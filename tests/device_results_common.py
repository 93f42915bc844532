"""Case driver of the device-resident route (mgb_align_batch_device, B200Aligner.align_tensors): the same reads go
through mgb_align_batch, and every column of the device route must equal the record route's mgb_alignment_t fields,
sequence, CIGAR and node bytes, per-read ranges and search counters. `device` is "cpu" under the host-emulation
library (its "device" memory is host memory) and "cuda:0" on the GPU."""
import ctypes
import dataclasses
import os

import numpy as np
import torch

import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, _pack
from metagraph_b200.config import cli_defaults

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EX = os.path.join(ROOT, "tests", "golden", "example_graphs")
COUNTERS = ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns", "num_reads_retried")
FIELDS = ("read_index", "orientation", "score", "offset", "query_begin", "query_len", "num_nodes", "sequence_len",
          "num_cigar_ops")


def records(al, reads):
    """mgb_align_batch's records as columns (numpy), and its stats"""
    L = al._L
    buf, offs = _pack(reads)
    res = al.align_batch_raw(buf, offs)
    try:
        n = L.mgb_results_num_alignments(res)
        alns = L.mgb_results_alignments(res)
        first, count = ctypes.c_uint64(), ctypes.c_uint32()
        read_first = [0]
        for r in range(len(reads)):
            L.mgb_results_read_range(res, r, ctypes.byref(first), ctypes.byref(count))
            assert first.value == read_first[-1]
            read_first.append(first.value + count.value)
        cols = {f: np.array([getattr(alns[i], f) for i in range(n)], dtype=np.int64) for f in FIELDS}
        seq, cig, nodes = [], [], []
        for i in range(n):
            x = alns[i]
            seq.append(ctypes.string_at(x.sequence, x.sequence_len))
            cig.append(np.ctypeslib.as_array(x.cigar, shape=(x.num_cigar_ops,)).astype(np.int64) if x.num_cigar_ops
                       else np.zeros(0, np.int64))
            nodes.append(np.ctypeslib.as_array(x.nodes, shape=(x.num_nodes,)).astype(np.uint64)
                         if x.num_nodes and x.nodes else np.zeros(0, np.uint64))
        stats = al.stats_of(res)
    finally:
        al.free_raw(res)
    return np.array(read_first, np.int64), cols, seq, cig, nodes, stats


def as_tensors(reads, device, offsets_on_device=False, odd_start=False):
    """reads packed into a uint8 tensor on `device` and int64 offsets. odd_start: the reads are a slice of a larger
    tensor that starts at an odd byte and ends exactly at the tensor's end."""
    buf, offs = _pack(reads)
    pad = 7 if odd_start else 0
    whole = torch.zeros(pad + len(buf), dtype=torch.uint8)
    whole[pad:] = torch.from_numpy(buf.copy())
    whole = whole.to(device)
    t = whole[pad:]
    o = torch.from_numpy(offs.astype(np.int64))
    return t, o.to(device) if offsets_on_device else o


def check(idx, cfg, reads, device, offsets_on_device=False, odd_start=False, counters=COUNTERS):
    """align_tensors against mgb_align_batch on the same reads (and the search counters named in `counters`); returns
    the device route's stats"""
    reads = [r.encode("latin1") if isinstance(r, str) else bytes(r) for r in reads]
    al = B200Aligner(idx, cfg)
    read_first, cols, seq, cig, nodes, st = records(al, reads)
    t, o = as_tensors(reads, device, offsets_on_device, odd_start)
    got = al.align_tensors(t, o)
    g = {f.name: getattr(got, f.name) for f in dataclasses.fields(got) if f.name != "stats"}
    for v in g.values():
        assert v.device == torch.device(device)
    g = {k: v.cpu().numpy() for k, v in g.items()}
    assert g["read_first"].tolist() == read_first.tolist()
    n = int(read_first[-1])
    for f in FIELDS:
        exp = cols[f]
        if f != "orientation":
            exp = exp.astype(np.int64)
        assert g[f].astype(np.int64).tolist() == exp.tolist(), f
    assert g["sequence_offsets"].tolist() == np.concatenate([[0], np.cumsum([len(s) for s in seq])]).astype(np.int64).tolist()
    assert g["sequence"].tobytes() == b"".join(seq)
    assert g["cigar_offsets"].tolist() == np.concatenate([[0], np.cumsum([len(c) for c in cig])]).astype(np.int64).tolist()
    assert (g["cigar"].astype(np.int64) & 0xffffffff).tolist() == (np.concatenate(cig + [np.zeros(0, np.int64)])).tolist()
    nodes_on = not cfg.result_nodes
    exp_nodes = np.concatenate(nodes + [np.zeros(0, np.uint64)]) if nodes_on else np.zeros(0, np.uint64)
    assert g["nodes"].view(np.uint64).tolist() == exp_nodes.tolist()
    n_off = np.concatenate([[0], np.cumsum([len(x) if nodes_on else 0 for x in nodes])]).astype(np.int64)
    assert g["node_offsets"].tolist() == n_off.tolist()
    assert len(g["read_index"]) == n
    diff = {c: (st[c], got.stats[c]) for c in counters if st[c] != got.stats[c]}
    assert not diff, diff
    return got.stats


# ------------------------------------------------------------------------------------------------ inputs ----
def read_fasta(path):
    seqs, cur = [], None
    for line in open(path):
        line = line.strip()
        if line.startswith(">"):
            if cur is not None:
                seqs.append(cur)
            cur = ""
        elif cur is not None:
            cur += line
    if cur is not None:
        seqs.append(cur)
    return seqs


def example_case(lib, device, protein):
    """an example graph (.dbg) with its query reads, the example sequences' windows, and short and empty reads"""
    name = "Protein" if protein else "DNA"
    boss = BOSSTable.from_dbg(os.path.join(EX, "test_%s_graph.dbg" % name), lib=lib)
    idx = DBGSuccinctIndex(boss, lib=lib)
    reads = read_fasta(os.path.join(EX, "test_%s_query.fa" % name))
    reads += [s[i:i + 120] for s in read_fasta(os.path.join(EX, "test_%s_sequences.fa" % name))[:20] for i in (0, 37)]
    reads += ["", "A", reads[0][:boss.k - 1]]
    try:
        for n_alt in (1, 4):
            check(idx, cli_defaults(boss.k, alphabet="protein" if protein else "dna", min_exact_match=0.0,
                                    num_alternative_paths=n_alt), reads, device)
    finally:
        idx.close()


def c1_case(lib, device, n_transcripts=120, max_len=1500, seed=7, k=12):
    """parity_common.c1_case's transcripts: the graph and the transcripts themselves as reads"""
    rng = np.random.default_rng(seed)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, max_len)])
    seqs = []
    for i in range(n_transcripts):
        L = 59 if i == 0 else (max_len if i == 1 else int(np.exp(rng.uniform(np.log(59), np.log(max_len)))))
        p = int(rng.integers(0, max_len - L + 1))
        t = base[p:p + L] if i % 3 else "".join(np.array(list("ACGT"))[rng.integers(0, 4, L)])
        seqs.append(P.mutate(rng, t, 0.01) if i % 3 == 1 else t)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    try:
        return check(idx, cli_defaults(k), seqs, device)
    finally:
        idx.close()


def mode_index(lib, seed, k, mode, G=3000, nreads=60, L=120, rate=0.03):
    """a BASIC (0), CANONICAL (1) or PRIMARY (2) graph over related sequences, and reads from them with errors, short
    and empty ones"""
    rng = np.random.default_rng(seed)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])
    seqs = [base, P.mutate(rng, base, 0.03)]
    src = seqs
    if mode == 1:
        seqs = seqs + [P.revcomp(s) for s in seqs]
    elif mode == 2:
        seqs = P.primary_contigs(seqs, k)
    g = O.OracleGraph(k, seqs)
    if mode:
        g.set_mode(mode)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), lib=lib, mode=mode)
    reads = []
    for i in range(nreads):
        s = src[int(rng.integers(0, len(src)))]
        p = int(rng.integers(0, len(s) - L))
        r = P.mutate(rng, s[p:p + int(rng.integers(k, L))], rate if i % 4 else 0.0)
        reads.append(P.revcomp(r) if i % 2 else r)
    reads += ["", "A", "ACGT" * 3, "N" * 40, base[:k - 1]]
    return idx, reads


def mode_case(lib, device, seed, mode, n_alt, nodes, both=True, **kw):
    k = 15 + seed
    idx, reads = mode_index(lib, seed, k, mode)
    try:
        cfg = cli_defaults(k, num_alternative_paths=n_alt, forward_and_reverse_complement=both,
                           result_nodes=nodes, min_exact_match=0.0)
        return check(idx, cfg, reads, device, **kw)
    finally:
        idx.close()


def _pcie_passes(st, n, offsets_on_device):
    """checks the PCIe bytes of a batch of n reads in which no read is answered before pass 0 against their formula;
    returns the number of align passes"""
    retried = st["num_reads_retried"]
    # up: offsets and k-mer offsets (upload_batch), pass 0's list of every read, then each retry list
    assert st["h2d_bytes"] == 16 * (n + 1) + 4 * n + 4 * retried
    # down: the device offsets, a 48-byte summary per pass, each retry list, the 32 bytes of totals
    rest = st["d2h_bytes"] - 32 - 4 * retried - (8 * (n + 1) if offsets_on_device else 0)
    assert rest % 48 == 0
    return rest // 48


def retry_case(lib, device, offsets_on_device=False):
    """parity_common's "retry" pressure input: about half its reads explore more columns than their arena holds at scale
    1 and are aligned again on a retry pass, whose list comes from k_pass_classify. Whether a read overflows its own
    arena does not depend on the other reads, so the retry count equals the record route's. No read is answered before
    pass 0 (min_seed_length < k), so every pass uploads its list. Returns (stats, passes)."""
    k, seqs, reads, cfg = P.pressure_input("retry")
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    try:
        st = check(idx, cfg, reads, device, offsets_on_device=offsets_on_device)
    finally:
        idx.close()
    assert st["num_reads_retried"] > 0
    passes = _pcie_passes(st, len(reads), offsets_on_device)
    assert passes >= 2
    return st, passes


def heap_retry_case(lib, device, monkeypatch, offsets_on_device=False):
    """pass 0's output heap (MGB_TEST_HEAP0) holds a few reads only, so most reads are answered by retry passes. The
    heap is shared: on the device, which reads find it full depends on the order in which their warps take space, so
    the retry count may differ from run to run and from the record route's. The columns and the DP counters may not.
    Forward strand only, so that no read is answered before pass 0. Returns (stats, passes)."""
    monkeypatch.setenv("MGB_TEST_HEAP0", "6000")
    idx, reads = mode_index(lib, 3, 19, 0, nreads=80)
    try:
        cfg = cli_defaults(19, num_alternative_paths=4, min_exact_match=0.0, forward_and_reverse_complement=False)
        st = check(idx, cfg, reads, device, offsets_on_device=offsets_on_device, counters=COUNTERS[:-1])
    finally:
        idx.close()
    assert st["num_reads_retried"] > 0
    passes = _pcie_passes(st, len(reads), offsets_on_device)
    assert passes >= 2
    return st, passes
