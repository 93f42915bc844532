"""Inputs and drivers for num_alternative_paths above 4 (up to kMaxAlt = 32): a gene-family graph on which reads map to
many places, run through a C-ABI library (the host emulation or the sm_90a product library) and compared with the
oracle, node paths included."""
import ctypes

import numpy as np

import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import SIZE_MAX, cli_defaults

MAX_ALT = 32              # align_core.cuh kMaxAlt
K = 21

# seeders the gene-family input runs under: exact k-mer seeds, MEMs, and sub-k seeds (min_seed_length < k)
SEEDERS = {
    "exact": dict(min_seed_length=K, max_seed_length=K),
    "mem": dict(min_seed_length=K, max_seed_length=SIZE_MAX),
    "subk": dict(min_seed_length=15, max_seed_length=SIZE_MAX),
}


def gene_family(seed=11, copies=40, unit_len=400, flank=300, unique=5000, n_reads=60, L=150):
    """(graph sequences, reads): `copies` copies of one unit, each diverged by 2-6 % and set between unique flanks, plus
    unique random sequence; 150 bp reads from the copies, half with 2 % errors, a third reverse-complemented."""
    rng = np.random.default_rng(seed)
    unit = P._random_seq(rng, unit_len)
    seqs, placed = [], []
    for _ in range(copies):
        copy = P.mutate(rng, unit, float(rng.uniform(0.02, 0.06)))
        seqs.append(P._random_seq(rng, flank) + copy + P._random_seq(rng, flank))
        placed.append((len(seqs) - 1, flank, flank + len(copy)))
    seqs.append(P._random_seq(rng, unique))
    reads = []
    for i in range(n_reads):
        s, a, b = placed[int(rng.integers(0, len(placed)))]
        p = int(rng.integers(max(0, a - L // 3), b - 2 * L // 3))
        r = seqs[s][p:p + L]
        if i % 2:
            r = P.mutate(rng, r, 0.02)
        if i % 3 == 0:
            r = P.revcomp(r)
        reads.append(r)
    return seqs, reads


def config(n_alt, seeder="exact", rel_score_cutoff=None, **kw):
    if rel_score_cutoff is not None:
        kw["rel_score_cutoff"] = rel_score_cutoff
    return cli_defaults(K, num_alternative_paths=n_alt, min_exact_match=0.0, **SEEDERS[seeder], **kw)


_graphs = {}


def family_graph(seed=11):
    if seed not in _graphs:
        seqs, reads = gene_family(seed)
        _graphs[seed] = (seqs, reads, O.OracleGraph(K, seqs))
    return _graphs[seed]


def record_counts(lines):
    """alignments per read in format_alignment(..., with_nodes=True) lines: header, query, then six fields per alignment
    and one node list per alignment (an unaligned read has six placeholder fields and no node list)"""
    return [(len(line.split("\t")) - 2) // 7 for line in lines]


def family_case(lib, cfg, seed=11):
    """gene-family input under cfg: library lines == oracle lines. Returns (lines, run statistics)."""
    return family_lines(lib, cfg, family_graph(seed)[1], seed)


def agg_hits(lib):
    """host emulation only: (replacements, duplicates dropped) the aggregator counted (align_core.cuh EmuAgg)"""
    from metagraph_b200 import _lib
    h = (ctypes.c_ulonglong * 2).in_dll(_lib.load_library(lib), "mgb_emu_agg_hits")
    return {"replace": h[0], "duplicate": h[1]}


def fuzz_case(lib, i):
    """random_case on a graph of several diverged copies of one sequence, with num_alternative_paths drawn from 5..32 and
    the seeder, strands, cut-off, x-drop and node budget drawn too. Returns the configuration's num_alternative_paths."""
    rng = np.random.default_rng(7000 + i)
    n_alt = int(rng.integers(5, MAX_ALT + 1))
    k = int(rng.choice([11, 15, 21, 31]))
    seeder = [dict(min_seed_length=k, max_seed_length=k), dict(min_seed_length=k, max_seed_length=SIZE_MAX),
              dict(min_seed_length=max(8, k - 6), max_seed_length=SIZE_MAX)][int(rng.integers(0, 3))]
    cfg = cli_defaults(k, num_alternative_paths=n_alt, min_exact_match=float(rng.choice([0.0, 0.0, 0.5])),
                       rel_score_cutoff=float(rng.choice([0.0, 0.5, 0.8, 0.95])),
                       forward_and_reverse_complement=bool(rng.random() < 0.8), xdrop=int(rng.integers(15, 60)),
                       max_nodes_per_seq_char=float(rng.choice([5.0, 10.0])), **seeder)
    G, nseq = int(rng.integers(600, 3000)), int(rng.integers(3, 9))
    P.random_case(lib, 7000 + i, k, G, 25, int(rng.integers(60, 200)), float(rng.choice([0.0, 0.02, 0.05])), cfg,
                  bool(rng.random() < 0.3), nseq)
    return n_alt


def config_k(k, n_alt, **kw):
    return cli_defaults(k, num_alternative_paths=n_alt, min_exact_match=0.0, **kw)


def mode_case(lib, n_alt, mode, seed=11):
    """the gene-family input on a CANONICAL-mode graph (the sequences and their reverse complements) or a PRIMARY graph
    (one k-mer of every reverse-complement pair, CanonicalDBG semantics): lines == oracle. Returns the lines."""
    seqs, reads, _ = family_graph(seed)
    if mode == "canonical":
        seqs = seqs + [P.revcomp(s) for s in seqs]
    else:
        seqs = P.primary_contigs(seqs, K)
    g = O.OracleGraph(K, seqs, mask=False)
    g.set_mode(1 if mode == "canonical" else 2)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(K, W, last, F), lib=lib, mode=1 if mode == "canonical" else 2)
    cfg = config(n_alt, "exact", 0.0)
    try:
        got, _ = P.run_lines(idx, cfg, reads)
    finally:
        idx.close()
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (mode, bad[:3], exp[bad[0]][:400], got[bad[0]][:400])
    return got


def spill_reads(seed=11):
    """the gene-family reads plus ten 200 bp reads from the copies: a staging limit of 160 stages some reads on chip and
    leaves the others in global memory (the knob lq_split of parity_common.SPILL_KNOBS)"""
    seqs, reads, _ = family_graph(seed)
    rng = np.random.default_rng(seed + 1)
    extra = []
    for i in range(10):
        s = seqs[int(rng.integers(0, len(seqs) - 1))]
        p = int(rng.integers(200, len(s) - 400))
        extra.append(P.revcomp(s[p:p + 200]) if i % 2 else s[p:p + 200])
    return reads + extra


def family_lines(lib, cfg, reads, seed=11):
    seqs, _, g = family_graph(seed)
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(K, seqs, lib=lib), lib=lib)
    try:
        got, stats = P.run_lines(idx, cfg, reads)
    finally:
        idx.close()
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (cfg.num_alternative_paths, bad[:3], exp[bad[0]][:400], got[bad[0]][:400])
    return got, stats


def spill_knob_matrix(lib, monkeypatch, n_alt=32):
    """the gene-family input at n_alt under every knob of parity_common.SPILL_KNOBS: lines == oracle, DP counters ==
    the default run's. Returns {knob: statistics}."""
    reads = spill_reads()
    cfg = config(n_alt, "subk", 0.0)
    out = {}
    for knob, env in P.SPILL_KNOBS:
        with monkeypatch.context() as mp:
            for var, val in env.items():
                mp.setenv(var, "160" if val is None else val)
            _, out[knob] = family_lines(lib, cfg, reads)
        diff = {c: (out["default"][c], out[knob][c]) for c in P.DP_COUNTERS if out[knob][c] != out["default"][c]}
        assert not diff, (knob, diff)
    return out


def heap_retry_case(lib, mp, n_alt=32):
    """pass 0's output heap (MGB_TEST_HEAP0) holds the records of a few reads only: the reads with n_alt records that do
    not fit are aligned again in a retry pass. Lines == oracle and DP counters == a run without the limit."""
    _, reads, _ = family_graph()
    cfg = config(n_alt, "exact", 0.0)
    _, base = family_lines(lib, cfg, reads)
    mp.setenv("MGB_TEST_HEAP0", "200000")
    got, stats = family_lines(lib, cfg, reads)
    assert sum(c == n_alt for c in record_counts(got)) >= 40
    diff = {c: (base[c], stats[c]) for c in P.DP_COUNTERS if base[c] != stats[c]}
    assert not diff, diff
    return stats


def check_limits(lib):
    """N = 32 is served; N = 33 is refused with MGB_ERR_UNSUPPORTED and a message naming the limit, by mgb_config_check
    (the aligner's constructor) and by mgb_align_batch"""
    import pytest
    from metagraph_b200 import _lib
    from metagraph_b200.aligner import B200Aligner
    seqs, reads, _ = family_graph()
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(K, seqs, lib=lib), lib=lib)
    try:
        al = B200Aligner(idx, config(MAX_ALT, "exact", 0.0))
        assert max(len(r) for r in al.align_batch([("", r) for r in reads[:8]])) == MAX_ALT
        with pytest.raises(_lib.MgbError, match=r"num_alternative_paths must be in \[1, 32\]") as e:
            B200Aligner(idx, config(MAX_ALT + 1))
        assert e.value.code == -4                                  # MGB_ERR_UNSUPPORTED
        al.config.num_alternative_paths = MAX_ALT + 1             # past the constructor: mgb_align_batch checks again
        with pytest.raises(_lib.MgbError, match=r"num_alternative_paths must be in \[1, 32\]") as e:
            al.align_batch([("", reads[0])])
        assert e.value.code == -4
    finally:
        idx.close()


def check_limits_shim(tmp_path, link_flags):
    """tests/cpp/test_alt_paths_shim.cpp: the C++ shim serves N = 32 and throws at construction for N = 33"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_alt_paths_shim")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(root, "tests", "cpp", "test_alt_paths_shim.cpp"),
                           "-o", exe] + link_flags)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "n32\t32" in out.stdout and "n33\tnum_alternative_paths must be in [1, 32]" in out.stdout, out.stdout


SHARD_WORKER = r'''
import os, sys
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch.distributed as dist
import alt_paths_common as A
import parity_common as P
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
from metagraph_b200.sharding import align_sharded
dist.init_process_group("gloo")
rank = dist.get_rank()
seqs, reads, g = A.family_graph()
batch = [("r%d" % i, r) for i, r in enumerate(reads)]
idx = DBGSuccinctIndex(BOSSTable.from_sequences(A.K, seqs, lib=LIB), lib=LIB)
cfg = A.config(8, "exact", 0.0)
fmt = lambda h, r: format_alignment(h, r, cfg.min_path_score, with_nodes=True)
lines = align_sharded(B200Aligner(idx, cfg), batch, fmt)
if rank == 0:
    single, _ = P.run_lines(idx, cfg, reads, [h for h, _ in batch])
    assert lines == single, (len(lines), len(single))
    assert lines == g.align_tsv(cfg, reads, headers=[h for h, _ in batch], with_nodes=True)
    counts = A.record_counts(lines)
    assert max(counts[:30]) == 8 and max(counts[30:]) == 8, counts
    print("SHARDING_OK", len(lines), sum(c == 8 for c in counts))
else:
    assert lines is None
dist.destroy_process_group()
'''


def check_sharding(tmp_path, lib, port=29523):
    """two gloo ranks align halves of the gene-family batch with N = 8 and gather on rank 0 (mgb_results_export /
    mgb_results_import): the gathered lines equal a single-rank run and the oracle"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "worker.py"
    script.write_text("ROOT = %r\nLIB = %r\n" % (root, lib) + SHARD_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                         capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert "SHARDING_OK 60" in out.stdout, out.stdout[-2000:]
