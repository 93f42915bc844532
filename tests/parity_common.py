"""Shared parity drivers: run the same inputs through the oracle and through a C-ABI library
(the sm_90a product library on a GPU, or the host-emulation build of the same kernel sources
on a CPU-only machine) and demand identical TSV lines + node paths."""
import json
import os

import numpy as np

import oracle_lib as O
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
from metagraph_b200.config import SIZE_MAX, cli_defaults, dna_scoring_matrix, struct_defaults
from test_oracle_golden import GOLD, make_cfg, read_fasta, read_fastq, revcomp

COMP = str.maketrans("ACGT", "TGCA")


def mutate(rng, r, rate):
    out = []
    for c in r:
        if rng.random() < rate:
            y = rng.random()
            if y < 0.8:
                out.append("ACGT"[int(rng.integers(0, 4))])
            elif y < 0.9:
                out.append(c); out.append("ACGT"[int(rng.integers(0, 4))])
        else:
            out.append(c)
    return "".join(out)


def run_lines(idx, cfg, reads, headers=None):
    headers = headers or [""] * len(reads)
    al = B200Aligner(idx, cfg)
    res = al.align_batch(list(zip(headers, reads)))
    return [format_alignment(h, r, cfg.min_path_score, with_nodes=True) for h, r in zip(headers, res)], al.last_stats


def check_goldens(lib):
    G = json.load(open(os.path.join(GOLD, "test_aligner_goldens.json")))
    for gold in G:
        g = O.OracleGraph(gold["k"], gold["refs"], mask=gold["mask"], dynamic=not gold["mask"])
        W, last, F, valid = g.arrays()
        idx = DBGSuccinctIndex(BOSSTable(gold["k"], W, last, F), valid=valid if gold["mask"] else None, lib=lib)
        query = revcomp(gold["query"]) if gold["rc_query"] else gold["query"]
        for uni in ([False, True] if gold["extend"] else [False]):
            cfg = make_cfg(gold["cfg"])
            if uni:
                cfg.max_seed_length = SIZE_MAX
            exp = g.align_tsv(cfg, [query], with_nodes=True)
            got, _ = run_lines(idx, cfg, [query])
            assert got == exp, (gold["name"], uni, exp, got)
        idx.close()


def check_mt(lib, both):
    _, seqs = read_fasta(os.path.join(GOLD, "genome.MT.fa"))
    names, reads = read_fastq(os.path.join(GOLD, "genome_MT1.fq"))
    boss = BOSSTable.from_sequences(11, seqs, lib=lib)
    g = O.OracleGraph(11, seqs, mask=False)
    W, last, F, _ = g.arrays()
    assert (boss.W == W).all() and (boss.last == last).all() and (boss.F == F).all()
    idx = DBGSuccinctIndex(boss, lib=lib)
    cfg = cli_defaults(11, min_exact_match=0.0, forward_and_reverse_complement=both)
    got, _ = run_lines(idx, cfg, reads, names)
    exp = g.align_tsv(cfg, reads, headers=names, with_nodes=True)
    assert got == exp
    return got


def random_case(lib, seed, k, G, nreads, L, rate, cfg, mask=False, nseq=1, oracle_stats=None):
    rng = np.random.default_rng(seed)
    seqs = ["".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])]
    seqs += [mutate(rng, seqs[0], 0.02) for _ in range(nseq - 1)]
    g = O.OracleGraph(k, seqs, mask=mask)
    W, last, F, valid = g.arrays()
    boss = BOSSTable.from_sequences(k, seqs, lib=lib)
    assert (boss.W == W).all() and (boss.last == last).all() and (boss.F == F).all()
    if mask:
        assert (boss.dummy_mask(lib=lib) == valid).all()
    idx = DBGSuccinctIndex(boss, valid=valid if mask else None, lib=lib)
    reads = []
    for i in range(nreads):
        s = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, max(1, len(s) - L)))
        r = mutate(rng, s[p:p + L], rate)
        if rng.random() < 0.5:
            r = r.translate(COMP)[::-1]
        if rng.random() < 0.05 and len(r) > 2:
            r = r[:len(r) // 2] + "N" + r[len(r) // 2 + 1:]
        reads.append(r)
    reads += ["", "A", "ACGT" * 3, "N" * 40]          # empty / shorter than k / all-invalid
    exp = g.align_tsv(cfg, reads, with_nodes=True, stats=oracle_stats)
    got, stats = run_lines(idx, cfg, reads)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (seed, bad[:3], exp[bad[0]], got[bad[0]])
    # map_to_nodes parity
    nodes = idx.map_to_nodes_sequentially(reads)
    for r, n in zip(reads, nodes):
        assert list(n) == list(g.map_to_nodes(r)), r
    idx.close()
    return stats


def whole_read_hits(lib):
    """test counter of the host-emulation build (None for the product library)"""
    import ctypes
    from metagraph_b200 import _lib
    L = _lib.load_library(lib)
    try:
        return ctypes.c_ulonglong.in_dll(L, "mgb_emu_whole_read_hits").value
    except ValueError:
        return None


# the aligner's spill / migration sites the host-emulation build counts (align_core.cuh EmuPath, same order)
EMU_PATHS = ("queue_migrate", "nn_migrate", "column_migrate", "arena_column", "unstaged_read", "general_column",
             "read_overflow", "ram_stop_general", "nodes_stop_general", "ram_stop_chain", "nodes_stop_chain", "conv_move")


def path_hits(lib):
    """test counters of the host-emulation build by path name (None for the product library)"""
    import ctypes
    from metagraph_b200 import _lib
    L = _lib.load_library(lib)
    try:
        hits = (ctypes.c_ulonglong * len(EMU_PATHS)).in_dll(L, "mgb_emu_path_hits")
    except ValueError:
        return None
    return dict(zip(EMU_PATHS, hits))


def exact_shortcut_case(lib, seed, k, cfg, nseq=3, G=3000, nreads=80, L=90):
    """Reads that match a path of the graph exactly (the exact-path shortcut of the extender applies to them) on a
    graph with variants and a tandem repeat, mixed with reads carrying errors; kernels (shortcut on) == oracle, and
    the shortcut switched off gives the same lines."""
    import dataclasses
    rng = np.random.default_rng(seed)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])
    unit = "".join(np.array(list("ACGT"))[rng.integers(0, 4, 7)])
    base = base[:G // 2] + unit * 12 + base[G // 2:]                 # a tandem repeat: nodes met more than once
    seqs = [base] + [mutate(rng, base, 0.01) for _ in range(nseq - 1)]
    g = O.OracleGraph(k, seqs)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    reads = []
    for i in range(nreads):
        sq = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, len(sq) - L))
        r = sq[p:p + L] if i % 4 else mutate(rng, sq[p:p + L], 0.03)
        reads.append(r.translate(COMP)[::-1] if i % 3 == 0 else r)
    reads.append(base[G // 2 - 20:G // 2 + 60])                      # runs into the repeat
    reads.append("ACGT" * (L // 4))
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    hits0 = whole_read_hits(lib)
    got, _ = run_lines(idx, cfg, reads)
    hits1 = whole_read_hits(lib)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (seed, bad[:3], exp[bad[0]], got[bad[0]])
    got2, _ = run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=True), reads)
    assert got2 == got
    if hits0 is not None:
        # host emulation: the whole-read form of the shortcut (exact seeder, both strands) answered reads in the first
        # run exactly when the configuration allows it, and none with the shortcut switched off
        exact = cfg.min_seed_length == k and cfg.max_seed_length == k and cfg.forward_and_reverse_complement
        assert (hits1 - hits0 >= nreads // 3) if exact else (hits1 == hits0), (hits0, hits1, exact)
        assert whole_read_hits(lib) == hits1
    full = sum(1 for r, l in zip(reads, got) if ("\t%d=\t" % len(r)) in l)
    assert full >= nreads // 2
    idx.close()


EXACT_SHORTCUT_CASES = [
    (101, 21, lambda k: cli_defaults(k)),                                           # MEM + sub-k seeds
    (102, 21, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k)),     # exact seeds (bench config)
    (103, 12, lambda k: cli_defaults(k, min_exact_match=0.0, left_end_bonus=0, right_end_bonus=0)),
    (104, 15, lambda k: cli_defaults(k, right_end_bonus=9)),                        # right bonus above match + left: no shortcut
    (105, 17, lambda k: cli_defaults(k, forward_and_reverse_complement=False)),
    (106, 13, lambda k: struct_defaults(xdrop=20, min_seed_length=k, max_seed_length=k)),
    (107, 19, lambda k: cli_defaults(k, num_alternative_paths=2)),                  # two reported paths: no shortcut
]

def whole_read_case(lib, seed, k, cfg, G=2500, L=70, n_path=40):
    """Reads around the whole-read form of the exact-path shortcut (exact seeder, both strands): reads that are paths
    of the graph on either strand, reads whose other strand has k-mers in the graph as well (the graph holds a region
    and its reverse complement; palindromes), reads of length k and k - 1, reads with an 'N' or one wrong base, a read
    that leaves the graph at its last base. Kernels == oracle, shortcut on and off."""
    import dataclasses
    rng = np.random.default_rng(seed)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])
    region = base[300:300 + 3 * L]
    pal = "".join(np.array(list("ACGT"))[rng.integers(0, 4, L // 2)])
    pal = pal + pal.translate(COMP)[::-1]                              # its own reverse complement
    seqs = [base, region.translate(COMP)[::-1], pal + base[:40]]
    g = O.OracleGraph(k, seqs)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    reads = []
    for i in range(n_path):
        p = int(rng.integers(0, G - L))
        r = base[p:p + L]
        reads.append(r.translate(COMP)[::-1] if i % 2 else r)
    for off in (0, 7, L, 2 * L - 3):                                   # both strands are paths of the graph
        reads.append(region[off:off + L]); reads.append(region[off:off + L].translate(COMP)[::-1])
    reads.append(base[290:290 + L])                                    # runs into the doubled region: other strand matches in part
    reads.append(base[300 + 3 * L - 20:300 + 3 * L - 20 + L])
    reads.append(pal); reads.append(pal[3:] + base[:3])
    for n in (k - 1, k, k + 1, 2 * k):
        reads.append(base[1000:1000 + n]); reads.append(base[1200:1200 + n].translate(COMP)[::-1])
    r = base[1500:1500 + L]
    reads.append(r[:30] + "N" + r[31:]); reads.append(r[:L - 1] + ("A" if r[L - 1] != "A" else "C"))
    reads.append(("T" if r[0] != "T" else "G") + r[1:]); reads.append(r[:k + 3] + ("A" if r[k + 3] != "A" else "C") + r[k + 4:])
    reads.append(base[G - L:] ); reads.append(base[G - L + 1:] + "A")
    reads.append("acgt" + base[2000:2000 + L - 4].lower())            # lower case input
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    hits0 = whole_read_hits(lib)
    got, _ = run_lines(idx, cfg, reads)
    hits = None if hits0 is None else whole_read_hits(lib) - hits0
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (seed, bad[:5], reads[bad[0]], exp[bad[0]], got[bad[0]])
    got2, _ = run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=True), reads)
    assert got2 == got
    idx.close()
    return hits


WHOLE_READ_CASES = [
    # (seed, k, config, whether the whole-read form may answer reads at all)
    (201, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k), True),
    (202, 21, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, rel_score_cutoff=0.0), True),
    (203, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, min_path_score=151), False),   # above 2 * L + 10
    (204, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, min_path_score=100), True),    # some reads pass
    (205, 17, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, seed_complexity_filter=True), False),
    (206, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, min_exact_match=1.0), True),
    (207, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, min_cell_score=120), True),    # forward min path score
    (208, 13, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, left_end_bonus=0, right_end_bonus=0,
                                     min_exact_match=0.0), True),
    (209, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, forward_and_reverse_complement=False), False),
    (210, 15, lambda k: cli_defaults(k, min_seed_length=k, max_seed_length=k, max_num_seeds_per_locus=1), True),
]


def nodeless_case(lib, seed=5, k=15, G=4000, nreads=60, L=80):
    """mgb_config_t::result_nodes = MGB_NODES_NONE: the same alignments (TSV fields identical to the oracle's),
    node arrays left on the device (nodes == NULL, num_nodes kept)."""
    import dataclasses
    rng = np.random.default_rng(seed)
    seqs = ["".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])]
    g = O.OracleGraph(k, seqs)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    reads = []
    for i in range(nreads):
        p = int(rng.integers(0, G - L))
        r = mutate(rng, seqs[0][p:p + L], 0.04)
        reads.append(r.translate(COMP)[::-1] if i % 2 else r)
    cfg = cli_defaults(k, min_exact_match=0.0)
    exp = g.align_tsv(cfg, reads)
    full = B200Aligner(idx, cfg).align_batch([("", r) for r in reads])
    slim = B200Aligner(idx, dataclasses.replace(cfg, result_nodes=1)).align_batch([("", r) for r in reads])
    n_aln = 0
    for r, e, a, b in zip(reads, exp, full, slim):
        assert format_alignment("", b, cfg.min_path_score) == e
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert len(y.nodes) == 0 and len(x.nodes) > 0
            n_aln += 1
    assert n_aln > nreads // 2
    idx.close()


def c1_case(lib, n_transcripts, max_len, seed=7, k=12):
    """BASELINE configs[0] shape (k=12 graph of transcripts, the transcripts themselves as reads, CLI
    defaults, ragged lengths from 59 bp up to max_len) on synthetic transcripts: related sequences
    (shared segments) so the graph branches. Returns (#reads, #reads aligned end to end)."""
    rng = np.random.default_rng(seed)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, max_len)])
    seqs = []
    for i in range(n_transcripts):
        L = 59 if i == 0 else (max_len if i == 1 else int(np.exp(rng.uniform(np.log(59), np.log(max_len)))))
        p = int(rng.integers(0, max_len - L + 1))
        t = base[p:p + L] if i % 3 else "".join(np.array(list("ACGT"))[rng.integers(0, 4, L)])
        seqs.append(mutate(rng, t, 0.01) if i % 3 == 1 else t)
    g = O.OracleGraph(k, seqs)
    boss = BOSSTable.from_sequences(k, seqs, lib=lib)
    W, last, F, _ = g.arrays()
    assert (boss.W == W).all() and (boss.last == last).all() and (boss.F == F).all()
    idx = DBGSuccinctIndex(boss, lib=lib)
    cfg = cli_defaults(k)
    exp = g.align_tsv(cfg, seqs, with_nodes=True, threads=8)
    got, _ = run_lines(idx, cfg, seqs)
    bad = [i for i in range(len(seqs)) if exp[i] != got[i]]
    assert not bad, (bad[:3], len(seqs[bad[0]]), exp[bad[0]][:300], got[bad[0]][:300])
    full = sum(1 for s_, l in zip(seqs, got) if l.split("\t")[6] == "%d=" % len(s_))
    idx.close()
    return len(seqs), full


def lowcx_genome(rng, n):
    """random sequence interleaved with homopolymers, di-/tri-nucleotide repeats and the odd N"""
    out = []
    while sum(len(x) for x in out) < n:
        y = rng.random()
        if y < 0.5:
            out.append("".join(np.array(list("ACGT"))[rng.integers(0, 4, int(rng.integers(20, 120)))]))
        elif y < 0.65:
            out.append("ACGT"[int(rng.integers(0, 4))] * int(rng.integers(5, 40)))
        elif y < 0.85:
            u = "".join(np.array(list("ACGT"))[rng.integers(0, 4, int(rng.integers(2, 5)))])
            out.append(u * int(rng.integers(3, 15)))
        else:
            out.append("".join(np.array(list("ACGT"))[rng.integers(0, 4, 12)]))
    return "".join(out)[:n]


def lowcx_case(lib, seed, k, exact):
    rng = np.random.default_rng(seed)
    seqs = [lowcx_genome(rng, 6000), lowcx_genome(rng, 3000)]
    g = O.OracleGraph(k, seqs)
    boss = BOSSTable.from_sequences(k, seqs, lib=lib)
    idx = DBGSuccinctIndex(boss, lib=lib)
    kw = dict(min_exact_match=0.0, seed_complexity_filter=True)
    if exact:
        kw.update(min_seed_length=k, max_seed_length=k)
    cfg = cli_defaults(k, **kw)
    reads = []
    for i in range(60):
        s_ = seqs[i % 2]
        p = int(rng.integers(0, len(s_) - 150))
        r = mutate(rng, s_[p:p + 150], 0.03)
        if i % 3 == 0:
            r = r.translate(COMP)[::-1]
        if i % 11 == 5:
            r = r[:70] + "N" + r[71:]
        reads.append(r)
    reads += ["A" * 150, "CA" * 60, "ACG" * 40, "", "AC"]
    exp_on = g.align_tsv(cfg, reads, with_nodes=True)
    got, _ = run_lines(idx, cfg, reads)
    bad = [i for i in range(len(reads)) if exp_on[i] != got[i]]
    assert not bad, (seed, bad[:3], exp_on[bad[0]][:200], got[bad[0]][:200])
    cfg.seed_complexity_filter = False
    exp_off = g.align_tsv(cfg, reads, with_nodes=True)
    idx.close()
    return sum(a != b for a, b in zip(exp_on, exp_off))      # reads whose result the filter changes


def concurrent_case(lib):
    """cli/align.cpp:440-475 runs align_batch from several worker threads on one shared graph: mgb_align_batch
    must be re-entrant (per-call workspaces, thread-local error state)."""
    import threading
    rng = np.random.default_rng(3)
    genome = "".join(np.array(list("ACGT"))[rng.integers(0, 4, 8000)])
    k = 21
    g = O.OracleGraph(k, [genome])
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, [genome], lib=lib), lib=lib)
    cfg = cli_defaults(k, min_exact_match=0.0)
    batches = []
    for t in range(6):
        reads = []
        for i in range(25):
            p = int(rng.integers(0, len(genome) - 120))
            r = mutate(rng, genome[p:p + 120], 0.04)
            reads.append(r.translate(COMP)[::-1] if i % 2 else r)
        batches.append(reads)
    exp = [g.align_tsv(cfg, b) for b in batches]
    got = [None] * len(batches)

    def work(t):
        al = B200Aligner(idx, cfg)
        got[t] = [format_alignment("", r, cfg.min_path_score) for r in al.align_batch([("", x) for x in batches[t]])]

    threads = [threading.Thread(target=work, args=(t,)) for t in range(len(batches))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert got == exp
    idx.close()



def primary_contigs(seqs, k):
    """Stand-in for `metagraph build --mode primary` (primary contigs of the canonical graph): one k-mer of every
    reverse-complement pair, emitted as maximal runs of consecutive k-mers not seen before on either strand.
    Which strand of a pair is kept depends on the reference's traversal order; alignments do not depend on it
    beyond node ids and tie order."""
    seen, out = set(), []
    for s in seqs:
        start = None
        for i in range(len(s) - k + 1):
            km = s[i:i + k]
            key = min(km, revcomp(km))
            if key in seen:
                if start is not None:
                    out.append(s[start:i + k - 1])
                    start = None
            else:
                seen.add(key)
                if start is None:
                    start = i
        if start is not None:
            out.append(s[start:])
    return out


# Known-answer tests of the reference's unit tests for the strand modes (tests/graph/test_aligner.cpp). Every entry:
# (name, k, graph sequences, mode, masked batch construction or dynamic add_sequence, config, query, check(fields)).
def mode_kats():
    from metagraph_b200.config import INT32_MIN
    lo = INT32_MIN + 100
    ref, query = "AAAAACTTTCGAGGCCAA", "GGGGGCTTTCGAGGCCAA"
    ref_rc = revcomp(ref)
    snp = dict(max_num_seeds_per_locus=SIZE_MAX, min_cell_score=lo, min_path_score=lo, min_seed_length=13)

    def check_snp(f):                                  # :1483-1539 align_suffix_seed_snp_canonical
        assert len(f) == 6
        strand, seq, score, _, cigar, off = f
        assert off == "5"
        assert (seq, cigar) in ((ref[5:], "5S13="), (ref_rc[:13], "13=5S"))
        assert int(score) == 26

    ref2, query2 = "AAAAGCTTTCGAGGCCAA", "AAAAGTTTTCGAGGCCAA"

    def check_both(f):                                 # :1541-1577 align_both_directions
        assert len(f) == 6
        strand, seq, score, _, cigar, off = f
        assert off == "0" and (seq, cigar) in ((ref2, "5=1X12="), (revcomp(ref2), "12=1X5="))
        assert int(score) == 2 * 17 - 1

    ref3 = "CTGCTGCGCCATCGCAACCCACGGTTGCTTTTTGAGTCGCTGCTCACGTTAGCCATCACACTGACGTTAAGCTGGCTTTCGATGCTGTATC"
    query3 = ("CTTACTGCTGCGCTCTTCGCAAACCCCACGGTTTCTTGTTTTGAGCTCGCCTGCTCACGATACCCATACACACTGACGTTCAAGCTGGCTTTCGATGTTGTATC")

    def one_path(f):                                   # :1773-1800 align_suffix_seed_no_full_seeds
        assert len(f) == 6

    _, transcripts = read_fasta(os.path.join(GOLD, "transcripts_100.fa"))
    query4 = ("TCGATCGATCGATCGATCGATCGACGATCGATCGATCGATCGATCGACGATCGAT"
              "CGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGA"
              "TCGATCGATCGATCGACGATCGATCGATCGATCGATCGACGATCGATCGATCGAT"
              "CGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGA"
              "TCGATCGACGATCGATCGATCGATCGATCGACGATCGATCGATCGATCGATCGAT"
              "CGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGA"
              "CGATCGATCGATCGATCGATCGACGATCGATCGATCGATCGATCGATCGATCGAT"
              "CGATCGATCGATCGATCGATCGA")

    def three_paths(f):                                # :1600-1631 align_low_similarity4_rep_primary
        assert len(f) == 18

    rep = dict(score_matrix=dna_scoring_matrix(2, -3, -3), gap_opening_penalty=-5, gap_extension_penalty=-2, xdrop=27,
               min_exact_match=0.0, max_nodes_per_seq_char=10.0, num_alternative_paths=3)
    # BASIC-mode tests of the same file that need the transcripts fixture or the complexity filter
    ref5 = "AGCTTCGAGGCCAA"

    def check_straight(f):                             # :338-381 align_straight_forward_and_reverse_complement_batch
        assert f == ["-", ref5, "28", "14", "14=", "0"]

    ref6 = ("AAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAGTGCTGGGATTATAGGTGTGAACCACCACACCTGGCTAATTTTTTTTGTGTGTGTGTGTGTTTTTTC")
    query6 = ("AAAAAAAAAAAAAAAAAAAAAAAAAAACGCCAAAAAGGGGGAATAGGGGGGGGGGAACCCCAACACCGGTATGTTTTTTTGTGTGTGGGGGATTTTTTTC")
    sim3 = dict(score_matrix=dna_scoring_matrix(2, -3, -3))

    def non_empty(f):                                  # :1345-1363 align_low_similarity3
        assert len(f) >= 6

    def empty(f):
        assert f == []

    match4 = ("TCGATCAATCGATCAATCGATCAACGATCAATCGATCAATCGATCAACGATCAAT"
              "CGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAA"
              "TCGATCAATCGATCAACGATCAATCGATCAATCGATCAACGATCAATCGATCAAT"
              "CGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAA"
              "TCGATCAACGATCAATCGATCAATCGATCAACGATCAATCGATCAATCGATCAAT"
              "CGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAATCGATCAA"
              "CGATCAATCGATCAATCGATCAACGATCAATCGATCAATCGATCAATCGATCAAT"
              "CGATCAATCGATCAATCGATC")

    def two_paths(f):                                  # :1365-1424 align_low_similarity4
        assert len(f) == 12 and f[:6] != f[6:] and int(f[2]) >= int(f[8])

    def exact(f):
        assert len(f) >= 6 and f[1] == match4 and f[4] == "%d=" % len(match4)

    sim4 = []
    for npc in (10.0, 50.0):
        for xd in (27, 30):
            for disc in (0.0, 1.0):
                c4 = dict(score_matrix=dna_scoring_matrix(2, -3, -3), gap_opening_penalty=-5, gap_extension_penalty=-2,
                          xdrop=xd, min_exact_match=disc, max_nodes_per_seq_char=npc, num_alternative_paths=2,
                          min_path_score=0, min_cell_score=0, min_seed_length=6)
                tag = "low_similarity4_%g_%d_%g" % (npc, xd, disc)
                sim4.append((tag, 6, transcripts, 0, True, c4, query4, two_paths if disc == 0.0 else empty))
                sim4.append((tag + "_match", 6, transcripts, 0, True, c4, match4, exact))
    return sim4 + [
        ("straight_fwd_rc_batch", 4, [ref5], 0, True, {}, revcomp(ref5), check_straight),
        ("low_similarity3", 27, [ref6], 0, True, sim3, query6, non_empty),
        ("low_similarity3_filter", 27, [ref6], 0, True, dict(sim3, seed_complexity_filter=True), query6, empty),
        ("snp_canonical", 18, [ref_rc, ref], 1, False, snp, query, check_snp),
        ("snp_primary", 18, [ref_rc], 2, False, snp, query, check_snp),
        ("both_directions", 7, [ref2, revcomp(ref2)], 1, True, {}, query2, check_both),
        ("no_full_seeds_0", 31, [ref3], 2, False, dict(snp, max_seed_length=0), query3, one_path),
        ("no_full_seeds_k100", 31, [ref3], 2, False, dict(snp, max_seed_length=131), query3, one_path),
        ("low_similarity4_rep_primary", 6, primary_contigs(transcripts, 6), 2, True, rep, query4, three_paths),
    ]


def check_mode_kats(lib=None, oracle_only=False):
    """The oracle must satisfy the reference's expectations; with a library, its lines must equal the oracle's."""
    graphs = {}
    for name, k, seqs, mode, masked, kw, query, check in mode_kats():
        key = (k, len(seqs), seqs[0][:64], mode, masked)
        if key not in graphs:
            g = O.OracleGraph(k, seqs, mask=masked, dynamic=not masked)
            g.set_mode(mode)
            idx = None
            if not oracle_only:
                W, last, F, valid = g.arrays()
                idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), valid=valid if masked else None, lib=lib, mode=mode)
            graphs[key] = (g, idx)
        g, idx = graphs[key]
        cfg = struct_defaults(**kw)
        exp = g.align_tsv(cfg, [query], with_nodes=True)
        n_aln = (len(exp[0].split("\t")) - 2) // 7
        check(exp[0].split("\t")[2:2 + 6 * n_aln])
        if oracle_only:
            continue
        got, _ = run_lines(idx, cfg, [query])
        assert got == exp, (name, exp, got)
    for g, idx in graphs.values():
        if idx is not None:
            idx.close()


def check_mt_canonical(lib, **kw):
    """CANONICAL-mode graph (sequences + their reverse complements, mode flag set): integration_tests/test_align.py:207-268."""
    _, seqs = read_fasta(os.path.join(GOLD, "genome.MT.fa"))
    names, reads = read_fastq(os.path.join(GOLD, "genome_MT1.fq"))
    seqs = seqs + [revcomp(s) for s in seqs]
    g = O.OracleGraph(11, seqs, mask=False)
    g.set_mode(1)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(11, W, last, F), lib=lib, mode=1)
    cfg = cli_defaults(11, min_exact_match=0.0, **kw)
    got, _ = run_lines(idx, cfg, reads, names)
    exp = g.align_tsv(cfg, reads, headers=names, with_nodes=True)
    idx.close()
    assert got == exp
    return got


def check_mt_primary(lib, **kw):
    """PRIMARY-mode graph behind CanonicalDBG semantics: integration_tests/test_align.py:270-300."""
    _, seqs = read_fasta(os.path.join(GOLD, "genome.MT.fa"))
    names, reads = read_fastq(os.path.join(GOLD, "genome_MT1.fq"))
    contigs = primary_contigs(seqs, 11)
    g = O.OracleGraph(11, contigs, mask=False)
    g.set_mode(2)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(11, W, last, F), lib=lib, mode=2)
    cfg = cli_defaults(11, min_exact_match=0.0, **kw)
    got, _ = run_lines(idx, cfg, reads, names)
    exp = g.align_tsv(cfg, reads, headers=names, with_nodes=True)
    # CanonicalDBG::map_to_nodes_sequentially (canonical_dbg.cpp:55-146) at the boundary
    probes = reads + [revcomp(r) for r in reads] + ["ACGT", "N" * 30]
    for r, nodes in zip(probes, idx.map_to_nodes_sequentially(probes)):
        assert list(nodes) == list(g.map_to_nodes(r)), r
    idx.close()
    assert got == exp
    return got


def fuzz_case(lib, seed, canonical=False, primary=False, k=None, nreads=25, threads=1):
    """One randomized (graph, reads, config) triple: k, graph shape (variants, repeats, dummy mask), scoring
    matrix, gap penalties, xdrop, seed lengths (exact / MEM / sub-k), seeds per locus, alternative paths,
    strands, end bonuses, cut-offs, node budget, left trim, complexity filter. Returns the mismatching reads."""
    rng = np.random.default_rng(1000 + seed)
    k_drawn = int(rng.integers(4, 34))
    k = k_drawn if k is None else k
    G = int(rng.integers(300, 4000))
    nseq = int(rng.integers(1, 4))
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])
    seqs = [base] + [mutate(rng, base, 0.03) for _ in range(nseq - 1)]
    if rng.random() < 0.3:      # repeats -> branching / cycles
        u = base[:int(rng.integers(k, 3 * k))]
        seqs.append(u * int(rng.integers(2, 5)) + base[50:120])
    match = int(rng.integers(1, 4)); mm1 = -int(rng.integers(1, 5)); mm2 = -int(rng.integers(1, 5))
    go = -int(rng.integers(2, 9)); ge = -int(rng.integers(1, min(-go, 4) + 1))
    kw = dict(score_matrix=dna_scoring_matrix(match, mm1, mm2), gap_opening_penalty=go, gap_extension_penalty=ge,
              xdrop=int(rng.integers(5, 60)), min_exact_match=float(rng.choice([0.0, 0.0, 0.3, 0.7])),
              rel_score_cutoff=float(rng.choice([0.0, 0.5, 0.8, 0.95])),
              num_alternative_paths=int(rng.integers(1, 4)),
              forward_and_reverse_complement=bool(rng.random() < 0.7),
              left_end_bonus=int(rng.integers(0, 7)), right_end_bonus=int(rng.integers(0, 7)),
              max_nodes_per_seq_char=float(rng.choice([5.0, 2.0, 12.0])),
              allow_left_trim=bool(rng.random() < 0.8),
              seed_complexity_filter=bool(rng.random() < 0.3))
    msl = int(rng.integers(2, k + 1)); kw["min_seed_length"] = msl
    kw["max_seed_length"] = int(rng.choice([k, SIZE_MAX, max(msl, k - 1), k + 5]))
    if kw["max_seed_length"] < msl: kw["max_seed_length"] = msl
    kw["max_num_seeds_per_locus"] = int(rng.choice([1000, 2, SIZE_MAX]))
    cfg = cli_defaults(k, **kw)
    mask = bool(rng.random() < 0.3)
    read_src = seqs
    if canonical:               # `build --mode canonical`: every sequence and its reverse complement
        seqs = seqs + [revcomp(s_) for s_ in seqs]
        read_src = seqs
    if primary:                 # `build --mode primary`: one k-mer of every reverse-complement pair
        seqs = primary_contigs(seqs, k)
    g = O.OracleGraph(k, seqs, mask=mask)
    if canonical or primary:
        g.set_mode(2 if primary else 1)
    W, last, F, valid = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), valid=valid if mask else None, lib=lib,
                           mode=2 if primary else 1 if canonical else 0)
    seqs = read_src
    reads = []
    for i in range(nreads):
        s_ = seqs[int(rng.integers(0, len(seqs)))]
        L = int(rng.integers(max(3, k - 3), 160))
        p = int(rng.integers(0, max(1, len(s_) - L)))
        r = mutate(rng, s_[p:p + L], float(rng.choice([0.0, 0.02, 0.08])))
        if rng.random() < 0.5: r = r.translate(COMP)[::-1]
        if rng.random() < 0.1 and len(r) > 5: r = r[:len(r)//2] + "N" + r[len(r)//2+1:]
        reads.append(r)
    try:
        exp = g.align_tsv(cfg, reads, with_nodes=True, threads=threads)
    except RuntimeError as err:                         # DBGAligner ctor: check_config_scores failed
        assert "too low" in str(err)
        import pytest
        from metagraph_b200 import _lib
        with pytest.raises(_lib.MgbError) as e2:
            run_lines(idx, cfg, reads)
        assert e2.value.code == -3                      # MGB_ERR_BAD_CONFIG
        idx.close()
        return [], None
    got, _ = run_lines(idx, cfg, reads)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    idx.close()
    return bad, (k, kw, mask, reads[bad[0]] if bad else None, exp[bad[0]] if bad else None, got[bad[0]] if bad else None)

AA = "ACDEFGHIKLMNPQRSTVWY"


def mutate_aa(rng, r, rate, indel=0.0):
    out = []
    for c in r:
        y = rng.random()
        if y < rate:
            out.append(AA[int(rng.integers(0, 20))])
        elif y < rate + indel / 2:
            out.append(c); out.append(AA[int(rng.integers(0, 20))])
        elif y < rate + indel:
            pass
        else:
            out.append(c)
    return "".join(out)


def protein_case(lib, seed, k, G, nreads, L, rate, cfg, mask=False, nseq=2, indel=0.0):
    """BASELINE configs[3] shape: protein alphabet (sigma = 27, BLOSUM62, forward strand only) through the
    alphabet-generic index layout; reads carry substitutions / indels, the odd 'X', 'B', 'Z', lower case
    and characters outside the alphabet (encoded as 'X', kmer/alphabets.hpp:29-38)."""
    rng = np.random.default_rng(seed)
    seqs = ["".join(np.array(list(AA))[rng.integers(0, 20, G)])]
    seqs += [mutate_aa(rng, seqs[0], 0.03) for _ in range(nseq - 1)]
    seqs[-1] = seqs[-1][:G // 2] + "XBZ" + seqs[-1][G // 2:]
    g = O.OracleGraph(k, seqs, alphabet="protein", mask=mask)
    W, last, F, valid = g.arrays()
    boss = BOSSTable.from_sequences(k, seqs, lib=lib, alphabet=1)
    assert (boss.W == W).all() and (boss.last == last).all() and (boss.F == F).all()
    if mask:
        assert (boss.dummy_mask(lib=lib) == valid).all()
    idx = DBGSuccinctIndex(boss, valid=valid if mask else None, lib=lib)
    reads = []
    for i in range(nreads):
        s_ = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, max(1, len(s_) - L)))
        r = mutate_aa(rng, s_[p:p + L], rate, indel)
        if i % 7 == 3 and len(r) > 4:
            r = r[:len(r) // 2] + "X*" + r[len(r) // 2 + 2:]
        if i % 5 == 1:
            r = r.lower()
        reads.append(r)
    reads += ["", "A", "ACDE", "X" * 30, "**********"]
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    got, stats = run_lines(idx, cfg, reads)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (seed, bad[:3], exp[bad[0]], got[bad[0]])
    nodes = idx.map_to_nodes_sequentially(reads)
    for r, n in zip(reads, nodes):
        assert list(n) == list(g.map_to_nodes(r)), r
    idx.close()
    n_aligned = sum(1 for l in got if l.split("\t")[3] != "*")
    return n_aligned, len(reads)


PROTEIN_CASES = [
    # seed, k, G, nreads, L, subst rate, cfg, mask, nseq, indel rate
    (21, 10, 3000, 40, 100, 0.05, lambda k: cli_defaults(k, alphabet="protein", min_exact_match=0.0), False, 2, 0.0),
    (22, 10, 3000, 40, 100, 0.03, lambda k: cli_defaults(k, alphabet="protein"), False, 3, 0.02),
    (23, 6, 1500, 30, 60, 0.08, lambda k: cli_defaults(k, alphabet="protein", min_exact_match=0.0,
                                                         num_alternative_paths=2), True, 2, 0.02),
    (24, 10, 4000, 30, 100, 0.0, lambda k: cli_defaults(k, alphabet="protein", min_seed_length=10,
                                                         max_seed_length=10), False, 1, 0.0),
    (25, 12, 3000, 30, 80, 0.05, lambda k: cli_defaults(k, alphabet="protein", min_exact_match=0.0,
                                                         min_seed_length=5), False, 2, 0.01),
]


def sd(**kw):
    return struct_defaults(**kw)


RANDOM_CASES = [
    # seed, k, G, nreads, L, rate, cfg, mask, nseq
    (1, 11, 3000, 40, 100, 0.0, lambda k: cli_defaults(k, min_exact_match=0.0), False, 1),
    (2, 11, 3000, 40, 100, 0.05, lambda k: cli_defaults(k, min_exact_match=0.0), False, 1),
    (3, 15, 5000, 40, 150, 0.05, lambda k: cli_defaults(k, min_exact_match=0.0), False, 3),
    (4, 31, 20000, 40, 150, 0.05, lambda k: cli_defaults(k, min_exact_match=0.0), False, 2),
    (5, 31, 20000, 40, 150, 0.0, lambda k: cli_defaults(k, min_seed_length=31, max_seed_length=31), False, 1),
    (6, 31, 20000, 40, 150, 0.03, lambda k: cli_defaults(k, min_seed_length=31, max_seed_length=31), False, 3),
    (7, 9, 2000, 30, 60, 0.05, lambda k: sd(), True, 2),
    (8, 7, 500, 30, 40, 0.08, lambda k: sd(xdrop=20), True, 2),
    (9, 21, 10000, 40, 120, 0.08, lambda k: cli_defaults(k, min_exact_match=0.0, num_alternative_paths=2), False, 4),
    (10, 12, 4000, 30, 300, 0.03, lambda k: cli_defaults(k), False, 2),
    (11, 31, 20000, 40, 150, 0.05,
     lambda k: cli_defaults(k, min_exact_match=0.0, forward_and_reverse_complement=False), False, 2),
    # large enough for the device-refined suffix-range levels (s > 8)
    (12, 31, 400000, 30, 150, 0.02, lambda k: cli_defaults(k, min_seed_length=31, max_seed_length=31), False, 1),
]


# Inputs that push k_align out of its on-chip working set, one per path (align_core.cuh): DP columns wider than the
# on-chip column buffers (created in arena scratch, or moved there mid-column by extend_ins_end), reads not staged on
# chip, the best-first queue and the next-nodes list moving to the arena, reads that overflow their arena and are retried
# with a larger one. The copies between the two places are warp-cooperative, so only the device can show a race in them;
# the host emulation shows that each input reaches its path (PRESSURE_TARGETS, path_hits).
PRESSURE_INPUTS = ("insertions", "insertions_cheap_gaps", "wide_band", "queue", "retry")
PRESSURE_TARGETS = {
    "insertions": ("column_migrate", "arena_column"),
    "insertions_cheap_gaps": ("column_migrate", "arena_column"),
    "wide_band": ("arena_column", "unstaged_read"),
    "queue": ("queue_migrate", "nn_migrate"),
    "retry": ("read_overflow",),
}


def _random_seq(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def pressure_input(name):
    """(k, graph sequences, reads, config) of one of PRESSURE_INPUTS"""
    if name in ("insertions", "insertions_cheap_gaps"):
        # 300 bp windows with 40 bp of random sequence inserted in the middle or put in place of the last 20 bp: under a
        # large x-drop the insertion runs of extend_ins_end grow a column past the on-chip buffers while it is computed
        rng = np.random.default_rng(301)
        k = 15
        genome = _random_seq(rng, 5000)
        reads = []
        for i in range(40):
            p = int(rng.integers(0, len(genome) - 300))
            w, ins = genome[p:p + 300], _random_seq(rng, 40)
            r = w[:150] + ins + w[150:] if i % 2 else w[:280] + ins
            reads.append(revcomp(r) if i % 3 == 0 else r)
        kw = dict(xdrop=1000) if name == "insertions" else dict(xdrop=300, gap_opening_penalty=-2, gap_extension_penalty=-1)
        return k, [genome], reads, cli_defaults(k, min_exact_match=0.0, **kw)
    if name == "wide_band":
        # no x-drop: a column spans the whole read. Reads of 249 .. 600 bp: the on-chip buffers are capped at 256 cells
        # and a batch with a read over 511 bp stages no query on chip (lq = 0)
        rng = np.random.default_rng(302)
        k = 13
        genome = _random_seq(rng, 1500)
        reads = []
        for i in range(10):
            L = 600 if i == 0 else 249 if i == 1 else int(rng.integers(249, 601))
            p = int(rng.integers(0, len(genome) - L))
            r = mutate(rng, genome[p:p + L], 0.03)
            reads.append(revcomp(r) if i % 2 else r)
        return k, [genome], reads, struct_defaults()
    if name == "queue":
        # tandem repeats on a low-complexity graph, three alternative paths and a large node budget: many columns wait in
        # the queue (and tie for the next-nodes list) at once, more than the on-chip queue holds
        rng = np.random.default_rng(303)
        k = 11
        base = lowcx_genome(rng, 4000)
        unit = _random_seq(rng, 7)
        seqs = [base, base[:600] + unit * 30 + base[600:1400], mutate(rng, base[2000:3500], 0.03)]
        reads = []
        for i in range(30):
            s_ = seqs[i % 3]
            p = int(rng.integers(0, len(s_) - 150))
            r = mutate(rng, s_[p:p + 150], 0.04)
            reads.append(revcomp(r) if i % 2 else r)
        reads.append(base[580:600] + unit * 14 + base[600:620])
        cfg = cli_defaults(k, min_seed_length=8, num_alternative_paths=3, max_nodes_per_seq_char=50.0, xdrop=60,
                           min_exact_match=0.0, rel_score_cutoff=0.0)
        return k, seqs, reads, cfg
    if name == "retry":
        # low-complexity sequence (homopolymers, short tandem repeats) with every seed kept, sub-k seeds, a large x-drop
        # and node budget: about half the reads from it explore more columns than their arena holds at scale 1 and are
        # retried with a larger one; the reads from the unique sequence in the same batch are not
        rng = np.random.default_rng(304)
        k = 15
        seqs = [lowcx_genome(rng, 3000), _random_seq(rng, 2000)]
        reads = []
        for i in range(30):
            s_, L = (seqs[0], 150) if i % 2 == 0 else (seqs[1], 110)
            p = int(rng.integers(0, len(s_) - L))
            r = mutate(rng, s_[p:p + L], 0.03)
            reads.append(revcomp(r) if i % 3 == 0 else r)
        cfg = cli_defaults(k, min_seed_length=6, max_num_seeds_per_locus=SIZE_MAX, max_nodes_per_seq_char=20.0,
                           xdrop=100, min_exact_match=0.0)
        return k, seqs, reads, cfg
    raise ValueError(name)


_pressure_expected = {}


def pressure_case(lib, name):
    """Runs the pressure input `name` through the library: lines == oracle (node paths included). Returns the run's
    statistics and, on the host emulation, how often it took each path (path_hits; None on the device). The index is
    built inside the call, so index-side knobs set in the environment apply."""
    k, seqs, reads, cfg = pressure_input(name)
    if name not in _pressure_expected:
        _pressure_expected[name] = O.OracleGraph(k, seqs).align_tsv(cfg, reads, with_nodes=True)
    exp = _pressure_expected[name]
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    h0 = path_hits(lib)
    got, stats = run_lines(idx, cfg, reads)
    h1 = path_hits(lib)
    idx.close()
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (name, bad[:3], exp[bad[0]][:300], got[bad[0]][:300])
    return stats, None if h0 is None else {p: h1[p] - h0[p] for p in EMU_PATHS}


# Knobs of api.cu that move k_align's on-chip limits or switch a path off (name, environment). Where a column, the queue
# or a query strand lives must change neither the lines nor the DP: every run equals the oracle, and its DP_COUNTERS
# equal those of the default run. The host chooses the smallest column buffer as 64 cells (the register path of the
# extender needs 40); a small queue or staging limit only makes the checks on every push and every read (n >= hp_cap,
# L + 1 <= lq) fire earlier. The k-mer hash and path index exist on the device only.
SPILL_KNOBS = (
    ("default", {}),
    ("bmax64", {"MGB_TEST_BMAX": "64"}),
    ("lq0", {"MGB_TEST_LQ": "0"}),
    ("lq_split", {"MGB_TEST_LQ": None}),                                 # pressure_lq_split: some reads staged, some not
    ("hcap1", {"MGB_TEST_HCAP": "1"}),
    ("hcap4", {"MGB_TEST_HCAP": "4"}),
    ("nofast", {"MGB_TEST_NOFAST": "1"}),                                # no register path: every column general
    ("nosubk", {"MGB_TEST_NOSUBK": "1"}),                                # sub-k seeds (min_seed_length < k) in k_align
    ("nopremap", {"MGB_TEST_NOPREMAP": "1", "MGB_NO_KMER_HASH": "1"}),   # premap runs only without the k-mer hash
    ("no_path_index", {"MGB_NO_PATH_INDEX": "1"}),
    ("wide", {"MGB_TEST_WIDE": "1"}),                                    # the alphabet-generic index layout
    ("pieces3", {"MGB_TEST_PIECES": "3"}),                               # retried reads in several pieces and heaps
    ("grid1", {"MGB_TEST_MAX_BLOCKS": "1"}),                             # one block of each read-path kernel: k_align's
                                                                         # 4 warps align every read, one after another
)
DP_COUNTERS = ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns")


def pressure_lq_split(name):
    """a staging limit (multiple of 16) that stages some reads of the input on chip and leaves others in global memory"""
    lens = [len(r) for r in pressure_input(name)[2]]
    fits = [lq for lq in range(16, 1024, 16) if min(lens) + 1 <= lq < max(lens) + 1]
    assert fits, (name, min(lens), max(lens))
    return fits[len(fits) // 2]


def pressure_knob_matrix(lib, name, monkeypatch, knobs=SPILL_KNOBS):
    """Runs the pressure input `name` under every knob: lines == oracle, DP counters == the default run's. Returns
    {knob: (statistics, path hits)}; path hits are None on the device."""
    out = {}
    for knob, env in knobs:
        with monkeypatch.context() as mp:
            for var, val in env.items():
                mp.setenv(var, str(pressure_lq_split(name)) if val is None else val)
            out[knob] = pressure_case(lib, name)
        base = out[knobs[0][0]][0]
        diff = {c: (base[c], out[knob][0][c]) for c in DP_COUNTERS if out[knob][0][c] != base[c]}
        assert not diff, (name, knob, diff)
    return out
