"""Parity tests proper: the sm_90a library (through the C-ABI) vs the oracle on a real GPU."""
import os

import numpy as np
import pytest

import parity_common as P

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)


def test_goldens_gpu():
    P.check_goldens(LIB)


@pytest.mark.parametrize("both", [False, True])
def test_mt_integration_gpu(both):
    P.check_mt(LIB, both)


@pytest.mark.parametrize("subk", [False, True])
def test_mt_canonical_gpu(subk):
    # integration_tests/test_align.py:207-268 (graph built with --mode canonical)
    got = P.check_mt_canonical(LIB, **({"min_seed_length": 10} if subk else {}))
    from test_oracle_canonical import CANONICAL, CANONICAL_SUBK
    for i, exp in (CANONICAL_SUBK if subk else CANONICAL):
        assert got[int(i)].split("\t")[:8] == exp.encode().decode("unicode_escape").split("\t")[:8]


@pytest.mark.parametrize("case", P.RANDOM_CASES, ids=[str(c[0]) for c in P.RANDOM_CASES])
def test_random_gpu(case):
    seed, k, G, n, L, rate, cfgf, mask, nseq = case
    P.random_case(LIB, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


@pytest.mark.parametrize("case", P.PROTEIN_CASES, ids=[str(c[0]) for c in P.PROTEIN_CASES])
def test_protein_gpu(case):
    """configs[3] shape: protein alphabet through the alphabet-generic kernel path."""
    seed, k, G, n, L, rate, cfgf, mask, nseq, indel = case
    aligned, total = P.protein_case(LIB, seed, k, G, n, L, rate, cfgf(k), mask, nseq, indel)
    assert aligned >= total // 2


def test_generic_layout_on_dna_gpu(monkeypatch):
    """The alphabet-generic index layout must reproduce the DNA goldens as well."""
    monkeypatch.setenv("MGB_TEST_WIDE", "1")
    P.check_goldens(LIB)
    P.check_mt(LIB, True)
    for case in P.RANDOM_CASES[:4] + P.RANDOM_CASES[6:8]:
        seed, k, G, n, L, rate, cfgf, mask, nseq = case
        P.random_case(LIB, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


def test_general_path_gpu(monkeypatch):
    """With the extender's register path switched off every column goes through the general path (S | E | F table
    format), with all 32 lanes sharing a column: the goldens, MT and the first random cases still equal the oracle."""
    monkeypatch.setenv("MGB_TEST_NOFAST", "1")
    P.check_goldens(LIB)
    P.check_mt(LIB, True)
    for case in P.RANDOM_CASES[:5]:
        seed, k, G, n, L, rate, cfgf, mask, nseq = case
        P.random_case(LIB, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


def test_seed_complexity_filter_gpu():
    """seed complexity filter on (CLI default): kernels vs oracle on low-complexity inputs."""
    for seed, k, exact in ((31, 15, False), (32, 21, True), (33, 31, False)):
        P.lowcx_case(LIB, seed, k, exact)


@pytest.mark.gpu
@pytest.mark.parametrize("case", P.WHOLE_READ_CASES, ids=[str(c[0]) for c in P.WHOLE_READ_CASES])
def test_whole_read_shortcut_gpu(case):
    seed, k, cfgf, _ = case
    P.whole_read_case(LIB, seed, k, cfgf(k))


@pytest.mark.gpu
@pytest.mark.parametrize("case", P.EXACT_SHORTCUT_CASES, ids=[str(c[0]) for c in P.EXACT_SHORTCUT_CASES])
def test_exact_path_shortcut_gpu(case):
    seed, k, cfgf = case
    P.exact_shortcut_case(LIB, seed, k, cfgf(k))


def test_nodeless_results_gpu():
    """MGB_NODES_NONE: identical alignments, node arrays stay on the device"""
    P.nodeless_case(LIB)


def test_concurrent_callers_gpu():
    """several host threads call mgb_align_batch on one index at the same time (cli/align.cpp:440-475)"""
    P.concurrent_case(LIB)


def test_c1_shape_gpu():
    """configs[0] shape: transcripts (59 bp .. 11 666 bp, the range of transcripts_1000.fa) aligned to
    their own k=12 graph at CLI defaults."""
    n, full = P.c1_case(LIB, 40, 11666)
    assert full >= n - 4


def test_random_gpu_in_pieces(monkeypatch):
    """Batch split into pieces on two streams / host threads (forced on small batches)."""
    monkeypatch.setenv("MGB_TEST_PIECES", "3")
    for case in P.RANDOM_CASES[:4]:
        seed, k, G, n, L, rate, cfgf, mask, nseq = case
        P.random_case(LIB, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


def test_c2_scale_properties():
    """BASELINE config[1] shape at reduced genome size: every error-free read must align end to end
    ({L}= with score 2L+10), forward reads on '+', reverse-complemented reads on '-', and the path must
    spell the read; a 2000-read sample is compared with the oracle line by line."""
    import oracle_lib as O
    from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
    from metagraph_b200.config import cli_defaults
    k, G, N = 31, 2_000_000, 140000      # > 128k reads: the batch runs as two pieces
    rng = np.random.default_rng(32)
    genome = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, G, dtype=np.uint8)]
    boss = BOSSTable.from_sequences(k, None, packed=(genome, np.array([0, G], dtype=np.uint64)))
    idx = DBGSuccinctIndex(boss)
    rng = np.random.default_rng(42)
    comp = np.zeros(256, np.uint8); comp[list(b"ACGT")] = list(b"TGCA")
    reads = []
    for i in range(N):
        p = int(rng.integers(0, G - 150))
        r = genome[p:p + 150]
        reads.append(bytes(comp[r][::-1] if i & 1 else r).decode())
    cfg = cli_defaults(k, min_seed_length=31, max_seed_length=31)
    al = B200Aligner(idx, cfg)
    res = al.align_batch([("", r) for r in reads])
    assert len(res) == N
    for i, (r, ar) in enumerate(zip(reads, res)):
        assert len(ar) == 1
        a = ar[0]
        assert a.get_cigar_string() == "150=" and a.score == 310 and a.offset == 0
        assert a.orientation == bool(i & 1)
        assert a.sequence == (r.translate(P.COMP)[::-1] if i & 1 else r)
        assert len(a.nodes) == 120
    o = O.OracleGraph(k, arrays=(boss.W, boss.last, boss.F))
    exp = o.align_tsv(cfg, reads[:2000], with_nodes=True, threads=8)
    got = [format_alignment("", r, 0, with_nodes=True) for r in res[:2000]]
    assert got == exp


def test_c1_transcripts_1000_gpu():
    """BASELINE configs[0] on the reference's own fixture: tests/data/transcripts_1000.fa (1000 records, 59 bp ..
    11 666 bp), k = 12 graph of the transcripts, the transcripts themselves as reads at CLI defaults. Kernels ==
    oracle line by line (node paths included); SURVEY 8c expects every read to align to itself end to end."""
    import os
    import oracle_lib as O
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import cli_defaults
    from test_oracle_golden import GOLD, read_fasta
    names, seqs = read_fasta(os.path.join(GOLD, "transcripts_1000.fa"))
    assert len(seqs) == 1000 and sum(len(s) for s in seqs) == 1490627
    k = 12
    boss = BOSSTable.from_sequences(k, seqs)
    idx = DBGSuccinctIndex(boss)
    cfg = cli_defaults(k)
    got, _ = P.run_lines(idx, cfg, seqs)
    g = O.OracleGraph(k, arrays=(boss.W, boss.last, boss.F))
    exp = g.align_tsv(cfg, seqs, with_nodes=True, threads=16)
    bad = [i for i in range(len(seqs)) if exp[i] != got[i]]
    assert not bad, (bad[:3], len(seqs[bad[0]]), exp[bad[0]][:200], got[bad[0]][:200])
    full = sum(1 for s_, l in zip(seqs, got) if l.split("\t")[6] == "%d=" % len(s_) and int(l.split("\t")[4]) == 2 * len(s_) + 10)
    assert full >= 990, full
    idx.close()


@pytest.mark.parametrize("which", ["dna", "protein"])
def test_example_dbg_graphs_gpu(which):
    """The two graph files the reference ships (examples/data/graphs/*.dbg, written by `metagraph build`): loaded
    with mgb_dbg_load, uploaded, and aligned against on the device; kernels == oracle on the example queries."""
    import os
    import oracle_lib as O
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import cli_defaults
    import test_dbg_loader as T
    dbg, fa, qfa, alpha, code = [c for c in T.CASES if c[3] == which][0]
    t = BOSSTable.from_dbg(os.path.join(T.EX, dbg))
    idx = DBGSuccinctIndex(t)
    reads = T.fasta(os.path.join(T.EX, qfa)) + [s[3:50] for s in T.fasta(os.path.join(T.EX, fa))]
    cfg = cli_defaults(t.k, alphabet=alpha)
    g = O.OracleGraph(t.k, arrays=(t.W, t.last, t.F), alphabet=alpha)
    exp = g.align_tsv(cfg, reads, with_nodes=True)
    got, _ = P.run_lines(idx, cfg, reads)
    assert got == exp
    idx.close()


def test_cpp_shim_on_device(tmp_path):
    """tests/cpp/test_shim.cpp (the IDBGAligner-shaped C++ shim) linked against the product library libmgb.so"""
    import subprocess
    from metagraph_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir = os.path.dirname(_lib.DEFAULT_LIB)
    exe = str(tmp_path / "test_shim_dev")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(root, "tests", "cpp", "test_shim.cpp"),
                           "-o", exe, "-L" + lib_dir, "-l:libmgb.so", "-Wl,-rpath," + lib_dir, "-fopenmp"])
    dbg = os.path.join(root, "tests", "golden", "example_graphs", "test_DNA_graph.dbg")
    out = subprocess.run([exe, dbg], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "q1\tAGCTNCGAGGCCAA\t4=1X9=\t24" in out.stdout and "dbg\t36=" in out.stdout
