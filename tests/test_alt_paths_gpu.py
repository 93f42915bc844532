"""num_alternative_paths from 5 to 32 on the sm_90a library: the inputs of test_alt_paths_emu.py on the device, where the
aggregator keeps one entry per lane of the warp, against the oracle with node paths."""
import os

import pytest

import alt_paths_common as A
import parity_common as P

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)

# (N, seeder, rel_score_cutoff or None for the CLI default 0.95): least number of reads (of 60) with exactly N records
REACH = [
    (5, "exact", None, 55), (8, "mem", None, 40), (16, "subk", 0.0, 40), (32, "exact", None, 18),
    (32, "subk", 0.0, 40), (16, "exact", None, 15), (8, "subk", None, 40), (32, "mem", 0.0, 40),
]


@pytest.mark.parametrize("n_alt,seeder,rel,least", REACH, ids=["%d-%s-%s" % c[:3] for c in REACH])
def test_gene_family_gpu(n_alt, seeder, rel, least):
    got, _ = A.family_case(LIB, A.config(n_alt, seeder, rel))
    counts = A.record_counts(got)
    print("N=%d %s rel=%s: %d reads with N records, %d with 5..N-1"
          % (n_alt, seeder, rel, sum(c == n_alt for c in counts), sum(5 <= c < n_alt for c in counts)))
    assert sum(c == n_alt for c in counts) >= least, counts
    assert max(counts) == n_alt
    if n_alt > 5:
        assert any(5 <= c < n_alt for c in counts), counts


@pytest.mark.parametrize("mode", ["basic", "canonical", "primary"])
def test_graph_modes_gpu(mode):
    """N = 16: random_case on a BASIC graph of four diverged copies, the gene-family input on CANONICAL and PRIMARY
    graphs (the CANONICAL-mode compilation of k_align serves both)"""
    if mode == "basic":
        seed, k, G, n, L, rate, _, mask, nseq = P.RANDOM_CASES[8]
        P.random_case(LIB, seed, k, G, n, L, rate, A.config_k(k, 16), mask, nseq)
    else:
        counts = A.record_counts(A.mode_case(LIB, 16, mode))
        assert sum(c == 16 for c in counts) >= 20, counts


def test_protein_generic_layout_gpu():
    seed, k, G, n, L, rate, _, mask, nseq, indel = P.PROTEIN_CASES[2]
    aligned, total = P.protein_case(LIB, seed, k, G, n, L, rate, A.config_k(k, 8, alphabet="protein"), mask, nseq,
                                    indel)
    assert aligned >= total // 2


def test_generic_layout_on_gene_family_gpu(monkeypatch):
    """the DNA input through the alphabet-generic compilation of k_align"""
    monkeypatch.setenv("MGB_TEST_WIDE", "1")
    A.family_case(LIB, A.config(32, "subk", 0.0))


@pytest.mark.parametrize("i", range(40))
def test_fuzz_n_alt_gpu(i):
    assert 5 <= A.fuzz_case(LIB, i) <= A.MAX_ALT


def test_spill_knobs_gpu(monkeypatch):
    """the gene-family input at N = 32 under every spill knob: lines == oracle, DP counters == the default run's"""
    A.spill_knob_matrix(LIB, monkeypatch)


def test_retry_many_records_gpu(monkeypatch):
    """pass 0's output heap too small for the reads with 32 records: they are retried, in one piece and in several"""
    for pieces in (None, "3"):
        with monkeypatch.context() as mp:
            if pieces:
                mp.setenv("MGB_TEST_PIECES", pieces)
            stats = A.heap_retry_case(LIB, mp)
        assert stats["num_reads_retried"] > 0, stats


def test_limits_gpu():
    A.check_limits(LIB)


def test_limits_shim_gpu(tmp_path):
    from metagraph_b200 import _lib
    lib_dir = os.path.dirname(_lib.DEFAULT_LIB)
    A.check_limits_shim(tmp_path, ["-L" + lib_dir, "-l:libmgb.so", "-Wl,-rpath," + lib_dir, "-fopenmp"])
