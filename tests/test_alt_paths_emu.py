"""num_alternative_paths from 5 to 32 (`metagraph align --align-alternative-alignments N`) on the host emulation of the
kernels: lines and node paths equal the oracle's on a gene-family graph where reads map to many places, and on the
random, canonical, primary and protein inputs; N = 33 is refused."""
import os
import subprocess

import pytest

import alt_paths_common as A
import parity_common as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")

# (N, seeder, rel_score_cutoff or None for the CLI default 0.95): least number of reads (of 60) with exactly N records
REACH = [
    (5, "exact", None, 55), (8, "mem", None, 40), (16, "subk", 0.0, 40), (32, "exact", None, 18),
    (32, "subk", 0.0, 40), (16, "exact", None, 15), (8, "subk", None, 40), (32, "mem", 0.0, 40),
]


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("n_alt,seeder,rel,least", REACH, ids=["%d-%s-%s" % c[:3] for c in REACH])
def test_gene_family_emu(n_alt, seeder, rel, least):
    h0 = A.agg_hits(EMU)
    got, _ = A.family_case(EMU, A.config(n_alt, seeder, rel))
    h1 = A.agg_hits(EMU)
    counts = A.record_counts(got)
    assert sum(c == n_alt for c in counts) >= least, counts
    assert max(counts) == n_alt
    if n_alt > 5:
        assert any(5 <= c < n_alt for c in counts), counts
    # the full aggregator gave an entry's slot to a better alignment
    assert h1["replace"] > h0["replace"]


def test_gene_family_duplicates_emu():
    """sub-k seeds find the same alignment more than once: the aggregator drops the copies"""
    h0 = A.agg_hits(EMU)
    A.family_case(EMU, A.config(16, "subk", 0.0))
    assert A.agg_hits(EMU)["duplicate"] > h0["duplicate"]


@pytest.mark.parametrize("mode", ["basic", "canonical", "primary"])
def test_graph_modes_emu(mode):
    """N = 16: random_case on a BASIC graph of four diverged copies, the gene-family input on CANONICAL and PRIMARY
    graphs"""
    if mode == "basic":
        seed, k, G, n, L, rate, _, mask, nseq = P.RANDOM_CASES[8]
        P.random_case(EMU, seed, k, G, n, L, rate, A.config_k(k, 16), mask, nseq)
    else:
        counts = A.record_counts(A.mode_case(EMU, 16, mode))
        assert sum(c == 16 for c in counts) >= 20, counts


def test_protein_generic_layout_emu():
    seed, k, G, n, L, rate, _, mask, nseq, indel = P.PROTEIN_CASES[2]
    aligned, total = P.protein_case(EMU, seed, k, G, n, L, rate, A.config_k(k, 8, alphabet="protein"), mask, nseq,
                                    indel)
    assert aligned >= total // 2


@pytest.mark.parametrize("i", range(25))
def test_fuzz_n_alt_emu(i):
    assert 5 <= A.fuzz_case(EMU, i) <= A.MAX_ALT


def test_spill_knobs_emu(monkeypatch):
    """the gene-family input at N = 32 under every spill knob: lines == oracle, DP counters == the default run's"""
    A.spill_knob_matrix(EMU, monkeypatch)


def test_retry_many_records_emu(monkeypatch):
    """pass 0's output heap too small for the reads with 32 records: they are retried, in one piece and in several"""
    for pieces in (None, "3"):
        with monkeypatch.context() as mp:
            if pieces:
                mp.setenv("MGB_TEST_PIECES", pieces)
            stats = A.heap_retry_case(EMU, mp)
        assert stats["num_reads_retried"] > 0, stats


def test_limits_emu():
    A.check_limits(EMU)


def test_limits_shim_emu(tmp_path):
    emu_dir = os.path.join(ROOT, "tests", "emu", "build")
    A.check_limits_shim(tmp_path, ["-L" + emu_dir, "-lmgb_emu", "-Wl,-rpath," + emu_dir, "-fopenmp"])


def test_sharded_export_import_gloo(tmp_path):
    """two gloo ranks, N = 8: shards carry reads with up to 8 records through mgb_results_export / _import, and the
    gathered lines equal a single-rank run"""
    A.check_sharding(tmp_path, EMU)
