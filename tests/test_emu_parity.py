"""Kernel logic vs oracle on a machine without a GPU: the kernel sources (metagraph_b200/csrc/*.cuh,
api.cu) compiled by g++ with one-lane warps (tests/emu/, test infrastructure) must reproduce the
oracle's TSV lines and node paths bit-exactly. The real sm_90a build is checked by test_gpu_parity.py."""
import os
import subprocess

import pytest

import parity_common as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


def test_goldens_emu():
    P.check_goldens(EMU)


@pytest.mark.parametrize("both", [False, True])
def test_mt_integration_emu(both):
    P.check_mt(EMU, both)


@pytest.mark.parametrize("subk", [False, True])
def test_mt_canonical_emu(subk, _emu_built):
    # integration_tests/test_align.py:207-268 (graph built with --mode canonical)
    got = P.check_mt_canonical(EMU, **({"min_seed_length": 10} if subk else {}))
    from test_oracle_canonical import CANONICAL, CANONICAL_SUBK
    for i, exp in (CANONICAL_SUBK if subk else CANONICAL):
        assert got[int(i)].split("\t")[:8] == exp.encode().decode("unicode_escape").split("\t")[:8]


def test_map_count_kmers_golden_emu():
    # `metagraph align --map --count-kmers` (integration_tests/test_align.py:58-87) through mgb_map_to_nodes
    from test_oracle_golden import GOLD, MAP_COUNTS, _map_counts, read_fasta, read_fastq
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
    _, seqs = read_fasta(os.path.join(GOLD, "genome.MT.fa"))
    _, reads = read_fastq(os.path.join(GOLD, "genome_MT1.fq"))
    boss = BOSSTable.from_sequences(11, seqs, lib=EMU)
    idx = DBGSuccinctIndex(boss, valid=boss.dummy_mask(lib=EMU), lib=EMU)
    assert [_map_counts(n) for n in idx.map_to_nodes_sequentially(reads)] == MAP_COUNTS
    idx.close()


def test_mode_known_answers_emu():
    # the reference's unit tests for CANONICAL / PRIMARY graphs (tests/graph/test_aligner.cpp:1483-1631, 1773-1800)
    P.check_mode_kats(EMU)


@pytest.mark.parametrize("subk", [False, True])
def test_mt_primary_emu(subk):
    # integration_tests/test_align.py:270-330 (graph built with --mode primary), CanonicalDBG semantics on device
    got = P.check_mt_primary(EMU, **({"min_seed_length": 10} if subk else {}))
    from test_oracle_canonical import CANONICAL, CANONICAL_SUBK
    for i, exp in (CANONICAL_SUBK if subk else CANONICAL):
        assert got[int(i)].split("\t")[:8] == exp.encode().decode("unicode_escape").split("\t")[:8]
    assert got[6].split("\t")[4] == "310" and (subk or got[5].split("\t")[4] == "22")


@pytest.mark.parametrize("case", P.RANDOM_CASES, ids=[str(c[0]) for c in P.RANDOM_CASES])
def test_random_emu(case):
    seed, k, G, n, L, rate, cfgf, mask, nseq = case
    P.random_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


@pytest.mark.parametrize("case", P.PROTEIN_CASES, ids=[str(c[0]) for c in P.PROTEIN_CASES])
def test_protein_emu(case):
    seed, k, G, n, L, rate, cfgf, mask, nseq, indel = case
    aligned, total = P.protein_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq, indel)
    assert aligned >= total // 2


def test_generic_layout_on_dna_emu(monkeypatch):
    """The alphabet-generic index layout (used for protein) must reproduce every DNA golden too."""
    monkeypatch.setenv("MGB_TEST_WIDE", "1")
    P.check_goldens(EMU)
    P.check_mt(EMU, True)
    for case in P.RANDOM_CASES[:4] + P.RANDOM_CASES[6:8]:
        seed, k, G, n, L, rate, cfgf, mask, nseq = case
        P.random_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


def test_general_path_emu(monkeypatch):
    """The emulation runs the extender's register path (one lane owning all 32 cells of a column) wherever the
    device does; with it switched off every column goes through the general path (S | E | F table format)."""
    monkeypatch.setenv("MGB_TEST_NOFAST", "1")
    P.check_goldens(EMU)
    P.check_mt(EMU, True)
    for case in P.RANDOM_CASES[:5]:
        seed, k, G, n, L, rate, cfgf, mask, nseq = case
        P.random_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


@pytest.mark.parametrize("case", P.EXACT_SHORTCUT_CASES, ids=[str(c[0]) for c in P.EXACT_SHORTCUT_CASES])
def test_exact_path_shortcut_emu(case):
    seed, k, cfgf = case
    P.exact_shortcut_case(EMU, seed, k, cfgf(k))


def test_nodeless_results_emu():
    P.nodeless_case(EMU)


def test_seed_complexity_filter_emu():
    """CLI default `seed_complexity_filter` (sdust restated from its definition, parity with the library
    unpinned): kernels vs oracle on reads and graphs full of homopolymers / short tandem repeats."""
    for seed, k, exact in ((31, 15, False), (32, 21, True), (33, 31, False)):
        P.lowcx_case(EMU, seed, k, exact)


def test_c1_shape_emu():
    """configs[0] shape: transcripts aligned to their own k=12 graph, ragged lengths up to 2.5 kbp. The batch holds
    reads over 511 bp, so no read is staged on chip; at the CLI's x-drop every DP column still fits the on-chip
    buffers (the arena-column paths are reached by the pressure inputs, test_pressure_inputs_reach_their_paths_emu)."""
    h0 = P.path_hits(EMU)
    n, full = P.c1_case(EMU, 10, 2500)
    h1 = P.path_hits(EMU)
    assert full >= n - 2
    assert h1["unstaged_read"] - h0["unstaged_read"] >= n


def test_c1_transcripts_subset_emu():
    """the first 40 records of the configs[0] fixture (up to 4.5 kbp) against the graph of all 1000"""
    import oracle_lib as O
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import cli_defaults
    from test_oracle_golden import GOLD, read_fasta
    _, seqs = read_fasta(os.path.join(GOLD, "transcripts_1000.fa"))
    boss = BOSSTable.from_sequences(12, seqs, lib=EMU)
    idx = DBGSuccinctIndex(boss, lib=EMU)
    cfg = cli_defaults(12)
    reads = seqs[:40]
    got, _ = P.run_lines(idx, cfg, reads)
    exp = O.OracleGraph(12, arrays=(boss.W, boss.last, boss.F)).align_tsv(cfg, reads, with_nodes=True, threads=8)
    assert got == exp
    idx.close()


def test_random_emu_in_pieces(monkeypatch):
    """mgb_align_batch splits big batches into pieces run by two host threads; force the split on a
    small batch (ragged piece boundaries, results merged in read order)."""
    monkeypatch.setenv("MGB_TEST_PIECES", "3")
    seed, k, G, n, L, rate, cfgf, mask, nseq = P.RANDOM_CASES[1]
    P.random_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq)
    monkeypatch.setenv("MGB_TEST_PIECES", "1000000")      # more pieces than reads: one read each
    seed, k, G, n, L, rate, cfgf, mask, nseq = P.RANDOM_CASES[2]
    P.random_case(EMU, seed, k, G, n, L, rate, cfgf(k), mask, nseq)


def test_concurrent_callers_emu():
    """cli/align.cpp:440-475 runs align_batch from several worker threads on one shared graph: mgb_align_batch
    must be re-entrant (per-call workspaces, thread-local error state)."""
    P.concurrent_case(EMU)


def test_unsupported_configs_fail_loudly():
    from metagraph_b200 import _lib
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex, B200Aligner
    from metagraph_b200.config import struct_defaults
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(4, ["AGCTTCGAGGCCAA"], lib=EMU), lib=EMU)
    for kw, code in ((dict(global_xdrop=False), -4),
                     (dict(num_alternative_paths=99), -4), (dict(min_cell_score=-2**31), -3)):
        with pytest.raises(_lib.MgbError) as e:
            B200Aligner(idx, struct_defaults(**kw)).align("AGCTTCGAGG")
        assert e.value.code == code


def test_graph_modes_fail_loudly():
    """DeBruijnGraph::Mode at the boundary: BASIC, CANONICAL and PRIMARY (CanonicalDBG semantics) are served; what is
    not (an unknown mode, a strand mode on a protein graph) is refused with an
    error code, never silently treated as BASIC."""
    from metagraph_b200 import _lib
    from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import cli_defaults
    boss = BOSSTable.from_sequences(5, ["AGCTTCGAGGCCAATTGACCGT"], lib=EMU)
    assert DBGSuccinctIndex(boss, lib=EMU, mode=1).mode == 1
    with pytest.raises(_lib.MgbError) as e:
        DBGSuccinctIndex(boss, lib=EMU, mode=3)
    assert e.value.code == -1                                           # MGB_ERR_INVALID_ARGUMENT
    idx = DBGSuccinctIndex(boss, lib=EMU, mode=2)
    B200Aligner(idx, cli_defaults(5)).align("AGCTTCGAGG")
    B200Aligner(idx, cli_defaults(5, min_seed_length=3)).align("AGCTTCGAGG")
    prot = BOSSTable.from_sequences(3, ["MKVLAAGIVGLLLAQ"], alphabet=1, lib=EMU)
    with pytest.raises(_lib.MgbError) as e:
        DBGSuccinctIndex(prot, lib=EMU, mode=1)
    assert e.value.code == -3                                           # MGB_ERR_BAD_CONFIG


@pytest.mark.parametrize("k", [43, 64, 85])
def test_boss_build_large_k(k):
    """mgb_boss_build beyond 128-bit packed k-mers (256-bit keys): same W / last / F as the oracle's constructor,
    which reproduces the reference-built graph files with either key width (MGO_FORCE_U256, MGB_TEST_WIDE_KEYS)."""
    import numpy as np
    import oracle_lib as O
    from metagraph_b200.aligner import BOSSTable
    rng = np.random.default_rng(k)
    seqs = ["".join(np.array(list("ACGT"))[rng.integers(0, 4, 700)]) for _ in range(3)]
    seqs.append(seqs[0][100:300] + "N" + seqs[1][50:250])
    boss = BOSSTable.from_sequences(k, seqs, lib=EMU)
    W, last, F, valid = O.OracleGraph(k, seqs, mask=True).arrays()
    assert (boss.W == W).all() and (boss.last == last).all() and (boss.F == F).all()
    assert (boss.dummy_mask(lib=EMU) == valid).all()


@pytest.mark.parametrize("case", P.WHOLE_READ_CASES, ids=[str(c[0]) for c in P.WHOLE_READ_CASES])
def test_whole_read_shortcut_emu(case):
    seed, k, cfgf, may = case
    hits = P.whole_read_case(EMU, seed, k, cfgf(k))
    assert (hits > 10) if may else (hits == 0), hits


def test_bad_min_cell_score_emu():
    """tests/graph/test_aligner.cpp:85-92 (bad_min_cell_score): the aligner's constructor throws for a configuration
    whose min_cell_score + lowest penalty underflows — here at construction too (mgb_config_check), with the
    reference's message, and the restatement agrees."""
    import oracle_lib as O
    from metagraph_b200 import _lib
    from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import INT32_MIN, dna_scoring_matrix, struct_defaults
    cfg = struct_defaults(score_matrix=dna_scoring_matrix(2, -1, -2), min_cell_score=INT32_MIN, min_path_score=INT32_MIN)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(3, [], lib=EMU), lib=EMU)      # build_graph_batch(3, {})
    with pytest.raises(_lib.MgbError, match="sum of min_cell_score and lowest penalty too low") as e:
        B200Aligner(idx, cfg)
    assert e.value.code == -3                                                       # MGB_ERR_BAD_CONFIG
    with pytest.raises(RuntimeError, match="sum of min_cell_score and lowest penalty too low"):
        O.OracleGraph(3, []).align_tsv(cfg, ["ACGT"])
    B200Aligner(idx, struct_defaults(score_matrix=dna_scoring_matrix(2, -1, -2)))   # the same graph with a sane config
    idx.close()


@pytest.mark.parametrize("name", P.PRESSURE_INPUTS)
def test_pressure_inputs_reach_their_paths_emu(name):
    """Each pressure input reaches the spill / migration / retry path it is built for (the emulation counts the
    aligner's sites), and the emulation equals the oracle on it. test_spill_paths_gpu.py runs the same bytes on the
    device, where the lanes of a warp share the copies to the arena."""
    stats, hits = P.pressure_case(EMU, name)
    for path in P.PRESSURE_TARGETS[name]:
        assert hits[path] > 0, (name, path, hits)
    if name == "retry":
        assert 0 < stats["num_reads_retried"] < len(P.pressure_input(name)[2]), stats


@pytest.mark.parametrize("name", P.PRESSURE_INPUTS)
def test_spill_knobs_emu(name, monkeypatch):
    """The knob matrix of test_spill_paths_gpu.py on the emulation: every run equals the oracle and the default run's
    DP counters, and the knobs that move an on-chip limit reach the path they move it to."""
    hits = {knob: h for knob, (_, h) in P.pressure_knob_matrix(EMU, name, monkeypatch).items()}
    assert hits["bmax64"]["arena_column"] > 0
    assert 0 < hits["lq_split"]["unstaged_read"] < hits["lq0"]["unstaged_read"]
    if name in ("queue", "retry"):                # the insertion and wide-band inputs never queue two columns
        assert hits["hcap1"]["queue_migrate"] > hits["hcap4"]["queue_migrate"] > hits["default"]["queue_migrate"]
        assert hits["nofast"]["general_column"] > hits["default"]["general_column"]
