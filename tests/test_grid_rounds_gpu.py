"""The read-path kernels past their first grid round. k_prepare, k_prepare_exact, k_premap, k_seed, k_seed_hash, k_subk,
k_exact_reads and k_align loop over their work with persistent or grid-stride loops; a round after the first reuses
shared tiles, a warp's arena and on-chip working set, and lanes of one warp can be in different rounds. The suite's
inputs otherwise fit into one round of every kernel.

Two ways to get further rounds, each checked line for line (node paths included) against the oracle:
- MGB_TEST_MAX_BLOCKS=n caps the grid of every read-path kernel at n blocks. The existing inputs run at n = 1 and n = 3
  (with three blocks the last round runs in only some of the blocks and ends partway through a tile), with read
  counts raised where a driver takes one.
- Batches of C3 and C2 shape at the default grid, where the real sizes give the rounds.
Each test names the kernels it targets and proves from the MGB_DEBUG launch lines that each ran at least two rounds
(items over the items one round of the launch covers); in the capped runs k_align's warps average at least four reads.
State carried from one read to the next (a convergence epoch, arena scratch, aggregator entries) can change how much DP
runs without changing a reported alignment, so every capped alignment call must also have the COUNTERS of the same call
at the default grid.
"""
import os
import re

import numpy as np
import pytest

import oracle_lib as O
import parity_common as P
import test_prepare_exact_gpu as PE
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
from metagraph_b200.config import cli_defaults
from test_exact_reads_gpu import COUNTERS, L, Case, substitute
from test_path_seed_gpu import boundary_reads, make_graph
from test_seed_hash_gpu import mixed_reads

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)

CAPS = (1, 3)
N_READS = 1000     # > 3 blocks x 256 reads: two rounds of the per-lane kernels at both caps

LAUNCH = re.compile(r"launch (\w+) grid=(\d+) block=(\d+) per_round=(\d+) items=(\d+|dev)")
LEFT_OVER = re.compile(r"k_prepare_exact answered \d+, left over (\d+)")


def launches(err):
    """[(kernel, grid, items one round covers, items)] of the MGB_DEBUG lines. A list the device holds (the reads
    k_prepare_exact left over) counts as the shortest such list of the call's pieces."""
    left = [int(n) for n in LEFT_OVER.findall(err)]
    out = []
    for name, grid, _, per_round, items in LAUNCH.findall(err):
        n = int(items) if items != "dev" else min(left, default=0)
        out.append((name, int(grid), int(per_round), n))
    return out


def rounds(err):
    """kernel -> the most rounds one of its launches ran"""
    r = {}
    for name, _, per_round, n in launches(err):
        r[name] = max(r.get(name, 0), -(-n // per_round))
    return r


def reads_per_warp(err):
    """reads per warp of k_align's largest launch"""
    n, warps = max((n, per_round) for name, _, per_round, n in launches(err) if name == "k_align")
    return n / warps


def assert_reach(err, targets, cap=None, per_warp=4):
    """every target kernel ran >= 2 rounds; capped: no launch above `cap` blocks, and k_align's warps average
    >= per_warp reads"""
    r = rounds(err)
    short = {t: r.get(t, 0) for t in targets if r.get(t, 0) < 2}
    assert not short, (short, r)
    if cap is not None:
        over = [l for l in launches(err) if l[1] > cap]
        assert not over, over[:3]
        if "k_align" in targets and per_warp:
            assert reads_per_warp(err) >= per_warp, (reads_per_warp(err), r)
    return r


def traced(monkeypatch, capfd, fn, env):
    """fn() under the environment `env` with MGB_DEBUG on: (its result, the MGB_DEBUG lines)"""
    with monkeypatch.context() as mp:
        mp.setenv("MGB_DEBUG", "1")
        for var, val in env.items():
            mp.setenv(var, val)
        capfd.readouterr()
        out = fn()
        err = capfd.readouterr().err
    return out, err


def capped(blocks, **env):
    return dict(env, MGB_TEST_MAX_BLOCKS=str(blocks))


def counted(monkeypatch, capfd, fn, env):
    """traced(fn) that also records the COUNTERS of every alignment call of the parity drivers (parity_common.run_lines):
    (result, MGB_DEBUG lines, [counters])"""
    calls = []
    run_lines = P.run_lines

    def recorded(*args, **kw):
        lines, stats = run_lines(*args, **kw)
        calls.append({c: stats[c] for c in COUNTERS})
        return lines, stats
    with monkeypatch.context() as mp:
        mp.setattr(P, "run_lines", recorded)
        out, err = traced(mp, capfd, fn, env)
    return out, err, calls


_default_grid = {}     # input -> the counters of its alignment calls at the default grid (both caps compare with them)


def grid_checked(key, monkeypatch, capfd, fn, blocks, env=None):
    """fn() with the grid capped at `blocks`: (result, MGB_DEBUG lines). Its alignment calls have the counters of the
    same calls at the default grid."""
    env = env or {}
    out, err, calls = counted(monkeypatch, capfd, fn, capped(blocks, **env))
    if key not in _default_grid:
        _default_grid[key] = counted(monkeypatch, capfd, fn, env)[2]
    assert calls == _default_grid[key], (key, blocks, calls, _default_grid[key])
    return out, err


def assert_default_grid_counters(runs, g, cfg, reads, monkeypatch, capfd):
    """test_prepare_exact_gpu.check's capped runs (route on and off, no node ids): the counters of the route-on run at the
    default grid"""
    with monkeypatch.context() as mp:
        mp.delenv("MGB_TEST_MAX_BLOCKS")
        base = PE.run(g.idx, cfg, reads, True, mp, capfd)[1]
    assert runs[0][1] == base and runs[1][1] == base, (runs[0][1], runs[1][1], base)


def exact_gate(cfg, k):
    """the configuration part of the whole-read exact answers (k_exact_reads, k_prepare_exact)"""
    return (cfg.min_seed_length == k and cfg.max_seed_length == k and cfg.forward_and_reverse_complement
            and not cfg.seed_complexity_filter and cfg.min_exact_match <= 1.0)


def seeding_targets(cfg, k):
    """the kernels an alignment call on a DNA graph with the k-mer hash index and path layout runs"""
    t = ["k_align"]
    if cfg.max_seed_length >= k and cfg.min_seed_length < k:
        t.append("k_subk")
    if cfg.max_seed_length >= k:
        t.append("k_seed_hash")
    t.append("k_prepare_exact" if exact_gate(cfg, k) else "k_prepare")
    return t


def exact_targets(cfg, k, route_off):
    """targets of a batch of mostly exact reads: with the exact gate the reads are answered ahead of k_align, by
    k_prepare_exact (its list of reads left over is short) or, with the route off, by k_exact_reads"""
    if not exact_gate(cfg, k):
        return set(seeding_targets(cfg, k))
    return {"k_prepare", "k_seed_hash", "k_exact_reads"} if route_off else {"k_prepare_exact"}


# ---------------------------------------------------------------------------------------------------------------------
# capped grids on the existing inputs

@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("case", P.RANDOM_CASES, ids=[str(c[0]) for c in P.RANDOM_CASES])
def test_random_grid_gpu(case, blocks, monkeypatch, capfd):
    """sub-k seeds, masked graphs, the device suffix levels; map_to_nodes through k_prepare and k_seed_hash"""
    seed, k, G, n, L_, rate, cfgf, mask, nseq = case
    cfg = cfgf(k)
    _, err = grid_checked(("random", seed), monkeypatch, capfd,
                          lambda: P.random_case(LIB, seed, k, G, max(n, N_READS), L_, rate, cfg, mask, nseq), blocks)
    assert_reach(err, set(seeding_targets(cfg, k)) | {"k_prepare", "k_seed_hash"}, blocks)


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("case", P.RANDOM_CASES, ids=[str(c[0]) for c in P.RANDOM_CASES])
def test_random_no_kmer_hash_grid_gpu(case, blocks, monkeypatch, capfd):
    """the same without the k-mer hash index: k_premap and k_seed"""
    seed, k, G, n, L_, rate, cfgf, mask, nseq = case
    cfg = cfgf(k)
    _, err = grid_checked(("random_no_kmer_hash", seed), monkeypatch, capfd,
                          lambda: P.random_case(LIB, seed, k, G, max(n, N_READS), L_, rate, cfg, mask, nseq), blocks,
                          {"MGB_NO_KMER_HASH": "1"})
    targets = {"k_prepare", "k_seed", "k_align"} | ({"k_premap"} if k >= 11 else set())
    if cfg.max_seed_length >= k and cfg.min_seed_length < k:
        targets.add("k_subk")
    if exact_gate(cfg, k):
        targets.add("k_exact_reads")         # without the hash index: from the node arrays, every read listed
    r = assert_reach(err, targets, blocks)
    assert "k_seed_hash" not in r and "k_prepare_exact" not in r, r


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("case", P.PROTEIN_CASES, ids=[str(c[0]) for c in P.PROTEIN_CASES])
def test_protein_grid_gpu(case, blocks, monkeypatch, capfd):
    """the alphabet-generic layout (its own compilation of k_prepare's successors: k_seed, k_subk, k_align)"""
    seed, k, G, n, L_, rate, cfgf, mask, nseq, indel = case
    cfg = cfgf(k)
    _, err = grid_checked(("protein", seed), monkeypatch, capfd,
                          lambda: P.protein_case(LIB, seed, k, G, max(n, N_READS), L_, rate, cfg, mask, nseq, indel), blocks)
    targets = {"k_prepare", "k_seed", "k_align"} | ({"k_subk"} if cfg.min_seed_length < k else set())
    assert_reach(err, targets, blocks)


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("case", P.WHOLE_READ_CASES, ids=[str(c[0]) for c in P.WHOLE_READ_CASES])
def test_whole_read_grid_gpu(case, blocks, monkeypatch, capfd):
    """whole-read exact answers, k_prepare_exact on and off: k_exact_reads gets every read when it is off"""
    seed, k, cfgf, _ = case
    cfg = cfgf(k)
    for env in ({}, {"MGB_TEST_NO_PREPARE_EXACT": "1"}):
        _, err = grid_checked(("whole_read", seed, bool(env)), monkeypatch, capfd,
                              lambda: P.whole_read_case(LIB, seed, k, cfg, n_path=N_READS), blocks, env)
        assert_reach(err, exact_targets(cfg, k, bool(env)), blocks)


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("case", P.EXACT_SHORTCUT_CASES, ids=[str(c[0]) for c in P.EXACT_SHORTCUT_CASES])
def test_exact_shortcut_grid_gpu(case, blocks, monkeypatch, capfd):
    seed, k, cfgf = case
    cfg = cfgf(k)
    for env in ({}, {"MGB_TEST_NO_PREPARE_EXACT": "1"}):
        _, err = grid_checked(("exact_shortcut", seed, bool(env)), monkeypatch, capfd,
                              lambda: P.exact_shortcut_case(LIB, seed, k, cfg, nreads=N_READS), blocks, env)
        # (the reads with errors, a quarter, reach k_align also when the others are answered ahead of it)
        assert_reach(err, exact_targets(cfg, k, bool(env)) | {"k_align"}, blocks)


@pytest.mark.parametrize("blocks", CAPS)
def test_prepare_exact_mixed_grid_gpu(blocks, monkeypatch, capfd):
    """the mixed reads of test_prepare_exact_gpu.py, drawn 19 times (> 1000 reads); the reads the route answered still
    equal the host restatement of its gate"""
    case = Case(31, 1831)
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = [r for _ in range(19) for r in case.mixed_reads()]
    runs = []
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    n = PE.check(g, reads, monkeypatch, capfd, runs=runs)
    assert 0 < n < len(reads)
    for run in runs[::2]:
        assert_reach(run[3], {"k_prepare_exact", "k_align"}, blocks)
    for run in runs[1::2]:
        assert_reach(run[3], {"k_prepare", "k_seed_hash", "k_exact_reads", "k_align"}, blocks)
    assert_default_grid_counters(runs, g, case.cfg, reads, monkeypatch, capfd)
    g.close()


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("n", [N_READS, 2 * 256 * 3 + 1])
def test_prepare_exact_tiles_grid_gpu(n, blocks, monkeypatch, capfd):
    """batches whose last round ends partway through a tile, or one read into a new round"""
    case = Case(31, 2200)
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(n)
    for i in range(0, n, 97):
        reads[i] = substitute(reads[i], (7 * i) % L)
    runs = []
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    PE.check(g, reads, monkeypatch, capfd, runs=runs)
    for run in runs[::2]:
        assert_reach(run[3], {"k_prepare_exact"}, blocks)
    for run in runs[1::2]:
        assert_reach(run[3], {"k_prepare", "k_seed_hash", "k_exact_reads"}, blocks)
    assert_default_grid_counters(runs, g, case.cfg, reads, monkeypatch, capfd)
    g.close()


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("kind,k", PE.CASES, ids=["%s-k%d" % c for c in PE.CASES])
def test_prepare_exact_path_ends_grid_gpu(kind, k, blocks, monkeypatch, capfd):
    """reads that start, end or cross where a path of the layout ends"""
    rng = np.random.default_rng(2100 + 10 * PE.CASES.index((kind, k)))
    pg = make_graph(kind, k, rng)
    g = PE.Graph(k, pg.seqs, monkeypatch)
    reads = boundary_reads(rng, pg)
    while len(reads) < N_READS:
        reads = reads + boundary_reads(rng, pg)
    reads = [reads[int(i)] for i in rng.permutation(len(reads))[:N_READS]]
    runs = []
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    n = PE.check(g, reads, monkeypatch, capfd, runs=runs)
    assert 0 < n < len(reads)
    for run in runs[::2]:
        assert_reach(run[3], {"k_prepare_exact"}, blocks)
    for run in runs[1::2]:
        assert_reach(run[3], {"k_prepare", "k_seed_hash", "k_exact_reads"}, blocks)
    assert_default_grid_counters(runs, g, cli_defaults(k, min_seed_length=k, max_seed_length=k), reads, monkeypatch,
                                 capfd)
    g.close()


@pytest.mark.parametrize("blocks", CAPS)
def test_prepare_exact_heap_full_grid_gpu(blocks, monkeypatch, capfd):
    """pass 0's heap holds no record, then room for some: the reads left over go round k_seed_hash, k_exact_reads (which
    overflow) and the retry pass"""
    case = Case(31, 2400)
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(N_READS)
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    monkeypatch.setenv("MGB_TEST_HEAP0", "64")
    runs = []
    PE.check(g, reads, monkeypatch, capfd, expect=0, runs=runs)
    for run in runs:
        assert_reach(run[3], {"k_seed_hash", "k_exact_reads"}, blocks)
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    assert_default_grid_counters(runs, g, cfg, reads, monkeypatch, capfd)
    # records of equal size: how many fit into the heap does not depend on the order they are allocated in
    monkeypatch.setenv("MGB_TEST_HEAP0", str(300 * 400))
    run = PE.run(g.idx, cfg, reads, True, monkeypatch, capfd)
    lines, stats, n, err = run
    assert lines == g.og.align_tsv(cfg, reads, with_nodes=True)
    assert 0 < n < len(reads) and stats["num_reads_retried"] > 0
    assert_reach(err, {"k_prepare_exact"}, blocks)
    assert_default_grid_counters([run, run], g, cfg, reads, monkeypatch, capfd)
    g.close()


# (seeds 205 and 212 draw configurations that take minutes at one block)
FUZZ = [(m, s, None) for m in ("basic", "canonical", "primary") for s in (200, 201, 202, 203, 204, 206, 207, 208, 209,
                                                                          210, 211, 215, 216)] + \
       [(m, s, k) for m in ("basic", "canonical", "primary") for s, k in ((213, 47), (214, 64))]


@pytest.mark.parametrize("mode,seed,k", FUZZ, ids=["%s-%d-%s" % f for f in FUZZ])
def test_fuzz_grid_gpu(mode, seed, k, monkeypatch, capfd):
    """randomized triples (parity_common.fuzz_case) with 800 reads (> 3 x 256), at one block (even seeds) or three"""
    blocks = 1 if seed % 2 == 0 else 3
    (bad, info), err = grid_checked(("fuzz", mode, seed, k), monkeypatch, capfd,
                                    lambda: P.fuzz_case(LIB, seed, canonical=mode == "canonical", primary=mode == "primary",
                                                        k=k, nreads=800, threads=os.cpu_count() or 1), blocks)
    assert not bad, (seed, info)
    if info is not None:                       # (None: the configuration is refused, as by the reference)
        k_, kw = info[0], info[1]
        gate = mode == "basic" and exact_gate(cli_defaults(k_, **kw), k_)
        # with the exact gate, error-free reads are answered ahead of k_align
        targets = {"k_prepare_exact"} if gate else {"k_prepare", "k_align"}
        assert_reach(err, targets, blocks, per_warp=4 if blocks == 1 else 0)


@pytest.mark.parametrize("blocks", CAPS)
def test_mt_grid_gpu(blocks, monkeypatch, capfd):
    """the MT goldens on CANONICAL and PRIMARY graphs. Seven reads: at one block k_align's four warps go round twice and
    the PRIMARY check's 16 probes take k_prepare round twice. At three blocks no kernel goes round twice (the inputs
    are fixed): only the lines and counters under the capped grid are checked there."""
    _, err = grid_checked(("mt_canonical",), monkeypatch, capfd, lambda: P.check_mt_canonical(LIB), blocks)
    assert_reach(err, {"k_align"} if blocks == 1 else set(), blocks, per_warp=0)
    _, err = grid_checked(("mt_primary",), monkeypatch, capfd, lambda: P.check_mt_primary(LIB), blocks)
    assert_reach(err, {"k_align", "k_prepare"} if blocks == 1 else set(), blocks, per_warp=0)


@pytest.mark.parametrize("blocks", CAPS)
@pytest.mark.parametrize("k", [31, 12])
@pytest.mark.parametrize("primary", [False, True], ids=["one_strand", "two_strands"])
def test_hashed_map_to_nodes_grid_gpu(k, primary, blocks, monkeypatch, capfd):
    """1 001 reads of 0 .. 11 666 bp with N characters through map_to_nodes_sequentially: lanes whose reads end early
    reach the path-run copy of k_seed_hash while others of the warp are still in an earlier round"""
    rng = np.random.default_rng(500 + k + primary)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, 14000)])
    seqs = [base, P.mutate(rng, base, 0.02)]
    g = O.OracleGraph(k, P.primary_contigs(seqs, k) if primary else seqs, mask=False)
    if primary:
        g.set_mode(2)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), mode=2 if primary else 0)
    reads = mixed_reads(rng, seqs, k, 1001)
    got, err = traced(monkeypatch, capfd, lambda: idx.map_to_nodes_sequentially(reads), capped(blocks))
    idx.close()
    bad = [i for i, (r, n) in enumerate(zip(reads, got)) if list(n) != list(g.map_to_nodes(r))]
    assert not bad, (len(bad), len(reads[bad[0]]), reads[bad[0]][:80])
    assert_reach(err, {"k_prepare", "k_seed_hash"}, blocks)


def test_pieces_grid_gpu(monkeypatch, capfd):
    """three pieces on two host threads, each with three blocks per kernel"""
    seed, k, G, n, L_, rate, cfgf, mask, nseq = P.RANDOM_CASES[3]
    cfg = cfgf(k)
    _, err = grid_checked(("pieces",), monkeypatch, capfd,
                          lambda: P.random_case(LIB, seed, k, G, 3 * N_READS, L_, rate, cfg, mask, nseq), 3,
                          {"MGB_TEST_PIECES": "3"})
    assert_reach(err, {"k_prepare", "k_subk", "k_seed_hash", "k_align"}, 3)
    assert len([l for l in launches(err) if l[0] == "k_align"]) >= 3


def test_grid1_knob_reach_gpu(monkeypatch, capfd):
    """the grid1 knob of parity_common.SPILL_KNOBS puts every read of a pressure input through k_align's four warps"""
    env = dict(P.SPILL_KNOBS)["grid1"]
    _, err = traced(monkeypatch, capfd, lambda: P.pressure_case(LIB, "queue"), env)
    assert max(l[1] for l in launches(err)) == 1
    assert_reach(err, {"k_align", "k_prepare"}, 1)


# ---------------------------------------------------------------------------------------------------------------------
# C3 and C2 shapes at the default grid

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, np.uint8)
COMP[list(b"ACGTN")] = list(b"TGCAN")


def mutate_rows(rng, rows, rate):
    """per base with probability `rate` an error: 80 % substitution, 10 % insertion after it, 10 % deletion (the
    split of parity_common.mutate), for a matrix of equal-length reads; returns the reads as str"""
    n, m = rows.shape
    ev = rng.random((n, m)) < rate
    kind = rng.random((n, m))
    sub, ins, dele = ev & (kind < 0.8), ev & (kind >= 0.8) & (kind < 0.9), ev & (kind >= 0.9)
    rows = np.where(sub, ACGT[rng.integers(0, 4, (n, m))], rows)
    pair = np.stack([rows, ACGT[rng.integers(0, 4, (n, m))]], axis=2).reshape(n, 2 * m)
    keep = np.stack([~dele, ins], axis=2).reshape(n, 2 * m)
    flat = pair[keep]
    ends = np.cumsum(keep.sum(axis=1))
    starts = ends - keep.sum(axis=1)
    raw = flat.tobytes().decode()
    return [raw[s:e] for s, e in zip(starts.tolist(), ends.tolist())]


def c3_genome(rng, G):
    """a random genome with tandem repeats, and three copies of it with 1 % substitutions"""
    g = ACGT[rng.integers(0, 4, G)]
    for p in rng.integers(0, G - 400, 40):
        unit = ACGT[rng.integers(0, 4, int(rng.integers(2, 9)))]
        rep = np.tile(unit, 300 // len(unit) + 1)[:300]
        g[p:p + 300] = rep
    copies = [g]
    for _ in range(3):
        c = g.copy()
        at = rng.random(G) < 0.01
        c[at] = ACGT[rng.integers(0, 4, int(at.sum()))]
        copies.append(c)
    return copies


def sample_reads(rng, copies, n, length):
    """n windows of `length` bp from the copies, every second one reverse complemented"""
    src = rng.integers(0, len(copies), n)
    pos = rng.integers(0, len(copies[0]) - length, n)
    idx = pos[:, None] + np.arange(length)[None, :]
    rows = np.stack(copies)[src[:, None], idx]
    rc = COMP[rows[1::2, ::-1]]
    rows[1::2] = rc
    return rows


def scale_index(copies, k):
    seqs = np.concatenate(copies)
    offs = np.cumsum([0] + [len(c) for c in copies]).astype(np.uint64)
    boss = BOSSTable.from_sequences(k, None, packed=(seqs, offs))
    return boss, DBGSuccinctIndex(boss)


def compare_with_oracle(boss, k, cfg, reads, results, chunk=50000):
    """results == the oracle's lines, node paths included, in chunks (the oracle on all host cores)"""
    o = O.OracleGraph(k, arrays=(boss.W, boss.last, boss.F))
    threads = os.cpu_count() or 1
    for lo in range(0, len(reads), chunk):
        exp = o.align_tsv(cfg, reads[lo:lo + chunk], with_nodes=True, threads=threads)
        got = [format_alignment("", r, cfg.min_path_score, with_nodes=True) for r in results[lo:lo + chunk]]
        bad = [i for i in range(len(exp)) if exp[i] != got[i]]
        assert not bad, (lo + bad[0], len(bad), exp[bad[0]][:300], got[bad[0]][:300])


def aligned(idx, cfg, reads, monkeypatch, capfd, env):
    """(results, counters, MGB_DEBUG lines) of one call"""
    def call():
        al = B200Aligner(idx, cfg)
        return al.align_batch([("", r) for r in reads]), al.last_stats
    (res, stats), err = traced(monkeypatch, capfd, call, env)
    return res, {c: stats[c] for c in COUNTERS}, err


def test_c3_shape_gpu(monkeypatch, capfd):
    """k = 31, a 2 Mbp genome with tandem repeats in four 1 %-diverged copies; 200 k reads of 150 bp with 5 % errors,
    half reverse complemented, the odd N and short read; CLI defaults with min_exact_match = 0 (sub-k seeds). Default
    pieces (three, on two host threads) and one piece: k_prepare, k_subk and k_align go round many times, k_seed_hash
    about three times in one piece."""
    k, G, n = 31, 2_000_000, 200_000
    rng = np.random.default_rng(3003)
    copies = c3_genome(rng, G)
    boss, idx = scale_index(copies, k)
    reads = mutate_rows(rng, sample_reads(rng, copies, n, 150), 0.05)
    del copies
    for i in range(0, n, 500):
        r = reads[i]
        reads[i] = r[:len(r) // 3] + "N" + r[len(r) // 3 + 1:]
    for i in range(250, n, 5000):
        reads[i] = reads[i][:int(rng.integers(0, 40))]
    cfg = cli_defaults(k, min_exact_match=0.0)
    res_p, cnt_p, err_p = aligned(idx, cfg, reads, monkeypatch, capfd, {})
    res_1, cnt_1, err_1 = aligned(idx, cfg, reads, monkeypatch, capfd, {"MGB_TEST_PIECES": "1"})
    idx.close()
    assert cnt_p == cnt_1
    assert len([l for l in launches(err_p) if l[0] == "k_align"]) >= 3
    assert_reach(err_p, {"k_prepare", "k_subk", "k_align"})
    assert_reach(err_1, {"k_prepare", "k_subk", "k_seed_hash", "k_align"})
    assert reads_per_warp(err_1) >= 20, reads_per_warp(err_1)
    same = [i for i in range(n) if format_alignment("", res_p[i], 0, with_nodes=True)
            != format_alignment("", res_1[i], 0, with_nodes=True)]
    assert not same, same[:3]
    del res_1
    compare_with_oracle(boss, k, cfg, reads, res_p)


def test_c2_shape_mixed_gpu(monkeypatch, capfd):
    """k = 31 exact seeder on a 2 Mbp genome; 300 k reads of 150 bp, 90 % error-free, 10 % with one substitution or an
    N. In one piece k_prepare_exact goes round twice and its left-over list feeds k_seed_hash, k_exact_reads and
    k_align; then with default pieces."""
    k, G, n = 31, 2_000_000, 300_000
    rng = np.random.default_rng(2002)
    genome = ACGT[rng.integers(0, 4, G)]
    boss, idx = scale_index([genome], k)
    rows = sample_reads(rng, [genome], n, 150)
    hit = np.flatnonzero(rng.random(n) < 0.1)
    at = rng.integers(0, 150, len(hit))
    is_n = rng.random(len(hit)) < 0.3
    rows[hit, at] = np.where(is_n, ord("N"), ACGT[(np.searchsorted(ACGT, rows[hit, at]) + 1) % 4])
    raw = rows.tobytes().decode()
    reads = [raw[150 * i:150 * (i + 1)] for i in range(n)]
    cfg = cli_defaults(k, min_seed_length=k, max_seed_length=k)
    res_1, cnt_1, err_1 = aligned(idx, cfg, reads, monkeypatch, capfd, {"MGB_TEST_PIECES": "1"})
    assert_reach(err_1, {"k_prepare_exact"})
    assert {"k_seed_hash", "k_exact_reads", "k_align"} <= set(rounds(err_1)), rounds(err_1)
    res_p, cnt_p, _ = aligned(idx, cfg, reads, monkeypatch, capfd, {})
    idx.close()
    assert cnt_p == cnt_1
    for lo in range(0, n, 50000):
        assert ([format_alignment("", r, 0, with_nodes=True) for r in res_p[lo:lo + 50000]]
                == [format_alignment("", r, 0, with_nodes=True) for r in res_1[lo:lo + 50000]]), lo
    del res_p
    compare_with_oracle(boss, k, cfg, reads, res_1)
