"""k_prepare_exact with its tiles staged in shared memory and the gate decided on packed 2-bit words: read lengths around
the word and tile boundaries (tile starts at every alignment mod 16), tiles too long to stage (read from global memory),
invalid bytes at every position mod 32, both strands, records with and without node ids, blocks that go round several
times (MGB_TEST_MAX_BLOCKS) and a heap that fills partway through a tile. Every case: oracle == route on == route off,
counters included, and the reads the route answered == the restated gate (test_prepare_exact_gpu.Graph)."""
import dataclasses
import re

import numpy as np
import pytest

from metagraph_b200.config import cli_defaults
from test_exact_reads_gpu import Case
from test_oracle_golden import revcomp
from test_prepare_exact_gpu import Graph, check, run

pytestmark = pytest.mark.gpu

TILE = 256
STAGE_MAX = 45 * 1024            # kernels.cuh kPrepStageMax


def lengths(k):
    return [k - 1, k, k + 1, 32, 33, 63, 64, 65, 150, 216, 217, 511]


def slices(case, rng, lens):
    """reads of the given lengths from the genome, every other one reverse complemented"""
    out = []
    for i, n in enumerate(lens):
        p = int(rng.integers(1200, len(case.base) - n))
        r = case.base[p:p + n]
        out.append(revcomp(r) if i % 2 else r)
    return out


def tiled_lengths(k, rng, tiles):
    """read lengths for `tiles` tiles of 256 reads whose byte ranges start at 0, 1, 2, ... mod 16"""
    lens = []
    for _ in range(tiles):
        t = [int(x) for x in rng.choice(lengths(k), TILE - 1)]
        last = 150 + (1 - sum(t) - 150) % 16            # the tile's bytes: 1 mod 16
        lens += t + [last]
    return lens


def rounds(err):
    """per k_prepare_exact launch: reads / reads per round (> 1: a second round)"""
    return [int(m[1]) / int(m[0]) for m in re.findall(r"launch k_prepare_exact grid=\d+ block=256 per_round=(\d+) items=(\d+)", err)]


@pytest.mark.parametrize("k", [31, 15])
def test_staged_lengths_gpu(k, monkeypatch, capfd):
    """lengths k - 1 .. 511 mixed, 16 tiles starting at every alignment mod 16, a few reads with a substitution"""
    case = Case(k, 2600 + k)
    rng = np.random.default_rng(2610 + k)
    g = Graph(k, case.seqs, monkeypatch)
    lens = tiled_lengths(k, rng, 16)
    starts = np.concatenate([[0], np.cumsum(lens)])[::TILE]
    assert len(set(int(s) % 16 for s in starts[:16])) == 16
    reads = slices(case, rng, lens)
    for i in rng.choice(len(reads), 40, replace=False):
        r = reads[i]
        j = int(rng.integers(0, len(r)))
        reads[i] = r[:j] + "ACGT"[("ACGT".index(r[j]) + 1) % 4] + r[j + 1:]
    n = check(g, reads, monkeypatch, capfd)
    assert 0 < n < len(reads)
    g.close()


def test_staged_fallback_tiles_gpu(monkeypatch, capfd):
    """511 bp reads among 150 bp ones: the first tile is longer than the staging budget and is read from global memory,
    the second one is staged"""
    case = Case(31, 2700)
    rng = np.random.default_rng(2701)
    lens = [511 if i % 6 == 0 else 150 for i in range(TILE)] + [511 if i % 30 == 0 else 150 for i in range(TILE)]
    tile_bytes = [sum(lens[:TILE]), sum(lens[TILE:])]
    assert tile_bytes[0] > STAGE_MAX and tile_bytes[1] + 80 < STAGE_MAX
    g = Graph(31, case.seqs, monkeypatch)
    reads = slices(case, rng, lens)
    n = check(g, reads, monkeypatch, capfd)
    assert n > len(reads) // 2
    g.close()


BAD = ["N", "lower", "\x00", "\xc1", "\xff"]


@pytest.mark.parametrize("bad", BAD, ids=["N", "lower", "nul", "c1", "ff"])
def test_staged_invalid_bytes_gpu(bad, monkeypatch, capfd):
    """one byte replaced at the first and the last position and at a position of every residue mod 32, on both strands
    (lower case is a valid byte: those reads are answered)"""
    case = Case(31, 2800)
    rng = np.random.default_rng(2801)
    g = Graph(31, case.seqs, monkeypatch)
    base = case.exact_reads(2 * 34)
    reads = []
    for i, r in enumerate(base):
        m = i // 2
        j = 0 if m == 32 else len(r) - 1 if m == 33 else m + 32 * int(rng.integers(0, (len(r) - 1 - m) // 32 + 1))
        c = r[j].lower() if bad == "lower" else bad
        reads.append(r[:j] + c + r[j + 1:])
    reads += case.exact_reads(20)
    if bad in ("N", "lower"):
        n = check(g, reads, monkeypatch, capfd)
    else:
        # bytes the oracle's C strings cannot carry: route on == route off, and the reads answered
        raw = [r.encode("latin1") for r in reads]
        n = g.expected(reads)
        cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
        for result_nodes in (0, 1):
            c = dataclasses.replace(cfg, result_nodes=result_nodes)
            on = run(g.idx, c, raw, True, monkeypatch, capfd)
            off = run(g.idx, c, raw, False, monkeypatch, capfd)
            assert on[0] == off[0] and on[1] == off[1]
            assert on[2] == n
    if bad == "lower":
        assert n == g.expected(base + reads[len(base):])
    else:
        assert n == g.expected(reads[len(base):]) and not any(g.answered(r, 511) for r in reads[:len(base)])
    g.close()


@pytest.mark.parametrize("blocks", [1, 3])
def test_staged_block_rounds_gpu(blocks, monkeypatch, capfd):
    """at most 1 / 3 blocks: every block stages several tiles in turn into the same shared memory"""
    case = Case(31, 2900)
    rng = np.random.default_rng(2901 + blocks)
    g = Graph(31, case.seqs, monkeypatch)
    reads = slices(case, rng, tiled_lengths(31, rng, 4)[:1000])
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    runs = []
    check(g, reads, monkeypatch, capfd, runs=runs)
    seen = [x for on in runs[::2] for x in rounds(on[3])]
    assert seen and min(seen) > 1, seen                 # some block takes a second tile
    g.close()


def test_staged_heap_partial_gpu(monkeypatch, capfd):
    """pass 0's heap fills partway through the first tile: the reads past it are left over, prepared and seeded, and the
    results are the oracle's and the route off's, with and without node ids"""
    case = Case(31, 3000)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(300)
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    gate = [g.answered(r, 511) for r in reads]
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", "1")          # one block: the tiles allocate in order
    for result_nodes, record in ((1, 32 + 8 + 152), (0, 32 + 8 * 120 + 8 + 152)):
        cap = 100 * record + record // 2
        # the first tile's answered reads take one allocation; those past the end of the heap are left over, and so
        # is the whole second tile
        expect = sum(1 for t in range(TILE) if gate[t] and (sum(gate[:t + 1]) * record) <= cap)
        assert 90 <= expect <= 100
        monkeypatch.setenv("MGB_TEST_HEAP0", str(cap))
        c = dataclasses.replace(cfg, result_nodes=result_nodes)
        lines, stats, n, _ = run(g.idx, c, reads, True, monkeypatch, capfd)
        assert lines == g.og.align_tsv(cfg, reads, with_nodes=not result_nodes)
        assert n == expect, (n, expect)
        off = run(g.idx, c, reads, False, monkeypatch, capfd)
        assert off[0] == lines
    g.close()
