"""k_prepare_exact's record runs: a warp whose 32 reads are all answered with records of one size writes its headers as
16-byte chunks, each lane its own record's OutAln, and the rest of the records as one run of words, lane i taking words
i, i + 32, ...; other warps write record after record. Warps of one read length at lengths whose records take word
counts that do and do not divide 32, and whose sizes are 0 and 8 mod 16; runs that start on and off a 16-byte boundary
(after a warp with one read not answered); both strands in every warp; warps of two record sizes, and warps of lengths
that round up to one record size without node ids; a tile too long to stage (its characters read from global memory).
Every case: oracle == route on == route off, with and without node ids, counters included
(test_prepare_exact_gpu.check)."""
import numpy as np
import pytest

from test_exact_reads_gpu import Case
from test_prepare_exact_gpu import Graph, check

pytestmark = pytest.mark.gpu

WARP = 32
STAGE_MAX = 45 * 1024            # kernels.cuh kPrepStageMax


def mutate(r, rng):
    """r with one substitution away from its ends (the read is then not answered)"""
    j = int(rng.integers(5, len(r) - 5))
    return r[:j] + "ACGT"[("ACGT".index(r[j]) + 1) % 4] + r[j + 1:]


def full_warps(g, reads):
    return sum(all(g.answered(r, 511) for r in reads[i:i + WARP]) for i in range(0, len(reads), WARP))


@pytest.mark.parametrize("k", [31, 15])
def test_runs_one_length_gpu(k, monkeypatch, capfd):
    """a warp per length, every read answered (reads alternate strands within each warp)"""
    case = Case(k, 3100 + k)
    g = Graph(k, case.seqs, monkeypatch)
    lens = [k, k + 1, 32, 40, 41, 63, 100, 150, 151, 160, 249, 250, 300]
    reads = [r for n in lens for r in case.exact_reads(WARP, n)]
    assert full_warps(g, reads) >= len(lens) - 2
    n = check(g, reads, monkeypatch, capfd)
    assert n >= len(reads) - 2 * WARP
    g.close()


def test_runs_unaligned_gpu(monkeypatch, capfd):
    """a warp with one read not answered leaves the next warp's run 8 bytes past a 16-byte boundary (records of 41 bp take
    an odd number of words); warps of two lengths and a warp with every other read not answered between full ones"""
    case = Case(31, 3200)
    rng = np.random.default_rng(3201)
    g = Graph(31, case.seqs, monkeypatch)
    reads = []
    one_off = case.exact_reads(WARP, 41)
    one_off[7] = mutate(one_off[7], rng)
    reads += one_off
    for n in (41, 150, 160, 63):
        reads += case.exact_reads(WARP, n)
    reads += [r for pair in zip(case.exact_reads(WARP // 2, 150), case.exact_reads(WARP // 2, 160)) for r in pair]
    reads += case.exact_reads(WARP, 41)
    half = case.exact_reads(WARP, 100)
    reads += [mutate(r, rng) if i % 2 else r for i, r in enumerate(half)]
    reads += case.exact_reads(WARP, 160)
    assert full_warps(g, reads) >= 4
    n = check(g, reads, monkeypatch, capfd)
    assert len(reads) - WARP // 2 - 1 - 2 * WARP <= n < len(reads)
    g.close()


def test_runs_one_size_gpu(monkeypatch, capfd):
    """lengths 145 .. 152 in one warp: without node ids their records are one size (the sequence is padded to 152) and the
    warp writes one run; with node ids the sizes differ and it writes record after record"""
    case = Case(31, 3300)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(WARP, 150)
    for i in range(2 * WARP):
        reads.append(case.exact_reads(2, 145 + i % 8)[i % 2])          # both strands
    reads += case.exact_reads(WARP, 151)
    assert full_warps(g, reads) >= 3
    n = check(g, reads, monkeypatch, capfd)
    assert n >= len(reads) - WARP
    g.close()


def test_runs_unstaged_tile_gpu(monkeypatch, capfd):
    """a tile of 256 reads of 200 bp is longer than the staging budget: its warps write their runs from characters read
    from global memory; the next tile (150 bp) is staged"""
    case = Case(31, 3400)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(256, 200) + case.exact_reads(256, 150)
    assert 200 * 256 > STAGE_MAX > 150 * 256 + 80
    assert full_warps(g, reads) >= 12
    n = check(g, reads, monkeypatch, capfd)
    assert n >= len(reads) - 4 * WARP
    g.close()
