"""k_seed_hash's short-list mode (kernels.cuh seed_hash_wide): when the reads to seed are at most one per warp of the
grid, each warp looks up every k-mer of its read in the hash index at once instead of walking the read.

- Node ids from both modes, forced with MGB_TEST_SEED_MODE=walk|wide, == the oracle's map_to_nodes and == each other,
  on the mixed reads of test_seed_hash_gpu (lengths below k to 11 666 bp, N characters, errors, random sequence), at
  k = 31 and k = 12, with one strand and with two.
- Alignments after k_prepare_exact, with 0, 1, a few, exactly as many and one more left-over reads than k_seed_hash
  has warps (so the mode the kernel picks changes between the last two), at the default grid and at grids capped to 1
  and 3 blocks (MGB_TEST_MAX_BLOCKS moves the point where the mode changes): results and counters identical with the
  mode picked and forced either way, == oracle.
- A batch shaped like the benchmark's (150 bp error-free reads of a random genome, k = 31, the exact seeder) where a
  handful of reads carry one substitution, so the list left over is short: route on == route off
  (MGB_TEST_NO_PREPARE_EXACT) == oracle, in each mode and grid."""
import re

import numpy as np
import pytest

import oracle_lib as O
import parity_common as P
import test_prepare_exact_gpu as PE
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from test_exact_reads_gpu import L, Case, random_seq, substitute
from test_oracle_golden import revcomp
from test_seed_hash_gpu import mixed_reads

pytestmark = pytest.mark.gpu

MODES = ["walk", "wide"]
SEED_THREADS = 128                      # kernels.cuh kSeedThreads: 4 warps per block of k_seed_hash
LEFT = re.compile(r"k_prepare_exact answered \d+, left over (\d+)")
TO_ALIGN = re.compile(r"k_exact_reads answered \d+, left to k_align (\d+)")


@pytest.mark.parametrize("k", [31, 12])
@pytest.mark.parametrize("primary", [False, True], ids=["one_strand", "two_strands"])
def test_seed_modes_map_to_nodes_gpu(k, primary, monkeypatch):
    rng = np.random.default_rng(700 + k + primary)
    base = random_seq(rng, 14000)
    seqs = [base, P.mutate(rng, base, 0.02)]
    graph_seqs = P.primary_contigs(seqs, k) if primary else seqs
    g = O.OracleGraph(k, graph_seqs, mask=False)
    if primary:
        g.set_mode(2)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), mode=2 if primary else 0)
    reads = mixed_reads(rng, seqs, k, 1001)
    want = [list(g.map_to_nodes(r)) for r in reads]
    got = {}
    for mode in MODES:
        monkeypatch.setenv("MGB_TEST_SEED_MODE", mode)
        got[mode] = [list(n) for n in idx.map_to_nodes_sequentially(reads)]
        bad = [i for i, n in enumerate(got[mode]) if n != want[i]]
        assert not bad, (mode, len(bad), len(reads[bad[0]]), reads[bad[0]][:80])
    # a batch of one read per call: the mode the kernel picks for a grid of one block
    monkeypatch.delenv("MGB_TEST_SEED_MODE")
    for i in range(0, len(reads), 97):
        assert [list(n) for n in idx.map_to_nodes_sequentially([reads[i]])] == [want[i]], i
    assert got["walk"] == got["wide"]
    idx.close()


def run_modes(g, cfg, reads, monkeypatch, capfd):
    """PE.run with the route on, the seeding mode picked by the kernel and forced either way: the one result, counters
    and answered count they all give, and the MGB_DEBUG lines of the first"""
    out = []
    for mode in [None] + MODES:
        if mode:
            monkeypatch.setenv("MGB_TEST_SEED_MODE", mode)
        out.append(PE.run(g.idx, cfg, reads, True, monkeypatch, capfd))
        monkeypatch.delenv("MGB_TEST_SEED_MODE", raising=False)
    for o in out[1:]:
        assert o[:3] == out[0][:3]
    return out[0]


@pytest.mark.parametrize("blocks", [None, 1, 3], ids=["grid", "blocks1", "blocks3"])
@pytest.mark.parametrize("n_left", ["0", "1", "3", "warps", "warps+1"])
def test_short_list_align_gpu(n_left, blocks, monkeypatch, capfd):
    """n_left reads with a substitution among 400 reads k_prepare_exact answers; `warps`: as many as k_seed_hash's grid
    has warps (16 for 400 reads, 4 / 12 at 1 / 3 blocks). == oracle in every mode, and both gates leave exactly the
    n_left reads."""
    warps = (400 + SEED_THREADS - 1) // SEED_THREADS * 4 if blocks is None else 4 * blocks
    n = {"warps": warps, "warps+1": warps + 1}.get(n_left) or int(n_left)
    case = Case(31, 7300 + n + (blocks or 0))
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = [r for r in case.exact_reads(600) if g.answered(r, 511)][:400]     # k_prepare_exact answers all 400
    assert len(reads) == 400
    for i in range(n):
        reads[2 * i] = substitute(reads[2 * i], (11 * i + 5) % L)
    if blocks:
        monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    lines, _, _, err = run_modes(g, cfg, reads, monkeypatch, capfd)
    assert lines == g.og.align_tsv(cfg, reads, with_nodes=True)
    assert [int(x) for x in LEFT.findall(err)] == [n]
    assert [int(x) for x in TO_ALIGN.findall(err)] == [n]
    g.close()


def c2_like(rng, G, n_reads, n_err):
    """a random genome of G bp and n_reads error-free 150 bp reads of it, half of them reverse-complemented, n_err of
    them with one substitution"""
    genome = random_seq(rng, G)
    reads = []
    for i in range(n_reads):
        p = int(rng.integers(0, G - L + 1))
        r = genome[p:p + L]
        reads.append(revcomp(r) if i % 2 else r)
    for i in rng.choice(n_reads, n_err, replace=False):
        reads[i] = substitute(reads[i], int(rng.integers(0, L)))
    return genome, reads


@pytest.mark.parametrize("blocks", [None, 1, 3], ids=["grid", "blocks1", "blocks3"])
def test_short_list_c2_shape_gpu(blocks, monkeypatch, capfd):
    """3 000 reads of a 60 kbp genome, 5 with one substitution: route on == route off == oracle (with and without node
    ids in the records) with the seeding mode picked and forced either way"""
    rng = np.random.default_rng(7400 + (blocks or 0))
    genome, reads = c2_like(rng, 60000, 3000, 5)
    g = PE.Graph(31, [genome], monkeypatch)
    if blocks:
        monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    answered = None
    for mode in [None] + MODES:
        if mode:
            monkeypatch.setenv("MGB_TEST_SEED_MODE", mode)
        runs = []
        n = PE.check(g, reads, monkeypatch, capfd, runs=runs)
        monkeypatch.delenv("MGB_TEST_SEED_MODE", raising=False)
        assert n == answered or answered is None
        answered = n
        left = [int(x) for x in TO_ALIGN.findall(runs[0][3])]
        assert left and 5 <= left[0] <= 10, left
    g.close()
