"""Whole-read exact answers ahead of k_align (k_exact_reads): with the exact seeder and both strands, a read whose k-mers
are all in the graph on one strand and none on the other is answered without the aligner, from the per-read summary of
the hashed seeding kernel or, on graphs without the k-mer hash index, from the node arrays. Kernels == oracle (TSV + node
paths, and records without node ids), shortcut on == off, the counters of batches that skip k_align, and identical
results and counters with and without the hash index."""
import dataclasses

import numpy as np
import pytest

import index_tables as IT
import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
from metagraph_b200.config import cli_defaults
from test_oracle_golden import revcomp

pytestmark = pytest.mark.gpu

COUNTERS = ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns", "num_reads_retried")
L = 150


def random_seq(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def substitute(r, i):
    return r[:i] + ("A" if r[i] != "A" else "C") + r[i + 1:]


class Case:
    """a graph of a random genome, a region of it stored in both orientations and a palindrome"""

    def __init__(self, k, seed):
        self.k = k
        self.rng = np.random.default_rng(seed)
        self.base = random_seq(self.rng, 8000)
        self.region = self.base[400:1000]
        half = random_seq(self.rng, 40)
        self.pal = half + revcomp(half)                                  # its own reverse complement
        self.seqs = [self.base, revcomp(self.region), self.pal + self.base[:50]]
        self.g = O.OracleGraph(k, self.seqs, mask=False)
        self.kmers = {s[i:i + k] for s in self.seqs for i in range(len(s) - k + 1)}
        self.cfg = cli_defaults(k, min_seed_length=k, max_seed_length=k)

    def index(self, monkeypatch, hashed):
        if hashed:
            monkeypatch.delenv("MGB_NO_KMER_HASH", raising=False)
        else:
            monkeypatch.setenv("MGB_NO_KMER_HASH", "1")
        W, last, F, _ = self.g.arrays()
        boss = BOSSTable(self.k, W, last, F)
        idx = DBGSuccinctIndex(boss)
        monkeypatch.delenv("MGB_NO_KMER_HASH", raising=False)
        if hashed:
            IT.assert_hashed(idx, boss)
        return idx

    def is_exact(self, r):
        """every k-mer of one strand of r in the graph and none of the other strand's"""
        k, rc = self.k, revcomp(r)
        f = [r[i:i + k] in self.kmers for i in range(len(r) - k + 1)]
        b = [rc[i:i + k] in self.kmers for i in range(len(r) - k + 1)]
        return len(r) >= k and ((all(f) and not any(b)) or (all(b) and not any(f)))

    def exact_reads(self, n, length=L):
        reads = []
        while len(reads) < n:
            p = int(self.rng.integers(1200, len(self.base) - length))
            r = self.base[p:p + length]
            r = revcomp(r) if len(reads) % 2 else r
            if self.is_exact(r):
                reads.append(r)
        return reads

    def mixed_reads(self):
        k = self.k
        reads = self.exact_reads(40)
        r = self.exact_reads(1)[0]
        reads += [substitute(r, 0), substitute(r, L // 2), substitute(r, L - 1), r[:70] + "N" + r[71:]]
        s = self.exact_reads(1, k + 1)[0]
        for n in (k - 1, k, k + 1):
            reads += [s[:n], revcomp(s[:n])]
        reads.append(self.exact_reads(1)[0].lower())
        reads.append("acgt" + self.exact_reads(1, L - 4)[0].lower())
        for off in (0, 9, 300):                                         # both strands are paths of the graph
            s = self.region[off:off + L]
            reads += [s, revcomp(s)]
        reads.append(self.base[380:380 + L])                             # runs into the doubled region
        reads += [self.pal, revcomp(self.pal + self.base[:40])]
        return reads


def check_oracle(case, idx, reads):
    """kernels == oracle with and without node ids in the records, shortcut on == off; returns (lines, stats)"""
    cfg = case.cfg
    got, stats = P.run_lines(idx, cfg, reads)
    exp = case.g.align_tsv(cfg, reads, with_nodes=True)
    bad = [i for i in range(len(reads)) if exp[i] != got[i]]
    assert not bad, (bad[:5], reads[bad[0]], exp[bad[0]], got[bad[0]])
    slim_cfg = dataclasses.replace(cfg, result_nodes=1)
    slim = B200Aligner(idx, slim_cfg).align_batch([("", r) for r in reads])
    assert [format_alignment("", a, cfg.min_path_score) for a in slim] == case.g.align_tsv(cfg, reads)
    off, _ = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=True), reads)
    assert off == got
    return got, stats


@pytest.mark.parametrize("k", [31, 15])
def test_exact_reads_mixed_gpu(k, monkeypatch):
    case = Case(k, 1300 + k)
    reads = case.mixed_reads()
    assert sum(case.is_exact(r.upper()) for r in reads) >= 40
    results = []
    for hashed in (True, False):
        idx = case.index(monkeypatch, hashed)
        got, stats = check_oracle(case, idx, reads)
        idx.close()
        results.append((got, {c: stats[c] for c in COUNTERS}))
    assert results[0] == results[1]


@pytest.mark.parametrize("k", [31, 15])
def test_exact_reads_all_exact_gpu(k, monkeypatch):
    """every read answered: k_align is not launched, the counters are those of one extension per read"""
    case = Case(k, 1400 + k)
    reads = case.exact_reads(300)
    one_more = reads[:-1] + [substitute(reads[-1], L // 2)]
    results = []
    for hashed in (True, False):
        idx = case.index(monkeypatch, hashed)
        got, stats = check_oracle(case, idx, reads)
        assert stats["num_extensions"] == len(reads)
        assert stats["num_seeds"] == sum(len(r) - k + 1 for r in reads)
        assert stats["dp_cells"] == 0 and stats["dp_columns"] == 0
        _, stats_one = P.run_lines(idx, case.cfg, one_more)
        assert stats["kernel_launches"] == stats_one["kernel_launches"] - 1      # no k_align
        idx.close()
        results.append((got, {c: stats[c] for c in COUNTERS}))
    assert results[0] == results[1]


def test_exact_reads_none_exact_gpu(monkeypatch):
    """no read answered: every read goes through k_align"""
    case = Case(31, 1500)
    reads = [substitute(r, int(i * 7) % L) for i, r in enumerate(case.exact_reads(100))]
    idx = case.index(monkeypatch, True)
    _, stats = check_oracle(case, idx, reads)
    idx.close()
    assert stats["dp_cells"] > 0


def test_exact_reads_long_read_gpu(monkeypatch):
    """a read over 511 bp in the batch: k_align does not stage the strands on chip, and the batch takes no exact
    answers (k_align's own exit required the staged strands); results still == oracle"""
    case = Case(31, 1600)
    reads = case.exact_reads(50)
    idx = case.index(monkeypatch, True)
    _, stats = check_oracle(case, idx, reads + case.exact_reads(1, 600))
    _, stats_short = P.run_lines(idx, case.cfg, reads + [substitute(reads[0], 5)])
    assert stats["kernel_launches"] == stats_short["kernel_launches"] - 1     # k_align only
    idx.close()
