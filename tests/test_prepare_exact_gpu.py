"""Whole-read exact answers from the raw reads along the path layout (k_prepare_exact, in place of k_prepare): with the
exact seeder and both strands, on graphs with the k-mer hash index and the path layout, a read whose primary strand runs
along one path with no reverse-complement bit set is answered before seeding; the others are prepared, seeded and go on
to k_exact_reads and k_align. Kernels == oracle (TSV + node paths, and records without node ids), results and counters
identical with the route on and off (MGB_TEST_NO_PREPARE_EXACT), and the number of reads the route answered (the
MGB_DEBUG line) equal to a restatement of its gate over the host reference of the graph."""
import dataclasses
import re

import numpy as np
import pytest

import index_tables as IT
import oracle_lib as O
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment
from metagraph_b200.config import cli_defaults
from test_exact_reads_gpu import COUNTERS, L, Case, random_seq, substitute
from test_oracle_golden import revcomp
from test_path_seed_gpu import boundary_reads, make_graph

pytestmark = pytest.mark.gpu

CODE = {"A": 0, "C": 1, "G": 2, "T": 3}


def pack(s):
    return sum(CODE[c] << (2 * i) for i, c in enumerate(s))


class Graph:
    """an index of `seqs` and the host reference of its tables"""

    def __init__(self, k, seqs, monkeypatch):
        monkeypatch.delenv("MGB_NO_KMER_HASH", raising=False)
        monkeypatch.delenv("MGB_NO_PATH_INDEX", raising=False)
        self.k = k
        self.og = O.OracleGraph(k, seqs, mask=False)
        W, last, F, _ = self.og.arrays()
        boss = BOSSTable(k, W, last, F)
        self.idx = DBGSuccinctIndex(boss)
        IT.assert_hashed(self.idx, boss)
        self.ref = IT.reference_for(boss)
        self.link, _ = self.ref.path_links()
        nodes = np.flatnonzero(self.ref.P)
        self.edge_of = dict(zip(self.ref.key[nodes].tolist(), nodes.tolist()))
        self.rc_set = set(nodes[self.ref.rc_in_K(nodes)].tolist())
        self.keys = set(self.ref.K.tolist())

    def answered(self, r, max_len):
        """the gate of exact_path_strand (kernels.cuh) restated: the read's primary strand starts on a DBG node and follows
        the kept links of the layout to its end, with no node whose reverse complement is a k-mer of the graph"""
        k, u = self.k, r.upper()
        if not k <= len(u) <= max_len or set(u) - set("ACGT"):
            return False
        rc = revcomp(u)
        f, b = pack(u[:k]) in self.keys, pack(rc[:k]) in self.keys
        if f == b:
            return False
        s = u if f else rc
        e = self.edge_of.get(pack(s[:k]))
        for t in range(len(s) - k + 1):
            if e is None or e in self.rc_set:
                return False
            if t + 1 < len(s) - k + 1:
                nxt = int(self.link[e])
                e = nxt if nxt and nxt == self.edge_of.get(pack(s[t + 1:t + 1 + k])) else None
        return True

    def expected(self, reads):
        """reads the route answers: none when a read over 511 bp keeps the batch's strands off chip"""
        max_len = 511 if max(len(r) for r in reads) <= 511 else 0
        return sum(self.answered(r, max_len) for r in reads)

    def close(self):
        self.idx.close()


def run(idx, cfg, reads, route, monkeypatch, capfd):
    """(TSV lines, counters, reads the route answered, the MGB_DEBUG lines)"""
    if route:
        monkeypatch.delenv("MGB_TEST_NO_PREPARE_EXACT", raising=False)
    else:
        monkeypatch.setenv("MGB_TEST_NO_PREPARE_EXACT", "1")
    monkeypatch.setenv("MGB_DEBUG", "1")
    capfd.readouterr()
    al = B200Aligner(idx, cfg)
    res = al.align_batch([("", r) for r in reads])
    err = capfd.readouterr().err
    monkeypatch.delenv("MGB_DEBUG")
    monkeypatch.delenv("MGB_TEST_NO_PREPARE_EXACT", raising=False)
    lines = [format_alignment("", a, cfg.min_path_score, with_nodes=not cfg.result_nodes) for a in res]
    stats = al.last_stats
    return (lines, {c: stats[c] for c in COUNTERS}, sum(int(m) for m in re.findall(r"k_prepare_exact answered (\d+)", err)),
            err)


def check(g, reads, monkeypatch, capfd, expect=None, runs=None):
    """route on == route off == oracle, with and without node ids in the records; returns the reads the route answered.
    runs: a list that receives what run() returned, route on and off, first without node ids in the records"""
    cfg = cli_defaults(g.k, min_seed_length=g.k, max_seed_length=g.k)
    expect = g.expected(reads) if expect is None else expect
    for result_nodes in (0, 1):
        c = dataclasses.replace(cfg, result_nodes=result_nodes)
        exp = g.og.align_tsv(cfg, reads, with_nodes=not result_nodes)
        on = run(g.idx, c, reads, True, monkeypatch, capfd)
        off = run(g.idx, c, reads, False, monkeypatch, capfd)
        if runs is not None:
            runs += [on, off]
        bad = [i for i in range(len(reads)) if exp[i] != on[0][i]]
        assert not bad, (result_nodes, len(bad), reads[bad[0]], exp[bad[0]], on[0][bad[0]])
        assert off[0] == on[0]
        assert off[1] == on[1], (result_nodes, on[1], off[1])
        assert off[2] == 0
        assert on[2] == expect, (result_nodes, on[2], expect)
    return expect


@pytest.mark.parametrize("k", [31, 15])
def test_prepare_exact_mixed_gpu(k, monkeypatch, capfd):
    """substitutions at 0, L/2 and L - 1, N, lower case, lengths k - 1, k and k + 1, a region stored in both orientations
    and palindromes; a batch of 54 reads (part of one tile)"""
    case = Case(k, 1800 + k)
    g = Graph(k, case.seqs, monkeypatch)
    reads = case.mixed_reads()
    n = check(g, reads, monkeypatch, capfd)
    assert 40 <= n < len(reads)
    g.close()


@pytest.mark.parametrize("k", [31, 15])
def test_prepare_exact_rc_bits_gpu(k, monkeypatch, capfd):
    """a piece of the genome (>= k) is also stored reverse complemented: reads over it see pl_rc bits on their run, have
    one probe hit and fall back; reads beside it are answered"""
    rng = np.random.default_rng(1900 + k)
    base = random_seq(rng, 6000)
    g = Graph(k, [base, revcomp(base[3000:3000 + k + 9])], monkeypatch)
    over = [base[p:p + L] for p in range(2900, 3000, 7)]
    beside = [base[p:p + L] for p in range(500, 2500, 97)]
    reads = over + [revcomp(r) for r in over] + beside + [revcomp(r) for r in beside]
    assert not any(g.answered(r, 511) for r in over)
    n = check(g, reads, monkeypatch, capfd)
    assert n == 2 * len(beside)
    g.close()


CASES = [("mutated", 31), ("tandem", 31), ("tandem", 12), ("both_orientations", 31), ("palindromes", 12)]


@pytest.mark.parametrize("kind,k", CASES, ids=["%s-k%d" % c for c in CASES])
def test_prepare_exact_path_ends_gpu(kind, k, monkeypatch, capfd):
    """reads that start, end or cross where a path of the layout ends (branches, cut cycles, a region in both
    orientations, palindromes)"""
    rng = np.random.default_rng(2100 + 10 * CASES.index((kind, k)))
    pg = make_graph(kind, k, rng)
    g = Graph(k, pg.seqs, monkeypatch)
    reads = boundary_reads(rng, pg)
    reads = [reads[int(i)] for i in rng.permutation(len(reads))[:700]]
    n = check(g, reads, monkeypatch, capfd)
    assert 0 < n < len(reads)
    g.close()


@pytest.mark.parametrize("n", [1, 255, 257, 300])
def test_prepare_exact_tiles_gpu(n, monkeypatch, capfd):
    """batch sizes that end partway through a tile of 256 reads"""
    case = Case(31, 2200)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(n)
    if n > 1:
        reads[n // 2] = substitute(reads[n // 2], L // 2)
    check(g, reads, monkeypatch, capfd)
    g.close()


@pytest.mark.parametrize("long_len", [511, 512])
def test_prepare_exact_long_read_gpu(long_len, monkeypatch, capfd):
    """a 511 bp read still lets the strands be staged on chip and is answered like the others; a 512 bp read keeps the
    route off for the whole batch"""
    case = Case(31, 2300)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(60) + case.exact_reads(1, long_len)
    n = check(g, reads, monkeypatch, capfd)
    assert n == (61 if long_len == 511 else 0)
    g.close()


def test_prepare_exact_heap_full_gpu(monkeypatch, capfd):
    """pass 0's heap holds no record (MGB_TEST_HEAP0): the route leaves every read over, they are prepared and seeded,
    overflow in k_exact_reads and are answered by the retry pass, as with the route off"""
    case = Case(31, 2400)
    g = Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(300)
    monkeypatch.setenv("MGB_TEST_HEAP0", "64")
    check(g, reads, monkeypatch, capfd, expect=0)
    # room for some of the records: the rest are left over; the results are the oracle's either way
    monkeypatch.setenv("MGB_TEST_HEAP0", str(100 * 400))
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    lines, stats, n, _ = run(g.idx, cfg, reads, True, monkeypatch, capfd)
    assert lines == g.og.align_tsv(cfg, reads, with_nodes=True)
    assert 0 < n < len(reads) and stats["num_reads_retried"] > 0
    g.close()
