"""Hashed seeding along the path layout (IndexView::pl_*): a walk that starts on a path of the graph follows it in
position order while the read matches, then falls back to the adjacency walk. Node ids of both strands == the oracle's
map_to_nodes, with the layout and without it (MGB_NO_PATH_INDEX), on graphs with many path boundaries: a genome and a
mutated copy, tandem repeats shorter than k (cycles, one of them with no way in or out), a region stored in both
orientations and planted palindromes. The reads cross boundaries, start and end at them, carry errors right past them, N
characters inside runs, and have lengths from below k to 11 666 bp. Whole-read exact answers, which read the seeding
kernel's per-read summary, are the same with and without the layout."""
import dataclasses

import numpy as np
import pytest

import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from test_exact_reads_gpu import COUNTERS, Case, check_oracle
from test_oracle_golden import revcomp
from test_seed_hash_gpu import mixed_reads
from test_seed_pairing import random_seq, role_reads, with_palindromes

pytestmark = pytest.mark.gpu


def substitute(r, i):
    return r[:i] + ("A" if r[i] != "A" else "C") + r[i + 1:]


@dataclasses.dataclass
class Graph:
    k: int
    seqs: list        # what the graph is built from
    sources: list     # what reads are drawn from
    sites: list       # (source, position) pairs: where a path of the graph may end


def branch_sites(k, seqs, sources):
    """positions i of the sources whose (k - 1)-mer ending before i has several children or the one starting at i
    several parents"""
    nxt, prv = {}, {}
    for s in seqs:
        for i in range(len(s) - k + 1):
            nxt.setdefault(s[i:i + k - 1], set()).add(s[i + k - 1])
            prv.setdefault(s[i + 1:i + k], set()).add(s[i])
    return [(j, i) for j, s in enumerate(sources) for i in range(k - 1, len(s) - k + 1)
            if len(nxt[s[i - k + 1:i]]) > 1 or len(prv[s[i:i + k - 1]]) > 1]


def make_graph(kind, k, rng):
    base = random_seq(rng, 12000)
    extra = []
    if kind == "mutated":
        seqs = [base, P.mutate(rng, base, 0.02)]
    elif kind == "tandem":
        unit = random_seq(rng, k // 2 + 3)                          # period < k: a cycle
        lone = random_seq(rng, k // 3 + 2)
        seqs = [base[:5000] + unit * 12 + base[5000:],
                lone * (3 * k // len(lone) + 3)]                    # every k-mer has one child and one parent: no head
        extra = [(0, 5000), (0, 5000 + 12 * len(unit))]
    elif kind == "both_orientations":
        seqs = [base, revcomp(base[3000:6000])]
        extra = [(0, 3000), (0, 6000)]                              # where the reverse strand's path starts / ends
    else:
        assert kind == "palindromes"
        seqs = [with_palindromes(rng, base, k, 60)]
        s = seqs[0]
        extra = [(0, i) for i in range(len(s) - k + 1) if s[i:i + k] == revcomp(s[i:i + k])]
    sources = seqs[:1] if kind == "both_orientations" else seqs
    return Graph(k, seqs, sources, branch_sites(k, seqs, sources) + extra)


def boundary_reads(rng, g):
    """reads that start or end at each offset around boundary sites, with an error right past the site or an N in the
    middle of a run"""
    k, reads = g.k, []
    for si in rng.permutation(len(g.sites))[:25]:
        src, m = g.sites[int(si)]
        s = g.sources[src]
        for d in range(-k - 2, 3):
            for L in (k, k + 1, 80):
                a = m + d
                if 0 <= a and a + L <= len(s):
                    reads.append(s[a:a + L])                        # starts near the site
                b = m - d
                if 0 <= b - L and b <= len(s):
                    reads.append(s[b - L:b])                        # ends near the site
        a = max(0, m - 60)
        r = s[a:a + 150]
        if m - a + 1 < len(r):
            reads.append(substitute(r, m - a + 1))                  # an error at the first character past the site
        if len(r) > 100:
            reads.append(r[:100] + "N" + r[101:])
    return reads + [revcomp(r) for r in reads[::3]]


CASES = [("mutated", 31), ("mutated", 12), ("tandem", 31), ("tandem", 12), ("both_orientations", 31),
         ("palindromes", 12)]


def index(g, monkeypatch, path):
    if path:
        monkeypatch.delenv("MGB_NO_PATH_INDEX", raising=False)
    else:
        monkeypatch.setenv("MGB_NO_PATH_INDEX", "1")
    og = O.OracleGraph(g.k, g.seqs, mask=False)
    W, last, F, _ = og.arrays()
    idx = DBGSuccinctIndex(BOSSTable(g.k, W, last, F))
    monkeypatch.delenv("MGB_NO_PATH_INDEX", raising=False)
    return og, idx


@pytest.mark.parametrize("kind,k", CASES, ids=["%s-k%d" % c for c in CASES])
def test_path_seed_gpu(kind, k, monkeypatch):
    rng = np.random.default_rng(2000 + 10 * CASES.index((kind, k)))
    g = make_graph(kind, k, rng)
    reads = boundary_reads(rng, g) + mixed_reads(rng, g.sources, k, 301) + role_reads(rng, g.sources[:1], k)
    sizes = []
    for path in (True, False):
        og, idx = index(g, monkeypatch, path)
        sizes.append(idx.device_bytes)
        seq = idx.map_to_nodes_sequentially(reads)
        fwd, rev = idx.map_to_nodes_strands(reads)
        idx.close()
        exp_f = [list(og.map_to_nodes(r)) for r in reads]
        exp_r = [list(og.map_to_nodes(revcomp(r))) for r in reads]
        bad = [i for i in range(len(reads)) if list(seq[i]) != exp_f[i]]
        assert not bad, (path, "sequentially", len(bad), reads[bad[0]][:80])
        bad = [i for i in range(len(reads)) if list(fwd[i]) != exp_f[i] or list(rev[i]) != exp_r[i]]
        assert not bad, (path, "strands", len(bad), reads[bad[0]][:80])
    assert sizes[0] > sizes[1]                                      # the layout was built


@pytest.mark.parametrize("k", [31, 15])
def test_path_seed_exact_reads_gpu(k, monkeypatch):
    """whole-read exact answers (from the seeding summary byte) with the layout == without it == the oracle"""
    case = Case(k, 1700 + k)
    reads = case.mixed_reads()
    results = []
    for path in (True, False):
        if not path:
            monkeypatch.setenv("MGB_NO_PATH_INDEX", "1")
        idx = case.index(monkeypatch, True)
        monkeypatch.delenv("MGB_NO_PATH_INDEX", raising=False)
        got, stats = check_oracle(case, idx, reads)
        idx.close()
        results.append((got, {c: stats[c] for c in COUNTERS}))
    assert results[0] == results[1]
