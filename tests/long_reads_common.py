"""Shared driver of the long-read tests: reads of 0.5 - 30 kbp with substitutions and indels, which need thousands of DP
columns per extension, overflow their first arenas and are aligned on a retry pass at scale 16 or 64. Every input runs
through a library and through the oracle, which must give identical TSV lines with node paths. With MGB_DEBUG set, the
run also returns how many align passes the call took (its `pass: classify` ticks) and, on the device, each pass's
`k_align grid` line: the warps launched, the arena bytes per warp and the arenas allocated."""
import dataclasses
import re

import numpy as np

import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults

# lengths: k = 31 graph of three haplotypes of a 30 kbp genome, 1 % apart; reads of LENGTHS bp with RATES errors
# (P.mutate: substitutions, insertions and deletions) on both strands. canonical / primary: the same reads on the graph built as
# `build --mode canonical` / `--mode primary` (as P.fuzz_case builds them). k11: sub-k seeds (min_seed_length 8)
# on a k = 11 graph. k47: the 256-bit-key build of the kernels. protein: 3 kbp reads with 5 % substitutions and 2 %
# indels, BLOSUM62, through the alphabet-generic layout. mixed: 2 000 150 bp reads with 5 % errors, 500 error-free
# 150 bp reads and 8 reads of 5 - 12 kbp in one batch under the exact seeder of the benchmark's C2 shape; a batch with a
# read over 511 bp stages no query on chip, which also turns its whole-read exact answers off, so every read of it goes
# through k_align. single20k / single30k: one read of 20 / 30 kbp with 5 % errors, alone in its batch.
LONG_INPUTS = ("lengths", "canonical", "primary", "k11", "k47", "protein", "mixed", "single20k", "single30k")
LENGTHS = (150, 600, 2000, 5000, 12000)
RATES = (0.02, 0.05, 0.12)

# configurations of `lengths`: CLI defaults (every read kept: min_exact_match 0) at x-drop 27 and 200, and with two
# alternative paths
LENGTHS_CFGS = ("x27", "x200", "alt2")

# align passes each input takes (its `pass: classify` ticks): pass p runs with arenas scaled by 4^p, so 4 passes means
# some read was aligned only at scale 64. The emulation and the device must agree on them. The protein reads fit their
# first arena: BLOSUM62's scores keep the x-drop band narrow.
PASSES = {("lengths", "x27"): 4, ("lengths", "x200"): 3, ("lengths", "alt2"): 4, ("canonical", "x27"): 4,
          ("primary", "x27"): 4, ("k11", "x27"): 3, ("k47", "x27"): 4, ("protein", "x27"): 1, ("mixed", "x27"): 4,
          ("single20k", "x27"): 4, ("single30k", "x27"): 4}

GRID = re.compile(r"k_align grid: (\d+) warps \((\d+) resident\), arena (\d+) bytes per warp, (\d+) arenas")
CLASSIFY = re.compile(r"\] reads \d+\+\d+ pass: classify")


@dataclasses.dataclass
class LongInput:
    k: int
    seqs: list           # sequences the graph is built from
    mode: int            # 0 BASIC, 1 CANONICAL, 2 PRIMARY
    alphabet: str
    reads: list
    cfgs: dict           # configuration name -> DBGAlignerConfig


def haplotypes():
    rng = np.random.default_rng(500)
    base = P._random_seq(rng, 30000)
    return [base] + [P.mutate(rng, base, 0.01) for _ in range(2)]


def _reads(rng, seqs, lengths, rates):
    """one read per (length, rate, strand), from the haplotypes in turn"""
    reads = []
    for L in lengths:
        for rate in rates:
            for strand in (0, 1):
                s_ = seqs[len(reads) % len(seqs)]
                p = int(rng.integers(0, len(s_) - L))
                r = P.mutate(rng, s_[p:p + L], rate)
                reads.append(P.revcomp(r) if strand else r)
    return reads


def long_input(name):
    hap = haplotypes()
    if name in ("lengths", "canonical", "primary"):
        k = 31
        reads = _reads(np.random.default_rng(501), hap, LENGTHS, RATES)
        cfgs = {"x27": cli_defaults(k, min_exact_match=0.0), "x200": cli_defaults(k, min_exact_match=0.0, xdrop=200),
                "alt2": cli_defaults(k, min_exact_match=0.0, num_alternative_paths=2)}
        if name == "canonical":
            return LongInput(k, hap + [P.revcomp(s_) for s_ in hap], 1, "dna", reads, {"x27": cfgs["x27"]})
        if name == "primary":
            return LongInput(k, P.primary_contigs(hap, k), 2, "dna", reads, {"x27": cfgs["x27"]})
        return LongInput(k, hap, 0, "dna", reads, cfgs)
    if name in ("k11", "k47"):
        k = 11 if name == "k11" else 47
        rng = np.random.default_rng(502 if name == "k11" else 503)
        reads = _reads(rng, hap, (600, 2000, 5000) if name == "k11" else (2000, 5000, 12000), (0.05, 0.12))
        kw = dict(min_seed_length=8) if name == "k11" else {}
        return LongInput(k, hap, 0, "dna", reads, {"x27": cli_defaults(k, min_exact_match=0.0, **kw)})
    if name == "protein":
        k = 10
        rng = np.random.default_rng(504)
        seqs = ["".join(np.array(list(P.AA))[rng.integers(0, 20, 10000)])]
        seqs.append(P.mutate_aa(rng, seqs[0], 0.01))
        reads = []
        for i in range(6):
            s_ = seqs[i % 2]
            p = int(rng.integers(0, len(s_) - 3000))
            reads.append(P.mutate_aa(rng, s_[p:p + 3000], 0.05, 0.02))
        return LongInput(k, seqs, 0, "protein", reads,
                         {"x27": cli_defaults(k, alphabet="protein", min_exact_match=0.0)})
    if name == "mixed":
        k = 31
        rng = np.random.default_rng(505)
        short = [P.mutate(rng, w, 0.05) for w in _windows(rng, hap, 2000, 150)]
        exact = _windows(rng, hap, 500, 150)
        long_ = [P.mutate(rng, w, 0.05) for w in _windows(rng, hap, 8, None)]
        reads = short + exact
        for i, r in enumerate(long_):                     # spread over the batch
            reads.insert(300 * i + 7, r)
        reads = [P.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
        return LongInput(k, hap, 0, "dna", reads,
                         {"x27": cli_defaults(k, min_seed_length=k, max_seed_length=k, min_exact_match=0.0)})
    if name in ("single20k", "single30k"):
        k = 31
        L = 20000 if name == "single20k" else 29900
        rng = np.random.default_rng(506 if name == "single20k" else 507)
        p = int(rng.integers(0, len(hap[1]) - L))
        return LongInput(k, hap, 0, "dna", [P.mutate(rng, hap[1][p:p + L], 0.05)],
                         {"x27": cli_defaults(k, min_exact_match=0.0)})
    raise ValueError(name)


def _windows(rng, seqs, n, L):
    """n windows of the haplotypes, of L bp each (None: 5 - 12 kbp)"""
    out = []
    for i in range(n):
        s_ = seqs[i % len(seqs)]
        n_bp = int(rng.integers(5000, 12001)) if L is None else L
        p = int(rng.integers(0, len(s_) - n_bp))
        out.append(s_[p:p + n_bp])
    return out


def cfg_names(name):
    return LENGTHS_CFGS if name == "lengths" else ("x27",)


class LongReads:
    """One input with its oracle graph and a cache of oracle answers per configuration, reused across libraries"""

    _inputs = {}
    _graphs = {}
    _oracle = {}             # (name, configuration name) -> (lines, stats)

    def __init__(self, name):
        self.name = name
        if name not in LongReads._inputs:
            inp = long_input(name)
            g = O.OracleGraph(inp.k, inp.seqs, alphabet=inp.alphabet)
            g.set_mode(inp.mode)
            LongReads._inputs[name], LongReads._graphs[name] = inp, g
        self.inp = LongReads._inputs[name]
        self.g = LongReads._graphs[name]

    def index(self, lib):
        W, last, F, _ = self.g.arrays()
        return DBGSuccinctIndex(BOSSTable(self.inp.k, W, last, F, alphabet=int(self.inp.alphabet == "protein")),
                                lib=lib, mode=self.inp.mode)

    def cfg(self, cfg_name, **kw):
        return dataclasses.replace(self.inp.cfgs[cfg_name], **kw)

    def oracle(self, cfg_name):
        key = (self.name, cfg_name)
        if key not in LongReads._oracle:
            st = {}
            lines = self.g.align_tsv(self.cfg(cfg_name), self.inp.reads, with_nodes=True, threads=8, stats=st)
            LongReads._oracle[key] = (lines, st)
        return LongReads._oracle[key]


@dataclasses.dataclass
class Run:
    stats: dict
    passes: int = None   # `pass: classify` ticks (MGB_DEBUG runs)
    grids: list = None   # per pass on the device: (warps, resident warps, arena bytes per warp, arenas)
    hits: dict = None    # emulation: path hits of the run


def check(lib, name, cfg_name="x27", trace=None, shortcut=True, idx=None):
    """lines == oracle for one input and configuration. trace = (monkeypatch, capfd): the run is made with MGB_DEBUG
    set and the result holds its passes and grid lines. shortcut=False: the exact-path shortcut off, and the five DP
    counters == the oracle's."""
    lr = LongReads(name)
    exp, ost = lr.oracle(cfg_name)
    cfg = lr.cfg(cfg_name, no_exact_path_shortcut=not shortcut)
    own = idx is None
    idx = lr.index(lib) if own else idx
    try:
        h0 = P.path_hits(lib)
        if trace is not None:
            mp, capfd = trace
            with mp.context() as m:
                m.setenv("MGB_DEBUG", "1")
                capfd.readouterr()
                got, st = P.run_lines(idx, cfg, lr.inp.reads)
                err = capfd.readouterr().err
        else:
            got, st = P.run_lines(idx, cfg, lr.inp.reads)
        h1 = P.path_hits(lib)
    finally:
        if own:
            idx.close()
    bad = [i for i in range(len(exp)) if exp[i] != got[i]]
    assert not bad, (name, cfg_name, len(bad), bad[:3], len(lr.inp.reads[bad[0]]), exp[bad[0]][:300],
                     got[bad[0]][:300])
    if not shortcut:
        diff = {c: (ost[c], st[c]) for c in P.DP_COUNTERS if ost[c] != st[c]}
        assert not diff, (name, cfg_name, diff)
    run = Run(st, hits=None if h0 is None else {p: h1[p] - h0[p] for p in P.EMU_PATHS})
    if trace is not None:
        run.passes = len(CLASSIFY.findall(err))
        run.grids = [tuple(int(x) for x in m.groups()) for m in GRID.finditer(err)]
    return run


def long_read_indices(name):
    """positions of the reads over 511 bp"""
    return [i for i, r in enumerate(LongReads(name).inp.reads) if len(r) > 511]
