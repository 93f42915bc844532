"""Shared driver of the budget tests: the extender's stop rules (max_ram_per_alignment, max_nodes_per_seq_char) at
budgets chosen from the oracle's own trace of its stop tests, and no_backtrack. Every run is compared with the oracle:
TSV lines with node paths, and with the exact-path shortcut off all five DP counters, which show that the kernel
explored exactly the columns the reference explores before it stopped."""
import dataclasses
import math

import numpy as np

import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import DBL_MAX, cli_defaults

# variants: k = 15 graph of 3 haplotypes, 150 bp reads with 5 % errors on both strands. Four of the pressure inputs.
# canonical / primary: the variant graph built as `build --mode canonical` / `--mode primary` (as fuzz_case builds
# them). protein: PROTEIN_CASES[0]'s shape (alphabet-generic layout, general path only). k47: the 256-bit-key
# instantiation. alt3: the variant graph reporting 3 alternative paths.
BUDGET_INPUTS = ("variants", "queue", "retry", "wide_band", "insertions", "canonical", "primary", "protein", "k47",
                 "alt3")
PRESSURE_BUDGET_INPUTS = ("queue", "retry", "wide_band", "insertions")


# quantiles of the distinct traced values at which the budgets are chosen (0 and 1: the extremes)
RAM_QUANTILES = (0.0, 0.01, 0.02, 0.05, 0.1, 0.15, 0.5, 0.9, 1.0)
NODE_QUANTILES = (0.0, 0.01, 0.02, 0.05, 0.1, 1.0)


@dataclasses.dataclass
class BudgetInput:
    k: int
    seqs: list           # sequences the graph is built from
    mode: int            # 0 BASIC, 1 CANONICAL, 2 PRIMARY
    alphabet: str
    reads: list
    cfg: object


def _variant_reads(rng, seqs, n, L, rate):
    reads = []
    for i in range(n):
        s_ = seqs[i % len(seqs)]
        p = int(rng.integers(0, len(s_) - L))
        r = P.mutate(rng, s_[p:p + L], rate)
        reads.append(P.revcomp(r) if i % 2 else r)
    return reads


def budget_input(name):
    if name in P.PRESSURE_INPUTS:
        k, seqs, reads, cfg = P.pressure_input(name)
        return BudgetInput(k, seqs, 0, "dna", reads, cfg)
    if name == "protein":
        seed, k, G, n, L, rate, cfgf, _, nseq, indel = P.PROTEIN_CASES[0]
        rng = np.random.default_rng(seed)
        seqs = ["".join(np.array(list(P.AA))[rng.integers(0, 20, G)])]
        seqs += [P.mutate_aa(rng, seqs[0], 0.03) for _ in range(nseq - 1)]
        reads = []
        for i in range(n):
            s_ = seqs[i % nseq]
            p = int(rng.integers(0, len(s_) - L))
            reads.append(P.mutate_aa(rng, s_[p:p + L], rate, indel))
        return BudgetInput(k, seqs, 0, "protein", reads, cfgf(k))
    k = 47 if name == "k47" else 15
    rng = np.random.default_rng(401 if name == "k47" else 400)
    base = P._random_seq(rng, 4000)
    hap = [base] + [P.mutate(rng, base, 0.02) for _ in range(2)]
    reads = _variant_reads(rng, hap, 30 if name in ("canonical", "primary", "k47") else 60, 150, 0.05)
    cfg = cli_defaults(k, min_exact_match=0.0, num_alternative_paths=3 if name == "alt3" else 1)
    if name == "canonical":
        return BudgetInput(k, hap + [P.revcomp(s_) for s_ in hap], 1, "dna", reads, cfg)
    if name == "primary":
        return BudgetInput(k, P.primary_contigs(hap, k), 2, "dna", reads, cfg)
    return BudgetInput(k, hap, 0, "dna", reads, cfg)


class Budgets:
    """One input with its oracle graph, its index in a library and a cache of oracle answers per configuration,
    reused across libraries and knobs."""

    _oracle = {}             # (name, config key) -> (lines, stats)
    _graphs = {}

    def __init__(self, name):
        self.name = name
        self.inp = budget_input(name)
        if name not in Budgets._graphs:
            g = O.OracleGraph(self.inp.k, self.inp.seqs, alphabet=self.inp.alphabet)
            g.set_mode(self.inp.mode)
            Budgets._graphs[name] = g
        self.g = Budgets._graphs[name]

    def index(self, lib):
        W, last, F, _ = self.g.arrays()
        return DBGSuccinctIndex(BOSSTable(self.inp.k, W, last, F, alphabet=int(self.inp.alphabet == "protein")),
                                lib=lib, mode=self.inp.mode)

    def cfg(self, **kw):
        return dataclasses.replace(self.inp.cfg, **kw)

    def oracle(self, cfg):
        key = (self.name, _cfg_key(cfg))
        if key not in Budgets._oracle:
            st = {}
            lines = self.g.align_tsv(cfg, self.inp.reads, with_nodes=True, stats=st)
            Budgets._oracle[key] = (lines, st)
        return Budgets._oracle[key]

    def trace(self):
        """all (bytes, table size, window size) the oracle's stop tests see with both budgets switched off"""
        t = self.g.budget_trace(self.cfg(max_ram_per_alignment=DBL_MAX, max_nodes_per_seq_char=DBL_MAX),
                                self.inp.reads)
        return np.concatenate([x for x in t if len(x)] or [np.zeros((0, 3), np.uint64)])

    def ram_budgets(self):
        """distinct traced byte counts v at 7 quantiles plus the extremes: v / 1e6 (the strict test does not fire at
        v) and the next double below it (it fires); then 0, the CLI's 200 MB, inf and NaN. Most quantiles are low:
        a late stop seldom changes the answer. The 0.9 quantile stops some of `retry`'s reads after their first try has
        overflowed its arena."""
        v = np.unique(self.trace()[:, 0])
        assert len(v) >= len(RAM_QUANTILES), (self.name, len(v))
        pick = sorted({int(v[int(round(q * (len(v) - 1)))]) for q in RAM_QUANTILES})
        pairs = [(b / 1e6, math.nextafter(b / 1e6, -math.inf)) for b in pick]
        return pairs, [0.0, 200.0, math.inf, math.nan]

    def node_budgets(self):
        """traced n / w at 4 quantiles plus the extremes: n / w (the test `>=` fires) and the next double above.
        Low quantiles, as for the RAM budgets."""
        t = self.trace()
        r = np.unique(t[:, 1].astype(np.float64) / t[:, 2].astype(np.float64))
        assert len(r) >= len(NODE_QUANTILES), (self.name, len(r))
        pick = sorted({float(r[int(round(q * (len(r) - 1)))]) for q in NODE_QUANTILES})
        return [(x, math.nextafter(x, math.inf)) for x in pick]


def _cfg_key(cfg):
    d = dataclasses.asdict(cfg)
    d.pop("no_exact_path_shortcut")            # the oracle has no shortcut; its answer is the same either way
    d.pop("result_nodes")
    d["score_matrix"] = tuple(map(tuple, d["score_matrix"]))
    return tuple(sorted((k, repr(v)) for k, v in d.items()))


def check_run(b, idx, cfg, what):
    """lines == oracle with the shortcut off and on, DP counters == oracle with it off. Returns (oracle lines, oracle
    stats, kernel statistics of the shortcut-off run)."""
    exp, ost = b.oracle(cfg)
    off, kst = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=True), b.inp.reads)
    bad = [i for i in range(len(exp)) if exp[i] != off[i]]
    assert not bad, (b.name, what, bad[:3], exp[bad[0]][:300], off[bad[0]][:300])
    diff = {c: (ost[c], kst[c]) for c in P.DP_COUNTERS if ost[c] != kst[c]}
    assert not diff, (b.name, what, diff)
    on, _ = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=False), b.inp.reads)
    bad = [i for i in range(len(exp)) if on[i] != off[i]]
    assert not bad, (b.name, what, "shortcut on", bad[:3], off[bad[0]][:300], on[bad[0]][:300])
    return exp, ost, kst


def budget_matrix(lib, name):
    """Every chosen RAM and node budget of one input through the library (see check_run), and the checks that show
    the budgets reach what they are meant to test: at least half of them change a read against the same
    configuration without that budget, at least one (v, next double below) pair changes the oracle's dp_columns,
    so the pair straddles a real stop, and on `retry` a budget that stops some search still leaves reads for the
    arena retry, which must restart them with an empty table.
    Returns the number of runs."""
    b = Budgets(name)
    idx = b.index(lib)
    runs = 0
    try:
        free_ram, free_st = b.oracle(b.cfg(max_ram_per_alignment=math.inf))
        pairs, extra = b.ram_budgets()
        changed, straddles, retried = 0, 0, 0
        for hi, lo in pairs:
            res = []
            for x in (hi, lo):
                exp, ost, kst = check_run(b, idx, b.cfg(max_ram_per_alignment=x), ("ram", x))
                changed += exp != free_ram
                res.append(ost["dp_columns"])
                if ost["dp_columns"] != free_st["dp_columns"] and kst["num_reads_retried"] > 0:
                    retried += 1
                runs += 1
            straddles += res[0] != res[1]
        for x in extra:
            exp, _, _ = check_run(b, idx, b.cfg(max_ram_per_alignment=x), ("ram", x))
            changed += exp != free_ram
            runs += 1
        n_ram = 2 * len(pairs) + len(extra)
        assert 2 * changed >= n_ram, (name, "ram budgets that change a read", changed, n_ram)
        assert straddles >= 1, (name, "no (v, nextafter) pair straddles a stop", pairs)
        if name == "retry":
            assert retried >= 1, (name, "no budget that stops a search leaves a read for the arena retry")

        free_nodes, _ = b.oracle(b.cfg(max_nodes_per_seq_char=DBL_MAX))
        changed = 0
        node_pairs = b.node_budgets()
        for x in [y for pr in node_pairs for y in pr]:
            exp, _, _ = check_run(b, idx, b.cfg(max_nodes_per_seq_char=x), ("nodes", x))
            changed += exp != free_nodes
            runs += 1
        assert 2 * changed >= 2 * len(node_pairs), (name, "node budgets that change a read", changed)
    finally:
        idx.close()
    return runs


def no_backtrack_case(lib, name):
    """no_backtrack: the extension reports the seed's alignment as it is (the exit before the backtrack), the
    exact-path shortcut is off for it; lines and counters == oracle"""
    b = Budgets(name)
    idx = b.index(lib)
    try:
        exp, _, _ = check_run(b, idx, b.cfg(no_backtrack=True), "no_backtrack")
    finally:
        idx.close()
    return exp


def shortcut_budget_cases(lib):
    """The whole-read and exact-path shortcut inputs at budgets that would end any extension at once (RAM 0 and NaN,
    0.01 nodes per character): the whole-read gates never read the budgets, so their answers must still equal the
    oracle's, shortcut on and off."""
    for seed, k, cfgf, _ in P.WHOLE_READ_CASES[:2]:
        for kw in (dict(max_ram_per_alignment=0.0), dict(max_ram_per_alignment=math.nan),
                   dict(max_nodes_per_seq_char=0.01)):
            P.whole_read_case(lib, seed, k, dataclasses.replace(cfgf(k), **kw))
    for seed, k, cfgf in P.EXACT_SHORTCUT_CASES[:3]:
        for kw in (dict(max_ram_per_alignment=0.0), dict(max_ram_per_alignment=math.nan),
                   dict(max_nodes_per_seq_char=0.01)):
            P.exact_shortcut_case(lib, seed, k, dataclasses.replace(cfgf(k), **kw))


# the knobs of pressure_knob_matrix that move where the budgets' copies run: the general loop without the register
# path (nofast), one block (grid1), several pieces and heaps (pieces3), no staged query (lq0), a small column buffer
BUDGET_KNOBS = tuple(kn for kn in P.SPILL_KNOBS if kn[0] in ("default", "nofast", "grid1", "pieces3", "lq0", "bmax64"))


def budget_knob_matrix(lib, name, monkeypatch):
    """one RAM budget and one node budget that bite, under every knob of BUDGET_KNOBS: lines == oracle, DP counters
    == the oracle's (shortcut off), and so == the default run's"""
    b = Budgets(name)
    pairs, _ = b.ram_budgets()
    free, _ = b.oracle(b.cfg(max_ram_per_alignment=math.inf))
    ram = next(lo for _, lo in pairs if b.oracle(b.cfg(max_ram_per_alignment=lo))[0] != free)
    free, _ = b.oracle(b.cfg(max_nodes_per_seq_char=DBL_MAX))
    nodes = next(x for x, _ in b.node_budgets() if b.oracle(b.cfg(max_nodes_per_seq_char=x))[0] != free)
    for knob, env in BUDGET_KNOBS:
        with monkeypatch.context() as mp:
            for var, val in env.items():
                mp.setenv(var, val)
            idx = b.index(lib)
            try:
                check_run(b, idx, b.cfg(max_ram_per_alignment=ram), (knob, "ram", ram))
                check_run(b, idx, b.cfg(max_nodes_per_seq_char=nodes), (knob, "nodes", nodes))
            finally:
                idx.close()


def random_counters_case(lib, case):
    """RANDOM_CASES with the shortcut off: the kernel's five DP counters == the oracle's"""
    seed, k, G, n, L, rate, cfgf, mask, nseq = case
    ost = {}
    kst = P.random_case(lib, seed, k, G, n, L, rate, dataclasses.replace(cfgf(k), no_exact_path_shortcut=True), mask,
                        nseq, oracle_stats=ost)
    diff = {c: (ost[c], kst[c]) for c in P.DP_COUNTERS if ost[c] != kst[c]}
    assert not diff, (seed, diff)


def stop_site_hits(lib):
    """one RAM budget and one node budget that stop searches early (the next double below the 0.1 quantile of the
    traced bytes, the 0.02 quantile of n / w) on every input; returns the emulation's path hits of these runs"""
    h0 = P.path_hits(lib)
    for name in BUDGET_INPUTS:
        b = Budgets(name)
        v = np.unique(b.trace()[:, 0])
        ram = math.nextafter(int(v[int(round(0.1 * (len(v) - 1)))]) / 1e6, -math.inf)
        nodes = b.node_budgets()[1][0]
        idx = b.index(lib)
        try:
            check_run(b, idx, b.cfg(max_ram_per_alignment=ram), ("ram", ram))
            check_run(b, idx, b.cfg(max_nodes_per_seq_char=nodes), ("nodes", nodes))
        finally:
            idx.close()
    h1 = P.path_hits(lib)
    return {p: h1[p] - h0[p] for p in P.EMU_PATHS}
