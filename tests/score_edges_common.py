"""Score edges: the kernels against the oracle on score matrices the other parity tests never draw (per-letter
diagonals, asymmetric and complement-asymmetric mismatches, mismatches at or above another letter's match, random N,
'$' and '\\0' rows), on min_cell_score / min_path_score away from their defaults, and on penalties at the bound of
check_config_scores. Every run: lines (node paths included) == oracle with the exact-path shortcut off, the five DP
counters == the oracle's, and the shortcut on gives the shortcut-off lines."""
import dataclasses

import numpy as np
import pytest

import oracle_lib as O
import parity_common as P
from metagraph_b200 import _lib
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import (INT32_MAX, INT32_MIN, NINF, SIZE_MAX, blosum62_scoring_matrix, cli_defaults,
                                   dna_scoring_matrix, struct_defaults, unit_scoring_matrix)

DNA = "ACGT"
PROTEIN = "ABCDEFGHIJKLMNOPQRSTUVWYZ"       # valid protein letters; 'X' is the alphabet's catch-all
COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}


def transpose(m):
    return [[m[b][a] for b in range(128)] for a in range(128)]


def complemented(m):
    """M'[a][b] = M[comp a][comp b] on ACGT (upper and lower case), the rest unchanged"""
    cmap = list(range(128))
    for a, b in COMP.items():
        cmap[ord(a)] = ord(b); cmap[ord(a.lower())] = ord(b.lower())
    return [[m[cmap[a]][cmap[b]] for b in range(128)] for a in range(128)]


def in_range(cfg):
    """ninf less the lowest matrix entry (or gap open), a gap open and a gap extension stays in int32: the reference's
    column update (extender.cpp:209-328) forms no sum outside int32, so its answer is defined (DESIGN.md §5)"""
    lo = min(min(min(r) for r in cfg.score_matrix), cfg.gap_opening_penalty)
    return NINF + lo + cfg.gap_opening_penalty + cfg.gap_extension_penalty >= INT32_MIN


def random_dna_matrix(rng):
    """per-letter diagonals 1..5, mismatches drawn per ordered pair (so M != M^T and M != complemented M), now and then
    one at or above another letter's match (the exact-path shortcut's gate turns off), random N column and row, random
    rows for '$' and '\\0'"""
    m = dna_scoring_matrix(2, -3, -3)
    diag = {c: int(rng.integers(1, 6)) for c in DNA}
    for a in DNA:
        for b in DNA:
            if a == b:
                m[ord(a)][ord(b)] = diag[a]
            elif rng.random() < 0.1:
                m[ord(a)][ord(b)] = int(rng.integers(min(diag.values()), 6))
            else:
                m[ord(a)][ord(b)] = -int(rng.integers(1, 7))
        m[ord(a)][ord("N")] = -int(rng.integers(0, 6))
        m[ord("N")][ord(a)] = -int(rng.integers(0, 6))
    for row in ("$", "\0"):
        for b in DNA + "N":
            m[ord(row)][ord(b)] = int(rng.integers(-6, 3))
    return m


def draw_cell_and_path_scores(rng, kw, match_sum):
    lo = min(min(min(r) for r in kw["score_matrix"]), kw["gap_opening_penalty"], kw["gap_extension_penalty"])
    kw["min_cell_score"] = int(rng.choice([NINF, INT32_MIN - lo, INT32_MIN - lo + 1, INT32_MIN - lo - 1, 0,
                                           int(rng.integers(1, 30))]))
    kw["min_path_score"] = int(rng.choice([-int(rng.integers(1, 100)), 0, int(rng.integers(1, max(2, match_sum)))]))


def check_text(idx, cfg, reads):
    """mgb_align_batch_text, TSV and JSON, == the host mirror over mgb_align_batch's records (text_common)"""
    import text_common as T
    T.check_text(idx, cfg, reads)


def _run(lib, idx, g, cfg, reads):
    """oracle lines and statistics, then the library shortcut off and on; returns the oracle lines or None when the
    oracle's constructor rejects the configuration (the library must reject it too)"""
    ost = {}
    try:
        exp = g.align_tsv(cfg, reads, with_nodes=True, stats=ost)
    except RuntimeError as err:                          # DBGAligner ctor: check_config_scores failed
        assert "too low" in str(err)
        with pytest.raises(_lib.MgbError) as e2:
            P.run_lines(idx, cfg, reads)
        assert e2.value.code == -3                       # MGB_ERR_BAD_CONFIG
        return None
    off, kst = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=True), reads)
    bad = [i for i in range(len(reads)) if exp[i] != off[i]]
    assert not bad, (bad[:3], reads[bad[0]], exp[bad[0]][:300], off[bad[0]][:300])
    diff = {c: (ost[c], kst[c]) for c in P.DP_COUNTERS if ost[c] != kst[c]}
    assert not diff, diff
    on, _ = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=False), reads)
    bad = [i for i in range(len(reads)) if on[i] != off[i]]
    assert not bad, ("shortcut on", bad[:3], off[bad[0]][:300], on[bad[0]][:300])
    return exp


def dna_matrix_case(lib, seed, mode, nreads=25, text=False):
    """One randomized DNA triple (mode 0 BASIC, 1 CANONICAL, 2 PRIMARY) under a random full matrix and random
    min_cell_score / min_path_score. text: also the text route (TSV and JSON) == the host mirror. Returns (#reads whose
    oracle lines differ under M^T, under complemented M), or None when the configuration is rejected."""
    rng = np.random.default_rng(7000 + 100 * mode + seed)
    k = int(rng.integers(5, 32))
    G = int(rng.integers(400, 3000))
    base = "".join(np.array(list(DNA))[rng.integers(0, 4, G)])
    seqs = [base] + [P.mutate(rng, base, 0.03) for _ in range(int(rng.integers(0, 3)))]
    if rng.random() < 0.3:
        seqs.append(base[:int(rng.integers(k, 3 * k))] * int(rng.integers(2, 4)) + base[50:120])
    m = random_dna_matrix(rng)
    go = -int(rng.integers(4, 10)); ge = -int(rng.integers(1, 4))
    kw = dict(score_matrix=m, gap_opening_penalty=go, gap_extension_penalty=ge, xdrop=int(rng.integers(8, 60)),
              min_exact_match=float(rng.choice([0.0, 0.0, 0.5])), rel_score_cutoff=float(rng.choice([0.0, 0.8, 0.95])),
              left_end_bonus=int(rng.integers(0, 7)), right_end_bonus=int(rng.integers(0, 7)),
              forward_and_reverse_complement=bool(rng.random() < 0.8), allow_left_trim=bool(rng.random() < 0.8))
    if rng.random() < 0.4:
        kw.update(min_seed_length=k, max_seed_length=k)
    else:
        kw.update(min_seed_length=int(rng.integers(max(2, k - 6), k + 1)), max_seed_length=int(rng.choice([k, SIZE_MAX])))
    draw_cell_and_path_scores(rng, kw, 3 * 100)
    cfg = cli_defaults(k, **kw)
    read_src = seqs
    if mode == 1:
        seqs = seqs + [P.revcomp(s_) for s_ in seqs]
        read_src = seqs
    if mode == 2:
        seqs = P.primary_contigs(seqs, k)
    mask = bool(rng.random() < 0.25)
    g = O.OracleGraph(k, seqs, mask=mask)
    if mode:
        g.set_mode(mode)
    W, last, F, valid = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), valid=valid if mask else None, lib=lib, mode=mode)
    reads = []
    for i in range(nreads):
        s_ = read_src[int(rng.integers(0, len(read_src)))]
        L = int(rng.integers(k, 150)); p = int(rng.integers(0, max(1, len(s_) - L)))
        r = P.mutate(rng, s_[p:p + L], float(rng.choice([0.0, 0.0, 0.03, 0.08])))
        if rng.random() < 0.5: r = P.revcomp(r)
        if rng.random() < 0.15 and len(r) > 5: r = r[:len(r) // 2] + "N" + r[len(r) // 2 + 1:]
        reads.append(r)
    try:
        exp = _run(lib, idx, g, cfg, reads)
        if exp is None:
            return None
        if text:
            check_text(idx, cfg, reads)
        diff_t = sum(a != b for a, b in zip(exp, g.align_tsv(dataclasses.replace(cfg, score_matrix=transpose(m)),
                                                              reads, with_nodes=True)))
        diff_c = sum(a != b for a, b in zip(exp, g.align_tsv(dataclasses.replace(cfg, score_matrix=complemented(m)),
                                                              reads, with_nodes=True)))
        return diff_t, diff_c
    finally:
        idx.close()


def dna_matrix_family(lib, seeds, mode, text=False):
    """dna_matrix_case over `seeds`: every triple == oracle; at least half the configurations are accepted, and the
    oracle's lines under M^T and under complemented M differ from those under M for some reads, so a kernel that scored
    with either would fail. Returns the cases' results (None: rejected by both sides)."""
    out = [dna_matrix_case(lib, s, mode, text=text) for s in seeds]
    ok = [o for o in out if o is not None]
    assert len(ok) >= len(out) // 2, (len(ok), len(out))
    assert sum(t for t, _ in ok) > 0 and sum(c for _, c in ok) > 0, ok
    return out


def protein_matrix(rng, kind):
    if kind == "blosum62":
        return blosum62_scoring_matrix()
    if kind == "unit":
        return unit_scoring_matrix(int(rng.integers(1, 4)), PROTEIN)
    m = blosum62_scoring_matrix()
    diag = {c: int(rng.integers(1, 8)) for c in PROTEIN + "X"}
    for a in PROTEIN + "X":
        for b in PROTEIN + "X":
            m[ord(a)][ord(b)] = diag[a] if a == b else int(rng.integers(-4, 2))
    return m


def protein_case(lib, seed, nreads=20, text=False):
    """One randomized protein triple through the alphabet-generic layout (kern_any): k 2..30 (256-bit keys above 25),
    a random 25-letter matrix, BLOSUM62 or a unit matrix, masked graphs, alternative paths 1..3, max_seed_length, left
    trim, x-drop and end bonuses. Returns the oracle lines, or None when the configuration is rejected."""
    rng = np.random.default_rng(8000 + seed)
    k = int(rng.integers(2, 31))
    G = int(rng.integers(300, 2000))
    seqs = ["".join(np.array(list(P.AA))[rng.integers(0, 20, G)])]
    seqs += [P.mutate_aa(rng, seqs[0], 0.04) for _ in range(int(rng.integers(0, 2)))]
    kind = ("random", "blosum62", "unit")[seed % 3]
    kw = dict(alphabet="protein", score_matrix=protein_matrix(rng, kind), gap_opening_penalty=-int(rng.integers(5, 12)),
              gap_extension_penalty=-int(rng.integers(1, 4)), xdrop=int(rng.integers(5, 60)),
              min_exact_match=float(rng.choice([0.0, 0.0, 0.5])), num_alternative_paths=int(rng.integers(1, 4)),
              left_end_bonus=int(rng.integers(0, 7)), right_end_bonus=int(rng.integers(0, 7)),
              allow_left_trim=bool(rng.random() < 0.7), min_seed_length=int(rng.integers(max(1, k - 5), k + 1)),
              max_seed_length=int(rng.choice([k, SIZE_MAX, k + 3])))
    draw_cell_and_path_scores(rng, kw, 5 * 80)
    cfg = cli_defaults(k, **kw)
    mask = bool(rng.random() < 0.3)
    g = O.OracleGraph(k, seqs, alphabet="protein", mask=mask)
    valid = g.arrays()[3]
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib, alphabet=1), valid=valid if mask else None, lib=lib)
    reads = []
    for i in range(nreads):
        s_ = seqs[int(rng.integers(0, len(seqs)))]
        L = int(rng.integers(max(2, k), 120)); p = int(rng.integers(0, max(1, len(s_) - L)))
        r = P.mutate_aa(rng, s_[p:p + L], float(rng.choice([0.0, 0.03, 0.08])), 0.01)
        if i % 6 == 5 and len(r) > 4:
            r = r[:len(r) // 2] + "X" + r[len(r) // 2 + 1:]
        reads.append(r)
    try:
        exp = _run(lib, idx, g, cfg, reads)
        if text and exp is not None:
            check_text(idx, cfg, reads)
        return exp
    finally:
        idx.close()


# ---------------------------------------------------------------------------------------------------------------------
# Whole-read gates with per-letter diagonals: A/T and C/G score differently, so a read and its reverse complement have
# different exact-match sums, and a threshold between the two makes the answer depend on which strand matches.

def strand_matrix(diag):
    m = dna_scoring_matrix(2, -3, -3)
    for c in DNA:
        m[ord(c)][ord(c)] = diag[c]
    return m


WHOLE_READ_DIAGS = ({"A": 4, "C": 2, "G": 3, "T": 1}, {"A": 1, "C": 3, "G": 5, "T": 2})


def diag_sum(m, r):
    return sum(m[ord(c)][ord(c)] for c in r.upper() if c in DNA)


def whole_read_gate_case(lib, seed, diag, which, text=False):
    """Reads that are paths of the graph on one strand (exact seeder, both strands: the whole-read form of the
    shortcut answers them) under a per-letter diagonal, with `which` (min_path_score or min_cell_score) set between
    the Σ diag of a read and of its reverse complement for many of the reads. Even reads match the graph's forward
    strand, odd ones its reverse complement. Kernel == oracle shortcut on and off; on each strand the threshold changes
    the oracle's answer for some reads and leaves others aligned. The odd reads then run again on their own (shortcut
    on, == oracle), so that a count of whole-read answers taken around that run comes from reverse-complement reads
    only. Returns the emulation's whole-read hits of the full run and of the odd-read run (None on the device)."""
    rng = np.random.default_rng(seed)
    k, L, G = 15, 60, 3000
    m = strand_matrix(diag)
    base = "".join(np.array(list(DNA))[rng.integers(0, 4, G)])
    g = O.OracleGraph(k, [base])
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, [base], lib=lib), lib=lib)
    reads = []
    for i in range(60):
        p = int(rng.integers(0, G - L))
        reads.append(P.revcomp(base[p:p + L]) if i % 2 else base[p:p + L])
    mids = sorted((diag_sum(m, r) + diag_sum(m, P.revcomp(r))) // 2 for r in reads)
    thr = mids[len(mids) // 2]
    kw = dict(score_matrix=m, min_seed_length=k, max_seed_length=k, left_end_bonus=0, right_end_bonus=0,
              min_exact_match=0.0)
    cfg0 = cli_defaults(k, **kw)
    cfg = cli_defaults(k, **dict(kw, **{which: thr}))
    base_lines = g.align_tsv(cfg0, reads, with_nodes=True)
    try:
        h0 = P.whole_read_hits(lib)
        exp = _run(lib, idx, g, cfg, reads)
        h1 = P.whole_read_hits(lib)
        for strand in (0, 1):
            pairs = [(a, b) for i, (a, b) in enumerate(zip(base_lines, exp)) if i % 2 == strand]
            changed = sum(a != b for a, b in pairs)
            kept = sum(a == b and b.split("\t")[3] != "*" for a, b in pairs)
            assert changed > 0 and kept > 0, (which, thr, strand, changed, kept)
        odd = reads[1::2]
        got, _ = P.run_lines(idx, cfg, odd)
        h2 = P.whole_read_hits(lib)
        assert got == exp[1::2]
        if text:
            check_text(idx, cfg, reads)
    finally:
        idx.close()
    return None if h0 is None else (h1 - h0, h2 - h1)


# ---------------------------------------------------------------------------------------------------------------------
# The exact-path shortcut's gate reads the matrix as the extender does, M[graph letter][read letter]
# (profile_score_[c][j], extender.cpp:41-59). A graph letter g that scores more against the read's q than q does
# itself turns the shortcut off, while M[q][g] below the match does not matter.

def snp_gate_matrix():
    """M[C][A] = 3 > M[A][A] = 2 > M[A][C] = -3 and M[C][C] = 4, the same on the other strand (G, T). No read letter q
    scores M[q][g] at or above its match against any graph letter g; read A against graph C scores above the match"""
    m = dna_scoring_matrix(2, -3, -3)
    m[ord("C")][ord("A")] = m[ord("G")][ord("T")] = 3
    m[ord("C")][ord("C")] = m[ord("G")][ord("G")] = 4
    return m


def shortcut_gate_snp_case(lib, mode, exact_seeder):
    """Two haplotypes that differ by A (base) / C (variant) at a few sites, reads that are exact paths of the A
    haplotype across a site, on both strands, in BASIC (mode 0) or CANONICAL (mode 1) mode. The reference's extension
    takes the C branch there (a mismatch that scores 3 beats the match's 2), so no read is answered as `{L}=`: a gate
    that tested M[q][g] would let the shortcut answer them so. Kernel == oracle, shortcut on == off."""
    rng = np.random.default_rng(61 + mode)
    k, L = 15, 80
    base = list("".join(np.array(list(DNA))[rng.integers(0, 4, 3000)]))
    sites = list(range(300, 2800, 250))
    for p in sites:
        base[p] = "A"
    base = "".join(base)
    var = "".join("C" if i in sites else c for i, c in enumerate(base))
    seqs = [base, var]
    if mode == 1:
        seqs = seqs + [P.revcomp(s_) for s_ in seqs]
    g = O.OracleGraph(k, seqs)
    if mode:
        g.set_mode(mode)
    W, last, F, _ = g.arrays()
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), lib=lib, mode=mode)
    reads = []
    for i, p in enumerate(sites):
        r = base[p - 40:p + 40]
        reads += [r, P.revcomp(r)]
    kw = dict(score_matrix=snp_gate_matrix(), min_exact_match=0.0)
    if exact_seeder:
        kw.update(min_seed_length=k, max_seed_length=k)
    cfg = cli_defaults(k, **kw)
    try:
        exp = _run(lib, idx, g, cfg, reads)
    finally:
        idx.close()
    crossed = sum(1 for line in exp if "X" in line.split("\t")[6])
    assert crossed == len(reads), [line.split("\t")[2:7] for line in exp]


# ---------------------------------------------------------------------------------------------------------------------
# The bound of check_config_scores. The reference accepts a configuration when min_cell_score plus its lowest penalty
# does not leave int32; its DP column still adds more than one penalty to ninf. Configurations where no such sum
# leaves int32 (in_range) are pinned: lines == oracle. The others are kept with "no error" asserted only: the
# reference's own scalar statements overflow there (DESIGN.md §5).

def _mat(match, mm, nsc):
    m = dna_scoring_matrix(match, mm, mm)
    for a in DNA:
        m[ord(a)][ord("N")] = nsc
    return m


def _sd(**kw):
    """struct defaults with the CLI's node and RAM budgets: no x-drop on a 3-5 kbp graph explores it all otherwise"""
    return struct_defaults(max_nodes_per_seq_char=5.0, max_ram_per_alignment=200.0, **kw)


def bound_configs(k):
    lo128 = INT32_MIN + 128
    return {
        "cli_pen100": cli_defaults(k, score_matrix=_mat(2, -40, -100), gap_opening_penalty=-100,
                                   gap_extension_penalty=-100, min_exact_match=0.0),
        "match127_go51": cli_defaults(k, score_matrix=_mat(127, -40, -100), gap_opening_penalty=-51,
                                      gap_extension_penalty=-100, min_exact_match=0.0),
        "pen100_xdrop1000": cli_defaults(k, score_matrix=_mat(2, -40, -100), gap_opening_penalty=-100,
                                         gap_extension_penalty=-100, min_exact_match=0.0, xdrop=1000),
        "pen128_xdrop1": _sd(score_matrix=_mat(127, -128, -128), gap_opening_penalty=-128,
                                         gap_extension_penalty=-128, min_cell_score=lo128, xdrop=1),
        "match127_bonus127": cli_defaults(k, score_matrix=_mat(127, -3, -3), left_end_bonus=127, right_end_bonus=127,
                                          min_exact_match=0.0),
        "match127_mild": _sd(score_matrix=_mat(127, -20, -5), gap_opening_penalty=-30,
                                         gap_extension_penalty=-7, left_end_bonus=127, right_end_bonus=3),
        "go_eq_ge": cli_defaults(k, gap_opening_penalty=-3, gap_extension_penalty=-3, min_exact_match=0.0),
        "ge3": cli_defaults(k, gap_opening_penalty=-8, gap_extension_penalty=-3, min_exact_match=0.0, xdrop=60),
        "ge7_xdrop_max": cli_defaults(k, score_matrix=_mat(3, -8, -2), gap_opening_penalty=-9,
                                      gap_extension_penalty=-7, min_exact_match=0.0, xdrop=INT32_MAX),
        "ge100_at_edge": _sd(score_matrix=_mat(2, -1, -1), gap_opening_penalty=-1,
                                         gap_extension_penalty=-98, xdrop=1),
        "xdrop1": cli_defaults(k, xdrop=1, min_exact_match=0.0),
        "xdrop_max": cli_defaults(k, xdrop=INT32_MAX, min_exact_match=0.0),
    }


def probe_input():
    """two 3 kbp haplotypes at k = 15, 40 reads of 150 bp with 5 % errors on both strands, an N run, an exact read"""
    rng = np.random.default_rng(9)
    base = "".join(np.array(list(DNA))[rng.integers(0, 4, 3000)])
    seqs = [base, P.mutate(rng, base, 0.03)]
    reads = []
    for i in range(40):
        p = int(rng.integers(0, 3000 - 150))
        r = P.mutate(rng, seqs[i % 2][p:p + 150], 0.05)
        reads.append(P.revcomp(r) if i % 2 else r)
    reads += ["N" * 30 + base[100:200], base[500:600]]
    return 15, seqs, reads


def bound_case(lib, name, inp="probe", text=False):
    """returns whether the configuration is pinned (in_range). text: also the text route, TSV and JSON == the host
    mirror where pinned; where not, TSV lines whose scores reach the top of the int32 range"""
    k, seqs, reads = probe_input() if inp == "probe" else P.pressure_input(inp)[:3]
    cfg = bound_configs(k)[name]
    g = O.OracleGraph(k, seqs)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs, lib=lib), lib=lib)
    try:
        if text and in_range(cfg):
            check_text(idx, cfg, reads)
        elif text:
            # unpinned: the text route runs and each TSV line holds the read and int32 scores. No comparison with the
            # records: with wrapped scores the search may end differently when the records carry node ids (their arena
            # retry differs), and a path can end in a deletion with one node more than its sequence spells
            import text_common as T
            heads = [b"read%d" % i for i in range(len(reads))]
            text = T.run_text(idx, cfg, [T.as_bytes(r) for r in reads], heads, False)[0]
            lines = text.decode("latin1").split("\n")
            assert lines[-1] == "" and len(lines) == len(reads) + 1
            for line, h, r in zip(lines, heads, reads):
                f = line.split("\t")
                assert f[0] == h.decode() and f[1] == r and (len(f) - 2) % 6 == 0, line[:300]
                for a in range(2, len(f), 6):
                    assert f[a + 2] == "*" or INT32_MIN <= int(f[a + 2]) <= INT32_MAX, line[:300]
        if in_range(cfg):
            assert _run(lib, idx, g, cfg, reads) is not None
            return True
        # accepted by the reference's constructor; the oracle is not run: past the range its scores wrap and its search
        # need not end within any memory
        for sc in (True, False):
            got, _ = P.run_lines(idx, dataclasses.replace(cfg, no_exact_path_shortcut=sc), reads)
            assert len(got) == len(reads)
        return False
    finally:
        idx.close()


BOUND_PINNED = ("match127_bonus127", "match127_mild", "go_eq_ge", "ge3", "ge7_xdrop_max", "ge100_at_edge", "xdrop1",
                "xdrop_max")
BOUND_UNPINNED = ("cli_pen100", "match127_go51", "pen100_xdrop1000", "pen128_xdrop1")
