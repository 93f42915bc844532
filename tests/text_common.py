"""Case driver of the text route (mgb_align_batch_text): the same reads go through mgb_align_batch (records with node
ids) and through mgb_align_batch_text in both formats. The text block must equal the host mirror
(aligner.format_alignment / format_alignment_json) over the records byte for byte, and both calls must report the same
alignment counts and search counters."""
import ctypes
import dataclasses

import numpy as np

import oracle_lib as O
import parity_common as P
from metagraph_b200 import _lib
from metagraph_b200.aligner import (B200Aligner, BOSSTable, DBGSuccinctIndex, _pack, format_alignment,
                                    format_alignment_json)
from metagraph_b200.config import SIZE_MAX, cli_defaults, dna_scoring_matrix

COUNTERS = ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns")


def as_bytes(x):
    return x.encode("latin1") if isinstance(x, str) else bytes(x)


def mirror_text(recs, headers, cfg, k, json):
    """the mirror's bytes: format_alignment(_json)(header, paths) + "\\n" per read (headers as latin1 text)"""
    out = []
    for h, p in zip(headers, recs):
        h = h.decode("latin1")
        out.append((format_alignment_json(h, p, k) if json else format_alignment(h, p, cfg.min_path_score)) + "\n")
    return "".join(out).encode("latin1")


def run_text(idx, cfg, reads, headers, json):
    """mgb_align_batch_text: (text, stats, number of alignments, per-read counts). Also checks that the text result set
    has no records and cannot be exported."""
    al = B200Aligner(idx, cfg)
    L = al._L
    buf, offs = _pack(reads)
    hbuf, hoffs = _pack(headers)
    res = al.align_batch_text_raw(buf, offs, hbuf, hoffs, json)
    try:
        text = al.text_of(res)
        stats = al.stats_of(res)
        n_alns = L.mgb_results_num_alignments(res)
        assert L.mgb_results_num_reads(res) == len(reads)
        first, count = ctypes.c_uint64(), ctypes.c_uint32()
        counts = []
        for r in range(len(reads)):
            L.mgb_results_read_range(res, r, ctypes.byref(first), ctypes.byref(count))
            assert first.value == sum(counts)
            counts.append(count.value)
        assert not L.mgb_results_alignments(res)
        scratch = np.zeros(1 << 16, np.uint8)
        assert L.mgb_results_export(res, scratch.ctypes.data, len(scratch)) == -1
    finally:
        al.free_raw(res)
    return text, stats, n_alns, counts


def first_difference(got, exp):
    g, e = got.split(b"\n"), exp.split(b"\n")
    for i, (a, b) in enumerate(zip(g, e)):
        if a != b:
            return i, a[:600], b[:600]
    return min(len(g), len(e)), len(g), len(e)


def check_text(idx, cfg, reads, headers=None, formats=(False, True)):
    """records vs text for one input; returns ({json: text}, records, record-route stats)"""
    reads = [as_bytes(r) for r in reads]
    headers = [as_bytes(h) for h in headers] if headers is not None else [b"read%d" % i for i in range(len(reads))]
    cfg_rec = dataclasses.replace(cfg, result_nodes=0)
    al = B200Aligner(idx, cfg_rec)
    recs = al.align_batch(list(zip(headers, reads)))
    st = al.last_stats
    out = {}
    for json in formats:
        text, stats, n_alns, counts = run_text(idx, cfg, reads, headers, json)
        exp = mirror_text(recs, headers, cfg, idx.k, json)
        assert text == exp, ("json" if json else "tsv", first_difference(text, exp))
        assert counts == [len(p) for p in recs]
        assert n_alns == sum(counts)
        diff = {c: (st[c], stats[c]) for c in COUNTERS if st[c] != stats[c]}
        assert not diff, diff
        retried = st["num_reads_retried"]
        if not json and stats["num_reads_retried"] != retried:
            # TSV records carry no node ids: a heap that overflows with them may not overflow without them
            nodeless = B200Aligner(idx, dataclasses.replace(cfg, result_nodes=1))
            nodeless.align_batch(list(zip(headers, reads)))
            retried = nodeless.last_stats["num_reads_retried"]
        assert stats["num_reads_retried"] == retried, (stats["num_reads_retried"], retried)
        assert stats["d2h_bytes"] >= len(text)
        out[json] = text
    return out, recs, st


# ------------------------------------------------------------------------------------------------ inputs ----
def goldens(lib):
    """the test_aligner goldens: (graph index, config, query) triples"""
    import json
    import os
    from test_oracle_golden import GOLD, make_cfg, revcomp
    for gold in json.load(open(os.path.join(GOLD, "test_aligner_goldens.json"))):
        g = O.OracleGraph(gold["k"], gold["refs"], mask=gold["mask"], dynamic=not gold["mask"])
        W, last, F, valid = g.arrays()
        idx = DBGSuccinctIndex(BOSSTable(gold["k"], W, last, F), valid=valid if gold["mask"] else None, lib=lib)
        query = revcomp(gold["query"]) if gold["rc_query"] else gold["query"]
        for uni in ([False, True] if gold["extend"] else [False]):
            cfg = make_cfg(gold["cfg"])
            if uni:
                cfg.max_seed_length = SIZE_MAX
            yield idx, cfg, [query]
        idx.close()


def random_inputs(lib, seed, k, G, nreads, L, rate, mask=False, nseq=1):
    """parity_common.random_case's graph and reads"""
    rng = np.random.default_rng(seed)
    seqs = ["".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])]
    seqs += [P.mutate(rng, seqs[0], 0.02) for _ in range(nseq - 1)]
    boss = BOSSTable.from_sequences(k, seqs, lib=lib)
    idx = DBGSuccinctIndex(boss, valid=boss.dummy_mask(lib=lib) if mask else None, lib=lib)
    reads = []
    for i in range(nreads):
        s = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, max(1, len(s) - L)))
        r = P.mutate(rng, s[p:p + L], rate)
        if rng.random() < 0.5:
            r = r.translate(P.COMP)[::-1]
        if rng.random() < 0.05 and len(r) > 2:
            r = r[:len(r) // 2] + "N" + r[len(r) // 2 + 1:]
        reads.append(r)
    reads += ["", "A", "ACGT" * 3, "N" * 40]
    return idx, reads, seqs


def random_case(lib, i, nreads=None):
    seed, k, G, n, L, rate, cfg, mask, nseq = P.RANDOM_CASES[i]
    idx, reads, _ = random_inputs(lib, seed, k, G, nreads or n, L, rate, mask, nseq)
    try:
        return check_text(idx, cfg(k) if callable(cfg) else cfg, reads)
    finally:
        idx.close()


def protein_case(lib, i):
    seed, k, G, nreads, L, rate, cfg, mask, nseq, indel = P.PROTEIN_CASES[i]
    rng = np.random.default_rng(seed)
    seqs = ["".join(np.array(list(P.AA))[rng.integers(0, 20, G)])]
    seqs += [P.mutate_aa(rng, seqs[0], 0.03) for _ in range(nseq - 1)]
    seqs[-1] = seqs[-1][:G // 2] + "XBZ" + seqs[-1][G // 2:]
    boss = BOSSTable.from_sequences(k, seqs, lib=lib, alphabet=1)
    idx = DBGSuccinctIndex(boss, valid=boss.dummy_mask(lib=lib) if mask else None, lib=lib)
    reads = []
    for j in range(nreads):
        s_ = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, max(1, len(s_) - L)))
        r = P.mutate_aa(rng, s_[p:p + L], rate, indel)
        if j % 7 == 3 and len(r) > 4:
            r = r[:len(r) // 2] + "X*" + r[len(r) // 2 + 2:]
        if j % 5 == 1:
            r = r.lower()
        reads.append(r)
    reads += ["", "A", "ACDE", "X" * 30, "**********"]
    try:
        return check_text(idx, cfg(k), reads)
    finally:
        idx.close()


def whole_read_case(lib, seed=3, k=15, nreads=60):
    """exact k-mer seeds on reads that are exact substrings of the graph: whole-read exact answers"""
    idx, reads, seqs = random_inputs(lib, seed, k, 3000, 0, 80, 0.0, nseq=2)
    rng = np.random.default_rng(seed)
    for i in range(nreads):
        s = seqs[i % 2]
        p = int(rng.integers(0, len(s) - 90))
        r = s[p:p + int(rng.integers(k, 90))]
        reads.append(P.revcomp(r) if i % 3 == 0 else r)
    cfg = cli_defaults(k, min_seed_length=k, max_seed_length=k)
    try:
        return check_text(idx, cfg, reads)
    finally:
        idx.close()


def fuzz_case(lib, seed, canonical=False, primary=False, nreads=25):
    """parity_common.fuzz_case's (graph, reads, config) triple on a CANONICAL or PRIMARY graph"""
    rng = np.random.default_rng(1000 + seed)
    k = int(rng.integers(4, 34))
    G = int(rng.integers(300, 4000))
    nseq = int(rng.integers(1, 4))
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, G)])
    seqs = [base] + [P.mutate(rng, base, 0.03) for _ in range(nseq - 1)]
    if rng.random() < 0.3:
        u = base[:int(rng.integers(k, 3 * k))]
        seqs.append(u * int(rng.integers(2, 5)) + base[50:120])
    match = int(rng.integers(1, 4)); mm1 = -int(rng.integers(1, 5)); mm2 = -int(rng.integers(1, 5))
    go = -int(rng.integers(2, 9)); ge = -int(rng.integers(1, min(-go, 4) + 1))
    kw = dict(score_matrix=dna_scoring_matrix(match, mm1, mm2), gap_opening_penalty=go, gap_extension_penalty=ge,
              xdrop=int(rng.integers(5, 60)), min_exact_match=float(rng.choice([0.0, 0.0, 0.3, 0.7])),
              rel_score_cutoff=float(rng.choice([0.0, 0.5, 0.8, 0.95])),
              num_alternative_paths=int(rng.integers(1, 4)),
              forward_and_reverse_complement=bool(rng.random() < 0.7),
              left_end_bonus=int(rng.integers(0, 7)), right_end_bonus=int(rng.integers(0, 7)),
              max_nodes_per_seq_char=float(rng.choice([5.0, 2.0, 12.0])),
              allow_left_trim=bool(rng.random() < 0.8),
              seed_complexity_filter=bool(rng.random() < 0.3))
    msl = int(rng.integers(2, k + 1)); kw["min_seed_length"] = msl
    kw["max_seed_length"] = int(rng.choice([k, SIZE_MAX, max(msl, k - 1), k + 5]))
    if kw["max_seed_length"] < msl:
        kw["max_seed_length"] = msl
    kw["max_num_seeds_per_locus"] = int(rng.choice([1000, 2, SIZE_MAX]))
    cfg = cli_defaults(k, **kw)
    mask = bool(rng.random() < 0.3)
    read_src = seqs
    if canonical:
        seqs = seqs + [P.revcomp(s_) for s_ in seqs]
        read_src = seqs
    if primary:
        seqs = P.primary_contigs(seqs, k)
    g = O.OracleGraph(k, seqs, mask=mask)
    if canonical or primary:
        g.set_mode(2 if primary else 1)
    W, last, F, valid = g.arrays()
    reads = []
    for i in range(nreads):
        s_ = read_src[int(rng.integers(0, len(read_src)))]
        L = int(rng.integers(max(3, k - 3), 160))
        p = int(rng.integers(0, max(1, len(s_) - L)))
        r = P.mutate(rng, s_[p:p + L], float(rng.choice([0.0, 0.02, 0.08])))
        if rng.random() < 0.5:
            r = r.translate(P.COMP)[::-1]
        if rng.random() < 0.1 and len(r) > 5:
            r = r[:len(r) // 2] + "N" + r[len(r) // 2 + 1:]
        reads.append(r)
    idx = DBGSuccinctIndex(BOSSTable(k, W, last, F), valid=valid if mask else None, lib=lib,
                           mode=2 if primary else 1 if canonical else 0)
    try:
        B200Aligner(idx, cfg)
    except _lib.MgbError as e:                     # check_config_scores: the text route refuses it the same way
        assert e.code == -3
        _assert_text_refused(idx, cfg, reads, -3)
        idx.close()
        return None
    try:
        return check_text(idx, cfg, reads)
    finally:
        idx.close()


def _assert_text_refused(idx, cfg, reads, code):
    L = idx._L
    c = cfg.to_c()
    buf, offs = _pack([as_bytes(r) for r in reads])
    hbuf, hoffs = _pack([b""] * len(reads))
    res = ctypes.c_void_p()
    for fmt in (1, 2):
        assert L.mgb_align_batch_text(idx.handle, ctypes.byref(c), buf.ctypes.data, offs.ctypes.data,
                                      hbuf.ctypes.data, hoffs.ctypes.data, len(reads), fmt, ctypes.byref(res)) == code


def family_case(lib, n_alt, seeder="exact", rel=0.0, reads=None):
    """the alternative-paths gene-family graph at num_alternative_paths = n_alt"""
    import alt_paths_common as A
    seqs, fam_reads, _ = A.family_graph()
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(A.K, seqs, lib=lib), lib=lib)
    try:
        return check_text(idx, A.config(n_alt, seeder, rel), reads or fam_reads)
    finally:
        idx.close()


def mt_index(lib):
    import os
    from test_oracle_golden import GOLD, read_fasta, read_fastq
    _, seqs = read_fasta(os.path.join(GOLD, "genome.MT.fa"))
    names, reads = read_fastq(os.path.join(GOLD, "genome_MT1.fq"))
    return DBGSuccinctIndex(BOSSTable.from_sequences(11, seqs, lib=lib), lib=lib), names, reads


def check_mt_goldens(lib):
    """the reference's MT TSV lines (integration_tests/test_align.py) and its two JSON golden files, straight out of
    the text block"""
    import os
    from test_oracle_golden import GOLD, MT_BOTH, MT_FWD
    idx, names, reads = mt_index(lib)
    try:
        for both, gold in ((False, MT_FWD), (True, MT_BOTH)):
            cfg = cli_defaults(11, min_exact_match=0.0, forward_and_reverse_complement=both)
            out, _, _ = check_text(idx, cfg, reads, names)
            lines = out[False].decode("latin1").split("\n")
            assert lines[-1] == "" and len(lines) == len(reads) + 1
            assert lines[:5] == gold
        for gold_file, edit in (("genome_MT1.align.json", False), ("genome_MT1.align.edit.json", True)):
            cfg = cli_defaults(11, min_exact_match=0.0, edit_distance=edit)
            out, _, _ = check_text(idx, cfg, reads, names, formats=(True,))
            gold = [l.rstrip() for l in open(os.path.join(GOLD, gold_file)) if l.strip()]
            assert out[True].decode("latin1").split("\n")[:5] == gold
    finally:
        idx.close()


ODD_HEADERS = [b"tab\there", b'quote"d', b"back\\slash", b"new\nline", b"ctl\x01\x1f", b"latin\xe9\xff\x80",
               b"", b"utf8 \xc3\xa9", b"plain"]


def odd_inputs_case(lib):
    """headers with tab, '"', '\\', newline, control bytes, bytes >= 0x80 and the empty header; reads that are empty,
    shorter than k, all N, lower case, or carry bytes >= 0x80 and JSON-special characters; unaligned reads under a
    non-zero min_path_score"""
    idx, reads, seqs = random_inputs(lib, 5, 15, 3000, 20, 100, 0.02)
    g = seqs[0]
    extra = [b"", b"ACG", b"N" * 50, g[100:220].lower().encode(), (g[300:360] + "\xe9\x80" + g[362:440]).encode("latin1"),
             (g[500:560] + '"\\\t' + g[563:640]).encode("latin1"), b"\x01\x02" + g[700:800].encode(),
             P.revcomp(g[900:1000]).lower().encode() + b"\xff", b"acgtRYKMBVDHUN`" * 3]
    reads = [as_bytes(r) for r in reads] + extra
    headers = [ODD_HEADERS[i % len(ODD_HEADERS)] + b"#%d" % i if i % 4 else ODD_HEADERS[i % len(ODD_HEADERS)]
               for i in range(len(reads))]
    try:
        out = []
        for mps in (0, 230):
            o, recs, _ = check_text(idx, cli_defaults(15, min_path_score=mps, min_exact_match=0.0), reads, headers)
            out.append((o, recs))
        assert sum(1 for p in out[1][1] if not len(p)) > sum(1 for p in out[0][1] if not len(p))
        assert b"\t*\t*\t230\t*\t*\t*\n" in out[1][0][False]
        return out
    finally:
        idx.close()


SHIM_BATCH = [(b"q1", b"AGCTNCGAGGCCAA"), (b'q\t2 "x"', b"TTGGCCTCGNAGCT"), (b"", b""), (b"q4", b"ACGTACGTNNN"),
              (b"q5", b"agctncgaggccaa")]


def check_shim(tmp_path, link_flags, lib):
    """tests/cpp/test_text_shim.cpp (B200Aligner::align_batch_text of the C++ shim) prints the same TSV and JSON blocks
    as the Python binding on the same library"""
    import os
    import subprocess
    from metagraph_b200.aligner import BOSSTable
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_text_shim")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(root, "tests", "cpp", "test_text_shim.cpp"), "-o", exe]
                          + link_flags)
    dbg = os.path.join(root, "tests", "golden", "example_graphs", "test_DNA_graph.dbg")
    out = subprocess.run([exe, dbg], capture_output=True)
    assert out.returncode == 0, out.stdout + out.stderr
    boss = BOSSTable.from_dbg(dbg, lib=lib)
    idx = DBGSuccinctIndex(boss, lib=lib)
    try:
        al = B200Aligner(idx, cli_defaults(boss.k, min_exact_match=0.0, num_alternative_paths=2))
        tsv, json = al.align_batch_text(SHIM_BATCH), al.align_batch_text(SHIM_BATCH, json=True)
    finally:
        idx.close()
    assert out.stdout == tsv + b"--\n" + json
    assert tsv.count(b"\n") == len(SHIM_BATCH) and b"q1\tAGCTNCGAGGCCAA\t" in tsv
    return tsv, json
