"""mgb_align_batch_text on the H100: the emulation's cases (tests/test_text_output_emu.py), the knobs that send reads down
other paths, capped grids on which k_text_size and k_text_write go round more than once, C2- and C3-shaped batches in
one piece and in several, and the C++ shim's text method. Every text block equals the host mirror over
mgb_align_batch's records byte for byte."""
import os
import re

import numpy as np
import pytest

import parity_common as P
import test_grid_rounds_gpu as G
import text_common as T
from metagraph_b200 import _lib
from metagraph_b200.aligner import B200Aligner, format_alignment, format_alignment_json
from metagraph_b200.config import cli_defaults

pytestmark = pytest.mark.gpu
LIB = None
LAUNCH = re.compile(r"launch (k_text_\w+) grid=(\d+) block=(\d+) per_round=(\d+) items=(\d+|dev)")
NAME = re.compile(rb'"name":"r(\d+)"')


def test_goldens_gpu():
    n = 0
    for idx, cfg, reads in T.goldens(LIB):
        T.check_text(idx, cfg, reads)
        n += 1
    assert n >= 47


@pytest.mark.parametrize("i", range(len(P.RANDOM_CASES)))
def test_random_gpu(i):
    T.random_case(LIB, i)


@pytest.mark.parametrize("i", range(len(P.PROTEIN_CASES)))
def test_protein_gpu(i):
    T.protein_case(LIB, i)


def test_whole_read_gpu():
    T.whole_read_case(LIB)


@pytest.mark.parametrize("mode", ["canonical", "primary"])
@pytest.mark.parametrize("seed", range(8))
def test_fuzz_modes_gpu(mode, seed):
    T.fuzz_case(LIB, seed, canonical=mode == "canonical", primary=mode == "primary")


@pytest.mark.parametrize("n_alt", [1, 5, 16, 32])
def test_alt_paths_gpu(n_alt):
    _, recs, _ = T.family_case(LIB, n_alt)
    assert max(len(p) for p in recs) == n_alt


def test_mt_goldens_gpu():
    T.check_mt_goldens(LIB)


def test_odd_inputs_gpu():
    T.odd_inputs_case(LIB)


def test_small_text_windows_gpu(monkeypatch):
    base, _, _ = T.family_case(LIB, 8)
    monkeypatch.setenv("MGB_TEST_TEXT_CAP", "997")
    assert T.family_case(LIB, 8)[0] == base


# knobs of test_spill_paths_gpu.py that send reads down other paths (index-build knobs are set before the index is made)
KNOBS = [("heap0", {"MGB_TEST_HEAP0": "60000"}), ("bmax64", {"MGB_TEST_BMAX": "64"}), ("pieces3", {"MGB_TEST_PIECES": "3"}),
         ("no_prepare_exact", {"MGB_TEST_NO_PREPARE_EXACT": "1"}), ("no_path_index", {"MGB_NO_PATH_INDEX": "1"}),
         ("wide", {"MGB_TEST_WIDE": "1"})]


@pytest.mark.parametrize("knob,env", KNOBS, ids=[k for k, _ in KNOBS])
def test_knobs_gpu(knob, env, monkeypatch):
    for var, val in env.items():
        monkeypatch.setenv(var, val)
    _, _, st = T.family_case(LIB, 32)
    if knob == "heap0":
        assert st["num_reads_retried"] > 0
    T.random_case(LIB, 5)          # exact k-mer seeds, k = 31: the whole-read routes
    T.whole_read_case(LIB)


def text_rounds(err):
    """per text kernel: the most rounds one launch went (k_text_write: at least, from the reads of the batch)"""
    out = {}
    for name, grid, block, per_round, items in LAUNCH.findall(err):
        n = int(items) if items != "dev" else None
        out.setdefault(name, []).append((int(per_round), n))
    return out


@pytest.mark.parametrize("blocks", [1, 3])
def test_text_grid_rounds_gpu(blocks, monkeypatch, capfd):
    """MGB_TEST_MAX_BLOCKS caps k_text_size and k_text_write: with 1 000 reads both go round at least twice, and the text
    is the same"""
    idx, reads, _ = T.random_inputs(LIB, 31, 15, 5000, 1000, 120, 0.03, nseq=2)
    cfg = cli_defaults(15, min_exact_match=0.0)
    try:
        capfd.readouterr()
        base, _, _ = T.check_text(idx, cfg, reads)
        monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
        monkeypatch.setenv("MGB_DEBUG", "1")
        capped, _, _ = T.check_text(idx, cfg, reads)
        err = capfd.readouterr().err
    finally:
        idx.close()
    assert capped == base
    r = text_rounds(err)
    assert len(r.get("k_text_size", [])) == 2 and len(r.get("k_text_write", [])) == 2, err[-2000:]
    for per_round, items in r["k_text_size"]:
        assert per_round == blocks * 8 and items == len(reads) and items >= 2 * per_round
    for per_round, _ in r["k_text_write"]:        # one window: every read of the batch
        assert per_round == blocks * 8 and len(reads) >= 2 * per_round


def test_text_shim_gpu(tmp_path):
    lib_dir = os.path.dirname(_lib.DEFAULT_LIB)
    T.check_shim(tmp_path, ["-L" + lib_dir, "-l:libmgb.so", "-Wl,-rpath," + lib_dir, "-fopenmp"], LIB)


# ------------------------------------------------------------------------------------------- at scale ----
def text_pair(idx, cfg, reads, headers, json, pieces):
    old = os.environ.get("MGB_TEST_PIECES")
    if pieces:
        os.environ["MGB_TEST_PIECES"] = str(pieces)
    try:
        al = B200Aligner(idx, cfg)
        return al.align_batch_text(list(zip(headers, reads)), json=json), al.last_stats
    finally:
        if pieces:
            if old is None:
                del os.environ["MGB_TEST_PIECES"]
            else:
                os.environ["MGB_TEST_PIECES"] = old


def check_scale(idx, k, cfg, reads, sample=20000, seed=0):
    """one piece == several pieces over the whole batch, in both formats; on a seeded sample of reads, located in the
    block by their line counts, text == the mirror over mgb_align_batch's records"""
    headers = [b"r%d" % i for i in range(len(reads))]
    rng = np.random.default_rng(seed)
    pick = np.sort(rng.choice(len(reads), min(sample, len(reads)), replace=False))
    recs = B200Aligner(idx, cfg).align_batch([(headers[i], reads[i]) for i in pick])
    for json in (False, True):
        one, st1 = text_pair(idx, cfg, reads, headers, json, 1)
        many, stp = text_pair(idx, cfg, reads, headers, json, None)
        assert one == many
        del many
        assert {c: st1[c] for c in T.COUNTERS} == {c: stp[c] for c in T.COUNTERS}
        lines = one.split(b"\n")
        del one
        assert lines[-1] == b""
        if not json:
            assert len(lines) == len(reads) + 1
            for j, i in enumerate(pick):
                exp = format_alignment(headers[i].decode(), recs[j], cfg.min_path_score).encode("latin1")
                assert lines[i] == exp, (i, lines[i][:300], exp[:300])
        else:
            # max(1, alignments) records per read, in read order: read i's records start where its name first appears
            first = {}
            r = -1
            for pos, line in enumerate(lines[:-1]):
                m = int(NAME.search(line).group(1))
                if m != r:
                    assert m == r + 1, (pos, m, r)
                    r = m
                    first[m] = pos
            assert r == len(reads) - 1
            for j, i in enumerate(pick):
                n = max(1, len(recs[j]))
                exp = format_alignment_json(headers[i].decode(), recs[j], k).encode("latin1")
                got = b"\n".join(lines[first[int(i)]:first[int(i)] + n])
                assert got == exp, (i, got[:300], exp[:300])


def test_c3_shape_text_gpu():
    k, Gn, n = 31, 2_000_000, 200_000
    rng = np.random.default_rng(3003)
    copies = G.c3_genome(rng, Gn)
    _, idx = G.scale_index(copies, k)
    reads = G.mutate_rows(rng, G.sample_reads(rng, copies, n, 150), 0.05)
    for i in range(0, n, 500):
        r = reads[i]
        reads[i] = r[:len(r) // 3] + "N" + r[len(r) // 3 + 1:]
    try:
        check_scale(idx, k, cli_defaults(k, min_exact_match=0.0), [r.encode() for r in reads])
    finally:
        idx.close()


def test_c2_shape_text_gpu():
    k, Gn, n = 31, 2_000_000, 140_000
    rng = np.random.default_rng(2002)
    genome = G.ACGT[rng.integers(0, 4, Gn)]
    _, idx = G.scale_index([genome], k)
    rows = G.sample_reads(rng, [genome], n, 150)
    hit = np.flatnonzero(rng.random(n) < 0.1)
    at = rng.integers(0, 150, len(hit))
    rows[hit, at] = ord("N")
    raw = rows.tobytes()
    reads = [raw[150 * i:150 * (i + 1)] for i in range(n)]
    try:
        check_scale(idx, k, cli_defaults(k, min_seed_length=k, max_seed_length=k), reads)
    finally:
        idx.close()
