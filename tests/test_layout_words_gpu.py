"""The whole-read gate's lookup tables (index.cuh IndexView::kh_pos and pl_word, built by k_layout_words) and the
pass-0 launch of k_align that reads its list's length from the device.

- Every kh_pos entry equals pl_pos[kh_vals[i]] of an in_graph edge and kPlNone otherwise (an empty slot, a dummy edge
  under the valid mask, an edge off the layout), and is kPlNone exactly where the host reference has no DBG node. Every
  pl_word is (pl_text[w], pl_stop[w] | pl_rc[w]) over all pl_n positions, the filler tail included. The tables are read
  through the test library tests/devlayout (the product's api.cu unchanged, plus read access).
- k_prepare_exact with the tables and with them left out (MGB_TEST_NO_LAYOUT_WORDS, read when the index is built)
  gives the same results, counters and answered reads, == oracle.
- k_align after k_exact_reads on pass 0 gets 0, 1 and many more reads than its resident warps, and a heap that
  overflows into the retry pass, at a capped grid (MGB_TEST_MAX_BLOCKS): results == oracle, and the reads it got are
  those the MGB_DEBUG lines report."""
import ctypes
import dataclasses
import os
import re

import numpy as np
import pytest

import index_tables as IT
import test_prepare_exact_gpu as PE
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from test_exact_reads_gpu import L, Case, substitute

pytestmark = pytest.mark.gpu

LAYOUT_LIB = os.path.join(IT.ROOT, "tests", "devlayout", "build", "libmgb_layout.so")
TABLES = {"kh_keys": np.uint64, "kh_vals": np.uint32, "kh_pos": np.uint32, "pl_pos": np.uint32, "pl_text": np.uint64,
          "pl_rc": np.uint32, "pl_stop": np.uint32, "pl_word": np.uint64, "valid": np.uint32}


def layout_tables(idx):
    """(n, kh_slots, pl_n), {name: host copy or None}"""
    L_ = idx._L
    L_.mgbl_layout_info.restype = ctypes.c_int
    L_.mgbl_layout_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L_.mgbl_layout_copy.restype = ctypes.c_int64
    L_.mgbl_layout_copy.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p]
    info = np.zeros(3, np.uint64)
    assert L_.mgbl_layout_info(idx.handle, info.ctypes.data) == 0
    out = {}
    for name, dt in TABLES.items():
        size = L_.mgbl_layout_copy(idx.handle, name.encode(), None)
        assert size >= 0, L_.mgb_last_error().decode()
        if not size:
            out[name] = None
            continue
        a = np.empty(size // np.dtype(dt).itemsize, dt)
        assert L_.mgbl_layout_copy(idx.handle, name.encode(), a.ctypes.data) == size
        out[name] = a
    return tuple(int(x) for x in info), out


def check_layout_words(boss, valid, idx):
    (n, slots, pl_n), T = layout_tables(idx)
    assert slots and pl_n, "no hash index or path layout (%s)" % IT.free_device_memory()
    assert T["kh_pos"] is not None and T["pl_word"] is not None, "no kh_pos / pl_word (%s)" % IT.free_device_memory()
    # kh_pos: pl_pos of the slot's edge when it is in_graph, else kPlNone
    keys, vals, pos = T["kh_keys"], T["kh_vals"].astype(np.int64), T["pl_pos"]
    e = np.where(keys != 0, vals, 0)
    ok = (e > 0) & (e <= n)
    if T["valid"] is not None:
        ok &= ((T["valid"][e >> 5] >> (e & 31).astype(np.uint32)) & 1).astype(bool)
    want = np.where(ok, pos[e], np.uint32(IT.PL_NONE)).astype(np.uint32)
    bad = np.flatnonzero(T["kh_pos"] != want)
    assert not len(bad), ("kh_pos", int(bad[0]), int(T["kh_pos"][bad[0]]), int(want[bad[0]]), len(bad))
    ref = IT.reference_for(boss, valid=valid)
    placed = (keys != 0) & ref.P[e]
    assert ((T["kh_pos"] != IT.PL_NONE) == placed).all(), "kh_pos: placed iff the slot holds a DBG node"
    # pl_word: (text, stop | rc, high half 0) per 32 positions, all pl_n of them
    w = T["pl_word"].reshape(-1, 2)
    assert len(w) == pl_n // 32 == len(T["pl_stop"]) == len(T["pl_rc"]) == len(T["pl_text"])
    assert (w[:, 0] == T["pl_text"]).all(), "pl_word text"
    assert (w[:, 1] == (T["pl_stop"] | T["pl_rc"]).astype(np.uint64)).all(), "pl_word mask"
    assert (T["pl_stop"][-(IT.PL_PAD // 32):] == 0xFFFFFFFF).all()        # the filler tail is covered
    return placed.sum()


SHAPES = [("mutated", 31), ("tandem", 12), ("circular", 3), ("both_orientations", 30), ("palindromes", 12),
          ("short_seqs", 31), ("one_kmer", 31)]
CASES = [(s, k, m) for s, k in SHAPES for m in (False, True)]


@pytest.mark.parametrize("shape,k,mask", CASES, ids=["%s-k%d%s" % (s, k, "-mask" if m else "") for s, k, m in CASES])
def test_layout_words_tables_gpu(shape, k, mask):
    rng = np.random.default_rng(6000 + 37 * k + CASES.index((shape, k, mask)))
    seqs = IT.shape_seqs(shape, k, rng, 20000)
    boss, valid, idx = IT.build_index(LAYOUT_LIB, k, seqs, mask=mask)
    assert check_layout_words(boss, valid, idx) > 0
    idx.close()


def test_layout_words_tables_4m_edges_gpu():
    rng = np.random.default_rng(4242)
    base = IT.random_seq(rng, 4_000_000)
    boss, valid, idx = IT.build_index(LAYOUT_LIB, 31, [base, IT.mutate(rng, base, 0.01)])
    assert boss.num_edges >= 4_000_000
    check_layout_words(boss, valid, idx)
    idx.close()


def test_layout_words_absent_gpu(monkeypatch):
    """MGB_TEST_NO_LAYOUT_WORDS leaves both tables out; the index is that much smaller"""
    rng = np.random.default_rng(6100)
    seqs = IT.shape_seqs("mutated", 31, rng, 20000)
    boss, _, idx = IT.build_index(LAYOUT_LIB, 31, seqs)
    monkeypatch.setenv("MGB_TEST_NO_LAYOUT_WORDS", "1")
    off = DBGSuccinctIndex(boss, lib=LAYOUT_LIB)
    monkeypatch.delenv("MGB_TEST_NO_LAYOUT_WORDS")
    (_, slots, pl_n), T = layout_tables(off)
    assert T["kh_pos"] is None and T["pl_word"] is None and pl_n
    assert idx.device_bytes - off.device_bytes == 4 * slots + pl_n // 2
    idx.close()
    off.close()


# ---------------------------------------------------------------------------------------------------------------------
# the route with the tables and without

def graphs(k, seqs, monkeypatch):
    """the test_prepare_exact_gpu Graph of `seqs`, and the same graph's index built without kh_pos / pl_word"""
    g = PE.Graph(k, seqs, monkeypatch)
    monkeypatch.setenv("MGB_TEST_NO_LAYOUT_WORDS", "1")
    W, last, F, _ = g.og.arrays()
    off =DBGSuccinctIndex(BOSSTable(k, W, last, F))
    monkeypatch.delenv("MGB_TEST_NO_LAYOUT_WORDS")
    assert g.idx.device_bytes > off.device_bytes          # the route's index has the tables, the other not
    return g, off


LEFT = re.compile(r"k_exact_reads answered \d+, left to k_align (\d+)")


@pytest.mark.parametrize("k", [31, 15])
def test_layout_words_route_gpu(k, monkeypatch, capfd):
    """mixed reads and reads across path ends: results (with and without node ids), headers, counters and the answered
    count identical with the tables and without them, == oracle"""
    case = Case(k, 6200 + k)
    g, off = graphs(k, case.seqs, monkeypatch)
    reads = case.mixed_reads() + case.exact_reads(300)
    for i in range(0, 300, 17):
        reads[-1 - i] = substitute(reads[-1 - i], (13 * i) % L)
    n = PE.check(g, reads, monkeypatch, capfd)              # with the tables, == oracle, == the route off
    assert 0 < n < len(reads)
    cfg = cli_defaults(k, min_seed_length=k, max_seed_length=k)
    for result_nodes in (0, 1):
        c = dataclasses.replace(cfg, result_nodes=result_nodes)
        on = PE.run(g.idx, c, reads, True, monkeypatch, capfd)
        without = PE.run(off, c, reads, True, monkeypatch, capfd)
        assert on[0] == without[0] and on[1] == without[1] and on[2] == without[2] == n
        assert LEFT.findall(on[3]) == LEFT.findall(without[3])
    off.close()
    g.close()


# ---------------------------------------------------------------------------------------------------------------------
# k_align on pass 0 without the host's read-back

def align_launch_items(err):
    return [int(m) for m in re.findall(r"launch k_align grid=\d+ block=\d+ per_round=\d+ items=(\d+)", err)]


@pytest.mark.parametrize("blocks", [1, 3])
@pytest.mark.parametrize("n_left", [0, 1, 200])
def test_align_list_on_device_gpu(n_left, blocks, monkeypatch, capfd):
    """n_left reads with a substitution among 400 error-free ones: k_align gets exactly those (0, 1, or far more than
    the 4 / 12 warps of 1 / 3 blocks), == oracle; a warp without a read does nothing, the counters are those of the
    default grid"""
    case = Case(31, 6300 + n_left)
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(400)
    for i in range(n_left):
        reads[2 * i] = substitute(reads[2 * i], (11 * i + 5) % L)
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    base = PE.run(g.idx, cfg, reads, True, monkeypatch, capfd)
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", str(blocks))
    lines, stats, n, err = PE.run(g.idx, cfg, reads, True, monkeypatch, capfd)
    assert lines == g.og.align_tsv(cfg, reads, with_nodes=True)
    assert stats == base[1] and n == base[2]
    assert [int(x) for x in LEFT.findall(err)] == [n_left]
    assert align_launch_items(err)[:1] == [n_left]               # pass 0's launch, with the resident grid
    assert stats["num_reads_retried"] == 0
    g.close()


def test_align_list_on_device_retry_gpu(monkeypatch, capfd):
    """pass 0's heap holds a few records (MGB_TEST_HEAP0): k_align's reads overflow and the retry pass answers them with
    the count read back; == oracle"""
    case = Case(31, 6400)
    g = PE.Graph(31, case.seqs, monkeypatch)
    reads = case.exact_reads(300)
    for i in range(0, 300, 3):
        reads[i] = substitute(reads[i], (7 * i) % L)
    cfg = cli_defaults(31, min_seed_length=31, max_seed_length=31)
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", "1")
    monkeypatch.setenv("MGB_TEST_HEAP0", str(60 * 400))
    lines, stats, n, err = PE.run(g.idx, cfg, reads, True, monkeypatch, capfd)
    assert lines == g.og.align_tsv(cfg, reads, with_nodes=True)
    assert stats["num_reads_retried"] > 0 and len(align_launch_items(err)) >= 2
    g.close()
