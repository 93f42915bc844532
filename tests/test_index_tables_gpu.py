"""Every table the device builds inside mgb_index_create / mgb_index_set_mode, entry by entry, against the numpy
restatement in index_tables.py: radj (k_radj_*), the adjacency records (bits 0..15 as the host built them, bits 16..20 of
k_adj_rc), the k-mer hash index (k_kmer_insert), the path layout (k_path_*), every suffix-range level (k_sfx_extend above
the host-built ones) and the PRIMARY rc tables (k_rc_tables). The graphs have the shapes where these builds go wrong:
many path ends, cycles with and without a way in, k-mers that are their own child or their own reverse complement, many
dummies, a graph far below one thread block and one of over 4 M edges. The index comes from the test library
(tests/devtables), which compiles the product's api.cu unchanged. A structure the graph should have and did not get is a
failure, with the free device memory in the message."""
import os

import numpy as np
import pytest

import index_tables as IT
import parity_common as P
from metagraph_b200.aligner import BOSSTable

pytestmark = pytest.mark.gpu

EX = os.path.join(IT.ROOT, "tests", "golden", "example_graphs")


def require(info, hashed, paths=None):
    paths = hashed if paths is None else paths
    if hashed:
        assert info.kh_slots, "no k-mer hash index for n = %d, k = %d (%s)" % (info.n, info.k, IT.free_device_memory())
    if paths:
        assert info.pl_n, "no path layout for n = %d, k = %d (%s)" % (info.n, info.k, IT.free_device_memory())


def check_device(boss, valid, idx, hashed, primary=False, emu_compare=True, wide=False):
    info = IT.index_info(idx)
    require(info, hashed)
    T = IT.read_tables(idx)
    ref = IT.reference_for(boss, valid=valid, sfx_len=info.sfx_len)
    out = IT.check_index(ref, T, info, hashed=hashed, primary=primary)
    if emu_compare:
        # the host-built parts of the adjacency records are what the emulation builds for the same graph
        from metagraph_b200.aligner import DBGSuccinctIndex
        e = DBGSuccinctIndex(boss, valid=valid, lib=IT.EMU_LIB, suffix_len=info.sfx_len)
        E = IT.read_tables(e, ["adj", "wadj", "radj", "sfx"])
        e.close()
        if wide:
            assert (E["wadj"] == T["wadj"]).all()
        else:
            assert (E["adj"][:, 0] == T["adj"][:, 0]).all()
            assert ((E["adj"][:, 1] & 0xFFFF) == (T["adj"][:, 1] & 0xFFFF)).all()
            assert not (E["adj"][:, 1] >> 16).any()
        assert (E["radj"][1:] == T["radj"][1:]).all()
        if T["sfx"] is not None:
            assert (E["sfx"] == T["sfx"]).all()
    return ref, T, info, out


CASES = [  # shape, k, options; hashed unless k > 31 or wide
    ("mutated", 31, {}), ("mutated", 16, {"mask": True}), ("tandem", 12, {}), ("tandem", 4, {}),
    ("homopolymer", 16, {}), ("circular", 3, {}), ("both_orientations", 30, {}), ("palindromes", 12, {}),
    ("short_seqs", 31, {"mask": True}), ("short_seqs", 12, {}), ("one_kmer", 31, {}), ("one_kmer", 3, {}),
    ("empty", 12, {}), ("mutated", 13, {"suffix_len": 12}),
    ("palindromes", 12, {"mode": 2}), ("both_orientations", 31, {"mode": 2}), ("mutated", 16, {"mode": 2}),
    ("mutated", 2, {}), ("mutated", 32, {}), ("mutated", 33, {}), ("mutated", 20, {"wide": True}),
]


@pytest.mark.parametrize("shape,k,kw", CASES, ids=["%s-k%d%s" % (s, k, "".join("-%s%s" % (a, b) for a, b in kw.items()))
                                                   for s, k, kw in CASES])
def test_device_tables(shape, k, kw, monkeypatch):
    rng = np.random.default_rng(3000 + 37 * k + CASES.index((shape, k, kw)))
    seqs = IT.shape_seqs(shape, k, rng, 20000)
    mode = kw.get("mode", 0)
    if mode == 2:
        seqs = P.primary_contigs(seqs, k)
    if kw.get("wide"):
        monkeypatch.setenv("MGB_TEST_WIDE", "1")
    boss, valid, idx = IT.build_index(IT.TABLES_LIB, k, seqs, mask=kw.get("mask", False),
                                      suffix_len=kw.get("suffix_len", 0), mode=mode)
    hashed = 3 <= k <= 31 and not kw.get("wide")
    ref, T, info, out = check_device(boss, valid, idx, hashed, primary=mode == 2, wide=kw.get("wide", False))
    if kw.get("suffix_len"):
        assert info.sfx_len == kw["suffix_len"]            # levels 9 .. 12 refined on the device
    if (shape, k) in (("mutated", 31), ("palindromes", 12)):
        names = IT.assert_corruptions_rejected(ref, T, info, np.random.default_rng(5), expect_hash=True)
        if mode == 2:
            assert {"rcs zeroed", "palin bit"} <= set(names)
    if shape == "tandem" and k == 12:
        assert out["cycles"] >= 1, out                      # the lone cycle, which has no head
    idx.close()


def test_device_tables_dbg_files():
    boss = BOSSTable.from_dbg(os.path.join(EX, "test_DNA_graph.dbg"), lib=IT.TABLES_LIB)
    assert boss.k == 20
    for mask in (False, True):
        boss, valid, idx = IT.build_index(IT.TABLES_LIB, boss.k, None, boss=boss, mask=mask)
        check_device(boss, valid, idx, hashed=True)
        idx.close()
    boss = BOSSTable.from_dbg(os.path.join(EX, "test_Protein_graph.dbg"), lib=IT.TABLES_LIB)
    boss, valid, idx = IT.build_index(IT.TABLES_LIB, boss.k, None, boss=boss, mask=True)
    check_device(boss, valid, idx, hashed=False, wide=True)
    idx.close()


@pytest.mark.parametrize("k,s", [(2, 0), (6, 5), (12, 0)])
def test_device_tables_protein(k, s):
    rng = np.random.default_rng(4000 + k)
    boss, valid, idx = IT.build_index(IT.TABLES_LIB, k, IT.protein_seqs(rng, 60, 500), suffix_len=s, alphabet=1)
    ref, T, info, _ = check_device(boss, valid, idx, hashed=False, wide=True)
    if s:
        assert info.sfx_len == s                           # levels 4 and 5 refined on the device
    idx.close()


def test_device_tables_4m_edges():
    """a random 4 Mbp genome and a 1 % mutated copy: long probe chains, many pointer-jumping rounds, grid-stride loops
    that wrap many times"""
    rng = np.random.default_rng(4242)
    base = IT.random_seq(rng, 4_000_000)
    boss, valid, idx = IT.build_index(IT.TABLES_LIB, 31, [base, IT.mutate(rng, base, 0.01)])
    assert boss.num_edges >= 4_000_000
    ref, T, info, out = check_device(boss, valid, idx, hashed=True, emu_compare=False)
    print("4M-edge graph:", out)
    idx.close()
