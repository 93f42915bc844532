"""The index tables of the host emulation against the numpy restatement in index_tables.py (radj, the adjacency records'
bits 0..15, every suffix-range level, the PRIMARY rc tables), and that restatement against the oracle: bwd, the per-edge
k-mer and the several-incoming flag of every edge. The emulation builds no hash index and no path layout; their
contracts are checked on the device (test_index_tables_gpu.py)."""
import subprocess

import numpy as np
import pytest

import index_tables as IT
import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable

EX = IT.os.path.join(IT.ROOT, "tests", "golden", "example_graphs")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", IT.os.path.join(IT.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


def oracle_graphs():
    rng = np.random.default_rng(41)
    yield "mutated-k12", BOSSTable.from_sequences(12, IT.shape_seqs("mutated", 12, rng, 1500), lib=IT.EMU_LIB), "dna"
    yield "short_seqs-k5", BOSSTable.from_sequences(5, IT.shape_seqs("short_seqs", 5, rng), lib=IT.EMU_LIB), "dna"
    yield "tandem-k2", BOSSTable.from_sequences(2, IT.shape_seqs("tandem", 2, rng, 300), lib=IT.EMU_LIB), "dna"
    yield "protein-k6", BOSSTable.from_sequences(6, IT.protein_seqs(rng, 10, 120), lib=IT.EMU_LIB, alphabet=1), \
        "protein"
    yield "test_DNA_graph", BOSSTable.from_dbg(IT.os.path.join(EX, "test_DNA_graph.dbg"), lib=IT.EMU_LIB), "dna"
    yield "test_Protein_graph", BOSSTable.from_dbg(IT.os.path.join(EX, "test_Protein_graph.dbg"), lib=IT.EMU_LIB), \
        "protein"


def test_reference_against_oracle():
    """bwd == BOSS::bwd, x(e) == get_node_sequence(e), the flag == !is_single_incoming, for every edge"""
    L = O.lib()
    for name, boss, alphabet in oracle_graphs():
        ref = IT.reference_for(boss, keep_codes=True)
        og = O.OracleGraph(boss.k, arrays=(boss.W, boss.last, boss.F), alphabet=alphabet)
        edges = range(1, ref.n + 1)
        bwd = np.array([L.mgo_boss_bwd(og.h, e) for e in edges])
        assert (bwd == ref.bwd[1:]).all(), (name, "bwd", int(np.flatnonzero(bwd != ref.bwd[1:])[0]) + 1)
        seqs = [og.node_sequence(e) for e in edges]
        mine = ref.kmer_strings(edges)
        bad = [e for e, a, b in zip(edges, seqs, mine) if a != b]
        assert not bad, (name, "k-mer", bad[0], seqs[bad[0] - 1], mine[bad[0] - 1])
        single = np.array([L.mgo_boss_is_single_incoming(og.h, e) for e in edges]).astype(bool)
        assert (single == ~ref.multi[1:]).all(), (name, "flag", int(np.flatnonzero(single == ref.multi[1:])[0]) + 1)
        assert (ref.clean[1:] == np.array(["$" not in s for s in seqs])).all(), name
        if alphabet == "dna":
            assert len(ref.K) == int(ref.clean.sum())


def emu_case(shape, k, mask=False, suffix_len=0, mode=0, seed=0, wide=False, monkeypatch=None):
    rng = np.random.default_rng(1000 + 31 * k + seed)
    seqs = IT.shape_seqs(shape, k, rng, 2500)
    if mode == 2:
        seqs = P.primary_contigs(seqs, k)
    if wide:
        monkeypatch.setenv("MGB_TEST_WIDE", "1")
    boss, valid, idx = IT.build_index(IT.EMU_LIB, k, seqs, mask=mask, suffix_len=suffix_len, mode=mode)
    if wide:
        monkeypatch.delenv("MGB_TEST_WIDE")
    return boss, valid, idx


EMU_CASES = [("mutated", 12, {}), ("mutated", 31, {"mask": True}), ("tandem", 4, {}), ("homopolymer", 16, {}),
             ("circular", 3, {}), ("short_seqs", 30, {"mask": True}), ("one_kmer", 31, {}), ("empty", 12, {}),
             ("mutated", 2, {}), ("mutated", 33, {}), ("mutated", 13, {"suffix_len": 10}),
             ("palindromes", 12, {"mode": 2}), ("both_orientations", 15, {"mode": 2}),
             ("mutated", 20, {"wide": True})]


@pytest.mark.parametrize("shape,k,kw", EMU_CASES, ids=["%s-k%d%s" % (s, k, "".join("-" + x for x in kw))
                                                       for s, k, kw in EMU_CASES])
def test_emu_tables(shape, k, kw, monkeypatch):
    boss, valid, idx = emu_case(shape, k, monkeypatch=monkeypatch, **kw)
    info = IT.index_info(idx)
    T = IT.read_tables(idx)
    assert info.kh_slots == 0 and info.pl_n == 0
    ref = IT.reference_for(boss, valid=valid, sfx_len=info.sfx_len)
    if kw.get("suffix_len"):
        assert info.sfx_len == kw["suffix_len"]
    IT.check_index(ref, T, info, hashed=False, primary=kw.get("mode") == 2)
    if shape == "mutated" and k == 12:
        IT.assert_corruptions_rejected(ref, T, info, np.random.default_rng(3), expect_hash=False)
    if kw.get("mode") == 2:
        names = [c[0] for c in IT.corruptions(ref, T, info, np.random.default_rng(4))]
        assert ("palin bit" in names) == (k % 2 == 0)
        assert "rcs zeroed" in names or k % 2       # planted palindromes: nodes whose reverse complement is a node
        IT.assert_corruptions_rejected(ref, T, info, np.random.default_rng(4), expect_hash=False)
    idx.close()


def test_emu_tables_protein():
    rng = np.random.default_rng(77)
    for k, s in ((2, 0), (6, 5), (12, 0)):
        boss, valid, idx = IT.build_index(IT.EMU_LIB, k, IT.protein_seqs(rng, 20, 200), suffix_len=s, alphabet=1)
        info = IT.index_info(idx)
        assert info.wide and info.sigma == 27
        ref = IT.reference_for(boss, sfx_len=info.sfx_len)
        IT.check_index(ref, IT.read_tables(idx), info, hashed=False)
        idx.close()
    boss = BOSSTable.from_dbg(IT.os.path.join(EX, "test_Protein_graph.dbg"), lib=IT.EMU_LIB)
    boss, valid, idx = IT.build_index(IT.EMU_LIB, boss.k, None, boss=boss, mask=True)
    info = IT.index_info(idx)
    IT.check_index(IT.reference_for(boss, valid=valid, sfx_len=info.sfx_len), IT.read_tables(idx), info, hashed=False)
    idx.close()
