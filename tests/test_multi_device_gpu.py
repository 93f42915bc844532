"""Index replicas and the multi-worker file driver on the device.

- mgb_index_replicate on the source's own device (and on device 1 when there is one): every table the test library
  reads equals the source's, array for array, and passes the table checks of test_index_tables_gpu, for a hashed
  graph, a PRIMARY graph after mgb_index_set_mode, the alphabet-generic layout and a graph of over 4 M edges.
- The knobs mgb_index_create honours, set while the replica is made: the replica holds what mgb_index_create builds
  under the same knob (so no test depends on how much memory other work leaves free).
- A replica aligns C2- and C3-shaped batches (bench.py's generators) to the same text as its source.
- `metagraph_b200 align --devices 0,0` and `0,0,0,0` on one GPU (and `0,1` on two): the same bytes as `--devices 0`
  for C2- and C3-shaped FASTQ files of 200 k reads in 20 or more chunks, TSV and JSON, plain and gzip."""
import gzip
import os

import numpy as np
import pytest

import bench
import index_tables as IT
import parity_common as P
from metagraph_b200 import _lib, cli
from metagraph_b200.aligner import B200Aligner, BOSSTable
from metagraph_b200.config import cli_defaults
from test_index_tables_gpu import check_device
from test_layout_words_gpu import LAYOUT_LIB, layout_tables

pytestmark = pytest.mark.gpu

try:
    N_DEV = _lib.load_library().mgb_device_count()
except ImportError:          # (collected without the built library: every test here is skipped without a GPU anyway)
    N_DEV = 0
TARGETS = [0, pytest.param(1, marks=pytest.mark.skipif(N_DEV < 2, reason="one visible device: no peer to copy to"))]
INFO = ("n", "kh_slots", "pl_n", "k", "sigma", "wide", "mode", "sfx_len")


def same_tables(a, b, names=None):
    ia, ib = IT.index_info(a), IT.index_info(b)
    assert [getattr(ia, f) for f in INFO] == [getattr(ib, f) for f in INFO]
    A, B = IT.read_tables(a, names), IT.read_tables(b, names)
    for name in A:
        assert (A[name] is None) == (B[name] is None), name
        if A[name] is not None:
            assert np.array_equal(A[name], B[name]), name


GRAPHS = [("mutated", 31, {}), ("palindromes", 12, {"mode": 2}), ("mutated", 20, {"wide": True})]


@pytest.mark.parametrize("device", TARGETS)
@pytest.mark.parametrize("shape,k,kw", GRAPHS, ids=["%s-k%d" % (s, k) + "".join("-%s" % a for a in kw)
                                                    for s, k, kw in GRAPHS])
def test_replica_tables(shape, k, kw, device, monkeypatch):
    rng = np.random.default_rng(7000 + k)
    seqs = IT.shape_seqs(shape, k, rng, 20000)
    mode = kw.get("mode", 0)
    if mode == 2:
        seqs = P.primary_contigs(seqs, k)
    if kw.get("wide"):
        monkeypatch.setenv("MGB_TEST_WIDE", "1")
    boss, valid, src = IT.build_index(IT.TABLES_LIB, k, seqs, mask=mode == 0, mode=mode)
    rep = src.replicate(device)
    try:
        same_tables(src, rep)
        src.close()                                  # the replica does not depend on its source
        hashed = not kw.get("wide")
        check_device(boss, valid, rep, hashed, primary=mode == 2, emu_compare=False, wide=kw.get("wide", False))
    finally:
        src.close()
        rep.close()


@pytest.mark.parametrize("device", TARGETS)
def test_replica_tables_4m_edges(device):
    rng = np.random.default_rng(4242)
    base = IT.random_seq(rng, 4_000_000)
    boss, valid, src = IT.build_index(IT.TABLES_LIB, 31, [base, IT.mutate(rng, base, 0.01)])
    assert boss.num_edges >= 4_000_000
    rep = src.replicate(device)
    try:
        same_tables(src, rep)
        check_device(boss, valid, rep, hashed=True, emu_compare=False)
    finally:
        src.close()
        rep.close()


KNOBS = [("MGB_NO_KMER_HASH", "1"), ("MGB_NO_PATH_INDEX", "1"), ("MGB_TEST_NO_LAYOUT_WORDS", "kh_pos"),
         ("MGB_TEST_NO_LAYOUT_WORDS", "pl_word"), ("MGB_TEST_NO_LAYOUT_WORDS", "both")]


@pytest.mark.parametrize("device", TARGETS)
@pytest.mark.parametrize("knob,value", KNOBS, ids=["%s=%s" % kv for kv in KNOBS])
def test_replica_knobs(knob, value, device, monkeypatch):
    """a replica made under a knob holds the tables mgb_index_create builds under it, with its source's contents (the
    hash index's slot order differs from build to build): without the hash index the adjacency records' bits 16..20
    are 0 again, and the path layout and its leaner copies go too"""
    rng = np.random.default_rng(11)
    seqs = IT.shape_seqs("mutated", 31, rng, 30000)
    lib = LAYOUT_LIB if knob == "MGB_TEST_NO_LAYOUT_WORDS" else IT.TABLES_LIB
    boss, valid, src = IT.build_index(lib, 31, seqs)
    monkeypatch.setenv(knob, value)
    rep = src.replicate(device)
    _, _, fresh = IT.build_index(lib, 31, None, boss=boss)
    monkeypatch.delenv(knob)
    try:
        if lib == LAYOUT_LIB:
            (info_r, R), (info_f, Fr), (_, S) = layout_tables(rep), layout_tables(fresh), layout_tables(src)
            assert info_r == info_f
            assert S["kh_pos"] is not None and S["pl_word"] is not None, IT.free_device_memory()
            assert (R["kh_pos"] is None) == (value != "pl_word") and (R["pl_word"] is None) == (value != "kh_pos")
        else:
            assert IT.index_info(src).pl_n, IT.free_device_memory()
            ir, i_f = IT.index_info(rep), IT.index_info(fresh)
            assert [getattr(ir, f) for f in INFO] == [getattr(i_f, f) for f in INFO]
            assert ir.pl_n == 0
            R, Fr, S = IT.read_tables(rep), IT.read_tables(fresh), IT.read_tables(src)
            if knob == "MGB_NO_KMER_HASH":
                assert ir.kh_slots == 0 and not (R["adj"][:, 1] >> 16).any() and (S["adj"][:, 1] >> 16).any()
                S["adj"] = Fr["adj"]
        for name in R:
            assert (R[name] is None) == (Fr[name] is None), name
            if R[name] is not None:
                assert np.array_equal(R[name], S[name]), name
    finally:
        for x in (src, rep, fresh):
            x.close()


def shaped_reads(genome, n):
    """C2: error-free reads, exact seeder; C3: 5 % errors, CLI-default seeder with --align-min-exact-match 0"""
    c2 = bench.make_reads(genome, n, 42)[0]
    c3 = bench.make_error_reads(genome, 0, 1, chunk=n)[0]
    return {"c2": (c2, cli_defaults(31, min_seed_length=31, max_seed_length=31)),
            "c3": (c3, cli_defaults(31, min_exact_match=0.0))}


@pytest.fixture(scope="module")
def small_graph():
    genome = bench.make_genome(2_000_000)
    return genome, BOSSTable.from_sequences(31, [genome.tobytes().decode()])


@pytest.mark.parametrize("device", TARGETS)
def test_replica_alignments(device, small_graph):
    from metagraph_b200.aligner import DBGSuccinctIndex
    genome, boss = small_graph
    src = DBGSuccinctIndex(boss, device=0)
    rep = src.replicate(device)
    try:
        n, L = 20000, bench.READ_LEN
        for shape, (buf, cfg) in shaped_reads(genome, n).items():
            batch = [(b"r%d" % i, buf[i * L:(i + 1) * L].tobytes()) for i in range(n)]
            for json in (False, True):
                exp = B200Aligner(src, cfg).align_batch_text(batch, json)
                assert exp.count(b"\n") >= n
                assert B200Aligner(rep, cfg).align_batch_text(batch, json) == exp, (shape, json)
    finally:
        src.close()
        rep.close()


def test_command_workers(small_graph, tmp_path, monkeypatch):
    genome, boss = small_graph
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, path, lib=None: boss))
    n, L = 200_000, bench.READ_LEN
    lists = ["0,0", "0,0,0,0"] + (["0,1"] if N_DEV >= 2 else [])
    for shape, (buf, _) in shaped_reads(genome, n).items():
        reads = buf.reshape(n, L)
        data = b"".join(b"@r%d\n%s\n+\n%s\n" % (i, reads[i].tobytes(), b"F" * L) for i in range(n))
        plain = str(tmp_path / (shape + ".fq"))
        open(plain, "wb").write(data)
        with gzip.open(plain + ".gz", "wb", compresslevel=1) as f:
            f.write(data)
        monkeypatch.setattr(cli, "CHUNK_BYTES", len(data) // 24)
        argv = ["-i", "graph.dbg"] + (["--align-min-seed-length", "31", "--align-max-seed-length", "31"]
                                      if shape == "c2" else ["--align-min-exact-match", "0"])
        for path in (plain, plain + ".gz"):
            for fmt in ([], ["--json"]):
                outs = {}
                for devices in ["0"] + lists:
                    out = str(tmp_path / ("out_%s.txt" % devices.replace(",", "_")))
                    assert cli.main(["align"] + argv + fmt + ["--devices", devices, "-o", out, path]) == 0
                    outs[devices] = open(out, "rb").read()
                assert outs["0"].count(b"\n") >= n
                for devices in lists:
                    assert outs[devices] == outs["0"], (shape, path, fmt, devices)
