"""BGZF input on the device: k_bgzf_inflate against zlib on the corpus and on a FASTQ of over 200 MB (3 000+ blocks) in
every strategy, the command on C2- and C3-shaped BGZF files against the same files plain, and blocks whose trailer
alone is wrong handed over as the gzip route handles them. (Payload mutations run on the emulation build only,
tests/test_bgzf_emu.py.)"""
import os
import zlib

import numpy as np
import pytest

import bench
import bgzf_common as B
import fastx_common as F
from metagraph_b200 import bgzf, cli
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex, bgzf_inflate
from test_multi_device_gpu import N_DEV, shaped_reads, small_graph  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def index():
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(11, ["ACGTACGTTGCAGGCATTACG"]), device=0)
    yield idx
    idx.close()


def served(index, data, text):
    got, c_consumed, n, refused = bgzf_inflate(index, data)
    assert (c_consumed, n, refused) == (len(data), B.n_blocks(data), False)
    assert got == text


def test_inflate_corpus(index):
    text = b"".join(F.corpus(n=2000))
    for strategy in B.STRATEGIES:
        for level in (0, 1, 6, 9):
            for flush in (None, zlib.Z_FULL_FLUSH):
                for block_text in (777, 65280 if level == 0 else 65536):
                    served(index, B.write(text, block_text, level, strategy, flush), text)
    for gen in (B.random_bytes, B.long_runs, B.far_repeats):
        t = gen(9, 2_000_000)
        served(index, B.write(t, 65280, 6), t)


@pytest.fixture(scope="module")
def big_fastq():
    text = B.fastq(np.random.default_rng(5), 640_000)
    assert len(text) >= 200_000_000
    return text


@pytest.mark.parametrize("level,strategy", [(6, s) for s in B.STRATEGIES] + [(1, "default"), (9, "default")])
def test_inflate_big(index, big_fastq, level, strategy):
    data = B.write(big_fastq, 65280, level, strategy)
    assert B.n_blocks(data) >= 3000
    served(index, data, big_fastq)


def _write_shapes(genome, tmp_path, n):
    files = {}
    for shape, (buf, _) in shaped_reads(genome, n).items():
        reads = buf.reshape(n, bench.READ_LEN)
        data = B.fastq_of(reads)
        plain = str(tmp_path / (shape + ".fq"))
        open(plain, "wb").write(data)
        open(plain + ".bgz", "wb").write(B.write(data, 65280, 6))
        files[shape] = (plain, plain + ".bgz", data)
    return files


def test_command_bgzf(small_graph, tmp_path, monkeypatch):  # noqa: F811
    genome, boss = small_graph
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, path, lib=None: boss))
    n = 200_000
    lists = ["0", "0,0", "0,0,0,0"] + (["0,1"] if N_DEV >= 2 else [])
    for shape, (plain, bgz, data) in _write_shapes(genome, tmp_path, n).items():
        monkeypatch.setattr(cli, "CHUNK_BYTES", len(data) // 24)
        argv = ["-i", "graph.dbg"] + (["--align-min-seed-length", "31", "--align-max-seed-length", "31"]
                                      if shape == "c2" else ["--align-min-exact-match", "0"])
        for fmt in ([], ["--json"]):
            out = str(tmp_path / "plain.txt")
            assert cli.main(["align"] + argv + fmt + ["-o", out, plain]) == 0
            exp = open(out, "rb").read()
            assert exp.count(b"\n") >= n
            for devices in lists:
                out = str(tmp_path / ("out_%s.txt" % devices.replace(",", "_")))
                assert cli.main(["align"] + argv + fmt + ["--devices", devices, "-o", out, bgz]) == 0
                assert open(out, "rb").read() == exp, (shape, fmt, devices)


@pytest.mark.parametrize("field", ["crc", "isize"])
def test_trailer_refused(index, small_graph, tmp_path, monkeypatch, capsys, field):  # noqa: F811
    """a valid payload under a wrong CRC32 or ISIZE: the block is refused, the rest of the file is handed over, and the
    command exits as the gzip route does"""
    genome, boss = small_graph
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, path, lib=None: boss))
    buf, _ = shaped_reads(genome, 20_000)["c2"]
    data = B.fastq_of(buf.reshape(20_000, bench.READ_LEN))
    good = B.write(data, 65280, 6, eof=False)
    at = bgzf.block(good)[0]
    size = bgzf.block(good, at)[0]
    blk = bytearray(good[at:at + size])
    blk[-8 if field == "crc" else -4] ^= 1
    bad = good[:at] + bytes(blk) + good[at + size:]
    assert bgzf_inflate(index, bad)[1:] == (at, 1, True)
    path = str(tmp_path / "bad.fq.gz")
    open(path, "wb").write(bad)
    for devices in ("0", "0,0"):
        monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, path, lib=None: boss))
        monkeypatch.setattr(cli, "CHUNK_BYTES", len(data) // 8)
        argv = ["-i", "graph.dbg", "--devices", devices]
        got = B.run(cli, argv, path, tmp_path, capsys)
        exp = B.gzip_route(monkeypatch, cli, argv, path, tmp_path, capsys)
        assert got[0] == exp[0] == 1 and "error: " in got[2], (got[2], exp[2])
