"""Plain gzip input on the device: the speculative inflater against zlib on the corpus and on a FASTQ of over 100 MB at
levels 1, 6 and 9 in every strategy the finder serves, the share of found candidates the chain confirms, and the
command on C2- and C3-shaped gzip files, one member over many stages, against the same files plain with one worker and
several. (Mutations and refusals run on the emulation build, tests/test_gzip_emu.py.)"""
import zlib

import numpy as np
import pytest

import bench
import bgzf_common as B
import fastx_common as F
from metagraph_b200 import cli
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex, gzip_inflate
from test_multi_device_gpu import N_DEV, shaped_reads, small_graph  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def index():
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(11, ["ACGTACGTTGCAGGCATTACG"]), device=0)
    yield idx
    idx.close()


def gz(text, level=6, strategy="default", flush=None):
    return b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + B.deflate(text, level, strategy, flush) + \
        (zlib.crc32(text)).to_bytes(4, "little") + (len(text) & 0xffffffff).to_bytes(4, "little")


def served(index, data, text, sub_bytes=0):
    got, c_used, refused, counts = gzip_inflate(index, data, sub_bytes=sub_bytes)
    assert (c_used, refused) == (len(data), False)
    assert got == text
    return counts


def test_inflate_corpus(index):
    text = b"".join(F.corpus(n=2000))
    for strategy in ("default", "filtered", "huffman", "rle"):
        for level in (1, 6, 9):
            for flush in (None, zlib.Z_FULL_FLUSH):
                for sub in (0, 1000):
                    served(index, gz(text, level, strategy, flush), text, sub)
    for gen in (B.random_bytes, B.long_runs, B.far_repeats):
        t = gen(9, 2_000_000)
        served(index, gz(t, 6), t)
        served(index, gz(t, 6), t, 3000)


@pytest.fixture(scope="module")
def big_fastq():
    text = B.fastq(np.random.default_rng(5), 330_000)
    assert len(text) >= 100_000_000
    return text


@pytest.mark.parametrize("level,strategy", [(6, s) for s in ("default", "filtered", "huffman", "rle")]
                         + [(1, "default"), (9, "default")])
def test_inflate_big(index, big_fastq, level, strategy):
    n_sub, found, confirmed = served(index, gz(big_fastq, level, strategy), big_fastq)
    assert n_sub >= 500 and confirmed >= 1
    if (level, strategy) == (6, "default"):
        assert found - confirmed < 0.01 * found, (found, confirmed)


def _write_shapes(genome, tmp_path, n):
    files = {}
    for shape, (buf, _) in shaped_reads(genome, n).items():
        reads = buf.reshape(n, bench.READ_LEN)
        data = B.fastq_of(reads)
        plain = str(tmp_path / (shape + ".fq"))
        open(plain, "wb").write(data)
        open(plain + ".gz", "wb").write(gz(data, 6))
        files[shape] = (plain, plain + ".gz", data)
    return files


def test_command_gzip(small_graph, tmp_path, monkeypatch):  # noqa: F811
    """one member staged in about 24 parts, with one worker and several, TSV and JSON"""
    genome, boss = small_graph
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, path, lib=None: boss))
    n = 200_000
    lists = ["0", "0,0", "0,0,0,0"] + (["0,1"] if N_DEV >= 2 else [])
    stages, handed = [], []
    orig = cli._Token._stage_gzip

    def stage(self, *a):
        stages.append(1)
        return orig(self, *a)

    monkeypatch.setattr(cli._Token, "_stage_gzip", stage)
    monkeypatch.setattr(cli._Token, "_hand_over", lambda self, *a: handed.append(1))
    for shape, (plain, gzp, data) in _write_shapes(genome, tmp_path, n).items():
        monkeypatch.setattr(cli, "CHUNK_BYTES", len(data) // 24)
        argv = ["-i", "graph.dbg"] + (["--align-min-seed-length", "31", "--align-max-seed-length", "31"]
                                      if shape == "c2" else ["--align-min-exact-match", "0"])
        for fmt in ([], ["--json"]):
            out = str(tmp_path / "plain.txt")
            assert cli.main(["align"] + argv + fmt + ["-o", out, plain]) == 0
            exp = open(out, "rb").read()
            assert exp.count(b"\n") >= n
            for devices in lists:
                stages.clear()
                handed.clear()
                out = str(tmp_path / ("out_%s.txt" % devices.replace(",", "_")))
                assert cli.main(["align"] + argv + fmt + ["--devices", devices, "-o", out, gzp]) == 0
                assert open(out, "rb").read() == exp, (shape, fmt, devices)
                assert len(stages) >= 10 and not handed
