"""Aligning files with several workers, on the host emulation: the stage / align split of the file route against the
one-shot call, the ordered multi-worker driver of `metagraph_b200 align --devices` against one worker and the oracle,
the --devices usage errors, and index replicas against their source."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import fastx_common as F
from metagraph_b200 import _lib, cli
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from test_cli_align import EX, GRAPHS, oracle_text

TIMERS = ("seed_kernel_ms", "align_kernel_ms", "h2d_ms", "d2h_ms")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.fixture(scope="module")
def dna():
    t = BOSSTable.from_dbg(os.path.join(EX, GRAPHS[0][0]), lib=F.EMU)
    idx = DBGSuccinctIndex(t, lib=F.EMU)
    yield B200Aligner(idx, cli_defaults(t.k))
    idx.close()


def split(al, data, at_eof, delim, fwd_rev, json):
    batch, consumed, ended = al.stage_fastx(data, at_eof, delim, fwd_rev)
    return al.align_staged_text(batch, json), consumed, ended


def counters(stats):
    return {k: v for k, v in stats.items() if k not in TIMERS}


def split_case(al, data, at_eof, delim, fwd_rev, json):
    one = al.align_fastx_text(data, at_eof, delim, fwd_rev, json)
    one_stats = counters(al.last_stats)
    assert split(al, data, at_eof, delim, fwd_rev, json) == one, (data, at_eof, delim, fwd_rev)
    assert counters(al.last_stats) == one_stats


@pytest.mark.parametrize("json", [False, True])
@pytest.mark.parametrize("i", range(len(F.KNOWN)))
def test_stage_align_known(dna, i, json):
    (data, at_eof, delim, fwd_rev), _ = F.KNOWN[i]
    split_case(dna, data, at_eof, delim, fwd_rev, json)


@pytest.mark.parametrize("json", [False, True])
def test_stage_align_corpus(dna, json):
    """the seeded corpus: FASTA of many lines, 4-line and multi-line FASTQ, CRLF, empty lines, truncated and malformed
    records, each as a last chunk and as a chunk with more to come, with and without a delimiter and the reverse
    complements"""
    for t in F.corpus(n=400):
        for at_eof in (True, False):
            for delim, fwd_rev in ((None, False), ("|", True)):
                split_case(dna, t, at_eof, delim, fwd_rev, json)


def test_stage_align_files(dna):
    """whole query files, one of them with every record made multi-line FASTQ, which the device route refuses"""
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    fq = b"".join(b"@%s c\n%s\n+\n%s\n" % (h, r, b"I" * len(r)) for h, r in zip(names, reads))
    for data in (open(os.path.join(EX, GRAPHS[0][1]), "rb").read(), fq, fq.replace(b"\n+\n", b"\n+\n\n")):
        for json in (False, True):
            split_case(dna, data, True, "|", False, json)
            split_case(dna, data, True, None, True, json)


def test_staged_buffer_reusable(dna):
    data = open(os.path.join(EX, GRAPHS[0][1]), "rb").read()
    exp = dna.align_fastx_text(data)
    for text in (data, data.replace(b"\n", b"\n\n")):        # the device route, and a chunk it refuses
        buf = np.frombuffer(text, np.uint8).copy()
        batch, consumed, ended = dna.stage_fastx(buf, True)
        buf[:] = ord("N")
        assert (dna.align_staged_text(batch), consumed, ended) == (exp[0], len(text), False)


def _rss():
    return int(open("/proc/self/statm").read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


def test_staged_batch_freed_unaligned(dna):
    """200 staged batches of a 1 MB chunk, freed unaligned: the parsed arrays (2 MB each) do not stay behind"""
    rng = np.random.default_rng(3)
    recs = [b">r%d\n%s\n" % (i, bytes(rng.choice(list(b"ACGT"), 200).tolist())) for i in range(5000)]
    data = b"".join(recs)
    dna.free_staged(dna.stage_fastx(data, True)[0])
    before = _rss()
    for _ in range(200):
        batch, consumed, _ = dna.stage_fastx(data, True)
        assert consumed == len(data)
        dna.free_staged(batch)
    assert _rss() - before < 64 << 20
    dna.free_staged(None)


def test_batch_of_another_index(dna):
    other = dna.graph.replicate(0)
    try:
        al = B200Aligner(other, dna.config)
        batch, _, _ = dna.stage_fastx(b">r\nACGT\n", True)
        with pytest.raises(_lib.MgbError) as e:
            al.align_staged_text(batch)
        assert e.value.code == -1
    finally:
        other.close()


# ---- the command ------------------------------------------------------------------------------------------------


def run_main(monkeypatch, tmp_path, argv, chunk_bytes):
    monkeypatch.setenv("MGB_LIB", F.EMU)
    monkeypatch.setattr(cli, "CHUNK_BYTES", chunk_bytes)
    out = str(tmp_path / "out.txt")
    assert cli.main(["align", "-o", out] + argv) == 0
    return open(out, "rb").read()


def _inputs(tmp_path, query):
    """the query file with a record of more than 8 chunks in front, plain and gzip"""
    names, reads = F.read_fasta(os.path.join(EX, query))
    long = (reads[0] * 40)[:4000]
    plain = str(tmp_path / ("long_" + query))
    with open(plain, "wb") as f:
        f.write(b">long\n" + b"".join(long[i:i + 70] + b"\n" for i in range(0, len(long), 70)))
        f.write(open(os.path.join(EX, query), "rb").read())
    gz = plain + ".gz"
    with gzip.open(gz, "wb") as f:
        f.write(open(plain, "rb").read())
    return plain, gz


@pytest.mark.parametrize("g", range(len(GRAPHS)))
def test_workers_match_one_worker(g, tmp_path, monkeypatch):
    dbg, query, alphabet = GRAPHS[g]
    graph = os.path.join(EX, dbg)
    plain, gz = _inputs(tmp_path, query)
    # the query file alone: the oracle's lines
    exp = oracle_text(dbg, query, alphabet)
    assert run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", "0,0,0", os.path.join(EX, query)], 300) == exp
    for path in (plain, gz):
        for fmt in ([], ["--json"]):
            one = run_main(monkeypatch, tmp_path, ["-i", graph] + fmt + [path], 300)
            assert one.count(b"\n") >= 3 and one.endswith(exp if not fmt else b"\n")
            for devices, chunk in (("0,0,0", 300), ("0,0", 97), ("all", 300), ("0,0,0", 1 << 20)):
                got = run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", devices] + fmt + [path], chunk)
                assert got == one, (path, fmt, devices, chunk)


def test_workers_early_end(tmp_path, monkeypatch):
    """a file that ends at a malformed record: the same text, and no chunk is read after the one that ended it"""
    reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))[1]
    good = b"".join(b"@g%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))
    bad = str(tmp_path / "bad.fq")
    open(bad, "wb").write(good * 4 + b"@r2\nACGT\n+\nII\n" + good * 200)
    graph = os.path.join(EX, GRAPHS[0][0])
    one = run_main(monkeypatch, tmp_path, ["-i", graph, bad], 256)
    assert one.count(b"\n") == 4 * len(reads)
    reads_at = []
    orig = cli._Chunks.next
    monkeypatch.setattr(cli._Chunks, "next", lambda self: reads_at.append(1) or orig(self))
    got = run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", "0,0,0,0", bad], 256)
    assert got == one
    assert len(reads_at) * 256 < len(good) * 6


@pytest.mark.parametrize("spec", ["1", "0,1", "-1", "x", "", "0,,0", "0;0"])
def test_devices_usage_error(spec, tmp_path, monkeypatch, capsys):
    """a bad --devices value is a usage error (exit 1) before the graph or any input is opened"""
    monkeypatch.setenv("MGB_LIB", F.EMU)
    opened = []
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, *a, **kw: opened.append(a)))
    assert cli.main(["align", "-i", os.path.join(EX, GRAPHS[0][0]), "--devices", spec,
                     os.path.join(EX, GRAPHS[0][1])]) == 1
    assert "--devices" in capsys.readouterr().err and not opened


def test_worker_error_stops_the_command(tmp_path, monkeypatch, capsys):
    """an error in one worker: `error: ...`, exit 1, nothing after the last text in order, every batch freed"""
    graph = os.path.join(EX, GRAPHS[0][0])
    plain, _ = _inputs(tmp_path, GRAPHS[0][1])
    one = run_main(monkeypatch, tmp_path, ["-i", graph, plain], 300)
    staged, freed = [], []
    orig_stage, orig_align, orig_free = B200Aligner.stage_fastx, B200Aligner.align_staged_text, B200Aligner.free_staged

    def stage(self, *a, **kw):
        r = orig_stage(self, *a, **kw)
        staged.append(r[0].value)
        return r

    def align(self, batch, json=False):
        freed.append(batch.value)
        if len(freed) == 3:
            orig_free(self, batch)
            raise RuntimeError("worker failed")
        return orig_align(self, batch, json)

    def free(self, batch):
        freed.append(batch.value)
        orig_free(self, batch)

    monkeypatch.setattr(B200Aligner, "stage_fastx", stage)
    monkeypatch.setattr(B200Aligner, "align_staged_text", align)
    monkeypatch.setattr(B200Aligner, "free_staged", free)
    monkeypatch.setattr(cli, "CHUNK_BYTES", 300)
    out = str(tmp_path / "err.txt")
    capsys.readouterr()
    assert cli.main(["align", "-i", graph, "--devices", "0,0,0", "-o", out, plain]) == 1
    assert "error: worker failed" in capsys.readouterr().err
    got = open(out, "rb").read()
    assert one.startswith(got) and len(got) < len(one)
    assert sorted(staged) == sorted(freed)


# ---- replicas ---------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("g,mode", [(0, 0), (0, 1), (0, 2), (1, 0)])
def test_replica_text(g, mode):
    dbg, query, _ = GRAPHS[g]
    t = BOSSTable.from_dbg(os.path.join(EX, dbg), lib=F.EMU)
    data = open(os.path.join(EX, query), "rb").read()
    src = DBGSuccinctIndex(t, lib=F.EMU, mode=mode)
    rep = src.replicate(0)
    try:
        cfg = cli_defaults(t.k, "dna" if g == 0 else "protein")
        exp = [B200Aligner(src, cfg).align_fastx_text(data, json=j)[0] for j in (False, True)]
        assert exp[0].count(b"\n") >= 2
        assert [B200Aligner(rep, cfg).align_fastx_text(data, json=j)[0] for j in (False, True)] == exp
        src.close()
        assert [B200Aligner(rep, cfg).align_fastx_text(data, json=j)[0] for j in (False, True)] == exp
        assert rep.replicate(0).replicate(0).num_edges == t.num_edges
    finally:
        src.close()
        rep.close()


def test_replica_bad_arguments(dna):
    for d in (-1, 1):
        with pytest.raises(_lib.MgbError) as e:
            dna.graph.replicate(d)
        assert e.value.code == -1
