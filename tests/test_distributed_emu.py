"""`metagraph_b200 align --distributed` under torchrun with gloo, on the host emulation: for 2 and 3 ranks, the same
bytes as the single-process command with the same chunk size (plain FASTA and FASTQ, BGZF, plain gzip, gzip files the
device route hands over to Python's gzip mid-file, --json / --fwd-and-reverse / --header-comment-delim, two files with
-o, a record longer than a chunk, a file that ends at a malformed record); the first error on one rank stops every
rank; the usage errors; gzip stream export and import; and sharding.align_sharded_text against align_batch_text and
the oracle."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import bgzf_common as B
import fastx_common as F
from metagraph_b200 import _lib, cli
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, GzipStream
from metagraph_b200.config import cli_defaults
from test_cli_align import EX, GRAPHS
from test_gzip_emu import member, stage_all

CHUNK = 512

# the command with cli.CHUNK_BYTES set, a note on stderr at every hand-over to Python's gzip, and optionally a failure
# injected into one rank's align_staged_text (MGB_TEST_FAIL="rank:call")
WORKER = r'''
import os, sys
sys.path.insert(0, ROOT)
from metagraph_b200 import cli
from metagraph_b200.aligner import B200Aligner
cli.CHUNK_BYTES = int(os.environ["MGB_TEST_CHUNK"])
hand_over = cli._Token._hand_over
def noted(self, *a):
    sys.stderr.write("HANDED_OVER\n")
    return hand_over(self, *a)
cli._Token._hand_over = noted
if os.environ.get("MGB_TEST_FAIL"):
    rank, call = (int(x) for x in os.environ["MGB_TEST_FAIL"].split(":"))
    if int(os.environ.get("RANK", "0")) == rank:
        align, calls = B200Aligner.align_staged_text, []
        def failing(self, batch, json=False):
            calls.append(1)
            if len(calls) == call:
                self.free_staged(batch)
                raise RuntimeError("injected failure")
            return align(self, batch, json)
        B200Aligner.align_staged_text = failing
sys.exit(cli.main(sys.argv[1:]))
'''


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.fixture(scope="module")
def worker(tmp_path_factory):
    p = tmp_path_factory.mktemp("worker") / "worker.py"
    p.write_text("ROOT = %r\n" % F.ROOT + WORKER)
    return str(p)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _env(chunk, fail=None):
    env = dict(os.environ, MGB_LIB=F.EMU, MGB_TEST_CHUNK=str(chunk), MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    env.pop("MGB_TEST_FAIL", None)
    if fail:
        env["MGB_TEST_FAIL"] = fail
    return env


def single(worker, argv, chunk=CHUNK):
    """(exit code, stdout, stderr) of the single-process command"""
    r = subprocess.run([sys.executable, worker, "align"] + argv, capture_output=True, env=_env(chunk), timeout=600)
    return r.returncode, r.stdout, r.stderr.decode()


def torchrun(worker, n, argv, chunk=CHUNK, fail=None, timeout=600):
    """(exit code, stdout, stderr) of `align --distributed` on n gloo ranks"""
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % n,
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), worker, "align",
                        "--distributed"] + argv, capture_output=True, env=_env(chunk, fail), timeout=timeout)
    return r.returncode, r.stdout, r.stderr.decode()


def _fastq(n_copies=40):
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    rng = np.random.default_rng(9)
    out = []
    for i in range(n_copies):
        for h, r in zip(names, reads):
            r = bytes(rng.permutation(np.frombuffer(r, np.uint8))) if i % 5 == 4 else r
            out.append(b"@%s_%d c%d\n%s\n+\n%s\n" % (h, i, i, r, b"F" * len(r)))
    return b"".join(out)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """name -> path: plain FASTA with a record of more than 8 chunks in front, FASTQ, BGZF, two-member gzip, and gzip
    whose device route hands over to Python's gzip mid-file (a large stored member after a dynamic one)"""
    d = tmp_path_factory.mktemp("inputs")
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    long = (reads[0] * 200)[:5000]
    fa = b">long\n" + b"".join(long[i:i + 70] + b"\n" for i in range(0, len(long), 70))
    fa += b"".join(b">%s_%d\n%s\n" % (h, i, r) for i in range(30) for h, r in zip(names, reads))
    fq = _fastq()
    half = len(fq) // 2
    big = _fastq(1200)
    assert len(big) > 3 * 32768
    data = {"long.fa": fa, "reads.fq": fq, "reads.fq.bgz": B.write(fq, 1000),
            "reads.fq.gz": member(fq[:half], 6, flg=8, name=b"r.fq") + member(fq[half:], 9),
            "stored.fq.gz": member(fq, 6) + member(big, 0),
            "bad_crc.fq.gz": member(fq, 6)[:-8] + bytes([member(fq, 6)[-8] ^ 1]) + member(fq, 6)[-7:]}
    out = {}
    for name, b in data.items():
        out[name] = str(d / name)
        open(out[name], "wb").write(b)
    assert cli.route_of(out["reads.fq.bgz"]) == "bgzf" and cli.route_of(out["reads.fq.gz"]) == "gzip"
    return out


GRAPH = os.path.join(EX, GRAPHS[0][0])
ORDER = ["long.fa", "reads.fq", "reads.fq.bgz", "reads.fq.gz", "stored.fq.gz"]


@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("fmt", [[], ["--json", "--fwd-and-reverse", "--header-comment-delim", "|"]],
                         ids=["tsv", "json-fwdrev-delim"])
def test_matches_single_process(worker, files, n, fmt):
    argv = ["-i", GRAPH] + fmt + [files[k] for k in ORDER]
    rc, exp, err = single(worker, argv)
    assert rc == 0, err
    assert exp.count(b"\n") > 500 and "HANDED_OVER" in err
    rc, got, err = torchrun(worker, n, argv)
    assert rc == 0, err[-3000:]
    assert "HANDED_OVER" in err
    assert got == exp


@pytest.mark.parametrize("n", [2, 3])
def test_bad_crc(worker, files, n):
    """the gzip route hands the member over, Python's gzip fails at its end: exit 1 and gzip's error on stderr"""
    argv = ["-i", GRAPH, files["bad_crc.fq.gz"]]
    rc, exp, exp_err = single(worker, argv)
    assert rc == 1 and "error: " in exp_err
    rc, got, err = torchrun(worker, n, argv)
    assert rc == 1
    line = [x for x in exp_err.splitlines() if x.startswith("error: ")]
    assert line and line[0] in err.splitlines()
    rc, good, _ = single(worker, ["-i", GRAPH, files["reads.fq"]])
    assert rc == 0 and good.startswith(exp) and good.startswith(got)


def test_two_files_outfile(worker, files, tmp_path):
    """-o is reopened for every input: it ends up with the last file's text"""
    out1, out2 = str(tmp_path / "one.txt"), str(tmp_path / "dist.txt")
    assert single(worker, ["-i", GRAPH, "-o", out1, files["reads.fq.gz"], files["long.fa"]])[0] == 0
    rc, stdout, err = torchrun(worker, 2, ["-i", GRAPH, "-o", out2, files["reads.fq.gz"], files["long.fa"]])
    assert rc == 0, err[-3000:]
    assert stdout == b"" and open(out2, "rb").read() == open(out1, "rb").read()
    assert open(out1, "rb").read().startswith(b"long\t")


def test_malformed_end(worker, tmp_path):
    """a file that ends at a malformed record: the text of the records before it"""
    reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))[1]
    good = b"".join(b"@g%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))
    bad = str(tmp_path / "bad.fq")
    open(bad, "wb").write(good * 40 + b"@r2\nACGT\n+\nII\n" + good * 200)
    rc, exp, _ = single(worker, ["-i", GRAPH, bad], 256)
    assert rc == 0 and exp.count(b"\n") == 40 * len(reads)
    rc, got, err = torchrun(worker, 3, ["-i", GRAPH, bad], 256)
    assert rc == 0, err[-3000:]
    assert got == exp


def _chunk_ends(path, chunk):
    """the output offsets at which the single-process command's chunks end"""
    t = BOSSTable.from_dbg(GRAPH, lib=F.EMU)
    idx = DBGSuccinctIndex(t, lib=F.EMU)
    ends = []

    class Out:
        def write(self, b):
            ends.append((ends[-1] if ends else 0) + len(b))
    try:
        cli.align_file(B200Aligner(idx, cli_defaults(t.k)), path, Out(), chunk_bytes=CHUNK)
    finally:
        idx.close()
    return [0] + ends


@pytest.mark.parametrize("fail", ["1:3", "0:2", "2:1", "2:2"])
def test_injected_failure(worker, files, fail):
    """rank r's k-th align_staged_text fails, which is chunk c = (k-1)*W + r: exit 1, the error on stderr, and the
    output is the single-process output of chunks 0 .. c-1 exactly"""
    argv = ["-i", GRAPH, files["reads.fq"]]
    rc, exp, _ = single(worker, argv)
    assert rc == 0
    rc, got, err = torchrun(worker, 3, argv, fail=fail)
    assert rc == 1
    assert "error: injected failure" in err.splitlines()
    r, k = (int(x) for x in fail.split(":"))
    ends = _chunk_ends(files["reads.fq"], CHUNK)
    c = (k - 1) * 3 + r
    assert c + 1 < len(ends)
    assert got == exp[:ends[c]]


@pytest.mark.parametrize("case", ["bad_outfile", "missing_input", "full_mid_file", "full_at_close"])
def test_output_errors(worker, files, tmp_path, case):
    """an error outside a stage or an align (rank 0 cannot open -o, an input does not exist, rank 0's writes fail in
    the middle of a file or when it closes -o): every rank stops at once with the single-process command's exit code,
    and rank 0 prints its error line"""
    if case.startswith("full") and not os.path.exists("/dev/full"):
        pytest.skip("no /dev/full, the device whose writes fail with ENOSPC")
    argv = {"bad_outfile": ["-o", str(tmp_path / "no" / "such" / "dir.tsv"), files["reads.fq"]],
            "missing_input": ["-o", str(tmp_path / "out.tsv"), files["reads.fq"], str(tmp_path / "missing.fq")],
            "full_mid_file": ["-o", "/dev/full", files["stored.fq.gz"], files["reads.fq"]],
            "full_at_close": ["-o", "/dev/full", files["reads.fq"]]}[case]
    rc, _, exp_err = single(worker, ["-i", GRAPH] + argv)
    assert rc == 1
    line = [x for x in exp_err.splitlines() if x.startswith(("error: ", "ERROR: "))]
    assert line
    rc, _, err = torchrun(worker, 2, ["-i", GRAPH] + argv, timeout=180)
    assert rc == 1 and line[0] in err.splitlines(), err[-3000:]


def test_usage_errors(monkeypatch, capsys):
    monkeypatch.setenv("MGB_LIB", F.EMU)
    opened = []
    monkeypatch.setattr(BOSSTable, "from_dbg", classmethod(lambda cls, *a, **kw: opened.append(a)))
    q = os.path.join(EX, GRAPHS[0][1])
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(v, raising=False)
    assert cli.main(["align", "-i", GRAPH, "--distributed", q]) == 1
    assert "RANK, WORLD_SIZE and LOCAL_RANK" in capsys.readouterr().err
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("WORLD_SIZE", "2")
    assert cli.main(["align", "-i", GRAPH, "--distributed", q]) == 1
    assert "LOCAL_RANK" in capsys.readouterr().err
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.setenv("RANK", "2")
    assert cli.main(["align", "-i", GRAPH, "--distributed", q]) == 1
    assert "bad RANK" in capsys.readouterr().err
    monkeypatch.setenv("RANK", "0")
    for devices in ("0", "all", "0,0"):
        assert cli.main(["align", "-i", GRAPH, "--distributed", "--devices", devices, q]) == 1
        assert "--devices cannot be combined with --distributed" in capsys.readouterr().err
    assert not opened


# ---- gzip stream export and import ----------------------------------------------------------------------------------


def test_gzip_stream_export_import():
    """stage part of a stream, export it, import it into a fresh stream and finish on another index: the same bytes as
    an uninterrupted run, at every point the stream can be cut"""
    t = BOSSTable.from_dbg(GRAPH, lib=F.EMU)
    a, b = DBGSuccinctIndex(t, lib=F.EMU), DBGSuccinctIndex(t, lib=F.EMU)
    try:
        cfg = cli_defaults(t.k)
        al_a, al_b = B200Aligner(a, cfg), B200Aligner(b, cfg)
        fq = B.fastq(np.random.default_rng(6), 3000)          # two members of several 32 KiB sub-ranges each
        third = len(fq) // 3
        data = member(fq[:third], 6) + member(fq[third:], 9, flg=8, name=b"x")
        exp = stage_all(al_a, data, 97, 400)
        assert exp == al_a.align_fastx_text(fq)[0] and exp.count(b"\n") == 3000
        text, n_stages, _ = _stage_cut(al_a, al_b, data, 97, 400, None)
        assert text == exp and n_stages >= 10
        inside = 0
        for cut in range(1, n_stages):
            text, _, state = _stage_cut(al_a, al_b, data, 97, 400, cut)
            assert state is not None and text == exp, cut       # the stream was cut, and finished on al_b
            inside += state[0]
        assert inside >= 2                                       # cuts inside a member, not only between members
    finally:
        a.close()
        b.close()


def _stage_cut(al_a, al_b, data, chunk, max_text, cut):
    """stage_all with the stream exported after `cut` stages and imported on al_b's index for the rest (cut None: not
    cut). Returns (text, stages, the stream's state at the cut or None when no cut was made)"""
    stream = GzipStream(al_a._L)
    al, state = al_a, None
    out, tail, cpend, at, c_eof, want, c_want = [], b"", b"", 0, False, 0, chunk
    try:
        for i in range(10 ** 6):
            if i == cut:
                block = stream.export()
                assert len(block) == stream._L.mgb_gzip_stream_export_bytes(stream.handle) > 32768
                state = stream.state()
                stream.close()
                stream = GzipStream.from_export(al_b._L, block)
                assert stream.state() == state and stream.export() == block
                al = al_b
            mt = max(max_text, want)
            while not c_eof and len(cpend) < c_want:
                nxt = data[at:at + chunk]
                at += len(nxt)
                c_eof = not nxt
                cpend += nxt
            batch, c_used, refused, consumed, ended, tail2 = al.stage_fastx_gzip(stream, tail, cpend, c_eof, mt)
            assert not refused
            out.append(al.align_staged_text(batch))
            cpend = cpend[c_used:]
            if ended or (c_eof and not cpend and not stream.state()[0]):
                return b"".join(out), i + 1, state
            c_want = 2 * max(c_want, len(cpend)) if c_used == 0 else chunk
            want = len(tail2) if consumed == 0 else 0
            tail = tail2
    finally:
        stream.close()


def test_gzip_stream_import_refuses():
    L = _lib.load_library(F.EMU)
    s = GzipStream(L)
    try:
        block = s.export()
    finally:
        s.close()
    assert GzipStream.from_export(L, block).state() == (False, 0)
    for bad in (block[:-1], b"", b"x" * len(block), block[:8] + b"\2" + block[9:], block[:12] + b"\x09" + block[13:]):
        with pytest.raises(_lib.MgbError) as e:
            GzipStream.from_export(L, bad)
        assert e.value.code == -1


# ---- align_sharded_text ---------------------------------------------------------------------------------------------

SHARDED = r'''
import os, sys
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch.distributed as dist
import oracle_lib as O
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from metagraph_b200.sharding import align_sharded_text
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")
dist.init_process_group("gloo")
rank = dist.get_rank()
rng = np.random.default_rng(5)
genome = "".join(np.array(list("ACGT"))[rng.integers(0, 4, 20000)])
comp = str.maketrans("ACGT", "TGCA")
reads = []
for i in range(37):
    p = int(rng.integers(0, len(genome) - 100)); r = genome[p:p + 100]
    reads.append(("r%d" % i, r.translate(comp)[::-1] if i % 3 == 0 else r))
k = 21
idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, [genome], lib=EMU), lib=EMU)
al = B200Aligner(idx, cli_defaults(k))
tsv, js = align_sharded_text(al, reads), align_sharded_text(al, reads, json=True)
few = align_sharded_text(al, reads[:1])                    # one rank's shard is empty
if rank == 0:
    assert tsv == al.align_batch_text(reads) and js == al.align_batch_text(reads, json=True)
    assert few == al.align_batch_text(reads[:1])
    exp = O.OracleGraph(k, [genome]).align_tsv(cli_defaults(k), [s for _, s in reads], headers=[h for h, _ in reads])
    assert tsv.decode().splitlines() == exp, (len(tsv), len(exp))
    assert js.count(b"\n") == len(reads)
    print("SHARDED_TEXT_OK", len(exp))
else:
    assert tsv is None and js is None and few is None
dist.destroy_process_group()
'''


def test_align_sharded_text_gloo(tmp_path):
    script = tmp_path / "sharded.py"
    script.write_text("ROOT = %r\n" % F.ROOT + SHARDED)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), str(script)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "SHARDED_TEXT_OK 37" in r.stdout
