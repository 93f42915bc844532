"""BGZF input on the host emulation: the inflater against zlib for every writer knob, the staged BGZF route against the
plain route's text, the command on BGZF files against the oracle with one worker and several, and files that are BGZF
only in part against the gzip route."""
import gzip
import os
import subprocess
import zlib

import numpy as np
import pytest

import bgzf_common as B
import fastx_common as F
from metagraph_b200 import bgzf, cli
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, bgzf_inflate
from metagraph_b200.config import cli_defaults
from test_cli_align import EX, GRAPHS, oracle_text


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.fixture(scope="module")
def dna():
    t = BOSSTable.from_dbg(os.path.join(EX, GRAPHS[0][0]), lib=F.EMU)
    idx = DBGSuccinctIndex(t, lib=F.EMU)
    yield B200Aligner(idx, cli_defaults(t.k))
    idx.close()


def inflates(index, data, text):
    """every block of data inflated on the device route, to zlib's text"""
    assert zlib.decompress(data, 31) == text or gzip.decompress(data) == text
    got, c_consumed, n, refused = bgzf_inflate(index, data)
    assert (c_consumed, n, refused) == (len(data), B.n_blocks(data), False)
    assert got == text


def test_eof_block(dna):
    assert bgzf_inflate(dna.graph, B.EOF_BLOCK) == (b"", 28, 1, False)
    assert bgzf_inflate(dna.graph, B.EOF_BLOCK * 3) == (b"", 84, 3, False)
    assert bgzf_inflate(dna.graph, b"") == (b"", 0, 0, False)


CORPUS = b"".join(F.corpus(n=300))


@pytest.mark.parametrize("strategy", list(B.STRATEGIES))
def test_inflate_knobs(dna, strategy):
    for level in range(10):
        for flush in (None, zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            for block_text in (1, 777, 65280 if level == 0 else 65536):
                text = CORPUS[:2000] if block_text == 1 else CORPUS
                inflates(dna.graph, B.write(text, block_text, level, strategy, flush), text)


@pytest.mark.parametrize("name", ["random", "runs", "far"])
@pytest.mark.parametrize("strategy", list(B.STRATEGIES))
def test_inflate_inputs(dna, name, strategy):
    """random bytes (stored blocks), runs (length-258 matches at distance 1) and repeats at distance 32 768"""
    gen = {"random": B.random_bytes, "runs": B.long_runs, "far": B.far_repeats}[name]
    text = gen(5, 400000)
    for level in (0, 1, 6, 9):
        for flush in (None, zlib.Z_FULL_FLUSH):
            # stored blocks add 5 bytes per 64 KiB: 65 280 bytes of text (bgzip's size) keep them in one block
            block_text = 65280 if name == "random" or level == 0 else 65536
            inflates(dna.graph, B.write(text, block_text, level, strategy, flush), text)


def test_inflate_stops(dna):
    """the walk stops at an incomplete block (refused only at the end of the input) and at a member that is not a
    BGZF block"""
    text = CORPUS[:100000]
    data = B.write(text, 20000, eof=False)
    first = bgzf.block(data)[0]
    assert bgzf_inflate(dna.graph, data[:first + 30], c_eof=False) == (text[:20000], first, 1, False)
    assert bgzf_inflate(dna.graph, data[:first + 30], c_eof=True) == (text[:20000], first, 1, True)
    assert bgzf_inflate(dna.graph, data[:first] + gzip.compress(b"x")) == (text[:20000], first, 1, True)
    assert bgzf_inflate(dna.graph, gzip.compress(text) + data) == (b"", 0, 0, True)


def stage_all(al, data, chunk, max_text, json, delim, fwd_rev):
    """the BGZF route by hand: compressed bytes in chunks of `chunk`, text up to max_text per stage"""
    out, tail, cpend, at, c_eof, want = [], b"", b"", 0, False, 0
    while True:
        mt = max(max_text, want)
        while not c_eof and bgzf.text_of(cpend, mt)[0] < mt:
            nxt = data[at:at + chunk]
            at += len(nxt)
            c_eof = not nxt
            cpend += nxt
        batch, c_used, refused, consumed, ended, tail2 = al.stage_fastx_bgzf(tail, cpend, c_eof, mt, delim, fwd_rev)
        assert not refused
        out.append(al.align_staged_text(batch, json))
        cpend = cpend[c_used:]
        if ended or (c_eof and not cpend):
            return b"".join(out)
        want = len(tail2) if consumed == 0 else 0
        tail = tail2


@pytest.mark.parametrize("json", [False, True])
def test_stage_matches_plain(dna, json):
    """TSV and JSON, --fwd-and-reverse and --header-comment-delim, compressed chunks from 1 byte up, and a record
    longer than max_text"""
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    fq = b"".join(b"@%s c%d\n%s\n+\n%s\n" % (h, i, r, b"I" * len(r)) for i, (h, r) in enumerate(zip(names, reads)))
    long = b">long x\n" + b"".join(reads[0][i % 40:i % 40 + 60] + b"\n" for i in range(60))
    for text in (open(os.path.join(EX, GRAPHS[0][1]), "rb").read(), fq, long + fq):
        for delim, fwd_rev in ((None, False), ("|", True)):
            exp = dna.align_fastx_text(text, True, delim, fwd_rev, json)[0]
            assert exp.count(b"\n") >= 2
            for block_text, chunk, max_text in ((500, 1, 300), (97, 64, 200), (65536, 1 << 20, 1 << 20),
                                                (300, 7, 1)):
                data = B.write(text, block_text)
                got = stage_all(dna, data, chunk, max_text, json, delim, fwd_rev)
                assert got == exp, (block_text, chunk, max_text, delim, fwd_rev)


def test_stage_refused_form(dna):
    """multi-line FASTQ, which the device parser refuses: the host restatement parses the inflated text"""
    text = b"@r1\nACGTACGTAC\nGTACGT\n+\nIIIIIIIIII\nIIIIII\n" * 50
    data = B.write(text, 300)
    exp = dna.align_fastx_text(text)[0]
    assert stage_all(dna, data, 100, 500, False, None, False) == exp


# ---- the command ------------------------------------------------------------------------------------------------


def run_main(monkeypatch, tmp_path, argv, chunk_bytes):
    monkeypatch.setenv("MGB_LIB", F.EMU)
    monkeypatch.setattr(cli, "CHUNK_BYTES", chunk_bytes)
    out = str(tmp_path / "out.txt")
    assert cli.main(["align", "-o", out] + argv) == 0
    return open(out, "rb").read()


@pytest.mark.parametrize("g", range(len(GRAPHS)))
def test_command_bgzf(g, tmp_path, monkeypatch):
    dbg, query, alphabet = GRAPHS[g]
    graph = os.path.join(EX, dbg)
    exp = oracle_text(dbg, query, alphabet)
    text = open(os.path.join(EX, query), "rb").read()
    for name, bt in (("q.bgz", 500), ("q.gz", 65536)):
        path = str(tmp_path / name)
        open(path, "wb").write(B.write(text, bt))
        assert bgzf.is_bgzf(path)
        for devices, chunk in (("0", 300), ("0", 1 << 20), ("0,0,0", 300), ("0,0", 97)):
            assert run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", devices, path], chunk) == exp
        one = run_main(monkeypatch, tmp_path, ["-i", graph, "--json", path], 300)
        assert run_main(monkeypatch, tmp_path, ["-i", graph, "--json", "--devices", "0,0,0", path], 300) == one
        assert run_main(monkeypatch, tmp_path, ["-i", graph, "--json", os.path.join(EX, query)], 300) == one


def _handover_files(text):
    """files that are BGZF only in part: name -> bytes"""
    good = B.write(text, 400, eof=False)
    cut = [0]
    at = 0
    while at < len(good):
        at += bgzf.block(good, at)[0]
        cut.append(at)
    mid = cut[len(cut) // 2]
    blk = good[mid:cut[len(cut) // 2 + 1]]
    bad_crc = blk[:-8] + bytes([blk[-8] ^ 1]) + blk[-7:]
    bad_isize = blk[:-4] + (int.from_bytes(blk[-4:], "little") + 1).to_bytes(4, "little")
    fname = gzip.compress(text[-500:])[:3] + b"\x08" + gzip.compress(text[-500:])[4:10] + b"name\x00" + \
        gzip.compress(text[-500:])[10:]
    return {
        "plain_after": good[:mid] + gzip.compress(text[-1000:]),
        "plain_first": gzip.compress(text[:700]) + good,
        "bad_crc": good[:mid] + bad_crc + good[mid + len(blk):],
        "bad_isize": good[:mid] + bad_isize + good[mid + len(blk):],
        "truncated": good[:-5],
        "zero_padding": good + B.EOF_BLOCK + b"\0" * 3000,
        "padding_then_block": good[:mid] + b"\0" * 100 + good[mid:],
        "garbage": good + b"garbage after the last member",
        "fname": good[:mid] + fname,
        "eof_blocks": good[:mid] + B.EOF_BLOCK * 3 + good[mid:] + B.EOF_BLOCK,
    }


@pytest.mark.parametrize("case", ["plain_after", "plain_first", "bad_crc", "bad_isize", "truncated", "zero_padding",
                                  "padding_then_block", "garbage", "fname", "eof_blocks"])
def test_handover(case, tmp_path, monkeypatch, capsys):
    """the same exit code as the gzip route on the same file, and the same bytes when it is 0"""
    monkeypatch.setenv("MGB_LIB", F.EMU)
    graph = os.path.join(EX, GRAPHS[0][0])
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    text = b"".join(b"@%s\n%s\n+\n%s\n" % (h, r, b"F" * len(r)) for h, r in zip(names, reads)) * 3
    path = str(tmp_path / ("in_%s.fq.gz" % case))
    open(path, "wb").write(_handover_files(text)[case])
    for devices in ("0", "0,0,0"):
        for chunk in (256, 1 << 20):
            monkeypatch.setattr(cli, "CHUNK_BYTES", chunk)
            argv = ["-i", graph, "--devices", devices]
            got = B.run(cli, argv, path, tmp_path, capsys)
            exp = B.gzip_route(monkeypatch, cli, argv, path, tmp_path, capsys)
            monkeypatch.setenv("MGB_LIB", F.EMU)
            monkeypatch.setattr(cli, "CHUNK_BYTES", chunk)
            assert got[0] == exp[0], (case, devices, chunk, got[2], exp[2])
            if exp[0] == 0:
                assert got[1] == exp[1] and got[1].count(b"\n") >= 3, (case, devices, chunk)
            else:
                assert got[2].startswith("error: ") and exp[2].startswith("error: ")
    if case == "plain_first":
        assert not bgzf.is_bgzf(path)


def test_grow_rule(tmp_path, monkeypatch):
    """a record of many chunks' text: each stage without a complete record is followed by one with twice the text"""
    graph = os.path.join(EX, GRAPHS[0][0])
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    long = (reads[0] * 40)[:6000]
    text = b">long\n" + b"".join(long[i:i + 70] + b"\n" for i in range(0, len(long), 70)) + \
        open(os.path.join(EX, GRAPHS[0][1]), "rb").read()
    plain = str(tmp_path / "q.fa")
    open(plain, "wb").write(text)
    path = str(tmp_path / "q.fa.bgz")
    open(path, "wb").write(B.write(text, 100))
    sizes = []
    orig = B200Aligner.stage_fastx_bgzf

    def stage(self, head, cbuf, *a, **kw):
        r = orig(self, head, cbuf, *a, **kw)
        sizes.append((len(head), r[3]))
        return r

    monkeypatch.setattr(B200Aligner, "stage_fastx_bgzf", stage)
    exp = run_main(monkeypatch, tmp_path, ["-i", graph, plain], 200)
    for devices in ("0", "0,0"):
        sizes.clear()
        assert run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", devices, path], 200) == exp
        # the record's 1.5 kB is staged 4 times at 200 bytes of text per stage, not 8
        grown = [(h, h2) for (h, c), (h2, _) in zip(sizes, sizes[1:]) if c == 0]
        assert len(grown) >= 3 and all(h2 >= max(2 * h, 200) for h, h2 in grown), sizes


UBSAN = "-fsanitize=undefined -fno-sanitize=alignment,vptr -fsanitize=float-cast-overflow"
UBSAN_EMU = os.path.join(F.ROOT, "tests", "emu", "build", "libmgb_emu_ubsan.so")

FUZZ = r"""
import sys, zlib
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np
import bgzf_common as B, fastx_common as F
from metagraph_b200 import bgzf
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex, bgzf_inflate
idx = DBGSuccinctIndex(BOSSTable.from_sequences(5, ["ACGTACGTTGCA"], lib=%(emu)r), lib=%(emu)r)
rng = np.random.default_rng(%(seed)d)
text = b"".join(F.corpus(n=200))[:60000]
srcs = [B.write(text[:3000], 65536, lvl, s) for s in B.STRATEGIES for lvl in (1, 6, 9)]
srcs += [B.write(B.random_bytes(3, 2000), 65536, 0), B.write(text[:2000], 65536, 6, "default", zlib.Z_FULL_FLUSH)]
n = served = 0
for it in range(%(n)d):
    src = srcs[it %% len(srcs)]
    size = bgzf.block(src)[0]
    blk = bytearray(src[:size])
    kind = it %% 3
    payload_at = 18
    if kind == 0:            # byte flips anywhere in the payload
        for _ in range(int(rng.integers(1, 4))):
            blk[payload_at + int(rng.integers(0, size - 26))] ^= 1 << int(rng.integers(0, 8))
    elif kind == 1:          # the dynamic Huffman header: the first bytes of the payload
        blk[payload_at + int(rng.integers(0, min(40, size - 26)))] ^= 1 << int(rng.integers(0, 8))
    else:                    # a truncated payload under a header that still claims the block's size
        cut = int(rng.integers(1, size - 26))
        p = bytes(blk[18:18 + cut])
        blk = bytearray(B.member(b"", p, crc=int.from_bytes(blk[-8:-4], "little"),
                                 isize=int.from_bytes(blk[-4:], "little")))
    blk = bytes(blk)
    try:
        exp = zlib.decompress(blk, 31)
    except zlib.error:
        exp = None
    got, c_used, nb, refused = bgzf_inflate(idx, blk)
    n += 1
    if not refused:
        served += 1
        assert exp is not None and got == exp, it
print("fuzz done", n, served)
"""


def test_mutation_fuzz_ubsan():
    """seeded byte flips in block payloads and dynamic Huffman headers, and truncated payloads, on the emulation built
    with UBSan (which also keeps the kernel's bounds asserts): every block inflates to zlib's bytes or is refused, and
    no `runtime error:` comes from the kernel sources"""
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu"), "OUT=build/libmgb_emu_ubsan.so",
                           "CXX=g++ " + UBSAN], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    env = dict(os.environ, UBSAN_OPTIONS="print_stacktrace=0:halt_on_error=0")
    import sys
    for seed in (1, 2):
        code = FUZZ % dict(root=F.ROOT, tests=os.path.join(F.ROOT, "tests"), emu=UBSAN_EMU, seed=seed, n=2000)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "fuzz done 2000" in r.stdout, r.stderr[-3000:]
        kernel = [l for l in r.stderr.splitlines() if "runtime error:" in l and "metagraph_b200/csrc/" in l]
        assert not kernel, "\n".join(sorted(set(kernel))[:20])
