"""Plain gzip input on the host emulation: the speculative inflater against zlib for every writer knob and forced
sub-range sizes, true block starts found at flush points, injected false candidates that never change a byte, the
staged gzip route against the plain route's text, the command against the oracle, and refusals against Python's gzip
route."""
import gzip
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import bgzf_common as B
import fastx_common as F
from metagraph_b200 import cli
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, GzipStream, gzip_inflate
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


def member(text, level=6, strategy="default", flush=None, flg=0, extra=b"", name=b"", comment=b""):
    """a gzip member (RFC 1952) around B.deflate's stream, with the optional header fields of `flg`"""
    hdr = struct.pack("<BBBBIBB", 31, 139, 8, flg, 0, 0, 255)
    if flg & 4:
        hdr += struct.pack("<H", len(extra)) + extra
    if flg & 8:
        hdr += name + b"\0"
    if flg & 16:
        hdr += comment + b"\0"
    if flg & 2:
        hdr += struct.pack("<H", zlib.crc32(hdr) & 0xffff)
    return hdr + B.deflate(text, level, strategy, flush) + struct.pack("<II", zlib.crc32(text), len(text) & 0xffffffff)


def inflates(index, data, text, sub_bytes=0):
    got, c_used, refused, counts = gzip_inflate(index, data, sub_bytes=sub_bytes)
    assert (c_used, refused) == (len(data), False)
    assert got == text
    return counts


CORPUS = b"".join(F.corpus(n=300))
FASTQ = B.fastq(np.random.default_rng(3), 3000)
STRATEGIES = ["default", "filtered", "huffman", "rle"]


@pytest.mark.parametrize("strategy", STRATEGIES)
def test_inflate_knobs(dna, strategy):
    """levels 1-9, no flush, sync flush and full flush, the default and a forced sub-range of a few hundred bytes"""
    for level in range(1, 10):
        for flush in (None, zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            for text in (CORPUS, FASTQ):
                data = member(text, level, strategy, flush)
                assert zlib.decompress(data, 31) == text
                for sub in (0, 300, 4000):
                    inflates(dna.graph, data, text, sub)


@pytest.mark.parametrize("name", ["random", "runs", "far"])
def test_inflate_inputs(dna, name):
    """random bytes (stored blocks), runs (length-258 matches at distance 1) and repeats at distance 32 768, which
    cross sub-range boundaries at every sub-range size and stage boundaries where a slot fills"""
    gen = {"random": B.random_bytes, "runs": B.long_runs, "far": B.far_repeats}[name]
    text = gen(5, 400000)
    for strategy in STRATEGIES:
        for level in (1, 6, 9):
            data = member(text, level, strategy)
            for sub in (0, 500, 7000):
                inflates(dna.graph, data, text, sub)


def test_far_repeats_confirmed(dna):
    """distance-32 768 matches resolved through the window chain: the text is split, and still equals zlib's"""
    text = B.far_repeats(7, 1_500_000)
    n_sub, found, confirmed = inflates(dna.graph, member(text, 6), text, 2000)
    assert confirmed >= 5 and found == confirmed


def test_multi_member(dna):
    text = FASTQ[:50000] + CORPUS + FASTQ[50000:]
    data = member(FASTQ[:50000], 1) + member(CORPUS, 9, flg=8, name=b"x.fa") + member(FASTQ[50000:], 6, flg=2 | 4 | 16,
                                                                                       extra=b"ab\x02\x00xy", comment=b"c")
    inflates(dna.graph, data, text, 0)
    inflates(dna.graph, data, text, 400)
    assert gzip_inflate(dna.graph, b"") == (b"", 0, False, (0, 0, 0))


def test_flush_points_found(dna):
    """a full flush ends a block at a byte boundary (an empty stored block) and the next block starts there: the finder
    started a few bytes before that point returns it, and the chain confirms it"""
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    third = len(FASTQ) // 3
    p1 = c.compress(FASTQ[:third]) + c.flush(zlib.Z_FULL_FLUSH)
    p2 = c.compress(FASTQ[third:2 * third]) + c.flush(zlib.Z_FULL_FLUSH)
    raw = p1 + p2 + c.compress(FASTQ[2 * third:]) + c.flush()
    data = member(b"")[:10] + raw + struct.pack("<II", zlib.crc32(FASTQ), len(FASTQ))
    for back in (1, 3, 7):
        sub = len(p1) - back                    # sub-range 1 starts `back` bytes before the block after the flush
        got, c_used, refused, (n_sub, found, confirmed) = gzip_inflate(dna.graph, data, sub_bytes=sub)
        assert got == FASTQ and not refused
        assert confirmed >= 1 and found >= 1


def test_false_candidates(dna):
    """candidates in the middle of blocks, inside a block header, past the member's end and everywhere wrong: the text
    never changes, only the confirmed count drops"""
    data = member(FASTQ, 6) + member(CORPUS, 6)
    text = FASTQ + CORPUS
    sub = 3000
    _, _, _, (n_sub, found, confirmed) = gzip_inflate(dna.graph, data, sub_bytes=sub)
    assert confirmed >= 3
    rng = np.random.default_rng(11)
    bits = len(data) * 8
    cases = {
        "mid_block": [int(x) for x in rng.integers(80, bits, 400)],
        "header": [80 + 5, 80 + 17, 80 + 40],
        "past_end": [bits - 20, bits + 100, bits * 2],
        "all_wrong": [80 + sub * 8 * j + 1 + int(rng.integers(0, 100)) for j in range(1, len(data) // sub + 1)],
    }
    for name, cands in cases.items():
        got, c_used, refused, counts = gzip_inflate(dna.graph, data, sub_bytes=sub, cands=sorted(cands))
        assert (got, c_used, refused) == (text, len(data), False), name
        assert counts[2] <= confirmed, name
    assert gzip_inflate(dna.graph, data, sub_bytes=sub, cands=cases["all_wrong"])[3][2] == 0


def test_inflate_refuses(dna):
    data = member(FASTQ, 6)
    assert gzip_inflate(dna.graph, b"not gzip")[2]
    assert gzip_inflate(dna.graph, data[:-3])[2]                                   # truncated trailer
    assert gzip_inflate(dna.graph, data[:len(data) // 2])[2]                       # truncated stream
    bad = data[:-8] + bytes([data[-8] ^ 1]) + data[-7:]
    assert gzip_inflate(dna.graph, bad)[2]
    assert gzip_inflate(dna.graph, data + b"garbage")[1:3] == (len(data), True)
    assert gzip_inflate(dna.graph, data[:len(data) // 2], c_eof=False)[2] is False


# ---- staging by hand ----------------------------------------------------------------------------------------------


def stage_all(al, data, chunk, max_text, json=False, delim=None, fwd_rev=False):
    """the gzip route by hand: compressed bytes in chunks of `chunk`, at least max_text of text per stage"""
    stream = GzipStream(al._L)
    out, tail, cpend, at, c_eof, want, c_want = [], b"", b"", 0, False, 0, chunk
    try:
        while True:
            mt = max(max_text, want)
            while not c_eof and len(cpend) < c_want:
                nxt = data[at:at + chunk]
                at += len(nxt)
                c_eof = not nxt
                cpend += nxt
            batch, c_used, refused, consumed, ended, tail2 = al.stage_fastx_gzip(stream, tail, cpend, c_eof, mt, delim,
                                                                                 fwd_rev)
            assert not refused
            out.append(al.align_staged_text(batch, json))
            cpend = cpend[c_used:]
            if ended or (c_eof and not cpend and not stream.state()[0]):
                return b"".join(out)
            c_want = 2 * max(c_want, len(cpend)) if c_used == 0 else chunk
            want = len(tail2) if consumed == 0 else 0
            tail = tail2
    finally:
        stream.close()


@pytest.mark.parametrize("json", [False, True])
def test_stage_matches_plain(dna, json):
    """TSV and JSON, --fwd-and-reverse and --header-comment-delim, compressed chunks from 1 byte up, multi-member
    files and every optional header field"""
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    fq = b"".join(b"@%s c%d\n%s\n+\n%s\n" % (h, i, r, b"I" * len(r)) for i, (h, r) in enumerate(zip(names, reads)))
    fa = open(os.path.join(EX, GRAPHS[0][1]), "rb").read()
    for text in (fa, fq):
        half = len(text) // 2
        files = [member(text), member(text[:half], 1, flg=8, name=b"q.fq") + member(text[half:], 9, flg=2 | 4 | 16,
                                                                                     extra=b"zz\x01\x00!", comment=b"c")]
        for delim, fwd_rev in ((None, False), ("|", True)):
            exp = dna.align_fastx_text(text, True, delim, fwd_rev, json)[0]
            assert exp.count(b"\n") >= 2
            for data in files:
                for chunk, max_text in ((1, 300), (97, 200), (1 << 20, 1 << 20), (7, 1)):
                    assert stage_all(dna, data, chunk, max_text, json, delim, fwd_rev) == exp, (chunk, max_text)


# ---- the command ------------------------------------------------------------------------------------------------


def run_main(monkeypatch, tmp_path, argv, chunk_bytes):
    monkeypatch.setenv("MGB_LIB", F.EMU)
    monkeypatch.setattr(cli, "CHUNK_BYTES", chunk_bytes)
    out = str(tmp_path / "out.txt")
    assert cli.main(["align", "-o", out] + argv) == 0
    return open(out, "rb").read()


@pytest.mark.parametrize("g", range(len(GRAPHS)))
def test_command_gzip(g, tmp_path, monkeypatch):
    dbg, query, alphabet = GRAPHS[g]
    graph = os.path.join(EX, dbg)
    exp = oracle_text(dbg, query, alphabet)
    text = open(os.path.join(EX, query), "rb").read()
    path = str(tmp_path / (query + ".gz"))
    with gzip.open(path, "wb") as f:            # FNAME set, as gzip writes it
        f.write(text)
    assert cli.route_of(path) == "gzip"
    stages, handed = [], []
    orig = cli._Token._stage_gzip

    def stage(self, *a):
        stages.append(1)
        return orig(self, *a)

    monkeypatch.setattr(cli._Token, "_stage_gzip", stage)
    monkeypatch.setattr(cli._Token, "_hand_over", lambda self, *a: handed.append(1))
    for devices in ("0", "0,0,0"):
        for chunk in (256, 1 << 20):
            stages.clear()
            handed.clear()
            assert run_main(monkeypatch, tmp_path, ["-i", graph, "--devices", devices, path], chunk) == exp
            assert stages and not handed


def _refusal_files(text):
    """files the gzip route refuses at some point: name -> bytes"""
    good = member(text, 6)
    mid = 10 + len(good) // 2
    blk = B.write(text[-3000:], 1000)
    return {
        "corrupt": good[:mid] + bytes([good[mid] ^ 0x10]) + good[mid + 1:],
        "bad_crc": good[:-8] + bytes([good[-8] ^ 1]) + good[-7:],
        "bad_isize": good[:-4] + struct.pack("<I", len(text) + 1),
        "truncated": good[:-5],
        "truncated_mid": good[:mid],
        "zero_padding": good + b"\0" * 3000,
        "garbage": good + b"garbage after the last member",
        "not_gzip": text,
        "level0": member(text, 0),
        "fixed": member(text, 6, "fixed"),
        "bgzf_after": good + blk,
        "two_members": member(text[:5000], 6) + good,
    }


@pytest.mark.parametrize("case", ["corrupt", "bad_crc", "bad_isize", "truncated", "truncated_mid", "zero_padding",
                                  "garbage", "not_gzip", "level0", "fixed", "bgzf_after", "two_members"])
def test_refusals(case, tmp_path, monkeypatch, capsys):
    """the same exit code as Python's gzip route on the same file, and the same bytes when it is 0"""
    monkeypatch.setenv("MGB_LIB", F.EMU)
    graph = os.path.join(EX, GRAPHS[0][0])
    names, reads = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))
    text = b"".join(b"@%s\n%s\n+\n%s\n" % (h, r, b"F" * len(r)) for h, r in zip(names, reads)) * 30
    path = str(tmp_path / ("in_%s.fq.gz" % case))
    open(path, "wb").write(_refusal_files(text)[case])
    assert cli.route_of(path) == "gzip"
    for devices in ("0", "0,0,0"):
        for chunk in (256, 1 << 20):
            argv = ["-i", graph, "--devices", devices]
            monkeypatch.setattr(cli, "CHUNK_BYTES", chunk)
            got = B.run(cli, argv, path, tmp_path, capsys)
            monkeypatch.setattr(cli, "route_of", lambda p: "host")
            exp = B.run(cli, argv, path, tmp_path, capsys)
            monkeypatch.undo()
            monkeypatch.setenv("MGB_LIB", F.EMU)
            assert got[0] == exp[0], (case, devices, chunk, got[2], exp[2])
            if exp[0] == 0:
                assert got[1] == exp[1], (case, devices, chunk)
            else:
                assert got[2].startswith("error: ") and exp[2].startswith("error: ")


def test_unsplit_member_handed_over(dna, tmp_path):
    """a stored or fixed-Huffman member larger than one sub-range's slot is refused at its first stage, before any of
    it is staged"""
    fq = B.fastq(np.random.default_rng(4), 8000)
    for data in (member(B.random_bytes(2, 1_500_000), 0), member(fq, 6, "fixed")):
        stream = GzipStream(dna._L)
        try:
            batch, c_used, refused, consumed, ended, tail = dna.stage_fastx_gzip(stream, b"", data, True, 1 << 20)
            dna.free_staged(batch)
            assert (c_used, refused, stream.state()) == (0, True, (False, 0))
        finally:
            stream.close()


UBSAN = "-fsanitize=undefined -fno-sanitize=alignment,vptr -fsanitize=float-cast-overflow"
UBSAN_EMU = os.path.join(F.ROOT, "tests", "emu", "build", "libmgb_emu_ubsan.so")

FUZZ = r"""
import sys, zlib, struct
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np
import bgzf_common as B, fastx_common as F
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex, gzip_inflate
idx = DBGSuccinctIndex(BOSSTable.from_sequences(5, ["ACGTACGTTGCA"], lib=%(emu)r), lib=%(emu)r)
rng = np.random.default_rng(%(seed)d)
text = B.fastq(np.random.default_rng(1), 400)
def member(t, lvl, s):
    return b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + B.deflate(t, lvl, s) + struct.pack("<II", zlib.crc32(t), len(t))
srcs = [member(text, lvl, s) for s in ("default", "huffman", "rle", "fixed") for lvl in (1, 6, 9)]
n = served = 0
for it in range(%(n)d):
    m = bytearray(srcs[it %% len(srcs)])
    kind = it %% 3
    if kind == 0:            # byte flips anywhere in the stream
        for _ in range(int(rng.integers(1, 4))):
            m[10 + int(rng.integers(0, len(m) - 18))] ^= 1 << int(rng.integers(0, 8))
    elif kind == 1:          # the first block's header
        m[10 + int(rng.integers(0, 40))] ^= 1 << int(rng.integers(0, 8))
    else:                    # a truncated stream
        m = m[:10 + int(rng.integers(1, len(m) - 10))]
    m = bytes(m)
    try:
        exp = zlib.decompress(m, 31)
    except zlib.error:
        exp = None
    sub = int(rng.choice([0, 200, 1000]))
    cands = None
    if it %% 2:              # injected candidates: anywhere, some true
        cands = sorted(int(x) for x in rng.integers(0, len(m) * 8 + 64, int(rng.integers(1, 40))))
    got, c_used, refused, counts = gzip_inflate(idx, m, sub_bytes=sub, cands=cands)
    n += 1
    if not refused:
        served += 1
        assert exp is not None and got == exp and c_used == len(m), it
print("fuzz done", n, served)
"""


def test_mutation_fuzz_ubsan():
    """seeded byte flips in members and their first block header, truncated members and injected candidates, on the
    emulation built with UBSan (which also keeps the decoder's bounds asserts): every member inflates to zlib's bytes or
    is refused, and no `runtime error:` comes from the kernel sources"""
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu"), "OUT=build/libmgb_emu_ubsan.so",
                           "CXX=g++ " + UBSAN], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    env = dict(os.environ, UBSAN_OPTIONS="print_stacktrace=0:halt_on_error=0")
    for seed in (1, 2):
        code = FUZZ % dict(root=F.ROOT, tests=os.path.join(F.ROOT, "tests"), emu=UBSAN_EMU, seed=seed, n=1500)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "fuzz done 1500" in r.stdout, r.stderr[-3000:]
        kernel = [l for l in r.stderr.splitlines() if "runtime error:" in l and "metagraph_b200/csrc/" in l]
        assert not kernel, "\n".join(sorted(set(kernel))[:20])
