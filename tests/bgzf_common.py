"""BGZF input: a BGZF writer on Python's zlib with the knobs the inflate tests sweep (level, strategy, text per block,
flushes inside a block), the inputs they inflate, and the command's gzip route as the reference for files that are BGZF
only in part."""
import concurrent.futures
import os
import struct
import zlib

import numpy as np

# the empty block htslib's bgzip ends every file with (SAM/BAM format specification, §4.1.2)
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def deflate(text, level=6, strategy="default", flush=None):
    """raw DEFLATE of text; flush (zlib.Z_SYNC_FLUSH / Z_FULL_FLUSH) after each third of it, which ends a DEFLATE
    block there and writes an empty stored block"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, STRATEGIES[strategy])
    if flush is None:
        return c.compress(text) + c.flush()
    t = len(text) // 3
    parts = [text[:t], text[t:2 * t], text[2 * t:]]
    return b"".join(c.compress(p) + c.flush(flush) for p in parts) + c.flush()


def member(text, payload, extra=b"", flg=4, crc=None, isize=None):
    """a gzip member with a BC subfield (after `extra`, other subfields) around a DEFLATE payload"""
    xf = extra + b"BC" + struct.pack("<HH", 2, 12 + 6 + len(extra) + len(payload) + 8 - 1)
    hdr = struct.pack("<BBBBIBBH", 31, 139, 8, flg, 0, 0, 255, len(xf)) + xf
    return hdr + payload + struct.pack("<II", zlib.crc32(text) if crc is None else crc,
                                       len(text) if isize is None else isize)


def write(text, block_text=65280, level=6, strategy="default", flush=None, eof=True):
    """text as BGZF: blocks of block_text bytes of text (the last one shorter), then the EOF block (zlib releases the
    GIL, so large texts are compressed on several threads)"""
    def one(i):
        t = text[i:i + block_text]
        p = deflate(t, level, strategy, flush)
        assert 18 + len(p) + 8 <= 65536, "block of %d bytes: lower block_text" % (18 + len(p) + 8)
        return member(t, p)

    starts = range(0, len(text), block_text)
    if len(text) > 1 << 24:
        with concurrent.futures.ThreadPoolExecutor(min(16, os.cpu_count() or 1)) as ex:
            out = list(ex.map(one, starts))
    else:
        out = [one(i) for i in starts]
    if eof:
        out.append(EOF_BLOCK)
    return b"".join(out)


def n_blocks(data):
    from metagraph_b200 import bgzf
    n = at = 0
    while at < len(data):
        b = bgzf.block(data, at)
        assert b not in (None, "cut")
        at += b[0]
        n += 1
    return n


def random_bytes(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def long_runs(seed, n):
    """runs of one byte of up to 2 000 bytes: matches of length 258 at distance 1"""
    rng = np.random.default_rng(seed)
    out = bytearray()
    while len(out) < n:
        out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 2000))
    return bytes(out[:n])


def far_repeats(seed, n):
    """a random 32 KiB segment repeated with a few changes: matches at distance 32 768"""
    rng = np.random.default_rng(seed)
    seg = bytearray(rng.integers(65, 70, 32768, dtype=np.uint8).tobytes())
    out = bytearray()
    while len(out) < n:
        seg[int(rng.integers(0, len(seg)))] = int(rng.integers(0, 256))
        out += seg
    return bytes(out[:n])


def fastq(rng, n, L=150):
    """n FASTQ reads of L bases with qualities drawn from a seeded distribution"""
    acgt = np.frombuffer(b"ACGT", np.uint8)
    q = np.frombuffer(b"#,:FFFFF", np.uint8)
    seqs = acgt[rng.integers(0, 4, (n, L))]
    quals = q[rng.integers(0, len(q), (n, L))]
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, seqs[i].tobytes(), quals[i].tobytes()) for i in range(n))


def fastq_of(reads):
    """FASTQ of the rows of a uint8 read matrix, with constant qualities as the command's other file tests write"""
    L = reads.shape[1]
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, reads[i].tobytes(), b"F" * L) for i in range(len(reads)))


def gzip_route(monkeypatch, cli, argv, path, tmp_path, capsys):
    """run() with the BGZF route turned off, which is the gzip route every .gz file took before it (this undoes the
    test's other monkeypatches too)"""
    from metagraph_b200 import bgzf
    monkeypatch.setattr(bgzf, "is_bgzf", lambda p: False)
    try:
        return run(cli, argv, path, tmp_path, capsys)
    finally:
        monkeypatch.undo()


def run(cli, argv, path, tmp_path, capsys):
    """(exit code, output bytes, stderr) of the command on `path`"""
    out = str(tmp_path / ("out_%d.txt" % len(os.listdir(str(tmp_path)))))
    capsys.readouterr()
    rc = cli.main(["align", "-o", out] + argv + [path])
    err = capsys.readouterr().err
    return rc, (open(out, "rb").read() if os.path.exists(out) else b""), err

