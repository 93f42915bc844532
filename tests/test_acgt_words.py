"""The word helpers of k_prepare_exact (metagraph_b200/csrc/acgt_words.cuh) built for the host (tests/devwords): packing
of raw bytes into 2-bit codes and their validity (every byte value at every position of a 32-byte window and every
alignment mod 4), the packed reverse complement, per-letter counts and the record characters, against a Python
restatement."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tests", "devwords", "build", "libmgb_words.so")
COMP = {ord("A"): ord("T"), ord("C"): ord("G"), ord("G"): ord("C"), ord("T"): ord("A")}


@pytest.fixture(scope="module")
def W():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "devwords")], stdout=subprocess.DEVNULL)
    L = ctypes.CDLL(LIB)
    u64, u32, p = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p
    for name, res, args in [("mgbw_pack32", u64, [p, ctypes.c_int, ctypes.POINTER(u32)]), ("mgbw_valid4", u32, [u32]),
                            ("mgbw_codes4", u32, [u32]), ("mgbw_rc32", u64, [u64]),
                            ("mgbw_count", None, [u64, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
                            ("mgbw_bytes8", u64, [p, ctypes.c_int]), ("mgbw_chars8", u64, [u64, ctypes.c_int])]:
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    return L


def valid(c):
    return (c & 0xDF) in b"ACGT"


def code(c):
    u = c & 0xDF
    return ((u >> 1) ^ (u >> 2)) & 3


def test_pack32_every_byte_everywhere(W):
    rng = np.random.default_rng(5)
    buf = (ctypes.c_uint8 * 80)()
    inv = ctypes.c_uint32()
    for align in range(4):
        for t in range(32):
            fill = rng.choice(np.frombuffer(b"ACGTacgt", np.uint8), 80)
            for v in range(256):
                for i in range(80):
                    buf[i] = int(fill[i])
                buf[align + t] = v
                got = W.mgbw_pack32(ctypes.addressof(buf), align, ctypes.byref(inv))
                win = [buf[align + i] for i in range(32)]
                bad = sum(1 << i for i, c in enumerate(win) if not valid(c))
                assert inv.value == bad, (align, t, v)
                want = sum(code(c) << (2 * i) for i, c in enumerate(win))
                assert got == want, (align, t, v)


def test_valid4_codes4_every_byte(W):
    for v in range(256):
        for j in range(4):
            x = (0x41434754 & ~(0xFF << (8 * j))) | (v << (8 * j))
            bs = [(x >> (8 * i)) & 0xFF for i in range(4)]
            assert W.mgbw_valid4(x) == sum((0xFF << (8 * i)) for i, c in enumerate(bs) if valid(c))
            assert W.mgbw_codes4(x) == sum(code(c) << (2 * i) for i, c in enumerate(bs))


def test_rc32_and_counts(W):
    rng = np.random.default_rng(6)
    counts = (ctypes.c_int * 4)()
    for _ in range(2000):
        codes = [int(c) for c in rng.integers(0, 4, 32)]
        w = sum(c << (2 * i) for i, c in enumerate(codes))
        assert W.mgbw_rc32(w) == sum((3 - c) << (2 * (31 - i)) for i, c in enumerate(codes))
        n = int(rng.integers(0, 33))
        for i in range(4):
            counts[i] = 0
        W.mgbw_count(w, n, counts)
        assert list(counts) == [codes[:n].count(c) for c in range(4)]


def test_chars8_and_bytes8(W):
    rng = np.random.default_rng(7)
    buf = (ctypes.c_uint8 * 32)()
    for _ in range(2000):
        raw = [int(c) for c in rng.choice(np.frombuffer(b"ACGTacgt", np.uint8), 32)]
        for i in range(32):
            buf[i] = raw[i]
        off = int(rng.integers(0, 16))
        x = W.mgbw_bytes8(ctypes.addressof(buf), off)
        assert x == sum(raw[off + j] << (8 * j) for j in range(8))
        up = [c & 0xDF for c in raw[off:off + 8]]
        assert W.mgbw_chars8(x, 0) == sum(c << (8 * j) for j, c in enumerate(up))
        assert W.mgbw_chars8(x, 1) == sum(COMP[c] << (8 * j) for j, c in enumerate(reversed(up)))
