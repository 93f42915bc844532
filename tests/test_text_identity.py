"""The `identity` field of the JSON records (matches / query_len, printed as "%.17g" with ".0" appended when the text has
no '.', 'e' or 'n'; aligner.py _json_value) as the text route's device code prints it (format_core.cuh
format_identity), against Python's own "%.17g": every pair 0 <= m <= q <= 4096, and seeded samples of q up to 2^32 - 1
with m in {0, 1, 2, q - 1, q, random}, which reach the exponent form and the widest shifts. Once on the host build of
the formatter and once on the sm_90a build."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "devtext", "build", "libmgb_text_emu.so")
DEV = os.path.join(ROOT, "tests", "devtext", "build", "libmgb_text.so")


def python_identity(m, q):
    t = "%.17g" % (m / q)
    return t if any(c in t for c in ".en") else t + ".0"


def formatted(lib, m, q):
    L = ctypes.CDLL(lib)
    m = np.ascontiguousarray(m, np.uint32)
    q = np.ascontiguousarray(q, np.uint32)
    out = np.zeros(len(m) * 32, np.uint8)
    rc = L.mgbt_identity(ctypes.c_void_p(m.ctypes.data), ctypes.c_void_p(q.ctypes.data), ctypes.c_uint64(len(m)),
                         ctypes.c_void_p(out.ctypes.data))
    assert rc == 0, rc
    return out.view("S32")


def all_pairs(q_lo, q_hi):
    q = np.concatenate([np.full(n + 1, n, np.uint32) for n in range(q_lo, q_hi)])
    m = np.concatenate([np.arange(n + 1, dtype=np.uint32) for n in range(q_lo, q_hi)])
    return m, q


def sampled_pairs(seed=17, n=60000):
    rng = np.random.default_rng(seed)
    q = np.concatenate([rng.integers(4097, 2 ** 32, n, dtype=np.uint64),
                        np.array([2 ** 32 - 1, 2 ** 32 - 2, 2 ** 31, 2 ** 31 + 1, 10 ** 9, 99999, 100000, 100001],
                                 np.uint64)])
    m = np.concatenate([np.zeros_like(q), np.ones_like(q), np.full_like(q, 2), q - 1, q,
                        (rng.random(len(q)) * (q + 1)).astype(np.uint64).clip(0, q)])
    q = np.tile(q, 6)
    # odd m over q = 2^18 .. 2^22: m / q has 18 .. 22 fraction digits ending in 5, so rounding to 17 significant digits
    # meets exact ties (round half to even)
    tq = np.repeat(2 ** np.arange(18, 23, dtype=np.uint64), 20000)
    tm = (rng.integers(0, tq // 2, dtype=np.uint64) * 2 + 1)
    return np.concatenate([m, tm]).astype(np.uint32), np.concatenate([q, tq]).astype(np.uint32)


def check(lib, m, q):
    got = formatted(lib, m, q)
    exp = np.array([python_identity(int(a), int(b)).encode() for a, b in zip(m.tolist(), q.tolist())], dtype="S32")
    bad = np.nonzero(got != exp)[0]
    assert not len(bad), [(int(m[i]), int(q[i]), got[i], exp[i]) for i in bad[:5]]
    return len(m)


def sweep(lib):
    n = 0
    for lo in range(1, 4097, 512):
        n += check(lib, *all_pairs(lo, min(lo + 512, 4097)))
    n += check(lib, *sampled_pairs())
    # the exponent form is reached (identity below 1e-4), and so is the rounding carry into a new decade
    m, q = sampled_pairs()
    assert any(b"e-" in x for x in formatted(lib, m, q))
    return n


def test_identity_sweep_emu():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "devtext")], stdout=subprocess.DEVNULL)
    assert sweep(EMU) > 8_000_000


@pytest.mark.gpu
def test_identity_sweep_gpu():
    assert os.path.exists(DEV), "build() makes %s" % DEV
    assert sweep(DEV) > 8_000_000
