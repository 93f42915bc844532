"""mgb_align_batch_text (`metagraph align` TSV lines and JSON records rendered by the library) on the host emulation of
the kernels: the text block equals the host mirror over mgb_align_batch's records byte for byte, in both formats, and
the reference's MT TSV lines and JSON goldens come straight out of it."""
import ctypes
import os
import subprocess

import pytest

import parity_common as P
import text_common as T
from metagraph_b200.aligner import B200Aligner, _pack
from metagraph_b200.config import cli_defaults

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


def test_goldens_emu():
    n = 0
    for idx, cfg, reads in T.goldens(EMU):
        T.check_text(idx, cfg, reads)
        n += 1
    assert n >= 47


@pytest.mark.parametrize("i", range(len(P.RANDOM_CASES) - 1))
def test_random_emu(i):
    T.random_case(EMU, i)


@pytest.mark.parametrize("i", range(len(P.PROTEIN_CASES)))
def test_protein_emu(i):
    T.protein_case(EMU, i)


def test_whole_read_emu():
    T.whole_read_case(EMU)


@pytest.mark.parametrize("mode", ["canonical", "primary"])
@pytest.mark.parametrize("seed", range(4))
def test_fuzz_modes_emu(mode, seed):
    T.fuzz_case(EMU, seed, canonical=mode == "canonical", primary=mode == "primary")


@pytest.mark.parametrize("n_alt", [1, 5, 16, 32])
def test_alt_paths_emu(n_alt):
    out, recs, _ = T.family_case(EMU, n_alt)
    assert max(len(p) for p in recs) == n_alt
    assert out[True].count(b'"is_secondary":true') == sum(max(0, len(p) - 1) for p in recs)


def test_mt_goldens_emu():
    T.check_mt_goldens(EMU)


def test_odd_inputs_emu():
    T.odd_inputs_case(EMU)


def test_small_text_windows_emu(monkeypatch):
    """a device byte budget small enough for dozens of windows (lines straddle them) gives the same text"""
    base, _, _ = T.family_case(EMU, 8)
    monkeypatch.setenv("MGB_TEST_TEXT_CAP", "997")
    small, _, _ = T.family_case(EMU, 8)
    assert small == base
    assert len(base[False]) > 30 * 997 and len(base[True]) > 30 * 997


def test_heap_retry_emu(monkeypatch):
    """pass 0's heap holds a few reads only: the others are answered from later passes' heaps, which the text route keeps
    on the device until it renders"""
    monkeypatch.setenv("MGB_TEST_HEAP0", "60000")
    _, _, st = T.family_case(EMU, 32)
    assert st["num_reads_retried"] > 0


def test_errors_emu():
    """an unknown format and a null header offset array are refused; mgb_results_text refuses a record set"""
    idx, reads, _ = T.random_inputs(EMU, 1, 11, 1000, 5, 60, 0.0)
    try:
        cfg = cli_defaults(11)
        al = B200Aligner(idx, cfg)
        L = al._L
        c = cfg.to_c()
        buf, offs = _pack(reads)
        hbuf, hoffs = _pack([b"h"] * len(reads))
        res = ctypes.c_void_p()
        for fmt in (0, 3, -1):
            assert L.mgb_align_batch_text(idx.handle, ctypes.byref(c), buf.ctypes.data, offs.ctypes.data,
                                          hbuf.ctypes.data, hoffs.ctypes.data, len(reads), fmt, ctypes.byref(res)) == -1
        assert L.mgb_align_batch_text(idx.handle, ctypes.byref(c), buf.ctypes.data, offs.ctypes.data,
                                      hbuf.ctypes.data, None, len(reads), 1, ctypes.byref(res)) == -1
        rec = al.align_batch_raw(buf, offs)
        p, n = ctypes.c_void_p(), ctypes.c_uint64()
        assert L.mgb_results_text(rec, ctypes.byref(p), ctypes.byref(n)) == -1
        al.free_raw(rec)
        assert al.align_batch_text([]) == b"" and al.align_batch_text([], json=True) == b""
    finally:
        idx.close()


def test_text_shim_emu(tmp_path):
    emu_dir = os.path.join(ROOT, "tests", "emu", "build")
    T.check_shim(tmp_path, ["-L" + emu_dir, "-lmgb_emu", "-Wl,-rpath," + emu_dir, "-fopenmp"], EMU)
