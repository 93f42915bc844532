"""mgb_align_batch_device / B200Aligner.align_tensors on the host emulation of the kernels (CPU tensors stand for device
memory there): every column equals mgb_align_batch's records over the same reads, retry passes come from
k_pass_classify's list, and the PCIe byte counts follow their formula."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import device_results_common as D
from metagraph_b200 import _lib
from metagraph_b200.aligner import B200Aligner
from metagraph_b200.config import cli_defaults

EMU = os.path.join(D.ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(D.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("protein", [False, True])
def test_example_graphs_emu(protein):
    D.example_case(EMU, "cpu", protein)


def test_c1_transcripts_emu():
    D.c1_case(EMU, "cpu")


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n_alt", [1, 4, 32])
def test_modes_emu(mode, n_alt):
    D.mode_case(EMU, "cpu", mode, mode, n_alt, nodes=0)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_no_nodes_emu(mode):
    D.mode_case(EMU, "cpu", mode + 3, mode, 4, nodes=1)


def test_forward_only_odd_slice_emu():
    D.mode_case(EMU, "cpu", 1, 0, 2, nodes=0, both=False, odd_start=True)


def test_retry_passes_emu():
    D.retry_case(EMU, "cpu")


def test_heap_retry_passes_emu(monkeypatch):
    D.heap_retry_case(EMU, "cpu", monkeypatch)


def test_empty_batches_emu():
    idx, _ = D.mode_index(EMU, 2, 15, 0, nreads=1)
    try:
        cfg = cli_defaults(15)
        D.check(idx, cfg, [], "cpu")
        D.check(idx, cfg, ["", "", "ACG"], "cpu")
    finally:
        idx.close()


def test_errors_emu():
    idx, reads = D.mode_index(EMU, 1, 15, 0, nreads=5)
    try:
        al = B200Aligner(idx, cli_defaults(15))
        t, o = D.as_tensors(reads, "cpu")
        L = al._L
        c = al.config.to_c()
        h = ctypes.c_void_p()
        # decreasing offsets
        bad = o.clone()
        bad[1], bad[2] = bad[2].item(), bad[1].item()
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), t.data_ptr(), bad.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == -1
        with pytest.raises(_lib.MgbError) as e:
            al.align_tensors(t, bad)
        assert e.value.code == -1
        # a config the record route refuses fails the same way, with the same text
        cfg = cli_defaults(15, num_alternative_paths=33)
        c2 = cfg.to_c()
        buf, offs = D._pack([r.encode() for r in reads])
        res = ctypes.c_void_p()
        rc = L.mgb_align_batch(idx.handle, ctypes.byref(c2), buf.ctypes.data, offs.ctypes.data, len(reads),
                               ctypes.byref(res))
        msg = L.mgb_last_error()
        assert rc != 0
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c2), t.data_ptr(), o.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == rc
        assert L.mgb_last_error() == msg
        # a null column for a non-empty array; mgb_device_results_free(NULL)
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), t.data_ptr(), o.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == 0
        z = _lib.mgb_device_sizes_t()
        assert L.mgb_device_results_sizes(h, ctypes.byref(z)) == 0 and z.n_alignments > 0
        cols = _lib.mgb_device_columns_t()
        assert L.mgb_device_results_write(h, ctypes.byref(cols), None) == -1
        L.mgb_device_results_free(h)
        L.mgb_device_results_free(None)
        # the Python layer: dtypes, shapes, offsets past the reads
        with pytest.raises(ValueError):
            al.align_tensors(t.to(torch.int8), o)
        with pytest.raises(ValueError):
            al.align_tensors(t, o.to(torch.int32))
        with pytest.raises(ValueError):
            al.align_tensors(t[:-1], o)
        with pytest.raises(ValueError):
            al.align_tensors(np.zeros(3, np.uint8), o)
    finally:
        idx.close()
