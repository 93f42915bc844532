"""mgb_align_batch_device / B200Aligner.align_tensors on the H100: every column equals mgb_align_batch's records over the
same reads (the cases of the emulation tests, plus C2- and C3-shaped batches at scale), offsets on the host and on the
device, reads produced on a side stream, and the refusals of pointers that are not on the index's device."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import device_results_common as D
from metagraph_b200 import _lib
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("protein", [False, True])
def test_example_graphs_gpu(protein):
    D.example_case(None, DEV, protein)


def test_c1_transcripts_gpu():
    D.c1_case(None, DEV)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n_alt", [1, 4, 32])
def test_modes_gpu(mode, n_alt):
    D.mode_case(None, DEV, mode, mode, n_alt, nodes=0)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_no_nodes_gpu(mode):
    D.mode_case(None, DEV, mode + 3, mode, 4, nodes=1)


@pytest.mark.parametrize("on_device", [False, True])
def test_input_forms_gpu(on_device):
    """offsets on the host or the device; reads as a slice from an odd byte to the very end of its tensor"""
    D.mode_case(None, DEV, 1, 0, 2, nodes=0, offsets_on_device=on_device, odd_start=True)
    D.mode_case(None, DEV, 2, 0, 2, nodes=0, both=False, offsets_on_device=on_device, odd_start=True)


@pytest.mark.parametrize("on_device", [False, True])
def test_retry_passes_gpu(on_device):
    D.retry_case(None, DEV, offsets_on_device=on_device)


@pytest.mark.parametrize("on_device", [False, True])
def test_heap_retry_passes_gpu(monkeypatch, on_device):
    D.heap_retry_case(None, DEV, monkeypatch, offsets_on_device=on_device)


def test_empty_batches_gpu():
    idx, _ = D.mode_index(None, 2, 15, 0, nreads=1)
    try:
        cfg = cli_defaults(15)
        D.check(idx, cfg, [], DEV)
        D.check(idx, cfg, ["", "", "ACG"], DEV, offsets_on_device=True)
    finally:
        idx.close()


def test_stream_order_gpu():
    """reads filled by a non-blocking copy from pinned memory on a side stream, aligned under that stream, and the
    columns read on it with no explicit synchronisation"""
    idx, reads = D.mode_index(None, 4, 19, 0, nreads=400)
    try:
        cfg = cli_defaults(19, min_exact_match=0.0)
        al = B200Aligner(idx, cfg)
        read_first, cols, seq, _, _, st = D.records(al, [r.encode() for r in reads])
        host, offs = D.as_tensors(reads, "cpu")
        host = host.pin_memory()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            dev = torch.empty(host.numel(), dtype=torch.uint8, device=DEV)
            dev.copy_(host, non_blocking=True)
            got = al.align_tensors(dev, offs.to(DEV, non_blocking=True))
            score_sum = got.score.to(torch.int64).sum()
            first = got.read_first.clone()
        s.synchronize()
        assert first.cpu().tolist() == read_first.tolist()
        assert int(score_sum) == int(cols["score"].sum())
    finally:
        idx.close()


def test_errors_gpu():
    idx, reads = D.mode_index(None, 1, 15, 0, nreads=5)
    try:
        al = B200Aligner(idx, cli_defaults(15))
        L = al._L
        c = al.config.to_c()
        h = ctypes.c_void_p()
        t, o = D.as_tensors(reads, DEV)
        host, _ = D.as_tensors(reads, "cpu")
        # a host pointer for the reads, or for offsets said to be on the device
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), host.data_ptr(), o.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == -1
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), t.data_ptr(), o.data_ptr(), 1, len(reads), None,
                                        ctypes.byref(h)) == -1
        with pytest.raises(ValueError):
            al.align_tensors(host, o)
        bad = o.clone()
        bad[1], bad[2] = bad[2].item(), bad[1].item()
        with pytest.raises(_lib.MgbError) as e:
            al.align_tensors(t, bad.to(DEV))
        assert e.value.code == -1
        c33 = cli_defaults(15, num_alternative_paths=33).to_c()
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c33), t.data_ptr(), o.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == -4
        assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), t.data_ptr(), o.data_ptr(), 0, len(reads), None,
                                        ctypes.byref(h)) == 0
        assert L.mgb_device_results_write(h, ctypes.byref(_lib.mgb_device_columns_t()), None) == -1
        L.mgb_device_results_free(h)
        L.mgb_device_results_free(None)
        if torch.cuda.device_count() > 1:
            other = t.to("cuda:1")
            assert L.mgb_align_batch_device(idx.handle, ctypes.byref(c), other.data_ptr(), o.data_ptr(), 0, len(reads),
                                            None, ctypes.byref(h)) == -1
    finally:
        idx.close()


# ---------------------------------------------------------------------------------------------- at scale ----
def _bench():
    sys.path.insert(0, D.ROOT)
    import bench
    return bench


def _scale_check(boss, cfg, buf, offs, sample=3000):
    """align_tensors against mgb_align_batch: fixed columns in full, sequence and CIGAR bytes of a sample"""
    idx = DBGSuccinctIndex(boss, device=0)
    try:
        al = B200Aligner(idx, cfg)
        L = al._L
        res = al.align_batch_raw(buf, offs)
        try:
            n = L.mgb_results_num_alignments(res)
            rec = np.ctypeslib.as_array(ctypes.cast(L.mgb_results_alignments(res), ctypes.POINTER(ctypes.c_uint8)),
                                        shape=(n * ctypes.sizeof(_lib.mgb_alignment_t),)).view(
                np.dtype({"names": list(D.FIELDS), "formats": ["<u4", "u1", "<i4", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4"],
                          "offsets": [0, 4, 8, 12, 16, 20, 24, 28, 32], "itemsize": ctypes.sizeof(_lib.mgb_alignment_t)}))
            st = al.stats_of(res)
            got = al.align_tensors(torch.from_numpy(buf).to(DEV), torch.from_numpy(offs.astype(np.int64)))
            for f in D.FIELDS:
                assert (getattr(got, f).cpu().numpy().astype(np.int64) == rec[f].astype(np.int64)).all(), f
            for c in D.COUNTERS:
                assert st[c] == got.stats[c], c
            alns = L.mgb_results_alignments(res)
            so, co = got.sequence_offsets.cpu().numpy(), got.cigar_offsets.cpu().numpy()
            sq, cg = got.sequence.cpu().numpy(), got.cigar.cpu().numpy()
            for i in np.random.default_rng(1).integers(0, n, min(n, sample)):
                x = alns[int(i)]
                assert sq[so[i]:so[i + 1]].tobytes() == ctypes.string_at(x.sequence, x.sequence_len)
                assert (cg[co[i]:co[i + 1]].astype(np.uint32)
                        == np.ctypeslib.as_array(x.cigar, shape=(x.num_cigar_ops,))).all()
            return n
        finally:
            al.free_raw(res)
    finally:
        idx.close()


def test_c2_shape_scale_gpu():
    """300 k error-free 150 bp reads past the first grid round, most answered by k_prepare_exact"""
    b = _bench()
    genome = b.make_genome(2_000_000)
    boss = BOSSTable.from_sequences(b.K, [genome.tobytes().decode()])
    buf, offs = b.make_reads(genome, 300_000, 42)
    cfg = cli_defaults(b.K, min_seed_length=b.K, max_seed_length=b.K, result_nodes=1)
    assert _scale_check(boss, cfg, buf, offs) >= 300_000


def test_c3_shape_scale_gpu():
    """C3's reads with 5 % errors against their genome"""
    b = _bench()
    genome = b.make_genome(2_000_000)
    boss = BOSSTable.from_sequences(b.K, [genome.tobytes().decode()])
    buf, offs = b.make_error_reads(genome, 0, 2, 0.05, 20_000)
    cfg = cli_defaults(b.K, min_exact_match=0.0, result_nodes=1)
    assert _scale_check(boss, cfg, buf, offs) > 0
