"""Read sharding across the GPUs of one box (SURVEY 8e): reads are independent units (dbg_aligner.cpp:263-354), the
index is replicated per HBM, there is no collective on the data path. Only the per-rank result sets travel: every
rank exports its results as one relocatable byte block (mgb_results_export: the records as the kernel packed
them), the sizes are all-gathered, the blocks go to rank 0 with point-to-point sends (NCCL over NVLink with device
tensors, gloo with CPU tensors in the CPU tests) and rank 0 rebuilds one result set per shard
(mgb_results_import) and emits them in input order. align_sharded_text gathers text instead: each rank renders its
shard on its own device and rank 0 concatenates the blocks (gather_blocks), which `align --distributed` uses too."""
import ctypes

import numpy as np

from . import _lib


def shard_range(n, rank, world):
    """contiguous range [n*rank/world, n*(rank+1)/world) of read indexes"""
    return (n * rank) // world, (n * (rank + 1)) // world


class ResultGather:
    """Gathers result sets on rank `dst`. Keeps its pinned staging buffers between calls."""

    def __init__(self, lib, device=None, dst=0):
        import torch
        self.L = lib
        self.dst = dst
        self.device = device if device is not None else torch.device("cpu")
        self.on_gpu = self.device.type == "cuda"
        self._send = None
        self._recv = {}

    def _host(self, cache, key, nbytes):
        import torch
        t = cache.get(key) if isinstance(cache, dict) else cache
        if t is None or t.numel() < nbytes:
            t = torch.empty(int(nbytes * 1.1) + 4096, dtype=torch.uint8, pin_memory=self.on_gpu)
            if isinstance(cache, dict):
                cache[key] = t
        return t

    def gather(self, res_handle, read_base):
        """res_handle: this rank's mgb_results_t*; read_base: index of the shard's first read in the whole batch.
        Returns on rank dst the list of (rank, imported results handle) in rank order (free each with
        mgb_results_free), elsewhere None."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        L = self.L
        nbytes = int(L.mgb_results_export_bytes(res_handle))
        self._send = self._host(self._send, None, nbytes)
        _lib.check(L, L.mgb_results_export(res_handle, self._send.data_ptr(), nbytes))
        meta = torch.tensor([nbytes, read_base], dtype=torch.int64, device=self.device)
        metas = [torch.zeros(2, dtype=torch.int64, device=self.device) for _ in range(world)]
        dist.all_gather(metas, meta)
        metas = [[int(x) for x in m.tolist()] for m in metas]
        if rank != self.dst:
            blk = self._send[:nbytes]
            blk = blk.to(self.device, non_blocking=True) if self.on_gpu else blk
            for q in dist.batch_isend_irecv([dist.P2POp(dist.isend, blk, self.dst)]):
                q.wait()
            return None
        out = []
        bufs = {}
        ops = []
        for r in range(world):
            if r == rank:
                continue
            bufs[r] = torch.empty(metas[r][0], dtype=torch.uint8, device=self.device)
            ops.append(dist.P2POp(dist.irecv, bufs[r], r))
        for q in (dist.batch_isend_irecv(ops) if ops else []):
            q.wait()
        for r in range(world):
            if r == rank:
                host, n = self._send, nbytes
            else:
                n = metas[r][0]
                host = self._host(self._recv, r, n)
                host[:n].copy_(bufs[r])
            h = ctypes.c_void_p()
            _lib.check(L, L.mgb_results_import(host.data_ptr(), n, metas[r][1], ctypes.byref(h)))
            out.append((r, h))
        return out


def gather_blocks(block, code=0, device=None, dst=0, tag=0):
    """Gathers one byte block per rank on rank `dst`, with one int (`code`) per rank that every rank learns: sizes and
    codes are all-gathered, and the blocks go to dst with point-to-point sends, as ResultGather sends its blocks
    (device: a CUDA device for NCCL, None for gloo with CPU tensors). Returns (codes, blocks): the codes in rank order
    on every rank, and on dst the blocks (bytes) in rank order, elsewhere None."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = device if device is not None else torch.device("cpu")
    meta = torch.tensor([len(block), code], dtype=torch.int64, device=dev)
    metas = [torch.zeros(2, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(metas, meta)
    metas = [[int(x) for x in m.tolist()] for m in metas]
    codes = [m[1] for m in metas]
    if rank != dst:
        if block:
            blk = torch.frombuffer(bytearray(block), dtype=torch.uint8).to(dev)
            for q in dist.batch_isend_irecv([dist.P2POp(dist.isend, blk, dst, tag=tag)]):
                q.wait()
        return codes, None
    bufs, ops = {}, []
    for r in range(world):
        if r != rank and metas[r][0]:
            bufs[r] = torch.empty(metas[r][0], dtype=torch.uint8, device=dev)
            ops.append(dist.P2POp(dist.irecv, bufs[r], r, tag=tag))
    for q in (dist.batch_isend_irecv(ops) if ops else []):
        q.wait()
    return codes, [bytes(block) if r == rank else bufs[r].cpu().numpy().tobytes() if r in bufs else b""
                   for r in range(world)]


def align_sharded(aligner, batch, format_fn, device=None):
    """Aligns this rank's shard of `batch` ([(header, seq)]) and gathers the results on rank 0, which formats them
    in input order with format_fn(header, AlignmentResults). Returns the list of entries on rank 0 (one per read,
    whatever format_fn returns -- multi-line strings included), None elsewhere."""
    import torch.distributed as dist
    from .aligner import _pack, results_of_handle
    rank, world = dist.get_rank(), dist.get_world_size()
    lo, hi = shard_range(len(batch), rank, world)
    mine = batch[lo:hi]
    buf, offsets = _pack([s for _, s in mine])
    res = aligner.align_batch_raw(buf, offsets)
    try:
        parts = ResultGather(aligner._L, device).gather(res, lo)
    finally:
        aligner.free_raw(res)
    if parts is None:
        return None
    out = []
    for r, h in parts:
        a, b = shard_range(len(batch), r, world)
        try:
            for (header, _), ar in zip(batch[a:b], results_of_handle(aligner._L, h, batch[a:b])):
                out.append(format_fn(header, ar))
        finally:
            aligner._L.mgb_results_free(h)
    return out


def align_sharded_text(aligner, batch, json=False, device=None):
    """What aligner.align_batch_text(batch, json) returns for the whole `batch` ([(header, seq)]), with the reads
    sharded across ranks: each rank renders its shard's TSV or JSON on its own device (mgb_align_batch_text) and rank 0
    gathers the text blocks (gather_blocks: NCCL with `device` a CUDA device, gloo with None). Returns the bytes on rank
    0, None elsewhere."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    lo, hi = shard_range(len(batch), rank, world)
    text = aligner.align_batch_text(batch[lo:hi], json) if hi > lo else b""
    _, blocks = gather_blocks(text, device=device)
    return None if blocks is None else b"".join(blocks)
