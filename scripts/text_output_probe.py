"""What the text route (mgb_align_batch_text) gains end to end: C2- and C3-shaped batches (bench.py's read generators and
configurations) timed from pinned host reads to the text in host memory, TSV and JSON, against mgb_align_batch with
records and no node ids (MGB_NODES_NONE); the host mirror's cost per line on a 10 k-read sample; bytes downloaded per
route; and the device time of k_text_size / k_text_scan / k_text_write from torch.profiler in a run of its own.
Prints the card and its power limit first, then one JSON line per measurement. G (genome bp, default 20 M) and N (reads,
default 1 M) come from the environment."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import K, make_error_reads, make_genome, make_reads  # noqa: E402
from metagraph_b200.aligner import (B200Aligner, BOSSTable, DBGSuccinctIndex, format_alignment,  # noqa: E402
                                    format_alignment_json, results_of_handle)
from metagraph_b200.config import cli_defaults  # noqa: E402

G = int(os.environ.get("G", 20_000_000))
N = int(os.environ.get("N", 1_000_000))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                   # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return out


def pinned(a, dtype):
    t = torch.empty(len(a), dtype=dtype, pin_memory=True)
    t.numpy()[:] = a
    return t


def emit(**kw):
    print(json.dumps(kw), flush=True)


def timed(fn, reps):
    fn()                                     # warm-up: workspaces, pinned pool
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def probe(shape, index, cfg, buf_np, off_np, reps):
    buf_t, off_t = pinned(buf_np, torch.uint8), pinned(off_np.astype(np.int64), torch.int64)
    buf, off = buf_t.numpy(), off_t.numpy().view(np.uint64)
    n = len(off) - 1
    names = np.frombuffer(b"".join(b"r%d" % i for i in range(n)), np.uint8).copy()
    noff = np.zeros(n + 1, np.uint64)
    noff[1:] = np.cumsum([len(b"r%d" % i) for i in range(n)])
    names_t, noff_t = pinned(names, torch.uint8), pinned(noff.astype(np.int64), torch.int64)
    hbuf, hoff = names_t.numpy(), noff_t.numpy().view(np.uint64)
    al = B200Aligner(index, cfg)
    L = al._L
    L.mgb_set_host_threads(os.cpu_count())

    def records():
        res = al.align_batch_raw(buf, off)
        st = al.stats_of(res)
        al.free_raw(res)
        return st

    def text(json_fmt):
        def run():
            res = al.align_batch_text_raw(buf, off, hbuf, hoff, json_fmt)
            st = al.stats_of(res)
            al.free_raw(res)
            return st
        return run

    out = {}
    for route, fn in (("records_nodes_none", records), ("text_tsv", text(False)), ("text_json", text(True))):
        ts = timed(fn, reps)
        st = fn()
        out[route] = np.median(ts)
        emit(shape=shape, route=route, reads=n, wall_ms=[round(t * 1e3, 2) for t in ts],
             median_ms=round(np.median(ts) * 1e3, 2), reads_per_s=round(n / np.median(ts)), d2h_bytes=st["d2h_bytes"],
             h2d_bytes=st["h2d_bytes"], d2h_bytes_per_read=round(st["d2h_bytes"] / n, 1))
    # the host mirror on a 10 k-read sample: records -> AlignmentResults -> lines
    m = min(10000, n)
    sub_off = off[:m + 1].copy()
    sub_buf = buf[:int(sub_off[-1])].copy()
    batch = [(b"r%d" % i, bytes(sub_buf[int(sub_off[i]):int(sub_off[i + 1])])) for i in range(m)]
    al_nodes = B200Aligner(index, cli_defaults(K, **{k: getattr(cfg, k) for k in ("min_seed_length", "max_seed_length",
                                                                                   "min_exact_match")}))
    res = al_nodes.align_batch_raw(sub_buf, sub_off)
    t0 = time.perf_counter()
    recs = results_of_handle(al_nodes._L, res, batch)
    t1 = time.perf_counter()
    tsv = [format_alignment(h.decode(), p, cfg.min_path_score) for (h, _), p in zip(batch, recs)]
    t2 = time.perf_counter()
    js = [format_alignment_json(h.decode(), p, K) for (h, _), p in zip(batch, recs)]
    t3 = time.perf_counter()
    al_nodes.free_raw(res)
    emit(shape=shape, route="python_mirror", reads=m, unpack_us_per_read=round((t1 - t0) / m * 1e6, 2),
         tsv_us_per_line=round((t2 - t1) / m * 1e6, 2), json_us_per_read=round((t3 - t2) / m * 1e6, 2),
         tsv_bytes_per_read=round(sum(len(x) + 1 for x in tsv) / m, 1),
         json_bytes_per_read=round(sum(len(x) + 1 for x in js) / m, 1))
    # device time of the text kernels, in a profiled run of its own
    for json_fmt in (False, True):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            text(json_fmt)()
        ker = {}
        for ev in prof.events():
            if "k_text" in ev.name:
                name = ev.name.split("k_text_")[1].split("(")[0].split("E")[0]
                ker["k_text_" + name] = ker.get("k_text_" + name, 0.0) + ev.device_time_total / 1e3
        emit(shape=shape, route="kernels_" + ("json" if json_fmt else "tsv"),
             device_ms={k: round(v, 3) for k, v in sorted(ker.items())})
    return out


def main():
    emit(card=card(), genome_bp=G, reads=N)
    genome = make_genome(G)
    boss = BOSSTable.from_sequences(K, None, packed=(genome, np.array([0, G], dtype=np.uint64)))
    index = DBGSuccinctIndex(boss)
    c2_buf, c2_off = make_reads(genome, N, 42)
    probe("C2", index, cli_defaults(K, min_seed_length=K, max_seed_length=K, result_nodes=1), c2_buf, c2_off, 3)
    del c2_buf, c2_off
    chunks = max(1, N // 250_000)
    c3_buf, c3_off = make_error_reads(genome, 0, chunks)
    probe("C3", index, cli_defaults(K, min_exact_match=0.0, result_nodes=1), c3_buf, c3_off, 2)
    index.close()


if __name__ == "__main__":
    main()
