"""Times the device-resident route (B200Aligner.align_tensors: reads in HBM, columns written into torch tensors on the
device) against the record route (align_batch_raw: reads from pinned host buffers, records unpacked on the host) over
the same reads, on bench.py's C2 and C3 shapes at reduced size, and checks that both give the same score sum.

    python scripts/device_results_probe.py [--reads-c2 N] [--reads-c3 N] [--genome G] [--steps S] [--warmup W]

Prints the card's name and power limit, then one JSON line per shape with the median time per 1 M reads of each route.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex  # noqa: E402
from metagraph_b200.config import cli_defaults  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome", type=int, default=20_000_000)
    ap.add_argument("--reads-c2", type=int, default=1_000_000)
    ap.add_argument("--reads-c3", type=int, default=500_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card: %s" % card, flush=True)
    genome = bench.make_genome(args.genome)
    boss = BOSSTable.from_sequences(bench.K, [genome.tobytes().decode()])
    idx = DBGSuccinctIndex(boss, device=0)
    shapes = {
        "c2": (bench.make_reads(genome, args.reads_c2, 42),
               cli_defaults(bench.K, min_seed_length=bench.K, max_seed_length=bench.K, result_nodes=1)),
        "c3": (bench.make_error_reads(genome, 0, max(1, args.reads_c3 // 50_000), 0.05, 50_000),
               cli_defaults(bench.K, min_exact_match=0.0, result_nodes=1)),
    }
    for name, ((buf, offs), cfg) in shapes.items():
        n = len(offs) - 1
        al = B200Aligner(idx, cfg)
        L = al._L
        hbuf = torch.from_numpy(buf).pin_memory()
        hoffs = torch.from_numpy(offs).pin_memory()
        hb, ho = hbuf.numpy(), hoffs.numpy()
        dreads = hbuf.to("cuda:0")
        doffs = torch.from_numpy(offs.astype(np.int64)).to("cuda:0")
        out = {}

        def device_route():
            out["dev"] = al.align_tensors(dreads, doffs)

        def record_route():
            res = al.align_batch_raw(hb, ho)
            try:
                k = L.mgb_results_num_alignments(res)
                a = L.mgb_results_alignments(res)
                rec = np.ctypeslib.as_array(ctypes.cast(a, ctypes.POINTER(ctypes.c_int32)), shape=(k * 16,))
                out["rec_score"] = int(rec.reshape(k, 16)[:, 2].astype(np.int64).sum()) if k else 0
                out["rec_stats"] = al.stats_of(res)
            finally:
                al.free_raw(res)

        t_rec = timed(record_route, args.steps, args.warmup)
        t_dev = timed(device_route, args.steps, args.warmup)
        dev_score = int(out["dev"].score.to(torch.int64).sum())
        assert dev_score == out["rec_score"], (dev_score, out["rec_score"])
        st = out["dev"].stats
        print(json.dumps({
            "shape": name, "reads": n, "card": card,
            "device_ms_per_1M": round(t_dev * 1e3 * 1e6 / n, 2), "record_ms_per_1M": round(t_rec * 1e3 * 1e6 / n, 2),
            "device_M_reads_s": round(n / t_dev / 1e6, 2), "record_M_reads_s": round(n / t_rec / 1e6, 2),
            "score_sum": dev_score, "device_h2d_bytes": st["h2d_bytes"], "device_d2h_bytes": st["d2h_bytes"],
            "record_h2d_bytes": out["rec_stats"]["h2d_bytes"], "record_d2h_bytes": out["rec_stats"]["d2h_bytes"],
            "retried": st["num_reads_retried"]}), flush=True)
    idx.close()


if __name__ == "__main__":
    main()
