"""Per-kernel device time of one call of bench.py's C2 workload (1 M x 150 bp reads, G = 100 Mbp, one piece, bench.py's
configuration: no node ids unless BENCH_RESULT_NODES=0), from a torch.profiler capture of the call, for each library
given (default: the product build). Prints, per library, the device-timed step (seed + align timers, mean of STEPS
calls without the profiler), then, for the capture with the median span, each kernel's, copy's and memset's device time
and the idle gap before it, and each kernel's total over all captures.
  python scripts/kernel_split.py [lib.so ...] [--trace-dir DIR]     (DIR: the chrome traces, one per library)
The graph is built once; each library uploads its own index."""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from torch.profiler import profile, ProfilerActivity
from bench import make_genome, make_reads, workload, K
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex


def gpu_line():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return "nvidia-smi not found"


def timeline(trace_path):
    """[(name, start_us, dur_us)] of the device work in a chrome trace, in start order"""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    out = [(e["name"].split("(")[0].split("<")[0], float(e["ts"]), float(e["dur"])) for e in ev
           if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    return sorted(out, key=lambda t: t[1])


def split(tl):
    """per-kernel time and the gaps: [(name, dur, gap_before)], span"""
    rows, end = [], None
    for name, ts, dur in tl:
        rows.append((name, dur, 0.0 if end is None else max(0.0, ts - end)))
        end = ts + dur if end is None else max(end, ts + dur)
    return rows, (end - tl[0][1]) if tl else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", default=[None])
    ap.add_argument("--trace-dir", default=None)
    ap.add_argument("--steps", type=int, default=int(os.environ.get("STEPS", 5)))
    ap.add_argument("--captures", type=int, default=int(os.environ.get("CAPTURES", 3)))
    args = ap.parse_args()
    wl = workload("c2", 1)
    G, N, cfg = wl["G"], wl["n_rank"], wl["cfg"]
    print("config c2 G %d reads %d result_nodes %d (%s); %s" % (G, N, cfg.result_nodes,
          "no node ids" if cfg.result_nodes else "node ids", gpu_line()), flush=True)
    genome = make_genome(G)
    buf, off = make_reads(genome, N, 42)
    boss = BOSSTable.from_sequences(K, None, packed=(genome, np.array([0, G], dtype=np.uint64)),
                                    threads=min(os.cpu_count() or 1, 32))
    tdir = args.trace_dir or tempfile.mkdtemp()
    os.makedirs(tdir, exist_ok=True)
    for lib in args.libs:
        tag = os.path.basename(lib) if lib else "libmgb.so"
        index = DBGSuccinctIndex(boss, lib=lib)
        al = B200Aligner(index, cfg)
        al.set_pipeline_pieces(1)
        for _ in range(2):
            al.free_raw(al.align_batch_raw(buf, off))
        st = []
        for _ in range(args.steps):
            res = al.align_batch_raw(buf, off); st.append(al.stats_of(res)); al.free_raw(res)
        seed = np.mean([s["seed_kernel_ms"] for s in st]); align = np.mean([s["align_kernel_ms"] for s in st])
        print("%s: step %.4f ms (seed %.4f align %.4f), %.1f M reads/s, launches %d, retried %d; index %.2f GB; %s"
              % (tag, seed + align, seed, align, N / (seed + align) / 1e3, st[-1]["kernel_launches"],
                 st[-1]["num_reads_retried"], index.device_bytes / 1e9, gpu_line()), flush=True)
        caps = []
        for c in range(args.captures):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                res = al.align_batch_raw(buf, off)
                torch.cuda.synchronize()
            al.free_raw(res)
            path = os.path.join(tdir, "%s.%d.pt.trace.json" % (tag, c))
            prof.export_chrome_trace(path)
            caps.append(split(timeline(path)))
        rows, span = sorted(caps, key=lambda x: x[1])[len(caps) // 2]
        print("  capture (median span of %d): span %.1f us" % (len(caps), span))
        for name, dur, gap in rows:
            print("    %-24s %9.1f us   gap before %7.1f us" % (name, dur, gap))
        tot = {}
        for name, dur, _ in rows:
            tot[name] = tot.get(name, 0.0) + dur
        print("  per kernel (all captures): " + ", ".join(
            "%s %.1f-%.1f us" % (n, min(sum(d for m, d, _ in r if m == n) for r, _ in caps),
                                 max(sum(d for m, d, _ in r if m == n) for r, _ in caps)) for n in tot), flush=True)
        del al
        index.close()


if __name__ == "__main__":
    main()
