"""The short left-over list of bench.py's C2 workload (1 M x 150 bp error-free reads, G = 100 Mbp, bench.py's
configuration): which reads both whole-read gates leave to k_align and why, and what seeding and aligning them costs.

1. One call with MGB_DEBUG: the lines api.cu prints for each read left to k_align (at most 8), i.e. the reason.
2. A batch of only those reads, aligned twice with L2 cold (a buffer larger than L2 written between calls) and twice
   warm: k_seed_hash and k_align device times from torch.profiler. Cold minus warm bounds how much of each kernel is
   memory latency.
3. The sweep that sets k_seed_hash's short-list threshold: one substitution in n of the 1 M reads (n = 1, 32, 1 k, 8 k by
   default), so that about n reads are left over, then k_seed_hash's device time with the walk and with the short-list
   mode forced (MGB_TEST_SEED_MODE), median of CAPTURES captures.
  python scripts/tail_probe.py [--lens 1,32,1024,8192] [--captures 3]      (library: MGB_LIB or the product build)"""
import argparse, os, re, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np
import torch
from torch.profiler import profile, ProfilerActivity
from bench import make_genome, make_reads, workload, K, READ_LEN
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from kernel_split import gpu_line, timeline


def stderr_of(fn):
    """fn()'s result and what the library wrote to fd 2 meanwhile"""
    with tempfile.TemporaryFile() as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            out = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return out, f.read().decode(errors="replace")


def kernel_times(al, buf, off, cold=None):
    """{kernel: device us} of one call, from a torch.profiler capture; `cold`: a tensor rewritten first"""
    if cold is not None:
        cold.add_(1)
        torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = al.align_batch_raw(buf, off)
        torch.cuda.synchronize()
    al.free_raw(res)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "t.pt.trace.json")
        prof.export_chrome_trace(path)
        out = {}
        for name, _, dur in timeline(path):
            name = name.split("::")[-1]
            out[name] = out.get(name, 0.0) + dur
    return out


def with_env(name, value, fn):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value
    try:
        return fn()
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lens", default="1,32,1024,8192")
    ap.add_argument("--captures", type=int, default=3)
    args = ap.parse_args()
    wl = workload("c2", 1)
    G, N, cfg = wl["G"], wl["n_rank"], wl["cfg"]
    print("config c2 G %d reads %d result_nodes %d; %s" % (G, N, cfg.result_nodes, gpu_line()), flush=True)
    genome = make_genome(G)
    buf, off = make_reads(genome, N, 42)
    boss = BOSSTable.from_sequences(K, None, packed=(genome, np.array([0, G], dtype=np.uint64)),
                                    threads=min(os.cpu_count() or 1, 32))
    index = DBGSuccinctIndex(boss)
    al = B200Aligner(index, cfg)
    al.set_pipeline_pieces(1)
    for _ in range(2):
        al.free_raw(al.align_batch_raw(buf, off))

    # ---- 1. the reads left to k_align and why
    _, err = stderr_of(lambda: with_env("MGB_DEBUG", "1", lambda: al.free_raw(al.align_batch_raw(buf, off))))
    lines = [l for l in err.splitlines() if "left over" in l or "left to k_align" in l]
    print("\n".join(lines), flush=True)
    left = [int(m) for m in re.findall(r"left to k_align: read (\d+)", err)]
    print("left to k_align: %s" % left, flush=True)

    # ---- 2. a batch of only those reads, L2 cold and warm
    if left:
        tbuf = np.concatenate([buf[int(off[r]):int(off[r + 1])] for r in left])
        toff = np.arange(len(left) + 1, dtype=np.uint64) * READ_LEN
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")       # > the 50 MB L2
        for mode in (None, "walk", "wide"):
            rows = []
            for kind in ("cold", "cold", "warm", "warm"):
                t = with_env("MGB_TEST_SEED_MODE", mode,
                             lambda: kernel_times(al, tbuf, toff, cold=flush if kind == "cold" else None))
                rows.append("%s seed %.1f align %.1f" % (kind, t.get("k_seed_hash", 0.0), t.get("k_align", 0.0)))
            print("tail only, seed mode %s: %s us" % (mode or "picked", "; ".join(rows)), flush=True)
        del flush

    # ---- 3. k_seed_hash per mode against the length of the list
    rng = np.random.default_rng(9)
    for n in [int(x) for x in args.lens.split(",")]:
        ebuf = buf.copy()
        for r in rng.choice(N, n, replace=False):
            p = int(off[r]) + READ_LEN // 2
            ebuf[p] = ord("A") if ebuf[p] != ord("A") else ord("C")
        res = {}
        for mode in ("walk", "wide", None):
            caps = [with_env("MGB_TEST_SEED_MODE", mode, lambda: kernel_times(al, ebuf, off))
                    for _ in range(args.captures)]
            res[mode or "picked"] = sorted(c.get("k_seed_hash", 0.0) for c in caps)[len(caps) // 2]
            res["align_" + (mode or "picked")] = sorted(c.get("k_align", 0.0) for c in caps)[len(caps) // 2]
        print("left over ~%d: k_seed_hash walk %.1f us, wide %.1f us, picked %.1f us; k_align %.1f / %.1f / %.1f us"
              % (n, res["walk"], res["wide"], res["picked"], res["align_walk"], res["align_wide"], res["align_picked"]),
              flush=True)
    del al
    index.close()


if __name__ == "__main__":
    main()
