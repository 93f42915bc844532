"""Compressed-input probe: the command's file route on a plain file, a gzip file and a BGZF file of the same reads.

  1. routes: 1 M reads per shape (C2 and C3, bench.py's generators; qualities drawn from a seeded distribution), written
     plain, as gzip level 6 (Python's gzip) and as BGZF level 6 (65 280 bytes of text per block, as bgzip writes). Four
     routes: plain, host gzip (the gzip file through Python's gzip, cli.route_of = "host"), device gzip (the same file
     on its own route) and BGZF. Each route is warmed up, then the four run alternately --repeats times, from the file
     on disk to TSV on disk with one worker (cli.align_file); the output files must be byte-identical. With more than
     one visible device the plain, device-gzip and BGZF files also run with every device once (`--devices all`).
  2. host gzip: Python's gzip.open(...).read(64 MiB) rate on this machine's CPU, over the gzip file.
  3. --profile (a run of its own): k_bgzf_inflate's device time over the BGZF file; the device time of every k_gzip_*
     kernel over the device-gzip route's stages (the command on the small index, so the alignment does not matter);
     and mgb_gzip_inflate's kernel time and speculation counts (sub-ranges, candidates found, confirmed) over the gzip
     file at several sub-range sizes. Times by torch.profiler, per 1 M reads and as GB/s of text.

Prints one JSON line per measurement with the card's name and power limit, read in the same run.

    python scripts/bgzf_probe.py [--reads 1000000] [--genome 100000000] [--repeats 3] [--profile] [--out F]
"""
import argparse
import gzip
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import bgzf_common as B  # noqa: E402
from metagraph_b200 import _lib, bgzf, cli  # noqa: E402
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, bgzf_inflate, gzip_inflate  # noqa: E402
from metagraph_b200.config import cli_defaults  # noqa: E402


def cards():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()
    except OSError:
        return None


def fastq(reads, seed):
    q = np.frombuffer(b"#,:FFFFFFF", np.uint8)
    quals = q[np.random.default_rng(seed).integers(0, len(q), reads.shape)]
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, reads[i].tobytes(), quals[i].tobytes()) for i in range(len(reads)))


def run_command(aligners, path, out_path, route=None):
    """the command's file route; route="host": the gzip file through Python's gzip"""
    orig = cli.route_of
    if route:
        cli.route_of = lambda p: route
    try:
        with open(out_path, "wb") as out:
            if len(aligners) == 1:
                cli.align_file(aligners[0], path, out)
            else:
                cli.align_file_workers(aligners, path, out)
    finally:
        cli.route_of = orig


GZIP_KERNELS = ("k_gzip_find", "k_gzip_decode", "k_gzip_window", "k_gzip_resolve", "k_gzip_crc")


def profile_gzip(index, path, n_reads, text_bytes):
    """the k_gzip_* kernels' device time over the command's stages of the gzip file (aligned on a small index), and
    mgb_gzip_inflate's over the whole file at several sub-range sizes, with its speculation counts"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    al = [B200Aligner(index, cli_defaults(11))]
    out = path + ".tsv"
    run_command(al, path, out)                           # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_command(al, path, out)
    ka = prof.key_averages()
    per = {k: sum(e.device_time_total for e in ka if k in e.key) / 1e3 for k in GZIP_KERNELS}
    total = sum(per.values())
    os.remove(out)
    r = {"command_kernel_ms_per_1M_reads": {k: v * 1e6 / n_reads for k, v in per.items()},
         "command_total_ms_per_1M_reads": total * 1e6 / n_reads, "command_text_GB_per_s": text_bytes / (total * 1e-3) / 1e9}
    data = open(path, "rb").read()
    subs = {}
    for sub in (8192, 16384, 32768, 65536):
        gzip_inflate(index, data, sub_bytes=sub)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            text, _, refused, counts = gzip_inflate(index, data, sub_bytes=sub)
        ka = prof.key_averages()
        ms = {k: sum(e.device_time_total for e in ka if k in e.key) / 1e3 for k in GZIP_KERNELS}
        subs[sub] = {"kernel_ms": ms, "total_ms_per_1M_reads": sum(ms.values()) * 1e6 / n_reads, "refused": refused,
                     "text_ok": len(text) == text_bytes, "sub_ranges": counts[0], "found": counts[1],
                     "confirmed": counts[2]}
    r["inflate_by_sub_bytes"] = subs
    return r


def profile_inflate(index, path, n_reads):
    """k_bgzf_inflate's device time over the file, in pieces of the blocks of about 64 MiB of text"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    data = open(path, "rb").read()
    pieces, at = [], 0
    while at < len(data):
        start, text = at, 0
        while at < len(data) and text < cli.CHUNK_BYTES:
            size, isize = bgzf.block(data, at)
            at += size
            text += isize
        pieces.append(data[start:at])
    bgzf_inflate(index, pieces[0])                       # warm-up
    torch.cuda.synchronize()
    text_bytes = 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for p in pieces:
            text_bytes += len(bgzf_inflate(index, p)[0])
    us = sum(e.device_time_total for e in prof.key_averages() if "k_bgzf_inflate" in e.key)
    return {"kernel_ms_per_1M_reads": us / 1e3 * 1e6 / n_reads, "text_GB_per_s": text_bytes / (us * 1e-6) / 1e9,
            "text_bytes": text_bytes, "kernel_ms": us / 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="only k_bgzf_inflate's device time, no routes timed")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = cards()
    n_dev = _lib.load_library().mgb_device_count()
    if not n_dev:
        raise SystemExit("no CUDA device: this probe measures on the GPU only")
    results = []

    def report(r):
        r["cards"] = card
        print(json.dumps(r), flush=True)
        results.append(r)

    n, L = args.reads, bench.READ_LEN
    genome = bench.make_genome(args.genome)
    shapes = {
        "c2": (bench.make_reads(genome, n, 42)[0], cli_defaults(31, min_seed_length=31, max_seed_length=31)),
        "c3": (bench.make_error_reads(genome, 0, (n + bench.CHUNK - 1) // bench.CHUNK)[0][:n * L],
               cli_defaults(31, min_exact_match=0.0)),
    }
    boss = None if args.profile else BOSSTable.from_sequences(31, [genome.tobytes().decode()])
    index = DBGSuccinctIndex(boss if boss else BOSSTable.from_sequences(11, ["ACGTACGTTGCAGGCATTACG"]), device=0)
    replicas = [index] + [index.replicate(d) for d in range(1, n_dev)] if not args.profile else [index]
    tmp = tempfile.mkdtemp()
    try:
        for shape, (buf, cfg) in shapes.items():
            text = fastq(buf.reshape(n, L), 7)
            paths = {"plain": os.path.join(tmp, shape + ".fq"), "gzip": os.path.join(tmp, shape + ".fq.gz"),
                     "bgzf": os.path.join(tmp, shape + ".bgzf.fq.gz")}
            open(paths["plain"], "wb").write(text)
            open(paths["bgzf"], "wb").write(B.write(text, 65280, 6))
            with gzip.open(paths["gzip"], "wb", compresslevel=6) as f:
                f.write(text)
            if args.profile:
                report({"measure": "k_bgzf_inflate", "shape": shape, "reads": n,
                        **profile_inflate(index, paths["bgzf"], n)})
                report({"measure": "k_gzip", "shape": shape, "reads": n,
                        **profile_gzip(index, paths["gzip"], n, len(text))})
                continue
            ratios = {k: len(text) / os.path.getsize(p) for k, p in paths.items()}
            routes = {"plain": (paths["plain"], None), "host_gzip": (paths["gzip"], "host"),
                      "gzip": (paths["gzip"], None), "bgzf": (paths["bgzf"], None)}
            # Python's gzip on this host's CPU
            t = time.perf_counter()
            with gzip.open(paths["gzip"], "rb") as f:
                while f.read(64 << 20):
                    pass
            gz_s = time.perf_counter() - t
            report({"measure": "host_gzip", "shape": shape, "text_bytes": len(text), "seconds": gz_s,
                    "MB_per_s": len(text) / gz_s / 1e6, "M_reads_per_s": n / gz_s / 1e6})
            al = [B200Aligner(index, cfg)]
            outs = {k: os.path.join(tmp, "%s.%s.tsv" % (shape, k)) for k in routes}
            for k, (p, route) in routes.items():                              # warm-up of every route
                run_command(al, p, outs[k], route)
            times = {k: [] for k in routes}
            for _ in range(args.repeats):
                for k, (p, route) in routes.items():
                    t = time.perf_counter()
                    run_command(al, p, outs[k], route)
                    times[k].append(time.perf_counter() - t)
            same = len({open(p, "rb").read() for p in outs.values()}) == 1
            med = {k: statistics.median(v) for k, v in times.items()}
            report({"measure": "routes", "shape": shape, "reads": n, "text_bytes": len(text), "ratio": ratios,
                    "outputs_equal": same, "M_reads_per_s_median": {k: n / v / 1e6 for k, v in med.items()},
                    "seconds": times})
            if n_dev > 1:
                al_all = [B200Aligner(r, cfg) for r in replicas]
                t_all = {}
                for k in ("plain", "gzip", "bgzf"):
                    run_command(al_all, paths[k], outs[k])
                    t = time.perf_counter()
                    run_command(al_all, paths[k], outs[k])
                    t_all[k] = time.perf_counter() - t
                same = len({open(outs[k], "rb").read() for k in ("plain", "gzip", "bgzf")}) == 1
                report({"measure": "routes_all_devices", "shape": shape, "devices": n_dev, "outputs_equal": same,
                        "M_reads_per_s": {k: n / v / 1e6 for k, v in t_all.items()}})
            for p in list(paths.values()) + list(outs.values()):
                os.remove(p)
    finally:
        for r in replicas:
            r.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
