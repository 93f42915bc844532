"""Multi-device probe: index replicas against builds, and `metagraph_b200 align --devices` against one worker.

  1. replicate: mgb_index_replicate of an index on device 0 to device 0 (and to every other visible device), timed
     against mgb_index_create of the same graph on device 0, alternating, on bench.py's 100 Mbp graph (--genome) and,
     with --genome-big, on a second graph.
  2. command: the command's file route (cli.align_file / cli.align_file_workers, the driver of `--devices`) on
     file_align_probe's 1 M-read C2 and C3 FASTQ files, with the worker lists `0`, `0,0` and every visible device once,
     alternating; the output files must be byte-identical.

Prints one JSON line per measurement with the card's name and power limit, read in the same run (and writes the list to
--out if given).

    python scripts/multi_device_probe.py [--reads 1000000] [--genome 100000000] [--genome-big 0] [--repeats 3] [--out F]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
from file_align_probe import write_fastq  # noqa: E402
from metagraph_b200 import _lib, cli  # noqa: E402
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex  # noqa: E402
from metagraph_b200.config import cli_defaults  # noqa: E402


def cards():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()
    except OSError:
        return None


def time_replicate(boss, n_dev, repeats):
    """seconds of mgb_index_create on device 0 and of mgb_index_replicate to each device, alternating"""
    src = DBGSuccinctIndex(boss, device=0)
    times = {"create": [], **{"replicate_to_%d" % d: [] for d in range(n_dev)}}
    try:
        for _ in range(repeats):
            t = time.perf_counter()
            DBGSuccinctIndex(boss, device=0).close()
            times["create"].append(time.perf_counter() - t)
            for d in range(n_dev):
                t = time.perf_counter()
                rep = src.replicate(d)
                times["replicate_to_%d" % d].append(time.perf_counter() - t)
                rep.close()
        return times, src.device_bytes
    finally:
        src.close()


def run_command(indexes, devices, cfg, path, out_path):
    aligners = [B200Aligner(indexes[d], cfg) for d in devices]
    with open(out_path, "wb") as out:
        if len(aligners) == 1:
            cli.align_file(aligners[0], path, out)
        else:
            cli.align_file_workers(aligners, path, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome", type=int, default=100_000_000)
    ap.add_argument("--genome-big", type=int, default=0, help="a second graph for the replicate timing (0: none)")
    ap.add_argument("--repeats", type=int, default=3)
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

    genome = bench.make_genome(args.genome)
    boss = BOSSTable.from_sequences(31, [genome.tobytes().decode()])
    for G, b in [(args.genome, boss)] + ([(args.genome_big, None)] if args.genome_big else []):
        if b is None:
            b = BOSSTable.from_sequences(31, [bench.make_genome(G).tobytes().decode()])
        times, dev_bytes = time_replicate(b, n_dev, args.repeats)
        report({"measure": "replicate", "genome": G, "edges": b.num_edges, "index_bytes": dev_bytes,
                "seconds_median": {k: statistics.median(v) for k, v in times.items()}, "seconds": times})
        del b

    indexes = {0: DBGSuccinctIndex(boss, device=0)}
    for d in range(1, n_dev):
        indexes[d] = indexes[0].replicate(d)
    lists = {"0": [0], "0,0": [0, 0]}
    if n_dev > 1:
        lists["all"] = list(range(n_dev))
    n, L = args.reads, bench.READ_LEN
    shapes = {
        "c2": (bench.make_reads(genome, n, 42)[0], cli_defaults(31, min_seed_length=31, max_seed_length=31)),
        "c3": (bench.make_error_reads(genome, 0, (n + bench.CHUNK - 1) // bench.CHUNK)[0][:n * L],
               cli_defaults(31, min_exact_match=0.0)),
    }
    tmp = tempfile.mkdtemp()
    try:
        for shape, (buf, cfg) in shapes.items():
            path = os.path.join(tmp, shape + ".fq")
            write_fastq(path, buf, n, L)
            outs = {k: os.path.join(tmp, "%s.%s.tsv" % (shape, k.replace(",", "_"))) for k in lists}
            for k, devs in lists.items():                                   # warm-up of every list
                run_command(indexes, devs, cfg, path, outs[k])
            times = {k: [] for k in lists}
            for _ in range(args.repeats):
                for k, devs in lists.items():
                    t = time.perf_counter()
                    run_command(indexes, devs, cfg, path, outs[k])
                    times[k].append(time.perf_counter() - t)
            same = len({open(p, "rb").read() for p in outs.values()}) == 1
            med = {k: statistics.median(v) for k, v in times.items()}
            report({"measure": "command", "shape": shape, "reads": n, "file_bytes": os.path.getsize(path),
                    "devices_visible": n_dev, "outputs_equal": same,
                    "reads_per_s_median": {k: n / v for k, v in med.items()}, "seconds": times})
            os.remove(path)
    finally:
        for ix in indexes.values():
            ix.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
