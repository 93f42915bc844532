"""File route probe: FASTQ file to output file on one GPU, three routes timed in one run.

  1. device:  the command's route (cli.align_file -> mgb_align_fastx_text: bytes up, records parsed on the device)
  2. host:    the host restatement of kseq_read (mgb_fastx_parse, device_route = 0) + mgb_align_batch_text
  3. arrays:  mgb_align_batch_text on reads already packed in host memory (bench.py's end-to-end shape; no parse)

Shapes: C2 (bench.py make_reads, seed 42, error-free) and C3-like (bench.py make_error_reads, 5 % errors), 1 M 150 bp
reads each, against bench.py's 100 Mbp genome (k = 31), written as 4-line FASTQ. Prints one JSON line per shape with
the median reads/s per route, the parse's device time per 1 M reads by kernel, scans included (torch.profiler over the
parse alone, a separate run) and H2D bytes per read,
plus the card's name and power limit (and writes the list to --out if given).

    python scripts/file_align_probe.py [--reads 1000000] [--genome 100000000] [--repeats 3] [--out FILE] [--parse-only]
"""
import argparse
import ctypes
import json
import statistics
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from metagraph_b200 import _lib, cli  # noqa: E402
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, parse_fastx  # noqa: E402
from metagraph_b200.config import cli_defaults  # noqa: E402


def write_fastq(path, buf, n, L):
    reads = buf.reshape(n, L)
    with open(path, "wb") as f:
        for lo in range(0, n, 100000):
            f.write(b"".join(b"@r%d\n%s\n+\n%s\n" % (i, reads[i].tobytes(), b"F" * L)
                             for i in range(lo, min(n, lo + 100000))))


def route_host(al, path, out_path, chunk=cli.CHUNK_BYTES):
    """host restatement + mgb_align_batch_text, chunk by chunk; returns (reads, h2d bytes)"""
    L = al._L
    c = al.config.to_c()
    n_reads = h2d = 0
    with open(path, "rb") as f, open(out_path, "wb") as out:
        pending = b""
        while True:
            nxt = f.read(chunk)
            at_eof = not nxt
            pending += nxt
            if not pending:
                break
            arr = np.frombuffer(pending, np.uint8)
            max_rec = pending.count(b"@") + pending.count(b">") + 1
            seqs, names = np.empty(len(pending) + 1, np.uint8), np.empty(len(pending) + 1, np.uint8)
            offs, noffs = np.empty(max_rec + 1, np.uint64), np.empty(max_rec + 1, np.uint64)
            n, consumed, ended, refused = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int(), ctypes.c_int()
            _lib.check(L, L.mgb_fastx_parse(None, arr.ctypes.data, len(pending), int(at_eof), None, 0, 0,
                                            seqs.ctypes.data, len(seqs), offs.ctypes.data, names.ctypes.data,
                                            len(names), noffs.ctypes.data, max_rec, ctypes.byref(n),
                                            ctypes.byref(consumed), ctypes.byref(ended), ctypes.byref(refused)))
            res = ctypes.c_void_p()
            _lib.check(L, L.mgb_align_batch_text(al.graph.handle, ctypes.byref(c), seqs.ctypes.data, offs.ctypes.data,
                                                 names.ctypes.data, noffs.ctypes.data, n.value, _lib.MGB_TEXT_TSV,
                                                 ctypes.byref(res)))
            out.write(al.text_of(res))
            h2d += al.stats_of(res)["h2d_bytes"]
            al.free_raw(res)
            n_reads += n.value
            if at_eof or ended.value:
                break
            pending = pending[consumed.value:]
    return n_reads, h2d


def route_device(al, path, out_path):
    h2d = 0
    orig = al.align_fastx_text

    def counted(*a, **kw):
        nonlocal h2d
        r = orig(*a, **kw)
        h2d += al.last_stats["h2d_bytes"]
        return r
    al.align_fastx_text = counted
    try:
        with open(out_path, "wb") as out:
            cli.align_file(al, path, out)
    finally:
        al.align_fastx_text = orig
    return h2d


def route_arrays(al, buf, offs, names, noffs, out_path):
    res = al.align_batch_text_raw(buf, offs, names, noffs)
    with open(out_path, "wb") as out:
        out.write(al.text_of(res))
    h2d = al.stats_of(res)["h2d_bytes"]
    al.free_raw(res)
    return h2d


def parse_device_ms(index, path, chunk=cli.CHUNK_BYTES):
    """device time of the parse alone, by kernel: mgb_fastx_parse (device route) over the file's chunks under
    torch.profiler (CUDA activities), no alignment and no text. The scans (k_text_scan) are the parse's own here."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    data = open(path, "rb").read()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pos, pending = 0, b""
        while True:
            pending += data[pos:pos + chunk]
            pos += chunk
            at_eof = pos >= len(data)
            _, _, consumed, _, refused = parse_fastx(pending, at_eof, index=index)
            assert not refused
            if at_eof:
                break
            pending = pending[consumed:]
        torch.cuda.synchronize()
    by_kernel = {}
    for e in prof.key_averages():
        if "k_fastx" in e.key or "k_text_scan" in e.key:       # kernel names come with their signatures
            by_kernel[e.key] = (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
    return by_kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--parse-only", action="store_true", help="only the parse's device time, no routes timed")
    args = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = None
    genome = bench.make_genome(args.genome)
    t0 = time.time()
    boss = BOSSTable.from_sequences(31, [genome.tobytes().decode()])
    index = DBGSuccinctIndex(boss, device=0)
    print("graph built in %.1f s" % (time.time() - t0), file=sys.stderr)
    n, L = args.reads, bench.READ_LEN
    shapes = {
        "c2": (bench.make_reads(genome, n, 42)[0],
               cli_defaults(31, min_seed_length=31, max_seed_length=31, result_nodes=1)),
        "c3": (bench.make_error_reads(genome, 0, (n + bench.CHUNK - 1) // bench.CHUNK)[0][:n * L],
               cli_defaults(31, min_exact_match=0.0, result_nodes=1)),
    }
    results = []
    tmp = tempfile.mkdtemp()
    for shape, (buf, cfg) in shapes.items():
        path = os.path.join(tmp, shape + ".fq")
        write_fastq(path, buf, n, L)
        al = B200Aligner(index, cfg)
        offs = np.arange(n + 1, dtype=np.uint64) * L
        hdr = [b"r%d" % i for i in range(n)]
        names = np.frombuffer(b"".join(hdr), np.uint8)
        noffs = np.zeros(n + 1, np.uint64)
        noffs[1:] = np.cumsum([len(h) for h in hdr])
        outs = {r: os.path.join(tmp, "%s.%s.tsv" % (shape, r)) for r in ("device", "host", "arrays")}
        if args.parse_only:
            parse = {k: v * 1e6 / n for k, v in parse_device_ms(index, path).items()}
            r = {"shape": shape, "card": card, "reads": n, "parse_device_ms_per_1M_reads": sum(parse.values()),
                 "parse_device_ms_per_1M_reads_by_kernel": parse}
            print(json.dumps(r))
            results.append(r)
            continue
        # warm-up of every route, then alternate them
        route_device(al, path, outs["device"]); route_host(al, path, outs["host"])
        route_arrays(al, buf, offs, names, noffs, outs["arrays"])
        times = {r: [] for r in outs}
        h2d = {}
        for _ in range(args.repeats):
            t = time.perf_counter(); h2d["device"] = route_device(al, path, outs["device"])
            times["device"].append(time.perf_counter() - t)
            t = time.perf_counter(); h2d["host"] = route_host(al, path, outs["host"])[1]
            times["host"].append(time.perf_counter() - t)
            t = time.perf_counter(); h2d["arrays"] = route_arrays(al, buf, offs, names, noffs, outs["arrays"])
            times["arrays"].append(time.perf_counter() - t)
        same = len({open(p, "rb").read() for p in outs.values()}) == 1
        try:
            per_m = 1e6 / n
            parse = {k: v * per_m for k, v in parse_device_ms(index, path).items()}
        except Exception as e:  # the measurement is reported as missing, not estimated
            print("profiler: %s" % e, file=sys.stderr)
            parse = None
        med = {k: statistics.median(v) for k, v in times.items()}
        r = {"shape": shape, "card": card, "reads": n, "file_bytes": os.path.getsize(path), "outputs_equal": same,
             "reads_per_s_median": {k: n / v for k, v in med.items()},
             "seconds": {k: v for k, v in times.items()},
             "h2d_bytes_per_read": {k: v / n for k, v in h2d.items()},
             "parse_device_ms_per_1M_reads": None if parse is None else sum(parse.values()),
             "parse_device_ms_per_1M_reads_by_kernel": parse}
        print(json.dumps(r))
        results.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
