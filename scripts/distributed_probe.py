"""`metagraph_b200 align --distributed` against the single-process command on one device.

Writes bench.py's 1 M-read C2 and C3 FASTQ files and the graph of its 100 Mbp genome once, then, alternating, for
--repeats rounds: the single-process file route (cli.align_file, what `--devices 0` runs), torchrun with 1 rank and
torchrun with 2 ranks on the same device (cli.align_file_distributed over gloo). Each run loads the saved graph and
builds its index (untimed), aligns each file once to warm up, then once timed: from a barrier to rank 0's last write.
The outputs must be byte-identical. Prints one JSON line per measurement with the cards' names and power limits, read
in the same run. More than one device, and more than one host, are not measured here.

    python scripts/distributed_probe.py [--reads 1000000] [--genome 100000000] [--repeats 3] [--out F]
"""
import argparse
import hashlib
import json
import os
import shutil
import socket
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SHAPES = {"c2": ["--align-min-seed-length", "31", "--align-max-seed-length", "31"],
          "c3": ["--align-min-exact-match", "0"]}


def cards():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()
    except OSError:
        return None


def worker(tmp, distributed):
    """one run: the index on this rank's device, each shape aligned once to warm up and once timed"""
    import numpy as np
    from metagraph_b200 import _lib, cli
    from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
    z = np.load(os.path.join(tmp, "graph.npz"))
    boss = BOSSTable(int(z["k"]), z["W"], z["last"], z["F"])
    rank, device = 0, 0
    if distributed:
        import torch.distributed as dist
        dist.init_process_group("gloo")
        rank = dist.get_rank()
        device = int(os.environ["LOCAL_RANK"]) % _lib.load_library().mgb_device_count()
    index = DBGSuccinctIndex(boss, device=device)
    res = {}
    try:
        for shape, argv in SHAPES.items():
            args = cli.parse_args(["-i", "graph.dbg"] + argv + ["x.fq"])
            al = B200Aligner(index, cli.config_of(args, boss.k, "dna"))
            path = os.path.join(tmp, shape + ".fq")
            out_path = os.path.join(tmp, "%s.%s.tsv" % (shape, "dist" if distributed else "single"))
            for timed in (False, True):
                if distributed:
                    dist.barrier()
                t = time.perf_counter()
                with open(out_path, "wb") if rank == 0 else open(os.devnull, "wb") as out:
                    if distributed:
                        cli.align_file_distributed(al, path, out if rank == 0 else None)
                    else:
                        cli.align_file(al, path, out)
                if timed:
                    res[shape] = time.perf_counter() - t
            if rank == 0:
                res[shape + "_sha1"] = hashlib.sha1(open(out_path, "rb").read()).hexdigest()
    finally:
        index.close()
        if distributed:
            dist.destroy_process_group()
    if rank == 0:
        print("RESULT " + json.dumps(res), flush=True)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run(tmp, mode):
    env = dict(os.environ, OMP_NUM_THREADS="1", MASTER_ADDR="127.0.0.1")
    env["CUDA_VISIBLE_DEVICES"] = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
    me = os.path.abspath(__file__)
    if mode == "single":
        cmd = [sys.executable, me, "--worker", tmp]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % int(mode[-1]),
               "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), me, "--worker", tmp, "--distributed"]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode:
        raise SystemExit("%s failed:\n%s" % (mode, r.stderr[-3000:]))
    return json.loads([x for x in r.stdout.splitlines() if x.startswith("RESULT ")][0][7:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome", type=int, default=100_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--distributed", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker, args.distributed)
    import numpy as np
    import bench
    from file_align_probe import write_fastq
    from metagraph_b200 import _lib
    from metagraph_b200.aligner import BOSSTable
    card = cards()
    if not _lib.load_library().mgb_device_count():
        raise SystemExit("no CUDA device: this probe measures on the GPU only")
    n, L = args.reads, bench.READ_LEN
    genome = bench.make_genome(args.genome)
    tmp = tempfile.mkdtemp()
    try:
        boss = BOSSTable.from_sequences(31, None, packed=(genome, np.array([0, len(genome)], dtype=np.uint64)))
        np.savez(os.path.join(tmp, "graph.npz"), k=boss.k, W=boss.W, last=boss.last, F=np.asarray(boss.F))
        write_fastq(os.path.join(tmp, "c2.fq"), bench.make_reads(genome, n, 42)[0], n, L)
        write_fastq(os.path.join(tmp, "c3.fq"),
                    bench.make_error_reads(genome, 0, (n + bench.CHUNK - 1) // bench.CHUNK)[0][:n * L], n, L)
        modes = ["single", "torchrun1", "torchrun2"]
        times = {m: {s: [] for s in SHAPES} for m in modes}
        sums = {s: set() for s in SHAPES}
        for _ in range(args.repeats):
            for m in modes:
                r = run(tmp, m)
                for s in SHAPES:
                    times[m][s].append(r[s])
                    sums[s].add(r[s + "_sha1"])
        results = []
        for s in SHAPES:
            med = {m: statistics.median(times[m][s]) for m in modes}
            r = {"measure": "distributed", "shape": s, "reads": n, "outputs_equal": len(sums[s]) == 1,
                 "M_reads_per_s_median": {m: n / v / 1e6 for m, v in med.items()}, "seconds": {m: times[m][s]
                                                                                              for m in modes},
                 "cards": card}
            print(json.dumps(r), flush=True)
            results.append(r)
        if args.out:
            with open(args.out, "w") as f:
                json.dump(results, f, indent=1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
