"""Cost of num_alternative_paths (--align-alternative-alignments N) on the device: C3-style reads (150 bp, 5 % substitutions,
half reverse-complemented, CLI defaults plus min_exact_match 0) against a graph with gene families (units of 400 bp in
20 copies diverged by 2-6 % between unique flanks, plus unique sequence). For N = 1, 4, 8, 32: device-timed reads/s
(seeding + k_align kernels, CUDA events, the batch as one piece as bench.py's `value`), k_align time, alignments
returned, and the arena bytes per warp and resident warps MGB_DEBUG prints. Prints one JSON line per N and a summary
line; --out FILE also writes the summary to FILE."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex, _pack   # noqa: E402
from metagraph_b200.config import cli_defaults                                       # noqa: E402

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = bytes.maketrans(b"ACGT", b"TGCA")


def graph(rng, families, copies, unit_len=400, flank=300, unique=2_000_000):
    seqs = []
    for _ in range(families):
        unit = rng.integers(0, 4, unit_len)
        for _ in range(copies):
            c = unit.copy()
            hit = rng.random(unit_len) < rng.uniform(0.02, 0.06)
            c[hit] = (c[hit] + rng.integers(1, 4, hit.sum())) % 4
            seqs.append(np.concatenate([rng.integers(0, 4, flank), c, rng.integers(0, 4, flank)]))
    seqs.append(rng.integers(0, 4, unique))
    return [ACGT[s].tobytes().decode() for s in seqs]


def reads(rng, seqs, n, L=150, rate=0.05):
    out = []
    for i in range(n):
        s = seqs[int(rng.integers(0, len(seqs) - 1))] if i % 2 else seqs[-1]
        p = int(rng.integers(0, len(s) - L))
        r = np.frombuffer(s[p:p + L].encode(), dtype=np.uint8).copy()
        hit = rng.random(L) < rate
        r[hit] = ACGT[rng.integers(0, 4, hit.sum())]
        b = r.tobytes()
        out.append(b.translate(COMP)[::-1].decode() if i % 3 == 0 else b.decode())
    return out


def debug_lines(aligner, buf, offsets):
    """one call with MGB_DEBUG set and stderr captured: the library reads the variable at every call"""
    os.environ["MGB_DEBUG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            aligner.free_raw(aligner.align_batch_raw(buf, offsets))
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["MGB_DEBUG"]
        f.seek(0)
        text = f.read()
    m = re.findall(r"k_align grid: (\d+) warps \((\d+) resident\), arena (\d+) bytes per warp", text)
    return [dict(grid_warps=int(a), resident_warps=int(b), arena_bytes_per_warp=int(c)) for a, b, c in m]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=200_000)
    ap.add_argument("--families", type=int, default=100)
    ap.add_argument("--copies", type=int, default=20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--n-alt", default="1,4,8,32")
    ap.add_argument("--out", default=None, help="also write the summary as JSON to this file")
    args = ap.parse_args()
    import torch
    rng = np.random.default_rng(2024)
    k = 31
    seqs = graph(rng, args.families, args.copies)
    rs = reads(rng, seqs, args.reads)
    index = DBGSuccinctIndex(BOSSTable.from_sequences(k, seqs), device=0)
    buf, offsets = _pack(rs)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = dict(gpu=smi, reads=args.reads, read_len=150, error_rate=0.05, k=k, families=args.families,
               copies=args.copies, graph_bp=sum(len(s) for s in seqs), runs=[])
    for n_alt in [int(x) for x in args.n_alt.split(",")]:
        cfg = cli_defaults(k, num_alternative_paths=n_alt, min_exact_match=0.0)
        al = B200Aligner(index, cfg)
        al.set_pipeline_pieces(1)
        al.free_raw(al.align_batch_raw(buf, offsets))          # warm-up
        dev_ms, align_ms, n_aln = [], [], 0
        for _ in range(args.steps):
            torch.cuda.synchronize()
            res = al.align_batch_raw(buf, offsets)
            st = al.stats_of(res)
            dev_ms.append(st["seed_kernel_ms"] + st["align_kernel_ms"])
            align_ms.append(st["align_kernel_ms"])
            n_aln = int(al._L.mgb_results_num_alignments(res))
            al.free_raw(res)
        dbg = debug_lines(al, buf, offsets)
        run = dict(n_alt=n_alt, device_ms=float(np.median(dev_ms)), k_align_ms=float(np.median(align_ms)),
                   reads_per_s=args.reads / (float(np.median(dev_ms)) / 1e3), alignments=n_aln, debug=dbg)
        out["runs"].append(run)
        print(json.dumps(run), flush=True)
    index.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
