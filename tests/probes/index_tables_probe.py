"""The index tables of the C2 bench graph (bench.make_genome, k = 31), built on the device by the test library, against
the numpy restatement of tests/index_tables.py: the whole hash index, adjacency records, radj and path layout, and a
random sample of 2^20 entries of the deepest suffix-range level (s = 15, 8.6 GB). Not part of pytest: the host needs
tens of GB for the reference.

usage: python tests/probes/index_tables_probe.py [GENOME_BP]   (default 100 000 000, the C2 graph)"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import index_tables as IT  # noqa: E402
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex  # noqa: E402


def step(what, t0):
    print("%7.1f s  %s" % (time.time() - t0, what), flush=True)


def main():
    G = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
    k = 31
    t0 = time.time()
    genome = bench.make_genome(G)
    boss = BOSSTable.from_sequences(k, None, packed=(genome, np.array([0, G], dtype=np.uint64)), lib=IT.TABLES_LIB)
    step("BOSS table: %d edges" % boss.num_edges, t0)
    idx = DBGSuccinctIndex(boss, lib=IT.TABLES_LIB)
    step("index built on the device", t0)
    info = IT.index_info(idx)
    assert info.kh_slots and info.pl_n, "hash index / path layout not built (%s)" % IT.free_device_memory()
    T = IT.read_tables(idx, [n for n in IT.TABLES if n != "sfx"])
    entries = 4 ** info.sfx_len
    rng = np.random.default_rng(15)
    sample = np.unique(rng.integers(0, entries, 1 << 20))
    chunk = 1 << 26
    got = np.empty((len(sample), 2), np.uint32)
    for c0 in range(0, entries, chunk):
        sel = (sample >= c0) & (sample < c0 + chunk)
        if sel.any():
            part = IT.read_table(idx, "sfx", 2 * c0, 2 * min(chunk, entries - c0)).reshape(-1, 2)
            got[sel] = part[sample[sel] - c0]
    import torch
    card = torch.cuda.get_device_name(0)
    idx.close()
    t1 = time.time()
    step("tables copied to the host", t0)
    ref = IT.reference_for(boss, sfx_len=info.sfx_len)
    step("reference", t0)
    IT.check_radj(ref, T, info)
    IT.check_adj(ref, T, info, True)
    step("radj and adjacency records", t0)
    longest = IT.check_hash(ref, T, info)
    step("hash index", t0)
    paths, cycles = IT.check_paths(ref, T, info)
    step("path layout", t0)
    IT.check_sfx(ref, {"sfx": got.reshape(-1)}, info, sample=sample)
    print("index tables of a %d bp genome, k = %d, on %s: %d edges, %d keys, longest probe %d slots, %d paths, "
          "%d cycles cut, suffix ranges s = %d (%d of %d entries sampled): all contracts hold "
          "(device build + copy %.0f s, host check %.0f s)"
          % (G, k, card, ref.n, len(ref.K), longest, paths, cycles, info.sfx_len, len(sample), entries,
             t1 - t0, time.time() - t1))


if __name__ == "__main__":
    main()
