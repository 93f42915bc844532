"""One bench-scale call of bench.py's C2 workload (BASELINE configs[1]: 1M x 150 bp reads, G = 100 Mbp, one piece) with
bench.py's own configuration (`workload("c2", 1)`: no node ids unless BENCH_RESULT_NODES=0), for probes and captures:
  MGB_DEBUG=1 MGB_LIB=metagraph_b200/_lib/libmgb_prep.so python scripts/profile_bench.py    (phase timers)
The numbers printed here are not bench values."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from bench import make_genome, make_reads, workload, K
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
wl = workload("c2", 1)
G = int(os.environ.get("G", wl["G"])); N = int(os.environ.get("N", wl["n_rank"]))
genome = make_genome(G)
boss = BOSSTable.from_sequences(K, None, packed=(genome, np.array([0, G], dtype=np.uint64)))
index = DBGSuccinctIndex(boss)
buf, off = make_reads(genome, N, 42)
al = B200Aligner(index, wl["cfg"])
al.set_pipeline_pieces(1)
res = al.align_batch_raw(buf, off); st = al.stats_of(res); al.free_raw(res)
print("config c2 G %d reads %d result_nodes %d (%s)" % (G, N, wl["cfg"].result_nodes,
      "no node ids" if wl["cfg"].result_nodes else "node ids"), flush=True)
print("seed_ms %.2f align_ms %.2f cols %d cells %d" % (st["seed_kernel_ms"], st["align_kernel_ms"], st["dp_columns"],
                                                      st["dp_cells"]), flush=True)
