"""k-mer seeding through the k-mer hash index (k <= 31 DNA graphs): node ids of every k-mer == the oracle's
map_to_nodes, on reads whose strands run side by side in one lane with different lengths and invalid characters."""
import numpy as np
import pytest

import index_tables as IT
import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from test_oracle_golden import revcomp

pytestmark = pytest.mark.gpu


def mixed_reads(rng, seqs, k, n):
    """n reads (n odd, so not a multiple of the strands a lane carries) of lengths below k, exactly k and several k up
    to 11 666 bp, with N characters at either end and in the middle, errors, reverse complements and random
    sequence that the graph does not have"""
    lens = [0, 1, k - 1, k, k + 1, 2 * k, 3 * k + 5, 150, 1000, 11666]
    reads = []
    for i in range(n):
        s = seqs[int(rng.integers(0, len(seqs)))]
        L = min(lens[int(rng.integers(0, len(lens)))], len(s))
        p = int(rng.integers(0, len(s) - L + 1))
        r = list(P.mutate(rng, s[p:p + L], float(rng.choice([0.0, 0.0, 0.01, 0.05]))))
        if i % 7 == 3:
            r = list("".join(np.array(list("ACGT"))[rng.integers(0, 4, len(r))]))
        if r and i % 5 == 1:
            r[0] = "N"
        if r and i % 5 == 2:
            r[-1] = "N"
        if len(r) > 2 and i % 3 == 0:
            for _ in range(int(rng.integers(1, 4))):
                r[int(rng.integers(0, len(r)))] = "N"
        r = "".join(r)
        reads.append(revcomp(r) if i % 2 else r)
    return reads


@pytest.mark.parametrize("k", [31, 12])
@pytest.mark.parametrize("primary", [False, True], ids=["one_strand", "two_strands"])
def test_hashed_map_to_nodes_gpu(k, primary):
    rng = np.random.default_rng(500 + k + primary)
    base = "".join(np.array(list("ACGT"))[rng.integers(0, 4, 14000)])
    seqs = [base, P.mutate(rng, base, 0.02)]
    graph_seqs = P.primary_contigs(seqs, k) if primary else seqs
    g = O.OracleGraph(k, graph_seqs, mask=False)
    if primary:
        g.set_mode(2)
    W, last, F, _ = g.arrays()
    boss = BOSSTable(k, W, last, F)
    idx = DBGSuccinctIndex(boss, mode=2 if primary else 0)
    IT.assert_hashed(idx, boss)
    reads = mixed_reads(rng, seqs, k, 1001)
    got = idx.map_to_nodes_sequentially(reads)
    bad = [i for i, (r, n) in enumerate(zip(reads, got)) if list(n) != list(g.map_to_nodes(r))]
    idx.close()
    assert not bad, (len(bad), len(reads[bad[0]]), reads[bad[0]][:80])
