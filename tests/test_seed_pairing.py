"""Both raw strands of every read mapped at once (mgb_map_to_nodes_strands): on graphs with the k-mer hash index a lane
walks a read's two strands together when exactly one of them starts in the graph, and skips the lookups of the other
strand's k-mers whose reverse complement the graph lacks. Node ids of both strands == the oracle's map_to_nodes of the
read and of its reverse complement, on graphs where reverse complements are absent, all present, or some present."""
import os
import subprocess

import numpy as np
import pytest

import index_tables as IT
import oracle_lib as O
import parity_common as P
from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
from test_oracle_golden import revcomp
from test_seed_hash_gpu import mixed_reads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_alphabet_pairing(tmp_path):
    """The walk's skip is sound only if, for a valid window on one strand, the mirrored window on the other strand is
    invalid or spells its reverse complement: checked over all 256 byte values with the library's own tables."""
    exe = str(tmp_path / "alphabet_pairing")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-DMGB_HOST_EMU", "-Wno-unknown-pragmas",
                           os.path.join(ROOT, "tests", "cpp", "alphabet_pairing.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "valid on both strands: 10" in out.stdout          # ACGTU, both cases


def random_seq(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def flip(c):
    return "ACGT"["ACGT".index(c) ^ 1]


def role_reads(rng, seqs, k):
    """reads whose first k-mers hit on strand 0 only, strand 1 only, both strands, neither strand"""
    reads = []
    for _ in range(40):
        s = seqs[int(rng.integers(0, len(seqs)))]
        p = int(rng.integers(0, len(s) - 200))
        q = int(rng.integers(0, len(s) - k))
        r = s[p:p + 150]
        reads.append(r)                                          # strand 0
        reads.append(revcomp(r))                                 # strand 1
        reads.append(r[:60] + revcomp(s[q:q + k]))               # both: the last k-mer is a reversed graph k-mer
        reads.append(flip(r[0]) + r[1:-1] + flip(r[-1]))         # neither
        reads.append(random_seq(rng, 3) + r[:50] + random_seq(rng, 3))      # neither, hits in the middle
        reads.append(r[:40] + "N" + r[41:90])                    # strand 0, an N in the middle
    return reads


def with_palindromes(rng, s, k, n):
    """s with n palindromic k-mers (k even: their reverse complement is themselves) planted at random places"""
    s = list(s)
    for _ in range(n):
        h = random_seq(rng, k // 2)
        p = int(rng.integers(0, len(s) - k))
        s[p:p + k] = list(h + revcomp(h))
    return "".join(s)


GRAPHS = ["absent", "all_present", "mixed", "k12_palindromes"]


@pytest.mark.gpu
@pytest.mark.parametrize("graph", GRAPHS)
def test_map_to_nodes_strands_gpu(graph):
    rng = np.random.default_rng(900 + GRAPHS.index(graph))
    k = 12 if graph == "k12_palindromes" else 31
    contigs = [random_seq(rng, 3000 + 500 * i) for i in range(8)]
    if graph == "k12_palindromes":
        contigs = [with_palindromes(rng, c, k, 20) for c in contigs]
    if graph == "all_present":
        graph_seqs = contigs + [revcomp(c) for c in contigs]
    elif graph == "mixed":
        graph_seqs = contigs + [revcomp(c) for c in contigs[::2]]
    else:
        graph_seqs = contigs
    g = O.OracleGraph(k, graph_seqs, mask=False)
    W, last, F, _ = g.arrays()
    boss = BOSSTable(k, W, last, F)
    idx = DBGSuccinctIndex(boss)
    IT.assert_hashed(idx, boss)
    reads = mixed_reads(rng, contigs, k, 1001) + role_reads(rng, contigs, k)
    fwd, rev = idx.map_to_nodes_strands(reads)
    idx.close()
    bad = [i for i, (r, f, b) in enumerate(zip(reads, fwd, rev))
           if list(f) != list(g.map_to_nodes(r)) or list(b) != list(g.map_to_nodes(revcomp(r)))]
    assert not bad, (len(bad), len(reads[bad[0]]), reads[bad[0]][:80])
