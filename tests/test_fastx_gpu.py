"""The file route on the H100: the sm_90a parser against the host restatement (the seeded corpus, and C2- and C3-shaped
FASTQ of 1 M records over several chunks), the reference's MT goldens through mgb_align_fastx_text, the whole command
against the oracle, long reads through the file route against mgb_align_batch_text, and a chunk aligned in three pieces
with the exact seeder (k_prepare_exact's word loads on the parsed reads) against mgb_align_batch_text."""
import os

import numpy as np
import pytest

import fastx_common as F
import text_common as T
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from test_oracle_golden import MT_BOTH, MT_FWD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev_index():
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(5, ["ACGTACGGTACCAGT"]), device=0)
    yield idx
    idx.close()


def test_device_parser_vs_host(dev_index):
    texts = F.corpus()
    n_device = 0
    for t in texts:
        for at_eof in (True, False):
            for delim, fr in ((None, False), ("|", True)):
                host = F.records(t, at_eof, delim, fr, lib=None)
                dev = F.records(t, at_eof, delim, fr, index=dev_index)
                assert dev[:4] == host[:4], (t, at_eof, delim, fr)
                assert dev[4] == (not F.parallel_form(t, at_eof)), (t, at_eof)
                n_device += not dev[4]
    assert n_device > len(texts)


def fastq_reads(n, L, seed, errors):
    """n reads of length L (C2: error-free, C3: 5 % substitutions) as 4-line FASTQ with comments on some headers"""
    rng = np.random.default_rng(seed)
    bases = np.frombuffer(b"ACGT", np.uint8)
    reads = bases[rng.integers(0, 4, (n, L))]
    if errors:
        hit = rng.random((n, L)) < errors
        reads[hit] = bases[rng.integers(0, 4, int(hit.sum()))]
    lines = []
    for i in range(n):
        r = reads[i].tobytes()
        lines.append(b"@read%d%s\n%s\n+\n%s\n" % (i, b" c=%d" % i if i % 3 == 0 else b"", r, b"F" * L))
    return b"".join(lines)


@pytest.mark.parametrize("shape", ["c2", "c3"])
def test_device_parser_large(shape, dev_index):
    data = fastq_reads(1_000_000, 150, 5 if shape == "c2" else 6, 0.0 if shape == "c2" else 0.05)
    chunk = 48 << 20 if shape == "c2" else 61 << 20          # records cross every chunk boundary
    pos, pending, n_dev, n_host, fr = 0, b"", 0, 0, shape == "c3"
    while True:
        pending += data[pos:pos + chunk]
        pos += chunk
        at_eof = pos >= len(data)
        dev = F.records(pending, at_eof, "|", fr, index=dev_index)
        host = F.records(pending, at_eof, "|", fr, lib=None)
        assert not dev[4] and dev[:4] == host[:4]
        n_dev += len(dev[1])
        if at_eof:
            break
        assert dev[2] < len(pending)
        pending = pending[dev[2]:]
    assert n_dev == (2 if fr else 1) * 1_000_000


def test_mt_goldens_file_route():
    idx, _, _ = T.mt_index(None)
    data = open(os.path.join(F.GOLD, "genome_MT1.fq"), "rb").read()
    try:
        for both, gold in ((False, MT_FWD), (True, MT_BOTH)):
            al = B200Aligner(idx, cli_defaults(11, min_exact_match=0.0, forward_and_reverse_complement=both))
            text, consumed, ended = al.align_fastx_text(data)
            assert (consumed, ended) == (len(data), False)
            assert text.decode().split("\n")[:5] == gold
        for gold_file, edit in (("genome_MT1.align.json", False), ("genome_MT1.align.edit.json", True)):
            al = B200Aligner(idx, cli_defaults(11, min_exact_match=0.0, edit_distance=edit))
            text, _, _ = al.align_fastx_text(data, json=True)
            gold = [l.rstrip() for l in open(os.path.join(F.GOLD, gold_file)) if l.strip()]
            assert text.decode().split("\n")[:5] == gold
    finally:
        idx.close()


def test_command_gpu(tmp_path):
    import test_cli_align as C
    C.command_case(tmp_path, None)


def test_long_reads_file_route():
    path = os.path.join(F.GOLD, "transcripts_1000.fa")
    data = open(path, "rb").read()
    names, reads = F.read_fasta(path)
    assert max(len(r) for r in reads) > 511
    genome = b"".join(reads[:200]).decode()
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(31, [genome]), device=0)
    try:
        al = B200Aligner(idx, cli_defaults(31))
        text, consumed, ended = al.align_fastx_text(data)
        assert (consumed, ended) == (len(data), False)
        assert text == al.align_batch_text(list(zip(names, reads)))
    finally:
        idx.close()


@pytest.mark.parametrize("json,fwd_rev", [(False, False), (True, False), (False, True)])
def test_pieces_gpu(json, fwd_rev, monkeypatch, capfd):
    F.pieces_case(None, json, fwd_rev, monkeypatch, capfd)
