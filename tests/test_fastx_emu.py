"""The file route on the CPU: the host restatement of kseq_read against known answers and the golden files, chunked
parsing against one-piece parsing, the host emulation of the device parser against the restatement on a seeded corpus,
and mgb_align_fastx_text against mgb_align_batch_text on the emulation."""
import os
import subprocess

import numpy as np
import pytest

import fastx_common as F
import text_common as T
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
from metagraph_b200.config import cli_defaults
from test_oracle_golden import read_fastq

EX = os.path.join(F.GOLD, "example_graphs")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.fixture(scope="module")
def emu_index():
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(5, ["ACGTACGGTACCAGT"], lib=F.EMU), lib=F.EMU)
    yield idx
    idx.close()


@pytest.mark.parametrize("i", range(len(F.KNOWN)))
def test_host_known_answers(i):
    (data, at_eof, delim, fr), exp = F.KNOWN[i]
    headers, reads, consumed, ended, refused = F.records(data, at_eof, delim, fr)
    assert (headers, reads, consumed, ended) == exp
    assert not refused


def test_host_golden_files():
    names, reads = read_fastq(os.path.join(F.GOLD, "genome_MT1.fq"))
    h, r, consumed, ended, _ = F.records(open(os.path.join(F.GOLD, "genome_MT1.fq"), "rb").read())
    assert (h, r, ended) == ([n.split()[0].encode() for n in names], [x.encode() for x in reads], False)
    for path in [os.path.join(F.GOLD, "transcripts_1000.fa"), os.path.join(EX, "test_DNA_query.fa"),
                 os.path.join(EX, "test_Protein_query.fa")]:
        data = open(path, "rb").read()
        h, r, consumed, ended, _ = F.records(data)
        assert (h, r, consumed, ended) == (*F.read_fasta(path), len(data), False), path


def chunked(data, sizes, delim=None, fr=False, index=None):
    """the records of data parsed chunk by chunk: each call gets the rest of the last one plus the next piece"""
    heads, reads, pending, pos, i = [], [], b"", 0, 0
    while True:
        take = sizes[i % len(sizes)]
        i += 1
        pending += data[pos:pos + take]
        pos += take
        at_eof = pos >= len(data)
        h, r, consumed, ended, _ = F.records(pending, at_eof, delim, fr, index=index)
        heads += h
        reads += r
        if ended or at_eof:
            return heads, reads, ended
        pending = pending[consumed:]


@pytest.mark.parametrize("seed", range(6))
def test_chunk_invariance(seed, emu_index):
    rng = np.random.default_rng(seed)
    data = b"".join([open(os.path.join(F.GOLD, "genome_MT1.fq"), "rb").read(),
                     open(os.path.join(F.GOLD, "transcripts_100.fa"), "rb").read()])
    if seed % 2:
        data = data.replace(b"\n", b"\r\n")
    whole = F.records(data, True, "|", seed >= 3)[:2]
    sizes = [int(x) for x in rng.integers(1, 3000, 50)]
    # seeds 4, 5: the first buffer is smaller than the longest record, which takes several grown buffers
    if seed >= 4:
        sizes = [7] + sizes
    assert chunked(data, sizes, "|", seed >= 3) == (*whole, False)
    assert chunked(data, sizes, "|", seed >= 3, index=emu_index) == (*whole, False)


def test_emu_parser_vs_host(emu_index):
    texts = F.corpus()
    assert len(texts) >= 2000
    n_device = 0
    for t in texts:
        for at_eof in (True, False):
            for delim, fr in ((None, False), ("|", True)):
                host = F.records(t, at_eof, delim, fr)
                dev = F.records(t, at_eof, delim, fr, index=emu_index)
                assert dev[:4] == host[:4], (t, at_eof, delim, fr)
                assert dev[4] == (not F.parallel_form(t, at_eof)), (t, at_eof)
                n_device += not dev[4]
    # both routes are exercised
    assert 0.2 < n_device / (len(texts) * 4) < 0.9


def _fastx(names, reads, fastq):
    if fastq:
        return b"".join(b"@%s\n%s\n+\n%s\n" % (h, r, b"I" * len(r)) for h, r in zip(names, reads))
    return b"".join(b">%s\n%s\n" % (h, r) for h, r in zip(names, reads))


@pytest.mark.parametrize("json", [False, True])
def test_emu_align_fastx_text(json):
    idx, names, reads = T.mt_index(F.EMU)
    try:
        names = [n.encode() + b" comment %d" % i for i, n in enumerate(names)]
        reads = [r.encode() for r in reads]
        cfg = cli_defaults(11, min_exact_match=0.0)
        al = B200Aligner(idx, cfg)
        for fastq, delim, fr in ((True, None, False), (False, "|", False), (True, "|", True)):
            data = _fastx(names, reads, fastq)
            assert not F.records(data, True, delim, fr, index=idx)[4]         # the device route parses it
            h, r = F.records(data, True, delim, fr)[:2]                         # the expected text: host-parsed records
            exp = al.align_batch_text(list(zip(h, r)), json=json)
            got, consumed, ended = al.align_fastx_text(data, True, delim, fr, json)
            assert (got, consumed, ended) == (exp, len(data), False)
            assert al.last_stats["h2d_bytes"] >= len(data)
        # a refused chunk (multi-line FASTQ) takes the host restatement and gives the same bytes
        data = _fastx(names, reads, True).replace(b"\n+\n", b"\n+\n\n")
        assert F.records(data, True, None, False, index=idx)[4]
        h, r = F.records(data, True, None, False)[:2]
        assert r == reads
        got, consumed, _ = al.align_fastx_text(data, True, None, False, json)
        assert got == al.align_batch_text(list(zip(h, r)), json=json) and consumed == len(data)
    finally:
        idx.close()


@pytest.mark.parametrize("json,fwd_rev", [(False, False), (True, False), (False, True)])
def test_emu_pieces(json, fwd_rev, monkeypatch, capfd):
    F.pieces_case(F.EMU, json, fwd_rev, monkeypatch, capfd)
