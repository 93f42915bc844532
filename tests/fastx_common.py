"""Cases of the file route (mgb_align_fastx_text, mgb_fastx_parse): known answers of the kseq_read restatement, a seeded
corpus of mutated FASTA/FASTQ texts, and a Python statement of the two forms the device parses in parallel."""
import os

import numpy as np

from metagraph_b200.aligner import parse_fastx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")

# (bytes, at_eof, comment delimiter, --fwd-and-reverse) -> (headers, reads, consumed, ended)
KNOWN = [
    # bytes before the first record are skipped byte by byte, even within a line
    ((b"junk\nxx>r1\nAC\n", True, None, False), ([b"r1"], [b"AC"], 14, False)),
    ((b"no record here\n", True, None, False), ([], [], 15, False)),
    # the name ends at the first isspace byte; it can be empty
    ((b">\nAC\n>\tc\nG\n", True, None, False), ([b"", b""], [b"AC", b"G"], 11, False)),
    # comments: printed only with a delimiter; an empty name leaves the comment alone (utils::join_strings)
    ((b">r1 some comment\nAC\n", True, None, False), ([b"r1"], [b"AC"], 20, False)),
    ((b">r1 some comment\nAC\n", True, "|", False), ([b"r1|some comment"], [b"AC"], 20, False)),
    ((b"> lone\nAC\n>r2 \nG\n", True, "|", False), ([b"lone", b"r2"], [b"AC", b"G"], 17, False)),
    ((b">r1\tx y\nAC\n", True, "", False), ([b"r1x y"], [b"AC"], 11, False)),
    # empty lines add nothing; sequence lines are concatenated
    ((b">r1\n\nAC\n\nGT\n\n>r2\n", True, None, False), ([b"r1", b"r2"], [b"ACGT", b""], 17, False)),
    # '@' at the start of a FASTA line starts a record, '+' makes the record FASTQ
    ((b">r1\nAC\n@r2\nGG\n", True, None, False), ([b"r1", b"r2"], [b"AC", b"GG"], 14, False)),
    ((b">r1\nAC\n+\nII\n>r2\nT\n", True, None, False), ([b"r1", b"r2"], [b"AC", b"T"], 18, False)),
    # multi-line FASTQ: quality lines are read until there are as many bytes as in the sequence
    ((b"@r1\nAC\nGT\n+x\nII\nII\n@r2\nA\n+\n@\n", True, None, False), ([b"r1", b"r2"], [b"ACGT", b"A"], 29, False)),
    # a quality line that starts with '@' or '+' is quality
    ((b"@r1\nAC\n+\n@+\n@r2\nG\n+\n+\n", True, None, False), ([b"r1", b"r2"], [b"AC", b"G"], 22, False)),
    # kseq_read's -2 ends the file there: quality too long, too short at the end, no quality line
    ((b"@r1\nAC\n+\nII\n@r2\nAC\n+\nIII\n@r3\nA\n+\nI\n", True, None, False), ([b"r1"], [b"AC"], 12, True)),
    ((b"@r1\nAC\n+\nII\n@r2\nACG\n+\nII\n", True, None, False), ([b"r1"], [b"AC"], 12, True)),
    ((b"@r1\nAC\n+\nII\n@r2\nAC\n+", True, None, False), ([b"r1"], [b"AC"], 12, True)),
    # truncation: a header byte at the end has no name (kseq_read returns -1); a record without '\n' at the end
    ((b">r1\nAC\n>", True, None, False), ([b"r1"], [b"AC"], 8, False)),
    ((b">r1\nAC", True, None, False), ([b"r1"], [b"AC"], 6, False)),
    ((b">r1 c", True, "|", False), ([b"r1|c"], [b""], 5, False)),
    # an empty FASTQ sequence takes one quality line, empty or not; at the end of the input it needs none
    ((b"@r1\n+\n\n@r2\n+\n", True, None, False), ([b"r1", b"r2"], [b"", b""], 13, False)),
    # chunks that end before the input does: only complete records, consumed = where the next chunk starts
    ((b">r1\nAC\n>r2\nGT\n", False, None, False), ([b"r1"], [b"AC"], 7, False)),
    ((b"@r1\nAC\n+\nII\n@r2\nGT\n+\nI", False, None, False), ([b"r1"], [b"AC"], 12, False)),
    ((b"@r1\nAC\n+\nII\n@r2\nGT\n+\nIII\n", False, None, False), ([b"r1"], [b"AC"], 12, True)),
    ((b">r1 comm", False, None, False), ([], [], 0, False)),
    # CR rule: one '\r' before a line's end is dropped (names end at it anyway)
    ((b">r1\r\nAC\r\nGT\r\n>r2 c\r\n\r\nA\r", True, "|", False), ([b"r1", b"r2|c"], [b"ACGT", b"A"], 24, False)),
    ((b"@r1\r\nACG\r\n+\r\nIII\r\n", True, None, False), ([b"r1"], [b"ACG"], 18, False)),
    # --fwd-and-reverse: the same header again with the reverse complement (IUPAC pairs, case kept, others as is)
    ((b">r1 c\nACGTN\n@r2\nacgtRYKMBVDHU*\n", True, "_", True),
     ([b"r1_c", b"r1_c", b"r2", b"r2"], [b"ACGTN", b"NACGT", b"acgtRYKMBVDHU*", b"*ADHBVKMRYacgt"], 31, False)),
]


def records(data, at_eof=True, delim=None, fwd_rev=False, index=None, lib=EMU):
    return parse_fastx(data, at_eof, delim, fwd_rev, index=index, lib=lib)


def parallel_form(data, at_eof):
    """True when the chunk has the FASTA form or the 4-line FASTQ form (fastx_core.cuh) and so is parsed on the
    device; mirrors the statement of the two forms, not the kernels"""
    if not data:
        return True
    lines = data.split(b"\n")
    partial = lines[-1] != b""
    if not partial:
        lines = lines[:-1]
    n_complete = len(lines) if (at_eof or not partial) else len(lines) - 1

    def clen(ln):
        return len(ln) - 1 if ln.endswith(b"\r") else len(ln)

    fasta = lines[0][:1] in (b">", b"@") and all(not l.startswith(b"+") for l in lines[:n_complete])
    if at_eof and partial and lines[-1] in (b">", b"@"):
        fasta = False
    if fasta:
        return True
    if at_eof and n_complete % 4:
        return False
    for i, l in enumerate(lines[:n_complete]):
        r = i % 4
        if r == 0 and not l.startswith(b"@"):
            return False
        if r == 1 and (not clen(l) or l[:1] in (b">", b"@", b"+")):
            return False
        if r == 2 and not l.startswith(b"+"):
            return False
        if r == 3 and clen(l) != clen(lines[i - 2]):
            return False
    return True


def _record(rng, fastq, nl, split=False):
    name = b"r%d" % rng.integers(0, 10 ** 6)
    if rng.random() < 0.3:
        name += b" " + bytes(rng.choice(list(b"abc xyz\t"), rng.integers(0, 8)).tolist())
    seq = bytes(rng.choice(list(b"ACGTNacgt"), rng.integers(0, 40)).tolist())
    if not fastq:
        parts, p = [], 0
        while p < len(seq):
            w = int(rng.integers(1, 20))
            parts.append(seq[p:p + w])
            p += w
        return b">" + name + nl + b"".join(x + nl for x in parts)
    qual = bytes(rng.choice(list(b"I@+#5"), len(seq)).tolist())
    if split:            # multi-line FASTQ: sequence and quality over two lines each
        h = len(seq) // 2
        return b"@" + name + nl + seq[:h] + nl + seq[h:] + nl + b"+ c" + nl + qual[:h] + nl + qual[h:] + nl
    return b"@" + name + nl + seq + nl + b"+" + nl + qual + nl


def mutate(rng, text):
    """one edit of a text: split or join lines, empty lines, CRLF, drop the final newline, truncate, stray bytes"""
    k = int(rng.integers(0, 8))
    if not text:
        return text
    p = int(rng.integers(0, len(text)))
    if k == 0:
        return text[:p] + b"\n" + text[p:]
    if k == 1:
        q = text.find(b"\n", p)
        return text if q < 0 else text[:q] + text[q + 1:]
    if k == 2:
        return text.replace(b"\n", b"\r\n")
    if k == 3:
        return text.rstrip(b"\n")
    if k == 4:
        return text[:p]
    if k == 5:
        return text[:p] + bytes([rng.choice(list(b">@+ \r"))]) + text[p:]
    if k == 6:
        q = text.find(b"\n", p)
        return text if q < 0 else text[:q + 1] + b"\n" + text[q + 1:]
    return text


def corpus(seed=11, n=2000):
    """n seeded texts: FASTA, 4-line FASTQ, multi-line FASTQ, mixed, each with 0-3 edits"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        nl = b"\r\n" if rng.random() < 0.15 else b"\n"
        kind = i % 4
        recs = [_record(rng, kind in (1, 2) or (kind == 3 and rng.random() < 0.5), nl, kind == 2)
                for _ in range(int(rng.integers(1, 8)))]
        text = b"".join(recs)
        for _ in range(int(rng.integers(0, 4))):
            text = mutate(rng, text)
        out.append(text)
    return out


def read_fasta(path):
    """(names up to the first whitespace, sequences)"""
    names, seqs = [], []
    for line in open(path, "rb"):
        line = line.rstrip(b"\n")
        if line.startswith(b">"):
            names.append(line[1:].split()[0] if line[1:].split() else b"")
            seqs.append(b"")
        elif line:
            seqs[-1] += line
    return names, seqs


def pieces_case(lib, json, fwd_rev, monkeypatch, capfd, k=31, n=3000, seed=17):
    """A chunk long enough to be aligned in three pieces (MGB_TEST_PIECES=3), of FASTQ reads whose lengths are not
    multiples of 16, so that every piece after the first starts inside a 16-byte word of the parsed reads, with the
    exact seeder (min = max seed length = k, no complexity filter), so that k_prepare_exact stages the reads with word
    loads. The file route's text equals mgb_align_batch_text's on the host-parsed records, and (MGB_DEBUG) the chunk
    ran in three pieces, each of which ran k_prepare_exact and answered reads in it on the device."""
    from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
    from metagraph_b200.config import cli_defaults
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    genome = acgt[rng.integers(0, 4, 40000)]
    comp = np.zeros(256, np.uint8)
    comp[list(b"ACGT")] = list(b"TGCA")
    recs = []
    for i in range(n):
        L = int(rng.integers(40, 180))
        L += L % 16 == 0
        p = int(rng.integers(0, len(genome) - L))
        r = genome[p:p + L].copy()
        if i % 4 == 0:
            r[int(rng.integers(0, L))] = acgt[int(rng.integers(0, 4))]
        if i % 2:
            r = comp[r][::-1]
        r = r.tobytes()
        recs.append(b"@q%d%s\n%s\n+\n%s\n" % (i, b" c%d" % i if i % 3 == 0 else b"", r, b"#" * len(r)))
    data = b"".join(recs)
    idx = DBGSuccinctIndex(BOSSTable.from_sequences(k, [genome.tobytes().decode()], lib=lib), lib=lib)
    try:
        al = B200Aligner(idx, cli_defaults(k, min_seed_length=k, max_seed_length=k))
        monkeypatch.setenv("MGB_TEST_PIECES", "3")
        h, r, _, _, _ = records(data, True, "|", fwd_rev, lib=lib)
        assert not records(data, True, "|", fwd_rev, index=idx)[4]
        exp = al.align_batch_text(list(zip(h, r)), json=json)
        assert exp.count(b"\n") >= len(r)
        got, consumed, ended = al.align_fastx_text(data, True, "|", fwd_rev, json)
        assert (consumed, ended) == (len(data), False)
        assert got == exp
        capfd.readouterr()
        monkeypatch.setenv("MGB_DEBUG", "1")
        got, _, _ = al.align_fastx_text(data, True, "|", fwd_rev, json)
        err = capfd.readouterr().err
        assert got == exp
        assert "3 pieces done" in err, err[-2000:]
        if lib is None:      # the host emulation builds no k-mer hash index, so k_prepare_exact runs on the device only
            answered = [int(l.split("answered ")[1].split(",")[0]) for l in err.splitlines()
                        if "k_prepare_exact answered" in l]
            assert len(answered) == 3 and min(answered) > 0, err[-2000:]
    finally:
        idx.close()
