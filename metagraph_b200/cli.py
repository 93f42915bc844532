"""`python -m metagraph_b200 align -i GRAPH.dbg [options] FILE...`: prints what `metagraph align` prints for the
FASTA/FASTQ files (plain, .gz or .bgz), aligned on one device (CUDA_VISIBLE_DEVICES picks it).

The files are read in chunks; each chunk is parsed, aligned and rendered by mgb_align_fastx_text, so only the file's
bytes go to the device and only the text comes back. A thread reads the next chunk while the device works on the
current one. Output is in input order, which is one of the orders the reference's thread pool can print.
"""
import argparse
import gzip
import os
import queue
import sys
import threading

from .config import SIZE_MAX, cli_defaults, dna_scoring_matrix

CHUNK_BYTES = 64 << 20

REFUSED = {  # options of `metagraph align` this command does not implement (DESIGN.md §7)
    "--map": "--map (k-mer mapping) is not implemented",
    "-a": "-a/--annotator (label-aware alignment) is not implemented",
    "--annotator": "-a/--annotator (label-aware alignment) is not implemented",
    "--align-chain": "--align-chain (seed chaining) is not implemented",
    "--align-post-chain": "--align-post-chain (post-alignment chaining) is not implemented",
}


class UsageError(Exception):
    pass


def _parser():
    p = argparse.ArgumentParser(prog="python -m metagraph_b200 align",
                                description="Align FASTA/FASTQ files to a de Bruijn graph as `metagraph align` does.")
    p.add_argument("-i", "--infile-base", dest="graph", required=True, help="graph (.dbg)")
    p.add_argument("files", nargs="+", metavar="FILE", help="FASTA/FASTQ files, plain or .gz/.bgz")
    p.add_argument("-o", "--outfile-base", dest="outfile", default=None,
                   help="output file; as in `metagraph align` it is reopened and truncated for every input file, so "
                        "it ends up with the output of the last one [stdout]")
    p.add_argument("--json", action="store_true", help="JSON records instead of TSV lines")
    p.add_argument("--fwd-and-reverse", action="store_true",
                   help="also align the reverse complement of each read, as a separate read under the same header")
    p.add_argument("--header-comment-delim", default=None, help="join the FASTA/FASTQ name and comment with this")
    p.add_argument("-p", "--parallel", type=int, default=1,
                   help="accepted for compatibility; changes no output (one device does the work)")
    p.add_argument("--batch-size", type=int, default=100000000,
                   help="accepted for compatibility; changes no output")
    p.add_argument("--align-only-forwards", action="store_true")
    p.add_argument("--align-edit-distance", action="store_true")
    p.add_argument("--align-no-seed-complexity-filter", action="store_true")
    p.add_argument("--align-match-score", type=int, default=2)
    p.add_argument("--align-mm-transition-penalty", type=int, default=3)
    p.add_argument("--align-mm-transversion-penalty", type=int, default=3)
    p.add_argument("--align-gap-open-penalty", type=int, default=6)
    p.add_argument("--align-gap-extension-penalty", type=int, default=2)
    p.add_argument("--align-end-bonus", type=int, default=5)
    p.add_argument("--align-alternative-alignments", type=int, default=1)
    p.add_argument("--align-min-path-score", type=int, default=0)
    p.add_argument("--align-xdrop", type=int, default=27)
    p.add_argument("--align-min-seed-length", type=int, default=19)
    p.add_argument("--align-max-seed-length", type=int, default=SIZE_MAX)
    p.add_argument("--align-max-num-seeds-per-locus", type=int, default=1000)
    p.add_argument("--align-max-nodes-per-seq-char", type=float, default=5.0)
    p.add_argument("--align-min-exact-match", type=float, default=0.7)
    p.add_argument("--align-max-ram", type=float, default=200.0)
    p.add_argument("--align-rel-score-cutoff", type=float, default=0.95)
    return p


def parse_args(argv):
    """the align arguments; UsageError for options the command refuses or values `metagraph align` rejects"""
    for a in argv:
        if a in REFUSED:
            raise UsageError(REFUSED[a])
    args = _parser().parse_args(argv)
    if args.outfile and args.outfile.endswith(".gfa"):
        raise UsageError("GFA output is not implemented")
    # config.cpp:532-564, 678-679
    if args.align_min_seed_length > args.align_max_seed_length:
        raise UsageError("min_seed_length must be <= max_seed_length")
    if min(args.align_mm_transition_penalty, args.align_mm_transversion_penalty, args.align_gap_open_penalty,
           args.align_gap_extension_penalty) < 0:
        raise UsageError("alignment penalties should be given as positive integers")
    if args.align_alternative_alignments == 0:
        raise UsageError("align-alternative-alignments must be > 0")
    return args


def config_of(args, k, alphabet):
    """the DBGAlignerConfig initialize_aligner_config (cli/align.cpp:33-69) builds from the arguments"""
    if alphabet not in ("dna", "protein"):
        raise UsageError("graphs over the %s alphabet are not supported" % alphabet)
    kw = dict(num_alternative_paths=args.align_alternative_alignments,
              min_seed_length=min(args.align_min_seed_length, k), max_seed_length=args.align_max_seed_length,
              max_num_seeds_per_locus=args.align_max_num_seeds_per_locus, min_path_score=args.align_min_path_score,
              xdrop=args.align_xdrop, min_exact_match=args.align_min_exact_match,
              max_nodes_per_seq_char=args.align_max_nodes_per_seq_char, max_ram_per_alignment=args.align_max_ram,
              rel_score_cutoff=args.align_rel_score_cutoff, gap_opening_penalty=-args.align_gap_open_penalty,
              gap_extension_penalty=-args.align_gap_extension_penalty,
              seed_complexity_filter=not args.align_no_seed_complexity_filter)
    if not args.align_edit_distance:        # set_scoring_matrix zeroes the end bonus for edit distance
        kw["left_end_bonus"] = kw["right_end_bonus"] = args.align_end_bonus
        if alphabet == "dna":
            kw["score_matrix"] = dna_scoring_matrix(args.align_match_score, -args.align_mm_transition_penalty,
                                                    -args.align_mm_transversion_penalty)
    if alphabet == "dna":                   # protein graphs have no reverse-complement strand
        kw["forward_and_reverse_complement"] = not args.align_only_forwards
    return cli_defaults(k, alphabet, args.align_edit_distance, **kw)


class _Chunks:
    """the file's bytes in chunks of `size`, read one chunk ahead on a thread; b"" at the end. close() stops the
    reader, so a file that ends at a malformed record is not read (or decompressed) to its end."""

    def __init__(self, f, size):
        self.q = queue.Queue(maxsize=1)
        self.stop = threading.Event()

        def reader():
            try:
                while not self.stop.is_set():
                    b = f.read(size)
                    while not self.stop.is_set():
                        try:
                            self.q.put(b, timeout=0.1)
                            break
                        except queue.Full:
                            pass
                    if not b:
                        return
            except BaseException as e:  # handed to the consumer
                self.q.put(e)

        self.t = threading.Thread(target=reader, daemon=True)
        self.t.start()

    def next(self):
        b = self.q.get()
        if isinstance(b, BaseException):
            raise b
        return b

    def close(self):
        self.stop.set()
        self.t.join()


def align_file(aligner, path, out, json=False, comment_delim=None, fwd_and_reverse=False, chunk_bytes=CHUNK_BYTES):
    """aligns one file and writes its text to `out`, chunk by chunk; returns the number of bytes written"""
    opener = gzip.open if path.endswith((".gz", ".bgz")) else open
    written = 0
    with opener(path, "rb") as f:
        chunks = _Chunks(f, chunk_bytes)
        try:
            pending, at_eof, want = b"", False, 0
            while True:
                # the rest of the last buffer, then at least one chunk; when the buffer held no complete record, as
                # many chunks as double it, so a record of n chunks is parsed O(log n) times, not n times
                while not at_eof:
                    nxt = chunks.next()
                    at_eof = not nxt
                    pending = pending + nxt if pending else nxt
                    if len(pending) >= want:
                        break
                if not pending:
                    break
                text, consumed, ended = aligner.align_fastx_text(pending, at_eof, comment_delim, fwd_and_reverse,
                                                                 json)
                out.write(text)
                written += len(text)
                if ended or at_eof:
                    break
                want = 2 * len(pending) if consumed == 0 else 0
                pending = pending[consumed:]
        finally:
            chunks.close()
    return written


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    if not argv or argv[0] != "align":
        sys.stderr.write("usage: python -m metagraph_b200 align -i GRAPH.dbg [options] FILE...\n")
        return 2
    try:
        args = parse_args(argv[1:])
        from .aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
        boss = BOSSTable.from_dbg(args.graph)
        alphabet = {0: "dna", 1: "protein"}.get(boss.alphabet, "code %d" % boss.alphabet)
        cfg = config_of(args, boss.k, alphabet)
    except UsageError as e:
        sys.stderr.write("error: %s\n" % e)
        return 1
    index = DBGSuccinctIndex(boss, device=0)
    aligner = B200Aligner(index, cfg)
    for path in args.files:
        if not os.path.exists(path):
            sys.stderr.write("ERROR: Cannot read from file %s\n" % path)
            return 1
        if args.outfile:
            with open(args.outfile, "wb") as out:       # reopened and truncated per input (cli/align.cpp:409-411)
                align_file(aligner, path, out, args.json, args.header_comment_delim, args.fwd_and_reverse)
        else:
            align_file(aligner, path, sys.stdout.buffer, args.json, args.header_comment_delim, args.fwd_and_reverse)
            sys.stdout.buffer.flush()
    index.close()
    return 0
