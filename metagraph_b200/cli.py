"""`python -m metagraph_b200 align -i GRAPH.dbg [options] FILE...`: prints what `metagraph align` prints for the
FASTA/FASTQ files (plain, .gz or .bgz), aligned on the devices --devices lists (CUDA_VISIBLE_DEVICES numbers them).

The files are read in chunks; each chunk is parsed, aligned and rendered on a device, so only the file's bytes go to
the device and only the text comes back. A thread reads the next chunk while the devices work. With one worker
(`--devices 0`, the default) each chunk is one mgb_align_fastx_text call. With several, worker i mod W stages chunk i
(mgb_fastx_stage: parse, and learn where its records end), hands the rest of the buffer on to the next worker and then
aligns its batch while the next chunk is staged. Output is in input order either way, the same bytes for any worker
list, and one of the orders the reference's thread pool can print.

A .gz/.bgz file whose first member is a BGZF block (htslib's bgzip) goes up compressed: each stage inflates its
blocks on the device (mgb_fastx_stage_bgzf) into the text it parses. From the first member the device route does not
serve on, the rest of the file is read by Python's gzip and takes the text route, so every file that is BGZF only in
part gives the bytes, or the error, it gives on the gzip route.

Any other .gz/.bgz file (plain gzip, as gzip and pigz write it) goes up compressed too: each stage inflates part of
a member on the device (mgb_fastx_stage_gzip), decoding the DEFLATE stream from many points at once. Where the device
route refuses, the file is reopened at the current member's start with Python's gzip, the text of that member already
staged is skipped, and the rest takes the text route: the same bytes, or the same error, as Python's gzip.

With --distributed the command is one rank of a torchrun job: rank c mod W stages and aligns chunk c, the token goes
from rank to rank as a small message (the file is read by offset on every rank), and rank 0 gathers and writes the
texts in chunk order; the same bytes as one process with the same chunk size (align_file_distributed).
"""
import argparse
import gzip
import os
import queue
import sys
import threading

from . import bgzf
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
                   help="accepted for compatibility; changes no output (--devices sets the workers)")
    p.add_argument("--devices", default=None, metavar="LIST",
                   help="comma-separated CUDA ordinals, one worker each (an ordinal listed twice runs two workers on "
                        "that device's one index), or `all`: every visible device once [0]")
    p.add_argument("--distributed", action="store_true",
                   help="run as one rank of a torchrun job (RANK, WORLD_SIZE and LOCAL_RANK from its environment): "
                        "rank c mod WORLD_SIZE aligns chunk c on device LOCAL_RANK mod the device count, and rank 0 "
                        "writes all the output")
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
    if args.distributed and args.devices is not None:
        raise UsageError("--devices cannot be combined with --distributed: each rank uses device LOCAL_RANK mod the "
                         "device count")
    if args.devices is None:
        args.devices = "0"
    return args


def dist_env():
    """(RANK, WORLD_SIZE, LOCAL_RANK) as torchrun sets them; UsageError when one is missing or bad"""
    try:
        rank, world, local = (int(os.environ[v]) for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"))
    except (KeyError, ValueError):
        raise UsageError("--distributed needs RANK, WORLD_SIZE and LOCAL_RANK in the environment (run it under "
                         "torchrun)")
    if not 0 <= rank < world or local < 0:
        raise UsageError("--distributed: bad RANK %d, WORLD_SIZE %d or LOCAL_RANK %d" % (rank, world, local))
    return rank, world, local


def devices_of(spec, count):
    """the worker list of --devices: ordinals below `count`, the number of visible devices"""
    if spec == "all":
        if not count:
            raise UsageError("--devices all: no CUDA device is visible")
        return list(range(count))
    try:
        devices = [int(x) for x in spec.split(",")]
    except ValueError:
        raise UsageError("--devices takes comma-separated CUDA ordinals or `all`, not %r" % spec)
    bad = [d for d in devices if not 0 <= d < count]
    if bad:
        raise UsageError("--devices: no CUDA device %d (%d visible)" % (bad[0], count))
    return devices


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


def route_of(path):
    """how a file is read: "plain" (the text as it is), "bgzf" (BGZF blocks inflated on the device), "gzip" (plain
    gzip inflated on the device) or "host" (Python's gzip, the route both device routes hand a file over to)"""
    if not path.endswith((".gz", ".bgz")):
        return "plain"
    return "bgzf" if bgzf.is_bgzf(path) else "gzip"


def align_file(aligner, path, out, json=False, comment_delim=None, fwd_and_reverse=False, chunk_bytes=CHUNK_BYTES):
    """aligns one file and writes its text to `out`, chunk by chunk; returns the number of bytes written"""
    route = route_of(path)
    if route in ("bgzf", "gzip"):
        return align_file_workers([aligner], path, out, json, comment_delim, fwd_and_reverse, chunk_bytes)
    opener = gzip.open if route == "host" else open
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


class _Token:
    """What passes from one stage to the next, held by one worker at a time: the text not yet consumed (`pending`) and
    the grow rule's `want`; on the device routes also the compressed bytes read but not yet staged (`cpend`, which
    starts at file offset `c_at`), and on the gzip route the stream's state and the compressed bytes a stage is
    given (`c_want`, doubled after a stage that could not make progress)."""

    def __init__(self, path, chunk_bytes, reader=None):
        """reader(file, chunk_bytes): what reads the file's chunks (_Chunks, one chunk ahead on a thread, by default)"""
        self.path, self.size = path, chunk_bytes
        self.pending, self.at_eof, self.want = b"", False, 0
        self.route = route_of(path)
        self.raw = self.route in ("bgzf", "gzip")
        self.cpend, self.c_at = b"", 0
        self.stream, self.m_at, self.c_want = None, 0, chunk_bytes
        self.files = [open(path, "rb") if self.raw else (gzip.open if self.route == "host" else open)(path, "rb")]
        self.chunks = (reader or _Chunks)(self.files[0], chunk_bytes)

    def _read(self):
        nxt = self.chunks.next()
        self.at_eof = not nxt
        return nxt

    def stage(self, al, halted, comment_delim, fwd_and_reverse):
        """reads and stages the next chunk: (batch, last), batch None when there is nothing left to stage; last: no
        stage follows this one"""
        if self.raw:
            stage = self._stage_bgzf if self.route == "bgzf" else self._stage_gzip
            return stage(al, halted, comment_delim, fwd_and_reverse)
        pending, want = self.pending, self.want
        while not self.at_eof and not halted():
            nxt = self._read()
            pending = pending + nxt if pending else nxt
            if len(pending) >= want:
                break
        if halted() or not pending:
            return None, True
        batch, consumed, ended = al.stage_fastx(pending, self.at_eof, comment_delim, fwd_and_reverse)
        if ended or self.at_eof:
            return batch, True
        self.want = 2 * len(pending) if consumed == 0 else 0
        self.pending = pending[consumed:]
        return batch, False

    def _stage_bgzf(self, al, halted, comment_delim, fwd_and_reverse):
        # at most chunk_bytes of text from blocks (or, after a stage with no complete record, as much text as that
        # stage held, so the next one holds twice as much), plus one block, plus the tail
        max_text = max(self.size, self.want)
        while not self.at_eof and not halted():
            text, other = bgzf.text_of(self.cpend, max_text)
            if text >= max_text or other:
                break
            nxt = self._read()
            self.cpend = self.cpend + nxt if self.cpend else nxt
        if halted():
            return None, True
        batch, c_used, c_refused, consumed, ended, tail = al.stage_fastx_bgzf(
            self.pending, self.cpend, self.at_eof, max_text, comment_delim, fwd_and_reverse)
        self.cpend, self.c_at = self.cpend[c_used:], self.c_at + c_used
        if ended:
            return batch, True
        if c_refused:
            self._hand_over(tail)
            return batch, False
        if self.at_eof and not self.cpend:
            return batch, True
        self.want = len(tail) if consumed == 0 else 0
        self.pending = tail
        return batch, False

    def _stage_gzip(self, al, halted, comment_delim, fwd_and_reverse):
        # at least c_want compressed bytes; the stage takes what max_text of text needs
        max_text = max(self.size, self.want)
        while not self.at_eof and len(self.cpend) < self.c_want and not halted():
            nxt = self._read()
            self.cpend = self.cpend + nxt if self.cpend else nxt
        if halted():
            return None, True
        if self.stream is None:
            from .aligner import GzipStream
            self.stream = GzipStream(al._L)
        in_member, member_text = self.stream.state()
        if not in_member:
            self.m_at = self.c_at
        batch, c_used, c_refused, consumed, ended, tail = al.stage_fastx_gzip(
            self.stream, self.pending, self.cpend, self.at_eof, max_text, comment_delim, fwd_and_reverse)
        self.cpend, self.c_at = self.cpend[c_used:], self.c_at + c_used
        if ended:
            return batch, True
        if c_refused:
            self._hand_over(tail, self.m_at, member_text)
            return batch, False
        if self.at_eof and not self.cpend and not self.stream.state()[0]:
            return batch, True
        self.c_want = 2 * max(self.c_want, len(self.cpend)) if c_used == 0 else self.size
        self.want = len(tail) if consumed == 0 else 0
        self.pending = tail
        return batch, False

    def _hand_over(self, tail, at=None, skip=0):
        """the rest of the file, from the member at `at` (c_at) on, through Python's gzip onto the text route, less
        the first `skip` bytes of text, which earlier stages took; zero bytes after a member are skipped as gzip skips
        them"""
        self.chunks.close()
        f = open(self.path, "rb")
        self.files.append(f)
        at = self.c_at if at is None else at
        f.seek(at)
        while True:
            b = f.read(1 << 16)
            z = len(b) - len(b.lstrip(b"\0"))
            if z < len(b) or not b:
                f.seek(at + z)
                break
            at += len(b)
        gz = gzip.GzipFile(fileobj=f, mode="rb")
        self.files.append(gz)
        while skip > 0:
            b = gz.read(min(skip, 1 << 24))
            if not b:
                break
            skip -= len(b)
        self.chunks = _Chunks(gz, self.size)
        self.raw, self.route, self.pending, self.at_eof, self.want, self.cpend = False, "host", tail, False, 0, b""

    def close(self):
        self.chunks.close()
        for f in reversed(self.files):
            f.close()
        if self.stream is not None:
            self.stream.close()


class _OffsetChunks:
    """_Chunks by file offset: chunk j is the file's bytes [j*size, (j+1)*size), the bytes the j-th read of _Chunks
    returns, so that any process can go on reading where another stopped; `n` counts the chunks read"""

    def __init__(self, f, size):
        self.f, self.size, self.n = f, size, 0

    def next(self):
        self.f.seek(self.n * self.size)
        self.n += 1
        return self.f.read(self.size)

    def close(self):
        pass


# token kinds between ranks: the state follows (LIVE); the file was handed over to Python's gzip on rank `held`
# (HELD); no chunk follows (OVER); a rank failed, so no rank stages (STOP)
_LIVE, _HELD, _OVER, _STOP = 0, 1, 2, 3
# what each rank reports for a round: its chunk's text (TEXT, LAST when no chunk follows it), no chunk and the file
# goes on (SKIP), no chunk and the file has ended (ENDED), or an error message (ERROR)
_TEXT, _LAST, _SKIP, _ENDED, _ERROR = 0, 1, 2, 3, 4
_TAG_TOKEN, _TAG_STATE, _TAG_TEXT = 1, 2, 3
# A token message is _TOKEN_INTS int64s -- kind, held, the _RankToken state in the order _TOKEN_STATE names it, and the
# length of the body -- then the body: the text tail and the gzip stream's state (mgb_gzip_stream_export).
_TOKEN_STATE = ("chunks_read", "at_eof", "want", "c_at", "m_at", "c_want", "tail_bytes", "stream_bytes")
_TOKEN_INTS = 2 + len(_TOKEN_STATE) + 1


class _RankToken(_Token):
    """The _Token of one rank of `align --distributed`. It reads the file by offset (_OffsetChunks), so its state
    crosses processes as a small message (dump / load): the chunks read and at_eof, c_at, the text tail and grow state,
    and on the gzip route the stream (mgb_gzip_stream_export). The compressed bytes not yet staged are the file's bytes
    from c_at to the end of the last chunk read, so the receiving rank reads them itself. Once handed over to Python's
    gzip (route "host") it stays on this rank."""

    def __init__(self, path, chunk_bytes):
        super().__init__(path, chunk_bytes, _OffsetChunks)

    def dump(self):
        """(the state, in _TOKEN_STATE's order; the body: the text tail then the stream's state)"""
        st = self.stream.export() if self.stream is not None else b""
        return [self.chunks.n, int(self.at_eof), self.want, self.c_at, self.m_at, self.c_want, len(self.pending),
                len(st)], self.pending + st

    def load(self, state, body, L):
        n, at_eof, self.want, self.c_at, self.m_at, self.c_want, n_pending, n_stream = state
        self.chunks.n, self.at_eof = n, bool(at_eof)
        self.pending = body[:n_pending]
        if self.stream is not None:
            self.stream.close()
            self.stream = None
        if n_stream:
            from .aligner import GzipStream
            self.stream = GzipStream.from_export(L, body[n_pending:n_pending + n_stream])
        if self.raw:
            f = self.files[0]
            f.seek(self.c_at)
            self.cpend = f.read(max(0, n * self.size - self.c_at))


def _token_msg(kind, held, token=None):
    """a token message (header ints, body) of this kind; the state of `token` when it is LIVE"""
    state, body = token.dump() if token is not None else ([0] * len(_TOKEN_STATE), b"")
    return [kind, held] + state + [len(body)], body


class DistributedError(RuntimeError):
    """the error that stopped `align --distributed` on some rank, raised on every rank"""


def align_file_distributed(aligner, path, out, json=False, comment_delim=None, fwd_and_reverse=False,
                           chunk_bytes=CHUNK_BYTES):
    """align_file across the ranks of the default process group (gloo): chunk c is staged and aligned by rank c mod W,
    and rank 0 writes every text to `out` (None elsewhere) in chunk order; the same bytes as align_file for the same
    chunk size. The ranks go in rounds of W chunks. In a round the token goes around the ring 0 -> 1 -> ... -> W-1 -> 0
    as a message (_RankToken.dump), each rank staging its chunk before it passes the token on and aligning it after;
    then the texts and one status per rank go to rank 0 (sharding.gather_blocks), which writes them. So a rank holds
    at most one staged batch and one text, and stages chunk c only after rank 0 has written text c - W. From a hand-over
    to Python's gzip on, the rank that made it stages every chunk, one per round.

    Every error on a rank becomes that rank's ERROR status: opening the file, staging, passing the token on, aligning,
    and on rank 0 writing (reported in the next round, whose token is then a STOP; when the file has no next round,
    rank 0 alone raises it and the caller's agreement after the file passes it on). Every rank learns every status, so
    the first error or the end of the file stops all of them after the same round: rank 0 writes the texts before the
    failed chunk, and every rank raises DistributedError with the error's message. Returns the bytes written."""
    import torch.distributed as dist
    from .sharding import gather_blocks
    rank, W = dist.get_rank(), dist.get_world_size()
    token, failed, written = None, None, 0
    try:
        token = _RankToken(path, chunk_bytes)
    except Exception as e:
        failed = str(e)
    msg = _token_msg(_LIVE, 0, token) if token is not None else _token_msg(_STOP, 0)    # rank 0's, for round 1
    try:
        while True:
            if rank:
                msg = _recv_token((rank - 1) % W)
            (kind, held), state, body = msg[0][:2], msg[0][2:-1], msg[1]
            batch, code, block, msg = None, _SKIP, b"", None
            if failed is None and (kind == _LIVE or (kind == _HELD and held == rank)):
                try:
                    if kind == _LIVE and W > 1:
                        token.load(state, body, aligner._L)
                    batch, last = token.stage(aligner, lambda: False, comment_delim, fwd_and_reverse)
                    code = _TEXT
                    if batch is None or last:
                        kind, code = _OVER, _LAST if batch is not None else _ENDED
                    elif token.route == "host":
                        kind, held = _HELD, rank
                    msg = _token_msg(kind, held, token if kind == _LIVE else None)
                except Exception as e:
                    if batch is not None:
                        aligner.free_staged(batch)
                        batch = None
                    failed = str(e)
            elif kind in (_OVER, _STOP):
                code = _ENDED
            if failed is not None:
                code, block, msg = _ERROR, failed.encode("utf-8", "replace"), _token_msg(_STOP, held)
            elif msg is None:
                msg = _token_msg(kind, held)
            sent = _send_token(msg, (rank + 1) % W) if W > 1 else []
            if batch is not None:
                try:
                    block = aligner.align_staged_text(batch, json)     # consumes the batch
                except Exception as e:
                    code, block = _ERROR, str(e).encode("utf-8", "replace")
            if rank == 0 and W > 1:
                msg = _recv_token(W - 1)
            for q in sent:
                q.wait()
            codes, blocks = gather_blocks(block, code, tag=_TAG_TEXT)
            block = None
            for r, c in enumerate(codes):
                if c == _ERROR:
                    error = blocks[r].decode("utf-8", "replace") if blocks is not None else "rank %d failed" % r
                    raise DistributedError(failed if rank == 0 and failed is not None else error)
                if c in (_TEXT, _LAST) and out is not None and failed is None:
                    try:
                        out.write(blocks[r])
                        written += len(blocks[r])
                    except Exception as e:      # reported in the next round
                        failed = str(e)
            if any(c in (_LAST, _ENDED) for c in codes):
                if failed is not None:
                    raise DistributedError(failed)
                return written
    finally:
        if token is not None:
            token.close()


def _send_token(msg, dst):
    """isends a token message (header ints, body bytes) to rank dst; returns the works to wait for"""
    import torch
    import torch.distributed as dist
    hdr, body = msg
    works = [dist.isend(torch.tensor(hdr, dtype=torch.int64), dst, tag=_TAG_TOKEN)]
    if body:
        works.append(dist.isend(torch.frombuffer(bytearray(body), dtype=torch.uint8), dst, tag=_TAG_STATE))
    return works


def _recv_token(src):
    """the token message rank src sent: (header ints, body bytes)"""
    import torch
    import torch.distributed as dist
    hdr = torch.zeros(_TOKEN_INTS, dtype=torch.int64)
    dist.recv(hdr, src, tag=_TAG_TOKEN)
    hdr = [int(x) for x in hdr.tolist()]
    body = b""
    if hdr[-1]:
        t = torch.empty(hdr[-1], dtype=torch.uint8)
        dist.recv(t, src, tag=_TAG_STATE)
        body = t.numpy().tobytes()
    return hdr, body


def align_file_workers(aligners, path, out, json=False, comment_delim=None, fwd_and_reverse=False,
                       chunk_bytes=CHUNK_BYTES):
    """align_file with one worker thread per aligner; the same bytes go to `out`. Chunk i is staged by worker i mod W,
    which holds the token (the rest of the last buffer and the grow rule of align_file) while it reads and stages, and
    hands it on before it aligns. A worker stages chunk i only once fewer than W texts wait ahead of the one to write
    next. The first error stops every worker and the reader: nothing after the last text in order is written, every
    staged batch is freed, every thread is joined, and the error is raised here."""
    W = len(aligners)
    cv = threading.Condition()
    st = dict(turn=0, n_chunks=None, next_out=0, error=None, stop=False)
    texts = {}

    def halted():
        return st["stop"] or st["error"] is not None

    def failed(e):
        with cv:
            if st["error"] is None:
                st["error"] = e
            cv.notify_all()

    def worker(w, al, token):
        i = w
        try:
            while True:
                with cv:
                    cv.wait_for(lambda: halted() or st["n_chunks"] is not None
                                or (st["turn"] == i and i <= st["next_out"] + W))
                    if halted() or st["n_chunks"] is not None:
                        return
                # this worker holds the token: it alone reads and stages until it hands the token on
                batch, last = token.stage(al, halted, comment_delim, fwd_and_reverse)
                if halted() and batch is None:
                    return
                if batch is None:
                    with cv:
                        st["n_chunks"] = i
                        cv.notify_all()
                    return
                with cv:
                    if last:
                        st["n_chunks"] = i + 1
                    st["turn"] = i + 1
                    cv.notify_all()
                    stop = halted()
                if stop:
                    al.free_staged(batch)
                    return
                text = al.align_staged_text(batch, json)      # consumes the batch
                with cv:
                    texts[i] = text
                    cv.notify_all()
                i += W
        except BaseException as e:
            failed(e)

    written = 0
    token = _Token(path, chunk_bytes)
    threads = []
    try:
        for w, al in enumerate(aligners):
            threads.append(threading.Thread(target=worker, args=(w, al, token)))
            threads[-1].start()
        while True:
            with cv:
                cv.wait_for(lambda: st["error"] is not None or st["next_out"] in texts
                            or st["n_chunks"] == st["next_out"])
                if st["error"] is not None or st["n_chunks"] == st["next_out"]:
                    break
                text = texts.pop(st["next_out"])
            out.write(text)
            written += len(text)
            with cv:
                st["next_out"] += 1
                cv.notify_all()
    except BaseException as e:
        failed(e)
    finally:
        with cv:
            st["stop"] = True
            cv.notify_all()
        for t in threads:
            t.join()
        token.close()
    if st["error"] is not None:
        raise st["error"]
    return written


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    if not argv or argv[0] != "align":
        sys.stderr.write("usage: python -m metagraph_b200 align -i GRAPH.dbg [options] FILE...\n")
        return 2
    try:
        args = parse_args(argv[1:])
        if args.distributed:
            env = dist_env()
        from . import _lib
        from .aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
        count = _lib.load_library().mgb_device_count()
        if args.distributed:
            if not count:
                raise UsageError("--distributed: no CUDA device is visible")
            return main_distributed(args, env[0], env[2] % count)
        devices = devices_of(args.devices, count)
        boss = BOSSTable.from_dbg(args.graph)
        alphabet = {0: "dna", 1: "protein"}.get(boss.alphabet, "code %d" % boss.alphabet)
        cfg = config_of(args, boss.k, alphabet)
    except UsageError as e:
        sys.stderr.write("error: %s\n" % e)
        return 1
    # the index is built once, on the first listed device, and copied device to device to the others, all at once
    indexes = {devices[0]: DBGSuccinctIndex(boss, device=devices[0])}
    try:
        errors = []

        def replicate(d):
            try:
                indexes[d] = indexes[devices[0]].replicate(d)
            except Exception as e:
                errors.append(e)

        threads = [threading.Thread(target=replicate, args=(d,)) for d in sorted(set(devices[1:]) - {devices[0]})]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        aligners = [B200Aligner(indexes[d], cfg) for d in devices]

        def align(path, out):
            if len(aligners) == 1:
                align_file(aligners[0], path, out, args.json, args.header_comment_delim, args.fwd_and_reverse,
                           CHUNK_BYTES)
            else:
                align_file_workers(aligners, path, out, args.json, args.header_comment_delim, args.fwd_and_reverse,
                                   CHUNK_BYTES)

        for path in args.files:
            if not os.path.exists(path):
                sys.stderr.write("ERROR: Cannot read from file %s\n" % path)
                return 1
            if args.outfile:
                with open(args.outfile, "wb") as out:       # reopened and truncated per input (cli/align.cpp:409-411)
                    align(path, out)
            else:
                align(path, sys.stdout.buffer)
                sys.stdout.buffer.flush()
    except Exception as e:
        sys.stderr.write("error: %s\n" % e)
        return 1
    finally:
        for ix in indexes.values():
            ix.close()
    return 0


def main_distributed(args, rank, device):
    """main() for one rank of `align --distributed`: every rank loads the graph and builds its own index on `device`,
    and the files are aligned one after the other by all ranks (align_file_distributed). Only rank 0 writes the output
    and the error. The ranks agree (_agree) after the set-up, before each file (it exists on every rank, and rank 0
    could open -o) and after it (rank 0 could write and close its output), so an error on any rank stops every rank
    with the same exit code; they meet at a barrier before they return, so no rank ends while rank 0 still writes."""
    import torch.distributed as dist
    from .aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
    dist.init_process_group("gloo")
    index = None
    try:
        error = None
        try:
            boss = BOSSTable.from_dbg(args.graph)
            alphabet = {0: "dna", 1: "protein"}.get(boss.alphabet, "code %d" % boss.alphabet)
            cfg = config_of(args, boss.k, alphabet)
            index = DBGSuccinctIndex(boss, device=device)
            aligner = B200Aligner(index, cfg)
        except Exception as e:
            error = "error: %s" % e
        if _agree(error, rank):
            return 1
        for path in args.files:
            out, error = None, None
            try:
                if not os.path.exists(path):
                    error = "ERROR: Cannot read from file %s" % path
                elif rank == 0:
                    # reopened and truncated per input (cli/align.cpp:409-411)
                    out = open(args.outfile, "wb") if args.outfile else sys.stdout.buffer
            except Exception as e:
                error = "error: %s" % e
            if _agree(error, rank):
                return 1
            try:
                align_file_distributed(aligner, path, out, args.json, args.header_comment_delim, args.fwd_and_reverse,
                                       CHUNK_BYTES)
            except Exception as e:
                error = "error: %s" % e
            if out is not None:
                try:
                    out.close() if args.outfile else out.flush()
                except Exception as e:
                    error = error or "error: %s" % e
            if _agree(error, rank):
                return 1
        return 0
    finally:
        if rank == 0:
            sys.stderr.flush()
        dist.barrier()
        if index is not None:
            index.close()
        dist.destroy_process_group()


def _agree(error, rank):
    """every rank's error line (None: no error) to every rank: True when some rank has one, which rank 0 then prints
    (the first in rank order)"""
    from .sharding import gather_blocks
    codes, lines = gather_blocks((error or "").encode("utf-8", "replace"), int(error is not None))
    if rank == 0 and any(codes):
        sys.stderr.write("%s\n" % lines[codes.index(1)].decode("utf-8", "replace"))
    return any(codes)
