"""Host-side mirror of the reference's aligner interface for the `metagraph align` hot path.

  BOSSTable          ~ boss::BOSS construction result (W / last / F)   [index build, untimed]
  DBGSuccinctIndex   ~ DBGSuccinct resident in HBM (mgb_index_t)
  B200Aligner        ~ IDBGAligner (graph/alignment/dbg_aligner.hpp:20-39): get_graph(),
                       get_config(), align_batch(batch, callback), align(query)
  AlignmentResults / Alignment ~ graph/alignment/alignment.hpp:132-406
  format_alignment   ~ cli/align.cpp:254-307 (TSV branch)

Everything computes through the C-ABI in include/mgb.h (metagraph_b200/_lib/libmgb.so).
"""
import ctypes
import dataclasses

import numpy as np

from . import _lib
from .config import DBGAlignerConfig, mgb_config_t

_OPS = "SX=DIG"


def _pack(seqs):
    """list of str/bytes -> (uint8 buffer, uint64 offsets)"""
    bs = [s.encode() if isinstance(s, str) else bytes(s) for s in seqs]
    offsets = np.zeros(len(bs) + 1, dtype=np.uint64)
    if bs:
        offsets[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64)
    buf = np.frombuffer(b"".join(bs), dtype=np.uint8) if bs else np.zeros(0, np.uint8)
    return np.ascontiguousarray(buf), offsets


class BOSSTable:
    """W / last / F arrays of a BOSS table (position 0 is the placeholder)."""

    def __init__(self, k, W, last, F, alphabet=0):
        self.k = int(k)
        self.W = np.ascontiguousarray(W, dtype=np.uint8)
        self.last = np.ascontiguousarray(last, dtype=np.uint8)
        self.F = np.ascontiguousarray(F, dtype=np.uint64)
        self.alphabet = alphabet

    @property
    def num_edges(self):
        return len(self.W) - 1

    @classmethod
    def from_sequences(cls, k, seqs, threads=0, force_source_dummies=False, lib=None, packed=None,
                       alphabet=0):
        """alphabet: 0 = DNA ("$ACGT"), 1 = protein ("$ABCDEFGHIJKLMNOPQRSTUVWYZX")"""
        L = _lib.load_library(lib)
        buf, offsets = packed if packed is not None else _pack(seqs)
        b = _lib.mgb_boss_t()
        rc = L.mgb_boss_build(buf.ctypes.data, offsets.ctypes.data, len(offsets) - 1, k, int(alphabet),
                              int(force_source_dummies), threads, ctypes.byref(b))
        if rc:
            raise _lib.MgbError(rc, "mgb_boss_build: " + L.mgb_boss_last_error().decode())
        try:
            n1 = b.n_plus_1
            W = np.ctypeslib.as_array(b.W, shape=(n1,)).copy()
            last = np.ctypeslib.as_array(b.last, shape=(n1,)).copy()
            F = np.array([b.F[i] for i in range(27 if alphabet == 1 else 5)], dtype=np.uint64)
        finally:
            L.mgb_boss_free(ctypes.byref(b))
        return cls(k, W, last, F, alphabet=int(alphabet))

    @classmethod
    def from_dbg(cls, path, lib=None):
        """Loads a graph written by the reference (`metagraph build` -> *.dbg; DBGSuccinct::load,
        dbg_succinct.cpp:690-712). Returns the table; .mode / .state carry the file's graph mode and BOSS state."""
        L = _lib.load_library(lib)
        b = _lib.mgb_boss_t()
        mode, state = ctypes.c_int(-1), ctypes.c_int(-1)
        rc = L.mgb_dbg_load(str(path).encode(), ctypes.byref(b), ctypes.byref(mode), ctypes.byref(state))
        if rc:
            raise _lib.MgbError(rc, "mgb_dbg_load: " + L.mgb_dbg_last_error().decode())
        try:
            n1 = b.n_plus_1
            W = np.ctypeslib.as_array(b.W, shape=(n1,)).copy()
            last = np.ctypeslib.as_array(b.last, shape=(n1,)).copy()
            F = np.array([b.F[i] for i in range(27 if b.alphabet == 1 else 5)], dtype=np.uint64)
            t = cls(b.k, W, last, F, alphabet=int(b.alphabet))
        finally:
            L.mgb_boss_free(ctypes.byref(b))
        t.mode, t.state = mode.value, state.value
        return t

    def dummy_mask(self, lib=None):
        """valid-edge bytes as DBGSuccinct::mask_dummy_kmers computes them"""
        L = _lib.load_library(lib)
        b = _lib.mgb_boss_t()
        b.n_plus_1 = len(self.W)
        b.W = self.W.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
        b.last = self.last.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
        for i in range(len(self.F)):
            b.F[i] = int(self.F[i])
        b.k = self.k
        b.alphabet = self.alphabet
        valid = np.zeros(len(self.W), np.uint8)
        _lib.check(L, L.mgb_boss_mask_dummy(ctypes.byref(b), valid.ctypes.data))
        return valid


def _split(out, nk):
    res, p = [], 0
    for n in nk:
        res.append(out[p:p + int(n)])
        p += int(n)
    return res


class DBGSuccinctIndex:
    """BOSS index resident in one GPU's HBM (DBGSuccinct's role for the aligner)."""

    def __init__(self, boss, valid=None, device=0, suffix_len=0, lib=None, mode=None):
        self._L = _lib.load_library(lib)
        self.k = boss.k
        if mode is None:        # a table read from a .dbg file carries the file's mode
            mode = getattr(boss, "mode", 0)
        h = ctypes.c_void_p()
        v = None
        if valid is not None:
            v = np.ascontiguousarray(valid, dtype=np.uint8)
        _lib.check(self._L, self._L.mgb_index_create(
            boss.W.ctypes.data, boss.last.ctypes.data, len(boss.W), boss.F.ctypes.data,
            v.ctypes.data if v is not None else None, boss.k, boss.alphabet, suffix_len, device,
            ctypes.byref(h)))
        self.handle = h
        self.device = int(device)
        if mode:     # DeBruijnGraph::Mode: 1 = CANONICAL (graph built from the sequences and their reverse complements)
            try:
                _lib.check(self._L, self._L.mgb_index_set_mode(h, int(mode)))
            except Exception:
                self.close()
                raise
        self.mode = mode

    def close(self):
        if self.handle:
            self._L.mgb_index_destroy(self.handle)
            self.handle = None

    def replicate(self, device):
        """a copy of this index on `device` (mgb_index_replicate: device to device, no rebuild), with its own handle"""
        h = ctypes.c_void_p()
        _lib.check(self._L, self._L.mgb_index_replicate(self.handle, int(device), ctypes.byref(h)))
        rep = DBGSuccinctIndex.__new__(DBGSuccinctIndex)
        rep._L, rep.k, rep.mode, rep.handle, rep.device = self._L, self.k, self.mode, h, int(device)
        return rep

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_k(self):
        return self.k

    @property
    def num_edges(self):
        return self._L.mgb_index_num_edges(self.handle)

    @property
    def device_bytes(self):
        return self._L.mgb_index_device_bytes(self.handle)

    def map_to_nodes_sequentially(self, seqs, packed=None):
        """node ids of all k-mers of each sequence (0 = missing); list of uint64 arrays"""
        buf, offsets = packed if packed is not None else _pack(seqs)
        lens = (offsets[1:] - offsets[:-1]).astype(np.int64)
        nk = np.maximum(lens - self.k + 1, 0)
        out = np.zeros(int(nk.sum()) + 1, dtype=np.uint64)
        _lib.check(self._L, self._L.mgb_map_to_nodes(self.handle, buf.ctypes.data, offsets.ctypes.data,
                                                     len(lens), out.ctypes.data))
        return _split(out, nk)

    def map_to_nodes_strands(self, seqs, packed=None):
        """node ids of all k-mers of each sequence and of its reverse complement in the stored graph, whatever the
        mode (no PRIMARY merge of the strands): two lists of uint64 arrays"""
        buf, offsets = packed if packed is not None else _pack(seqs)
        lens = (offsets[1:] - offsets[:-1]).astype(np.int64)
        nk = np.maximum(lens - self.k + 1, 0)
        fwd = np.zeros(int(nk.sum()) + 1, dtype=np.uint64)
        rev = np.zeros(int(nk.sum()) + 1, dtype=np.uint64)
        _lib.check(self._L, self._L.mgb_map_to_nodes_strands(self.handle, buf.ctypes.data, offsets.ctypes.data,
                                                             len(lens), fwd.ctypes.data, rev.ctypes.data))
        return _split(fwd, nk), _split(rev, nk)


class Alignment:
    __slots__ = ("orientation", "score", "offset", "query_begin", "query_len", "nodes", "sequence", "cigar")

    def get_cigar_string(self):
        return "".join("%d%s" % (int(x) >> 3, _OPS[int(x) & 7]) for x in self.cigar)

    def get_num_matches(self):
        return int(sum(int(x) >> 3 for x in self.cigar if int(x) & 7 == 2))

    def __repr__(self):   # fmt::formatter<Alignment> (alignment.hpp:418-435)
        return "%s\t%s\t%d\t%d\t%s\t%d" % ("-" if self.orientation else "+", self.sequence, self.score,
                                           self.get_num_matches(), self.get_cigar_string(), self.offset)


_COMP = {}
for _f, _t in zip("ABCDGHKMRTUVY", "TVGHCDMKYAABR"):      # COMPL_TAB (seq_tools/reverse_complement.hpp:31-48)
    _COMP[_f] = _t
    _COMP[_f.lower()] = _t.lower()
_COMP["`"] = "@"


def reverse_complement(seq):
    return "".join(_COMP.get(c, c) for c in reversed(seq))


def _json_value(v):
    """Json::StreamWriterBuilder with indentation "" (jsoncpp): sorted keys, no blanks, doubles as %.17g"""
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, float):
        t = "%.17g" % v
        return t if any(c in t for c in ".en") else t + ".0"
    if isinstance(v, str):
        out = ['"']
        for ch in v:
            if ch in '"\\':
                out.append("\\" + ch)
            elif ch == "\n":
                out.append("\\n")
            elif ch == "\t":
                out.append("\\t")
            elif ord(ch) < 0x20:
                out.append("\\u%04x" % ord(ch))
            else:
                out.append(ch)
        out.append('"')
        return "".join(out)
    if isinstance(v, list):
        return "[" + ",".join(_json_value(x) for x in v) + "]"
    return "{" + ",".join(_json_value(k) + ":" + _json_value(v[k]) for k in sorted(v)) + "}"


def _path_json(nodes, cigar, node_size, query_view, offset, label):
    """path_json (alignment.cpp:704-880), derived there from GraphAligner's vg.proto"""
    ops = [(int(x) & 7, int(x) >> 3) for x in cigar]          # (Cigar::Operator, length); 0 = CLIPPED
    it = 1 if ops and ops[0][0] == 0 else 0
    cigar_offset = 0
    qpos = 0
    path = {"mapping": []}
    cur_pos = offset
    position = {"node_id": int(nodes[0])}
    if cur_pos:
        position["offset"] = cur_pos
    mapping = {"position": position, "edit": []}
    while cur_pos < node_size and it < len(ops):                # the first node
        op, n = ops[it]
        if op == 0:                                             # trailing clipping
            it += 1
            cigar_offset = 0
            continue
        next_pos = min(node_size, cur_pos + (n - cigar_offset))
        next_size = next_pos - cur_pos
        edit = {}
        if op == 1:                                             # MISMATCH
            edit = {"from_length": next_size, "to_length": next_size, "sequence": query_view[qpos:qpos + next_size]}
            qpos += next_size
        elif op == 4:                                           # INSERTION
            edit = {"to_length": next_size, "sequence": query_view[qpos:qpos + next_size]}
            qpos += next_size
            next_pos = cur_pos
        elif op == 3:                                           # DELETION
            edit = {"from_length": next_size}
        elif op == 2:                                           # MATCH
            edit = {"from_length": next_size, "to_length": next_size}
            qpos += next_size
        cigar_offset += next_size
        cur_pos = next_pos
        mapping["edit"].append(edit)
        if cigar_offset == n:
            it += 1
            cigar_offset = 0
    rank = 1
    mapping["rank"] = rank
    if not mapping["edit"]:
        del mapping["edit"]
    path["mapping"].append(mapping)
    for node in nodes[1:]:                                      # one character per further node
        rank += 1
        mapping = {"position": {"node_id": int(node), "offset": node_size - 1}, "edit": []}
        op, n = ops[it]
        if op in (4, 0):
            length = n - cigar_offset
            mapping["edit"].append({"to_length": length, "sequence": query_view[qpos:qpos + length]})
            qpos += length
            it += 1
            cigar_offset = 0
            op, n = ops[it]
        if op == 1:
            edit = {"from_length": 1, "to_length": 1, "sequence": query_view[qpos:qpos + 1]}
            qpos += 1
        elif op == 3:
            edit = {"from_length": 1}
        else:
            edit = {"from_length": 1, "to_length": 1}
            qpos += 1
        cigar_offset += 1
        if cigar_offset == n:
            cigar_offset = 0
            it += 1
        mapping["edit"].append(edit)
        mapping["rank"] = rank
        path["mapping"].append(mapping)
    path["length"] = len(nodes)
    if int(nodes[0]) == int(nodes[-1]):
        path["is_circular"] = True
    path["name"] = label
    return path


def alignment_to_json(a, strand_query, node_size, is_secondary, read_name, label=""):
    """Alignment::to_json (alignment.cpp:882-963). strand_query = the query strand `a` was aligned to
    (a None alignment gives the record of an unaligned read)."""
    out = {"name": read_name, "sequence": strand_query}
    if a is None:
        return out
    if a.sequence:
        out.setdefault("annotation", {})["ref_sequence"] = a.sequence
    if not a.query_len:
        return out
    out.setdefault("annotation", {})["cigar"] = a.get_cigar_string()
    view = strand_query[a.query_begin:a.query_begin + a.query_len]
    if len(a.nodes):
        out["path"] = _path_json(a.nodes, a.cigar, node_size, view, a.offset, label)
    out["score"] = int(a.score)
    if a.query_begin:
        out["query_position"] = int(a.query_begin)
        out["soft_clipped"] = True
    if is_secondary:
        out["is_secondary"] = True
    out["identity"] = a.get_num_matches() / a.query_len if a.query_len else 0.0
    out["read_mapped"] = bool(a.query_len)
    if a.orientation:
        out["read_on_reverse_strand"] = True
    return out


def format_alignment_json(header, paths, k):
    """cli/align.cpp:289-304, JSON branch: one line per alignment (without the trailing newline)"""
    lines = []
    for i, a in enumerate(paths):
        q = reverse_complement(paths.get_query()) if a.orientation else paths.get_query()
        lines.append(_json_value(alignment_to_json(a, q, k, i > 0, header)))
    if not paths:
        lines.append(_json_value(alignment_to_json(None, "", k, False, header)))
    return "\n".join(lines)


class AlignmentResults(list):
    """Alignments of one read (alignment.hpp:366-406)."""

    def __init__(self, query):
        super().__init__()
        # upper-cased copy, bytes >= 128 -> 127 (alignment.cpp:1357-1358)
        self.query = "".join(chr(127) if ord(c) >= 128 else c.upper() for c in query)

    def get_query(self):
        return self.query


def format_alignment(header, paths, min_path_score=0, with_nodes=False):
    """cli/align.cpp:254-307, TSV branch (without the trailing newline)"""
    out = "%s\t%s" % (header, paths.get_query())
    if not paths:
        return out + "\t*\t*\t%d\t*\t*\t*" % min_path_score
    for a in paths:
        out += "\t" + repr(a)
    if with_nodes:
        for a in paths:
            out += "\t" + ",".join(str(int(n)) for n in a.nodes)
    return out


def results_of_handle(L, res, seq_batch):
    """AlignmentResults of every read of a mgb_results_t (seq_batch: the (header, sequence) pairs it was made from)"""
    alns = L.mgb_results_alignments(res)
    out = []
    first, count = ctypes.c_uint64(), ctypes.c_uint32()
    for r, (header, seq) in enumerate(seq_batch):
        ar = AlignmentResults(seq if isinstance(seq, str) else seq.decode("latin1"))
        L.mgb_results_read_range(res, r, ctypes.byref(first), ctypes.byref(count))
        for i in range(first.value, first.value + count.value):
            x = alns[i]
            a = Alignment()
            a.orientation = bool(x.orientation); a.score = x.score; a.offset = x.offset
            a.query_begin = x.query_begin; a.query_len = x.query_len
            a.nodes = np.ctypeslib.as_array(x.nodes, shape=(x.num_nodes,)).copy() if (x.num_nodes and x.nodes) else np.zeros(0, np.uint64)
            a.sequence = ctypes.string_at(x.sequence, x.sequence_len).decode("latin1")
            a.cigar = np.ctypeslib.as_array(x.cigar, shape=(x.num_cigar_ops,)).copy()
            ar.append(a)
        out.append(ar)
    return out


@dataclasses.dataclass
class DeviceAlignments:
    """Alignments of B200Aligner.align_tensors as torch tensors on the index's device. The alignments of read r are
    [read_first[r], read_first[r + 1]); alignment i has the fields of mgb_alignment_t (int32 for the uint32 ones), its
    path spelling sequence[sequence_offsets[i]:sequence_offsets[i + 1]], its CIGAR words ((len << 3) | op) and node ids
    likewise. nodes is empty when the config's result_nodes is MGB_NODES_NONE."""
    read_first: object          # int64 [n_reads + 1]
    read_index: object          # int32 [n_alignments]
    orientation: object         # uint8
    score: object               # int32
    offset: object
    query_begin: object
    query_len: object
    num_nodes: object
    sequence_len: object
    num_cigar_ops: object
    sequence: object            # uint8 [sequence bytes]
    sequence_offsets: object    # int64 [n_alignments + 1]
    cigar: object               # int32 [CIGAR ops]
    cigar_offsets: object       # int64 [n_alignments + 1]
    nodes: object               # int64 [node ids]
    node_offsets: object        # int64 [n_alignments + 1]
    stats: dict


def _column_dtypes(torch):
    i32, i64 = torch.int32, torch.int64
    return {"read_first": i64, "read_index": i32, "orientation": torch.uint8, "score": i32, "offset": i32,
            "query_begin": i32, "query_len": i32, "num_nodes": i32, "sequence_len": i32, "num_cigar_ops": i32,
            "sequence": torch.uint8, "sequence_offsets": i64, "cigar": i32, "cigar_offsets": i64, "nodes": i64,
            "node_offsets": i64}


class B200Aligner:
    """IDBGAligner over the H100 kernels (Seeder = SuffixSeeder<UniMEMSeeder>, Extender =
    DefaultColumnExtender, as DBGAligner<> in dbg_aligner.hpp:42-45)."""

    def __init__(self, graph, config=None):
        self.graph = graph
        self.config = config or DBGAlignerConfig()
        self._L = graph._L
        self.last_stats = None
        # the DBGAligner constructor throws for a configuration it cannot run (dbg_aligner.cpp:55-56)
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        _lib.check(self._L, self._L.mgb_config_check(self.graph.handle, ctypes.byref(c)))

    def get_graph(self):
        return self.graph

    def get_config(self):
        return self.config

    def has_coordinates(self):
        return False

    def align_batch_raw(self, buf, offsets):
        """Runs mgb_align_batch on packed reads; returns the opaque results handle."""
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        res = ctypes.c_void_p()
        _lib.check(self._L, self._L.mgb_align_batch(self.graph.handle, ctypes.byref(c), buf.ctypes.data,
                                                    offsets.ctypes.data, len(offsets) - 1, ctypes.byref(res)))
        return res

    def free_raw(self, res):
        self._L.mgb_results_free(res)

    def set_pipeline_pieces(self, max_pieces):
        """mgb_set_pipeline_pieces: cap on the pieces a batch is split into (0 = automatic)."""
        self._L.mgb_set_pipeline_pieces(int(max_pieces))

    def stats_of(self, res):
        st = self._L.mgb_results_stats(res).contents
        return {n: getattr(st, n) for n, _ in _lib.mgb_stats_t._fields_}

    def align_tensors(self, reads, offsets):
        """mgb_align_batch_device: aligns reads already in GPU memory and returns DeviceAlignments on that device.

        reads: 1-D torch.uint8 tensor with stride 1 on the index's device (a slice that starts anywhere in its storage
        is fine); offsets: int64 tensor [n + 1] on the CPU or on that device, read r = reads[offsets[r]:offsets[r + 1]].
        The work is ordered after what is queued on torch's current stream, and the columns are written on it. With the
        host-emulation library (tests) the "device" is the host and both tensors are CPU tensors."""
        import torch
        emu = hasattr(self._L, "mgb_emu_whole_read_hits")
        device = torch.device("cpu") if emu else torch.device("cuda", self.graph.device)
        if not isinstance(reads, torch.Tensor) or not isinstance(offsets, torch.Tensor):
            raise ValueError("align_tensors takes torch tensors")
        if reads.dtype != torch.uint8 or reads.dim() != 1 or (reads.numel() > 1 and reads.stride(0) != 1):
            raise ValueError("reads must be a 1-D torch.uint8 tensor with stride 1")
        if reads.device != device:
            raise ValueError("reads must be on %s (the index's device), not %s" % (device, reads.device))
        if offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1:
            raise ValueError("offsets must be a 1-D torch.int64 tensor of n_reads + 1 entries")
        if offsets.device not in (torch.device("cpu"), device):
            raise ValueError("offsets must be on the CPU or on %s, not %s" % (device, offsets.device))
        n_reads = offsets.numel() - 1
        if n_reads >= 1 << 32:
            raise ValueError("at most 2^32 - 1 reads per batch")
        offsets = offsets.contiguous()
        first, last = offsets[[0, -1]].tolist()
        if first < 0 or last > reads.numel():
            raise ValueError("offsets [%d, %d] outside the %d bytes of reads" % (first, last, reads.numel()))
        on_device = not emu and offsets.device == device
        stream = None if emu else torch.cuda.current_stream(device).cuda_stream
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        h = ctypes.c_void_p()
        _lib.check(self._L, self._L.mgb_align_batch_device(self.graph.handle, ctypes.byref(c), reads.data_ptr() or None,
                                                           offsets.data_ptr(), int(on_device), n_reads, stream,
                                                           ctypes.byref(h)))
        try:
            z = _lib.mgb_device_sizes_t()
            _lib.check(self._L, self._L.mgb_device_results_sizes(h, ctypes.byref(z)))
            st = self._L.mgb_device_results_stats(h).contents
            stats = {n: getattr(st, n) for n, _ in _lib.mgb_stats_t._fields_}
            count = {"read_first": z.n_reads + 1, "sequence": z.sequence_bytes, "cigar": z.cigar_ops, "nodes": z.nodes,
                     "sequence_offsets": z.n_alignments + 1, "cigar_offsets": z.n_alignments + 1,
                     "node_offsets": z.n_alignments + 1}
            out = {n: torch.empty(count.get(n, z.n_alignments), dtype=dt, device=device)
                   for n, dt in _column_dtypes(torch).items()}
            cols = _lib.mgb_device_columns_t(**{n: (t.data_ptr() if t.numel() else None) for n, t in out.items()})
            _lib.check(self._L, self._L.mgb_device_results_write(h, ctypes.byref(cols), stream))
        finally:
            self._L.mgb_device_results_free(h)
        self.last_stats = stats
        return DeviceAlignments(stats=stats, **out)

    def align_batch(self, seq_batch, callback=None):
        """seq_batch: list of (header, sequence). Calls callback(header, AlignmentResults) in input
        order (dbg_aligner.cpp:263, 353) and returns the list of AlignmentResults."""
        seqs = [s for _, s in seq_batch]
        buf, offsets = _pack(seqs)
        res = self.align_batch_raw(buf, offsets)
        try:
            self.last_stats = self.stats_of(res)
            out = results_of_handle(self._L, res, seq_batch)
            if callback:
                for (header, _), ar in zip(seq_batch, out):
                    callback(header, ar)
            return out
        finally:
            self.free_raw(res)

    def align_batch_text_raw(self, buf, offsets, hbuf, hoffsets, json=False):
        """Runs mgb_align_batch_text on packed reads and headers; returns the opaque results handle."""
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        res = ctypes.c_void_p()
        fmt = _lib.MGB_TEXT_JSON if json else _lib.MGB_TEXT_TSV
        _lib.check(self._L, self._L.mgb_align_batch_text(self.graph.handle, ctypes.byref(c), buf.ctypes.data,
                                                         offsets.ctypes.data, hbuf.ctypes.data, hoffsets.ctypes.data,
                                                         len(offsets) - 1, fmt, ctypes.byref(res)))
        return res

    def text_of(self, res):
        """the text block of a result set of mgb_align_batch_text, as bytes"""
        p, n = ctypes.c_void_p(), ctypes.c_uint64()
        _lib.check(self._L, self._L.mgb_results_text(res, ctypes.byref(p), ctypes.byref(n)))
        # (ctypes.string_at takes a C int size: blocks of 2 GiB and more are copied through an array type)
        return bytes((ctypes.c_char * n.value).from_address(p.value)) if n.value else b""

    def align_batch_text(self, seq_batch, json=False):
        """seq_batch: list of (header, sequence), str or bytes. Returns what `metagraph align` prints for them, rendered
        on the device: the concatenation of format_alignment(header, paths, min_path_score) + "\\n" per read (json=False)
        or of format_alignment_json(header, paths, k) + "\\n" (json=True), in input order, as bytes."""
        buf, offsets = _pack([s for _, s in seq_batch])
        hbuf, hoffsets = _pack([h for h, _ in seq_batch])
        res = self.align_batch_text_raw(buf, offsets, hbuf, hoffsets, json)
        try:
            self.last_stats = self.stats_of(res)
            return self.text_of(res)
        finally:
            self.free_raw(res)

    def align_fastx_text_raw(self, buf, at_eof=True, comment_delim=None, fwd_and_reverse=False, json=False):
        """Runs mgb_align_fastx_text on one chunk of FASTA/FASTQ bytes (a uint8 array or bytes); returns (results
        handle, consumed, ended)."""
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        arr = np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else buf
        res, consumed, ended = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_int()
        fmt = _lib.MGB_TEXT_JSON if json else _lib.MGB_TEXT_TSV
        flags = _lib.MGB_FASTX_FWD_AND_REVERSE if fwd_and_reverse else 0
        delim = None if comment_delim is None else _as_bytes(comment_delim)
        _lib.check(self._L, self._L.mgb_align_fastx_text(self.graph.handle, ctypes.byref(c), arr.ctypes.data, len(arr),
                                                         int(bool(at_eof)), delim, flags, fmt, ctypes.byref(consumed),
                                                         ctypes.byref(ended), ctypes.byref(res)))
        return res, consumed.value, bool(ended.value)

    def align_fastx_text(self, buf, at_eof=True, comment_delim=None, fwd_and_reverse=False, json=False):
        """What `metagraph align` prints for the complete FASTA/FASTQ records of buf, rendered on the device.
        Returns (text, consumed, ended): bytes of buf up to the end of the last complete record, and whether a
        malformed record ended the input (see mgb_align_fastx_text)."""
        res, consumed, ended = self.align_fastx_text_raw(buf, at_eof, comment_delim, fwd_and_reverse, json)
        try:
            self.last_stats = self.stats_of(res)
            return self.text_of(res), consumed, ended
        finally:
            self.free_raw(res)

    def stage_fastx(self, buf, at_eof=True, comment_delim=None, fwd_and_reverse=False):
        """mgb_fastx_stage: parses the complete records of one chunk (a uint8 array or bytes) and returns (batch
        handle, consumed, ended) as soon as the boundary is known; buf may be reused at once. The batch is aligned by
        align_staged_text or freed by free_staged."""
        arr = np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else buf
        batch, consumed, ended = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_int()
        flags = _lib.MGB_FASTX_FWD_AND_REVERSE if fwd_and_reverse else 0
        delim = None if comment_delim is None else _as_bytes(comment_delim)
        _lib.check(self._L, self._L.mgb_fastx_stage(self.graph.handle, arr.ctypes.data, len(arr), int(bool(at_eof)),
                                                    delim, flags, ctypes.byref(consumed), ctypes.byref(ended),
                                                    ctypes.byref(batch)))
        return batch, consumed.value, bool(ended.value)

    def align_staged_text(self, batch, json=False):
        """mgb_align_fastx_batch_text: the text of a staged batch, as align_fastx_text would have returned it; the
        batch is consumed, also when this raises"""
        c = self.config.to_c() if not isinstance(self.config, mgb_config_t) else self.config
        res = ctypes.c_void_p()
        fmt = _lib.MGB_TEXT_JSON if json else _lib.MGB_TEXT_TSV
        _lib.check(self._L, self._L.mgb_align_fastx_batch_text(self.graph.handle, ctypes.byref(c), batch, fmt,
                                                               ctypes.byref(res)))
        try:
            self.last_stats = self.stats_of(res)
            return self.text_of(res)
        finally:
            self.free_raw(res)

    def free_staged(self, batch):
        self._L.mgb_fastx_batch_free(batch)

    def stage_fastx_bgzf(self, head, cbuf, c_eof, max_text, comment_delim=None, fwd_and_reverse=False):
        """mgb_fastx_stage_bgzf: stages the text `head` followed by the text of the complete BGZF blocks at the start of
        cbuf (bytes), inflated on the device until their text reaches max_text. Returns (batch, c_consumed, c_refused,
        consumed, ended, tail): compressed bytes taken, whether the member after them is left to the host, the text
        consumed and ended as stage_fastx returns them, and the text after the last complete record, as bytes."""
        hbuf = _as_bytes(head)
        cb = np.frombuffer(cbuf, np.uint8) if isinstance(cbuf, (bytes, bytearray, memoryview)) else cbuf
        batch, c_consumed, c_refused = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_int()
        consumed, ended = ctypes.c_uint64(), ctypes.c_int()
        flags = _lib.MGB_FASTX_FWD_AND_REVERSE if fwd_and_reverse else 0
        delim = None if comment_delim is None else _as_bytes(comment_delim)
        _lib.check(self._L, self._L.mgb_fastx_stage_bgzf(
            self.graph.handle, hbuf, len(hbuf), cb.ctypes.data, len(cb), int(bool(c_eof)), int(max_text), delim, flags,
            ctypes.byref(c_consumed), ctypes.byref(c_refused), ctypes.byref(consumed), ctypes.byref(ended),
            ctypes.byref(batch)))
        p, n = ctypes.c_void_p(), ctypes.c_uint64()
        try:
            _lib.check(self._L, self._L.mgb_fastx_batch_tail(batch, ctypes.byref(p), ctypes.byref(n)))
            tail = bytes((ctypes.c_char * n.value).from_address(p.value)) if n.value else b""
        except BaseException:
            self.free_staged(batch)
            raise
        return batch, c_consumed.value, bool(c_refused.value), consumed.value, bool(ended.value), tail

    def stage_fastx_gzip(self, stream, head, cbuf, c_eof, max_text, comment_delim=None, fwd_and_reverse=False):
        """mgb_fastx_stage_gzip: stages the text `head` followed by the text of the plain gzip stream `stream` (a
        GzipStream) whose next bytes are cbuf, inflated on the device up to a confirmed block boundary once the text
        reaches max_text, or to the member's end. Returns what stage_fastx_bgzf returns; c_refused: nothing of the
        stream was staged and the stream is where it was."""
        hbuf = _as_bytes(head)
        cb = np.frombuffer(cbuf, np.uint8) if isinstance(cbuf, (bytes, bytearray, memoryview)) else cbuf
        batch, c_consumed, c_refused = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_int()
        consumed, ended = ctypes.c_uint64(), ctypes.c_int()
        flags = _lib.MGB_FASTX_FWD_AND_REVERSE if fwd_and_reverse else 0
        delim = None if comment_delim is None else _as_bytes(comment_delim)
        _lib.check(self._L, self._L.mgb_fastx_stage_gzip(
            self.graph.handle, stream.handle, hbuf, len(hbuf), cb.ctypes.data, len(cb), int(bool(c_eof)),
            int(max_text), delim, flags, ctypes.byref(c_consumed), ctypes.byref(c_refused), ctypes.byref(consumed),
            ctypes.byref(ended), ctypes.byref(batch)))
        p, n = ctypes.c_void_p(), ctypes.c_uint64()
        try:
            _lib.check(self._L, self._L.mgb_fastx_batch_tail(batch, ctypes.byref(p), ctypes.byref(n)))
            tail = bytes((ctypes.c_char * n.value).from_address(p.value)) if n.value else b""
        except BaseException:
            self.free_staged(batch)
            raise
        return batch, c_consumed.value, bool(c_refused.value), consumed.value, bool(ended.value), tail

    def align(self, query):
        return self.align_batch([("", query)])[0]


class GzipStream:
    """mgb_gzip_stream_t: where a plain gzip stream's next stage starts, kept in host memory between stages"""

    def __init__(self, L):
        self._L = L                 # the library the stages run in
        self.handle = ctypes.c_void_p()
        _lib.check(self._L, self._L.mgb_gzip_stream_create(ctypes.byref(self.handle)))

    def state(self):
        """(inside a member, text of that member staged so far)"""
        m, t = ctypes.c_int(), ctypes.c_uint64()
        _lib.check(self._L, self._L.mgb_gzip_stream_state(self.handle, ctypes.byref(m), ctypes.byref(t)))
        return bool(m.value), t.value

    def export(self):
        """mgb_gzip_stream_export: the stream's state as bytes, which from_export rebuilds in any process"""
        n = int(self._L.mgb_gzip_stream_export_bytes(self.handle))
        buf = ctypes.create_string_buffer(n)
        _lib.check(self._L, self._L.mgb_gzip_stream_export(self.handle, buf, n))
        return buf.raw

    @classmethod
    def from_export(cls, L, block):
        """mgb_gzip_stream_import: a new stream in library L with the state `block` (from export) holds"""
        s = cls.__new__(cls)
        s._L, s.handle = L, ctypes.c_void_p()
        block = bytes(block)
        _lib.check(L, L.mgb_gzip_stream_import(block, len(block), ctypes.byref(s.handle)))
        return s

    def close(self):
        if self.handle:
            self._L.mgb_gzip_stream_free(self.handle)
            self.handle = ctypes.c_void_p()


def _as_bytes(x):
    return x.encode("latin1") if isinstance(x, str) else bytes(x)


def bgzf_inflate(index, cbuf, c_eof=True):
    """mgb_bgzf_inflate: the text of the complete BGZF blocks at the start of cbuf (bytes), inflated on index's device.
    Returns (text, c_consumed, n_blocks, refused)."""
    from . import bgzf
    L = index._L
    cbuf = bytes(cbuf)
    cb = np.frombuffer(cbuf, np.uint8) if cbuf else np.zeros(1, np.uint8)
    cap = bgzf.text_of(cbuf)[0] + 1
    out = np.zeros(cap, np.uint8)
    n, c_consumed, n_blocks, refused = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int()
    _lib.check(L, L.mgb_bgzf_inflate(index.handle, cb.ctypes.data, len(cbuf), int(bool(c_eof)), out.ctypes.data, cap,
                                     ctypes.byref(n), ctypes.byref(c_consumed), ctypes.byref(n_blocks),
                                     ctypes.byref(refused)))
    return out[:n.value].tobytes(), c_consumed.value, n_blocks.value, bool(refused.value)


def gzip_inflate(index, cbuf, c_eof=True, sub_bytes=0, cands=None):
    """mgb_gzip_inflate: the gzip members of cbuf (bytes) inflated on index's device, with sub-ranges of sub_bytes
    compressed bytes (0: the default) and, when given, the candidate block starts `cands` (bit offsets in cbuf) in
    place of the finder's. Returns (text, c_consumed, refused, (sub-ranges, candidates found, candidates confirmed))."""
    L = index._L
    cbuf = bytes(cbuf)
    cb = np.frombuffer(cbuf, np.uint8) if cbuf else np.zeros(1, np.uint8)
    cd = np.asarray(cands if cands is not None else [0], np.uint64)
    counts = np.zeros(3, np.uint64)
    n, c_consumed, refused = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int()
    cap = 4 * len(cbuf) + 1024
    while True:
        out = np.zeros(cap, np.uint8)
        rc = L.mgb_gzip_inflate(index.handle, cb.ctypes.data, len(cbuf), int(bool(c_eof)), int(sub_bytes),
                                cd.ctypes.data if cands is not None else None, len(cands) if cands is not None else 0,
                                out.ctypes.data, cap, ctypes.byref(n), ctypes.byref(c_consumed), ctypes.byref(refused),
                                counts.ctypes.data)
        if rc == -5 and n.value > cap:          # MGB_ERR_OVERFLOW: again with room for the whole text
            cap = n.value
            continue
        _lib.check(L, rc)
        return out[:n.value].tobytes(), c_consumed.value, bool(refused.value), tuple(int(x) for x in counts)


def parse_fastx(buf, at_eof=True, comment_delim=None, fwd_and_reverse=False, index=None, lib=None):
    """The records mgb_align_fastx_text aligns for these arguments (mgb_fastx_parse): with index, as its device
    parses them; without, by the host restatement of kseq_read. Returns (headers, reads, consumed, ended, refused),
    headers and reads as lists of bytes; refused: the device route left the chunk to the host restatement."""
    L = index._L if index is not None else _lib.load_library(lib)
    data = bytes(buf)
    arr = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
    delim = None if comment_delim is None else _as_bytes(comment_delim)
    copies = 2 if fwd_and_reverse else 1
    # every record starts at a '>' or '@' byte
    max_rec = copies * (data.count(b">") + data.count(b"@") + 1)
    max_seq = copies * len(data) + 1
    max_name = copies * (len(data) + max_rec * len(delim or b"")) + 1
    seqs, names = np.zeros(max_seq, np.uint8), np.zeros(max_name, np.uint8)
    offs, noffs = np.zeros(max_rec + 1, np.uint64), np.zeros(max_rec + 1, np.uint64)
    n, consumed, ended, refused = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L, L.mgb_fastx_parse(index.handle if index is not None else None, arr.ctypes.data, len(data),
                                    int(bool(at_eof)), delim, _lib.MGB_FASTX_FWD_AND_REVERSE if fwd_and_reverse else 0,
                                    int(index is not None), seqs.ctypes.data, max_seq, offs.ctypes.data,
                                    names.ctypes.data, max_name, noffs.ctypes.data, max_rec, ctypes.byref(n),
                                    ctypes.byref(consumed), ctypes.byref(ended), ctypes.byref(refused)))
    n = n.value
    sb, nb = seqs.tobytes(), names.tobytes()
    reads = [sb[int(offs[i]):int(offs[i + 1])] for i in range(n)]
    headers = [nb[int(noffs[i]):int(noffs[i + 1])] for i in range(n)]
    return headers, reads, consumed.value, bool(ended.value), bool(refused.value)
