"""ctypes wrapper around oracle/build/libmgo.so (CPU restatement; test infrastructure only)."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "build", "libmgo.so")


def build_oracle():
    srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle"))
            if f.endswith((".cpp", ".hpp"))]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")],
                              stdout=subprocess.DEVNULL)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build_oracle()
        L = ctypes.CDLL(LIB)
        u64, vp, cp, i = ctypes.c_uint64, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int
        L.mgo_config_sizeof.restype = u64
        L.mgo_graph_build.restype = vp
        L.mgo_graph_build.argtypes = [cp, i, ctypes.POINTER(cp), i, i, i, i]
        L.mgo_graph_from_arrays.restype = vp
        L.mgo_graph_from_arrays.argtypes = [cp, i, vp, vp, u64, vp, i]
        L.mgo_graph_free.argtypes = [vp]
        L.mgo_graph_set_mode.argtypes = [vp, ctypes.c_int]
        for f in ("mgo_graph_num_edges", "mgo_graph_num_nodes"):
            getattr(L, f).restype = u64
            getattr(L, f).argtypes = [vp]
        L.mgo_graph_mask_dummy.argtypes = [vp, i]
        L.mgo_graph_get_arrays.argtypes = [vp, vp, vp, vp, vp]
        L.mgo_map_to_nodes.restype = u64
        L.mgo_map_to_nodes.argtypes = [vp, cp, u64, vp]
        L.mgo_call_outgoing.restype = i
        L.mgo_call_outgoing.argtypes = [vp, u64, i, vp, vp]
        for f in ("mgo_boss_fwd", "mgo_boss_bwd", "mgo_boss_pred_last", "mgo_boss_succ_last",
                  "mgo_boss_rank_last", "mgo_boss_select_last", "mgo_boss_is_single_incoming"):
            getattr(L, f).restype = u64
            getattr(L, f).argtypes = [vp, u64]
        for f in ("mgo_boss_pick_edge", "mgo_boss_rank_W"):
            getattr(L, f).restype = u64
            getattr(L, f).argtypes = [vp, u64, i]
        L.mgo_node_sequence.argtypes = [vp, u64, vp]
        L.mgo_seeds.restype = u64
        L.mgo_seeds.argtypes = [vp, cp, vp, cp, u64, i, vp, u64, vp]
        L.mgo_align_tsv.restype = vp
        L.mgo_align_tsv.argtypes = [vp, cp, vp, ctypes.POINTER(cp), ctypes.POINTER(cp), u64, i, i, vp]
        L.mgo_align_budget_trace.restype = ctypes.POINTER(u64)
        L.mgo_align_budget_trace.argtypes = [vp, cp, vp, ctypes.POINTER(cp), u64, vp]
        L.mgo_free.argtypes = [vp]
        _lib = L
    return _lib


class Stats(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in
                ("num_seeds", "num_extensions", "num_explored_nodes", "dp_cells", "dp_columns")]


class OracleGraph:
    """DBGSuccinct restatement. mask=True mimics the unit-test graphs (dummy k-mers masked),
    mask=False mimics `metagraph align` (mask dropped, cli/align.cpp:335-339)."""

    def __init__(self, k, seqs=None, alphabet="dna", mask=False, suffix_index=0, arrays=None,
                 dynamic=False):
        import numpy as np
        self.k = k
        self.alphabet = alphabet.encode()
        L = lib()
        if arrays is not None:
            W, last, F = arrays
            W = np.ascontiguousarray(W, dtype=np.uint8)
            last = np.ascontiguousarray(last, dtype=np.uint8)
            F = np.ascontiguousarray(F, dtype=np.uint64)
            self.h = L.mgo_graph_from_arrays(self.alphabet, k, W.ctypes.data, last.ctypes.data,
                                             len(W), F.ctypes.data, suffix_index)
        else:
            arr = (ctypes.c_char_p * len(seqs))(*[s.encode() for s in seqs])
            self.h = L.mgo_graph_build(self.alphabet, k, arr, len(seqs), int(mask), suffix_index,
                                       int(dynamic))
        if not self.h:
            raise RuntimeError("oracle graph construction failed")

    def set_mode(self, mode):
        """0 = BASIC, 1 = CANONICAL (graph built from the sequences plus their reverse complements),
        2 = PRIMARY (graph built from primary contigs; the aligner wraps it into CanonicalDBG)"""
        lib().mgo_graph_set_mode(self.h, int(mode))

    def __del__(self):
        if getattr(self, "h", None):
            lib().mgo_graph_free(self.h)
            self.h = None

    @property
    def num_edges(self):
        return lib().mgo_graph_num_edges(self.h)

    @property
    def num_nodes(self):
        return lib().mgo_graph_num_nodes(self.h)

    def set_mask(self, on):
        lib().mgo_graph_mask_dummy(self.h, int(on))

    def arrays(self):
        import numpy as np
        n1 = self.num_edges + 1
        sigma = 27 if self.alphabet == b"protein" else 5
        W = np.zeros(n1, np.uint8); last = np.zeros(n1, np.uint8)
        F = np.zeros(sigma, np.uint64); valid = np.zeros(n1, np.uint8)
        lib().mgo_graph_get_arrays(self.h, W.ctypes.data, last.ctypes.data, F.ctypes.data,
                                   valid.ctypes.data)
        return W, last, F, valid

    def map_to_nodes(self, seq):
        import numpy as np
        out = np.zeros(max(1, len(seq)), np.uint64)
        n = lib().mgo_map_to_nodes(self.h, seq.encode(), len(seq), out.ctypes.data)
        return out[:n].copy()

    def suffix_match_first(self, s, min_match_length):
        """first node of call_nodes_with_suffix_matching_longest_prefix (0: none)"""
        f = lib().mgo_suffix_match_first
        f.restype = ctypes.c_uint64
        f.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint64]
        return int(f(self.h, s.encode(), len(s), min_match_length))

    def outgoing(self, node, rc=False):
        import numpy as np
        nodes = np.zeros(64, np.uint64)
        chars = ctypes.create_string_buffer(64)
        n = lib().mgo_call_outgoing(self.h, int(node), int(rc), nodes.ctypes.data, chars)
        return [(int(nodes[j]), chars.raw[j:j + 1].decode()) for j in range(n)]

    def node_sequence(self, node):
        buf = ctypes.create_string_buffer(self.k + 8)
        lib().mgo_node_sequence(self.h, int(node), buf)
        return buf.value.decode()

    def seeds(self, cfg, seq, orientation=False):
        import numpy as np
        c = cfg.to_c()
        out = np.zeros(5 * 65536, np.uint64)
        nm = ctypes.c_uint64(0)
        n = lib().mgo_seeds(self.h, self.alphabet, ctypes.byref(c), seq.encode(), len(seq),
                            int(orientation), out.ctypes.data, 65536, ctypes.byref(nm))
        return [tuple(int(x) for x in out[5 * j:5 * j + 5]) for j in range(min(n, 65536))], nm.value

    def align_tsv(self, cfg, reads, headers=None, threads=1, with_nodes=False, stats=None):
        """Returns one TSV line (without the newline) per read."""
        c = cfg.to_c()
        n = len(reads)
        headers = headers or [""] * n
        H = (ctypes.c_char_p * n)(*[h.encode() for h in headers])
        S = (ctypes.c_char_p * n)(*[s.encode() if isinstance(s, str) else s for s in reads])
        st = Stats()
        p = lib().mgo_align_tsv(self.h, self.alphabet, ctypes.byref(c), H, S, n, threads,
                                int(with_nodes), ctypes.byref(st))
        txt = ctypes.string_at(p).decode()
        lib().mgo_free(p)
        if txt.startswith("ERROR:"):
            raise RuntimeError(txt)
        if stats is not None:
            stats.update({k: getattr(st, k) for k, _ in Stats._fields_})
        lines = txt.split("\n")
        assert lines[-1] == ""
        return lines[:-1]

    def budget_trace(self, cfg, reads):
        """Every evaluation of the extender's node and RAM budgets, per read: a list with one (n, 3) uint64 array
        per read whose rows are (table_size_bytes_, table.size(), window.size()) at the stop tests."""
        import numpy as np
        c = cfg.to_c()
        n = len(reads)
        S = (ctypes.c_char_p * n)(*[s.encode() if isinstance(s, str) else s for s in reads])
        ends = np.zeros(max(1, n), np.uint64)
        p = lib().mgo_align_budget_trace(self.h, self.alphabet, ctypes.byref(c), S, n, ends.ctypes.data)
        if not p:
            raise RuntimeError("oracle aligner failed")
        total = int(ends[n - 1]) if n else 0
        flat = np.ctypeslib.as_array(p, shape=(max(1, 3 * total),))[:3 * total].reshape(total, 3).copy()
        lib().mgo_free(ctypes.cast(p, ctypes.c_void_p))
        bounds = [0] + [int(e) for e in ends[:n]]
        return [flat[bounds[i]:bounds[i + 1]] for i in range(n)]


def is_low_complexity(seq):
    """oracle restatement of sdust(seq, T=20, W=64) finding at least one interval"""
    b = seq.encode() if isinstance(seq, str) else seq
    return bool(lib().mgo_is_low_complexity(b, len(b)))


def parse_tsv_line(line, with_nodes=False):
    """-> (header, query, [alignments]) each alignment = dict(strand, seq, score, nm, cigar, offset[, nodes])"""
    f = line.split("\t")
    header, query = f[0], f[1]
    rest = f[2:]
    alns = []
    if rest[:2] == ["*", "*"]:
        return header, query, alns
    n_aln = len(rest) // (7 if with_nodes else 6)
    for a in range(n_aln):
        r = rest[6 * a:6 * a + 6]
        d = dict(strand=r[0], seq=r[1], score=int(r[2]), nm=int(r[3]), cigar=r[4], offset=int(r[5]))
        if with_nodes:
            d["nodes"] = [int(x) for x in rest[6 * n_aln + a].split(",") if x]
        alns.append(d)
    return header, query, alns
