"""What each table of a built index must hold, restated on the host in numpy from W, last, F and the dummy mask alone.

The tables (index.cuh IndexView) are read through the test library's accessor (tests/devtables/index_tables.cu):
libmgb_tables.so on the GPU, libmgb_emu.so in the host emulation. Each check_* function raises AssertionError with
the first entry that breaks its contract. Notation: x(e) is the k-mer of edge e, "clean" if it holds no '$';
key(e) = sum_p (code_p - 1) << 2p; P = {e : in_graph(e) and x(e) clean} are the DBG nodes the seeding walk stores;
K is the set of keys of the clean k-mers. The contracts never compare hash slot positions or path positions between
builds: both come from atomic races on the device.
"""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES_LIB = os.path.join(ROOT, "tests", "devtables", "build", "libmgb_tables.so")
EMU_LIB = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")

PL_NONE = 0xFFFFFFFF      # index.cuh kPlNone
PL_PAD = 256              # index.cuh kPlPad
KEY_FLAG = np.uint64(1 << 63)


class IndexInfo(ctypes.Structure):
    _fields_ = [("n", ctypes.c_uint64), ("kh_slots", ctypes.c_uint64), ("pl_n", ctypes.c_uint64),
                ("k", ctypes.c_uint32), ("sigma", ctypes.c_uint32), ("wide", ctypes.c_uint32),
                ("mode", ctypes.c_uint32), ("sfx_len", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


# table name -> (dtype, entries per row)
TABLES = {"adj": (np.uint32, 2), "wadj": (np.uint32, 4), "radj": (np.uint32, 2), "kh_keys": (np.uint64, 1),
          "kh_vals": (np.uint32, 1), "pl_node": (np.uint32, 1), "pl_pos": (np.uint32, 1), "pl_text": (np.uint64, 1),
          "pl_rc": (np.uint32, 1), "pl_stop": (np.uint32, 1), "sfx": (np.uint32, 1), "rcs": (np.uint32, 1),
          "rcp": (np.uint32, 1), "palin": (np.uint32, 1), "valid": (np.uint32, 1)}


def _accessor(L):
    if not getattr(L, "_mgbt_ready", False):
        L.mgbt_index_info.restype = ctypes.c_int
        L.mgbt_index_info.argtypes = [ctypes.c_void_p, ctypes.POINTER(IndexInfo)]
        L.mgbt_index_copy.restype = ctypes.c_int64
        L.mgbt_index_copy.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p,
                                      ctypes.c_uint64]
        L._mgbt_ready = True
    return L


def index_info(idx):
    L = _accessor(idx._L)
    info = IndexInfo()
    assert L.mgbt_index_info(idx.handle, ctypes.byref(info)) == 0, L.mgb_last_error().decode()
    return info


def table_bytes(idx, name):
    L = _accessor(idx._L)
    size = L.mgbt_index_copy(idx.handle, name.encode(), 0, None, 0)
    assert size >= 0, L.mgb_last_error().decode()
    return size


def read_table(idx, name, first=0, count=None):
    """host copy of table `name` (rows first .. first + count), None if the index does not hold it"""
    L = _accessor(idx._L)
    dtype, width = TABLES[name]
    row = np.dtype(dtype).itemsize * width
    size = table_bytes(idx, name)
    if size == 0:
        return None
    if count is None:
        count = size // row - first
    out = np.empty((count, width) if width > 1 else count, dtype)
    if count:
        got = L.mgbt_index_copy(idx.handle, name.encode(), first * row, out.ctypes.data, count * row)
        assert got == size, L.mgb_last_error().decode()
    return out


def read_tables(idx, names=None):
    return {nm: read_table(idx, nm) for nm in (names or TABLES)}


# ---------------------------------------------------------------------------------------------------------------
# packed k-mers
# ---------------------------------------------------------------------------------------------------------------
def revcomp_keys(keys, length):
    """reverse complement of 2-bit packed strings of `length` characters (position p in bits 2p, 2p + 1)"""
    x = keys.astype(np.uint64)
    for shift, mask in ((2, 0x3333333333333333), (4, 0x0F0F0F0F0F0F0F0F), (8, 0x00FF00FF00FF00FF),
                        (16, 0x0000FFFF0000FFFF), (32, 0x00000000FFFFFFFF)):
        m = np.uint64(mask)
        x = ((x >> np.uint64(shift)) & m) | ((x & m) << np.uint64(shift))
    x = x >> np.uint64(64 - 2 * length)
    return x ^ np.uint64((1 << (2 * length)) - 1)


def kh_slot_of(keys, slots):
    """index.cuh kh_slot_of: the high 64 bits of a 64 x 64-bit product, from 32-bit halves"""
    m = np.uint64(slots >> 2)
    assert slots >> 2 < 1 << 32
    with np.errstate(over="ignore"):
        h = keys.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    x = h ^ (h >> np.uint64(29))
    lo, hi = x & np.uint64(0xFFFFFFFF), x >> np.uint64(32)
    return (((hi * m) + ((lo * m) >> np.uint64(32))) >> np.uint64(32)) << np.uint64(2)


def member(sorted_keys, q):
    i = np.searchsorted(sorted_keys, q)
    i[i == len(sorted_keys)] = 0
    return (sorted_keys[i] == q) if len(sorted_keys) else np.zeros(len(q), bool)


def bits_of(words, n_bits):
    """bit q of a little-endian uint32 bit array, for q < n_bits"""
    return np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")[:n_bits].astype(bool)


# ---------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------
class Reference:
    """The graph's per-edge facts, from W / last / F / valid only (BOSS semantics, boss.cpp):
      rnode[e]   rank of e's source node; ones[r - 1] its last edge
      nlv[e]     last character of e's source node
      tnode[e]   rank of the node fwd(e) enters (0: none: a '$' edge other than the root's)
      bwd[e]     the un-flagged edge entering e's source node (1 at the root)
      first[e]   x(e)[0]; clean[e]; key[e] (DNA); sidx[e] the suffix-table index of the source node's last s
                 characters (-1 if they hold '$')"""

    def __init__(self, W, last, F, k, valid=None, sfx_len=0, keep_codes=False):
        W = np.asarray(W, np.uint8)
        self.k = k = int(k)
        self.sigma = sigma = len(F)
        self.n = n = len(W) - 1
        self.F = F = np.asarray(F, np.uint64).astype(np.int64)
        pos = np.arange(n + 1, dtype=np.int64)
        lastb = np.asarray(last, np.uint8).astype(bool)
        lastb[0] = False
        rank_last = np.cumsum(lastb)                         # set bits in [1, i]
        self.ones = np.flatnonzero(lastb)
        self.num_nodes = len(self.ones)
        self.rnode = np.concatenate([[0], rank_last[:-1] + 1])
        nlv = np.searchsorted(F, pos, side="left") - 1          # boss.cpp:679-690: largest c with F[c] < i
        nlv[0] = 0
        self.nlv = nlv.astype(np.uint8)
        self.label = (W % sigma).astype(np.uint8)
        self.label[0] = 0
        NF = rank_last[F]
        # fwd (boss.cpp:642-652): the j-th un-flagged c enters the (NF[c] + j)-th node; flagged edges share the target of
        # the un-flagged one before them
        rank_w = np.zeros(n + 1, np.int64)
        for c in range(sigma):
            cnt = np.cumsum(W == c)
            cnt -= int(W[0] == c)
            m = self.label == c
            rank_w[m] = cnt[m]
        tnode = NF[self.label.astype(np.int64)] + rank_w
        has = (self.label != 0) | (rank_w == 1)                 # '$' edges: only the root's (the first un-flagged '$')
        has[0] = False
        tnode[~has] = 0
        tnode[(tnode < 1) | (tnode > self.num_nodes)] = 0
        self.tnode = tnode
        bwd_node = np.zeros(self.num_nodes + 1, np.int64)
        enter = (W < sigma) & (self.label != 0) & (tnode > 0)
        enter[0] = False
        bwd_node[tnode[enter]] = pos[enter]
        self.bwd = bwd_node[self.rnode]
        self.bwd[self.rnode == 1] = 1
        self.bwd[0] = 0
        assert (bwd_node[2:] > 0).all(), "a node other than the root without an un-flagged incoming edge"
        # incoming edges per node, counted from fwd
        indeg = np.bincount(tnode[tnode > 0], minlength=self.num_nodes + 1)
        self.multi = indeg[self.rnode] > 1
        self.multi[0] = False
        self.valid = None if valid is None else np.asarray(valid, np.uint8).astype(bool)
        self.in_graph = np.ones(n + 1, bool) if valid is None else self.valid.copy()
        self.in_graph[0] = False
        # the k-mers: node characters from the last one backwards through bwd, the label last
        self.sfx_len = s = min(int(sfx_len), k - 1)
        dna = sigma == 5 and k <= 32                            # keys in 64 bits
        lab =self.label.astype(np.uint64)
        self.clean = self.label != 0
        tail_ok = np.ones(n + 1, bool)                          # node characters 1 .. k - 2 clean
        key =np.where(lab > 0, lab - np.uint64(1), 0).astype(np.uint64) << np.uint64(2 * (k - 1)) if dna else None
        sidx = np.zeros(n + 1, np.int64)
        sclean = np.ones(n + 1, bool)
        codes = np.zeros((n + 1, k), np.uint8) if keep_codes else None
        if keep_codes:
            codes[:, k - 1] = self.label
        cur = pos.copy()
        for t in range(k - 1):
            p = k - 2 - t                                       # node position
            c = self.nlv[cur]
            if keep_codes:
                codes[:, p] = c
            nz = c != 0
            self.clean &= nz
            if p >= 1:
                tail_ok &= nz
            if dna:
                key |= np.where(nz, c.astype(np.uint64) - np.uint64(1), 0).astype(np.uint64) << np.uint64(2 * p)
            if t < s:
                sclean &= nz
                sidx += np.where(nz, c.astype(np.int64) - 1, 0) * (sigma - 1) ** (s - 1 - t)
            if t + 1 < k - 1:
                cur = self.bwd[cur]
        self.first = c
        self.clean_suffix = (self.label != 0) & tail_ok         # x[1..k) clean
        self.node_clean = (self.first != 0) & tail_ok           # x[0..k-1) clean
        self.clean[0] = self.clean_suffix[0] = self.node_clean[0] = False
        self.codes = codes
        self.key = key
        self.sidx = np.where(sclean, sidx, -1) if s else None
        if self.sidx is not None:
            self.sidx[0] = -1
        self.P = self.in_graph & self.clean
        if dna:
            ck = key[self.clean]
            self.K = np.sort(ck)
            assert len(np.unique(self.K)) == len(self.K), "two clean edges spell the same k-mer"

    def kmer_strings(self, edges):
        alph = "$ACGT" if self.sigma == 5 else "$ABCDEFGHIJKLMNOPQRSTUVWYZX"
        return ["".join(alph[c] for c in self.codes[e]) for e in edges]

    # --- forward adjacency records (index_build.hpp) ---
    @property
    def adj(self):
        if getattr(self, "_adj", None) is None:
            self._adj = self.adj_expected()
        return self._adj

    def adj_expected(self):
        """(x, all, ok) per edge: last edge of the target node, the target node's labels, the labels of its edges that
        are valid non-'$' DBG nodes; nothing for '$' edges other than edge 1"""
        n, sig = self.n, self.sigma
        lab = self.label.astype(np.int64)
        w_all = np.bincount(self.rnode[1:], weights=(1 << lab[1:]).astype(np.float64), minlength=self.num_nodes + 1)
        okm = (lab != 0) & self.in_graph
        okm[0] = False
        w_ok = np.bincount(self.rnode[1:], weights=np.where(okm[1:], 1 << lab[1:], 0).astype(np.float64),
                           minlength=self.num_nodes + 1)
        w_all, w_ok = w_all.astype(np.uint32), w_ok.astype(np.uint32)
        x = np.zeros(n + 1, np.uint32)
        a = np.zeros(n + 1, np.uint32)
        o = np.zeros(n + 1, np.uint32)
        t = self.tnode
        m = (t > 0) & ((self.label != 0) | (np.arange(n + 1) == 1))
        x[m] = self.ones[t[m] - 1]
        a[m] = w_all[t[m]]
        o[m] = w_ok[t[m]]
        assert sig <= 32
        return x, a, o

    def adj_children(self, x, a, c):
        """index.cuh adj_child for label c of every record"""
        has = (x > 0) & (((a >> np.uint32(c)) & np.uint32(1)) > 0)
        below = a & np.uint32((1 << c) - 1)
        pa, pb = np.bitwise_count(a).astype(np.int64), np.bitwise_count(below).astype(np.int64)
        child = x.astype(np.int64) - pa + 1 + pb
        return np.where(has, child, 0)

    def rc_in_K(self, edges):
        return member(self.K, revcomp_keys(self.key[edges], self.k))

    # --- path layout ---
    def path_links(self):
        """kept links e -> c of the path layout (0: none) and the number of cycles cut"""
        x, a, o = self.adj
        e = np.flatnonzero(self.P)
        okm = o[e]
        single = np.bitwise_count(okm) == 1
        e = e[single]
        lab = (np.log2(okm[single].astype(np.float64))).astype(np.int64)
        child = np.zeros(len(e), np.int64)
        for c in range(1, 5):
            m = lab == c
            child[m] = self.adj_children(x[e[m]], a[e[m]], c)
        keep = (child > 0) & self.clean[child]
        e, child = e[keep], child[keep]
        # pred(c) = the smallest e linking to c (e is ascending)
        _, firsts = np.unique(child, return_index=True)
        link = np.zeros(self.n + 1, np.int64)
        link[e[firsts]] = child[firsts]
        # cycles: components of kept links without a head (every node of one has a kept incoming link)
        import scipy.sparse as sp
        from scipy.sparse.csgraph import connected_components
        src = np.flatnonzero(link)
        g = sp.coo_matrix((np.ones(len(src), np.int8), (src, link[src])), shape=(self.n + 1, self.n + 1)).tocsr()
        _, comp = connected_components(g, directed=False)
        has_in = np.zeros(self.n + 1, bool)
        has_in[link[src]] = True
        head = self.P & ~has_in
        comp_has_head = np.zeros(comp.max() + 1, bool)
        comp_has_head[comp[head]] = True
        on_cycle = self.P & ~comp_has_head[comp]
        cyc = np.flatnonzero(on_cycle)
        n_cycles = 0
        if len(cyc):
            smallest = np.full(comp.max() + 1, np.iinfo(np.int64).max)
            np.minimum.at(smallest, comp[cyc], cyc)
            into_min = cyc[link[cyc] == smallest[comp[cyc]]]
            n_cycles = len(into_min)
            link[into_min] = 0
        return link, n_cycles


def reference_for(boss, valid=None, sfx_len=0, keep_codes=False):
    return Reference(boss.W, boss.last, boss.F, boss.k, valid=valid, sfx_len=sfx_len, keep_codes=keep_codes)


# ---------------------------------------------------------------------------------------------------------------
# checkers
# ---------------------------------------------------------------------------------------------------------------
def _first_bad(mask, what, *cols):
    bad = np.flatnonzero(mask)
    if len(bad):
        i = bad[0]
        raise AssertionError("%s: %d entries, first at %d: %s" % (what, len(bad), i,
                                                                    ", ".join(str(c[i]) for c in cols)))


def check_radj(ref, T, info):
    r = T["radj"]
    assert r is not None, "radj: absent"
    assert r.shape == (ref.n + 1, 2), "radj: shape %s" % (r.shape,)
    shift = 7 if info.wide else 3
    exp_y = ref.first.astype(np.uint32) | (ref.multi.astype(np.uint32) << np.uint32(shift))
    e = np.arange(ref.n + 1)
    _first_bad(r[1:, 0] != ref.bwd[1:], "radj bwd", e[1:], r[1:, 0], ref.bwd[1:])
    char_mask = np.uint32((1 << shift) - 1)
    _first_bad((r[1:, 1] & char_mask) != ref.first[1:], "radj first character", e[1:], r[1:, 1], ref.first[1:])
    _first_bad(r[1:, 1] != exp_y[1:], "radj several-incoming flag", e[1:], r[1:, 1], exp_y[1:])


def check_adj(ref, T, info, hashed):
    """bits 0..15 of the DNA records (or the generic layout's wadj), and the reverse-complement bits 16..20"""
    x, a, o = ref.adj
    e = np.arange(ref.n + 1)
    if info.wide:
        w = T["wadj"]
        assert w is not None and T["adj"] is None, "wadj: absent"
        got = w[1:]
        _first_bad((got[:, 0] != x[1:]) | (got[:, 1] != a[1:]) | (got[:, 2] != o[1:]) | (got[:, 3] != 0),
                   "wadj", e[1:], got[:, 0], got[:, 1], got[:, 2], x[1:], a[1:], o[1:])
        return
    r = T["adj"]
    assert r is not None, "adj: absent"
    low = a | (o << np.uint32(8))
    _first_bad((r[1:, 0] != x[1:]) | ((r[1:, 1] & np.uint32(0xFFFF)) != low[1:]), "adj bits 0..15",
               e[1:], r[1:, 0], r[1:, 1], x[1:], low[1:])
    rc = np.zeros(ref.n + 1, np.uint32)
    if hashed:
        for c in range(1, 5):
            ch = ref.adj_children(x, a, c)
            has = np.flatnonzero(ch)
            chs = ch[has]
            bit = ~ref.clean[chs]
            cl = ref.clean[chs]
            bit[cl] = ref.rc_in_K(chs[cl])
            rc[has[bit]] |= np.uint32(1 << (16 + c))
    high = r[1:, 1] & np.uint32(0xFFFF0000)
    _first_bad(high != rc[1:], "adj reverse-complement bits", e[1:], r[1:, 1], rc[1:])


def kh_slots_for(n):
    """api.cu: a load factor of 0.7 plus 64 slots, in whole buckets of 4"""
    return ((int((n + 1) / 0.7) + 64) + 3) & ~3


def check_hash(ref, T, info, rng=None):
    """returns the longest probe (slots read by one lookup)"""
    keys, vals = T["kh_keys"], T["kh_vals"]
    assert keys is not None and vals is not None, "hash index: absent"
    S = int(info.kh_slots)
    assert S == kh_slots_for(ref.n) and len(keys) == S and len(vals) == S, "kh_slots %d, expected %d" % (
        S, kh_slots_for(ref.n))
    occ = keys != 0
    sk = keys[occ]
    assert ((sk & KEY_FLAG) != 0).all(), "hash keys: a key without bit 63"
    got = np.sort(sk & ~KEY_FLAG)
    assert len(got) == len(ref.K), "hash keys: %d keys, %d clean k-mers" % (len(got), len(ref.K))
    d = np.flatnonzero(got != ref.K)
    assert not len(d), "hash keys: key set differs, first at sorted position %d: %x vs %x" % (d[0], got[d[0]],
                                                                                            ref.K[d[0]])
    # kh_vals: the key's edge
    edges = np.flatnonzero(ref.clean)
    order = np.argsort(ref.key[edges], kind="stable")
    key_sorted, edge_sorted = ref.key[edges][order], edges[order]
    slot = np.flatnonzero(occ)
    exp = edge_sorted[np.searchsorted(key_sorted, sk & ~KEY_FLAG)]
    _first_bad(vals[slot] != exp, "kh_vals", slot, vals[slot], exp)
    # no empty slot between a key's home and its slot
    home = kh_slot_of(sk, S).astype(np.int64)
    E = np.concatenate([[0], np.cumsum(~occ)])
    empties = np.where(home <= slot, E[slot] - E[home], E[S] - E[home] + E[slot])
    _first_bad(empties != 0, "hash probe chain: an empty slot before the key", slot, home, empties)
    # lookups: every key finds its edge, as many keys outside K find nothing
    got_e, probes = kh_lookup(keys, vals, ref.K | KEY_FLAG)
    exp_e = edge_sorted[np.searchsorted(key_sorted, ref.K)]
    _first_bad(got_e != exp_e, "kh_lookup of a key", ref.K, got_e, exp_e)
    rng = rng or np.random.default_rng(1)
    kmask = np.uint64((1 << (2 * ref.k)) - 1)
    miss = rng.integers(0, 1 << 63, size=len(ref.K), dtype=np.uint64) & kmask
    miss = miss[~member(ref.K, miss)]
    got_m, probes_m = kh_lookup(keys, vals, miss | KEY_FLAG)
    _first_bad(got_m != 0, "kh_lookup of a key not in the graph", miss, got_m)
    return int(max(probes.max(initial=0), probes_m.max(initial=0)))


def kh_lookup(keys, vals, q):
    """index.cuh kh_lookup for every query (with bit 63): (edge or 0, slots read)"""
    S = len(keys)
    res = np.zeros(len(q), np.int64)
    probes = np.zeros(len(q), np.int64)
    i = kh_slot_of(q, S).astype(np.int64)
    act = np.arange(len(q))
    step = 0
    while len(act):
        step += 1
        s = keys[i]
        hit = s == q[act]
        res[act[hit]] = vals[i[hit]]
        done = hit | (s == 0)
        probes[act[done]] = step
        act, i = act[~done], i[~done] + 1
        i[i == S] = 0
        assert step <= S, "kh_lookup: no empty slot in the table"
    return res, probes


def check_paths(ref, T, info):
    """returns (number of paths, number of cycles cut)"""
    node, pos, text, rcb, stop = T["pl_node"], T["pl_pos"], T["pl_text"], T["pl_rc"], T["pl_stop"]
    assert node is not None, "path layout: absent"
    N, k = int(info.pl_n), ref.k
    assert N % 64 == 0 and N >= PL_PAD and len(node) == N, "pl_n %d" % N
    assert len(pos) == ref.n + 1 and len(text) == N // 32 and len(rcb) == N // 32 and len(stop) == N // 32
    e = np.arange(ref.n + 1)
    placed = pos != PL_NONE
    _first_bad(placed != ref.P, "pl_pos: placed iff a DBG node with a clean k-mer", e, pos, ref.P)
    P = np.flatnonzero(ref.P)
    p = pos[P].astype(np.int64)
    assert (p < N).all(), "pl_pos past pl_n"
    _first_bad(node[p] != P, "pl_node[pl_pos[e]] != e", P, p, node[p])
    assert np.count_nonzero(node) == len(P), "pl_node: %d nodes, |P| = %d" % (np.count_nonzero(node), len(P))
    assert not node[N - PL_PAD:].any(), "pl_node: the last kPlPad positions are not fillers"
    link, n_cycles = ref.path_links()
    src = np.flatnonzero(link)
    _first_bad(pos[link[src]].astype(np.int64) != pos[src].astype(np.int64) + 1, "path link not kept in place",
               src, link[src], pos[src], pos[link[src]])
    tails = P[link[P] == 0]
    tp = pos[tails].astype(np.int64)
    for j in range(1, k):
        q = tp + j
        _first_bad((q >= N) | (node[np.minimum(q, N - 1)] != 0), "a path end not followed by k - 1 fillers",
                   tails, tp, np.full(len(tails), j))
    # text: x(e) at pl_pos[e] .. + k - 1
    for j in range(k):
        q = p + j
        ch = (text[q >> 5] >> ((q & 31) * 2).astype(np.uint64)) & np.uint64(3)
        exp = (ref.key[P] >> np.uint64(2 * j)) & np.uint64(3)
        _first_bad(ch != exp, "pl_text", P, p, np.full(len(P), j), ch, exp)
    is_node = node != 0
    _first_bad(bits_of(stop, N) != ~is_node, "pl_stop", np.arange(N), node)
    exp_rc = np.zeros(N, bool)
    exp_rc[p] = ref.rc_in_K(P)
    _first_bad(bits_of(rcb, N) != exp_rc, "pl_rc", np.arange(N), node)
    heads = len(P) - len(src)
    return heads, n_cycles


def check_sfx(ref, T, info, sample=None):
    """the suffix-range table at its deepest level; `sample`: check these entries only (T["sfx"] then holds their
    pairs, in the same order)"""
    s, sig = int(info.sfx_len), ref.sigma
    assert s == ref.sfx_len, "sfx_len %d, expected %d" % (s, ref.sfx_len)
    if s == 0:
        assert T["sfx"] is None
        return
    entries = (sig - 1) ** s
    e = np.flatnonzero(ref.sidx >= 0)
    v = ref.sidx[e]
    order = np.argsort(v, kind="stable")
    vs, es = v[order], e[order]
    uniq, starts, counts = np.unique(vs, return_index=True, return_counts=True)
    lo, hi = es[starts], es[starts + counts - 1]
    _first_bad(hi - lo + 1 != counts, "suffix ranges: edges with one s-mer not contiguous", uniq, lo, hi, counts)
    idx = np.arange(entries) if sample is None else np.asarray(sample, np.int64)
    got = np.asarray(T["sfx"], np.int64).reshape(-1, 2)
    assert len(got) == len(idx), "sfx: %d entries, expected %d" % (len(got), len(idx))
    if not len(uniq):
        uniq = lo = hi = np.zeros(1, np.int64) - 1
    j = np.searchsorted(uniq, idx)
    j[j == len(uniq)] = 0
    present = uniq[j] == idx
    eb = np.where(present, lo[j], 1)
    ee = np.where(present, hi[j] + 1, 1)
    bad = np.where(present, (got[:, 0] != eb) | (got[:, 1] != ee), got[:, 0] < got[:, 1])
    _first_bad(bad, "sfx range", idx, got[:, 0], got[:, 1], eb, ee)


def check_rc_tables(ref, T, info):
    """PRIMARY graphs: rcs / rcp / palin"""
    k, n = ref.k, ref.n
    rcs, rcp, pal = T["rcs"], T["rcp"], T["palin"]
    assert rcs is not None and rcp is not None, "rc tables: absent"
    # node (k - 1)-mer -> its last edge, over the nodes whose characters are all clean
    nmask = np.uint64((1 << (2 * (k - 1))) - 1)
    last_e = ref.ones
    cl = ref.node_clean[last_e]
    nk = ref.key[last_e[cl]] & nmask
    order = np.argsort(nk)
    nk, ne = nk[order], last_e[cl][order]

    def find(q):
        j = np.searchsorted(nk, q)
        j[j == len(nk)] = 0
        return np.where(nk[j] == q, ne[j], 0) if len(nk) else np.zeros(len(q), np.int64)

    e = np.arange(n + 1)
    exp_s = np.zeros(n + 1, np.int64)
    m = ref.clean_suffix.copy()
    exp_s[m] = find(revcomp_keys(ref.key[m] >> np.uint64(2), k - 1))
    exp_p = np.zeros(n + 1, np.int64)
    m = ref.node_clean.copy()
    exp_p[m] = find(revcomp_keys(ref.key[m] & nmask, k - 1))
    _first_bad(rcs[1:] != exp_s[1:], "rcs", e[1:], rcs[1:], exp_s[1:])
    _first_bad(rcp[1:] != exp_p[1:], "rcp", e[1:], rcp[1:], exp_p[1:])
    if k % 2:
        assert pal is None, "palin on an odd k"
        return
    assert pal is not None, "palin: absent"
    exp_pal = ref.clean & (revcomp_keys(ref.key, k) == ref.key)
    got = bits_of(pal, n + 1)
    _first_bad(got != exp_pal, "palin", e, got, exp_pal)


def check_index(ref, T, info, hashed, paths=None, primary=False):
    """every contract of an index; returns a dict of what was measured"""
    out = {"n": ref.n}
    assert info.n == ref.n and info.k == ref.k and info.sigma == ref.sigma
    check_radj(ref, T, info)
    check_adj(ref, T, info, hashed)
    check_sfx(ref, T, info)
    if hashed:
        out["keys"] = len(ref.K)
        out["longest_probe"] = check_hash(ref, T, info)
    else:
        assert info.kh_slots == 0 and T["kh_keys"] is None, "a hash index where none belongs"
    if paths is None:
        paths = hashed
    if paths:
        out["paths"], out["cycles"] = check_paths(ref, T, info)
    else:
        assert info.pl_n == 0 and T["pl_node"] is None, "a path layout where none belongs"
    if primary:
        check_rc_tables(ref, T, info)
    return out


# ---------------------------------------------------------------------------------------------------------------
# graphs with the shapes where the build kernels can go wrong
# ---------------------------------------------------------------------------------------------------------------
def random_seq(rng, n, alphabet="ACGT"):
    return "".join(np.array(list(alphabet))[rng.integers(0, len(alphabet), n)])


def revcomp(s):
    return s.translate(str.maketrans("ACGT", "TGCA"))[::-1]


def mutate(rng, s, rate, alphabet="ACGT"):
    a = np.array(list(s))
    hit = rng.random(len(a)) < rate
    a[hit] = np.array(list(alphabet))[rng.integers(0, len(alphabet), int(hit.sum()))]
    return "".join(a)


def shape_seqs(shape, k, rng, size=6000):
    """sequences of a graph of the given shape"""
    base = random_seq(rng, size)
    if shape == "mutated":                       # a genome and a 2 % mutated copy: many path ends
        return [base, mutate(rng, base, 0.02)]
    if shape == "tandem":                        # a cycle with a way in and out, and a lone cycle with no head
        unit = random_seq(rng, max(1, k // 2 + 1))
        lone = random_seq(rng, max(1, k // 3 + 1))
        return [base[:size // 2] + unit * (3 * k // len(unit) + 4) + base[size // 2:],
                lone * (3 * k // len(lone) + 3)]
    if shape == "homopolymer":                   # k-mers that are their own child
        return [base[:1000] + "A" * (2 * k + 5) + base[1000:2000] + "C" * (k + 1) + base[2000:3000] + "G" * 3 * k]
    if shape == "circular":
        return [base[:2000] + base[:k - 1]]
    if shape == "both_orientations":
        return [base, revcomp(base[1000:3000])]
    if shape == "palindromes":                   # k-mers that are their own reverse complement (even k)
        s = list(base)
        for _ in range(60):
            h = random_seq(rng, k // 2)
            p = int(rng.integers(0, len(s) - k))
            s[p:p + k] = list(h + revcomp(h))
        return ["".join(s)]
    if shape == "short_seqs":                    # many source and sink dummies
        return [random_seq(rng, int(rng.integers(k, 3 * k + 2))) for _ in range(400)]
    if shape == "one_kmer":
        return [base[:k]]
    if shape == "empty":
        return []
    raise ValueError(shape)


def protein_seqs(rng, n_seq=40, length=400):
    aa = "ACDEFGHIKLMNPQRSTVWY"
    base = [random_seq(rng, length, aa) for _ in range(n_seq)]
    return base + [mutate(rng, s, 0.05, aa) for s in base[:10]]


def build_index(lib, k, seqs, mask=False, suffix_len=0, mode=0, alphabet=0, boss=None):
    """(boss, valid or None, index) from the given library"""
    from metagraph_b200.aligner import BOSSTable, DBGSuccinctIndex
    if boss is None:
        boss = BOSSTable.from_sequences(k, seqs, lib=lib, alphabet=alphabet)
    valid = boss.dummy_mask(lib=lib) if mask else None
    idx = DBGSuccinctIndex(boss, valid=valid, suffix_len=suffix_len, lib=lib, mode=mode)
    return boss, valid, idx


# ---------------------------------------------------------------------------------------------------------------
# corruptions of host copies: every checker must reject each one
# ---------------------------------------------------------------------------------------------------------------
def _copy(T):
    return {k: (None if v is None else v.copy()) for k, v in T.items()}


def corruptions(ref, T, info, rng):
    """(name, corrupted tables, checker, message fragment) for each corruption the tables allow"""
    out = []
    shift = 7 if info.wide else 3
    e = int(rng.integers(1, ref.n + 1))
    for what, f in (("bwd", lambda r: r.__setitem__((e, 0), r[e, 0] + 1)),
                    ("character", lambda r: r.__setitem__((e, 1), r[e, 1] ^ 1)),
                    ("flag", lambda r: r.__setitem__((e, 1), r[e, 1] ^ (1 << shift)))):
        C = _copy(T)
        f(C["radj"])
        out.append(("radj " + what, C, check_radj, "radj"))
    if T["sfx"] is not None:
        C = _copy(T)
        got = C["sfx"].reshape(-1, 2)
        present = np.flatnonzero(got[:, 0] < got[:, 1])
        i = int(present[rng.integers(0, len(present))])
        got[i, int(rng.integers(0, 2))] += 1
        out.append(("sfx bound", C, check_sfx, "sfx range"))
    if T["rcs"] is not None and T["rcs"].any():
        C = _copy(T)
        nz = np.flatnonzero(C["rcs"])
        C["rcs"][nz[rng.integers(0, len(nz))]] = 0
        out.append(("rcs zeroed", C, check_rc_tables, "rcs"))
    if T["palin"] is not None:
        C = _copy(T)
        C["palin"][e >> 5] ^= np.uint32(1 << (e & 31))
        out.append(("palin bit", C, check_rc_tables, "palin"))
    if T["kh_keys"] is None:
        return out
    keys = T["kh_keys"]
    occ = np.flatnonzero(keys)
    i = int(occ[rng.integers(0, len(occ))])
    C = _copy(T)
    C["kh_keys"][i] = 0
    out.append(("key dropped", C, check_hash, "hash keys"))
    C = _copy(T)
    C["kh_vals"][i] ^= 1
    out.append(("kh_vals entry", C, check_hash, "kh_vals"))
    # a key moved behind an empty slot: to the second empty slot after its own
    S = len(keys)
    empty = np.flatnonzero(keys == 0)
    j0 = empty[np.searchsorted(empty, i) % len(empty)]
    j1 = int(empty[(np.searchsorted(empty, j0) + 1) % len(empty)])
    C = _copy(T)
    C["kh_keys"][j1], C["kh_vals"][j1] = keys[i], T["kh_vals"][i]
    C["kh_keys"][i] = 0
    assert S > 8
    out.append(("key behind an empty slot", C, check_hash, "empty slot before the key"))
    # an adj reverse-complement bit, both ways
    a = T["adj"]
    hi = (a[:, 1] >> np.uint32(17)) & np.uint32(15)
    ones = np.flatnonzero(hi)
    if len(ones):
        r = int(ones[rng.integers(0, len(ones))])
        c = int(np.flatnonzero([(int(hi[r]) >> b) & 1 for b in range(4)])[0]) + 1
        C = _copy(T)
        C["adj"][r, 1] ^= np.uint32(1 << (16 + c))
        out.append(("adj rc bit 1 -> 0", C, lambda ref, T, info: check_adj(ref, T, info, True), "reverse-complement"))
    zeros = np.flatnonzero(hi != 15)
    r = int(zeros[rng.integers(0, len(zeros))])
    c = int(np.flatnonzero([((int(hi[r]) >> b) & 1) == 0 for b in range(4)])[0]) + 1
    C = _copy(T)
    C["adj"][r, 1] ^= np.uint32(1 << (16 + c))
    out.append(("adj rc bit 0 -> 1", C, lambda ref, T, info: check_adj(ref, T, info, True), "reverse-complement"))
    if T["pl_node"] is None:
        return out
    pos, node = T["pl_pos"], T["pl_node"]
    P = np.flatnonzero(pos != PL_NONE)
    e1, e2 = (int(x) for x in rng.choice(P, 2, replace=False))
    C = _copy(T)
    C["pl_pos"][e1], C["pl_pos"][e2] = pos[e2], pos[e1]
    C["pl_node"][pos[e1]], C["pl_node"][pos[e2]] = e2, e1
    out.append(("pl_node / pl_pos swap", C, check_paths, ""))
    # a kept link broken: a path's last node moved one position on
    link, _ = ref.path_links()
    src = np.flatnonzero(link)
    tails = src[link[link[src]] == 0]
    if len(tails):
        t = int(link[tails[rng.integers(0, len(tails))]])
        p = int(pos[t])
        C = _copy(T)
        C["pl_node"][p], C["pl_node"][p + 1] = 0, t
        C["pl_pos"][t] = p + 1
        out.append(("kept link broken", C, check_paths, "path link"))
    q = int(pos[e1])
    C = _copy(T)
    C["pl_rc"][q >> 5] ^= np.uint32(1 << (q & 31))
    out.append(("pl_rc bit", C, check_paths, "pl_rc"))
    C = _copy(T)
    C["pl_stop"][q >> 5] ^= np.uint32(1 << (q & 31))
    out.append(("pl_stop bit", C, check_paths, "pl_stop"))
    C = _copy(T)
    C["pl_text"][q >> 5] ^= np.uint64(1 << (2 * (q & 31)))
    out.append(("pl_text character", C, check_paths, "pl_text"))
    return out


def assert_corruptions_rejected(ref, T, info, rng, expect_hash):
    """every corruption of the host copies makes its checker fail; returns the names"""
    names = []
    for name, C, checker, msg in corruptions(ref, T, info, rng):
        try:
            checker(ref, C, info)
        except AssertionError as ex:
            assert msg in str(ex), (name, str(ex))
        else:
            raise AssertionError("corruption not detected: " + name)
        names.append(name)
    want = {"radj bwd", "radj character", "radj flag"}
    if T["sfx"] is not None:
        want.add("sfx bound")
    if expect_hash:
        want |= {"key dropped", "kh_vals entry", "key behind an empty slot", "adj rc bit 0 -> 1", "adj rc bit 1 -> 0",
                 "pl_node / pl_pos swap", "kept link broken", "pl_rc bit", "pl_stop bit", "pl_text character"}
    assert want <= set(names), want - set(names)
    return names


def free_device_memory():
    import torch
    free, total = torch.cuda.mem_get_info(0)
    return "%.1f of %.1f GB free on the device" % (free / 1e9, total / 1e9)


def assert_hashed(idx, boss, valid=None):
    """the index (any library) holds the k-mer hash index: it takes at least 12 bytes per hash slot more device memory
    than the same graph built under MGB_NO_KMER_HASH"""
    from metagraph_b200.aligner import DBGSuccinctIndex
    old = os.environ.get("MGB_NO_KMER_HASH")
    os.environ["MGB_NO_KMER_HASH"] = "1"
    try:
        plain = DBGSuccinctIndex(boss, valid=valid, lib=idx._L._name)
    finally:
        if old is None:
            del os.environ["MGB_NO_KMER_HASH"]
        else:
            os.environ["MGB_NO_KMER_HASH"] = old
    extra = idx.device_bytes - plain.device_bytes
    plain.close()
    assert extra >= 12 * kh_slots_for(boss.num_edges), (
        "the index was built without the k-mer hash index (%d more bytes than without it; %s)"
        % (extra, free_device_memory()))
