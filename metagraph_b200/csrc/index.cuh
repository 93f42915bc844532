// Flat BOSS index in HBM and the rank/select primitives on top of it.
//
// Layout (DNA, sigma = 5): one 64-byte block per 64 consecutive BOSS edges
//     words 0..7   W, 4 bits per edge (edge j: (w[j>>3] >> 4*(j&7)) & 15; 0xF = padding / W[0])
//     words 8..9   `last`, 1 bit per edge
//     word  10     number of set `last` bits before the block
//     words 11..15 number of W == c (c = 0..4, un-flagged) before the block
// so one 64-byte (two sector) access answers get_W, get_last, rank_W and rank_last for any
// position of the block.  A quad (4 consecutive lanes) loads a block with one 16-byte load
// per lane.  Auxiliary arrays: blk_rank (compact copy of word 10), sel_last / sel_W (block
// of every 64th set bit / 32nd occurrence) for select, the optional dummy mask and the
// suffix-range table (boss.hpp:516-525).
//
// Semantics follow graph/representation/succinct/boss.{hpp,cpp} (cited per function);
// only the values returned are observable, the layout is ours.
#pragma once
#include "common.cuh"

#if !defined(__CUDACC__)
struct uint2 { uint32_t x, y; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
#endif

namespace mgb {

static constexpr int kSigmaDNA = 5;
#ifndef MGB_MAX_SIGMA
#define MGB_MAX_SIGMA 32
#endif
static constexpr int kMaxSigma = MGB_MAX_SIGMA;   // alphabet-generic ("wide") layout: sigma <= 32 (protein: 27)
// MGB_WIDE(ix): is the index in the alphabet-generic layout? A translation unit built with
// -DMGB_NARROW_ONLY / -DMGB_WIDE_ONLY serves one layout only and drops the branches (kernels.cuh).
#if defined(MGB_NARROW_ONLY)
#define MGB_WIDE(ix) false
#elif defined(MGB_WIDE_ONLY)
#define MGB_WIDE(ix) true
#else
#define MGB_WIDE(ix) ((ix).wide != 0)
#endif
static constexpr int kBlkEdges = 64;
static constexpr int kBlkWords = 16;
static constexpr int kSelLastRate = 64;
static constexpr int kSelWRate = 32;
static constexpr uint32_t kPlNone = 0xFFFFFFFFu;    // IndexView::pl_pos of an edge that is not a DBG node
static constexpr uint64_t kPlPad = 256;             // filler positions after the last path (a multiple of 64)

struct IndexView {
    const uint32_t *blocks;     // nblk * 16 words
    const uint32_t *blk_rank;   // nblk + 1
    const uint32_t *sel_last;   // ceil(ones / 64) + 1 (sentinel = last block)
    const uint32_t *sel_W[kSigmaDNA];   // per symbol, ceil(cnt / 32) + 1
    const uint32_t *valid;      // bit per edge or nullptr (mask dropped)
    const uint32_t *sfx;        // 2 words per indexed suffix: [begin, end) edge range
    const uint2 *adj;           // per edge: forward adjacency record (see adj_* below), or nullptr
    const uint2 *radj;          // per edge: reverse adjacency record (see load_radj), or nullptr
    // k-mer -> edge hash index (DNA block layout, k <= 31; kh_slots == 0: absent). Open addressing, linear probing:
    // kh_keys[i] = packed k-mer | 1 << 63 (0 = empty), kh_vals[i] = its BOSS edge. What BOSS::map_to_edge
    // (boss.hpp:766-777: index() over k-1 characters, then pick_edge) answers with ~60 dependent block loads, this
    // answers with one or two: HBM capacity traded for latency, as with the adjacency records.
    const unsigned long long *kh_keys;
    const uint32_t *kh_vals;
    uint64_t kh_slots;
    // Path layout (graphs with the k-mer hash index; pl_n == 0: absent). The DBG nodes are covered by disjoint paths
    // (each step from a node to its child), laid out one after another in a position space of pl_n positions, with k - 1
    // filler positions after every path (k_path_* in kernels.cuh builds it):
    //   pl_node[p]  the node whose k-mer starts at position p, 0 at a filler position
    //   pl_text     the characters of the positions, 2 bits each (position i in bits 2i.. of the packed words, as the
    //               hash keys); the k-mer of pl_node[p] is pl_text[p .. p + k)
    //   pl_rc       1 bit per position: the reverse complement of pl_node[p]'s k-mer is in the hash index (the meaning
    //               of the adjacency records' bits 16..20)
    //   pl_stop     1 bit per position: pl_node[p] == 0
    //   pl_pos[e]   the position of edge e, kPlNone unless e is a DBG node
    // The arrays end with at least kPlPad filler positions, so readers may run ahead of a path's end.
    // Two leaner copies for the whole-read gate (exact_path_strand), nullptr when the memory is not there (or the layout
    // is absent); every reader falls back to the arrays above:
    //   kh_pos[i]   per hash slot: pl_pos[kh_vals[i]] of an in_graph edge, else kPlNone (an empty slot too)
    //   pl_word[w]  positions 32w .. 32w + 31 in one 16-byte word: x = pl_text[w], y = pl_stop[w] | pl_rc[w] (high
    //               half 0), over the same pl_n positions
    const uint32_t *pl_node;
    const uint32_t *pl_pos;
    const unsigned long long *pl_text;
    const uint32_t *pl_rc;
    const uint32_t *pl_stop;
    const uint32_t *kh_pos;
    const ulonglong2 *pl_word;
    uint64_t pl_n;
    uint64_t n;                 // number of edges (ids 1..n)
    uint32_t nblk;
    uint32_t k;                 // DBG k; BOSS node length = k - 1
    uint32_t sfx_len;
    uint32_t sigma;
    uint64_t F[kMaxSigma];
    uint64_t NF[kMaxSigma];
    uint32_t total_W[kMaxSigma];
    uint64_t num_ones;
    // Alphabet-generic layout (any sigma <= 32; used for protein, kmer/alphabets.hpp:29-38). Plain arrays
    // per 64-edge block, no lane cooperation: every lane of a group does the same scalar work.
    //   wW     one byte per edge (0xFF = padding / position 0)
    //   wl     4 words per block: `last` bits (2 words), set bits before the block, 0
    //   wrank  kMaxSigma words per block: number of W == c (un-flagged) before the block
    //   wsel   per symbol (offset wsel_off[c]): block of every 32nd occurrence, as sel_W
    //   wadj   4 words per edge: last edge of the target node, label mask (all), label mask (valid
    //          DBG nodes), 0 -- the adj record with sigma-bit masks
    // radj is shared; its y word holds the first character in bits 0..6 and the multi-incoming flag in
    // bit 7 here (bits 0..2 / bit 3 in the DNA layout).
    uint32_t mode;              // DeBruijnGraph::Mode: 0 BASIC, 1 CANONICAL (graph holds both strands),
                                // 2 PRIMARY (one k-mer of every reverse-complement pair; CanonicalDBG semantics)
    // PRIMARY graphs only (canonical_dbg.cpp, node_first_cache.cpp:122-176, one u32 per edge e with k-mer x):
    //   rcs[e]  last edge of the BOSS node rc(x[1..k)) or 0   (get_suffix_rc: where children of x enter on the rc strand)
    //   rcp[e]  last edge of the BOSS node rc(x[0..k-1)) or 0 (get_prefix_rc: where parents of x leave on the rc strand)
    //   palin   bit per edge: x is its own reverse complement (even k only, else nullptr)
    const uint32_t *rcs;
    const uint32_t *rcp;
    const uint32_t *palin;
    uint32_t wide;
    const uint8_t *wW;
    const uint32_t *wl;
    const uint32_t *wrank;
    const uint32_t *wsel;
    uint32_t wsel_off[kMaxSigma];
    const uint32_t *wadj;
};

// ---------------------------------------------------------------------------------------
// A 64-byte block held by a quad (device) or by the single host lane (emulation).
// ---------------------------------------------------------------------------------------
#if MGB_DEVICE_CODE
struct Line { uint32_t x, y, z, w; };
static constexpr int kGroup = 4;
MGB_D int glane() { return quad_lane(); }
MGB_D Line load_line(const IndexView &ix, uint32_t blk) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(ix.blocks) + (size_t)blk * 4 + quad_lane());
    Line l; l.x = v.x; l.y = v.y; l.z = v.z; l.w = v.w;
    return l;
}
MGB_D uint32_t line_word(const Line &l, int idx) {
    int c = idx & 3;
    uint32_t v = c == 0 ? l.x : c == 1 ? l.y : c == 2 ? l.z : l.w;
    return qbcast(v, idx >> 2);
}
MGB_D uint32_t gsum_or(uint32_t s) {   // lanes 2,3 contribute 0 to sums over W words
    s += qxor(s, 1);
    s |= qxor(s, 2);
    return s;
}
MGB_D uint32_t gmin(uint32_t s) {
    uint32_t o = qxor(s, 1); s = o < s ? o : s;
    o = qxor(s, 2); s = o < s ? o : s;
    return s;
}
MGB_D unsigned gballot(bool p) { return (__ballot_sync(quad_mask(), p) >> (threadIdx.x & 28)) & 0xFu; }
MGB_D uint32_t ldg32(const uint32_t *p) { return __ldg(p); }
#else
struct Line { uint32_t w16[16]; };
static constexpr int kGroup = 1;
inline int glane() { return 0; }
inline Line load_line(const IndexView &ix, uint32_t blk) {
    Line l;
    for (int i = 0; i < 16; ++i) l.w16[i] = ix.blocks[(size_t)blk * 16 + i];
    return l;
}
inline uint32_t line_word(const Line &l, int idx) { return l.w16[idx]; }
inline uint32_t gsum_or(uint32_t s) { return s; }
inline uint32_t gmin(uint32_t s) { return s; }
inline unsigned gballot(bool p) { return p ? 1u : 0u; }
inline uint32_t ldg32(const uint32_t *p) { return *p; }
#endif

// one bit per nibble of x that equals c
MGB_HD uint32_t nib_eq(uint32_t x, uint32_t c) {
    uint32_t y = x ^ (c * 0x11111111u);
    y |= y >> 1;
    y |= y >> 2;
    return ~y & 0x11111111u;
}
// nibble positions 0..m of a word (m may be < 0 or > 7)
MGB_HD uint32_t nib_prefix(int m) {
    return m < 0 ? 0u : (m >= 7 ? 0x11111111u : (0x11111111u >> (4 * (7 - m))));
}
MGB_HD uint32_t nib_suffix(int m) {   // nibble positions m..7
    return m <= 0 ? 0x11111111u : (m > 7 ? 0u : (0x11111111u << (4 * m)));
}

// number of W == c among in-block offsets [0, off]
MGB_HD uint32_t line_count_W(const Line &l, int off, uint32_t c) {
    uint32_t cnt = 0;
#if MGB_DEVICE_CODE
    int q = quad_lane();
    if (q < 2) {
        int base = 32 * q;
        cnt += popc32(nib_eq(l.x, c) & nib_prefix(off - base));
        cnt += popc32(nib_eq(l.y, c) & nib_prefix(off - base - 8));
        cnt += popc32(nib_eq(l.z, c) & nib_prefix(off - base - 16));
        cnt += popc32(nib_eq(l.w, c) & nib_prefix(off - base - 24));
    }
    cnt = gsum_or(cnt);
#else
    for (int t = 0; t < 8; ++t)
        cnt += popc32(nib_eq(l.w16[t], c) & nib_prefix(off - 8 * t));
#endif
    return cnt;
}

MGB_HD uint32_t line_get_W(const Line &l, int off) {
    return (line_word(l, off >> 3) >> (4 * (off & 7))) & 15u;
}
MGB_HD bool line_get_last(const Line &l, int off) {
    return (line_word(l, 8 + (off >> 5)) >> (off & 31)) & 1u;
}
MGB_HD uint32_t line_count_last(const Line &l, int off) {   // set bits at offsets [0, off]
    uint32_t lo = line_word(l, 8), hi = line_word(l, 9);
    if (off < 32)
        return popc32(lo & (off == 31 ? 0xffffffffu : ((2u << off) - 1u)));
    off -= 32;
    return popc32(lo) + popc32(hi & (off == 31 ? 0xffffffffu : ((2u << off) - 1u)));
}


// ---------------------------------------------------------------------------------------
// Alphabet-generic primitives (IndexView::wide): same contracts as the block versions below.
// ---------------------------------------------------------------------------------------
MGB_HD uint32_t wide_get_W(const IndexView &ix, uint64_t e) { return ix.wW[e]; }
MGB_HD bool wide_get_last(const IndexView &ix, uint64_t e) {
    return (ix.wl[(e >> 6) * 4 + ((e >> 5) & 1)] >> (e & 31)) & 1u;
}
MGB_HD uint32_t bytes_eq(uint32_t x, uint32_t c) {        // bit 8j set iff byte j of x == c
    uint32_t y = x ^ (c * 0x01010101u);
    y |= y >> 4; y |= y >> 2; y |= y >> 1;
    return ~y & 0x01010101u;
}
MGB_HD uint64_t wide_rank_W(const IndexView &ix, uint64_t i, uint32_t c) {
    if (i == 0) return 0;
    const uint64_t b = i >> 6;
    uint64_t r = ix.wrank[b * kMaxSigma + c];
    const uint32_t *w = reinterpret_cast<const uint32_t*>(ix.wW + (b << 6));
    const int off = (int)(i & 63);                         // positions [0, off] of the block
    for (int t = 0; 4 * t <= off; ++t) {
        uint32_t m = bytes_eq(w[t], c);
        const int rem = off - 4 * t;                       // bytes 0..rem of this word count
        if (rem < 3) m &= (1u << (8 * rem + 1)) - 1u;
        r += popc32(m);
    }
    return r;
}
MGB_HD uint64_t wide_rank_last(const IndexView &ix, uint64_t i) {
    if (i == 0) return 0;
    const uint32_t *l = ix.wl + (i >> 6) * 4;
    int off = (int)(i & 63);
    uint32_t r = l[2];
    if (off < 32) return r + popc32(l[0] & (off == 31 ? 0xffffffffu : ((2u << off) - 1u)));
    off -= 32;
    return r + popc32(l[0]) + popc32(l[1] & (off == 31 ? 0xffffffffu : ((2u << off) - 1u)));
}
MGB_HD uint64_t wide_select_last(const IndexView &ix, uint64_t r) {
    if (r == 0) return 0;
    uint64_t j = (r - 1) / kSelLastRate;
    uint32_t b = ix.sel_last[j], b1 = ix.sel_last[j + 1];
    while (b < b1 && ix.blk_rank[b + 1] < r) ++b;          // largest block with blk_rank[b] < r
    const uint32_t *l = ix.wl + (size_t)b * 4;
    int t = (int)(r - l[2]);
    int plo = popc32(l[0]);
    int pos = t <= plo ? nth_set32(l[0], t) : 32 + nth_set32(l[1], t - plo);
    return ((uint64_t)b << 6) + pos;
}
MGB_HD uint64_t wide_select_W(const IndexView &ix, uint32_t c, uint64_t r) {
    uint64_t j = (r - 1) / kSelWRate;
    const uint32_t *sel = ix.wsel + ix.wsel_off[c];
    uint32_t b = sel[j], b1 = sel[j + 1];
    while (b < b1 && ix.wrank[(size_t)(b + 1) * kMaxSigma + c] < r) ++b;
    int t = (int)(r - ix.wrank[(size_t)b * kMaxSigma + c]);
    const uint32_t *w = reinterpret_cast<const uint32_t*>(ix.wW + ((uint64_t)b << 6));
    for (int q = 0; q < 16; ++q) {
        uint32_t m = bytes_eq(w[q], c);
        int pc = popc32(m);
        if (t <= pc) return ((uint64_t)b << 6) + 4 * q + (nth_set32(m, t) >> 3);
        t -= pc;
    }
    return 0;   // unreachable for r <= total_W[c]
}
MGB_HD uint64_t wide_pred_last(const IndexView &ix, uint64_t i) {
    while (i) {
        const uint32_t *l = ix.wl + (i >> 6) * 4;
        int off = (int)(i & 63);
        uint64_t bits = ((uint64_t)l[1] << 32) | l[0];
        bits &= off == 63 ? ~0ull : ((2ull << off) - 1ull);
        if (bits) {
            uint32_t h = (uint32_t)(bits >> 32);
            int p = h ? 63 - clz32(h) : 31 - clz32((uint32_t)bits);
            return (i & ~63ull) + p;
        }
        if ((i >> 6) == 0) return 0;
        i = (i & ~63ull) - 1;
    }
    return 0;
}
MGB_HD uint64_t wide_succ_last(const IndexView &ix, uint64_t i) {
    while (i <= ix.n) {
        const uint32_t *l = ix.wl + (i >> 6) * 4;
        int off = (int)(i & 63);
        uint64_t bits = ((((uint64_t)l[1] << 32) | l[0]) >> off) << off;
        if (bits) {
            uint32_t lo = (uint32_t)bits;
            int p = lo ? ffs32(lo) - 1 : 32 + ffs32((uint32_t)(bits >> 32)) - 1;
            return (i & ~63ull) + p;
        }
        i = (i & ~63ull) + 64;
    }
    return ix.n + 1;
}
MGB_HD uint64_t wide_succ_W2(const IndexView &ix, uint64_t i, uint32_t d, uint32_t *w) {
    for (; i <= ix.n; ++i) {
        // whole words ahead are skipped when they hold neither symbol
        if ((i & 3) == 0) {
            const uint32_t x = *reinterpret_cast<const uint32_t*>(ix.wW + i);
            if (!(bytes_eq(x, d) | bytes_eq(x, d + ix.sigma))) { i += 3; continue; }
        }
        const uint32_t v = ix.wW[i];
        if (v == d || v == d + ix.sigma) { *w = v; return i; }
    }
    *w = 0;
    return ix.n + 1;
}

// A cached block: re-loaded only when another block is touched.
struct LineCache {
    Line line;
    uint32_t blk;
    bool valid_;
    MGB_HD LineCache() : blk(0), valid_(false) {}
    MGB_HD void touch(const IndexView &ix, uint64_t edge) {
        uint32_t b = (uint32_t)(edge >> 6);
        if (!valid_ || b != blk) { line = load_line(ix, b); blk = b; valid_ = true; }
    }
    MGB_HD uint32_t get_W(const IndexView &ix, uint64_t e) {
        if (MGB_WIDE(ix)) return wide_get_W(ix, e);
        touch(ix, e); return line_get_W(line, (int)(e & 63));
    }
    MGB_HD bool get_last(const IndexView &ix, uint64_t e) {
        if (MGB_WIDE(ix)) return wide_get_last(ix, e);
        touch(ix, e); return line_get_last(line, (int)(e & 63));
    }
};

// boss.cpp:437-441; positions [1..i], un-flagged symbol c only
MGB_HD uint64_t rank_W(const IndexView &ix, LineCache &lc, uint64_t i, uint32_t c) {
    if (MGB_WIDE(ix)) return wide_rank_W(ix, i, c);
    if (i == 0) return 0;
    lc.touch(ix, i);
    return (uint64_t)line_word(lc.line, 11 + c) + line_count_W(lc.line, (int)(i & 63), c);
}
// boss.cpp:577-581
MGB_HD uint64_t rank_last(const IndexView &ix, LineCache &lc, uint64_t i) {
    if (MGB_WIDE(ix)) return wide_rank_last(ix, i);
    if (i == 0) return 0;
    lc.touch(ix, i);
    return (uint64_t)line_word(lc.line, 10) + line_count_last(lc.line, (int)(i & 63));
}

// boss.cpp:588-592: position of the r-th set bit of `last` (r >= 1); leaves its block in lc
MGB_HD uint64_t select_last(const IndexView &ix, LineCache &lc, uint64_t r) {
    if (MGB_WIDE(ix)) return wide_select_last(ix, r);
    if (r == 0) return 0;
    uint64_t j = (r - 1) / kSelLastRate;
    uint32_t b = ldg32(ix.sel_last + j), b1 = ldg32(ix.sel_last + j + 1);
    // largest block b in [b, b1] with blk_rank[b] < r
    for (uint32_t base = b + 1; base <= b1; base += kGroup) {
        uint32_t cand = base + glane();
        bool p = cand <= b1 && ldg32(ix.blk_rank + cand) < r;
        int cnt = popc32(gballot(p));
        b += cnt;
        if (cnt < kGroup) break;
    }
    lc.touch(ix, (uint64_t)b << 6);
    int t = (int)(r - line_word(lc.line, 10));
    uint32_t lo = line_word(lc.line, 8), hi = line_word(lc.line, 9);
    int plo = popc32(lo);
    int pos = t <= plo ? nth_set32(lo, t) : 32 + nth_set32(hi, t - plo);
    return ((uint64_t)b << 6) + pos;
}

// wavelet_tree::select(c, r) (wavelet_tree.cpp:352-357) for un-flagged c, r >= 1
MGB_HD uint64_t select_W(const IndexView &ix, LineCache &lc, uint32_t c, uint64_t r) {
    if (MGB_WIDE(ix)) return wide_select_W(ix, c, r);
    uint64_t j = (r - 1) / kSelWRate;
    uint32_t b = ldg32(ix.sel_W[c] + j), b1 = ldg32(ix.sel_W[c] + j + 1);
    for (uint32_t base = b + 1; base <= b1; base += kGroup) {
        uint32_t cand = base + glane();
        bool p = cand <= b1 && ldg32(ix.blocks + (size_t)cand * kBlkWords + 11 + c) < r;
        int cnt = popc32(gballot(p));
        b += cnt;
        if (cnt < kGroup) break;
    }
    lc.touch(ix, (uint64_t)b << 6);
    int t = (int)(r - line_word(lc.line, 11 + c));   // t-th occurrence inside the block
    // every lane scans the 8 W words (uniform result)
    int pos = -1;
    for (int w = 0; w < 8 && pos < 0; ++w) {
        uint32_t m = nib_eq(line_word(lc.line, w), c);
        int pc = popc32(m);
        if (t <= pc) pos = 8 * w + (nth_set32(m, t) >> 2);
        else t -= pc;
    }
    return ((uint64_t)b << 6) + pos;
}

// boss.cpp:598-607: last set bit of `last` in [1..i], 0 if none
MGB_HD uint64_t pred_last(const IndexView &ix, LineCache &lc, uint64_t i) {
    if (MGB_WIDE(ix)) return wide_pred_last(ix, i);
    while (i) {
        lc.touch(ix, i);
        int off = (int)(i & 63);
        uint32_t lo = line_word(lc.line, 8), hi = line_word(lc.line, 9);
        uint64_t bits = ((uint64_t)hi << 32) | lo;
        bits &= off == 63 ? ~0ull : ((2ull << off) - 1ull);
        if (bits) {
            uint32_t h = (uint32_t)(bits >> 32);
            int p = h ? 63 - clz32(h) : 31 - clz32((uint32_t)bits);
            return (i & ~63ull) + p;
        }
        if ((i >> 6) == 0) return 0;
        i = (i & ~63ull) - 1;
    }
    return 0;
}

// boss.cpp:613-617: first set bit of `last` at a position >= i; n + 1 if none
MGB_HD uint64_t succ_last(const IndexView &ix, LineCache &lc, uint64_t i) {
    if (MGB_WIDE(ix)) return wide_succ_last(ix, i);
    while (i <= ix.n) {
        lc.touch(ix, i);
        int off = (int)(i & 63);
        uint32_t lo = line_word(lc.line, 8), hi = line_word(lc.line, 9);
        uint64_t bits = (((uint64_t)hi << 32) | lo) >> off << off;
        if (bits) {
            uint32_t l = (uint32_t)bits;
            int p = l ? ffs32(l) - 1 : 32 + ffs32((uint32_t)(bits >> 32)) - 1;
            return (i & ~63ull) + p;
        }
        i = (i & ~63ull) + 64;
    }
    return ix.n + 1;
}

// boss.cpp:679-690
MGB_HD uint32_t node_last_value(const IndexView &ix, uint64_t i) {
    if (i == 0) return 0;
    for (uint32_t c = 0; c < ix.sigma; ++c)
        if (ix.F[c] >= i) return c - 1;
    return ix.sigma - 1;
}

// boss.cpp:642-652
MGB_HD uint64_t fwd(const IndexView &ix, LineCache &lc, uint64_t i, uint32_t c) {
    return select_last(ix, lc, ix.NF[c] + rank_W(ix, lc, i, c));
}

// Forward adjacency record of edge e (denormalised DBGSuccinct::call_outgoing_kmers,
// dbg_succinct.cpp:110-139 = fwd + pred_last + get_W of the target node, in one 8-byte load):
//   x        last edge of the target node of e (0: e is a sink dummy, no outgoing edges)
//   y[0:5)   labels ($ACGT) present among the target node's edges (flagged ones included)
//   y[8:13)  labels whose edge is a valid, non-'$' DBG node (in_graph)
//   y[16:21) graphs with the k-mer hash index only (DNA block layout, k <= 31): labels c whose edge's k-mer has its
//            reverse complement in the hash index (kh_lookup != 0, in_graph or not), or whose k-mer is not a valid
//            key. 0 tells k_seed_hash that the other strand's k-mer at the mirrored position is missing. Set by
//            k_adj_rc; other layouts and the host emulation leave these bits 0 and never read them.
// Edges of a node are sorted by label, so the edge with label c is first + popc(mask & ((1<<c)-1)).
MGB_HD uint2 load_adj(const IndexView &ix, uint64_t e) {
#if MGB_DEVICE_CODE
    return __ldg(ix.adj + e);
#else
    return ix.adj[e];
#endif
}
MGB_HD uint64_t adj_child(uint2 a, uint32_t c) {   // edge with label c out of the target node, 0 if none
    uint32_t all = a.y & 31u;
    if (!a.x || !((all >> c) & 1u)) return 0;
    uint64_t first = (uint64_t)a.x - popc32(all) + 1;
    return first + popc32(all & ((1u << c) - 1u));
}
// The record in decoded form, from either layout: `last` = last edge of the target node (0: none),
// `all` / `ok` = label masks (bit c), as described above.
struct Adj { uint32_t last, all, ok; };
MGB_HD Adj adj_decode(uint2 a) { Adj r; r.last = a.x; r.all = a.y & 31u; r.ok = (a.y >> 8) & 31u; return r; }
MGB_HD Adj load_adj_any(const IndexView &ix, uint64_t e) {
    if (!MGB_WIDE(ix)) return adj_decode(load_adj(ix, e));
    const uint32_t *p = ix.wadj + e * 4;
    Adj r; r.last = p[0]; r.all = p[1]; r.ok = p[2];
    return r;
}
MGB_HD uint64_t adj_child(const Adj &a, uint32_t c) {
    if (!a.last || !((a.all >> c) & 1u)) return 0;
    return (uint64_t)a.last - popc32(a.all) + 1 + popc32(a.all & ((1u << c) - 1u));
}
// fields of the y word of a reverse adjacency record
MGB_HD uint32_t radj_char(const IndexView &ix, uint32_t y) { return MGB_WIDE(ix) ? (y & 127u) : (y & 7u); }
MGB_HD bool radj_multi(const IndexView &ix, uint32_t y) { return MGB_WIDE(ix) ? ((y >> 7) & 1u) : ((y >> 3) & 1u); }

// Reverse adjacency record of edge e (backward extension through the RCDBG view, rc_dbg.hpp:86-97):
//   x        bwd(e): first (un-flagged) edge entering the source node of e (boss.cpp:623-636)
//   y[0:3)   first character of e's own k-mer = node_last_value(bwd^{k-2}(e))
//            (NodeFirstCache::get_first_char, node_first_cache.cpp:10-24)
//   y[3]     the source node of e has more than one incoming edge (!BOSS::is_single_incoming)
MGB_HD uint2 load_radj(const IndexView &ix, uint64_t e) {
#if MGB_DEVICE_CODE
    return __ldg(ix.radj + e);
#else
    return ix.radj[e];
#endif
}

// boss.cpp:623-636
MGB_HD uint64_t bwd(const IndexView &ix, LineCache &lc, uint64_t i) {
    uint64_t target_node = rank_last(ix, lc, i - 1) + 1;
    if (target_node == 1) return 1;
    uint32_t c = node_last_value(ix, i);
    return select_W(ix, lc, c, target_node - ix.NF[c]);
}

// boss.cpp:710-722
MGB_HD uint64_t pick_edge(const IndexView &ix, LineCache &lc, uint64_t edge, uint32_t c) {
    do {
        uint32_t w = lc.get_W(ix, edge);
        if (w == c || w == c + ix.sigma) return edge;
    } while (--edge && !lc.get_last(ix, edge));
    return 0;
}

// First position p >= i with W[p] in { d, d + sigma } (boss.cpp:515-570 succ_W with two
// symbols); returns n + 1 and *w = 0 if none.
MGB_HD uint64_t succ_W2(const IndexView &ix, LineCache &lc, uint64_t i, uint32_t d, uint32_t *w) {
    if (MGB_WIDE(ix)) return wide_succ_W2(ix, i, d, w);
    while (i <= ix.n) {
        lc.touch(ix, i);
        int off = (int)(i & 63);
        uint32_t best = 64;
#if MGB_DEVICE_CODE
        int q = quad_lane();
        if (q < 2) {
            uint32_t ws[4] = { lc.line.x, lc.line.y, lc.line.z, lc.line.w };
#pragma unroll
            for (int t = 3; t >= 0; --t) {
                int base = 32 * q + 8 * t;
                uint32_t m = (nib_eq(ws[t], d) | nib_eq(ws[t], d + ix.sigma)) & nib_suffix(off - base);
                if (m) best = base + ((ffs32(m) - 1) >> 2);
            }
        }
        best = gmin(best);
#else
        for (int t = 7; t >= 0; --t) {
            uint32_t x = lc.line.w16[t];
            uint32_t m = (nib_eq(x, d) | nib_eq(x, d + ix.sigma)) & nib_suffix(off - 8 * t);
            if (m) best = 8 * t + ((ffs32(m) - 1) >> 2);
        }
#endif
        if (best < 64) {
            uint64_t p = (i & ~63ull) + best;
            if (p > ix.n) break;
            *w = line_get_W(lc.line, (int)best);
            return p;
        }
        i = (i & ~63ull) + 64;
    }
    *w = 0;
    return ix.n + 1;
}

// dbg_succinct.cpp:934-939
MGB_HD bool in_graph(const IndexView &ix, uint64_t node) {
    if (node == 0 || node > ix.n) return false;
    if (!ix.valid) return true;
    return (ldg32(ix.valid + (node >> 5)) >> (node & 31)) & 1u;
}

// boss.hpp:682-693. Both ends are advanced together so their loads overlap.
MGB_HD bool tighten_range(const IndexView &ix, uint64_t *rl, uint64_t *ru, uint32_t s) {
    LineCache la, lb;
    uint64_t rk_rl = rank_W(ix, la, *rl - 1, s) + 1;
    uint64_t rk_ru = rank_W(ix, lb, *ru, s);
    if (rk_rl > rk_ru) return false;
    *rl = select_last(ix, la, ix.NF[s] + rk_rl - 1) + 1;
    *ru = select_last(ix, lb, ix.NF[s] + rk_ru);
    return true;
}

// boss.hpp:636-680 (codes must be < sigma)
MGB_HD void initial_range(const IndexView &ix, const uint8_t *begin, int len,
                          uint64_t *rl, uint64_t *ru, int *offset) {
    bool use_sfx = ix.sfx_len && (int)ix.sfx_len <= len;
    if (use_sfx) {
        for (uint32_t i = 0; i < ix.sfx_len; ++i)
            if (begin[i] == 0) use_sfx = false;
    }
    if (use_sfx) {
        uint64_t index = 0;
        for (int i = (int)ix.sfx_len - 1; i >= 0; --i)
            index = index * (ix.sigma - 1) + (begin[i] - 1);
        *rl = ldg32(ix.sfx + 2 * index);
        *ru = (uint64_t)ldg32(ix.sfx + 2 * index + 1) - 1;
        *offset = ix.sfx_len;
    } else {
        uint32_t s = begin[0];
        *rl = ix.F[s] + 1 < ix.n + 1 ? ix.F[s] + 1 : ix.n + 1;
        *ru = s + 1 < ix.sigma ? ix.F[s + 1] : ix.n;
        *offset = 1;
    }
}

// boss.hpp:695-718: last edge of the node spelled by codes[0..len) (len == k - 1), 0 if absent.
// Codes equal to sigma are invalid.
MGB_HD uint64_t boss_index(const IndexView &ix, const uint8_t *codes, int len) {
    for (int i = 0; i < len; ++i)
        if (codes[i] >= ix.sigma) return 0;
    uint64_t rl, ru; int off;
    initial_range(ix, codes, len, &rl, &ru, &off);
    if (rl > ru) return 0;
    for (int i = off; i < len; ++i)
        if (!tighten_range(ix, &rl, &ru, codes[i])) return 0;
    return ru;
}

// boss_index for codes known to be valid (all < sigma, none 0) with the suffix-table slot of
// codes[0..sfx_len) already known (map_to_edges keeps it as a rolling value)
MGB_HD uint64_t boss_index_slot(const IndexView &ix, const uint8_t *codes, int len, uint64_t slot) {
    uint64_t rl = ldg32(ix.sfx + 2 * slot);
    uint64_t ru = (uint64_t)ldg32(ix.sfx + 2 * slot + 1) - 1;
    if (rl > ru) return 0;
    for (int i = (int)ix.sfx_len; i < len; ++i)
        if (!tighten_range(ix, &rl, &ru, codes[i])) return 0;
    return ru;
}

// boss.hpp:720-764: longest matching prefix of codes[0..len) (len <= k - 1) and its edge
// range; *matched = number of matched characters (0 -> (0, 0)).
// min_len > 0: the caller discards matches shorter than min_len, so a miss in a suffix table of
// length <= min_len is final (*matched = 0) and the walk from the first character is skipped.
MGB_HD void boss_index_range(const IndexView &ix, const uint8_t *codes, int len,
                             uint64_t *first, uint64_t *lst, int *matched, int min_len = 0) {
    if (len == 0) { *first = 1; *lst = 1; *matched = 0; return; }
    for (int i = 0; i < len; ++i)
        if (codes[i] >= ix.sigma) { *first = 0; *lst = 0; *matched = 0; return; }
    uint64_t rl, ru; int off;
    initial_range(ix, codes, len, &rl, &ru, &off);
    if (rl > ru) {
        if (off > 1 && off <= min_len) { *first = 0; *lst = 0; *matched = 0; return; }
        uint32_t s = codes[0];
        rl = ix.F[s] + 1 < ix.n + 1 ? ix.F[s] + 1 : ix.n + 1;
        ru = s + 1 < ix.sigma ? ix.F[s + 1] : ix.n;
        if (rl > ru) { *first = 0; *lst = 0; *matched = 0; return; }
        off = 1;
    }
    int i = off;
    for (; i < len; ++i)
        if (!tighten_range(ix, &rl, &ru, codes[i])) break;
    LineCache lc;
    *first = succ_last(ix, lc, rl);
    *lst = ru;
    *matched = i;
}

// ---------------------------------------------------------------------------------------
// k-mer hash index: key = sum over positions p of (code_p - 1) << 2p (codes 1..4), k <= 31
// ---------------------------------------------------------------------------------------
// Buckets of 4 keys = one 32-byte sector. A k-mer's home is the first slot of its bucket; insertion takes the first free
// slot from there on (running into the following buckets when its own is full), so a lookup reads whole buckets in
// order and stops at the first empty slot: ~1.2 sectors per probe at a load factor of 0.7, hit or miss (one key per
// slot with linear probing needs ~6 for a miss).
MGB_HD uint64_t kh_slot_of(uint64_t key, uint64_t slots) {
    const uint64_t h = key * 0x9E3779B97F4A7C15ull;
#if MGB_DEVICE_CODE
    return __umul64hi(h ^ (h >> 29), slots >> 2) << 2;
#else
    return (uint64_t)(((unsigned __int128)(h ^ (h >> 29)) * (slots >> 2)) >> 64) << 2;
#endif
}
// reverse complement of the packed k-mer `key` (k <= 31): position p takes 3 - (the code at k - 1 - p, minus 1), as
// the complement of DNA code c is 5 - c
MGB_HD uint64_t kh_revcomp(uint64_t key, uint32_t k) {
    uint64_t r = 0;
    for (uint32_t p = 0; p < k; ++p) { r = (r << 2) | (key & 3u); key >>= 2; }
    return r ^ ((1ull << (2 * k)) - 1);
}
// edge of the k-mer `key62`, 0 if the graph does not have it (kh_slots is a multiple of 4)
MGB_HD uint64_t kh_lookup(const IndexView &ix, uint64_t key62) {
    const unsigned long long key = key62 | (1ull << 63);
    uint64_t i = kh_slot_of(key, ix.kh_slots);
    while (true) {
#if MGB_DEVICE_CODE
        const ulonglong2 a = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + i));
        const ulonglong2 b = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + i + 2));
        const unsigned long long k0 = a.x, k1 = a.y, k2 = b.x, k3 = b.y;
#else
        const unsigned long long k0 = ix.kh_keys[i], k1 = ix.kh_keys[i + 1], k2 = ix.kh_keys[i + 2], k3 = ix.kh_keys[i + 3];
#endif
        if (k0 == key) return ix.kh_vals[i];
        if (k0 == 0) return 0;
        if (k1 == key) return ix.kh_vals[i + 1];
        if (k1 == 0) return 0;
        if (k2 == key) return ix.kh_vals[i + 2];
        if (k2 == 0) return 0;
        if (k3 == key) return ix.kh_vals[i + 3];
        if (k3 == 0) return 0;
        i += 4;
        if (i >= ix.kh_slots) i = 0;
    }
}

} // namespace mgb
