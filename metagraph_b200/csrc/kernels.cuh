// Kernel-side code of the C-ABI library: per-item device functions, the kernels and their launchers.
//
// The product library compiles this file twice (no relocatable device code, so the two sets of device
// functions never meet):
//   api.cu          -DMGB_NARROW_ONLY, MGB_KERNEL_NS = kern_dna : DNA block layout only; the branches
//                   to the alphabet-generic index layout are compiled out of the hot kernels
//   api_generic.cu  -DMGB_WIDE_ONLY,   MGB_KERNEL_NS = kern_any : alphabet-generic layout only (protein)
//   api_canonical.cu -DMGB_NARROW_ONLY -DMGB_CANONICAL_ONLY -DMGB_ALIGN_KERNEL_ONLY, MGB_KERNEL_NS = kern_canon :
//                   k_align for CANONICAL-mode DNA graphs; the other two sets compile that mode's branches out
// The host-emulation build (tests/emu) includes it once with the layout chosen at run time.
#pragma once
#include "align_core.cuh"
#include "acgt_words.cuh"
#if !defined(MGB_HOST_EMU)
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#endif

#ifndef MGB_KERNEL_NS
#define MGB_KERNEL_NS kern_dna
#endif

namespace mgb {

struct ReadHdr {              // per read, written by the align kernel
    uint32_t status, n_aln;
    uint64_t heap_off;
    ReadStats stats;
};

// ---------------------------------------------------------------------------------------
// kernels (device) / loops (host emulation)
// ---------------------------------------------------------------------------------------
struct PrepArgs {
    const char *seqs; const uint64_t *offsets; uint32_t n_reads;
    char *qf, *qr; uint8_t *cf, *cr;
    uint8_t code_of[256];     // KmerExtractorBOSS::encode of the index's alphabet
};

MGB_HD void prepare_read(const PrepArgs &a, uint32_t r) {
    const uint64_t b = a.offsets[r];
    const int L = (int)(a.offsets[r + 1] - b);
    for (int i = wlane(); i < L; i += kWarp) {
        uint8_t f = sanitize_char((uint8_t)a.seqs[b + i]);
        uint8_t rc = complement_char(sanitize_char((uint8_t)a.seqs[b + L - 1 - i]));
        a.qf[b + i] = (char)f; a.qr[b + i] = (char)rc;
        a.cf[b + i] = a.code_of[f]; a.cr[b + i] = a.code_of[rc];
    }
}

struct SeedArgs {
    IndexView ix;
    const uint8_t *cf, *cr; const uint64_t *offsets; const uint64_t *koff;
    uint64_t *nodes_f, *nodes_r; uint32_t n_reads; uint32_t n_strands;
    uint32_t hinted;           // 1: k_premap ran, hint_f / hint_r hold its verdicts
    uint32_t *hint_f, *hint_r;
    // k_seed_hash only (nullptr: not written): per read, which kinds of node id the walk stored, as ExactArgs::summary
    // reads them (1: a 0 on the forward strand, 2: a non-zero one; 4 / 8: the same on the reverse strand; 0 if L < k)
    uint8_t *summary;
    // k_seed_hash only: the reads to seed, list[0 .. *n_list) (built on the device by k_prepare_exact); nullptr: all
    // n_reads reads
    const uint32_t *list; const unsigned int *n_list;
    // k_seed_hash only: 0 picks the walk or the short-list mode by the number of reads; 1 / 2 force the walk / the
    // short-list mode (MGB_TEST_SEED_MODE=walk|wide, test knob)
    uint32_t seed_mode;
};

MGB_HD void seed_item(const SeedArgs &a, uint64_t item) {
    uint32_t r = (uint32_t)(item / a.n_strands);
    uint32_t s = (uint32_t)(item % a.n_strands);
    const uint64_t b = a.offsets[r];
    const int L = (int)(a.offsets[r + 1] - b);
    const uint32_t *hints = a.hinted ? (s ? a.hint_r : a.hint_f) + (a.koff[r] >> 5) + r : nullptr;
    map_to_edges(a.ix, (s ? a.cr : a.cf) + b, L, (s ? a.nodes_r : a.nodes_f) + a.koff[r], hints);
}
// first pass (premap_kmer) for strand s of read r: one k-mer per lane, one hint word per 32 k-mers
// (the words of read r start at word koff[r] / 32 + r of the strand's hint array)
MGB_HD void premap_item(const SeedArgs &a, uint32_t r, uint32_t s) {
    const uint64_t b = a.offsets[r];
    const int L = (int)(a.offsets[r + 1] - b);
    const int nk = L - (int)a.ix.k + 1;
    if (nk <= 0) return;
    const uint8_t *codes = (s ? a.cr : a.cf) + b;
    uint32_t *hw = (s ? a.hint_r : a.hint_f) + (a.koff[r] >> 5) + r;
    for (int base = 0; base < nk; base += 32) {
        unsigned word = 0;
        for (int o = 0; o < 32; o += kWarp) {                 // one pass on the device
            const int i = base + o + wlane();
            word |= wballot(i < nk && premap_kmer(a.ix, codes, i) != 0) << o;
        }
        if (wlane() == 0) hw[base >> 5] = word;
    }
}

// Sub-k seeding, lookup part (SuffixSeeder::generate_seeds, aligner_seeder_methods.cpp:215-238 ->
// dbg_succinct.cpp:307-330 -> BOSS::index_range, boss.hpp:720-764): the longest prefix of the query at
// every position without a full k-mer hit and its edge range. The lookups are independent of each other,
// so they run GPU-wide, one quad per 16 positions of a strand, before the per-read kernel; k_align
// keeps the order-dependent part (enumeration, per-locus rules, merging with the MEM seeds).
struct SubkArgs {
    IndexView ix;
    const uint8_t *cf, *cr; const uint64_t *offsets, *koff; const uint64_t *nodes_f, *nodes_r;
    uint32_t n_reads, n_strands, min_seed_length, max_len;     // max_len = min(max_seed_length, k - 1)
    uint32_t *first_f, *last_f, *first_r, *last_r; uint8_t *len_f, *len_r;
};
#ifndef MGB_SUBK_CHUNK
#define MGB_SUBK_CHUNK 1
#endif
static constexpr int kSubkChunk = MGB_SUBK_CHUNK;
MGB_HD void subk_item(const SubkArgs &a, uint32_t r, uint32_t s, uint32_t chunk) {
    const uint64_t b = a.offsets[r];
    const int L = (int)(a.offsets[r + 1] - b);
    const int K = (int)a.ix.k;
    if (L < (int)a.min_seed_length) return;
    const int n_pos = L - (int)a.min_seed_length + 1;
    const uint8_t *codes = (s ? a.cr : a.cf) + b;
    const uint64_t *nodes = L >= K ? (s ? a.nodes_r : a.nodes_f) + a.koff[r] : nullptr;
    uint32_t *of = (s ? a.first_r : a.first_f) + b, *ol = (s ? a.last_r : a.last_f) + b;
    uint8_t *on = (s ? a.len_r : a.len_f) + b;
    const int nk = L >= K ? L - K + 1 : 0;
    for (int i = (int)chunk * kSubkChunk; i < n_pos && i < (int)(chunk + 1) * kSubkChunk; ++i) {
        uint64_t first = 0, lst = 0; int matched = 0;
        uint8_t code = 0xFF;                              // not computed: a full k-mer matches here
        if (!(i < nk && nodes && nodes[i] != 0)) {
            const int len = (int)a.max_len < L - i ? (int)a.max_len : L - i;
            bool ok = len >= (int)a.min_seed_length;
            for (int t = 0; t < len && ok; ++t) ok = codes[i + t] < a.ix.sigma;
            if (ok) boss_index_range(a.ix, codes + i, len < K - 1 ? len : K - 1, &first, &lst, &matched, (int)a.min_seed_length);
            code = (uint8_t)matched;
        }
        if (glane() == 0) { of[i] = (uint32_t)first; ol[i] = (uint32_t)lst; on[i] = code; }
    }
}

struct AlignArgs {
    IndexView ix; DevConfig cfg; Caps caps;
    WarpLayout lay;             // arena regions of a warp (offsets)
    SmemLayout slay;            // on-chip working set of a warp (offsets)
    int use_fast;               // 0 disables the register fast path (test knob)
    unsigned long long *phase_out;   // MGB_PHASE_TIMERS builds: cycles per phase (setup, seeds, fwd, backtrack, align total)
    const char *qf, *qr; const uint8_t *cf, *cr; const uint64_t *offsets, *koff;
    const uint64_t *nodes_f, *nodes_r;
    const uint32_t *sub_first_f, *sub_last_f, *sub_first_r, *sub_last_r;    // k_subk results or nullptr
    const uint8_t *sub_len_f, *sub_len_r;
    const uint32_t *read_list; uint32_t n_list;
    const unsigned int *n_list_dev;   // non-null: the list's length is *n_list_dev (<= n_list), written by an earlier kernel
    char *arena; size_t arena_stride;
    uint32_t n_arenas;          // arenas at `arena`: k_align hands them to its warps in the order they start
    ReadHdr *hdr; char *heap; uint64_t heap_cap; unsigned long long *heap_used;
    unsigned int *next;         // next[0]: the next read of the list; next[3]: the next arena
};

// aligns read r with the warp's arena and on-chip working set and writes its record and alignments
MGB_HD void align_read(const AlignArgs &a, uint32_t r, const WarpMem &mem, const WarpSmem &sm) {
    ReadAligner al(a.ix, a.cfg, a.caps, mem, sm);
    al.use_fast = a.use_fast != 0;
    const uint64_t b = a.offsets[r];
    const int L = (int)(a.offsets[r + 1] - b);
    const bool has_k = L >= (int)a.ix.k;
    if (a.sub_len_f) {
        al.subk_first[0] = a.sub_first_f + b; al.subk_last[0] = a.sub_last_f + b; al.subk_len[0] = a.sub_len_f + b;
        if (a.sub_len_r) { al.subk_first[1] = a.sub_first_r + b; al.subk_last[1] = a.sub_last_r + b; al.subk_len[1] = a.sub_len_r + b; }
    }
    const uint64_t ko = has_k ? a.koff[r] : 0;
    int n = al.run(L, a.qf + b, a.qr + b, a.cf + b, a.cr + b,
                   has_k ? a.nodes_f + ko : nullptr,
                   has_k && a.cfg.forward_and_reverse_complement ? a.nodes_r + ko : nullptr);
#if defined(MGB_PHASE_TIMERS) && MGB_DEVICE_CODE
    if (wlane() == 0 && a.phase_out) {
        for (int p = 0; p < 8; ++p) atomicAdd((unsigned long long*)a.phase_out + p, (unsigned long long)al.phase_cycles[p]);
    }
#endif
    ReadHdr h;
    h.status = al.overflow ? MGB_READ_OVERFLOW : MGB_READ_OK;
    h.n_aln = 0; h.heap_off = 0; h.stats = al.stats;
    if (!al.overflow && n) {
        // bytes: per alignment OutAln + nodes*8 + cigar*4 + seq (padded to 8), from the aggregator's keys on chip
        const AggKey *keys = sm.agg();
        const int32_t *ord = sm.agg_ord();
        uint64_t bytes = 0;
        for (int i = 0; i < n; ++i) {
            const AggKey ak = keys[i];
            bytes += sizeof(OutAln) + (a.cfg.result_nodes ? 0ull : 8ull * ak.n_nodes) + ((4ull * ak.n_cigar + 7) & ~7ull)
                   + (((uint64_t)ak.seq_len + 7) & ~7ull);
        }
        unsigned long long off = 0;
#if MGB_DEVICE_CODE
        if (wlane() == 0) off = atomicAdd(a.heap_used, (unsigned long long)bytes);
        off = wbcast64(off, 0);
#else
        off = *a.heap_used; *a.heap_used += bytes;
#endif
        if (off + bytes > a.heap_cap) {
            h.status = MGB_READ_OVERFLOW;
        } else {
            h.n_aln = n; h.heap_off = off;
            char *p = a.heap + off;
            for (int i = 0; i < n; ++i) {
                const AlnSlot sl = mem.slot(a.lay.slot_agg + ord[i]);
                const AggKey ak = keys[ord[i]];
                OutAln o;
                o.orientation = ak.orientation; o.score = ak.score; o.offset = ak.offset;
                o.query_begin = ak.clip; o.query_len = ak.q_len;
                o.n_nodes = ak.n_nodes; o.seq_len = ak.seq_len; o.n_cigar = ak.n_cigar;
                if (wlane() == 0) *(OutAln*)p = o;
                p += sizeof(OutAln);
                if (!a.cfg.result_nodes) {
                    uint64_t *pn = (uint64_t*)p;
                    for (int t = wlane(); t < ak.n_nodes; t += kWarp) pn[t] = sl.nodes[t];
                    p += 8ull * ak.n_nodes;
                }
                uint32_t *pc = (uint32_t*)p;
                for (int t = wlane(); t < ak.n_cigar; t += kWarp) pc[t] = sl.cigar[t];
                p += (4ull * ak.n_cigar + 7) & ~7ull;
                for (int t = wlane(); t < ak.seq_len; t += kWarp) p[t] = sl.seq[t];
                p += ((uint64_t)ak.seq_len + 7) & ~7ull;
            }
        }
    }
    if (wlane() == 0) {
        a.hdr[r] = h;
        mem.epoch_store()[0] = sm.ctx()[0].conv_epoch; mem.epoch_store()[1] = sm.ctx()[1].conv_epoch;
    }
    wsync();
}

// once per arena: convergence-table slots start with epoch 0 (never equal to a live epoch)
MGB_HD void init_arena(const AlignArgs &a, char *arena) {
    const WarpMem mem { arena, &a.lay };
    for (int e = 0; e < 2; ++e)
        for (uint32_t i = wlane(); i < a.caps.hash_size; i += kWarp) mem.conv_slots(e)[i].epoch = 0;
    if (wlane() == 0) { mem.epoch_store()[0] = 0; mem.epoch_store()[1] = 0; }
    wsync();
}

// Whole-read exact answers (k_exact_reads, run over a pass's reads before k_align). With the exact seeder
// (min_seed_length = max_seed_length = k) and both strands asked for, a read whose k-mers are all in the graph on one
// strand and none on the other has one alignment: {L}= along that strand's own nodes, score Σ diag + both end bonuses,
// L - k + 1 seeds and one extension. build_seeds would give the matching strand one seed per k-mer (num_matching = L) and
// the other strand none; the matching strand goes first, its first seed starts the read, extend() takes the exact-path
// shortcut (DESIGN.md §3.3), the result enters the empty aggregator and every later seed is dropped. Such a read is
// answered here, without the aligner's set-up; every other read goes on to k_align. The host evaluates the configuration
// part of the gate (cfg.exact_shortcut, both strands, BASIC mode, the exact seeder, no complexity filter,
// min_exact_match <= 1) and launches nothing when it fails.
struct ExactArgs {
    uint32_t k;
    int32_t end_bonus;            // left_end_bonus + right_end_bonus
    int32_t min_score;            // max(0, min_cell_score, min_path_score): extend()'s threshold on a forward extension
                                  // when both strands are aligned, and the empty aggregator's
    uint32_t max_len;             // longest read answered: k_align's own exit needed both strands staged on chip
                                  // (L + 1 <= lq) and room for L characters and L - k + 1 nodes in an alignment slot
    uint32_t result_nodes;        // DevConfig::result_nodes: records without node ids
    int8_t diag[128];             // DevConfig::diag
    const char *qf, *qr; const uint64_t *offsets, *koff, *nodes_f, *nodes_r;
    const uint8_t *summary;       // SeedArgs::summary, or nullptr: the same bits from nodes_f / nodes_r
    const uint32_t *list; uint32_t n_list;
    const unsigned int *n_list_dev;                  // non-null: the list's length is *n_list_dev (<= n_list)
    uint32_t *rest; unsigned int *n_rest;            // the reads left to k_align
    ReadHdr *hdr; char *heap; uint64_t heap_cap; unsigned long long *heap_used;
};

// The strand (0 / 1) whose alignment answers read r, or -1; *b / *L: the read's start and length, *score: the alignment's
// score. One lane, no collectives.
MGB_HD int exact_read_strand(const ExactArgs &a, const int8_t *diag, uint32_t r, uint64_t *b, int *L, score_t *score) {
    *b = a.offsets[r];
    *L = (int)(a.offsets[r + 1] - *b);
    const int n = *L, k = (int)a.k;
    if (n < k || n > (int)a.max_len) return -1;
    unsigned bits;                                       // 1: a missing forward k-mer, 2: a present one; 4 / 8: reverse
    if (a.summary) {
        bits = a.summary[r];
    } else {
        const uint64_t *nf = a.nodes_f + a.koff[r], *nr = a.nodes_r + a.koff[r];
        bits = 0;
        for (int i = 0; i < n - k + 1; ++i) bits |= (nf[i] ? 2u : 1u) | (nr[i] ? 8u : 4u);
    }
    const int s = bits == (2u | 4u) ? 0 : bits == (1u | 8u) ? 1 : -1;
    if (s < 0) return -1;
    // Σ diag over the strand (prepared characters are < 128), read as aligned 8-byte words (the strand buffers are padded
    // past their end)
    const char *q = (s ? a.qr : a.qf) + *b;
    const uintptr_t lo = (uintptr_t)q, hi = lo + (uintptr_t)n;
    int sum = 0;
    for (uintptr_t w = lo & ~(uintptr_t)7; w < hi; w += 8) {
        const unsigned long long x = *reinterpret_cast<const unsigned long long*>(w);
        const int j0 = w < lo ? (int)(lo - w) : 0, j1 = hi - w < 8 ? (int)(hi - w) : 8;
        for (int j = j0; j < j1; ++j) sum += diag[(x >> (8 * j)) & 0x7Fu];
    }
    const score_t full = sum + a.end_bonus;
    if (full < a.min_score) return -1;
#if defined(MGB_HOST_EMU)
    ++mgb_emu_whole_read_hits;
#endif
    *score = full;
    return s;
}

// bytes of the record: OutAln | node ids (unless result_nodes) | one CIGAR op | sequence, each part padded to 8 (align_read)
MGB_HD uint32_t exact_read_bytes(const ExactArgs &a, int L) {
    return (uint32_t)sizeof(OutAln) + (a.result_nodes ? 0u : 8u * (uint32_t)(L - (int)a.k + 1)) + 8u + (((uint32_t)L + 7u) & ~7u);
}

// The one layout of a whole-read exact answer ({L}= along strand s, L - k + 1 nodes): writes the record of read r at heap
// offset `off` and the read's header, the same bytes align_read writes for it, padding as zeros; a record past the end
// of the heap marks the read MGB_READ_OVERFLOW (the next pass retries it). node(t) / chr(t): the strand's node id t and
// prepared character t. Lanes `lane` of `width` share the copies.
template <class Node, class Chr>
MGB_HD void exact_record_write(const ExactArgs &a, uint32_t r, int L, int s, score_t score, uint64_t off, Node node, Chr chr,
                               int lane, int width) {
    const int nk = L - (int)a.k + 1;
    ReadHdr h;
    h.status = MGB_READ_OK; h.n_aln = 1; h.heap_off = off;
    h.stats.num_seeds = (uint32_t)nk; h.stats.num_extensions = 1;
    h.stats.num_explored_nodes = 0; h.stats.dp_columns = 0; h.stats.dp_cells = 0;
    if (off + exact_read_bytes(a, L) > a.heap_cap) {
        h.status = MGB_READ_OVERFLOW; h.n_aln = 0; h.heap_off = 0;
    } else {
        char *p = a.heap + off;
        if (lane == 0) {
            OutAln o;
            o.orientation = (uint32_t)s; o.score = score; o.offset = 0; o.query_begin = 0; o.query_len = (uint32_t)L;
            o.n_nodes = (uint32_t)nk; o.seq_len = (uint32_t)L; o.n_cigar = 1;
            *reinterpret_cast<OutAln*>(p) = o;
        }
        p += sizeof(OutAln);
        if (!a.result_nodes) {
            for (int t = lane; t < nk; t += width) reinterpret_cast<uint64_t*>(p)[t] = node(t);
            p += 8ull * nk;
        }
        if (lane == 0) *reinterpret_cast<unsigned long long*>(p) = cig_pack(OP_M, (uint32_t)L);
        p += 8;
        for (int t = lane; t < ((L + 7) & ~7); t += width) p[t] = t < L ? chr(t) : 0;
    }
    if (lane == 0) a.hdr[r] = h;
}

// exact_record_write from the seeding kernel's node arrays and the prepared strands
MGB_HD void exact_read_write(const ExactArgs &a, uint32_t r, uint64_t b, int L, int s, score_t score, uint64_t off,
                             int lane, int width) {
    const uint64_t *qn = (s ? a.nodes_r : a.nodes_f) + a.koff[r];
    const char *q = (s ? a.qr : a.qf) + b;
    exact_record_write(a, r, L, s, score, off, [qn](int t) { return qn[t]; }, [q](int t) { return q[t]; }, lane, width);
}

#if MGB_DEVICE_CODE
// One k-mer lookup in the hash index (kh_lookup) in three parts, so that a lane keeps several in flight: issue() loads
// the k-mer's bucket (nothing when `on` is false), find() settles it (a full bucket without the k-mer continues in the
// next one, rare at this load factor), value() loads the edge (0: not in the graph).
struct KhProbe {
    unsigned long long want;
    uint64_t slot;
    ulonglong2 ka, kb;
    int h;
    MGB_D void issue(const IndexView &ix, unsigned long long key, bool on) {
        want = key | (1ull << 63);
        slot = kh_slot_of(want, ix.kh_slots);
        ka = make_ulonglong2(0ull, 0ull); kb = ka;
        if (on) {
            ka = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + slot));
            kb = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + slot + 2));
        }
    }
    MGB_D void find(const IndexView &ix) {
        h = ka.x == want ? 0 : ka.y == want ? 1 : kb.x == want ? 2 : kb.y == want ? 3 : -1;
        bool more = h < 0 && ka.x != 0 && ka.y != 0 && kb.x != 0 && kb.y != 0;     // never when not issued
        while (more) {
            slot += 4; if (slot >= ix.kh_slots) slot = 0;
            const ulonglong2 x = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + slot));
            const ulonglong2 y = __ldg(reinterpret_cast<const ulonglong2*>(ix.kh_keys + slot + 2));
            h = x.x == want ? 0 : x.y == want ? 1 : y.x == want ? 2 : y.y == want ? 3 : -1;
            more = h < 0 && x.x != 0 && x.y != 0 && y.x != 0 && y.y != 0;
        }
    }
    MGB_D uint64_t value(const IndexView &ix) const { return h >= 0 ? __ldg(ix.kh_vals + slot + h) : 0u; }
};
#endif

// Whole-read exact answers straight from the raw characters (k_prepare_exact, in place of k_prepare): a read is answered
// here only if
//   1. k <= L <= max_len, and every character is A, C, G or T (after sanitize_char);
//   2. of the position-0 k-mers of the two strands exactly one is in the hash index (the primary strand), its edge is
//      in_graph and has a place p on the path layout;
//   3. pl_text[p .. p + L) is the primary strand, no pl_stop bit is set in [p, p + L - k + 1) and no pl_rc bit in the same
//      range;
//   4. Σ diag over the primary strand plus both end bonuses >= min_score.
// k_seed_hash would then walk the read paired (2), and the primary's walk would stay on the path to the end (3: each next
// character is the path's, the path goes on): it stores pl_node[p .. p + nk) on the primary. Every secondary k-mer is the
// reverse complement of a primary k-mer (1: no invalid window) whose pl_rc bit is 0, so its lookup misses and it stores 0.
// So exact_read_strand would take the primary with the same score (4), and the record is exact_record_write's with
// node ids pl_node[p + t]. Every other read is prepared as by prepare_read and seeded; k_exact_reads still answers the
// exact ones among them (across a path end, with a pl_rc bit set, ...). DESIGN.md §3.3.
struct PrepExactArgs {
    IndexView ix;                // with the k-mer hash index and the path layout
    PrepArgs prep;                // the raw reads, and the strand buffers of the reads left over
    ExactArgs ex;                 // k, end_bonus, min_score, max_len, result_nodes, diag; hdr and the heap
    uint32_t *list; unsigned int *n_list;            // the reads left over (prepared, to be seeded)
    unsigned long long *phase_out;   // MGB_PREP_TIMERS builds: cycles per PrepPhase, summed over the threads
    uint32_t stage_bytes;            // k_prepare_exact's shared memory for a tile's characters (prep_stage_bytes)
};

// k_prepare_exact stages a tile's characters in shared memory from the 16-byte word holding its first byte to
// kPrepStageSlack bytes past its last (the word reads of exact_path_strand go up to 35 past a read), rounded up to 16
// bytes: 256 * L_max + 80 bytes hold any tile of 256 reads, at most kPrepStageMax (below the 48 KB a block may use without opting in;
// a longer tile is read from global memory). The read buffer is padded by 64 bytes, so the copy stays inside it.
static constexpr uint32_t kPrepStageSlack = 48, kPrepStageMax = 45 * 1024;
MGB_HOSTDEV uint32_t prep_stage_bytes(uint32_t L_max) {
    const uint64_t need = 256ull * L_max + 32 + kPrepStageSlack;          // rounding both ends to 16 adds <= 30
    return need < kPrepStageMax ? (uint32_t)need : kPrepStageMax;
}

// MGB_PREP_TIMERS builds (scripts/build_variant.sh): clock64 cycles of each thread of k_prepare_exact per phase, printed
// per read under MGB_DEBUG. A thread's time from one lap to the next goes to the phase named at the lap; a read that
// leaves the gate early adds its time to the next phase the thread reaches. Compiled out of the product build.
enum PrepPhase : int { PREP_STAGE, PREP_KEYS, PREP_LOOKUP, PREP_STOPRC, PREP_TEXT, PREP_ALLOC, PREP_WRITE, PREP_LEFT,
                       PREP_N_PHASES };
struct PrepTimer {
#if defined(MGB_PREP_TIMERS) && MGB_DEVICE_CODE
    long long c[PREP_N_PHASES] = {}, t0 = 0;
    MGB_D void start() { t0 = clock64(); }
    MGB_D void lap(int ph) { const long long t = clock64(); c[ph] += t - t0; t0 = t; }
#else
    MGB_HD void start() {}
    MGB_HD void lap(int) {}
#endif
};

MGB_HD unsigned long long ldg64(const unsigned long long *p) {
#if MGB_DEVICE_CODE
    return __ldg(p);
#else
    return *p;
#endif
}
MGB_HD ulonglong2 ldg128(const ulonglong2 *p) {
#if MGB_DEVICE_CODE
    return __ldg(p);
#else
    return *p;
#endif
}
// The primary strand (0 / 1) of a read if it is answered here (conditions above), else -1; raw / n: its characters
// and length, *pos: its place p on the path, *score: the alignment's score. One lane, no collectives. The characters
// are read as aligned 4-byte words (acgt_pack32: up to 35 bytes past the read must be readable) and handled as 2-bit
// codes 32 at a time; both strands run the same word operations. The path layout is read in chunks of kPathChunk
// characters, all words of a chunk loaded before any is used. With kh_pos and pl_word (IndexView) a read's index
// accesses are the two buckets, one kh_pos entry and one 16-byte pl_word per 32 positions, three dependent steps;
// without them, kh_vals then pl_pos, and pl_stop, pl_rc and pl_text words apart.
static constexpr int kPathChunk = 160;
static constexpr int kChunkWords = kPathChunk / 32;
MGB_HD int exact_path_strand(const PrepExactArgs &a, const uint8_t *raw, int n, uint32_t *pos, score_t *score,
                             PrepTimer &tm) {
    const IndexView &ix = a.ix;
    const int K = (int)a.ex.k;
    if (n < K || n > (int)a.ex.max_len) return -1;
    // ---- the position-0 k-mers of both strands: codes [0, k) forward, [L - k, L) reverse-complemented. Their
    // characters are checked with the whole read below; an invalid one only makes a lookup that cannot matter.
    uint32_t inv;
    const unsigned long long kf = acgt_pack32(raw, &inv) & codes_mask(K);
    const unsigned long long kr = rc_codes32(acgt_pack32(raw + (n - K), &inv)) >> (2 * (32 - K));
    tm.lap(PREP_KEYS);
    int s;
    uint32_t p;
#if MGB_DEVICE_CODE
    {
        KhProbe pf, pr;                                     // both lookups in flight
        pf.issue(ix, kf, true); pr.issue(ix, kr, true);
        pf.find(ix); pr.find(ix);
        if ((pf.h >= 0) == (pr.h >= 0)) return -1;          // (a found k-mer's edge is never 0)
        s = pf.h >= 0 ? 0 : 1;
        const uint64_t i = s ? pr.slot + pr.h : pf.slot + pf.h;
#if defined(MGB_PROBE_NO_LAYOUT)
        // probe build (scripts/build_variant.sh), wrong results by design: no load after the buckets (no kh_pos,
        // kh_vals, pl_pos or layout words), every read whose primary k-mer is found passes the layout checks at p = 0
        p = 0; (void)i;
#else
        if (ix.kh_pos) {
            p = __ldg(ix.kh_pos + i);
        } else {
            const uint64_t e = __ldg(ix.kh_vals + i);
            p = in_graph(ix, e) ? __ldg(ix.pl_pos + e) : kPlNone;
        }
#endif
    }
#else
    {
        const uint64_t ef = kh_lookup(ix, kf), er = kh_lookup(ix, kr);
        if ((ef != 0) == (er != 0)) return -1;
        s = ef ? 0 : 1;
        const uint64_t e = s ? er : ef;
        p = in_graph(ix, e) ? ix.pl_pos[e] : kPlNone;
    }
#endif
    tm.lap(PREP_LOOKUP);
    if (p == kPlNone) return -1;
    const int nk = n - K + 1;
    int cnt[4] = { 0, 0, 0, 0 };                            // A, C, G, T on the primary strand
    for (int i0 = 0; i0 < n; i0 += kPathChunk) {
        // ---- the layout words of path positions [P, P + kPathChunk): pl_stop / pl_rc over [p, p + nk) (a 0 stop bit
        // at p + 1 .. p + nk - 1 keeps the path going, p is a node), pl_text over [p, p + L); all issued first
        const uint32_t P = p + (uint32_t)i0, w0 = P >> 5;
        const uint32_t se = p + (uint32_t)(i0 + kPathChunk < nk ? i0 + kPathChunk : nk);
        const uint32_t te = p + (uint32_t)(i0 + kPathChunk < n ? i0 + kPathChunk : n);
        uint32_t sr[kChunkWords + 1];                       // pl_stop | pl_rc
        unsigned long long tx[kChunkWords + 1];
#if defined(MGB_PROBE_NO_LAYOUT) && MGB_DEVICE_CODE
        (void)se; (void)te;
        for (int t = 0; t <= kChunkWords; ++t) { tx[t] = 0ull; sr[t] = 0u; }
#else
        if (ix.pl_word) {
#if MGB_DEVICE_CODE
            #pragma unroll
#endif
            for (int t = 0; t <= kChunkWords; ++t) {
                const uint32_t q = (w0 + (uint32_t)t) << 5;
                const ulonglong2 w = q < te ? ldg128(ix.pl_word + w0 + t) : ulonglong2{ 0ull, 0ull };
                tx[t] = w.x;
                sr[t] = q < se ? (uint32_t)w.y : 0u;
            }
        } else {
            uint32_t st[kChunkWords + 1], rc[kChunkWords + 1];
#if MGB_DEVICE_CODE
            #pragma unroll
#endif
            for (int t = 0; t <= kChunkWords; ++t) {
                const uint32_t q = (w0 + (uint32_t)t) << 5;
                st[t] = q < se ? ldg32(ix.pl_stop + w0 + t) : 0u;
                rc[t] = q < se ? ldg32(ix.pl_rc + w0 + t) : 0u;
                tx[t] = q < te ? ldg64(ix.pl_text + w0 + t) : 0ull;
            }
#if MGB_DEVICE_CODE
            #pragma unroll
#endif
            for (int t = 0; t <= kChunkWords; ++t) sr[t] = st[t] | rc[t];
        }
#endif
        uint32_t stop = 0;
#if MGB_DEVICE_CODE
        #pragma unroll
#endif
        for (int t = 0; t <= kChunkWords; ++t) {
            const uint32_t q = (w0 + (uint32_t)t) << 5;
            if (q < se) {
                uint32_t m = q < P ? ~0u << (P - q) : ~0u;
                if (se - q < 32) m &= (1u << (se - q)) - 1u;
                stop |= sr[t] & m;
            }
        }
        tm.lap(PREP_STOPRC);
        // ---- the primary strand's codes i0 + 32 j .. against pl_text, every character checked for A/C/G/T, the
        // per-letter counts on the way. Strand 1's code i is 3 - code n - 1 - i forward: the 32 bytes ending there,
        // reverse-complemented (near the read's start, the bytes from 0 and the codes shifted into place).
        const uint32_t sh = 2 * (P & 31);
        unsigned long long diff = 0;
        uint32_t bad = 0;
#if MGB_DEVICE_CODE
        #pragma unroll
#endif
        for (int j = 0; j < kChunkWords; ++j) {
            const int i = i0 + 32 * j;
            if (i < n) {
                const int m = n - i < 32 ? n - i : 32;
                const int q = s ? n - i - 32 : i;
                const unsigned long long x = acgt_pack32(raw + (q > 0 ? q : 0), &inv);
                const unsigned long long xr = rc_codes32(x) >> (q < 0 ? -2 * q : 0);
                const unsigned long long c = s ? xr : x, cm = codes_mask(m);
                bad |= inv & (m < 32 ? (1u << m) - 1u : ~0u);
                unsigned long long t = tx[j] >> sh;
                if (sh) t |= tx[j + 1] << (64 - sh);
                diff |= (c ^ t) & cm;
                acgt_count(c, cm, cnt);
            }
        }
        tm.lap(PREP_TEXT);
#if defined(MGB_PROBE_NO_LAYOUT) && MGB_DEVICE_CODE
        diff = 0;
#endif
        if (stop || bad || diff) return -1;
    }
    const score_t full = cnt[0] * a.ex.diag['A'] + cnt[1] * a.ex.diag['C'] + cnt[2] * a.ex.diag['G']
                       + cnt[3] * a.ex.diag['T'] + a.ex.end_bonus;
    if (full < a.ex.min_score) return -1;
#if defined(MGB_HOST_EMU)
    ++mgb_emu_path_read_hits;
#endif
    *pos = p; *score = full;
    return s;
}

// Word wi of the record of a read exact_path_strand answered (raw / L / s / p / score: its characters, length, strand,
// place on the path and score): exact_record_write's bytes with node ids pl_node[p + t] and the strand's characters from
// the raw read (sanitize_char, complement_char: the read is all A/C/G/T), padding as zeros.
static_assert(sizeof(OutAln) == 32, "OutAln is four words");
MGB_HD unsigned long long exact_path_word(const PrepExactArgs &a, const uint8_t *raw, int L, int s, uint32_t p,
                                          score_t score, uint32_t wi) {
    const uint32_t nk = (uint32_t)(L - (int)a.ex.k + 1), nn = a.ex.result_nodes ? 0u : nk;
    if (wi < 4) {            // OutAln: orientation, score | offset, query_begin | query_len, n_nodes | seq_len, n_cigar
        const uint32_t lo = wi == 0 ? (uint32_t)s : wi == 1 ? 0u : (uint32_t)L;
        const uint32_t hi = wi == 0 ? (uint32_t)score : wi == 1 ? 0u : wi == 2 ? nk : 1u;
        return lo | (unsigned long long)hi << 32;
    }
    wi -= 4;
    if (wi < nn) return ldg32(a.ix.pl_node + p + wi);
    wi -= nn;
    if (wi == 0) return cig_pack(OP_M, (uint32_t)L);
    const int j = 8 * (int)(wi - 1);                    // characters j .. j + 7 of the strand
    const int q = s ? L - 8 - j : j;                    // ... from the raw bytes q .. q + 7
    unsigned long long x = bytes8_at(raw + (q > 0 ? q : 0));
    if (q < 0) x <<= -8 * q;
    x = acgt_chars8(x, s != 0);
    if (L - j < 8) x &= (1ull << (8 * (L - j))) - 1;
    return x;
}
// the record of such a read at heap offset `off` (which fits), lanes `lane` of `width` one word each
MGB_HD void exact_path_write(const PrepExactArgs &a, const uint8_t *raw, int L, int s, uint32_t p, score_t score,
                             uint64_t off, int lane, int width) {
    unsigned long long *o = reinterpret_cast<unsigned long long*>(a.ex.heap + off);
    const uint32_t nw = exact_read_bytes(a.ex, L) / 8;
    for (uint32_t wi = (uint32_t)lane; wi < nw; wi += (uint32_t)width) o[wi] = exact_path_word(a, raw, L, s, p, score, wi);
}
// ... and word qi (< 5) of its header, exact_record_write's: status, n_aln | heap_off | num_seeds, num_extensions |
// num_explored_nodes, dp_columns | dp_cells
static_assert(sizeof(ReadHdr) == 40 && MGB_READ_OK == 0, "ReadHdr is five words");
MGB_HD unsigned long long exact_path_hdr_word(const ExactArgs &a, int L, uint64_t off, int qi) {
    return qi == 0 ? 1ull << 32 : qi == 1 ? off : qi == 2 ? (uint32_t)(L - (int)a.k + 1) | 1ull << 32 : 0ull;
}
MGB_HD void exact_path_hdr(const ExactArgs &a, uint32_t r, int L, uint64_t off) {
    unsigned long long *h = reinterpret_cast<unsigned long long*>(a.hdr + r);
    for (int qi = 0; qi < 5; ++qi) h[qi] = exact_path_hdr_word(a, L, off, qi);
}

// One refinement level of the suffix-range table (boss.hpp:651-655 index order: the appended
// character is the most significant digit): entry o = idx + (c-1)*cur_num of the new table is
// tighten_range(cur[idx], c).
struct SfxArgs { IndexView ix; const uint32_t *cur; uint32_t *nxt; uint64_t cur_num; };

MGB_HD void sfx_extend_item(const SfxArgs &a, uint64_t o) {
    const uint64_t idx = o % a.cur_num;
    const uint32_t c = (uint32_t)(o / a.cur_num) + 1;
    uint64_t rl = a.cur[2 * idx], ru = (uint64_t)a.cur[2 * idx + 1] - 1;
    uint32_t b = 1, e = 1;
    if (rl <= ru && tighten_range(a.ix, &rl, &ru, c)) { b = (uint32_t)rl; e = (uint32_t)(ru + 1); }
    if (glane() == 0) { a.nxt[2 * o] = b; a.nxt[2 * o + 1] = e; }
}

// Reverse adjacency construction (index.cuh load_radj): per edge bwd(e) + "source node has several
// incoming edges", then k-2 gather rounds c_{j+1}[e] = c_j[bwd(e)] that move the last node character
// (boss.cpp:679-690) to the first position of the k-mer.
struct RadjArgs { IndexView ix; uint32_t *bwd_arr; uint8_t *c_cur; uint8_t *c_nxt; uint8_t *multi; uint2 *radj; uint64_t n;
                  // k-mer hash index build (nullptr: not built): the packed k-mer of every edge, accumulated over the same
                  // gather rounds that move the node's last character to the first position
                  unsigned long long *kmer; };
static constexpr unsigned long long kKmerBad = ~0ull;      // the k-mer holds a '$'
inline uint32_t radj_multi_shift(const IndexView &ix) { return ix.wide ? 7u : 3u; }   // index.cuh radj_multi

MGB_HD void radj_bwd_item(const RadjArgs &a, uint64_t e) {
    LineCache lc;
    uint64_t x = bwd(a.ix, lc, e);
    uint32_t d = node_last_value(a.ix, e);
    uint32_t multi = 0;
    if (x + 1 <= a.ix.n) {
        uint32_t w;
        succ_W2(a.ix, lc, x + 1, d, &w);
        multi = w == d + a.ix.sigma;
    }
    if (a.kmer) {
        // last two characters of the k-mer: the edge label and the node's last character
        const uint32_t lab = lc.get_W(a.ix, e) % a.ix.sigma;
        const uint32_t K = a.ix.k;
        if (glane() == 0)
            a.kmer[e] = (lab == 0 || d == 0) ? kKmerBad
                      : ((unsigned long long)(lab - 1) << (2 * (K - 1))) | ((unsigned long long)(d - 1) << (2 * (K - 2)));
    }
    if (glane() == 0) { a.bwd_arr[e] = (uint32_t)x; a.c_cur[e] = (uint8_t)d; a.multi[e] = (uint8_t)multi; }
}

// PRIMARY graphs: the rc-strand jump tables of IndexView (rcs / rcp / palin) for edge e. The k-mer is spelled
// through the reverse adjacency records (BOSS::get_node_seq, boss.cpp:953-973), its two (k-1)-mers are reverse
// complemented and looked up (NodeFirstCache::get_suffix_rc / get_prefix_rc, node_first_cache.cpp:122-176).
constexpr int kMaxPrimaryK = 128;
struct RcArgs { IndexView ix; uint32_t *rcs; uint32_t *rcp; uint32_t *palin; uint64_t n; };
MGB_HD void rc_tables_item(const RcArgs &a, uint64_t e) {
    const IndexView &ix = a.ix;
    const int K = (int)ix.k;
    uint8_t km[kMaxPrimaryK];
    {
        LineCache lc;
        km[K - 1] = (uint8_t)(lc.get_W(ix, e) % ix.sigma);
        uint64_t cur = e;
        for (int i = K - 2; i >= 0; --i) {
            km[i] = (uint8_t)node_last_value(ix, cur);
            cur = load_radj(ix, cur).x;
        }
    }
    uint8_t rc[kMaxPrimaryK];
    uint32_t r_s = 0, r_p = 0;
    bool clean = true;                                   // no '$' in x[1..k)
    for (int i = 1; i < K; ++i) clean = clean && km[i] != 0;
    if (clean) {
        for (int t = 0; t < K - 1; ++t) rc[t] = (uint8_t)(ix.sigma - km[K - 1 - t]);
        uint64_t first, lst; int matched;
        boss_index_range(ix, rc, K - 1, &first, &lst, &matched);
        if (matched == K - 1) r_s = (uint32_t)lst;
    }
    if (km[0] != 0) {                                    // then x[0..k-1) holds no '$' at all
        for (int t = 0; t < K - 1; ++t) rc[t] = (uint8_t)(ix.sigma - km[K - 2 - t]);
        uint64_t first, lst; int matched;
        boss_index_range(ix, rc, K - 1, &first, &lst, &matched);
        if (matched == K - 1) r_p = (uint32_t)lst;
    }
    bool pal = a.palin != nullptr && clean && km[0] != 0;
    for (int t = 0; t < K && pal; ++t) pal = km[t] == ix.sigma - km[K - 1 - t];
    if (glane() == 0) {
        a.rcs[e] = r_s; a.rcp[e] = r_p;
        if (pal) {
#if MGB_DEVICE_CODE
            atomicOr(a.palin + (e >> 5), 1u << (e & 31));
#else
            a.palin[e >> 5] |= 1u << (e & 31);
#endif
        }
    }
}

} // namespace mgb

#if !defined(MGB_HOST_EMU)
namespace MGB_KERNEL_NS {
using namespace mgb;

#if !defined(MGB_ALIGN_KERNEL_ONLY)
__global__ void __launch_bounds__(128) k_radj_bwd(RadjArgs a) {
    uint64_t quad = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    uint64_t nquads = ((uint64_t)gridDim.x * blockDim.x) >> 2;
    for (uint64_t e = 1 + quad; e <= a.n; e += nquads) radj_bwd_item(a, e);
}

__global__ void __launch_bounds__(128) k_sfx_extend(SfxArgs a) {
    uint64_t quad = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    uint64_t nquads = ((uint64_t)gridDim.x * blockDim.x) >> 2;
    const uint64_t total = a.cur_num * (a.ix.sigma - 1);
    for (uint64_t o = quad; o < total; o += nquads) sfx_extend_item(a, o);
}

// Sub-k lookups (subk_item) for 32 query positions of one strand per warp. Most positions end with one load: the
// first sfx_len characters do not occur in the graph, and a miss in a suffix-range table no longer than
// min_seed_length is final (boss_index_range). So every LANE first settles its own position against the table;
// only the survivors (a matched prefix of at least sfx_len characters: near an error on the matching strand) go
// through the quad-cooperative range search, 8 at a time. (One quad per position kept 4 lanes on every one-load
// miss.) Same results as subk_item(), which the host emulation still runs.
__global__ void __launch_bounds__(128) k_subk(SubkArgs a, uint32_t chunks_per_strand) {
    const IndexView &ix = a.ix;
    const int K = (int)ix.k;
    const int lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint32_t blocks32 = (chunks_per_strand * (uint32_t)kSubkChunk + 31) / 32;    // 32-position blocks per strand
    const uint64_t per_read = (uint64_t)a.n_strands * blocks32;
    const uint64_t items = (uint64_t)a.n_reads * per_read;
    const int S = (int)ix.sfx_len;
    const uint64_t base = ix.sigma - 1;
    for (uint64_t it = warp; it < items; it += nwarps) {
        const uint32_t r = (uint32_t)(it / per_read), rem = (uint32_t)(it % per_read);
        const uint32_t s = rem / blocks32, blk = rem % blocks32;
        const uint64_t b = a.offsets[r];
        const int L = (int)(a.offsets[r + 1] - b);
        if (L < (int)a.min_seed_length) continue;
        const int n_pos = L - (int)a.min_seed_length + 1;
        const uint8_t *codes = (s ? a.cr : a.cf) + b;
        const uint64_t *nodes = L >= K ? (s ? a.nodes_r : a.nodes_f) + a.koff[r] : nullptr;
        uint32_t *of = (s ? a.first_r : a.first_f) + b, *ol = (s ? a.last_r : a.last_f) + b;
        uint8_t *on = (s ? a.len_r : a.len_f) + b;
        const int nk = L >= K ? L - K + 1 : 0;
        const int i = (int)blk * 32 + lane;
        // ---- per lane: positions that need no search
        bool survivor = false;
        int len = 0;
        if (i < n_pos) {
            if (i < nk && nodes && nodes[i] != 0) {
                of[i] = 0; ol[i] = 0; on[i] = 0xFF;                 // a full k-mer matches here: not computed
            } else {
                len = (int)a.max_len < L - i ? (int)a.max_len : L - i;
                bool ok = len >= (int)a.min_seed_length;
                bool zero = false;
                for (int t = 0; t < len && ok; ++t) { const uint32_t c = codes[i + t]; ok = c < ix.sigma; zero = zero || c == 0; }
                const int qlen = len < K - 1 ? len : K - 1;         // what boss_index_range is asked for
                survivor = ok;
                if (ok && S && S <= qlen && S <= (int)a.min_seed_length && !zero && S > 1) {
                    uint64_t slot = 0;
                    for (int j = S - 1; j >= 0; --j) slot = slot * base + (codes[i + j] - 1);
                    const uint32_t rl = ldg32(ix.sfx + 2 * slot), ru1 = ldg32(ix.sfx + 2 * slot + 1);
                    if (rl >= ru1) survivor = false;                // empty range: matched = 0, final
                }
                if (!survivor) { of[i] = 0; ol[i] = 0; on[i] = 0; }
            }
        }
        // ---- the survivors, 8 per round, one quad each
        uint32_t todo = __ballot_sync(0xffffffffu, survivor);
        while (todo) {
            // the (lane >> 2)-th set bit of `todo` is this quad's position, if there are that many
            const int q = lane >> 2;
            const int src = popc32(todo) > q ? nth_set32(todo, q + 1) : -1;
            if (src >= 0) {
                const int pi = (int)blk * 32 + src;
                const int plen = (int)a.max_len < L - pi ? (int)a.max_len : L - pi;
                uint64_t first = 0, lst = 0; int matched = 0;
                boss_index_range(ix, codes + pi, plen < K - 1 ? plen : K - 1, &first, &lst, &matched, (int)a.min_seed_length);
                if (glane() == 0) { of[pi] = (uint32_t)first; ol[pi] = (uint32_t)lst; on[pi] = (uint8_t)matched; }
            }
            // drop the (up to) 8 lowest set bits
            for (int t = 0; t < 8 && todo; ++t) todo &= todo - 1;
        }
    }
}

// one warp per read strand
__global__ void __launch_bounds__(256) k_premap(SeedArgs a) {
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / kWarp;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) / kWarp;
    const uint64_t items = (uint64_t)a.n_reads * a.n_strands;
    for (uint64_t it = warp; it < items; it += nwarps) premap_item(a, (uint32_t)(it / a.n_strands), (uint32_t)(it % a.n_strands));
}

// BOSS::map_to_edges (boss.cpp:996-1045) for 32 read strands per warp, one per lane. The two regimes of the walk
// have opposite shapes, so the warp alternates between them instead of letting every strand run its own loop:
//   cold  a k-mer is looked up from scratch (BOSS::index: suffix-range table + tighten_range steps over 64-byte
//         blocks): quad-cooperative, 8 strands at a time, the strand's state fetched from / returned to its lane;
//   warm  the next k-mer is the child of the current edge: ONE 8-byte adjacency load per step and lane, 32
//         independent pointer chases per warp, all lanes in the same three-instruction-deep loop.
// (One quad per strand running both regimes kept 8 of 32 lanes busy on average: 8 quads in 8 different states.)
// Same results as map_to_edges() in seed_core.cuh, which the host emulation still runs. Graphs with the k-mer hash
// index take k_seed_hash instead.
__global__ void __launch_bounds__(128) k_seed(SeedArgs a) {
    const IndexView &ix = a.ix;
    const int K = (int)ix.k;
    const int lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t items = (uint64_t)a.n_reads * a.n_strands;
    const int S = (ix.sfx_len && (int)ix.sfx_len <= K - 1) ? (int)ix.sfx_len : 0;
    const uint64_t base = ix.sigma - 1;
    for (uint64_t chunk = warp * 32; chunk < items; chunk += nwarps * 32) {
        const uint64_t item = chunk + lane;
        // this lane's strand
        const uint8_t *codes = nullptr; uint64_t *out = nullptr; const uint32_t *hints = nullptr;
        int nk = 0;
        if (item < items) {
            const uint32_t r = (uint32_t)(item / a.n_strands), s = (uint32_t)(item % a.n_strands);
            const uint64_t b = a.offsets[r];
            const int L = (int)(a.offsets[r + 1] - b);
            nk = L >= K ? L - K + 1 : 0;
            codes = (s ? a.cr : a.cf) + b;
            out = (s ? a.nodes_r : a.nodes_f) + a.koff[r];
            hints = a.hinted ? (s ? a.hint_r : a.hint_f) + (a.koff[r] >> 5) + r : nullptr;
        }
        int pos = 0;                 // first k-mer not resolved yet
        uint64_t edge = 0;           // warm: the edge of k-mer pos - 1
        while (__any_sync(0xffffffffu, pos < nk)) {
            if (pos >= nk) edge = 0;
            // ---- cold: strands without an edge look for their next k-mer that exists. The quads take the waiting
            // strands in lane order, 8 per round (quad q serves the q-th waiting lane)
            uint32_t waiting = __ballot_sync(0xffffffffu, edge == 0 && pos < nk);
            while (waiting) {
                const int q = lane >> 2;
                const bool need = popc32(waiting) > q;
                const int src = need ? nth_set32(waiting, q + 1) : 0;
                const uint64_t codes_s = __shfl_sync(0xffffffffu, (unsigned long long)codes, src);
                const uint64_t hints_s = __shfl_sync(0xffffffffu, (unsigned long long)hints, src);
                const uint64_t out_s = __shfl_sync(0xffffffffu, (unsigned long long)out, src);
                const int nk_s = __shfl_sync(0xffffffffu, nk, src);
                int i = __shfl_sync(0xffffffffu, pos, src);
                uint64_t found = 0;
                if (need) {                                            // uniform within the quad
                    const uint8_t *cd = (const uint8_t*)codes_s;
                    const uint32_t *hn = (const uint32_t*)hints_s;
                    LineCache lc;
                    for (; i < nk_s; ++i) {
                        if (hn) { i = next_hint(hn, nk_s, i); if (i >= nk_s) break; }
                        // map_to_edge (boss.hpp:766-777)
                        bool valid = true, zero = false;
                        for (int j = 0; j < K; ++j) { const uint32_t c = cd[i + j]; valid = valid && c < ix.sigma; zero = zero || c == 0; }
                        uint64_t e = 0;
                        if (valid) {
                            if (S && !zero) {
                                uint64_t slot = 0;
                                for (int j = S - 1; j >= 0; --j) slot = slot * base + (cd[i + j] - 1);
                                e = boss_index_slot(ix, cd + i, K - 1, slot);
                            } else {
                                e = boss_index(ix, cd + i, K - 1);
                            }
                            if (e) e = pick_edge(ix, lc, e, cd[i + K - 1]);
                        }
                        if (e) { found = e; break; }
                    }
                    if (found && glane() == 0) ((uint64_t*)out_s)[i] = in_graph(ix, found) ? found : 0;
                }
                // back to the strand's lane: the r-th waiting lane was served by quad r (if r < 8)
                const int my_rank = popc32(waiting & ((1u << lane) - 1u));
                const bool served = ((waiting >> lane) & 1u) && my_rank < 8;
                const uint64_t f_back = __shfl_sync(0xffffffffu, (unsigned long long)found, 4 * (my_rank & 7));
                const int i_back = __shfl_sync(0xffffffffu, i, 4 * (my_rank & 7));
                if (served) {
                    edge = f_back;
                    pos = f_back ? i_back + 1 : nk;                    // nothing left to find: the strand is done
                }
                for (int t = 0; t < 8 && waiting; ++t) waiting &= waiting - 1;
            }
            // ---- warm: every lane with an edge follows it (boss.cpp:1024-1043) until its next k-mer is missing; the
            // warp goes back to cold lookups once 8 strands wait for one (a full round of quads), or nobody is warm
            while (true) {
                const bool warm = edge != 0 && pos < nk;
                // one warp reduction counts both kinds of lanes: warm ones in the low byte, waiting ones above
                const uint32_t cnt = __reduce_add_sync(0xffffffffu, warm ? 1u : ((edge == 0 && pos < nk) ? 256u : 0u));
                if (!(cnt & 255u) || (cnt >> 8) >= 8u) break;
                if (warm) {
                    const uint32_t c = codes[pos + K - 1];
                    if (c >= ix.sigma) {                               // invalid character: this k-mer and the walk end
                        out[pos] = 0; edge = 0; ++pos;
                    } else if (!MGB_WIDE(ix)) {
                        const uint2 ar = load_adj(ix, edge);
                        edge = adj_child(ar, c);
                        out[pos] = (edge && ((ar.y >> (8 + c)) & 1u)) ? edge : 0;
                        ++pos;
                    } else {
                        const Adj ar = load_adj_any(ix, edge);
                        edge = adj_child(ar, c);
                        out[pos] = (edge && ((ar.ok >> c) & 1u)) ? edge : 0;
                        ++pos;
                    }
                }
            }
            if (pos >= nk) edge = 0;
        }
    }
}

#if !defined(MGB_WIDE_ONLY)
// k_seed_hash: threads per block and the blocks per SM its registers are sized for (build-time probes,
// scripts/build_variant.sh -D...; DESIGN.md §3.2 has the measurements).
#ifndef MGB_SEED_THREADS
#define MGB_SEED_THREADS 128
#endif
#ifndef MGB_SEED_MIN_BLOCKS
#define MGB_SEED_MIN_BLOCKS 5
#endif
static constexpr int kSeedThreads = MGB_SEED_THREADS;

// The characters of a strand in order, read 8 at a time: w0 is the aligned 8-byte word holding the next character,
// w1 the word after it, loaded 8 characters before it is needed. Words are only loaded if they hold a character of the
// strand (an aligned word never crosses a page). One byte load per character instead measured 19 % slower on c2 (2 strands per lane): with
// tens of thousands of strands in flight, their lines do not stay in L1 from one character to the next.
struct CodeStream {
    const uint8_t *p;             // next character
    int left;                     // characters from p to the end of the strand
    unsigned long long w0, w1;
    MGB_D void start(const uint8_t *codes, int L) {
        p = codes; left = L; w0 = 0; w1 = 0;
        const unsigned long long *w = reinterpret_cast<const unsigned long long*>((uintptr_t)codes & ~(uintptr_t)7);
        if (L > 0) w0 = __ldg(w);
        if (L > 8 - (int)((uintptr_t)codes & 7)) w1 = __ldg(w + 1);
    }
    MGB_D uint32_t next() {
        const uint32_t c = (uint32_t)(w0 >> (8 * ((uintptr_t)p & 7))) & 0xFFu;
        ++p; --left;
        if (((uintptr_t)p & 7) == 0) {
            w0 = w1;
            w1 = left > 8 ? __ldg(reinterpret_cast<const unsigned long long*>(p) + 1) : 0ull;
        }
        return c;
    }
};
// The same backwards, from the last character of the strand: w0 holds the next character, w1 is the word before it.
struct CodeStreamDown {
    const uint8_t *p;             // next character
    int left;                     // characters from the start of the strand to p, p included
    unsigned long long w0, w1;
    MGB_D void start(const uint8_t *codes, int L) {
        p = codes + L - 1; left = L; w0 = 0; w1 = 0;
        const unsigned long long *w = reinterpret_cast<const unsigned long long*>((uintptr_t)p & ~(uintptr_t)7);
        if (L > 0) w0 = __ldg(w);
        if (L > 1 + (int)((uintptr_t)p & 7)) w1 = __ldg(w - 1);
    }
    MGB_D uint32_t next() {
        const uint32_t c = (uint32_t)(w0 >> (8 * ((uintptr_t)p & 7))) & 0xFFu;
        --left;
        if (((uintptr_t)p & 7) == 0) {
            w0 = w1;
            w1 = left > 8 ? __ldg(reinterpret_cast<const unsigned long long*>(p) - 2) : 0ull;
        }
        --p;
        return c;
    }
};

// Packed k-mer at position 0 of a strand (key = sum of (code_p - 1) << 2p); *last_bad = position of its last invalid
// character, -1 if none. The stream is left at position k.
MGB_D unsigned long long first_kmer(CodeStream &cs, const uint8_t *codes, int L, int K, uint32_t sigma, int *last_bad) {
    cs.start(codes, L);
    unsigned long long key = 0;
    int bad = -1;
    for (int j = 0; j < K; ++j) {
        const uint32_t c = cs.next();
        if (c < 1 || c >= sigma) bad = j;
        key = (key >> 2) | ((unsigned long long)((c - 1) & 3u) << (2 * (K - 1)));
    }
    *last_bad = bad;
    return key;
}

// Node ids of a strand leave in whole 32-byte sectors: s0..s3 are the slots of the sector being filled (slot q of
// node id i is (address / 8) % 4). A sector the strand shares with a neighbouring read gets single stores of the
// strand's own slots. Single 8-byte stores left sectors partly written in L2, and evicting one of those most likely
// costs the DRAM (ECC, no write mask) a read-modify-write (c2 prepare + seed: 19.3 ms -> 14.8 ms).
struct SectorOut {
    uint64_t s0, s1, s2, s3;
    MGB_D void clear() { s0 = s1 = s2 = s3 = 0; }
    MGB_D void put(int q, uint64_t v) {
        s0 = q == 0 ? v : s0; s1 = q == 1 ? v : s1; s2 = q == 2 ? v : s2; s3 = q == 3 ? v : s3;
    }
    MGB_D void flush(uint64_t *sec, int lo, int hi) {      // slots lo..hi
        if (lo == 0 && hi == 3) {
            reinterpret_cast<ulonglong2*>(sec)[0] = make_ulonglong2(s0, s1);
            reinterpret_cast<ulonglong2*>(sec)[1] = make_ulonglong2(s2, s3);
        } else {
            if (lo == 0) sec[0] = s0;
            if (lo <= 1 && hi >= 1) sec[1] = s1;
            if (lo <= 2 && hi >= 2) sec[2] = s2;
            if (hi == 3) sec[3] = s3;
        }
    }
    // ascending walk: node id v of k-mer `pos` of nk; stored once the sector is full or the strand ends. Zeros are
    // stored too.
    MGB_D void put_up(uint64_t *out, int pos, int nk, uint64_t v) {
        uint64_t *pa = out + pos;
        const int q = (int)(((uintptr_t)pa >> 3) & 3);
        put(q, v);
        if (q == 3 || pos == nk - 1) flush(pa - q, pos < q ? q - pos : 0, q);
    }
    // descending walk: node id v of k-mer j, sectors filled from slot 3 down. A sector of zeros is not stored: the
    // node arrays start zero-filled. (Slots of the first sector above the strand's last k-mer are 0 after clear().)
    MGB_D void put_down(uint64_t *out, int j, int nk, uint64_t v) {
        uint64_t *pa = out + j;
        const int q = (int)(((uintptr_t)pa >> 3) & 3);
        put(q, v);
        if ((q == 0 || j == 0) && (s0 | s1 | s2 | s3)) {
            const int hi = q + (nk - 1 - j);
            flush(pa - q, q, hi < 3 ? hi : 3);
        }
    }
};

// A walk along the path layout (IndexView::pl_*): the character, reverse-complement and stop bits of position q, read
// sequentially, each array by the aligned word that holds q. Words are loaded only when q enters them; the filler
// padding at the end of the layout keeps that inside the arrays. The node ids are not read here: k_seed_hash copies the
// run a whole warp at a time once the walk leaves it.
struct PathWalk {
    uint32_t q;                   // position of the k-mer the next step would reach
    bool on;                      // still on the path
    unsigned long long tw;        // pl_text word holding position q + k - 1 (the last character of q's k-mer)
    uint32_t rw, sw;              // pl_rc / pl_stop words holding q
    MGB_D void load(const IndexView &ix, bool all) {
        const uint32_t qt = q + ix.k - 1;
        if (all || (qt & 31) == 0) tw = __ldg(ix.pl_text + (qt >> 5));
        if (all || (q & 31) == 0) { rw = __ldg(ix.pl_rc + (q >> 5)); sw = __ldg(ix.pl_stop + (q >> 5)); }
    }
    // the walk's k-mer is the one of edge e (stored, so a DBG node): start after its position, if it has one
    MGB_D void start(const IndexView &ix, uint64_t e, bool stored) {
        const uint32_t p = stored && ix.pl_n ? __ldg(ix.pl_pos + e) : kPlNone;
        on = p != kPlNone;
        q = p + 1;
        tw = 0; rw = 0; sw = ~0u;
        if (on) load(ix, true);
    }
    // the next k-mer, whose last character is c (valid), is the one at q
    MGB_D bool next_is(const IndexView &ix, uint32_t c) const {
        return on && ((tw >> (2 * ((q + ix.k - 1) & 31))) & 3u) == c - 1 && !((sw >> (q & 31)) & 1u);
    }
    MGB_D bool rc() const { return (rw >> (q & 31)) & 1u; }
    MGB_D void step(const IndexView &ix) { ++q; load(ix, false); }
};

// k_seed_hash's short-list mode: one read per warp, every k-mer of the read looked up in the hash index on its own
// (map_to_edge for each k-mer, the lookup the walk below saves loads on), kSeedWideDepth lookups in flight per lane.
// A k-mer's node id is its edge if that is in_graph, else 0 (so is a window with an invalid character); the summary
// bits come from a warp-wide OR. There is no chain of dependent loads: a read costs about one round trip per
// kSeedWideDepth * 32 k-mers, where the walk's lane waits on one adjacency record or bucket per k-mer once it leaves the
// path layout. Kept out of line so that the walk's code and registers stay as they are. Warp w takes items w,
// w + warps, ...
static constexpr int kSeedWideDepth = 4;
// the short-list mode runs when the items are at most kSeedWideRounds per warp of the grid (DESIGN.md §3.2)
#ifndef MGB_SEED_WIDE_ROUNDS
#define MGB_SEED_WIDE_ROUNDS 1
#endif
static constexpr uint32_t kSeedWideRounds = MGB_SEED_WIDE_ROUNDS;
__device__ __noinline__ void seed_hash_wide(const SeedArgs &a, uint32_t n_items) {
    const IndexView &ix = a.ix;
    const int K = (int)ix.k;
    const uint32_t sigma = ix.sigma;
    const int ns = (int)a.n_strands;
    const int lane = (int)(threadIdx.x & 31);
    const uint32_t warps = gridDim.x * blockDim.x / kWarp;
    for (uint32_t it = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp; it < n_items; it += warps) {
        const uint32_t r = a.list ? __ldg(a.list + it) : it;
        const uint64_t b = a.offsets[r];
        const int L = (int)(a.offsets[r + 1] - b);
        const int nk = L >= K ? L - K + 1 : 0;
        const uint64_t ko = a.koff[r];
        const int n = ns * nk;                        // item j: k-mer j % nk of strand j / nk
        uint32_t seen = 0;                            // SeedArgs::summary bits of this lane's k-mers
        for (int base = 0; base < n; base += kWarp * kSeedWideDepth) {
            KhProbe p[kSeedWideDepth];
            #pragma unroll
            for (int d = 0; d < kSeedWideDepth; ++d) {
                const int j = base + d * kWarp + lane;
                const int s = j >= nk ? 1 : 0, i = j - s * nk;
                bool ok = j < n;
                unsigned long long key = 0;
                if (ok) {
                    const uint8_t *c = (s ? a.cr : a.cf) + b + i;
                    for (int t = 0; t < K; ++t) {
                        const uint32_t x = __ldg(c + t);
                        ok = ok && x >= 1 && x < sigma;
                        key |= (unsigned long long)((x - 1) & 3u) << (2 * t);
                    }
                }
                p[d].issue(ix, key, ok);
            }
            #pragma unroll
            for (int d = 0; d < kSeedWideDepth; ++d) p[d].find(ix);
            #pragma unroll
            for (int d = 0; d < kSeedWideDepth; ++d) {
                const int j = base + d * kWarp + lane;
                if (j < n) {
                    const int s = j >= nk ? 1 : 0, i = j - s * nk;
                    const uint64_t found = p[d].value(ix);
                    const bool store = found != 0 && in_graph(ix, found);
                    ((s ? a.nodes_r : a.nodes_f) + ko)[i] = store ? found : 0;
                    seen |= (store ? 2u : 1u) << (2 * s);
                }
            }
        }
        seen = __reduce_or_sync(0xffffffffu, seen);
        if (a.summary && lane == 0) a.summary[r] = (uint8_t)seen;
    }
}

// BOSS::map_to_edges (boss.cpp:996-1045) on graphs with the k-mer hash index (DNA block layout, k <= 31), one read per
// lane. A strand walked in order costs one load per k-mer: the adjacency record of the previous k-mer's edge while the
// walk is warm (boss.cpp:1024-1043), the k-mer's bucket (+ the value on a hit) when it is cold (map_to_edge,
// boss.hpp:766-777); the packed k-mer is a rolling value. The characters come from CodeStream, off the chain of the walk.
//
// With both strands, the lane first looks up position 0 of each. If exactly one of them hits, the read runs PAIRED:
// that strand (the primary) is walked in order, and the other one (the secondary) backwards in the same steps. The
// secondary's k-mer at j = nk - 1 - t is the reverse complement of the primary's at t when both windows are valid
// (pinned for the alphabet tables by tests/test_seed_pairing.py), and a random genome hardly ever holds both. So when
// the primary's k-mer at t came from a warm step, bit 16 + c of the record it came from (k_adj_rc) settles the
// secondary's k-mer with no load whenever it is 0. Otherwise the secondary looks it up cold. The secondary runs one step
// behind, so its lookup is issued together with the primary's load of the next step. Its key is a rolling value of its
// own characters, read backwards. Its first k-mer (position 0) is the probe's miss. If both probes hit (CANONICAL-mode
// graphs, regions stored in both orientations) or neither does (an error in the first k-mer), the strands are walked
// one after the other. (c2 prepare + seed: 14.8 ms -> 7.2 ms, DESIGN.md §3.2.)
//
// With the path layout, the strand walked in order starts at its probe's position on the path (PathWalk) and stays on the
// path while each next character is the path's and the path goes on: k-mer t is then the string stored at q, so its node
// id is pl_node[q] and pl_rc[q] stands in for the adjacency record's reverse-complement bit. Such a step loads nothing
// but the layout's character and bit words in order (one per 32 steps); when the secondary needs no lookup either it
// skips the lookup code altogether. The run's node ids are copied at the end of the pass, by the warp together. At the
// first mismatch, invalid character or path end the walk goes on as above from the last node on the path, and does not
// return to it. (c2 k_seed_hash: 6.0 ms -> 2.85 ms, DESIGN.md §3.2.)
//
// Steps are written with selects rather than branches: lanes in different regimes issue together. Persistent grid:
// lane t of n_lanes takes the reads t + n_lanes * round, or those entries of a.list (the reads k_prepare_exact left over).
// A short list (at most kSeedWideRounds reads per warp of the grid, decided alike by every thread) goes to
// seed_hash_wide instead: a lane's walk is a chain of dependent loads, and with few reads nothing hides its latency.
__global__ void __launch_bounds__(kSeedThreads, MGB_SEED_MIN_BLOCKS) k_seed_hash(const __grid_constant__ SeedArgs a) {
    const IndexView &ix = a.ix;
    const int K = (int)ix.k;
    const int top = 2 * (K - 1);                                      // shift of the newest character in the key
    const unsigned long long mask = (1ull << (2 * K)) - 1;
    const uint32_t sigma = ix.sigma;
    const bool two = a.n_strands == 2;
    const uint32_t lanes = gridDim.x * blockDim.x;
    const uint32_t n_items = a.list ? *a.n_list : a.n_reads;
    if (a.seed_mode == 2 || (a.seed_mode == 0 && n_items <= kSeedWideRounds * (lanes / kWarp))) {
        seed_hash_wide(a, n_items);
        return;
    }
    for (uint32_t it = blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += lanes) {
        const uint32_t r = a.list ? __ldg(a.list + it) : it;
        const uint64_t b = a.offsets[r];
        const int L = (int)(a.offsets[r + 1] - b);
        const int nk = L >= K ? L - K + 1 : 0;
        if (nk == 0) { if (a.summary) a.summary[r] = 0; continue; }
        const uint64_t ko = a.koff[r];
        // ---- position 0 of both strands, the two lookups in flight together
        uint64_t f0, f1;
        {
            CodeStream c0, c1;
            int bad0, bad1 = 0;
            const unsigned long long k0 = first_kmer(c0, a.cf + b, L, K, sigma, &bad0);
            const unsigned long long k1 = two ? first_kmer(c1, a.cr + b, L, K, sigma, &bad1) : 0ull;
            KhProbe p0, p1;
            p0.issue(ix, k0, bad0 < 0); p1.issue(ix, k1, two && bad1 < 0);
            p0.find(ix); p1.find(ix);
            f0 = p0.value(ix); f1 = p1.value(ix);
        }
        const bool paired = two && ((f0 != 0) != (f1 != 0));
        const int passes = two && !paired ? 2 : 1;
        uint32_t seen = 0;                    // SeedArgs::summary of the read: bit 0 / 1 (forward), 2 / 3 (reverse)
        for (int pass = 0; pass < passes; ++pass) {
            // the strand walked in order (the primary when paired) ...
            const bool sp = paired ? f0 == 0 : pass == 1;
            const int sh = sp ? 2 : 0;        // its bits in `seen`; the secondary's are at 2 - sh
            CodeStream cs;
            int last_bad;
            unsigned long long key = first_kmer(cs, (sp ? a.cr : a.cf) + b, L, K, sigma, &last_bad);
            uint64_t edge = sp ? f1 : f0;                              // its k-mer at 0, from the probe
            uint64_t *out = (sp ? a.nodes_r : a.nodes_f) + ko;
            SectorOut so;
            so.clear();
            const bool store0 = edge != 0 && in_graph(ix, edge);
            so.put_up(out, 0, nk, store0 ? edge : 0);
            seen |= (store0 ? 2u : 1u) << sh;
            PathWalk pw;
            pw.start(ix, edge, store0 && nk > 1);
            // ... and the secondary, backwards: characters L - 1 .. nk of its k-mer at nk - 1 first
            CodeStreamDown ds;
            ds.start((sp ? a.cf : a.cr) + b, paired ? L : 0);
            uint64_t *out2 = (sp ? a.nodes_f : a.nodes_r) + ko;
            unsigned long long key2 = 0;
            int bad2 = 0x7fffffff;                                     // lowest position of an invalid character read
            for (int i = 0; paired && i < K - 1; ++i) {
                const uint32_t c = ds.next();
                if (c < 1 || c >= sigma) bad2 = L - 1 - i;
                key2 = (key2 << 2) | ((c - 1) & 3u);
            }
            SectorOut so2;
            so2.clear();
            bool look2 = true;                 // the secondary's next k-mer needs a lookup (the probe was a cold hit)
            for (int t = 1; t < nk; ++t) {
                // ---- issue: the primary's record or bucket for k-mer t, the secondary's bucket for k-mer nk - t
                const uint32_t c = cs.next();
                if (c < 1 || c >= sigma) last_bad = t + K - 1;
                key = (key >> 2) | ((unsigned long long)((c - 1) & 3u) << top);
                const bool ok = last_bad < t;                          // a k-mer without an invalid character
                // on the path: the k-mer t - 1 is the one at q - 1, so k-mer t is the one at q if its last character is
                // q's and q is on the same path. Leaving it, the walk goes on from the last node on it.
                const bool path = ok && pw.next_is(ix, c);
                if (pw.on && !path) { if (ok) edge = __ldg(ix.pl_node + pw.q - 1); pw.on = false; }
                const bool warm = ok && edge != 0 && !path, cold = ok && edge == 0;
                const int j = nk - t;
                const uint32_t c2 = ds.next();
                if (c2 < 1 || c2 >= sigma) bad2 = j;
                key2 = ((key2 << 2) | ((c2 - 1) & 3u)) & mask;
                const bool cold2 = paired && look2 && bad2 >= j + K;
                if (path && !cold2) {                                  // no lookup on either strand: the short way
                    look2 = pw.rc();
                    pw.step(ix);
                    seen |= 2u << sh;
                    if (paired) { so2.put_down(out2, j, nk, 0); seen |= 1u << (2 - sh); }
                    continue;
                }
                uint2 ar = make_uint2(0u, 0u);
                if (warm) ar = load_adj(ix, edge);
                KhProbe p, p2;
                p.issue(ix, key, cold); p2.issue(ix, key2, cold2);
                p.find(ix); p2.find(ix);
                const uint64_t found = p.value(ix), found2 = p2.value(ix);
                // ---- consume: the k-mers' edges, stored if they are nodes of the graph
                const uint64_t child = adj_child(ar, c);              // 0 unless warm (ar = 0)
                const bool child_ok = (ar.y >> (8 + c)) & 1u;
                look2 = path ? pw.rc() : !(warm && child != 0 && !((ar.y >> (16 + c)) & 1u));
                if (path) {
                    pw.step(ix);                                       // stored by the copy below
                    seen |= 2u << sh;
                } else {
                    edge = warm ? child : found;                       // 0 when the window is invalid
                    const bool store = warm ? (child != 0 && child_ok) : (found != 0 && in_graph(ix, found));
                    so.put_up(out, t, nk, store ? edge : 0);            // (store: edge != 0)
                    seen |= (store ? 2u : 1u) << sh;
                }
                if (paired) {
                    const bool store2 = found2 != 0 && in_graph(ix, found2);
                    so2.put_down(out2, j, nk, store2 ? found2 : 0);
                    seen |= (store2 ? 2u : 1u) << (2 - sh);
                }
            }
            if (paired) {
                so2.put_down(out2, 0, nk, 0);                          // the probe's miss
                seen |= 1u << (2 - sh);
            }
            // ---- the path run: k-mers 0 .. t of a lane that took t steps on the path are pl_node[p .. q) (p: the
            // position of the probe's node, loaded again), copied by the lanes here together, 32 node ids per
            // instruction. The copy comes after the lane's own stores: SectorOut may have written stale slots of the
            // run's sectors.
            const uint32_t from = pw.q != kPlNone + 1 ? __ldg(ix.pl_pos + (sp ? f1 : f0)) : pw.q;
            const unsigned grp = __activemask();
            const int width = __popc(grp), rank = __popc(grp & ((1u << (threadIdx.x & 31)) - 1u));
            __syncwarp(grp);
            for (unsigned todo = __ballot_sync(grp, pw.q - from > 1); todo; todo &= todo - 1) {
                const int src = __ffs(todo) - 1;
                uint64_t *dst = reinterpret_cast<uint64_t*>(__shfl_sync(grp, (unsigned long long)out, src));
                const uint32_t f = __shfl_sync(grp, from, src), len = __shfl_sync(grp, pw.q - from, src);
                for (uint32_t i = rank; i < len; i += width) dst[i] = __ldg(ix.pl_node + f + i);
            }
        }
        if (a.summary) a.summary[r] = (uint8_t)seen;
    }
}
#endif // !MGB_WIDE_ONLY

#endif // MGB_ALIGN_KERNEL_ONLY

#ifndef MGB_ALIGN_MIN_BLOCKS
#define MGB_ALIGN_MIN_BLOCKS 4
#endif
#ifndef MGB_ALIGN_THREADS
#define MGB_ALIGN_THREADS 128
#endif
static constexpr int kAlignThreads = MGB_ALIGN_THREADS;
static constexpr int kWarpsPerBlock = kAlignThreads / kWarp;   // reads in flight per block of k_align
// one warp per read; a warp that finds the list done before its first read touches nothing (the host may launch more
// warps than a list whose length only the device knows needs)
__device__ __forceinline__ unsigned int align_take(const AlignArgs &a, int which = 0) {
    unsigned int t = 0;
    if (wlane() == 0) t = atomicAdd(a.next + which, 1u);
    return wbcast(t, 0);
}
__global__ void __launch_bounds__(kAlignThreads, MGB_ALIGN_MIN_BLOCKS) k_align(const __grid_constant__ AlignArgs a) {
    const uint32_t n_list = a.n_list_dev ? __ldg(a.n_list_dev) : a.n_list;
    // the warp's arena, numbered in the order the warps start rather than by warp id: a pass allocates one arena per
    // read at most, and fewer when device memory holds fewer; a warp left without one aligns nothing
    const unsigned int slot = align_take(a, 3);
    if (slot >= a.n_arenas) return;
    unsigned int t = align_take(a);
    if (t >= n_list) return;
    char *arena = a.arena + (size_t)slot * a.arena_stride;
    extern __shared__ __align__(16) char smem_raw[];
    char *smem = smem_raw + (threadIdx.x / kWarp) * a.slay.total;
    init_arena(a, arena);
    // the warp's arena and on-chip working set: base + offsets from the kernel parameters
    const WarpMem mem { arena, &a.lay };
    const WarpSmem sm { smem, &a.slay };
    for (; t < n_list; t = align_take(a)) align_read(a, a.read_list[t], mem, sm);
}

// Grid of a read-path kernel (k_prepare, k_prepare_exact, k_premap, k_seed, k_seed_hash, k_subk, k_exact_reads, k_align):
// `blocks`, or fewer under MGB_TEST_MAX_BLOCKS=n (test knob: at most n blocks, so that the kernels' persistent and
// grid-stride loops run several rounds on small inputs). Read on every launch; host code only.
static inline uint64_t read_path_grid(uint64_t blocks) {
    if (const char *e = std::getenv("MGB_TEST_MAX_BLOCKS")) {
        const long long n = std::atoll(e);
        if (n > 0 && (uint64_t)n < blocks) blocks = (uint64_t)n;
    }
    return blocks;
}
// MGB_DEBUG=1: one line per read-path launch on stderr: the grid, the threads per block, the items (reads, strands,
// 32-position blocks of a strand) one round of the kernel's loop covers and, when the host knows it, the number of items
// (items=dev: a length the device holds)
static inline void log_launch(const char *kernel, uint64_t grid, int threads, uint64_t per_round, long long items) {
    if (!std::getenv("MGB_DEBUG")) return;
    char n[24];
    if (items >= 0) std::snprintf(n, sizeof(n), "%lld", items); else std::snprintf(n, sizeof(n), "dev");
    std::fprintf(stderr, "[mgb] launch %s grid=%llu block=%d per_round=%llu items=%s\n", kernel,
                 (unsigned long long)grid, threads, (unsigned long long)per_round, n);
}

// launchers (the only entry points the host code uses)
#if !defined(MGB_ALIGN_KERNEL_ONLY)
cudaError_t launch_radj_bwd(unsigned grid, const RadjArgs &a) { k_radj_bwd<<<grid, 128>>>(a); return cudaGetLastError(); }
cudaError_t launch_sfx_extend(unsigned grid, const SfxArgs &a) { k_sfx_extend<<<grid, 128>>>(a); return cudaGetLastError(); }
cudaError_t launch_subk(unsigned grid, cudaStream_t s, const SubkArgs &a, uint32_t chunks_per_strand) {
    grid = (unsigned)read_path_grid(grid);
    log_launch("k_subk", grid, 128, (uint64_t)grid * 4,          // one warp per 32 positions of a strand
               (long long)a.n_reads * a.n_strands * ((chunks_per_strand * (uint32_t)kSubkChunk + 31) / 32));
    k_subk<<<grid, 128, 0, s>>>(a, chunks_per_strand);
    return cudaGetLastError();
}
cudaError_t launch_premap(unsigned grid, cudaStream_t s, const SeedArgs &a) {
    grid = (unsigned)read_path_grid(grid);
    log_launch("k_premap", grid, 256, (uint64_t)grid * 8, (long long)a.n_reads * a.n_strands);     // a warp per strand
    k_premap<<<grid, 256, 0, s>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_seed(unsigned grid, cudaStream_t s, const SeedArgs &a) {
    grid = (unsigned)read_path_grid(grid);
    log_launch("k_seed", grid, 128, (uint64_t)grid * 128, (long long)a.n_reads * a.n_strands);     // a lane per strand
    k_seed<<<grid, 128, 0, s>>>(a);
    return cudaGetLastError();
}
#if !defined(MGB_WIDE_ONLY)
// persistent grid: as many blocks as are resident at once, or fewer when the reads do not fill them
cudaError_t launch_seed_hash(int num_sms, cudaStream_t s, const SeedArgs &a) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_seed_hash, kSeedThreads, 0);
    if (e != cudaSuccess) return e;
    const uint64_t need = ((uint64_t)a.n_reads + kSeedThreads - 1) / kSeedThreads;     // one read per lane
    const uint64_t resident = (uint64_t)per_sm * num_sms;
    const unsigned grid = (unsigned)read_path_grid(need < resident ? need : resident);
    log_launch("k_seed_hash", grid, kSeedThreads, (uint64_t)grid * kSeedThreads, a.list ? -1 : (long long)a.n_reads);
    k_seed_hash<<<grid, kSeedThreads, 0, s>>>(a);
    return cudaGetLastError();
}
#endif
#endif
cudaError_t launch_align(unsigned grid, size_t smem_block, cudaStream_t s, const AlignArgs &a) {
    k_align<<<grid, kAlignThreads, smem_block, s>>>(a);
    return cudaGetLastError();
}
// raises the kernel's dynamic shared memory limit to `smem_limit` and reports the resident blocks per SM
// for blocks of `smem_block` bytes
cudaError_t align_occupancy(size_t smem_limit, size_t smem_block, int *blocks_per_sm) {
    cudaError_t e = cudaFuncSetAttribute(k_align, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k_align, kAlignThreads, smem_block);
}

#if !defined(MGB_WIDE_ONLY) && !defined(MGB_ALIGN_KERNEL_ONLY)
// PRIMARY graphs are DNA graphs in the block layout: first translation unit only
__global__ void __launch_bounds__(128) k_rc_tables(RcArgs a) {
    uint64_t quad = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    uint64_t nquads = ((uint64_t)gridDim.x * blockDim.x) >> 2;
    for (uint64_t e = 1 + quad; e <= a.n; e += nquads) rc_tables_item(a, e);
}
// alphabet-independent kernels live in the first translation unit only
__global__ void __launch_bounds__(256) k_prepare(PrepArgs a) {
    uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp;
    uint32_t nwarps = (gridDim.x * blockDim.x) / kWarp;
    for (uint32_t r = warp; r < a.n_reads; r += nwarps) prepare_read(a, r);
}

// Whole-read exact answers for the reads of a.list, a tile of kExactThreads reads per block and round. Each thread
// decides for one read (exact_read_strand: its loads are independent of the other reads', so a warp has 32 reads' loads
// in flight); a block prefix sum of the record sizes gives the answered reads one heap allocation per tile, and the
// others one append to a.rest. Then each warp writes its answered records one after the other, 32 lanes per record.
// Persistent grid. No index structure is read.
static constexpr int kExactThreads = 256;
// the length of a.list (loaded again each round: holding it across the loop made ptxas spill)
__device__ __forceinline__ uint32_t exact_list_len(const ExactArgs &a) { return a.n_list_dev ? __ldg(a.n_list_dev) : a.n_list; }
__global__ void __launch_bounds__(kExactThreads) k_exact_reads(const __grid_constant__ ExactArgs a) {
    constexpr int kWarps = kExactThreads / 32;
    __shared__ int8_t diag[128];
    __shared__ unsigned long long s_off[kWarps];        // per warp: heap offset of its first record
    __shared__ uint32_t s_bytes[kWarps], s_left[kWarps], s_slot[kWarps];
    for (int i = threadIdx.x; i < 128; i += kExactThreads) diag[i] = a.diag[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned below = (1u << lane) - 1u;
    for (uint64_t base = (uint64_t)blockIdx.x * kExactThreads; base < exact_list_len(a); base += (uint64_t)gridDim.x * kExactThreads) {
        const uint32_t n_list = exact_list_len(a);
        const uint64_t t = base + threadIdx.x;
        uint32_t r = 0; uint64_t b = 0; int L = 0, s = -1; score_t score = 0;
        if (t < n_list) {
            r = a.list[t];
            s = exact_read_strand(a, diag, r, &b, &L, &score);
        }
        const uint32_t bytes = s >= 0 ? exact_read_bytes(a, L) : 0u;
        uint32_t inc = bytes;                                          // inclusive prefix sum over the warp
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
        const unsigned left = __ballot_sync(0xffffffffu, t < n_list && s < 0);
        if (lane == 31) s_bytes[w] = inc;
        if (lane == 0) s_left[w] = (uint32_t)__popc(left);
        __syncthreads();
        if (w == 0) {                                                  // the same over the warps, one atomic each
            const uint32_t v = lane < kWarps ? s_bytes[lane] : 0u, c = lane < kWarps ? s_left[lane] : 0u;
            uint32_t vi = v, ci = c;
            #pragma unroll
            for (int d = 1; d < kWarps; d <<= 1) {
                const uint32_t ov = __shfl_up_sync(0xffffffffu, vi, d), oc = __shfl_up_sync(0xffffffffu, ci, d);
                if (lane >= d) { vi += ov; ci += oc; }
            }
            const uint32_t tv = __shfl_sync(0xffffffffu, vi, kWarps - 1), tc = __shfl_sync(0xffffffffu, ci, kWarps - 1);
            unsigned long long off = 0; unsigned int slot = 0;
            if (lane == 0) {
                if (tv) off = atomicAdd(a.heap_used, (unsigned long long)tv);
                if (tc) slot = atomicAdd(a.n_rest, tc);
            }
            off = __shfl_sync(0xffffffffu, off, 0); slot = __shfl_sync(0xffffffffu, slot, 0);
            if (lane < kWarps) { s_off[lane] = off + (vi - v); s_slot[lane] = slot + (ci - c); }
        }
        __syncthreads();
        if ((left >> lane) & 1u) a.rest[s_slot[w] + __popc(left & below)] = r;
        const unsigned long long my_off = s_off[w] + (inc - bytes);
        for (unsigned todo = __ballot_sync(0xffffffffu, s >= 0); todo; todo &= todo - 1) {
            const int j = __ffs(todo) - 1;
            exact_read_write(a, __shfl_sync(0xffffffffu, r, j), __shfl_sync(0xffffffffu, (unsigned long long)b, j),
                             __shfl_sync(0xffffffffu, L, j), __shfl_sync(0xffffffffu, s, j),
                             __shfl_sync(0xffffffffu, score, j), __shfl_sync(0xffffffffu, my_off, j), lane, 32);
        }
    }
}
cudaError_t launch_exact_reads(int num_sms, cudaStream_t s, const ExactArgs &a) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_exact_reads, kExactThreads, 0);
    if (e != cudaSuccess) return e;
    const uint64_t need = ((uint64_t)a.n_list + kExactThreads - 1) / kExactThreads;
    const uint64_t resident = (uint64_t)per_sm * num_sms;
    const unsigned grid = (unsigned)read_path_grid(need < resident ? need : resident);
    log_launch("k_exact_reads", grid, kExactThreads, (uint64_t)grid * kExactThreads,
               a.n_list_dev ? -1 : (long long)a.n_list);
    k_exact_reads<<<grid, kExactThreads, 0, s>>>(a);
    return cudaGetLastError();
}

// Exclusive prefix sum of v over the threads of the block, with one atomicAdd of the block's total to *ctr: the thread's
// share of what the atomic handed out. s_sum / s_base: kWarps words of shared memory each.
template <int kWarps, class C>
__device__ __forceinline__ C tile_alloc(uint32_t v, C *ctr, uint32_t *s_sum, C *s_base) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
    if (lane == 31) s_sum[w] = inc;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < kWarps ? s_sum[lane] : 0u;
        uint32_t xi = x;
        #pragma unroll
        for (int d = 1; d < kWarps; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, xi, d); if (lane >= d) xi += o; }
        const uint32_t total = __shfl_sync(0xffffffffu, xi, kWarps - 1);
        C base = 0;
        if (lane == 0 && total) base = atomicAdd(ctr, (C)total);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (lane < kWarps) s_base[lane] = base + (xi - x);
    }
    __syncthreads();
    return s_base[w] + (inc - v);
}

// Whole-read exact answers from the raw reads (exact_path_strand), in place of k_prepare, a tile of kPrepExactThreads
// reads per block and round, one read per thread. The block first copies the tile's characters to shared memory with
// coalesced 16-byte loads (a tile longer than a.stage_bytes is read from global memory through the same code). The
// answered reads of a tile take one heap allocation (a record that does not fit makes its read a left-over one), the
// left-over reads one append to a.list. A warp whose reads are all answered with records of one size writes its headers
// and records as runs of words across its lanes (no loads but node ids; DESIGN.md §3.3); other warps write a header per
// thread and the records one after the other, 32 lanes each. Each warp then prepares its left-over reads (prepare_read),
// one after the other. Persistent grid.
static constexpr int kPrepExactThreads = 256;
#if defined(MGB_PROBE_NO_WRITES)
// probe build (scripts/build_variant.sh), wrong results by design: no header or record stores (the host zeroes the
// headers, so every answered read comes back with no alignment)
static constexpr bool kPrepWrites = false;
#else
static constexpr bool kPrepWrites = true;
#endif
static_assert(kPrepExactThreads == 256, "prep_stage_bytes sizes tiles of 256 reads");
// MGB_PREP_TIMERS builds: a warp's sums of the phase cycles added to a.phase_out
__device__ __forceinline__ void prep_timer_flush(const PrepExactArgs &a, const PrepTimer &tm) {
#if defined(MGB_PREP_TIMERS)
    for (int ph = 0; ph < PREP_N_PHASES; ++ph) {
        unsigned long long v = (unsigned long long)tm.c[ph];
        for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        if ((threadIdx.x & 31) == 0 && a.phase_out) atomicAdd(a.phase_out + ph, v);
    }
#else
    (void)a; (void)tm;
#endif
}
// 5 blocks per SM (<= 51 registers): more reads in flight; with fewer, the kernel is latency-bound (DESIGN.md §3.3)
__global__ void __launch_bounds__(kPrepExactThreads, 5) k_prepare_exact(const __grid_constant__ PrepExactArgs a) {
    constexpr int kWarps = kPrepExactThreads / 32;
    extern __shared__ uint4 s_tile[];                   // a.stage_bytes: the tile's raw characters
    __shared__ unsigned long long s_off[kWarps];
    __shared__ uint32_t s_bytes[kWarps], s_left[kWarps], s_slot[kWarps];
    const int lane = threadIdx.x & 31;
    const uint32_t n_reads = a.prep.n_reads;
    PrepTimer tm;
    for (uint64_t base = (uint64_t)blockIdx.x * kPrepExactThreads; base < n_reads; base += (uint64_t)gridDim.x * kPrepExactThreads) {
        tm.start();
        // ---- the tile's bytes [offsets[base], offsets[end]) and the slack the word reads go past them, in 16-byte
        // words from the one holding the first byte; a tile that does not fit is read from global memory instead
        const uint64_t end = base + kPrepExactThreads < n_reads ? base + kPrepExactThreads : n_reads;
        const uint64_t lo16 = a.prep.offsets[base] & ~15ull;
        const uint64_t n16 = (((a.prep.offsets[end] + kPrepStageSlack + 15) & ~15ull) - lo16) >> 4;
        const uint4 *src = reinterpret_cast<const uint4*>(a.prep.seqs + lo16);
        const bool staged = n16 * 16 <= a.stage_bytes;
        if (staged) {
            #pragma unroll 4
            for (uint32_t i = threadIdx.x; i < n16; i += kPrepExactThreads) s_tile[i] = __ldg(src + i);
        }
        __syncthreads();
        const uint8_t *tile = reinterpret_cast<const uint8_t*>(staged ? s_tile : src);
        tm.lap(PREP_STAGE);
        const uint32_t r = (uint32_t)(base + threadIdx.x);
        const uint8_t *raw = nullptr;
        int L = 0, s = -1; uint32_t p = 0; score_t score = 0;
        if (r < n_reads) {
            const uint64_t b = a.prep.offsets[r];
            L = (int)(a.prep.offsets[r + 1] - b);
            raw = tile + (b - lo16);
            s = exact_path_strand(a, raw, L, &p, &score, tm);
        }
        tm.lap(PREP_TEXT);
        const uint32_t bytes = s >= 0 ? exact_read_bytes(a.ex, L) : 0u;
        const unsigned long long off = tile_alloc<kWarps>(bytes, a.ex.heap_used, s_bytes, s_off);
        if (s >= 0 && off + bytes > a.ex.heap_cap) s = -1;
        const bool left = r < n_reads && s < 0;
        const uint32_t slot = tile_alloc<kWarps>(left ? 1u : 0u, a.n_list, s_left, s_slot);
        if (left) a.list[slot] = r;
        tm.lap(PREP_ALLOC);
        // ---- the answered reads' headers and records. The allocation goes in thread order, so a warp's answered
        // records are one run of the heap. A warp whose 32 reads are all answered with records of one size (without
        // node ids: lengths that round up to one multiple of 8) writes its headers as one run of 16-byte chunks, each
        // lane its own record's OutAln, and the rest of its records as one run of 8-byte words from lane 0's offset,
        // lane i words i, i + 32, ...; other warps write a header per thread and the records one after the other.
        const unsigned ans = __ballot_sync(0xffffffffu, s >= 0);
        const uint32_t R = __shfl_sync(0xffffffffu, bytes, 0);
        unsigned long long *hw = reinterpret_cast<unsigned long long*>(a.ex.hdr + (r - lane));
        if (kPrepWrites && __all_sync(0xffffffffu, s >= 0 && bytes == R) && ((uintptr_t)hw & 15) == 0) {
            // the header array and so the warp's 1280 bytes of headers start on a 16-byte boundary
            #pragma unroll
            for (int c = lane; c < 96; c += 32) {                    // 80 chunks; every lane takes part in the shuffles
                const int q = c < 80 ? 2 * c : 0, i0 = q / 5, i1 = (q + 1) / 5;
                ulonglong2 v;
                v.x = exact_path_hdr_word(a.ex, __shfl_sync(0xffffffffu, L, i0), __shfl_sync(0xffffffffu, off, i0), q % 5);
                v.y = exact_path_hdr_word(a.ex, __shfl_sync(0xffffffffu, L, i1), __shfl_sync(0xffffffffu, off, i1),
                                          (q + 1) % 5);
                if (c < 80) reinterpret_cast<ulonglong2*>(hw)[c] = v;
            }
            // each lane its own record's OutAln (words 0-3); then word g of the records' words 4 .. nw - 1 is word
            // 4 + g % nb of lane g / nb's record, every lane taking nb of them (past word 0 the score is not used)
            unsigned long long *o = reinterpret_cast<unsigned long long*>(a.ex.heap + off);
            const ulonglong2 h0 = make_ulonglong2(exact_path_word(a, raw, L, s, p, score, 0), exact_path_word(a, raw, L, s, p, score, 1));
            const ulonglong2 h1 = make_ulonglong2(exact_path_word(a, raw, L, s, p, score, 2), exact_path_word(a, raw, L, s, p, score, 3));
            if (((uintptr_t)o & 15) == 0) {
                reinterpret_cast<ulonglong2*>(o)[0] = h0; reinterpret_cast<ulonglong2*>(o)[1] = h1;
            } else {
                o[0] = h0.x; o[1] = h0.y; o[2] = h1.x; o[3] = h1.y;
            }
            o = reinterpret_cast<unsigned long long*>(a.ex.heap + __shfl_sync(0xffffffffu, off, 0)) + 4;
            // each word's record: its read's place in the tile, and its length and strand, from the record's lane. They
            // go in one shuffle when both fit in 16 bits: a staged tile is smaller than 64 KB, and every L is below R
            // (warp-uniform, so is the choice)
            const uint32_t ro = (uint32_t)(raw - tile), ls = (uint32_t)L << 1 | (uint32_t)s, nw = R >> 3, nb = nw - 4;
            const bool packed = staged && R < (1u << 15);
            uint32_t j = (uint32_t)lane / nb, wi = (uint32_t)lane - j * nb;
            for (uint32_t g = (uint32_t)lane; g < 32 * nb; g += 32) {
                uint32_t rj, lj;
                if (packed) {
                    const uint32_t x = __shfl_sync(0xffffffffu, ro << 16 | ls, j);
                    rj = x >> 16; lj = x & 0xFFFFu;
                } else {
                    rj = __shfl_sync(0xffffffffu, ro, j); lj = __shfl_sync(0xffffffffu, ls, j);
                }
                const uint32_t pj = a.ex.result_nodes ? 0u : __shfl_sync(0xffffffffu, p, j);
                o[j * nw + wi] = exact_path_word(a, tile + rj, (int)(lj >> 1), (int)(lj & 1u), pj, 0, 4 + wi);
                for (wi += 32; wi >= nb; wi -= nb) ++j;
            }
        } else if (kPrepWrites && ans) {
            if (s >= 0) exact_path_hdr(a.ex, r, L, off);
            for (unsigned todo = ans; todo; todo &= todo - 1) {
                const int j = __ffs(todo) - 1;
                exact_path_write(a, reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, (unsigned long long)raw, j)),
                                 __shfl_sync(0xffffffffu, L, j), __shfl_sync(0xffffffffu, s, j), __shfl_sync(0xffffffffu, p, j),
                                 __shfl_sync(0xffffffffu, score, j), __shfl_sync(0xffffffffu, off, j), lane, 32);
            }
        }
        tm.lap(PREP_WRITE);
        for (unsigned todo = __ballot_sync(0xffffffffu, left); todo; todo &= todo - 1)
            prepare_read(a.prep, __shfl_sync(0xffffffffu, r, __ffs(todo) - 1));
        __syncthreads();                                 // the tile's characters are read up to here
        tm.lap(PREP_LEFT);
    }
    prep_timer_flush(a, tm);
}
cudaError_t launch_prepare_exact(int num_sms, cudaStream_t s, const PrepExactArgs &a) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_prepare_exact, kPrepExactThreads, a.stage_bytes);
    if (e != cudaSuccess) return e;
    const uint64_t need = ((uint64_t)a.prep.n_reads + kPrepExactThreads - 1) / kPrepExactThreads;
    const uint64_t resident = (uint64_t)per_sm * num_sms;
    const unsigned grid = (unsigned)read_path_grid(need < resident ? need : resident);
    log_launch("k_prepare_exact", grid, kPrepExactThreads, (uint64_t)grid * kPrepExactThreads, a.prep.n_reads);
    k_prepare_exact<<<grid, kPrepExactThreads, a.stage_bytes, s>>>(a);
    return cudaGetLastError();
}
// round r (0-based) brings character k - 3 - r of every edge's k-mer to c_nxt[e]; kmer_shift = 2 * (k - 3 - r)
__global__ void __launch_bounds__(256) k_radj_gather(RadjArgs a, int kmer_shift) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = 1 + t; e <= a.n; e += nt) {
        const uint8_t c = a.c_cur[a.bwd_arr[e]];
        a.c_nxt[e] = c;
        if (a.kmer) {
            const unsigned long long km = a.kmer[e];
            if (km != kKmerBad) a.kmer[e] = c == 0 ? kKmerBad : (km | ((unsigned long long)(c - 1) << kmer_shift));
        }
    }
}
// k-mer hash index: one slot per k-mer without '$' (every such edge spells a distinct k-mer)
__global__ void __launch_bounds__(256) k_kmer_insert(const unsigned long long *kmer, uint64_t n, unsigned long long *keys,
                                                     uint32_t *vals, uint64_t slots) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = 1 + t; e <= n; e += nt) {
        const unsigned long long km = kmer[e];
        if (km == kKmerBad) continue;
        const unsigned long long key = km | (1ull << 63);
        uint64_t i = kh_slot_of(key, slots);
        while (atomicCAS(keys + i, 0ull, key) != 0ull) { if (++i == slots) i = 0; }
        vals[i] = (uint32_t)e;
    }
}
// Reverse-complement bits of the forward adjacency records (index.cuh load_adj, y[16:21)), once the hash index is
// complete: for every label c != '$' out of e's target node, is the reverse complement of that child's k-mer in the
// index? A k-mer that is no valid key gets the bit too, so k_seed_hash then looks it up rather than skip it. Each
// thread writes its own records only. `ix` carries the finished hash index.
__global__ void __launch_bounds__(256) k_adj_rc(IndexView ix, uint2 *adj, const unsigned long long *kmer) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = 1 + t; e <= ix.n; e += nt) {
        const uint2 a = adj[e];
        uint32_t bits = 0;
        for (uint32_t c = 1; c < 5; ++c) {
            const uint64_t child = adj_child(a, c);
            if (!child) continue;
            const unsigned long long km = kmer[child];
            if (km == kKmerBad || kh_lookup(ix, kh_revcomp(km, ix.k))) bits |= 1u << (16 + c);
        }
        if (bits) adj[e].y = a.y | bits;
    }
}
// Clears y[16:21) of every forward adjacency record: a replica that leaves out the hash index (mgb_index_replicate)
// holds the records mgb_index_create builds without it.
__global__ void __launch_bounds__(256) k_adj_clear_rc(uint2 *adj, uint64_t n) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = 1 + t; e <= n; e += nt) adj[e].y &= ~(0x1Fu << 16);
}

// Path layout (IndexView::pl_*), built once the hash index is complete. Its nodes are the DBG nodes the seeding walk
// stores (in_graph, a k-mer without '$'). A node whose target has exactly one such child links to it; a child that several
// nodes link to keeps the smallest of them, the others end their paths. Cycles (tandem repeats shorter than k, circular
// inputs) are cut at their smallest node. Positions come from pointer jumping over `jump`, one word per edge:
//   0                          not a DBG node
//   next | dist << 32          not done: `next` is dist steps ahead on the path
//   tail | dist << 32 | kJDone done: the path's last node is dist steps ahead (k_path_heads then puts the tail's
//                              position in place of its own id, dist 0)
// Cycle nodes never get done; k_path_cycle_* then hold (next | smallest node seen << 32) instead. Edge ids are < 2^31.
struct PathArgs {
    IndexView ix;                        // with the hash index
    const unsigned long long *kmer;      // per edge (RadjArgs::kmer)
    uint32_t *pred;                      // per edge: the node linking to it, kPlNone if none; k_path_place: pl_pos
    unsigned long long *jump;            // per edge, as above
    uint32_t *node; unsigned int *text, *rc, *stop;           // pl_node / pl_text / pl_rc cleared, pl_stop all
                                                              // ones (k_path_place)
    unsigned long long *total;           // positions handed out (k_path_heads)
    unsigned int *count;                 // nodes that got done in a round / cycle nodes
};
static constexpr unsigned long long kJDone = 1ull << 63;
MGB_D bool path_node(const PathArgs &a, uint64_t e) { return in_graph(a.ix, e) && a.kmer[e] != kKmerBad; }
// the child that DBG node e links to if it is the only one, else 0
MGB_D uint64_t path_child(const PathArgs &a, uint64_t e) {
    const uint2 ar = a.ix.adj[e];
    const uint32_t ok = (ar.y >> 8) & 31u;
    if (popc32(ok) != 1) return 0;
    const uint64_t c = adj_child(ar, (uint32_t)ffs32(ok) - 1);
    return c && a.kmer[c] != kKmerBad ? c : 0;
}
MGB_D void count_warp(unsigned int *count, bool p) {
    const unsigned m = __ballot_sync(0xffffffffu, p);
    if (m && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(count, (unsigned)__popc(m));
}
#define MGB_EDGE_LOOP(e, n) \
    for (uint64_t e = 1 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e <= (n); e += (uint64_t)gridDim.x * blockDim.x)
__global__ void __launch_bounds__(256) k_path_pred(PathArgs a) {
    MGB_EDGE_LOOP(e, a.ix.n) {
        if (!path_node(a, e)) continue;
        const uint64_t c = path_child(a, e);
        if (c) atomicMin(a.pred + c, (uint32_t)e);
    }
}
__global__ void __launch_bounds__(256) k_path_link(PathArgs a) {
    MGB_EDGE_LOOP(e, a.ix.n) {
        unsigned long long j = 0;
        if (path_node(a, e)) {
            const uint64_t c = path_child(a, e);
            j = c && a.pred[c] == (uint32_t)e ? (1ull << 32) | c : kJDone | e;
        }
        a.jump[e] = j;
    }
}
// One round of pointer jumping, in place: a word read from another node is a valid (next, dist) pair whether or not that
// node has jumped in this round yet. *count: the nodes that got done. (The block-uniform loop keeps the ballot whole.)
__global__ void __launch_bounds__(256) k_path_jump(PathArgs a) {
    const uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < a.ix.n; base += nt) {
        const uint64_t e = 1 + base + threadIdx.x;
        bool done = false;
        if (e <= a.ix.n) {
            const unsigned long long x = a.jump[e];
            if (x && !(x & kJDone)) {
                const unsigned long long y = a.jump[(uint32_t)x];
                const unsigned long long d = ((x >> 32) + (y >> 32)) & 0x7FFFFFFFull;   // (cycle nodes: wraps, unused)
                a.jump[e] = (y & (kJDone | 0xFFFFFFFFull)) | (d << 32);
                done = (y & kJDone) != 0;
            }
        }
        count_warp(a.count, done);
    }
}
// the nodes left undone are on cycles: each starts with itself as the smallest node seen; *count: how many
__global__ void __launch_bounds__(256) k_path_cycle_init(PathArgs a) {
    const uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < a.ix.n; base += nt) {
        const uint64_t e = 1 + base + threadIdx.x;
        bool cyc = false;
        if (e <= a.ix.n) {
            const unsigned long long x = a.jump[e];
            cyc = x && !(x & kJDone);
            if (cyc) a.jump[e] = (e << 32) | path_child(a, e);
        }
        count_warp(a.count, cyc);
    }
}
// one doubling round of the smallest node over the cycle ahead
__global__ void __launch_bounds__(256) k_path_cycle_min(PathArgs a) {
    MGB_EDGE_LOOP(e, a.ix.n) {
        const unsigned long long x = a.jump[e];
        if (!x || (x & kJDone)) continue;
        const unsigned long long y = a.jump[(uint32_t)x];
        const unsigned long long m = (x >> 32) < (y >> 32) ? (x >> 32) : (y >> 32);
        a.jump[e] = (m << 32) | (y & 0xFFFFFFFFull);
    }
}
// the cycle node whose child is the cycle's smallest node becomes a tail, the smallest node a head
__global__ void __launch_bounds__(256) k_path_cycle_cut(PathArgs a) {
    MGB_EDGE_LOOP(e, a.ix.n) {
        const unsigned long long x = a.jump[e];
        if (!x || (x & kJDone)) continue;
        const uint64_t c = path_child(a, e);
        if (c == (x >> 32)) { a.jump[e] = kJDone | e; a.pred[c] = kPlNone; }
        else a.jump[e] = (1ull << 32) | c;
    }
}
// every head takes the positions of its path and the k - 1 filler positions after it, and leaves the tail's position in
// the tail's word
__global__ void __launch_bounds__(256) k_path_heads(PathArgs a) {
    MGB_EDGE_LOOP(e, a.ix.n) {
        if (a.pred[e] != kPlNone) continue;
        const unsigned long long x = a.jump[e];
        if (!x) continue;
        const uint64_t d = (x >> 32) & 0x7FFFFFFFull;
        const unsigned long long base = atomicAdd(a.total, (unsigned long long)(d + a.ix.k));
        a.jump[(uint32_t)x] = kJDone | ((base + d) & 0xFFFFFFFFull);
    }
}
// pl_pos, pl_node, pl_text (every node its first character, a tail all k), pl_rc and pl_stop
__global__ void __launch_bounds__(256) k_path_place(PathArgs a) {
    const int K = (int)a.ix.k;
    MGB_EDGE_LOOP(e, a.ix.n) {
        const unsigned long long x = a.jump[e];
        if (!x) { a.pred[e] = kPlNone; continue; }
        const uint64_t d = (x >> 32) & 0x7FFFFFFFull;
        const uint64_t pos = d == 0 ? (uint32_t)x : (uint32_t)a.jump[(uint32_t)x] - d;
        a.pred[e] = (uint32_t)pos;
        a.node[pos] = (uint32_t)e;
        atomicAnd(a.stop + (pos >> 5), ~(1u << (pos & 31)));
        const unsigned long long km = a.kmer[e];
        for (int i = 0; i < (d == 0 ? K : 1); ++i) {
            const uint64_t q = pos + i;
            atomicOr(a.text + (q >> 4), (unsigned)((km >> (2 * i)) & 3u) << (2 * (q & 15)));
        }
        if (kh_lookup(a.ix, kh_revcomp(km, a.ix.k))) atomicOr(a.rc + (pos >> 5), 1u << (pos & 31));
    }
}
#undef MGB_EDGE_LOOP
// IndexView::kh_pos and pl_word from the finished hash index and path layout in `ix` (either output may be null: not
// built)
__global__ void __launch_bounds__(256) k_layout_words(IndexView ix, uint32_t *kh_pos, ulonglong2 *pl_word) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (uint64_t)gridDim.x * blockDim.x;
    if (kh_pos) {
        for (uint64_t i = t; i < ix.kh_slots; i += nt) {
            const uint64_t e = ix.kh_keys[i] ? ix.kh_vals[i] : 0u;
            kh_pos[i] = in_graph(ix, e) ? ix.pl_pos[e] : kPlNone;
        }
    }
    if (pl_word) {
        for (uint64_t w = t; w < ix.pl_n / 32; w += nt)
            pl_word[w] = make_ulonglong2(ix.pl_text[w], ix.pl_stop[w] | ix.pl_rc[w]);
    }
}
__global__ void __launch_bounds__(256) k_radj_pack(RadjArgs a, uint32_t multi_shift) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t nt = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = 1 + t; e <= a.n; e += nt)
        a.radj[e] = make_uint2(a.bwd_arr[e], (uint32_t)a.c_cur[e] | ((uint32_t)a.multi[e] << multi_shift));
}
#endif

} // namespace MGB_KERNEL_NS
#endif
