// Seed-and-extend for one read, executed by one warp.
//
// Restates, on device data structures, the reference's per-read pipeline
//   DBGAligner::align_batch / align_both_directions / align_core   (dbg_aligner.cpp:251-384, 531-758)
//   ExactSeeder / MEMSeeder(UniMEM) / SuffixSeeder                 (aligner_seeder_methods.cpp:37-424)
//   SeedFilteringExtender + DefaultColumnExtender                  (aligner_extender_methods.cpp:66-1034)
//   Alignment::{trim_offset, reverse_complement (RCDBG)}           (alignment.cpp:177-190, 540-561)
//   AlignmentAggregator (unlabeled queue)                          (aligner_aggregator.hpp:59-202)
// Execution model: scalar state is warp-uniform (every lane holds the same value and takes
// the same branch; scalar stores are issued by all lanes with identical values), DP columns
// and copies are strided over the 32 lanes, rank/select go through the quad primitives of
// index.cuh. All dynamic containers live in a per-warp arena in HBM (no malloc); running out
// of arena marks the read MGB_READ_OVERFLOW and the host re-runs it with a larger arena.
#pragma once
#include "index.cuh"
#include "seed_core.cuh"

// Graph mode seen by the aligner (DeBruijnGraph::Mode): the product library compiles k_align per mode
// (kernels.cuh); the host-emulation build decides at run time.
#if defined(MGB_CANONICAL_ONLY)
#define MGB_CANONICAL(cfg) true
#elif defined(MGB_BASIC_ONLY)
#define MGB_CANONICAL(cfg) false
#else
#define MGB_CANONICAL(cfg) ((cfg).canonical != 0)
#endif
// PRIMARY graph behind CanonicalDBG semantics (node ids above ix.n denote reverse complements): only ever true
// in the CANONICAL-mode compilation
#if defined(MGB_BASIC_ONLY)
#define MGB_PRIMARY(ix) false
#else
#define MGB_PRIMARY(ix) ((ix).mode == 2)
#endif

namespace mgb {

// ------------------------------------------------------------------------------------
// Configuration as consumed on the device (DBGAlignerConfig, aligner_config.hpp:18-94)
// ------------------------------------------------------------------------------------
struct DevConfig {
    uint32_t num_alternative_paths;
    uint32_t min_seed_length;      // after the DBGAligner ctor normalisation (dbg_aligner.cpp:37-48)
    uint32_t max_seed_length;      // saturated to 0xffffffff
    uint64_t max_num_seeds_per_locus;
    score_t min_cell_score, min_path_score, xdrop;
    double min_exact_match, max_nodes_per_seq_char, max_ram_per_alignment, rel_score_cutoff;
    int32_t gap_open, gap_ext, left_end_bonus, right_end_bonus;
    uint8_t forward_and_reverse_complement, allow_left_trim, no_backtrack;
    uint8_t seed_complexity_filter;   // sdust on seed windows (aligner_seeder_methods.cpp:21-29), DNA only
    int32_t ge_shift;              // log2(-gap_ext) if that is a power of two, else -1 (extend_ins_end's division)
    int8_t diag[128];              // score_matrix[c][c]
    int8_t prof[kMaxSigma + 1][128];   // score_matrix[decode(i)][q], row sigma = '\0'
    uint8_t opmatch[kMaxSigma + 1][128]; // kCharToOp[decode(i)][q] == MATCH (aligner_cigar.cpp:11-51)
    uint8_t code_of[256];              // KmerExtractorBOSS::encode (kmer_extractor.cpp:30-44); invalid = sigma
    char letters[kMaxSigma + 1];       // alphabet, "$ACGT" / "$ABCDEFGHIJKLMNOPQRSTUVWYZX"
    uint32_t sigma;
    uint32_t has_complement;           // DNA: reverse complement defined
    uint32_t canonical;                // graph in CANONICAL mode (holds both strands): dbg_aligner.cpp:224-226, 646-656
    uint32_t result_nodes;             // mgb_config_t::result_nodes (MGB_NODES_*)
    uint32_t exact_shortcut;           // the scores allow the exact-path shortcut (lower_config) and it is not switched off
};

// largest num_alternative_paths served: the aggregator keeps one entry per lane of the warp that aligns the read
static constexpr int kMaxAlt = 32;
static constexpr int kMaxOut = kMaxSigma;     // max outgoing edges handled per column

enum ReadStatus : uint32_t { MGB_READ_OK = 0, MGB_READ_OVERFLOW = 1 };

// Capacities of the per-warp arena (host chooses them from the batch's longest read).
struct Caps {
    uint32_t L_max;            // longest read
    uint32_t max_cols;         // DP table columns
    uint32_t max_cells;        // DP cells (each = S,E,F)
    uint32_t hash_size;        // conv-checker hash slots, power of two
    uint32_t max_conv_entries;
    uint32_t max_conv_cells;
    uint32_t max_seeds;        // per strand
    uint32_t aln_nodes, aln_seq, aln_cigar;   // per alignment slot
    uint32_t n_alt;            // num_alternative_paths: the arena holds 3 * n_alt + 2 alignment slots
};

// Cells of a column in the DP table arena (ColMeta::fmt):
//   FMT_FULL     S[size+5] | E[size+5] | F[size+5]                       (general path, any width)
//   FMT_COMPACT  S[capr] | 32 flag bytes | F[capr] reserved, not written  (register path, size + 5 <= 32;
//   FMT_COMPACT_F  ... F written                                           capr = size + 5 rounded up to 8)
// A compact column keeps, instead of E and F, the four comparisons the backtrack makes with them (one byte
// per cell, see CF_*); F is only written when a later column may have to read it (the column waits in the
// queue, or a general-path child is created from it).
enum : uint8_t { FMT_FULL = 0, FMT_COMPACT = 1, FMT_COMPACT_F = 2 };
enum : uint8_t { CF_INS = 1,      // S == E                          (extender.cpp:943, insertion start)
                 CF_INS_EXT = 2,  // E[j] == E[j-1] + gap_ext        (:947-957, insertion run)
                 CF_DEL = 4,      // S == F                          (:972, deletion start)
                 CF_DEL_EXT = 8 };// F[j] == F_parent[row] + score + gap_ext  (:976-997, deletion run)
struct ColMeta {              // DefaultColumnExtender::DPTColumn (extender.hpp:129-147)
    uint64_t node;
    uint32_t parent;
    uint32_t cells_off;       // index of the first cell in the cells arena
    int32_t size;             // S.size()
    int32_t trim;
    int32_t offset;
    int32_t max_pos;
    int32_t score;            // added score (always 0 on real edges)
    uint8_t c;                // upper-cased character
    uint8_t is_tip;
    uint8_t started;          // prev_starts membership
    uint8_t fmt;              // FMT_*
    uint32_t pad0, pad1;      // 48 bytes: three 16-byte stores
};

struct HeapItem { int32_t score, neg_off_diag; uint32_t idx; int32_t max_score; };
struct BtStart { int32_t score, neg_off_diag, neg_i, pos; };
// convergence-table slot with the entry stored inline (one 32-byte load per probe)
struct ConvSlot { uint64_t key; uint32_t epoch; int32_t start, size, seg_start, seg_cap; uint32_t seg_off; };
struct SeedRec { uint32_t clip, len, offset, n_nodes; uint64_t node0; uint32_t alive, pad; };

struct AlnHdr {
    int32_t q_len;        // query_view size
    int32_t n_nodes, seq_len, n_cigar;
    int32_t score;
    uint32_t offset;
    uint32_t orientation;
    uint32_t used;
};

struct AlnSlot { AlnHdr *h; uint64_t *nodes; char *seq; uint32_t *cigar; };

// An aggregator entry's key, kept on chip: the fields LocalAlignmentLess orders by (score, query length, orientation,
// clipping) and the header fields Alignment::operator== compares before the arrays.
struct AggKey { int32_t score, q_len; uint32_t orientation; int32_t clip; uint32_t offset; int32_t seq_len, n_cigar, n_nodes; };

// Per-strand state. Lives in shared memory so that it can be indexed with a run-time strand
// number without forcing the aligner object out of registers.
struct StrandCtx {
    const char *q;               // upper-cased query strand (on-chip copy if staged)
    int32_t *ps;                 // suffix sums of self-match scores (extender.cpp:26-36)
    const uint8_t *codes;        // alphabet codes of q
    const uint64_t *qnodes;      // map_to_nodes_sequentially (nullptr if L < k)
    SeedRec *seeds;
    ConvSlot *conv_slots; score_t *conv_cells;      // convergence table of the extender built on this strand
    uint32_t conv_epoch, conv_n, conv_cells_used;
    int32_t n_seeds; uint32_t num_matching;
    uint32_t table_cap;          // std::vector<DPTColumn>::capacity() emulation
    uint32_t num_ext, explored_prev;
    uint32_t rc;                 // set_graph(): 1 = RCDBG view
    uint32_t implicit_seeds;     // 1: seeds are the set bits of `mask` (one k-mer seed per matched k-mer)
    uint32_t *mask;              // alive bits of implicit seeds (shared memory)
    // BOSS::index_range per query position from k_subk (nullptr: computed here); sub_len 0xFF = not computed
    const uint32_t *sub_first, *sub_last; const uint8_t *sub_len;
};

// Per-read output record header; followed in the output heap by packed alignments.
struct OutAln {
    uint32_t orientation; int32_t score; uint32_t offset; uint32_t query_begin, query_len;
    uint32_t n_nodes, seq_len, n_cigar;
};

// One alignment of a read's packed records (OutAln | node ids unless result_nodes | CIGAR | sequence, each part padded
// to 8, as k_align and the whole-read writers pack them): the reader every consumer of the heaps goes through
struct RecView {
    OutAln o; const uint64_t *nodes; const uint32_t *cigar; const char *seq;
};
MGB_HOSTDEV const char *rec_next(const char *p, bool no_nodes, RecView *v) {
    v->o = *reinterpret_cast<const OutAln*>(p);
    p += sizeof(OutAln);
    v->nodes = no_nodes ? nullptr : reinterpret_cast<const uint64_t*>(p);
    if (!no_nodes) p += 8ull * v->o.n_nodes;
    v->cigar = reinterpret_cast<const uint32_t*>(p); p += (4ull * v->o.n_cigar + 7) & ~7ull;
    v->seq = p; p += ((uint64_t)v->o.seq_len + 7) & ~7ull;
    return p;
}

struct ReadStats { uint32_t num_seeds, num_extensions, num_explored_nodes, dp_columns; uint64_t dp_cells; };
#if defined(MGB_HOST_EMU)
extern "C" unsigned long long mgb_emu_whole_read_hits;   // host emulation (tests) only: reads answered by exact_read_strand()
extern "C" unsigned long long mgb_emu_path_read_hits;    // ... and by exact_path_strand()
// host emulation (tests) only: how often the aligner leaves its on-chip working set, so that a test can show which of
// these paths its inputs reach. The order is part of the test interface (tests/parity_common.py EMU_PATHS).
enum EmuPath : int {
    EMU_QUEUE_MIGRATE,        // heap_push: the best-first queue moves to the arena
    EMU_NN_MIGRATE,           // nn_push: the next-nodes list moves to the arena
    EMU_COLUMN_MIGRATE,       // extend_ins_end: an on-chip column moves to arena scratch mid-column
    EMU_ARENA_COLUMN,         // a column (root or child) created in arena scratch: wider than the on-chip buffers
    EMU_UNSTAGED_READ,        // a read whose strands are not staged on chip (L + 1 > lq)
    EMU_GENERAL_COLUMN,       // a child column computed by the general path
    EMU_READ_OVERFLOW,        // a read marked MGB_READ_OVERFLOW (retried with a larger arena)
    EMU_RAM_STOP_GENERAL,     // the general loop ends an extension on max_ram_per_alignment
    EMU_NODES_STOP_GENERAL,   // the general loop ends an extension on max_nodes_per_seq_char
    EMU_RAM_STOP_CHAIN,       // chain_loop ends an extension on max_ram_per_alignment
    EMU_NODES_STOP_CHAIN,     // chain_loop ends an extension on max_nodes_per_seq_char
    EMU_CONV_MOVE,            // conv_grow: a convergence-table entry outgrows its segment and moves to a new one
    EMU_N_PATHS
};
extern "C" unsigned long long mgb_emu_path_hits[EMU_N_PATHS];
#define MGB_EMU_HIT(path) __atomic_fetch_add(&mgb_emu_path_hits[path], 1ull, __ATOMIC_RELAXED)
// host emulation (tests) only: what the aggregator did with an alignment offered to it (mgb_emu_agg_hits[EmuAgg])
enum EmuAgg : int {
    EMU_AGG_REPLACE,          // it took the slot of the smallest entry of a full aggregator
    EMU_AGG_DUPLICATE,        // it was dropped as equal to an entry
    EMU_N_AGG
};
extern "C" unsigned long long mgb_emu_agg_hits[EMU_N_AGG];
#define MGB_EMU_AGG(ev) __atomic_fetch_add(&mgb_emu_agg_hits[ev], 1ull, __ATOMIC_RELAXED)
#else
#define MGB_EMU_HIT(path) ((void)0)
#define MGB_EMU_AGG(ev) ((void)0)
#endif

#if defined(MGB_PHASE_TIMERS) && MGB_DEVICE_CODE
#define MGB_TIC(var) long long var = clock64()
#define MGB_TOC(var, slot) phase_cycles[slot] += clock64() - var
#define MGB_COUNT(slot) ++phase_cycles[slot]
#else
#define MGB_COUNT(slot)
#define MGB_TIC(var)
#define MGB_TOC(var, slot)
#endif

// alignment slots: seed, tmp, ext[n_alt], bwd[n_alt], agg[n_alt]; the first bwd and agg slots depend on the configuration
// and are in WarpLayout (slot_bwd, slot_agg)
enum { SLOT_SEED = 0, SLOT_TMP = 1, SLOT_EXT = 2 };

// ------------------------------------------------------------------------------------
// Arena carving (shared by host sizing code and the kernel)
// ------------------------------------------------------------------------------------
MGB_HOSTDEV size_t align_up(size_t x) { return (x + 15) & ~(size_t)15; }

// State handed to / taken back from the extender's chain loop (ReadAligner::chain_loop, run by chain_entry in
// an aligner of its own): the extension's constants, the column that is the sole candidate, and the running values.
struct ChainIO {
    int e, rc, start, wlen, seed_off_m1, sh_offset, seed_seq_len, force_fixed, seed_is_query;
    score_t partial_sum_offset;
    const char *seed_seq; const uint64_t *seed_nodes; uint64_t seed_node0;
    uint32_t cells_limit;
    uint32_t ci; uint64_t c_node; int c_offset, c_trim; uint32_t c_bm; int c_pb;
    HeapItem cur_it;
    score_t cutoff, best_score, min_cell_score;
    uint64_t table_size_bytes; uint32_t n_cols, cells_used;
    uint64_t pf_node; uint2 pf_adj;
    int stop;                    // 1: the extension is over (queue empty), 2: column ci is left to the general code
    bool overflow;
    uint64_t dp_cells; uint32_t dp_columns;
};
struct WarpMem; struct WarpSmem;
#if MGB_DEVICE_CODE
static __device__ __forceinline__
#else
static inline
#endif
void chain_entry(const IndexView &ix, const DevConfig &cfg, const Caps &caps, const WarpMem &m, const WarpSmem &sm, int L,
                 ChainIO *io);

// Regions of a warp's arena as BYTE OFFSETS from its base. The layout is the same for every warp, so it is
// computed once on the host and travels in the kernel parameters (constant bank): a region's address is
// base + constant, no pointer table has to live in registers or on the stack.
struct WarpLayout {
    uint64_t cols, cells, heap, next_nodes, starts, conv_slots[2], conv_cells[2], seeds[2], psum[2];
    uint64_t slot0, slot_stride, slot_nodes, slot_seq, slot_cigar;      // alignment slot s starts at slot0 + s * slot_stride
    uint32_t slot_bwd, slot_agg;                                        // first slot of the bwd[] and agg[] groups
    uint64_t bt_ops, bt_path, bt_seq;
    uint64_t sfx_min;       // per query position: current min_seed_length (SuffixSeeder)
    uint64_t sfx_first, sfx_last, sfx_len;   // index_range result per query position
    // seed complexity filter: 3-mer codes / equal-3-mer masks (scratch) and, per strand, the largest start of a
    // low-complexity 3-mer interval ending at or before each 3-mer (see build_lowcx)
    uint64_t lc_word, lc_eq, lc_max[2];
    uint64_t epoch_store;   // conv-table epochs survive across the reads a warp processes
    uint64_t total;

    MGB_HOSTDEV size_t carve(const Caps &c) {
        size_t o = 0;
        auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes); return (uint64_t)r; };
        epoch_store = take(16);
        cols = take(sizeof(ColMeta) * c.max_cols);
        cells = take(sizeof(score_t) * 3 * (size_t)c.max_cells);
        heap = take(sizeof(HeapItem) * c.max_cols);
        next_nodes = take(sizeof(HeapItem) * c.max_cols);
        starts = take(sizeof(BtStart) * 2 * c.max_cols);
        for (int e = 0; e < 2; ++e) {
            conv_slots[e] = take(sizeof(ConvSlot) * c.hash_size);
            conv_cells[e] = take(sizeof(score_t) * c.max_conv_cells);
            seeds[e] = take(sizeof(SeedRec) * c.max_seeds);
            psum[e] = take(sizeof(int32_t) * (c.L_max + 8));
        }
        slot0 = o;
        take(sizeof(AlnHdr));
        slot_nodes = take(8 * (size_t)c.aln_nodes) - slot0;
        slot_seq = take(c.aln_seq) - slot0;
        slot_cigar = take(4 * (size_t)c.aln_cigar) - slot0;
        slot_stride = o - slot0;
        slot_bwd = 2 + c.n_alt;
        slot_agg = 2 + 2 * c.n_alt;
        o = slot0 + slot_stride * (2 + 3 * (size_t)c.n_alt);
        bt_ops = take(4 * (size_t)c.aln_cigar);
        bt_path = take(8 * (size_t)c.aln_nodes);
        bt_seq = take(c.aln_seq);
        sfx_min = take(c.L_max + 8);
        sfx_first = take(4 * ((size_t)c.L_max + 8)); sfx_last = take(4 * ((size_t)c.L_max + 8));
        sfx_len = take(c.L_max + 8);
        lc_word = take(c.L_max + 8); lc_eq = take(8 * ((size_t)c.L_max + 8));
        lc_max[0] = take(4 * ((size_t)c.L_max + 8)); lc_max[1] = take(4 * ((size_t)c.L_max + 8));
        total = o;
        return o;
    }
};

struct WarpMem {
    char *base; const WarpLayout *lay;
    MGB_HD ColMeta* cols() const { return (ColMeta*)(base + lay->cols); }
    MGB_HD score_t* cells() const { return (score_t*)(base + lay->cells); }
    MGB_HD HeapItem* heap() const { return (HeapItem*)(base + lay->heap); }
    MGB_HD HeapItem* next_nodes() const { return (HeapItem*)(base + lay->next_nodes); }
    MGB_HD BtStart* starts() const { return (BtStart*)(base + lay->starts); }
    MGB_HD ConvSlot* conv_slots(int e) const { return (ConvSlot*)(base + lay->conv_slots[e]); }
    MGB_HD score_t* conv_cells(int e) const { return (score_t*)(base + lay->conv_cells[e]); }
    MGB_HD SeedRec* seeds(int e) const { return (SeedRec*)(base + lay->seeds[e]); }
    MGB_HD int32_t* psum(int e) const { return (int32_t*)(base + lay->psum[e]); }
    MGB_HD AlnSlot slot(int s) const {
        char *p = base + lay->slot0 + (uint64_t)s * lay->slot_stride;
        AlnSlot a; a.h = (AlnHdr*)p; a.nodes = (uint64_t*)(p + lay->slot_nodes); a.seq = p + lay->slot_seq;
        a.cigar = (uint32_t*)(p + lay->slot_cigar);
        return a;
    }
    MGB_HD uint32_t* bt_ops() const { return (uint32_t*)(base + lay->bt_ops); }
    MGB_HD uint64_t* bt_path() const { return (uint64_t*)(base + lay->bt_path); }
    MGB_HD char* bt_seq() const { return base + lay->bt_seq; }
    MGB_HD uint8_t* sfx_min() const { return (uint8_t*)(base + lay->sfx_min); }
    MGB_HD uint32_t* sfx_first() const { return (uint32_t*)(base + lay->sfx_first); }
    MGB_HD uint32_t* sfx_last() const { return (uint32_t*)(base + lay->sfx_last); }
    MGB_HD uint8_t* sfx_len() const { return (uint8_t*)(base + lay->sfx_len); }
    MGB_HD uint8_t* lc_word() const { return (uint8_t*)(base + lay->lc_word); }
    MGB_HD uint64_t* lc_eq() const { return (uint64_t*)(base + lay->lc_eq); }
    MGB_HD int32_t* lc_max(int s) const { return (int32_t*)(base + lay->lc_max[s]); }
    MGB_HD uint32_t* epoch_store() const { return (uint32_t*)(base + lay->epoch_store); }
};

// Per-warp on-chip working set (shared memory on the device, a heap block in the host emulation), again as
// offsets from the warp's base: two DP column buffers (parent / child ping-pong), the query strands and their
// suffix sums, the best-first queue, the outgoing-edge scratch and the aggregator's keys.
struct SmemLayout {
    int bmax, lq, hcap;       // column buffer cells; staged query capacity in characters (0: not staged); queue entries
    uint32_t buf0, psum0, psum1, q0, q1, ctx, mask0, mask1, heap, nn, out_nodes, out_scores, out_chars, total;
    uint32_t agg, agg_ord;    // AggKey per aggregator entry; the entries in output order (run())
    uint32_t prof0, prof1;    // DNA block layout only: per query position the scores against A, C, G, T, one byte each
    uint32_t has_prof;
    MGB_HOSTDEV size_t carve(int bmax_, int lq_, int hcap_, int n_alt, bool with_prof = false) {
        size_t o = 0;
        auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes); return (uint32_t)r; };
        bmax = bmax_; lq = lq_; hcap = hcap_;
        buf0 = take(sizeof(score_t) * 6 * (size_t)bmax);      // two buffers, each: S[bmax] | E[bmax] | F[bmax]
        psum0 = take(4 * ((size_t)lq + 8)); psum1 = take(4 * ((size_t)lq + 8));
        q0 = take((size_t)lq + 8); q1 = take((size_t)lq + 8);
        ctx = take(sizeof(StrandCtx) * 2);
        mask0 = take(4 * ((size_t)lq / 32 + 2)); mask1 = take(4 * ((size_t)lq / 32 + 2));   // (lq / 32 + 2) words each
        heap = take(sizeof(HeapItem) * hcap);
        nn = take(sizeof(HeapItem) * hcap);
        out_nodes = take(8 * kMaxOut);
        out_scores = take(4 * kMaxOut); out_chars = take(kMaxOut);
        agg = take(sizeof(AggKey) * (size_t)n_alt); agg_ord = take(4 * (size_t)n_alt);
        has_prof = with_prof && lq > 0 ? 1u : 0u;
        prof0 = prof1 = 0;
        if (has_prof) { prof0 = take(4 * ((size_t)lq + 8)); prof1 = take(4 * ((size_t)lq + 8)); }
        total = (uint32_t)o;
        return o;
    }
};
struct WarpSmem {
    char *base; const SmemLayout *lay;
    MGB_HD int bmax() const { return lay->bmax; }
    MGB_HD int lq() const { return lay->lq; }
    MGB_HD int hcap() const { return lay->hcap; }
    MGB_HD score_t* buf(int b) const { return (score_t*)(base + lay->buf0) + (size_t)b * 3 * lay->bmax; }
    MGB_HD int32_t* psum0() const { return (int32_t*)(base + lay->psum0); }
    MGB_HD int32_t* psum1() const { return (int32_t*)(base + lay->psum1); }
    MGB_HD char* q0() const { return base + lay->q0; }
    MGB_HD char* q1() const { return base + lay->q1; }
    MGB_HD StrandCtx* ctx() const { return (StrandCtx*)(base + lay->ctx); }
    MGB_HD uint32_t* mask0() const { return (uint32_t*)(base + lay->mask0); }
    MGB_HD uint32_t* mask1() const { return (uint32_t*)(base + lay->mask1); }
    MGB_HD HeapItem* heap() const { return (HeapItem*)(base + lay->heap); }
    MGB_HD HeapItem* nn() const { return (HeapItem*)(base + lay->nn); }
    MGB_HD uint64_t* out_nodes() const { return (uint64_t*)(base + lay->out_nodes); }
    MGB_HD int32_t* out_scores() const { return (int32_t*)(base + lay->out_scores); }
    MGB_HD uint8_t* out_chars() const { return (uint8_t*)(base + lay->out_chars); }
    MGB_HD AggKey* agg() const { return (AggKey*)(base + lay->agg); }
    MGB_HD int32_t* agg_ord() const { return (int32_t*)(base + lay->agg_ord); }
    MGB_HD uint32_t* prof4(int s) const { return (uint32_t*)(base + (s ? lay->prof1 : lay->prof0)); }
};

MGB_HOSTDEV uint32_t cig_pack(uint32_t op, uint32_t len) { return (len << 3) | op; }
MGB_HOSTDEV uint32_t cig_op(uint32_t x) { return x & 7u; }
MGB_HOSTDEV uint32_t cig_len(uint32_t x) { return x >> 3; }
enum { OP_S = 0, OP_X = 1, OP_M = 2, OP_D = 3, OP_I = 4, OP_G = 5 };

// ------------------------------------------------------------------------------------
// The per-read aligner
// ------------------------------------------------------------------------------------
struct ReadAligner {
    const IndexView &ix;
    const DevConfig &cfg;
    const Caps &caps;
    const WarpMem m;             // base + constant offsets: two small objects that live in registers
    const WarpSmem sm;

    // read
    int L;
    StrandCtx *cx;               // sm.ctx: per-strand state (query, seeds, extender bookkeeping)

    bool overflow;
    ReadStats stats;


    // DP table of the extension in flight
    uint32_t n_cols;
    uint32_t cells_used;
    int n_agg;

    MGB_HD ReadAligner(const IndexView &ix_, const DevConfig &cfg_, const Caps &caps_, const WarpMem &m_,
                       const WarpSmem &sm_)
        : ix(ix_), cfg(cfg_), caps(caps_), m(m_), sm(sm_), cx(sm_.ctx()) {}

    // --------------------------------------------------------------------------------
    // small helpers
    // --------------------------------------------------------------------------------
    // committed columns (layouts: see ColMeta); S always starts at cells_off
    MGB_HD static int capr_of(int size) { return (size + 5 + 7) & ~7; }
    MGB_HD score_t& cellS(const ColMeta &c, int j) { return m.cells()[(size_t)c.cells_off + j]; }
    MGB_HD score_t& cellE(const ColMeta &c, int j) { return m.cells()[(size_t)c.cells_off + (c.size + 5) + j]; }    // FMT_FULL
    MGB_HD score_t& cellF(const ColMeta &c, int j) {
        return m.cells()[(size_t)c.cells_off + (c.fmt == FMT_FULL ? 2 * (c.size + 5) : capr_of(c.size) + 8) + j];
    }
    MGB_HD uint32_t cell_flags(const ColMeta &c, int j) {                                                          // compact
        return reinterpret_cast<const uint8_t*>(m.cells() + (size_t)c.cells_off + capr_of(c.size))[j];
    }
    // the backtrack's comparisons with E and F (extender.cpp:943-999), from the cells or from the flag bytes
    MGB_HD bool bt_is_ins(const ColMeta &c, int j, score_t sv) {
        return c.fmt == FMT_FULL ? sv == cellE(c, j) : (cell_flags(c, j) & CF_INS) != 0;
    }
    MGB_HD bool bt_ins_ext(const ColMeta &c, int j) {
        return c.fmt == FMT_FULL ? cellE(c, j) == wadd(cellE(c, j - 1), cfg.gap_ext) : (cell_flags(c, j) & CF_INS_EXT) != 0;
    }
    MGB_HD bool bt_is_del(const ColMeta &c, int j, score_t sv) {
        return c.fmt == FMT_FULL ? sv == cellF(c, j) : (cell_flags(c, j) & CF_DEL) != 0;
    }
    MGB_HD bool bt_del_ext(const ColMeta &c, const ColMeta &p, int pos) {
        return c.fmt == FMT_FULL ? cellF(c, pos - c.trim) == wadd(wadd(cellF(p, pos - p.trim), c.score), cfg.gap_ext)
                                 : (cell_flags(c, pos - c.trim) & CF_DEL_EXT) != 0;
    }

    MGB_HD int prof_score(int s, int x, int code) const {   // profile_score_[code][x]
        return (x >= 1 && x <= L) ? cfg.prof[code][(uint8_t)cx[s].q[x - 1]] : 0;
    }
    MGB_HD bool prof_is_match(int s, int x, int code) const {
        return (x >= 1 && x <= L) ? cfg.opmatch[code][(uint8_t)cx[s].q[x - 1]] : false;
    }
    MGB_HD uint32_t encode_char(uint8_t ch) const { return cfg.code_of[ch]; }

    MGB_HD int aln_clipping(const AlnSlot &a) const {
        return a.h->n_cigar && cig_op(a.cigar[0]) == OP_S ? (int)cig_len(a.cigar[0]) : 0;
    }
    MGB_HD int aln_end_clipping(const AlnSlot &a) const {
        int n = a.h->n_cigar;
        return n && cig_op(a.cigar[n - 1]) == OP_S ? (int)cig_len(a.cigar[n - 1]) : 0;
    }

    MGB_HD void copy_slot(int dst, int src) {
        const AlnSlot d = m.slot(dst); const AlnSlot s = m.slot(src);
        wsync();
        AlnHdr h = *s.h;
        for (int i = wlane(); i < h.n_nodes; i += kWarp) d.nodes[i] = s.nodes[i];
        for (int i = wlane(); i < h.seq_len; i += kWarp) d.seq[i] = s.seq[i];
        for (int i = wlane(); i < h.n_cigar; i += kWarp) d.cigar[i] = s.cigar[i];
        *d.h = h;
        wsync();
    }

    // Alignment(const Seed&, config) (alignment.hpp:154-165) materialised into a slot
    MGB_HD void seed_to_slot(int slot, int s, const SeedRec &sd) {
        const AlnSlot a = m.slot(slot);
        wsync();
        for (int i = wlane(); i < (int)sd.n_nodes; i += kWarp)
            a.nodes[i] = sd.n_nodes == 1 ? sd.node0 : cx[s].qnodes[sd.clip + i];
        for (int i = wlane(); i < (int)sd.len; i += kWarp) a.seq[i] = cx[s].q[sd.clip + i];
        int end_clip = L - (int)sd.clip - (int)sd.len;
        int nc = 0;
        if (sd.clip) a.cigar[nc++] = cig_pack(OP_S, sd.clip);
        a.cigar[nc++] = cig_pack(OP_M, sd.len);
        if (end_clip) a.cigar[nc++] = cig_pack(OP_S, end_clip);
        AlnHdr h;
        h.q_len = sd.len; h.n_nodes = sd.n_nodes; h.seq_len = sd.len; h.n_cigar = nc;
        h.score = cx[s].ps[sd.clip] - cx[s].ps[sd.clip + sd.len]
                + (!sd.clip ? cfg.left_end_bonus : 0) + (!end_clip ? cfg.right_end_bonus : 0);
        h.offset = sd.offset; h.orientation = s; h.used = 1;
        *a.h = h;
        wsync();
    }

    // alignment.cpp:177-190 (no npos nodes on this path)
    MGB_HD void trim_offset(int slot) {
        const AlnSlot a = m.slot(slot);
        AlnHdr h = *a.h;
        if (!h.offset || h.n_nodes <= 1) return;
        int trim = imin((int)h.offset, h.n_nodes - 1);
        wsync();
        // shift nodes down by `trim` (chunked so that reads precede overlapping writes)
        for (int base = 0; base < h.n_nodes - trim; base += kWarp) {
            int i = base + wlane();
            uint64_t v = i < h.n_nodes - trim ? a.nodes[i + trim] : 0;
            wsync();
            if (i < h.n_nodes - trim) a.nodes[i] = v;
            wsync();
        }
        h.offset -= trim; h.n_nodes -= trim;
        *a.h = h;
        wsync();
    }

    // alignment.cpp:540-561, RCDBG branch. Returns false if the alignment became empty.
    MGB_HD bool reverse_complement_slot(int slot) {
        trim_offset(slot);
        const AlnSlot a = m.slot(slot);
        AlnHdr h = *a.h;
        if (h.offset) { h.used = 0; h.n_nodes = 0; *a.h = h; return false; }
        wsync();
        for (int base = 0; base < (h.n_cigar + 1) / 2; base += kWarp) {
            int i = base + wlane();
            if (i < h.n_cigar / 2) {
                uint32_t x = a.cigar[i], y = a.cigar[h.n_cigar - 1 - i];
                a.cigar[i] = y; a.cigar[h.n_cigar - 1 - i] = x;
            }
        }
        for (int base = 0; base < (h.n_nodes + 1) / 2; base += kWarp) {
            int i = base + wlane();
            if (i < h.n_nodes / 2) {
                uint64_t x = a.nodes[i], y = a.nodes[h.n_nodes - 1 - i];
                a.nodes[i] = y; a.nodes[h.n_nodes - 1 - i] = x;
            }
        }
        for (int base = 0; base < (h.seq_len + 1) / 2; base += kWarp) {
            int i = base + wlane();
            if (i < (h.seq_len + 1) / 2) {
                int jj = h.seq_len - 1 - i;
                char x = complement_char(a.seq[i]), y = complement_char(a.seq[jj]);
                a.seq[i] = y; a.seq[jj] = x;
            }
        }
        h.orientation ^= 1u;
        *a.h = h;
        wsync();
        h.q_len = L - aln_clipping(a) - aln_end_clipping(a);
        *a.h = h;
        wsync();
        return true;
    }

    // alignment.cpp:563-702 on a plain DBGSuccinct (CANONICAL-mode graph, no RCDBG view): the path of the
    // reverse complement is looked up in the graph itself. Returns false if the alignment became empty.
    MGB_HD bool reverse_complement_slot_plain(int slot) {
        trim_offset(slot);
        const AlnSlot a = m.slot(slot);
        AlnHdr h = *a.h;
        const int K = ix.k;
        uint8_t *codes = (uint8_t*)m.bt_seq();                    // scratch (not in use outside backtrack)
        auto kill = [&]() { h.used = 0; h.n_nodes = 0; *a.h = h; wsync(); return false; };
        // reverse_complement_seq_path (sequence_graph.cpp:563-573) of a.seq[0..len): complement in place, map
        auto rc_seq_path = [&](int len) {
            wsync();
            for (int base = 0; base < (len + 1) / 2; base += kWarp) {
                int i = base + wlane();
                if (i < (len + 1) / 2) {
                    int jj = len - 1 - i;
                    char x = complement_char(a.seq[i]), y = complement_char(a.seq[jj]);
                    a.seq[i] = y; a.seq[jj] = x;
                }
            }
            wsync();
            for (int i = wlane(); i < len; i += kWarp) codes[i] = (uint8_t)encode_char((uint8_t)a.seq[i]);
            for (int i = wlane(); i < len - K + 1; i += kWarp) a.nodes[i] = 0;
            wsync();
            map_to_edges(ix, codes, len, a.nodes);
            wsync();
        };
        if ((int)caps.aln_seq < K + 8 || (int)caps.aln_nodes < 2) { overflow = true; return false; }
        if (!h.offset) {
            if (h.seq_len < K) return kill();
            rc_seq_path(h.seq_len);
            h.n_nodes = h.seq_len - K + 1;
        } else {
            // one node, its first `offset` characters are not part of the alignment: rebuild the whole k-mer
            const int off = (int)h.offset;
            const uint64_t node = a.nodes[0];
            wsync();
            for (int i = wlane(); i < h.seq_len; i += kWarp) codes[K + i] = (uint8_t)a.seq[i];   // stash
            wsync();
            {   // BOSS::get_node_str + edge label: last characters first (boss.cpp:663-690)
                uint64_t e = node;
                for (int i = K - 2; i >= 0; --i) {
                    const uint32_t c = node_last_value(ix, e);
                    if (i < off) a.seq[i] = cfg.letters[c];
                    e = (uint64_t)load_radj(ix, e).x;         // bwd(e)
                }
            }
            wsync();
            for (int i = wlane(); i < h.seq_len; i += kWarp) a.seq[off + i] = (char)codes[K + i];
            wsync();
            if (a.seq[0] == '$') {
                // starts in a source dummy k-mer: walk forward along the last outgoing edge until the k-mer is
                // real (:572-640), then take the reverse complement of that k-mer
                LineCache lc;
                uint64_t edge = node;
                uint32_t label = lc.get_W(ix, edge) % ix.sigma;
                int len = off + h.seq_len;                       // == K
                for (int i = 0; i < off; ++i) {
                    edge = fwd(ix, lc, edge, label);
                    label = lc.get_W(ix, edge) % ix.sigma;
                    if (label == 0) return kill();
                    if (len >= (int)caps.aln_seq) { overflow = true; return false; }
                    a.seq[len++] = cfg.letters[label];
                }
                wsync();
                for (int base = 0; base < K; base += kWarp) {     // seq = seq.substr(off)
                    int i = base + wlane();
                    char v = i < K ? a.seq[off + i] : 0;
                    wsync();
                    if (i < K) a.seq[i] = v;
                    wsync();
                }
                rc_seq_path(K);
                if (a.nodes[0] == 0) return kill();
                wsync();
                for (int base = 0; base < K - off; base += kWarp) {     // keep the last K - off characters
                    int i = base + wlane();
                    char v = i < K - off ? a.seq[off + i] : 0;
                    wsync();
                    if (i < K - off) a.seq[i] = v;
                    wsync();
                }
            } else {
                rc_seq_path(K);
                if (a.nodes[0] == 0) return kill();
                // drop the ending that corresponds to the added prefix: first incoming node each time
                // (adjacent_incoming_nodes, dbg_succinct.cpp:176-193)
                uint64_t cur = a.nodes[0];
                for (int i = 0; i < off; ++i) {
                    const uint2 r = load_radj(ix, cur);
                    const uint32_t d = node_last_value(ix, cur);
                    uint64_t edge = r.x, found = 0;
                    LineCache lc;
                    while (true) {
                        if (in_graph(ix, edge)) { found = edge; break; }
                        if (!radj_multi(ix, r.y)) break;
                        if (++edge > ix.n) break;
                        uint32_t w;
                        edge = succ_W2(ix, lc, edge, d, &w);
                        if (w != d + ix.sigma) break;
                    }
                    if (!found) return kill();
                    cur = found;
                }
                wsync();
                a.nodes[0] = cur;
                wsync();
            }
            h.n_nodes = 1;
            h.seq_len = K - off;
        }
        wsync();
        for (int base = 0; base < (h.n_cigar + 1) / 2; base += kWarp) {
            int i = base + wlane();
            if (i < h.n_cigar / 2) {
                uint32_t x = a.cigar[i], y = a.cigar[h.n_cigar - 1 - i];
                a.cigar[i] = y; a.cigar[h.n_cigar - 1 - i] = x;
            }
        }
        h.orientation ^= 1u;
        *a.h = h;
        wsync();
        h.q_len = L - aln_clipping(a) - aln_end_clipping(a);
        *a.h = h;
        wsync();
        return true;
    }
    // alignment.cpp:563-702 on a PRIMARY graph behind CanonicalDBG: reverse_complement_seq_path flips the node ids
    // (canonical_dbg.cpp:555-565) instead of mapping the sequence. Returns false if the alignment became empty.
    MGB_HD bool reverse_complement_slot_primary(int slot) {
        trim_offset(slot);
        const AlnSlot a = m.slot(slot);
        AlnHdr h = *a.h;
        const int K = ix.k;
        auto kill = [&]() { h.used = 0; h.n_nodes = 0; *a.h = h; wsync(); return false; };
        auto rc_seq = [&](int len) {
            wsync();
            for (int base = 0; base < (len + 1) / 2; base += kWarp) {
                int i = base + wlane();
                if (i < (len + 1) / 2) {
                    int jj = len - 1 - i;
                    char x = complement_char(a.seq[i]), y = complement_char(a.seq[jj]);
                    a.seq[i] = y; a.seq[jj] = x;
                }
            }
            wsync();
        };
        if ((int)caps.aln_seq < 2 * K + 8) { overflow = true; return false; }
        if (!h.offset) {
            rc_seq(h.seq_len);
            for (int base = 0; base < (h.n_nodes + 1) / 2; base += kWarp) {
                int i = base + wlane();
                if (i < (h.n_nodes + 1) / 2) {
                    uint64_t x = canon_flip(a.nodes[i]), y = canon_flip(a.nodes[h.n_nodes - 1 - i]);
                    a.nodes[i] = y; a.nodes[h.n_nodes - 1 - i] = x;
                }
            }
            wsync();
        } else {
            const int off = (int)h.offset;
            uint64_t node = a.nodes[0];
            const uint64_t base_node = node > ix.n ? node - ix.n : node;
            uint8_t *stash = (uint8_t*)m.bt_seq();                 // scratch (not in use outside backtrack)
            wsync();
            for (int i = wlane(); i < h.seq_len; i += kWarp) stash[i] = (uint8_t)a.seq[i];
            wsync();
            // the first `off` characters of CanonicalDBG::get_node_sequence(node) (:423-432)
            if (node == base_node) {
                uint64_t e = node;
                for (int i = K - 2; i >= 0; --i) {
                    const uint32_t c = node_last_value(ix, e);
                    if (i < off) a.seq[i] = cfg.letters[c];
                    e = (uint64_t)load_radj(ix, e).x;
                }
            } else {                                             // reverse complement of the stored k-mer
                LineCache lc;
                uint64_t e = base_node;
                for (int t = 0; t < off; ++t) {
                    const uint32_t c = t == 0 ? lc.get_W(ix, base_node) % ix.sigma : node_last_value(ix, e);
                    a.seq[t] = (char)complement_char((uint8_t)cfg.letters[c]);
                    if (t > 0) e = (uint64_t)load_radj(ix, e).x;
                }
            }
            wsync();
            for (int i = wlane(); i < h.seq_len; i += kWarp) a.seq[off + i] = (char)stash[i];
            wsync();
            if (a.seq[0] == '$') {
                if (node != base_node) return kill();            // reverse complement of a sink dummy k-mer (:592-597)
                int num_sentinels = 0;
                for (int i = 0; i < off + h.seq_len; ++i) if (a.seq[i] == '$') num_sentinels = i + 1;
                const int num_first_steps = imin(off, num_sentinels);
                LineCache lc;
                uint64_t edge = node;
                uint32_t label = lc.get_W(ix, edge) % ix.sigma;
                int len = off + h.seq_len;                       // == K
                for (int i = 0; i < num_first_steps; ++i) {
                    edge = fwd(ix, lc, edge, label);
                    label = lc.get_W(ix, edge) % ix.sigma;
                    if (label == 0) return kill();
                    if (len >= (int)caps.aln_seq) { overflow = true; return false; }
                    node = edge;
                    wsync();
                    a.seq[len++] = cfg.letters[label];
                }
                for (int i = num_first_steps; i < off; ++i) {    // last non-'$' child through the wrapper (:624-646)
                    const int n = canon_out(node, sm.out_nodes(), sm.out_chars());
                    wsync();
                    if (n > kMaxOut) { overflow = true; return false; }
                    if (!n) return kill();
                    if (len >= (int)caps.aln_seq) { overflow = true; return false; }
                    node = sm.out_nodes()[n - 1];
                    a.seq[len++] = (char)sm.out_chars()[n - 1];
                    wsync();
                }
                wsync();
                for (int base = 0; base < K; base += kWarp) {     // seq = seq.substr(off)
                    int i = base + wlane();
                    char v = i < K ? a.seq[off + i] : 0;
                    wsync();
                    if (i < K) a.seq[i] = v;
                    wsync();
                }
                rc_seq(K);
                node = canon_flip(node);
                for (int base = 0; base < K - off; base += kWarp) {     // keep the last K - off characters
                    int i = base + wlane();
                    char v = i < K - off ? a.seq[off + i] : 0;
                    wsync();
                    if (i < K - off) a.seq[i] = v;
                    wsync();
                }
            } else {
                rc_seq(K);
                node = canon_flip(node);
                // drop the ending that corresponds to the added prefix: first incoming node each time (:667-690)
                for (int i = 0; i < off; ++i) {
                    uint64_t sent = 0;
                    const int n = canon_in(node, sm.out_nodes(), sm.out_chars(), &sent);
                    wsync();
                    if (n > kMaxOut) { overflow = true; return false; }
                    if (!n && !sent) return kill();
                    node = n ? sm.out_nodes()[0] : sent;
                    wsync();
                }
            }
            wsync();
            a.nodes[0] = node;
            h.n_nodes = 1;
            h.seq_len = K - off;
        }
        wsync();
        for (int base = 0; base < (h.n_cigar + 1) / 2; base += kWarp) {
            int i = base + wlane();
            if (i < h.n_cigar / 2) {
                uint32_t x = a.cigar[i], y = a.cigar[h.n_cigar - 1 - i];
                a.cigar[i] = y; a.cigar[h.n_cigar - 1 - i] = x;
            }
        }
        h.orientation ^= 1u;
        *a.h = h;
        wsync();
        h.q_len = L - aln_clipping(a) - aln_end_clipping(a);
        *a.h = h;
        wsync();
        return true;
    }
    // Alignment::reverse_complement against the graph view the backward extender works on
    MGB_HD bool reverse_complement_for_bwd(int slot) {
        if (MGB_CANONICAL(cfg) && MGB_PRIMARY(ix)) return reverse_complement_slot_primary(slot);
        return MGB_CANONICAL(cfg) ? reverse_complement_slot_plain(slot) : reverse_complement_slot(slot);
    }

    // --------------------------------------------------------------------------------
    // graph access for the extender
    // --------------------------------------------------------------------------------
    // DBGSuccinct::call_outgoing_kmers (dbg_succinct.cpp:110-139); '$' targets are skipped
    // as the extender does (extender.cpp:381-384). Returns the number of (node, char) pairs.
    MGB_HD int outgoing_fwd(uint64_t node, uint64_t *nodes, uint8_t *chars) {
        // the record of the most recently created column was requested while its DP was computed
        const Adj a = (!MGB_WIDE(ix) && node == pf_node) ? adj_decode(pf_adj) : load_adj_any(ix, node);
        if (!a.last) return 0;
        const uint32_t all = a.all, ok = a.ok;
        const uint64_t first = (uint64_t)a.last - popc32(all) + 1;
        int n = 0;
        for (uint32_t c = 1; c < ix.sigma; ++c) {
            if (!((ok >> c) & 1u)) continue;
            if (n < kMaxOut) { nodes[n] = first + popc32(all & ((1u << c) - 1u)); chars[n] = cfg.letters[c]; }
            ++n;
        }
        return n;
    }

    // RCDBG::call_outgoing_kmers (rc_dbg.hpp:86-97) -> NodeFirstCache::call_incoming_kmers
    // (node_first_cache.cpp:40-50): incoming nodes in call_incoming_to_target order
    // (boss.cpp:766-786) with the complement of their first character, through the reverse
    // adjacency records.
    MGB_HD int outgoing_rc(uint64_t node, uint64_t *nodes, uint8_t *chars) {
        const uint2 r = load_radj(ix, node);
        const uint32_t d = node_last_value(ix, node);
        int n = 0;
        uint64_t edge = r.x;
        LineCache lc;
        while (true) {
            if (in_graph(ix, edge)) {
                const uint32_t c = radj_char(ix, load_radj(ix, edge).y);
                uint8_t ch = complement_char((uint8_t)cfg.letters[c]);
                if (ch != '$') {
                    if (n < kMaxOut) { nodes[n] = edge; chars[n] = ch; }
                    ++n;
                }
            }
            if (!radj_multi(ix, r.y)) break;             // single incoming edge
            if (++edge > ix.n) break;
            uint32_t w;
            edge = succ_W2(ix, lc, edge, d, &w);
            if (w != d + ix.sigma) break;
        }
        return n;
    }

    // --------------------------------------------------------------------------------
    // CanonicalDBG over a PRIMARY graph (canonical_dbg.cpp): nodes 1..n are the stored k-mers, n+1..2n their
    // reverse complements. The rc-strand jumps that the reference answers with k-1 bwd steps and an index
    // lookup behind LRU caches (NodeFirstCache) are one load from IndexView::rcs / rcp here.
    // --------------------------------------------------------------------------------
    MGB_HD uint64_t canon_flip(uint64_t node) const {            // CanonicalDBG::reverse_complement(node), :521-553
        if (node > ix.n) return node - ix.n;
        if ((ix.k & 1u) || !ix.palin) return node + ix.n;
        return ((ix.palin[node >> 5] >> (node & 31)) & 1u) ? node : node + ix.n;
    }
    MGB_HD static bool has_char(const uint8_t *chars, int n, uint8_t ch) {
        bool f = false;
        for (int t = 0; t < n && t < kMaxOut; ++t) f = f || chars[t] == ch;
        return f;
    }
    // call_outgoing_kmers (:158-243) of a stored node: its children in the base graph, then the parents of its
    // reverse complement that no base child covers. Non-'$' children in callback order; *sentinel receives the
    // '$' child the reference reports when there is no other (has_sentinel_, :238-242), 0 if none.
    MGB_HD int canon_base_out(uint64_t base, uint64_t *nodes, uint8_t *chars, uint64_t *sentinel) {
        const Adj a = load_adj_any(ix, base);
        int n = 0;
        uint64_t dollar = 0;
        if (a.last) {
            const uint64_t first = (uint64_t)a.last - popc32(a.all) + 1;
            if ((a.all & 1u) && in_graph(ix, first)) dollar = first;
            for (uint32_t c = 1; c < ix.sigma; ++c) {
                if (!((a.ok >> c) & 1u)) continue;
                if (n < kMaxOut) { nodes[n] = first + popc32(a.all & ((1u << c) - 1u)); chars[n] = cfg.letters[c]; }
                ++n;
            }
        }
        const int max_children = (int)ix.sigma - (ix.valid ? 0 : 1);
        if (n < max_children) {
            const uint64_t rc_edge = ix.rcs[base];
            if (rc_edge) {
                // NodeFirstCache::call_incoming_edges (node_first_cache.cpp:26-38) of the rc node
                const uint2 r = load_radj(ix, rc_edge);
                const uint32_t d = node_last_value(ix, rc_edge);
                uint64_t edge = r.x;
                LineCache lc;
                while (true) {
                    if (in_graph(ix, edge)) {
                        const uint32_t c = radj_char(ix, load_radj(ix, edge).y);
                        if (c != 0) {
                            const uint8_t ch = (uint8_t)cfg.letters[ix.sigma - c];
                            if (!has_char(chars, n, ch)) {
                                if (n < kMaxOut) { nodes[n] = canon_flip(edge); chars[n] = ch; }
                                ++n;
                            }
                        }                               // a '$' seen through the rc strand is never reported (:209-233)
                    }
                    if (!radj_multi(ix, r.y)) break;
                    if (++edge > ix.n) break;
                    uint32_t w;
                    edge = succ_W2(ix, lc, edge, d, &w);
                    if (w != d + ix.sigma) break;
                }
            }
        }
        if (sentinel) *sentinel = (!ix.valid && dollar && n == 0) ? dollar : 0;
        return n;
    }
    // call_incoming_kmers (:245-336) of a stored node, same conventions
    MGB_HD int canon_base_in(uint64_t base, uint64_t *nodes, uint8_t *chars, uint64_t *sentinel) {
        int n = 0;
        uint64_t dollar = 0;
        {   // DBGSuccinct::call_incoming_kmers through the reverse adjacency records
            const uint2 r = load_radj(ix, base);
            const uint32_t d = node_last_value(ix, base);
            uint64_t edge = r.x;
            LineCache lc;
            while (true) {
                if (in_graph(ix, edge)) {
                    const uint32_t c = radj_char(ix, load_radj(ix, edge).y);
                    if (c != 0) {
                        if (n < kMaxOut) { nodes[n] = edge; chars[n] = (uint8_t)cfg.letters[c]; }
                        ++n;
                    } else {
                        dollar = edge;
                    }
                }
                if (!radj_multi(ix, r.y)) break;
                if (++edge > ix.n) break;
                uint32_t w;
                edge = succ_W2(ix, lc, edge, d, &w);
                if (w != d + ix.sigma) break;
            }
        }
        const int max_parents = (int)ix.sigma - (ix.valid ? 0 : 1);
        if (n < max_parents) {
            const uint64_t rc_edge = ix.rcp[base];
            if (rc_edge) {
                LineCache lc;
                // BOSS::call_outgoing (boss.hpp:779-784): the edges of the rc node, last one first
                uint64_t edge = rc_edge;
                do {
                    if (in_graph(ix, edge)) {
                        const uint32_t c = lc.get_W(ix, edge) % ix.sigma;
                        if (c != 0) {
                            const uint8_t ch = (uint8_t)cfg.letters[ix.sigma - c];
                            if (!has_char(chars, n, ch)) {
                                if (n < kMaxOut) { nodes[n] = canon_flip(edge); chars[n] = ch; }
                                ++n;
                            }
                        }
                    }
                } while (--edge && !lc.get_last(ix, edge));
            }
        }
        if (sentinel) *sentinel = (!ix.valid && dollar && n == 0) ? dollar : 0;
        return n;
    }
    // flips a neighbour list onto the other strand (:163-172, :250-259)
    MGB_HD void canon_flip_list(int n, uint64_t *nodes, uint8_t *chars, uint64_t *sentinel) {
        for (int t = 0; t < n && t < kMaxOut; ++t) { nodes[t] = canon_flip(nodes[t]); chars[t] = complement_char(chars[t]); }
        if (sentinel && *sentinel) *sentinel = canon_flip(*sentinel);
    }
    MGB_HD int canon_out(uint64_t node, uint64_t *nodes, uint8_t *chars, uint64_t *sentinel = nullptr) {
        if (node <= ix.n) return canon_base_out(node, nodes, chars, sentinel);
        int n = canon_base_in(node - ix.n, nodes, chars, sentinel);
        canon_flip_list(n, nodes, chars, sentinel);
        return n;
    }
    MGB_HD int canon_in(uint64_t node, uint64_t *nodes, uint8_t *chars, uint64_t *sentinel = nullptr) {
        if (node <= ix.n) return canon_base_in(node, nodes, chars, sentinel);
        int n = canon_base_out(node - ix.n, nodes, chars, sentinel);
        canon_flip_list(n, nodes, chars, sentinel);
        return n;
    }

    // dbg_succinct.cpp:617-630
    MGB_HD bool has_multiple_outgoing(uint64_t node) {
        if (MGB_PRIMARY(ix)) {                               // canonical_dbg.cpp:366-380
            uint64_t sent;
            return canon_out(node, sm.out_nodes(), sm.out_chars(), &sent) > 1;
        }
        // !get_last(fwd(node, d) - 1): the target node has more than one edge
        const Adj a = load_adj_any(ix, node);
        return a.last && popc32(a.all) > 1;
    }
    // dbg_succinct.cpp:662-680
    MGB_HD bool has_single_incoming(uint64_t node) {
        if (MGB_PRIMARY(ix)) {                               // canonical_dbg.cpp:382-392
            uint64_t sent;
            int n = canon_in(node, sm.out_nodes(), sm.out_chars(), &sent);
            return n + (sent ? 1 : 0) == 1;
        }
        if (node == 1) return false;
        if (!ix.valid) return !radj_multi(ix, load_radj(ix, node).y);   // mask dropped: !multi-incoming
        LineCache lc;
        uint64_t x = bwd(ix, lc, node);
        uint32_t w = node_last_value(ix, node);
        bool first_valid = !ix.valid || in_graph(ix, x);
        if (x + 1 == ix.n + 1) return first_valid;
        uint32_t wn;
        if (first_valid) {
            // BOSS::is_single_incoming (boss.cpp:803-816)
            succ_W2(ix, lc, x + 1, w, &wn);
            return wn != w + ix.sigma;
        }
        // num_incoming_to_target(x, w) == 2
        int indeg = 1;
        uint64_t e = x;
        while (++e <= ix.n) {
            e = succ_W2(ix, lc, e, w, &wn);
            if (wn != w + ix.sigma) break;
            ++indeg;
            if (indeg > 2) break;
        }
        return indeg == 2;
    }

    // --------------------------------------------------------------------------------
    // seeding (aligner_seeder_methods.cpp)
    // --------------------------------------------------------------------------------
    MGB_HD uint64_t qnode(int s, int i) const { return cx[s].qnodes ? cx[s].qnodes[i] : 0; }

    MGB_HD void push_seed(int s, uint32_t clip, uint32_t len, uint32_t off, uint32_t nn, uint64_t node0) {
        if (cx[s].n_seeds >= (int)caps.max_seeds) { overflow = true; return; }
        SeedRec r; r.clip = clip; r.len = len; r.offset = off; r.n_nodes = nn; r.node0 = node0;
        r.alive = 1; r.pad = 0;
        cx[s].seeds[cx[s].n_seeds++] = r;
    }

    // ExactSeeder::num_exact_matching (:49-65)
    MGB_HD uint32_t num_exact_matching(int s, int nk) {
        const int k = ix.k;
        // lane-parallel: a matched k-mer at i contributes min(k, distance to the previous match run end)
        // sequential restatement is cheap enough (nk <= L) and avoids subtle differences
        uint32_t nm = 0; int last_match_count = 0;
        for (int i = 0; i < nk; ++i) {
            if (qnode(s, i)) {
                int j = i + 1;
                while (j < nk && qnode(s, j)) ++j;
                nm += k + (j - i) - 1 - last_match_count;
                last_match_count = k;
                i = j - 1;
            } else if (last_match_count) {
                --last_match_count;
            }
        }
        return nm;
    }

    // --------------------------------------------------------------------------------
    // Seed complexity filter: is_low_complexity(window) = sdust(window, T = 20, W = 64) reports an interval
    // (aligner_seeder_methods.cpp:21-29). sdust is not vendored; restated from its definition (oracle:
    // is_low_complexity, parity unpinned): some interval of l + 1 <= 62 consecutive valid 3-mers has
    // 10 * sum_t c_t (c_t - 1) / 2 > 20 * l. Computed once per strand: lc_max[b] = the largest start a such
    // that (a .. b') qualifies for some b' <= b; a window of words [i, i + nt) is low-complexity iff
    // lc_max[i + nt - 1] >= i.
    // --------------------------------------------------------------------------------
    MGB_HD void build_lowcx(int s) {
        const uint8_t *cd = cx[s].codes;
        const int n_w = L - 2;
        if (n_w <= 0) return;
        uint8_t *wd = m.lc_word(); uint64_t *eq = m.lc_eq(); int32_t *mx = m.lc_max(s);
        for (int j = wlane(); j < n_w; j += kWarp) {
            const uint32_t a = cd[j], b = cd[j + 1], c = cd[j + 2];
            const bool ok = a >= 1 && a <= 4 && b >= 1 && b <= 4 && c >= 1 && c <= 4;
            wd[j] = ok ? (uint8_t)(((a - 1) << 4) | ((b - 1) << 2) | (c - 1)) : (uint8_t)0xFF;
        }
        wsync();
        // eq[a] bit d-1: 3-mer a + d equals 3-mer a (d = 1..61, inside the same run of valid 3-mers)
        for (int a = wlane(); a < n_w; a += kWarp) {
            uint64_t e = 0;
            const uint8_t w = wd[a];
            if (w != 0xFF)
                for (int d = 1; d <= 61 && a + d < n_w; ++d) {
                    const uint8_t x = wd[a + d];
                    if (x == 0xFF) break;
                    if (x == w) e |= 1ull << (d - 1);
                }
            eq[a] = e;
        }
        wsync();
        // largest qualifying start per end: growing the interval to the left by 3-mer a adds the number of its
        // occurrences in (a, b] to the score
        for (int base = 0; base < n_w; base += kWarp) {
            const int b = base + wlane();
            int best = -1;
            if (b < n_w && wd[b] != 0xFF) {
                int r = 0;
                for (int a = b - 1; a >= 0 && b - a <= 61; --a) {
                    if (wd[a] == 0xFF) break;
                    const int span = b - a;
                    const uint64_t mk = eq[a] & ((1ull << span) - 1ull);
                    r += popc32((uint32_t)mk) + popc32((uint32_t)(mk >> 32));
                    if (r * 10 > 20 * span) { best = a; break; }
                }
            }
            if (b < n_w) mx[b] = best;
        }
        wsync();
        // running maximum over the ends
        int carry = -1;
        for (int base = 0; base < n_w; base += kWarp) {
            const int b = base + wlane();
            int v = b < n_w ? (int)mx[b] : -1;
            v = imax(wscan_max(v), carry);
            if (b < n_w) mx[b] = v;
            carry = wbcast(v, kWarp - 1);
        }
        wsync();
    }
    // window = characters [i, i + len) of strand s (clamped to the read as substr() does); lane-divergent i allowed
    MGB_HD bool low_complexity(int s, int i, int len) const {
        if (len > L - i) len = L - i;
        const int nt = len - 2;
        if (nt < 2) return false;
        return (int)m.lc_max(s)[i + nt - 1] >= i;
    }

    // ExactSeeder::get_seeds (:67-93)
    MGB_HD void exact_seeds(int s, int nk) {
        const int k = ix.k;
        if (cx[s].num_matching < cfg.min_exact_match * L) return;
        if (cfg.max_seed_length < (uint32_t)k) return;
        for (int i = 0; i < nk; ++i) {
            uint64_t nd = qnode(s, i);
            if (nd && !(cfg.seed_complexity_filter && low_complexity(s, i, k))) push_seed(s, i, k, 0, 1, nd);
        }
    }

    // MEMSeeder::get_seeds (:360-424) with the UniMEM terminator (seeder.hpp:116-135)
    MGB_HD void mem_seeds(int s, int nk) {
        const int k = ix.k;
        if ((uint32_t)k >= cfg.max_seed_length) { exact_seeds(s, nk); return; }
        if (cx[s].num_matching < cfg.min_exact_match * L) return;
        int i = 0;
        while (i < nk) {
            if (!qnode(s, i)) { ++i; continue; }
            // [i, next): run of matched nodes ending at the first terminator (inclusive)
            int j = i;
            while (true) {
                uint64_t nd = qnode(s, j);
                bool term = j + 1 == nk || !qnode(s, j + 1)
                            || has_multiple_outgoing(nd) || !has_single_incoming(nd);
                ++j;
                if (term) break;
            }
            int mem_length = (j - i) + k - 1;
            if (mem_length >= (int)cfg.min_seed_length)
                push_seed(s, i, mem_length, 0, j - i, qnode(s, i));
            i = j;
        }
    }

    // first index >= pos (< n) whose bit equals `want`; n if none
    MGB_HD int mask_next(const uint32_t *mask, int n, int pos, bool want) const {
        while (pos < n) {
            uint32_t wd = mask[pos >> 5];
            if (!want) wd = ~wd;
            wd &= ~0u << (pos & 31);
            if (wd) { int r = (pos & ~31) + ffs32(wd) - 1; return r < n ? r : n; }
            pos = (pos & ~31) + 32;
        }
        return n;
    }

    // Second half of DBGSuccinct::call_nodes_with_suffix_matching_longest_prefix
    // (dbg_succinct.cpp:355-393, max_num_allowed_matches == SIZE_MAX): enumerate the nodes whose
    // k-mer suffix matches, given the BOSS range [first, lst] found by index_range. Appends one
    // seed per node at query position `pos`; returns their number (seeds beyond the capacity set
    // `overflow`).
    MGB_HD int suffix_enumerate(int s, int pos, int matched, uint64_t first, uint64_t lst, uint64_t *first_node) {
        LineCache lc;
        const uint64_t rank_first = rank_last(ix, lc, first);
        const uint64_t rank_lst = rank_last(ix, lc, lst);
        int count = 0;
        for (uint64_t r = rank_first; r <= rank_lst && !overflow; ++r) {
            LineCache l2;
            const uint64_t e = select_last(ix, l2, r);
            const uint2 ra = load_radj(ix, e);
            const uint32_t d = node_last_value(ix, e);
            uint64_t edge = ra.x;
            while (true) {
                if (in_graph(ix, edge)) {
                    if (count == 0) *first_node = edge;
                    ++count;
                    push_seed(s, pos, matched, ix.k - matched, 1, edge);
                    if (overflow) break;
                }
                if (!radj_multi(ix, ra.y)) break;
                if (++edge > ix.n) break;
                uint32_t w;
                edge = succ_W2(ix, l2, edge, d, &w);
                if (w != d + ix.sigma) break;
            }
        }
        return count;
    }

    // suffix_to_prefix (aligner_seeder_methods.cpp:95-139): the nodes whose k-mer starts with the `len0` characters
    // that select the BOSS range [rl0, ru0] (a set of nodes ending in them), found by extending the range one
    // character at a time, last pushed first. Counts the valid nodes; with `emit` each becomes a seed of the
    // reverse-complement node at query position `pos`. `stack`: scratch of 3 words per entry.
    MGB_HD int suffix_to_prefix(int s, int pos, uint64_t rl0, uint64_t ru0, int len0, bool emit,
                                uint32_t *stack, int stack_cap) {
        const int bk = (int)ix.k - 1;                         // boss.get_k()
        int count = 0;
        if (len0 == bk) {
            for (uint64_t e = rl0; e <= ru0 && !overflow; ++e)
                if (in_graph(ix, e)) { ++count; if (emit) push_seed(s, pos, len0, ix.k - len0, 1, canon_flip(e)); }
            return count;
        }
        int sp = 0;
        wsync();
        stack[0] = (uint32_t)rl0; stack[1] = (uint32_t)ru0; stack[2] = (uint32_t)len0; sp = 1;
        wsync();
        while (sp && !overflow) {
            --sp;
            const uint64_t rl = stack[3 * sp], ru = stack[3 * sp + 1];
            const int len = (int)stack[3 * sp + 2] + 1;
            wsync();
            for (uint32_t c = 1; c < ix.sigma && !overflow; ++c) {
                uint64_t nrl = rl, nru = ru;
                if (!tighten_range(ix, &nrl, &nru, c)) continue;
                if (len == bk) {
                    for (uint64_t e = nrl; e <= nru && !overflow; ++e)
                        if (in_graph(ix, e)) { ++count; if (emit) push_seed(s, pos, len0, ix.k - len0, 1, canon_flip(e)); }
                } else {
                    if (sp >= stack_cap) { overflow = true; break; }
                    stack[3 * sp] = (uint32_t)nrl; stack[3 * sp + 1] = (uint32_t)nru; stack[3 * sp + 2] = (uint32_t)len;
                    ++sp;
                }
            }
            wsync();
        }
        return count;
    }

    // Second half of SuffixSeeder::generate_seeds on a PRIMARY graph (CanonicalDBG): sub-k matches of the query
    // (:216-249) AND of its reverse complement (:251-314) compete per query position, so the seeds of a position are
    // only known after both passes. Pass A replays the reference's bookkeeping (min_seed_length per position, which
    // source holds the current seeds) while only counting nodes; pass B emits the survivors in position order with
    // the aggregation rules (:316-357). m.sfx_* hold the forward lookups; scratch lives in the (idle) DP cell arena.
    MGB_HD void build_seeds_subk_primary(int s, int n_base, const SeedRec *base_seeds, int n_pos) {
        const int k = ix.k;
        const int min_len = (int)cfg.min_seed_length;
        const int stack_cap = 4 * k + 8;
        if ((uint64_t)3 * n_pos + 3 * (uint64_t)stack_cap > 3ull * caps.max_cells) { overflow = true; return; }
        uint32_t *rc_first = (uint32_t*)m.cells(), *rc_last = rc_first + n_pos;
        uint32_t *meta = rc_last + n_pos;                         // fwd length | rc length << 8
        uint32_t *stack = meta + n_pos;
        for (int i = wlane(); i < n_pos; i += kWarp) meta[i] = 0;
        wsync();
        // ---- pass A, forward matches (:216-249) ----
        {
            int b_next = 0;
            const int last_full_id = L >= k ? L - k + 1 : n_pos;
            int lf_count = 0; uint64_t lf_node = 0;
            for (int i = 0; i < n_pos; ++i) {
                int n_here = 0; uint64_t node_here = 0;
                if (b_next < n_base && (int)base_seeds[b_next].clip == i) {
                    node_here = base_seeds[b_next].node0; ++b_next; n_here = 1;
                } else if (m.sfx_min()[i] != k) {
                    const int min_here = m.sfx_min()[i];
                    const int matched = m.sfx_len()[i];
                    if (matched >= min_here && matched > 0
                            && !(cfg.seed_complexity_filter && low_complexity(s, i, min_here))) {
                        uint64_t first_node = 0;
                        const int keep = cx[s].n_seeds;
                        int cnt = suffix_enumerate(s, i, matched, m.sfx_first()[i], m.sfx_last()[i], &first_node);
                        if (overflow) return;
                        cx[s].n_seeds = keep;                     // counted only
                        const bool skip = i >= last_full_id && cnt == 1 && last_full_id >= 1
                                    && m.sfx_min()[last_full_id - 1] == k && lf_count == 1 && first_node == lf_node;
                        if (cnt != 0 && !skip) {
                            wsync();
                            m.sfx_min()[i] = (uint8_t)matched;
                            meta[i] = (uint32_t)matched;
                            int sl = matched;
                            for (int j = i + 1; j < n_pos && sl > (int)m.sfx_min()[j]; ++j) m.sfx_min()[j] = (uint8_t)(sl--);
                            wsync();
                            n_here = cnt; node_here = first_node;
                        }
                    }
                }
                if (i == last_full_id - 1) { lf_count = n_here; lf_node = n_here ? node_here : 0; }
            }
        }
        // ---- pass A, matches of the reverse complement (:251-314) ----
        const uint8_t *rc_codes = cx[1 - s].codes;
        for (int i = 0; i + min_len <= L && !overflow; ++i) {
            int max_len = imin(imin((int)(cfg.max_seed_length < 0x7fffffffu ? cfg.max_seed_length : 0x7fffffffu), k - 1), L - i);
            int j_min = L - i - max_len;
            const int j_max = L - i - min_len;
            while (j_min <= j_max && (int)m.sfx_min()[j_min] > max_len) { ++j_min; --max_len; }
            if (j_min > j_max) continue;
            uint64_t first = 0, lst = 0; int matched = 0;
            boss_index_range(ix, rc_codes + i, max_len, &first, &lst, &matched, min_len);
            const int seed_length = matched;
            if (seed_length < min_len) continue;
            const int j = L - i - seed_length;
            if (seed_length < (int)m.sfx_min()[j]
                    || (cfg.seed_complexity_filter && low_complexity(s, j, seed_length)))
                continue;
            LineCache lc;
            const uint64_t lo = pred_last(ix, lc, first - 1) + 1;
            const int cnt = suffix_to_prefix(s, j, lo, lst, seed_length, false, stack, stack_cap);
            if (overflow) return;
            if (!cnt) continue;
            wsync();
            // append_suffix_seed (:195-213): longer than what the position holds -> replaces it
            m.sfx_min()[j] = (uint8_t)seed_length;
            rc_first[j] = (uint32_t)lo; rc_last[j] = (uint32_t)lst;
            meta[j] = (meta[j] & 0xffu) | ((uint32_t)seed_length << 8);
            int sl = seed_length;
            for (int jj = j + 1; jj < n_pos && sl > (int)m.sfx_min()[jj]; ++jj) m.sfx_min()[jj] = (uint8_t)(sl--);
            wsync();
        }
        if (overflow) return;
        // ---- pass B: aggregation in query order (:316-357) ----
        int b_next = 0;
        uint32_t nm = 0; int last_end = 0;
        for (int i = 0; i < n_pos; ++i) {
            const int pos_first = cx[s].n_seeds;
            if (b_next < n_base && (int)base_seeds[b_next].clip == i) {
                if (cx[s].n_seeds >= (int)caps.max_seeds - n_base) { overflow = true; return; }
                cx[s].seeds[cx[s].n_seeds++] = base_seeds[b_next++];
            } else {
                const int cur = m.sfx_min()[i];
                const int fl = (int)(meta[i] & 0xffu), rl_ = (int)((meta[i] >> 8) & 0xffu);
                uint64_t cnt = 0;
                if (fl && fl == cur) {
                    uint64_t fn = 0;
                    cnt += (uint64_t)suffix_enumerate(s, i, fl, m.sfx_first()[i], m.sfx_last()[i], &fn);
                }
                if (!overflow && rl_ && rl_ == cur)
                    cnt += (uint64_t)suffix_to_prefix(s, i, rc_first[i], rc_last[i], rl_, true, stack, stack_cap);
                if (overflow) return;
                if (cx[s].n_seeds > (int)caps.max_seeds - n_base) { overflow = true; return; }
                if (cnt > cfg.max_num_seeds_per_locus) cx[s].n_seeds = pos_first;
            }
            if (cx[s].n_seeds > pos_first) {
                const SeedRec &bk = cx[s].seeds[cx[s].n_seeds - 1];
                int begin = bk.clip, end = begin + (int)bk.len;
                if (begin < last_end) nm += end - begin - (last_end - begin);
                else nm += end - begin;
                last_end = end;
            }
        }
        cx[s].num_matching = nm;
    }

    // SuffixSeeder<UniMEMSeeder>::generate_seeds (:153-358), non-canonical part
    MGB_HD void build_seeds(int s) {
        const int k = ix.k;
        const int nk = L >= k ? L - k + 1 : 0;
        cx[s].n_seeds = 0;
        // Exact seeder with staged query (the BASELINE configs[1] path): one k-mer seed per matched
        // k-mer, kept as a bit mask on chip instead of a seed array
        if ((int)cfg.min_seed_length >= k && (uint32_t)k >= cfg.max_seed_length && sm.lq() && L + 1 <= sm.lq()) {
            uint32_t *mask = cx[s].mask;
            const uint64_t *qn = cx[s].qnodes;
            const int nw = (nk + 31) / 32;
            int total = 0;
            for (int w = 0; w < nw; ++w) {
                unsigned word = 0;
                for (int b = 0; b < 32; b += kWarp) {        // one pass on the device
                    int i = 32 * w + b + wlane();
                    word |= wballot(i < nk && qn[i] != 0) << b;
                }
                mask[w] = word;
                total += popc32(word);
            }
            mask[nw] = 0;
            wsync();
            // ExactSeeder::num_exact_matching (:49-65) over the runs of set bits
            uint32_t nm = 0; int pos = 0, prev_end = -1;
            while (pos < nk) {
                int i = mask_next(mask, nk, pos, true);
                if (i >= nk) break;
                int j = mask_next(mask, nk, i, false);
                int lmc = prev_end < 0 ? 0 : imax(k - (i - prev_end), 0);
                nm += k + (j - i) - 1 - lmc;
                prev_end = j; pos = j;
            }
            cx[s].num_matching = nm;
            cx[s].implicit_seeds = 1;
            if (cfg.seed_complexity_filter) {            // low-complexity k-mers give no seed (:84)
                total = 0;
                for (int w = 0; w < nw; ++w) {
                    unsigned drop = 0;
                    for (int b = 0; b < 32; b += kWarp) {
                        int i = 32 * w + b + wlane();
                        drop |= wballot(i < nk && low_complexity(s, i, k)) << b;
                    }
                    mask[w] &= ~drop;
                    total += popc32(mask[w]);
                }
                wsync();
            }
            // ExactSeeder::get_seeds (:67-93)
            if (L < (int)cfg.min_seed_length || (double)nm < cfg.min_exact_match * L || cfg.max_seed_length < (uint32_t)k)
                total = 0;
            cx[s].n_seeds = total;
            return;
        }
        cx[s].num_matching = num_exact_matching(s, nk);
        if (L < (int)cfg.min_seed_length) return;
        const bool mem_only = (int)cfg.min_seed_length >= k;

        // base (MEM) seeds first; they are merged with the sub-k seeds in query order below
        const int n_pos = L - (int)cfg.min_seed_length + 1;
        if (!mem_only) for (int i = wlane(); i < n_pos; i += kWarp) m.sfx_min()[i] = (uint8_t)cfg.min_seed_length;
        wsync();
        mem_seeds(s, nk);
        if (mem_only) return;
        const int n_base = cx[s].n_seeds;
        if (overflow) return;
        if (2 * n_base > (int)caps.max_seeds) { overflow = true; return; }
        SeedRec *base_seeds = cx[s].seeds + caps.max_seeds - n_base;   // scratch at the end of the array
        wsync();
        for (int i = n_base - 1; i >= 0; --i) base_seeds[i] = cx[s].seeds[i];
        for (int b = 0; b < n_base; ++b) {
            SeedRec sd = base_seeds[b];
            for (int j = 0; j < (int)sd.n_nodes; ++j) m.sfx_min()[sd.clip + j] = (uint8_t)k;
            if ((int)(sd.clip + sd.n_nodes) < n_pos) m.sfx_min()[sd.clip + sd.n_nodes] = (uint8_t)k;
        }
        wsync();
        cx[s].n_seeds = 0;

        // BOSS::index_range (boss.hpp:720-764) of every position not covered by a base seed, one
        // position per lane group (the searches are independent; only their use below is ordered)
        const uint32_t msl_u = cfg.max_seed_length < (uint32_t)(k - 1) ? cfg.max_seed_length : (uint32_t)(k - 1);
        {
            const int groups = kWarp / kGroup;
            const int g = wlane() / kGroup;
            for (int base = 0; base < n_pos; base += groups) {
                const int i = base + g;
                if (i < n_pos && m.sfx_min()[i] != k && cx[s].sub_len && cx[s].sub_len[i] != 0xFF) {
                    if (glane() == 0) {                   // looked up by k_subk
                        m.sfx_first()[i] = cx[s].sub_first[i]; m.sfx_last()[i] = cx[s].sub_last[i];
                        m.sfx_len()[i] = cx[s].sub_len[i];
                    }
                } else if (i < n_pos && m.sfx_min()[i] != k) {
                    const int len = imin((int)msl_u, L - i);
                    uint64_t first = 0, lst = 0; int matched = 0;
                    bool ok = len >= (int)cfg.min_seed_length;
                    const uint8_t *cd = cx[s].codes + i;
                    for (int t = 0; t < len && ok; ++t) ok = cd[t] < ix.sigma;
                    // matches shorter than min_seed_length are never used below (sfx_min[i] >= min_seed_length)
                    if (ok) boss_index_range(ix, cd, imin(len, k - 1), &first, &lst, &matched, (int)cfg.min_seed_length);
                    if (glane() == 0) {
                        m.sfx_first()[i] = (uint32_t)first; m.sfx_last()[i] = (uint32_t)lst; m.sfx_len()[i] = (uint8_t)matched;
                    }
                }
            }
        }
        wsync();

        if (MGB_CANONICAL(cfg) && MGB_PRIMARY(ix)) { build_seeds_subk_primary(s, n_base, base_seeds, n_pos); return; }

        int b_next = 0;
        const int last_full_id = L >= k ? L - k + 1 : n_pos;
        // state of suffix_seeds[last_full_id - 1] for the skip rule (:240-244)
        int lf_count = 0; uint64_t lf_node = 0;
        uint32_t nm = 0; int last_end = 0;
        for (int i = 0; i < n_pos; ++i) {
            const int pos_first = cx[s].n_seeds;
            int n_here = 0;
            if (b_next < n_base && (int)base_seeds[b_next].clip == i) {
                // a full seed at this position (offset 0): emitted as is (:334-337)
                if (cx[s].n_seeds >= (int)caps.max_seeds - n_base) { overflow = true; return; }
                cx[s].seeds[cx[s].n_seeds++] = base_seeds[b_next++];
                n_here = 1;
            } else if (m.sfx_min()[i] != k) {
                const int min_here = m.sfx_min()[i];
                const int matched = m.sfx_len()[i];
                // call_nodes_with_suffix_matching_longest_prefix (:231-238): nothing below min_match_length;
                // a low-complexity window of the current minimum length is skipped altogether (:226-229)
                if (matched >= min_here && matched > 0
                        && !(cfg.seed_complexity_filter && low_complexity(s, i, min_here))) {
                    uint64_t first_node = 0;
                    // capacity: the scratch copy of the base seeds lives at the end of the array
                    int cnt = suffix_enumerate(s, i, matched, m.sfx_first()[i], m.sfx_last()[i], &first_node);
                    if (overflow) return;
                    if (cx[s].n_seeds > (int)caps.max_seeds - n_base) { overflow = true; return; }
                    const bool skip = i >= last_full_id && cnt == 1 && last_full_id >= 1
                                && m.sfx_min()[last_full_id - 1] == k && lf_count == 1 && first_node == lf_node;
                    if (cnt == 0 || skip) {
                        cx[s].n_seeds = pos_first;
                    } else {
                        // append_suffix_seed (:195-213) for every alternative node
                        m.sfx_min()[i] = (uint8_t)matched;
                        int sl = matched;
                        for (int j = i + 1; j < n_pos && sl > (int)m.sfx_min()[j]; ++j)
                            m.sfx_min()[j] = (uint8_t)(sl--);
                        n_here = cnt;
                        // a locus with too many alternatives is dropped at aggregation (:340-345)
                        if ((uint64_t)cnt > cfg.max_num_seeds_per_locus) cx[s].n_seeds = pos_first;
                    }
                }
            }
            if (i == last_full_id - 1) {
                lf_count = n_here;
                lf_node = (n_here && cx[s].n_seeds > pos_first) ? cx[s].seeds[pos_first].node0 : 0;
            }
            // aggregation (:316-357): num_matching counts the span of the last seed emitted here
            if (cx[s].n_seeds > pos_first) {
                const SeedRec &bk = cx[s].seeds[cx[s].n_seeds - 1];
                int begin = bk.clip, end = begin + (int)bk.len;
                if (begin < last_end) nm += end - begin - (last_end - begin);
                else nm += end - begin;
                last_end = end;
            }
        }
        cx[s].num_matching = nm;
    }

    // --------------------------------------------------------------------------------
    // convergence filter (SeedFilteringExtender, extender.cpp:66-207)
    // Open-addressing table keyed by node id; the per-node score vector lives in a
    // segment of the conv cell arena, indexed by absolute query position.
    // --------------------------------------------------------------------------------
    // first probe of `key`; mask = hash_size - 1
    MGB_HD static uint32_t hash_node(uint64_t key, uint32_t mask) {
        uint32_t h = (uint32_t)key * 0x9E3779B1u ^ (uint32_t)(key >> 32) * 0x85EBCA77u;
        h ^= h >> 15;
        return h & mask;
    }
    MGB_HD void conv_clear(int e) {
        StrandCtx &t = cx[e];
        t.explored_prev += t.conv_n;
        t.conv_n = 0; t.conv_cells_used = 0;
        ++t.conv_epoch;
    }
    // returns the slot index or -1; *out = slot contents. No collectives: may be called with
    // lane-divergent keys.
    // *free_at (optional) = the free slot the probe sequence ended on when the key is absent (-1: none)
    MGB_HD int conv_find(const ConvSlot *slots, uint32_t epoch, uint64_t key, ConvSlot *out,
                         bool use_prefetch = false, int *free_at = nullptr) {
        uint32_t h = hash_node(key, caps.hash_size - 1);
        if (free_at) *free_at = -1;
        for (uint32_t probe = 0; probe < caps.hash_size; ++probe) {
            uint32_t p = (h + probe) & (caps.hash_size - 1);
            ConvSlot sl = (use_prefetch && probe == 0 && key == pf_key && p == pf_slot_idx) ? pf_slot : slots[p];
            if (sl.epoch != epoch) { if (free_at) *free_at = (int)p; return -1; }
            if (sl.key == key) { *out = sl; return (int)p; }
        }
        return -1;
    }
    // new entry covering [start, start + size) in the free slot conv_find ended on for this key, cells uninitialised.
    // conv_find ends on no free slot only when every slot is taken, which the load test below rejects first
    MGB_HD bool conv_insert(int e, uint64_t key, int start, int size, ConvSlot *out, int free_at) {
        StrandCtx &t = cx[e];
        const uint32_t n_entries = t.conv_n, cells_used = t.conv_cells_used;
        if (n_entries >= caps.max_conv_entries || 2 * (n_entries + 1) > caps.hash_size || free_at < 0) {
            overflow = true; return false;
        }
        int seg_start = imax(0, start - 8);
        int seg_cap = imin(L + 1, start + size + 8) - seg_start;
        if (cells_used + seg_cap > caps.max_conv_cells) { overflow = true; return false; }
        ConvSlot sl; sl.key = key; sl.epoch = t.conv_epoch; sl.start = start; sl.size = size;
        sl.seg_start = seg_start; sl.seg_cap = seg_cap; sl.seg_off = cells_used;
        t.conv_cells_used = cells_used + seg_cap;
        t.conv_n = n_entries + 1;
        t.conv_slots[free_at] = sl;
        *out = sl;
        return true;
    }
    // make the stored vector cover [new_start, new_end) (superset of the current range),
    // new cells = ninf. Mirrors vec.insert(begin, n, ninf) / resize(n, ninf).
    MGB_HD bool conv_grow(int e, int slot, ConvSlot *en, int new_start, int new_end) {
        StrandCtx &t = cx[e];
        score_t *cells = t.conv_cells;
        int old_start = en->start, old_end = en->start + en->size;
        if (new_start < en->seg_start || new_end > en->seg_start + en->seg_cap) {
            const uint32_t cells_used = t.conv_cells_used;
            int seg_start = imax(0, new_start - 16);
            int seg_cap = imin(L + 1, new_end + 16) - seg_start;
            if (cells_used + seg_cap > caps.max_conv_cells) { overflow = true; return false; }
            MGB_EMU_HIT(EMU_CONV_MOVE);
            score_t *src = cells + en->seg_off, *dst = cells + cells_used;
            wsync();
            for (int p = old_start + wlane(); p < old_end; p += kWarp)
                dst[p - seg_start] = src[p - en->seg_start];
            en->seg_off = cells_used; en->seg_start = seg_start; en->seg_cap = seg_cap;
            t.conv_cells_used = cells_used + seg_cap;
        }
        score_t *c = cells + en->seg_off;
        for (int p = new_start + wlane(); p < old_start; p += kWarp) c[p - en->seg_start] = kNinf;
        for (int p = old_end + wlane(); p < new_end; p += kWarp) c[p - en->seg_start] = kNinf;
        en->start = new_start; en->size = new_end - new_start;
        t.conv_slots[slot] = *en;
        wsync();
        return true;
    }

    // The entry of `key`, made to cover [start, start + size) (extender.cpp:113-141, 165-194): a new entry (cells
    // uninitialised) or the stored one, grown with ninf cells. Returns what was found: CONV_NEW, CONV_DISJOINT (the range
    // lies before or after the stored one), CONV_OVERLAP, or CONV_FAILED (table or cells full: overflow is set).
    enum : int { CONV_FAILED, CONV_NEW, CONV_DISJOINT, CONV_OVERLAP };
    MGB_HD int conv_entry(int e, uint64_t key, int start, int size, bool use_prefetch, ConvSlot *en) {
        StrandCtx &t = cx[e];
        int free_at;
        const int slot = conv_find(t.conv_slots, t.conv_epoch, key, en, use_prefetch, &free_at);
        if (slot < 0) return conv_insert(e, key, start, size, en, free_at) ? CONV_NEW : CONV_FAILED;
        const bool disjoint = start + size <= en->start || start >= en->start + en->size;
        const int ns = imin(start, en->start), ne = imax(start + size, en->start + en->size);
        if ((ns != en->start || ne != en->start + en->size) && !conv_grow(e, slot, en, ns, ne)) return CONV_FAILED;
        return disjoint ? CONV_DISJOINT : CONV_OVERLAP;
    }

    // extender.cpp:100-156; sv = S[s_first .. s_first + size) of the column being committed
    MGB_HD score_t update_seed_filter(int e, uint64_t node, int query_start, const score_t *sv, int size) {
        score_t mx = kNinf;
        for (int j = wlane(); j < size; j += kWarp) mx = imax(mx, sv[j]);
        mx = wreduce_max(mx);
        if (node == 0) return mx;
        StrandCtx &t = cx[e];
        ConvSlot en;
        const int got = conv_entry(e, node + ((!MGB_CANONICAL(cfg) && t.rc) ? ix.n : 0), query_start, size, false, &en);
        if (got == CONV_FAILED) return kNinf;
        score_t *v = t.conv_cells + en.seg_off + (query_start - en.seg_start);
        if (got != CONV_OVERLAP) {                       // new, or before / after the stored range: stored as is
            for (int j = wlane(); j < size; j += kWarp) v[j] = sv[j];
            wsync();
            return mx;
        }
        score_t max_changed = kNinf;
        for (int j = wlane(); j < size; j += kWarp) {
            score_t sj = sv[j];
            score_t vj = v[j];
            if ((double)sj > (double)vj * cfg.rel_score_cutoff) {
                vj = imax(vj, sj);
                v[j] = vj;
                max_changed = imax(max_changed, vj);
            }
        }
        max_changed = wreduce_max(max_changed);
        wsync();
        return max_changed;
    }

    // The cells [s_first, size) of a register-path column (lane l holds cell l * kCPL + c in S[c]) written into a
    // convergence entry whose cells v0 points to, indexed by cell: stored as they are (a new entry, or a range before or
    // after the stored one; returns their maximum), or merged with the stored cells (:143-153; returns the largest cell
    // that changed, ninf if none).
    MGB_HD static score_t conv_store_regs(score_t *v0, const score_t (&S)[kCPL], int s_first, int size) {
        const int j0 = wlane() * kCPL;
        score_t mx = kNinf;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const int j = j0 + c;
            if (j >= s_first && j < size) { v0[j] = S[c]; mx = imax(mx, S[c]); }
        }
        mx = wreduce_max(mx);
        wsync();
        return mx;
    }
    MGB_HD static score_t conv_merge_regs(score_t *v0, const score_t (&S)[kCPL], int s_first, int size,
                                          double rel_score_cutoff) {
        const int j0 = wlane() * kCPL;
        score_t max_changed = kNinf;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const int j = j0 + c;
            if (j >= s_first && j < size) {
                score_t vj = v0[j];
                if ((double)S[c] > (double)vj * rel_score_cutoff) {
                    vj = imax(vj, S[c]);
                    v0[j] = vj;
                    max_changed = imax(max_changed, vj);
                }
            }
        }
        max_changed = wreduce_max(max_changed);
        wsync();
        return max_changed;
    }

    // update_seed_filter (extender.cpp:100-156) for a column of the register path: the passed range is cells
    // [s_first, size)
    MGB_HD score_t update_seed_filter_regs(int e, uint64_t node, int query_start, const score_t (&S)[kCPL],
                                           int s_first, int size) {
        if (node == 0) {
            const int j0 = wlane() * kCPL;
            score_t mx = kNinf;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
            for (int c = 0; c < kCPL; ++c)
                if (j0 + c >= s_first && j0 + c < size) mx = imax(mx, S[c]);
            return wreduce_max(mx);
        }
        StrandCtx &t = cx[e];
        ConvSlot en;
        const int got = conv_entry(e, node + ((!MGB_CANONICAL(cfg) && t.rc) ? ix.n : 0), query_start, size - s_first,
                                   true, &en);
        if (got == CONV_FAILED) return kNinf;
        score_t *v0 = t.conv_cells + en.seg_off + (query_start - s_first - en.seg_start);   // indexed by cell
        return got == CONV_OVERLAP ? conv_merge_regs(v0, S, s_first, size, cfg.rel_score_cutoff)
                                   : conv_store_regs(v0, S, s_first, size);
    }

    // extender.cpp:158-207 (every cell of [query_start, query_end) ends up at -ninf)
    MGB_HD void filter_nodes(int e, uint64_t node, int query_start, int query_end) {
        const score_t mscore = -kNinf;
        StrandCtx &t = cx[e];
        ConvSlot en;
        if (conv_entry(e, node, query_start, query_end - query_start, false, &en) == CONV_FAILED) return;
        score_t *c = t.conv_cells + en.seg_off;
        for (int p = query_start + wlane(); p < query_end; p += kWarp) c[p - en.seg_start] = mscore;
        wsync();
    }

    // extender.cpp:66-88 (lane-divergent arguments allowed)
    MGB_HD bool check_seed_vals(const ConvSlot *slots, const score_t *cells, uint32_t epoch, bool rc,
                                uint64_t last_node, int pos, score_t score) {
        uint64_t key = last_node + (rc ? ix.n : 0);
        ConvSlot en;
        if (conv_find(slots, epoch, key, &en) < 0) return true;
        if (pos < en.start || pos - en.start >= en.size) return true;
        return cells[en.seg_off + (pos - en.seg_start)] < score;
    }

    // --------------------------------------------------------------------------------
    // best-first queue (std::priority_queue<TableIt>, extender.cpp:477-504); lives in shared
    // memory and migrates to the arena when it outgrows it
    // --------------------------------------------------------------------------------
    HeapItem *hp, *np;           // heap / next_nodes storage
    int hp_cap, np_cap;

    MGB_HD bool heap_less(const HeapItem &a, const HeapItem &b) const {   // std::less<TableIt>
        if (a.score != b.score) return a.score < b.score;
        if (a.neg_off_diag != b.neg_off_diag) return a.neg_off_diag < b.neg_off_diag;
        if (a.idx != b.idx) return a.idx < b.idx;
        return a.max_score < b.max_score;
    }
    MGB_HD void heap_push(int &n, HeapItem it) {
        if (n >= hp_cap) {
            if (hp == m.heap()) { overflow = true; return; }
            MGB_EMU_HIT(EMU_QUEUE_MIGRATE);
            for (int t = wlane(); t < n; t += kWarp) m.heap()[t] = hp[t];
            wsync();
            hp = m.heap(); hp_cap = caps.max_cols;
        }
        int i = n++;
        while (i > 0) {
            int p = (i - 1) >> 1;
            HeapItem pi = hp[p];
            if (!heap_less(pi, it)) break;
            hp[i] = pi;
            i = p;
        }
        hp[i] = it;
    }
    MGB_HD HeapItem heap_pop(int &n) {
        HeapItem top = hp[0];
        HeapItem last = hp[--n];
        int i = 0;
        while (true) {
            int l = 2 * i + 1, r = l + 1;
            if (l >= n) break;
            int c = l;
            if (r < n && heap_less(hp[l], hp[r])) c = r;
            HeapItem ci = hp[c];
            if (!heap_less(last, ci)) break;
            hp[i] = ci;
            i = c;
        }
        if (n > 0) hp[i] = last;
        return top;
    }
    MGB_HD void nn_push(int &n, HeapItem it) {
        if (n >= np_cap) {
            if (np == m.next_nodes()) { overflow = true; return; }
            MGB_EMU_HIT(EMU_NN_MIGRATE);
            for (int t = wlane(); t < n; t += kWarp) m.next_nodes()[t] = np[t];
            wsync();
            np = m.next_nodes(); np_cap = caps.max_cols;
        }
        np[n++] = it;
    }

    // --------------------------------------------------------------------------------
    // DP columns
    // --------------------------------------------------------------------------------
    // std::vector<score_t> capacity after DPTColumn::create(size0) + p push_backs + reserve(size + 5)
    MGB_HD static uint32_t vec_capacity(int size0, int size_final) {
        uint32_t cap = size0 + 5;
        if (size_final == size0) return cap;
        while ((uint32_t)size_final > cap) cap *= 2;
        if ((uint32_t)size_final + 5 > cap) cap = size_final + 5;
        return cap;
    }
    // std::vector<DPTColumn>::capacity() once the table holds n columns (table_cap: the capacity before)
    MGB_HD static uint32_t table_capacity(uint32_t table_cap, uint32_t n) {
        return n > table_cap ? (table_cap ? 2 * table_cap : 1) : table_cap;
    }
    // what a column adds to table_size_bytes (extender.cpp:466-469, 705-711): the DPTColumns the table grew by from
    // cap_before to cap, and the capacity of the column's S, E and F
    MGB_HD static uint64_t column_bytes(uint32_t cap_before, uint32_t cap, int size0, int size) {
        return 136ull * (cap - cap_before) + 3ull * vec_capacity(size0, size) * 4;
    }
    // the end of a child column's step (:681-719): false when the column is dropped (pop(table.size() - 1)); otherwise
    // its bytes are counted, and the x-drop cutoff and best_score follow its maximum
    MGB_HD static bool accept_column(bool in_seed, score_t max_val, bool has_extension, uint32_t cap_before, uint32_t cap,
                                     int size0, int size, score_t xdrop, score_t &cutoff, score_t &best_score,
                                     uint64_t &table_size_bytes) {
        if (!in_seed && (max_val < cutoff || !has_extension)) return false;
        table_size_bytes += column_bytes(cap_before, cap, size0, size);
        if ((int64_t)max_val - cutoff > xdrop) cutoff = max_val - xdrop;
        best_score = imax(best_score, max_val);
        return true;
    }
    MGB_HD static ColMeta make_col(uint64_t node, uint32_t parent, uint8_t c, int offset, int max_pos, int trim,
                                   score_t score, uint8_t fmt, int size, uint32_t cells_off) {
        ColMeta col;
        col.node = node; col.parent = parent; col.c = c;
        col.offset = offset; col.max_pos = max_pos; col.trim = trim; col.score = score;
        col.is_tip = 0; col.started = 0; col.fmt = fmt; col.pad0 = col.pad1 = 0;
        col.size = size; col.cells_off = cells_off;
        return col;
    }
    // global_xdrop (:525-546), before a column is expanded whose best cell (par_max) is below best_score: the budget
    // that ends the extension, the table's columns per window character or its bytes; BUDGET_NONE if neither
    enum : int { BUDGET_NONE, BUDGET_NODES, BUDGET_RAM };
    MGB_HD static int budget_stop(const DevConfig &cfg, score_t par_max, score_t best_score, uint32_t n_cols, int wlen,
                                  uint64_t table_size_bytes) {
        if (par_max >= best_score) return BUDGET_NONE;
        if ((double)n_cols / wlen >= cfg.max_nodes_per_seq_char) return BUDGET_NODES;
        if ((double)table_size_bytes / 1000000 > cfg.max_ram_per_alignment) return BUDGET_RAM;
        return BUDGET_NONE;
    }

    // Working buffer of the column being computed: S | E | F with stride `cap`
    struct Scratch { score_t *S, *E, *F; int cap; bool on_chip; };

    MGB_HD Scratch scratch_smem(int b) const {
        Scratch r; r.S = sm.buf(b); r.E = r.S + sm.bmax(); r.F = r.E + sm.bmax(); r.cap = sm.bmax(); r.on_chip = true;
        return r;
    }
    // arena scratch above the commit area of the column in flight; `cells` must be the largest
    // size the column can reach (so that an arena scratch never has to move)
    MGB_HD bool scratch_arena(int cells, Scratch *r) {
        uint64_t need = (uint64_t)cells_used + 3ull * (cells + 8) /*commit*/ + 3ull * (cells + 8) /*scratch*/;
        if (need > 3ull * caps.max_cells) { overflow = true; return false; }
        r->cap = cells + 8;
        r->S = m.cells() + cells_used + 3ull * (cells + 8);
        r->E = r->S + r->cap; r->F = r->E + r->cap; r->on_chip = false;
        return true;
    }

    // extend_ins_end (extender.cpp:293-328); returns the new size. `sc` may migrate to the arena.
    MGB_HD int extend_ins_end(Scratch &sc, int size, int max_size, score_t cutoff) {
        if (size >= max_size) return size;
        score_t ins = imax(wadd(sc.S[size - 1], cfg.gap_open), wadd(sc.E[size - 1], cfg.gap_ext));
        if (ins < cutoff) return size;
        const uint32_t diff = (uint32_t)ins - (uint32_t)cutoff;              // ins >= cutoff
        const uint32_t extra = cfg.gap_ext < 0 ? diff / (uint32_t)(-cfg.gap_ext) : 0x7fffffffu;
        const uint32_t room = (uint32_t)(max_size - size - 1);
        int cnt = 1 + (int)(extra < room ? extra : room);
        if (size + cnt + 5 > sc.cap) {
            Scratch big;                               // only an on-chip scratch can be too small
            if (!sc.on_chip || !scratch_arena(max_size, &big)) { overflow = true; return size; }
            MGB_EMU_HIT(EMU_COLUMN_MIGRATE);
            for (int t = wlane(); t < size + 5 && t < sc.cap; t += kWarp) {
                big.S[t] = sc.S[t]; big.E[t] = sc.E[t]; big.F[t] = sc.F[t];
            }
            wsync();
            sc = big;
        }
        for (int t = wlane(); t < cnt + 5; t += kWarp) {
            score_t v = t < cnt ? wadd(ins, t * cfg.gap_ext) : kNinf;
            sc.S[size + t] = v; sc.E[size + t] = v; sc.F[size + t] = kNinf;
        }
        wsync();
        return size + cnt;
    }

    // update_column (extender.cpp:209-290), restated as a max-plus scan (see DESIGN.md).
    // pS / pF: parent's S / F shifted so that index j is the same absolute row as child row j.
    MGB_HD void update_column(int s, const score_t *pS, const score_t *pF, Scratch &sc, int size0,
                              int n, int prof_base, score_t cutoff, int code, score_t add, bool use_del) {
        const int n4 = (n + 3) & ~3;
        const score_t go = cfg.gap_open, ge = cfg.gap_ext;
        int carry = wadd(kNinf, ge);                       // a[-1] = E[0] + ge, E[0] = ninf
        for (int base = 0; base < n4; base += kWarp) {
            int j = base + wlane();
            bool act = j < n4;
            score_t mval = kNinf, del = kNinf;
            if (act) {
                score_t match = kNinf;
                if (j) match = wadd(wadd(pS[j - 1], prof_score(s, prof_base + j, code)), add);
                if (use_del) del = wadd(imax(wadd(pS[j], go), wadd(pF[j], ge)), add);
                mval = imax(match, del);
            }
            // a[j] = m[j] + go - j*ge ; E[j+1] = prefmax(a)[j] + j*ge
            int a = act ? wsub(wadd(mval, go), j * ge) : INT32_MIN;
            int incl = wscan_max(a);
            incl = imax(incl, carry);
            int excl = wshfl_up1(incl, carry);         // prefix max over i < j (incl. a[-1])
            if (act) {
                score_t e_j = j ? wadd(excl, (j - 1) * ge) : kNinf;    // E[j]
                score_t sv = imax(mval, e_j);
                sc.F[j] = del;
                sc.E[j + 1] = wadd(incl, j * ge);                      // E[j + 1]
                sc.S[j] = sv > cutoff - 1 ? sv : kNinf;
            }
            carry = wbcast(incl, kWarp - 1);
        }
        wsync();
        if (size0 > imax(1, n)) {                      // scalar tail (:284-289)
            int j = size0 - 1;
            score_t t = imax(wadd(wadd(pS[j - 1], add), prof_score(s, prof_base + j, code)), sc.E[j]);
            if (t >= cutoff) sc.S[j] = t;
            wsync();
        }
    }

    // copy a finished column (incl. 5 padding cells) into the DP table; returns cells_off
    MGB_HD uint32_t commit_column(const Scratch &sc, int size) {
        const int cap = size + 5;
        const uint32_t off = cells_used;
        score_t *dst = m.cells() + off;
        for (int t = wlane(); t < cap; t += kWarp) {
            dst[t] = sc.S[t]; dst[cap + t] = sc.E[t]; dst[2 * cap + t] = sc.F[t];
        }
        cells_used += 3 * cap;
        return off;
    }

    // --------------------------------------------------------------------------------
    // Register path: a DP column of up to 32 cells (incl. its 5 padding cells) held in registers, lane l owning
    // cells [l * kCPL, (l + 1) * kCPL). Fuses DPTColumn::create, update_column, extend_ins_end and the flag bytes
    // of the compact table format. In the host emulation the single lane owns all 32 cells, so the same code
    // is exercised on machines without a GPU.
    // --------------------------------------------------------------------------------
    struct RegCol { score_t S[kCPL], E[kCPL], F[kCPL]; uint8_t fl[kCPL]; };

    // value of cell `idx` of a lane-distributed array, broadcast to the warp
    MGB_HD static score_t cell_bcast(const score_t (&v)[kCPL], int idx) {
        score_t x = v[0];
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 1; c < kCPL; ++c) if ((idx & (kCPL - 1)) == c) x = v[c];
        return wbcast(x, idx / kCPL);
    }
    // dst[j] = v[j - j0] for the lane's cells j < limit
    MGB_HD static void store_cells(score_t *dst, int j0, const score_t (&v)[kCPL], int limit) {
#if MGB_DEVICE_CODE
        if (j0 < limit) dst[j0] = v[0];
#else
        for (int c = 0; c < kCPL && j0 + c < limit; ++c) dst[j0 + c] = v[c];
#endif
    }
    MGB_HD static void store_flags(uint8_t *dst, int j0, const uint8_t (&v)[kCPL]) {
#if MGB_DEVICE_CODE
        dst[j0] = v[0];
#else
        for (int c = 0; c < kCPL; ++c) dst[j0 + c] = v[c];
#endif
    }

    // update_column (extender.cpp:209-290, max-plus scan form) + extend_ins_end (:293-328) for a child column
    // whose n4 <= 28 and size0 <= 27. pS / pF: the parent's S / F shifted to the child's rows. Returns the final
    // size, or -1 when the column outgrows the register path (nothing has been stored then).
    template <class ProfFn>
    MGB_HD static int reg_column(ProfFn prof, const score_t *pS, const score_t *pF, int n, int size0, int max_size,
                                 score_t add, bool use_del, score_t cutoff, score_t go, score_t ge, int ge_shift, RegCol &r) {
        const int j0 = wlane() * kCPL;
        const int n4 = (n + 3) & ~3;
        score_t mval[kCPL], pr[kCPL], psm1[kCPL], pfv[kCPL];
        int aloc[kCPL];
        score_t prev = (j0 >= 1 && j0 <= n4) ? pS[j0 - 1] : kNinf;
        int loc = INT32_MIN;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const int j = j0 + c;
            const bool act = j < n4;
            const score_t ps_j = act ? pS[j] : kNinf;
            const score_t pf_j = act ? pF[j] : kNinf;
            pr[c] = prof(j);
            psm1[c] = prev; pfv[c] = pf_j;
            const score_t match = (act && j) ? wadd(wadd(prev, pr[c]), add) : kNinf;
            // (DPX add-max forms of max(S + go, F + ge) and of the running maximum)
            const score_t del = (act && use_del) ? wadd(iaddmax(ps_j, go, wadd(pf_j, ge)), add) : kNinf;
            mval[c] = imax(match, del);
            r.F[c] = act ? del : kNinf;
            // a[j] = m[j] + go - j*ge ; E[j+1] = prefmax(a)[j] + j*ge
            if (act) loc = iaddmax(mval[c], go - j * ge, loc);
            aloc[c] = loc;
            prev = ps_j;                                   // pS[j] for cell j + 1 (valid while j + 1 <= n4)
        }
        // prefix max over the previous lanes (incl. a[-1] = E[0] + ge, E[0] = ninf)
        const int lane_incl = imax(wscan_max(loc), wadd(kNinf, ge));
        const int lane_excl = wshfl_up1(lane_incl, wadd(kNinf, ge));
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const int j = j0 + c;
            const int excl = c ? imax(lane_excl, aloc[c ? c - 1 : 0]) : lane_excl;      // prefix max over i < j
            const score_t E_j = (j >= 1 && j <= n4) ? wadd(excl, (j - 1) * ge) : kNinf;
            score_t S_j = kNinf;
            if (j < n4) { const score_t sv = imax(mval[c], E_j); S_j = sv > cutoff - 1 ? sv : kNinf; }
            if (size0 > imax(1, n) && j == size0 - 1) {                                 // scalar tail (:284-289)
                const score_t tt = imax(wadd(wadd(psm1[c], add), pr[c]), E_j);
                if (tt >= cutoff) S_j = tt;
            }
            r.S[c] = S_j; r.E[c] = E_j;
        }
        // extend_ins_end (:293-328)
        int size = size0;
        if (size0 < max_size) {
            const score_t s_last = cell_bcast(r.S, size0 - 1), e_last = cell_bcast(r.E, size0 - 1);
            const score_t ins = imax(wadd(s_last, go), wadd(e_last, ge));
            if (ins >= cutoff) {
                const uint32_t diff = (uint32_t)ins - (uint32_t)cutoff;                  // ins >= cutoff
                const uint32_t extra = ge_shift >= 0 ? diff >> ge_shift
                                     : (ge < 0 ? diff / (uint32_t)(-ge) : 0x7fffffffu);
                const uint32_t room = (uint32_t)(max_size - size0 - 1);
                const int cnt = 1 + (int)(extra < room ? extra : room);
                if (size0 + cnt > 27) return -1;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
                for (int c = 0; c < kCPL; ++c) {
                    const int j = j0 + c;
                    if (j >= size0) {
                        const bool in = j < size0 + cnt;
                        r.S[c] = in ? wadd(ins, (j - size0) * ge) : kNinf;
                        r.E[c] = r.S[c]; r.F[c] = kNinf;
                    }
                }
                size = size0 + cnt;
            }
        }
        // what the backtrack asks of E and F (see CF_*)
        score_t e_prev = wshfl_up1(r.E[kCPL - 1], kNinf);
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            r.fl[c] = (uint8_t)((r.S[c] == r.E[c] ? CF_INS : 0) | (r.E[c] == wadd(e_prev, ge) ? CF_INS_EXT : 0)
                              | (r.S[c] == r.F[c] ? CF_DEL : 0) | (r.F[c] == wadd(wadd(pfv[c], add), ge) ? CF_DEL_EXT : 0));
            e_prev = r.E[c];
        }
        return size;
    }

    // per-column scan (:643-669) of a register column of `size` cells whose cell j is row begin + j: the smallest
    // finite and the largest score, max_pos (the row of the largest score nearest to the diagonal diag_i, the lowest
    // such row on ties) and has_extension (in the seed, or a cell reaches ext_cut with the suffix sum psb[j] added).
    // One reduction over the key (|off-diagonal| << 5) | j finds max_pos; the key fits while L < 2^25.
    struct ColScan { score_t min, max; int max_pos; bool has_extension; };
    MGB_HD static ColScan reg_scan(const RegCol &r, int size, int begin, int diag_i, bool in_seed, const int32_t *psb,
                                   score_t ext_cut) {
        const int j0 = wlane() * kCPL;
        score_t mn = 0x7fffffff, bs = INT32_MIN;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const bool cell = j0 + c < size;
            const score_t v = r.S[c];
            if (cell && v != kNinf) mn = imin(mn, v);
            if (cell) bs = imax(bs, v);
        }
        ColScan sc;
        sc.min = wreduce_min(mn);
        sc.max = wreduce_max(bs);
        int bkey = 0x7fffffff; bool he = false;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) {
            const int j = j0 + c;
            const bool cell = j < size;
            if (cell && r.S[c] == sc.max) bkey = imin(bkey, (iabs(j + begin - diag_i) << 5) | j);
            if (!in_seed && cell && wadd(r.S[c], psb[j]) >= ext_cut) he = true;
        }
        sc.max_pos = (wreduce_min(bkey) & 31) + begin;
        sc.has_extension = in_seed || wballot(he) != 0;
        return sc;
    }
    // commit of a register column in the compact format, in whole 32-byte sectors: S and the flag bytes to the DP table
    // at the first multiple of 8 cells from cells_used, S and F to the on-chip child buffer child_S (F at
    // child_S + 2 * bmax). Returns the cells' offset; cells_used moves past them and the space reserved for F.
    MGB_HD static uint32_t commit_compact(const RegCol &r, int size, score_t *cells, uint32_t &cells_used, score_t *child_S,
                                          int bmax) {
        const int j0 = wlane() * kCPL;
        const int capr = capr_of(size);
        const uint32_t off = (cells_used + 7u) & ~7u;
        cells_used = off + 2 * capr + 8;
        score_t *dst = cells + off;
        store_cells(dst, j0, r.S, capr);
        store_flags(reinterpret_cast<uint8_t*>(dst + capr), j0, r.fl);
        store_cells(child_S, j0, r.S, 32); store_cells(child_S + 2 * bmax, j0, r.F, 32);
        return off;
    }
    // band of a register column under cutoff: bit j set for the cells j < size with S >= cutoff
    MGB_HD static uint32_t reg_band(const RegCol &r, int size, score_t cutoff) {
        const int j0 = wlane() * kCPL;
        uint32_t bits = 0;
#if MGB_DEVICE_CODE
#pragma unroll
#endif
        for (int c = 0; c < kCPL; ++c) if (j0 + c < size && r.S[c] >= cutoff) bits |= 1u << c;
        return kCPL == 32 ? bits : wreduce_or(bits << (j0 & 31));
    }

    // --------------------------------------------------------------------------------
    // DefaultColumnExtender::extend (extender.cpp:412-772) + backtrack (:800-1034)
    //   e      extender (query strand) index, seed in slot `seed_slot`
    //   results are written to slots out_base .. out_base + n_out
    // The reference's nested loops (queue rounds -> next_nodes -> outgoing edges) run here as ONE loop whose
    // iteration creates one child column: `t >= n_out` means "take the next parent off the queue".
    // --------------------------------------------------------------------------------
    MGB_HD int extend(int e, int seed_slot, score_t min_path_score, bool force_fixed_seed, int out_base) {
        const int s = e;                                 // query strand of this extender
        const AlnSlot seed = m.slot(seed_slot);
        const AlnHdr sh = *seed.h;
        bool rc = false;
        const int K = ix.k;
        const score_t xdrop = cfg.xdrop;
        score_t cutoff = 0;
        int start = 0, wlen = 1, seed_off_m1 = 0, seed_seq_len = 0;
        score_t partial_sum_offset = 0;
        const char *seed_seq = nullptr;
        uint64_t seed_node0 = 0;
        int res0 = -1, res1 = -1;                         // columns resident in sm.buf(0) / sm.buf(1)
        ColMeta last_col = ColMeta(); uint32_t last_idx = 0xffffffffu;  // newest committed column (register copy)
        bool last_band_valid = false; uint32_t last_band_mask = 0; score_t last_band_cutoff = 0;
        // (L < 2^25: reg_scan's key holds a cell's distance to the diagonal and its row in one int)
        const bool reg_path = use_fast && sm.bmax() >= 40 && (sm.bmax() & 3) == 0 && L < (1 << 25);
        const bool chain_ok = !MGB_WIDE(ix) && !MGB_PRIMARY(ix) && sm.lay->has_prof && L + 1 <= sm.lq();
        uint32_t cells_limit = 0;
        score_t min_cell_score = 0, best_score = 0;
        int heap_n = 0, nn_n = 0;
        bool go = sh.used;                                // nothing to extend from a seed slot that was dropped
        if (go) {
            rc = !MGB_CANONICAL(cfg) && cx[e].rc;        // the RCDBG view is never used on CANONICAL / PRIMARY graphs
            ++cx[e].num_ext;
            min_path_score = imax(0, min_path_score);
            n_cols = 0; cells_used = 0;
            hp = sm.heap(); hp_cap = sm.hcap(); np = sm.nn(); np_cap = sm.hcap();
            pf_node = 0; pf_key = ~0ull; pf_slot_idx = 0;
            cutoff = imax(-xdrop, kNinf + 1);
            start = aln_clipping(seed);
            wlen = L - start;                             // |window|
            seed_off_m1 = (int)sh.offset - 1;             // seed_offset
            seed_seq_len = sh.seq_len;
            partial_sum_offset = cx[s].ps[start + wlen];
            // seed characters: for plain seeds the sequence equals the query substring (staged on chip)
            seed_seq = seed_is_query ? cx[s].q + start : seed.seq;
            seed_node0 = seed.nodes[0];
            if ((uint64_t)3 * (wlen + 16) > 3ull * caps.max_cells) { overflow = true; go = false; }
            // committing a column is safe while cells_used <= cells_limit (room for it and the next scratch)
            cells_limit = (uint32_t)(3ull * caps.max_cells - 6ull * (wlen + 16));
        }

        // ---------------- exact-path shortcut (DESIGN.md): every k-mer of this strand is in the graph and the seed
        // starts the read. The extension below would walk exactly those nodes first (their columns hold the best
        // score so far, so the queue pops them before anything else), the backtrack would start from the last of
        // them at the end of the read -- every other start scores less: a shorter alignment misses matches and the
        // end bonus, any mismatch or gap costs more than the match it replaces, and another path cannot spell the
        // same characters -- and walk the diagonal back: {L}=, the read's own nodes. lower_config() checked what this
        // needs from the scores (cfg.exact_shortcut).
        shortcut_hit = false;
        if (go && cfg.exact_shortcut && !force_fixed_seed && seed_is_query && start == 0 && sh.offset == 0 && !rc
                && !MGB_CANONICAL(cfg) && !MGB_PRIMARY(ix) && L >= K && cx[s].qnodes != nullptr) {
            const uint64_t *qn = cx[s].qnodes;
            const int nk = L - K + 1;
            bool miss = false;
            for (int i2 = wlane(); i2 < nk; i2 += kWarp) miss = miss || qn[i2] == 0;
            const score_t full = cx[s].ps[0] - cx[s].ps[L] + cfg.left_end_bonus + cfg.right_end_bonus;
            if (!wballot(miss) && full >= min_path_score) {
                if ((int)caps.aln_nodes < nk || (int)caps.aln_seq < L || (int)caps.aln_cigar < 1) overflow = true;
                else {
                    const AlnSlot o = m.slot(out_base);
                    wsync();
                    for (int i2 = wlane(); i2 < nk; i2 += kWarp) o.nodes[i2] = qn[i2];
                    for (int i2 = wlane(); i2 < L; i2 += kWarp) o.seq[i2] = cx[s].q[i2];
                    o.cigar[0] = cig_pack(OP_M, L);
                    AlnHdr h;
                    h.q_len = L; h.n_nodes = nk; h.seq_len = L; h.n_cigar = 1; h.score = full; h.offset = 0;
                    h.orientation = sh.orientation; h.used = 1;
                    *o.h = h;
                    wsync();
                    shortcut_hit = true;
                }
                go = false;
            }
        }

        // root column (:455-470)
        if (go) {
            Scratch sc;
            bool have_sc = true;
            if (1 + 8 <= sm.bmax()) sc = scratch_smem(0);
            else { have_sc = scratch_arena(wlen + 1, &sc); MGB_EMU_HIT(EMU_ARENA_COLUMN); }
            if (have_sc) {
                for (int t = wlane(); t < 1 + 5; t += kWarp) { sc.S[t] = kNinf; sc.E[t] = kNinf; sc.F[t] = kNinf; }
                wsync();
                sc.S[0] = cfg.left_end_bonus && !start ? cfg.left_end_bonus : 0;
                wsync();
                int size = extend_ins_end(sc, 1, wlen + 1, cutoff);
                if (!overflow) {
                    m.cols()[n_cols++] = make_col(seed_node0, 0xffffffffu, 0, seed_off_m1, 0, 0, 0, FMT_FULL, size,
                                                  commit_column(sc, size));
                    if (sc.on_chip) res0 = 0;
                    cx[e].table_cap = table_capacity(cx[e].table_cap, n_cols);
                    stats.dp_cells += size; ++stats.dp_columns;
                    table_size_bytes = column_bytes(0, cx[e].table_cap, 1, size);   // the table's whole capacity
                    wsync();
                }
            }
            if (overflow) go = false;
        }

        MGB_TIC(t_fwd);
        if (go) { HeapItem r0; r0.score = 0; r0.neg_off_diag = 0; r0.idx = 0; r0.max_score = 0; heap_push(heap_n, r0); }
        bool finished = false;

        // the parent being expanded and what its children share
        uint32_t i = 0;
        int t = 0, n_out = 0;                             // children t .. n_out - 1 of column i are still to be made
        bool plain_out = false;                           // all added scores are 0 (not stored)
        bool one_reg = false; uint64_t one_node = 0; uint8_t one_ch = 0;   // a single plain child, kept in registers
        int next_offset = 0, begin = 0, size0 = 0, n = 0, shift = 0, cb = 0, pb = -1;
        bool in_seed = false;
        const score_t *parS = nullptr, *parF = nullptr;
        uint8_t par_fmt = FMT_FULL;

        while (go && !overflow && !finished) {
            // ---------------- chain: the column just committed is the only candidate (:477-504 would push it and
            // pop it again), sits in an on-chip buffer and its band under the current cutoff is known. In a
            // linear stretch of the graph every column is like that: chain_loop() (run by chain_entry, with the
            // running values handed over in a ChainIO) creates such columns one after the other until something
            // unusual turns up, which it leaves to the general code below.
            {
                const bool chain = reg_path && chain_ok && t >= n_out && heap_n == 0 && nn_n == 1
                                   && np[0].idx == last_idx && last_band_valid && last_band_cutoff == cutoff
                                   && (res0 == (int)last_idx || res1 == (int)last_idx);
                if (chain) {
                    ChainIO io;
                    io.e = e; io.rc = rc; io.start = start; io.wlen = wlen; io.seed_off_m1 = seed_off_m1;
                    io.sh_offset = (int)sh.offset; io.seed_seq_len = seed_seq_len; io.force_fixed = force_fixed_seed;
                    io.seed_is_query = seed_is_query; io.partial_sum_offset = partial_sum_offset;
                    io.seed_seq = seed_seq; io.seed_nodes = seed.nodes; io.seed_node0 = seed_node0; io.cells_limit = cells_limit;
                    io.ci = last_idx; io.c_node = last_col.node; io.c_offset = last_col.offset; io.c_trim = last_col.trim;
                    io.c_bm = last_band_mask; io.c_pb = res1 == (int)last_idx ? 1 : 0;
                    io.cur_it = np[0];
                    io.cutoff = cutoff; io.best_score = best_score; io.min_cell_score = min_cell_score;
                    io.table_size_bytes = table_size_bytes; io.n_cols = n_cols; io.cells_used = cells_used;
                    io.pf_node = pf_node; io.pf_adj = pf_adj;
                    io.stop = 0; io.overflow = false; io.dp_cells = 0; io.dp_columns = 0;
                    chain_entry(ix, cfg, caps, m, sm, L, &io);
                    cutoff = io.cutoff; best_score = io.best_score; min_cell_score = io.min_cell_score;
                    table_size_bytes = io.table_size_bytes; n_cols = io.n_cols; cells_used = io.cells_used;
                    pf_node = io.pf_node; pf_adj = io.pf_adj;
                    stats.dp_cells += io.dp_cells; stats.dp_columns += io.dp_columns;
                    if (io.overflow) overflow = true;
                    // the general code finds: an empty queue (stop 1), or column ci as the one entry of
                    // next_nodes (stop 2); its register copy is re-read from the table, its band re-computed
                    if (io.stop == 1) nn_n = 0; else { np[0] = io.cur_it; nn_n = 1; }
                    last_idx = 0xffffffffu; last_band_valid = false;
                    res0 = io.c_pb == 0 ? (int)io.ci : -1; res1 = io.c_pb == 1 ? (int)io.ci : -1;
                }
            }
            if (overflow) continue;
            if (t >= n_out) {
                // ---------------- next parent: queue round / next_nodes (:477-504) ----------------
                if (!nn_n) {
                    if (!heap_n) { finished = true; continue; }
                    nn_push(nn_n, heap_pop(heap_n));
                    while (heap_n && hp[0].score == np[nn_n - 1].score) nn_push(nn_n, heap_pop(heap_n));
                    if (overflow) continue;
                }
                i = np[--nn_n].idx;
                t = 0; n_out = 0;
                // `last_col` is the register copy of column `last_idx`; the popped column takes it over
                if (i != last_idx) { last_col = m.cols()[i]; last_idx = i; last_band_valid = false; }
                const ColMeta &par = last_col;
                next_offset = par.offset + 1;
                in_seed = (uint32_t)(next_offset - (int)sh.offset) < (uint32_t)seed_seq_len;
                par_fmt = par.fmt;
                // parent cells: on chip if it is one of the two most recent columns
                pb = res0 == (int)i ? 0 : (res1 == (int)i ? 1 : -1);
                if (pb >= 0) { parS = sm.buf(pb); parF = parS + 2 * sm.bmax(); }
                else {
                    parS = m.cells() + par.cells_off;
                    parF = parS + (par.fmt == FMT_FULL ? 2 * (par.size + 5) : capr_of(par.size) + 8);
                }
                cb = pb >= 0 ? 1 - pb : 0;                // buffer for the children

                if (const int b = budget_stop(cfg, parS[par.max_pos - par.trim], best_score, n_cols, wlen, table_size_bytes)) {
                    MGB_EMU_HIT(b == BUDGET_NODES ? EMU_NODES_STOP_GENERAL : EMU_RAM_STOP_GENERAL);
                    heap_n = 0; nn_n = 0;
                    continue;
                }
                // band within the xdrop cutoff (:549-560)
                int prev_end;
                if (last_band_valid && last_band_cutoff == cutoff) {
                    // band recorded when the column was committed (same cutoff): no second pass
                    if (!last_band_mask) continue;
                    begin = ffs32(last_band_mask) - 1 + par.trim;
                    prev_end = 32 - clz32(last_band_mask) + par.trim;
                } else {
                    int lo = 0x7fffffff, hi = -1;
                    for (int j = wlane(); j < par.size; j += kWarp) {
                        if (parS[j] >= cutoff) { lo = imin(lo, j); hi = imax(hi, j); }
                    }
                    lo = wreduce_min(lo); hi = wreduce_max(hi);
                    if (hi < 0) continue;                 // prev_end <= begin
                    begin = lo + par.trim; prev_end = hi + 1 + par.trim;
                }

                // call_outgoing (:330-387)
                plain_out = false; one_reg = false;
                {
                    const uint32_t seed_pos = (uint32_t)(next_offset - (int)sh.offset);
                    if (in_seed && next_offset < K) {
                        one_node = seed_node0; one_ch = (uint8_t)seed_seq[seed_pos];
                        one_reg = true; plain_out = true; n_out = 1;
                    } else if (in_seed && force_fixed_seed) {
                        const int node_i = next_offset - K + 1;
                        const uint64_t next_node = seed.nodes[node_i];
                        one_node = next_node; one_ch = (uint8_t)seed_seq[seed_pos];
                        if (next_node) { one_reg = true; plain_out = true; }
                        else {
                            sm.out_nodes()[0] = next_node; sm.out_chars()[0] = one_ch;
                            sm.out_scores()[0] = !par.node ? cfg.gap_ext : cfg.gap_open;
                            wsync();
                        }
                        n_out = 1;
                    } else if (MGB_PRIMARY(ix)) {          // extender.cpp:361-380 (the hint equals the node's sequence)
                        n_out = canon_out(par.node, sm.out_nodes(), sm.out_chars());
                        plain_out = true;
                        wsync();
                    } else if (!rc) {
                        // DBGSuccinct::call_outgoing_kmers through the adjacency record; the record of the most
                        // recently created column was requested while its DP was computed
                        const Adj a = (!MGB_WIDE(ix) && par.node == pf_node) ? adj_decode(pf_adj) : load_adj_any(ix, par.node);
                        plain_out = true;
                        if (a.last) {
                            const uint32_t all = a.all, ok = a.ok & ~1u;
                            const uint64_t first = (uint64_t)a.last - popc32(all) + 1;
                            n_out = popc32(ok);
                            if (n_out == 1) {
                                const uint32_t c = (uint32_t)ffs32(ok) - 1;
                                one_node = first + popc32(all & ((1u << c) - 1u)); one_ch = (uint8_t)cfg.letters[c];
                                one_reg = true;
                            } else if (n_out > 1 && n_out <= kMaxOut) {
                                int k2 = 0;
                                for (uint32_t c = 1; c < ix.sigma; ++c) {
                                    if (!((ok >> c) & 1u)) continue;
                                    sm.out_nodes()[k2] = first + popc32(all & ((1u << c) - 1u)); sm.out_chars()[k2] = cfg.letters[c];
                                    ++k2;
                                }
                                wsync();
                            }
                        }
                    } else {
                        n_out = outgoing_rc(par.node, sm.out_nodes(), sm.out_chars());
                        plain_out = true;
                        wsync();
                    }
                    if (n_out > kMaxOut) { overflow = true; continue; }
                }
                if (n_out == 0) { m.cols()[i].is_tip = 1; continue; }

                const int end = imin(prev_end, wlen) + 1;
                size0 = end - begin;
                n = prev_end - begin;                     // parent rows inside the band
                shift = begin - par.trim;
            }

            // ---------------- child t of column i (:562-770) ----------------
            const int tc = t++;
            uint8_t ch = one_reg ? one_ch : sm.out_chars()[tc];
            if (ch >= 'a' && ch <= 'z') ch -= 32;          // toupper (:564)
            const uint64_t cnode = one_reg ? one_node : sm.out_nodes()[tc];
            const score_t add = plain_out ? 0 : sm.out_scores()[tc];
            if (n_cols >= caps.max_cols) { overflow = true; continue; }
            const int code = encode_char(ch);
            const int diag_i = next_offset - seed_off_m1;

            // ---- register path: the whole column (incl. its 5 padding cells) fits 32 cells (n4 <= 28, final
            // size <= 27). Fuses DPTColumn::create, update_column, extend_ins_end, the per-column scan, the
            // table commit (compact format) and the convergence filter.
            if (reg_path && n <= 28 && size0 <= 27) {
                {   // requests whose latency overlaps the DP below
                    if (!rc && cnode && !MGB_WIDE(ix) && !MGB_PRIMARY(ix)) { pf_node = cnode; pf_adj = load_adj(ix, cnode); }
                    pf_key = cnode + (rc ? ix.n : 0);
                    pf_slot_idx = hash_node(pf_key, caps.hash_size - 1);
                    pf_slot = cx[e].conv_slots[pf_slot_idx];
                }
                RegCol r;
                const int prof_base = start + begin;
                const int size = reg_column([&](int j) { return prof_score(s, prof_base + j, code); }, parS + shift, parF + shift,
                                            n, size0, wlen + 1 - begin, add, next_offset > 1, cutoff, cfg.gap_open, cfg.gap_ext,
                                            cfg.ge_shift, r);
                if (size >= 0) {
                    MGB_COUNT(5);
                    const uint32_t cap_before = cx[e].table_cap;
                    cx[e].table_cap = table_capacity(cap_before, n_cols + 1);
                    stats.dp_cells += size; ++stats.dp_columns;
                    const ColScan scan = reg_scan(r, size, begin, diag_i, in_seed, cx[s].ps + start + begin,
                                                (score_t)((double)best_score * cfg.rel_score_cutoff + (double)partial_sum_offset));
                    min_cell_score = imin(min_cell_score, scan.min);
                    if (!accept_column(in_seed, scan.max, scan.has_extension, cap_before, cx[e].table_cap, size0, size, xdrop,
                                       cutoff, best_score, table_size_bytes))
                        continue;
                    if (cells_used > cells_limit) { overflow = true; continue; }
                    const uint32_t off = commit_compact(r, size, m.cells(), cells_used, sm.buf(cb), sm.bmax());
                    const ColMeta col = make_col(cnode, i, ch, next_offset, scan.max_pos, begin, add, FMT_COMPACT, size, off);
                    const uint32_t idx = n_cols;
                    m.cols()[n_cols++] = col;
                    last_col = col; last_idx = idx;
                    // band of this column under the (updated) cutoff, for when it is expanded
                    last_band_mask = reg_band(r, size, cutoff); last_band_cutoff = cutoff; last_band_valid = true;
                    if (cb) res1 = (int)idx; else res0 = (int)idx;
                    wsync();
                    // convergence filter from registers (update_seed_filter)
                    const int s_first = begin ? 0 : 1;
                    const int vec_offset = start + begin - (begin ? 1 : 0);
                    const score_t converged = update_seed_filter_regs(e, cnode, vec_offset, r.S, s_first, size);
                    if (overflow) continue;
                    if (converged != kNinf) {
                        HeapItem it; it.score = converged; it.neg_off_diag = -iabs(scan.max_pos - diag_i);
                        it.idx = idx; it.max_score = scan.max;
                        if (nn_n && converged == np[0].score) nn_push(nn_n, it);
                        else if (heap_n == 0 && nn_n == 0 && t == n_out) {
                            // sole candidate: pushing it and popping it in the next round is the
                            // identity; np[0] must still hold it for the tie test above. It is expanded from
                            // the on-chip buffer next, so its F never has to be read from the table
                            np[0] = it; nn_n = 1;
                            continue;
                        } else heap_push(heap_n, it);
                        // the column waits in the queue: a later expansion reads its F from the table
                        store_cells(m.cells() + off + capr_of(size) + 8, wlane() * kCPL, r.F, capr_of(size));
                        m.cols()[idx].fmt = FMT_COMPACT_F; last_col.fmt = FMT_COMPACT_F;
                    }
                    continue;
                }
            }
            // ---- general path: columns of any width, S | E | F in the table
            MGB_COUNT(6);
            MGB_EMU_HIT(EMU_GENERAL_COLUMN);
            if (par_fmt == FMT_COMPACT && pb >= 0) {
                // the backtrack compares the F of a general-path column with its parent's (:976-997): write the
                // parent's F (still on chip) into the space its compact record reserves for it
                const ColMeta pc = m.cols()[i];
                score_t *dstF = m.cells() + pc.cells_off + capr_of(pc.size) + 8;
                for (int j = wlane(); j < pc.size + 5; j += kWarp) dstF[j] = parF[j];
                m.cols()[i].fmt = FMT_COMPACT_F; par_fmt = FMT_COMPACT_F;
                if (last_idx == i) last_col.fmt = FMT_COMPACT_F;
                wsync();
            }
            Scratch sc;
            if (size0 + 8 <= sm.bmax()) { sc = scratch_smem(cb); if (cb) res1 = -1; else res0 = -1; }
            else { MGB_EMU_HIT(EMU_ARENA_COLUMN); if (!scratch_arena(wlen + 1 - begin, &sc)) continue; }
            // DPTColumn::create: everything (incl. padding) = ninf (extender.cpp:389-410)
            for (int j = wlane(); j < size0 + 5; j += kWarp) { sc.S[j] = kNinf; sc.E[j] = kNinf; sc.F[j] = kNinf; }
            wsync();
            const uint32_t cap_before = cx[e].table_cap;
            cx[e].table_cap = table_capacity(cap_before, n_cols + 1);

            update_column(s, parS + shift, parF + shift, sc, size0, n, start + begin, cutoff,
                          code, add, next_offset > 1);
            const int size = extend_ins_end(sc, size0, wlen + 1 - begin, cutoff);
            if (overflow) continue;
            stats.dp_cells += size; ++stats.dp_columns;

            // per-column scan (:643-669)
            bool has_extension = in_seed;
            const score_t extension_cutoff
                = (score_t)((double)best_score * cfg.rel_score_cutoff + (double)partial_sum_offset);
            int max_pos;
            {
                score_t mn = 0x7fffffff; score_t bs = INT32_MIN; int bd = 0x7fffffff, bj = 0x7fffffff;
                bool he = false;
                for (int j = wlane(); j < size; j += kWarp) {
                    score_t v = sc.S[j];
                    if (v != kNinf) mn = imin(mn, v);
                    int d = iabs(j + begin - diag_i);
                    if (v > bs || (v == bs && d < bd)) { bs = v; bd = d; bj = j; }
                    if (wadd(v, cx[s].ps[start + begin + j]) >= extension_cutoff) he = true;
                }
                min_cell_score = imin(min_cell_score, wreduce_min(mn));
                score_t gbs = wreduce_max(bs);
                int gd = wreduce_min(bs == gbs ? bd : 0x7fffffff);
                int gj = wreduce_min(bs == gbs && bd == gd ? bj : 0x7fffffff);
                max_pos = gj + begin;
                if (!has_extension && wballot(he)) has_extension = true;
            }
            const score_t max_val = sc.S[max_pos - begin];

            if (!accept_column(in_seed, max_val, has_extension, cap_before, cx[e].table_cap, size0, size, xdrop, cutoff,
                               best_score, table_size_bytes))
                continue;
            if ((uint64_t)cells_used + 3ull * (size + 5) + 3ull * (wlen + 16) > 3ull * caps.max_cells) {
                overflow = true; continue;
            }
            const ColMeta col = make_col(cnode, i, ch, next_offset, max_pos, begin, add, FMT_FULL, size, commit_column(sc, size));
            const uint32_t idx = n_cols;
            m.cols()[n_cols++] = col;
            last_col = col; last_idx = idx; last_band_valid = false;
            if (sc.on_chip) { if (cb) res1 = (int)idx; else res0 = (int)idx; }

            const int vec_offset = start + begin - (begin ? 1 : 0);
            const int s_first = begin ? 0 : 1;
            score_t converged = update_seed_filter(e, col.node, vec_offset, sc.S + s_first, size - s_first);
            if (overflow) continue;
            if (converged != kNinf) {
                HeapItem it; it.score = converged; it.neg_off_diag = -iabs(max_pos - diag_i);
                it.idx = idx; it.max_score = max_val;
                if (nn_n && converged == np[0].score) nn_push(nn_n, it);
                else heap_push(heap_n, it);
            }
        }
        if (shortcut_hit) return 1;
        if (!go || overflow) return 0;
        wsync();
        MGB_TOC(t_fwd, 2);

        if (cfg.no_backtrack) {
            copy_slot(out_base, seed_slot);
            return 1;
        }
        MGB_TIC(t_bt);
        int n_res = backtrack(e, seed_slot, min_path_score, start, wlen, min_cell_score, out_base);
        for (int r = 0; r < n_res; ++r) trim_offset(out_base + r);
        MGB_TOC(t_bt, 3);
        return n_res;
    }

    // The extender's chain loop (see extend()): one child column per iteration of the column that is the sole
    // candidate, registers only, no queue traffic. It runs in an aligner of its own (chain_entry) and takes the
    // running values from io, where it leaves them again; everything it reads more than once is copied into locals first.
    // Leaves with io.stop = 1 (the extension is over: nothing is left in the queue) or 2 (column io.ci stays the
    // sole candidate and the general code expands it: several children, a column too wide for the register path,
    // a seed node missing from the graph, a convergence-table entry that has to move, ...).
    MGB_HD void chain_loop(ChainIO &io) {
        const int e = io.e, s = io.e;
        const bool rc = io.rc != 0;
        const int start = io.start, wlen = io.wlen, seed_off_m1 = io.seed_off_m1, sh_offset = io.sh_offset;
        const int seed_seq_len = io.seed_seq_len, K = (int)ix.k;
        const bool force_fixed = io.force_fixed != 0, seed_is_q = io.seed_is_query != 0;
        const char *seed_seq = io.seed_seq; const uint64_t *seed_nodes = io.seed_nodes;
        const uint64_t seed_node0 = io.seed_node0;
        const score_t go = cfg.gap_open, ge = cfg.gap_ext, xdrop = cfg.xdrop;
        const int ge_shift = cfg.ge_shift;
        const double rsc = cfg.rel_score_cutoff, pso = (double)io.partial_sum_offset;
        const uint32_t max_cols = caps.max_cols, hash_mask = caps.hash_size - 1;
        const uint32_t max_conv_entries = caps.max_conv_entries, max_conv_cells = caps.max_conv_cells, hash_size = caps.hash_size;
        const uint64_t n_edges = ix.n;
        const uint32_t sigma = ix.sigma;
        const uint2 *adj = ix.adj, *radj = ix.radj;
        const uint32_t *valid = ix.valid;
        uint32_t letters = 0;                              // '$ACGT': letters of symbols 1..4, one byte each
        for (int c = 1; c <= 4; ++c) letters |= (uint32_t)(uint8_t)cfg.letters[c] << (8 * (c - 1));
        ColMeta *cols = m.cols();
        score_t *cells = m.cells();
        StrandCtx &tc = cx[e];
        ConvSlot *cslots = tc.conv_slots; score_t *ccells = tc.conv_cells;
        const uint32_t epoch = tc.conv_epoch;
        uint32_t conv_n = tc.conv_n, conv_used = tc.conv_cells_used, t_cap = tc.table_cap;
        const int32_t *ps = cx[s].ps;
        const uint32_t *p4 = sm.prof4(s);
        const uint8_t *qcodes = cx[s].codes;
        score_t *buf0 = sm.buf(0);
        const int bmax = sm.bmax();
        const int Lq = L;

        uint32_t ci = io.ci; uint64_t c_node = io.c_node;
        int c_offset = io.c_offset, c_trim = io.c_trim, c_pb = io.c_pb;
        uint32_t c_bm = io.c_bm;
        HeapItem cur_it = io.cur_it;
        score_t c_maxval = cur_it.max_score;
        score_t cutoff = io.cutoff, best_score = io.best_score, min_cell_score = io.min_cell_score;
        uint64_t table_bytes = io.table_size_bytes;
        uint32_t ncols = io.n_cols, cused = io.cells_used;
        const uint32_t cells_limit = io.cells_limit;
        uint64_t pfn = io.pf_node; uint2 pfa = io.pf_adj;
        uint32_t made = 0; uint64_t made_cells = 0;
        int stop = 0;
        bool ovf = false;

        while (!stop) {                                    // every exit sets stop
            if (const int b = budget_stop(cfg, c_maxval, best_score, ncols, wlen, table_bytes)) {
                MGB_EMU_HIT(b == BUDGET_NODES ? EMU_NODES_STOP_CHAIN : EMU_RAM_STOP_CHAIN); stop = 1; break;
            }
            if (!c_bm) { stop = 1; break; }                    // no band: no children
            const int begin = ffs32(c_bm) - 1 + c_trim;
            const int prev_end = 32 - clz32(c_bm) + c_trim;
            const int noff = c_offset + 1;
            const uint32_t seed_pos = (uint32_t)(noff - sh_offset);
            const bool in_seed = seed_pos < (uint32_t)seed_seq_len;
            uint64_t cnode; uint32_t code; uint8_t ch;
            // call_outgoing (:330-387), a single plain child
            if (in_seed && (noff < K || force_fixed)) {
                cnode = noff < K ? seed_node0 : seed_nodes[noff - K + 1];
                if (!cnode) { stop = 2; break; }               // (fixed seed: a node the graph does not have)
                ch = (uint8_t)seed_seq[seed_pos];
                code = seed_is_q ? qcodes[start + seed_pos] : cfg.code_of[ch];
            } else if (!rc) {
                const uint2 a = c_node == pfn ? pfa : adj[c_node];
                const uint32_t all = a.y & 31u, ok = a.x ? ((a.y >> 8) & 30u) : 0u;
                if (!ok) { cols[ci].is_tip = 1; stop = 1; break; }
                if (ok & (ok - 1u)) { stop = 2; break; }
                code = (uint32_t)ffs32(ok) - 1;
                cnode = (uint64_t)a.x - popc32(all) + 1 + popc32(all & ((1u << code) - 1u));
                ch = (uint8_t)(letters >> (8 * (code - 1)));
            } else {
                // RCDBG::call_outgoing_kmers through the reverse adjacency records, single incoming edge
                const uint2 rr = radj[c_node];
                if ((rr.y >> 3) & 1u) { stop = 2; break; }     // several incoming edges
                const uint64_t edge = rr.x;
                uint32_t c = 0;
                if (edge != 0 && edge <= n_edges && (!valid || ((valid[edge >> 5] >> (edge & 31)) & 1u)))
                    c = radj[edge].y & 7u;
                if (!c) { cols[ci].is_tip = 1; stop = 1; break; }   // no incoming k-mer, or its first character is '$'
                code = sigma - c;                                   // complement
                ch = (uint8_t)(letters >> (8 * (code - 1)));
                cnode = edge;
            }
            if (code < 1 || code > 4) { stop = 2; break; }
            if (ch >= 'a' && ch <= 'z') ch -= 32;              // toupper (:564)
            if (ncols >= max_cols) { ovf = true; stop = 1; break; }
            const int size0 = imin(prev_end, wlen) + 1 - begin;
            const int n = prev_end - begin;
            if (n > 28 || size0 > 27) { stop = 2; break; }
            // requests whose latency overlaps the DP below: the child's adjacency record, its convergence slot
            if (!rc) { pfn = cnode; pfa = adj[cnode]; }
            const uint64_t key = cnode + (rc ? n_edges : 0);
            uint32_t hp = hash_node(key, hash_mask);
            ConvSlot sl = cslots[hp];

            const score_t *pS = buf0 + (size_t)c_pb * 3 * bmax + (begin - c_trim);
            const int prof_base = start + begin;
            const int sh = 8 * ((int)code - 1);
            RegCol r;
            const int size = reg_column([&](int j) { const int x = prof_base + j;
                                                     return x <= Lq ? (int)(int8_t)(p4[x] >> sh) : 0; },
                                        pS, pS + 2 * bmax, n, size0, wlen + 1 - begin, 0, noff > 1, cutoff, go, ge,
                                        ge_shift, r);
            if (size < 0) { stop = 2; break; }
            const int diag_i = noff - seed_off_m1;
            const ColScan scan = reg_scan(r, size, begin, diag_i, in_seed, ps + start + begin,
                                          in_seed ? 0 : (score_t)((double)best_score * rsc + pso));
            // ---- convergence filter, first half (update_seed_filter, :100-156): find the node's entry. Cases
            // that move data around are left to the general code before anything has been written
            const int s_first = begin ? 0 : 1;
            const int qstart = start + begin - (begin ? 1 : 0);
            const int n_pass = size - s_first;
            bool hit = false;
            {
                uint32_t probes = 0;
                while (sl.epoch == epoch && sl.key != key && probes < hash_size) { hp = (hp + 1) & hash_mask; sl = cslots[hp]; ++probes; }
                hit = sl.epoch == epoch && sl.key == key;
            }
            int new_end = 0;
            if (!hit) {
                const int seg_start = imax(0, qstart - 8);
                const int seg_cap = imin(Lq + 1, qstart + n_pass + 8) - seg_start;
                if (conv_n >= max_conv_entries || 2 * (conv_n + 1) > hash_size || conv_used + seg_cap > max_conv_cells) {
                    stop = 2; break;                           // (the general code reports the overflow)
                }
                sl.key = key; sl.epoch = epoch; sl.start = qstart; sl.size = n_pass;
                sl.seg_start = seg_start; sl.seg_cap = seg_cap; sl.seg_off = conv_used;
            } else {
                // the node was met before (seed columns share the seed's node): only the in-place cases -- the
                // passed range overlaps the stored one and ends at or after its end, inside the segment
                new_end = imax(qstart + n_pass, sl.start + sl.size);
                if (qstart < sl.start || qstart >= sl.start + sl.size || new_end > sl.seg_start + sl.seg_cap) {
                    stop = 2; break;
                }
            }

            const uint32_t cap_before = t_cap;
            t_cap = table_capacity(t_cap, ncols + 1);
            made_cells += size; ++made;
            min_cell_score = imin(min_cell_score, scan.min);
            if (!accept_column(in_seed, scan.max, scan.has_extension, cap_before, t_cap, size0, size, xdrop, cutoff,
                               best_score, table_bytes)) {
                stop = 1; break;
            }
            if (cused > cells_limit) { ovf = true; stop = 1; break; }
            const uint32_t off = commit_compact(r, size, cells, cused, buf0 + (size_t)(1 - c_pb) * 3 * bmax, bmax);
            const uint32_t idx = ncols;
            cols[ncols++] = make_col(cnode, ci, ch, noff, scan.max_pos, begin, 0, FMT_COMPACT, size, off);
            const uint32_t bm_new = reg_band(r, size, cutoff);

            // ---- convergence filter, second half
            score_t converged;
            score_t *c0 = ccells + sl.seg_off + (qstart - s_first - sl.seg_start);              // indexed by cell
            if (!hit) {
                conv_used += sl.seg_cap; ++conv_n;
                cslots[hp] = sl;
                converged = conv_store_regs(c0, r.S, s_first, size);
            } else {
                const int old_end = sl.start + sl.size;
                if (new_end > old_end) {                       // vec.resize(n, ninf)
                    score_t *cseg = ccells + sl.seg_off;
                    for (int p = old_end + wlane(); p < new_end; p += kWarp) cseg[p - sl.seg_start] = kNinf;
                    sl.size = new_end - sl.start;
                    cslots[hp] = sl;
                    wsync();
                }
                converged = conv_merge_regs(c0, r.S, s_first, size, rsc);
            }
            // the new column becomes the parent
            ci = idx; c_node = cnode; c_offset = noff; c_trim = begin; c_bm = bm_new; c_pb = 1 - c_pb;
            c_maxval = scan.max;
            cur_it.score = converged; cur_it.neg_off_diag = -iabs(scan.max_pos - diag_i); cur_it.idx = idx;
            cur_it.max_score = scan.max;
            if (converged == kNinf) { stop = 1; break; }
        }
        tc.table_cap = t_cap; tc.conv_n = conv_n; tc.conv_cells_used = conv_used;
        io.ci = ci; io.c_pb = c_pb; io.cur_it = cur_it;
        io.cutoff = cutoff; io.best_score = best_score; io.min_cell_score = min_cell_score;
        io.table_size_bytes = table_bytes; io.n_cols = ncols; io.cells_used = cused;
        io.pf_node = pfn; io.pf_adj = pfa;
        io.stop = stop; io.overflow = ovf; io.dp_cells = made_cells; io.dp_columns = made;
    }

    long long phase_cycles[8] = {0,0,0,0,0,0,0,0};   // MGB_PHASE_TIMERS: setup, seeds, fwd loop, backtrack, rest
    bool seed_is_query;          // the seed in SLOT_SEED is a plain query substring
    bool shortcut_hit = false;   // the last extend() call took the exact-path shortcut
    bool use_fast = true;        // register fast path for narrow columns (device only)
    uint64_t pf_node; uint2 pf_adj;        // software prefetch: adjacency record of the newest column
    uint64_t pf_key; ConvSlot pf_slot; uint32_t pf_slot_idx;   // ... and its first conv-table probe
    uint64_t table_size_bytes;

    MGB_HD void cig_append(int &n_ops, uint32_t op) {       // Cigar::append(op, 1)
        if (n_ops && cig_op(m.bt_ops()[n_ops - 1]) == op) m.bt_ops()[n_ops - 1] += 8u;
        else {
            if (n_ops >= (int)caps.aln_cigar - 4) { overflow = true; return; }
            m.bt_ops()[n_ops++] = cig_pack(op, 1);
        }
    }

    MGB_HD int backtrack(int e, int seed_slot, score_t min_path_score, int start, int wlen,
                         score_t min_cell_score, int out_base) {
        const int s = e;
        const AlnSlot seed = m.slot(seed_slot);
        const AlnHdr sh = *seed.h;
        const int K = ix.k;
        const int seed_clipping = start;
        const int seed_off_m1 = (int)sh.offset - 1;
        const int k_minus_1 = K - 1;
        const int last_pos = wlen;
        const int seed_dist = imax(K, sh.seq_len) - 1;
        const score_t min_start_score = min_path_score;
        const int min_trace_length = K - (int)sh.offset;
        const score_t right_end_bonus = cfg.right_end_bonus;

        // start candidates (:815-867), two slots per column
        for (uint32_t i = wlane(); i < n_cols; i += kWarp) {
            BtStart a, b; a.score = INT32_MIN; b.score = INT32_MIN;
            a.neg_off_diag = b.neg_off_diag = a.neg_i = b.neg_i = a.pos = b.pos = 0;
            if (i >= 1) {
                const ColMeta col = m.cols()[i];
                if (col.offset >= seed_dist) {
                    const ColMeta par = m.cols()[col.parent];
                    const int code = encode_char(col.c);
                    for (int which = 0; which < 2; ++which) {
                        int start_pos;
                        if (which == 0) start_pos = col.max_pos;
                        else {
                            if (!(col.size + col.trim == wlen + 1 && col.max_pos != last_pos)) continue;
                            start_pos = last_pos;
                        }
                        if (start_pos < par.trim + 1) continue;
                        int pos = start_pos - col.trim, pos_p = start_pos - par.trim - 1;
                        score_t sv = cellS(col, pos), sp = cellS(par, pos_p);
                        if (sv == kNinf || sp == kNinf) continue;
                        score_t end_bonus = start_pos == last_pos ? right_end_bonus : 0;
                        if (wadd(sv, end_bonus) >= min_start_score) {
                            bool is_match = sv == wadd(wadd(sp, col.score), prof_score(s, seed_clipping + start_pos, code))
                                && prof_is_match(s, seed_clipping + start_pos, code);
                            if (is_match || start_pos == last_pos || col.is_tip) {
                                BtStart &o = which ? b : a;
                                o.score = wadd(sv, end_bonus);
                                o.neg_off_diag = -iabs(start_pos - col.offset + seed_off_m1);
                                o.neg_i = -(int)i; o.pos = start_pos;
                            }
                        }
                    }
                }
            }
            m.starts()[2 * i] = a; m.starts()[2 * i + 1] = b;
        }
        wsync();

        int n_ext = 0;
        score_t best_score = INT32_MIN;
        const uint32_t n_cand = 2 * n_cols;

        while (true) {
            // pop the largest remaining start (heap order of :873-879)
            BtStart best; best.score = INT32_MIN; best.neg_off_diag = INT32_MIN; best.neg_i = INT32_MIN; best.pos = INT32_MIN;
            uint32_t best_idx = 0xffffffffu;
            for (uint32_t c = wlane(); c < n_cand; c += kWarp) {
                BtStart x = m.starts()[c];
                if (x.score == INT32_MIN) continue;
                bool gt = x.score != best.score ? x.score > best.score
                        : x.neg_off_diag != best.neg_off_diag ? x.neg_off_diag > best.neg_off_diag
                        : x.neg_i != best.neg_i ? x.neg_i > best.neg_i : x.pos > best.pos;
                if (best_idx == 0xffffffffu || gt) { best = x; best_idx = c; }
            }
            {
                int has = best_idx != 0xffffffffu;
                int v0 = wreduce_max(has ? best.score : INT32_MIN);
                if (!wballot(has)) break;
                bool ok = has && best.score == v0;
                int v1 = wreduce_max(ok ? best.neg_off_diag : INT32_MIN); ok = ok && best.neg_off_diag == v1;
                int v2 = wreduce_max(ok ? best.neg_i : INT32_MIN); ok = ok && best.neg_i == v2;
                int v3 = wreduce_max(ok ? best.pos : INT32_MIN); ok = ok && best.pos == v3;
                unsigned who = wballot(ok);
                int src = ffs32(who) - 1;
                best.score = v0; best.neg_off_diag = v1; best.neg_i = v2; best.pos = v3;
                best_idx = wbcast(best_idx, src);
            }
            m.starts()[best_idx].score = INT32_MIN;
            wsync();

            if (n_ext >= (int)cfg.num_alternative_paths) break;          // terminate_backtrack_start
            uint32_t j = (uint32_t)(-best.neg_i);
            if (m.cols()[j].started) continue;                             // skip_backtrack_start
            m.cols()[j].started = 1;

            score_t score = best.score;
            if ((int64_t)score - min_cell_score < best_score) break;

            int n_ops = 0, n_path = 0, n_seq = 0, n_trace = 0;
            int pos = best.pos;
            const int end_pos = pos;
            int align_offset = sh.offset;
            bool path_back_nonzero = false;

            // pending CIGAR run lives in registers (Cigar::append merges equal neighbours)
            uint32_t cur_op = 0xffu, cur_len = 0;
            auto cig_add = [&](uint32_t op) {
                if (op == cur_op) { ++cur_len; return; }
                if (cur_len) {
                    if (n_ops >= (int)caps.aln_cigar - 4) { overflow = true; return; }
                    m.bt_ops()[n_ops++] = cig_pack(cur_op, cur_len);
                }
                cur_op = op; cur_len = 1;
            };
            ColMeta col = m.cols()[j];
            ColMeta par = m.cols()[col.parent];
            // the grand-parent's record is requested one step ahead so that a move to the parent costs
            // no dependent round trip
            ColMeta gpar = par;
            if (par.parent != 0xffffffffu) gpar = m.cols()[par.parent];
            bool try_run = true;
            while (j) {
                // Diagonal runs, one warp-wide step: lane t examines column j - t at query position
                // pos - t, assuming that j, j-1, ... is a parent chain and that every step before it was a
                // (mis)match (:961-970). The longest prefix of lanes for which this holds is exactly what
                // the sequential walk would do, and is committed at once.
                if (try_run) {
                    const int t = wlane();
                    bool good = false, is_m = false;
                    ColMeta c_t;
                    c_t.offset = 0; c_t.node = 0; c_t.c = 0; c_t.max_pos = -1;
                    if ((uint32_t)t < j) {
                        c_t = m.cols()[j - t];
                        const ColMeta p_t = m.cols()[j - t - 1];
                        const int pos_t = pos - t;
                        const int ci = pos_t - c_t.trim, pi = pos_t - p_t.trim - 1;
                        if (c_t.parent == j - t - 1 && pos_t > 0 && ci >= 0 && ci < c_t.size && pi >= 0 && pi < p_t.size) {
                            const score_t sv = cellS(c_t, ci);
                            const bool ins = bt_is_ins(c_t, ci, sv) && (t || cur_op == 0xffu || cur_op != OP_D);
                            const int code = encode_char(c_t.c);
                            good = sv != kNinf && !ins
                                && sv == wadd(wadd(cellS(p_t, pi), c_t.score), prof_score(s, seed_clipping + pos_t, code));
                            is_m = prof_is_match(s, seed_clipping + pos_t, code);
                        }
                    }
                    const uint32_t bad = ~wballot(good);
                    const int n_good = bad ? ffs32(bad) - 1 : kWarp;
                    try_run = n_good == kWarp;                // a short run ends on a step of another kind
                    if (n_good) {
                        const bool mine = t < n_good;
                        const bool has_node = mine && c_t.offset >= k_minus_1;
                        const uint32_t node_mask = wballot(has_node);
                        const uint32_t nz_mask = wballot(has_node && c_t.node != 0);
                        const uint32_t m_mask = wballot(mine && is_m);
                        if (n_seq + n_good > (int)caps.aln_seq || n_path + popc32(node_mask) > (int)caps.aln_nodes) {
                            overflow = true; return 0;
                        }
                        if (mine) {
                            m.bt_seq()[n_seq + t] = c_t.c;
                            if (pos - t == c_t.max_pos) m.cols()[j - t].started = 1;
                            if (has_node) m.bt_path()[n_path + popc32(node_mask & ((1u << t) - 1u))] = c_t.node;
                        }
                        if (node_mask) path_back_nonzero = (nz_mask >> (31 - clz32(node_mask))) & 1u;
                        for (int b = 0; b < n_good; ) {          // Cigar::append per run of equal ops
                            const bool mb = (m_mask >> b) & 1u;
                            const uint32_t valid = n_good >= 32 ? 0xffffffffu : ((1u << n_good) - 1u);
                            const uint32_t diff = (mb ? ~m_mask : m_mask) & valid & ~((1u << b) - 1u);
                            const int end = diff ? ffs32(diff) - 1 : n_good;
                            const uint32_t op = mb ? OP_M : OP_X;
                            if (op == cur_op) cur_len += end - b;
                            else {
                                if (cur_len) {
                                    if (n_ops >= (int)caps.aln_cigar - 4) { overflow = true; return 0; }
                                    m.bt_ops()[n_ops++] = cig_pack(cur_op, cur_len);
                                }
                                cur_op = op; cur_len = end - b;
                            }
                            b = end;
                        }
                        n_trace += n_good; n_seq += n_good; n_path += popc32(node_mask);
                        pos -= n_good;
                        align_offset = imin(wbcast(c_t.offset, n_good - 1), k_minus_1);
                        j -= n_good;
                        col = m.cols()[j];
                        if (j) {
                            par = m.cols()[col.parent];
                            gpar = par;
                            if (par.parent != 0xffffffffu) gpar = m.cols()[par.parent];
                        }
                        continue;
                    }
                }
                try_run = true;
                const int trim = col.trim, trim_p = par.trim;
                align_offset = imin(col.offset, k_minus_1);
                if (pos == col.max_pos) m.cols()[j].started = 1;
                const int code = encode_char(col.c);
                const score_t sv = cellS(col, pos - trim);
                const uint32_t last_op = cur_op;

                if (sv == kNinf) {
                    j = 0;
                } else if (pos && bt_is_ins(col, pos - trim, sv) && (last_op == 0xffu || last_op != OP_D)) {
                    // insertion run (:943-959)
                    bool again = true;
                    while (again) {
                        cig_add(OP_I);
                        again = bt_ins_ext(col, pos - trim);
                        --pos;
                    }
                } else if (pos && pos >= trim_p + 1
                        && sv == wadd(wadd(cellS(par, pos - trim_p - 1), col.score),
                                      prof_score(s, seed_clipping + pos, code))) {
                    ++n_trace;
                    if (n_seq >= (int)caps.aln_seq) { overflow = true; return 0; }
                    m.bt_seq()[n_seq++] = col.c;
                    cig_add(prof_is_match(s, seed_clipping + pos, code) ? OP_M : OP_X);
                    if (col.offset >= k_minus_1) {
                        if (n_path >= (int)caps.aln_nodes) { overflow = true; return 0; }
                        m.bt_path()[n_path++] = col.node; path_back_nonzero = col.node != 0;
                    }
                    --pos;
                    j = col.parent;
                    col = par;
                    if (j) { par = gpar; if (par.parent != 0xffffffffu) gpar = m.cols()[par.parent]; }
                } else if (bt_is_del(col, pos - trim, sv) && (last_op == 0xffu || last_op != OP_I)) {
                    // deletion run (:972-999)
                    bool again = true;
                    while (again && j) {
                        align_offset = imin(col.offset, k_minus_1);
                        again = bt_del_ext(col, par, pos);
                        ++n_trace;
                        if (n_seq >= (int)caps.aln_seq) { overflow = true; return 0; }
                        m.bt_seq()[n_seq++] = col.c;
                        cig_add(OP_D);
                        if (col.offset >= k_minus_1) {
                            if (n_path >= (int)caps.aln_nodes) { overflow = true; return 0; }
                            m.bt_path()[n_path++] = col.node; path_back_nonzero = col.node != 0;
                        }
                        j = col.parent;
                        col = par;
                        if (j) { par = gpar; if (par.parent != 0xffffffffu) gpar = m.cols()[par.parent]; }
                    }
                } else {
                    break;                                   // backtracking failed
                }
                if (overflow) return 0;
            }
            if (cur_len) {
                if (n_ops >= (int)caps.aln_cigar - 4) { overflow = true; return 0; }
                m.bt_ops()[n_ops++] = cig_pack(cur_op, cur_len);
            }
            wsync();

            if (n_trace >= min_trace_length && n_path && path_back_nonzero) {
                const ColMeta cj = j ? col : m.cols()[0];
                score_t cur_cell_score = cellS(cj, pos - cj.trim);
                best_score = imax(best_score, wsub(score, cur_cell_score));
                if ((int64_t)score - min_cell_score < best_score) break;

                const ColMeta root = m.cols()[0];
                if (score >= min_start_score
                        && (!pos || cur_cell_score == 0)
                        && (pos || cur_cell_score == cellS(root, 0))
                        && (cfg.allow_left_trim || !j)) {
                    // construct_alignment (:774-798)
                    const AlnSlot o = m.slot(out_base + n_ext);
                    wsync();
                    for (int t = wlane(); t < n_path; t += kWarp) o.nodes[t] = m.bt_path()[n_path - 1 - t];
                    for (int t = wlane(); t < n_seq; t += kWarp) o.seq[t] = m.bt_seq()[n_seq - 1 - t];
                    int lead = start + pos;
                    int tail = L - start - end_pos;
                    int nc = 0;
                    if (lead) nc = 1;
                    for (int t = wlane(); t < n_ops; t += kWarp) o.cigar[nc + t] = m.bt_ops()[n_ops - 1 - t];
                    if (lead) o.cigar[0] = cig_pack(OP_S, lead);
                    nc += n_ops;
                    if (tail) o.cigar[nc++] = cig_pack(OP_S, tail);
                    AlnHdr h;
                    h.q_len = end_pos - pos; h.n_nodes = n_path; h.seq_len = n_seq; h.n_cigar = nc;
                    h.score = score; h.offset = align_offset; h.orientation = sh.orientation; h.used = 1;
                    *o.h = h;
                    wsync();
                    ++n_ext;
                }
            }
        }

        if (n_ext == 0 && sh.score >= min_path_score) {
            copy_slot(out_base, seed_slot);
            n_ext = 1;
        }
        return n_ext;
    }

    // --------------------------------------------------------------------------------
    // aggregator (aligner_aggregator.hpp:59-149, unlabeled queue)
    // Entry i lives in slot lay->slot_agg + i and its key in sm.agg()[i]: on the device lane i owns entry i (n_agg <=
    // kMaxAlt = kWarp), so a question about all entries is one pass and one warp collective; the one-lane emulation
    // runs the same loops over all entries.
    // --------------------------------------------------------------------------------
    MGB_HD static bool key_less(const AggKey &a, const AggKey &b) {      // LocalAlignmentLess
        if (a.score != b.score) return b.score > a.score;
        if (a.q_len != b.q_len) return a.q_len > b.q_len;
        if (a.orientation != b.orientation) return a.orientation > b.orientation;
        return a.clip > b.clip;
    }
    MGB_HD static bool key_same_hdr(const AggKey &a, const AggKey &b) {  // operator=='s fields before the arrays
        return a.orientation == b.orientation && a.offset == b.offset && a.score == b.score && a.q_len == b.q_len
            && a.seq_len == b.seq_len && a.n_cigar == b.n_cigar && a.n_nodes == b.n_nodes;
    }
    MGB_HD AggKey agg_key(const AlnSlot &a) const {
        const AlnHdr h = *a.h;
        AggKey k;
        k.score = h.score; k.q_len = h.q_len; k.orientation = h.orientation; k.clip = aln_clipping(a);
        k.offset = h.offset; k.seq_len = h.seq_len; k.n_cigar = h.n_cigar; k.n_nodes = h.n_nodes;
        return k;
    }
    // Alignment::operator== for two alignments whose keys pass key_same_hdr: query views, sequences, CIGARs, node paths
    MGB_HD bool aln_same_arrays(const AlnSlot &a, const AggKey &x, const AlnSlot &b, const AggKey &y) {
        bool diff = false;
        for (int i = wlane(); i < x.q_len; i += kWarp)
            if (cx[x.orientation].q[x.clip + i] != cx[y.orientation].q[y.clip + i]) diff = true;
        for (int i = wlane(); i < x.seq_len; i += kWarp) if (a.seq[i] != b.seq[i]) diff = true;
        for (int i = wlane(); i < x.n_cigar; i += kWarp) if (a.cigar[i] != b.cigar[i]) diff = true;
        for (int i = wlane(); i < x.n_nodes; i += kWarp) if (a.nodes[i] != b.nodes[i]) diff = true;
        return !wballot(diff);
    }
    // Position of entry i in a stable sort of the entries by LocalAlignmentLess: descending (get_alignments' order) or
    // ascending (position 0 is the entry std::min_element returns, the first of the minimal ones). An entry j comes
    // before i if it is strictly on i's side of the order or, being equivalent to i, has the lower index.
    MGB_HD int agg_rank(int i, bool desc) const {
        const AggKey *keys = sm.agg();
        const AggKey a = keys[i];
        int r = 0;
        for (int j = 0; j < n_agg; ++j) {
            if (j == i) continue;
            const AggKey b = keys[j];
            const AggKey &x = desc ? a : b, &y = desc ? b : a;
            r += j < i ? !key_less(y, x) : key_less(x, y);
        }
        return r;
    }
    MGB_HD score_t agg_global_cutoff() {
        if (!n_agg) return kNinf;
        // the score of std::max_element's entry is the largest score
        score_t mx = INT32_MIN;
        for (int i = wlane(); i < n_agg; i += kWarp) mx = imax(mx, sm.agg()[i].score);
        const score_t cur_max = wreduce_max(mx);
        return cur_max > 0 ? (score_t)((double)cur_max * cfg.rel_score_cutoff) : cur_max;
    }
    MGB_HD void agg_add(int slot) {
        const AlnSlot a = m.slot(slot);
        const AggKey nk = agg_key(a);
        AggKey *keys = sm.agg();
        const int agg0 = (int)m.lay->slot_agg;
        int dst = n_agg;
        if (n_agg) {
            if (nk.score < agg_global_cutoff()) return;
            // duplicates: a ballot of the entries whose header fields match, then the arrays of those only
            uint32_t cand = 0;
            for (int b = 0; b < n_agg; b += kWarp) {             // one pass on the device
                const int i = b + wlane();
                cand |= wballot(i < n_agg && key_same_hdr(keys[i], nk)) << b;
            }
            for (; cand; cand &= cand - 1) {
                const int i = ffs32(cand) - 1;
                if (aln_same_arrays(a, nk, m.slot(agg0 + i), keys[i])) { MGB_EMU_AGG(EMU_AGG_DUPLICATE); return; }
            }
            if (n_agg == (int)cfg.num_alternative_paths) {
                // *std::min_element(q_, cmp_) = alignment, unless alignment is smaller still
                uint32_t first = 0;
                for (int b = 0; b < n_agg; b += kWarp) {
                    const int i = b + wlane();
                    first |= wballot(i < n_agg && agg_rank(i, false) == 0) << b;
                }
                dst = ffs32(first) - 1;
                if (key_less(nk, keys[dst])) return;
                MGB_EMU_AGG(EMU_AGG_REPLACE);
            }
        }
        copy_slot(agg0 + dst, slot);
        keys[dst] = nk;
        if (dst == n_agg) ++n_agg;
        wsync();
    }
    MGB_HD score_t get_min_path_score() { return imax(cfg.min_path_score, agg_global_cutoff()); }

    // --------------------------------------------------------------------------------
    // drivers (dbg_aligner.cpp:360-384, 657-755)
    // --------------------------------------------------------------------------------
    // check_seed for a plain seed (Alignment(seed): last node, pos = |query_view| + clipping - 1, score)
    MGB_HD bool check_seed_rec(const ConvSlot *slots, const score_t *cells, uint32_t epoch, bool rc,
                               const uint64_t *nodes_s, const int32_t *pss, const SeedRec &sd) {
        uint64_t last_node = sd.n_nodes == 1 ? sd.node0 : nodes_s[sd.clip + sd.n_nodes - 1];
        int end_clip = L - (int)sd.clip - (int)sd.len;
        score_t score = pss[sd.clip] - pss[sd.clip + sd.len]
            + (!sd.clip ? cfg.left_end_bonus : 0) + (!end_clip ? cfg.right_end_bonus : 0);
        return check_seed_vals(slots, cells, epoch, rc, last_node, (int)sd.len + (int)sd.clip - 1, score);
    }

    MGB_HD void set_seed(int e) { conv_clear(e); }

    // Seeds of query strand s, in order (dbg_aligner.cpp:360-384 align_core when `both` is false,
    // :657-736 aln_both otherwise: forward extension, then backward extension of left-clipped
    // results through the reverse-complement graph view).
    MGB_HD void align_strand(int s, bool both) {
        const int fe = s, be = 1 - s;
        const int nk = L >= (int)ix.k ? L - (int)ix.k + 1 : 0;
        cx[fe].rc = 0;
        if (both) cx[be].rc = MGB_CANONICAL(cfg) ? 0 : 1;     // use_rcdbg (dbg_aligner.cpp:646-650)
        const int n_seeds_s = cx[s].n_seeds;
        SeedRec *seeds_s = cx[s].seeds;
        const bool implicit = cx[s].implicit_seeds != 0;
        stats.num_seeds += n_seeds_s;
        if (!n_seeds_s) return;
        int i = implicit ? mask_next(cx[s].mask, nk, 0, true) : 0;
        while (true) {
            // next live seed
            if (!implicit) while (i < n_seeds_s && !seeds_s[i].alive) ++i;
            if (overflow || (implicit ? i >= nk : i >= n_seeds_s)) break;
            SeedRec sd;
            if (implicit) {
                sd.clip = i; sd.len = ix.k; sd.offset = 0; sd.n_nodes = 1; sd.node0 = cx[s].qnodes[i];
                sd.alive = 1; sd.pad = 0;
            } else {
                sd = seeds_s[i];
            }
            seed_to_slot(SLOT_SEED, s, sd);
            seed_is_query = true;
            const score_t mps_fwd = both ? cfg.min_cell_score : get_min_path_score();
            // One call site for both kinds of extension (the forward one, then the backward ones it
            // spawns): the extender is by far the largest piece of code and must exist once.
            // A backward seed dropped by an earlier backward extension stays in its slot, unused: extend() does
            // nothing for it.
            const int bwd0 = (int)m.lay->slot_bwd;
            int n_rc = 0;
            for (int it = 0; !overflow && it <= n_rc; ++it) {
                const int r = it - 1;
                const bool ext_ok = it == 0 || m.slot(SLOT_EXT + r).h->used;
                if (it == 0) {
                    set_seed(fe);
                } else if (ext_ok) {
                    // align_core(ManualSeeder(rc_of_alignments), bwd_extender, ..., force_fixed_seed = true)
                    set_seed(be);
                    seed_is_query = false;
                }
                const int n_ext = extend(it ? be : fe, it ? SLOT_EXT + r : SLOT_SEED,
                                         (ext_ok && it) ? get_min_path_score() : mps_fwd, it != 0, it ? bwd0 : SLOT_EXT);
                // results of this extension: one loop (and one agg_add site: the aggregator's comparison
                // code is large) for the forward case (aggregate, then reverse-complement the clipped
                // ones for the backward pass) and the backward case (reverse-complement back, then aggregate)
                for (int r0 = 0; ext_ok && !overflow && r0 < n_ext; ++r0) {
                    const int slot = (it ? bwd0 : SLOT_EXT) + r0;
                    // is_reversible (:652-656): on a CANONICAL-mode graph an alignment to the reverse strand
                    // with no offset is reported as its reverse complement
                    const bool reversible = MGB_CANONICAL(cfg) && m.slot(slot).h->orientation && !m.slot(slot).h->offset;
                    // pass 0 reports the result, pass 1 (forward case only) turns a left-clipped result into
                    // a seed of the backward extension; both go through the one reverse-complement call site
                    #pragma unroll 1
                    for (int pass = 0; pass < 2; ++pass) {
                        bool add = false, need_rc;
                        int target = slot;
                        if (pass == 0) {
                            if (it == 0) {
                                add = !both || m.slot(slot).h->score >= get_min_path_score();
                                need_rc = add && reversible;              // :680-684
                                if (need_rc) { copy_slot(SLOT_TMP, slot); target = SLOT_TMP; }
                            } else {
                                need_rc = !MGB_CANONICAL(cfg) || reversible;   // use_rcdbg || is_reversible (:710-722)
                                add = true;
                            }
                        } else {
                            if (it != 0 || !both) break;
                            if (!aln_clipping(m.slot(slot)) || m.slot(slot).h->offset) break;
                            need_rc = true;
                        }
                        bool ok = true;
                        if (need_rc) ok = reverse_complement_for_bwd(target);
                        if (overflow) break;
                        if (!ok) break;                                   // the alignment cannot be reversed
                        if (pass == 0) {
                            if (it != 0 && need_rc) {
                                const AlnHdr h = *m.slot(slot).h;
                                int clip = aln_clipping(m.slot(slot)), eclip = aln_end_clipping(m.slot(slot));
                                for (int t = 0; t < h.n_nodes && !overflow; ++t)
                                    filter_nodes(fe, m.slot(slot).nodes[t], clip, L - eclip);
                            }
                            if (add) agg_add(target);
                        } else {
                            if (n_rc != r0) copy_slot(SLOT_EXT + n_rc, slot);
                            ++n_rc;
                        }
                    }
                }
                if (ext_ok && !overflow && it != 0) {
                    for (int r2 = r + 1; r2 < n_rc; ++r2) {
                        const AlnSlot a = m.slot(SLOT_EXT + r2);
                        if (!a.h->used) continue;
                        const AlnHdr h = *a.h;
                        if (!check_seed_vals(cx[be].conv_slots, cx[be].conv_cells, cx[be].conv_epoch, !MGB_CANONICAL(cfg) && cx[be].rc != 0,
                                             a.nodes[h.n_nodes - 1], h.q_len + aln_clipping(a) - 1, h.score))
                            a.h->used = 0;
                    }
                }
            }
            if (!overflow && shortcut_hit) {
                // exact-path shortcut: the extension it replaces covers every later seed of the strand (their last
                // node and position lie on the matched path with at least the seed's score, DESIGN.md)
                wsync();
                if (implicit) {
                    uint32_t *mask = cx[s].mask;
                    for (int w = i >> 5; 32 * w < nk; ++w) {
                        const uint32_t keep = 32 * w + 31 <= i ? ~0u : (32 * w > i ? 0u : ((2u << (i & 31)) - 1u));
                        mask[w] &= keep;
                    }
                } else {
                    for (int j = i + 1 + wlane(); j < n_seeds_s; j += kWarp) seeds_s[j].alive = 0;
                }
                shortcut_hit = false;
                wsync();
            } else if (!overflow) {
                // later seeds already covered by this extension are dropped (:731-734, :379-382);
                // independent probes, one seed per lane
                wsync();
                const ConvSlot *slots = cx[fe].conv_slots; const score_t *cells = cx[fe].conv_cells;
                const uint32_t epoch = cx[fe].conv_epoch;
                const uint64_t *nodes_s = cx[s].qnodes; const int32_t *pss = cx[s].ps;
                if (implicit) {
                    uint32_t *mask = cx[s].mask;
                    for (int w = (i + 1) >> 5; 32 * w < nk; ++w) {
                        const uint32_t word = mask[w];
                        uint32_t nw = 0;
                        for (int b = 0; b < 32; b += kWarp) {    // one pass on the device
                            const int bit = b + wlane();
                            const int jj = 32 * w + bit;
                            bool alive = jj > i && ((word >> bit) & 1u);
                            if (alive) {
                                SeedRec c; c.clip = jj; c.len = ix.k; c.offset = 0; c.n_nodes = 1;
                                c.node0 = nodes_s[jj]; c.alive = 1; c.pad = 0;
                                alive = check_seed_rec(slots, cells, epoch, false, nodes_s, pss, c);
                            }
                            nw |= wballot(alive) << b;
                        }
                        // bits at positions <= i in the first word stay as they are
                        if (32 * w <= i) { uint32_t lowmask = (i & 31) == 31 ? ~0u : ((2u << (i & 31)) - 1u); nw |= word & lowmask; }
                        mask[w] = nw;
                    }
                } else {
                    for (int j = i + 1 + wlane(); j < n_seeds_s; j += kWarp) {
                        if (seeds_s[j].alive && !check_seed_rec(slots, cells, epoch, false, nodes_s, pss, seeds_s[j]))
                            seeds_s[j].alive = 0;
                    }
                }
                wsync();
            }
            i = implicit ? mask_next(cx[s].mask, nk, i + 1, true) : i + 1;
        }
    }

    // suffix sums of the self-match scores (extender.cpp:26-36)
    MGB_HD void build_psum(int s) {
        // sequential suffix sum chunked over the warp
        int carry = 0;
        if (wlane() == 0) cx[s].ps[L] = 0;
        for (int base = L - 1; base >= 0; base -= kWarp) {
            int i = base - wlane();
            int v = i >= 0 ? cfg.diag[(uint8_t)cx[s].q[i]] : 0;
            v = wscan_add(v);
            v += carry;
            if (i >= 0) cx[s].ps[i] = v;
            carry = wbcast(v, kWarp - 1);
        }
        wsync();
    }

    // DNA block layout: scores of query position x (1-based, as prof_score) against A, C, G, T in one word, so that
    // the chain loop reads one shared-memory word per DP cell instead of the query character and then the table
    MGB_HD void build_prof4(int s) {
        uint32_t *p4 = sm.prof4(s);
        const char *q = cx[s].q;
        for (int x = wlane(); x < sm.lq() + 8; x += kWarp) {
            uint32_t w = 0;
            if (x >= 1 && x <= L) {
                const uint8_t ch = (uint8_t)q[x - 1];
                w = (uint32_t)(uint8_t)cfg.prof[1][ch] | ((uint32_t)(uint8_t)cfg.prof[2][ch] << 8)
                  | ((uint32_t)(uint8_t)cfg.prof[3][ch] << 16) | ((uint32_t)(uint8_t)cfg.prof[4][ch] << 24);
            }
            p4[x] = w;
        }
        wsync();
    }

    // whole pipeline for one read; returns the number of aggregator entries, sm.agg_ord() lists them in output order
    // optional: per-position index_range results of both strands (k_subk), set before run()
    const uint32_t *subk_first[2] = { nullptr, nullptr }, *subk_last[2] = { nullptr, nullptr };
    const uint8_t *subk_len[2] = { nullptr, nullptr };
    MGB_HD int run(int L_, const char *qf, const char *qr, const uint8_t *cf, const uint8_t *cr,
                   const uint64_t *nf, const uint64_t *nr) {
        MGB_TIC(t_setup);
        L = L_;
        overflow = false; n_agg = 0; seed_is_query = false;
        const bool both = cfg.forward_and_reverse_complement;
        wsync();
        // per-strand context + alignment slot table (shared memory; constant indices only here)
        {
            StrandCtx c0, c1;
            c0.q = qf; c1.q = qr; c0.codes = cf; c1.codes = cr; c0.qnodes = nf; c1.qnodes = nr;
            c0.ps = m.psum(0); c1.ps = m.psum(1);
            c0.seeds = m.seeds(0); c1.seeds = m.seeds(1);
            c0.conv_slots = m.conv_slots(0); c1.conv_slots = m.conv_slots(1);
            c0.conv_cells = m.conv_cells(0); c1.conv_cells = m.conv_cells(1);
            c0.conv_epoch = m.epoch_store()[0]; c1.conv_epoch = m.epoch_store()[1];
            c0.conv_n = c1.conv_n = 0; c0.conv_cells_used = c1.conv_cells_used = 0;
            c0.n_seeds = c1.n_seeds = 0; c0.num_matching = c1.num_matching = 0;
            c0.table_cap = c1.table_cap = 0; c0.num_ext = c1.num_ext = 0;
            c0.explored_prev = c1.explored_prev = 0; c0.rc = c1.rc = 0;
            c0.implicit_seeds = c1.implicit_seeds = 0; c0.mask = sm.mask0(); c1.mask = sm.mask1();
            c0.sub_first = subk_first[0]; c0.sub_last = subk_last[0]; c0.sub_len = subk_len[0];
            c1.sub_first = subk_first[1]; c1.sub_last = subk_last[1]; c1.sub_len = subk_len[1];
            // stage the query strands (and their suffix sums) on chip when they fit
            if (L + 1 <= sm.lq()) {
                for (int i = wlane(); i < L; i += kWarp) { sm.q0()[i] = qf[i]; sm.q1()[i] = qr[i]; }
                c0.q = sm.q0(); c1.q = sm.q1(); c0.ps = sm.psum0(); c1.ps = sm.psum1();
            } else MGB_EMU_HIT(EMU_UNSTAGED_READ);
            sm.ctx()[0] = c0; sm.ctx()[1] = c1;
        }
        wsync();
        stats.num_seeds = stats.num_extensions = stats.num_explored_nodes = stats.dp_columns = 0;
        stats.dp_cells = 0;
        if (MGB_CANONICAL(cfg) && MGB_PRIMARY(ix) && L >= (int)ix.k) {
            // CanonicalDBG::map_to_nodes_sequentially (:55-146) from the two per-strand maps of the stored k-mers: a
            // k-mer missing on its own strand takes the id of its reverse complement + n; the other strand's path is
            // the flipped one (reverse_complement_seq_path, dbg_aligner.cpp:224-230). Idempotent (overflow retries).
            uint64_t *nf_w = const_cast<uint64_t*>(cx[0].qnodes), *nr_w = const_cast<uint64_t*>(cx[1].qnodes);
            const int nk = L - (int)ix.k + 1;
            wsync();
            for (int i = wlane(); i < nk; i += kWarp) {
                const uint64_t f = nf_w[i], r = nr_w[nk - 1 - i];
                const uint64_t mf = f ? f : (r ? (r > ix.n ? r : r + ix.n) : 0);
                nf_w[i] = mf;
                nr_w[nk - 1 - i] = mf ? canon_flip(mf) : 0;
            }
            wsync();
        }
        build_psum(0);
        if (both) build_psum(1);
        if (!MGB_WIDE(ix) && sm.lay->has_prof && L + 1 <= sm.lq()) { build_prof4(0); if (both) build_prof4(1); }
        if (cfg.seed_complexity_filter) { build_lowcx(0); if (both) build_lowcx(1); }
        MGB_TOC(t_setup, 0);
        MGB_TIC(t_seeds);
        #pragma unroll 1
        for (int s = 0; s < (both ? 2 : 1) && !overflow; ++s) {           // one call site: the seeder is large
            build_seeds(s);
            if (overflow) break;
            if ((double)L * cfg.min_exact_match > (double)cx[s].num_matching) { cx[s].n_seeds = 0; cx[s].num_matching = 0; }
        }
        int first = 0, n_pass = 1;
        if (both) {
            // the strand with more exact-match bases first; the other only if it is close (:738-755)
            uint32_t fm = cx[0].num_matching, bm = cx[1].num_matching;
            first = fm >= bm ? 0 : 1;
            uint32_t hi = first ? bm : fm, lo = first ? fm : bm;
            n_pass = (double)lo >= (double)hi * cfg.rel_score_cutoff ? 2 : 1;
        }
        MGB_TOC(t_seeds, 1);
        MGB_TIC(t_align);
        for (int pass = 0; !overflow && pass < n_pass; ++pass)
            align_strand(pass ? 1 - first : first, both);
        MGB_TOC(t_align, 4);
        if (overflow) return 0;
        stats.num_extensions += cx[0].num_ext + cx[1].num_ext;
        stats.num_explored_nodes += cx[0].explored_prev + cx[0].conv_n + cx[1].explored_prev + cx[1].conv_n;
        // AlignmentAggregator::get_alignments: descending LocalAlignmentLess order, ties in entry order
        for (int i = wlane(); i < n_agg; i += kWarp) sm.agg_ord()[agg_rank(i, true)] = i;
        wsync();
        return n_agg;
    }
};

#if MGB_DEVICE_CODE
static __device__ __forceinline__
#else
static inline
#endif
void chain_entry(const IndexView &ix, const DevConfig &cfg, const Caps &caps, const WarpMem &m, const WarpSmem &sm, int L,
                 ChainIO *io) {
    ReadAligner al(ix, cfg, caps, m, sm);
    al.L = L;
    al.chain_loop(*io);
}

} // namespace mgb
