// Device-resident batches (mgb_align_batch_device): the two per-read host steps of the record route done on the device.
//
//   k_pass_classify  after an align pass, over the pass's reads: a finished read's pass id goes into pass_of, a read
//                    that overflowed its arena is appended to the retry list (warp-aggregated), and the search
//                    counters of the finished reads are summed into a PassSummary, the only thing the host reads back
//                    when no read overflowed. The record and text routes run the same classify_read on the host.
//   k_columns_size   after the last pass, one warp per read: the read's alignments, sequence bytes, CIGAR ops and node
//                    ids, walking its records in the heap of the pass that answered it.
//   k_columns_write  after the four scans of those counts, one warp per read: the records as the caller's columns
//                    (mgb_device_columns_t), the fixed fields by lane 0, the ragged arrays spread over the lanes.
//
// The host emulation (MGB_HOST_EMU) runs the same per-read functions in loops.
#pragma once
#include <string.h>
#include "common.cuh"
#include "kernels.cuh"
#include "../../include/mgb.h"

namespace mgb {

constexpr int kColumnsMaxPasses = 8;    // heaps a batch can be answered from (api.cu kMaxPasses)

// a pass's classification: the counters of the finished reads, how many reads overflowed and the longest of them (it
// sizes the next pass's arena); on the device route the host reads back only this after a pass with no overflow
struct PassSummary {
    unsigned long long num_seeds, num_extensions, num_explored_nodes, dp_cells, dp_columns;
    unsigned int n_retry, max_retry_len;
};
static_assert(sizeof(PassSummary) == 48, "PassSummary is what crosses PCIe per pass");

struct ClassifyArgs {
    const uint32_t *list; uint32_t n_list;     // the pass's reads; list == nullptr: reads 0 .. n_list - 1
    const ReadHdr *hdr; const uint64_t *offsets;
    uint8_t *pass_of; uint32_t pass;
    PassSummary *sum; uint32_t *retry;         // sum zeroed before the launch; retry holds n_list entries
};

// read r of the pass: true when it overflowed (the caller appends it); otherwise its pass and counters are recorded
MGB_HOSTDEV bool classify_read(const ClassifyArgs &a, uint32_t r, PassSummary &acc) {
    const ReadHdr h = a.hdr[r];
    if (h.status == MGB_READ_OVERFLOW) {
        const uint32_t L = (uint32_t)(a.offsets[r + 1] - a.offsets[r]);
        if (L > acc.max_retry_len) acc.max_retry_len = L;
        return true;
    }
    a.pass_of[r] = (uint8_t)a.pass;
    acc.num_seeds += h.stats.num_seeds; acc.num_extensions += h.stats.num_extensions;
    acc.num_explored_nodes += h.stats.num_explored_nodes; acc.dp_cells += h.stats.dp_cells;
    acc.dp_columns += h.stats.dp_columns;
    return false;
}

struct ColumnsArgs {
    const ReadHdr *hdr; const uint8_t *pass_of;
    const char *heap[kColumnsMaxPasses];
    uint32_t n_reads, no_nodes;
    // per read: alignments, sequence bytes, CIGAR ops, node ids; after the scans the read's first element of each,
    // cnt[i][n_reads] the totals
    uint64_t *cnt[4];
    mgb_device_columns_t dst;                 // k_columns_write
};

MGB_HD const char *read_records(const ColumnsArgs &a, uint32_t r) {
    return a.heap[a.pass_of[r]] + a.hdr[r].heap_off;
}

// every lane walks the read's records (the loads are broadcasts); lane 0 stores the counts
MGB_HD void columns_size_read(const ColumnsArgs &a, uint32_t r) {
    const uint32_t n = a.hdr[r].n_aln;
    uint64_t seq = 0, cig = 0, nodes = 0;
    const char *p = n ? read_records(a, r) : nullptr;
    for (uint32_t i = 0; i < n; ++i) {
        RecView v;
        p = rec_next(p, a.no_nodes, &v);
        seq += v.o.seq_len; cig += v.o.n_cigar; nodes += a.no_nodes ? 0 : v.o.n_nodes;
    }
    if (wlane() == 0) { a.cnt[0][r] = n; a.cnt[1][r] = seq; a.cnt[2][r] = cig; a.cnt[3][r] = nodes; }
}

// dst[0, n) = src[0, n) over the lanes of a warp: elements up to dst's first 16-byte boundary one by one, then one
// 16-byte store per lane and round, built from element loads (src, in the heap, is only 8-byte aligned), then the tail
template <class T> MGB_HD void warp_copy(T *dst, const T *src, uint64_t n) {
    constexpr uint64_t E = 16 / sizeof(T);
    uint64_t head = ((16 - ((uintptr_t)dst & 15)) & 15) / sizeof(T);
    if (head > n) head = n;
    for (uint64_t i = wlane(); i < head; i += kWarp) dst[i] = src[i];
    const uint64_t words = (n - head) / E;
    for (uint64_t w = wlane(); w < words; w += kWarp) {
#if MGB_DEVICE_CODE
        union { T e[E]; uint4 v; } u;
#else
        struct { T e[E]; } u;
#endif
        const T *s = src + head + w * E;
        for (uint64_t e = 0; e < E; ++e) u.e[e] = s[e];
#if MGB_DEVICE_CODE
        *reinterpret_cast<uint4*>(dst + head + w * E) = u.v;
#else
        memcpy(dst + head + w * E, u.e, 16);
#endif
    }
    for (uint64_t i = head + words * E + wlane(); i < n; i += kWarp) dst[i] = src[i];
}

MGB_HD void columns_write_read(const ColumnsArgs &a, uint32_t r) {
    const mgb_device_columns_t &d = a.dst;
    const uint32_t n = a.hdr[r].n_aln;
    const uint64_t j0 = a.cnt[0][r];
    uint64_t seq = a.cnt[1][r], cig = a.cnt[2][r], nodes = a.cnt[3][r];
    if (wlane() == 0) d.read_first[r] = j0;
    const char *p = n ? read_records(a, r) : nullptr;
    for (uint32_t i = 0; i < n; ++i) {
        RecView v;
        p = rec_next(p, a.no_nodes, &v);
        const uint64_t j = j0 + i;
        if (wlane() == 0) {
            d.read_index[j] = r; d.orientation[j] = (uint8_t)v.o.orientation; d.score[j] = v.o.score;
            d.offset[j] = v.o.offset; d.query_begin[j] = v.o.query_begin; d.query_len[j] = v.o.query_len;
            d.num_nodes[j] = v.o.n_nodes; d.sequence_len[j] = v.o.seq_len; d.num_cigar_ops[j] = v.o.n_cigar;
            d.sequence_offsets[j] = seq; d.cigar_offsets[j] = cig; d.node_offsets[j] = nodes;
        }
        warp_copy(d.sequence + seq, v.seq, v.o.seq_len);
        warp_copy(d.cigar + cig, v.cigar, v.o.n_cigar);
        if (!a.no_nodes) warp_copy(d.nodes + nodes, v.nodes, v.o.n_nodes);
        seq += v.o.seq_len; cig += v.o.n_cigar; nodes += a.no_nodes ? 0 : v.o.n_nodes;
    }
}

// the closing entries: read_first[n_reads] and the three offset arrays at [n_alignments]
MGB_HD void columns_write_ends(const ColumnsArgs &a) {
    const uint64_t n_aln = a.cnt[0][a.n_reads];
    a.dst.read_first[a.n_reads] = n_aln;
    a.dst.sequence_offsets[n_aln] = a.cnt[1][a.n_reads];
    a.dst.cigar_offsets[n_aln] = a.cnt[2][a.n_reads];
    a.dst.node_offsets[n_aln] = a.cnt[3][a.n_reads];
}

#if MGB_DEVICE_CODE
// a lane per read of the list; every lane of a warp runs the same rounds, so the ballot sees the whole warp
__global__ void __launch_bounds__(256) k_pass_classify(const __grid_constant__ ClassifyArgs a) {
    PassSummary acc;
    memset(&acc, 0, sizeof(acc));
    const uint32_t lane = threadIdx.x & 31, stride = gridDim.x * blockDim.x;
    for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < a.n_list; base += stride) {
        const uint32_t t = base + lane;
        uint32_t r = 0;
        bool over = false;
        if (t < a.n_list) { r = a.list ? a.list[t] : t; over = classify_read(a, r, acc); }
        const unsigned m = __ballot_sync(0xffffffffu, over);
        if (!m) continue;
        uint32_t at = 0;
        if (lane == 0) at = atomicAdd(&a.sum->n_retry, (unsigned)__popc(m));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (over) a.retry[at + __popc(m & ((1u << lane) - 1))] = r;
    }
    unsigned long long *c = &acc.num_seeds;
    for (int i = 0; i < 5; ++i)
        for (int o = 16; o; o >>= 1) c[i] += __shfl_xor_sync(0xffffffffu, c[i], o);
    for (int o = 16; o; o >>= 1) acc.max_retry_len = max(acc.max_retry_len, __shfl_xor_sync(0xffffffffu, acc.max_retry_len, o));
    if (lane == 0) {
        unsigned long long *s = &a.sum->num_seeds;
        for (int i = 0; i < 5; ++i) if (c[i]) atomicAdd(s + i, c[i]);
        if (acc.max_retry_len) atomicMax(&a.sum->max_retry_len, acc.max_retry_len);
    }
}

__global__ void __launch_bounds__(256) k_columns_size(const __grid_constant__ ColumnsArgs a) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp, nw = (gridDim.x * blockDim.x) / kWarp;
    for (uint32_t r = warp; r < a.n_reads; r += nw) columns_size_read(a, r);
}

__global__ void __launch_bounds__(256) k_columns_write(const __grid_constant__ ColumnsArgs a) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp, nw = (gridDim.x * blockDim.x) / kWarp;
    if (blockIdx.x == 0 && threadIdx.x == 0) columns_write_ends(a);
    for (uint32_t r = warp; r < a.n_reads; r += nw) columns_write_read(a, r);
}
#endif

} // namespace mgb
