// FASTA/FASTQ records parsed on the device (mgb_align_fastx_text): one chunk of raw file bytes becomes the packed
// seqs/offsets and names/name_offsets arrays the align route and the text kernels read, without leaving device memory.
//
// A chunk is parsed in parallel when it has one of two forms, decided line by line (DESIGN.md §8):
//   FASTA form: no complete line starts with '+'; line 0 and every line that starts with '>' or '@' is a header, every
//               other line (empty ones included) is sequence;
//   4-line FASTQ form: line 4i starts with '@', line 4i+1 is non-empty and starts with none of '>', '@', '+', line 4i+2
//               starts with '+', line 4i+3 is as long as line 4i+1.
// In both, a record is what kseq_read returns for it (fastx_host.hpp restates kseq_read for every other chunk). Line
// lengths follow the CR rule: one '\r' before a line's end is not part of the line.
//
// Steps: k_fastx_count / k_fastx_lines find the '\n' of each 4 KiB tile (16-byte loads) and write their positions;
// k_fastx_classify checks every line against both forms; k_fastx_roles gives each line of the chosen form its header
// flag, sequence bytes and header bytes, which are scanned; k_fastx_records (FASTA) lists the header lines; k_fastx_gather
// copies each record's header and sequence lines with a warp, and with MGB_FASTX_FWD_AND_REVERSE its reverse complement
// after it. Byte positions in a chunk are 32-bit: a chunk is shorter than 4 GiB.
#pragma once
#include <stdint.h>
#include "common.cuh"

namespace mgb {

constexpr uint32_t kFastxTile = 4096;             // bytes per block of the line scan: 256 threads x 16 bytes
constexpr uint32_t kFastxMaxDelim = 32;           // --header-comment-delim bytes the device route copies
constexpr uint32_t kFastxFastaBad = 1, kFastxFastqBad = 2;

// isspace() in the C locale: what ends a record's name (kseq_read reads the name with KS_SEP_SPACE)
MGB_HOSTDEV bool fastx_space(uint8_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

// the complement reverse_complement() applies (seq_tools/reverse_complement.hpp): A/T, C/G and the IUPAC pairs B/V,
// D/H, K/M, R/Y in both cases, U -> A, '`' -> '@', every other byte unchanged
MGB_HOSTDEV uint8_t fastx_complement(uint8_t c) {
    const uint8_t u = c & 0xDF, low = c & 0x20;
    if (c == '`') return '@';
    if (c < 'A' || (c > 'Z' && c < 'a') || c > 'z') return c;
    uint8_t r = u;
    switch (u) {
        case 'A': r = 'T'; break;
        case 'T': case 'U': r = 'A'; break;
        case 'C': r = 'G'; break;
        case 'G': r = 'C'; break;
        case 'B': r = 'V'; break;
        case 'V': r = 'B'; break;
        case 'D': r = 'H'; break;
        case 'H': r = 'D'; break;
        case 'K': r = 'M'; break;
        case 'M': r = 'K'; break;
        case 'R': r = 'Y'; break;
        case 'Y': r = 'R'; break;
        default: break;
    }
    return (uint8_t)(r | low);
}

// what k_fastx_classify leaves for the host (zeroed before it runs)
struct FastxSummary {
    uint32_t flags;          // kFastxFastaBad | kFastxFastqBad
    uint32_t n_hdr;          // FASTA form: header lines (the partial last line included)
    uint32_t last_hdr;       // FASTA form: 1 + byte where the last header line starts (0: none)
    uint32_t q_cut;          // FASTQ form: 1 + byte where line 4 * (complete lines / 4) starts (0: no such line)
};

struct FastxArgs {
    const uint8_t *buf; uint32_t n; uint32_t at_eof;
    uint32_t n_tiles;
    uint64_t *tile_nl;       // per tile: '\n' count, then (scanned) the first '\n' index of the tile; [n_tiles] = total
    uint32_t *nl;            // line i ends at nl[i] (its '\n', or n for the partial last line); nl[n_nl] = n
    uint32_t n_nl, n_lines;
    FastxSummary *sum;
    int fastq;               // the form k_fastx_roles and k_fastx_gather apply
    uint64_t *lh, *ls, *ln;  // per line: header flag, sequence bytes, header bytes; after the scans their offsets
    uint32_t *rec_line;      // FASTA: header line of record r; [n_hdr] = n_lines
    uint32_t n_rec, fwd_rev;
    char delim[kFastxMaxDelim]; uint32_t dlen; int has_delim;
    char *seqs; uint64_t *offsets; char *names; uint64_t *name_offsets;
};

MGB_HOSTDEV uint32_t fastx_line_begin(const FastxArgs &a, uint32_t i) { return i ? a.nl[i - 1] + 1 : 0; }

// the line [b, e) without the '\r' the CR rule drops
MGB_HOSTDEV uint32_t fastx_content_end(const FastxArgs &a, uint32_t b, uint32_t e) {
    return e > b && a.buf[e - 1] == '\r' ? e - 1 : e;
}

// a header line's name [b + 1, *name_end) and comment [*com_b, ce): kseq_read's name ends at the first isspace byte,
// the comment is the rest of the line
MGB_HOSTDEV void fastx_header_parts(const FastxArgs &a, uint32_t b, uint32_t ce, uint32_t *name_end, uint32_t *com_b) {
    uint32_t q = b + 1;
    while (q < ce && !fastx_space(a.buf[q])) ++q;
    *name_end = q;
    *com_b = q < ce ? q + 1 : ce;
}

// the header as `metagraph align` prints it: the name, or utils::join_strings({name, comment}, delim, true) when a
// delimiter is given and the comment is not empty (cli/align.cpp:430-435)
MGB_HOSTDEV uint32_t fastx_header_bytes(const FastxArgs &a, uint32_t name_len, uint32_t com_len) {
    if (!a.has_delim || !com_len) return name_len;
    return name_len ? name_len + a.dlen + com_len : com_len;
}

// line i against both forms
MGB_HOSTDEV void fastx_classify_line(const FastxArgs &a, uint32_t i, uint32_t *bad, bool *hdr_a, uint32_t *q_cut) {
    const uint32_t b = fastx_line_begin(a, i), e = a.nl[i], raw = e - b;
    const int f = raw ? a.buf[b] : -1;
    const bool complete = i < a.n_nl || a.at_eof;
    const uint32_t clen = fastx_content_end(a, b, e) - b;
    const bool hdr = f == '>' || f == '@';
    *hdr_a = hdr;
    if (complete && f == '+') *bad |= kFastxFastaBad;
    if (i == 0 && !hdr) *bad |= kFastxFastaBad;
    // a header byte that ends the input: kseq_read reads no name and returns -1 (the host restatement decides)
    if (a.at_eof && i >= a.n_nl && raw == 1 && hdr) *bad |= kFastxFastaBad;
    const uint32_t n_complete = a.at_eof ? a.n_lines : a.n_nl;
    if (i == n_complete / 4 * 4) *q_cut = b + 1;
    if (!complete) return;
    switch (i & 3) {
        case 0: if (f != '@') *bad |= kFastxFastqBad; break;
        case 1: if (!clen || f == '>' || f == '@' || f == '+') *bad |= kFastxFastqBad; break;
        case 2: if (f != '+') *bad |= kFastxFastqBad; break;
        default: {
            const uint32_t sb = fastx_line_begin(a, i - 2);
            if (clen != fastx_content_end(a, sb, a.nl[i - 2]) - sb) *bad |= kFastxFastqBad;
        }
    }
    if (i == 0 && a.at_eof && n_complete % 4) *bad |= kFastxFastqBad;
}

// line i of the chosen form: header flag, sequence bytes, header bytes
MGB_HOSTDEV void fastx_role_line(const FastxArgs &a, uint32_t i) {
    const uint32_t b = fastx_line_begin(a, i), e = a.nl[i];
    const uint32_t ce = fastx_content_end(a, b, e);
    const int f = e > b ? a.buf[b] : -1;
    const bool hdr = a.fastq ? (i & 3) == 0 : f == '>' || f == '@';
    uint64_t s = 0, h = 0;
    if (hdr) {
        uint32_t name_end, com_b;
        fastx_header_parts(a, b, ce, &name_end, &com_b);
        h = fastx_header_bytes(a, name_end - b - 1, ce - com_b);
    } else if (!a.fastq || (i & 3) == 1) {
        s = ce - b;
    }
    a.lh[i] = hdr; a.ls[i] = s; a.ln[i] = h;
}

// record r with one warp: its header and sequence lines into the packed arrays, and the offsets of the copies
MGB_HD void fastx_gather_record(const FastxArgs &a, uint32_t r) {
    const uint32_t h = a.fastq ? 4 * r : a.rec_line[r];
    const uint32_t h2 = a.fastq ? 4 * r + 2 : a.rec_line[r + 1];
    const uint64_t S = a.ls[h], S2 = a.ls[h2], N = a.ln[h], N2 = a.ln[h + 1];
    const uint64_t len = S2 - S, nlen = N2 - N;
    const int copies = a.fwd_rev ? 2 : 1;
    const uint64_t sb = copies * S, nb = copies * N;      // where the record's forward copy starts
    const int lane = wlane();
    if (lane == 0) {
        const uint64_t o = (uint64_t)copies * r;
        a.offsets[o] = sb; a.name_offsets[o] = nb;
        if (a.fwd_rev) { a.offsets[o + 1] = sb + len; a.name_offsets[o + 1] = nb + nlen; }
        if (r + 1 == a.n_rec) { a.offsets[o + copies] = sb + copies * len; a.name_offsets[o + copies] = nb + copies * nlen; }
    }
    // header: name, then delimiter and comment (fastx_header_bytes)
    const uint32_t hb = fastx_line_begin(a, h), hce = fastx_content_end(a, hb, a.nl[h]);
    uint32_t name_end, com_b;
    fastx_header_parts(a, hb, hce, &name_end, &com_b);
    const uint32_t name_len = name_end - hb - 1, com_len = hce - com_b;
    const bool with_com = a.has_delim && com_len;
    const uint32_t d_at = name_len, c_at = with_com && name_len ? name_len + a.dlen : 0;
    for (int c = 0; c < copies; ++c) {
        char *dst = a.names + nb + (uint64_t)c * nlen;
        if (!with_com || name_len)
            for (uint32_t t = lane; t < name_len; t += kWarp) dst[t] = (char)a.buf[hb + 1 + t];
        if (with_com) {
            if (name_len) for (uint32_t t = lane; t < a.dlen; t += kWarp) dst[d_at + t] = a.delim[t];
            for (uint32_t t = lane; t < com_len; t += kWarp) dst[c_at + t] = (char)a.buf[com_b + t];
        }
    }
    // sequence lines (h, h2)
    char *fwd = a.seqs + sb, *rc = a.seqs + sb + len;
    for (uint32_t j = h + 1; j < h2; ++j) {
        const uint32_t b = fastx_line_begin(a, j), ce = fastx_content_end(a, b, a.nl[j]);
        const uint64_t q = a.ls[j] - S;
        for (uint32_t t = lane; t < ce - b; t += kWarp) {
            const uint8_t x = a.buf[b + t];
            fwd[q + t] = (char)x;
            if (a.fwd_rev) rc[len - 1 - (q + t)] = (char)fastx_complement(x);
        }
    }
}

#if MGB_DEVICE_CODE
MGB_D uint32_t fastx_nl16(const uint8_t *buf, uint32_t n, uint32_t at, uint32_t *mask) {
    const uint4 w = *reinterpret_cast<const uint4*>(buf + at);
    const uint32_t x[4] = { w.x, w.y, w.z, w.w };
    uint32_t m = 0;
    #pragma unroll
    for (int j = 0; j < 4; ++j) {
        // bytes equal to '\n': zero bytes of x ^ 0x0a0a0a0a
        const uint32_t v = x[j] ^ 0x0a0a0a0au;
        const uint32_t z = __vcmpeq4(v, 0u);             // 0xff per matching byte
        m |= ((z & 0x01u) | ((z >> 7) & 0x02u) | ((z >> 14) & 0x04u) | ((z >> 21) & 0x08u)) << (4 * j);
    }
    if (at + 16 > n) m &= at >= n ? 0u : (1u << (n - at)) - 1u;
    *mask = m;
    return __popc(m);
}

// per tile: number of '\n'
__global__ void __launch_bounds__(256) k_fastx_count(const __grid_constant__ FastxArgs a) {
    __shared__ uint32_t part[8];
    for (uint32_t tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        uint32_t m;
        uint32_t c = fastx_nl16(a.buf, a.n, tile * kFastxTile + threadIdx.x * 16, &m);
        for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = c;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t s = 0;
            for (int w = 0; w < 8; ++w) s += part[w];
            a.tile_nl[tile] = s;
        }
        __syncthreads();
    }
}

// the '\n' positions of every tile at the tile's scanned offset; nl[n_nl] = n
__global__ void __launch_bounds__(256) k_fastx_lines(const __grid_constant__ FastxArgs a) {
    __shared__ uint32_t part[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const uint32_t at = tile * kFastxTile + threadIdx.x * 16;
        uint32_t m;
        const uint32_t c = fastx_nl16(a.buf, a.n, at, &m);
        uint32_t x = c;                                   // inclusive scan within the warp
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
        if (lane == 31) part[warp] = x;
        __syncthreads();
        uint32_t before = 0;
        for (int w = 0; w < warp; ++w) before += part[w];
        uint64_t o = a.tile_nl[tile] + before + x - c;
        while (m) { const int j = __ffs(m) - 1; a.nl[o++] = at + j; m &= m - 1; }
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.nl[a.n_nl] = a.n;
}

__global__ void __launch_bounds__(256) k_fastx_classify(const __grid_constant__ FastxArgs a) {
    uint32_t bad = 0, n_hdr = 0, last = 0, q_cut = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_lines; i += gridDim.x * blockDim.x) {
        bool hdr;
        fastx_classify_line(a, i, &bad, &hdr, &q_cut);
        if (hdr) { ++n_hdr; last = fastx_line_begin(a, i) + 1 > last ? fastx_line_begin(a, i) + 1 : last; }
    }
    for (int d = 16; d; d >>= 1) {
        bad |= __shfl_xor_sync(0xffffffffu, bad, d);
        n_hdr += __shfl_xor_sync(0xffffffffu, n_hdr, d);
        const uint32_t l = __shfl_xor_sync(0xffffffffu, last, d); last = l > last ? l : last;
        const uint32_t q = __shfl_xor_sync(0xffffffffu, q_cut, d); q_cut = q > q_cut ? q : q_cut;
    }
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicOr(&a.sum->flags, bad);
        if (n_hdr) atomicAdd(&a.sum->n_hdr, n_hdr);
        if (last) atomicMax(&a.sum->last_hdr, last);
        if (q_cut) atomicMax(&a.sum->q_cut, q_cut);
    }
}

__global__ void __launch_bounds__(256) k_fastx_roles(const __grid_constant__ FastxArgs a) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_lines; i += gridDim.x * blockDim.x)
        fastx_role_line(a, i);
}

// FASTA: record lh[i] starts at header line i
__global__ void __launch_bounds__(256) k_fastx_records(const __grid_constant__ FastxArgs a) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_lines; i += gridDim.x * blockDim.x)
        if (a.lh[i + 1] != a.lh[i]) a.rec_line[a.lh[i]] = i;
    if (blockIdx.x == 0 && threadIdx.x == 0) a.rec_line[a.lh[a.n_lines]] = a.n_lines;
}

// Exclusive scan of a per-line array over the whole grid, in tiles of kFastxScanTile elements: k_fastx_scan_up sums each
// tile with coalesced loads, the tile sums are scanned, and k_fastx_scan_down scans each tile in shared memory from its
// tile's offset and writes it back coalesced. The per-line arrays hold millions of elements per chunk; one block reading
// a contiguous segment per thread (k_text_scan) took 17.5 ms of the parse's 18.7 ms device time per 1 M FASTQ reads on
// an H100 (DESIGN.md §6).
constexpr uint32_t kFastxScanTile = 4096;        // 256 threads x 16 elements

__global__ void __launch_bounds__(256) k_fastx_scan_up(const uint64_t *v, uint32_t n, uint64_t *tile_sum) {
    __shared__ uint64_t part[8];
    const uint64_t base = (uint64_t)blockIdx.x * kFastxScanTile;
    uint64_t x = 0;
    #pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint64_t i = base + j * 256 + threadIdx.x;
        if (i < n) x += v[i];
    }
    for (int d = 16; d; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t t = 0;
        for (int w = 0; w < 8; ++w) t += part[w];
        tile_sum[blockIdx.x] = t;
    }
}

// tile_sum: scanned (tile_sum[n_tiles] = total, which goes to v[n])
__global__ void __launch_bounds__(256) k_fastx_scan_down(uint64_t *v, uint32_t n, const uint64_t *tile_sum,
                                                         uint32_t n_tiles) {
    __shared__ uint64_t s[kFastxScanTile + kFastxScanTile / 16];     // one pad word per thread's 16: fewer conflicts
    __shared__ uint64_t part[8];
    const uint64_t base = (uint64_t)blockIdx.x * kFastxScanTile;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    auto at = [](uint32_t i) { return i + (i >> 4); };
    #pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint32_t i = j * 256 + t;
        s[at(i)] = base + i < n ? v[base + i] : 0;
    }
    __syncthreads();
    uint64_t x = 0;
    #pragma unroll
    for (int j = 0; j < 16; ++j) x += s[at(t * 16 + j)];
    uint64_t inc = x;
    for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += y; }
    if (lane == 31) part[warp] = inc;
    __syncthreads();
    uint64_t run = tile_sum[blockIdx.x] + inc - x;
    for (int w = 0; w < warp; ++w) run += part[w];
    #pragma unroll
    for (int j = 0; j < 16; ++j) { const uint64_t y = s[at(t * 16 + j)]; s[at(t * 16 + j)] = run; run += y; }
    __syncthreads();
    #pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint32_t i = j * 256 + t;
        if (base + i < n) v[base + i] = s[at(i)];
    }
    if (blockIdx.x == 0 && t == 0) v[n] = tile_sum[n_tiles];
}

// one warp per record
__global__ void __launch_bounds__(256) k_fastx_gather(const __grid_constant__ FastxArgs a) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, nw = gridDim.x * blockDim.x / 32;
    for (uint32_t r = warp; r < a.n_rec; r += nw) fastx_gather_record(a, r);
}
#endif

} // namespace mgb
