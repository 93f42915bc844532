// Ordinary gzip members inflated on the device (mgb_fastx_stage_gzip, mgb_gzip_inflate): one DEFLATE stream decoded
// from many points at once (DESIGN.md §8 "Plain gzip input").
//
// A stage's compressed bits, from the stream's position `start`, are split into sub-ranges of sub_bits. Sub-range 0
// starts at `start`, a true block boundary. For every later one, k_gzip_find looks for the first bit offset that parses
// as a dynamic-Huffman block header (a lane prefilter over kWarp consecutive offsets, then bgzf_dynamic's full check
// on a survivor). k_gzip_decode then decodes every sub-range with a candidate, one warp each, with the decoder of
// bgzf_core.cuh writing 16-bit symbols: a byte, or a marker 0x8000 | i for byte i of the 32 KiB window before the
// sub-range's start, which is not known yet. Each decode stops at the first block end at or past the next candidate,
// at a final block, or keeps the last block end it reached when it fails. The host confirms the chain from sub-range
// 0 (a sub-range is confirmed when a confirmed decode ended exactly at its candidate), so a false candidate can only
// shorten a stage. k_gzip_window then resolves the 32 KiB windows along the confirmed chain, k_gzip_resolve turns the
// symbols into text, and k_gzip_crc computes CRC32 parts of it for the host to combine.
#pragma once
#include "bgzf_core.cuh"

namespace mgb {

constexpr uint32_t kGzipWindow = 32768;
constexpr uint64_t kGzipNone = ~0ull;            // no candidate in the sub-range
constexpr uint32_t kGzipCrcPiece = 4096;         // text bytes per CRC32 part
constexpr int kGzipWarps = 4;                    // warps per block of k_gzip_find / k_gzip_decode
// decode results besides the decoder's own (kBgzfBadStream: invalid, kBgzfBadSize: the slot is full)
enum : uint32_t { kGzipStop = 0, kGzipFinal = 4, kGzipShort = 5, kGzipSkipped = 6 };

// one sub-range's decode: it stopped at bit `end`, a block end, with `len` symbols; reach: how far before its start a
// back-reference reached
struct GzipSub {
    uint64_t end;
    uint32_t len, reach, status, pad;
};

// a confirmed sub-range: its symbols, and where its text goes
struct GzipLink {
    uint64_t sym_off, t_off;
    uint32_t len, pad;
};

struct GzipArgs {
    const uint8_t *cbuf;
    uint64_t cbytes;          // cbuf[0, cbytes) on the device
    uint64_t start, sub_bits; // the stream's bit position; sub-range size
    uint32_t n_sub, cap;      // sub-ranges; symbols per sub-range slot
    uint64_t *cand;           // per sub-range: the bit offset of its first block, or kGzipNone
    GzipSub *res;
    uint16_t *sym;            // sub-range j's symbols at sym + j * cap
    const GzipLink *links;    // the confirmed chain
    uint32_t n_links;
    uint8_t *win;             // n_links + 1 windows of 32 KiB: win[0] is the stream's, win[i + 1] follows link i
    uint8_t *text;            // the links' text, n_text bytes
    uint64_t n_text;
    uint32_t *crc_parts;      // CRC32 of text piece p (kGzipCrcPiece bytes)
};

// 64 bits of c[0, n) from bit p on (zeros past n)
MGB_HD uint64_t gzip_bits64(const uint8_t *c, uint64_t n, uint64_t p) {
    const uint64_t b = p >> 3;
    uint64_t v = 0;
    for (int k = 0; k < 8 && b + k < n; ++k) v |= (uint64_t)c[b + k] << (8 * k);
    const uint32_t s = (uint32_t)(p & 7);
    if (s) v = (v >> s) | (b + 8 < n ? (uint64_t)c[b + 8] << (64 - s) : 0);
    return v;
}

// the cheap test of one bit offset: BTYPE 10, HLIT <= 29, HDIST <= 29 and a complete code-length code
MGB_HD bool gzip_prefilter(const uint8_t *c, uint64_t n, uint64_t p) {
    const uint64_t h = gzip_bits64(c, n, p);
    if (((h >> 1) & 3) != 2 || ((h >> 3) & 31) > 29 || ((h >> 8) & 31) > 29) return false;
    const uint32_t ncode = (uint32_t)((h >> 13) & 15) + 4;
    const uint64_t g = gzip_bits64(c, n, p + 17);
    uint32_t count[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    for (uint32_t i = 0; i < ncode; ++i) ++count[(g >> (3 * i)) & 7];
    int left = 1;
    for (int l = 1; l < 8; ++l) {
        left = 2 * left - (int)count[l];
        if (left < 0) return false;
    }
    return left == 0;
}

// a bit reader at bit p of c[0, n); false when n ends first
MGB_HD bool gzip_reader_at(BgzfBits &r, const uint8_t *c, uint64_t n, uint64_t p) {
    r.p = c; r.pos = p >> 3; r.end = n; r.buf = 0; r.cnt = 0;
    if (!bgzf_need(r, (uint32_t)(p & 7))) return false;
    bgzf_take(r, (uint32_t)(p & 7));
    return true;
}

// the full test (warp-uniform p): the whole dynamic header parses, as the decoder would read it
MGB_HD bool gzip_header_at(const uint8_t *c, uint64_t n, uint64_t p, BgzfShared &sh) {
    BgzfBits r;
    if (!gzip_reader_at(r, c, n, p) || !bgzf_need(r, 3)) return false;
    bgzf_take(r, 3);
    const bool ok = bgzf_dynamic(r, sh) == kBgzfOk;
    wsync();
    return ok;
}

// sub-range j's candidate: sub-range 0 starts at the stream's position; the others at the first offset in their range
// that passes both tests
MGB_HD void gzip_find_sub(const GzipArgs &a, uint32_t j, BgzfShared &sh) {
    if (j == 0) {
        if (wlane() == 0) a.cand[0] = a.start;
        return;
    }
    const uint64_t lo = a.start + j * a.sub_bits, bits = a.cbytes * 8;
    const uint64_t hi = lo + a.sub_bits < bits ? lo + a.sub_bits : bits;
    uint64_t found = kGzipNone;
    for (uint64_t p0 = lo; p0 < hi && found == kGzipNone; p0 += kWarp) {
        const uint64_t p = p0 + wlane();
        unsigned m = wballot(p < hi && gzip_prefilter(a.cbuf, a.cbytes, p));
        while (m) {
#if MGB_DEVICE_CODE
            const int l = __ffs(m) - 1;
#else
            const int l = __builtin_ctz(m);
#endif
            m &= m - 1;
            if (gzip_header_at(a.cbuf, a.cbytes, p0 + l, sh)) { found = p0 + l; break; }
        }
    }
    if (wlane() == 0) a.cand[j] = found;
    wsync();
}

// where a speculative decode writes: symbols, with back-references before the sub-range's start as window markers
struct GzipSink {
    uint16_t *out;
    uint32_t cap, far;        // far: the farthest a back-reference reached before the start
    MGB_HD bool reach(uint32_t o, uint32_t dist) {
        if (dist > o + kGzipWindow) return false;
        if (dist > o && dist - o > far) far = dist - o;
        return true;
    }
    MGB_HD void lit(uint32_t o, uint32_t sym) { if (wlane() == 0) out[o] = (uint16_t)sym; }
    // every source symbol is before o, so the lanes copy at once; a source before the start becomes a marker
    MGB_HD void match(uint32_t o, uint32_t len, uint32_t dist) {
        MGB_BGZF_ASSERT(dist >= 1 && dist <= o + kGzipWindow && len <= cap - o);
        wsync();
        for (uint32_t i = wlane(); i < len; i += kWarp) {
            const int64_t src = (int64_t)o - dist + (i < dist ? i : i % dist);
            out[o + i] = src >= 0 ? out[src] : (uint16_t)(0x8000u | (uint32_t)(kGzipWindow + src));
        }
        wsync();
    }
    MGB_HD void stored(uint32_t o, const uint8_t *src, uint32_t len) {
        for (uint32_t i = wlane(); i < len; i += kWarp) out[o + i] = src[i];
        wsync();
    }
};

// sub-range j decoded from its candidate until the first block end at or past the next candidate, a final block, a
// full slot, the end of the input or an invalid code; end/len: the last block end reached
MGB_HD void gzip_decode_sub(const GzipArgs &a, uint32_t j, BgzfShared &sh) {
    const uint64_t start = a.cand[j];
    GzipSub out;
    out.end = start; out.len = 0; out.reach = 0; out.pad = 0;
    if (start == kGzipNone) {
        out.status = kGzipSkipped;
    } else {
        uint64_t stop = kGzipNone;
        for (uint32_t k = j + 1; k < a.n_sub && stop == kGzipNone; ++k) stop = a.cand[k];
        GzipSink s{a.sym + (uint64_t)j * a.cap, a.cap, 0};
        BgzfBits r;
        uint32_t o = 0, last = 0, status = gzip_reader_at(r, a.cbuf, a.cbytes, start) ? (uint32_t)kBgzfOk : (uint32_t)kGzipShort;
        while (status == kBgzfOk) {
            status = bgzf_block(r, sh, s, &o, &last);
            wsync();
            if (status != kBgzfOk) break;
            out.end = r.pos * 8 - r.cnt;
            out.len = o;
            if (last) status = kGzipFinal;
            else if (out.end >= stop) break;
        }
        // an invalid code read with the whole input loaded may be cut off by its end: more input decides
        if (status == kBgzfBadStream && r.pos == r.end) status = kGzipShort;
        out.status = status;
        out.reach = s.far;
    }
    if (wlane() == 0) a.res[j] = out;
    wsync();
}

MGB_HD uint8_t gzip_byte(uint16_t sym, const uint8_t *win) { return sym < 256 ? (uint8_t)sym : win[sym & 0x7fff]; }

// byte x of the window after link i: its last symbols, or the end of its own window when it is shorter than 32 KiB
MGB_HD void gzip_window_at(const GzipArgs &a, uint32_t i, uint32_t x) {
    const GzipLink l = a.links[i];
    const uint8_t *w = a.win + (uint64_t)i * kGzipWindow;
    const uint32_t k = kGzipWindow - x;
    a.win[(uint64_t)(i + 1) * kGzipWindow + x] = k <= l.len ? gzip_byte(a.sym[l.sym_off + l.len - k], w) : w[x + l.len];
}

MGB_HD void gzip_resolve_at(const GzipArgs &a, uint32_t i, uint32_t x) {
    const GzipLink &l = a.links[i];
    a.text[l.t_off + x] = gzip_byte(a.sym[l.sym_off + x], a.win + (uint64_t)i * kGzipWindow);
}

// CRC32 of text piece p (crc: the byte table)
MGB_HD void gzip_crc_piece(const GzipArgs &a, uint64_t p, const uint32_t *crc) {
    const uint64_t b = p * kGzipCrcPiece, e = b + kGzipCrcPiece < a.n_text ? b + kGzipCrcPiece : a.n_text;
    uint32_t c = 0xffffffffu;
    for (uint64_t i = b; i < e; ++i) c = crc[(c ^ a.text[i]) & 0xff] ^ (c >> 8);
    a.crc_parts[p] = ~c;
}

#if MGB_DEVICE_CODE
__global__ void __launch_bounds__(32 * kGzipWarps) k_gzip_find(const __grid_constant__ GzipArgs a) {
    __shared__ BgzfShared sh[kGzipWarps];
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, nw = gridDim.x * blockDim.x / 32;
    for (uint32_t j = warp; j < a.n_sub; j += nw) gzip_find_sub(a, j, sh[threadIdx.x / 32]);
}

__global__ void __launch_bounds__(32 * kGzipWarps) k_gzip_decode(const __grid_constant__ GzipArgs a) {
    __shared__ BgzfShared sh[kGzipWarps];
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, nw = gridDim.x * blockDim.x / 32;
    for (uint32_t j = warp; j < a.n_sub; j += nw) gzip_decode_sub(a, j, sh[threadIdx.x / 32]);
}

// one block walks the chain: window i + 1 needs window i
__global__ void __launch_bounds__(1024) k_gzip_window(const __grid_constant__ GzipArgs a) {
    for (uint32_t i = 0; i < a.n_links; ++i) {
        for (uint32_t x = threadIdx.x; x < kGzipWindow; x += blockDim.x) gzip_window_at(a, i, x);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_gzip_resolve(const __grid_constant__ GzipArgs a) {
    for (uint32_t i = blockIdx.x; i < a.n_links; i += gridDim.x)
        for (uint32_t x = threadIdx.x; x < a.links[i].len; x += blockDim.x) gzip_resolve_at(a, i, x);
}

__global__ void __launch_bounds__(256) k_gzip_crc(const __grid_constant__ GzipArgs a) {
    __shared__ uint32_t crc[256];
    for (uint32_t n = threadIdx.x; n < 256; n += blockDim.x) {
        uint32_t c = n;
        for (int k = 0; k < 8; ++k) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1;
        crc[n] = c;
    }
    __syncthreads();
    const uint64_t pieces = (a.n_text + kGzipCrcPiece - 1) / kGzipCrcPiece;
    for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < pieces; p += (uint64_t)gridDim.x * blockDim.x)
        gzip_crc_piece(a, p, crc);
}
#endif

} // namespace mgb
