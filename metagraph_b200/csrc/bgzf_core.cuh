// BGZF blocks inflated on the device (mgb_fastx_stage_bgzf, mgb_bgzf_inflate): one warp per block, its text written
// straight to its offset in the buffer the FASTX parser reads (DESIGN.md §8 "Compressed input").
//
// A BGZF block is a gzip member of at most 64 KiB of text whose header carries its compressed size, so the host lists
// the blocks (payload, CRC32, ISIZE, text offset) without inflating anything and every block is inflated on its own.
// The warp decodes the DEFLATE stream in lock-step: every lane reads the same bits and decodes the same symbols (warp-
// uniform control flow), lane 0 writes literals, and back-references and stored blocks are copied by the whole warp.
// Huffman codes are canonical count/symbol tables in shared memory, decoded a bit at a time; the code-length code,
// lit/len and distance codes are checked for over-subscription and incompleteness as zlib's inflate_table checks them.
// Every payload read is bounded by the payload's end, every write by ISIZE and every distance by the bytes produced.
// The block is refused (status != 0), never faulted, when any check fails, when the stream does not end in the
// payload's last byte, or when the output's CRC32 or length differs from the trailer.
#pragma once
#include <stdint.h>
#include "common.cuh"
#if !MGB_DEVICE_CODE
#include <cassert>
#define MGB_BGZF_ASSERT(x) assert(x)      // the bounds the checks below establish, asserted in the emulation build
#else
#define MGB_BGZF_ASSERT(x) ((void)0)
#endif

namespace mgb {

constexpr uint32_t kBgzfMaxText = 65536;        // ISIZE of a BGZF block is at most 64 KiB
constexpr int kBgzfWarps = 4;                    // warps per block of k_bgzf_inflate
constexpr int kBgzfCrcParts = 32;                // the output's CRC32 is computed in this many parts and combined
enum : uint32_t { kBgzfOk = 0, kBgzfBadStream = 1, kBgzfBadSize = 2, kBgzfBadCrc = 3 };

struct BgzfBlock {
    uint64_t c_off;          // the DEFLATE payload is cbuf[c_off, c_off + c_len)
    uint64_t t_off;          // where the block's text goes: text + t_off
    uint32_t c_len, crc, isize, pad;
};

struct BgzfArgs {
    const uint8_t *cbuf;
    const BgzfBlock *blocks;
    uint32_t n_blocks;
    uint8_t *text;
    uint32_t *status;        // per block: kBgzfOk, or why it was refused
};

// one warp's working set: the CRC32 byte table, a canonical code each for lit/len (or the code-length code) and
// distances, and the code lengths being read
struct BgzfShared {
    uint32_t crc[256];
    uint32_t part[kBgzfCrcParts];
    uint16_t lcount[16], lsym[288];
    uint16_t dcount[16], dsym[32];
    uint8_t lens[320];
};

#if MGB_DEVICE_CODE
#define MGB_BGZF_TABLE __constant__ const
#else
#define MGB_BGZF_TABLE static const
#endif
MGB_BGZF_TABLE uint16_t kBgzfLenBase[29] = { 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67,
                                             83, 99, 115, 131, 163, 195, 227, 258 };
MGB_BGZF_TABLE uint8_t kBgzfLenExtra[29] = { 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5,
                                             5, 5, 0 };
MGB_BGZF_TABLE uint16_t kBgzfDistBase[30] = { 1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513,
                                              769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577 };
MGB_BGZF_TABLE uint8_t kBgzfDistExtra[30] = { 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10,
                                              11, 11, 12, 12, 13, 13 };
MGB_BGZF_TABLE uint8_t kBgzfClOrder[19] = { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };

// a * b modulo the CRC-32 polynomial, bit-reflected (x^0 is bit 31)
MGB_HOSTDEV uint32_t crc_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}

// x^(8n) modulo the polynomial: crc32(A || B) = crc_multmodp(crc_x8n(|B|), crc32(A)) ^ crc32(B)
MGB_HOSTDEV uint32_t crc_x8n(uint64_t n) {
    uint32_t p = 1u << 31, sq = 1u << 30;            // x^0, x^1
    for (int i = 0; i < 3; ++i) sq = crc_multmodp(sq, sq);
    for (; n; n >>= 1) {
        if (n & 1) p = crc_multmodp(sq, p);
        sq = crc_multmodp(sq, sq);
    }
    return p;
}

// the payload's bits, least significant first; pos: the next byte to load
struct BgzfBits {
    const uint8_t *p;
    uint64_t pos, end, buf;
    uint32_t cnt;
};

MGB_HD void bgzf_fill(BgzfBits &r) {
    while (r.cnt <= 56 && r.pos < r.end) {
        MGB_BGZF_ASSERT(r.pos < r.end);
        r.buf |= (uint64_t)r.p[r.pos++] << r.cnt;
        r.cnt += 8;
    }
}
// false when the payload ends before n bits
MGB_HD bool bgzf_need(BgzfBits &r, uint32_t n) {
    if (r.cnt < n) bgzf_fill(r);
    return r.cnt >= n;
}
MGB_HD uint32_t bgzf_take(BgzfBits &r, uint32_t n) {
    MGB_BGZF_ASSERT(n <= r.cnt);
    const uint32_t v = (uint32_t)(r.buf & ((1ull << n) - 1));
    r.buf >>= n;
    r.cnt -= n;
    return v;
}

// The canonical code of lens[0, n) into count/symbol (lane 0 writes, the warp reads after the sync). Returns 0 for a
// complete code, 1 for the incomplete codes zlib accepts for lit/len and distances (at most one code, of length 1) and
// -1 for any other: over-subscribed or incomplete. A code-length code must be complete.
MGB_HD int bgzf_build(const uint8_t *lens, int n, uint16_t *count, uint16_t *symbol) {
    if (wlane() == 0) {
        uint16_t offs[16];
        for (int l = 0; l < 16; ++l) count[l] = 0;
        for (int s = 0; s < n; ++s) ++count[lens[s]];
        offs[1] = 0;
        for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + count[l];
        for (int s = 0; s < n; ++s) if (lens[s]) symbol[offs[lens[s]]++] = (uint16_t)s;
    }
    wsync();
    int left = 1, max = 0;
    for (int l = 1; l < 16; ++l) {
        left = 2 * left - count[l];
        if (left < 0) return -1;
        if (count[l]) max = l;
    }
    return left == 0 ? 0 : max <= 1 ? 1 : -1;
}

// the next symbol of a code (puff's decode: one bit at a time along the canonical code); -1: none in 15 bits, or the
// payload ends inside the code
MGB_HD int bgzf_decode(BgzfBits &r, const uint16_t *count, const uint16_t *symbol) {
    bgzf_need(r, 15);
    int code = 0, first = 0, index = 0;
    for (uint32_t len = 1; len <= 15 && len <= r.cnt; ++len) {
        code |= (int)((r.buf >> (len - 1)) & 1);
        const int c = count[len];
        if (code - c < first) {
            bgzf_take(r, len);
            return symbol[index + (code - first)];
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

// out[o, o + len) = out[o - dist, ...) repeated with period dist: every source byte was written before the copy
MGB_HD void bgzf_match(uint8_t *out, uint32_t o, uint32_t len, uint32_t dist, uint32_t isize) {
    MGB_BGZF_ASSERT(dist >= 1 && dist <= o && len <= isize - o);
    wsync();
    for (uint32_t i = wlane(); i < len; i += kWarp) out[o + i] = out[o - dist + (i < dist ? i : i % dist)];
    wsync();
}

// Where a block's output goes. BgzfByteSink: the bytes of a BGZF block (k_bgzf_inflate); a sink with the same members
// writes the 16-bit symbols of a speculative decode (gzip_core.cuh). cap: the most output the sink takes; reach: whether
// a back-reference of `dist` from output position o is valid for the sink.
struct BgzfByteSink {
    uint8_t *out;
    uint32_t cap;
    MGB_HD bool reach(uint32_t o, uint32_t dist) const { return dist <= o; }
    MGB_HD void lit(uint32_t o, uint32_t sym) { if (wlane() == 0) out[o] = (uint8_t)sym; }
    MGB_HD void match(uint32_t o, uint32_t len, uint32_t dist) { bgzf_match(out, o, len, dist, cap); }
    MGB_HD void stored(uint32_t o, const uint8_t *src, uint32_t len) {
        for (uint32_t i = wlane(); i < len; i += kWarp) out[o + i] = src[i];
        wsync();
    }
};

// lit/len symbols up to end-of-block into the sink at [*o, cap)
template <class Sink> MGB_HD uint32_t bgzf_codes(BgzfBits &r, BgzfShared &sh, Sink &s, uint32_t *o) {
    for (;;) {
        int sym = bgzf_decode(r, sh.lcount, sh.lsym);
        if (sym < 0) return kBgzfBadStream;
        if (sym < 256) {
            if (*o >= s.cap) return kBgzfBadSize;
            s.lit(*o, (uint32_t)sym);
            ++*o;
            continue;
        }
        if (sym == 256) return kBgzfOk;
        sym -= 257;
        if (sym >= 29 || !bgzf_need(r, kBgzfLenExtra[sym])) return kBgzfBadStream;
        const uint32_t len = kBgzfLenBase[sym] + bgzf_take(r, kBgzfLenExtra[sym]);
        const int ds = bgzf_decode(r, sh.dcount, sh.dsym);
        if (ds < 0 || ds >= 30 || !bgzf_need(r, kBgzfDistExtra[ds])) return kBgzfBadStream;
        const uint32_t dist = kBgzfDistBase[ds] + bgzf_take(r, kBgzfDistExtra[ds]);
        if (!s.reach(*o, dist)) return kBgzfBadStream;
        if (len > s.cap - *o) return kBgzfBadSize;
        s.match(*o, len, dist);
        *o += len;
    }
}

// a dynamic block's header: the code-length code, then the lit/len and distance code lengths, then both codes
MGB_HD uint32_t bgzf_dynamic(BgzfBits &r, BgzfShared &sh) {
    if (!bgzf_need(r, 14)) return kBgzfBadStream;
    const uint32_t nlen = bgzf_take(r, 5) + 257, ndist = bgzf_take(r, 5) + 1, ncode = bgzf_take(r, 4) + 4;
    if (nlen > 286 || ndist > 30) return kBgzfBadStream;
    for (uint32_t i = 0; i < 19; ++i) {
        uint32_t l = 0;
        if (i < ncode) {
            if (!bgzf_need(r, 3)) return kBgzfBadStream;
            l = bgzf_take(r, 3);
        }
        if (wlane() == 0) sh.lens[kBgzfClOrder[i]] = (uint8_t)l;
    }
    wsync();
    if (bgzf_build(sh.lens, 19, sh.lcount, sh.lsym) != 0) return kBgzfBadStream;
    uint32_t idx = 0, prev = 0;
    while (idx < nlen + ndist) {
        const int sym = bgzf_decode(r, sh.lcount, sh.lsym);
        if (sym < 0) return kBgzfBadStream;
        uint32_t l = (uint32_t)sym, rep = 1;
        if (sym == 16) {
            if (idx == 0 || !bgzf_need(r, 2)) return kBgzfBadStream;
            l = prev;
            rep = 3 + bgzf_take(r, 2);
        } else if (sym == 17) {
            if (!bgzf_need(r, 3)) return kBgzfBadStream;
            l = 0;
            rep = 3 + bgzf_take(r, 3);
        } else if (sym == 18) {
            if (!bgzf_need(r, 7)) return kBgzfBadStream;
            l = 0;
            rep = 11 + bgzf_take(r, 7);
        }
        if (rep > nlen + ndist - idx) return kBgzfBadStream;
        if (wlane() == 0) for (uint32_t j = 0; j < rep; ++j) sh.lens[idx + j] = (uint8_t)l;
        idx += rep;
        prev = l;
    }
    wsync();
    if (sh.lens[256] == 0) return kBgzfBadStream;                 // no end-of-block code
    wsync();
    if (bgzf_build(sh.lens, (int)nlen, sh.lcount, sh.lsym) < 0) return kBgzfBadStream;
    if (bgzf_build(sh.lens + nlen, (int)ndist, sh.dcount, sh.dsym) < 0) return kBgzfBadStream;
    return kBgzfOk;
}

MGB_HD void bgzf_fixed(BgzfShared &sh) {
    if (wlane() == 0) for (int s = 0; s < 288; ++s) sh.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
    bgzf_build(sh.lens, 288, sh.lcount, sh.lsym);
    wsync();
    if (wlane() == 0) for (int s = 0; s < 32; ++s) sh.lens[s] = 5;
    bgzf_build(sh.lens, 32, sh.dcount, sh.dsym);
    wsync();
}

MGB_HD void bgzf_crc_table(BgzfShared &sh) {
    for (uint32_t n = wlane(); n < 256; n += kWarp) {
        uint32_t c = n;
        for (int k = 0; k < 8; ++k) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1;
        sh.crc[n] = c;
    }
    wsync();
}

// CRC32 of out[0, n): kBgzfCrcParts parts of the output, one per lane on the device, combined in order
MGB_HD uint32_t bgzf_crc(BgzfShared &sh, const uint8_t *out, uint32_t n) {
    const uint32_t step = (n + kBgzfCrcParts - 1) / kBgzfCrcParts;
    for (int j = wlane(); j < kBgzfCrcParts; j += kWarp) {
        const uint32_t b = j * step < n ? j * step : n, e = b + step < n ? b + step : n;
        uint32_t c = 0xffffffffu;
        for (uint32_t i = b; i < e; ++i) c = sh.crc[(c ^ out[i]) & 0xff] ^ (c >> 8);
        sh.part[j] = ~c;
    }
    wsync();
    const uint32_t z = crc_x8n(step);
    uint32_t crc = 0;
    for (int j = 0; j < kBgzfCrcParts && j * step < n; ++j) {
        const bool tail = (uint64_t)(j + 1) * step >= n;
        crc = crc_multmodp(tail ? crc_x8n(n - j * step) : z, crc) ^ sh.part[j];
    }
    return crc;
}

// one DEFLATE block (header and body) into the sink at *o; *last: its BFINAL bit
template <class Sink> MGB_HD uint32_t bgzf_block(BgzfBits &r, BgzfShared &sh, Sink &s, uint32_t *o, uint32_t *last) {
    if (!bgzf_need(r, 3)) return kBgzfBadStream;
    *last = bgzf_take(r, 1);
    const uint32_t type = bgzf_take(r, 2);
    if (type == 0) {                                  // stored: LEN, NLEN from the next byte boundary
        bgzf_take(r, r.cnt & 7);
        if (!bgzf_need(r, 32)) return kBgzfBadStream;
        const uint32_t len = bgzf_take(r, 16), nlen = bgzf_take(r, 16);
        if (len != (~nlen & 0xffff)) return kBgzfBadStream;
        // the bytes still in the bit buffer go back to the payload
        const uint64_t at = r.pos - r.cnt / 8;
        r.pos = at; r.buf = 0; r.cnt = 0;
        if (len > r.end - at) return kBgzfBadStream;
        if (len > s.cap - *o) return kBgzfBadSize;
        MGB_BGZF_ASSERT(at + len <= r.end && *o + len <= s.cap);
        s.stored(*o, r.p + at, len);
        r.pos += len;
        *o += len;
        return kBgzfOk;
    }
    if (type == 1) {
        bgzf_fixed(sh);
        return bgzf_codes(r, sh, s, o);
    }
    if (type == 2) {
        const uint32_t status = bgzf_dynamic(r, sh);
        return status == kBgzfOk ? bgzf_codes(r, sh, s, o) : status;
    }
    return kBgzfBadStream;
}

// block b with one warp: inflate, then check the stream's end, the length and the CRC32 against the trailer
MGB_HD void bgzf_inflate_block(const BgzfArgs &a, uint32_t b, BgzfShared &sh) {
    const BgzfBlock blk = a.blocks[b];
    BgzfByteSink out{a.text + blk.t_off, blk.isize};
    BgzfBits r;
    r.p = a.cbuf; r.pos = blk.c_off; r.end = blk.c_off + blk.c_len; r.buf = 0; r.cnt = 0;
    uint32_t o = 0, status = kBgzfOk, last = 0;
    while (!last && status == kBgzfOk) {
        status = bgzf_block(r, sh, out, &o, &last);
        wsync();
    }
    // the stream ends in the payload's last byte (the trailer follows it), and holds ISIZE bytes
    if (status == kBgzfOk && (r.pos != r.end || r.cnt >= 8)) status = kBgzfBadStream;
    if (status == kBgzfOk && o != blk.isize) status = kBgzfBadSize;
    if (status == kBgzfOk && bgzf_crc(sh, out.out, o) != blk.crc) status = kBgzfBadCrc;
    if (wlane() == 0) a.status[b] = status;
    wsync();
}

#if MGB_DEVICE_CODE
__global__ void __launch_bounds__(32 * kBgzfWarps) k_bgzf_inflate(const __grid_constant__ BgzfArgs a) {
    __shared__ BgzfShared sh[kBgzfWarps];
    BgzfShared &w = sh[threadIdx.x / 32];
    bgzf_crc_table(w);
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, nw = gridDim.x * blockDim.x / 32;
    for (uint32_t b = warp; b < a.n_blocks; b += nw) bgzf_inflate_block(a, b, w);
}
#endif

} // namespace mgb
