// DNA reads as words: 2-bit codes of raw A/C/G/T bytes four at a time, their validity, the reverse complement of packed
// codes and per-letter counts (k_prepare_exact, kernels.cuh exact_path_strand). Codes: A 0, C 1, G 2, T 3, upper or
// lower case; code i of a packed word sits in bits 2i, 2i + 1, as in the hash keys and IndexView::pl_text.
// Host and device; tests/devwords builds them for the host.
#pragma once
#include "common.cuh"

namespace mgb {

// per byte: 0xFF where the bytes of x and y are equal, else 0 (__vcmpeq4)
MGB_HOSTDEV uint32_t bytes_eq4(uint32_t x, uint32_t y) {
#if defined(__CUDA_ARCH__)
    return __vcmpeq4(x, y);
#else
    uint32_t m = 0;
    for (int j = 0; j < 32; j += 8) m |= ((x >> j) & 0xFFu) == ((y >> j) & 0xFFu) ? 0xFFu << j : 0u;
    return m;
#endif
}

// per byte of x: 0xFF if it is A, C, G or T in either case, else 0. x & 0xDF folds the case of letters and keeps bit 7,
// so a byte >= 128 matches none of the four.
MGB_HOSTDEV uint32_t acgt_valid4(uint32_t x) {
    const uint32_t u = x & 0xDFDFDFDFu;
    return bytes_eq4(u, 0x41414141u) | bytes_eq4(u, 0x43434343u) | bytes_eq4(u, 0x47474747u) | bytes_eq4(u, 0x54545454u);
}

// the 2-bit codes of the four bytes of x, byte j in bits 2j, 2j + 1 (((u >> 1) ^ (u >> 2)) & 3 per byte, u = byte & 0xDF;
// meaningful where acgt_valid4 is set)
MGB_HOSTDEV uint32_t acgt_codes4(uint32_t x) {
    const uint32_t u = x & 0xDFDFDFDFu;
    const uint32_t c = ((u >> 1) ^ (u >> 2)) & 0x03030303u;       // one code per byte
    const uint32_t t = c | (c >> 6);                                 // bytes 0, 1 -> bits 0-3; bytes 2, 3 -> bits 16-19
    return (t & 0xFu) | ((t >> 12) & 0xF0u);
}

// the 4 bytes at p (any alignment) from the aligned words around them: lo = the word at p & ~3, hi = the next one
MGB_HOSTDEV uint32_t bytes_funnel(uint32_t lo, uint32_t hi, uint32_t byte_shift) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, 8 * byte_shift);
#else
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (8 * byte_shift));
#endif
}

// the 8 bytes at p (any alignment), byte j in bits 8j; reads the aligned 4-byte words that hold them (up to 11 bytes
// past p)
MGB_HOSTDEV uint64_t bytes8_at(const uint8_t *p) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t *w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3), w1 = w[1];
    return bytes_funnel(w[0], w1, sh) | (uint64_t)bytes_funnel(w1, w[2], sh) << 32;
}

// the codes of the 32 bytes at p (any alignment), and in *invalid one bit per byte that is not A/C/G/T (bit t: byte
// p[t]). Reads the aligned 4-byte words that hold p[0 .. 32), so up to 35 bytes past p must be readable.
MGB_HOSTDEV uint64_t acgt_pack32(const uint8_t *p, uint32_t *invalid) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t *w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3);
    uint32_t prev = w[0], bad = 0;
    uint64_t codes = 0;
#if defined(__CUDA_ARCH__)
    #pragma unroll
#endif
    for (int g = 0; g < 8; ++g) {
        const uint32_t next = w[g + 1];
        const uint32_t x = bytes_funnel(prev, next, sh);
        prev = next;
        const uint32_t v = acgt_valid4(x);
        const uint32_t nv = ~v & 0x80808080u;                        // bit 7 of each invalid byte
        bad |= (((nv >> 7) | (nv >> 14) | (nv >> 21) | (nv >> 28)) & 0xFu) << (4 * g);
        codes |= (uint64_t)acgt_codes4(x) << (8 * g);
    }
    *invalid = bad;
    return codes;
}

// the reverse complement of the 32 codes of w: code i of the result is 3 - code 31 - i of w
MGB_HOSTDEV uint64_t rc_codes32(uint64_t w) {
#if defined(__CUDA_ARCH__)
    uint64_t r = __brevll(w);
#else
    uint64_t r = w;
    r = ((r >> 1) & 0x5555555555555555ull) | ((r & 0x5555555555555555ull) << 1);
    r = ((r >> 2) & 0x3333333333333333ull) | ((r & 0x3333333333333333ull) << 2);
    r = ((r >> 4) & 0x0F0F0F0F0F0F0F0Full) | ((r & 0x0F0F0F0F0F0F0F0Full) << 4);
    r = ((r >> 8) & 0x00FF00FF00FF00FFull) | ((r & 0x00FF00FF00FF00FFull) << 8);
    r = ((r >> 16) & 0x0000FFFF0000FFFFull) | ((r & 0x0000FFFF0000FFFFull) << 16);
    r = (r >> 32) | (r << 32);
#endif
    r = ((r >> 1) & 0x5555555555555555ull) | ((r & 0x5555555555555555ull) << 1);     // the two bits of each code back
    return ~r;
}

MGB_HOSTDEV int popc64(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return __popcll(x);
#else
    return __builtin_popcountll(x);
#endif
}

// per-letter counts of the codes of w under mask (both bits of each counted code set): c[0..3] += A, C, G, T
MGB_HOSTDEV void acgt_count(uint64_t w, uint64_t mask, int c[4]) {
    const uint64_t lo = w & mask & 0x5555555555555555ull, hi = (w >> 1) & mask & 0x5555555555555555ull;
    const int t = popc64(lo & hi), g = popc64(hi & ~lo), cc = popc64(lo & ~hi);
    c[0] += popc64(mask & 0x5555555555555555ull) - t - g - cc; c[1] += cc; c[2] += g; c[3] += t;
}

// the codes 0 .. n of a packed word (n <= 32): its low 2n bits
MGB_HOSTDEV uint64_t codes_mask(int n) { return n >= 32 ? ~0ull : (1ull << (2 * n)) - 1; }

// 8 characters of a DNA strand as stored in a record, from the 8 raw A/C/G/T bytes x (byte j: character j): upper case
// (sanitize_char) or, if rc, the reverse complement (character j is complement_char of byte 7 - j, upper case)
MGB_HOSTDEV uint64_t acgt_chars8(uint64_t x, bool rc) {
    uint64_t u = x & 0xDFDFDFDFDFDFDFDFull;
    if (!rc) return u;
#if defined(__CUDA_ARCH__)
    const uint32_t lo = (uint32_t)u, hi = (uint32_t)(u >> 32);
    u = (uint64_t)__byte_perm(lo, 0, 0x0123) << 32 | __byte_perm(hi, 0, 0x0123);
#else
    u = __builtin_bswap64(u);
#endif
    // A 0x41 <-> T 0x54 differ by 0x15, C 0x43 <-> G 0x47 by 0x04; bit 1 is set in C and G only
    return u ^ 0x1515151515151515ull ^ (((u >> 1) & 0x0101010101010101ull) * 0x11u);
}

} // namespace mgb
