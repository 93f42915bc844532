// Text rendering of alignments as `metagraph align` prints them (cli/align.cpp:254-307): the TSV line of a read and the
// JSON records of Alignment::to_json (alignment.cpp:704-963). The bytes are those of the host mirror in
// metagraph_b200/aligner.py (format_alignment, format_alignment_json), which is pinned against the reference's goldens.
//
// Every function is a template over a sink, so that one definition serves both passes of the text route (api.cu
// k_text_size / k_text_write): CountSink only adds up the bytes a read's text takes, WriteSink stores them. Control flow
// is uniform across the warp: every lane computes the same scalar values and positions; scalar bytes are stored by lane
// 0, the long copies (query, its reverse complement, path sequence, escaped strings) are spread over the lanes.
#pragma once
#include <string.h>
#include "common.cuh"

namespace mgb {

// ---------------------------------------------------------------------------------------
// sinks
// ---------------------------------------------------------------------------------------
// JSON string escaping of _json_value (aligner.py): '"' and '\' get a backslash, \n and \t their escapes, other bytes
// below 0x20 \u00XX; everything else (bytes >= 0x80 included) is copied
MGB_HOSTDEV uint32_t json_esc_len(uint8_t c) {
    return (c == '"' || c == '\\' || c == '\n' || c == '\t') ? 2u : c < 0x20 ? 6u : 1u;
}

struct CountSink {
    uint64_t pos = 0;
    MGB_HD void put(char) { ++pos; }
    template <class F> MGB_HD void copy(uint32_t n, F) { pos += n; }
    // f(i): byte i of a string of n bytes, written escaped
    template <class F> MGB_HD void escaped(uint32_t n, F f) {
        for (uint32_t b = 0; b < n; b += kWarp) {
            const uint32_t i = b + wlane();
            pos += (uint64_t)wreduce_add(i < n ? (int)json_esc_len((uint8_t)f(i)) : 0);
        }
    }
};

// Stores bytes [lo, hi) of the text at out[0, hi - lo); the others are counted and dropped (a read's text may straddle
// two windows of the output buffer)
struct WriteSink {
    char *out;
    uint64_t lo, hi, pos;
    MGB_HD void at(uint64_t p, char c) const { if (p >= lo && p < hi) out[p - lo] = c; }
    MGB_HD bool touches(uint64_t n) const { return pos + n > lo && pos < hi; }
    MGB_HD void put(char c) { if (wlane() == 0) at(pos, c); ++pos; }
    template <class F> MGB_HD void copy(uint32_t n, F f) {
        if (touches(n))
            for (uint32_t i = wlane(); i < n; i += kWarp) at(pos + i, f(i));
        pos += n;
    }
    template <class F> MGB_HD void escaped(uint32_t n, F f) {
        for (uint32_t b = 0; b < n; b += kWarp) {
            const uint32_t i = b + wlane();
            const uint8_t c = i < n ? (uint8_t)f(i) : 0;
            const int len = i < n ? (int)json_esc_len(c) : 0;
            const int incl = wscan_add(len);
            const uint64_t p = pos + (uint64_t)(incl - len);
            if (len == 1) at(p, (char)c);
            else if (len == 2) { at(p, '\\'); at(p + 1, c == '\n' ? 'n' : c == '\t' ? 't' : (char)c); }
            else if (len == 6) {
                const char *hex = "0123456789abcdef";
                at(p, '\\'); at(p + 1, 'u'); at(p + 2, '0'); at(p + 3, '0'); at(p + 4, hex[c >> 4]); at(p + 5, hex[c & 15]);
            }
            pos += (uint64_t)wbcast(incl, kWarp - 1);
        }
    }
};

template <class S> MGB_HD void put_str(S &s, const char *lit) { for (; *lit; ++lit) s.put(*lit); }

template <class S> MGB_HD void put_u64(S &s, uint64_t v) {
    char d[20];
    int n = 0;
    do { d[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) s.put(d[--n]);
}
template <class S> MGB_HD void put_i64(S &s, int64_t v) {
    if (v < 0) { s.put('-'); put_u64(s, (uint64_t)0 - (uint64_t)v); } else put_u64(s, (uint64_t)v);
}

// ---------------------------------------------------------------------------------------
// identity: matches / query_len as jsoncpp and Python print a double, "%.17g" (+ ".0" when the text has no '.', 'e'
// or 'n'), exactly and correctly rounded without printf.
// d = m / q is the IEEE quotient, so d in [0, 1]; with 0 < m <= q < 2^32, d >= 2^-32 > 1e-10, i.e. its decimal exponent
// X is in [-10, 0]. d = M 2^-e with M < 2^53, e <= 84. Seventeen significant digits are round(d 10^p), p = 16 - X <= 26:
// M 10^p = M 5^p 2^p and M 5^p < 2^53 5^26 < 2^114 fits in 128 bits, so the digits are (M 5^p) >> (e - p), rounded
// half-even on the bits shifted out.
// ---------------------------------------------------------------------------------------
typedef unsigned __int128 u128_t;

MGB_HOSTDEV u128_t pow5_u128(int p) { u128_t r = 1; for (int i = 0; i < p; ++i) r *= 5u; return r; }

// writes the text into buf (at most 24 bytes), returns its length
MGB_HOSTDEV int format_identity(uint32_t m, uint32_t q, char *buf) {
    if (m == 0 || q == 0) { buf[0] = '0'; buf[1] = '.'; buf[2] = '0'; return 3; }
    const double d = (double)m / (double)q;
    uint64_t bits;
    memcpy(&bits, &d, 8);
    const int E = (int)((bits >> 52) & 0x7ff);             // normal: d >= 2^-32
    const uint64_t M = (bits & ((1ull << 52) - 1)) | (1ull << 52);
    const int e = 1075 - E;                                // d = M 2^-e, 52 <= e <= 84
    // X = largest x in [-10, 0] with d >= 10^x  <=>  M 5^-x >= 2^(e + x)
    int X = -10;
    for (int x = 0; x > -10; --x)
        if (((u128_t)M * pow5_u128(-x)) >= ((u128_t)1 << (e + x))) { X = x; break; }
    const int p = 16 - X, sh = e - p;                      // sh >= 52 - 26 > 0
    const u128_t N = (u128_t)M * pow5_u128(p);
    uint64_t T = (uint64_t)(N >> sh);
    const u128_t rem = N & (((u128_t)1 << sh) - 1), half = (u128_t)1 << (sh - 1);
    if (rem > half || (rem == half && (T & 1))) ++T;
    if (T == 100000000000000000ull) { T = 10000000000000000ull; ++X; }
    char dig[17];
    for (int i = 16; i >= 0; --i) { dig[i] = (char)('0' + T % 10); T /= 10; }
    int nd = 17;
    while (nd > 1 && dig[nd - 1] == '0') --nd;             // %g drops trailing zeros
    int n = 0;
    if (X >= -4) {                                         // fixed notation (X <= 0 here)
        if (X == 0) {
            buf[n++] = dig[0];
            if (nd > 1) { buf[n++] = '.'; for (int i = 1; i < nd; ++i) buf[n++] = dig[i]; }
            else { buf[n++] = '.'; buf[n++] = '0'; }      // "1" -> "1.0"
        } else {
            buf[n++] = '0'; buf[n++] = '.';
            for (int i = 0; i < -X - 1; ++i) buf[n++] = '0';
            for (int i = 0; i < nd; ++i) buf[n++] = dig[i];
        }
    } else {                                               // exponent form: d[.ddd]e-XX
        buf[n++] = dig[0];
        if (nd > 1) { buf[n++] = '.'; for (int i = 1; i < nd; ++i) buf[n++] = dig[i]; }
        buf[n++] = 'e'; buf[n++] = '-';
        const int ex = -X;
        buf[n++] = (char)('0' + ex / 10); buf[n++] = (char)('0' + ex % 10);
    }
    return n;
}

template <class S> MGB_HD void put_identity(S &s, uint32_t m, uint32_t q) {
    char buf[24];
    const int n = format_identity(m, q, buf);
    for (int i = 0; i < n; ++i) s.put(buf[i]);
}

// ---------------------------------------------------------------------------------------
// one read and its alignments
// ---------------------------------------------------------------------------------------
// AlignmentResults' query (alignment.cpp:1357-1358): upper-cased, bytes >= 0x80 -> 0x7F
MGB_HOSTDEV char query_char(uint8_t c) { return c >= 0x80 ? (char)0x7f : (c >= 'a' && c <= 'z') ? (char)(c - 32) : (char)c; }
// the mirror's reverse_complement table (COMPL_TAB, seq_tools/reverse_complement.hpp:31-48) on upper-cased characters
MGB_HOSTDEV char iupac_complement(char c) {
    switch (c) {
        case 'A': return 'T'; case 'B': return 'V'; case 'C': return 'G'; case 'D': return 'H'; case 'G': return 'C';
        case 'H': return 'D'; case 'K': return 'M'; case 'M': return 'K'; case 'R': return 'Y'; case 'T': return 'A';
        case 'U': return 'A'; case 'V': return 'B'; case 'Y': return 'R'; case '`': return '@';
        default: return c;
    }
}

// what the renderers need of one record (OutAln and its arrays)
struct TextAln {
    uint32_t orientation; int32_t score; uint32_t offset, query_begin, query_len;
    uint32_t n_nodes, seq_len, n_cigar;
    const uint64_t *nodes;     // nullptr on the TSV route (records without node ids)
    const uint32_t *cigar;     // (len << 3) | op
    const char *seq;
};

// the raw read and its header
struct TextRead {
    const char *seq; uint32_t len;
    const char *name; uint32_t name_len;
};

MGB_HOSTDEV uint64_t cigar_matches(const TextAln &a) {
    uint64_t m = 0;
    for (uint32_t i = 0; i < a.n_cigar; ++i) if ((a.cigar[i] & 7u) == 2u) m += a.cigar[i] >> 3;
    return m;
}

template <class S> MGB_HD void put_cigar(S &s, const TextAln &a) {
    const char *ops = "SX=DIG";
    for (uint32_t i = 0; i < a.n_cigar; ++i) { put_u64(s, a.cigar[i] >> 3); s.put(ops[a.cigar[i] & 7u]); }
}

// the strand the alignment was made on: the query or its reverse complement, character i
struct StrandQuery {
    const char *raw; uint32_t len; uint32_t rc;
    MGB_HD char operator()(uint32_t i) const {
        return rc ? iupac_complement(query_char((uint8_t)raw[len - 1 - i])) : query_char((uint8_t)raw[i]);
    }
};

// TSV line of a read (format_alignment, without node lists): tsv_head, then tsv_aln per alignment or tsv_unaligned
template <class S> MGB_HD void tsv_head(S &s, const TextRead &rd) {
    const char *nm = rd.name, *q = rd.seq;
    s.copy(rd.name_len, [nm](uint32_t i) { return nm[i]; });
    s.put('\t');
    s.copy(rd.len, [q](uint32_t i) { return query_char((uint8_t)q[i]); });
}
template <class S> MGB_HD void tsv_unaligned(S &s, int32_t min_path_score) {
    put_str(s, "\t*\t*\t"); put_i64(s, min_path_score); put_str(s, "\t*\t*\t*");
}
// fmt::formatter<Alignment> (alignment.hpp:418-435), preceded by a tab
template <class S> MGB_HD void tsv_aln(S &s, const TextAln &a) {
    s.put('\t'); s.put(a.orientation ? '-' : '+'); s.put('\t');
    const char *sq = a.seq;
    s.copy(a.seq_len, [sq](uint32_t i) { return sq[i]; });
    s.put('\t'); put_i64(s, a.score);
    s.put('\t'); put_u64(s, cigar_matches(a));
    s.put('\t'); put_cigar(s, a);
    s.put('\t'); put_u64(s, a.offset);
}

// a JSON string of n bytes f(i)
template <class S, class F> MGB_HD void json_str(S &s, uint32_t n, F f) { s.put('"'); s.escaped(n, f); s.put('"'); }

// bytes [from, from + n) of the query view (slices clamp at its end, as Python's do)
template <class S> MGB_HD void json_view(S &s, const StrandQuery &sq, uint32_t vbegin, uint32_t vlen, uint64_t from, uint64_t n) {
    const uint64_t a = from < vlen ? from : vlen, b = from + n < vlen ? from + n : vlen;
    json_str(s, (uint32_t)(b - a), [sq, vbegin, a](uint32_t i) { return sq(vbegin + (uint32_t)a + i); });
}

// _path_json (aligner.py; path_json, alignment.cpp:704-880), label ""
template <class S> MGB_HD void json_path(S &s, const TextAln &a, const StrandQuery &sq, uint32_t node_size) {
    const uint32_t nops = a.n_cigar, vb = a.query_begin, vl = a.query_len;
    auto op_of = [&](uint32_t it) -> uint32_t { return it < nops ? (a.cigar[it] & 7u) : 2u; };
    auto len_of = [&](uint32_t it) -> uint64_t { return it < nops ? (uint64_t)(a.cigar[it] >> 3) : ~0ull; };
    uint32_t it = (nops && op_of(0) == 0) ? 1 : 0;
    uint64_t cigar_offset = 0, qpos = 0;
    uint64_t cur_pos = a.offset;
    s.put('{');
    if (a.nodes[0] == a.nodes[a.n_nodes - 1]) put_str(s, "\"is_circular\":true,");
    put_str(s, "\"length\":"); put_u64(s, a.n_nodes); put_str(s, ",\"mapping\":[{");
    bool any = false;
    while (cur_pos < node_size && it < nops) {               // the first node
        const uint32_t op = op_of(it); const uint64_t n = len_of(it);
        if (op == 0) { ++it; cigar_offset = 0; continue; }     // trailing clipping
        uint64_t next_pos = cur_pos + (n - cigar_offset) < node_size ? cur_pos + (n - cigar_offset) : node_size;
        const uint64_t next_size = next_pos - cur_pos;
        put_str(s, any ? ",{" : "\"edit\":[{");
        any = true;
        if (op == 1) {                                         // MISMATCH
            put_str(s, "\"from_length\":"); put_u64(s, next_size); put_str(s, ",\"sequence\":");
            json_view(s, sq, vb, vl, qpos, next_size); put_str(s, ",\"to_length\":"); put_u64(s, next_size);
            qpos += next_size;
        } else if (op == 4) {                                  // INSERTION
            put_str(s, "\"sequence\":"); json_view(s, sq, vb, vl, qpos, next_size);
            put_str(s, ",\"to_length\":"); put_u64(s, next_size);
            qpos += next_size;
            next_pos = cur_pos;
        } else if (op == 3) {                                  // DELETION
            put_str(s, "\"from_length\":"); put_u64(s, next_size);
        } else if (op == 2) {                                  // MATCH
            put_str(s, "\"from_length\":"); put_u64(s, next_size); put_str(s, ",\"to_length\":"); put_u64(s, next_size);
            qpos += next_size;
        }
        s.put('}');
        cigar_offset += next_size;
        cur_pos = next_pos;
        if (cigar_offset == n) { ++it; cigar_offset = 0; }
    }
    if (any) put_str(s, "],");
    put_str(s, "\"position\":{\"node_id\":"); put_u64(s, a.nodes[0]);
    if (a.offset) { put_str(s, ",\"offset\":"); put_u64(s, a.offset); }
    put_str(s, "},\"rank\":1}");
    for (uint32_t j = 1; j < a.n_nodes; ++j) {                 // one character per further node
        put_str(s, ",{\"edit\":[");
        uint32_t op = op_of(it); uint64_t n = len_of(it);
        if (op == 4 || op == 0) {
            const uint64_t length = n - cigar_offset;
            put_str(s, "{\"sequence\":"); json_view(s, sq, vb, vl, qpos, length);
            put_str(s, ",\"to_length\":"); put_u64(s, length); put_str(s, "},");
            qpos += length; ++it; cigar_offset = 0;
            op = op_of(it); n = len_of(it);
        }
        if (op == 1) {
            put_str(s, "{\"from_length\":1,\"sequence\":"); json_view(s, sq, vb, vl, qpos, 1); put_str(s, ",\"to_length\":1}");
            ++qpos;
        } else if (op == 3) {
            put_str(s, "{\"from_length\":1}");
        } else {
            put_str(s, "{\"from_length\":1,\"to_length\":1}");
            ++qpos;
        }
        if (++cigar_offset == n) { cigar_offset = 0; ++it; }
        put_str(s, "],\"position\":{\"node_id\":"); put_u64(s, a.nodes[j]);
        put_str(s, ",\"offset\":"); put_i64(s, (int64_t)node_size - 1);
        put_str(s, "},\"rank\":"); put_u64(s, j + 1); s.put('}');
    }
    put_str(s, "],\"name\":\"\"}");
}

template <class S> MGB_HD void json_name(S &s, const TextRead &rd) {
    const char *nm = rd.name;
    put_str(s, "\"name\":");
    json_str(s, rd.name_len, [nm](uint32_t i) { return nm[i]; });
}

// Alignment::to_json (alignment_to_json in aligner.py) with sorted keys, and its newline
template <class S> MGB_HD void json_aln(S &s, const TextRead &rd, const TextAln &a, bool secondary, uint32_t node_size) {
    const StrandQuery sq { rd.seq, rd.len, a.orientation };
    const char *seq = a.seq;
    s.put('{');
    if (a.seq_len || a.query_len) {
        put_str(s, "\"annotation\":{");
        if (a.query_len) { put_str(s, "\"cigar\":\""); put_cigar(s, a); s.put('"'); }
        if (a.seq_len) {
            put_str(s, a.query_len ? ",\"ref_sequence\":" : "\"ref_sequence\":");
            json_str(s, a.seq_len, [seq](uint32_t i) { return seq[i]; });
        }
        put_str(s, "},");
    }
    if (a.query_len) {
        put_str(s, "\"identity\":"); put_identity(s, (uint32_t)cigar_matches(a), a.query_len); s.put(',');
        if (secondary) put_str(s, "\"is_secondary\":true,");
    }
    json_name(s, rd);
    if (a.query_len) {
        if (a.n_nodes) { put_str(s, ",\"path\":"); json_path(s, a, sq, node_size); }
        if (a.query_begin) { put_str(s, ",\"query_position\":"); put_u64(s, a.query_begin); }
        put_str(s, ",\"read_mapped\":true");
        if (a.orientation) put_str(s, ",\"read_on_reverse_strand\":true");
        put_str(s, ",\"score\":"); put_i64(s, a.score);
    }
    put_str(s, ",\"sequence\":");
    json_str(s, rd.len, sq);
    if (a.query_len && a.query_begin) put_str(s, ",\"soft_clipped\":true");
    put_str(s, "}\n");
}

// the record of an unaligned read
template <class S> MGB_HD void json_unaligned(S &s, const TextRead &rd) {
    s.put('{'); json_name(s, rd); put_str(s, ",\"sequence\":\"\"}\n");
}

} // namespace mgb
