// Host-side helpers shared by the C-ABI implementation: config validation / lowering
// (DBGAligner ctor, dbg_aligner.cpp:33-61) and arena sizing.
#pragma once
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/mgb.h"
#include "align_core.cuh"

namespace mgb {

// DBGAlignerConfig::check_config_scores (aligner_config.cpp:39-66)
inline bool check_config_scores(const mgb_config_t &c) {
    int8_t min_penalty = 127;
    for (int i = 0; i < 128; ++i)
        for (int j = 0; j < 128; ++j)
            if (c.score_matrix[i][j] < min_penalty) min_penalty = c.score_matrix[i][j];
    if (c.gap_opening_penalty * 2 >= min_penalty) return false;
    if (c.gap_opening_penalty < min_penalty) min_penalty = c.gap_opening_penalty;
    if (c.gap_extension_penalty < min_penalty) min_penalty = c.gap_extension_penalty;
    return (int64_t)c.min_cell_score >= (int64_t)INT32_MIN - min_penalty;
}

// Alphabets of the BOSS graph (kmer/alphabets.hpp:29-38 protein, :64-79 DNA) and
// KmerExtractorBOSS::encode (kmer_extractor.cpp:30-44): unknown characters (and bytes >= 128) map to
// `sigma` for DNA (invalid) and to 'X' = 26 for protein (a regular symbol).
struct AlphabetTables {
    uint32_t sigma;
    bool has_complement;
    char letters[kMaxSigma + 1];
    uint8_t code_of[256];
    const char *valid_upper;      // letters that score as a match with themselves (alphabets.hpp:85-161)
};
inline bool alphabet_tables(int alphabet, AlphabetTables *t) {
    std::memset(t, 0, sizeof(*t));
    if (alphabet == MGB_ALPHABET_DNA) {
        t->sigma = 5; t->has_complement = true;
        std::strcpy(t->letters, "$ACGT");
        std::memset(t->code_of, 5, sizeof(t->code_of));
        for (int i = 1; i < 5; ++i) { t->code_of[(int)t->letters[i]] = i; t->code_of[(int)t->letters[i] + 32] = i; }
        t->code_of[(int)'U'] = t->code_of[(int)'u'] = 4;
        t->valid_upper = "ACGT";
        return true;
    }
    if (alphabet == MGB_ALPHABET_PROTEIN) {
        t->sigma = 27; t->has_complement = false;
        std::strcpy(t->letters, "$ABCDEFGHIJKLMNOPQRSTUVWYZX");
        std::memset(t->code_of, 26, sizeof(t->code_of));
        for (int i = 1; i < 26; ++i) { t->code_of[(int)t->letters[i]] = i; t->code_of[(int)t->letters[i] + 32] = i; }
        t->valid_upper = "ABCDEFGHIJKLMNOPQRSTUVWYZ";
        return true;
    }
    return false;
}

// DBGAlignerConfig::score_matrix_blosum62 (aligner_config.cpp:207-255): the standard BLOSUM62 table for
// the 23 letters below, -4 elsewhere, +1 on the rest of the diagonal
inline void blosum62_matrix(int8_t m[128][128]) {
    static const char order[] = "ARNDCQEGHILKMFPSTWYVBZX";
    static const int8_t b62[23][23] = {
    {  4, -1, -2, -2,  0, -1, -1,  0, -2, -1, -1, -1, -1, -2, -1,  1,  0, -3, -2,  0, -2, -1,  0 },
    { -1,  5,  0, -2, -3,  1,  0, -2,  0, -3, -2,  2, -1, -3, -2, -1, -1, -3, -2, -3, -1,  0, -1 },
    { -2,  0,  6,  1, -3,  0,  0,  0,  1, -3, -3,  0, -2, -3, -2,  1,  0, -4, -2, -3,  3,  0, -1 },
    { -2, -2,  1,  6, -3,  0,  2, -1, -1, -3, -4, -1, -3, -3, -1,  0, -1, -4, -3, -3,  4,  1, -1 },
    {  0, -3, -3, -3,  9, -3, -4, -3, -3, -1, -1, -3, -1, -2, -3, -1, -1, -2, -2, -1, -3, -3, -2 },
    { -1,  1,  0,  0, -3,  5,  2, -2,  0, -3, -2,  1,  0, -3, -1,  0, -1, -2, -1, -2,  0,  3, -1 },
    { -1,  0,  0,  2, -4,  2,  5, -2,  0, -3, -3,  1, -2, -3, -1,  0, -1, -3, -2, -2,  1,  4, -1 },
    {  0, -2,  0, -1, -3, -2, -2,  6, -2, -4, -4, -2, -3, -3, -2,  0, -2, -2, -3, -3, -1, -2, -1 },
    { -2,  0,  1, -1, -3,  0,  0, -2,  8, -3, -3, -1, -2, -1, -2, -1, -2, -2,  2, -3,  0,  0, -1 },
    { -1, -3, -3, -3, -1, -3, -3, -4, -3,  4,  2, -3,  1,  0, -3, -2, -1, -3, -1,  3, -3, -3, -1 },
    { -1, -2, -3, -4, -1, -2, -3, -4, -3,  2,  4, -2,  2,  0, -3, -2, -1, -2, -1,  1, -4, -3, -1 },
    { -1,  2,  0, -1, -3,  1,  1, -2, -1, -3, -2,  5, -1, -3, -1,  0, -1, -3, -2, -2,  0,  1, -1 },
    { -1, -1, -2, -3, -1,  0, -2, -3, -2,  1,  2, -1,  5,  0, -2, -1, -1, -1, -1,  1, -3, -1, -1 },
    { -2, -3, -3, -3, -2, -3, -3, -3, -1,  0,  0, -3,  0,  6, -4, -2, -2,  1,  3, -1, -3, -3, -1 },
    { -1, -2, -2, -1, -3, -1, -1, -2, -2, -3, -3, -1, -2, -4,  7, -1, -1, -4, -3, -2, -2, -1, -2 },
    {  1, -1,  1,  0, -1,  0,  0,  0, -1, -2, -2,  0, -1, -2, -1,  4,  1, -3, -2, -2,  0,  0,  0 },
    {  0, -1,  0, -1, -1, -1, -1, -2, -2, -1, -1, -1, -1, -2, -1,  1,  5, -2, -2,  0, -1, -1,  0 },
    { -3, -3, -4, -4, -2, -2, -3, -2, -2, -3, -2, -3, -1,  1, -4, -3, -2, 11,  2, -3, -4, -3, -2 },
    { -2, -2, -2, -3, -2, -1, -2, -3,  2, -1, -1, -2, -1,  3, -3, -2, -2,  2,  7, -1, -3, -2, -1 },
    {  0, -3, -3, -3, -1, -2, -2, -3, -3,  3,  1, -2,  1, -1, -2, -2,  0, -3, -1,  4, -3, -2, -1 },
    { -2, -1,  3,  4, -3,  0,  1, -1,  0, -3, -4,  0, -3, -3, -2,  0, -1, -4, -3, -3,  4,  1, -1 },
    { -1,  0,  0,  1, -3,  3,  4, -2,  0, -3, -3,  1, -1, -3, -1,  0, -1, -3, -2, -2,  1,  4, -1 },
    {  0, -1, -1, -1, -2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -2,  0,  0, -2, -1, -1, -1, -1, -1 }
    };
    std::memset(m, -4, 128 * 128);
    for (int i = 0; i < 128; ++i) m[i][i] = 1;
    for (int i = 0; i < 23; ++i)
        for (int j = 0; j < 23; ++j) m[(int)order[i]][(int)order[j]] = b62[i][j];
}

// Returns MGB_OK or an error code; fills `d`.
inline int lower_config(const mgb_config_t &c, uint32_t k, int alphabet, DevConfig *d, std::string *err) {
    AlphabetTables at;
    if (!alphabet_tables(alphabet, &at)) { *err = "unknown alphabet"; return MGB_ERR_UNSUPPORTED; }

    if (!c.global_xdrop) { *err = "global_xdrop = false is not supported"; return MGB_ERR_UNSUPPORTED; }
    if (c.num_alternative_paths < 1 || c.num_alternative_paths > (uint64_t)kMaxAlt) {
        *err = "num_alternative_paths must be in [1, " + std::to_string(kMaxAlt) + "]";
        return MGB_ERR_UNSUPPORTED;
    }
    if (!check_config_scores(c)) {
        *err = "Error: sum of min_cell_score and lowest penalty too low.";   // dbg_aligner.cpp:55-56
        return MGB_ERR_BAD_CONFIG;
    }
    std::memset(d, 0, sizeof(*d));
    uint64_t min_seed = c.min_seed_length ? c.min_seed_length : k;
    uint64_t max_seed = c.max_seed_length ? c.max_seed_length : k;
    if (min_seed > max_seed) { uint64_t t = min_seed; min_seed = max_seed; max_seed = t; }
    d->num_alternative_paths = (uint32_t)c.num_alternative_paths;
    d->min_seed_length = min_seed > 0xffffffffull ? 0xffffffffu : (uint32_t)min_seed;
    d->max_seed_length = max_seed > 0xffffffffull ? 0xffffffffu : (uint32_t)max_seed;
    d->max_num_seeds_per_locus = c.max_num_seeds_per_locus;
    d->min_cell_score = c.min_cell_score; d->min_path_score = c.min_path_score; d->xdrop = c.xdrop;
    if (c.xdrop <= 0) { *err = "xdrop must be positive"; return MGB_ERR_BAD_CONFIG; }
    d->min_exact_match = c.min_exact_match; d->max_nodes_per_seq_char = c.max_nodes_per_seq_char;
    d->max_ram_per_alignment = c.max_ram_per_alignment; d->rel_score_cutoff = c.rel_score_cutoff;
    d->gap_open = c.gap_opening_penalty; d->gap_ext = c.gap_extension_penalty;
    d->ge_shift = -1;
    for (int sh = 0; sh < 8; ++sh) if (-(int)c.gap_extension_penalty == (1 << sh)) d->ge_shift = sh;
    d->left_end_bonus = c.left_end_bonus; d->right_end_bonus = c.right_end_bonus;
    // protein builds compile the reverse-complement strand out (dbg_aligner.cpp:224-229, 289-293)
    d->forward_and_reverse_complement = c.forward_and_reverse_complement && at.has_complement;
    d->allow_left_trim = c.allow_left_trim; d->no_backtrack = c.no_backtrack;
    // is_low_complexity() is compiled to `false` in protein builds (aligner_seeder_methods.cpp:30-34)
    d->seed_complexity_filter = c.seed_complexity_filter && at.has_complement;
    if (c.result_nodes > 1) { *err = "result_nodes must be MGB_NODES_U64 or MGB_NODES_NONE"; return MGB_ERR_INVALID_ARGUMENT; }
    d->result_nodes = c.result_nodes;
    {   // exact-path shortcut (align_core.cuh extend()): one reported alignment, backtracking on, every letter of the
        // alphabet scores strictly best against itself and positively, gaps cost, the end bonuses are not negative
        // and the left one (plus a match) is not outweighed by the right one (later seeds are covered)
        bool ok = !c.no_exact_path_shortcut && c.num_alternative_paths == 1 && !c.no_backtrack
                  && c.gap_opening_penalty < 0 && c.gap_extension_penalty < 0
                  && c.left_end_bonus >= 0 && c.right_end_bonus >= 0 && !std::getenv("MGB_NO_EXACT_SHORTCUT");
        for (uint32_t i = 1; i < at.sigma && ok; ++i) {
            const int q = (unsigned char)at.letters[i];
            const int m = c.score_matrix[q][q];
            if (m <= 0 || m + c.left_end_bonus < c.right_end_bonus || !std::strchr(at.valid_upper, q)) ok = false;
            for (uint32_t x = 1; x < at.sigma && ok; ++x) {
                const int g = (unsigned char)at.letters[x];
                if (g != q && c.score_matrix[g][q] >= m) ok = false;
            }
        }
        // ... and ninf less a mismatch (or gap open), a gap open and an extension stays in int32: past that the reference's
        // column update wraps (DESIGN.md §5) and the argument for the shortcut does not hold
        int lo = c.gap_opening_penalty;
        for (int a = 0; a < 128; ++a)
            for (int b = 0; b < 128; ++b) lo = std::min(lo, (int)c.score_matrix[a][b]);
        ok = ok && (int64_t)kNinf + lo + c.gap_opening_penalty + c.gap_extension_penalty >= INT32_MIN;
        d->exact_shortcut = ok ? 1 : 0;
    }
    d->sigma = at.sigma; d->has_complement = at.has_complement ? 1 : 0;
    std::memcpy(d->letters, at.letters, sizeof(d->letters));
    std::memcpy(d->code_of, at.code_of, sizeof(d->code_of));
    const int sigma = (int)at.sigma;
    for (int q = 0; q < 128; ++q) {
        d->diag[q] = c.score_matrix[q][q];
        for (int i = 0; i <= sigma; ++i) {
            int ch = i < sigma ? at.letters[i] : 0;
            d->prof[i][q] = c.score_matrix[ch][q];
            // kCharToOp (aligner_cigar.cpp:11-51): MATCH iff same valid letter, any case
            int uq = (q >= 'a' && q <= 'z') ? q - 32 : q;
            d->opmatch[i][q] = (i >= 1 && i < sigma && uq == ch && std::strchr(at.valid_upper, ch)) ? 1 : 0;
        }
    }
    return MGB_OK;
}

// Arena capacities for reads up to L_max; `scale` = 1, 4, 16, ... on overflow retries.
inline Caps choose_caps(uint32_t L_max, const DevConfig &d, uint32_t k, uint32_t scale) {
    Caps c;
    uint32_t L = L_max < 16 ? 16 : L_max;
    c.L_max = L_max;
    uint64_t cols = (uint64_t)scale * (8ull * L + 256);
    uint64_t band = (uint64_t)L + 6;
    if (d.gap_ext < 0 && d.xdrop < (1 << 20)) {
        uint64_t b = 2ull * (d.xdrop / (-d.gap_ext)) + 16;
        if (b < band) band = b;
    }
    c.max_cols = (uint32_t)(cols > 0x3fffffffull ? 0x3fffffffull : cols);
    uint64_t cells = cols * (band + 5) + 4ull * (L + 16);
    c.max_cells = (uint32_t)(cells > 0x7fffffffull / 3 ? 0x7fffffffull / 3 : cells);
    uint32_t hs = 1024;
    while (hs < 4 * c.max_cols && hs < (1u << 30)) hs <<= 1;
    c.hash_size = hs;
    c.max_conv_entries = c.max_cols;
    uint64_t ccells = cols * (band + 24);
    c.max_conv_cells = (uint32_t)(ccells > 0x7fffffffull ? 0x7fffffffull : ccells);
    c.max_seeds = scale * (4 * L + 64);
    c.aln_nodes = scale * (3 * L + 128 + k);
    c.aln_seq = scale * (3 * L + 128 + 2 * k);
    c.aln_cigar = scale * (2 * L + 64);
    c.n_alt = d.num_alternative_paths;
    return c;
}

inline size_t arena_bytes(const Caps &c) {
    WarpLayout l;
    return l.carve(c);
}

} // namespace mgb
