// The property k_seed_hash's paired walk relies on (kernels.cuh): for every byte of a read, if its code on one strand
// is a valid DNA code, its code on the other strand is either invalid or the complement (5 - code). Codes are those
// k_prepare writes: code_of[sanitize_char(ch)] forward, code_of[complement_char(sanitize_char(ch))] reverse.
// Prints the number of bytes valid on both strands; exits 1 on a violation.
#include <cstdio>

#include "../../metagraph_b200/csrc/host_common.hpp"

int main() {
    mgb::AlphabetTables t;
    if (!mgb::alphabet_tables(MGB_ALPHABET_DNA, &t)) return 2;
    int both = 0, bad = 0;
    for (int ch = 0; ch < 256; ++ch) {
        const uint8_t s = mgb::sanitize_char((uint8_t)ch);
        const int f = t.code_of[s], r = t.code_of[mgb::complement_char(s)];
        const bool fv = f >= 1 && f < (int)t.sigma, rv = r >= 1 && r < (int)t.sigma;
        if (fv && rv) {
            ++both;
            if (f + r != 5) { std::printf("byte %d: forward code %d, reverse code %d\n", ch, f, r); ++bad; }
        }
    }
    std::printf("valid on both strands: %d\n", both);
    return bad ? 1 : 0;
}
