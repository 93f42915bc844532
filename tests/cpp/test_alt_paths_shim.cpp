// The C++ IDBGAligner-shaped shim (metagraph_b200/csrc/b200_aligner.hpp) with --align-alternative-alignments N: N = 32
// is served and returns up to 32 alignments of a read that maps to many places; N = 33 throws at construction with the
// library's message. Linked by tests/test_alt_paths_*.py against a C-ABI library.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../metagraph_b200/csrc/b200_aligner.hpp"

int main() {
    // 40 copies of a 30 bp unit with one substitution each, between unique flanks
    const std::string unit = "ACGTTGCATGCCTAGGATCCGATTACAGGC";
    std::string flank_a = "TTGACCAGTAGGCTTAACGGTCAAGTCC", flank_b = "GGCATCGATCGTAAGCTTGCAAGCTTAC";
    std::string refs;
    std::vector<uint64_t> offsets = { 0 };
    for (int c = 0; c < 40; ++c) {
        std::string copy = unit;
        copy[(c * 7) % unit.size()] = "ACGT"[(c + 1) % 4] == copy[(c * 7) % unit.size()] ? 'T' : "ACGT"[(c + 1) % 4];
        std::string fa = flank_a, fb = flank_b;
        fa[c % fa.size()] = "ACGT"[c % 4]; fb[(3 * c) % fb.size()] = "ACGT"[(c + 2) % 4];
        refs += fa + copy + fb;
        offsets.push_back(refs.size());
    }
    mgb_boss_t boss;
    if (mgb_boss_build(refs.data(), offsets.data(), 40, 11, MGB_ALPHABET_DNA, 0, 1, &boss) != MGB_OK) return 2;
    mgb_shim::B200Graph graph(boss.W, boss.last, boss.n_plus_1, boss.F, nullptr, 11);
    mgb_boss_free(&boss);
    mgb_config_t cfg;
    mgb_config_init_cli(&cfg, 11, MGB_ALPHABET_DNA);
    cfg.min_exact_match = 0.0;
    cfg.rel_score_cutoff = 0.0;
    cfg.num_alternative_paths = 32;
    size_t n32 = 0;
    try {
        n32 = mgb_shim::B200Aligner(graph, cfg).align(unit).alignments.size();
    } catch (const std::runtime_error &e) {
        std::printf("n32 threw\t%s\n", e.what());
        return 1;
    }
    std::printf("n32\t%zu\n", n32);
    cfg.num_alternative_paths = 33;
    std::string msg = "no exception";
    try { mgb_shim::B200Aligner a(graph, cfg); } catch (const std::runtime_error &e) { msg = e.what(); }
    std::printf("n33\t%s\n", msg.c_str());
    return n32 == 32 && msg.find("[1, 32]") != std::string::npos ? 0 : 1;
}
