// The C++ shim's text method (metagraph_b200/csrc/b200_aligner.hpp B200Aligner::align_batch_text): reads the graph file
// given as argv[1], aligns a small batch with headers and writes the TSV block, a line "--", then the JSON block to
// stdout. tests/test_text_output_*.py compare both blocks with the Python binding's text of the same batch.
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../metagraph_b200/csrc/b200_aligner.hpp"

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    try {
        mgb_shim::B200Graph graph(argv[1]);
        mgb_config_t cfg;
        mgb_config_init_cli(&cfg, graph.get_k(), MGB_ALPHABET_DNA);
        cfg.min_exact_match = 0.0;
        cfg.num_alternative_paths = 2;
        mgb_shim::B200Aligner aligner(graph, cfg);
        const std::vector<mgb_shim::B200Aligner::Query> batch = {
            { "q1", "AGCTNCGAGGCCAA" }, { "q\t2 \"x\"", "TTGGCCTCGNAGCT" }, { "", "" }, { "q4", "ACGTACGTNNN" },
            { "q5", "agctncgaggccaa" },
        };
        std::string tsv, json;
        aligner.align_batch_text(batch, false, &tsv);
        aligner.align_batch_text(batch, true, &json);
        std::fwrite(tsv.data(), 1, tsv.size(), stdout);
        std::printf("--\n");
        std::fwrite(json.data(), 1, json.size(), stdout);
    } catch (const std::runtime_error &e) {
        std::printf("threw\t%s\n", e.what());
        return 1;
    }
    return 0;
}
