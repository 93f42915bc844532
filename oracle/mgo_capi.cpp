// ORACLE — TEST INFRASTRUCTURE ONLY (see mgo_graph.hpp header).
// Plain C entry points so that tests/ and bench.py (cpu_baseline / --impl reference)
// can drive the CPU restatement through ctypes.
#include "mgo_align.hpp"

#include <cstdlib>
#include <thread>

using namespace mgo;

extern "C" {

// Same field order as include/mgb.h:mgb_config_t (checked by tests/test_abi.py).
struct mgo_config_t {
    uint64_t num_alternative_paths;
    uint64_t min_seed_length;
    uint64_t max_seed_length;
    uint64_t max_num_seeds_per_locus;
    int32_t min_cell_score;
    int32_t min_path_score;
    int32_t xdrop;
    int32_t reserved0;
    double min_exact_match;
    double max_nodes_per_seq_char;
    double max_ram_per_alignment;
    double rel_score_cutoff;
    int8_t gap_opening_penalty;
    int8_t gap_extension_penalty;
    int8_t left_end_bonus;
    int8_t right_end_bonus;
    uint8_t forward_and_reverse_complement;
    uint8_t global_xdrop;
    uint8_t allow_left_trim;
    uint8_t no_backtrack;
    uint8_t seed_complexity_filter;
    uint8_t reserved1[7];
    int8_t score_matrix[128][128];
};

struct mgo_stats_t {
    uint64_t num_seeds, num_extensions, num_explored_nodes, dp_cells, dp_columns;
};

static const Alphabet& alph_of(const char *name) {
    return std::string(name) == "protein" ? Alphabet::protein() : Alphabet::dna();
}

static DBGAlignerConfig to_config(const mgo_config_t &c, const Alphabet &a) {
    DBGAlignerConfig r;
    r.num_alternative_paths = c.num_alternative_paths;
    r.min_seed_length = c.min_seed_length;
    r.max_seed_length = c.max_seed_length;
    r.max_num_seeds_per_locus = c.max_num_seeds_per_locus;
    r.min_cell_score = c.min_cell_score;
    r.min_path_score = c.min_path_score;
    r.xdrop = c.xdrop;
    r.min_exact_match = c.min_exact_match;
    r.max_nodes_per_seq_char = c.max_nodes_per_seq_char;
    r.max_ram_per_alignment = c.max_ram_per_alignment;
    r.rel_score_cutoff = c.rel_score_cutoff;
    r.gap_opening_penalty = c.gap_opening_penalty;
    r.gap_extension_penalty = c.gap_extension_penalty;
    r.left_end_bonus = c.left_end_bonus;
    r.right_end_bonus = c.right_end_bonus;
    r.forward_and_reverse_complement = c.forward_and_reverse_complement;
    r.global_xdrop = c.global_xdrop;
    r.allow_left_trim = c.allow_left_trim;
    r.no_backtrack = c.no_backtrack;
    r.seed_complexity_filter = c.seed_complexity_filter;
    std::memcpy(r.score_matrix, c.score_matrix, sizeof(r.score_matrix));
    r.alphabet = &a;
    return r;
}

uint64_t mgo_config_sizeof() { return sizeof(mgo_config_t); }

void* mgo_graph_build(const char *alphabet, int K, const char **seqs, int n,
                      int mask_dummy, int suffix_index_len, int dynamic_like) {
    try {
        std::vector<std::string> s(seqs, seqs + n);
        auto *g = new DBGSuccinct();
        g->boss = BOSS::build(alph_of(alphabet), K - 1, s, dynamic_like != 0);
        if (suffix_index_len) g->boss.index_suffix_ranges(suffix_index_len);
        if (mask_dummy) g->mask_dummy_kmers();
        return g;
    } catch (...) { return nullptr; }
}

// DeBruijnGraph::Mode of the graph: 0 BASIC, 1 CANONICAL (the caller built it from the sequences and their
// reverse complements, as `metagraph build --mode canonical` does), 2 PRIMARY (the caller built it from contigs
// that hold one k-mer of every reverse-complement pair; the aligner wraps it into CanonicalDBG as the CLI does)
void mgo_graph_set_mode(void *gp, int mode) { static_cast<DBGSuccinct*>(gp)->mode = mode; }

void* mgo_graph_from_arrays(const char *alphabet, int K, const uint8_t *W, const uint8_t *last,
                            uint64_t n_plus_1, const uint64_t *F, int suffix_index_len) {
    try {
        const Alphabet &a = alph_of(alphabet);
        auto *g = new DBGSuccinct();
        g->boss = BOSS::from_arrays(a, K - 1, std::vector<uint8_t>(W, W + n_plus_1),
                                    std::vector<uint8_t>(last, last + n_plus_1),
                                    std::vector<uint64_t>(F, F + a.sigma));
        if (suffix_index_len) g->boss.index_suffix_ranges(suffix_index_len);
        return g;
    } catch (...) { return nullptr; }
}

void mgo_graph_free(void *g) { delete static_cast<DBGSuccinct*>(g); }
uint64_t mgo_graph_num_edges(void *g) { return static_cast<DBGSuccinct*>(g)->boss.num_edges(); }
uint64_t mgo_graph_num_nodes(void *g) { return static_cast<DBGSuccinct*>(g)->num_nodes(); }
void mgo_graph_mask_dummy(void *g, int on) {
    auto *d = static_cast<DBGSuccinct*>(g);
    if (on) d->mask_dummy_kmers(); else d->reset_mask();
}

// W, last: n+1 bytes each; F: sigma entries; valid: n+1 bytes (all 1 except [0] when unmasked)
void mgo_graph_get_arrays(void *g, uint8_t *W, uint8_t *last, uint64_t *F, uint8_t *valid) {
    auto *d = static_cast<DBGSuccinct*>(g);
    std::memcpy(W, d->boss.W.data(), d->boss.W.size());
    std::memcpy(last, d->boss.last.data(), d->boss.last.size());
    std::memcpy(F, d->boss.F.data(), d->boss.F.size() * 8);
    if (valid) {
        for (uint64_t i = 0; i < d->boss.W.size(); ++i) valid[i] = d->in_graph(i);
    }
}

uint64_t mgo_map_to_nodes(void *g, const char *seq, uint64_t len, uint64_t *out) {
    const DBGSuccinct *dbg = static_cast<DBGSuccinct*>(g);
    // a PRIMARY graph is seen through the CanonicalDBG wrapper, as under `metagraph align`
    auto nodes = dbg->mode == 2 ? CanonicalDBG(*dbg).map_to_nodes_sequentially(std::string_view(seq, len))
                                : dbg->map_to_nodes_sequentially(std::string_view(seq, len));
    std::copy(nodes.begin(), nodes.end(), out);
    return nodes.size();
}

// First node DBGSuccinct::call_nodes_with_suffix_matching_longest_prefix reports for `str` (0: none), what
// `metagraph align --map --align-length L` with L < k keeps per position (cli/align.cpp:113-131).
uint64_t mgo_suffix_match_first(void *g, const char *str, uint64_t len, uint64_t min_match_length) {
    const DBGSuccinct *dbg = static_cast<DBGSuccinct*>(g);
    uint64_t first = 0;
    dbg->call_nodes_with_suffix_matching_longest_prefix(std::string_view(str, len),
        [&](uint64_t node, uint64_t) { if (!first) first = node; }, min_match_length);
    return first;
}

// Outgoing (rc = 0) or RCDBG-outgoing (rc = 1) (node, char) pairs in reference order.
int mgo_call_outgoing(void *g, uint64_t node, int rc, uint64_t *nodes, char *chars) {
    GraphView v { static_cast<DBGSuccinct*>(g), rc != 0 };
    int n = 0;
    v.call_outgoing_kmers(node, [&](node_index nn, char c) { nodes[n] = nn; chars[n] = c; ++n; });
    return n;
}

// BOSS primitives for test_boss.cpp-style known-answer checks
uint64_t mgo_boss_fwd(void *g, uint64_t i) {
    auto &b = static_cast<DBGSuccinct*>(g)->boss;
    return b.fwd(i, b.get_W(i) % b.alph_size);
}
uint64_t mgo_boss_bwd(void *g, uint64_t i) { return static_cast<DBGSuccinct*>(g)->boss.bwd(i); }
uint64_t mgo_boss_pick_edge(void *g, uint64_t i, int c) {
    return static_cast<DBGSuccinct*>(g)->boss.pick_edge(i, c);
}
uint64_t mgo_boss_pred_last(void *g, uint64_t i) { return static_cast<DBGSuccinct*>(g)->boss.pred_last(i); }
uint64_t mgo_boss_succ_last(void *g, uint64_t i) { return static_cast<DBGSuccinct*>(g)->boss.succ_last(i); }
uint64_t mgo_boss_rank_W(void *g, uint64_t i, int c) { return static_cast<DBGSuccinct*>(g)->boss.rank_W(i, c); }
uint64_t mgo_boss_rank_last(void *g, uint64_t i) { return static_cast<DBGSuccinct*>(g)->boss.rank_last(i); }
uint64_t mgo_boss_select_last(void *g, uint64_t i) { return static_cast<DBGSuccinct*>(g)->boss.select_last(i); }
// 1 if the source node of edge i has a single incoming edge (BOSS::is_single_incoming(bwd(i), last character))
uint64_t mgo_boss_is_single_incoming(void *g, uint64_t i) {
    auto &b = static_cast<DBGSuccinct*>(g)->boss;
    return b.is_single_incoming(b.bwd(i), b.get_node_last_value(i)) ? 1 : 0;
}
void mgo_node_sequence(void *g, uint64_t node, char *out) {
    std::string s = static_cast<DBGSuccinct*>(g)->get_node_sequence(node);
    std::memcpy(out, s.data(), s.size());
    out[s.size()] = 0;
}

// Seeds of one strand: returns count; each seed -> (clipping, length, offset, first node, num nodes)
// is_low_complexity (aligner_seeder_methods.cpp:21-29) on a raw character string
int mgo_is_low_complexity(const char *seq, uint64_t len) { return is_low_complexity(std::string_view(seq, len)) ? 1 : 0; }

uint64_t mgo_seeds(void *gp, const char *alphabet, const mgo_config_t *cfg, const char *seq,
                   uint64_t len, int orientation, uint64_t *out, uint64_t max_out,
                   uint64_t *num_matching) {
    auto *g = static_cast<DBGSuccinct*>(gp);
    DBGAligner aligner(*g, to_config(*cfg, alph_of(alphabet)));
    AlignmentResults r(std::string_view(seq, len));
    std::string_view q = r.get_query(orientation);
    std::vector<node_index> nodes;
    if (aligner.get_config().max_seed_length >= g->get_k())
        nodes = g->map_to_nodes_sequentially(q);
    else if (q.size() >= g->get_k())
        nodes.resize(q.size() - g->get_k() + 1);
    SeederOutput so = run_seeder(*g, aligner.get_config(), q, orientation, std::move(nodes));
    *num_matching = so.num_matching;
    uint64_t n = 0;
    for (const Seed &s : so.seeds) {
        if (n + 1 > max_out) break;
        out[5 * n + 0] = s.clipping; out[5 * n + 1] = s.query_view.size();
        out[5 * n + 2] = s.offset; out[5 * n + 3] = s.nodes[0]; out[5 * n + 4] = s.nodes.size();
        ++n;
    }
    return so.seeds.size();
}

// Aligns `n` reads with `num_threads` worker threads (contiguous chunks, one aligner per
// chunk — the reference's structure, cli/align.cpp:422-480) and returns a malloc'd
// NUL-terminated buffer with one TSV line per read in input order (cli/align.cpp:254-307).
// If with_nodes != 0 every alignment gets an extra trailing field: comma-joined node ids.
char* mgo_align_tsv(void *gp, const char *alphabet, const mgo_config_t *cfg,
                    const char **headers, const char **seqs, uint64_t n, int num_threads,
                    int with_nodes, mgo_stats_t *stats_out) {
    auto *g = static_cast<DBGSuccinct*>(gp);
    const Alphabet &a = alph_of(alphabet);
    DBGAlignerConfig config = to_config(*cfg, a);
    if (num_threads < 1) num_threads = 1;
    std::vector<std::string> outs(num_threads);
    std::vector<AlignStats> stats(num_threads);
    std::vector<std::string> errors(num_threads);
    auto work = [&](int t) {
        try {
            uint64_t b = n * t / num_threads, e = n * (t + 1) / num_threads;
            std::vector<std::pair<std::string, std::string>> batch;
            for (uint64_t i = b; i < e; ++i) batch.emplace_back(headers[i], seqs[i]);
            DBGAligner aligner(*g, config);
            aligner.align_batch(batch, [&](const std::string &h, AlignmentResults &&r) {
                if (!with_nodes) {
                    outs[t] += format_alignment(h, r, config.min_path_score);
                } else {
                    std::string line = format_alignment(h, r, config.min_path_score);
                    line.pop_back();
                    for (const auto &aln : r.alignments) {
                        line += "\t";
                        for (size_t j = 0; j < aln.get_nodes().size(); ++j)
                            line += (j ? "," : "") + std::to_string(aln.get_nodes()[j]);
                    }
                    outs[t] += line + "\n";
                }
            }, &stats[t]);
        } catch (const std::exception &ex) { errors[t] = ex.what(); }
    };
    if (num_threads == 1) {
        work(0);
    } else {
        std::vector<std::thread> th;
        for (int t = 0; t < num_threads; ++t) th.emplace_back(work, t);
        for (auto &x : th) x.join();
    }
    std::string all;
    for (int t = 0; t < num_threads; ++t) {
        if (!errors[t].empty()) { all = "ERROR: " + errors[t]; break; }
        all += outs[t];
    }
    if (stats_out) {
        std::memset(stats_out, 0, sizeof(*stats_out));
        for (auto &s : stats) {
            stats_out->num_seeds += s.num_seeds; stats_out->num_extensions += s.num_extensions;
            stats_out->num_explored_nodes += s.num_explored_nodes;
            stats_out->dp_cells += s.dp_cells; stats_out->dp_columns += s.dp_columns;
        }
    }
    char *buf = static_cast<char*>(std::malloc(all.size() + 1));
    std::memcpy(buf, all.data(), all.size());
    buf[all.size()] = 0;
    return buf;
}

// Aligns `n` reads on the calling thread as mgo_align_tsv does and reports every evaluation of the extender's
// node and RAM budgets (DefaultColumnExtender::extend: the column's best cell is below the best score so far).
// Each evaluation is a triple (table_size_bytes_, table.size(), window.size()); read_ends[i] is the number of
// triples of reads 0..i. Returns a malloc'd array of all triples, or NULL if the aligner threw.
uint64_t* mgo_align_budget_trace(void *gp, const char *alphabet, const mgo_config_t *cfg, const char **seqs,
                                 uint64_t n, uint64_t *read_ends) {
    auto *g = static_cast<DBGSuccinct*>(gp);
    const Alphabet &a = alph_of(alphabet);
    std::vector<uint64_t> trace;
    try {
        DBGAligner aligner(*g, to_config(*cfg, a));
        std::vector<std::pair<std::string, std::string>> batch;
        for (uint64_t i = 0; i < n; ++i) batch.emplace_back(std::string(), seqs[i]);
        uint64_t i = 0;
        budget_trace = &trace;
        // align_batch finishes a read before it moves on to the next one
        aligner.align_batch(batch, [&](const std::string&, AlignmentResults&&) { read_ends[i++] = trace.size() / 3; });
        budget_trace = nullptr;
    } catch (...) {
        budget_trace = nullptr;
        return nullptr;
    }
    auto *out = static_cast<uint64_t*>(std::malloc(std::max<size_t>(1, trace.size()) * sizeof(uint64_t)));
    std::copy(trace.begin(), trace.end(), out);
    return out;
}

void mgo_free(void *p) { std::free(p); }

} // extern "C"
