// C++ host shim: the reference's aligner interface over the C-ABI of include/mgb.h.
//
//   class IDBGAligner (graph/alignment/dbg_aligner.hpp:20-39)
//       get_graph(), get_config(), align_batch(batch, callback), has_coordinates(), align(query)
//
// Inside the metagraph tree compile with -DMGB_WITH_METAGRAPH: B200Aligner then derives from
// mtg::graph::align::IDBGAligner and hands back real AlignmentResults / Alignment objects
// (alignment.hpp:132-406), so cli/align.cpp:452-458 only has to construct it instead of
// DBGAligner<>. Stand-alone (this repository, where the reference's third-party dependencies are
// absent) the same class works on the POD mirror types below; tests/cpp/test_shim.cpp uses that.
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/mgb.h"

#ifdef MGB_WITH_METAGRAPH
#include "graph/alignment/dbg_aligner.hpp"
#include "graph/representation/succinct/dbg_succinct.hpp"
#endif

namespace mgb_shim {

// ---- index: DBGSuccinct -> HBM ----------------------------------------------------------
class B200Graph {
  public:
    // W / last / F exactly as boss::BOSS holds them (boss.hpp:499-525); valid = dummy mask or
    // nullptr (`metagraph align` drops it, cli/align.cpp:335-339)
    B200Graph(const uint8_t *W, const uint8_t *last, uint64_t n_plus_1, const uint64_t *F,
              const uint8_t *valid, uint32_t k, int device = 0, int alphabet = MGB_ALPHABET_DNA) : k_(k) {
        if (mgb_index_create(W, last, n_plus_1, F, valid, k, alphabet, 0, device, &index_) != MGB_OK)
            throw std::runtime_error(mgb_last_error());
    }
    // A graph file written by `metagraph build` (DBGSuccinct::load, dbg_succinct.cpp:690-712), for callers
    // that do not link MetaGraph. BASIC, CANONICAL and PRIMARY graphs (the latter answer with CanonicalDBG semantics, as under `metagraph align`).
    explicit B200Graph(const std::string &dbg_path, int device = 0) {
        mgb_boss_t boss;
        int mode = -1, state = -1;
        if (mgb_dbg_load(dbg_path.c_str(), &boss, &mode, &state) != MGB_OK)
            throw std::runtime_error(std::string("cannot load ") + dbg_path + ": " + mgb_dbg_last_error());
        k_ = boss.k;
        int rc = mgb_index_create(boss.W, boss.last, boss.n_plus_1, boss.F, nullptr, boss.k,
                                  boss.alphabet, 0, device, &index_);
        mgb_boss_free(&boss);
        if (rc != MGB_OK) throw std::runtime_error(mgb_last_error());
        set_mode(mode);
    }
#ifdef MGB_WITH_METAGRAPH
    // Flatten a loaded DBGSuccinct (get_W / get_last / get_F are public on boss::BOSS).
    explicit B200Graph(const mtg::graph::DBGSuccinct &dbg, int device = 0) : k_(dbg.get_k()) {
        const auto &boss = dbg.get_boss();
        const uint64_t n1 = boss.num_edges() + 1;
        std::vector<uint8_t> W(n1, 0), last(n1, 0), valid;
        // get_W is a wavelet-tree access (a few rank operations): read-only, so all cores share the pass; for a
        // graph that is on disk anyway the .dbg constructor above decodes the tree level by level instead
        #pragma omp parallel for schedule(static)
        for (uint64_t i = 1; i < n1; ++i) { W[i] = boss.get_W(i); last[i] = boss.get_last(i); }
        std::vector<uint64_t> F(boss.alph_size);
        for (size_t c = 0; c < F.size(); ++c) F[c] = boss.get_F(c);
        if (dbg.get_mask()) {
            valid.assign(n1, 0);
            #pragma omp parallel for schedule(static)
            for (uint64_t i = 1; i < n1; ++i) valid[i] = (*dbg.get_mask())[i];
        }
        if (mgb_index_create(W.data(), last.data(), n1, F.data(), valid.empty() ? nullptr : valid.data(),
                             k_, boss.alph_size == 27 ? MGB_ALPHABET_PROTEIN : MGB_ALPHABET_DNA, 0, device,
                             &index_) != MGB_OK)
            throw std::runtime_error(mgb_last_error());
        set_mode(static_cast<int>(dbg.get_mode()));
    }
#endif
    // DeBruijnGraph::Mode of the graph (sequence_graph.hpp:160): 0 BASIC, 1 CANONICAL, 2 PRIMARY
    void set_mode(int mode) {
        if (mgb_index_set_mode(index_, mode) != MGB_OK) {
            std::string err = mgb_last_error();
            mgb_index_destroy(index_);
            index_ = nullptr;
            throw std::runtime_error(err);
        }
    }
    ~B200Graph() { mgb_index_destroy(index_); }
    B200Graph(const B200Graph&) = delete;
    B200Graph& operator=(const B200Graph&) = delete;
    uint32_t get_k() const { return k_; }
    const mgb_index_t* handle() const { return index_; }
  private:
    mgb_index_t *index_ = nullptr;
    uint32_t k_;
};

#ifndef MGB_WITH_METAGRAPH
// POD mirrors of Alignment / AlignmentResults for stand-alone use
struct Alignment {
    bool orientation = false;
    int32_t score = 0;
    size_t offset = 0, query_begin = 0, query_len = 0;
    std::vector<uint64_t> nodes;
    std::string sequence;
    std::vector<std::pair<uint8_t, uint32_t>> cigar;   // (Cigar::Operator, length)
    std::string cigar_string() const {
        static const char ops[] = "SX=DIG";
        std::string s;
        for (auto &p : cigar) s += std::to_string(p.second) + ops[p.first];
        return s;
    }
};
struct AlignmentResults {
    std::string query;               // upper-cased (alignment.cpp:1357-1358)
    std::vector<Alignment> alignments;
};
typedef mgb_config_t DBGAlignerConfig;
#endif

class B200Aligner
#ifdef MGB_WITH_METAGRAPH
    : public mtg::graph::align::IDBGAligner
#endif
{
  public:
    typedef std::pair<std::string, std::string> Query;
#ifdef MGB_WITH_METAGRAPH
    typedef mtg::graph::align::AlignmentResults Results;
    B200Aligner(const mtg::graph::DeBruijnGraph &graph, const B200Graph &index,
                const mtg::graph::align::DBGAlignerConfig &config)
          : graph_(graph), index_(index), config_(config) { lower(config); check(); }
    const mtg::graph::DeBruijnGraph& get_graph() const override { return graph_; }
    const mtg::graph::align::DBGAlignerConfig& get_config() const override { return config_; }
    bool has_coordinates() const override { return false; }
#else
    typedef AlignmentResults Results;
    B200Aligner(const B200Graph &index, const mgb_config_t &config) : index_(index), c_(config) { check(); }
    const mgb_config_t& get_config() const { return c_; }
    bool has_coordinates() const { return false; }
#endif
    typedef std::function<void(const std::string&, Results&&)> AlignmentCallback;

    // dbg_aligner.cpp:251-355: callback(header, results) in input order
    void align_batch(const std::vector<Query> &batch, const AlignmentCallback &callback) const
#ifdef MGB_WITH_METAGRAPH
        override
#endif
    {
        std::string seqs;
        std::vector<uint64_t> offsets(batch.size() + 1, 0);
        for (size_t i = 0; i < batch.size(); ++i) {
            seqs += batch[i].second;
            offsets[i + 1] = seqs.size();
        }
        mgb_results_t *res_raw = nullptr;
        int rc = mgb_align_batch(index_.handle(), &c_, seqs.data(), offsets.data(),
                                 (uint32_t)batch.size(), &res_raw);
        if (rc != MGB_OK) throw std::runtime_error(mgb_last_error());
        // freed on every way out, a throwing callback included
        struct ResultsFree { void operator()(mgb_results_t *r) const { mgb_results_free(r); } };
        std::unique_ptr<mgb_results_t, ResultsFree> res_guard(res_raw);
        const mgb_results_t *res = res_raw;
        const mgb_alignment_t *alns = mgb_results_alignments(res);
        for (size_t i = 0; i < batch.size(); ++i) {
            uint64_t first; uint32_t count;
            mgb_results_read_range(res, (uint32_t)i, &first, &count);
#ifdef MGB_WITH_METAGRAPH
            using namespace mtg::graph::align;
            Results paths(batch[i].second);
            for (uint64_t a = first; a < first + count; ++a) {
                const mgb_alignment_t &x = alns[a];
                Cigar cigar;
                for (uint32_t t = 0; t < x.num_cigar_ops; ++t)
                    cigar.append(static_cast<Cigar::Operator>(x.cigar[t] & 7), x.cigar[t] >> 3);
                size_t clipping = cigar.trim_clipping();
                const std::string &q = paths.get_query(x.orientation);
                paths.emplace_back(std::string_view(q.data() + x.query_begin, x.query_len),
                                   std::vector<Alignment::node_index>(x.nodes, x.nodes + x.num_nodes),
                                   std::string(x.sequence, x.sequence_len), x.score, std::move(cigar),
                                   clipping, x.orientation, x.offset);
            }
#else
            Results paths;
            for (char ch : batch[i].second) {
                int8_t c = (int8_t)ch;
                paths.query.push_back(c >= 0 ? (char)toupper(c) : (char)127);
            }
            for (uint64_t a = first; a < first + count; ++a) {
                const mgb_alignment_t &x = alns[a];
                Alignment al;
                al.orientation = x.orientation; al.score = x.score; al.offset = x.offset;
                al.query_begin = x.query_begin; al.query_len = x.query_len;
                al.nodes.assign(x.nodes, x.nodes + x.num_nodes);
                al.sequence.assign(x.sequence, x.sequence_len);
                for (uint32_t t = 0; t < x.num_cigar_ops; ++t)
                    al.cigar.emplace_back((uint8_t)(x.cigar[t] & 7), x.cigar[t] >> 3);
                paths.alignments.push_back(std::move(al));
            }
#endif
            callback(batch[i].first, std::move(paths));
        }
    }

    // What `metagraph align` prints for the batch (cli/align.cpp:254-307), rendered on the device by mgb_align_batch_text:
    // one TSV line per query, or with json = true one JSON record per alignment, each ending in '\n', in batch order,
    // appended to *out. No AlignmentResults are built; the node ids never leave the device.
    void align_batch_text(const std::vector<Query> &batch, bool json, std::string *out) const {
        std::string seqs, names;
        std::vector<uint64_t> offsets(batch.size() + 1, 0), name_offsets(batch.size() + 1, 0);
        for (size_t i = 0; i < batch.size(); ++i) {
            names += batch[i].first;
            name_offsets[i + 1] = names.size();
            seqs += batch[i].second;
            offsets[i + 1] = seqs.size();
        }
        mgb_results_t *res = nullptr;
        int rc = mgb_align_batch_text(index_.handle(), &c_, seqs.data(), offsets.data(), names.data(),
                                      name_offsets.data(), (uint32_t)batch.size(), json ? MGB_TEXT_JSON : MGB_TEXT_TSV,
                                      &res);
        if (rc != MGB_OK) throw std::runtime_error(mgb_last_error());
        const char *text = nullptr;
        uint64_t bytes = 0;
        rc = mgb_results_text(res, &text, &bytes);
        if (rc == MGB_OK) out->append(text, bytes);
        std::string err = rc == MGB_OK ? "" : mgb_last_error();
        mgb_results_free(res);
        if (rc != MGB_OK) throw std::runtime_error(err);
    }

    Results align(const std::string &query) const {   // IDBGAligner::align (dbg_aligner.cpp:22-31)
        Results result;
        align_batch({ Query{ std::string{}, query } },
                    [&](const std::string&, Results &&r) { result = std::move(r); });
        return result;
    }

  private:
    // the DBGAligner constructor throws for a configuration it cannot run (dbg_aligner.cpp:55-56): so does this one
    void check() const {
        if (mgb_config_check(index_.handle(), &c_) != MGB_OK) throw std::runtime_error(mgb_last_error());
    }
#ifdef MGB_WITH_METAGRAPH
    void lower(const mtg::graph::align::DBGAlignerConfig &c) {
        std::memset(&c_, 0, sizeof(c_));
        c_.num_alternative_paths = c.num_alternative_paths;
        c_.min_seed_length = c.min_seed_length; c_.max_seed_length = c.max_seed_length;
        c_.max_num_seeds_per_locus = c.max_num_seeds_per_locus;
        c_.min_cell_score = c.min_cell_score; c_.min_path_score = c.min_path_score; c_.xdrop = c.xdrop;
        c_.min_exact_match = c.min_exact_match; c_.max_nodes_per_seq_char = c.max_nodes_per_seq_char;
        c_.max_ram_per_alignment = c.max_ram_per_alignment; c_.rel_score_cutoff = c.rel_score_cutoff;
        c_.gap_opening_penalty = c.gap_opening_penalty; c_.gap_extension_penalty = c.gap_extension_penalty;
        c_.left_end_bonus = c.left_end_bonus; c_.right_end_bonus = c.right_end_bonus;
        c_.forward_and_reverse_complement = c.forward_and_reverse_complement;
        c_.global_xdrop = c.global_xdrop; c_.allow_left_trim = c.allow_left_trim;
        c_.no_backtrack = c.no_backtrack; c_.seed_complexity_filter = c.seed_complexity_filter;
        for (int i = 0; i < 128; ++i)
            for (int j = 0; j < 128; ++j) c_.score_matrix[i][j] = c.score_matrix[i][j];
        if (c.chain_alignments || c.post_chain_alignments)
            throw std::runtime_error("B200Aligner: chaining is not supported");
    }
    const mtg::graph::DeBruijnGraph &graph_;
#endif
    const B200Graph &index_;
#ifdef MGB_WITH_METAGRAPH
    mtg::graph::align::DBGAlignerConfig config_;
#endif
    mgb_config_t c_;
};

} // namespace mgb_shim
