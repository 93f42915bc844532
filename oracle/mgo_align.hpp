// ORACLE — TEST INFRASTRUCTURE ONLY (see mgo_graph.hpp header).
//
// CPU restatement of graph/alignment/* for the `metagraph align` hot path:
// DBGAlignerConfig, Cigar, Seed/Alignment, ExactSeeder / MEMSeeder(UniMEM) /
// SuffixSeeder, SeedFilteringExtender + DefaultColumnExtender, the unlabeled
// AlignmentAggregator and DBGAligner::{align_batch, align_both_directions,
// align_core}.  Out of scope (SURVEY §8): chaining, labels, CanonicalDBG, JSON.
#pragma once
#include "mgo_graph.hpp"

#include <limits>
#include <map>
#include <memory>
#include <unordered_map>
#include <unordered_set>

namespace mgo {

typedef int32_t score_t;

// graph/alignment/aligner_config.hpp:18-94
// aligner_seeder_methods.cpp:21-35 (protein builds: always false)
bool is_low_complexity(std::string_view s, int T = 20, int W = 64);

struct DBGAlignerConfig {
    size_t num_alternative_paths = 1;
    size_t min_seed_length = 0;
    size_t max_seed_length = 0;
    size_t max_num_seeds_per_locus = std::numeric_limits<size_t>::max();
    static constexpr score_t ninf = std::numeric_limits<score_t>::min() + 100;
    score_t min_cell_score = ninf;
    score_t min_path_score = 0;
    score_t xdrop = std::numeric_limits<score_t>::max();
    double min_exact_match = 0.0;
    double max_nodes_per_seq_char = std::numeric_limits<double>::max();
    double max_ram_per_alignment = std::numeric_limits<double>::max();
    double rel_score_cutoff = 0.0;
    int8_t gap_opening_penalty = -5;
    int8_t gap_extension_penalty = -2;
    int8_t left_end_bonus = 0;
    int8_t right_end_bonus = 0;
    bool forward_and_reverse_complement = true;
    bool global_xdrop = true;
    bool allow_left_trim = true;
    bool no_backtrack = false;
    bool seed_complexity_filter = false; // sdust is un-vendored: restated from its definition, parity unpinned (mgo_align.cpp)
    int8_t score_matrix[128][128];
    const Alphabet *alphabet = &Alphabet::dna();

    DBGAlignerConfig() { std::memset(score_matrix, 0, sizeof(score_matrix)); }

    score_t score_sequences(std::string_view a, std::string_view b) const {
        score_t s = 0;
        for (size_t i = 0; i < a.size(); ++i) s += score_matrix[(int)a[i]][(int)b[i]];
        return s;
    }
    score_t match_score(std::string_view q) const { return score_sequences(q, q); }
    bool check_config_scores() const;                                  // aligner_config.cpp:39-66
    void set_dna_scoring_matrix(int8_t match, int8_t transition, int8_t transversion); // :164-183
    void set_unit_scoring_matrix(int8_t match);                        // :185-205
    void set_blosum62();                                               // :207-255
};

// graph/alignment/aligner_cigar.hpp:16-109
class Cigar {
  public:
    enum Operator : int8_t { CLIPPED, MISMATCH, MATCH, DELETION, INSERTION, NODE_INSERTION };
    typedef uint32_t LengthType;
    typedef std::pair<Operator, LengthType> value_type;

    Cigar(Operator op = CLIPPED, LengthType num = 0) : cigar_(num ? 1 : 0, std::make_pair(op, num)) {}
    size_t size() const { return cigar_.size(); }
    bool empty() const { return cigar_.empty(); }
    std::string to_string() const;
    void append(Operator op, LengthType num = 1);
    void append(Cigar &&other);
    LengthType trim_clipping();
    LengthType trim_end_clipping();
    LengthType get_clipping() const {
        return cigar_.size() && cigar_.front().first == CLIPPED ? cigar_.front().second : 0;
    }
    LengthType get_end_clipping() const {
        return cigar_.size() && cigar_.back().first == CLIPPED ? cigar_.back().second : 0;
    }
    void extend_clipping(LengthType n);
    std::vector<value_type>& data() { return cigar_; }
    const std::vector<value_type>& data() const { return cigar_; }
    bool operator==(const Cigar &o) const { return cigar_ == o.cigar_; }
    size_t get_num_matches() const;
    bool is_valid(std::string_view reference, std::string_view query) const;
  private:
    std::vector<value_type> cigar_;
};

// alignment.hpp:32-98
struct Seed {
    std::string_view query_view;
    std::vector<node_index> nodes;
    bool orientation = false;
    size_t offset = 0;
    Cigar::LengthType clipping = 0;
    Cigar::LengthType end_clipping = 0;
    bool empty() const { return nodes.empty(); }
    size_t size() const { return nodes.size(); }
};

// alignment.hpp:132-331
class Alignment {
  public:
    Alignment() {}
    Alignment(std::string_view query, std::vector<node_index> &&nodes, std::string &&sequence,
              score_t score, Cigar &&cigar, size_t clipping, bool orientation, size_t offset)
          : query_view_(query), nodes_(std::move(nodes)), orientation_(orientation),
            offset_(offset), sequence_(std::move(sequence)), score_(score),
            cigar_(Cigar::CLIPPED, clipping) { cigar_.append(std::move(cigar)); }
    Alignment(const Seed &seed, const DBGAlignerConfig &config);       // alignment.hpp:154-165

    std::string_view get_query_view() const { return query_view_; }
    bool empty() const { return nodes_.empty(); }
    const std::vector<node_index>& get_nodes() const { return nodes_; }
    std::string_view get_sequence() const { return sequence_; }
    size_t get_offset() const { return offset_; }
    size_t size() const { return nodes_.size(); }
    bool get_orientation() const { return orientation_; }
    score_t get_score() const { return score_; }
    const Cigar& get_cigar() const { return cigar_; }
    Cigar::LengthType get_clipping() const { return cigar_.get_clipping(); }
    Cigar::LengthType get_end_clipping() const { return cigar_.get_end_clipping(); }

    void extend_query_begin(const char *begin);                        // alignment.hpp:209-214
    void extend_query_end(const char *end);                            // alignment.hpp:216-222
    size_t trim_offset();                                              // alignment.cpp:177-190
    void reverse_complement(const GraphView &graph, std::string_view query_rev_comp); // :540-702 (RCDBG branch)
    bool is_valid(const GraphView &graph, const DBGAlignerConfig *config) const;      // :1316-1345

    bool operator==(const Alignment &o) const {
        return orientation_ == o.orientation_ && offset_ == o.offset_ && score_ == o.score_
            && query_view_ == o.query_view_ && sequence_ == o.sequence_
            && cigar_ == o.cigar_ && nodes_ == o.nodes_;
    }
    score_t extra_score = 0;

  private:
    std::string_view query_view_;
    std::vector<node_index> nodes_;
    bool orientation_ = false;
    size_t offset_ = 0;
    std::string sequence_;
    score_t score_ = 0;
    Cigar cigar_;
};

// alignment.hpp:337-348
struct LocalAlignmentLess {
    bool operator()(const Alignment &a, const Alignment &b) const {
        return std::make_tuple(b.get_score(), a.get_query_view().size(),
                               a.get_orientation(), a.get_clipping())
            > std::make_tuple(a.get_score(), b.get_query_view().size(),
                              b.get_orientation(), b.get_clipping());
    }
};

// alignment.hpp:366-406, alignment.cpp:1348-1372
class AlignmentResults {
  public:
    explicit AlignmentResults(std::string_view query = {});
    AlignmentResults(const AlignmentResults&) = delete;
    AlignmentResults(AlignmentResults&&) = default;
    AlignmentResults& operator=(AlignmentResults&&) = default;
    const std::string& get_query(bool rc = false) const { return rc ? *query_rc_ : *query_; }
    std::vector<Alignment> alignments;
  private:
    // heap-allocated so that string_views stay valid when the object is moved
    std::unique_ptr<std::string> query_, query_rc_;
};

// Per-read counters (dbg_aligner.cpp:341-351 trace line)
struct AlignStats {
    size_t num_seeds = 0, num_extensions = 0, num_explored_nodes = 0;
    uint64_t dp_cells = 0, dp_columns = 0;
};

// dbg_aligner.hpp:42-99 with Seeder = SuffixSeeder<UniMEMSeeder>, Extender = DefaultColumnExtender
class DBGAligner {
  public:
    DBGAligner(const DBGSuccinct &graph, const DBGAlignerConfig &config); // dbg_aligner.cpp:33-61
    const DBGAlignerConfig& get_config() const { return config_; }
    // dbg_aligner.cpp:251-355; callback(header, results) in input order
    void align_batch(const std::vector<std::pair<std::string, std::string>> &batch,
                     const std::function<void(const std::string&, AlignmentResults&&)> &callback,
                     AlignStats *stats = nullptr) const;
    AlignmentResults align(std::string_view query) const;
  private:
    const DBGSuccinct &graph_;
    // PRIMARY graphs are aligned to through the CanonicalDBG wrapper, as `metagraph align` does
    // (cli/align.cpp primary_to_canonical; dbg_aligner.cpp:52-53 asserts it)
    std::unique_ptr<CanonicalDBG> canonical_;
    DBGAlignerConfig config_;
};

// Not in the reference: when non-null, the extender of the calling thread appends one triple
// (table_size_bytes_, table.size(), window.size()) each time it evaluates its node and RAM budgets
// (the stop tests of DefaultColumnExtender::extend). Test infrastructure for the budget tests.
extern thread_local std::vector<uint64_t> *budget_trace;

// cli/align.cpp:254-307 (TSV branch) + alignment.hpp:418-435
std::string format_alignment(const std::string &header, const AlignmentResults &paths,
                             score_t min_path_score);

// exposed for unit tests of the seeding stage
struct SeederOutput {
    std::vector<Seed> seeds;
    size_t num_matching = 0;
};
SeederOutput run_seeder(const DBGSuccinct &graph, const DBGAlignerConfig &config,
                        std::string_view query, bool orientation,
                        std::vector<node_index> &&nodes, const CanonicalDBG *canon = nullptr);

} // namespace mgo
