// ORACLE — TEST INFRASTRUCTURE ONLY (see mgo_graph.hpp header).
// Restatement of graph/alignment/* (reference paths relative to metagraph/src).
#include "mgo_align.hpp"

#include <cctype>
#include <cmath>
#include <queue>
#include <stdexcept>

namespace mgo {

static constexpr score_t ninf = DBGAlignerConfig::ninf;

// ---------------------------------------------------------------------------
// DBGAlignerConfig (aligner_config.cpp)
// ---------------------------------------------------------------------------
bool DBGAlignerConfig::check_config_scores() const {
    int8_t min_penalty_score = std::numeric_limits<int8_t>::max();
    for (int i = 0; i < 128; ++i)
        for (int j = 0; j < 128; ++j)
            min_penalty_score = std::min(min_penalty_score, score_matrix[i][j]);
    if (gap_opening_penalty * 2 >= min_penalty_score)
        return false;
    min_penalty_score = std::min({ min_penalty_score, gap_opening_penalty, gap_extension_penalty });
    if (min_cell_score >= std::numeric_limits<score_t>::min() - min_penalty_score)
        return true;
    return false;
}

void DBGAlignerConfig::set_dna_scoring_matrix(int8_t match, int8_t transition, int8_t transversion) {
    std::memset(score_matrix, transversion, sizeof(score_matrix));
    score_matrix['A']['G'] = score_matrix['G']['A'] = transition;
    score_matrix['C']['T'] = score_matrix['T']['C'] = transition;
    for (char c : std::string("ACGT")) score_matrix[(int)c][(int)c] = match;
}

// letters counted as valid by the non-BOSS alphabets (kmer/alphabets.hpp:85-161):
// DNA "ACGT"; protein: every letter except 'X' (code 25 == invalid code)
static std::string valid_upper_letters(const Alphabet &a) {
    return a.sigma == 5 ? std::string("ACGT") : std::string("ABCDEFGHIJKLMNOPQRSTUVWYZ");
}

void DBGAlignerConfig::set_unit_scoring_matrix(int8_t match) {
    std::memset(score_matrix, -match, sizeof(score_matrix));
    for (char c : valid_upper_letters(*alphabet)) score_matrix[(int)c][(int)c] = match;
}

void DBGAlignerConfig::set_blosum62() {
    // Standard BLOSUM62 (public NCBI table), rows/cols in the order below.
    static const char *order = "ARNDCQEGHILKMFPSTWYVBZX";
    static const int8_t b62[23][23] = {
        { 4,-1,-2,-2, 0,-1,-1, 0,-2,-1,-1,-1,-1,-2,-1, 1, 0,-3,-2, 0,-2,-1, 0},
        {-1, 5, 0,-2,-3, 1, 0,-2, 0,-3,-2, 2,-1,-3,-2,-1,-1,-3,-2,-3,-1, 0,-1},
        {-2, 0, 6, 1,-3, 0, 0, 0, 1,-3,-3, 0,-2,-3,-2, 1, 0,-4,-2,-3, 3, 0,-1},
        {-2,-2, 1, 6,-3, 0, 2,-1,-1,-3,-4,-1,-3,-3,-1, 0,-1,-4,-3,-3, 4, 1,-1},
        { 0,-3,-3,-3, 9,-3,-4,-3,-3,-1,-1,-3,-1,-2,-3,-1,-1,-2,-2,-1,-3,-3,-2},
        {-1, 1, 0, 0,-3, 5, 2,-2, 0,-3,-2, 1, 0,-3,-1, 0,-1,-2,-1,-2, 0, 3,-1},
        {-1, 0, 0, 2,-4, 2, 5,-2, 0,-3,-3, 1,-2,-3,-1, 0,-1,-3,-2,-2, 1, 4,-1},
        { 0,-2, 0,-1,-3,-2,-2, 6,-2,-4,-4,-2,-3,-3,-2, 0,-2,-2,-3,-3,-1,-2,-1},
        {-2, 0, 1,-1,-3, 0, 0,-2, 8,-3,-3,-1,-2,-1,-2,-1,-2,-2, 2,-3, 0, 0,-1},
        {-1,-3,-3,-3,-1,-3,-3,-4,-3, 4, 2,-3, 1, 0,-3,-2,-1,-3,-1, 3,-3,-3,-1},
        {-1,-2,-3,-4,-1,-2,-3,-4,-3, 2, 4,-2, 2, 0,-3,-2,-1,-2,-1, 1,-4,-3,-1},
        {-1, 2, 0,-1,-3, 1, 1,-2,-1,-3,-2, 5,-1,-3,-1, 0,-1,-3,-2,-2, 0, 1,-1},
        {-1,-1,-2,-3,-1, 0,-2,-3,-2, 1, 2,-1, 5, 0,-2,-1,-1,-1,-1, 1,-3,-1,-1},
        {-2,-3,-3,-3,-2,-3,-3,-3,-1, 0, 0,-3, 0, 6,-4,-2,-2, 1, 3,-1,-3,-3,-1},
        {-1,-2,-2,-1,-3,-1,-1,-2,-2,-3,-3,-1,-2,-4, 7,-1,-1,-4,-3,-2,-2,-1,-2},
        { 1,-1, 1, 0,-1, 0, 0, 0,-1,-2,-2, 0,-1,-2,-1, 4, 1,-3,-2,-2, 0, 0, 0},
        { 0,-1, 0,-1,-1,-1,-1,-2,-2,-1,-1,-1,-1,-2,-1, 1, 5,-2,-2, 0,-1,-1, 0},
        {-3,-3,-4,-4,-2,-2,-3,-2,-2,-3,-2,-3,-1, 1,-4,-3,-2,11, 2,-3,-4,-3,-2},
        {-2,-2,-2,-3,-2,-1,-2,-3, 2,-1,-1,-2,-1, 3,-3,-2,-2, 2, 7,-1,-3,-2,-1},
        { 0,-3,-3,-3,-1,-2,-2,-3,-3, 3, 1,-2, 1,-1,-2,-2, 0,-3,-1, 4,-3,-2,-1},
        {-2,-1, 3, 4,-3, 0, 1,-1, 0,-3,-4, 0,-3,-3,-2, 0,-1,-4,-3,-3, 4, 1,-1},
        {-1, 0, 0, 1,-3, 3, 4,-2, 0,-3,-3, 1,-1,-3,-1, 0,-1,-3,-2,-2, 1, 4,-1},
        { 0,-1,-1,-1,-2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-2, 0, 0,-2,-1,-1,-1,-1,-1}
    };
    for (int i = 0; i < 128; ++i) {
        for (int j = 0; j < 128; ++j) score_matrix[i][j] = -4;
        score_matrix[i][i] = 1; // J, O, U (aligner_config.cpp:238-243)
    }
    for (int i = 0; i < 23; ++i)
        for (int j = 0; j < 23; ++j)
            score_matrix[(int)order[i]][(int)order[j]] = b62[i][j];
}

// is_low_complexity (aligner_seeder_methods.cpp:21-35) = sdust(seq, T = 20, W = 64) finds at least one
// interval. sdust (hmusta/sdust, a fork of lh3/sdust = symmetric DUST, Morgulis et al. 2006) is NOT vendored
// in the reference tree; this restates its published definition — PARITY UNPINNED against the library:
// over the 3-mers of every maximal A/C/G/T run, an interval of l + 1 consecutive 3-mers (at most W - 2 of
// them) is low-complexity when 10 * sum_t c_t (c_t - 1) / 2 > T * l, c_t = occurrences of 3-mer t in it;
// some interval is "perfect" (reported) iff some interval exceeds the threshold.
bool is_low_complexity(std::string_view s, int T, int W) {
    auto nt4 = [](char c) -> int {
        switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2;
                     case 'T': case 't': case 'U': case 'u': return 3; default: return 4; }
    };
    const int max_words = W - 2;
    std::vector<int> words;          // 3-mer at every position of the current run
    size_t i = 0;
    auto scan_run = [&]() -> bool {
        const int n = (int)words.size();
        for (int a = 0; a < n; ++a) {
            int cnt[64] = { 0 };
            int r = 0;
            for (int b = a; b < n && b - a < max_words; ++b) {
                r += cnt[words[b]]++;
                if (b > a && r * 10 > T * (b - a)) return true;
            }
        }
        return false;
    };
    while (i <= s.size()) {
        int run = 0, w = 0;
        words.clear();
        for (; i < s.size() && nt4(s[i]) < 4; ++i) {
            w = ((w << 2) | nt4(s[i])) & 63;
            if (++run >= 3) words.push_back(w);
        }
        if (scan_run()) return true;
        ++i;                         // skip the non-ACGT character (or step past the end)
    }
    return false;
}

// aligner_cigar.cpp:11-51: kCharToOp
static Cigar::Operator char_to_op(const Alphabet &a, char ref, char q) {
    // MATCH iff both are the same valid letter, case-insensitively
    if (ref < 0 || q < 0) return Cigar::MISMATCH;
    char ur = toupper(ref), uq = toupper(q);
    if (ur != uq) return Cigar::MISMATCH;
    return valid_upper_letters(a).find(ur) != std::string::npos ? Cigar::MATCH : Cigar::MISMATCH;
}

// ---------------------------------------------------------------------------
// Cigar (aligner_cigar.cpp)
// ---------------------------------------------------------------------------
std::string Cigar::to_string() const {
    static const char op_str[] = "SX=DIG";
    std::string s;
    for (const auto &p : cigar_) s += std::to_string(p.second) + op_str[p.first];
    return s;
}

void Cigar::append(Operator op, LengthType num) {
    if (!num) return;
    if (cigar_.empty() || cigar_.back().first != op) cigar_.emplace_back(op, num);
    else cigar_.back().second += num;
}

void Cigar::append(Cigar &&other) {
    if (other.empty()) return;
    append(other.cigar_.front().first, other.cigar_.front().second);
    cigar_.insert(cigar_.end(), std::next(other.cigar_.begin()), other.cigar_.end());
}

Cigar::LengthType Cigar::trim_clipping() {
    if (cigar_.size() && cigar_.front().first == CLIPPED) {
        LengthType r = cigar_.front().second;
        cigar_.erase(cigar_.begin());
        return r;
    }
    return 0;
}

Cigar::LengthType Cigar::trim_end_clipping() {
    if (cigar_.size() && cigar_.back().first == CLIPPED) {
        LengthType r = cigar_.back().second;
        cigar_.pop_back();
        return r;
    }
    return 0;
}

void Cigar::extend_clipping(LengthType n) {
    if (cigar_.front().first != CLIPPED) cigar_.insert(cigar_.begin(), value_type(CLIPPED, n));
    else cigar_.front().second += n;
}

size_t Cigar::get_num_matches() const {
    size_t n = 0;
    for (const auto &p : cigar_) n += (p.first == MATCH) * p.second;
    return n;
}

bool Cigar::is_valid(std::string_view reference, std::string_view query) const {
    auto ref_it = reference.begin();
    auto alt_it = query.begin();
    for (size_t i = 0; i < cigar_.size(); ++i) {
        const auto &op = cigar_[i];
        if (!op.second) return false;
        switch (op.first) {
            case CLIPPED:
                if ((ref_it != reference.begin() || alt_it != query.begin())
                        && (ref_it != reference.end() || alt_it != query.end())) {
                    if (alt_it > query.end() - op.second) return false;
                    alt_it += op.second;
                }
                break;
            case MATCH:
            case MISMATCH:
                if (ref_it > reference.end() - op.second) return false;
                if (alt_it > query.end() - op.second) return false;
                if (std::equal(ref_it, ref_it + op.second, alt_it) == (op.first != MATCH)) return false;
                ref_it += op.second; alt_it += op.second;
                break;
            case INSERTION:
                if (i && cigar_[i - 1].first == DELETION) return false;
                if (alt_it > query.end() - op.second) return false;
                alt_it += op.second;
                break;
            case DELETION:
                if (i && cigar_[i - 1].first == INSERTION) return false;
                if (ref_it > reference.end() - op.second) return false;
                ref_it += op.second;
                break;
            case NODE_INSERTION: break;
        }
    }
    return ref_it == reference.end() && alt_it == query.end();
}

// aligner_config.cpp:68-126
static score_t score_cigar(const DBGAlignerConfig &c, std::string_view reference,
                           std::string_view query, const Cigar &cigar) {
    if (cigar.empty()) return 0;
    score_t score = (!cigar.get_clipping() ? c.left_end_bonus : 0)
                    + (!cigar.get_end_clipping() ? c.right_end_bonus : 0);
    size_t ref_i = 0, alt_i = 0;
    auto it = cigar.data().begin();
    if (it->first == Cigar::CLIPPED) ++it;
    for (; it != cigar.data().end(); ++it) {
        switch (it->first) {
            case Cigar::CLIPPED:
                if (it + 1 != cigar.data().end()) alt_i += it->second;
                break;
            case Cigar::MATCH:
                score += c.match_score(reference.substr(ref_i, it->second));
                ref_i += it->second; alt_i += it->second;
                break;
            case Cigar::MISMATCH:
                score += c.score_sequences(reference.substr(ref_i, it->second),
                                           query.substr(alt_i, it->second));
                ref_i += it->second; alt_i += it->second;
                break;
            case Cigar::INSERTION:
                score += c.gap_opening_penalty + (it->second - 1) * c.gap_extension_penalty;
                alt_i += it->second;
                break;
            case Cigar::DELETION:
                score += c.gap_opening_penalty + (it->second - 1) * c.gap_extension_penalty;
                ref_i += it->second;
                break;
            case Cigar::NODE_INSERTION:
                score += c.gap_opening_penalty + (it->second - 1) * c.gap_extension_penalty;
                break;
        }
    }
    return score;
}

// ---------------------------------------------------------------------------
// Alignment
// ---------------------------------------------------------------------------
Alignment::Alignment(const Seed &seed, const DBGAlignerConfig &config)
      : query_view_(seed.query_view), nodes_(seed.nodes), orientation_(seed.orientation),
        offset_(seed.offset), sequence_(seed.query_view),
        score_(config.match_score(seed.query_view)
                 + (!seed.clipping ? config.left_end_bonus : 0)
                 + (!seed.end_clipping ? config.right_end_bonus : 0)),
        cigar_(Cigar::CLIPPED, seed.clipping) {
    cigar_.append(Cigar::MATCH, query_view_.size());
    cigar_.append(Cigar::CLIPPED, seed.end_clipping);
}

void Alignment::extend_query_begin(const char *begin) {
    const char *full_query_begin = query_view_.data() - get_clipping();
    if (full_query_begin > begin)
        cigar_.extend_clipping(full_query_begin - begin);
}

void Alignment::extend_query_end(const char *end) {
    const char *full_query_end = query_view_.data() + query_view_.size() + get_end_clipping();
    if (full_query_end < end)
        cigar_.append(Cigar::CLIPPED, end - full_query_end);
}

size_t Alignment::trim_offset() {
    if (!offset_ || nodes_.size() <= 1)
        return 0;
    size_t first_dummy = (std::find(nodes_.begin(), nodes_.end(), npos) - nodes_.begin()) - 1;
    size_t trim = std::min(std::min(offset_, nodes_.size() - 1), first_dummy);
    offset_ -= trim;
    nodes_.erase(nodes_.begin(), nodes_.begin() + trim);
    return trim;
}

void Alignment::reverse_complement(const GraphView &graph, std::string_view query_rev_comp) {
    trim_offset();
    if (graph.rc) {
        // alignment.cpp:547-561
        if (offset_) {
            *this = Alignment();
        } else {
            std::reverse(cigar_.data().begin(), cigar_.data().end());
            std::reverse(nodes_.begin(), nodes_.end());
            reverse_complement_inplace(sequence_);
            orientation_ = !orientation_;
            query_view_ = { query_rev_comp.data() + get_clipping(),
                            query_rev_comp.size() - get_clipping() - get_end_clipping() };
        }
        return;
    }
    // alignment.cpp:563-702 on a CANONICAL-mode DBGSuccinct (the path of the reverse complement is looked up in
    // the graph itself) or on a PRIMARY graph behind CanonicalDBG (the node ids are flipped)
    const DBGSuccinct &dbg = *graph.g;
    const CanonicalDBG *canonical = graph.canon;
    auto rc_seq_path = [&]() {                                // reverse_complement_seq_path, sequence_graph.cpp:563-573
        if (canonical) {
            canonical->reverse_complement(sequence_, nodes_);
            return;
        }
        reverse_complement_inplace(sequence_);
        nodes_ = dbg.map_to_nodes_sequentially(sequence_);
    };
    if (!offset_) {
        rc_seq_path();
    } else {
        sequence_ = graph.get_node_sequence(nodes_[0]).substr(0, offset_) + sequence_;
        if (sequence_[0] == '$') {
            // starts in a source dummy k-mer: walk forward (always the last outgoing edge) until the k-mer is
            // real, then take its reverse complement (:572-640)
            size_t num_sentinels = sequence_.find_last_of('$') + 1;
            if (canonical && nodes_[0] != canonical->get_base_node(nodes_[0])) {
                *this = Alignment();                          // reverse complement of a sink dummy k-mer
                return;
            }
            size_t num_first_steps = canonical ? std::min(offset_, num_sentinels) : offset_;
            const BOSS &boss = dbg.boss;
            edge_index edge = nodes_[0];
            TAlphabet edge_label = boss.get_W(edge) % boss.alph_size;
            for (size_t i = 0; i < num_first_steps; ++i) {
                edge = boss.fwd(edge, edge_label);
                edge_label = boss.get_W(edge) % boss.alph_size;
                if (edge_label == 0) { *this = Alignment(); return; }
                nodes_[0] = dbg.validate_edge(edge);
                sequence_.push_back(boss.alph->decode(edge_label));
            }
            for (size_t i = num_first_steps; i < offset_; ++i) {
                node_index next_node = 0;
                char last_char = 0;
                canonical->call_outgoing_kmers(nodes_[0], [&](node_index next, char c) {
                    if (c == '$')
                        return;
                    next_node = next;
                    last_char = c;
                });
                if (!next_node) { *this = Alignment(); return; }
                nodes_[0] = next_node;
                sequence_.push_back(last_char);
            }
            sequence_ = sequence_.substr(offset_);
            rc_seq_path();
            if (std::find(nodes_.begin(), nodes_.end(), npos) != nodes_.end()) { *this = Alignment(); return; }
            sequence_.assign(sequence_.data() + offset_, dbg.get_k() - offset_);
        } else {
            rc_seq_path();
            if (std::find(nodes_.begin(), nodes_.end(), npos) != nodes_.end()) { *this = Alignment(); return; }
            // trim the ending that corresponds to the added prefix (:667-690): first incoming node each time
            for (size_t i = 0; i < offset_; ++i) {
                size_t indegree = 0;
                node_index first_prev = npos;
                graph.adjacent_incoming_nodes(nodes_[0], [&](node_index prev) { if (++indegree == 1) first_prev = prev; });
                if (!indegree) { *this = Alignment(); return; }
                nodes_[0] = first_prev;
                sequence_.pop_back();
            }
        }
    }
    std::reverse(cigar_.data().begin(), cigar_.data().end());
    orientation_ = !orientation_;
    query_view_ = { query_rev_comp.data() + get_clipping(),
                    query_rev_comp.size() - get_clipping() - get_end_clipping() };
}

// alignment.cpp:1239-1314 (no npos nodes: chaining is out of scope)
static std::string spell_path(const GraphView &graph, const std::vector<node_index> &path, size_t offset) {
    std::string seq;
    if (path.empty()) return seq;
    seq += graph.get_node_sequence(path.front()).substr(offset);
    for (size_t i = 1; i < path.size(); ++i) {
        char next = '\0';
        graph.call_outgoing_kmers(path[i - 1], [&](node_index nn, char c) {
            if (nn == path[i]) next = c;
        });
        if (!next) throw std::runtime_error("invalid edge");
        seq += next;
    }
    return seq;
}

bool Alignment::is_valid(const GraphView &graph, const DBGAlignerConfig *config) const {
    if (empty()) return true;
    try {
        if (spell_path(graph, nodes_, offset_) != sequence_) return false;
    } catch (const std::runtime_error&) { return false; }
    if (!cigar_.is_valid(sequence_, query_view_)) return false;
    if (config && score_ != score_cigar(*config, sequence_, query_view_, cigar_) + extra_score)
        return false;
    return true;
}

AlignmentResults::AlignmentResults(std::string_view query) {
    query_ = std::make_unique<std::string>();
    query_->reserve(std::max(query.size(), sizeof(std::string)) + 8);
    for (char ch : query) {
        int8_t c = ch;
        query_->push_back(c >= 0 ? toupper(c) : 127);
    }
    query_rc_ = std::make_unique<std::string>(*query_);
    reverse_complement_inplace(*query_rc_);
}

// ---------------------------------------------------------------------------
// Seeders (aligner_seeder_methods.cpp)
// ---------------------------------------------------------------------------
namespace {

struct SeederBase {
    const DBGSuccinct &graph;
    std::string_view query;
    bool orientation;
    std::vector<node_index> query_nodes;
    const DBGAlignerConfig &config;
    size_t num_matching = 0;
    const CanonicalDBG *canon = nullptr;       // set when the aligner's graph is a PRIMARY graph behind CanonicalDBG

    bool has_multiple_outgoing(node_index n) const {
        return canon ? canon->has_multiple_outgoing(n) : graph.has_multiple_outgoing(n);
    }
    bool has_single_incoming(node_index n) const {
        return canon ? canon->has_single_incoming(n) : graph.has_single_incoming(n);
    }

    // :49-65
    size_t num_exact_matching() const {
        size_t nm = 0, last_match_count = 0;
        size_t k = graph.get_k();
        for (auto it = query_nodes.begin(); it != query_nodes.end(); ++it) {
            if (*it) {
                auto jt = std::find(it + 1, query_nodes.end(), node_index(0));
                nm += k + std::distance(it, jt) - 1 - last_match_count;
                last_match_count = k;
                it = jt - 1;
            } else if (last_match_count) {
                --last_match_count;
            }
        }
        return nm;
    }

    // ExactSeeder::get_seeds :67-93
    std::vector<Seed> exact_seeds() const {
        size_t k = graph.get_k();
        if (num_matching < config.min_exact_match * query.size())
            return {};
        std::vector<Seed> seeds;
        if (config.max_seed_length < k)
            return seeds;
        size_t end_clipping = query.size() - k;
        for (size_t i = 0; i < query_nodes.size(); ++i, --end_clipping) {
            if (query_nodes[i] != npos) {
                if (config.seed_complexity_filter && config.alphabet->sigma == 5
                        && is_low_complexity(query.substr(i, k)))
                    continue;                                              // :84
                Seed s;
                s.query_view = query.substr(i, k);
                s.nodes = { query_nodes[i] };
                s.orientation = orientation;
                s.offset = 0; s.clipping = i; s.end_clipping = end_clipping;
                seeds.push_back(std::move(s));
            }
        }
        return seeds;
    }

    // MEMSeeder::get_seeds :360-424 with the UniMEM terminator (seeder.hpp:116-135)
    std::vector<Seed> mem_seeds() const {
        size_t k = graph.get_k();
        if (k >= config.max_seed_length)
            return exact_seeds();
        if (num_matching < config.min_exact_match * query.size())
            return {};
        std::vector<uint8_t> flags(query_nodes.size(), 0);
        for (size_t i = 0; i < flags.size(); ++i) {
            if (query_nodes[i] != npos) {
                flags[i] = 2 | (i + 1 == query_nodes.size()
                                || query_nodes[i + 1] == npos
                                || has_multiple_outgoing(query_nodes[i])
                                || !has_single_incoming(query_nodes[i]));
            }
        }
        std::vector<Seed> seeds;
        auto it = flags.begin();
        while ((it = std::find_if(it, flags.end(), [](uint8_t f) { return f & 2; })) != flags.end()) {
            auto next = std::find_if(it, flags.end(),
                                     [](uint8_t f) { return (f & 1) == 1 || (f & 2) == 0; });
            if (next != flags.end() && ((*next) & 2))
                ++next;
            size_t i = it - flags.begin();
            size_t mem_length = (next - it) + k - 1;
            if (mem_length >= config.min_seed_length) {
                Seed s;
                s.query_view = query.substr(i, mem_length);
                s.nodes.assign(query_nodes.begin() + i, query_nodes.begin() + i + (next - it));
                s.orientation = orientation;
                s.offset = 0; s.clipping = i; s.end_clipping = query.size() - i - mem_length;
                seeds.push_back(std::move(s));
            }
            it = next;
        }
        return seeds;
    }

    // SuffixSeeder<UniMEMSeeder>::generate_seeds :153-358
    std::vector<Seed> suffix_seeds() {
        std::vector<Seed> seeds_;
        size_t k = graph.get_k();
        if (query.size() < config.min_seed_length)
            return seeds_;
        if (config.min_seed_length >= k)
            return mem_seeds();

        size_t n_pos = query.size() - config.min_seed_length + 1;
        std::vector<std::vector<Seed>> suffix_seeds(n_pos);
        std::vector<size_t> min_seed_length(n_pos, config.min_seed_length);

        for (auto &&seed : mem_seeds()) {
            size_t i = seed.clipping;
            for (size_t j = 0; j < seed.size(); ++j)
                min_seed_length[i + j] = k;
            if (i + seed.size() < min_seed_length.size())
                min_seed_length[i + seed.size()] = k;
            suffix_seeds[i].emplace_back(std::move(seed));
        }

        auto append_suffix_seed = [&](size_t i, node_index alt_node, size_t seed_length) {
            std::string_view seed_seq = query.substr(i, seed_length);
            if (seed_length > min_seed_length[i])
                suffix_seeds[i].clear();
            min_seed_length[i] = seed_length;
            Seed s;
            s.query_view = seed_seq;
            s.nodes = { alt_node };
            s.orientation = orientation;
            s.offset = k - seed_length;
            s.clipping = i;
            s.end_clipping = query.size() - i - seed_seq.size();
            suffix_seeds[i].push_back(std::move(s));
            for (++i; i < min_seed_length.size() && seed_length > min_seed_length[i]; ++i) {
                min_seed_length[i] = seed_length--;
                suffix_seeds[i].clear();
            }
        };

        size_t last_full_id = query.size() >= k ? query.size() - k + 1 : min_seed_length.size();
        for (size_t i = 0; i < min_seed_length.size(); ++i) {
            size_t max_seed_length = std::min({ config.max_seed_length, k - 1, query.size() - i });
            size_t seed_length = 0;
            std::vector<node_index> alt_nodes;
            if (config.seed_complexity_filter && config.alphabet->sigma == 5
                    && is_low_complexity(query.substr(i, min_seed_length[i])))
                continue;                                                  // :226-229
            graph.call_nodes_with_suffix_matching_longest_prefix(
                query.substr(i, max_seed_length),
                [&](node_index alt, uint64_t len) { seed_length = len; alt_nodes.push_back(alt); },
                min_seed_length[i]);
            if (i >= last_full_id && alt_nodes.size() == 1
                    && min_seed_length[last_full_id - 1] == k
                    && suffix_seeds[last_full_id - 1].size() == 1
                    && alt_nodes[0] == suffix_seeds[last_full_id - 1][0].nodes[0])
                continue;
            for (node_index alt : alt_nodes)
                append_suffix_seed(i, alt, seed_length);
        }

        if (canon) {
            // sub-k matches of the reverse complement (:251-314): a prefix of query_rc[i..] that is the suffix
            // of nodes, turned into nodes whose reverse complement starts with the match (suffix_to_prefix :95-139)
            const BOSS &boss = graph.boss;
            std::string query_rc(query);
            reverse_complement_inplace(query_rc);
            for (size_t i = 0; i + config.min_seed_length <= query_rc.size(); ++i) {
                size_t max_seed_length = std::min({ config.max_seed_length, k - 1, query.size() - i });
                size_t j_min = query_rc.size() - i - max_seed_length;
                size_t j_max = query_rc.size() - i - config.min_seed_length;
                while (j_min <= j_max && min_seed_length[j_min] > max_seed_length) {
                    ++j_min;
                    --max_seed_length;
                }
                if (j_min > j_max)
                    continue;
                std::vector<TAlphabet> encoded = boss.alph->encode(std::string_view(query_rc.data() + i, max_seed_length));
                auto [first, last, end] = boss.index_range(encoded.data(), encoded.data() + encoded.size());
                size_t seed_length = end - encoded.data();
                size_t j = query_rc.size() - i - seed_length;
                if (seed_length < config.min_seed_length
                        || seed_length < min_seed_length[j]
                        || (config.seed_complexity_filter && config.alphabet->sigma == 5
                                && is_low_complexity(query.substr(j, seed_length))))
                    continue;
                typedef std::tuple<edge_index, edge_index, size_t> Range;
                auto call_nodes_in_range = [&](const Range &r) {
                    for (edge_index e = std::get<0>(r); e <= std::get<1>(r); ++e) {
                        node_index node = graph.validate_edge(e);
                        if (node)
                            append_suffix_seed(j, canon->reverse_complement(node), seed_length);
                    }
                };
                Range start { boss.pred_last(first - 1) + 1, last, seed_length };
                if (std::get<2>(start) == boss.k_) {
                    call_nodes_in_range(start);
                    continue;
                }
                std::vector<Range> range_stack { start };
                while (range_stack.size()) {
                    Range cur = range_stack.back();
                    range_stack.pop_back();
                    ++std::get<2>(cur);
                    for (TAlphabet c = 1; c < boss.alph_size; ++c) {
                        Range next = cur;
                        if (boss.tighten_range(&std::get<0>(next), &std::get<1>(next), c)) {
                            if (std::get<2>(next) == boss.k_)
                                call_nodes_in_range(next);
                            else
                                range_stack.push_back(next);
                        }
                    }
                }
            }
        }

        num_matching = 0;
        size_t last_end = 0;
        for (size_t i = 0; i < suffix_seeds.size(); ++i) {
            std::vector<Seed> &pos_seeds = suffix_seeds[i];
            if (pos_seeds.empty())
                continue;
            bool first_no_offset = !pos_seeds[0].offset;
            size_t n_pos_seeds = pos_seeds.size();
            if (first_no_offset) {
                seeds_.emplace_back(std::move(pos_seeds[0]));
            } else if (n_pos_seeds <= config.max_num_seeds_per_locus) {
                for (auto &&s : pos_seeds) seeds_.emplace_back(std::move(s));
            }
            if (first_no_offset || n_pos_seeds <= config.max_num_seeds_per_locus) {
                size_t begin = seeds_.back().clipping;
                size_t end = begin + seeds_.back().query_view.size();
                if (begin < last_end) num_matching += end - begin - (last_end - begin);
                else num_matching += end - begin;
                last_end = end;
            }
        }
        return seeds_;
    }
};

} // namespace

SeederOutput run_seeder(const DBGSuccinct &graph, const DBGAlignerConfig &config,
                        std::string_view query, bool orientation,
                        std::vector<node_index> &&nodes, const CanonicalDBG *canon) {
    SeederBase s { graph, query, orientation, std::move(nodes), config, 0, canon };
    s.num_matching = s.num_exact_matching();
    SeederOutput out;
    out.seeds = s.suffix_seeds();
    out.num_matching = s.num_matching;
    return out;
}

// ---------------------------------------------------------------------------
// Extender (aligner_extender_methods.{hpp,cpp})
// ---------------------------------------------------------------------------
// Stop-test trace of the calling thread (mgo_align_budget_trace): while set, the extender appends
// (table_size_bytes_, table.size(), window.size()) every time it evaluates the node and RAM budgets.
thread_local std::vector<uint64_t> *budget_trace = nullptr;

namespace {

constexpr size_t kPadding = 5;

// std::vector<score_t> with observable capacity/padding, as relied upon by
// update_column's 16-byte block accesses (extender.cpp:389-410, 317-325).
struct PVec {
    std::vector<score_t> buf; // buf.size() == capacity
    size_t sz = 0;
    size_t size() const { return sz; }
    size_t capacity() const { return buf.size(); }
    score_t& operator[](size_t i) { return buf[i]; }
    const score_t& operator[](size_t i) const { return buf[i]; }
    score_t* data() { return buf.data(); }
    const score_t* data() const { return buf.data(); }
    score_t& back() { return buf[sz - 1]; }
    void push_back(score_t v) {
        if (sz == buf.size())
            buf.resize(std::max<size_t>(1, 2 * buf.size()), ninf); // libstdc++ doubling
        buf[sz++] = v;
    }
    void reserve(size_t n) { if (n > buf.size()) buf.resize(n, ninf); }
    void fill_padding() { std::fill(buf.begin() + sz, buf.end(), ninf); }
};

struct DPTColumn {
    PVec S, E, F;
    node_index node;
    size_t parent_i;
    char c;
    ssize_t offset;
    ssize_t max_pos;
    ssize_t trim;
    size_t xdrop_cutoff_i;
    score_t score;

    static DPTColumn create(size_t size, node_index node, size_t parent_i, char c, ssize_t offset,
                            ssize_t max_pos, ssize_t trim, size_t xdrop_cutoff_i, score_t score) {
        DPTColumn col;
        col.S.buf.assign(size + kPadding, ninf); col.S.sz = size;
        col.E.buf.assign(size + kPadding, ninf); col.E.sz = size;
        col.F.buf.assign(size + kPadding, ninf); col.F.sz = size;
        col.node = node; col.parent_i = parent_i; col.c = c; col.offset = offset;
        col.max_pos = max_pos; col.trim = trim; col.xdrop_cutoff_i = xdrop_cutoff_i; col.score = score;
        return col;
    }
};
constexpr size_t kSizeofDPTColumn = 136; // sizeof(DefaultColumnExtender::DPTColumn) on LP64/libstdc++

// simde_mm_add_epi32 lane: adds modulo 2^32 (the scalar statements of extender.cpp stay plain int adds)
inline score_t add_epi32(score_t a, score_t b) { return (score_t)((uint32_t)a + (uint32_t)b); }

// extender.cpp:209-290, lane-for-lane
void update_column(size_t prev_end, const score_t *S_prev_v, const score_t *F_prev_v,
                   PVec &S_v, PVec &E_v, PVec &F_v, const score_t *profile_scores,
                   score_t xdrop_cutoff, const DBGAlignerConfig &config_, score_t init_score,
                   size_t offset) {
    constexpr size_t width = kPadding - 1;
    const score_t gap_open = config_.gap_opening_penalty;
    const score_t gap_extend = config_.gap_extension_penalty;
    for (size_t j = 0; j < prev_end; j += width) {
        score_t match[4], del_score[4];
        for (size_t l = 0; l < 4; ++l) {
            if (j) {
                match[l] = add_epi32(add_epi32(S_prev_v[j + l - 1], profile_scores[j + l]), init_score);
            } else if (l) {
                match[l] = add_epi32(add_epi32(S_prev_v[l - 1], profile_scores[l]), init_score);
            } else {
                match[l] = ninf;
            }
            del_score[l] = offset > 1
                ? add_epi32(std::max(add_epi32(S_prev_v[j + l], gap_open), add_epi32(F_prev_v[j + l], gap_extend)), init_score)
                : ninf;
            F_v[j + l] = del_score[l];
            match[l] = std::max(match[l], del_score[l]);
            E_v[j + l + 1] = add_epi32(match[l], gap_open);
        }
        E_v[j + 1] = std::max(E_v[j] + gap_extend, E_v[j + 1]);
        E_v[j + 2] = std::max(E_v[j + 1] + gap_extend, E_v[j + 2]);
        E_v[j + 3] = std::max(E_v[j + 2] + gap_extend, E_v[j + 3]);
        E_v[j + 4] = std::max(E_v[j + 3] + gap_extend, E_v[j + 4]);
        for (size_t l = 0; l < 4; ++l) {
            score_t m = std::max(match[l], E_v[j + l]);
            S_v[j + l] = m > xdrop_cutoff - 1 ? m : ninf;
        }
    }
    if (S_v.size() > std::max(size_t{1}, prev_end)) {
        size_t j = S_v.size() - 1;
        score_t match = std::max(S_prev_v[j - 1] + init_score + profile_scores[j], E_v[j]);
        if (match >= xdrop_cutoff)
            S_v[j] = match;
    }
}

// extender.cpp:293-328
void extend_ins_end(PVec &S, PVec &E, PVec &F, size_t max_size, score_t xdrop_cutoff,
                    const DBGAlignerConfig &config_) {
    if (S.size() < max_size) {
        score_t ins_score = std::max(S.back() + config_.gap_opening_penalty,
                                     E.back() + config_.gap_extension_penalty);
        if (ins_score >= xdrop_cutoff) {
            S.push_back(ins_score);
            E.push_back(ins_score);
            F.push_back(ninf);
            while (E.back() + config_.gap_extension_penalty >= xdrop_cutoff && E.size() < max_size) {
                E.push_back(E.back() + config_.gap_extension_penalty);
                S.push_back(E.back());
                F.push_back(ninf);
            }
            S.reserve(S.size() + kPadding);
            E.reserve(E.size() + kPadding);
            F.reserve(F.size() + kPadding);
            S.fill_padding(); E.fill_padding(); F.fill_padding();
        }
    }
}

class Extender {
  public:
    Extender(const DBGSuccinct &graph, const DBGAlignerConfig &config, std::string_view query)
          : graph_{ &graph, false }, config_(config), query_size_(query.size()), query_(query) {
        const Alphabet &al = *config.alphabet;
        // extender.cpp:22-60
        partial_sums_.assign(query_.size(), 0);
        for (size_t i = 0; i < query_.size(); ++i)
            partial_sums_[i] = config_.score_matrix[(int)query_[i]][(int)query_[i]];
        for (size_t i = query_.size(); i-- > 1; )
            partial_sums_[i - 1] += partial_sums_[i];
        partial_sums_.push_back(0);
        profile_score_.resize(al.sigma + 1);
        profile_op_.resize(al.sigma + 1);
        for (int i = 0; i <= al.sigma; ++i) {
            profile_score_[i].assign(query_.size() + kPadding, 0);
            profile_op_[i].assign(query_.size() + kPadding, Cigar::CLIPPED);
            char c = i != al.sigma ? al.decode(i) : '\0';
            for (size_t j = 0; j < query_.size(); ++j) {
                profile_score_[i][j + 1] = config_.score_matrix[(int)c][(int)query_[j]];
                profile_op_[i][j + 1] = char_to_op(al, c, query_[j]);
            }
        }
    }

    void set_graph(const GraphView &g) { graph_ = g; }
    size_t num_extensions() const { return num_extensions_; }
    size_t num_explored_nodes() const { return explored_nodes_previous_ + conv_checker_.size(); }
    uint64_t dp_cells = 0, dp_columns = 0;

    std::vector<Alignment> get_extensions(const Alignment &seed, score_t min_path_score,
                                          bool force_fixed_seed) {
        // set_seed (:90-98)
        seed_ = &seed;
        explored_nodes_previous_ += conv_checker_.size();
        conv_checker_.clear();
        return extend(min_path_score, force_fixed_seed);
    }

    // :66-88
    bool check_seed(const Alignment &seed) const {
        if (seed.empty())
            return false;
        node_index node = seed.get_nodes().back();
        if (graph_.rc)
            node += graph_.max_index();
        auto it = conv_checker_.find(node);
        if (it == conv_checker_.end())
            return true;
        size_t pos = seed.get_query_view().size() + seed.get_clipping() - 1;
        const auto &[start, vec] = it->second;
        return pos < start || pos - start >= vec.size() || vec[pos - start] < seed.get_score();
    }

    // :158-207
    bool filter_nodes(node_index node, size_t query_start, size_t query_end) {
        constexpr score_t mscore = -ninf;
        size_t size = query_end - query_start;
        auto it = conv_checker_.find(node);
        if (it == conv_checker_.end()) {
            conv_checker_.emplace(node, ScoreVec(query_start, std::vector<score_t>(size, mscore)));
            return true;
        }
        auto &[start, vec] = it->second;
        if (query_start + size <= start) {
            vec.insert(vec.begin(), start - query_start, ninf);
            std::fill(vec.begin(), vec.begin() + size, mscore);
            start = query_start;
            return true;
        }
        if (query_start >= start + vec.size()) {
            vec.insert(vec.end(), query_start - start - vec.size(), ninf);
            vec.insert(vec.end(), size, mscore);
            return true;
        }
        if (query_start < start) {
            vec.insert(vec.begin(), start - query_start, ninf);
            start = query_start;
        }
        if (query_start + size > start + vec.size())
            vec.resize(query_start + size - start, ninf);
        bool converged = true;
        score_t *v = vec.data() + query_start - start;
        for (size_t j = 0; j < size; ++j) {
            if (mscore > v[j]) { converged = false; v[j] = mscore; }
        }
        return !converged;
    }

  private:
    typedef std::pair<size_t, std::vector<score_t>> ScoreVec;
    GraphView graph_;
    const DBGAlignerConfig &config_;
    const Alignment *seed_ = nullptr;
    size_t query_size_;
    std::unordered_map<node_index, ScoreVec> conv_checker_;
    size_t explored_nodes_previous_ = 0;

    std::string_view query_;
    std::vector<DPTColumn> table;
    size_t table_capacity_ = 0;      // std::vector<DPTColumn>::capacity() survives clear()
    size_t table_size_bytes_ = 0;
    std::unordered_set<size_t> prev_starts;
    score_t xdrop_cutoff_ = 0;        // global_xdrop: one shared cutoff (xdrop_cutoffs_[0])
    std::vector<std::pair<size_t, score_t>> xdrop_cutoffs_;
    size_t num_extensions_ = 0;
    std::vector<score_t> partial_sums_;
    std::vector<std::vector<score_t>> profile_score_;
    std::vector<std::vector<Cigar::Operator>> profile_op_;
    std::vector<score_t> scores_reached_;
    score_t min_cell_score_ = 0;

    void table_emplace_back(DPTColumn &&col) {
        if (table.size() == table_capacity_)
            table_capacity_ = std::max<size_t>(1, 2 * table_capacity_);
        table.emplace_back(std::move(col));
    }

    // :100-156
    score_t update_seed_filter(node_index node, size_t query_start,
                               const score_t *s_begin, const score_t *s_end) {
        if (node == npos)
            return *std::max_element(s_begin, s_end);
        if (graph_.rc)
            node += graph_.max_index();
        size_t size = s_end - s_begin;
        auto it = conv_checker_.find(node);
        if (it == conv_checker_.end()) {
            conv_checker_.emplace(node, ScoreVec(query_start, { s_begin, s_end }));
            return *std::max_element(s_begin, s_end);
        }
        auto &[start, vec] = it->second;
        if (query_start + size <= start) {
            vec.insert(vec.begin(), start - query_start, ninf);
            std::copy(s_begin, s_end, vec.begin());
            start = query_start;
            return *std::max_element(s_begin, s_end);
        }
        if (query_start >= start + vec.size()) {
            vec.insert(vec.end(), query_start - start - vec.size(), ninf);
            vec.insert(vec.end(), s_begin, s_end);
            return *std::max_element(s_begin, s_end);
        }
        if (query_start < start) {
            vec.insert(vec.begin(), start - query_start, ninf);
            start = query_start;
        }
        if (query_start + size > start + vec.size())
            vec.resize(query_start + size - start, ninf);
        score_t max_changed_value = ninf;
        score_t *v = vec.data() + query_start - start;
        for (size_t j = 0; j < size; ++j) {
            if (s_begin[j] > v[j] * config_.rel_score_cutoff) {
                v[j] = std::max(v[j], s_begin[j]);
                max_changed_value = std::max(max_changed_value, v[j]);
            }
        }
        return max_changed_value;
    }

    // :330-387
    template <class CB>
    void call_outgoing(node_index node, CB &&callback, size_t table_i, bool force_fixed_seed) {
        size_t next_offset = table[table_i].offset + 1;
        size_t seed_pos = next_offset - seed_->get_offset();
        bool in_seed = seed_pos < seed_->get_sequence().size();
        if (in_seed && next_offset < graph_.get_k()) {
            callback(seed_->get_nodes().front(), seed_->get_sequence()[seed_pos], 0);
        } else if (in_seed && force_fixed_seed) {
            size_t node_i = next_offset - graph_.get_k() + 1;
            node_index next_node = seed_->get_nodes()[node_i];
            char next_c = seed_->get_sequence()[seed_pos];
            callback(next_node, next_c, next_node
                ? 0
                : (!node ? config_.gap_extension_penalty : config_.gap_opening_penalty));
        } else {
            graph_.call_outgoing_kmers(node, [&](node_index next, char c) {
                if (c != '$')
                    callback(next, c, 0);
            });
        }
    }

    // :412-772 (target_length = 0, target_node = npos, trim_offset_after_extend = true,
    //           trim_query_suffix = 0, added_xdrop = 0: the only values on this path)
    std::vector<Alignment> extend(score_t min_path_score, bool force_fixed_seed) {
        ++num_extensions_;
        min_path_score = std::max(0, min_path_score);
        table.clear();
        prev_starts.clear();

        score_t xdrop = config_.xdrop;
        xdrop_cutoffs_.assign(1, std::make_pair(0u, std::max(-xdrop, ninf + 1)));
        if (!config_.global_xdrop)
            scores_reached_.assign(1, 0);

        size_t start = seed_->get_clipping();
        std::string_view window(seed_->get_query_view().data(),
                                query_.data() + query_.size() - seed_->get_query_view().data());
        score_t partial_sum_offset = partial_sums_.at(start + window.size());
        ssize_t seed_offset = static_cast<ssize_t>(seed_->get_offset()) - 1;

        table_emplace_back(DPTColumn::create(1, seed_->get_nodes().front(), static_cast<size_t>(-1),
                                             '\0', seed_offset, 0, 0, 0u, 0));
        {
            auto &col = table[0];
            col.S[0] = config_.left_end_bonus && !seed_->get_clipping() ? config_.left_end_bonus : 0;
            extend_ins_end(col.S, col.E, col.F, window.size() + 1 - col.trim,
                           xdrop_cutoffs_[col.xdrop_cutoff_i].second, config_);
            table_size_bytes_ = kSizeofDPTColumn * table_capacity_
                + (col.S.capacity() + col.E.capacity() + col.F.capacity()) * sizeof(score_t);
            dp_cells += col.S.size(); ++dp_columns;
        }

        using TableIt = std::tuple<score_t, ssize_t, size_t, score_t>;
        min_cell_score_ = 0;
        score_t best_score = 0;
        std::priority_queue<TableIt> queue;
        queue.emplace(0, 0, 0, 0);
        std::vector<size_t> tips;

        while (queue.size()) {
            std::vector<TableIt> next_nodes{ queue.top() };
            queue.pop();
            while (queue.size() && std::get<0>(queue.top()) == std::get<0>(next_nodes.back())) {
                next_nodes.push_back(queue.top());
                queue.pop();
            }

            while (next_nodes.size()) {
                size_t i = std::get<2>(next_nodes.back());
                next_nodes.pop_back();

                std::vector<std::tuple<node_index, char, score_t>> outgoing;
                size_t next_offset = table[i].offset + 1;
                ssize_t begin = 0;
                ssize_t prev_end = window.size() + 1;
                size_t prev_xdrop_cutoff_i = table[i].xdrop_cutoff_i;
                score_t prev_xdrop_cutoff = xdrop_cutoffs_[prev_xdrop_cutoff_i].second;
                bool in_seed = next_offset - seed_->get_offset() < seed_->get_sequence().size();

                {
                    const DPTColumn &col = table[i];
                    const PVec &S = col.S;
                    double node_counter = config_.global_xdrop ? table.size()
                                                               : next_offset - seed_offset;
                    if (S[col.max_pos - col.trim] < best_score) {
                        if (budget_trace) {
                            budget_trace->push_back(table_size_bytes_);
                            budget_trace->push_back(table.size());
                            budget_trace->push_back(window.size());
                        }
                        if (node_counter / window.size() >= config_.max_nodes_per_seq_char) {
                            if (config_.global_xdrop) {
                                queue = std::priority_queue<TableIt>();
                                next_nodes.clear();
                            }
                            continue;
                        }
                        if (static_cast<double>(table_size_bytes_) / 1'000'000
                                > config_.max_ram_per_alignment) {
                            queue = std::priority_queue<TableIt>();
                            next_nodes.clear();
                            continue;
                        }
                    }
                    // band within the xdrop cutoff (:549-560)
                    {
                        size_t b = 0;
                        while (b < S.size() && S[b] < prev_xdrop_cutoff) ++b;
                        size_t e = S.size();
                        while (e > 0 && S[e - 1] < prev_xdrop_cutoff) --e;
                        begin = b + col.trim;
                        prev_end = e + col.trim;
                    }
                    if (prev_end <= begin)
                        continue;
                    call_outgoing(col.node, [&](node_index next, char c, score_t s) {
                        c = toupper(c);
                        outgoing.emplace_back(next, c, s);
                    }, i, force_fixed_seed);
                    if (outgoing.empty()) {
                        tips.push_back(i);
                        continue;
                    }
                }

                size_t end = std::min(static_cast<size_t>(prev_end), window.size()) + 1;

                for (const auto &[next, c, score] : outgoing) {
                    bool forked = outgoing.size() > 1;
                    bool forked_xdrop = !config_.global_xdrop && forked;
                    size_t xdrop_cutoffs_sizediff = xdrop_cutoffs_.capacity();
                    if (forked_xdrop) {
                        xdrop_cutoffs_.emplace_back(table.size(), prev_xdrop_cutoff);
                        xdrop_cutoffs_sizediff = xdrop_cutoffs_.capacity() - xdrop_cutoffs_sizediff;
                    } else {
                        xdrop_cutoffs_sizediff = 0;
                    }

                    size_t table_sizediff = table_capacity_;
                    table_emplace_back(DPTColumn::create(end - begin, next, i, c,
                        static_cast<ssize_t>(next_offset), begin, begin,
                        forked_xdrop ? xdrop_cutoffs_.size() - 1 : prev_xdrop_cutoff_i, score));

                    const DPTColumn &prev = table[i];
                    DPTColumn &cur = table.back();
                    PVec &S = cur.S, &E = cur.E, &F = cur.F;
                    const PVec &S_prev = prev.S, &F_prev = prev.F;
                    const ssize_t trim = cur.trim, trim_prev = prev.trim;
                    const ssize_t offset = cur.offset;
                    ssize_t &max_pos = cur.max_pos;
                    score_t &xdrop_cutoff = xdrop_cutoffs_[cur.xdrop_cutoff_i].second;

                    update_column(prev_end - trim,
                                  S_prev.data() + trim - trim_prev,
                                  F_prev.data() + trim - trim_prev,
                                  S, E, F,
                                  profile_score_[config_.alphabet->encode(c)].data() + start + trim,
                                  xdrop_cutoff, config_, score, offset);
                    extend_ins_end(S, E, F, window.size() + 1 - trim, xdrop_cutoff, config_);
                    dp_cells += S.size(); ++dp_columns;

                    ssize_t cur_offset = begin;
                    ssize_t diag_i = offset - seed_offset;
                    bool has_extension = in_seed;
                    const score_t *partial_sums = &partial_sums_[start + trim];
                    score_t extension_cutoff
                        = best_score * config_.rel_score_cutoff + partial_sum_offset;
                    score_t max_diff = ninf;

                    size_t scores_reached_sizediff = 0;
                    bool scores_reached_cutoff = true;
                    if (!config_.global_xdrop) {
                        scores_reached_sizediff = scores_reached_.capacity();
                        scores_reached_.resize(S.size() + trim + 1, ninf);
                        scores_reached_sizediff = scores_reached_.capacity() - scores_reached_sizediff;
                    }

                    for (size_t j = 0; j < S.size(); ++j, ++cur_offset) {
                        if (S[j] != ninf)
                            min_cell_score_ = std::min(min_cell_score_, S[j]);
                        if (std::make_pair(S[j], std::abs(max_pos - diag_i))
                                > std::make_pair(S[max_pos - begin], std::abs(cur_offset - diag_i))) {
                            max_pos = j + begin;
                        }
                        if (!config_.global_xdrop) {
                            scores_reached_[trim + j] = std::max(scores_reached_[trim + j], S[j]);
                            scores_reached_cutoff
                                = (S[j] >= scores_reached_[trim + j] * config_.rel_score_cutoff);
                        }
                        if (!has_extension && scores_reached_cutoff
                                && S[j] + partial_sums[j] >= extension_cutoff) {
                            has_extension = true;
                        }
                        if (static_cast<size_t>(trim - trim_prev) < S_prev.size()
                                && S[j] - S_prev[j + trim - trim_prev] > max_diff) {
                            max_diff = S[j] - S_prev[j + trim - trim_prev];
                        }
                    }

                    score_t max_val = S[max_pos - trim];

                    // target_length == 0: static_cast<size_t>(offset - seed_offset) < 1 is
                    // never true for a child column; `else if (target_length)` is dead.
                    if (static_cast<size_t>(offset - seed_offset) < 1)
                        has_extension = true;

                    if (!in_seed && max_val < xdrop_cutoff) {
                        table.pop_back();
                        if (forked_xdrop) xdrop_cutoffs_.pop_back();
                        continue;
                    }
                    if (!in_seed && !has_extension) {
                        table.pop_back();
                        if (forked_xdrop) xdrop_cutoffs_.pop_back();
                        continue;
                    }

                    table_sizediff = table_capacity_ - table_sizediff;
                    table_size_bytes_ += kSizeofDPTColumn * table_sizediff
                        + (S.capacity() + E.capacity() + F.capacity()) * sizeof(score_t)
                        + sizeof(score_t) * scores_reached_sizediff
                        + sizeof(std::pair<size_t, score_t>) * xdrop_cutoffs_sizediff;

                    if (max_val - xdrop_cutoff > xdrop)
                        xdrop_cutoff = max_val - xdrop;

                    best_score = std::max(best_score, max_val);

                    size_t vec_offset = start + begin - static_cast<bool>(begin);
                    score_t *s_begin = S.data() + !begin;
                    score_t *s_end = S.data() + S.size();

                    score_t converged_score = update_seed_filter(next, vec_offset, s_begin, s_end);
                    if (converged_score != ninf) {
                        TableIt next_score { converged_score, -std::abs(max_pos - diag_i),
                                             table.size() - 1, max_val };
                        if (next_nodes.size() && converged_score == std::get<0>(next_nodes[0])) {
                            next_nodes.emplace_back(std::move(next_score));
                        } else {
                            queue.emplace(std::move(next_score));
                        }
                    }
                }
            }
        }

        if (config_.no_backtrack)
            return { *seed_ };

        std::sort(tips.begin(), tips.end());
        auto extensions = backtrack(min_path_score, window, config_.right_end_bonus, tips);
        for (auto &extension : extensions)
            extension.trim_offset();
        return extensions;
    }

    // :774-798
    Alignment construct_alignment(Cigar cigar, size_t clipping, std::string_view window,
                                  std::vector<node_index> final_path, std::string match,
                                  score_t score, size_t offset, score_t extra_score) const {
        cigar.append(Cigar::CLIPPED, clipping);
        std::reverse(cigar.data().begin(), cigar.data().end());
        std::reverse(final_path.begin(), final_path.end());
        std::reverse(match.begin(), match.end());
        Alignment extension(window, std::move(final_path), std::move(match), score,
                            std::move(cigar), 0, seed_->get_orientation(), offset);
        extension.extend_query_begin(query_.data());
        extension.extend_query_end(query_.data() + query_.size());
        extension.extra_score = extra_score;
        return extension;
    }

    // :800-1034 (target_node == npos)
    std::vector<Alignment> backtrack(score_t min_path_score, std::string_view window,
                                     score_t right_end_bonus, const std::vector<size_t> &tips) {
        std::vector<Alignment> extensions;
        const Alphabet &al = *config_.alphabet;
        size_t seed_clipping = seed_->get_clipping();
        ssize_t seed_offset = static_cast<ssize_t>(seed_->get_offset() - 1);
        ssize_t k_minus_1 = graph_.get_k() - 1;
        ssize_t last_pos = window.size();
        ssize_t seed_dist = std::max(graph_.get_k(), seed_->get_sequence().size()) - 1;
        score_t min_start_score = min_path_score;
        size_t min_trace_length = graph_.get_k() - seed_->get_offset();

        std::vector<std::tuple<score_t, ssize_t, ssize_t, ssize_t>> indices;
        indices.reserve(table.size());
        auto it = tips.begin();
        for (size_t i = 1; i < table.size(); ++i) {
            while (it != tips.end() && i > *it)
                ++it;

            auto check_and_add_pos = [&](ssize_t start_pos, bool is_tip) {
                const DPTColumn &col = table[i];
                const DPTColumn &par = table[col.parent_i];
                if (start_pos < par.trim + 1)
                    return;
                size_t pos = start_pos - col.trim;
                size_t pos_p = start_pos - par.trim - 1;
                if (col.S[pos] == ninf || par.S[pos_p] == ninf)
                    return;
                score_t end_bonus = start_pos == last_pos ? right_end_bonus : 0;
                TAlphabet s = al.encode(col.c);
                if (col.S[pos] + end_bonus >= min_start_score) {
                    bool is_match = col.S[pos] == par.S[pos_p] + col.score
                                        + profile_score_[s][seed_clipping + start_pos]
                        && profile_op_[s][seed_clipping + start_pos] == Cigar::MATCH;
                    if (is_match || start_pos == last_pos || is_tip) {
                        indices.emplace_back(col.S[pos] + end_bonus,
                                             -std::abs(start_pos - col.offset + seed_offset),
                                             -static_cast<ssize_t>(i), start_pos);
                    }
                }
            };

            if (table[i].offset < seed_dist)
                continue;

            bool is_tip = (it != tips.end() && i == *it);
            check_and_add_pos(table[i].max_pos, is_tip);

            if (table[i].S.size() + table[i].trim == window.size() + 1
                    && table[i].max_pos != last_pos) {
                check_and_add_pos(last_pos, is_tip);
            }
        }

        // heap order == descending order of the (unique) tuples
        std::sort(indices.begin(), indices.end());

        score_t best_score = std::numeric_limits<score_t>::min();

        for (auto rit = indices.rbegin(); rit != indices.rend(); ++rit) {
            const auto &[start_score, neg_off_diag, neg_j_start, start_pos] = *rit;

            if (extensions.size() >= config_.num_alternative_paths)
                break;

            size_t j = -neg_j_start;
            if (!prev_starts.emplace(j).second)
                continue;

            std::vector<node_index> path;
            std::vector<size_t> trace;
            Cigar ops;
            std::string seq;
            score_t score = start_score;

            if (score - min_cell_score_ < best_score)
                break;

            size_t dummy_counter = 0;
            ssize_t pos = start_pos;
            ssize_t end_pos = pos;
            size_t align_offset = seed_->get_offset();
            score_t extra_score = 0;

            auto append_node = [&](node_index node, char c, ssize_t offset, Cigar::Operator op) {
                seq += c;
                ops.append(op);
                if (offset >= k_minus_1) {
                    path.emplace_back(node);
                    if (!node) {
                        ++dummy_counter;
                    } else if (dummy_counter) {
                        ops.append(Cigar::NODE_INSERTION, dummy_counter);
                        extra_score -= config_.gap_opening_penalty
                            + (dummy_counter - 1) * config_.gap_extension_penalty;
                        dummy_counter = 0;
                    }
                }
            };

            while (j) {
                const DPTColumn &col = table[j];
                const DPTColumn &par = table[col.parent_i];
                const PVec &S = col.S, &E = col.E, &F = col.F;
                const PVec &S_p = par.S;
                const ssize_t trim = col.trim, trim_p = par.trim;

                align_offset = std::min(col.offset, k_minus_1);

                if (pos == col.max_pos)
                    prev_starts.emplace(j);

                TAlphabet s = al.encode(col.c);

                if (S[pos - trim] == ninf) {
                    j = 0;
                } else if (pos && S[pos - trim] == E[pos - trim]
                        && (ops.empty() || ops.data().back().first != Cigar::DELETION)) {
                    Cigar::Operator last_op = Cigar::INSERTION;
                    while (last_op == Cigar::INSERTION) {
                        ops.append(last_op);
                        last_op = E[pos - trim] == E[pos - trim - 1] + config_.gap_extension_penalty
                            ? Cigar::INSERTION
                            : Cigar::MATCH;
                        --pos;
                    }
                } else if (pos && pos >= trim_p + 1
                        && S[pos - trim] == S_p[pos - trim_p - 1] + col.score
                            + profile_score_[s][seed_clipping + pos]) {
                    trace.emplace_back(j);
                    extra_score += col.score;
                    append_node(col.node, col.c, col.offset, profile_op_[s][seed_clipping + pos]);
                    --pos;
                    j = col.parent_i;
                } else if (S[pos - trim] == F[pos - trim]
                        && (ops.empty() || ops.data().back().first != Cigar::INSERTION)) {
                    Cigar::Operator last_op = Cigar::DELETION;
                    while (last_op == Cigar::DELETION && j) {
                        const DPTColumn &c2 = table[j];
                        const DPTColumn &p2 = table[c2.parent_i];
                        align_offset = std::min(c2.offset, k_minus_1);
                        last_op = c2.F[pos - c2.trim]
                                == p2.F[pos - p2.trim] + c2.score + config_.gap_extension_penalty
                            ? Cigar::DELETION
                            : Cigar::MATCH;
                        trace.emplace_back(j);
                        extra_score += c2.score;
                        append_node(c2.node, c2.c, c2.offset, Cigar::DELETION);
                        j = c2.parent_i;
                    }
                } else {
                    break;
                }
            }

            if (trace.size() >= min_trace_length && path.size() && path.back()) {
                score_t cur_cell_score = table[j].S[pos - table[j].trim];
                best_score = std::max(best_score, score - cur_cell_score);
                if (score - min_cell_score_ < best_score)
                    break;

                if (score >= min_start_score
                        && (!pos || cur_cell_score == 0)
                        && (pos || cur_cell_score == table[0].S[0])
                        && (config_.allow_left_trim || !j)) {
                    extensions.emplace_back(construct_alignment(
                        ops, pos, window.substr(pos, end_pos - pos), path, seq, score,
                        align_offset, extra_score));
                }
            }
        }

        if (extensions.empty() && seed_->get_score() >= min_path_score)
            extensions.emplace_back(*seed_);

        return extensions;
    }
};

// aligner_aggregator.hpp (unlabeled queue only)
class Aggregator {
  public:
    explicit Aggregator(const DBGAlignerConfig &config) : config_(config) {}

    bool add_alignment(Alignment &&alignment) {
        if (q_.empty()) {
            q_.emplace_back(std::move(alignment));
            return true;
        }
        if (alignment.get_score() < get_global_cutoff())
            return false;
        for (const auto &aln : q_)
            if (alignment == aln)
                return false;
        if (q_.size() < config_.num_alternative_paths) {
            q_.emplace_back(std::move(alignment));
            return true;
        }
        auto min_it = std::min_element(q_.begin(), q_.end(), cmp_);
        if (cmp_(alignment, *min_it))
            return false;
        *min_it = std::move(alignment);
        return true;
    }

    score_t get_global_cutoff() const {
        if (q_.empty())
            return config_.ninf;
        score_t cur_max = std::max_element(q_.begin(), q_.end(), cmp_)->get_score();
        return cur_max > 0 ? cur_max * config_.rel_score_cutoff : cur_max;
    }

    std::vector<Alignment> get_alignments() {
        std::vector<Alignment> out = std::move(q_);
        q_.clear();
        // descending; ties (std::sort leaves them unspecified in the reference) keep insertion order
        std::stable_sort(out.begin(), out.end(),
                         [&](const Alignment &a, const Alignment &b) { return cmp_(b, a); });
        return out;
    }

  private:
    const DBGAlignerConfig &config_;
    std::vector<Alignment> q_;
    LocalAlignmentLess cmp_;
};

std::vector<Alignment> seeds_to_alignments(const std::vector<Seed> &seeds,
                                           const DBGAlignerConfig &config) {
    // ISeeder::get_alignments (seeder.hpp:20-29)
    std::vector<Alignment> alignments;
    alignments.reserve(seeds.size());
    for (const Seed &seed : seeds) {
        alignments.emplace_back(seed, config);
        alignments.back().trim_offset();
    }
    return alignments;
}

// dbg_aligner.cpp:360-384
template <class Callback, class GetMinPathScore>
void align_core(std::vector<Alignment> seeds, Extender &extender, Callback &&callback,
                GetMinPathScore &&get_min_path_score, bool force_fixed_seed) {
    for (size_t i = 0; i < seeds.size(); ++i) {
        if (seeds[i].empty())
            continue;
        score_t min_path_score = get_min_path_score(seeds[i]);
        for (auto &&extension : extender.get_extensions(seeds[i], min_path_score, force_fixed_seed))
            callback(std::move(extension));
        for (size_t j = i + 1; j < seeds.size(); ++j) {
            if (seeds[j].size() && !extender.check_seed(seeds[j]))
                seeds[j] = Alignment(); // filter_seed with no labels (:105-107)
        }
    }
}

} // namespace

// ---------------------------------------------------------------------------
// DBGAligner
// ---------------------------------------------------------------------------
DBGAligner::DBGAligner(const DBGSuccinct &graph, const DBGAlignerConfig &config)
      : graph_(graph), config_(config) {
    if (graph_.mode == 2)
        canonical_ = std::make_unique<CanonicalDBG>(graph_);
    if (!config_.min_seed_length)
        config_.min_seed_length = graph_.get_k();
    if (!config_.max_seed_length)
        config_.max_seed_length = graph_.get_k();
    std::tie(config_.min_seed_length, config_.max_seed_length)
        = std::make_pair(std::min(config_.min_seed_length, config_.max_seed_length),
                         std::max(config_.min_seed_length, config_.max_seed_length));
    if (!config_.check_config_scores())
        throw std::runtime_error("Error: sum of min_cell_score and lowest penalty too low.");
}

AlignmentResults DBGAligner::align(std::string_view query) const {
    AlignmentResults result;
    align_batch({ { std::string{}, std::string(query) } },
                [&](const std::string&, AlignmentResults &&r) { result = std::move(r); });
    return result;
}

void DBGAligner::align_batch(const std::vector<std::pair<std::string, std::string>> &batch,
                             const std::function<void(const std::string&, AlignmentResults&&)> &callback,
                             AlignStats *stats) const {
    // dbg_aligner.cpp:224-226, 646-656
    const CanonicalDBG *canon = canonical_.get();         // CanonicalDBG::get_mode() == CANONICAL (canonical_dbg.hpp:83)
    const bool canonical = graph_.mode == 1 || canon;
    const bool both = (canonical || config_.forward_and_reverse_complement) && config_.alphabet->sigma == 5;
    const bool use_rcdbg = !canonical && config_.forward_and_reverse_complement;
    GraphView fwd_graph { &graph_, false, canon };
    GraphView rc_graph { &graph_, use_rcdbg, canon };
    auto map_nodes = [&](std::string_view seq) {
        return canon ? canon->map_to_nodes_sequentially(seq) : graph_.map_to_nodes_sequentially(seq);
    };
    auto is_reversible = [&](const Alignment &a) { return canonical && a.get_orientation() && !a.get_offset(); };

    for (const auto &[header, query] : batch) {
        AlignmentResults paths(query);
        std::string_view this_query = paths.get_query(false);
        std::string_view reverse = paths.get_query(true);

        // build_seeders (:193-248)
        std::vector<node_index> nodes;
        if (config_.max_seed_length >= graph_.get_k()) {
            nodes = map_nodes(query);
        } else if (this_query.size() >= graph_.get_k()) {
            nodes.resize(this_query.size() - graph_.get_k() + 1);
        }
        std::vector<node_index> nodes_rc;
        if (both) {
            nodes_rc = nodes;
            if (config_.max_seed_length >= graph_.get_k()) {
                std::string dummy(query);
                reverse_complement_inplace(dummy);
                if (canon) canon->reverse_complement(dummy, nodes_rc);   // reverse_complement_seq_path,
                else nodes_rc = map_nodes(dummy);                        // sequence_graph.cpp:563-573
            }
        }
        SeederOutput seeder = run_seeder(graph_, config_, this_query, false, std::move(nodes), canon);
        if (this_query.size() * config_.min_exact_match > seeder.num_matching)
            seeder = SeederOutput();
        SeederOutput seeder_rc;
        if (both) {
            seeder_rc = run_seeder(graph_, config_, reverse, true, std::move(nodes_rc), canon);
            if (reverse.size() * config_.min_exact_match > seeder_rc.num_matching)
                seeder_rc = SeederOutput();
        }

        Aggregator aggregator(config_);
        auto add_alignment = [&](Alignment &&a) { aggregator.add_alignment(std::move(a)); };
        auto get_min_path_score = [&](const Alignment&) {
            return std::max(config_.min_path_score, aggregator.get_global_cutoff());
        };

        Extender extender(graph_, config_, this_query);
        size_t num_seeds = 0;

        if (both) {
            Extender extender_rc(graph_, config_, reverse);

            // align_both_directions (:531-758), non-chaining branch
            auto aln_both = [&](std::string_view q, std::string_view q_rc,
                                std::vector<Alignment> &&seeds,
                                Extender &fwd_extender, Extender &bwd_extender) {
                fwd_extender.set_graph(fwd_graph);
                bwd_extender.set_graph(rc_graph);
                num_seeds += seeds.size();
                if (seeds.empty())
                    return;
                for (size_t i = 0; i < seeds.size(); ++i) {
                    if (seeds[i].empty())
                        continue;
                    score_t min_path_score = config_.min_cell_score;
                    auto extensions = fwd_extender.get_extensions(seeds[i], min_path_score, false);
                    std::vector<Alignment> rc_of_alignments;
                    for (Alignment &path : extensions) {
                        if (path.get_score() >= get_min_path_score(path)) {
                            if (is_reversible(path)) {                        // :680-684
                                Alignment out_path = path;
                                out_path.reverse_complement(fwd_graph, q_rc);
                                add_alignment(std::move(out_path));
                            } else {
                                add_alignment(Alignment(path));
                            }
                        }
                        if (!path.get_clipping() || path.get_offset())
                            continue;
                        path.reverse_complement(rc_graph, q_rc);
                        if (path.empty())
                            continue;
                        rc_of_alignments.emplace_back(std::move(path));
                    }
                    align_core(std::move(rc_of_alignments), bwd_extender,
                        [&](Alignment &&path) {
                            if (use_rcdbg || is_reversible(path)) {           // :710-722
                                path.reverse_complement(rc_graph, q);
                                if (path.empty())
                                    return;
                                for (node_index node : path.get_nodes()) {
                                    fwd_extender.filter_nodes(node, path.get_clipping(),
                                                              q.size() - path.get_end_clipping());
                                }
                            }
                            add_alignment(std::move(path));
                        },
                        get_min_path_score, true);
                    for (size_t j = i + 1; j < seeds.size(); ++j) {
                        if (seeds[j].size() && !fwd_extender.check_seed(seeds[j]))
                            seeds[j] = Alignment();
                    }
                }
            };

            size_t fwd_num_matches = seeder.num_matching;
            size_t bwd_num_matches = seeder_rc.num_matching;
            auto fwd_seeds = seeds_to_alignments(seeder.seeds, config_);
            auto bwd_seeds = seeds_to_alignments(seeder_rc.seeds, config_);
            if (fwd_num_matches >= bwd_num_matches) {
                aln_both(this_query, reverse, std::move(fwd_seeds), extender, extender_rc);
                if (bwd_num_matches >= fwd_num_matches * config_.rel_score_cutoff)
                    aln_both(reverse, this_query, std::move(bwd_seeds), extender_rc, extender);
            } else {
                aln_both(reverse, this_query, std::move(bwd_seeds), extender_rc, extender);
                if (fwd_num_matches >= bwd_num_matches * config_.rel_score_cutoff)
                    aln_both(this_query, reverse, std::move(fwd_seeds), extender, extender_rc);
            }
            if (stats) {
                stats->num_extensions += extender_rc.num_extensions();
                stats->num_explored_nodes += extender_rc.num_explored_nodes();
                stats->dp_cells += extender_rc.dp_cells;
                stats->dp_columns += extender_rc.dp_columns;
            }
        } else {
            num_seeds += seeder.seeds.size();
            align_core(seeds_to_alignments(seeder.seeds, config_), extender, add_alignment,
                       get_min_path_score, false);
        }
        if (stats) {
            stats->num_seeds += num_seeds;
            stats->num_extensions += extender.num_extensions();
            stats->num_explored_nodes += extender.num_explored_nodes();
            stats->dp_cells += extender.dp_cells;
            stats->dp_columns += extender.dp_columns;
        }

        // chain_alignments is the identity unless post_chain_alignments (chainer.cpp:560-561)
        for (auto &&alignment : aggregator.get_alignments())
            paths.alignments.emplace_back(std::move(alignment));

        callback(header, std::move(paths));
    }
}

std::string format_alignment(const std::string &header, const AlignmentResults &paths,
                             score_t min_path_score) {
    std::string sout = header + "\t" + paths.get_query();
    if (paths.alignments.empty()) {
        sout += "\t*\t*\t" + std::to_string(min_path_score) + "\t*\t*\t*\n";
    } else {
        for (const auto &a : paths.alignments) {
            sout += "\t";
            sout += a.get_orientation() ? "-" : "+";
            sout += "\t" + std::string(a.get_sequence()) + "\t" + std::to_string(a.get_score())
                + "\t" + std::to_string(a.get_cigar().get_num_matches())
                + "\t" + a.get_cigar().to_string() + "\t" + std::to_string(a.get_offset());
        }
        sout += "\n";
    }
    return sout;
}

} // namespace mgo
