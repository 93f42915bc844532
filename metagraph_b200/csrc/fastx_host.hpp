// Host restatement of htslib's kseq_read as seq_io::FastaParser drives it (seq_io/sequence_io.hpp:349-438), over one
// chunk of a file held in memory. It parses every chunk the device parser (fastx_core.cuh) refuses, and it is what the
// device parser is tested against.
//
// Per record: skip bytes up to a '>' or '@'; the name runs to the first isspace byte, the rest of that line is the
// comment; sequence lines follow until a line that starts with '>', '@' or '+' (empty lines add nothing). After '+' the
// rest of that line is skipped and quality lines are read until they hold at least as many bytes as the sequence; no
// quality line, or a length that differs, is kseq_read's -2, which ends FastaParser's iteration: that record and the
// rest of the file are dropped (*ended = 1). Every line read to its end loses one '\r' before that end (the CR rule).
#pragma once
#include <cstring>
#include <string>
#include <vector>
#include "fastx_core.cuh"

namespace mgb {

struct FastxRecords {
    std::vector<char> seqs, names;
    std::vector<uint64_t> offsets{ 0 }, name_offsets{ 0 };
    void add(const std::string &header, const char *seq, size_t len) {
        seqs.insert(seqs.end(), seq, seq + len);
        names.insert(names.end(), header.begin(), header.end());
        offsets.push_back(seqs.size());
        name_offsets.push_back(names.size());
    }
};

// Parses the complete records of buf[0, n). at_eof: nothing follows buf. delim: --header-comment-delim (nullptr: none).
// *consumed: bytes up to the end of the last complete record (or of bytes skipped before a record). *ended: the input
// ended at a malformed record.
inline void fastx_parse_host(const char *buf, uint64_t n, bool at_eof, const char *delim, bool fwd_rev,
                             FastxRecords *out, uint64_t *consumed, int *ended) {
    *consumed = 0; *ended = 0;
    uint64_t p = 0;
    bool have_hdr = false;                 // kseq's last_char: the record's header byte was read by the previous one
    // the end of the line that starts at i ('\n' or n); false: the line runs past the chunk
    auto line_end = [&](uint64_t i, uint64_t *e) {
        const void *q = i < n ? std::memchr(buf + i, '\n', n - i) : nullptr;
        *e = q ? (uint64_t)((const char*)q - buf) : n;
        return q || at_eof;
    };
    auto content_end = [&](uint64_t b, uint64_t e) { return e > b && buf[e - 1] == '\r' ? e - 1 : e; };
    auto next_line = [&](uint64_t e) { return e < n ? e + 1 : n; };
    std::string name, comment, seq, header;
    for (;;) {
        if (!have_hdr) {
            while (p < n && buf[p] != '>' && buf[p] != '@') ++p;
            if (p == n) { *consumed = n; return; }
            ++p;
        }
        *consumed = p - 1;
        // name (KS_SEP_SPACE); a header byte that ends the input has none and kseq_read returns -1
        uint64_t q = p, e;
        while (q < n && !fastx_space((uint8_t)buf[q])) ++q;
        if (q == n && !at_eof) return;
        if (q == p && q == n) { *consumed = n; return; }
        name.assign(buf + p, q - p);
        comment.clear();
        if (q < n && buf[q] == '\n') {
            p = q + 1;
        } else if (q == n) {
            p = n;
        } else {
            if (!line_end(q + 1, &e)) return;
            comment.assign(buf + q + 1, content_end(q + 1, e) - (q + 1));
            p = next_line(e);
        }
        // sequence lines
        seq.clear();
        int c = -1;
        for (;;) {
            if (p == n) { if (!at_eof) return; c = -1; break; }
            c = (uint8_t)buf[p];
            if (c == '>' || c == '@' || c == '+') { ++p; break; }
            if (c == '\n') { ++p; continue; }
            if (!line_end(p, &e)) return;
            seq.append(buf + p, content_end(p, e) - p);
            p = next_line(e);
        }
        if (c == '+') {
            // the rest of the '+' line, then quality lines until there are at least as many bytes as in the sequence
            const void *nl = p < n ? std::memchr(buf + p, '\n', n - p) : nullptr;
            if (!nl) { if (at_eof) *ended = 1; return; }
            p = (uint64_t)((const char*)nl - buf) + 1;
            uint64_t ql = 0;
            for (;;) {
                if (p == n) { if (!at_eof) return; break; }
                if (!line_end(p, &e)) return;
                ql += content_end(p, e) - p;
                p = next_line(e);
                if (ql >= seq.size()) break;
            }
            if (ql != seq.size()) { *ended = 1; return; }
        }
        // the header `metagraph align` prints (cli/align.cpp:430-435; utils::join_strings drops an empty name)
        if (delim && !comment.empty()) header = name.empty() ? comment : name + delim + comment;
        else header = name;
        out->add(header, seq.data(), seq.size());
        if (fwd_rev) {
            std::string rc(seq.rbegin(), seq.rend());
            for (char &x : rc) x = (char)fastx_complement((uint8_t)x);
            out->add(header, rc.data(), rc.size());
        }
        if (c < 0) { *consumed = n; return; }
        have_hdr = c != '+';
        *consumed = have_hdr ? p - 1 : p;
    }
}

} // namespace mgb
