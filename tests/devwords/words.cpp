// TEST INFRASTRUCTURE ONLY: the word helpers of k_prepare_exact (metagraph_b200/csrc/acgt_words.cuh) built for the host,
// so that tests/test_acgt_words.py can sweep them against a Python restatement. The product library never contains it.
#include "../../metagraph_b200/csrc/acgt_words.cuh"

extern "C" {

// buf: at least off + 36 bytes, 4-byte aligned; the 32 bytes at buf + off: codes, invalid bits
uint64_t mgbw_pack32(const uint8_t *buf, int off, uint32_t *invalid) { return mgb::acgt_pack32(buf + off, invalid); }
uint32_t mgbw_valid4(uint32_t x) { return mgb::acgt_valid4(x); }
uint32_t mgbw_codes4(uint32_t x) { return mgb::acgt_codes4(x); }
uint64_t mgbw_rc32(uint64_t w) { return mgb::rc_codes32(w); }
void mgbw_count(uint64_t w, int n, int *c) { mgb::acgt_count(w, mgb::codes_mask(n), c); }
uint64_t mgbw_bytes8(const uint8_t *buf, int off) { return mgb::bytes8_at(buf + off); }
uint64_t mgbw_chars8(uint64_t x, int rc) { return mgb::acgt_chars8(x, rc != 0); }

}
