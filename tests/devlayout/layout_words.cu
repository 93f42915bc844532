// TEST INFRASTRUCTURE ONLY: read access to the whole-read gate's lookup tables of a built index (IndexView::kh_pos,
// pl_word) and to the tables they are built from, for tests/test_layout_words_gpu.py.
//
// This file compiles the product's api.cu as it is and adds two entry points, so the tables come from the same
// mgb_index_create code and kernels as the product's. __graft_entry__.build() links it with the product's other
// objects into tests/devlayout/build/libmgb_layout.so. The product library never contains it.
#include "../../metagraph_b200/csrc/api.cu"

namespace {

struct LayoutRef { const void *p; uint64_t bytes; };

LayoutRef layout_table(const mgb_index_t *idx, const char *name) {
    const IndexView &v = idx->view;
    const std::string s(name);
    if (s == "kh_keys") return { v.kh_keys, v.kh_keys ? v.kh_slots * 8 : 0 };
    if (s == "kh_vals") return { v.kh_vals, v.kh_vals ? v.kh_slots * 4 : 0 };
    if (s == "kh_pos") return { v.kh_pos, v.kh_pos ? v.kh_slots * 4 : 0 };
    if (s == "pl_pos") return { v.pl_pos, v.pl_n ? (v.n + 1) * 4 : 0 };
    if (s == "pl_text") return { v.pl_text, v.pl_n ? v.pl_n / 4 : 0 };
    if (s == "pl_rc") return { v.pl_rc, v.pl_n ? v.pl_n / 8 : 0 };
    if (s == "pl_stop") return { v.pl_stop, v.pl_n ? v.pl_n / 8 : 0 };
    if (s == "pl_word") return { v.pl_word, v.pl_word ? v.pl_n / 2 : 0 };
    if (s == "valid") return { v.valid, v.valid ? ((v.n + 1 + 31) / 32 + 1) * 4 : 0 };
    return { nullptr, UINT64_MAX };
}

} // namespace

extern "C" {

// n (edges), kh_slots, pl_n of the index
int mgbl_layout_info(const mgb_index_t *idx, uint64_t *out) {
    if (!idx || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    out[0] = idx->view.n; out[1] = idx->view.kh_slots; out[2] = idx->view.pl_n;
    return MGB_OK;
}

// Size in bytes of table `name` (0: the index does not hold it), or -1 for an unknown name; copies all of it to dst
// when dst is not null
int64_t mgbl_layout_copy(const mgb_index_t *idx, const char *name, void *dst) {
    if (!idx || !name) { fail(MGB_ERR_INVALID_ARGUMENT, "null argument"); return -1; }
    const LayoutRef t = layout_table(idx, name);
    if (t.bytes == UINT64_MAX) { fail(MGB_ERR_INVALID_ARGUMENT, std::string("unknown table ") + name); return -1; }
    if (!dst || !t.bytes) return (int64_t)t.bytes;
    cudaError_t e = cudaSetDevice(idx->device);
    if (e == cudaSuccess) e = cudaMemcpy(dst, t.p, t.bytes, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { fail(MGB_ERR_CUDA, std::string("cudaMemcpy: ") + cudaGetErrorString(e)); return -1; }
    return (int64_t)t.bytes;
}

} // extern "C"
