// TEST INFRASTRUCTURE ONLY: read access to the tables of a built index (IndexView), for tests/index_tables.py.
//
// This file compiles the product's api.cu as it is and adds two entry points, so the tables the tests read come from
// the same mgb_index_create / mgb_index_set_mode code (and, in the nvcc build, the same kernels) as the product's.
// __graft_entry__.build() links it with the product's other objects into tests/devtables/build/libmgb_tables.so;
// tests/emu/Makefile compiles it with -DMGB_HOST_EMU into libmgb_emu.so. The product library never contains it.
#include "../../metagraph_b200/csrc/api.cu"

namespace {

struct TableRef { const void *p; uint64_t bytes; };

TableRef table_of(const mgb_index_t *idx, const char *name) {
    const IndexView &v = idx->view;
    const uint64_t n1 = v.n + 1;
    const std::string s(name);
    uint64_t sfx_entries = 0;
    if (v.sfx && v.sfx_len) {
        sfx_entries = 1;
        for (uint32_t i = 0; i < v.sfx_len; ++i) sfx_entries *= v.sigma - 1;
    }
    if (s == "adj") return { v.adj, v.adj ? n1 * 8 : 0 };
    if (s == "wadj") return { v.wide ? v.wadj : nullptr, v.wide ? n1 * 16 : 0 };
    if (s == "radj") return { v.radj, v.radj ? n1 * 8 : 0 };
    if (s == "kh_keys") return { v.kh_keys, v.kh_keys ? v.kh_slots * 8 : 0 };
    if (s == "kh_vals") return { v.kh_vals, v.kh_vals ? v.kh_slots * 4 : 0 };
    if (s == "pl_node") return { v.pl_node, v.pl_n ? v.pl_n * 4 : 0 };
    if (s == "pl_pos") return { v.pl_pos, v.pl_n ? n1 * 4 : 0 };
    if (s == "pl_text") return { v.pl_text, v.pl_n ? v.pl_n / 4 : 0 };
    if (s == "pl_rc") return { v.pl_rc, v.pl_n ? v.pl_n / 8 : 0 };
    if (s == "pl_stop") return { v.pl_stop, v.pl_n ? v.pl_n / 8 : 0 };
    if (s == "sfx") return { v.sfx, sfx_entries * 8 };
    if (s == "rcs") return { v.rcs, v.rcs ? n1 * 4 : 0 };
    if (s == "rcp") return { v.rcp, v.rcp ? n1 * 4 : 0 };
    if (s == "palin") return { v.palin, v.palin ? ((v.n >> 5) + 1) * 4 : 0 };
    if (s == "valid") return { v.valid, v.valid ? ((n1 + 31) / 32 + 1) * 4 : 0 };
    return { nullptr, UINT64_MAX };
}

} // namespace

extern "C" {

struct mgbt_index_info_t {
    uint64_t n, kh_slots, pl_n;
    uint32_t k, sigma, wide, mode, sfx_len, reserved;
};

int mgbt_index_info(const mgb_index_t *idx, mgbt_index_info_t *out) {
    if (!idx || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    const IndexView &v = idx->view;
    out->n = v.n; out->kh_slots = v.kh_slots; out->pl_n = v.pl_n;
    out->k = v.k; out->sigma = v.sigma; out->wide = v.wide; out->mode = v.mode; out->sfx_len = v.sfx_len;
    out->reserved = 0;
    return MGB_OK;
}

// Size in bytes of table `name` (0: the index does not hold it), or -1 for an unknown name. Copies bytes
// [offset, offset + count) of it to dst when dst is not null; offset + count must not run past its end.
int64_t mgbt_index_copy(const mgb_index_t *idx, const char *name, uint64_t offset, void *dst, uint64_t count) {
    if (!idx || !name) { fail(MGB_ERR_INVALID_ARGUMENT, "null argument"); return -1; }
    const TableRef t = table_of(idx, name);
    if (t.bytes == UINT64_MAX) { fail(MGB_ERR_INVALID_ARGUMENT, std::string("unknown table ") + name); return -1; }
    if (!dst || !count) return (int64_t)t.bytes;
    if (offset > t.bytes || count > t.bytes - offset) { fail(MGB_ERR_INVALID_ARGUMENT, "range past the table's end"); return -1; }
    const char *src = static_cast<const char*>(t.p) + offset;
#if defined(MGB_HOST_EMU)
    std::memcpy(dst, src, count);
#else
    cudaError_t e = cudaSetDevice(idx->device);
    if (e == cudaSuccess) e = cudaMemcpy(dst, src, count, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { fail(MGB_ERR_CUDA, std::string("cudaMemcpy: ") + cudaGetErrorString(e)); return -1; }
#endif
    return (int64_t)t.bytes;
}

} // extern "C"
