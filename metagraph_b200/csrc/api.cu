// C-ABI (include/mgb.h) of the H100-native `metagraph align` hot path: index upload, the three
// sm_90a kernels (query preparation, quad-per-strand exact seeding, warp-per-read
// seed-and-extend) and result unpacking.
//
// When compiled by g++ with -DMGB_HOST_EMU (tests/emu/ only) the same logic runs with
// one-lane "warps" on host memory so that it can be checked against the oracle on a machine
// without a GPU. That build is test infrastructure; the product library is always the nvcc
// build and has no CPU path.
#include <algorithm>
#include <atomic>
#include <thread>
#include <chrono>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>
#include <string>
#include <vector>
#if defined(_OPENMP)
#include <omp.h>
#endif

// Threads per OpenMP team of the result-unpacking loops. They are short, memory-bound loops that run on two
// pipeline lanes at once: beyond a few cores they gain nothing, and with one team per lane as wide as a
// 128-thread host the teams spend their time spinning against each other (scripts/e2e_probe.py times the call by
// piece, lane and thread count). mgb_set_host_threads() can only lower the number.
[[maybe_unused]] static inline int host_team() {
#if defined(_OPENMP)
    const int n = omp_get_max_threads();
    return n < 16 ? (n < 1 ? 1 : n) : 16;
#else
    return 1;
#endif
}

// memcpy of n bytes in 4 MiB chunks, on host_team() threads when there are more than four chunks
static void parallel_copy(char *dst, const char *src, uint64_t n) {
    const int64_t chunks = (int64_t)((n + (1 << 22) - 1) >> 22);
    #pragma omp parallel for schedule(static) num_threads(host_team()) if (chunks > 4)
    for (int64_t c = 0; c < chunks; ++c) {
        const uint64_t o = (uint64_t)c << 22;
        std::memcpy(dst + o, src + o, std::min<uint64_t>(1ull << 22, n - o));
    }
}

#include "../../include/mgb.h"
#if !defined(MGB_HOST_EMU)
#define MGB_NARROW_ONLY 1        // this translation unit's kernels: DNA block layout only (see kernels.cuh)
#define MGB_BASIC_ONLY 1         // ... and BASIC-mode graphs only (api_canonical.cu holds the CANONICAL-mode k_align)
#endif
#define MGB_KERNEL_NS kern_dna
#include "kernels.cuh"
#include "format_core.cuh"
#include "fastx_core.cuh"
#include "gzip_core.cuh"
#include "columns_core.cuh"
#include "fastx_host.hpp"
#include "host_common.hpp"
#include "index_build.hpp"

#if !defined(MGB_HOST_EMU)
#include <cuda_runtime.h>
#endif

using namespace mgb;

// A plain gzip stream between stages, in host memory so that the next stage may run on any device: where the next
// stage starts, and the state of the member it is in (DESIGN.md §8 "Plain gzip input").
struct mgb_gzip_stream {
    bool in_member = false;
    uint32_t bit = 0;                     // bits of the next input's first byte already decoded
    uint64_t member_text = 0;             // text of the member staged so far (ISIZE is it modulo 2^32)
    uint32_t crc = 0;                     // its CRC32
    std::vector<uint8_t> window = std::vector<uint8_t>(kGzipWindow, 0);   // its last 32 KiB, right-aligned
    uint64_t c_bits = 0, text = 0;        // compressed bits and text so far: the ratio that sizes a stage
};

namespace {

thread_local std::string g_err;

int fail(int code, const std::string &msg) { g_err = msg; return code; }

void add_stats(mgb_stats_t &t, const mgb_stats_t &u) {
    t.num_seeds += u.num_seeds; t.num_extensions += u.num_extensions;
    t.num_explored_nodes += u.num_explored_nodes; t.dp_cells += u.dp_cells; t.dp_columns += u.dp_columns;
    t.num_reads_retried += u.num_reads_retried; t.seed_kernel_ms += u.seed_kernel_ms;
    t.align_kernel_ms += u.align_kernel_ms; t.h2d_ms += u.h2d_ms; t.d2h_ms += u.d2h_ms;
    t.h2d_bytes += u.h2d_bytes; t.d2h_bytes += u.d2h_bytes; t.kernel_launches += u.kernel_launches;
}


#if !defined(MGB_HOST_EMU)
} // namespace
// the same kernels compiled for the alphabet-generic layout (api_generic.cu)
namespace kern_any {
cudaError_t launch_radj_bwd(unsigned grid, const mgb::RadjArgs &a);
cudaError_t launch_sfx_extend(unsigned grid, const mgb::SfxArgs &a);
cudaError_t launch_seed(unsigned grid, cudaStream_t s, const mgb::SeedArgs &a);
cudaError_t launch_premap(unsigned grid, cudaStream_t s, const mgb::SeedArgs &a);
cudaError_t launch_subk(unsigned grid, cudaStream_t s, const mgb::SubkArgs &a, uint32_t chunks_per_strand);
cudaError_t launch_align(unsigned grid, size_t smem_block, cudaStream_t s, const mgb::AlignArgs &a);
cudaError_t align_occupancy(size_t smem_limit, size_t smem_block, int *blocks_per_sm);
}
// k_align for CANONICAL-mode DNA graphs (api_canonical.cu)
namespace kern_canon {
cudaError_t launch_align(unsigned grid, size_t smem_block, cudaStream_t s, const mgb::AlignArgs &a);
cudaError_t align_occupancy(size_t smem_limit, size_t smem_block, int *blocks_per_sm);
}
namespace {
#endif

#if !defined(MGB_HOST_EMU)
#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) \
    return fail(MGB_ERR_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)
#endif

// ---------------------------------------------------------------------------------------
// device memory helpers
// ---------------------------------------------------------------------------------------
// sync: waits for the stream's work (MGB_ERR_CUDA with the CUDA error text if it failed); record / elapsed_ms: the
// workspace's events ev[i], which the device timers of mgb_stats_t are measured between. The emulation runs every
// operation when it is issued, so these do nothing there.
#if defined(MGB_HOST_EMU)
struct Stream { int dummy; };
inline int dev_alloc(void **p, size_t bytes, Stream&) { *p = std::calloc(1, bytes ? bytes : 1); return *p ? 0 : MGB_ERR_CUDA; }
inline void dev_free(void *p, Stream&) { std::free(p); }
inline int h2d(void *d, const void *h, size_t bytes, Stream&) { std::memcpy(d, h, bytes); return 0; }
inline int d2h(void *h, const void *d, size_t bytes, Stream&) { std::memcpy(h, d, bytes); return 0; }
inline int dev_zero(void *d, size_t bytes, Stream&) { std::memset(d, 0, bytes); return 0; }
inline int sync(Stream&) { return 0; }
inline void record(Stream&, int) {}
inline float elapsed_ms(Stream&, int, int) { return 0; }
#else
struct Stream { cudaStream_t s = nullptr; cudaEvent_t *ev = nullptr; };
inline int dev_alloc(void **p, size_t bytes, Stream &st) {
    cudaError_t e = cudaMallocAsync(p, bytes ? bytes : 16, st.s);
    if (e != cudaSuccess) { g_err = std::string("cudaMallocAsync: ") + cudaGetErrorString(e); return MGB_ERR_CUDA; }
    return 0;
}
inline void dev_free(void *p, Stream &st) { if (p) cudaFreeAsync(p, st.s); }
inline int h2d(void *d, const void *h, size_t bytes, Stream &st) {
    cudaError_t e = cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st.s);
    if (e != cudaSuccess) { g_err = std::string("H2D: ") + cudaGetErrorString(e); return MGB_ERR_CUDA; }
    return 0;
}
inline int d2h(void *h, const void *d, size_t bytes, Stream &st) {
    cudaError_t e = cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st.s);
    if (e != cudaSuccess) { g_err = std::string("D2H: ") + cudaGetErrorString(e); return MGB_ERR_CUDA; }
    return 0;
}
inline int dev_zero(void *d, size_t bytes, Stream &st) {
    cudaError_t e = cudaMemsetAsync(d, 0, bytes, st.s);
    if (e != cudaSuccess) { g_err = std::string("memset: ") + cudaGetErrorString(e); return MGB_ERR_CUDA; }
    return 0;
}
inline int sync(Stream &st) {
    cudaError_t e = cudaStreamSynchronize(st.s);
    if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    return 0;
}
inline void record(Stream &st, int i) { cudaEventRecord(st.ev[i], st.s); }
inline float elapsed_ms(Stream &st, int from, int to) { float ms = 0; cudaEventElapsedTime(&ms, st.ev[from], st.ev[to]); return ms; }
#endif

// Host buffers that receive the packed results. On the device build they are pinned and
// recycled through a process-wide pool (cudaHostAlloc of GB-sized buffers costs 100s of ms), so a
// mgb_results_t owns its buffers zero-copy and hands them back in mgb_results_free().
struct HostBuf { char *p = nullptr; size_t cap = 0; };
#if defined(MGB_HOST_EMU)
inline HostBuf hostbuf_acquire(size_t bytes) { HostBuf b; b.cap = bytes ? bytes : 1; b.p = (char*)std::malloc(b.cap); return b; }
inline void hostbuf_release(HostBuf b) { std::free(b.p); }
#else
struct PinnedPool {
    std::mutex mu;
    std::vector<HostBuf> free_list;
    HostBuf acquire(size_t bytes) {
        {
            std::lock_guard<std::mutex> lk(mu);
            size_t best = free_list.size();
            for (size_t i = 0; i < free_list.size(); ++i)
                if (free_list[i].cap >= bytes && (best == free_list.size() || free_list[i].cap < free_list[best].cap)) best = i;
            if (best != free_list.size()) { HostBuf b = free_list[best]; free_list.erase(free_list.begin() + best); return b; }
        }
        HostBuf b;
        size_t want = bytes + bytes / 8 + 4096;
        if (cudaHostAlloc((void**)&b.p, want, cudaHostAllocDefault) != cudaSuccess) { b.p = nullptr; b.cap = 0; return b; }
        b.cap = want;
        return b;
    }
    void release(HostBuf b) {
        if (!b.p) return;
        std::lock_guard<std::mutex> lk(mu);
        if (free_list.size() >= 32) { cudaFreeHost(b.p); return; }
        free_list.push_back(b);
    }
};
PinnedPool g_pinned_pool;
inline HostBuf hostbuf_acquire(size_t bytes) { return g_pinned_pool.acquire(bytes); }
inline void hostbuf_release(HostBuf b) { g_pinned_pool.release(b); }
#endif

// Device working memory of one call. On the device build the buffers belong to a Workspace that the
// index keeps between calls (slot i = the i-th request of the call): cudaMalloc of GB-sized arenas per
// call is slow, and stream-ordered pools stall when two streams trade memory back and forth.
// Every DevBufs takes consecutive slots of one region, and an allocation past the region's end fails, in both builds.
constexpr int kMaxPasses = 6;          // align_piece gives up on a read after six passes
struct Region { const char *name; size_t base, end; };
constexpr Region kBatchSlots { "batch", 0, 32 };              // the batch's buffers; the file route's parse
constexpr Region kArenaSlots { "arena", 32, 33 };             // the align pass's arena
constexpr Region kPassHeapSlots { "pass heap", 33, 40 };      // record route: the heap, list and counters of a pass
// text and columns routes: every pass keeps its heap on the device until the text or the columns are made from it
inline Region kept_heap_slots(int pass) { return { "kept heap", 40 + 8 * (size_t)pass, 48 + 8 * (size_t)pass }; }
constexpr Region kInflateSlots { "inflate", 88, 96 };        // plain gzip input: a stage's decode scratch
constexpr Region kTextSlots { "text", 96, SIZE_MAX };         // text route: the headers and the text
static_assert(40 + 8 * kMaxPasses <= kTextSlots.base, "the kept heaps end below the text region");
static_assert(kMaxPasses <= kColumnsMaxPasses, "ColumnsArgs holds a heap per pass");

#if defined(MGB_HOST_EMU)
struct Workspace {};
#else
struct Workspace {
    std::vector<void*> ptr;
    std::vector<size_t> cap;
    cudaStream_t stream = nullptr;       // created on first use, kept with the buffers
    cudaEvent_t ev[6] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };
    int ready() {
        if (stream) return 0;
        cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        for (auto &x : ev) if (e == cudaSuccess) e = cudaEventCreate(&x);
        if (e != cudaSuccess) { g_err = std::string("stream/event creation: ") + cudaGetErrorString(e); return MGB_ERR_CUDA; }
        return 0;
    }
    ~Workspace() {
        for (void *p : ptr) if (p) cudaFree(p);
        for (auto &x : ev) if (x) cudaEventDestroy(x);
        if (stream) cudaStreamDestroy(stream);
    }
    int get(size_t slot, size_t bytes, void **out) {
        if (slot >= ptr.size()) { ptr.resize(slot + 1, nullptr); cap.resize(slot + 1, 0); }
        if (cap[slot] < bytes || !ptr[slot]) {
            if (ptr[slot]) cudaFree(ptr[slot]);
            ptr[slot] = nullptr; cap[slot] = 0;
            size_t want = bytes + bytes / 8 + 256;
            cudaError_t e = cudaMalloc(&ptr[slot], want);
            if (e != cudaSuccess) { cudaGetLastError(); want = bytes ? bytes : 16; e = cudaMalloc(&ptr[slot], want); }
            if (e != cudaSuccess) {
                ptr[slot] = nullptr;
                g_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
                return MGB_ERR_CUDA;
            }
            cap[slot] = want;
        }
        *out = ptr[slot];
        return 0;
    }
};
#endif
struct DevBufs {               // (the emulation build frees what it took on scope exit)
    Stream &st;
    Workspace *ws;
    Region region;
    size_t slot;
    std::vector<void*> owned;
    DevBufs(Stream &s, Workspace *w, Region r) : st(s), ws(w), region(r), slot(r.base) {}
    ~DevBufs() { for (void *p : owned) dev_free(p, st); }
    template <class T> int alloc(T **p, size_t count) {
        if (slot >= region.end) return fail(MGB_ERR_CUDA, std::string("workspace region '") + region.name + "' is full");
        void *v = nullptr;
#if defined(MGB_HOST_EMU)
        ++slot;
        if (int rc = dev_alloc(&v, count * sizeof(T), st)) return rc;
        owned.push_back(v);
#else
        if (int rc = ws->get(slot++, count * sizeof(T), &v)) return rc;
#endif
        *p = (T*)v;
        return 0;
    }
#if !defined(MGB_HOST_EMU)
    size_t capacity_of_next() const { return slot < ws->cap.size() ? ws->cap[slot] : 0; }
#endif
};

} // namespace

// ---------------------------------------------------------------------------------------
// opaque types
// ---------------------------------------------------------------------------------------
struct mgb_index {
    // owns its device buffers and cached workspaces: every error path of mgb_index_create releases what was uploaded
    ~mgb_index();
    IndexView view;            // device pointers (host pointers in the emulation build)
    int device = 0;
    uint64_t device_bytes = 0;
    int num_sms = 1;
    struct DevArray { const void *p; size_t bytes; };
    std::vector<DevArray> bufs;        // every device array the index owns (the device build)
    void keep(const void *p, size_t bytes) { bufs.push_back({ p, bytes }); device_bytes += bytes; }
#if defined(MGB_HOST_EMU)
    std::vector<uint32_t> rc_host;   // PRIMARY graphs: rcs / rcp / palin (mgb_index_set_mode)
#endif
    int alphabet = MGB_ALPHABET_DNA;
    AlphabetTables at;
    // working memory recycled between calls (at most 4 sets are kept)
    mutable std::mutex ws_mu;
    mutable std::vector<Workspace*> ws_free;
    Workspace* ws_acquire() const {
        std::lock_guard<std::mutex> lk(ws_mu);
        if (ws_free.empty()) return new Workspace();
        Workspace *w = ws_free.back(); ws_free.pop_back(); return w;
    }
    void ws_release(Workspace *w) const {
        std::lock_guard<std::mutex> lk(ws_mu);
        if (ws_free.size() < 4) ws_free.push_back(w); else delete w;
    }
#if defined(MGB_HOST_EMU)
    HostIndex host;
    std::vector<uint2> radj_host;
#endif
};

mgb_index::~mgb_index() {
#if !defined(MGB_HOST_EMU)
    if (!bufs.empty()) { cudaSetDevice(device); for (const DevArray &b : bufs) cudaFree(const_cast<void*>(b.p)); }
#endif
    for (Workspace *w : ws_free) delete w;
}

struct mgb_results {
    uint32_t n_reads = 0;
    std::vector<uint64_t> first;
    std::vector<uint32_t> count;
    mgb_alignment_t *alns = nullptr;         // n_alns records in read order, inside alns_buf
    uint64_t n_alns = 0;
    HostBuf alns_buf;
    std::vector<HostBuf> heaps;              // host copies of the output heaps (recycled on free)
    std::vector<uint64_t> heap_bytes;        // used bytes of each heap
    // where the packed records of read r start: heap src_heap[r], byte src_off[r] (mgb_results_export)
    std::vector<uint64_t> src_off;
    std::vector<uint32_t> src_heap;
    uint32_t result_nodes = 0;
    // a text result set (mgb_align_batch_text): MGB_TEXT_TSV / MGB_TEXT_JSON, and the block (no records, no heaps)
    int text_format = 0;
    HostBuf text;
    uint64_t text_bytes = 0;
    ~mgb_results() {
        for (HostBuf b : heaps) hostbuf_release(b);
        if (alns_buf.p) hostbuf_release(alns_buf);
        if (text.p) hostbuf_release(text);
    }
    mgb_stats_t stats;
};

namespace {
// A workspace of the index held for the duration of a call, with its stream and events. ready() makes the index's
// device current. The destructor waits for the call's work on the stream before the workspace goes back; that wait is
// unchecked, so the call's own result and error text stand.
struct CallWorkspace {
    const mgb_index_t *ix; Workspace *w; Stream st; bool ready_ = false;
    explicit CallWorkspace(const mgb_index_t *i) : ix(i), w(i->ws_acquire()) {}
    ~CallWorkspace() {
        if (ready_) { const std::string err = g_err; sync(st); g_err = err; }
        ix->ws_release(w);
    }
    int ready() {
#if !defined(MGB_HOST_EMU)
        CUDA_TRY(cudaSetDevice(ix->device));
        if (int rc = w->ready()) return rc;
        st.s = w->stream; st.ev = w->ev;
#endif
        ready_ = true;
        return MGB_OK;
    }
};
} // namespace

#if !defined(MGB_HOST_EMU)
// IndexView::pl_word (0.5 bytes per position) and kh_pos (4 bytes per hash slot), the whole-read gate's leaner copies of
// the path layout, once the layout is in place. Each is built only if half the device memory (at least 16 GB) stays
// free after it: the aligner sizes its working memory from what is free, and on a 1 B-node graph (C3) the 6.2 GB of both
// tables left an 80 GB H100 short at align time. Without them the gate reads the layout arrays. MGB_TEST_NO_LAYOUT_WORDS (test knob) leaves out kh_pos (value "kh_pos"),
// pl_word ("pl_word") or both (any other value).
static int build_layout_words(mgb_index *idx) {
    IndexView &v = idx->view;
    if (!v.pl_n || !v.kh_slots) return MGB_OK;
    const char *no = std::getenv("MGB_TEST_NO_LAYOUT_WORDS");
    const bool want_word = !no || !std::strcmp(no, "kh_pos"), want_pos = !no || !std::strcmp(no, "pl_word");
    const uint64_t word_bytes = v.pl_n / 32 * 16, pos_bytes = v.kh_slots * 4;
    ulonglong2 *pl_word = nullptr; uint32_t *kh_pos = nullptr;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    double left = (double)free_b;
    const double keep = std::max(16e9, 0.5 * (double)total_b);
    if (want_word && left - word_bytes >= keep && cudaMalloc((void**)&pl_word, word_bytes) == cudaSuccess)
        left -= word_bytes;
    else pl_word = nullptr;
    if (!want_pos || left - pos_bytes < keep || cudaMalloc((void**)&kh_pos, pos_bytes) != cudaSuccess) kh_pos = nullptr;
    cudaGetLastError();
    if (!pl_word && !kh_pos) return MGB_OK;
    kern_dna::k_layout_words<<<(unsigned)idx->num_sms * 16, 256>>>(v, kh_pos, pl_word);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(pl_word); cudaFree(kh_pos);
        return fail(MGB_ERR_CUDA, std::string("layout words: ") + cudaGetErrorString(e));
    }
    if (pl_word) { idx->keep(pl_word, word_bytes); v.pl_word = pl_word; }
    if (kh_pos) { idx->keep(kh_pos, pos_bytes); v.kh_pos = kh_pos; }
    return MGB_OK;
}

// Path layout of a graph with the k-mer hash index (IndexView::pl_*, kernels.cuh k_path_*), from the per-edge k-mers
// of the hash build. Skipped, leaving the seeding walk as it is without it, when the device memory is not there (it
// keeps the same 16 GB for the aligner's working memory as the hash index) or MGB_NO_PATH_INDEX is set.
static int build_path_layout(mgb_index *idx, const unsigned long long *kmer) {
    const uint64_t n = idx->view.n;
    if (std::getenv("MGB_NO_PATH_INDEX") || n >= (1ull << 31)) return MGB_OK;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    // pred + jump during the build; pl_pos stays, and the positions take about 4.5 bytes per edge
    if ((double)free_b < 1.2 * 16.5 * (n + 1) || (double)free_b - 8.6 * (n + 1) < 16e9) return MGB_OK;
    kern_dna::PathArgs a;
    std::memset(&a, 0, sizeof(a));
    a.ix = idx->view; a.kmer = kmer;
    struct Counters { unsigned long long total; unsigned int count; };
    Counters *ctr = nullptr;
    auto drop = [&]() {
        cudaGetLastError();
        cudaFree(a.pred); cudaFree(a.jump); cudaFree(a.node); cudaFree(a.text); cudaFree(a.rc); cudaFree(a.stop); cudaFree(ctr);
        return MGB_OK;
    };
    if (cudaMalloc((void**)&a.pred, (n + 1) * 4) != cudaSuccess || cudaMalloc((void**)&a.jump, (n + 1) * 8) != cudaSuccess
            || cudaMalloc((void**)&ctr, sizeof(Counters)) != cudaSuccess)
        return drop();
    a.total = &ctr->total; a.count = &ctr->count;
    cudaError_t e = cudaMemset(a.pred, 0xFF, (n + 1) * 4);
    if (e == cudaSuccess) e = cudaMemset(ctr, 0, sizeof(Counters));
    const unsigned grid = (unsigned)idx->num_sms * 16;
    auto check = [&](const char *what) -> int {
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e == cudaSuccess) return MGB_OK;
        drop();
        return fail(MGB_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
    };
    // *count after one launch of kernel f
    auto counted = [&](void (*f)(kern_dna::PathArgs)) -> unsigned {
        unsigned c = 0;
        if (e == cudaSuccess) e = cudaMemset(a.count, 0, 4);
        if (e == cudaSuccess) { f<<<grid, 256>>>(a); e = cudaGetLastError(); }
        if (e == cudaSuccess) e = cudaMemcpy(&c, a.count, 4, cudaMemcpyDeviceToHost);
        return c;
    };
    auto rank = [&]() { while (e == cudaSuccess && counted(kern_dna::k_path_jump)) {} };
    kern_dna::k_path_pred<<<grid, 256>>>(a);
    kern_dna::k_path_link<<<grid, 256>>>(a);
    rank();
    const unsigned cycle_nodes = counted(kern_dna::k_path_cycle_init);
    if (cycle_nodes) {
        for (unsigned w = 1; ; w *= 2) {               // the smallest node over windows of 2w >= every cycle's length
            kern_dna::k_path_cycle_min<<<grid, 256>>>(a);
            if (w >= cycle_nodes) break;
        }
        kern_dna::k_path_cycle_cut<<<grid, 256>>>(a);
        rank();
    }
    kern_dna::k_path_heads<<<grid, 256>>>(a);
    unsigned long long used = 0;
    if (e == cudaSuccess) e = cudaMemcpy(&used, a.total, 8, cudaMemcpyDeviceToHost);
    if (int rc = check("path layout")) return rc;
    const uint64_t n_pos = ((used + 63) & ~63ull) + kPlPad;
    if (n_pos >= (1ull << 32)) return drop();
    cudaMemGetInfo(&free_b, &total_b);
    const uint64_t bytes = n_pos * 4 + n_pos / 4 + 2 * (n_pos / 8);
    if ((double)free_b < 1.2 * bytes || cudaMalloc((void**)&a.node, n_pos * 4) != cudaSuccess
            || cudaMalloc((void**)&a.text, n_pos / 4) != cudaSuccess || cudaMalloc((void**)&a.rc, n_pos / 8) != cudaSuccess
            || cudaMalloc((void**)&a.stop, n_pos / 8) != cudaSuccess)
        return drop();
    e = cudaMemset(a.node, 0, n_pos * 4);
    if (e == cudaSuccess) e = cudaMemset(a.text, 0, n_pos / 4);
    if (e == cudaSuccess) e = cudaMemset(a.rc, 0, n_pos / 8);
    if (e == cudaSuccess) e = cudaMemset(a.stop, 0xFF, n_pos / 8);
    if (e == cudaSuccess) kern_dna::k_path_place<<<grid, 256>>>(a);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (int rc = check("path layout")) return rc;
    cudaFree(a.jump); cudaFree(ctr);
    idx->keep(a.pred, (n + 1) * 4); idx->keep(a.node, n_pos * 4); idx->keep(a.text, n_pos / 4); idx->keep(a.rc, n_pos / 8);
    idx->keep(a.stop, n_pos / 8);
    idx->view.pl_pos = a.pred; idx->view.pl_node = a.node;
    idx->view.pl_text = reinterpret_cast<const unsigned long long*>(a.text);
    idx->view.pl_rc = a.rc; idx->view.pl_stop = a.stop;
    idx->view.pl_n = n_pos;
    return build_layout_words(idx);
}
#endif

#if !defined(MGB_HOST_EMU)
// what an index sets up on the device it lives on (the current device)
static void device_setup(int device) {
    {   // Every access of this path to the index and to the per-read arenas is a single 8 .. 64-byte record at a
        // data-dependent address; L2 may fetch whole 128-byte lines from HBM for them. MGB_L2_FETCH=32 / 64 asks for
        // smaller fetches (process-wide): fewer bytes, but the access rate, not the bytes, is what HBM limits on this
        // path, so the default is left alone unless MGB_L2_FETCH is set.
        size_t gran = 0;
        if (const char *e = std::getenv("MGB_L2_FETCH")) gran = (size_t)std::atoi(e);
        if (gran) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
        cudaGetLastError();
    }
    {   // keep stream-ordered allocations cached between calls
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            uint64_t thr = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
    }
}

// f(field, name, opt) for every pointer of the view: the table's name and, for the tables mgb_index_create builds only
// when the device memory is there (and no knob leaves them out), which one it is
enum class Opt { none, hash, path, pl_word, kh_pos };
template <class F> static void each_table(IndexView &v, F &&f) {
    f(v.blocks, "blocks", Opt::none); f(v.blk_rank, "blk_rank", Opt::none); f(v.sel_last, "sel_last", Opt::none);
    for (auto &p : v.sel_W) f(p, "sel_W", Opt::none);
    f(v.valid, "valid", Opt::none); f(v.sfx, "sfx", Opt::none); f(v.adj, "adj", Opt::none);
    f(v.radj, "radj", Opt::none);
    f(v.kh_keys, "kh_keys", Opt::hash); f(v.kh_vals, "kh_vals", Opt::hash);
    f(v.pl_node, "pl_node", Opt::path); f(v.pl_pos, "pl_pos", Opt::path); f(v.pl_text, "pl_text", Opt::path);
    f(v.pl_rc, "pl_rc", Opt::path); f(v.pl_stop, "pl_stop", Opt::path);
    f(v.kh_pos, "kh_pos", Opt::kh_pos); f(v.pl_word, "pl_word", Opt::pl_word);
    f(v.rcs, "rcs", Opt::none); f(v.rcp, "rcp", Opt::none); f(v.palin, "palin", Opt::none);
    f(v.wW, "wW", Opt::none); f(v.wl, "wl", Opt::none); f(v.wrank, "wrank", Opt::none); f(v.wsel, "wsel", Opt::none);
    f(v.wadj, "wadj", Opt::none);
}
#endif

extern "C" {

const char* mgb_last_error(void) { return g_err.c_str(); }

int mgb_device_count(void) {
#if defined(MGB_HOST_EMU)
    return 1;
#else
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
#endif
}

int mgb_index_create(const uint8_t *W, const uint8_t *last, uint64_t n_plus_1, const uint64_t *F,
                     const uint8_t *valid, uint32_t k, int alphabet, uint32_t suffix_len,
                     int device, mgb_index_t **out) {
    if (!W || !last || !F || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    std::unique_ptr<mgb_index> idx(new mgb_index());
    if (!alphabet_tables(alphabet, &idx->at)) return fail(MGB_ERR_UNSUPPORTED, "unknown alphabet");
    idx->alphabet = alphabet;
    const uint32_t sigma = idx->at.sigma;
    const bool force_wide = std::getenv("MGB_TEST_WIDE") != nullptr;   // test knob: generic layout for DNA
    HostIndex hloc;
#if defined(MGB_HOST_EMU)
    HostIndex &h = idx->host;
#else
    HostIndex &h = hloc;
#endif
    if (suffix_len == 0) {
        // reference default 12 (cli/config/config.cpp:24-25). Here: as long as the table has at most
        // ~12 entries per edge and 2^30 entries (8 GiB): a cold k-mer lookup that misses in the table
        // costs one load instead of a chain of tighten_range steps, and on a strand that does not match
        // every k-mer is a cold lookup. HBM capacity is traded for latency.
        uint64_t n = n_plus_1 - 1;
        suffix_len = 1;
        uint64_t entries = sigma - 1;
        while (suffix_len < 15 && suffix_len + 1 <= k - 1 && entries * (sigma - 1) <= 12 * n + 1024
               && entries * (sigma - 1) <= (1ull << 30) + (1ull << 26)) {
            entries *= sigma - 1; ++suffix_len;
        }
    }
    // levels up to 8 are refined on the host, the rest by k_sfx_extend on the device
    const uint32_t sfx_target = suffix_len > k - 1 ? k - 1 : suffix_len;
    // (host levels: at most 4^8 = 65k entries' worth)
    uint32_t sfx_host = 0;
    for (uint64_t e = 1; sfx_host < sfx_target && e * (sigma - 1) <= 65536; e *= sigma - 1) ++sfx_host;
    if (sfx_host == 0 && sfx_target) sfx_host = 1;
    try {
        build_host_index(W, last, n_plus_1, F, valid, k, sfx_host, &h, sigma, force_wide);
    } catch (const std::exception &e) {
        return fail(MGB_ERR_INVALID_ARGUMENT, e.what());
    }
#if defined(MGB_HOST_EMU)
    (void)device; (void)hloc;
    idx->view = h.view();
    {
        uint64_t cur_num = 1;
        for (uint32_t i = 0; i < sfx_host; ++i) cur_num *= (sigma - 1);
        for (uint32_t len = sfx_host + 1; len <= sfx_target && sfx_host >= 1; ++len) {
            const uint64_t nxt_num = cur_num * (sigma - 1);
            std::vector<uint32_t> nxt(2 * nxt_num);
            SfxArgs sa { idx->view, idx->view.sfx, nxt.data(), cur_num };
            sa.ix.sfx = nullptr; sa.ix.sfx_len = 0;
            for (uint64_t o = 0; o < nxt_num; ++o) sfx_extend_item(sa, o);
            h.sfx.swap(nxt);
            cur_num = nxt_num;
            idx->view.sfx = h.sfx.data(); idx->view.sfx_len = len;
        }
    }
    {
        const uint64_t n = idx->view.n;
        std::vector<uint32_t> bwd_arr(n + 1, 0);
        std::vector<uint8_t> c0(n + 1, 0), c1(n + 1, 0), multi(n + 1, 0);
        idx->radj_host.assign(n + 1, uint2{0, 0});
        RadjArgs ra { idx->view, bwd_arr.data(), c0.data(), c1.data(), multi.data(), idx->radj_host.data(), n, nullptr };
        for (uint64_t e = 1; e <= n; ++e) radj_bwd_item(ra, e);
        for (uint32_t r = 0; r + 2 < k; ++r) {
            for (uint64_t e = 1; e <= n; ++e) ra.c_nxt[e] = ra.c_cur[bwd_arr[e]];
            std::swap(ra.c_cur, ra.c_nxt);
        }
        for (uint64_t e = 1; e <= n; ++e)
            idx->radj_host[e] = uint2{ bwd_arr[e], (uint32_t)ra.c_cur[e] | ((uint32_t)multi[e] << radj_multi_shift(idx->view)) };
        idx->view.radj = idx->radj_host.data();
    }
    idx->device_bytes = h.blocks.size() * 4 + h.wW.size();
#else
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(MGB_ERR_NO_DEVICE, "no CUDA device available (the kernels have no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(MGB_ERR_INVALID_ARGUMENT, "bad device ordinal");
    CUDA_TRY(cudaSetDevice(device));
    idx->device = device;
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    idx->num_sms = prop.multiProcessorCount;
    device_setup(device);
    IndexView v = h.view();
    auto upload = [&](const std::vector<uint32_t> &src, const uint32_t **dst) -> int {
        if (src.empty()) { *dst = nullptr; return 0; }
        void *p = nullptr;
        cudaError_t e = cudaMalloc(&p, src.size() * 4);
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
        idx->keep(p, src.size() * 4);
        e = cudaMemcpy(p, src.data(), src.size() * 4, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMemcpy: ") + cudaGetErrorString(e));
        *dst = (const uint32_t*)p;
        return 0;
    };
    int rc;
    if ((rc = upload(h.blocks, &v.blocks))) return rc;
    if ((rc = upload(h.blk_rank, &v.blk_rank))) return rc;
    if ((rc = upload(h.sel_last, &v.sel_last))) return rc;
    for (int c = 0; c < kSigmaDNA; ++c)
        if ((rc = upload(h.sel_W[c], &v.sel_W[c]))) return rc;
    if ((rc = upload(h.valid, &v.valid))) return rc;
    if ((rc = upload(h.sfx, &v.sfx))) return rc;
    if (h.wide) {
        std::vector<uint32_t> wW32((h.wW.size() + 3) / 4);
        std::memcpy(wW32.data(), h.wW.data(), h.wW.size());
        const uint32_t *p32 = nullptr;
        if ((rc = upload(wW32, &p32))) return rc;
        v.wW = (const uint8_t*)p32;
        if ((rc = upload(h.wl, &v.wl))) return rc;
        if ((rc = upload(h.wrank, &v.wrank))) return rc;
        if ((rc = upload(h.wsel, &v.wsel))) return rc;
        if ((rc = upload(h.wadj, &v.wadj))) return rc;
        v.adj = nullptr;
    } else {
        void *p = nullptr;
        cudaError_t e = cudaMalloc(&p, h.adj.size() * sizeof(uint2));
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMalloc(adj): ") + cudaGetErrorString(e));
        idx->keep(p, h.adj.size() * sizeof(uint2));
        e = cudaMemcpy(p, h.adj.data(), h.adj.size() * sizeof(uint2), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMemcpy(adj): ") + cudaGetErrorString(e));
        v.adj = (const uint2*)p;
    }
    idx->view = v;
    // deeper suffix-range levels on the device
    {
        uint64_t cur_num = 1;
        for (uint32_t i = 0; i < sfx_host; ++i) cur_num *= (sigma - 1);
        const uint32_t *cur = v.sfx;
        for (uint32_t len = sfx_host + 1; len <= sfx_target && sfx_host >= 1; ++len) {
            uint32_t *nxt = nullptr;
            const uint64_t nxt_num = cur_num * (sigma - 1);
            cudaError_t e = cudaMalloc((void**)&nxt, nxt_num * 8);
            if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMalloc(sfx): ") + cudaGetErrorString(e));
            SfxArgs sa { idx->view, cur, nxt, cur_num };
            sa.ix.sfx = nullptr; sa.ix.sfx_len = 0;
            uint64_t blocks = std::min<uint64_t>((nxt_num + 31) / 32, (uint64_t)idx->num_sms * 32);
            e = idx->view.wide ? kern_any::launch_sfx_extend((unsigned)blocks, sa) : kern_dna::launch_sfx_extend((unsigned)blocks, sa);
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { cudaFree(nxt); return fail(MGB_ERR_CUDA, std::string("k_sfx_extend: ") + cudaGetErrorString(e)); }   // (idx's destructor frees the rest)
            // the previous level is no longer needed (the host-built one is freed with the index)
            if (len > sfx_host + 1) {
                cudaFree((void*)cur);
                idx->bufs.erase(std::find_if(idx->bufs.begin(), idx->bufs.end(), [&](const mgb_index::DevArray &b) { return b.p == cur; }));
                idx->device_bytes -= cur_num * 8;
            }
            idx->keep(nxt, nxt_num * 8);
            cur = nxt; cur_num = nxt_num;
            idx->view.sfx = nxt; idx->view.sfx_len = len;
        }
    }
    // reverse adjacency records
    {
        const uint64_t n = idx->view.n;
        uint32_t *bwd_arr = nullptr; uint8_t *c0 = nullptr, *c1 = nullptr, *multi = nullptr; uint2 *radj = nullptr;
        cudaError_t e = cudaMalloc((void**)&bwd_arr, (n + 1) * 4);
        if (e == cudaSuccess) e = cudaMalloc((void**)&c0, n + 1);
        if (e == cudaSuccess) e = cudaMalloc((void**)&c1, n + 1);
        if (e == cudaSuccess) e = cudaMalloc((void**)&multi, n + 1);
        if (e == cudaSuccess) e = cudaMalloc((void**)&radj, (n + 1) * sizeof(uint2));
        if (e != cudaSuccess) {
            cudaFree(bwd_arr); cudaFree(c0); cudaFree(c1); cudaFree(multi); cudaFree(radj);     // cudaFree(nullptr) is a no-op
            return fail(MGB_ERR_CUDA, std::string("cudaMalloc(radj): ") + cudaGetErrorString(e));
        }
        cudaMemset(bwd_arr, 0, 4); cudaMemset(c0, 0, 1); cudaMemset(c1, 0, 1); cudaMemset(multi, 0, 1);
        cudaMemset(radj, 0, sizeof(uint2));
        // k-mer hash index (index.cuh kh_*): DNA block layout, k <= 31 (62-bit keys). The k-mer of every edge falls out
        // of the gather rounds below; 12 bytes per slot at a load factor of 0.7. Skipped (the seeding kernel then looks
        // k-mers up through the suffix-range table and tighten_range) if the memory is not there or MGB_NO_KMER_HASH is set.
        unsigned long long *kmer = nullptr, *kh_keys = nullptr; uint32_t *kh_vals = nullptr;
        const uint64_t kh_slots = (((uint64_t)((double)(n + 1) / 0.7) + 64) + 3) & ~3ull;     // whole buckets of 4
        if (!idx->view.wide && k >= 3 && k <= 31 && !std::getenv("MGB_NO_KMER_HASH")) {
            size_t free_b = 0, total_b = 0;
            cudaMemGetInfo(&free_b, &total_b);
            if ((double)free_b > 1.2 * (8.0 * (n + 1) + 12.0 * kh_slots) + 16e9
                    && cudaMalloc((void**)&kmer, (n + 1) * 8) == cudaSuccess) {
                if (cudaMalloc((void**)&kh_keys, kh_slots * 8) != cudaSuccess
                        || cudaMalloc((void**)&kh_vals, kh_slots * 4) != cudaSuccess) {
                    cudaGetLastError();
                    cudaFree(kmer); cudaFree(kh_keys); cudaFree(kh_vals);
                    kmer = nullptr; kh_keys = nullptr; kh_vals = nullptr;
                } else {
                    cudaMemset(kmer, 0xFF, 8);                  // position 0: no k-mer
                    cudaMemset(kh_keys, 0, kh_slots * 8);
                }
            } else cudaGetLastError();
        }
        RadjArgs ra { idx->view, bwd_arr, c0, c1, multi, radj, n, kmer };
        const unsigned grid = (unsigned)idx->num_sms * 16;
        e = idx->view.wide ? kern_any::launch_radj_bwd(grid, ra) : kern_dna::launch_radj_bwd(grid, ra);
        for (uint32_t r = 0; r + 2 < k; ++r) {          // k - 2 bwd steps
            kern_dna::k_radj_gather<<<grid, 256>>>(ra, 2 * ((int)k - 3 - (int)r));
            std::swap(ra.c_cur, ra.c_nxt);
        }
        kern_dna::k_radj_pack<<<grid, 256>>>(ra, radj_multi_shift(idx->view));
        if (kmer) {
            kern_dna::k_kmer_insert<<<grid, 256>>>(kmer, n, kh_keys, kh_vals, kh_slots);
            IndexView hv = idx->view;
            hv.kh_keys = kh_keys; hv.kh_vals = kh_vals; hv.kh_slots = kh_slots;
            kern_dna::k_adj_rc<<<grid, 256>>>(hv, const_cast<uint2*>(hv.adj), kmer);
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        cudaFree(bwd_arr); cudaFree(c0); cudaFree(c1); cudaFree(multi);
        if (e != cudaSuccess) {
            cudaFree(kmer); cudaFree(radj); cudaFree(kh_keys); cudaFree(kh_vals);
            return fail(MGB_ERR_CUDA, std::string("radj / k-mer hash build: ") + cudaGetErrorString(e));
        }
        idx->keep(radj, (n + 1) * sizeof(uint2));
        idx->view.radj = radj;
        if (kh_keys) {
            idx->keep(kh_keys, kh_slots * 8); idx->keep(kh_vals, kh_slots * 4);
            idx->view.kh_keys = kh_keys; idx->view.kh_vals = kh_vals; idx->view.kh_slots = kh_slots;
            rc = build_path_layout(idx.get(), kmer);
        }
        cudaFree(kmer);
        if (rc) return rc;
    }
#endif
    *out = idx.release();
    return MGB_OK;
}

int mgb_index_set_mode(mgb_index_t *index, int mode) {
    if (!index) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (mode < 0 || mode > 2) return fail(MGB_ERR_INVALID_ARGUMENT, "mode must be 0 (BASIC), 1 (CANONICAL) or 2 (PRIMARY)");
    if (mode != 0 && !index->at.has_complement)
        return fail(MGB_ERR_BAD_CONFIG, "CANONICAL / PRIMARY modes need a DNA graph");
    if (mode != 0 && index->view.wide)
        return fail(MGB_ERR_UNSUPPORTED, "CANONICAL / PRIMARY modes are served on the DNA block layout only");
    if (mode == 2 && !index->view.rcs) {
        // PRIMARY graph: the rc-strand jump tables of the CanonicalDBG semantics (IndexView::rcs / rcp / palin)
        if (index->view.k > (uint32_t)kMaxPrimaryK)
            return fail(MGB_ERR_UNSUPPORTED, "PRIMARY graphs: k above 128 is not supported");
        const uint64_t n = index->view.n;
        const bool even_k = index->view.k % 2 == 0;
        const size_t pal_words = (n >> 5) + 1;
#if defined(MGB_HOST_EMU)
        index->rc_host.assign(2 * (n + 1) + (even_k ? pal_words : 0), 0);
        RcArgs ra { index->view, index->rc_host.data(), index->rc_host.data() + (n + 1),
                    even_k ? index->rc_host.data() + 2 * (n + 1) : nullptr, n };
        for (uint64_t e = 1; e <= n; ++e) rc_tables_item(ra, e);
#else
        CUDA_TRY(cudaSetDevice(index->device));
        uint32_t *buf = nullptr;
        const size_t words = 2 * (n + 1) + (even_k ? pal_words : 0);
        cudaError_t e = cudaMalloc((void**)&buf, words * 4);
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("cudaMalloc(rc tables): ") + cudaGetErrorString(e));
        cudaMemset(buf, 0, words * 4);
        RcArgs ra { index->view, buf, buf + (n + 1), even_k ? buf + 2 * (n + 1) : nullptr, n };
        kern_dna::k_rc_tables<<<(unsigned)index->num_sms * 16, 128>>>(ra);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { cudaFree(buf); return fail(MGB_ERR_CUDA, std::string("rc tables: ") + cudaGetErrorString(e)); }
        index->keep(buf, words * 4);
#endif
        index->view.rcs = ra.rcs; index->view.rcp = ra.rcp; index->view.palin = ra.palin;
    }
    index->view.mode = (uint32_t)mode;
    return MGB_OK;
}

void mgb_index_destroy(mgb_index_t *index) { delete index; }

int mgb_index_replicate(const mgb_index_t *src, int device, mgb_index_t **out) {
    if (!src || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    std::unique_ptr<mgb_index> idx(new mgb_index());
    idx->alphabet = src->alphabet;
    idx->at = src->at;
#if defined(MGB_HOST_EMU)
    if (device != 0) return fail(MGB_ERR_INVALID_ARGUMENT, "bad device ordinal");
    // the emulated index has none of the tables that depend on free memory; its arrays are host vectors
    idx->host = src->host;
    idx->radj_host = src->radj_host;
    idx->rc_host = src->rc_host;
    idx->device_bytes = src->device_bytes;
    const IndexView &s = src->view;
    IndexView v = idx->host.view();
    v.sfx_len = s.sfx_len;
    v.mode = s.mode;
    v.radj = idx->radj_host.data();
    auto rc_of = [&](const uint32_t *p) { return p ? idx->rc_host.data() + (p - src->rc_host.data()) : nullptr; };
    v.rcs = rc_of(s.rcs); v.rcp = rc_of(s.rcp); v.palin = rc_of(s.palin);
    idx->view = v;
#else
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(MGB_ERR_NO_DEVICE, "no CUDA device available (the kernels have no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(MGB_ERR_INVALID_ARGUMENT, "bad device ordinal");
    CUDA_TRY(cudaSetDevice(device));
    idx->device = device;
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    idx->num_sms = prop.multiProcessorCount;
    device_setup(device);
    // the source's arrays the view points into (not the host-built suffix level the deeper ones replaced), and the
    // table each one holds
    IndexView v = src->view;
    struct Copy { const mgb_index::DevArray *from; const char *name; Opt opt; void *to; };
    std::vector<Copy> copies;
    const char *stray = nullptr;
    each_table(v, [&](auto &field, const char *name, Opt opt) {
        if (!field) return;
        const char *p = reinterpret_cast<const char*>(field);
        for (const mgb_index::DevArray &b : src->bufs) {
            if (p < (const char*)b.p || p >= (const char*)b.p + b.bytes) continue;
            for (const Copy &c : copies) if (c.from == &b) return;
            copies.push_back({ &b, name, opt, nullptr });
            return;
        }
        stray = name;
    });
    if (stray) return fail(MGB_ERR_INVALID_ARGUMENT, std::string("table ") + stray + " is not an array of the index");
    struct Undo {                // frees the copies unless they went to the replica
        std::vector<Copy> &c; cudaStream_t s = nullptr; bool done = false;
        ~Undo() {
            if (s) cudaStreamDestroy(s);
            if (!done) for (Copy &x : c) cudaFree(x.to);
        }
    } undo { copies };
    // allocates the arrays of one table class; the first that fails, else nullptr (and none of the class is kept)
    auto alloc = [&](Opt opt) -> const Copy* {
        for (Copy &c : copies) {
            if (c.opt != opt || cudaMalloc(&c.to, c.from->bytes) == cudaSuccess) continue;
            cudaGetLastError();
            for (Copy &d : copies) if (d.opt == opt) { cudaFree(d.to); d.to = nullptr; }
            return &c;
        }
        return nullptr;
    };
    if (const Copy *c = alloc(Opt::none)) return fail(MGB_ERR_CUDA, std::string("cudaMalloc(") + c->name + ") failed");
    // The optional tables follow mgb_index_create's rules on this device, in its order, each checked with the free
    // memory the build would see there: less the temporaries the build holds at that point (7 bytes per edge for the
    // radj rounds, 8 for the per-edge k-mers, 12 for the path layout's pred and jump arrays).
    const double n1 = (double)(v.n + 1);
    size_t free_b = 0, total_b = 0;
    auto free_now = [&]() { cudaMemGetInfo(&free_b, &total_b); return (double)free_b; };
    bool hash = v.kh_slots && !std::getenv("MGB_NO_KMER_HASH")
                && free_now() - 7 * n1 > 1.2 * (8.0 * n1 + 12.0 * v.kh_slots) + 16e9 && !alloc(Opt::hash);
    bool path = hash && v.pl_n && !std::getenv("MGB_NO_PATH_INDEX");
    if (path) {
        const double f = free_now() - 8 * n1, pl = (double)v.pl_n;
        path = f >= 1.2 * 16.5 * n1 && f - 8.6 * n1 >= 16e9
               && f - 12 * n1 >= 1.2 * (pl * 4 + pl / 4 + 2 * (pl / 8)) && !alloc(Opt::path);
    }
    if (path) {
        const char *no = std::getenv("MGB_TEST_NO_LAYOUT_WORDS");
        const double keep = std::max(16e9, 0.5 * (double)total_b), word_bytes = (double)(v.pl_n / 32 * 16);
        double left = free_now() - 8 * n1;
        if (v.pl_word && (!no || !std::strcmp(no, "kh_pos")) && left - word_bytes >= keep && !alloc(Opt::pl_word))
            left -= word_bytes;
        if (v.kh_pos && (!no || !std::strcmp(no, "pl_word")) && left - 4.0 * v.kh_slots >= keep) alloc(Opt::kh_pos);
    }
    CUDA_TRY(cudaStreamCreateWithFlags(&undo.s, cudaStreamNonBlocking));
    for (const Copy &c : copies) {
        if (!c.to) continue;
        const cudaError_t e = device == src->device
            ? cudaMemcpyAsync(c.to, c.from->p, c.from->bytes, cudaMemcpyDeviceToDevice, undo.s)
            : cudaMemcpyPeerAsync(c.to, device, c.from->p, src->device, c.from->bytes, undo.s);
        if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("copy of ") + c.name + ": " + cudaGetErrorString(e));
    }
    // re-point the view; a table left out is absent, as in an index built without it
    each_table(v, [&](auto &field, const char *, Opt) {
        using P = std::remove_reference_t<decltype(field)>;
        const char *p = reinterpret_cast<const char*>(field);
        for (const Copy &c : copies) {
            const char *b = (const char*)c.from->p;
            if (p && p >= b && p < b + c.from->bytes) { field = c.to ? reinterpret_cast<P>((char*)c.to + (p - b)) : nullptr; return; }
        }
    });
    if (!hash) v.kh_slots = 0;
    if (!path) v.pl_n = 0;
    if (src->view.kh_slots && !hash)         // y[16:21) is defined only with the hash index
        kern_dna::k_adj_clear_rc<<<(unsigned)idx->num_sms * 16, 256, 0, undo.s>>>(const_cast<uint2*>(v.adj), v.n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(undo.s);
    if (e != cudaSuccess) return fail(MGB_ERR_CUDA, std::string("index replica copy: ") + cudaGetErrorString(e));
    for (const Copy &c : copies) if (c.to) idx->keep(c.to, c.from->bytes);
    undo.done = true;
    idx->view = v;
#endif
    *out = idx.release();
    return MGB_OK;
}

uint64_t mgb_index_num_edges(const mgb_index_t *index) { return index->view.n; }
uint64_t mgb_index_device_bytes(const mgb_index_t *index) { return index->device_bytes; }
uint32_t mgb_index_k(const mgb_index_t *index) { return index->view.k; }

void mgb_config_init(mgb_config_t *c) {
    std::memset(c, 0, sizeof(*c));
    c->num_alternative_paths = 1;
    c->max_num_seeds_per_locus = UINT64_MAX;
    c->min_cell_score = INT32_MIN + 100;
    c->min_path_score = 0;
    c->xdrop = INT32_MAX;
    c->max_nodes_per_seq_char = 1.7976931348623157e308;
    c->max_ram_per_alignment = 1.7976931348623157e308;
    c->gap_opening_penalty = -5; c->gap_extension_penalty = -2;
    c->forward_and_reverse_complement = 1; c->global_xdrop = 1; c->allow_left_trim = 1;
    // dna_scoring_matrix(2, -1, -2) (aligner_config.cpp:164-183)
    std::memset(c->score_matrix, -2, sizeof(c->score_matrix));
    c->score_matrix['A']['G'] = c->score_matrix['G']['A'] = -1;
    c->score_matrix['C']['T'] = c->score_matrix['T']['C'] = -1;
    for (const char *p = "ACGT"; *p; ++p) c->score_matrix[(int)*p][(int)*p] = 2;
}

void mgb_config_init_cli(mgb_config_t *c, uint32_t k, int alphabet) {
    mgb_config_init(c);
    c->min_seed_length = k < 19 ? k : 19;           // cli/align.cpp:42-43
    c->max_seed_length = UINT64_MAX;
    c->max_num_seeds_per_locus = 1000;
    c->xdrop = 27;
    c->min_exact_match = 0.7;
    c->max_nodes_per_seq_char = 5.0;
    c->max_ram_per_alignment = 200;
    c->rel_score_cutoff = 0.95;
    c->gap_opening_penalty = -6; c->gap_extension_penalty = -2;
    c->left_end_bonus = 5; c->right_end_bonus = 5;
    std::memset(c->score_matrix, -3, sizeof(c->score_matrix));
    for (const char *p = "ACGT"; *p; ++p) c->score_matrix[(int)*p][(int)*p] = 2;
    if (alphabet == MGB_ALPHABET_PROTEIN) {              // set_scoring_matrix (aligner_config.cpp:128-163)
        blosum62_matrix(c->score_matrix);
        c->forward_and_reverse_complement = 0;           // no reverse complement (dbg_aligner.cpp:224-229)
    }
}

} // extern "C"

namespace {

struct Batch {                 // device-resident read batch
    uint32_t n_reads = 0; uint64_t total_chars = 0, total_kmers = 0; uint32_t L_max = 0;
    char *seqs = nullptr, *qf = nullptr, *qr = nullptr; uint8_t *cf = nullptr, *cr = nullptr;
    uint64_t *offsets = nullptr, *koff = nullptr, *nodes_f = nullptr, *nodes_r = nullptr;
};

// dev_seqs: seqs is device memory (the file route's parsed reads, 16-byte aligned, 64 bytes of slack after the last
// read) and is read in place
int upload_batch(const mgb_index_t *index, const char *seqs, const uint64_t *offsets, uint32_t n_reads,
                 bool need_rc_nodes, Stream &st, DevBufs &bufs, Batch *b, std::vector<uint64_t> *koff_host,
                 mgb_stats_t *stats, bool dev_seqs = false) {
    const uint32_t k = index->view.k;
    b->n_reads = n_reads;
    b->total_chars = offsets[n_reads];
    koff_host->assign(n_reads + 1, 0);
    for (uint32_t r = 0; r < n_reads; ++r) {
        if (offsets[r + 1] < offsets[r]) return fail(MGB_ERR_INVALID_ARGUMENT, "offsets must be non-decreasing");
        uint64_t L = offsets[r + 1] - offsets[r];
        if (L > 0x3fffffffull) return fail(MGB_ERR_INVALID_ARGUMENT, "read too long");
        if (L > b->L_max) b->L_max = (uint32_t)L;
        (*koff_host)[r + 1] = (*koff_host)[r] + (L >= k ? L - k + 1 : 0);
    }
    b->total_kmers = (*koff_host)[n_reads];
    int rc;
    const size_t pad = 64;
    if (dev_seqs) b->seqs = const_cast<char*>(seqs);
    else if ((rc = bufs.alloc(&b->seqs, b->total_chars + pad))) return rc;
    if ((rc = bufs.alloc(&b->qf, b->total_chars + pad))) return rc;
    if ((rc = bufs.alloc(&b->qr, b->total_chars + pad))) return rc;
    if ((rc = bufs.alloc(&b->cf, b->total_chars + pad))) return rc;
    if ((rc = bufs.alloc(&b->cr, b->total_chars + pad))) return rc;
    if ((rc = bufs.alloc(&b->offsets, (size_t)n_reads + 1))) return rc;
    if ((rc = bufs.alloc(&b->koff, (size_t)n_reads + 1))) return rc;
    if ((rc = bufs.alloc(&b->nodes_f, b->total_kmers + 1))) return rc;
    if (need_rc_nodes && (rc = bufs.alloc(&b->nodes_r, b->total_kmers + 1))) return rc;
    if (!dev_seqs && (rc = h2d(b->seqs, seqs, b->total_chars, st))) return rc;
    if ((rc = h2d(b->offsets, offsets, ((size_t)n_reads + 1) * 8, st))) return rc;
    if ((rc = h2d(b->koff, koff_host->data(), ((size_t)n_reads + 1) * 8, st))) return rc;
    stats->h2d_bytes += (dev_seqs ? 0 : b->total_chars) + 2 * ((size_t)n_reads + 1) * 8;
    return 0;
}

int launch_prepare(const mgb_index_t *index, const Batch &b, Stream &st, int num_sms) {
    PrepArgs a { b.seqs, b.offsets, b.n_reads, b.qf, b.qr, b.cf, b.cr, {0} };
    std::memcpy(a.code_of, index->at.code_of, sizeof(a.code_of));
#if defined(MGB_HOST_EMU)
    (void)st; (void)num_sms;
    for (uint32_t r = 0; r < b.n_reads; ++r) prepare_read(a, r);
#else
    if (!b.n_reads) return 0;
    const unsigned blocks = (unsigned)kern_dna::read_path_grid(std::min<uint64_t>((b.n_reads + 7) / 8, (uint64_t)num_sms * 8));
    kern_dna::log_launch("k_prepare", blocks, 256, (uint64_t)blocks * 8, b.n_reads);     // a warp per read
    kern_dna::k_prepare<<<blocks, 256, 0, st.s>>>(a);
    CUDA_TRY(cudaGetLastError());
#endif
    return 0;
}

// summary: SeedArgs::summary (k_seed_hash writes it; nullptr on graphs without the k-mer hash index); list / n_list:
// SeedArgs::list (k_seed_hash only)
int launch_seed(const mgb_index_t *index, const Batch &b, uint32_t n_strands, Stream &st, DevBufs &bufs,
                uint8_t *summary, uint64_t *n_launches = nullptr, const uint32_t *list = nullptr,
                const unsigned int *n_list = nullptr) {
    SeedArgs a { index->view, b.cf, b.cr, b.offsets, b.koff, b.nodes_f, b.nodes_r, b.n_reads, n_strands, 0, nullptr, nullptr,
                 summary, list, n_list, 0 };
    // MGB_TEST_SEED_MODE=walk|wide: test knob, k_seed_hash's walk or short-list mode whatever the list's length
    if (const char *e = std::getenv("MGB_TEST_SEED_MODE")) a.seed_mode = !std::strcmp(e, "walk") ? 1 : !std::strcmp(e, "wide") ? 2 : 0;
    uint64_t items = (uint64_t)b.n_reads * n_strands;
    // first pass (k_premap): rules out the k-mers the suffix-range table has no node for; the node arrays
    // are zero-filled, so the second pass only visits what is left
    const bool premap = index->view.sfx_len && index->view.sfx_len <= index->view.k - 1 && b.total_kmers
                        && !index->view.kh_slots               // (the k-mer hash index answers every k-mer with one load)
                        && !std::getenv("MGB_TEST_NOPREMAP");
    if (premap) {
        const size_t words = (size_t)(b.total_kmers >> 5) + b.n_reads + 2;
        int rc;
        if ((rc = bufs.alloc(&a.hint_f, words))) return rc;
        if (n_strands > 1 && (rc = bufs.alloc(&a.hint_r, words))) return rc;
        a.hinted = 1;
    }
    if (n_launches) *n_launches += premap ? 2 : 1;
#if defined(MGB_HOST_EMU)
    (void)st;
    if (premap)
        for (uint64_t it = 0; it < items; ++it) premap_item(a, (uint32_t)(it / n_strands), (uint32_t)(it % n_strands));
    if (list) {
        for (uint32_t t = 0; t < *n_list; ++t)
            for (uint32_t s = 0; s < n_strands; ++s) seed_item(a, (uint64_t)list[t] * n_strands + s);
    } else {
        for (uint64_t it = 0; it < items; ++it) seed_item(a, it);
    }
#else
    if (!items) return 0;
    if (premap) {
        const uint64_t pb = std::min<uint64_t>((items + 7) / 8, (uint64_t)index->num_sms * 16);
        CUDA_TRY(index->view.wide ? kern_any::launch_premap((unsigned)pb, st.s, a) : kern_dna::launch_premap((unsigned)pb, st.s, a));
    }
    if (index->view.kh_slots) {
        CUDA_TRY(kern_dna::launch_seed_hash(index->num_sms, st.s, a));
        return 0;
    }
    // one strand per lane, 128 strands per block; enough blocks to fill the machine, grid-stride beyond that
    uint64_t blocks = std::min<uint64_t>((items + 127) / 128, (uint64_t)index->num_sms * 16);
    CUDA_TRY(index->view.wide ? kern_any::launch_seed((unsigned)blocks, st.s, a) : kern_dna::launch_seed((unsigned)blocks, st.s, a));
#endif
    return 0;
}

// whole-read exact answers (kernels.cuh ExactArgs) for the reads of a.list; the others are appended to a.rest
int launch_exact_reads(const mgb_index_t *index, const ExactArgs &a, Stream &st) {
#if defined(MGB_HOST_EMU)
    (void)index; (void)st;
    const uint32_t n_list = a.n_list_dev ? *a.n_list_dev : a.n_list;
    for (uint32_t t = 0; t < n_list; ++t) {
        const uint32_t r = a.list[t];
        uint64_t b; int L; score_t score;
        const int s = exact_read_strand(a, a.diag, r, &b, &L, &score);
        if (s < 0) { a.rest[(*a.n_rest)++] = r; continue; }
        exact_read_write(a, r, b, L, s, score, *a.heap_used, 0, 1);
        *a.heap_used += exact_read_bytes(a, L);
    }
#else
    if (a.n_list) CUDA_TRY(kern_dna::launch_exact_reads(index->num_sms, st.s, a));
#endif
    return 0;
}

// whole-read exact answers from the raw reads (kernels.cuh PrepExactArgs), in place of launch_prepare; the reads left
// over are prepared and listed in a.list
int launch_prepare_exact(const mgb_index_t *index, const PrepExactArgs &a, Stream &st) {
#if defined(MGB_HOST_EMU)
    (void)index; (void)st;
    for (uint32_t r = 0; r < a.prep.n_reads; ++r) {
        uint64_t b; int L; uint32_t p; score_t score;
        PrepTimer tm;
        b = a.prep.offsets[r]; L = (int)(a.prep.offsets[r + 1] - b);
        const uint8_t *raw = reinterpret_cast<const uint8_t*>(a.prep.seqs) + b;
        int s = exact_path_strand(a, raw, L, &p, &score, tm);
        const uint64_t off = *a.ex.heap_used;
        if (s >= 0) {
            *a.ex.heap_used += exact_read_bytes(a.ex, L);
            if (off + exact_read_bytes(a.ex, L) > a.ex.heap_cap) s = -1;
        }
        if (s >= 0) {
            exact_path_hdr(a.ex, r, L, off);
            exact_path_write(a, raw, L, s, p, score, off, 0, 1);
            continue;
        }
        a.list[(*a.n_list)++] = r;
        prepare_read(a.prep, r);
    }
#else
    if (a.prep.n_reads) CUDA_TRY(kern_dna::launch_prepare_exact(index->num_sms, st.s, a));
#endif
    return 0;
}

// ---------------------------------------------------------------------------------------
// text route (mgb_align_batch_text): the TSV lines or JSON records of a piece's reads, rendered from the records the
// align passes left in their heaps (format_core.cuh). Independent of the index layout and the graph mode, so compiled
// in this translation unit only.
// ---------------------------------------------------------------------------------------
struct TextArgs {
    const char *seqs; const uint64_t *offsets;       // the piece's raw reads
    const char *names; const uint64_t *name_off;     // and their headers
    const ReadHdr *hdr;                              // per read: n_aln and heap_off of the pass that answered it
    const uint8_t *pass;                             // ... and that pass
    const char *heap[kMaxPasses];                    // the output heap of every pass (PassState::heap)
    uint32_t n_reads, k, json, result_nodes;
    int32_t min_path_score;
    uint64_t *off;         // k_text_size: bytes of each read's text; after the scan its offset, off[n_reads] = total
    char *out; uint64_t lo, hi;                      // k_text_write: bytes [lo, hi) of the text, at out[0, hi - lo)
};

// the text of read r (its line, or one JSON record per alignment) into sink s
template <class S> MGB_HD void text_read(const TextArgs &a, uint32_t r, S &s) {
    const uint64_t b = a.offsets[r], nb = a.name_off[r];
    const TextRead rd { a.seqs + b, (uint32_t)(a.offsets[r + 1] - b), a.names + nb, (uint32_t)(a.name_off[r + 1] - nb) };
    const uint32_t n_aln = a.hdr[r].n_aln;
    const char *p = n_aln ? a.heap[a.pass[r]] + a.hdr[r].heap_off : nullptr;
    if (!a.json) tsv_head(s, rd);
    for (uint32_t i = 0; i < n_aln; ++i) {
        RecView v;
        p = rec_next(p, a.result_nodes != 0, &v);
        const OutAln &o = v.o;
        const TextAln t { o.orientation, o.score, o.offset, o.query_begin, o.query_len, o.n_nodes, o.seq_len, o.n_cigar,
                          v.nodes, v.cigar, v.seq };
        if (a.json) json_aln(s, rd, t, i > 0, a.k); else tsv_aln(s, t);
    }
    if (!a.json) {
        if (!n_aln) tsv_unaligned(s, a.min_path_score);
        s.put('\n');
    } else if (!n_aln) {
        json_unaligned(s, rd);
    }
}

// reads [*r0, *r1) are those whose text meets bytes [lo, hi) (off: exclusive offsets, every read's text >= 1 byte)
MGB_HOSTDEV void text_window(const uint64_t *off, uint32_t n, uint64_t lo, uint64_t hi, uint32_t *r0, uint32_t *r1) {
    uint32_t a = 0, b = n;                 // first read whose text ends after lo
    while (a < b) { const uint32_t m = (a + b) / 2; if (off[m + 1] > lo) b = m; else a = m + 1; }
    *r0 = a;
    b = n;                                 // first read whose text starts at or after hi
    while (a < b) { const uint32_t m = (a + b) / 2; if (off[m] >= hi) b = m; else a = m + 1; }
    *r1 = a;
}

#if !defined(MGB_HOST_EMU)
// one warp per read
__global__ void __launch_bounds__(256) k_text_size(const __grid_constant__ TextArgs a) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp, nw = (gridDim.x * blockDim.x) / kWarp;
    for (uint32_t r = warp; r < a.n_reads; r += nw) {
        CountSink c;
        text_read(a, r, c);
        if (wlane() == 0) a.off[r] = c.pos;
    }
}

// exclusive scan of off[0, n) in place, total at off[n]: one block, a contiguous segment per thread
__global__ void __launch_bounds__(1024) k_text_scan(uint64_t *off, uint32_t n) {
    __shared__ uint64_t part[1024];
    const uint32_t t = threadIdx.x, seg = (n + 1023) / 1024;
    const uint64_t b = (uint64_t)t * seg < n ? (uint64_t)t * seg : n, e = b + seg < n ? b + seg : n;
    uint64_t sum = 0;
    for (uint64_t i = b; i < e; ++i) sum += off[i];
    part[t] = sum;
    __syncthreads();
    for (uint32_t d = 1; d < 1024; d <<= 1) {
        const uint64_t v = t >= d ? part[t - d] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    uint64_t run = part[t] - sum;
    for (uint64_t i = b; i < e; ++i) { const uint64_t v = off[i]; off[i] = run; run += v; }
    if (t == 1023) off[n] = part[1023];
}

// one warp per read of the window [a.lo, a.hi)
__global__ void __launch_bounds__(256) k_text_write(const __grid_constant__ TextArgs a) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / kWarp, nw = (gridDim.x * blockDim.x) / kWarp;
    uint32_t r0, r1;
    text_window(a.off, a.n_reads, a.lo, a.hi, &r0, &r1);
    for (uint32_t r = r0 + warp; r < r1; r += nw) {
        WriteSink w { a.out, a.lo, a.hi, a.off[r] };
        text_read(a, r, w);
    }
}
#endif

// Renders the text of a piece's reads into `host` (pinned; acquired here, *bytes long): the size pass, the scan, 8 bytes
// read back, then windows of at most `cap` bytes rendered and downloaded one after the other.
int render_text(const mgb_index_t *index, TextArgs &ta, DevBufs &tb, Stream &st, HostBuf *host, uint64_t *bytes,
                mgb_stats_t *stats) {
    *bytes = 0;
    int rc;
    if ((rc = tb.alloc(&ta.off, (size_t)ta.n_reads + 1))) return rc;
    uint64_t total = 0;
#if defined(MGB_HOST_EMU)
    (void)index;
    for (uint32_t r = 0; r < ta.n_reads; ++r) { CountSink c; text_read(ta, r, c); ta.off[r] = c.pos; }
    for (uint32_t r = 0; r < ta.n_reads; ++r) { const uint64_t v = ta.off[r]; ta.off[r] = total; total += v; }
    ta.off[ta.n_reads] = total;
#else
    {
        const unsigned grid = (unsigned)kern_dna::read_path_grid(std::min<uint64_t>((ta.n_reads + 7) / 8, (uint64_t)index->num_sms * 16));
        kern_dna::log_launch("k_text_size", grid, 256, (uint64_t)grid * 8, ta.n_reads);     // a warp per read
        k_text_size<<<grid, 256, 0, st.s>>>(ta);
        k_text_scan<<<1, 1024, 0, st.s>>>(ta.off, ta.n_reads);
        CUDA_TRY(cudaGetLastError());
    }
#endif
    if ((rc = d2h(&total, ta.off + ta.n_reads, 8, st)) || (rc = sync(st))) return rc;
    stats->kernel_launches += 2;
    stats->d2h_bytes += 8;
    *host = hostbuf_acquire(total);
    if (!host->p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
    *bytes = total;
    // device bytes of one window (MGB_TEST_TEXT_CAP: test knob, so that small inputs take many windows)
    uint64_t cap = 256ull << 20;
    if (const char *e = std::getenv("MGB_TEST_TEXT_CAP")) cap = std::max<long long>(1, std::atoll(e));
    cap = std::min<uint64_t>(cap, std::max<uint64_t>(total, 1));
    if ((rc = tb.alloc(&ta.out, cap))) return rc;
    for (uint64_t lo = 0; lo < total; lo += cap) {
        ta.lo = lo; ta.hi = std::min(total, lo + cap);
#if defined(MGB_HOST_EMU)
        uint32_t r0, r1;
        text_window(ta.off, ta.n_reads, ta.lo, ta.hi, &r0, &r1);
        for (uint32_t r = r0; r < r1; ++r) { WriteSink w { ta.out, ta.lo, ta.hi, ta.off[r] }; text_read(ta, r, w); }
#else
        const unsigned grid = (unsigned)kern_dna::read_path_grid(std::min<uint64_t>((ta.n_reads + 7) / 8, (uint64_t)index->num_sms * 16));
        kern_dna::log_launch("k_text_write", grid, 256, (uint64_t)grid * 8, -1);       // a warp per read of the window
        k_text_write<<<grid, 256, 0, st.s>>>(ta);
        CUDA_TRY(cudaGetLastError());
#endif
        if ((rc = d2h(host->p + lo, ta.out, ta.hi - ta.lo, st))) return rc;
        stats->kernel_launches += 1;
    }
    if ((rc = sync(st))) return rc;
    stats->d2h_bytes += total;
    return 0;
}

// ---------------------------------------------------------------------------------------
// file route (mgb_align_fastx_text): one chunk of FASTA/FASTQ bytes parsed into reads and headers on the device
// (fastx_core.cuh). The parsed arrays stay in the workspace of the call; only their offsets come back.
// ---------------------------------------------------------------------------------------
struct FastxDev {
    bool refused = false;                      // the chunk has neither parallel form: the host restatement parses it
    char *seqs = nullptr, *names = nullptr;    // device arrays
    std::vector<uint64_t> offsets, name_offsets;
    uint64_t consumed = 0;
};

// exclusive scan of off[0, n) in place, total at off[n] (fastx_core.cuh k_fastx_scan_up / _down; the tile sums, a
// thousandth of the elements, by k_text_scan's one block)
int scan_u64(uint64_t *off, uint32_t n, Stream &st, DevBufs &bufs) {
#if defined(MGB_HOST_EMU)
    (void)st; (void)bufs;
    uint64_t t = 0;
    for (uint32_t i = 0; i < n; ++i) { const uint64_t v = off[i]; off[i] = t; t += v; }
    off[n] = t;
#else
    const uint32_t n_tiles = (n + kFastxScanTile - 1) / kFastxScanTile;
    uint64_t *tile_sum = nullptr;
    if (int rc = bufs.alloc(&tile_sum, (size_t)n_tiles + 1)) return rc;
    if (n_tiles) k_fastx_scan_up<<<n_tiles, 256, 0, st.s>>>(off, n, tile_sum);
    k_text_scan<<<1, 1024, 0, st.s>>>(tile_sum, n_tiles);
    k_fastx_scan_down<<<n_tiles ? n_tiles : 1, 256, 0, st.s>>>(off, n, tile_sum, n_tiles);
    CUDA_TRY(cudaGetLastError());
#endif
    return 0;
}

// the chunk's text in device memory: fastx_text_bytes(bytes) bytes, the chunk at the front
inline uint64_t fastx_text_bytes(uint64_t bytes) { return (bytes + kFastxTile - 1) / kFastxTile * kFastxTile + 16; }

// whether the device route takes a chunk of this size and delimiter at all
inline bool fastx_dev_takes(uint64_t bytes, const char *delim) {
    return bytes < 0xffffffffull && (!delim || std::strlen(delim) <= kFastxMaxDelim);
}

// the records of the chunk d_buf[0, bytes) (device memory of fastx_text_bytes(bytes) bytes, last: its last byte)
int fastx_parse_text(const mgb_index_t *index, const uint8_t *d_buf, uint64_t bytes, uint8_t last, bool at_eof,
                     const char *delim, bool fwd_rev, Stream &st, DevBufs &bufs, FastxDev *out, mgb_stats_t *stats) {
    if (!fastx_dev_takes(bytes, delim)) { out->refused = true; return 0; }
    int rc;
    FastxArgs a;
    std::memset(&a, 0, sizeof(a));
    a.n = (uint32_t)bytes; a.at_eof = at_eof; a.fwd_rev = fwd_rev;
    a.n_tiles = (uint32_t)((bytes + kFastxTile - 1) / kFastxTile);
    if (delim) { a.has_delim = 1; a.dlen = (uint32_t)std::strlen(delim); std::memcpy(a.delim, delim, a.dlen); }
    if ((rc = bufs.alloc(&a.tile_nl, (size_t)a.n_tiles + 1))) return rc;
    if ((rc = bufs.alloc(&a.sum, 1))) return rc;
    if ((rc = dev_zero(a.sum, sizeof(FastxSummary), st))) return rc;
    a.buf = d_buf;
    [[maybe_unused]] const unsigned tiles_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(a.n_tiles, (uint64_t)index->num_sms * 8));
    // line ends
    uint64_t n_nl = 0;
#if defined(MGB_HOST_EMU)
    for (uint32_t t = 0; t < a.n_tiles; ++t) {
        uint64_t c = 0;
        for (uint32_t i = t * kFastxTile; i < a.n && i < (t + 1) * kFastxTile; ++i) c += a.buf[i] == '\n';
        a.tile_nl[t] = c;
    }
#else
    if (a.n_tiles) {
        k_fastx_count<<<tiles_grid, 256, 0, st.s>>>(a);
        CUDA_TRY(cudaGetLastError());
    }
#endif
    if ((rc = scan_u64(a.tile_nl, a.n_tiles, st, bufs))) return rc;
    if ((rc = d2h(&n_nl, a.tile_nl + a.n_tiles, 8, st)) || (rc = sync(st))) return rc;
    a.n_nl = (uint32_t)n_nl;
    a.n_lines = a.n_nl + (bytes && last != '\n' ? 1 : 0);
    if ((rc = bufs.alloc(&a.nl, (size_t)a.n_nl + 1))) return rc;
    [[maybe_unused]] const unsigned lines_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)a.n_lines + 255) / 256,
                                                                                   (uint64_t)index->num_sms * 8));
    FastxSummary sum;
    std::memset(&sum, 0, sizeof(sum));
#if defined(MGB_HOST_EMU)
    {
        uint64_t o = 0;
        for (uint32_t i = 0; i < a.n; ++i) if (a.buf[i] == '\n') a.nl[o++] = i;
        a.nl[a.n_nl] = a.n;
        for (uint32_t i = 0; i < a.n_lines; ++i) {
            bool hdr;
            fastx_classify_line(a, i, &sum.flags, &hdr, &sum.q_cut);
            if (hdr) { ++sum.n_hdr; sum.last_hdr = fastx_line_begin(a, i) + 1; }
        }
    }
#else
    if (a.n_tiles) k_fastx_lines<<<tiles_grid, 256, 0, st.s>>>(a);
    else k_fastx_lines<<<1, 32, 0, st.s>>>(a);        // (nl[0] = 0 for an empty chunk)
    if (a.n_lines) k_fastx_classify<<<lines_grid, 256, 0, st.s>>>(a);
    CUDA_TRY(cudaGetLastError());
    if ((rc = d2h(&sum, a.sum, sizeof(sum), st))) return rc;
#endif
    if ((rc = sync(st))) return rc;
    stats->kernel_launches += 6;
    stats->d2h_bytes += 8 + sizeof(sum);
    if ((sum.flags & kFastxFastaBad) && (sum.flags & kFastxFastqBad)) { out->refused = true; return 0; }
    a.fastq = (sum.flags & kFastxFastaBad) != 0;
    uint32_t n_rec;
    if (a.fastq) {
        n_rec = (at_eof ? a.n_lines : a.n_nl) / 4;
        out->consumed = sum.q_cut ? sum.q_cut - 1 : bytes;
    } else {
        n_rec = at_eof ? sum.n_hdr : sum.n_hdr ? sum.n_hdr - 1 : 0;
        out->consumed = at_eof ? bytes : sum.last_hdr ? sum.last_hdr - 1 : 0;
    }
    const uint64_t copies = fwd_rev ? 2 : 1, n_out = copies * n_rec;
    if (n_out > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "more than 2^32 - 1 records in one chunk");
    out->offsets.assign(n_out + 1, 0);
    out->name_offsets.assign(n_out + 1, 0);
    // the packed arrays: at most `copies` times the chunk's bytes (and a delimiter per record), and the slack the read
    // kernels' word loads go past the last read
    if ((rc = bufs.alloc(&out->seqs, copies * bytes + 128))) return rc;
    if ((rc = bufs.alloc(&out->names, copies * (bytes + (uint64_t)n_rec * a.dlen) + 128))) return rc;
    if (!n_rec) return 0;
    a.n_rec = n_rec;
    a.seqs = out->seqs; a.names = out->names;
    if ((rc = bufs.alloc(&a.lh, (size_t)a.n_lines + 1))) return rc;
    if ((rc = bufs.alloc(&a.ls, (size_t)a.n_lines + 1))) return rc;
    if ((rc = bufs.alloc(&a.ln, (size_t)a.n_lines + 1))) return rc;
    if (!a.fastq && (rc = bufs.alloc(&a.rec_line, (size_t)sum.n_hdr + 1))) return rc;
    if ((rc = bufs.alloc(&a.offsets, n_out + 1))) return rc;
    if ((rc = bufs.alloc(&a.name_offsets, n_out + 1))) return rc;
#if defined(MGB_HOST_EMU)
    for (uint32_t i = 0; i < a.n_lines; ++i) fastx_role_line(a, i);
#else
    k_fastx_roles<<<lines_grid, 256, 0, st.s>>>(a);
    CUDA_TRY(cudaGetLastError());
#endif
    if ((rc = scan_u64(a.lh, a.n_lines, st, bufs)) || (rc = scan_u64(a.ls, a.n_lines, st, bufs))
        || (rc = scan_u64(a.ln, a.n_lines, st, bufs)))
        return rc;
#if defined(MGB_HOST_EMU)
    if (!a.fastq) {
        for (uint32_t i = 0; i < a.n_lines; ++i) if (a.lh[i + 1] != a.lh[i]) a.rec_line[a.lh[i]] = i;
        a.rec_line[a.lh[a.n_lines]] = a.n_lines;
    }
    for (uint32_t r = 0; r < n_rec; ++r) fastx_gather_record(a, r);
#else
    if (!a.fastq) k_fastx_records<<<lines_grid, 256, 0, st.s>>>(a);
    {
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)n_rec + 7) / 8, (uint64_t)index->num_sms * 16));
        k_fastx_gather<<<grid, 256, 0, st.s>>>(a);       // a warp per record
    }
    CUDA_TRY(cudaGetLastError());
#endif
    stats->kernel_launches += a.fastq ? 11 : 12;
    if ((rc = d2h(out->offsets.data(), a.offsets, (n_out + 1) * 8, st))) return rc;
    if ((rc = d2h(out->name_offsets.data(), a.name_offsets, (n_out + 1) * 8, st)) || (rc = sync(st))) return rc;
    stats->d2h_bytes += 16 * (n_out + 1);
    return 0;
}

// the chunk buf[0, bytes) (host memory) uploaded and parsed
int fastx_parse_dev(const mgb_index_t *index, const char *buf, uint64_t bytes, bool at_eof, const char *delim,
                    bool fwd_rev, Stream &st, DevBufs &bufs, FastxDev *out, mgb_stats_t *stats) {
    if (!fastx_dev_takes(bytes, delim)) { out->refused = true; return 0; }
    uint8_t *d_buf = nullptr;
    int rc;
    if ((rc = bufs.alloc(&d_buf, fastx_text_bytes(bytes)))) return rc;
    if (bytes && (rc = h2d(d_buf, buf, bytes, st))) return rc;
    stats->h2d_bytes += bytes;
    return fastx_parse_text(index, d_buf, bytes, bytes ? (uint8_t)buf[bytes - 1] : 0, at_eof, delim, fwd_rev, st, bufs,
                            out, stats);
}

// ---------------------------------------------------------------------------------------
// BGZF input (mgb_fastx_stage_bgzf, mgb_bgzf_inflate): the blocks of a compressed buffer listed on the host from their
// headers, and inflated on the device (bgzf_core.cuh) into the text the parser reads
// ---------------------------------------------------------------------------------------
inline uint32_t rd16(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8; }
inline uint32_t rd32(const uint8_t *p) { return rd16(p) | rd16(p + 2) << 16; }

struct BgzfWalk {
    std::vector<BgzfBlock> blocks;
    uint64_t c_end = 0;      // compressed bytes of the blocks
    uint64_t text = 0;       // their text (the sum of ISIZE)
    bool refused = false;    // the member at c_end is not a BGZF block (or is cut off by the end of the input)
    std::vector<uint64_t> member;      // where each block's member starts
};

// The complete BGZF blocks at the start of c[0, n), until their text reaches max_text. A member is a BGZF block when its
// header is ID1 ID2 CM FLG = 31 139 8 4 (FEXTRA only), its extra field holds a BC subfield of SLEN 2 (BSIZE; other
// subfields are skipped) and ISIZE <= 64 KiB. One header per block is read.
void bgzf_walk(const uint8_t *c, uint64_t n, bool c_eof, uint64_t max_text, BgzfWalk *w) {
    uint64_t at = 0;
    while (w->text < max_text && at < n) {
        const uint8_t *h = c + at;
        const uint64_t left = n - at;
        if (left < 12) { w->refused = c_eof; break; }
        if (h[0] != 31 || h[1] != 139 || h[2] != 8 || h[3] != 4) { w->refused = true; break; }
        const uint32_t xlen = rd16(h + 10);
        if (left < 12 + (uint64_t)xlen) { w->refused = c_eof; break; }
        int64_t bsize = -1;
        uint32_t p = 0;
        while (p + 4 <= xlen) {
            const uint32_t slen = rd16(h + 12 + p + 2);
            if (slen > xlen - p - 4) break;
            if (h[12 + p] == 'B' && h[12 + p + 1] == 'C' && slen == 2) bsize = rd16(h + 12 + p + 4);
            p += 4 + slen;
        }
        const uint64_t size = (uint64_t)bsize + 1;
        if (p != xlen || bsize < 0 || size < 12 + (uint64_t)xlen + 8) { w->refused = true; break; }
        if (left < size) { w->refused = c_eof; break; }
        const uint32_t isize = rd32(h + size - 4);
        if (isize > kBgzfMaxText) { w->refused = true; break; }
        BgzfBlock b;
        b.c_off = at + 12 + xlen; b.t_off = w->text;
        b.c_len = (uint32_t)(size - 12 - xlen - 8); b.crc = rd32(h + size - 8); b.isize = isize; b.pad = 0;
        w->blocks.push_back(b);
        w->member.push_back(at);
        w->text += isize;
        at += size;
    }
    w->c_end = at;
}

// The blocks of w inflated on the device after head[0, head_bytes): *d_text (device memory of
// fastx_text_bytes(*text_bytes) bytes) holds the head and the text of the blocks before the first one the device
// refuses; *n_ok: those blocks. The last byte of the text is in *last.
int bgzf_inflate_dev(const mgb_index_t *index, const uint8_t *cbuf, BgzfWalk &w, const char *head, uint64_t head_bytes,
                     Stream &st, DevBufs &bufs, uint8_t **d_text, uint64_t *text_bytes, uint64_t *n_ok, uint8_t *last,
                     mgb_stats_t *stats) {
    (void)index;
    const uint64_t n = w.blocks.size();
    if (n > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "more than 2^32 - 1 BGZF blocks in one call");
    int rc;
    BgzfArgs a;
    std::memset(&a, 0, sizeof(a));
    a.n_blocks = (uint32_t)n;
    if ((rc = bufs.alloc(d_text, fastx_text_bytes(head_bytes + w.text)))) return rc;
    if (head_bytes && (rc = h2d(*d_text, head, head_bytes, st))) return rc;
    stats->h2d_bytes += head_bytes;
    std::vector<uint32_t> status(n, 0);
    if (n) {
        uint8_t *d_c = nullptr;
        BgzfBlock *d_blocks = nullptr;
        if ((rc = bufs.alloc(&d_c, w.c_end)) || (rc = bufs.alloc(&d_blocks, n)) || (rc = bufs.alloc(&a.status, n)))
            return rc;
        if ((rc = h2d(d_c, cbuf, w.c_end, st)) || (rc = h2d(d_blocks, w.blocks.data(), n * sizeof(BgzfBlock), st)))
            return rc;
        stats->h2d_bytes += w.c_end + n * sizeof(BgzfBlock);
        a.cbuf = d_c; a.blocks = d_blocks; a.text = *d_text + head_bytes;
#if defined(MGB_HOST_EMU)
        BgzfShared sh;
        bgzf_crc_table(sh);
        for (uint32_t b = 0; b < a.n_blocks; ++b) bgzf_inflate_block(a, b, sh);
#else
        const unsigned grid = (unsigned)std::min<uint64_t>((n + kBgzfWarps - 1) / kBgzfWarps, (uint64_t)index->num_sms * 16);
        k_bgzf_inflate<<<grid, 32 * kBgzfWarps, 0, st.s>>>(a);
        CUDA_TRY(cudaGetLastError());
#endif
        stats->kernel_launches += 1;
        if ((rc = d2h(status.data(), a.status, n * 4, st)) || (rc = sync(st))) return rc;
        stats->d2h_bytes += n * 4;
    }
    uint64_t ok = 0;
    while (ok < n && status[ok] == kBgzfOk) ++ok;
    if (ok < n) { w.c_end = w.member[ok]; w.refused = true; }
    *n_ok = ok;
    *text_bytes = head_bytes + (ok < n ? w.blocks[ok].t_off : w.text);
    *last = 0;
    if (*text_bytes > head_bytes) {
        if ((rc = d2h(last, *d_text + *text_bytes - 1, 1, st)) || (rc = sync(st))) return rc;
        stats->d2h_bytes += 1;
    } else if (head_bytes) {
        *last = (uint8_t)head[head_bytes - 1];
    }
    return 0;
}

// ---------------------------------------------------------------------------------------
// Plain gzip input (mgb_fastx_stage_gzip, mgb_gzip_inflate): member headers and trailers read on the host, the DEFLATE
// stream decoded speculatively on the device (gzip_core.cuh)
// ---------------------------------------------------------------------------------------
constexpr uint64_t kGzipSubBytes = 32768;        // compressed bytes per sub-range of a stage

// The gzip member header (RFC 1952) at c[0, n): its length; 0 when n ends inside it; -1 when the bytes are not a header
// this route serves (not gzip, not DEFLATE, or reserved flag bits). FHCRC is skipped unchecked, as Python's gzip does.
int64_t gzip_header(const uint8_t *c, uint64_t n) {
    if ((n > 0 && c[0] != 31) || (n > 1 && c[1] != 139) || (n > 2 && c[2] != 8) || (n > 3 && (c[3] & 0xe0))) return -1;
    if (n < 10) return 0;
    const uint8_t flg = c[3];
    uint64_t at = 10;
    if (flg & 4) {
        if (n < at + 2) return 0;
        at += 2 + rd16(c + at);
    }
    for (uint8_t f : { (uint8_t)8, (uint8_t)16 }) {
        if (!(flg & f)) continue;
        while (at < n && c[at]) ++at;
        if (at >= n) return 0;
        ++at;
    }
    if (flg & 2) at += 2;
    return at <= n ? (int64_t)at : 0;
}

struct GzipCounts { uint64_t n_sub = 0, found = 0, confirmed = 0; };

// What one stage did: it staged `text` bytes after the head, took c_used whole bytes, refused the input (the stream
// is unchanged), or ended a member.
struct GzipStage {
    uint64_t text = 0, c_used = 0;
    bool refused = false, member_end = false;
};

// One stage of stream s over c[0, n) (the first byte's first s->bit bits already decoded when in a member): the
// member header if the stream is between members, then the DEFLATE stream from its position to the last confirmed
// block end, or to the member's end and its checked trailer. *d_text (fastx_text_bytes of head + text, from bufs)
// holds head then the text; *last: its last byte. Nothing is staged and s is unchanged when the stage refuses or
// needs more input (c_used 0, not refused). inject: candidate bit offsets in c that replace the finder.
// hand_over_unsplit: refuse a member whose first stage confirmed no candidate (see mgb_fastx_stage_gzip).
int gzip_stage_dev(const mgb_index_t *index, mgb_gzip_stream *s, const uint8_t *c, uint64_t n, bool c_eof,
                   uint64_t max_text, uint64_t sub_bytes, const std::vector<uint64_t> *inject,
                   bool hand_over_unsplit, const char *head,
                   uint64_t head_bytes, Stream &st, DevBufs &bufs, uint8_t **d_text, uint8_t *last, GzipStage *out,
                   GzipCounts *counts, mgb_stats_t *stats) {
    (void)index;
    int rc;
    *out = GzipStage();
    mgb_gzip_stream g = *s;
    uint64_t hdr = 0;
    bool go = n > 0;
    if (!g.in_member && n) {
        const int64_t h = gzip_header(c, n);
        if (h < 0 || (h == 0 && c_eof)) out->refused = true;
        go = h > 0;
        if (h > 0) {
            hdr = (uint64_t)h;
            g.in_member = true; g.bit = 0; g.member_text = 0; g.crc = 0;
            std::fill(g.window.begin(), g.window.end(), 0);
        }
    } else if (!g.in_member) {
        go = false;                                                   // the end of the input, between members
    }
    const uint64_t start = hdr * 8 + g.bit, sub_bits = sub_bytes * 8;
    if (g.in_member && start >= n * 8) {
        go = false;
        if (c_eof) out->refused = true;                               // cut off after the header or a block
    }
    std::unique_ptr<DevBufs> ib;
    GzipArgs a;
    std::memset(&a, 0, sizeof(a));
    std::vector<GzipSub> res;
    std::vector<uint64_t> cand;
    std::vector<GzipLink> links;
    uint64_t end = start, text = 0;
    bool final = false;
    if (go) {
        // as many sub-ranges as max_text needs at the stream's ratio so far (3 before any text), and the bytes their
        // decodes may run into
        const double ratio = g.c_bits ? std::max(1.0, 8.0 * g.text / g.c_bits) : 3.0;
        const uint64_t all = (n * 8 - start + sub_bits - 1) / sub_bits;
        uint64_t n_sub = std::min<uint64_t>(all, (uint64_t)std::min(1e12, (double)max_text / (ratio * sub_bytes)) + 2);
        uint64_t up = std::min<uint64_t>(n, (start + n_sub * sub_bits) / 8 + std::max<uint64_t>(4 * sub_bytes, 262144));
        uint64_t cap = std::max<uint64_t>(16 * sub_bytes, 262144);
        bool retried = false;
        for (;;) {
            if (n_sub > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "too many gzip sub-ranges in one stage");
            ib.reset(new DevBufs(st, bufs.ws, kInflateSlots));
            a.start = start; a.sub_bits = sub_bits; a.n_sub = (uint32_t)n_sub; a.cap = (uint32_t)cap; a.cbytes = up;
            uint8_t *d_c = nullptr;
            if ((rc = ib->alloc(&d_c, up)) || (rc = ib->alloc(&a.cand, n_sub)) || (rc = ib->alloc(&a.res, n_sub))
                || (rc = ib->alloc(&a.sym, n_sub * cap)))
                return rc;
            a.cbuf = d_c;
            if ((rc = h2d(d_c, c, up, st))) return rc;
            stats->h2d_bytes += up;
            cand.assign(n_sub, kGzipNone);
            if (inject) {
                cand[0] = start;
                for (uint64_t p : *inject)
                    if (p > start && p < up * 8) {
                        const uint64_t j = (p - start) / sub_bits;
                        if (j < n_sub && p < cand[j]) cand[j] = p;
                    }
                if ((rc = h2d(a.cand, cand.data(), n_sub * 8, st))) return rc;
            }
#if defined(MGB_HOST_EMU)
            BgzfShared sh;
            if (!inject) for (uint32_t j = 0; j < a.n_sub; ++j) gzip_find_sub(a, j, sh);
            for (uint32_t j = 0; j < a.n_sub; ++j) gzip_decode_sub(a, j, sh);
#else
            const unsigned grid = (unsigned)std::min<uint64_t>((n_sub + kGzipWarps - 1) / kGzipWarps, (uint64_t)index->num_sms * 16);
            if (!inject) k_gzip_find<<<grid, 32 * kGzipWarps, 0, st.s>>>(a);
            k_gzip_decode<<<grid, 32 * kGzipWarps, 0, st.s>>>(a);
            CUDA_TRY(cudaGetLastError());
#endif
            stats->kernel_launches += inject ? 1 : 2;
            res.resize(n_sub);
            if ((rc = d2h(cand.data(), a.cand, n_sub * 8, st)) || (rc = d2h(res.data(), a.res, n_sub * sizeof(GzipSub), st))
                || (rc = sync(st)))
                return rc;
            stats->d2h_bytes += n_sub * (8 + sizeof(GzipSub));
            // the chain: sub-range 0 starts at a block boundary; the sub-range whose candidate a confirmed decode ended
            // at exactly is confirmed too, and every block end a confirmed decode passed is the stream's
            links.clear();
            end = start; text = 0; final = false;
            uint64_t j = 0, confirmed = 0;
            uint32_t why = kGzipStop;
            for (;;) {
                const GzipSub &r = res[j];
                if (r.reach > g.member_text + text) { why = kBgzfBadStream; break; }     // before the member's start
                if (r.len) links.push_back(GzipLink{ j * cap, head_bytes + text, r.len, 0 });
                text += r.len;
                end = r.end;
                if (r.status == kGzipFinal) { final = true; break; }
                if (r.status != kGzipStop) { why = r.status; break; }
                const uint64_t k = (r.end - start) / sub_bits;
                if (k <= j || k >= n_sub || cand[k] != r.end) break;
                ++confirmed;
                if (text >= max_text) break;
                j = k;
            }
            counts->n_sub += n_sub;
            counts->confirmed += confirmed;
            for (uint64_t k = 1; k < n_sub; ++k) counts->found += cand[k] != kGzipNone && cand[k] <= end;
            if (why == kBgzfBadStream) { out->refused = true; break; }
            if (end > start || final) {
                // a member's first stage that decoded on one warp alone is a member the finder cannot see into
                // (stored or fixed-Huffman blocks): the command leaves it to the host whole
                if (hand_over_unsplit && g.member_text == 0 && !final && n_sub >= 2 && confirmed == 0 && !retried)
                    out->refused = true;
                break;
            }
            // no block ended: a block larger than the slot or than the bytes uploaded gets one sub-range with room
            retried = true;
            if (why == kBgzfBadSize && cap < (1ull << 28)) { n_sub = 1; cap *= 8; continue; }
            if (why == kGzipShort && up < n) { n_sub = 1; up = n; continue; }
            if (why == kBgzfBadSize || c_eof) out->refused = true;            // too large, or cut off
            go = false;
            break;
        }
        if (out->refused) go = false;
    }
    // the trailer: CRC32 and ISIZE of the member, after its last byte
    const uint64_t tb = (end + 7) / 8;
    if (go && final && tb + 8 > n) {
        if (c_eof) out->refused = true;
        go = false;
    }
    if ((rc = bufs.alloc(d_text, fastx_text_bytes(head_bytes + (go ? text : 0))))) return rc;
    if (head_bytes && (rc = h2d(*d_text, head, head_bytes, st))) return rc;
    stats->h2d_bytes += head_bytes;
    *last = head_bytes ? (uint8_t)head[head_bytes - 1] : 0;
    if (!go) return 0;
    if (links.size() > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "too many gzip sub-ranges in one stage");
    const uint64_t n_links = links.size(), pieces = (text + kGzipCrcPiece - 1) / kGzipCrcPiece;
    std::vector<uint32_t> parts(pieces);
    if (n_links) {
        GzipLink *d_links = nullptr;
        if ((rc = ib->alloc(&d_links, n_links)) || (rc = ib->alloc(&a.win, (n_links + 1) * kGzipWindow))
            || (rc = ib->alloc(&a.crc_parts, pieces)))
            return rc;
        if ((rc = h2d(d_links, links.data(), n_links * sizeof(GzipLink), st)) || (rc = h2d(a.win, g.window.data(), kGzipWindow, st)))
            return rc;
        stats->h2d_bytes += n_links * sizeof(GzipLink) + kGzipWindow;
        a.links = d_links; a.n_links = (uint32_t)n_links; a.text = *d_text; a.n_text = text;
#if defined(MGB_HOST_EMU)
        for (uint32_t i = 0; i < a.n_links; ++i)
            for (uint32_t x = 0; x < kGzipWindow; ++x) gzip_window_at(a, i, x);
        for (uint32_t i = 0; i < a.n_links; ++i)
            for (uint32_t x = 0; x < links[i].len; ++x) gzip_resolve_at(a, i, x);
        // the CRC32 parts run over the new text, after the head
        a.text = *d_text + head_bytes;
        BgzfShared sh;
        bgzf_crc_table(sh);
        for (uint64_t p = 0; p < pieces; ++p) gzip_crc_piece(a, p, sh.crc);
#else
        k_gzip_window<<<1, 1024, 0, st.s>>>(a);
        k_gzip_resolve<<<(unsigned)std::min<uint64_t>(n_links, (uint64_t)index->num_sms * 16), 256, 0, st.s>>>(a);
        a.text = *d_text + head_bytes;
        k_gzip_crc<<<(unsigned)std::max<uint64_t>(1, std::min<uint64_t>((pieces + 255) / 256, (uint64_t)index->num_sms * 8)), 256, 0, st.s>>>(a);
        CUDA_TRY(cudaGetLastError());
#endif
        stats->kernel_launches += 3;
        if ((rc = d2h(parts.data(), a.crc_parts, pieces * 4, st))
            || (rc = d2h(g.window.data(), a.win + n_links * kGzipWindow, kGzipWindow, st))
            || (rc = d2h(last, *d_text + head_bytes + text - 1, 1, st)) || (rc = sync(st)))
            return rc;
        stats->d2h_bytes += pieces * 4 + kGzipWindow + 1;
    }
    uint32_t crc = 0;
    const uint32_t whole = crc_x8n(kGzipCrcPiece);
    for (uint64_t p = 0; p < pieces; ++p)
        crc = crc_multmodp(p + 1 < pieces ? whole : crc_x8n(text - p * kGzipCrcPiece), crc) ^ parts[p];
    g.crc = crc_multmodp(crc_x8n(text), g.crc) ^ crc;
    g.member_text += text;
    g.text += text;
    g.c_bits += end - start;
    if (final) {
        if (rd32(c + tb) != g.crc || rd32(c + tb + 4) != (uint32_t)g.member_text) {
            out->refused = true;
            *last = head_bytes ? (uint8_t)head[head_bytes - 1] : 0;
            return 0;
        }
        g.in_member = false; g.bit = 0;
        out->c_used = tb + 8;
        out->member_end = true;
    } else {
        out->c_used = end / 8; g.bit = (uint32_t)(end % 8);
    }
    out->text = text;
    *s = g;
    return 0;
}

// k-mer to node ids of every read on `strands` strands: the forward strand's into out_f, the reverse complement's into
// *out_r (resized to the batch's k-mers); *koff: where each read's k-mers start
static int map_nodes(const mgb_index_t *index, const char *seqs, const uint64_t *offsets, uint32_t n, uint32_t strands,
                     uint64_t *out_f, std::vector<uint64_t> *out_r, std::vector<uint64_t> *koff) {
    CallWorkspace cw(index);
    if (int rc = cw.ready()) return rc;
    DevBufs bufs(cw.st, cw.w, kBatchSlots);
    Batch b; mgb_stats_t stats; std::memset(&stats, 0, sizeof(stats));
    int rc = upload_batch(index, seqs, offsets, n, strands == 2, cw.st, bufs, &b, koff, &stats);
    if (!rc) rc = dev_zero(b.nodes_f, (b.total_kmers + 1) * 8, cw.st);
    if (!rc && strands == 2) rc = dev_zero(b.nodes_r, (b.total_kmers + 1) * 8, cw.st);
    if (!rc) rc = launch_prepare(index, b, cw.st, index->num_sms);
    if (!rc) rc = launch_seed(index, b, strands, cw.st, bufs, nullptr);
    if (!rc) rc = d2h(out_f, b.nodes_f, b.total_kmers * 8, cw.st);
    if (!rc && strands == 2) { out_r->resize(b.total_kmers + 1); rc = d2h(out_r->data(), b.nodes_r, b.total_kmers * 8, cw.st); }
    if (!rc) rc = sync(cw.st);
    return rc;
}

} // namespace

extern "C" {

int mgb_map_to_nodes(const mgb_index_t *index, const char *seqs, const uint64_t *offsets,
                     uint32_t n_seqs, uint64_t *out_nodes) {
    if (!index || !seqs || !offsets || !out_nodes) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    // PRIMARY graph: CanonicalDBG::map_to_nodes_sequentially (canonical_dbg.cpp:55-146) = both strands mapped in
    // the stored graph; a k-mer missing on its own strand takes the id of its reverse complement + n
    const bool primary = index->view.mode == 2;
    std::vector<uint64_t> rev, koff;
    if (int rc = map_nodes(index, seqs, offsets, n_seqs, primary ? 2 : 1, out_nodes, &rev, &koff)) return rc;
    if (primary) {
        const uint64_t n = index->view.n;
        for (uint32_t r = 0; r < n_seqs; ++r) {
            const uint64_t lo = koff[r], nk = koff[r + 1] - koff[r];
            for (uint64_t i = 0; i < nk; ++i) {
                const uint64_t rv = rev[lo + nk - 1 - i];
                if (!out_nodes[lo + i] && rv) out_nodes[lo + i] = rv + n;
            }
        }
    }
    return MGB_OK;
}

int mgb_map_to_nodes_strands(const mgb_index_t *index, const char *seqs, const uint64_t *offsets,
                             uint32_t n_seqs, uint64_t *out_fwd, uint64_t *out_rc) {
    if (!index || !seqs || !offsets || !out_fwd || !out_rc) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (!index->at.has_complement) return fail(MGB_ERR_BAD_CONFIG, "a reverse-complement strand needs a DNA graph");
    std::vector<uint64_t> rev, koff;
    if (int rc = map_nodes(index, seqs, offsets, n_seqs, 2, out_fwd, &rev, &koff)) return rc;
    std::memcpy(out_rc, rev.data(), 8 * koff[n_seqs]);
    return MGB_OK;
}

} // extern "C"

// MGB_DEBUG, when k_prepare_exact ran and at most 8 reads reach k_align on pass 0: one line per such read with what
// turned it down at each whole-read gate, read back from the device. exact_path_strand (kernels.cuh, conditions 1-4):
// the length limit, whether the position-0 k-mer of each strand has a node (f0 / r0), the primary's place p on the path,
// the first k-mer offset from p with a pl_stop or pl_rc bit, the first character that is not A/C/G/T or differs from
// pl_text, and the score. exact_read_strand: the length limit, the summary bits (answered only as 0x6 or 0x9) and the
// score against the threshold. Host code, never on a timed path.
static void debug_left_over(const IndexView &ix, const PrepExactArgs &pa, const ExactArgs &ea, const char *seqs,
                            const uint64_t *offsets, const std::vector<uint64_t> &koff, const Batch &b,
                            const uint8_t *summary, const uint32_t *d_rest, uint32_t n, uint32_t lo, uint32_t n_reads,
                            Stream &st) {
    std::vector<uint32_t> rest(n);
    if (d2h(rest.data(), d_rest, 4ull * n, st) || sync(st)) return;
    const int k = (int)ix.k;
    for (uint32_t r : rest) {
        const char *raw = seqs + offsets[r];
        const int L = (int)(offsets[r + 1] - offsets[r]), nk = L - k + 1;
        std::string path = "length", read = "length";
        uint8_t bits = 0;
        if (summary) d2h(&bits, summary + r, 1, st);
        uint64_t n0[2] = { 0, 0 };
        uint32_t p = kPlNone;
        if (nk > 0) {
            d2h(&n0[0], b.nodes_f + koff[r], 8, st);
            d2h(&n0[1], b.nodes_r + koff[r], 8, st);
        }
        sync(st);
        const int s = (n0[0] != 0) == (n0[1] != 0) ? -1 : n0[0] ? 0 : 1;
        // the primary strand's characters, upper case (N: not A/C/G/T); Σ diag over them
        std::string q(L > 0 ? L : 0, 'N');
        for (int i = 0; i < L; ++i) {
            const char c = (char)std::toupper((unsigned char)(s == 1 ? raw[L - 1 - i] : raw[i]));
            const char *at = std::strchr("ACGT", c);
            q[i] = !c || !at ? 'N' : s == 1 ? "TGCA"[at - "ACGT"] : c;
        }
        long score = ea.end_bonus;
        for (char c : q) score += ea.diag[(uint8_t)c & 0x7F];
        if (nk > 0 && L <= (int)pa.ex.max_len) {
            if (s < 0) {
                path = "probe";
            } else {
                if (ix.pl_n) d2h(&p, ix.pl_pos + n0[s], 4, st);
                sync(st);
                if (p == kPlNone) {
                    path = "no path position";
                } else {
                    const uint32_t w0 = p >> 5, w1 = (p + (uint32_t)L + 31) >> 5;
                    std::vector<uint32_t> sw(w1 - w0 + 1), rw(w1 - w0 + 1);
                    std::vector<unsigned long long> tw(w1 - w0 + 1);
                    d2h(sw.data(), ix.pl_stop + w0, 4ull * sw.size(), st);
                    d2h(rw.data(), ix.pl_rc + w0, 4ull * rw.size(), st);
                    d2h(tw.data(), ix.pl_text + w0, 8ull * tw.size(), st);
                    sync(st);
                    int stop = -1, rcb = -1, bad = -1, diff = -1;
                    for (int t = nk - 1; t >= 0; --t) {
                        const uint32_t x = p + (uint32_t)t - (w0 << 5);
                        if ((sw[x >> 5] >> (x & 31)) & 1u) stop = t;
                        if ((rw[x >> 5] >> (x & 31)) & 1u) rcb = t;
                    }
                    for (int i = L - 1; i >= 0; --i) {
                        const char *acgt = std::strchr("ACGT", q[i]);
                        const uint32_t x = p + (uint32_t)i - (w0 << 5);
                        if (q[i] == 'N') bad = i;
                        else if ((int)((tw[x >> 5] >> (2 * (x & 31))) & 3u) != (int)(acgt - "ACGT")) diff = i;
                    }
                    char buf[160];
                    std::snprintf(buf, sizeof(buf), "p=%u stop@%d rc@%d invalid@%d mismatch@%d", p, stop, rcb, bad, diff);
                    path = stop >= 0 || rcb >= 0 || bad >= 0 || diff >= 0 ? buf
                         : score < pa.ex.min_score ? std::string(buf) + " threshold" : std::string(buf) + " (answers)";
                }
            }
        }
        if (nk > 0 && L <= (int)ea.max_len) {
            read = bits == 0x6 || bits == 0x9 ? (score < ea.min_score ? "threshold" : "(answers)") : "summary bits";
        }
        std::fprintf(stderr, "[mgb] reads %u+%u left to k_align: read %u L=%d f0=%d r0=%d | exact_path_strand: %s | "
                     "exact_read_strand: summary=0x%x score=%ld min=%d: %s\n", lo, n_reads, r, L,
                     n0[0] != 0, n0[1] != 0, path.c_str(), bits, score, ea.min_score, read.c_str());
    }
}

// Where a call's alignments go. records: mgb_alignment_t on the host (mgb_align_batch); text: TSV or JSON rendered on
// the device (mgb_align_batch_text and the file route); columns: the caller's device arrays (mgb_align_batch_device),
// with every pass classified on the device. The text and columns routes keep every pass's heap on the device.
enum class Route { records, text, columns };

// What is the same for every piece of one call
struct Call {
    const mgb_index_t *index;
    const DevConfig &dcfg;
    Route route;
    const char *seqs; const uint64_t *offsets;          // the batch's reads
    const char *names; const uint64_t *name_offsets;    // text route: their headers
    int text_format;                                    // text route: MGB_TEXT_TSV / MGB_TEXT_JSON
    int32_t min_path_score;
    bool dev_input;          // reads (and headers) are device memory (the file and columns routes), offsets host memory
};

// One contiguous range of reads [lo, lo + n) of a batch, processed start to finish on its own
// stream: upload, prepare + seed, align passes, download, materialisation. Pieces of one batch are
// independent (IDBGAligner::align_batch treats every query separately, dbg_aligner.cpp:251-355), so
// the download and unpacking of one piece overlap the kernels of the next.
struct Piece {
    uint32_t lo = 0, n_reads = 0;
    // views into the arrays of the enclosing mgb_results: entries of reads [lo, lo + n_reads), and a
    // region of n_reads * num_alternative_paths records that receives n_alns of them (piece-local
    // indices in `first`)
    uint64_t *first = nullptr;
    uint32_t *count = nullptr;
    mgb_alignment_t *alns = nullptr;
    uint64_t n_alns = 0;
    std::vector<HostBuf> heaps;
    std::vector<uint64_t> heap_bytes;
    uint64_t *src_off = nullptr; uint32_t *src_heap = nullptr;   // views into the enclosing mgb_results
    HostBuf text;                    // text route: the piece's text
    uint64_t text_bytes = 0;
    mgb_stats_t stats = {};
    int rc = 0; std::string err;
    ~Piece() { for (HostBuf b : heaps) hostbuf_release(b); if (text.p) hostbuf_release(text); }
};

// MGB_DEBUG=1: wall-clock split of a piece on stderr
struct Ticks {
    bool on; uint32_t lo, n_reads;
    std::chrono::steady_clock::time_point last = std::chrono::steady_clock::now();
    void operator()(const char *what) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        std::fprintf(stderr, "[mgb] reads %u+%u %-28s %8.2f ms\n", lo, n_reads, what,
                     std::chrono::duration<double, std::milli>(now - last).count());
        last = now;
    }
};

// offsets all[lo .. lo + n] relative to base: in place when base is 0, else rebased into *local
static const uint64_t *rebase_offsets(const uint64_t *all, uint32_t lo, uint32_t n, uint64_t base,
                                      std::vector<uint64_t> *local) {
    if (!base) return all + lo;
    local->resize((size_t)n + 1);
    for (uint32_t r = 0; r <= n; ++r) (*local)[r] = all[lo + r] - base;
    return local->data();
}

// the packed records of one read as `count` mgb_alignment_t
static void unpack_records(const char *p, uint32_t count, bool no_nodes, uint32_t read_index, mgb_alignment_t *dst) {
    for (uint32_t i = 0; i < count; ++i) {
        RecView v;
        p = rec_next(p, no_nodes, &v);
        const OutAln &o = v.o;
        mgb_alignment_t al;
        std::memset(&al, 0, sizeof(al));
        al.read_index = read_index; al.orientation = (uint8_t)o.orientation; al.score = o.score;
        al.offset = o.offset; al.query_begin = o.query_begin; al.query_len = o.query_len;
        al.num_nodes = o.n_nodes; al.sequence_len = o.seq_len; al.num_cigar_ops = o.n_cigar;
        al.nodes = v.nodes; al.cigar = v.cigar; al.sequence = v.seq;
        dst[i] = al;
    }
}

// output heap of a pass over n reads: generous first guess, doubled on retry passes (MGB_TEST_HEAP0: test knob,
// pass 0's capacity in bytes)
static uint64_t heap_cap_of(const Batch &b, const DevConfig &dcfg, uint32_t k, uint64_t n, uint32_t scale) {
    const uint64_t per_read = sizeof(OutAln) + 9ull * (b.L_max + 64 + k) + 4ull * 64;
    uint64_t cap = n * per_read * dcfg.num_alternative_paths * scale + 4096;
    if (const char *e = std::getenv("MGB_TEST_HEAP0")) if (scale == 1) cap = std::min<uint64_t>(cap, std::atoll(e));
    return cap;
}

// longest read with a whole-read exact answer: k_align's own exit needed both strands staged on chip
// (L + 1 <= lq) and room for L characters and L - k + 1 nodes in an alignment slot
static uint32_t exact_max_len(const Caps &caps, uint32_t k, int lq) {
    const uint64_t max_len = std::min<uint64_t>({ lq > 0 ? (uint64_t)lq - 1 : 0, caps.aln_seq,
                                                 (uint64_t)caps.aln_nodes + k - 1 });
    return caps.aln_cigar >= 1 ? (uint32_t)max_len : 0;
}

// the configuration part of the whole-read gate (kernels.cuh ExactArgs), over the batch's arrays
static void exact_args(const Batch &b, const DevConfig &dcfg, uint32_t k, const Caps &caps, int lq,
                       const uint8_t *summary, ReadHdr *hdr, ExactArgs *ea) {
    std::memset(ea, 0, sizeof(*ea));
    ea->k = k;
    ea->end_bonus = dcfg.left_end_bonus + dcfg.right_end_bonus;
    ea->min_score = std::max({ 0, (int)dcfg.min_cell_score, (int)dcfg.min_path_score });
    ea->max_len = exact_max_len(caps, k, lq);
    ea->result_nodes = dcfg.result_nodes;
    std::memcpy(ea->diag, dcfg.diag, sizeof(ea->diag));
    ea->qf = b.qf; ea->qr = b.qr; ea->offsets = b.offsets; ea->koff = b.koff;
    ea->nodes_f = b.nodes_f; ea->nodes_r = b.nodes_r; ea->summary = summary;
    ea->hdr = hdr;
}

// sub-k seeding (min_seed_length < k): the independent index_range lookups run GPU-wide ahead of k_align
static int launch_subk(const mgb_index_t *index, const SubkArgs &sk, uint32_t L_max, Stream &st) {
    const uint32_t chunks = (L_max + kSubkChunk - 1) / kSubkChunk;
#if defined(MGB_HOST_EMU)
    (void)index; (void)st;
    for (uint32_t r = 0; r < sk.n_reads; ++r)
        for (uint32_t s = 0; s < sk.n_strands; ++s)
            for (uint32_t c = 0; c < chunks; ++c) subk_item(sk, r, s, c);
#else
    // one warp per 32 query positions of a strand, 4 warps per block
    const uint64_t items = (uint64_t)sk.n_reads * sk.n_strands * ((chunks * kSubkChunk + 31) / 32);
    const uint64_t blocks = std::min<uint64_t>((items + 3) / 4, (uint64_t)index->num_sms * 16);
    CUDA_TRY(index->view.wide ? kern_any::launch_subk((unsigned)blocks, st.s, sk, chunks)
                              : kern_dna::launch_subk((unsigned)blocks, st.s, sk, chunks));
#endif
    return 0;
}

// text route: the piece's headers go up ahead of its reads, and the text's arguments that do not come from the passes
// are set
static int upload_headers(const Call &c, uint32_t n_reads, const char *names, const uint64_t *name_offs, Stream &st,
                          DevBufs &text_bufs, TextArgs *ta, mgb_stats_t *stats) {
    const uint64_t name_bytes = name_offs[n_reads];
    char *d_names = c.dev_input ? const_cast<char*>(names) : nullptr; uint64_t *d_name_off = nullptr;
    int rc = c.dev_input ? 0 : text_bufs.alloc(&d_names, name_bytes + 64);
    if (!rc) rc = text_bufs.alloc(&d_name_off, (size_t)n_reads + 1);
    if (!rc && name_bytes && !c.dev_input) rc = h2d(d_names, names, name_bytes, st);
    if (!rc) rc = h2d(d_name_off, name_offs, ((size_t)n_reads + 1) * 8, st);
    stats->h2d_bytes += (c.dev_input ? 0 : name_bytes) + ((size_t)n_reads + 1) * 8;
    ta->names = d_names; ta->name_off = d_name_off;
    ta->n_reads = n_reads; ta->k = c.index->view.k; ta->json = c.text_format == MGB_TEXT_JSON;
    ta->result_nodes = c.dcfg.result_nodes; ta->min_path_score = c.min_path_score;
    return rc;
}

// What prepare_and_seed leaves for the align passes
struct Seeded {
    bool exact_reads = false;        // the configuration allows whole-read exact answers (kernels.cuh ExactArgs)
    bool prep_exact = false;         // k_prepare_exact ran: pass 0's heap, counters and list are in pa / next0 / rest0
    bool subk = false;               // sub-k seeding ran (sk)
    uint8_t *summary = nullptr;      // k_seed_hash's per-read summary
    ReadHdr *hdr = nullptr;          // per read: status, n_aln, heap offset and stats of the pass that answered it
    PrepExactArgs pa;
    // k_align's next read, the reads k_exact_reads leaves, the length of pa.list, k_align's next arena
    unsigned int *next0 = nullptr; uint32_t *rest0 = nullptr;
    SubkArgs sk;
};

// query preparation (k_prepare, or k_prepare_exact with its whole-read answers), exact seeding and sub-k seeding;
// device events 1 and 2 mark the start and the end of the kernels
static int prepare_and_seed(const Call &c, const Batch &b, int lq, Stream &st, DevBufs &bufs, Seeded *sd,
                            mgb_stats_t *stats) {
    const mgb_index_t *index = c.index; const DevConfig &dcfg = c.dcfg;
    const uint32_t k = index->view.k, n_reads = b.n_reads;
    const bool both = dcfg.forward_and_reverse_complement;
    const bool map_nodes = dcfg.max_seed_length >= k;
    // The seeding kernel of graphs with the k-mer hash index summarises what it stored per read; without it the
    // whole-read gate reads the node arrays instead.
    sd->exact_reads = dcfg.exact_shortcut && both && index->view.mode == 0 && dcfg.min_seed_length == k
                      && dcfg.max_seed_length == k && !dcfg.seed_complexity_filter && dcfg.min_exact_match <= 1.0;
    int rc;
    if (sd->exact_reads && index->view.kh_slots && (rc = bufs.alloc(&sd->summary, (size_t)n_reads + 1))) return rc;
    if ((rc = dev_zero(b.nodes_f, (b.total_kmers + 1) * 8, st))) return rc;
    if (both && (rc = dev_zero(b.nodes_r, (b.total_kmers + 1) * 8, st))) return rc;
    if ((rc = bufs.alloc(&sd->hdr, (size_t)n_reads + 1))) return rc;
#if defined(MGB_PROBE_NO_WRITES)
    if ((rc = dev_zero(sd->hdr, ((size_t)n_reads + 1) * sizeof(ReadHdr), st))) return rc;     // k_prepare_exact stores none
#endif
    // Whole-read exact answers from the raw reads, in place of k_prepare (kernels.cuh PrepExactArgs), on graphs with
    // the k-mer hash index and the path layout: the reads left over are prepared, seeded and go on as before. Pass 0's
    // heap, its counters and the list exist before the kernel runs; pass 0 takes them over.
    // MGB_TEST_NO_PREPARE_EXACT: test knob, the route off.
    PrepExactArgs &pa = sd->pa;
    std::memset(&pa, 0, sizeof(pa));
    sd->prep_exact = sd->exact_reads && index->view.kh_slots && index->view.pl_n
                     && exact_max_len(choose_caps(b.L_max, dcfg, k, 1), k, lq) >= k
                     && !std::getenv("MGB_TEST_NO_PREPARE_EXACT");
    if (sd->prep_exact) {
        pa.ix = index->view;
        pa.prep = PrepArgs { b.seqs, b.offsets, b.n_reads, b.qf, b.qr, b.cf, b.cr, {0} };
        std::memcpy(pa.prep.code_of, index->at.code_of, sizeof(pa.prep.code_of));
        exact_args(b, dcfg, k, choose_caps(b.L_max, dcfg, k, 1), lq, sd->summary, sd->hdr, &pa.ex);
        pa.stage_bytes = prep_stage_bytes(b.L_max);
        pa.ex.heap_cap = heap_cap_of(b, dcfg, k, n_reads, 1);
        if ((rc = bufs.alloc(&pa.ex.heap, pa.ex.heap_cap)) || (rc = bufs.alloc(&pa.ex.heap_used, 1))
            || (rc = bufs.alloc(&sd->next0, 4)) || (rc = bufs.alloc(&pa.list, (size_t)n_reads + 1))
            || (rc = bufs.alloc(&sd->rest0, (size_t)n_reads + 1)) || (rc = dev_zero(pa.ex.heap_used, 8, st))
            || (rc = dev_zero(sd->next0, 16, st)))
            return rc;
        pa.n_list = sd->next0 + 2;
#if defined(MGB_PREP_TIMERS) && !defined(MGB_HOST_EMU)
        if ((rc = bufs.alloc(&pa.phase_out, PREP_N_PHASES)) || (rc = dev_zero(pa.phase_out, 8 * PREP_N_PHASES, st))) return rc;
#endif
    }
    record(st, 1);
    rc = sd->prep_exact ? launch_prepare_exact(index, pa, st) : launch_prepare(index, b, st, index->num_sms);
    stats->kernel_launches += 1;
    if (rc) return rc;
    if (map_nodes && (rc = launch_seed(index, b, both ? 2 : 1, st, bufs, sd->summary, &stats->kernel_launches,
                                       sd->prep_exact ? pa.list : nullptr, sd->prep_exact ? pa.n_list : nullptr)))
        return rc;
    SubkArgs &sk = sd->sk;
    std::memset(&sk, 0, sizeof(sk));
    sd->subk = map_nodes && dcfg.min_seed_length < k && b.total_chars && !std::getenv("MGB_TEST_NOSUBK");
    if (sd->subk) {
        sk.ix = index->view; sk.cf = b.cf; sk.cr = b.cr; sk.offsets = b.offsets; sk.koff = b.koff;
        sk.nodes_f = b.nodes_f; sk.nodes_r = b.nodes_r; sk.n_reads = n_reads; sk.n_strands = both ? 2 : 1;
        sk.min_seed_length = dcfg.min_seed_length;
        sk.max_len = dcfg.max_seed_length < k - 1 ? dcfg.max_seed_length : k - 1;
        const size_t nc = b.total_chars + 64;
        if ((rc = bufs.alloc(&sk.first_f, nc)) || (rc = bufs.alloc(&sk.last_f, nc)) || (rc = bufs.alloc(&sk.len_f, nc)))
            return rc;
        if (both && ((rc = bufs.alloc(&sk.first_r, nc)) || (rc = bufs.alloc(&sk.last_r, nc))
                     || (rc = bufs.alloc(&sk.len_r, nc))))
            return rc;
        if ((rc = launch_subk(index, sk, b.L_max, st))) return rc;
        stats->kernel_launches += 1;
    }
    record(st, 2);
    return 0;
}

// The shape of one align pass: the per-read caps, arena and on-chip layout, and how many warps and arenas k_align gets
struct PassPlan {
    Caps caps; SmemLayout slay;
    size_t stride = 0, smem_per_warp = 0;      // arena and shared-memory bytes per warp
    int blocks_per_sm = 1;
    uint32_t n_warps = 1, n_arenas = 1;
};

static int pass_plan(const Call &c, const Batch &b, uint32_t L_pass, uint32_t scale, int lq, uint32_t n_pass,
                     const DevBufs &arena_bufs, PassPlan *p) {
    const mgb_index_t *index = c.index; const DevConfig &dcfg = c.dcfg;
    p->caps = choose_caps(L_pass, dcfg, index->view.k, scale);
    p->stride = arena_bytes(p->caps);
    // on-chip working set per warp: the column buffers hold the widest column the x-drop band
    // allows (choose_caps' estimate; at least 64 cells, the register path of the extender needs 40) of
    // reads up to 248 bp; wider columns spill to the arena scratch
    uint64_t band_est = (uint64_t)b.L_max + 9;
    if (dcfg.gap_ext < 0 && dcfg.xdrop < (1 << 20))
        band_est = std::min<uint64_t>(band_est, 2ull * (dcfg.xdrop / (-dcfg.gap_ext)) + 16 + 8);
    int bmax = band_est <= 256 ? std::max(64, (int)((band_est + 31) & ~31ull)) : 256;
    int hcap = 16;
    // test knobs: force the spill paths (arena scratch, queue migration)
    if (const char *e = std::getenv("MGB_TEST_BMAX")) bmax = std::atoi(e);
    if (const char *e = std::getenv("MGB_TEST_HCAP")) hcap = std::atoi(e);
    p->smem_per_warp = p->slay.carve(bmax, lq, hcap, (int)dcfg.num_alternative_paths, !index->view.wide);
#if defined(MGB_HOST_EMU)
    (void)n_pass; (void)arena_bufs;           // one lane aligns the reads one after the other in one arena
#else
    const size_t smem_block = p->smem_per_warp * kern_dna::kWarpsPerBlock;
    {
        // driver queries serialise against running work: ask once per shared-memory size
        static std::mutex occ_mu;
        static std::map<std::pair<int, size_t>, int> occ_cache;
        std::lock_guard<std::mutex> lk(occ_mu);
        const int variant = index->view.wide ? 1 : index->view.mode != 0 ? 2 : 0;    // which k_align
        auto key = std::make_pair(index->device * 4 + variant, smem_block);
        auto it = occ_cache.find(key);
        if (it == occ_cache.end()) {
            // the shared memory limit is a high-water mark per device and kernel: keep the largest
            size_t mx = smem_block;
            for (auto &kv : occ_cache) if (kv.first.first == key.first) mx = std::max(mx, kv.first.second);
            CUDA_TRY(variant == 1 ? kern_any::align_occupancy(mx, smem_block, &p->blocks_per_sm)
                   : variant == 2 ? kern_canon::align_occupancy(mx, smem_block, &p->blocks_per_sm)
                                  : kern_dna::align_occupancy(mx, smem_block, &p->blocks_per_sm));
            occ_cache[key] = p->blocks_per_sm;
        } else p->blocks_per_sm = it->second;
    }
    if (p->blocks_per_sm < 1) p->blocks_per_sm = 1;
    const uint64_t wpb = kern_dna::kWarpsPerBlock;        // warps (reads in flight) per block
    uint64_t n_warps = (uint64_t)index->num_sms * p->blocks_per_sm * wpb;
    if (n_warps > ((uint64_t)n_pass + wpb - 1) / wpb * wpb) n_warps = ((uint64_t)n_pass + wpb - 1) / wpb * wpb;
    n_warps = kern_dna::read_path_grid(n_warps / wpb) * wpb;    // (MGB_TEST_MAX_BLOCKS)
    // one arena per warp that can take a read, and as many as fit in 60 % of the free memory (at least one)
    uint64_t n_arenas = std::min<uint64_t>(n_warps, n_pass);
    if (p->stride * n_arenas > arena_bufs.capacity_of_next()) {
        size_t free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        const uint64_t mem_arenas = (uint64_t)(free_b * 0.6 + arena_bufs.capacity_of_next()) / (p->stride ? p->stride : 1);
        n_arenas = std::max<uint64_t>(1, std::min(n_arenas, mem_arenas));
        n_warps = std::min(n_warps, (n_arenas + wpb - 1) / wpb * wpb);
    }
    p->n_warps = (uint32_t)n_warps; p->n_arenas = (uint32_t)n_arenas;
#endif
    return 0;
}

// k_align over a.read_list (its length a.n_list, or *a.n_list_dev when set); n_align: the reads it gets, for MGB_DEBUG
static int launch_align(const mgb_index_t *index, const AlignArgs &a, const PassPlan &p, uint32_t n_align, bool dbg,
                        Stream &st) {
#if defined(MGB_HOST_EMU)
    (void)index; (void)n_align; (void)dbg; (void)st;
    const uint32_t n = a.n_list_dev ? *a.n_list_dev : a.n_list;
    if (n) init_arena(a, a.arena);
    std::vector<char> smem_emu(p.smem_per_warp + 64);
    const WarpMem mem_emu { a.arena, &a.lay };
    const WarpSmem sm_emu { smem_emu.data(), &a.slay };
    for (uint32_t t = 0; t < n; ++t) align_read(a, a.read_list[t], mem_emu, sm_emu);
#else
    const uint64_t wpb = kern_dna::kWarpsPerBlock;
    const uint32_t grid = (uint32_t)(std::min<uint64_t>(p.n_warps, ((uint64_t)a.n_list + wpb - 1) / wpb * wpb) / wpb);
    if (dbg) {         // every pass; per_round: warps launched with an arena, each aligning one read at a time
        char launched[128] = "";          // (one fprintf: pieces on two host threads print at once)
        if (a.n_list) std::snprintf(launched, sizeof(launched), "; launch k_align grid=%u block=%d per_round=%llu items=%u",
                                    grid, kern_dna::kAlignThreads,
                                    (unsigned long long)std::min<uint64_t>((uint64_t)grid * wpb, p.n_arenas), n_align);
        std::fprintf(stderr, "[mgb] k_align grid: %u warps (%llu resident), arena %zu bytes per warp, %u arenas%s\n",
                     p.n_warps, (unsigned long long)index->num_sms * p.blocks_per_sm * wpb, p.stride, p.n_arenas, launched);
    }
    const size_t smem_block = p.smem_per_warp * kern_dna::kWarpsPerBlock;
    if (a.n_list) {
        CUDA_TRY(index->view.wide ? kern_any::launch_align(grid, smem_block, st.s, a)
               : index->view.mode != 0 ? kern_canon::launch_align(grid, smem_block, st.s, a)
                                       : kern_dna::launch_align(grid, smem_block, st.s, a));
    }
#endif
    return 0;
}

// MGB_DEBUG on pass 0 after k_prepare_exact: how many reads each whole-read stage answered, and why the last few
// were left over
static void debug_exact_counts(const Call &c, uint32_t lo, const Batch &b, const std::vector<uint64_t> &koff,
                               const char *seqs, const uint64_t *offsets, const Seeded &sd, const ExactArgs &ea,
                               const uint32_t n_rest[2], Stream &st) {
    const uint32_t n_reads = b.n_reads;
    std::fprintf(stderr, "[mgb] reads %u+%u k_prepare_exact answered %u, left over %u\n", lo, n_reads,
                 n_reads - n_rest[1], n_rest[1]);
    std::fprintf(stderr, "[mgb] reads %u+%u k_exact_reads answered %u, left to k_align %u\n", lo, n_reads,
                 n_rest[1] - n_rest[0], n_rest[0]);
    if (n_rest[0] <= 8 && !c.dev_input)
        debug_left_over(c.index->view, sd.pa, ea, seqs, offsets, koff, b, sd.summary, ea.rest, n_rest[0], lo, n_reads, st);
#if defined(MGB_PREP_TIMERS) && !defined(MGB_HOST_EMU)
    unsigned long long ph[PREP_N_PHASES];
    if (cudaMemcpy(ph, sd.pa.phase_out, sizeof(ph), cudaMemcpyDeviceToHost) != cudaSuccess) return;
    const double nr = n_reads ? (double)n_reads : 1.0;
    std::fprintf(stderr, "[mgb] k_prepare_exact cycles/read: stage %.0f keys %.0f lookup %.0f stop_rc %.0f "
                 "text %.0f alloc %.0f write %.0f left %.0f\n", ph[PREP_STAGE] / nr, ph[PREP_KEYS] / nr,
                 ph[PREP_LOOKUP] / nr, ph[PREP_STOPRC] / nr, ph[PREP_TEXT] / nr, ph[PREP_ALLOC] / nr,
                 ph[PREP_WRITE] / nr, ph[PREP_LEFT] / nr);
#endif
}

// The align passes of a piece so far. Whether run_pass classifies a pass on the host (into read_heap) or on the device
// (into pass_of), it leaves the next pass's list in read order, its length and its longest read here.
struct PassState {
    std::vector<uint32_t> list;      // the pass's reads; empty on pass 0 after k_prepare_exact until its launches are in
    uint32_t n_pass = 0;
    uint32_t L_retry = 0;            // the longest read of list, after the first pass: it sizes the next pass's arena
    const char *heap[kMaxPasses] = {};   // every pass's output heap on the device
    std::vector<uint8_t> read_heap;  // host classification: the pass that answered each read (its heap of the piece)
    ReadHdr *hdr_host = nullptr;     // host classification: the headers of the pass, downloaded
    uint8_t *pass_of = nullptr;      // device classification: read_heap on the device
    float align_ms = 0, d2h_ms = 0;
    void all_reads(uint32_t n) { list.resize(n); std::iota(list.begin(), list.end(), 0u); }
};

// k_pass_classify's work one read after the other: the host classification, and the device one in the emulation build.
// a.retry may be a.list, which is then compacted in place.
static void classify_reads(const ClassifyArgs &a) {
    for (uint32_t t = 0; t < a.n_list; ++t) {
        const uint32_t r = a.list ? a.list[t] : t;
        if (classify_read(a, r, *a.sum)) { MGB_EMU_HIT(EMU_READ_OVERFLOW); a.retry[a.sum->n_retry++] = r; }
    }
}

// The classification on the device (k_pass_classify): only the summary comes back, into *sum, and the list of the reads
// that overflowed when there are any, into ps->list.
static int classify_pass(const Call &c, const Batch &b, const Seeded &sd, int pass, const uint32_t *d_list,
                         uint32_t n_list, DevBufs &heap_bufs, Stream &st, PassState *ps, PassSummary *sum, Piece *res) {
    constexpr size_t kSumWords = sizeof(PassSummary) / 4;
    uint32_t *d_block = nullptr;                 // the summary, then the retry list
    int rc;
    if ((rc = heap_bufs.alloc(&d_block, kSumWords + n_list)) || (rc = dev_zero(d_block, sizeof(PassSummary), st))) return rc;
    const ClassifyArgs a { d_list, n_list, sd.hdr, b.offsets, ps->pass_of, (uint32_t)pass,
                           reinterpret_cast<PassSummary*>(d_block), d_block + kSumWords };
#if defined(MGB_HOST_EMU)
    (void)c;
    classify_reads(a);
#else
    if (n_list) {
        const unsigned grid = (unsigned)kern_dna::read_path_grid(std::min<uint64_t>((n_list + 255) / 256, (uint64_t)c.index->num_sms * 8));
        kern_dna::log_launch("k_pass_classify", grid, 256, (uint64_t)grid * 256, n_list);     // a lane per read
        k_pass_classify<<<grid, 256, 0, st.s>>>(a);
        CUDA_TRY(cudaGetLastError());
    }
#endif
    record(st, 3);
    if ((rc = d2h(sum, a.sum, sizeof(*sum), st)) || (rc = sync(st))) return rc;
    ps->list.resize(sum->n_retry);
    if (sum->n_retry && ((rc = d2h(ps->list.data(), a.retry, (size_t)sum->n_retry * 4, st)) || (rc = sync(st)))) return rc;
    record(st, 4);
    if ((rc = sync(st))) return rc;
    ps->d2h_ms += elapsed_ms(st, 3, 4);
    std::sort(ps->list.begin(), ps->list.end());     // read order, as the host classification leaves it
    res->stats.d2h_bytes += sizeof(PassSummary) + (uint64_t)sum->n_retry * 4;
    res->stats.kernel_launches += n_list ? 1 : 0;
    return 0;
}

// One align pass over ps->list: its buffers (or those pass 0 takes over from k_prepare_exact), k_exact_reads and
// k_align, then the classification of the reads, on the columns route on the device, on the others on the host after
// the download of the headers (and on the record route the heap). The reads that overflowed their arena become
// ps->list, the next pass's reads.
static int run_pass(const Call &c, const Batch &b, const Seeded &sd, const PassPlan &p, int pass, uint32_t scale,
                    int lq, const char *seqs, const uint64_t *offsets, const std::vector<uint64_t> &koff,
                    DevBufs &arena_bufs, DevBufs &heap_bufs, Stream &st, Ticks &tick, PassState *ps, Piece *res) {
    const mgb_index_t *index = c.index;
    const uint32_t k = index->view.k, n_reads = b.n_reads, n_pass = ps->n_pass;
    const bool listed = pass == 0 && sd.prep_exact;      // pass 0 after k_prepare_exact
    const uint64_t heap_cap = listed ? sd.pa.ex.heap_cap : heap_cap_of(b, c.dcfg, k, n_pass, scale);
    char *d_arena = nullptr, *d_heap = nullptr; uint32_t *d_list = nullptr, *d_rest = nullptr;
    unsigned long long *d_used = nullptr; unsigned int *d_next = nullptr;
    int rc;
    if ((rc = arena_bufs.alloc(&d_arena, p.stride * p.n_arenas))) return rc;
    if (listed) {
        d_heap = sd.pa.ex.heap; d_list = sd.pa.list; d_used = sd.pa.ex.heap_used; d_next = sd.next0; d_rest = sd.rest0;
    } else {
        if ((rc = heap_bufs.alloc(&d_heap, heap_cap)) || (rc = heap_bufs.alloc(&d_list, n_pass))
            || (rc = heap_bufs.alloc(&d_used, 1))
            || (rc = heap_bufs.alloc(&d_next, 4))        // k_align's next read and arena; the reads k_exact_reads leaves
            || (sd.exact_reads && (rc = heap_bufs.alloc(&d_rest, n_pass))))
            return rc;
    }
    ps->heap[pass] = d_heap;
    tick("pass: arena/heap alloc");
    if (!listed && ((rc = h2d(d_list, ps->list.data(), (size_t)n_pass * 4, st)) || (rc = dev_zero(d_used, 8, st))
                    || (rc = dev_zero(d_next, 16, st))))
        return rc;
    // only the columns route counts the list in h2d_bytes (the record route's count is the one bench.py reports)
    if (!listed && c.route == Route::columns) res->stats.h2d_bytes += (uint64_t)n_pass * 4;
    // the read-dependent part of the gate (exact_read_strand); max_len keeps what k_align's own exit required
    ExactArgs ea;
    std::memset(&ea, 0, sizeof(ea));
    if (sd.exact_reads) {
        exact_args(b, c.dcfg, k, p.caps, lq, sd.summary, sd.hdr, &ea);
        ea.list = d_list; ea.n_list = n_pass; ea.n_list_dev = listed ? sd.pa.n_list : nullptr;
        ea.rest = d_rest; ea.n_rest = d_next + 1;
        ea.heap = d_heap; ea.heap_cap = heap_cap; ea.heap_used = d_used;
    }
    const bool run_exact = sd.exact_reads && ea.max_len >= k;
    AlignArgs a;
    a.ix = index->view; a.cfg = c.dcfg; a.caps = p.caps; a.lay.carve(p.caps); a.slay = p.slay;
    a.use_fast = std::getenv("MGB_TEST_NOFAST") ? 0 : 1; a.phase_out = nullptr;
#if defined(MGB_PHASE_TIMERS) && !defined(MGB_HOST_EMU)
    unsigned long long *d_phase = nullptr;
    if ((rc = heap_bufs.alloc(&d_phase, 8)) || (rc = dev_zero(d_phase, 64, st))) return rc;
    a.phase_out = d_phase;
#endif
    const SubkArgs &sk = sd.sk;
    a.qf = b.qf; a.qr = b.qr; a.cf = b.cf; a.cr = b.cr; a.offsets = b.offsets; a.koff = b.koff;
    a.nodes_f = b.nodes_f; a.nodes_r = b.nodes_r;
    a.sub_first_f = sd.subk ? sk.first_f : nullptr; a.sub_last_f = sk.last_f; a.sub_len_f = sd.subk ? sk.len_f : nullptr;
    a.sub_first_r = sk.first_r; a.sub_last_r = sk.last_r;
    a.sub_len_r = sd.subk && c.dcfg.forward_and_reverse_complement ? sk.len_r : nullptr;
    a.read_list = d_list; a.n_list = n_pass; a.n_list_dev = nullptr;
    a.arena = d_arena; a.arena_stride = p.stride; a.n_arenas = p.n_arenas;
    a.hdr = sd.hdr; a.heap = d_heap; a.heap_cap = heap_cap; a.heap_used = d_used; a.next = d_next;
    record(st, 3);
    // reads k_align gets (after run_exact: known on the host once the pass is done, or at once when read back)
    uint32_t n_align = a.n_list;
    bool align_dev = false;         // k_align reads the length of its list from the device
    if (run_exact) {
        // k_align takes only the reads left over. On pass 0 it reads their count from the device and the host
        // launches the grid it sized for the whole list without waiting; retry passes read the count back
        // and size the grid by it. MGB_DEBUG reads it back on pass 0 too, for its lines.
        if ((rc = launch_exact_reads(index, ea, st))) return rc;
        align_dev = pass == 0;
        uint32_t n_rest[2] = { 0, 0 };          // and after k_prepare_exact, the length of its list
        if ((!align_dev || tick.on) && ((rc = d2h(n_rest, d_next + 1, listed ? 8 : 4, st)) || (rc = sync(st)))) return rc;
        if (listed && tick.on) debug_exact_counts(c, res->lo, b, koff, seqs, offsets, sd, ea, n_rest, st);
        a.read_list = d_rest;
        if (align_dev) a.n_list_dev = d_next + 1;      // (a.n_list, the whole list's length, bounds it)
        else a.n_list = n_rest[0];
        n_align = n_rest[0];
        res->stats.kernel_launches += 1;
    }
    if ((rc = launch_align(index, a, p, n_align, tick.on, st))) return rc;
    record(st, 4);
    unsigned long long used = 0;
    if ((rc = d2h(&used, d_used, 8, st))) return rc;
    if (align_dev && !tick.on && (rc = d2h(&n_align, d_next + 1, 4, st))) return rc;
    if ((rc = sync(st))) return rc;
    ps->align_ms += elapsed_ms(st, 3, 4);
    record(st, 3);
    tick("pass: h2d+seed+align kernels");
    if (n_align) res->stats.kernel_launches += 1;       // (a k_align over an empty list aligns nothing)
#if defined(MGB_PHASE_TIMERS) && !defined(MGB_HOST_EMU)
    unsigned long long ph[8];
    cudaMemcpy(ph, a.phase_out, 64, cudaMemcpyDeviceToHost);
    std::fprintf(stderr, "[phase cycles/read] setup %.0f seeds %.0f fwd %.0f backtrack %.0f align_total %.0f; columns/read: register path %.1f, general path %.1f (reads %u)\n",
                 (double)ph[0] / n_align, (double)ph[1] / n_align, (double)ph[2] / n_align,
                 (double)ph[3] / n_align, (double)ph[4] / n_align, (double)ph[5] / n_align,
                 (double)ph[6] / n_align, n_align);
#endif
    PassSummary sum = {};
    if (c.route == Route::columns) {
        if ((rc = classify_pass(c, b, sd, pass, listed ? nullptr : d_list, n_pass, heap_bufs, st, ps, &sum, res)))
            return rc;
    } else {
        if (used > heap_cap) used = heap_cap;
        if (c.route == Route::text) used = 0;      // the records stay on the device
        else {
            HostBuf heap_host = hostbuf_acquire((size_t)used + 16);
            tick("pass: host buffer");
            if (!heap_host.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
            res->heaps.push_back(heap_host);
            res->heap_bytes.push_back(used);
            if (used && (rc = d2h(heap_host.p, d_heap, used, st))) return rc;
        }
        if ((rc = d2h(ps->hdr_host, sd.hdr, (size_t)n_reads * sizeof(ReadHdr), st)) || (rc = sync(st))) return rc;
        record(st, 4);
        if ((rc = sync(st))) return rc;
        ps->d2h_ms += elapsed_ms(st, 3, 4);
        res->stats.d2h_bytes += used + (size_t)n_reads * sizeof(ReadHdr);
        tick("pass: d2h");
        if (listed) ps->all_reads(n_reads);
        classify_reads(ClassifyArgs { ps->list.data(), n_pass, ps->hdr_host, offsets, ps->read_heap.data(),
                                      (uint32_t)pass, &sum, ps->list.data() });
        tick("pass: classify");
    }
    mgb_stats_t &s = res->stats;
    s.num_seeds += sum.num_seeds; s.num_extensions += sum.num_extensions; s.num_explored_nodes += sum.num_explored_nodes;
    s.dp_cells += sum.dp_cells; s.dp_columns += sum.dp_columns; s.num_reads_retried += sum.n_retry;
    ps->list.resize(sum.n_retry);
    ps->n_pass = sum.n_retry;
    ps->L_retry = sum.max_retry_len;
    return 0;
}

// record route: mgb_alignment_t records in read order (res->first), from the heaps the passes downloaded
static void materialise(const Call &c, const PassState &ps, Piece *res) {
    const uint32_t n_reads = res->n_reads;
    for (uint32_t r = 0; r < n_reads; ++r) { res->src_off[r] = ps.hdr_host[r].heap_off; res->src_heap[r] = ps.read_heap[r]; }
    #pragma omp parallel for schedule(static) num_threads(host_team()) if (n_reads > 20000)
    for (int64_t r = 0; r < (int64_t)n_reads; ++r)
        unpack_records(res->heaps[res->src_heap[r]].p + res->src_off[r], res->count[r], c.dcfg.result_nodes != 0,
                       res->lo + (uint32_t)r, res->alns + res->first[r]);
}

// What every route runs on one piece of res->n_reads reads (seqs and offsets relative to the piece), after the caller
// has recorded event 0: upload, preparation and seeding, and the align passes until no read overflows its arena. Every
// pass's heap buffers go into the caller's heap_keep, so the heaps can outlive the call; ps comes prepared for the
// route's classification (read_heap and hdr_host, or pass_of).
static int align_piece(const Call &c, const char *seqs, const uint64_t *offsets, CallWorkspace &cw, DevBufs &bufs,
                       std::deque<DevBufs> &heap_keep, Ticks &tick, Batch *b, Seeded *sd, PassState *ps, Piece *res) {
    const uint32_t n_reads = res->n_reads;
    Stream &st = cw.st;
    std::vector<uint64_t> koff;
    int rc = upload_batch(c.index, seqs, offsets, n_reads, c.dcfg.forward_and_reverse_complement, st, bufs, b, &koff,
                          &res->stats, c.dev_input);
    if (rc) return rc;
    tick("upload_batch (host part)");
    // query length k_align stages on chip (0: none; MGB_TEST_LQ: test knob that forces the unstaged path)
    int lq = b->L_max + 1 <= 512 ? (int)((b->L_max + 1 + 15) & ~15u) : 0;
    if (const char *e = std::getenv("MGB_TEST_LQ")) lq = std::atoi(e);
    if ((rc = prepare_and_seed(c, *b, lq, st, bufs, sd, &res->stats))) return rc;

    // align passes: all reads with scale 1, overflowed reads again with larger arenas. Pass 0 after k_prepare_exact
    // takes its list from the device and needs the host's copy of all n_reads only once it is done: filling it first
    // would delay the launches behind it.
    ps->n_pass = n_reads;
    if (!sd->prep_exact) ps->all_reads(n_reads);
    for (int pass = 0; ps->n_pass; ++pass) {
        const uint32_t scale = 1u << (2 * pass);
        if (pass == kMaxPasses) return fail(MGB_ERR_OVERFLOW, "a read exceeded the largest per-read work arena");
        // the arena fits the longest read of the pass: on a retry pass the reads that overflowed, not the batch
        const uint32_t L_pass = pass ? ps->L_retry : b->L_max;
        DevBufs arena_bufs(st, cw.w, kArenaSlots);
        DevBufs &heap_bufs = heap_keep.emplace_back(st, cw.w, c.route == Route::records ? kPassHeapSlots
                                                                                        : kept_heap_slots(pass));
        PassPlan plan;
        if ((rc = pass_plan(c, *b, L_pass, scale, lq, ps->n_pass, arena_bufs, &plan))
            || (rc = run_pass(c, *b, *sd, plan, pass, scale, lq, seqs, offsets, koff, arena_bufs, heap_bufs, st, tick,
                              ps, res)))
            return rc;
    }
    res->stats.h2d_ms = elapsed_ms(st, 0, 1);
    res->stats.seed_kernel_ms = elapsed_ms(st, 1, 2);
    res->stats.align_kernel_ms = ps->align_ms; res->stats.d2h_ms = ps->d2h_ms;
    return MGB_OK;
}

// The record and text routes on one piece of a call: the piece's offsets rebased, its headers uploaded (text route),
// align_piece, then the text rendered on the device or the records materialised on the host.
static int align_range(const Call &c, uint32_t lo, uint32_t n_reads, Piece *res) {
    const mgb_index_t *index = c.index;
    Ticks tick { std::getenv("MGB_DEBUG") != nullptr, lo, n_reads };
    res->lo = lo; res->n_reads = n_reads;
    const bool text = c.route == Route::text;
    // offsets relative to the first character of the piece
    // (device-resident reads: the piece starts at the 16-byte word that holds its first character, as the kernels'
    // word reads assume)
    std::vector<uint64_t> offs_local, name_offs_local;
    const uint64_t base = c.dev_input ? c.offsets[lo] & ~15ull : c.offsets[lo];
    const uint64_t *offsets = rebase_offsets(c.offsets, lo, n_reads, base, &offs_local);
    const char *seqs = c.seqs ? c.seqs + base : nullptr;
    const uint64_t *name_offs = text ? rebase_offsets(c.name_offsets, lo, n_reads, c.name_offsets[lo], &name_offs_local) : nullptr;
    const char *names = text && c.names ? c.names + c.name_offsets[lo] : nullptr;

    CallWorkspace cw(index);
    Stream &st = cw.st;
    int rc = cw.ready();
    if (rc) return rc;
    HostBuf hdr_buf = hostbuf_acquire(((size_t)n_reads + 1) * sizeof(ReadHdr));
    if (!hdr_buf.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
    struct HdrGuard { HostBuf b; ~HdrGuard() { hostbuf_release(b); } } hdr_guard{ hdr_buf };
    PassState ps;
    ps.hdr_host = (ReadHdr*)hdr_buf.p;
    ps.read_heap.assign(n_reads, 0);
    DevBufs bufs(st, cw.w, kBatchSlots), text_bufs(st, cw.w, kTextSlots);
    std::deque<DevBufs> heap_keep;       // the text route keeps every pass's heap until the text is rendered
    record(st, 0);
    tick("setup");
    TextArgs ta;
    std::memset(&ta, 0, sizeof(ta));
    if (text && (rc = upload_headers(c, n_reads, names, name_offs, st, text_bufs, &ta, &res->stats))) return rc;
    Batch b; Seeded sd;
    if ((rc = align_piece(c, seqs, offsets, cw, bufs, heap_keep, tick, &b, &sd, &ps, res))) return rc;
    // each read's records in read order: the last pass's headers hold the count of every read, from the pass that
    // answered it
    uint64_t pos = 0;
    for (uint32_t r = 0; r < n_reads; ++r) { res->count[r] = ps.hdr_host[r].n_aln; res->first[r] = pos; pos += res->count[r]; }
    res->n_alns = pos;
    if (text && n_reads) {      // every read's pass goes up (its heap offset is in sd.hdr already), then the text comes down
        uint8_t *d_pass = nullptr;
        rc = text_bufs.alloc(&d_pass, n_reads);
        if (!rc) rc = h2d(d_pass, ps.read_heap.data(), n_reads, st);
        res->stats.h2d_bytes += n_reads;
        ta.seqs = b.seqs; ta.offsets = b.offsets; ta.hdr = sd.hdr; ta.pass = d_pass;
        std::copy(ps.heap, ps.heap + kMaxPasses, ta.heap);
        if (rc || (rc = render_text(index, ta, text_bufs, st, &res->text, &res->text_bytes, &res->stats))) return rc;
        tick("text");
    }
    tick("free device buffers");
    if (!text) {
        materialise(c, ps, res);
        tick("materialise");
    }
    return MGB_OK;
}

static std::atomic<uint32_t> g_max_pieces{0};      // 0 = automatic
#if defined(MGB_HOST_EMU)
extern "C" { unsigned long long mgb_emu_whole_read_hits = 0, mgb_emu_path_read_hits = 0; unsigned long long mgb_emu_path_hits[EMU_N_PATHS] = {};
             unsigned long long mgb_emu_agg_hits[EMU_N_AGG] = {}; }
#endif

extern "C" {

void mgb_set_pipeline_pieces(uint32_t max_pieces) { g_max_pieces.store(max_pieces); }

void mgb_set_host_threads(int n) {
#if defined(_OPENMP)
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int mgb_config_check(const mgb_index_t *index, const mgb_config_t *config) {
    if (!index || !config) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    DevConfig dcfg;
    std::string err;
    const int rc = lower_config(*config, index->view.k, index->alphabet, &dcfg, &err);
    return rc ? fail(rc, err) : MGB_OK;
}

} // extern "C"

// the configuration of an align call on the device: lower_config, then the graph mode's override
static int call_config(const mgb_index_t *index, const mgb_config_t &config, DevConfig *dcfg) {
    std::string err;
    if (const int rc = lower_config(config, index->view.k, index->alphabet, dcfg, &err)) return fail(rc, err);
    if (index->view.mode != 0) {                  // CANONICAL-mode graph, or a PRIMARY one with CanonicalDBG semantics
        dcfg->canonical = 1;                      // (get_mode() == CANONICAL): both strands, no RCDBG view
        dcfg->forward_and_reverse_complement = 1; // (dbg_aligner.cpp:224-226)
    }
    return MGB_OK;
}

// mgb_align_batch (text_format 0) and mgb_align_batch_text (MGB_TEXT_TSV / MGB_TEXT_JSON, with the headers)
// dev_input: seqs and names are device memory (the file route's parsed chunk), the offsets host memory
static int align_batch(const mgb_index_t *index, const mgb_config_t *config, const char *seqs, const uint64_t *offsets,
                       const char *names, const uint64_t *name_offsets, uint32_t n_reads, int text_format,
                       mgb_results_t **out, bool dev_input = false) {
    DevConfig dcfg;
    if (const int rc = call_config(index, *config, &dcfg)) return rc;
    // the text route: TSV lines print no node ids, so its records carry none; JSON records need them on the device
    if (text_format) dcfg.result_nodes = text_format == MGB_TEXT_TSV ? MGB_NODES_NONE : MGB_NODES_U64;


    // pieces of >= 64k reads, at most 8; two host threads keep two pieces in flight
    const uint32_t kMinPiece = 65536, kMaxPieces = 8;
    uint32_t n_pieces = std::min<uint32_t>(kMaxPieces, n_reads / kMinPiece);
#if defined(MGB_HOST_EMU)
    n_pieces = 1;
#endif
    if (uint32_t cap = g_max_pieces.load()) n_pieces = std::min<uint32_t>(std::max<uint32_t>(n_pieces, 1), cap);
    if (const char *e = std::getenv("MGB_TEST_PIECES")) n_pieces = (uint32_t)std::atoi(e);   // test knob
    if (n_pieces < 1) n_pieces = 1;
    if (n_pieces > n_reads) n_pieces = n_reads ? n_reads : 1;

    const bool dbg_time = std::getenv("MGB_DEBUG") != nullptr;
    const auto t_begin = std::chrono::steady_clock::now();
    auto since = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count(); };

    // every piece writes its records straight into the result arrays: a read has at most
    // num_alternative_paths alignments, so piece i owns the record region starting at lo_i * num_alt
    std::unique_ptr<mgb_results> res(new mgb_results());
    std::memset(&res->stats, 0, sizeof(res->stats));
    res->n_reads = n_reads;
    res->first.assign(n_reads, 0);
    res->count.assign(n_reads, 0);
    res->result_nodes = dcfg.result_nodes;
    res->text_format = text_format;
    const uint64_t num_alt = dcfg.num_alternative_paths;
    if (!text_format) {
        res->src_off.assign(n_reads, 0);
        res->src_heap.assign(n_reads, 0);
        res->alns_buf = hostbuf_acquire(((size_t)n_reads * num_alt + 1) * sizeof(mgb_alignment_t));
        if (!res->alns_buf.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
        res->alns = (mgb_alignment_t*)res->alns_buf.p;
    }

    std::vector<Piece> pieces(n_pieces);
    auto piece_lo = [&](uint32_t i) { return (uint32_t)((uint64_t)n_reads * i / n_pieces); };
    for (uint32_t i = 0; i < n_pieces; ++i) {
        pieces[i].first = res->first.data() + piece_lo(i);
        pieces[i].count = res->count.data() + piece_lo(i);
        if (!text_format) {
            pieces[i].alns = res->alns + (uint64_t)piece_lo(i) * num_alt;
            pieces[i].src_off = res->src_off.data() + piece_lo(i);
            pieces[i].src_heap = res->src_heap.data() + piece_lo(i);
        }
    }
    const Call call { index, dcfg, text_format ? Route::text : Route::records, seqs, offsets, names, name_offsets,
                      text_format, config->min_path_score, dev_input };
    std::atomic<uint32_t> next{0};
    std::atomic<bool> failed{false};
    auto lane = [&]() {
        for (uint32_t i; !failed.load() && (i = next.fetch_add(1)) < n_pieces; ) {
            Piece &pc = pieces[i];
            pc.rc = align_range(call, piece_lo(i), piece_lo(i + 1) - piece_lo(i), &pc);
            if (pc.rc) { pc.err = g_err; failed.store(true); }
        }
    };
    // two host threads keep two pieces in flight (MGB_TEST_LANES: measurement knob)
    uint32_t n_lanes = 2;
    if (const char *e = std::getenv("MGB_TEST_LANES")) n_lanes = std::max(1, std::atoi(e));
    n_lanes = std::min(n_lanes, n_pieces);
    std::vector<std::thread> others;
    for (uint32_t t = 1; t < n_lanes; ++t) others.emplace_back(lane);
    lane();
    for (std::thread &t : others) t.join();
    for (Piece &pc : pieces)
        if (pc.rc) return fail(pc.rc, pc.err);
    if (dbg_time) std::fprintf(stderr, "[mgb] %u pieces done at %.2f ms\n", n_pieces, since());

    // close the gaps between the regions (none if every read produced num_alt alignments)
    uint64_t total = 0;
    for (uint32_t i = 0; i < n_pieces; ++i) {
        Piece &pc = pieces[i];
        const uint64_t region = (uint64_t)pc.lo * num_alt;
        if (!text_format && total != region) {
            std::memmove(res->alns + total, res->alns + region, pc.n_alns * sizeof(mgb_alignment_t));
        }
        if (total) {
            const int64_t n = pc.n_reads;
            #pragma omp parallel for schedule(static) num_threads(host_team()) if (n > 50000)
            for (int64_t r = 0; r < n; ++r) pc.first[r] += total;
        }
        total += pc.n_alns;
        {   // heap ids of the piece become ids in the merged list
            const uint32_t base = (uint32_t)res->heaps.size();
            if (base) for (uint32_t r = 0; r < pc.n_reads; ++r) pc.src_heap[r] += base;
        }
        for (HostBuf b : pc.heaps) res->heaps.push_back(b);
        for (uint64_t b : pc.heap_bytes) res->heap_bytes.push_back(b);
        pc.heaps.clear();
        add_stats(res->stats, pc.stats);
    }
    res->n_alns = total;
    if (text_format) {
        // the pieces' blocks in piece order: one piece hands its buffer over, several are copied into one block
        uint64_t bytes = 0;
        for (Piece &pc : pieces) bytes += pc.text_bytes;
        if (n_pieces == 1 && pieces[0].text.p) {
            res->text = pieces[0].text; pieces[0].text = HostBuf();
        } else {
            res->text = hostbuf_acquire(bytes);
            if (!res->text.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
            uint64_t at = 0;
            for (Piece &pc : pieces) {
                parallel_copy(res->text.p + at, pc.text.p, pc.text_bytes);
                at += pc.text_bytes;
            }
        }
        res->text_bytes = bytes;
    }
    if (dbg_time) std::fprintf(stderr, "[mgb] merged at %.2f ms\n", since());
    *out = res.release();
    return MGB_OK;
}

extern "C" {

int mgb_align_batch(const mgb_index_t *index, const mgb_config_t *config, const char *seqs,
                    const uint64_t *offsets, uint32_t n_reads, mgb_results_t **out) {
    if (!index || !config || !offsets || !out || (!seqs && n_reads && offsets[n_reads]))
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    return align_batch(index, config, seqs, offsets, nullptr, nullptr, n_reads, 0, out);
}

int mgb_align_batch_text(const mgb_index_t *index, const mgb_config_t *config, const char *seqs,
                         const uint64_t *offsets, const char *headers, const uint64_t *header_offsets,
                         uint32_t n_reads, int format, mgb_results_t **out) {
    if (!index || !config || !offsets || !out || (!seqs && n_reads && offsets[n_reads]))
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (format != MGB_TEXT_TSV && format != MGB_TEXT_JSON)
        return fail(MGB_ERR_INVALID_ARGUMENT, "format must be MGB_TEXT_TSV or MGB_TEXT_JSON");
    if (!header_offsets || (!headers && n_reads && header_offsets[n_reads]))
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    for (uint32_t r = 0; r < n_reads; ++r)
        if (header_offsets[r + 1] < header_offsets[r]) return fail(MGB_ERR_INVALID_ARGUMENT, "header offsets must be non-decreasing");
    return align_batch(index, config, seqs, offsets, headers, header_offsets, n_reads, format, out);
}

// the chunk's records on the device route, or the host restatement's when the device route refuses the chunk
// (or device_route is false); *parse: the file route's own copies and launches
static int fastx_parse(const mgb_index_t *index, const char *buf, uint64_t bytes, bool at_eof, const char *delim,
                       bool fwd_rev, bool device_route, Stream &st, DevBufs &bufs, FastxDev *dev, FastxRecords *host,
                       uint64_t *consumed, int *ended, mgb_stats_t *parse) {
    *consumed = 0; *ended = 0;
    dev->refused = !device_route;
    if (device_route) {
        const int rc = fastx_parse_dev(index, buf, bytes, at_eof, delim, fwd_rev, st, bufs, dev, parse);
        if (rc) return rc;
    }
    if (dev->refused) fastx_parse_host(buf, bytes, at_eof, delim, fwd_rev, host, consumed, ended);
    else *consumed = dev->consumed;
    return MGB_OK;
}

} // extern "C"

// ---------------------------------------------------------------------------------------
// device-resident batches (mgb_align_batch_device), the columns route: align_piece on reads already in device memory,
// one piece on one stream; the records stay in the pass heaps, which the handle holds, until the caller's columns are
// written (columns_core.cuh)
// ---------------------------------------------------------------------------------------
struct mgb_device_results {
    explicit mgb_device_results(const mgb_index_t *ix) : cw(ix) {}
    ~mgb_device_results();
    CallWorkspace cw;                 // the working memory the columns are read from, held until the handle is freed
    std::deque<DevBufs> bufs;         // the batch's buffers, every pass's heap and the columns' counts
    ColumnsArgs ca;
    mgb_device_sizes_t sizes;
    mgb_stats_t stats;
#if !defined(MGB_HOST_EMU)
    mutable cudaEvent_t written = nullptr;     // recorded after the last mgb_device_results_write
#endif
};

mgb_device_results::~mgb_device_results() {
#if !defined(MGB_HOST_EMU)
    if (written) { cudaEventSynchronize(written); cudaEventDestroy(written); }
#endif
}

#if !defined(MGB_HOST_EMU)
static bool on_device(const void *p, int device) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == device;
}
#endif

static int align_device(const mgb_index_t *index, const mgb_config_t *config, const char *d_seqs, const uint64_t *offsets,
                        bool offsets_on_device, uint32_t n_reads, void *stream, mgb_device_results *res) {
    DevConfig dcfg;
    int rc = call_config(index, *config, &dcfg);
    if (rc) return rc;
    Piece piece;
    piece.n_reads = n_reads;
    mgb_stats_t &stats = piece.stats;
    CallWorkspace &cw = res->cw;
    if ((rc = cw.ready())) return rc;
    Stream &st = cw.st;
#if !defined(MGB_HOST_EMU)
    if ((d_seqs && !on_device(d_seqs, index->device)) || (offsets_on_device && !on_device(offsets, index->device)))
        return fail(MGB_ERR_INVALID_ARGUMENT, "the reads (and device offsets) must be device memory on the index's device");
    {   // the caller's work queued on its stream comes first
        cudaEvent_t ev;
        CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        cudaError_t e = cudaEventRecord(ev, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(st.s, ev, 0);
        cudaEventDestroy(ev);
        CUDA_TRY(e);
    }
#else
    (void)stream;
#endif
    record(st, 0);
    // the offsets on the host, relative to the first read (upload_batch checks them)
    std::vector<uint64_t> offs((size_t)n_reads + 1);
    if (offsets_on_device) {
        if ((rc = d2h(offs.data(), offsets, offs.size() * 8, st)) || (rc = sync(st))) return rc;
        stats.d2h_bytes += offs.size() * 8;
    } else {
        std::memcpy(offs.data(), offsets, offs.size() * 8);
    }
    const uint64_t base = offs[0];
    if (offs[n_reads] < base) return fail(MGB_ERR_INVALID_ARGUMENT, "offsets must be non-decreasing");
    const uint64_t chars = offs[n_reads] - base;
    if (!d_seqs && chars) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    for (uint64_t &o : offs) o -= base;
    // The reads are copied into the batch's own buffer first: k_prepare_exact's word loads and the other kernels' reads
    // past a read's end assume a 16-byte-aligned base and 64 bytes of slack, which a caller's buffer need not have.
    DevBufs &bufs = res->bufs.emplace_back(st, cw.w, kBatchSlots);
    char *seqs = nullptr;
    if ((rc = bufs.alloc(&seqs, chars + 64))) return rc;
#if defined(MGB_HOST_EMU)
    if (chars) std::memcpy(seqs, d_seqs + base, chars);
#else
    if (chars) CUDA_TRY(cudaMemcpyAsync(seqs, d_seqs + base, chars, cudaMemcpyDeviceToDevice, st.s));
#endif
    DevBufs &cb = res->bufs.emplace_back(st, cw.w, kTextSlots);
    PassState ps;
    if ((rc = cb.alloc(&ps.pass_of, (size_t)n_reads + 1))) return rc;
    const Call c { index, dcfg, Route::columns, seqs, offs.data(), nullptr, nullptr, 0, config->min_path_score, true };
    Ticks tick { std::getenv("MGB_DEBUG") != nullptr, 0, n_reads };
    Batch b; Seeded sd;
    if ((rc = align_piece(c, seqs, offs.data(), cw, bufs, res->bufs, tick, &b, &sd, &ps, &piece))) return rc;

    // every read's alignments, sequence bytes, CIGAR ops and node ids; their scans; the totals come down
    ColumnsArgs &ca = res->ca;
    std::memset(&ca, 0, sizeof(ca));
    ca.hdr = sd.hdr; ca.pass_of = ps.pass_of;
    std::copy(ps.heap, ps.heap + kMaxPasses, ca.heap);
    ca.n_reads = n_reads; ca.no_nodes = dcfg.result_nodes != 0;
    for (uint64_t *&x : ca.cnt) if ((rc = cb.alloc(&x, (size_t)n_reads + 1))) return rc;
#if defined(MGB_HOST_EMU)
    for (uint32_t r = 0; r < n_reads; ++r) columns_size_read(ca, r);
#else
    if (n_reads) {
        const unsigned grid = (unsigned)kern_dna::read_path_grid(std::min<uint64_t>((n_reads + 7) / 8, (uint64_t)index->num_sms * 16));
        kern_dna::log_launch("k_columns_size", grid, 256, (uint64_t)grid * 8, n_reads);     // a warp per read
        k_columns_size<<<grid, 256, 0, st.s>>>(ca);
        CUDA_TRY(cudaGetLastError());
    }
#endif
    for (uint64_t *x : ca.cnt) if ((rc = scan_u64(x, n_reads, st, cb))) return rc;
    uint64_t tot[4];
    for (int i = 0; i < 4; ++i) if ((rc = d2h(&tot[i], ca.cnt[i] + n_reads, 8, st))) return rc;
    if ((rc = sync(st))) return rc;
    stats.d2h_bytes += sizeof(tot);
    stats.kernel_launches += (n_reads ? 1 : 0) + 4 * (n_reads ? 3 : 2);
    res->sizes = mgb_device_sizes_t { n_reads, tot[0], tot[1], tot[2], tot[3] };
    res->stats = stats;
    return MGB_OK;
}

extern "C" {

int mgb_align_batch_device(const mgb_index_t *index, const mgb_config_t *config, const char *d_seqs,
                           const uint64_t *offsets, int offsets_on_device, uint32_t n_reads, void *stream,
                           mgb_device_results_t **out) {
    if (!index || !config || !offsets || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    std::unique_ptr<mgb_device_results> res(new mgb_device_results(index));
    if (const int rc = align_device(index, config, d_seqs, offsets, offsets_on_device != 0, n_reads, stream, res.get()))
        return rc;
    *out = res.release();
    return MGB_OK;
}

int mgb_device_results_sizes(const mgb_device_results_t *res, mgb_device_sizes_t *sizes) {
    if (!res || !sizes) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    *sizes = res->sizes;
    return MGB_OK;
}

const mgb_stats_t *mgb_device_results_stats(const mgb_device_results_t *res) { return res ? &res->stats : nullptr; }

int mgb_device_results_write(const mgb_device_results_t *res, const mgb_device_columns_t *dst, void *stream) {
    if (!res || !dst) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    const mgb_device_sizes_t &z = res->sizes;
    const mgb_device_columns_t &d = *dst;
    if (!d.read_first || !d.sequence_offsets || !d.cigar_offsets || !d.node_offsets
        || (z.n_alignments && (!d.read_index || !d.orientation || !d.score || !d.offset || !d.query_begin || !d.query_len
                               || !d.num_nodes || !d.sequence_len || !d.num_cigar_ops))
        || (z.sequence_bytes && !d.sequence) || (z.cigar_ops && !d.cigar) || (z.nodes && !d.nodes))
        return fail(MGB_ERR_INVALID_ARGUMENT, "a column with at least one element has a null pointer");
    ColumnsArgs a = res->ca;
    a.dst = d;
#if defined(MGB_HOST_EMU)
    (void)stream;
    columns_write_ends(a);
    for (uint32_t r = 0; r < a.n_reads; ++r) columns_write_read(a, r);
#else
    const mgb_index_t *index = res->cw.ix;
    CUDA_TRY(cudaSetDevice(index->device));
    const unsigned grid = (unsigned)std::max<uint64_t>(1, kern_dna::read_path_grid(
        std::min<uint64_t>((a.n_reads + 7) / 8, (uint64_t)index->num_sms * 16)));
    kern_dna::log_launch("k_columns_write", grid, 256, (uint64_t)grid * 8, a.n_reads);     // a warp per read
    k_columns_write<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    if (!res->written) CUDA_TRY(cudaEventCreateWithFlags(&res->written, cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(res->written, (cudaStream_t)stream));
#endif
    return MGB_OK;
}

void mgb_device_results_free(mgb_device_results_t *res) { delete res; }

} // extern "C"

// A chunk's records between mgb_fastx_stage and mgb_align_fastx_batch_text: the stage's workspace (its "batch" region
// holds the parsed arrays on the device) and stream, the host restatement's records for a refused chunk, and the
// parse's own copies and launches, which the result set reports. A BGZF stage also keeps the text the host holds: the
// whole text when the host restatement parsed it, else text[consumed, end); the tail starts at tail_at.
struct mgb_fastx_batch {
    CallWorkspace cw;
    DevBufs bufs;
    FastxDev dev;
    FastxRecords host;
    mgb_stats_t parse;
    std::vector<char> text;
    uint64_t tail_at = 0;
    explicit mgb_fastx_batch(const mgb_index_t *index) : cw(index), bufs(cw.st, cw.w, kBatchSlots) {
        std::memset(&parse, 0, sizeof(parse));
    }
};

// The records of a compressed stage's text d_text[0, text_bytes) (device memory of fastx_text_bytes(text_bytes)
// bytes; last: its last byte) parsed into batch b, which keeps text[consumed, end) for the next stage's head (the whole
// text when the host restatement parses it).
static int stage_text(const mgb_index_t *index, mgb_fastx_batch *b, const uint8_t *d_text, uint64_t text_bytes,
                      uint8_t last, bool at_eof, const char *comment_delim, bool fwd_rev, uint64_t *consumed,
                      int *ended) {
    Stream &st = b->cw.st;
    int rc;
    *consumed = 0; *ended = 0;
    if ((rc = fastx_parse_text(index, d_text, text_bytes, last, at_eof, comment_delim, fwd_rev, st, b->bufs, &b->dev,
                               &b->parse)))
        return rc;
    if (b->dev.refused) {            // the host restatement parses the inflated text
        b->text.resize(text_bytes);
        if ((text_bytes && (rc = d2h(b->text.data(), d_text, text_bytes, st))) || (rc = sync(st))) return rc;
        b->parse.d2h_bytes += text_bytes;
        fastx_parse_host(b->text.data(), text_bytes, at_eof, comment_delim, fwd_rev, &b->host, consumed, ended);
        b->tail_at = *consumed;
    } else {
        *consumed = b->dev.consumed;
        b->text.resize(text_bytes - *consumed);
        if ((b->text.size() && (rc = d2h(b->text.data(), d_text + *consumed, b->text.size(), st))) || (rc = sync(st)))
            return rc;
        b->parse.d2h_bytes += b->text.size();
    }
    const std::vector<uint64_t> &offs = b->dev.refused ? b->host.offsets : b->dev.offsets;
    if (offs.size() - 1 > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "more than 2^32 - 1 records in one chunk");
    return MGB_OK;
}

extern "C" {

int mgb_fastx_stage(const mgb_index_t *index, const char *buf, uint64_t bytes, int at_eof, const char *comment_delim,
                    int flags, uint64_t *consumed, int *ended, mgb_fastx_batch_t **out) {
    if (!index || !consumed || !ended || !out || (!buf && bytes)) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (flags & ~MGB_FASTX_FWD_AND_REVERSE) return fail(MGB_ERR_INVALID_ARGUMENT, "unknown flags");
    std::unique_ptr<mgb_fastx_batch> b(new mgb_fastx_batch(index));
    int rc = b->cw.ready();
    if (rc) return rc;
    rc = fastx_parse(index, buf, bytes, at_eof != 0, comment_delim, (flags & MGB_FASTX_FWD_AND_REVERSE) != 0, true,
                     b->cw.st, b->bufs, &b->dev, &b->host, consumed, ended, &b->parse);
    if (rc) return rc;
    const std::vector<uint64_t> &offs = b->dev.refused ? b->host.offsets : b->dev.offsets;
    if (offs.size() - 1 > 0xffffffffull) return fail(MGB_ERR_OVERFLOW, "more than 2^32 - 1 records in one chunk");
    *out = b.release();
    return MGB_OK;
}

int mgb_align_fastx_batch_text(const mgb_index_t *index, const mgb_config_t *config, mgb_fastx_batch_t *batch,
                               int format, mgb_results_t **out) {
    std::unique_ptr<mgb_fastx_batch> b(batch);
    if (!index || !config || !batch || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (b->cw.ix != index) return fail(MGB_ERR_INVALID_ARGUMENT, "the batch was staged on another index");
    if (format != MGB_TEXT_TSV && format != MGB_TEXT_JSON)
        return fail(MGB_ERR_INVALID_ARGUMENT, "format must be MGB_TEXT_TSV or MGB_TEXT_JSON");
    const FastxDev &dev = b->dev;
    const FastxRecords &host = b->host;
    const std::vector<uint64_t> &offs = dev.refused ? host.offsets : dev.offsets;
    const uint32_t n = (uint32_t)(offs.size() - 1);
    const int rc = dev.refused ? align_batch(index, config, host.seqs.data(), host.offsets.data(), host.names.data(),
                                             host.name_offsets.data(), n, format, out)
                               : align_batch(index, config, dev.seqs, dev.offsets.data(), dev.names,
                                             dev.name_offsets.data(), n, format, out, true);
    if (rc) return rc;
    add_stats((*out)->stats, b->parse);
    return MGB_OK;
}

void mgb_fastx_batch_free(mgb_fastx_batch_t *batch) { delete batch; }

int mgb_fastx_stage_bgzf(const mgb_index_t *index, const char *head, uint64_t head_bytes, const uint8_t *cbuf,
                         uint64_t cbytes, int c_eof, uint64_t max_text, const char *comment_delim, int flags,
                         uint64_t *c_consumed, int *c_refused, uint64_t *consumed, int *ended,
                         mgb_fastx_batch_t **out) {
    if (!index || !c_consumed || !c_refused || !consumed || !ended || !out || (!head && head_bytes) || (!cbuf && cbytes))
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (flags & ~MGB_FASTX_FWD_AND_REVERSE) return fail(MGB_ERR_INVALID_ARGUMENT, "unknown flags");
    const bool fwd_rev = (flags & MGB_FASTX_FWD_AND_REVERSE) != 0;
    std::unique_ptr<mgb_fastx_batch> b(new mgb_fastx_batch(index));
    int rc = b->cw.ready();
    if (rc) return rc;
    BgzfWalk w;
    bgzf_walk(cbuf, cbytes, c_eof != 0, max_text, &w);
    uint8_t *d_text = nullptr, last = 0;
    uint64_t text_bytes = 0, n_ok = 0;
    if ((rc = bgzf_inflate_dev(index, cbuf, w, head, head_bytes, b->cw.st, b->bufs, &d_text, &text_bytes, &n_ok, &last,
                               &b->parse)))
        return rc;
    const bool at_eof = c_eof && w.c_end == cbytes && !w.refused;
    if ((rc = stage_text(index, b.get(), d_text, text_bytes, last, at_eof, comment_delim, fwd_rev, consumed, ended)))
        return rc;
    *c_consumed = w.c_end;
    *c_refused = w.refused ? 1 : 0;
    *out = b.release();
    return MGB_OK;
}

int mgb_gzip_stream_create(mgb_gzip_stream_t **out) {
    if (!out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    *out = new mgb_gzip_stream();
    return MGB_OK;
}

void mgb_gzip_stream_free(mgb_gzip_stream_t *stream) { delete stream; }

int mgb_gzip_stream_state(const mgb_gzip_stream_t *stream, int *in_member, uint64_t *member_text) {
    if (!stream || !in_member || !member_text) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    *in_member = stream->in_member ? 1 : 0;
    *member_text = stream->in_member ? stream->member_text : 0;
    return MGB_OK;
}

// Relocatable form of a gzip stream (what the token carries between processes): header, then the 32 KiB window.
namespace {
struct GzipStreamHdr { uint64_t magic; uint32_t in_member, bit; uint64_t member_text; uint32_t crc, window;
                       uint64_t c_bits, text; };
const uint64_t kGzipStreamMagic = 0x314d525453475a47ull;     // "GZGSTRM1"
}
uint64_t mgb_gzip_stream_export_bytes(const mgb_gzip_stream_t *stream) {
    (void)stream;
    return sizeof(GzipStreamHdr) + kGzipWindow;
}
int mgb_gzip_stream_export(const mgb_gzip_stream_t *s, void *dst, uint64_t capacity) {
    if (!s || !dst) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (capacity < mgb_gzip_stream_export_bytes(s)) return fail(MGB_ERR_INVALID_ARGUMENT, "export buffer too small");
    GzipStreamHdr h { kGzipStreamMagic, s->in_member ? 1u : 0u, s->bit, s->member_text, s->crc, kGzipWindow,
                      s->c_bits, s->text };
    std::memcpy(dst, &h, sizeof(h));
    std::memcpy((char*)dst + sizeof(h), s->window.data(), kGzipWindow);
    return MGB_OK;
}
int mgb_gzip_stream_import(const void *block, uint64_t bytes, mgb_gzip_stream_t **out) {
    if (!block || !out) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    GzipStreamHdr h;
    if (bytes < sizeof(h)) return fail(MGB_ERR_INVALID_ARGUMENT, "bad gzip stream block");
    std::memcpy(&h, block, sizeof(h));
    if (h.magic != kGzipStreamMagic || h.window != kGzipWindow || bytes < sizeof(h) + kGzipWindow || h.in_member > 1
        || h.bit > 7)
        return fail(MGB_ERR_INVALID_ARGUMENT, "bad gzip stream block");
    std::unique_ptr<mgb_gzip_stream> s(new mgb_gzip_stream());
    s->in_member = h.in_member != 0; s->bit = h.bit; s->member_text = h.member_text; s->crc = h.crc;
    s->c_bits = h.c_bits; s->text = h.text;
    std::memcpy(s->window.data(), (const char*)block + sizeof(h), kGzipWindow);
    *out = s.release();
    return MGB_OK;
}

int mgb_fastx_stage_gzip(const mgb_index_t *index, mgb_gzip_stream_t *stream, const char *head, uint64_t head_bytes,
                         const uint8_t *cbuf, uint64_t cbytes, int c_eof, uint64_t max_text, const char *comment_delim,
                         int flags, uint64_t *c_consumed, int *c_refused, uint64_t *consumed, int *ended,
                         mgb_fastx_batch_t **out) {
    if (!index || !stream || !c_consumed || !c_refused || !consumed || !ended || !out || (!head && head_bytes)
        || (!cbuf && cbytes))
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (flags & ~MGB_FASTX_FWD_AND_REVERSE) return fail(MGB_ERR_INVALID_ARGUMENT, "unknown flags");
    std::unique_ptr<mgb_fastx_batch> b(new mgb_fastx_batch(index));
    int rc = b->cw.ready();
    if (rc) return rc;
    uint8_t *d_text = nullptr, last = 0;
    GzipStage g;
    GzipCounts counts;
    if ((rc = gzip_stage_dev(index, stream, cbuf, cbytes, c_eof != 0, max_text, kGzipSubBytes, nullptr, true, head,
                             head_bytes, b->cw.st, b->bufs, &d_text, &last, &g, &counts, &b->parse)))
        return rc;
    const bool at_eof = c_eof && g.c_used == cbytes && !g.refused && !stream->in_member;
    if ((rc = stage_text(index, b.get(), d_text, head_bytes + g.text, last, at_eof, comment_delim,
                         (flags & MGB_FASTX_FWD_AND_REVERSE) != 0, consumed, ended)))
        return rc;
    *c_consumed = g.c_used;
    *c_refused = g.refused ? 1 : 0;
    *out = b.release();
    return MGB_OK;
}

int mgb_gzip_inflate(const mgb_index_t *index, const uint8_t *cbuf, uint64_t cbytes, int c_eof, uint64_t sub_bytes,
                     const uint64_t *cands, uint64_t n_cands, char *out, uint64_t out_cap, uint64_t *out_bytes,
                     uint64_t *c_consumed, int *refused, uint64_t *counts) {
    if (!index || (!cbuf && cbytes) || (!cands && n_cands) || (!out && out_cap) || !out_bytes || !c_consumed
        || !refused || !counts)
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    CallWorkspace cw(index);
    int rc = cw.ready();
    if (rc) return rc;
    mgb_stats_t stats;
    std::memset(&stats, 0, sizeof(stats));
    mgb_gzip_stream s;
    GzipCounts cnt;
    std::vector<char> text;
    uint64_t at = 0;
    bool ref = false;
    for (;;) {
        std::vector<uint64_t> inject;
        for (uint64_t i = 0; i < n_cands; ++i) if (cands[i] >= at * 8) inject.push_back(cands[i] - at * 8);
        DevBufs bufs(cw.st, cw.w, kBatchSlots);
        uint8_t *d_text = nullptr, last = 0;
        GzipStage g;
        if ((rc = gzip_stage_dev(index, &s, cbuf + at, cbytes - at, c_eof != 0, UINT64_MAX,
                                 sub_bytes ? sub_bytes : kGzipSubBytes, cands ? &inject : nullptr, false, nullptr, 0,
                                 cw.st,
                                 bufs, &d_text, &last, &g, &cnt, &stats)))
            return rc;
        if (g.text) {
            text.resize(text.size() + g.text);
            if ((rc = d2h(text.data() + text.size() - g.text, d_text, g.text, cw.st)) || (rc = sync(cw.st))) return rc;
        }
        at += g.c_used;
        ref = g.refused;
        if (ref || (!g.c_used && !g.member_end)) break;
    }
    counts[0] = cnt.n_sub; counts[1] = cnt.found; counts[2] = cnt.confirmed;
    *out_bytes = text.size();
    *c_consumed = at;
    *refused = ref ? 1 : 0;
    if (text.size() > out_cap) return fail(MGB_ERR_OVERFLOW, "output buffer too small");
    if (text.size()) std::memcpy(out, text.data(), text.size());
    return MGB_OK;
}

int mgb_fastx_batch_tail(const mgb_fastx_batch_t *batch, const char **tail, uint64_t *bytes) {
    if (!batch || !tail || !bytes) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    *tail = batch->text.data() + batch->tail_at;
    *bytes = batch->text.size() - batch->tail_at;
    return MGB_OK;
}

int mgb_bgzf_inflate(const mgb_index_t *index, const uint8_t *cbuf, uint64_t cbytes, int c_eof, char *out,
                     uint64_t out_cap, uint64_t *out_bytes, uint64_t *c_consumed, uint64_t *n_blocks, int *refused) {
    if (!index || (!cbuf && cbytes) || (!out && out_cap) || !out_bytes || !c_consumed || !n_blocks || !refused)
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    CallWorkspace cw(index);
    int rc = cw.ready();
    if (rc) return rc;
    DevBufs bufs(cw.st, cw.w, kBatchSlots);
    mgb_stats_t stats;
    std::memset(&stats, 0, sizeof(stats));
    BgzfWalk w;
    bgzf_walk(cbuf, cbytes, c_eof != 0, UINT64_MAX, &w);
    uint8_t *d_text = nullptr, last = 0;
    uint64_t text_bytes = 0, n_ok = 0;
    if ((rc = bgzf_inflate_dev(index, cbuf, w, nullptr, 0, cw.st, bufs, &d_text, &text_bytes, &n_ok, &last, &stats)))
        return rc;
    if (text_bytes > out_cap) return fail(MGB_ERR_OVERFLOW, "output buffer too small");
    if ((text_bytes && (rc = d2h(out, d_text, text_bytes, cw.st))) || (rc = sync(cw.st))) return rc;
    *out_bytes = text_bytes;
    *c_consumed = w.c_end;
    *n_blocks = n_ok;
    *refused = w.refused ? 1 : 0;
    return MGB_OK;
}

int mgb_align_fastx_text(const mgb_index_t *index, const mgb_config_t *config, const char *buf, uint64_t bytes,
                         int at_eof, const char *comment_delim, int flags, int format, uint64_t *consumed, int *ended,
                         mgb_results_t **out) {
    if (!index || !config || !consumed || !ended || !out || (!buf && bytes)) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (format != MGB_TEXT_TSV && format != MGB_TEXT_JSON)
        return fail(MGB_ERR_INVALID_ARGUMENT, "format must be MGB_TEXT_TSV or MGB_TEXT_JSON");
    mgb_fastx_batch_t *batch = nullptr;
    const int rc = mgb_fastx_stage(index, buf, bytes, at_eof, comment_delim, flags, consumed, ended, &batch);
    return rc ? rc : mgb_align_fastx_batch_text(index, config, batch, format, out);
}

int mgb_fastx_parse(const mgb_index_t *index, const char *buf, uint64_t bytes, int at_eof, const char *comment_delim,
                    int flags, int device_route, char *seqs, uint64_t max_seq_bytes, uint64_t *offsets, char *names,
                    uint64_t max_name_bytes, uint64_t *name_offsets, uint64_t max_records, uint64_t *n_records,
                    uint64_t *consumed, int *ended, int *refused) {
    if ((device_route && !index) || (!buf && bytes) || !seqs || !offsets || !names || !name_offsets || !n_records
        || !consumed || !ended || !refused)
        return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (flags & ~MGB_FASTX_FWD_AND_REVERSE) return fail(MGB_ERR_INVALID_ARGUMENT, "unknown flags");
    FastxDev dev;
    FastxRecords host;
    mgb_stats_t parse;
    std::memset(&parse, 0, sizeof(parse));
    const bool fwd_rev = flags & MGB_FASTX_FWD_AND_REVERSE;
    auto fits = [&](const std::vector<uint64_t> &o, const std::vector<uint64_t> &no) {
        return o.size() - 1 <= max_records && o.back() <= max_seq_bytes && no.back() <= max_name_bytes;
    };
    if (!device_route) {
        Stream st;
        DevBufs none(st, nullptr, kBatchSlots);
        fastx_parse(index, buf, bytes, at_eof != 0, comment_delim, fwd_rev, false, st, none, &dev, &host, consumed,
                    ended, &parse);
    } else {
        CallWorkspace cw(index);
        int rc = cw.ready();
        if (rc) return rc;
        DevBufs bufs(cw.st, cw.w, kBatchSlots);
        if ((rc = fastx_parse(index, buf, bytes, at_eof != 0, comment_delim, fwd_rev, true, cw.st, bufs, &dev, &host,
                              consumed, ended, &parse)))
            return rc;
        if (!dev.refused) {
            if (!fits(dev.offsets, dev.name_offsets)) return fail(MGB_ERR_OVERFLOW, "output arrays too small");
            if ((rc = d2h(seqs, dev.seqs, dev.offsets.back(), cw.st))) return rc;
            if ((rc = d2h(names, dev.names, dev.name_offsets.back(), cw.st)) || (rc = sync(cw.st))) return rc;
            std::memcpy(offsets, dev.offsets.data(), dev.offsets.size() * 8);
            std::memcpy(name_offsets, dev.name_offsets.data(), dev.name_offsets.size() * 8);
            *n_records = dev.offsets.size() - 1;
            *refused = 0;
            return MGB_OK;
        }
    }
    *refused = device_route ? 1 : 0;
    if (!fits(host.offsets, host.name_offsets)) return fail(MGB_ERR_OVERFLOW, "output arrays too small");
    std::memcpy(seqs, host.seqs.data(), host.seqs.size());
    std::memcpy(names, host.names.data(), host.names.size());
    std::memcpy(offsets, host.offsets.data(), host.offsets.size() * 8);
    std::memcpy(name_offsets, host.name_offsets.data(), host.name_offsets.size() * 8);
    *n_records = host.offsets.size() - 1;
    return MGB_OK;
}

int mgb_results_text(const mgb_results_t *results, const char **text, uint64_t *bytes) {
    if (!results || !text || !bytes) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (!results->text_format) return fail(MGB_ERR_INVALID_ARGUMENT, "not a text result set (mgb_align_batch_text)");
    *text = results->text.p ? results->text.p : "";
    *bytes = results->text_bytes;
    return MGB_OK;
}

// Relocatable form of a result set (what a rank ships to rank 0, SURVEY 8e): header, per-read record counts and
// positions, then the packed records exactly as the kernel wrote them (OutAln | nodes | cigar | sequence).
namespace {
struct ExportHdr { uint64_t magic, n_reads, n_alns, n_heaps, result_nodes, total_bytes; };
const uint64_t kExportMagic = 0x3142474d53455231ull;      // "1RESMGB1"
}
uint64_t mgb_results_export_bytes(const mgb_results_t *r) {
    if (r->text_format) return 0;                // a text result set has no records to export
    uint64_t b = sizeof(ExportHdr) + (uint64_t)r->n_reads * (8 + 4 + 4) + 8 * r->heap_bytes.size();
    b = (b + 15) & ~15ull;
    for (uint64_t h : r->heap_bytes) b += (h + 15) & ~15ull;
    return b;
}
int mgb_results_export(const mgb_results_t *r, void *dst, uint64_t capacity) {
    if (!r || !dst) return fail(MGB_ERR_INVALID_ARGUMENT, "null argument");
    if (r->text_format) return fail(MGB_ERR_INVALID_ARGUMENT, "a text result set (mgb_align_batch_text) has no records to export");
    const uint64_t total = mgb_results_export_bytes(r);
    if (capacity < total) return fail(MGB_ERR_INVALID_ARGUMENT, "export buffer too small");
    char *p = (char*)dst;
    ExportHdr h { kExportMagic, r->n_reads, r->n_alns, r->heap_bytes.size(), r->result_nodes, total };
    std::memcpy(p, &h, sizeof(h)); p += sizeof(h);
    std::memcpy(p, r->src_off.data(), 8ull * r->n_reads); p += 8ull * r->n_reads;
    std::memcpy(p, r->count.data(), 4ull * r->n_reads); p += 4ull * r->n_reads;
    std::memcpy(p, r->src_heap.data(), 4ull * r->n_reads); p += 4ull * r->n_reads;
    std::memcpy(p, r->heap_bytes.data(), 8 * r->heap_bytes.size()); p += 8 * r->heap_bytes.size();
    p = (char*)dst + (((uint64_t)(p - (char*)dst) + 15) & ~15ull);
    for (size_t i = 0; i < r->heaps.size(); ++i) {
        parallel_copy(p, r->heaps[i].p, r->heap_bytes[i]);
        p += (r->heap_bytes[i] + 15) & ~15ull;
    }
    return MGB_OK;
}
int mgb_results_import(const void *blob, uint64_t bytes, uint32_t read_index_base, mgb_results_t **out) {
    if (!blob || !out || bytes < sizeof(ExportHdr)) return fail(MGB_ERR_INVALID_ARGUMENT, "bad export blob");
    ExportHdr h; std::memcpy(&h, blob, sizeof(h));
    if (h.magic != kExportMagic || h.total_bytes > bytes || h.n_reads > 0xffffffffull)
        return fail(MGB_ERR_INVALID_ARGUMENT, "bad export blob");
    std::unique_ptr<mgb_results> res(new mgb_results());
    std::memset(&res->stats, 0, sizeof(res->stats));
    const uint32_t n = (uint32_t)h.n_reads;
    res->n_reads = n; res->n_alns = h.n_alns; res->result_nodes = (uint32_t)h.result_nodes;
    res->first.assign(n, 0); res->count.assign(n, 0); res->src_off.assign(n, 0); res->src_heap.assign(n, 0);
    const char *p = (const char*)blob + sizeof(h);
    std::memcpy(res->src_off.data(), p, 8ull * n); p += 8ull * n;
    std::memcpy(res->count.data(), p, 4ull * n); p += 4ull * n;
    std::memcpy(res->src_heap.data(), p, 4ull * n); p += 4ull * n;
    res->heap_bytes.assign(h.n_heaps, 0);
    std::memcpy(res->heap_bytes.data(), p, 8 * h.n_heaps); p += 8 * h.n_heaps;
    p = (const char*)blob + (((uint64_t)(p - (const char*)blob) + 15) & ~15ull);
    // the records are referenced in place: one host buffer takes over the heaps
    uint64_t heaps_total = 0;
    for (uint64_t b : res->heap_bytes) heaps_total += (b + 15) & ~15ull;
    if ((uint64_t)(p - (const char*)blob) + heaps_total > bytes) return fail(MGB_ERR_INVALID_ARGUMENT, "truncated export blob");
    HostBuf hb = hostbuf_acquire(heaps_total + 16);
    if (!hb.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
    res->heaps.push_back(hb);
    std::vector<uint64_t> heap_base(h.n_heaps, 0);
    {
        uint64_t o = 0;
        for (size_t i = 0; i < h.n_heaps; ++i) { heap_base[i] = o; o += (res->heap_bytes[i] + 15) & ~15ull; }
        parallel_copy(hb.p, p, heaps_total);
    }
    res->alns_buf = hostbuf_acquire((h.n_alns + 1) * sizeof(mgb_alignment_t));
    if (!res->alns_buf.p) return fail(MGB_ERR_CUDA, "host buffer allocation failed");
    res->alns = (mgb_alignment_t*)res->alns_buf.p;
    uint64_t pos = 0;
    for (uint32_t r = 0; r < n; ++r) { res->first[r] = pos; pos += res->count[r]; }
    if (pos != h.n_alns) return fail(MGB_ERR_INVALID_ARGUMENT, "inconsistent export blob");
    const bool no_nodes = res->result_nodes != 0;
    #pragma omp parallel for schedule(static) num_threads(host_team()) if (n > 20000)
    for (int64_t r = 0; r < (int64_t)n; ++r) {
        if (!res->count[r]) continue;
        unpack_records(hb.p + heap_base[res->src_heap[r]] + res->src_off[r], res->count[r], no_nodes,
                       read_index_base + (uint32_t)r, res->alns + res->first[r]);
    }
    // after the import the records live in heap 0 at the rebased offsets
    for (uint32_t r = 0; r < n; ++r) { res->src_off[r] += heap_base[res->src_heap[r]]; res->src_heap[r] = 0; }
    res->heap_bytes.assign(1, heaps_total);
    *out = res.release();
    return MGB_OK;
}

uint32_t mgb_results_num_reads(const mgb_results_t *r) { return r->n_reads; }
void mgb_results_read_range(const mgb_results_t *r, uint32_t read, uint64_t *first, uint32_t *count) {
    *first = r->first[read]; *count = r->count[read];
}
uint64_t mgb_results_num_alignments(const mgb_results_t *r) { return r->n_alns; }
const mgb_alignment_t* mgb_results_alignments(const mgb_results_t *r) { return r->alns; }
const mgb_stats_t* mgb_results_stats(const mgb_results_t *r) { return &r->stats; }
void mgb_results_free(mgb_results_t *r) { delete r; }

} // extern "C"
