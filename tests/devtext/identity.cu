// TEST INFRASTRUCTURE ONLY: the `identity` formatter of the text route (format_core.cuh format_identity, "%.17g" of
// matches / query_len) over arrays, so that tests/test_text_identity*.py can sweep it against Python's "%.17g". Built
// for sm_90a by __graft_entry__.build() (tests/devtext/build/libmgb_text.so) and for the host by tests/devtext/Makefile
// (g++ -DMGB_HOST_EMU: tests/devtext/build/libmgb_text_emu.so). The product library never contains it.
#include "../../metagraph_b200/csrc/format_core.cuh"
#if !defined(MGB_HOST_EMU)
#include <cuda_runtime.h>
#endif

static constexpr int kTextWidth = 32;     // bytes per result, NUL-terminated

#if !defined(MGB_HOST_EMU)
__global__ void k_identity(const uint32_t *m, const uint32_t *q, uint64_t n, char *out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        char buf[24];
        const int len = mgb::format_identity(m[i], q[i], buf);
        char *o = out + i * kTextWidth;
        for (int j = 0; j < kTextWidth; ++j) o[j] = j < len ? buf[j] : 0;
    }
}
#endif

extern "C" {

// out: n * 32 bytes; returns 0, or a CUDA error code
int mgbt_identity(const uint32_t *m, const uint32_t *q, uint64_t n, char *out) {
#if defined(MGB_HOST_EMU)
    for (uint64_t i = 0; i < n; ++i) {
        char buf[24];
        const int len = mgb::format_identity(m[i], q[i], buf);
        for (int j = 0; j < kTextWidth; ++j) out[i * kTextWidth + j] = j < len ? buf[j] : 0;
    }
    return 0;
#else
    uint32_t *dm = nullptr, *dq = nullptr; char *dout = nullptr;
    cudaError_t e = cudaMalloc(&dm, n * 4 + 4);
    if (e == cudaSuccess) e = cudaMalloc(&dq, n * 4 + 4);
    if (e == cudaSuccess) e = cudaMalloc(&dout, n * kTextWidth + 1);
    if (e == cudaSuccess) e = cudaMemcpy(dm, m, n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dq, q, n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n) {
        k_identity<<<(unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096), 256>>>(dm, dq, n, dout);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, n * kTextWidth, cudaMemcpyDeviceToHost);
    cudaFree(dm); cudaFree(dq); cudaFree(dout);
    return (int)e;
#endif
}

} // extern "C"
