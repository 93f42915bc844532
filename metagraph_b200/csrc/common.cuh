// Warp / quad cooperation primitives for the sm_90a kernels.
//
// All device logic is written as "warp-uniform scalar control flow + lane-parallel vector
// loops": every lane of a warp executes the same branch on the same scalar values, global
// stores of scalars are done by lane 0 and vector work is strided over the lanes.
//
// The same sources also compile with plain g++ when MGB_HOST_EMU is defined. In that mode a
// "warp" is one lane wide, every collective degenerates to the identity, and the logic can
// be exercised on a machine without a GPU (tests/emu/, test infrastructure only — the
// product library never contains or calls the host instantiation).
#pragma once
#include <stdint.h>

// MGB_HD: kernel logic. Device-only under nvcc, plain inline under g++ (host emulation).
// MGB_HOSTDEV: helpers shared by host sizing code and kernels (no collectives inside).
#if defined(__CUDACC__)
#define MGB_HD __device__ __forceinline__
#define MGB_D __device__ __forceinline__
#define MGB_HOSTDEV __host__ __device__ __forceinline__
#define MGB_DEVICE_CODE 1
#else
#define MGB_HD inline
#define MGB_D inline
#define MGB_HOSTDEV inline
#define MGB_DEVICE_CODE 0
#endif

namespace mgb {

typedef int32_t score_t;
static constexpr score_t kNinf = INT32_MIN + 100;   // aligner_config.hpp:31

// A read is aligned by one warp of kWarp lanes; "scalar" values are uniform within the warp. The host
// emulation is a one-lane warp. kCPL is the number of DP cells a lane owns in the register path of the
// extender (a column of up to 32 cells): 1 on the device, 32 in the emulation.
#if MGB_DEVICE_CODE
static constexpr int kWarp = 32;
static constexpr int kCPL = 1;
MGB_D int wlane() { return threadIdx.x & (kWarp - 1); }
MGB_D unsigned wmask() { return 0xffffffffu; }
MGB_D void wsync() { __syncwarp(wmask()); }
template <class T> MGB_D T wbcast(T v, int src) { return __shfl_sync(wmask(), v, src, kWarp); }
MGB_D uint64_t wbcast64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(wmask(), (uint32_t)v, src, kWarp);
    uint32_t hi = __shfl_sync(wmask(), (uint32_t)(v >> 32), src, kWarp);
    return ((uint64_t)hi << 32) | lo;
}
MGB_D int wreduce_max(int v) { return __reduce_max_sync(wmask(), v); }
MGB_D int wreduce_min(int v) { return __reduce_min_sync(wmask(), v); }
MGB_D int wreduce_add(int v) { return __reduce_add_sync(wmask(), v); }
MGB_D unsigned wreduce_or(unsigned v) { return __reduce_or_sync(wmask(), v); }
MGB_D unsigned wballot(bool p) { return __ballot_sync(wmask(), p); }
// inclusive prefix max over the lanes of the warp
MGB_D int wscan_max(int v) {
#pragma unroll
    for (int d = 1; d < kWarp; d <<= 1) {
        int o = __shfl_up_sync(wmask(), v, d, kWarp);
        if (wlane() >= d) v = o > v ? o : v;
    }
    return v;
}
// inclusive prefix sum over the lanes of the warp
MGB_D int wscan_add(int v) {
#pragma unroll
    for (int d = 1; d < kWarp; d <<= 1) {
        int o = __shfl_up_sync(wmask(), v, d, kWarp);
        if (wlane() >= d) v += o;
    }
    return v;
}
MGB_D int wshfl_up1(int v, int fill) {
    int o = __shfl_up_sync(wmask(), v, 1, kWarp);
    return wlane() == 0 ? fill : o;
}
MGB_D int popc32(uint32_t x) { return __popc(x); }
MGB_D int ffs32(uint32_t x) { return __ffs(x); }            // 1-based, 0 if none
MGB_D int clz32(uint32_t x) { return __clz(x); }
// position (0-based) of the t-th (1-based) set bit of x; x must have >= t bits
MGB_D int nth_set32(uint32_t x, int t) { return __fns(x, 0, t); }
// lanes of a quad (4 consecutive lanes) cooperate on one 64-byte index block
MGB_D unsigned quad_mask() { return 0xFu << (threadIdx.x & 28); }
MGB_D int quad_lane() { return threadIdx.x & 3; }
MGB_D uint32_t qbcast(uint32_t v, int src) { return __shfl_sync(quad_mask(), v, src, 4); }
MGB_D uint32_t qxor(uint32_t v, int m) { return __shfl_xor_sync(quad_mask(), v, m, 4); }
#else
static constexpr int kWarp = 1;
static constexpr int kCPL = 32;      // the single host lane owns all 32 cells of a register-path column
inline int wlane() { return 0; }
inline void wsync() {}
template <class T> inline T wbcast(T v, int) { return v; }
inline uint64_t wbcast64(uint64_t v, int) { return v; }
inline int wreduce_max(int v) { return v; }
inline int wreduce_min(int v) { return v; }
inline int wreduce_add(int v) { return v; }
inline unsigned wreduce_or(unsigned v) { return v; }
inline int wscan_add(int v) { return v; }
inline unsigned wballot(bool p) { return p ? 1u : 0u; }
inline int wscan_max(int v) { return v; }
inline int wshfl_up1(int, int fill) { return fill; }
inline int popc32(uint32_t x) { return __builtin_popcount(x); }
inline int ffs32(uint32_t x) { return __builtin_ffs((int)x); }
inline int clz32(uint32_t x) { return x ? __builtin_clz(x) : 32; }
inline int nth_set32(uint32_t x, int t) {
    for (int i = 0; i < 32; ++i)
        if ((x >> i) & 1u) { if (--t == 0) return i; }
    return -1;
}
#endif

// a + b and a - b modulo 2^32. Past the scores the reference keeps in range (ninf plus more than one penalty, DESIGN.md
// §5) its epi32 column update wraps; these wrap the same way, with no undefined behaviour in the host build.
MGB_HOSTDEV int wadd(int a, int b) { return (int)((uint32_t)a + (uint32_t)b); }
MGB_HOSTDEV int wsub(int a, int b) { return (int)((uint32_t)a - (uint32_t)b); }

// max(a + b, c), a + b modulo 2^32: one DPX instruction (VIADDMNMX) on the device
MGB_HD int iaddmax(int a, int b, int c) {
#if MGB_DEVICE_CODE
    return __viaddmax_s32(a, b, c);
#else
    const int t = wadd(a, b);
    return t > c ? t : c;
#endif
}
MGB_HOSTDEV int imin(int a, int b) { return a < b ? a : b; }
MGB_HOSTDEV int imax(int a, int b) { return a > b ? a : b; }
MGB_HOSTDEV int iabs(int a) { return a < 0 ? -a : a; }

} // namespace mgb
