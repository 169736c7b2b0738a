// Shared pieces of the coefficient-builder translation units (hermite.cu, natural.cu, fill.cu):
// packed fp32x2 helpers, grid sizing, argument checks and the test-only kernel selectors.
#pragma once
#include "common.cuh"

namespace tcde {

static constexpr int kThreads = 256;

// two-float arithmetic: one IEEE rounding per lane and operation, never contracted into an FMA
typedef float2 f2;
__device__ __forceinline__ f2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk2(f2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// kernel selectors for tests / benchmarks (tcde_set_natural_variant, defined in fill.cu)
extern int g_fill_variant;            // 0 = scan / ballot warp-per-path gap fill when they fit, 1 = one thread per
                                      // series, 2 = never the scan kernel
extern int g_natural_variant;         // 0 = warp per path / windowed CTA sweeps when they fit, 1 = one thread per
                                      // series, 2 = never the warp-per-path kernel

static int persistent_grid(const void* kernel, int threads, size_t smem, int64_t n_items) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    int64_t g = (int64_t)sm_count() * per_sm;
    if (g > n_items) g = n_items;
    if (g < 1) g = 1;
    return (int)g;
}

static constexpr size_t kMaxSmem = 200 * 1024;

static int check_shape(const void* x, const void* out, int64_t n_paths, int64_t length, int64_t channels, int dtype) {
    TCDE_CHECK_ARG(x != nullptr && out != nullptr, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1, "n_paths=%lld channels=%lld", (long long)n_paths,
                   (long long)channels);
    TCDE_CHECK_ARG(length >= 2, "length=%lld (need at least 2 knots, misc.py:96-98)", (long long)length);
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_SUPPORTED(length < (1 << 24) && channels < (1 << 20), "length / channels too large");
    return TCDE_OK;
}


}  // namespace tcde
