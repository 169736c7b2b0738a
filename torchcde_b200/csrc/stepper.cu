// Elementwise pieces of the adaptive (dopri5) driver as single launches (sm_90a).
//
// One attempted Dormand-Prince step forms six stage states  y + dt * sum_j beta_ij k_j  and one
// error estimate  |sum_j e_j k_j| / (atol + rtol * max(|y0|, |y1|)).  Written with torch operators
// that is ~60 small launches per attempt on states of a few MB -- more time than the six vector-field
// evaluations between them.  Here each combination is ONE streaming kernel over the state (any shape,
// fp32 / fp64, up to 7 terms, coefficients passed by value), and the error norm is ONE kernel that
// leaves per-CTA partial sums of squares (summed in a fixed order by the caller: deterministic).
#include "common.cuh"

namespace tcde {
namespace stepper {

constexpr int kMaxTerms = 7;
constexpr int kThreads = 256;

template <typename T> struct Terms {
    const T* k[kMaxTerms];
    T c[kMaxTerms];
    int n;
};

template <typename T>
__global__ void __launch_bounds__(kThreads)
combine_kernel(T* out, const T* base, const Terms<T> terms, int64_t n) {     // out may alias base
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += stride) {
        T v = base ? base[i] : T(0);
#pragma unroll
        for (int j = 0; j < kMaxTerms; ++j)
            if (j < terms.n) v = fma(terms.c[j], terms.k[j][i], v);
        out[i] = v;
    }
}

// partial[cta] = sum over the CTA's elements of (err / tol)^2, err = sum_j c_j k_j,
// tol = atol + rtol * max(|y0|, |y1|)    (torchdiffeq rk_common._compute_error_ratio, restated)
template <typename T>
__global__ void __launch_bounds__(kThreads)
error_kernel(const T* __restrict__ y0, const T* __restrict__ y1, const Terms<T> terms, T atol, T rtol, int64_t n,
             double* __restrict__ partial) {
    __shared__ double warp_sums[kThreads / 32];
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    double acc = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += stride) {
        T e = T(0);
#pragma unroll
        for (int j = 0; j < kMaxTerms; ++j)
            if (j < terms.n) e = fma(terms.c[j], terms.k[j][i], e);
        const T tol = atol + rtol * fmax(fabs(y0[i]), fabs(y1[i]));
        const double r = (double)(e / tol);
        acc += r * r;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += warp_sums[w];
        partial[blockIdx.x] = s;
    }
}

// _VectorField.forward's last line (solver.py:129-135) for an arbitrary func: out[p][h] = scale * sum_c f[p][h][c] * dx[p][c].
// torch.matmul hands this (batch of [H x C] . [C]) to a batched cuBLAS kernel: 62 us for 65,536 x 8 x 3 (100 GB/s); streamed
// it is a few microseconds.  dx may be a strided view (the stages of a step side by side): dx_stride elements per path.
template <typename T>
__global__ void __launch_bounds__(kThreads)
contract_kernel(const T* __restrict__ f, const T* __restrict__ dx, T* __restrict__ out, int64_t n_rows, int hidden, int channels,
                int64_t dx_stride, T scale) {
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n_rows; i += stride) {     // i = path * hidden + h
        const int64_t p = i / hidden;
        const T* fr = f + i * channels;
        const T* dr = dx + p * dx_stride;
        T acc = T(0);
        for (int c = 0; c < channels; ++c) acc = fma(fr[c], dr[c], acc);
        out[i] = scale * acc;
    }
}

static int stepper_grid(int64_t n) {
    int64_t g = (n + kThreads * 4 - 1) / (kThreads * 4);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

template <typename T>
static Terms<T> make_terms(const void* const* ks, const double* coefs, int n_terms) {
    Terms<T> t;
    t.n = n_terms;
    for (int j = 0; j < kMaxTerms; ++j) {
        t.k[j] = (j < n_terms) ? (const T*)ks[j] : nullptr;
        t.c[j] = (j < n_terms) ? (T)coefs[j] : T(0);
    }
    return t;
}

}  // namespace stepper
}  // namespace tcde

using namespace tcde;

extern "C" int tcde_linear_combination(void* out, const void* base, const void* const* terms, const double* coefs,
                                       int n_terms, int64_t n, int dtype, void* stream) {
    TCDE_CHECK_ARG(out != nullptr && n >= 0, "null output or negative size");
    TCDE_CHECK_ARG(n_terms >= 0 && n_terms <= stepper::kMaxTerms, "n_terms=%d (at most %d)", n_terms, stepper::kMaxTerms);
    TCDE_CHECK_ARG(n_terms == 0 || (terms != nullptr && coefs != nullptr), "null term list");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    for (int j = 0; j < n_terms; ++j) TCDE_CHECK_ARG(terms[j] != nullptr, "term %d is null", j);
    if (n == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = stepper::stepper_grid(n);
    if (dtype == TCDE_F32)
        stepper::combine_kernel<float><<<grid, stepper::kThreads, 0, s>>>((float*)out, (const float*)base,
                                                                         stepper::make_terms<float>(terms, coefs, n_terms), n);
    else
        stepper::combine_kernel<double><<<grid, stepper::kThreads, 0, s>>>((double*)out, (const double*)base,
                                                                          stepper::make_terms<double>(terms, coefs, n_terms), n);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

extern "C" int tcde_field_contract(const void* field, const void* dx, void* out, int64_t n_paths, int64_t hidden, int64_t channels,
                                   int64_t dx_stride, double scale, int dtype, void* stream) {
    TCDE_CHECK_ARG(field && dx && out, "null pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && hidden >= 1 && channels >= 1 && dx_stride >= channels, "bad sizes");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_SUPPORTED(hidden < (1ll << 31) && channels < (1ll << 31), "hidden / channels too large");
    const int64_t n = n_paths * hidden;
    if (n == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = stepper::stepper_grid(n * 4);
    if (dtype == TCDE_F32)
        stepper::contract_kernel<float><<<grid, stepper::kThreads, 0, s>>>((const float*)field, (const float*)dx, (float*)out, n, (int)hidden,
                                                                          (int)channels, dx_stride, (float)scale);
    else
        stepper::contract_kernel<double><<<grid, stepper::kThreads, 0, s>>>((const double*)field, (const double*)dx, (double*)out, n,
                                                                           (int)hidden, (int)channels, dx_stride, scale);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

extern "C" int64_t tcde_error_ratio_partials(int64_t n) { return n < 0 ? -1 : (int64_t)stepper::stepper_grid(n); }

extern "C" int tcde_error_ratio_sumsq(const void* y0, const void* y1, const void* const* terms, const double* coefs,
                                      int n_terms, double atol, double rtol, int64_t n, int dtype, void* partials,
                                      void* stream) {
    TCDE_CHECK_ARG(y0 && y1 && partials && terms && coefs, "null pointer");
    TCDE_CHECK_ARG(n_terms >= 1 && n_terms <= stepper::kMaxTerms, "n_terms=%d (1..%d)", n_terms, stepper::kMaxTerms);
    TCDE_CHECK_ARG(n >= 1, "n=%lld", (long long)n);
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    for (int j = 0; j < n_terms; ++j) TCDE_CHECK_ARG(terms[j] != nullptr, "term %d is null", j);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = stepper::stepper_grid(n);
    if (dtype == TCDE_F32)
        stepper::error_kernel<float><<<grid, stepper::kThreads, 0, s>>>((const float*)y0, (const float*)y1,
                                                                       stepper::make_terms<float>(terms, coefs, n_terms),
                                                                       (float)atol, (float)rtol, n, (double*)partials);
    else
        stepper::error_kernel<double><<<grid, stepper::kThreads, 0, s>>>((const double*)y0, (const double*)y1,
                                                                        stepper::make_terms<double>(terms, coefs, n_terms),
                                                                        atol, rtol, n, (double*)partials);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}
