// Shared device/host helpers for the torchcde_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/torchcde_b200.h"

namespace tcde {

// ---- error plumbing (nothing throws across the C ABI) ------------------------------------
void set_error(const char* fmt, ...);
int cuda_failed(cudaError_t e, const char* what);

#define TCDE_CHECK_ARG(cond, ...)                 \
    do {                                          \
        if (!(cond)) {                            \
            tcde::set_error(__VA_ARGS__);         \
            return TCDE_ERR_ARGUMENT;             \
        }                                         \
    } while (0)

#define TCDE_CHECK_SUPPORTED(cond, ...)           \
    do {                                          \
        if (!(cond)) {                            \
            tcde::set_error(__VA_ARGS__);         \
            return TCDE_ERR_UNSUPPORTED;          \
        }                                         \
    } while (0)

#define TCDE_CHECK_CUDA(call)                                         \
    do {                                                              \
        cudaError_t e_ = (call);                                      \
        if (e_ != cudaSuccess) return tcde::cuda_failed(e_, #call);   \
    } while (0)

int sm_count();

// ---- arithmetic that must round exactly once per operation --------------------------------
// The reference is a chain of separate torch elementwise ops, i.e. one IEEE rounding per
// +,-,*,/ and never a fused multiply-add.  Kernels that promise bit-identical results use
// these wrappers so that nvcc cannot contract a*b+c into an FMA.
template <typename T> struct exact;
template <> struct exact<float> {
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
};
template <> struct exact<double> {
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
};

template <typename T> __device__ __forceinline__ bool is_nan(T v) { return v != v; }

// ---- 1-D bulk (TMA) shared -> global store -------------------------------------------------
// cp.async.bulk moves a contiguous, 16-byte-aligned byte range with one instruction issued by
// one thread; SASS shows it as UBLKCP.  The async proxy must see the generic-proxy writes to
// shared memory first, hence the proxy fence before the CTA barrier that precedes the issue.
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bulk_store(void* gmem, const void* smem, uint32_t bytes) {
    uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem), "r"(s), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// ---- 16-byte cp.async (LDGSTS) global -> shared --------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
    uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- arguments of the tensor-core solve (solve_tc.cu), filled in by the C entry points of solve_simt.cu ----
struct UmmaArgs {
    const float* control;
    const float* weight;
    const float* bias;
    const float* z0;
    float* out;
    const float* step_dt;
    const int32_t* stage_index;
    const float* stage_frac;
    const int32_t* out_step;
    const int32_t* out_mode;
    const float* out_slope;
    int64_t n_paths;
    int64_t n_rows;
    int control_kind, method, n_stages, n_steps, n_out;
    float sign;
    float* stage_dump;    // optional [n_steps * n_stages][n_paths][32]: the input of every stage (for the adjoint);
                          // reversible Heun: the checkpoints [slot][3][n_paths][32] (y, z, f of every ckpt_stride-th step)
    int ckpt_stride;      // reversible Heun only
    // the Runge-Kutta backward (tcde_cdeint_fixed_linear_backward) only: the schedule arrays above are reversed, out
    // receives dL/dz0 [n_paths][32] and stage_dump (optional) the cotangent of every stage's slope, in the forward's slots
    const float* grad_out;       // [n_paths][n_out][32] output gradients
    const int32_t* inj_range;    // [n_steps + 2]: grid state r (r = 0: the end of the solve) adds the entries
                                 // inj_range[r] .. inj_range[r + 1] - 1
    const int32_t* inj_out;      // output index of each entry
    const float* inj_weight;     // its weight
};
bool solve_tc_supported(int H, int C);
// tensor-core kernel (solve_tc.cu): Runge-Kutta state in registers; mode 0 = 3xTF32 operand split, mode 1 = 2xFP16 with
// per-path power-of-two scaling
int solve_tc_f32(const UmmaArgs& a, int H, int C, int mode, cudaStream_t stream);
int current_solve_variant();          // tcde_set_solve_variant: 0 auto, 1 CUDA-core, 2 / 3 tensor cores 3xTF32, 4 tensor cores 2xFP16

// parameter gradients of a whole backward solve on the tensor cores (param_grad_mma.cu): mode 0 = 3xTF32, 1 = 2xBF16 split
int param_grad_mma_grid(int64_t n_paths, int64_t n_stage_total);
int param_grad_mma_f32(const float* control, int control_kind, int64_t n_rows, const float* z_stages, const float* a_stages,
                       const int32_t* stage_index, const float* stage_frac, const float* stage_weight, int n_stage_total,
                       float* scratch, int64_t n_paths, int mode, int grid, cudaStream_t stream);

}  // namespace tcde
