// Small device helpers shared by the tensor-core kernels (solve_tc.cu, solve_dopri5.cu, param_grad_mma.cu):
// shared-memory addresses, the 128-byte swizzle of the operand tiles, TF32 rounding and two-float arithmetic.
#pragma once
#include "common.cuh"

namespace tcde {
namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }


// 128-byte-swizzled tile of 32-float rows: row r is the 128 bytes at r*128; its 16-byte chunk c lives at chunk position
// c ^ (r & 7), so that eight consecutive rows read at the same chunk hit eight different bank groups (ldmatrix).
__device__ __forceinline__ uint32_t swz(int row, int k) {          // element offset of (row, k) in floats
    return (uint32_t)row * 32u + (uint32_t)((((k >> 2) ^ (row & 7)) << 2) | (k & 3));
}
__device__ __forceinline__ float tf32_hi(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}

// ---- two-float arithmetic, one IEEE rounding per lane and operation (never contracted into an FMA except fma2) ------
typedef float2 f2;
__device__ __forceinline__ f2 pk(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk(f2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

}  // namespace umma
}  // namespace tcde
