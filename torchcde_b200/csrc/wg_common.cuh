// What the fused fixed-step solves on the tensor cores share across kernel files (sm_90a): the Runge-Kutta combination and
// the output interpolation on a lane's state values, and the warpgroup-MMA primitives of the 2xFP16 split in the fragment
// layout of cdeint_wgmma_kernel (solve_tc.cu, whose header comment describes that layout).  Used by solve_tc.cu (linear
// field) and solve_mlp.cu (MLP field).
#pragma once
#include "tc_common.cuh"

namespace tcde {
namespace tc {

// One Runge-Kutta combination on NV state values of the calling thread: kv = the stage's slopes, the next stage input ends
// up in zin.  Returns true when the stage completed a step.
template <int NV>
__device__ __forceinline__ bool rk_combine(const UmmaArgs& a, int sub, float dt, const float* y, float* k1, float* s23,
                                           const float* kv, float* zin) {
    using E = exact<float>;
    const f2 dt2 = pk(dt, dt);
    if (a.method == TCDE_RK4_38) {
        const float third = (float)(1.0 / 3.0);
        const f2 th2 = pk(third, third);
        if (sub == 0) {
#pragma unroll
            for (int h = 0; h < NV; h += 2) {
                k1[h] = kv[h]; k1[h + 1] = kv[h + 1];
                upk(add2(pk(y[h], y[h + 1]), mul2(mul2(dt2, pk(kv[h], kv[h + 1])), th2)), zin[h], zin[h + 1]);
            }
        } else if (sub == 1) {
#pragma unroll
            for (int h = 0; h < NV; h += 2) {
                s23[h] = kv[h]; s23[h + 1] = kv[h + 1];
                upk(add2(pk(y[h], y[h + 1]), mul2(dt2, sub2(pk(kv[h], kv[h + 1]), mul2(pk(k1[h], k1[h + 1]), th2)))),
                    zin[h], zin[h + 1]);
            }
        } else if (sub == 2) {
#pragma unroll
            for (int h = 0; h < NV; h += 2) {
                const f2 k2p = pk(s23[h], s23[h + 1]), k3p = pk(kv[h], kv[h + 1]);
                upk(add2(pk(y[h], y[h + 1]), mul2(dt2, add2(sub2(pk(k1[h], k1[h + 1]), k2p), k3p))), zin[h], zin[h + 1]);
                upk(add2(k2p, k3p), s23[h], s23[h + 1]);
            }
        } else {
            const f2 three = pk(3.f, 3.f), eighth = pk(0.125f, 0.125f);
#pragma unroll
            for (int h = 0; h < NV; h += 2) {
                const f2 sum = add2(add2(pk(k1[h], k1[h + 1]), mul2(three, pk(s23[h], s23[h + 1]))), pk(kv[h], kv[h + 1]));
                upk(add2(pk(y[h], y[h + 1]), mul2(mul2(sum, dt2), eighth)), zin[h], zin[h + 1]);
            }
            return true;
        }
        return false;
    }
    if (a.method == TCDE_MIDPOINT) {
        if (sub == 0) {
            const float half = E::mul(0.5f, dt);
#pragma unroll
            for (int h = 0; h < NV; ++h) zin[h] = E::add(y[h], E::mul(kv[h], half));
            return false;
        }
#pragma unroll
        for (int h = 0; h < NV; ++h) zin[h] = E::add(y[h], E::mul(dt, kv[h]));
        return true;
    }
#pragma unroll
    for (int h = 0; h < NV; ++h) zin[h] = E::add(y[h], E::mul(dt, kv[h]));
    return true;
}

// The transpose of rk_combine for a field whose Jacobian J_s does not depend on the state (the linear field): the stages of
// a step in reverse, sub 0 being its last stage.  yb = the cotangent ybar' of the step's end state, su = the sum of the
// stage products so far, run = rk4's running combination, kv = u_s = J_s^T kappa_s of the stage just evaluated; the next
// stage's kappa (the cotangent of its slope) ends up in kap.  rk4 (kappa_4 = dt/8 ybar', rk_backward_first):
//   kappa_3 = dt (3/8 ybar' + u_4),  kappa_2 = dt (3/8 ybar' - u_4 + u_3),  kappa_1 = dt (1/8 ybar' + u_4 - u_3/3 + u_2/3);
// midpoint: kappa_1 = dt/2 u_2.  Returns true when the stage closed the step: yb then holds ybar' + sum_s u_s, the
// cotangent of the step's start state.  T: float (the tensor-core kernels) or double; A: any argument struct with `method`.
template <int NV, typename A, typename T>
__device__ __forceinline__ bool rk_backward_combine(const A& a, int sub, T dt, T* yb, T* su, T* run, const T* kv, T* kap) {
    using E = exact<T>;
    if (a.method == TCDE_RK4_38) {
        const T third = (T)(1.0 / 3.0);
        if (sub == 0) {
#pragma unroll
            for (int h = 0; h < NV; ++h) {
                su[h] = kv[h];
                run[h] = kv[h];
                kap[h] = E::mul(dt, E::add(E::mul(T(0.375), yb[h]), kv[h]));
            }
        } else if (sub == 1) {
#pragma unroll
            for (int h = 0; h < NV; ++h) {
                kap[h] = E::mul(dt, E::add(E::sub(E::mul(T(0.375), yb[h]), run[h]), kv[h]));
                run[h] = E::sub(run[h], E::mul(kv[h], third));
                su[h] = E::add(su[h], kv[h]);
            }
        } else if (sub == 2) {
#pragma unroll
            for (int h = 0; h < NV; ++h) {
                kap[h] = E::mul(dt, E::add(E::add(E::mul(T(0.125), yb[h]), run[h]), E::mul(kv[h], third)));
                su[h] = E::add(su[h], kv[h]);
            }
        } else {
#pragma unroll
            for (int h = 0; h < NV; ++h) yb[h] = E::add(yb[h], E::add(su[h], kv[h]));
            return true;
        }
        return false;
    }
    if (a.method == TCDE_MIDPOINT) {
        if (sub == 0) {
            const T half = E::mul(T(0.5), dt);
#pragma unroll
            for (int h = 0; h < NV; ++h) {
                su[h] = kv[h];
                kap[h] = E::mul(half, kv[h]);
            }
            return false;
        }
#pragma unroll
        for (int h = 0; h < NV; ++h) yb[h] = E::add(yb[h], E::add(su[h], kv[h]));
        return true;
    }
#pragma unroll
    for (int h = 0; h < NV; ++h) yb[h] = E::add(yb[h], kv[h]);
    return true;
}

// kappa of a step's last stage from the cotangent ybar' of its end state: dt/8 ybar' (rk4), dt ybar' (midpoint, euler)
template <int NV, typename A, typename T>
__device__ __forceinline__ void rk_backward_first(const A& a, T dt, const T* yb, T* kap) {
    using E = exact<T>;
    const T c = (a.method == TCDE_RK4_38) ? E::mul(T(0.125), dt) : dt;
#pragma unroll
    for (int h = 0; h < NV; ++h) kap[h] = E::mul(c, yb[h]);
}

// The outputs that fall on the step just completed (y = its start, zin = its end); write(j, v) stores output j.
template <int NV, typename Write>
__device__ __forceinline__ void step_outputs(const UmmaArgs& a, int step, int& jn, int& next_out, const float* y,
                                             const float* zin, Write write) {
    using E = exact<float>;
    while (next_out == step) {
        const int mode = a.out_mode[jn];
        if (mode == 0) write(jn, y);
        else if (mode == 1) write(jn, zin);
        else {
            const float slope_w = a.out_slope[jn];
            float v[NV];
#pragma unroll
            for (int h = 0; h < NV; ++h) v[h] = E::add(y[h], E::mul(slope_w, E::sub(zin[h], y[h])));
            write(jn, v);
        }
        ++jn;
        next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
    }
}

namespace wg {

constexpr int kThreads = 128;                    // one warpgroup
constexpr int kPaths = 64;                       // the M of the wgmma tile
constexpr int kNV = 16;                          // state values per lane: 2 rows x 8 hidden units
constexpr int kN = 64;                           // output columns per chunk: hidden units 8c .. 8c + 7
constexpr int kChunks = kCols / kN;
constexpr int kAcc = kN / 2;                     // accumulator registers per chunk
constexpr int kDxSlot = 16 * kCh * 4;           // per warp: the scaled dX/dt of its 16 rows (solve_tc.cu's wg::field)
constexpr int kXch = BSmem<1>::bytes;            // the four warps' dX/dt slots, after the B tile and the bias
constexpr int kRowSlot = 6 * 32 * 8;             // per warp and buffer: spline rows, [2][b | 2c | 3d][32] float2
constexpr int kRows = kXch + 4 * kDxSlot;        // the four warps' two buffers each
constexpr int kFetch = kRows + 8 * kRowSlot;     // per thread: its two spline-row sources (16 bytes), then its buffer
constexpr int kSmem = kFetch + kThreads * 20 + 1024;   // slack for the 1024-byte alignment of the swizzled B tile

// shared-memory matrix descriptor of a K-major, 128-byte-swizzled operand whose 8-row swizzle atoms are 1024 bytes apart
__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// desc_sw128(addr + off) from base = desc_sw128(addr), for a shared-memory address addr + off below 2^18 (every shared
// address is) and off a multiple of 16: the start-address field (bits 0-13) is then (addr + off) >> 4, with no carry
__device__ __forceinline__ uint64_t desc_add(uint64_t base, uint32_t off) { return base + (off >> 4); }

__device__ __forceinline__ void mma_m64n64k16(float* d, const uint32_t* a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
// cp.async of 8 bytes to the shared address s; an 8-byte load from one
__device__ __forceinline__ void cp_async8(uint32_t s, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ float2 lds_f2(uint32_t s) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(s) : "memory");
    return v;
}
__device__ __forceinline__ void mma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void mma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void mma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads or writes of an accumulator across the asynchronous MMAs that own it
__device__ __forceinline__ void pin(float* d) {
#pragma unroll
    for (int i = 0; i < kAcc; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// The quad reduce-scatter that closes the contraction of chunk c (hidden units 8c .. 8c + 7): p[j][r] = the lane's
// partial sum over its two channels of unit 8c + j, row r.  Leaves in kv[8 r + 2 c + e] the sums of the units 8c + 2q + e
// the lane owns, added in the order (q, q ^ 1) + (q ^ 2, q ^ 3).
__device__ __forceinline__ void reduce_chunk(const float (*p)[2], int c, int q, float* kv) {
    const bool odd = q & 1, upper = q >> 1;
    // xor 1: keep the hidden units j with (j >> 1) & 1 == q & 1, that is 8c + 4h + 2 (q & 1) + e
    float u[2][2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float got = __shfl_xor_sync(0xffffffffu, odd ? p[4 * h + e][r] : p[4 * h + 2 + e][r], 1);
                u[h][e][r] = (odd ? p[4 * h + 2 + e][r] : p[4 * h + e][r]) + got;
            }
    // xor 2: lanes 0, 1 keep h = 0, lanes 2, 3 h = 1: the units 8c + 2q + e
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float got = __shfl_xor_sync(0xffffffffu, upper ? u[0][e][r] : u[1][e][r], 2);
            kv[8 * r + 2 * c + e] = (upper ? u[1][e][r] : u[0][e][r]) + got;
        }
}

}  // namespace wg

}  // namespace tc
}  // namespace tcde
