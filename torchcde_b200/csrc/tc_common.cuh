// The linear vector field of one warp's 32 paths on the tensor cores (warp-level mma.sync, sm_90a), used by the 3xTF32
// fixed-step solve (solve_tc.cu) and the device-controlled dopri5 attempts (solve_dopri5.cu).  prepare_b<1>'s operand B, with
// its rows permuted (prepare_b<1, true>), is also the B of the 2xFP16 fixed-step solve's wgmma (a K-major 128-byte-swizzled
// tile).
//
// One evaluation is the product D[32 paths x 256] = z[32 x 32] . W^T[32 x 256] + bias followed by the contraction
// kv[h] = sum_c D[h * 8 + c] dX/dt[c].  fp32 accuracy on the tensor pipe comes from a two-way operand split:
//   * MODE 1 (2xFP16): z and W each become hi + lo FP16 pieces; z_lo.W_hi + z_hi.W_lo + z_hi.W_hi is 6 m16n8k16 MMAs per
//     16 x 8 output block.  FP16 has TF32's 11-bit significand (hi + lo = 22 bits) but only 5 exponent bits, so every path's
//     row is scaled by its own power of two (exact) so that max(|z_k|, bias floor) lands in [2^13, 2^14); the weights get one
//     global power of two.  The inverse scales are folded into the path's dX/dt before the contraction;
//   * MODE 0 (3xTF32): the same three products with TF32 pieces, 12 m16n8k8 MMAs per output block.
// The bias enters as the accumulator's initial value (scaled like the product in MODE 1).
//
// Each warp owns a private scratch (its 32 operand rows and their dX/dt) and never synchronises with other warps.  Lane l
// holds the path of row lane_row(l): with that assignment the reduction of the contraction over the four lanes of a quad
// (a reduce-scatter, three shuffles per hidden unit) leaves every lane with the full kv of its own row.
#pragma once
#include <cuda_fp16.h>

#include "umma.cuh"

namespace tcde {
namespace tc {

using namespace umma;

constexpr int kHid = 32, kCh = 8, kCols = kHid * kCh;

// row of the warp's 32-row operand tile that lane l evaluates: (l >> 2) + 8 * rho(l & 3), rho(q) = 2 (q & 1) + (q >> 1)
__device__ __forceinline__ int lane_row(int lane) { return (lane >> 2) + 8 * (2 * (lane & 1) + ((lane >> 1) & 1)); }

// shared memory of operand B (the split weights) and the bias, per CTA
template <int MODE> struct BSmem {
    static constexpr int tile = 0;                                        // MODE 1: [256][hi 32 | lo 32 halves]; MODE 0: hi, lo [256][32]
    static constexpr int bias = tile + (MODE == 0 ? 2 : 1) * kCols * 128; // [256] floats (MODE 1: times the weight scale)
    static constexpr int red = bias + kCols * 4;                          // 32 floats of reduction scratch
    static constexpr int bytes = red + 128;
};
// per-warp scratch: the operand rows of the warp's 32 paths, then per row dX/dt (8 floats) and the bias scale
template <int MODE> struct WarpSmem {
    static constexpr int a = 0;
    static constexpr int dx = (MODE == 0 ? 2 : 1) * 32 * 128;
    static constexpr int dx_stride = 12;                                  // floats per row
    static constexpr int bytes = dx + 32 * dx_stride * 4;                 // a multiple of 128
};

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {          // (lo, hi) -> f16x2, round to nearest even
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ void unpack_h2(uint32_t h, float& lo, float& hi) {
    asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}" : "=f"(lo), "=f"(hi) : "r"(h));
}
__device__ __forceinline__ int exponent_of(float m) { return (int)((__float_as_uint(m) >> 23) & 0xFFu); }   // biased
__device__ __forceinline__ float pow2_biased(int e) { return __uint_as_float((uint32_t)e << 23); }          // 2^(e-127)

__device__ __forceinline__ void ldsm_x4(const void* p, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(p))
                 : "memory");
}
__device__ __forceinline__ void mma_f16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Tile row of weight row n = 8h + c in the column-permuted MODE 1 tile of the fused solve (prepare_b<1, true>): within each
// 64-row chunk i, row 8j + 2q + e holds unit h = 8i + 2q + (j >> 2), channel c = 4e + (j & 3), so that lane q of a
// wgmma m64n64 accumulator (columns 8j + 2q + e) holds the two whole units 8i + 2q, 8i + 2q + 1 x all eight channels.
__device__ __forceinline__ int field_tile_row(int n) {
    const int h = n >> 3, c = n & 7;
    return 64 * (h >> 3) + 8 * (4 * (h & 1) + (c & 3)) + 2 * ((h >> 1) & 3) + (c >> 2);
}

// Operand B and the bias of the linear field weight [256][32], bias [256] (called by every thread of the CTA; contains
// __syncthreads).  MODE 1 returns the scales the rows need through inv_w_scale and beta (2^(ex(max|bias|) - ex(max|W|))).
// PERM (MODE 1 only): weight row n and its bias go to tile row field_tile_row(n) instead of n.
template <int MODE, bool PERM = false>
__device__ __forceinline__ void prepare_b(unsigned char* bsm, const float* weight, const float* bias, int tid, int n_threads,
                                          float& inv_w_scale, float& beta) {
    using S = BSmem<MODE>;
    float* b_bias = reinterpret_cast<float*>(bsm + S::bias);
    if (MODE == 0) {
        float* b_hi = reinterpret_cast<float*>(bsm + S::tile);
        float* b_lo = b_hi + kCols * 32;
        for (int e = tid; e < kCols * kHid; e += n_threads) {
            const int n = e >> 5, k = e & 31;
            const float w = weight[e];                     // weight[n][k], n = h*C + c
            const float hi = tf32_hi(w);
            b_hi[swz(n, k)] = hi;
            b_lo[swz(n, k)] = tf32_hi(w - hi);
        }
        for (int n = tid; n < kCols; n += n_threads) b_bias[n] = bias[n];
        inv_w_scale = 1.f;
        beta = 0.f;
        return;
    }
    float* red = reinterpret_cast<float*>(bsm + S::red);
    float wmax = 0.f, bmax = 0.f;
    for (int e = tid; e < kCols * kHid; e += n_threads) wmax = fmaxf(wmax, fabsf(weight[e]));
    for (int e = tid; e < kCols; e += n_threads) bmax = fmaxf(bmax, fabsf(bias[e]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
        bmax = fmaxf(bmax, __shfl_xor_sync(0xffffffffu, bmax, o));
    }
    if ((tid & 31) == 0) { red[tid >> 5] = wmax; red[16 + (tid >> 5)] = bmax; }
    __syncthreads();
    wmax = 0.f; bmax = 0.f;
    for (int w = 0; w < n_threads / 32; ++w) { wmax = fmaxf(wmax, red[w]); bmax = fmaxf(bmax, red[16 + w]); }
    __syncthreads();                                                              // red may be reused by the caller
    const int eb = min(max(exponent_of(bmax), 40), 215);
    const int ew = (wmax > 0.f) ? min(max(exponent_of(wmax), 40), 215) : (bmax > 0.f ? eb : 127);
    const float w_scale = pow2_biased(127 + 13 - (ew - 127));                    // max |W| * w_scale in [2^13, 2^14)
    inv_w_scale = pow2_biased(127 - 13 + (ew - 127));
    beta = (bmax > 0.f) ? pow2_biased(min(max(127 + eb - ew, 2), 250)) : 0.f;    // 2^(ex(bmax) - ex(wmax))
    __half* bt = reinterpret_cast<__half*>(bsm + S::tile);
    for (int e = tid; e < kCols * kHid; e += n_threads) {
        const int n = (PERM ? field_tile_row(e >> 5) : e >> 5), k = e & 31;     // n: the tile row (swizzled by n & 7)
        const float w = weight[e] * w_scale;
        const __half hi = __float2half_rn(w);
        const __half lo = __float2half_rn(w - __half2float(hi));
        bt[n * 64 + ((((k >> 3)) ^ (n & 7)) << 3) + (k & 7)] = hi;
        bt[n * 64 + ((((k >> 3) + 4) ^ (n & 7)) << 3) + (k & 7)] = lo;
    }
    for (int n = tid; n < kCols; n += n_threads) b_bias[PERM ? field_tile_row(n) : n] = bias[n] * w_scale;   // exact
}

// Row `row` of the warp's operand tile from z (32 floats).  MODE 1: z times the path's own power of two s, split into
// hi | lo halves (one 128-byte swizzled row); returns 1 / (s * weight scale), to be folded into dX/dt, and s through
// row_scale.  MODE 0: TF32 hi and lo rows; returns 1.
template <int MODE>
__device__ __forceinline__ float store_row(const float* z, unsigned char* a_tile, int row, float beta, float inv_w_scale, float& row_scale) {
    if (MODE == 0) {
        float* a_hi = reinterpret_cast<float*>(a_tile);
        float* a_lo = a_hi + 32 * 32;
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) {
            float4 hi, lo;
            hi.x = tf32_hi(z[4 * c4 + 0]); hi.y = tf32_hi(z[4 * c4 + 1]);
            hi.z = tf32_hi(z[4 * c4 + 2]); hi.w = tf32_hi(z[4 * c4 + 3]);
            lo.x = tf32_hi(__fsub_rn(z[4 * c4 + 0], hi.x)); lo.y = tf32_hi(__fsub_rn(z[4 * c4 + 1], hi.y));
            lo.z = tf32_hi(__fsub_rn(z[4 * c4 + 2], hi.z)); lo.w = tf32_hi(__fsub_rn(z[4 * c4 + 3], hi.w));
            const uint32_t off = (uint32_t)row * 32u + (uint32_t)((c4 ^ (row & 7)) << 2);
            *reinterpret_cast<float4*>(a_hi + off) = hi;
            *reinterpret_cast<float4*>(a_lo + off) = lo;
        }
        row_scale = 1.f;
        return 1.f;
    }
    float mx[8];                          // a tree, not a 32-long dependent chain
#pragma unroll
    for (int k = 0; k < 8; ++k) mx[k] = fmaxf(fmaxf(fabsf(z[k]), fabsf(z[k + 8])), fmaxf(fabsf(z[k + 16]), fabsf(z[k + 24])));
    const float m = fmaxf(fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3])), fmaxf(fmaxf(fmaxf(mx[4], mx[5]), fmaxf(mx[6], mx[7])), beta));
    const int e = min(max(exponent_of(m), 30), 224);
    const float s = pow2_biased(127 + 13 - (e - 127));
    uint32_t hi_h[16], lo_h[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float s0 = __fmul_rn(z[2 * j], s), s1 = __fmul_rn(z[2 * j + 1], s);
        float h0, h1;
        hi_h[j] = pack_h2(s0, s1);
        unpack_h2(hi_h[j], h0, h1);
        lo_h[j] = pack_h2(__fsub_rn(s0, h0), __fsub_rn(s1, h1));
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        *reinterpret_cast<uint4*>(a_tile + row * 128 + ((c ^ (row & 7)) << 4)) =
            make_uint4(hi_h[4 * c], hi_h[4 * c + 1], hi_h[4 * c + 2], hi_h[4 * c + 3]);
        *reinterpret_cast<uint4*>(a_tile + row * 128 + (((c + 4) ^ (row & 7)) << 4)) =
            make_uint4(lo_h[4 * c], lo_h[4 * c + 1], lo_h[4 * c + 2], lo_h[4 * c + 3]);
    }
    row_scale = s;
    return pow2_biased(127 - 13 + (e - 127)) * inv_w_scale;
}

// One evaluation of the field for the calling lane's path (every lane of the warp calls it together): z = the path's state,
// dx = its dX/dt (times the sign of the time direction); returns kv[h] = sum_c (W z + b)[h * 8 + c] dx[c].
template <int MODE>
__device__ __forceinline__ void warp_field(const float* z, const float* dx, float* kv, unsigned char* ws, const unsigned char* bsm,
                                           float beta, float inv_w_scale) {
    using S = BSmem<MODE>;
    using W = WarpSmem<MODE>;
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    const int row = lane_row(lane);
    __syncwarp();                                             // the previous evaluation's reads of the scratch are done
    float row_scale;
    const float inv = store_row<MODE>(z, ws + W::a, row, beta, inv_w_scale, row_scale);
    float* dxs = reinterpret_cast<float*>(ws + W::dx);
    *reinterpret_cast<float4*>(dxs + row * W::dx_stride) = make_float4(dx[0] * inv, dx[1] * inv, dx[2] * inv, dx[3] * inv);
    *reinterpret_cast<float4*>(dxs + row * W::dx_stride + 4) = make_float4(dx[4] * inv, dx[5] * inv, dx[6] * inv, dx[7] * inv);
    dxs[row * W::dx_stride + 8] = row_scale;
    __syncwarp();

    // A fragments: [piece hi / lo][m tile][k step][4]
    constexpr int kSteps = (MODE == 0) ? 4 : 2;
    uint32_t af[2][2][kSteps][4];
    {
        const unsigned char* a_tile = ws + W::a;
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int j = 0; j < kSteps; ++j) {
                    const int r = 16 * m + (lane & 15);
                    const int chunk = (MODE == 0 ? 0 : 4 * p) + 2 * j + (lane >> 4);
                    const unsigned char* base = a_tile + (MODE == 0 ? p * 32 * 128 : 0);
                    ldsm_x4(base + r * 128 + ((chunk ^ (r & 7)) << 4), af[p][m][j]);
                }
    }
    // dX/dt (2 channels) and bias scale of the four rows this lane's accumulators cover: g, g + 8, g + 16, g + 24
    float d[4][2], sc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 v = *reinterpret_cast<const float2*>(dxs + (g + 8 * j) * W::dx_stride + 2 * q);
        d[j][0] = v.x; d[j][1] = v.y;
        sc[j] = dxs[(g + 8 * j) * W::dx_stride + 8];
    }
    const float* b_bias = reinterpret_cast<const float*>(bsm + S::bias);
    const bool odd = q & 1, upper = (q >> 1) & 1;
#pragma unroll
    for (int h = 0; h < kHid; ++h) {
        const int n = 8 * h + (lane & 7);                     // B row this lane addresses for ldmatrix
        uint32_t bh[2 * kSteps], bl[2 * kSteps];
        if (MODE == 0) {
            const unsigned char* hi = bsm + S::tile;
            const unsigned char* lo = hi + kCols * 128;
            ldsm_x4(hi + n * 128 + (((lane >> 3) ^ (n & 7)) << 4), bh);
            ldsm_x4(hi + n * 128 + (((4 + (lane >> 3)) ^ (n & 7)) << 4), bh + 4);
            ldsm_x4(lo + n * 128 + (((lane >> 3) ^ (n & 7)) << 4), bl);
            ldsm_x4(lo + n * 128 + (((4 + (lane >> 3)) ^ (n & 7)) << 4), bl + 4);
        } else {
            const unsigned char* bt = bsm + S::tile;
            ldsm_x4(bt + n * 128 + (((lane >> 3) ^ (n & 7)) << 4), bh);
            ldsm_x4(bt + n * 128 + (((4 + (lane >> 3)) ^ (n & 7)) << 4), bl);
        }
        const float2 bb = *reinterpret_cast<const float2*>(b_bias + 8 * h + 2 * q);
        float c[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
            c[m][0] = bb.x * sc[2 * m]; c[m][1] = bb.y * sc[2 * m];
            c[m][2] = bb.x * sc[2 * m + 1]; c[m][3] = bb.y * sc[2 * m + 1];
#pragma unroll
            for (int j = 0; j < kSteps; ++j) {                // small terms first
                if (MODE == 0) mma_tf32(c[m], af[1][m][j], bh[2 * j], bh[2 * j + 1]);
                else mma_f16(c[m], af[1][m][j], bh[2 * j], bh[2 * j + 1]);
            }
#pragma unroll
            for (int j = 0; j < kSteps; ++j) {
                if (MODE == 0) mma_tf32(c[m], af[0][m][j], bl[2 * j], bl[2 * j + 1]);
                else mma_f16(c[m], af[0][m][j], bl[2 * j], bl[2 * j + 1]);
            }
#pragma unroll
            for (int j = 0; j < kSteps; ++j) {
                if (MODE == 0) mma_tf32(c[m], af[0][m][j], bh[2 * j], bh[2 * j + 1]);
                else mma_f16(c[m], af[0][m][j], bh[2 * j], bh[2 * j + 1]);
            }
        }
        // partial contraction of the lane's two channels for rows g, g + 8, g + 16, g + 24
        const float p0 = fmaf(c[0][1], d[0][1], c[0][0] * d[0][0]);
        const float p1 = fmaf(c[0][3], d[1][1], c[0][2] * d[1][0]);
        const float p2 = fmaf(c[1][1], d[2][1], c[1][0] * d[2][0]);
        const float p3 = fmaf(c[1][3], d[3][1], c[1][2] * d[3][0]);
        // reduce-scatter over the quad: lanes with odd q keep rows g + 16, g + 24, then q >> 1 picks the first or second
        const float r0 = __shfl_xor_sync(0xffffffffu, odd ? p0 : p2, 1);
        const float r1 = __shfl_xor_sync(0xffffffffu, odd ? p1 : p3, 1);
        const float u0 = (odd ? p2 : p0) + r0, u1 = (odd ? p3 : p1) + r1;
        const float r2 = __shfl_xor_sync(0xffffffffu, upper ? u0 : u1, 2);
        kv[h] = (upper ? u1 : u0) + r2;
    }
}

}  // namespace tc
}  // namespace tcde
