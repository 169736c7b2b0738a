// Parameter gradients of a whole backward solve on the tensor cores (sm_90a, warp-level mma.sync).
//
//     dL/dW[hC+c][k] = sum over stages e, paths p of  U[(e,p)][hC+c] z_e[p][k],    U = w_e a_e[p][h] dX_e[p][c]
//     dL/db[hC+c]    = sum over (e, p) of U[(e,p)][hC+c]
// is ONE product G[256 x 40] = U^T [256 x pairs] . [z | 1 | 0...] [pairs x 40] over all (stage, path) pairs.  Work item =
// (stage, tile of 64 paths), dealt to persistent CTAs; the CTA stages z, a and w_e dX/dt of the item in shared memory
// (fp32), and warp w owns the output rows n = 32w .. 32w + 31 (hidden units 4w .. 4w + 3) for all 40 columns: 2 x 5
// accumulator blocks of 16 x 8.  Operand fragments are built straight from the fp32 tiles (U = a dX formed on the fly)
// with a two-way split, three MMAs per block and K step (lo.hi + hi.lo + hi.hi):
//   * MODE 1: BF16 pieces, m16n8k16 (8 + 8 significant bits; BF16 keeps fp32's exponent range, so no scaling);
//   * MODE 0: TF32 pieces, m16n8k8 (11 + 11 bits).
// Each item is accumulated in fresh registers and then added to the CTA's running sums with ordinary fp32 adds, so the
// tensor core never accumulates more than 64 pairs.  Per-CTA partial sums go to scratch in the layout of the CUDA-core
// kernel (solve_vjp.cu), whose fixed-order reduction adds them into the caller's gradients.
#include <cuda_bf16.h>

#include "tc_common.cuh"

namespace tcde {
namespace pg {

using namespace tc;

constexpr int H = 32, C = 8, TB = 64;
constexpr int kThreads = 256;                       // 8 warps x 32 output rows
constexpr int kParams = H * C * H + H * C;
constexpr int ZS = H + 1, DS = C + 1;               // padded rows of the staged tiles
constexpr int kNT = 5;                              // column blocks: z (4 x 8) + [1, 0 x 7]

__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ float bf_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// hi / lo pieces of two values packed as one operand register (MODE 1) or of one value (MODE 0: v1 unused)
template <int MODE> __device__ __forceinline__ void split(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    if (MODE == 1) {
        const float h0 = bf_round(v0), h1 = bf_round(v1);
        hi = pack_bf2(h0, h1);
        lo = pack_bf2(__fsub_rn(v0, h0), __fsub_rn(v1, h1));
    } else {
        const float h0 = tf32_hi(v0);
        hi = __float_as_uint(h0);
        lo = __float_as_uint(tf32_hi(__fsub_rn(v0, h0)));
    }
}
template <int MODE> __device__ __forceinline__ void mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    if (MODE == 1) mma_bf16(c, a, b0, b1);
    else mma_tf32(c, a, b0, b1);
}

template <int MODE>
__global__ void __launch_bounds__(kThreads, 2)
param_grad_mma_kernel(const float* __restrict__ control, int control_kind, int64_t n_rows, const float* __restrict__ z_stages,
                      const float* __restrict__ a_stages, const int32_t* __restrict__ stage_index,
                      const float* __restrict__ stage_frac, const float* __restrict__ stage_weight, int n_stage_total,
                      float* __restrict__ scratch, int64_t n_paths) {
    __shared__ float zR[TB * ZS];
    __shared__ float aR[TB * ZS];
    __shared__ float dxs[TB * DS];
    using E = exact<float>;
    constexpr int KS = (MODE == 1) ? 16 : 8;          // pairs per K step
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const bool cubic = (control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * C : C;
    float acc[2][kNT][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int t = 0; t < kNT; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[m][t][i] = 0.f;
    // column `col` of the B operand for pair j: z[j][col], then the bias column of ones, then zeros
    auto zval = [&](int j, int col) { return col < H ? zR[j * ZS + col] : (col == H ? 1.f : 0.f); };

    const int64_t n_tiles = (n_paths + TB - 1) / TB;
    const int64_t n_items = n_tiles * n_stage_total;
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int e = (int)(item / n_tiles);
        const int64_t path0 = (item - (int64_t)e * n_tiles) * TB;
        const float we = stage_weight[e];
        if (we == 0.f) continue;                      // uniform per CTA
        const int index = stage_index[e];
        const float frac = stage_frac[e];
        __syncthreads();                              // the previous item is done with the tiles
        const float* zs = z_stages + ((int64_t)e * n_paths + path0) * H;
        const float* as = a_stages + ((int64_t)e * n_paths + path0) * H;
        for (int v = tid; v < TB * (H / 4); v += kThreads) {
            const int lp = v >> 3, k4 = v & 7;
            float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), av = zv;
            if (path0 + lp < n_paths) {
                zv = reinterpret_cast<const float4*>(zs)[v];
                av = reinterpret_cast<const float4*>(as)[v];
            }
            float* zr = zR + lp * ZS + 4 * k4;
            float* ar = aR + lp * ZS + 4 * k4;
            zr[0] = zv.x; zr[1] = zv.y; zr[2] = zv.z; zr[3] = zv.w;
            ar[0] = av.x; ar[1] = av.y; ar[2] = av.z; ar[3] = av.w;
        }
        for (int v = tid; v < TB * C; v += kThreads) {
            const int lp = v >> 3, c = v & 7;
            int64_t p = path0 + lp;
            if (p >= n_paths) p = n_paths - 1;        // its z and a rows are zero
            const float* r = control + (p * n_rows + index) * row_stride + (cubic ? C : 0) + c;
            // dX/dt (interpolation_cubic.py:331-336), times the stage's weight
            const float d = cubic ? E::add(r[0], E::mul(E::add(r[C], E::mul(r[2 * C], frac)), frac)) : r[0];
            dxs[lp * DS + c] = d * we;
        }
        __syncthreads();

        float part[2][kNT][4];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int t = 0; t < kNT; ++t)
#pragma unroll
                for (int i = 0; i < 4; ++i) part[m][t][i] = 0.f;
#pragma unroll 1
        for (int j0 = 0; j0 < TB; j0 += KS) {
            // B fragments (k = pair, n = column 8t + g): b0 covers pairs 2q, 2q+1 (MODE 1) / q (MODE 0), b1 the same + KS / 2
            uint32_t bh[kNT][2], bl[kNT][2];
#pragma unroll
            for (int t = 0; t < kNT; ++t)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int col = 8 * t + g;
                    if (MODE == 1) {
                        const int j = j0 + 2 * q + 8 * r;
                        split<1>(zval(j, col), zval(j + 1, col), bh[t][r], bl[t][r]);
                    } else {
                        split<0>(zval(j0 + q + 4 * r, col), 0.f, bh[t][r], bl[t][r]);
                    }
                }
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                // A fragments (m = output row n = 8 h + c, k = pair): rows g / g + 8 of the block are hidden units h0 / h0 + 1
                // with channel g; register r * 2 + hh holds pair offset r * KS / 2, hidden unit h0 + hh
                const int h0 = 4 * warp + 2 * m;
                uint32_t ah[4], al[4];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        if (MODE == 1) {
                            const int j = j0 + 2 * q + 8 * r;
                            split<1>(aR[j * ZS + h0 + hh] * dxs[j * DS + g], aR[(j + 1) * ZS + h0 + hh] * dxs[(j + 1) * DS + g],
                                     ah[2 * r + hh], al[2 * r + hh]);
                        } else {
                            const int j = j0 + q + 4 * r;
                            split<0>(aR[j * ZS + h0 + hh] * dxs[j * DS + g], 0.f, ah[2 * r + hh], al[2 * r + hh]);
                        }
                    }
#pragma unroll
                for (int t = 0; t < kNT; ++t) {              // small terms first
                    mma<MODE>(part[m][t], al, bh[t][0], bh[t][1]);
                    mma<MODE>(part[m][t], ah, bl[t][0], bl[t][1]);
                    mma<MODE>(part[m][t], ah, bh[t][0], bh[t][1]);
                }
            }
        }
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int t = 0; t < kNT; ++t)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[m][t][i] += part[m][t][i];
    }
    // accumulator (m, t): rows n0 = 32 w + 16 m + g and n0 + 8, columns 8 t + 2 q, + 1
    float* mine = scratch + (size_t)blockIdx.x * kParams;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
        const int n0 = 32 * warp + 16 * m + g;
#pragma unroll
        for (int t = 0; t < kNT - 1; ++t) {
            const int k = 8 * t + 2 * q;
            *reinterpret_cast<float2*>(mine + n0 * H + k) = make_float2(acc[m][t][0], acc[m][t][1]);
            *reinterpret_cast<float2*>(mine + (n0 + 8) * H + k) = make_float2(acc[m][t][2], acc[m][t][3]);
        }
        if (q == 0) {                                 // column 32: the bias gradient
            mine[H * C * H + n0] = acc[m][kNT - 1][0];
            mine[H * C * H + n0 + 8] = acc[m][kNT - 1][2];
        }
    }
}

}  // namespace pg

int param_grad_mma_grid(int64_t n_paths, int64_t n_stage_total) {
    return capped_grid(((n_paths + pg::TB - 1) / pg::TB) * n_stage_total, 2);
}

int param_grad_mma_f32(const float* control, int control_kind, int64_t n_rows, const float* z_stages, const float* a_stages,
                       const int32_t* stage_index, const float* stage_frac, const float* stage_weight, int n_stage_total,
                       float* scratch, int64_t n_paths, int mode, int grid, cudaStream_t stream) {
    return launch((mode & 1) ? pg::param_grad_mma_kernel<1> : pg::param_grad_mma_kernel<0>, grid, pg::kThreads, 0,
                  stream, control, control_kind, n_rows, z_stages, a_stages, stage_index, stage_frac, stage_weight,
                  n_stage_total, scratch, n_paths);
}

}  // namespace tcde
