// One stage of the continuous adjoint of hot path (ii): the README-form linear vector field and
// its vector-Jacobian products in ONE launch (sm_90a, fp32, hidden = 32, channels = 8).
//
// torchdiffeq's odeint_adjoint (the reference's default, solver.py:144 / 226-227) integrates the
// augmented state (z, a, dL/dW, dL/db) backwards in time; every stage of that solve needs
//     f[p][h]      = sf * sum_c (b[hC+c] + sum_k W[hC+c][k] z[p][k]) dX[p][c]
//     vz[p][k]     = sv * sum_h a[p][h] sum_c W[hC+c][k] dX[p][c]                 (a^T df/dz)
//     gW[hC+c][k] += sg * sum_p a[p][h] dX[p][c] z[p][k]                           (a^T df/dW)
//     gb[hC+c]    += sg * sum_p a[p][h] dX[p][c]                                   (a^T df/db)
// (sf, sv: the signs of the reversed-time solve; sg: sign times the Runge-Kutta weight of the stage)
// which the generic path gets from autograd (~40 launches and a 64 MB intermediate per stage).
// Here a persistent CTA walks tiles of 64 paths.  f and vz are the same register-tiled product as
// the forward CUDA-core kernel (solve_simt.cu), once with (z, W) and once with (a, W regrouped as
// [(k, c)][h]): thread (group of 8 paths, output unit) accumulates 8 x 4 products per pass and
// contracts them with dX.  The parameter gradients are a product over PATHS: thread (h, 4 k's) keeps
// its 8 x 4 block of dL/dW in registers across all tiles of the CTA and adds a[p][h] dX[p][c] z[p][k]
// path by path; per-CTA partial sums go to a scratch buffer and a second small kernel adds them
// (times s) into the caller's gradient tensors -- no atomics, deterministic for a given grid.
#include "common.cuh"

namespace tcde {
namespace vjp {

constexpr int H = 32, C = 8, Q = C / 4;
constexpr int TB = 64;                 // paths per tile
constexpr int TBp = TB + 4;            // padded row of the transposed stage inputs
constexpr int ST = 8;                  // paths per thread in the two products
constexpr int kThreads = 256;
constexpr int kParams = H * C * H + H * C;      // dL/dW then dL/db

struct alignas(16) F4 { float v[4]; };

// shared memory (floats)
constexpr int oW1 = 0;                          // [k][q][h][4]   W[(h C + 4q + j)][k]
constexpr int oW2 = oW1 + H * C * H;            // [h][q][k][4]   the same numbers, grouped by output k
constexpr int oB = oW2 + H * C * H;             // [q][h][4]
constexpr int oZT = oB + H * C;                 // [k][TBp]   z transposed
constexpr int oAT = oZT + H * TBp;              // [h][TBp]   a transposed
constexpr int oZR = oAT + H * TBp;              // [p][H]
constexpr int oAR = oZR + TB * H;               // [p][H]
constexpr int oDX = oAR + TB * H;               // [p][C]
constexpr int kSmemFloats = oDX + TB * C;

__global__ void __launch_bounds__(kThreads, 2)
field_vjp_kernel(const float* __restrict__ control, int control_kind, int64_t n_rows, const float* __restrict__ weight,
                 const float* __restrict__ bias, const float* __restrict__ z, const float* __restrict__ a,
                 float* __restrict__ f_out, float* __restrict__ vz_out, float* __restrict__ scratch, int64_t n_paths,
                 int index, float frac, float f_scale, float vjp_scale) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<float>;
    float* smem = reinterpret_cast<float*>(smem_raw);
    float* W1 = smem + oW1;
    float* W2 = smem + oW2;
    float* Bs = smem + oB;
    float* zT = smem + oZT;
    float* aT = smem + oAT;
    float* zR = smem + oZR;
    float* aR = smem + oAR;
    float* dxs = smem + oDX;
    const int tid = threadIdx.x;

    for (int e = tid; e < H * C * H; e += kThreads) {
        const int j = e & 3;
        int r = e >> 2;
        const int u = r % H; r /= H;             // h for W1, k for W2
        const int q = r % Q;
        const int v = r / Q;                     // k for W1, h for W2
        const int c = 4 * q + j;
        W1[e] = weight[((int64_t)u * C + c) * H + v];
        W2[e] = weight[((int64_t)v * C + c) * H + u];
    }
    for (int e = tid; e < H * C; e += kThreads) {
        const int j = e & 3;
        const int r = e >> 2;
        const int h = r % H, q = r / H;
        Bs[e] = bias[h * C + 4 * q + j];
    }

    const bool cubic = (control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * C : C;
    const int g = tid >> 5, u = tid & 31;        // products: paths 8g .. 8g+7, output unit u (h, then k)
    const int lp0 = g * ST;
    const int gh = tid & 31, gkt = tid >> 5;     // parameter gradients: row block h, columns 4 gkt .. 4 gkt + 3
    float gw[C][4], gb[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
        gb[c] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) gw[c][j] = 0.f;
    }

    const int64_t n_tiles = (n_paths + TB - 1) / TB;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t path0 = tile * TB;
        __syncthreads();                          // the previous tile (and the weight staging) is done with smem
        // ---- stage inputs: z and a rows (zero beyond the batch), dX/dt of every path --------------
        for (int e = tid; e < TB * (H / 4); e += kThreads) {
            const int lp = e >> 3, k4 = e & 7;
            const int64_t p = path0 + lp;
            F4 zv = {{0.f, 0.f, 0.f, 0.f}}, av = zv;
            if (p < n_paths) {
                zv = *reinterpret_cast<const F4*>(z + p * H + 4 * k4);
                av = *reinterpret_cast<const F4*>(a + p * H + 4 * k4);
            }
            *reinterpret_cast<F4*>(zR + lp * H + 4 * k4) = zv;
            *reinterpret_cast<F4*>(aR + lp * H + 4 * k4) = av;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                zT[(4 * k4 + j) * TBp + lp] = zv.v[j];
                aT[(4 * k4 + j) * TBp + lp] = av.v[j];
            }
        }
        for (int e = tid; e < TB * Q; e += kThreads) {
            const int lp = e / Q, q = e - lp * Q;
            int64_t p = path0 + lp;
            if (p >= n_paths) p = n_paths - 1;
            const float* r = control + (p * n_rows + index) * row_stride + (cubic ? C : 0) + 4 * q;
            F4 o;
#pragma unroll
            for (int j = 0; j < 4; ++j)           // interpolation_cubic.py:331-336, one rounding per operation
                o.v[j] = cubic ? E::add(r[j], E::mul(E::add(r[C + j], E::mul(r[2 * C + j], frac)), frac)) : r[j];
            *reinterpret_cast<F4*>(dxs + lp * C + 4 * q) = o;
        }
        __syncthreads();

        // ---- f = (W z + b) . dX   and   vz = (W^T-regrouped a) . dX: the same tiled product twice ---
#pragma unroll 1
        for (int which = 0; which < 2; ++which) {
            const float* in = (which == 0 ? zT : aT) + lp0;
            const float* wt = (which == 0 ? W1 : W2) + u * 4;
            float res[ST];
#pragma unroll
            for (int s = 0; s < ST; ++s) res[s] = 0.f;
#pragma unroll 1
            for (int q = 0; q < Q; ++q) {
                float acc[ST][4];
                const F4 b4 = *reinterpret_cast<const F4*>(Bs + (q * H + u) * 4);
#pragma unroll
                for (int s = 0; s < ST; ++s)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[s][j] = (which == 0) ? b4.v[j] : 0.f;
#pragma unroll 4
                for (int k = 0; k < H; ++k) {
                    const F4 i0 = *reinterpret_cast<const F4*>(in + k * TBp);
                    const F4 i1 = *reinterpret_cast<const F4*>(in + k * TBp + 4);
                    const F4 w4 = *reinterpret_cast<const F4*>(wt + ((size_t)k * Q + q) * H * 4);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
#pragma unroll
                        for (int s = 0; s < 4; ++s) {
                            acc[s][j] = fmaf(i0.v[s], w4.v[j], acc[s][j]);
                            acc[4 + s][j] = fmaf(i1.v[s], w4.v[j], acc[4 + s][j]);
                        }
                    }
                }
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    const F4 d4 = *reinterpret_cast<const F4*>(dxs + (lp0 + s) * C + 4 * q);
#pragma unroll
                    for (int j = 0; j < 4; ++j) res[s] = fmaf(acc[s][j], d4.v[j], res[s]);
                }
            }
            float* dst = (which == 0) ? f_out : vz_out;
            const float mult = (which == 0) ? f_scale : vjp_scale;
#pragma unroll
            for (int s = 0; s < ST; ++s) {
                const int64_t p = path0 + lp0 + s;
                if (p < n_paths) dst[p * H + u] = res[s] * mult;
            }
        }

        // ---- parameter gradients of this tile: gw[c][j] += a[p][h] dX[p][c] z[p][4 gkt + j] ---------
#pragma unroll 2
        for (int lp = 0; lp < TB; ++lp) {
            const float av = aR[lp * H + gh];
            const F4 d0 = *reinterpret_cast<const F4*>(dxs + lp * C);
            const F4 d1 = *reinterpret_cast<const F4*>(dxs + lp * C + 4);
            const F4 z4 = *reinterpret_cast<const F4*>(zR + lp * H + 4 * gkt);
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const float ad = av * (c < 4 ? d0.v[c] : d1.v[c - 4]);
                gb[c] += ad;
#pragma unroll
                for (int j = 0; j < 4; ++j) gw[c][j] = fmaf(ad, z4.v[j], gw[c][j]);
            }
        }
    }

    // ---- per-CTA partial sums: scratch[cta][(h C + c) H + k] and, after them, [h C + c] ---------------
    float* mine = scratch + (size_t)blockIdx.x * kParams;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        F4 o;
#pragma unroll
        for (int j = 0; j < 4; ++j) o.v[j] = gw[c][j];
        *reinterpret_cast<F4*>(mine + ((size_t)gh * C + c) * H + 4 * gkt) = o;
        if (gkt == 0) mine[H * C * H + gh * C + c] = gb[c];
    }
}

// grad[e] += scale * sum over CTAs of scratch[cta][e].  A CTA owns 32 elements; each of its 8 warps sums every
// 8th CTA's partial (128-byte coalesced rows), then warp 0 adds the 8 results in a fixed order: 8,448 elements x
// ~300 partial sums are a latency problem, not a bandwidth one, and one thread per element left most SMs idle.
__global__ void __launch_bounds__(256)
field_vjp_reduce_kernel(const float* __restrict__ scratch, int n_ctas, float scale, float* __restrict__ grad_weight,
                        float* __restrict__ grad_bias) {
    __shared__ float parts[8][32];
    const int lane = threadIdx.x & 31, part = threadIdx.x >> 5;
    const int e = blockIdx.x * 32 + lane;
    float s = 0.f;
    if (e < kParams)
        for (int cta = part; cta < n_ctas; cta += 8) s += scratch[(size_t)cta * kParams + e];
    parts[part][lane] = s;
    __syncthreads();
    if (part != 0 || e >= kParams) return;
    float total = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) total += parts[w][lane];
    if (e < H * C * H) {
        if (grad_weight) grad_weight[e] += scale * total;
    } else if (grad_bias) {
        grad_bias[e - H * C * H] += scale * total;
    }
}

// The parameter gradients of a WHOLE fixed-step backward solve in one launch, from the stage inputs that the
// two decoupled tensor-core solves left in HBM.  For the linear field the adjoint state does not depend on z
// (da/ds = a^T df/dz has no z in it), so z and a are each an ordinary fused solve; what couples them is only
//     dL/dW[hC+c][k] = sum over stages e, paths p of  w_e a_e[p][h] dX_e[p][c] z_e[p][k]       (w_e = ds * RK weight)
// Work item = (stage, tile of 64 paths); a persistent CTA keeps its 8 x 4 block per thread in registers over all
// its items, exactly like the per-stage kernel above, and leaves per-CTA partial sums in scratch.
__global__ void __launch_bounds__(kThreads, 3)
param_grad_kernel(const float* __restrict__ control, int control_kind, int64_t n_rows, const float* __restrict__ z_stages,
                  const float* __restrict__ a_stages, const int32_t* __restrict__ stage_index,
                  const float* __restrict__ stage_frac, const float* __restrict__ stage_weight, int n_stage_total,
                  float* __restrict__ scratch, int64_t n_paths) {
    __shared__ __align__(16) float zR[TB * H];
    __shared__ __align__(16) float aR[TB * H];
    __shared__ __align__(16) float dxs[TB * C];
    using E = exact<float>;
    const int tid = threadIdx.x;
    const bool cubic = (control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * C : C;
    const int gh = tid & 31, gkt = tid >> 5;
    float gw[C][4], gb[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
        gb[c] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) gw[c][j] = 0.f;
    }
    const int64_t n_tiles = (n_paths + TB - 1) / TB;
    const int64_t n_items = n_tiles * n_stage_total;
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int e = (int)(item / n_tiles);
        const int64_t path0 = (item - (int64_t)e * n_tiles) * TB;
        const float we = stage_weight[e];
        if (we == 0.f) continue;                  // e.g. the first stage of the midpoint rule (uniform per CTA)
        const int index = stage_index[e];
        const float frac = stage_frac[e];
        __syncthreads();                          // the previous item is done with the tiles
        const float* zs = z_stages + ((int64_t)e * n_paths + path0) * H;
        const float* as = a_stages + ((int64_t)e * n_paths + path0) * H;
        for (int v = tid; v < TB * (H / 4); v += kThreads) {
            const int lp = v >> 3;
            F4 zv = {{0.f, 0.f, 0.f, 0.f}}, av = zv;
            if (path0 + lp < n_paths) {
                zv = *reinterpret_cast<const F4*>(zs + 4 * v);
                av = *reinterpret_cast<const F4*>(as + 4 * v);
            }
            *reinterpret_cast<F4*>(zR + 4 * v) = zv;
            *reinterpret_cast<F4*>(aR + 4 * v) = av;
        }
        for (int v = tid; v < TB * Q; v += kThreads) {
            const int lp = v / Q, q = v - lp * Q;
            int64_t p = path0 + lp;
            if (p >= n_paths) p = n_paths - 1;
            const float* r = control + (p * n_rows + index) * row_stride + (cubic ? C : 0) + 4 * q;
            F4 o;
#pragma unroll
            for (int j = 0; j < 4; ++j) {         // dX/dt (interpolation_cubic.py:331-336), times the stage's weight
                const float d = cubic ? E::add(r[j], E::mul(E::add(r[C + j], E::mul(r[2 * C + j], frac)), frac)) : r[j];
                o.v[j] = d * we;
            }
            *reinterpret_cast<F4*>(dxs + lp * C + 4 * q) = o;
        }
        __syncthreads();
#pragma unroll 2
        for (int lp = 0; lp < TB; ++lp) {
            const float av = aR[lp * H + gh];
            const F4 d0 = *reinterpret_cast<const F4*>(dxs + lp * C);
            const F4 d1 = *reinterpret_cast<const F4*>(dxs + lp * C + 4);
            const F4 z4 = *reinterpret_cast<const F4*>(zR + lp * H + 4 * gkt);
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const float ad = av * (c < 4 ? d0.v[c] : d1.v[c - 4]);
                if (gkt == 0) gb[c] += ad;        // warp-uniform: one warp per row block owns the bias gradient
#pragma unroll
                for (int j = 0; j < 4; ++j) gw[c][j] = fmaf(ad, z4.v[j], gw[c][j]);
            }
        }
    }
    float* mine = scratch + (size_t)blockIdx.x * kParams;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        F4 o;
#pragma unroll
        for (int j = 0; j < 4; ++j) o.v[j] = gw[c][j];
        *reinterpret_cast<F4*>(mine + ((size_t)gh * C + c) * H + 4 * gkt) = o;
        if (gkt == 0) mine[H * C * H + gh * C + c] = gb[c];
    }
}

static int param_grad_grid(int64_t n_paths, int64_t n_stage_total) {
    const int64_t items = ((n_paths + TB - 1) / TB) * n_stage_total;
    int64_t g = (int64_t)sm_count() * 3;
    if (g > items) g = items;
    if (g < 1) g = 1;
    return (int)g;
}

static int vjp_grid(int64_t n_paths) {
    int64_t tiles = (n_paths + TB - 1) / TB;
    int64_t g = (int64_t)sm_count() * 2;
    if (g > tiles) g = tiles;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace vjp
}  // namespace tcde

using namespace tcde;

extern "C" int64_t tcde_vector_field_linear_vjp_scratch_bytes(int64_t n_paths, int64_t channels, int64_t hidden) {
    if (n_paths < 0 || channels != vjp::C || hidden != vjp::H) return -1;
    return (int64_t)vjp::vjp_grid(n_paths) * vjp::kParams * (int64_t)sizeof(float);
}

extern "C" int tcde_vector_field_linear_vjp(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                            const void* bias, const void* z, const void* a, void* f_out,
                                            void* vjp_z_out, void* grad_weight, void* grad_bias, void* scratch,
                                            int64_t n_paths, int64_t channels, int64_t hidden, int32_t index,
                                            double frac, double f_scale, double vjp_scale, double grad_scale,
                                            int dtype, void* stream) {
    TCDE_CHECK_ARG(control && weight && bias && z && a && f_out && vjp_z_out && scratch, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(index >= 0 && index < n_rows, "index=%d outside [0, %lld)", index, (long long)n_rows);
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == vjp::H && channels == vjp::C,
                         "the fused adjoint stage is built for fp32, hidden=%d, channels=%d (got dtype=%d, hidden=%lld, "
                         "channels=%lld)", vjp::H, vjp::C, dtype, (long long)hidden, (long long)channels);
    TCDE_CHECK_ARG(((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(scratch)) & 15) == 0,
                   "z, a and scratch must be 16-byte aligned");
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int grid = vjp::vjp_grid(n_paths);
    const size_t smem = (size_t)vjp::kSmemFloats * sizeof(float);
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(vjp::field_vjp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    vjp::field_vjp_kernel<<<grid, vjp::kThreads, smem, s>>>(
        (const float*)control, control_kind, n_rows, (const float*)weight, (const float*)bias, (const float*)z,
        (const float*)a, (float*)f_out, (float*)vjp_z_out, (float*)scratch, n_paths, (int)index, (float)frac,
        (float)f_scale, (float)vjp_scale);
    TCDE_CHECK_CUDA(cudaGetLastError());
    if (grad_weight || grad_bias) {
        vjp::field_vjp_reduce_kernel<<<(vjp::kParams + 31) / 32, 256, 0, s>>>((const float*)scratch, grid, (float)grad_scale,
                                                                                (float*)grad_weight, (float*)grad_bias);
        TCDE_CHECK_CUDA(cudaGetLastError());
    }
    return TCDE_OK;
}

extern "C" int64_t tcde_linear_field_param_grads_scratch_bytes(int64_t n_paths, int64_t n_stages_total, int64_t channels,
                                                              int64_t hidden) {
    if (n_paths < 0 || n_stages_total < 1 || channels != vjp::C || hidden != vjp::H) return -1;
    const int64_t g1 = vjp::param_grad_grid(n_paths, n_stages_total), g2 = param_grad_mma_grid(n_paths, n_stages_total);
    return (g1 > g2 ? g1 : g2) * vjp::kParams * (int64_t)sizeof(float);
}

extern "C" int tcde_linear_field_param_grads(const void* control, int control_kind, int64_t n_rows, const void* z_stages,
                                             const void* a_stages, const int32_t* stage_index, const void* stage_frac,
                                             const void* stage_weight, int64_t n_stages_total, void* grad_weight,
                                             void* grad_bias, void* scratch, int64_t n_paths, int64_t channels,
                                             int64_t hidden, double scale, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && z_stages && a_stages && stage_index && stage_frac && stage_weight && scratch,
                   "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_stages_total >= 1 && n_stages_total < (1ll << 31), "bad sizes");
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == vjp::H && channels == vjp::C,
                         "built for fp32, hidden=%d, channels=%d (got dtype=%d, hidden=%lld, channels=%lld)", vjp::H,
                         vjp::C, dtype, (long long)hidden, (long long)channels);
    TCDE_CHECK_ARG(((reinterpret_cast<uintptr_t>(z_stages) | reinterpret_cast<uintptr_t>(a_stages) |
                     reinterpret_cast<uintptr_t>(scratch)) & 15) == 0, "stage buffers and scratch must be 16-byte aligned");
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int grid;
    const int variant = current_solve_variant();
    if (variant != 1) {
        // tensor cores: 2xBF16 split by default (and for 4 / 5), 3xTF32 for the variants that select it for the solve
        const int mode = (variant == 2 || variant == 3 || variant == 6) ? 0 : 1;
        grid = param_grad_mma_grid(n_paths, n_stages_total);
        const int rc = param_grad_mma_f32((const float*)control, control_kind, n_rows, (const float*)z_stages,
                                          (const float*)a_stages, stage_index, (const float*)stage_frac,
                                          (const float*)stage_weight, (int)n_stages_total, (float*)scratch, n_paths, mode,
                                          grid, s);
        if (rc != TCDE_OK) return rc;
    } else {
        grid = vjp::param_grad_grid(n_paths, n_stages_total);
        vjp::param_grad_kernel<<<grid, vjp::kThreads, 0, s>>>((const float*)control, control_kind, n_rows,
                                                             (const float*)z_stages, (const float*)a_stages,
                                                             stage_index, (const float*)stage_frac,
                                                             (const float*)stage_weight, (int)n_stages_total,
                                                             (float*)scratch, n_paths);
        TCDE_CHECK_CUDA(cudaGetLastError());
    }
    if (grad_weight || grad_bias) {
        vjp::field_vjp_reduce_kernel<<<(vjp::kParams + 31) / 32, 256, 0, s>>>((const float*)scratch, grid, (float)scale,
                                                                              (float*)grad_weight, (float*)grad_bias);
        TCDE_CHECK_CUDA(cudaGetLastError());
    }
    return TCDE_OK;
}
