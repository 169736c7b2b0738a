// The fused fixed-step CDE solve for the MLP vector field of the reference's examples (sm_90a):
//   f(t, z) = tanh(W2 relu(W1 z + b1) + b2).view(H, C) @ dX/dt(t)
// (example/time_series_classification.py:20-51: Linear(H, W) -> ReLU -> Linear(W, H * C) -> tanh), with the schedule,
// controls, Runge-Kutta methods and outputs of tcde_cdeint_fixed_linear.  Two kernels:
//   * cdeint_mlp_wgmma_kernel (fp32, H = 32, C = 8, W = 128): the 2xFP16 split of cdeint_wgmma_kernel for both products,
//     two warpgroups per CTA sharing one copy of the split weights;
//   * cdeint_mlp_simt_kernel<T, HM> (fp32 / fp64, H <= HM, any C and W): one thread per path on the CUDA cores; the fp64
//     instantiation is the reference solve of the parity tests.
#include "wg_common.cuh"

namespace tcde {

template <typename T> struct MlpArgs {
    const T* control;        // cubic: [P][n_rows][4C]   linear: slopes [P][n_rows][C]
    const T* w1;             // [W][H]
    const T* b1;             // [W]
    const T* w2;             // [H*C][W]
    const T* b2;             // [H*C]
    const T* z0;             // [P][H]
    T* out;                  // [P][n_out][H]
    const T* step_dt;
    const int32_t* stage_index;
    const T* stage_frac;
    const int32_t* out_step;
    const int32_t* out_mode;
    const T* out_slope;
    int64_t n_paths, n_rows;
    int C, H, W;
    int control_kind, method, n_stages, n_steps, n_out;
    T sign;
};

__device__ __forceinline__ float tanh_of(float v) { return tanhf(v); }
__device__ __forceinline__ double tanh_of(double v) { return tanh(v); }

template <typename T, int N> struct alignas(sizeof(T) * N) Pack { T v[N]; };

// ---- CUDA cores: one thread per path ----------------------------------------------------------------------------------
//
// The state (y, k1, k2 + k3, stage input) sits in registers, HM values each, guarded by the runtime H.  The second product
// runs in chunks of NT outputs n = h C + c held in registers: for every hidden unit w, relu(W1[w] . z + b1[w]) is formed in
// registers and multiplied into the chunk, so no activation is stored; with H C > NT the first product is recomputed per
// chunk.  tanh of a finished chunk, times dX/dt[c], is added to the slope of unit h in the thread's column of shared
// memory, in increasing c like the reference's matmul order.  When they fit, the weights are staged once per CTA in shared
// memory as W1 [W][Hp] and W2^T [W][Nq] (zero padded), so every load is a 16-byte broadcast feeding four FMAs; otherwise
// they are read from global memory at warp-uniform addresses (one broadcast per warp through the L1).
constexpr int kMlpSimtThreads = 128;
constexpr int kMlpChunk = 32;                                  // NT: outputs per chunk

template <typename T> struct MlpSimtLayout {
    int Hp, Nq;                                                 // H and H*C rounded up to 4 and to NT
    size_t w1, w2t, b1, b2, cols, total;                        // offsets in elements of T; total in bytes
    bool staged;
};

template <typename T> static MlpSimtLayout<T> mlp_simt_layout(int H, int C, int W, bool stage) {
    MlpSimtLayout<T> l;
    l.Hp = (H + 3) / 4 * 4;
    l.Nq = (H * C + kMlpChunk - 1) / kMlpChunk * kMlpChunk;
    l.staged = stage;
    size_t off = 0;
    if (stage) {
        l.w1 = off; off += (size_t)W * l.Hp;
        l.w2t = off; off += (size_t)W * l.Nq;
        l.b1 = off; off += (size_t)W;
        l.b2 = off; off += (size_t)l.Nq;
        off = (off + 3) / 4 * 4;
    } else {
        l.w1 = l.w2t = l.b1 = l.b2 = 0;
    }
    l.cols = off; off += (size_t)(C + H) * kMlpSimtThreads;       // per thread: dX/dt [C], slopes [H]
    l.total = off * sizeof(T);
    return l;
}

template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads) cdeint_mlp_simt_kernel(const MlpArgs<T> a, const MlpSimtLayout<T> lay) {
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    if (lay.staged) {
        for (int e = tid; e < W * Hp; e += nt) {
            const int w = e / Hp, k = e - w * Hp;
            smem[lay.w1 + e] = k < H ? a.w1[(size_t)w * H + k] : T(0);
        }
        for (int e = tid; e < W * Nq; e += nt) {
            const int w = e / Nq, n = e - w * Nq;
            smem[lay.w2t + e] = n < HC ? a.w2[(size_t)n * W + w] : T(0);
        }
        for (int e = tid; e < W; e += nt) smem[lay.b1 + e] = a.b1[e];
        for (int e = tid; e < Nq; e += nt) smem[lay.b2 + e] = e < HC ? a.b2[e] : T(0);
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;                                // dxs[c * nt]: dX/dt channel c
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: slope of hidden unit h
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);

    auto write_out = [&](int j, const T* v) {
        if (!live) return;
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) a.out[(path * a.n_out + j) * H + h] = v[h];
    };

    T y[HM], k1[HM], s23[HM], zin[HM], kv[HM];
#pragma unroll
    for (int h = 0; h < HM; ++h) {
        y[h] = (h < H) ? a.z0[lp * H + h] : T(0);
        k1[h] = T(0); s23[h] = T(0); zin[h] = y[h];
    }
    int jn = 0;
    while (jn < a.n_out && a.out_step[jn] < 0) { write_out(jn, y); ++jn; }

    const int total = a.n_steps * a.n_stages;
    const T third = T(1.0 / 3.0);
    int step = 0, sub = 0;
    T dt = a.step_dt[0];
    for (int st = 0; st < total; ++st) {
        // dX/dt of this stage (interpolation_cubic.py:331-336), times the sign of the time direction
        {
            const T* r = crow + (int64_t)a.stage_index[st] * (cubic ? 4 * C : C);
            const T fr = a.stage_frac[st];
            for (int c = 0; c < C; ++c) {
                const T v = cubic ? E::add(r[c], E::mul(E::add(r[C + c], E::mul(r[2 * C + c], fr)), fr)) : r[c];
                dxs[(size_t)c * nt] = a.sign < T(0) ? -v : v;
            }
            for (int h = 0; h < H; ++h) kvs[(size_t)h * nt] = T(0);
        }
        for (int n0 = 0; n0 < HC; n0 += kMlpChunk) {
            T acc[kMlpChunk];
#pragma unroll
            for (int j = 0; j < kMlpChunk; ++j)
                acc[j] = lay.staged ? smem[lay.b2 + n0 + j] : (n0 + j < HC ? __ldg(a.b2 + n0 + j) : T(0));
            for (int w = 0; w < W; ++w) {
                // hidden unit w: relu(W1[w] . z + b1[w])
                T u;
                if (lay.staged) {
                    u = smem[lay.b1 + w];
                    const T* wr = smem + lay.w1 + (size_t)w * Hp;
#pragma unroll
                    for (int k4 = 0; k4 < HM / 4; ++k4) {
                        if (4 * k4 < Hp) {
                            const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);
#pragma unroll
                            for (int i = 0; i < 4; ++i) u = fma(w4.v[i], zin[4 * k4 + i], u);
                        }
                    }
                } else {
                    u = __ldg(a.b1 + w);
                    const T* wr = a.w1 + (size_t)w * H;
#pragma unroll
                    for (int k = 0; k < HM; ++k)
                        if (k < H) u = fma(__ldg(wr + k), zin[k], u);
                }
                u = u > T(0) ? u : T(0);
                if (lay.staged) {
                    const T* wc = smem + lay.w2t + (size_t)w * Nq + n0;
#pragma unroll
                    for (int j4 = 0; j4 < kMlpChunk / 4; ++j4) {
                        const P4 w4 = *reinterpret_cast<const P4*>(wc + 4 * j4);
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[4 * j4 + i] = fma(w4.v[i], u, acc[4 * j4 + i]);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < kMlpChunk; ++j)
                        if (n0 + j < HC) acc[j] = fma(__ldg(a.w2 + (size_t)(n0 + j) * W + w), u, acc[j]);
                }
            }
            // tanh, times dX/dt, into the slopes: output n = h C + c
            int h = n0 / C, c = n0 - h * C;
#pragma unroll
            for (int j = 0; j < kMlpChunk; ++j) {
                if (n0 + j < HC) {
                    kvs[(size_t)h * nt] = fma(tanh_of(acc[j]), dxs[(size_t)c * nt], kvs[(size_t)h * nt]);
                    if (++c == C) { c = 0; ++h; }
                }
            }
        }
#pragma unroll
        for (int h = 0; h < HM; ++h) kv[h] = (h < H) ? kvs[(size_t)h * nt] : T(0);
        // Runge-Kutta combination (oracle/odeint_port.py), one rounding per operation
        bool step_done = true;
        if (a.method == TCDE_RK4_38) {
            step_done = (sub == 3);
#pragma unroll
            for (int h = 0; h < HM; ++h) {
                if (sub == 0) {
                    k1[h] = kv[h];
                    zin[h] = E::add(y[h], E::mul(E::mul(dt, kv[h]), third));
                } else if (sub == 1) {
                    s23[h] = kv[h];
                    zin[h] = E::add(y[h], E::mul(dt, E::sub(kv[h], E::mul(k1[h], third))));
                } else if (sub == 2) {
                    zin[h] = E::add(y[h], E::mul(dt, E::add(E::sub(k1[h], s23[h]), kv[h])));
                    s23[h] = E::add(s23[h], kv[h]);
                } else {
                    const T sum = E::add(E::add(k1[h], E::mul(T(3), s23[h])), kv[h]);
                    zin[h] = E::add(y[h], E::mul(E::mul(sum, dt), T(0.125)));
                }
            }
        } else if (a.method == TCDE_MIDPOINT && sub == 0) {
            step_done = false;
            const T half = E::mul(T(0.5), dt);
#pragma unroll
            for (int h = 0; h < HM; ++h) zin[h] = E::add(y[h], E::mul(kv[h], half));
        } else {
#pragma unroll
            for (int h = 0; h < HM; ++h) zin[h] = E::add(y[h], E::mul(dt, kv[h]));
        }
        if (!step_done) {
            ++sub;
            continue;
        }
        // the outputs in (t0, t1] of this step (linear interpolation)
        while (jn < a.n_out && a.out_step[jn] == step) {
            const int mode = a.out_mode[jn];
            if (mode == 0) write_out(jn, y);
            else if (mode == 1) write_out(jn, zin);
            else {
                const T slope = a.out_slope[jn];
                T v[HM];
#pragma unroll
                for (int h = 0; h < HM; ++h) v[h] = E::add(y[h], E::mul(slope, E::sub(zin[h], y[h])));
                write_out(jn, v);
            }
            ++jn;
        }
#pragma unroll
        for (int h = 0; h < HM; ++h) y[h] = zin[h];
        ++step;
        sub = 0;
        if (step < a.n_steps) dt = a.step_dt[step];
    }
}

template <typename T, int HM>
static int launch_mlp_simt(const MlpArgs<T>& a, cudaStream_t stream) {
    auto kern = cdeint_mlp_simt_kernel<T, HM>;
    constexpr size_t kMax = 200 * 1024;
    MlpSimtLayout<T> lay = mlp_simt_layout<T>(a.H, a.C, a.W, true);
    if (lay.total > kMax) lay = mlp_simt_layout<T>(a.H, a.C, a.W, false);
    TCDE_CHECK_SUPPORTED(lay.total <= kMax, "MLP solve: hidden=%d channels=%d do not fit the CUDA-core kernel's shared "
                         "memory", a.H, a.C);
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.total));
    const int64_t ctas = (a.n_paths + kMlpSimtThreads - 1) / kMlpSimtThreads;
    TCDE_CHECK_SUPPORTED(ctas < (1ll << 31), "too many paths");
    kern<<<(unsigned)ctas, kMlpSimtThreads, lay.total, stream>>>(a, lay);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

template <typename T>
static int solve_mlp_simt(const MlpArgs<T>& a, cudaStream_t stream) {
    TCDE_CHECK_SUPPORTED(a.H <= 32, "MLP solve: hidden=%d > 32 is not built for the CUDA-core kernel", a.H);
    if (a.H <= 8) return launch_mlp_simt<T, 8>(a, stream);
    return launch_mlp_simt<T, 32>(a, stream);
}

// ---- tensor cores: 2xFP16 wgmma, H = 32, C = 8, W = 128 --------------------------------------------------------------
//
// Each warpgroup owns 64 paths in cdeint_wgmma_kernel's fragment layout (lane (g, q) of warp w: rows 16 w + g and
// 16 w + g + 8, hidden units 8 i + 2 q + e).  Per stage:
//   1. u = z W1^T + b1 (K = 32, N = 128): two chunks of N = 64, six m64n64k16 wgmmas each, A = the stage input split into
//      FP16 hi + lo with a per-row power of two exactly as in wg::field;
//   2. h = relu(u) in registers, unscaled exactly (powers of two), re-scaled per row and split into FP16 hi + lo A
//      fragments straight from the accumulator layout: accumulator columns 16 k + 8 t + 2 q + e of a row are the A columns
//      of k step k, so no shared-memory round trip;
//   3. v = h W2^T + b2 (K = 128, N = 256) in four chunks of N = 64 (hidden units 8 c .. 8 c + 7), 24 wgmmas each (eight k
//      steps x three split products, small terms first), two accumulators alternating as in wg::field;
//   4. tanhf of the unscaled accumulator (the accurate tanh: tanh.approx.f32's ~5e-4 relative error is far above the
//      fp32 bar), contracted with dX/dt and reduced over the quad by wg::reduce_chunk.
// Shared memory: W1's tile [128 rows][hi 32 | lo 32] (16 KB) and W2's [hi, lo][k block 0, 1][256 rows][64 halves] (128 KB),
// all K-major with the 128-byte swizzle, plus the scaled biases: 145 KB, one copy for the CTA's two warpgroups.
namespace tc {
namespace mlp {

constexpr int kWidth = 128;
constexpr int kGroups = 2;                                   // warpgroups per CTA
constexpr int kThreads = kGroups * wg::kThreads;
constexpr int kPaths = kGroups * wg::kPaths;
constexpr int kW2Region = kCols * 128;                       // one (piece, k block) region of W2's tile
struct Smem {
    static constexpr int w1 = 0;
    static constexpr int w2 = w1 + kWidth * 128;
    static constexpr int b1 = w2 + 4 * kW2Region;
    static constexpr int b2 = b1 + kWidth * 4;
    static constexpr int red = b2 + kCols * 4;
    static constexpr int bytes = red + 4 * (kThreads / 32) * 4;
};
constexpr int kSmem = Smem::bytes + 1024;                    // slack for the 1024-byte alignment of the tiles

// max |x| of two arrays over the CTA (all threads call it; contains __syncthreads)
__device__ __forceinline__ void cta_max(float* red, int tid, float& a, float& b, float& c, float& d) {
    float v[4] = {a, b, c, d};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[i] = fmaxf(v[i], __shfl_xor_sync(0xffffffffu, v[i], o));
        if ((tid & 31) == 0) red[i * (kThreads / 32) + (tid >> 5)] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[i] = 0.f;
        for (int w = 0; w < kThreads / 32; ++w) v[i] = fmaxf(v[i], red[i * (kThreads / 32) + w]);
    }
    a = v[0]; b = v[1]; c = v[2]; d = v[3];
}

// prepare_b<1>'s scales: one power of two for the weights (max |W| lands in [2^13, 2^14)), its inverse, and the bias floor
// of the per-row scale
__device__ __forceinline__ void split_scales(float wmax, float bmax, float& w_scale, float& inv_w_scale, float& beta) {
    const int eb = min(max(exponent_of(bmax), 40), 215);
    const int ew = (wmax > 0.f) ? min(max(exponent_of(wmax), 40), 215) : (bmax > 0.f ? eb : 127);
    w_scale = pow2_biased(127 + 13 - (ew - 127));
    inv_w_scale = pow2_biased(127 - 13 + (ew - 127));
    beta = (bmax > 0.f) ? pow2_biased(min(max(127 + eb - ew, 2), 250)) : 0.f;
}

// the power of two that brings max(|row|, floor) = m into [2^13, 2^14), and its inverse
__device__ __forceinline__ void row_scale(float m, float& rs, float& inv) {
    const int e = min(max(exponent_of(m), 30), 224);
    rs = pow2_biased(127 + 13 - (e - 127));
    inv = pow2_biased(127 - 13 + (e - 127));
}

__device__ __forceinline__ void split_h2(float s0, float s1, uint32_t& hi, uint32_t& lo) {
    float h0, h1;
    hi = pack_h2(s0, s1);
    unpack_h2(hi, h0, h1);
    lo = pack_h2(__fsub_rn(s0, h0), __fsub_rn(s1, h1));
}

struct Scales {
    float inv1, beta1, inv2, beta2;                          // per weight tile: 1 / weight scale, bias floor
};

__device__ __forceinline__ Scales prepare(unsigned char* smem, const float* w1, const float* b1, const float* w2,
                                          const float* b2, int tid) {
    float* red = reinterpret_cast<float*>(smem + Smem::red);
    float m1 = 0.f, mb1 = 0.f, m2 = 0.f, mb2 = 0.f;
    for (int e = tid; e < kWidth * kHid; e += kThreads) m1 = fmaxf(m1, fabsf(w1[e]));
    for (int e = tid; e < kWidth; e += kThreads) mb1 = fmaxf(mb1, fabsf(b1[e]));
    for (int e = tid; e < kCols * kWidth; e += kThreads) m2 = fmaxf(m2, fabsf(w2[e]));
    for (int e = tid; e < kCols; e += kThreads) mb2 = fmaxf(mb2, fabsf(b2[e]));
    cta_max(red, tid, m1, mb1, m2, mb2);
    Scales s;
    float s1, s2;
    split_scales(m1, mb1, s1, s.inv1, s.beta1);
    split_scales(m2, mb2, s2, s.inv2, s.beta2);
    __half* t1 = reinterpret_cast<__half*>(smem + Smem::w1);
    for (int e = tid; e < kWidth * kHid; e += kThreads) {     // [128 rows][hi k 0..31 | lo k 0..31], 16-byte chunks swizzled
        const int n = e >> 5, k = e & 31;
        const float w = w1[e] * s1;
        const __half hi = __float2half_rn(w);
        const __half lo = __float2half_rn(w - __half2float(hi));
        t1[n * 64 + (((k >> 3) ^ (n & 7)) << 3) + (k & 7)] = hi;
        t1[n * 64 + ((((k >> 3) + 4) ^ (n & 7)) << 3) + (k & 7)] = lo;
    }
    __half* t2 = reinterpret_cast<__half*>(smem + Smem::w2);
    for (int e = tid; e < kCols * kWidth; e += kThreads) {    // region (piece, k block): [256 rows][64 halves], swizzled
        const int n = e >> 7, k = e & 127, kb = k >> 6, kk = k & 63;
        const float w = w2[e] * s2;
        const __half hi = __float2half_rn(w);
        const __half lo = __float2half_rn(w - __half2float(hi));
        const int at = n * 64 + (((kk >> 3) ^ (n & 7)) << 3) + (kk & 7);
        t2[(0 * 2 + kb) * (kW2Region / 2) + at] = hi;
        t2[(1 * 2 + kb) * (kW2Region / 2) + at] = lo;
    }
    float* sb1 = reinterpret_cast<float*>(smem + Smem::b1);
    float* sb2 = reinterpret_cast<float*>(smem + Smem::b2);
    for (int n = tid; n < kWidth; n += kThreads) sb1[n] = b1[n] * s1;   // powers of two: exact
    for (int n = tid; n < kCols; n += kThreads) sb2[n] = b2[n] * s2;
    return s;
}

// One evaluation of the MLP field for the warpgroup's 64 rows: kv = tanh(W2 relu(W1 zin + b1) + b2) . dx in the fragment
// layout; dx: the lane's two channels of both rows, times the sign of the time direction.  mid() runs during the second
// product (the caller's next dX/dt hides behind the MMAs).
template <typename Mid>
__device__ __forceinline__ void field(const float* zin, const float (*dx)[2], const Scales& sc, const float* sb1,
                                      const float* sb2, uint32_t tile1, uint32_t tile2, int q, float* kv, Mid mid) {
    using namespace wg;
    // 1. u = z W1^T + b1, row-scaled: A from the stage input as in wg::field
    float rs[2], inv[2];
    uint32_t ahi[2][4], alo[2][4];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float m = sc.beta1;
#pragma unroll
        for (int h = 0; h < 8; ++h) m = fmaxf(m, fabsf(zin[8 * r + h]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        row_scale(m, rs[r], inv[r]);
        inv[r] *= sc.inv1;
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int t = 0; t < 4; ++t) {                          // register t: row t & 1, columns 16 k + 8 (t >> 1) + 2q, +1
            const int r = t & 1, v = 8 * r + 4 * k + 2 * (t >> 1);
            split_h2(__fmul_rn(zin[v], rs[r]), __fmul_rn(zin[v + 1], rs[r]), ahi[k][t], alo[k][t]);
        }
    float u[2][kAcc];                                         // column 64 c + 8 j + 2 q + e of row r at u[c][4 j + 2 r + e]
#pragma unroll
    for (int c = 0; c < 2; ++c) {
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {
            const float2 bb = *reinterpret_cast<const float2*>(sb1 + c * kN + 8 * j + 2 * q);
            u[c][4 * j + 0] = bb.x * rs[0]; u[c][4 * j + 1] = bb.y * rs[0];
            u[c][4 * j + 2] = bb.x * rs[1]; u[c][4 * j + 3] = bb.y * rs[1];
        }
    }
    mma_fence();
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const uint32_t rows = tile1 + c * kN * 128;
        mma_m64n64k16(u[c], alo[0], desc_sw128(rows + 0));    // z_lo . W1_hi
        mma_m64n64k16(u[c], alo[1], desc_sw128(rows + 32));
        mma_m64n64k16(u[c], ahi[0], desc_sw128(rows + 64));   // z_hi . W1_lo
        mma_m64n64k16(u[c], ahi[1], desc_sw128(rows + 96));
        mma_m64n64k16(u[c], ahi[0], desc_sw128(rows + 0));    // z_hi . W1_hi
        mma_m64n64k16(u[c], ahi[1], desc_sw128(rows + 32));
    }
    mma_commit();
    mma_wait<0>();
    pin(u[0]);
    pin(u[1]);

    // 2. h = relu(u) unscaled, then the second product's row scale and its hi / lo A fragments [k step][4]
    float m2[2] = {sc.beta2, sc.beta2};
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int i = 0; i < kAcc; ++i) {
            const int r = (i >> 1) & 1;
            const float h = fmaxf(__fmul_rn(u[c][i], inv[r]), 0.f);
            u[c][i] = h;
            m2[r] = fmaxf(m2[r], h);
        }
    float inv2[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 1));
        m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 2));
        row_scale(m2[r], rs[r], inv2[r]);
        inv2[r] *= sc.inv2;
    }
    uint32_t bhi[8][4], blo[8][4];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int t = 0; t < 4; ++t) {                          // A column 16 k + 8 (t >> 1) + 2 q = u column 64 c + 8 j + 2 q
            const int r = t & 1, c = k >> 2, j = 2 * (k & 3) + (t >> 1);
            split_h2(__fmul_rn(u[c][4 * j + 2 * r], rs[r]), __fmul_rn(u[c][4 * j + 2 * r + 1], rs[r]), bhi[k][t],
                     blo[k][t]);
        }

    // 3. v = h W2^T + b2 in four chunks of 64 columns, 4. tanh, contraction with dX/dt
    float acc[2][kAcc];
    auto issue = [&](int chunk, float* d) {
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {
            const float2 bb = *reinterpret_cast<const float2*>(sb2 + chunk * kN + 8 * j + 2 * q);
            d[4 * j + 0] = bb.x * rs[0]; d[4 * j + 1] = bb.y * rs[0];
            d[4 * j + 2] = bb.x * rs[1]; d[4 * j + 3] = bb.y * rs[1];
        }
        mma_fence();
        const uint32_t rows = tile2 + chunk * kN * 128;
        const uint32_t hi = rows, lo = rows + 2 * kW2Region;  // piece regions; k block kb at + kb * kW2Region
#pragma unroll
        for (int k = 0; k < 8; ++k)                            // h_lo . W2_hi
            mma_m64n64k16(d, blo[k], desc_sw128(hi + (k >> 2) * kW2Region + 32 * (k & 3)));
#pragma unroll
        for (int k = 0; k < 8; ++k)                            // h_hi . W2_lo
            mma_m64n64k16(d, bhi[k], desc_sw128(lo + (k >> 2) * kW2Region + 32 * (k & 3)));
#pragma unroll
        for (int k = 0; k < 8; ++k)                            // h_hi . W2_hi
            mma_m64n64k16(d, bhi[k], desc_sw128(hi + (k >> 2) * kW2Region + 32 * (k & 3)));
        mma_commit();
    };
    issue(0, acc[0]);
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        float* d = acc[c & 1];
        if (c + 1 < kChunks) {
            issue(c + 1, acc[(c + 1) & 1]);
            mma_wait<1>();
        } else {
            mma_wait<0>();
        }
        pin(d);
        if (c == kChunks / 2) mid();
        float p[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float f0 = tanhf(__fmul_rn(d[4 * j + 2 * r], inv2[r]));
                const float f1 = tanhf(__fmul_rn(d[4 * j + 2 * r + 1], inv2[r]));
                p[j][r] = fmaf(f1, dx[r][1], __fmul_rn(f0, dx[r][0]));
            }
        reduce_chunk(p, c, q, kv);
    }
}

__global__ void __launch_bounds__(kThreads, 1) cdeint_mlp_wgmma_kernel(const UmmaArgs a, const float* w2, const float* b2) {
    using E = exact<float>;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((1024u - (smem_u32(smem_unaligned) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const Scales sc = prepare(smem, a.weight, a.bias, w2, b2, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the tiles are read by wgmma (the async proxy)
    __syncthreads();
    const float* sb1 = reinterpret_cast<const float*>(smem + Smem::b1);
    const float* sb2 = reinterpret_cast<const float*>(smem + Smem::b2);
    const uint32_t tile1 = smem_u32(smem + Smem::w1), tile2 = smem_u32(smem + Smem::w2);

    const int64_t first = (int64_t)blockIdx.x * kPaths + (tid >> 7) * wg::kPaths;
    if (first >= a.n_paths) return;                            // a whole warpgroup past the batch; no CTA barrier follows
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_f2 = (cubic ? 4 * kCh : kCh) / 2;
    const float sign = (a.sign < 0.f) ? -1.f : 1.f;
    int64_t path[2];
    bool live[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        path[r] = first + 16 * warp + g + 8 * r;
        live[r] = path[r] < a.n_paths;
    }
    const int64_t lpath0 = live[0] ? path[0] : a.n_paths - 1;
    const int row1 = (int)((live[1] ? path[1] : a.n_paths - 1) - lpath0);
    const float2* crow = reinterpret_cast<const float2*>(a.control + lpath0 * a.n_rows * (2 * row_f2) + (cubic ? kCh : 0)) + q;
    auto fetch = [&](int interval, float2 (*raw)[3]) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2* src = crow + (r * row1 * a.n_rows + interval) * row_f2;
            raw[r][0] = __ldg(src);
            if (cubic) { raw[r][1] = __ldg(src + 4); raw[r][2] = __ldg(src + 8); }
        }
    };
    // dX/dt (interpolation_cubic.py:331-336) at fraction fr, channels 2q, 2q + 1 of both rows, times the sign
    auto slope = [&](const float2 (*raw)[3], float fr, float (*dx)[2]) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (cubic) {
                dx[r][0] = E::add(raw[r][0].x, E::mul(E::add(raw[r][1].x, E::mul(raw[r][2].x, fr)), fr));
                dx[r][1] = E::add(raw[r][0].y, E::mul(E::add(raw[r][1].y, E::mul(raw[r][2].y, fr)), fr));
            } else {
                dx[r][0] = raw[r][0].x;
                dx[r][1] = raw[r][0].y;
            }
            dx[r][0] = E::mul(dx[r][0], sign);
            dx[r][1] = E::mul(dx[r][1], sign);
        }
    };
    auto write_out = [&](int j, const float* v) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!live[r]) continue;
            float2* dst = reinterpret_cast<float2*>(a.out + (path[r] * a.n_out + j) * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[4 * i] = make_float2(v[8 * r + 2 * i], v[8 * r + 2 * i + 1]);
        }
    };

    float y[wg::kNV], k1[wg::kNV], s23[wg::kNV], zin[wg::kNV];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int64_t lpath = live[r] ? path[r] : a.n_paths - 1;
        const float2* zp = reinterpret_cast<const float2*>(a.z0 + lpath * kHid) + q;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 v = zp[4 * i];
            y[8 * r + 2 * i] = v.x; y[8 * r + 2 * i + 1] = v.y;
        }
    }
#pragma unroll
    for (int h = 0; h < wg::kNV; ++h) { k1[h] = 0.f; s23[h] = 0.f; zin[h] = y[h]; }
    int jn = 0;
    int next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
    while (jn < a.n_out && next_out < 0) {                    // outputs at the initial time
        write_out(jn, y);
        ++jn;
        next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
    }

    const int n_st = a.n_steps * a.n_stages;
    float dx[2][2];
    {
        float2 raw[2][3];
        fetch(a.stage_index[0], raw);
        slope(raw, a.stage_frac[0], dx);
    }
    int step = 0, sub = 0;
    float dt = a.step_dt[0];
    for (int st = 0; st < n_st; ++st) {
        float2 nxt[2][3];
        float dx_next[2][2];
        if (st + 1 < n_st) fetch(a.stage_index[st + 1], nxt);
        float kv[wg::kNV];
        field(zin, dx, sc, sb1, sb2, tile1, tile2, q, kv, [&] {
            if (st + 1 < n_st) slope(nxt, a.stage_frac[st + 1], dx_next);
        });
        if (rk_combine<wg::kNV>(a, sub, dt, y, k1, s23, kv, zin)) {
            step_outputs<wg::kNV>(a, step, jn, next_out, y, zin, write_out);
#pragma unroll
            for (int h = 0; h < wg::kNV; ++h) y[h] = zin[h];
            ++step;
            sub = 0;
            if (step < a.n_steps) dt = a.step_dt[step];
        } else {
            ++sub;
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) { dx[r][0] = dx_next[r][0]; dx[r][1] = dx_next[r][1]; }
    }
}

}  // namespace mlp
}  // namespace tc

static bool mlp_tc_shape(int64_t H, int64_t C, int64_t W) { return H == tc::kHid && C == tc::kCh && W == tc::mlp::kWidth; }

// Where automatic selection runs the CUDA-core kernel: the shapes at which it measured faster than cdeint's stage loop on
// an H100 (DESIGN 4.2): at most 8 hidden units (the HM = 8 instantiation) or one chunk of outputs (H C <= 32).  Elsewhere
// it recomputes the first product per chunk of 32 outputs and runs at low occupancy, and was 1.3-4.5x (fp32) and up to
// 13.6x (fp64) slower than the loop, so automatic selection refuses the shape and the caller keeps its stage loop.
static bool mlp_simt_preferred(int64_t H, int64_t C) { return H <= 8 || H * C <= kMlpChunk; }

}  // namespace tcde

using namespace tcde;

extern "C" int tcde_cdeint_fixed_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                                     const void* w2, const void* b2, const void* z0, void* out, int64_t n_paths,
                                     int64_t channels, int64_t hidden, int64_t width, int method, int64_t n_steps,
                                     const void* step_dt, const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                     const int32_t* out_step, const int32_t* out_mode, const void* out_slope, double sign,
                                     int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z0 && out, "null data pointer");
    TCDE_CHECK_ARG(step_dt && stage_index && stage_frac && out_step && out_mode && out_slope, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && width >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(n_steps >= 1 && n_out >= 1, "n_steps=%lld n_out=%lld", (long long)n_steps, (long long)n_out);
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    TCDE_CHECK_ARG(method == TCDE_EULER || method == TCDE_MIDPOINT || method == TCDE_RK4_38, "method=%d", method);
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    TCDE_CHECK_SUPPORTED(width < (1 << 20) && channels < (1 << 20) && hidden * channels < (1 << 20), "MLP too wide");
    if (n_paths == 0) return TCDE_OK;
    const int n_stages = (method == TCDE_RK4_38) ? 4 : (method == TCDE_MIDPOINT) ? 2 : 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int variant = current_solve_variant();
    const bool simt_ok = variant == 1 || mlp_simt_preferred(hidden, channels);
    if (dtype == TCDE_F32) {
        // 0: the tensor-core kernel where it is built for the shape and the buffers are 16-byte aligned, else the CUDA
        // cores where they beat the stage loop; 1: the CUDA cores; 4 / 5: the tensor-core kernel or TCDE_ERR_UNSUPPORTED;
        // 2 / 3 / 6 (3xTF32): not built
        const bool aligned = ((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(z0) |
                               reinterpret_cast<uintptr_t>(out)) & 15) == 0;
        const bool tc_ok = mlp_tc_shape(hidden, channels, width) && aligned;
        TCDE_CHECK_SUPPORTED(variant <= 1 || variant == 4 || variant == 5,
                             "MLP solve: solve variant %d (3xTF32) is not built for the MLP field", variant);
        if (variant >= 4) {
            TCDE_CHECK_SUPPORTED(tc_ok, "MLP solve: the tensor-core kernel is built for hidden=32, channels=8, width=128 "
                                 "with 16-byte aligned control, z0 and out (got %lld, %lld, %lld)", (long long)hidden,
                                 (long long)channels, (long long)width);
        }
        if (variant >= 4 || (variant == 0 && tc_ok)) {
            UmmaArgs u{(const float*)control, (const float*)w1, (const float*)b1, (const float*)z0, (float*)out,
                       (const float*)step_dt, stage_index, (const float*)stage_frac, out_step, out_mode,
                       (const float*)out_slope, n_paths, n_rows, control_kind, method, n_stages, (int)n_steps, (int)n_out,
                       (float)sign, nullptr, 0};
            const int64_t grid = (n_paths + tc::mlp::kPaths - 1) / tc::mlp::kPaths;
            TCDE_CHECK_SUPPORTED(grid < (1ll << 31), "too many paths");
            TCDE_CHECK_CUDA(cudaFuncSetAttribute(tc::mlp::cdeint_mlp_wgmma_kernel,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, tc::mlp::kSmem));
            tc::mlp::cdeint_mlp_wgmma_kernel<<<(unsigned)grid, tc::mlp::kThreads, tc::mlp::kSmem, s>>>(
                u, (const float*)w2, (const float*)b2);
            TCDE_CHECK_CUDA(cudaGetLastError());
            return TCDE_OK;
        }
        MlpArgs<float> a{(const float*)control, (const float*)w1, (const float*)b1, (const float*)w2, (const float*)b2,
                         (const float*)z0, (float*)out, (const float*)step_dt, stage_index, (const float*)stage_frac,
                         out_step, out_mode, (const float*)out_slope, n_paths, n_rows, (int)channels, (int)hidden,
                         (int)width, control_kind, method, n_stages, (int)n_steps, (int)n_out, (float)sign};
        TCDE_CHECK_SUPPORTED(simt_ok, "MLP solve: at hidden=%lld channels=%lld the CUDA-core kernel is slower than the "
                             "stage loop; automatic selection does not run it (variant 1 forces it)", (long long)hidden,
                             (long long)channels);
        return solve_mlp_simt(a, s);
    }
    TCDE_CHECK_SUPPORTED(simt_ok, "MLP solve: at hidden=%lld channels=%lld the CUDA-core kernel is slower than the stage "
                         "loop; automatic selection does not run it (variant 1 forces it)", (long long)hidden,
                         (long long)channels);
    MlpArgs<double> a{(const double*)control, (const double*)w1, (const double*)b1, (const double*)w2, (const double*)b2,
                      (const double*)z0, (double*)out, (const double*)step_dt, stage_index, (const double*)stage_frac,
                      out_step, out_mode, (const double*)out_slope, n_paths, n_rows, (int)channels, (int)hidden,
                      (int)width, control_kind, method, n_stages, (int)n_steps, (int)n_out, sign};
    return solve_mlp_simt(a, s);
}
