// The fused fixed-step CDE solve for the MLP vector field of the reference's examples (sm_90a):
//   f(t, z) = tanh(W2 relu(W1 z + b1) + b2).view(H, C) @ dX/dt(t)
// (example/time_series_classification.py:20-51: Linear(H, W) -> ReLU -> Linear(W, H * C) -> tanh), with the schedule,
// controls, Runge-Kutta methods and outputs of tcde_cdeint_fixed_linear.  Two kernels:
//   * cdeint_mlp_wgmma_kernel (fp32, H = 32, C = 8, W = 128): the 2xFP16 split of cdeint_wgmma_kernel for both products,
//     two warpgroups per CTA sharing one copy of the split weights;
//   * cdeint_mlp_simt_kernel<T, HM, DUMP> (fp32 / fp64, H <= HM, any C and W): one thread per path on the CUDA cores; the
//     fp64 instantiation is the reference solve of the parity tests.
// Each has a stage-dump variant, a Runge-Kutta backward and a parameter-gradient kernel for cdeint(..., adjoint=False).
#include <optional>
#include <type_traits>

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

// extra: more values per thread after the slopes (tcde_vector_field_mlp_vjp keeps f there, H of them)
template <typename T> static MlpSimtLayout<T> mlp_simt_layout(int H, int C, int W, bool stage,
                                                                int nt = kMlpSimtThreads, int extra = 0) {
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
    l.cols = off; off += (size_t)(C + H + extra) * nt;            // per thread: dX/dt [C], slopes [H], extra
    l.total = off * sizeof(T);
    return l;
}

// The field evaluation that the forward and the backward kernels share, so that the backward's dX/dt, ReLU masks and tanh
// values are the forward's bits.  Macros rather than __forceinline__ functions: the forward kernel expands them in place,
// token for token the code it had before the backward kernels existed, so its instructions are unchanged (as functions,
// the same code came out with a different register allocation).  They read the caller's a, lay, smem, tid, nt, crow,
// cubic, zin and H, C, W, HC, Hp, Nq, and the types E and P4.
//
// The weights in shared memory as W1 [W][Hp] and W2^T [W][Nq] (zero padded), by the CTA's nt threads (tid: this one)
#define TCDE_MLP_STAGE_WEIGHTS()                                                                                       \
    for (int e = tid; e < W * Hp; e += nt) {                                                                           \
        const int w = e / Hp, k = e - w * Hp;                                                                          \
        smem[lay.w1 + e] = k < H ? a.w1[(size_t)w * H + k] : T(0);                                                     \
    }                                                                                                                  \
    for (int e = tid; e < W * Nq; e += nt) {                                                                           \
        const int w = e / Nq, n = e - w * Nq;                                                                          \
        smem[lay.w2t + e] = n < HC ? a.w2[(size_t)n * W + w] : T(0);                                                   \
    }                                                                                                                  \
    for (int e = tid; e < W; e += nt) smem[lay.b1 + e] = a.b1[e];                                                      \
    for (int e = tid; e < Nq; e += nt) smem[lay.b2 + e] = e < HC ? a.b2[e] : T(0);

// dX/dt at (interval, fr) (interpolation_cubic.py:331-336), times the sign of the time direction, into dxs[c * nt]
#define TCDE_MLP_SLOPE(interval, frac)                                                                                 \
    const T* r = crow + (int64_t)(interval) * (cubic ? 4 * C : C);                                                     \
    const T fr = (frac);                                                                                               \
    for (int c = 0; c < C; ++c) {                                                                                      \
        const T v = cubic ? E::add(r[c], E::mul(E::add(r[C + c], E::mul(r[2 * C + c], fr)), fr)) : r[c];             \
        dxs[(size_t)c * nt] = a.sign < T(0) ? -v : v;                                                                  \
    }

// u = the pre-activation W1[w] . z + b1[w] of hidden unit w
#define TCDE_MLP_PRE(u, w)                                                                                             \
    T u;                                                                                                               \
    if (lay.staged) {                                                                                                  \
        u = smem[lay.b1 + w];                                                                                          \
        const T* wr = smem + lay.w1 + (size_t)w * Hp;                                                                  \
        _Pragma("unroll") for (int k4 = 0; k4 < HM / 4; ++k4) {                                                        \
            if (4 * k4 < Hp) {                                                                                         \
                const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);                                               \
                _Pragma("unroll") for (int i = 0; i < 4; ++i) u = fma(w4.v[i], zin[4 * k4 + i], u);                    \
            }                                                                                                          \
        }                                                                                                              \
    } else {                                                                                                           \
        u = __ldg(a.b1 + w);                                                                                           \
        const T* wr = a.w1 + (size_t)w * H;                                                                            \
        _Pragma("unroll") for (int k = 0; k < HM; ++k) if (k < H) u = fma(__ldg(wr + k), zin[k], u);                  \
    }

// acc [NT] = W2 relu(W1 z + b1) + b2 for the outputs n0 .. n0 + NT - 1
#define TCDE_MLP_CHUNK(acc, n0)                                                                                        \
    _Pragma("unroll") for (int j = 0; j < kMlpChunk; ++j)                                                              \
        acc[j] = lay.staged ? smem[lay.b2 + n0 + j] : (n0 + j < HC ? __ldg(a.b2 + n0 + j) : T(0));                     \
    for (int w = 0; w < W; ++w) {                                                                                      \
        TCDE_MLP_PRE(u, w)                                                                                             \
        u = u > T(0) ? u : T(0);                                                                                       \
        if (lay.staged) {                                                                                              \
            const T* wc = smem + lay.w2t + (size_t)w * Nq + n0;                                                        \
            _Pragma("unroll") for (int j4 = 0; j4 < kMlpChunk / 4; ++j4) {                                             \
                const P4 w4 = *reinterpret_cast<const P4*>(wc + 4 * j4);                                               \
                _Pragma("unroll") for (int i = 0; i < 4; ++i) acc[4 * j4 + i] = fma(w4.v[i], u, acc[4 * j4 + i]);      \
            }                                                                                                          \
        } else {                                                                                                       \
            _Pragma("unroll") for (int j = 0; j < kMlpChunk; ++j)                                                      \
                if (n0 + j < HC) acc[j] = fma(__ldg(a.w2 + (size_t)(n0 + j) * W + w), u, acc[j]);                      \
        }                                                                                                              \
    }

// DUMP: the input of every stage also goes to stage_dump[stage][path][H] (the forward state of the backward kernels)
template <typename T, int HM, bool DUMP>
__global__ void __launch_bounds__(kMlpSimtThreads) cdeint_mlp_simt_kernel(const MlpArgs<T> a, const MlpSimtLayout<T> lay,
                                                                          T* stage_dump) {
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    if (lay.staged) {
        TCDE_MLP_STAGE_WEIGHTS()
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
        if (DUMP && live) {
            T* dst = stage_dump + ((int64_t)st * a.n_paths + path) * H;
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) dst[h] = zin[h];
        }
        // dX/dt of this stage (interpolation_cubic.py:331-336), times the sign of the time direction
        {
            TCDE_MLP_SLOPE(a.stage_index[st], a.stage_frac[st])
            for (int h = 0; h < H; ++h) kvs[(size_t)h * nt] = T(0);
        }
        for (int n0 = 0; n0 < HC; n0 += kMlpChunk) {
            T acc[kMlpChunk];
            TCDE_MLP_CHUNK(acc, n0)
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

// The layout of a CUDA-core kernel of nt threads per CTA with `extra` values per thread after the slopes: the weights
// staged when everything fits in kMlpSimtMaxSmem bytes, else read from global memory; none if neither fits
constexpr size_t kMlpSimtMaxSmem = 200 * 1024;
template <typename T>
static std::optional<MlpSimtLayout<T>> mlp_simt_fit(int H, int C, int W, int nt, int extra) {
    for (const bool stage : {true, false}) {
        const MlpSimtLayout<T> lay = mlp_simt_layout<T>(H, C, W, stage, nt, extra);
        if (lay.total <= kMlpSimtMaxSmem) return lay;
    }
    return std::nullopt;
}

// kern(a, layout, args...) on the CUDA cores: one thread per path in CTAs of nt threads, the layout fitted for them
template <typename T, typename... P, typename... A>
static int mlp_launch_simt(void (*kern)(P...), const MlpArgs<T>& a, int nt, int extra, cudaStream_t s,
                           const A&... args) {
    const auto lay = mlp_simt_fit<T>(a.H, a.C, a.W, nt, extra);
    TCDE_CHECK_SUPPORTED(lay.has_value(), "MLP kernel on the CUDA cores: hidden=%d channels=%d width=%d do not fit its "
                         "shared memory", a.H, a.C, a.W);
    return launch(kern, (a.n_paths + nt - 1) / nt, nt, lay->total, s, a, *lay, args...);
}

// f(std::integral_constant<int, HM>()) at the CUDA-core instantiation hm (8 or 32)
template <typename F> static int mlp_hm(int hm, F&& f) {
    return hm == 8 ? f(std::integral_constant<int, 8>()) : f(std::integral_constant<int, 32>());
}

// ---- the backward of the CUDA-core solve (cdeint(..., adjoint=False)): one thread per path ---------------------------
//
// The transposed Runge-Kutta recurrence of cdeint_mlp_backward_kernel (rk_backward_combine, the host-reversed tables, the
// same output-gradient injection), with the stage product at the forward's stage input z_s (read back from its dump)
//   u_s = W1^T (mask . W2^T g),   g[(h, c)] = (1 - y^2)[(h, c)] kappa_s[h] dX_s[c],   mask = (W1 z_s + b1 > 0)
// formed chunk by chunk: TCDE_MLP_CHUNK recomputes the chunk's v = W2 h + b2 (the forward's bits, so y = tanh(v) and the ReLU
// mask are the forward's), g of its NT outputs stays in registers, and a second pass over the hidden units recomputes
// each pre-activation for its mask and adds W1[w] (mask_w W2[chunk, w] . g) to u.  u is linear in g, so nothing of
// width W is kept per thread.  dX/dt and kappa sit in the thread's column of shared memory, as the forward's dX/dt and
// slopes do (their index runs with the output n = h C + c).

struct MlpIgnore {
    template <typename... Args> __device__ __forceinline__ void operator()(Args...) const {}
};

// For every chunk: chunk(n0, g) with g [NT] (zero past H C), then unit(w, pre_w, W2[n0 .., w] . g) for every hidden unit;
// tanh_out(h, c, y) sees every output's tanh value as g is formed (tcde_vector_field_mlp_vjp forms f from them)
template <typename T, int HM, typename Chunk, typename Unit, typename Tanh = MlpIgnore, typename Z = const T*>
__device__ __forceinline__ void mlp_vjp(const MlpArgs<T>& a, const MlpSimtLayout<T>& lay, const T* smem, Z zin,
                                        const T* dxs, const T* kvs, int nt, Chunk chunk, Unit unit,
                                        Tanh tanh_out = Tanh()) {
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    for (int n0 = 0; n0 < HC; n0 += kMlpChunk) {
        T gc[kMlpChunk];
        TCDE_MLP_CHUNK(gc, n0)
        int h = n0 / C, c = n0 - h * C;
#pragma unroll
        for (int j = 0; j < kMlpChunk; ++j) {
            if (n0 + j < HC) {
                const T y = tanh_of(gc[j]);
                tanh_out(h, c, y);
                gc[j] = E::mul(E::sub(T(1), E::mul(y, y)), E::mul(kvs[(size_t)h * nt], dxs[(size_t)c * nt]));
                if (++c == C) { c = 0; ++h; }
            } else {
                gc[j] = T(0);
            }
        }
        chunk(n0, gc);
        for (int w = 0; w < W; ++w) {
            TCDE_MLP_PRE(pre, w)
            T sv = T(0);
            if (lay.staged) {
                const T* wc = smem + lay.w2t + (size_t)w * Nq + n0;
#pragma unroll
                for (int j4 = 0; j4 < kMlpChunk / 4; ++j4) {
                    const P4 w4 = *reinterpret_cast<const P4*>(wc + 4 * j4);
#pragma unroll
                    for (int i = 0; i < 4; ++i) sv = fma(w4.v[i], gc[4 * j4 + i], sv);
                }
            } else {
#pragma unroll
                for (int j = 0; j < kMlpChunk; ++j)
                    if (n0 + j < HC) sv = fma(__ldg(a.w2 + (size_t)(n0 + j) * W + w), gc[j], sv);
            }
            unit(n0, w, pre, sv);
        }
    }
}

template <typename T> struct MlpSimtBwd {
    const T* z_dump;              // the forward's stage inputs [n_total][n_paths][H]
    T* kappa_dump;                // kappa_s in the same slots (may be null)
    const T* grad_out;            // [n_paths][n_out][H]
    const int32_t* inj_range;
    const int32_t* inj_out;
    const T* inj_weight;
};

// a.step_dt, a.stage_index, a.stage_frac: the host-reversed tables; a.out: dL/dz0 [n_paths][H]
template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads) cdeint_mlp_simt_backward_kernel(const MlpArgs<T> a,
                                                                                   const MlpSimtLayout<T> lay,
                                                                                   const MlpSimtBwd<T> b) {
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    if (lay.staged) {
        TCDE_MLP_STAGE_WEIGHTS()
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: kappa of hidden unit h
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);

    // v += the output gradients that land on grid state r (counted from the end of the solve)
    auto inject = [&](int r, T* v) {
        for (int e = b.inj_range[r]; e < b.inj_range[r + 1]; ++e) {
            const T wt = b.inj_weight[e];
            const T* src = b.grad_out + (lp * a.n_out + b.inj_out[e]) * H;
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) v[h] = E::add(v[h], E::mul(wt, src[h]));
        }
    };

    T yb[HM], su[HM], run[HM], kap[HM];
#pragma unroll
    for (int h = 0; h < HM; ++h) { yb[h] = T(0); su[h] = T(0); run[h] = T(0); }
    inject(0, yb);
    tc::rk_backward_first<HM>(a, a.step_dt[0], yb, kap);

    const int n_st = a.n_steps * a.n_stages;
    const int64_t plane = a.n_paths * H;
    const T* z_at = b.z_dump + (int64_t)(n_st - 1) * plane + lp * H;     // stage st's forward slot, walking down
    T* k_at = b.kappa_dump ? b.kappa_dump + (int64_t)(n_st - 1) * plane + lp * H : nullptr;
    int step = 0, sub = 0;
    T dt = a.step_dt[0];
    for (int st = 0; st < n_st; ++st) {
        T zs[HM], kv[HM];
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            zs[h] = (h < H) ? z_at[h] : T(0);
            kv[h] = T(0);
            if (h < H) {
                kvs[(size_t)h * nt] = kap[h];
                if (k_at && live) k_at[h] = kap[h];
            }
        }
        z_at -= plane;
        if (k_at) k_at -= plane;
        {
            TCDE_MLP_SLOPE(a.stage_index[st], a.stage_frac[st])
        }
        mlp_vjp<T, HM>(a, lay, smem, zs, dxs, kvs, nt, [](int, const T*) {}, [&](int, int w, T pre, T sv) {
            if (!(pre > T(0))) return;
            if (lay.staged) {
                const T* wr = smem + lay.w1 + (size_t)w * lay.Hp;
#pragma unroll
                for (int k4 = 0; k4 < HM / 4; ++k4) {
                    if (4 * k4 < lay.Hp) {
                        const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);
#pragma unroll
                        for (int i = 0; i < 4; ++i) kv[4 * k4 + i] = fma(w4.v[i], sv, kv[4 * k4 + i]);
                    }
                }
            } else {
                const T* wr = a.w1 + (size_t)w * H;
#pragma unroll
                for (int k = 0; k < HM; ++k)
                    if (k < H) kv[k] = fma(__ldg(wr + k), sv, kv[k]);
            }
        });
        if (tc::rk_backward_combine<HM>(a, sub, dt, yb, su, run, kv, kap)) {
            ++step;
            sub = 0;
            inject(step, yb);
            if (step < a.n_steps) {
                dt = a.step_dt[step];
                tc::rk_backward_first<HM>(a, dt, yb, kap);
            }
        } else {
            ++sub;
        }
    }
    if (live) {
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) a.out[path * H + h] = yb[h];
    }
}

// ---- the parameter gradients of the CUDA-core backward ---------------------------------------------------------------
//
//   dW2 = sum_e g_e h_e^T,  db2 = sum_e g_e,  dW1 = sum_e ub_e z_e^T,  db1 = sum_e ub_e
// over the items e = (stage, path).  A block is one stage x NI paths, one thread per item, dealt to a persistent grid.
// Each thread recomputes its g and ub with mlp_vjp (the backward's code on the dumped z_s and kappa_s) and stages g [HC],
// h [W], ub [W] and z [H] in shared memory, item-minor; the CTA then adds the block's items, in order, to the running
// sums of the parameter entries each thread owns (entry p, p + NI, ...), kept in the CTA's row of the scratch.
// mlp_simt_param_reduce_kernel adds the rows in CTA order: two runs give the same bits.
struct MlpSimtPg {
    int ni;                        // items per block = threads per CTA
    int rs;                        // staging row stride in elements (ni + 1)
    size_t g, h, ub, z;            // staging offsets in elements of T: g [HC][rs], h [W][rs], ub [W][rs], z [H][rs]
    size_t total;                  // bytes of dynamic shared memory
};
constexpr int kMlpPgCtasPerSm = 4;

// the per-CTA parameter vector [W1 | b1 | W2 | b2]
static int64_t mlp_simt_n_params(int64_t H, int64_t C, int64_t W) { return W * H + W + H * C * W + H * C; }

// The staging of ni items after the weights and the per-thread columns of lay (lay built for ni threads)
template <typename T> static MlpSimtPg mlp_simt_pg_layout(const MlpSimtLayout<T>& lay, int H, int C, int W, int ni) {
    MlpSimtPg p;
    p.ni = ni;
    p.rs = ni + 1;
    size_t off = lay.total / sizeof(T);
    p.g = off; off += (size_t)H * C * p.rs;
    p.h = off; off += (size_t)W * p.rs;
    p.ub = off; off += (size_t)W * p.rs;
    p.z = off; off += (size_t)H * p.rs;
    p.total = off * sizeof(T);
    return p;
}

// The widest block (ni_max, ni_max / 2, ... 32 items) whose staging fits, with the weights staged if they fit too; false
// if none does.  Not mlp_simt_fit: the staging after the columns decides, and its rows are ni + 1 elements apart.
template <typename T>
static bool mlp_simt_pg_pick(int H, int C, int W, int ni_max, MlpSimtLayout<T>& lay, MlpSimtPg& pg) {
    for (int ni = ni_max; ni >= 32; ni /= 2) {
        for (int stage = 1; stage >= 0; --stage) {
            lay = mlp_simt_layout<T>(H, C, W, stage != 0, ni);
            pg = mlp_simt_pg_layout<T>(lay, H, C, W, ni);
            if (pg.total <= kMlpSimtMaxSmem) return true;
        }
    }
    return false;
}

template <typename T> struct MlpSimtPgArgs {
    const T* z_stages;            // [n_total][n_paths][H]
    const T* kappa;               // [n_total][n_paths][H]
    T* scratch;                   // [gridDim.x][n_params]
    int64_t n_params;
    int n_total;                  // stages of the solve
};

// a.stage_index, a.stage_frac: the forward's tables
template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads) mlp_simt_param_grad_kernel(const MlpArgs<T> a,
                                                                              const MlpSimtLayout<T> lay,
                                                                              const MlpSimtPg pg,
                                                                              const MlpSimtPgArgs<T> p) {
    using E = exact<T>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq, rs = pg.rs;
    if (lay.staged) {
        TCDE_MLP_STAGE_WEIGHTS()
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;
    T* gs = smem + pg.g + tid;                                     // this item's column of each staging array
    T* hs = smem + pg.h + tid;
    T* us = smem + pg.ub + tid;
    T* zt = smem + pg.z + tid;
    T* mine = p.scratch + (int64_t)blockIdx.x * p.n_params;
    for (int64_t e = tid; e < p.n_params; e += nt) mine[e] = T(0);
    __syncthreads();
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int64_t n_tiles = (a.n_paths + nt - 1) / nt;
    const int64_t n_blocks = n_tiles * p.n_total;
    const int64_t plane = a.n_paths * H;
    const int64_t o_b1 = (int64_t)W * H, o_w2 = o_b1 + W, o_b2 = o_w2 + (int64_t)HC * W;
    for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const int st = (int)(blk / n_tiles);
        const int64_t path = (blk - (int64_t)st * n_tiles) * nt + tid;
        const bool live = path < a.n_paths;
        const int64_t lp = live ? path : a.n_paths - 1;
        T zs[HM];
        const T* zp = p.z_stages + st * plane + lp * H;
        const T* kp = p.kappa + st * plane + lp * H;
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            zs[h] = (h < H) ? zp[h] : T(0);
            if (h < H) {
                kvs[(size_t)h * nt] = live ? kp[h] : T(0);         // a dead item adds zero
                zt[(size_t)h * rs] = zs[h];
            }
        }
        const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);
        {
            TCDE_MLP_SLOPE(a.stage_index[st], a.stage_frac[st])
        }
        mlp_vjp<T, HM>(a, lay, smem, zs, dxs, kvs, nt,
                       [&](int n0, const T* g) {
#pragma unroll
                           for (int j = 0; j < kMlpChunk; ++j)
                               if (n0 + j < HC) gs[(size_t)(n0 + j) * rs] = g[j];
                       },
                       [&](int n0, int w, T pre, T sv) {
                           const T m = pre > T(0) ? sv : T(0);
                           if (n0 == 0) {
                               hs[(size_t)w * rs] = pre > T(0) ? pre : T(0);
                               us[(size_t)w * rs] = m;
                           } else {
                               us[(size_t)w * rs] += m;
                           }
                       });
        __syncthreads();
        // the block's items, in order, into the entries this thread owns
        for (int64_t e = tid; e < p.n_params; e += nt) {
            const T* x;
            const T* y = nullptr;
            if (e < o_b1) { x = smem + pg.ub + (size_t)(e / H) * rs; y = smem + pg.z + (size_t)(e % H) * rs; }
            else if (e < o_w2) { x = smem + pg.ub + (size_t)(e - o_b1) * rs; }
            else if (e < o_b2) { x = smem + pg.g + (size_t)((e - o_w2) / W) * rs; y = smem + pg.h + (size_t)((e - o_w2) % W) * rs; }
            else { x = smem + pg.g + (size_t)(e - o_b2) * rs; }
            T s = mine[e];
            if (y) {
                for (int i = 0; i < nt; ++i) s = fma(x[i], y[i], s);
            } else {
                for (int i = 0; i < nt; ++i) s += x[i];
            }
            mine[e] = s;
        }
        __syncthreads();                                           // the staging is rewritten next
    }
}

// grads += scale * the per-CTA sums, added in CTA order
template <typename T>
__global__ void mlp_simt_param_reduce_kernel(const T* scratch, int n_parts, int64_t n_params, int64_t o_b1, int64_t o_w2,
                                             int64_t o_b2, T scale, T* gw1, T* gb1, T* gw2, T* gb2) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_params) return;
    T s = T(0);
    for (int q = 0; q < n_parts; ++q) s += scratch[(int64_t)q * n_params + i];
    s *= scale;
    if (i < o_b1) { if (gw1) gw1[i] += s; }
    else if (i < o_w2) { if (gb1) gb1[i - o_b1] += s; }
    else if (i < o_b2) { if (gw2) gw2[i - o_w2] += s; }
    else if (gb2) gb2[i - o_b2] += s;
}

// ---- one evaluation of the field, and one adjoint stage, on the CUDA cores (tcde_vector_field_mlp[_vjp]) --------------
//
// One thread per path at one time (index, frac), with the forward's code: f[h] = sum_c tanh(v[(h, c)]) dX_c in increasing
// c, accumulated in the thread's column of shared memory.  With VJP the same pass through mlp_vjp (kappa = the cotangent
// a, in the slope column) also gives f from its tanh values, and a^T df/dz = W1^T (mask . W2^T g) as the Runge-Kutta
// backward forms u_s.  The parameter part is mlp_simt_param_grad_kernel over this one stage, which reads the stage's
// (index, frac) from the device: block 0's thread 0 stores them into q_index / q_frac.
template <typename T> struct MlpFieldEval {
    const T* adj;                 // the cotangent a [n_paths][H] (VJP)
    T* vjp_out;                   // vjp_scale a^T df/dz [n_paths][H] (VJP)
    int32_t* q_index;             // where the stage's interval index and fraction go (VJP, may be null)
    T* q_frac;
    int32_t index;
    T frac, f_scale, vjp_scale;
};

// The per-thread values after the slopes: f [H], and with VJP in fp64 at HM = 32 also the a^T df/dz accumulator [H] and z
// zero padded to Hp (held in registers there beside the chunk, they spill; the first product reads z up to Hp)
template <typename T, int HM, bool VJP> __host__ __device__ constexpr bool mlp_field_kv_shared() {
    return VJP && sizeof(T) == 8 && HM == 32;
}
template <typename T, int HM, bool VJP> static int mlp_field_extra(int H) {
    return !VJP ? 0 : mlp_field_kv_shared<T, HM, VJP>() ? 2 * H + (H + 3) / 4 * 4 : H;
}

// a.z0: z [n_paths][H]; a.out: f_scale f [n_paths][H]; a.sign = 1
template <typename T, int HM, bool VJP>
__global__ void __launch_bounds__(kMlpSimtThreads) mlp_field_kernel(const MlpArgs<T> a, const MlpSimtLayout<T> lay,
                                                                    const MlpFieldEval<T> e) {
    constexpr bool kKvShared = mlp_field_kv_shared<T, HM, VJP>();
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    if (lay.staged) {
        TCDE_MLP_STAGE_WEIGHTS()
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: a of hidden unit h (VJP)
    T* fs = kvs + (size_t)(VJP ? H : 0) * nt;                      // fs[h * nt]: f of hidden unit h
    T* kvx = fs + (size_t)H * nt;                                  // kvx[k * nt]: a^T df/dz_k (kKvShared)
    T* zx = kvx + (size_t)H * nt;                                  // zx[k * nt]: z_k, zero for k >= H (kKvShared)
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);
    if (VJP && e.q_index && blockIdx.x == 0 && tid == 0) {
        *e.q_index = e.index;
        *e.q_frac = e.frac;
    }
    T zin[HM];
#pragma unroll
    for (int h = 0; h < HM; ++h) {
        zin[h] = (h < H) ? a.z0[lp * H + h] : T(0);
        if (h < H) {
            fs[(size_t)h * nt] = T(0);
            if (VJP) kvs[(size_t)h * nt] = e.adj[lp * H + h];
        }
    }
    {
        TCDE_MLP_SLOPE(e.index, e.frac)
    }
    if (!VJP) {
        for (int n0 = 0; n0 < HC; n0 += kMlpChunk) {
            T acc[kMlpChunk];
            TCDE_MLP_CHUNK(acc, n0)
            int h = n0 / C, c = n0 - h * C;
#pragma unroll
            for (int j = 0; j < kMlpChunk; ++j) {
                if (n0 + j < HC) {
                    fs[(size_t)h * nt] = fma(tanh_of(acc[j]), dxs[(size_t)c * nt], fs[(size_t)h * nt]);
                    if (++c == C) { c = 0; ++h; }
                }
            }
        }
    } else {
        T kv[HM];
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            kv[h] = T(0);
            if (kKvShared && h < H) kvx[(size_t)h * nt] = T(0);
            if (kKvShared && h < Hp) zx[(size_t)h * nt] = zin[h];           // zin is zero past H
        }
        struct Column {                                            // z read from the thread's column (kKvShared)
            const T* p;
            int nt;
            __device__ __forceinline__ T operator[](int k) const { return p[(size_t)k * nt]; }
        };
        using Z = std::conditional_t<kKvShared, Column, const T*>;
        Z zarg;
        if constexpr (kKvShared) zarg = Column{zx, nt};
        else zarg = zin;
        mlp_vjp<T, HM>(
            a, lay, smem, zarg, dxs, kvs, nt, [](int, const T*) {},
            [&](int, int w, T pre, T sv) {
                if (!(pre > T(0))) return;
                auto add = [&](int k, T wv) {
                    if constexpr (kKvShared) kvx[(size_t)k * nt] = fma(wv, sv, kvx[(size_t)k * nt]);
                    else kv[k] = fma(wv, sv, kv[k]);
                };
                if (lay.staged) {
                    const T* wr = smem + lay.w1 + (size_t)w * lay.Hp;
#pragma unroll
                    for (int k4 = 0; k4 < HM / 4; ++k4) {
                        if (4 * k4 < lay.Hp) {
                            const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if (!kKvShared || 4 * k4 + i < H) add(4 * k4 + i, w4.v[i]);
                        }
                    }
                } else {
                    const T* wr = a.w1 + (size_t)w * H;
#pragma unroll
                    for (int k = 0; k < HM; ++k)
                        if (k < H) add(k, __ldg(wr + k));
                }
            },
            [&](int h, int c, T y) { fs[(size_t)h * nt] = fma(y, dxs[(size_t)c * nt], fs[(size_t)h * nt]); });
        if (live) {
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) e.vjp_out[path * H + h] = E::mul(e.vjp_scale, kKvShared ? kvx[(size_t)h * nt] : kv[h]);
        }
    }
    if (live) {
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) a.out[path * H + h] = VJP ? E::mul(e.f_scale, fs[(size_t)h * nt]) : fs[(size_t)h * nt];
    }
}

// ---- torchsde's reversible Heun (cdeint(..., backend="torchsde")) on the CUDA cores: one thread per path ---------------
//
// The forward (tcde_cdeint_reversible_heun_mlp) evaluates the field at z_0 = y_0 and then once per step, with the forward's
// own TCDE_MLP_CHUNK into the slope column:
//   z_{n+1} = 2 y_n - z_n + f_n dt_n,  f_{n+1} = F(t_{n+1}, z_{n+1}),  y_{n+1} = y_n + (f_n + f_{n+1}) (0.5 dt_n)
// rounded once per operation in the order of the linear field's kernel (solve_simt.cu), with its output weights and its
// checkpoint layout.  The segment backward (tcde_reversible_heun_mlp_backward_segment) is the recurrence of
// reversible_backward_kernel (solve_tc.cu) with one mlp_vjp pass per step at the reconstructed z_m: its tanh hook gives
// f_m = F(z_m) (the forward's bits) and its units J^T fbar_m.
// y, z, f (and in the backward ybar, zbar, z_m, J^T fbar) are register arrays, or where those would spill (fp64 forward at
// HM = 32, every HM = 32 backward) the thread's columns of shared memory after the slopes.
template <typename T, int HM> __host__ __device__ constexpr bool mlp_rev_fwd_shared() { return sizeof(T) == 8 && HM == 32; }
template <int HM> __host__ __device__ constexpr bool mlp_rev_bwd_shared() { return HM == 32; }
// the backward at HM = 32 runs 64 threads per CTA, so that its columns fit shared memory in fp64
template <int HM> __host__ __device__ constexpr int mlp_rev_bwd_threads() { return HM == 32 ? 64 : kMlpSimtThreads; }
// per-thread values after the slopes: forward y [H], z [Hp], f [H]; backward f_m [H], then y, z, f, ybar, zbar,
// J^T fbar [H] and z_m [Hp] (z and z_m are read up to Hp by the first product)
template <typename T, int HM> static int mlp_rev_fwd_extra(int H) {
    return mlp_rev_fwd_shared<T, HM>() ? 2 * H + (H + 3) / 4 * 4 : 0;
}
template <int HM> static int mlp_rev_bwd_extra(int H) { return mlp_rev_bwd_shared<HM>() ? 7 * H + (H + 3) / 4 * 4 : H; }

template <typename T, int HM, bool SHARED, int NT> struct MlpRevVec {          // HM registers, zero past H
    T v[HM];
    __device__ __forceinline__ void bind(T*) {}
    __device__ __forceinline__ T& operator[](int k) { return v[k]; }
    __device__ __forceinline__ const T* arg() const { return v; }
};
// the thread's column of shared memory for a CTA of NT threads (a compile-time stride: immediate address offsets)
template <typename T, int HM, int NT> struct MlpRevVec<T, HM, true, NT> {
    T* p;
    __device__ __forceinline__ void bind(T* col) { p = col; }
    __device__ __forceinline__ T& operator[](int k) const { return p[k * NT]; }
    __device__ __forceinline__ MlpRevVec arg() const { return *this; }
};

// a.out_slope: the output weights [2][n_out] (w1, then w0); a.stage_index / a.stage_frac: the N + 1 evaluation points;
// ckpt (may be null): [ceil(N / ckpt_stride) + 1][3][n_paths][H]
template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads, 1) cdeint_mlp_rev_kernel(const MlpArgs<T> a, const MlpSimtLayout<T> lay,
                                                                         T* ckpt, int ckpt_stride) {
    constexpr bool kShared = mlp_rev_fwd_shared<T, HM>();
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x;
    constexpr int nt = kMlpSimtThreads;
    const int H = a.H, C = a.C, W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
    if (lay.staged) {
        TCDE_MLP_STAGE_WEIGHTS()
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: F(z_st) of hidden unit h
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);
    MlpRevVec<T, HM, kShared, nt> y, zin, f;                          // zin: z_st, the input of evaluation st
    y.bind(kvs + (size_t)H * nt);
    zin.bind(kvs + (size_t)2 * H * nt);
    f.bind(kvs + (size_t)(2 * H + Hp) * nt);
#pragma unroll
    for (int h = 0; h < HM; ++h) {
        const T v = (h < H) ? a.z0[lp * H + h] : T(0);
        if (!kShared || h < H) { y[h] = v; f[h] = T(0); }
        if (!kShared || h < Hp) zin[h] = v;
    }
    int jn = 0;
    while (jn < a.n_out && a.out_step[jn] < 0) {                   // outputs at t_0: y_0 itself
        if (live) {
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) a.out[(path * a.n_out + jn) * H + h] = y[h];
        }
        ++jn;
    }
    for (int st = 0; st <= a.n_steps; ++st) {
        {
            TCDE_MLP_SLOPE(a.stage_index[st], a.stage_frac[st])
            for (int h = 0; h < H; ++h) kvs[(size_t)h * nt] = T(0);
        }
        for (int n0 = 0; n0 < HC; n0 += kMlpChunk) {
            T acc[kMlpChunk];
            TCDE_MLP_CHUNK(acc, n0)
            int h = n0 / C, c = n0 - h * C;
#pragma unroll
            for (int j = 0; j < kMlpChunk; ++j) {
                if (n0 + j < HC) {
                    kvs[(size_t)h * nt] = fma(tanh_of(acc[j]), dxs[(size_t)c * nt], kvs[(size_t)h * nt]);
                    if (++c == C) { c = 0; ++h; }
                }
            }
        }
        if (st > 0) {
            // step n = st - 1 ends: y_{n+1}, and the outputs w0 y_n + w1 y_{n+1} of this step (torchsde's linear_interp)
            const T half = E::mul(T(0.5), a.step_dt[st - 1]);
            while (jn < a.n_out && a.out_step[jn] == st - 1) {
                const T w1 = a.out_slope[jn], w0 = a.out_slope[a.n_out + jn];
                if (live) {
#pragma unroll
                    for (int h = 0; h < HM; ++h)
                        if (h < H)
                            a.out[(path * a.n_out + jn) * H + h] =
                                E::add(E::mul(w0, y[h]), E::mul(w1, E::add(y[h], E::mul(E::add(f[h], kvs[(size_t)h * nt]),
                                                                                         half))));
                }
                ++jn;
            }
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) y[h] = E::add(y[h], E::mul(E::add(f[h], kvs[(size_t)h * nt]), half));
        }
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) f[h] = kvs[(size_t)h * nt];
        if (ckpt && live && (st % ckpt_stride == 0 || st == a.n_steps)) {
            T* base = ckpt + (int64_t)((st + ckpt_stride - 1) / ckpt_stride) * 3 * a.n_paths * H + path * H;
#pragma unroll
            for (int h = 0; h < HM; ++h) {
                if (h < H) {
                    base[h] = y[h];
                    base[a.n_paths * H + h] = zin[h];
                    base[2 * a.n_paths * H + h] = f[h];
                }
            }
        }
        if (st < a.n_steps) {
            const T dt = a.step_dt[st];
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) zin[h] = E::add(E::sub(E::mul(T(2), y[h]), zin[h]), E::mul(f[h], dt));
        }
    }
}

template <typename T> struct MlpRevBwd {
    const T* ckpt_lo;             // [3][n_paths][H]: y, z, f of step lo
    const T* ckpt_hi;             // ... of step hi
    T* carry;                     // [2][n_paths][H]: ybar, zbar of step hi in (not read when hi = N), of step lo out
    const T* g;                   // [n_paths][n_out][H] output gradients
    const int32_t* inj_range;     // [N + 1][2]: the outputs [first, end) whose gradient lands on y_m
    T* dump_z;                    // [hi - lo, + 1 when hi = N][n_paths][H]: z_m, in slot m - lo
    T* dump_a;                    // ... fbar_m
    int lo, hi;
};

// a.step_dt [N], a.stage_index / a.stage_frac [N + 1], a.out_step [n_out], a.out_slope [2][n_out] (w1, then w0)
template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads, 1) mlp_rev_backward_kernel(const MlpArgs<T> a, const MlpSimtLayout<T> lay,
                                                                           const MlpRevBwd<T> b) {
    constexpr bool kShared = mlp_rev_bwd_shared<HM>();
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x;
    constexpr int nt = mlp_rev_bwd_threads<HM>();
    const int H = a.H, C = a.C, Hp = lay.Hp;
    if (lay.staged) {
        const int W = a.W, HC = a.H * a.C, Nq = lay.Nq;
        TCDE_MLP_STAGE_WEIGHTS()
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: fbar_m, the cotangent of mlp_vjp
    T* fs = kvs + (size_t)H * nt;                                  // fs[h * nt]: f_m = F(z_m) from its tanh values
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);
    MlpRevVec<T, HM, kShared, nt> y, z, f, yb, zb, kv, zm;             // kv: J^T fbar_m; zm: z_m
    {
        T* col = fs + (size_t)H * nt;
        const size_t step = (size_t)H * nt;
        y.bind(col);
        z.bind(col + step);
        f.bind(col + 2 * step);
        yb.bind(col + 3 * step);
        zb.bind(col + 4 * step);
        kv.bind(col + 5 * step);
        zm.bind(col + 6 * step);
    }
#pragma unroll
    for (int h = 0; h < HM; ++h) {
        if (!kShared || h < H) { y[h] = T(0); z[h] = T(0); f[h] = T(0); yb[h] = T(0); zb[h] = T(0); kv[h] = T(0); }
        if (!kShared || h < Hp) zm[h] = T(0);
    }
    const int64_t plane = a.n_paths * H;
    auto load = [&](auto& v, const T* base) {
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) v[h] = base[lp * H + h];
    };
    auto store = [&](T* base, auto& v) {
        if (!live) return;
#pragma unroll
        for (int h = 0; h < HM; ++h)
            if (h < H) base[path * H + h] = v[h];
    };
    auto store_fbar = [&](T* base) {
        if (!live) return;
        for (int h = 0; h < H; ++h) base[path * H + h] = kvs[(size_t)h * nt];
    };
    // v += the output gradients that land on y_m: weight w0 when the output's step is m, 1 at t_0, w1 otherwise
    auto inject = [&](int m, auto& v) {
        for (int j = b.inj_range[2 * m]; j < b.inj_range[2 * m + 1]; ++j) {
            const int os = a.out_step[j];
            const T w = (os == m) ? a.out_slope[a.n_out + j] : (os < 0 ? T(1) : a.out_slope[j]);
            const T* src = b.g + (lp * a.n_out + j) * H;
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) v[h] = fma(w, src[h], v[h]);
        }
    };
    // one pass at evaluation point m: fs = F(z_m), kv = J_F(z_m)^T fbar (fbar in kvs)
    auto vjp = [&](int m) {
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            if (h < H) {
                fs[(size_t)h * nt] = T(0);
                kv[h] = T(0);
            }
        }
        {
            TCDE_MLP_SLOPE(a.stage_index[m], a.stage_frac[m])
        }
        mlp_vjp<T, HM>(
            a, lay, smem, zm.arg(), dxs, kvs, nt, [](int, const T*) {},
            [&](int, int w, T pre, T sv) {
                if (!(pre > T(0))) return;
                if (lay.staged) {
                    const T* wr = smem + lay.w1 + (size_t)w * lay.Hp;
#pragma unroll
                    for (int k4 = 0; k4 < HM / 4; ++k4) {
                        if (4 * k4 < lay.Hp) {
                            const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if (!kShared || 4 * k4 + i < H) kv[4 * k4 + i] = fma(w4.v[i], sv, kv[4 * k4 + i]);
                        }
                    }
                } else {
                    const T* wr = a.w1 + (size_t)w * H;
#pragma unroll
                    for (int k = 0; k < HM; ++k)
                        if (k < H) kv[k] = fma(__ldg(wr + k), sv, kv[k]);
                }
            },
            [&](int h, int c, T yv) { fs[(size_t)h * nt] = fma(yv, dxs[(size_t)c * nt], fs[(size_t)h * nt]); });
    };

    load(y, b.ckpt_hi);
    load(z, b.ckpt_hi + plane);
    load(f, b.ckpt_hi + 2 * plane);
    const bool close = b.hi == a.n_steps;
    if (!close) {
        load(yb, b.carry);
        load(zb, b.carry + plane);
    }
    // m = N (when hi = N) closes the solve: ybar_N = its output gradients, fbar_N = ybar_N dt_{N-1} / 2, z_N from the
    // checkpoint, zbar_N = J^T fbar_N; it is dumped in the last slot
    for (int m = close ? b.hi : b.hi - 1; m >= b.lo; --m) {
        const bool last = m == a.n_steps;
        const T d = last ? T(0) : a.step_dt[m], dp = m > 0 ? a.step_dt[m - 1] : T(0);
        const T hd = E::mul(T(0.5), d), hdp = E::mul(T(0.5), dp);
        // ybar_m = ybar + 2 zbar + (output gradients on y_m);  fbar_m = ybar dt_m / 2 + zbar dt_m + ybar_m dt_{m-1} / 2
        if (!last) {
#pragma unroll
            for (int h = 0; h < HM; ++h) {
                if (h < H) {
                    kvs[(size_t)h * nt] = E::add(E::mul(yb[h], hd), E::mul(zb[h], d));
                    yb[h] = E::add(yb[h], E::mul(T(2), zb[h]));
                }
            }
        }
        inject(m, yb);
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            if (h < H) kvs[(size_t)h * nt] = last ? E::mul(yb[h], hdp) : E::add(kvs[(size_t)h * nt], E::mul(yb[h], hdp));
        }
        if (last) {
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) zm[h] = z[h];
        } else if (m == b.lo) {
            load(zm, b.ckpt_lo + plane);
        } else {
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) zm[h] = E::sub(E::sub(E::mul(T(2), y[h]), z[h]), E::mul(f[h], d));
        }
        vjp(m);
        store(b.dump_z + (int64_t)(m - b.lo) * plane, zm);
        store_fbar(b.dump_a + (int64_t)(m - b.lo) * plane);
        if (m == b.lo) {
            load(y, b.ckpt_lo);
            load(f, b.ckpt_lo + 2 * plane);
        } else if (!last) {
#pragma unroll
            for (int h = 0; h < HM; ++h) {
                if (h < H) {
                    y[h] = E::sub(y[h], E::mul(E::add(fs[(size_t)h * nt], f[h]), hd));
                    f[h] = fs[(size_t)h * nt];
                }
            }
        }
        // zbar_m = J^T fbar_m - zbar (zbar = 0 before step N)
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            if (h < H) {
                z[h] = zm[h];
                zb[h] = E::sub(kv[h], zb[h]);
            }
        }
    }
    store(b.carry, yb);
    store(b.carry + plane, zb);
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

// max |x| of two arrays over the CTA of NT threads (all threads call it; contains __syncthreads)
template <int NT>
__device__ __forceinline__ void cta_max(float* red, int tid, float& a, float& b, float& c, float& d) {
    float v[4] = {a, b, c, d};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[i] = fmaxf(v[i], __shfl_xor_sync(0xffffffffu, v[i], o));
        if ((tid & 31) == 0) red[i * (NT / 32) + (tid >> 5)] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[i] = 0.f;
        for (int w = 0; w < NT / 32; ++w) v[i] = fmaxf(v[i], red[i * (NT / 32) + w]);
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

// the split weight tiles and scaled biases in shared memory, by a CTA of NT threads
template <int NT = kThreads>
__device__ __forceinline__ Scales prepare(unsigned char* smem, const float* w1, const float* b1, const float* w2,
                                          const float* b2, int tid) {
    float* red = reinterpret_cast<float*>(smem + Smem::red);
    float m1 = 0.f, mb1 = 0.f, m2 = 0.f, mb2 = 0.f;
    for (int e = tid; e < kWidth * kHid; e += NT) m1 = fmaxf(m1, fabsf(w1[e]));
    for (int e = tid; e < kWidth; e += NT) mb1 = fmaxf(mb1, fabsf(b1[e]));
    for (int e = tid; e < kCols * kWidth; e += NT) m2 = fmaxf(m2, fabsf(w2[e]));
    for (int e = tid; e < kCols; e += NT) mb2 = fmaxf(mb2, fabsf(b2[e]));
    cta_max<NT>(red, tid, m1, mb1, m2, mb2);
    Scales s;
    float s1, s2;
    split_scales(m1, mb1, s1, s.inv1, s.beta1);
    split_scales(m2, mb2, s2, s.inv2, s.beta2);
    __half* t1 = reinterpret_cast<__half*>(smem + Smem::w1);
    for (int e = tid; e < kWidth * kHid; e += NT) {     // [128 rows][hi k 0..31 | lo k 0..31], 16-byte chunks swizzled
        const int n = e >> 5, k = e & 31;
        const float w = w1[e] * s1;
        const __half hi = __float2half_rn(w);
        const __half lo = __float2half_rn(w - __half2float(hi));
        t1[n * 64 + (((k >> 3) ^ (n & 7)) << 3) + (k & 7)] = hi;
        t1[n * 64 + ((((k >> 3) + 4) ^ (n & 7)) << 3) + (k & 7)] = lo;
    }
    __half* t2 = reinterpret_cast<__half*>(smem + Smem::w2);
    for (int e = tid; e < kCols * kWidth; e += NT) {    // region (piece, k block): [256 rows][64 halves], swizzled
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
    for (int n = tid; n < kWidth; n += NT) sb1[n] = b1[n] * s1;   // powers of two: exact
    for (int n = tid; n < kCols; n += NT) sb2[n] = b2[n] * s2;
    return s;
}

// Steps 1 and 2 of field for the warpgroup's 64 rows: h = relu(W1 zin + b1), unscaled, into u (column 64 c + 8 j + 2 q + e
// of row r at u[c][4 j + 2 r + e]), and the second product's row scales rs / inv2 (times 1 / weight scale) and hi / lo A
// fragments [k step][4].  The backward kernels call it too, so that their ReLU masks and tanh values are the forward's bits.
__device__ __forceinline__ void hidden_layer(const float* zin, const Scales& sc, const float* sb1, uint32_t tile1, int q,
                                             float (*u)[wg::kAcc], float* rs, float* inv2, uint32_t (*bhi)[4],
                                             uint32_t (*blo)[4]) {
    using namespace wg;
    // 1. u = z W1^T + b1, row-scaled: A from the stage input as in wg::field
    float inv[2];
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
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 1));
        m2[r] = fmaxf(m2[r], __shfl_xor_sync(0xffffffffu, m2[r], 2));
        row_scale(m2[r], rs[r], inv2[r]);
        inv2[r] *= sc.inv2;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int t = 0; t < 4; ++t) {                          // A column 16 k + 8 (t >> 1) + 2 q = u column 64 c + 8 j + 2 q
            const int r = t & 1, c = k >> 2, j = 2 * (k & 3) + (t >> 1);
            split_h2(__fmul_rn(u[c][4 * j + 2 * r], rs[r]), __fmul_rn(u[c][4 * j + 2 * r + 1], rs[r]), bhi[k][t],
                     blo[k][t]);
        }
}

// Step 3 of field for one chunk (hidden units 8 chunk .. 8 chunk + 7): d = (h W2^T + b2) of the chunk's 64 columns, scaled
// by the rows' rs and the weight scale, as 24 wgmmas committed as one group (small terms first)
__device__ __forceinline__ void issue_v(int chunk, float* d, const float* sb2, const float* rs, uint32_t tile2, int q,
                                        const uint32_t (*bhi)[4], const uint32_t (*blo)[4]) {
    using namespace wg;
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
        const float2 bb = *reinterpret_cast<const float2*>(sb2 + chunk * kN + 8 * j + 2 * q);
        d[4 * j + 0] = bb.x * rs[0]; d[4 * j + 1] = bb.y * rs[0];
        d[4 * j + 2] = bb.x * rs[1]; d[4 * j + 3] = bb.y * rs[1];
    }
    mma_fence();
    const uint32_t rows = tile2 + chunk * kN * 128;
    const uint32_t hi = rows, lo = rows + 2 * kW2Region;      // piece regions; k block kb at + kb * kW2Region
#pragma unroll
    for (int k = 0; k < 8; ++k)                                // h_lo . W2_hi
        mma_m64n64k16(d, blo[k], desc_sw128(hi + (k >> 2) * kW2Region + 32 * (k & 3)));
#pragma unroll
    for (int k = 0; k < 8; ++k)                                // h_hi . W2_lo
        mma_m64n64k16(d, bhi[k], desc_sw128(lo + (k >> 2) * kW2Region + 32 * (k & 3)));
#pragma unroll
    for (int k = 0; k < 8; ++k)                                // h_hi . W2_hi
        mma_m64n64k16(d, bhi[k], desc_sw128(hi + (k >> 2) * kW2Region + 32 * (k & 3)));
    mma_commit();
}

// One evaluation of the MLP field for the warpgroup's 64 rows: kv = tanh(W2 relu(W1 zin + b1) + b2) . dx in the fragment
// layout; dx: the lane's two channels of both rows, times the sign of the time direction.  mid() runs during the second
// product (the caller's next dX/dt hides behind the MMAs).
template <typename Mid>
__device__ __forceinline__ void field(const float* zin, const float (*dx)[2], const Scales& sc, const float* sb1,
                                      const float* sb2, uint32_t tile1, uint32_t tile2, int q, float* kv, Mid mid) {
    using namespace wg;
    float u[2][kAcc], rs[2], inv2[2];
    uint32_t bhi[8][4], blo[8][4];
    hidden_layer(zin, sc, sb1, tile1, q, u, rs, inv2, bhi, blo);

    // 3. v = h W2^T + b2 in four chunks of 64 columns, 4. tanh, contraction with dX/dt
    float acc[2][kAcc];
    issue_v(0, acc[0], sb2, rs, tile2, q, bhi, blo);
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        float* d = acc[c & 1];
        if (c + 1 < kChunks) {
            issue_v(c + 1, acc[(c + 1) & 1], sb2, rs, tile2, q, bhi, blo);
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

// DUMP: the input of every stage also goes to a.stage_dump[stage][path][32] (the forward state of the backward kernels)
template <bool DUMP>
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
    float* dump_at = a.stage_dump;
    for (int st = 0; st < n_st; ++st) {
        if (DUMP) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!live[r]) continue;
                float2* dst = reinterpret_cast<float2*>(dump_at + path[r] * kHid) + q;
#pragma unroll
                for (int i = 0; i < 4; ++i) dst[4 * i] = make_float2(zin[8 * r + 2 * i], zin[8 * r + 2 * i + 1]);
            }
            dump_at += a.n_paths * kHid;
        }
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

// ---- the backward of the tensor-core solve (cdeint(..., adjoint=False)): the transposed Runge-Kutta recurrence ---------
//
// F_s(z) = tanh(v).view(H, C) dX_s with v = W2 h + b2, h = relu(W1 z + b1), so the stage product is
//   u_s = J_s^T kappa_s = W1^T (mask . W2^T g),   g[(h, c)] = (1 - y^2)[(h, c)] kappa_s[h] dX_s[c],   mask = (h > 0),
// evaluated at the forward's stage input z_s (read back from its dump).  hidden_layer and issue_v recompute h and v with
// the forward's own code, so the mask and tanh values are the forward's bits.  The two transposed products read the
// forward's K-major tiles as MN-major B operands through ldmatrix.trans and run as warp-level m16n8k16 MMAs on the same
// fragment layout (2xFP16 split, per-row powers of two, small terms first).  g (256 columns) is too large to keep as A
// fragments next to h's, so each warp parks its 16 rows of g in shared memory (fp32) and scales them by the exact row
// max; that tile is why the CTA holds ONE warpgroup: 145 KB of weights + 4 x 16.5 KB of g fit in 227 KB, 8 warps' would not.
constexpr int kBwdThreads = wg::kThreads;
constexpr int kGStride = kCols + 8;                          // floats per row of a warp's g tile (rows g, g + 4 8 banks apart)
struct BwdSmem {
    static constexpr int g = Smem::bytes;                    // per warp: [16 rows][kGStride] floats
    static constexpr int bytes = g + (kBwdThreads / 32) * 16 * kGStride * 4;
};
constexpr int kBwdSmem = BwdSmem::bytes + 1024;

__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr)
                 : "memory");
}

// g of one chunk (columns 64 c + 8 j + 2 q + e: unit 8 c + j, channel 2 q + e) from its scaled accumulator d:
// gc[4 j + 2 r + e] = (1 - y^2) kc[r][j] dx[r][e], kc[r][j] = kappa of unit 8 c + j of row r
__device__ __forceinline__ void slope_cotangent(const float* d, const float* inv2, const float (*kc)[8], const float (*dx)[2],
                                                float* gc) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float y = tanhf(__fmul_rn(d[4 * j + 2 * r + e], inv2[r]));
                gc[4 * j + 2 * r + e] = __fmul_rn(__fsub_rn(1.f, __fmul_rn(y, y)), __fmul_rn(kc[r][j], dx[r][e]));
            }
}

// hd = g W2 (K = 256, N = 128) for the warp's 16 rows: g from the warp's tile gt scaled per row by rsg, W2 from the
// forward's tile.  hd[j][2 r + e]: column 8 j + 2 q + e of row g + 8 r.
__device__ __forceinline__ void hdot_product(const float* gt, const float* rsg, uint32_t tile2, int lane, float (*hd)[4]) {
    const int g = lane >> 2, q = lane & 3;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) hd[j][i] = 0.f;
    const int nl = (lane & 7) + 8 * ((lane >> 3) & 1);       // the W2 row (within the k step) this lane addresses
#pragma unroll 1
    for (int ks = 0; ks < kCols / 16; ++ks) {
        uint32_t ahi[4], alo[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {                          // register t: row t & 1, columns 16 ks + 8 (t >> 1) + 2 q, +1
            const int r = t & 1;
            const float2 v = *reinterpret_cast<const float2*>(gt + (g + 8 * r) * kGStride + 16 * ks + 8 * (t >> 1) + 2 * q);
            split_h2(__fmul_rn(v.x, rsg[r]), __fmul_rn(v.y, rsg[r]), ahi[t], alo[t]);
        }
        const int n = 16 * ks + nl;
#pragma unroll
        for (int np = 0; np < 8; ++np) {
            const int chunk = 2 * np + (lane >> 4);            // W2 columns 8 chunk .. 8 chunk + 7
            const uint32_t at = tile2 + (chunk >> 3) * kW2Region + n * 128 + (((chunk & 7) ^ (n & 7)) << 4);
            uint32_t bh[4], bl[4];
            ldsm_x4_t(at, bh);
            ldsm_x4_t(at + 2 * kW2Region, bl);
#pragma unroll
            for (int h = 0; h < 2; ++h) {                      // small terms first
                mma_f16(hd[2 * np + h], alo, bh[2 * h], bh[2 * h + 1]);
                mma_f16(hd[2 * np + h], ahi, bl[2 * h], bl[2 * h + 1]);
                mma_f16(hd[2 * np + h], ahi, bh[2 * h], bh[2 * h + 1]);
            }
        }
    }
}

// max |x| over each of the lane's two rows, reduced over the quad
__device__ __forceinline__ void quad_row_max(float* m) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
    }
}

// The part of a stage's backward both kernels share: g of every chunk into the warp's tile gt, then ub = mask . (W2^T g)
// unscaled (ub[j][2 r + e]: hidden unit 8 j + 2 q + e of row r).  kap: the lane's kappa in the state layout.
__device__ __forceinline__ void stage_ubar(const float* zs, const float* kap, const float (*dx)[2], const Scales& sc,
                                           const float* sb1, const float* sb2, uint32_t tile1, uint32_t tile2, int lane,
                                           float* gt, float (*ub)[4]) {
    using namespace wg;
    const int g = lane >> 2, q = lane & 3;
    float u[2][kAcc], rs[2], inv2[2];
    uint32_t bhi[8][4], blo[8][4];
    hidden_layer(zs, sc, sb1, tile1, q, u, rs, inv2, bhi, blo);
    uint32_t mask[2] = {0u, 0u};
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int i = 0; i < kAcc; ++i) mask[c] |= (u[c][i] > 0.f ? 1u : 0u) << i;
    float acc[2][kAcc], gmax[2] = {0.f, 0.f};
    issue_v(0, acc[0], sb2, rs, tile2, q, bhi, blo);
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
        float* d = acc[c & 1];
        if (c + 1 < kChunks) {
            issue_v(c + 1, acc[(c + 1) & 1], sb2, rs, tile2, q, bhi, blo);
            mma_wait<1>();
        } else {
            mma_wait<0>();
        }
        pin(d);
        float kc[2][8], gc[kAcc];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int r = 0; r < 2; ++r) kc[r][j] = __shfl_sync(0xffffffffu, kap[8 * r + 2 * c + (j & 1)], (lane & ~3) | (j >> 1));
        slope_cotangent(d, inv2, kc, dx, gc);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                *reinterpret_cast<float2*>(gt + (g + 8 * r) * kGStride + 64 * c + 8 * j + 2 * q) =
                    make_float2(gc[4 * j + 2 * r], gc[4 * j + 2 * r + 1]);
                gmax[r] = fmaxf(gmax[r], fmaxf(fabsf(gc[4 * j + 2 * r]), fabsf(gc[4 * j + 2 * r + 1])));
            }
    }
    __syncwarp();
    quad_row_max(gmax);
    float rsg[2], invg[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) row_scale(gmax[r], rsg[r], invg[r]);
    hdot_product(gt, rsg, tile2, lane, ub);
    __syncwarp();                                              // the tile is rewritten next
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = i >> 1;
            const float v = __fmul_rn(__fmul_rn(ub[j][i], invg[r]), sc.inv2);
            ub[j][i] = ((mask[j >> 3] >> (4 * (j & 7) + i)) & 1u) ? v : 0.f;
        }
}

// kv = W1^T ub (K = 128, N = 32) in the state layout kv[8 r + 2 i + e] (unit 8 i + 2 q + e of row r)
__device__ __forceinline__ void input_product(const float (*ub)[4], float inv1, uint32_t tile1, int lane, float* kv) {
    float m[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) m[i >> 1] = fmaxf(m[i >> 1], fabsf(ub[j][i]));
    quad_row_max(m);
    float rs[2], inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) row_scale(m[r], rs[r], inv[r]);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
    const int nl = (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
    for (int kk = 0; kk < kWidth / 16; ++kk) {
        uint32_t ahi[4], alo[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {                          // A column 16 kk + 8 (t >> 1) + 2 q = ub tile 2 kk + (t >> 1)
            const int r = t & 1, j = 2 * kk + (t >> 1);
            split_h2(__fmul_rn(ub[j][2 * r], rs[r]), __fmul_rn(ub[j][2 * r + 1], rs[r]), ahi[t], alo[t]);
        }
        const int n = 16 * kk + nl;                            // W1 row = hidden unit
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int chunk = 2 * p + (lane >> 4);
            uint32_t bh[4], bl[4];
            ldsm_x4_t(tile1 + n * 128 + ((chunk ^ (n & 7)) << 4), bh);
            ldsm_x4_t(tile1 + n * 128 + (((chunk + 4) ^ (n & 7)) << 4), bl);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                mma_f16(acc[2 * p + h], alo, bh[2 * h], bh[2 * h + 1]);
                mma_f16(acc[2 * p + h], ahi, bl[2 * h], bl[2 * h + 1]);
                mma_f16(acc[2 * p + h], ahi, bh[2 * h], bh[2 * h + 1]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int e = 0; e < 2; ++e) kv[8 * r + 2 * i + e] = __fmul_rn(__fmul_rn(acc[i][2 * r + e], inv[r]), inv1);
}

// The lane's rows of the warpgroup's 64 paths, the control reads and dX/dt of cdeint_mlp_wgmma_kernel, for the backward
// kernels (path0: the first of the 64)
struct BwdRows {
    int64_t path[2], lpath[2];
    bool live[2];
    const float2* crow;
    int row1, row_f2;
    bool cubic;
    float sign;

    __device__ __forceinline__ BwdRows(const float* control, int control_kind, int64_t n_rows, int64_t n_paths,
                                       int64_t path0, int warp, int g, int q, float sgn) {
        cubic = (control_kind == TCDE_CONTROL_CUBIC);
        row_f2 = (cubic ? 4 * kCh : kCh) / 2;
        sign = sgn;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            path[r] = path0 + 16 * warp + g + 8 * r;
            live[r] = path[r] < n_paths;
            lpath[r] = live[r] ? path[r] : n_paths - 1;
        }
        row1 = (int)(lpath[1] - lpath[0]);
        crow = reinterpret_cast<const float2*>(control + lpath[0] * n_rows * (2 * row_f2) + (cubic ? kCh : 0)) + q;
    }
    __device__ __forceinline__ void fetch(int64_t n_rows, int interval, float2 (*raw)[3]) const {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2* src = crow + (r * row1 * n_rows + interval) * row_f2;
            raw[r][0] = __ldg(src);
            if (cubic) { raw[r][1] = __ldg(src + 4); raw[r][2] = __ldg(src + 8); }
        }
    }
    // dX/dt at fraction fr, channels 2q, 2q + 1 of both rows, times the sign (the forward's slope, bit for bit)
    __device__ __forceinline__ void slope(const float2 (*raw)[3], float fr, float (*dx)[2]) const {
        using E = exact<float>;
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
    }
    // the lane's 16 values of a [path][32] block (dead rows read the last path)
    __device__ __forceinline__ void load(const float* base, int q, float* v) const {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2* src = reinterpret_cast<const float2*>(base + lpath[r] * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 t = src[4 * i];
                v[8 * r + 2 * i] = t.x; v[8 * r + 2 * i + 1] = t.y;
            }
        }
    }
    __device__ __forceinline__ void store(float* base, int q, const float* v) const {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!live[r]) continue;
            float2* dst = reinterpret_cast<float2*>(base + path[r] * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[4 * i] = make_float2(v[8 * r + 2 * i], v[8 * r + 2 * i + 1]);
        }
    }
};

// The Runge-Kutta backward of the MLP field on the host-reversed schedule (a.step_dt etc. reversed, as in
// tcde_cdeint_fixed_linear_backward): the state is the cotangent ybar, the output gradients a.grad_out are added at every
// grid state (a.inj_*), kappa_s goes to a.stage_dump (when given) in the forward's slot, dL/dz0 to a.out.  z_dump: the
// forward's stage inputs.
__global__ void __launch_bounds__(kBwdThreads, 1) cdeint_mlp_backward_kernel(const UmmaArgs a, const float* w2,
                                                                             const float* b2, const float* z_dump) {
    using E = exact<float>;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((1024u - (smem_u32(smem_unaligned) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const Scales sc = prepare<kBwdThreads>(smem, a.weight, a.bias, w2, b2, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const float* sb1 = reinterpret_cast<const float*>(smem + Smem::b1);
    const float* sb2 = reinterpret_cast<const float*>(smem + Smem::b2);
    const uint32_t tile1 = smem_u32(smem + Smem::w1), tile2 = smem_u32(smem + Smem::w2);
    float* gt = reinterpret_cast<float*>(smem + BwdSmem::g) + warp * 16 * kGStride;
    const BwdRows rows(a.control, a.control_kind, a.n_rows, a.n_paths, (int64_t)blockIdx.x * wg::kPaths, warp, g, q,
                       a.sign < 0.f ? -1.f : 1.f);

    // v += the output gradients that land on grid state r (counted from the end of the solve)
    auto inject = [&](int r, float* v) {
        for (int e = a.inj_range[r]; e < a.inj_range[r + 1]; ++e) {
            const int j = a.inj_out[e];
            const float w = a.inj_weight[e];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const float2* src = reinterpret_cast<const float2*>(a.grad_out + (rows.lpath[rr] * a.n_out + j) * kHid) + q;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 t = src[4 * i];
                    v[8 * rr + 2 * i] = E::add(v[8 * rr + 2 * i], E::mul(w, t.x));
                    v[8 * rr + 2 * i + 1] = E::add(v[8 * rr + 2 * i + 1], E::mul(w, t.y));
                }
            }
        }
    };

    float yb[wg::kNV], su[wg::kNV], run[wg::kNV], kap[wg::kNV];
#pragma unroll
    for (int h = 0; h < wg::kNV; ++h) { yb[h] = 0.f; su[h] = 0.f; run[h] = 0.f; }
    inject(0, yb);
    rk_backward_first<wg::kNV>(a, a.step_dt[0], yb, kap);

    const int n_st = a.n_steps * a.n_stages;
    const int64_t plane = a.n_paths * kHid;
    const float* z_at = z_dump + (int64_t)(n_st - 1) * plane;     // stage st's forward slot, walking down
    float* k_at = a.stage_dump ? a.stage_dump + (int64_t)(n_st - 1) * plane : nullptr;
    float dx[2][2];
    {
        float2 raw[2][3];
        rows.fetch(a.n_rows, a.stage_index[0], raw);
        rows.slope(raw, a.stage_frac[0], dx);
    }
    int step = 0, sub = 0;
    float dt = a.step_dt[0];
    for (int st = 0; st < n_st; ++st) {
        if (k_at) {
            rows.store(k_at, q, kap);
            k_at -= plane;
        }
        float zs[wg::kNV];
        rows.load(z_at, q, zs);
        z_at -= plane;
        float2 nxt[2][3];
        if (st + 1 < n_st) rows.fetch(a.n_rows, a.stage_index[st + 1], nxt);
        float ub[16][4], kv[wg::kNV];
        stage_ubar(zs, kap, dx, sc, sb1, sb2, tile1, tile2, lane, gt, ub);
        input_product(ub, sc.inv1, tile1, lane, kv);
        if (st + 1 < n_st) rows.slope(nxt, a.stage_frac[st + 1], dx);
        if (rk_backward_combine<wg::kNV>(a, sub, dt, yb, su, run, kv, kap)) {
            ++step;
            sub = 0;
            inject(step, yb);
            if (step < a.n_steps) {
                dt = a.step_dt[step];
                rk_backward_first<wg::kNV>(a, dt, yb, kap);
            }
        } else {
            ++sub;
        }
    }
    rows.store(a.out, q, yb);
}

// ---- the parameter gradients of the backward: dW2, db2 (blockIdx.y = chunk b < 4) and dW1, db1 (blockIdx.y = 4) --------
//
//   dW2 = sum_e g_e h_e^T,  db2 = sum_e g_e,  dW1 = sum_e ub_e z_e^T,  db1 = sum_e ub_e
// over the items e = (stage, path), with g and ub recomputed from (z_s, kappa_s, dX_s) as the backward kernel forms them
// (they are far too large to store).  Work item = one stage x 64 paths, dealt to persistent CTAs of one warpgroup; each
// CTA's y index picks what it accumulates, so its accumulators stay in registers:
//   * y = b < 4: v of chunk b only (its 64 columns of g need h but one quarter of the second product); g_b and h go to
//     shared memory and G_b^T [H | 1] (K = 64 items, M = 64, N = 128 + a column of ones for db2) runs as m16n8k16 MMAs;
//   * y = 4: the whole ub (stage_ubar), then ub^T [z | 1] (M = 128, N = 32 + ones).
// Operands are split into two BF16 pieces (no scaling; three MMAs, small terms first), each item is accumulated in
// fresh registers and added to the CTA's running sums in fp32, and the per-CTA sums are added in a fixed order by
// mlp_param_reduce_kernel: two runs give the same bits.
constexpr int kPgY = wg::kChunks + 1;
constexpr int kPgParams = kWidth * kHid + kWidth + kCols * kWidth + kCols;   // [W1 | b1 | W2 | b2]
constexpr int kOffB1 = kWidth * kHid, kOffW2 = kOffB1 + kWidth, kOffB2 = kOffW2 + kCols * kWidth;
constexpr int kGS = wg::kN + 4, kHS = kWidth + 4, kZS = kHid + 4;             // padded fp32 staging rows
struct PgSmem {
    static constexpr int stage = BwdSmem::g;                 // y < 4: G [64][kGS], H [64][kHS]; y = 4: the g tiles, then
    static constexpr int h = stage + 64 * kGS * 4;           // per warp ub [16][kHS] and z [16][kZS] in its own tile
    static constexpr int bytes_b = h + 64 * kHS * 4;
    static constexpr int bytes = bytes_b > BwdSmem::bytes ? bytes_b : BwdSmem::bytes;
};
constexpr int kPgSmem = PgSmem::bytes + 1024;

__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ float bf_round(float x) { return __uint_as_float(pack_bf2(x, 0.f) << 16); }
__device__ __forceinline__ void split_bf2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    const float h0 = bf_round(v0), h1 = bf_round(v1);
    hi = pack_bf2(h0, h1);
    lo = pack_bf2(__fsub_rn(v0, h0), __fsub_rn(v1, h1));
}
__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[m][t] += sum over the 64 items i of A[i][row] B[i][col] for the warp's MT m-tiles of rows and NT n-tiles of columns
// (the last n-tile: a column of ones, then zeros).  a(i, row), b(i, col): the staged fp32 values.
template <int MT, int NT, typename FA, typename FB>
__device__ __forceinline__ void outer_items(float (*acc)[NT][4], int row0, int lane, FA a, FB b) {
    const int g = lane >> 2, q = lane & 3;
    float part[MT][NT][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) part[m][t][i] = 0.f;
#pragma unroll 1
    for (int i0 = 0; i0 < 64; i0 += 16) {
        uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int r = 0; r < 2; ++r) {                      // b0 / b1: items i0 + 2 q (+1) + 8 r, column 8 t + g
                const int i = i0 + 2 * q + 8 * r, col = 8 * t + g;
                if (t == NT - 1) {
                    const float one = (g == 0) ? 1.f : 0.f;
                    bh[t][r] = pack_bf2(one, one);
                    bl[t][r] = 0u;
                } else {
                    split_bf2(b(i, col), b(i + 1, col), bh[t][r], bl[t][r]);
                }
            }
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            uint32_t ah[4], al[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {                      // register t: row g + 8 (t & 1), items i0 + 2 q + 8 (t >> 1), +1
                const int row = row0 + 16 * m + g + 8 * (t & 1), i = i0 + 2 * q + 8 * (t >> 1);
                split_bf2(a(i, row), a(i + 1, row), ah[t], al[t]);
            }
#pragma unroll
            for (int t = 0; t < NT; ++t) {
                mma_bf16(part[m][t], al, bh[t][0], bh[t][1]);
                mma_bf16(part[m][t], ah, bl[t][0], bl[t][1]);
                mma_bf16(part[m][t], ah, bh[t][0], bh[t][1]);
            }
        }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[m][t][i] += part[m][t][i];
}

struct PgArgs {
    const float* control;
    const float* w1;
    const float* b1;
    const float* w2;
    const float* b2;
    const float* z_stages;        // [n_total][n_paths][32]
    const float* kappa;           // [n_total][n_paths][32]
    const int32_t* stage_index;   // [n_total] (forward order)
    const float* stage_frac;
    float* scratch;               // [gridDim.x][kPgParams]
    int64_t n_paths, n_rows;
    int control_kind, n_total;
    float sign;
};

__global__ void __launch_bounds__(kBwdThreads, 1) mlp_param_grad_kernel(const PgArgs a) {
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((1024u - (smem_u32(smem_unaligned) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const Scales sc = prepare<kBwdThreads>(smem, a.w1, a.b1, a.w2, a.b2, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const float* sb1 = reinterpret_cast<const float*>(smem + Smem::b1);
    const float* sb2 = reinterpret_cast<const float*>(smem + Smem::b2);
    const uint32_t tile1 = smem_u32(smem + Smem::w1), tile2 = smem_u32(smem + Smem::w2);
    const int b = blockIdx.y;
    float* gs = reinterpret_cast<float*>(smem + PgSmem::stage);
    float* hs = reinterpret_cast<float*>(smem + PgSmem::h);
    float* wt = reinterpret_cast<float*>(smem + BwdSmem::g) + warp * 16 * kGStride;      // y = 4: the warp's g tile
    float* mine = a.scratch + (size_t)blockIdx.x * kPgParams;

    const int64_t n_tiles = (a.n_paths + wg::kPaths - 1) / wg::kPaths;
    const int64_t n_items = n_tiles * a.n_total;
    const int64_t plane = a.n_paths * kHid;
    if (b < wg::kChunks) {
        float acc[1][17][4];
#pragma unroll
        for (int t = 0; t < 17; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[0][t][i] = 0.f;
        for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int e = (int)(item / n_tiles);
            const int64_t path0 = (item - (int64_t)e * n_tiles) * wg::kPaths;
            const BwdRows rows(a.control, a.control_kind, a.n_rows, a.n_paths, path0, warp, g, q, a.sign < 0.f ? -1.f : 1.f);
            float zs[wg::kNV], dx[2][2], kc[2][8];
            rows.load(a.z_stages + e * plane, q, zs);
            {
                float2 raw[2][3];
                rows.fetch(a.n_rows, a.stage_index[e], raw);
                rows.slope(raw, a.stage_frac[e], dx);
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {                      // kappa of the chunk's units 8 b .. 8 b + 7 (zero on dead rows)
                const float4* src = reinterpret_cast<const float4*>(a.kappa + e * plane + rows.lpath[r] * kHid + 8 * b);
                const float4 k0 = src[0], k1 = src[1];
                const float live = rows.live[r] ? 1.f : 0.f;
                kc[r][0] = k0.x * live; kc[r][1] = k0.y * live; kc[r][2] = k0.z * live; kc[r][3] = k0.w * live;
                kc[r][4] = k1.x * live; kc[r][5] = k1.y * live; kc[r][6] = k1.z * live; kc[r][7] = k1.w * live;
            }
            float u[2][wg::kAcc], rs[2], inv2[2], d[wg::kAcc], gc[wg::kAcc];
            uint32_t bhi[8][4], blo[8][4];
            hidden_layer(zs, sc, sb1, tile1, q, u, rs, inv2, bhi, blo);
            issue_v(b, d, sb2, rs, tile2, q, bhi, blo);
            wg::mma_wait<0>();
            wg::pin(d);
            slope_cotangent(d, inv2, kc, dx, gc);
            __syncthreads();                                   // the previous item's outer product is done with the tiles
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = 16 * warp + g + 8 * r;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    *reinterpret_cast<float2*>(gs + row * kGS + 8 * j + 2 * q) = make_float2(gc[4 * j + 2 * r], gc[4 * j + 2 * r + 1]);
#pragma unroll
                    for (int c = 0; c < 2; ++c)
                        *reinterpret_cast<float2*>(hs + row * kHS + 64 * c + 8 * j + 2 * q) =
                            make_float2(u[c][4 * j + 2 * r], u[c][4 * j + 2 * r + 1]);
                }
            }
            __syncthreads();
            outer_items<1, 17>(acc, 16 * warp, lane, [&](int i, int row) { return gs[i * kGS + row]; },
                               [&](int i, int col) { return hs[i * kHS + col]; });
        }
        // accumulator t: rows n = 16 w + g (+8) of chunk b, columns 8 t + 2 q (+1); t = 16, column 0: db2
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int n = 64 * b + 16 * warp + g + 8 * r;
#pragma unroll
            for (int t = 0; t < 16; ++t)
                *reinterpret_cast<float2*>(mine + kOffW2 + n * kWidth + 8 * t + 2 * q) =
                    make_float2(acc[0][t][2 * r], acc[0][t][2 * r + 1]);
            if (q == 0) mine[kOffB2 + n] = acc[0][16][2 * r];
        }
        return;
    }
    float acc[2][5][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int t = 0; t < 5; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[m][t][i] = 0.f;
    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int e = (int)(item / n_tiles);
        const int64_t path0 = (item - (int64_t)e * n_tiles) * wg::kPaths;
        const BwdRows rows(a.control, a.control_kind, a.n_rows, a.n_paths, path0, warp, g, q, a.sign < 0.f ? -1.f : 1.f);
        float zs[wg::kNV], kap[wg::kNV], dx[2][2];
        rows.load(a.z_stages + e * plane, q, zs);
        rows.load(a.kappa + e * plane, q, kap);
#pragma unroll
        for (int h = 0; h < wg::kNV; ++h)
            if (!rows.live[h >> 3]) kap[h] = 0.f;
        {
            float2 raw[2][3];
            rows.fetch(a.n_rows, a.stage_index[e], raw);
            rows.slope(raw, a.stage_frac[e], dx);
        }
        __syncthreads();                                       // the previous item's outer product is done with the tiles
        float ub[16][4];
        stage_ubar(zs, kap, dx, sc, sb1, sb2, tile1, tile2, lane, wt, ub);
        float* us = wt;                                        // the warp's rows: ub [16][kHS], then z [16][kZS]
        float* zt = wt + 16 * kHS;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = g + 8 * r;
#pragma unroll
            for (int j = 0; j < 16; ++j)
                *reinterpret_cast<float2*>(us + row * kHS + 8 * j + 2 * q) = make_float2(ub[j][2 * r], ub[j][2 * r + 1]);
#pragma unroll
            for (int i = 0; i < 4; ++i)
                *reinterpret_cast<float2*>(zt + row * kZS + 8 * i + 2 * q) = make_float2(zs[8 * r + 2 * i], zs[8 * r + 2 * i + 1]);
        }
        __syncthreads();
        const float* base = reinterpret_cast<const float*>(smem + BwdSmem::g);
        outer_items<2, 5>(acc, 32 * warp, lane,
                          [&](int i, int row) { return base[(i >> 4) * 16 * kGStride + (i & 15) * kHS + row]; },
                          [&](int i, int col) { return base[(i >> 4) * 16 * kGStride + 16 * kHS + (i & 15) * kZS + col]; });
    }
    // accumulator (m, t): rows k = 32 w + 16 m + g (+8), columns 8 t + 2 q (+1); t = 4, column 0: db1
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int k = 32 * warp + 16 * m + g + 8 * r;
#pragma unroll
            for (int t = 0; t < 4; ++t)
                *reinterpret_cast<float2*>(mine + k * kHid + 8 * t + 2 * q) = make_float2(acc[m][t][2 * r], acc[m][t][2 * r + 1]);
            if (q == 0) mine[kOffB1 + k] = acc[m][4][2 * r];
        }
}

// grads += scale * the per-CTA sums, added in CTA order
__global__ void mlp_param_reduce_kernel(const float* scratch, int n_parts, float scale, float* gw1, float* gb1, float* gw2,
                                        float* gb2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kPgParams) return;
    float s = 0.f;
    for (int p = 0; p < n_parts; ++p) s += scratch[(size_t)p * kPgParams + i];
    s *= scale;
    if (i < kOffB1) { if (gw1) gw1[i] += s; }
    else if (i < kOffW2) { if (gb1) gb1[i - kOffB1] += s; }
    else if (i < kOffB2) { if (gw2) gw2[i - kOffW2] += s; }
    else if (gb2) gb2[i - kOffB2] += s;
}

}  // namespace mlp
}  // namespace tc

template <typename T>
static MlpArgs<T> mlp_simt_args(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                                const void* w2, const void* b2, const void* z0, void* out, int64_t n_paths,
                                int64_t channels, int64_t hidden, int64_t width, int method, int64_t n_steps,
                                const void* step_dt, const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                const int32_t* out_step, const int32_t* out_mode, const void* out_slope, double sign) {
    const int n_stages = (method == TCDE_RK4_38) ? 4 : (method == TCDE_MIDPOINT) ? 2 : 1;
    return MlpArgs<T>{(const T*)control, (const T*)w1, (const T*)b1, (const T*)w2, (const T*)b2, (const T*)z0, (T*)out,
                      (const T*)step_dt, stage_index, (const T*)stage_frac, out_step, out_mode, (const T*)out_slope,
                      n_paths, n_rows, (int)channels, (int)hidden, (int)width, control_kind, method, n_stages,
                      (int)n_steps, (int)n_out, (T)sign};
}

// the persistent grid of mlp_simt_param_grad_kernel (independent of the dtype: the scratch size has no dtype)
static int64_t mlp_simt_param_grid(int64_t n_paths, int64_t n_total, int ni) {
    return capped_grid(((n_paths + ni - 1) / ni) * n_total, kMlpPgCtasPerSm);
}

// the items per block of the parameter gradients at this shape (sized for 8-byte elements, so that both dtypes use the
// same grid and scratch), or 0 if no block fits in shared memory
static int mlp_simt_param_items(int64_t H, int64_t C, int64_t W) {
    MlpSimtLayout<double> lay;
    MlpSimtPg pg;
    return mlp_simt_pg_pick<double>((int)H, (int)C, (int)W, kMlpSimtThreads, lay, pg) ? pg.ni : 0;
}

template <typename T>
static int mlp_simt_param_grads(const MlpArgs<T>& a, int hm, const T* z_stages, const T* kappa, int64_t n_total,
                                void* grad_w1, void* grad_b1, void* grad_w2, void* grad_b2, void* scratch, double scale,
                                cudaStream_t s) {
    const int ni = mlp_simt_param_items(a.H, a.C, a.W);
    TCDE_CHECK_SUPPORTED(ni > 0, "MLP parameter gradients: hidden=%d channels=%d width=%d do not fit the CUDA-core "
                         "kernel's shared memory", a.H, a.C, a.W);
    // the same block width as the scratch was sized for; fp32 may then also stage the weights
    MlpSimtLayout<T> lay;
    MlpSimtPg pg;
    TCDE_CHECK_SUPPORTED(mlp_simt_pg_pick<T>(a.H, a.C, a.W, ni, lay, pg) && pg.ni == ni,
                         "MLP parameter gradients: the shape does not fit");
    const int64_t grid = mlp_simt_param_grid(a.n_paths, n_total, ni);
    const int64_t n_params = mlp_simt_n_params(a.H, a.C, a.W);
    const MlpSimtPgArgs<T> p{z_stages, kappa, (T*)scratch, n_params, (int)n_total};
    const int rc = mlp_hm(hm, [&](auto HM) {
        return launch(mlp_simt_param_grad_kernel<T, HM.value>, grid, ni, pg.total, s, a, lay, pg, p);
    });
    if (rc != TCDE_OK || !(grad_w1 || grad_b1 || grad_w2 || grad_b2)) return rc;
    const int64_t o_b1 = (int64_t)a.W * a.H, o_w2 = o_b1 + a.W, o_b2 = o_w2 + (int64_t)a.H * a.C * a.W;
    return launch(mlp_simt_param_reduce_kernel<T>, (n_params + 255) / 256, 256, 0, s, (const T*)scratch, (int)grid,
                      n_params, o_b1, o_w2, o_b2, (T)scale, (T*)grad_w1, (T*)grad_b1, (T*)grad_w2, (T*)grad_b2);
}

// the parameter-gradient scratch of tcde_vector_field_mlp_vjp starts after the stage's (index, frac)
constexpr int64_t kMlpFieldScratchHead = 16;

// One field evaluation (no cotangent) or one adjoint stage: at most three launches (the field kernel, then with a
// parameter gradient mlp_simt_param_grad_kernel over this one stage and mlp_simt_param_reduce_kernel)
template <typename T>
static int mlp_field_eval(int hm, const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                          const void* w2, const void* b2, const void* z, void* f_out, int64_t n_paths, int64_t channels,
                          int64_t hidden, int64_t width, int32_t index, double frac, const void* adj, void* vjp_out,
                          void* grad_w1, void* grad_b1, void* grad_w2, void* grad_b2, void* scratch, double f_scale,
                          double vjp_scale, double grad_scale, cudaStream_t s) {
    const bool grads = grad_w1 || grad_b1 || grad_w2 || grad_b2;
    int32_t* q_index = grads ? static_cast<int32_t*>(scratch) : nullptr;
    T* q_frac = grads ? reinterpret_cast<T*>(static_cast<char*>(scratch) + 8) : nullptr;
    const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, z, f_out, n_paths, channels,
                                          hidden, width, TCDE_EULER, 1, nullptr, q_index, q_frac, 1, nullptr, nullptr,
                                          nullptr, 1.0);
    const MlpFieldEval<T> e{(const T*)adj, (T*)vjp_out, q_index, q_frac, index, (T)frac, (T)f_scale, (T)vjp_scale};
    const auto field = [&](auto vjp) {
        constexpr bool VJP = decltype(vjp)::value;
        return mlp_hm(hm, [&](auto HM) {
            return mlp_launch_simt(mlp_field_kernel<T, HM.value, VJP>, a, kMlpSimtThreads,
                                   mlp_field_extra<T, HM.value, VJP>(a.H), s, e);
        });
    };
    const int rc = adj == nullptr ? field(std::false_type()) : field(std::true_type());
    if (rc != TCDE_OK || !grads) return rc;
    return mlp_simt_param_grads(a, hm, (const T*)z, (const T*)adj, 1, grad_w1, grad_b1, grad_w2, grad_b2,
                                static_cast<char*>(scratch) + kMlpFieldScratchHead, grad_scale, s);
}

static int64_t mlp_param_grid(int64_t n_paths, int64_t n_total) {
    return capped_grid(((n_paths + tc::wg::kPaths - 1) / tc::wg::kPaths) * n_total, 1);
}

// ---- the backward of cdeint(..., adjoint=False) under the host-driven dopri5 (tcde_dopri5_mlp_backward) ---------------
//
// The transposed Dormand-Prince recurrence of dopri5_backward_kernel (solve_dopri5.cu) for this field, one thread per path
// over one record chunk, last step first.  J depends on the state here, so every J^T is one mlp_vjp pass at the
// evaluation's recorded input and location (the forward's ReLU masks and tanh values, as in the Runge-Kutta backward).
// Items [step_item[n], step_item[n + 1]) of the chunk are the evaluations of step n: 6 (stages 2..7; stage 7's input is
// y_{n+1}), or 7 when k1 of step n is a fresh start slope f(t_n, y_n) (step 0 of the solve, and the step after a jump of
// jump_t), whose item then comes first.  (A, K): the cotangents of y_{n+1} and of the evaluation k7 (= k1 of step n + 1
// under FSAL: zero when that one was fresh).  Per step:
//   kappa7 = K + inj;  Zbar7 = A + J7^T kappa7 + inj, to y_n (weight 1) and k_j (beta[5][j - 1] dt);  stages i = 6 .. 2:
//   kappa_i = the accumulated cotangent of k_i, Zbar_i = J_i^T kappa_i to y_n and k_j, j < i;  (A, K) = (ybar_n, kbar_1);
//   a fresh k1 gets its own J^T at y_n into A, and K = 0.
// The output cotangents enter through the transposed dense output (adaptive.dopri5_backward_tables); kappa of every
// evaluation goes to its item, for tcde_mlp_field_param_grads.  The cotangents of k2..k6 sit in the thread's shared-memory
// columns, so that the stages run as one loop (one mlp_vjp site); A, K, J^T kappa and the input as the reversible
// backward keeps its vectors (registers at HM = 8, 64-thread CTAs with shared columns at HM = 32).
template <typename T> struct MlpDp5Bwd {
    const T* rec_z;               // [n_items][n_paths][H]: the evaluations' inputs
    T* kappa;                     // [n_items][n_paths][H], or null
    const T* grad_out;            // [n_paths][n_out][H]
    T* carry;                     // [2][n_paths][H]: (A, K) after the chunk's last step in, before its first step out
    const T* coef;                // [n_steps][36]: beta[s][j] dt_n, rows s = 0..5 zero padded, as the forward combined
    const int32_t* step_item;     // [n_steps + 1]
    const int32_t* inj_range;     // [n_steps + 1]: the injections of step n are [inj_range[n], inj_range[n + 1])
    const int32_t* inj_out;       // [n_inj]: output index
    const T* inj_w;               // [n_inj][8]: weights on (y_n, y_{n+1}, k1, k3, k4, k5, k6, k7)
    int n_steps;
};
enum { kDpY0 = 0, kDpY1 = 1, kDpK1 = 2, kDpK7 = 7 };               // inj_w columns; k_j (j = 3..6) is column j

template <int HM> __host__ __device__ constexpr bool mlp_dp5_bwd_shared() { return HM == 32; }
// per-thread values after the slopes: the cotangents of k2..k6 [5H], then at HM = 32 A, K, J^T kappa [H] and z [Hp]
template <int HM> static int mlp_dp5_bwd_extra(int H) {
    return 5 * H + (mlp_dp5_bwd_shared<HM>() ? 3 * H + (H + 3) / 4 * 4 : 0);
}

// a.stage_index / a.stage_frac: the items' locations; a.sign: the sign of the solve's time direction
template <typename T, int HM>
__global__ void __launch_bounds__(kMlpSimtThreads, 1) dopri5_mlp_backward_kernel(const MlpArgs<T> a,
                                                                              const MlpSimtLayout<T> lay,
                                                                              const MlpDp5Bwd<T> b) {
    constexpr bool kShared = mlp_dp5_bwd_shared<HM>();
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* smem = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x;
    constexpr int nt = mlp_rev_bwd_threads<HM>();
    const int H = a.H, C = a.C;
    if (lay.staged) {
        const int W = a.W, HC = a.H * a.C, Hp = lay.Hp, Nq = lay.Nq;
        TCDE_MLP_STAGE_WEIGHTS()
        __syncthreads();
    }
    T* dxs = smem + lay.cols + tid;
    T* kvs = dxs + (size_t)C * nt;                                 // kvs[h * nt]: kappa of the evaluation transposed
    T* park = kvs + (size_t)H * nt;                                // park[((j - 2) * H + h) * nt]: cotangent of k_j
    const int64_t path = (int64_t)blockIdx.x * nt + tid;
    const bool live = path < a.n_paths;
    const int64_t lp = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const T* crow = a.control + lp * a.n_rows * (cubic ? 4 * C : C) + (cubic ? C : 0);
    MlpRevVec<T, HM, kShared, nt> A, K, kv, zm;                    // kv: J^T kappa; zm: the evaluation's input
    {
        T* col = park + (size_t)5 * H * nt;
        const size_t step = (size_t)H * nt;
        A.bind(col);
        K.bind(col + step);
        kv.bind(col + 2 * step);
        zm.bind(col + 3 * step);
    }
    struct Col {                                                   // the cotangent of k_j in the thread's column
        T* p;
        __device__ __forceinline__ T& operator[](int k) const { return p[(size_t)k * nt]; }
    };
    auto kbar = [&](int j) { return Col{park + (size_t)(j - 2) * H * nt}; };
    const int64_t plane = a.n_paths * H;
#pragma unroll
    for (int h = 0; h < HM; ++h) {
        if (!kShared || h < H) {
            A[h] = h < H ? b.carry[lp * H + h] : T(0);
            K[h] = h < H ? b.carry[plane + lp * H + h] : T(0);
            kv[h] = T(0);
        }
        if (!kShared || h < lay.Hp) zm[h] = T(0);
    }
    // v += the step's output cotangents with weight column col
    auto inject = [&](int e0, int e1, int col, auto&& v) {
        for (int e = e0; e < e1; ++e) {
            const T w = b.inj_w[8 * e + col];
            const T* src = b.grad_out + (lp * a.n_out + b.inj_out[e]) * H;
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) v[h] = fma(w, src[h], v[h]);
        }
    };
    // kv = J^T kappa (kappa in kvs) at item e's input and location; kappa also goes to item e of b.kappa
    auto transposed = [&](int e) {
        const T* zsrc = b.rec_z + (int64_t)e * plane + lp * H;
        T* kdst = b.kappa ? b.kappa + (int64_t)e * plane + path * H : nullptr;
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            if (h < H) {
                zm[h] = zsrc[h];
                kv[h] = T(0);
                if (kdst && live) kdst[h] = kvs[(size_t)h * nt];
            }
        }
        {
            TCDE_MLP_SLOPE(a.stage_index[e], a.stage_frac[e])
        }
        mlp_vjp<T, HM>(
            a, lay, smem, zm.arg(), dxs, kvs, nt, [](int, const T*) {},
            [&](int, int w, T pre, T sv) {
                if (!(pre > T(0))) return;
                if (lay.staged) {
                    const T* wr = smem + lay.w1 + (size_t)w * lay.Hp;
#pragma unroll
                    for (int k4 = 0; k4 < HM / 4; ++k4) {
                        if (4 * k4 < lay.Hp) {
                            const P4 w4 = *reinterpret_cast<const P4*>(wr + 4 * k4);
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if (!kShared || 4 * k4 + i < H) kv[4 * k4 + i] = fma(w4.v[i], sv, kv[4 * k4 + i]);
                        }
                    }
                } else {
                    const T* wr = a.w1 + (size_t)w * H;
#pragma unroll
                    for (int k = 0; k < HM; ++k)
                        if (k < H) kv[k] = fma(__ldg(wr + k), sv, kv[k]);
                }
            });
    };

    for (int n = b.n_steps - 1; n >= 0; --n) {
        const T* cs = b.coef + (int64_t)n * 36;
        const int e0 = b.inj_range[n], e1 = b.inj_range[n + 1];
        const int first = b.step_item[n];
        const bool fresh = b.step_item[n + 1] - first == 7;
        const int s2 = first + (fresh ? 1 : 0);                    // the item of stage 2
        // the evaluations of step n, last first: i = 7 .. 2 its stages, i = 1 its fresh start slope
        for (int i = 7; i >= (fresh ? 1 : 2); --i) {
            if (i == 7) inject(e0, e1, kDpK7, K);
#pragma unroll
            for (int h = 0; h < HM; ++h)
                if (h < H) kvs[(size_t)h * nt] = (i == 7 || i == 1) ? K[h] : kbar(i)[h];
            transposed(i == 1 ? first : s2 + i - 2);
            if (i == 7) {
#pragma unroll
                for (int h = 0; h < HM; ++h)
                    if (h < H) A[h] = E::add(A[h], kv[h]);
                inject(e0, e1, kDpY1, A);
                // Zbar7 (in A) -> y_n (A stays), k1 (K), k2 .. k6
#pragma unroll
                for (int h = 0; h < HM; ++h) {
                    if (h < H) {
                        const T z = A[h];
                        K[h] = E::mul(cs[30], z);
                        for (int j = 2; j <= 6; ++j) kbar(j)[h] = E::mul(cs[30 + j - 1], z);
                    }
                }
                inject(e0, e1, kDpY0, A);
                inject(e0, e1, kDpK1, K);
                for (int j = 3; j <= 6; ++j) inject(e0, e1, j, kbar(j));
            } else if (i == 1) {
#pragma unroll
                for (int h = 0; h < HM; ++h) {
                    if (h < H) {
                        A[h] = E::add(A[h], kv[h]);
                        K[h] = T(0);
                    }
                }
            } else {
                const T* c = cs + (i - 2) * 6;
#pragma unroll
                for (int h = 0; h < HM; ++h) {
                    if (h < H) {
                        A[h] = E::add(A[h], kv[h]);
                        K[h] = fma(c[0], kv[h], K[h]);
                        for (int j = 2; j < i; ++j) kbar(j)[h] = fma(c[j - 1], kv[h], kbar(j)[h]);
                    }
                }
            }
        }
    }
    if (live) {
#pragma unroll
        for (int h = 0; h < HM; ++h) {
            if (h < H) {
                b.carry[path * H + h] = A[h];
                b.carry[plane + path * H + h] = K[h];
            }
        }
    }
}

// ---- which kernels serve an entry point: the one route policy of the MLP field ----------------------------------------
//
// What is asked, then what serves it (every ask first needs 1 <= width, channels < 2^20 and hidden * channels < 2^20).
// "simt shapes": hidden <= 8 (the HM = 8 instantiations) or hidden * channels <= 32 (one chunk of outputs); "tc": fp32
// at hidden 32, channels 8, width 128 with 16-byte aligned buffers; "CUDA-core route": fp32 or fp64 at the simt shapes
// under solve variant 0 (hidden <= 8) or variant 1.
//   solve                fp32: tc under variant 0 (if not tc, as fp64) and only tc under 4 / 5; 2 / 3 / 6 (3xTF32) not
//                        built.  fp64 under any variant: the CUDA cores at the simt shapes, or at hidden <= 32 under 1.
//   stages, backward,    tc under variant 0, 4 or 5 past the simt shapes, the CUDA-core route at them.
//   param_grads
//   param_scratch        as param_grads, whatever the dtype and the variant.
//   field                the CUDA-core route; by default also only fp32 at hidden * channels <= 32 and width <= 128.
//   reversible           the CUDA-core route; by default also only hidden * channels <= 32.
//   dopri5_backward      the CUDA-core route.
// For field, reversible and dopri5_backward the width must also let the kernels' layouts (mlp_simt_fit, with 8-byte
// elements: one answer for both dtypes) and, but for the dopri5 backward, the parameter-gradient staging fit shared memory.
// Elsewhere TCDE_ERR_UNSUPPORTED, and the caller keeps its own route (the stage loop, autograd, torch operators).
//
// Why, from measurements on an H100 (DESIGN 4.2, 8 and "torchsde backend"):
//   * past the simt shapes the CUDA-core forward recomputes the first product per chunk of 32 outputs and runs at low
//     occupancy: 1.3-4.5x (fp32) and up to 13.6x (fp64) slower than cdeint's stage loop;
//   * at hidden 32, channels 1 a training step on the CUDA-core backprop was slower per sequence than the torch-operator
//     loop, so variant 0 runs it only at hidden <= 8 (variant 1 forces the HM = 32 kernels);
//   * an adjoint=True training step on the field kernels beat autograd per stage only at fp32, hidden * channels <= 32 and
//     width <= 128; fp64, channels 14 and width 366 at hidden 8 measured 0.13-0.83x of autograd's speed;
//   * reversible Heun beat the torch-operator forward and per-step autograd at (8, 3, 128) fp32 and fp64 and at
//     (5, 3, 37), but was 7.7x slower at (8, 14, 128): four chunks, the backward recomputes the first product per chunk
//     and its parameter gradients stage 112 outputs per item.
enum MlpAsk { kMlpSolve, kMlpStages, kMlpBackward, kMlpParamGrads, kMlpParamScratch, kMlpField, kMlpReversible,
              kMlpDopri5Backward };

struct MlpRoute {
    bool tc;                      // the tensor-core kernels
    int hm;                       // else the CUDA-core instantiation: HM = 8 up to 8 hidden units, else 32
};

// The checks of the entry points' enum arguments.  The solve and the reversible Heun and dopri5 entries reject an unknown
// dtype as an argument; to the others it is a dtype the route policy does not serve.
static int mlp_check_args(MlpAsk ask, int control_kind, int dtype, int method = TCDE_EULER) {
    if (ask == kMlpSolve || ask == kMlpReversible || ask == kMlpDopri5Backward) TCDE_TRY(check_dtype(dtype));
    TCDE_TRY(check_control_kind(control_kind));
    return check_method(method);
}

static int mlp_check_shape(int64_t hidden, int64_t channels, int64_t width) {
    TCDE_CHECK_ARG(channels >= 1 && hidden >= 1 && width >= 1, "bad sizes");
    TCDE_CHECK_SUPPORTED(width < (1 << 20) && channels < (1 << 20) && hidden * channels < (1 << 20), "MLP too wide");
    return TCDE_OK;
}

static int mlp_route(MlpAsk ask, int64_t hidden, int64_t channels, int64_t width, int dtype, bool aligned,
                     const char* what, MlpRoute* r) {
    TCDE_TRY(mlp_check_shape(hidden, channels, width));
    const int variant = current_solve_variant();
    const bool simt = hidden <= 8 || hidden * channels <= kMlpChunk;
    const bool tc_shape = hidden == tc::kHid && channels == tc::kCh && width == tc::mlp::kWidth;
    *r = MlpRoute{false, hidden <= 8 ? 8 : 32};
    if (ask == kMlpParamScratch) {
        r->tc = !simt;
        TCDE_CHECK_SUPPORTED(simt ? mlp_simt_param_items(hidden, channels, width) > 0 : tc_shape,
                             "%s: hidden=%lld channels=%lld width=%lld are not served", what, (long long)hidden,
                             (long long)channels, (long long)width);
        return TCDE_OK;
    }
    if (ask == kMlpSolve) {
        if (dtype == TCDE_F32) {
            TCDE_CHECK_SUPPORTED(variant != kVariantTf32,
                                 "%s: solve variant %d (3xTF32) is not built for the MLP field", what, variant);
            TCDE_CHECK_SUPPORTED(variant <= kVariantSimt || (tc_shape && aligned),
                                 "%s: the tensor-core kernel is built for "
                                 "hidden=32, channels=8, width=128 with 16-byte aligned control, z0 and out (got %lld, "
                                 "%lld, %lld)", what, (long long)hidden, (long long)channels, (long long)width);
            r->tc = variant == kVariantFp16 || (variant == kVariantAuto && tc_shape && aligned);
            if (r->tc) return TCDE_OK;
        }
        TCDE_CHECK_SUPPORTED(simt || variant == kVariantSimt,
                             "%s: at hidden=%lld channels=%lld the CUDA-core kernel is slower than "
                             "the stage loop; automatic selection does not run it (variant 1 forces it)", what,
                             (long long)hidden, (long long)channels);
        TCDE_CHECK_SUPPORTED(hidden <= 32, "%s: hidden=%lld > 32 is not built for the CUDA-core kernel", what,
                             (long long)hidden);
        return TCDE_OK;
    }
    if (!simt) {
        r->tc = true;
        TCDE_CHECK_SUPPORTED((ask == kMlpStages || ask == kMlpBackward || ask == kMlpParamGrads) && dtype == TCDE_F32 &&
                                 tc_shape && (variant == kVariantAuto || variant == kVariantFp16),
                             "%s is built for fp32, hidden=32, channels=8, width=128 on the tensor-core kernel where it "
                             "has one, else for the CUDA-core shapes (hidden <= 8, or hidden * channels <= 32 under solve "
                             "variant 1; got dtype=%d, %lld, %lld, %lld, solve variant %d)", what, dtype,
                             (long long)hidden, (long long)channels, (long long)width, variant);
        TCDE_CHECK_SUPPORTED(aligned, "%s: the tensor-core kernel needs 16-byte aligned buffers", what);
        return TCDE_OK;
    }
    TCDE_CHECK_SUPPORTED(hidden <= 8 || variant == kVariantSimt,
                         "%s: at hidden=%lld the CUDA-core route is slower than the stage "
                         "loop; automatic selection does not run it (variant 1 forces it)", what, (long long)hidden);
    TCDE_CHECK_SUPPORTED((dtype == TCDE_F32 || dtype == TCDE_F64) && variant <= kVariantSimt,
                         "%s on the CUDA cores is built for "
                         "fp32 / fp64 under solve variant 0 or 1 (got dtype=%d, solve variant %d)", what, dtype,
                         variant);
    TCDE_CHECK_SUPPORTED(ask != kMlpField || variant == kVariantSimt ||
                             (dtype == TCDE_F32 && hidden * channels <= kMlpChunk && width <= 128),
                         "%s: at dtype=%d hidden=%lld channels=%lld width=%lld it is slower than autograd per stage; "
                         "automatic selection does not run it (variant 1 forces it)", what, dtype, (long long)hidden,
                         (long long)channels, (long long)width);
    TCDE_CHECK_SUPPORTED(ask != kMlpReversible || variant == kVariantSimt || hidden * channels <= kMlpChunk,
                         "%s: at hidden=%lld channels=%lld the backward is slower than per-step autograd; automatic "
                         "selection does not run it (variant 1 forces it)", what, (long long)hidden, (long long)channels);
    const int H = (int)hidden, C = (int)channels, W = (int)width;
    const bool fits = mlp_hm(r->hm, [&](auto HM) {
        const bool staging = mlp_simt_param_items(H, C, W) > 0;
        switch (ask) {
        case kMlpField:
            return staging && mlp_simt_fit<double>(H, C, W, kMlpSimtThreads, mlp_field_extra<double, HM.value, true>(H));
        case kMlpReversible:
            return staging && mlp_simt_fit<double>(H, C, W, kMlpSimtThreads, mlp_rev_fwd_extra<double, HM.value>(H)) &&
                   mlp_simt_fit<double>(H, C, W, mlp_rev_bwd_threads<HM.value>(), mlp_rev_bwd_extra<HM.value>(H));
        case kMlpDopri5Backward:
            return mlp_simt_fit<double>(H, C, W, mlp_rev_bwd_threads<HM.value>(), mlp_dp5_bwd_extra<HM.value>(H))
                .has_value();
        default:
            return true;          // the solve's layouts are fitted at launch
        }
    });
    TCDE_CHECK_SUPPORTED(fits, "%s: hidden=%lld channels=%lld width=%lld do not fit the CUDA-core kernels' shared memory",
                         what, (long long)hidden, (long long)channels, (long long)width);
    return TCDE_OK;
}

// The fixed-step solve, with a stage dump when stage_dump is set
static int mlp_fixed_solve(const MlpRoute& r, const void* control, int control_kind, int64_t n_rows, const void* w1,
                           const void* b1, const void* w2, const void* b2, const void* z0, void* out, void* stage_dump,
                           int64_t n_paths, int64_t channels, int64_t hidden, int64_t width, int method,
                           int64_t n_steps, const void* step_dt, const int32_t* stage_index, const void* stage_frac,
                           int64_t n_out, const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                           double sign, int dtype, cudaStream_t s) {
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, z0, out, n_paths, channels,
                                              hidden, width, method, n_steps, step_dt, stage_index, stage_frac, n_out,
                                              out_step, out_mode, out_slope, sign);
        if (r.tc) {
            const UmmaArgs u{(const float*)a.control, (const float*)a.w1, (const float*)a.b1, (const float*)a.z0,
                             (float*)a.out, (const float*)a.step_dt, a.stage_index, (const float*)a.stage_frac,
                             a.out_step, a.out_mode, (const float*)a.out_slope, a.n_paths, a.n_rows, a.control_kind,
                             a.method, a.n_stages, a.n_steps, a.n_out, (float)a.sign, (float*)stage_dump, 0};
            return launch(stage_dump ? tc::mlp::cdeint_mlp_wgmma_kernel<true> : tc::mlp::cdeint_mlp_wgmma_kernel<false>,
                              (n_paths + tc::mlp::kPaths - 1) / tc::mlp::kPaths, tc::mlp::kThreads, tc::mlp::kSmem, s,
                              u, (const float*)w2, (const float*)b2);
        }
        return mlp_hm(r.hm, [&](auto HM) {
            return mlp_launch_simt(stage_dump ? cdeint_mlp_simt_kernel<T, HM.value, true>
                                              : cdeint_mlp_simt_kernel<T, HM.value, false>,
                                   a, kMlpSimtThreads, 0, s, (T*)stage_dump);
        });
    });
}

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
    TCDE_TRY(mlp_check_args(kMlpSolve, control_kind, dtype, method));
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    TCDE_TRY(mlp_check_shape(hidden, channels, width));
    if (n_paths == 0) return TCDE_OK;
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpSolve, hidden, channels, width, dtype, aligned16(control, z0, out), "the MLP solve", &r));
    return mlp_fixed_solve(r, control, control_kind, n_rows, w1, b1, w2, b2, z0, out, nullptr, n_paths, channels, hidden,
                           width, method, n_steps, step_dt, stage_index, stage_frac, n_out, out_step, out_mode,
                           out_slope, sign, dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int tcde_cdeint_fixed_mlp_stages(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                            const void* b1, const void* w2, const void* b2, const void* z0, void* out,
                                            void* stage_dump, int64_t n_paths, int64_t channels, int64_t hidden,
                                            int64_t width, int method, int64_t n_steps, const void* step_dt,
                                            const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                            const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                                            double sign, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z0 && out && stage_dump, "null data pointer");
    TCDE_CHECK_ARG(step_dt && stage_index && stage_frac && out_step && out_mode && out_slope, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_steps >= 1 && n_out >= 1, "bad sizes");
    TCDE_TRY(mlp_check_args(kMlpStages, control_kind, dtype, method));
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpStages, hidden, channels, width, dtype, aligned16(control, z0, out, stage_dump),
                       "the MLP stage-dump solve", &r));
    TCDE_CHECK_SUPPORTED(r.tc || n_paths * hidden * n_steps * 4 < (1ll << 62), "stage dump too large");
    if (n_paths == 0) return TCDE_OK;
    return mlp_fixed_solve(r, control, control_kind, n_rows, w1, b1, w2, b2, z0, out, stage_dump, n_paths, channels,
                           hidden, width, method, n_steps, step_dt, stage_index, stage_frac, n_out, out_step, out_mode,
                           out_slope, sign, dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int tcde_cdeint_fixed_mlp_backward(
    const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1, const void* w2, const void* b2,
    const void* stage_dump, const void* grad_out, void* grad_z0, void* kappa_dump, int64_t n_paths, int64_t channels,
    int64_t hidden, int64_t width, int method, int64_t n_steps, const void* step_dt_rev, const int32_t* stage_index_rev,
    const void* stage_frac_rev, int64_t n_out, const int32_t* inj_range, const int32_t* inj_out, const void* inj_weight,
    double sign, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && stage_dump && grad_out && grad_z0, "null data pointer");
    TCDE_CHECK_ARG(step_dt_rev && stage_index_rev && stage_frac_rev && inj_range && inj_out && inj_weight,
                   "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_steps >= 1 && n_out >= 1, "bad sizes");
    TCDE_TRY(mlp_check_args(kMlpBackward, control_kind, dtype, method));
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpBackward, hidden, channels, width, dtype,
                       aligned16(control, stage_dump, grad_out, grad_z0, kappa_dump),
                       "the MLP Runge-Kutta backward", &r));
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, nullptr, grad_z0, n_paths,
                                              channels, hidden, width, method, n_steps, step_dt_rev, stage_index_rev,
                                              stage_frac_rev, n_out, nullptr, nullptr, nullptr, sign);
        if (r.tc) {
            const UmmaArgs u{(const float*)control, (const float*)w1, (const float*)b1, nullptr, (float*)grad_z0,
                             (const float*)step_dt_rev, stage_index_rev, (const float*)stage_frac_rev, nullptr, nullptr,
                             nullptr, n_paths, n_rows, control_kind, method, a.n_stages, (int)n_steps, (int)n_out,
                             (float)sign, (float*)kappa_dump, 0, (const float*)grad_out, inj_range, inj_out,
                             (const float*)inj_weight};
            return launch(tc::mlp::cdeint_mlp_backward_kernel, (n_paths + tc::wg::kPaths - 1) / tc::wg::kPaths,
                              tc::mlp::kBwdThreads, tc::mlp::kBwdSmem, s, u, (const float*)w2, (const float*)b2,
                              (const float*)stage_dump);
        }
        const MlpSimtBwd<T> b{(const T*)stage_dump, (T*)kappa_dump, (const T*)grad_out, inj_range, inj_out,
                              (const T*)inj_weight};
        return mlp_hm(r.hm, [&](auto HM) {
            return mlp_launch_simt(cdeint_mlp_simt_backward_kernel<T, HM.value>, a, kMlpSimtThreads, 0, s, b);
        });
    });
}

extern "C" int64_t tcde_mlp_field_param_grads_scratch_bytes(int64_t n_paths, int64_t n_stages_total, int64_t channels,
                                                           int64_t hidden, int64_t width) {
    MlpRoute r;
    if (n_paths < 0 || n_stages_total < 1 ||
        mlp_route(kMlpParamScratch, hidden, channels, width, TCDE_F32, true, "the MLP parameter-gradient scratch",
                  &r) != TCDE_OK)
        return -1;
    if (r.tc) return mlp_param_grid(n_paths, n_stages_total) * tc::mlp::kPgParams * (int64_t)sizeof(float);
    // the CUDA-core kernel, sized for 8-byte elements
    return mlp_simt_param_grid(n_paths, n_stages_total, mlp_simt_param_items(hidden, channels, width)) *
           mlp_simt_n_params(hidden, channels, width) * (int64_t)sizeof(double);
}

extern "C" int tcde_mlp_field_param_grads(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                          const void* b1, const void* w2, const void* b2, const void* z_stages,
                                          const void* kappa_stages, const int32_t* stage_index, const void* stage_frac,
                                          int64_t n_stages_total, void* grad_w1, void* grad_b1, void* grad_w2,
                                          void* grad_b2, void* scratch, int64_t n_paths, int64_t channels, int64_t hidden,
                                          int64_t width, double sign, double scale, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z_stages && kappa_stages && stage_index && stage_frac && scratch,
                   "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_stages_total >= 1 && n_stages_total < (1ll << 31), "bad sizes");
    TCDE_TRY(mlp_check_args(kMlpParamGrads, control_kind, dtype));
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpParamGrads, hidden, channels, width, dtype,
                       aligned16(control, z_stages, kappa_stages, scratch),
                       "the MLP parameter gradients", &r));
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (r.tc) {
        const int64_t grid = mlp_param_grid(n_paths, n_stages_total);
        tc::mlp::PgArgs a{(const float*)control, (const float*)w1, (const float*)b1, (const float*)w2, (const float*)b2,
                          (const float*)z_stages, (const float*)kappa_stages, stage_index, (const float*)stage_frac,
                          (float*)scratch, n_paths, n_rows, control_kind, (int)n_stages_total, (float)sign};
        TCDE_CHECK_CUDA(cudaFuncSetAttribute(tc::mlp::mlp_param_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             tc::mlp::kPgSmem));
        tc::mlp::mlp_param_grad_kernel<<<dim3((unsigned)grid, tc::mlp::kPgY), tc::mlp::kBwdThreads, tc::mlp::kPgSmem,
                                         s>>>(a);
        TCDE_CHECK_CUDA(cudaGetLastError());
        if (!(grad_w1 || grad_b1 || grad_w2 || grad_b2)) return TCDE_OK;
        return launch(tc::mlp::mlp_param_reduce_kernel, (tc::mlp::kPgParams + 255) / 256, 256, 0, s,
                          (const float*)scratch, (int)grid, (float)scale, (float*)grad_w1, (float*)grad_b1,
                          (float*)grad_w2, (float*)grad_b2);
    }
    // the forward's stage tables; the solve's method and steps do not matter here
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        return mlp_simt_param_grads(mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, nullptr, nullptr,
                                                     n_paths, channels, hidden, width, TCDE_EULER, 1, nullptr,
                                                     stage_index, stage_frac, 1, nullptr, nullptr, nullptr, sign),
                                    r.hm, (const T*)z_stages, (const T*)kappa_stages, n_stages_total, grad_w1, grad_b1,
                                    grad_w2, grad_b2, scratch, scale, s);
    });
}

extern "C" int tcde_vector_field_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                                     const void* w2, const void* b2, const void* z, void* out, int64_t n_paths,
                                     int64_t channels, int64_t hidden, int64_t width, int32_t index, double frac,
                                     int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z && out, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && width >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(index >= 0 && index < n_rows, "index=%d outside [0, %lld)", index, (long long)n_rows);
    TCDE_TRY(mlp_check_args(kMlpField, control_kind, dtype));
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpField, hidden, channels, width, dtype, true, "the MLP field evaluation", &r));
    if (n_paths == 0) return TCDE_OK;
    return by_dtype(dtype, [&](auto t) {
        return mlp_field_eval<decltype(t)>(r.hm, control, control_kind, n_rows, w1, b1, w2, b2, z, out, n_paths,
                                           channels, hidden, width, index, frac, nullptr, nullptr, nullptr, nullptr,
                                           nullptr, nullptr, nullptr, 1.0, 1.0, 1.0, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int64_t tcde_vector_field_mlp_vjp_scratch_bytes(int64_t n_paths, int64_t channels, int64_t hidden,
                                                           int64_t width) {
    MlpRoute r;
    if (n_paths < 0 ||
        mlp_route(kMlpField, hidden, channels, width, TCDE_F32, true, "the MLP adjoint stage", &r) != TCDE_OK)
        return -1;
    return kMlpFieldScratchHead + mlp_simt_param_grid(n_paths, 1, mlp_simt_param_items(hidden, channels, width)) *
                                      mlp_simt_n_params(hidden, channels, width) * (int64_t)sizeof(double);
}

extern "C" int tcde_vector_field_mlp_vjp(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                         const void* b1, const void* w2, const void* b2, const void* z, const void* a,
                                         void* f_out, void* vjp_z_out, void* grad_w1, void* grad_b1, void* grad_w2,
                                         void* grad_b2, void* scratch, int64_t n_paths, int64_t channels, int64_t hidden,
                                         int64_t width, int32_t index, double frac, double f_scale, double vjp_scale,
                                         double grad_scale, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z && a && f_out && vjp_z_out && scratch, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && width >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(index >= 0 && index < n_rows, "index=%d outside [0, %lld)", index, (long long)n_rows);
    TCDE_TRY(mlp_check_args(kMlpField, control_kind, dtype));
    TCDE_CHECK_ARG(aligned16(scratch), "scratch must be 16-byte aligned");
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpField, hidden, channels, width, dtype, true, "the MLP adjoint stage", &r));
    if (n_paths == 0) return TCDE_OK;
    return by_dtype(dtype, [&](auto t) {
        return mlp_field_eval<decltype(t)>(r.hm, control, control_kind, n_rows, w1, b1, w2, b2, z, f_out, n_paths,
                                           channels, hidden, width, index, frac, a, vjp_z_out, grad_w1, grad_b1, grad_w2,
                                           grad_b2, scratch, f_scale, vjp_scale, grad_scale,
                                           static_cast<cudaStream_t>(stream));
    });
}

extern "C" int tcde_cdeint_reversible_heun_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                               const void* b1, const void* w2, const void* b2, const void* z0, void* out,
                                               void* checkpoints, int64_t checkpoint_stride, int64_t n_paths,
                                               int64_t channels, int64_t hidden, int64_t width, int64_t n_steps,
                                               const void* step_dt, const int32_t* stage_index, const void* stage_frac,
                                               int64_t n_out, const int32_t* out_step, const void* out_weights, int dtype,
                                               void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && z0 && out, "null data pointer");
    TCDE_CHECK_ARG(step_dt && stage_index && stage_frac && out_step && out_weights, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && width >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(n_steps >= 1 && n_out >= 1, "n_steps=%lld n_out=%lld", (long long)n_steps, (long long)n_out);
    TCDE_CHECK_ARG(checkpoint_stride >= 1 && checkpoint_stride < (1ll << 30), "checkpoint_stride=%lld",
                   (long long)checkpoint_stride);
    TCDE_TRY(mlp_check_args(kMlpReversible, control_kind, dtype));
    TCDE_CHECK_SUPPORTED(n_steps + 1 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpReversible, hidden, channels, width, dtype, true, "the MLP reversible Heun solve",
                       &r));
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, z0, out, n_paths, channels,
                                              hidden, width, TCDE_REVERSIBLE_HEUN, n_steps, step_dt, stage_index,
                                              stage_frac, n_out, out_step, nullptr, out_weights, 1.0);
        return mlp_hm(r.hm, [&](auto HM) {
            return mlp_launch_simt(cdeint_mlp_rev_kernel<T, HM.value>, a, kMlpSimtThreads,
                                   mlp_rev_fwd_extra<T, HM.value>(a.H), s, (T*)checkpoints, (int)checkpoint_stride);
        });
    });
}

extern "C" int tcde_reversible_heun_mlp_backward_segment(
    const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1, const void* w2, const void* b2,
    const void* ckpt_lo, const void* ckpt_hi, void* carry, const void* g, int64_t n_out, const int32_t* out_step,
    const void* out_weights, const int32_t* inj_range, int64_t n_steps, const void* step_dt, const int32_t* stage_index,
    const void* stage_frac, int64_t lo, int64_t hi, int64_t n_paths, int64_t channels, int64_t hidden, int64_t width,
    void* dump_z, void* dump_a, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && ckpt_lo && ckpt_hi && carry && g && dump_z && dump_a,
                   "null data pointer");
    TCDE_CHECK_ARG(out_step && out_weights && inj_range && step_dt && stage_index && stage_frac, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && width >= 1 && n_rows >= 1 && n_out >= 1, "bad sizes");
    TCDE_CHECK_ARG(lo >= 0 && hi > lo && hi <= n_steps && n_steps + 1 < (1ll << 31), "lo=%lld hi=%lld n_steps=%lld",
                   (long long)lo, (long long)hi, (long long)n_steps);
    TCDE_TRY(mlp_check_args(kMlpReversible, control_kind, dtype));
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpReversible, hidden, channels, width, dtype, true, "the MLP reversible backward", &r));
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, nullptr, nullptr, n_paths,
                                              channels, hidden, width, TCDE_REVERSIBLE_HEUN, n_steps, step_dt,
                                              stage_index, stage_frac, n_out, out_step, nullptr, out_weights, 1.0);
        const MlpRevBwd<T> b{(const T*)ckpt_lo, (const T*)ckpt_hi, (T*)carry, (const T*)g, inj_range, (T*)dump_z,
                             (T*)dump_a, (int)lo, (int)hi};
        return mlp_hm(r.hm, [&](auto HM) {
            return mlp_launch_simt(mlp_rev_backward_kernel<T, HM.value>, a, mlp_rev_bwd_threads<HM.value>(),
                                   mlp_rev_bwd_extra<HM.value>(a.H), s, b);
        });
    });
}

extern "C" int tcde_dopri5_mlp_backward(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                        const void* b1, const void* w2, const void* b2, const void* rec_z,
                                        const void* grad_out, void* carry, void* kappa, const void* coef,
                                        const int32_t* step_item, const int32_t* item_index, const void* item_frac,
                                        const int32_t* inj_range, const int32_t* inj_out, const void* inj_w, int64_t n_out,
                                        int64_t n_steps, int64_t n_paths, int64_t channels, int64_t hidden, int64_t width,
                                        double sign, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && w1 && b1 && w2 && b2 && rec_z && grad_out && carry, "null data pointer");
    TCDE_CHECK_ARG(coef && step_item && item_index && item_frac && inj_range && inj_out && inj_w, "null table pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_out >= 2 && n_out < (1ll << 31) && n_steps >= 0 &&
                       n_steps < (1ll << 24) && channels >= 1 && hidden >= 1 && width >= 1, "bad sizes");
    TCDE_TRY(mlp_check_args(kMlpDopri5Backward, control_kind, dtype));
    TCDE_CHECK_ARG(sign == 1.0 || sign == -1.0, "sign=%g", sign);
    MlpRoute r;
    TCDE_TRY(mlp_route(kMlpDopri5Backward, hidden, channels, width, dtype, true, "the MLP dopri5 backward", &r));
    TCDE_CHECK_SUPPORTED(n_paths * hidden * 7 * n_steps < (1ll << 62), "record too large");
    if (n_paths == 0 || n_steps == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return by_dtype(dtype, [&](auto t) {
        using T = decltype(t);
        const MlpArgs<T> a = mlp_simt_args<T>(control, control_kind, n_rows, w1, b1, w2, b2, nullptr, nullptr, n_paths,
                                              channels, hidden, width, TCDE_EULER, n_steps, nullptr, item_index,
                                              item_frac, n_out, nullptr, nullptr, nullptr, sign);
        const MlpDp5Bwd<T> b{(const T*)rec_z, (T*)kappa, (const T*)grad_out, (T*)carry, (const T*)coef, step_item,
                             inj_range, inj_out, (const T*)inj_w, (int)n_steps};
        return mlp_hm(r.hm, [&](auto HM) {
            return mlp_launch_simt(dopri5_mlp_backward_kernel<T, HM.value>, a, mlp_rev_bwd_threads<HM.value>(),
                                   mlp_dp5_bwd_extra<HM.value>(a.H), s, b);
        });
    });
}
