// Hot path (ii): the fused fixed-step CDE solve on the FP32/FP64 CUDA-core pipe (sm_90a).
//
// One persistent-state kernel replaces what the reference does with ~10^4 small launches and
// ~4*10^3 host syncs per solve (SURVEY.md 3.1): for every Runge-Kutta stage it evaluates the
// spline derivative dX/dt (interpolation_cubic.py:331-336), the README-form linear vector
// field (README.md:42-49), the f.dX/dt contraction (solver.py:130) and the stage combination
// of torchdiffeq's fixed-grid solvers (restated in oracle/odeint_port.py), keeping the hidden
// state in registers for all steps and touching HBM only for the coefficient rows, z0 and the
// requested outputs.
//
// Roofline (SURVEY.md 8d): ~17.6 MFLOP and ~25 KB per path at (L=256, C=8, H=32), i.e. ~700
// flop/byte -- this kernel is bound by the FP32 FMA pipe, not by HBM.  It is therefore built
// like a register-tiled SGEMM: a CTA owns TB paths; thread (g, h) owns hidden unit h of ST
// consecutive paths and accumulates an ST x CT tile of  z . W^T  per channel chunk, with the
// stage input z^T and W^T staged in shared memory ([k][path] and [k][chunk][h][4] so that
// every shared-memory access is a conflict-free or broadcast 128-bit load).  The tensor-core
// variant lives in solve_tc.cu; this file is also the generic-shape path.
#include "common.cuh"

namespace tcde {

template <typename T, int N> struct alignas(sizeof(T) * N) Pack { T v[N]; };

template <typename T> struct SolveArgs {
    const T* control;        // cubic: [P][n_rows][4C]   linear: slopes [P][n_rows][C]
    const T* weight;         // [H*C][H]
    const T* bias;           // [H*C]
    const T* z0;             // [P][H]
    T* out;                  // [P][n_out][H]
    const T* step_dt;        // [n_steps]
    const int32_t* stage_index;   // [n_steps][n_stages]
    const T* stage_frac;          // [n_steps][n_stages]
    const int32_t* out_step;      // [n_out]
    const int32_t* out_mode;      // [n_out]
    const T* out_slope;           // [n_out]
    int64_t n_paths;
    int64_t n_rows;
    int C, Cp, H;
    int control_kind, method, n_stages;
    int n_steps, n_out;
    int groups;              // path groups per CTA (TB = groups * ST)
    int threads;
    T sign;
    // single evaluation mode (tcde_vector_field_linear): z0 is z, out[p][h] receives f(z) . dX/dt at
    // (eval_index, eval_frac) and the kernel returns after the first stage; no schedule is read
    int eval_only, eval_index;
    T eval_frac;
};

// Shared-memory carve-up (all offsets in elements of T; every region 16-byte aligned):
//   Ws   [H][Cp/4][H][4]     W^T, n = (chunk4, h, lane-in-chunk)
//   bs   [Cp/4][H][4]        bias in the same order
//   zin  [2][H][TBp]         stage input, transposed; TBp = TB + 4 (conflict-free column writes)
//   dxs  [2][TB][Cp]         dX/dt of the current / next stage
//   raw  [TB][3*Cp]          cp.async landing zone for the next stage's (b, 2c, 3d) rows
//   kst  [2][ST][threads]    Runge-Kutta stage slopes parked between stages (frees 2*ST registers
//                            per thread so that two CTAs fit per SM next to the 64 accumulators)
template <typename T> struct SolveSmem {
    size_t ws, bs, zin, dxs, raw, kst, total;
    int TB, TBp;
};

template <typename T> static SolveSmem<T> solve_smem_layout(int H, int Cp, int groups, int ST, int threads) {
    SolveSmem<T> s;
    s.TB = groups * ST;
    s.TBp = s.TB + 4;
    size_t off = 0;
    s.ws = off; off += (size_t)H * Cp * H;
    s.bs = off; off += (size_t)Cp * H;
    s.zin = off; off += (size_t)2 * H * s.TBp;
    s.dxs = off; off += (size_t)2 * s.TB * Cp;
    s.raw = off; off += (size_t)s.TB * 3 * Cp;
    s.kst = off; off += (size_t)2 * ST * threads;
    s.total = off * sizeof(T);
    return s;
}

template <typename T, int ST, int CT>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 && ST * CT >= 64) ? 2 : 1)
cdeint_simt_kernel(const SolveArgs<T> a, const SolveSmem<T> lay) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    using P4 = Pack<T, 4>;
    T* smem = reinterpret_cast<T*>(smem_raw);
    T* Ws = smem + lay.ws;
    T* bs = smem + lay.bs;
    T* zin = smem + lay.zin;
    T* dxs = smem + lay.dxs;
    T* raw = smem + lay.raw;
    T* kst = smem + lay.kst + threadIdx.x;    // slot (which, s) of this thread at kst[(which*ST + s) * threads]

    const int H = a.H, C = a.C, Cp = a.Cp;
    const int TB = lay.TB, TBp = lay.TBp;
    const int tid = threadIdx.x;
    const int nthreads = a.threads;
    const int nq = Cp / 4;                       // 4-channel chunks
    const int64_t path0 = (int64_t)blockIdx.x * TB;

    // ---- one-time staging of W^T and bias ------------------------------------------------
    for (int e = tid; e < H * Cp * H; e += nthreads) {
        // destination order (k, q, h, j); source weight[(h*C + c)][k] with c = 4q + j
        const int j = e & 3;
        int r = e >> 2;
        const int h = r % H; r /= H;
        const int q = r % nq;
        const int k = r / nq;
        const int c = 4 * q + j;
        Ws[e] = (c < C) ? a.weight[((int64_t)h * C + c) * H + k] : T(0);
    }
    for (int e = tid; e < Cp * H; e += nthreads) {
        const int j = e & 3;
        int r = e >> 2;
        const int h = r % H;
        const int q = r / H;
        const int c = 4 * q + j;
        bs[e] = (c < C) ? a.bias[h * C + c] : T(0);
    }

    // ---- thread roles --------------------------------------------------------------------
    const bool worker = tid < a.groups * H;
    const int g = worker ? tid / H : 0;
    const int h = worker ? tid - g * H : 0;
    const int lp0 = g * ST;                      // first local path of this thread

    // dX/dt producer items: (local path, 4-channel chunk); item i -> path i / nq, chunk i % nq
    const int n_items = TB * nq;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * C : C;
    const bool vec_ok = ((C & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.control) & 15) == 0);

    auto fetch_rows = [&](int idx) {             // asynchronous: lands in raw[], consumed by the issuing thread
        for (int it = tid; it < n_items; it += nthreads) {
            const int lp = it / nq, q = it - lp * nq;
            int64_t p = path0 + lp;
            if (p >= a.n_paths) p = a.n_paths - 1;
            const T* src = a.control + (p * a.n_rows + idx) * row_stride + (cubic ? C : 0) + 4 * q;
            T* dst = raw + (size_t)lp * 3 * Cp + 4 * q;
            const int parts = cubic ? 3 : 1;
            for (int w = 0; w < parts; ++w) {
                if (vec_ok) {
                    if (sizeof(T) == 4) cp_async16(dst + w * Cp, src + w * C);
                    else { cp_async16(dst + w * Cp, src + w * C); cp_async16(dst + w * Cp + 2, src + w * C + 2); }
                } else {
                    for (int j = 0; j < 4; ++j)
                        if (4 * q + j < C) {
                            if (sizeof(T) == 4) cp_async4(dst + w * Cp + j, src + w * C + j);
                            else dst[w * Cp + j] = src[w * C + j];
                        }
                }
            }
        }
        cp_async_commit();
    };
    auto produce_dx = [&](T frac, T* dst_dx) {   // interpolation_cubic.py:331-336, one rounding per op
        cp_async_wait<0>();
        for (int it = tid; it < n_items; it += nthreads) {
            const int lp = it / nq, q = it - lp * nq;
            const T* r = raw + (size_t)lp * 3 * Cp + 4 * q;
            P4 o;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                T v = T(0);
                if (4 * q + j < C) {
                    if (cubic) v = E::add(r[j], E::mul(E::add(r[Cp + j], E::mul(r[2 * Cp + j], frac)), frac));
                    else v = r[j];
                }
                o.v[j] = v;
            }
            *reinterpret_cast<P4*>(dst_dx + (size_t)lp * Cp + 4 * q) = o;
        }
    };

    // ---- state ---------------------------------------------------------------------------
    T y[ST];
#pragma unroll
    for (int s = 0; s < ST; ++s) {
        int64_t p = path0 + lp0 + s;
        if (p >= a.n_paths) p = a.n_paths - 1;
        y[s] = worker ? a.z0[p * H + h] : T(0);
    }
    auto park = [&](int which, int s, T v) { kst[(size_t)(which * ST + s) * nthreads] = v; };
    auto parked = [&](int which, int s) -> T { return kst[(size_t)(which * ST + s) * nthreads]; };
    auto write_out = [&](int j, const T* v) {
        if (!worker) return;
#pragma unroll
        for (int s = 0; s < ST; ++s) {
            const int64_t p = path0 + lp0 + s;
            if (p < a.n_paths) a.out[(p * a.n_out + j) * H + h] = v[s];
        }
    };
    int jn = 0;
    if (!a.eval_only) {
        while (jn < a.n_out && a.out_step[jn] < 0) { write_out(jn, y); ++jn; }
    }

    // stage 0 inputs
    if (worker) {
#pragma unroll
        for (int s = 0; s < ST; ++s) zin[(size_t)h * TBp + lp0 + s] = y[s];
    }
    fetch_rows(a.eval_only ? a.eval_index : a.stage_index[0]);
    produce_dx(a.eval_only ? a.eval_frac : a.stage_frac[0], dxs);
    __syncthreads();

    const int n_stages = a.n_stages;
    const int total = a.eval_only ? 1 : a.n_steps * n_stages;
    const T third = T(1.0 / 3.0);
    int step = 0, sub = 0;
    T dt = a.eval_only ? T(0) : a.step_dt[0];

    for (int st = 0; st < total; ++st) {
        const int cur = st & 1, nxt = cur ^ 1;
        const bool more = (st + 1 < total);
        T next_frac = T(0);
        if (more) {
            fetch_rows(a.stage_index[st + 1]);
            next_frac = a.stage_frac[st + 1];
        }
        // ---- f(z) . dX/dt for this thread's (ST paths, hidden unit h) ----------------------
        T kv[ST];
#pragma unroll
        for (int s = 0; s < ST; ++s) kv[s] = T(0);
        if (worker) {
            const T* zc = zin + (size_t)cur * H * TBp + lp0;
            const T* dc = dxs + (size_t)cur * TB * Cp + (size_t)lp0 * Cp;
            for (int q0 = 0; q0 < nq; q0 += CT / 4) {
                const T* wk = Ws + ((size_t)q0 * H + h) * 4;
                {
                    T acc[ST][CT];
#pragma unroll
                    for (int cc = 0; cc < CT / 4; ++cc) {
                        const P4 b4 = *reinterpret_cast<const P4*>(bs + ((size_t)(q0 + cc) * H + h) * 4);
#pragma unroll
                        for (int s = 0; s < ST; ++s)
#pragma unroll
                            for (int j = 0; j < 4; ++j) acc[s][cc * 4 + j] = b4.v[j];
                    }
#pragma unroll 2
                    for (int k = 0; k < H; ++k) {
                        T zv[ST], wv[CT];
#pragma unroll
                        for (int s4 = 0; s4 < ST / 4; ++s4) {
                            const P4 z4 = *reinterpret_cast<const P4*>(zc + (size_t)k * TBp + 4 * s4);
#pragma unroll
                            for (int j = 0; j < 4; ++j) zv[4 * s4 + j] = z4.v[j];
                        }
#pragma unroll
                        for (int cc = 0; cc < CT / 4; ++cc) {
                            const P4 w4 = *reinterpret_cast<const P4*>(wk + (size_t)k * Cp * H + (size_t)cc * H * 4);
#pragma unroll
                            for (int j = 0; j < 4; ++j) wv[4 * cc + j] = w4.v[j];
                        }
#pragma unroll
                        for (int s = 0; s < ST; ++s)
#pragma unroll
                            for (int c = 0; c < CT; ++c) acc[s][c] = fma(zv[s], wv[c], acc[s][c]);
                    }
#pragma unroll
                    for (int s = 0; s < ST; ++s) {
#pragma unroll
                        for (int cc = 0; cc < CT / 4; ++cc) {
                            const P4 d4 = *reinterpret_cast<const P4*>(dc + (size_t)s * Cp + 4 * (q0 + cc));
#pragma unroll
                            for (int j = 0; j < 4; ++j) kv[s] = fma(acc[s][cc * 4 + j], d4.v[j], kv[s]);
                        }
                    }
                }
            }
            if (a.sign < T(0)) {
#pragma unroll
                for (int s = 0; s < ST; ++s) kv[s] = -kv[s];
            }
        }
        if (a.eval_only) {                       // out[p][h] = f(z) . dX/dt, nothing else
            if (worker) {
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    const int64_t p = path0 + lp0 + s;
                    if (p < a.n_paths) a.out[p * H + h] = kv[s];
                }
            }
            return;
        }
        // ---- Runge-Kutta combination (oracle/odeint_port.py, one rounding per op) ----------
        bool step_done = false;
        T zn[ST];
        if (a.method == TCDE_RK4_38) {
            // 3/8 rule.  Slot 0 keeps k1; slot 1 keeps k2, then k2 + k3 (all that the last
            // combination needs), so only y[] stays in registers across the stage GEMMs.
            if (sub == 0) {
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    park(0, s, kv[s]);
                    zn[s] = E::add(y[s], E::mul(E::mul(dt, kv[s]), third));
                }
            } else if (sub == 1) {
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    park(1, s, kv[s]);
                    zn[s] = E::add(y[s], E::mul(dt, E::sub(kv[s], E::mul(parked(0, s), third))));
                }
            } else if (sub == 2) {
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    const T k2 = parked(1, s);
                    zn[s] = E::add(y[s], E::mul(dt, E::add(E::sub(parked(0, s), k2), kv[s])));
                    park(1, s, E::add(k2, kv[s]));
                }
            } else {
#pragma unroll
                for (int s = 0; s < ST; ++s) {
                    const T sum = E::add(E::add(parked(0, s), E::mul(T(3), parked(1, s))), kv[s]);
                    zn[s] = E::add(y[s], E::mul(E::mul(sum, dt), T(0.125)));
                }
                step_done = true;
            }
        } else if (a.method == TCDE_MIDPOINT) {
            if (sub == 0) {
                const T half = E::mul(T(0.5), dt);
#pragma unroll
                for (int s = 0; s < ST; ++s) zn[s] = E::add(y[s], E::mul(kv[s], half));
            } else {
#pragma unroll
                for (int s = 0; s < ST; ++s) zn[s] = E::add(y[s], E::mul(dt, kv[s]));
                step_done = true;
            }
        } else {
#pragma unroll
            for (int s = 0; s < ST; ++s) zn[s] = E::add(y[s], E::mul(dt, kv[s]));
            step_done = true;
        }
        if (step_done) {
            // requested output times that fall in (t0, t1] of this step (linear interpolation)
            while (jn < a.n_out && a.out_step[jn] == step) {
                const int mode = a.out_mode[jn];
                if (mode == 0) write_out(jn, y);
                else if (mode == 1) write_out(jn, zn);
                else {
                    const T slope = a.out_slope[jn];
                    T v[ST];
#pragma unroll
                    for (int s = 0; s < ST; ++s) v[s] = E::add(y[s], E::mul(slope, E::sub(zn[s], y[s])));
                    write_out(jn, v);
                }
                ++jn;
            }
#pragma unroll
            for (int s = 0; s < ST; ++s) y[s] = zn[s];
            ++step;
            sub = 0;
            if (step < a.n_steps) dt = a.step_dt[step];
        } else {
            ++sub;
        }
        if (more) {
            if (worker) {
                T* zo = zin + (size_t)nxt * H * TBp + (size_t)h * TBp + lp0;
#pragma unroll
                for (int s4 = 0; s4 < ST / 4; ++s4) {
                    P4 o;
#pragma unroll
                    for (int j = 0; j < 4; ++j) o.v[j] = zn[4 * s4 + j];
                    *reinterpret_cast<P4*>(zo + 4 * s4) = o;
                }
            }
            produce_dx(next_frac, dxs + (size_t)nxt * TB * Cp);
            __syncthreads();
        }
    }
}

// One vector-field evaluation f(z) . dX/dt at a given (index, frac) -- the building block the
// adaptive (dopri5) driver calls.  Same data flow as one stage of the solve kernel, with z
// read from / the result written to global memory.
template <typename T>
__global__ void __launch_bounds__(256)
vector_field_kernel(const T* __restrict__ control, int control_kind, int64_t n_rows, const T* __restrict__ weight,
                    const T* __restrict__ bias, const T* __restrict__ z, T* __restrict__ out, int64_t n_paths, int C,
                    int H, int index, T frac) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    T* zs = reinterpret_cast<T*>(smem_raw);      // [paths_per_cta][H]
    T* dx = zs + (size_t)(blockDim.x / H) * H;   // [paths_per_cta][C]
    const int ppc = blockDim.x / H;
    const int lp = threadIdx.x / H, h = threadIdx.x - lp * H;
    const int64_t p = (int64_t)blockIdx.x * ppc + lp;
    const bool live = (lp < ppc) && (p < n_paths);
    const bool cubic = (control_kind == TCDE_CONTROL_CUBIC);
    if (live) zs[lp * H + h] = z[p * H + h];
    for (int e = threadIdx.x; e < ppc * C; e += blockDim.x) {
        const int l = e / C, c = e - l * C;
        const int64_t pp = (int64_t)blockIdx.x * ppc + l;
        T v = T(0);
        if (pp < n_paths) {
            if (cubic) {
                const T* r = control + (pp * n_rows + index) * 4 * C;
                v = E::add(r[C + c], E::mul(E::add(r[2 * C + c], E::mul(r[3 * C + c], frac)), frac));
            } else {
                v = control[(pp * n_rows + index) * C + c];
            }
        }
        dx[e] = v;
    }
    __syncthreads();
    if (!live) return;
    T res = T(0);
    for (int c = 0; c < C; ++c) {
        const T* w = weight + ((int64_t)h * C + c) * H;
        T acc = bias[h * C + c];
        for (int k = 0; k < H; ++k) acc = fma(zs[lp * H + k], w[k], acc);
        res = fma(acc, dx[lp * C + c], res);
    }
    out[p * H + h] = res;
}

template <typename T, int ST, int CT>
static int launch_solve_ct(SolveArgs<T> a, cudaStream_t stream) {
    auto kern = cdeint_simt_kernel<T, ST, CT>;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    int g_max = 256 / a.H;
    if (g_max < 1) g_max = 1;
    if (g_max > 32) g_max = 32;
    const int64_t need_groups = (a.n_paths + ST - 1) / ST;
    if (g_max > need_groups) g_max = (int)need_groups;
    // Every path costs the same, so a launch is a sequence of equal "waves" of resident CTAs.
    // Pick the CTA size (path groups per CTA) that wastes the least of the last wave:
    // cost = waves * (paths resident per SM in a wave).
    const int sms = sm_count();
    int best_g = 0;
    double best_cost = 0;
    SolveSmem<T> best_lay{};
    for (int g = g_max; g >= (g_max + 1) / 2; --g) {
        const int threads = ((g * a.H + 31) / 32) * 32;
        SolveSmem<T> lay = solve_smem_layout<T>(a.H, a.Cp, g, ST, threads);
        if (lay.total > 220 * 1024) continue;
        int occ = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, lay.total) != cudaSuccess || occ < 1)
            continue;
        const int64_t ctas = (a.n_paths + lay.TB - 1) / lay.TB;
        const int64_t slots = (int64_t)sms * occ;
        const int64_t waves = (ctas + slots - 1) / slots;
        const int64_t resident = ctas < slots ? (ctas + sms - 1) / sms : occ;
        const double cost = (double)waves * (double)resident * g;
        if (best_g == 0 || cost < best_cost) {
            best_g = g;
            best_cost = cost;
            best_lay = lay;
        }
    }
    TCDE_CHECK_SUPPORTED(best_g > 0,
                         "fused solve: hidden=%d channels=%d does not fit the CUDA-core kernel's shared memory", a.H,
                         a.C);
    a.groups = best_g;
    a.threads = ((best_g * a.H + 31) / 32) * 32;
    const int64_t ctas = (a.n_paths + best_lay.TB - 1) / best_lay.TB;
    TCDE_CHECK_SUPPORTED(ctas < (1ll << 31), "too many paths");
    kern<<<(unsigned)ctas, a.threads, best_lay.total, stream>>>(a, best_lay);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

template <typename T, int ST>
static int launch_solve(const SolveArgs<T>& a_in, cudaStream_t stream) {
    SolveArgs<T> a = a_in;
    TCDE_CHECK_SUPPORTED(a.H <= 256, "fused solve: hidden=%d > 256 is not supported by the CUDA-core kernel", a.H);
    a.Cp = ((a.C + 3) / 4) * 4;
    if (a.Cp % 8 == 0) return launch_solve_ct<T, ST, 8>(a, stream);
    return launch_solve_ct<T, ST, 4>(a, stream);
}

int solve_simt_f32(const SolveArgs<float>& a, cudaStream_t s) { return launch_solve<float, 8>(a, s); }
int solve_simt_f64(const SolveArgs<double>& a, cudaStream_t s) { return launch_solve<double, 4>(a, s); }

template <typename T>
static int launch_field(const void* control, int control_kind, int64_t n_rows, const void* weight, const void* bias,
                        const void* z, void* out, int64_t n_paths, int C, int H, int index, double frac,
                        cudaStream_t stream) {
    TCDE_CHECK_SUPPORTED(H <= 256, "vector field: hidden=%d > 256", H);
    {
        // the register-tiled stage of the fused solve, run for exactly one evaluation
        SolveArgs<T> a{};
        a.control = (const T*)control; a.weight = (const T*)weight; a.bias = (const T*)bias;
        a.z0 = (const T*)z; a.out = (T*)out;
        a.n_paths = n_paths; a.n_rows = n_rows; a.C = C; a.H = H;
        a.control_kind = control_kind; a.method = TCDE_EULER; a.n_stages = 1; a.n_steps = 1; a.n_out = 1;
        a.sign = T(1);
        a.eval_only = 1; a.eval_index = index; a.eval_frac = (T)frac;
        const int rc = launch_solve<T, (sizeof(T) == 4 ? 8 : 4)>(a, stream);
        if (rc != TCDE_ERR_UNSUPPORTED) return rc;
    }
    const int ppc = 256 / H;
    const int threads = ppc * H;
    const size_t smem = (size_t)ppc * (H + C) * sizeof(T);
    TCDE_CHECK_SUPPORTED(smem <= 48 * 1024, "vector field: channels=%d too large", C);
    const int64_t ctas = (n_paths + ppc - 1) / ppc;
    vector_field_kernel<T><<<(unsigned)ctas, threads, smem, stream>>>(
        (const T*)control, control_kind, n_rows, (const T*)weight, (const T*)bias, (const T*)z, (T*)out, n_paths, C, H,
        index, (T)frac);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

// ---- tensor-core variant (solve_tc.cu) ---------------------------------------------------------
#ifndef TCDE_DEFAULT_TC_MODE
#define TCDE_DEFAULT_TC_MODE 1      // bit 0: 2xFP16 operand split (6 MMAs per 16 x 8 block) instead of 3xTF32 (12)
#endif
static int g_solve_variant = 0;     // 0 auto, 1 CUDA-core kernel, 2 / 3 tensor cores 3xTF32, 4 tensor cores 2xFP16
int current_solve_variant() { return g_solve_variant; }

}  // namespace tcde

using namespace tcde;

extern "C" int tcde_set_solve_variant(int variant) {
    TCDE_CHECK_ARG(variant >= 0 && (variant & 15) <= 6,
                   "variant=%d (0 auto, 1 CUDA-core kernel, 3 / 4 tensor-core kernel with the 3xTF32 / 2xFP16 operand split; "
                   "2, 6 / 5 are aliases of 3 / 4)", variant);
    g_solve_variant = variant & 15;      // bits above 15 (profiling switches of earlier kernels) are accepted and ignored
    return TCDE_OK;
}

extern "C" int tcde_vector_field_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                        const void* bias, const void* z, void* out, int64_t n_paths, int64_t channels,
                                        int64_t hidden, int32_t index, double frac, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && weight && bias && z && out, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(index >= 0 && index < n_rows, "index=%d outside [0, %lld)", index, (long long)n_rows);
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (dtype == TCDE_F32)
        return launch_field<float>(control, control_kind, n_rows, weight, bias, z, out, n_paths, (int)channels,
                                   (int)hidden, index, frac, s);
    return launch_field<double>(control, control_kind, n_rows, weight, bias, z, out, n_paths, (int)channels,
                                (int)hidden, index, frac, s);
}

static int solve_fixed_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                              const void* bias, const void* z0, void* out, int64_t n_paths, int64_t channels,
                              int64_t hidden, int method, int64_t n_steps, const void* step_dt,
                              const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                              const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                              double sign, int dtype, void* stage_dump, void* stream) {
    TCDE_CHECK_ARG(control && weight && bias && z0 && out, "null data pointer");
    TCDE_CHECK_ARG(step_dt && stage_index && stage_frac && out_step && out_mode && out_slope, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && channels >= 1 && hidden >= 1 && n_rows >= 1, "bad sizes");
    TCDE_CHECK_ARG(n_steps >= 1 && n_out >= 1, "n_steps=%lld n_out=%lld", (long long)n_steps, (long long)n_out);
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    TCDE_CHECK_ARG(method == TCDE_EULER || method == TCDE_MIDPOINT || method == TCDE_RK4_38, "method=%d", method);
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    if (n_paths == 0) return TCDE_OK;
    const int n_stages = (method == TCDE_RK4_38) ? 4 : (method == TCDE_MIDPOINT) ? 2 : 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (dtype == TCDE_F32) {
        // auto: the tensor-core kernel wherever it is built for the shape (parity-tested against the
        // CUDA-core kernel and the fp64 oracle), the CUDA-core kernel for every other shape
        const bool tc_ok = solve_tc_supported((int)hidden, (int)channels) &&
                           ((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(z0) |
                             reinterpret_cast<uintptr_t>(out)) & 15) == 0;
        const bool want_tc = (g_solve_variant >= 2) || (g_solve_variant == 0 && tc_ok);
        if (want_tc) {
            UmmaArgs u{(const float*)control, (const float*)weight, (const float*)bias, (const float*)z0, (float*)out,
                       (const float*)step_dt, stage_index, (const float*)stage_frac, out_step, out_mode,
                       (const float*)out_slope, n_paths, n_rows, control_kind, method, n_stages, (int)n_steps,
                       (int)n_out, (float)sign, (float*)stage_dump};
            // 2 / 3 / 6 = 3xTF32 split, 4 / 5 = 2xFP16 split (2, 5, 6: aliases from the development history)
            const int mode = (g_solve_variant == 2 || g_solve_variant == 3 || g_solve_variant == 6) ? 0
                             : (g_solve_variant == 4 || g_solve_variant == 5) ? 1 : TCDE_DEFAULT_TC_MODE;
            return solve_tc_f32(u, (int)hidden, (int)channels, mode, s);
        }
        TCDE_CHECK_SUPPORTED(stage_dump == nullptr, "the stage dump is written by the tensor-core solve only "
                             "(fp32, hidden=32, channels=8, 16-byte aligned buffers)");
        SolveArgs<float> a{(const float*)control, (const float*)weight, (const float*)bias, (const float*)z0,
                           (float*)out, (const float*)step_dt, stage_index, (const float*)stage_frac, out_step,
                           out_mode, (const float*)out_slope, n_paths, n_rows, (int)channels, 0, (int)hidden,
                           control_kind, method, n_stages, (int)n_steps, (int)n_out, 0, 0, (float)sign, 0, 0, 0.f};
        return solve_simt_f32(a, s);
    }
    TCDE_CHECK_SUPPORTED(stage_dump == nullptr, "the stage dump is written by the fp32 tensor-core solve only");
    SolveArgs<double> a{(const double*)control, (const double*)weight, (const double*)bias, (const double*)z0,
                        (double*)out, (const double*)step_dt, stage_index, (const double*)stage_frac, out_step,
                        out_mode, (const double*)out_slope, n_paths, n_rows, (int)channels, 0, (int)hidden,
                        control_kind, method, n_stages, (int)n_steps, (int)n_out, 0, 0, (double)sign, 0, 0, 0.0};
    return solve_simt_f64(a, s);
}

extern "C" int tcde_cdeint_fixed_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                        const void* bias, const void* z0, void* out, int64_t n_paths, int64_t channels,
                                        int64_t hidden, int method, int64_t n_steps, const void* step_dt,
                                        const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                        const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                                        double sign, int dtype, void* stream) {
    return solve_fixed_linear(control, control_kind, n_rows, weight, bias, z0, out, n_paths, channels, hidden, method,
                              n_steps, step_dt, stage_index, stage_frac, n_out, out_step, out_mode, out_slope, sign, dtype,
                              nullptr, stream);
}

extern "C" int tcde_cdeint_fixed_linear_stages(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                               const void* bias, const void* z0, void* out, void* stage_dump,
                                               int64_t n_paths, int64_t channels, int64_t hidden, int method,
                                               int64_t n_steps, const void* step_dt, const int32_t* stage_index,
                                               const void* stage_frac, int64_t n_out, const int32_t* out_step,
                                               const int32_t* out_mode, const void* out_slope, double sign, int dtype,
                                               void* stream) {
    TCDE_CHECK_ARG(stage_dump != nullptr, "null stage dump");
    return solve_fixed_linear(control, control_kind, n_rows, weight, bias, z0, out, n_paths, channels, hidden, method,
                              n_steps, step_dt, stage_index, stage_frac, n_out, out_step, out_mode, out_slope, sign, dtype,
                              stage_dump, stream);
}
