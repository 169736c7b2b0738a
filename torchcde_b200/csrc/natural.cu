// Hot path (i): batched spline-coefficient construction (sm_90a) -- natural cubic splines (NaN-free knots and the per-series version with missing values).
//
// The builders are HBM-bound streaming kernels (SURVEY.md 8d: ~1 flop per byte).  The design rules
// that matter are the memory ones: coalesced 128-bit loads, results staged in shared memory and
// written back as contiguous 1-D bulk (TMA) stores, persistent CTAs sized from the SM count.
// Arithmetic uses tcde::exact<> (one rounding per operation, no FMA contraction) wherever the header
// promises bit-identical results.
#include "builders_common.cuh"

namespace tcde {

// =========================================================================================
// Natural cubic spline, NaN-free knots  (interpolation_cubic.py:7-53, misc.py:13-67)
// =========================================================================================
// The knots are shared by the whole batch (misc.py:83), so the eliminated diagonal and the
// forward multipliers of the Thomas solve are batch independent: one tiny kernel forms them
// once (the reference recomputes them for every series).  workspace = [rdt | rdt2 | mult | rnd].
template <typename T>
__global__ void natural_prep_kernel(const T* __restrict__ t, T* __restrict__ ws, int L) {
    using E = exact<T>;
    T* rdt = ws;
    T* rdt2 = ws + L;
    T* mult = ws + 2 * L;
    T* rnd = ws + 3 * L;
    __shared__ int s_wf, s_wb;
    for (int i = threadIdx.x; i < L - 1; i += blockDim.x) {
        const T t0 = t ? t[i] : T(i), t1 = t ? t[i + 1] : T(i + 1);
        const T r = E::div(T(1), E::sub(t1, t0));
        rdt[i] = r;
        rdt2[i] = E::mul(r, r);
    }
    if (threadIdx.x == 0) { s_wf = 0; s_wb = 0; }
    __syncthreads();
    if (threadIdx.x == 0) {
        rdt[L - 1] = T(0);
        rdt2[L - 1] = T(0);
        // diag[i] = 2 * (rdt[i] + rdt[i-1]) with the out-of-range terms absent (cubic.py:31-35)
        T nd = E::mul(T(2), rdt[0]);
        T r_prev = rdt[0];
        // mult[0] is unused by the sweeps (0); for two knots it carries t1 - t0 (cubic.py:18)
        mult[0] = (L > 2) ? T(0) : E::sub(t ? t[1] : T(1), t ? t[0] : T(0));
        rnd[0] = E::div(T(1), nd);
        for (int i = 1; i < L; ++i) {
            const T r_cur = (i < L - 1) ? rdt[i] : T(0);
            const T diag = E::mul(T(2), E::add(r_cur, r_prev));
            const T w = E::div(r_prev, nd);                      // misc.py:59
            nd = E::sub(diag, E::mul(w, r_prev));                // misc.py:60
            mult[i] = w;
            rnd[i] = E::div(T(1), nd);
            r_prev = r_cur;
        }
    }
    __syncthreads();
    // Window sizes for the parallel sweeps of natural_win_kernel: the forward recurrence
    // f[i] = rhs[i] - mult[i] f[i-1] forgets f[i-w] by the factor prod |mult|, the backward one
    // k[i] = (f[i] - rdt[i] k[i+1]) rnd[i] forgets k[i+w] by prod |rdt rnd|; both factors are
    // ~0.27 per knot for a diagonally dominant system.  A window is long enough when that
    // product is below eps/16 (or it reaches the end of the series, where the start is exact).
    if (L > 2) {
        const T tol = (sizeof(T) == 4) ? T(3.7e-9) : T(1.4e-17);
        int wf = 0, wb = 0;
        for (int i = 1 + threadIdx.x; i < L; i += blockDim.x) {
            T prod = T(1);
            int w = 0;
            for (int j = i; j >= 1 && prod > tol; --j) { prod *= fabs(mult[j]); ++w; }
            wf = max(wf, w);
        }
        for (int i = threadIdx.x; i < L - 1; i += blockDim.x) {
            T prod = T(1);
            int w = 0;
            for (int j = i; j < L - 1 && prod > tol; ++j) { prod *= fabs(rdt[j] * rnd[j]); ++w; }
            wb = max(wb, w);
        }
        atomicMax(&s_wf, wf);
        atomicMax(&s_wb, wb);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        ws[4 * L] = T(s_wf);
        ws[4 * L + 1] = T(s_wb);
    }
}

// Natural cubic spline, parallel version.  One path at a time per CTA; thread = (series, chunk of
// G consecutive knots).  Each thread runs the two Thomas recurrences over its chunk preceded by
// a warm-up window (sizes from natural_prep_kernel), so all 256 threads sweep concurrently
// instead of one thread per series walking all L knots: the sweeps stop being the
// latency-bound phase that ncu showed (issue slots 28% busy, DRAM 11%).  The result equals the
// sequential recurrence up to a truncated influence below eps/16 -- the same few-ulp class as
// replacing the division by a multiplication with 1/nd.
template <typename T>
__global__ void __launch_bounds__(kThreads)
natural_win_kernel(const T* __restrict__ x, const T* __restrict__ ws, T* __restrict__ out, int64_t n_paths, int L,
                   int C, int Lp, int G, int TR, int use_bulk, int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    const int row_elems = 4 * C;
    T* ot0 = reinterpret_cast<T*>(smem_raw);
    T* ot1 = ot0 + (size_t)TR * row_elems;
    T* rdt = ot1 + (size_t)TR * row_elems;
    T* rdt2 = rdt + L;
    T* mult = rdt2 + L;
    T* rnd = mult + L;
    T* xs = rnd + L + 8;                 // [C][Lp]
    T* fs = xs + (size_t)C * Lp;         // forward-sweep values
    T* ks = fs + (size_t)C * Lp;         // knot slopes

    const int tid = threadIdx.x;
    for (int e = tid; e < 4 * L + 2; e += kThreads) rdt[e] = ws[e];
    __syncthreads();
    const int wf = (int)rdt[4 * L], wb = (int)rdt[4 * L + 1];
    const int n_chunks = (L + G - 1) / G;
    const int n_items = C * n_chunks;
    const int di = kThreads / C, dc = kThreads - di * C;
    const bool vec4 = (sizeof(T) == 4) && ((C & 3) == 0) && L > 2 && use_bulk &&
                      (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    bool saw_nan = false;
    int buf = 0;

    for (int64_t p = blockIdx.x; p < n_paths; p += gridDim.x) {
        __syncthreads();                 // the previous path's coefficient phase is done with xs / ks
        if (vec4) {                      // 128-bit coalesced loads, transposed to [c][i]
            const float4* xg4 = reinterpret_cast<const float4*>(x + p * (int64_t)L * C);
            const int Q = C >> 2;
            int i = tid / Q, q = tid - (tid / Q) * Q;
            const int dq_i = kThreads / Q, dq_q = kThreads - dq_i * Q;
            for (int e = tid; e < L * Q; e += kThreads) {
                const float4 v4 = xg4[e];
                saw_nan |= is_nan(v4.x) | is_nan(v4.y) | is_nan(v4.z) | is_nan(v4.w);
                T* dst = xs + (4 * q) * Lp + i;
                dst[0] = (T)v4.x; dst[Lp] = (T)v4.y; dst[2 * Lp] = (T)v4.z; dst[3 * Lp] = (T)v4.w;
                i += dq_i;
                q += dq_q;
                if (q >= Q) { q -= Q; ++i; }
            }
        } else {
            const T* xg = x + p * (int64_t)L * C;
            int i = tid / C, c = tid - (tid / C) * C;
            for (int e = tid; e < L * C; e += kThreads) {
                const T v = xg[e];
                saw_nan |= is_nan(v);
                xs[c * Lp + i] = v;
                i += di;
                c += dc;
                if (c >= C) { c -= C; ++i; }
            }
        }
        __syncthreads();
        if (L > 2) {
            const bool pairs = (sizeof(T) == 4) && ((C & 1) == 0);
            if (pairs) {
                // two series per thread, packed arithmetic: half the instructions of the scalar sweeps
                const int C2 = C >> 1;
                const int n_pair_items = C2 * n_chunks;
                for (int it = tid; it < n_pair_items; it += kThreads) {     // forward sweep (misc.py:58-61)
                    const int c = 2 * (it % C2), j = it / C2;
                    const int g0 = j * G, g1 = min(g0 + G, L);
                    const float* x0 = reinterpret_cast<const float*>(xs) + c * Lp;
                    float* f0 = reinterpret_cast<float*>(fs) + c * Lp;
                    int i = max(g0 - wf, 0);
                    f2 f = pk2(0.f, 0.f);
                    const f2 three = pk2(3.f, 3.f);
                    f2 x_lo = pk2(x0[i], x0[Lp + i]);
                    f2 sc_prev = pk2(0.f, 0.f);
                    if (i > 0) {
                        const float r2 = (float)rdt2[i - 1];
                        sc_prev = mul2(mul2(three, sub2(x_lo, pk2(x0[i - 1], x0[Lp + i - 1]))), pk2(r2, r2));
                    }
                    for (; i < g1; ++i) {
                        // scaled difference 3 (x[i+1] - x[i]) / dt_i^2; rdt2[L-1] = 0 closes the system (cubic.py:36-39)
                        const int in = min(i + 1, L - 1);
                        const f2 x_hi = pk2(x0[in], x0[Lp + in]);
                        const float r2 = (float)rdt2[i];
                        const f2 sc = mul2(mul2(three, sub2(x_hi, x_lo)), pk2(r2, r2));
                        x_lo = x_hi;
                        const float m = (float)mult[i];
                        f = sub2(add2(sc, sc_prev), mul2(pk2(m, m), f));
                        sc_prev = sc;
                        if (i >= g0) upk2(f, f0[i], f0[Lp + i]);
                    }
                }
            } else {
                for (int it = tid; it < n_items; it += kThreads) {
                    const int c = it % C, j = it / C;
                    const int g0 = j * G, g1 = min(g0 + G, L);
                    const T* xr = xs + c * Lp;
                    T* fr = fs + c * Lp;
                    int i = max(g0 - wf, 0);
                    T f = T(0);
                    T x_lo = xr[i];
                    T sc_prev = (i > 0) ? E::mul(E::mul(T(3), E::sub(x_lo, xr[i - 1])), rdt2[i - 1]) : T(0);
                    for (; i < g1; ++i) {
                        const T x_hi = xr[min(i + 1, L - 1)];
                        const T sc = E::mul(E::mul(T(3), E::sub(x_hi, x_lo)), rdt2[i]);      // rdt2[L-1] = 0
                        x_lo = x_hi;
                        f = E::sub(E::add(sc, sc_prev), E::mul(mult[i], f));     // cubic.py:36-39, misc.py:61
                        sc_prev = sc;
                        if (i >= g0) fr[i] = f;
                    }
                }
            }
            __syncthreads();
            if (pairs) {
                const int C2 = C >> 1;
                const int n_pair_items = C2 * n_chunks;
                for (int it = tid; it < n_pair_items; it += kThreads) {     // back substitution (misc.py:63-65)
                    const int c = 2 * (it % C2), j = it / C2;
                    const int g0 = j * G, g1 = min(g0 + G, L);
                    const float* f0 = reinterpret_cast<const float*>(fs) + c * Lp;
                    float* k0 = reinterpret_cast<float*>(ks) + c * Lp;
                    f2 k = pk2(0.f, 0.f);
                    for (int i = min(g1 - 1 + wb, L - 1); i >= g0; --i) {
                        const float rd = (float)rdt[i], rn = (float)rnd[i];
                        k = mul2(sub2(pk2(f0[i], f0[Lp + i]), mul2(pk2(rd, rd), k)), pk2(rn, rn));
                        if (i < g1) upk2(k, k0[i], k0[Lp + i]);
                    }
                }
            } else {
                for (int it = tid; it < n_items; it += kThreads) {
                    const int c = it % C, j = it / C;
                    const int g0 = j * G, g1 = min(g0 + G, L);
                    const T* fr = fs + c * Lp;
                    T* kr = ks + c * Lp;
                    T k = T(0);
                    for (int i = min(g1 - 1 + wb, L - 1); i >= g0; --i) {
                        k = E::mul(E::sub(fr[i], E::mul(rdt[i], k)), rnd[i]);    // misc.py:63-65 (rdt[L-1] = 0)
                        if (i < g1) kr[i] = k;
                    }
                }
            }
        }
        __syncthreads();
        if (vec4) {
            // coefficient rows straight from registers to global memory: thread = (interval, 4 channels), four
            // 128-bit stores that each fill whole 32-byte sectors (a warp completes its 128-byte lines across
            // the four instructions).  No staging tile: the shared memory saved doubles the resident CTAs.
            const int Q = C >> 2;
            float4* og4 = reinterpret_cast<float4*>(out + p * (int64_t)(L - 1) * row_elems);
            int i = tid / Q, q = tid - (tid / Q) * Q;
            const int dq_i = kThreads / Q, dq_q = kThreads - dq_i * Q;
            for (int e = tid; e < (L - 1) * Q; e += kThreads) {
                const float rd = (float)rdt[i], rd2 = (float)rdt2[i];
                const f2 rdp = pk2(rd, rd), rd2p = pk2(rd2, rd2);
                float av[4], bv[4], cv[4], dv[4];
#pragma unroll
                for (int j = 0; j < 4; j += 2) {
                    const float* xr0 = reinterpret_cast<const float*>(xs) + (4 * q + j) * Lp + i;
                    const float* kr0 = reinterpret_cast<const float*>(ks) + (4 * q + j) * Lp + i;
                    const f2 xl = pk2(xr0[0], xr0[Lp]), xh = pk2(xr0[1], xr0[Lp + 1]);
                    const f2 kl = pk2(kr0[0], kr0[Lp]), kh = pk2(kr0[1], kr0[Lp + 1]);
                    const f2 six = mul2(pk2(2.f, 2.f), mul2(pk2(3.f, 3.f), sub2(xh, xl)));
                    const f2 sr = mul2(six, rdp);
                    const f2 c2 = mul2(sub2(sub2(sr, mul2(pk2(4.f, 4.f), kl)), mul2(pk2(2.f, 2.f), kh)), rdp);   // :45-47
                    const f2 d3 = mul2(sub2(mul2(pk2(3.f, 3.f), add2(kl, kh)), sr), rd2p);                          // :48-50
                    upk2(xl, av[j], av[j + 1]);
                    upk2(kl, bv[j], bv[j + 1]);
                    upk2(c2, cv[j], cv[j + 1]);
                    upk2(d3, dv[j], dv[j + 1]);
                }
                float4* row = og4 + (size_t)i * (4 * Q) + q;
                row[0] = make_float4(av[0], av[1], av[2], av[3]);
                row[Q] = make_float4(bv[0], bv[1], bv[2], bv[3]);
                row[2 * Q] = make_float4(cv[0], cv[1], cv[2], cv[3]);
                row[3 * Q] = make_float4(dv[0], dv[1], dv[2], dv[3]);
                i += dq_i;
                q += dq_q;
                if (q >= Q) { q -= Q; ++i; }
            }
            continue;
        }
        for (int r0 = 0; r0 < L - 1; r0 += TR, buf ^= 1) {
            const int nr = min(TR, L - 1 - r0);
            if (use_bulk && tid == 0) bulk_wait_read<1>();
            __syncthreads();
            T* ot = buf ? ot1 : ot0;
            int i = tid / C, c = tid - (tid / C) * C;
            for (int e = tid; e < nr * C; e += kThreads) {
                const int r = r0 + i;
                const T* xr = xs + c * Lp + r;
                const T* kr = ks + c * Lp + r;
                const T xl = xr[0], xh = xr[1];
                T b, two_c, three_d;
                if (L == 2) {
                    b = E::div(E::sub(xh, xl), mult[0]);
                    two_c = T(0);
                    three_d = T(0);
                } else {
                    const T kl = kr[0], kh = kr[1];
                    const T six = E::mul(T(2), E::mul(T(3), E::sub(xh, xl)));
                    const T sr = E::mul(six, rdt[r]);
                    b = kl;
                    two_c = E::mul(E::sub(E::sub(sr, E::mul(T(4), kl)), E::mul(T(2), kh)), rdt[r]);
                    three_d = E::mul(E::add(-sr, E::mul(T(3), E::add(kl, kh))), rdt2[r]);
                }
                T* row = ot + (size_t)i * row_elems + c;
#pragma unroll
                for (int kq = 0; kq < 4; ++kq) {
                    const int w = (kq + i) & 3;
                    const T v = (w == 0) ? xl : (w == 1) ? b : (w == 2) ? two_c : three_d;
                    row[w * C] = v;
                }
                i += di;
                c += dc;
                if (c >= C) { c -= C; ++i; }
            }
            T* gp = out + (p * (int64_t)(L - 1) + r0) * row_elems;
            if (use_bulk) {
                fence_proxy_async_smem();
                __syncthreads();
                if (tid == 0) {
                    bulk_store(gp, ot, (uint32_t)((size_t)nr * row_elems * sizeof(T)));
                    bulk_commit();
                }
            } else {
                __syncthreads();
                for (int e = tid; e < nr * row_elems; e += kThreads) gp[e] = ot[e];
            }
        }
    }
    if (use_bulk && tid == 0) bulk_wait_read<0>();
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}

// Natural cubic spline, one WARP per path (fp32, channels % 4 == 0).  No CTA barrier after the
// prologue: a warp loads its path with 128-bit loads into its own shared-memory tile kept in
// the global [knot][channel] order, sweeps it with lane = (channel pair, chunk of G knots) --
// 64-bit shared loads feed the packed fp32x2 pipe directly -- and writes the coefficient rows
// with four 128-bit stores per (interval, 4 channels).  The back substitution overwrites the
// forward-sweep values in place (warm-up reads of the neighbouring chunk happen before a
// __syncwarp, the chunk's own stores after it), so a path needs two tiles, not three.
// Chunk c of a tile starts at word c * (G * C + padw) with padw chosen so that consecutive
// chunks start C banks apart: the sweeps' strided accesses are conflict free.  The per-knot
// constants are stored already duplicated for the packed pipe, at index i + i / G (one slot of
// padding per chunk, same reason).  ~2.2 K warp-instructions per path against ~10 K for the
// CTA-per-path kernel (whose chunks of 4 knots re-ran a 16-knot warm-up each).
static constexpr int kNatPrefetch = 16;     // 128-bit loads per lane kept in flight for the next path
static constexpr int kNatMaxWarps = 12;

__global__ void __launch_bounds__(32 * kNatMaxWarps)
natural_warp_kernel(const float* __restrict__ x, const float* __restrict__ ws, float* __restrict__ out,
                    int64_t n_paths, int L, int C, int lgG, int padw, int tile_words, int stage_words,
                    int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int G = 1 << lgG;
    const int nct = (L + G - 1) >> lgG;
    const int Lc = L + nct + 1;
    const int Lc2 = (Lc + 1) & ~1;
    float2* cA = reinterpret_cast<float2*>(smem_raw);          // [i + i/G] = (rdt2, mult)
    float2* cB = cA + Lc2;                                      // [i + i/G] = (rdt, rnd)
    float2* cC = cB + Lc2;                                      // [i] = (rdt, rdt2)
    float* tiles = reinterpret_cast<float*>(cC + ((L + 1) & ~1));
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const float rd = ws[i], rd2 = ws[L + i], m = ws[2 * L + i], rn = ws[3 * L + i];
        const int pi = i + (i >> lgG);
        cA[pi] = make_float2(rd2, m);
        cB[pi] = make_float2(rd, rn);
        cC[i] = make_float2(rd, rd2);
    }
    __syncthreads();
    const int wf = (int)ws[4 * L], wb = (int)ws[4 * L + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    float* xs = tiles + (size_t)warp * (2 * tile_words + stage_words);
    float* fk = xs + tile_words;
    float* stage = fk + tile_words;                     // stage_words: coefficient rows staged for a bulk store
    const int C2 = C >> 1, Q = C >> 2;
    const int n_items = C2 * nct;
    const int n_vec = L * Q;
    const int dq_i = 32 / Q, dq_q = 32 - dq_i * Q;
    const int row_step = C + padw;                     // from the last knot of a chunk to the first of the next
    const f2 three = pk2(3.f, 3.f), two = pk2(2.f, 2.f), four = pk2(4.f, 4.f);
    bool saw_nan = false;
    const int RR = stage_words / (4 * C);              // rows per bulk store
    int rl_pre[2], q_pre[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        rl_pre[u] = (lane + 32 * u) / Q;
        q_pre[u] = lane + 32 * u - rl_pre[u] * Q;
    }
    auto word = [&](int i) { return i * C + (i >> lgG) * padw; };

    // The next path's knots are requested before the current path is swept: the DRAM latency of a
    // warp's only global loads is covered by its own arithmetic, not by other warps.
    float4 pre[kNatPrefetch];
    auto request = [&](int64_t path) {
        const float4* xg4 = reinterpret_cast<const float4*>(x + path * (int64_t)L * C);
#pragma unroll
        for (int k = 0; k < kNatPrefetch; ++k)
            if (lane + 32 * k < n_vec) pre[k] = __ldg(xg4 + lane + 32 * k);
    };
    const int64_t stride = (int64_t)gridDim.x * n_warps;
    int64_t p = (int64_t)blockIdx.x * n_warps + warp;
    if (p < n_paths) request(p);

    for (; p < n_paths; p += stride) {
        __syncwarp();                                   // the previous path's coefficient phase has read xs / fk
        {
            int i = lane / Q, q = lane - (lane / Q) * Q;
#pragma unroll
            for (int k = 0; k < kNatPrefetch; ++k) {
                if (lane + 32 * k < n_vec) {
                    const float4 v = pre[k];
                    saw_nan |= is_nan(v.x) | is_nan(v.y) | is_nan(v.z) | is_nan(v.w);
                    *reinterpret_cast<float4*>(xs + word(i) + 4 * q) = v;
                }
                i += dq_i;
                q += dq_q;
                if (q >= Q) { q -= Q; ++i; }
            }
            const float4* xg4 = reinterpret_cast<const float4*>(x + p * (int64_t)L * C);
#pragma unroll 4
            for (int e = lane + 32 * kNatPrefetch; e < n_vec; e += 32) {       // longer paths: the rest, directly
                const float4 v = __ldg(xg4 + e);
                saw_nan |= is_nan(v.x) | is_nan(v.y) | is_nan(v.z) | is_nan(v.w);
                *reinterpret_cast<float4*>(xs + word(i) + 4 * q) = v;
                i += dq_i;
                q += dq_q;
                if (q >= Q) { q -= Q; ++i; }
            }
        }
        if (p + stride < n_paths) request(p + stride);
        __syncwarp();
        for (int base = 0; base < n_items; base += 32) {             // forward sweep (misc.py:58-61)
            const int it = base + lane;
            if (it >= n_items) continue;
            const int pr = it % C2, j = it / C2;
            const int g0 = j << lgG, g1 = min(g0 + G, L);
            int i = max(g0 - wf, 0);
            const float* px = xs + 2 * pr + word(i);               // x[i]; the forward value of knot i goes to
            const float2* pa = cA + i + (i >> lgG);                // px + tile_words
            f2 f = pk2(0.f, 0.f), sc_prev = pk2(0.f, 0.f);
            f2 x_lo = *reinterpret_cast<const f2*>(px);
            if (i > 0) {
                const float2 a = cA[i - 1 + ((i - 1) >> lgG)];
                const f2 x_before = *reinterpret_cast<const f2*>(xs + 2 * pr + word(i - 1));
                sc_prev = mul2(mul2(three, sub2(x_lo, x_before)), pk2(a.x, a.x));
            }
            // scaled difference 3 (x[i+1] - x[i]) / dt_i^2; rdt2[L-1] = 0 closes the system (cubic.py:36-39)
            auto knot = [&](const f2 x_hi, const float2 a, float* dst, bool keep) {
                const f2 sc = mul2(mul2(three, sub2(x_hi, x_lo)), pk2(a.x, a.x));
                x_lo = x_hi;
                f = sub2(add2(sc, sc_prev), mul2(pk2(a.y, a.y), f));
                sc_prev = sc;
                if (keep) *reinterpret_cast<f2*>(dst) = f;
            };
            while (i < g1) {                                         // chunk by chunk: warm-up chunks, then its own
                const int seg_end = min((i | (G - 1)) + 1, g1);
                const bool keep = i >= g0;
                int r = seg_end - 1 - i;
                for (; r >= 4; r -= 4) {                             // loads of four knots ahead of their stores
                    f2 xh[4];
                    float2 aa[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        xh[u] = *reinterpret_cast<const f2*>(px + (u + 1) * C);
                        aa[u] = pa[u];
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) knot(xh[u], aa[u], const_cast<float*>(px) + u * C + tile_words, keep);
                    px += 4 * C;
                    pa += 4;
                }
                for (; r > 0; --r) {
                    knot(*reinterpret_cast<const f2*>(px + C), *pa, const_cast<float*>(px) + tile_words, keep);
                    px += C;
                    ++pa;
                }
                const int step = (seg_end == L) ? 0 : row_step;      // the right neighbour of the last knot is itself
                knot(*reinterpret_cast<const f2*>(px + step), *pa, const_cast<float*>(px) + tile_words, keep);
                px += step;
                pa += 2;
                i = seg_end;
            }
        }
        __syncwarp();
        for (int base = 0; base < n_items; base += 32) {             // back substitution (misc.py:63-65), in place
            const int it = base + lane;
            const bool active = it < n_items;
            const int pr = active ? it % C2 : 0, j = active ? it / C2 : 0;
            const int g0 = j << lgG, g1 = min(g0 + G, L);
            int i = min(g1 - 1 + wb, L - 1);
            float* pf = fk + 2 * pr + word(i);
            const float2* pb = cB + i + (i >> lgG);
            f2 k = pk2(0.f, 0.f);
            if (active) {
                while (i >= g1) {                                    // warm-up in the chunks to the right: reads only
                    const int seg_lo = max(i & ~(G - 1), g1);        // g1 is a chunk boundary whenever this loop runs
                    for (; i > seg_lo; --i) {
                        const float2 b = *pb;
                        k = mul2(sub2(*reinterpret_cast<const f2*>(pf), mul2(pk2(b.x, b.x), k)), pk2(b.y, b.y));
                        pf -= C;
                        --pb;
                    }
                    const float2 b = *pb;
                    k = mul2(sub2(*reinterpret_cast<const f2*>(pf), mul2(pk2(b.x, b.x), k)), pk2(b.y, b.y));
                    pf -= row_step;
                    pb -= 2;
                    i = seg_lo - 1;
                }
            }
            __syncwarp();
            if (active) {
                for (; i >= g0 + 3; i -= 4) {                       // loads of four knots ahead of their stores
                    f2 fv[4];
                    float2 bb[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        fv[u] = *reinterpret_cast<const f2*>(pf - u * C);
                        bb[u] = *(pb - u);
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        k = mul2(sub2(fv[u], mul2(pk2(bb[u].x, bb[u].x), k)), pk2(bb[u].y, bb[u].y));
                        *reinterpret_cast<f2*>(pf - u * C) = k;
                    }
                    pf -= 4 * C;
                    pb -= 4;
                }
                for (; i >= g0; --i) {
                    const float2 b = *pb;
                    k = mul2(sub2(*reinterpret_cast<const f2*>(pf), mul2(pk2(b.x, b.x), k)), pk2(b.y, b.y));
                    *reinterpret_cast<f2*>(pf) = k;
                    pf -= C;
                    --pb;
                }
            }
        }
        __syncwarp();
        {
            // coefficient rows: RR whole rows per round (two items per lane, loads of both ahead of the math), staged
            // in shared memory exactly as they lie in global memory and written by one bulk (TMA) store of the warp's
            // elected lane.  Lane = (row, 4 channels); its four 16-byte blocks go to the staging row in an order
            // rotated by the row number, which spreads the lanes of one store instruction over the banks (rows are
            // 16 C bytes apart).  The staging buffer is reused once the previous bulk store has read it.
            float* og = out + p * (int64_t)(L - 1) * 4 * C;
            for (int r0 = 0; r0 < L - 1; r0 += RR) {
                const int n_it = min(RR, L - 1 - r0) * Q;
                for (int base = 0; base < n_it; base += 64) {
                    int rl[2], qq[2];
                    bool valid[2];
                    float4 xl[2], xh[2], kl[2], kh[2];
                    float2 rr[2];
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int it = base + lane + 32 * u;
                        rl[u] = base == 0 ? rl_pre[u] : it / Q;
                        qq[u] = base == 0 ? q_pre[u] : it - (it / Q) * Q;
                        valid[u] = it < n_it;
                        if (valid[u]) {
                            const int i = r0 + rl[u];
                            const int w0 = word(i) + 4 * qq[u], w1 = word(i + 1) + 4 * qq[u];
                            xl[u] = *reinterpret_cast<const float4*>(xs + w0);
                            xh[u] = *reinterpret_cast<const float4*>(xs + w1);
                            kl[u] = *reinterpret_cast<const float4*>(fk + w0);
                            kh[u] = *reinterpret_cast<const float4*>(fk + w1);
                            rr[u] = cC[i];
                        }
                    }
                    if (base == 0) {
                        if (lane == 0) bulk_wait_read<0>();
                        __syncwarp();
                    }
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        if (!valid[u]) continue;
                        const f2 rdp = pk2(rr[u].x, rr[u].x), rd2p = pk2(rr[u].y, rr[u].y);
                        float4 cv, dv;
                        {
                            const f2 l = pk2(kl[u].x, kl[u].y), h = pk2(kh[u].x, kh[u].y);
                            const f2 sr = mul2(mul2(two, mul2(three, sub2(pk2(xh[u].x, xh[u].y), pk2(xl[u].x, xl[u].y)))), rdp);
                            upk2(mul2(sub2(sub2(sr, mul2(four, l)), mul2(two, h)), rdp), cv.x, cv.y);   // cubic.py:45-47
                            upk2(mul2(sub2(mul2(three, add2(l, h)), sr), rd2p), dv.x, dv.y);             // cubic.py:48-50
                        }
                        {
                            const f2 l = pk2(kl[u].z, kl[u].w), h = pk2(kh[u].z, kh[u].w);
                            const f2 sr = mul2(mul2(two, mul2(three, sub2(pk2(xh[u].z, xh[u].w), pk2(xl[u].z, xl[u].w)))), rdp);
                            upk2(mul2(sub2(sub2(sr, mul2(four, l)), mul2(two, h)), rdp), cv.z, cv.w);
                            upk2(mul2(sub2(mul2(three, add2(l, h)), sr), rd2p), dv.z, dv.w);
                        }
                        // rotate (a, b, 2c, 3d) left by rl & 3: two conditional stages of register selects
                        const bool r1 = rl[u] & 1, r2 = rl[u] & 2;
                        const float4 v0 = r1 ? kl[u] : xl[u], v1 = r1 ? cv : kl[u], v2 = r1 ? dv : cv, v3 = r1 ? xl[u] : dv;
                        const float4 u0 = r2 ? v2 : v0, u1 = r2 ? v3 : v1, u2 = r2 ? v0 : v2, u3 = r2 ? v1 : v3;
                        float4* row = reinterpret_cast<float4*>(stage) + (size_t)rl[u] * (4 * Q) + qq[u];
                        const int b0 = rl[u] & 3;
                        row[b0 * Q] = u0;
                        row[((b0 + 1) & 3) * Q] = u1;
                        row[((b0 + 2) & 3) * Q] = u2;
                        row[((b0 + 3) & 3) * Q] = u3;
                    }
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    bulk_store(og + (size_t)r0 * 4 * C, stage, (uint32_t)(n_it * 64));     // an item is 4 x 16 bytes
                    bulk_commit();
                }
            }
        }
    }
    if (lane == 0) bulk_wait_read<0>();
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}

// One CTA per group of S paths.  Phase 1: coalesced load, transposed into shared memory as
// [series][knot] so that the thread that owns a series walks contiguous words.  Phase 2: one
// thread per series runs the forward sweep and the back substitution in shared memory.
// Phase 3: all threads turn (x, slope) into the [a|b|2c|3d] rows, staged per tile and written
// with bulk stores exactly like the Hermite kernel.
template <typename T>
__global__ void __launch_bounds__(kThreads)
natural_kernel(const T* __restrict__ x, const T* __restrict__ ws, T* __restrict__ out, int64_t n_paths, int L, int C,
               int S, int Lp, int TR, int use_bulk, int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    const int row_elems = 4 * C;
    const int path_stride = C * Lp + 1;
    T* ot0 = reinterpret_cast<T*>(smem_raw);
    T* ot1 = ot0 + (size_t)TR * row_elems;
    T* rdt = ot1 + (size_t)TR * row_elems;
    T* rdt2 = rdt + L;
    T* mult = rdt2 + L;
    T* rnd = mult + L;
    T* xs = rnd + L;
    T* ks = xs + (size_t)S * path_stride;

    const int tid = threadIdx.x;
    for (int e = tid; e < 4 * L; e += kThreads) rdt[e] = ws[e];
    bool saw_nan = false;
    int buf = 0;
    const int64_t n_groups = (n_paths + S - 1) / S;
    const int di = kThreads / C, dc = kThreads - di * C;

    for (int64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
        const int64_t p0 = grp * S;
        const int np = (int)min((int64_t)S, n_paths - p0);
        __syncthreads();   // previous group's phase 3 is done with xs / ks
        {
            const T* xg = x + p0 * L * C;
            int i = tid / C, c = tid - (tid / C) * C, p = 0;
            while (i >= L) { i -= L; ++p; }
            const int total = np * L * C;
            for (int e = tid; e < total; e += kThreads) {
                const T v = xg[e];
                saw_nan |= is_nan(v);
                xs[p * path_stride + c * Lp + i] = v;
                i += di;
                c += dc;
                if (c >= C) { c -= C; ++i; }
                while (i >= L) { i -= L; ++p; }
            }
        }
        __syncthreads();
        if (tid < np * C && L > 2) {
            const int p = tid / C, c = tid - p * C;
            const T* xr = xs + p * path_stride + c * Lp;
            T* kr = ks + p * path_stride + c * Lp;
            // forward sweep (misc.py:58-61); rhs[i] = scaled[i] + scaled[i-1] (cubic.py:36-39)
            T x_lo = xr[0], x_hi = xr[1];
            T scaled_prev = E::mul(E::mul(T(3), E::sub(x_hi, x_lo)), rdt2[0]);
            T f = scaled_prev;
            kr[0] = f;
            for (int i = 1; i < L; ++i) {
                T rhs;
                if (i < L - 1) {
                    x_lo = x_hi;
                    x_hi = xr[i + 1];
                    const T scaled = E::mul(E::mul(T(3), E::sub(x_hi, x_lo)), rdt2[i]);
                    rhs = E::add(scaled, scaled_prev);
                    scaled_prev = scaled;
                } else {
                    rhs = E::add(T(0), scaled_prev);
                }
                f = E::sub(rhs, E::mul(mult[i], f));
                kr[i] = f;
            }
            // back substitution (misc.py:63-65), dividing by nd as a multiplication by 1/nd
            T k = E::mul(f, rnd[L - 1]);
            kr[L - 1] = k;
            for (int i = L - 2; i >= 0; --i) {
                k = E::mul(E::sub(kr[i], E::mul(rdt[i], k)), rnd[i]);
                kr[i] = k;
            }
        }
        __syncthreads();
        // phase 3
        for (int p = 0; p < np; ++p) {
            for (int r0 = 0; r0 < L - 1; r0 += TR, buf ^= 1) {
                const int nr = min(TR, L - 1 - r0);
                if (use_bulk && tid == 0) bulk_wait_read<1>();
                __syncthreads();
                T* ot = buf ? ot1 : ot0;
                int i = tid / C, c = tid - (tid / C) * C;
                for (int e = tid; e < nr * C; e += kThreads) {
                    const int r = r0 + i;
                    const T* xr = xs + p * path_stride + c * Lp + r;
                    const T* kr = ks + p * path_stride + c * Lp + r;
                    const T xl = xr[0], xh = xr[1];
                    T b, two_c, three_d;
                    if (L == 2) {                       // cubic.py:16-20
                        b = E::div(E::sub(xh, xl), mult[0]);
                        two_c = T(0);
                        three_d = T(0);
                    } else {
                        const T kl = kr[0], kh = kr[1];
                        const T six = E::mul(T(2), E::mul(T(3), E::sub(xh, xl)));
                        const T sr = E::mul(six, rdt[r]);
                        b = kl;
                        two_c = E::mul(E::sub(E::sub(sr, E::mul(T(4), kl)), E::mul(T(2), kh)), rdt[r]);      // :45-47
                        three_d = E::mul(E::add(-sr, E::mul(T(3), E::add(kl, kh))), rdt2[r]);                // :48-50
                    }
                    T* row = ot + (size_t)i * row_elems + c;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int w = (k + i) & 3;
                        const T v = (w == 0) ? xl : (w == 1) ? b : (w == 2) ? two_c : three_d;
                        row[w * C] = v;
                    }
                    i += di;
                    c += dc;
                    if (c >= C) { c -= C; ++i; }
                }
                T* gp = out + ((p0 + p) * (int64_t)(L - 1) + r0) * row_elems;
                if (use_bulk) {
                    fence_proxy_async_smem();
                    __syncthreads();
                    if (tid == 0) {
                        bulk_store(gp, ot, (uint32_t)((size_t)nr * row_elems * sizeof(T)));
                        bulk_commit();
                    }
                } else {
                    __syncthreads();
                    for (int e = tid; e < nr * row_elems; e += kThreads) gp[e] = ot[e];
                }
            }
        }
    }
    if (use_bulk && tid == 0) bulk_wait_read<0>();
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}

// =========================================================================================
// Natural cubic spline with missing values, one thread per series  (cubic.py:56-167)
// =========================================================================================
// Irregular path: each series has its own set of observed knots, so the tridiagonal system
// differs per series.  scratch holds, per series, 3 rows of length L in a [row][knot][series]
// layout (coalesced across the warp): compacted rhs/solution, eliminated diagonal, and the
// knot slopes.  Exact arithmetic (the reference order) throughout.
template <typename T, bool UNIT>
__global__ void __launch_bounds__(128)
natural_missing_kernel(const T* __restrict__ x, const T* __restrict__ t, T* __restrict__ out, T* __restrict__ scratch,
                       int64_t n_series, int L, int C, int version) {
    using E = exact<T>;
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n_series) return;
    const int64_t p = g / C;
    const int c = (int)(g - p * C);
    const T* xs = x + p * L * C + c;
    T* os = out + p * (int64_t)(L - 1) * 4 * C + c;
    auto time_of = [&](int i) -> T { return UNIT ? T(i) : t[i]; };
    // scratch rows, element (row, j) of this series at scratch[(row * L + j) * n_series + g]
    auto S0 = [&](int j) -> T& { return scratch[((int64_t)0 * L + j) * n_series + g]; };   // rhs -> fwd -> slope
    auto S1 = [&](int j) -> T& { return scratch[((int64_t)1 * L + j) * n_series + g]; };   // eliminated diagonal
    auto S2 = [&](int j) -> T& { return scratch[((int64_t)2 * L + j) * n_series + g]; };   // compacted value
    auto S3 = [&](int j) -> T& { return scratch[((int64_t)3 * L + j) * n_series + g]; };   // compacted time

    // first / last observation
    int first = -1, last = -1;
    for (int i = 0; i < L; ++i) {
        if (!is_nan(xs[(int64_t)i * C])) {
            if (first < 0) first = i;
            last = i;
        }
    }
    const int rows = L - 1;
    if (first < 0) {                                             // cubic.py:85-92
        for (int i = 0; i < rows; ++i)
            for (int w = 0; w < 4; ++w) os[((int64_t)i * 4 + w) * C] = T(0);
        return;
    }
    const T vfirst = xs[(int64_t)first * C], vlast = xs[(int64_t)last * C];
    // compact the (imputed) observed knots: cubic.py:101-133
    int m = 0;
    for (int i = 0; i < L; ++i) {
        T v = xs[(int64_t)i * C];
        if (is_nan(v)) {
            if (version == 0) {
                if (i == 0) v = vfirst;
                else if (i == L - 1) v = vlast;
            } else {
                if (i < first) v = vfirst;
                else if (i > last) v = vlast;
            }
        }
        if (!is_nan(v)) {
            S2(m) = v;
            S3(m) = time_of(i);
            ++m;
        }
    }
    // m >= 2 always (both ends are observed after imputation)
    if (m > 2) {
        // system of cubic.py:23-39 on the compacted knots, Thomas solve of misc.py:52-65
        T rprev = E::div(T(1), E::sub(S3(1), S3(0)));
        T scaled_prev = E::mul(E::mul(T(3), E::sub(S2(1), S2(0))), E::mul(rprev, rprev));
        T nd = E::mul(T(2), rprev);
        T f = scaled_prev;
        S0(0) = f;
        S1(0) = nd;
        for (int j = 1; j < m; ++j) {
            T diag, rhs, rcur = T(0);
            if (j < m - 1) {
                rcur = E::div(T(1), E::sub(S3(j + 1), S3(j)));
                const T scaled = E::mul(E::mul(T(3), E::sub(S2(j + 1), S2(j))), E::mul(rcur, rcur));
                diag = E::mul(T(2), E::add(rcur, rprev));
                rhs = E::add(scaled, scaled_prev);
                scaled_prev = scaled;
            } else {
                diag = E::mul(T(2), E::add(T(0), rprev));
                rhs = E::add(T(0), scaled_prev);
            }
            const T w = E::div(rprev, nd);
            nd = E::sub(diag, E::mul(w, rprev));
            f = E::sub(rhs, E::mul(w, f));
            S0(j) = f;
            S1(j) = nd;
            rprev = rcur;
        }
        T k = E::div(f, nd);
        S0(m - 1) = k;
        for (int j = m - 2; j >= 0; --j) {
            const T up = E::div(T(1), E::sub(S3(j + 1), S3(j)));
            k = E::div(E::sub(S0(j), E::mul(up, k)), S1(j));
            S0(j) = k;
        }
    }
    // walk the original intervals; piece q spans compacted knots q, q+1   (cubic.py:147-162)
    int q = -1;
    T pa = T(0), pb = T(0), pc = T(0), pd = T(0), anchor = T(0);
    int next_obs = 0;   // index into compacted knots of the next observed time
    for (int i = 0; i < rows; ++i) {
        const T ti = time_of(i);
        if (next_obs < m && ti >= S3(next_obs)) {
            q = next_obs;
            ++next_obs;
            anchor = S3(q);
            const T xl = S2(q), xh = S2(q + 1);
            if (m == 2) {                                        // cubic.py:16-20
                pa = xl;
                pb = E::div(E::sub(xh, xl), E::sub(S3(1), S3(0)));
                pc = T(0);
                pd = T(0);
            } else {
                const T r = E::div(T(1), E::sub(S3(q + 1), S3(q)));
                const T r2 = E::mul(r, r);
                const T kl = S0(q), kh = S0(q + 1);
                const T six = E::mul(T(2), E::mul(T(3), E::sub(xh, xl)));
                const T sr = E::mul(six, r);
                pa = xl;
                pb = kl;
                pc = E::mul(E::sub(E::sub(sr, E::mul(T(4), kl)), E::mul(T(2), kh)), r);
                pd = E::mul(E::add(-sr, E::mul(T(3), E::add(kl, kh))), r2);
            }
        }
        const T off = E::sub(anchor, ti);
        const T inner = E::mul(E::sub(E::mul(T(0.5), pc), E::div(E::mul(pd, off), T(3))), off);
        os[((int64_t)i * 4 + 0) * C] = E::add(pa, E::mul(E::sub(inner, pb), off));
        os[((int64_t)i * 4 + 1) * C] = E::add(pb, E::mul(E::sub(E::mul(pd, off), pc), off));
        os[((int64_t)i * 4 + 2) * C] = E::sub(pc, E::mul(E::mul(T(2), pd), off));
        os[((int64_t)i * 4 + 3) * C] = pd;
    }
}


template <typename T>
static int launch_natural(const T* x, const T* t, T* out, T* ws, int64_t n_paths, int L, int C, int32_t* flags,
                          cudaStream_t stream) {
    natural_prep_kernel<T><<<1, 128, 0, stream>>>(t, ws, L);
    TCDE_CHECK_CUDA(cudaGetLastError());
    const size_t row_bytes = (size_t)4 * C * sizeof(T);
    int TR = (int)(8192 / row_bytes);
    if (TR < 1) TR = 1;
    if (TR > L - 1) TR = L - 1;
    if constexpr (sizeof(T) == 4) {
        // warp per path: fp32, 128-bit rows, two tiles per warp in shared memory
        if ((C & 3) == 0 && L > 2 && aligned16(out) && aligned16(x) && g_natural_variant == 0) {
            const int C2 = C / 2;
            const int n_chunks = C2 >= 32 ? 1 : 32 / C2;
            int lgG = 0;
            while ((1 << lgG) * n_chunks < L) ++lgG;
            const int G = 1 << lgG;
            const int nct = (L + G - 1) / G;
            const int padw = (int)((((int64_t)C - (int64_t)G * C) % 32 + 32) % 32);
            const int tile_words = L * C + nct * padw;
            const int rows_per_round = C / 4 >= 32 ? 2 : 64 / (C / 4);       // two (row, 4 channels) items per lane
            const int stage_words = rows_per_round * 4 * C;
            const size_t fixed = (size_t)2 * ((L + nct + 2) & ~1) * 8 + (size_t)((L + 1) & ~1) * 8;
            const size_t per_warp = (size_t)(2 * tile_words + stage_words) * 4;
            int wpc = fixed < 220 * 1024 ? (int)((220 * 1024 - fixed) / per_warp) : 0;
            if (wpc > kNatMaxWarps) wpc = kNatMaxWarps;
            if (wpc >= 2) {
                const size_t smem_k = fixed + wpc * per_warp;
                auto kw = natural_warp_kernel;
                TCDE_CHECK_CUDA(cudaFuncSetAttribute(kw, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k));
                int64_t grid = (n_paths + wpc - 1) / wpc;
                if (grid > sm_count()) grid = sm_count();
                kw<<<(int)grid, 32 * wpc, smem_k, stream>>>((const float*)x, (const float*)ws, (float*)out, n_paths, L, C,
                                                           lgG, padw, tile_words, stage_words, flags);
                TCDE_CHECK_CUDA(cudaGetLastError());
                return TCDE_OK;
            }
        }
    }
    {
        // parallel windowed sweeps: one path per CTA iteration, thread = (series, chunk of G knots)
        const int Lpw = ((L + 31) / 32) * 32 + 1;
        int G = (int)(((int64_t)L * C + kThreads - 1) / kThreads);
        if (G < 4) G = 4;
        // coefficient tiles: at least one (interval, 4-channel) item per thread and tile (a tile costs two
        // CTA barriers and a bulk store), at most 16 KB per staging buffer
        int TRw = TR;
        while (TRw < L - 1 && (size_t)TRw * (C / 4 > 0 ? C / 4 : 1) < (size_t)kThreads && (size_t)(2 * TRw) * row_bytes <= 16384) TRw *= 2;
        if (TRw > L - 1) TRw = L - 1;
        const bool direct = (sizeof(T) == 4) && ((C & 3) == 0) && L > 2 && aligned16(out) && aligned16(x);
        const int TR = direct ? 1 : TRw;      // the vectorised path stores rows straight to global memory
        const size_t smem_w = 2 * TR * row_bytes + (size_t)(4 * L + 8) * sizeof(T) + (size_t)3 * C * Lpw * sizeof(T) + 16;
        if (smem_w <= 64 * 1024 && g_natural_variant != 1) {
            auto kw = natural_win_kernel<T>;
            TCDE_CHECK_CUDA(cudaFuncSetAttribute(kw, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_w));
            const int grid = persistent_grid((const void*)kw, kThreads, smem_w, n_paths);
            kw<<<grid, kThreads, smem_w, stream>>>(x, ws, out, n_paths, L, C, Lpw, G, TR, aligned16(out) ? 1 : 0, flags);
            TCDE_CHECK_CUDA(cudaGetLastError());
            return TCDE_OK;
        }
    }
    int cp = 1;
    while (cp < C && cp < 32) cp <<= 1;
    const int Lp = ((L + 31) / 32) * 32 + 32 / cp;
    const size_t per_path = (size_t)2 * ((size_t)C * Lp + 1) * sizeof(T);
    const size_t fixed = 2 * TR * row_bytes + (size_t)4 * L * sizeof(T) + 16;
    int S = (32 + C - 1) / C;
    while (S > 1 && fixed + S * per_path > 100 * 1024) --S;
    const size_t smem = fixed + S * per_path;
    TCDE_CHECK_SUPPORTED(smem <= kMaxSmem,
                         "natural cubic: length=%d x channels=%d needs %zu bytes of shared memory (max %zu)", L, C,
                         smem, kMaxSmem);
    const int use_bulk = aligned16(out) ? 1 : 0;
    auto kern = natural_kernel<T>;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t n_groups = (n_paths + S - 1) / S;
    const int grid = persistent_grid((const void*)kern, kThreads, smem, n_groups);
    kern<<<grid, kThreads, smem, stream>>>(x, ws, out, n_paths, L, C, S, Lp, TR, use_bulk, flags);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}


}  // namespace tcde

using namespace tcde;

extern "C" int tcde_natural_cubic_coeffs(const void* x, const void* t, void* coeffs, void* workspace, int64_t n_paths,
                                         int64_t length, int64_t channels, int dtype, int32_t* flags, void* stream) {
    int rc = check_shape(x, coeffs, n_paths, length, channels, dtype);
    if (rc != TCDE_OK) return rc;
    TCDE_CHECK_ARG(workspace != nullptr, "null workspace");
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (dtype == TCDE_F32)
        return launch_natural<float>((const float*)x, (const float*)t, (float*)coeffs, (float*)workspace, n_paths,
                                     (int)length, (int)channels, flags, s);
    return launch_natural<double>((const double*)x, (const double*)t, (double*)coeffs, (double*)workspace, n_paths,
                                  (int)length, (int)channels, flags, s);
}

extern "C" int64_t tcde_natural_cubic_missing_scratch_bytes(int64_t n_paths, int64_t length, int64_t channels,
                                                            int dtype) {
    const int64_t elem = (dtype == TCDE_F64) ? 8 : 4;
    return 4 * length * n_paths * channels * elem;
}

extern "C" int tcde_natural_cubic_coeffs_missing(const void* x, const void* t, void* coeffs, void* scratch,
                                                 int64_t n_paths, int64_t length, int64_t channels, int version,
                                                 int dtype, void* stream) {
    int rc = check_shape(x, coeffs, n_paths, length, channels, dtype);
    if (rc != TCDE_OK) return rc;
    TCDE_CHECK_ARG(scratch != nullptr, "null scratch");
    TCDE_CHECK_ARG(version == 0 || version == 1, "version=%d", version);
    const int64_t n_series = n_paths * channels;
    if (n_series == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int threads = 128;
    const int64_t blocks = (n_series + threads - 1) / threads;
    TCDE_CHECK_SUPPORTED(blocks < (1ll << 31), "too many series");
    const int L = (int)length, C = (int)channels;
    if (dtype == TCDE_F32) {
        if (t) natural_missing_kernel<float, false><<<(unsigned)blocks, threads, 0, s>>>((const float*)x, (const float*)t, (float*)coeffs, (float*)scratch, n_series, L, C, version);
        else natural_missing_kernel<float, true><<<(unsigned)blocks, threads, 0, s>>>((const float*)x, nullptr, (float*)coeffs, (float*)scratch, n_series, L, C, version);
    } else {
        if (t) natural_missing_kernel<double, false><<<(unsigned)blocks, threads, 0, s>>>((const double*)x, (const double*)t, (double*)coeffs, (double*)scratch, n_series, L, C, version);
        else natural_missing_kernel<double, true><<<(unsigned)blocks, threads, 0, s>>>((const double*)x, nullptr, (double*)coeffs, (double*)scratch, n_series, L, C, version);
    }
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

