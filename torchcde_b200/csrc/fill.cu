// Hot path (i): batched spline-coefficient construction (sm_90a) -- gap fill, forward fill, rectilinear preparation, NaN flag.
//
// The builders are HBM-bound streaming kernels (SURVEY.md 8d: ~1 flop per byte).  The design rules
// that matter are the memory ones: coalesced 128-bit loads, results staged in shared memory and
// written back as contiguous 1-D bulk (TMA) stores, persistent CTAs sized from the SM count.
// Arithmetic uses tcde::exact<> (one rounding per operation, no FMA contraction) wherever the header
// promises bit-identical results.
#include "builders_common.cuh"

namespace tcde {

// =========================================================================================
// Per-series scans: linear gap fill, forward fill, rectilinear preparation
// =========================================================================================
// One thread per scalar series, walking the length dimension.  A warp covers 32/C paths x C
// channels, so every load/store instruction touches whole 32-byte sectors (C >= 8 floats) and
// the four sectors of a 128-byte line are consumed by four consecutive iterations (L1 hits).
// Loads do not depend on the scan state, so they are issued eight steps ahead.
template <typename T, bool UNIT>
__global__ void __launch_bounds__(kThreads)
linear_fill_kernel(const T* __restrict__ x, const T* __restrict__ t, T* __restrict__ out, int64_t n_series, int L,
                   int C) {
    using E = exact<T>;
    const int64_t g = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (g >= n_series) return;
    const int64_t p = g / C;
    const int c = (int)(g - p * C);
    const T* xs = x + p * L * C + c;
    T* os = out + p * L * C + c;

    auto time_of = [&](int i) -> T { return UNIT ? T(i) : t[i]; };
    // interpolation_linear.py:60-69: x[j] = lo + ((t_j - t_lo) / (t_hi - t_lo)) * (hi - lo)
    auto bridge = [&](int lo, T vlo, int hi, T vhi) {
        const T tl = time_of(lo);
        const T span = E::sub(time_of(hi), tl);
        const T rise = E::sub(vhi, vlo);
        for (int j = lo + 1; j < hi; ++j) {
            const T ratio = E::div(E::sub(time_of(j), tl), span);
            os[(int64_t)j * C] = E::add(vlo, E::mul(ratio, rise));
        }
    };

    int prev = -1;
    T vprev = T(0);
    for (int i0 = 0; i0 < L; i0 += 8) {
        T ahead[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) ahead[k] = (i0 + k < L) ? xs[(int64_t)(i0 + k) * C] : T(0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int i = i0 + k;
            if (i < L && !is_nan(ahead[k])) {
                const T v = ahead[k];
                if (prev < 0) {
                    if (i > 0) {            // :31-32 the first entry takes the first observation
                        os[0] = v;
                        bridge(0, v, i, v);
                    }
                } else if (i - prev > 1) {
                    bridge(prev, vprev, i, v);
                }
                os[(int64_t)i * C] = v;
                prev = i;
                vprev = v;
            }
        }
    }
    if (prev < 0) {                         // :19-21 nothing observed: the zero path
        for (int i = 0; i < L; ++i) os[(int64_t)i * C] = T(0);
    } else if (prev < L - 1) {              // :33-34 the last entry takes the last observation
        os[(int64_t)(L - 1) * C] = vprev;
        bridge(prev, vprev, L - 1, vprev);
    }
}

// Warp-per-path variant of the gap fill for length <= 32 * kFillRounds.  ncu on the
// thread-per-series kernel above: 70% of issue slots busy at 16% of HBM peak -- the data-dependent
// bridge loops diverge within a warp.  Here a warp stages its path in shared memory
// ([channel][position], conflict-free) and lane l owns positions l, l+32, ...; "nearest
// observation before / after" comes from warp ballots and bit scans (no loops, no divergence),
// every lane then applies the reference's interpolation formula once per element, and the
// filled tile is copied out with 128-bit coalesced stores.
constexpr int kFillRounds = 8;
template <typename T, bool UNIT>
__global__ void __launch_bounds__(kThreads)
linear_fill_warp_kernel(const T* __restrict__ x, const T* __restrict__ t, T* __restrict__ out, int64_t n_paths, int L,
                        int C, int Lp) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T* tile = reinterpret_cast<T*>(smem_raw) + (size_t)warp * C * Lp;
    const int rounds = (L + 31) >> 5;
    const int64_t warps_total = (int64_t)gridDim.x * (kThreads / 32);
    auto time_of = [&](int i) -> T { return UNIT ? T(i) : t[i]; };

    for (int64_t p = (int64_t)blockIdx.x * (kThreads / 32) + warp; p < n_paths; p += warps_total) {
        const T* xg = x + p * (int64_t)L * C;
        T* og = out + p * (int64_t)L * C;
        __syncwarp();
        const int di = 32 / C, dc = 32 - di * C;
        const bool vec4 = (sizeof(T) == 4) && ((C & 3) == 0) && (32 % (C >> 2) == 0) &&
                          ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
        if (vec4) {                                         // 128-bit coalesced loads, transposed to [c][i]
            const int Q = C >> 2, qi = 32 / Q;              // lane -> (row offset lane / Q, quad lane % Q)
            const int q = lane % Q;
            const float4* xg4 = reinterpret_cast<const float4*>(xg);
            for (int i = lane / Q; i < L; i += qi) {
                const float4 v4 = xg4[(size_t)i * Q + q];
                T* dst = tile + (4 * q) * Lp + i;
                dst[0] = (T)v4.x; dst[Lp] = (T)v4.y; dst[2 * Lp] = (T)v4.z; dst[3 * Lp] = (T)v4.w;
            }
        } else {
            int i = lane / C, c = lane - (lane / C) * C;
            for (int e = lane; e < L * C; e += 32) {        // coalesced load, transposed to [c][i]
                tile[c * Lp + i] = xg[e];
                i += di;
                c += dc;
                if (c >= C) { c -= C; ++i; }
            }
        }
        __syncwarp();
        for (int c = 0; c < C; ++c) {
            T* row = tile + c * Lp;
            T v[kFillRounds];
            uint32_t m[kFillRounds];
#pragma unroll
            for (int k = 0; k < kFillRounds; ++k) {
                const int i = 32 * k + lane;
                v[k] = (k < rounds && i < L) ? row[i] : T(0);
                m[k] = __ballot_sync(0xffffffffu, k < rounds && i < L && !is_nan(v[k]));
            }
            // first / last observation of the series, and per round the nearest ones outside it
            int first = L, last = -1;
#pragma unroll
            for (int k = 0; k < kFillRounds; ++k) {
                if (m[k]) {
                    if (first == L) first = 32 * k + __ffs(m[k]) - 1;
                    last = 32 * k + 31 - __clz(m[k]);
                }
            }
            if (first == L) {                               // nothing observed: the zero path
#pragma unroll
                for (int k = 0; k < kFillRounds; ++k)
                    if (k < rounds && 32 * k + lane < L) row[32 * k + lane] = T(0);
                continue;
            }
            const T v_first = row[first], v_last = row[last];
            __syncwarp();
            // first observation in any LATER round, per round (one backward pass instead of a search per round)
            int later_first[kFillRounds];
            {
                int carry = L;
#pragma unroll
                for (int k = kFillRounds - 1; k >= 0; --k) {
                    later_first[k] = carry;
                    if (m[k]) carry = 32 * k + __ffs(m[k]) - 1;
                }
            }
            int carry_prev = -1;
            const uint32_t le_mask = 0xffffffffu >> (31 - lane);
#pragma unroll
            for (int k = 0; k < kFillRounds; ++k) {
                const int i = 32 * k + lane;
                const bool hole = (k < rounds) && (i < L) && is_nan(v[k]);
                if (__any_sync(0xffffffffu, hole)) {        // whole rounds without a gap are skipped (warp-uniform)
                    const uint32_t below = m[k] & le_mask;
                    const int prv = below ? 32 * k + 31 - __clz(below) : carry_prev;
                    const uint32_t above = m[k] >> lane;
                    const int nxt = above ? i + __ffs(above) - 1 : later_first[k];
                    if (hole) {
                        int lo_i, hi_i;
                        T lo_v, hi_v;
                        if (prv < 0) {                      // before the first observation
                            lo_i = 0; hi_i = first; lo_v = v_first; hi_v = v_first;
                        } else if (nxt >= L) {              // after the last observation
                            lo_i = last; hi_i = L - 1; lo_v = v_last; hi_v = v_last;
                        } else {
                            lo_i = prv; hi_i = nxt; lo_v = row[prv]; hi_v = row[nxt];
                        }
                        T filled;
                        if (i == lo_i) filled = lo_v;       // an imputed end point itself
                        else if (i == hi_i) filled = hi_v;
                        else {
                            const T tl = time_of(lo_i);
                            const T ratio = E::div(E::sub(time_of(i), tl), E::sub(time_of(hi_i), tl));
                            filled = E::add(lo_v, E::mul(ratio, E::sub(hi_v, lo_v)));
                        }
                        v[k] = filled;
                    }
                }
                if (m[k]) carry_prev = 32 * k + 31 - __clz(m[k]);
            }
            __syncwarp();                                   // every gather from row[] is done
#pragma unroll
            for (int k = 0; k < kFillRounds; ++k)
                if (k < rounds && 32 * k + lane < L) row[32 * k + lane] = v[k];
        }
        __syncwarp();
        if (vec4) {
            const int Q = C >> 2, qi = 32 / Q;
            const int q = lane % Q;
            float4* og4 = reinterpret_cast<float4*>(og);
            for (int i = lane / Q; i < L; i += qi) {
                const T* src = tile + (4 * q) * Lp + i;
                og4[(size_t)i * Q + q] = make_float4((float)src[0], (float)src[Lp], (float)src[2 * Lp], (float)src[3 * Lp]);
            }
        } else {
            int i = lane / C, c = lane - (lane / C) * C;
            for (int e = lane; e < L * C; e += 32) {
                og[e] = tile[c * Lp + i];
                i += di;
                c += dc;
                if (c >= C) { c -= C; ++i; }
            }
        }
    }
}

// Scan variant of the gap fill: lane = (channel, chunk of G consecutive positions) of one path, for
// channels <= 32.  ncu on the ballot kernel above: 115 warp-instructions per 32 elements, issue
// bound at 19% of HBM peak.  Here the warp's tile stays in the global [position][channel] order
// (128-bit loads and stores on both sides, chunks padded so that the 32 lanes hit 32 banks) and
// every lane walks its chunk backward once: each hole is overwritten with a NaN whose payload holds
// the distances to the next observation and to the next hole of the chunk, which threads the holes
// into a list.  A few shuffles hand every chunk the nearest observation of the chunks before and
// after it.  Then the lane hops along its list of holes only (30% of the positions in the
// benchmark) and replaces each by the reference's interpolation formula; the end points of a gap
// are fetched once per gap.
template <typename T> struct nan_code;
template <> struct nan_code<float> {
    static constexpr uint32_t quiet = 0x7FC00000u;
    __device__ static int get(float v) { return (int)(__float_as_uint(v) & 0x3FFFFFu); }
    __device__ static float make(int i) { return __uint_as_float(quiet | (uint32_t)i); }
};
template <> struct nan_code<double> {
    static constexpr unsigned long long quiet = 0x7FF8000000000000ull;
    __device__ static int get(double v) { return (int)((unsigned long long)__double_as_longlong(v) & 0x3FFFFFull); }
    __device__ static double make(int i) { return __longlong_as_double((long long)(quiet | (unsigned long long)i)); }
};
constexpr int kFillNone = 0x3FFFFF;          // no observation
constexpr int kFillDist = 11;                // payload = distance to next observation | distance to next hole << 11

// The in-place gap fill of ONE path held in a warp's shared-memory tile ([position][channel] order, chunk padding
// ``padw``): shared by the stand-alone fill kernel and by the fused series -> Hermite kernel below.  Returns whether
// this lane's chunk held a hole.  Must be called by the whole warp (shuffles); the caller separates it from the loads
// and from the readers of the tile with __syncwarp().
template <typename T, bool UNIT>
__device__ __forceinline__ bool fill_tile_in_place(T* tile, const T* ts, int L, int C, int lgG,
                                                   int padw, int lane) {
    using E = exact<T>;
    const int G = 1 << lgG;
    const int nch = (L + G - 1) >> lgG;                     // chunks in use (<= 32 / C)
    const int c = lane % C, j = lane / C;
    const bool active = j < nch;
    const int g0 = j << lgG, g1 = min(g0 + G, L);
    const unsigned full = 0xffffffffu;
    auto word = [&](int i) { return i * C + (i >> lgG) * padw; };
    auto time_of = [&](int i) -> T { return UNIT ? T(i) : ts[i]; };
    // backward: thread the holes (payload: distance to the next observation / next hole of the chunk, 0 = none)
    int first_idx = kFillNone, last_idx = -1, head = -1;
    T last_val = T(0);
    if (active) {
        T* ptr = tile + word(g1 - 1) + c;
        for (int i = g1 - 1; i >= g0; --i, ptr -= C) {
            const T w = *ptr;
            if (is_nan(w)) {
                const int d_obs = first_idx == kFillNone ? 0 : first_idx - i;
                const int d_hole = head < 0 ? 0 : head - i;
                *ptr = nan_code<T>::make(d_obs | (d_hole << kFillDist));
                head = i;
            } else {
                if (last_idx < 0) { last_idx = i; last_val = w; }
                first_idx = i;
            }
        }
    }
    // nearest observation in the chunks after (position) and before (position, value) this one
    int after = kFillNone, before = -1;
    T before_val = T(0);
    for (int d = 1; d < nch; ++d) {
        const int fa = __shfl_down_sync(full, first_idx, C * d);
        const int la = __shfl_up_sync(full, last_idx, C * d);
        const T lv = __shfl_up_sync(full, last_val, C * d);
        if (after == kFillNone && j + d < nch) after = fa;
        if (before < 0 && j - d >= 0) { before = la; before_val = lv; }
    }
    const int series_first = __shfl_sync(full, first_idx != kFillNone ? first_idx : after, c);
    const int series_last = __shfl_sync(full, last_idx >= 0 ? last_idx : before, c + C * (nch - 1));
    if (active) {
        if (series_first == kFillNone) {                // nothing observed: the zero path (linear.py:19-21)
            T* ptr = tile + word(g0) + c;
            for (int i = g0; i < g1; ++i, ptr += C) *ptr = T(0);
        } else {
            const T v_first = tile[word(series_first) + c], v_last = tile[word(series_last) + c];
            // the ends of the series count as observations carrying the first / last value (linear.py:31-34)
            int prev_idx = before >= 0 ? before : 0;
            T prev_val = before >= 0 ? before_val : v_first;
            const int far_idx = after != kFillNone ? after : L - 1;
            const T far_val = after != kFillNone ? tile[word(after) + c] : v_last;
            T* base = tile + word(g0) + c;              // a chunk has no padding inside
            T lo_t = T(0), span = T(1), rise = T(0);
            for (int i = head, visited = -2; i >= 0;) {
                T* ptr = base + (i - g0) * C;
                const int code = nan_code<T>::get(*ptr);
                const int d_obs = code & ((1 << kFillDist) - 1), d_hole = code >> kFillDist;
                if (i != visited + 1) {                 // a new gap: fetch its end points
                    if (i > g0) {
                        prev_idx = i - 1;
                        prev_val = ptr[-C];
                    }
                    const int hi_i = d_obs ? i + d_obs : far_idx;
                    const T hi_v = d_obs ? ptr[d_obs * C] : far_val;
                    lo_t = time_of(prev_idx);
                    span = E::sub(time_of(hi_i), lo_t);
                    rise = E::sub(hi_v, prev_val);
                }
                // linear.py:60-69: x[j] = lo + ((t_j - t_lo) / (t_hi - t_lo)) * (hi - lo)
                *ptr = E::add(prev_val, E::mul(E::div(E::sub(time_of(i), lo_t), span), rise));
                visited = i;
                i = d_hole ? i + d_hole : -1;
            }
            // an imputed end point is a copy of the observation, not an interpolation
            if (g0 == 0 && series_first > 0) tile[c] = v_first;
            if (g1 == L && series_last < L - 1) tile[word(L - 1) + c] = v_last;
        }
    }
    return head >= 0;
}

// OUT = 0: the filled series (linear_interpolation_coeffs).  OUT = 1: the Hermite coefficients with backward
// differences of the filled series (interpolation_hermite_cubic_bdiff.py:23-44 = fill, then :8-20) straight from the
// warp's tile -- one launch, the filled series never goes to HBM, and no NaN flag has to travel to the host to decide
// whether a fill is needed: a path without holes skips the fill (one vote per path after the loads).
template <typename T, bool UNIT, int OUT>
__global__ void __launch_bounds__(kThreads)
linear_fill_scan_kernel(const T* __restrict__ x, const T* __restrict__ t, T* __restrict__ out, int64_t n_paths, int L,
                        int C, int lgG, int padw, int tile_words, int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    T* ts = reinterpret_cast<T*>(smem_raw);                 // knot times (absent for unit knots)
    T* tiles = ts + (UNIT ? 0 : ((L + 3) & ~3));
    if (!UNIT) {
        for (int i = threadIdx.x; i < L; i += blockDim.x) ts[i] = t[i];
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T* tile = tiles + (size_t)warp * tile_words;
    const unsigned full = 0xffffffffu;
    auto word = [&](int i) { return i * C + (i >> lgG) * padw; };
    const bool vec4 = (sizeof(T) == 4) && ((C & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const int Q = C >> 2;
    const int64_t warps_total = (int64_t)gridDim.x * (kThreads / 32);
    bool saw_nan = false;

    for (int64_t p = (int64_t)blockIdx.x * (kThreads / 32) + warp; p < n_paths; p += warps_total) {
        const T* xg = x + p * (int64_t)L * C;
        __syncwarp();                                       // the previous path has been copied out
        bool hole = false;
        if (vec4) {
            const float4* xg4 = reinterpret_cast<const float4*>(xg);
            const int dq_i = 32 / Q, dq_q = 32 - dq_i * Q;
            int i = lane / Q, q = lane - (lane / Q) * Q;
#pragma unroll 8
            for (int e = lane; e < L * Q; e += 32) {
                const float4 v = __ldg(xg4 + e);
                hole |= is_nan(v.x) | is_nan(v.y) | is_nan(v.z) | is_nan(v.w);
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(tile) + word(i) + 4 * q) = v;
                i += dq_i;
                q += dq_q;
                if (q >= Q) { q -= Q; ++i; }
            }
        } else {
            const int di = 32 / C, dc = 32 - di * C;
            int i = lane / C, cc = lane - (lane / C) * C;
#pragma unroll 4
            for (int e = lane; e < L * C; e += 32) {
                const T v = xg[e];
                hole |= is_nan(v);
                tile[word(i) + cc] = v;
                i += di;
                cc += dc;
                if (cc >= C) { cc -= C; ++i; }
            }
        }
        __syncwarp();
        if (__any_sync(full, hole)) {
            saw_nan = true;
            fill_tile_in_place<T, UNIT>(tile, ts, L, C, lgG, padw, lane);
            __syncwarp();
        }
        if (OUT == 0) {
            T* og = out + p * (int64_t)L * C;
            if (vec4) {
                float4* og4 = reinterpret_cast<float4*>(og);
                const int dq_i = 32 / Q, dq_q = 32 - dq_i * Q;
                int i = lane / Q, q = lane - (lane / Q) * Q;
#pragma unroll 8
                for (int e = lane; e < L * Q; e += 32) {
                    og4[e] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(tile) + word(i) + 4 * q);
                    i += dq_i;
                    q += dq_q;
                    if (q >= Q) { q -= Q; ++i; }
                }
            } else {
                const int di = 32 / C, dc = 32 - di * C;
                int i = lane / C, cc = lane - (lane / C) * C;
#pragma unroll 4
                for (int e = lane; e < L * C; e += 32) {
                    og[e] = tile[word(i) + cc];
                    i += di;
                    cc += dc;
                    if (cc >= C) { cc -= C; ++i; }
                }
            }
        } else {
            // interval r of channel c: (a, b, 2c, 3d) from the knots r-1, r, r+1 (operation order of bdiff.py:8-20, :36-43)
            T* og = out + p * (int64_t)(L - 1) * 4 * C;
            if (vec4) {
                float4* og4 = reinterpret_cast<float4*>(og);
                const float* tf = reinterpret_cast<const float*>(tile);
                const float* tsf = reinterpret_cast<const float*>(ts);
                const int dq_i = 32 / Q, dq_q = 32 - dq_i * Q;
                int r = lane / Q, q = lane - (lane / Q) * Q;
#pragma unroll 2
                for (int e = lane; e < (L - 1) * Q; e += 32) {
                    const float4 lo = *reinterpret_cast<const float4*>(tf + word(r) + 4 * q);
                    const float4 hi = *reinterpret_cast<const float4*>(tf + word(r + 1) + 4 * q);
                    const float4 pp = (r > 0) ? *reinterpret_cast<const float4*>(tf + word(r - 1) + 4 * q) : lo;
                    const float xl[4] = {lo.x, lo.y, lo.z, lo.w}, xh[4] = {hi.x, hi.y, hi.z, hi.w};
                    const float xq[4] = {pp.x, pp.y, pp.z, pp.w};
                    float b[4], c2[4], d3[4];
                    float dt = 1.f, dtp = 1.f, inv_sq = 1.f;
                    if (!UNIT) {
                        dt = exact<float>::sub(tsf[r + 1], tsf[r]);
                        dtp = (r > 0) ? exact<float>::sub(tsf[r], tsf[r - 1]) : dt;
                        inv_sq = exact<float>::div(1.f, exact<float>::mul(dt, dt));
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        using F = exact<float>;
                        if (UNIT) {
                            const float dn = F::sub(xh[k], xl[k]);
                            const float dp = (r > 0) ? F::sub(xl[k], xq[k]) : dn;
                            const float bend = F::sub(dn, dp);
                            c2[k] = F::mul(2.f, F::add(F::sub(F::mul(3.f, bend), dn), dp));
                            d3[k] = F::sub(bend, c2[k]);
                            b[k] = dp;
                        } else {
                            const float dn = F::div(F::sub(xh[k], xl[k]), dt);
                            const float dp = (r > 0) ? F::div(F::sub(xl[k], xq[k]), dtp) : dn;
                            const float inner = F::add(F::sub(F::mul(3.f, F::sub(dn, dp)), dn), dp);
                            c2[k] = F::div(F::mul(2.f, inner), dt);
                            d3[k] = F::sub(F::mul(inv_sq, F::sub(dn, dp)), F::div(c2[k], dt));
                            b[k] = dp;
                        }
                    }
                    float4* row = og4 + (size_t)r * 4 * Q + q;
                    __stcs(row, lo);
                    __stcs(row + Q, make_float4(b[0], b[1], b[2], b[3]));
                    __stcs(row + 2 * Q, make_float4(c2[0], c2[1], c2[2], c2[3]));
                    __stcs(row + 3 * Q, make_float4(d3[0], d3[1], d3[2], d3[3]));
                    r += dq_i;
                    q += dq_q;
                    if (q >= Q) { q -= Q; ++r; }
                }
            } else {
                const int di = 32 / C, dc = 32 - di * C;
                int r = lane / C, cc = lane - (lane / C) * C;
                for (int e = lane; e < (L - 1) * C; e += 32) {
                    const T xl = tile[word(r) + cc], xh = tile[word(r + 1) + cc];
                    T b, two_c, three_d;
                    if (UNIT) {
                        const T dn = E::sub(xh, xl);
                        const T dp = (r > 0) ? E::sub(xl, tile[word(r - 1) + cc]) : dn;
                        const T bend = E::sub(dn, dp);
                        two_c = E::mul(T(2), E::add(E::sub(E::mul(T(3), bend), dn), dp));
                        three_d = E::sub(bend, two_c);
                        b = dp;
                    } else {
                        const T dt = E::sub(ts[r + 1], ts[r]);
                        const T dn = E::div(E::sub(xh, xl), dt);
                        const T dp = (r > 0) ? E::div(E::sub(xl, tile[word(r - 1) + cc]), E::sub(ts[r], ts[r - 1])) : dn;
                        const T inner = E::add(E::sub(E::mul(T(3), E::sub(dn, dp)), dn), dp);
                        two_c = E::div(E::mul(T(2), inner), dt);
                        const T inv_sq = E::div(T(1), E::mul(dt, dt));
                        three_d = E::sub(E::mul(inv_sq, E::sub(dn, dp)), E::div(two_c, dt));
                        b = dp;
                    }
                    T* row = og + (size_t)r * 4 * C + cc;
                    row[0] = xl;
                    row[C] = b;
                    row[2 * C] = two_c;
                    row[3 * C] = three_d;
                    r += di;
                    cc += dc;
                    if (cc >= C) { cc -= C; ++r; }
                }
            }
        }
    }
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}

// misc.forward_fill (misc.py:103-126) and _prepare_rectilinear_interpolation
// (interpolation_linear.py:87-128).  RECT = false: out has L rows; RECT = true: 2L-1 rows, row
// 2i = held[i], row 2i+1 = held[i] except the time channel which takes held[i+1].
template <typename T, bool RECT>
__global__ void __launch_bounds__(kThreads)
hold_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t n_series, int L, int C, int time_index,
            int32_t* __restrict__ flags) {
    const int64_t g = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (g >= n_series) return;
    const int64_t p = g / C;
    const int c = (int)(g - p * C);
    const T* xs = x + p * L * C + c;
    const int out_rows = RECT ? 2 * L - 1 : L;
    T* os = out + p * out_rows * C + c;
    const bool is_time = RECT && (c == time_index);
    int32_t seen = 0;
    T held = xs[0];
    if (is_nan(held)) seen |= TCDE_FLAG_NAN_SEEN | TCDE_FLAG_NAN_FIRST_ROW | (is_time ? TCDE_FLAG_NAN_TIME : 0);
    for (int i0 = 0; i0 < L; i0 += 8) {
        T ahead[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) ahead[k] = (i0 + k < L) ? xs[(int64_t)(i0 + k) * C] : T(0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int i = i0 + k;
            if (i < L) {
                const T v = ahead[k];
                const T before = held;
                if (!is_nan(v)) held = v;
                else seen |= TCDE_FLAG_NAN_SEEN | (is_time ? TCDE_FLAG_NAN_TIME : 0);
                if (RECT) {
                    if (i > 0) os[(int64_t)(2 * i - 1) * C] = is_time ? held : before;
                    os[(int64_t)(2 * i) * C] = held;
                } else {
                    os[(int64_t)i * C] = held;
                }
            }
        }
    }
    if (seen && flags != nullptr) atomicOr(flags, seen);
}


// torch.isnan(x).any() of interpolation_linear.py:169 as one pass that only sets a flag.
template <typename T>
__global__ void __launch_bounds__(kThreads)
nan_flag_kernel(const T* __restrict__ x, int64_t n, int32_t* __restrict__ flags) {
    bool seen = false;
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += stride) seen |= is_nan(x[i]);
    if (__syncthreads_or(seen) && threadIdx.x == 0) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}


int g_fill_variant = 0;
int g_natural_variant = 0;

// Launch of the scan kernel (OUT = 0 filled series, 1 Hermite coefficients); TCDE_ERR_UNSUPPORTED (without setting an error
// message) when the shape does not fit a warp's shared-memory tile.
static int launch_fill_scan(const void* x, const void* t, void* out, int64_t n_paths, int L, int C, int dtype,
                            int32_t* flags, cudaStream_t s, int what) {
    if (!(C <= 32 && L < kFillNone)) return TCDE_ERR_UNSUPPORTED;
    // lane = (channel, chunk of positions), tile in the global layout
    const size_t elem = (dtype == TCDE_F32) ? 4 : 8;
    const int n_chunks = 32 / C;
    int lgG = 0;
    while ((1 << lgG) * n_chunks < L) ++lgG;
    const int G = 1 << lgG;
    const int nct = (L + G - 1) / G;
    const int bank_words = (int)(128 / elem);
    const int padw = (int)((((int64_t)C - (int64_t)G * C) % bank_words + bank_words) % bank_words);
    const int tile_words = (L * C + nct * padw + 3) & ~3;
    const size_t smem = (t ? (size_t)((L + 3) & ~3) * elem : 0) + (size_t)(kThreads / 32) * tile_words * elem;
    if (!(smem <= 100 * 1024 && lgG < kFillDist)) return TCDE_ERR_UNSUPPORTED;   // hole-list distances are 11-bit
    const void* kern;
    if (what == 0)
        kern = (dtype == TCDE_F32)
            ? (t ? (const void*)linear_fill_scan_kernel<float, false, 0> : (const void*)linear_fill_scan_kernel<float, true, 0>)
            : (t ? (const void*)linear_fill_scan_kernel<double, false, 0> : (const void*)linear_fill_scan_kernel<double, true, 0>);
    else
        kern = (dtype == TCDE_F32)
            ? (t ? (const void*)linear_fill_scan_kernel<float, false, 1> : (const void*)linear_fill_scan_kernel<float, true, 1>)
            : (t ? (const void*)linear_fill_scan_kernel<double, false, 1> : (const void*)linear_fill_scan_kernel<double, true, 1>);
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = persistent_grid(kern, kThreads, smem, (n_paths + kThreads / 32 - 1) / (kThreads / 32));
    const int Li = L, Ci = C;
    void* args[] = {(void*)&x, (void*)&t, (void*)&out, (void*)&n_paths, (void*)&Li, (void*)&Ci, (void*)&lgG,
                    (void*)&padw, (void*)&tile_words, (void*)&flags};
    TCDE_CHECK_CUDA(cudaLaunchKernel(kern, dim3(grid), dim3(kThreads), args, smem, s));
    return TCDE_OK;
}


}  // namespace tcde

using namespace tcde;

extern "C" int tcde_hermite_bdiff_coeffs_series(const void* x, const void* t, void* coeffs, int64_t n_paths, int64_t length,
                                                int64_t channels, int dtype, int32_t* flags, void* stream) {
    int rc = check_shape(x, coeffs, n_paths, length, channels, dtype);
    if (rc != TCDE_OK) return rc;
    if (n_paths == 0) return TCDE_OK;
    rc = launch_fill_scan(x, t, coeffs, n_paths, (int)length, (int)channels, dtype, flags, static_cast<cudaStream_t>(stream), 1);
    TCDE_CHECK_SUPPORTED(rc != TCDE_ERR_UNSUPPORTED,
                         "fused fill + Hermite: a path of length=%lld x channels=%lld does not fit a warp's shared-memory tile "
                         "(run tcde_linear_fill, then tcde_hermite_bdiff_coeffs)", (long long)length, (long long)channels);
    return rc;
}

extern "C" int tcde_linear_fill(const void* x, const void* t, void* out, int64_t n_paths, int64_t length,
                                int64_t channels, int dtype, int32_t* flags, void* stream) {
    int rc = check_shape(x, out, n_paths, length, channels, dtype);
    if (rc != TCDE_OK) return rc;
    const int64_t n_series = n_paths * channels;
    if (n_series == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int L = (int)length, C = (int)channels;
    if (g_fill_variant == 0) {
        rc = launch_fill_scan(x, t, out, n_paths, L, C, dtype, flags, s, 0);
        if (rc != TCDE_ERR_UNSUPPORTED) return rc;
    }
    if (flags != nullptr) {               // the other kernels do not report: a separate pass over x
        rc = tcde_nan_flag(x, n_series * L, dtype, flags, stream);
        if (rc != TCDE_OK) return rc;
    }
    {
        // warp-per-path kernel when a path fits a warp's shared-memory tile
        const int Lp = ((L + 31) / 32) * 32 + 1;
        const size_t elem = (dtype == TCDE_F32) ? 4 : 8;
        const size_t smem = (size_t)(kThreads / 32) * C * Lp * elem;
        if (L <= 32 * kFillRounds && smem <= 72 * 1024 && g_fill_variant != 1) {
            const void* kern = (dtype == TCDE_F32)
                ? (t ? (const void*)linear_fill_warp_kernel<float, false> : (const void*)linear_fill_warp_kernel<float, true>)
                : (t ? (const void*)linear_fill_warp_kernel<double, false> : (const void*)linear_fill_warp_kernel<double, true>);
            TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const int grid = persistent_grid(kern, kThreads, smem, (n_paths + kThreads / 32 - 1) / (kThreads / 32));
            const int Li = L, Ci = C, Lpi = Lp;
            void* args[] = {(void*)&x, (void*)&t, (void*)&out, (void*)&n_paths, (void*)&Li, (void*)&Ci, (void*)&Lpi};
            TCDE_CHECK_CUDA(cudaLaunchKernel(kern, dim3(grid), dim3(kThreads), args, smem, s));
            return TCDE_OK;
        }
    }
    const int64_t blocks = (n_series + kThreads - 1) / kThreads;
    TCDE_CHECK_SUPPORTED(blocks < (1ll << 31), "too many series");
    if (dtype == TCDE_F32) {
        if (t) linear_fill_kernel<float, false><<<(unsigned)blocks, kThreads, 0, s>>>((const float*)x, (const float*)t, (float*)out, n_series, L, C);
        else linear_fill_kernel<float, true><<<(unsigned)blocks, kThreads, 0, s>>>((const float*)x, nullptr, (float*)out, n_series, L, C);
    } else {
        if (t) linear_fill_kernel<double, false><<<(unsigned)blocks, kThreads, 0, s>>>((const double*)x, (const double*)t, (double*)out, n_series, L, C);
        else linear_fill_kernel<double, true><<<(unsigned)blocks, kThreads, 0, s>>>((const double*)x, nullptr, (double*)out, n_series, L, C);
    }
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

template <bool RECT>
static int launch_hold(const void* x, void* out, int64_t n_paths, int64_t length, int64_t channels, int64_t time_index,
                       int dtype, int32_t* flags, void* stream) {
    int rc = check_shape(x, out, n_paths, length, channels, dtype, RECT ? 2 : 1);
    if (rc != TCDE_OK) return rc;
    if (RECT) TCDE_CHECK_ARG(time_index >= 0 && time_index < channels, "time_index=%lld", (long long)time_index);
    const int64_t n_series = n_paths * channels;
    if (n_series == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int64_t blocks = (n_series + kThreads - 1) / kThreads;
    TCDE_CHECK_SUPPORTED(blocks < (1ll << 31), "too many series");
    if (dtype == TCDE_F32)
        hold_kernel<float, RECT><<<(unsigned)blocks, kThreads, 0, s>>>((const float*)x, (float*)out, n_series, (int)length, (int)channels, (int)time_index, flags);
    else
        hold_kernel<double, RECT><<<(unsigned)blocks, kThreads, 0, s>>>((const double*)x, (double*)out, n_series, (int)length, (int)channels, (int)time_index, flags);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

extern "C" int tcde_forward_fill(const void* x, void* out, int64_t n_paths, int64_t length, int64_t channels,
                                 int dtype, int32_t* flags, void* stream) {
    return launch_hold<false>(x, out, n_paths, length, channels, 0, dtype, flags, stream);
}

extern "C" int tcde_rectilinear_prepare(const void* x, void* out, int64_t n_paths, int64_t length, int64_t channels,
                                        int64_t time_index, int dtype, int32_t* flags, void* stream) {
    return launch_hold<true>(x, out, n_paths, length, channels, time_index, dtype, flags, stream);
}


extern "C" int tcde_nan_flag(const void* x, int64_t n, int dtype, int32_t* flags, void* stream) {
    TCDE_CHECK_ARG(x != nullptr && flags != nullptr && n >= 0, "null pointer or negative size");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    if (n == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int64_t blocks = (n + kThreads * 8 - 1) / (kThreads * 8);
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    if (dtype == TCDE_F32) nan_flag_kernel<float><<<(unsigned)blocks, kThreads, 0, s>>>((const float*)x, n, flags);
    else nan_flag_kernel<double><<<(unsigned)blocks, kThreads, 0, s>>>((const double*)x, n, flags);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

extern "C" int tcde_set_natural_variant(int variant) {
    TCDE_CHECK_ARG(variant >= 0 && variant <= 2,
                   "variant=%d (0 parallel kernels, 1 one thread per series, 2 CTA-per-path natural kernel)", variant);
    g_natural_variant = variant;
    g_fill_variant = variant;
    return TCDE_OK;
}

