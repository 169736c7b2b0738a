// Hot path (i): batched spline-coefficient construction (sm_90a) -- Hermite cubic with backward differences.
//
// The builders are HBM-bound streaming kernels (SURVEY.md 8d: ~1 flop per byte).  The design rules
// that matter are the memory ones: coalesced 128-bit loads, results staged in shared memory and
// written back as contiguous 1-D bulk (TMA) stores, persistent CTAs sized from the SM count.
// Arithmetic uses tcde::exact<> (one rounding per operation, no FMA contraction) wherever the header
// promises bit-identical results.
#include "builders_common.cuh"

namespace tcde {

// =========================================================================================
// Hermite cubic with backward differences  (interpolation_hermite_cubic_bdiff.py:5-44)
// =========================================================================================
// Work item = (path, tile of TR consecutive intervals).  The CTA stages the TR+2 knot rows it
// needs in shared memory, every thread produces the four coefficients of its (interval,
// channel) elements into a shared output tile laid out exactly like global memory
// ([row][a|b|2c|3d][channel]), and one thread issues a single bulk store of the tile (the
// tile is a contiguous byte range of the output).  Two output tiles alternate so that the
// store of tile n overlaps the computation of tile n+1.
// A row too wide for one tile in shared memory (fp64 channels >= 2,327) is split into channel tiles of at most CW
// channels: work item = (path, row tile, channel tile), and the tile's four CW-wide parts per row are stored with
// plain stores (they are not one contiguous byte range of the output; the launcher passes use_bulk = 0).
template <typename T, bool UNIT>
__global__ void __launch_bounds__(kThreads)
hermite_kernel(const T* __restrict__ x, const T* __restrict__ t, T* __restrict__ out, int64_t n_paths, int L, int C,
               int CW, int TR, int tiles_per_path, int use_bulk, int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<T>;
    T* ot0 = reinterpret_cast<T*>(smem_raw);
    T* ot1 = ot0 + (size_t)TR * 4 * CW;
    T* xs = ot1 + (size_t)TR * 4 * CW;
    T* ts = xs + (size_t)(TR + 2) * CW;

    const int tid = threadIdx.x;
    const int ctiles = (C + CW - 1) / CW;
    const int64_t n_items = n_paths * tiles_per_path * ctiles;
    bool saw_nan = false;
    int buf = 0;

    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x, buf ^= 1) {
        const int64_t pt = item / ctiles;
        const int c0 = (int)(item - pt * ctiles) * CW;
        const int cw = min(CW, C - c0);                      // channels of this tile (C when the row is not split)
        const int row_elems = 4 * cw;
        const int di = kThreads / cw, dc = kThreads - di * cw;   // (row, channel) advance per thread-stride
        const int64_t p = pt / tiles_per_path;
        const int tile = (int)(pt - p * tiles_per_path);
        const int r0 = tile * TR;
        const int nr = min(TR, L - 1 - r0);
        if (use_bulk && tid == 0) bulk_wait_read<1>();   // the store that last read ot[buf] has drained

        // knot rows r0-1 .. r0+nr ; row -1 does not exist for the first tile
        const T* xp = x + (p * L + r0 - 1) * C + c0;
        const int ne = (nr + 2) * cw;
        if (cw == C) {
            for (int e = (r0 == 0 ? C : 0) + tid; e < ne; e += kThreads) xs[e] = xp[e];
        } else {
            for (int e = (r0 == 0 ? cw : 0) + tid; e < ne; e += kThreads) {
                const int row = e / cw;
                xs[e] = xp[(int64_t)row * C + (e - row * cw)];
            }
        }
        if (!UNIT) {
            for (int e = (r0 == 0 ? 1 : 0) + tid; e < nr + 2; e += kThreads) ts[e] = t[r0 - 1 + e];
        }
        __syncthreads();

        T* ot = buf ? ot1 : ot0;
        int i = tid / cw, c = tid - (tid / cw) * cw;
        for (int e = tid; e < nr * cw; e += kThreads) {
            const T xl = xs[(i + 1) * cw + c];
            const T xh = xs[(i + 2) * cw + c];
            saw_nan |= is_nan(xl) | is_nan(xh);
            const bool first = (r0 + i == 0);
            T b, two_c, three_d;
            if (UNIT) {
                // dt == 1 exactly: every division by dt and the 1/dt^2 factor are exact identities
                const T dn = E::sub(xh, xl);
                const T dp = first ? dn : E::sub(xl, xs[i * cw + c]);
                const T bend = E::sub(dn, dp);
                const T inner = E::add(E::sub(E::mul(T(3), bend), dn), dp);
                two_c = E::mul(T(2), inner);
                three_d = E::sub(bend, two_c);
                b = dp;
            } else {
                const T dt = E::sub(ts[i + 2], ts[i + 1]);
                const T dn = E::div(E::sub(xh, xl), dt);                       // bdiff.py:39
                const T dp = first ? dn : E::div(E::sub(xl, xs[i * cw + c]), E::sub(ts[i + 1], ts[i]));
                const T inner = E::add(E::sub(E::mul(T(3), E::sub(dn, dp)), dn), dp);
                two_c = E::div(E::mul(T(2), inner), dt);                        // bdiff.py:17
                const T inv_sq = E::div(T(1), E::mul(dt, dt));
                three_d = E::sub(E::mul(inv_sq, E::sub(dn, dp)), E::div(two_c, dt));   // bdiff.py:18
                b = dp;
            }
            // four stores per thread; rotating which coefficient goes first by row spreads a
            // warp's stores over all 32 banks (rows are 4C words apart)
            T* row = ot + (size_t)i * row_elems + c;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int w = (k + i) & 3;
                const T v = (w == 0) ? xl : (w == 1) ? b : (w == 2) ? two_c : three_d;
                row[w * cw] = v;
            }
            i += di;
            c += dc;
            if (c >= cw) { c -= cw; ++i; }
        }
        T* gp = out + (p * (int64_t)(L - 1) + r0) * 4 * C;
        if (cw != C) {                                     // one channel tile: rows 4C apart, parts C apart
            __syncthreads();
            for (int e = tid; e < nr * row_elems; e += kThreads) {
                const int r = e / row_elems, rem = e - r * row_elems;
                const int w = rem / cw;
                gp[(int64_t)r * 4 * C + (int64_t)w * C + c0 + (rem - w * cw)] = ot[e];
            }
        } else if (use_bulk) {
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
    if (use_bulk && tid == 0) bulk_wait_read<0>();
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}

// Vectorised fp32 variant for channels % 4 == 0 (the BASELINE shapes): one thread produces a whole
// (interval, 4-channel) block -- three 128-bit read-only loads of the neighbouring knot rows
// straight from global memory (each row is reused by three intervals and hits L1), 4-wide
// arithmetic, four 128-bit shared stores -- so the instruction count per output byte is ~4x
// lower than the scalar kernel's (which ncu showed to be issue-bound at ~40% of HBM peak), and
// a tile needs one CTA barrier instead of two.
template <bool UNIT>
__global__ void __launch_bounds__(kThreads)
hermite_vec4_kernel(const float* __restrict__ x, const float* __restrict__ t, float* __restrict__ out,
                    int64_t n_paths, int L, int C, int TR, int tiles_per_path, int32_t* __restrict__ flags) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using E = exact<float>;
    const int Q = C >> 2;                                   // 16-byte chunks per coefficient part
    const int row_chunks = 4 * Q;
    float4* ot0 = reinterpret_cast<float4*>(smem_raw);
    float4* ot1 = ot0 + (size_t)TR * row_chunks;
    const int tid = threadIdx.x;
    const int di = kThreads / Q, dq = kThreads - di * Q;
    const int i_first = tid / Q, q_first = tid - i_first * Q;
    const int64_t n_items = n_paths * tiles_per_path;
    bool saw_nan = false;
    int buf = 0;

    for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x, buf ^= 1) {
        const int64_t p = item / tiles_per_path;
        const int tile = (int)(item - p * tiles_per_path);
        const int r0 = tile * TR;
        const int nr = min(TR, L - 1 - r0);
        const float4* xp = reinterpret_cast<const float4*>(x + p * (int64_t)L * C);
        float4* ot = buf ? ot1 : ot0;
        if (tid == 0) bulk_wait_read<1>();
        __syncthreads();                                    // ot[buf] is free again (and visible to all)
        int i = i_first, q = q_first;
        for (int e = tid; e < nr * Q; e += kThreads) {
            const int r = r0 + i;
            const float4 lo = __ldg(xp + (size_t)r * Q + q);
            const float4 hi = __ldg(xp + (size_t)(r + 1) * Q + q);
            const float4 pp = (r > 0) ? __ldg(xp + (size_t)(r - 1) * Q + q) : lo;
            saw_nan |= is_nan(lo.x) | is_nan(lo.y) | is_nan(lo.z) | is_nan(lo.w) | is_nan(hi.x) | is_nan(hi.y) |
                       is_nan(hi.z) | is_nan(hi.w);
            const float xl[4] = {lo.x, lo.y, lo.z, lo.w}, xh[4] = {hi.x, hi.y, hi.z, hi.w};
            const float xq[4] = {pp.x, pp.y, pp.z, pp.w};
            float b[4], c2[4], d3[4];
            float dt = 1.f, dtp = 1.f, inv_sq = 1.f;
            if (!UNIT) {
                dt = E::sub(t[r + 1], t[r]);
                dtp = (r > 0) ? E::sub(t[r], t[r - 1]) : dt;
                inv_sq = E::div(1.f, E::mul(dt, dt));
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (UNIT) {
                    const float dn = E::sub(xh[j], xl[j]);
                    const float dp = (r > 0) ? E::sub(xl[j], xq[j]) : dn;
                    const float bend = E::sub(dn, dp);
                    c2[j] = E::mul(2.f, E::add(E::sub(E::mul(3.f, bend), dn), dp));
                    d3[j] = E::sub(bend, c2[j]);
                    b[j] = dp;
                } else {
                    const float dn = E::div(E::sub(xh[j], xl[j]), dt);
                    const float dp = (r > 0) ? E::div(E::sub(xl[j], xq[j]), dtp) : dn;
                    const float inner = E::add(E::sub(E::mul(3.f, E::sub(dn, dp)), dn), dp);
                    c2[j] = E::div(E::mul(2.f, inner), dt);
                    d3[j] = E::sub(E::mul(inv_sq, E::sub(dn, dp)), E::div(c2[j], dt));
                    b[j] = dp;
                }
            }
            float4* row = ot + (size_t)i * row_chunks + q;
#pragma unroll
            for (int k = 0; k < 4; ++k) {                   // rotate the part order by row: conflict-free 128-bit stores
                const int w = (k + i) & 3;
                float4 v;
                if (w == 0) v = lo;
                else if (w == 1) v = make_float4(b[0], b[1], b[2], b[3]);
                else if (w == 2) v = make_float4(c2[0], c2[1], c2[2], c2[3]);
                else v = make_float4(d3[0], d3[1], d3[2], d3[3]);
                row[w * Q] = v;
            }
            i += di;
            q += dq;
            if (q >= Q) { q -= Q; ++i; }
        }
        fence_proxy_async_smem();
        __syncthreads();
        if (tid == 0) {
            bulk_store(out + (p * (int64_t)(L - 1) + r0) * 4 * C, ot, (uint32_t)((size_t)nr * row_chunks * 16));
            bulk_commit();
        }
    }
    if (tid == 0) bulk_wait_read<0>();
    if (saw_nan && flags != nullptr) atomicOr(flags, TCDE_FLAG_NAN_SEEN);
}


static int launch_hermite_vec4(const float* x, const float* t, float* out, int64_t n_paths, int L, int C,
                               int32_t* flags, cudaStream_t stream) {
    const size_t row_bytes = (size_t)16 * C;
    int TR = (int)(16384 / row_bytes);
    if (TR < 1) TR = 1;
    if (TR > L - 1) TR = L - 1;
    const size_t smem = 2 * TR * row_bytes + 16;
    const int tiles = (L - 1 + TR - 1) / TR;
    auto kern = t ? hermite_vec4_kernel<false> : hermite_vec4_kernel<true>;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = persistent_grid((const void*)kern, kThreads, smem, n_paths * tiles);
    kern<<<grid, kThreads, smem, stream>>>(x, t, out, n_paths, L, C, TR, tiles, flags);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

template <typename T>
static int launch_hermite(const T* x, const T* t, T* out, int64_t n_paths, int L, int C, int32_t* flags,
                          cudaStream_t stream) {
    if (sizeof(T) == 4 && (C & 3) == 0 && C <= 512 && aligned16(x) && aligned16(out))
        return launch_hermite_vec4((const float*)x, (const float*)t, (float*)out, n_paths, L, C, flags, stream);
    const size_t row_bytes = (size_t)4 * C * sizeof(T);
    int TR = (int)(16384 / row_bytes);
    if (TR < 1) TR = 1;
    if (TR > L - 1) TR = L - 1;
    auto smem_of = [&](int cw) {
        return 2 * TR * (size_t)4 * cw * sizeof(T) + (size_t)(TR + 2) * cw * sizeof(T) + (size_t)(TR + 2) * sizeof(T) + 16;
    };
    // rows too wide for one tile (TR = 1 then): split the channels into the fewest tiles that fit, of equal width
    int CW = C;
    if (smem_of(C) > kMaxSmem) {
        const int cw_max = (int)((kMaxSmem - smem_of(0)) / (smem_of(1) - smem_of(0)));
        const int ctiles = (C + cw_max - 1) / cw_max;
        CW = (C + ctiles - 1) / ctiles;
    }
    const size_t smem = smem_of(CW);
    const int tiles = (L - 1 + TR - 1) / TR;
    const int use_bulk = (CW == C && aligned16(out)) ? 1 : 0;
    auto kern = t ? hermite_kernel<T, false> : hermite_kernel<T, true>;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = persistent_grid((const void*)kern, kThreads, smem, n_paths * tiles * ((C + CW - 1) / CW));
    kern<<<grid, kThreads, smem, stream>>>(x, t, out, n_paths, L, C, CW, TR, tiles, use_bulk, flags);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}


}  // namespace tcde

using namespace tcde;

extern "C" int tcde_hermite_bdiff_coeffs(const void* x, const void* t, void* coeffs, int64_t n_paths, int64_t length,
                                         int64_t channels, int dtype, int32_t* flags, void* stream) {
    int rc = check_shape(x, coeffs, n_paths, length, channels, dtype);
    if (rc != TCDE_OK) return rc;
    if (n_paths == 0) return TCDE_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (dtype == TCDE_F32)
        return launch_hermite<float>((const float*)x, (const float*)t, (float*)coeffs, n_paths, (int)length,
                                     (int)channels, flags, s);
    return launch_hermite<double>((const double*)x, (const double*)t, (double*)coeffs, n_paths, (int)length,
                                  (int)channels, flags, s);
}

