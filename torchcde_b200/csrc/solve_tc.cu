// Hot path (ii): the fused fixed-step CDE solve on the tensor cores (sm_90a).
//
// Two kernels share the schedule, the controls, the Runge-Kutta combination and the outputs:
//   * cdeint_wgmma_kernel (2xFP16 split, the default): one warpgroup per 64 paths, warpgroup-level wgmma.mma_async with the
//     Runge-Kutta state kept in the MMA fragment layout (below);
//   * cdeint_tc_kernel (3xTF32 split): thread = path, warp = 32 paths, warp-level mma.sync through tc_common.cuh's
//     warp_field<0>.
// Each Runge-Kutta stage is
//   * dX/dt of the stage from the path's spline row (b | 2c | 3d of the interval, from HBM; the next stage's row is
//     requested before the current stage's products so that its latency hides behind them: into registers in the 3xTF32
//     kernel, into shared memory by cp.async in the 2xFP16 one);
//   * the field W z + b as a [paths x 32] . [32 x 256] product on the tensor cores with a two-way operand split
//     (tc_common.cuh), contracted with dX/dt in registers;
//   * the Runge-Kutta combination in registers, one rounding per operation in the order of oracle/odeint_port.py.
// The Runge-Kutta state y, k1 and the running k2 + k3 stay in registers for the whole solve.  With a stage dump (the adjoint's
// stage trajectory) every stage input is also written to HBM.
#include "wg_common.cuh"

namespace tcde {

namespace tc {

// torchsde's reversible Heun (zero diffusion) on NV state values: the slots y, f (k1) and z (s23) hold y_n, f_n and the z
// the current evaluation kv = f(t_st, z) was made at.  Evaluation 0 is the prologue f(t_0, y_0); evaluation st > 0 ends
// step st - 1:  y_{n+1} = y_n + (f_n + f_{n+1}) (0.5 dt_n), outputs w0 y_n + w1 y_{n+1} (out_slope = [w1..., w0...]).
// ckpt(slot, y, z, f) stores the state of every ckpt_stride-th step and of the last; zin receives the next evaluation's
// input z_{n+1} = 2 y_n - z_n + f_n dt_n.
template <int NV, typename Write, typename Ckpt>
__device__ __forceinline__ void rev_heun_combine(const UmmaArgs& a, int st, int& step, float& dt, float* y, float* f,
                                                 float* z, const float* kv, float* zin, int& jn, Write write, Ckpt ckpt) {
    using E = exact<float>;
    if (st == 0) {
#pragma unroll
        for (int h = 0; h < NV; ++h) z[h] = y[h];                       // z_0 = y_0
    } else {
        const float half = E::mul(0.5f, dt);
        float yn[NV];
#pragma unroll
        for (int h = 0; h < NV; ++h) yn[h] = E::add(y[h], E::mul(E::add(f[h], kv[h]), half));
        while (jn < a.n_out && a.out_step[jn] == step) {
            const float w1 = a.out_slope[jn], w0 = a.out_slope[a.n_out + jn];
            float v[NV];
#pragma unroll
            for (int h = 0; h < NV; ++h) v[h] = E::add(E::mul(w0, y[h]), E::mul(w1, yn[h]));
            write(jn, v);
            ++jn;
        }
#pragma unroll
        for (int h = 0; h < NV; ++h) y[h] = yn[h];
        ++step;
    }
    if (step % a.ckpt_stride == 0 || step == a.n_steps) ckpt((step + a.ckpt_stride - 1) / a.ckpt_stride, y, z, kv);
    if (step < a.n_steps) {
        dt = a.step_dt[step];
#pragma unroll
        for (int h = 0; h < NV; ++h) {
            zin[h] = E::add(E::sub(E::mul(2.f, y[h]), z[h]), E::mul(kv[h], dt));
            f[h] = kv[h];
            z[h] = zin[h];
        }
    }
}

// ---- 3xTF32 split: thread = path, warp-level mma.sync ---------------------------------------------------------------

constexpr int kWarps = 4;
constexpr int kThreads = 32 * kWarps;            // 128 paths per CTA

struct Smem {
    static constexpr int b = 0;
    static constexpr int warps = (BSmem<0>::bytes + 127) & ~127;
    static constexpr int total = warps + kWarps * WarpSmem<0>::bytes;
};

// REV: reversible Heun (rev_heun_combine, checkpoints through the stage-dump pointer) instead of the Runge-Kutta methods
template <bool DUMP, bool REV>
__global__ void __launch_bounds__(kThreads, 2) cdeint_tc_kernel(const UmmaArgs a) {
    using S = Smem;
    using E = exact<float>;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((128u - (smem_u32(smem_unaligned) & 127u)) & 127u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float inv_w_scale, beta;
    prepare_b<0>(smem + S::b, a.weight, a.bias, tid, kThreads, inv_w_scale, beta);
    __syncthreads();

    const int64_t warp_path0 = (int64_t)blockIdx.x * kThreads + warp * 32;
    if (warp_path0 >= a.n_paths) return;                      // no CTA-wide barrier follows
    unsigned char* ws = smem + S::warps + warp * WarpSmem<0>::bytes;
    const int64_t path = warp_path0 + lane_row(lane);
    const bool live = path < a.n_paths;
    const int64_t lpath = live ? path : a.n_paths - 1;
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_floats = cubic ? 4 * kCh : kCh;
    // the part of a spline row that dX/dt reads: b | 2c | 3d (cubic), the slope (linear)
    const float4* crow = reinterpret_cast<const float4*>(a.control + lpath * a.n_rows * row_floats + (cubic ? kCh : 0));
    const int row_f4 = row_floats / 4;
    const float sign = (a.sign < 0.f) ? -1.f : 1.f;

    auto fetch = [&](int interval, float4* raw) {
        const float4* src = crow + (int64_t)interval * row_f4;
        raw[0] = __ldg(src); raw[1] = __ldg(src + 1);
        if (cubic) { raw[2] = __ldg(src + 2); raw[3] = __ldg(src + 3); raw[4] = __ldg(src + 4); raw[5] = __ldg(src + 5); }
    };
    auto write_out = [&](int j, const float* v) {
        if (!live) return;
        float4* dst = reinterpret_cast<float4*>(a.out + (path * a.n_out + j) * kHid);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
    };
    auto dump = [&](int stage_no, const float* z) {
        if (!DUMP || REV || !live) return;
        float4* dst = reinterpret_cast<float4*>(a.stage_dump + ((int64_t)stage_no * a.n_paths + path) * kHid);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(z[4 * c4], z[4 * c4 + 1], z[4 * c4 + 2], z[4 * c4 + 3]);
    };

    float y[kHid], k1[kHid], s23[kHid], zin[kHid];
    {
        const float4* zp = reinterpret_cast<const float4*>(a.z0 + lpath * kHid);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) {
            const float4 v = zp[c4];
            y[4 * c4] = v.x; y[4 * c4 + 1] = v.y; y[4 * c4 + 2] = v.z; y[4 * c4 + 3] = v.w;
        }
#pragma unroll
        for (int h = 0; h < kHid; ++h) { k1[h] = 0.f; s23[h] = 0.f; zin[h] = y[h]; }
    }
    int jn = 0;
    int next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
    while (jn < a.n_out && next_out < 0) {                    // outputs at the initial time
        write_out(jn, y);
        ++jn;
        next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
    }

    const int n_st = a.n_steps * a.n_stages + (REV ? 1 : 0);
    float4 raw[6], nxt[6];
    fetch(a.stage_index[0], raw);
    int step = 0, sub = 0;
    float dt = a.step_dt[0];
    for (int st = 0; st < n_st; ++st) {
        dump(st, zin);
        // dX/dt of this stage (interpolation_cubic.py:331-336) times the sign of the time direction
        float dx[kCh];
        {
            const float fr = a.stage_frac[st];
            if (cubic) {
                const float* b = reinterpret_cast<const float*>(raw);
#pragma unroll
                for (int c = 0; c < kCh; ++c) dx[c] = E::mul(E::add(b[c], E::mul(E::add(b[kCh + c], E::mul(b[2 * kCh + c], fr)), fr)), sign);
            } else {
                const float* b = reinterpret_cast<const float*>(raw);
#pragma unroll
                for (int c = 0; c < kCh; ++c) dx[c] = E::mul(b[c], sign);
            }
        }
        if (st + 1 < n_st) fetch(a.stage_index[st + 1], nxt);

        float kv[kHid];
        warp_field<0>(zin, dx, kv, ws, smem + S::b, beta, inv_w_scale);

        if (REV) {
            rev_heun_combine<kHid>(a, st, step, dt, y, k1, s23, kv, zin, jn, write_out,
                                   [&](int slot, const float* vy, const float* vz, const float* vf) {
                                       if (!DUMP || !live) return;
                                       const float* src[3] = {vy, vz, vf};
#pragma unroll
                                       for (int w = 0; w < 3; ++w) {
                                           float4* dst = reinterpret_cast<float4*>(
                                               a.stage_dump + (((int64_t)slot * 3 + w) * a.n_paths + path) * kHid);
#pragma unroll
                                           for (int c4 = 0; c4 < 8; ++c4)
                                               dst[c4] = make_float4(src[w][4 * c4], src[w][4 * c4 + 1], src[w][4 * c4 + 2],
                                                                     src[w][4 * c4 + 3]);
                                       }
                                   });
        } else if (rk_combine<kHid>(a, sub, dt, y, k1, s23, kv, zin)) {
            step_outputs<kHid>(a, step, jn, next_out, y, zin, write_out);
#pragma unroll
            for (int h = 0; h < kHid; ++h) y[h] = zin[h];
            ++step;
            sub = 0;
            if (step < a.n_steps) dt = a.step_dt[step];
        } else {
            ++sub;
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) raw[j] = nxt[j];
    }
}

// ---- 2xFP16 split: one warpgroup per 64 paths, wgmma.mma_async ------------------------------------------------------
//
// The CTA is one warpgroup and its 64 paths are the M = 64 rows of every wgmma.  Lane (g, q) = (lane >> 2, lane & 3) of
// warp w owns rows 16 w + g and 16 w + g + 8 (the rows of its A and accumulator fragments) and, of each of these rows, the
// hidden units 8 i + 2 q + e (i < 4, e < 2): exactly the columns of the A fragment of the next stage, so the operand is
// built in registers from the Runge-Kutta state.  Its 16 values of a state vector sit at index 8 r + 2 i + e (r = row).
// The product runs in chunks of kN = 64 output columns (eight hidden units x eight channels): z_lo.W_hi, z_hi.W_lo and
// z_hi.W_hi (small terms first) are six m64n64k16 wgmmas onto an accumulator that starts at the scaled bias, with A from
// registers and B (prepare_b<1, true>'s [256 rows][hi 32 | lo 32] halves, 128-byte swizzled) through one shared-memory
// descriptor per product and k step.  Two accumulators alternate: the chunk after the current one is in flight on the
// tensor core while the current one is contracted with dX/dt.  Chunk c holds hidden units 8c .. 8c + 7 with its rows
// permuted (field_tile_row) so that accumulator column 8j + 2q + e is unit 8c + 2q + (j >> 2), channel 4e + (j & 3): each
// lane holds all eight channels of exactly the units 8c + 2q + e it owns, and the contraction closes inside the lane.  The
// lane gets all eight channels of dX/dt from its quad through a per-warp shared-memory slot once per stage.  The sum is
// (P_0 + P_1) + (P_2 + P_3) with P_k = the products of channels 2k, 2k + 1, the order in which the quad reduce-scatter of
// the unpermuted layout (wg::reduce_chunk) added them, so the bits are the same.
// N = 64 issues half the wgmmas of N = 32 for the same flops; scripts/wgmma_probe.py measures what that saves.

namespace wg {

// One evaluation of the linear field for the warpgroup's 64 rows: kv = (W zin + b) . dx in the fragment layout above.
// beta, inv_w_scale: prepare_b<1, true>'s scales of the tile at b_tile (bias at b_bias).  dx: the lane's two channels of
// both rows; xch: the warp's kDxSlot bytes of shared memory, through which the quad shares them.  HOLD: all eight
// channels of both rows stay in registers for the whole evaluation (four 16-byte loads); otherwise they are read again,
// one float at a time, for each chunk and row, which holds 16 registers fewer (the Runge-Kutta backward and
// reversible_backward_kernel have no room for them; 16-byte loads there spill).  b_desc = desc_sw128 of the tile: each
// wgmma's descriptor is b_desc plus a constant.
template <bool HOLD>
__device__ __forceinline__ void field(const float* zin, const float (*dx)[2], float beta, float inv_w_scale,
                                      const float* b_bias, uint64_t b_desc, float* xch, int g, int q, float* kv) {
    // Each row scaled by its own power of two so that max(|z|, bias floor) lands in [2^13, 2^14), split into FP16
    // hi + lo A fragments [k step][4]; the inverse scales are folded into dX/dt, which goes to the quad's row of xch.
    float rs[2];
    uint32_t ahi[2][4], alo[2][4];
    __syncwarp();                                         // the previous evaluation's reads of xch are done
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float m = beta;
#pragma unroll
        for (int h = 0; h < 8; ++h) m = fmaxf(m, fabsf(zin[8 * r + h]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        const int e = min(max(exponent_of(m), 30), 224);
        rs[r] = pow2_biased(127 + 13 - (e - 127));
        const float inv = pow2_biased(127 - 13 + (e - 127)) * inv_w_scale;
        *reinterpret_cast<float2*>(xch + (g + 8 * r) * kCh + 2 * q) =
            make_float2(__fmul_rn(dx[r][0], inv), __fmul_rn(dx[r][1], inv));
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int t = 0; t < 4; ++t) {                     // register t: row t & 1, columns 16 k + 8 (t >> 1) + 2q, +1
            const int r = t & 1, v = 8 * r + 4 * k + 2 * (t >> 1);
            const float s0 = __fmul_rn(zin[v], rs[r]), s1 = __fmul_rn(zin[v + 1], rs[r]);
            float h0, h1;
            ahi[k][t] = pack_h2(s0, s1);
            unpack_h2(ahi[k][t], h0, h1);
            alo[k][t] = pack_h2(__fsub_rn(s0, h0), __fsub_rn(s1, h1));
        }
    __syncwarp();                                         // xch holds the quad's dX/dt
    float dxs[2][kCh];                                    // all eight channels of rows g and g + 8
    auto load_row = [&](int r) {
        const float4 lo = *reinterpret_cast<const float4*>(xch + (g + 8 * r) * kCh);
        const float4 hi = *reinterpret_cast<const float4*>(xch + (g + 8 * r) * kCh + 4);
        dxs[r][0] = lo.x; dxs[r][1] = lo.y; dxs[r][2] = lo.z; dxs[r][3] = lo.w;
        dxs[r][4] = hi.x; dxs[r][5] = hi.y; dxs[r][6] = hi.z; dxs[r][7] = hi.w;
    };
    auto reload_row = [&](int r) {
#pragma unroll
        for (int k = 0; k < kCh; ++k) dxs[r][k] = xch[(g + 8 * r) * kCh + k];
    };
    if (HOLD) { load_row(0); load_row(1); }

    float acc[2][kAcc];
    auto issue = [&](int chunk, float* d) {
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {                // bias of columns 8 (8 chunk + j) + 2q, +1 times the row scales
            const float2 bb = *reinterpret_cast<const float2*>(b_bias + chunk * kN + 8 * j + 2 * q);
            d[4 * j + 0] = bb.x * rs[0]; d[4 * j + 1] = bb.y * rs[0];
            d[4 * j + 2] = bb.x * rs[1]; d[4 * j + 3] = bb.y * rs[1];
        }
        mma_fence();
        const uint32_t rows = chunk * kN * 128;
        mma_m64n64k16(d, alo[0], desc_add(b_desc, rows + 0));    // z_lo . W_hi
        mma_m64n64k16(d, alo[1], desc_add(b_desc, rows + 32));
        mma_m64n64k16(d, ahi[0], desc_add(b_desc, rows + 64));   // z_hi . W_lo
        mma_m64n64k16(d, ahi[1], desc_add(b_desc, rows + 96));
        mma_m64n64k16(d, ahi[0], desc_add(b_desc, rows + 0));    // z_hi . W_hi
        mma_m64n64k16(d, ahi[1], desc_add(b_desc, rows + 32));
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
        // the contraction of the lane's units 8c + 2q + u, rows g and g + 8: d[4 j + 2 r + e] is unit 8c + 2q + (j >> 2),
        // channel 4e + (j & 3), so channels 2k, 2k + 1 of unit u sit at j = 4u + 2 (k & 1) + {0, 1}, e = k >> 1
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!HOLD) reload_row(r);
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                float p[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int j = 4 * u + 2 * (k & 1), e = k >> 1;
                    p[k] = fmaf(d[4 * (j + 1) + 2 * r + e], dxs[r][2 * k + 1],
                                __fmul_rn(d[4 * j + 2 * r + e], dxs[r][2 * k]));
                }
                kv[8 * r + 2 * c + u] = (p[0] + p[1]) + (p[2] + p[3]);
            }
        }
    }
}

}  // namespace wg

// REV: reversible Heun (rev_heun_combine, checkpoints through the stage-dump pointer) instead of the Runge-Kutta methods.
// BWD: the Runge-Kutta backward of the linear field (rk_backward_combine) on the host-reversed schedule: the state is the
// cotangent ybar, the field product runs on the regrouped weight W2[(k, c)][h] = W[(h, c)][k] with a zero bias, so that
// the stage product is J_s^T kappa_s; the output gradients are added at every grid state (a.inj_*), the stage inputs
// kappa_s go to the forward's dump slots (last slot first) and dL/dz0 to a.out.
template <bool DUMP, bool REV, bool BWD = false>
__global__ void __launch_bounds__(wg::kThreads, 3) cdeint_wgmma_kernel(const UmmaArgs a) {
    using S = BSmem<1>;
    using E = exact<float>;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((1024u - (smem_u32(smem_unaligned) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    float inv_w_scale, beta;
    prepare_b<1, true>(smem, a.weight, a.bias, tid, wg::kThreads, inv_w_scale, beta);
    if (a.sign < 0.f) inv_w_scale = -inv_w_scale;       // the sign of the time direction: dX/dt is negated exactly either way
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the tile is read by wgmma (the async proxy)
    __syncthreads();

    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_f2 = (cubic ? 4 * kCh : kCh) / 2;
    int64_t path[2];
    bool live[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        path[r] = (int64_t)blockIdx.x * wg::kPaths + 16 * warp + g + 8 * r;
        live[r] = path[r] < a.n_paths;
    }
    // channels 2q, 2q + 1 of b (cubic; +4, +8: 2c, 3d) or of the slope (linear) in the spline rows of row 0; row 1's are
    // row1 paths further (8, or fewer where the batch ends and the reads are clamped)
    const int64_t lpath0 = live[0] ? path[0] : a.n_paths - 1;
    const int row1 = (int)((live[1] ? path[1] : a.n_paths - 1) - lpath0);
    const float2* crow = reinterpret_cast<const float2*>(a.control + lpath0 * a.n_rows * (2 * row_f2) + (cubic ? kCh : 0)) + q;

    // These pieces travel to shared memory by cp.async, a stage ahead of their use, into one of two per-warp buffers of
    // [row r][b | 2c | 3d][lane] float2: held in registers across the products they would push the stage over the
    // register cap.  Each lane reads back only what it copied itself.  The lane's two source rows and its buffer address
    // are kept in its fetch slot (wg::kFetch) and read back once per stage: at the register cap the compiler would
    // otherwise recompute them from the lane's paths every stage, about 60 integer instructions.
    {
        const float2* src1 = crow + (int64_t)row1 * a.n_rows * row_f2;
        reinterpret_cast<ulonglong2*>(smem + wg::kFetch)[tid] =
            make_ulonglong2(reinterpret_cast<uint64_t>(crow), reinterpret_cast<uint64_t>(src1));
        reinterpret_cast<uint32_t*>(smem + wg::kFetch + wg::kThreads * 16)[tid] =
            smem_u32(smem + wg::kRows + warp * 2 * wg::kRowSlot + lane * 8);
    }
    const ulonglong2* fetch_src = reinterpret_cast<const ulonglong2*>(smem + wg::kFetch) + tid;
    const uint32_t* fetch_dst = reinterpret_cast<const uint32_t*>(smem + wg::kFetch + wg::kThreads * 16) + tid;
    const int row_bytes = row_f2 * 8;
    auto fetch = [&](int interval, int buf) {
        const ulonglong2 base = *fetch_src;
        const uint32_t dst = *fetch_dst + buf * wg::kRowSlot;
        const int64_t off = (int64_t)interval * row_bytes;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const char* src = reinterpret_cast<const char*>(r ? base.y : base.x) + off;
            wg::cp_async8(dst + 3 * r * 256, src);
            if (cubic) { wg::cp_async8(dst + (3 * r + 1) * 256, src + 32); wg::cp_async8(dst + (3 * r + 2) * 256, src + 64); }
        }
        cp_async_commit();
    };
    // the lane's 16 values of a [path][32] row pair: float2 at column 8 i + 2 q of row r
    auto store_rows = [&](float* base, int64_t stride_rows, int64_t row_off, const float* v) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!live[r]) continue;
            float2* dst = reinterpret_cast<float2*>(base + (path[r] * stride_rows + row_off) * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[4 * i] = make_float2(v[8 * r + 2 * i], v[8 * r + 2 * i + 1]);
        }
    };
    auto write_out = [&](int j, const float* v) { store_rows(a.out, a.n_out, j, v); };
    // BWD: v += the output gradients that land on grid state r (counted from the end of the solve)
    auto inject = [&](int r, float* v) {
        for (int e = a.inj_range[r]; e < a.inj_range[r + 1]; ++e) {
            const int j = a.inj_out[e];
            const float w = a.inj_weight[e];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int64_t lpath = live[rr] ? path[rr] : a.n_paths - 1;
                const float2* src = reinterpret_cast<const float2*>(a.grad_out + (lpath * a.n_out + j) * kHid) + q;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 t = src[4 * i];
                    v[8 * rr + 2 * i] = E::add(v[8 * rr + 2 * i], E::mul(w, t.x));
                    v[8 * rr + 2 * i + 1] = E::add(v[8 * rr + 2 * i + 1], E::mul(w, t.y));
                }
            }
        }
    };

    float y[wg::kNV], k1[wg::kNV], s23[wg::kNV], zin[wg::kNV];
    int jn = 0, next_out = 0;
    if constexpr (BWD) {
#pragma unroll
        for (int h = 0; h < wg::kNV; ++h) { y[h] = 0.f; k1[h] = 0.f; s23[h] = 0.f; }
        inject(0, y);
        rk_backward_first<wg::kNV>(a, a.step_dt[0], y, zin);
    } else {
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
        next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
        while (jn < a.n_out && next_out < 0) {                    // outputs at the initial time
            write_out(jn, y);
            ++jn;
            next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
        }
    }

    const float* b_bias = reinterpret_cast<const float*>(smem + S::bias);
    const uint64_t b_desc = wg::desc_sw128(smem_u32(smem + S::tile));
    float* xch = reinterpret_cast<float*>(smem + wg::kXch + warp * wg::kDxSlot);
    const int n_st = a.n_steps * a.n_stages + (REV ? 1 : 0);
    // dX/dt (interpolation_cubic.py:331-336) of a stage at fraction fr of its interval, channels 2q, 2q + 1 of both rows,
    // from the rows fetched into buffer buf
    auto slope = [&](int buf, float fr, float (*dx)[2]) {
        cp_async_wait<0>();
        const uint32_t raw = *fetch_dst + buf * wg::kRowSlot;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2 b = wg::lds_f2(raw + 3 * r * 256);
            if (cubic) {
                const float2 c2 = wg::lds_f2(raw + (3 * r + 1) * 256), d3 = wg::lds_f2(raw + (3 * r + 2) * 256);
                dx[r][0] = E::add(b.x, E::mul(E::add(c2.x, E::mul(d3.x, fr)), fr));
                dx[r][1] = E::add(b.y, E::mul(E::add(c2.y, E::mul(d3.y, fr)), fr));
            } else {
                dx[r][0] = b.x;
                dx[r][1] = b.y;
            }
        }
    };
    // stage st's [path][32] block (BWD: the forward's slot of stage st, walking down from the last)
    float* dump_at = BWD ? a.stage_dump + (int64_t)(n_st - 1) * a.n_paths * kHid : a.stage_dump;
    fetch(a.stage_index[0], 0);
    int step = 0, sub = 0;
    float dt = a.step_dt[0];
    for (int st = 0; st < n_st; ++st) {
        if (DUMP && !REV) {
            store_rows(dump_at, 1, 0, zin);
            if (BWD) dump_at -= a.n_paths * kHid;
            else dump_at += a.n_paths * kHid;
        }
        float dx[2][2];
        slope(st & 1, a.stage_frac[st], dx);
        // the next stage's spline rows; their latency hides behind this stage's products
        if (st + 1 < n_st) fetch(a.stage_index[st + 1], (st + 1) & 1);

        float kv[wg::kNV];
        wg::field<!BWD>(zin, dx, beta, inv_w_scale, b_bias, b_desc, xch, g, q, kv);

        if (REV) {
            rev_heun_combine<wg::kNV>(a, st, step, dt, y, k1, s23, kv, zin, jn, write_out,
                                      [&](int slot, const float* vy, const float* vz, const float* vf) {
                                          if (!DUMP) return;
                                          float* base = a.stage_dump + (int64_t)slot * 3 * a.n_paths * kHid;
                                          store_rows(base, 1, 0, vy);
                                          store_rows(base + a.n_paths * kHid, 1, 0, vz);
                                          store_rows(base + 2 * a.n_paths * kHid, 1, 0, vf);
                                      });
        } else if constexpr (BWD) {
            if (rk_backward_combine<wg::kNV>(a, sub, dt, y, k1, s23, kv, zin)) {
                ++step;
                sub = 0;
                inject(step, y);
                if (step < a.n_steps) {
                    dt = a.step_dt[step];
                    rk_backward_first<wg::kNV>(a, dt, y, zin);
                }
            } else {
                ++sub;
            }
        } else if (rk_combine<wg::kNV>(a, sub, dt, y, k1, s23, kv, zin)) {
            step_outputs<wg::kNV>(a, step, jn, next_out, y, zin, write_out);
#pragma unroll
            for (int h = 0; h < wg::kNV; ++h) y[h] = zin[h];
            ++step;
            sub = 0;
            if (step < a.n_steps) dt = a.step_dt[step];
        } else {
            ++sub;
        }
    }
    if constexpr (BWD) store_rows(a.out, 1, 0, y);
}


// ---- the reversible Heun backward: one launch per checkpoint segment ---------------------------------------------------
//
// The transpose of rev_heun_combine, run backwards over the steps m = hi - 1 .. lo of one segment in the wgmma fragment
// layout (one warpgroup per 64 paths, the lane's 16 values as in cdeint_wgmma_kernel).  State per lane: y, z, f of step
// m + 1 and the adjoints ybar, zbar.  Per step:
//   ybar_m = ybar + 2 zbar + (output gradients on y_m);   fbar_m = ybar dt_m / 2 + zbar dt_m + ybar_m dt_{m-1} / 2;
//   z_m = 2 y - z - f dt_m (at m = lo: the checkpoint's z);
//   f_m = F(z_m) with (W, b) and J_F(z_m)^T fbar_m = sum_c dX_c (W2 fbar_m) with the regrouped W2, both wg::field products
//   at dX/dt(t_m) from two B tiles;  y_m = y - (f_m + f) dt_m / 2 (at m = lo: the checkpoint's y, f);
//   zbar_m = J^T fbar_m - zbar;
// and (z_m, fbar_m) go to the segment's dump, which tcde_linear_field_param_grads contracts into dL/dW, dL/db.
struct RevBwdArgs {
    const float* control;
    const float* weight;          // [256][32]
    const float* bias;            // [256]
    const float* weight_t;        // W2[(k, c)][h] = W[(h, c)][k]
    const float* zeros;           // [256] zeros: W2's bias
    const float* ckpt_lo;         // [3][n_paths][32]: y, z, f of step lo
    const float* ckpt_hi;         // ... of step hi
    float* carry;                 // [2][n_paths][32]: ybar, zbar of step hi in, of step lo out
    const float* g;               // [n_paths][n_out][32] output gradients
    const int32_t* out_step;      // [n_out]
    const float* out_weights;     // [2][n_out]: w1, then w0
    const int32_t* inj_range;     // [N + 1][2]: the outputs [first, end) that touch y_m
    const float* step_dt;
    const int32_t* stage_index;   // [N + 1]
    const float* stage_frac;
    float* dump_z;                // [hi - lo][n_paths][32]
    float* dump_a;
    int64_t n_paths, n_rows;
    int control_kind, n_out, lo, hi;
};

constexpr int kRevTile = (BSmem<1>::bytes + 1023) & ~1023;
constexpr int kRevSmem = 2 * kRevTile + 4 * wg::kDxSlot + 1024;     // two B tiles, the warps' dX/dt slots, alignment

__global__ void __launch_bounds__(wg::kThreads, 2) reversible_backward_kernel(const RevBwdArgs a) {
    using S = BSmem<1>;
    using E = exact<float>;
    constexpr int NV = wg::kNV;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((1024u - (smem_u32(smem_unaligned) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    float inv_f, beta_f, inv_g, beta_g;
    prepare_b<1, true>(smem, a.weight, a.bias, tid, wg::kThreads, inv_f, beta_f);
    prepare_b<1, true>(smem + kRevTile, a.weight_t, a.zeros, tid, wg::kThreads, inv_g, beta_g);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const float* bias_f = reinterpret_cast<const float*>(smem + S::bias);
    const float* bias_g = reinterpret_cast<const float*>(smem + kRevTile + S::bias);
    const uint64_t desc_f = wg::desc_sw128(smem_u32(smem + S::tile));
    const uint64_t desc_g = wg::desc_sw128(smem_u32(smem + kRevTile + S::tile));
    float* xch = reinterpret_cast<float*>(smem + 2 * kRevTile + warp * wg::kDxSlot);

    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_f2 = (cubic ? 4 * kCh : kCh) / 2;
    int64_t path[2], lpath[2];
    bool live[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        path[r] = (int64_t)blockIdx.x * wg::kPaths + 16 * warp + g + 8 * r;
        live[r] = path[r] < a.n_paths;
        lpath[r] = live[r] ? path[r] : a.n_paths - 1;
    }
    auto load_rows = [&](const float* base, int64_t stride_rows, int64_t row_off, float* v) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2* src = reinterpret_cast<const float2*>(base + (lpath[r] * stride_rows + row_off) * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 t = src[4 * i];
                v[8 * r + 2 * i] = t.x; v[8 * r + 2 * i + 1] = t.y;
            }
        }
    };
    auto store_rows = [&](float* base, const float* v) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!live[r]) continue;
            float2* dst = reinterpret_cast<float2*>(base + path[r] * kHid) + q;
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[4 * i] = make_float2(v[8 * r + 2 * i], v[8 * r + 2 * i + 1]);
        }
    };
    // dX/dt of evaluation point m: channels 2q, 2q + 1 of both rows
    auto slope_at = [&](int m, float (*dx)[2]) {
        const int interval = a.stage_index[m];
        const float fr = a.stage_frac[m];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2* src = reinterpret_cast<const float2*>(a.control + (lpath[r] * a.n_rows + interval) * (2 * row_f2) +
                                                                (cubic ? kCh : 0)) + q;
            const float2 b = __ldg(src);
            if (cubic) {
                const float2 c2 = __ldg(src + 4), d3 = __ldg(src + 8);
                dx[r][0] = E::add(b.x, E::mul(E::add(c2.x, E::mul(d3.x, fr)), fr));
                dx[r][1] = E::add(b.y, E::mul(E::add(c2.y, E::mul(d3.y, fr)), fr));
            } else {
                dx[r][0] = b.x;
                dx[r][1] = b.y;
            }
        }
    };

    const int64_t plane = a.n_paths;
    float y[NV], z[NV], f[NV], yb[NV], zb[NV];
    load_rows(a.ckpt_hi, 1, 0, y);
    load_rows(a.ckpt_hi + plane * kHid, 1, 0, z);
    load_rows(a.ckpt_hi + 2 * plane * kHid, 1, 0, f);
    load_rows(a.carry, 1, 0, yb);
    load_rows(a.carry + plane * kHid, 1, 0, zb);
    for (int m = a.hi - 1; m >= a.lo; --m) {
        const float d = a.step_dt[m], dp = m > 0 ? a.step_dt[m - 1] : 0.f;
        const float hd = E::mul(0.5f, d), hdp = E::mul(0.5f, dp);
        float ybm[NV], fb[NV], zm[NV];
#pragma unroll
        for (int h = 0; h < NV; ++h) ybm[h] = E::add(yb[h], E::mul(2.f, zb[h]));
        for (int j = a.inj_range[2 * m]; j < a.inj_range[2 * m + 1]; ++j) {
            const int os = a.out_step[j];
            const float w = (os == m) ? a.out_weights[a.n_out + j] : (os < 0 ? 1.f : a.out_weights[j]);
            float gv[NV];
            load_rows(a.g, a.n_out, j, gv);
#pragma unroll
            for (int h = 0; h < NV; ++h) ybm[h] = fmaf(w, gv[h], ybm[h]);
        }
#pragma unroll
        for (int h = 0; h < NV; ++h) fb[h] = E::add(E::add(E::mul(yb[h], hd), E::mul(zb[h], d)), E::mul(ybm[h], hdp));
        if (m == a.lo) {
            load_rows(a.ckpt_lo + plane * kHid, 1, 0, zm);
        } else {
#pragma unroll
            for (int h = 0; h < NV; ++h) zm[h] = E::sub(E::sub(E::mul(2.f, y[h]), z[h]), E::mul(f[h], d));
        }
        float dx[2][2];
        slope_at(m, dx);
        float kf[NV], kg[NV];
        wg::field<false>(zm, dx, beta_f, inv_f, bias_f, desc_f, xch, g, q, kf);
        wg::field<false>(fb, dx, beta_g, inv_g, bias_g, desc_g, xch, g, q, kg);
        store_rows(a.dump_z + (int64_t)(m - a.lo) * plane * kHid, zm);
        store_rows(a.dump_a + (int64_t)(m - a.lo) * plane * kHid, fb);
        if (m == a.lo) {
            load_rows(a.ckpt_lo, 1, 0, y);
            load_rows(a.ckpt_lo + 2 * plane * kHid, 1, 0, f);
        } else {
#pragma unroll
            for (int h = 0; h < NV; ++h) {
                y[h] = E::sub(y[h], E::mul(E::add(kf[h], f[h]), hd));
                f[h] = kf[h];
            }
        }
#pragma unroll
        for (int h = 0; h < NV; ++h) {
            z[h] = zm[h];
            zb[h] = E::sub(kg[h], zb[h]);
            yb[h] = ybm[h];
        }
    }
    store_rows(a.carry, yb);
    store_rows(a.carry + plane * kHid, zb);
}

}  // namespace tc

int solve_tc_f32(const UmmaArgs& a, int H, int C, int mode, cudaStream_t stream) {
    TCDE_CHECK_SUPPORTED(H == tc::kHid && C == tc::kCh, "tensor-core solve: built for hidden=32, channels=8 (got %d, %d)", H, C);
    TCDE_CHECK_SUPPORTED(aligned16(a.control, a.z0, a.out), "tensor-core solve: control, z0 and out must be 16-byte aligned");
    TCDE_CHECK_SUPPORTED(aligned16(a.stage_dump), "tensor-core solve: the stage dump must be 16-byte aligned");
    // mode: bit 0 = operand split (0 = 3xTF32, 1 = 2xFP16)
    const bool rev = (a.method == TCDE_REVERSIBLE_HEUN);
    if (mode & 1)
        return launch(rev ? (a.stage_dump ? tc::cdeint_wgmma_kernel<true, true> : tc::cdeint_wgmma_kernel<false, true>)
                          : (a.stage_dump ? tc::cdeint_wgmma_kernel<true, false> : tc::cdeint_wgmma_kernel<false, false>),
                      (a.n_paths + tc::wg::kPaths - 1) / tc::wg::kPaths, tc::wg::kThreads, tc::wg::kSmem, stream, a);
    return launch(rev ? (a.stage_dump ? tc::cdeint_tc_kernel<true, true> : tc::cdeint_tc_kernel<false, true>)
                      : (a.stage_dump ? tc::cdeint_tc_kernel<true, false> : tc::cdeint_tc_kernel<false, false>),
                  (a.n_paths + tc::kThreads - 1) / tc::kThreads, tc::kThreads,
                  tc::Smem::total + 128, stream, a);               // slack for the 128-byte alignment of the tiles
}

}  // namespace tcde

using namespace tcde;

extern "C" int tcde_reversible_heun_linear_backward_segment(
    const void* control, int control_kind, int64_t n_rows, const void* weight, const void* bias, const void* weight_t,
    const void* zeros, const void* ckpt_lo, const void* ckpt_hi, void* carry, const void* g, int64_t n_out,
    const int32_t* out_step, const void* out_weights, const int32_t* inj_range, const void* step_dt,
    const int32_t* stage_index, const void* stage_frac, int64_t lo, int64_t hi, int64_t n_paths, int64_t channels,
    int64_t hidden, void* dump_z, void* dump_a, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && weight && bias && weight_t && zeros && ckpt_lo && ckpt_hi && carry && g && dump_z && dump_a,
                   "null data pointer");
    TCDE_CHECK_ARG(out_step && out_weights && inj_range && step_dt && stage_index && stage_frac, "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_out >= 1 && lo >= 0 && hi > lo && hi < (1ll << 31), "bad sizes");
    TCDE_TRY(check_control_kind(control_kind));
    LinearRoute r;
    TCDE_TRY(linear_route(kLinBackward, hidden, channels, dtype, true, "the reversible backward kernel is ", &r));
    TCDE_CHECK_SUPPORTED(aligned16(control, ckpt_lo, ckpt_hi, carry, g, dump_z, dump_a),
                         "reversible backward: buffers must be 16-byte aligned");
    if (n_paths == 0) return TCDE_OK;
    const tc::RevBwdArgs a{(const float*)control, (const float*)weight, (const float*)bias, (const float*)weight_t,
                           (const float*)zeros, (const float*)ckpt_lo, (const float*)ckpt_hi, (float*)carry,
                           (const float*)g, out_step, (const float*)out_weights, inj_range, (const float*)step_dt,
                           stage_index, (const float*)stage_frac, (float*)dump_z, (float*)dump_a, n_paths, n_rows,
                           control_kind, (int)n_out, (int)lo, (int)hi};
    return launch(tc::reversible_backward_kernel, (n_paths + tc::wg::kPaths - 1) / tc::wg::kPaths, tc::wg::kThreads,
                  tc::kRevSmem, static_cast<cudaStream_t>(stream), a);
}

extern "C" int tcde_cdeint_fixed_linear_backward(
    const void* control, int control_kind, int64_t n_rows, const void* weight_t, const void* zeros, const void* grad_out,
    void* grad_z0, void* kappa_dump, int64_t n_paths, int64_t channels, int64_t hidden, int method, int64_t n_steps,
    const void* step_dt_rev, const int32_t* stage_index_rev, const void* stage_frac_rev, int64_t n_out,
    const int32_t* inj_range, const int32_t* inj_out, const void* inj_weight, double sign, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && weight_t && zeros && grad_out && grad_z0, "null data pointer");
    TCDE_CHECK_ARG(step_dt_rev && stage_index_rev && stage_frac_rev && inj_range && inj_out && inj_weight,
                   "null schedule pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && n_steps >= 1 && n_out >= 1, "bad sizes");
    TCDE_TRY(check_control_kind(control_kind));
    TCDE_TRY(check_method(method));
    TCDE_CHECK_SUPPORTED(n_steps * 4 < (1ll << 31) && n_out < (1ll << 31), "schedule too long");
    LinearRoute r;
    TCDE_TRY(linear_route(kLinBackward, hidden, channels, dtype, true, "the Runge-Kutta backward kernel is ", &r));
    TCDE_CHECK_SUPPORTED(aligned16(control, grad_out, grad_z0, kappa_dump),
                         "Runge-Kutta backward: control, grad_out, grad_z0 and the dump must be 16-byte aligned");
    if (n_paths == 0) return TCDE_OK;
    const int n_stages = (method == TCDE_RK4_38) ? 4 : (method == TCDE_MIDPOINT) ? 2 : 1;
    const UmmaArgs u{(const float*)control, (const float*)weight_t, (const float*)zeros, nullptr, (float*)grad_z0,
                     (const float*)step_dt_rev, stage_index_rev, (const float*)stage_frac_rev, nullptr, nullptr, nullptr,
                     n_paths, n_rows, control_kind, method, n_stages, (int)n_steps, (int)n_out, (float)sign,
                     (float*)kappa_dump, 0, (const float*)grad_out, inj_range, inj_out, (const float*)inj_weight};
    return launch(kappa_dump ? tc::cdeint_wgmma_kernel<true, false, true> : tc::cdeint_wgmma_kernel<false, false, true>,
                  (n_paths + tc::wg::kPaths - 1) / tc::wg::kPaths, tc::wg::kThreads, tc::wg::kSmem,
                  static_cast<cudaStream_t>(stream), u);
}
