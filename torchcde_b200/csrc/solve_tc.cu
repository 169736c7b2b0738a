// Hot path (ii): the fused fixed-step CDE solve on the tensor cores (sm_90a, warp-level mma.sync).
//
// Thread = path, warp = 32 paths, and the warps of a CTA never wait for each other after the one-time setup of operand B.
// Each Runge-Kutta stage of a warp is
//   * dX/dt of the stage from the path's spline row (read straight from HBM: b | 2c | 3d of the interval, 96 bytes per path;
//     the next stage's row is requested before the current stage's products so that its latency hides behind them);
//   * the field W z + b of the warp's 32 paths as a [32 x 32] . [32 x 256] product on the tensor cores with a two-way
//     operand split (tc_common.cuh: MODE 1 = 2xFP16 with per-path power-of-two scaling, 6 MMAs per 16 x 8 block; MODE 0 =
//     3xTF32, 12 MMAs), contracted with dX/dt in registers; every lane ends with the 32 slopes of its own path;
//   * the Runge-Kutta combination in registers, one rounding per operation in the order of oracle/odeint_port.py.
// The Runge-Kutta state y, k1 and the running k2 + k3 stay in registers for the whole solve.  With a stage dump (the adjoint's
// stage trajectory) every stage input is also written to HBM.
#include "tc_common.cuh"

namespace tcde {

namespace tc {

constexpr int kWarps = 4;
constexpr int kThreads = 32 * kWarps;            // 128 paths per CTA

template <int MODE> struct Smem {
    static constexpr int b = 0;
    static constexpr int warps = (BSmem<MODE>::bytes + 127) & ~127;
    static constexpr int total = warps + kWarps * WarpSmem<MODE>::bytes;
};

template <int MODE, bool DUMP>
__global__ void __launch_bounds__(kThreads, 2) cdeint_tc_kernel(const UmmaArgs a) {
    using S = Smem<MODE>;
    using E = exact<float>;
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((128u - (smem_u32(smem_unaligned) & 127u)) & 127u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float inv_w_scale, beta;
    prepare_b<MODE>(smem + S::b, a.weight, a.bias, tid, kThreads, inv_w_scale, beta);
    __syncthreads();

    const int64_t warp_path0 = (int64_t)blockIdx.x * kThreads + warp * 32;
    if (warp_path0 >= a.n_paths) return;                      // no CTA-wide barrier follows
    unsigned char* ws = smem + S::warps + warp * WarpSmem<MODE>::bytes;
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
        if (!DUMP || !live) return;
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

    const int n_st = a.n_steps * a.n_stages;
    const float third = (float)(1.0 / 3.0);
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
        warp_field<MODE>(zin, dx, kv, ws, smem + S::b, beta, inv_w_scale);

        // Runge-Kutta combination; the next stage input ends up in zin
        bool step_done = false;
        const f2 dt2 = pk(dt, dt);
        if (a.method == TCDE_RK4_38) {
            const f2 th2 = pk(third, third);
            if (sub == 0) {
#pragma unroll
                for (int h = 0; h < kHid; h += 2) {
                    k1[h] = kv[h]; k1[h + 1] = kv[h + 1];
                    upk(add2(pk(y[h], y[h + 1]), mul2(mul2(dt2, pk(kv[h], kv[h + 1])), th2)), zin[h], zin[h + 1]);
                }
            } else if (sub == 1) {
#pragma unroll
                for (int h = 0; h < kHid; h += 2) {
                    s23[h] = kv[h]; s23[h + 1] = kv[h + 1];
                    upk(add2(pk(y[h], y[h + 1]), mul2(dt2, sub2(pk(kv[h], kv[h + 1]), mul2(pk(k1[h], k1[h + 1]), th2)))),
                        zin[h], zin[h + 1]);
                }
            } else if (sub == 2) {
#pragma unroll
                for (int h = 0; h < kHid; h += 2) {
                    const f2 k2p = pk(s23[h], s23[h + 1]), k3p = pk(kv[h], kv[h + 1]);
                    upk(add2(pk(y[h], y[h + 1]), mul2(dt2, add2(sub2(pk(k1[h], k1[h + 1]), k2p), k3p))), zin[h], zin[h + 1]);
                    upk(add2(k2p, k3p), s23[h], s23[h + 1]);
                }
            } else {
                const f2 three = pk(3.f, 3.f), eighth = pk(0.125f, 0.125f);
#pragma unroll
                for (int h = 0; h < kHid; h += 2) {
                    const f2 sum = add2(add2(pk(k1[h], k1[h + 1]), mul2(three, pk(s23[h], s23[h + 1]))), pk(kv[h], kv[h + 1]));
                    upk(add2(pk(y[h], y[h + 1]), mul2(mul2(sum, dt2), eighth)), zin[h], zin[h + 1]);
                }
                step_done = true;
            }
        } else if (a.method == TCDE_MIDPOINT) {
            if (sub == 0) {
                const float half = E::mul(0.5f, dt);
#pragma unroll
                for (int h = 0; h < kHid; ++h) zin[h] = E::add(y[h], E::mul(kv[h], half));
            } else {
#pragma unroll
                for (int h = 0; h < kHid; ++h) zin[h] = E::add(y[h], E::mul(dt, kv[h]));
                step_done = true;
            }
        } else {
#pragma unroll
            for (int h = 0; h < kHid; ++h) zin[h] = E::add(y[h], E::mul(dt, kv[h]));
            step_done = true;
        }
        if (step_done) {
            while (next_out == step) {
                const int mode = a.out_mode[jn];
                if (mode == 0) write_out(jn, y);
                else if (mode == 1) write_out(jn, zin);
                else {
                    const float slope_w = a.out_slope[jn];
                    float v[kHid];
#pragma unroll
                    for (int h = 0; h < kHid; ++h) v[h] = E::add(y[h], E::mul(slope_w, E::sub(zin[h], y[h])));
                    write_out(jn, v);
                }
                ++jn;
                next_out = (jn < a.n_out) ? a.out_step[jn] : 0x7fffffff;
            }
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

}  // namespace tc

bool solve_tc_supported(int H, int C) { return H == tc::kHid && C == tc::kCh; }

template <int MODE> static int launch_tc(const UmmaArgs& a, cudaStream_t stream) {
    const int64_t grid = (a.n_paths + tc::kThreads - 1) / tc::kThreads;
    TCDE_CHECK_SUPPORTED(grid < (1ll << 31), "too many paths");
    auto kern = a.stage_dump ? tc::cdeint_tc_kernel<MODE, true> : tc::cdeint_tc_kernel<MODE, false>;
    const int smem = tc::Smem<MODE>::total + 128;             // slack for the 128-byte alignment of the tiles
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<(unsigned)grid, tc::kThreads, smem, stream>>>(a);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

int solve_tc_f32(const UmmaArgs& a, int H, int C, int mode, cudaStream_t stream) {
    TCDE_CHECK_SUPPORTED(solve_tc_supported(H, C), "tensor-core solve: built for hidden=32, channels=8 (got %d, %d)", H, C);
    TCDE_CHECK_SUPPORTED((reinterpret_cast<uintptr_t>(a.control) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.z0) & 15) == 0 &&
                             (reinterpret_cast<uintptr_t>(a.out) & 15) == 0,
                         "tensor-core solve: control, z0 and out must be 16-byte aligned");
    TCDE_CHECK_SUPPORTED(a.stage_dump == nullptr || (reinterpret_cast<uintptr_t>(a.stage_dump) & 15) == 0,
                         "tensor-core solve: the stage dump must be 16-byte aligned");
    // mode: bit 0 = operand split (0 = 3xTF32, 1 = 2xFP16)
    return (mode & 1) ? launch_tc<1>(a, stream) : launch_tc<0>(a, stream);
}

}  // namespace tcde
