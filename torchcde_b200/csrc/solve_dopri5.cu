// BASELINE config 4 (cdeint's default method): Dormand-Prince 5(4) with the step controller ON THE DEVICE.
//
// What the reference does here (torchcde/solver.py:226-227 -> torchdiffeq's adaptive solver, restated in
// torchcde_b200/adaptive.py): per attempted step six vector-field evaluations, ~60 elementwise launches, and one
// device->host read of the error ratio that decides accept / reject and the next step size.  Round 1 cut that to
// 6 field launches + 7 combination launches + 1 host read per attempt (0.95 s at 65,536 paths).
//
// Here ONE launch is one attempted step of the whole batch, and the host never reads anything per attempt:
//   * launch n first DECIDES attempt n-1: every CTA sums the per-CTA partial sums of squares that launch n-1 left
//     (fixed order => all CTAs agree bit for bit), forms the RMS error ratio over the WHOLE batch (torchdiffeq's norm
//     couples the batch, SURVEY 8e), accepts or rejects, and runs torchdiffeq's step-size rule in double precision.
//     The control block (t, dt, which state buffer is current, counters, done flag) is double buffered in global
//     memory: launch n reads slot (n-1)&1 and CTA 0 writes slot n&1.  The host enqueues launches blindly in chunks and
//     reads the done flag once per chunk; launches after the end are no-ops.
//   * on acceptance each thread evaluates torchdiffeq's 4th-order dense output for its own path at every requested
//     time inside the accepted step (y0, y1, y_mid, f0, f1 are all still in HBM / L2: the state is double buffered);
//   * then the attempt itself: the six new slopes k2..k7 (k1 is FSAL) through the same warp-level tensor-core field as the
//     fixed-step solve (tc_common.cuh: 2xFP16 split, each warp evaluates its own 32 paths); y, k1, k2/k6 live in
//     registers, k3..k5 in shared memory (k2's coefficient is zero in
//     the 5th-order weights, the error weights and the dense output, so k6 takes its registers); stage times ->
//     spline interval and fraction with the reference's bucketize semantics on the device; error partial sums of
//     (err / (atol + rtol max(|y0|, |y1|)))^2 in double; candidate (y1, k7) into the other state buffer.
//
// PAIRED mode (the backward pass of cdeint(adjoint=True) with dopri5, weight2 != NULL): the batch is a VIRTUAL batch of
// 2 n_ctrl paths -- paths [0, n_ctrl) carry the state z with (weight, bias), paths [n_ctrl, 2 n_ctrl) the adjoint state a
// with the regrouped, negated weight (for this linear field da/ds = a^T df/dz does not involve z: two linear CDEs that share
// the control and the step-size controller; the RMS error norm runs over both halves).  The parameter gradients
// dL/dW, dL/db = integral of (a (x) dX) (x) (z | 1) are NOT carried as a third state: g' does not depend on g, so
// integrating it with the same Runge-Kutta method is the quadrature  sum over accepted steps of dt * b_i * G(stage i) --
// every attempt leaves the inputs of its stages 1, 3, 4, 5, 6 (the non-zero b_i) in slot [number of accepted steps so far]
// of two trajectories (a rejected attempt is simply overwritten by the next one), the controller writes the accepted steps'
// quadrature nodes (spline interval, fraction, dt * b_i), and ONE launch of the parameter-gradient GEMM
// (tcde_linear_field_param_grads) contracts them afterwards.  (Not part of the error norm: in the host-driven adjoint the 8,448
// parameter-gradient components are 0.2 % of the packed state's RMS.)
#include "tc_common.cuh"

namespace tcde {

namespace dp5 {

using namespace tc;

constexpr int kRows = 128;                        // paths per tile
constexpr int kTiles = 2;
constexpr int kThreads = kRows * kTiles;          // 256: thread = path
constexpr int kCtl = 24;                          // doubles per control slot

// control slot fields (doubles; the integer ones hold exact small integers); the host side names them adaptive.CTL_*
enum { C_T = 0, C_DT, C_TEND, C_RTOL, C_ATOL, C_CUR, C_DONE, C_PENDING, C_NACC, C_NREJ, C_NEXT_OUT, C_NPART, C_NEED_MID, C_RATIO, C_LAUNCHES,
       C_OVERFLOW,     // paired mode: the trajectory slots are full -- the solve pauses (done = 1) until the caller has contracted them
       C_BASE };       // paired mode: accepted steps already contracted; slot of an attempt = accepted steps - base

__constant__ double c_alpha[6] = {1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9, 1.0, 1.0};
__constant__ double c_beta[6][6] = {
    {1.0 / 5, 0, 0, 0, 0, 0},
    {3.0 / 40, 9.0 / 40, 0, 0, 0, 0},
    {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0, 0},
    {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0, 0},
    {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656, 0},
    {35.0 / 384, 0.0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84},
};
__constant__ double c_err[7] = {35.0 / 384 - 1951.0 / 21600, 0.0, 500.0 / 1113 - 22642.0 / 50085, 125.0 / 192 - 451.0 / 720,
                                -2187.0 / 6784 - -12231.0 / 42400, 11.0 / 84 - 649.0 / 6300, -1.0 / 60.0};
__constant__ double c_mid[7] = {6025192743.0 / 30085553152.0 / 2, 0.0, 51252292925.0 / 65400821598.0 / 2, -2691868925.0 / 45128329728.0 / 2,
                                187940372067.0 / 1594534317056.0 / 2, -1776094331.0 / 19743644256.0 / 2, 11237099.0 / 235043384.0 / 2};

struct Args {
    const float* control;     // [n_paths][n_rows][4C] cubic rows or [n_paths][n_rows][C] linear slopes
    const float* knots;       // [n_rows + 1] in the coefficient dtype
    const float* weight;
    const float* bias;
    float* state;             // [5][n_paths][32]: Y0, Y1, F0, F1, MID
    double* partials;         // [2][grid]
    double* ctl;              // [2][kCtl]
    float* out;               // [n_paths][n_out][32]
    const double* out_times;  // [n_out], increasing (already negated for a decreasing t)
    int64_t n_paths, n_rows;
    int control_kind, n_out, seq;
    float sign;               // +1, or -1 for a decreasing t (the field is then -f(-s, y))
    // paired mode (all null / zero otherwise)
    const float* weight2;     // weights of the second half of the virtual batch
    const float* bias2;
    int64_t n_ctrl;           // paths of the control: n_paths, or n_paths / 2 in paired mode
    float* dump_z;            // [max_slots][5][n_ctrl][32]: stage inputs of the first half
    float* dump_a;            // ... of the second half
    int32_t* q_index;         // [max_slots * 5] quadrature nodes of the accepted steps
    float* q_frac;
    float* q_weight;
    int max_slots;
    // recording mode (the forward pass of cdeint(adjoint=False) with gradients; null otherwise): every attempt leaves its
    // step, its stage locations and the inputs of its six evaluations in slot [accepted steps so far - C_BASE]
    float* rec_z;             // [max_slots][6][n_paths][32]: inputs of stages 2..7 (stage 7's is the step's result y1); may be null
    double* rec_step;         // [max_slots][2]: (t, dt)
    int32_t* rec_index;       // [max_slots][6]: spline interval and fraction of stages 2..7
    float* rec_frac;
};

struct Smem {
    static constexpr int b = 0;                                   // operand B (W_hi | W_lo) + bias: tc_common.cuh
    static constexpr int a = (BSmem<1>::bytes + 127) & ~127;      // [kThreads / 32] per-warp operand scratch
    static constexpr int raw = a + (kThreads / 32) * WarpSmem<1>::bytes;   // [kTiles][6][128] float4
    static constexpr int park = raw + kTiles * 6 * kRows * 16;    // [kTiles][3][32][128] floats: k3, k4, k5
    static constexpr int misc = park + kTiles * 3 * kHid * kRows * 4;      // decision + coefficient tables
    static constexpr int total = misc + 1024;
};

// what thread 0 decides for the whole CTA (identically in every CTA)
struct Plan {
    double t, dt;             // the attempt of THIS launch starts at t with step dt
    double t_lo, t_hi, dt_old;  // the step accepted by this launch's decision (for the dense output)
    int cur;                  // state buffer holding (y, f) at t
    int idle;                 // nothing to do at all (the solve had finished before this launch)
    int done;                 // no attempt in this launch
    int emit_lo, emit_hi;     // output indices [emit_lo, emit_hi) fall inside the accepted step
    int old_cur;              // buffer that held the accepted step's start
    int need_mid;
    float cs[6][6];           // (float)(beta[s][j] * dt)
    float ce[7], cm[7];
    float stage_frac[6];
    int stage_index[6];
    float rtol, atol;
    int slot;                 // paired mode: trajectory slot of this attempt = accepted steps so far
};

// stage time -> (spline interval, fraction): the time in the state dtype, then the coefficient dtype (both float here), then
// bucketize - 1 (the reference's _interpret_t on the device)
__device__ __forceinline__ void locate_stage(const Args& a, double ti, int& idx, float& frac) {
    const float tk = (float)((double)a.sign * ti);
    int lo = 0, hi = (int)a.n_rows + 1;                    // lower_bound over knots[0 .. n_rows]
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.knots[mid] < tk) lo = mid + 1; else hi = mid;
    }
    idx = min(max(lo - 1, 0), (int)a.n_rows - 1);
    frac = tk - a.knots[idx];
}

__device__ __forceinline__ double next_step(double dt, double ratio) {           // adaptive._next_step
    if (ratio == 0.0) return dt * 10.0;
    double dfactor = 0.2;
    if (ratio < 1.0) dfactor = 1.0;
    const double f = 0.9 / pow(ratio, 0.2);
    return dt * fmin(10.0, fmax(f, dfactor));
}

// One launch of the solve.  RECORD: the recording mode (Args::rec_*); the kernels with RECORD = false are the plain and
// paired modes.
template <bool RECORD>
__device__ __forceinline__ void attempt(const Args& a) {
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((128u - (smem_u32(smem_unaligned) & 127u)) & 127u);
    Plan* plan = reinterpret_cast<Plan*>(smem + Smem::misc);
    double* cta_sums = reinterpret_cast<double*>(smem + Smem::misc + 896);
    const int tid = threadIdx.x, warp = tid >> 5;
    const int64_t n_elem = a.n_paths * kHid;
    const int64_t plane = n_elem;                     // floats per state buffer

    // ---- 1. decide the previous attempt, plan this one (thread 0; every CTA computes the same thing) ----------------
    if (tid == 0) {
        const double* in = a.ctl + ((a.seq + 1) & 1) * kCtl;
        double t = in[C_T], dt = in[C_DT];
        const double t_end = in[C_TEND], rtol = in[C_RTOL], atol = in[C_ATOL];
        int cur = (int)in[C_CUR], done = (int)in[C_DONE], pending = (int)in[C_PENDING];
        int nacc = (int)in[C_NACC], nrej = (int)in[C_NREJ], next_out = (int)in[C_NEXT_OUT];
        double ratio = in[C_RATIO];
        Plan p;
        p.idle = done;
        p.emit_lo = p.emit_hi = 0;
        p.t_lo = p.t_hi = t;
        p.dt_old = dt;
        p.old_cur = cur;
        if (!done && pending) {
            const double* part = a.partials + (size_t)((a.seq + 1) & 1) * gridDim.x;
            const int n_part = (int)in[C_NPART];
            double s = 0.0;
            for (int i = 0; i < n_part; ++i) s += part[i];
            ratio = sqrt(s / (double)n_elem);
            if (ratio <= 1.0) {
                p.t_lo = t;
                p.t_hi = t + dt;
                // paired mode clips the last step to the end of the segment (below): land on it exactly
                if (a.weight2 != nullptr && p.t_hi >= t_end - 1e-13 * fmax(1.0, fabs(t_end))) p.t_hi = t_end;
                p.old_cur = cur;
                cur ^= 1;
                const int slot_acc = nacc - (int)in[C_BASE];
                if (a.weight2 != nullptr && blockIdx.x == 0) {
                    // the accepted step's quadrature nodes for the parameter gradients: stages 1, 3, 4, 5, 6
                    const double cq[5] = {0.0, c_alpha[1], c_alpha[2], c_alpha[3], 1.0};
                    const int bq[5] = {0, 2, 3, 4, 5};
                    for (int k = 0; k < 5; ++k) {
                        int idx;
                        float fr;
                        locate_stage(a, (cq[k] == 1.0) ? t + dt : t + cq[k] * dt, idx, fr);
                        a.q_index[slot_acc * 5 + k] = idx;
                        a.q_frac[slot_acc * 5 + k] = fr;
                        a.q_weight[slot_acc * 5 + k] = (float)(c_beta[5][bq[k]] * dt);
                    }
                }
                ++nacc;
                p.emit_lo = next_out;
                while (next_out < a.n_out && a.out_times[next_out] <= p.t_hi) ++next_out;
                p.emit_hi = next_out;
                t = p.t_hi;
                if (next_out >= a.n_out) done = 1;
            } else {
                ++nrej;
            }
            dt = next_step(dt, ratio);
        }
        int overflow = (int)in[C_OVERFLOW];
        const int base = (int)in[C_BASE];
        if ((a.weight2 != nullptr || RECORD) && !done && nacc - base >= a.max_slots) {   // no trajectory slot left for another attempt
            overflow = 1;
            done = 1;
        }
        p.slot = nacc - base;
        // paired mode: the parameter gradients are a quadrature over WHOLE accepted steps, so the last step of a segment must end
        // at the segment's end instead of running past it and interpolating back (what the plain solve, like torchdiffeq, does)
        if (a.weight2 != nullptr && !done && t + dt > t_end) dt = t_end - t;
        p.t = t;
        p.dt = dt;
        p.cur = cur;
        p.done = done;
        p.need_mid = (!done && next_out < a.n_out && a.out_times[next_out] <= t + dt) ? 1 : 0;
        p.rtol = (float)rtol;
        p.atol = (float)atol;
        if (!done) {
            for (int s = 0; s < 6; ++s) {
                for (int j = 0; j < 6; ++j) p.cs[s][j] = (float)(c_beta[s][j] * dt);
                const double ti = (c_alpha[s] == 1.0) ? t + dt : t + c_alpha[s] * dt;
                locate_stage(a, ti, p.stage_index[s], p.stage_frac[s]);
                if (RECORD && blockIdx.x == 0) {
                    a.rec_index[p.slot * 6 + s] = p.stage_index[s];
                    a.rec_frac[p.slot * 6 + s] = p.stage_frac[s];
                }
            }
            if (RECORD && blockIdx.x == 0) {
                a.rec_step[2 * p.slot] = t;
                a.rec_step[2 * p.slot + 1] = dt;
            }
            for (int j = 0; j < 7; ++j) {
                p.ce[j] = (float)(c_err[j] * dt);
                p.cm[j] = (float)(c_mid[j] * dt);
            }
        }
        *plan = p;
        if (blockIdx.x == 0) {
            double* o = a.ctl + (a.seq & 1) * kCtl;
            o[C_T] = t; o[C_DT] = dt; o[C_TEND] = t_end; o[C_RTOL] = rtol; o[C_ATOL] = atol;
            o[C_CUR] = cur; o[C_DONE] = done; o[C_PENDING] = done ? 0 : 1; o[C_NACC] = nacc; o[C_NREJ] = nrej;
            o[C_NEXT_OUT] = next_out; o[C_NPART] = gridDim.x; o[C_NEED_MID] = p.need_mid; o[C_RATIO] = ratio;
            o[C_LAUNCHES] = in[C_LAUNCHES] + 1.0;
            o[C_OVERFLOW] = overflow;
            o[C_BASE] = base;
        }
    }
    __syncthreads();
    if (plan->idle) return;

    const int64_t n_pairs = (a.n_paths + kRows * kTiles - 1) / (kRows * kTiles);
    const int t_ = warp >> 2;                         // tile of this thread
    const int r = (warp & 3) * 32 + lane_row(tid & 31);   // its row in the tile: the row warp_field evaluates for this lane

    // ---- 2. dense output of the step that was just accepted, for the thread's own paths ---------------------------
    if (plan->emit_hi > plan->emit_lo) {
        const float* Y0 = a.state + (size_t)plan->old_cur * plane;
        const float* Y1 = a.state + (size_t)(plan->old_cur ^ 1) * plane;
        const float* F0 = a.state + (size_t)(2 + plan->old_cur) * plane;
        const float* F1 = a.state + (size_t)(2 + (plan->old_cur ^ 1)) * plane;
        const float* MID = a.state + (size_t)4 * plane;
        const float dtf = (float)plan->dt_old, two_dt = (float)(2.0 * plan->dt_old);
        for (int64_t pair = blockIdx.x; pair < n_pairs; pair += gridDim.x) {
            const int64_t path = (pair * kTiles + t_) * kRows + r;
            if (path >= a.n_paths) continue;
            for (int c4 = 0; c4 < 8; ++c4) {
                const float4 y0 = reinterpret_cast<const float4*>(Y0 + path * kHid)[c4];
                const float4 y1 = reinterpret_cast<const float4*>(Y1 + path * kHid)[c4];
                const float4 f0 = reinterpret_cast<const float4*>(F0 + path * kHid)[c4];
                const float4 f1 = reinterpret_cast<const float4*>(F1 + path * kHid)[c4];
                const float4 ym = reinterpret_cast<const float4*>(MID + path * kHid)[c4];
                const float y0v[4] = {y0.x, y0.y, y0.z, y0.w}, y1v[4] = {y1.x, y1.y, y1.z, y1.w};
                const float f0v[4] = {f0.x, f0.y, f0.z, f0.w}, f1v[4] = {f1.x, f1.y, f1.z, f1.w};
                const float ymv[4] = {ym.x, ym.y, ym.z, ym.w};
                float c1[4], c2[4], c3[4], c4v[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {           // adaptive.Dopri5._fit (torchdiffeq _interp_fit)
                    c4v[q] = two_dt * (f1v[q] - f0v[q]) - 8.f * (y1v[q] + y0v[q]) + 16.f * ymv[q];
                    c3[q] = dtf * (5.f * f0v[q] - 3.f * f1v[q]) + 18.f * y0v[q] + 14.f * y1v[q] - 32.f * ymv[q];
                    c2[q] = dtf * (f1v[q] - 4.f * f0v[q]) - 11.f * y0v[q] - 5.f * y1v[q] + 16.f * ymv[q];
                    c1[q] = dtf * f0v[q];
                }
                for (int j = plan->emit_lo; j < plan->emit_hi; ++j) {
                    const double x = (a.out_times[j] - plan->t_lo) / (plan->t_hi - plan->t_lo);
                    const float x1 = (float)x, x2 = (float)(x * x), x3 = (float)(x * x * x), x4 = (float)(x * x * x * x);
                    float v[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) v[q] = (((y0v[q] + x1 * c1[q]) + x2 * c2[q]) + x3 * c3[q]) + x4 * c4v[q];
                    reinterpret_cast<float4*>(a.out + (path * a.n_out + j) * kHid)[c4] = make_float4(v[0], v[1], v[2], v[3]);
                }
            }
        }
    }
    if (plan->done) return;

    // ---- 3. the attempt --------------------------------------------------------------------------------------------
    float inv_w_scale, beta;
    prepare_b<1>(smem + Smem::b, a.weight, a.bias, tid, kThreads, inv_w_scale, beta);
    __syncthreads();

    unsigned char* ws = smem + Smem::a + warp * WarpSmem<1>::bytes;
    float4* raw = reinterpret_cast<float4*>(smem + Smem::raw) + (size_t)t_ * 6 * kRows + r;
    float* park = reinterpret_cast<float*>(smem + Smem::park) + (size_t)t_ * 3 * kHid * kRows + r;      // [slot][h][row]
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * kCh : kCh;
    const float* Ycur = a.state + (size_t)plan->cur * plane;
    const float* Fcur = a.state + (size_t)(2 + plan->cur) * plane;
    float* Ynew = a.state + (size_t)(plan->cur ^ 1) * plane;
    float* Fnew = a.state + (size_t)(2 + (plan->cur ^ 1)) * plane;
    float* MID = a.state + (size_t)4 * plane;
    const float rtol = plan->rtol, atol = plan->atol, sign = a.sign;
    const bool need_mid = plan->need_mid != 0;
    double err_acc = 0.0;

    const bool paired = a.weight2 != nullptr;         // then n_ctrl is a multiple of 256: no partial tiles, no pair across the halves
    int cur_half = 0;
    for (int64_t pair = blockIdx.x; pair < n_pairs; pair += gridDim.x) {
        const int64_t path = (pair * kTiles + t_) * kRows + r;
        const bool tile_live = (pair * kTiles + t_) * kRows < a.n_paths;
        const int half = (paired && pair * kTiles * kRows >= a.n_ctrl) ? 1 : 0;
        if (half != cur_half) {                       // CTA-uniform: switch the operand B to the adjoint state's weights
            __syncthreads();                          // every warp is done reading the old weights
            prepare_b<1>(smem + Smem::b, a.weight2, a.bias2, tid, kThreads, inv_w_scale, beta);
            __syncthreads();
            cur_half = half;
        }
        if (!tile_live) continue;                     // whole tile beyond the batch: its four warps skip together
        const bool live = path < a.n_paths;
        const int64_t lpath = live ? path : a.n_paths - 1;
        const int64_t cpath = lpath - (half ? a.n_ctrl : 0);      // the control's path (both halves share it)
        const float* crow = a.control + cpath * a.n_rows * row_stride + (cubic ? kCh : 0);
        float* dump = paired ? (half ? a.dump_a : a.dump_z) + ((size_t)plan->slot * 5 * a.n_ctrl + cpath) * kHid : nullptr;
        auto dump_stage = [&](int k, const float* v) {           // input of quadrature stage k (0..4) of this attempt
            if (!paired) return;
            float4* dst = reinterpret_cast<float4*>(dump + (size_t)k * a.n_ctrl * kHid);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        };

        auto record_stage = [&](int k, const float* v) {         // input of stage k + 2 (0..5) of this attempt
            if (!RECORD || !live || a.rec_z == nullptr) return;
            float4* dst = reinterpret_cast<float4*>(a.rec_z + ((size_t)(plan->slot * 6 + k) * a.n_paths + path) * kHid);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        };

        auto fetch_row = [&](int idx) {
            const float* src = crow + (int64_t)idx * row_stride;
            const int parts = cubic ? 6 : 2;
            for (int j = 0; j < parts; ++j) cp_async16(&raw[j * kRows], src + 4 * j);
            cp_async_commit();
        };
        // one field evaluation: dX/dt of stage s, the next stage's row requested, then the tensor-core product + contraction
        auto evaluate = [&](const float* z, int s, float* kv, auto&& shadow) {
            cp_async_wait<0>();
            f2 dx2[kCh / 2];
            {
                const float4 b0 = raw[0], b1 = raw[kRows];
                if (cubic) {
                    const float4 c0 = raw[2 * kRows], c1 = raw[3 * kRows], d0 = raw[4 * kRows], d1 = raw[5 * kRows];
                    const float frac = plan->stage_frac[s];
                    const f2 fr = pk(frac, frac);
                    dx2[0] = add2(pk(b0.x, b0.y), mul2(add2(pk(c0.x, c0.y), mul2(pk(d0.x, d0.y), fr)), fr));
                    dx2[1] = add2(pk(b0.z, b0.w), mul2(add2(pk(c0.z, c0.w), mul2(pk(d0.z, d0.w), fr)), fr));
                    dx2[2] = add2(pk(b1.x, b1.y), mul2(add2(pk(c1.x, c1.y), mul2(pk(d1.x, d1.y), fr)), fr));
                    dx2[3] = add2(pk(b1.z, b1.w), mul2(add2(pk(c1.z, c1.w), mul2(pk(d1.z, d1.w), fr)), fr));
                } else {
                    dx2[0] = pk(b0.x, b0.y); dx2[1] = pk(b0.z, b0.w); dx2[2] = pk(b1.x, b1.y); dx2[3] = pk(b1.z, b1.w);
                }
                const f2 p2 = pk(sign, sign);
#pragma unroll
                for (int q = 0; q < 4; ++q) dx2[q] = mul2(dx2[q], p2);
            }
            float dx[kCh];
#pragma unroll
            for (int q = 0; q < 4; ++q) upk(dx2[q], dx[2 * q], dx[2 * q + 1]);
            if (s + 1 < 6) fetch_row(plan->stage_index[s + 1]);
            shadow();
            warp_field<1>(z, dx, kv, ws, smem + Smem::b, beta, inv_w_scale);
        };
        auto nothing = [] {};

        float y[kHid], k1[kHid], kA[kHid], kv[kHid];
        {
            const float4* yp = reinterpret_cast<const float4*>(Ycur + lpath * kHid);
            const float4* fp = reinterpret_cast<const float4*>(Fcur + lpath * kHid);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) {
                const float4 v = yp[c4], w = fp[c4];
                y[4 * c4] = v.x; y[4 * c4 + 1] = v.y; y[4 * c4 + 2] = v.z; y[4 * c4 + 3] = v.w;
                k1[4 * c4] = w.x; k1[4 * c4 + 1] = w.y; k1[4 * c4 + 2] = w.z; k1[4 * c4 + 3] = w.w;
            }
        }
        fetch_row(plan->stage_index[0]);
        dump_stage(0, y);

        // stage inputs y + sum_j c[s][j] k_j, fma in the order of adaptive._combine (zero weights skipped)
        // s = 0: k1
#pragma unroll
        for (int h = 0; h < kHid; ++h) kv[h] = fmaf(plan->cs[0][0], k1[h], y[h]);
        record_stage(0, kv);
        evaluate(kv, 0, kA, nothing);                                        // kA = k2
        // s = 1: k1, k2
#pragma unroll
        for (int h = 0; h < kHid; ++h) kv[h] = fmaf(plan->cs[1][1], kA[h], fmaf(plan->cs[1][0], k1[h], y[h]));
        dump_stage(1, kv);
        record_stage(1, kv);
        evaluate(kv, 1, kv, nothing);                                        // kv = k3
#pragma unroll
        for (int h = 0; h < kHid; ++h) park[(size_t)(0 * kHid + h) * kRows] = kv[h];
        // s = 2: k1, k2, k3
#pragma unroll
        for (int h = 0; h < kHid; ++h)
            kv[h] = fmaf(plan->cs[2][2], kv[h], fmaf(plan->cs[2][1], kA[h], fmaf(plan->cs[2][0], k1[h], y[h])));
        dump_stage(2, kv);
        record_stage(2, kv);
        evaluate(kv, 2, kv, nothing);                                        // kv = k4
#pragma unroll
        for (int h = 0; h < kHid; ++h) park[(size_t)(1 * kHid + h) * kRows] = kv[h];
        // s = 3: k1..k4
#pragma unroll
        for (int h = 0; h < kHid; ++h) {
            float v = fmaf(plan->cs[3][1], kA[h], fmaf(plan->cs[3][0], k1[h], y[h]));
            v = fmaf(plan->cs[3][2], park[(size_t)(0 * kHid + h) * kRows], v);
            kv[h] = fmaf(plan->cs[3][3], kv[h], v);
        }
        dump_stage(3, kv);
        record_stage(3, kv);
        evaluate(kv, 3, kv, nothing);                                        // kv = k5
#pragma unroll
        for (int h = 0; h < kHid; ++h) park[(size_t)(2 * kHid + h) * kRows] = kv[h];
        // s = 4: k1..k5
#pragma unroll
        for (int h = 0; h < kHid; ++h) {
            float v = fmaf(plan->cs[4][1], kA[h], fmaf(plan->cs[4][0], k1[h], y[h]));
            v = fmaf(plan->cs[4][2], park[(size_t)(0 * kHid + h) * kRows], v);
            v = fmaf(plan->cs[4][3], park[(size_t)(1 * kHid + h) * kRows], v);
            kv[h] = fmaf(plan->cs[4][4], kv[h], v);
        }
        dump_stage(4, kv);
        record_stage(4, kv);
        evaluate(kv, 4, kA, nothing);                                        // kA = k6 (k2 is not used again)
        // s = 5: the 5th-order solution y1 = y + dt (b1 k1 + b3 k3 + b4 k4 + b5 k5 + b6 k6); k7 = f(t + dt, y1)
        float y1[kHid];
#pragma unroll
        for (int h = 0; h < kHid; ++h) {
            float v = fmaf(plan->cs[5][0], k1[h], y[h]);
            v = fmaf(plan->cs[5][2], park[(size_t)(0 * kHid + h) * kRows], v);
            v = fmaf(plan->cs[5][3], park[(size_t)(1 * kHid + h) * kRows], v);
            v = fmaf(plan->cs[5][4], park[(size_t)(2 * kHid + h) * kRows], v);
            y1[h] = fmaf(plan->cs[5][5], kA[h], v);
        }
        record_stage(5, y1);
        float e6[kHid];                                   // error estimate without its k7 term, formed in the MMAs' shadow
        evaluate(y1, 5, kv, [&] {
            if (live) {
                float4* dst = reinterpret_cast<float4*>(Ynew + path * kHid);
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(y1[4 * c4], y1[4 * c4 + 1], y1[4 * c4 + 2], y1[4 * c4 + 3]);
            }
#pragma unroll
            for (int h = 0; h < kHid; ++h) {
                float v = plan->ce[0] * k1[h];                                        // fma(c, k, 0)
                v = fmaf(plan->ce[2], park[(size_t)(0 * kHid + h) * kRows], v);
                v = fmaf(plan->ce[3], park[(size_t)(1 * kHid + h) * kRows], v);
                v = fmaf(plan->ce[4], park[(size_t)(2 * kHid + h) * kRows], v);
                e6[h] = fmaf(plan->ce[5], kA[h], v);
            }
            if (need_mid) {                               // y_mid without its k7 term goes through k1's registers
#pragma unroll
                for (int h = 0; h < kHid; ++h) {
                    float v = fmaf(plan->cm[0], k1[h], y[h]);
                    v = fmaf(plan->cm[2], park[(size_t)(0 * kHid + h) * kRows], v);
                    v = fmaf(plan->cm[3], park[(size_t)(1 * kHid + h) * kRows], v);
                    v = fmaf(plan->cm[4], park[(size_t)(2 * kHid + h) * kRows], v);
                    k1[h] = fmaf(plan->cm[5], kA[h], v);
                }
            }
        });                                               // kv = k7
        if (live) {
            float4* dst = reinterpret_cast<float4*>(Fnew + path * kHid);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) dst[c4] = make_float4(kv[4 * c4], kv[4 * c4 + 1], kv[4 * c4 + 2], kv[4 * c4 + 3]);
            if (need_mid) {
                float4* md = reinterpret_cast<float4*>(MID + path * kHid);
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4)
                    md[c4] = make_float4(fmaf(plan->cm[6], kv[4 * c4], k1[4 * c4]), fmaf(plan->cm[6], kv[4 * c4 + 1], k1[4 * c4 + 1]),
                                         fmaf(plan->cm[6], kv[4 * c4 + 2], k1[4 * c4 + 2]), fmaf(plan->cm[6], kv[4 * c4 + 3], k1[4 * c4 + 3]));
            }
#pragma unroll
            for (int h = 0; h < kHid; ++h) {
                const float e = fmaf(plan->ce[6], kv[h], e6[h]);
                const float tol = atol + rtol * fmaxf(fabsf(y[h]), fabsf(y1[h]));
                const double q = (double)(e / tol);
                err_acc += q * q;
            }
        }
    }

    // ---- 4. this CTA's partial sum of squares (fixed order: lanes, then warps) ------------------------------------
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) err_acc += __shfl_down_sync(0xffffffffu, err_acc, off);
    if ((tid & 31) == 0) cta_sums[warp] = err_acc;
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += cta_sums[w];
        a.partials[(size_t)(a.seq & 1) * gridDim.x + blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(kThreads, 1) dopri5_attempt_kernel(const Args a) { attempt<false>(a); }
__global__ void __launch_bounds__(kThreads, 1) dopri5_record_kernel(const Args a) { attempt<true>(a); }

// ---- the backward pass of the recording mode: the transposed Dormand-Prince recurrence over the accepted steps --------
//
// For this linear field J = df/dz does not depend on z, so the cotangents need no forward state.  Per step n (last to
// first), with A the cotangent of y_{n+1} and K the cotangent still pending on the evaluation k7 of step n (= k1 of step
// n + 1, one evaluation under FSAL):
//   kappa7 = K + injections;  Zbar7 = A + J7^T kappa7 + injections;  then stages 6 .. 2: kappa_i = the accumulated cotangent
//   of k_i, Zbar_i = J_i^T kappa_i, and Zbar_i flows to y_n (weight 1) and to k_j, j < i (weight (float)(beta[i-2][j-1] dt));
//   the new A is the cotangent of y_n, the new K that of k1.
// The output cotangents enter through the transposed dense output (y_mid folded into y_n and the k_j on the host): weights
// [y_n, y_{n+1}, k1, k3, k4, k5, k6, k7] per (step, output).  kappa_i goes to item 6n + i - 2 of the record, the slot of its
// evaluation's input, for tcde_linear_field_param_grads.
struct BwdArgs {
    const float* control;
    const float* weight_t;    // [256][32] W with rows regrouped as (k, c): the field product with it is J^T
    const float* zeros;       // [256] zero bias
    const float* grad_out;    // [n_paths][n_out][32]
    float* carry;             // [2][n_paths][32]: (A, K) at step n_steps, replaced by (A, K) at step 0
    float* kappa;             // [n_steps][6][n_paths][32], or null
    const float* coef;        // [n_steps][36]: (float)(beta[s][j] dt_n), as the forward's Plan.cs
    const int32_t* stage_index;   // [n_steps][6]: the forward's stage locations
    const float* stage_frac;
    const int32_t* inj_range;     // [n_steps + 1]: injections of step n are [inj_range[n], inj_range[n + 1])
    const int32_t* inj_out;       // [n_inj]: output index
    const float* inj_w;           // [n_inj][8]
    int64_t n_paths, n_rows;
    int control_kind, n_out, n_steps;
    float sign;
};
enum { W_Y0 = 0, W_Y1, W_K1, W_K3, W_K4, W_K5, W_K6, W_K7 };

struct BwdSmem {
    static constexpr int b = 0;
    static constexpr int a = (BSmem<1>::bytes + 127) & ~127;
    static constexpr int park = a + (kThreads / 32) * WarpSmem<1>::bytes;   // [4][32][kThreads] floats: cotangents of k2..k5
    static constexpr int total = park + 4 * kHid * kThreads * 4;
};

__global__ void __launch_bounds__(kThreads, 1) dopri5_backward_kernel(const BwdArgs a) {
    extern __shared__ unsigned char smem_unaligned[];
    unsigned char* smem = smem_unaligned + ((128u - (smem_u32(smem_unaligned) & 127u)) & 127u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float inv_w_scale, beta;
    prepare_b<1>(smem + BwdSmem::b, a.weight_t, a.zeros, tid, kThreads, inv_w_scale, beta);
    __syncthreads();
    unsigned char* ws = smem + BwdSmem::a + warp * WarpSmem<1>::bytes;
    float* park = reinterpret_cast<float*>(smem + BwdSmem::park) + tid;          // cotangent of k_j: park[((j - 2) * 32 + h) * kThreads]
    const bool cubic = (a.control_kind == TCDE_CONTROL_CUBIC);
    const int row_stride = cubic ? 4 * kCh : kCh;
    const size_t item = (size_t)a.n_paths * kHid;

    for (int64_t w = (int64_t)blockIdx.x * (kThreads / 32) + warp; w * 32 < a.n_paths; w += (int64_t)gridDim.x * (kThreads / 32)) {
        const int64_t path = w * 32 + lane;
        const bool live = path < a.n_paths;
        const int64_t lpath = live ? path : a.n_paths - 1;
        const float* crow = a.control + lpath * a.n_rows * row_stride + (cubic ? kCh : 0);
        const float* grow = a.grad_out + lpath * a.n_out * kHid;

        // v = J^T v at stage location s of step n (every lane of the warp together)
        auto transposed = [&](int n, int s, float* v) {
            const int idx = a.stage_index[n * 6 + s];
            const float frac = a.stage_frac[n * 6 + s];
            const float4* src = reinterpret_cast<const float4*>(crow + (int64_t)idx * row_stride);
            float dx[kCh];
            if (cubic) {
                float r[24];
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const float4 q = src[j];
                    r[4 * j] = q.x; r[4 * j + 1] = q.y; r[4 * j + 2] = q.z; r[4 * j + 3] = q.w;
                }
#pragma unroll
                for (int c = 0; c < kCh; ++c)
                    dx[c] = __fmul_rn(__fadd_rn(r[c], __fmul_rn(__fadd_rn(r[8 + c], __fmul_rn(r[16 + c], frac)), frac)), a.sign);
            } else {
                const float4 q0 = src[0], q1 = src[1];
                dx[0] = q0.x * a.sign; dx[1] = q0.y * a.sign; dx[2] = q0.z * a.sign; dx[3] = q0.w * a.sign;
                dx[4] = q1.x * a.sign; dx[5] = q1.y * a.sign; dx[6] = q1.z * a.sign; dx[7] = q1.w * a.sign;
            }
            warp_field<1>(v, dx, v, ws, smem + BwdSmem::b, beta, inv_w_scale);
        };
        auto store = [&](float* dst, const float* v) {
            if (!live || dst == nullptr) return;
            float4* d = reinterpret_cast<float4*>(dst + path * kHid);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) d[c4] = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        };
        auto load = [&](const float* src, float* v) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) {
                const float4 q = s4[c4];
                v[4 * c4] = q.x; v[4 * c4 + 1] = q.y; v[4 * c4 + 2] = q.z; v[4 * c4 + 3] = q.w;
            }
        };

        float A[kHid], K[kHid], v[kHid];
        load(a.carry + lpath * kHid, A);
        load(a.carry + item + lpath * kHid, K);
        for (int n = a.n_steps - 1; n >= 0; --n) {
            const float* cs = a.coef + n * 36;
            float* kap = a.kappa;                                      // null: no parameter gradient wanted
            const int e0 = a.inj_range[n], e1 = a.inj_range[n + 1];
            // stage 7: kappa7 = K + injections, then Zbar7 = A + J7^T kappa7 + injections (in A)
#pragma unroll
            for (int h = 0; h < kHid; ++h) v[h] = K[h];
            for (int e = e0; e < e1; ++e) {
                float gv[kHid];
                load(grow + a.inj_out[e] * kHid, gv);
                const float wk = a.inj_w[8 * e + W_K7];
#pragma unroll
                for (int h = 0; h < kHid; ++h) v[h] = fmaf(wk, gv[h], v[h]);
            }
            store(kap ? kap + ((size_t)n * 6 + 5) * item : nullptr, v);
            transposed(n, 5, v);
#pragma unroll
            for (int h = 0; h < kHid; ++h) A[h] += v[h];
            for (int e = e0; e < e1; ++e) {
                float gv[kHid];
                load(grow + a.inj_out[e] * kHid, gv);
                const float wy = a.inj_w[8 * e + W_Y1];
#pragma unroll
                for (int h = 0; h < kHid; ++h) A[h] = fmaf(wy, gv[h], A[h]);
            }
            // Zbar7 -> y_n (K now holds ybar_n), k1 (v), k2..k5 (park), k6 (A)
#pragma unroll
            for (int h = 0; h < kHid; ++h) {
                K[h] = A[h];
                v[h] = cs[5 * 6 + 0] * A[h];
#pragma unroll
                for (int j = 2; j <= 5; ++j) park[((j - 2) * kHid + h) * kThreads] = cs[5 * 6 + j - 1] * A[h];
                A[h] = cs[5 * 6 + 5] * A[h];
            }
            for (int e = e0; e < e1; ++e) {
                float gv[kHid];
                load(grow + a.inj_out[e] * kHid, gv);
                const float* we = a.inj_w + 8 * e;
#pragma unroll
                for (int h = 0; h < kHid; ++h) {
                    K[h] = fmaf(we[W_Y0], gv[h], K[h]);
                    v[h] = fmaf(we[W_K1], gv[h], v[h]);
#pragma unroll
                    for (int j = 3; j <= 5; ++j)
                        park[((j - 2) * kHid + h) * kThreads] = fmaf(we[W_K3 + j - 3], gv[h], park[((j - 2) * kHid + h) * kThreads]);
                    A[h] = fmaf(we[W_K6], gv[h], A[h]);
                }
            }
            // stages 6 .. 2: A = kappa_i on entry
#pragma unroll
            for (int i = 6; i >= 2; --i) {
                store(kap ? kap + ((size_t)n * 6 + i - 2) * item : nullptr, A);
                transposed(n, i - 2, A);                                   // A = Zbar_i
                const float* c = cs + (i - 2) * 6;
#pragma unroll
                for (int h = 0; h < kHid; ++h) {
                    K[h] += A[h];
                    v[h] = fmaf(c[0], A[h], v[h]);
#pragma unroll
                    for (int j = 2; j <= i - 2; ++j)
                        park[((j - 2) * kHid + h) * kThreads] = fmaf(c[j - 1], A[h], park[((j - 2) * kHid + h) * kThreads]);
                    if (i > 2) A[h] = fmaf(c[i - 2], A[h], park[((i - 3) * kHid + h) * kThreads]);   // kappa_{i-1}
                }
            }
#pragma unroll
            for (int h = 0; h < kHid; ++h) {
                A[h] = K[h];
                K[h] = v[h];
            }
        }
        store(a.carry, A);
        store(a.carry + item, K);
    }
}

}  // namespace dp5

}  // namespace tcde

using namespace tcde;

extern "C" int tcde_dopri5_linear_grid(int64_t n_paths) {
    if (n_paths < 1) return -1;
    const int64_t pairs = (n_paths + dp5::kRows * dp5::kTiles - 1) / (dp5::kRows * dp5::kTiles);
    return (int)(pairs < sm_count() ? pairs : sm_count());
}

static int launch_attempts(dp5::Args a, int64_t first_seq, int64_t n_launches, cudaStream_t s,
                           void (*kernel)(const dp5::Args) = dp5::dopri5_attempt_kernel) {
    constexpr int smem = dp5::Smem::total + 1024;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = tcde_dopri5_linear_grid(a.n_paths);
    for (int64_t i = 0; i < n_launches; ++i) {
        a.seq = (int)((first_seq + i) & 0x3fffffff);
        kernel<<<grid, dp5::kThreads, smem, s>>>(a);
    }
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}

extern "C" int tcde_dopri5_linear_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                           const void* weight, const void* bias, void* state, void* partials, void* ctl,
                                           void* out, const void* out_times, int64_t n_out, int64_t n_paths, int64_t channels,
                                           int64_t hidden, double sign, int64_t first_seq, int64_t n_launches, int dtype,
                                           void* stream) {
    TCDE_CHECK_ARG(control && knots && weight && bias && state && partials && ctl && out && out_times, "null pointer");
    TCDE_CHECK_ARG(n_paths >= 1 && n_rows >= 1 && n_out >= 2 && n_launches >= 0 && first_seq >= 0, "bad sizes");
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d", control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == dp5::kHid && channels == dp5::kCh,
                         "device-controlled dopri5: built for float32, hidden=32, channels=8");
    TCDE_CHECK_SUPPORTED(((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                         "device-controlled dopri5: control, state and out must be 16-byte aligned");
    TCDE_CHECK_SUPPORTED(n_paths * 32 * 5 < (1ll << 40), "batch too large");
    dp5::Args a{(const float*)control, (const float*)knots, (const float*)weight, (const float*)bias, (float*)state,
                (double*)partials, (double*)ctl, (float*)out, (const double*)out_times, n_paths, n_rows, control_kind,
                (int)n_out, 0, (float)sign, nullptr, nullptr, n_paths, nullptr, nullptr, nullptr, nullptr, nullptr, 0};
    return launch_attempts(a, first_seq, n_launches, static_cast<cudaStream_t>(stream));
}

extern "C" int tcde_dopri5_linear_paired_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                                  const void* weight, const void* bias, const void* weight2, const void* bias2,
                                                  void* state, void* partials, void* ctl, void* out, const void* out_times,
                                                  int64_t n_out, int64_t n_ctrl, int64_t channels, int64_t hidden, double sign,
                                                  void* dump_z, void* dump_a, int32_t* q_index, void* q_frac, void* q_weight,
                                                  int64_t max_slots, int64_t first_seq, int64_t n_launches, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && knots && weight && bias && weight2 && bias2 && state && partials && ctl && out && out_times, "null pointer");
    TCDE_CHECK_ARG(dump_z && dump_a && q_index && q_frac && q_weight && max_slots >= 1 && max_slots < (1ll << 24), "null trajectory / bad slot count");
    TCDE_CHECK_ARG(n_ctrl >= 1 && n_rows >= 1 && n_out >= 2 && n_launches >= 0 && first_seq >= 0, "bad sizes");
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d", control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == dp5::kHid && channels == dp5::kCh,
                         "device-controlled dopri5: built for float32, hidden=32, channels=8");
    TCDE_CHECK_SUPPORTED(n_ctrl % (dp5::kRows * dp5::kTiles) == 0,
                         "device-controlled dopri5 adjoint: the batch (%lld paths) must be a multiple of %d", (long long)n_ctrl,
                         dp5::kRows * dp5::kTiles);
    TCDE_CHECK_SUPPORTED(((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(out) |
                           reinterpret_cast<uintptr_t>(dump_z) | reinterpret_cast<uintptr_t>(dump_a)) & 15) == 0,
                         "device-controlled dopri5: control, state, out and the trajectories must be 16-byte aligned");
    TCDE_CHECK_SUPPORTED(n_ctrl * 2 * 32 * 5 < (1ll << 40), "batch too large");
    dp5::Args a{(const float*)control, (const float*)knots, (const float*)weight, (const float*)bias, (float*)state,
                (double*)partials, (double*)ctl, (float*)out, (const double*)out_times, 2 * n_ctrl, n_rows, control_kind,
                (int)n_out, 0, (float)sign, (const float*)weight2, (const float*)bias2, n_ctrl, (float*)dump_z, (float*)dump_a,
                q_index, (float*)q_frac, (float*)q_weight, (int)max_slots};
    return launch_attempts(a, first_seq, n_launches, static_cast<cudaStream_t>(stream));
}

extern "C" int tcde_dopri5_linear_record_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                                  const void* weight, const void* bias, void* state, void* partials, void* ctl,
                                                  void* out, const void* out_times, int64_t n_out, int64_t n_paths,
                                                  int64_t channels, int64_t hidden, double sign, void* rec_z, void* rec_step,
                                                  int32_t* rec_index, void* rec_frac, int64_t max_slots, int64_t first_seq,
                                                  int64_t n_launches, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && knots && weight && bias && state && partials && ctl && out && out_times, "null pointer");
    TCDE_CHECK_ARG(rec_step && rec_index && rec_frac && max_slots >= 1 && max_slots < (1ll << 24), "null record / bad slot count");
    TCDE_CHECK_ARG(n_paths >= 1 && n_rows >= 1 && n_out >= 2 && n_launches >= 0 && first_seq >= 0, "bad sizes");
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d", control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == dp5::kHid && channels == dp5::kCh,
                         "device-controlled dopri5: built for float32, hidden=32, channels=8");
    TCDE_CHECK_SUPPORTED(((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(out) |
                           reinterpret_cast<uintptr_t>(rec_z)) & 15) == 0,
                         "device-controlled dopri5: control, state, out and the record must be 16-byte aligned");
    TCDE_CHECK_SUPPORTED(n_paths * 32 * 6 * max_slots < (1ll << 40), "record too large");
    dp5::Args a{(const float*)control, (const float*)knots, (const float*)weight, (const float*)bias, (float*)state,
                (double*)partials, (double*)ctl, (float*)out, (const double*)out_times, n_paths, n_rows, control_kind,
                (int)n_out, 0, (float)sign, nullptr, nullptr, n_paths, nullptr, nullptr, nullptr, nullptr, nullptr,
                (int)max_slots, (float*)rec_z, (double*)rec_step, rec_index, (float*)rec_frac};
    return launch_attempts(a, first_seq, n_launches, static_cast<cudaStream_t>(stream), dp5::dopri5_record_kernel);
}

extern "C" int tcde_dopri5_linear_backward(const void* control, int control_kind, int64_t n_rows, const void* weight_t,
                                           const void* zeros, const void* grad_out, void* carry, void* kappa, const void* coef,
                                           const int32_t* stage_index, const void* stage_frac, const int32_t* inj_range,
                                           const int32_t* inj_out, const void* inj_w, int64_t n_out, int64_t n_steps,
                                           int64_t n_paths, int64_t channels, int64_t hidden, double sign, int dtype,
                                           void* stream) {
    TCDE_CHECK_ARG(control && weight_t && zeros && grad_out && carry && coef && stage_index && stage_frac && inj_range &&
                   (inj_out || n_steps == 0) && inj_w, "null pointer");
    TCDE_CHECK_ARG(n_paths >= 1 && n_rows >= 1 && n_out >= 2 && n_steps >= 0 && n_steps < (1ll << 24), "bad sizes");
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d", control_kind);
    TCDE_CHECK_SUPPORTED(dtype == TCDE_F32 && hidden == dp5::kHid && channels == dp5::kCh,
                         "dopri5 backward: built for float32, hidden=32, channels=8");
    TCDE_CHECK_SUPPORTED(((reinterpret_cast<uintptr_t>(control) | reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(carry) |
                           reinterpret_cast<uintptr_t>(kappa)) & 15) == 0,
                         "dopri5 backward: control, grad_out, carry and kappa must be 16-byte aligned");
    if (n_steps == 0) return TCDE_OK;
    dp5::BwdArgs a{(const float*)control, (const float*)weight_t, (const float*)zeros, (const float*)grad_out, (float*)carry,
                   (float*)kappa, (const float*)coef, stage_index, (const float*)stage_frac, inj_range, inj_out,
                   (const float*)inj_w, n_paths, n_rows, control_kind, (int)n_out, (int)n_steps, (float)sign};
    constexpr int smem = dp5::BwdSmem::total + 1024;
    TCDE_CHECK_CUDA(cudaFuncSetAttribute(dp5::dopri5_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int64_t warps = (n_paths + 31) / 32;
    const int64_t blocks = (warps + dp5::kThreads / 32 - 1) / (dp5::kThreads / 32);
    const int grid = (int)(blocks < sm_count() ? blocks : sm_count());
    dp5::dopri5_backward_kernel<<<grid, dp5::kThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}
