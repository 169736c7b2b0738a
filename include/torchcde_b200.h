/*
 * torchcde_b200 -- C ABI of the H100-native Neural-CDE hot path.
 *
 * The reference (patrick-kidger/torchcde) is pure Python and has no FFI of its own; the
 * drop-in boundary is its Python API (SURVEY.md 8b).  This header is the boundary one level
 * below: the entry points the Python host layer (torchcde_b200/*.py) binds with ctypes, and
 * that a reference maintainer would bind the same way (INTEGRATION.md shows the stubs).
 * Each entry point names the reference function whose arithmetic it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types.  All data pointers are DEVICE
 *     pointers owned by the caller, contiguous, row-major.  Nothing is allocated inside.
 *   - `dtype`: TCDE_F32 or TCDE_F64 -- the dtype of every floating-point buffer of the call.
 *   - `stream`: a cudaStream_t passed as void* (NULL = legacy default stream).  Every call
 *     only enqueues work on that stream and returns; it never synchronises.
 *   - return value: TCDE_OK (0) or a negative tcde_status; tcde_last_error() gives the text
 *     of the last failure on the calling thread.  Nothing throws across the boundary.
 *   - a "series" is one scalar time series (one batch element, one channel); a "path" is one
 *     batch element with all its channels: x[n_paths][length][channels].
 *   - spline coefficient rows follow the reference layout (interpolation_cubic.py:297-305):
 *     coeffs[n_paths][length-1][4*channels] with row = [a | b | 2c | 3d].
 */
#ifndef TORCHCDE_B200_H
#define TORCHCDE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TCDE_ABI_VERSION 2

#if defined(__GNUC__)
#define TCDE_API __attribute__((visibility("default")))
#else
#define TCDE_API
#endif

enum tcde_dtype { TCDE_F32 = 0, TCDE_F64 = 1 };

enum tcde_status {
    TCDE_OK = 0,
    TCDE_ERR_ARGUMENT = -1,     /* null pointer, non-positive size, unknown enum */
    TCDE_ERR_UNSUPPORTED = -2,  /* shape outside what the kernels are built for (message says which) */
    TCDE_ERR_CUDA = -3          /* a CUDA runtime call failed (message carries cudaGetErrorString) */
};

enum tcde_control { TCDE_CONTROL_CUBIC = 0, TCDE_CONTROL_LINEAR = 1 };
enum tcde_method { TCDE_EULER = 0, TCDE_MIDPOINT = 1, TCDE_RK4_38 = 2, TCDE_REVERSIBLE_HEUN = 3 };

/* flag bits written by the builders into *flags (a device int32, may be NULL) */
#define TCDE_FLAG_NAN_SEEN 1        /* at least one NaN in x */
#define TCDE_FLAG_NAN_TIME 2        /* rectilinear: NaN in the time channel */
#define TCDE_FLAG_NAN_FIRST_ROW 4   /* rectilinear: NaN in the first row of some channel */

TCDE_API int tcde_abi_version(void);
TCDE_API const char* tcde_last_error(void);
/* number of SMs / compute capability of the current device; 0 on success */
TCDE_API int tcde_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- hot path (i): coefficient construction ------------------------------------------- */

/* hermite_cubic_coefficients_with_backward_differences on NaN-free knots
 * (interpolation_hermite_cubic_bdiff.py:5-44, after the linear fill at :33).
 * x[n_paths][length][channels] -> coeffs[n_paths][length-1][4*channels].
 * t: length knots, or NULL for the default 0,1,...,length-1 (misc.py:79-80).
 * Bit-identical to the reference's fp32/fp64 result at any channel count (rows too wide for one shared-memory tile
 * are split into channel tiles).  Sets TCDE_FLAG_NAN_SEEN if x holds a
 * NaN (the caller then runs tcde_linear_fill and calls again, as the reference does). */
TCDE_API int tcde_hermite_bdiff_coeffs(const void* x, const void* t, void* coeffs, int64_t n_paths, int64_t length,
                              int64_t channels, int dtype, int32_t* flags, void* stream);

/* hermite_cubic_coefficients_with_backward_differences of a series that MAY hold NaNs -- the whole reference function
 * (interpolation_hermite_cubic_bdiff.py:23-44: linear_interpolation_coeffs at :33, then the coefficients at :36-43) as ONE
 * launch: a warp holds a path in shared memory, fills its gaps in place (only if it has any) and writes the coefficient
 * rows; the filled series never goes to HBM and no flag has to reach the host to pick a branch.  Bit-identical to
 * tcde_linear_fill followed by tcde_hermite_bdiff_coeffs.  flags (optional): TCDE_FLAG_NAN_SEEN.
 * TCDE_ERR_UNSUPPORTED when a path does not fit a warp's tile (channels > 32, or length x channels beyond ~3,000
 * fp32 values): the caller runs the two kernels. */
TCDE_API int tcde_hermite_bdiff_coeffs_series(const void* x, const void* t, void* coeffs, int64_t n_paths, int64_t length,
                                     int64_t channels, int dtype, int32_t* flags, void* stream);

/* linear_interpolation_coeffs with missing values, per series
 * (interpolation_linear.py:13-84): all-NaN -> zeros; missing ends take the first / last
 * observation; interior gaps are interpolated in time.  x -> out, same shape.  Bit-identical.
 * flags (optional): TCDE_FLAG_NAN_SEEN is set when x held a NaN -- without it out is a copy of x and the
 * caller returns x itself like the reference (interpolation_linear.py:169-171), with no separate isnan pass. */
TCDE_API int tcde_linear_fill(const void* x, const void* t, void* out, int64_t n_paths, int64_t length,
                     int64_t channels, int dtype, int32_t* flags, void* stream);

/* torch.isnan(x).any() (the branch selector at interpolation_linear.py:169 and
 * interpolation_cubic.py:176) over n elements: sets TCDE_FLAG_NAN_SEEN in *flags. */
TCDE_API int tcde_nan_flag(const void* x, int64_t n, int dtype, int32_t* flags, void* stream);

/* misc.forward_fill along the length dim (misc.py:103-126); leading NaNs stay NaN.  length >= 1. */
TCDE_API int tcde_forward_fill(const void* x, void* out, int64_t n_paths, int64_t length, int64_t channels,
                      int dtype, int32_t* flags, void* stream);

/* _prepare_rectilinear_interpolation (interpolation_linear.py:87-128):
 * x[n_paths][length][channels] -> out[n_paths][2*length-1][channels].
 * Sets TCDE_FLAG_NAN_TIME / TCDE_FLAG_NAN_FIRST_ROW for the caller's assertion / warning. */
TCDE_API int tcde_rectilinear_prepare(const void* x, void* out, int64_t n_paths, int64_t length, int64_t channels,
                             int64_t time_index, int dtype, int32_t* flags, void* stream);

/* natural cubic spline on NaN-free knots (interpolation_cubic.py:7-53 + the Thomas solve of
 * misc.py:13-67).  workspace: device scratch of 4*length + 8 elements of `dtype` (the eliminated
 * diagonal, shared by every series, is formed once there).  fp tolerance: a few ulp (the
 * back-substitution multiplies by a reciprocal instead of dividing).  Sets
 * TCDE_FLAG_NAN_SEEN like the Hermite builder. */
TCDE_API int tcde_natural_cubic_coeffs(const void* x, const void* t, void* coeffs, void* workspace, int64_t n_paths,
                              int64_t length, int64_t channels, int dtype, int32_t* flags, void* stream);

/* natural cubic spline with missing values, per series (interpolation_cubic.py:56-167).
 * version 0 = natural_cubic_spline_coeffs (ends copied), 1 = natural_cubic_coeffs (ends
 * filled).  scratch: device memory of tcde_natural_cubic_missing_scratch_bytes() bytes. */
TCDE_API int64_t tcde_natural_cubic_missing_scratch_bytes(int64_t n_paths, int64_t length, int64_t channels, int dtype);
TCDE_API int tcde_natural_cubic_coeffs_missing(const void* x, const void* t, void* coeffs, void* scratch, int64_t n_paths,
                                      int64_t length, int64_t channels, int version, int dtype, void* stream);

/* ---- hot path (ii): spline evaluation and the fused fixed-step solve ------------------- */

/* CubicSpline.evaluate / .derivative (interpolation_cubic.py:324-336) or
 * LinearInterpolation.evaluate / .derivative (interpolation_linear.py:212-225) at n_times
 * query points whose interval index / fraction the host already located
 * (index[n_times] int32, frac[n_times]).  out[n_paths][n_times][channels].
 * control = coeffs (cubic) or knot values (linear, with knot_t[length]). */
TCDE_API int tcde_spline_eval(const void* control, const void* knot_t, const int32_t* index, const void* frac,
                     void* out, int64_t n_paths, int64_t n_rows, int64_t channels, int64_t n_times,
                     int control_kind, int derivative, int dtype, void* stream);

/* One evaluation of the CDE vector field for the README-form linear func
 * (solver.py:117-135 with func = Linear(H, H*C).view(H, C)):
 *   out[p][h] = sum_c (bias[h*C+c] + sum_k weight[h*C+c][k] z[p][k]) * dXdt[p][c]
 * with dXdt taken from the control at (index, frac).  Used by the adaptive driver. */
TCDE_API int tcde_vector_field_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                             const void* bias, const void* z, void* out, int64_t n_paths, int64_t channels,
                             int64_t hidden, int32_t index, double frac, int dtype, void* stream);

/* The same evaluation together with its vector-Jacobian products -- one stage of torchdiffeq's
 * odeint_adjoint (the reference's default, solver.py:144 and :226-227), which the stock stack gets
 * from autograd:
 *   f_out[p][h]        = f_scale * field as above
 *   vjp_z_out[p][k]    = vjp_scale * sum_h a[p][h] d f[p][h] / d z[p][k]
 *   grad_weight[n][k] += grad_scale * sum_p sum_h a[p][h] d f[p][h] / d weight[n][k]      (n = h*C + c)
 *   grad_bias[n]      += grad_scale * sum_p sum_h a[p][h] d f[p][h] / d bias[n]
 * (the scales carry the signs of the reversed-time solve and the Runge-Kutta weight of the stage, so a
 * fixed-step backward solve accumulates the parameter gradients in place).
 * grad_weight / grad_bias may be NULL.  scratch: device buffer of
 * tcde_vector_field_linear_vjp_scratch_bytes(...) bytes (per-CTA partial sums; -1 = shape not built).
 * Built for fp32, hidden = 32, channels = 8 (TCDE_ERR_UNSUPPORTED otherwise: the caller keeps autograd). */
TCDE_API int64_t tcde_vector_field_linear_vjp_scratch_bytes(int64_t n_paths, int64_t channels, int64_t hidden);
TCDE_API int tcde_vector_field_linear_vjp(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                 const void* bias, const void* z, const void* a, void* f_out, void* vjp_z_out,
                                 void* grad_weight, void* grad_bias, void* scratch, int64_t n_paths, int64_t channels,
                                 int64_t hidden, int32_t index, double frac, double f_scale, double vjp_scale,
                                 double grad_scale, int dtype, void* stream);

/* The fused fixed-step solve: everything torchdiffeq's fixed-grid odeint does for
 * cdeint(X, func, z0, t, method in {euler, midpoint, rk4}, options={step_size})
 * (solver.py:224-236; stepping restated in oracle/odeint_port.py) in ONE kernel launch:
 * spline derivative, linear vector field, f.dX/dt contraction, Runge-Kutta combination and
 * output interpolation, with the state in registers across all steps.
 *
 *   control      cubic: coeffs[n_paths][n_rows][4C];  linear: slopes[n_paths][n_rows][C]
 *   weight,bias  Linear(H, H*C): weight[H*C][H], bias[H*C]
 *   z0           [n_paths][H]
 *   out          [n_paths][n_out][H]      (time on dim -2, like solver.py:234-236)
 *   schedule (host-built with the reference's own torch ops, torchcde_b200/schedule.py):
 *     step_dt[n_steps]                     step width, already in the state dtype
 *     stage_index[n_steps][n_stages] int32 interval index of every stage time (bit-exact
 *                                          with CubicSpline._interpret_t), stage_frac same shape
 *     out_step[n_out] int32                step after which output j is produced (-1: j is z0)
 *     out_mode[n_out] int32                0 = copy step start, 1 = copy step end, 2 = interpolate
 *     out_slope[n_out]                     interpolation weight for mode 2
 *   sign         +1, or -1 for a decreasing t (field negated, torchdiffeq's time reversal)
 */
TCDE_API int tcde_cdeint_fixed_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                             const void* bias, const void* z0, void* out, int64_t n_paths, int64_t channels,
                             int64_t hidden, int method, int64_t n_steps, const void* step_dt,
                             const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                             const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                             double sign, int dtype, void* stream);

/* tcde_cdeint_fixed_linear that also stores the INPUT of every stage:
 * stage_dump[n_steps * n_stages][n_paths][hidden].  Served by the tensor-core kernel only (fp32, hidden = 32,
 * channels = 8, 16-byte aligned buffers; TCDE_ERR_UNSUPPORTED otherwise).  The backward solve of odeint_adjoint
 * uses it twice: for a linear field the adjoint state a obeys da/ds = a^T df/dz, which does not involve z, so
 * z(s) and a(s) are two ordinary solves (the second with the regrouped, negated weight and no bias). */
TCDE_API int tcde_cdeint_fixed_linear_stages(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                    const void* bias, const void* z0, void* out, void* stage_dump, int64_t n_paths,
                                    int64_t channels, int64_t hidden, int method, int64_t n_steps, const void* step_dt,
                                    const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                    const int32_t* out_step, const int32_t* out_mode, const void* out_slope,
                                    double sign, int dtype, void* stream);

/* The backward pass of tcde_cdeint_fixed_linear_stages through its own discrete operations (cdeint(..., adjoint=False) of a
 * fixed-step solve): the transposed Runge-Kutta recurrence of every step, in reverse, in ONE launch.  For the linear field
 * F_s(v) = sign (W v + b) . dX(t_s) the Jacobian J_s does not depend on v, so the forward state is never needed:
 *   rk4       kappa_4 = dt/8 ybar',  kappa_3 = dt (3/8 ybar' + u_4),  kappa_2 = dt (3/8 ybar' - u_4 + u_3),
 *             kappa_1 = dt (1/8 ybar' + u_4 - u_3/3 + u_2/3),  with u_s = J_s^T kappa_s;
 *   midpoint  kappa_2 = dt ybar',  kappa_1 = dt/2 u_2;      euler  kappa_1 = dt ybar';
 *   ybar = ybar' + sum_s u_s,
 * where ybar' is the cotangent of the step's end state after its output gradients were added.  J_s^T w = sign sum_c
 * dX_c(t_s) W_c^T w is the field product with weight_t[(k, c)][h] = weight[(h, c)][k] and the bias `zeros` (hidden *
 * channels zeros).
 *   grad_out     [n_paths][n_out][hidden] output gradients;  grad_z0 [n_paths][hidden] receives dL/dz0
 *   kappa_dump   (may be NULL) [n_steps * n_stages][n_paths][hidden] receives kappa of forward stage (i, s) in slot
 *                i * n_stages + s, the slot of that stage's input in the forward dump; tcde_linear_field_param_grads
 *                over the two dumps with stage_weight = sign gives dL/dW and dL/db
 *   step_dt_rev[n_steps], stage_index_rev / stage_frac_rev[n_steps * n_stages]: the forward schedule's arrays reversed
 *   inj_range[n_steps + 2], inj_out[], inj_weight[]: grid state r (r = 0 the end of the solve, r = n_steps z0) adds
 *                inj_weight[e] * grad_out[:, inj_out[e]] for e in [inj_range[r], inj_range[r + 1]) -- an output copied from
 *                a step's start or end lands there with weight 1, one interpolated at slope s lands on the start with
 *                1 - s and on the end with s
 * fp32, hidden = 32, channels = 8, 16-byte aligned buffers (TCDE_ERR_UNSUPPORTED otherwise); the field product is the
 * 2xFP16 warpgroup MMA of the fused solve. */
TCDE_API int tcde_cdeint_fixed_linear_backward(const void* control, int control_kind, int64_t n_rows, const void* weight_t,
                                      const void* zeros, const void* grad_out, void* grad_z0, void* kappa_dump,
                                      int64_t n_paths, int64_t channels, int64_t hidden, int method, int64_t n_steps,
                                      const void* step_dt_rev, const int32_t* stage_index_rev, const void* stage_frac_rev,
                                      int64_t n_out, const int32_t* inj_range, const int32_t* inj_out,
                                      const void* inj_weight, double sign, int dtype, void* stream);

/* The fused fixed-step solve of tcde_cdeint_fixed_linear for the MLP vector field of the reference's examples
 * (example/time_series_classification.py:20-51, func = Linear(H, W) -> ReLU -> Linear(W, H*C) -> tanh -> view(H, C)):
 *   f(t, z) = tanh(w2 relu(w1 z + b1) + b2).view(H, C) @ dX/dt(t)
 * in ONE launch, with the same control, schedule, output and sign arguments.
 *   w1, b1       Linear(H, W): w1[W][H], b1[W]         (`width` = W; a missing bias is a zero vector)
 *   w2, b2       Linear(W, H*C): w2[H*C][W], b2[H*C]
 * float32 runs the kernel that tcde_set_solve_variant selects: by default the tensor-core kernel (2xFP16 warpgroup MMA for
 * both products, accurate tanhf) at hidden = 32, channels = 8, width = 128 when control, z0 and out are 16-byte aligned,
 * else the CUDA-core kernel where it beats a stage loop (hidden <= 8 or hidden * channels <= 32; TCDE_ERR_UNSUPPORTED
 * elsewhere, so that the caller keeps its own loop); variant 1 the CUDA-core kernel at any shape it is built for;
 * variants 4 / 5 the tensor-core kernel or TCDE_ERR_UNSUPPORTED; variants 2 / 3 / 6 (3xTF32) TCDE_ERR_UNSUPPORTED.
 * float64 runs the CUDA-core kernel, by default at the same shapes and with variant 1 at any.  The
 * CUDA-core kernel takes hidden <= 32 and any width (weights in shared memory when they fit, else read from global
 * memory) and channels whose per-path scratch (C + H values) fits its shared memory; TCDE_ERR_UNSUPPORTED otherwise. */
TCDE_API int tcde_cdeint_fixed_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                          const void* w2, const void* b2, const void* z0, void* out, int64_t n_paths, int64_t channels,
                          int64_t hidden, int64_t width, int method, int64_t n_steps, const void* step_dt,
                          const int32_t* stage_index, const void* stage_frac, int64_t n_out, const int32_t* out_step,
                          const int32_t* out_mode, const void* out_slope, double sign, int dtype, void* stream);

/* tcde_cdeint_fixed_mlp that also stores the INPUT of every stage: stage_dump[n_steps * n_stages][n_paths][hidden] (the
 * forward state of tcde_cdeint_fixed_mlp_backward).  The outputs equal tcde_cdeint_fixed_mlp's bit for bit.  Served by the
 * tensor-core kernel at fp32, hidden = 32, channels = 8, width = 128 with 16-byte aligned control, z0, out and dump under
 * solve variant 0, 4 or 5, and by the CUDA-core kernel (fp32 or fp64, any alignment) at hidden <= 8 under solve variant
 * 0 or 1, and under variant 1 also at hidden * channels <= 32 (the other shapes where tcde_cdeint_fixed_mlp runs it by
 * default; by default they are refused because the backward there is slower than a stage loop); TCDE_ERR_UNSUPPORTED
 * otherwise. */
TCDE_API int tcde_cdeint_fixed_mlp_stages(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                 const void* b1, const void* w2, const void* b2, const void* z0, void* out,
                                 void* stage_dump, int64_t n_paths, int64_t channels, int64_t hidden, int64_t width,
                                 int method, int64_t n_steps, const void* step_dt, const int32_t* stage_index,
                                 const void* stage_frac, int64_t n_out, const int32_t* out_step, const int32_t* out_mode,
                                 const void* out_slope, double sign, int dtype, void* stream);

/* The backward pass of tcde_cdeint_fixed_mlp_stages through its own discrete operations (cdeint(..., adjoint=False)): the
 * transposed Runge-Kutta recurrence of tcde_cdeint_fixed_linear_backward (same kappa / ybar formulas, reversed schedule
 * arrays and output-gradient lists inj_*) in ONE launch, with the stage product of the MLP field at the forward's stage
 * input z_s (stage_dump, read from the last slot down):
 *   u_s = J_s^T kappa_s = W1^T (mask . W2^T g),  g[(h, c)] = (1 - y^2)[(h, c)] kappa_s[h] sign dX_c(t_s),
 *   y = tanh(W2 h + b2),  h = relu(W1 z_s + b1),  mask = (h > 0)
 * (h and y recomputed by the forward's own code, so the mask and tanh values are the forward's bits).  grad_z0
 * [n_paths][hidden] receives dL/dz0; kappa_dump (may be NULL) [n_steps * n_stages][n_paths][hidden] receives kappa_s in the
 * slot of stage s's input in stage_dump, for tcde_mlp_field_param_grads.  Same support as tcde_cdeint_fixed_mlp_stages
 * (on the tensor-core kernel, grad_out and grad_z0 16-byte aligned too). */
TCDE_API int tcde_cdeint_fixed_mlp_backward(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                   const void* b1, const void* w2, const void* b2, const void* stage_dump,
                                   const void* grad_out, void* grad_z0, void* kappa_dump, int64_t n_paths, int64_t channels,
                                   int64_t hidden, int64_t width, int method, int64_t n_steps, const void* step_dt_rev,
                                   const int32_t* stage_index_rev, const void* stage_frac_rev, int64_t n_out,
                                   const int32_t* inj_range, const int32_t* inj_out, const void* inj_weight, double sign,
                                   int dtype, void* stream);

/* The parameter gradients of tcde_cdeint_fixed_mlp_backward from its two dumps (z_stages = the forward's stage inputs,
 * kappa_stages = the backward's kappa, both [n_stages_total][n_paths][hidden]):
 *   grad_w2 += scale sum g h^T,  grad_b2 += scale sum g,  grad_w1 += scale sum ubar z^T,  grad_b1 += scale sum ubar
 * over every (stage, path), with g and ubar = mask . W2^T g recomputed as the backward forms them (dX/dt from the control at
 * (stage_index[e], stage_frac[e]) times `sign`).  Any gradient pointer may be NULL.  Tensor cores (2xBF16 split) at
 * 32 / 8 / 128, the CUDA cores at the CUDA-core shapes; a fixed-order reduction: two calls give the same bits.  Same
 * support as tcde_cdeint_fixed_mlp_stages, except that a CUDA-core width whose staging does not fit shared memory is
 * refused; scratch of tcde_mlp_field_param_grads_scratch_bytes (-1: not built for the shape; it has no dtype argument, so
 * at the CUDA-core shapes it is the size for 8-byte elements). */
TCDE_API int64_t tcde_mlp_field_param_grads_scratch_bytes(int64_t n_paths, int64_t n_stages_total, int64_t channels,
                                                 int64_t hidden, int64_t width);
TCDE_API int tcde_mlp_field_param_grads(const void* control, int control_kind, int64_t n_rows, const void* w1,
                               const void* b1, const void* w2, const void* b2, const void* z_stages,
                               const void* kappa_stages, const int32_t* stage_index, const void* stage_frac,
                               int64_t n_stages_total, void* grad_w1, void* grad_b1, void* grad_w2, void* grad_b2,
                               void* scratch, int64_t n_paths, int64_t channels, int64_t hidden, int64_t width,
                               double sign, double scale, int dtype, void* stream);

/* One evaluation of the MLP vector field of tcde_cdeint_fixed_mlp at one time, for an adaptive driver (the counterpart of
 * tcde_vector_field_linear):
 *   out[p][h] = sum_c tanh(w2 relu(w1 z[p] + b1) + b2)[h*C+c] * dXdt[p][c]
 * with dXdt from the control at (index, frac), in the CUDA-core solve's arithmetic.  Built where the CUDA-core kernels
 * of tcde_cdeint_fixed_mlp_stages run (fp32 or fp64; hidden <= 8, and under solve variant 1 also hidden * channels <= 32;
 * widths whose parameter-gradient staging fits shared memory).  By default served only at fp32 with hidden * channels
 * <= 32 and width <= 128, where an adjoint=True training step on them measured faster than autograd per stage; solve
 * variant 1 forces the rest.  TCDE_ERR_UNSUPPORTED elsewhere, the tensor-core shape fp32 32 / 8 / 128 included, so that
 * the caller keeps its torch-operator field. */
TCDE_API int tcde_vector_field_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                          const void* w2, const void* b2, const void* z, void* out, int64_t n_paths, int64_t channels,
                          int64_t hidden, int64_t width, int32_t index, double frac, int dtype, void* stream);

/* The same evaluation together with its vector-Jacobian products -- one stage of the adjoint backward solve, with the
 * scale convention of tcde_vector_field_linear_vjp:
 *   f_out      = f_scale * f                        vjp_z_out = vjp_scale * a^T df/dz
 *   grad_w1 += grad_scale * sum_p a^T df/dw1, and likewise grad_b1, grad_w2, grad_b2 (each may be NULL)
 * At most three launches: the field and a^T df/dz in one pass (f_out equals tcde_vector_field_mlp's out bit for bit at
 * f_scale = 1), then, with a parameter gradient, the parameter-gradient kernel of tcde_mlp_field_param_grads over this
 * one stage and its fixed-order reduction (two calls give the same bits).  scratch: 16-byte aligned device buffer of
 * tcde_vector_field_mlp_vjp_scratch_bytes(...) bytes (-1: the shape is not served at fp32; the query has no dtype, the
 * size fits both, and a call with n_paths = 0 gives the verdict for a dtype).  Same support as tcde_vector_field_mlp. */
TCDE_API int64_t tcde_vector_field_mlp_vjp_scratch_bytes(int64_t n_paths, int64_t channels, int64_t hidden,
                                                int64_t width);
TCDE_API int tcde_vector_field_mlp_vjp(const void* control, int control_kind, int64_t n_rows, const void* w1,
                              const void* b1, const void* w2, const void* b2, const void* z, const void* a, void* f_out,
                              void* vjp_z_out, void* grad_w1, void* grad_b1, void* grad_w2, void* grad_b2, void* scratch,
                              int64_t n_paths, int64_t channels, int64_t hidden, int64_t width, int32_t index,
                              double frac, double f_scale, double vjp_scale, double grad_scale, int dtype,
                              void* stream);

/* torchsde's reversible Heun method with zero diffusion (cdeint(..., backend="torchsde", method="reversible_heun")) for
 * the same linear field, in ONE launch:
 *   z_{n+1} = 2 y_n - z_n + f_n dt_n,  f_{n+1} = f(t_{n+1}, z_{n+1}),  y_{n+1} = y_n + (f_n + f_{n+1}) (0.5 dt_n)
 * starting from z_0 = y_0, f_0 = f(t_0, y_0).  float32 runs the kernel that tcde_set_solve_variant selects, as
 * tcde_cdeint_fixed_linear does: by default the tensor-core kernel with the 2xFP16 split (warpgroup MMA) at hidden =
 * 32, channels = 8 when control, z0, out and checkpoints are 16-byte aligned, else the CUDA-core kernel; variant 3 the
 * 3xTF32 tensor-core kernel; variant 1 the CUDA-core kernel.  float64 runs the CUDA-core kernel, at any shape whose
 * weights fit its shared memory.  Schedule (torchcde_b200/schedule.py, build_sde_schedule):
 *   step_dt[n_steps]; stage_index / stage_frac[n_steps + 1]: the evaluation points t_0 .. t_N;
 *   out_step[n_out] (-1: output j is y_0); out_weights[2][n_out]: w1 of every output, then w0, and output j is
 *   w0 y_n + w1 y_{n+1} of its step n (torchsde's linear_interp).
 * checkpoints (may be NULL): [ceil(n_steps / checkpoint_stride) + 1][3][n_paths][hidden] receives (y, z, f) of every step
 * that is a multiple of checkpoint_stride and of the last step -- the restart points of the reversible backward. */
TCDE_API int tcde_cdeint_reversible_heun_linear(const void* control, int control_kind, int64_t n_rows, const void* weight,
                                       const void* bias, const void* z0, void* out, void* checkpoints,
                                       int64_t checkpoint_stride, int64_t n_paths, int64_t channels, int64_t hidden,
                                       int64_t n_steps, const void* step_dt, const int32_t* stage_index,
                                       const void* stage_frac, int64_t n_out, const int32_t* out_step,
                                       const void* out_weights, int dtype, void* stream);

/* One checkpoint segment [lo, hi] of the reversible Heun backward (fp32, hidden = 32, channels = 8), in one launch: walks the
 * steps m = hi - 1 .. lo in reverse, reconstructing z_m, f_m = F(z_m), y_m algebraically from step m + 1 (the state of step lo
 * is taken from its checkpoint), running the adjoint recurrence of (y, z, f) and adding the output gradients
 * g[n_paths][n_out][hidden] (inj_range[N + 1][2]: the outputs [first, end) that touch y_m; weight w0 when out_step == m,
 * 1 when out_step < 0, w1 otherwise).  J_F^T fbar is the same field product with weight_t[(k, c)][h] = weight[(h, c)][k] and
 * the bias `zeros` (256 zeros).  ckpt_lo / ckpt_hi: [3][n_paths][hidden] (y, z, f) of steps lo and hi; carry [2][n_paths]
 * [hidden]: (ybar, zbar) of step hi in, of step lo out.  dump_z / dump_a [hi - lo][n_paths][hidden] receive (z_m, fbar_m)
 * for tcde_linear_field_param_grads (weights 1) to contract into dL/dW, dL/db. */
TCDE_API int tcde_reversible_heun_linear_backward_segment(
    const void* control, int control_kind, int64_t n_rows, const void* weight, const void* bias, const void* weight_t,
    const void* zeros, const void* ckpt_lo, const void* ckpt_hi, void* carry, const void* g, int64_t n_out,
    const int32_t* out_step, const void* out_weights, const int32_t* inj_range, const void* step_dt,
    const int32_t* stage_index, const void* stage_frac, int64_t lo, int64_t hi, int64_t n_paths, int64_t channels,
    int64_t hidden, void* dump_z, void* dump_a, int dtype, void* stream);

/* torchsde's reversible Heun method (as tcde_cdeint_reversible_heun_linear: the same step, schedule, output weights and
 * checkpoint layout) for the MLP vector field of tcde_cdeint_fixed_mlp, in ONE launch on the CUDA cores (one thread per
 * path, the field in the arithmetic of the fixed-step CUDA-core solve; fp32 or fp64):
 *   z_{n+1} = 2 y_n - z_n + f_n dt_n,  f_{n+1} = F(t_{n+1}, z_{n+1}),  y_{n+1} = y_n + (f_n + f_{n+1}) (0.5 dt_n)
 * from z_0 = y_0, f_0 = F(t_0, y_0), one rounding per operation.  checkpoints (may be NULL):
 * [ceil(n_steps / checkpoint_stride) + 1][3][n_paths][hidden] receives (y, z, f) of every step that is a multiple of
 * checkpoint_stride and of the last step.  Served at the CUDA-core shapes of tcde_cdeint_fixed_mlp_stages: by default
 * hidden <= 8 with hidden * channels <= 32 (fp32 and fp64; where a training step on it measured faster than per-step
 * autograd), under solve variant 1 every hidden * channels <= 32 or hidden <= 8; widths whose parameter-gradient staging
 * fits shared memory.  TCDE_ERR_UNSUPPORTED elsewhere (the tensor-core shape 32 / 8 / 128 and solve variant 4 included),
 * so that the caller keeps its own solve. */
TCDE_API int tcde_cdeint_reversible_heun_mlp(const void* control, int control_kind, int64_t n_rows, const void* w1,
                                    const void* b1, const void* w2, const void* b2, const void* z0, void* out,
                                    void* checkpoints, int64_t checkpoint_stride, int64_t n_paths, int64_t channels,
                                    int64_t hidden, int64_t width, int64_t n_steps, const void* step_dt,
                                    const int32_t* stage_index, const void* stage_frac, int64_t n_out,
                                    const int32_t* out_step, const void* out_weights, int dtype, void* stream);

/* One checkpoint segment [lo, hi] of the reversible Heun backward of tcde_cdeint_reversible_heun_mlp, in one launch (one
 * thread per path): the recurrence of tcde_reversible_heun_linear_backward_segment (same ckpt_lo / ckpt_hi, carry, g,
 * out_step, out_weights, inj_range and schedule arrays) with one pass of the field's vector-Jacobian product per step at
 * the reconstructed z_m, which gives f_m = F(z_m) (the forward's bits) and J_F(z_m)^T fbar_m together.  When hi == n_steps
 * the launch first closes step N: ybar_N = the output gradients on y_N, fbar_N = ybar_N dt_{N-1} / 2, zbar_N =
 * J_F(z_N)^T fbar_N (carry is not read).  dump_z / dump_a [hi - lo + (hi == n_steps)][n_paths][hidden] receive (z_m,
 * fbar_m) in slot m - lo, step N in the last slot: tcde_mlp_field_param_grads over them (stage_index / stage_frac offset
 * by lo, n_stages_total = the dump's length, sign and scale 1) adds dL/dW1, db1, dW2, db2.  Same support as
 * tcde_cdeint_reversible_heun_mlp. */
TCDE_API int tcde_reversible_heun_mlp_backward_segment(
    const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1, const void* w2, const void* b2,
    const void* ckpt_lo, const void* ckpt_hi, void* carry, const void* g, int64_t n_out, const int32_t* out_step,
    const void* out_weights, const int32_t* inj_range, int64_t n_steps, const void* step_dt, const int32_t* stage_index,
    const void* stage_frac, int64_t lo, int64_t hi, int64_t n_paths, int64_t channels, int64_t hidden, int64_t width,
    void* dump_z, void* dump_a, int dtype, void* stream);

/* The backward pass of cdeint(adjoint=False) with dopri5 for the MLP field of tcde_cdeint_fixed_mlp, over one record chunk
 * of a host-driven solve, its n_steps accepted steps last to first, in ONE launch (one thread per path, fp32 or fp64): the
 * transposed Dormand-Prince recurrence of tcde_dopri5_linear_backward, with J^T of every evaluation formed at its recorded
 * input (the forward's ReLU masks and tanh values).
 *   rec_z     [n_items][n_paths][hidden]: the inputs of the chunk's evaluations, n_items = step_item[n_steps]; the items
 *             of step n are [step_item[n], step_item[n + 1]): stages 2..7 (stage 7's input is the step's result), preceded
 *             by the step's own start slope f(t_n, y_n) when k1 of step n is not the previous step's k7 (step 0 of the
 *             solve, and the step after a jump of jump_t): 7 items then, 6 otherwise
 *   item_index int32 / item_frac [n_items]: the spline interval and fraction of every evaluation
 *   grad_out  [n_paths][n_out][hidden]: dL/d(outputs)
 *   carry     [2][n_paths][hidden]: in, the cotangent of the state after the chunk's last step and the cotangent still
 *             pending on that step's last evaluation (zero for the last chunk); out, the same before the chunk's first step
 *             (the second is zero when that step's start slope was its own evaluation)
 *   kappa     [n_items][n_paths][hidden] or NULL: the cotangent of every evaluation, in its item, for
 *             tcde_mlp_field_param_grads (item_index / item_frac, n_items, sign = the solve's, scale 1)
 *   coef      [n_steps][36]: beta[s][j] dt of the Dormand-Prince tableau in the state dtype, rows s = 0..5, zero padded
 *   inj_range int32 [n_steps + 1], inj_out int32 [n_inj], inj_w [n_inj][8]: as tcde_dopri5_linear_backward's, in the state
 *             dtype
 *   sign      +1, or -1 for a decreasing t solved in -t (dX/dt is negated)
 * Served where tcde_cdeint_fixed_mlp_stages runs the CUDA cores (by default hidden <= 8, fp32 and fp64; under solve variant 1
 * also hidden * channels <= 32) at widths whose columns fit shared memory; TCDE_ERR_UNSUPPORTED elsewhere, the tensor-core
 * shape 32 / 8 / 128 included.  n_paths == 0 validates the problem and launches nothing. */
TCDE_API int tcde_dopri5_mlp_backward(const void* control, int control_kind, int64_t n_rows, const void* w1, const void* b1,
                             const void* w2, const void* b2, const void* rec_z, const void* grad_out, void* carry,
                             void* kappa, const void* coef, const int32_t* step_item, const int32_t* item_index,
                             const void* item_frac, const int32_t* inj_range, const int32_t* inj_out, const void* inj_w,
                             int64_t n_out, int64_t n_steps, int64_t n_paths, int64_t channels, int64_t hidden,
                             int64_t width, double sign, int dtype, void* stream);

/* The parameter gradients of a whole backward solve (the stage trajectories of tcde_cdeint_fixed_linear_stages, or any
 * other list of (z, a, stage) triples) in one launch:
 *   grad_weight[h*C+c][k] += scale * sum_e sum_p stage_weight[e] * a_stages[e][p][h] * dXdt_e[p][c] * z_stages[e][p][k]
 *   grad_bias[h*C+c]      += scale * sum_e sum_p stage_weight[e] * a_stages[e][p][h] * dXdt_e[p][c]
 * with dXdt_e from the control at (stage_index[e], stage_frac[e]) and stage_weight[e] = step * Runge-Kutta weight
 * (device arrays of length n_stages_total).  fp32, hidden = 32, channels = 8. */
TCDE_API int64_t tcde_linear_field_param_grads_scratch_bytes(int64_t n_paths, int64_t n_stages_total, int64_t channels,
                                                    int64_t hidden);
TCDE_API int tcde_linear_field_param_grads(const void* control, int control_kind, int64_t n_rows, const void* z_stages,
                                  const void* a_stages, const int32_t* stage_index, const void* stage_frac,
                                  const void* stage_weight, int64_t n_stages_total, void* grad_weight, void* grad_bias,
                                  void* scratch, int64_t n_paths, int64_t channels, int64_t hidden, double scale,
                                  int dtype, void* stream);

/* Elementwise pieces of the adaptive driver that stands in for torchdiffeq's dopri5 (the reference's default
 * method, solver.py:226-227): out[i] = base[i] + sum_j coefs[j] * terms[j][i]  (base may be NULL; at most 7
 * terms; `terms` / `coefs` are HOST arrays of device pointers / doubles, read at launch; out may alias base). */
TCDE_API int tcde_linear_combination(void* out, const void* base, const void* const* terms, const double* coefs,
                            int n_terms, int64_t n, int dtype, void* stream);

/* The contraction that closes _VectorField.forward for an arbitrary func (solver.py:129-135):
 * out[p][h] = scale * sum_c field[p][h][c] * dx[p * dx_stride + c]   (field [n_paths][hidden][channels] contiguous, out
 * [n_paths][hidden]; dx may be a strided view, e.g. one stage of the per-step dX/dt block; scale = -1 for reversed time).
 * torch.matmul runs this as a batched cuBLAS kernel at ~100 GB/s; streamed it is HBM bound. */
TCDE_API int tcde_field_contract(const void* field, const void* dx, void* out, int64_t n_paths, int64_t hidden, int64_t channels,
                        int64_t dx_stride, double scale, int dtype, void* stream);

/* Grouped forms of tcde_spline_eval and tcde_field_contract for the members of a TupleControl (misc.py:129-166) and a
 * tuple state (solver.py:131-133): one launch serves every member, each with its own sizes and pointers, and every
 * output element is bit-equal to the single-member entry's on that member alone.  `members` is a HOST array read at
 * launch; up to 16 members go in one launch, a longer list is launched in chunks of 16.  A member with no output
 * elements may carry NULL pointers.  All members share `dtype` (and, for the evaluation, `derivative`). */
typedef struct tcde_spline_member {
    const void* control;       /* as tcde_spline_eval: rows [n_paths][n_rows][4C] (cubic) or [n_paths][n_rows][C] (linear) */
    const void* knot_t;        /* linear: knots [n_rows] (NULL = 0, 1, 2, ...); unused for cubic */
    const int32_t* index;      /* [n_times] interval index of every query, located on the host from THIS member's knots */
    const void* frac;          /* [n_times] */
    void* out;                 /* [n_paths][n_times][channels] */
    int64_t n_paths, n_rows, channels, n_times;
    int32_t control_kind, reserved;
} tcde_spline_member;
TCDE_API int tcde_spline_eval_grouped(const tcde_spline_member* members, int n_members, int derivative, int dtype,
                                      void* stream);

typedef struct tcde_contract_member {
    const void* field;         /* [n_paths][hidden][channels] contiguous */
    const void* dx;            /* dx[p * dx_stride + c] */
    void* out;                 /* [n_paths][hidden] */
    int64_t n_paths, hidden, channels, dx_stride;
} tcde_contract_member;
/* out_k = scale * field_k @ dx_k for every member k, as tcde_field_contract computes it */
TCDE_API int tcde_field_contract_grouped(const tcde_contract_member* members, int n_members, double scale, int dtype,
                                         void* stream);

/* The error ratio of one attempted step (rk_common._compute_error_ratio, restated): with
 * err = sum_j coefs[j] * terms[j] and tol = atol + rtol * max(|y0|, |y1|), partials[c] receives the sum over
 * CTA c's elements of (err / tol)^2; the RMS norm is sqrt(sum(partials) / n).  partials: device double
 * [tcde_error_ratio_partials(n)]. */
TCDE_API int64_t tcde_error_ratio_partials(int64_t n);
TCDE_API int tcde_error_ratio_sumsq(const void* y0, const void* y1, const void* const* terms, const double* coefs,
                           int n_terms, double atol, double rtol, int64_t n, int dtype, void* partials, void* stream);

/* Device-controlled Dormand-Prince 5(4) for the linear vector field (float32, hidden = 32, channels = 8) -- replaces what
 * the reference obtains from torchdiffeq's adaptive solver behind torchcde/solver.py:226-227 (default method of cdeint).
 * ONE launch = one attempted step of the whole batch; accept / reject, the step-size rule and the dense output at the
 * requested times run on the device, so the host only reads the control block once per chunk of launches.
 *   state     float  [5][n_paths][32]: Y0, Y1, F0, F1, MID.  Before the first launch Y0 = y(t0), F0 = f(t0, y(t0)).
 *   partials  double [2][tcde_dopri5_linear_grid(n_paths)]
 *   ctl       double [2][24]: slot 1 is read by launch 0.  Fields: 0 t, 1 dt, 2 t_end, 3 rtol, 4 atol, 5 current state
 *             buffer, 6 done, 7 pending (an undecided attempt exists), 8 accepted, 9 rejected, 10 next output index (>= 1),
 *             11 number of partials, 12 need_mid, 13 last error ratio, 14 launches.  Launch seq reads slot (seq + 1) & 1
 *             and writes slot seq & 1.
 *   out       float  [n_paths][n_out][32]; the caller writes out[:, 0] = y(t0).  out_times: device double [n_out], increasing
 *             (negated for a decreasing t, sign = -1).
 * Enqueues launches first_seq .. first_seq + n_launches - 1 on the stream; launches after the end are no-ops. */
TCDE_API int tcde_dopri5_linear_grid(int64_t n_paths);
TCDE_API int tcde_dopri5_linear_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                const void* weight, const void* bias, void* state, void* partials, void* ctl, void* out,
                                const void* out_times, int64_t n_out, int64_t n_paths, int64_t channels, int64_t hidden,
                                double sign, int64_t first_seq, int64_t n_launches, int dtype, void* stream);

/* The backward pass of cdeint(adjoint=True) with dopri5 for the linear field, controller on the device (torchdiffeq's
 * odeint_adjoint behind torchcde/solver.py:226-227 with the default method): a VIRTUAL batch of 2 n_ctrl paths -- the first half
 * the state z with (weight, bias), the second half the adjoint state a with (weight2, bias2) = the regrouped, negated weight and a
 * zero bias -- advances with one step-size controller (RMS error norm over both halves).  state [5][2 n_ctrl][32], out
 * [2 n_ctrl][n_out][32], ctl / partials as for tcde_dopri5_linear_attempts (grid for 2 n_ctrl paths); ctl field 15 = slots full, 16 = slot base.
 * Every attempt stores the inputs of its stages 1, 3, 4, 5, 6 into slot [accepted steps so far] of dump_z / dump_a
 * [max_slots][5][n_ctrl][32]; for every accepted step the controller writes the five quadrature nodes q_index / q_frac /
 * q_weight [max_slots * 5] (spline interval, fraction, dt * b_i), so that ONE call of tcde_linear_field_param_grads over
 * 5 * accepted stages yields dL/dW, dL/db.  When the slots are full the solve pauses (done = 1, field 15 = 1): the caller
 * contracts the filled slots, sets field 16 to the number of accepted steps, clears fields 6 and 15 of the slot just
 * read, and enqueues more launches.
 * n_ctrl must be a multiple of 256.  float32, hidden = 32, channels = 8. */
TCDE_API int tcde_dopri5_linear_paired_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                       const void* weight, const void* bias, const void* weight2, const void* bias2, void* state,
                                       void* partials, void* ctl, void* out, const void* out_times, int64_t n_out, int64_t n_ctrl,
                                       int64_t channels, int64_t hidden, double sign, void* dump_z, void* dump_a,
                                       int32_t* q_index, void* q_frac, void* q_weight, int64_t max_slots, int64_t first_seq,
                                       int64_t n_launches, int dtype, void* stream);

/* The forward pass of cdeint(adjoint=False) with dopri5 for the linear field when gradients are wanted: the attempts of
 * tcde_dopri5_linear_attempts (same outputs, same accepted and rejected steps, bit for bit) that also record what the
 * backward pass needs.  Every attempt writes into slot [accepted steps so far - ctl field 16] (a rejected attempt is
 * overwritten by the next one):
 *   rec_step  double [max_slots][2]: (t, dt) of the step
 *   rec_index int32 / rec_frac float [max_slots][6]: spline interval and fraction of stages 2..7 (stage 7 at t + dt)
 *   rec_z     float  [max_slots][6][n_paths][32]: the inputs of stages 2..7, the last one being the step's result; may be NULL
 *             (no parameter gradient wanted)
 * When the slots are full the solve pauses as in tcde_dopri5_linear_paired_attempts (done = 1, field 15 = 1): the caller
 * keeps the filled record, passes fresh storage, sets field 16 to the number of accepted steps, clears fields 6 and 15 of
 * the slot just read and enqueues more launches.  Same support as tcde_dopri5_linear_attempts; rec_z 16-byte aligned. */
TCDE_API int tcde_dopri5_linear_record_attempts(const void* control, int control_kind, int64_t n_rows, const void* knots,
                                       const void* weight, const void* bias, void* state, void* partials, void* ctl, void* out,
                                       const void* out_times, int64_t n_out, int64_t n_paths, int64_t channels, int64_t hidden,
                                       double sign, void* rec_z, void* rec_step, int32_t* rec_index, void* rec_frac,
                                       int64_t max_slots, int64_t first_seq, int64_t n_launches, int dtype, void* stream);

/* The backward pass of that record over n_steps accepted steps, last to first, in ONE launch: the transposed
 * Dormand-Prince recurrence of the linear field (J^T by the field product on weight_t = W.view(H,C,H).permute(2,1,0)
 * .reshape(H*C,H) with a zero bias).
 *   grad_out  float [n_paths][n_out][32]: dL/d(outputs)
 *   carry     float [2][n_paths][32]: in, the cotangent of the state after the last step and the cotangent still pending on
 *             that step's last evaluation (zero for the last step of the solve); out, the same at the first step's start
 *             (the second is the cotangent of the start slope f(t0, z0), whose J^T and parameter gradients are the caller's)
 *   kappa     float [n_steps][6][n_paths][32] or NULL: the cotangent of every evaluation, in the item of its input in rec_z,
 *             for tcde_linear_field_param_grads with item weight = sign
 *   coef      float [n_steps][36]: (float)(beta[s][j] * dt) of the Dormand-Prince tableau, rows s = 0..5, zero padded
 *   stage_index / stage_frac [n_steps][6]: the record's
 *   inj_range int32 [n_steps + 1], inj_out int32 [n_inj], inj_w float [n_inj][8]: the outputs step n emits and their
 *             weights on (y_n, y_{n+1}, k1, k3, k4, k5, k6, k7) -- the transposed dense output with y_mid folded in
 * Same support as tcde_dopri5_linear_attempts; control, grad_out, carry and kappa 16-byte aligned. */
TCDE_API int tcde_dopri5_linear_backward(const void* control, int control_kind, int64_t n_rows, const void* weight_t,
                                const void* zeros, const void* grad_out, void* carry, void* kappa, const void* coef,
                                const int32_t* stage_index, const void* stage_frac, const int32_t* inj_range,
                                const int32_t* inj_out, const void* inj_w, int64_t n_out, int64_t n_steps, int64_t n_paths,
                                int64_t channels, int64_t hidden, double sign, int dtype, void* stream);

/* Logsignatures of windows of piecewise-linear paths -- replaces the per-window call of the optional third-party package
 * at torchcde/log_ode.py:56-58 (``signatory.Logsignature(depth)``, default "words" basis).  x [n_paths][length][channels]
 * (NaN free); window w spans the points window_index[w] .. window_index[w + 1] (device int32 [n_windows + 1]); words: device
 * int32 [n_words][2] = (level, flat index i_1 * C^(k-1) + ... + i_k) of the Lyndon words; out [n_paths][n_windows][n_words].
 * channels^1 + ... + channels^depth must not exceed tcde_logsignature_max_terms(). */
TCDE_API int64_t tcde_logsignature_max_terms(void);
TCDE_API int tcde_logsignature_windows(const void* x, int64_t n_paths, int64_t length, int64_t channels,
                              const int32_t* window_index, int64_t n_windows, int depth, const int32_t* words, int64_t n_words,
                              void* out, int dtype, void* stream);

/* Natural-cubic / gap-fill kernel choice: 0 = the parallel kernels (windowed sweeps, warp per path)
 * when the path fits shared memory (default), 1 = one thread per series, 2 = parallel kernels
 * but the CTA-per-path natural-cubic kernel instead of the warp-per-path one.  For tests / benchmarks. */
TCDE_API int tcde_set_natural_variant(int variant);

/* Which kernel tcde_cdeint_fixed_linear, tcde_cdeint_reversible_heun_linear and tcde_cdeint_fixed_mlp launch for
 * float32: 0 = automatic (the tensor-core kernel where it is built for the shape: hidden = 32, channels = 8, and for the
 * MLP width = 128; the CUDA-core kernel otherwise, for the MLP only at hidden <= 8 or hidden * channels <= 32), 1 =
 * CUDA-core kernel (for the MLP also in float64 at every shape it is built for), 3 / 4 = tensor-core kernel (solve_tc.cu,
 * solve_mlp.cu) with the 3xTF32 / the 2xFP16 operand split (TCDE_ERR_UNSUPPORTED for other shapes; the MLP field has
 * no 3xTF32 kernel); 2 and 6 are aliases of 3, 5 of 4; bits above 15 are ignored.
 * Process-wide; meant for tests and benchmarks. */
TCDE_API int tcde_set_solve_variant(int variant);

#ifdef __cplusplus
}
#endif
#endif /* TORCHCDE_B200_H */
