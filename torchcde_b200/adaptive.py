"""Adaptive (dopri5) stepping and the adjoint backward pass -- this package's own drivers.

Where the reference calls ``torchdiffeq.odeint`` / ``odeint_adjoint`` with the default method
(solver.py:226-227; ``example/time_series_classification.py:83-86`` uses dopri5 + adjoint), we
run the drivers below instead.  They restate the *published* algorithms of torchdiffeq 0.2.x
(``_impl/rk_common.py`` ``RKAdaptiveStepsizeODESolver`` with the Dormand-Prince tableau,
``_impl/adjoint.py``) -- the package itself is not installable here, so, like the fixed-step
port, the stepping is "parity unpinned" against a torchdiffeq binary; an adaptive solver's
output is only defined up to its tolerances anyway, and that is what the tests check
(against tight-tolerance fp64 solutions).

Design for the GPU: time, step size and the controller live on the HOST as Python floats
(double precision, the dtype torchdiffeq uses for them); the state, the seven stage slopes and
the error estimate live on the device; each attempted step costs exactly one device->host
read (the error ratio), which is also what torchdiffeq pays (``if accept_step``).  The error
norm is the RMS over the *whole* state tensor, so a batch shares one step sequence
(SURVEY.md 8e caveat 1).  The vector field is a callable ``field(t_float, y) -> dy``; for the
linear vector field it is one fused kernel launch (``tcde_vector_field_linear``).

The backward pass of ``adjoint=True`` for the flagship linear field (fp32, hidden 32, channels 8) does not go
through autograd: a fixed-step backward solve is three launches per segment (``_fused_fixed_backward`` ->
``linear_field.AdjointStage.segment``), an adaptive one gets the field and its vector-Jacobian products from one launch
per evaluation (``tcde_vector_field_linear_vjp``); the stage combinations and the error ratio of a dopri5
attempt are single launches too (``tcde_linear_combination`` / ``tcde_error_ratio_sumsq``).  The examples' MLP field
gets the same per-evaluation layer at its CUDA-core shapes (``mlp_field.MlpAdjointStage``, one call of
``tcde_vector_field_mlp_vjp`` per stage, for dopri5 and the fixed-step methods alike).
"""
import ctypes
import math

import torch

from . import _lib

# Dormand-Prince 5(4), FSAL.  alpha, beta (rows), solution weights, error weights, midpoint weights
_ALPHA = (1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0)
_BETA = (
    (1 / 5,),
    (3 / 40, 9 / 40),
    (44 / 45, -56 / 15, 32 / 9),
    (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
    (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656),
    (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84),
)
_C_ERROR = (
    35 / 384 - 1951 / 21600, 0.0, 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720,
    -2187 / 6784 - -12231 / 42400, 11 / 84 - 649 / 6300, -1.0 / 60.0,
)
_C_MID = (
    6025192743 / 30085553152 / 2, 0.0, 51252292925 / 65400821598 / 2, -2691868925 / 45128329728 / 2,
    187940372067 / 1594534317056 / 2, -1776094331 / 19743644256 / 2, 11237099 / 235043384 / 2,
)
_ORDER = 5


def _rms(x):
    return float(x.detach().pow(2).mean().sqrt())


# The error norm of a tuple state (TupleControl).  torchdiffeq flattens a tuple ``y0`` into one vector and, unless told
# otherwise, measures its adaptive steps with the *mixed* norm: the largest of the members' RMS norms, for the error ratio
# and for the initial step alike (_impl/misc.py ``_mixed_norm`` -- recalled, not verified: torchdiffeq is not installed
# here, see DESIGN.md section 3).  This switch is the one place that choice is made; "rms" would measure the packed state
# as one tensor.
TUPLE_NORM = "mixed"


class MixedNorm:
    """max over the segments of a packed vector (``sizes`` elements each, end to end) of each segment's RMS; a segment
    without elements contributes nothing."""

    def __init__(self, sizes):
        self.sizes = [int(n) for n in sizes]
        self.offsets = [sum(self.sizes[:i]) for i in range(len(self.sizes))]

    def __call__(self, x):
        flat = x.detach().reshape(-1)
        return max((_rms(flat[o:o + n]) for o, n in zip(self.offsets, self.sizes) if n), default=0.0)


def tuple_norm(sizes):
    """The norm of a packed tuple state whose members have ``sizes`` elements (see ``TUPLE_NORM``)."""
    return MixedNorm(sizes) if TUPLE_NORM == "mixed" else _rms


def _kernels_apply(*tensors):
    """The single-launch kernels serve plain CUDA float tensors of one shape outside autograd; anything else
    (CPU tensors, states that are being differentiated with adjoint=False) keeps the torch operators."""
    first = tensors[0]
    if not (first.is_cuda and first.dtype in (torch.float32, torch.float64) and first.numel() > 0):
        return False
    grad = torch.is_grad_enabled()
    for x in tensors:
        if x.shape != first.shape or x.dtype != first.dtype or x.device != first.device or not x.is_contiguous():
            return False
        if grad and x.requires_grad:
            return False
    return True


def _term_arrays(ks, coefs):
    n = len(ks)
    return (ctypes.c_void_p * n)(*[k.data_ptr() for k in ks]), (ctypes.c_double * n)(*coefs), n


def _combine(base, ks, weights, dt, out=None):
    """base + sum_j (weights[j] * dt) * ks[j], skipping zero weights -- one launch of ``tcde_linear_combination``
    where that applies (``base`` may be None for a pure combination; ``out`` may alias ``base``)."""
    pairs = [(k, w * dt) for k, w in zip(ks, weights) if w != 0.0]
    terms = [k for k, _ in pairs]
    if terms and len(terms) <= 7 and _kernels_apply(*(terms + ([base] if base is not None else []))):
        out = torch.empty_like(terms[0]) if out is None else out
        ptrs, coefs, n = _term_arrays(terms, [c for _, c in pairs])
        with torch.cuda.device(out.device):
            _lib.call("tcde_linear_combination", _lib.ptr(out), _lib.ptr(base), ptrs, coefs, n, out.numel(),
                      _lib.dtype_code(out.dtype), _lib.stream_of(out))
        return out
    res = base if base is not None else torch.zeros_like(ks[0])
    for k, c in pairs:
        res = res + k * c
    if out is not None:
        out.copy_(res)
        return out
    return res


def _error_ratio(y0, y1, ks, weights, dt, atol, rtol, norm):
    """norm(err / (atol + rtol max(|y0|, |y1|))) with err = dt sum_j weights[j] ks[j]; for the default RMS norm one
    launch of ``tcde_error_ratio_sumsq`` plus the sum of its per-CTA partials (the one host read per attempt)."""
    pairs = [(k, w * dt) for k, w in zip(ks, weights) if w != 0.0]
    terms = [k for k, _ in pairs]
    if isinstance(norm, MixedNorm) and terms and len(terms) <= 7 and _kernels_apply(y0, y1, *terms):
        # one tcde_error_ratio_sumsq per member range of the packed state, one host read for all of them
        lib, size = _lib.load(), y0.element_size()
        segs = [(o, n) for o, n in zip(norm.offsets, norm.sizes) if n]
        n_parts = [lib.tcde_error_ratio_partials(n) for _, n in segs]
        partials = torch.empty(sum(n_parts), dtype=torch.float64, device=y0.device)
        coefs = [c for _, c in pairs]
        at = 0
        with torch.cuda.device(y0.device):
            for (o, n), m in zip(segs, n_parts):
                _, cf, n_terms = _term_arrays(terms, coefs)
                ptrs = (ctypes.c_void_p * n_terms)(*[k.data_ptr() + o * size for k in terms])
                _lib.call("tcde_error_ratio_sumsq", ctypes.c_void_p(y0.data_ptr() + o * size),
                          ctypes.c_void_p(y1.data_ptr() + o * size), ptrs, cf, n_terms, float(atol), float(rtol), n,
                          _lib.dtype_code(y0.dtype), ctypes.c_void_p(partials.data_ptr() + at * 8), _lib.stream_of(y0))
                at += m
        sums = partials.cpu().tolist()
        ratios, at = [], 0
        for (_, n), m in zip(segs, n_parts):
            ratios.append(math.sqrt(math.fsum(sums[at:at + m]) / n))
            at += m
        return max(ratios, default=0.0)
    if norm is _rms and terms and len(terms) <= 7 and _kernels_apply(y0, y1, *terms):
        n_part = _lib.load().tcde_error_ratio_partials(y0.numel())
        partials = torch.empty(n_part, dtype=torch.float64, device=y0.device)
        ptrs, coefs, n = _term_arrays(terms, [c for _, c in pairs])
        with torch.cuda.device(y0.device):
            _lib.call("tcde_error_ratio_sumsq", _lib.ptr(y0), _lib.ptr(y1), ptrs, coefs, n, float(atol), float(rtol),
                      y0.numel(), _lib.dtype_code(y0.dtype), _lib.ptr(partials), _lib.stream_of(y0))
        return float(partials.sum().div_(y0.numel()).sqrt_())
    err = _combine(None, ks, weights, dt)
    tol = atol + rtol * torch.max(y0.abs(), y1.abs())
    return norm(err / tol)


def _initial_step(field, t0, y0, f0, rtol, atol, norm=_rms):
    """Hairer's starting step (torchdiffeq ``_select_initial_step`` with order - 1 = 4)."""
    scale = atol + y0.abs() * rtol
    d0 = norm(y0 / scale)
    d1 = norm(f0 / scale)
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    f1 = field(t0 + h0, y0 + h0 * f0)
    d2 = norm((f1 - f0) / scale) / h0
    if d1 <= 1e-15 and d2 <= 1e-15:
        h1 = max(1e-6, h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1.0 / _ORDER)
    return min(100 * h0, h1)


def _next_step(dt, ratio, safety=0.9, ifactor=10.0, dfactor=0.2):
    if ratio == 0:
        return dt * ifactor
    if ratio < 1:
        dfactor = 1.0
    return dt * min(ifactor, max(safety / ratio ** (1.0 / _ORDER), dfactor))


class Dopri5:
    """One adaptive solve of dy/dt = field(t, y) over increasing output times ``t`` (floats)."""

    def __init__(self, field, y0, rtol, atol, first_step=None, max_num_steps=2 ** 31 - 1, norm=None, jump_t=None):
        self.field, self.rtol, self.atol = field, float(rtol), float(atol)
        self.max_num_steps = max_num_steps
        self.norm = norm or _rms
        self.first_step = first_step
        self.y0 = y0
        self.n_accepted = 0
        self.n_rejected = 0
        # times at which the field is discontinuous (README.md:194-200, `options=dict(jump_t=X.grid_points)`):
        # no step may straddle one, and the slope is re-evaluated just after it
        self.jump_t = sorted(float(v) for v in jump_t) if jump_t is not None else []

    # Hooks of a solve that records what its backward pass needs (mlp_field.Dopri5MlpBackprop); as defined here they
    # leave the solve as it is.
    def _stage_out(self, s):
        """Where the input of stage s + 2 of the current attempt is written (None: a new tensor)."""
        return None

    def _stage_done(self, s):
        """Called after the evaluation of stage s + 2 of the current attempt."""

    def _start_slope(self, t, y, *nudge):
        """f(t, y) where a step starts from a slope of its own: at t0, and just after a jump of ``jump_t``."""
        return self.field(t, y, *nudge)

    def _accepted(self, t, dt, t_new):
        """Called when the attempt (t, dt) is accepted, before the next start slope; it ends at t_new."""

    def _stages(self, t0, dt, y0, f0):
        ks = [f0]
        y1 = y0
        for s, (alpha, beta) in enumerate(zip(_ALPHA, _BETA)):
            ti = t0 + dt if alpha == 1.0 else t0 + alpha * dt
            y1 = _combine(y0, ks, beta, dt, out=self._stage_out(s))
            ks.append(self.field(ti, y1))
            self._stage_done(s)
        # the last beta row equals the solution weights (FSAL): y1 is the 5th-order solution
        return y1, ks

    def _attempt(self, t0, dt, y0, f0):
        y1, ks = self._stages(t0, dt, y0, f0)
        return y1, ks, _error_ratio(y0, y1, ks, _C_ERROR, dt, self.atol, self.rtol, self.norm)

    def integrate(self, times, targets=None, steps=None):
        """``targets``: optional 1-D tensor holding the same output times; when given, the dense output is evaluated at
        the tensor entries so that autograd sees the dependence on the requested times (adjoint=False).  ``steps``: the
        accepted steps ``[(t, dt), ...]`` of an earlier solve of the same problem (``cdeint.last_stats["steps"]``); the
        solve then takes exactly those steps, without the controller -- a replay of that discrete solve."""
        out = [self.y0]
        t0 = times[0]
        y0 = self.y0
        f0 = self._start_slope(t0, y0)
        if steps is not None:
            steps = list(steps)
            dt = steps[0][1] if steps else 0.0
        else:
            dt = self.first_step if self.first_step is not None else _initial_step(self.field, t0, y0, f0, self.rtol,
                                                                                   self.atol, self.norm)
        t_lo, t_hi = t0, t0
        coeff = None
        jumps = [v for v in self.jump_t if v > t0]
        for n_target, target in enumerate(times[1:], 1):
            tries = 0
            while target > t_hi:
                if tries >= self.max_num_steps:
                    raise RuntimeError("max_num_steps exceeded ({}>={})".format(tries, self.max_num_steps))
                step = dt
                if steps is not None:
                    if self.n_accepted == len(steps):
                        raise RuntimeError("dopri5 replay: the recorded steps end at t = {}".format(t_hi))
                    step = steps[self.n_accepted][1]
                # a recorded step that ends on a jump is jumps[0] - t_hi, which t_hi + step may round onto or below the jump
                on_jump = bool(jumps) and t_hi < jumps[0] and (jumps[0] < t_hi + step
                                                                or (steps is not None and jumps[0] - t_hi == step))
                if on_jump:
                    step = jumps[0] - t_hi
                if steps is None:
                    y1, ks, ratio = self._attempt(t_hi, step, y0, f0)
                else:                            # a recorded step: accepted, no error estimate
                    (y1, ks), ratio = self._stages(t_hi, step, y0, f0), 0.0
                if ratio <= 1:
                    t_new = jumps[0] if on_jump else t_hi + step
                    self._accepted(t_hi, step, t_new)
                    if t_new >= target:          # the dense output is only ever evaluated inside the last step
                        y_mid = _combine(y0, ks, _C_MID, step)
                        coeff = self._fit(y0, y1, y_mid, ks[0], ks[-1], step)
                    t_lo, t_hi = t_hi, t_new
                    y0, f0 = y1, ks[-1]
                    if on_jump:
                        jumps.pop(0)
                        f0 = self._start_slope(t_hi, y0, 1)      # the slope just AFTER the discontinuity
                    self.n_accepted += 1
                else:
                    self.n_rejected += 1
                dt = _next_step(step, ratio)
                tries += 1
            out.append(self._evaluate(coeff, t_lo, t_hi, target if targets is None else targets[n_target]))
        return torch.stack(out, dim=0)

    @staticmethod
    def _fit(y0, y1, y_mid, f0, f1, dt):
        a = 2 * dt * (f1 - f0) - 8 * (y1 + y0) + 16 * y_mid
        b = dt * (5 * f0 - 3 * f1) + 18 * y0 + 14 * y1 - 32 * y_mid
        c = dt * (f1 - 4 * f0) - 11 * y0 - 5 * y1 + 16 * y_mid
        return (y0, dt * f0, c, b, a)

    @staticmethod
    def _evaluate(coeff, t_lo, t_hi, t):
        x = (t - t_lo) / (t_hi - t_lo)
        total = coeff[0] + x * coeff[1]
        power = x
        for cf in coeff[2:]:
            power = power * x
            total = total + power * cf
        return total


def odeint_dopri5(field, y0, times, rtol, atol, options=None, targets=None, norm=None, steps=None):
    """``times``: increasing Python floats.  Returns (len(times), *y0.shape).  ``norm``: the error norm (default RMS).
    ``steps``: replay these accepted ``(t, dt)`` instead of running the controller (``Dopri5.integrate``)."""
    options = dict(options or {})
    jump_t = options.pop("jump_t", None)
    if isinstance(jump_t, torch.Tensor):
        jump_t = jump_t.detach().cpu().tolist()
    solver = Dopri5(field, y0, rtol, atol, first_step=options.pop("first_step", None),
                    max_num_steps=options.pop("max_num_steps", 2 ** 31 - 1), norm=norm, jump_t=jump_t)
    if options:
        raise NotImplementedError("dopri5: unsupported options {}".format(sorted(options)))
    out = solver.integrate(list(times), targets, steps)
    return out, solver


# ----------------------------------------------------- dopri5 with the controller on the device (linear field)
_DEVICE_CHUNK = 48          # launches enqueued between two reads of the done flag

# One control slot of solve_dopri5.cu: CTL_SIZE doubles, fields in the order of its C_* enum.  Launch n reads slot
# (n - 1) & 1 and writes slot n & 1; the integer fields hold exact small integers.
CTL_SIZE = 24
(CTL_T, CTL_DT, CTL_TEND, CTL_RTOL, CTL_ATOL, CTL_CUR, CTL_DONE, CTL_PENDING, CTL_NACC, CTL_NREJ, CTL_NEXT_OUT,
 CTL_NPART, CTL_NEED_MID, CTL_RATIO, CTL_LAUNCHES, CTL_OVERFLOW, CTL_BASE) = range(17)


def initial_control(t0, dt, t_end, rtol, atol):
    """The two control slots before launch 0: slot 1 (what launch 0 reads) holds the start, no attempt pending."""
    ctl = torch.zeros(2, CTL_SIZE, dtype=torch.float64)
    ctl[1, CTL_T], ctl[1, CTL_DT], ctl[1, CTL_TEND] = t0, dt, t_end
    ctl[1, CTL_RTOL], ctl[1, CTL_ATOL] = rtol, atol
    ctl[1, CTL_NEXT_OUT] = 1
    return ctl


def device_dopri5_available(z0, channels):
    return (z0.is_cuda and z0.dtype == torch.float32 and z0.size(-1) == 32 and channels == 8 and z0.numel() > 0)


def device_controller(launch, field, v0, times, rtol, atol, first_step, underflow, on_overflow=None):
    """The host loop of the device-controlled dopri5 kernels: ``launch(state, partials, ctl, out, out_times, first_seq)``
    enqueues ``_DEVICE_CHUNK`` attempts from ``v0``, one control slot is read per chunk; ``field`` only gives the start
    slope and Hairer's first step.  ``on_overflow(last)`` empties full trajectory slots before the solve resumes;
    ``underflow`` is the error message.  Returns ``(out (paths, len(times), H), the last control slot, stats)``."""
    dev = v0.device
    n_paths, hidden = v0.shape
    with torch.cuda.device(dev), torch.no_grad():
        f0 = field(times[0], v0)
        dt = first_step if first_step is not None else _initial_step(field, times[0], v0, f0, rtol, atol)
        state = torch.empty(5, n_paths, hidden, dtype=torch.float32, device=dev)
        state[0].copy_(v0)
        state[2].copy_(f0)
        partials = torch.zeros(2, _lib.load().tcde_dopri5_linear_grid(n_paths), dtype=torch.float64, device=dev)
        ctl = initial_control(times[0], dt, times[-1], rtol, atol).to(dev)
        out = torch.empty(n_paths, len(times), hidden, dtype=torch.float32, device=dev)
        out[:, 0].copy_(v0)
        out_times = torch.tensor(times, dtype=torch.float64, device=dev)
        seq = 0
        while True:
            launch(state, partials, ctl, out, out_times, seq)
            seq += _DEVICE_CHUNK
            last = ctl[(seq - 1) & 1].cpu()              # the one host read per chunk
            if last[CTL_DONE] != 0:
                if last[CTL_OVERFLOW] == 0:
                    break
                on_overflow(last)
                # hand the slots back and resume where the device paused
                resume = last.clone()
                resume[CTL_DONE], resume[CTL_OVERFLOW], resume[CTL_BASE] = 0.0, 0.0, last[CTL_NACC]
                ctl[(seq - 1) & 1].copy_(resume)
                continue
            if not math.isfinite(float(last[CTL_DT])) or float(last[CTL_DT]) == 0.0 or seq > 10_000_000:
                raise RuntimeError(underflow.format(float(last[CTL_T])))
    return out, last, {"n_accepted": int(last[CTL_NACC]), "n_rejected": int(last[CTL_NREJ]), "launches": seq}


def dense_output_weights(x, dt):
    """The weights of ``Dopri5._evaluate(Dopri5._fit(y0, y1, y_mid, f0, f1, dt), 0, 1, x)`` on (y0, y1, y_mid, f0, f1):
    the dense output is linear in them."""
    x2, x3, x4 = x * x, x * x * x, x * x * x * x
    return (1.0 - 11.0 * x2 + 18.0 * x3 - 8.0 * x4, -5.0 * x2 + 14.0 * x3 - 8.0 * x4, 16.0 * x2 - 32.0 * x3 + 16.0 * x4,
            dt * (x - 4.0 * x2 + 5.0 * x3 - 2.0 * x4), dt * (x2 - 3.0 * x3 + 2.0 * x4))


def dopri5_backward_tables(steps, times, dtype=torch.float32, ends=None):
    """The host tables of ``tcde_dopri5_linear_backward`` / ``tcde_dopri5_mlp_backward`` for the accepted ``steps``
    [(t, dt), ...] of a solve over the increasing output times ``times``, in double, cast to ``dtype`` (the state dtype:
    the coefficients the forward's combinations used) at the end:
      coef [n, 36]: beta[s][j] * dt, the forward's own stage coefficients;
      inj_range [n + 1], inj_out [m], inj_w [m, 8]: the outputs each step emits (the kernel's rule: the first accepted step
      whose end is at or past the output time; output 0 is y(t0) itself) and their weights on (y_n, y_{n+1}, k1, k3, k4,
      k5, k6, k7) -- ``dense_output_weights`` with y_mid = y_n + dt sum_j c_mid[j] k_j folded in.
    ``ends``: where each step ended as the solve took it (a step cut at a jump of ``jump_t`` ends exactly on the jump,
    which t + dt may miss by a rounding); default t + dt."""
    import numpy as np
    n = len(steps)
    np_dtype = np.float64 if dtype == torch.float64 else np.float32
    dts = np.array([dt for _t, dt in steps], dtype=np.float64)
    beta = np.zeros((6, 6))
    for s, row in enumerate(_BETA):
        beta[s, :len(row)] = row
    coef = (beta.reshape(1, 36) * dts.reshape(n, 1)).astype(np_dtype)
    inj_range, inj_out, inj_w = [0], [], []
    nxt = 1
    for i, (t, dt) in enumerate(steps):
        t_hi = t + dt if ends is None else ends[i]
        while nxt < len(times) and times[nxt] <= t_hi:
            w_y0, w_y1, w_ym, w_f0, w_f1 = dense_output_weights((times[nxt] - t) / (t_hi - t), dt)
            cm = [c * dt * w_ym for c in _C_MID]
            inj_out.append(nxt)
            inj_w.append([w_y0 + w_ym, w_y1, w_f0 + cm[0], cm[2], cm[3], cm[4], cm[5], w_f1 + cm[6]])
            nxt += 1
        inj_range.append(len(inj_out))
    return {"coef": torch.from_numpy(coef), "inj_range": torch.tensor(inj_range, dtype=torch.int32),
            "inj_out": torch.tensor(inj_out or [0], dtype=torch.int32),
            "inj_w": torch.tensor(inj_w or [[0.0] * 8], dtype=torch.float64).to(dtype)}


# ------------------------------------------------------------------------- fixed grids (generic)
def odeint_fixed(field, y0, times, method, step_size):
    """Fixed-grid euler / midpoint / rk4 (3/8 rule) on float times -- used by the adjoint pass."""
    t0, t_end = times[0], times[-1]
    if step_size is None:
        grid = list(times)
    else:
        n = int(math.ceil((t_end - t0) / step_size + 1))
        grid = [t0 + i * step_size for i in range(n)]
        grid[-1] = t_end
    out = [y0]
    y = y0
    j = 1
    for a, b in zip(grid[:-1], grid[1:]):
        dt = b - a
        if method == "rk4":
            k1 = field(a, y)
            k2 = field(a + dt / 3, y + dt * k1 / 3)
            k3 = field(a + dt * 2 / 3, y + dt * (k2 - k1 / 3))
            k4 = field(b, y + dt * (k1 - k2 + k3))
            y1 = y + (k1 + 3 * (k2 + k3) + k4) * (dt * 0.125)
        elif method == "midpoint":
            y1 = y + dt * field(a + dt / 2, y + field(a, y) * (dt / 2))
        else:
            y1 = y + dt * field(a, y)
        while j < len(times) and b >= times[j]:
            if times[j] == b:
                out.append(y1)
            else:
                out.append(y + ((times[j] - a) / (b - a)) * (y1 - y))
            j += 1
        y = y1
    return torch.stack(out, dim=0)


# ------------------------------------------------------------------------------------- adjoint
def _packing(shapes):
    """``pack(parts)`` / ``unpack(flat)`` of the adjoint's augmented state: tensors of ``shapes`` end to end."""
    sizes = [s.numel() for s in shapes]

    def pack(parts):
        return torch.cat([p.reshape(-1) for p in parts])

    def unpack(flat):
        outs, off = [], 0
        for shape, n in zip(shapes, sizes):
            outs.append(flat[off:off + n].view(shape))
            off += n
        return outs

    return pack, unpack


class _Adjoint(torch.autograd.Function):
    """Continuous adjoint (torchdiffeq ``odeint_adjoint``): the forward pass keeps only the outputs;
    the backward pass integrates ``(y, a_y, a_params)`` backwards between consecutive output times
    with the same solver family, evaluating the vector field under autograd for its VJPs."""

    @staticmethod
    def forward(ctx, forward_solve, vf, times, solve_aug, fused_vjp, fixed_spec, flipped, t_tensor, y0, *params):
        ctx.vf, ctx.times, ctx.solve_aug, ctx.fused_vjp, ctx.fixed_spec = vf, times, solve_aug, fused_vjp, fixed_spec
        ctx.flipped = flipped
        ctx.t_needs_grad = t_tensor is not None and t_tensor.requires_grad
        ctx.t_meta = None if t_tensor is None else (t_tensor.dtype, t_tensor.device)
        with torch.no_grad():
            ys = forward_solve(y0)
        ctx.save_for_backward(ys, *params)
        return ys

    @staticmethod
    def backward(ctx, grad_ys):
        ys, *params = ctx.saved_tensors
        vf, times = ctx.vf, ctx.times
        params = tuple(params)
        if ctx.fused_vjp is not None and ctx.fixed_spec is not None and not ctx.t_needs_grad:
            with torch.no_grad():
                a_y, a_p = _fused_fixed_backward(ctx.fused_vjp, times, ys, grad_ys, *ctx.fixed_spec)
            return (None, None, None, None, None, None, None, None, a_y, *a_p)
        if ctx.t_needs_grad:
            return _Adjoint._backward_with_times(ctx, ys, params, grad_ys)
        if ctx.fused_vjp is not None and ctx.fused_vjp.adaptive_spec is not None:
            with torch.no_grad():
                done = _device_adaptive_backward(ctx.fused_vjp, times, ys, grad_ys)
            if done is not None:
                return (None, None, None, None, None, None, None, None, done[0], *done[1])
        pack, unpack = _packing([ys[0].shape, ys[0].shape] + [p.shape for p in params])

        def aug_field(t, flat):
            y, a_y, *_ = unpack(flat)
            if ctx.fused_vjp is not None:
                # one launch: the field and its three vector-Jacobian products with the cotangent -a_y
                f, vjp_y, vjp_p = ctx.fused_vjp(t, y, a_y, -1.0)
                return pack([f, vjp_y] + vjp_p)
            with torch.enable_grad():
                y_ = y.detach().requires_grad_(True)
                f = vf(t, y_)
                # retain_graph: the part of the graph that is shared between calls (views of a coefficient tensor that is
                # itself an adjoint parameter) must survive, like in torchdiffeq's augmented dynamics
                grads = torch.autograd.grad(f, (y_,) + params, -a_y, allow_unused=True, retain_graph=True)
            vjp_y = grads[0] if grads[0] is not None else torch.zeros_like(y)
            vjp_p = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads[1:], params)]
            return pack([f.detach(), vjp_y] + vjp_p)

        with torch.no_grad():
            a_y = grad_ys[-1].clone()
            a_p = [torch.zeros_like(p) for p in params]
            for i in range(len(times) - 1, 0, -1):
                flat0 = pack([ys[i], a_y] + a_p)
                # integrate from times[i] back to times[i-1]: substitute s = -t
                flat1 = ctx.solve_aug(lambda s, v: -aug_field(-s, v), flat0, [-times[i], -times[i - 1]])[-1]
                _, a_y, *a_p = [x.clone() for x in unpack(flat1)]
                a_y = a_y + grad_ys[i - 1]
        return (None, None, None, None, None, None, None, None, a_y, *a_p)

    @staticmethod
    def _backward_with_times(ctx, ys, params, grad_ys):
        """The same backward solve with torchdiffeq's time gradients: the augmented state carries one more scalar,
        the integral of -a^T df/dt, and every output time t_i gets dL/dt_i = <f(t_i, y_i), dL/dy_i> (``odeint_adjoint``
        with ``t.requires_grad``).  Autograd serves the field (its time dependence is the control's dX/dt)."""
        vf, times = ctx.vf, ctx.times
        pack, unpack = _packing([torch.Size([]), ys[0].shape, ys[0].shape] + [p.shape for p in params])

        def aug_field(t, flat):
            _, y, a_y, *_ = unpack(flat)
            with torch.enable_grad():
                t_ = torch.tensor(t, dtype=torch.float64, device=ys.device, requires_grad=True)
                y_ = y.detach().requires_grad_(True)
                f = vf(t_, y_)
                grads = torch.autograd.grad(f, (t_, y_) + params, -a_y, allow_unused=True, retain_graph=True)
            vjp_t = grads[0].to(ys.dtype) if grads[0] is not None else torch.zeros((), dtype=ys.dtype, device=ys.device)
            vjp_y = grads[1] if grads[1] is not None else torch.zeros_like(y)
            vjp_p = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads[2:], params)]
            return pack([vjp_t, f.detach(), vjp_y] + vjp_p)

        with torch.no_grad():
            time_vjps = [None] * len(times)
            a_t = torch.zeros((), dtype=ys.dtype, device=ys.device)
            a_y = grad_ys[-1].clone()
            a_p = [torch.zeros_like(p) for p in params]
            for i in range(len(times) - 1, 0, -1):
                f_i = vf(times[i], ys[i])
                d_cur = (f_i.reshape(-1) * grad_ys[i].reshape(-1)).sum()
                a_t = a_t - d_cur
                time_vjps[i] = d_cur
                flat0 = pack([a_t, ys[i], a_y] + a_p)
                flat1 = ctx.solve_aug(lambda s, v: -aug_field(-s, v), flat0, [-times[i], -times[i - 1]])[-1]
                a_t, _, a_y, *a_p = [x.clone() for x in unpack(flat1)]
                a_y = a_y + grad_ys[i - 1]
            time_vjps[0] = a_t
            grad_t = torch.stack(time_vjps)
            if ctx.flipped:                # the solve ran in s = -t
                grad_t = -grad_t
            grad_t = grad_t.to(dtype=ctx.t_meta[0], device=ctx.t_meta[1])
        return (None, None, None, None, None, None, None, grad_t, a_y, *a_p)


def _device_adaptive_backward(stage, times, ys, grad_ys):
    """The dopri5 backward solve of ``_Adjoint`` with the controller on the device (``stage.adaptive_segment``), segment by
    segment between the output times like torchdiffeq's ``odeint_adjoint``.  Returns ``(a_y, grads)`` or None when a segment
    could not run there (the host-driven backward then starts from scratch)."""
    rtol, atol = stage.adaptive_spec
    grads = stage.new_grads()
    gw = next((g for g, r in zip(grads, stage.roles) if r == "w"), None)
    gb = next((g for g, r in zip(grads, stage.roles) if r == "b"), None)
    from .solver import cdeint
    totals = {}
    a_y = grad_ys[-1].clone()
    for i in range(len(times) - 1, 0, -1):
        try:
            a_lo = stage.adaptive_segment(times[i], times[i - 1], ys[i], a_y, rtol, atol, gw, gb, stage.slots_hint)
        except NotImplementedError:           # TCDE_ERR_UNSUPPORTED from a kernel: the host-driven backward takes any problem
            a_lo = None
        if a_lo is None:
            return None
        for key, val in stage.adaptive_stats.items():
            totals[key] = max(totals.get(key, 0), val) if key == "slots" else totals.get(key, 0) + val
        a_y = a_lo + grad_ys[i - 1]
    try:
        cdeint.last_adjoint_stats = dict(totals, device_controlled=True)
    except Exception:
        pass
    return a_y, grads


def _fused_fixed_backward(stage, times, ys, grad_ys, method, step_size):
    """The backward solve of ``_Adjoint`` for a fixed-step method when the fused adjoint stage kernel serves the
    field: same grid, same stage times and the same Runge-Kutta combinations as ``odeint_fixed`` on the packed
    state, but (z, a) stay one (2, ..., H) tensor that the kernel reads and writes directly, and the parameter
    gradients -- whose slopes do not depend on themselves -- are accumulated in place by the kernel with the
    stage's weight, instead of being carried through ``torch.cat`` as 8,448 extra state components."""
    grads = stage.new_grads()
    unweighted = [None] * len(grads)
    shape = ys[0].shape
    U = torch.empty((2,) + tuple(shape), dtype=ys.dtype, device=ys.device)
    V = torch.empty_like(U)
    K = [torch.empty_like(U) for _ in range(4)]
    a_y = grad_ys[-1].clone()

    def field(idx, frac, state, out, weight):
        # d(z, a)/ds = (-f, +a^T df/dz), d(grad)/ds = +a^T df/dp  (s = -t), the latter times the stage weight
        stage.launch(idx, frac, state[0], state[1], out[0], out[1], *(unweighted if weight == 0.0 else grads),
                     f_scale=-1.0, vjp_scale=1.0, grad_scale=weight)

    for i in range(len(times) - 1, 0, -1):
        # whole segment in three launches (two tensor-core solves that keep their stage inputs + one contraction)
        a_lo = stage.segment(times[i], times[i - 1], ys[i], a_y, method, step_size, *grads)
        if a_lo is not None:
            a_y = a_lo + grad_ys[i - 1]
            continue
        s0, s_end = -times[i], -times[i - 1]
        if step_size is None:
            grid = [s0, s_end]
        else:
            n = int(math.ceil((s_end - s0) / step_size + 1))
            grid = [s0 + j * step_size for j in range(n)]
            grid[-1] = s_end
        stage_times = []
        for lo, hi in zip(grid[:-1], grid[1:]):
            ds = hi - lo
            if method == "rk4":
                stage_times += [lo, lo + ds / 3, lo + ds * 2 / 3, hi]
            elif method == "midpoint":
                stage_times += [lo, lo + ds / 2]
            else:
                stage_times += [lo]
        index, frac = stage.locate_many([-s for s in stage_times])
        U[0].copy_(ys[i])
        U[1].copy_(a_y)
        e = 0
        for lo, hi in zip(grid[:-1], grid[1:]):
            ds = hi - lo
            if method == "rk4":
                # the 3/8 rule of odeint_fixed, each stage state / the step itself as one combination launch
                field(index[e], frac[e], U, K[0], ds * 0.125)
                _combine(U, K[:1], (1.0 / 3,), ds, out=V)
                field(index[e + 1], frac[e + 1], V, K[1], ds * 0.375)
                _combine(U, K[:2], (-1.0 / 3, 1.0), ds, out=V)
                field(index[e + 2], frac[e + 2], V, K[2], ds * 0.375)
                _combine(U, K[:3], (1.0, -1.0, 1.0), ds, out=V)
                field(index[e + 3], frac[e + 3], V, K[3], ds * 0.125)
                _combine(U, K, (0.125, 0.375, 0.375, 0.125), ds, out=U)
                e += 4
            elif method == "midpoint":
                field(index[e], frac[e], U, K[0], 0.0)
                torch.add(U, K[0], alpha=ds / 2, out=V)
                field(index[e + 1], frac[e + 1], V, K[1], ds)
                U.add_(K[1], alpha=ds)
                e += 2
            else:
                field(index[e], frac[e], U, K[0], ds)
                U.add_(K[0], alpha=ds)
                e += 1
        a_y = U[1] + grad_ys[i - 1]
    return a_y, grads


def solve_with_adjoint(forward_solve, vf, times, solve_aug, y0, params, fused_vjp=None, fixed_spec=None, t_tensor=None,
                       flipped=False):
    """``forward_solve(y0) -> ys`` (time first); ``vf(t_float, y)`` differentiable in y and ``params``.

    ``fused_vjp(params)``, if given, returns ``None`` or a callable ``(t, y, a, scale) -> (f, scale * a^T df/dy,
    [scale * a^T df/dp for p in params])`` that replaces autograd in the backward solve."""
    params = tuple(p for p in params if p.requires_grad and p is not t_tensor)
    stage = fused_vjp(params) if fused_vjp is not None else None
    return _Adjoint.apply(forward_solve, vf, times, solve_aug, stage, fixed_spec, flipped, t_tensor, y0, *params)
