"""``cdeint`` -- the host side of hot path (ii).

Same signature, validation, exception types/messages, defaults and output layout as the
reference adapter (torchcde/solver.py:144-245).  What differs is what happens where the
reference leaves for torchdiffeq (solver.py:226-227): nothing is dispatched to torchdiffeq or
torchsde.  For the fixed-step methods the whole solve -- spline derivative, vector field,
contraction, Runge-Kutta combination, output interpolation -- is ONE launch of the fused
kernel (``tcde_cdeint_fixed_linear``) when the vector field is the README-form linear map;
any other ``func`` runs through this package's own on-GPU stage loop, which keeps the
reference's arithmetic but issues no per-stage host syncs.
"""
import bisect
import math
import warnings
import weakref

import numpy as np

import torch

from . import _lib, adaptive
from .controls import CubicSpline, LinearInterpolation, _schedule_knots
from .schedule import FIXED_METHODS, ScheduleCache, build_schedule, locate

_schedules = ScheduleCache()


# ------------------------------------------------------------------------------ vector fields
class LinearVectorField(torch.nn.Module):
    """The README's vector field (README.md:42-49): ``Linear(H, H*C)(z).view(..., H, C)``.

    ``cdeint`` recognises this class (and structurally identical user modules) and fuses it.
    """

    def __init__(self, hidden_channels, input_channels, bias=True, device=None, dtype=None):
        super().__init__()
        self.hidden_channels = hidden_channels
        self.input_channels = input_channels
        self.linear = torch.nn.Linear(hidden_channels, hidden_channels * input_channels, bias=bias, device=device,
                                      dtype=dtype)

    def forward(self, t, z):
        return self.linear(z).view(*z.shape[:-1], self.hidden_channels, self.input_channels)


_recognised = weakref.WeakKeyDictionary()


def _single_linear(func):
    """The one ``nn.Linear`` of ``func`` if ``func`` consists of nothing else, otherwise None."""
    if not isinstance(func, torch.nn.Module) or hasattr(func, "prod"):
        return None
    mods = [m for m in func.modules() if m is not func]
    if len(mods) != 1 or not isinstance(mods[0], torch.nn.Linear):
        return None
    if len(list(func.parameters())) != len(list(mods[0].parameters())) or len(list(func.buffers())) != 0:
        return None
    return mods[0]


def linear_field_of(func, z0, channels, times):
    """Return ``(weight, bias)`` if ``func(t, z)`` is exactly ``Linear(H, H*C)(z).view(..., H, C)``.

    ``LinearVectorField`` is trusted; any other module made of a single ``nn.Linear`` of the
    right shape is *probed*: it must reproduce the linear map bit for bit on random states at
    several distinct times of the integration interval (so a module that adds an activation, or
    scales by a function of ``t``, is never mistaken for a linear field -- probing at ``(t[0], z0)``
    alone is degenerate for ``z0 == 0`` or ``t[0] in {0, 1}``)."""
    hidden = z0.size(-1)
    if isinstance(func, LinearVectorField):
        lin = func.linear
        if lin.in_features == hidden and lin.out_features == hidden * channels:
            return lin.weight, lin.bias
        return None
    lin = _single_linear(func)
    if lin is None or lin.in_features != hidden or lin.out_features != hidden * channels:
        return None
    try:
        known = _recognised.get(func)
    except TypeError:
        known = None
    if known is None:
        known = _probe(func, lin, z0, channels, times)
        try:
            _recognised[func] = known
        except TypeError:
            pass
    return (lin.weight, lin.bias) if known else None


def _probe(func, lin, z0, channels, times):
    """Bit-exact comparison of ``func`` with its ``nn.Linear`` on random (non-degenerate) states of z0's own
    shape (user modules may hard-code the batch size) at four distinct times, none of them 0 or 1."""
    hidden = z0.size(-1)
    if z0.numel() * channels > (1 << 27):
        # too large to probe at full shape: only the explicit LinearVectorField gets the fused kernel
        return False
    lo, hi = float(times[0]), float(times[-1])
    span = hi - lo if hi != lo else 1.0
    probe_times = [lo + 0.6180339887 * span, lo + 0.2718281828 * span + 0.0137, hi + 0.5772156649, lo - 0.4142135624]
    gen = torch.Generator(device=z0.device).manual_seed(0x5eed)
    with torch.no_grad():
        for i, tv in enumerate(probe_times):
            zp = torch.randn(z0.shape, generator=gen, device=z0.device, dtype=z0.dtype) * (0.5 + 1.3 * i) + 0.21 * i
            tp = torch.tensor(tv, dtype=z0.dtype, device=z0.device)
            try:
                got = func(tp, zp)
            except Exception:
                warnings.warn("torchcde_b200.cdeint: `func` looks like a single nn.Linear but could not be probed. "
                              "Falling back to the generic stage loop; use torchcde_b200.LinearVectorField to get the "
                              "fused kernel.")
                return False
            want = torch.nn.functional.linear(zp, lin.weight, lin.bias).view(*zp.shape[:-1], hidden, channels)
            if not (isinstance(got, torch.Tensor) and got.shape == want.shape and got.dtype == want.dtype
                    and torch.equal(got, want)):
                return False
    return True


def _check_linear_problem(control, weight, bias, z0):
    """One validator for every kernel-backed route (fused solve, kernel field, kernel vjp): the control's
    coefficients, the weight and the bias must share z0's dtype and CUDA device -- the kernels receive raw
    pointers, so a mismatch would be reinterpreted memory, not an exception (the reference raises a dtype /
    device RuntimeError from its torch ops in the same situations)."""
    _lib.require_cuda(z0, control, weight, bias)
    for name, ten in (("the control's coefficients", control), ("func's weight", weight), ("func's bias", bias)):
        if ten is None:
            continue
        if ten.dtype != z0.dtype:
            raise RuntimeError("torchcde_b200.cdeint: z0 is {} but {} are {}; they must match."
                               .format(z0.dtype, name, ten.dtype))
        if ten.device != z0.device:
            raise RuntimeError("torchcde_b200.cdeint: z0 is on {} but {} are on {}; they must be on the same device."
                               .format(z0.device, name, ten.device))


# ------------------------------------------------------------------------------- validation
def _shape_error_base(control_shape, z0):
    if control_shape[:-1] != z0.shape[:-1]:
        raise ValueError("X.derivative did not return a tensor with the same number of batch dimensions as z0. "
                         "X.derivative returned shape {} (meaning {} batch dimensions), whilst z0 has shape {} "
                         "(meaning {} batch dimensions)."
                         "".format(tuple(control_shape), tuple(control_shape[:-1]), tuple(z0.shape),
                                   tuple(z0.shape[:-1])))


def _shape_error_forward(control_shape, system_shape, z0):
    _shape_error_base(control_shape, z0)
    if system_shape[:-2] != z0.shape[:-1]:
        raise ValueError("func did not return a tensor with the same number of batch dimensions as z0. func returned "
                         "shape {} (meaning {} batch dimensions), whilst z0 has shape {} (meaning {} batch"
                         " dimensions)."
                         "".format(tuple(system_shape), tuple(system_shape[:-2]), tuple(z0.shape),
                                   tuple(z0.shape[:-1])))
    if system_shape[-2] != z0.size(-1):
        raise ValueError("func did not return a tensor with the same number of hidden channels as z0. func returned "
                         "shape {} (meaning {} channels), whilst z0 has shape {} (meaning {} channels)."
                         "".format(tuple(system_shape), system_shape[-2], tuple(z0.shape), z0.size(-1)))
    if system_shape[-1] != control_shape[-1]:
        raise ValueError("func did not return a tensor with the same number of input channels as X.derivative "
                         "returned. func returned shape {} (meaning {} channels), whilst X.derivative returned shape "
                         "{} (meaning {} channels)."
                         "".format(tuple(system_shape), system_shape[-1], tuple(control_shape),
                                   control_shape[-1]))


def _shape_error_prod(control_shape, field_shape, z0):
    _shape_error_base(control_shape, z0)
    if field_shape != z0.shape:
        raise ValueError("func.prod did not return a tensor with the same shape as z0. func.prod returned shape {} "
                         "whilst z0 has shape {}."
                         "".format(tuple(field_shape), tuple(z0.shape)))


def _control_signature(X):
    """(kind, batch shape, channels, n_intervals) of a built-in control without evaluating it."""
    if isinstance(X, CubicSpline):
        return _lib.CONTROL_CUBIC, tuple(X._b.shape[:-2]), X._b.size(-1), X._b.size(-2)
    if isinstance(X, LinearInterpolation):
        return _lib.CONTROL_LINEAR, tuple(X._coeffs.shape[:-2]), X._coeffs.size(-1), X._coeffs.size(-2) - 1
    return None


# --------------------------------------------------------------------------------- the solve
def _fused_solve(X, weight, bias, z0, t, method, step_size):
    kind, batch, channels, n_rows = _control_signature(X)
    hidden = z0.size(-1)
    dtype = z0.dtype
    code = _lib.dtype_code(dtype)
    control = X._rows() if kind == _lib.CONTROL_CUBIC else X._derivs
    _check_linear_problem(control, weight, bias, z0)
    with torch.cuda.device(z0.device):
        control = control.detach().reshape(-1, control.size(-2), control.size(-1))
        if not control.is_contiguous():
            control = control.contiguous()
        zf = z0.detach().reshape(-1, hidden).contiguous()
        w = weight.detach().contiguous()
        b = (bias.detach() if bias is not None else torch.zeros(hidden * channels, dtype=dtype, device=z0.device))
        b = b.contiguous()
        sched, (floats, ints, v) = _schedules.get(t, _schedule_knots(X), n_rows, method, step_size, dtype, z0.device)
        out = torch.empty(zf.size(0), sched.n_out, hidden, dtype=dtype, device=z0.device)
        _lib.call("tcde_cdeint_fixed_linear", _lib.ptr(control), kind, n_rows, _lib.ptr(w), _lib.ptr(b),
                  _lib.ptr(zf), _lib.ptr(out), zf.size(0), channels, hidden, _lib.METHODS[method], sched.n_steps,
                  _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), sched.n_out,
                  _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]), float(sched.sign), code,
                  _lib.stream_of(zf))
    return out.view(*z0.shape[:-1], sched.n_out, hidden)


def _derivative_at(X, index, frac):
    """dX/dt from a known interval (Python int) and fraction: the reference's arithmetic
    (interpolation_cubic.py:331-336 / interpolation_linear.py:222-225) as differentiable torch
    ops, without the 0-dim-tensor indexing that forces a host sync per stage."""
    if isinstance(X, CubicSpline):
        inner = X._two_c[..., index, :] + X._three_d[..., index, :] * frac
        return X._b[..., index, :] + inner * frac
    coeffs, knots = X._coeffs, X._t
    return (coeffs[..., index + 1, :] - coeffs[..., index, :]) / (knots[index + 1] - knots[index])


def _generic_solve(X, func, z0, t, method, step_size, is_prod, known_control):
    """This package's own fixed-step driver for an arbitrary ``func`` / ``func.prod``
    (solver.py:117-135 semantics): torch ops on the GPU, differentiable, one pass, no host
    sync inside the time loop for the built-in controls."""
    n_rows = _control_signature(X)[3] if known_control else None
    dtype = z0.dtype
    third, two_thirds_ = 1 / 3, 2 / 3
    if known_control:
        sched = build_schedule(t, _schedule_knots(X), n_rows, method, step_size, dtype)
        idx = sched.stage_index.tolist()
        frac_dev = sched.stage_frac.to(z0.device)
    else:
        sched = build_schedule(t, torch.zeros(2), 1, method, step_size, dtype)
    times_dev = sched.stage_times.to(z0.device)
    dts = sched.step_dt.to(z0.device)
    slopes = sched.out_slope.to(z0.device)
    sign = sched.sign
    if torch.is_grad_enabled() and (t.requires_grad or (known_control and X._t.requires_grad)):
        # gradients with respect to the output times / the knots (test_tricks.py:21-49): the same grid, stage times,
        # fractions and output weights as the host schedule, but as torch expressions of ``t`` and ``X._t`` on the
        # device (torchdiffeq builds its grid from the ``t`` tensor too, so autograd sees the same dependence)
        tt = (t if sign > 0 else -t).to(z0.device)
        n_grid = sched.grid.numel()
        if step_size is None:
            grid_t = tt
        else:
            inner = tt[0] + torch.arange(n_grid - 1, dtype=tt.dtype, device=tt.device) * step_size
            grid_t = torch.cat([inner, tt[-1:]])
        g0, g1 = grid_t[:-1], grid_t[1:]
        gdt = g1 - g0
        if method == "rk4":
            st = torch.stack([g0, g0 + gdt * third, g0 + gdt * two_thirds_, g1], dim=1)
        elif method == "midpoint":
            st = torch.stack([g0, g0 + 0.5 * gdt], dim=1)
        else:
            st = g0.unsqueeze(1)
        times_dev = (st if sign > 0 else -st).to(dtype)
        dts = gdt.to(dtype)
        if known_control:
            index_dev = sched.stage_index.to(z0.device).long()
            frac_dev = times_dev.to(X._t.dtype) - X._t[index_dev]
        steps = sched.out_step.clamp(min=0).to(z0.device).long()
        slopes = ((tt - g0[steps]) / (g1[steps] - g0[steps])).to(dtype)

    def field(i, s, z):
        ts = times_dev[i, s]
        if known_control:
            dx = _derivative_at(X, idx[i][s], frac_dev[i, s])
        else:
            dx = X.derivative(ts)
        if is_prod:
            out = func.prod(ts, z, dx)
        else:
            out = (func(ts, z) @ dx.unsqueeze(-1)).squeeze(-1)
        return out if sign > 0 else -1.0 * out

    outs = [None] * sched.n_out
    j = 0
    while j < sched.n_out and int(sched.out_step[j]) < 0:
        outs[j] = z0
        j += 1
    y = z0
    third, two_thirds = 1 / 3, 2 / 3
    for i in range(sched.n_steps):
        dt = dts[i]
        if method == "rk4":
            k1 = field(i, 0, y)
            k2 = field(i, 1, y + dt * k1 * third)
            k3 = field(i, 2, y + dt * (k2 - k1 * third))
            k4 = field(i, 3, y + dt * (k1 - k2 + k3))
            y1 = y + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
        elif method == "midpoint":
            k1 = field(i, 0, y)
            y1 = y + dt * field(i, 1, y + k1 * (0.5 * dt))
        else:
            y1 = y + dt * field(i, 0, y)
        while j < sched.n_out and int(sched.out_step[j]) == i:
            mode = int(sched.out_mode[j])
            if mode == 0:
                outs[j] = y
            elif mode == 1:
                outs[j] = y1
            else:
                outs[j] = y + slopes[j] * (y1 - y)
            j += 1
        y = y1
    return torch.stack(outs, dim=-2)


# ------------------------------------------------- generic func, no autograd: kernels + optional CUDA graph
_graphs = {}


def _generic_solve_kernels(X, func, z0, t, method, step_size, is_prod, use_graph=False):
    """The fixed-step stage loop for an arbitrary ``func`` when nothing needs a gradient: the control's derivative of
    the four stages of a step is ONE launch of ``tcde_spline_eval`` (the reference: ~10 small kernels and 4 host syncs
    per stage, interpolation_cubic.py:315-336), every Runge-Kutta combination is ONE launch of
    ``tcde_linear_combination``; only ``func`` itself and the ``f @ dX`` contraction stay torch operators (they are the
    user's code).  With ``use_graph`` the whole time loop is captured into a CUDA graph once per (func, X, shapes,
    schedule) and replayed -- for small states the loop is launch-bound (12 launches per stage), which is what a graph
    removes.  The graph reads ``func``'s parameters and X's coefficients from their own storage, so in-place updates of
    either are seen by a replay; a different ``func`` / ``X`` object captures anew."""
    kind, _, channels, n_rows = _control_signature(X)
    dtype, device = z0.dtype, z0.device
    sched = build_schedule(t, _schedule_knots(X), n_rows, method, step_size, dtype)
    n_stages = sched.n_stages
    control = (X._rows() if kind == _lib.CONTROL_CUBIC else X._coeffs).detach()
    knots = X._t.detach().to(device=device, dtype=control.dtype).contiguous()
    index_dev = sched.stage_index.to(device)
    frac_dev = sched.stage_frac.to(device=device, dtype=control.dtype)
    times_dev = sched.stage_times.to(device)
    sign = sched.sign
    from .controls import _eval_kernel
    from .adaptive import _combine

    def run(y0):
        outs = [None] * sched.n_out
        j = 0
        while j < sched.n_out and int(sched.out_step[j]) < 0:
            outs[j] = y0
            j += 1
        y = y0
        for i in range(sched.n_steps):
            # dX/dt of this step's stages: (..., n_stages, C) in one launch
            dxs = _eval_kernel(control, knots, control.size(-2), channels, index_dev[i], frac_dev[i], kind, True)

            def field(s, z):
                ts = times_dev[i, s]
                dx = dxs[..., s, :]
                if is_prod:
                    out = func.prod(ts, z, dx)
                    out = out if sign > 0 else -1.0 * out
                    return out if out.is_contiguous() else out.contiguous()
                # solver.py:129-135: f(t, z) @ dX/dt as one streaming launch (the sign of a reversed solve folded in)
                f = func(ts, z)
                if (f.shape != z.shape + (channels,) or f.dtype != dtype or dxs.dtype != dtype or not f.is_cuda
                        or dxs.shape[:-2] != z.shape[:-1]):
                    out = (f @ dx.unsqueeze(-1)).squeeze(-1)          # an unusual func output: let torch broadcast / promote
                    out = out if sign > 0 else -1.0 * out
                    return out if out.is_contiguous() else out.contiguous()
                f = f if f.is_contiguous() else f.contiguous()
                out = torch.empty_like(z)
                _lib.call("tcde_field_contract", _lib.ptr(f), _lib.ptr(dx), _lib.ptr(out), z.numel() // z.size(-1), z.size(-1),
                          channels, n_stages * channels, float(sign),
                          _lib.dtype_code(dtype), _lib.stream_of(z))
                return out

            dt = float(sched.step_dt[i])
            if method == "rk4":
                k1 = field(0, y)
                k2 = field(1, _combine(y, [k1], (1 / 3,), dt))
                k3 = field(2, _combine(y, [k1, k2], (-1 / 3, 1.0), dt))
                k4 = field(3, _combine(y, [k1, k2, k3], (1.0, -1.0, 1.0), dt))
                y1 = _combine(y, [k1, k2, k3, k4], (0.125, 0.375, 0.375, 0.125), dt)
            elif method == "midpoint":
                k1 = field(0, y)
                y1 = _combine(y, [field(1, _combine(y, [k1], (0.5,), dt))], (1.0,), dt)
            else:
                y1 = _combine(y, [field(0, y)], (1.0,), dt)
            while j < sched.n_out and int(sched.out_step[j]) == i:
                mode = int(sched.out_mode[j])
                outs[j] = y if mode == 0 else y1 if mode == 1 else _combine(y, [y1, y], (1.0, -1.0), float(sched.out_slope[j]))
                j += 1
            y = y1
        return torch.stack(outs, dim=-2)

    zc = z0.detach().contiguous()
    if not use_graph:
        return run(zc)
    key = (id(func), id(X), tuple(zc.shape), dtype, str(device), method, step_size, tuple(float(v) for v in t.detach().cpu().tolist()))
    hit = _graphs.get(key)
    if hit is None:
        static_in = zc.clone()
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):                      # warm-up outside the capture (lazy initialisations)
            run(static_in)
        torch.cuda.current_stream(device).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = run(static_in)
        # func / X are kept alive because their ids are the key; ``run`` is kept because its closure owns the device
        # copies of the schedule and of the control rows whose addresses the captured kernels read
        hit = (graph, static_in, static_out, func, X, run)
        if len(_graphs) >= 8:
            _graphs.clear()
        _graphs[key] = hit
    graph, static_in, static_out = hit[:3]
    static_in.copy_(zc)
    graph.replay()
    return static_out.clone()


# ------------------------------------------------------- fields for the host-driven drivers
def _host_locator(X, state_dtype):
    """``(t_float, nudge) -> (interval index, fraction)`` with exactly the casts the reference stack
    applies to a stage time (to the state dtype by the solver, to the coefficient dtype by
    ``_interpret_t``), evaluated on the CPU so that no device sync is needed per stage."""
    knots = _schedule_knots(X)
    n_rows = _control_signature(X)[3]
    # scalar version of ``schedule.locate``: numpy scalars round exactly like the tensor casts, ``bisect_left`` is
    # ``torch.bucketize`` (right=False), and none of it goes through the torch dispatcher (this runs once per
    # vector-field evaluation of the adaptive and adjoint drivers)
    state_t = np.dtype(str(state_dtype).replace("torch.", "")).type
    knot_t = np.dtype(str(knots.dtype).replace("torch.", "")).type
    knot_list = knots.tolist()
    knot_vals = [knot_t(v) for v in knot_list]

    def where(t, nudge=0):
        tt = state_t(t)
        if nudge:
            tt = np.nextafter(tt, tt + state_t(1))
        tk = knot_t(tt)
        index = min(max(bisect.bisect_left(knot_list, float(tk)) - 1, 0), n_rows - 1)
        return index, float(tk - knot_vals[index])

    return where


def _kernel_field(X, weight, bias, z0):
    """f(t, y) = (Linear(y).view(H, C)) @ dX/dt(t) as ONE launch of ``tcde_vector_field_linear``."""
    kind, _, channels, n_rows = _control_signature(X)
    hidden = z0.size(-1)
    code = _lib.dtype_code(z0.dtype)
    control = X._rows() if kind == _lib.CONTROL_CUBIC else X._derivs
    _check_linear_problem(control, weight, bias, z0)
    control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
    w = weight.detach().contiguous()
    b = bias.detach().contiguous() if bias is not None else torch.zeros(hidden * channels, dtype=z0.dtype,
                                                                        device=z0.device)
    where = _host_locator(X, z0.dtype)

    def field(t, y, nudge=0):
        index, frac = where(t, nudge)
        yf = y.reshape(-1, hidden)
        if not yf.is_contiguous():
            yf = yf.contiguous()
        out = torch.empty_like(yf)
        with torch.cuda.device(y.device):
            _lib.call("tcde_vector_field_linear", _lib.ptr(control), kind, n_rows, _lib.ptr(w), _lib.ptr(b),
                      _lib.ptr(yf), _lib.ptr(out), yf.size(0), channels, hidden, index, float(frac), code,
                      _lib.stream_of(yf))
        return out.view_as(y)

    return field


def _kernel_vjp(X, weight, bias, z0, params):
    """The adjoint stage of the linear field as ONE launch of ``tcde_vector_field_linear_vjp``:
    ``(t, y, a, scale) -> (f, scale * a^T df/dy, [scale * a^T df/dp for p in params])``, or ``None`` when the
    kernel is not built for this problem (then autograd serves the backward solve)."""
    kind, _, channels, n_rows = _control_signature(X)
    hidden = z0.size(-1)
    roles = []
    for p in params:
        if p is weight:
            roles.append("w")
        elif bias is not None and p is bias:
            roles.append("b")
        else:
            return None                       # a parameter that is not the linear map: autograd knows how
    control_check = X._rows() if kind == _lib.CONTROL_CUBIC else X._derivs
    _check_linear_problem(control_check, weight, bias, z0)
    if z0.dtype != torch.float32:
        return None
    n_paths = z0.numel() // hidden
    scratch_bytes = _lib.load().tcde_vector_field_linear_vjp_scratch_bytes(n_paths, channels, hidden)
    if scratch_bytes < 0:
        return None
    code = _lib.dtype_code(z0.dtype)
    control = X._rows() if kind == _lib.CONTROL_CUBIC else X._derivs
    control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
    w = weight.detach().contiguous()
    b = bias.detach().contiguous() if bias is not None else torch.zeros(hidden * channels, dtype=z0.dtype,
                                                                        device=z0.device)
    scratch = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=z0.device)
    where = _host_locator(X, z0.dtype)
    knots = _schedule_knots(X)

    def launch(index, frac, y, a, f_out, vjp_out, gw, gb, f_scale, vjp_scale, grad_scale):
        with torch.cuda.device(y.device):
            _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(control), kind, n_rows, _lib.ptr(w), _lib.ptr(b),
                      _lib.ptr(y), _lib.ptr(a), _lib.ptr(f_out), _lib.ptr(vjp_out), _lib.ptr(gw), _lib.ptr(gb),
                      _lib.ptr(scratch), y.numel() // hidden, channels, hidden, index, float(frac), float(f_scale),
                      float(vjp_scale), float(grad_scale), code, _lib.stream_of(y))

    def stage(t, y, a, scale):
        index, frac = where(t)
        yf = y.reshape(-1, hidden).contiguous()
        af = a.reshape(-1, hidden).contiguous()
        f = torch.empty_like(yf)
        vjp_y = torch.empty_like(yf)
        gw = torch.zeros_like(w) if "w" in roles else None
        gb = torch.zeros_like(b) if "b" in roles else None
        launch(index, frac, yf, af, f, vjp_y, gw, gb, 1.0, scale, scale)
        return f.view_as(y), vjp_y.view_as(y), [gw if r == "w" else gb for r in roles]

    def locate_many(times):
        """Interval index / fraction of a list of stage times, with the casts of ``_host_locator``, in one go."""
        tt = torch.tensor(times, dtype=torch.float64).to(z0.dtype)
        frac, index = locate(knots, tt.to(knots.dtype), n_rows)
        return index.tolist(), frac.tolist()

    regrouped = []            # -W with rows regrouped as (k, c) and columns h: the "weight" of the adjoint state's own CDE

    def segment(t_hi, t_lo, y_hi, a_hi, method, step_size, gw, gb):
        """One segment [t_hi -> t_lo] of a fixed-step backward solve WITHOUT a launch per stage.  For this linear
        field d a/ds = a^T df/dz does not involve z, so z(s) and a(s) are two ordinary fused solves (tensor-core
        kernel, reversed time), each leaving the input of every stage in HBM; one more launch contracts the two
        trajectories with dX/dt and the Runge-Kutta weights into dL/dW, dL/db.  Returns a(t_lo), or None when the
        tensor-core kernel or the memory for the two trajectories (2 x stages x paths x 128 bytes) is not available."""
        lib = _lib.load()
        yf = y_hi.reshape(-1, hidden).contiguous()
        af = a_hi.reshape(-1, hidden).contiguous()
        n_paths = yf.size(0)
        tt = torch.tensor([t_hi, t_lo], dtype=torch.float64)
        sched, (_floats, _ints, v) = _schedules.get(tt, knots, n_rows, method, step_size, z0.dtype, z0.device)
        n_total = sched.n_steps * sched.n_stages
        scratch_bytes = lib.tcde_linear_field_param_grads_scratch_bytes(n_paths, n_total, channels, hidden)
        if scratch_bytes < 0:
            return None
        need = 2 * n_total * n_paths * hidden * 4
        with torch.cuda.device(z0.device):
            free, _total = torch.cuda.mem_get_info()
            if need + scratch_bytes > 0.7 * free:
                return None
            if not regrouped:
                regrouped.append(w.view(hidden, channels, hidden).permute(2, 1, 0).contiguous()
                                 .view(hidden * channels, hidden).neg_())
                regrouped.append(torch.zeros_like(b))
            z_stages = torch.empty(n_total, n_paths, hidden, dtype=z0.dtype, device=z0.device)
            a_stages = torch.empty_like(z_stages)
            ends = torch.empty(2, n_paths, sched.n_out, hidden, dtype=z0.dtype, device=z0.device)
            try:
                for which, (start, dump, ww, bb) in enumerate(((yf, z_stages, w, b),
                                                               (af, a_stages, regrouped[0], regrouped[1]))):
                    _lib.call("tcde_cdeint_fixed_linear_stages", _lib.ptr(control), kind, n_rows, _lib.ptr(ww),
                              _lib.ptr(bb), _lib.ptr(start), _lib.ptr(ends[which]), _lib.ptr(dump), n_paths, channels,
                              hidden, _lib.METHODS[method], sched.n_steps, _lib.ptr(v["step_dt"]),
                              _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), sched.n_out,
                              _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]),
                              float(sched.sign), code, _lib.stream_of(yf))
            except NotImplementedError:
                return None
            rk = {"rk4": (0.125, 0.375, 0.375, 0.125), "midpoint": (0.0, 1.0), "euler": (1.0,)}[method]
            weights = (sched.step_dt.to(torch.float64).unsqueeze(1) * torch.tensor(rk, dtype=torch.float64)).reshape(-1)
            weights = weights.to(z0.dtype).to(z0.device)
            scratch2 = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=z0.device)
            _lib.call("tcde_linear_field_param_grads", _lib.ptr(control), kind, n_rows, _lib.ptr(z_stages),
                      _lib.ptr(a_stages), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), _lib.ptr(weights),
                      n_total, _lib.ptr(gw), _lib.ptr(gb), _lib.ptr(scratch2), n_paths, channels, hidden, 1.0, code,
                      _lib.stream_of(yf))
        return ends[1][:, -1].reshape(a_hi.shape)

    def adaptive_segment(t_hi, t_lo, y_hi, a_hi, rtol, atol, gw, gb, slots_hint):
        """One segment [t_hi -> t_lo] of the dopri5 backward solve with the step controller on the device
        (``tcde_dopri5_linear_paired_attempts``): the state z and the adjoint state a advance as one virtual batch of
        2 x paths under one controller, every attempt leaves the inputs of its five weighted stages in the slot of the
        step it would become, and one launch of the parameter-gradient GEMM over the accepted steps' stages adds
        dL/dW, dL/db into ``gw`` / ``gb``.  Returns a(t_lo), or None (not built for this problem / out of memory / more
        accepted steps than slots) -- the caller then runs the host-driven backward."""
        from . import adaptive
        lib = _lib.load()
        yf = y_hi.reshape(-1, hidden).contiguous()
        af = a_hi.reshape(-1, hidden).contiguous()
        n_paths = yf.size(0)
        if hidden != 32 or channels != 8 or n_paths % 256 != 0 or n_paths == 0:
            return None
        with torch.cuda.device(z0.device):
            if not regrouped:
                regrouped.append(w.view(hidden, channels, hidden).permute(2, 1, 0).contiguous()
                                 .view(hidden * channels, hidden).neg_())
                regrouped.append(torch.zeros_like(b))
            w2, b2 = regrouped
            if not fields:
                fields.append(_kernel_field(X, w, b, z0))
                fields.append(_kernel_field(X, w2, b2, z0))

            def field_v(s_time, v):                  # the virtual batch's slope in s = -t (start slope, Hairer's first step)
                return torch.cat([-fields[0](-s_time, v[:n_paths]), -fields[1](-s_time, v[n_paths:])])

            s0, s1 = -float(t_hi), -float(t_lo)
            v0 = torch.cat([yf, af])
            f0 = field_v(s0, v0)
            dt = adaptive._initial_step(field_v, s0, v0, f0, rtol, atol)
            # trajectory slots: enough for a few hundred accepted steps, at most a quarter of the free memory; when they are
            # full the device pauses, the filled slots are contracted into the gradients and the solve goes on
            free, _total = torch.cuda.mem_get_info()
            per_slot = 2 * 5 * n_paths * hidden * 4
            max_slots = int(min(max(16, slots_hint), 256, 0.25 * free // per_slot))
            if max_slots < 8:
                return None
            dev = z0.device
            state = torch.empty(5, 2 * n_paths, hidden, dtype=torch.float32, device=dev)
            state[0].copy_(v0)
            state[2].copy_(f0)
            grid = lib.tcde_dopri5_linear_grid(2 * n_paths)
            partials = torch.zeros(2, grid, dtype=torch.float64, device=dev)
            ctl = adaptive.initial_control(s0, dt, s1, rtol, atol).to(dev)
            out = torch.empty(2 * n_paths, 2, hidden, dtype=torch.float32, device=dev)
            out[:, 0].copy_(v0)
            out_times = torch.tensor([s0, s1], dtype=torch.float64, device=dev)
            dump_z = torch.empty(max_slots * 5, n_paths, hidden, dtype=torch.float32, device=dev)
            dump_a = torch.empty_like(dump_z)
            q_index = torch.zeros(max_slots * 5, dtype=torch.int32, device=dev)
            q_frac = torch.zeros(max_slots * 5, dtype=torch.float32, device=dev)
            q_weight = torch.zeros(max_slots * 5, dtype=torch.float32, device=dev)
            knots_dev = knots.detach().to(device=dev, dtype=torch.float32).contiguous()
            stream = _lib.stream_of(yf)
            scratch_cache = {}

            def contract(n_steps):                   # dL/dW, dL/db += the quadrature over the first n_steps slots
                n_total = 5 * n_steps
                if n_total <= 0 or (gw is None and gb is None):
                    return
                scratch_bytes = lib.tcde_linear_field_param_grads_scratch_bytes(n_paths, n_total, channels, hidden)
                if scratch_bytes < 0:
                    raise RuntimeError("dopri5 adjoint: the parameter-gradient kernel is not built for this problem")
                if scratch_cache.get("n", 0) < scratch_bytes:
                    scratch_cache["buf"] = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=dev)
                    scratch_cache["n"] = scratch_bytes
                _lib.call("tcde_linear_field_param_grads", _lib.ptr(control), kind, n_rows, _lib.ptr(dump_z), _lib.ptr(dump_a),
                          _lib.ptr(q_index), _lib.ptr(q_frac), _lib.ptr(q_weight), n_total, _lib.ptr(gw), _lib.ptr(gb),
                          _lib.ptr(scratch_cache["buf"]), n_paths, channels, hidden, 1.0, code, stream)

            seq, base, flushes = 0, 0, 0
            while True:
                _lib.call("tcde_dopri5_linear_paired_attempts", _lib.ptr(control), kind, n_rows, _lib.ptr(knots_dev), _lib.ptr(w),
                          _lib.ptr(b), _lib.ptr(w2), _lib.ptr(b2), _lib.ptr(state), _lib.ptr(partials), _lib.ptr(ctl),
                          _lib.ptr(out), _lib.ptr(out_times), 2, n_paths, channels, hidden, -1.0, _lib.ptr(dump_z),
                          _lib.ptr(dump_a), _lib.ptr(q_index), _lib.ptr(q_frac), _lib.ptr(q_weight), max_slots, seq,
                          adaptive._DEVICE_CHUNK, _lib.F32, stream)
                seq += adaptive._DEVICE_CHUNK
                last = ctl[(seq - 1) & 1].cpu()
                if last[adaptive.CTL_DONE] != 0:
                    contract(int(last[adaptive.CTL_NACC]) - base)
                    if last[adaptive.CTL_OVERFLOW] == 0:
                        break
                    # slots full: the filled ones are contracted; hand the slots back and resume where the device paused
                    base = int(last[adaptive.CTL_NACC])
                    flushes += 1
                    resume = last.clone()
                    resume[adaptive.CTL_DONE], resume[adaptive.CTL_OVERFLOW] = 0.0, 0.0
                    resume[adaptive.CTL_BASE] = float(base)
                    ctl[(seq - 1) & 1].copy_(resume)
                    continue
                if not math.isfinite(float(last[adaptive.CTL_DT])) or float(last[adaptive.CTL_DT]) == 0.0 or seq > 10_000_000:
                    raise RuntimeError("dopri5 adjoint: step size underflow / non-finite error estimate at s = {}".format(
                        float(last[adaptive.CTL_T])))
            n_acc = int(last[adaptive.CTL_NACC])
            stage.adaptive_stats = {"n_accepted": n_acc, "n_rejected": int(last[adaptive.CTL_NREJ]), "launches": seq,
                                    "slots": max_slots, "flushes": flushes}
            return out[n_paths:, 1].reshape(a_hi.shape).clone()

    fields = []
    stage.launch = launch
    stage.locate_many = locate_many
    stage.segment = segment
    stage.adaptive_segment = adaptive_segment
    stage.adaptive_spec = None
    stage.roles = roles
    stage.new_grads = lambda: [torch.zeros_like(w) if r == "w" else torch.zeros_like(b) for r in roles]
    return stage


def _torch_field(X, func, is_prod, known_control, z0):
    """The reference's ``_VectorField.forward`` (solver.py:117-135) as differentiable torch ops.  ``t`` is a Python
    float, or a 0-dim tensor when the gradient with respect to time is wanted (the adjoint's time vjps)."""
    where = _host_locator(X, z0.dtype) if known_control else None

    def field(t, y, nudge=0):
        if isinstance(t, torch.Tensor):
            tf = float(t.detach())
            ts = t.to(device=y.device, dtype=z0.dtype)
        else:
            tf = t
            ts = torch.tensor(t, dtype=torch.float64).to(z0.dtype).to(y.device)
        if nudge:
            ts = torch.nextafter(ts, ts + 1)
        if known_control:
            index, frac = where(tf, nudge)
            if torch.is_grad_enabled() and (ts.requires_grad or X._t.requires_grad):
                frac = ts.to(X._t.dtype) - X._t[index]          # differentiable in the time and in the knots
            dx = _derivative_at(X, index, frac)
        else:
            dx = X.derivative(ts)
        if is_prod:
            return func.prod(ts, y, dx)
        return (func(ts, y) @ dx.unsqueeze(-1)).squeeze(-1)

    return field


def _reverse(field):
    return lambda s, y, nudge=0: -1.0 * field(-s, y)


def _time_first_to_reference_layout(out):
    dims = range(1, out.dim() - 1)
    return out.permute(*dims, 0, -1)


def cdeint(X, func, z0, t, adjoint=True, backend="torchdiffeq", **kwargs):
    r"""Solves a system of controlled differential equations
    ``z_t = z_{t_0} + \int_{t_0}^t f(s, z_s) dX_s``  (reference: torchcde/solver.py:144-245).

    Arguments, defaults, errors and the returned layout ``(..., len(t), hidden_channels)`` follow
    the reference.  ``**kwargs`` are the torchdiffeq keyword arguments the reference forwards
    (``method``, ``options={'step_size': ...}``, ``rtol``, ``atol``, ``adjoint_*``).

    Supported in this round: ``backend="torchdiffeq"`` semantics with the fixed-step methods
    ``euler``, ``midpoint`` and ``rk4`` (torchdiffeq's 3/8 rule).  With a ``CubicSpline`` or
    ``LinearInterpolation`` control and a linear ``func`` (``LinearVectorField`` or any module
    that is exactly one ``nn.Linear`` + ``view``) the solve is one fused CUDA kernel.  Gradients:
    ``adjoint=True`` runs this package's continuous-adjoint backward (fused kernels for the linear
    field), ``adjoint=False`` backpropagates through the differentiable generic stage loop.
    """
    # Reduce the default values for the tolerances because CDEs are difficult to solve with the default high tolerances.
    if 'atol' not in kwargs:
        kwargs['atol'] = 1e-6
    if 'rtol' not in kwargs:
        kwargs['rtol'] = 1e-4
    if adjoint:
        if "adjoint_atol" not in kwargs:
            kwargs["adjoint_atol"] = kwargs["atol"]
        if "adjoint_rtol" not in kwargs:
            kwargs["adjoint_rtol"] = kwargs["rtol"]

    if not hasattr(X, 'derivative'):
        raise ValueError("X must have a 'derivative' method.")
    if isinstance(z0, (tuple, list)):
        raise NotImplementedError("torchcde_b200.cdeint: tuple / list states (TupleControl) are outside the fused hot "
                                  "path; pass a single tensor state.")
    if not isinstance(z0, torch.Tensor):
        raise ValueError("z0 must either a tensor or a tuple/list of tensors.")
    if backend == "torchsde":
        raise NotImplementedError("torchcde_b200.cdeint: the torchsde backend is out of scope (SURVEY.md section 2, "
                                  "row 8); use backend='torchdiffeq' semantics with a fixed-step method.")
    if backend != "torchdiffeq":
        raise ValueError(f"Unrecognised backend={backend}")

    method = kwargs.get("method", None) or "dopri5"          # torchdiffeq's default
    options = dict(kwargs.get("options", None) or {})
    if method not in FIXED_METHODS and method != "dopri5":
        raise NotImplementedError(
            "torchcde_b200.cdeint: method={!r} is not built. Available: torchdiffeq's fixed-step {} and the adaptive "
            "'dopri5' (its default).".format(method, FIXED_METHODS))
    step_size = options.pop("step_size", None) if method in FIXED_METHODS else None
    # this package's extension: capture the stage loop of a generic ``func`` in a CUDA graph (see _generic_solve_kernels)
    use_graph = bool(options.pop("cuda_graph", False)) if method in FIXED_METHODS else False
    if method in FIXED_METHODS and options:
        raise NotImplementedError("torchcde_b200.cdeint: unsupported solver options {}".format(sorted(options)))
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(t)

    is_prod = hasattr(func, 'prod')
    sig = _control_signature(X)
    # the ONE host read of the output times (a device->host copy only if the caller put ``t`` on the GPU; the
    # schedule -- grid, interval index of every stage -- is host arithmetic, like torchdiffeq's own grid construction)
    times = [float(v) for v in t.detach().cpu().tolist()]

    if adjoint and 'adjoint_params' not in kwargs:
        for buffer in X.buffers():
            if buffer.requires_grad:
                warnings.warn("One of the inputs to the control path X requires gradients but "
                              "`kwargs['adjoint_params']` has not been passed. This is probably a mistake: these "
                              "inputs will not receive a gradient when using the adjoint method. Either have the input "
                              "not require gradients (if that was unintended), or include it (and every other "
                              "parameter needing gradients) in `adjoint_params`. For example:\n"
                              "```\n"
                              "coeffs = ...\n"
                              "func = ...\n"
                              "X = CubicSpline(coeffs)\n"
                              "adjoint_params = tuple(func.parameters()) + (coeffs,)\n"
                              "cdeint(X=X, func=func, ..., adjoint_params=adjoint_params)\n"
                              "```")

    # ---- what kind of problem is this? -----------------------------------------------------------
    field_params = None
    if sig is not None and not is_prod:
        kind, batch, channels, _ = sig
        field_params = linear_field_of(func, z0, channels, times) if times else None
    if field_params is not None:
        # shapes are checked from metadata: nothing is evaluated on the batch
        _shape_error_forward(batch + (channels,), tuple(z0.shape[:-1]) + (z0.size(-1), channels), z0)
    else:
        # the reference's own compatibility check (solver.py:44-100): one evaluation at t[0]
        _lib.require_cuda(z0)
        control_gradient = X.derivative(t[0].detach())
        if not isinstance(control_gradient, torch.Tensor):
            raise ValueError("z0 is a tensor and so X.derivative must return a tensor as well.")
        if is_prod:
            vector_field = func.prod(t[0], z0, control_gradient)
            if not isinstance(vector_field, torch.Tensor):
                raise ValueError("z0 is a tensor and so func.prod must return a tensor as well.")
            _shape_error_prod(tuple(control_gradient.shape), tuple(vector_field.shape), z0)
        else:
            system = func(t[0], z0)
            if not isinstance(system, torch.Tensor):
                raise ValueError("z0 is a tensor and so func must return a tensor as well.")
            _shape_error_forward(tuple(control_gradient.shape), tuple(system.shape), z0)
    _lib.require_cuda(z0)

    if 'adjoint_params' in kwargs:
        adjoint_params = tuple(kwargs['adjoint_params'])
    else:
        adjoint_params = tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()
    differentiable = (z0, t) + tuple(X.buffers()) + (tuple(func.parameters()) if isinstance(func, torch.nn.Module)
                                                     else ()) + adjoint_params
    wants_grad = torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad
                                                 for x in differentiable)

    flipped = len(times) > 1 and times[0] > times[1]
    if flipped:
        times = [-v for v in times]
    if any(b <= a for a, b in zip(times[:-1], times[1:])):
        raise ValueError("t must be strictly increasing or decreasing")
    if method == "dopri5" and options.get("jump_t", None) is not None:
        jumps = options["jump_t"]
        jumps = jumps.detach().cpu().tolist() if isinstance(jumps, torch.Tensor) else list(jumps)
        options["jump_t"] = sorted(-float(v) for v in jumps) if flipped else sorted(float(v) for v in jumps)

    def fast_field():
        f = _kernel_field(X, field_params[0], field_params[1], z0) if field_params is not None \
            else _torch_field(X, func, is_prod, sig is not None, z0)
        return _reverse(f) if flipped else f

    def autograd_field():
        f = _torch_field(X, func, is_prod, sig is not None, z0)
        return _reverse(f) if flipped else f

    rtol, atol = kwargs['rtol'], kwargs['atol']

    def forward_values(y0):
        """Outputs only, time first, by the fastest route."""
        if method in FIXED_METHODS:
            if field_params is not None:
                try:
                    out = _fused_solve(X, field_params[0], field_params[1], y0, t, method, step_size)
                    return out.movedim(-2, 0)
                except NotImplementedError:
                    # a shape the fused kernels are not built for (e.g. hidden * channels * hidden beyond the
                    # shared-memory budget of the CUDA-core kernel): this package's own stage loop takes any shape
                    pass
            if sig is not None and not torch.is_grad_enabled() and y0.is_cuda and y0.dtype in (torch.float32, torch.float64) \
                    and sig[1] == tuple(y0.shape[:-1]):
                return _generic_solve_kernels(X, func, y0, t, method, step_size, is_prod, use_graph).movedim(-2, 0)
            return _generic_solve(X, func, y0, t, method, step_size, is_prod, sig is not None).movedim(-2, 0)
        if (field_params is not None and adaptive.device_dopri5_available(y0, sig[2]) and not options.get("jump_t")
                and set(options) <= {"first_step", "jump_t"}):
            # config 4's forward pass: the whole adaptive loop on the device, one launch per attempted step
            kind = sig[0]
            control = X._rows() if kind == _lib.CONTROL_CUBIC else X._derivs
            _check_linear_problem(control, field_params[0], field_params[1], y0)
            control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
            bias = field_params[1]
            bias = bias.detach().contiguous() if bias is not None else torch.zeros(
                field_params[0].size(0), dtype=y0.dtype, device=y0.device)
            knots = X._t.detach().to(device=y0.device, dtype=y0.dtype).contiguous()
            out, stats = adaptive.odeint_dopri5_device(control, kind, sig[3], knots, field_params[0].detach().contiguous(), bias,
                                                       fast_field(), y0, times, rtol, atol, -1.0 if flipped else 1.0,
                                                       options.get("first_step"))
            cdeint.last_stats = stats
            return out
        out, solver_obj = adaptive.odeint_dopri5(fast_field(), y0, times, rtol, atol, options)
        cdeint.last_stats = {"n_accepted": solver_obj.n_accepted, "n_rejected": solver_obj.n_rejected,
                             "device_controlled": False}
        return out

    if not wants_grad:
        with torch.no_grad():
            return _time_first_to_reference_layout(forward_values(z0))

    if adjoint:
        a_rtol, a_atol = kwargs["adjoint_rtol"], kwargs["adjoint_atol"]
        a_method = kwargs.get("adjoint_method", None) or method
        a_options = dict(kwargs.get("adjoint_options", None) or ({"step_size": step_size} if step_size else {}))

        def solve_aug(f, v, ts):
            if a_method in FIXED_METHODS:
                return adaptive.odeint_fixed(f, v, ts, a_method, a_options.get("step_size", None))
            return adaptive.odeint_dopri5(f, v, ts, a_rtol, a_atol)[0]

        t_grad = t if t.requires_grad else None

        def fused_vjp(params):
            # decreasing t, gradients with respect to the output times, or parameters that are not the linear map
            # (the control's coefficients or knots in ``adjoint_params``): autograd serves the backward solve
            if field_params is None or flipped or t_grad is not None:
                return None
            st = _kernel_vjp(X, field_params[0], field_params[1], z0, params)
            if (st is not None and a_method not in FIXED_METHODS and adaptive.device_dopri5_available(z0, sig[2])
                    and not kwargs.get("adjoint_options", None)):
                # dopri5 backward with the controller on the device; the forward pass's step count sizes the trajectory slots
                st.adaptive_spec = (a_rtol, a_atol)
            return st

        fixed_spec = (a_method, a_options.get("step_size", None)) if a_method in FIXED_METHODS else None
        ys = adaptive.solve_with_adjoint(forward_values, autograd_field(), times, solve_aug, z0, adjoint_params,
                                         fused_vjp, fixed_spec, t_grad, flipped)
        return _time_first_to_reference_layout(ys)

    # adjoint=False: backpropagate through the solver's own operations, like torchdiffeq.odeint
    if method in FIXED_METHODS:
        return _generic_solve(X, func, z0, t, method, step_size, is_prod, sig is not None)
    targets = None
    if t.requires_grad:
        targets = (-t if flipped else t).to(z0.device)
    ys = adaptive.odeint_dopri5(autograd_field(), z0, times, rtol, atol, options, targets)[0]
    return _time_first_to_reference_layout(ys)
