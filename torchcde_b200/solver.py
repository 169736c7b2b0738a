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
import warnings

import torch

from . import _lib, adaptive
from .controls import CubicSpline, _control_signature, _eval_kernel, _schedule_knots
from .linear_field import (LinearFieldKernels, LinearVectorField, _reverse, dopri5_backprop, fixed_backprop,  # noqa: F401
                           linear_field_of)
from .mlp_field import MlpFieldKernels, dopri5_mlp_backprop, mlp_backprop, mlp_field_of
from .schedule import FIXED_METHODS, build_schedule, host_locator


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
def _stage_loop(sched, y0, fields_of_step):
    """The fixed-step time loop of ``sched`` from ``y0`` when nothing needs a gradient: ``fields_of_step(i)`` evaluates
    dX/dt once for step i and returns ``field(s, z)``, the vector field at stage s of that step.  Every Runge-Kutta
    combination and output interpolation is ONE launch of ``tcde_linear_combination``.  Returns the list of outputs."""
    combine = adaptive._combine
    outs = [None] * sched.n_out
    j = 0
    while j < sched.n_out and int(sched.out_step[j]) < 0:
        outs[j] = y0
        j += 1
    y = y0
    for i in range(sched.n_steps):
        field = fields_of_step(i)
        dt = float(sched.step_dt[i])
        if sched.method == "rk4":
            k1 = field(0, y)
            k2 = field(1, combine(y, [k1], (1 / 3,), dt))
            k3 = field(2, combine(y, [k1, k2], (-1 / 3, 1.0), dt))
            k4 = field(3, combine(y, [k1, k2, k3], (1.0, -1.0, 1.0), dt))
            y1 = combine(y, [k1, k2, k3, k4], (0.125, 0.375, 0.375, 0.125), dt)
        elif sched.method == "midpoint":
            k1 = field(0, y)
            y1 = combine(y, [field(1, combine(y, [k1], (0.5,), dt))], (1.0,), dt)
        else:
            y1 = combine(y, [field(0, y)], (1.0,), dt)
        while j < sched.n_out and int(sched.out_step[j]) == i:
            mode = int(sched.out_mode[j])
            outs[j] = y if mode == 0 else y1 if mode == 1 else combine(y, [y1, y], (1.0, -1.0), float(sched.out_slope[j]))
            j += 1
        y = y1
    return outs


_graphs = {}


def _graph_replay(run, zc, state_key, func, X, method, step_size, t):
    """``run(zc)`` as a replay of a CUDA graph of ``run``, captured once per (func, X, state, schedule) -- for small
    states the stage loop is launch-bound (12 launches per stage), which is what a graph removes.  The graph reads
    ``func``'s parameters and X's coefficients from their own storage, so in-place updates of either
    (``optimizer.step()``) are seen by a replay.  The cache key is everything a replay cannot see change: the ``func``
    and ``X`` objects, the state (``state_key``: its shape, or its members' shapes), dtype and device, the method, step
    and output times, the ``training`` flag of every submodule of ``func`` (a branch on ``self.training`` is baked into
    the capture), and the storage address, shape and dtype of every parameter and buffer of ``func`` and of every buffer
    of ``X`` (``p.data = ...``, ``module.double().float()`` or ``load_state_dict(..., assign=True)`` give a parameter
    new storage, which the captured kernels would not read; a view of the same storage can start at the same address
    with another extent).  The cache entry keeps those tensors alive, so no address in a key can be reused while its
    graph is cached."""
    dtype, device = zc.dtype, zc.device
    modules = list(func.modules()) if isinstance(func, torch.nn.Module) else []
    read = [x for m in modules for x in m.parameters(recurse=False)] + \
        [x for m in modules for x in m.buffers(recurse=False)] + list(X.buffers())
    key = (id(func), id(X), state_key, dtype, str(device), method, step_size,
           tuple(float(v) for v in t.detach().cpu().tolist()), tuple(m.training for m in modules),
           tuple((x.data_ptr(), tuple(x.shape), x.dtype) for x in read))
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
        # func / X are kept alive because their ids are the key, the tensors in ``read`` because their addresses are;
        # ``run`` is kept because its closure owns the device copies of the schedule and of the control rows whose
        # addresses the captured kernels read
        hit = (graph, static_in, static_out, func, X, run, read)
        if len(_graphs) >= 8:
            _graphs.clear()
        _graphs[key] = hit
    graph, static_in, static_out = hit[:3]
    static_in.copy_(zc)
    graph.replay()
    return static_out.clone()


def _generic_solve_kernels(X, func, z0, t, method, step_size, is_prod, use_graph=False):
    """The fixed-step stage loop for an arbitrary ``func`` when nothing needs a gradient: the control's derivative of
    the four stages of a step is ONE launch of ``tcde_spline_eval`` (the reference: ~10 small kernels and 4 host syncs
    per stage, interpolation_cubic.py:315-336), every Runge-Kutta combination is ONE launch of
    ``tcde_linear_combination``; only ``func`` itself and the ``f @ dX`` contraction stay torch operators (they are the
    user's code).  With ``use_graph`` the whole time loop is captured into a CUDA graph and replayed
    (``_graph_replay``)."""
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

    def fields_of_step(i):
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

        return field

    def run(y0):
        return torch.stack(_stage_loop(sched, y0, fields_of_step), dim=-2)

    zc = z0.detach().contiguous()
    if not use_graph:
        return run(zc)
    return _graph_replay(run, zc, tuple(zc.shape), func, X, method, step_size, t)


def _host_locator(X, state_dtype):
    """``schedule.host_locator`` of a built-in control: ``(t_float, nudge) -> (interval index, fraction)``."""
    return host_locator(_schedule_knots(X), _control_signature(X)[3], state_dtype)


def _kernel_field(X, weight, bias, z0):
    """f(t, y) = (Linear(y).view(H, C)) @ dX/dt(t) as ONE launch of ``tcde_vector_field_linear``."""
    return LinearFieldKernels(X, weight, bias, z0).field()


# the one call through which cdeint gets the adjoint stage of a linear field: ``_kernel_vjp(kernels, params)``
_kernel_vjp = LinearFieldKernels.adjoint_stage
# and of the examples' MLP field: ``_mlp_vjp(mlp, params)``
_mlp_vjp = MlpFieldKernels.adjoint_stage


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


def _warn_control_gradients(X, adjoint, kwargs):
    """The reference's warning (solver.py:198-213) when the control needs a gradient the adjoint will not give it."""
    if not (adjoint and 'adjoint_params' not in kwargs):
        return
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


def _oriented_times(times, method, options):
    """A decreasing ``t`` is solved as the increasing ``-t`` (torchdiffeq's reversal); ``options["jump_t"]`` follows."""
    flipped = len(times) > 1 and times[0] > times[1]
    if flipped:
        times = [-v for v in times]
    if any(b <= a for a, b in zip(times[:-1], times[1:])):
        raise ValueError("t must be strictly increasing or decreasing")
    if method == "dopri5" and options.get("jump_t", None) is not None:
        jumps = options["jump_t"]
        jumps = jumps.detach().cpu().tolist() if isinstance(jumps, torch.Tensor) else list(jumps)
        options["jump_t"] = sorted(-float(v) for v in jumps) if flipped else sorted(float(v) for v in jumps)
    return times, flipped


def _time_first_to_reference_layout(out):
    dims = range(1, out.dim() - 1)
    return out.permute(*dims, 0, -1)


def _linear_field_or_check(X, func, z0, t, times, sig, is_prod):
    """``(weight, bias)`` when ``func`` is the README-form linear field on a built-in control, whose shapes are then
    checked from metadata (nothing is evaluated on the batch); otherwise None, after the reference's own compatibility
    check (solver.py:44-100): one evaluation at t[0]."""
    if sig is not None and not is_prod and times:
        field_params = linear_field_of(func, z0, sig[2], times)
        if field_params is not None:
            _shape_error_forward(sig[1] + (sig[2],), tuple(z0.shape[:-1]) + (z0.size(-1), sig[2]), z0)
            return field_params
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
    return None


def _adjoint_params(func, kwargs):
    """``kwargs['adjoint_params']``, by default the parameters of ``func``."""
    if 'adjoint_params' in kwargs:
        return tuple(kwargs['adjoint_params'])
    return tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()


def _wants_grad(states, t, X, func, adjoint_params):
    """Whether grad mode is on and a gradient is wanted for a tensor of ``states``, the output times ``t``, the
    control, ``func`` or ``adjoint_params``."""
    # a user-defined control need not be a module: all it must have is ``derivative``
    differentiable = tuple(states) + (t,) + (tuple(X.buffers()) if isinstance(X, torch.nn.Module) else ()) + \
        (tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()) + adjoint_params
    return torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad for x in differentiable)


def _adjoint_solve(kwargs, method, step_size, norm_of=None):
    """The backward solve of ``adjoint=True``: ``solve_aug(f, v, ts)`` with ``adjoint_method`` (the forward's method by
    default), and ``(method, step_size)`` of that solve when it is a fixed-step one, else None.  ``norm_of(v)``: the
    error norm of a dopri5 backward on the augmented state ``v`` (default RMS)."""
    a_method = kwargs.get("adjoint_method", None) or method
    if a_method in FIXED_METHODS:
        a_options = dict(kwargs.get("adjoint_options", None) or ({"step_size": step_size} if step_size else {}))
        a_step = a_options.get("step_size", None)
        return (lambda f, v, ts: adaptive.odeint_fixed(f, v, ts, a_method, a_step)), (a_method, a_step)
    a_rtol, a_atol = kwargs["adjoint_rtol"], kwargs["adjoint_atol"]

    def solve_aug(f, v, ts):
        return adaptive.odeint_dopri5(f, v, ts, a_rtol, a_atol, norm=None if norm_of is None else norm_of(v))[0]

    return solve_aug, None


def _host_dopri5(field, y0, times, rtol, atol, options, norm=None):
    """The host-driven dopri5 solve of the outputs (``adaptive.odeint_dopri5``); its step counts go to
    ``cdeint.last_stats``."""
    out, solver_obj = adaptive.odeint_dopri5(field, y0, times, rtol, atol, options, norm=norm)
    cdeint.last_stats = {"n_accepted": solver_obj.n_accepted, "n_rejected": solver_obj.n_rejected,
                         "device_controlled": False}
    return out


def cdeint(X, func, z0, t, adjoint=True, backend="torchdiffeq", **kwargs):
    r"""Solves a system of controlled differential equations
    ``z_t = z_{t_0} + \int_{t_0}^t f(s, z_s) dX_s``  (reference: torchcde/solver.py:144-245).

    Arguments, defaults, errors and the returned layout ``(..., len(t), hidden_channels)`` follow
    the reference.  ``**kwargs`` are the torchdiffeq keyword arguments the reference forwards
    (``method``, ``options={'step_size': ...}``, ``rtol``, ``atol``, ``adjoint_*``).

    Supported in this round: ``backend="torchdiffeq"`` semantics with the fixed-step methods
    ``euler``, ``midpoint`` and ``rk4`` (torchdiffeq's 3/8 rule).  With a ``CubicSpline`` or
    ``LinearInterpolation`` control and a linear ``func`` (``LinearVectorField`` or any module
    that is exactly one ``nn.Linear`` + ``view``) the solve is one fused CUDA kernel, and likewise
    for the examples' MLP field (``Linear -> ReLU -> Linear -> tanh``).  The default ``dopri5`` runs
    this package's own adaptive driver; its field is one launch per evaluation for both fields where
    their kernels serve the shape (the MLP's: fp32, hidden * channels <= 32, width <= 128).  Gradients:
    ``adjoint=True`` runs this package's continuous-adjoint backward (fused kernels for the linear
    field, and one call per stage for the MLP field at the same shapes as its dopri5 field, with
    dopri5 or a fixed-step method), ``adjoint=False`` backpropagates through the solve: for the
    linear field at fp32, hidden 32, channels 8 with gradients for z0 / weight / bias in three
    launches (``linear_field.FixedBackprop``), likewise for the examples' MLP field at fp32, hidden
    32, channels 8, width 128 with gradients for z0 and its two layers (``mlp_field.MlpBackprop``),
    for the linear field under dopri5 from a recording device-controlled forward and one transposed
    Dormand-Prince launch per record chunk (``linear_field.Dopri5Backprop``; ``cdeint.last_stats["steps"]``
    then lists the accepted ``(t, dt)``, in ``-t`` for a decreasing ``t``), for the examples' MLP field
    under dopri5 at its CUDA-core shapes from a recording host-driven forward and one transposed
    Dormand-Prince launch per record chunk (``mlp_field.Dopri5MlpBackprop``, same ``last_stats``),
    otherwise through the differentiable generic stage loop.

    ``backend="torchsde"`` is built for ``method="reversible_heun"`` (torchsde's reversible Heun
    method with zero diffusion, fixed step ``dt``, default 1e-3; ``z0`` of shape (batch, hidden),
    increasing ``t``).  ``adjoint=True`` gives the exact gradient of the discrete solve by running it
    backwards algebraically from checkpoints (``reversible.py``); ``t`` receives no gradient.
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
    is_tuple = isinstance(z0, (tuple, list))
    if not is_tuple and not isinstance(z0, torch.Tensor):
        raise ValueError("z0 must either a tensor or a tuple/list of tensors.")
    if backend == "torchsde" and is_tuple:
        raise NotImplementedError("torchcde_b200.cdeint: backend='torchsde' is built for a single tensor state; a tuple / "
                                  "list state (TupleControl) runs with backend='torchdiffeq'.")
    if backend == "torchsde":
        if not isinstance(t, torch.Tensor):
            t = torch.as_tensor(t)
        from .reversible import cdeint_reversible        # (reversible.py builds on this module's helpers)
        return cdeint_reversible(X, func, z0, t, adjoint, kwargs)
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

    if is_tuple:
        # one CDE driven by several controls (TupleControl): the members packed into one state (tuple_solver.py)
        from .tuple_solver import cdeint_tuple
        _warn_control_gradients(X, adjoint, kwargs)
        times, flipped = _oriented_times(times, method, options)
        return cdeint_tuple(X, func, z0, t, adjoint, kwargs, method, step_size, use_graph, options, times, flipped,
                            is_prod)
    _warn_control_gradients(X, adjoint, kwargs)

    # ---- what kind of problem is this? -----------------------------------------------------------
    field_params = _linear_field_or_check(X, func, z0, t, times, sig, is_prod)
    _lib.require_cuda(z0)
    adjoint_params = _adjoint_params(func, kwargs)
    wants_grad = _wants_grad((z0,), t, X, func, adjoint_params)

    times, flipped = _oriented_times(times, method, options)

    def autograd_field():
        f = _torch_field(X, func, is_prod, sig is not None, z0)
        return _reverse(f) if flipped else f

    rtol, atol = kwargs['rtol'], kwargs['atol']

    def host_dopri5_field(owner, y0):
        """The field of the host-driven dopri5 (before ``_reverse``): the kernel owner's where it answers one evaluation,
        else the torch operators."""
        if owner is not None:
            field = owner.field()
            try:
                # one evaluation before the solve: the kernel field refuses a shape (e.g. hidden > 256, or the MLP's
                # tensor-core shape) on every call, so a field that answers here answers every attempt
                field(-times[0] if flipped else times[0], y0)
                return field
            except NotImplementedError:
                pass                                          # the torch-operator field takes any shape
        return _torch_field(X, func, is_prod, sig is not None, z0)

    def forward_values(y0):
        """Outputs only, time first, by the fastest route."""
        if method in FIXED_METHODS:
            if kernels is not None:
                try:
                    return kernels.solve(y0, t, method, step_size).movedim(-2, 0)
                except NotImplementedError:
                    # a shape the fused kernels are not built for (e.g. hidden * channels * hidden beyond the
                    # shared-memory budget of the CUDA-core kernel): this package's own stage loop takes any shape
                    pass
            if mlp is not None:
                try:
                    return mlp.solve(y0, t, method, step_size).movedim(-2, 0)
                except NotImplementedError:
                    # a shape or solve variant the MLP kernels are not built for: the stage loop below
                    pass
            if sig is not None and not torch.is_grad_enabled() and y0.is_cuda and y0.dtype in (torch.float32, torch.float64) \
                    and sig[1] == tuple(y0.shape[:-1]):
                return _generic_solve_kernels(X, func, y0, t, method, step_size, is_prod, use_graph).movedim(-2, 0)
            return _generic_solve(X, func, y0, t, method, step_size, is_prod, sig is not None).movedim(-2, 0)
        if (kernels is not None and adaptive.device_dopri5_available(y0, sig[2]) and not options.get("jump_t")
                and set(options) <= {"first_step", "jump_t"}):
            # config 4's forward pass: the whole adaptive loop on the device, one launch per attempted step
            try:
                out, cdeint.last_stats = kernels.dopri5(y0, times, rtol, atol, -1.0 if flipped else 1.0,
                                                        options.get("first_step"))
                return out
            except NotImplementedError:
                # a problem the device controller is not built for (e.g. control rows off a 16-byte boundary): the
                # host-driven loop below takes it, with the kernel field
                pass

        field = host_dopri5_field(kernels if kernels is not None else mlp, y0)
        return _host_dopri5(_reverse(field) if flipped else field, y0, times, rtol, atol, options)

    # adjoint=False with gradients: the kernel routes serve gradients for z0 and the field's parameters; a gradient for
    # anything else (t, the control's knots or coefficients) keeps the torch-operator solve
    route_may_serve = (not adjoint and wants_grad and sig is not None and not t.requires_grad
                       and not any(b.requires_grad for b in X.buffers()))
    # the routes that call a kernel own the problem; building it checks dtypes and devices (the adjoint=False routes
    # build their own where they serve the problem)
    kernel_forward = adjoint or not wants_grad
    kernels = None
    if field_params is not None and kernel_forward:
        kernels = LinearFieldKernels(X, field_params[0], field_params[1], z0)
    # the examples' MLP field: the fixed-step forward is one launch, a dopri5 field evaluation and an adjoint stage one
    # call each where its CUDA-core kernels serve the shape
    mlp_params = mlp = None
    if field_params is None and sig is not None and not is_prod and times and (kernel_forward or route_may_serve):
        mlp_params = mlp_field_of(func, z0, sig[2], times)
        if mlp_params is not None and kernel_forward:
            mlp = MlpFieldKernels(X, mlp_params, z0)

    if not wants_grad:
        with torch.no_grad():
            return _time_first_to_reference_layout(forward_values(z0))

    if adjoint:
        solve_aug, fixed_spec = _adjoint_solve(kwargs, method, step_size)
        t_grad = t if t.requires_grad else None

        def fused_vjp(params):
            # decreasing t, gradients with respect to the output times, or parameters that are not the field's own
            # (the control's coefficients or knots in ``adjoint_params``): autograd serves the backward solve
            if flipped or t_grad is not None:
                return None
            if kernels is None:
                return _mlp_vjp(mlp, params) if mlp is not None else None
            st = _kernel_vjp(kernels, params)
            if (st is not None and fixed_spec is None and adaptive.device_dopri5_available(z0, sig[2])
                    and not kwargs.get("adjoint_options", None)):
                # dopri5 backward with the controller on the device; the forward pass's step count sizes the trajectory slots
                st.adaptive_spec = (kwargs["adjoint_rtol"], kwargs["adjoint_atol"])
            return st

        ys = adaptive.solve_with_adjoint(forward_values, autograd_field(), times, solve_aug, z0, adjoint_params,
                                         fused_vjp, fixed_spec, t_grad, flipped)
        return _time_first_to_reference_layout(ys)

    # adjoint=False: backpropagate through the solver's own operations, like torchdiffeq.odeint, or through a kernel
    # route's solve where one serves the problem (linear_field.FixedBackprop / Dopri5Backprop, mlp_field.MlpBackprop /
    # Dopri5MlpBackprop)
    if method in FIXED_METHODS:
        loop = lambda y0: _generic_solve(X, func, y0, t, method, step_size, is_prod, True)  # noqa: E731
        ys = None
        if route_may_serve and field_params is not None:
            ys = fixed_backprop(X, field_params, z0, t, method, step_size, loop)
        elif route_may_serve and mlp_params is not None:
            ys = mlp_backprop(X, mlp_params, z0, t, method, step_size, loop)
        return ys if ys is not None else _generic_solve(X, func, z0, t, method, step_size, is_prod, sig is not None)

    def replay(steps):
        return lambda y0: _time_first_to_reference_layout(
            adaptive.odeint_dopri5(autograd_field(), y0, times, rtol, atol, options, steps=steps)[0])

    sign, done = -1.0 if flipped else 1.0, None
    if route_may_serve and field_params is not None:
        done = dopri5_backprop(X, field_params, z0, times, rtol, atol, sign, options, replay)
    elif route_may_serve and mlp_params is not None:
        # the dopri5 field of the same call without gradients
        done = dopri5_mlp_backprop(X, mlp_params, z0, lambda owner: host_dopri5_field(owner, z0), times, rtol, atol, sign,
                                   options, replay)
    if done is not None:
        ys, cdeint.last_stats = done
        return ys
    targets = None
    if t.requires_grad:
        targets = (-t if flipped else t).to(z0.device)
    ys = adaptive.odeint_dopri5(autograd_field(), z0, times, rtol, atol, options, targets)[0]
    return _time_first_to_reference_layout(ys)
