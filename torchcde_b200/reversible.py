"""``cdeint(..., backend="torchsde", method="reversible_heun")``: torchsde's reversible Heun method for a CDE, whose
diffusion is zero (the reference's ``_VectorField`` has ``g = 0``), and its exact, checkpointed reversible backward.

Forward.  torchsde's fixed-step ``integrate`` loop (``schedule.build_sde_schedule``: grid by repeated addition of ``dt``
in ``t``'s dtype, last step clipped, outputs by linear interpolation between the bracketing grid states) with the step

    z_{n+1} = 2 y_n - z_n + f_n dt_n,   f_{n+1} = f(t_{n+1}, z_{n+1}),   y_{n+1} = y_n + (f_n + f_{n+1}) (0.5 dt_n)

from ``z_0 = y_0``, ``f_0 = f(t_0, y_0)``: one evaluation of the vector field per step.  On a built-in control the whole
solve is one launch of the kernel owner's forward: ``tcde_cdeint_reversible_heun_linear`` for the README's linear field,
``tcde_cdeint_reversible_heun_mlp`` for the examples' MLP field where the C dispatch serves its shape; any other ``func``
runs as torch operators (differentiable, which is what ``adjoint=False`` backpropagates through).

Backward (``adjoint=True``).  The gradient of the discrete forward solve, found by running the step backwards
algebraically -- ``z_n = 2 y_{n+1} - z_{n+1} - f_{n+1} dt_n``, ``f_n = F(n, z_n)``, ``y_n = y_{n+1} - (f_n + f_{n+1})
dt_n / 2`` -- while the adjoints of (y, z, f) run the transposed recurrence.  In fp32 the reconstruction drifts (the
backward dynamics amplify rounding), so the forward keeps ``(y, z, f)`` every ``CHECKPOINT_STRIDE`` steps and at the
end, and each segment of the backward restarts from its saved end state; that is a deliberate departure from torchsde,
which reconstructs the whole solve from the final state.  The memory is the checkpoints plus O(1) states, independent of
the number of output times.  Where the kernels solved the forward and every parameter is one of the field's own, the
kernel owner (``LinearFieldKernels`` or ``MlpFieldKernels``) runs each segment as one segment launch ((z_m, fbar_m)
dumped) and one parameter-gradient launch over that dump: for the linear field in fp32 (hidden 32, channels 8)
``tcde_reversible_heun_linear_backward_segment`` (the two field products of a step on the tensor cores; step N closed by
``tcde_vector_field_linear_vjp``) and ``tcde_linear_field_param_grads``; for the MLP field
``tcde_reversible_heun_mlp_backward_segment`` (one vector-Jacobian pass per step on the CUDA cores, step N closed in the
same launch) and ``tcde_mlp_field_param_grads``.  Otherwise each step is one ``torch.autograd.grad`` of ``F``, which
covers any ``func``, control coefficients in ``adjoint_params`` and the linear field in fp64; an MLP field whose
parameters the kernels do not serve also keeps the torch-operator forward.

``t`` is a constant here: it receives no gradient.

The step count is ``(t[-1] - t[0]) / dt``, and the schedule is built on the host one step at a time, like torchsde's loop.
torchsde's default ``dt = 1e-3`` over a long span therefore means many steps: 255,000 over a span of 255, with
checkpoints of 3 states per 16 steps (about 125 GB at 65,536 paths x 32 hidden).  Pass the step you mean; the forward
refuses a checkpoint buffer that does not fit in the free device memory, with a message that says so.
"""
import bisect
import types

import torch

from . import _lib
from .controls import _control_signature, _schedule_knots
from .linear_field import LinearFieldKernels, linear_field_of
from .mlp_field import MlpFieldKernels, mlp_field_of
from .schedule import build_sde_schedule, locate
from .solver import _derivative_at, _shape_error_forward, _shape_error_prod

# the forward keeps (y, z, f) of every CHECKPOINT_STRIDE-th step; the backward restarts every segment from them
CHECKPOINT_STRIDE = 16
DEFAULT_DT = 1e-3                     # torchsde's default step
_ACCEPTED = {"method", "dt", "adjoint_method", "adjoint_params", "rtol", "atol", "adjoint_rtol", "adjoint_atol",
             "adaptive"}


def _check_arguments(z0, t, kwargs):
    method = kwargs.get("method", None)
    if method != "reversible_heun":
        raise NotImplementedError(
            "torchcde_b200.cdeint: the torchsde backend is built for method='reversible_heun' only (got method={!r}). "
            "midpoint, euler, rk4 and dopri5 are available as backend='torchdiffeq'.".format(method))
    if kwargs.get("adaptive", False):
        raise NotImplementedError("torchcde_b200.cdeint: torchsde backend: adaptive stepping is not built; "
                                  "reversible_heun runs with the fixed step dt.")
    unknown = sorted(set(kwargs) - _ACCEPTED)
    if unknown:
        raise NotImplementedError("torchcde_b200.cdeint: torchsde backend: unsupported arguments {} (built: dt, "
                                  "adjoint_method, adjoint_params)".format(unknown))
    if kwargs.get("adjoint_method", None) not in (None, "adjoint_reversible_heun"):
        raise NotImplementedError("torchcde_b200.cdeint: torchsde backend: adjoint_method={!r} is not built; the backward "
                                  "is 'adjoint_reversible_heun'.".format(kwargs["adjoint_method"]))
    if z0.dim() != 2:
        raise ValueError("torchcde_b200.cdeint: the torchsde backend takes z0 of shape (batch, hidden_channels); got "
                         "shape {}.".format(tuple(z0.shape)))
    if t.dim() != 1 or t.numel() < 2 or not bool((t[1:] > t[:-1]).all()):
        raise ValueError("torchcde_b200.cdeint: the torchsde backend needs t one dimensional and strictly increasing.")
    dt = kwargs.get("dt", None)
    return DEFAULT_DT if dt is None else float(dt)


def _roles(field_params, params):
    """The index in ``field_params`` (a missing bias is None) of every parameter, or None when one is not the field's."""
    roles = []
    for p in params:
        role = next((i for i, q in enumerate(field_params) if q is not None and p is q), None)
        if role is None:
            return None
        roles.append(role)
    return roles


class _Problem:
    """One reversible Heun problem: the schedule, the torch-operator field and, for the linear or the MLP field, the
    kernel owner (``LinearFieldKernels`` or ``MlpFieldKernels``)."""

    def __init__(self, X, func, z0, t, dt, kernels, params):
        self.X, self.func, self.kernels, self.params = X, func, kernels, params
        self.is_prod = hasattr(func, "prod")
        sig = _control_signature(X)
        self.known = sig is not None
        knots = _schedule_knots(X) if self.known else torch.zeros(2, dtype=t.dtype)
        n_rows = sig[3] if self.known else 1
        self.sched = build_sde_schedule(t, knots, n_rows, dt, z0.dtype)
        s = self.sched
        self.dts = s.step_dt.tolist()
        self.n_out = s.n_out
        self.out_step = s.out_step.tolist()
        self.w1 = s.out_slope[:s.n_out].tolist()
        self.w0 = s.out_slope[s.n_out:].tolist()
        self.index = s.stage_index.tolist()
        self.frac_state = s.stage_frac.tolist()
        dev = z0.device
        if self.known:
            # the fraction in the coefficient dtype, as _interpret_t forms it
            frac, _ = locate(knots, s.grid.to(knots.dtype), n_rows)
            self.frac_dev = frac.to(dev)
        self.grid_dev = s.grid.to(dev)

    # ---- the vector field as torch operators --------------------------------------------------------------------------
    def field(self, n, z):
        """F(n, z) = f(t_n, z) dX/dt(t_n)."""
        tn = self.grid_dev[n]
        if self.known:
            dx = _derivative_at(self.X, self.index[n], self.frac_dev[n])
        else:
            dx = self.X.derivative(tn)
        if self.is_prod:
            return self.func.prod(tn, z, dx)
        return (self.func(tn, z) @ dx.unsqueeze(-1)).squeeze(-1)

    def torch_forward(self, y0, keep_checkpoints):
        """The forward solve as torch operators (differentiable when grad mode is on).  Returns the outputs
        ``(batch, n_out, hidden)`` and, with ``keep_checkpoints``, {step: (y, z, f)}."""
        n_steps = self.sched.n_steps
        outs = [None] * self.n_out
        ckpts = {}
        y, z = y0, y0
        f = self.field(0, y0)
        if keep_checkpoints:
            ckpts[0] = (y, z, f)
        j = 0
        while j < self.n_out and self.out_step[j] < 0:
            outs[j] = y0
            j += 1
        for n in range(n_steps):
            d = self.dts[n]
            z1 = 2 * y - z + f * d
            f1 = self.field(n + 1, z1)
            y1 = y + (f + f1) * (0.5 * d)
            while j < self.n_out and self.out_step[j] == n:
                outs[j] = self.w0[j] * y + self.w1[j] * y1
                j += 1
            y, z, f = y1, z1, f1
            if keep_checkpoints and ((n + 1) % CHECKPOINT_STRIDE == 0 or n + 1 == n_steps):
                ckpts[n + 1] = (y, z, f)
        return torch.stack(outs, dim=-2), ckpts

    # ---- the kernels of the linear or the MLP field ------------------------------------------------------------------
    def kernel_forward(self, y0, keep_checkpoints):
        """ONE launch of the kernel owner's solve (``reversible_forward``); the same return values as ``torch_forward``."""
        k, s = self.kernels, self.sched
        n_paths, hidden = y0.size(0), k.hidden
        n_slots = -(-s.n_steps // CHECKPOINT_STRIDE) + 1
        with torch.cuda.device(k.device):
            _floats, _ints, v = s.device_buffers(k.device)
            zf = y0.detach().contiguous()
            out = torch.empty(n_paths, s.n_out, hidden, dtype=k.dtype, device=k.device)
            ck = None
            if keep_checkpoints:
                need = n_slots * 3 * n_paths * hidden * zf.element_size()
                free, _total = torch.cuda.mem_get_info()
                if need > free:
                    raise RuntimeError(
                        "torchcde_b200.cdeint: torchsde backend: {} steps need {:.1f} GiB of checkpoints for the backward "
                        "({} states of {} paths every {} steps), more than the {:.1f} GiB free; use a larger dt."
                        .format(s.n_steps, need / 2 ** 30, 3 * n_slots, n_paths, CHECKPOINT_STRIDE, free / 2 ** 30))
                ck = torch.empty(n_slots, 3, n_paths, hidden, dtype=k.dtype, device=k.device)
            k.reversible_forward(s, v, zf, out, ck, CHECKPOINT_STRIDE)
        ckpts = {}
        if keep_checkpoints:
            ckpts["slots"], ckpts["views"] = ck, v
            for slot in range(n_slots):
                step = min(slot * CHECKPOINT_STRIDE, s.n_steps)
                ckpts[step] = (ck[slot, 0], ck[slot, 1], ck[slot, 2])
        return out, ckpts

    def forward(self, y0, keep_checkpoints=False):
        if self.kernels is not None:
            try:
                return self.kernel_forward(y0, keep_checkpoints)
            except NotImplementedError:
                # a shape the kernels are not built for: the torch-operator solve takes any shape
                self.kernels = None
        return self.torch_forward(y0, keep_checkpoints)

    # ---- the backward -------------------------------------------------------------------------------------------------
    def fused_roles(self, ckpts):
        """The index of every parameter in the kernel owner's ``field_params`` when its segment kernel serves the backward
        (the field solved by the kernel, ``reversible_backward_served``, every parameter one of the field's own), else
        None."""
        k = self.kernels
        if k is None or "slots" not in ckpts or not k.reversible_backward_served:
            return None
        return _roles(k.field_params, self.params)

    def _injection(self, m):
        """The outputs [first, end) whose gradient lands on y_m, and their weights."""
        first = bisect.bisect_left(self.out_step, m - 1)
        end = bisect.bisect_right(self.out_step, m)
        weights = [self.w0[j] if self.out_step[j] == m else (1.0 if self.out_step[j] < 0 else self.w1[j])
                   for j in range(first, end)]
        return first, end, weights

    def fused_backward(self, ckpts, g, roles):
        """The backward with the kernel owner's launches: per checkpoint segment, last first, ``reversible_segment`` (the
        recurrence over the segment, (ybar, zbar) carried between launches, (z_m, fbar_m) dumped; the segment that ends at
        step N also closes it) and ``reversible_param_grads`` over that dump."""
        k, s = self.kernels, self.sched
        n_steps, n_paths, dev = s.n_steps, g.size(0), k.device
        tensors = k.field_tensors
        grads = [torch.zeros_like(tensors[r]) for r in roles]
        by_role = [None] * len(tensors)
        for r, acc in zip(roles, grads):
            if by_role[r] is None:
                by_role[r] = acc
        ck = ckpts["slots"]
        with torch.cuda.device(dev):
            ranges = []
            for m in range(n_steps + 1):
                first, end, _w = self._injection(m)
                ranges += [first, end]
            dump_z = torch.empty(CHECKPOINT_STRIDE + 1, n_paths, k.hidden, dtype=k.dtype, device=dev)
            bw = types.SimpleNamespace(
                problem=self, views=ckpts["views"], inj=torch.tensor(ranges, dtype=torch.int32).to(dev),
                carry=torch.empty(2, n_paths, k.hidden, dtype=k.dtype, device=dev), g=g, last=ck[-1], dump_z=dump_z,
                dump_a=torch.empty_like(dump_z), grads=by_role, stream=_lib.stream_of(g))
            for slot in range(ck.size(0) - 2, -1, -1):
                lo = slot * CHECKPOINT_STRIDE
                hi = min(lo + CHECKPOINT_STRIDE, n_steps)
                n_dump = k.reversible_segment(bw, lo, hi, ck[slot], ck[slot + 1])
                if any(acc is not None for acc in by_role):
                    k.reversible_param_grads(bw, lo, n_dump)
            return bw.carry[0] + bw.carry[1], grads

    def autograd_vjp(self, n, z, a, grads):
        with torch.enable_grad():
            zz = z.detach().requires_grad_(True)
            f = self.field(n, zz)
            got = torch.autograd.grad(f, (zz,) + tuple(self.params), a, allow_unused=True)
        for acc, gi in zip(grads, got[1:]):
            if gi is not None:
                acc.add_(gi)
        return f.detach(), got[0] if got[0] is not None else torch.zeros_like(z)

    def backward(self, ckpts, g):
        """dL/dy0 and dL/dparams of the forward solve that left ``ckpts``, for output gradients ``g``
        ``(batch, n_out, hidden)``."""
        roles = self.fused_roles(ckpts)
        if roles is not None:
            return self.fused_backward(ckpts, g, roles)
        n_steps, dts = self.sched.n_steps, self.dts
        grads = [torch.zeros_like(p) for p in self.params]
        vjp = self.autograd_vjp
        with torch.cuda.device(g.device):
            inject = {}                                  # step -> sum of w g_j that lands on y_step
            for j in range(self.n_out):
                n = self.out_step[j]
                if n < 0:
                    inject[0] = inject.get(0, 0) + g[:, j]
                    continue
                inject[n] = inject.get(n, 0) + self.w0[j] * g[:, j]
                inject[n + 1] = inject.get(n + 1, 0) + self.w1[j] * g[:, j]
            y, z, f = ckpts[n_steps]
            ybar = torch.zeros_like(y) + inject.get(n_steps, 0)
            fbar = ybar * (0.5 * dts[n_steps - 1])
            _f, zbar = vjp(n_steps, z, fbar, grads)
            for m in range(n_steps - 1, -1, -1):
                d = dts[m]
                ybar_m = ybar + 2 * zbar + inject.get(m, 0)
                fbar = ybar * (0.5 * d) + zbar * d
                if m > 0:
                    fbar = fbar + ybar_m * (0.5 * dts[m - 1])
                saved = ckpts.get(m)
                z_m = saved[1] if saved is not None else 2 * y - z - f * d
                f_m, vz = vjp(m, z_m, fbar, grads)
                if saved is not None:
                    y_m, f_m = saved[0], saved[2]
                else:
                    y_m = y - (f_m + f) * (0.5 * d)
                zbar = vz - zbar
                ybar = ybar_m
                y, z, f = y_m, z_m, f_m
            return ybar + zbar, grads


class _ReversibleAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, problem, y0, *params):
        with torch.no_grad():
            out, ckpts = problem.forward(y0, keep_checkpoints=True)
        ctx.problem, ctx.ckpts = problem, ckpts
        return out

    @staticmethod
    def backward(ctx, g):
        with torch.no_grad():
            gy0, gparams = ctx.problem.backward(ctx.ckpts, g.contiguous())
        ctx.ckpts = None
        return (None, gy0) + tuple(gparams)


def _mlp_kernels(X, mlp_params, z0, params):
    """``MlpFieldKernels`` of the recognised MLP field, or None when its kernels cannot serve the problem: a dtype other
    than fp32 / fp64, a parameter or the control on another dtype or device, or (``params`` not None: the adjoint
    backward) a parameter that is not the MLP's own.  Shapes are the C dispatch's call, at the first launch."""
    if z0.dtype not in (torch.float32, torch.float64):
        return None
    if any(p is not None and (p.dtype != z0.dtype or p.device != z0.device) for p in mlp_params):
        return None
    if params is not None and _roles(mlp_params, params) is None:
        return None
    try:
        return MlpFieldKernels(X, mlp_params, z0)
    except RuntimeError:
        return None                      # the control's dtype or device: the torch operators report it as today


def cdeint_reversible(X, func, z0, t, adjoint, kwargs):
    """``cdeint(..., backend="torchsde")``; ``kwargs`` as ``cdeint`` received them (tolerances injected)."""
    dt = _check_arguments(z0, t, kwargs)
    _lib.require_cuda(z0)

    sig = _control_signature(X)
    is_prod = hasattr(func, "prod")
    times = [float(v) for v in t.detach().cpu().tolist()]
    field_params = None
    if sig is not None and not is_prod:
        field_params = linear_field_of(func, z0, sig[2], times)
    if field_params is not None:
        _shape_error_forward(sig[1] + (sig[2],), tuple(z0.shape[:-1]) + (z0.size(-1), sig[2]), z0)
    else:
        dx = X.derivative(t[0].detach())
        if is_prod:
            _shape_error_prod(tuple(dx.shape), tuple(func.prod(t[0], z0, dx).shape), z0)
        else:
            _shape_error_forward(tuple(dx.shape), tuple(func(t[0], z0).shape), z0)

    if "adjoint_params" in kwargs:
        params = tuple(kwargs["adjoint_params"])
    else:
        params = tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()
    differentiable = (z0,) + tuple(X.buffers()) + (tuple(func.parameters()) if isinstance(func, torch.nn.Module)
                                                    else ()) + params
    wants_grad = torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad for x in differentiable)
    grad_params = tuple(p for p in params if isinstance(p, torch.Tensor) and p.requires_grad)

    kernels = None
    if field_params is not None and (adjoint or not wants_grad) and z0.dtype in (torch.float32, torch.float64):
        kernels = LinearFieldKernels(X, field_params[0], field_params[1], z0)
    elif sig is not None and not is_prod and (adjoint or not wants_grad):
        # the examples' MLP field: its kernels serve the forward and, for its own parameters, the backward; anything else
        # keeps the torch-operator forward and the per-step autograd backward
        mlp_params = mlp_field_of(func, z0, sig[2], times)
        if mlp_params is not None:
            kernels = _mlp_kernels(X, mlp_params, z0, grad_params if wants_grad else None)
    problem = _Problem(X, func, z0, t, dt, kernels, params)
    if not wants_grad:
        with torch.no_grad():
            return problem.forward(z0)[0]
    if adjoint:
        problem.params = grad_params
        return _ReversibleAdjoint.apply(problem, z0, *grad_params)
    problem.kernels = None
    return problem.torch_forward(z0, keep_checkpoints=False)[0]
