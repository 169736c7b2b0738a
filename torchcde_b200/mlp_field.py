"""The MLP vector field of the reference's examples and ``MlpFieldKernels``, the owner of its fused fixed-step solve.

example/time_series_classification.py:20-51 trains ``func(t, z) = tanh(Linear(W, H*C)(relu(Linear(H, W)(z)))).view(H, C)``.
``mlp_field_of`` recognises a user module that computes exactly that (no new class to adopt), and ``cdeint`` then runs
its fixed-step forward as ONE launch of ``tcde_cdeint_fixed_mlp``; ``cdeint(..., adjoint=False)`` with gradients runs
``MlpBackprop`` (three launches) where it is built for the problem.  At the CUDA-core shapes ``MlpFieldKernels.field`` and
``MlpAdjointStage`` give the host-driven dopri5 one launch per field evaluation and the ``adjoint=True`` backward one
launch per stage (``tcde_vector_field_mlp`` / ``tcde_vector_field_mlp_vjp``); ``cdeint(..., adjoint=False)`` with dopri5
runs ``Dopri5MlpBackprop`` there (a recording host-driven forward, one backward launch per record chunk).  Under ``backend="torchsde"``
(``reversible.py``) ``MlpFieldKernels`` supplies the reversible Heun forward and its segment backward on the CUDA cores."""
import functools
import math
import weakref

import torch

from . import _lib, adaptive, backprop
from .controls import _control_signature, _schedule_knots
from .linear_field import AdjointStage, _check_linear_problem, _probe, _reverse, _schedules
from .schedule import backward_views, host_locator

# module -> {training flag: index of the accepted layer ordering, or -1}; kept apart from the linear probe's cache
_recognised = weakref.WeakKeyDictionary()
# submodules that hold no state and behave the same in training and evaluation mode
_STATELESS = (torch.nn.Linear, torch.nn.ReLU, torch.nn.Tanh, torch.nn.Identity, torch.nn.Sequential)


def _two_linears(func):
    """The orderings ``(L1, L2)`` of the two ``nn.Linear`` of ``func`` if its parameters are exactly theirs, it has no
    buffers and every other submodule is a ReLU, Tanh, Identity or Sequential (a Dropout or any module whose forward may
    depend on its mode or state is refused: the probe sees one mode only), otherwise []."""
    if not isinstance(func, torch.nn.Module) or hasattr(func, "prod"):
        return []
    if any(type(m) not in _STATELESS for m in func.modules() if m is not func):
        return []
    lins = [m for m in func.modules() if isinstance(m, torch.nn.Linear)]
    if len(lins) != 2 or len(list(func.buffers())) != 0:
        return []
    own = {id(p) for lin in lins for p in lin.parameters()}
    if {id(p) for p in func.parameters()} != own or len(own) != sum(len(list(lin.parameters())) for lin in lins):
        return []
    return [lins, lins[::-1]]


def _mlp(l1, l2):
    def field(z):
        return torch.tanh(torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(z, l1.weight, l1.bias)),
                                                     l2.weight, l2.bias))
    return field


def mlp_field_of(func, z0, channels, times):
    """Return ``(W1, b1, W2, b2)`` (a bias may be None) if ``func(t, z)`` is exactly
    ``tanh(F.linear(relu(F.linear(z, W1, b1)), W2, b2)).view(..., H, C)`` for two ``nn.Linear`` of ``func``, else None.

    Like ``linear_field_of``, the module is *probed*: it must reproduce that map bit for bit on random states at four
    times of the integration interval, so a module with another activation, no tanh, a dependence on ``t``, a scaled
    output or a third layer is never taken for it.  Both orderings of the two layers are tried when both fit the shapes.
    The outcome is cached per module and training flag."""
    hidden = z0.size(-1)
    fits = [(l1, l2) for l1, l2 in _two_linears(func) if l1.in_features == hidden
            and l2.in_features == l1.out_features and l2.out_features == hidden * channels]
    if not fits:
        return None
    if z0.numel() * channels > (1 << 27):
        return None                       # too large to probe at this batch size; not a verdict on the module
    # the verdict is kept per training flag: the module's own forward may branch on it
    try:
        verdicts = _recognised.setdefault(func, {})
    except TypeError:
        verdicts = {}
    known = verdicts.get(func.training)
    if known is None:
        known = next((i for i, (l1, l2) in enumerate(fits)
                      if _probe(func, _mlp(l1, l2), z0, channels, times, "a two-layer MLP", None)), -1)
        verdicts[func.training] = known
    if known < 0:
        return None
    l1, l2 = fits[known]
    return l1.weight, l1.bias, l2.weight, l2.bias


class MlpFieldKernels:
    """The fused fixed-step solve of one problem: a built-in control ``X``, the MLP field ``params = (W1, b1, W2, b2)``
    (a bias may be None: zeros are passed) and the state ``z0``.  Construction validates dtypes and devices."""

    def __init__(self, X, params, z0):
        w1, b1, w2, b2 = params
        self.kind, _, self.channels, self.n_rows = _control_signature(X)
        self.hidden, self.width = z0.size(-1), w1.size(0)
        self.n_paths = math.prod(z0.shape[:-1])
        self.dtype, self.device = z0.dtype, z0.device
        self.params = params                   # the parameters themselves, to recognise them in adjoint_params
        control = X._rows() if self.kind == _lib.CONTROL_CUBIC else X._derivs
        _check_linear_problem(control, w1, b1, z0)
        _check_linear_problem(control, w2, b2, z0)
        self.control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
        zeros = lambda n: torch.zeros(n, dtype=z0.dtype, device=z0.device)  # noqa: E731
        self.w1, self.w2 = w1.detach().contiguous(), w2.detach().contiguous()
        self.b1 = (b1.detach() if b1 is not None else zeros(self.width)).contiguous()
        self.b2 = (b2.detach() if b2 is not None else zeros(self.hidden * self.channels)).contiguous()
        self.knots = _schedule_knots(X)

    def solve(self, y0, t, method, step_size):
        """The fixed-step solve as ONE launch of ``tcde_cdeint_fixed_mlp``: ``(..., len(t), H)``.  Raises
        NotImplementedError for a shape or solve variant no kernel is built for."""
        with torch.cuda.device(self.device):
            zf = y0.detach().reshape(-1, self.hidden).contiguous()
            sched, (_floats, _ints, v) = _schedules.get(t, self.knots, self.n_rows, method, step_size, self.dtype,
                                                        self.device)
            out = torch.empty(zf.size(0), sched.n_out, self.hidden, dtype=self.dtype, device=self.device)
            if zf.size(0) > 0:            # an empty batch: nothing to launch (its null data pointers would be refused)
                _lib.call("tcde_cdeint_fixed_mlp", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w1),
                          _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(zf), _lib.ptr(out),
                          zf.size(0), self.channels, self.hidden, self.width, _lib.METHODS[sched.method],
                          sched.n_steps, _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]),
                          sched.n_out, _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]),
                          float(sched.sign), _lib.dtype_code(self.dtype), _lib.stream_of(zf))
        return out.view(*y0.shape[:-1], sched.n_out, self.hidden)

    @functools.cached_property
    def where(self):
        """``(t, nudge) -> (interval index, fraction)`` of a stage time: ``schedule.host_locator``."""
        return host_locator(self.knots, self.n_rows, self.dtype)

    def field(self):
        """f(t, y) = tanh(W2 relu(W1 y + b1) + b2).view(H, C) @ dX/dt(t) as ONE launch of ``tcde_vector_field_mlp``.
        Raises NotImplementedError, on every call, for a shape, dtype or solve variant the kernel is not built for."""
        hidden = self.hidden
        code = _lib.dtype_code(self.dtype)

        def field(t, y, nudge=0):
            index, frac = self.where(t, nudge)
            yf = y.reshape(-1, hidden).contiguous()
            out = torch.empty_like(yf)
            if yf.size(0) == 0:           # an empty batch: nothing to launch (its null data pointers would be refused)
                return out.view_as(y)
            with torch.cuda.device(y.device):
                _lib.call("tcde_vector_field_mlp", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w1),
                          _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(yf), _lib.ptr(out), yf.size(0),
                          self.channels, hidden, self.width, index, float(frac), code, _lib.stream_of(yf))
            return out.view_as(y)

        return field

    # ---- torchsde's reversible Heun (reversible._Problem): the forward, the segment backward, the parameter gradients ----
    # Which shapes, dtypes and solve variants they serve is the C dispatch's call; where it admits the forward it serves the
    # backward.  A missing bias is the kernels' zero vector, which takes no gradient.
    reversible_backward_served = True

    @property
    def field_params(self):
        return self.params

    @property
    def field_tensors(self):
        return self.w1, self.b1, self.w2, self.b2

    def reversible_forward(self, sched, v, z0, out, ckpt, stride):
        """ONE launch of ``tcde_cdeint_reversible_heun_mlp``; NotImplementedError where it is not built."""
        _lib.call("tcde_cdeint_reversible_heun_mlp", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w1),
                  _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(z0), _lib.ptr(out), _lib.ptr(ckpt),
                  stride, z0.size(0), self.channels, self.hidden, self.width, sched.n_steps, _lib.ptr(v["step_dt"]),
                  _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), sched.n_out, _lib.ptr(v["out_step"]),
                  _lib.ptr(v["out_slope"]), _lib.dtype_code(self.dtype), _lib.stream_of(z0))

    def reversible_segment(self, bw, lo, hi, ck_lo, ck_hi):
        """ONE launch of ``tcde_reversible_heun_mlp_backward_segment`` over steps [lo, hi] (the segment that ends at step N
        also closes it and dumps it last).  Returns the number of dumped steps."""
        p, v = bw.problem, bw.views
        n_steps = p.sched.n_steps
        _lib.call("tcde_reversible_heun_mlp_backward_segment", _lib.ptr(self.control), self.kind, self.n_rows,
                  _lib.ptr(self.w1), _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(ck_lo),
                  _lib.ptr(ck_hi), _lib.ptr(bw.carry), _lib.ptr(bw.g), p.n_out, _lib.ptr(v["out_step"]),
                  _lib.ptr(v["out_slope"]), _lib.ptr(bw.inj), n_steps, _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]),
                  _lib.ptr(v["stage_frac"]), lo, hi, bw.g.size(0), self.channels, self.hidden, self.width,
                  _lib.ptr(bw.dump_z), _lib.ptr(bw.dump_a), _lib.dtype_code(self.dtype), bw.stream)
        return hi - lo + (1 if hi == n_steps else 0)

    def reversible_param_grads(self, bw, lo, n):
        """dW1, db1, dW2, db2 += the segment's dump of ``n`` steps from ``lo`` (``param_grads``, its scratch kept on ``bw``)."""
        if getattr(bw, "scratch", None) is None:
            bw.scratch = self.param_grad_scratch(bw.g.size(0), bw.dump_z.size(0))
        v = bw.views
        self.param_grads(bw.dump_z, bw.dump_a, v["stage_index"][lo:], v["stage_frac"][lo:], n, bw.grads, bw.scratch)

    def param_grad_scratch_bytes(self, n_paths, n_total):
        return _lib.load().tcde_mlp_field_param_grads_scratch_bytes(n_paths, n_total, self.channels, self.hidden,
                                                                    self.width)

    def param_grad_scratch(self, n_paths, n_total):
        """The scratch of ``param_grads`` for ``n_paths`` paths and up to ``n_total`` stages."""
        return torch.empty(max(self.param_grad_scratch_bytes(n_paths, n_total) // 4, 4), dtype=torch.float32,
                           device=self.device)

    def param_grads(self, z_stages, a_stages, index, frac, n_total, grads, scratch, weight=1.0):
        """``grads`` (dW1, db1, dW2, db2, None where not wanted) += ``weight`` times the sum over ``n_total`` stages of
        a^T df/dtheta at the stage inputs ``z_stages`` and cotangents ``a_stages`` ``[stage][paths][H]`` (``z_stages`` may
        keep the batch shape): ONE call of ``tcde_mlp_field_param_grads`` (its kernel and its fixed-order reduction)."""
        _lib.call("tcde_mlp_field_param_grads", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w1),
                  _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(z_stages), _lib.ptr(a_stages),
                  _lib.ptr(index), _lib.ptr(frac), n_total, *(_lib.ptr(g) for g in grads), _lib.ptr(scratch),
                  a_stages.size(1), self.channels, self.hidden, self.width, float(weight), 1.0,
                  _lib.dtype_code(self.dtype), _lib.stream_of(z_stages))

    def adjoint_stage(self, params):
        """The adjoint stage of this problem for ``params``, or None when the kernel is not built for it (then autograd
        serves the backward solve): every parameter must be W1, b1, W2 or b2, and the shape one the CUDA-core kernels
        serve (the scratch query answers -1 elsewhere, the tensor-core shape included)."""
        roles = []
        for p in params:
            role = next((i for i, q in enumerate(self.params) if q is not None and p is q), None)
            if role is None:
                return None                       # a parameter that is not the MLP's: autograd knows how
            roles.append(role)
        if self.dtype not in (torch.float32, torch.float64):
            return None
        scratch_bytes = _lib.load().tcde_vector_field_mlp_vjp_scratch_bytes(self.n_paths, self.channels, self.hidden,
                                                                             self.width)
        if scratch_bytes < 0:
            return None
        # one scratch per backward: the stage's launches reuse it
        scratch = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=self.device)
        # the scratch query has no dtype: the dispatch's verdict on this dtype and solve variant comes from a call with
        # no paths, which validates the problem and launches nothing (the scratch stands in for the per-path buffers,
        # the control's among them, which is empty for an empty batch)
        s = _lib.ptr(scratch)
        try:
            with torch.cuda.device(self.device):
                _lib.call("tcde_vector_field_mlp_vjp", s, self.kind, self.n_rows, _lib.ptr(self.w1),
                          _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), s, s, s, s, None, None, None, None, s,
                          0, self.channels, self.hidden, self.width, 0, 0.0, 1.0, 1.0, 1.0, _lib.dtype_code(self.dtype),
                          _lib.stream_of(scratch))
        except NotImplementedError:
            return None
        return MlpAdjointStage(self, roles, scratch)


class MlpAdjointStage:
    """The adjoint stage of the MLP field: ``stage(t, y, a, scale) -> (f, scale * a^T df/dy, [scale * a^T df/dp for p in
    params])`` as ONE call of ``tcde_vector_field_mlp_vjp`` (at most three launches), with what ``adaptive._Adjoint`` and
    ``adaptive._fused_fixed_backward`` use of ``linear_field.AdjointStage``; it has no whole-segment route and no
    device-controlled dopri5 backward.  ``roles``: the index in (W1, b1, W2, b2) of each parameter."""

    adaptive_spec = None

    def __init__(self, kernels, roles, scratch):
        self.kernels, self.roles, self.scratch = kernels, roles, scratch

    def _tensors(self):
        k = self.kernels
        return k.w1, k.b1, k.w2, k.b2

    def new_grads(self):
        return [torch.zeros_like(self._tensors()[r]) for r in self.roles]

    def launch(self, index, frac, y, a, f_out, vjp_out, *grads, f_scale, vjp_scale, grad_scale):
        """``grads``: one tensor (or None) per parameter, in the order of ``params``, += grad_scale * a^T df/dp."""
        k = self.kernels
        slots = [None] * 4
        for r, g in zip(self.roles, grads):
            slots[r] = g
        if y.numel() == 0:
            return
        with torch.cuda.device(y.device):
            _lib.call("tcde_vector_field_mlp_vjp", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1), _lib.ptr(k.b1),
                      _lib.ptr(k.w2), _lib.ptr(k.b2), _lib.ptr(y), _lib.ptr(a), _lib.ptr(f_out), _lib.ptr(vjp_out),
                      *(_lib.ptr(g) for g in slots), _lib.ptr(self.scratch), y.numel() // k.hidden, k.channels,
                      k.hidden, k.width, index, float(frac), float(f_scale), float(vjp_scale), float(grad_scale),
                      _lib.dtype_code(k.dtype), _lib.stream_of(y))

    def __call__(self, t, y, a, scale):
        k = self.kernels
        index, frac = k.where(t)
        yf = y.reshape(-1, k.hidden).contiguous()
        af = a.reshape(-1, k.hidden).contiguous()
        f = torch.empty_like(yf)
        vjp_y = torch.empty_like(yf)
        grads = self.new_grads()
        self.launch(index, frac, yf, af, f, vjp_y, *grads, f_scale=1.0, vjp_scale=scale, grad_scale=scale)
        return f.view_as(y), vjp_y.view_as(y), grads

    locate_many = AdjointStage.locate_many

    def segment(self, *args):
        """No whole-segment backward for this field: the fixed-step backward runs stage by stage."""
        return None


class MlpBackprop:
    """``cdeint(..., adjoint=False)`` of a fixed-step solve of the MLP field with gradients for any of z0, W1, b1, W2, b2:
    the exact gradient of the discrete solve in three launches, as
    ``linear_field.FixedBackprop`` does for the linear field, on the tensor cores at fp32 32 / 8 / 128 and on the CUDA
    cores (fp32, fp64) where the CUDA-core forward runs by default; the C dispatch owns that policy.  The forward is the
    stage-dump solve
    (``tcde_cdeint_fixed_mlp_stages``: the outputs of the same call without gradients, bit for bit); the backward is ONE
    launch of ``tcde_cdeint_fixed_mlp_backward`` (the transposed Runge-Kutta recurrence over every step at the dumped stage
    inputs) and, with parameter gradients, ONE launch of ``tcde_mlp_field_param_grads`` over the two dumps.
    ``differentiable(z0)``: the torch-operator solve of the same problem, which a backward with ``create_graph``
    differentiates instead."""

    def __init__(self, kernels, t, method, step_size, loop):
        self.kernels, self.method, self.differentiable = kernels, method, loop
        self.sched, (_floats, _ints, self.views) = _schedules.get(t, kernels.knots, kernels.n_rows, method, step_size,
                                                                  kernels.dtype, kernels.device)
        self.n_total = self.sched.n_steps * self.sched.n_stages
        self.want_params = any(p is not None and p.requires_grad for p in kernels.field_params)

    def forward(self, z0):
        """(the outputs ``(..., n_out, H)``, [the input of every stage ``[n_steps * n_stages][paths][H]``]).  Raises
        ``NoRoom`` when the stage dump, and with a parameter gradient its kappa copy and the scratch, do not fit."""
        k, sched, v = self.kernels, self.sched, self.views
        scratch_bytes = k.param_grad_scratch_bytes(k.n_paths, self.n_total) if self.want_params else None
        elt = torch.empty(0, dtype=k.dtype).element_size()
        if not backprop.fits(k.device, self.n_total * k.n_paths * k.hidden * elt, scratch_bytes):
            raise backprop.NoRoom()
        with torch.cuda.device(k.device):
            zf = z0.detach().reshape(-1, k.hidden).contiguous()
            out = torch.empty(zf.size(0), sched.n_out, k.hidden, dtype=k.dtype, device=k.device)
            dump = torch.empty(self.n_total, zf.size(0), k.hidden, dtype=k.dtype, device=k.device)
            if zf.size(0) > 0:
                _lib.call("tcde_cdeint_fixed_mlp_stages", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1),
                          _lib.ptr(k.b1), _lib.ptr(k.w2), _lib.ptr(k.b2), _lib.ptr(zf), _lib.ptr(out), _lib.ptr(dump),
                          zf.size(0), k.channels, k.hidden, k.width, _lib.METHODS[sched.method], sched.n_steps,
                          _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), sched.n_out,
                          _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]), float(sched.sign),
                          _lib.dtype_code(k.dtype), _lib.stream_of(zf))
        return out.view(*z0.shape[:-1], sched.n_out, k.hidden), [dump]

    def backward(self, g, z0, saved, want):
        """(dL/dz0, [dL/dW1, dL/db1, dL/dW2, dL/db2] with None where ``want`` is False) for output gradients ``g``."""
        k, sched = self.kernels, self.sched
        (dump,), hidden, dev = saved, k.hidden, k.device
        with torch.cuda.device(dev):
            gf = backprop.cotangent(g, sched.n_out, hidden)
            n_paths = gf.size(0)
            gz = torch.empty(n_paths, hidden, dtype=k.dtype, device=dev)
            kappa = torch.empty_like(dump) if any(want) else None
            grads = [torch.zeros_like(p) if w else None for p, w in zip((k.w1, k.b1, k.w2, k.b2), want)]
            if n_paths > 0:
                tables = backward_views(sched, dev)
                _lib.call("tcde_cdeint_fixed_mlp_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1),
                          _lib.ptr(k.b1), _lib.ptr(k.w2), _lib.ptr(k.b2), _lib.ptr(dump), _lib.ptr(gf), _lib.ptr(gz),
                          _lib.ptr(kappa), n_paths, k.channels, hidden, k.width, _lib.METHODS[sched.method], sched.n_steps,
                          _lib.ptr(tables["step_dt"]), _lib.ptr(tables["stage_index"]), _lib.ptr(tables["stage_frac"]),
                          sched.n_out, _lib.ptr(tables["inj_range"]), _lib.ptr(tables["inj_out"]),
                          _lib.ptr(tables["inj_weight"]), float(sched.sign), _lib.dtype_code(k.dtype), _lib.stream_of(gf))
                if kappa is not None:
                    k.param_grads(dump, kappa, self.views["stage_index"], self.views["stage_frac"], self.n_total, grads,
                                  k.param_grad_scratch(n_paths, self.n_total), sched.sign)
        return gz.view(g.shape[:-2] + (hidden,)), grads


def _backprop_kernels(X, params, z0):
    """The kernels of a problem the MLP backprop routes may serve (z0 fp32 or fp64 on a CUDA device, the parameters and
    the control of its dtype and device), else None.  Which shapes, dtypes and solve variants are served is the C
    dispatch's call: a refusal (``TCDE_ERR_UNSUPPORTED``, as a -1 scratch size or NotImplementedError) keeps the
    torch-operator solve."""
    if (z0.dtype not in (torch.float32, torch.float64) or not z0.is_cuda
            or any(p is not None and (p.dtype != z0.dtype or p.device != z0.device) for p in params)):
        return None
    k = MlpFieldKernels(X, params, z0)
    if k.control.dtype != z0.dtype or k.control.device != z0.device:
        return None
    return k


def mlp_backprop(X, params, z0, t, method, step_size, loop):
    """``cdeint(..., adjoint=False)``'s outputs ``(..., n_out, H)`` on the three-launch route of ``MlpBackprop``, or None
    when the route does not serve the problem (the caller runs the torch-operator solve ``loop``).  ``params``: (W1, b1,
    W2, b2) of the recognised field, a bias may be None (the kernels' zero vector, which wants no gradient)."""
    k = _backprop_kernels(X, params, z0)
    return None if k is None else backprop.run(MlpBackprop(k, t, method, step_size, loop), z0, params)


class _Located:
    """The field of a host-driven dopri5 that keeps the location ``where(t, nudge)`` of its last evaluation: the
    locator the field itself calls, with the arguments it receives (under ``_reverse`` that is -s without the nudge)."""

    def __init__(self, field, where):
        self.field, self.where, self.loc = field, where, None

    def __call__(self, t, y, nudge=0):
        self.loc = self.where(t, nudge)
        return self.field(t, y, nudge)


class _RecordingDopri5(adaptive.Dopri5):
    """``adaptive.Dopri5`` whose hooks fill the record of ``Dopri5MlpBackprop``: every attempt writes the inputs of its
    evaluations 2..7 into the items of the step it would become (a rejected attempt's are overwritten by the next one), a
    start slope of its own writes its input into the item before them, and the locations come from ``_Located``."""

    def __init__(self, route, located, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.route, self.located = route, located
        self.fresh = None                      # the location of the current step's own start slope, if it has one
        self.locs = [None] * 6

    def _start_slope(self, t, y, *nudge):
        f = super()._start_slope(t, y, *nudge)
        c = self.route.room()
        c["z"][c["items"]].copy_(y)
        self.fresh = self.located.loc
        return f

    def _stage_out(self, s):
        c = self.route.room()
        return c["z"][c["items"] + (self.fresh is not None) + s]

    def _stage_done(self, s):
        self.locs[s] = self.located.loc

    def _accepted(self, t, dt, t_new):
        c = self.route.chunks[-1]
        locs = ([self.fresh] if self.fresh is not None else []) + self.locs
        c["locs"] += locs
        c["items"] += len(locs)
        c["step_item"].append(c["items"])
        self.route.steps.append((t, dt))
        self.route.ends.append(t_new)
        self.fresh = None


class Dopri5MlpBackprop:
    """``cdeint(..., adjoint=False)`` of the host-driven dopri5 solve of the MLP field with gradients for any of z0, W1,
    b1, W2, b2: the exact gradient of the discrete solve, without autograd, where the CUDA-core kernels serve the shape
    (the C dispatch's policy, ``tcde_dopri5_mlp_backward``).

    The forward is ``adaptive.Dopri5`` under ``no_grad`` with the field the same call without gradients uses, so its
    outputs and accepted / rejected steps are that call's, bit for bit; its hooks record, per accepted step, the inputs and
    locations of its evaluations 2..7 and of its own start slope where it has one (step 0, and after a jump of
    ``jump_t``), in chunks of ``slots`` steps.  The backward is, per chunk and last chunk first, ONE launch of
    ``tcde_dopri5_mlp_backward`` (the transposed Dormand-Prince recurrence, J^T at the recorded inputs) and, with a
    parameter gradient, ONE call of ``tcde_mlp_field_param_grads`` over (input, kappa) of the chunk's evaluations.
    ``replay(steps)``: the differentiable torch-operator solve of the same problem taking the recorded steps, which a
    backward with ``create_graph`` differentiates instead.  Memory: the first chunk is checked before the solve starts and
    each further one before it is taken; a chunk that does not fit discards the partial solve (``NoRoom``)."""

    slots = 64                # accepted steps per record chunk

    def __init__(self, kernels, field, times, rtol, atol, sign, options, replay):
        self.kernels, self.field, self.times, self.rtol, self.atol = kernels, field, list(times), rtol, atol
        self.sign, self.options, self.replay = float(sign), options, replay
        self.want_params = any(p is not None and p.requires_grad for p in kernels.field_params)
        # a step takes 6 items, 7 with a start slope of its own: only step 0 has one unless jump_t is given
        self.cap = 7 * self.slots if options.get("jump_t") else 6 * self.slots + 1

    def differentiable(self, z0):
        return self.replay(self.steps)(z0)

    def fits(self, n_paths):
        """Whether one more record chunk fits (``backprop.fits``)."""
        k = self.kernels
        chunk = self.cap * n_paths * k.hidden * torch.empty(0, dtype=k.dtype).element_size()
        return backprop.fits(k.device, chunk,
                             k.param_grad_scratch_bytes(n_paths, self.cap) if self.want_params else None)

    def room(self):
        """The chunk the current step records into: a fresh one when the last is full (``NoRoom`` if it does not fit)."""
        if len(self.chunks[-1]["step_item"]) > self.slots:
            if not self.fits(self.n_paths):
                raise backprop.NoRoom()
            self._new_chunk()
        return self.chunks[-1]

    def _new_chunk(self):
        k = self.kernels
        self.chunks.append({"z": torch.empty((self.cap,) + self.shape, dtype=k.dtype, device=k.device),
                            "items": 0, "step_item": [0], "locs": []})

    def forward(self, z0):
        """(the outputs ``(..., len(times), H)``, the record: per chunk its evaluations' inputs, interval indices and
        fractions and its steps' first items).  Raises ``NoRoom`` (nothing kept) when the record does not fit."""
        k = self.kernels
        with torch.cuda.device(k.device), torch.no_grad():
            y0 = z0.detach()
            self.shape, self.n_paths = tuple(y0.shape), k.n_paths
            if not self.fits(self.n_paths):
                raise backprop.NoRoom()
            self.chunks, self.steps, self.ends = [], [], []
            self._new_chunk()
            located = _Located(self.field, k.where)
            opts = self.options
            solver = _RecordingDopri5(self, located, _reverse(located) if self.sign < 0 else located, y0, self.rtol,
                                      self.atol, first_step=opts.get("first_step"),
                                      max_num_steps=opts.get("max_num_steps", 2 ** 31 - 1), jump_t=opts.get("jump_t"))
            out = solver.integrate(self.times)
            record = []
            for c in self.chunks:
                n_items = c["items"]
                record += [c["z"][:n_items],
                           torch.tensor([i for i, _f in c["locs"]] or [0], dtype=torch.int32).to(k.device),
                           torch.tensor([f for _i, f in c["locs"]] or [0.0], dtype=k.dtype).to(k.device),
                           torch.tensor(c["step_item"], dtype=torch.int32).to(k.device)]
            self.counts = [len(c["step_item"]) - 1 for c in self.chunks]
            self.chunks = None                 # the record lives as long as its holder (the autograd shell saves it)
        self.stats = {"n_accepted": solver.n_accepted, "n_rejected": solver.n_rejected, "device_controlled": False,
                      "steps": list(self.steps)}
        return out.movedim(0, -2), record

    def backward(self, g, z0, saved, want):
        """(dL/dz0, [dL/dW1, dL/db1, dL/dW2, dL/db2] with None where ``want`` is False) for output gradients ``g``
        ``(..., len(times), H)`` from ``forward``'s record ``saved``."""
        k = self.kernels
        hidden, dev, n_out, code = k.hidden, k.device, len(self.times), _lib.dtype_code(k.dtype)
        with torch.cuda.device(dev):
            gf = backprop.cotangent(g, n_out, hidden)
            n_paths = gf.size(0)
            stream = _lib.stream_of(gf)
            grads = [torch.zeros_like(p) if w else None for p, w in zip((k.w1, k.b1, k.w2, k.b2), want)]
            params = any(want)
            tables = adaptive.dopri5_backward_tables(self.steps, self.times, k.dtype, self.ends)
            coef, inj_range = tables["coef"].to(dev), tables["inj_range"].to(dev)
            inj_out, inj_w = tables["inj_out"].to(dev), tables["inj_w"].to(dev)
            carry = torch.zeros(2, n_paths, hidden, dtype=k.dtype, device=dev)
            kappa = torch.empty(self.cap, n_paths, hidden, dtype=k.dtype, device=dev) if params else None
            scratch = k.param_grad_scratch(n_paths, self.cap) if params else None
            starts = [sum(self.counts[:i]) for i in range(len(self.counts))]
            for i in range(len(self.counts) - 1, -1, -1):
                (z, index, frac, step_item), n, lo = saved[4 * i:4 * i + 4], self.counts[i], starts[i]
                if n <= 0:
                    continue
                _lib.call("tcde_dopri5_mlp_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1),
                          _lib.ptr(k.b1), _lib.ptr(k.w2), _lib.ptr(k.b2), _lib.ptr(z), _lib.ptr(gf), _lib.ptr(carry),
                          _lib.ptr(kappa), _lib.ptr(coef[lo:lo + n]), _lib.ptr(step_item), _lib.ptr(index),
                          _lib.ptr(frac), _lib.ptr(inj_range[lo:lo + n + 1]), _lib.ptr(inj_out), _lib.ptr(inj_w), n_out,
                          n, n_paths, k.channels, hidden, k.width, self.sign, code, stream)
                if params:
                    k.param_grads(z, kappa, index, frac, z.size(0), grads, scratch, self.sign)
            # step 0's start slope f(t0, z0) was closed by the first chunk's launch: carry[1] is zero
            gz = carry[0] + gf[:, 0]
        return gz.view(g.shape[:-2] + (hidden,)), grads


def dopri5_mlp_backprop(X, params, z0, field_of, times, rtol, atol, sign, options, replay):
    """``cdeint(..., adjoint=False)``'s outputs ``(..., len(times), H)`` and statistics on the route of
    ``Dopri5MlpBackprop``, or None when the route does not serve the problem (the caller runs the torch-operator dopri5).
    ``field_of(kernels)``: the dopri5 field of the same call without gradients (before ``_reverse``); ``times``: increasing
    floats (negated when ``sign`` < 0); ``options``: the host driver's (``jump_t`` oriented like ``times``); ``replay(steps)``
    returns the torch-operator solve ``z0 -> outputs`` on ``steps``."""
    if len(times) < 2 or not set(options) <= {"first_step", "jump_t", "max_num_steps"}:
        return None
    k = _backprop_kernels(X, params, z0)
    if k is None or k.n_paths == 0:
        return None
    route = Dopri5MlpBackprop(k, None, times, rtol, atol, sign, options, replay)
    if route.want_params and k.param_grad_scratch_bytes(k.n_paths, route.cap) < 0:
        return None                            # the parameter-gradient staging does not fit this width
    # the dispatch's verdict on the problem, from a call with no paths (it validates and launches nothing; one small
    # buffer stands in for the per-path and table pointers)
    s = torch.zeros(4, dtype=torch.float64, device=k.device)
    p = _lib.ptr(s)
    try:
        with torch.cuda.device(k.device):
            _lib.call("tcde_dopri5_mlp_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1), _lib.ptr(k.b1),
                      _lib.ptr(k.w2), _lib.ptr(k.b2), p, p, p, None, p, p, p, p, p, p, p, len(times), 0, 0, k.channels,
                      k.hidden, k.width, float(sign), _lib.dtype_code(k.dtype), _lib.stream_of(s))
    except NotImplementedError:
        return None
    with torch.no_grad():
        route.field = field_of(k)
    ys = backprop.run(route, z0, params)
    return None if ys is None else (ys, route.stats)
