"""The README's linear vector field and ``LinearFieldKernels``, the owner of every kernel route of ``cdeint`` for one
(control, linear field, z0) problem: fused fixed-step solve, kernel field, device-controlled dopri5, adjoint stage."""
import functools
import math
import warnings
import weakref

import torch

from . import _lib, adaptive, backprop
from .controls import _control_signature, _schedule_knots
from .schedule import ScheduleCache, backward_views, host_locator, locate

_schedules = ScheduleCache()


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
        known = _probe(func, lambda z: torch.nn.functional.linear(z, lin.weight, lin.bias), z0, channels, times,
                       "a single nn.Linear", "torchcde_b200.LinearVectorField")
        try:
            _recognised[func] = known
        except TypeError:
            pass
    return (lin.weight, lin.bias) if known else None


def _probe(func, field, z0, channels, times, looks_like, remedy):
    """Bit-exact comparison of ``func`` with ``field(z).view(..., H, C)`` on random (non-degenerate) states of z0's own
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
                warnings.warn("torchcde_b200.cdeint: `func` looks like {} but could not be probed. Falling back to the "
                              "generic stage loop{}.".format(looks_like, "; use {} to get the fused kernel".format(remedy)
                                                             if remedy else ""))
                return False
            want = field(zp).view(*zp.shape[:-1], hidden, channels)
            if not (isinstance(got, torch.Tensor) and got.shape == want.shape and got.dtype == want.dtype
                    and torch.equal(got, want)):
                return False
    return True


def _check_linear_problem(control, weight, bias, z0):
    """The control's coefficients, the weight and the bias must share z0's dtype and CUDA device -- the kernels receive
    raw pointers, so a mismatch would be reinterpreted memory, not an exception (the reference raises a dtype / device
    RuntimeError from its torch ops in the same situations)."""
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


def _reverse(field):
    return lambda s, y, nudge=0: -1.0 * field(-s, y)


class LinearFieldKernels:
    """The kernel routes of one problem: a built-in control ``X``, the linear field ``(weight, bias)`` (``bias`` may be
    None) and the state ``z0``.  Construction validates the problem; the adjoint's regrouped weights, the scalar locator
    and the parameter-gradient scratch are made on first use."""

    def __init__(self, X, weight, bias, z0):
        self.kind, _, self.channels, self.n_rows = _control_signature(X)
        self.hidden = z0.size(-1)
        self.n_paths = math.prod(z0.shape[:-1])
        self.dtype, self.device = z0.dtype, z0.device
        control = X._rows() if self.kind == _lib.CONTROL_CUBIC else X._derivs
        _check_linear_problem(control, weight, bias, z0)
        self.control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
        self.weight, self.bias = weight, bias          # the parameters themselves, to recognise them in adjoint_params
        self.w = weight.detach().contiguous()
        self.b = (bias.detach() if bias is not None else
                  torch.zeros(self.hidden * self.channels, dtype=z0.dtype, device=z0.device)).contiguous()
        self.knots = _schedule_knots(X)
        self.time_knots = X._t
        self._scratch = None

    @functools.cached_property
    def where(self):
        """``(t, nudge) -> (interval index, fraction)`` of a stage time: ``schedule.host_locator``."""
        return host_locator(self.knots, self.n_rows, self.dtype)

    def solve(self, y0, t, method, step_size):
        """The fixed-step solve as ONE launch of ``tcde_cdeint_fixed_linear``: ``(..., len(t), H)``."""
        with torch.cuda.device(self.device):
            zf = y0.detach().reshape(-1, self.hidden).contiguous()
            sched, (_floats, _ints, v) = _schedules.get(t, self.knots, self.n_rows, method, step_size, self.dtype,
                                                        self.device)
            out = torch.empty(zf.size(0), sched.n_out, self.hidden, dtype=self.dtype, device=self.device)
            if zf.size(0) > 0:            # an empty batch: nothing to launch (its null data pointers would be refused)
                self._fixed(sched, v, self.w, self.b, zf, out)
        return out.view(*y0.shape[:-1], sched.n_out, self.hidden)

    def _fixed(self, sched, v, w, b, z, out, dump=None):
        """One fused solve on ``sched`` (device views ``v``); with ``dump`` it also keeps every stage's input there."""
        name, dumps = ("tcde_cdeint_fixed_linear", ()) if dump is None else ("tcde_cdeint_fixed_linear_stages",
                                                                             (_lib.ptr(dump),))
        _lib.call(name, _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(w), _lib.ptr(b), _lib.ptr(z),
                  _lib.ptr(out), *dumps, z.size(0), self.channels, self.hidden, _lib.METHODS[sched.method],
                  sched.n_steps, _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]),
                  sched.n_out, _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]),
                  float(sched.sign), _lib.dtype_code(self.dtype), _lib.stream_of(z))

    def field(self, weight=None, bias=None):
        """f(t, y) = (Linear(y).view(H, C)) @ dX/dt(t) as ONE launch of ``tcde_vector_field_linear``.  ``weight``,
        ``bias``: contiguous tensors of the problem's dtype and device in place of its own (the adjoint's weights)."""
        w = self.w if weight is None else weight
        b = self.b if bias is None else bias
        hidden = self.hidden
        code = _lib.dtype_code(self.dtype)

        def field(t, y, nudge=0):
            index, frac = self.where(t, nudge)
            yf = y.reshape(-1, hidden).contiguous()
            out = torch.empty_like(yf)
            with torch.cuda.device(y.device):
                _lib.call("tcde_vector_field_linear", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(w),
                          _lib.ptr(b), _lib.ptr(yf), _lib.ptr(out), yf.size(0), self.channels, hidden, index,
                          float(frac), code, _lib.stream_of(yf))
            return out.view_as(y)

        return field

    @functools.cached_property
    def transposed_weights(self):
        """W with rows regrouped as (k, c) and columns h, and a zero bias: the field product with them is J^T w."""
        h, c = self.hidden, self.channels
        return self.w.view(h, c, h).permute(2, 1, 0).contiguous().view(h * c, h), torch.zeros_like(self.b)

    @functools.cached_property
    def adjoint_weights(self):
        """-W with rows regrouped as (k, c) and columns h, and a zero bias: the weights of the adjoint state's own CDE."""
        w2, zeros = self.transposed_weights
        return w2.neg(), zeros

    def param_grad_scratch_bytes(self, n_paths, n_total):
        return _lib.load().tcde_linear_field_param_grads_scratch_bytes(n_paths, n_total, self.channels, self.hidden)

    def param_grads(self, z_stages, a_stages, index, frac, weights, n_total, gw, gb):
        """``gw``, ``gb`` += the quadrature sum over ``n_total`` stages of ``weights * a^T df/dW, a^T df/db`` (ONE launch
        of ``tcde_linear_field_param_grads``).  Returns False, launching nothing, when the kernel is not built for it."""
        n_paths = z_stages.size(1)
        nbytes = self.param_grad_scratch_bytes(n_paths, n_total)
        if nbytes < 0:
            return False
        if self._scratch is None or 4 * self._scratch.numel() < nbytes:
            self._scratch = torch.empty(max(nbytes // 4, 4), dtype=torch.float32, device=self.device)
        _lib.call("tcde_linear_field_param_grads", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(z_stages),
                  _lib.ptr(a_stages), _lib.ptr(index), _lib.ptr(frac), _lib.ptr(weights), n_total, _lib.ptr(gw),
                  _lib.ptr(gb), _lib.ptr(self._scratch), n_paths, self.channels, self.hidden, 1.0,
                  _lib.dtype_code(self.dtype), _lib.stream_of(z_stages))
        return True

    # ---- torchsde's reversible Heun (reversible._Problem): the forward, the segment backward, the parameter gradients ----
    @property
    def field_params(self):
        return self.weight, self.bias

    @property
    def field_tensors(self):
        return self.w, self.b

    @property
    def reversible_backward_served(self):
        """The segment kernel is built for fp32 at hidden 32, channels 8."""
        return self.dtype == torch.float32 and self.hidden == 32 and self.channels == 8

    def reversible_forward(self, sched, v, z0, out, ckpt, stride):
        """ONE launch of ``tcde_cdeint_reversible_heun_linear`` on ``build_sde_schedule``'s tables (device views ``v``)."""
        _lib.call("tcde_cdeint_reversible_heun_linear", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w),
                  _lib.ptr(self.b), _lib.ptr(z0), _lib.ptr(out), _lib.ptr(ckpt), stride, z0.size(0), self.channels,
                  self.hidden, sched.n_steps, _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]),
                  sched.n_out, _lib.ptr(v["out_step"]), _lib.ptr(v["out_slope"]), _lib.dtype_code(self.dtype),
                  _lib.stream_of(z0))

    def reversible_segment(self, bw, lo, hi, ck_lo, ck_hi):
        """ONE launch of ``tcde_reversible_heun_linear_backward_segment`` over steps [lo, hi]; the segment that ends at
        step N first closes it (ybar_N from the outputs, zbar_N = J_F(z_N)^T fbar_N and its parameter gradients by one
        launch of ``tcde_vector_field_linear_vjp``).  Returns the number of dumped steps."""
        p, v = bw.problem, bw.views
        n_steps, n_paths = p.sched.n_steps, bw.g.size(0)
        gw, gb = bw.grads
        if hi == n_steps:
            first, end, weights = p._injection(n_steps)
            bw.carry[0].zero_()
            for j, w in zip(range(first, end), weights):
                bw.carry[0].add_(bw.g[:, j], alpha=w)
            fbar = bw.carry[0] * (0.5 * p.dts[n_steps - 1])
            z_n = bw.last[1].contiguous()
            f_tmp = torch.empty_like(z_n)
            scratch_bytes = _lib.load().tcde_vector_field_linear_vjp_scratch_bytes(n_paths, self.channels, self.hidden)
            scratch = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=self.device)
            _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w),
                      _lib.ptr(self.b), _lib.ptr(z_n), _lib.ptr(fbar), _lib.ptr(f_tmp), _lib.ptr(bw.carry[1]),
                      _lib.ptr(gw), _lib.ptr(gb), _lib.ptr(scratch), n_paths, self.channels, self.hidden,
                      p.index[n_steps], float(p.frac_state[n_steps]), 1.0, 1.0, 1.0, _lib.F32, bw.stream)
        w_t, zeros = self.transposed_weights
        _lib.call("tcde_reversible_heun_linear_backward_segment", _lib.ptr(self.control), self.kind, self.n_rows,
                  _lib.ptr(self.w), _lib.ptr(self.b), _lib.ptr(w_t), _lib.ptr(zeros), _lib.ptr(ck_lo), _lib.ptr(ck_hi),
                  _lib.ptr(bw.carry), _lib.ptr(bw.g), p.n_out, _lib.ptr(v["out_step"]), _lib.ptr(v["out_slope"]),
                  _lib.ptr(bw.inj), _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]), lo, hi,
                  n_paths, self.channels, self.hidden, _lib.ptr(bw.dump_z), _lib.ptr(bw.dump_a), _lib.F32, bw.stream)
        return hi - lo

    def reversible_param_grads(self, bw, lo, n):
        """dL/dW, dL/db += the segment's dump of ``n`` steps from ``lo`` (``param_grads`` with weights 1)."""
        gw, gb = bw.grads
        if getattr(bw, "ones", None) is None:
            bw.ones = torch.ones(bw.dump_z.size(0), dtype=torch.float32, device=self.device)
        v = bw.views
        if not self.param_grads(bw.dump_z, bw.dump_a, v["stage_index"][lo:lo + n], v["stage_frac"][lo:lo + n], bw.ones,
                                n, gw, gb):
            raise RuntimeError("reversible backward: the parameter-gradient kernel is not built for this problem")

    def dopri5(self, y0, times, rtol, atol, sign, first_step=None):
        """The same algorithm as ``adaptive.Dopri5.integrate`` with accept / reject, the step-size rule and the dense
        output on the device (``tcde_dopri5_linear_attempts``: one launch per attempted step, no host read per attempt).
        The kernel field only gives the slope at the start and Hairer's initial step.  ``times``: increasing floats
        (already negated when ``sign`` < 0).  Returns ``(out (len(times), *y0.shape), stats)``."""
        field = self.field() if sign > 0 else _reverse(self.field())
        yf = y0.detach().reshape(-1, self.hidden).contiguous()
        knots = self.time_knots.detach().to(device=self.device, dtype=torch.float32).contiguous()
        stream = _lib.stream_of(yf)

        def launch(state, partials, ctl, out, out_times, first_seq):
            _lib.call("tcde_dopri5_linear_attempts", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(knots),
                      _lib.ptr(self.w), _lib.ptr(self.b), _lib.ptr(state), _lib.ptr(partials), _lib.ptr(ctl),
                      _lib.ptr(out), _lib.ptr(out_times), len(times), yf.size(0), self.channels, self.hidden,
                      float(sign), first_seq, adaptive._DEVICE_CHUNK, _lib.F32, stream)

        out, _last, stats = adaptive.device_controller(launch, field, yf, times, rtol, atol, first_step,
                                                       "dopri5: step size underflow / non-finite error estimate at t = {}")
        return out.movedim(1, 0).reshape(len(times), *y0.shape), dict(stats, device_controlled=True)

    def adjoint_stage(self, params):
        """The adjoint stage of this problem for ``params``, or None when the kernel is not built for it (then autograd
        serves the backward solve): fp32 only, and every parameter must be the weight or the bias."""
        roles = []
        for p in params:
            if p is self.weight:
                roles.append("w")
            elif self.bias is not None and p is self.bias:
                roles.append("b")
            else:
                return None                       # a parameter that is not the linear map: autograd knows how
        if self.dtype != torch.float32:
            return None
        scratch_bytes = _lib.load().tcde_vector_field_linear_vjp_scratch_bytes(self.n_paths, self.channels, self.hidden)
        if scratch_bytes < 0:
            return None
        return AdjointStage(self, roles, torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=self.device))


def _backprop_kernels(X, field_params, z0):
    """The kernels of a problem the linear backprop routes are built for (fp32, hidden 32, channels 8, the control's
    floating buffers and the parameters fp32 on z0's device), else None: nothing is built, so a mismatched call keeps
    the torch operators' own dtype and device errors."""
    if (z0.dtype != torch.float32 or z0.size(-1) != 32 or _control_signature(X)[2] != 8
            or any(b.dtype != torch.float32 or b.device != z0.device for b in X.buffers() if b.is_floating_point())
            or any(p is not None and (p.dtype != torch.float32 or p.device != z0.device) for p in field_params)):
        return None
    return LinearFieldKernels(X, field_params[0], field_params[1], z0)


class FixedBackprop:
    """``cdeint(..., adjoint=False)`` of a fixed-step solve of this linear field with gradients for z0, the weight and /
    or the bias: the exact gradient of the discrete solve in three launches.  The forward is the stage-dump solve
    (``tcde_cdeint_fixed_linear_stages``: the outputs are those of the same call without gradients, bit for bit); the
    backward is ONE launch of ``tcde_cdeint_fixed_linear_backward`` (the transposed Runge-Kutta recurrence over every
    step, the cotangent kappa of every stage dumped in the forward's slot) and ONE launch of
    ``tcde_linear_field_param_grads`` over the two dumps (neither without a parameter gradient).
    ``differentiable(z0)``: the torch-operator solve of the same problem, which a backward with ``create_graph``
    differentiates instead."""

    def __init__(self, kernels, t, method, step_size, loop):
        self.kernels, self.method, self.differentiable = kernels, method, loop
        self.sched, (_floats, _ints, self.views) = _schedules.get(t, kernels.knots, kernels.n_rows, method, step_size,
                                                                  kernels.dtype, kernels.device)
        self.want_params = any(p is not None and p.requires_grad for p in kernels.field_params)

    def forward(self, z0):
        """(the outputs ``(..., n_out, H)``, [the input of every stage ``[n_steps * n_stages][paths][H]``]).  Raises
        ``NoRoom`` when the stage dump, and with a parameter gradient its kappa copy and the scratch, do not fit."""
        k, sched = self.kernels, self.sched
        n_total = sched.n_steps * sched.n_stages
        scratch_bytes = k.param_grad_scratch_bytes(k.n_paths, n_total) if self.want_params else None
        if not backprop.fits(k.device, n_total * k.n_paths * k.hidden * 4, scratch_bytes):
            raise backprop.NoRoom()
        with torch.cuda.device(k.device):
            zf = z0.detach().reshape(-1, k.hidden).contiguous()
            out = torch.empty(*z0.shape[:-1], sched.n_out, k.hidden, dtype=k.dtype, device=k.device)
            dump = torch.empty(n_total, zf.size(0), k.hidden, dtype=k.dtype, device=k.device)
            if zf.size(0) > 0:
                k._fixed(sched, self.views, k.w, k.b, zf, out.view(-1, sched.n_out, k.hidden), dump)
        return out, [dump]

    def backward(self, g, z0, saved, want):
        """(dL/dz0, [dL/dW, dL/db], None where ``want`` is False) for output gradients ``g`` ``(..., n_out, H)``."""
        k, sched = self.kernels, self.sched
        (dump,), (want_w, want_b) = saved, want
        hidden, dev = k.hidden, k.device
        n_total = sched.n_steps * sched.n_stages
        with torch.cuda.device(dev):
            gf = backprop.cotangent(g, sched.n_out, hidden)
            n_paths = gf.size(0)
            gz = torch.empty(n_paths, hidden, dtype=k.dtype, device=dev)
            kappa = torch.empty_like(dump) if want_w or want_b else None
            if n_paths > 0:
                tables = backward_views(sched, dev)
                w_t, zeros = k.transposed_weights
                _lib.call("tcde_cdeint_fixed_linear_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(w_t),
                          _lib.ptr(zeros), _lib.ptr(gf), _lib.ptr(gz), _lib.ptr(kappa), n_paths, k.channels, hidden,
                          _lib.METHODS[sched.method], sched.n_steps, _lib.ptr(tables["step_dt"]),
                          _lib.ptr(tables["stage_index"]), _lib.ptr(tables["stage_frac"]), sched.n_out,
                          _lib.ptr(tables["inj_range"]), _lib.ptr(tables["inj_out"]), _lib.ptr(tables["inj_weight"]),
                          float(sched.sign), _lib.F32, _lib.stream_of(gf))
            gw = torch.zeros_like(k.w) if want_w else None
            gb = torch.zeros_like(k.b) if want_b else None
            if (gw is not None or gb is not None) and n_paths > 0:
                weights = torch.full((n_total,), float(sched.sign), dtype=k.dtype, device=dev)
                if not k.param_grads(dump, kappa, self.views["stage_index"], self.views["stage_frac"], weights, n_total,
                                     gw, gb):
                    raise RuntimeError("cdeint backward: the parameter-gradient kernel is not built for this problem")
        return gz.view(g.shape[:-2] + (hidden,)), [gw, gb]


def fixed_backprop(X, field_params, z0, t, method, step_size, loop):
    """``cdeint(..., adjoint=False)``'s outputs ``(..., n_out, H)`` on the three-launch route of ``FixedBackprop``, or
    None when the route does not serve the problem (the caller runs the torch-operator solve ``loop``).  The stage-dump
    solve refuses the CUDA-core kernel's shapes and misaligned rows before it launches anything."""
    k = _backprop_kernels(X, field_params, z0)
    return None if k is None else backprop.run(FixedBackprop(k, t, method, step_size, loop), z0, k.field_params)


class Dopri5Backprop:
    """``cdeint(..., adjoint=False)`` of the device-controlled dopri5 solve of this linear field with gradients for z0, the
    weight and / or the bias: the exact gradient of the discrete solve, without autograd.

    The forward is the recording mode of the device controller (``tcde_dopri5_linear_record_attempts``: the outputs and
    the accepted / rejected steps of the same call without gradients, bit for bit); every accepted step leaves its (t, dt),
    its stage locations and, with a parameter gradient, the inputs of its six evaluations in a slot.  The slots come in
    chunks of ``slots`` steps; a full chunk pauses the device, which resumes on a fresh chunk.  The backward is, per chunk
    and last chunk first, ONE launch of ``tcde_dopri5_linear_backward`` (the transposed Dormand-Prince recurrence) and,
    with a parameter gradient, ONE launch of ``tcde_linear_field_param_grads`` over (stage input, kappa); then one launch of
    ``tcde_vector_field_linear_vjp`` closes the start slope f(t0, z0).  ``replay(steps)``: the differentiable
    torch-operator solve of the same problem taking the recorded steps, which a backward with ``create_graph``
    differentiates instead (the forward cannot know which backward will come, so it records either way).  Memory: the
    first chunk is checked before the solve starts, each further chunk when the device pauses for it; a chunk that does
    not fit discards the partial solve and the caller runs the torch-operator solve from the start."""

    slots = 64                # accepted steps per record chunk

    def __init__(self, kernels, times, rtol, atol, sign, first_step, replay):
        self.kernels, self.times, self.rtol, self.atol = kernels, list(times), rtol, atol
        self.sign, self.first_step, self.replay = float(sign), first_step, replay
        self.want_params = any(p is not None and p.requires_grad for p in kernels.field_params)

    def differentiable(self, z0):
        return self.replay(self.steps)(z0)

    def fits(self, n_paths):
        """Whether one more record chunk fits (``backprop.fits``; without a parameter gradient nothing is recorded)."""
        k = self.kernels
        if not self.want_params:
            return backprop.fits(k.device, 0)
        return backprop.fits(k.device, self.slots * 6 * n_paths * k.hidden * 4,
                             k.param_grad_scratch_bytes(n_paths, 6 * self.slots))

    def _new_chunk(self, n_paths):
        k, dev = self.kernels, self.kernels.device
        return {"z": torch.empty(self.slots * 6, n_paths, k.hidden, dtype=torch.float32, device=dev)
                if self.want_params else None,
                "step": torch.zeros(self.slots, 2, dtype=torch.float64, device=dev),
                "index": torch.zeros(self.slots, 6, dtype=torch.int32, device=dev),
                "frac": torch.zeros(self.slots, 6, dtype=torch.float32, device=dev)}

    def forward(self, z0):
        """(the outputs ``(..., len(times), H)``, the record: per chunk its stage inputs (None without a parameter
        gradient), stage intervals and fractions).  The route keeps only the accepted steps on the host, so the record
        lives exactly as long as its holder.  Raises ``NoRoom`` (nothing kept) when the record does not fit."""
        k = self.kernels
        with torch.cuda.device(k.device):
            yf = z0.detach().reshape(-1, k.hidden).contiguous()
            n_paths = yf.size(0)
            if not self.fits(n_paths):
                raise backprop.NoRoom()
            field = k.field() if self.sign > 0 else _reverse(k.field())
            knots = k.time_knots.detach().to(device=k.device, dtype=torch.float32).contiguous()
            stream = _lib.stream_of(yf)
            chunks = [self._new_chunk(n_paths)]

            def launch(state, partials, ctl, out, out_times, first_seq):
                c = chunks[-1]
                _lib.call("tcde_dopri5_linear_record_attempts", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(knots),
                          _lib.ptr(k.w), _lib.ptr(k.b), _lib.ptr(state), _lib.ptr(partials), _lib.ptr(ctl), _lib.ptr(out),
                          _lib.ptr(out_times), len(self.times), n_paths, k.channels, k.hidden, self.sign, _lib.ptr(c["z"]),
                          _lib.ptr(c["step"]), _lib.ptr(c["index"]), _lib.ptr(c["frac"]), self.slots, first_seq,
                          adaptive._DEVICE_CHUNK, _lib.F32, stream)

            def grow(last):                          # the chunk is full: the device resumes on a fresh one
                if not self.fits(n_paths):
                    raise backprop.NoRoom()
                chunks.append(self._new_chunk(n_paths))

            out, _last, stats = adaptive.device_controller(
                launch, field, yf, self.times, self.rtol, self.atol, self.first_step,
                "dopri5: step size underflow / non-finite error estimate at t = {}", on_overflow=grow)
            n_acc = stats["n_accepted"]
            self.counts = [min(self.slots, n_acc - i * self.slots) for i in range(len(chunks))]
            steps = torch.cat([c["step"][:n] for c, n in zip(chunks, self.counts)]).cpu()
            self.steps = [(float(t), float(dt)) for t, dt in steps.tolist()]
        self.stats = dict(stats, device_controlled=True, steps=list(self.steps))
        record = [x for c in chunks for x in (c["z"], c["index"], c["frac"])]
        return out.view(*z0.shape[:-1], len(self.times), k.hidden), record

    def backward(self, g, z0, saved, want):
        """(dL/dz0, [dL/dW, dL/db], None where ``want`` is False) for output gradients ``g`` ``(..., len(times), H)`` from
        the solve of ``z0`` and its record ``saved`` (``forward``'s)."""
        k = self.kernels
        hidden, dev, n_out = k.hidden, k.device, len(self.times)
        want_w, want_b = want
        with torch.cuda.device(dev):
            gf = backprop.cotangent(g, n_out, hidden)
            n_paths = gf.size(0)
            stream = _lib.stream_of(gf)
            gw = torch.zeros_like(k.w) if want_w else None
            gb = torch.zeros_like(k.b) if want_b else None
            params = gw is not None or gb is not None
            tables = adaptive.dopri5_backward_tables(self.steps, self.times)
            coef, inj_range = tables["coef"].to(dev), tables["inj_range"].to(dev)
            inj_out, inj_w = tables["inj_out"].to(dev), tables["inj_w"].to(dev)
            w_t, zeros = k.transposed_weights
            carry = torch.zeros(2, n_paths, hidden, dtype=torch.float32, device=dev)
            kappa = torch.empty(self.slots * 6, n_paths, hidden, dtype=torch.float32, device=dev) if params else None
            weights = torch.full((self.slots * 6,), self.sign, dtype=torch.float32, device=dev) if params else None
            for i in range(len(self.counts) - 1, -1, -1):
                (stage_z, stage_index, stage_frac), n = saved[3 * i:3 * i + 3], self.counts[i]
                lo = i * self.slots
                if n <= 0:
                    continue
                _lib.call("tcde_dopri5_linear_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(w_t),
                          _lib.ptr(zeros), _lib.ptr(gf), _lib.ptr(carry), _lib.ptr(kappa), _lib.ptr(coef[lo:lo + n]),
                          _lib.ptr(stage_index), _lib.ptr(stage_frac), _lib.ptr(inj_range[lo:lo + n + 1]), _lib.ptr(inj_out),
                          _lib.ptr(inj_w), n_out, n, n_paths, k.channels, hidden, self.sign, _lib.F32, stream)
                if params and not k.param_grads(stage_z, kappa, stage_index.view(-1), stage_frac.view(-1), weights, 6 * n,
                                                gw, gb):
                    raise RuntimeError("cdeint backward: the parameter-gradient kernel is not built for this problem")
            # the start slope f(t0, z0): its cotangent is carry[1]
            index, frac = k.where(self.sign * self.times[0])
            z0 = z0.detach().reshape(-1, hidden).contiguous()
            f_tmp, vjp = torch.empty_like(z0), torch.empty_like(z0)
            scratch_bytes = _lib.load().tcde_vector_field_linear_vjp_scratch_bytes(n_paths, k.channels, hidden)
            scratch = torch.empty(max(scratch_bytes // 4, 4), dtype=torch.float32, device=dev)
            _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w), _lib.ptr(k.b),
                      _lib.ptr(z0), _lib.ptr(carry[1]), _lib.ptr(f_tmp), _lib.ptr(vjp), _lib.ptr(gw), _lib.ptr(gb),
                      _lib.ptr(scratch), n_paths, k.channels, hidden, index, float(frac), 1.0, self.sign, self.sign,
                      _lib.F32, stream)
            gz = carry[0] + vjp + gf[:, 0]
        return gz.view(g.shape[:-2] + (hidden,)), [gw, gb]


def dopri5_backprop(X, field_params, z0, times, rtol, atol, sign, options, replay):
    """``cdeint(..., adjoint=False)``'s outputs ``(..., len(times), H)`` and statistics on the route of ``Dopri5Backprop``,
    or None when the route does not serve the problem (the caller runs the torch-operator solve).  ``times``: increasing
    floats (negated when ``sign`` < 0); ``options``: the host driver's (the device controller takes ``first_step`` and no
    ``jump_t``); ``replay(steps)`` returns the torch-operator solve ``z0 -> outputs`` on ``steps``.  The recording solve
    refuses control rows off a 16-byte boundary before it launches anything."""
    if options.get("jump_t") or not set(options) <= {"first_step", "jump_t"} or len(times) < 2:
        return None
    k = _backprop_kernels(X, field_params, z0)
    if k is None or k.n_paths == 0:
        return None
    route = Dopri5Backprop(k, times, rtol, atol, sign, options.get("first_step"), replay)
    ys = backprop.run(route, z0, k.field_params)
    return None if ys is None else (ys, route.stats)


class AdjointStage:
    """The adjoint stage of the linear field: ``stage(t, y, a, scale) -> (f, scale * a^T df/dy, [scale * a^T df/dp for
    p in params])`` as ONE launch of ``tcde_vector_field_linear_vjp``, plus the whole-segment backward routes that
    ``adaptive._Adjoint`` tries first; fp32 only.  ``roles``: "w" or "b" for each parameter."""

    adaptive_spec = None      # (rtol, atol) when the dopri5 backward may run with the controller on the device
    slots_hint = 256          # trajectory slots asked for by that backward
    adaptive_stats = None     # statistics of the last adaptive_segment

    def __init__(self, kernels, roles, scratch):
        self.kernels, self.roles, self.scratch = kernels, roles, scratch

    def new_grads(self):
        k = self.kernels
        return [torch.zeros_like(k.w) if r == "w" else torch.zeros_like(k.b) for r in self.roles]

    def _by_role(self, grads):
        """(dL/dW, dL/db) out of one tensor (or None) per parameter in the order of ``params``."""
        gw = next((g for g, r in zip(grads, self.roles) if r == "w"), None)
        gb = next((g for g, r in zip(grads, self.roles) if r == "b"), None)
        return gw, gb

    def launch(self, index, frac, y, a, f_out, vjp_out, *grads, f_scale, vjp_scale, grad_scale):
        """``grads``: one tensor (or None) per parameter, in the order of ``params``, += grad_scale * a^T df/dp."""
        k = self.kernels
        gw, gb = self._by_role(grads)
        with torch.cuda.device(y.device):
            _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w),
                      _lib.ptr(k.b), _lib.ptr(y), _lib.ptr(a), _lib.ptr(f_out), _lib.ptr(vjp_out), _lib.ptr(gw),
                      _lib.ptr(gb), _lib.ptr(self.scratch), y.numel() // k.hidden, k.channels, k.hidden, index,
                      float(frac), float(f_scale), float(vjp_scale), float(grad_scale), _lib.F32, _lib.stream_of(y))

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

    def locate_many(self, times):
        """Interval index / fraction of a list of stage times, with the casts of ``schedule.host_locator``, in one go."""
        k = self.kernels
        tt = torch.tensor(times, dtype=torch.float64).to(k.dtype)
        frac, index = locate(k.knots, tt.to(k.knots.dtype), k.n_rows)
        return index.tolist(), frac.tolist()

    def segment(self, t_hi, t_lo, y_hi, a_hi, method, step_size, *grads):
        """One segment [t_hi -> t_lo] of a fixed-step backward solve WITHOUT a launch per stage.  For this linear
        field d a/ds = a^T df/dz does not involve z, so z(s) and a(s) are two ordinary fused solves (tensor-core
        kernel, reversed time), each leaving the input of every stage in HBM; one more launch contracts the two
        trajectories with dX/dt and the Runge-Kutta weights into dL/dW, dL/db.  Returns a(t_lo), or None when the
        tensor-core kernel or the memory for the two trajectories (2 x stages x paths x 128 bytes) is not available.
        ``grads``: one tensor per parameter, in the order of ``params``."""
        k = self.kernels
        gw, gb = self._by_role(grads)
        hidden, dtype, dev = k.hidden, k.dtype, k.device
        yf = y_hi.reshape(-1, hidden).contiguous()
        af = a_hi.reshape(-1, hidden).contiguous()
        n_paths = yf.size(0)
        tt = torch.tensor([t_hi, t_lo], dtype=torch.float64)
        sched, (_floats, _ints, v) = _schedules.get(tt, k.knots, k.n_rows, method, step_size, dtype, dev)
        n_total = sched.n_steps * sched.n_stages
        if not backprop.fits(dev, n_total * n_paths * hidden * 4, k.param_grad_scratch_bytes(n_paths, n_total)):
            return None
        with torch.cuda.device(dev):
            w2, b2 = k.adjoint_weights
            z_stages = torch.empty(n_total, n_paths, hidden, dtype=dtype, device=dev)
            a_stages = torch.empty_like(z_stages)
            ends = torch.empty(2, n_paths, sched.n_out, hidden, dtype=dtype, device=dev)
            try:
                for which, (start, dump, ww, bb) in enumerate(((yf, z_stages, k.w, k.b), (af, a_stages, w2, b2))):
                    k._fixed(sched, v, ww, bb, start, ends[which], dump)
            except NotImplementedError:
                return None
            rk = {"rk4": (0.125, 0.375, 0.375, 0.125), "midpoint": (0.0, 1.0), "euler": (1.0,)}[method]
            weights = (sched.step_dt.to(torch.float64).unsqueeze(1) * torch.tensor(rk, dtype=torch.float64)).reshape(-1)
            weights = weights.to(dtype).to(dev)
            k.param_grads(z_stages, a_stages, v["stage_index"], v["stage_frac"], weights, n_total, gw, gb)
        return ends[1][:, -1].reshape(a_hi.shape)

    def adaptive_segment(self, t_hi, t_lo, y_hi, a_hi, rtol, atol, gw, gb, slots_hint):
        """One segment [t_hi -> t_lo] of the dopri5 backward solve with the step controller on the device
        (``tcde_dopri5_linear_paired_attempts``): the state z and the adjoint state a advance as one virtual batch of
        2 x paths under one controller, every attempt leaves the inputs of its five weighted stages in the slot of the
        step it would become, and one launch of the parameter-gradient GEMM over the accepted steps' stages adds
        dL/dW, dL/db into ``gw`` / ``gb``.  Returns a(t_lo), or None (not built for this problem / out of memory / more
        accepted steps than slots) -- the caller then runs the host-driven backward."""
        k = self.kernels
        hidden, dev = k.hidden, k.device
        yf = y_hi.reshape(-1, hidden).contiguous()
        af = a_hi.reshape(-1, hidden).contiguous()
        n_paths = yf.size(0)
        if hidden != 32 or k.channels != 8 or n_paths % 256 != 0 or n_paths == 0:
            return None
        with torch.cuda.device(dev):
            w2, b2 = k.adjoint_weights
            fz, fa = k.field(), k.field(w2, b2)

            def field_v(s_time, v):                  # the virtual batch's slope in s = -t (start slope, Hairer's first step)
                return torch.cat([-fz(-s_time, v[:n_paths]), -fa(-s_time, v[n_paths:])])

            # trajectory slots: enough for a few hundred accepted steps, at most a quarter of the free memory; when they are
            # full the device pauses, the filled slots are contracted into the gradients and the solve goes on
            free, _total = torch.cuda.mem_get_info()
            per_slot = 2 * 5 * n_paths * hidden * 4
            max_slots = int(min(max(16, slots_hint), 256, 0.25 * free // per_slot))
            if max_slots < 8:
                return None
            dump_z = torch.empty(max_slots * 5, n_paths, hidden, dtype=torch.float32, device=dev)
            dump_a = torch.empty_like(dump_z)
            q_index = torch.zeros(max_slots * 5, dtype=torch.int32, device=dev)
            q_frac = torch.zeros(max_slots * 5, dtype=torch.float32, device=dev)
            q_weight = torch.zeros(max_slots * 5, dtype=torch.float32, device=dev)
            knots = k.time_knots.detach().to(device=dev, dtype=torch.float32).contiguous()
            stream = _lib.stream_of(yf)

            def launch(state, partials, ctl, out, out_times, first_seq):
                _lib.call("tcde_dopri5_linear_paired_attempts", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(knots),
                          _lib.ptr(k.w), _lib.ptr(k.b), _lib.ptr(w2), _lib.ptr(b2), _lib.ptr(state), _lib.ptr(partials),
                          _lib.ptr(ctl), _lib.ptr(out), _lib.ptr(out_times), 2, n_paths, k.channels, hidden, -1.0,
                          _lib.ptr(dump_z), _lib.ptr(dump_a), _lib.ptr(q_index), _lib.ptr(q_frac), _lib.ptr(q_weight),
                          max_slots, first_seq, adaptive._DEVICE_CHUNK, _lib.F32, stream)

            def contract(last):                      # dL/dW, dL/db += the quadrature over the filled slots
                n_total = 5 * int(last[adaptive.CTL_NACC] - last[adaptive.CTL_BASE])
                if n_total <= 0 or (gw is None and gb is None):
                    return
                if not k.param_grads(dump_z, dump_a, q_index, q_frac, q_weight, n_total, gw, gb):
                    raise RuntimeError("dopri5 adjoint: the parameter-gradient kernel is not built for this problem")

            flushes = []

            def flush(last):                         # the slots are full: empty them before the device goes on
                contract(last)
                flushes.append(last)

            out, last, stats = adaptive.device_controller(
                launch, field_v, torch.cat([yf, af]), [-float(t_hi), -float(t_lo)], rtol, atol, None,
                "dopri5 adjoint: step size underflow / non-finite error estimate at s = {}", on_overflow=flush)
            contract(last)
        self.adaptive_stats = dict(stats, slots=max_slots, flushes=len(flushes))
        return out[n_paths:, 1].reshape(a_hi.shape).clone()
