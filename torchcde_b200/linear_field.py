"""The README's linear vector field and ``LinearFieldKernels``, the owner of every kernel route of ``cdeint`` for one
(control, linear field, z0) problem: fused fixed-step solve, kernel field, device-controlled dopri5, adjoint stage."""
import functools
import math
import warnings
import weakref

import torch

from . import _lib, adaptive
from .controls import _control_signature, _schedule_knots
from .schedule import ScheduleCache, host_locator, locate

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
    def adjoint_weights(self):
        """-W with rows regrouped as (k, c) and columns h, and a zero bias: the weights of the adjoint state's own CDE."""
        h, c = self.hidden, self.channels
        return self.w.view(h, c, h).permute(2, 1, 0).contiguous().view(h * c, h).neg_(), torch.zeros_like(self.b)

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

    def launch(self, index, frac, y, a, f_out, vjp_out, gw, gb, f_scale, vjp_scale, grad_scale):
        k = self.kernels
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
        gw = torch.zeros_like(k.w) if "w" in self.roles else None
        gb = torch.zeros_like(k.b) if "b" in self.roles else None
        self.launch(index, frac, yf, af, f, vjp_y, gw, gb, 1.0, scale, scale)
        return f.view_as(y), vjp_y.view_as(y), [gw if r == "w" else gb for r in self.roles]

    def locate_many(self, times):
        """Interval index / fraction of a list of stage times, with the casts of ``schedule.host_locator``, in one go."""
        k = self.kernels
        tt = torch.tensor(times, dtype=torch.float64).to(k.dtype)
        frac, index = locate(k.knots, tt.to(k.knots.dtype), k.n_rows)
        return index.tolist(), frac.tolist()

    def segment(self, t_hi, t_lo, y_hi, a_hi, method, step_size, gw, gb):
        """One segment [t_hi -> t_lo] of a fixed-step backward solve WITHOUT a launch per stage.  For this linear
        field d a/ds = a^T df/dz does not involve z, so z(s) and a(s) are two ordinary fused solves (tensor-core
        kernel, reversed time), each leaving the input of every stage in HBM; one more launch contracts the two
        trajectories with dX/dt and the Runge-Kutta weights into dL/dW, dL/db.  Returns a(t_lo), or None when the
        tensor-core kernel or the memory for the two trajectories (2 x stages x paths x 128 bytes) is not available."""
        k = self.kernels
        hidden, dtype, dev = k.hidden, k.dtype, k.device
        yf = y_hi.reshape(-1, hidden).contiguous()
        af = a_hi.reshape(-1, hidden).contiguous()
        n_paths = yf.size(0)
        tt = torch.tensor([t_hi, t_lo], dtype=torch.float64)
        sched, (_floats, _ints, v) = _schedules.get(tt, k.knots, k.n_rows, method, step_size, dtype, dev)
        n_total = sched.n_steps * sched.n_stages
        scratch_bytes = k.param_grad_scratch_bytes(n_paths, n_total)
        if scratch_bytes < 0:
            return None
        need = 2 * n_total * n_paths * hidden * 4
        with torch.cuda.device(dev):
            free, _total = torch.cuda.mem_get_info()
            if need + scratch_bytes > 0.7 * free:
                return None
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
