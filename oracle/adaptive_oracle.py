"""fp64 restatement of the adaptive Dormand-Prince solve and of the continuous adjoint -- TEST INFRASTRUCTURE ONLY.

What this pins
--------------
``torchcde_b200/adaptive.py`` and ``torchcde_b200/csrc/solve_dopri5.cu`` each write the Dormand-Prince constants down
themselves, so comparing the two only shows that they agree with each other.  This module takes the tableau from an
independent source and restates the algorithm the package documents (DESIGN.md sections 3 and 4.2):

  * A, the 5th-order weights b5 and the nodes c are SciPy's ``RK45`` arrays (Dormand & Prince 1980, "A family of
    embedded Runge-Kutta formulae", J. Comp. Appl. Math. 6, 19-26).  The midpoint weights of the dense output are
    ``RK45.P @ [1/2, 1/4, 1/8, 1/16]``.
  * The error weights b5 - b4* are NOT ``RK45.E``.  torchdiffeq's dopri5 estimates the error with the embedded 4th-order
    weights of Shampine (1986, "Some practical Runge-Kutta formulas", Math. Comp. 46, 135-150), written below as
    fractions; ``RK45.E`` belongs to the original Dormand-Prince pair (last weight 1/40 instead of 1/60).
  * The dense output is the quartic through y0, y1 and y_mid with the end slopes dt f0 and dt f1, found by solving that
    5 x 5 system.
  * The controller is torchdiffeq's: RMS norm of err / (atol + rtol max(|y0|, |y1|)), accept when the ratio is <= 1,
    safety 0.9, ifactor 10, dfactor 0.2 (1 when the ratio is below 1), exponent 1/5, Hairer's initial step.

Everything is plain torch fp64, on the device the control lives on (the CPU, or for batches of tens of thousands of
paths the GPU's generic fp64 operators).  The field of a linear CDE comes from ``cde_oracle`` (its spline derivatives and
``linear_field``), the fixed-step grids from ``odeint_port``.  Nothing here imports ``torchcde_b200``.
"""
from fractions import Fraction

import numpy as np
import torch
from scipy.integrate._ivp.rk import RK45

from . import cde_oracle, odeint_port

# ------------------------------------------------------------------------------------------------------ the tableau
A = [[float(v) for v in row] for row in RK45.A]                 # rows of stages 1..6 (row 0 is empty)
B5 = [float(v) for v in RK45.B]                                 # 5th-order weights of k1..k6 (k7 has weight 0)
C = [float(v) for v in RK45.C]                                  # nodes of stages 1..6; stage 7 sits at t + dt
# the error weights b5 - b4*: b5 of Dormand & Prince (the FSAL stage k7 has weight 0) minus Shampine's b4*
B5_EXACT = (Fraction(35, 384), Fraction(0), Fraction(500, 1113), Fraction(125, 192), Fraction(-2187, 6784),
            Fraction(11, 84), Fraction(0))
B4_SHAMPINE = (Fraction(1951, 21600), Fraction(0), Fraction(22642, 50085), Fraction(451, 720),
               Fraction(-12231, 42400), Fraction(649, 6300), Fraction(1, 60))
E = [float(b - b4) for b, b4 in zip(B5_EXACT, B4_SHAMPINE)]
MID = [float(v) for v in RK45.P @ np.array([1 / 2, 1 / 4, 1 / 8, 1 / 16])]
ORDER = 5                                                        # of the step-size rule: exponent 1 / ORDER
QUAD_STAGES = (0, 2, 3, 4, 5)                                    # stages with a non-zero b5: the adjoint's quadrature


def rms(x):
    return float(x.pow(2).mean().sqrt())


# ----------------------------------------------------------------------------------------------- one attempted step
def attempt(field, t, dt, y, k1):
    """One Dormand-Prince attempt from (t, y) with k1 = f(t, y).  Returns a dict with ``y1`` (5th order), ``ks`` (k1..k7,
    k7 = f(t + dt, y1)), ``err`` = dt sum (b5 - b4*) k, ``y_mid`` (the solution at t + dt/2 of the dense output) and
    ``inputs`` (the state each of the seven stages was evaluated at)."""
    ks, inputs = [k1], [y]
    for i in range(1, 6):
        yi = y + dt * sum(A[i][j] * ks[j] for j in range(i) if A[i][j] != 0.0)
        inputs.append(yi)
        ks.append(field(t + dt if C[i] == 1.0 else t + C[i] * dt, yi))
    y1 = y + dt * sum(B5[j] * ks[j] for j in range(6) if B5[j] != 0.0)
    inputs.append(y1)
    ks.append(field(t + dt, y1))
    err = dt * sum(E[j] * ks[j] for j in range(7) if E[j] != 0.0)
    y_mid = y + dt * sum(MID[j] * ks[j] for j in range(7) if MID[j] != 0.0)
    return {"y1": y1, "ks": ks, "err": err, "y_mid": y_mid, "inputs": inputs}


def error_ratio(err, y0, y1, rtol, atol):
    return rms(err / (atol + rtol * torch.max(y0.abs(), y1.abs())))


def next_step(dt, ratio, safety=0.9, ifactor=10.0, dfactor=0.2):
    if ratio == 0.0:
        return dt * ifactor
    if ratio < 1.0:
        dfactor = 1.0
    return dt * min(ifactor, max(safety * ratio ** (-1.0 / ORDER), dfactor))


def initial_step(field, t0, y0, f0, rtol, atol):
    """Hairer, Norsett & Wanner, Solving ODEs I, II.4 (starting step size) for an order-4 error estimate."""
    scale = atol + rtol * y0.abs()
    d0, d1 = rms(y0 / scale), rms(f0 / scale)
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    d2 = rms((field(t0 + h0, y0 + h0 * f0) - f0) / scale) / h0
    if max(d1, d2) <= 1e-15:
        h1 = max(1e-6, h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1.0 / 5)
    return min(100 * h0, h1)


# ---------------------------------------------------------------------------------------------------- dense output
_M = np.array([[1, 0, 0, 0, 0],             # p(0)  = y0
               [1, 1, 1, 1, 1],             # p(1)  = y1
               [1, 1 / 2, 1 / 4, 1 / 8, 1 / 16],   # p(1/2) = y_mid
               [0, 1, 0, 0, 0],             # p'(0) = dt f0
               [0, 1, 2, 3, 4]], dtype=np.float64)   # p'(1) = dt f1
_M_INV = torch.from_numpy(np.linalg.inv(_M))


def dense_coefficients(y0, y1, y_mid, f0, f1, dt):
    """Coefficients c_0..c_4 of p(x) = sum c_m x^m, x = (t - t0) / dt."""
    rhs = torch.stack([y0, y1, y_mid, dt * f0, dt * f1])
    return torch.einsum("mk,k...->m...", _M_INV.to(rhs), rhs)


def dense_evaluate(coeff, x):
    return sum(c * x ** m for m, c in enumerate(coeff))


# ---------------------------------------------------------------------------------------------------- the drivers
class Record:
    """One attempted step: start time, step, decision, error ratio (the drivers fill it in)."""

    def __init__(self, t, dt, accepted, ratio):
        self.t, self.dt, self.accepted, self.ratio = t, dt, accepted, ratio


def _clip_end(t_hi, t_end):
    """Where the paired adjoint lands an accepted step that reaches the end of its segment."""
    return t_end if t_hi >= t_end - 1e-13 * max(1.0, abs(t_end)) else t_hi


def solve(field, y0, times, rtol, atol, first_step=None, clip=False, replay=None, on_accept=None):
    """dopri5 over increasing float ``times`` starting from ``y0``.

    Free running (``replay`` None): the driver makes its own decisions.  Replay: ``replay`` is a list of
    ``(t, dt, accepted)`` -- e.g. what a device recorded -- and the driver takes those steps and decisions instead, from
    its own fp64 state.  ``clip``: the last step ends exactly at ``times[-1]`` (the paired adjoint).  ``on_accept(t, dt,
    result)`` is called for every accepted step.  Returns ``(outputs (len(times), ...), records, first_dt)``."""
    t = times[0]
    y = y0
    f = field(t, y)
    dt = first_step if first_step is not None else initial_step(field, t, y, f, rtol, atol)
    first_dt = dt
    out = [y0]
    records = []
    nxt = 1
    while nxt < len(times):
        if replay is not None:
            if len(records) == len(replay):
                raise RuntimeError("replay ran out of attempts at t = {}".format(t))
            rt, dt, accepted = replay[len(records)]
            assert abs(rt - t) <= 1e-12 * max(1.0, abs(t)), (rt, t)
            t = rt
        elif clip and t + dt > times[-1]:
            dt = times[-1] - t
        res = attempt(field, t, dt, y, f)
        ratio = error_ratio(res["err"], y, res["y1"], rtol, atol)
        if replay is None:
            accepted = ratio <= 1.0
        records.append(Record(t, dt, accepted, ratio))
        if accepted:
            t_hi = _clip_end(t + dt, times[-1]) if clip else t + dt
            if on_accept is not None:
                on_accept(t, dt, res)
            coeff = None
            while nxt < len(times) and times[nxt] <= t_hi:
                if coeff is None:
                    coeff = dense_coefficients(y, res["y1"], res["y_mid"], f, res["ks"][6], dt)
                out.append(dense_evaluate(coeff, (times[nxt] - t) / (t_hi - t)))
                nxt += 1
            t, y, f = t_hi, res["y1"], res["ks"][6]
        if replay is None:
            dt = next_step(dt, ratio)
    return torch.stack(out), records, first_dt


# ---------------------------------------------------------------------------------------------------- the control
class _Control:
    """dX/dt of a cubic spline (``control`` = its coefficient rows) or a linear interpolation (``control`` = its knot
    values) in fp64.  ``time_dtype``: the dtype a stage time is rounded to before the interval lookup (the state's dtype
    in the reference stack)."""

    def __init__(self, control, knots, kind, time_dtype):
        self.control = control.double()
        self.knots = knots.double().to(self.control.device)
        self.kind, self.time_dtype = kind, time_dtype

    def time(self, t):
        return float(torch.tensor(float(t), dtype=torch.float64).to(self.time_dtype))

    def _dxdt_at(self, ts):
        """dX/dt at the fp64 tensor ``ts`` (differentiable in ``ts`` and in the knots)."""
        if self.kind == "cubic":
            return cde_oracle.cubic_derivative(self.control, self.knots, ts)
        return cde_oracle.linear_derivative(self.control, self.knots, ts)

    def dxdt(self, t):
        return self._dxdt_at(torch.tensor(self.time(t), dtype=torch.float64, device=self.knots.device))

    def locate(self, t):
        """(interval, fraction) of a stage time with the lookup the field uses."""
        frac, index = cde_oracle.locate(self.knots.cpu(), self.time(t), self.control.size(-2) - (self.kind == "linear"))
        return int(index), float(frac)


# -------------------------------------------------------------------------------------------- the linear CDE field
class LinearCDE(_Control):
    """f(t, z) = Linear(H, H C)(z).view(H, C) @ dX/dt(t) in fp64 for a cubic spline (``control`` = its coefficient
    rows) or a linear interpolation (``control`` = its knot values).  ``time_dtype``: the dtype a stage time is rounded
    to before the interval lookup (the state's dtype in the reference stack)."""

    def __init__(self, control, knots, weight, bias, kind, time_dtype=torch.float64):
        super().__init__(control, knots, kind, time_dtype)
        self.weight, self.bias = weight.double(), bias.double()
        self.hidden = self.weight.size(1)
        self.channels = self.weight.size(0) // self.hidden

    def __call__(self, t, z):
        return cde_oracle.linear_field(self.weight, self.bias, z, self.dxdt(t))

    def vjp(self, t, z, a):
        """(f, a^T df/dz, a^T df/dW, a^T df/db) by fp64 autograd of ``cde_oracle.linear_field``."""
        w = self.weight.clone().requires_grad_(True)
        b = self.bias.clone().requires_grad_(True)
        zz = z.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            f = cde_oracle.linear_field(w, b, zz, self.dxdt(t))
            gz, gw, gb = torch.autograd.grad(f, (zz, w, b), a)
        return f.detach(), gz, gw, gb

    def regrouped(self):
        """The adjoint state's own linear CDE: a^T df/dz = -Linear(-W regrouped, 0)(a) @ dX/dt."""
        h, c = self.hidden, self.channels
        w2 = -self.weight.view(h, c, h).permute(2, 1, 0).reshape(h * c, h)
        return LinearCDE(self.control, self.knots, w2, torch.zeros_like(self.bias), self.kind, self.time_dtype)


# ------------------------------------------------------------------------------------------ the CDE of any field
class FuncCDE(_Control):
    """f(t, z) = g(t, z) @ dX/dt(t) in fp64 for any fp64 callable ``g(t, z) -> (..., H, C)``, or with ``prod`` the
    callable's own product f(t, z) = g(t, z, dX/dt(t)).  ``g`` gets the stage time as a 0-dim fp64 tensor holding it
    rounded to ``time_dtype``, as the package passes it to ``func`` (under a decreasing ``t`` the time of the original
    frame, as torchdiffeq's reversal ``func(-s)`` does).  ``params``: the fp64 leaf tensors ``g`` reads, created with
    ``requires_grad``; they are what ``vjp`` and ``fixed_adjoint`` differentiate unless told otherwise."""

    def __init__(self, control, knots, g, kind, time_dtype=torch.float64, params=(), prod=False):
        super().__init__(control, knots, kind, time_dtype)
        self.g, self.params, self.prod = g, list(params), prod

    def _field(self, ts, z):
        dx = self._dxdt_at(ts)
        if self.prod:
            return self.g(ts, z, dx)
        return (self.g(ts, z) @ dx.unsqueeze(-1)).squeeze(-1)

    def __call__(self, t, z):
        return self._field(torch.tensor(self.time(t), dtype=torch.float64, device=self.knots.device), z)

    def vjp(self, t, z, a, params=None, with_t=False):
        """(f, a^T df/dz, [a^T df/dp for p in params]) by fp64 autograd; with ``with_t`` also a^T df/dt.  The rounding
        of the stage time to ``time_dtype`` passes the time gradient through unchanged, like ``t.to(dtype)``."""
        params = self.params if params is None else list(params)
        t_ = torch.tensor(float(t), dtype=torch.float64, device=self.knots.device, requires_grad=True)
        zz = z.detach().clone().requires_grad_(True)
        wrt = [zz] + params + ([t_] if with_t else [])
        with torch.enable_grad():
            f = self._field(t_ + (self.time(t) - float(t)), zz)
            grads = torch.autograd.grad(f, wrt, a, allow_unused=True)
        grads = [torch.zeros_like(x) if g is None else g for g, x in zip(grads, wrt)]
        gz, gp = grads[0], grads[1:1 + len(params)]
        return (f.detach(), gz, gp, grads[-1]) if with_t else (f.detach(), gz, gp)


# ------------------------------------------------------------------------------------------------ the fixed adjoint
def fixed_adjoint(cde, ys, grad_ys, times, method, step_size, params=None, with_t=False):
    """torchdiffeq ``odeint_adjoint`` for a fixed-grid method: (z, a, dL/dparams) integrated from t_i back to t_{i-1}
    by ``odeint_port`` (its grid for the reversed segment, its stages), grad_ys[i-1] added at every output time.
    ``ys``, ``grad_ys``: (len(times), P, H).

    A ``LinearCDE`` differentiates (W, b) and returns (dL/dz0, dL/dW, dL/db).  A ``FuncCDE`` differentiates ``params``
    (default: its own list) and returns (dL/dz0, [dL/dp], dL/dt or None).  ``with_t`` (FuncCDE only): the gradients of
    the output times, as ``odeint_adjoint`` forms them when ``t.requires_grad`` -- the augmented state carries the
    integral of -a^T df/dt, ``<f(t_i, y_i), dL/dy_i>`` is dL/dt_i and is subtracted from that integral at every output
    t_i > t_0, and dL/dt_0 is what the integral holds at the end.  Everything is in the frame of ``times`` itself, so a
    decreasing ``times`` needs no sign flip."""
    linear = isinstance(cde, LinearCDE)
    if linear:
        assert params is None and not with_t
        params = [cde.weight, cde.bias]
    elif params is None:
        params = cde.params
    shape_z = ys[0].shape
    n_z = ys[0].numel()
    sizes = [p.numel() for p in params]
    dev = ys.device

    def vjp(t, z, a):
        if linear:
            f, gz, gw, gb = cde.vjp(t, z, a)
            return f, gz, [gw, gb], None
        return cde.vjp(t, z, a, params, with_t) + (() if with_t else (None,))

    def aug(t, v):
        z, a = v[:n_z].view(shape_z), v[n_z:2 * n_z].view(shape_z)
        f, gz, gp, gt = vjp(float(t), z, a)
        parts = [f, -gz] + [-g for g in gp] + ([-gt] if with_t else [])
        return torch.cat([x.reshape(-1) for x in parts])

    a = grad_ys[-1].double().clone()
    gp = [torch.zeros(n, dtype=torch.float64, device=dev) for n in sizes]
    a_t = torch.zeros(1, dtype=torch.float64, device=dev)
    time_grads = [None] * len(times)
    for i in range(len(times) - 1, 0, -1):
        if with_t:
            d_cur = (cde(times[i], ys[i].double()) * grad_ys[i].double()).sum().reshape(1)
            time_grads[i] = d_cur
            a_t = a_t - d_cur
        v0 = torch.cat([ys[i].double().reshape(-1), a.reshape(-1)] + gp + ([a_t] if with_t else []))
        seg = torch.tensor([times[i], times[i - 1]], dtype=torch.float64)
        v1 = odeint_port.odeint(aug, v0, seg, method=method, options={"step_size": step_size})[-1]
        a = v1[n_z:2 * n_z].view(shape_z) + grad_ys[i - 1].double()
        gp = list(torch.split(v1[2 * n_z:2 * n_z + sum(sizes)], sizes))
        if with_t:
            a_t = v1[-1:]
    if linear:
        return a, gp[0].view_as(cde.weight), gp[1]
    time_grads[0] = a_t
    grads_t = torch.cat(time_grads) if with_t else None
    return a, [g.view_as(p) for g, p in zip(gp, params)], grads_t


class PairedSegment:
    """One segment t_hi -> t_lo of the dopri5 adjoint as the device runs it (DESIGN 4.2): in s = -t the virtual state
    (z, a) -- z with (W, b), a with the regrouped, negated W and a zero bias -- under ONE controller (RMS over both
    halves), the last step clipped to the end of the segment, and dL/dW, dL/db as the quadrature
    sum over accepted steps of dt b_i (a_i (x) dX_i) (x) [z_i | 1] at stages 1, 3, 4, 5, 6."""

    def __init__(self, cde):
        self.cde, self.adj = cde, cde.regrouped()

    def field(self, s, v):
        return torch.stack([-self.cde(-s, v[0]), -self.adj(-s, v[1])])

    def run(self, t_hi, t_lo, z_hi, a_hi, rtol, atol, first_step=None, replay=None):
        """Returns a dict: ``a_lo``, ``z_lo``, ``gw``, ``gb``, ``records``, ``first_dt`` and ``steps`` -- per accepted
        step its ``t``, ``dt``, stage ``inputs`` (5 x (2, P, H)) and quadrature ``nodes`` [(interval, fraction, weight)]."""
        cde = self.cde
        h, c = cde.hidden, cde.channels
        gw = torch.zeros(h, c, h, dtype=torch.float64, device=cde.weight.device)
        gb = torch.zeros(h, c, dtype=torch.float64, device=cde.weight.device)
        steps = []

        def on_accept(s, dt, res):
            inputs, nodes = [], []
            for q in QUAD_STAGES:
                sq = s + dt if C[q] == 1.0 else s + C[q] * dt
                w = B5[q] * dt
                v = res["inputs"][q]
                dx = cde.dxdt(-sq)
                gw.add_(w * torch.einsum("ph,pc,pk->hck", v[1], dx, v[0]))
                gb.add_(w * torch.einsum("ph,pc->hc", v[1], dx))
                inputs.append(v)
                nodes.append(cde.locate(-sq) + (w,))
            steps.append({"t": s, "dt": dt, "inputs": inputs, "nodes": nodes})

        v0 = torch.stack([z_hi.double(), a_hi.double()])
        out, records, first_dt = solve(self.field, v0, [-float(t_hi), -float(t_lo)], rtol, atol, first_step=first_step,
                                       clip=True, replay=replay, on_accept=on_accept)
        return {"z_lo": out[-1][0], "a_lo": out[-1][1], "gw": gw.reshape(h * c, h), "gb": gb.reshape(-1),
                "records": records, "first_dt": first_dt, "steps": steps}


def paired_adjoint(cde, ys, grad_ys, times, rtol, atol):
    """The whole dopri5 backward pass, segment by segment between the output times.  Returns (dL/dz0, dL/dW, dL/db)."""
    seg = PairedSegment(cde)
    a = grad_ys[-1].double().clone()
    gw = torch.zeros_like(cde.weight)
    gb = torch.zeros_like(cde.bias)
    for i in range(len(times) - 1, 0, -1):
        r = seg.run(times[i], times[i - 1], ys[i], a, rtol, atol)
        a = r["a_lo"] + grad_ys[i - 1].double()
        gw, gb = gw + r["gw"], gb + r["gb"]
    return a, gw, gb
