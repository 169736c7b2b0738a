"""GPU: the dopri5 forward solve, the fixed-step adjoint and the dopri5 adjoint against the independent fp64 oracle of
their own algorithms (oracle/adaptive_oracle.py: tableau from SciPy, Shampine's error weights, the dense output as the
solution of its defining conditions, torchdiffeq's controller and odeint_adjoint).

The device-controlled solves are driven ONE launch per call (``n_launches=1``; ``first_seq`` says which launch it is), so
that after every launch the control slot, the candidate state, the per-CTA error partials and the adjoint's trajectory
slots can be read and checked against the oracle step started from the device's own state -- no accumulation, tight bars.
The whole solve is then replayed by the oracle with the device's step sequence.  The oracle's arithmetic runs in fp64 on
the GPU through torch's generic operators (cuBLAS DGEMM), none of this package's kernels."""
import math

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import cde_oracle as O
from oracle import odeint_port
from torchcde_b200 import _lib, adaptive, solver
from torchcde_b200.adaptive import (CTL_BASE, CTL_DONE, CTL_DT, CTL_NACC, CTL_NEED_MID, CTL_NEXT_OUT, CTL_NPART,
                                    CTL_NREJ, CTL_OVERFLOW, CTL_PENDING, CTL_RATIO, CTL_T, CTL_TEND, CTL_CUR)

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, C = 32, 8


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _problem(batch, length, kind, seed=0, dtype=torch.float32, hidden=H):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(batch, length, C, generator=gen, device=DEV, dtype=torch.float64).cumsum(1)
         / math.sqrt(length)).to(dtype)
    z0 = torch.randn(batch, hidden, generator=gen, device=DEV, dtype=torch.float64).to(dtype)
    torch.manual_seed(seed)
    func = cde.LinearVectorField(hidden, C, dtype=dtype).to(DEV)
    with torch.no_grad():
        X = (cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x)) if kind == "cubic"
             else cde.LinearInterpolation(x))
    return X, func, z0


def _oracle_cde(X, func, kind, pick=None):
    control = (X._rows() if kind == "cubic" else X._coeffs).detach()
    if pick is not None:
        control = control[pick]
    return AO.LinearCDE(control.double(), X._t.detach().double().cpu(), func.linear.weight.detach().double(),
                        func.linear.bias.detach().double(), kind, time_dtype=func.linear.weight.dtype)


def _device_args(X, func, kind):
    code = _lib.CONTROL_CUBIC if kind == "cubic" else _lib.CONTROL_LINEAR
    control = (X._rows() if kind == "cubic" else X._derivs).detach().contiguous()
    knots = X._t.detach().to(DEV, torch.float32).contiguous()
    return code, control, control.size(-2), knots, func.linear.weight.detach().contiguous(), \
        func.linear.bias.detach().contiguous()


class _Worst:
    """Largest measured error / bar of each check (printed, so that a run with -s reports them)."""

    def __init__(self, name):
        self.name, self.items = name, {}

    def note(self, key, err, bar):
        assert err <= bar, (self.name, key, err, bar)
        e, b = self.items.get(key, (0.0, bar))
        if err / bar >= e / b:
            self.items[key] = (err, bar)

    def report(self):
        print("\n[{}] ".format(self.name) + "; ".join("{}: {:.3g} (bar {:.3g})".format(k, e, b)
                                                    for k, (e, b) in sorted(self.items.items())))


def _path_err(got, want):
    """max over elements of |got - want| / (that path's max |want|)."""
    scale = want.abs().amax(dim=-1, keepdim=True).clamp_min(1e-30)
    return float(((got.double() - want) / scale).abs().max())


# ----------------------------------------------------------------------------------------- the controller's decision
def _check_decision(prev, now, prev_partials, n_elem, worst, clip):
    """Launch n decided attempt n-1 from the partials launch n-1 left: bit-exact RMS in index order, accept iff
    ratio <= 1, torchdiffeq's step-size rule in double.  Returns None (nothing pending) or whether it accepted."""
    if prev[CTL_PENDING] == 0:
        return None
    s = 0.0
    for v in prev_partials[:int(prev[CTL_NPART])].tolist():
        s += v
    ratio = math.sqrt(s / n_elem)
    assert now[CTL_RATIO] == ratio, (now[CTL_RATIO], ratio)
    accepted = now[CTL_NACC] == prev[CTL_NACC] + 1
    assert accepted == (ratio <= 1.0)
    assert now[CTL_NREJ] == prev[CTL_NREJ] + (0 if accepted else 1)
    t_want = prev[CTL_T]
    if accepted:
        t_want = prev[CTL_T] + prev[CTL_DT]
        if clip and t_want >= prev[CTL_TEND] - 1e-13 * max(1.0, abs(prev[CTL_TEND])):
            t_want = prev[CTL_TEND]
    assert now[CTL_T] == t_want
    dt_want = AO.next_step(prev[CTL_DT], ratio)
    if clip and now[CTL_DONE] == 0 and now[CTL_T] + dt_want > now[CTL_TEND]:
        dt_want = now[CTL_TEND] - now[CTL_T]
    worst.note("dt rel (CUDA pow)", abs(now[CTL_DT] - dt_want) / dt_want, 1e-14)
    return accepted


def _check_attempt(field, t, dt, y, k1, y1, k7, ratio, rtol, atol, worst, mid=None):
    """One attempt against the oracle's attempt from the device's own (y, k1).  y etc.: (..., paths, H) fp64."""
    worst.note("k1 vs fp64 field", _path_err(k1, field(t, y)), 1e-5)
    res = AO.attempt(field, t, dt, y, k1)
    worst.note("y1", _path_err(y1, res["y1"]), 1e-5)
    worst.note("k7", _path_err(k7, res["ks"][6]), 1e-5)
    kmax = torch.stack([k.abs().amax(dim=-1, keepdim=True) for k in res["ks"]]).amax(dim=0)
    if mid is not None:
        # y_mid - y is dt * O(k): the bar is set by the k's fp32 error, not by y's scale
        bar = 1e-6 * y.abs().amax(dim=-1, keepdim=True) + 5e-6 * dt * kmax
        worst.note("y_mid / bar", float(((mid - res["y_mid"]).abs() / bar).max()), 1.0)
    tol = atol + rtol * torch.max(y.abs(), res["y1"].abs())
    r_or = AO.rms(res["err"] / tol)
    bar = 1e-3 * r_or + AO.rms(1e-6 * dt * kmax / tol)
    worst.note("ratio vs oracle / bar", abs(ratio - r_or) / bar, 1.0)
    return res


# ---------------------------------------------------------------------------------- (a) dopri5 forward, launch by launch
def _forward_launch_by_launch(X, func, kind, z0, times, rtol, atol, worst, first_step=None, field=None, flipped=False):
    """tcde_dopri5_linear_attempts one launch per call.  ``times``: increasing floats (negated for a decreasing t).
    ``field``: the oracle field in the solve's time (None: only the controller is checked).  Returns the outputs
    (paths, len(times), H), the attempt records, the first step, and per accepted step the number of outputs emitted."""
    code, control, n_rows, knots, w, b = _device_args(X, func, kind)
    sign = -1.0 if flipped else 1.0
    yf = z0.reshape(-1, H).contiguous()
    n_paths = yf.size(0)
    kfield = solver._kernel_field(X, w, b, z0)
    if flipped:
        kfield = solver._reverse(kfield)
    f0 = kfield(times[0], yf)
    dt0 = first_step if first_step is not None else adaptive._initial_step(kfield, times[0], yf, f0, rtol, atol)
    state = torch.empty(5, n_paths, H, dtype=torch.float32, device=DEV)
    state[0].copy_(yf)
    state[2].copy_(f0)
    grid = _lib.load().tcde_dopri5_linear_grid(n_paths)
    partials = torch.zeros(2, grid, dtype=torch.float64, device=DEV)
    ctl = adaptive.initial_control(times[0], dt0, times[-1], rtol, atol).to(DEV)
    out = torch.empty(n_paths, len(times), H, dtype=torch.float32, device=DEV)
    out[:, 0].copy_(yf)
    out_times = torch.tensor(times, dtype=torch.float64, device=DEV)
    prev, prev_part = ctl[1].cpu().tolist(), None
    records, emitted = [], []
    n = 0
    while True:
        _lib.call("tcde_dopri5_linear_attempts", _lib.ptr(control), code, n_rows, _lib.ptr(knots), _lib.ptr(w),
                  _lib.ptr(b), _lib.ptr(state), _lib.ptr(partials), _lib.ptr(ctl), _lib.ptr(out), _lib.ptr(out_times),
                  len(times), n_paths, C, H, sign, n, 1, _lib.F32, _lib.stream_of(yf))
        now = ctl[n & 1].cpu().tolist()
        accepted = _check_decision(prev, now, prev_part, n_paths * H, worst, clip=False)
        if accepted is not None:
            records[-1][2] = accepted
            if accepted:
                emitted.append(int(now[CTL_NEXT_OUT] - prev[CTL_NEXT_OUT]))
        if now[CTL_DONE]:
            break
        part = partials[n & 1].cpu()
        records.append([now[CTL_T], now[CTL_DT], None])
        if field is not None:
            cur = int(now[CTL_CUR])
            st = state.double()
            s = 0.0
            for v in part.tolist():
                s += v
            _check_attempt(field, now[CTL_T], now[CTL_DT], st[cur], st[2 + cur], st[1 - cur], st[3 - cur],
                           math.sqrt(s / (n_paths * H)), rtol, atol, worst, st[4] if now[CTL_NEED_MID] else None)
        prev, prev_part = now, part
        n += 1
        assert n < 100_000
    assert all(r[2] is not None for r in records)
    return out, [tuple(r) for r in records], dt0, emitted


_FORWARD_CASES = {
    # name: (kind, batch, length, times, rtol, atol, first_step)
    "cubic-1": ("cubic", 1, 10, [0.0, 3.7, 9.0], 1e-4, 1e-6, None),
    "linear-129-dense": ("linear", 129, 8, [0.0, 0.02, 0.05, 0.1, 0.125, 2.2, 7.0], 1e-3, 1e-5, 0.125),
    "cubic-300-decreasing": ("cubic", 300, 9, [8.0, 5.5, 2.25, 0.0], 1e-4, 1e-6, None),
    "linear-300-decreasing": ("linear", 300, 9, [8.0, 5.5, 0.0], 1e-4, 1e-6, None),
    "linear-256-knot-stages": ("linear", 256, 16, [0.0, 15.0], 1e-4, 1e-6, 5.0),
    "cubic-grid-stride": ("cubic", None, 8, [0.0, 3.3, 7.0], 1e-4, 1e-6, None),
}


@pytest.mark.parametrize("case", sorted(_FORWARD_CASES))
def test_dopri5_forward_attempt_by_attempt(case):
    kind, batch, length, t_list, rtol, atol, first_step = _FORWARD_CASES[case]
    batch = batch or 256 * (_sm_count() + 3)            # more tile pairs than CTAs: the grid-stride loop runs
    worst = _Worst("dopri5 forward " + case)
    X, func, z0 = _problem(batch, length, kind, seed=len(case))
    cde_or = _oracle_cde(X, func, kind)
    flipped = t_list[0] > t_list[1]
    times = [-v for v in t_list] if flipped else list(t_list)
    field = (lambda s, y: -cde_or(-s, y)) if flipped else cde_or
    with torch.no_grad():
        out, records, dt0, emitted = _forward_launch_by_launch(X, func, kind, z0, times, rtol, atol, worst,
                                                               first_step, field, flipped)
    n_acc = sum(r[2] for r in records)
    assert n_acc >= 3
    if first_step is None:
        f0 = field(times[0], z0.double())
        want = AO.initial_step(field, times[0], z0.double(), f0, rtol, atol)
        worst.note("first dt rel", abs(dt0 - want) / want, 1e-3)
    if case == "linear-129-dense":
        # three outputs inside the first step, one exactly at its end (0.125 = t0 + first_step)
        assert records[0][2] and emitted[0] == 4, (records[:2], emitted[:2])
    if case == "linear-256-knot-stages":
        # first attempt: stage times 1, 4 and 5 are knots; bucketize puts each into the interval on its left
        assert records[0][:2] == (0.0, 5.0)
    # the whole solve replayed by the oracle on every path, with the device's steps and decisions
    want, rep, _ = AO.solve(field, z0.double(), times, rtol, atol, replay=records)
    assert len(rep) == len(records)
    scale = float(want.abs().max())
    worst.note("outputs vs replay", float((out.double() - want.movedim(0, 1)).abs().max()) / scale, 2e-5)
    # cdeint (48 launches per host read) returns exactly these bits
    with torch.no_grad():
        got = cde.cdeint(X, func, z0, torch.tensor(t_list, dtype=torch.float64), adjoint=False, rtol=rtol, atol=atol,
                         options={} if first_step is None else {"first_step": first_step})
    assert cde.cdeint.last_stats["device_controlled"] and cde.cdeint.last_stats["n_accepted"] == n_acc
    assert torch.equal(got, out)
    worst.report()


# -------------------------------------------------------------------------------------- (b) the host driver in fp64
@pytest.mark.parametrize("kind", ["cubic", "linear"])
def test_host_dopri5_fp64_against_the_free_running_oracle(kind, monkeypatch):
    """adaptive.Dopri5 with the fp64 kernel field (hidden 16: the host-driven route) makes the oracle's decisions.  The
    solve stays inside one spline interval: where a step straddles a knot the error estimate jumps with the knot's position
    inside the step, so fp64 rounding alone would let two correct drivers drift apart there."""
    worst = _Worst("host dopri5 fp64 " + kind)
    X, func, z0 = _problem(40, 10, kind, seed=2, dtype=torch.float64, hidden=16)
    cde_or = _oracle_cde(X, func, kind)
    t = [1.05, 1.3, 1.62, 1.95]
    rtol, atol = 1e-9, 1e-11
    firsts = []
    real = adaptive._initial_step

    def record(*a, **k):
        firsts.append(real(*a, **k))
        return firsts[-1]
    monkeypatch.setattr(adaptive, "_initial_step", record)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, torch.tensor(t, dtype=torch.float64), adjoint=False, rtol=rtol, atol=atol)
    stats = cde.cdeint.last_stats
    assert not stats["device_controlled"]
    want, records, dt0 = AO.solve(cde_or, z0.double(), t, rtol, atol)
    worst.note("first dt rel", abs(firsts[0] - dt0) / dt0, 1e-12)
    worst.note("outputs", float((out - want.movedim(0, 1)).abs().max()) / float(want.abs().max()), 1e-10)
    assert stats["n_accepted"] == sum(r.accepted for r in records) > 10
    assert stats["n_rejected"] == sum(not r.accepted for r in records)
    worst.report()


# ---------------------------------------------------------------------------------- (c) fixed-step adjoint vs oracle
_ADJ_T = [0.35, 2.3, 5.9, 8.45]           # output times off the knots; the step 0.4 divides none of the segments
_ADJ_CACHE = {}


def _adjoint_problem(kind):
    if kind not in _ADJ_CACHE:
        X, func, z0 = _problem(200, 10, kind, seed=7)
        g = torch.randn(len(_ADJ_T), 200, H, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
        _ADJ_CACHE[kind] = (X, func, z0, g, {})
    return _ADJ_CACHE[kind]


def _oracle_fixed_adjoint(kind, method):
    X, func, z0, g, done = _adjoint_problem(kind)
    if method not in done:
        cde_or = _oracle_cde(X, func, kind)
        ys = odeint_port.odeint(cde_or, z0.double(), torch.tensor(_ADJ_T, dtype=torch.float64), method=method,
                                  options={"step_size": 0.4})
        done[method] = AO.fixed_adjoint(cde_or, ys, g.double(), _ADJ_T, method, 0.4)
    return done[method]


@pytest.mark.parametrize("route,variant", [("three-launch", 0), ("three-launch", 1), ("three-launch", 2),
                                           ("per-stage", 0)])
@pytest.mark.parametrize("kind", ["cubic", "linear"])
@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
def test_fixed_step_adjoint_against_the_oracle(method, kind, route, variant, monkeypatch):
    """cdeint(adjoint=True) for a fixed-step method against torchdiffeq's odeint_adjoint in fp64: dL/dz0 within 1e-5 of
    its scale, dL/dW and dL/db within 2e-4 (variant 0: 2xBF16 contraction) / 3e-5 (variants 1, 2)."""
    worst = _Worst("fixed adjoint {} {} {} v{}".format(method, kind, route, variant))
    X, func, z0, g, _ = _adjoint_problem(kind)
    want = _oracle_fixed_adjoint(kind, method)
    real = solver._kernel_vjp
    used = []

    def probe(*a, **k):
        st = real(*a, **k)
        inner = st.segment

        def segment(*sa, **sk):
            res = None if route == "per-stage" else inner(*sa, **sk)
            used.append(res is not None)
            return res
        st.segment = segment
        return st
    monkeypatch.setattr(solver, "_kernel_vjp", probe)
    if variant == 1:
        # variant 1 is the CUDA-core solve, which keeps no stage inputs: select it for the contraction only
        real_call = _lib.call

        def call(name, *args):
            if name != "tcde_linear_field_param_grads":
                return real_call(name, *args)
            real_call("tcde_set_solve_variant", 1)
            try:
                return real_call(name, *args)
            finally:
                real_call("tcde_set_solve_variant", 0)
        monkeypatch.setattr(_lib, "call", call)
    try:
        _lib.call("tcde_set_solve_variant", 0 if variant == 1 else variant)
        zz = z0.clone().requires_grad_(True)
        func.zero_grad()
        out = cde.cdeint(X, func, zz, torch.tensor(_ADJ_T, dtype=torch.float64), adjoint=True, method=method, options={"step_size": 0.4})
        (out * g.movedim(0, 1)).sum().backward()
        torch.cuda.synchronize()
    finally:
        _lib.call("tcde_set_solve_variant", 0)
    assert used == [route == "three-launch"] * (len(_ADJ_T) - 1)
    got = (zz.grad, func.linear.weight.grad, func.linear.bias.grad)
    bars = (1e-5, 2e-4 if variant == 0 else 3e-5, 2e-4 if variant == 0 else 3e-5)
    for name, a, b, bar in zip(("dL/dz0", "dL/dW", "dL/db"), got, want, bars):
        worst.note(name, float((a.double() - b).abs().max()) / float(b.abs().max()), bar)
    worst.report()


# ------------------------------------------------------------------------ (d) dopri5 adjoint, launch by launch
def _paired_launch_by_launch(X, func, kind, z_hi, a_hi, t_hi, t_lo, rtol, atol, max_slots, worst, check=True,
                             cde_or=None, pick=None):
    """One segment t_hi -> t_lo of the dopri5 adjoint through tcde_dopri5_linear_paired_attempts, one launch per call,
    the trajectory slots contracted (tcde_linear_field_param_grads) whenever the device pauses.  ``check``: compare
    every attempt's stage inputs and every accepted step's quadrature nodes with the oracle (``cde_or``).  Returns
    (z(t_lo), a(t_lo), dL/dW, dL/db, records, first step, flushes)."""
    code, control, n_rows, knots, w, b = _device_args(X, func, kind)
    n_paths = z_hi.size(0)
    w2 = w.view(H, C, H).permute(2, 1, 0).contiguous().view(H * C, H).neg()
    b2 = torch.zeros_like(b)
    seg = AO.PairedSegment(cde_or) if cde_or is not None else None
    v0 = torch.cat([z_hi, a_hi]).contiguous()
    s0, s1 = -float(t_hi), -float(t_lo)
    fz, fa = solver._kernel_field(X, w, b, z_hi), solver._kernel_field(X, w2, b2, z_hi)
    f0 = torch.cat([-fz(-s0, z_hi), -fa(-s0, a_hi)])
    dt0 = adaptive._initial_step(lambda s, v: torch.cat([-fz(-s, v[:n_paths]), -fa(-s, v[n_paths:])]), s0, v0, f0,
                                 rtol, atol)
    state = torch.empty(5, 2 * n_paths, H, dtype=torch.float32, device=DEV)
    state[0].copy_(v0)
    state[2].copy_(f0)
    grid = _lib.load().tcde_dopri5_linear_grid(2 * n_paths)
    partials = torch.zeros(2, grid, dtype=torch.float64, device=DEV)
    ctl = adaptive.initial_control(s0, dt0, s1, rtol, atol).to(DEV)
    out = torch.empty(2 * n_paths, 2, H, dtype=torch.float32, device=DEV)
    out[:, 0].copy_(v0)
    out_times = torch.tensor([s0, s1], dtype=torch.float64, device=DEV)
    dump_z = torch.empty(max_slots * 5, n_paths, H, dtype=torch.float32, device=DEV)
    dump_a = torch.empty_like(dump_z)
    q_index = torch.zeros(max_slots * 5, dtype=torch.int32, device=DEV)
    q_frac = torch.zeros(max_slots * 5, dtype=torch.float32, device=DEV)
    q_weight = torch.zeros(max_slots * 5, dtype=torch.float32, device=DEV)
    gw, gb = torch.zeros_like(w), torch.zeros_like(b)
    knots32 = X._t.detach().float().cpu()
    lib = _lib.load()

    def contract(n_steps):
        n_total = 5 * n_steps
        if n_total == 0:
            return
        nbytes = lib.tcde_linear_field_param_grads_scratch_bytes(n_paths, n_total, C, H)
        scratch = torch.empty(max(nbytes // 4, 4), dtype=torch.float32, device=DEV)
        _lib.call("tcde_linear_field_param_grads", _lib.ptr(control), code, n_rows, _lib.ptr(dump_z), _lib.ptr(dump_a),
                  _lib.ptr(q_index), _lib.ptr(q_frac), _lib.ptr(q_weight), n_total, _lib.ptr(gw), _lib.ptr(gb),
                  _lib.ptr(scratch), n_paths, C, H, 1.0, _lib.F32, _lib.stream_of(z_hi))

    prev, prev_part = ctl[1].cpu().tolist(), None
    records, flushes, n = [], 0, 0
    while True:
        _lib.call("tcde_dopri5_linear_paired_attempts", _lib.ptr(control), code, n_rows, _lib.ptr(knots), _lib.ptr(w),
                  _lib.ptr(b), _lib.ptr(w2), _lib.ptr(b2), _lib.ptr(state), _lib.ptr(partials), _lib.ptr(ctl),
                  _lib.ptr(out), _lib.ptr(out_times), 2, n_paths, C, H, -1.0, _lib.ptr(dump_z), _lib.ptr(dump_a),
                  _lib.ptr(q_index), _lib.ptr(q_frac), _lib.ptr(q_weight), max_slots, n, 1, _lib.F32,
                  _lib.stream_of(z_hi))
        now = ctl[n & 1].cpu().tolist()
        accepted = _check_decision(prev, now, prev_part, 2 * n_paths * H, worst, clip=True)
        if accepted is not None:
            records[-1][2] = accepted
            if accepted and check:
                # the accepted step's quadrature nodes: the reference's interval lookup of the float32 stage time
                slot = int(prev[CTL_NACC] - prev[CTL_BASE])
                t, dt = prev[CTL_T], prev[CTL_DT]
                qi = q_index[slot * 5:slot * 5 + 5].cpu()
                qf = q_frac[slot * 5:slot * 5 + 5].cpu()
                qw = q_weight[slot * 5:slot * 5 + 5].cpu()
                for k, q in enumerate(AO.QUAD_STAGES):
                    tq = torch.tensor(-(t + dt if AO.C[q] == 1.0 else t + AO.C[q] * dt), dtype=torch.float64).float()
                    frac, index = O.locate(knots32, tq, n_rows)
                    assert int(qi[k]) == int(index) and bool(qf[k] == frac), (k, int(qi[k]), int(index), qf[k], frac)
                    assert bool(qw[k] == torch.tensor(AO.B5[q] * dt, dtype=torch.float64).float()), k
        n += 1
        if now[CTL_DONE]:
            contract(int(now[CTL_NACC] - now[CTL_BASE]))
            if now[CTL_OVERFLOW] == 0:
                break
            # the slots are full: contract them, hand them back, resume where the device paused
            flushes += 1
            now[CTL_DONE], now[CTL_OVERFLOW], now[CTL_BASE] = 0.0, 0.0, now[CTL_NACC]
            ctl[(n - 1) & 1].copy_(torch.tensor(now, dtype=torch.float64))
            prev, prev_part = now, None
            continue
        part = partials[(n - 1) & 1].cpu()
        records.append([now[CTL_T], now[CTL_DT], None])
        if check:
            cur = int(now[CTL_CUR])
            st = state.double().view(5, 2, n_paths, H)
            s = 0.0
            for v in part.tolist():
                s += v
            res = _check_attempt(seg.field, now[CTL_T], now[CTL_DT], st[cur], st[2 + cur], st[1 - cur], st[3 - cur],
                                 math.sqrt(s / (2 * n_paths * H)), rtol, atol, worst)
            slot = int(now[CTL_NACC] - now[CTL_BASE])
            for k, q in enumerate(AO.QUAD_STAGES):
                want = res["inputs"][q]
                worst.note("dump z", _path_err(dump_z[slot * 5 + k], want[0]), 1e-5)
                worst.note("dump a", _path_err(dump_a[slot * 5 + k], want[1]), 1e-5)
        prev, prev_part = now, part
        assert n < 100_000
    torch.cuda.synchronize()
    return (out[:n_paths, 1], out[n_paths:, 1], gw, gb, [tuple(r) for r in records], dt0, flushes)


@pytest.mark.parametrize("kind,batch,slots", [("cubic", 256, 64), ("linear", 512, 64), ("cubic", 512, 16),
                                              ("cubic", None, 64)])
def test_dopri5_adjoint_attempt_by_attempt(kind, batch, slots):
    """tcde_dopri5_linear_paired_attempts for one segment: every decision, every attempt's stage inputs in its trajectory
    slot, every accepted step's quadrature nodes, then a(t_lo), dL/dW and dL/db against the oracle's replay.  The largest
    batch has more tile pairs than CTAs, so one CTA switches from z's weights to the adjoint's inside its loop; 16 slots
    make the device pause and resume."""
    batch = batch or 256 * (_sm_count() + 3)
    worst = _Worst("dopri5 adjoint {} {} slots {}".format(kind, batch, slots))
    X, func, z0 = _problem(batch, 10, kind, seed=batch + slots)
    gen = torch.Generator(device=DEV).manual_seed(5)
    a_hi = torch.randn(batch, H, generator=gen, device=DEV)
    cde_or = _oracle_cde(X, func, kind)
    rtol, atol = 1e-5, 1e-7
    t_hi, t_lo = 9.0, 0.5
    with torch.no_grad():
        z_lo, a_lo, gw, gb, records, dt0, flushes = _paired_launch_by_launch(
            X, func, kind, z0, a_hi, t_hi, t_lo, rtol, atol, slots, worst, cde_or=cde_or)
    n_acc = sum(r[2] for r in records)
    assert n_acc > 16 and (flushes >= 1 or slots > 16), (n_acc, flushes)
    want = AO.PairedSegment(cde_or).run(t_hi, t_lo, z0.double(), a_hi.double(), rtol, atol, replay=records)
    for name, got, ref, bar in (("z(t_lo)", z_lo, want["z_lo"], 2e-5), ("a(t_lo)", a_lo, want["a_lo"], 2e-5),
                                ("dL/dW", gw, want["gw"], 2e-4), ("dL/db", gb, want["gb"], 2e-4)):
        worst.note(name, float((got.double() - ref).abs().max()) / float(ref.abs().max()), bar)
    worst.report()


# ----------------------------------------------------------------------------------------------- (e) BASELINE sizes
def _picked(batch, count=24):
    return torch.linspace(0, batch - 1, count, device=DEV).round().long()


def test_config3_training_step_against_the_oracle(monkeypatch):
    """BASELINE config 3 training step: 65,536 x 256, rk4 with step 1, adjoint=True, a loss on 24 paths spread over the
    batch.  Every other path has a = 0 and adds exactly nothing to dL/dW, dL/db, so the fp64 oracle on those 24 paths
    is the full reference."""
    worst = _Worst("config 3 training step")
    batch, length = 65536, 256
    X, func, z0 = _problem(batch, length, "cubic", seed=31)
    pick = _picked(batch)
    g = torch.randn(len(pick), H, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)
    real = solver._kernel_vjp
    used = []

    def probe(*a, **k):
        st = real(*a, **k)
        inner = st.segment
        st.segment = lambda *sa, **sk: used.append(inner(*sa, **sk)) or used[-1]
        return st
    monkeypatch.setattr(solver, "_kernel_vjp", probe)
    zz = z0.clone().requires_grad_(True)
    out = cde.cdeint(X, func, zz, X.interval, adjoint=True, method="rk4", options={"step_size": 1.0})
    (out[pick, -1] * g).sum().backward()
    assert len(used) == 1 and used[0] is not None                    # the three-launch route
    rest = torch.ones(batch, dtype=torch.bool, device=DEV)
    rest[pick] = False
    assert not bool(zz.grad[rest].any())
    cde_or = _oracle_cde(X, func, "cubic", pick)
    times = [0.0, float(length - 1)]
    ys = odeint_port.odeint(cde_or, z0[pick].double(), torch.tensor(times, dtype=torch.float64), method="rk4",
                              options={"step_size": 1.0})
    worst.note("forward", float((out[pick].detach().double().movedim(0, 1) - ys).abs().max()) / float(ys.abs().max()),
               1e-5)
    grad_ys = torch.stack([torch.zeros_like(g), g]).double()
    wz, ww, wb = AO.fixed_adjoint(cde_or, ys, grad_ys, times, "rk4", 1.0)
    for name, a, b, bar in (("dL/dz0", zz.grad[pick], wz, 1e-5), ("dL/dW", func.linear.weight.grad, ww, 2e-4),
                            ("dL/db", func.linear.bias.grad, wb, 2e-4)):
        worst.note(name, float((a.double() - b).abs().max()) / float(b.abs().max()), bar)
    worst.report()


def test_config4_forward_and_backward_replayed():
    """BASELINE config 4 (dopri5 at cdeint's defaults, 65,536 x 256): forward and one backward segment recorded one launch
    at a time (every decision checked bit for bit), then replayed by the oracle on 24 paths spread over the batch."""
    worst = _Worst("config 4")
    batch, length = 65536, 256
    rtol, atol = 1e-4, 1e-6
    X, func, z0 = _problem(batch, length, "cubic", seed=41)
    pick = _picked(batch)
    cde_or = _oracle_cde(X, func, "cubic", pick)
    times = [0.0, float(length - 1)]
    with torch.no_grad():
        out, records, _, _ = _forward_launch_by_launch(X, func, "cubic", z0, times, rtol, atol, worst)
    want, _, _ = AO.solve(cde_or, z0[pick].double(), times, rtol, atol, replay=records)
    worst.note("forward vs replay", float((out[pick].double().movedim(0, 1) - want).abs().max())
               / float(want.abs().max()), 2e-5)
    a_hi = torch.zeros(batch, H, device=DEV)
    a_hi[pick] = torch.randn(len(pick), H, generator=torch.Generator(device=DEV).manual_seed(6), device=DEV)
    z_hi = out[:, -1].contiguous()
    with torch.no_grad():
        z_lo, a_lo, gw, gb, brecords, _, _ = _paired_launch_by_launch(X, func, "cubic", z_hi, a_hi, times[-1], times[0],
                                                                      rtol, atol, 128, worst, check=False)
    print("config 4: forward {} attempts ({} accepted), backward {} attempts ({} accepted)".format(
        len(records), sum(r[2] for r in records), len(brecords), sum(r[2] for r in brecords)))
    rep = AO.PairedSegment(cde_or).run(times[-1], times[0], z_hi[pick].double(), a_hi[pick].double(), rtol, atol,
                                       replay=brecords)
    assert not bool(a_lo[~torch.isin(torch.arange(batch, device=DEV), pick)].any())
    # z went 255 time units forward and back again: ~1,000 fp32 steps
    for name, got, ref, bar in (("z(0)", z_lo[pick], rep["z_lo"], 1e-4), ("a(0)", a_lo[pick], rep["a_lo"], 2e-5),
                                ("dL/dW", gw, rep["gw"], 2e-4), ("dL/db", gb, rep["gb"], 2e-4)):
        worst.note(name, float((got.double() - ref).abs().max()) / float(ref.abs().max()), bar)
    worst.report()
