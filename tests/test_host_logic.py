"""Host-side logic that needs no GPU: validation, the fixed-step schedule, func recognition."""
import pytest
import torch

import torchcde_b200 as cde
from oracle import cde_oracle as O
from oracle import odeint_port
from torchcde_b200 import schedule, solver


def test_validation_errors_match_reference_wording():
    f = cde.hermite_cubic_coefficients_with_backward_differences
    with pytest.raises(ValueError, match="floating point"):
        f(torch.zeros(3, 2, dtype=torch.int64))
    with pytest.raises(ValueError, match="at least two dimensions"):
        f(torch.zeros(3))
    with pytest.raises(ValueError, match="monotonically increasing"):
        f(torch.zeros(3, 2), torch.tensor([0.0, 2.0, 1.0]))
    with pytest.raises(ValueError, match="one dimensional"):
        cde.natural_cubic_coeffs(torch.zeros(3, 2), torch.zeros(3, 1))
    with pytest.raises(ValueError, match="time dimension of X must equal"):
        cde.linear_interpolation_coeffs(torch.zeros(3, 2), torch.tensor([0.0, 1.0]))
    with pytest.raises(ValueError, match="at least 2"):
        cde.natural_cubic_spline_coeffs(torch.zeros(1, 2))
    with pytest.raises(ValueError, match="invalid coeffs"):
        cde.CubicSpline(torch.zeros(2, 3, 7))


def test_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="no CPU path"):
        cde.hermite_cubic_coefficients_with_backward_differences(torch.zeros(2, 5, 3))
    X = cde.CubicSpline(torch.zeros(2, 4, 8))
    with pytest.raises(RuntimeError, match="no CPU path"):
        X.derivative(torch.tensor(0.5))
    with pytest.raises(RuntimeError, match="no CPU path"):
        cde.cdeint(X, cde.LinearVectorField(3, 2), torch.zeros(2, 3), X.interval, adjoint=False, method="rk4",
                   options={"step_size": 1.0})


def test_cdeint_argument_errors():
    X = cde.CubicSpline(torch.zeros(2, 4, 8))
    f = cde.LinearVectorField(3, 2)
    z0 = torch.zeros(2, 3)
    with pytest.raises(ValueError, match="Unrecognised backend"):
        cde.cdeint(X, f, z0, X.interval, backend="nope", method="rk4")
    with pytest.raises(ValueError, match="'derivative' method"):
        cde.cdeint(object(), f, z0, X.interval, method="rk4")
    with pytest.raises(NotImplementedError, match="not built"):
        cde.cdeint(X, f, z0, X.interval, method="bosh3")
    with pytest.raises(ValueError, match="batch dimensions"):
        cde.cdeint(X, f, torch.zeros(5, 3), X.interval, adjoint=False, method="rk4")
    with pytest.raises(NotImplementedError, match="torchsde"):
        cde.cdeint(X, f, z0, X.interval, backend="torchsde")


def test_spline_buffers_are_views_with_reference_names():
    coeffs = torch.randn(2, 5, 12)
    X = cde.CubicSpline(coeffs)
    assert [n for n, _ in X.named_buffers()] == ["_t", "_a", "_b", "_two_c", "_three_d"]
    assert X._b.data_ptr() == coeffs[..., 3:6].data_ptr()          # interpolation_cubic.py:297-305
    assert X.interval.tolist() == [0.0, 5.0] and X.grid_points.numel() == 6
    lin = cde.LinearInterpolation(torch.randn(2, 5, 3))
    assert [n for n, _ in lin.named_buffers()] == ["_t", "_coeffs", "_derivs"]     # interpolation_linear.py:191-193


# the fixed-step schedules of tests/test_gpu_fixed_routes.py on 40 knots: name: (t, step_size, uneven knots)
FIXED_SCHEDULES = {
    "F1": ([0.0, 0.5], 1.0, False),                             # one clipped step
    "F2": (None, None, False),                                  # t = every knot, no step_size
    "F3": ([0.0, 0.3, 0.35, 0.9, 7.0, 39.0], 1.0, False),       # three outputs inside step 0, outputs on grid points
    "F4": ([0.0, 9.8], 0.7, False),                             # float32 t: a zero-length last step
    "F5": ([0.0, 10.0001], 1.0, False),                         # a last step of 1e-4
    "F6": ([0.0, 7.75, 39.0], 3.0, False),                      # every rk4 stage on a knot
    "F7": ([0.5, 20.0, 30.1], 2.5, True),                       # uneven knots, steps longer than intervals
    "F8": ([39.0, 20.5, 3.0, 0.0], 0.5, False),                 # decreasing t
}


def fixed_schedule_knots(uneven, seed=0):
    """40 float32 knots: 0..39, or widths drawn in [0.6, 1.4)."""
    if not uneven:
        return torch.arange(40, dtype=torch.float32)
    widths = 0.6 + 0.8 * torch.rand(39, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    return torch.cat([torch.zeros(1, dtype=torch.float64), widths.cumsum(0)]).float()


_SCHEDULE_CASES = [pytest.param(m, s, None, id="{}-{}".format(m, s)) for m, s in
                   [("rk4", 1.0), ("rk4", 0.4), ("midpoint", 0.5), ("euler", 0.25), ("rk4", None)]]
_SCHEDULE_CASES += [pytest.param(m, FIXED_SCHEDULES[n][1], n, id="{}-{}".format(m, n))
                    for n in FIXED_SCHEDULES for m in ("rk4", "midpoint", "euler")]


@pytest.mark.parametrize("dtype_t", [torch.float32, torch.float64])
@pytest.mark.parametrize("method,step,sname", _SCHEDULE_CASES)
def test_schedule_reproduces_the_stage_by_stage_arithmetic(dtype_t, method, step, sname, monkeypatch):
    """Drive the oracle's solver with a recording field and compare every stage's interval and
    fraction, computed one stage at a time the reference's way, with the batched table; and every
    output's step, mode (start / end / interpolated) and slope with where the oracle's ``_between``
    places it."""
    if sname is None:
        knots = (torch.rand(12, dtype=torch.float64) + 0.2).cumsum(0).float()
        lo, hi = float(knots[0]), float(knots[-1])
        t = torch.tensor([lo, lo + 0.37 * (hi - lo), lo + 0.5 * (hi - lo), hi], dtype=dtype_t)
    else:
        ts, _step, uneven = FIXED_SCHEDULES[sname]
        knots = fixed_schedule_knots(uneven)
        t = knots.to(dtype_t) if ts is None else torch.tensor(ts, dtype=dtype_t)
    n_intervals = knots.numel() - 1
    n_stages = schedule.N_STAGES[method]
    seen, placed = [], []

    def field(s, y):
        frac, idx = O.locate(knots, s, n_intervals)
        seen.append((int(idx), float(frac)))
        return y * 0

    real_between = odeint_port._between

    def between(t0, t1, y0, y1, tj):
        # called after the stages of the step that ends at t1
        mode = 0 if tj == t0 else 1 if tj == t1 else 2
        slope = float(((tj - t0) / (t1 - t0)).to(torch.float32)) if mode == 2 else 0.0
        placed.append((len(seen) // n_stages - 1, mode, slope))
        return real_between(t0, t1, y0, y1, tj)

    monkeypatch.setattr(odeint_port, "_between", between)
    options = {} if step is None else {"step_size": step}
    odeint_port.odeint(field, torch.zeros(1), t, method=method, options=options)
    sched = schedule.build_schedule(t, knots, n_intervals, method, step, torch.float32)
    flat_idx = sched.stage_index.reshape(-1).tolist()
    flat_frac = sched.stage_frac.reshape(-1).tolist()
    assert len(seen) == len(flat_idx) == sched.n_steps * n_stages
    assert [s[0] for s in seen] == flat_idx                 # interval indices: bit exact
    assert [s[1] for s in seen] == flat_frac
    assert sched.out_step[0] == -1 and sched.n_out == t.numel()
    table = list(zip(sched.out_step.tolist(), sched.out_mode.tolist(), sched.out_slope.tolist()))[1:]
    assert table == placed                                  # output placement: bit exact
    dts = sched.step_dt.tolist()
    if sname == "F4" and dtype_t == torch.float32:
        assert dts[-1] == 0.0 and sched.n_steps == 15       # 14 * 0.7 is 9.8 in float32: the last step has no length
    if sname == "F5":
        assert 0 < dts[-1] < 2e-4
    if sname == "F6" and method == "rk4":
        assert all(f in (0.0, 1.0) for f in flat_frac)      # every stage on a knot


def test_schedule_knot_semantics_and_reversal():
    knots = torch.linspace(0, 255, 256)
    s = schedule.build_schedule(torch.tensor([0.0, 255.0]), knots, 255, "rk4", 1.0, torch.float32)
    assert s.n_steps == 255 and s.stage_index[0].tolist() == [0, 0, 0, 0]
    # step n > 0: k1 sits exactly on knot n and reads interval n-1 with fraction 1 (SURVEY 8a row 2)
    assert s.stage_index[7].tolist() == [6, 7, 7, 7] and float(s.stage_frac[7, 0]) == 1.0
    r = schedule.build_schedule(torch.tensor([255.0, 0.0]), knots, 255, "rk4", 1.0, torch.float32)
    assert r.sign == -1.0 and r.stage_index[0].tolist() == [254, 254, 254, 253]
    with pytest.raises(ValueError):
        schedule.build_schedule(torch.tensor([0.0, 1.0, 0.5]), knots, 255, "rk4", 1.0, torch.float32)


def test_linear_field_recognition():
    z0 = torch.randn(4, 3)
    t0 = [0.0, 1.0]                  # the integration interval: the probe picks its own non-degenerate times in it
    good = cde.LinearVectorField(3, 2)
    assert solver.linear_field_of(good, z0, 2, t0)[0] is good.linear.weight
    assert solver.linear_field_of(good, z0, 5, t0) is None            # wrong channel count

    class Readme(torch.nn.Module):                                     # README.md:42-49
        def __init__(self):
            super().__init__()
            self.linear = torch.nn.Linear(3, 6)

        def forward(self, t, z):
            return self.linear(z).view(4, 3, 2)

    class WithTanh(Readme):
        def forward(self, t, z):
            return self.linear(z).view(4, 3, 2).tanh()

    class Transposed(Readme):
        def forward(self, t, z):
            return self.linear(z).view(4, 2, 3).transpose(-1, -2)

    assert solver.linear_field_of(Readme(), z0, 2, t0) is not None
    assert solver.linear_field_of(WithTanh(), z0, 2, t0) is None
    assert solver.linear_field_of(Transposed(), z0, 2, t0) is None
    assert solver.linear_field_of(lambda t, z: z, z0, 2, t0) is None

    # ADVICE r01 (high): modules that agree with their nn.Linear only at a degenerate probe point (t = 0, z = 0)
    class DecaysInTime(Readme):
        def forward(self, t, z):
            return self.linear(z).view(4, 3, 2) * torch.exp(-t)

    class TanhInside(Readme):
        def forward(self, t, z):
            return self.linear(torch.tanh(z)).view(4, 3, 2)

    zeros = torch.zeros(4, 3)
    assert solver.linear_field_of(DecaysInTime(), zeros, 2, [0.0, 1.0]) is None
    assert solver.linear_field_of(TanhInside(), zeros, 2, [0.0, 1.0]) is None
    assert solver.linear_field_of(Readme(), zeros, 2, [0.0, 1.0]) is not None


def test_scalar_host_locator_equals_the_tensor_one():
    """solver._host_locator (numpy scalars + bisect, once per field evaluation of the adaptive / adjoint drivers)
    gives the bits of schedule.locate (torch casts + bucketize) -- also on the knots and one ulp after them."""
    import numpy as np
    from torchcde_b200 import solver
    from torchcde_b200.schedule import locate

    class FakeControl:
        pass

    gen = torch.Generator().manual_seed(3)
    for knot_dtype in (torch.float32, torch.float64):
        for state_dtype in (torch.float32, torch.float64):
            knots = (torch.rand(40, generator=gen, dtype=torch.float64) + 0.01).cumsum(0).to(knot_dtype)
            X = FakeControl()
            orig = (solver._schedule_knots, solver._control_signature)
            solver._schedule_knots = lambda _x: knots
            solver._control_signature = lambda _x: ("cubic", (), 1, 39)
            try:
                where = solver._host_locator(X, state_dtype)
            finally:
                solver._schedule_knots, solver._control_signature = orig
            times = (torch.rand(500, generator=gen, dtype=torch.float64) * 30 - 2).tolist() + knots.tolist()
            times += [float(np.nextafter(np.float32(v), np.float32(1e9))) for v in knots.tolist()]
            for nudge in (0, 1):
                for t in times:
                    tt = torch.tensor(t, dtype=torch.float64).to(state_dtype)
                    if nudge:
                        tt = torch.nextafter(tt, tt + 1)
                    frac, index = locate(knots, tt.to(knot_dtype), 39)
                    assert where(t, nudge) == (int(index), float(frac))


@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
def test_fused_fixed_backward_logic_against_the_generic_adjoint_on_cpu(method):
    """adaptive._fused_fixed_backward (grid, stage times, Runge-Kutta weights of the in-place parameter-gradient
    accumulation, segment bookkeeping) with a torch-CPU stand-in for the stage kernel, against the generic
    adjoint that integrates the packed state (y, a, dL/dW, dL/db) with autograd -- fp64, same algorithm."""
    from torchcde_b200 import adaptive
    torch.manual_seed(0)
    P, H, C = 5, 4, 3
    W = (torch.randn(H * C, H, dtype=torch.float64) / 2).requires_grad_(True)
    b = torch.randn(H * C, dtype=torch.float64).requires_grad_(True)
    y0 = torch.randn(P, H, dtype=torch.float64)
    phase = torch.arange(P, dtype=torch.float64).unsqueeze(1)
    freq = 0.3 * (1 + torch.arange(C, dtype=torch.float64)).unsqueeze(0)

    def dx_at(t):
        return torch.cos(freq * t + phase)                                   # dX/dt, (P, C)

    def vf(t, y):
        g = torch.nn.functional.linear(y, W, b).view(*y.shape[:-1], H, C)
        return (g @ dx_at(t).unsqueeze(-1)).squeeze(-1)

    class Stage:
        roles = ["w", "b"]

        @staticmethod
        def new_grads():
            return [torch.zeros_like(W), torch.zeros_like(b)]

        @staticmethod
        def locate_many(times):
            return [0] * len(times), list(times)                              # the "fraction" carries the time

        @staticmethod
        def segment(*args, **kwargs):
            return None                                                       # exercise the per-stage route

        @staticmethod
        def launch(index, frac, y, a, f_out, vjp_out, gw, gb, f_scale, vjp_scale, grad_scale):
            dx = dx_at(frac)
            w3 = W.detach().view(H, C, H)
            g = torch.nn.functional.linear(y, W.detach(), b.detach()).view(P, H, C)
            f_out.copy_(f_scale * (g * dx.unsqueeze(1)).sum(-1))
            vjp_out.copy_(vjp_scale * torch.einsum("ph,pc,hck->pk", a, dx, w3))
            if gw is not None:
                gw += grad_scale * torch.einsum("ph,pc,pk->hck", a, dx, y).reshape(H * C, H)
            if gb is not None:
                gb += grad_scale * torch.einsum("ph,pc->hc", a, dx).reshape(H * C)

    times = [0.0, 1.3, 2.0]
    step = 0.25

    def forward_solve(y):
        return adaptive.odeint_fixed(vf, y, times, method, step)

    def solve_aug(f, v, ts):
        return adaptive.odeint_fixed(f, v, ts, method, step)

    grads = []
    for fused in (True, False):
        yy = y0.clone().requires_grad_(True)
        W.grad = b.grad = None
        ys = adaptive.solve_with_adjoint(forward_solve, vf, times, solve_aug, yy, (W, b),
                                         (lambda params: Stage) if fused else None, (method, step))
        (ys[1].pow(2).sum() + ys[2].sum()).backward()
        grads.append((yy.grad.clone(), W.grad.clone(), b.grad.clone()))
    for got, want in zip(*grads):
        assert torch.allclose(got, want, rtol=1e-10, atol=1e-12)
