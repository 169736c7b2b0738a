"""Anchor the restated fixed-grid stepping (oracle/odeint_port.py) without torchdiffeq.

No torchdiffeq binary exists on this machine, so the stepping arithmetic is "parity
unpinned"; these are the independent checks SURVEY 8(c) lists: analytic solutions of the
reference's own test fixtures, convergence order, and the grid / output-time rules.
"""
import math

import torch

from oracle import cde_oracle as O
from oracle import odeint_port


def _smooth_path(batch, length, channels, seed):
    gen = torch.Generator().manual_seed(seed)
    tau = torch.linspace(0, 1, length, dtype=torch.float64).view(1, length, 1)
    freq = torch.rand(batch, 1, channels, generator=gen, dtype=torch.float64) * 2 + 0.5
    phase = torch.rand(batch, 1, channels, generator=gen, dtype=torch.float64)
    return torch.sin(2 * math.pi * (freq * tau + phase))


def _decay_solve(coeffs, knots, z0, method, h, channels):
    # test_cdeint.py:54-55: func(t, z) = -z expanded over the input channels
    def field(s, z):
        dx = O.cubic_derivative(coeffs, knots, s)
        system = -z.unsqueeze(-1).expand(*z.shape, channels)
        return (system @ dx.unsqueeze(-1)).squeeze(-1)
    t = torch.stack([knots[0], knots[-1]])
    return odeint_port.odeint(field, z0, t, method=method, options={"step_size": h})[-1]


def test_analytic_solution_and_convergence_order():
    x = _smooth_path(3, 9, 2, seed=5)
    coeffs = O.natural_cubic_coeffs(x)
    knots = O.knot_times(9, torch.float64)
    z0 = torch.randn(3, 4, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    # dz = -z * sum_c dX_c  =>  z(T) = z0 * exp(-sum_c (X_c(T) - X_c(0)))
    exact = z0 * torch.exp(-(x[:, -1] - x[:, 0]).sum(-1, keepdim=True))
    for method, order in (("euler", 1), ("midpoint", 2), ("rk4", 4)):
        errs = [(_decay_solve(coeffs, knots, z0, method, h, 2) - exact).abs().max().item()
                for h in (1 / 8, 1 / 16, 1 / 32, 1 / 64)]
        rates = [math.log2(errs[i] / errs[i + 1]) for i in range(3)]
        assert abs(rates[-1] - order) < 0.35, (method, errs, rates)
    assert errs[-1] < 1e-6       # rk4 at h = 1/64


def test_rk4_is_the_three_eighths_rule():
    # y' = t^3 + y is integrated exactly in t by neither tableau, but they differ; check the 3/8 stage times
    seen = []

    def field(s, y):
        seen.append(float(s))
        return y

    odeint_port.odeint(field, torch.ones(1, dtype=torch.float64), torch.tensor([0.0, 3.0], dtype=torch.float64),
                       method="rk4", options={"step_size": 3.0})
    assert seen == [0.0, 1.0, 2.0, 3.0]
    seen.clear()
    odeint_port.odeint(field, torch.ones(1, dtype=torch.float64), torch.tensor([0.0, 1.0], dtype=torch.float64),
                       method="midpoint", options={"step_size": 1.0})
    assert seen == [0.0, 0.5]


def test_grid_construction_and_output_interpolation():
    t = torch.tensor([0.0, 0.7, 2.0, 2.5])
    grid = odeint_port.make_time_grid(t, 1.0)
    assert grid.tolist() == [0.0, 1.0, 2.0, 2.5]               # last entry overwritten by t[-1]
    assert odeint_port.make_time_grid(t, None) is t
    # y' = 1: every method is exact, and outputs inside a step are linear interpolants
    out = odeint_port.odeint(lambda s, y: torch.ones_like(y), torch.zeros(2), t, method="rk4",
                             options={"step_size": 1.0})
    assert torch.allclose(out[:, 0], t)
    assert out.shape == (4, 2)


def test_stage_time_is_cast_to_state_dtype():
    kinds = []
    odeint_port.odeint(lambda s, y: (kinds.append(s.dtype), y)[1], torch.ones(1, dtype=torch.float32),
                       torch.tensor([0.0, 1.0], dtype=torch.float64), method="euler", options={"step_size": 0.5})
    assert set(kinds) == {torch.float32}


def test_reversed_time():
    out = odeint_port.odeint(lambda s, y: torch.ones_like(y), torch.zeros(1, dtype=torch.float64),
                             torch.tensor([1.0, 0.0], dtype=torch.float64), method="rk4", options={"step_size": 0.25})
    assert torch.allclose(out[-1], torch.tensor([-1.0], dtype=torch.float64))


# ---------------------------------------------------------------------------------------------------------------------
# Independent anchors (torchdiffeq is not installed, scripts/probe_torchdiffeq.py):
# a generic explicit Runge-Kutta written from the published Butcher tableaux in numpy fp64 -- no code shared with
# oracle/odeint_port.py -- and scipy's adaptive integrators as ground truth.
_TABLEAUX = {
    # name: (c, A (strictly lower triangular rows), b)
    "euler": ([0.0], [[]], [1.0]),
    "midpoint": ([0.0, 0.5], [[], [0.5]], [0.0, 1.0]),
    # Kutta's 3/8 rule: what torchdiffeq calls "rk4" (rk_common.rk4_alt_step_func)
    "rk4": ([0.0, 1 / 3, 2 / 3, 1.0], [[], [1 / 3], [-1 / 3, 1.0], [1.0, -1.0, 1.0]], [1 / 8, 3 / 8, 3 / 8, 1 / 8]),
}


def _np_field(t, y):
    import numpy as np
    return np.array([math.sin(3 * t) * y[1] - 0.5 * y[0] ** 3, math.cos(t) - y[0] * y[2], 0.3 * y[1] - 0.2 * y[2] + math.sin(t)])


def _butcher_solve(method, t_out, h, y0):
    """Fixed grid t0, t0+h, ... (last point = t_end), outputs by linear interpolation inside the step that covers them."""
    import numpy as np
    c, A, b = _TABLEAUX[method]
    t0, t_end = t_out[0], t_out[-1]
    n = int(math.ceil((t_end - t0) / h + 1))
    grid = [t0 + h * i for i in range(n)]
    if grid[-1] >= t_end:
        grid[-1] = t_end
    else:
        grid.append(t_end)
    outs = [np.array(y0, dtype=np.float64)]
    y = np.array(y0, dtype=np.float64)
    nxt = 1
    for ta, tb in zip(grid[:-1], grid[1:]):
        dt = tb - ta
        ks = []
        for ci, row in zip(c, A):
            yi = y + dt * sum((a * k for a, k in zip(row, ks)), np.zeros_like(y))
            ks.append(_np_field(ta + ci * dt, yi))
        y_new = y + dt * sum(bi * k for bi, k in zip(b, ks))
        while nxt < len(t_out) and tb >= t_out[nxt]:
            w = (t_out[nxt] - ta) / (tb - ta)
            outs.append(y + w * (y_new - y))
            nxt += 1
        y = y_new
    return np.stack(outs)


def test_independent_butcher_tableau_solver_agrees_with_the_port():
    import numpy as np

    def field(t, y):
        t = float(t)
        return torch.stack([math.sin(3 * t) * y[1] - 0.5 * y[0] ** 3, math.cos(t) - y[0] * y[2],
                            0.3 * y[1] - 0.2 * y[2] + math.sin(t)])

    y0 = [0.7, -0.4, 1.1]
    t_out = [0.0, 0.37, 1.0, 2.6, 3.05]
    for method in ("euler", "midpoint", "rk4"):
        for h in (0.25, 0.1):
            want = _butcher_solve(method, t_out, h, y0)
            got = odeint_port.odeint(field, torch.tensor(y0, dtype=torch.float64), torch.tensor(t_out, dtype=torch.float64),
                                     method=method, options={"step_size": h}).numpy()
            assert np.allclose(got, want, rtol=0, atol=1e-12), (method, h, np.abs(got - want).max())


def test_independent_scipy_ground_truth_and_orders():
    import numpy as np
    from scipy.integrate import solve_ivp

    y0 = [0.7, -0.4, 1.1]
    t_out = [0.0, 1.0, 3.0]
    truth = solve_ivp(_np_field, (0.0, 3.0), y0, method="DOP853", rtol=1e-13, atol=1e-13, t_eval=t_out).y.T

    def field(t, y):
        t = float(t)
        return torch.stack([math.sin(3 * t) * y[1] - 0.5 * y[0] ** 3, math.cos(t) - y[0] * y[2],
                            0.3 * y[1] - 0.2 * y[2] + math.sin(t)])

    for method, order in (("euler", 1), ("midpoint", 2), ("rk4", 4)):
        errs = []
        for h in (0.1, 0.05):          # grid points hit every output time: no interpolation error in the way
            got = odeint_port.odeint(field, torch.tensor(y0, dtype=torch.float64), torch.tensor(t_out, dtype=torch.float64),
                                     method=method, options={"step_size": h}).numpy()
            errs.append(np.abs(got - truth).max())
        assert errs[0] < {1: 0.3, 2: 2e-2, 4: 2e-4}[order]
        rate = math.log2(errs[0] / errs[1])
        assert order - 0.4 < rate < order + 0.6, (method, errs, rate)
