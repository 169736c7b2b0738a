"""The reversible Heun oracle and the torchsde schedule, on the CPU (no GPU): the oracle's backward against autograd
through its own forward, its convergence order against SciPy, the schedule against the oracle's loop bit for bit, and
the argument errors of cdeint(backend="torchsde")."""
import math

import numpy as np
import pytest
import scipy.integrate
import torch

import torchcde_b200 as cde
from oracle import cde_oracle as O
from oracle import reversible_oracle as R
from torchcde_b200 import schedule

D = torch.float64


def _mlp_field(hidden, gen):
    w1 = (torch.randn(hidden, hidden, generator=gen, dtype=D) / math.sqrt(hidden)).requires_grad_(True)
    b1 = (0.1 * torch.randn(hidden, generator=gen, dtype=D)).requires_grad_(True)
    w2 = (torch.randn(hidden, hidden, generator=gen, dtype=D) / math.sqrt(hidden)).requires_grad_(True)

    def f(t, z):
        return torch.tanh(z @ w1.T + b1 + torch.cos(t)) @ w2.T

    return f, (w1, b1, w2)


def _linear_cubic_field(hidden, channels, length, gen):
    coeffs = (0.3 * torch.randn(3, length - 1, 4 * channels, generator=gen, dtype=D)).requires_grad_(True)
    knots = torch.arange(length, dtype=D)
    weight = (torch.randn(hidden * channels, hidden, generator=gen, dtype=D) / math.sqrt(hidden)).requires_grad_(True)
    bias = (0.1 * torch.randn(hidden * channels, generator=gen, dtype=D)).requires_grad_(True)
    return R.linear_cde_field(coeffs, knots, weight, bias), (weight, bias, coeffs)


def _linear_linear_field(hidden, channels, length, gen):
    slopes = (0.3 * torch.randn(3, length - 1, channels, generator=gen, dtype=D)).requires_grad_(True)
    knots = torch.arange(length, dtype=D)
    weight = (torch.randn(hidden * channels, hidden, generator=gen, dtype=D) / math.sqrt(hidden)).requires_grad_(True)
    bias = (0.1 * torch.randn(hidden * channels, generator=gen, dtype=D)).requires_grad_(True)
    return R.linear_control_field(slopes, knots, weight, bias), (weight, bias, slopes)


@pytest.mark.parametrize("field", ["mlp", "linear_cubic", "linear_linear"])
@pytest.mark.parametrize("checkpoint_every", [None, 4])
def test_oracle_backward_is_the_gradient_of_its_forward(field, checkpoint_every):
    gen = torch.Generator().manual_seed(3)
    hidden = 6
    if field == "mlp":
        f, params = _mlp_field(hidden, gen)
        ts = torch.tensor([0.0, 0.35, 0.4, 1.3, 2.05], dtype=D)
        dt = 0.07
    else:
        make = _linear_cubic_field if field == "linear_cubic" else _linear_linear_field
        f, params = make(hidden, 3, 6, gen)
        ts = torch.tensor([0.0, 1.0, 2.5, 4.6, 5.0], dtype=D)
        dt = 0.3 if field == "linear_cubic" else 0.5           # 0.5: every other step ends on a knot
    y0 = torch.randn(3, hidden, generator=gen, dtype=D).requires_grad_(True)
    g = torch.randn(ts.numel(), 3, hidden, generator=gen, dtype=D)
    ys, _ = R.integrate(f, y0, ts, dt)
    want = torch.autograd.grad((ys * g).sum(), (y0,) + params)
    got_y0, got_p = R.reversible_backward(f, params, y0.detach(), ts, dt, g, checkpoint_every)
    for w, gg in zip(want, (got_y0,) + tuple(got_p)):
        assert (gg - w).abs().max() <= 1e-10 * w.abs().max()


@pytest.mark.parametrize("uneven", [False, True])
def test_oracle_linear_control_is_the_pinned_linear_derivative(uneven):
    """linear_control_field on a control's own slopes against cde_oracle.linear_derivative (pinned to the reference),
    at every knot, between knots and at both ends: same interval rule, same field."""
    gen = torch.Generator().manual_seed(9)
    length, channels, hidden = 7, 3, 4
    knots = torch.arange(length, dtype=D)
    if uneven:
        knots = torch.cat([torch.zeros(1, dtype=D), (0.4 + torch.rand(length - 1, generator=gen, dtype=D)).cumsum(0)])
    x = torch.randn(2, length, channels, generator=gen, dtype=D)
    slopes = O.linear_slopes(x, knots)
    weight = torch.randn(hidden * channels, hidden, generator=gen, dtype=D)
    bias = torch.randn(hidden * channels, generator=gen, dtype=D)
    z = torch.randn(2, hidden, generator=gen, dtype=D)
    f = R.linear_control_field(slopes, knots, weight, bias)
    mids = (knots[1:] + knots[:-1]) / 2
    for t in torch.cat([knots, mids, knots[1:] - 1e-9 * (knots[1:] - knots[:-1])]):
        want_dx = O.linear_derivative(x, knots, t)
        assert torch.equal(R.linear_derivative(slopes, knots, t), want_dx), float(t)
        assert torch.equal(f(t, z), O.linear_field(weight, bias, z, want_dx)), float(t)
    # a knot t_n takes the slope of interval n - 1 (the first knot: interval 0)
    for n in range(1, length):
        assert torch.equal(R.linear_derivative(slopes, knots, knots[n]), slopes[:, n - 1])
    assert torch.equal(R.linear_derivative(slopes, knots, knots[0]), slopes[:, 0])


def test_oracle_converges_at_order_two():
    """y' = (A0 + sin(t) A1) y against SciPy's DOP853: the error ratio over a halving of dt is 4."""
    gen = torch.Generator().manual_seed(5)
    a0 = 0.5 * torch.randn(4, 4, generator=gen, dtype=D)
    a1 = 0.5 * torch.randn(4, 4, generator=gen, dtype=D)
    y0 = torch.randn(1, 4, generator=gen, dtype=D)

    def f(t, y):
        return y @ (a0 + torch.sin(t) * a1).T

    ts = torch.tensor([0.0, 1.0, 2.0], dtype=D)
    sol = scipy.integrate.solve_ivp(lambda t, y: (a0 + math.sin(t) * a1).numpy() @ y, (0.0, 2.0), y0[0].numpy(),
                                    method="DOP853", rtol=1e-13, atol=1e-13, t_eval=[1.0, 2.0])
    want = torch.from_numpy(np.ascontiguousarray(sol.y.T))
    errs = []
    for dt in (0.02, 0.01, 0.005):
        ys, _ = R.integrate(f, y0, ts, dt)
        errs.append((ys[1:, 0] - want).abs().max().item())
    orders = [math.log2(errs[i] / errs[i + 1]) for i in range(2)]
    assert all(1.9 < o < 2.1 for o in orders), orders


@pytest.mark.parametrize("dtype_t", [torch.float32, torch.float64])
@pytest.mark.parametrize("ts,dt", [
    ([0.0, 1.0, 2.0, 3.0], 0.3),                       # dt does not divide the span: clipped last step
    ([0.0, 0.11, 0.12, 0.13, 0.5, 0.7], 0.25),         # several outputs inside one step
    ([0.0, 0.1, 1.7], 1e-2),
    ([0.5, 2.0, 6.75], 1.0),
])
def test_sde_schedule_is_the_oracles_loop(dtype_t, ts, dt):
    t = torch.tensor(ts, dtype=dtype_t)
    knots = torch.arange(8, dtype=torch.float32)
    seen = []

    def f(tt, y):
        seen.append(tt)
        return torch.zeros_like(y)

    _, rec = R.integrate(f, torch.zeros(1, 1, dtype=torch.float32), t, dt)
    s = schedule.build_sde_schedule(t, knots, 7, dt, torch.float32)
    grid = torch.stack(rec["grid"])
    assert s.grid.dtype == dtype_t and torch.equal(s.grid, grid)
    assert torch.equal(torch.stack(seen), grid)                    # the prologue at t_0, then one evaluation per step
    assert s.n_steps == grid.numel() - 1 and s.step_dt.numel() == s.n_steps
    assert torch.equal(s.step_dt, (grid[1:] - grid[:-1]).float())
    assert s.out_step.tolist() == [-1] + [n for n, _, _ in rec["outputs"]]       # output at t_0 is y_0
    w0 = torch.stack([torch.zeros((), dtype=dtype_t)] + [w for _, w, _ in rec["outputs"]]).float()
    w1 = torch.stack([torch.zeros((), dtype=dtype_t)] + [w for _, _, w in rec["outputs"]]).float()
    assert torch.equal(s.out_slope, torch.cat([w1, w0]))
    tk = grid.to(torch.float32)
    index = (torch.bucketize(tk, knots) - 1).clamp(0, 6)
    assert torch.equal(s.stage_index, index.int()) and torch.equal(s.stage_frac, tk - knots[index])


def test_torchsde_argument_errors_need_no_gpu():
    X = cde.CubicSpline(torch.zeros(2, 4, 8))
    f = cde.LinearVectorField(3, 2)
    z0 = torch.zeros(2, 3)
    t = X.interval
    for kw in ({}, {"method": "srk"}, {"method": "midpoint"}):
        with pytest.raises(NotImplementedError, match="torchsde") as info:
            cde.cdeint(X, f, z0, t, backend="torchsde", **kw)
        assert "torchdiffeq" in str(info.value)
    for kw in ({"adaptive": True}, {"bm": object()}, {"options": {}}, {"names": {}},
               {"adjoint_method": "midpoint"}):
        with pytest.raises(NotImplementedError):
            cde.cdeint(X, f, z0, t, backend="torchsde", method="reversible_heun", **kw)
    with pytest.raises(ValueError, match="batch, hidden"):
        cde.cdeint(X, f, torch.zeros(1, 2, 3), t, backend="torchsde", method="reversible_heun")
    with pytest.raises(ValueError, match="strictly increasing"):
        cde.cdeint(X, f, z0, torch.tensor([0.0, 2.0, 1.0]), backend="torchsde", method="reversible_heun")
    with pytest.raises(ValueError, match="strictly increasing"):
        cde.cdeint(X, f, z0, torch.tensor([3.0, 0.0]), backend="torchsde", method="reversible_heun", dt=0.5)
    with pytest.raises(RuntimeError, match="no CPU path"):
        cde.cdeint(X, f, z0, t, backend="torchsde", method="reversible_heun", dt=0.5, rtol=1e-3,
                   adjoint_method="adjoint_reversible_heun")
