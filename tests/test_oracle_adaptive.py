"""The fp64 dopri5 / adjoint oracle (oracle/adaptive_oracle.py) anchored without trusting it: order conditions of its
tableau, SciPy's own Runge-Kutta step, the defining conditions and order of the dense output, a DOP853 solution, and
finite differences of a fine forward solve for the adjoint gradients."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
from scipy.integrate import solve_ivp
from scipy.integrate._ivp.rk import RK45, rk_step

from oracle import adaptive_oracle as AO
from oracle import cde_oracle as O
from oracle import odeint_port


# ------------------------------------------------------------------------------------------------ order conditions
def _conditions(A, b, c):
    """(computed, exact) for the 17 rooted-tree conditions of order <= 5 (Butcher): index = order - 1."""
    A, b, c = np.asarray(A), np.asarray(b), np.asarray(c)
    Ac, Ac2, Ac3 = A @ c, A @ c ** 2, A @ c ** 3
    AAc = A @ Ac
    out = [[(b.sum(), 1)], [(b @ c, 1 / 2)],
           [(b @ c ** 2, 1 / 3), (b @ Ac, 1 / 6)],
           [(b @ c ** 3, 1 / 4), (b @ (c * Ac), 1 / 8), (b @ Ac2, 1 / 12), (b @ AAc, 1 / 24)],
           [(b @ c ** 4, 1 / 5), (b @ (c ** 2 * Ac), 1 / 10), (b @ Ac ** 2, 1 / 20), (b @ (c * Ac2), 1 / 15),
            (b @ (c * AAc), 1 / 30), (b @ Ac3, 1 / 20), (b @ (A @ (c * Ac)), 1 / 40), (b @ (A @ Ac2), 1 / 60),
            (b @ (A @ AAc), 1 / 120)]]
    return out


def _full_tableau():
    """7-stage form: row 6 (the FSAL stage at t + dt) is b5."""
    A = np.zeros((7, 7))
    A[:6, :5] = RK45.A
    A[6, :6] = RK45.B
    c = np.append(RK45.C, 1.0)
    return A, c


def test_tableau_rows_and_source():
    A, c = _full_tableau()
    assert np.allclose(A.sum(axis=1), c, rtol=0, atol=1e-15)
    assert AO.B5 == [float(v) for v in RK45.B] and AO.C == [float(v) for v in RK45.C]
    assert all(float(e) == v for e, v in zip(AO.B5_EXACT[:6], RK45.B))
    # the midpoint weights are SciPy's dense output at x = 1/2
    assert np.allclose(AO.MID, RK45.P @ [1 / 2, 1 / 4, 1 / 8, 1 / 16], rtol=0, atol=1e-16)
    # the error weights are Shampine's pair, not the original Dormand-Prince pair SciPy uses (RK45.E, last weight 1/40)
    assert AO.E[6] == -1 / 60 and RK45.E[6] == 1 / 40
    assert max(abs(a - b) for a, b in zip(AO.E, RK45.E)) > 1e-3


def test_order_conditions():
    A, c = _full_tableau()
    for order, conds in enumerate(_conditions(A, np.append(RK45.B, 0.0), c), 1):
        for got, want in conds:
            assert abs(got - want) < 1e-14, (order, got, want)
    b4 = np.array([float(v) for v in AO.B4_SHAMPINE])
    assert np.allclose(np.array(AO.B5_EXACT, dtype=float) - b4, AO.E, rtol=0, atol=1e-16)
    conds = _conditions(A, b4, c)
    for order in range(4):
        for got, want in conds[order]:
            assert abs(got - want) < 1e-14, (order + 1, got, want)
    # order 5 fails: the error estimate is of order 4 (b4* integrates t^3 exactly, t^4 not)
    assert max(abs(got - want) for got, want in conds[4]) > 1e-4
    nodes = [Fraction(0), Fraction(1, 5), Fraction(3, 10), Fraction(4, 5), Fraction(8, 9), Fraction(1), Fraction(1)]
    assert np.allclose(nodes, c, rtol=0, atol=1e-16)
    for k in range(4):
        assert sum(b * cc ** k for b, cc in zip(AO.B4_SHAMPINE, nodes)) == Fraction(1, k + 1)
    assert sum(b * cc ** 4 for b, cc in zip(AO.B4_SHAMPINE, nodes)) != Fraction(1, 5)


# ------------------------------------------------------------------------------------------------------- one step
def _nonlinear(t, y):
    return np.array([y[1] + 0.3 * np.sin(t), -np.sin(y[0]) - 0.1 * y[1] * y[2], 0.5 * y[0] * y[1] - y[2] ** 2])


def _torch_field(fun):
    return lambda t, y: torch.from_numpy(fun(t, y.numpy()))


@pytest.mark.parametrize("h", [0.7, 0.05, -0.2])
def test_one_attempt_equals_scipy_rk_step(h):
    t, y = 0.4, np.array([0.3, -1.1, 0.8])
    f = _nonlinear(t, y)
    K = np.empty((RK45.n_stages + 1, 3))
    y_new, f_new = rk_step(_nonlinear, t, y, f, h, RK45.A, RK45.B, RK45.C, K)
    res = AO.attempt(_torch_field(_nonlinear), t, h, torch.from_numpy(y), torch.from_numpy(f))
    assert np.allclose(res["y1"].numpy(), y_new, rtol=0, atol=1e-14)
    assert np.allclose(res["ks"][6].numpy(), f_new, rtol=0, atol=1e-14)
    for j in range(7):
        assert np.allclose(res["ks"][j].numpy(), K[j], rtol=0, atol=1e-14), j
    y4 = y + h * sum(float(b) * K[j] for j, b in enumerate(AO.B4_SHAMPINE))
    assert np.allclose(res["err"].numpy(), y_new - y4, rtol=0, atol=1e-14)
    ymid = y + h * K.T @ (RK45.P @ [1 / 2, 1 / 4, 1 / 8, 1 / 16])
    assert np.allclose(res["y_mid"].numpy(), ymid, rtol=0, atol=1e-14)


# --------------------------------------------------------------------------------------------------- dense output
def test_dense_output_conditions_and_order():
    torch.manual_seed(0)
    y0, y1, ym, f0, f1 = (torch.randn(5, dtype=torch.float64) for _ in range(5))
    dt = 0.37
    cf = AO.dense_coefficients(y0, y1, ym, f0, f1, dt)
    deriv = [m * c for m, c in enumerate(cf)][1:]
    assert torch.allclose(AO.dense_evaluate(cf, 0.0), y0, rtol=0, atol=1e-13)
    assert torch.allclose(AO.dense_evaluate(cf, 1.0), y1, rtol=0, atol=1e-13)
    assert torch.allclose(AO.dense_evaluate(cf, 0.5), ym, rtol=0, atol=1e-13)
    assert torch.allclose(deriv[0], dt * f0, rtol=0, atol=1e-13)
    assert torch.allclose(sum(deriv), dt * f1, rtol=0, atol=1e-13)
    # y' = lam y: the dense output inside one step has a local error O(h^5)
    lam, errs = -1.3, []
    for h in (0.2, 0.1, 0.05):
        y = torch.tensor([1.0], dtype=torch.float64)
        field = lambda t, v: lam * v                       # noqa: E731
        res = AO.attempt(field, 0.0, h, y, field(0.0, y))
        cf = AO.dense_coefficients(y, res["y1"], res["y_mid"], res["ks"][0], res["ks"][6], h)
        errs.append(abs(float(AO.dense_evaluate(cf, 0.3)) - math.exp(lam * 0.3 * h)))
    for a, b in zip(errs[:-1], errs[1:]):
        assert 4.5 < math.log2(a / b) < 5.6, errs


# ---------------------------------------------------------------------------------------- a linear CDE test problem
def _cde(kind="cubic", batch=2, length=6, channels=2, hidden=3, seed=0):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / math.sqrt(length)
    knots = O.knot_times(length, torch.float64)
    control = O.hermite_backward_difference_coeffs(x) if kind == "cubic" else x
    weight = torch.randn(hidden * channels, hidden, generator=gen, dtype=torch.float64) / math.sqrt(hidden)
    bias = torch.randn(hidden * channels, generator=gen, dtype=torch.float64) / 2
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64)
    return AO.LinearCDE(control, knots, weight, bias, kind), z0


def test_free_running_driver_against_dop853():
    """On a smooth problem the solution lands within the tolerance of a DOP853 solution at rtol 1e-13."""
    times = [0.0, 1.3, 2.0, 4.75, 5.0]
    y0 = np.array([0.3, -1.1, 0.8])
    rtol, atol = 1e-8, 1e-10
    out, records, _ = AO.solve(_torch_field(_nonlinear), torch.from_numpy(y0), times, rtol, atol)
    assert sum(r.accepted for r in records) > 10
    want = solve_ivp(_nonlinear, (times[0], times[-1]), y0, method="DOP853", rtol=1e-13, atol=1e-13, t_eval=times).y.T
    assert float((np.abs(out.numpy() - want) / (atol + rtol * np.abs(want))).max()) <= 5.0


@pytest.mark.parametrize("kind", ["cubic", "linear"])
def test_free_running_driver_converges_on_a_cde(kind):
    """A spline control is not smooth at its knots (dX/dt jumps for a linear one), so the global error is a larger
    multiple of the tolerance there; it still shrinks in proportion to it.  Reference: DOP853 restarted at every knot."""
    cde, z0 = _cde(kind)
    times = [0.0, 1.3, 2.0, 4.75, 5.0]

    def fun(t, y):
        return cde(t, torch.from_numpy(y).view_as(z0)).reshape(-1).numpy()

    y, ends = z0.reshape(-1).numpy(), {0.0: z0.reshape(-1).numpy()}
    edges = sorted(set([float(k) for k in range(6)] + times))
    for a, b in zip(edges[:-1], edges[1:]):
        inside = (lambda t, v, a=a, b=b: fun(min(max(t, a + 1e-12), b - 1e-12), v))
        y = solve_ivp(inside, (a, b), y, method="DOP853", rtol=1e-13, atol=1e-14).y[:, -1]
        ends[b] = y
    want = torch.from_numpy(np.stack([ends[t] for t in times])).view(len(times), *z0.shape)
    errs = [float((AO.solve(cde, z0, times, rtol, rtol * 1e-2)[0] - want).abs().max()) for rtol in (1e-6, 1e-8, 1e-10)]
    assert errs[0] < 1e-2 and errs[1] < errs[0] / 20 and errs[2] < errs[1] / 20, errs


# ------------------------------------------------------------------------------------------------- adjoint gradients
_TIMES = [0.0, 2.0, 5.0]


def _fd_truth(cde, z0, g, eps=1e-5, step=1 / 64):
    """Central differences of L = sum_i <g_i, z(t_i)> over every entry of (z0, W, b), all perturbed copies in one fine
    fp64 rk4 solve (odeint_port)."""
    theta = [z0, cde.weight, cde.bias]
    sizes = [p.numel() for p in theta]
    n = sum(sizes)
    flat = torch.cat([p.reshape(-1) for p in theta])
    copies = flat.repeat(2 * n, 1)
    idx = torch.arange(n)
    copies[2 * idx, idx] += eps
    copies[2 * idx + 1, idx] -= eps
    zc, wc, bc = torch.split(copies, sizes, dim=1)
    zc = zc.view(2 * n, *z0.shape)
    wc, bc = wc.view(2 * n, *cde.weight.shape), bc.view(2 * n, 1, -1)
    h, c = cde.hidden, cde.channels

    def field(t, z):
        system = (torch.einsum("nik,npk->npi", wc, z) + bc).view(*z.shape, c)
        return (system @ cde.dxdt(float(t)).unsqueeze(-1)).squeeze(-1)

    ys = odeint_port.odeint(field, zc, torch.tensor(_TIMES, dtype=torch.float64), method="rk4",
                            options={"step_size": step})
    loss = torch.einsum("inph,iph->n", ys, g)
    grad = (loss[0::2] - loss[1::2]) / (2 * eps)
    gz, gw, gb = torch.split(grad, sizes)
    return gz.view_as(z0), gw.view_as(cde.weight), gb


def _forward(cde, z0):
    return odeint_port.odeint(cde, z0, torch.tensor(_TIMES, dtype=torch.float64), method="rk4",
                              options={"step_size": 1 / 64})


def _rel_err(got, want):
    return max(float((a - b).abs().max()) / float(b.abs().max()) for a, b in zip(got, want))


@pytest.fixture(scope="module")
def adjoint_problem():
    cde, z0 = _cde("cubic", seed=3)
    g = torch.randn(len(_TIMES), *z0.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    return cde, z0, g, _fd_truth(cde, z0, g), _forward(cde, z0)


@pytest.mark.parametrize("method,order", [("rk4", 4), ("midpoint", 2), ("euler", 1)])
def test_fixed_adjoint_converges_to_finite_differences(adjoint_problem, method, order):
    cde, z0, g, truth, ys = adjoint_problem
    steps = (1 / 4, 1 / 8, 1 / 16) if method != "euler" else (1 / 16, 1 / 32, 1 / 64)
    errs = [_rel_err(AO.fixed_adjoint(cde, ys, g, _TIMES, method, h), truth) for h in steps]
    for a, b in zip(errs[:-1], errs[1:]):
        assert order - 0.3 < math.log2(a / b) < order + 0.6, (method, errs)


def test_paired_adjoint_converges_to_finite_differences(adjoint_problem):
    cde, z0, g, truth, ys = adjoint_problem
    errs = [_rel_err(AO.paired_adjoint(cde, ys, g, _TIMES, rtol, rtol * 1e-2), truth) for rtol in (1e-5, 1e-7, 1e-9)]
    assert errs[0] < 1e-3 and errs[1] < errs[0] / 10 and errs[2] < errs[1] / 10 and errs[2] < 1e-7, errs


# ------------------------------------------------------------------------------------------------------- FuncCDE
def _linear_func_cde(cde):
    """The LinearCDE's field as a FuncCDE of an nn.Linear + view, with W and b as its parameters."""
    lin = torch.nn.Linear(cde.hidden, cde.hidden * cde.channels, dtype=torch.float64)
    with torch.no_grad():
        lin.weight.copy_(cde.weight)
        lin.bias.copy_(cde.bias)
    h = cde.hidden

    def g(t, z):
        return lin(z).view(*z.shape[:-1], h, -1)

    return AO.FuncCDE(cde.control, cde.knots, g, cde.kind, cde.time_dtype, params=[lin.weight, lin.bias])


@pytest.mark.parametrize("kind", ["cubic", "linear"])
def test_func_cde_of_a_linear_module_is_the_linear_cde_bit_for_bit(kind):
    cde, z0 = _cde(kind, seed=4)
    fc = _linear_func_cde(cde)
    a = torch.randn(z0.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    for t in (0.0, 0.7, 2.0, 3.25, 5.0):
        with torch.no_grad():
            assert torch.equal(fc(t, z0), cde(t, z0))
        f, gz, gw, gb = cde.vjp(t, z0, a)
        f2, gz2, (gw2, gb2) = fc.vjp(t, z0, a)
        for got, want in ((f2, f), (gz2, gz), (gw2, gw), (gb2, gb)):
            assert torch.equal(got, want)
        assert fc.locate(t) == cde.locate(t)


@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
def test_generalised_fixed_adjoint_on_a_linear_field(adjoint_problem, method):
    """The parameter-list form of fixed_adjoint on the FuncCDE of a linear module gives LinearCDE's (W, b) form bit for
    bit."""
    cde, z0, g, _truth, ys = adjoint_problem
    gz, gw, gb = AO.fixed_adjoint(cde, ys, g, _TIMES, method, 1 / 4)
    gz2, (gw2, gb2), gt = AO.fixed_adjoint(_linear_func_cde(cde), ys, g, _TIMES, method, 1 / 4)
    assert gt is None
    assert torch.equal(gz2, gz) and torch.equal(gw2, gw) and torch.equal(gb2, gb)


@pytest.mark.parametrize("times", [[2.1, 2.45, 2.9], [2.9, 2.45, 2.1]])
def test_time_channel_of_fixed_adjoint_matches_central_differences(times):
    """dL/dt from the augmented state (the integral of -a^T df/dt, <f, dL/dy> at every output) for a field that reads
    ``t`` itself, against central differences of a fine fp64 solve in every output time, on increasing and decreasing
    t.  The times lie inside one spline interval: across a knot the second derivative of the control jumps, and the fine
    solve's error would then move with its grid by more than the bar."""
    cde, z0 = _cde("cubic", seed=6)
    h = cde.hidden
    v = torch.randn(h * cde.channels, generator=torch.Generator().manual_seed(7), dtype=torch.float64) / 4
    w, b = cde.weight.clone().requires_grad_(True), cde.bias.clone().requires_grad_(True)

    def g(t, z):
        return torch.tanh(torch.nn.functional.linear(z, w, b) + t * v).view(*z.shape[:-1], h, -1)

    fc = AO.FuncCDE(cde.control, cde.knots, g, "cubic", params=[w, b])
    gy = torch.randn(len(times), *z0.shape, generator=torch.Generator().manual_seed(8), dtype=torch.float64)

    def loss(ts):
        # 160 rk4 steps per segment, so that every output is a grid point (no interpolation) and the grid moves with t
        ys, y = [z0], z0
        with torch.no_grad():
            for lo, hi in zip(ts[:-1], ts[1:]):
                grid = torch.linspace(lo, hi, 161, dtype=torch.float64)
                y = odeint_port.odeint(fc, y, grid, method="rk4")[-1]
                ys.append(y)
        ys = torch.stack(ys)
        return float((ys * gy).sum()), ys

    _, ys = loss(times)
    _gz, _gp, gt = AO.fixed_adjoint(fc, ys, gy, times, "rk4", 1 / 64, with_t=True)
    gt = gt.detach()
    eps = 1e-5
    fd = []
    for j in range(len(times)):
        up, down = list(times), list(times)
        up[j] += eps
        down[j] -= eps
        fd.append((loss(up)[0] - loss(down)[0]) / (2 * eps))
    fd = torch.tensor(fd, dtype=torch.float64)
    assert float((gt - fd).abs().max() / fd.abs().max()) < 1e-6, (gt, fd)


def test_paired_segment_quadrature_is_the_integral_of_the_parameter_gradient(adjoint_problem):
    """The quadrature over accepted steps equals integrating dL/dW as a third state with the same Runge-Kutta steps
    (g' does not depend on g), so it agrees with a fine fixed-step adjoint of the same segment."""
    cde, z0, g, truth, ys = adjoint_problem
    seg = AO.PairedSegment(cde).run(_TIMES[2], _TIMES[1], ys[2], g[2], 1e-10, 1e-12)
    assert seg["records"][-1].accepted and abs(seg["steps"][-1]["t"] + seg["steps"][-1]["dt"] + _TIMES[1]) < 1e-12
    _, gw, gb = AO.fixed_adjoint(cde, ys[1:], torch.cat([torch.zeros_like(g[:1]), g[2:]]), _TIMES[1:], "rk4", 1 / 64)
    assert _rel_err((seg["gw"], seg["gb"]), (gw, gb)) < 1e-8
