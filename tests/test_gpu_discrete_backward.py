"""cdeint(adjoint=False) of the fixed-step linear field with gradients: the three-launch route (stage-dump forward, the
transposed Runge-Kutta recurrence of tcde_cdeint_fixed_linear_backward, one parameter-gradient launch) against fp64
autograd through the oracle's own discrete solve, and the torch-operator solve wherever the route does not serve.

Reference: ``odeint_port.odeint`` driving ``adaptive_oracle.LinearCDE`` built from fp64 leaves of W and b, on fp64 copies
of the kernel's rounded inputs (the continuous adjoint ``fixed_adjoint`` differs from this gradient by the step error,
so it is not the reference here).  Bars: dL/dz0 within 1e-5 of each path's scale, dL/dW and dL/db within 2e-4 of their
scale, the bars of the fused adjoint."""
import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port
from test_gpu_fixed_routes import (CONTROLS, DEV, F32, FIXED_SCHEDULES, _case, _control, _global_err, _misaligned_control,
                                   _options, _path_err, _pattern, _variant)
from torchcde_b200 import _lib, solver

pytestmark = pytest.mark.gpu
GRAD_BAR = {"z0": 1e-5, "w": 2e-4, "b": 2e-4}
ROUTE = ["tcde_cdeint_fixed_linear_stages", "tcde_cdeint_fixed_linear_backward", "tcde_linear_field_param_grads"]
LOOP = "the torch-operator solve"


class _Calls:
    """The names of the library calls made while it is installed."""

    def __init__(self, monkeypatch):
        self.names = []
        real = _lib.call

        def call(name, *args):
            self.names.append(name)
            return real(name, *args)

        monkeypatch.setattr(_lib, "call", call)


def _refuse_loop(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("the torch-operator solve served the kernel route")

    monkeypatch.setattr(solver, "_generic_solve", refuse)


def _count_loop(monkeypatch):
    used = []
    real = solver._generic_solve

    def loop(*args, **kwargs):
        used.append(True)
        return real(*args, **kwargs)

    monkeypatch.setattr(solver, "_generic_solve", loop)
    return used


def _problem(control, sname, batch=1000, roles="wb", shape=None, method="rk4"):
    """(X, func, z0 leaf, t, step, the parameters that want a gradient)."""
    X, func, z0, t, step = _case(32, 8, F32, control, sname, batch if shape is None else shape[0] * shape[1],
                                 bias=roles != "no_bias")
    lin = func.linear
    params = {"w": lin.weight, "b": lin.bias}
    if roles in ("w", "z0"):
        lin.bias.requires_grad_(False)
    if roles in ("b", "z0"):
        lin.weight.requires_grad_(False)
    if shape is not None:
        src = X._rows() if control == "cubic" else X._coeffs
        X = _control(src.view(*shape, *src.shape[1:]), None if X._default_knots else X._t, control)
        z0 = z0.view(*shape, 32)
    want = [n for n, p in params.items() if p is not None and p.requires_grad]
    return X, func, z0.clone().requires_grad_(True), t, step, want


def _run(X, func, z0, t, step, method, g, retain=False):
    """(outputs, dL/dz0, {name: dL/dparam}) of one cdeint(adjoint=False) call and one backward; leaves the leaves clean."""
    lin = func.linear
    for p in (z0, lin.weight, lin.bias):
        if p is not None:
            p.grad = None
    out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    out.backward(g, retain_graph=retain)
    grads = {n: p.grad for n, p in (("w", lin.weight), ("b", lin.bias)) if p is not None and p.requires_grad}
    return out, z0.grad, grads


_oracles = {}


def _oracle(X, func, z0, t, step, method, g, control, key):
    """(outputs, dL/dz0, dL/dW, dL/db) in fp64 by autograd through odeint_port.odeint on LinearCDE."""
    if key not in _oracles:
        rows = (X._rows() if control == "cubic" else X._coeffs).detach()
        rows = rows.reshape(-1, rows.size(-2), rows.size(-1)).double()
        lin = func.linear
        w = lin.weight.detach().double().clone().requires_grad_(True)
        b = (lin.bias.detach().double() if lin.bias is not None else torch.zeros(w.size(0), dtype=torch.float64,
                                                                                 device=DEV)).clone().requires_grad_(True)
        field = AO.LinearCDE(rows, X._t.detach().cpu(), w, b, control, time_dtype=F32)
        zz = z0.detach().reshape(-1, 32).double().clone().requires_grad_(True)
        with torch.enable_grad():
            ys = odeint_port.odeint(field, zz, t, method=method, options=_options(step)).movedim(0, 1)
            gz, gw, gb = torch.autograd.grad(ys, (zz, w, b), g.detach().reshape(ys.shape).double())
        _oracles[key] = (ys.detach(), gz, gw, gb)
    return _oracles[key]


def _check(what, gz, grads, want):
    _ys, wz, ww, wb = want
    err = _path_err(gz.reshape(-1, 32), wz)
    print("discrete backward dL/dz0 | {}: {:.2e}".format(what, err))
    assert err <= GRAD_BAR["z0"], (what, err)
    for name, ref in (("w", ww), ("b", wb)):
        if name in grads:
            err = _global_err(grads[name], ref)
            print("discrete backward dL/d{} | {}: {:.2e}".format(name, what, err))
            assert err <= GRAD_BAR[name], (what, name, err)


def _route_case(monkeypatch, control, sname, method="rk4", batch=1000, roles="wb", shape=None, pattern="dense"):
    X, func, z0, t, step, want = _problem(control, sname, batch, roles, shape, method)
    g = _pattern(pattern, tuple(z0.shape[:-1]), t.numel(), 32)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, method, g)
    assert calls.names == (ROUTE if want else ROUTE[:2]), calls.names
    assert sorted(grads) == sorted(want)
    ref = _oracle(X, func, z0, t, step, method, g, control, (control, sname, method, z0.numel(), roles, pattern))
    return out, gz, grads, ref, g


# ---- 1. the route against the oracle --------------------------------------------------------------------------------
SCHEDULE_CASES = [(c, s, "rk4") for c in CONTROLS for s in FIXED_SCHEDULES]
SCHEDULE_CASES += [(c, s, m) for c in CONTROLS for s in ("F3", "F8") for m in ("midpoint", "euler")]


@pytest.mark.parametrize("control,sname,method", SCHEDULE_CASES)
def test_route_matches_the_discrete_oracle(control, sname, method, monkeypatch):
    out, gz, grads, ref, _g = _route_case(monkeypatch, control, sname, method)
    assert _path_err(out, ref[0]) <= 1e-5
    _check("{} {} {}".format(control, sname, method), gz, grads, ref)


@pytest.mark.parametrize("batch", [1, 63, 64, 65, 129, 1000, (5, 13)])
@pytest.mark.parametrize("control", CONTROLS)
def test_tile_edges_and_batch_shapes(control, batch, monkeypatch):
    shape = batch if isinstance(batch, tuple) else None
    out, gz, grads, ref, _g = _route_case(monkeypatch, control, "F3", batch=1 if shape else batch, shape=shape)
    assert gz.shape == out.shape[:-2] + (32,)
    _check("{} batch {}".format(control, batch), gz, grads, ref)


@pytest.mark.parametrize("roles", ["wb", "w", "b", "no_bias", "z0"])
@pytest.mark.parametrize("control", CONTROLS)
def test_parameter_roles(control, roles, monkeypatch):
    """W and b, W only, b only, a field without bias, and z0 alone (no parameter gradient: no dumps, no third launch)."""
    _out, gz, grads, ref, _g = _route_case(monkeypatch, control, "F3", batch=129, roles=roles)
    _check("{} roles {}".format(control, roles), gz, grads, ref)


@pytest.mark.parametrize("pattern", ["last_output", "odd_paths_zero", "tiny", "huge", "first_output"])
@pytest.mark.parametrize("control", CONTROLS)
def test_gradient_patterns(control, pattern, monkeypatch):
    """The last output only, zero on odd paths (their dL/dz0 exactly zero), scaled by 2^-60 / 2^60, or output 0 only (z0
    itself: dL/dz0 = g[:, 0] bit for bit and no parameter gradient)."""
    _out, gz, grads, ref, g = _route_case(monkeypatch, control, "F3", batch=129, pattern=pattern)
    if pattern == "first_output":
        assert torch.equal(gz, g[:, 0])
        assert not grads["w"].any() and not grads["b"].any()
        return
    if pattern == "odd_paths_zero":
        assert not gz[1::2].any()
    _check("{} pattern {}".format(control, pattern), gz, grads, ref)


@pytest.mark.parametrize("control", CONTROLS)
def test_dl_dz0_against_a_finite_difference_of_the_oracle(control):
    """The outputs are affine in z0, so sum g . (out(z0 + d) - out(z0)) of the fp64 oracle equals sum dL/dz0 . d."""
    X, func, z0, t, step, _want = _problem(control, "F3")
    g = _pattern("dense", (z0.size(0),), t.numel(), 32)
    _out, gz, _grads = _run(X, func, z0, t, step, "rk4", g)
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    field = AO.LinearCDE(rows.double(), X._t.detach().cpu(), func.linear.weight.detach().double(),
                         func.linear.bias.detach().double(), control, time_dtype=F32)
    d = torch.randn(z0.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64).to(DEV)
    with torch.no_grad():
        solve = [odeint_port.odeint(field, z, t, method="rk4", options=_options(step)).movedim(0, 1)
                 for z in (z0.detach().double(), z0.detach().double() + d)]
    lhs = (g.double() * (solve[1] - solve[0])).sum(dim=(1, 2))
    rhs = (gz.double() * d).sum(dim=1)
    scale = (g.double().abs() * (solve[1] - solve[0]).abs()).sum(dim=(1, 2))
    err = ((lhs - rhs).abs() / scale).max().item()
    print("discrete backward finite difference | {}: {:.2e}".format(control, err))
    assert err <= GRAD_BAR["z0"]


# ---- 2. consistency -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sname", ["F3", "F8"])
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_equal_the_no_grad_call_and_backward_is_deterministic(control, sname):
    X, func, z0, t, step, _want = _problem(control, sname)
    g = _pattern("dense", (z0.size(0),), t.numel(), 32)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    assert torch.equal(out, plain)
    out2, gz2, grads2 = _run(X, func, z0, t, step, "rk4", g)
    assert torch.equal(out2, out) and torch.equal(gz2, gz)
    assert all(torch.equal(grads2[n], grads[n]) for n in grads)


@pytest.mark.parametrize("sname,method", [("F3", "rk4"), ("F8", "rk4"), ("F3", "midpoint"), ("F8", "euler")])
@pytest.mark.parametrize("control", CONTROLS)
def test_gradients_agree_with_the_torch_operator_solve(control, sname, method, monkeypatch):
    X, func, z0, t, step, _want = _problem(control, sname, 129, method=method)
    g = _pattern("dense", (z0.size(0),), t.numel(), 32)
    _out, gz, grads = _run(X, func, z0, t, step, method, g)
    grads = {n: v.clone() for n, v in grads.items()}
    monkeypatch.setattr(solver, "fixed_backprop", lambda *args: None)
    used = _count_loop(monkeypatch)
    _out, lz, lgrads = _run(X, func, z0, t, step, method, g)
    assert used == [True]
    _check("vs torch loop {} {} {}".format(control, sname, method), gz, grads, (None, lz, lgrads["w"], lgrads["b"]))


# ---- 3. what keeps the torch-operator solve -------------------------------------------------------------------------
FALLBACKS = ["t", "knots", "coefficients", "fp64", "16x4", "variant1", "misaligned", "memory"]


@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_keep_the_torch_operator_solve(case, monkeypatch):
    hidden, channels, dtype = (16, 4, F32) if case == "16x4" else (32, 8, torch.float64 if case == "fp64" else F32)
    X, func, z0, t, step = _case(hidden, channels, dtype, "cubic", "F3", 65)
    if case == "misaligned":
        X = _misaligned_control(X, "cubic")
    if case == "t":
        t = t.clone().requires_grad_(True)
    if case in ("knots", "coefficients"):
        src = X._rows().detach().clone()
        knots = torch.arange(40, dtype=F32, device=DEV)
        if case == "knots":
            knots.requires_grad_(True)
        else:
            src.requires_grad_(True)
        X = cde.CubicSpline(src, t=knots)
    if case == "memory":
        monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a, **k: (1 << 20, 80 << 30))
    z0 = z0.clone().requires_grad_(True)
    g = torch.randn(65, t.numel(), hidden, generator=torch.Generator().manual_seed(5), dtype=dtype).to(DEV)
    used = _count_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    with _variant(1 if case == "variant1" else 0):
        out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
        out.backward(g)
    assert used == [True], case
    assert "tcde_cdeint_fixed_linear_backward" not in calls.names
    gz = z0.grad.clone()
    # the same solve, the route declined by cdeint itself: the same bits
    monkeypatch.setattr(solver, "fixed_backprop", lambda *args: None)
    z1 = z0.detach().clone().requires_grad_(True)
    with _variant(1 if case == "variant1" else 0):
        out1 = cde.cdeint(X, func, z1, t, adjoint=False, method="rk4", options=_options(step))
        out1.backward(g)
    assert torch.equal(out, out1) and torch.equal(gz, z1.grad)


# ---- 4. create_graph ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("control", CONTROLS)
def test_create_graph_matches_the_torch_operator_solve(control, monkeypatch):
    """A second-order quantity, d ||dL/dz0||^2 / dW, is the torch-operator solve's: the kernels give no higher-order
    derivatives, so a backward with create_graph differentiates that solve on the saved inputs."""
    X, func, z0, t, step, _want = _problem(control, "F3", 65)
    g = _pattern("dense", (65,), t.numel(), 32)

    def second_order():
        z = z0.detach().clone().requires_grad_(True)
        out = cde.cdeint(X, func, z, t, adjoint=False, method="rk4", options=_options(step))
        gz, = torch.autograd.grad(out, z, g, create_graph=True)
        return torch.autograd.grad(gz.pow(2).sum(), func.linear.weight)[0]

    calls = _Calls(monkeypatch)
    got = second_order()
    assert calls.names[:1] == ["tcde_cdeint_fixed_linear_stages"]
    assert "tcde_cdeint_fixed_linear_backward" not in calls.names
    monkeypatch.setattr(solver, "fixed_backprop", lambda *args: None)
    want = second_order()
    assert got.abs().max() > 0
    assert _global_err(got, want) <= 1e-5


# ---- 5. full scale --------------------------------------------------------------------------------------------------
def test_config3_full_scale(monkeypatch):
    """B = 65,536, L = 256, C = 8, H = 32, rk4 step 1: dL/dz0 of the first 1,024 paths against the oracle; the parameter
    gradients of a 4,096-path call against it too."""
    gen = torch.Generator().manual_seed(11)
    B, L = 65536, 256
    x = (torch.randn(B, L, 8, generator=gen) / 16).cumsum(1).to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    z0 = torch.randn(B, 32, generator=gen).to(DEV)
    func = cde.LinearVectorField(32, 8).to(DEV)
    t = torch.tensor([0.0, float(L - 1)], dtype=torch.float64)
    g = torch.randn(B, 2, 32, generator=gen).to(DEV)
    _refuse_loop(monkeypatch)
    for n in (B, 4096):
        X = cde.CubicSpline(coeffs[:n])
        z = z0[:n].clone().requires_grad_(True)
        _out, gz, grads = _run(X, func, z, t, 1.0, "rk4", g[:n])
        m = min(n, 1024)
        Xo = cde.CubicSpline(coeffs[:m])
        ref = _oracle(Xo, func, z0[:m], t, 1.0, "rk4", g[:m], "cubic", ("config3", m))
        err = _path_err(gz[:m], ref[1])
        print("config 3 dL/dz0, {} paths: {:.2e}".format(n, err))
        assert err <= GRAD_BAR["z0"]
        if n == 4096:
            ref = _oracle(X, func, z0[:n], t, 1.0, "rk4", g[:n], "cubic", ("config3", n))
            _check("config 3, 4096 paths", gz, grads, ref)
