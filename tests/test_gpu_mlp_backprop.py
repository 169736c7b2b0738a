"""cdeint(adjoint=False) of the examples' MLP field with gradients: the three-launch route (stage-dump forward,
tcde_cdeint_fixed_mlp_backward, tcde_mlp_field_param_grads) against fp64 autograd through the oracle's own discrete solve,
and the torch-operator solve wherever the route does not serve.

Reference: ``odeint_port.odeint`` driving ``adaptive_oracle.FuncCDE`` with the MLP as its field (the ``MlpCDE`` of
test_gpu_mlp_field), built from fp64 leaves of W1, b1, W2, b2 on fp64 copies of the kernel's rounded inputs.  Bars: those
of the linear route, dL/dz0 within 1e-5 of each path's scale, every parameter gradient within 2e-4 of its scale.

ReLU kinks: where a stage's pre-activation lies within the fp32 error of the trajectory of zero, the route and the fp64
oracle take opposite sides of the kink and that one path's gradient jumps (DESIGN 5, generic routes).  The rule of the
generic-route tests applies (with a wider KINK_BAR for longer steps): every path within KINK_BAR, all but 1 in 32 within the bar, and the paths over the bar are
run once more with a zero output gradient (their dL/dz0 must then be exactly zero), after which every path and every
parameter gradient must meet the bars.  (Flagging paths whose smallest |W1 z + b1| falls under 1e-4 of the stage's
largest flags almost every path over a whole solve: 981 of 1,000 on F1.)  One case raises b1 so that every
pre-activation stays positive: there no path may be set aside."""
import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port
from test_gpu_discrete_backward import GRAD_BAR, _Calls, _count_loop, _refuse_loop
from test_gpu_fixed_routes import _global_err, _pattern
from test_gpu_mlp_field import (CONTROLS, DEV, F32, METHODS, SCHEDULES, _case, _control, _misaligned_control, _options,
                                _path_err, _variant)
from torchcde_b200 import solver

pytestmark = pytest.mark.gpu
ROUTE = ["tcde_cdeint_fixed_mlp_stages", "tcde_cdeint_fixed_mlp_backward", "tcde_mlp_field_param_grads"]
PARAMS = ("w1", "b1", "w2", "b2")
# a kink's jump is O(dt |W1| |W2|) of the path's scale: 6.8e-2 measured on F6 (the longest steps) with midpoint, 1.0e-2
# with the last output's gradient only; the count (1 in 32) and the bars once kinked paths are set aside are the check
KINK_BAR = 0.1


def _leaves(func):
    l1, l2 = func.linear1, func.linear2
    return {"w1": l1.weight, "b1": l1.bias, "w2": l2.weight, "b2": l2.bias}


def _problem(control, sname, batch=1000, roles="all", shape=None, method="rk4", hidden=32, channels=8, width=128,
             dtype=F32):
    """(X, func, z0 leaf, t, step, the parameter names that want a gradient).  roles: "all", "no_bias", "z0" or one name."""
    n = batch if shape is None else shape[0] * shape[1]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, control, sname, n, bias=roles != "no_bias")
    for name, p in _leaves(func).items():
        if p is not None and roles not in ("all", "no_bias") and name != roles:
            p.requires_grad_(False)
    if shape is not None:
        src = X._rows() if control == "cubic" else X._coeffs
        X = _control(src.view(*shape, *src.shape[1:]), None if X._default_knots else X._t, control)
        z0 = z0.view(*shape, hidden)
    want = [n for n, p in _leaves(func).items() if p is not None and p.requires_grad]
    return X, func, z0.clone().requires_grad_(True), t, step, want


def _run(X, func, z0, t, step, method, g):
    """(outputs, dL/dz0, {name: dL/dparam}) of one cdeint(adjoint=False) call and one backward."""
    leaves = _leaves(func)
    for p in [z0] + list(leaves.values()):
        if p is not None:
            p.grad = None
    out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    out.backward(g)
    return out, z0.grad, {n: p.grad for n, p in leaves.items() if p is not None and p.requires_grad}


class _Oracle:
    """fp64 autograd through odeint_port.odeint on the MLP CDE: ``ys``; ``grads(g)`` = (dL/dz0, {name: dL/dparam})."""

    def __init__(self, X, func, z0, t, step, method, control):
        rows = (X._rows() if control == "cubic" else X._coeffs).detach()
        rows = rows.reshape(-1, rows.size(-2), rows.size(-1)).double()
        leaves = _leaves(func)
        self.names = [n for n in PARAMS if leaves[n] is not None]
        self.p = {n: leaves[n].detach().double().clone().requires_grad_(True) for n in self.names}
        w1, w2 = self.p["w1"], self.p["w2"]
        b1 = self.p.get("b1", torch.zeros(w1.size(0), dtype=torch.float64, device=DEV))
        b2 = self.p.get("b2", torch.zeros(w2.size(0), dtype=torch.float64, device=DEV))
        hidden = w1.size(1)
        self.zz = z0.detach().reshape(-1, hidden).double().clone().requires_grad_(True)

        def g(_t, z):
            return torch.tanh(torch.relu(z @ w1.T + b1) @ w2.T + b2).view(*z.shape[:-1], hidden, -1)

        field = AO.FuncCDE(rows, X._t.detach().cpu(), g, control, z0.dtype)
        with torch.enable_grad():
            self.ys = odeint_port.odeint(field, self.zz, t, method=method, options=_options(step)).movedim(0, 1)

    def grads(self, g):
        got = torch.autograd.grad(self.ys, [self.zz] + [self.p[n] for n in self.names],
                                  g.detach().reshape(self.ys.shape).double(), retain_graph=True)
        return got[0], dict(zip(self.names, got[1:]))


def _check(what, gz, grads, ref_gz, ref_grads):
    err = _path_err(gz.reshape(ref_gz.shape), ref_gz)
    print("mlp backprop dL/dz0 | {}: {:.2e}".format(what, err))
    assert err <= GRAD_BAR["z0"], (what, err)
    for name, got in grads.items():
        err = _global_err(got, ref_grads[name])
        print("mlp backprop dL/d{} | {}: {:.2e}".format(name, what, err))
        assert err <= GRAD_BAR["w"], (what, name, err)


def _compare(what, run, oracle, g):
    """run(g) -> (out, dL/dz0, grads) against the oracle under the kink rule; returns (out, dL/dz0, grads, kinked paths)."""
    out, gz, grads = run(g)
    n_out = g.size(-2)
    ref_gz, ref_grads = oracle.grads(g)
    got = gz.detach().double().reshape(ref_gz.shape)
    errs = ((got - ref_gz).abs().amax(dim=1) / ref_gz.abs().amax(dim=1).clamp_min(1e-300))
    kinked = errs > GRAD_BAR["z0"]
    print("mlp backprop dL/dz0 before setting kinks aside | {}: {:.2e}, {} kinked".format(
        what, float(errs.max()) if errs.numel() else 0.0, int(kinked.sum())))
    assert int(kinked.sum()) <= errs.numel() // 32, (what, int(kinked.sum()))
    assert errs.numel() == 0 or float(errs.max()) <= KINK_BAR, (what, float(errs.max()))
    if kinked.any():
        g = g.clone()
        g.view(-1, n_out, g.size(-1))[kinked] = 0
        out, gz, grads = run(g)
        assert not gz.reshape(-1, gz.size(-1))[kinked].any()
        ref_gz, ref_grads = oracle.grads(g)
    _check(what, gz, grads, ref_gz, ref_grads)
    return out, gz, grads, kinked


def _route_case(monkeypatch, control, sname, method="rk4", batch=1000, roles="all", shape=None, pattern="dense",
                prep=None):
    """Runs the route on a problem and checks it against the oracle; returns (out, dL/dz0, grads, kinked paths)."""
    X, func, z0, t, step, want = _problem(control, sname, batch, roles, shape, method)
    if prep is not None:
        with torch.no_grad():
            prep(func)
    oracle = _Oracle(X, func, z0, t, step, method, control)
    g = _pattern(pattern, tuple(z0.shape[:-1]), t.numel(), 32)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)

    def run(gg):
        calls.names.clear()
        got = _run(X, func, z0, t, step, method, gg)
        # (the module's recognition probe evaluates the control once: tcde_spline_eval)
        assert [n for n in calls.names if n != "tcde_spline_eval"] == (ROUTE if want else ROUTE[:2]), calls.names
        return got

    out, gz, grads, kinked = _compare("{} {} {} {} {} {}".format(control, sname, method, batch, roles, pattern), run,
                                      oracle, g)
    assert sorted(grads) == sorted(want)
    assert _path_err(out.reshape(oracle.ys.shape), oracle.ys) <= 1e-5
    return out, gz, grads, kinked


# ---- 1. the route against the oracle --------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sname", SCHEDULES)
@pytest.mark.parametrize("control", CONTROLS)
def test_route_matches_the_discrete_oracle(control, sname, method, monkeypatch):
    _route_case(monkeypatch, control, sname, method)


@pytest.mark.parametrize("batch", [1, 63, 64, 65, 127, 128, 129, 257])
@pytest.mark.parametrize("control", CONTROLS)
def test_tile_edges(control, batch, monkeypatch):
    _route_case(monkeypatch, control, "F3", batch=batch)


@pytest.mark.parametrize("roles", ["all", "w1", "b2", "z0", "no_bias"])
@pytest.mark.parametrize("control", CONTROLS)
def test_parameter_roles(control, roles, monkeypatch):
    """All parameters, W1 only, b2 only, z0 alone (no kappa dump, no third launch), and both biases absent."""
    _route_case(monkeypatch, control, "F3", batch=129, roles=roles)


@pytest.mark.parametrize("pattern", ["last_output", "odd_paths_zero", "tiny", "huge", "first_output"])
@pytest.mark.parametrize("control", CONTROLS)
def test_gradient_patterns(control, pattern, monkeypatch):
    """The last output only, zero on odd paths (their dL/dz0 exactly zero), scaled by 2^-60 / 2^60, or output 0 only (z0
    itself: dL/dz0 = g[:, 0] bit for bit and every parameter gradient exactly zero)."""
    if pattern == "first_output":
        X, func, z0, t, step, _want = _problem(control, "F3", 129)
        g = _pattern(pattern, (129,), t.numel(), 32)
        _refuse_loop(monkeypatch)
        _out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
        assert torch.equal(gz, g[:, 0])
        assert all(not v.any() for v in grads.values()) and len(grads) == 4
        return
    _out, gz, _grads, _kinked = _route_case(monkeypatch, control, "F3", batch=129, pattern=pattern)
    if pattern == "odd_paths_zero":
        assert not gz[1::2].any()


@pytest.mark.parametrize("control", CONTROLS)
def test_positive_pre_activations_every_path(control, monkeypatch):
    """W1 scaled down and b1 raised so that every pre-activation stays positive: no kink path, the bars on every path."""
    def prep(func):
        func.linear1.weight.mul_(0.1)
        func.linear1.bias.add_(3.0)

    _out, _gz, _grads, kinked = _route_case(monkeypatch, control, "F3", batch=257, prep=prep)
    assert not kinked.any()


def test_a_dead_hidden_unit_gets_exactly_zero_gradient(monkeypatch):
    """A zero row of W1 with a zero bias entry: that unit is relu(0) = 0 at every stage, so its row of dL/dW1 and its
    entry of dL/db1 are exactly zero."""
    def prep(func):
        func.linear1.weight[5].zero_()
        func.linear1.bias[5] = 0.0

    _out, _gz, grads, _kinked = _route_case(monkeypatch, "cubic", "F3", batch=129, prep=prep)
    assert not grads["w1"][5].any() and grads["b1"][5].item() == 0.0


# ---- 2. consistency -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_equal_the_no_grad_call_and_backward_is_deterministic(control, monkeypatch):
    X, func, z0, t, step, _want = _problem(control, "F3", 300)
    g = _pattern("dense", (300,), t.numel(), 32)
    _refuse_loop(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    grads = {n: v.clone() for n, v in grads.items()}
    gz = gz.clone()
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    assert torch.equal(out, plain)
    out2, gz2, grads2 = _run(X, func, z0, t, step, "rk4", g)
    assert torch.equal(out2, out) and torch.equal(gz2, gz)
    assert all(torch.equal(grads2[n], grads[n]) for n in grads)


@pytest.mark.parametrize("control", CONTROLS)
def test_batch_dimensions_are_flattened_bit_for_bit(control, monkeypatch):
    X, func, z0, t, step, _want = _problem(control, "F3", 100)
    g = _pattern("dense", (100,), t.numel(), 32)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    gz, grads = gz.clone(), {n: v.clone() for n, v in grads.items()}
    X4, _f, z4, _t, _s, _w = _problem(control, "F3", shape=(4, 25))
    out4, gz4, grads4 = _run(X4, func, z4, t, step, "rk4", g.view(4, 25, *g.shape[1:]))
    assert out4.shape == (4, 25, t.numel(), 32)
    assert torch.equal(out4.reshape(out.shape), out) and torch.equal(gz4.reshape(gz.shape), gz)
    assert all(torch.equal(grads4[n], grads[n]) for n in grads)


def test_an_empty_batch(monkeypatch):
    X, func, z0, t, step, _want = _problem("cubic", "F3", 0)
    _refuse_loop(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", torch.zeros(0, t.numel(), 32, device=DEV))
    assert out.shape == (0, t.numel(), 32) and gz.shape == (0, 32)
    assert all(not v.any() for v in grads.values())


# ---- 3. what keeps the torch-operator solve -------------------------------------------------------------------------
FALLBACKS = ["fp64", "16x4", "w48", "variant1", "misaligned", "t", "coefficients"]


@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_keep_the_torch_operator_solve(case, monkeypatch):
    hidden, channels = (16, 4) if case == "16x4" else (32, 8)
    width = 48 if case == "w48" else 128
    dtype = torch.float64 if case == "fp64" else F32
    X, func, z0, t, step, _want = _problem("cubic", "F3", 65, hidden=hidden, channels=channels, width=width,
                                           dtype=dtype)
    if case == "misaligned":
        X = _misaligned_control(X, "cubic")
    if case == "t":
        t = t.clone().requires_grad_(True)
    if case == "coefficients":
        X = cde.CubicSpline(X._rows().detach().clone().requires_grad_(True), t=None if X._default_knots else X._t)
    oracle = _Oracle(X, func, z0, t.detach(), step, "rk4", "cubic")
    g = _pattern("dense", (65,), t.numel(), hidden).to(dtype)
    used = _count_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    with _variant(1 if case == "variant1" else 0):
        _compare("fallback " + case, lambda gg: _run(X, func, z0, t, step, "rk4", gg), oracle, g)
    assert used and all(used), case
    assert "tcde_cdeint_fixed_mlp_backward" not in calls.names


@pytest.mark.parametrize("control", CONTROLS)
def test_create_graph_matches_the_torch_operator_solve(control, monkeypatch):
    """A second-order quantity, d ||dL/dz0||^2 / dW2, is the torch-operator solve's: a backward with create_graph
    differentiates that solve on the saved inputs."""
    X, func, z0, t, step, _want = _problem(control, "F3", 65)
    g = _pattern("dense", (65,), t.numel(), 32)

    def second_order():
        z = z0.detach().clone().requires_grad_(True)
        out = cde.cdeint(X, func, z, t, adjoint=False, method="rk4", options=_options(step))
        gz, = torch.autograd.grad(out, z, g, create_graph=True)
        return torch.autograd.grad(gz.pow(2).sum(), func.linear2.weight)[0]

    calls = _Calls(monkeypatch)
    got = second_order()
    assert [n for n in calls.names if n != "tcde_spline_eval"][:1] == ["tcde_cdeint_fixed_mlp_stages"]
    assert "tcde_cdeint_fixed_mlp_backward" not in calls.names
    monkeypatch.setattr(solver, "mlp_backprop", lambda *args: None)
    want = second_order()
    assert got.abs().max() > 0
    assert _global_err(got, want) <= 1e-5


# ---- 4. full scale --------------------------------------------------------------------------------------------------
def test_config3_full_scale(monkeypatch):
    """B = 65,536, L = 256, (H, C, W) = (32, 8, 128), rk4 step 1, output gradients on 256 sampled paths only: the whole
    route against the oracle on those paths (the dumps pass 2^32 bytes, so their offsets must be 64-bit)."""
    gen = torch.Generator().manual_seed(11)
    B, L = 65536, 256
    x = (torch.randn(B, L, 8, generator=gen) / 16).cumsum(1).to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    z0 = torch.randn(B, 32, generator=gen).to(DEV).requires_grad_(True)
    _X, func, _z, _t, _s = _case(32, 8, 128, F32, "cubic", "F3", 1)
    t = torch.tensor([0.0, float(L - 1)], dtype=torch.float64)
    sample = torch.randperm(B, generator=gen)[:256].sort().values.to(DEV)
    oracle = _Oracle(cde.CubicSpline(coeffs[sample]), func, z0[sample], t, 1.0, "rk4", "cubic")
    gs = torch.randn(256, 2, 32, generator=gen).to(DEV)
    X = cde.CubicSpline(coeffs)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    mask = torch.ones(B, dtype=torch.bool, device=DEV)
    mask[sample] = False

    def run(gg):
        calls.names.clear()
        g = torch.zeros(B, 2, 32, device=DEV)
        g[sample] = gg
        _out, gz, grads = _run(X, func, z0, t, 1.0, "rk4", g)
        assert [n for n in calls.names if n != "tcde_spline_eval"] == ROUTE, calls.names
        assert not gz[mask].any()
        return _out, gz[sample], grads

    _compare("config 3, 256 sampled paths", run, oracle, gs)
