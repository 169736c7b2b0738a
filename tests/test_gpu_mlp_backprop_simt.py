"""cdeint(adjoint=False) of the examples' MLP field with gradients at the CUDA-core shapes (hidden <= 8 or hidden *
channels <= 32, fp32 and fp64): the three-launch route (stage-dump forward, tcde_cdeint_fixed_mlp_backward,
tcde_mlp_field_param_grads, each on its CUDA-core branch) against fp64 autograd through the oracle's own discrete solve,
and the torch-operator solve wherever the route does not serve.  By default the route serves hidden <= 8 (the HM = 8
kernels); the HM = 32 kernels (hidden 16 / channels 2, hidden 32 / channels 1) run under solve variant 1.

Reference and kink rule: those of test_gpu_mlp_backprop (``_Oracle``, ``_compare``).  Bars: fp32 those of the
tensor-core route (dL/dz0 within 1e-5 of each path's scale, parameters within 2e-4 of their scale), fp64 1e-10 and
1e-9.  In fp64 no path may be set aside as kinked: route and oracle both run fp64, so a real kink would need a
pre-activation within about 1e-15 of zero, and a set-aside path points to an error."""
import copy

import pytest
import torch

import torchcde_b200 as cde
from test_gpu_discrete_backward import GRAD_BAR, _Calls, _count_loop, _refuse_loop
from test_gpu_fixed_routes import _global_err, _pattern
from test_gpu_mlp_backprop import ROUTE, _compare, _Oracle, _problem, _run
from test_gpu_mlp_field import (CONTROLS, DEV, F32, F64, METHODS, SCHEDULES, _case, _misaligned_control,
                                _offset_copy, _options, _path_err, _variant)
from torchcde_b200 import solver

pytestmark = pytest.mark.gpu
BARS = {F32: {"z0": 1e-5, "w": 2e-4, "out": 1e-5}, F64: {"z0": 1e-10, "w": 1e-9, "out": 1e-10}}
SHAPES = [(8, 3, 128), (5, 3, 48), (8, 16, 128), (16, 2, 128), (32, 1, 128), (1, 1, 33)]
DTYPES = {"fp32": F32, "fp64": F64}


def _bars(monkeypatch, dtype):
    for k in ("z0", "w"):
        monkeypatch.setitem(GRAD_BAR, k, BARS[dtype][k])


def _variant_of(hidden):
    return 0 if hidden <= 8 else 1


def _route_case(monkeypatch, control, sname="F3", method="rk4", batch=129, roles="all", shape=(8, 3, 128), dtype=F32,
                pattern="dense", prep=None, batch_shape=None):
    """The route on one problem against the oracle; returns (out, dL/dz0, grads, kinked paths)."""
    hidden, channels, width = shape
    X, func, z0, t, step, want = _problem(control, sname, batch, roles, batch_shape, method, hidden, channels, width,
                                          dtype)
    if prep is not None:
        with torch.no_grad():
            prep(func)
    _bars(monkeypatch, dtype)
    oracle = _Oracle(X, func, z0, t, step, method, control)
    g = _pattern(pattern, tuple(z0.shape[:-1]), t.numel(), hidden).to(dtype)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)

    def run(gg):
        calls.names.clear()
        got = _run(X, func, z0, t, step, method, gg)
        assert [n for n in calls.names if n != "tcde_spline_eval"] == (ROUTE if want else ROUTE[:2]), calls.names
        return got

    what = "{} {} {} {} {} {} {} {}".format(control, sname, method, shape, dtype, batch, roles, pattern)
    with _variant(_variant_of(hidden)):
        out, gz, grads, kinked = _compare(what, run, oracle, g)
    assert sorted(grads) == sorted(want)
    assert dtype != F64 or not kinked.any(), (what, int(kinked.sum()))
    assert out.dtype == dtype and gz.dtype == dtype
    assert _path_err(out.reshape(oracle.ys.shape), oracle.ys) <= BARS[dtype]["out"]
    return out, gz, grads, kinked


# ---- 1. shapes, dtypes, controls, schedules, methods ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "{}x{}w{}".format(*s))
def test_shapes_match_the_discrete_oracle(shape, control, dtype, monkeypatch):
    _route_case(monkeypatch, control, shape=shape, dtype=DTYPES[dtype])


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sname", SCHEDULES)
@pytest.mark.parametrize("control", CONTROLS)
def test_examples_shape_every_schedule_and_method(control, sname, method, monkeypatch):
    _route_case(monkeypatch, control, sname, method, batch=257)


# ---- 2. batch edges, parameter roles, gradient patterns -------------------------------------------------------------
@pytest.mark.parametrize("batch", [1, 127, 128, 129, 257])
@pytest.mark.parametrize("control", CONTROLS)
def test_batch_edges(control, batch, monkeypatch):
    _route_case(monkeypatch, control, batch=batch)


@pytest.mark.parametrize("roles", ["all", "w1", "b2", "z0", "no_bias"])
@pytest.mark.parametrize("control", CONTROLS)
def test_parameter_roles(control, roles, monkeypatch):
    """All parameters, W1 only, b2 only, z0 alone (no kappa dump, no third launch), and both biases absent."""
    _route_case(monkeypatch, control, roles=roles)


@pytest.mark.parametrize("pattern", ["last_output", "odd_paths_zero", "tiny", "huge"])
@pytest.mark.parametrize("control", CONTROLS)
def test_gradient_patterns(control, pattern, monkeypatch):
    _out, gz, _grads, _kinked = _route_case(monkeypatch, control, pattern=pattern)
    if pattern == "odd_paths_zero":
        assert not gz[1::2].any()


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_first_output_gradient_is_z0_itself(dtype, monkeypatch):
    """Output 0 is z0: dL/dz0 = g[:, 0] bit for bit and every parameter gradient exactly zero."""
    dt = DTYPES[dtype]
    X, func, z0, t, step, _want = _problem("cubic", "F3", 129, hidden=8, channels=3, width=128, dtype=dt)
    g = _pattern("first_output", (129,), t.numel(), 8).to(dt)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    _out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    assert [n for n in calls.names if n != "tcde_spline_eval"] == ROUTE
    assert torch.equal(gz, g[:, 0])
    assert all(not v.any() for v in grads.values()) and len(grads) == 4


def test_positive_pre_activations_every_path(monkeypatch):
    """W1 scaled down and b1 raised so that every pre-activation stays positive: no path is set aside."""
    def prep(func):
        func.linear1.weight.mul_(0.1)
        func.linear1.bias.add_(3.0)

    _out, _gz, _grads, kinked = _route_case(monkeypatch, "cubic", batch=257, prep=prep)
    assert not kinked.any()


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_a_dead_hidden_unit_gets_exactly_zero_gradient(dtype, monkeypatch):
    def prep(func):
        func.linear1.weight[5].zero_()
        func.linear1.bias[5] = 0.0

    _out, _gz, grads, _kinked = _route_case(monkeypatch, "cubic", dtype=DTYPES[dtype], prep=prep)
    assert not grads["w1"][5].any() and grads["b1"][5].item() == 0.0


# ---- 3. consistency -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("shape", [(8, 3, 128), (32, 1, 128)], ids=["8x3", "32x1"])
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_equal_the_no_grad_call_and_backward_is_deterministic(control, shape, dtype, monkeypatch):
    dt = DTYPES[dtype]
    X, func, z0, t, step, _want = _problem(control, "F3", 300, hidden=shape[0], channels=shape[1], width=shape[2],
                                           dtype=dt)
    g = _pattern("dense", (300,), t.numel(), shape[0]).to(dt)
    _refuse_loop(monkeypatch)
    with _variant(_variant_of(shape[0])):
        out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
        grads = {n: v.clone() for n, v in grads.items()}
        gz = gz.clone()
        with torch.no_grad():
            plain = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
        out2, gz2, grads2 = _run(X, func, z0, t, step, "rk4", g)
    assert torch.equal(out, plain)
    assert torch.equal(out2, out) and torch.equal(gz2, gz)
    assert all(torch.equal(grads2[n], grads[n]) for n in grads)


def test_batch_dimensions_are_flattened_bit_for_bit(monkeypatch):
    X, func, z0, t, step, _want = _problem("cubic", "F3", 100, hidden=8, channels=3)
    g = _pattern("dense", (100,), t.numel(), 8)
    _refuse_loop(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    gz, grads = gz.clone(), {n: v.clone() for n, v in grads.items()}
    X4, _f, z4, _t, _s, _w = _problem("cubic", "F3", shape=(4, 25), hidden=8, channels=3)
    out4, gz4, grads4 = _run(X4, func, z4, t, step, "rk4", g.view(4, 25, *g.shape[1:]))
    assert out4.shape == (4, 25, t.numel(), 8)
    assert torch.equal(out4.reshape(out.shape), out) and torch.equal(gz4.reshape(gz.shape), gz)
    assert all(torch.equal(grads4[n], grads[n]) for n in grads)


def test_an_empty_batch(monkeypatch):
    X, func, z0, t, step, _want = _problem("cubic", "F3", 0, hidden=8, channels=3)
    _refuse_loop(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", torch.zeros(0, t.numel(), 8, device=DEV))
    assert out.shape == (0, t.numel(), 8) and gz.shape == (0, 8)
    assert all(not v.any() for v in grads.values())


@pytest.mark.parametrize("where", ["control", "z0"])
def test_misaligned_buffers_give_the_aligned_bits(where, monkeypatch):
    X, func, z0, t, step, _want = _problem("cubic", "F3", 129, hidden=8, channels=3)
    g = _pattern("dense", (129,), t.numel(), 8)
    _refuse_loop(monkeypatch)
    out, gz, grads = _run(X, func, z0, t, step, "rk4", g)
    gz, grads = gz.clone(), {n: v.clone() for n, v in grads.items()}
    if where == "control":
        X = _misaligned_control(X, "cubic")
    else:
        z0 = _offset_copy(z0.detach()).requires_grad_(True)
    calls = _Calls(monkeypatch)
    out2, gz2, grads2 = _run(X, func, z0, t, step, "rk4", g)
    assert [n for n in calls.names if n != "tcde_spline_eval"] == ROUTE
    assert torch.equal(out2, out) and torch.equal(gz2, gz)
    assert all(torch.equal(grads2[n], grads[n]) for n in grads)


def test_create_graph_matches_the_torch_operator_solve(monkeypatch):
    X, func, z0, t, step, _want = _problem("cubic", "F3", 65, hidden=8, channels=3)
    g = _pattern("dense", (65,), t.numel(), 8)

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


# ---- 4. what keeps the torch-operator solve -------------------------------------------------------------------------
# w512: (8, 3) at width 512, whose parameter-gradient staging does not fit shared memory (scratch size -1)
REFUSALS = ["16x4", "16x4_variant1", "16x2", "32x1", "w512", "variant4", "variant5", "t", "coefficients"]


@pytest.mark.parametrize("case", REFUSALS)
def test_refusals_keep_the_torch_operator_solve(case, monkeypatch):
    hidden, channels = {"16x4": (16, 4), "16x2": (16, 2), "32x1": (32, 1)}.get(case.split("_")[0], (8, 3))
    X, func, z0, t, step, _want = _problem("cubic", "F3", 65, hidden=hidden, channels=channels,
                                           width=512 if case == "w512" else 128)
    if case == "t":
        t = t.clone().requires_grad_(True)
    if case == "coefficients":
        X = cde.CubicSpline(X._rows().detach().clone().requires_grad_(True), t=None if X._default_knots else X._t)
    variant = {"16x4_variant1": 1, "variant4": 4, "variant5": 5}.get(case, 0)
    oracle = _Oracle(X, func, z0, t.detach(), step, "rk4", "cubic")
    g = _pattern("dense", (65,), t.numel(), hidden)
    used = _count_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    with _variant(variant):
        _compare("refusal " + case, lambda gg: _run(X, func, z0, t, step, "rk4", gg), oracle, g)
    assert used and all(used), case
    assert "tcde_cdeint_fixed_mlp_backward" not in calls.names


# ---- 5. full scale --------------------------------------------------------------------------------------------------
def _full_scale(monkeypatch, hidden, channels, L, seed):
    """B = 65,536 paths of length L, rk4 step 1, output gradients on 256 sampled paths only, against the oracle there."""
    gen = torch.Generator().manual_seed(seed)
    B = 65536
    x = (torch.randn(B, L, channels, generator=gen) / 16).cumsum(1).to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    del x
    z0 = torch.randn(B, hidden, generator=gen).to(DEV).requires_grad_(True)
    _X, func, _z, _t, _s = _case(hidden, channels, 128, F32, "cubic", "F3", 1)
    t = torch.tensor([0.0, float(L - 1)], dtype=torch.float64)
    sample = torch.randperm(B, generator=gen)[:256].sort().values.to(DEV)
    oracle = _Oracle(cde.CubicSpline(coeffs[sample]), func, z0[sample], t, 1.0, "rk4", "cubic")
    gs = torch.randn(256, 2, hidden, generator=gen).to(DEV)
    X = cde.CubicSpline(coeffs)
    _refuse_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    mask = torch.ones(B, dtype=torch.bool, device=DEV)
    mask[sample] = False

    def run(gg):
        calls.names.clear()
        g = torch.zeros(B, 2, hidden, device=DEV)
        g[sample] = gg
        _out, gz, grads = _run(X, func, z0, t, 1.0, "rk4", g)
        assert [n for n in calls.names if n != "tcde_spline_eval"] == ROUTE, calls.names
        assert not gz[mask].any()
        return _out[sample], gz[sample], grads

    with _variant(_variant_of(hidden)):
        _compare("full scale {}x{} L={}".format(hidden, channels, L), run, oracle, gs)


def test_full_scale_examples_shape(monkeypatch):
    _full_scale(monkeypatch, 8, 3, 256, 11)


def test_full_scale_dump_past_2_31_elements(monkeypatch):
    """(32, 1, 128) at L = 260 (solve variant 1): 1,036 stages x 65,536 paths x 32 = 2.17e9 elements per dump, so offsets
    must be 64-bit."""
    _full_scale(monkeypatch, 32, 1, 260, 12)


def test_long_solve_error_is_the_fp32_trajectorys(monkeypatch):
    """Why the fp32 dL/dz0 of the 1,036-stage case above sits near its bar: on its 256 sampled paths (the same inputs),
    the fp64 CUDA-core route meets the fp64 bars on every path against its own fp64 reference, so the kernels compute
    the discrete gradient; and the fp32 torch-operator loop, which rounds the same trajectory in fp32 through other
    operations, is as far from the oracle on the same paths (the same two ReLU-kink paths over 1e-5).  The error is the
    conditioning of a long fp32 solve, not the route's."""
    gen = torch.Generator().manual_seed(12)
    B, L, hidden = 65536, 260, 32
    x = (torch.randn(B, L, 1, generator=gen) / 16).cumsum(1)
    z0_all = torch.randn(B, hidden, generator=gen)
    _X, func, _z, _t, _s = _case(hidden, 1, 128, F32, "cubic", "F3", 1)
    t = torch.tensor([0.0, float(L - 1)], dtype=torch.float64)
    sample = torch.randperm(B, generator=gen)[:256].sort().values
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x[sample].to(DEV))
    z0 = z0_all[sample].to(DEV)
    gs = torch.randn(256, 2, hidden, generator=gen).to(DEV)
    # the oracle takes the state's dtype for its stage times, as the solvers do: fp64 states solve a slightly different
    # discrete problem, with its own reference
    refs = {dt: _Oracle(cde.CubicSpline(coeffs.to(dt)), copy.deepcopy(func).to(dt), z0.to(dt), t, 1.0, "rk4",
                        "cubic").grads(gs.to(dt)) for dt in (F32, F64)}
    calls = _Calls(monkeypatch)

    def errs(gz, grads):
        ref_gz, ref_grads = refs[gz.dtype]
        got = gz.detach().double()
        per_path = (got - ref_gz).abs().amax(1) / ref_gz.abs().amax(1)
        return per_path, {n: _global_err(v, ref_grads[n]) for n, v in grads.items()}

    def route(dtype):
        f = copy.deepcopy(func).to(dtype)
        zz = z0.to(dtype).clone().requires_grad_(True)
        calls.names.clear()
        with _variant(1):
            _out, gz, grads = _run(cde.CubicSpline(coeffs.to(dtype)), f, zz, t, 1.0, "rk4", gs.to(dtype))
        assert [n for n in calls.names if n not in ("tcde_spline_eval", "tcde_set_solve_variant")] == ROUTE, calls.names
        return errs(gz, {"w1": f.linear1.weight.grad, "w2": f.linear2.weight.grad})

    r32, p32 = route(F32)
    r64, p64 = route(F64)
    with monkeypatch.context() as m:
        m.setattr(solver, "mlp_backprop", lambda *args: None)
        f = copy.deepcopy(func)
        zz = z0.clone().requires_grad_(True)
        _out, gz, _g = _run(cde.CubicSpline(coeffs), f, zz, t, 1.0, "rk4", gs)
        l32, q32 = errs(gz, {"w1": f.linear1.weight.grad, "w2": f.linear2.weight.grad})
    for name, e, p in (("route fp32", r32, p32), ("loop fp32", l32, q32), ("route fp64", r64, p64)):
        print("long solve dL/dz0 | {}: worst {:.2e}, median {:.2e}, paths over 1e-5 {}; dW1 {:.2e}, dW2 {:.2e}".format(
            name, float(e.max()), float(e.median()), int((e > 1e-5).sum()), p["w1"], p["w2"]))
    assert float(r64.max()) <= BARS[F64]["z0"] and max(p64.values()) <= BARS[F64]["w"]
    assert float(r32.median()) <= 2 * float(l32.median()) and float(r32.max()) <= 2 * float(l32.max())
    assert all(p32[n] <= 2 * q32[n] for n in p32)
