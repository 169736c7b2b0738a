"""cdeint(adjoint=False) of the device-controlled dopri5 solve of the linear field with gradients: the recording forward
(tcde_dopri5_linear_record_attempts), the transposed Dormand-Prince recurrence (tcde_dopri5_linear_backward) and one
parameter-gradient launch per record chunk, against fp64 autograd through the oracle's dopri5 replayed on the route's
own accepted steps, and the torch-operator solve wherever the route does not serve.

Once the steps are fixed the paths are independent, so the oracle may replay a subset of them.  Bars: dL/dz0 within 1e-5
of each path's scale, dL/dW and dL/db within 2e-4 of their scale (the bars of the fixed-step route)."""
import math

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from torchcde_b200 import _lib, adaptive, linear_field, solver

DEV = "cuda"
GRAD_BAR = {"z0": 1e-5, "w": 2e-4, "b": 2e-4}
RECORD, BACKWARD = "tcde_dopri5_linear_record_attempts", "tcde_dopri5_linear_backward"
PARAMS, VJP = "tcde_linear_field_param_grads", "tcde_vector_field_linear_vjp"
CONTROLS = ["cubic", "linear"]


def _path_err(got, want):
    got, want = got.detach().double(), want.detach().double().to(got.device)
    dims = tuple(range(1, want.dim()))
    err = (got - want).abs().amax(dim=dims)
    return (err / want.abs().amax(dim=dims).clamp_min(1e-300)).max().item()


def _global_err(got, want):
    got, want = got.detach().double(), want.detach().double().to(got.device)
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


class _Calls:
    """The names of the library calls made while it is installed."""

    def __init__(self, monkeypatch):
        self.names = []
        real = _lib.call

        def call(name, *args):
            self.names.append(name)
            return real(name, *args)

        monkeypatch.setattr(_lib, "call", call)


def _problem(control, batch, length=24, seed=0, roles="wb"):
    """(X, func, z0 leaf, the parameters that want a gradient); ``batch`` an int or a batch shape."""
    shape = batch if isinstance(batch, tuple) else (batch,)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(*shape, length, 8, generator=gen, device=DEV).cumsum(-2) / math.sqrt(length)
    z0 = torch.randn(*shape, 32, generator=gen, device=DEV)
    torch.manual_seed(seed + 1)
    func = cde.LinearVectorField(32, 8, bias=roles != "no_bias").to(DEV)
    lin = func.linear
    if roles in ("w", "z0"):
        lin.bias.requires_grad_(False)
    if roles in ("b", "z0"):
        lin.weight.requires_grad_(False)
    with torch.no_grad():
        X = cde.LinearInterpolation(x) if control == "linear" else \
            cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    want = [n for n, p in (("w", lin.weight), ("b", lin.bias)) if p is not None and p.requires_grad]
    return X, func, z0.requires_grad_(True), want


def _run(X, func, z0, t, g, **kwargs):
    """(outputs, dL/dz0, {name: dL/dparam}, stats) of one cdeint(adjoint=False) call and one backward."""
    lin = func.linear
    for p in (z0, lin.weight, lin.bias):
        if p is not None:
            p.grad = None
    out = cde.cdeint(X, func, z0, t, adjoint=False, **kwargs)
    stats = dict(cde.cdeint.last_stats)
    out.backward(g)
    grads = {n: p.grad.clone() for n, p in (("w", lin.weight), ("b", lin.bias)) if p is not None and p.requires_grad}
    return out.detach(), z0.grad.clone(), grads, stats


def _oracle(X, func, z0, t, g, control, steps, m=None):
    """(outputs, dL/dz0, dL/dW, dL/db) of the first ``m`` paths in fp64 by autograd through adaptive_oracle.solve on
    LinearCDE, replaying the accepted ``steps`` (in the solve's time: -t for a decreasing t)."""
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    rows = rows.reshape(-1, rows.size(-2), rows.size(-1))
    zz = z0.detach().reshape(-1, 32)
    gg = g.detach().reshape(zz.size(0), -1, 32)
    if m is not None:
        rows, zz, gg = rows[:m], zz[:m], gg[:m]
    lin = func.linear
    w = lin.weight.detach().double().clone().requires_grad_(True)
    b = (lin.bias.detach().double() if lin.bias is not None else
         torch.zeros(w.size(0), dtype=torch.float64, device=DEV)).clone().requires_grad_(True)
    cde_field = AO.LinearCDE(rows.double(), X._t.detach().cpu(), w, b, control, time_dtype=torch.float32)
    times = [float(v) for v in t.tolist()]
    field = cde_field
    if times[0] > times[-1]:
        times = [-v for v in times]

        def field(s, z):
            return -cde_field(-s, z)
    zz = zz.double().clone().requires_grad_(True)
    with torch.enable_grad():
        ys, _records, _dt = AO.solve(field, zz, times, 1e-4, 1e-6, replay=[(s, d, True) for s, d in steps])
        ys = ys.movedim(0, 1)
        gz, gw, gb = torch.autograd.grad(ys, (zz, w, b), gg.double())
    return ys.detach(), gz, gw, gb


def _check(what, gz, grads, want, m=None):
    _ys, wz, ww, wb = want
    err = _path_err(gz.reshape(-1, 32)[:m], wz)
    print("dopri5 backprop dL/dz0 | {}: {:.2e}".format(what, err))
    assert err <= GRAD_BAR["z0"], (what, err)
    for name, ref in (("w", ww), ("b", wb)):
        if name in grads:
            err = _global_err(grads[name], ref)
            print("dopri5 backprop dL/d{} | {}: {:.2e}".format(name, what, err))
            assert err <= GRAD_BAR[name], (what, name, err)


def _refuse_host_driver(monkeypatch):
    def refuse(*args, **kwargs):
        if kwargs.get("steps") is None:
            raise AssertionError("the torch-operator dopri5 served the kernel route")
        return real(*args, **kwargs)

    real = adaptive.odeint_dopri5
    monkeypatch.setattr(adaptive, "odeint_dopri5", refuse)


def _route_case(monkeypatch, control, t, batch=129, roles="wb", g=None, **kwargs):
    X, func, z0, want = _problem(control, batch, roles=roles)
    if g is None:
        g = torch.randn(*z0.shape[:-1], t.numel(), 32, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    _refuse_host_driver(monkeypatch)
    calls = _Calls(monkeypatch)
    out, gz, grads, stats = _run(X, func, z0, t, g, **kwargs)
    assert RECORD in calls.names and BACKWARD in calls.names and calls.names[-1] == VJP, calls.names
    assert (PARAMS in calls.names) == bool(want), calls.names
    assert sorted(grads) == sorted(want)
    ref = _oracle(X, func, z0, t, g, control, stats["steps"])
    assert _path_err(out.reshape(-1, t.numel(), 32), ref[0]) <= 1e-4
    return X, func, z0, out, gz, grads, stats, ref, g


# ---- 1. the route against the oracle --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["dense", "decreasing", "first_step", "t0_only"])
@pytest.mark.parametrize("control", CONTROLS)
def test_route_matches_the_replayed_oracle(control, case, monkeypatch):
    kwargs = {"options": {"first_step": 0.05}} if case == "first_step" else {}
    t = torch.tensor([23.0, 9.5, 3.25, 0.0] if case == "decreasing" else [0.0, 0.7, 5.3, 11.0, 23.0],
                     dtype=torch.float64)
    g = None
    if case == "t0_only":
        g = torch.zeros(129, t.numel(), 32, device=DEV)
        g[:, 0] = torch.randn(129, 32, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    _X, _f, _z0, _out, gz, grads, stats, ref, g = _route_case(monkeypatch, control, t, g=g, **kwargs)
    assert stats["n_accepted"] == len(stats["steps"]) >= 3
    if case == "t0_only":
        # output 0 is z0 itself: dL/dz0 = g[:, 0] bit for bit, no parameter gradient
        assert torch.equal(gz, g[:, 0])
        assert not grads["w"].any() and not grads["b"].any()
        return
    if case == "first_step":
        assert stats["steps"][0][1] == 0.05
    _check("{} {}".format(control, case), gz, grads, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_inside_one_step_and_on_a_step_end(control, monkeypatch):
    """The accepted steps do not depend on the output times between t0 and the end: place three outputs inside one step
    and one exactly on a step's end."""
    X, func, z0, _want = _problem(control, 129)
    cde.cdeint(X, func, z0, torch.tensor([0.0, 23.0], dtype=torch.float64), adjoint=False)
    steps = cde.cdeint.last_stats["steps"]
    (ta, da), (tb, db) = max(steps[:-1], key=lambda s: s[1]), steps[len(steps) // 2]
    t = torch.tensor(sorted({0.0, ta + 0.2 * da, ta + 0.5 * da, ta + 0.9 * da, tb + db, 23.0}), dtype=torch.float64)
    _X, _f, _z0, _out, gz, grads, stats, ref, _g = _route_case(monkeypatch, control, t)
    assert stats["steps"] == steps
    _check("{} outputs inside a step / on a step end".format(control), gz, grads, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 127, 128, 129, 1000, (5, 13)])
def test_tile_edges_and_batch_shapes(batch, monkeypatch):
    t = torch.tensor([0.0, 7.0, 23.0], dtype=torch.float64)
    _X, _f, z0, out, gz, grads, _stats, ref, _g = _route_case(monkeypatch, "cubic", t, batch=batch)
    assert gz.shape == z0.shape and out.shape == z0.shape[:-1] + (3, 32)
    _check("batch {}".format(batch), gz, grads, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("roles", ["wb", "w", "b", "no_bias", "z0"])
def test_parameter_roles(roles, monkeypatch):
    """W and b, W only, b only, a field without bias, and z0 alone (no record of stage inputs, no parameter launch)."""
    t = torch.tensor([0.0, 7.0, 23.0], dtype=torch.float64)
    _X, _f, _z0, _out, gz, grads, _stats, ref, _g = _route_case(monkeypatch, "linear", t, roles=roles)
    _check("roles {}".format(roles), gz, grads, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("control", CONTROLS)
def test_record_overflows_into_new_chunks(control, monkeypatch):
    """Three slots per chunk: the device pauses and resumes several times, the backward runs chunk by chunk, and the outputs
    and step counts still equal the no-grad call's."""
    monkeypatch.setattr(linear_field.Dopri5Backprop, "slots", 3)
    t = torch.tensor([0.0, 5.0, 23.0], dtype=torch.float64)
    X, func, z0, out, gz, grads, stats, ref, _g = _route_case(monkeypatch, control, t)
    n_chunks = -(-stats["n_accepted"] // 3)
    assert n_chunks >= 3
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False)
        plain_stats = cde.cdeint.last_stats
    assert torch.equal(out, plain)
    assert (plain_stats["n_accepted"], plain_stats["n_rejected"]) == (stats["n_accepted"], stats["n_rejected"])
    _check("{} {} chunks".format(control, n_chunks), gz, grads, ref)


# ---- 2. bits ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("decreasing", [False, True])
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_equal_the_no_grad_call_and_backward_is_deterministic(control, decreasing):
    X, func, z0, _want = _problem(control, 1000)
    t = torch.tensor([23.0, 11.0, 0.0] if decreasing else [0.0, 11.0, 23.0], dtype=torch.float64)
    g = torch.randn(1000, 3, 32, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV)
    out, gz, grads, stats = _run(X, func, z0, t, g)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False)
        plain_stats = dict(cde.cdeint.last_stats)
    assert torch.equal(out, plain)
    assert (plain_stats["n_accepted"], plain_stats["n_rejected"]) == (stats["n_accepted"], stats["n_rejected"])
    assert plain_stats["device_controlled"] and stats["device_controlled"]
    out2, gz2, grads2, _stats2 = _run(X, func, z0, t, g)
    assert torch.equal(out2, out) and torch.equal(gz2, gz)
    assert all(torch.equal(grads2[n], grads[n]) for n in grads)


@pytest.mark.gpu
def test_backward_releases_the_record_while_the_outputs_live():
    """The record (the stage inputs of every accepted step) is saved for the backward, not held by the graph node: after
    out.backward(g) it is freed although ``out`` is still bound -- as in a training loop, where the last step's outputs
    are alive while the next forward runs.  retain_graph keeps it for a second backward."""
    X, func, z0, _want = _problem("cubic", 4096)
    t = torch.tensor([0.0, 23.0], dtype=torch.float64)
    g = torch.randn(4096, 2, 32, generator=torch.Generator(device=DEV).manual_seed(13), device=DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    out = cde.cdeint(X, func, z0, t, adjoint=False)
    record = cde.cdeint.last_stats["n_accepted"] * 6 * 4096 * 32 * 4
    assert torch.cuda.memory_allocated() - before >= record
    out.backward(g)
    torch.cuda.synchronize()
    left = torch.cuda.memory_allocated() - before
    # what may stay: out, the gradients of z0, W and b, and the parameter-gradient kernel's cached scratch
    allowed = out.numel() * 4 + z0.numel() * 4 + (256 * 32 + 256) * 4 + (16 << 20)
    print("record {:.1f} MiB, left after the backward {:.1f} MiB".format(record / 2 ** 20, left / 2 ** 20))
    assert record > 4 * allowed and left <= allowed, (left, allowed, record)
    gz = z0.grad.clone()
    z0.grad = None
    out = cde.cdeint(X, func, z0, t, adjoint=False)
    out.backward(g, retain_graph=True)
    out.backward(g)
    assert torch.equal(z0.grad, 2 * gz)


@pytest.mark.gpu
def test_parameter_gradients_over_many_chunks_at_a_large_batch(monkeypatch):
    """4,096 paths, length 64, eight slots per chunk: dL/dW and dL/db accumulate over many chunks, against the oracle over
    every path."""
    monkeypatch.setattr(linear_field.Dopri5Backprop, "slots", 8)
    t = torch.tensor([0.0, 21.5, 63.0], dtype=torch.float64)
    X, func, z0, _want = _problem("cubic", 4096, length=64, seed=5)
    g = torch.randn(4096, 3, 32, generator=torch.Generator(device=DEV).manual_seed(17), device=DEV)
    _out, gz, grads, stats = _run(X, func, z0, t, g)
    assert stats["n_accepted"] > 4 * 8
    ref = _oracle(X, func, z0, t, g, "cubic", stats["steps"])
    _check("4,096 paths, {} chunks".format(-(-stats["n_accepted"] // 8)), gz, grads, ref)


# ---- 3. create_graph --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_create_graph_differentiates_the_replay_of_the_recorded_steps(monkeypatch):
    X, func, z0, _want = _problem("cubic", 65)
    t = torch.tensor([0.0, 9.0, 23.0], dtype=torch.float64)
    g = torch.randn(65, 3, 32, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV)

    def second_order(solve):
        z = z0.detach().clone().requires_grad_(True)
        gz, = torch.autograd.grad(solve(z), z, g, create_graph=True)
        return torch.autograd.grad(gz.pow(2).sum(), func.linear.weight)[0]

    calls = _Calls(monkeypatch)
    got = second_order(lambda z: cde.cdeint(X, func, z, t, adjoint=False))
    steps = cde.cdeint.last_stats["steps"]
    assert calls.names.count(RECORD) >= 1 and BACKWARD not in calls.names
    field = solver._torch_field(X, func, False, True, z0)
    want = second_order(lambda z: adaptive.odeint_dopri5(field, z, [0.0, 9.0, 23.0], 1e-4, 1e-6, steps=steps)[0]
                        .movedim(0, 1))
    assert got.abs().max() > 0
    assert _global_err(got, want) <= 1e-6


# ---- 4. what keeps the torch-operator solve -------------------------------------------------------------------------
FALLBACKS = ["t", "knots", "coefficients", "fp64", "16x4", "jump_t", "memory"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_keep_the_torch_operator_solve(case, monkeypatch):
    hidden, channels = (16, 4) if case == "16x4" else (32, 8)
    dtype = torch.float64 if case == "fp64" else torch.float32
    gen = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(65, 12, channels, generator=gen, device=DEV, dtype=dtype).cumsum(1) / 4
    z0 = torch.randn(65, hidden, generator=gen, device=DEV, dtype=dtype)
    torch.manual_seed(4)
    func = cde.LinearVectorField(hidden, channels).to(device=DEV, dtype=dtype)
    t = torch.tensor([0.0, 4.0, 11.0], dtype=torch.float64)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    knots = None
    if case == "knots":
        knots = torch.arange(12, dtype=dtype, device=DEV).requires_grad_(True)
    if case == "coefficients":
        coeffs = coeffs.clone().requires_grad_(True)
    if case == "t":
        t = t.clone().requires_grad_(True)
    kwargs = {"options": {"jump_t": torch.arange(12.0)}} if case == "jump_t" else {}
    if case == "memory":
        monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a, **k: (1 << 20, 80 << 30))
    g = torch.randn(65, 3, hidden, generator=gen, device=DEV, dtype=dtype)

    def run():
        X = cde.CubicSpline(coeffs, t=knots)
        z = z0.clone().requires_grad_(True)
        out = cde.cdeint(X, func, z, t, adjoint=False, **kwargs)
        out.backward(g)
        return out.detach(), z.grad

    calls = _Calls(monkeypatch)
    out, gz = run()
    names = list(calls.names)
    assert RECORD not in names and BACKWARD not in names, case
    # the same solve with the route declined by cdeint itself: the same library calls, the same bits
    monkeypatch.setattr(solver, "dopri5_backprop", lambda *args: None)
    calls.names.clear()
    out1, gz1 = run()
    assert calls.names == names, case
    assert torch.equal(out, out1) and torch.equal(gz, gz1), case


# ---- 5. full scale ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_scale(monkeypatch):
    """B = 65,536, L = 256, C = 8, H = 32 with cdeint's default tolerances: dL/dz0 of the first 1,024 paths against the
    oracle replaying the route's steps."""
    B, L = 65536, 256
    gen = torch.Generator(device=DEV).manual_seed(11)
    x = (torch.randn(B, L, 8, generator=gen, device=DEV) / 16).cumsum(1)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    z0 = torch.randn(B, 32, generator=gen, device=DEV).requires_grad_(True)
    torch.manual_seed(12)
    func = cde.LinearVectorField(32, 8).to(DEV)
    t = torch.tensor([0.0, float(L - 1)], dtype=torch.float64)
    g = torch.randn(B, 2, 32, generator=gen, device=DEV)
    _refuse_host_driver(monkeypatch)
    _out, gz, grads, stats = _run(X, func, z0, t, g)
    print("full scale: {} accepted, {} rejected".format(stats["n_accepted"], stats["n_rejected"]))
    assert all(torch.isfinite(v).all() for v in grads.values())
    ref = _oracle(X, func, z0, t, g, "cubic", stats["steps"], m=1024)
    err = _path_err(gz[:1024], ref[1])
    print("full scale dL/dz0, 1,024 paths: {:.2e}".format(err))
    assert err <= GRAD_BAR["z0"]


# ---- 6. the host tables (no GPU) ------------------------------------------------------------------------------------
def test_injection_weights_equal_autograd_of_the_dense_output():
    """Each output's weights on (y_n, y_{n+1}, k1, k3, k4, k5, k6, k7) equal fp64 autograd of Dopri5._fit / _evaluate with
    y_mid = y_n + dt sum_j c_mid[j] k_j."""
    steps = [(0.0, 0.3), (0.3, 0.45), (0.75, 1.5)]
    times = [0.0, 0.1, 0.3, 0.31, 0.5, 0.75, 2.0, 2.25]
    tables = adaptive.dopri5_backward_tables(steps, times)
    assert tables["inj_range"].tolist() == [0, 2, 5, 7]
    assert tables["inj_out"].tolist() == [1, 2, 3, 4, 5, 6, 7]
    for n, (t_lo, dt) in enumerate(steps):
        for e in range(int(tables["inj_range"][n]), int(tables["inj_range"][n + 1])):
            y0, y1, *ks = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (0.3, -1.1, 0.7, 0.2, -0.4,
                                                                                              1.3, 0.9, -0.6, 0.5)]
            y_mid = y0 + sum(c * dt * k for c, k in zip(adaptive._C_MID, ks))
            coeff = adaptive.Dopri5._fit(y0, y1, y_mid, ks[0], ks[6], dt)
            out = adaptive.Dopri5._evaluate(coeff, t_lo, t_lo + dt, times[int(tables["inj_out"][e])])
            want = torch.autograd.grad(out, (y0, y1, ks[0], ks[2], ks[3], ks[4], ks[5], ks[6]), allow_unused=True)
            want = torch.stack([w if w is not None else torch.zeros((), dtype=torch.float64) for w in want])
            assert torch.allclose(tables["inj_w"][e].double(), want, rtol=1e-6, atol=1e-6), (n, e)
    coef = tables["coef"].view(-1, 6, 6)
    assert coef[1, 5, 5].item() == torch.tensor((11 / 84) * 0.45, dtype=torch.float32).item()
