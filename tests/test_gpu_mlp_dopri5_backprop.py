"""cdeint(adjoint=False) of the host-driven dopri5 solve of the examples' MLP field with gradients: the recording forward
(``adaptive.Dopri5`` with the field of the call without gradients, its hooks filling the record), one launch of
``tcde_dopri5_mlp_backward`` (the transposed Dormand-Prince recurrence, J^T at the recorded inputs) and one
``tcde_mlp_field_param_grads`` call per record chunk, against fp64 autograd through the oracle's dopri5 replayed on the
route's own accepted steps; and the torch-operator dopri5 wherever the route does not serve.

Every case proves its route: the library calls are recorded, the backward runs with ``torch.autograd.grad`` patched to
raise, and the outputs and step counts are those of the same call under ``no_grad``, bit for bit.  Bars (those of the MLP
adjoint tests): fp32 dL/dz0 within 1e-5 of each path's scale (the relu-kink rule: all but 1 path in 32, every path within
KINK_BAR) and dL/dtheta within 2e-4 of its scale; fp64 1e-10 for both, no path set aside."""
import copy

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from test_gpu_generic_routes import KINK_BAR, SoftplusMLP, _control, _global_err, _inputs
from test_gpu_mlp_adjoint import _check_paths, _func, _report
from test_gpu_mlp_field import _variant
from torchcde_b200 import _lib, adaptive, mlp_field, solver

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
CONTROLS = ["cubic", "linear"]
BACKWARD, PARAMS = "tcde_dopri5_mlp_backward", "tcde_mlp_field_param_grads"
BARS = {F32: (1e-5, 2e-4), F64: (1e-10, 1e-10)}
RTOL, ATOL = 1e-4, 1e-6


def _problem(shape, dtype, control, batch, bias=True, length=None):
    """(X, func, z0) on ``batch`` paths (an int or a batch shape) of the generic-routes inputs (paths repeated past 1000)."""
    hidden, channels, width = shape
    dims = batch if isinstance(batch, tuple) else (batch,)
    n = 1
    for d in dims:
        n *= d
    if length is None:
        x, knots, coeffs, z0 = _inputs(channels, hidden, False)
    else:
        x, knots, coeffs, z0 = _inputs(channels, hidden, False, paths=min(n, 1000), length=length)
    reps = -(-n // x.size(0))
    src = (coeffs if control == "cubic" else x).repeat(reps, 1, 1)[:n].to(dtype)
    src = src.reshape(*dims, src.size(-2), src.size(-1))
    return _control(src, None, control), _func(channels, hidden, width, dtype, bias), \
        z0.repeat(reps, 1)[:n].to(dtype).reshape(*dims, hidden)


def _fc(X, func, control, dtype, m=None):
    """FuncCDE on fp64 copies of the first ``m`` paths' control rows and of the module."""
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    rows = rows.reshape(-1, rows.size(-2), rows.size(-1))[:m].double()
    f64 = copy.deepcopy(func).double()
    for q in f64.parameters():
        q.requires_grad_(True)
    return AO.FuncCDE(rows, X._t.detach().cpu(), f64, control, time_dtype=dtype, params=list(f64.parameters()))


def _after(t, dtype):
    """The first time after ``t`` in the state dtype: where the driver takes the slope after a jump point."""
    tt = torch.tensor(t, dtype=dtype)
    return float(torch.nextafter(tt, tt + 1))


def _oracle(X, func, control, dtype, z0, t_list, g, steps, jumps=(), m=None):
    """(outputs, dL/dz0, [dL/dtheta]) of the first ``m`` paths by fp64 autograd through adaptive_oracle.solve replaying
    the accepted ``steps`` (in -t for a decreasing t); with ``jumps``, segment by segment between them, the slope after a
    jump taken just after it."""
    fc = _fc(X, func, control, dtype, m)
    hidden = z0.size(-1)
    zz = z0.detach().reshape(-1, hidden)[:m].double().clone().requires_grad_(True)
    gg = g.detach().reshape(-1, len(t_list), hidden)[:m].double().to(DEV)
    times, field = list(t_list), fc
    if times[0] > times[-1]:
        times = [-v for v in times]

        def field(s, z):
            return -fc(-s, z)
    replay = [(s, d, True) for s, d in steps]
    with torch.enable_grad():
        if not jumps:
            ys = AO.solve(field, zz, times, RTOL, ATOL, replay=replay)[0]
        else:
            y, outs = zz, [zz]
            edges = sorted(set([times[0], times[-1]] + [j for j in jumps if times[0] < j < times[-1]]))
            for lo, hi in zip(edges[:-1], edges[1:]):
                seg = [r for r in replay if lo <= r[0] < hi]
                inner = [v for v in times if lo < v < hi]
                start = (lambda s, v, lo=lo: field(_after(lo, dtype) if s == lo else s, v)) if lo in jumps else field
                want = AO.solve(start, y, [lo] + inner + [hi], RTOL, ATOL, replay=seg)[0]
                outs += list(want[1:1 + len(inner)]) + ([want[-1]] if hi in times else [])
                y = want[-1]
            ys = torch.stack(outs)
        ys = ys.movedim(0, 1)
        grads = torch.autograd.grad(ys, [zz] + fc.params, gg)
    return ys.detach(), grads[0], list(grads[1:])


class _Calls:
    def __init__(self, monkeypatch):
        self.names = []
        real = _lib.call

        def call(name, *args):
            self.names.append(name)
            return real(name, *args)

        monkeypatch.setattr(_lib, "call", call)


def _no_autograd(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("autograd ran in the backward")
    monkeypatch.setattr(torch.autograd, "grad", refuse)


def _leaves(func, roles):
    """The parameters that want a gradient: ``roles`` among "z0", "l1", "l2" (bias=False modules have no biases)."""
    for lin, name in ((func.linear1, "l1"), (func.linear2, "l2")):
        for p in lin.parameters():
            p.requires_grad_(name in roles)
    return [p for p in func.parameters() if p.requires_grad]


def _run(X, func, z0, t, g, roles=("z0", "l1", "l2"), monkeypatch=None, **kwargs):
    """One cdeint(adjoint=False) call and one backward on the route (its calls recorded, autograd refused in the
    backward): (outputs, dL/dz0 or None, [dL/dtheta], stats, backward calls)."""
    params = _leaves(func, roles)
    zz = z0.clone().requires_grad_("z0" in roles)
    calls = _Calls(monkeypatch)
    out = cde.cdeint(X, func, zz, t, adjoint=False, **kwargs)
    stats = dict(cde.cdeint.last_stats)
    n_fwd = len(calls.names)
    assert out.grad_fn is not None and type(out.grad_fn).__name__ == "_Dopri5MlpBackpropFnBackward", out.grad_fn
    with monkeypatch.context() as m:
        _no_autograd(m)
        out.backward(g)
    backward = calls.names[n_fwd:]
    assert backward.count(BACKWARD) >= 1 and set(backward) <= {BACKWARD, PARAMS}, backward
    assert (PARAMS in backward) == bool(params), backward
    grads = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    return out.detach(), (zz.grad.clone() if zz.requires_grad else None), grads, stats, backward


def _path_errs(got, want):
    got = got.detach().double()
    want = want.detach().double().to(got.device)
    return ((got - want).abs().amax(dim=1) / want.abs().amax(dim=1).clamp_min(1e-300)).cpu()


def _plain(X, func, z0, t, **kwargs):
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, **kwargs)
    return out, dict(cde.cdeint.last_stats)


def _g(shape, dtype, seed=11):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=F64).to(DEV, dtype)


def _case(shape, dtype, control, t_list, batch=129, roles=("z0", "l1", "l2"), bias=True, jumps=False,
          monkeypatch=None, t_device="cpu", m=None, what="", **kwargs):
    X, func, z0 = _problem(shape, dtype, control, batch, bias)
    t = torch.tensor(t_list, dtype=F64, device=t_device)
    if jumps:
        kwargs["options"] = dict(kwargs.get("options", {}), jump_t=X.grid_points)
    plain, plain_stats = _plain(X, func, z0, t, **kwargs)
    g = _g(plain.shape, dtype)
    out, gz, grads, stats, backward = _run(X, func, z0, t, g, roles, monkeypatch, **kwargs)
    assert torch.equal(out, plain)
    assert (stats["n_accepted"], stats["n_rejected"]) == (plain_stats["n_accepted"], plain_stats["n_rejected"])
    assert stats["device_controlled"] is False and len(stats["steps"]) == stats["n_accepted"]
    jump_list = [(-v if t_list[0] > t_list[-1] else v) for v in X.grid_points.tolist()] if jumps else ()
    ys, wz, wp = _oracle(X, func, control, dtype, z0, t_list, g, stats["steps"], jump_list, m)
    bar_z, bar_p = BARS[dtype]
    what = "{} {} {} {}".format(shape, control, "fp32" if dtype == F32 else "fp64", what)
    hidden = z0.size(-1)
    _report("outputs vs replay | " + what, _global_err(out.reshape(-1, len(t_list), hidden)[:m], ys),
            2e-5 if dtype == F32 else 1e-10)
    if gz is not None:
        _check_paths("dopri5 backprop dL/dz0 | " + what, gz.reshape(-1, hidden)[:m], wz, bar_z, dtype)
        kinked = _path_errs(gz.reshape(-1, hidden)[:m], wz) > bar_z
        if kinked.any() and grads:
            # a path at a relu kink (fp32 only: _check_paths allows 1 in 32) also moves dL/dtheta, which sums over the
            # paths: once more without its output gradients (the steps and every other path are unchanged)
            print("{}: {} path(s) at a relu kink".format(what, int(kinked.sum())))
            g = g.clone()
            g.reshape(-1, len(t_list), hidden)[:kinked.numel()][kinked.to(g.device)] = 0.0
            _o, gz, grads, stats2, _b = _run(X, func, z0, t, g, roles, monkeypatch, **kwargs)
            assert stats2["steps"] == stats["steps"]
            ys, wz, wp = _oracle(X, func, control, dtype, z0, t_list, g, stats["steps"], jump_list, m)
            assert not (_path_errs(gz.reshape(-1, hidden)[:m], wz) > bar_z).any()
    want = dict(zip([id(p) for p in func.parameters()], wp))
    for p, got in zip([p for p in func.parameters() if p.requires_grad], grads):
        _report("dopri5 backprop dL/dtheta | " + what, _global_err(got, want[id(p)]), bar_p)
    return X, func, z0, t, g, out, gz, grads, stats, backward


# ---- 1. the route against the oracle --------------------------------------------------------------------------------
T_DEFAULT = [0.0, 0.7, 5.3, 11.0, 23.0]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("control", CONTROLS)
def test_examples_shape_matches_the_replayed_oracle(control, dtype, monkeypatch):
    _case((8, 3, 128), {"fp32": F32, "fp64": F64}[dtype], control, T_DEFAULT, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,control,dtype,variant", [
    ((8, 14, 128), "cubic", F32, 0),        # the logsignature example's depth-3 width: the torch-operator field forward
    ((8, 14, 128), "linear", F64, 0),
    ((4, 2, 37), "linear", F32, 0),         # an odd width
    ((10, 3, 128), "cubic", F32, 1),        # HM = 32, under solve variant 1
    ((16, 2, 64), "linear", F64, 1),
], ids=["8x14_fp32", "8x14_fp64", "4x2w37", "10x3_v1", "16x2_v1_fp64"])
def test_other_shapes_match_the_replayed_oracle(shape, control, dtype, variant, monkeypatch):
    with _variant(variant):
        _, _, _, _, _, _, _, _, stats, backward = _case(shape, dtype, control, T_DEFAULT, batch=96,
                                                        monkeypatch=monkeypatch)
    assert backward.count(BACKWARD) == -(-stats["n_accepted"] // mlp_field.Dopri5MlpBackprop.slots)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["decreasing", "first_step", "t_on_gpu", "several_in_one_step"])
def test_times_and_options(case, monkeypatch):
    t_list = {"decreasing": [23.0, 9.5, 3.25, 0.0],
              "several_in_one_step": [0.0, 0.3, 0.3001, 0.3002, 0.3003, 7.0]}.get(case, T_DEFAULT)
    kwargs = {"options": {"first_step": 0.05}} if case == "first_step" else {}
    res = _case((8, 3, 128), F32, "cubic", t_list, monkeypatch=monkeypatch, what=case,
                t_device=DEV if case == "t_on_gpu" else "cpu", **kwargs)
    stats = res[-2]
    if case == "first_step":
        assert stats["steps"][0][1] == 0.05
    if case == "decreasing":
        assert all(s <= -0.0 for s, _d in stats["steps"][1:]) and stats["steps"][0][0] == -23.0


@pytest.mark.gpu
@pytest.mark.parametrize("control", CONTROLS)
def test_outputs_on_a_step_end_and_inside_one_step(control, monkeypatch):
    # the solve's steps do not depend on the output times inside (0, 23): an output exactly on the end of step 5 (which
    # emits it with x = 1) and two inside step 6
    res = _case((8, 3, 128), F32, control, [0.0, 23.0], batch=64, monkeypatch=monkeypatch, what="two outputs")
    s5, d5 = res[-2]["steps"][5]
    s6, d6 = res[-2]["steps"][6]
    t_list = [0.0, s5 + d5, s6 + 0.25 * d6, s6 + 0.75 * d6, 23.0]
    res2 = _case((8, 3, 128), F32, control, t_list, batch=64, monkeypatch=monkeypatch, what="step end")
    assert res2[-2]["steps"] == res[-2]["steps"]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
def test_jump_t_on_a_linear_control(dtype, monkeypatch):
    """options=dict(jump_t=X.grid_points): every step after a knot starts from a slope of its own, which gets its own
    item, J^T and parameter-gradient contribution."""
    dt = {"fp32": F32, "fp64": F64}[dtype]
    res = _case((8, 3, 128), dt, "linear", [0.0, 2.7, 6.0, 11.5], jumps=True, monkeypatch=monkeypatch, what="jump_t")
    X, stats = res[0], res[-2]
    knots = X.grid_points.tolist()
    starts = [s for s, _d in stats["steps"]]
    assert sum(1 for s in starts if s in knots) >= 5
    for s, d in stats["steps"]:
        assert not any(s < j < s + d for j in knots), (s, d)



@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 129, (3, 43)], ids=["1", "129", "3x43"])
def test_batch_edges(batch, monkeypatch):
    _case((8, 3, 128), F32, "cubic", T_DEFAULT, batch=batch, monkeypatch=monkeypatch, what="batch {}".format(batch))


@pytest.mark.gpu
@pytest.mark.parametrize("roles,bias", [(("z0",), True), (("l1",), True), (("l2",), True), (("z0", "l1", "l2"), False)],
                         ids=["z0_only", "layer1_only", "layer2_only", "no_bias"])
def test_parameter_roles(roles, bias, monkeypatch):
    res = _case((8, 3, 128), F32, "cubic", T_DEFAULT, roles=roles, bias=bias, monkeypatch=monkeypatch,
                what="roles {} bias {}".format(roles, bias))
    gz, grads = res[6], res[7]
    assert (gz is not None) == ("z0" in roles)
    assert len(grads) == 2 * sum(1 for r in ("l1", "l2") if r in roles) // (1 if bias else 2)


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [True, False], ids=["exact_multiple", "partial_last"])
def test_three_slot_chunks(exact, monkeypatch):
    monkeypatch.setattr(mlp_field.Dopri5MlpBackprop, "slots", 3)
    X, func, z0 = _problem((8, 3, 128), F32, "cubic", 64)
    t_end = None
    for cand in [23.0, 22.0, 21.0, 20.0, 19.0, 18.0, 17.0, 16.0, 15.0, 14.0, 13.0]:
        _plain(X, func, z0, torch.tensor([0.0, cand], dtype=F64))
        if (cde.cdeint.last_stats["n_accepted"] % 3 == 0) == exact:
            t_end = cand
            break
    assert t_end is not None
    res = _case((8, 3, 128), F32, "cubic", [0.0, 0.5 * t_end, t_end], batch=64, monkeypatch=monkeypatch,
                what="3-slot chunks")
    stats, backward = res[-2], res[-1]
    assert (stats["n_accepted"] % 3 == 0) == exact
    n_chunks = -(-stats["n_accepted"] // 3)
    assert backward.count(BACKWARD) == n_chunks and backward.count(PARAMS) == n_chunks


# ---- 2. autograd modes ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_create_graph_matches_the_torch_replay(monkeypatch):
    X, func, z0 = _problem((8, 3, 128), F32, "cubic", 32)
    t = torch.tensor([0.0, 3.0, 9.0], dtype=F64)

    zz = z0.clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    out = cde.cdeint(X, func, zz, t, adjoint=False)
    assert type(out.grad_fn).__name__ == "_Dopri5MlpBackpropFnBackward"
    steps = cde.cdeint.last_stats["steps"]
    # a cotangent that does not depend on the outputs (the route's forward field and the replay's differ in rounding)
    c = _g(out.shape, F32, seed=5)
    (gz,) = torch.autograd.grad((out * c).sum(), zz, create_graph=True)
    (gz ** 2).sum().backward()
    gz, gzz, gw = gz.detach(), zz.grad.clone(), func.linear1.weight.grad.clone()
    # the torch-operator replay of the route's own steps, differentiated twice by autograd
    zz = z0.clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    field = solver._torch_field(X, func, False, True, z0)
    ys = adaptive.odeint_dopri5(field, zz, t.tolist(), RTOL, ATOL, steps=steps)[0].movedim(0, -2)
    (rgz,) = torch.autograd.grad((ys * c).sum(), zz, create_graph=True)
    (rgz ** 2).sum().backward()
    assert _global_err(gz, rgz) <= 1e-6
    assert _global_err(gzz, zz.grad) <= 1e-6
    assert _global_err(gw, func.linear1.weight.grad) <= 1e-6


@pytest.mark.gpu
def test_retain_graph_and_two_runs_give_the_same_bits(monkeypatch):
    X, func, z0 = _problem((8, 3, 128), F32, "linear", 129)
    t = torch.tensor(T_DEFAULT, dtype=F64)
    g = _g((129, len(T_DEFAULT), 8), F32)
    runs = []
    for _ in range(2):
        zz = z0.clone().requires_grad_(True)
        for p in func.parameters():
            p.grad = None
        out = cde.cdeint(X, func, zz, t, adjoint=False)
        out.backward(g, retain_graph=True)
        first = [zz.grad.clone()] + [p.grad.clone() for p in func.parameters()]
        zz.grad = None
        for p in func.parameters():
            p.grad = None
        out.backward(g)
        second = [zz.grad.clone()] + [p.grad.clone() for p in func.parameters()]
        assert all(torch.equal(a, b) for a, b in zip(first, second))
        runs.append((out.detach(), first))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


# ---- 3. refusals keep the torch-operator dopri5 and its bits --------------------------------------------------------
def _grads_of(X, func, z0, t, g, coeffs=None, t_grad=False):
    zz = z0.clone().requires_grad_(True)
    tt = t.clone().requires_grad_(t_grad)
    for p in func.parameters():
        p.grad = None
    out = cde.cdeint(X, func, zz, tt, adjoint=False)
    assert type(out.grad_fn).__name__ != "_Dopri5MlpBackpropFnBackward"
    out.backward(g)
    res = [out.detach(), zz.grad] + [p.grad for p in func.parameters()]
    if coeffs is not None:
        res.append(coeffs.grad)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tensor_core_shape", "t_requires_grad", "coefficients", "softplus", "hidden16_variant0",
                                  "wide", "no_room_first_chunk", "no_room_later_chunk"])
def test_refusals_keep_the_torch_operator_route(case, monkeypatch):
    shape = {"tensor_core_shape": (32, 8, 128), "hidden16_variant0": (16, 2, 64), "wide": (8, 3, 400)}.get(case,
                                                                                                           (8, 3, 128))
    X, func, z0 = _problem(shape, F32, "cubic", 64)
    t = torch.tensor([0.0, 2.5, 12.0], dtype=F64)
    coeffs = None
    if case == "coefficients":
        coeffs = _inputs(3, 8, False)[2][:64].clone().requires_grad_(True)
        X = cde.CubicSpline(coeffs)
    if case == "softplus":
        torch.manual_seed(3)
        func = SoftplusMLP(8, 3, 128).to(DEV)
    g = _g((64, 3, shape[0]), F32)
    # today's route: the new one switched off
    with monkeypatch.context() as m:
        m.setattr(solver, "dopri5_mlp_backprop", lambda *a, **k: None)
        want = _grads_of(X, func, z0, t, g, coeffs, case == "t_requires_grad")
    if case.startswith("no_room"):
        monkeypatch.setattr(mlp_field.Dopri5MlpBackprop, "slots", 3)
        real = torch.cuda.mem_get_info
        seen = []

        def mem_get_info(*args):
            seen.append(1)
            free, total = real(*args)
            return (0 if case == "no_room_first_chunk" or len(seen) > 2 else free), total
        monkeypatch.setattr(torch.cuda, "mem_get_info", mem_get_info)
    calls = _Calls(monkeypatch)
    got = _grads_of(X, func, z0, t, g, coeffs, case == "t_requires_grad")
    # at most the dispatch's verdict (a call with no paths) before the forward
    assert calls.names.count(BACKWARD) <= 1 and PARAMS not in calls.names, calls.names
    if case == "no_room_later_chunk":
        assert len(seen) > 2                       # the route began and gave up at a later chunk
    for a, b in zip(got, want):
        assert (a is None and b is None) or torch.equal(a, b)


# ---- 4. full scale --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_scale(monkeypatch):
    """B = 65,536, L = 256, (8, 3, 128), cubic control, fp32 (the inputs of the MLP adjoint's full-scale test), against
    fp64 autograd of the replay on 256 of the paths (the only ones with an output cotangent).  Over this long solve (about
    350 accepted fp32 steps) the route's gradients sit farther from the fp64 replay than the bars of the short cases, so,
    as the MLP adjoint's full-scale test does for its worst paths, they are held to the distance of fp32 autograd through
    the same discrete solve (the torch-operator replay of the route's steps on those paths): dL/dz0 per path within twice
    it plus 1e-5 for all but 1 in 32, every path within KINK_BAR; dL/dtheta, with the paths over the first bar set aside
    (the relu-kink rule), within twice it plus 2e-4."""
    gen = torch.Generator().manual_seed(21)
    x = (torch.randn(65536, 256, 3, generator=gen) / 16).cumsum(1).to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    del x
    X, func, z0 = cde.CubicSpline(coeffs), _func(3, 8, 128, F32), torch.randn(65536, 8, generator=gen).to(DEV)
    t, m = torch.tensor([0.0, 255.0], dtype=F64), 256
    g = _g((z0.size(0), 2, 8), F32)
    g[m:] = 0.0                    # dL/dtheta of the sampled paths alone (the steps do not depend on g)
    Xm = cde.CubicSpline(coeffs[:m])

    def measure(g):
        out, gz, grads, stats, backward = _run(X, func, z0, t, g, monkeypatch=monkeypatch)
        ys, wz, wp = _oracle(X, func, "cubic", F32, z0, [0.0, 255.0], g, stats["steps"], m=m)
        # fp32 autograd through the torch-operator replay of the same steps on the sampled paths
        zz = z0[:m].clone().requires_grad_(True)
        field = solver._torch_field(Xm, func, False, True, zz)
        with torch.enable_grad():
            ya = adaptive.odeint_dopri5(field, zz, [0.0, 255.0], RTOL, ATOL, steps=stats["steps"])[0].movedim(0, -2)
            az, *ap = torch.autograd.grad(ya, [zz] + list(func.parameters()), g[:m])
        _report("outputs vs replay | full scale", _global_err(out[:m], ys), 2e-5)
        print("full scale: {} accepted, {} rejected, {} chunks".format(stats["n_accepted"], stats["n_rejected"],
                                                                     backward.count(BACKWARD)))
        return _path_errs(gz[:m], wz), _path_errs(az, wz), [(_global_err(a, w), _global_err(b, w))
                                                             for a, b, w in zip(grads, ap, wp)]

    e_route, e_auto, e_theta = measure(g)
    print("full scale dL/dz0 vs fp64, median / worst: route {:.2e} / {:.2e}, fp32 autograd {:.2e} / {:.2e}".format(
        e_route.median(), e_route.max(), e_auto.median(), e_auto.max()))
    excess = (e_route - 2 * e_auto).sort().values
    _report("dopri5 backprop dL/dz0 | full scale, beyond twice fp32 autograd's distance (all but 1 in 32)",
            float(excess[-(1 + m // 32)]), 1e-5)
    _report("dopri5 backprop dL/dz0 at a relu kink | full scale", float(e_route.max()), KINK_BAR)
    kinked = e_route - 2 * e_auto > 1e-5
    if kinked.any():
        # dL/dtheta sums over the paths, the kinked ones included: once more without their output gradients
        g[:m][kinked.to(DEV)] = 0.0
        e_route, e_auto, e_theta = measure(g)
    for e, a in e_theta:
        print("full scale dL/dtheta vs fp64 ({} kinked paths set aside): route {:.2e}, fp32 autograd {:.2e}".format(
            int(kinked.sum()), e, a))
        _report("dopri5 backprop dL/dtheta | full scale, beyond twice fp32 autograd's distance", e - 2 * a, 2e-4)


# ---- 5. without a GPU -----------------------------------------------------------------------------------------------
def test_fp64_tables_against_the_float32_default():
    steps = [(0.0, 0.37), (0.37, 0.9), (1.27, 1.13), (2.4, 0.6)]
    times = [0.0, 0.2, 1.27, 2.0, 3.0]
    t32 = adaptive.dopri5_backward_tables(steps, times)
    t64 = adaptive.dopri5_backward_tables(steps, times, torch.float64)
    assert t32["coef"].dtype == torch.float32 and t32["inj_w"].dtype == torch.float32
    assert t64["coef"].dtype == torch.float64 and t64["inj_w"].dtype == torch.float64
    assert torch.equal(t64["coef"].float(), t32["coef"]) and torch.equal(t64["inj_w"].float(), t32["inj_w"])
    assert torch.equal(t64["inj_range"], t32["inj_range"]) and torch.equal(t64["inj_out"], t32["inj_out"])
    assert t64["coef"][1, 0] == 0.2 * 0.9                       # beta[0][0] dt in double
    # ends: a step cut at a jump ends on it even where t + dt does not reach it
    ends = [0.37, 1.27, 2.4, 3.0000000000000004]
    t_end = adaptive.dopri5_backward_tables(steps, times + [3.0000000000000004], torch.float64, ends)
    assert t_end["inj_range"].tolist()[-1] == 5


def test_entry_rejects_bad_arguments_before_any_cuda_call():
    p = lambda: _lib.ctypes.c_void_p(16)  # noqa: E731  (never dereferenced: the checks come first)

    def call(*over, **named):
        args = dict(control=p(), kind=0, n_rows=4, w1=p(), b1=p(), w2=p(), b2=p(), rec_z=p(), grad_out=p(), carry=p(),
                    kappa=None, coef=p(), step_item=p(), item_index=p(), item_frac=p(), inj_range=p(), inj_out=p(),
                    inj_w=p(), n_out=3, n_steps=2, n_paths=10, channels=3, hidden=8, width=128, sign=1.0,
                    dtype=_lib.F32, stream=None)
        args.update(named)
        return _lib.call(BACKWARD, *args.values())

    with pytest.raises(ValueError, match="null data pointer"):
        call(rec_z=None)
    with pytest.raises(ValueError, match="null table pointer"):
        call(step_item=None)
    with pytest.raises(ValueError, match="bad sizes"):
        call(n_out=1)
    with pytest.raises(ValueError, match="bad sizes"):
        call(n_steps=-1)
    with pytest.raises(ValueError, match="dtype"):
        call(dtype=7)
    with pytest.raises(ValueError, match="sign"):
        call(sign=0.5)
    # the policy: the tensor-core shape, hidden 16 without solve variant 1
    with pytest.raises(NotImplementedError):
        call(hidden=32, channels=8, width=128, n_paths=0)
    with pytest.raises(NotImplementedError):
        call(hidden=16, channels=2, width=64, n_paths=0)
    assert call(n_paths=0) == 0                                  # served: nothing launched
    assert call(dtype=_lib.F64, n_paths=0) == 0
