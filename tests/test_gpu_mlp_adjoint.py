"""The per-evaluation kernels of the examples' MLP field against the fp64 oracle: ``tcde_vector_field_mlp`` (one launch
per field evaluation of the host-driven dopri5) and ``tcde_vector_field_mlp_vjp`` (one call per stage of the
``adjoint=True`` backward, for dopri5 and the fixed-step methods).  They serve the CUDA-core shapes (hidden <= 8 by
default, hidden * channels <= 32 under solve variant 1; fp32 and fp64); everywhere else the old routes keep the call.

Reference: ``adaptive_oracle.FuncCDE`` over an fp64 copy of the module and of the kernels' own rounded inputs
(``test_gpu_generic_routes._oracle``), ``AO.fixed_adjoint`` for the fixed-step backward and ``AO.solve`` replaying the
host loop's own step decisions for dopri5.  Every case proves its route: the names of the library calls are recorded and
the other routes are patched to raise.  fp32 kink rule (DESIGN 5): a path with a hidden unit whose oracle
pre-activation lies within fp32 rounding of 0 may take the other side of the relu, so its cotangent is zeroed (kernel
level) or it is held to KINK_BAR (whole solves)."""
import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from test_gpu_generic_routes import (KINK_BAR, Func, SoftplusMLP, _Attempts, _Calls, _check_host_attempts, _control,
                                     _global_err, _grad_pattern, _inputs, _options, _oracle, _path_err, _times,
                                     _ys_for_oracle)
from test_gpu_mlp_field import _variant
from test_host_logic import FIXED_SCHEDULES
from torchcde_b200 import _lib, solver
from torchcde_b200.mlp_field import MlpAdjointStage, MlpFieldKernels

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
CONTROLS = ["cubic", "linear"]
FIELD, VJP = "tcde_vector_field_mlp", "tcde_vector_field_mlp_vjp"
KERNEL_BAR = {F32: 1e-5, F64: 1e-12}

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[MLP adjoint, worst of each check] " + "; ".join(
        "{}: {:.2e} (bar {:.0e})".format(k, e, b) for k, (e, b) in sorted(_WORST.items())))


def _report(what, err, bar):
    key = what.split(" |")[0]
    if err > _WORST.get(key, (-1.0, bar))[0]:
        _WORST[key] = (err, bar)
    assert err <= bar, (what, err, bar)


def _func(channels, hidden, width, dtype, bias=True, seed=0):
    torch.manual_seed(500 + seed + 7 * hidden + channels + width)
    func = Func(channels, hidden, width).to(DEV).to(dtype)
    if not bias:
        func.linear1.bias = None
        func.linear2.bias = None
    return func


def _problem(hidden, channels, width, dtype, control, batch, uneven=False, bias=True):
    """(X, func, z0) on the first ``batch`` of up to 1000 paths of 40 knots (batch > 1000: the paths repeated)."""
    x, knots, coeffs, z0 = _inputs(channels, hidden, uneven)
    reps = -(-batch // 1000) if batch else 1
    src = (coeffs if control == "cubic" else x).repeat(reps, 1, 1)[:batch].to(dtype)
    kt = None if knots is None else knots.to(dtype)
    return _control(src, kt, control), _func(channels, hidden, width, dtype, bias), z0.repeat(reps, 1)[:batch].to(dtype)


def _variant_for(shape, dtype):
    """The solve variant under which the stage serves ``shape``: 0 where the dispatch runs it by default (fp32, hidden *
    channels <= 32, width <= 128), else 1, which forces it."""
    hidden, channels, width = shape
    return 0 if dtype == F32 and hidden <= 8 and hidden * channels <= 32 and width <= 128 else 1


def _params(func):
    return (func.linear1.weight, func.linear1.bias, func.linear2.weight, func.linear2.bias)


def _kinked(func, z, dtype):
    """Paths with a hidden unit whose fp64 pre-activation is within fp32 rounding of 0 (none in fp64)."""
    if dtype == F64:
        return torch.zeros(z.size(0), dtype=torch.bool, device=z.device)
    w1 = func.linear1.weight.detach().double()
    b1 = func.linear1.bias.detach().double() if func.linear1.bias is not None else torch.zeros(w1.size(0), device=DEV,
                                                                                                dtype=F64)
    zz = z.detach().double()
    pre = zz @ w1.T + b1
    scale = zz.abs() @ w1.abs().T + b1.abs()
    return (pre.abs() <= 4 * 2.0 ** -24 * scale).any(dim=1)


# ---- 1. the two entries -------------------------------------------------------------------------------------------
def _kernel_case(shape, dtype, control, batch, t, uneven=False, bias=True, scales=(1.0, 1.0, 1.0), want=(1, 1, 1, 1),
                 accumulate=False, monkeypatch=None):
    with _variant(_variant_for(shape, dtype)):
        return _kernel_case_at(shape, dtype, control, batch, t, uneven, bias, scales, want, accumulate, monkeypatch)


def _kernel_case_at(shape, dtype, control, batch, t, uneven, bias, scales, want, accumulate, monkeypatch):
    hidden, channels, width = shape
    X, func, z0 = _problem(hidden, channels, width, dtype, control, batch, uneven, bias)
    k = MlpFieldKernels(X, _params(func), z0)
    index, frac = k.where(t)
    gen = torch.Generator().manual_seed(batch + hidden)
    a = torch.randn(batch, hidden, generator=gen, dtype=F64).to(DEV)
    kinked = _kinked(func, z0, dtype)
    a[kinked] = 0.0
    a = a.to(dtype)
    params = [p for p in _params(func) if p is not None]
    chosen = [p for p, w in zip(_params(func), want) if w and p is not None]
    stage = k.adjoint_stage(chosen)
    assert isinstance(stage, MlpAdjointStage)
    grads = stage.new_grads()
    if accumulate:
        for g in grads:
            g.copy_(torch.randn(g.shape, generator=gen, dtype=F64).to(g))
    before = [g.clone() for g in grads]
    f_out, vjp_out = torch.empty_like(z0), torch.empty_like(z0)
    f_scale, vjp_scale, grad_scale = scales
    calls = _Calls(monkeypatch)
    stage.launch(index, frac, z0, a, f_out, vjp_out, *grads, f_scale=f_scale, vjp_scale=vjp_scale,
                 grad_scale=grad_scale)
    field = k.field()(t, z0)
    assert calls.names == ([VJP, FIELD] if batch else []), calls.names          # an empty batch launches nothing
    assert torch.equal(f_out, field * f_scale)
    fc = _oracle(X, func, control, dtype)
    chosen64 = [q for q, p in zip(fc.params, params) if any(p is c for c in chosen)]
    f, gz, gp = fc.vjp(t, z0.double(), a.double(), chosen64)
    bar = KERNEL_BAR[dtype]
    what = "{} {} {} batch {} t {} | {}".format(shape, dtype, control, batch, t, int(kinked.sum()))
    if batch:
        _report("field f | " + what, _path_err(f_out, f_scale * f), bar)
        _report("vjp a^T df/dz | " + what, _path_err(vjp_out, vjp_scale * gz), bar)
    for g, g0, want_g in zip(grads, before, gp):
        expect = g0.double() + grad_scale * want_g
        _report("vjp a^T df/dtheta | " + what, _global_err(g, expect) if expect.abs().max() > 0 else
                float(g.abs().max()), bar)
    assert int(kinked.sum()) <= max(1, batch // 32), (what, int(kinked.sum()))
    return index, frac, k


KERNEL_SHAPES = [(8, 3, 128), (8, 14, 128), (1, 1, 1), (5, 3, 37)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("shape", KERNEL_SHAPES, ids=lambda s: "{}x{}w{}".format(*s))
def test_kernels_match_fp64_autograd(shape, control, dtype, monkeypatch):
    dt = {"fp32": F32, "fp64": F64}[dtype]
    _kernel_case(shape, dt, control, 129, 7.3, monkeypatch=monkeypatch)
    _kernel_case(shape, dt, control, 129, 20.0, uneven=True, bias=False, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [0, 1, 127, 128, 129, 3000])
def test_batch_edges(batch, monkeypatch):
    _kernel_case((8, 3, 128), F32, "cubic", batch, 11.6, monkeypatch=monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("where", ["first", "last", "knot"])
def test_first_and_last_interval_and_frac_zero(where, control, monkeypatch):
    t = {"first": 0.0, "last": 39.0, "knot": 17.0}[where]
    index, frac, k = _kernel_case((8, 3, 128), F64, control, 129, t, monkeypatch=monkeypatch)
    if where == "first":
        assert (index, frac) == (0, 0.0)
    elif where == "last":
        assert index == k.n_rows - 1, (index, k.n_rows)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
def test_scales_null_gradients_and_accumulation(dtype, monkeypatch):
    dt = {"fp32": F32, "fp64": F64}[dtype]
    _kernel_case((8, 3, 128), dt, "cubic", 300, 5.5, scales=(-1.0, -0.75, -0.3), want=(1, 0, 0, 1), accumulate=True,
                 monkeypatch=monkeypatch)
    _kernel_case((8, 3, 128), dt, "linear", 300, 5.5, scales=(1.0, 2.5, 0.125), want=(0, 1, 1, 0), accumulate=True,
                 monkeypatch=monkeypatch)


def _max_width(hidden, channels):
    lib = _lib.load()
    w = 1
    while lib.tcde_vector_field_mlp_vjp_scratch_bytes(1000, channels, hidden, 2 * w) > 0:
        w *= 2
    lo, hi = w, 2 * w
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if lib.tcde_vector_field_mlp_vjp_scratch_bytes(1000, channels, hidden, mid) > 0 else (lo, mid)
    return lo


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
def test_width_at_the_shared_memory_limit(dtype, monkeypatch):
    with _variant(1):                           # past width 128 only solve variant 1 runs the stage
        width = _max_width(8, 3)
    assert 128 < width < 4096
    _kernel_case((8, 3, width), {"fp32": F32, "fp64": F64}[dtype], "cubic", 129, 9.1, monkeypatch=monkeypatch)


@pytest.mark.gpu
def test_two_calls_give_the_same_bits(monkeypatch):
    X, func, z0 = _problem(8, 3, 128, F32, "cubic", 3000)
    stage = MlpFieldKernels(X, _params(func), z0).adjoint_stage([p for p in _params(func)])
    a = torch.randn_like(z0)
    runs = [stage(4.4, z0, a, -1.0) for _ in range(2)]
    assert all(torch.equal(x, y) for x, y in zip(runs[0][:2], runs[1][:2]))
    assert all(torch.equal(x, y) for x, y in zip(runs[0][2], runs[1][2]))


def test_scratch_query_follows_the_served_shapes():
    lib = _lib.load()
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 3, 8, 128) > 0
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(0, 3, 8, 128) > 0
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 8, 32, 128) == -1       # the tensor-core shape
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 2, 16, 128) == -1       # hidden 16 under variant 0
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 4, 8, 128) > 0          # hidden * channels = 32
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 5, 8, 128) == -1        # slower: hidden * channels > 32
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 3, 8, 129) == -1        # slower: width > 128
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(100, 3, 8, 1 << 20) == -1
    assert lib.tcde_vector_field_mlp_vjp_scratch_bytes(-1, 3, 8, 128) == -1


def test_null_pointers_are_rejected_before_any_cuda_call():
    lib = _lib.load()
    p = lambda: _lib.ctypes.c_void_p(16)  # noqa: E731  (never dereferenced: the checks come first)
    with pytest.raises(ValueError, match="null data pointer"):
        _lib.call(FIELD, None, 0, 4, p(), p(), p(), p(), p(), p(), 10, 3, 8, 128, 0, 0.0, _lib.F32, None)
    with pytest.raises(ValueError, match="null data pointer"):
        _lib.call(VJP, p(), 0, 4, p(), p(), p(), p(), p(), p(), p(), None, None, None, None, None, p(), 10, 3, 8, 128, 0,
                  0.0, 1.0, 1.0, 1.0, _lib.F32, None)
    with pytest.raises(ValueError, match="index"):
        _lib.call(FIELD, p(), 0, 4, p(), p(), p(), p(), p(), p(), 10, 3, 8, 128, 4, 0.0, _lib.F32, None)
    assert lib is _lib.load()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["32x8_fp32", "16x2_variant0", "fp16_code", "fp64_default", "8x14_default",
                                  "w129_default"])
def test_refusals(case, monkeypatch):
    """The tensor-core shape, hidden 16, another dtype, and by default the shapes where the stage measured slower than
    autograd (fp64, hidden * channels > 32, width > 128)."""
    shape, dtype = {"32x8_fp32": ((32, 8, 128), F32), "16x2_variant0": ((16, 2, 128), F32),
                    "fp16_code": ((8, 3, 128), F32), "fp64_default": ((8, 3, 128), F64),
                    "8x14_default": ((8, 14, 128), F32), "w129_default": ((8, 3, 129), F32)}[case]
    X, func, z0 = _problem(*shape, dtype, "cubic", 65)
    k = MlpFieldKernels(X, _params(func), z0)
    if case != "fp16_code":
        with pytest.raises(NotImplementedError):
            k.field()(3.0, z0)
        assert k.adjoint_stage(list(func.parameters())) is None
    scratch = torch.empty(1 << 20, device=DEV)
    code = 7 if case == "fp16_code" else _lib.dtype_code(dtype)
    with pytest.raises(NotImplementedError):
        _lib.call(VJP, _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1), _lib.ptr(k.b1), _lib.ptr(k.w2),
                  _lib.ptr(k.b2), _lib.ptr(z0), _lib.ptr(z0), _lib.ptr(scratch), _lib.ptr(scratch), None, None, None,
                  None, _lib.ptr(scratch), 65, k.channels, k.hidden, k.width, 1, 0.5, 1.0, 1.0, 1.0, code,
                  _lib.stream_of(z0))
    with pytest.raises(NotImplementedError):
        _lib.call(FIELD, _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(k.w1), _lib.ptr(k.b1), _lib.ptr(k.w2),
                  _lib.ptr(k.b2), _lib.ptr(z0), _lib.ptr(scratch), 65, k.channels, k.hidden, k.width, 1, 0.5, code,
                  _lib.stream_of(z0))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("shape", [(16, 2, 128), (10, 3, 128), (9, 3, 37)], ids=lambda s: "{}x{}w{}".format(*s))
def test_hidden_past_8_runs_under_variant_1(shape, dtype, monkeypatch):
    """The HM = 32 kernels at hidden 16 and at hidden 9 and 10, which are not multiples of 4: in fp64 the stage reads z
    from a shared column whose padding up to the next multiple of 4 must be zeros."""
    dt = {"fp32": F32, "fp64": F64}[dtype]
    _kernel_case(shape, dt, "cubic", 129, 6.2, monkeypatch=monkeypatch)
    _kernel_case(shape, dt, "linear", 300, 31.4, uneven=True, bias=False, scales=(-1.0, 0.5, -2.0), accumulate=True,
                 monkeypatch=monkeypatch)


# ---- 2. the fixed-step adjoint=True ---------------------------------------------------------------------------------
ADJ_PATHS = 96
FIXED_CASES = [(s, "rk4") for s in FIXED_SCHEDULES] + [("F3", "midpoint"), ("F3", "euler")]


def _no_autograd(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("autograd ran in the backward")
    monkeypatch.setattr(torch.autograd, "grad", refuse)


def _check_paths(what, got, want, bar, dtype):
    got = got.detach().double().reshape(-1, got.size(-1))
    want = want.detach().double().to(got.device).reshape(got.shape)
    errs = ((got - want).abs().amax(dim=1) / want.abs().amax(dim=1).clamp_min(1e-300)).cpu()
    if dtype == F64:
        _report(what, float(errs.max()), bar)
        return
    _report(what + " (all but 1 in 32)", float(errs.sort().values[-(1 + errs.numel() // 32)]), bar)
    _report(what.split(" |")[0] + " at a relu kink |" + what.split(" |")[1], float(errs.max()), KINK_BAR)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("shape", [(8, 3, 128), (8, 14, 128)], ids=["8x3", "8x14"])
@pytest.mark.parametrize("sname,method", FIXED_CASES)
def test_fixed_step_adjoint_matches_the_oracle(sname, method, shape, control, dtype, monkeypatch):
    _fixed_case(sname, method, shape, control, {"fp32": F32, "fp64": F64}[dtype], monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("shape", [(10, 3, 128), (9, 3, 37)], ids=["10x3", "9x3w37"])
def test_fixed_step_adjoint_under_variant_1(shape, dtype, monkeypatch):
    """cdeint(adjoint=True) reaches the HM = 32 stage at hidden 9 and 10 under solve variant 1."""
    _fixed_case("F3", "rk4", shape, "cubic", {"fp32": F32, "fp64": F64}[dtype], monkeypatch)


def _fixed_case(sname, method, shape, control, dt, monkeypatch):
    with _variant(_variant_for(shape, dt)):
        _fixed_case_at(sname, method, shape, control, dt, monkeypatch)


def _fixed_case_at(sname, method, shape, control, dt, monkeypatch):
    dtype = "fp32" if dt == F32 else "fp64"
    hidden, channels, width = shape
    ts, step, uneven = FIXED_SCHEDULES[sname]
    X, func, z0 = _problem(hidden, channels, width, dt, control, ADJ_PATHS, uneven)
    t, step = _times(sname)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    decreasing = sname == "F8"                        # decreasing t keeps the autograd-per-stage backward
    calls = _Calls(monkeypatch)
    with monkeypatch.context() as m:
        if not decreasing:
            _no_autograd(m)
        zz = z0.clone().requires_grad_(True)
        out = cde.cdeint(X, func, zz, t, adjoint=True, method=method, options=_options(step))
        n_fwd = len(calls.names)
        g = _grad_pattern(out.shape).to(DEV, dt)
        out.backward(g)
    assert torch.equal(out.detach(), plain)
    backward = calls.names[n_fwd:]
    if decreasing:
        assert VJP not in backward
    else:
        n_stages = {"rk4": 4, "midpoint": 2, "euler": 1}[method]
        assert backward.count(VJP) % n_stages == 0 and backward.count(VJP) > 0, backward
        assert set(backward) <= {VJP, "tcde_linear_combination"}, set(backward)
    fc = _oracle(X, func, control, dt)
    wz, wp, _ = AO.fixed_adjoint(fc, _ys_for_oracle(out), g.double().movedim(-2, 0), t.tolist(), method, step)
    what = "{} {} {} {} {}".format(shape, control, sname, method, dtype)
    _check_paths("fixed adjoint dL/dz0 | " + what, zz.grad, wz, 1e-10 if dt == F64 else 1e-5, dt)
    for p, want in zip(func.parameters(), wp):
        _report("fixed adjoint dL/dtheta | " + what, _global_err(p.grad, want), 1e-10 if dt == F64 else 2e-4)


@pytest.mark.gpu
def test_one_vjp_call_per_stage(monkeypatch):
    """rk4 step 1 over t = 0 .. 39: 39 steps x 4 stages calls, one per stage, and nothing else but the combinations."""
    X, func, z0 = _problem(8, 3, 128, F32, "cubic", 200)
    zz = z0.clone().requires_grad_(True)
    out = cde.cdeint(X, func, zz, torch.tensor([0.0, 39.0], dtype=F64), adjoint=True, method="rk4",
                     options={"step_size": 1.0})
    calls = _Calls(monkeypatch)
    _no_autograd(monkeypatch)
    out.backward(torch.ones_like(out))
    assert calls.names.count(VJP) == 39 * 4
    assert set(calls.names) == {VJP, "tcde_linear_combination"}


# ---- 3. the host-driven dopri5 forward ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("shape", [(8, 3, 128), (8, 14, 128)], ids=["8x3", "8x14"])
def test_dopri5_forward_attempt_by_attempt(shape, control, monkeypatch):
    hidden, channels, width = shape
    X, func, z0 = _problem(hidden, channels, width, F32, control, 200)
    with _variant(_variant_for(shape, F32)):
        _dopri5_forward(X, func, z0, shape, control, monkeypatch)


def _dopri5_forward(X, func, z0, shape, control, monkeypatch):
    attempts = _Attempts(monkeypatch)
    calls = _Calls(monkeypatch)
    monkeypatch.setattr(solver, "_torch_field", lambda *a: (_ for _ in ()).throw(AssertionError("torch field ran")))
    t_list, rtol, atol = [0.0, 2.7, 5.0], 1e-4, 1e-6
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, torch.tensor(t_list, dtype=F64), adjoint=False, rtol=rtol, atol=atol)
    (records,) = attempts.lists()
    # (tcde_spline_eval: cdeint's compatibility check of X.derivative at t[0])
    assert set(calls.names) <= {FIELD, "tcde_linear_combination", "tcde_error_ratio_sumsq", "tcde_spline_eval"}
    # the probe, the start slope, Hairer's second evaluation and six per attempt
    assert calls.names.count(FIELD) == 3 + 6 * len(records)
    fc = _oracle(X, func, control, F32)
    what = "{} {}".format(shape, control)
    replay = _check_host_attempts(records, fc, rtol, atol, what)
    want, _rec, _ = AO.solve(fc, z0.double(), t_list, rtol, atol, replay=replay)
    _report("dopri5 outputs vs replay | " + what, _global_err(out.movedim(-2, 0), want), 2e-5)


# ---- 4. the examples' exact call ------------------------------------------------------------------------------------
def _examples_call(monkeypatch, dtype, control, batch=64):
    X, func, z0 = _problem(8, 3, 128, dtype, control, batch)
    attempts = _Attempts(monkeypatch)
    calls = _Calls(monkeypatch)
    zz = z0.clone().requires_grad_(True)
    t = torch.tensor([0.0, 2.6, 5.0], dtype=F64)
    out = cde.cdeint(X=X, z0=zz, func=func, t=t)
    n_fwd = len(calls.names)
    g = _grad_pattern(out.shape, 14).to(DEV, dtype)
    with monkeypatch.context() as m:
        _no_autograd(m)
        out.backward(g)
    backward = calls.names[n_fwd:]
    # the forward: the field, and the stage's one validation call (no paths, nothing launched)
    assert FIELD in calls.names[:n_fwd] and calls.names[:n_fwd].count(VJP) == 1
    assert FIELD not in backward and backward.count(VJP) > 0
    return X, func, z0, zz, t.tolist(), out, g, attempts.lists()


EXAMPLES_BARS = {F32: (2e-5, 2e-4), F64: (1e-9, 1e-9)}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp64"])
@pytest.mark.parametrize("control", CONTROLS)
def test_examples_call_replayed_by_the_oracle(control, dtype, monkeypatch):
    """cdeint(X, func, z0, X.interval)'s defaults: dopri5 with adjoint=True, rtol 1e-4, atol 1e-6.  The forward solve and
    every backward segment are replayed by the oracle (on the augmented field) from the package's own attempts: a(t0)
    and dL/dtheta within 2e-5 and 2e-4 in fp32 (kink rule), 1e-9 in fp64."""
    dt = {"fp32": F32, "fp64": F64}[dtype]
    with _variant(_variant_for((8, 3, 128), dt)):
        X, func, z0, zz, t_list, out, g, solves = _examples_call(monkeypatch, dt, control)
    rtol, atol = 1e-4, 1e-6
    assert len(solves) == 1 + len(t_list) - 1
    fc = _oracle(X, func, control, dt)
    what = "{} {}".format(control, dtype)
    replay = _check_host_attempts(solves[0], fc, rtol, atol, "examples forward " + what)
    want_out = AO.solve(fc, z0.double(), t_list, rtol, atol, replay=replay)[0]
    _report("examples call outputs vs replay | " + what, _global_err(out.movedim(-2, 0), want_out),
            2e-5 if dt == F32 else 1e-10)
    params = fc.params
    sizes = [p.numel() for p in params]
    n_z = z0.numel()
    ys, gys = _ys_for_oracle(out), g.double().movedim(-2, 0)

    def aug_s(s, v):
        z, a = v[:n_z].view(z0.shape), v[n_z:2 * n_z].view(z0.shape)
        f, gz, gp = fc.vjp(-s, z, a, params)
        return -torch.cat([x.reshape(-1) for x in [f, -gz] + [-p for p in gp]])

    a = gys[-1]
    gp = [torch.zeros(n, dtype=F64, device=DEV) for n in sizes]
    for seg, i in zip(solves[1:], range(len(t_list) - 1, 0, -1)):
        v0 = torch.cat([ys[i].reshape(-1), a.reshape(-1)] + gp)
        replay = _check_host_attempts(seg, aug_s, rtol, atol, "examples adjoint {} segment {}".format(what, i),
                                      part=lambda v: v[:n_z])
        v1 = AO.solve(aug_s, v0, [-t_list[i], -t_list[i - 1]], rtol, atol, replay=replay)[0][-1]
        a = v1[n_z:2 * n_z].view(z0.shape) + gys[i - 1]
        gp = list(torch.split(v1[2 * n_z:], sizes))
    bar_a, bar_p = EXAMPLES_BARS[dt]
    _check_paths("examples call a(t0) | " + what, zz.grad, a, bar_a, dt)
    for p, want in zip(func.parameters(), gp):
        _report("examples call dL/dtheta | " + what, _global_err(p.grad, want.view_as(p)), bar_p)


# ---- 5. exclusions keep their old route and their old bits ----------------------------------------------------------
def _run_adjoint(X, func, z0, t, method, step, params=None):
    zz = z0.clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    kwargs = {} if params is None else {"adjoint_params": tuple(params)}
    opts = {} if method == "dopri5" else {"method": method, "options": _options(step)}
    out = cde.cdeint(X, func, zz, t, **opts, **kwargs)
    out.backward(_grad_pattern(out.shape, 16).to(DEV, out.dtype))
    return [out.detach(), zz.grad] + [p.grad for p in func.parameters()] + [t.grad if t.requires_grad else None]


EXCLUSIONS = ["t_requires_grad", "coefficients", "decreasing_t", "32x8", "softplus"]


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["rk4", "dopri5"])
@pytest.mark.parametrize("case", EXCLUSIONS)
def test_exclusions_keep_the_old_route_and_bits(case, method, monkeypatch):
    shape = (32, 8, 128) if case == "32x8" else (8, 3, 128)
    X, func, z0 = _problem(*shape, F32, "cubic", 64)
    t = torch.tensor([0.0, 2.5, 6.0], dtype=F64)
    params = None
    if case == "softplus":
        torch.manual_seed(3)
        func = SoftplusMLP(8, 3, 128).to(DEV)
    if case == "t_requires_grad":
        t = t.clone().requires_grad_(True)
    if case == "decreasing_t":
        t = t.flip(0)
    if case == "coefficients":
        rows = X._rows().detach().clone().requires_grad_(True)
        X = cde.CubicSpline(rows)
        params = list(func.parameters()) + [rows]

    def run():
        return _run_adjoint(X, func, z0, t, method, 0.5, params)

    calls = _Calls(monkeypatch)
    new = run()
    assert VJP not in calls.names
    with monkeypatch.context() as m:
        m.setattr(solver, "_mlp_vjp", lambda *a: None)           # the autograd-per-stage backward, same forward
        old = run()
    for x, y in zip(new, old):
        assert (x is None and y is None) or torch.equal(x, y)


# ---- 6. full scale --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_scale_training_step(monkeypatch):
    """One rk4 step-1 adjoint=True training step at B = 65,536, L = 256, (8, 3, 128), against the autograd adjoint of
    the same call: dL/dtheta within 2e-4 and dL/dz0 per path within 1e-5 for all but 1 in 32.  The worst paths (where
    the two fp32 routes part at relu kinks) are held to the fp64 oracle instead: on the 8 worst, the kernels' route is
    no farther from it than twice the autograd route's distance (plus 1e-5)."""
    gen = torch.Generator().manual_seed(21)
    B, L = 65536, 256
    x = (torch.randn(B, L, 3, generator=gen) / 16).cumsum(1).to(DEV)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    del x
    func = _func(3, 8, 128, F32)
    z0 = torch.randn(B, 8, generator=gen).to(DEV)
    t = torch.tensor([0.0, float(L - 1)], dtype=F64)

    def step():
        zz = z0.clone().requires_grad_(True)
        for p in func.parameters():
            p.grad = None
        out = cde.cdeint(X, func, zz, t, adjoint=True, method="rk4", options={"step_size": 1.0})
        out[:, -1].sum().backward()
        return out.detach(), zz.grad, [p.grad.clone() for p in func.parameters()]

    calls = _Calls(monkeypatch)
    out, gz, gp = step()
    assert calls.names.count(VJP) == 1 + (L - 1) * 4                   # the validation call, then one per stage
    with monkeypatch.context() as m:
        m.setattr(solver, "_mlp_vjp", lambda *a: None)
        _o, wz, wp = step()
    for got, want in zip(gp, wp):
        _report("full scale dL/dtheta | rk4 B=65536", _global_err(got, want), 2e-4)
    errs = ((gz.double() - wz.double()).abs().amax(1) / wz.double().abs().amax(1)).cpu()
    _report("full scale dL/dz0 (all but 1 in 32) | rk4 B=65536", float(errs.sort().values[-(1 + B // 32)]), 1e-5)
    # kink accounting: the paths where the two fp32 routes part are relu-kink paths of a long fp32 solve -- against the
    # fp64 oracle of the same discrete solve, the kernels' route is no farther than the autograd route (within 2x)
    worst = errs.topk(8).indices.sort().values.to(DEV)
    rows = X._rows()[worst]
    fc = _oracle(cde.CubicSpline(rows), func, "cubic", F32)
    gys = torch.zeros(2, worst.numel(), 8, dtype=F64, device=DEV)
    gys[-1] = 1.0
    ref, _wp, _ = AO.fixed_adjoint(fc, _ys_for_oracle(out[worst]), gys, t.tolist(), "rk4", 1.0)
    e_new = float(((gz[worst].double() - ref).abs().amax(1) / ref.abs().amax(1)).max())
    e_old = float(((wz[worst].double() - ref).abs().amax(1) / ref.abs().amax(1)).max())
    print("full scale worst paths vs the fp64 oracle: kernels {:.2e}, autograd {:.2e}, between them {:.2e}".format(
        e_new, e_old, float(errs.max())))
    assert e_new <= 2 * e_old + 1e-5, (e_new, e_old)
