"""The fused fixed-step solve of the examples' MLP field (``tcde_cdeint_fixed_mlp``) on every kernel route, against an
fp64 oracle at the schedule, tile and control edges.

Routes: the wgmma kernel at hidden 32 / channels 8 / width 128 (variant 0), the CUDA-core kernel in fp32 and fp64 (auto
at 8 / 3 and 5 / 3, variant 1 at 32 / 8 and 16 / 4, where auto leaves the shape to the stage loop), each at widths 128
and 48.  Schedules: ``test_host_logic.FIXED_SCHEDULES``
on 40 knots.  Reference: ``odeint_port.odeint`` driving ``MlpCDE`` below -- ``adaptive_oracle.FuncCDE`` with the MLP as
its field -- in fp64 on fp64 copies of the kernel's own rounded inputs.  Bars are fractions of each path's own scale."""
import contextlib
import functools

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port
from test_host_logic import FIXED_SCHEDULES, fixed_schedule_knots
from torchcde_b200 import _lib, solver

pytestmark = pytest.mark.gpu
DEV = "cuda"
PATHS, LENGTH = 1000, 40
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-10}
CONTROLS = ["cubic", "linear"]
METHODS = ["rk4", "midpoint", "euler"]
SCHEDULES = list(FIXED_SCHEDULES)

# name: (hidden, channels, width, dtype, solve variant)
ROUTES = {"wgmma": (32, 8, 128, F32, 0)}
for _w in (128, 48):
    for _h, _c in ((32, 8), (8, 3), (5, 3), (16, 4)):
        # auto runs the CUDA-core kernel only at H <= 8 or H C <= 32 (where it beats the stage loop); variant 1 forces it
        _v = 0 if (_h <= 8 or _h * _c <= 32) else 1
        ROUTES["simt{}x{}w{}".format(_h, _c, _w)] = (_h, _c, _w, F32, _v)
        ROUTES["f64_{}x{}w{}".format(_h, _c, _w)] = (_h, _c, _w, F64, _v)
TILE_ROUTES = ["wgmma", "simt32x8w128"]

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[MLP field, worst of each check] " + "; ".join(
        "{}: {:.2e} (bar {:.0e})".format(k, e, b) for k, (e, b) in sorted(_WORST.items())))


def _report(what, err, bar):
    print("mlp {}: {:.2e} of scale (bar {:.0e})".format(what, err, bar))
    key = what.split(" |")[0]
    if err > _WORST.get(key, (-1.0, bar))[0]:
        _WORST[key] = (err, bar)
    assert err <= bar, (what, err, bar)


def _path_err(got, want):
    """max over paths (dim 0) of max |got - want| / max |want| on that path (NaN if got holds a NaN)."""
    got, want = got.detach().double(), want.detach().double().to(got.device)
    if want.numel() == 0:
        return 0.0
    dims = tuple(range(1, want.dim()))
    err = (got - want).abs().amax(dim=dims)
    return (err / want.abs().amax(dim=dims).clamp_min(1e-300)).max().item()


@contextlib.contextmanager
def _variant(v):
    _lib.call("tcde_set_solve_variant", v)
    try:
        yield
    finally:
        _lib.call("tcde_set_solve_variant", 0)


def _options(step):
    return {} if step is None else {"step_size": step}


def MlpCDE(control, knots, w1, b1, w2, b2, kind, time_dtype):
    """f(t, z) = tanh(W2 relu(W1 z + b1) + b2).view(H, C) @ dX/dt(t) in fp64: ``adaptive_oracle.FuncCDE`` with the MLP
    as its ``g``."""
    w1, b1, w2, b2 = (x.double() for x in (w1, b1, w2, b2))
    hidden = w1.size(1)

    def g(t, z):
        u = torch.relu(z @ w1.T + b1)
        return torch.tanh(u @ w2.T + b2).view(*z.shape[:-1], hidden, -1)

    return AO.FuncCDE(control, knots, g, kind, time_dtype)


class Func(torch.nn.Module):
    """example/time_series_classification.py:20-51's CDEFunc (the width a parameter)."""

    def __init__(self, input_channels, hidden_channels, width=128, bias=True):
        super().__init__()
        self.input_channels, self.hidden_channels = input_channels, hidden_channels
        self.linear1 = torch.nn.Linear(hidden_channels, width, bias=bias)
        self.linear2 = torch.nn.Linear(width, input_channels * hidden_channels, bias=bias)

    def forward(self, t, z):
        z = self.linear1(z)
        z = z.relu()
        z = self.linear2(z)
        z = z.tanh()
        return z.view(*z.shape[:-1], self.hidden_channels, self.input_channels)


# ---- problems --------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _inputs(hidden, channels, width, uneven):
    """fp32 inputs on the device: paths (random walk), knots (None: 0..39), Hermite coefficients, z0, and W1, b1, W2, b2
    in nn.Linear's default ranges."""
    gen = torch.Generator().manual_seed(131 * hidden + 7 * channels + width)
    x = (torch.randn(PATHS, LENGTH, channels, generator=gen, dtype=F64) / 4).cumsum(1).float()
    z0 = torch.randn(PATHS, hidden, generator=gen, dtype=F64).float()

    def uniform(shape, fan_in):
        return ((2 * torch.rand(*shape, generator=gen, dtype=F64) - 1) * fan_in ** -0.5).float().to(DEV)

    params = (uniform((width, hidden), hidden), uniform((width,), hidden), uniform((hidden * channels, width), width),
              uniform((hidden * channels,), width))
    knots = fixed_schedule_knots(True).to(DEV) if uneven else None
    x = x.to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots)
    return x, knots, coeffs, z0.to(DEV), params


def _control(src, knots, control):
    return cde.CubicSpline(src, t=knots) if control == "cubic" else cde.LinearInterpolation(src, t=knots)


def _times(sname):
    ts, step, uneven = FIXED_SCHEDULES[sname]
    if ts is None:
        return fixed_schedule_knots(uneven).double(), step
    return torch.tensor(ts, dtype=F32 if sname == "F4" else F64), step


def _case(hidden, channels, width, dtype, control, sname, batch=PATHS, bias=True):
    """(X, func, z0, t, step_size) of the first ``batch`` paths in ``dtype`` (fp64: the fp32 values, cast)."""
    x, knots, coeffs, z0, (w1, b1, w2, b2) = _inputs(hidden, channels, width, FIXED_SCHEDULES[sname][2])
    kt = None if knots is None else knots.to(dtype)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    func = Func(channels, hidden, width, bias=bias).to(device=DEV, dtype=dtype)
    with torch.no_grad():
        func.linear1.weight.copy_(w1)
        func.linear2.weight.copy_(w2)
        if bias:
            func.linear1.bias.copy_(b1)
            func.linear2.bias.copy_(b2)
    t, step = _times(sname)
    return _control(src, kt, control), func, z0[:batch].to(dtype), t, step


def _oracle_field(X, func, control, dtype):
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    rows = rows.reshape(-1, rows.size(-2), rows.size(-1))
    l1, l2 = func.linear1, func.linear2

    def bias(lin):
        return lin.bias.detach() if lin.bias is not None else torch.zeros(lin.out_features, device=DEV)

    return MlpCDE(rows.double(), X._t.detach().cpu(), l1.weight.detach(), bias(l1), l2.weight.detach(), bias(l2),
                  control, time_dtype=dtype)


_solves = {}


def _reference(hidden, channels, width, dtype, control, sname, method, bias=True):
    """The oracle's outputs (PATHS, n_out, H) in fp64 on the device, one solve per problem."""
    key = (hidden, channels, width, dtype, control, sname, method, bias)
    if key not in _solves:
        X, func, z0, t, step = _case(hidden, channels, width, dtype, control, sname, bias=bias)
        with torch.no_grad():
            ys = odeint_port.odeint(_oracle_field(X, func, control, dtype), z0.double(), t, method=method,
                                    options=_options(step))
        _solves[key] = ys.movedim(0, 1)
    return _solves[key]


def _refuse_loop(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("the generic stage loop served a kernel route")

    monkeypatch.setattr(solver, "_generic_solve_kernels", refuse)
    monkeypatch.setattr(solver, "_generic_solve", refuse)


def _forward(monkeypatch, X, func, z0, t, step, method, variant):
    """cdeint's no-grad forward under solve variant ``variant``; the fused kernel must serve it, not the stage loop."""
    _refuse_loop(monkeypatch)
    with _variant(variant), torch.no_grad():
        return cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))


def _offset_copy(x):
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    view = buf[1:].view(x.shape)
    view.copy_(x)
    assert view.data_ptr() % 16 != 0
    return view


def _misaligned_control(X, control):
    knots = None if X._default_knots else X._t
    if control == "cubic":
        return cde.CubicSpline(_offset_copy(X._rows()), t=knots)
    Y = cde.LinearInterpolation(X._coeffs, t=knots)
    Y._derivs = _offset_copy(Y._derivs)
    return Y


# ---- 1. the forward route table --------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sname", SCHEDULES)
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", list(ROUTES))
def test_forward_routes_match_the_oracle(route, control, sname, method, monkeypatch):
    hidden, channels, width, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, control, sname)
    want = _reference(hidden, channels, width, dtype, control, sname, method)
    out = _forward(monkeypatch, X, func, z0, t, step, method, variant)
    assert out.shape == want.shape and out.dtype == dtype
    assert torch.equal(out[:, 0], z0)
    _report("forward {} | {} {} {} {}".format("fp64" if dtype == F64 else "fp32", route, control, sname, method),
            _path_err(out, want), BAR[dtype])


def test_the_variants_run_distinct_kernels(monkeypatch):
    """The wgmma and CUDA-core kernels round differently: bit-equal outputs would mean the switch did nothing."""
    X, func, z0, t, step = _case(32, 8, 128, F32, "cubic", "F3")
    tc = _forward(monkeypatch, X, func, z0, t, step, "rk4", 0)
    assert not torch.equal(tc, _forward(monkeypatch, X, func, z0, t, step, "rk4", 1))
    assert torch.equal(tc, _forward(monkeypatch, X, func, z0, t, step, "rk4", 4))


# ---- 2. tiles, batch shapes, buffers ---------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("batch", [1, 63, 64, 65, 127, 128, 129, 257])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", TILE_ROUTES)
def test_forward_tile_edges_match_the_oracle(route, control, batch, method, monkeypatch):
    """Batches on both sides of 64 paths per warpgroup and 128 paths per CTA (both kernels)."""
    hidden, channels, width, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, control, "F3", batch)
    want = _reference(hidden, channels, width, dtype, control, "F3", method)[:batch]
    out = _forward(monkeypatch, X, func, z0, t, step, method, variant)
    assert out.shape == want.shape
    assert torch.equal(out[:, 0], z0)
    _report("tile edges | {} {} {} batch {}".format(route, control, method, batch), _path_err(out, want), BAR[dtype])


@pytest.mark.parametrize("route", ["wgmma", "simt32x8w128", "simt5x3w48", "f64_32x8w128"])
@pytest.mark.parametrize("control", CONTROLS)
def test_batch_dimensions_are_flattened_bit_for_bit(route, control, monkeypatch):
    hidden, channels, width, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, control, "F3", 100)
    src = X._rows() if control == "cubic" else X._coeffs
    knots = None if X._default_knots else X._t
    X4 = _control(src.view(4, 25, *src.shape[1:]), knots, control)
    flat = _forward(monkeypatch, X, func, z0, t, step, "rk4", variant)
    nested = _forward(monkeypatch, X4, func, z0.view(4, 25, hidden), t, step, "rk4", variant)
    assert nested.shape == (4, 25, t.numel(), hidden)
    assert torch.equal(nested.reshape(flat.shape), flat)


@pytest.mark.parametrize("route", ["wgmma", "simt8x3w128", "f64_32x8w128"])
def test_an_empty_batch(route, monkeypatch):
    hidden, channels, width, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, "cubic", "F3", 0)
    out = _forward(monkeypatch, X, func, z0, t, step, "rk4", variant)
    assert out.shape == (0, t.numel(), hidden) and out.dtype == dtype


def _served_by_the_loop(monkeypatch, variant, X, func, z0, t, step):
    """cdeint under ``variant`` where tcde_cdeint_fixed_mlp must refuse the problem: (output, refused calls, loop runs)."""
    refused, looped = [], []
    real_call, real_loop = _lib.call, solver._generic_solve_kernels

    def call(name, *args):
        try:
            return real_call(name, *args)
        except NotImplementedError:
            refused.append(name)
            raise

    def loop(*args, **kwargs):
        looped.append(True)
        return real_loop(*args, **kwargs)

    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(solver, "_generic_solve_kernels", loop)
    with _variant(variant), torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    monkeypatch.undo()
    return out, refused, looped


def _misaligned(X, z0, control, where):
    return (_misaligned_control(X, control), z0) if where == "control" else (X, _offset_copy(z0))


@pytest.mark.parametrize("where", ["control", "z0"])
@pytest.mark.parametrize("control", CONTROLS)
def test_misaligned_buffers_at_the_tensor_core_shape(control, where, monkeypatch):
    """Control rows or z0 at a 4-byte offset at 32 / 8 / 128: the wgmma kernel cannot take them and the CUDA-core kernel
    is slower than the stage loop there, so both auto and a forced variant 4 refuse and cdeint answers from its loop;
    a forced variant 1 runs the CUDA-core kernel, bit-equal to variant 1 on aligned buffers."""
    X, func, z0, t, step = _case(32, 8, 128, F32, control, "F3")
    Xm, zm = _misaligned(X, z0, control, where)
    want = _reference(32, 8, 128, F32, control, "F3", "rk4")
    for variant in (0, 4):
        out, refused, looped = _served_by_the_loop(monkeypatch, variant, Xm, func, zm, t, step)
        assert refused == ["tcde_cdeint_fixed_mlp"] and looped == [True]
        _report("stage loop after a refusal | {} {} v{}".format(control, where, variant), _path_err(out, want), BAR[F32])
    out = _forward(monkeypatch, Xm, func, zm, t, step, "rk4", 1)
    assert torch.equal(out, _forward(monkeypatch, X, func, z0, t, step, "rk4", 1))
    _report("misaligned | {} {} v1".format(control, where), _path_err(out, want), BAR[F32])


@pytest.mark.parametrize("where", ["control", "z0"])
@pytest.mark.parametrize("control", CONTROLS)
def test_misaligned_buffers_run_the_cuda_core_kernel(control, where, monkeypatch):
    """At 8 / 3 / 128 auto runs the CUDA-core kernel, which reads element by element: misaligned buffers give the bits of
    aligned ones."""
    X, func, z0, t, step = _case(8, 3, 128, F32, control, "F3")
    Xm, zm = _misaligned(X, z0, control, where)
    out = _forward(monkeypatch, Xm, func, zm, t, step, "rk4", 0)
    assert torch.equal(out, _forward(monkeypatch, X, func, z0, t, step, "rk4", 0))
    _report("misaligned | {} {} 8x3".format(control, where), _path_err(out, _reference(8, 3, 128, F32, control, "F3",
                                                                                         "rk4")), BAR[F32])


@pytest.mark.parametrize("route", ["simt16x4w128", "simt32x8w48", "f64_32x8w128", "f64_16x4w48"])
def test_auto_leaves_slow_cuda_core_shapes_to_the_stage_loop(route, monkeypatch):
    """Where the CUDA-core kernel is slower than the stage loop (H > 8 and H C > 32), auto refuses the shape and the
    loop answers within the bar; variant 1 still runs the kernel."""
    hidden, channels, width, dtype, variant = ROUTES[route]
    assert variant == 1
    X, func, z0, t, step = _case(hidden, channels, width, dtype, "cubic", "F3")
    want = _reference(hidden, channels, width, dtype, "cubic", "F3", "rk4")
    out, refused, looped = _served_by_the_loop(monkeypatch, 0, X, func, z0, t, step)
    assert refused == ["tcde_cdeint_fixed_mlp"] and looped == [True]
    _report("stage loop at a slow shape | {}".format(route), _path_err(out, want), BAR[dtype])


@pytest.mark.parametrize("route", ["wgmma", "simt32x8w128", "simt8x3w48", "f64_16x4w128"])
@pytest.mark.parametrize("control", CONTROLS)
def test_both_biases_absent(route, control, monkeypatch):
    hidden, channels, width, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, width, dtype, control, "F3", bias=False)
    want = _reference(hidden, channels, width, dtype, control, "F3", "rk4", bias=False)
    out = _forward(monkeypatch, X, func, z0, t, step, "rk4", variant)
    _report("no bias | {} {}".format(route, control), _path_err(out, want), BAR[dtype])


def test_the_3xtf32_variant_is_not_built_for_the_mlp(monkeypatch):
    X, func, z0, t, step = _case(32, 8, 128, F32, "cubic", "F3", 65)
    kern = solver.MlpFieldKernels(X, (func.linear1.weight, func.linear1.bias, func.linear2.weight, func.linear2.bias),
                                  z0)
    with _variant(3), pytest.raises(NotImplementedError):
        kern.solve(z0, t, "rk4", step)


# ---- 3. full scale ---------------------------------------------------------------------------------------------------
def test_full_scale_against_the_fp64_kernel(monkeypatch):
    """All 65,536 paths of a length-256 cubic control at (32, 8, 128), rk4 with step 1: the wgmma kernel within 1e-5 of
    each path's scale of the fp64 CUDA-core kernel on the same fp32-rounded inputs."""
    gen = torch.Generator().manual_seed(5)
    batch, length = 65536, 256
    x = (torch.randn(batch, length, 8, generator=gen) / 4).cumsum(1).to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    del x
    z0 = torch.randn(batch, 32, generator=gen).to(DEV)
    torch.manual_seed(6)
    func = Func(8, 32).to(DEV)
    t = torch.tensor([0.0, 100.0, 255.0])
    out = _forward(monkeypatch, cde.CubicSpline(coeffs), func, z0, t, 1.0, "rk4", 0)
    coeffs64 = coeffs.double()
    del coeffs
    want = _forward(monkeypatch, cde.CubicSpline(coeffs64), func.double(), z0.double(), t, 1.0, "rk4", 1)
    _report("full scale | 65,536 paths", _path_err(out, want), BAR[F32])


# ---- 4. recognition through cdeint -----------------------------------------------------------------------------------
class BenchField(torch.nn.Module):
    """bench.py's generic_mlp_field_rk4 workload."""

    def __init__(self):
        super().__init__()
        self.linear1 = torch.nn.Linear(8, 128)
        self.linear2 = torch.nn.Linear(128, 24)

    def forward(self, tt, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], 8, 3)


def _bench_problem():
    gen = torch.Generator().manual_seed(8)
    x = (torch.randn(300, 30, 3, generator=gen) / 4).cumsum(1).to(DEV)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    z0 = torch.randn(300, 8, generator=gen).to(DEV)
    return X, z0, torch.tensor([0.0, 12.5, 29.0])


def test_the_examples_and_the_benchmarks_fields_take_the_fused_route(monkeypatch):
    X, z0, t = _bench_problem()
    torch.manual_seed(9)
    for func in (Func(3, 8), BenchField()):
        func = func.to(DEV)
        out = _forward(monkeypatch, X, func, z0, t, 1.0, "rk4", 0)
        monkeypatch.undo()
        with torch.no_grad():
            loop = solver._generic_solve_kernels(X, func, z0, t, "rk4", 1.0, False)
        assert not torch.equal(out, loop)                       # a different kernel: not the stage loop's bits
        assert _path_err(out, loop) < 1e-5


def _variant_field(body):
    class Variant(BenchField):
        def forward(self, tt, z):
            return body(self, tt, z).view(*z.shape[:-1], 8, 3)
    return Variant()


REJECTED = {
    "softplus": lambda m, t, z: m.linear2(torch.nn.functional.softplus(m.linear1(z))).tanh(),
    "sigmoid": lambda m, t, z: m.linear2(torch.sigmoid(m.linear1(z))).tanh(),
    "no_tanh": lambda m, t, z: m.linear2(m.linear1(z).relu()),
    "depends_on_t": lambda m, t, z: m.linear2(m.linear1(z).relu()).tanh() * (1 + 0.01 * t),
    "scaled_output": lambda m, t, z: 2 * m.linear2(m.linear1(z).relu()).tanh(),
    "relu_after_tanh": lambda m, t, z: m.linear2(m.linear1(z).relu()).tanh().relu(),
}


@pytest.mark.parametrize("name", list(REJECTED))
def test_rejected_fields_run_the_stage_loop(name, monkeypatch):
    """Fields the probe rejects never reach tcde_cdeint_fixed_mlp: cdeint returns the stage loop's own result."""
    X, z0, t = _bench_problem()
    torch.manual_seed(10)
    func = _variant_field(REJECTED[name]).to(DEV)
    called = []
    real_call = _lib.call
    monkeypatch.setattr(_lib, "call", lambda n, *a: called.append(n) or real_call(n, *a))
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options={"step_size": 1.0})
        loop = solver._generic_solve_kernels(X, func, z0, t, "rk4", 1.0, False)
    assert "tcde_cdeint_fixed_mlp" not in called
    assert torch.equal(out, loop)


# ---- 5. gradients ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("control", CONTROLS)
def test_adjoint_forward_is_fused_and_backward_unchanged(control, method, monkeypatch):
    """adjoint=True: the outputs are those of the no-grad call bit for bit (the fused forward), and the autograd-per-stage
    backward gives dL/dz0 within 1e-5 and dL/dtheta within 2e-4 of the same call in fp64."""
    X, func, z0, t, step = _case(32, 8, 128, F32, control, "F3", 65)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    grads = {}
    for dtype in (F32, F64):
        knots = None if X._default_knots else X._t.double()
        Xd = X if dtype == F32 else _control((X._rows() if control == "cubic" else X._coeffs).double(), knots, control)
        fd = func if dtype == F32 else Func(8, 32).to(device=DEV, dtype=F64)
        if dtype == F64:
            fd.load_state_dict({k: v.double() for k, v in func.state_dict().items()})
        fd.zero_grad()
        zz = z0.to(dtype).clone().requires_grad_(True)
        out = cde.cdeint(Xd, fd, zz, t, adjoint=True, method=method, options=_options(step))
        if dtype == F32:
            assert torch.equal(out.detach(), plain)
        g = torch.randn(out.shape, generator=torch.Generator().manual_seed(3), dtype=F64).to(device=DEV, dtype=dtype)
        out.backward(g)
        grads[dtype] = [zz.grad] + [p.grad for p in fd.parameters()]
    _report("adjoint dL/dz0 | {} {}".format(control, method), _path_err(grads[F32][0], grads[F64][0]), 1e-5)
    for got, want in zip(grads[F32][1:], grads[F64][1:]):
        err = ((got.double() - want).abs().max() / want.abs().max()).item()
        _report("adjoint dL/dtheta | {} {}".format(control, method), err, 2e-4)


# ---- 6. the stage loop, with a field the probe rejects ---------------------------------------------------------------
class _SoftplusField(BenchField):
    def forward(self, tt, z):
        z = self.linear2(torch.nn.functional.softplus(self.linear1(z))).tanh()
        return z.view(*z.shape[:-1], 8, 3)


@pytest.mark.parametrize("method,step", [("rk4", 1.0), ("midpoint", 0.5), ("euler", 0.25)])
def test_generic_field_kernel_loop_and_cuda_graph(method, step):
    """The checks of test_gpu_round2's stage-loop test, with a softplus MLP (which the probe rejects, so the stage loop
    still serves it): kernel loop vs the torch-operator loop, CUDA graph vs kernel loop, a replay reads the new z0, and
    reversed time."""
    torch.manual_seed(0)
    x = torch.randn(64, 20, 3, device=DEV).cumsum(1) / 4
    func = _SoftplusField().to(DEV)
    z0 = torch.randn(64, 8, device=DEV)
    t = torch.tensor([0.0, 7.3, 19.0])
    for make in (lambda: cde.CubicSpline(cde.natural_cubic_coeffs(x)), lambda: cde.LinearInterpolation(x)):
        X = make()
        with torch.no_grad():
            fast = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options={"step_size": step})
            graph = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options={"step_size": step, "cuda_graph": True})
            again = cde.cdeint(X, func, z0 * 0.5, t, adjoint=False, method=method,
                               options={"step_size": step, "cuda_graph": True})
            half = cde.cdeint(X, func, z0 * 0.5, t, adjoint=False, method=method, options={"step_size": step})
            slow = solver._generic_solve(X, func, z0, t, method, step, False, True)
            direct = solver._generic_solve_kernels(X, func, z0, t, method, step, False)
        assert fast.shape == (64, 3, 8)
        assert torch.equal(fast, direct)
        assert torch.allclose(fast, slow, rtol=1e-5, atol=1e-5)
        assert torch.allclose(graph, fast, rtol=1e-6, atol=1e-6)
        assert torch.allclose(again, half, rtol=1e-6, atol=1e-6)
        t_rev = torch.tensor([19.0, 7.3, 0.0])
        with torch.no_grad():
            fast_rev = cde.cdeint(X, func, z0, t_rev, adjoint=False, method=method, options={"step_size": step})
            slow_rev = solver._generic_solve(X, func, z0, t_rev, method, step, False, True)
        assert torch.allclose(fast_rev, slow_rev, rtol=1e-5, atol=1e-5)
