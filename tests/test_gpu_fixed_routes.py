"""The fixed-step Runge-Kutta solve (rk4, midpoint, euler) on every kernel route, its stage dump and its three-launch
adjoint, against the fp64 oracle at the schedule, tile and control edges.

Routes: the wgmma kernel (variant 0), the 3xTF32 kernel (variant 3), the CUDA-core kernel at hidden 32 / channels 8
(variant 1) and at other shapes, and the fp64 kernel.  Schedules (``test_host_logic.FIXED_SCHEDULES``, 40 knots): one
clipped step, ``step_size=None``, several outputs inside one step, a zero-length and a 1e-4 last step, every rk4 stage on a
knot, uneven knots with steps longer than intervals, decreasing time.  Reference: ``odeint_port.odeint`` driving
``adaptive_oracle.LinearCDE`` in fp64 (torch's generic fp64 operators on the GPU, none of this package's kernels) on fp64
copies of the kernel's own rounded inputs, stage times rounded to the state dtype, one solve per (shape, dtype, control,
schedule, method) shared by every route; gradients by ``adaptive_oracle.fixed_adjoint``.  Bars are fractions of each
path's own scale (dL/dW, dL/db: of the tensor's scale)."""
import contextlib
import functools

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port
from test_host_logic import FIXED_SCHEDULES, fixed_schedule_knots
from torchcde_b200 import _lib, linear_field, solver
from torchcde_b200.linear_field import LinearFieldKernels

pytestmark = pytest.mark.gpu
DEV = "cuda"
PATHS, LENGTH = 1000, 40                 # 1,000 paths: a partial tile for both tensor-core kernels
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-10}
GRAD_BAR = {"z0": 1e-5, "w": 2e-4, "b": 2e-4}
CONTROLS = ["cubic", "linear"]
METHODS = ["rk4", "midpoint", "euler"]
SCHEDULES = list(FIXED_SCHEDULES)

# name: (hidden, channels, dtype, solve variant)
ROUTES = {
    "wgmma": (32, 8, F32, 0),             # the default: 2xFP16 warpgroup MMA
    "tf32": (32, 8, F32, 3),              # 3xTF32 mma.sync
    "simt": (32, 8, F32, 1),              # the CUDA-core kernel at the tensor-core shape
    "f64": (32, 8, F64, 0),
    "simt16x4": (16, 4, F32, 0), "simt5x3": (5, 3, F32, 0), "simt64x8": (64, 8, F32, 0),
    "simt16x4_f64": (16, 4, F64, 0), "simt5x3_f64": (5, 3, F64, 0), "simt64x4_f64": (64, 4, F64, 0),
}
TC_ROUTES = ["wgmma", "tf32", "simt"]

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[fixed routes, worst of each check] " + "; ".join(
        "{}: {:.2e} (bar {:.0e})".format(k, e, b) for k, (e, b) in sorted(_WORST.items())))


def _report(what, err, bar):
    print("fixed {}: {:.2e} of scale (bar {:.0e})".format(what, err, bar))
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


def _global_err(got, want):
    got, want = got.detach().double(), want.detach().double().to(got.device)
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


@contextlib.contextmanager
def _variant(v):
    _lib.call("tcde_set_solve_variant", v)
    try:
        yield
    finally:
        _lib.call("tcde_set_solve_variant", 0)


def _options(step):
    return {} if step is None else {"step_size": step}


# ---- problems --------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _inputs(hidden, channels, uneven):
    """The fp32 inputs of one problem shape on the device: paths (random walk, N(0, 1/16^2) increments), knots (None:
    the default 0..39), their Hermite coefficients, z0, and W, b in nn.Linear's default range."""
    gen = torch.Generator().manual_seed(31 * hidden + channels)
    x = (torch.randn(PATHS, LENGTH, channels, generator=gen, dtype=F64) / 16).cumsum(1).float()
    z0 = torch.randn(PATHS, hidden, generator=gen, dtype=F64).float()
    bound = hidden ** -0.5
    w = ((2 * torch.rand(hidden * channels, hidden, generator=gen, dtype=F64) - 1) * bound).float()
    b = ((2 * torch.rand(hidden * channels, generator=gen, dtype=F64) - 1) * bound).float()
    knots = fixed_schedule_knots(True).to(DEV) if uneven else None
    x = x.to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots)
    return x, knots, coeffs, z0.to(DEV), w.to(DEV), b.to(DEV)


def _control(src, knots, control):
    return cde.CubicSpline(src, t=knots) if control == "cubic" else cde.LinearInterpolation(src, t=knots)


def _times(sname):
    """(t on the CPU, step_size): t in float64, F4's in float32 (the zero-length last step), F2's = every knot."""
    ts, step, uneven = FIXED_SCHEDULES[sname]
    if ts is None:
        return fixed_schedule_knots(uneven).double(), step
    return torch.tensor(ts, dtype=F32 if sname == "F4" else F64), step


def _case(hidden, channels, dtype, control, sname, batch=PATHS, bias=True):
    """(X, func, z0, t, step_size) of the first ``batch`` paths in ``dtype`` (fp64: the fp32 values, cast).  The cubic
    control takes the fp32 Hermite coefficients, the linear one the knot values (it forms its own slopes)."""
    x, knots, coeffs, z0, w, b = _inputs(hidden, channels, FIXED_SCHEDULES[sname][2])
    kt = None if knots is None else knots.to(dtype)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    func = cde.LinearVectorField(hidden, channels, bias=bias).to(device=DEV, dtype=dtype)
    with torch.no_grad():
        func.linear.weight.copy_(w)
        if bias:
            func.linear.bias.copy_(b)
    t, step = _times(sname)
    return _control(src, kt, control), func, z0[:batch].to(dtype), t, step


def _oracle_field(X, func, control, dtype):
    """adaptive_oracle.LinearCDE on fp64 copies of the kernel's inputs: the Hermite rows or the knot values, the knots
    (in the control's dtype, then widened exactly), W and b (zero without bias); stage times rounded to ``dtype``."""
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    rows = rows.reshape(-1, rows.size(-2), rows.size(-1))
    w = func.linear.weight.detach()
    b = func.linear.bias.detach() if func.linear.bias is not None else torch.zeros(w.size(0), device=w.device)
    return AO.LinearCDE(rows.double(), X._t.detach().cpu(), w.double(), b.double(), control, time_dtype=dtype)


class _Recording:
    """The oracle field, keeping the state every stage is evaluated at (odeint_port calls it once per stage, in order)."""

    def __init__(self, field):
        self.field, self.inputs = field, []

    def __call__(self, t, y):
        self.inputs.append(y)
        return self.field(t, y)


def _solve_oracle(hidden, channels, dtype, control, sname, method, record):
    X, func, z0, t, step = _case(hidden, channels, dtype, control, sname)
    field = _Recording(_oracle_field(X, func, control, dtype))
    with torch.no_grad():
        ys = odeint_port.odeint(field, z0.double(), t, method=method, options=_options(step))
    return ys.movedim(0, 1), (field.inputs if record else None)


_solves = {}                              # one oracle solve per (shape, dtype, control, schedule, method)


def _reference(hidden, channels, dtype, control, sname, method):
    """The oracle's outputs (PATHS, n_out, H) in fp64 on the device."""
    key = (hidden, channels, dtype, control, sname, method)
    if key not in _solves:
        _solves[key] = _solve_oracle(hidden, channels, dtype, control, sname, method, False)[0]
    return _solves[key]


@functools.lru_cache(maxsize=2)
def _stage_reference(control, sname, method):
    """(outputs, the input of every stage in order) of the 32 / 8 fp32 problem: what the stage dump must hold."""
    return _solve_oracle(32, 8, F32, control, sname, method, True)


def _forward(monkeypatch, X, func, z0, t, step, method, variant):
    """cdeint's forward under solve variant ``variant``; the fused kernel must serve it, not the stage loop."""
    def refuse(*args, **kwargs):
        raise AssertionError("the generic stage loop served a kernel route")

    monkeypatch.setattr(solver, "_generic_solve_kernels", refuse)
    monkeypatch.setattr(solver, "_generic_solve", refuse)
    with _variant(variant), torch.no_grad():
        return cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))


def _offset_copy(x):
    """A copy of ``x`` whose data starts one element (4 or 8 bytes) past a 16-byte boundary."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    view = buf[1:].view(x.shape)
    view.copy_(x)
    assert view.data_ptr() % 16 != 0
    return view


def _misaligned_control(X, control):
    """The same control with its kernel rows (Hermite rows / slopes) in misaligned storage."""
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
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, dtype, control, sname)
    want = _reference(hidden, channels, dtype, control, sname, method)
    out = _forward(monkeypatch, X, func, z0, t, step, method, variant)
    assert out.shape == want.shape and out.dtype == dtype
    assert torch.equal(out[:, 0], z0)
    _report("forward {} | {} {} {} {}".format("fp64" if dtype == F64 else "fp32", route, control, sname, method),
            _path_err(out, want), BAR[dtype])


# ---- 2. tile edges ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sname", ["F3", "F8"])
@pytest.mark.parametrize("batch", [1, 63, 64, 65, 127, 128, 129, 257])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", TC_ROUTES)
def test_forward_tile_edges_match_the_oracle(route, control, batch, sname, method, monkeypatch):
    """Batches on both sides of 64 paths per warpgroup (wgmma) and 128 paths per CTA (3xTF32)."""
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, dtype, control, sname, batch)
    want = _reference(hidden, channels, dtype, control, sname, method)[:batch]
    out = _forward(monkeypatch, X, func, z0, t, step, method, variant)
    assert out.shape == want.shape and out.dtype == dtype
    assert torch.equal(out[:, 0], z0)
    _report("tile edges | {} {} {} {} batch {}".format(route, control, sname, method, batch), _path_err(out, want),
            BAR[dtype])


# ---- 3. the variant switch -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("control", CONTROLS)
def test_the_variants_run_distinct_kernels(control, monkeypatch):
    """wgmma, 3xTF32 and the CUDA-core kernel round differently: bit-equal outputs would mean the switch did nothing."""
    outs = {}
    for route in TC_ROUTES:
        X, func, z0, t, step = _case(32, 8, F32, control, "F3")
        outs[route] = _forward(monkeypatch, X, func, z0, t, step, "rk4", ROUTES[route][3])
    for a, b in (("wgmma", "tf32"), ("wgmma", "simt"), ("tf32", "simt")):
        assert not torch.equal(outs[a], outs[b]), (a, b)


# ---- 4. alignment and batch shape ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("where", ["control", "z0"])
@pytest.mark.parametrize("control", CONTROLS)
def test_misaligned_buffers_run_the_cuda_core_kernel(control, where, dtype, monkeypatch):
    """Control rows or z0 at a 4-byte (fp32) / 8-byte (fp64) offset: auto selects the CUDA-core kernel, which reads them
    element by element; its fp32 output is bit-equal to variant 1 on aligned buffers."""
    X, func, z0, t, step = _case(32, 8, dtype, control, "F3")
    Xm, zm = (_misaligned_control(X, control), z0) if where == "control" else (X, _offset_copy(z0))
    out = _forward(monkeypatch, Xm, func, zm, t, step, "rk4", 0)
    assert torch.equal(out[:, 0], z0)
    _report("misaligned | {} {} {}".format(control, where, dtype), _path_err(out, _reference(32, 8, dtype, control,
                                                                                           "F3", "rk4")), BAR[dtype])
    if dtype == F32:
        assert torch.equal(out, _forward(monkeypatch, X, func, z0, t, step, "rk4", 1))


@pytest.mark.parametrize("variant", [3, 4])
@pytest.mark.parametrize("where", ["control", "z0"])
@pytest.mark.parametrize("control", CONTROLS)
def test_forced_tensor_core_variant_refuses_misaligned_buffers(control, where, variant, monkeypatch):
    """A forced tensor-core variant cannot take misaligned buffers: the kernel call raises NotImplementedError and
    cdeint answers from its stage loop instead, still within the bar."""
    X, func, z0, t, step = _case(32, 8, F32, control, "F3")
    if where == "control":
        X = _misaligned_control(X, control)
    else:
        z0 = _offset_copy(z0)
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
    assert refused == ["tcde_cdeint_fixed_linear"] and looped == [True]
    _report("stage loop after a refusal | {} {} v{}".format(control, where, variant),
            _path_err(out, _reference(32, 8, F32, control, "F3", "rk4")), BAR[F32])


@pytest.mark.parametrize("route", ["wgmma", "tf32", "simt", "f64", "simt5x3"])
@pytest.mark.parametrize("control", CONTROLS)
def test_batch_dimensions_are_flattened_bit_for_bit(route, control, monkeypatch):
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, dtype, control, "F3", 100)
    src = X._rows() if control == "cubic" else X._coeffs
    knots = None if X._default_knots else X._t
    X4 = _control(src.view(4, 25, *src.shape[1:]), knots, control)
    flat = _forward(monkeypatch, X, func, z0, t, step, "rk4", variant)
    nested = _forward(monkeypatch, X4, func, z0.view(4, 25, hidden), t, step, "rk4", variant)
    assert nested.shape == (4, 25, t.numel(), hidden)
    assert torch.equal(nested.reshape(flat.shape), flat)


@pytest.mark.parametrize("route", ["wgmma", "tf32", "simt", "f64", "simt5x3"])
@pytest.mark.parametrize("control", CONTROLS)
def test_an_empty_batch(route, control, monkeypatch):
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, dtype, control, "F3", 0)
    out = _forward(monkeypatch, X, func, z0, t, step, "rk4", variant)
    assert out.shape == (0, t.numel(), hidden) and out.dtype == dtype


# ---- 5. the stage dump -----------------------------------------------------------------------------------------------
GUARD_ROWS = 128                          # one 3xTF32 CTA of paths: where a partial tile's masked writes would land


def _guarded(shape, rows, dtype):
    """A NaN-filled tensor of ``shape`` followed by ``rows`` NaN rows of 32 values: (tensor, guard)."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + rows * 32,), float("nan"), dtype=dtype, device=DEV)
    return buf[:n].view(shape), buf[n:]


def _fixed_solve(kernels, z0, t, step, method, dump=None):
    sched, (_floats, _ints, v) = linear_field._schedules.get(t, kernels.knots, kernels.n_rows, method, step,
                                                              kernels.dtype, kernels.device)
    out, guard = _guarded((z0.size(0), sched.n_out, kernels.hidden), GUARD_ROWS, kernels.dtype)
    kernels._fixed(sched, v, kernels.w, kernels.b, z0, out, dump)
    return sched, out, guard


def _dump_buffer(kernels, z0, t, step, method):
    sched = linear_field._schedules.get(t, kernels.knots, kernels.n_rows, method, step, kernels.dtype,
                                        kernels.device)[0]
    return _guarded((sched.n_steps * sched.n_stages, z0.size(0), kernels.hidden), GUARD_ROWS, kernels.dtype)


DUMP_CASES = [(r, m, c, s, b) for r in ("wgmma", "tf32") for m in METHODS for c in CONTROLS
              for s in ("F3", "F4", "F6", "F8") for b in (1, 65, 129, 1000)]


@pytest.mark.parametrize("route,method,control,sname,batch", DUMP_CASES)
def test_stage_dump_holds_the_oracle_stage_inputs(route, method, control, sname, batch):
    """tcde_cdeint_fixed_linear_stages: the same output bits as the plain solve, and slot s = the input of stage s
    (step-major, Runge-Kutta stage minor) on every path; nothing written past the last path."""
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, step = _case(hidden, channels, dtype, control, sname, batch)
    kernels = LinearFieldKernels(X, func.linear.weight, func.linear.bias, z0)
    dump, dump_guard = _dump_buffer(kernels, z0, t, step, method)
    with _variant(variant), torch.no_grad():
        _s, plain, _g = _fixed_solve(kernels, z0, t, step, method)
        _s, out, out_guard = _fixed_solve(kernels, z0, t, step, method, dump)
    assert torch.equal(out, plain)
    assert out_guard.isnan().all() and dump_guard.isnan().all()
    _want, inputs = _stage_reference(control, sname, method)
    assert len(inputs) == dump.size(0)
    worst = max(_path_err(dump[e], inputs[e][:batch]) for e in range(dump.size(0)))
    _report("stage dump | {} {} {} {} batch {}".format(route, method, control, sname, batch), worst, BAR[F32])


@pytest.mark.parametrize("case", ["cuda_core", "fp64", "16x4", "16x4_tf32", "misaligned_wgmma", "misaligned_tf32"])
def test_stage_dump_refusals(case):
    """Only the fp32 tensor-core kernels at 32 / 8 write a stage dump, into 16-byte aligned memory; everything else is
    TCDE_ERR_UNSUPPORTED (NotImplementedError), so the adjoint falls back instead of reading a dump nobody wrote."""
    route = {"cuda_core": "simt", "fp64": "f64", "16x4": "simt16x4", "16x4_tf32": "simt16x4"}.get(case, "wgmma")
    hidden, channels, dtype, variant = ROUTES[route]
    variant = 3 if case.endswith("tf32") else variant
    X, func, z0, t, step = _case(hidden, channels, dtype, "cubic", "F3", 65)
    kernels = LinearFieldKernels(X, func.linear.weight, func.linear.bias, z0)
    dump, _guard = _dump_buffer(kernels, z0, t, step, "rk4")
    if case.startswith("misaligned"):
        dump = _offset_copy(dump)
    with _variant(variant), torch.no_grad(), pytest.raises(NotImplementedError):
        _fixed_solve(kernels, z0, t, step, "rk4", dump)


# ---- 6. the three-launch adjoint -------------------------------------------------------------------------------------
def _pattern(name, shape, n_out, hidden):
    gen = torch.Generator().manual_seed(7)
    n = 1
    for s in shape:
        n *= s
    g = torch.randn(n, n_out, hidden, generator=gen, dtype=F64)
    if name == "last_output":
        g[:, :-1] = 0
    elif name == "odd_paths_zero":
        g[1::2] = 0
    elif name == "first_output":
        g[:, 1:] = 0
    elif name == "tiny":
        g *= 2.0 ** -60
    elif name == "huge":
        g *= 2.0 ** 60
    return g.float().to(DEV).view(*shape, n_out, hidden)


def _run_adjoint(monkeypatch, X, func, z0, t, step, method, g, route):
    """cdeint(adjoint=True) and one backward with output gradients g: (dL/dz0, per segment whether the three-launch
    route served it).  ``route="per-stage"``: the three-launch route is declined, the per-stage kernel loop runs."""
    used = []
    real = solver._kernel_vjp

    def probe(*args, **kwargs):
        st = real(*args, **kwargs)
        inner = st.segment

        def segment(*sa, **sk):
            res = None if route == "per-stage" else inner(*sa, **sk)
            used.append(res is not None)
            return res
        st.segment = segment
        return st

    monkeypatch.setattr(solver, "_kernel_vjp", probe)
    zz = z0.detach().clone().requires_grad_(True)
    out = cde.cdeint(X, func, zz, t, adjoint=True, method=method, options=_options(step))
    out.backward(g)
    return zz.grad, used


_adjoints = {}                            # one oracle backward per problem, shared by the two routes


def _oracle_adjoint(key, X, func, z0, t, step, method, g, control):
    if key not in _adjoints:
        field = _oracle_field(X, func, control, F32)
        hidden = z0.size(-1)
        with torch.no_grad():
            ys = odeint_port.odeint(field, z0.detach().reshape(-1, hidden).double(), t, method=method,
                                    options=_options(step))
            gys = g.detach().reshape(-1, t.numel(), hidden).movedim(1, 0).double()
            _adjoints[key] = AO.fixed_adjoint(field, ys, gys, t.tolist(), method, step)
    return _adjoints[key]


def _adjoint_case(monkeypatch, control, sname, method, batch, route, roles="wb", pattern="dense", shape=None,
                  misaligned=False):
    X, func, z0, t, step = _case(32, 8, F32, control, sname, batch, bias=roles != "no_bias")
    lin = func.linear
    if roles == "w":
        lin.bias.requires_grad_(False)
    elif roles == "b":
        lin.weight.requires_grad_(False)
    shape = shape or (batch,)
    g = _pattern(pattern, shape, t.numel(), 32)
    Xr, zr = X, z0
    if len(shape) > 1:
        src = X._rows() if control == "cubic" else X._coeffs
        Xr = _control(src.view(*shape, *src.shape[1:]), None if X._default_knots else X._t, control)
        zr = z0.view(*shape, 32)
    if misaligned:
        Xr = _misaligned_control(Xr, control)
    gz, used = _run_adjoint(monkeypatch, Xr, func, zr, t, step, method, g, route)
    key = (control, sname, method, batch, roles == "no_bias", pattern)
    wz, ww, wb = _oracle_adjoint(key, X, func, z0, t, step, method, g, control)
    got = {"z0": gz.reshape(-1, 32)}
    want = {"z0": wz, "w": ww, "b": wb}
    for name, p in (("w", lin.weight), ("b", lin.bias)):
        if p is not None and p.requires_grad:
            got[name] = p.grad
        elif p is not None:
            assert p.grad is None
    return got, want, used, g, t.numel()


def _check_grads(what, got, want):
    for name, g in got.items():
        err = _path_err(g, want[name]) if name == "z0" else _global_err(g, want[name])
        _report("adjoint dL/d{} | {}".format(name, what), err, GRAD_BAR[name])


ADJ_ROUTES = ["three-launch", "per-stage"]
ADJ_CASES = [(c, s, m, b, r) for c in CONTROLS for s in ("F2", "F3", "F6") for m in METHODS for b in (1, 64, 65, 129)
             for r in ADJ_ROUTES]


@pytest.mark.parametrize("control,sname,method,batch,route", ADJ_CASES)
def test_adjoint_routes_match_the_oracle(control, sname, method, batch, route, monkeypatch):
    got, want, used, _g, n_out = _adjoint_case(monkeypatch, control, sname, method, batch, route)
    assert used == [route == "three-launch"] * (n_out - 1)
    _check_grads("{} {} {} {} batch {}".format(route, control, sname, method, batch), got, want)


@pytest.mark.parametrize("route", ADJ_ROUTES)
@pytest.mark.parametrize("roles", ["wb", "w", "b", "no_bias"])
@pytest.mark.parametrize("control", CONTROLS)
def test_adjoint_parameter_roles(control, roles, route, monkeypatch):
    """W and b, W only (a null grad_bias), b only (a null grad_weight) and a field without bias, at F3."""
    got, want, used, _g, n_out = _adjoint_case(monkeypatch, control, "F3", "rk4", 65, route, roles=roles)
    assert used == [route == "three-launch"] * (n_out - 1)
    _check_grads("{} {} roles {}".format(route, control, roles), got, want)


@pytest.mark.parametrize("route", ADJ_ROUTES)
@pytest.mark.parametrize("pattern", ["last_output", "odd_paths_zero", "tiny", "huge", "first_output"])
@pytest.mark.parametrize("control", CONTROLS)
def test_adjoint_gradient_patterns(control, pattern, route, monkeypatch):
    """Output gradients on the last output only, zero on odd paths, scaled by 2^-60 / 2^60 (relative bars), or on output
    0 only (which is z0 itself: dL/dz0 = g[:, 0] and no parameter gradient, bit for bit), at F3."""
    got, want, used, g, n_out = _adjoint_case(monkeypatch, control, "F3", "rk4", 65, route, pattern=pattern)
    assert used == [route == "three-launch"] * (n_out - 1)
    if pattern == "first_output":
        assert torch.equal(got["z0"], g[:, 0])
        assert not got["w"].any() and not got["b"].any()
        return
    if pattern == "odd_paths_zero":
        assert not got["z0"][1::2].any()                      # paths are independent
    _check_grads("{} {} pattern {}".format(route, control, pattern), got, want)


@pytest.mark.parametrize("route", ADJ_ROUTES)
@pytest.mark.parametrize("control", CONTROLS)
def test_adjoint_multi_dimensional_batch(control, route, monkeypatch):
    got, want, used, _g, n_out = _adjoint_case(monkeypatch, control, "F3", "rk4", 65, route, shape=(5, 13))
    assert used == [route == "three-launch"] * (n_out - 1)
    _check_grads("{} {} batch (5, 13)".format(route, control), got, want)


@pytest.mark.parametrize("control", CONTROLS)
def test_adjoint_with_a_misaligned_control_runs_per_stage(control, monkeypatch):
    """The tensor-core solve refuses misaligned control rows, so every segment declines the three-launch route and the
    per-stage kernel loop serves the whole backward."""
    got, want, used, _g, n_out = _adjoint_case(monkeypatch, control, "F3", "rk4", 65, "three-launch", misaligned=True)
    assert used == [False] * (n_out - 1)
    _check_grads("misaligned {}".format(control), got, want)
