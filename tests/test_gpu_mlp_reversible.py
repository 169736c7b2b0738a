"""cdeint(backend="torchsde", method="reversible_heun") of the examples' MLP field on its CUDA-core kernels: the forward
(tcde_cdeint_reversible_heun_mlp) and its checkpoints against the fp64 oracle, the segment backward
(tcde_reversible_heun_mlp_backward_segment + tcde_mlp_field_param_grads per segment) against fp64 autograd through the
oracle, the launches each takes, the refusals that keep the torch-operator route, determinism and memory.

References are fp64 copies of the kernel's own inputs run through oracle/reversible_oracle.py; bars are fractions of each
path's own scale.  fp32 gradients: the kink rule of test_gpu_mlp_backprop (a path whose dL/dz0 misses the bar sits on a
ReLU kink the fp32 forward crossed on the other side; at most 1/32 of the paths are set aside, their output gradients
zeroed, and everything is compared again); fp64 sets no path aside."""
import contextlib
import functools

import pytest
import torch

import torchcde_b200 as cde
from oracle import reversible_oracle as R
from test_gpu_reversible import CONTROLS, LENGTH, PATHS, SCHEDULES, STRIDE, _path_err, _variant
from torchcde_b200 import _lib, reversible
from torchcde_b200.mlp_field import MlpFieldKernels

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-10}
GRAD_BAR = {F32: {"z0": 1e-5, "w": 2e-4}, F64: {"z0": 1e-9, "w": 1e-9}}
KINK_BAR = 1e-2
FWD, SEG, PG = "tcde_cdeint_reversible_heun_mlp", "tcde_reversible_heun_mlp_backward_segment", "tcde_mlp_field_param_grads"
_WORST = {}

# name: (hidden, channels, width, solve variant)
SHAPES = {
    "examples": (8, 3, 128, 0),
    "odd": (5, 3, 37, 0),
    "unit": (1, 1, 1, 0),
    "hm32": (16, 2, 48, 1),              # hidden > 8: the HM = 32 kernels, forced by variant 1
}


class Func(torch.nn.Module):
    """The examples' field: Linear(H, W) -> ReLU -> Linear(W, H C) -> tanh, viewed (H, C)."""

    def __init__(self, hidden, channels, width, bias=True, act=torch.relu):
        super().__init__()
        self.linear1 = torch.nn.Linear(hidden, width, bias=bias)
        self.linear2 = torch.nn.Linear(width, hidden * channels, bias=bias)
        self.hidden, self.channels, self.act = hidden, channels, act

    def forward(self, t, z):
        return torch.tanh(self.linear2(self.act(self.linear1(z)))).view(*z.shape[:-1], self.hidden, self.channels)


@functools.lru_cache(maxsize=None)
def _inputs(hidden, channels, width, uneven):
    """fp32 inputs of one shape: random-walk paths, knots (None: 0..LENGTH-1), Hermite coefficients, z0, the MLP."""
    gen = torch.Generator().manual_seed(131 * hidden + 7 * channels + width)
    x = (torch.randn(PATHS, LENGTH, channels, generator=gen, dtype=F64) / 16).cumsum(1).float()
    z0 = torch.randn(PATHS, hidden, generator=gen, dtype=F64).float()

    def uniform(shape, fan_in):
        return ((2 * torch.rand(*shape, generator=gen, dtype=F64) - 1) * fan_in ** -0.5).float().to(DEV)

    params = (uniform((width, hidden), hidden), uniform((width,), hidden), uniform((hidden * channels, width), width),
              uniform((hidden * channels,), width))
    knots = None
    if uneven:
        widths = 0.6 + 0.8 * torch.rand(LENGTH - 1, generator=gen, dtype=F64)
        knots = torch.cat([torch.zeros(1, dtype=F64), widths.cumsum(0)]).float().to(DEV)
    x = x.to(DEV)
    return x, knots, cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots), z0.to(DEV), params


def _case(shape, dtype, control, sname, batch=PATHS, bias=True):
    """(X, func, z0, t, dt) of the first ``batch`` paths in ``dtype`` (fp64: the fp32 values, cast)."""
    hidden, channels, width, _v = SHAPES[shape] if isinstance(shape, str) else shape
    ts, dt, t_dtype, uneven = SCHEDULES[sname]
    x, knots, coeffs, z0, (w1, b1, w2, b2) = _inputs(hidden, channels, width, uneven)
    kt = None if knots is None else knots.to(dtype)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    X = cde.CubicSpline(src, t=kt) if control == "cubic" else cde.LinearInterpolation(src, t=kt)
    func = Func(hidden, channels, width, bias=bias).to(device=DEV, dtype=dtype)
    with torch.no_grad():
        func.linear1.weight.copy_(w1)
        func.linear2.weight.copy_(w2)
        if bias:
            func.linear1.bias.copy_(b1)
            func.linear2.bias.copy_(b2)
    return X, func, z0[:batch].to(dtype), torch.tensor(ts, dtype=t_dtype), dt


def _oracle_field(X, func):
    """R's drift on fp64 copies of the kernel's inputs (the control's rows, W1, b1, W2, b2; the knots in the control's
    dtype, as _interpret_t locates a time).  Returns (f, [parameter leaves that require grad])."""
    leaves = [p.detach().double().cpu().requires_grad_(True) for p in func.parameters()]
    w1, w2 = leaves[0], leaves[-2] if len(leaves) == 4 else leaves[1]
    b1, b2 = (leaves[1], leaves[3]) if len(leaves) == 4 else (None, None)
    knots = X._t.detach().cpu()
    cubic = isinstance(X, cde.CubicSpline)
    rows = (X._rows() if cubic else X._derivs).detach().double().cpu()
    hidden = func.hidden

    def f(t, z):
        dx = R.cubic_derivative(rows, knots, t) if cubic else R.linear_derivative(rows, knots, t)
        m = torch.tanh(torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(z, w1, b1)), w2, b2))
        return (m.view(*z.shape[:-1], hidden, -1) @ dx.unsqueeze(-1)).squeeze(-1)

    return f, leaves


class _Calls:
    """The names of the library calls cdeint makes and the library serves (a refused call raises and is not listed; the
    module probe's and shape check's own calls are left out)."""

    def __init__(self, monkeypatch):
        self.names = []
        orig = _lib.call

        def spy(name, *args):
            rc = orig(name, *args)
            if "mlp" in name or "reversible" in name or "vjp" in name:
                self.names.append(name)
            return rc

        monkeypatch.setattr(_lib, "call", spy)


def _no_autograd(monkeypatch):
    def refuse(self, *args):
        raise AssertionError("per-step autograd served the MLP kernel route")

    monkeypatch.setattr(reversible._Problem, "autograd_vjp", refuse)


def _cdeint(X, func, z0, t, dt, **kw):
    return cde.cdeint(X, func, z0, t.to(DEV), backend="torchsde", method="reversible_heun", dt=dt, **kw)


# ---- the forward -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sname", list(SCHEDULES))
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_forward_matches_the_oracle(monkeypatch, shape, dtype, control, sname):
    X, func, z0, t, dt = _case(shape, dtype, control, sname)
    calls = _Calls(monkeypatch)

    def refuse(self, *args):
        raise AssertionError("the torch-operator solve served the MLP kernel route")

    monkeypatch.setattr(reversible._Problem, "torch_forward", refuse)
    with _variant(SHAPES[shape][3]), torch.no_grad():
        out = _cdeint(X, func, z0, t, dt)
    assert calls.names == [FWD], calls.names
    f, _ = _oracle_field(X, func)
    with torch.no_grad():
        ys, _rec = R.integrate(f, z0.double().cpu(), t, dt)
    err = _path_err(out, ys.movedim(0, 1))
    _WORST[("forward", dtype)] = max(_WORST.get(("forward", dtype), 0.0), err)
    print("mlp reversible forward {} {} {} {}: {:.2e} (worst {:.2e})".format(shape, dtype, control, sname, err,
                                                                            _WORST[("forward", dtype)]))
    assert err <= BAR[dtype], err
    assert torch.equal(out[:, 0], z0)


@pytest.mark.parametrize("shape", ["examples", "odd", "hm32"])
@pytest.mark.parametrize("sname", ["S3", "S4", "S5", "S6"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_checkpoints_match_the_oracle_states(shape, sname, dtype):
    X, func, z0, t, dt = _case(shape, dtype, "cubic", sname)
    params = tuple(p for p in (func.linear1.weight, func.linear1.bias, func.linear2.weight, func.linear2.bias))
    with _variant(SHAPES[shape][3]), torch.no_grad():
        problem = reversible._Problem(X, func, z0, t.to(DEV), dt, MlpFieldKernels(X, params, z0), params)
        out, ckpts = problem.kernel_forward(z0, keep_checkpoints=True)
        bare, _ = problem.kernel_forward(z0, keep_checkpoints=False)
        plain = _cdeint(X, func, z0, t, dt)
    assert torch.equal(out, bare) and torch.equal(out, plain)
    with _variant(SHAPES[shape][3]):
        y0 = z0.clone().requires_grad_(True)
        graded = _cdeint(X, func, y0, t, dt)
    assert torch.equal(graded.detach(), out)
    f, _ = _oracle_field(X, func)
    with torch.no_grad():
        _ys, rec = R.integrate(f, z0.double().cpu(), t, dt)
    n_steps = problem.sched.n_steps
    steps = sorted(k for k in ckpts if isinstance(k, int))
    assert steps == sorted(set(list(range(0, n_steps, STRIDE)) + [n_steps]))
    bar = 2e-5 if dtype == F32 else BAR[dtype]        # y, z and f, each to its own per-path scale
    for step in steps:
        for got, want in zip(ckpts[step], rec["states"][step]):
            assert _path_err(got, want) <= bar, (step, _path_err(got, want))


# ---- the backward ------------------------------------------------------------------------------------------------------
PATTERNS = ["dense", "last", "first", "boundaries"]
ROLES = {"all": None, "z0_w2": ("linear2.weight",), "biases": ("linear1.bias", "linear2.bias"), "no_bias": None}


def _grads(X, func, z0, t, dt, g, names):
    """cdeint's dL/dz0 and the parameter gradients on the kernel route."""
    params = tuple(p for n, p in func.named_parameters() if names is None or n in names)
    y0 = z0.clone().requires_grad_(True)
    out = _cdeint(X, func, y0, t, dt, adjoint_params=params)
    got = torch.autograd.grad((out * g).sum(), (y0,) + params)
    return out.detach(), got[0], dict(zip([n for n, p in func.named_parameters() if names is None or n in names],
                                          got[1:]))


def _reference_grads(X, func, z0, t, dt, g, names):
    f, leaves = _oracle_field(X, func)
    pnames = [n for n, _p in func.named_parameters()]
    y0 = z0.detach().double().cpu().requires_grad_(True)
    ys, _ = R.integrate(f, y0, t, dt)
    got = torch.autograd.grad((ys.movedim(0, 1) * g.double().cpu()).sum(), [y0] + leaves)
    return got[0], {n: v for n, v in zip(pnames, got[1:]) if names is None or n in names}


def _pattern(pattern, n_out, hidden, dtype, batch, t, dt):
    gen = torch.Generator().manual_seed(5)
    g = torch.randn(batch, n_out, hidden, generator=gen, dtype=F64)
    if pattern == "last":
        g[:, :-1] = 0
    elif pattern == "first":
        g[:, 1:] = 0
    elif pattern == "boundaries":                 # only outputs at multiples of the stride
        keep = [j for j, tv in enumerate(t.tolist()) if (tv - t[0].item()) / dt % STRIDE == 0]
        mask = torch.zeros(n_out, dtype=torch.bool)
        mask[keep] = True
        g[:, ~mask] = 0
    return g.to(dtype).to(DEV)


def _backward_case(monkeypatch, shape, dtype, control, sname, pattern="dense", roles="all", batch=300):
    X, func, z0, t, dt = _case(shape, dtype, control, sname, batch=batch, bias=roles != "no_bias")
    names = ROLES[roles]
    n_out = t.numel()
    g = _pattern(pattern, n_out, func.hidden, dtype, batch, t, dt)
    calls = _Calls(monkeypatch)
    _no_autograd(monkeypatch)
    with _variant(SHAPES[shape][3]):
        out, gz, grads = _grads(X, func, z0, t, dt, g, names)
    n_steps = reversible._Problem(X, func, z0, t.to(DEV), dt, None, ()).sched.n_steps
    n_seg = -(-n_steps // STRIDE)
    assert calls.names == [FWD] + [SEG, PG] * n_seg, calls.names
    ref_gz, ref = _reference_grads(X, func, z0, t, dt, g, names)
    errs = (gz.double().cpu() - ref_gz).abs().amax(dim=1) / ref_gz.abs().amax(dim=1).clamp_min(1e-300)
    kinked = errs > GRAD_BAR[dtype]["z0"]
    print("mlp reversible backward {} {} {} {} {} {}: dL/dz0 {:.2e} before setting {} kinked paths aside".format(
        shape, dtype, control, sname, pattern, roles, errs.max().item(), int(kinked.sum())))
    assert dtype == F32 or not kinked.any()
    assert int(kinked.sum()) <= batch // 32 and errs.max().item() <= KINK_BAR
    if kinked.any():
        g = g.clone()
        g[kinked.to(DEV)] = 0
        with _variant(SHAPES[shape][3]):
            out, gz, grads = _grads(X, func, z0, t, dt, g, names)
        ref_gz, ref = _reference_grads(X, func, z0, t, dt, g, names)
    assert sorted(grads) == sorted(ref)
    worst = {"z0": _path_err(gz, ref_gz)}
    for n, v in grads.items():
        worst[n] = ((v.double().cpu() - ref[n]).abs().max() / ref[n].abs().max().clamp_min(1e-300)).item()
    for n, e in worst.items():
        key = ("backward", dtype, "z0" if n == "z0" else "w")
        _WORST[key] = max(_WORST.get(key, 0.0), e)
        assert e <= GRAD_BAR[dtype]["z0" if n == "z0" else "w"], (n, e)
    print("  errors {} (worst so far {})".format({n: "{:.1e}".format(e) for n, e in worst.items()},
                                                 {k[1:]: "{:.1e}".format(v) for k, v in _WORST.items()}))
    return gz, grads


@pytest.mark.parametrize("sname", ["S2", "S4", "S5", "S6", "S8"])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_backward_matches_autograd_through_the_oracle(monkeypatch, dtype, control, sname):
    _backward_case(monkeypatch, "examples", dtype, control, sname)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_backward_output_gradient_patterns(monkeypatch, dtype, pattern):
    _backward_case(monkeypatch, "examples", dtype, "cubic", "S5", pattern=pattern)


@pytest.mark.parametrize("roles", list(ROLES))
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_backward_parameter_roles(monkeypatch, dtype, roles):
    _backward_case(monkeypatch, "examples", dtype, "linear", "S4", roles=roles)


@pytest.mark.parametrize("shape", ["odd", "unit", "hm32"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_backward_other_shapes(monkeypatch, shape, dtype):
    _backward_case(monkeypatch, shape, dtype, "cubic", "S5")


# ---- refusals keep the torch-operator forward and the per-step autograd backward ------------------------------------
@contextlib.contextmanager
def _parent_route(monkeypatch):
    """The route before the MLP kernels existed: the module is not taken for the MLP field."""
    with monkeypatch.context() as m:
        m.setattr(reversible, "mlp_field_of", lambda *args: None)
        yield


REFUSALS = ["tensor_core_shape", "softplus", "coeffs_in_params", "too_wide", "hm32_without_variant", "four_chunks"]


@pytest.mark.parametrize("refusal", REFUSALS)
def test_refusals_keep_the_torch_route(monkeypatch, refusal):
    shape = {"tensor_core_shape": (32, 8, 128, 0), "too_wide": (8, 3, 400, 0), "hm32_without_variant": (16, 2, 48, 0),
             "four_chunks": (8, 14, 128, 0)}
    X, func, z0, t, dt = _case(shape.get(refusal, SHAPES["examples"]), F32, "cubic", "S5", batch=200)
    if refusal == "softplus":
        func.act = torch.nn.functional.softplus
    extra = ()
    if refusal == "coeffs_in_params":
        coeffs = _inputs(8, 3, 128, False)[2][:200].clone().requires_grad_(True)
        X = cde.CubicSpline(coeffs)
        extra = (coeffs,)
    params = tuple(func.parameters()) + extra
    g = _pattern("dense", t.numel(), func.hidden, F32, 200, t, dt)

    def run():
        y0 = z0.clone().requires_grad_(True)
        out = _cdeint(X, func, y0, t, dt, adjoint_params=params)
        return (out.detach(),) + torch.autograd.grad((out * g).sum(), (y0,) + params)

    calls = _Calls(monkeypatch)
    got = run()
    assert not [n for n in calls.names if n in (FWD, SEG)], calls.names
    with _parent_route(monkeypatch):
        want = run()
    for a, b in zip(got, want):
        assert torch.equal(a, b)


# ---- determinism, memory, full scale ----------------------------------------------------------------------------------
def _problem(batch, length, dtype=F32, seed=4):
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(batch, length, 3, generator=gen, dtype=F64) / 16).cumsum(1).to(dtype)
    z0 = torch.randn(batch, 8, generator=gen, dtype=F64).to(dtype).to(DEV)
    torch.manual_seed(seed)
    func = Func(8, 3, 128).to(device=DEV, dtype=dtype)
    return cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV)), z0, func


def _backward_peak(coeffs, z0, func, dt):
    X = cde.CubicSpline(coeffs)
    ts = torch.tensor([0.0, coeffs.size(1) - 1.0], device=DEV)
    y0 = z0.clone().requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = cde.cdeint(X, func, y0, ts, backend="torchsde", method="reversible_heun", dt=dt)
    loss = out[:, -1].square().sum()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss.backward()
    torch.cuda.synchronize()
    grads = (y0.grad.clone(),) + tuple(p.grad.clone() for p in func.parameters())
    func.zero_grad()
    return torch.cuda.max_memory_allocated() - base, grads


def test_backward_memory_and_determinism(monkeypatch):
    paths = 8192
    coeffs, z0, func = _problem(paths, 256)
    _no_autograd(monkeypatch)
    state = paths * 8 * 4
    peak1, g1 = _backward_peak(coeffs, z0, func, 1.0)
    _peak, g1b = _backward_peak(coeffs, z0, func, 1.0)
    for a, b in zip(g1, g1b):
        assert torch.equal(a, b)
    peak4, _ = _backward_peak(coeffs, z0, func, 0.25)
    slots = lambda n: -(-n // STRIDE) + 1   # noqa: E731
    extra_ckpt = (slots(1020) - slots(255)) * 3 * state
    print("mlp reversible backward peak: dt 1 {:.1f} MiB, dt 0.25 {:.1f} MiB, extra checkpoints {:.1f} MiB".format(
        peak1 / 2 ** 20, peak4 / 2 ** 20, extra_ckpt / 2 ** 20))
    assert peak4 - peak1 <= extra_ckpt + 40 * state, (peak1, peak4, extra_ckpt)
    # checkpoints plus O(1) states: the checkpoints, two dumps of 17 steps, the carry and a few more states, and the
    # parameter-gradient scratch (one row of parameters per CTA of its persistent grid)
    scratch = _lib.load().tcde_mlp_field_param_grads_scratch_bytes(paths, STRIDE + 1, 3, 8, 128)
    assert peak1 <= slots(255) * 3 * state + 2 * (STRIDE + 1) * state + 16 * state + scratch + (4 << 20), (peak1, scratch)


def test_full_scale_fp32_against_the_fp64_kernel():
    coeffs, z0, func = _problem(65536, 256, seed=6)
    ts = torch.tensor([0.0, 100.5, 255.0], device=DEV)
    with torch.no_grad():
        out = cde.cdeint(cde.CubicSpline(coeffs), func, z0, ts, backend="torchsde", method="reversible_heun", dt=1.0)
        f64 = Func(8, 3, 128).to(device=DEV, dtype=F64)
        f64.load_state_dict({k: v.double() for k, v in func.state_dict().items()})
        ref = cde.cdeint(cde.CubicSpline(coeffs.double()), f64, z0.double(), ts.double(), backend="torchsde",
                         method="reversible_heun", dt=1.0)
    err = _path_err(out, ref)
    print("mlp reversible forward at B = 65,536, L = 256 vs the fp64 kernel: {:.2e} of scale".format(err))
    assert err <= 1e-5, err
