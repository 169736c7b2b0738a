"""cdeint(backend="torchsde", method="reversible_heun") on the GPU: the fused forward against the fp64 oracle and the
fp64 kernel, the reversible backward against autograd, its memory and its determinism.

The table-driven tests below run every kernel route of the forward (wgmma, 3xTF32, CUDA-core fp32 and fp64, at hidden
32 / channels 8 and at other shapes) on both controls and on schedules chosen at the edges of the checkpoint stride
(N < 16, N = 16, N = 16k + 1, outputs on segment boundaries, several outputs in one step, float32 grids, uneven knots),
check the checkpoint buffer slot by slot, and run the segment backward over the same schedules, parameter roles and
output-gradient patterns.  References: the fp64 oracle on the same fp32-rounded inputs, one solve per (shape, dtype,
control, schedule) shared by every route; bars are fractions of each path's own scale."""
import contextlib
import functools

import pytest
import torch

import torchcde_b200 as cde
from oracle import cde_oracle as O
from oracle import reversible_oracle as R
from torchcde_b200 import _lib, reversible
from torchcde_b200.linear_field import LinearFieldKernels

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _problem(batch, length, channels=8, hidden=32, seed=0, dtype=torch.float32):
    """Bench-like data: a random walk with N(0, (1/16)^2) increments, its Hermite spline, nn.Linear default init."""
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(batch, length, channels, generator=gen, dtype=torch.float64) / 16).cumsum(1).to(dtype)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64).to(dtype)
    torch.manual_seed(seed)
    func = cde.LinearVectorField(hidden, channels).to(device=DEV, dtype=dtype)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV))
    return coeffs, z0.to(DEV), func


def _oracle(coeffs, func, z0, ts, dt):
    """The fp64 oracle on the same (rounded) inputs: (outputs (batch, len(ts), H), field, params)."""
    w = func.linear.weight.detach().double().cpu().requires_grad_(True)
    b = func.linear.bias.detach().double().cpu().requires_grad_(True)
    c = coeffs.detach().double().cpu()
    f = R.linear_cde_field(c, torch.arange(c.size(1) + 1, dtype=torch.float64), w, b)
    y0 = z0.detach().double().cpu()
    ys, _ = R.integrate(f, y0, ts.double().cpu(), dt)
    return ys.movedim(0, 1), f, (w, b)


def _err(got, want):
    return (got.double().cpu() - want.double().cpu()).abs().max().item(), want.abs().max().item()


@pytest.mark.parametrize("dtype,bar", [(torch.float32, 1e-5), (torch.float64, 1e-10)])
def test_fused_forward_matches_the_oracle(dtype, bar):
    coeffs, z0, func = _problem(1000, 20, dtype=dtype)          # 1,000 paths: partial tiles
    X = cde.CubicSpline(coeffs)
    ts = torch.tensor([0.0, 0.3, 0.35, 5.0, 11.9, 19.0], dtype=torch.float64)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, ts.to(DEV), backend="torchsde", method="reversible_heun", dt=0.4)
    want, _, _ = _oracle(coeffs, func, z0, ts, 0.4)
    assert out.shape == (1000, ts.numel(), 32)
    err, scale = _err(out, want)
    print("forward {} vs oracle: {:.2e} of scale".format(dtype, err / scale))
    assert err <= bar * scale, (err, scale)
    assert torch.equal(out[:, 0], z0)


def test_fused_forward_config3_against_fp64_kernel():
    coeffs, z0, func = _problem(65536, 256)
    ts = torch.tensor([0.0, 100.5, 255.0], device=DEV)
    with torch.no_grad():
        out = cde.cdeint(cde.CubicSpline(coeffs), func, z0, ts, backend="torchsde", method="reversible_heun", dt=1.0)
        f64 = cde.LinearVectorField(32, 8).to(device=DEV, dtype=torch.float64)
        f64.load_state_dict({k: v.double() for k, v in func.state_dict().items()})
        ref = cde.cdeint(cde.CubicSpline(coeffs.double()), f64, z0.double(), ts.double(), backend="torchsde",
                         method="reversible_heun", dt=1.0)
    err = (out.double() - ref).abs().amax(dim=(1, 2))
    scale = ref.abs().amax(dim=(1, 2)).clamp(min=1.0)
    print("config 3 forward vs fp64 kernel: {:.2e} of scale".format((err / scale).max().item()))
    assert bool((err <= 1e-5 * scale).all()), (err / scale).max().item()


def test_fused_backward_matches_autograd_through_the_oracle():
    coeffs, z0, func = _problem(300, 256, seed=1)                # 300 paths: a partial tile
    ts = torch.tensor([0.0, 64.0, 130.25, 255.0], dtype=torch.float64)
    gen = torch.Generator().manual_seed(7)
    g = torch.randn(300, ts.numel(), 32, generator=gen, dtype=torch.float64)
    X = cde.CubicSpline(coeffs)
    y0 = z0.clone().requires_grad_(True)
    routes = []
    orig = reversible._Problem.fused_backward

    def spy(self, *args):
        routes.append("segment kernel")
        return orig(self, *args)

    reversible._Problem.fused_backward = spy
    try:
        out = cde.cdeint(X, func, y0, ts.to(DEV), backend="torchsde", method="reversible_heun", dt=1.0)
        (out.double() * g.to(DEV)).sum().backward()
    finally:
        reversible._Problem.fused_backward = orig
    assert routes == ["segment kernel"]           # one launch per checkpoint segment served the backward
    want, f, (w, b) = _oracle(coeffs, func, z0, ts, 1.0)
    y0d = z0.detach().double().cpu().requires_grad_(True)
    ys, _ = R.integrate(f, y0d, ts, 1.0)
    gy0, gw, gb = torch.autograd.grad((ys.movedim(0, 1) * g).sum(), (y0d, w, b))
    for got, ref, bar in ((y0.grad, gy0, 1e-5), (func.linear.weight.grad, gw, 2e-4), (func.linear.bias.grad, gb, 2e-4)):
        err, scale = _err(got, ref)
        print("fused backward: {:.2e} of scale (bar {:.0e})".format(err / scale, bar))
        assert err <= bar * scale, (err, scale)


class _MLP(torch.nn.Module):
    def __init__(self, hidden, channels, dtype):
        super().__init__()
        self.l1 = torch.nn.Linear(hidden, 48, dtype=dtype)
        self.l2 = torch.nn.Linear(48, hidden * channels, dtype=dtype)
        self.hidden, self.channels = hidden, channels

    def forward(self, t, z):
        return torch.tanh(self.l2(torch.nn.functional.softplus(self.l1(z)))).view(*z.shape[:-1], self.hidden,
                                                                                    self.channels)


@pytest.mark.parametrize("dtype,bar", [(torch.float32, 1e-5), (torch.float64, 1e-10)])
@pytest.mark.parametrize("field", ["mlp", "linear_with_coeffs"])
def test_torch_operator_backward_matches_autograd(dtype, bar, field):
    coeffs, z0, func = _problem(64, 40, channels=4, hidden=16, seed=2, dtype=dtype)
    coeffs = coeffs.clone().requires_grad_(True)
    if field == "mlp":
        func = _MLP(16, 4, dtype).to(DEV)
        params = tuple(func.parameters())
    else:
        params = tuple(func.parameters()) + (coeffs,)
    ts = torch.tensor([0.0, 7.3, 20.0, 39.0], device=DEV)
    gen = torch.Generator().manual_seed(3)
    g = torch.randn(64, 4, 16, generator=gen, dtype=dtype).to(DEV)
    grads = []
    for adjoint in (True, False):
        y0 = z0.clone().requires_grad_(True)
        X = cde.CubicSpline(coeffs)
        out = cde.cdeint(X, func, y0, ts, adjoint=adjoint, backend="torchsde", method="reversible_heun", dt=0.7,
                         adjoint_params=params)
        grads.append(torch.autograd.grad((out * g).sum(), (y0,) + params))
    worst = max(((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item() for a, b in zip(*grads))
    print("torch-operator backward {} {}: {:.2e}".format(field, dtype, worst))
    for a, b in zip(*grads):
        assert (a - b).abs().max() <= bar * b.abs().max().clamp(min=1e-30)


@pytest.mark.parametrize("culprit", ["func", "func.prod", "X.derivative"])
def test_a_non_tensor_answer_raises_the_reference_value_error(culprit):
    """The reference's compatibility check: a ``func``, ``func.prod`` or ``X.derivative`` that answers with something
    other than a tensor is a ValueError, before any solve."""
    coeffs, z0, _func = _problem(4, 6, channels=4, hidden=16)
    X = cde.CubicSpline(coeffs)
    func = lambda t, z: [z]                                                         # noqa: E731
    if culprit == "func.prod":
        func = type("Prod", (), {"prod": staticmethod(lambda t, z, dx: [z])})()
    elif culprit == "X.derivative":
        X = type("Control", (), {"derivative": staticmethod(lambda t: [t])})()
    with pytest.raises(ValueError, match="z0 is a tensor and so {} must return a tensor as well".format(culprit)):
        cde.cdeint(X, func, z0, torch.tensor([0.0, 5.0], device=DEV), backend="torchsde", method="reversible_heun",
                   dt=0.5)


def _backward_peak(coeffs, z0, func, dt):
    X = cde.CubicSpline(coeffs)
    ts = torch.tensor([0.0, 255.0], device=DEV)
    y0 = z0.clone().requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = cde.cdeint(X, func, y0, ts, backend="torchsde", method="reversible_heun", dt=dt)
    loss = out[:, -1].square().sum()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()          # the peak of the backward, checkpoints and outputs included
    loss.backward()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, (y0.grad.clone(), func.linear.weight.grad.clone(),
                                                      func.linear.bias.grad.clone())


def test_backward_memory_and_determinism():
    paths = 8192
    coeffs, z0, func = _problem(paths, 256, seed=4)
    state = paths * 32 * 4
    peak1, g1 = _backward_peak(coeffs, z0, func, 1.0)
    func.zero_grad()
    _peak1b, g1b = _backward_peak(coeffs, z0, func, 1.0)
    for a, b in zip(g1, g1b):
        assert torch.equal(a, b)                                  # bit-identical gradients
    func.zero_grad()
    peak4, _ = _backward_peak(coeffs, z0, func, 0.25)
    slots = lambda n: -(-n // reversible.CHECKPOINT_STRIDE) + 1   # noqa: E731
    extra_ckpt = (slots(1020) - slots(255)) * 3 * state
    # beyond the extra checkpoints, a step's temporaries are a few states
    print("backward peak: dt 1 {} MiB, dt 0.25 {} MiB, extra checkpoints {} MiB".format(peak1 >> 20, peak4 >> 20,
                                                                                      extra_ckpt >> 20))
    assert peak4 - peak1 <= extra_ckpt + 32 * state, (peak1, peak4, extra_ckpt)
    rk4_trajectory = 2 * 1020 * paths * 128                       # both stage dumps of the rk4 adjoint at step 1
    assert peak1 < rk4_trajectory, (peak1, rk4_trajectory)


# ---- the route x control x schedule tables ---------------------------------------------------------------------------
PATHS, LENGTH = 1000, 40                 # 1,000 paths: a partial tile for both tensor-core kernels
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-10}
CONTROLS = ["cubic", "linear"]
STRIDE = reversible.CHECKPOINT_STRIDE

# name: (t, dt, dtype of t, uneven knots)
SCHEDULES = {
    "S1": ([0.0, 0.5], 1.0, F64, False),                        # one clipped step: N = 1
    "S2": ([0.0, 15.0], 1.0, F64, False),                       # N = 15, shorter than one stride
    "S3": ([0.0, 16.0], 1.0, F64, False),                       # N = 16: the last checkpoint is slot 1
    "S4": ([0.0, 17.0], 1.0, F64, False),                       # N = 17: a one-step last segment
    "S5": ([0.0, 16.0, 32.0], 1.0, F64, False),                 # outputs on segment boundaries (w1 = 1)
    "S6": ([0.0, 0.1, 0.2, 0.25, 9.0, 9.7], 0.7, F64, False),   # several outputs in one step; a clipped last step
    "S7": ([0.0, 1.0, 3.0], 0.1, F32, False),                   # float32 grid by repeated addition
    "S8": ([2.5, 7.75, 11.0], 0.3, F64, True),                  # uneven knots (the builders' t=)
}

# name: (hidden, channels, dtype, solve variant)
ROUTES = {
    "wgmma": (32, 8, F32, 0),             # the default: 2xFP16 warpgroup MMA
    "tf32": (32, 8, F32, 3),              # 3xTF32 mma.sync
    "simt": (32, 8, F32, 1),              # the CUDA-core kernel at the tensor-core shape
    "f64": (32, 8, F64, 0),
    "simt16x4": (16, 4, F32, 0), "simt16x4_f64": (16, 4, F64, 0),
    "simt5x3": (5, 3, F32, 0), "simt5x3_f64": (5, 3, F64, 0),
    # fp64 at 64 x 8 would stage 256 KB of weights in shared memory: no kernel; that shape runs as torch operators
    "simt64x8": (64, 8, F32, 0), "simt64x4_f64": (64, 4, F64, 0),
}


@contextlib.contextmanager
def _variant(v):
    _lib.call("tcde_set_solve_variant", v)
    try:
        yield
    finally:
        _lib.call("tcde_set_solve_variant", 0)


@functools.lru_cache(maxsize=None)
def _inputs(hidden, channels, uneven):
    """The fp32 inputs of one problem shape on the device: paths (random walk, N(0, 1/16^2) increments), knots (None:
    the default 0..39), their Hermite coefficients, z0, and W, b in nn.Linear's default range."""
    gen = torch.Generator().manual_seed(97 * hidden + channels)
    x = (torch.randn(PATHS, LENGTH, channels, generator=gen, dtype=F64) / 16).cumsum(1).float()
    z0 = torch.randn(PATHS, hidden, generator=gen, dtype=F64).float()
    bound = hidden ** -0.5
    w = ((2 * torch.rand(hidden * channels, hidden, generator=gen, dtype=F64) - 1) * bound).float()
    b = ((2 * torch.rand(hidden * channels, generator=gen, dtype=F64) - 1) * bound).float()
    knots = None
    if uneven:                            # widths in [0.6, 1.4): neither integers nor evenly spaced
        widths = 0.6 + 0.8 * torch.rand(LENGTH - 1, generator=gen, dtype=F64)
        knots = torch.cat([torch.zeros(1, dtype=F64), widths.cumsum(0)]).float().to(DEV)
    x = x.to(DEV)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots)
    return x, knots, coeffs, z0.to(DEV), w.to(DEV), b.to(DEV)


def _case(hidden, channels, dtype, control, sname, batch=PATHS, bias=True, leaf=False):
    """(X, func, z0, t, dt) of the first ``batch`` paths in ``dtype`` (fp64: the fp32 values, cast).  The cubic control
    takes the fp32 Hermite coefficients; the linear one forms its own slopes.  ``leaf``: the control is built from a
    fresh leaf that requires grad, returned as a sixth value."""
    ts, dt, t_dtype, uneven = SCHEDULES[sname]
    x, knots, coeffs, z0, w, b = _inputs(hidden, channels, uneven)
    kt = None if knots is None else knots.to(dtype)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    if leaf:
        src = src.clone().requires_grad_(True)
    X = cde.CubicSpline(src, t=kt) if control == "cubic" else cde.LinearInterpolation(src, t=kt)
    func = cde.LinearVectorField(hidden, channels, bias=bias).to(device=DEV, dtype=dtype)
    with torch.no_grad():
        func.linear.weight.copy_(w)
        if bias:
            func.linear.bias.copy_(b)
    case = (X, func, z0[:batch].to(dtype), torch.tensor(ts, dtype=t_dtype), dt)
    return case + (src,) if leaf else case


def _oracle_field(X, func, wrt=()):
    """R's field on fp64 copies of the kernel's own inputs: the control's rows (Hermite coefficients, or the slopes
    ``_derivs``), W and b.  The knots keep the control's dtype: like ``_interpret_t``, the oracle casts a grid time to
    it before locating it (in fp32, t = 0.7 * 10 = 7.000000000000001 is the knot 7, which takes interval 6).  The copies
    named in ``wrt`` ("w", "b", "rows", or "x": the linear control's slopes formed from its knot values) are leaves that
    require grad.  Returns (f, {name: leaf})."""
    leaves = {"w": func.linear.weight.detach().double().cpu()}
    if func.linear.bias is not None:
        leaves["b"] = func.linear.bias.detach().double().cpu()
    knots = X._t.detach().cpu()
    cubic = isinstance(X, cde.CubicSpline)
    if "x" in wrt:
        leaves["x"] = X._coeffs.detach().double().cpu()
    else:
        leaves["rows"] = (X._rows() if cubic else X._derivs).detach().double().cpu()
    for name in wrt:
        leaves[name].requires_grad_(True)
    rows = O.linear_slopes(leaves["x"], knots.double()) if "x" in wrt else leaves["rows"]
    make = R.linear_cde_field if cubic else R.linear_control_field
    return make(rows, knots, leaves["w"], leaves.get("b")), leaves


_solves = {}                              # one oracle solve per (shape, dtype, control, schedule), shared by routes


def _reference(hidden, channels, dtype, control, sname):
    """The oracle's outputs (PATHS, n_out, H) and its states {step: (y, z, f)} at every step."""
    key = (hidden, channels, dtype, control, sname)
    if key not in _solves:
        X, func, z0, t, dt = _case(hidden, channels, dtype, control, sname)
        f, _ = _oracle_field(X, func)
        with torch.no_grad():
            ys, rec = R.integrate(f, z0.double().cpu(), t, dt)
        _solves[key] = (ys.movedim(0, 1), rec["states"])
    return _solves[key]


def _forward(monkeypatch, X, func, z0, t, dt, variant):
    """cdeint's forward; the kernel must serve it (the torch-operator solve takes over shapes no kernel fits)."""
    def refuse(self, *args):
        raise AssertionError("the torch-operator solve served a kernel route")

    monkeypatch.setattr(reversible._Problem, "torch_forward", refuse)
    with _variant(variant), torch.no_grad():
        return cde.cdeint(X, func, z0, t.to(DEV), backend="torchsde", method="reversible_heun", dt=dt)


def _path_err(got, want):
    """max over paths (dim 0) of max |got - want| / max |want| on that path."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    dims = tuple(range(1, want.dim()))
    err = (got - want).abs().amax(dim=dims)
    return (err / want.abs().amax(dim=dims).clamp_min(1e-300)).max().item()


def _global_err(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


def _report(what, err, bar):
    print("reversible {}: {:.2e} of scale (bar {:.0e})".format(what, err, bar))
    assert err <= bar, (what, err, bar)


@pytest.mark.parametrize("sname", list(SCHEDULES))
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", list(ROUTES))
def test_forward_routes_match_the_oracle(route, control, sname, monkeypatch):
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, dt = _case(hidden, channels, dtype, control, sname)
    want, _states = _reference(hidden, channels, dtype, control, sname)
    out = _forward(monkeypatch, X, func, z0, t, dt, variant)
    assert out.shape == want.shape and out.dtype == dtype
    assert torch.equal(out[:, 0], z0)
    _report("forward {} {} {}".format(route, control, sname), _path_err(out, want), BAR[dtype])


@pytest.mark.parametrize("batch", [1, 63, 64, 65, 127, 128, 129])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", ["wgmma", "tf32", "simt"])
def test_forward_tile_edges_match_the_oracle(route, control, batch, monkeypatch):
    """Batches on both sides of 64 paths per warpgroup (wgmma) and 128 paths per CTA (3xTF32), at S4."""
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, dt = _case(hidden, channels, dtype, control, "S4", batch)
    want, _states = _reference(hidden, channels, dtype, control, "S4")
    out = _forward(monkeypatch, X, func, z0, t, dt, variant)
    assert out.shape == (batch,) + want.shape[1:]
    assert torch.equal(out[:, 0], z0)
    _report("forward {} {} batch {}".format(route, control, batch), _path_err(out, want[:batch]), BAR[dtype])


@pytest.mark.parametrize("sname", ["S1", "S2", "S3", "S4", "S5", "S7"])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("route", list(ROUTES))
def test_checkpoints_hold_the_oracle_states(route, control, sname):
    """The checkpointing forward: outputs bit-equal to the plain forward, ceil(N / 16) + 1 slots, slot s = (y, z, f) of
    step min(16 s, N), each state within the bar of the oracle's state at that step."""
    hidden, channels, dtype, variant = ROUTES[route]
    X, func, z0, t, dt = _case(hidden, channels, dtype, control, sname)
    _want, states = _reference(hidden, channels, dtype, control, sname)
    kernels = LinearFieldKernels(X, func.linear.weight, func.linear.bias, z0)
    problem = reversible._Problem(X, func, z0, t, dt, kernels, tuple(func.parameters()))
    with _variant(variant), torch.no_grad():
        plain, _ = problem.kernel_forward(z0, keep_checkpoints=False)
        out, ckpts = problem.kernel_forward(z0, keep_checkpoints=True)
    assert torch.equal(out, plain)
    n_steps = problem.sched.n_steps
    slots = ckpts["slots"]
    n_slots = -(-n_steps // STRIDE) + 1
    assert slots.shape == (n_slots, 3, z0.size(0), hidden)
    steps = [min(STRIDE * s, n_steps) for s in range(n_slots)]
    assert sorted(k for k in ckpts if isinstance(k, int)) == steps
    worst = 0.0
    for s, step in enumerate(steps):
        for plane in range(3):                              # y, z, f
            assert ckpts[step][plane].data_ptr() == slots[s, plane].data_ptr()
            worst = max(worst, _path_err(slots[s, plane], states[step][plane]))
    _report("checkpoints {} {} {} (N = {})".format(route, control, sname, n_steps), worst, BAR[dtype])


# ---- the backward ----------------------------------------------------------------------------------------------------
def _run_backward(monkeypatch, X, func, z0, t, dt, g, adjoint_params=None):
    """One backward through cdeint(adjoint=True) with output gradients g: (dL/dz0, the routes that served it)."""
    served = []
    orig = reversible._Problem.fused_backward

    def spy(self, *args):
        served.append("segment kernel")
        return orig(self, *args)

    monkeypatch.setattr(reversible._Problem, "fused_backward", spy)
    y0 = z0.clone().requires_grad_(True)
    kwargs = {} if adjoint_params is None else {"adjoint_params": adjoint_params}
    out = cde.cdeint(X, func, y0, t.to(DEV), backend="torchsde", method="reversible_heun", dt=dt, adjoint=True,
                     **kwargs)
    out.backward(g)
    return y0.grad, served


def _reference_grads(X, func, z0, sname, g, wrt):
    """dL/dz0 and dL/d(each of ``wrt``) by torch.autograd through the fp64 oracle forward."""
    ts, dt, t_dtype, _uneven = SCHEDULES[sname]
    f, leaves = _oracle_field(X, func, wrt)
    y0 = z0.detach().double().cpu().requires_grad_(True)
    ys, _ = R.integrate(f, y0, torch.tensor(ts, dtype=t_dtype), dt)
    got = torch.autograd.grad((ys.movedim(0, 1) * g.double().cpu()).sum(), [y0] + [leaves[k] for k in wrt])
    return dict(zip(["z0"] + list(wrt), got))


def _pattern(name, batch, n_out, hidden, dtype):
    gen = torch.Generator().manual_seed(7)
    g = torch.randn(batch, n_out, hidden, generator=gen, dtype=F64)
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
    return g.to(dtype).to(DEV)


# bars: dL/dz0 per path; dL/dW, dL/db (the 2xBF16 contraction) and the control's gradient of the scale of the tensor
GRAD_BARS = {F32: {"z0": 1e-5, "w": 2e-4, "b": 2e-4, "rows": 1e-5, "x": 1e-5},
             F64: {"z0": 1e-10, "w": 1e-10, "b": 1e-10, "rows": 1e-10, "x": 1e-10}}


def _check_grads(what, got, want, dtype):
    for name, g in got.items():
        err = _path_err(g, want[name]) if name == "z0" else _global_err(g, want[name])
        _report("backward {} d/d{}".format(what, name), err, GRAD_BARS[dtype][name])


def _backward_case(monkeypatch, control, sname, batch, pattern="dense", roles="wb", dtype=F32):
    X, func, z0, t, dt = _case(32, 8, dtype, control, sname, batch, bias=roles != "no_bias")
    lin = func.linear
    if roles == "w":
        lin.bias.requires_grad_(False)
    elif roles == "b":
        lin.weight.requires_grad_(False)
    g = _pattern(pattern, batch, len(SCHEDULES[sname][0]), 32, dtype)
    gz, served = _run_backward(monkeypatch, X, func, z0, t, dt, g)
    wrt = {"wb": ["w", "b"], "w": ["w"], "b": ["b"], "no_bias": ["w"]}[roles]
    got = {"z0": gz}
    for name in wrt:
        got[name] = (lin.weight if name == "w" else lin.bias).grad
    for name, p in (("w", lin.weight), ("b", lin.bias)):
        if p is not None and name not in wrt:
            assert p.grad is None
    return got, _reference_grads(X, func, z0, sname, g, wrt), served, g


BACKWARD_CASES = [(65, s) for s in ("S1", "S2", "S3", "S4", "S5", "S6", "S7")] + [(b, s) for b in (1, 1000)
                                                                                 for s in ("S4", "S6")]


@pytest.mark.parametrize("batch,sname", BACKWARD_CASES)
@pytest.mark.parametrize("control", CONTROLS)
def test_segment_backward_matches_autograd_through_the_oracle(control, batch, sname, monkeypatch):
    got, want, served, _g = _backward_case(monkeypatch, control, sname, batch)
    assert served == ["segment kernel"]
    _check_grads("{} {} batch {}".format(control, sname, batch), got, want, F32)


@pytest.mark.parametrize("roles", ["wb", "w", "b", "no_bias"])
@pytest.mark.parametrize("control", CONTROLS)
def test_segment_backward_parameter_roles(control, roles, monkeypatch):
    """W and b, W only (a null grad_bias), b only (a null grad_weight) and a field without bias, at S6."""
    got, want, served, _g = _backward_case(monkeypatch, control, "S6", 65, roles=roles)
    assert served == ["segment kernel"]
    _check_grads("{} roles {}".format(control, roles), got, want, F32)


@pytest.mark.parametrize("pattern", ["dense", "last_output", "odd_paths_zero", "tiny", "huge", "first_output"])
@pytest.mark.parametrize("control", CONTROLS)
def test_segment_backward_gradient_patterns(control, pattern, monkeypatch):
    """Output gradients with zero rows (whole paths, or every output but one: rows of fbar that are exactly zero through
    the zero-bias product J_F^T fbar) and scaled by 2^-60 / 2^60 (relative bars), at S6."""
    got, want, served, g = _backward_case(monkeypatch, control, "S6", 65, pattern=pattern)
    assert served == ["segment kernel"]
    if pattern == "first_output":
        # output 0 is z0 itself: dL/dz0 = g[:, 0] and no parameter gradient, exactly
        assert torch.equal(got["z0"], g[:, 0])
        assert not got["w"].any() and not got["b"].any()
        return
    if pattern == "odd_paths_zero":
        assert not got["z0"][1::2].any()                      # paths are independent
    _check_grads("{} pattern {}".format(control, pattern), got, want, F32)


@pytest.mark.parametrize("sname", ["S4", "S6"])
@pytest.mark.parametrize("control", CONTROLS)
def test_per_step_backward_with_control_gradients(control, sname, monkeypatch):
    """The control's coefficients in adjoint_params: the per-step autograd backward from the wgmma forward's
    checkpoints, the coefficient gradient included."""
    X, func, z0, t, dt, leaf = _case(32, 8, F32, control, sname, 65, leaf=True)
    g = _pattern("dense", 65, len(SCHEDULES[sname][0]), 32, F32)
    params = (func.linear.weight, func.linear.bias, leaf)
    gz, served = _run_backward(monkeypatch, X, func, z0, t, dt, g, adjoint_params=params)
    assert served == []
    name = "rows" if control == "cubic" else "x"
    want = _reference_grads(X, func, z0, sname, g, ["w", "b", name])
    got = {"z0": gz, "w": func.linear.weight.grad, "b": func.linear.bias.grad, name: leaf.grad}
    _check_grads("per-step {} {}".format(control, sname), got, want, F32)


@pytest.mark.parametrize("sname", ["S4", "S6"])
@pytest.mark.parametrize("control", CONTROLS)
def test_fp64_backward_matches_autograd_through_the_oracle(control, sname, monkeypatch):
    got, want, served, _g = _backward_case(monkeypatch, control, sname, 65, dtype=F64)
    assert served == []
    _check_grads("fp64 {} {}".format(control, sname), got, want, F64)
