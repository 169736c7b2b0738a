"""The routes of cdeint that serve every ``func`` that is not one fused kernel, against the fp64 oracle.

Routes:
  1. the stage-kernel loop (``solver._generic_solve_kernels``: ``tcde_spline_eval`` once per step, ``tcde_field_contract``
     per stage, ``tcde_linear_combination`` per Runge-Kutta combination) -- fixed step, no gradient;
  2. its CUDA graph (``options={"cuda_graph": True}``) and the graph cache ``solver._graphs``;
  3. the torch-operator loop (``solver._generic_solve``) -- fixed step, ``adjoint=False`` with gradients;
  4. the fixed-step ``adjoint=True`` backward through ``adaptive.odeint_fixed`` under autograd;
  5. the host-driven dopri5 (``adaptive.Dopri5``) with ``tcde_linear_combination`` and ``tcde_error_ratio_sumsq``;
  6. the dopri5 ``adjoint=True`` backward on the packed augmented state.
Fields (none of them runs a fused kernel): a softplus MLP at 32 / 8 (width 64), a field that reads t at 5 / 3,
``LinearVectorField(128, 8)`` (recognised, but its shape is refused by the fused kernels), a ``prod`` field at 4 / 2,
H = C = 1, a field that returns a non-contiguous (H, C) view, and for the dopri5 and adjoint rows the examples' MLP at
32 / 8 / 128 (its fixed-step forward is one fused kernel).  Schedules: ``test_host_logic.FIXED_SCHEDULES`` on 40 knots;
the stage-kernel loop runs every schedule with rk4 in fp32 and fp64, and midpoint and euler at F3 (several outputs
inside a step) and F8 (decreasing t) in fp32 -- the stepper arithmetic that differs between the methods is the same on
every schedule, so the other 24 (schedule, method) pairs per field would add runtime, not coverage.

Reference: ``odeint_port.odeint`` and ``adaptive_oracle`` driving ``adaptive_oracle.FuncCDE`` -- an fp64 copy of the
module on fp64 copies of the kernel's own rounded inputs, stage times rounded to the state dtype -- with torch's generic
fp64 operators on the GPU, none of this package's kernels.  Every case proves its route: the other routes are patched to
raise, and the names of the library calls are recorded.  Bars are fractions of each path's own scale (parameter
gradients: of the tensor's scale)."""
import copy
import functools
import math

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port
from test_host_logic import FIXED_SCHEDULES, fixed_schedule_knots
from torchcde_b200 import _lib, adaptive, solver
from torchcde_b200.linear_field import LinearFieldKernels
from torchcde_b200.mlp_field import MlpFieldKernels

pytestmark = pytest.mark.gpu
DEV = "cuda"
PATHS, LENGTH = 1000, 40
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-10}
DTYPES = {"fp32": F32, "fp64": F64}
CONTROLS = ["cubic", "linear"]
METHODS = ["rk4", "midpoint", "euler"]
SCHEDULES = list(FIXED_SCHEDULES)
LOOP_KERNELS = {"tcde_spline_eval", "tcde_field_contract", "tcde_linear_combination"}
STEPPERS = {"tcde_field_contract", "tcde_linear_combination", "tcde_error_ratio_sumsq"}

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[generic routes, worst of each check] " + "; ".join(
        "{}: {:.2e} (bar {:.0e})".format(k, e, b) for k, (e, b) in sorted(_WORST.items())))


def _report(what, err, bar):
    print("generic {}: {:.2e} (bar {:.0e})".format(what, err, bar))
    key = what.split(" |")[0]
    if err > _WORST.get(key, (-1.0, bar))[0]:
        _WORST[key] = (err, bar)
    assert err <= bar, (what, err, bar)


def _path_err(got, want):
    """max over paths (dim 0) of max |got - want| / max |want| on that path (NaN if got holds a NaN)."""
    got, want = got.detach().double(), want.detach().double().to(got.device)
    if want.numel() == 0:
        return 0.0
    want = want.reshape(want.size(0), -1) if want.dim() > 1 else want.reshape(1, -1)
    got = got.reshape(want.shape)
    err = (got - want).abs().amax(dim=1)
    return (err / want.abs().amax(dim=1).clamp_min(1e-300)).max().item()


def _global_err(got, want):
    got, want = got.detach().double(), want.detach().double().to(got.device)
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


def _options(step, **extra):
    return dict({} if step is None else {"step_size": step}, **extra)


# ---- fields ----------------------------------------------------------------------------------------------------------
class SoftplusMLP(torch.nn.Module):
    def __init__(self, hidden=32, channels=8, width=64):
        super().__init__()
        self.hidden, self.channels = hidden, channels
        self.linear1 = torch.nn.Linear(hidden, width)
        self.linear2 = torch.nn.Linear(width, hidden * channels)

    def forward(self, t, z):
        z = self.linear2(torch.nn.functional.softplus(self.linear1(z))).tanh()
        return z.view(*z.shape[:-1], self.hidden, self.channels)


class TimeField(torch.nn.Module):
    """tanh(Linear(z) + t v): the only field here whose value depends on the stage time itself."""

    def __init__(self, hidden=5, channels=3):
        super().__init__()
        self.hidden = hidden
        self.linear = torch.nn.Linear(hidden, hidden * channels)
        self.v = torch.nn.Parameter(torch.randn(hidden * channels) / 8)

    def forward(self, t, z):
        return torch.tanh(self.linear(z) + t * self.v).view(*z.shape[:-1], self.hidden, -1)


class ProdField(torch.nn.Module):
    """A field given by its product with dX/dt: f(t, z) = tanh(Linear(z)).view(H, C) @ dX/dt - z |dX/dt|^2 / 4."""

    def __init__(self, hidden=4, channels=2):
        super().__init__()
        self.hidden = hidden
        self.linear = torch.nn.Linear(hidden, hidden * channels)

    def prod(self, t, z, dxdt):
        m = torch.tanh(self.linear(z)).view(*z.shape[:-1], self.hidden, -1)
        return (m @ dxdt.unsqueeze(-1)).squeeze(-1) - 0.25 * z * (dxdt * dxdt).sum(-1, keepdim=True)


class TanhLinear(torch.nn.Module):
    def __init__(self, hidden=1, channels=1):
        super().__init__()
        self.hidden = hidden
        self.linear = torch.nn.Linear(hidden, hidden * channels)

    def forward(self, t, z):
        return torch.tanh(self.linear(z)).view(*z.shape[:-1], self.hidden, -1)


class TransposedField(torch.nn.Module):
    """Returns the transpose of a (C, H) view: an (H, C) tensor that is not contiguous."""

    def __init__(self, hidden=6, channels=4):
        super().__init__()
        self.hidden, self.channels = hidden, channels
        self.linear = torch.nn.Linear(hidden, hidden * channels)

    def forward(self, t, z):
        out = torch.tanh(self.linear(z)).view(*z.shape[:-1], self.channels, self.hidden).transpose(-1, -2)
        assert not out.is_contiguous()
        return out


class Func(torch.nn.Module):
    """example/time_series_classification.py's CDEFunc."""

    def __init__(self, input_channels=8, hidden_channels=32, width=128):
        super().__init__()
        self.input_channels, self.hidden_channels = input_channels, hidden_channels
        self.linear1 = torch.nn.Linear(hidden_channels, width)
        self.linear2 = torch.nn.Linear(width, input_channels * hidden_channels)

    def forward(self, t, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], self.hidden_channels, self.input_channels)


# name: (hidden, channels, constructor)
FIELDS = {
    "softplus": (32, 8, lambda: SoftplusMLP(32, 8, 64)),
    "time": (5, 3, lambda: TimeField(5, 3)),
    "linear128x8": (128, 8, lambda: cde.LinearVectorField(128, 8)),
    "prod": (4, 2, lambda: ProdField(4, 2)),
    "h1c1": (1, 1, lambda: TanhLinear(1, 1)),
    "transposed": (6, 4, lambda: TransposedField(6, 4)),
    "examples": (32, 8, lambda: Func(8, 32, 128)),
}
LOOP_FIELDS = [f for f in FIELDS if f != "examples"]          # the examples' fixed-step forward is one fused kernel


def _func(name, dtype, seed=0):
    """The field's module with parameters drawn in fp32 (fp64: the same values, cast)."""
    torch.manual_seed(1000 + 17 * seed + sum(map(ord, name)))
    return FIELDS[name][2]().to(DEV).to(dtype)


@functools.lru_cache(maxsize=None)
def _inputs(channels, hidden, uneven, paths=PATHS, length=LENGTH):
    """fp32 inputs on the device: paths (random walk, N(0, 1/4^2) increments), knots (None: 0..length-1), their
    Hermite coefficients and z0."""
    gen = torch.Generator().manual_seed(97 * channels + hidden + paths + length)
    x = (torch.randn(paths, length, channels, generator=gen, dtype=F64) / 4).cumsum(1).float().to(DEV)
    z0 = torch.randn(paths, hidden, generator=gen, dtype=F64).float().to(DEV)
    knots = fixed_schedule_knots(True).to(DEV) if uneven else None
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots)
    return x, knots, coeffs, z0


def _control(src, knots, control):
    return cde.CubicSpline(src, t=knots) if control == "cubic" else cde.LinearInterpolation(src, t=knots)


def _times(sname):
    ts, step, uneven = FIXED_SCHEDULES[sname]
    if ts is None:
        return fixed_schedule_knots(uneven).double(), step
    return torch.tensor(ts, dtype=F32 if sname == "F4" else F64), step


def _case(field, dtype, control, sname, batch=PATHS):
    """(X, func, z0, t, step_size) of the first ``batch`` paths in ``dtype``."""
    hidden, channels, _ = FIELDS[field]
    x, knots, coeffs, z0 = _inputs(channels, hidden, FIXED_SCHEDULES[sname][2])
    kt = None if knots is None else knots.to(dtype)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    t, step = _times(sname)
    return _control(src, kt, control), _func(field, dtype), z0[:batch].to(dtype), t, step


def _oracle(X, func, control, dtype):
    """FuncCDE on fp64 copies of the control's rows (cubic) / knot values (linear), its knots and the module."""
    rows = (X._rows() if control == "cubic" else X._coeffs).detach()
    rows = rows.reshape(-1, rows.size(-2), rows.size(-1)).double()
    f64 = copy.deepcopy(func).double()
    prod = hasattr(func, "prod")
    return AO.FuncCDE(rows, X._t.detach().cpu(), f64.prod if prod else f64, control, time_dtype=dtype,
                      params=list(f64.parameters()), prod=prod)


_solves = {}


def _reference(field, dtype, control, sname, method):
    """The oracle's outputs (PATHS, n_out, H) in fp64, one solve per problem."""
    key = (field, dtype, control, sname, method)
    if key not in _solves:
        X, func, z0, t, step = _case(field, dtype, control, sname)
        with torch.no_grad():
            ys = odeint_port.odeint(_oracle(X, func, control, dtype), z0.double(), t, method=method,
                                    options=_options(step))
        _solves[key] = ys.movedim(0, 1)
    return _solves[key]


class _Calls:
    """Records the names of the library calls (and which of them refused the problem)."""

    def __init__(self, monkeypatch):
        self.names, self.refused = [], []
        real = _lib.call

        def call(name, *args):
            self.names.append(name)
            try:
                return real(name, *args)
            except NotImplementedError:
                self.refused.append(name)
                raise

        monkeypatch.setattr(_lib, "call", call)


def _refuse(monkeypatch, *names):
    """Patch the named routes to raise: ``loop`` (_generic_solve_kernels), ``torch`` (_generic_solve), ``mlp`` (the MLP
    kernels), ``linear`` (the fused linear solve; it may still refuse the problem itself), ``device`` (device dopri5)."""
    def raiser(what):
        def refuse(*args, **kwargs):
            raise AssertionError("{} served a case of another route".format(what))
        return refuse

    if "loop" in names:
        monkeypatch.setattr(solver, "_generic_solve_kernels", raiser("the stage-kernel loop"))
    if "torch" in names:
        monkeypatch.setattr(solver, "_generic_solve", raiser("the torch-operator loop"))
    if "mlp" in names:
        monkeypatch.setattr(MlpFieldKernels, "solve", raiser("the fused MLP solve"))
    if "linear" in names:
        real = LinearFieldKernels.solve

        def solve(self, *args, **kwargs):
            out = real(self, *args, **kwargs)
            raise AssertionError("the fused linear solve served a case of another route")
        monkeypatch.setattr(LinearFieldKernels, "solve", solve)
    if "device" in names:
        monkeypatch.setattr(LinearFieldKernels, "dopri5", raiser("the device-controlled dopri5"))


def _loop(monkeypatch, X, func, z0, t, step, method, **extra):
    """cdeint's no-grad fixed-step call, which the stage-kernel loop must serve: (output, calls)."""
    _refuse(monkeypatch, "torch", "mlp", "linear")
    calls = _Calls(monkeypatch)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step, **extra))
    monkeypatch.undo()
    return out, calls


def _check_loop_calls(calls, field):
    want = LOOP_KERNELS - ({"tcde_field_contract"} if field == "prod" else set())
    assert want <= set(calls.names), calls.names
    assert set(calls.refused) <= {"tcde_cdeint_fixed_linear"}, calls.refused
    assert (field == "linear128x8") == ("tcde_cdeint_fixed_linear" in calls.refused)


# ---- 1. the stage-kernel loop ----------------------------------------------------------------------------------------
LOOP_CASES = [(f, d, c, s, m) for f in LOOP_FIELDS for d in ("fp32", "fp64") for c in CONTROLS for s in SCHEDULES
              for m in METHODS if m == "rk4" or (d == "fp32" and s in ("F3", "F8"))]


@pytest.mark.parametrize("field,dtype,control,sname,method", LOOP_CASES)
def test_stage_kernel_loop_matches_the_oracle(field, dtype, control, sname, method, monkeypatch):
    dtype = DTYPES[dtype]
    X, func, z0, t, step = _case(field, dtype, control, sname)
    want = _reference(field, dtype, control, sname, method)
    out, calls = _loop(monkeypatch, X, func, z0, t, step, method)
    _check_loop_calls(calls, field)
    assert out.shape == want.shape and out.dtype == dtype
    assert torch.equal(out[:, 0], z0)
    _report("loop {} | {} {} {} {}".format("fp64" if dtype == F64 else "fp32", field, control, sname, method),
            _path_err(out, want), BAR[dtype])


@pytest.mark.parametrize("shape", [(), (1,), (3, 7), (257,), (0,)])
@pytest.mark.parametrize("control", CONTROLS)
def test_stage_kernel_loop_batch_shapes(control, shape, monkeypatch):
    n = math.prod(shape)
    X, func, z0, t, step = _case("softplus", F32, control, "F3", max(n, 1))
    src = (X._rows() if control == "cubic" else X._coeffs)[:n]
    Xs = _control(src.reshape(*shape, *src.shape[1:]), None, control)
    zs = z0[:n].reshape(*shape, 32)
    if n == 0:
        with torch.no_grad():
            out = cde.cdeint(Xs, func, zs, t, adjoint=False, method="rk4", options=_options(step))
        assert out.shape == (0, t.numel(), 32)
        return
    out, calls = _loop(monkeypatch, Xs, func, zs, t, step, "rk4")
    assert out.shape == (*shape, t.numel(), 32)
    _check_loop_calls(calls, "softplus")
    want = _reference("softplus", F32, control, "F3", "rk4")[:n]
    _report("loop batch shape | {} {}".format(control, shape), _path_err(out.reshape(n, t.numel(), 32), want),
            BAR[F32])


def test_stage_kernel_loop_past_the_grid_cap(monkeypatch):
    """A state of 1.2 M elements: more than the 8 CTAs per SM x 256 threads x 4 elements the stepper kernels launch
    (1.08 M on 132 SMs), so their grid-stride loops run more than once."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    paths = 240_000
    assert paths * 5 > n_sm * 8 * 256 * 4
    gen = torch.Generator(device=DEV).manual_seed(3)
    x = (torch.randn(paths, 10, 3, generator=gen, device=DEV) / 4).cumsum(1)
    z0 = torch.randn(paths, 5, generator=gen, device=DEV)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    func = _func("time", F32)
    t = torch.tensor([0.0, 4.3, 9.0], dtype=F64)
    out, calls = _loop(monkeypatch, X, func, z0, t, 0.5, "rk4")
    _check_loop_calls(calls, "time")
    with torch.no_grad():
        want = odeint_port.odeint(_oracle(X, func, "cubic", F32), z0.double(), t, method="rk4",
                                  options={"step_size": 0.5}).movedim(0, 1)
    _report("loop past the grid cap | 240,000 x 5", _path_err(out, want), BAR[F32])


class DerivativeOnly:
    """A user-defined control: nothing but a ``derivative`` method (here, that of a built-in spline)."""

    def __init__(self, X):
        self.X = X

    def derivative(self, t):
        return self.X.derivative(t)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("sname", ["F3", "F8"])
def test_a_user_defined_control_runs_the_torch_operator_loop(sname, method, monkeypatch):
    """An unknown control has no kernel rows: even without gradients the torch-operator loop serves it."""
    X, func, z0, t, step = _case("time", F32, "cubic", sname)
    _refuse(monkeypatch, "loop", "mlp", "linear")
    calls = _Calls(monkeypatch)
    with torch.no_grad():
        out = cde.cdeint(DerivativeOnly(X), func, z0, t, adjoint=False, method=method, options=_options(step))
    assert not STEPPERS & set(calls.names)
    assert torch.equal(out[:, 0], z0)
    _report("user-defined control | {} {}".format(sname, method),
            _path_err(out, _reference("time", F32, "cubic", sname, method)), BAR[F32])


# ---- 2. the CUDA graph -----------------------------------------------------------------------------------------------
class _Captures:
    def __init__(self, monkeypatch):
        self.count = 0
        real = torch.cuda.CUDAGraph

        def make(*args, **kwargs):
            self.count += 1
            return real(*args, **kwargs)

        monkeypatch.setattr(torch.cuda, "CUDAGraph", make)


def _graph(X, func, z0, t, step, method="rk4"):
    with torch.no_grad():
        return cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step, cuda_graph=True))


@pytest.mark.parametrize("sname,method", [("F3", "rk4"), ("F8", "rk4"), ("F3", "midpoint"), ("F8", "euler")])
@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("field", ["softplus", "time", "prod", "transposed"])
def test_cuda_graph_replays_the_loop_bit_for_bit(field, control, sname, method, monkeypatch):
    solver._graphs.clear()
    X, func, z0, t, step = _case(field, F32, control, sname)
    plain, _calls = _loop(monkeypatch, X, func, z0, t, step, method)
    caps = _Captures(monkeypatch)
    first = _graph(X, func, z0, t, step, method)
    again = _graph(X, func, z0 * 0.5, t, step, method)          # a new z0 is read
    assert caps.count == 1
    assert torch.equal(first, plain)
    half, _calls = _loop(monkeypatch, X, func, z0 * 0.5, t, step, method)
    assert torch.equal(again, half)
    _report("graph | {} {} {} {}".format(field, control, sname, method),
            _path_err(first, _reference(field, F32, control, sname, method)), BAR[F32])


@pytest.mark.parametrize("control", CONTROLS)
def test_cuda_graph_sees_in_place_updates_and_captures_new_problems(control, monkeypatch):
    solver._graphs.clear()
    X0, func, z0, t, step = _case("time", F32, control, "F3", 200)
    X = _control((X0._rows() if control == "cubic" else X0._coeffs).clone(), None, control)
    _graph(X, func, z0, t, step)
    # in-place updates of parameters and of the control's coefficients (an optimizer step): no new capture
    with torch.no_grad():
        func.v.mul_(-2.0)
        func.linear.weight.add_(0.01)
        (X._rows() if control == "cubic" else X._coeffs).mul_(1.5)
    out = _graph(X, func, z0, t, step)
    assert len(solver._graphs) == 1
    want = _loop(monkeypatch, X, func, z0, t, step, "rk4")[0]
    assert not torch.equal(out, _loop(monkeypatch, X0, _func("time", F32), z0, t, step, "rk4")[0])
    assert torch.equal(out, want)
    # another control of the same shape, and new output times: captured anew, and answered correctly
    Y, _f, _z, _t, _s = _case("time", F32, control, "F3", 200)
    Y = _control((Y._rows() if control == "cubic" else Y._coeffs).flip(0).contiguous(), None, control)
    for XX, tt in ((Y, t), (X, torch.tensor([0.0, 0.45, 12.0, 39.0], dtype=F64))):
        got = _graph(XX, func, z0, tt, step)
        assert torch.equal(got, _loop(monkeypatch, XX, func, z0, tt, step, "rk4")[0])
    assert len(solver._graphs) == 3


def test_a_ninth_key_clears_the_graph_cache(monkeypatch):
    solver._graphs.clear()
    X, func, z0, t, step = _case("softplus", F32, "cubic", "F3", 64)
    caps = _Captures(monkeypatch)
    outs = []
    for k in range(9):
        tt = torch.tensor([0.0, 1.0 + k, 39.0], dtype=F64)
        outs.append((tt, _graph(X, func, z0, tt, step)))
        assert len(solver._graphs) == (k + 1 if k < 8 else 1)
    assert caps.count == 9
    for tt, got in outs:
        assert torch.equal(got, _loop(monkeypatch, X, func, z0, tt, step, "rk4")[0])


class TrainingBranch(SoftplusMLP):
    """A field that branches on ``self.training`` (as dropout or a batch statistic would)."""

    def forward(self, t, z):
        out = super().forward(t, z)
        return out * 0.5 if self.training else out


def test_cuda_graph_follows_the_training_flag(monkeypatch):
    """Captured in train mode, called after .eval(): the eval-mode field must answer, not a replay of train mode."""
    solver._graphs.clear()
    X, _f, z0, t, step = _case("softplus", F32, "cubic", "F3", 128)
    torch.manual_seed(5)
    func = TrainingBranch().to(DEV)
    train = _graph(X, func, z0, t, step)
    func.eval()
    evaluated = _graph(X, func, z0, t, step)
    want = _loop(monkeypatch, X, func, z0, t, step, "rk4")[0]
    assert not torch.equal(train, want)
    assert torch.equal(evaluated, want)
    func.train()
    assert torch.equal(_graph(X, func, z0, t, step), train)


@pytest.mark.parametrize("how", ["data", "double_float", "load_state_dict_assign"])
def test_cuda_graph_follows_replaced_parameter_storage(how, monkeypatch):
    """A parameter given new storage must be read from there.  The old tensors are kept referenced (``keep``), so a
    replay that still read them would read live memory holding the old values, and fail on the result."""
    solver._graphs.clear()
    X, func, z0, t, step = _case("softplus", F32, "cubic", "F3", 128)
    before = _graph(X, func, z0, t, step)
    keep = [p.data for p in func.parameters()]
    if how == "data":
        func.linear1.weight.data = func.linear1.weight.data * 1.5
    elif how == "double_float":
        func.double().float()
        with torch.no_grad():
            func.linear2.bias.add_(0.25)
    else:
        state = {k: v.clone() * (0.5 if k == "linear2.weight" else 1.0) for k, v in func.state_dict().items()}
        func.load_state_dict(state, assign=True)
    assert any(p.data_ptr() != k.data_ptr() for p, k in zip(func.parameters(), keep))
    after = _graph(X, func, z0, t, step)
    want = _loop(monkeypatch, X, func, z0, t, step, "rk4")[0]
    assert not torch.equal(before, want)
    assert torch.equal(after, want)
    del keep


# ---- 3. the torch-operator loop (adjoint=False with gradients) -------------------------------------------------------
GRAD_PATHS = 64


def _grad_pattern(shape, seed=11):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=F64)


def _oracle_grads(X, func, control, z0, t, step, method, g, dtype=F32):
    """Outputs, dL/dz0 and dL/dtheta by fp64 autograd through the oracle's own discrete solve."""
    fc = _oracle(X, func, control, dtype)
    zz = z0.detach().double().clone().requires_grad_(True)
    with torch.enable_grad():
        ys = odeint_port.odeint(fc, zz, t, method=method, options=_options(step)).movedim(0, 1)
        grads = torch.autograd.grad(ys, [zz] + fc.params, g.to(DEV))
    return ys.detach(), grads[0], list(grads[1:])


TORCH_CASES = [(f, c, s, m) for f in LOOP_FIELDS for c in CONTROLS for s in ("F3", "F8") for m in METHODS
               if m == "rk4" or s == "F3"]


@pytest.mark.parametrize("field,control,sname,method", TORCH_CASES)
def test_torch_operator_loop_gradients_match_the_oracle(field, control, sname, method, monkeypatch):
    X, func, z0, t, step = _case(field, F32, control, sname, GRAD_PATHS)
    _refuse(monkeypatch, "loop", "mlp", "linear")
    calls = _Calls(monkeypatch)
    zz = z0.clone().requires_grad_(True)
    out = cde.cdeint(X, func, zz, t, adjoint=False, method=method, options=_options(step))
    g = _grad_pattern(out.shape)
    out.backward(g.to(DEV, F32))
    assert not STEPPERS & set(calls.names), calls.names
    ys, gz, gp = _oracle_grads(X, func, control, z0, t, step, method, g)
    what = "{} {} {} {}".format(field, control, sname, method)
    _report("torch loop outputs | " + what, _path_err(out, ys), 1e-5)
    # at H = 1 a path is one number, which may cross zero: there the bar is a fraction of the whole state's scale
    _report("torch loop dL/dz0 | " + what, (_global_err if field == "h1c1" else _path_err)(zz.grad, gz), 1e-5)
    for p, want in zip(func.parameters(), gp):
        _report("torch loop dL/dtheta | " + what, _global_err(p.grad, want), 3e-5)


@pytest.mark.parametrize("direction", ["increasing", "decreasing"])
@pytest.mark.parametrize("control", CONTROLS)
def test_torch_operator_loop_time_and_knot_gradients(control, direction, monkeypatch):
    """dL/dt and dL/dknots (t.requires_grad, X._t.requires_grad) in fp64 against central differences of the oracle's
    fp64 discrete solve, on F7's uneven knots and times, increasing and reversed.  (No stage time may sit on a knot
    here: there the interval, and with it the one-sided derivative in the knot, would change with the perturbation.)"""
    paths = 16
    X0, func, z0, t, step = _case("time", F64, control, "F7", paths)
    if direction == "decreasing":
        t = t.flip(0)
    src = (X0._rows() if control == "cubic" else X0._coeffs).detach()
    knots = X0._t.detach().clone()
    g = _grad_pattern((paths, t.numel(), 5), 12)

    def oracle_loss(tt, kk):
        fc = _oracle(_control(src, kk, control), func, control, F64)
        with torch.no_grad():
            ys = odeint_port.odeint(fc, z0.double(), tt, method="rk4", options=_options(step)).movedim(0, 1)
        return float((ys * g.to(DEV)).sum())

    _refuse(monkeypatch, "loop", "mlp", "linear")
    tt = t.double().clone().requires_grad_(True)
    kk = knots.clone().requires_grad_(True)
    out = cde.cdeint(_control(src, kk, control), func, z0, tt, adjoint=False, method="rk4", options=_options(step))
    out.backward(g.to(DEV))
    eps = 1e-5
    for name, base, got in (("t", t.double(), tt.grad), ("knots", knots, kk.grad)):
        fd = torch.zeros_like(base)
        for j in range(base.numel()):
            up, down = base.clone(), base.clone()
            up[j] += eps
            down[j] -= eps
            args_up = (up, knots) if name == "t" else (t.double(), up)
            args_down = (down, knots) if name == "t" else (t.double(), down)
            fd[j] = (oracle_loss(*args_up) - oracle_loss(*args_down)) / (2 * eps)
        _report("torch loop dL/d{} | {} {}".format(name, control, direction), _global_err(got, fd), 1e-5)


# ---- 4. the fixed-step adjoint=True ----------------------------------------------------------------------------------
ADJ_PATHS = 96
ADJ_CASES = [(f, c, s, m) for f in ("time", "softplus", "examples") for c in CONTROLS for s in SCHEDULES
             for m in METHODS if m == "rk4" or s == "F3"]
ADJ_CASES += [(f, "cubic", "F3", "rk4") for f in ("prod", "h1c1", "transposed", "linear128x8")]


def _adjoint_run(X, func, z0, t, step, method, g, params=None, t_grad=False):
    zz = z0.clone().requires_grad_(True)
    tt = t.clone().requires_grad_(True) if t_grad else t
    kwargs = {} if params is None else {"adjoint_params": tuple(params)}
    out = cde.cdeint(X, func, zz, tt, adjoint=True, method=method, options=_options(step), **kwargs)
    out.backward(g.to(DEV, out.dtype))
    return out, zz.grad, (tt.grad if t_grad else None)


# The examples' field has relu kinks: where a stage's pre-activation is within the fp32 error of the backward trajectory of
# zero, the package and the fp64 oracle take different sides of the kink, and the Jacobian of that stage -- so that path's
# adjoint -- jumps by O(dt |W1| |W2|), 1e-3 of the path's scale (DESIGN 5, generic routes).  The values are continuous,
# the gradients of the other paths are not affected: every path within KINK_BAR, and all but 1 in 32 within the bar.
KINK_BAR = 5e-3


def _check_adjoint_paths(what, field, got, want, bar):
    """Per-path check of dL/dz0; returns the paths over ``bar`` (only the examples' field may have any: at a kink)."""
    got = got.detach().double().reshape(-1, got.size(-1))
    want = want.detach().double().to(got.device).reshape(got.shape)
    errs = ((got - want).abs().amax(dim=1) / want.abs().amax(dim=1).clamp_min(1e-300)).cpu()
    if field != "examples":
        _report(what, float(errs.max()), bar)
        return errs > bar
    _report(what + " (all but 1 in 32)", float(errs.sort().values[-(1 + errs.numel() // 32)]), bar)
    _report(what.split(" |")[0] + " at a relu kink |" + what.split(" |")[1], float(errs.max()), KINK_BAR)
    return errs > bar


def _ys_for_oracle(out):
    return out.detach().double().movedim(-2, 0).reshape(out.size(-2), -1, out.size(-1))


@pytest.mark.parametrize("field,control,sname,method", ADJ_CASES)
def test_fixed_step_adjoint_matches_the_oracle(field, control, sname, method, monkeypatch):
    X, func, z0, t, step = _case(field, F32, control, sname, ADJ_PATHS)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    _refuse(monkeypatch, "torch", "linear")
    g = _grad_pattern(plain.shape)
    out, gz, _ = _adjoint_run(X, func, z0, t, step, method, g)
    assert torch.equal(out.detach(), plain)
    fc = _oracle(X, func, control, F32)
    wz, wp, _ = AO.fixed_adjoint(fc, _ys_for_oracle(out), g.movedim(-2, 0).to(DEV), t.tolist(), method, step)
    what = "{} {} {} {}".format(field, control, sname, method)
    kinked = _check_adjoint_paths("adjoint dL/dz0 | " + what, field, gz, wz, 1e-5)
    if kinked.any():
        # dL/dtheta sums over the paths, the kinked ones included: once more without their output gradients (the stage
        # times, and z along the backward solve, do not depend on g, so no other path meets a kink)
        g[kinked] = 0.0
        for p in func.parameters():
            p.grad = None
        _o, gz, _ = _adjoint_run(X, func, z0, t, step, method, g)
        wz, wp, _ = AO.fixed_adjoint(fc, _ys_for_oracle(out), g.movedim(-2, 0).to(DEV), t.tolist(), method, step)
        assert not _check_adjoint_paths("adjoint dL/dz0 | kinked paths without gradient " + what, field, gz, wz,
                                        1e-5).any()
    for p, want in zip(func.parameters(), wp):
        _report("adjoint dL/dtheta | " + what, _global_err(p.grad, want), 2e-4)


@pytest.mark.parametrize("sname", ["F3", "F7", "F8"])
@pytest.mark.parametrize("control", CONTROLS)
def test_fixed_step_adjoint_of_coefficients_and_times(control, sname, monkeypatch):
    """The control's coefficients in ``adjoint_params`` and dL/dt with ``t.requires_grad``, on increasing (F3, F7) and
    decreasing (F8) t."""
    X, func, z0, t, step = _case("time", F32, control, sname, ADJ_PATHS)
    src = (X._rows() if control == "cubic" else X._coeffs).detach().clone().requires_grad_(True)
    Xg = _control(src, None if X._default_knots else X._t, control)
    with torch.no_grad():
        plain = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    g = _grad_pattern(plain.shape, 13)
    out, gz, gt = _adjoint_run(Xg, func, z0, t.double(), step, "rk4", g,
                               params=list(func.parameters()) + [src], t_grad=True)
    fc = _oracle(X, func, control, F32)
    fc.control.requires_grad_(True)
    wz, wp, wt = AO.fixed_adjoint(fc, _ys_for_oracle(out), g.movedim(-2, 0).to(DEV), t.tolist(), "rk4", step,
                                  params=fc.params + [fc.control], with_t=True)
    what = "{} {}".format(control, sname)
    _report("adjoint dL/dz0 | coefficients and times " + what, _path_err(gz, wz), 1e-5)
    for p, want in zip(list(func.parameters()) + [src], wp):
        _report("adjoint dL/dtheta | coefficients and times " + what, _global_err(p.grad, want), 2e-4)
    _report("adjoint dL/dt | " + what, _global_err(gt, wt), 2e-4)


# ---- 5. the host-driven dopri5 ---------------------------------------------------------------------------------------
class _Attempts:
    """Wraps Dopri5._attempt: per solver object, every attempt's (t, dt, y0, f0, y1, ks, ratio)."""

    def __init__(self, monkeypatch):
        self.solves = {}
        real = adaptive.Dopri5._attempt

        def attempt(solver_obj, t0, dt, y0, f0):
            y1, ks, ratio = real(solver_obj, t0, dt, y0, f0)
            if not hasattr(solver_obj, "_test_index"):           # (ids are reused once a solver is collected)
                solver_obj._test_index = len(self.solves)
            self.solves.setdefault(solver_obj._test_index, []).append(
                (t0, dt, y0.detach().clone(), f0.detach().clone(), y1.detach().clone(), [k.detach().clone() for k in ks],
                 ratio))
            return y1, ks, ratio

        monkeypatch.setattr(adaptive.Dopri5, "_attempt", attempt)

    def lists(self):
        return list(self.solves.values())


# k1, y1, k7 of one attempt: the bar of test_gpu_adjoint_oracle, per path.  At H = 1 a path is one number, which may
# cross zero: there the bar is a fraction of the whole state's scale.
ATTEMPT_BAR = 1e-5


def _after(t):
    """The first fp32 time after ``t``: where the driver takes the slope after a jump point."""
    t32 = torch.tensor(t, dtype=F32)
    return float(torch.nextafter(t32, t32 + 1))


def _check_host_attempts(records, field_or, rtol, atol, what, jumps=(), err=_path_err, part=None):
    """``part``: the slice of the state the k1, y1, k7 and y_mid checks compare (default: all of it)."""
    part = part or (lambda v: v)
    """Each attempt against AO.attempt from the driver's own state; accept iff ratio <= 1; the next step by AO.next_step
    exactly (unless a jump point shortened it).  Returns the (t, dt, accepted) list for AO.solve's replay."""
    worst = {}

    def note(key, err, bar):
        worst[key] = max(worst.get(key, 0.0), err / bar)
        assert err <= bar, (what, key, err, bar)

    replay = []
    for n, (t0, dt, y0, f0, y1, ks, ratio) in enumerate(records):
        y = y0.double()
        note("k1", err(part(f0), part(field_or(_after(t0) if t0 in jumps else t0, y))), ATTEMPT_BAR)
        res = AO.attempt(field_or, t0, dt, y, f0.double())
        note("y1", err(part(y1), part(res["y1"])), ATTEMPT_BAR)
        note("k7", err(part(ks[-1]), part(res["ks"][6])), ATTEMPT_BAR)
        kmax = torch.stack([k.abs().amax(dim=-1, keepdim=True) for k in res["ks"]]).amax(dim=0)
        mid = adaptive._combine(y0, ks, adaptive._C_MID, dt)
        bar = 1e-6 * y.abs().amax(dim=-1, keepdim=True) + 5e-6 * abs(dt) * kmax
        note("y_mid", float((part((mid.double() - res["y_mid"]).abs() / bar)).max()), 1.0)
        tol = atol + rtol * torch.max(y.abs(), res["y1"].abs())
        r_or = AO.rms(res["err"] / tol)
        note("ratio", abs(ratio - r_or) / (1e-3 * r_or + AO.rms(1e-6 * abs(dt) * kmax / tol)), 1.0)
        accepted = ratio <= 1.0
        replay.append((t0, dt, accepted))
        if n + 1 < len(records):
            t_next, dt_next = records[n + 1][:2]
            assert t_next == (t0 + dt if accepted else t0) or t_next in jumps, (n, t0, dt, t_next)
            on_jump = any(t_next < j < t_next + AO.next_step(dt, ratio) for j in jumps)
            if not on_jump:
                # 0.9 / r^(1/5) here, 0.9 r^(-1/5) in the oracle: the two roundings differ by an ulp at times
                want = AO.next_step(dt, ratio)
                note("next dt rel", abs(dt_next - want) / want, 1e-15)
    for key, val in worst.items():
        _report("dopri5 {} / bar | {}".format(key, what), val, 1.0)
    return replay


DP_LENGTH = 10
DP_PATHS = 200
DP_CASES = {
    # name: (times, rtol, atol, options)
    "increasing": ([0.0, 2.7, 5.0], 1e-4, 1e-6, {}),
    "decreasing": ([5.0, 3.5, 1.25, 0.0], 1e-4, 1e-6, {}),
    "first_step": ([0.3, 0.35, 0.9, 5.0], 1e-4, 1e-6, {"first_step": 0.2}),
    "t_on_gpu": ([0.0, 2.4, 4.5], 1e-4, 1e-6, {}),
}


def _dp_case(field, dtype, control, batch=DP_PATHS):
    hidden, channels, _ = FIELDS[field]
    x, _k, coeffs, z0 = _inputs(channels, hidden, False, PATHS, DP_LENGTH)
    src = (coeffs if control == "cubic" else x)[:batch].to(dtype)
    return _control(src, None, control), _func(field, dtype, seed=1), z0[:batch].to(dtype)


def _routes_for_dopri5(monkeypatch, field):
    _refuse(monkeypatch, "loop", "torch", "mlp", "linear", "device")


DP_FIELDS = ["softplus", "time", "linear128x8", "prod", "h1c1", "transposed", "examples"]


# every field on increasing t; decreasing t, first_step and t on the GPU on the field that reads t
DP_ROWS = [(f, c, "increasing") for f in DP_FIELDS for c in CONTROLS]
DP_ROWS += [("time", c, case) for case in DP_CASES if case != "increasing" for c in CONTROLS]


@pytest.mark.parametrize("field,control,case", DP_ROWS)
def test_host_dopri5_attempt_by_attempt(field, control, case, monkeypatch):
    t_list, rtol, atol, options = DP_CASES[case]
    X, func, z0 = _dp_case(field, F32, control)
    _routes_for_dopri5(monkeypatch, field)
    attempts = _Attempts(monkeypatch)
    calls = _Calls(monkeypatch)
    firsts = []
    real_first = adaptive._initial_step
    monkeypatch.setattr(adaptive, "_initial_step", lambda *a: firsts.append(real_first(*a)) or firsts[-1])
    t = torch.tensor(t_list, dtype=F64, device=DEV if case == "t_on_gpu" else "cpu")
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, rtol=rtol, atol=atol, options=dict(options))
    assert not cde.cdeint.last_stats["device_controlled"]
    assert {"tcde_linear_combination", "tcde_error_ratio_sumsq"} <= set(calls.names)
    assert ("tcde_vector_field_linear" in calls.names) == (field == "linear128x8")
    (records,) = attempts.lists()
    assert cde.cdeint.last_stats["n_accepted"] + cde.cdeint.last_stats["n_rejected"] == len(records)
    fc = _oracle(X, func, control, F32)
    flipped = t_list[0] > t_list[1]
    times = [-v for v in t_list] if flipped else list(t_list)
    field_or = (lambda s, y: -fc(-s, y)) if flipped else fc
    what = "{} {} {}".format(field, control, case)
    replay = _check_host_attempts(records, field_or, rtol, atol, what,
                                  err=_global_err if field == "h1c1" else _path_err)
    if "first_step" in options:
        assert records[0][1] == options["first_step"] and not firsts
    else:
        want = AO.initial_step(field_or, times[0], z0.double(), field_or(times[0], z0.double()), rtol, atol)
        _report("dopri5 first dt rel | " + what, abs(records[0][1] - want) / want, 1e-3)
    want, _rec, _ = AO.solve(field_or, z0.double(), times, rtol, atol, replay=replay)
    _report("dopri5 outputs vs replay | " + what, _global_err(out.movedim(-2, 0), want), 2e-5)


@pytest.mark.parametrize("control", CONTROLS)
def test_host_dopri5_stops_at_jump_points(control, monkeypatch):
    """``jump_t`` at every knot: no step straddles one, the step after a jump restarts from the slope just after it."""
    X, func, z0 = _dp_case("time", F32, control)
    _routes_for_dopri5(monkeypatch, "time")
    attempts = _Attempts(monkeypatch)
    t_list, rtol, atol = [0.0, 2.7, 5.0], 1e-4, 1e-6
    jumps = [float(v) for v in range(DP_LENGTH)]
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, torch.tensor(t_list, dtype=F64), adjoint=False, rtol=rtol, atol=atol,
                         options={"jump_t": X.grid_points})
    (records,) = attempts.lists()
    for t0, dt, *_ in records:
        assert not any(t0 < j < t0 + dt for j in jumps), (t0, dt)
    assert sum(1 for r in records if r[0] in jumps) >= 5
    fc = _oracle(X, func, control, F32)
    replay = _check_host_attempts(records, fc, rtol, atol, "time {} jump_t".format(control), jumps)
    # the oracle's driver has no jump handling: replay it segment by segment between the jumps, restarting the slope
    y, outs = z0.double(), [z0.double()]
    edges = sorted(set([t_list[0], t_list[-1]] + [j for j in jumps if t_list[0] < j < t_list[-1]]))
    for lo, hi in zip(edges[:-1], edges[1:]):
        seg = [r for r in replay if lo <= r[0] < hi]
        inner = [v for v in t_list if lo < v < hi]
        start = (lambda t, v, lo=lo: fc(_after(lo) if t == lo else t, v)) if lo in jumps else fc
        want_seg = AO.solve(start, y, [lo] + inner + [hi], rtol, atol, replay=seg)[0]
        outs += list(want_seg[1:1 + len(inner)]) + ([want_seg[-1]] if hi in t_list else [])
        y = want_seg[-1]
    _report("dopri5 outputs vs replay | jump_t {}".format(control), _global_err(out.movedim(-2, 0), torch.stack(outs)),
            2e-5)


@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("field", ["time", "prod", "linear128x8"])
def test_host_dopri5_fp64_against_the_free_running_oracle(field, control, monkeypatch):
    """In fp64, inside one spline interval (where a step straddling a knot would make the decisions depend on rounding):
    the oracle's own step sequence and outputs within 1e-10."""
    X, func, z0 = _dp_case(field, F64, control, 64)
    _routes_for_dopri5(monkeypatch, field)
    t_list, rtol, atol = [4.05, 4.3, 4.62, 4.95], 1e-9, 1e-11
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, torch.tensor(t_list, dtype=F64), adjoint=False, rtol=rtol, atol=atol)
    stats = cde.cdeint.last_stats
    want, records, _ = AO.solve(_oracle(X, func, control, F64), z0.double(), t_list, rtol, atol)
    assert stats["n_accepted"] == sum(r.accepted for r in records) > 5
    assert stats["n_rejected"] == sum(not r.accepted for r in records)
    _report("dopri5 fp64 outputs | {} {}".format(field, control), _global_err(out.movedim(-2, 0), want), 1e-10)


def test_host_dopri5_is_deterministic_on_a_large_state(monkeypatch):
    """1.2 M state elements (past the stepper kernels' grid cap): two runs give the same ratios, steps and outputs, bit
    for bit (the error partials are summed in a fixed order)."""
    gen = torch.Generator(device=DEV).manual_seed(4)
    x = (torch.randn(240_000, DP_LENGTH, 3, generator=gen, device=DEV) / 4).cumsum(1)
    z0 = torch.randn(240_000, 5, generator=gen, device=DEV)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    func = _func("time", F32)
    runs = []
    for _ in range(2):
        attempts = _Attempts(monkeypatch)
        with torch.no_grad():
            out = cde.cdeint(X, func, z0, torch.tensor([0.0, 9.0], dtype=F64), adjoint=False)
        (records,) = attempts.lists()
        runs.append(([(r[0], r[1], r[6]) for r in records], out))
        monkeypatch.undo()
    assert len(runs[0][0]) > 5
    assert runs[0][0] == runs[1][0]
    assert torch.equal(runs[0][1], runs[1][1])


def _misaligned_cubic(X):
    rows = X._rows()
    buf = torch.empty(rows.numel() + 1, dtype=rows.dtype, device=rows.device)
    view = buf[1:].view(rows.shape)
    view.copy_(rows)
    assert view.data_ptr() % 16 != 0
    return cde.CubicSpline(view)


@pytest.mark.parametrize("case", ["misaligned_cubic", "hidden_300"])
def test_dopri5_falls_back_where_the_kernels_refuse(case, monkeypatch):
    """The default method on a problem a dopri5 kernel refuses answers from the host driver, like the fixed-step methods
    answer from their stage loop: control rows off a 16-byte boundary (the device controller's refusal) run the host
    driver with the kernel field; hidden 300 (the kernel field's refusal) runs it with the torch-operator field."""
    if case == "misaligned_cubic":
        X, func, z0 = _dp_case("softplus", F32, "cubic", 256)
        torch.manual_seed(3)
        func = cde.LinearVectorField(32, 8).to(DEV)
        X = _misaligned_cubic(X)
    else:
        x = _inputs(2, 300, False, PATHS, DP_LENGTH)[0][:64]
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
        torch.manual_seed(4)
        func = cde.LinearVectorField(300, 2).to(DEV)
        z0 = torch.randn(64, 300, generator=torch.Generator().manual_seed(5)).to(DEV)
    calls = _Calls(monkeypatch)
    attempts = _Attempts(monkeypatch)
    t_list, rtol, atol = [0.0, 3.7, 9.0], 1e-4, 1e-6
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, torch.tensor(t_list, dtype=F64))
    assert not cde.cdeint.last_stats["device_controlled"]
    want_refused = "tcde_dopri5_linear_attempts" if case == "misaligned_cubic" else "tcde_vector_field_linear"
    assert want_refused in calls.refused
    if case == "misaligned_cubic":                                  # the kernel field served every attempt
        assert "tcde_vector_field_linear" in calls.names and "tcde_vector_field_linear" not in calls.refused
    fc = AO.LinearCDE(X._rows().detach().double(), X._t.detach().cpu(), func.linear.weight.detach().double(),
                      func.linear.bias.detach().double(), "cubic", time_dtype=F32)
    (records,) = attempts.lists()
    replay = _check_host_attempts(records, fc, rtol, atol, "fallback " + case)
    want, _rec, _ = AO.solve(fc, z0.double(), t_list, rtol, atol, replay=replay)
    _report("dopri5 outputs vs replay | fallback " + case, _global_err(out.movedim(-2, 0), want), 2e-5)


# ---- 6. the dopri5 adjoint=True --------------------------------------------------------------------------------------
DP_ADJ_PATHS = 64


@pytest.mark.parametrize("control", CONTROLS)
@pytest.mark.parametrize("field", ["time", "softplus", "prod", "examples"])
def test_dopri5_adjoint_replayed_by_the_oracle(field, control, monkeypatch):
    """The backward's attempts on the packed augmented state (z, a, dL/dtheta), segment by segment, replayed by the
    oracle on FuncCDE's augmented field: a(t_0) within 2e-5, dL/dtheta within 2e-4 of the replay.  The examples' field
    is the examples' training step (dopri5, adjoint=True); at its relu kinks the adjoint part of one attempt may jump
    (KINK_BAR), so its attempts are compared on z, the part of the state whose slope is continuous."""
    X, func, z0 = _dp_case(field, F32, control, DP_ADJ_PATHS)
    _refuse(monkeypatch, "loop", "torch", "mlp", "linear", "device")
    attempts = _Attempts(monkeypatch)
    t_list, rtol, atol = [0.0, 2.6, 5.0], 1e-4, 1e-6
    zz = z0.clone().requires_grad_(True)
    out = cde.cdeint(X, func, zz, torch.tensor(t_list, dtype=F64), rtol=rtol, atol=atol)
    g = _grad_pattern(out.shape, 14)
    out.backward(g.to(DEV, F32))
    solves = attempts.lists()
    assert len(solves) == 1 + len(t_list) - 1                     # the forward solve, then one per segment
    fc = _oracle(X, func, control, F32)
    params = fc.params
    sizes = [p.numel() for p in params]
    n_z = z0.numel()
    ys = _ys_for_oracle(out)
    gys = g.movedim(-2, 0).to(DEV)

    def aug(t, v):
        z, a = v[:n_z].view(z0.shape), v[n_z:2 * n_z].view(z0.shape)
        f, gz, gp = fc.vjp(t, z, a, params)
        return torch.cat([x.reshape(-1) for x in [f, -gz] + [-p for p in gp]])

    def aug_s(s, v):                                               # the package's backward runs in s = -t
        return -aug(-s, v)

    a = gys[-1]
    gp = [torch.zeros(n, dtype=F64, device=DEV) for n in sizes]
    for seg, i in zip(solves[1:], range(len(t_list) - 1, 0, -1)):
        v0 = torch.cat([ys[i].reshape(-1), a.reshape(-1)] + gp)
        replay = _check_host_attempts(seg, aug_s, rtol, atol, "adjoint {} {} segment {}".format(field, control, i),
                                      part=(lambda v: v[:n_z]) if field == "examples" else None)
        v1 = AO.solve(aug_s, v0, [-t_list[i], -t_list[i - 1]], rtol, atol, replay=replay)[0][-1]
        a = v1[n_z:2 * n_z].view(z0.shape) + gys[i - 1]
        gp = list(torch.split(v1[2 * n_z:], sizes))
    what = "{} {}".format(field, control)
    _check_adjoint_paths("dopri5 adjoint a(t0) | " + what, field, zz.grad, a, 2e-5)
    for p, want in zip(func.parameters(), gp):
        _report("dopri5 adjoint dL/dtheta | " + what, _global_err(p.grad, want.view_as(p)), 2e-4)
