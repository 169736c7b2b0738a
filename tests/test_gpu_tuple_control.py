"""TupleControl and tuple states of cdeint (reference misc.py:129-166, solver.py:68-98, 131-133, 238-243).

CPU: TupleControl's construction, ``state_dict`` keys and ``grid_points``; cdeint's tuple argument errors message for
message; the fp64 tuple oracle's anchors (one member = the tensor oracle bit for bit, decoupled members = separate
solves).  GPU: the grouped entries bit-equal to per-member calls at the size, alignment and member-count edges; every
tuple route against the fp64 oracle (``oracle/tuple_oracle.py``) with the bars of test_gpu_generic_routes.py, each route
proving itself by the library calls it makes; invariants; the reference's own ``test_tuple_input``."""
import copy

import pytest
import torch

import torchcde_b200 as cde
from oracle import adaptive_oracle as AO
from oracle import odeint_port, reference_loader
from oracle import tuple_oracle as TO
from test_gpu_generic_routes import BAR, _Calls, _global_err, _path_err, _times
from test_host_logic import FIXED_SCHEDULES
from torchcde_b200 import _lib, adaptive, solver, tuple_solver

F32, F64 = torch.float32, torch.float64
DEV = "cuda"


# ============================================================================================================ CPU
def _cubic_cpu(batch, length, channels, t=None, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return cde.CubicSpline(torch.randn(*batch, length - 1, 4 * channels, generator=gen), t=t)


def test_tuple_control_construction_errors():
    with pytest.raises(ValueError, match="^Expected one or more controls to batch together.$"):
        cde.TupleControl()
    a = _cubic_cpu((2,), 10, 2)
    b = _cubic_cpu((), 6, 1)                 # interval [0, 5] against [0, 9]
    with pytest.raises(ValueError, match="^Can only batch togehter controls over the same interval.$"):
        cde.TupleControl(a, b)


def test_tuple_control_state_dict_keys_and_exports():
    a = _cubic_cpu((2,), 10, 2)
    b = cde.LinearInterpolation(torch.randn(10, 3))
    X = cde.TupleControl(a, b)
    # the reference's keys: a ModuleList named ``controls`` of the members' own buffers
    assert list(X.state_dict()) == ["controls.0._t", "controls.0._a", "controls.0._b", "controls.0._two_c",
                                    "controls.0._three_d", "controls.1._t", "controls.1._coeffs", "controls.1._derivs"]
    assert isinstance(X.controls, torch.nn.ModuleList)
    assert cde.misc.TupleControl is cde.TupleControl and "TupleControl" in cde.__all__
    assert torch.equal(X.interval, a.interval)


def test_tuple_control_grid_points():
    a = _cubic_cpu((2,), 10, 2)
    b = cde.LinearInterpolation(torch.randn(3, 10, 1))
    assert torch.equal(cde.TupleControl(a, b).grid_points, a.grid_points)
    uneven = torch.tensor([0.0, 0.5, 2.0, 3.5, 5.0, 6.0, 7.25, 8.0, 8.5, 9.0])
    c = cde.LinearInterpolation(torch.randn(10, 1), t=uneven)
    d = _cubic_cpu((), 4, 1, t=torch.tensor([0.0, 3.0, 6.0, 9.0]))      # other length, same interval
    for X in (cde.TupleControl(a, c), cde.TupleControl(a, d)):
        with pytest.raises(RuntimeError, match="^Batch of controls have different grid points.$"):
            X.grid_points


class _UserControl(torch.nn.Module):
    """A control of the user's own: ``derivative`` answers with whatever it was given."""

    def __init__(self, answer):
        super().__init__()
        self.answer = answer

    def derivative(self, t):
        return self.answer


def _z(*shape):
    return torch.zeros(*shape)


# (control answer, func output, is_prod, z0) -> the reference's message (solver.py:68-98)
_ERROR_CASES = {
    "dx-not-tuple": (_z(2, 1), (_z(2, 3, 1),), False, (_z(2, 3),),
                     "z0 is a tuple/list and so X.derivative must return a tuple/list as well."),
    "dx-length": ((_z(2, 1), _z(1)), (_z(2, 3, 1),), False, (_z(2, 3),),
                  "z0 and X.derivative(t) must be tuples of the same length."),
    "func-not-tuple": ((_z(2, 1),), _z(2, 3, 1), False, (_z(2, 3),),
                       "z0 is a tuple/list and so func must return a tuple/list as well."),
    "func-length": ((_z(2, 1),), (_z(2, 3, 1), _z(3, 1)), False, (_z(2, 3),),
                    "z0 and func(t, z) must be tuples of the same length."),
    "dx-member": ((1.0,), (_z(2, 3, 1),), False, (_z(2, 3),), "X.derivative must return a tensor or tuple of tensors."),
    "func-member": ((_z(2, 1),), (1.0,), False, (_z(2, 3),), "func must return a tensor or tuple/list of tensors."),
    "dx-batch": ((_z(4, 1),), (_z(2, 3, 1),), False, (_z(2, 3),),
                 "X.derivative did not return a tensor with the same number of batch dimensions as z0. X.derivative "
                 "returned shape (4, 1) (meaning (4,) batch dimensions), whilst z0 has shape (2, 3) (meaning (2,) batch "
                 "dimensions)."),
    "func-hidden": ((_z(2, 1),), (_z(2, 4, 1),), False, (_z(2, 3),),
                    "func did not return a tensor with the same number of hidden channels as z0. func returned shape "
                    "(2, 4, 1) (meaning 4 channels), whilst z0 has shape (2, 3) (meaning 3 channels)."),
    "func-channels": ((_z(2, 1),), (_z(2, 3, 2),), False, (_z(2, 3),),
                      "func did not return a tensor with the same number of input channels as X.derivative returned. "
                      "func returned shape (2, 3, 2) (meaning 2 channels), whilst X.derivative returned shape (2, 1) "
                      "(meaning 1 channels)."),
    "prod-not-tuple": ((_z(2, 1),), _z(2, 3), True, (_z(2, 3),),
                       "z0 is a tuple/list and so func.prod must return a tuple/list as well."),
    "prod-length": ((_z(2, 1),), (_z(2, 3), _z(3)), True, (_z(2, 3),),
                    "z0 and func.prod(t, z, dXdt) must be tuples of the same length."),
    "prod-member": ((_z(2, 1),), (1.0,), True, (_z(2, 3),), "func.prod must return a tensor or tuple/list of tensors."),
    "prod-shape": ((_z(2, 1),), (_z(2, 4),), True, (_z(2, 3),),
                   "func.prod did not return a tensor with the same shape as z0. func.prod returned shape (2, 4) whilst "
                   "z0 has shape (2, 3)."),
}


def _error_problem(name):
    answer, result, is_prod, z0, _ = _ERROR_CASES[name]
    X = _UserControl(answer)
    if is_prod:
        class F:
            def prod(self, t, z, dxdt):
                return result
        return X, F(), z0
    return X, (lambda t, z: result), z0


@pytest.mark.parametrize("name", list(_ERROR_CASES))
def test_cdeint_tuple_argument_errors_match_the_reference(name):
    X, func, z0 = _error_problem(name)
    t = torch.tensor([0.0, 1.0])
    with pytest.raises(ValueError) as got:
        cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options={"step_size": 0.5})
    assert str(got.value) == _ERROR_CASES[name][4]
    if reference_loader.reference_available():
        ref = reference_loader.load_reference()
        with pytest.raises(ValueError) as want:
            ref.solver._check_compatability(X, func, z0, t)
        assert str(got.value) == str(want.value)


def test_torchsde_backend_names_the_tuple_state():
    X, func, z0 = _error_problem("dx-batch")
    with pytest.raises(NotImplementedError, match="tuple / list state"):
        cde.cdeint(X, func, z0, torch.tensor([0.0, 1.0]), backend="torchsde", method="reversible_heun")


# ---- the oracle's anchors -------------------------------------------------------------------------------------------
def _oracle_members(seed=0):
    gen = torch.Generator().manual_seed(seed)
    rows_a = torch.randn(3, 9, 4 * 2, generator=gen, dtype=F64) / 4       # cubic, 3 paths, 2 channels, knots 0..9
    knots_b = torch.tensor([0.0, 0.7, 2.0, 2.9, 4.4, 5.0, 6.5, 7.1, 8.0, 9.0], dtype=F64)
    x_b = torch.randn(4, 10, 1, generator=gen, dtype=F64).cumsum(1) / 4   # linear, 4 paths, 1 channel, uneven knots
    wa = torch.randn(3, 3 * 2, generator=gen, dtype=F64) / 2
    wb = torch.randn(2, 2, generator=gen, dtype=F64) / 2
    ga = lambda t, z: torch.tanh(z @ wa).view(*z.shape[:-1], 3, 2)      # noqa: E731
    gb = lambda t, z: torch.sin(z @ wb + t).unsqueeze(-1)              # noqa: E731
    za = torch.randn(3, 3, generator=gen, dtype=F64)
    zb = torch.randn(4, 2, generator=gen, dtype=F64)
    return (rows_a, torch.arange(10, dtype=F64), "cubic", ga, za), (x_b, knots_b, "linear", gb, zb)


@pytest.mark.parametrize("method,step", [("rk4", 0.5), ("midpoint", 0.3), ("euler", 0.25), ("rk4", None)])
def test_oracle_one_member_equals_the_tensor_oracle(method, step):
    (rows, knots, kind, g, z0), _ = _oracle_members()
    t = torch.tensor([0.0, 2.5, 9.0], dtype=F64)
    tensor = odeint_port.odeint(AO.FuncCDE(rows, knots, g, kind), z0, t, method=method,
                                options={} if step is None else {"step_size": step})
    packed = TO.Packed(TO.TupleFuncCDE([(rows, knots, kind)], lambda ts, zs: (g(ts, zs[0]),)), [z0.shape])
    tup = odeint_port.odeint(packed, packed.pack([z0]), t, method=method,
                             options={} if step is None else {"step_size": step})
    assert torch.equal(packed.unpack(tup)[0], tensor)


@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
def test_oracle_decoupled_members_equal_separate_solves(method):
    a, b = _oracle_members(1)
    t = torch.tensor([9.0, 4.0, 0.0], dtype=F64)                         # decreasing t
    cde_t = TO.TupleFuncCDE([a[:3], b[:3]], lambda ts, zs: (a[3](ts, zs[0]), b[3](ts, zs[1])))
    packed = TO.Packed(cde_t, [a[4].shape, b[4].shape])
    ys = packed.unpack(odeint_port.odeint(packed, packed.pack([a[4], b[4]]), t, method=method,
                                          options={"step_size": 0.5}))
    for m, y in zip((a, b), ys):
        alone = odeint_port.odeint(AO.FuncCDE(m[0], m[1], m[3], m[2]), m[4], t, method=method, options={"step_size": 0.5})
        assert torch.equal(y, alone)


def test_oracle_mixed_norm_is_the_largest_member_rms():
    norm = TO.mixed_norm([2, 0, 3])
    x = torch.tensor([3.0, 4.0, 1.0, 1.0, 1.0], dtype=F64)
    assert norm(x) == pytest.approx((12.5) ** 0.5)
    assert adaptive.MixedNorm([2, 0, 3])(x) == norm(x)


# ============================================================================================================ GPU
gpu = pytest.mark.gpu


def _spline_member(kind, batch, channels, knots, dtype, gen, misalign):
    """(control rows view, knots, n_rows): cubic rows [batch][L-1][4C] / linear values [batch][L][C], one element off a
    16-byte boundary when ``misalign``."""
    n_rows = knots.numel() - 1 if kind == "cubic" else knots.numel()
    width = 4 * channels if kind == "cubic" else channels
    n = batch * n_rows * width
    buf = torch.randn(n + 1, generator=gen, dtype=F64).to(dtype).to(DEV)
    rows = (buf[1:] if misalign else buf[:n]).view(batch, n_rows, width)
    return rows, knots.to(DEV, dtype), n_rows


def _queries(knots, n, gen, dtype):
    t = torch.rand(n, generator=gen, dtype=F64) * float(knots[-1] - knots[0]) + float(knots[0])
    t[0], t[-1] = float(knots[0]), float(knots[-1])
    kk = knots.cpu().to(dtype)
    index = (torch.bucketize(t.to(dtype), kk) - 1).clamp(0, kk.numel() - 2)
    return index.to(torch.int32).to(DEV), (t.to(dtype) - kk[index]).to(DEV)


GUARD = 7


def _guarded(n, dtype):
    """A buffer of n elements with GUARD NaN-patterned elements on each side: (inner view, whole buffer)."""
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device=DEV)
    buf[:GUARD] = -123.0
    buf[-GUARD:] = 456.0
    return buf[GUARD:GUARD + n], buf


def _uneven_knots(length, seed):
    w = 0.6 + 0.8 * torch.rand(length - 1, generator=torch.Generator().manual_seed(seed), dtype=F64)
    k = torch.cat([torch.zeros(1, dtype=F64), w.cumsum(0)])
    return k / k[-1] * (length - 1)


def _member_specs():
    """Mixed kinds, channels 1 / 3 / 8 / 33, batches 0 / 1 / 63 / 1000, default and uneven knots, rows on and off a
    16-byte boundary; 20 members, more than one launch's 16."""
    specs = []
    kinds, chans, batches = ["cubic", "linear"], [1, 3, 8, 33], [0, 1, 63, 1000]
    for k in range(20):
        specs.append((kinds[k % 2], batches[(k // 2) % 4], chans[k % 4], k % 3 == 0, k % 5 == 1))
    return specs


@gpu
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("derivative", [1, 0])
@pytest.mark.parametrize("n_members", [1, 3, 20])
def test_grouped_spline_eval_is_bit_equal_to_per_member_calls(dtype, derivative, n_members):
    gen = torch.Generator().manual_seed(5 + n_members)
    specs = _member_specs()[:n_members] if n_members != 3 else [_member_specs()[i] for i in (2, 4, 9)]
    descs = (_lib.SplineMember * len(specs))()
    keep, wants = [], []
    for d, (kind, batch, channels, uneven, misalign) in zip(descs, specs):
        knots = _uneven_knots(17, batch + channels) if uneven else torch.arange(17, dtype=F64)
        rows, kt, n_rows = _spline_member(kind, batch, channels, knots, dtype, gen, misalign)
        index, frac = _queries(knots, 5, gen, dtype)
        inner, whole = _guarded(batch * 5 * channels, dtype)
        want = torch.zeros(max(batch * 5 * channels, 1), dtype=dtype, device=DEV)
        if batch:
            _lib.call("tcde_spline_eval", _lib.ptr(rows), _lib.ptr(kt), _lib.ptr(index), _lib.ptr(frac), _lib.ptr(want),
                      batch, n_rows, channels, 5, _lib.CONTROL_CUBIC if kind == "cubic" else _lib.CONTROL_LINEAR,
                      derivative, _lib.dtype_code(dtype), _lib.stream_of(rows))
        d.control, d.knot_t, d.index, d.frac, d.out = (rows.data_ptr(), kt.data_ptr(), index.data_ptr(),
                                                       frac.data_ptr(), inner.data_ptr())
        d.n_paths, d.n_rows, d.channels, d.n_times = batch, n_rows, channels, 5
        d.control_kind = _lib.CONTROL_CUBIC if kind == "cubic" else _lib.CONTROL_LINEAR
        keep += [rows, kt, index, frac]
        wants.append((inner, whole, want[:batch * 5 * channels]))
    _lib.call("tcde_spline_eval_grouped", descs, len(specs), derivative, _lib.dtype_code(dtype),
              _lib.stream_of(keep[0]))
    torch.cuda.synchronize()
    for inner, whole, want in wants:
        assert torch.equal(inner, want)
        assert (whole[:GUARD] == -123.0).all() and (whole[-GUARD:] == 456.0).all()


@gpu
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("n_members", [1, 4, 20])
def test_grouped_field_contract_is_bit_equal_to_per_member_calls(dtype, n_members):
    gen = torch.Generator().manual_seed(11 + n_members)
    specs = _member_specs()[:n_members] if n_members != 4 else [_member_specs()[i] for i in (1, 3, 6, 8)]
    descs = (_lib.ContractMember * len(specs))()
    keep, wants = [], []
    for k, (d, (_, batch, channels, _u, misalign)) in enumerate(zip(descs, specs)):
        hidden = [1, 5, 32, 7][k % 4]
        stride = channels * (1 + k % 4)                      # the stages of a step side by side
        f = torch.randn(batch * hidden * channels + 1, generator=gen, dtype=F64).to(dtype).to(DEV)
        f = f[1:] if misalign else f[:-1]
        dx = torch.randn(batch * stride + 1, generator=gen, dtype=F64).to(dtype).to(DEV)
        dx = dx[1:] if misalign else dx[:-1]
        inner, whole = _guarded(batch * hidden, dtype)
        want = torch.zeros(max(batch * hidden, 1), dtype=dtype, device=DEV)
        if batch:
            _lib.call("tcde_field_contract", _lib.ptr(f), _lib.ptr(dx), _lib.ptr(want), batch, hidden, channels, stride,
                      -1.0, _lib.dtype_code(dtype), _lib.stream_of(f))
        d.field, d.dx, d.out = f.data_ptr(), dx.data_ptr(), inner.data_ptr()
        d.n_paths, d.hidden, d.channels, d.dx_stride = batch, hidden, channels, stride
        keep += [f, dx]
        wants.append((inner, whole, want[:batch * hidden]))
    _lib.call("tcde_field_contract_grouped", descs, len(specs), -1.0, _lib.dtype_code(dtype), _lib.stream_of(keep[0]))
    torch.cuda.synchronize()
    for inner, whole, want in wants:
        assert torch.equal(inner, want)
        assert (whole[:GUARD] == -123.0).all() and (whole[-GUARD:] == 456.0).all()


@gpu
def test_grouped_entries_report_argument_errors():
    descs = (_lib.SplineMember * 1)()
    descs[0].n_paths, descs[0].n_rows, descs[0].channels, descs[0].n_times, descs[0].control_kind = 2, 3, 1, 1, 0
    with pytest.raises(ValueError, match="member 0: null data pointer"):
        _lib.call("tcde_spline_eval_grouped", descs, 1, 1, _lib.F32, None)
    c = (_lib.ContractMember * 1)()
    c[0].n_paths, c[0].hidden, c[0].channels, c[0].dx_stride = 1, 1, 2, 1
    with pytest.raises(ValueError, match="member 0: bad sizes"):
        _lib.call("tcde_field_contract_grouped", c, 1, 1.0, _lib.F32, None)


# ---- routes against the oracle -------------------------------------------------------------------------------------
PATHS, LENGTH = 600, 40


class TupleField(torch.nn.Module):
    """Member A (H 5, C 3) reads the stage time; member B (H 4, C 2) also reads member A's state (coupled members)."""

    def __init__(self):
        super().__init__()
        self.la = torch.nn.Linear(5, 15)
        self.v = torch.nn.Parameter(torch.randn(15) / 8)
        self.lb = torch.nn.Linear(4, 8)
        self.cb = torch.nn.Linear(5, 8, bias=False)

    def forward(self, t, z):
        za, zb = z
        fa = torch.tanh(self.la(za) + t * self.v).view(*za.shape[:-1], 5, 3)
        cross = self.cb(za) if za.shape[:-1] == zb.shape[:-1] else 0.0
        fb = torch.tanh(self.lb(zb) + cross).view(*zb.shape[:-1], 4, 2)
        return fa, fb


class TupleProd(torch.nn.Module):
    """A tuple field given by its products: member i's is tanh(Linear(z_i)).view(H, C) @ dX_i - z_i |dX_i|^2 / 4."""

    def __init__(self):
        super().__init__()
        self.la, self.lb = torch.nn.Linear(5, 15), torch.nn.Linear(4, 8)

    def prod(self, t, z, dx):
        out = []
        for zi, di, lin, c in zip(z, dx, (self.la, self.lb), (3, 2)):
            m = torch.tanh(lin(zi)).view(*zi.shape[:-1], -1, c)
            out.append((m @ di.unsqueeze(-1)).squeeze(-1) - 0.25 * zi * (di * di).sum(-1, keepdim=True))
        return tuple(out)


def _tuple_case(dtype, uneven, paths=PATHS, prod=False, seed=0):
    """(X, func, z0, src) on the device: member A a cubic spline on the default knots 0..39, member B a linear
    interpolation on its own knots (uneven: widths in [0.6, 1.4) scaled to [0, 39])."""
    gen = torch.Generator().manual_seed(31 + seed)
    xa = (torch.randn(paths, LENGTH, 3, generator=gen, dtype=F64) / 4).cumsum(1).to(dtype).to(DEV)
    xb = (torch.randn(paths, LENGTH, 2, generator=gen, dtype=F64) / 4).cumsum(1).to(dtype).to(DEV)
    kb = (_uneven_knots(LENGTH, 3) if uneven else torch.arange(LENGTH, dtype=F64)).to(dtype).to(DEV)
    ca = cde.hermite_cubic_coefficients_with_backward_differences(xa)
    X = cde.TupleControl(cde.CubicSpline(ca), cde.LinearInterpolation(xb, t=kb))
    torch.manual_seed(77 + seed)
    func = (TupleProd() if prod else TupleField()).to(DEV).to(dtype)
    z0 = (torch.randn(paths, 5, generator=gen, dtype=F64).to(dtype).to(DEV),
          torch.randn(paths, 4, generator=gen, dtype=F64).to(dtype).to(DEV))
    return X, func, z0, (ca, xb, kb)


def _tuple_oracle(X, func, dtype, z0):
    a, b = X.controls
    f64 = copy.deepcopy(func).double()
    prod = hasattr(func, "prod")
    members = [(a._rows().detach().double(), a._t.detach().cpu(), "cubic"),
               (b._coeffs.detach().double(), b._t.detach().cpu(), "linear")]
    t_cde = TO.TupleFuncCDE(members, f64.prod if prod else f64, time_dtype=dtype, prod=prod)
    return TO.Packed(t_cde, [z.shape for z in z0]), f64


def _options(step, **extra):
    return dict({} if step is None else {"step_size": step}, **extra)


def _refuse_torch_loop(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("the torch-operator loop served a grouped-loop case")
    monkeypatch.setattr(solver, "_generic_solve", refuse)
    monkeypatch.setattr(solver, "_generic_solve_kernels", refuse)


def _n_steps(t, step, method, dtype):
    from torchcde_b200.schedule import build_schedule
    return build_schedule(t, torch.arange(LENGTH, dtype=dtype), LENGTH - 1, method, step, dtype).n_steps


_LOOP_CASES = [("rk4", s, F32) for s in FIXED_SCHEDULES] + [(m, s, F32) for m in ("midpoint", "euler")
                                                              for s in ("F3", "F8")] + [("rk4", "F3", F64)]


@gpu
@pytest.mark.parametrize("method,sname,dtype", _LOOP_CASES,
                         ids=["{}-{}-{}".format(m, s, "fp32" if d == F32 else "fp64") for m, s, d in _LOOP_CASES])
def test_grouped_loop_matches_the_oracle(method, sname, dtype, monkeypatch):
    X, func, z0, _ = _tuple_case(dtype, FIXED_SCHEDULES[sname][2] or sname in ("F3", "F8"))
    t, step = _times(sname)
    _refuse_torch_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=_options(step))
    monkeypatch.undo()
    n_steps = _n_steps(t, step, method, dtype)
    assert calls.names.count("tcde_spline_eval_grouped") == n_steps
    assert calls.names.count("tcde_field_contract_grouped") == n_steps * {"rk4": 4, "midpoint": 2, "euler": 1}[method]
    # per-member evaluations: only the reference's one compatibility evaluation at t[0], before the loop
    loop = calls.names[calls.names.index("tcde_spline_eval_grouped"):]
    assert calls.names.count("tcde_spline_eval") == 2 and "tcde_spline_eval" not in loop
    assert "tcde_field_contract" not in calls.names
    packed, _ = _tuple_oracle(X, func, dtype, z0)
    with torch.no_grad():
        want = packed.unpack(odeint_port.odeint(packed, packed.pack([z.double() for z in z0]), t.to(DEV),
                                                method=method, options=_options(step)))
    for o, w, z in zip(out, want, z0):
        assert o.shape == z.shape[:-1] + (t.numel(), z.size(-1)) and o.dtype == dtype
        assert torch.equal(o[:, 0], z)
        assert _path_err(o, w.movedim(0, 1)) <= BAR[dtype]


@gpu
def test_prod_field_runs_the_grouped_evaluation(monkeypatch):
    X, func, z0, _ = _tuple_case(F32, True, prod=True)
    t, step = _times("F3")
    _refuse_torch_loop(monkeypatch)
    calls = _Calls(monkeypatch)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    monkeypatch.undo()
    assert "tcde_spline_eval_grouped" in calls.names and "tcde_field_contract_grouped" not in calls.names
    packed, _ = _tuple_oracle(X, func, F32, z0)
    with torch.no_grad():
        want = packed.unpack(odeint_port.odeint(packed, packed.pack([z.double() for z in z0]), t.to(DEV), method="rk4",
                                                options=_options(step)))
    for o, w in zip(out, want):
        assert _path_err(o, w.movedim(0, 1)) <= BAR[F32]


@gpu
def test_one_member_tuple_equals_the_tensor_state_loop():
    X, func, z0, _ = _tuple_case(F32, False)
    a = X.controls[0]
    t, step = _times("F3")
    fa = lambda t, z: torch.tanh(func.la(z) + t * func.v).view(*z.shape[:-1], 5, 3)     # noqa: E731
    with torch.no_grad():
        tensor = cde.cdeint(a, fa, z0[0], t, adjoint=False, method="rk4", options=_options(step))
        tup = cde.cdeint(cde.TupleControl(a), lambda t, z: (fa(t, z[0]),), (z0[0],), t, adjoint=False, method="rk4",
                         options=_options(step))
    assert isinstance(tup, tuple) and len(tup) == 1
    assert torch.equal(tup[0], tensor)


@gpu
def test_cuda_graph_replays_the_grouped_loop_and_runs_are_deterministic():
    X, func, z0, _ = _tuple_case(F32, True)
    t, step = _times("F8")
    with torch.no_grad():
        eager = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
        again = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
        graph = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step, cuda_graph=True))
        replay = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step, cuda_graph=True))
    for e, a, g, r in zip(eager, again, graph, replay):
        assert torch.equal(e, a) and torch.equal(e, g) and torch.equal(e, r)
    assert any(k[1] == id(X) for k in tuple_solver._graphs)


@gpu
def test_adjoint_false_gradients_match_fp64_autograd_through_the_oracle():
    X, func, z0, (ca, xb, kb) = _tuple_case(F32, True, paths=48)
    ca = ca.detach().requires_grad_(True)
    xb = xb.detach().requires_grad_(True)
    X = cde.TupleControl(cde.CubicSpline(ca), cde.LinearInterpolation(xb, t=kb))
    z0 = tuple(z.detach().requires_grad_(True) for z in z0)
    t, step = _times("F3")
    out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=_options(step))
    gen = torch.Generator().manual_seed(3)
    ws = [torch.randn(o.shape, generator=gen, dtype=F64).to(DEV) for o in out]
    params = list(func.parameters())
    got = torch.autograd.grad(sum((o.double() * w).sum() for o, w in zip(out, ws)), list(z0) + params + [ca, xb])

    ca64 = ca.detach().double().requires_grad_(True)
    xb64 = xb.detach().double().requires_grad_(True)
    z64 = [z.detach().double().requires_grad_(True) for z in z0]
    f64 = copy.deepcopy(func).double()
    t_cde = TO.TupleFuncCDE([(ca64, X.controls[0]._t.detach().cpu(), "cubic"), (xb64, kb.cpu(), "linear")], f64,
                            time_dtype=F32)
    packed = TO.Packed(t_cde, [z.shape for z in z0])
    ys = packed.unpack(odeint_port.odeint(packed, packed.pack(z64), t.to(DEV), method="rk4", options=_options(step)))
    want = torch.autograd.grad(sum((y.movedim(0, -2) * w).sum() for y, w in zip(ys, ws)),
                               z64 + list(f64.parameters()) + [ca64, xb64])
    for g, w in zip(got, want):
        assert _global_err(g, w) <= 1e-4


@gpu
def test_adjoint_false_time_and_knot_gradients_of_decoupled_members_are_the_tensor_states():
    """Decoupled members: the tuple's gradients with respect to t and to member B's knots are the sums of the two
    tensor-state solves' (each pinned by test_gpu_generic_routes.py)."""
    _, _, z0, (ca, xb, kb) = _tuple_case(F64, True, paths=16)
    torch.manual_seed(5)
    la, lb = torch.nn.Linear(5, 15).to(DEV).double(), torch.nn.Linear(4, 8).to(DEV).double()
    fa = lambda t, z: torch.tanh(la(z) + t).view(*z.shape[:-1], 5, 3)      # noqa: E731
    fb = lambda t, z: torch.tanh(lb(z) * t).view(*z.shape[:-1], 4, 2)      # noqa: E731

    def grads(tuple_state):
        t = torch.tensor([0.0, 0.3, 0.35, 0.9, 7.0, 39.0], dtype=F64, device=DEV, requires_grad=True)
        k = kb.detach().clone().requires_grad_(True)
        A, B = cde.CubicSpline(ca), cde.LinearInterpolation(xb, t=k)
        if tuple_state:
            out = cde.cdeint(cde.TupleControl(A, B), lambda s, z: (fa(s, z[0]), fb(s, z[1])), z0, t, adjoint=False,
                             method="rk4", options={"step_size": 1.0})
        else:
            out = (cde.cdeint(A, fa, z0[0], t, adjoint=False, method="rk4", options={"step_size": 1.0}),
                   cde.cdeint(B, fb, z0[1], t, adjoint=False, method="rk4", options={"step_size": 1.0}))
        return torch.autograd.grad(sum(o.pow(2).sum() for o in out), [t, k])

    for g, w in zip(grads(True), grads(False)):
        assert _global_err(g, w) <= 1e-10


def _record_attempts(monkeypatch):
    records = []
    real = adaptive.Dopri5._attempt

    def attempt(self, t0, dt, y0, f0):
        y1, ks, ratio = real(self, t0, dt, y0, f0)
        records.append((t0, dt, ratio <= 1, ratio))
        return y1, ks, ratio
    monkeypatch.setattr(adaptive.Dopri5, "_attempt", attempt)
    return records


@gpu
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_dopri5_matches_the_oracle_on_the_device_step_sequence(dtype, monkeypatch):
    X, func, z0, _ = _tuple_case(dtype, True, paths=200)
    t = torch.tensor([0.0, 3.5, 17.0, 39.0], dtype=F64)
    rtol, atol = (1e-4, 1e-6) if dtype == F32 else (1e-7, 1e-9)
    records = _record_attempts(monkeypatch)
    _refuse_torch_loop(monkeypatch)
    monkeypatch.setattr(tuple_solver, "torch_field", lambda *a: (_ for _ in ()).throw(AssertionError("torch field")))
    calls = _Calls(monkeypatch)
    with torch.no_grad():
        out = cde.cdeint(X, func, z0, t, rtol=rtol, atol=atol)
    monkeypatch.undo()
    stats = cde.cdeint.last_stats
    assert stats["n_accepted"] + stats["n_rejected"] == len(records) and not stats["device_controlled"]
    assert calls.names.count("tcde_error_ratio_sumsq") == 2 * len(records)          # one per member per attempt
    n_eval = calls.names.count("tcde_spline_eval_grouped")
    assert n_eval == calls.names.count("tcde_field_contract_grouped") == 6 * len(records) + 2
    packed, _ = _tuple_oracle(X, func, dtype, z0)
    with torch.no_grad():
        ys, recs, first = TO.solve_mixed(packed, packed.pack([z.double() for z in z0]), t.tolist(), rtol, atol,
                                         [z.numel() for z in z0], replay=[(r[0], r[1], r[2]) for r in records])
    assert first == pytest.approx(records[0][1], rel=1e-3 if dtype == F32 else 1e-9)
    for (t0, dt, acc, ratio), rec in zip(records, recs):
        if abs(rec.ratio - 1.0) > 0.1:           # the oracle, from its own fp64 state, takes the same decisions
            assert acc == (rec.ratio <= 1.0), (t0, dt, ratio, rec.ratio)
    for o, w in zip(out, packed.unpack(ys)):
        assert _global_err(o.movedim(-2, 0), w) <= (2e-5 if dtype == F32 else 1e-9)


@gpu
def test_adjoint_true_gradients_match_the_oracle_gradient():
    """The continuous adjoint of a fixed-step rk4 solve (steps on every knot of both members, so every step sees a smooth
    field) against fp64 autograd through the oracle's solve on the same grid: the two differ by the rk4 error of the
    backward solve, far below the adjoint bar of test_gpu_generic_routes.py (2e-4)."""
    X, func, z0, _ = _tuple_case(F64, False, paths=24)
    z0 = tuple(z.detach().requires_grad_(True) for z in z0)
    t = torch.tensor([0.0, 12.0, 39.0], dtype=F64)
    out = cde.cdeint(X, func, z0, t, method="rk4", options={"step_size": 0.1})
    gen = torch.Generator().manual_seed(4)
    ws = [torch.randn(o.shape, generator=gen, dtype=F64).to(DEV) for o in out]
    params = list(func.parameters())
    got = torch.autograd.grad(sum((o * w).sum() for o, w in zip(out, ws)), list(z0) + params)
    packed, f64 = _tuple_oracle(X, func, F64, z0)
    z64 = [z.detach().double().requires_grad_(True) for z in z0]
    ys = packed.unpack(odeint_port.odeint(packed, packed.pack(z64), t.to(DEV), method="rk4", options={"step_size": 0.1}))
    want = torch.autograd.grad(sum((y.movedim(0, -2) * w).sum() for y, w in zip(ys, ws)),
                               z64 + list(f64.parameters()))
    for g, w in zip(got, want):
        assert _global_err(g, w) <= 2e-4


@gpu
def test_adjoint_true_fixed_step_honours_adjoint_params():
    X, func, z0, _ = _tuple_case(F32, False, paths=32)
    z0 = tuple(z.detach().requires_grad_(True) for z in z0)
    out = cde.cdeint(X, func, z0, torch.tensor([0.0, 39.0]), method="rk4", options={"step_size": 1.0},
                     adjoint_params=())
    out[1].sum().backward()
    assert all(p.grad is None for p in func.parameters())
    assert z0[0].grad is not None and z0[1].grad.abs().sum() > 0


@gpu
def test_members_with_batch_shapes_2_and_scalar():
    """Decoupled members with batch shapes (2,) and (): each member's output is its own tensor-state solve's."""
    gen = torch.Generator().manual_seed(8)
    xa = torch.rand(2, 10, 2, generator=gen).to(DEV)
    xb = torch.rand(10, 1, generator=gen).to(DEV)
    A, B = cde.CubicSpline(cde.natural_cubic_coeffs(xa)), cde.CubicSpline(cde.natural_cubic_coeffs(xb))
    fa = lambda t, z: z.sigmoid().unsqueeze(-1).repeat_interleave(2, dim=-1)     # noqa: E731
    fb = lambda t, z: z.tanh().unsqueeze(-1)                                     # noqa: E731
    z0 = (torch.rand(2, 3, generator=gen).to(DEV), torch.rand(5, generator=gen).to(DEV))
    X = cde.TupleControl(A, B)
    opts = {"step_size": 0.5}
    with torch.no_grad():
        fixed = cde.cdeint(X, lambda t, z: (fa(t, z[0]), fb(t, z[1])), z0, X.interval, adjoint=False, method="rk4",
                           options=opts)
        alone = (cde.cdeint(A, fa, z0[0], X.interval, adjoint=False, method="rk4", options=opts),
                 cde.cdeint(B, fb, z0[1], X.interval, adjoint=False, method="rk4", options=opts))
        adapt = cde.cdeint(X, lambda t, z: (fa(t, z[0]), fb(t, z[1])), z0, X.interval)
    assert fixed[0].shape == (2, 2, 3) and fixed[1].shape == (2, 5) and adapt[1].shape == (2, 5)
    for f, a, d in zip(fixed, alone, adapt):
        assert _global_err(f, a) <= 1e-6
        assert _global_err(d, a) <= 1e-2              # dopri5 at rtol 1e-4 against rk4 at step 0.5


@gpu
def test_reference_test_tuple_input():
    # test/test_cdeint.py::test_tuple_input, with ``import torchcde_b200 as torchcde`` and ``.cuda()``
    torchcde = cde
    xa = torch.rand(2, 10, 2).cuda()
    xb = torch.rand(10, 1).cuda()

    coeffs_a = torchcde.natural_cubic_coeffs(xa)
    coeffs_b = torchcde.natural_cubic_coeffs(xb)
    spline_a = torchcde.CubicSpline(coeffs_a)
    spline_b = torchcde.CubicSpline(coeffs_b)
    X = torchcde.TupleControl(spline_a, spline_b)

    def func(t, z):
        za, zb = z
        return za.sigmoid().unsqueeze(-1).repeat_interleave(2, dim=-1), zb.tanh().unsqueeze(-1)

    z0 = torch.rand(2, 3).cuda(), torch.rand(5, requires_grad=True, device="cuda")
    out = torchcde.cdeint(X=X, func=func, z0=z0, t=X.interval, adjoint_params=())
    out[0].sum().backward()
    assert (z0[1].grad == 0).all()

