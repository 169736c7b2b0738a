"""GPU: dopri5 (this package's own adaptive driver) and the adjoint backward pass.

An adaptive solver's output is defined only up to its tolerances, so these tests compare with
tight fixed-step fp64 oracle solutions and with autograd through the fixed-step loop."""
import math

import pytest
import torch

import torchcde_b200 as cde
from oracle import cde_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _problem(batch, length, channels, hidden, seed, dtype=torch.float32):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / math.sqrt(length)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64)
    torch.manual_seed(seed)
    func = cde.LinearVectorField(hidden, channels, dtype=dtype)
    return x.to(dtype), z0.to(dtype), func


def test_readme_example_default_call_runs_dopri5_with_adjoint():
    """BASELINE config 1: the README call verbatim (README.md:29-55): default method and adjoint."""
    batch, length, input_channels, hidden_channels = 1, 10, 2, 3
    torch.manual_seed(0)
    t = torch.linspace(0, 1, length)
    x = torch.cat([t.view(1, length, 1), torch.rand(batch, length, input_channels - 1)], dim=2).to(DEV)

    class F(torch.nn.Module):
        def __init__(self):
            super(F, self).__init__()
            self.linear = torch.nn.Linear(hidden_channels, hidden_channels * input_channels)

        def forward(self, t, z):
            return self.linear(z).view(batch, hidden_channels, input_channels)

    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    X = cde.CubicSpline(coeffs)
    func = F().to(DEV)
    z0 = torch.rand(batch, hidden_channels, device=DEV)
    out = cde.cdeint(X=X, func=func, z0=z0, t=X.interval)
    assert out.shape == (batch, 2, hidden_channels) and out.requires_grad
    out[:, -1].sum().backward()
    assert func.linear.weight.grad is not None and bool(torch.isfinite(func.linear.weight.grad).all())
    want = O.cdeint_linear(coeffs.cpu().double(), O.knot_times(length, torch.float64),
                           func.linear.weight.detach().cpu().double(), func.linear.bias.detach().cpu().double(),
                           z0.cpu().double(), torch.tensor([0.0, 9.0], dtype=torch.float64), "rk4", 1 / 32)
    err = float((out.detach().cpu().double() - want).abs().max())
    assert err < 2e-2 * max(1.0, float(want.abs().max())), err      # default rtol=1e-4 accumulated over 9 time units


def _exact_piecewise_linear(x, weight, bias, z0, t_end_index):
    """For a piecewise-LINEAR control dX/dt is constant on every interval, so the linear CDE is an
    affine constant-coefficient ODE there: one matrix exponential per interval gives the exact
    solution (fp64) -- an oracle that involves no time stepping at all."""
    batch, length, channels = x.shape
    hidden = z0.size(-1)
    w = weight.view(hidden, channels, hidden)
    b = bias.view(hidden, channels)
    z = torch.cat([z0, torch.ones(batch, 1, dtype=z0.dtype)], dim=1)
    outs = {0: z0.clone()}
    for i in range(length - 1):
        dx = x[:, i + 1] - x[:, i]                                   # unit knots: slope == increment
        m = torch.zeros(batch, hidden + 1, hidden + 1, dtype=z0.dtype)
        m[:, :hidden, :hidden] = torch.einsum("hck,bc->bhk", w, dx)
        m[:, :hidden, hidden] = torch.einsum("hc,bc->bh", b, dx)
        z = torch.einsum("bij,bj->bi", torch.linalg.matrix_exp(m), z)
        outs[i + 1] = z[:, :hidden].clone()
    return outs[t_end_index]


def test_dopri5_cubic_control_matches_fine_fixed_step_solution():
    x, z0, func = _problem(64, 24, 8, 32, seed=4)
    func = func.to(DEV)
    with torch.no_grad():
        control = O.hermite_backward_difference_coeffs(x)
        X = cde.CubicSpline(control.to(DEV))
        t = torch.tensor([0.0, 7.5, 23.0])
        out = cde.cdeint(X, func, z0.to(DEV), t, adjoint=False, rtol=1e-6, atol=1e-8)
        want = O.cdeint_linear(control.double(), O.knot_times(24, torch.float64),
                               func.linear.weight.detach().cpu().double(), func.linear.bias.detach().cpu().double(),
                               z0.double(), t.double(), "rk4", 1 / 16, "cubic")
    scale = float(want.abs().max())
    assert float((out.cpu().double() - want).abs().max()) < 2e-4 * scale


def test_dopri5_linear_control_matches_exact_matrix_exponential():
    x, z0, func = _problem(48, 12, 8, 32, seed=5)
    func = func.to(DEV)
    with torch.no_grad():
        X = cde.LinearInterpolation(x.to(DEV))
        out = cde.cdeint(X, func, z0.to(DEV), X.interval, adjoint=False, rtol=1e-6, atol=1e-8)
        want = _exact_piecewise_linear(x.double(), func.linear.weight.detach().cpu().double(),
                                       func.linear.bias.detach().cpu().double(), z0.double(), 11)
    scale = float(want.abs().max())
    assert float((out[:, -1].cpu().double() - want).abs().max()) < 5e-4 * scale


def test_dopri5_jump_t_on_linear_control():
    """README.md:194-200: with a piecewise-linear control pass the knots as jump_t; same answer, far fewer steps."""
    from torchcde_b200 import adaptive
    x, z0, func = _problem(16, 12, 8, 32, seed=6)
    func = func.to(DEV)
    counts = []
    with torch.no_grad():
        X = cde.LinearInterpolation(x.to(DEV))
        plain = cde.cdeint(X, func, z0.to(DEV), X.interval, adjoint=False, rtol=1e-6, atol=1e-8)
        counts.append((cde.cdeint.last_stats["n_accepted"], cde.cdeint.last_stats["n_rejected"]))     # device-controlled driver
        jumped = cde.cdeint(X, func, z0.to(DEV), X.interval, adjoint=False, rtol=1e-6, atol=1e-8,
                            options=dict(jump_t=X.grid_points))
        counts.append((cde.cdeint.last_stats["n_accepted"], cde.cdeint.last_stats["n_rejected"]))     # host driver (jump_t)
        assert not cde.cdeint.last_stats["device_controlled"]
    want = _exact_piecewise_linear(x.double(), func.linear.weight.detach().cpu().double(),
                                   func.linear.bias.detach().cpu().double(), z0.double(), 11)
    scale = float(want.abs().max())
    assert float((jumped[:, -1].cpu().double() - want).abs().max()) < 5e-4 * scale
    assert float((plain[:, -1].cpu().double() - want).abs().max()) < 5e-4 * scale
    assert sum(counts[1]) < sum(counts[0])              # fewer attempted steps with jump_t


def test_generic_func_shapes_like_reference_test_cdeint():
    """test_cdeint.py:6-46: sigmoid field, float64 output times with a float32 state, 0-2 batch dims."""
    gen = torch.Generator().manual_seed(11)
    for method, kw in (("rk4", {"options": {"step_size": 1.0}}), ("dopri5", {})):
        for batch_dims in ((), (2,), (2, 1)):
            values = torch.rand(*batch_dims, 17, 2, generator=gen).to(DEV)
            with torch.no_grad():
                X = cde.CubicSpline(cde.natural_cubic_coeffs(values))
            variable = torch.rand(*[1 for _ in batch_dims], 1, 2, generator=gen).to(DEV)

            def f(t, z):
                return z.sigmoid().unsqueeze(-1) + variable

            z0 = torch.rand(*batch_dims, 4, generator=gen).to(DEV)
            start, end = X.interval
            out_times = torch.rand(5, dtype=torch.float64, generator=gen).sort().values.to(DEV) * (end - start) + start
            with torch.no_grad():
                out = cde.cdeint(X, f, z0, out_times, method=method, rtol=1e-1, atol=1e-1, adjoint=False, **kw)
            assert out.shape == (*batch_dims, 5, 4)


def test_prod_interface_and_gradient():
    """test_cdeint.py:86-99: func.prod(t, z, dXdt) with the analytic solution z0 exp(-(X(T)-X(0)))."""
    x = torch.rand(2, 5, 1, device=DEV, dtype=torch.float64)
    with torch.no_grad():
        X = cde.CubicSpline(cde.natural_cubic_coeffs(x))

    class F:
        def prod(self, t, z, dXdt):
            assert t.shape == () and z.shape == (2, 3) and dXdt.shape == (2, 1)
            return -z * dXdt

    z0 = torch.rand(2, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    out = cde.cdeint(X=X, func=F(), z0=z0, t=X.interval, adjoint_params=(), rtol=1e-8, atol=1e-10)
    exact = z0.detach() * torch.exp(-(x[:, -1] - x[:, 0]))
    assert torch.allclose(out[:, -1].detach(), exact, rtol=1e-5, atol=1e-7)
    out.sum().backward()
    assert torch.allclose(z0.grad, 1 + torch.exp(-(x[:, -1] - x[:, 0])).expand_as(z0), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("method,kw", [("rk4", {"options": {"step_size": 0.03125}}), ("dopri5", {})])
def test_adjoint_gradients_match_backprop_through_the_solver(method, kw):
    """adjoint=True (continuous adjoint, fused forward) vs adjoint=False (autograd through the stage
    loop): same gradients up to discretisation error (test_tricks.py checks existence only)."""
    x, z0, func = _problem(5, 9, 3, 4, seed=8, dtype=torch.float64)
    func = func.to(DEV)
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV))
    X = cde.CubicSpline(coeffs)
    t = torch.tensor([0.0, 3.3, 8.0], dtype=torch.float64)
    grads = []
    for adjoint in (True, False):
        zz = z0.to(DEV).clone().requires_grad_(True)
        func.zero_grad()
        out = cde.cdeint(X, func, zz, t, adjoint=adjoint, method=method, rtol=1e-9, atol=1e-11, **kw)
        (out[:, 1].pow(2).sum() + out[:, 2].sum()).backward()
        grads.append((zz.grad.clone(), func.linear.weight.grad.clone(), func.linear.bias.grad.clone()))
    tol = 2e-3 if method == "rk4" else 1e-5
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=tol, atol=tol * float(b.abs().max()))


def _vjp_reference(control, kind, weight, bias, z, a, index, frac, scale):
    """fp64 autograd statement of what tcde_vector_field_linear_vjp returns."""
    w = weight.double().clone().requires_grad_(True)
    b = bias.double().clone().requires_grad_(True)
    zz = z.double().clone().requires_grad_(True)
    c = control.double()
    channels = b.numel() // zz.size(-1)
    if kind == "cubic":
        row = c[:, index]
        dx = row[:, channels:2 * channels] + (row[:, 2 * channels:3 * channels] + row[:, 3 * channels:] * frac) * frac
    else:
        dx = c[:, index]
    f = (torch.nn.functional.linear(zz, w, b).view(zz.size(0), zz.size(1), channels) @ dx.unsqueeze(-1)).squeeze(-1)
    gz, gw, gb = torch.autograd.grad(f, (zz, w, b), a.double() * scale)
    return f.detach(), gz, gw, gb


@pytest.mark.parametrize("n_paths", [1, 63, 64, 65, 1000, 20011])
@pytest.mark.parametrize("kind", ["cubic", "linear"])
def test_fused_adjoint_stage_against_autograd(n_paths, kind):
    """tcde_vector_field_linear_vjp (hidden 32, channels 8, fp32): field value, a^T df/dz and the parameter
    gradients (accumulated onto what the buffers already hold) vs fp64 autograd of the same expression."""
    from torchcde_b200 import _lib
    gen = torch.Generator().manual_seed(n_paths)
    hidden, channels, n_rows = 32, 8, 5
    width = 4 * channels if kind == "cubic" else channels
    control = torch.randn(n_paths, n_rows, width, generator=gen).to(DEV)
    weight = (torch.randn(hidden * channels, hidden, generator=gen) / math.sqrt(hidden)).to(DEV)
    bias = torch.randn(hidden * channels, generator=gen).to(DEV)
    z = torch.randn(n_paths, hidden, generator=gen).to(DEV)
    a = torch.randn(n_paths, hidden, generator=gen).to(DEV)
    index, frac, scale = 3, 0.37, -0.75
    f = torch.empty_like(z)
    vz = torch.empty_like(z)
    gw0 = torch.randn(hidden * channels, hidden, generator=gen).to(DEV)
    gb0 = torch.randn(hidden * channels, generator=gen).to(DEV)
    gw, gb = gw0.clone(), gb0.clone()
    nbytes = _lib.load().tcde_vector_field_linear_vjp_scratch_bytes(n_paths, channels, hidden)
    assert nbytes > 0
    scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=DEV)
    code = _lib.dtype_code(z.dtype)
    _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(control), _lib.CONTROL_CUBIC if kind == "cubic" else
              _lib.CONTROL_LINEAR, n_rows, _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(z), _lib.ptr(a), _lib.ptr(f),
              _lib.ptr(vz), _lib.ptr(gw), _lib.ptr(gb), _lib.ptr(scratch), n_paths, channels, hidden, index, frac, 1.0,
              scale, scale, code, _lib.stream_of(z))
    wf, wz, ww, wb = _vjp_reference(control, kind, weight, bias, z, a, index, frac, scale)

    def close(got, want, tol=2e-5):
        return float((got.double() - want).abs().max()) <= tol * max(1.0, float(want.abs().max()))

    assert close(f, wf) and close(vz, wz)
    assert close(gw - gw0, ww, 5e-5) and close(gb - gb0, wb, 5e-5)
    # the forward-only entry point returns the same field
    f2 = torch.empty_like(z)
    _lib.call("tcde_vector_field_linear", _lib.ptr(control), _lib.CONTROL_CUBIC if kind == "cubic" else
              _lib.CONTROL_LINEAR, n_rows, _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(z), _lib.ptr(f2), n_paths, channels,
              hidden, index, frac, code, _lib.stream_of(z))
    assert close(f, f2.double(), 1e-6)
    with pytest.raises(NotImplementedError):
        _lib.call("tcde_vector_field_linear_vjp", _lib.ptr(control), _lib.CONTROL_LINEAR, n_rows, _lib.ptr(weight),
                  _lib.ptr(bias), _lib.ptr(z), _lib.ptr(a), _lib.ptr(f), _lib.ptr(vz), None, None, _lib.ptr(scratch),
                  n_paths, 4, 16, index, frac, 1.0, scale, scale, code, _lib.stream_of(z))


@pytest.mark.parametrize("method,kw", [("rk4", {"options": {"step_size": 0.25}}), ("midpoint", {"options": {"step_size": 0.25}}),
                                       ("dopri5", {})])
def test_fused_adjoint_matches_the_autograd_adjoint(method, kw, monkeypatch):
    """cdeint(adjoint=True) at the flagship field shape (hidden 32, channels 8, fp32): the backward solve that
    uses the fused stage kernel gives the gradients of the one that uses autograd (same algorithm, same steps)."""
    from torchcde_b200 import solver
    x, z0, func = _problem(37, 12, 8, 32, seed=5)
    func = func.to(DEV)
    with torch.no_grad():
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV)))
    t = torch.tensor([0.0, 4.5, 11.0])
    grads, used = [], []
    real = solver._kernel_vjp
    for fused in (True, False):
        def probe(*args, _fused=fused, **kwargs):
            stage = real(*args, **kwargs) if _fused else None
            used.append(stage is not None)
            return stage
        monkeypatch.setattr(solver, "_kernel_vjp", probe)
        zz = z0.to(DEV).clone().requires_grad_(True)
        func.zero_grad()
        out = cde.cdeint(X, func, zz, t, adjoint=True, method=method, rtol=1e-5, atol=1e-7, **kw)
        (out[:, 1].pow(2).sum() + out[:, 2].sum()).backward()
        grads.append((zz.grad.clone(), func.linear.weight.grad.clone(), func.linear.bias.grad.clone()))
    assert used == [True, False]
    # fixed steps: the two backward solves do the same arithmetic up to summation order.  dopri5: its error norm is
    # dominated by the parameter-gradient components (|dL/dW| ~ 100 vs |a| ~ 1), so rtol=1e-5 on the whole state
    # leaves ~1e-2 relative freedom on the small components and the two runs may pick different steps
    rtol, scale = (5e-2, 5e-3) if method == "dopri5" else (2e-3, 2e-4)
    for got, want in zip(*grads):
        assert torch.allclose(got, want, rtol=rtol, atol=scale * float(want.abs().max()))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(1,), (257, 3), (100003,), (8, 33, 32)])
def test_stepper_kernels_against_torch(dtype, shape):
    """tcde_linear_combination / tcde_error_ratio_sumsq (the elementwise part of a dopri5 attempt) vs torch."""
    from torchcde_b200 import adaptive
    gen = torch.Generator().manual_seed(len(shape))
    ks = [torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype).to(DEV) for _ in range(7)]
    y0 = torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype).to(DEV)
    weights = (0.3, 0.0, -1.25, 2.0, 0.5, -0.75, 0.125)
    dt = 0.37
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for base in (y0, None):
        with torch.no_grad():
            got = adaptive._combine(base, ks, weights, dt)
        want = sum(k.double() * (w * dt) for k, w in zip(ks, weights)) + (0 if base is None else base.double())
        assert got.dtype == dtype and torch.allclose(got.double(), want, rtol=tol, atol=tol)
    y1 = y0 + 0.1 * ks[0]
    with torch.no_grad():
        got = adaptive._error_ratio(y0, y1, ks, weights, dt, 1e-6, 1e-4, adaptive._rms)
    err = sum(k.double() * (w * dt) for k, w in zip(ks, weights))
    want = float((err / (1e-6 + 1e-4 * torch.max(y0.double().abs(), y1.double().abs()))).pow(2).mean().sqrt())
    assert abs(got - want) <= 1e-4 * want
    # under autograd the torch operators are kept (adjoint=False differentiates through the solver)
    yg = y0.clone().requires_grad_(True)
    out = adaptive._combine(yg, ks, weights, dt)
    assert out.requires_grad


@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
def test_trajectory_backward_matches_the_per_stage_backward(method, monkeypatch):
    """Fixed-step adjoint at the flagship field shape: the three-launch backward (two tensor-core solves that keep
    their stage inputs + one contraction into dL/dW, dL/db) vs the per-stage fused backward vs autograd."""
    from torchcde_b200 import solver
    x, z0, func = _problem(300, 14, 8, 32, seed=11)
    func = func.to(DEV)
    with torch.no_grad():
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV)))
    t = torch.tensor([0.0, 4.5, 13.0])
    kw = {"options": {"step_size": 0.5}}
    real = solver._kernel_vjp
    grads, used = {}, {}
    for mode in ("trajectory", "per_stage", "autograd"):
        def probe(*args, _mode=mode, **kwargs):
            stage = real(*args, **kwargs)
            if _mode == "autograd":
                return None
            if _mode == "per_stage":
                stage.segment = lambda *a, **k: None
            else:
                inner = stage.segment

                def counted(*a, **k):
                    res = inner(*a, **k)
                    used[_mode] = used.get(_mode, 0) + (res is not None)
                    return res
                stage.segment = counted
            return stage
        monkeypatch.setattr(solver, "_kernel_vjp", probe)
        zz = z0.to(DEV).clone().requires_grad_(True)
        func.zero_grad()
        out = cde.cdeint(X, func, zz, t, adjoint=True, method=method, **kw)
        (out[:, 1].pow(2).sum() + out[:, 2].sum()).backward()
        grads[mode] = (zz.grad.clone(), func.linear.weight.grad.clone(), func.linear.bias.grad.clone())
    assert used.get("trajectory") == 2                        # both segments took the three-launch route
    for mode in ("per_stage", "autograd"):
        for got, want in zip(grads["trajectory"], grads[mode]):
            assert torch.allclose(got, want, rtol=2e-3, atol=2e-4 * float(want.abs().max())), mode


@pytest.mark.parametrize("n_paths,n_stages", [(1, 1), (31, 3), (32, 2), (33, 5), (1000, 8), (4099, 40)])
@pytest.mark.parametrize("kind", ["cubic", "linear"])
def test_parameter_gradient_kernels_against_einsum(n_paths, n_stages, kind):
    """tcde_linear_field_param_grads on the tensor cores (variant 0: 2xBF16 operand split; variant 2: 3xTF32) and on the
    CUDA cores (variant 1) vs an fp64 einsum over (stage, path): ragged path blocks, zero-weight stages, accumulation onto
    existing gradients.  Bars: fp32-class (3e-5 of the largest entry) for the TF32 / CUDA-core kernels, 2e-4 for the BF16
    split (16 significant bits per operand: ample for a gradient)."""
    from torchcde_b200 import _lib
    gen = torch.Generator().manual_seed(n_paths + n_stages)
    hidden, channels, n_rows = 32, 8, 6
    width = 4 * channels if kind == "cubic" else channels
    control = torch.randn(n_paths, n_rows, width, generator=gen).to(DEV)
    z = torch.randn(n_stages, n_paths, hidden, generator=gen).to(DEV)
    a = torch.randn(n_stages, n_paths, hidden, generator=gen).to(DEV)
    index = torch.randint(0, n_rows, (n_stages,), generator=gen, dtype=torch.int32)
    frac = torch.rand(n_stages, generator=gen)
    weight = torch.randn(n_stages, generator=gen)
    if n_stages > 2:
        weight[1] = 0.0
    c64 = control.double().cpu()
    want_w = torch.zeros(hidden, channels, hidden, dtype=torch.float64)
    want_b = torch.zeros(hidden, channels, dtype=torch.float64)
    for e in range(n_stages):
        row = c64[:, int(index[e])]
        f = float(frac[e])
        if kind == "cubic":
            dx = row[:, channels:2 * channels] + (row[:, 2 * channels:3 * channels] + row[:, 3 * channels:] * f) * f
        else:
            dx = row
        ae, ze = a[e].double().cpu(), z[e].double().cpu()
        want_w += float(weight[e]) * torch.einsum("ph,pc,pk->hck", ae, dx, ze)
        want_b += float(weight[e]) * torch.einsum("ph,pc->hc", ae, dx)
    want_w, want_b = want_w.reshape(hidden * channels, hidden), want_b.reshape(-1)
    nbytes = _lib.load().tcde_linear_field_param_grads_scratch_bytes(n_paths, n_stages, channels, hidden)
    assert nbytes > 0
    scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=DEV)
    code = _lib.dtype_code(z.dtype)
    scale = -0.5
    index_d, frac_d, weight_d = index.to(DEV), frac.to(DEV), weight.to(DEV)     # kept alive across the launches
    try:
        for variant in (0, 1, 2):
            _lib.call("tcde_set_solve_variant", variant)
            gw0 = torch.randn(hidden * channels, hidden, generator=gen).to(DEV)
            gb0 = torch.randn(hidden * channels, generator=gen).to(DEV)
            gw, gb = gw0.clone(), gb0.clone()
            _lib.call("tcde_linear_field_param_grads", _lib.ptr(control), _lib.CONTROL_CUBIC if kind == "cubic" else
                      _lib.CONTROL_LINEAR, n_rows, _lib.ptr(z), _lib.ptr(a), _lib.ptr(index_d),
                      _lib.ptr(frac_d), _lib.ptr(weight_d), n_stages, _lib.ptr(gw), _lib.ptr(gb),
                      _lib.ptr(scratch), n_paths, channels, hidden, scale, code, _lib.stream_of(z))
            torch.cuda.synchronize()
            for got, want in (((gw - gw0).double().cpu(), scale * want_w), ((gb - gb0).double().cpu(), scale * want_b)):
                bar = 2e-4 if variant == 0 else 3e-5
                assert float((got - want).abs().max()) <= bar * max(1.0, float(want.abs().max())), variant
    finally:
        _lib.call("tcde_set_solve_variant", 0)


@pytest.mark.parametrize("kind", ["cubic", "linear"])
@pytest.mark.parametrize("slots", [None, 16])
def test_device_controlled_dopri5_adjoint_matches_the_host_driven_adjoint(kind, slots, monkeypatch):
    """cdeint(adjoint=True) with the default dopri5: the backward pass with the controller on the device
    (tcde_dopri5_linear_paired_attempts: z and the adjoint state as one virtual batch, parameter gradients by quadrature over
    the accepted steps' stage inputs) against this package's host-driven adjoint (one fused field + vjp launch per evaluation)
    at a tolerance tight enough to compare them; two segments between three output times; with 16 trajectory slots the
    device has to pause and hand the slots back several times."""
    from torchcde_b200 import adaptive, solver
    torch.manual_seed(11)
    B, L, C, H = 512, 14, 8, 32
    x = torch.randn(B, L, C, device=DEV).cumsum(1) / 3
    X = (cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x)) if kind == "cubic"
         else cde.LinearInterpolation(x))
    func = cde.LinearVectorField(H, C).to(DEV)
    with torch.no_grad():
        func.linear.weight.mul_(0.5)
    z0 = torch.randn(B, H, device=DEV)
    t = torch.tensor([0.0, 5.5, L - 1.0], device=DEV)
    kw = {"rtol": 1e-6, "atol": 1e-8}

    def run():
        zz = z0.clone().requires_grad_(True)
        func.zero_grad()
        out = cde.cdeint(X, func, zz, t, adjoint=True, **kw)
        (out[:, -1].sum() + (out[:, 1] ** 2).sum()).backward()
        return out.detach(), zz.grad.clone(), func.linear.weight.grad.clone(), func.linear.bias.grad.clone()

    if slots is not None:
        real = solver._kernel_vjp

        def with_few_slots(*a, **k):
            st = real(*a, **k)
            if st is not None:
                st.slots_hint = slots
            return st

        monkeypatch.setattr(solver, "_kernel_vjp", with_few_slots)
    cde.cdeint.last_adjoint_stats = None
    out_d, gz_d, gw_d, gb_d = run()
    stats = cde.cdeint.last_adjoint_stats
    assert stats is not None and stats["device_controlled"] and stats["n_accepted"] > 10
    if slots is not None:
        assert stats["flushes"] >= 1 and stats["slots"] == 16
    monkeypatch.setattr(adaptive, "_device_adaptive_backward", lambda *a, **k: None)
    cde.cdeint.last_adjoint_stats = None
    out_h, gz_h, gw_h, gb_h = run()
    assert cde.cdeint.last_adjoint_stats is None
    assert torch.equal(out_d, out_h)
    for got, want in ((gz_d, gz_h), (gw_d, gw_h), (gb_d, gb_h)):
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 2e-3 * scale, (float((got - want).abs().max()), scale)
