"""GPU parity, hot path (ii): spline evaluation and the fused fixed-step solve through the C ABI.

Tolerances.  Interval indices: bit exact.  Spline evaluation: bit exact.  The solve: fp64 to
1e-10 relative; fp32 to 1e-5 of the solution scale (10x inside the north_star's rtol 1e-4; the
observed error is ~5e-7 of scale, VERDICT r01) -- the reference's own addmm/bmm reduction order
is not reproducible, so two fp32 runs of the *reference* on different hardware differ by ~1e-6
(SURVEY 8d: fp32 vs fp64 of one algorithm ~1e-6 median)."""
import math

import pytest
import torch

import torchcde_b200 as cde
from conftest import Golden, same
from oracle import cde_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _assert_close(got, want, dtype):
    want = want.to(torch.float64)
    got = got.detach().cpu().to(torch.float64)
    scale = max(1.0, float(want.abs().max()))
    rtol, atol = (1e-5, 1e-5 * scale) if dtype == torch.float32 else (1e-10, 1e-10 * scale)
    err = (got - want).abs()
    assert bool((err <= atol + rtol * want.abs()).all()), "max err {:.3e} at scale {:.3e}".format(float(err.max()), scale)


def test_evaluation_fixtures_bit_exact():
    g = Golden("evaluation")
    for i in range(g.count):
        k = "e{:02d}".format(i)
        x = g.t(k + "_in_x").to(DEV)
        t = g.t(k + "_in_t").to(DEV) if g.has(k + "_in_t") else None
        q = g.t(k + "_in_query").to(DEV)
        spline = cde.CubicSpline(g.t(k + "_ref_coeffs").to(DEV), t)
        linear = cde.LinearInterpolation(x, t)
        frac, index = spline._interpret_t(q)
        assert torch.equal(index.cpu(), g.t(k + "_ref_index")), k                 # bit exact indices
        assert torch.equal(frac.cpu(), g.t(k + "_ref_frac")), k
        assert same(spline.evaluate(q).cpu(), g.t(k + "_ref_cubic_eval")), k
        assert same(spline.derivative(q).cpu(), g.t(k + "_ref_cubic_deriv")), k
        assert same(linear.evaluate(q).cpu(), g.t(k + "_ref_linear_eval")), k
        assert same(linear.derivative(q).cpu(), g.t(k + "_ref_linear_deriv")), k
        # shapes for scalar and 2-D query times (README.md:137-138)
        assert spline.derivative(q[0]).shape == (*x.shape[:-2], x.size(-1))
        assert spline.evaluate(q[:6].view(2, 3)).shape == (*x.shape[:-2], 2, 3, x.size(-1))


def _solve_fixture(g, k, dev_dtype=None):
    control = g.t(k + "_in_control")
    kind = g.s(k + "_kind")
    knots = g.t(k + "_in_knots") if g.has(k + "_in_knots") else None
    w, b, z0, t = g.t(k + "_in_weight"), g.t(k + "_in_bias"), g.t(k + "_in_z0"), g.t(k + "_in_t")
    hidden, channels = z0.size(-1), w.size(0) // z0.size(-1)
    func = cde.LinearVectorField(hidden, channels, dtype=control.dtype)
    with torch.no_grad():
        func.linear.weight.copy_(w)
        func.linear.bias.copy_(b)
    func = func.to(DEV)
    kd = None if knots is None else knots.to(DEV)
    X = cde.CubicSpline(control.to(DEV), kd) if kind == "cubic" else cde.LinearInterpolation(control.to(DEV), kd)
    step = g.f(k + "_step")
    options = {} if step < 0 else {"step_size": step}
    return X, func, z0.to(DEV), t.to(DEV), g.s(k + "_method"), options


def test_solve_fixtures_fused_kernel():
    g = Golden("solves")
    for i in range(g.count):
        k = "s{:02d}".format(i)
        X, func, z0, t, method, options = _solve_fixture(g, k)
        with torch.no_grad():
            out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=options)
            field = cde.solver._lib  # noqa: F841  (the call above went through the C ABI)
        want = g.t(k + "_ref_out")
        assert out.shape == want.shape, k
        _assert_close(out, want, want.dtype)


def test_solve_fixtures_generic_stage_loop_and_readme_module():
    """The same fixtures through (a) a README-style user module that must be *recognised* and
    fused, and (b) a non-linear wrapper that must take the generic on-GPU stage loop."""
    g = Golden("solves")
    for i in (0, 2, 5, 9):
        k = "s{:02d}".format(i)
        X, func, z0, t, method, options = _solve_fixture(g, k)
        hidden, channels = func.hidden_channels, func.input_channels

        class Readme(torch.nn.Module):
            def __init__(self, lin):
                super().__init__()
                self.linear = lin

            def forward(self, t, z):
                return self.linear(z).view(*z.shape[:-1], hidden, channels)

        class Opaque:                              # not an nn.Module: cannot be recognised
            def __init__(self, f):
                self.f = f

            def __call__(self, t, z):
                return self.f(t, z)

        want = g.t(k + "_ref_out")
        with torch.no_grad():
            a = cde.cdeint(X, Readme(func.linear), z0, t, adjoint=False, method=method, options=options)
            b = cde.cdeint(X, Opaque(func), z0, t, adjoint=False, method=method, options=options)
        _assert_close(a, want, want.dtype)
        _assert_close(b, want, want.dtype)


def test_vector_field_kernel_against_reference_field():
    g = Golden("solves")
    from torchcde_b200 import _lib
    for i in range(g.count):
        k = "s{:02d}".format(i)
        X, func, z0, t, method, options = _solve_fixture(g, k)
        kind = g.s(k + "_kind")
        probe = g.t(k + "_in_probe").to(DEV)
        frac, index = X._interpret_t(probe)
        control = X._rows() if kind == "cubic" else X._derivs
        flat = control.reshape(-1, control.size(-2), control.size(-1)).contiguous()
        zf = z0.reshape(-1, z0.size(-1)).contiguous()
        out = torch.empty_like(zf)
        _lib.call("tcde_vector_field_linear", _lib.ptr(flat), 0 if kind == "cubic" else 1, flat.size(1),
                  _lib.ptr(func.linear.weight.detach().contiguous()), _lib.ptr(func.linear.bias.detach().contiguous()),
                  _lib.ptr(zf), _lib.ptr(out), zf.size(0), func.input_channels, func.hidden_channels, int(index),
                  float(frac), _lib.dtype_code(zf.dtype), _lib.stream_of(zf))
        _assert_close(out.view_as(z0), g.t(k + "_ref_field"), zf.dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("batch,length,channels,hidden", [(200, 64, 8, 32), (37, 20, 3, 5), (1, 10, 2, 3),
                                                          (64, 30, 4, 64), (9, 12, 12, 16), (130, 40, 1, 7),
                                                          (77, 25, 8, 16), (50, 18, 16, 24)])
def test_fused_solve_against_fp64_oracle(dtype, batch, length, channels, hidden):
    gen = torch.Generator().manual_seed(batch * 7 + hidden)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / math.sqrt(length)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64)
    torch.manual_seed(hidden)
    lin = torch.nn.Linear(hidden, hidden * channels).double()
    co64 = O.hermite_backward_difference_coeffs(x)
    knots = O.knot_times(length, torch.float64)
    func = cde.LinearVectorField(hidden, channels, dtype=dtype)
    with torch.no_grad():
        func.linear.weight.copy_(lin.weight)
        func.linear.bias.copy_(lin.bias)
    func = func.to(DEV)
    X = cde.CubicSpline(co64.to(dtype).to(DEV))
    t_out = torch.tensor([0.0, 0.4 * (length - 1), length - 1.0], dtype=dtype)
    for method, step in (("rk4", 1.0), ("midpoint", 0.5), ("euler", 0.25)):
        with torch.no_grad():
            out = cde.cdeint(X, func, z0.to(dtype).to(DEV), t_out.to(DEV), adjoint=False, method=method,
                             options={"step_size": step})
            # oracle on the SAME rounded inputs, in fp64
            want = O.cdeint_linear(co64.to(dtype).double(), knots, func.linear.weight.detach().cpu().double(),
                                   func.linear.bias.detach().cpu().double(), z0.to(dtype).double(), t_out.double(),
                                   method, step)
        _assert_close(out, want, dtype)


def test_config1_readme_example():
    """BASELINE config 1: the README example shapes (batch 1, length 10, 2 channels, 3 hidden)."""
    torch.manual_seed(0)
    batch, length, input_channels, hidden_channels = 1, 10, 2, 3
    t = torch.linspace(0, 1, length)
    x = torch.cat([t.view(1, length, 1), torch.rand(batch, length, input_channels - 1)], dim=2)
    func = cde.LinearVectorField(hidden_channels, input_channels)
    z0 = torch.rand(batch, hidden_channels)
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV))
        X = cde.CubicSpline(coeffs)
        out = cde.cdeint(X=X, func=func.to(DEV), z0=z0.to(DEV), t=X.interval, adjoint=False, method="rk4",
                         options=dict(step_size=0.5))
        func = func.cpu()
        want = O.cdeint_linear(O.hermite_backward_difference_coeffs(x), O.knot_times(length, torch.float32),
                               func.linear.weight, func.linear.bias, z0, torch.tensor([0.0, 9.0]), "rk4", 0.5)
    assert out.shape == (1, 2, 3)
    _assert_close(out, want, torch.float32)


def test_analytic_solution_of_reference_fixture():
    """test_cdeint.py:54-55 as a linear field: W = 0, bias = -1 on ... no: f(z) = -z expanded over
    C=2 channels is linear with weight rows -e_h; z(T) = z0 exp(-sum_c (X_c(T) - X_c(0)))."""
    hidden, channels, length = 3, 2, 9
    tau = torch.linspace(0, 1, length, dtype=torch.float64).view(1, length, 1)
    x = torch.sin(2 * math.pi * (tau * torch.tensor([0.7, 1.3], dtype=torch.float64) + 0.1)).expand(4, length, channels)
    func = cde.LinearVectorField(hidden, channels, dtype=torch.float64)
    with torch.no_grad():
        func.linear.bias.zero_()
        func.linear.weight.zero_()
        for h in range(hidden):
            for c in range(channels):
                func.linear.weight[h * channels + c, h] = -1.0
    z0 = torch.randn(4, hidden, dtype=torch.float64)
    exact = z0 * torch.exp(-(x[:, -1] - x[:, 0]).sum(-1, keepdim=True))
    with torch.no_grad():
        X = cde.CubicSpline(cde.natural_cubic_coeffs(x.contiguous().to(DEV)))
        errs = []
        for h in (0.25, 0.125, 0.0625):
            out = cde.cdeint(X, func.to(DEV), z0.to(DEV), X.interval, adjoint=False, method="rk4",
                             options={"step_size": h})
            errs.append(float((out[:, -1].cpu() - exact).abs().max()))
    assert errs[-1] < 1e-5 and math.log2(errs[0] / errs[1]) > 3.3 and math.log2(errs[1] / errs[2]) > 3.3, errs


def test_full_size_config3_properties():
    """BASELINE config 3 (batch 65536, length 256, 8 channels, 32 hidden, fp32, rk4 step 1):
    a slice of the full launch must equal the oracle and be independent of the rest of the batch."""
    gen = torch.Generator(device=DEV).manual_seed(0)
    B, L, C, H = 65536, 256, 8, 32
    x = torch.randn(B, L, C, generator=gen, device=DEV).cumsum(1) / math.sqrt(L)
    z0 = torch.randn(B, H, generator=gen, device=DEV)
    torch.manual_seed(1)
    func = cde.LinearVectorField(H, C).to(DEV)
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
        X = cde.CubicSpline(coeffs)
        out = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
        assert out.shape == (B, 2, H) and bool(torch.isfinite(out).all())
        assert torch.equal(out[:, 0], z0)
        again = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
        assert torch.equal(out, again)                                         # deterministic
        pick = torch.arange(0, B, 2731, device=DEV)[:24]
        sub = cde.cdeint(cde.CubicSpline(coeffs[pick].contiguous()), func, z0[pick].contiguous(), X.interval,
                         adjoint=False, method="rk4", options={"step_size": 1.0})
        assert torch.equal(sub, out[pick])                                     # batch independence, bitwise
        want = O.cdeint_linear(coeffs[pick].cpu().double(), O.knot_times(L, torch.float64),
                               func.linear.weight.detach().cpu().double(), func.linear.bias.detach().cpu().double(),
                               z0[pick].cpu().double(), torch.tensor([0.0, L - 1.0], dtype=torch.float64), "rk4", 1.0)
    _assert_close(out[pick], want, torch.float32)


def test_gradients_flow_through_the_generic_loop():
    """Training still works: when anything requires grad the differentiable stage loop is used."""
    torch.manual_seed(3)
    x = torch.randn(6, 8, 2, device=DEV).cumsum(1) / 3
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    X = cde.CubicSpline(coeffs)
    func = cde.LinearVectorField(4, 2).to(DEV)
    z0 = torch.randn(6, 4, device=DEV, requires_grad=True)
    out = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
    out[:, -1].sum().backward()
    assert z0.grad is not None and func.linear.weight.grad is not None
    with torch.no_grad():
        fused = cde.cdeint(X, func, z0.detach(), X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
    _assert_close(out.detach(), fused.cpu(), torch.float32)


# ------------------------------------------------------------------ tensor-core variant
def _set_variant(v):
    from torchcde_b200 import _lib
    _lib.call("tcde_set_solve_variant", v)


@pytest.mark.parametrize("variant", [2, 3, 4, 4 + 16 * 32, 4 + 16 * 2])
@pytest.mark.parametrize("batch", [1, 100, 128, 129, 256, 300, 1000])
def test_tensor_core_variant_matches_cuda_core_and_oracle(batch, variant):
    """The tensor-core kernel solve_tc.cu -- 2 / 3: 3xTF32, 4: 2xFP16 with per-path power-of-two scaling; the + 16 * k
    variants carry flag bits the library accepts and ignores -- against solve_simt.cu and the fp64 oracle, including
    partial warps and CTAs (batch not a multiple of 32 / 128)."""
    length, channels, hidden = 40, 8, 32
    gen = torch.Generator().manual_seed(batch)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / math.sqrt(length)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64).float()
    torch.manual_seed(5)
    func = cde.LinearVectorField(hidden, channels).to(DEV)
    co = O.hermite_backward_difference_coeffs(x).float()
    X = cde.CubicSpline(co.to(DEV))
    Xl = cde.LinearInterpolation(x.float().to(DEV))
    t_out = torch.tensor([0.0, 11.3, 25.0, length - 1.0])
    try:
        for method, step in (("rk4", 1.0), ("midpoint", 0.5), ("euler", 0.5)):
            for control, kind in ((X, "cubic"), (Xl, "linear")):
                with torch.no_grad():
                    _set_variant(1)
                    simt = cde.cdeint(control, func, z0.to(DEV), t_out, adjoint=False, method=method,
                                      options={"step_size": step})
                    _set_variant(variant)
                    tc = cde.cdeint(control, func, z0.to(DEV), t_out, adjoint=False, method=method,
                                    options={"step_size": step})
                    data = co.double() if kind == "cubic" else x.float().double()
                    want = O.cdeint_linear(data, O.knot_times(length, torch.float64),
                                           func.linear.weight.detach().cpu().double(),
                                           func.linear.bias.detach().cpu().double(), z0.double(), t_out.double(),
                                           method, step, kind)
                _assert_close(tc, want, torch.float32)
                _assert_close(simt, want, torch.float32)
                assert torch.equal(tc[:, 0], z0.to(DEV))
    finally:
        _set_variant(0)


@pytest.mark.parametrize("variant", [2, 3, 4, 4 + 16 * 16, 4 + 16 * 2])
def test_tensor_core_variant_full_size(variant):
    gen = torch.Generator(device=DEV).manual_seed(0)
    B, L, C, H = 65536, 256, 8, 32
    x = torch.randn(B, L, C, generator=gen, device=DEV).cumsum(1) / math.sqrt(L)
    z0 = torch.randn(B, H, generator=gen, device=DEV)
    torch.manual_seed(1)
    func = cde.LinearVectorField(H, C).to(DEV)
    try:
        with torch.no_grad():
            coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
            X = cde.CubicSpline(coeffs)
            t = torch.tensor([0.0, L - 1.0])
            _set_variant(variant)
            out = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options={"step_size": 1.0})
            again = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options={"step_size": 1.0})
            assert torch.equal(out, again) and bool(torch.isfinite(out).all())
            pick = torch.arange(0, B, 2731, device=DEV)[:24]
            want = O.cdeint_linear(coeffs[pick].cpu().double(), O.knot_times(L, torch.float64),
                                   func.linear.weight.detach().cpu().double(),
                                   func.linear.bias.detach().cpu().double(), z0[pick].cpu().double(),
                                   torch.tensor([0.0, L - 1.0], dtype=torch.float64), "rk4", 1.0)
        _assert_close(out[pick], want, torch.float32)
    finally:
        _set_variant(0)


@pytest.mark.parametrize("variant", [1, 2, 3, 4, 4 + 16 * 32])
def test_decreasing_output_times(variant):
    """A decreasing t is integrated as -t with the field negated (torchdiffeq's time reversal)."""
    length, channels, hidden, batch = 20, 8, 32, 70
    gen = torch.Generator().manual_seed(77)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / math.sqrt(length)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64).float()
    torch.manual_seed(9)
    func = cde.LinearVectorField(hidden, channels).to(DEV)
    co = O.hermite_backward_difference_coeffs(x).float()
    X = cde.CubicSpline(co.to(DEV))
    t_out = torch.tensor([length - 1.0, 12.5, 3.0, 0.0])
    try:
        _set_variant(variant)
        with torch.no_grad():
            out = cde.cdeint(X, func, z0.to(DEV), t_out, adjoint=False, method="rk4", options={"step_size": 0.5})
            want = O.cdeint_linear(co.double(), O.knot_times(length, torch.float64),
                                   func.linear.weight.detach().cpu().double(), func.linear.bias.detach().cpu().double(),
                                   z0.double(), t_out.double(), "rk4", 0.5)
        _assert_close(out, want, torch.float32)
    finally:
        _set_variant(0)


def test_control_with_own_knots_on_device():
    """Non-default knots live on the device: the schedule reads them back once (one sync), results as usual."""
    length, channels, hidden, batch = 15, 8, 32, 33
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(batch, length, channels, generator=gen, dtype=torch.float64).cumsum(1) / 4
    knots = (torch.rand(length, generator=gen, dtype=torch.float64) + 0.3).cumsum(0)
    z0 = torch.randn(batch, hidden, generator=gen, dtype=torch.float64)
    torch.manual_seed(2)
    func = cde.LinearVectorField(hidden, channels).to(DEV)
    co = O.hermite_backward_difference_coeffs(x.float(), knots.float())
    X = cde.CubicSpline(co.to(DEV), knots.float().to(DEV))
    with torch.no_grad():
        out = cde.cdeint(X, func, z0.float().to(DEV), X.interval, adjoint=False, method="rk4", options={"step_size": 0.25})
        want = O.cdeint_linear(co.double(), knots.float().double(), func.linear.weight.detach().cpu().double(),
                               func.linear.bias.detach().cpu().double(), z0.float().double(),
                               torch.stack([knots.float()[0], knots.float()[-1]]).double(), "rk4", 0.25)
    _assert_close(out, want, torch.float32)


@pytest.mark.parametrize("batch,chunk", [(700, 256), (1000, 96), (64, 4096)])
def test_host_pipelines_equal_the_device_resident_solve(batch, chunk):
    """hostio.cdeint_from_host / cdeint_from_host_series (chunked H2D -> [coefficients ->] solve -> D2H on several
    streams) return the bits of one device-resident cdeint: paths are independent, chunking changes nothing.
    Chunk counts above and below the number of pipeline slots, ragged last chunk, buffers reused across calls."""
    from torchcde_b200 import hostio
    gen = torch.Generator().manual_seed(batch)
    length, channels, hidden = 24, 8, 32
    x = (torch.randn(batch, length, channels, generator=gen).cumsum(1) / math.sqrt(length))
    z0 = torch.randn(batch, hidden, generator=gen)
    torch.manual_seed(4)
    func = cde.LinearVectorField(hidden, channels).to(DEV)
    t = torch.tensor([0.0, 7.5, length - 1.0])
    kw = dict(method="rk4", options={"step_size": 0.5})
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV))
        want = cde.cdeint(cde.CubicSpline(coeffs), func, z0.to(DEV), t, adjoint=False, **kw).cpu()
        x_host, z_host, c_host = x.pin_memory(), z0.pin_memory(), coeffs.cpu().pin_memory()
        for _ in range(2):                                       # second round: cached pipeline buffers
            got = hostio.cdeint_from_host(c_host, func, z_host, t, chunk_paths=chunk, **kw)
            torch.cuda.synchronize()
            assert torch.equal(got, want)
            got = hostio.cdeint_from_host_series(x_host, func, z_host, t, chunk_paths=chunk, **kw)
            torch.cuda.synchronize()
            assert torch.equal(got, want)
        lin = cde.LinearInterpolation(x.to(DEV))
        want_lin = cde.cdeint(lin, func, z0.to(DEV), t, adjoint=False, **kw).cpu()
        got = hostio.cdeint_from_host(x_host, func, z_host, t, kind="linear", chunk_paths=chunk, **kw)
        torch.cuda.synchronize()
        assert torch.equal(got, want_lin)
