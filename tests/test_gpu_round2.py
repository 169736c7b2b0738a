"""Round-2 GPU tests: full-batch parity of the tensor-core solve, the ADVICE r01 regressions and the
reference-compatibility details added in round 2.  Everything here goes through the C ABI on the device."""
import math

import pytest
import torch

import torchcde_b200 as cde

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bench_problem(batch, nan_fraction=0.0, seed=0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    L, C, H = 256, 8, 32
    x = torch.randn(batch, L, C, generator=gen, device=DEV).cumsum(1) / math.sqrt(L)
    if nan_fraction:
        hole = torch.rand(x.shape, generator=gen, device=DEV) < nan_fraction
        hole[:, 0] = False
        hole[:, -1] = False
        x = x.masked_fill(hole, float("nan"))
    z0 = torch.randn(batch, H, generator=gen, device=DEV)
    torch.manual_seed(1)
    func = cde.LinearVectorField(H, C).to(DEV)
    return x, z0, func


@pytest.mark.parametrize("nan_fraction", [0.0, 0.3])
def test_full_batch_fp32_tensor_core_solve_against_fp64_kernel(nan_fraction):
    """ALL 65,536 paths of BASELINE config 3 (and of a 30 %-NaN config-2 -> config-3 pipeline): the fp32 tensor-core
    solve against the fp64 CUDA-core solve (itself oracle-checked to 1e-10 in test_gpu_solve.py) on the same
    fp32-rounded coefficients.  Bar: 1e-5 of the solution scale on every element."""
    B = 65536
    x, z0, func = _bench_problem(B, nan_fraction)
    opts = {"step_size": 1.0}
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
        assert bool(torch.isfinite(coeffs).all())
        X = cde.CubicSpline(coeffs)
        got = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options=opts)
        f64 = cde.LinearVectorField(32, 8, dtype=torch.float64).to(DEV)
        f64.linear.weight.copy_(func.linear.weight.double())
        f64.linear.bias.copy_(func.linear.bias.double())
        worst, scale = 0.0, 0.0
        for lo in range(0, B, 16384):                      # fp64 coefficients of 16,384 paths: 1 GiB at a time
            Xd = cde.CubicSpline(coeffs[lo:lo + 16384].double())
            want = cde.cdeint(Xd, f64, z0[lo:lo + 16384].double(), Xd.interval, adjoint=False, method="rk4", options=opts)
            worst = max(worst, float((got[lo:lo + 16384].double() - want).abs().max()))
            scale = max(scale, float(want.abs().max()))
    assert math.isfinite(scale) and scale > 1.0
    assert worst <= 1e-5 * scale, "max |fp32 tensor-core - fp64| = {:.3e} at scale {:.3e}".format(worst, scale)


def test_large_hidden_linear_field_falls_back_to_the_stage_loop():
    """ADVICE r01 (medium): hidden=128, channels=8 does not fit the fused kernels; the reference handles it, so must we."""
    torch.manual_seed(0)
    x = torch.randn(5, 12, 8, device=DEV).cumsum(1) / 4
    func = cde.LinearVectorField(128, 8).to(DEV)
    with torch.no_grad():
        func.linear.weight.mul_(0.3)
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
        z0 = torch.randn(5, 128, device=DEV)
        out = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})

        class Opaque:
            def __call__(self, t, z):
                return func(t, z)

        want = cde.cdeint(X, Opaque(), z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
    assert out.shape == (5, 2, 128)
    assert torch.allclose(out, want, rtol=1e-5, atol=1e-5)


def test_kernel_backed_routes_reject_mismatched_dtype_and_device():
    """ADVICE r01 (medium): dopri5 / adjoint routes hand raw pointers to the kernels -- a float64 spline with a
    float32 state, or a field left on the CPU, must raise a clean RuntimeError like the reference's torch ops do."""
    torch.manual_seed(0)
    x = torch.randn(4, 9, 8, device=DEV).cumsum(1) / 3
    with torch.no_grad():
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    func = cde.LinearVectorField(32, 8).to(DEV)
    z0 = torch.randn(4, 32, device=DEV)
    X64 = cde.CubicSpline(coeffs.double())
    for kwargs in ({"method": "rk4", "options": {"step_size": 1.0}}, {}):           # fixed step and the default dopri5
        with pytest.raises(RuntimeError, match="must match"):
            with torch.no_grad():
                cde.cdeint(X64, func, z0, X64.interval, adjoint=False, **kwargs)
        with pytest.raises(RuntimeError):
            with torch.no_grad():
                cde.cdeint(cde.CubicSpline(coeffs), cde.LinearVectorField(32, 8), z0, X64.interval, adjoint=False, **kwargs)
    zg = z0.clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match="must match"):
        cde.cdeint(X64, func, zg, X64.interval, adjoint=True, method="rk4", options={"step_size": 1.0})
    # the device is still healthy (no sticky error): a correct call works
    with torch.no_grad():
        X = cde.CubicSpline(coeffs)
        out = cde.cdeint(X, func, z0, X.interval, adjoint=False, method="rk4", options={"step_size": 1.0})
    assert bool(torch.isfinite(out).all())


def test_linear_interpolation_state_dict_matches_the_reference_keys():
    """ADVICE r01 (low): reference checkpoints of LinearInterpolation hold ``_t``, ``_coeffs``, ``_derivs``
    (interpolation_linear.py:191-193) and must load with strict=True; slopes follow a load."""
    torch.manual_seed(0)
    a = torch.randn(3, 7, 2, device=DEV)
    b = torch.randn(3, 7, 2, device=DEV)
    Xa, Xb = cde.LinearInterpolation(a), cde.LinearInterpolation(b)
    assert sorted(Xa.state_dict().keys()) == ["_coeffs", "_derivs", "_t"]
    want = (a[:, 1:] - a[:, :-1]) / 1.0
    assert torch.equal(Xa._derivs, want)
    Xb.load_state_dict(Xa.state_dict(), strict=True)
    assert torch.equal(Xb._derivs, want) and torch.equal(Xb.derivative(torch.tensor(2.5, device=DEV)), want[:, 2])
    # a module built on the CPU and moved afterwards carries the same slopes
    Xc = cde.LinearInterpolation(a.cpu()).to(DEV)
    assert torch.equal(Xc._derivs, want)


class _MlpField(torch.nn.Module):
    """The vector field of example/time_series_classification.py:37-51 (MLP + tanh)."""

    def __init__(self, input_channels, hidden_channels):
        super().__init__()
        self.input_channels, self.hidden_channels = input_channels, hidden_channels
        self.linear1 = torch.nn.Linear(hidden_channels, 128)
        self.linear2 = torch.nn.Linear(128, input_channels * hidden_channels)

    def forward(self, t, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], self.hidden_channels, self.input_channels)


@pytest.mark.parametrize("method,step", [("rk4", 1.0), ("midpoint", 0.5), ("euler", 0.25)])
def test_generic_field_kernel_loop_and_cuda_graph(method, step):
    """SURVEY 8(f)1: an arbitrary func runs through this package's stage loop -- dX/dt of a step's stages in one launch,
    Runge-Kutta combinations as single launches, optionally the whole loop as one CUDA graph -- with the numbers of the
    differentiable torch-operator loop (which is what autograd uses)."""
    from torchcde_b200 import solver
    torch.manual_seed(0)
    x = torch.randn(64, 20, 3, device=DEV).cumsum(1) / 4
    func = _MlpField(3, 8).to(DEV)
    z0 = torch.randn(64, 8, device=DEV)
    t = torch.tensor([0.0, 7.3, 19.0])
    for make in (lambda: cde.CubicSpline(cde.natural_cubic_coeffs(x)), lambda: cde.LinearInterpolation(x)):
        X = make()
        with torch.no_grad():
            fast = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options={"step_size": step})
            graph = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options={"step_size": step, "cuda_graph": True})
            again = cde.cdeint(X, func, z0 * 0.5, t, adjoint=False, method=method, options={"step_size": step, "cuda_graph": True})
            half = cde.cdeint(X, func, z0 * 0.5, t, adjoint=False, method=method, options={"step_size": step})
            slow = solver._generic_solve(X, func, z0, t, method, step, False, True)
        assert fast.shape == (64, 3, 8)
        assert torch.allclose(fast, slow, rtol=1e-5, atol=1e-5)
        assert torch.allclose(graph, fast, rtol=1e-6, atol=1e-6)
        assert torch.allclose(again, half, rtol=1e-6, atol=1e-6)          # the replay really read the new z0
        # reversed time: the sign is folded into the contraction kernel (tcde_field_contract)
        t_rev = torch.tensor([19.0, 7.3, 0.0])
        with torch.no_grad():
            fast_rev = cde.cdeint(X, func, z0, t_rev, adjoint=False, method=method, options={"step_size": step})
            slow_rev = solver._generic_solve(X, func, z0, t_rev, method, step, False, True)
        assert torch.allclose(fast_rev, slow_rev, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_field_contract_kernel_against_matmul(dtype):
    """solver.py:129-135: (f @ dX.unsqueeze(-1)).squeeze(-1) as tcde_field_contract, with dX a strided view."""
    from torchcde_b200 import _lib
    torch.manual_seed(3)
    P, H, C, S = 77, 13, 5, 4
    f = torch.randn(P, H, C, device=DEV, dtype=dtype)
    dxs = torch.randn(P, S, C, device=DEV, dtype=dtype)
    for s in range(S):
        for scale in (1.0, -1.0):
            out = torch.empty(P, H, device=DEV, dtype=dtype)
            _lib.call("tcde_field_contract", _lib.ptr(f), _lib.ptr(dxs[:, s]), _lib.ptr(out), P, H, C, S * C, scale,
                      _lib.dtype_code(dtype), _lib.stream_of(f))
            want = scale * (f.double() @ dxs[:, s].double().unsqueeze(-1)).squeeze(-1)
            tol = 1e-5 if dtype == torch.float32 else 1e-13
            assert torch.allclose(out.double(), want, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(7, 256, 8), (5, 33, 3), (3, 2, 1), (4, 100, 32), (2, 700, 4), (6, 17, 5)])
@pytest.mark.parametrize("with_t", [False, True])
def test_fused_fill_and_hermite_is_bit_identical_to_the_two_kernels(dtype, shape, with_t):
    """VERDICT r01 item 8: hermite_cubic_coefficients_with_backward_differences of a series with gaps is ONE launch
    (tcde_hermite_bdiff_coeffs_series); it must reproduce tcde_linear_fill -> tcde_hermite_bdiff_coeffs bit for bit,
    gaps at the ends, all-NaN channels and gap-free paths included."""
    from torchcde_b200 import _lib
    gen = torch.Generator(device=DEV).manual_seed(shape[1] * 31 + shape[2])
    P, L, C = shape
    x = torch.randn(P, L, C, generator=gen, device=DEV, dtype=dtype).cumsum(1)
    hole = torch.rand(P, L, C, generator=gen, device=DEV) < 0.35
    hole[0] = False                                       # a path without gaps
    if P > 2:
        hole[1, :, 0] = True                              # an all-NaN channel
        hole[2, : L // 2, -1] = True                      # a missing start
        hole[2, -1, 0] = True                             # a missing end
    x = x.masked_fill(hole, float("nan"))
    t = (torch.rand(L, generator=gen, device=DEV, dtype=dtype) + 0.1).cumsum(0) if with_t else None
    code = _lib.dtype_code(dtype)
    filled = torch.empty_like(x)
    want = torch.empty(P, L - 1, 4 * C, device=DEV, dtype=dtype)
    got = torch.full_like(want, float("nan"))
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    stream = _lib.stream_of(x)
    _lib.call("tcde_linear_fill", _lib.ptr(x), _lib.ptr(t), _lib.ptr(filled), P, L, C, code, None, stream)
    _lib.call("tcde_hermite_bdiff_coeffs", _lib.ptr(filled), _lib.ptr(t), _lib.ptr(want), P, L, C, code, None, stream)
    assert bool(torch.isfinite(want).all())
    try:
        _lib.call("tcde_hermite_bdiff_coeffs_series", _lib.ptr(x), _lib.ptr(t), _lib.ptr(got), P, L, C, code, _lib.ptr(flags), stream)
        fused = True
    except NotImplementedError:                           # eight warp tiles of this shape do not fit shared memory (fp64 at 256 x 8)
        fused = False
    assert fused or L * C * x.element_size() * 8 > 90 * 1024
    if fused:
        assert torch.equal(got, want)
        assert int(flags.item()) & _lib.FLAG_NAN_SEEN
    # and the public builder (which now calls the fused entry) agrees with the differentiable restatement
    pub = cde.hermite_cubic_coefficients_with_backward_differences(x, t)
    assert torch.equal(pub, want)


def test_fused_fill_and_hermite_reports_unsupported_shapes_and_the_builder_falls_back():
    from torchcde_b200 import _lib
    x = torch.randn(2, 9, 40, device=DEV)                 # channels > 32: no warp tile
    x[0, 3, 5] = float("nan")
    out = torch.empty(2, 8, 160, device=DEV)
    with pytest.raises(NotImplementedError):
        _lib.call("tcde_hermite_bdiff_coeffs_series", _lib.ptr(x), None, _lib.ptr(out), 2, 9, 40, _lib.dtype_code(x.dtype),
                  None, _lib.stream_of(x))
    got = cde.hermite_cubic_coefficients_with_backward_differences(x)
    want = cde.hermite_cubic_coefficients_with_backward_differences(cde.linear_interpolation_coeffs(x))
    assert bool(torch.isfinite(got).all()) and torch.equal(got, want)
