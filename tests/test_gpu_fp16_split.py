"""The 2xFP16 operand split of solve_tc.cu (variant 4) on inputs that stress its per-path scaling: states far from
1 in magnitude, wide dynamic range inside a row, zero / tiny / huge bias, zero weight; for rk4 and for reversible Heun
(torchsde backend, dt = 1).  Reference = the fp64 CUDA-core solve of the same method on the same fp32-rounded inputs;
bar = 1e-5 of each path's own solution scale (the 3xTF32 kernel, variant 3, must meet the same bar: the two splits
carry the same 22 significand bits)."""
import math

import pytest
import torch

import torchcde_b200 as cde
from torchcde_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _solve(X, func, z0, variant, method):
    t = X.interval
    _lib.call("tcde_set_solve_variant", variant)
    try:
        with torch.no_grad():
            if method == "reversible_heun":
                return cde.cdeint(X, func, z0, t, backend="torchsde", method="reversible_heun", dt=1.0)
            return cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options={"step_size": 1.0})
    finally:
        _lib.call("tcde_set_solve_variant", 0)


CASES = ["plain", "tiny_state", "huge_state", "wide_rows", "no_bias", "tiny_bias", "huge_bias", "zero_weight",
         "zero_state"]


# the method axis: the reversible Heun instantiations form their stage input as z = 2 y - z + f dt rather than
# y + dt k; the rk4 cases keep their plain case names as ids
@pytest.mark.parametrize("variant", [3, 4])
@pytest.mark.parametrize("method,case", [("rk4", c) for c in CASES] + [("reversible_heun", c) for c in CASES],
                         ids=CASES + ["reversible_heun-" + c for c in CASES])
def test_split_precision_under_scaling(method, case, variant):
    torch.manual_seed(11)
    B, L, C, H = 300, 24, 8, 32
    x = (torch.randn(B, L, C, dtype=torch.float64).cumsum(1) / math.sqrt(L)).float().to(DEV)
    z0 = torch.randn(B, H, dtype=torch.float64).float().to(DEV)
    func = cde.LinearVectorField(H, C).to(DEV)
    with torch.no_grad():
        func.linear.weight.mul_(0.5)
        if case == "tiny_state":
            z0 *= 1e-9
            func.linear.bias.zero_()
        elif case == "huge_state":
            z0 *= 3e7
        elif case == "wide_rows":
            z0 *= torch.exp(4.0 * torch.randn(B, H, device=DEV))
        elif case == "no_bias":
            func.linear.bias.zero_()
        elif case == "tiny_bias":
            func.linear.bias.mul_(1e-12)
            z0 *= 1e-8
        elif case == "huge_bias":
            func.linear.bias.mul_(1e6)
        elif case == "zero_weight":
            func.linear.weight.zero_()
        elif case == "zero_state":
            z0.zero_()
        coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    X = cde.CubicSpline(coeffs)
    got = _solve(X, func, z0, variant, method)
    f64 = cde.LinearVectorField(H, C, dtype=torch.float64).to(DEV)
    with torch.no_grad():
        f64.linear.weight.copy_(func.linear.weight.double())
        f64.linear.bias.copy_(func.linear.bias.double())
    want = _solve(cde.CubicSpline(coeffs.double()), f64, z0.double(), 1, method)
    assert bool(torch.isfinite(want).all())
    scale = want.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-300)      # per path
    err = ((got.double() - want).abs() / scale).max().item()
    print("split {} {} variant {}: {:.2e} of path scale".format(method, case, variant, err))
    assert err <= 1e-5, "{} {} variant {}: max error / path scale = {:.3e}".format(method, case, variant, err)
