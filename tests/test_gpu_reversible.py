"""cdeint(backend="torchsde", method="reversible_heun") on the GPU: the fused forward against the fp64 oracle and the
fp64 kernel, the reversible backward against autograd, its memory and its determinism."""

import pytest
import torch

import torchcde_b200 as cde
from oracle import reversible_oracle as R
from torchcde_b200 import reversible

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
