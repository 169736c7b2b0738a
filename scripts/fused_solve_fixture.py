#!/usr/bin/env python
"""The exact output bits of the fused 2xFP16 tensor-core solve on fixed, seeded inputs (1,000 paths on 40 knots, hidden 32,
channels 8), for tests/golden/fused_solve_bits.npz and tests/test_gpu_fused_solve_bits.py.

    python scripts/fused_solve_fixture.py OUT.npz

Cases, on the fixed-step schedules F1-F8 of tests/test_host_logic.py:
  * fwd/<F>/<method>/<control>: cdeint's outputs (cdeint_wgmma_kernel) for rk4, midpoint, euler, cubic and linear control;
  * dump/<F>/<method>: the stage-dump solve's outputs and stage inputs, and tcde_cdeint_fixed_linear_backward's dL/dz0
    and kappa dump for seeded output gradients (the BWD kernel);
  * rev/<F>: reversible Heun's outputs without and with checkpoints, and dL/dz0 of its backward (one launch of
    reversible_backward_kernel per checkpoint segment).
Each array is kept as the SHA-256 of its bytes (so -0.0 and +0.0 differ) and, for a readable failure, the last output,
stage or state of four of its paths: 0, 63, 64 (both sides of the first 64-path tile) and 999 (the partial last tile)."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torchcde_b200 as cde  # noqa: E402
from test_host_logic import FIXED_SCHEDULES, fixed_schedule_knots  # noqa: E402
from torchcde_b200 import _lib  # noqa: E402
from torchcde_b200.linear_field import FixedBackprop, LinearFieldKernels  # noqa: E402
from torchcde_b200.schedule import backward_tables  # noqa: E402

PATHS, LENGTH, HIDDEN, CHANNELS = 1000, 40, 32, 8
SAMPLE = [0, 63, 64, 999]
METHODS = ("rk4", "midpoint", "euler")
DUMP_SCHEDULES = ("F3", "F4", "F6", "F8")
REV_SCHEDULES = ("F3", "F7")


def _inputs(dev, uneven):
    gen = torch.Generator().manual_seed(2024)
    x = (torch.randn(PATHS, LENGTH, CHANNELS, generator=gen, dtype=torch.float64) / 16).cumsum(1).float()
    z0 = torch.randn(PATHS, HIDDEN, generator=gen, dtype=torch.float64).float()
    bound = HIDDEN ** -0.5
    w = ((2 * torch.rand(HIDDEN * CHANNELS, HIDDEN, generator=gen, dtype=torch.float64) - 1) * bound).float()
    b = ((2 * torch.rand(HIDDEN * CHANNELS, generator=gen, dtype=torch.float64) - 1) * bound).float()
    knots = fixed_schedule_knots(True).to(dev) if uneven else None
    x = x.to(dev)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x, t=knots)
    func = cde.LinearVectorField(HIDDEN, CHANNELS).to(dev)
    with torch.no_grad():
        func.linear.weight.copy_(w)
        func.linear.bias.copy_(b)
    return x, knots, coeffs, z0.to(dev), func


def _problem(dev, sname, control):
    ts, step, uneven = FIXED_SCHEDULES[sname]
    x, knots, coeffs, z0, func = _inputs(dev, uneven)
    if ts is None:
        t = fixed_schedule_knots(uneven).double()
    else:
        t = torch.tensor(ts, dtype=torch.float32 if sname == "F4" else torch.float64)
    X = cde.CubicSpline(coeffs, t=knots) if control == "cubic" else cde.LinearInterpolation(x, t=knots)
    return X, func, z0, t, step


def _grads(shape, dev):
    gen = torch.Generator().manual_seed(7)
    return torch.randn(*shape, generator=gen, dtype=torch.float64).float().to(dev)


def compute(dev):
    """{case name: float32 array} of the current build on ``dev``."""
    got = {}
    with torch.no_grad():
        for sname in FIXED_SCHEDULES:
            for method in METHODS:
                for control in ("cubic", "linear"):
                    X, func, z0, t, step = _problem(dev, sname, control)
                    opts = {} if step is None else {"step_size": step}
                    out = cde.cdeint(X, func, z0, t, adjoint=False, method=method, options=opts)
                    got["fwd/{}/{}/{}".format(sname, method, control)] = out
        for sname in DUMP_SCHEDULES:
            for method in METHODS:
                X, func, z0, t, step = _problem(dev, sname, "cubic")
                k = LinearFieldKernels(X, func.linear.weight, func.linear.bias, z0)
                route = FixedBackprop(k, t, method, step, None)
                out, dump = route.forward(z0)
                sched = route.sched
                g = _grads(out.shape, dev)
                n_total = sched.n_steps * sched.n_stages
                gz = torch.empty(PATHS, HIDDEN, device=dev)
                kappa = torch.empty_like(dump)
                tables = backward_tables(sched)
                floats = torch.cat([tables["step_dt"], tables["stage_frac"], tables["inj_weight"]]).to(dev)
                ints = torch.cat([tables["stage_index"], tables["inj_range"], tables["inj_out"]]).to(dev)
                ns, nr = sched.n_steps, tables["inj_range"].numel()
                w_t, zeros = k.transposed_weights
                _lib.call("tcde_cdeint_fixed_linear_backward", _lib.ptr(k.control), k.kind, k.n_rows, _lib.ptr(w_t),
                          _lib.ptr(zeros), _lib.ptr(g), _lib.ptr(gz), _lib.ptr(kappa), PATHS, CHANNELS, HIDDEN,
                          _lib.METHODS[method], ns, _lib.ptr(floats[:ns]), _lib.ptr(ints[:n_total]),
                          _lib.ptr(floats[ns:ns + n_total]), sched.n_out, _lib.ptr(ints[n_total:n_total + nr]),
                          _lib.ptr(ints[n_total + nr:]), _lib.ptr(floats[ns + n_total:]), float(sched.sign), _lib.F32,
                          _lib.stream_of(g))
                name = "dump/{}/{}/".format(sname, method)
                got[name + "out"], got[name + "stages"] = out, dump.transpose(0, 1)
                got[name + "dl_dz0"], got[name + "kappa"] = gz, kappa.transpose(0, 1)
    for sname in REV_SCHEDULES:
        X, func, z0, t, _step = _problem(dev, sname, "cubic")
        with torch.no_grad():
            got["rev/{}/out".format(sname)] = cde.cdeint(X, func, z0, t, backend="torchsde", method="reversible_heun",
                                                          dt=0.4)
        y0 = z0.clone().requires_grad_(True)
        out = cde.cdeint(X, func, y0, t, adjoint=True, backend="torchsde", method="reversible_heun", dt=0.4)
        out.backward(_grads(out.shape, dev))
        got["rev/{}/out_ckpt".format(sname)] = out.detach()
        got["rev/{}/dl_dz0".format(sname)] = y0.grad
    torch.cuda.synchronize(dev)
    return {name: v.detach().float().contiguous().cpu().numpy() for name, v in got.items()}


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def sample(a):
    """The values of ``a`` [paths, ...] kept beside its digest: the last slot of axis 1 (outputs, stages) of the SAMPLE
    paths, or their whole rows for a [paths, hidden] array."""
    a = a[SAMPLE]
    return np.ascontiguousarray(a[:, -1] if a.ndim == 3 else a)


def main():
    dev = torch.device("cuda:0")
    got = compute(dev)
    fixture = {}
    for name, a in got.items():
        assert a.shape[0] == PATHS, (name, a.shape)
        fixture[name + "#sha256"] = digest(a)
        fixture[name + "#sample"] = sample(a)
    np.savez_compressed(sys.argv[1], **fixture)
    print("{} arrays, {} bytes, to {}".format(len(got), sum(a.nbytes for a in got.values()), sys.argv[1]))


if __name__ == "__main__":
    main()
