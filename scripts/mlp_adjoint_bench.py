"""Time one adjoint=True training step (forward + ``out[:, -1].sum().backward()``) of cdeint with the examples' MLP field
(hidden 8, channels 3, width 128; cubic control of length 256) on two routes, alternated in one process:

  * ``kernels``: the field of the host-driven dopri5 is one launch of tcde_vector_field_mlp per evaluation and every
    backward stage one call of tcde_vector_field_mlp_vjp;
  * ``autograd``: the route before those kernels -- the torch-operator field (``MlpFieldKernels.field`` declines) and an
    autograd vector-Jacobian product per backward stage (``solver._mlp_vjp`` declines).

``--hidden / --channels / --width / --dtype`` time other shapes the kernels serve.  Two workloads: the examples' default call ``cdeint(X, func, z0, X.interval)`` (dopri5, adjoint=True, rtol 1e-4, atol
1e-6) and rk4 with step 1 (the forward is the fused solve on both routes).  Each step is bracketed by device
synchronisations; medians over the repetitions, the peak allocated memory of each step, the accepted and rejected steps
of the forward dopri5 solve, and dL/dz0 and dL/dW2 of the kernel route against the autograd route's.  The card's name,
power limit and SM clock are read in the same run.  ``--profile DIR``: instead, one step of each route and workload under
torch.profiler, the per-kernel CUDA times written to DIR/mlp_adjoint_kernels.txt.
usage: python scripts/mlp_adjoint_bench.py [--batch 65536] [--reps 3] [--workloads dopri5,rk4] [--hidden 8]
                                          [--channels 3] [--width 128] [--dtype fp32] [--profile DIR]"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import torchcde_b200 as cde  # noqa: E402
from torchcde_b200 import solver  # noqa: E402
from torchcde_b200.mlp_field import MlpFieldKernels  # noqa: E402

L, C, H, W = 256, 3, 8, 128
DTYPE = torch.float32
dev = torch.device("cuda")


class Func(torch.nn.Module):
    """example/time_series_classification.py:20-51's CDEFunc."""

    def __init__(self):
        super().__init__()
        self.linear1 = torch.nn.Linear(H, W)
        self.linear2 = torch.nn.Linear(W, C * H)

    def forward(self, t, z):
        return self.linear2(self.linear1(z).relu()).tanh().view(*z.shape[:-1], H, C)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (v.strip() for v in line.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "power.limit": "unknown", "clocks.sm": "unknown"}


def problem(batch):
    gen = torch.Generator(device=dev).manual_seed(0)
    x = (torch.randn(batch, L, C, generator=gen, device=dev) / 16).cumsum(1)
    X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x).to(DTYPE))
    torch.manual_seed(0)
    return X, Func().to(dev, DTYPE), torch.randn(batch, H, generator=gen, device=dev).to(DTYPE)


@contextlib.contextmanager
def route(name):
    """``autograd``: the kernels decline, as for a shape they are not built for."""
    if name == "kernels":
        yield
        return
    real_vjp, real_field = solver._mlp_vjp, MlpFieldKernels.field

    def declined(self):
        def field(*args, **kwargs):
            raise NotImplementedError("declined")
        return field

    solver._mlp_vjp, MlpFieldKernels.field = (lambda *args: None), declined
    try:
        yield
    finally:
        solver._mlp_vjp, MlpFieldKernels.field = real_vjp, real_field


def step(workload, X, func, z0):
    zz = z0.clone().requires_grad_(True)
    for p in func.parameters():
        p.grad = None
    if workload == "dopri5":
        out = cde.cdeint(X=X, z0=zz, func=func, t=X.interval)
    else:
        out = cde.cdeint(X=X, z0=zz, func=func, t=X.interval, method="rk4", options={"step_size": 1.0})
    stats = dict(cde.cdeint.last_stats) if workload == "dopri5" else {}
    out[:, -1].sum().backward()
    return zz.grad, func.linear2.weight.grad.clone(), stats


def rel(got, want, per_path):
    got, want = got.double(), want.double()
    if per_path:
        return float(((got - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-300)).max())
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


def main():
    global H, C, W, DTYPE
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="dopri5,rk4")
    ap.add_argument("--hidden", type=int, default=H)
    ap.add_argument("--channels", type=int, default=C)
    ap.add_argument("--width", type=int, default=W)
    ap.add_argument("--dtype", default="fp32", choices=["fp32", "fp64"])
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    H, C, W = args.hidden, args.channels, args.width
    DTYPE = {"fp32": torch.float32, "fp64": torch.float64}[args.dtype]
    if not torch.cuda.is_available():
        raise SystemExit("mlp_adjoint_bench: no CUDA device")
    X, func, z0 = problem(args.batch)
    workloads = args.workloads.split(",")
    routes = ("kernels", "autograd")
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "mlp_adjoint_kernels.txt"), "w") as f:
            for wl in workloads:
                for name in routes:
                    with route(name):
                        step(wl, X, func, z0)                         # warm-up outside the trace
                        torch.cuda.synchronize()
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            step(wl, X, func, z0)
                            torch.cuda.synchronize()
                    f.write("== {} {} batch {}\n".format(wl, name, args.batch))
                    f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25) + "\n")
        print(json.dumps({"profile": os.path.join(args.profile, "mlp_adjoint_kernels.txt")}))
        return
    info = card()
    for wl in workloads:
        times = {n: [] for n in routes}
        peak, grads, stats = {}, {}, {}
        for name in routes:                                          # warm-up: every route once
            with route(name):
                step(wl, X, func, z0)
        for _ in range(args.reps):
            for name in routes:
                with route(name):
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    gz, gw2, st = step(wl, X, func, z0)
                    torch.cuda.synchronize()
                    times[name].append(time.perf_counter() - t0)
                    peak[name] = torch.cuda.max_memory_allocated() / 2 ** 30
                    grads[name], stats[name] = (gz, gw2), st
        med = {n: statistics.median(v) for n, v in times.items()}
        print(json.dumps({
            "workload": wl, "batch": args.batch, "shape": [H, C, W], "dtype": args.dtype, "length": L,
            "reps": args.reps,
            "median_s": {n: round(v, 4) for n, v in med.items()},
            "speedup_kernels_over_autograd": round(med["autograd"] / med["kernels"], 3),
            "peak_gib": {n: round(v, 3) for n, v in peak.items()},
            "forward_steps": {n: {k: stats[n].get(k) for k in ("n_accepted", "n_rejected")} for n in routes},
            "dz0_rel_vs_autograd": rel(grads["kernels"][0], grads["autograd"][0], True),
            "dW2_rel_vs_autograd": rel(grads["kernels"][1], grads["autograd"][1], False),
            "gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock": info.get("clocks.sm"),
            "sm_clock_max": info.get("clocks.max.sm")}))


if __name__ == "__main__":
    main()
