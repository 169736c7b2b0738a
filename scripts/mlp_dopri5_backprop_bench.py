"""Time one training step (forward + backward of a random cotangent on the outputs) of cdeint with its default method,
dopri5, and default tolerances (rtol 1e-4, atol 1e-6) at batch 65,536, length 256, cubic control, and the examples' MLP
field (Linear(H, W) -> ReLU -> Linear(W, H C) -> tanh) at (H, C, W) = (8, 3, 128) by default, on three routes,
alternated in one process:

  * ``backprop``: adjoint=False on the recording host-driven forward, one tcde_dopri5_mlp_backward launch and one
    tcde_mlp_field_param_grads call per record chunk (mlp_field.Dopri5MlpBackprop);
  * ``adjoint``: adjoint=True, the examples' default call (the host-driven forward, one tcde_vector_field_mlp_vjp call per
    stage of the backward where the shape is served);
  * ``torch_loop``: adjoint=False on the torch-operator dopri5 (the route declined): one autograd graph over every accepted
    step.  It runs at the largest halving of the batch whose step fits (reported as ``batch``).

Each step is bracketed by device synchronisations; medians over the repetitions, the peak allocated memory of each
route (for ``backprop``: the record and the backward's buffers), its accepted / rejected step counts, and its dL/dz0
against the backprop route's on the same paths.  The card's name, power limit and SM clock are read in the same run.
usage: python scripts/mlp_dopri5_backprop_bench.py [--batch 65536] [--reps 3] [--hidden 8 --channels 3 --width 128]
       [--dtype fp32|fp64] [--variant 0|1]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import torchcde_b200 as cde  # noqa: E402
from torchcde_b200 import adaptive, solver  # noqa: E402

L = 256
H, C, W = 8, 3, 128
DTYPE = torch.float32
dev = torch.device("cuda")


class Func(torch.nn.Module):
    """example/time_series_classification.py's CDEFunc."""

    def __init__(self, input_channels, hidden_channels, width):
        super().__init__()
        self.input_channels, self.hidden_channels = input_channels, hidden_channels
        self.linear1 = torch.nn.Linear(hidden_channels, width)
        self.linear2 = torch.nn.Linear(width, input_channels * hidden_channels)

    def forward(self, t, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], self.hidden_channels, self.input_channels)


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
    x = (torch.randn(batch, L, C, generator=gen, device=dev).cumsum(1) / math.sqrt(L)).to(DTYPE)
    z0 = torch.randn(batch, H, generator=gen, device=dev).to(DTYPE)
    g = torch.randn(batch, 2, H, generator=gen, device=dev).to(DTYPE)
    torch.manual_seed(1)
    func = Func(C, H, W).to(dev).to(DTYPE)
    with torch.no_grad():
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    return X, func, z0, g


def step(route, X, func, z0, g):
    """(seconds, dL/dz0, stats, peak bytes) of one training step on ``route``."""
    z = z0.clone().requires_grad_(True)
    func.zero_grad(set_to_none=True)
    t = torch.tensor([0.0, L - 1.0], dtype=torch.float64)
    real, real_solve = solver.dopri5_mlp_backprop, adaptive.odeint_dopri5
    stats = {}
    if route == "torch_loop":
        def solve(*args, **kwargs):                       # the torch-operator solve leaves no last_stats: count here
            out, solver_obj = real_solve(*args, **kwargs)
            stats.update(n_accepted=solver_obj.n_accepted, n_rejected=solver_obj.n_rejected)
            return out, solver_obj

        solver.dopri5_mlp_backprop = lambda *args: None
        adaptive.odeint_dopri5 = solve
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = cde.cdeint(X, func, z, t, adjoint=route == "adjoint")
        if route != "torch_loop":
            stats = dict(cde.cdeint.last_stats)
        if route == "backprop":
            assert type(out.grad_fn).__name__ == "_Dopri5MlpBackpropFnBackward", "the route declined the problem"
        out.backward(g)
        torch.cuda.synchronize()
        seconds = time.perf_counter() - t0
    finally:
        solver.dopri5_mlp_backprop, adaptive.odeint_dopri5 = real, real_solve
    stats.pop("steps", None)
    return seconds, z.grad, stats, torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--hidden", type=int, default=8)
    ap.add_argument("--channels", type=int, default=3)
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--dtype", choices=["fp32", "fp64"], default="fp32")
    ap.add_argument("--variant", type=int, default=0)
    args = ap.parse_args()
    global H, C, W, DTYPE
    H, C, W, DTYPE = args.hidden, args.channels, args.width, {"fp32": torch.float32, "fp64": torch.float64}[args.dtype]
    if not torch.cuda.is_available():
        raise SystemExit("mlp_dopri5_backprop_bench.py measures on a GPU; none is visible")
    from torchcde_b200 import _lib
    _lib.call("tcde_set_solve_variant", args.variant)
    full = problem(args.batch)
    # the torch-operator route at the largest halving of the batch whose step fits
    loop_batch = args.batch
    while True:
        small = problem(loop_batch) if loop_batch != args.batch else full
        try:
            step("torch_loop", *small)
            break
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            loop_batch //= 2
            if loop_batch < 256:
                raise
    runs = {"backprop": full, "adjoint": full, "torch_loop": small}
    for name, prob in runs.items():                       # warm-up of every route
        step(name, *prob)
    times = {name: [] for name in runs}
    last = {}
    for _ in range(args.reps):
        for name, prob in runs.items():
            sec, gz, stats, peak = step(name, *prob)
            times[name].append(sec)
            last[name] = (gz, stats, peak)
    ref_gz = last["backprop"][0]
    result = {"card": card(), "length": L, "hidden": H, "channels": C, "width": W, "dtype": args.dtype,
              "variant": args.variant, "reps": args.reps}
    for name in runs:
        gz, stats, peak = last[name]
        m = gz.size(0)
        err = ((gz - ref_gz[:m]).abs().max() / ref_gz[:m].abs().max()).item()
        if name == "torch_loop" and m != ref_gz.size(0):
            err = None                                    # a different batch has its own step sequence
        result[name] = {"batch": m, "median_s": statistics.median(times[name]), "all_s": times[name],
                        "median_s_per_sequence": statistics.median(times[name]) / m,
                        "peak_gib": peak / 2 ** 30, "n_accepted": stats.get("n_accepted"),
                        "n_rejected": stats.get("n_rejected"), "dl_dz0_vs_backprop": err}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
