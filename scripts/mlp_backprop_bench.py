"""Time one training step (forward + ``out[:, -1].sum().backward()``) of cdeint at length 256 with the examples' MLP field
(by default config 3: channels 8, hidden 32, width 128; cubic control, rk4, step 1) on three routes, alternated in one
process:

  * ``backprop``: adjoint=False on the three-launch discrete backward (stage-dump solve, tcde_cdeint_fixed_mlp_backward,
    tcde_mlp_field_param_grads);
  * ``torch_loop``: adjoint=False on the torch-operator solve (the route declined), at half the largest halving of the
    batch whose autograd graph fits on its own (reported as ``batch``), so that it also fits next to the other routes;
  * ``adjoint``: adjoint=True (the fused forward, three launches per output segment backwards).

Each step is bracketed by device synchronisations; medians over the repetitions, the peak allocated memory of each
route, and each route's dL/dz0 and dL/dW2 against the backprop route's on the same batch.  The card's name, power limit
and SM clock are read in the same run.  ``--profile DIR``: instead, one step of each route under torch.profiler, the
per-kernel CUDA times written to DIR/mlp_backprop_kernels.txt.
usage: python scripts/mlp_backprop_bench.py [--batch 65536] [--reps 3] [--hidden 32] [--channels 8] [--width 128]
                                           [--profile DIR]"""
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
from torchcde_b200 import solver  # noqa: E402


class Func(torch.nn.Module):
    """example/time_series_classification.py:20-51's CDEFunc."""

    def __init__(self):
        super().__init__()
        self.linear1 = torch.nn.Linear(H, W)
        self.linear2 = torch.nn.Linear(W, C * H)

    def forward(self, t, z):
        return self.linear2(self.linear1(z).relu()).tanh().view(*z.shape[:-1], H, C)

L, C, H, W = 256, 8, 32, 128
dev = torch.device("cuda")


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
    x = torch.randn(batch, L, C, generator=gen, device=dev).cumsum(1) / math.sqrt(L)
    z0 = torch.randn(batch, H, generator=gen, device=dev)
    torch.manual_seed(1)
    func = Func().to(dev)
    with torch.no_grad():
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
    return X, func, z0


def step(route, X, func, z0):
    """One timed training step: (seconds, peak bytes, dL/dz0, dL/dW2)."""
    real = solver.mlp_backprop
    if route == "torch_loop":
        solver.mlp_backprop = lambda *args: None
    try:
        zz = z0.clone().requires_grad_(True)
        func.zero_grad()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = cde.cdeint(X, func, zz, X.interval, adjoint=route == "adjoint", method="rk4", options={"step_size": 1.0})
        out[:, -1].sum().backward()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dt, torch.cuda.max_memory_allocated(), zz.grad, func.linear2.weight.grad.clone()
    finally:
        solver.mlp_backprop = real


def rel(got, want, per_path):
    got, want = got.double(), want.double()
    if per_path:
        return ((got - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-300)).max().item()
    return ((got - want).abs().max() / want.abs().max()).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--hidden", type=int, default=32)
    ap.add_argument("--channels", type=int, default=8)
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    global C, H, W
    C, H, W = args.channels, args.hidden, args.width
    info = card()
    full = problem(args.batch)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        step("backprop", *full)
        step("adjoint", *full)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step("backprop", *full)
            step("adjoint", *full)
        os.makedirs(args.profile, exist_ok=True)
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
        with open(os.path.join(args.profile, "mlp_backprop_kernels.txt"), "w") as f:
            f.write(json.dumps(info) + "\n" + table)
        print(table)
        return
    # the largest batch (full, then halvings) whose torch-operator step fits in memory
    loop_batch = args.batch
    while True:
        try:
            sub = full if loop_batch == args.batch else tuple(
                [cde.CubicSpline(full[0]._rows()[:loop_batch]), full[1], full[2][:loop_batch]])
            step("torch_loop", *sub)
            break
        except torch.OutOfMemoryError:
            torch.cuda.empty_cache()
            loop_batch //= 2
    # once more halved: the timed loop runs alongside the other routes' inputs and gradients
    loop_batch //= 2
    loop_problem = (cde.CubicSpline(full[0]._rows()[:loop_batch]), full[1], full[2][:loop_batch])
    torch.cuda.empty_cache()
    runs = {"backprop": (full, args.batch), "torch_loop": (loop_problem, loop_batch), "adjoint": (full, args.batch)}
    for name, (prob, _b) in runs.items():             # warm-up of every route
        step(name, *prob)
    times = {name: [] for name in runs}
    peak, grads = {}, {}
    for _ in range(args.reps):
        for name, (prob, _b) in runs.items():
            dt, mem, gz, gw = step(name, *prob)
            times[name].append(dt)
            peak[name] = max(peak.get(name, 0), mem)
            grads[name] = (gz, gw)
            del gz, gw
    ref_loop = step("backprop", *loop_problem)[2:] if loop_batch != args.batch else grads["backprop"]
    for name, (_prob, batch) in runs.items():
        ref = ref_loop if name == "torch_loop" else grads["backprop"]
        gz, gw = grads[name]
        print(json.dumps({
            "route": name, "batch": batch, "median_s": statistics.median(times[name]), "all_s": times[name],
            "sequences_per_s": batch / statistics.median(times[name]), "peak_gib": peak[name] / 2 ** 30,
            "dl_dz0_vs_backprop": rel(gz, ref[0], True), "dl_dw2_vs_backprop": rel(gw, ref[1], False),
            "gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock": info.get("clocks.sm"),
            "max_sm_clock": info.get("clocks.max.sm"), "hidden": H, "channels": C, "width": W}), flush=True)


if __name__ == "__main__":
    main()
