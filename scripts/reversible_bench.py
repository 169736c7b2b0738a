"""Reversible Heun (backend="torchsde") against the rk4 adjoint training step at config 3 (65,536 paths, 256 knots,
8 channels, hidden 32), dt = step = 1, alternating in one process.  Prints the card and its power limit, the forward
and forward + backward times (median of --reps), the peak memory of the backward and the error of each method's
outputs against a fine fp64 solve (rk4, step 1/16) on the first 1,024 paths."""
import argparse
import json
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchcde_b200 as cde  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    args = ap.parse_args()
    dev = "cuda"
    gen = torch.Generator().manual_seed(0)
    x = (torch.randn(args.batch, 256, 8, generator=gen) / 16).cumsum(1).to(dev)
    z0 = torch.randn(args.batch, 32, generator=gen).to(dev)
    torch.manual_seed(0)
    func = cde.LinearVectorField(32, 8).to(dev)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    X = cde.CubicSpline(coeffs)
    ts = X.interval
    calls = {
        "reversible_heun": lambda y0, adj: cde.cdeint(X, func, y0, ts, adjoint=adj, backend="torchsde",
                                                      method="reversible_heun", dt=1.0),
        "rk4": lambda y0, adj: cde.cdeint(X, func, y0, ts, adjoint=adj, method="rk4", options={"step_size": 1.0}),
    }
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    times = {k: {"forward": [], "train": [], "peak_backward": 0} for k in calls}
    for rep in range(args.reps + 1):                  # the first round warms up
        for name, call in calls.items():
            with torch.no_grad():
                a, b = ev(), ev()
                a.record()
                call(z0, False)
                b.record()
                torch.cuda.synchronize()
            if rep > 0:
                times[name]["forward"].append(a.elapsed_time(b))
            y0 = z0.clone().requires_grad_(True)
            func.zero_grad()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            a, b = ev(), ev()
            a.record()
            out = call(y0, True)
            loss = out[:, -1].square().sum()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            loss.backward()
            b.record()
            torch.cuda.synchronize()
            if rep > 0:
                times[name]["train"].append(a.elapsed_time(b))
                times[name]["peak_backward"] = max(times[name]["peak_backward"],
                                                   torch.cuda.max_memory_allocated() - base)
            del out, loss, y0
    # accuracy against a fine fp64 solve on the first 1,024 paths
    n = 1024
    f64 = cde.LinearVectorField(32, 8).to(device=dev, dtype=torch.float64)
    f64.load_state_dict({k: v.double() for k, v in func.state_dict().items()})
    X64 = cde.CubicSpline(coeffs[:n].double())
    with torch.no_grad():
        fine = cde.cdeint(X64, f64, z0[:n].double(), ts.double(), adjoint=False, method="rk4",
                          options={"step_size": 1 / 16})
        Xs = cde.CubicSpline(coeffs[:n])
        got = {"reversible_heun": cde.cdeint(Xs, func, z0[:n], ts, backend="torchsde", method="reversible_heun", dt=1.0),
               "rk4": cde.cdeint(Xs, func, z0[:n], ts, adjoint=False, method="rk4", options={"step_size": 1.0})}
    scale = fine.abs().max().item()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    result = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "batch": args.batch}
    for name in calls:
        result[name] = {"forward_ms": round(med(times[name]["forward"]), 3),
                        "forward_backward_ms": round(med(times[name]["train"]), 3),
                        "peak_backward_MiB": round(times[name]["peak_backward"] / 2 ** 20, 1),
                        "max_err_vs_fine_fp64_of_scale": (got[name].double() - fine).abs().max().item() / scale}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
