"""Reversible Heun (backend="torchsde") against the rk4 adjoint training step, dt = step = 1, alternating in one process.
Prints the card and its power limit, the forward and forward + backward times (median of --reps), the peak memory of the
backward and the error of each route's outputs against a fine fp64 solve (rk4, step 1/16) on the first 1,024 paths.

--field linear (default): config 3 (65,536 paths, 256 knots, 8 channels, hidden 32) with the README's linear field;
routes: reversible Heun and rk4 adjoint=True.
--field mlp: the examples' MLP field (Linear(H, W) -> ReLU -> Linear(W, H C) -> tanh) at --hidden / --channels / --width
/ --dtype; routes: reversible Heun on its kernels, the same solve as torch operators with per-step autograd (forced by an
equivalent module the kernels do not recognise: it holds a Dropout(p=0)), and as context rk4 adjoint=True and
adjoint=False.  --variant sets the solve variant (1 forces the CUDA-core kernels at hidden > 8)."""
import argparse
import json
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchcde_b200 as cde  # noqa: E402
from torchcde_b200 import _lib  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


class Mlp(torch.nn.Module):
    """The examples' field; with ``hidden_dropout`` an equivalent module (Dropout(p=0) in eval mode changes nothing) that
    the kernels' probe refuses, so cdeint runs it as torch operators."""

    def __init__(self, hidden, channels, width, hidden_dropout=False):
        super().__init__()
        self.linear1 = torch.nn.Linear(hidden, width)
        self.linear2 = torch.nn.Linear(width, hidden * channels)
        self.drop = torch.nn.Dropout(0.0) if hidden_dropout else torch.nn.Identity()
        self.hidden, self.channels = hidden, channels

    def forward(self, t, z):
        return torch.tanh(self.linear2(self.drop(self.linear1(z).relu()))).view(*z.shape[:-1], self.hidden,
                                                                                 self.channels)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--field", choices=["linear", "mlp"], default="linear")
    ap.add_argument("--hidden", type=int, default=None)
    ap.add_argument("--channels", type=int, default=None)
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--dtype", choices=["float32", "float64"], default="float32")
    ap.add_argument("--variant", type=int, default=0)
    args = ap.parse_args()
    mlp = args.field == "mlp"
    hidden = args.hidden or (8 if mlp else 32)
    channels = args.channels or (3 if mlp else 8)
    dtype = getattr(torch, args.dtype)
    dev = "cuda"
    _lib.call("tcde_set_solve_variant", args.variant)
    gen = torch.Generator().manual_seed(0)
    x = (torch.randn(args.batch, 256, channels, generator=gen, dtype=torch.float64) / 16).cumsum(1).to(dev, dtype)
    z0 = torch.randn(args.batch, hidden, generator=gen, dtype=torch.float64).to(dev, dtype)
    torch.manual_seed(0)
    if mlp:
        func = Mlp(hidden, channels, args.width).to(dev, dtype).eval()
        twin = Mlp(hidden, channels, args.width, hidden_dropout=True).to(dev, dtype).eval()
        twin.load_state_dict(func.state_dict())
    else:
        func = cde.LinearVectorField(hidden, channels).to(dev, dtype)
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x)
    X = cde.CubicSpline(coeffs)
    ts = X.interval

    def rev(f):
        return lambda X_, y0, adj: cde.cdeint(X_, f, y0, ts, adjoint=adj, backend="torchsde", method="reversible_heun",
                                              dt=1.0)

    def rk4(adjoint):
        return lambda X_, y0, adj: cde.cdeint(X_, func, y0, ts, adjoint=adjoint if adj else False, method="rk4",
                                              options={"step_size": 1.0})

    calls = {"reversible_heun": rev(func)}
    if mlp:
        calls["reversible_heun_torch_ops"] = rev(twin)
        calls["rk4_adjoint"] = rk4(True)
        calls["rk4_backprop"] = rk4(False)
    else:
        calls["rk4"] = rk4(True)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    times = {k: {"forward": [], "train": [], "peak_backward": 0} for k in calls}
    for rep in range(args.reps + 1):                  # the first round warms up
        for name, call in calls.items():
            with torch.no_grad():
                a, b = ev(), ev()
                a.record()
                call(X, z0, False)
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
            out = call(X, y0, True)
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
    f64 = (Mlp(hidden, channels, args.width) if mlp else cde.LinearVectorField(hidden, channels)).to(dev, torch.float64)
    f64.load_state_dict({k: v.double() for k, v in func.state_dict().items()})
    with torch.no_grad():
        fine = cde.cdeint(cde.CubicSpline(coeffs[:n].double()), f64, z0[:n].double(), ts.double(), adjoint=False,
                          method="rk4", options={"step_size": 1 / 16})
        Xs = cde.CubicSpline(coeffs[:n])
        got = {name: call(Xs, z0[:n], False) for name, call in calls.items()}
    scale = fine.abs().max().item()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    result = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "batch": args.batch,
              "field": args.field, "hidden": hidden, "channels": channels, "dtype": args.dtype, "variant": args.variant}
    if mlp:
        result["width"] = args.width
    for name in calls:
        result[name] = {"forward_ms": round(med(times[name]["forward"]), 3),
                        "forward_backward_ms": round(med(times[name]["train"]), 3),
                        "peak_backward_MiB": round(times[name]["peak_backward"] / 2 ** 20, 1),
                        "max_err_vs_fine_fp64_of_scale": (got[name].double() - fine).abs().max().item() / scale}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
