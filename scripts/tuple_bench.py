"""Time a no-grad rk4 cdeint of a tuple state on the GPU: the grouped stage loop, the same loop with one launch per
member, and the torch-operator tuple loop, alternated in one process.

Problem (a training-size batch): 65,536 paths of length 256, two members -- a cubic spline with 8 channels driving a
hidden state of 32, a linear interpolation with 3 channels driving a hidden state of 8 -- each with a small MLP field
(Linear(H, 64) -> softplus -> Linear(64, H C) -> tanh), rk4 with step 1 over the whole interval (255 steps).

Usage: python scripts/tuple_bench.py [--paths N] [--length L] [--reps R] [--out FILE]
Prints one JSON line (and writes it to FILE): milliseconds per solve (median over R), library calls per step, the
largest difference between the variants' outputs, and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torchcde_b200 as cde  # noqa: E402
from torchcde_b200 import _lib, solver, tuple_solver  # noqa: E402


class MLP(torch.nn.Module):
    def __init__(self, hidden, channels, width=64):
        super().__init__()
        self.hidden, self.channels = hidden, channels
        self.l1, self.l2 = torch.nn.Linear(hidden, width), torch.nn.Linear(width, hidden * channels)

    def forward(self, t, z):
        return self.l2(torch.nn.functional.softplus(self.l1(z))).tanh().view(*z.shape[:-1], self.hidden, self.channels)


class TupleMLP(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a, self.b = MLP(32, 8), MLP(8, 3)

    def forward(self, t, z):
        return self.a(t, z[0]), self.b(t, z[1])


def per_member_calls():
    """Patch the library binding so that every grouped call runs as one launch per member (same kernels, same bits)."""
    real = _lib.call

    def call(name, *args):
        if name in ("tcde_spline_eval_grouped", "tcde_field_contract_grouped"):
            descs, n = args[0], args[1]
            for k in range(n):
                one = (type(descs[k]) * 1)(descs[k])
                real(name, one, 1, *args[2:])
            return 0
        return real(name, *args)
    return call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tuple_bench.py measures on a GPU and found none")
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(0)
    xa = (torch.randn(args.paths, args.length, 8, generator=gen) / 8).cumsum(1).to(dev)
    xb = (torch.randn(args.paths, args.length, 3, generator=gen) / 8).cumsum(1).to(dev)
    X = cde.TupleControl(cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(xa)),
                         cde.LinearInterpolation(xb))
    torch.manual_seed(0)
    func = TupleMLP().to(dev)
    z0 = (torch.randn(args.paths, 32, generator=gen).to(dev), torch.randn(args.paths, 8, generator=gen).to(dev))
    t = X.interval
    opts = {"step_size": 1.0}
    n_steps = args.length - 1
    packing = tuple_solver.Packing(z0)

    def grouped():
        return cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=opts)

    def member_launches():
        real = _lib.call
        _lib.call = per_member_calls()
        try:
            return grouped()
        finally:
            _lib.call = real

    def torch_loop():
        prod = tuple_solver._PackedProd(func, False, packing)
        ys = solver._generic_solve(X, prod, packing.pack(z0), t, "rk4", 1.0, True, False)
        return packing.outputs(ys)

    variants = {"grouped": grouped, "per_member": member_launches, "torch_ops": torch_loop}
    def launches_per_step(per_member):
        """library calls (each one launch here) per step of the grouped loop, or of its per-member form"""
        real, names = _lib.call, []

        def counting(n, *a):
            names.append(n)
            return real(n, *a)
        _lib.call = counting
        if per_member:
            _lib.call = per_member_calls()               # splits each grouped call, then counts the launches
        try:
            with torch.no_grad():
                grouped()
        finally:
            _lib.call = real
        return len(names) / n_steps

    calls = {"grouped": launches_per_step(False), "per_member": launches_per_step(True)}

    times = {k: [] for k in variants}
    outs = {}
    with torch.no_grad():
        for k, f in variants.items():                      # warm-up
            outs[k] = f()
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for k, f in variants.items():                  # alternated
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                f()
                end.record()
                torch.cuda.synchronize()
                times[k].append(start.elapsed_time(end))
    diff = {k: max(float((a - b).abs().max()) for a, b in zip(outs[k], outs["grouped"])) for k in outs}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": smi, "paths": args.paths, "length": args.length, "steps": n_steps,
           "ms_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
           "ms_all": times,
           "library_calls_per_step": calls,
           "max_abs_diff_vs_grouped": diff}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
