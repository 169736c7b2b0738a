"""The examples' MLP vector field (Linear(H, 128) -> ReLU -> Linear(128, H*C) -> tanh) under cdeint's fixed-step rk4:
the fused solve (``tcde_cdeint_fixed_mlp``, automatic and forced CUDA-core routes) against this package's stage loop and
its CUDA graph, at B = 65,536 paths, length 256, step 1, (H, C) = (8, 3) and (32, 8).

The routes alternate within every repetition in one process (CUDA events, medians of ``--reps``).  Also printed: the
card's name and power limit, the MMA flops the 2xFP16 tensor-core kernel executes (three split products per layer)
against the 989 TFLOP/s dense-fp16 datasheet figure, and the adjoint=True training step (forward + backward) with the
fused forward against the stage-loop forward.

    python scripts/mlp_bench.py [--reps 5] [--train-reps 3]
"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchcde_b200 as cde  # noqa: E402
from torchcde_b200 import _lib, solver  # noqa: E402

B, L, WIDTH = 65536, 256, 128
DENSE_FP16_TFLOPS = 989.0


class Func(torch.nn.Module):
    def __init__(self, channels, hidden):
        super().__init__()
        self.channels, self.hidden = channels, hidden
        self.linear1 = torch.nn.Linear(hidden, WIDTH)
        self.linear2 = torch.nn.Linear(WIDTH, hidden * channels)

    def forward(self, t, z):
        z = self.linear2(self.linear1(z).relu()).tanh()
        return z.view(*z.shape[:-1], self.hidden, self.channels)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                # noqa: BLE001 -- the numbers still print, without the limit
        q = "unknown ({})".format(exc)
    return name, q


def time_ms(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


@contextlib.contextmanager
def variant(v):
    _lib.call("tcde_set_solve_variant", v)
    try:
        yield
    finally:
        _lib.call("tcde_set_solve_variant", 0)


@contextlib.contextmanager
def without_mlp_route():
    real = solver.mlp_field_of
    solver.mlp_field_of = lambda *a, **k: None
    try:
        yield
    finally:
        solver.mlp_field_of = real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--train-reps", type=int, default=3)
    args = ap.parse_args()
    name, limits = card()
    print("card: {} | power.limit, clocks.max.sm: {}".format(name, limits))
    dev = torch.device("cuda:0")
    t = torch.tensor([0.0, L - 1.0])
    opts = {"step_size": 1.0}
    report = {"card": name, "power_limit_and_max_sm_clock": limits, "shapes": {}}
    for hidden, channels in ((8, 3), (32, 8)):
        gen = torch.Generator().manual_seed(0)
        x = (torch.randn(B, L, channels, generator=gen) / 4).cumsum(1).to(dev)
        X = cde.CubicSpline(cde.hermite_cubic_coefficients_with_backward_differences(x))
        del x
        z0 = torch.randn(B, hidden, generator=gen).to(dev)
        torch.manual_seed(1)
        func = Func(channels, hidden).to(dev)
        holder = {}

        def fused():
            holder["fused"] = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=opts)

        def cuda_core():
            with variant(1):
                holder["cuda_core"] = cde.cdeint(X, func, z0, t, adjoint=False, method="rk4", options=opts)

        def loop():
            holder["loop"] = solver._generic_solve_kernels(X, func, z0, t, "rk4", 1.0, False, False)

        def graph():
            holder["graph"] = solver._generic_solve_kernels(X, func, z0, t, "rk4", 1.0, False, True)

        routes = {"fused_auto": fused, "fused_cuda_core": cuda_core, "stage_loop": loop, "stage_loop_cuda_graph": graph}
        with torch.no_grad():
            for fn in routes.values():                      # warm-up: module loads, graph capture
                fn()
            times = {k: [] for k in routes}
            for _ in range(args.reps):
                for k, fn in routes.items():
                    times[k].append(time_ms(fn))
        med = {k: statistics.median(v) for k, v in times.items()}
        err = {k: ((holder[k] - holder["loop"]).abs().amax(dim=(1, 2)) /
                   holder["loop"].abs().amax(dim=(1, 2)).clamp_min(1e-30)).max().item() for k in ("fused", "cuda_core")}
        row = {"ms_median": med, "ms_all": times, "max_path_rel_diff_vs_stage_loop": err,
               "speedup_vs_cuda_graph": med["stage_loop_cuda_graph"] / med["fused_auto"]}
        if (hidden, channels) == (32, 8):
            stages = 4 * (L - 1)
            mma = 3 * 2 * (hidden * WIDTH + WIDTH * hidden * channels)      # per path and stage, three split products
            tflops = B * stages * mma / (med["fused_auto"] * 1e-3) / 1e12
            row["mma_tflops_executed"] = tflops
            row["share_of_989_dense_fp16"] = tflops / DENSE_FP16_TFLOPS

        # adjoint=True training step: fused forward vs the stage-loop forward, the same autograd-per-stage backward
        def train():
            zz = z0.clone().requires_grad_(True)
            func.zero_grad()
            out = cde.cdeint(X, func, zz, t, adjoint=True, method="rk4", options=opts)
            out[:, -1].sum().backward()

        def train_loop():
            with without_mlp_route():
                train()

        train()
        train_loop()
        tt = {"fused_forward": [], "stage_loop_forward": []}
        for _ in range(args.train_reps):
            tt["fused_forward"].append(time_ms(train))
            tt["stage_loop_forward"].append(time_ms(train_loop))
        row["adjoint_training_step_ms_median"] = {k: statistics.median(v) for k, v in tt.items()}
        row["adjoint_training_step_ms_all"] = tt
        report["shapes"]["H{}_C{}".format(hidden, channels)] = row
        print(json.dumps({"H": hidden, "C": channels, **row}), flush=True)
        del X, z0, holder
        torch.cuda.empty_cache()
    print(json.dumps(report))


if __name__ == "__main__":
    main()
