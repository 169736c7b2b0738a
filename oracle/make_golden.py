"""Generate tests/golden/*.npz from the LIVE reference -- run where a reference checkout exists.

    python -m oracle.make_golden

Every array under ``ref_*`` keys is an output of the unmodified reference code imported
from the reference checkout (``oracle/reference_loader.py``); the ``in_*`` arrays are the seeded
inputs that produced them.  Nothing here is computed by the oracle or by the CUDA path.
The only non-reference arithmetic involved is the fixed-grid stepping inside the
``cdeint`` fixtures, which is ``oracle/odeint_port.py`` standing where torchdiffeq would
(those files are named ``solve_*`` and carry ``stepping='odeint_port'``).

The first fixture re-states the known-answer tensors hard-coded in the reference's own
test (test/test_linear_interpolation.py:125-137) so that they are pinned even if the
reference tree is not around.
"""
import math
import os
import warnings

import numpy as np
import torch

from . import reference_loader

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
NAN = float("nan")


def _np(x):
    return x.detach().cpu().numpy()


def _holes(x, frac, gen, keep_ends=False, kill_channel=None):
    mask = torch.rand(x.shape, generator=gen) < frac
    if keep_ends:
        mask[..., 0, :] = False
        mask[..., -1, :] = False
    x = x.clone()
    x[mask] = NAN
    if kill_channel is not None:
        x[0, :, kill_channel] = NAN          # one series with no observation at all
    return x


def builders(ref):
    """Coefficient builders: every (dtype, t, NaN pattern) combination, small shapes."""
    gen = torch.Generator().manual_seed(1234)
    cases = {}
    n = 0
    for dtype in (torch.float32, torch.float64):
        for shape in ((3, 9, 2), (2, 2, 6, 3), (4, 2, 1), (5, 2, 2), (7, 4), (2, 33, 8)):
            length = shape[-2]
            for own_t in (False, True):
                x = torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype)
                t = ((torch.rand(length, generator=gen, dtype=torch.float64) + 0.1).cumsum(0)).to(dtype) \
                    if own_t else None
                for pattern in ("dense", "interior", "ragged", "sparse"):
                    if pattern == "dense":
                        xin = x
                    elif pattern == "interior":
                        xin = _holes(x, 0.3, gen, keep_ends=True)
                    elif pattern == "ragged":
                        xin = _holes(x, 0.4, gen, kill_channel=0 if len(shape) > 2 else None)
                    else:
                        xin = _holes(x, 0.85, gen)
                    key = "c{:03d}".format(n)
                    n += 1
                    cases[key + "_in_x"] = _np(xin)
                    if t is not None:
                        cases[key + "_in_t"] = _np(t)
                    cases[key + "_ref_linear"] = _np(ref.linear_interpolation_coeffs(xin, t))
                    cases[key + "_ref_hermite"] = _np(ref.hermite_cubic_coefficients_with_backward_differences(xin, t))
                    cases[key + "_ref_natural_v1"] = _np(ref.natural_cubic_coeffs(xin, t))
                    cases[key + "_ref_natural_v0"] = _np(ref.natural_cubic_spline_coeffs(xin, t))
                    cases[key + "_ref_ffill"] = _np(ref.misc.forward_fill(xin))
    cases["count"] = np.array(n)
    np.savez_compressed(os.path.join(OUT, "builders.npz"), **cases)
    return n


def rectilinear(ref):
    cases = {}
    # known answers written out in the reference's own test (test_linear_interpolation.py:125-137)
    x = torch.tensor([[[0.1, 0.4], [0.2, NAN], [0.9, 1.1]],
                      [[0.2, NAN], [0.3, 2.0], [0.3, NAN]]])
    known = torch.tensor([[[0.1, 0.4], [0.2, 0.4], [0.2, 0.4], [0.9, 0.4], [0.9, 1.1]],
                          [[0.2, 2.0], [0.3, 2.0], [0.3, 2.0], [0.3, 2.0], [0.3, 2.0]]])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = ref.linear_interpolation_coeffs(x, rectilinear=0)
        assert torch.equal(got, known)
        cases["k_in_x"] = _np(x)
        cases["k_known"] = _np(known)
        cases["k_ref_swapped"] = _np(ref.linear_interpolation_coeffs(x[:, :, [1, 0]], rectilinear=1))
        gen = torch.Generator().manual_seed(99)
        n = 0
        for dtype in (torch.float32, torch.float64):
            for shape, tc in (((4, 7, 3), 0), ((2, 3, 5, 4), 2), ((6, 2), 1), ((3, 20, 5), 4)):
                x = torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype)
                x[..., tc] = x[..., tc].abs().cumsum(-1) if x.dim() == 2 else x[..., tc].abs().cumsum(-1)
                xin = _holes(x, 0.35, gen)
                xin[..., tc] = x[..., tc]
                key = "r{:02d}".format(n)
                n += 1
                cases[key + "_in_x"] = _np(xin)
                cases[key + "_time_index"] = np.array(tc)
                cases[key + "_ref"] = _np(ref.linear_interpolation_coeffs(xin, rectilinear=tc))
    cases["count"] = np.array(n)
    np.savez_compressed(os.path.join(OUT, "rectilinear.npz"), **cases)
    return n


def evaluation(ref):
    """CubicSpline / LinearInterpolation evaluate, derivative and (bit-exact) interval indices."""
    gen = torch.Generator().manual_seed(7)
    cases = {}
    n = 0
    for dtype in (torch.float32, torch.float64):
        for shape in ((3, 9, 2), (2, 2, 6, 3), (5, 1), (2, 257, 4)):
            length = shape[-2]
            for own_t in (False, True):
                x = torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype)
                t = ((torch.rand(length, generator=gen, dtype=torch.float64) + 0.1).cumsum(0)).to(dtype) \
                    if own_t else None
                coeffs = ref.natural_cubic_coeffs(x, t)
                spline = ref.CubicSpline(coeffs, t)
                knots_x = ref.linear_interpolation_coeffs(x, t)
                linear = ref.LinearInterpolation(knots_x, t)
                grid = spline.grid_points
                span = float(grid[-1] - grid[0])
                inside = torch.rand(40, generator=gen, dtype=torch.float64) * span * 1.2 + float(grid[0]) - 0.1 * span
                thirds = (grid[:-1, None] + (grid[1:] - grid[:-1])[:, None]
                          * torch.tensor([1 / 3, 2 / 3], dtype=dtype)).flatten()[:60]
                just_above = torch.nextafter(grid, grid + 1)[:30]
                query = torch.cat([grid[:30], just_above, thirds, inside.to(dtype)])
                frac, index = spline._interpret_t(query)
                key = "e{:02d}".format(n)
                n += 1
                cases[key + "_in_x"] = _np(x)
                if t is not None:
                    cases[key + "_in_t"] = _np(t)
                cases[key + "_in_query"] = _np(query)
                cases[key + "_ref_coeffs"] = _np(coeffs)
                cases[key + "_ref_index"] = _np(index)
                cases[key + "_ref_frac"] = _np(frac)
                cases[key + "_ref_cubic_eval"] = _np(spline.evaluate(query))
                cases[key + "_ref_cubic_deriv"] = _np(spline.derivative(query))
                cases[key + "_ref_linear_eval"] = _np(linear.evaluate(query))
                cases[key + "_ref_linear_deriv"] = _np(linear.derivative(query))
    cases["count"] = np.array(n)
    np.savez_compressed(os.path.join(OUT, "evaluation.npz"), **cases)
    return n


class _ReadmeFunc(torch.nn.Module):
    """The README's vector field (README.md:42-49), batch-shape agnostic."""

    def __init__(self, hidden, channels, dtype, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.hidden, self.channels = hidden, channels
        self.linear = torch.nn.Linear(hidden, hidden * channels).to(dtype)

    def forward(self, t, z):
        return self.linear(z).view(*z.shape[:-1], self.hidden, self.channels)


def solves(ref):
    """Reference ``cdeint`` + ``_VectorField`` run end to end, stepping by oracle/odeint_port.py."""
    gen = torch.Generator().manual_seed(2024)
    cases = {"stepping": np.array("odeint_port")}
    n = 0
    plans = (
        # (batch shape, L, C, H, builder, control, method, step, t kind)
        ((6,), 12, 3, 4, "hermite", "cubic", "rk4", 1.0, "interval"),
        ((6,), 12, 3, 4, "hermite", "cubic", "rk4", 0.5, "inner64"),
        ((2, 3), 9, 2, 5, "natural", "cubic", "midpoint", 1.0, "knots"),
        ((4,), 17, 8, 32, "hermite", "cubic", "rk4", 1.0, "interval"),
        ((4,), 17, 8, 32, "hermite", "cubic", "euler", 0.25, "inner"),
        ((3,), 10, 2, 3, "linear", "linear", "rk4", 1.0, "interval"),
        ((3,), 10, 2, 3, "linear", "linear", "midpoint", 0.5, "inner"),
        ((5,), 8, 4, 6, "hermite", "cubic", "rk4", None, "knots"),
        ((5,), 8, 4, 6, "hermite_t", "cubic", "rk4", 0.3, "inner"),
        ((1,), 10, 2, 3, "hermite", "cubic", "rk4", 1.0, "reversed"),
    )
    with torch.no_grad():
        for dtype in (torch.float32, torch.float64):
            for bshape, length, chan, hid, builder, kind, method, step, tkind in plans:
                x = (torch.randn(*bshape, length, chan, generator=gen, dtype=torch.float64).cumsum(-2)
                     / math.sqrt(length)).to(dtype)
                t_knots = None
                if builder == "hermite":
                    control = ref.hermite_cubic_coefficients_with_backward_differences(x)
                elif builder == "hermite_t":
                    t_knots = ((torch.rand(length, generator=gen, dtype=torch.float64) + 0.2).cumsum(0)).to(dtype)
                    control = ref.hermite_cubic_coefficients_with_backward_differences(x, t_knots)
                elif builder == "natural":
                    control = ref.natural_cubic_coeffs(x)
                else:
                    control = ref.linear_interpolation_coeffs(x)
                X = ref.CubicSpline(control, t_knots) if kind == "cubic" else ref.LinearInterpolation(control, t_knots)
                lo, hi = X.interval
                if tkind == "interval":
                    t = X.interval
                elif tkind == "knots":
                    t = X.grid_points
                elif tkind == "inner":
                    w = torch.rand(5, generator=gen, dtype=torch.float64).sort().values.to(dtype)
                    t = torch.cat([lo.view(1), lo + (hi - lo) * w, hi.view(1)])
                elif tkind == "inner64":      # float64 output times with a float32 state (test_cdeint.py:43)
                    w = torch.rand(5, generator=gen, dtype=torch.float64).sort().values
                    t = torch.cat([lo.view(1).double(), lo.double() + (hi - lo).double() * w, hi.view(1).double()])
                else:
                    t = torch.stack([hi, lo])
                func = _ReadmeFunc(hid, chan, dtype, seed=100 + n)
                z0 = torch.randn(*bshape, hid, generator=gen, dtype=torch.float64).to(dtype)
                options = {} if step is None else {"step_size": step}
                out = ref.cdeint(X, func, z0, t, adjoint=False, method=method, options=options)
                # one bare vector-field evaluation straight from the reference (solver.py:117-135)
                vf = ref.solver._VectorField(X, func, True, False)
                probe = torch.as_tensor(float(lo) + 0.37 * float(hi - lo), dtype=dtype)
                key = "s{:02d}".format(n)
                n += 1
                cases[key + "_in_control"] = _np(control)
                if t_knots is not None:
                    cases[key + "_in_knots"] = _np(t_knots)
                cases[key + "_in_weight"] = _np(func.linear.weight)
                cases[key + "_in_bias"] = _np(func.linear.bias)
                cases[key + "_in_z0"] = _np(z0)
                cases[key + "_in_t"] = _np(t)
                cases[key + "_kind"] = np.array(kind)
                cases[key + "_method"] = np.array(method)
                cases[key + "_step"] = np.array(-1.0 if step is None else step)
                cases[key + "_ref_out"] = _np(out)
                cases[key + "_in_probe"] = _np(probe)
                cases[key + "_ref_field"] = _np(vf(probe, z0))
    cases["count"] = np.array(n)
    np.savez_compressed(os.path.join(OUT, "solves.npz"), **cases)
    return n


def main():
    torch.set_num_threads(1)
    os.makedirs(OUT, exist_ok=True)
    ref = reference_loader.load_reference()
    print("builders   :", builders(ref))
    print("rectilinear:", rectilinear(ref))
    print("evaluation :", evaluation(ref))
    print("solves     :", solves(ref))
    for name in sorted(os.listdir(OUT)):
        print("  {:20s} {:8d} B".format(name, os.path.getsize(os.path.join(OUT, name))))


if __name__ == "__main__":
    main()
