"""Write tests/golden/reference_live.npz: inputs and the reference package's own outputs (and gradients) for the tests that
compare against the reference itself (tests/test_diff_formulas.py, tests/test_oracle_pinned.py fresh inputs,
tests/test_gpu_logsig.py whole transform).  The tests read these arrays, so they run where the reference tree is absent.

    python -m oracle.make_reference_golden        (needs the reference tree: see oracle/reference_loader.py)

Every case is keyed ``<group>__<case number>__<field>``.  Inputs are generated exactly as the tests generated them before
they became self-contained."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import reference_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_live.npz")


def _data(seed, batch=(3,), length=9, channels=2, nan=0.0, irregular=True):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(*batch, length, channels, generator=gen, dtype=torch.float64)
    if nan:
        hole = torch.rand(x.shape, generator=gen) < nan
        x = x.masked_fill(hole, float("nan"))
    t = torch.rand(length, generator=gen, dtype=torch.float64).add(0.2).cumsum(0) if irregular else None
    return x, t


def _value_and_grads(fn, x, t, seed):
    """fn(x, t), a seeded cotangent, and the gradients of <fn, cotangent> w.r.t. x (and t) with NaN outputs masked."""
    xb = x.clone().requires_grad_(True)
    tb = None if t is None else t.clone().requires_grad_(True)
    want = fn(xb, tb)
    ok = ~torch.isnan(want)
    cot = torch.randn(want.shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * ok
    res = {"want": want.detach(), "cot": cot}
    if want.requires_grad:
        ins = [xb] + ([tb] if t is not None else [])
        grads = torch.autograd.grad(torch.where(ok, want, torch.zeros_like(want)), ins, cot, allow_unused=True)
        for name, g in zip(("gx", "gt"), grads):
            res[name] = torch.zeros(1, dtype=torch.float64) if g is None else torch.nan_to_num(g)
    return res


def diff_cases(ref):
    """tests/test_diff_formulas.py: builders' values and gradients."""
    builders = {"hermite": ref.hermite_cubic_coefficients_with_backward_differences, "natural1": ref.natural_cubic_coeffs,
                "natural0": ref.natural_cubic_spline_coeffs, "linear": ref.linear_interpolation_coeffs}
    out = {}
    n = 0
    for nan in (0.0, 0.35):
        for irregular in (False, True):
            for seed, batch, length in ((0, (3,), 9), (1, (2, 2), 6), (2, (), 2), (3, (4,), 3)):
                x, t = _data(seed, batch, length, 2, nan, irregular)
                if nan:
                    x[..., 1, :] = float("nan") if length > 2 else x[..., 1, :]
                    if batch:
                        x[0] = float("nan")
                        x[-1][..., 0, :] = float("nan")
                        x[-1][..., -1, 0] = float("nan")
                for name, fn in builders.items():
                    if name == "linear" and not nan:
                        continue
                    key = "diff__{}__".format(n)
                    out[key + "group"] = np.array([nan, float(irregular)])
                    out[key + "builder"] = np.array(name)
                    out[key + "seed"] = np.array(seed)
                    out[key + "x"] = x.numpy()
                    if t is not None:
                        out[key + "t"] = t.numpy()
                    for field, v in _value_and_grads(fn, x, t, seed).items():
                        out[key + field] = v.numpy()
                    n += 1
                if nan:
                    key = "diff__{}__".format(n)
                    out[key + "group"] = np.array([nan, float(irregular)])
                    out[key + "builder"] = np.array("ffill")
                    out[key + "x"] = x.numpy()
                    out[key + "want"] = ref.misc.forward_fill(x).numpy()
                    n += 1
    # rectilinear
    x, _ = _data(5, (3,), 7, 3, 0.3, False)
    x[..., 0] = torch.arange(7, dtype=torch.float64)
    x[:, 0, :] = 1.0
    out["rect__x"] = x.numpy()
    out["rect__want"] = ref.linear_interpolation_coeffs(x, rectilinear=0).numpy()
    # evaluation formulas
    x, t = _data(7, (2, 3), 8, 2, 0.0, True)
    coeffs = ref.natural_cubic_coeffs(x, t)
    spline = ref.CubicSpline(coeffs, t)
    linear = ref.LinearInterpolation(x, t)
    query = torch.tensor([t[0] - 0.3, t[0], t[2], 0.5 * (t[3] + t[4]), t[-1], t[-1] + 1.0], dtype=torch.float64)
    out["eval__x"], out["eval__t"], out["eval__coeffs"] = x.numpy(), t.numpy(), coeffs.numpy()
    for i, q in enumerate((query, query[3], query.view(2, 3))):
        key = "eval__{}__".format(i)
        frac, index = spline._interpret_t(q)
        _, lindex = linear._interpret_t(q)
        out[key + "q"] = q.numpy()
        out[key + "index"] = np.asarray(index.numpy() if torch.is_tensor(index) else index)
        out[key + "lindex"] = np.asarray(lindex.numpy() if torch.is_tensor(lindex) else lindex)
        out[key + "cubic_eval"] = spline.evaluate(q).numpy()
        out[key + "cubic_deriv"] = spline.derivative(q).numpy()
        out[key + "linear_eval"] = linear.evaluate(q).numpy()
        out[key + "linear_deriv"] = linear.derivative(q).numpy()
    return out


def fresh_cases(ref):
    """tests/test_oracle_pinned.py: the builders on fresh seeded inputs, fp32 and fp64, with and without knots."""
    out = {}
    gen = torch.Generator().manual_seed(31337)
    n = 0
    for dtype in (torch.float32, torch.float64):
        for shape in ((4, 11, 3), (2, 2, 5, 2), (6, 2, 1)):
            x = torch.randn(shape, generator=gen, dtype=torch.float64).to(dtype)
            t = (torch.rand(shape[-2], generator=gen, dtype=torch.float64) + 0.05).cumsum(0).to(dtype)
            for frac in (0.0, 0.25, 0.7):
                xin = x.clone()
                xin[torch.rand(shape, generator=gen) < frac] = float("nan")
                for tt in (None, t):
                    key = "fresh__{}__".format(n)
                    out[key + "x"] = xin.numpy()
                    if tt is not None:
                        out[key + "t"] = tt.numpy()
                    out[key + "linear"] = ref.linear_interpolation_coeffs(xin, tt).numpy()
                    out[key + "hermite"] = ref.hermite_cubic_coefficients_with_backward_differences(xin, tt).numpy()
                    out[key + "natural1"] = ref.natural_cubic_coeffs(xin, tt).numpy()
                    out[key + "natural0"] = ref.natural_cubic_spline_coeffs(xin, tt).numpy()
                    out[key + "ffill"] = ref.misc.forward_fill(xin).numpy()
                    n += 1
    return out


def logsig_cases(ref):
    """tests/test_gpu_logsig.py: the reference's whole log-signature transform, the oracle standing in for signatory."""
    from oracle import logsig_oracle as O
    import types
    log_ode = sys.modules[ref.__name__ + ".log_ode"]
    mod = types.ModuleType("signatory")

    class Logsignature:
        def __init__(self, depth):
            self.depth = depth

        def __call__(self, paths):
            return torch.tensor(np.stack([O.logsignature(p.detach().cpu().double().numpy(), self.depth) for p in paths]),
                                dtype=paths.dtype)

    mod.Logsignature = Logsignature
    mod.logsignature_channels = lambda channels, depth: len(O.lyndon_words(channels, depth))
    saved = getattr(log_ode, "signatory", None)
    log_ode.signatory = mod
    out = {}
    try:
        torch.manual_seed(1)
        cases = (((2,), 11, 2, 3, 2.5, False, 0.0), ((3,), 9, 3, 2, 4.0, True, 0.3), ((2, 2), 7, 1, 4, 1.0, False, 0.2),
                 ((1,), 6, 2, 2, 10.0, True, 0.0))
        for i, (batch, length, channels, depth, window, irregular, nan) in enumerate(cases):
            x = torch.randn(*batch, length, channels, dtype=torch.float64)
            if nan:
                hole = torch.rand(x.shape) < nan
                hole[..., 0, :] = False
                hole[..., -1, :] = False
                x = x.masked_fill(hole, float("nan"))
            t = (torch.rand(length, dtype=torch.float64) + 0.3).cumsum(0) if irregular else None
            key = "logsig__{}__".format(i)
            out[key + "x"] = x.numpy()
            out[key + "depth"] = np.array(depth)
            out[key + "window"] = np.array(window)
            if t is not None:
                out[key + "t"] = t.numpy()
            out[key + "want"] = ref.logsig_windows(x, depth, window, t).numpy()
            want_v, want_t = ref.logsignature_windows(x, depth, window, t)
            out[key + "want_v"], out[key + "want_t"] = want_v.numpy(), want_t.numpy()
    finally:
        log_ode.signatory = saved
    return out


def main():
    ref = reference_loader.load_reference()
    out = {}
    out.update(diff_cases(ref))
    out.update(fresh_cases(ref))
    out.update(logsig_cases(ref))
    np.savez_compressed(OUT, **out)
    print("wrote {} arrays to {} ({} bytes)".format(len(out), OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
