"""Write tests/golden/reference_live.npz: inputs and the reference package's own outputs (and gradients) for the tests that
compare against the reference itself (tests/test_diff_formulas.py, tests/test_oracle_pinned.py fresh inputs,
tests/test_gpu_logsig.py and tests/test_gpu_logsig_routes.py whole transform and its gradients,
tests/test_logsig_oracle.py window bookkeeping).  The tests read these arrays, so they run where the reference tree is absent.

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


class _OracleLogsignature(torch.autograd.Function):
    """signatory.Logsignature's call on (paths, length, C), differentiable: forward = the oracle, backward = the oracle's
    exact (complex-step) Jacobian."""

    @staticmethod
    def forward(ctx, paths, depth):
        from oracle import logsig_oracle as O
        ctx.save_for_backward(paths)
        ctx.depth = depth
        return torch.tensor(np.stack([O.logsignature(p.detach().cpu().double().numpy(), depth) for p in paths]),
                            dtype=paths.dtype)

    @staticmethod
    def backward(ctx, grad):
        from oracle import logsig_oracle as O
        paths, = ctx.saved_tensors
        out = [np.einsum("w,wlc->lc", g, O.logsignature_jacobian(p.double().numpy(), ctx.depth))
               for g, p in zip(grad.double().numpy(), paths.detach())]
        return torch.tensor(np.stack(out), dtype=paths.dtype), None


def _with_signatory(ref, call):
    """Run the reference's log_ode.py with a stand-in ``signatory`` whose Logsignature(depth)(paths) is ``call(paths,
    depth)``; returns a function that runs ``fn(ref)`` under the stand-in."""
    from oracle import logsig_oracle as O
    import types
    log_ode = sys.modules[ref.__name__ + ".log_ode"]
    mod = types.ModuleType("signatory")

    class Logsignature:
        def __init__(self, depth):
            self.depth = depth

        def __call__(self, paths):
            return call(paths, self.depth)

    mod.Logsignature = Logsignature
    mod.logsignature_channels = lambda channels, depth: len(O.lyndon_words(channels, depth))

    def run(fn):
        saved = getattr(log_ode, "signatory", None)
        log_ode.signatory = mod
        try:
            return fn()
        finally:
            log_ode.signatory = saved
    return run


def logsig_cases(ref):
    """tests/test_gpu_logsig.py: the reference's whole log-signature transform, the oracle standing in for signatory."""
    run = _with_signatory(ref, _OracleLogsignature.apply)

    def cases():
        out = {}
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
        return out
    return run(cases)


# (batch, length, channels, depth, window, t: "none" / "regular" / "irregular" / "inside" / "outside", NaN holes)
# "inside" / "outside": t = 0, 1, ... with the knot at 2 moved to just inside / just outside torch.allclose's
# tolerance of the window end at 2, so that the end is / is not taken as that observation.
LOGSIG_GRAD_CASES = (
    ((3,), 8, 2, 1, 2.0, "regular", False),
    ((2,), 9, 2, 2, 2.5, "irregular", False),
    ((2, 3), 7, 2, 3, 1.7, "irregular", True),
    ((2,), 6, 3, 4, 2.0, "regular", True),
    ((2,), 7, 2, 2, 2.0, "inside", False),
    ((2,), 7, 2, 2, 2.0, "outside", True),
    ((3,), 10, 1, 4, 3.0, "none", True),
    ((1,), 12, 2, 4, 4.5, "irregular", False),
)


def logsig_grad_cases(ref):
    """The reference's logsig_windows / logsignature_windows and their gradients in x and t for a seeded cotangent, with
    the oracle and its Jacobian standing in for signatory (so the window knots, NaN fill, clip, scaling and cumsum
    are differentiated through the reference's own code)."""
    run = _with_signatory(ref, _OracleLogsignature.apply)

    def cases():
        out = {}
        gen = torch.Generator().manual_seed(4242)
        for i, (batch, length, channels, depth, window, kind, nan) in enumerate(LOGSIG_GRAD_CASES):
            x = torch.randn(*batch, length, channels, generator=gen, dtype=torch.float64)
            if nan:
                hole = torch.rand(x.shape, generator=gen) < 0.3
                hole[..., 0, 0] = True                  # holes in the first and the last row
                hole[..., -1, -1] = True
                x = x.masked_fill(hole, float("nan"))
            if kind == "irregular":
                t = (torch.rand(length, generator=gen, dtype=torch.float64) + 0.3).cumsum(0)
            elif kind == "none":
                t = None
            else:
                t = torch.arange(length, dtype=torch.float64)
                tol = 1e-8 + 1e-5 * 2.0
                t[2] = 2.0 + {"regular": 0.0, "inside": 0.5 * tol, "outside": 2.0 * tol}[kind]
            key = "logsig_grad__{}__".format(i)
            out[key + "x"] = x.numpy()
            out[key + "depth"] = np.array(depth)
            out[key + "window"] = np.array(window)
            if t is not None:
                out[key + "t"] = t.numpy()
            for name in ("logsig", "logsignature"):
                xb = x.clone().requires_grad_(True)
                tb = None if t is None else t.clone().requires_grad_(True)
                if name == "logsig":
                    outs = (ref.logsig_windows(xb, depth, window, tb),)
                else:
                    outs = ref.logsignature_windows(xb, depth, window, tb)
                cots = tuple(torch.randn(o.shape, generator=gen, dtype=torch.float64) for o in outs)
                ins = [xb] + ([tb] if tb is not None else [])
                live = [(o, c) for o, c in zip(outs, cots) if o.requires_grad]     # the times need a differentiable t
                grads = torch.autograd.grad([o for o, _ in live], ins, [c for _, c in live], allow_unused=True)
                prefix = key + name + "__"
                for field, v in zip(("want", "want_t"), outs):
                    out[prefix + field] = v.detach().numpy()
                for field, v in zip(("cot", "cot_t"), cots):
                    out[prefix + field] = v.numpy()
                for field, g, like in zip(("gx", "gt"), grads, ins):
                    out[prefix + field] = (torch.zeros_like(like) if g is None else g).detach().numpy()
        return out
    return run(cases)


def logsig_spy_cases(ref):
    """The lengths of the window slices the reference hands to signatory (log_ode.py:57), which are its window end
    positions in the merged knots: on random fp32 and fp64 ``t``, and on ``t`` with an interior knot placed at the
    edge of torch.allclose's tolerance of a window end, +- a few ulps."""
    lengths = []

    def spy(paths, depth):
        lengths.append(paths.size(-2))
        return torch.zeros(paths.size(0), 1, dtype=paths.dtype)

    run = _with_signatory(ref, spy)
    out = {}
    rng = np.random.default_rng(777)
    n = 0
    for trial in range(300):
        dtype = (np.float32, np.float64)[trial % 2]
        length = int(rng.integers(3, 30))
        t = (rng.random(length) + 0.05).cumsum() if trial % 5 else np.arange(length, dtype=np.float64)
        t = t.astype(dtype)
        window = float(rng.choice([0.5, 1.0, 2.0, rng.uniform(0.3, 4.0), float(t[-1] - t[0]) / rng.integers(1, 6)]))
        if trial % 3 == 0:
            tt = torch.from_numpy(t)
            pieces = int((((tt[-1] - tt[0]) / window).ceil()).item())
            ends = torch.linspace(tt[0], tt[0] + pieces * window, pieces + 1, dtype=tt.dtype).numpy()
            if pieces >= 2:
                end = float(ends[int(rng.integers(1, pieces))])
                k = int(np.clip(np.searchsorted(t, end), 1, length - 2))
                side = rng.choice([-1.0, 1.0])
                edge = (end - 1e-8) / (1 + 1e-5) if side < 0 else (end + 1e-8) / (1 - 1e-5)   # |end - v| = tol(v)
                v = dtype(edge)
                for _ in range(abs(int(rng.integers(-2, 3)))):
                    v = np.nextafter(v, dtype(np.inf if rng.random() < 0.5 else -np.inf))
                if t[k - 1] < v < t[k + 1]:
                    t[k] = v
        x = torch.zeros(1, length, 1, dtype=torch.from_numpy(t).dtype)
        del lengths[:]
        run(lambda: ref.logsig_windows(x, 1, window, torch.from_numpy(t)))
        key = "logsig_spy__{}__".format(n)
        out[key + "t"] = t
        out[key + "window"] = np.array(window)
        out[key + "lengths"] = np.array(lengths, dtype=np.int64)
        n += 1
    out["logsig_spy__count"] = np.array(n)
    return out


def main():
    ref = reference_loader.load_reference()
    out = {}
    out.update(diff_cases(ref))
    out.update(fresh_cases(ref))
    out.update(logsig_cases(ref))
    out.update(logsig_grad_cases(ref))
    out.update(logsig_spy_cases(ref))
    np.savez_compressed(OUT, **out)
    print("wrote {} arrays to {} ({} bytes)".format(len(out), OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
