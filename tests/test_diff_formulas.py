"""torchcde_b200/_diff.py (the torch-operator restatements that serve BACKWARD passes of the kernel-backed builders)
against the reference package: same values and the same gradients with respect to the data and the knots, with and
without missing values.  CPU, fp64.  The reference's values, cotangents and gradients are stored in
tests/golden/reference_live.npz (oracle/make_reference_golden.py)."""
import os

import numpy as np
import pytest
import torch

from torchcde_b200 import _diff

_Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz"))
_OURS = {"hermite": _diff.hermite, "natural1": lambda a, b: _diff.natural(a, b, 1), "natural0": lambda a, b: _diff.natural(a, b, 0),
         "linear": _diff.linear_fill}


def _t(key):
    return torch.from_numpy(_Z[key]) if key in _Z.files else None


def _cases(prefix):
    n = 0
    while prefix + "__{}__x".format(n) in _Z.files:
        yield prefix + "__{}__".format(n)
        n += 1


def _compare(ours, key):
    x, t = _t(key + "x"), _t(key + "t")
    want, cot = _t(key + "want"), _t(key + "cot")
    xa = x.clone().requires_grad_(True)
    ta = None if t is None else t.clone().requires_grad_(True)
    got = ours(xa, ta)
    assert got.shape == want.shape
    nan_same = torch.isnan(got) == torch.isnan(want)
    assert bool(nan_same.all())
    ok = ~torch.isnan(want)
    assert torch.allclose(got[ok], want[ok], rtol=1e-9, atol=1e-11), float((got[ok] - want[ok]).abs().max())
    if key + "gx" not in _Z.files:       # e.g. linear coefficients without NaN return their input
        return
    ins_a = [xa] + ([ta] if t is not None else [])
    ga = torch.autograd.grad(torch.where(ok, got, torch.zeros_like(got)), ins_a, cot, allow_unused=True)
    for a, name in zip(ga, ("gx", "gt")):
        b = _t(key + name)
        a = torch.zeros(1, dtype=torch.float64) if a is None else torch.nan_to_num(a)
        assert torch.allclose(a, b, rtol=1e-7, atol=1e-9), float((a - b).abs().max())


@pytest.mark.parametrize("nan", [0.0, 0.35])
@pytest.mark.parametrize("irregular", [False, True])
def test_builders_values_and_gradients_match_the_reference(nan, irregular):
    keys = [k for k in _cases("diff") if tuple(_Z[k + "group"]) == (nan, float(irregular))]
    assert len(keys) == (20 if nan else 12)
    for key in keys:
        builder = str(_Z[key + "builder"])
        if builder == "ffill":
            ff, mine = _t(key + "want"), _diff.forward_fill(_t(key + "x"))
            assert bool(((ff == mine) | (torch.isnan(ff) & torch.isnan(mine))).all()), key
        else:
            _compare(_OURS[builder], key)


def test_rectilinear_matches_the_reference():
    got = _diff.linear_fill(_diff.rectilinear(_t("rect__x"), 0), None)
    assert torch.allclose(got, _t("rect__want"))


def test_evaluation_formulas_match_the_reference():
    x, t, coeffs = _t("eval__x"), _t("eval__t"), _t("eval__coeffs")
    c = x.size(-1)
    a, b, two_c, three_d = coeffs[..., :c], coeffs[..., c:2 * c], coeffs[..., 2 * c:3 * c], coeffs[..., 3 * c:]
    for i in range(3):
        key = "eval__{}__".format(i)
        q, index, lindex = _t(key + "q"), _t(key + "index"), _t(key + "lindex")
        for deriv in (False, True):
            want = _t(key + ("cubic_deriv" if deriv else "cubic_eval"))
            got = _diff.cubic_eval(a, b, two_c, three_d, t, q, index, deriv)
            assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
            want = _t(key + ("linear_deriv" if deriv else "linear_eval"))
            got = _diff.linear_eval(x, t, q, lindex, deriv)
            assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
