"""The fused 2xFP16 tensor-core solve keeps its output bits: cdeint_wgmma_kernel's forward (rk4, midpoint, euler; cubic
and linear control; schedules F1-F8), its stage dump, the Runge-Kutta backward's dL/dz0 and kappa dump, and reversible
Heun's forward and checkpointed backward, against tests/golden/fused_solve_bits.npz (scripts/fused_solve_fixture.py).
A change of the kernels' layout or instruction order must leave every bit, the sign of zeros included, where it was."""
import importlib.util
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "fused_solve_bits.npz")

pytestmark = pytest.mark.gpu


def _generator():
    spec = importlib.util.spec_from_file_location("fused_solve_fixture",
                                                  os.path.join(ROOT, "scripts", "fused_solve_fixture.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_fused_solve_bits_match_the_fixture():
    gen = _generator()
    want = np.load(FIXTURE)
    got = gen.compute(torch.device("cuda:0"))
    names = sorted({k.split("#")[0] for k in want.files})
    assert sorted(got) == names
    bad = []
    for name in names:
        a = got[name]
        sample, ref = gen.sample(a).view(np.int32), want[name + "#sample"].view(np.int32)
        if not np.array_equal(gen.digest(a), want[name + "#sha256"]) or not np.array_equal(sample, ref):
            bad.append("{}: bits differ; {} of the {} sampled values".format(name, int((sample != ref).sum()), ref.size))
    assert not bad, "\n".join(bad)
