"""The C dispatch of the MLP and linear fields keeps every verdict: which (entry point, hidden, channels, width, dtype,
solve variant, control kind, method, null or misaligned pointer, batch) it serves, refuses or rejects, with which message
for the linear field, where the MLP's shared-memory bounds lie, and what the scratch queries and the dopri5 grid answer,
against tests/golden/dispatch.npz (scripts/dispatch_fixture.py).  Every call returns before any launch, so no GPU is
needed."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "dispatch.npz")


def _generator():
    spec = importlib.util.spec_from_file_location("dispatch_fixture", os.path.join(ROOT, "scripts", "dispatch_fixture.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_dispatch_verdicts_match_the_fixture():
    want = np.load(FIXTURE)
    got = _generator().records()
    assert sorted(got) == sorted(want.files)
    # scratch sizes and the dopri5 grid scale with the SM count: exact values where it is the fixture's, served (>= 0)
    # or not elsewhere
    same_sms = int(got["sm_count"]) == int(want["sm_count"])
    bad = []
    for key in sorted(want.files):
        if key == "sm_count":
            continue
        a, b = got[key], want[key]
        if key.startswith(("bytes/", "grid/")) and not same_sms:
            a, b = np.sign(a), np.sign(b)
        if a.shape != b.shape or not np.array_equal(a, b):
            n = int((a != b).sum()) if a.shape == b.shape else "shape"
            bad.append("{}: {} of {} verdicts differ".format(key, n, b.size))
    assert not bad, "\n".join(bad)
