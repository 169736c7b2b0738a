"""oracle/logsig_oracle.py against mathematics that does not depend on any implementation (the package it stands in for,
signatory, is not installable offline): level 1 = total increment, level 2 = Levy areas, a straight line has nothing above
level 1, Chen's identity, invariance under re-sampling, and the number of Lyndon words (Witt's formula)."""
import numpy as np

from oracle import logsig_oracle as O


def test_level_one_and_levy_area():
    rng = np.random.default_rng(0)
    path = rng.standard_normal((7, 3))
    ls = O.logsignature(path, 2)
    words = O.lyndon_words(3, 2)
    assert words == [(0,), (1,), (2,), (0, 1), (0, 2), (1, 2)]
    assert np.allclose(ls[:3], path[-1] - path[0])
    x = path - path[0]
    dx = np.diff(path, axis=0)
    mid = 0.5 * (x[1:] + x[:-1])
    for q, (i, j) in enumerate(words[3:], 3):
        area = 0.5 * np.sum(mid[:, i] * dx[:, j] - mid[:, j] * dx[:, i])       # 1/2 int (x_i dx_j - x_j dx_i), exact for linear pieces
        assert np.isclose(ls[q], area)


def test_straight_line_and_resampling():
    rng = np.random.default_rng(1)
    a, b = rng.standard_normal(4), rng.standard_normal(4)
    line = np.stack([a + s * (b - a) for s in (0.0, 0.2, 0.7, 1.0)])
    ls = O.logsignature(line, 4)
    assert np.allclose(ls[:4], b - a) and np.allclose(ls[4:], 0.0, atol=1e-13)
    path = rng.standard_normal((5, 2))
    finer = np.concatenate([[path[0]], *[[0.5 * (path[i] + path[i + 1]), path[i + 1]] for i in range(4)]])
    assert np.allclose(O.logsignature(path, 4), O.logsignature(finer, 4))


def test_chen_identity_and_counts():
    rng = np.random.default_rng(2)
    path = rng.standard_normal((9, 2))
    whole = O.signature(path, 4)
    parts = O._mul(O.signature(path[:5], 4), O.signature(path[4:], 4), 4)
    for k in range(5):
        assert np.allclose(whole[k], parts[k])
    # Witt: number of Lyndon words of length n over c letters = (1/n) sum_{d | n} mu(d) c^(n/d)
    assert [len([w for w in O.lyndon_words(3, 4) if len(w) == n]) for n in (1, 2, 3, 4)] == [3, 3, 8, 18]
    from torchcde_b200.log_ode import lyndon_words, logsignature_channels
    for c, d in ((1, 3), (2, 5), (3, 4), (5, 2)):
        assert lyndon_words(c, d) == O.lyndon_words(c, d)
        assert logsignature_channels(c, d) == len(O.lyndon_words(c, d))


def test_window_knots_bookkeeping():
    """log_ode.py:18-40 as restated in torchcde_b200.log_ode._window_knots: the merged knot sequence stays sorted, every
    window end sits at the position it is given, end points that coincide with observation times are not duplicated, and
    the last window is clipped to the final time."""
    import math
    import random
    import torch
    from torchcde_b200.log_ode import _window_knots

    random.seed(1)
    torch.manual_seed(1)
    for trial in range(300):
        n = random.randint(2, 30)
        dtype = random.choice([torch.float32, torch.float64])
        t = torch.linspace(0, n - 1, n, dtype=dtype) if trial % 3 == 0 else (torch.rand(n, dtype=torch.float64) + 0.05).cumsum(0).to(dtype)
        wl = random.choice([0.5, 1.0, 2.0, float(t[-1] - t[0]) / random.randint(1, 5), random.uniform(0.3, 4.0)])
        ends, positions, extra = _window_knots(t, wl)
        # the last end is the linspace end clipped to the final time; it can round to just below it, and then it is
        # within torch.allclose of the final time and still names the last knot (positions[-1] below)
        last = t[0] + (ends.numel() - 1) * wl
        assert float(ends[0]) == float(t[0]) and float(ends[-1]) == min(float(last), float(t[-1]))
        assert torch.allclose(ends[-1], t[-1])
        assert ends.numel() == int(math.ceil(float((t[-1] - t[0]) / wl))) + 1 or ends.numel() == int((((t[-1] - t[0]) / wl).ceil()).item()) + 1
        merged = torch.cat([t] + extra).sort().values if extra else t
        assert all(b > a for a, b in zip(positions[:-1], positions[1:]))
        assert merged.numel() == n + len(extra) and positions[-1] == merged.numel() - 1
        for e, p in zip(ends.tolist(), positions):
            assert abs(float(merged[p]) - e) <= 1e-8 + 1e-5 * abs(e)


def test_jacobian_matches_central_differences_and_level_one():
    """The complex-step Jacobian against central differences, and level 1 (the total increment) is exactly -1 at the
    first point, +1 at the last and 0 in between, channel by channel."""
    rng = np.random.default_rng(3)
    for length, channels, depth in ((5, 2, 4), (3, 3, 3), (6, 1, 2), (2, 2, 5)):
        path = rng.standard_normal((length, channels))
        jac = O.logsignature_jacobian(path, depth)
        assert jac.shape == (len(O.lyndon_words(channels, depth)), length, channels)
        h = 1e-6
        num = np.zeros_like(jac)
        for p in range(length):
            for c in range(channels):
                e = np.zeros_like(path)
                e[p, c] = h
                num[:, p, c] = (O.logsignature(path + e, depth) - O.logsignature(path - e, depth)) / (2 * h)
        assert np.abs(jac - num).max() <= 1e-7 * max(1.0, np.abs(jac).max()), (length, channels, depth)
        level_one = np.zeros((channels, length, channels))
        for c in range(channels):
            level_one[c, 0, c], level_one[c, -1, c] = -1.0, 1.0
        assert np.array_equal(jac[:channels], level_one)
        real = O.logsignature(path, depth)
        assert np.allclose(O.logsignature(path.astype(complex), depth).real, real, rtol=1e-14, atol=1e-14)


def test_jacobian_agrees_with_chen_across_a_split_window():
    """The signature of a path is the product of the signatures of its two halves (Chen), so perturbing a point of the
    first half moves the whole path's logsignature as the chain rule through that product says.  The whole path's
    Jacobian at a point of the first half, pushed through the product by complex step on the first half alone, must
    agree with the Jacobian of the whole; at the point the halves share, both halves move."""
    rng = np.random.default_rng(4)
    depth = 4
    path = rng.standard_normal((7, 2))
    words = O.lyndon_words(2, depth)
    whole = O.logsignature_jacobian(path, depth)
    second = O.signature(path[3:], depth)
    h = 1e-30
    for p in range(3):
        for c in range(2):
            z = path[:4].astype(complex)
            z[p, c] += 1j * h
            log = O.log_tensor(O._mul(O.signature(z, depth), second, depth), depth)
            chen = np.array([log[len(w)][w] for w in words]).imag / h
            assert np.allclose(chen, whole[:, p, c], rtol=1e-12, atol=1e-12), (p, c)
    # the point shared by the halves: the second half's start moves too
    z = path.astype(complex)
    z[3, 0] += 1j * h
    log = O.log_tensor(O._mul(O.signature(z[:4], depth), O.signature(z[3:], depth), depth), depth)
    assert np.allclose(np.array([log[len(w)][w] for w in words]).imag / h, whole[:, 3, 0], rtol=1e-12, atol=1e-12)


def test_window_positions_match_the_reference_slices():
    """The window end positions of _window_knots against the lengths of the window slices the reference's own log_ode.py
    handed to signatory (tests/golden/reference_live.npz, oracle/make_reference_golden.py): random fp32 and fp64 ``t``,
    and ``t`` with a knot a few ulps either side of torch.allclose's tolerance of a window end, where the comparison has
    to be made in ``t``'s dtype."""
    import os
    import torch
    from torchcde_b200.log_ode import _window_knots

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz"))
    count = int(z["logsig_spy__count"])
    assert count >= 300
    for i in range(count):
        key = "logsig_spy__{}__".format(i)
        t = torch.from_numpy(z[key + "t"])
        lengths = z[key + "lengths"].tolist()
        _, positions, extra = _window_knots(t, float(z[key + "window"]))
        assert [b - a + 1 for a, b in zip(positions[:-1], positions[1:])] == lengths, (i, t.dtype)
        assert positions[0] == 0 and positions[-1] == t.numel() + len(extra) - 1
