"""``logsig_windows`` / ``logsignature_windows`` on every route, against the fp64 oracle (oracle/logsig_oracle.py) per
window and per level, and against the reference's own log_ode.py (tests/golden/reference_live.npz) in value and gradient.

Routes (every case records which one served it):
  1. the kernel ``tcde_logsignature_windows`` (csrc/logsig.cu), one thread per (path, window), no graph;
  2. the same kernel forward with the torch-operator backward ``log_ode._windows_formula`` (``_diff.KernelForward``) when
     ``x`` or ``t`` requires grad;
  3. ``_windows_formula`` forward and backward for the shapes the kernel refuses (channels > 16, depth > 6, or more than
     640 terms in levels 1..depth).

Per-window errors: consecutive output rows are differenced to recover each window's logsignature, and a level-k word's
error is measured against ``(window path length)^k / k!`` (the bound on a level-k term), so an error confined to a high
level is not hidden by the size of level 1.  Bars: 1e-12 (fp64) and 1e-5 (fp32) of that scale; a window of 200 or more
segments accumulates one rounding per segment and gets ``4 * n_segments * eps`` of its dtype instead."""
import math
import os

import numpy as np
import pytest
import torch

import torchcde_b200 as cde
from oracle import logsig_oracle as O
from torchcde_b200 import _lib, log_ode

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64 = torch.float32, torch.float64
BAR = {F32: 1e-5, F64: 1e-12}
EPS = {F32: float(np.finfo(np.float32).eps), F64: float(np.finfo(np.float64).eps)}
KERNEL = "tcde_logsignature_windows"
# (channels, depth) at and just inside the kernel's limits: channels <= 16, depth <= 6, C + ... + C^depth <= 640
SHAPES = [(16, 2), (8, 3), (4, 4), (3, 5), (2, 6), (1, 6), (16, 1)]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz")

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[log-ODE routes, worst per-window error per dtype and level] " + "; ".join(
        "{} level {}: {:.2e} (bar {:.1e})".format(dtype, level, e, bar) for (dtype, level, bar), e in sorted(_WORST.items())))


@pytest.fixture
def routes(monkeypatch):
    """Record, in order, every call of the log-ODE kernel (``<name>:refused`` when it refuses the shape) and of the torch
    formula, letting both run."""
    seen = []
    real_call, real_formula = _lib.call, log_ode._windows_formula

    def call(name, *args):
        if name != KERNEL:
            return real_call(name, *args)
        try:
            rc = real_call(name, *args)
        except NotImplementedError:
            seen.append(KERNEL + ":refused")
            raise
        seen.append(KERNEL)
        return rc

    def formula(*args):
        seen.append("formula")
        return real_formula(*args)

    monkeypatch.setattr(_lib, "call", call)
    monkeypatch.setattr(log_ode, "_windows_formula", formula)
    return seen


def _report(dtype, level, err, bar):
    key = ("fp32" if dtype == F32 else "fp64", level, bar)
    _WORST[key] = max(err, _WORST.get(key, 0.0))


def _windows_of(rows):
    """(..., 1 + W, words) cumsummed output -> (..., W, words) per-window logsignatures, in fp64."""
    rows = rows.detach().double().cpu()
    return (rows[..., 1:, :] - rows[..., :-1, :]).numpy()


def _check_window(got, path, depth, dtype, what, bar=None):
    """got: (words,) one window's logsignature; path: (points, C) fp64 the window's points.  Per-level bar."""
    want = O.logsignature(path, depth)
    words = O.lyndon_words(path.shape[1], depth)
    segments = path.shape[0] - 1
    length = float(np.linalg.norm(np.diff(path, axis=0), axis=1).sum())
    if bar is None:
        bar = 4 * segments * EPS[dtype] if segments >= 200 else BAR[dtype]
    levels = np.array([len(w) for w in words])
    for k in sorted(set(levels.tolist())):               # one channel has no words above level 1
        scale = max(length ** k / math.factorial(k), 1e-300)
        err = float(np.abs(got[levels == k] - want[levels == k]).max()) / scale
        _report(dtype, k, err, bar)
        assert err <= bar, (what, "level", k, err, bar)


def _grid_knots(segments, dtype):
    """Knots on [0, len(segments)] whose unit windows hold ``segments[w]`` segments each: the window ends are integers and
    fall on knots, so no knot is added and the windows are the slices between consecutive integer knots."""
    knots = [0.0]
    for w, n in enumerate(segments):
        knots += [w + (j + 1) / n for j in range(n)]
    return torch.tensor(knots, dtype=F64).to(dtype)


def _path(gen, n_paths, points, channels, step):
    """Random walks from the origin (row 0 of the output is then 0, so differencing rows loses nothing to it)."""
    inc = torch.randn(n_paths, points - 1, channels, generator=gen, dtype=F64) * step
    return torch.cat([torch.zeros(n_paths, 1, channels, dtype=F64), inc.cumsum(1)], dim=1)


# ------------------------------------------------------------------------------------- kernel vs oracle, per window
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("channels,depth", SHAPES)
def test_kernel_per_window_and_level(routes, channels, depth, dtype):
    """Windows of 1, 2, 7 and 200 segments, unit and 1e-3 increments."""
    gen = torch.Generator().manual_seed(100 * channels + depth)
    segments = [1, 2, 7, 200]
    t = _grid_knots(segments, dtype)
    bounds = np.cumsum([0] + segments)
    for step in (1.0, 1e-3):
        x = _path(gen, 2, t.numel(), channels, step).to(dtype)
        got = cde.logsig_windows(x.to(DEV), depth, 1.0, t.to(DEV))
        assert got.shape == (2, len(segments) + 1, log_ode.logsignature_channels(channels, depth))
        assert got.grad_fn is None
        sigs = _windows_of(got)
        xd = x.double().numpy()
        for p in range(2):
            for w, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
                _check_window(sigs[p, w], xd[p, lo:hi + 1], depth, dtype, (channels, depth, step, p, segments[w]))
    assert routes == [KERNEL] * 2


@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("n_paths,n_windows", [(1, 1), (1, 127), (2, 64), (3, 43), (600, 110)],
                         ids=["items1", "items127", "items128", "items129", "items66000"])
def test_kernel_across_the_thread_blocks(routes, n_paths, n_windows, dtype):
    """(path, window) counts around the 128-thread block and over 65,536: windows of 3 segments at (3, 3).  Every window
    against the torch formula in fp64; the first and last windows, both sides of every block boundary up to the third,
    and a random sample against the oracle."""
    channels, depth = 3, 3
    gen = torch.Generator().manual_seed(n_paths * 1000 + n_windows)
    x = _path(gen, n_paths, 3 * n_windows + 1, channels, 0.5).to(dtype)
    got = cde.logsig_windows(x.to(DEV), depth, 3.0)
    assert routes == [KERNEL]
    sigs = _windows_of(got).reshape(n_paths * n_windows, -1)
    xd = x.double()
    table = log_ode._word_table(channels, depth)
    formula = log_ode._windows_formula(xd.to(DEV), list(range(0, 3 * n_windows + 1, 3)), depth, table)
    full = np.abs(sigs - formula.reshape(n_paths * n_windows, -1).cpu().numpy()).max()
    assert full <= 50 * BAR[dtype], full
    items = n_paths * n_windows
    sample = {0, items - 1} | {i for b in (127, 128, 255, 256, 383, 384) for i in (b - 1, b) if i < items}
    sample |= set(np.random.default_rng(items).integers(0, items, size=min(items, 40)).tolist())
    for i in sorted(sample):
        p, w = divmod(i, n_windows)
        _check_window(sigs[i], xd[p, 3 * w:3 * w + 4].numpy(), depth, dtype, (n_paths, n_windows, i))


# --------------------------------------------------------------------------- whole transform vs the reference's code
def _reference_cases():
    z = np.load(GOLDEN)
    n = 0
    while "logsig_grad__{}__x".format(n) in z.files:
        n += 1
    return z, n


@pytest.mark.parametrize("case", range(8))
def test_whole_transform_and_gradients_against_the_reference(routes, case):
    """Values of logsig_windows and logsignature_windows (values and times) and their gradients in x and t against the
    reference's log_ode.py run with the oracle (and its Jacobian) as signatory: regular, irregular and default t, NaN
    holes in the first and last rows, a window end just inside and just outside torch.allclose of an observation, batch
    dimensions (2, 3), depths 1 to 4."""
    z, n = _reference_cases()
    assert n == 8
    key = "logsig_grad__{}__".format(case)
    x = torch.from_numpy(z[key + "x"])
    depth, window = int(z[key + "depth"]), float(z[key + "window"])
    t = torch.from_numpy(z[key + "t"]) if key + "t" in z.files else None
    for name in ("logsig", "logsignature"):
        prefix = key + name + "__"
        xb = x.to(DEV).requires_grad_(True)
        tb = None if t is None else t.to(DEV).requires_grad_(True)
        outs = (cde.logsig_windows(xb, depth, window, tb),) if name == "logsig" else \
            cde.logsignature_windows(xb, depth, window, tb)
        fields = ("want", "want_t")[:len(outs)]
        cots = ("cot", "cot_t")[:len(outs)]
        for out, field in zip(outs, fields):
            want = torch.from_numpy(z[prefix + field])
            assert out.shape == want.shape and out.dtype == want.dtype, (name, field)
            assert torch.allclose(out.detach().cpu(), want, rtol=1e-9, atol=1e-12), (name, field)
        live = [(o, torch.from_numpy(z[prefix + c]).to(DEV)) for o, c in zip(outs, cots) if o.requires_grad]
        ins = [xb] + ([tb] if tb is not None else [])
        grads = torch.autograd.grad([o for o, _ in live], ins, [c for _, c in live], allow_unused=True)
        for g, field, like in zip(grads, ("gx", "gt"), ins):
            got = torch.zeros_like(like) if g is None else g
            want = torch.from_numpy(z[prefix + field])
            scale = max(1.0, float(want.abs().max()))
            assert torch.allclose(got.cpu(), want, rtol=1e-9, atol=1e-12 * scale), (name, field)
    assert routes == [KERNEL, "formula"] * 2


# ----------------------------------------------------------------------------------- gradient in x vs the Jacobian
def _jacobian_grad(x, segments, depth, cot):
    """The gradient of <logsig_windows(x), cot> from the oracle's Jacobian: x (points, C) fp64 on unit windows of
    ``segments``; cot (1 + W, words).  Row w of the output is x[0] (level 1) plus the sum of windows 1..w."""
    channels = x.shape[1]
    per_window = np.flip(np.cumsum(np.flip(cot[1:], 0), 0), 0)        # d<out, cot>/d(window w) = sum of rows >= w
    grad = np.zeros_like(x)
    grad[0] += cot[:, :channels].sum(0)
    lo = 0
    for w, n in enumerate(segments):
        jac = O.logsignature_jacobian(x[lo:lo + n + 1], depth)
        grad[lo:lo + n + 1] += np.einsum("q,qlc->lc", per_window[w], jac)
        lo += n
    return grad


@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("channels,depth", SHAPES)
def test_gradient_in_x_against_the_jacobian(routes, channels, depth, dtype):
    """The forward grid's windows of 1, 2 and 7 segments (11 points), unit and 1e-3 increments."""
    gen = torch.Generator().manual_seed(7 * channels + depth)
    segments = [1, 2, 7]
    t = _grid_knots(segments, dtype).to(DEV)
    for step in (1.0, 1e-3):
        x = _path(gen, 1, t.numel(), channels, step)
        xb = x.to(dtype).to(DEV).requires_grad_(True)
        out = cde.logsig_windows(xb, depth, 1.0, t)
        cot = torch.randn(out.shape, generator=gen, dtype=F64)
        got, = torch.autograd.grad(out, xb, cot.to(dtype).to(DEV))
        want = _jacobian_grad(xb.detach().double().cpu()[0].numpy(), segments, depth, cot.to(dtype).double()[0].numpy())
        scale = max(1.0, float(np.abs(want).max()))
        err = float(np.abs(got.double().cpu()[0].numpy() - want).max()) / scale
        assert err <= (1e-12 if dtype == F64 else 1e-5), (channels, depth, step, err)
    assert routes == [KERNEL, "formula"] * 2


def test_gradcheck_and_no_graph_without_grad():
    """torch.autograd.gradcheck in fp64 through both functions (x and t; window ends between observations, so the
    fill of the added knots is differentiated too), and no KernelForward node when nothing requires grad."""
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 5, 2, generator=gen, dtype=F64).to(DEV).requires_grad_(True)
    t = (torch.rand(5, generator=gen, dtype=F64) + 0.4).cumsum(0).to(DEV).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda xx: cde.logsig_windows(xx, 3, 1.3), (x,))
    # t[0] also places the window ends through linspace, which (as in the reference) carries no gradient: hold it fixed
    t0, rest = t[:1].detach(), t[1:].detach().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda xx, tt: cde.logsignature_windows(xx, 2, 0.9, torch.cat([t0, tt])), (x, rest))

    def names(fn):
        seen, stack = set(), [fn]
        while stack:
            node = stack.pop()
            if node is not None and node not in seen:
                seen.add(node)
                stack += [f for f, _ in node.next_functions]
        return {type(node).__name__ for node in seen}

    assert "KernelForwardBackward" in names(cde.logsig_windows(x, 3, 1.3).grad_fn)
    assert cde.logsig_windows(x.detach(), 3, 1.3).grad_fn is None
    with torch.no_grad():
        assert cde.logsig_windows(x, 3, 1.3).grad_fn is None
    values, times = cde.logsignature_windows(x.detach(), 2, 0.9, t.detach())
    assert t.requires_grad and cde.logsignature_windows(x.detach(), 2, 0.9, t)[1].grad_fn is not None
    assert values.grad_fn is None and times.grad_fn is None


# ------------------------------------------------------------------------------------------------------------ edges
def _transform_oracle(x, t, depth, window):
    """The whole transform in fp64 on the host for x without NaNs: ends as torch builds them, every end that is not within
    torch.allclose of an observation becomes a knot filled linearly, the oracle on every window, rows cumsummed; plus the
    end points.  x (..., L, C) fp64, t (L,) any float dtype."""
    knots = t.double().numpy()
    ends_t, positions, extra = log_ode._window_knots(t.cpu(), window)
    merged = np.sort(np.concatenate([knots] + [e.detach().double().numpy() for e in extra]))
    flat = x.reshape(-1, x.shape[-2], x.shape[-1]).numpy()
    filled = np.stack([np.stack([np.interp(merged, knots, p[:, c]) for c in range(p.shape[1])], 1) for p in flat])
    words = len(O.lyndon_words(x.shape[-1], depth))
    rows = np.zeros((flat.shape[0], len(positions), words))
    rows[:, 0, :x.shape[-1]] = filled[:, 0]
    for w, (lo, hi) in enumerate(zip(positions[:-1], positions[1:])):
        rows[:, w + 1] = [O.logsignature(p[lo:hi + 1], depth) for p in filled]
    return rows.cumsum(1), ends_t.detach().double().numpy(), positions, filled


def _check_rows(got, want, dtype, what):
    """Per-window comparison of cumsummed outputs, bar relative to each window's own scale (max 1)."""
    gw, ww = _windows_of(got), want[..., 1:, :] - want[..., :-1, :]
    scale = np.maximum(np.abs(ww).max(-1, keepdims=True), 1.0)
    err = float((np.abs(gw - ww.reshape(gw.shape)) / scale.reshape(*gw.shape[:-1], 1)).max()) if gw.size else 0.0
    assert err <= 10 * BAR[dtype], (what, err)
    first = got.detach().double().cpu().numpy()[..., 0, :]
    assert np.abs(first - want[..., 0, :].reshape(first.shape)).max() <= BAR[dtype] * max(1.0, np.abs(want).max())


def test_empty_batch_and_nested_batch_dimensions(routes):
    x = torch.zeros(0, 6, 2, dtype=F64, device=DEV)
    got = cde.logsig_windows(x, 3, 2.0)
    assert got.shape == (0, 4, 5)
    values, times = cde.logsignature_windows(torch.zeros(2, 0, 6, 2, dtype=F32, device=DEV), 2, 2.5)
    assert values.shape == (2, 0, 3, 3) and values.dtype == F32 and times.tolist() == [0.0, 2.5, 5.0]
    assert cde.logsig_windows(torch.zeros(0, 6, 17, dtype=F64, device=DEV), 1, 2.0).shape == (0, 4, 17)
    assert routes == []
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(2, 3, 9, 2, generator=gen, dtype=F64)
    t = (torch.rand(9, generator=gen, dtype=F64) + 0.2).cumsum(0)
    got = cde.logsig_windows(x.to(DEV), 3, 1.1, t.to(DEV))
    want, _, _, _ = _transform_oracle(x, t, 3, 1.1)
    assert got.shape == (2, 3) + want.shape[1:]
    _check_rows(got, want.reshape(got.shape), F64, "nested")
    assert routes == [KERNEL]


def test_non_contiguous_x_and_fp32_x_with_fp64_t(routes):
    gen = torch.Generator().manual_seed(10)
    base = torch.randn(8, 3, 2, generator=gen, dtype=F64).to(DEV)          # (L, paths, C): x = base.transpose(0, 1)
    x = base.transpose(0, 1)
    assert not x.is_contiguous()
    assert torch.equal(cde.logsig_windows(x, 4, 2.0), cde.logsig_windows(x.contiguous(), 4, 2.0))
    xb = x.detach().requires_grad_(True)
    g1, = torch.autograd.grad(cde.logsig_windows(xb, 4, 2.0).sum(), xb)
    xc = x.contiguous().requires_grad_(True)
    g2, = torch.autograd.grad(cde.logsig_windows(xc, 4, 2.0).sum(), xc)
    assert torch.allclose(g1, g2, rtol=1e-14, atol=1e-14)
    t = (torch.rand(8, generator=gen, dtype=F64) + 0.25).cumsum(0)
    x32 = torch.randn(3, 8, 2, generator=gen, dtype=F64).float()
    values, times = cde.logsignature_windows(x32.to(DEV), 3, 0.7, t.to(DEV))
    assert values.dtype == F32 and times.dtype == F64
    rows, ends, positions, _ = _transform_oracle(x32.double(), t, 3, 0.7)
    assert np.array_equal(times.cpu().numpy(), ends)
    widths = np.diff(ends).astype(np.float32).astype(np.float64)
    sig = rows[:, 1:] - rows[:, :-1]
    want = np.concatenate([rows[:, :1], sig * widths[:, None]], 1).cumsum(1)
    _check_rows(values, want, F32, "fp32 x, fp64 t")


def test_logsignature_windows_scaling(routes):
    """Each window's logsignature times its width (the last window clipped to the final time), cumsummed, and the end
    points returned as the times."""
    gen = torch.Generator().manual_seed(11)
    x = torch.randn(2, 10, 3, generator=gen, dtype=F64)
    t = (torch.rand(10, generator=gen, dtype=F64) + 0.5).cumsum(0)
    values, times = cde.logsignature_windows(x.to(DEV), 3, 1.6, t.to(DEV))
    rows, ends, _, _ = _transform_oracle(x, t, 3, 1.6)
    assert ends[-1] == float(t[-1]) and np.diff(ends)[-1] < 1.6
    assert np.array_equal(times.cpu().numpy(), ends)
    sig = rows[:, 1:] - rows[:, :-1]
    want = np.concatenate([rows[:, :1], sig * np.diff(ends)[:, None]], 1).cumsum(1)
    _check_rows(values, want, F64, "scaling")
    plain = cde.logsig_windows(x.to(DEV), 3, 1.6, t.to(DEV))
    _check_rows(plain, rows, F64, "unscaled")
    assert routes == [KERNEL] * 2


@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("channels,depth", [(5, 4), (17, 1), (2, 7)])
def test_refused_shapes_run_the_formula(routes, channels, depth, dtype):
    """Shapes beyond the kernel (780 terms, 17 channels, depth 7): the kernel refuses them and the torch formula serves
    the forward and the backward, against the oracle and its Jacobian.  In fp32 at depth 7 the logarithm's powers of the
    signature, up to 7! times a level-7 term, round visibly at that level: its bar is 1e-4 (measured 4.9e-5 on an H100)."""
    gen = torch.Generator().manual_seed(channels * 10 + depth)
    segments = [1, 2, 7]
    t = _grid_knots(segments, dtype)
    x = _path(gen, 2, t.numel(), channels, 0.7).to(dtype)
    got = cde.logsig_windows(x.to(DEV), depth, 1.0, t.to(DEV))
    assert routes == [KERNEL + ":refused", "formula"]
    sigs = _windows_of(got)
    bounds = np.cumsum([0] + segments)
    for p in range(2):
        for w, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
            _check_window(sigs[p, w], x.double()[p, lo:hi + 1].numpy(), depth, dtype, (channels, depth, p, w),
                          bar=1e-4 if dtype == F32 and depth > 6 else None)
    if dtype == F64:
        xb = x[:1].to(DEV).requires_grad_(True)
        out = cde.logsig_windows(xb, depth, 1.0, t.to(DEV))
        cot = torch.randn(out.shape, generator=gen, dtype=F64)
        got, = torch.autograd.grad(out, xb, cot.to(DEV))
        want = _jacobian_grad(x[0].double().numpy(), segments, depth, cot[0].numpy())
        assert np.abs(got[0].cpu().numpy() - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    with pytest.raises(NotImplementedError):                # other refusals still raise: a dtype without a kernel
        cde.logsig_windows(x.to(DEV).half(), depth, 1.0)
