"""CPU restatement of the torchcde hot path -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Everything here is plain ``torch`` CPU arithmetic in the dtype of the inputs, written so
that every floating-point operation happens in the same order as in the reference (no
fused multiply-add anywhere: each torch elementwise op rounds once), which is what lets
``tests/`` demand bit-equality for path (i).  Citations are to the reference repository.

Pinning: ``tests/test_oracle_pinned.py`` checks each function below bit-for-bit against the
committed fixtures in ``tests/golden/`` (generated from the live reference by
``oracle/make_golden.py``) and, against the live
reference again.  The solve (``cdeint_linear``) is pinned for its vector field only; its
time stepping is ``oracle/odeint_port.py`` -- see that file's header for "parity unpinned".
"""
import torch

from . import odeint_port


# ----------------------------------------------------------------------------- helpers
def knot_times(length, dtype, device="cpu"):
    """Default knots 0, 1, ..., length-1  (misc.py:79-80)."""
    return torch.linspace(0, length - 1, length, dtype=dtype, device=device)


def check_path(x, t):
    """Input validation of misc.py:70-100 (same exception type and wording)."""
    if not x.is_floating_point():
        raise ValueError("X must both be floating point.")
    if x.ndimension() < 2:
        raise ValueError("X must have at least two dimensions, corresponding to time and channels. It instead has "
                         "shape {}.".format(tuple(x.shape)))
    if t is None:
        t = knot_times(x.size(-2), x.dtype, x.device)
    if not t.is_floating_point():
        raise ValueError("t must both be floating point.")
    if t.dim() != 1:
        raise ValueError("t must be one dimensional. It instead has shape {}.".format(tuple(t.shape)))
    if t.numel() > 1 and not bool((t[1:] > t[:-1]).all()):
        raise ValueError("t must be monotonically increasing.")
    if x.size(-2) != t.size(0):
        raise ValueError("The time dimension of X must equal the length of t. X has shape {} and t has shape {}, "
                         "corresponding to time dimensions of {} and {} respectively."
                         .format(tuple(x.shape), tuple(t.shape), x.size(-2), t.size(0)))
    if t.size(0) < 2:
        raise ValueError("Must have a time dimension of size at least 2. It instead has shape {}, corresponding to a "
                         "time dimension of size {}.".format(tuple(t.shape), t.size(0)))
    return t


def _observed_neighbours(valid):
    """For a (..., L, C) boolean mask: index of the nearest observation at-or-before and
    at-or-after every position (-1 / L where there is none)."""
    length = valid.size(-2)
    pos = torch.arange(length).view(length, 1).expand_as(valid)
    before = torch.where(valid, pos, torch.full_like(pos, -1)).cummax(dim=-2).values
    after = torch.where(valid, pos, torch.full_like(pos, length)).flip(-2).cummin(dim=-2).values.flip(-2)
    return before, after


# ------------------------------------------------------------- linear knots / NaN handling
def fill_gaps_linear(x, t=None):
    """``linear_interpolation_coeffs`` without ``rectilinear`` (interpolation_linear.py:13-84,
    :165-171), vectorised over every scalar series instead of recursing one at a time.

    Per series: all-NaN -> zeros (:19-21); a missing first / last entry takes the first /
    last observation (:31-34); every other missing entry is interpolated *in time* between
    the nearest observations either side, as ``prev + ratio * (next - prev)`` with
    ``ratio = (t - t_prev) / (t_next - t_prev)`` (:60-69).  No NaN at all -> the input
    object itself is returned (:169-171).
    """
    t = check_path(x, t)
    missing = torch.isnan(x)
    if not bool(missing.any()):
        return x
    length = x.size(-2)
    valid = ~missing
    before, after = _observed_neighbours(valid)
    seen = valid.any(dim=-2, keepdim=True)
    first = after[..., :1, :].clamp(max=length - 1)
    last = before[..., -1:, :].clamp(min=0)

    y = x.clone()
    y[..., :1, :] = torch.where(missing[..., :1, :], x.gather(-2, first), x[..., :1, :])
    y[..., -1:, :] = torch.where(missing[..., -1:, :], x.gather(-2, last), x[..., -1:, :])

    hole = torch.isnan(y)
    before, after = _observed_neighbours(~hole)
    lo = before.clamp(min=0)
    hi = after.clamp(max=length - 1)
    y_lo = y.gather(-2, lo)
    y_hi = y.gather(-2, hi)
    t_here = t.view(length, 1).expand_as(y)
    t_lo = t[lo]
    t_hi = t[hi]
    ratio = (t_here - t_lo) / (t_hi - t_lo)
    filled = y_lo + ratio * (y_hi - y_lo)
    y = torch.where(hole, filled, y)
    return torch.where(seen, y, torch.zeros_like(y))


def carry_forward(x, dim=-2):
    """``misc.forward_fill`` (misc.py:103-126): each entry takes the most recent observation
    along ``dim``; entries before the first observation stay NaN (index 0 is gathered)."""
    missing = torch.isnan(x)
    if not bool(missing.any()):
        return x
    xm = x.movedim(dim, -1)
    mm = missing.movedim(dim, -1)
    pos = torch.arange(xm.size(-1)).expand_as(xm)
    src = torch.where(mm, torch.zeros_like(pos), pos).cummax(dim=-1).values
    return xm.gather(-1, src).movedim(-1, dim)


def rectilinear_knots(x, time_index):
    """``_prepare_rectilinear_interpolation`` (interpolation_linear.py:87-128): carry values
    forward, double every row, and advance the time channel by one row -> length 2L-1."""
    channels = x.size(-1)
    assert isinstance(time_index, int), \
        "Index of the time channel must be an integer in [0, {}]".format(channels - 1)
    assert 0 <= time_index < channels, \
        "Time index must be in [0, {}], was given {}.".format(channels - 1, time_index)
    assert not bool(torch.isnan(x[..., time_index]).any()), \
        "There exist nan values in the time column which is not allowed."
    held = carry_forward(x)
    length = x.size(-2)
    out = torch.empty(*x.shape[:-2], 2 * length - 1, channels, dtype=x.dtype)
    out[..., 0::2, :] = held
    out[..., 1::2, :] = held[..., :-1, :]
    out[..., 1::2, time_index] = held[..., 1:, time_index]
    return out


def linear_knots(x, t=None, rectilinear=None):
    """``linear_interpolation_coeffs`` (interpolation_linear.py:131-171)."""
    if rectilinear is not None:
        x = rectilinear_knots(x, rectilinear)
    return fill_gaps_linear(x, t)


# ------------------------------------------------------------------ Hermite (backward diff)
def hermite_backward_difference_coeffs(x, t=None):
    """``hermite_cubic_coefficients_with_backward_differences``
    (interpolation_hermite_cubic_bdiff.py:5-44).  Row i of the result is
    ``[a | b | 2c | 3d]`` for interval i with the slope at knot i taken as the backward
    difference (the first slope repeated, so interval 0 is exactly linear)."""
    knots = fill_gaps_linear(x, t)
    if t is None:
        t = knot_times(knots.size(-2), knots.dtype)
    lo = knots[..., :-1, :]
    hi = knots[..., 1:, :]
    dt = (t[1:] - t[:-1]).unsqueeze(-1)
    slope_next = (hi - lo) / dt                                             # :39
    slope_prev = torch.cat((slope_next[..., :1, :], slope_next[..., :-1, :]), dim=-2)   # :10
    rise = hi - lo
    b = slope_prev
    two_c = 2 * (3 * (rise / dt - b) - slope_next + slope_prev) / dt        # :17
    three_d = (1 / dt ** 2) * (slope_next - b) - two_c / dt                 # :18
    return torch.cat([lo, b, two_c, three_d], dim=-1)                       # :19


# --------------------------------------------------------------------- natural cubic spline
def thomas_shared(rhs, upper, diag, lower):
    """Thomas algorithm of misc.py:13-67 for a system whose three diagonals are 1-D and
    shared by every series in ``rhs`` (..., k).  The eliminated diagonal and the
    multipliers depend only on the diagonals, so they are formed once (the reference
    broadcasts them to the batch and recomputes identical numbers per series)."""
    k = rhs.size(-1)
    new_diag = [diag[0]]
    mult = [None]
    for i in range(1, k):
        w = lower[i - 1] / new_diag[i - 1]
        mult.append(w)
        new_diag.append(diag[i] - w * upper[i - 1])
    fwd = [rhs[..., 0]]
    for i in range(1, k):
        fwd.append(rhs[..., i] - mult[i] * fwd[i - 1])
    sol = [None] * k
    sol[k - 1] = fwd[k - 1] / new_diag[k - 1]
    for i in range(k - 2, -1, -1):
        sol[i] = (fwd[i] - upper[i] * sol[i + 1]) / new_diag[i]
    return torch.stack(sol, dim=-1)


def natural_cubic_rows(t, x):
    """``_natural_cubic_spline_coeffs_without_missing_values`` (interpolation_cubic.py:7-53)
    for ``x`` of shape (..., length) (channels already moved to a batch dim)."""
    length = x.size(-1)
    if length == 2:
        a = x[..., :1]
        b = (x[..., 1:] - x[..., :1]) / (t[..., 1:] - t[..., :1])
        zero = torch.zeros(*x.shape[:-1], 1, dtype=x.dtype)
        return a, b, zero, zero.clone()
    rdt = (t[1:] - t[:-1]).reciprocal()
    rdt2 = rdt ** 2
    three_rise = 3 * (x[..., 1:] - x[..., :-1])
    six_rise = 2 * three_rise
    scaled = three_rise * rdt2
    diag = torch.empty(length, dtype=x.dtype)
    diag[:-1] = rdt
    diag[-1] = 0
    diag[1:] += rdt
    diag *= 2
    rhs = torch.empty_like(x)
    rhs[..., :-1] = scaled
    rhs[..., -1] = 0
    rhs[..., 1:] += scaled
    slope = thomas_shared(rhs, rdt, diag, rdt)
    a = x[..., :-1]
    b = slope[..., :-1]
    two_c = (six_rise * rdt - 4 * slope[..., :-1] - 2 * slope[..., 1:]) * rdt
    three_d = (-six_rise * rdt + 3 * (slope[..., :-1] + slope[..., 1:])) * rdt2
    return a, b, two_c, three_d


def _natural_cubic_series_with_gaps(t, x, version):
    """One scalar series with NaNs (interpolation_cubic.py:78-167).  Returns four (L-1,) rows."""
    length = x.size(0)
    seen = ~torch.isnan(x)
    if not bool(seen.any()):
        z = torch.zeros(length - 1, dtype=x.dtype)
        return z, z.clone(), z.clone(), z.clone()
    where = torch.nonzero(seen).flatten()
    first, last = int(where[0]), int(where[-1])
    x = x.clone()
    if version == 0:                      # :101-118  copy the first/last observation to the ends
        if not seen[0]:
            x[0] = x[first]
        if not seen[-1]:
            x[-1] = x[last]
    else:                                 # :119-131  fill backward / forward from them
        x[:first] = x[first]
        x[last + 1:] = x[last]
    seen = ~torch.isnan(x)
    tk = t[seen]
    xk = x[seen]
    pa, pb, pc, pd = natural_cubic_rows(tk, xk)
    # :147-162  re-expand piece p (anchored at tk[p]) about every original knot t[i] inside it
    piece = (seen.cumsum(0) - 1)[:-1].clamp(max=tk.numel() - 2)
    offset = tk[piece] - t[:-1]
    pa, pb, pc, pd = pa[piece], pb[piece], pc[piece], pd[piece]
    inner = (0.5 * pc - pd * offset / 3) * offset
    a = pa + (inner - pb) * offset
    b = pb + (pd * offset - pc) * offset
    two_c = pc - 2 * pd * offset
    return a, b, two_c, pd


def natural_cubic_coeffs(x, t=None, version=1):
    """``natural_cubic_coeffs`` (version=1) / ``natural_cubic_spline_coeffs`` (version=0)
    (interpolation_cubic.py:173-265)."""
    t = check_path(x, t)
    xt = x.transpose(-1, -2)
    if bool(torch.isnan(x).any()):
        flat = xt.reshape(-1, xt.size(-1))
        rows = [_natural_cubic_series_with_gaps(t, s, version) for s in flat]
        a, b, two_c, three_d = (torch.stack([r[j] for r in rows]).reshape(*xt.shape[:-1], -1) for j in range(4))
    else:
        a, b, two_c, three_d = natural_cubic_rows(t, xt)
    return torch.cat([a.transpose(-1, -2), b.transpose(-1, -2),
                      two_c.transpose(-1, -2), three_d.transpose(-1, -2)], dim=-1)


# ------------------------------------------------------------------------- spline evaluation
def locate(knots, t, n_intervals):
    """``_interpret_t`` (interpolation_cubic.py:315-322, interpolation_linear.py:203-210):
    interval index = clamp(#knots strictly below t  - 1, 0, n_intervals-1); a knot t_n
    (n > 0) therefore belongs to interval n-1.  Returns (fraction, int64 index)."""
    t = torch.as_tensor(t, dtype=knots.dtype)
    index = (torch.bucketize(t, knots) - 1).clamp(0, n_intervals - 1)
    return t - knots[index], index


def cubic_parts(coeffs):
    c = coeffs.size(-1) // 4
    if c * 4 != coeffs.size(-1):
        raise ValueError("Passed invalid coeffs.")
    return coeffs[..., :c], coeffs[..., c:2 * c], coeffs[..., 2 * c:3 * c], coeffs[..., 3 * c:]


def cubic_derivative(coeffs, knots, t):
    """``CubicSpline.derivative`` (interpolation_cubic.py:331-336)."""
    _, b, two_c, three_d = cubic_parts(coeffs)
    frac, index = locate(knots, t, coeffs.size(-2))
    frac = frac.unsqueeze(-1)
    inner = two_c[..., index, :] + three_d[..., index, :] * frac
    return b[..., index, :] + inner * frac


def cubic_evaluate(coeffs, knots, t):
    """``CubicSpline.evaluate`` (interpolation_cubic.py:324-329)."""
    a, b, two_c, three_d = cubic_parts(coeffs)
    frac, index = locate(knots, t, coeffs.size(-2))
    frac = frac.unsqueeze(-1)
    inner = 0.5 * two_c[..., index, :] + three_d[..., index, :] * frac / 3
    inner = b[..., index, :] + inner * frac
    return a[..., index, :] + inner * frac


def linear_slopes(knots_x, knots_t):
    """``LinearInterpolation.__init__`` slopes (interpolation_linear.py:189)."""
    return (knots_x[..., 1:, :] - knots_x[..., :-1, :]) / (knots_t[1:] - knots_t[:-1]).unsqueeze(-1)


def linear_derivative(knots_x, knots_t, t):
    """``LinearInterpolation.derivative`` (interpolation_linear.py:222-225)."""
    slopes = linear_slopes(knots_x, knots_t)
    _, index = locate(knots_t, t, slopes.size(-2))
    return slopes[..., index, :]


def linear_evaluate(knots_x, knots_t, t):
    """``LinearInterpolation.evaluate`` (interpolation_linear.py:212-220)."""
    frac, index = locate(knots_t, t, knots_x.size(-2) - 1)
    frac = frac.unsqueeze(-1)
    lo = knots_x[..., index, :]
    hi = knots_x[..., index + 1, :]
    width = knots_t[index + 1] - knots_t[index]
    return lo + frac * (hi - lo) / width.unsqueeze(-1)


# ------------------------------------------------------------------------------- the solve
def linear_field(weight, bias, z, dxdt):
    """README-form vector field contracted with dX/dt:
    ``Linear(H, H*C)(z).view(..., H, C) @ dXdt`` (README.md:42-49 + solver.py:126-130)."""
    hidden = z.size(-1)
    system = torch.nn.functional.linear(z, weight, bias).view(*z.shape[:-1], hidden, -1)
    return (system @ dxdt.unsqueeze(-1)).squeeze(-1)


def cdeint_linear(control, knots, weight, bias, z0, t, method="rk4", step_size=None, kind="cubic"):
    """``cdeint(X, func, z0, t, adjoint=False, method=..., options={'step_size': ...})`` for a
    ``CubicSpline`` (kind='cubic', ``control`` = coeffs) or ``LinearInterpolation``
    (kind='linear', ``control`` = knot values) and the README linear ``func``.
    Returns (..., len(t), H) like solver.py:234-236."""
    if kind == "cubic":
        def dxdt(s):
            return cubic_derivative(control, knots, s)
    elif kind == "linear":
        def dxdt(s):
            return linear_derivative(control, knots, s)
    else:
        raise ValueError(kind)

    def field(s, z):
        return linear_field(weight, bias, z, dxdt(s))

    options = {} if step_size is None else {"step_size": step_size}
    out = odeint_port.odeint(field, z0, t, method=method, options=options)
    dims = range(1, out.dim() - 1)
    return out.permute(*dims, 0, -1)
