"""``logsig_windows`` / ``logsignature_windows`` -- the log-ODE preprocessing transform (reference torchcde/log_ode.py:15-133).

Same arguments, window construction, NaN handling and return values as the reference.  The reference computes each
window's logsignature with the optional third-party package ``signatory`` (log_ode.py:1-8, :56-58) in a Python loop over
the windows; here all windows of all paths are ONE launch of ``tcde_logsignature_windows`` (csrc/logsig.cu), which restates
what ``signatory.Logsignature(depth)`` computes for a piecewise-linear path in its default "words" basis: the coefficients
of the Lyndon words (ordered by length, then lexicographically) of the logarithm of the signature in the truncated tensor
algebra.  ``signatory`` itself is not installable offline, so -- like the ODE stepping -- this is anchored on an independent
fp64 restatement (oracle/logsig_oracle.py) and on analytic facts (level 1 = increments, level 2 = Levy areas, a straight
line has no higher terms, Chen's identity across windows), not on the package's binary.

Gradients: the reference is differentiable through ``signatory`` in ``x`` and, through the clip of the last window end,
the linear fill of the added knots and the widths of ``logsignature_windows``, in ``t``.  Here the kernel's output
carries a torch-operator backward (``_windows_formula``, through ``_diff.KernelForward``), and the knots are built on
``t`` itself.  The same formula is the forward pass of the shapes the kernel refuses (more than 16 channels, depth over
6, or more than 640 terms), which the reference computes too.
"""
import torch

from . import _diff, _lib
from .coeffs import linear_interpolation_coeffs, validate_input_path


def lyndon_words(channels, depth):
    """All Lyndon words over ``range(channels)`` of length <= depth, ordered by length, then lexicographically (Duval)."""
    words = []
    w = [-1]
    while w:
        w[-1] += 1
        if len(w) <= depth:
            words.append(tuple(w))
        m = len(w)
        while len(w) < depth:
            w.append(w[-m])
        while w and w[-1] == channels - 1:
            w.pop()
    return sorted(words, key=lambda u: (len(u), u))


def logsignature_channels(channels, depth):
    """Number of logsignature channels (``signatory.logsignature_channels``; Witt's formula summed over the levels)."""
    return len(lyndon_words(channels, depth))


def _window_knots(t, window_length):
    """The window end points (in ``t``'s dtype, the last one clipped to the final time), where each of them sits in the
    merged knot sequence, and the end points that are not already observation times -- the bookkeeping of log_ode.py:18-40
    as one merge of two sorted lists on the host.  The end points are on ``t``'s device and keep its autograd graph through
    the clip, as the reference's do (its ``linspace`` carries no gradient)."""
    knots = t.detach().cpu()
    n_windows = int(((knots[-1] - knots[0]) / window_length).ceil().item())
    ends = torch.linspace(knots[0], knots[0] + n_windows * window_length, n_windows + 1, dtype=t.dtype)
    ends = torch.min(ends.to(t.device), t.max())
    knots = knots.tolist()
    rtol, atol = 1e-5, 1e-8                        # torch.allclose's defaults: when an end point counts as an observation time
    positions, extra = [], []
    k = 0
    for i, end in enumerate(ends.tolist()):
        while True:
            same = abs(end - knots[k]) <= atol + rtol * abs(knots[k])
            if same or end <= knots[k]:
                break
            k += 1
        positions.append(k + len(extra))
        if not same:
            extra.append(ends[i:i + 1])
    return ends, positions, extra


def _word_table(channels, depth):
    """(level, flat index) of every Lyndon word, the first letter most significant."""
    table = []
    for w in lyndon_words(channels, depth):
        flat = 0
        for letter in w:
            flat = flat * channels + letter
        table.append((len(w), flat))
    return table


def _tensor_mul(a, b, depth):
    """Product in the truncated tensor algebra; an element is a list of levels 0..depth of shape (..., C^k), the first
    factor's letters most significant in the flat index."""
    out = []
    for k in range(depth + 1):
        acc = a[0] * b[k]
        for j in range(1, k + 1):
            acc = acc + (a[j].unsqueeze(-1) * b[k - j].unsqueeze(-2)).flatten(-2)
        out.append(acc)
    return out


def _windows_formula(x, positions, depth, table):
    """Every window's logsignature with torch operators, batched over (path, window): x (P, L, C) filled, positions the
    window ends' indices into L.  Every window is padded to the longest with zero increments (exp(0) is the identity),
    Chen's product runs over the segment index as a pairwise tree, the logarithm is Horner's
    log(1 + X) = X (1 - X (1/2 - X (1/3 - ...))), and the Lyndon words are gathered.  This is the backward pass of the
    kernel, and the forward pass of the shapes the kernel does not take.  Returns (P, windows, words)."""
    channels = x.size(-1)
    first = torch.tensor(positions[:-1], device=x.device)
    counts = torch.tensor(positions[1:], device=x.device) - first
    n = 1
    while n < max(b - a for a, b in zip(positions[:-1], positions[1:])):
        n *= 2
    step = torch.arange(n, device=x.device)
    index = (first.unsqueeze(-1) + step).clamp(max=x.size(-2) - 2)                    # (W, n) segment indices
    dx = x[..., 1:, :] - x[..., :-1, :]
    inc = dx[..., index, :] * (step < counts.unsqueeze(-1)).unsqueeze(-1).to(x.dtype)  # (P, W, n, C)
    levels = [torch.ones_like(inc[..., :1]), inc]
    for k in range(2, depth + 1):
        levels.append((levels[-1].unsqueeze(-1) * inc.unsqueeze(-2)).flatten(-2) / k)
    while levels[0].size(-2) > 1:
        levels = _tensor_mul([v[..., 0::2, :] for v in levels], [v[..., 1::2, :] for v in levels], depth)
    s = [torch.zeros_like(levels[0].squeeze(-2))] + [v.squeeze(-2) for v in levels[1:]]   # signature - 1
    r = [torch.full_like(s[0], 1.0 / depth)] + [torch.zeros_like(v) for v in s[1:]]
    for m in range(depth - 1, 0, -1):
        r = [-v for v in _tensor_mul(s, r, depth)]
        r[0] = r[0] + 1.0 / m
    log = torch.cat(_tensor_mul(s, r, depth)[1:], dim=-1)
    offsets = [0, 0]
    for k in range(1, depth):
        offsets.append(offsets[-1] + channels ** k)
    return log[..., [offsets[level] + flat for level, flat in table]]


def _windows_kernel(x, positions, depth, table):
    """tcde_logsignature_windows: the same as ``_windows_formula``, one thread per (path, window)."""
    n_windows = len(positions) - 1
    with torch.cuda.device(x.device):
        window_index = torch.tensor(positions, dtype=torch.int32, device=x.device)
        word_table = torch.tensor(table, dtype=torch.int32, device=x.device).flatten()
        sigs = torch.empty(x.size(0), n_windows, len(table), dtype=x.dtype, device=x.device)
        _lib.call("tcde_logsignature_windows", _lib.ptr(x), x.size(0), x.size(1), x.size(2), _lib.ptr(window_index),
                  n_windows, depth, _lib.ptr(word_table), len(table), _lib.ptr(sigs), _lib.dtype_code(x.dtype),
                  _lib.stream_of(x))
    return sigs


def _logsignature_windows(x, depth, window_length, t, _version):
    t = validate_input_path(x, t)
    _lib.require_cuda(x)
    _lib.dtype_code(x.dtype)
    if _version not in (0, 1):
        raise RuntimeError
    new_t, new_t_indices, new_t_unique = _window_knots(t, window_length)
    batch_dimensions = x.shape[:-2]
    channels = x.size(-1)

    if len(new_t_unique) > 0:                       # window ends that are not observations: NaN rows, filled linearly below
        t_merged, indices = torch.cat([t, *new_t_unique]).sort()
        missing = torch.full((1,), float('nan'), dtype=x.dtype, device=x.device).expand(*batch_dimensions, 1, channels)
        x = torch.cat([x, missing], dim=-2)[..., indices.clamp(0, x.size(-2)).to(x.device), :]
    else:
        t_merged = t
    x = linear_interpolation_coeffs(x, t_merged.to(device=x.device, dtype=x.dtype))   # the gap-fill kernel

    table = _word_table(channels, depth)
    n_windows = len(new_t_indices) - 1
    flat_x = x.reshape(-1, x.size(-2), channels)
    if flat_x.size(0) == 0:
        sigs = flat_x.new_zeros(0, n_windows, len(table))
    else:
        try:
            sigs = _diff.with_kernel_forward(lambda xx: _windows_kernel(xx.contiguous(), new_t_indices, depth, table),
                                             lambda xx: _windows_formula(xx, new_t_indices, depth, table), flat_x)
        except NotImplementedError:
            # channels, depth or channels + ... + channels^depth beyond the kernel's per-thread storage (logsig.cu)
            sigs = _windows_formula(flat_x, new_t_indices, depth, table)
    sigs = sigs.view(*batch_dimensions, n_windows, len(table))
    if _version == 0:
        widths = (new_t[1:] - new_t[:-1]).to(device=x.device, dtype=x.dtype)
        sigs = sigs * widths.unsqueeze(-1)
    first_increment = torch.cat([x[..., :1, :], x.new_zeros(*batch_dimensions, 1, len(table) - channels)], dim=-1)
    logsignatures = torch.cat([first_increment, sigs], dim=-2).cumsum(dim=-2)
    if _version == 0:
        return logsignatures, new_t.to(x.device)
    return logsignatures


def logsignature_windows(x, depth, window_length, t=None):
    """DEPRECATED variant kept for backward compatibility (log_ode.py:80-107): returns ``(values, times)`` with each window's
    logsignature scaled by the window's width."""
    return _logsignature_windows(x, depth, window_length, t, _version=0)


def logsig_windows(x, depth, window_length, t=None):
    """Logsignatures over windows, as in the log-ODE method (log_ode.py:110-133): ``(..., length, channels)`` ->
    ``(..., 1 + number of windows, logsignature_channels(channels, depth))``; the corresponding times are 0, 1, 2, ..."""
    return _logsignature_windows(x, depth, window_length, t, _version=1)
