"""Logsignature of a piecewise-linear path -- TEST INFRASTRUCTURE ONLY (never imported by torchcde_b200/).

What this stands in for: ``signatory.Logsignature(depth)`` (reference call site torchcde/log_ode.py:56-58; optional
third-party C++ package, ``signatory`` in setup.py's extras, not vendored, not installable offline).  PARITY UNPINNED
against the package's binary; pinned instead on mathematics that does not depend on any implementation
(tests/test_logsig_oracle.py): level 1 = total increment, level 2 = Levy areas, a straight line has no terms above level 1,
Chen's identity, invariance under re-sampling of linear pieces.

Written to share NO code path with csrc/logsig.cu: dense ``numpy`` tensors per level (level k has shape (C,)*k), the
signature as the ordered product of the segments' tensor exponentials, the logarithm as the plain power series
``sum_n (-1)^(n+1) x^n / n`` with explicitly formed powers, fp64 throughout.
"""
import numpy as np


def _mul(a, b, depth):
    """Product in the truncated tensor algebra: a, b = lists [level0 scalar, level1 (C,), level2 (C, C), ...]."""
    out = []
    for k in range(depth + 1):
        acc = None
        for j in range(k + 1):
            term = np.multiply.outer(a[j], b[k - j])
            acc = term if acc is None else acc + term
        out.append(acc)
    return out


def _exp(dx, depth):
    levels = [np.array(1.0)]
    for k in range(1, depth + 1):
        levels.append(np.multiply.outer(levels[-1], dx) / k)
    return levels


def signature(path, depth):
    """path: (length, C) float64 -> [1, S1, ..., S_depth]."""
    c = path.shape[1]
    sig = [np.array(1.0)] + [np.zeros((c,) * k) for k in range(1, depth + 1)]
    for p in range(path.shape[0] - 1):
        sig = _mul(sig, _exp(path[p + 1] - path[p], depth), depth)
    return sig


def log_tensor(sig, depth):
    c = sig[1].shape[0]
    x = [np.array(0.0)] + [np.array(s) for s in sig[1:]]
    total = [np.array(0.0)] + [np.zeros((c,) * k) for k in range(1, depth + 1)]
    power = [np.array(1.0)] + [np.zeros((c,) * k) for k in range(1, depth + 1)]
    for n in range(1, depth + 1):
        power = _mul(power, x, depth)
        for k in range(depth + 1):
            total[k] = total[k] + ((-1.0) ** (n + 1)) * power[k] / n
    return total


def lyndon_words(channels, depth):
    """Brute force: a word is Lyndon iff it is strictly smaller than all of its proper rotations."""
    import itertools
    words = []
    for k in range(1, depth + 1):
        for w in itertools.product(range(channels), repeat=k):
            if all(w < w[i:] + w[:i] for i in range(1, k)):
                words.append(w)
    return words


def logsignature(path, depth):
    """Coefficients of the Lyndon words (by length, then lexicographically) of log(signature).  A complex ``path`` stays
    complex (the arithmetic is the same), which is what ``logsignature_jacobian`` differentiates through."""
    path = np.asarray(path)
    path = path.astype(np.complex128 if np.iscomplexobj(path) else np.float64)
    log = log_tensor(signature(path, depth), depth)
    return np.array([log[len(w)][w] for w in lyndon_words(path.shape[1], depth)])


def logsignature_jacobian(path, depth, h=1e-30):
    """d logsignature / d path, shape (n_words, length, C), by complex-step differentiation: imag(f(x + i h e_j)) / h.
    ``logsignature`` is built from +, * and / only, so there is no subtractive cancellation: the result is exact to
    rounding for any small ``h``."""
    path = np.asarray(path, dtype=np.float64)
    length, channels = path.shape
    cols = []
    for p in range(length):
        for c in range(channels):
            z = path.astype(np.complex128)
            z[p, c] += 1j * h
            cols.append(logsignature(z, depth).imag / h)
    return np.stack(cols, axis=-1).reshape(-1, length, channels)
