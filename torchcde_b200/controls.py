"""Control paths: ``CubicSpline`` and ``LinearInterpolation``.

Same constructor arguments, buffer names (``_t, _a, _b, _two_c, _three_d`` /
``_t, _coeffs, _derivs``), properties and ``evaluate`` / ``derivative`` contract as the
reference (interpolation_base.py:5-22, interpolation_cubic.py:268-346,
interpolation_linear.py:174-225).  The buffers are *views* of the coefficient tensor, as in
the reference (:297-305).  Evaluation at a tensor of times runs ``tcde_spline_eval`` (one
launch, no host sync); the interval index of every query time is computed with the
reference's own ``bucketize`` arithmetic so it is bit-exact.  ``evaluate`` / ``derivative`` are
differentiable in the coefficients, the knots and the query times (backward pass: ``_diff.py``).
"""
import abc

import torch

from . import _diff, _lib
from .schedule import locate


class InterpolationBase(torch.nn.Module, metaclass=abc.ABCMeta):
    @property
    @abc.abstractmethod
    def grid_points(self):
        raise NotImplementedError

    @property
    @abc.abstractmethod
    def interval(self):
        raise NotImplementedError

    @abc.abstractmethod
    def evaluate(self, t):
        raise NotImplementedError

    @abc.abstractmethod
    def derivative(self, t):
        raise NotImplementedError


def _schedule_knots(X):
    """The control's knots as a CPU tensor for the host-side schedule.  Default knots are the
    integers 0..n (exact in any float dtype), so they are rebuilt on the CPU instead of being read
    back from the device -- that keeps ``cdeint`` free of host syncs."""
    knots = X._t
    if X._default_knots:
        n = knots.numel()
        return torch.linspace(0, n - 1, n, dtype=knots.dtype)
    return knots.detach().cpu()


def _control_signature(X):
    """(kind, batch shape, channels, n_intervals) of a built-in control without evaluating it."""
    if isinstance(X, CubicSpline):
        return _lib.CONTROL_CUBIC, tuple(X._b.shape[:-2]), X._b.size(-1), X._b.size(-2)
    if isinstance(X, LinearInterpolation):
        return _lib.CONTROL_LINEAR, tuple(X._coeffs.shape[:-2]), X._coeffs.size(-1), X._coeffs.size(-2) - 1
    return None


def _eval_kernel(control, knots, n_rows, channels, index, frac, kind, derivative):
    """control: (..., n_rows, width) -> (..., *t.shape, channels) through the C ABI."""
    _lib.require_cuda(control)
    code = _lib.dtype_code(control.dtype)
    batch = control.shape[:-2]
    flat = control.reshape(-1, control.size(-2), control.size(-1))
    if not flat.is_contiguous():
        flat = flat.contiguous()
    tshape = index.shape
    idx = index.reshape(-1).to(torch.int32).contiguous()
    fr = frac.reshape(-1).to(control.dtype).contiguous()
    n_times = idx.numel()
    out = torch.empty(flat.size(0), n_times, channels, dtype=control.dtype, device=control.device)
    with torch.cuda.device(control.device):
        _lib.call("tcde_spline_eval", _lib.ptr(flat), _lib.ptr(knots), _lib.ptr(idx), _lib.ptr(fr), _lib.ptr(out),
                  flat.size(0), n_rows, channels, n_times, kind, int(derivative), code, _lib.stream_of(flat))
    return out.view(*batch, *tshape, channels)


class CubicSpline(InterpolationBase):
    """Piecewise cubic control from ``natural_cubic_coeffs`` / ``hermite_cubic_coefficients_with_
    backward_differences`` coefficients (interpolation_cubic.py:268-336)."""

    def __init__(self, coeffs, t=None, **kwargs):
        super(CubicSpline, self).__init__(**kwargs)

        self._default_knots = t is None
        if t is None:
            t = torch.linspace(0, coeffs.size(-2), coeffs.size(-2) + 1, dtype=coeffs.dtype, device=coeffs.device)

        channels = coeffs.size(-1) // 4
        if channels * 4 != coeffs.size(-1):  # check that it's a multiple of 4
            raise ValueError("Passed invalid coeffs.")

        self.register_buffer('_t', t)
        self.register_buffer('_a', coeffs[..., :channels])
        self.register_buffer('_b', coeffs[..., channels:2 * channels])
        self.register_buffer('_two_c', coeffs[..., 2 * channels:3 * channels])
        self.register_buffer('_three_d', coeffs[..., 3 * channels:])
        self._coeffs_ref = [coeffs]      # the whole rows, for the kernels (not a buffer: it aliases the four views)

    @property
    def grid_points(self):
        return self._t

    @property
    def interval(self):
        return torch.stack([self._t[0], self._t[-1]])

    @property
    def channels(self):
        return self._b.size(-1)

    def _rows(self):
        """The (..., L-1, 4C) coefficient tensor the four buffers are views of."""
        coeffs = self._coeffs_ref[0]
        if coeffs.device != self._b.device or coeffs.dtype != self._b.dtype:
            # the module was moved / cast after construction: rebuild the rows from the buffers
            coeffs = torch.cat([self._a, self._b, self._two_c, self._three_d], dim=-1)
            self._coeffs_ref[0] = coeffs
        return coeffs

    def _interpret_t(self, t):
        maxlen = self._b.size(-2) - 1
        t = torch.as_tensor(t, dtype=self._b.dtype, device=self._b.device)
        return locate(self._t, t, maxlen + 1)

    def _eval(self, t, derivative):
        t = torch.as_tensor(t, dtype=self._b.dtype, device=self._b.device)
        fractional_part, index = self._interpret_t(t)

        def kernel(*_):
            knots = self._t.detach().to(self._b.dtype).contiguous()
            return _eval_kernel(self._rows().detach(), knots, self._b.size(-2), self.channels, index,
                                fractional_part.detach(), _lib.CONTROL_CUBIC, derivative)

        # differentiable in the coefficients, the knots and the query times like the reference's torch operators
        # (interpolation_cubic.py:315-336): the backward pass recomputes the polynomial with torch operators
        return _diff.with_kernel_forward(
            kernel, lambda a, b, c, d, k, tt: _diff.cubic_eval(a, b, c, d, k.to(tt.dtype), tt, index, derivative),
            self._a, self._b, self._two_c, self._three_d, self._t, t)

    def evaluate(self, t):
        return self._eval(t, False)

    def derivative(self, t):
        return self._eval(t, True)


class NaturalCubicSpline(CubicSpline):
    """Deprecated alias kept for backward compatibility (interpolation_cubic.py:339-346)."""


class LinearInterpolation(InterpolationBase):
    """Piecewise linear control (interpolation_linear.py:174-225)."""

    def __init__(self, coeffs, t=None, **kwargs):
        super(LinearInterpolation, self).__init__(**kwargs)

        self._default_knots = t is None
        if t is None:
            t = torch.linspace(0, coeffs.size(-2) - 1, coeffs.size(-2), dtype=coeffs.dtype, device=coeffs.device)

        # slopes per interval, precomputed and registered like the reference (interpolation_linear.py:189-193:
        # state_dict keys ``_t``, ``_coeffs``, ``_derivs``); on the GPU they come from the evaluation kernel (the same
        # ``(x[i+1] - x[i]) / (t[i+1] - t[i])``, bit-identical); a module built from CPU tensors (to be moved with
        # ``.to(device)`` before use) forms them with the reference's own two torch ops
        def slopes(c, k):
            return (c[..., 1:, :] - c[..., :-1, :]) / (k[1:] - k[:-1]).unsqueeze(-1)

        if coeffs.is_cuda:
            def kernel(c, k):
                n = c.size(-2) - 1
                index = torch.arange(n, device=c.device)
                frac = torch.zeros(n, dtype=c.dtype, device=c.device)
                knots = k.to(device=c.device, dtype=c.dtype).contiguous()
                return _eval_kernel(c, knots, c.size(-2), c.size(-1), index, frac, _lib.CONTROL_LINEAR, True)

            derivs = _diff.with_kernel_forward(kernel, slopes, coeffs, t)
        else:
            derivs = slopes(coeffs, t)

        self.register_buffer('_t', t)
        self.register_buffer('_coeffs', coeffs)
        self.register_buffer('_derivs', derivs)

    @property
    def grid_points(self):
        return self._t

    @property
    def interval(self):
        return torch.stack([self._t[0], self._t[-1]])

    @property
    def channels(self):
        return self._coeffs.size(-1)

    def _interpret_t(self, t):
        maxlen = self._coeffs.size(-2) - 2
        t = torch.as_tensor(t, dtype=self._coeffs.dtype, device=self._coeffs.device)
        return locate(self._t, t, maxlen + 1)

    def _eval(self, t, derivative):
        t = torch.as_tensor(t, dtype=self._coeffs.dtype, device=self._coeffs.device)
        fractional_part, index = self._interpret_t(t)

        def kernel(*_):
            knots = self._t.detach().to(self._coeffs.dtype).contiguous()
            return _eval_kernel(self._coeffs.detach(), knots, self._coeffs.size(-2), self.channels, index,
                                fractional_part.detach(), _lib.CONTROL_LINEAR, derivative)

        return _diff.with_kernel_forward(
            kernel, lambda c, k, tt: _diff.linear_eval(c, k.to(tt.dtype), tt, index, derivative), self._coeffs, self._t, t)

    def evaluate(self, t):
        return self._eval(t, False)

    def derivative(self, t):
        return self._eval(t, True)
