"""torchcde_b200 -- an H100-native (sm_90a) Neural-CDE solve path with the torchcde API.

Drop-in names (reference torchcde/__init__.py:1-9): ``cdeint``, ``CubicSpline``,
``LinearInterpolation``, ``natural_cubic_coeffs``, ``natural_cubic_spline_coeffs``,
``linear_interpolation_coeffs``, ``hermite_cubic_coefficients_with_backward_differences``,
``InterpolationBase``.  The arithmetic lives in hand-written CUDA behind the C ABI of
``include/torchcde_b200.h``; this package is the thin Python host layer.  CUDA tensors only:
there is no CPU path and no PyTorch-eager fallback.

``logsig_windows`` / ``logsignature_windows`` (the log-ODE transform) run on a kernel of this package instead of the optional
``signatory`` dependency.  ``cdeint(..., backend="torchsde", method="reversible_heun")`` is torchsde's reversible Heun
method with an exact, checkpointed reversible backward (``reversible.py``); the other torchsde methods are not built.
Not provided (outside the hot path, SURVEY.md section 2): ``TupleControl``.
"""
from . import misc
from .coeffs import (hermite_cubic_coefficients_with_backward_differences, linear_interpolation_coeffs,
                     natural_cubic_coeffs, natural_cubic_spline_coeffs)
from .controls import CubicSpline, InterpolationBase, LinearInterpolation, NaturalCubicSpline
from .log_ode import logsig_windows, logsignature_windows
from .solver import LinearVectorField, cdeint

__version__ = "0.1.0"

__all__ = [
    "InterpolationBase", "natural_cubic_spline_coeffs", "natural_cubic_coeffs", "CubicSpline",
    "linear_interpolation_coeffs", "LinearInterpolation", "hermite_cubic_coefficients_with_backward_differences",
    "logsignature_windows", "logsig_windows", "cdeint", "LinearVectorField", "NaturalCubicSpline", "misc",
]
