"""Restatement of torchdiffeq's fixed-grid ``odeint`` -- TEST INFRASTRUCTURE ONLY.

What this stands in for
-----------------------
``torchcde.cdeint`` contains no time stepping.  It hands a vector field to
``torchdiffeq.odeint`` (reference call site: torchcde/solver.py:226-227).  torchdiffeq
is a third-party dependency pinned only as ``torchdiffeq>=0.2.0`` (setup.py:51); it is
not vendored in the reference repository, not installed here and not installable (no
network).  This module restates the *published* algorithm of torchdiffeq 0.2.x's
fixed-grid solvers (its ``_impl/fixed_grid.py``, ``_impl/solvers.py``
``FixedGridODESolver``, ``_impl/rk_common.py`` ``rk4_alt_step_func`` and the time
normalisation of ``_impl/misc.py``) so that the reference ``cdeint`` can be executed
end to end with this module installed in ``sys.modules['torchdiffeq']``.

PARITY UNPINNED for the stepping arithmetic: there is no torchdiffeq binary on this
machine to diff against.  It is anchored instead on (tests/test_oracle_solver.py):
  * the analytic solutions of the reference's own test fixtures
    (test_cdeint.py:54-55 ``func = -z`` and :90-95 ``prod = -z * dXdt``);
  * observed convergence order 1 / 2 / 4 for euler / midpoint / rk4;
  * explicit midpoint with the field evaluated at ``t + dt/2`` (test_cdeint.py:49-63).

Semantics restated (all of them matter for bit-level interval selection downstream):
  * the grid is ``arange(ceil((t[-1]-t[0])/h + 1)) * h + t[0]`` in ``t``'s dtype with
    the last entry overwritten by ``t[-1]``; without ``step_size`` the grid is ``t``;
  * ``rk4`` is the 3/8-rule: stages at ``t0, t0 + dt/3, t0 + 2dt/3, t1`` and
    ``dy = (k1 + 3 (k2 + k3) + k4) * dt / 8``;
  * ``midpoint``: ``dy = dt * f(t0 + dt/2, y0 + f(t0, y0) * dt/2)``; ``euler``:
    ``dy = dt * f(t0, y0)``;
  * stage times are formed in ``t``'s dtype and cast to the state's dtype just before
    the vector field is called;
  * requested output times strictly inside a step are linearly interpolated between
    the step's end points; an output time equal to an end point copies that end point;
  * a decreasing ``t`` is integrated as ``-t`` with the field ``-f(-t, y)``;
  * the result is stacked with time on dim 0.
"""
import torch

_FIXED_METHODS = ("euler", "midpoint", "rk4")

_THIRD = 1 / 3
_TWO_THIRDS = 2 / 3


class _CastTime:
    """Cast the stage time to the state's real dtype before calling the field."""

    def __init__(self, field):
        self.field = field

    def __call__(self, t, y):
        return self.field(t.to(y.abs().dtype), y)


class _Reversed:
    def __init__(self, field):
        self.field = field

    def __call__(self, t, y):
        return -1.0 * self.field(-t, y)


def make_time_grid(t, step_size):
    if step_size is None:
        return t
    first, last = t[0], t[-1]
    count = torch.ceil((last - first) / step_size + 1).item()
    grid = torch.arange(0, count, dtype=t.dtype, device=t.device) * step_size + first
    grid[-1] = t[-1]
    return grid


def _step_euler(f, t0, dt, t1, y0):
    return dt * f(t0, y0)


def _step_midpoint(f, t0, dt, t1, y0):
    half = 0.5 * dt
    k1 = f(t0, y0)
    return dt * f(t0 + half, y0 + k1 * half)


def _step_rk4_38(f, t0, dt, t1, y0):
    k1 = f(t0, y0)
    k2 = f(t0 + dt * _THIRD, y0 + dt * k1 * _THIRD)
    k3 = f(t0 + dt * _TWO_THIRDS, y0 + dt * (k2 - k1 * _THIRD))
    k4 = f(t1, y0 + dt * (k1 - k2 + k3))
    return (k1 + 3 * (k2 + k3) + k4) * dt * 0.125


_STEPPERS = {"euler": _step_euler, "midpoint": _step_midpoint, "rk4": _step_rk4_38}


def _between(t0, t1, y0, y1, t):
    if t == t0:
        return y0
    if t == t1:
        return y1
    slope = (t - t0) / (t1 - t0)
    return y0 + slope * (y1 - y0)


def odeint(func, y0, t, *, rtol=1e-7, atol=1e-9, method=None, options=None, **unused):
    if method not in _FIXED_METHODS:
        raise NotImplementedError(
            "oracle odeint port restates only the fixed-grid methods {}; got method={!r}".format(
                _FIXED_METHODS, method))
    options = dict(options or {})
    step_size = options.pop("step_size", None)
    if options:
        raise NotImplementedError("oracle odeint port: unsupported options {}".format(sorted(options)))
    if not isinstance(y0, torch.Tensor):
        raise NotImplementedError("oracle odeint port: tensor state only")

    field = func
    flipped = len(t) > 1 and bool(t[0] > t[1])
    if flipped:
        t = -t
        field = _Reversed(field)
    if not bool((t[1:] > t[:-1]).all()):
        raise ValueError("t must be strictly increasing or decreasing")
    if t.device != y0.device:
        t = t.to(y0.device)
    field = _CastTime(field)

    stepper = _STEPPERS[method]
    grid = make_time_grid(t, step_size)
    assert grid[0] == t[0] and grid[-1] == t[-1]

    out = torch.empty(len(t), *y0.shape, dtype=y0.dtype, device=y0.device)
    out[0] = y0
    nxt = 1
    y = y0
    for t0, t1 in zip(grid[:-1], grid[1:]):
        dt = t1 - t0
        y_new = y + stepper(field, t0, dt, t1, y)
        while nxt < len(t) and t1 >= t[nxt]:
            out[nxt] = _between(t0, t1, y, y_new, t[nxt])
            nxt += 1
        y = y_new
    return out


def odeint_adjoint(func, y0, t, *, rtol=1e-7, atol=1e-9, method=None, options=None,
                   adjoint_rtol=None, adjoint_atol=None, adjoint_method=None, adjoint_options=None,
                   adjoint_params=None, **unused):
    """Forward values only: identical to ``odeint`` (the adjoint changes gradients, not outputs)."""
    return odeint(func, y0, t, rtol=rtol, atol=atol, method=method, options=options)
