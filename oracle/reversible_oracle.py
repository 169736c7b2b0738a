"""fp64 oracle of torchsde's reversible Heun solve and of its reversible backward (test infrastructure; shares no code
with the package).

torchsde is not installed here and cannot be installed.  What follows about its internals is RECALLED, NOT VERIFIED
against its source:
  * ``sdeint(..., method="reversible_heun")`` uses a fixed step ``dt`` (default 1e-3) unless ``adaptive=True``;
  * ``integrate``: ``prev_t = curr_t = ts[0]``; for every output time ``out_t`` in ``ts[1:]``, ``while curr_t < out_t:
    next_t = min(curr_t + dt, ts[-1])`` and one step; the output is ``linear_interp(prev_t, prev_y, curr_t, curr_y,
    out_t)``; output 0 is ``y0``.  The grid is built by repeated addition in ``ts``'s dtype and steps on across output
    times; the last step is clipped;
  * ``linear_interp`` -- restated here in the two-weight form
    ``(t1 - t) / (t1 - t0) * y0 + (t - t0) / (t1 - t0) * y1``;
  * the step (diffusion zero, as the reference's ``_VectorField`` has ``g = 0``), from ``z0 = y0``,
    ``f0 = f(t0, y0)``:  ``z1 = 2 * y0 - z0 + f0 * dt``, ``f1 = f(t1, z1)``, ``y1 = y0 + (f0 + f1) * (0.5 * dt)``,
    with ``dt = t1 - t0`` and the field evaluated at the grid time ``t1``;
  * ``y0`` is 2-D ``(batch, hidden)`` and ``ts`` strictly increasing.

The backward recurrence below is the transpose of that step, derived by hand; its checkpointed variant restarts from
saved ``(y, z, f)`` states instead of reconstructing the whole solve from the final state (torchsde's algorithm as
recalled).  Tests check it against ``torch.autograd`` through ``integrate``.
"""
import torch


def linear_interp(t0, y0, t1, y1, t):
    w0 = (t1 - t) / (t1 - t0)
    w1 = (t - t0) / (t1 - t0)
    return w0 * y0 + w1 * y1, (w0, w1)


def step(f, t0, t1, y0, extra):
    f0, z0 = extra
    dt = t1 - t0
    z1 = 2 * y0 - z0 + f0 * dt
    f1 = f(t1, z1)
    y1 = y0 + (f0 + f1) * (0.5 * dt)
    return y1, (f1, z1)


def integrate(f, y0, ts, dt, keep=None):
    """torchsde's fixed-step loop.  ``f(t, y)``: the drift, ``t`` a 0-dim tensor of ``ts``'s dtype.  Returns
    ``(ys (len(ts), *y0.shape), record)``; ``record``: ``grid`` (list of 0-dim tensors), ``outputs`` (list of
    ``(step n, w0, w1)`` per output after the first) and ``states`` {step: (y, z, f)} for the steps in ``keep``
    (a callable of the step number, or None for all)."""
    prev_t = curr_t = ts[0]
    prev_y = curr_y = y0
    extra = (f(ts[0], y0), y0)
    grid = [curr_t]
    states = {0: (y0, y0, extra[0])}
    outputs = []
    ys = [y0]
    for out_t in ts[1:]:
        while curr_t < out_t:
            next_t = min(curr_t + dt, ts[-1])
            prev_t, prev_y = curr_t, curr_y
            curr_y, extra = step(f, curr_t, next_t, curr_y, extra)
            curr_t = next_t
            grid.append(curr_t)
            n = len(grid) - 1
            if keep is None or keep(n):
                states[n] = (curr_y, extra[1], extra[0])
        y, (w0, w1) = linear_interp(prev_t, prev_y, curr_t, curr_y, out_t)
        ys.append(y)
        outputs.append((len(grid) - 2, w0, w1))
    states[len(grid) - 1] = (curr_y, extra[1], extra[0])
    return torch.stack(ys, dim=0), {"grid": grid, "outputs": outputs, "states": states}


def reversible_backward(f, params, y0, ts, dt, grad_ys, checkpoint_every=None):
    """dL/dy0 and dL/dparams of ``integrate`` for output gradients ``grad_ys`` (same shape as its output), by running
    the solve backwards algebraically.  ``checkpoint_every``: restart from the saved state of every k-th step (and the
    last); None reconstructs everything from the final state."""
    params = tuple(params)
    with torch.no_grad():
        keep = (lambda n: False) if checkpoint_every is None else (lambda n: n % checkpoint_every == 0)
        _ys, rec = integrate(f, y0, ts, dt, keep)
    grid = rec["grid"]
    N = len(grid) - 1
    saved = rec["states"]
    if checkpoint_every is None:
        saved = {N: saved[N]}
    dts = [grid[n + 1] - grid[n] for n in range(N)]
    # adjoint of y_n from the outputs
    yin = {0: grad_ys[0].clone()}
    for j, (n, w0, w1) in enumerate(rec["outputs"], start=1):
        yin[n] = yin.get(n, 0) + w0 * grad_ys[j]
        yin[n + 1] = yin.get(n + 1, 0) + w1 * grad_ys[j]
    gparams = [torch.zeros_like(p) for p in params]

    def close_f(n, z, fbar):
        """f(t_n, z), and J^T fbar; adds dF/dparams^T fbar into gparams."""
        with torch.enable_grad():
            zz = z.detach().requires_grad_(True)
            out = f(grid[n], zz)
            got = torch.autograd.grad(out, (zz,) + params, fbar, allow_unused=True)
        for acc, g in zip(gparams, got[1:]):
            if g is not None:
                acc += g
        return out.detach(), got[0]

    y, z, fv = saved[N]
    ybar = torch.zeros_like(y0) + yin.get(N, 0)
    _, zbar = close_f(N, z, ybar * (dts[N - 1] / 2))
    for n in range(N - 1, -1, -1):
        d = dts[n]
        # the step n -> n + 1 backwards: its z and y equations
        z_n = 2 * y - z - fv * d
        ybar_n = ybar + 2 * zbar + yin.get(n, 0)
        fbar_n = ybar * (d / 2) + d * zbar
        if n > 0:
            fbar_n = fbar_n + ybar_n * (dts[n - 1] / 2)
        if n in saved:
            z_n = saved[n][1]
        f_n, jz = close_f(n, z_n, fbar_n)
        y_n = y - (f_n + fv) * (d / 2)
        if n in saved:
            y_n, f_n = saved[n][0], saved[n][2]
        zbar = jz - zbar
        ybar = ybar_n
        y, z, fv = y_n, z_n, f_n
    return ybar + zbar, gparams


def cubic_derivative(coeffs, knots, t):
    """dX/dt of a cubic spline with rows (a, b, 2c, 3d) at a 0-dim time (``_interpret_t`` then the polynomial)."""
    ch = coeffs.size(-1) // 4
    tt = t.to(knots.dtype)
    i = int(torch.bucketize(tt, knots).sub(1).clamp(0, knots.numel() - 2))
    fr = tt - knots[i]
    row = coeffs[..., i, :]
    b, c2, d3 = row[..., ch:2 * ch], row[..., 2 * ch:3 * ch], row[..., 3 * ch:]
    return b + (c2 + d3 * fr) * fr


def linear_derivative(slopes, knots, t):
    """dX/dt of a piecewise linear control with per-interval rows ``slopes`` at a 0-dim time: ``_interpret_t``'s
    interval, so a knot t_n (n > 0) takes the slope of interval n - 1.  Like ``_interpret_t`` (and ``cubic_derivative``)
    the time is cast to the knots' dtype first: pass the knots in the control's dtype to locate times as it does."""
    tt = t.to(knots.dtype)
    i = int(torch.bucketize(tt, knots).sub(1).clamp(0, slopes.size(-2) - 1))
    return slopes[..., i, :]


def _product_field(derivative, weight, bias):
    hidden = weight.size(1)

    def f(t, z):
        dx = derivative(t)
        m = torch.nn.functional.linear(z, weight, bias).view(*z.shape[:-1], hidden, -1)
        return (m @ dx.unsqueeze(-1)).squeeze(-1)

    return f


def linear_cde_field(coeffs, knots, weight, bias):
    """f(t, z) = (weight z + bias).view(H, C) . dX/dt(t) with a cubic control."""
    return _product_field(lambda t: cubic_derivative(coeffs, knots, t), weight, bias)


def linear_control_field(slopes, knots, weight, bias):
    """f(t, z) = (weight z + bias).view(H, C) . dX/dt(t) with a linear control given by its own slopes (the ``_derivs``
    rows of ``LinearInterpolation``); ``bias`` may be None."""
    return _product_field(lambda t: linear_derivative(slopes, knots, t), weight, bias)
