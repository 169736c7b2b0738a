"""Host-side schedule of a fixed-step solve: which spline interval every Runge-Kutta stage
reads, with what fraction, and where the requested outputs fall.

The fused kernel (csrc/solve_simt.cu) takes no times at all -- only this table.  The table is
built here with the *same torch operations, in the same dtypes and order,* as the reference
stack would execute them one stage at a time:

  * the time grid and stage times of torchdiffeq's fixed-grid solvers (published algorithm,
    restated independently in oracle/odeint_port.py: grid = arange(ceil((t1-t0)/h + 1)) * h + t0
    with the last entry replaced by t[-1]; rk4 = 3/8 rule with stages at t0, t0+dt/3,
    t0+2dt/3, t1; midpoint at t0, t0+dt/2), formed in ``t``'s dtype and cast to the state dtype;
  * ``CubicSpline._interpret_t`` (interpolation_cubic.py:315-322): cast to the coefficient
    dtype, ``bucketize(t, knots) - 1`` clamped to ``[0, n_intervals - 1]``, ``frac = t - knots[idx]``.

Because it is literally ``torch.bucketize`` on the same numbers, the interval indices are
bit-exact with the reference by construction (a knot t_n, n > 0, belongs to interval n-1).
Everything here is O(number of steps) scalar work on the CPU.
"""
import bisect
import collections

import numpy as np
import torch

_ONE_THIRD = 1 / 3
_TWO_THIRDS = 2 / 3

FIXED_METHODS = ("euler", "midpoint", "rk4")
N_STAGES = {"euler": 1, "midpoint": 2, "rk4": 4}


class Schedule:
    """CPU tensors describing one fixed-step solve (see include/torchcde_b200.h)."""

    __slots__ = ("method", "n_steps", "n_stages", "n_out", "sign", "step_dt", "stage_index", "stage_frac",
                 "out_step", "out_mode", "out_slope", "grid", "stage_times")

    def device_buffers(self, device):
        """Pack into two device tensors (one float, one int32) and return them with the views."""
        floats = torch.cat([self.step_dt, self.stage_frac.reshape(-1), self.out_slope]).to(device)
        ints = torch.cat([self.stage_index.reshape(-1), self.out_step, self.out_mode]).to(device)
        # (a reversible Heun schedule has one evaluation point more than steps and two output weights per output)
        ns, nst, no, nw = self.n_steps, self.stage_index.numel(), self.n_out, self.out_slope.numel()
        views = {
            "step_dt": floats[:ns], "stage_frac": floats[ns:ns + nst], "out_slope": floats[ns + nst:ns + nst + nw],
            "stage_index": ints[:nst], "out_step": ints[nst:nst + no], "out_mode": ints[nst + no:nst + 2 * no],
        }
        return floats, ints, views


def fixed_time_grid(t, step_size):
    if step_size is None:
        return t
    start, end = t[0], t[-1]
    niters = torch.ceil((end - start) / step_size + 1).item()
    grid = torch.arange(0, niters, dtype=t.dtype, device=t.device) * step_size + start
    grid[-1] = t[-1]
    return grid


def locate(knots, times, n_intervals):
    """The reference's ``_interpret_t`` on a tensor of times: (fraction, int64 index)."""
    times = torch.as_tensor(times, dtype=knots.dtype, device=knots.device)
    index = torch.bucketize(times.detach(), knots.detach()).sub(1).clamp(0, n_intervals - 1)
    return times - knots[index], index


def host_locator(knots, n_rows, state_dtype):
    """``(t_float, nudge) -> (interval index, fraction)``: the scalar version of ``locate`` with exactly the casts the
    reference stack applies to a stage time (to the state dtype by the solver, to the coefficient dtype by
    ``_interpret_t``), evaluated on the CPU so that no device sync is needed per stage.  ``knots``: CPU tensor."""
    # numpy scalars round exactly like the tensor casts, ``bisect_left`` is ``torch.bucketize`` (right=False), and none
    # of it goes through the torch dispatcher (this runs once per vector-field evaluation of the adaptive and adjoint
    # drivers)
    state_t = np.dtype(str(state_dtype).replace("torch.", "")).type
    knot_t = np.dtype(str(knots.dtype).replace("torch.", "")).type
    knot_list = knots.tolist()
    knot_vals = [knot_t(v) for v in knot_list]

    def where(t, nudge=0):
        tt = state_t(t)
        if nudge:
            tt = np.nextafter(tt, tt + state_t(1))
        tk = knot_t(tt)
        index = min(max(bisect.bisect_left(knot_list, float(tk)) - 1, 0), n_rows - 1)
        return index, float(tk - knot_vals[index])

    return where


def build_schedule(t, knots, n_intervals, method, step_size, state_dtype):
    """``t``: requested output times (1-D, any float dtype); ``knots``: the control's grid points
    (1-D, coefficient dtype); ``state_dtype``: dtype of z0 (the kernel's compute dtype)."""
    if method not in FIXED_METHODS:
        raise ValueError("fixed-step schedule: unknown method {!r}".format(method))
    t = t.detach().cpu()
    knots = knots.detach().cpu()
    if t.dim() != 1 or t.numel() < 2:
        raise ValueError("t must be one dimensional with at least two entries.")
    if not t.is_floating_point():
        raise ValueError("t must be floating point.")
    sign = 1.0
    if bool(t[0] > t[1]):
        t = -t
        sign = -1.0
    if not bool((t[1:] > t[:-1]).all()):
        raise ValueError("t must be strictly increasing or decreasing")

    grid = fixed_time_grid(t, step_size)
    if grid.numel() < 2 or not (grid[0] == t[0] and grid[-1] == t[-1]):
        raise ValueError("fixed-step schedule: the time grid does not span t (step_size={})".format(step_size))
    t0, t1 = grid[:-1], grid[1:]
    dt = t1 - t0
    if method == "rk4":
        stages = torch.stack([t0, t0 + dt * _ONE_THIRD, t0 + dt * _TWO_THIRDS, t1], dim=1)
    elif method == "midpoint":
        stages = torch.stack([t0, t0 + 0.5 * dt], dim=1)
    else:
        stages = t0.unsqueeze(1)
    stages = stages.to(state_dtype)          # the solver hands the field a time in the state's dtype
    if sign < 0:
        stages = -stages                      # time reversal: f is evaluated at -t and negated
    frac, index = locate(knots, stages, n_intervals)

    n_out = t.numel()
    out_step = torch.full((n_out,), -1, dtype=torch.int32)
    out_mode = torch.zeros(n_out, dtype=torch.int32)
    out_slope = torch.zeros(n_out, dtype=state_dtype)
    where = torch.searchsorted(t1.contiguous(), t[1:].contiguous(), right=False)   # first step with t1 >= t[j]
    for j in range(1, n_out):
        i = int(where[j - 1])
        out_step[j] = i
        if t[j] == t0[i]:
            out_mode[j] = 0
        elif t[j] == t1[i]:
            out_mode[j] = 1
        else:
            out_mode[j] = 2
            out_slope[j] = ((t[j] - t0[i]) / (t1[i] - t0[i])).to(state_dtype)

    s = Schedule()
    s.method = method
    s.n_steps = int(dt.numel())
    s.n_stages = N_STAGES[method]
    s.n_out = n_out
    s.sign = sign
    s.step_dt = dt.to(state_dtype).contiguous()
    s.stage_index = index.to(torch.int32).contiguous()
    s.stage_frac = frac.to(state_dtype).contiguous()
    s.out_step, s.out_mode, s.out_slope = out_step, out_mode, out_slope
    s.grid = grid
    s.stage_times = stages
    return s


def backward_tables(sched):
    """The tables of ``tcde_cdeint_fixed_linear_backward`` for a fixed-step ``sched`` (CPU tensors): the step widths and
    the stage intervals / fractions in reverse order, and the output gradients every grid state receives, as a list of
    (output, weight) entries grouped by grid state counted from the end (``inj_range[r] .. inj_range[r + 1] - 1`` belong
    to grid state ``n_steps - r``).  Output j after step i lands on that step's start (mode 0, or ``out_step = -1``: z0)
    or end (mode 1) with weight 1, or, interpolated at slope s (mode 2), on the start with ``1 - s`` and on the end with
    ``s`` -- the derivatives of ``y + s (y1 - y)``, formed in the state dtype."""
    n_steps = sched.n_steps
    by_state = [[] for _ in range(n_steps + 1)]
    one_minus = (1 - sched.out_slope).tolist()
    slopes = sched.out_slope.tolist()
    for j, (step, mode) in enumerate(zip(sched.out_step.tolist(), sched.out_mode.tolist())):
        if step < 0 or mode == 0:
            by_state[max(step, 0)].append((j, 1.0))
        elif mode == 1:
            by_state[step + 1].append((j, 1.0))
        else:
            by_state[step].append((j, one_minus[j]))
            by_state[step + 1].append((j, slopes[j]))
    entries = [e for state in reversed(by_state) for e in state]
    inj_range = [0]
    for state in reversed(by_state):
        inj_range.append(inj_range[-1] + len(state))
    return {
        "step_dt": sched.step_dt.flip(0),
        "stage_index": sched.stage_index.reshape(-1).flip(0),
        "stage_frac": sched.stage_frac.reshape(-1).flip(0),
        "inj_range": torch.tensor(inj_range, dtype=torch.int32),
        "inj_out": torch.tensor([j for j, _w in entries], dtype=torch.int32),
        "inj_weight": torch.tensor([w for _j, w in entries], dtype=sched.out_slope.dtype),
    }


def backward_views(sched, device):
    """``backward_tables(sched)`` on ``device`` in two copies: the float tables packed into one buffer, the int tables
    into another, returned as views named like the tables."""
    tables = backward_tables(sched)
    views = {}
    for names in (("step_dt", "stage_frac", "inj_weight"), ("stage_index", "inj_range", "inj_out")):
        packed = torch.cat([tables[n] for n in names]).to(device)
        views.update(zip(names, packed.split([tables[n].numel() for n in names])))
    return views


def build_sde_schedule(t, knots, n_intervals, dt, state_dtype):
    """The schedule of torchsde's fixed-step ``integrate`` loop with the reversible Heun method, in the table format of
    ``build_schedule`` (``tcde_cdeint_reversible_heun_linear`` reads it):

      * the grid is made by repeated addition in ``t``'s dtype, ``next_t = min(curr_t + dt, t[-1])``, stepping on across
        the output times; the last step is clipped and may be very small;
      * ``stage_index`` / ``stage_frac`` locate the ``N + 1`` evaluation points ``t_0 .. t_N`` (the prologue f(t_0, y_0),
        then one evaluation at the end of every step), cast to the coefficient dtype like ``_interpret_t``;
      * output ``j > 0`` is torchsde's ``linear_interp`` between the two grid states that bracket ``t[j]``,
        ``w0 * y_n + w1 * y_{n+1}`` with ``w0 = (t_{n+1} - t[j]) / dt_n`` and ``w1 = (t[j] - t_n) / dt_n`` formed in ``t``'s
        dtype; ``out_step[j] = n`` and ``out_slope`` holds ``[w1 of every output, w0 of every output]``; output 0 is
        ``y_0`` (``out_step = -1``).

    ``t`` must be 1-D and strictly increasing (torchsde integrates forwards only)."""
    t = t.detach().cpu()
    knots = knots.detach().cpu()
    if t.dim() != 1 or t.numel() < 2:
        raise ValueError("t must be one dimensional with at least two entries.")
    if not t.is_floating_point():
        raise ValueError("t must be floating point.")
    if not bool((t[1:] > t[:-1]).all()):
        raise ValueError("torchsde backend: t must be strictly increasing")
    dt = float(dt)
    if not dt > 0:
        raise ValueError("torchsde backend: dt must be positive, got {}".format(dt))
    end = t[-1]
    grid = [t[0]]
    curr = t[0]
    n_out = t.numel()
    out_step = torch.full((n_out,), -1, dtype=torch.int32)
    w0 = torch.zeros(n_out, dtype=t.dtype)
    w1 = torch.zeros(n_out, dtype=t.dtype)
    for j in range(1, n_out):
        out_t = t[j]
        while curr < out_t:
            curr = min(curr + dt, end)
            grid.append(curr)
        t0, t1 = grid[-2], grid[-1]
        out_step[j] = len(grid) - 2
        w0[j] = (t1 - out_t) / (t1 - t0)
        w1[j] = (out_t - t0) / (t1 - t0)
    grid = torch.stack(grid)
    frac, index = locate(knots, grid.to(knots.dtype), n_intervals)

    s = Schedule()
    s.method = "reversible_heun"
    s.n_steps = grid.numel() - 1
    s.n_stages = 1
    s.n_out = n_out
    s.sign = 1.0
    s.step_dt = (grid[1:] - grid[:-1]).to(state_dtype).contiguous()
    s.stage_index = index.to(torch.int32).contiguous()
    s.stage_frac = frac.to(state_dtype).contiguous()
    s.out_step = out_step
    s.out_mode = torch.zeros(n_out, dtype=torch.int32)
    s.out_slope = torch.cat([w1, w0]).to(state_dtype).contiguous()
    s.grid = grid
    s.stage_times = grid
    return s


class ScheduleCache:
    """Value-keyed LRU of device-resident schedules (the build is ~0.3 ms of tiny CPU ops)."""

    def __init__(self, capacity=16):
        self.capacity = capacity
        self.entries = collections.OrderedDict()

    def get(self, t, knots, n_intervals, method, step_size, state_dtype, device):
        t_cpu = t.detach().cpu()
        k_cpu = knots.detach().cpu()
        key = (t_cpu.dtype, t_cpu.numpy().tobytes(), k_cpu.dtype, k_cpu.numpy().tobytes(), n_intervals, method,
               None if step_size is None else float(step_size), state_dtype, str(device))
        hit = self.entries.get(key)
        if hit is not None:
            self.entries.move_to_end(key)
            return hit
        sched = build_schedule(t_cpu, k_cpu, n_intervals, method, step_size, state_dtype)
        packed = sched.device_buffers(device)
        self.entries[key] = (sched, packed)
        if len(self.entries) > self.capacity:
            self.entries.popitem(last=False)
        return sched, packed
