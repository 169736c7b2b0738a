"""fp64 restatement of a CDE with a tuple state (TupleControl) -- TEST INFRASTRUCTURE ONLY.

The reference (torchcde misc.py:129-166, solver.py:131-133) drives one CDE with several controls: member i of the state
evolves by ``f_i(t, z) @ dX_i/dt`` where ``(f_1, ..., f_K) = g(t, (z_1, ..., z_K))``, or by ``g.prod``'s own products.
torchdiffeq solves a tuple ``y0`` by flattening it into one vector (members end to end); that is what ``Packed`` does,
so ``odeint_port.odeint`` and the dopri5 below integrate the packed vector.

RECALLED, UNVERIFIED (torchdiffeq is not installed here): for a tuple state torchdiffeq's adaptive solvers use the
*mixed* norm, the largest of the members' RMS norms, both for the error ratio and for Hairer's initial step
(``_impl/misc.py`` ``_mixed_norm``).  ``solve_mixed`` restates ``adaptive_oracle.solve`` with that norm.

Everything is plain torch fp64.  Nothing here imports ``torchcde_b200``.
"""
import torch

from . import adaptive_oracle as A


class TupleFuncCDE:
    """The tuple field in fp64.  ``members``: ``adaptive_oracle.FuncCDE``-style controls given as ``(control, knots,
    kind)``; ``g(t, zs) -> tuple of (..., H_i, C_i)`` (or with ``prod`` ``g(t, zs, dxs) -> tuple of (..., H_i)``).  ``g``
    gets the stage time as a 0-dim fp64 tensor rounded to ``time_dtype``, as ``FuncCDE`` passes it."""

    def __init__(self, members, g, time_dtype=torch.float64, prod=False):
        self.controls = [A._Control(c, k, kind, time_dtype) for c, k, kind in members]
        self.g, self.prod, self.time_dtype = g, prod, time_dtype

    def time(self, t):
        return self.controls[0].time(t)

    def field_at(self, ts, zs):
        dxs = [c._dxdt_at(ts) for c in self.controls]
        if self.prod:
            return tuple(self.g(ts, zs, dxs))
        return tuple((f @ d.unsqueeze(-1)).squeeze(-1) for f, d in zip(self.g(ts, zs), dxs))

    def __call__(self, t, zs):
        return self.field_at(torch.tensor(self.time(t), dtype=torch.float64, device=self.controls[0].knots.device), zs)


class Packed:
    """A tuple field on the packed state: ``shapes`` of the members, ``pack`` / ``unpack`` of tuples."""

    def __init__(self, cde, shapes):
        self.cde, self.shapes = cde, [tuple(s) for s in shapes]
        self.sizes = [int(torch.Size(s).numel()) for s in self.shapes]

    def pack(self, parts):
        return torch.cat([p.reshape(-1) for p in parts])

    def unpack(self, flat):
        out, off = [], 0
        for s, n in zip(self.shapes, self.sizes):
            out.append(flat[..., off:off + n].reshape(*flat.shape[:-1], *s))
            off += n
        return tuple(out)

    def __call__(self, t, y):
        return self.pack(self.cde(t, self.unpack(y)))


def mixed_norm(sizes):
    """max over the members (``sizes`` elements each, end to end) of their RMS; empty members contribute nothing."""
    def norm(x):
        flat, off, best = x.reshape(-1), 0, 0.0
        for n in sizes:
            if n:
                best = max(best, A.rms(flat[off:off + n]))
            off += n
        return best
    return norm


def initial_step(field, t0, y0, f0, rtol, atol, norm):
    """``adaptive_oracle.initial_step`` with ``norm`` in place of the RMS."""
    scale = atol + rtol * y0.abs()
    d0, d1 = norm(y0 / scale), norm(f0 / scale)
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    d2 = norm((field(t0 + h0, y0 + h0 * f0) - f0) / scale) / h0
    if max(d1, d2) <= 1e-15:
        h1 = max(1e-6, h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1.0 / 5)
    return min(100 * h0, h1)


def solve_mixed(field, y0, times, rtol, atol, sizes, first_step=None, replay=None):
    """``adaptive_oracle.solve`` (free running, or replaying ``(t, dt, accepted)`` decisions) with the mixed norm of a
    packed tuple state.  Returns ``(outputs (len(times), numel), records, first_dt)``."""
    norm = mixed_norm(sizes)
    t, y = times[0], y0
    f = field(t, y)
    dt = first_step if first_step is not None else initial_step(field, t, y, f, rtol, atol, norm)
    first_dt = dt
    out, records, nxt = [y0], [], 1
    while nxt < len(times):
        if replay is not None:
            if len(records) == len(replay):
                raise RuntimeError("replay ran out of attempts at t = {}".format(t))
            rt, dt, accepted = replay[len(records)]
            t = rt
        res = A.attempt(field, t, dt, y, f)
        ratio = norm(res["err"] / (atol + rtol * torch.max(y.abs(), res["y1"].abs())))
        if replay is None:
            accepted = ratio <= 1.0
        records.append(A.Record(t, dt, accepted, ratio))
        if accepted:
            t_hi = t + dt
            coeff = None
            while nxt < len(times) and times[nxt] <= t_hi:
                if coeff is None:
                    coeff = A.dense_coefficients(y, res["y1"], res["y_mid"], f, res["ks"][6], dt)
                out.append(A.dense_evaluate(coeff, (times[nxt] - t) / (t_hi - t)))
                nxt += 1
            t, y, f = t_hi, res["y1"], res["ks"][6]
        if replay is None:
            dt = A.next_step(dt, ratio)
    return torch.stack(out), records, first_dt
