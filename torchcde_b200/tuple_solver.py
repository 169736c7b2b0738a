"""``cdeint`` with a tuple / list state: one CDE driven by several controls (a ``TupleControl``, misc.py:129-166).

The reference hands a tuple state to torchdiffeq, which flattens it into one vector and solves that (the vector field is
``tuple(f_i @ dX_i/dt)``, solver.py:131-133).  Here, too, the members live end to end in one packed buffer, so every
Runge-Kutta combination, dopri5 stage and adjoint step is one operation on it, and ``func`` sees a tuple of views:

  * no gradient, fixed step, every member a built-in control: the grouped stage loop.  Per step ONE launch of
    ``tcde_spline_eval_grouped`` evaluates every member's dX/dt at every stage (each member's intervals located on its own
    knots by the host schedule); per stage ``func`` runs, then ONE launch of ``tcde_field_contract_grouped`` forms every
    member's ``f_i @ dX_i``.  ``options={"cuda_graph": True}`` captures the loop like the tensor-state loop.
  * dopri5: ``adaptive.Dopri5`` on the packed state with the same grouped field (one evaluation and one contraction
    launch per field evaluation) and the mixed error norm of ``adaptive.tuple_norm``.
  * ``adjoint=True``: ``adaptive.solve_with_adjoint`` on the packed state, autograd per stage of the backward solve.
  * gradients with ``adjoint=False``, and members that are not this package's controls: the differentiable generic
    loop of ``solver._generic_solve`` / the torch-operator field through ``X.derivative(t)``.
"""
import torch

from . import _lib, adaptive
from .controls import TupleControl, _control_signature, _schedule_knots
from .linear_field import _reverse
from .schedule import FIXED_METHODS, build_schedule, host_locator


# ------------------------------------------------------------------------------- validation (solver.py:68-98)
def check_compatability(X, func, z0, t, is_prod, shape_error_forward, shape_error_prod):
    """The tuple branch of the reference's ``_check_compatability``, message for message."""
    control_gradient = X.derivative(t[0].detach())
    if is_prod:
        vector_field = func.prod(t[0], tuple(z0), control_gradient)
    else:
        system = func(t[0], tuple(z0))
    if not isinstance(control_gradient, (tuple, list)):
        raise ValueError("z0 is a tuple/list and so X.derivative must return a tuple/list as well.")
    if len(z0) != len(control_gradient):
        raise ValueError("z0 and X.derivative(t) must be tuples of the same length.")
    if is_prod:
        if not isinstance(vector_field, (tuple, list)):
            raise ValueError("z0 is a tuple/list and so func.prod must return a tuple/list as well.")
        if len(z0) != len(vector_field):
            raise ValueError("z0 and func.prod(t, z, dXdt) must be tuples of the same length.")
        for control_gradient_, vector_field_, z0_ in zip(control_gradient, vector_field, z0):
            if not isinstance(control_gradient_, torch.Tensor):
                raise ValueError("X.derivative must return a tensor or tuple of tensors.")
            if not isinstance(vector_field_, torch.Tensor):
                raise ValueError("func.prod must return a tensor or tuple/list of tensors.")
            shape_error_prod(tuple(control_gradient_.shape), tuple(vector_field_.shape), z0_)
    else:
        if not isinstance(system, (tuple, list)):
            raise ValueError("z0 is a tuple/list and so func must return a tuple/list as well.")
        if len(z0) != len(system):
            raise ValueError("z0 and func(t, z) must be tuples of the same length.")
        for control_gradient_, system_, z0_ in zip(control_gradient, system, z0):
            if not isinstance(control_gradient_, torch.Tensor):
                raise ValueError("X.derivative must return a tensor or tuple of tensors.")
            if not isinstance(system_, torch.Tensor):
                raise ValueError("func must return a tensor or tuple/list of tensors.")
            shape_error_forward(tuple(control_gradient_.shape), tuple(system_.shape), z0_)


# ------------------------------------------------------------------------------------------------ the packed state
class Packing:
    """Members of a tuple state end to end in one vector (torchdiffeq's flattening of a tuple ``y0``)."""

    def __init__(self, z0):
        self.shapes = [tuple(z.shape) for z in z0]
        self.sizes = [z.numel() for z in z0]
        self.offsets = [sum(self.sizes[:i]) for i in range(len(self.sizes))]
        self.numel = sum(self.sizes)

    def pack(self, parts):
        return torch.cat([p.reshape(-1) for p in parts])

    def views(self, flat):
        """Member views of ``flat`` (..., numel): (..., *shape_i)."""
        lead = tuple(flat.shape[:-1])
        return tuple(flat[..., o:o + n].view(*lead, *s) for o, n, s in zip(self.offsets, self.sizes, self.shapes))

    def outputs(self, ys):
        """(len(t), numel) -> the reference's output tuple, time at dim -2 of every member (solver.py:238-243)."""
        return tuple(y.movedim(0, -2) for y in self.views(ys))


class _PackedProd:
    """The tuple vector field as a ``prod`` on the packed state, for the tensor-state drivers of ``solver``."""

    def __init__(self, func, is_prod, packing):
        self.func, self.is_prod, self.packing = func, is_prod, packing

    def prod(self, t, z, dx):
        zs = self.packing.views(z)
        if self.is_prod:
            return self.packing.pack(self.func.prod(t, zs, dx))
        return self.packing.pack([(f @ d.unsqueeze(-1)).squeeze(-1) for f, d in zip(self.func(t, zs), dx)])


# --------------------------------------------------------------------------------------- the grouped kernel field
class GroupedControls:
    """The members of a ``TupleControl`` of built-in controls as ``tcde_spline_eval_grouped`` reads them."""

    def __init__(self, controls, device):
        self.members = []
        for X in controls:
            kind, batch, channels, n_rows = _control_signature(X)
            rows = (X._rows() if kind == _lib.CONTROL_CUBIC else X._coeffs).detach()
            flat = rows.reshape(-1, rows.size(-2), rows.size(-1)).contiguous()
            knots = X._t.detach().to(device=device, dtype=rows.dtype).contiguous()
            self.members.append((X, kind, batch, channels, n_rows, flat, knots))
        self.dtype = self.members[0][5].dtype

    def evaluate(self, index, frac):
        """dX/dt of member k at the queries ``index[k]`` (int32) / ``frac[k]`` (device, 1-D) in ONE launch; returns the
        tensors (*batch_k, n_times_k, C_k)."""
        outs = []
        descs = (_lib.SplineMember * len(self.members))()
        for d, (X, kind, batch, channels, _, flat, knots), idx, fr in zip(descs, self.members, index, frac):
            out = torch.empty(flat.size(0), idx.numel(), channels, dtype=flat.dtype, device=flat.device)
            d.control, d.knot_t, d.index, d.frac, d.out = (flat.data_ptr(), knots.data_ptr(), idx.data_ptr(),
                                                           fr.data_ptr(), out.data_ptr())
            d.n_paths, d.n_rows, d.channels, d.n_times, d.control_kind = (flat.size(0), flat.size(-2), channels,
                                                                          idx.numel(), kind)
            if out.numel() == 0:
                d.control = d.knot_t = d.index = d.frac = d.out = None
            outs.append(out.view(*batch, idx.numel(), channels))
        with torch.cuda.device(self.members[0][5].device):
            _lib.call("tcde_spline_eval_grouped", descs, len(self.members), 1, _lib.dtype_code(self.dtype),
                      _lib.stream_of(self.members[0][5]))
        return outs


def _apply_field(func, is_prod, ts, zs, dxs, stage, packing, out, sign):
    """``out`` (packed) <- sign * tuple(f_i @ dX_i) at ``stage`` of the per-member dX/dt blocks ``dxs`` (*B_i, S, C_i): ONE
    launch of ``tcde_field_contract_grouped`` for every member whose ``f_i`` is the plain (*B_i, H_i, C_i) tensor; a member
    with an unusual output (other shape or dtype, broadcasting) gets the torch contraction, alone."""
    parts = packing.views(out)
    dx_at = tuple(d[..., stage, :] for d in dxs)
    if is_prod:
        res = func.prod(ts, zs, dx_at)
        for p, r in zip(parts, res):
            p.copy_(r if sign > 0 else -1.0 * r)
        return out
    fs = func(ts, zs)
    descs = []
    for f, d, z, p in zip(fs, dxs, zs, parts):
        if z.numel() == 0:
            continue
        channels = d.size(-1)
        if (f.shape != z.shape + (channels,) or f.dtype != out.dtype or d.dtype != out.dtype or not f.is_cuda
                or d.shape[:-2] != z.shape[:-1]):
            r = (f @ d[..., stage, :].unsqueeze(-1)).squeeze(-1)          # let torch broadcast / promote
            p.copy_(r if sign > 0 else -1.0 * r)
            continue
        f = f if f.is_contiguous() else f.contiguous()
        descs.append((f, d.data_ptr() + stage * channels * d.element_size(), p.data_ptr(), z.numel() // z.size(-1),
                      z.size(-1), channels, d.size(-2) * channels))
    if descs:
        arr = (_lib.ContractMember * len(descs))()
        for a, (f, dx_ptr, out_ptr, n_paths, hidden, channels, stride) in zip(arr, descs):
            a.field, a.dx, a.out = f.data_ptr(), dx_ptr, out_ptr
            a.n_paths, a.hidden, a.channels, a.dx_stride = n_paths, hidden, channels, stride
        _lib.call("tcde_field_contract_grouped", arr, len(descs), float(sign), _lib.dtype_code(out.dtype),
                  _lib.stream_of(out))
    return out


# ---------------------------------------------------------------------------- no gradient, fixed step: grouped loop
_graphs = {}


def grouped_solve(X, func, z0, t, method, step_size, is_prod, packing, use_graph=False):
    """The fixed-step stage loop of a tuple state (the tuple form of ``solver._generic_solve_kernels``).  ``z0``: the
    packed state.  Returns (len(t), numel)."""
    dtype, device = z0.dtype, z0.device
    gc = GroupedControls(list(X.controls), device)
    scheds = [build_schedule(t, _schedule_knots(m[0]), m[4], method, step_size, dtype) for m in gc.members]
    sched = scheds[0]          # grid, stage times, outputs: the same for every member (they depend on t only)
    index_dev = [s.stage_index.to(device=device, dtype=torch.int32) for s in scheds]
    frac_dev = [s.stage_frac.to(device=device, dtype=gc.dtype) for s in scheds]
    times_dev = sched.stage_times.to(device)
    sign = sched.sign
    from .adaptive import _combine

    def run(y0):
        outs = [None] * sched.n_out
        j = 0
        while j < sched.n_out and int(sched.out_step[j]) < 0:
            outs[j] = y0
            j += 1
        y = y0
        for i in range(sched.n_steps):
            dxs = gc.evaluate([ix[i] for ix in index_dev], [fr[i] for fr in frac_dev])       # every member, every stage

            def field(s, z):
                return _apply_field(func, is_prod, times_dev[i, s], packing.views(z), dxs, s, packing,
                                    torch.empty_like(z), sign)

            dt = float(sched.step_dt[i])
            if method == "rk4":
                k1 = field(0, y)
                k2 = field(1, _combine(y, [k1], (1 / 3,), dt))
                k3 = field(2, _combine(y, [k1, k2], (-1 / 3, 1.0), dt))
                k4 = field(3, _combine(y, [k1, k2, k3], (1.0, -1.0, 1.0), dt))
                y1 = _combine(y, [k1, k2, k3, k4], (0.125, 0.375, 0.375, 0.125), dt)
            elif method == "midpoint":
                k1 = field(0, y)
                y1 = _combine(y, [field(1, _combine(y, [k1], (0.5,), dt))], (1.0,), dt)
            else:
                y1 = _combine(y, [field(0, y)], (1.0,), dt)
            while j < sched.n_out and int(sched.out_step[j]) == i:
                mode = int(sched.out_mode[j])
                outs[j] = y if mode == 0 else y1 if mode == 1 else _combine(y, [y1, y], (1.0, -1.0), float(sched.out_slope[j]))
                j += 1
            y = y1
        return torch.stack(outs, dim=0)

    zc = z0.detach().contiguous()
    if not use_graph:
        return run(zc)
    # the cache key of solver._generic_solve_kernels, over every member: what a replay cannot see change
    modules = list(func.modules()) if isinstance(func, torch.nn.Module) else []
    read = [x for m in modules for x in m.parameters(recurse=False)] + \
        [x for m in modules for x in m.buffers(recurse=False)] + list(X.buffers())
    key = (id(func), id(X), tuple(packing.shapes), dtype, str(device), method, step_size,
           tuple(float(v) for v in t.detach().cpu().tolist()), tuple(m.training for m in modules),
           tuple((x.data_ptr(), tuple(x.shape), x.dtype) for x in read))
    hit = _graphs.get(key)
    if hit is None:
        static_in = zc.clone()
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):                      # warm-up outside the capture (lazy initialisations)
            run(static_in)
        torch.cuda.current_stream(device).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = run(static_in)
        hit = (graph, static_in, static_out, func, X, run, read)
        if len(_graphs) >= 8:
            _graphs.clear()
        _graphs[key] = hit
    graph, static_in, static_out = hit[:3]
    static_in.copy_(zc)
    graph.replay()
    return static_out.clone()


def grouped_field(X, func, is_prod, packing, dtype, device):
    """``field(t_float, y_packed, nudge=0)`` of the host-driven dopri5: each member's interval and fraction from its own
    host locator, then one grouped evaluation and one grouped contraction."""
    gc = GroupedControls(list(X.controls), device)
    locators = [host_locator(_schedule_knots(m[0]), m[4], dtype) for m in gc.members]

    def field(t, y, nudge=0):
        ts = torch.tensor(float(t), dtype=torch.float64).to(dtype).to(device)
        if nudge:
            ts = torch.nextafter(ts, ts + 1)
        where = [loc(float(t), nudge) for loc in locators]
        index = torch.tensor([w[0] for w in where], dtype=torch.int32).to(device)
        frac = torch.tensor([w[1] for w in where], dtype=torch.float64).to(gc.dtype).to(device)
        dxs = gc.evaluate([index[k:k + 1] for k in range(len(where))], [frac[k:k + 1] for k in range(len(where))])
        return _apply_field(func, is_prod, ts, packing.views(y), dxs, 0, packing, torch.empty_like(y), 1.0)

    return field


def torch_field(X, func, is_prod, packing, dtype):
    """The reference's ``_VectorField.forward`` on the packed state as differentiable torch ops (``X.derivative``)."""
    prod = _PackedProd(func, is_prod, packing)

    def field(t, y, nudge=0):
        ts = t.to(device=y.device, dtype=dtype) if isinstance(t, torch.Tensor) else \
            torch.tensor(t, dtype=torch.float64).to(dtype).to(y.device)
        if nudge:
            ts = torch.nextafter(ts, ts + 1)
        return prod.prod(ts, y, X.derivative(ts))

    return field


# ----------------------------------------------------------------------------------------------------- the driver
def cdeint_tuple(X, func, z0, t, adjoint, kwargs, method, step_size, use_graph, options, times, flipped, is_prod):
    """``solver.cdeint`` for a tuple / list ``z0`` (after its argument parsing).  Returns the reference's output tuple."""
    from .solver import _generic_solve, _shape_error_forward, _shape_error_prod
    check_compatability(X, func, z0, t, is_prod, _shape_error_forward, _shape_error_prod)
    _lib.require_cuda(*z0)
    packing = Packing(z0)
    y0 = packing.pack(z0)
    dtype, device = y0.dtype, y0.device
    controls = list(X.controls) if isinstance(X, TupleControl) else None
    built_in = (controls is not None and y0.is_cuda and dtype in (torch.float32, torch.float64)
                and all(_control_signature(m) is not None for m in controls)
                and all(b.device == device and b.dtype == dtype for m in controls for b in m.buffers()))

    if 'adjoint_params' in kwargs:
        adjoint_params = tuple(kwargs['adjoint_params'])
    else:
        adjoint_params = tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()
    differentiable = tuple(z0) + (t,) + (tuple(X.buffers()) if isinstance(X, torch.nn.Module) else ()) + \
        (tuple(func.parameters()) if isinstance(func, torch.nn.Module) else ()) + adjoint_params
    wants_grad = torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad
                                                 for x in differentiable)
    rtol, atol = kwargs['rtol'], kwargs['atol']
    prod = _PackedProd(func, is_prod, packing)

    def forward_values(v0):
        """Outputs only, time first, packed: (len(t), numel)."""
        if method in FIXED_METHODS:
            if built_in and not torch.is_grad_enabled():
                return grouped_solve(X, func, v0, t, method, step_size, is_prod, packing, use_graph)
            return _generic_solve(X, prod, v0, t, method, step_size, True, False)
        field = grouped_field(X, func, is_prod, packing, dtype, device) if built_in and not torch.is_grad_enabled() \
            else torch_field(X, func, is_prod, packing, dtype)
        out, solver_obj = adaptive.odeint_dopri5(_reverse(field) if flipped else field, v0, times, rtol, atol, options,
                                                 norm=adaptive.tuple_norm(packing.sizes))
        from .solver import cdeint
        cdeint.last_stats = {"n_accepted": solver_obj.n_accepted, "n_rejected": solver_obj.n_rejected,
                             "device_controlled": False}
        return out

    if not wants_grad:
        with torch.no_grad():
            return packing.outputs(forward_values(y0))

    def autograd_field():
        f = torch_field(X, func, is_prod, packing, dtype)
        return _reverse(f) if flipped else f

    if adjoint:
        a_rtol, a_atol = kwargs["adjoint_rtol"], kwargs["adjoint_atol"]
        a_method = kwargs.get("adjoint_method", None) or method
        a_options = dict(kwargs.get("adjoint_options", None) or ({"step_size": step_size} if step_size else {}))
        t_grad = t if t.requires_grad else None
        n_params = sum(p.numel() for p in adjoint_params if p.requires_grad and p is not t_grad)

        def solve_aug(f, v, ts):
            if a_method in FIXED_METHODS:
                return adaptive.odeint_fixed(f, v, ts, a_method, a_options.get("step_size", None))
            # the augmented state (a_t?, y, a, params): the tuple norm on y and on a, the RMS of the rest
            lead = v.numel() - 2 * packing.numel - n_params
            sizes = ([lead] if lead else []) + packing.sizes + packing.sizes + ([n_params] if n_params else [])
            return adaptive.odeint_dopri5(f, v, ts, a_rtol, a_atol, norm=adaptive.tuple_norm(sizes))[0]

        ys = adaptive.solve_with_adjoint(forward_values, autograd_field(), times, solve_aug, y0, adjoint_params,
                                         None, None, t_grad, flipped)
        return packing.outputs(ys)

    # adjoint=False: backpropagate through the solver's own operations, like torchdiffeq.odeint
    if method in FIXED_METHODS:
        return packing.outputs(_generic_solve(X, prod, y0, t, method, step_size, True, False))
    targets = (-t if flipped else t).to(device) if t.requires_grad else None
    ys = adaptive.odeint_dopri5(autograd_field(), y0, times, rtol, atol, options, targets,
                                norm=adaptive.tuple_norm(packing.sizes))[0]
    return packing.outputs(ys)
