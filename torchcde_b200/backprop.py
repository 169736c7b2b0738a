"""What the ``cdeint(..., adjoint=False)`` kernel routes share: one autograd shell, one memory bound, the cotangent layout.

A route is any object with
  * ``forward(z0) -> (out, saved)``: the solve's outputs and the tensors its backward needs (the record; None entries
    allowed); it raises ``NoRoom`` or ``NotImplementedError`` before anything the caller can see has run;
  * ``backward(g, z0, saved, want) -> (dL/dz0, [dL/dp or None for p in params])``, ``want[i]`` telling whether params[i]
    wants a gradient;
  * ``differentiable(z0)``: the torch-operator solve of the same problem, which a backward with ``create_graph``
    differentiates instead (the kernels give no higher-order derivatives)."""
import functools

import torch


class NoRoom(Exception):
    """The record of a route's forward would not fit in the device memory."""


def fits(device, record_bytes, scratch_bytes=None):
    """Whether a record of ``record_bytes`` fits in 0.7 of the free memory of ``device``; with a parameter gradient
    (``scratch_bytes`` not None), the record, its kappa copy and the parameter-gradient scratch (a negative size: the
    kernel is not built for the problem)."""
    need = record_bytes
    if scratch_bytes is not None:
        if scratch_bytes < 0:
            return False
        need = 2 * record_bytes + scratch_bytes
    with torch.cuda.device(device):
        free, _total = torch.cuda.mem_get_info()
    return need <= 0.7 * free


def cotangent(g, n_out, hidden):
    """The output gradients ``g`` as ``(paths, n_out, hidden)``: contiguous and 16-byte aligned, as the kernels read them."""
    gf = g.reshape(-1, n_out, hidden)
    if not gf.is_contiguous() or gf.data_ptr() % 16:
        gf = gf.clone(memory_format=torch.contiguous_format)
    return gf


class _Backprop(torch.autograd.Function):
    @staticmethod
    def forward(ctx, route, z0, *params):
        out, saved = route.forward(z0)
        ctx.route = route                      # host-side metadata only: the record goes through save_for_backward, so a
        ctx.save_for_backward(z0, *params, *saved)                                      # backward frees it
        return out

    @staticmethod
    def backward(ctx, g):
        z0, *rest = ctx.saved_tensors
        want_z, *want = ctx.needs_input_grad[1:]
        params, saved = rest[:len(want)], rest[len(want):]
        if torch.is_grad_enabled():
            # create_graph: differentiate the torch-operator solve of the same problem, whose gradients are themselves
            # differentiable
            inputs = [x for x, w in zip([z0] + params, [want_z] + want) if w]
            got = iter(torch.autograd.grad(ctx.route.differentiable(z0), inputs, g, create_graph=True,
                                           allow_unused=True))
            return (None,) + tuple(next(got) if w else None for w in [want_z] + want)
        gz, grads = ctx.route.backward(g, z0, saved, want)
        return (None, gz if want_z else None) + tuple(grads)


@functools.cache
def _shell(route_class):
    """The shell under the route's own name: the outputs' ``grad_fn`` is a ``_<Route>FnBackward``."""
    return type("_{}Fn".format(route_class.__name__.lstrip("_")), (_Backprop,), {})


def run(route, z0, params):
    """The outputs of ``route``'s solve of ``z0``, differentiable in ``z0`` and ``params`` (a None entry stands for a
    missing bias), or None when the forward declines the problem: nothing the caller can see has run, so it runs the
    torch-operator solve from the start."""
    try:
        return _shell(type(route)).apply(route, z0, *params)
    except (NoRoom, NotImplementedError):
        return None
