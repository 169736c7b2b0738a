"""The autograd shell of the adjoint=False kernel routes (``torchcde_b200.backprop``) on the CPU, with a pure-torch route
in place of the kernels: where the gradients land, which backward runs, when the record is freed, and how a route
declines."""
import weakref

import pytest
import torch

from torchcde_b200 import backprop


class _Route:
    """out = z0 @ w + b, with b optional; the record is a copy of z0.  The backward is the hand-written vjp."""

    def __init__(self, w, b, decline=None):
        self.w, self.b, self.decline = w, b, decline
        self.records, self.backwards, self.differentiated = [], 0, 0

    def forward(self, z0):
        if self.decline is not None:
            raise self.decline
        record = z0.detach().clone()
        self.records.append(weakref.ref(record))
        out = record @ self.w.detach()
        if self.b is not None:
            out = out + self.b.detach()
        return out, [record, None]

    def backward(self, g, z0, saved, want):
        record, nothing = saved
        assert nothing is None and torch.equal(record, z0)
        self.backwards += 1
        gw = record.t() @ g if want[0] else None
        gb = g.sum(0) if want[1] else None
        return g @ self.w.detach().t(), [gw, gb]

    def differentiable(self, z0):
        self.differentiated += 1
        return z0 @ self.w + (self.b if self.b is not None else 0)


def _leaves(bias=True, want_w=True):
    gen = torch.Generator().manual_seed(0)
    z0 = torch.randn(5, 3, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(3, 4, generator=gen, dtype=torch.float64, requires_grad=want_w)
    b = torch.randn(4, generator=gen, dtype=torch.float64, requires_grad=True) if bias else None
    return z0, w, b


def _no_autograd(monkeypatch):
    def refuse(*args, **kwargs):
        raise AssertionError("autograd ran in the backward")
    monkeypatch.setattr(torch.autograd, "grad", refuse)


@pytest.mark.parametrize("bias,want_w", [(True, True), (False, True), (True, False)])
def test_gradients_land_on_their_inputs(bias, want_w, monkeypatch):
    """A missing bias (None) and a parameter that wants no gradient get none; the others get the route's."""
    z0, w, b = _leaves(bias, want_w)
    route = _Route(w, b)
    out = backprop.run(route, z0, [w, b])
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    with monkeypatch.context() as m:
        _no_autograd(m)
        out.backward(g)
    assert type(out.grad_fn).__name__ == "_RouteFnBackward" and out.grad_fn.route is route
    assert route.backwards == 1 and route.differentiated == 0
    assert torch.equal(z0.grad, g @ w.detach().t())
    assert (w.grad is not None) == want_w
    if want_w:
        assert torch.equal(w.grad, z0.detach().t() @ g)
    if b is not None:
        assert torch.equal(b.grad, g.sum(0))


def test_create_graph_differentiates_the_torch_solve():
    z0, w, b = _leaves()
    route = _Route(w, b)
    out = backprop.run(route, z0, [w, b])
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    gz, gw = torch.autograd.grad(out, (z0, w), g, create_graph=True)
    assert route.differentiated == 1 and route.backwards == 0
    assert gz.requires_grad and torch.allclose(gz, g @ w.detach().t())
    (second,) = torch.autograd.grad(gz.pow(2).sum(), w)
    assert torch.allclose(second, 2 * (g @ w.detach().t()).t() @ g)


def test_backward_frees_the_record_while_the_outputs_live():
    z0, w, b = _leaves()
    route = _Route(w, b)
    out = backprop.run(route, z0, [w, b])
    g = torch.ones_like(out)
    out.backward(g, retain_graph=True)                   # retain_graph keeps the record for a second backward
    assert route.records[0]() is not None
    out.backward(g)
    assert route.backwards == 2 and route.records[0]() is None
    assert torch.equal(z0.grad, 2 * (g @ w.detach().t()))


@pytest.mark.parametrize("decline", [backprop.NoRoom(), NotImplementedError("not built")], ids=["no_room", "not_built"])
def test_a_declining_forward_returns_none(decline):
    z0, w, b = _leaves()
    assert backprop.run(_Route(w, b, decline), z0, [w, b]) is None
