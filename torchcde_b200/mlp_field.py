"""The MLP vector field of the reference's examples and ``MlpFieldKernels``, the owner of its fused fixed-step solve.

example/time_series_classification.py:20-51 trains ``func(t, z) = tanh(Linear(W, H*C)(relu(Linear(H, W)(z)))).view(H, C)``.
``mlp_field_of`` recognises a user module that computes exactly that (no new class to adopt), and ``cdeint`` then runs
its fixed-step forward as ONE launch of ``tcde_cdeint_fixed_mlp``."""
import math
import weakref

import torch

from . import _lib
from .controls import _control_signature, _schedule_knots
from .linear_field import _check_linear_problem, _probe, _schedules

# module -> {training flag: index of the accepted layer ordering, or -1}; kept apart from the linear probe's cache
_recognised = weakref.WeakKeyDictionary()
# submodules that hold no state and behave the same in training and evaluation mode
_STATELESS = (torch.nn.Linear, torch.nn.ReLU, torch.nn.Tanh, torch.nn.Identity, torch.nn.Sequential)


def _two_linears(func):
    """The orderings ``(L1, L2)`` of the two ``nn.Linear`` of ``func`` if its parameters are exactly theirs, it has no
    buffers and every other submodule is a ReLU, Tanh, Identity or Sequential (a Dropout or any module whose forward may
    depend on its mode or state is refused: the probe sees one mode only), otherwise []."""
    if not isinstance(func, torch.nn.Module) or hasattr(func, "prod"):
        return []
    if any(type(m) not in _STATELESS for m in func.modules() if m is not func):
        return []
    lins = [m for m in func.modules() if isinstance(m, torch.nn.Linear)]
    if len(lins) != 2 or len(list(func.buffers())) != 0:
        return []
    own = {id(p) for lin in lins for p in lin.parameters()}
    if {id(p) for p in func.parameters()} != own or len(own) != sum(len(list(lin.parameters())) for lin in lins):
        return []
    return [lins, lins[::-1]]


def _mlp(l1, l2):
    def field(z):
        return torch.tanh(torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(z, l1.weight, l1.bias)),
                                                     l2.weight, l2.bias))
    return field


def mlp_field_of(func, z0, channels, times):
    """Return ``(W1, b1, W2, b2)`` (a bias may be None) if ``func(t, z)`` is exactly
    ``tanh(F.linear(relu(F.linear(z, W1, b1)), W2, b2)).view(..., H, C)`` for two ``nn.Linear`` of ``func``, else None.

    Like ``linear_field_of``, the module is *probed*: it must reproduce that map bit for bit on random states at four
    times of the integration interval, so a module with another activation, no tanh, a dependence on ``t``, a scaled
    output or a third layer is never taken for it.  Both orderings of the two layers are tried when both fit the shapes.
    The outcome is cached per module and training flag."""
    hidden = z0.size(-1)
    fits = [(l1, l2) for l1, l2 in _two_linears(func) if l1.in_features == hidden
            and l2.in_features == l1.out_features and l2.out_features == hidden * channels]
    if not fits:
        return None
    if z0.numel() * channels > (1 << 27):
        return None                       # too large to probe at this batch size; not a verdict on the module
    # the verdict is kept per training flag: the module's own forward may branch on it
    try:
        verdicts = _recognised.setdefault(func, {})
    except TypeError:
        verdicts = {}
    known = verdicts.get(func.training)
    if known is None:
        known = next((i for i, (l1, l2) in enumerate(fits)
                      if _probe(func, _mlp(l1, l2), z0, channels, times, "a two-layer MLP", None)), -1)
        verdicts[func.training] = known
    if known < 0:
        return None
    l1, l2 = fits[known]
    return l1.weight, l1.bias, l2.weight, l2.bias


class MlpFieldKernels:
    """The fused fixed-step solve of one problem: a built-in control ``X``, the MLP field ``params = (W1, b1, W2, b2)``
    (a bias may be None: zeros are passed) and the state ``z0``.  Construction validates dtypes and devices."""

    def __init__(self, X, params, z0):
        w1, b1, w2, b2 = params
        self.kind, _, self.channels, self.n_rows = _control_signature(X)
        self.hidden, self.width = z0.size(-1), w1.size(0)
        self.n_paths = math.prod(z0.shape[:-1])
        self.dtype, self.device = z0.dtype, z0.device
        control = X._rows() if self.kind == _lib.CONTROL_CUBIC else X._derivs
        _check_linear_problem(control, w1, b1, z0)
        _check_linear_problem(control, w2, b2, z0)
        self.control = control.detach().reshape(-1, control.size(-2), control.size(-1)).contiguous()
        zeros = lambda n: torch.zeros(n, dtype=z0.dtype, device=z0.device)  # noqa: E731
        self.w1, self.w2 = w1.detach().contiguous(), w2.detach().contiguous()
        self.b1 = (b1.detach() if b1 is not None else zeros(self.width)).contiguous()
        self.b2 = (b2.detach() if b2 is not None else zeros(self.hidden * self.channels)).contiguous()
        self.knots = _schedule_knots(X)

    def solve(self, y0, t, method, step_size):
        """The fixed-step solve as ONE launch of ``tcde_cdeint_fixed_mlp``: ``(..., len(t), H)``.  Raises
        NotImplementedError for a shape or solve variant no kernel is built for."""
        with torch.cuda.device(self.device):
            zf = y0.detach().reshape(-1, self.hidden).contiguous()
            sched, (_floats, _ints, v) = _schedules.get(t, self.knots, self.n_rows, method, step_size, self.dtype,
                                                        self.device)
            out = torch.empty(zf.size(0), sched.n_out, self.hidden, dtype=self.dtype, device=self.device)
            if zf.size(0) > 0:            # an empty batch: nothing to launch (its null data pointers would be refused)
                _lib.call("tcde_cdeint_fixed_mlp", _lib.ptr(self.control), self.kind, self.n_rows, _lib.ptr(self.w1),
                          _lib.ptr(self.b1), _lib.ptr(self.w2), _lib.ptr(self.b2), _lib.ptr(zf), _lib.ptr(out),
                          zf.size(0), self.channels, self.hidden, self.width, _lib.METHODS[sched.method],
                          sched.n_steps, _lib.ptr(v["step_dt"]), _lib.ptr(v["stage_index"]), _lib.ptr(v["stage_frac"]),
                          sched.n_out, _lib.ptr(v["out_step"]), _lib.ptr(v["out_mode"]), _lib.ptr(v["out_slope"]),
                          float(sched.sign), _lib.dtype_code(self.dtype), _lib.stream_of(zf))
        return out.view(*y0.shape[:-1], sched.n_out, self.hidden)
