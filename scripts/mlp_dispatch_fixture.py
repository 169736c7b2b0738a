#!/usr/bin/env python
"""The verdicts of the MLP field's C dispatch, for tests/golden/mlp_dispatch.npz and tests/test_mlp_dispatch_cpu.py.

    python scripts/mlp_dispatch_fixture.py OUT.npz

Every entry point of solve_mlp.cu is called with no paths, so each call validates its arguments, consults the route
policy and returns before any launch: no device is needed, and nothing runs on one where there is.  One small buffer
stands in for every pointer.  Recorded, at solve variants 0 to 6:
  * rc/<entry>: the return code over hidden x channels x width x dtype (fp32, fp64, an invalid code) x variant;
  * edge/<entry>: the largest admitted width below 2^20 (0 if none) per hidden x channels x dtype x variant, found by
    bisection as tests/test_gpu_mlp_adjoint.py does: where each shared-memory bound lies;
  * align/<entry>: at the tensor-core shape (32, 8, 128) in fp32, the return code with each pointer argument in turn
    4 bytes off 16-byte alignment, per variant;
  * the two scratch queries' byte counts over n_paths x hidden x channels x width x variant, and their edges.
The scratch sizes scale with the SM count; sm_count holds the one they were made with (132 without a GPU)."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchcde_b200 import _lib  # noqa: E402

HIDDEN = (1, 4, 5, 8, 9, 16, 32, 33)
CHANNELS = (1, 2, 3, 4, 5, 8, 14)
WIDTH = (1, 37, 48, 128, 129, 366, 1 << 20)
DTYPES = (_lib.F32, _lib.F64, 7)
VARIANTS = tuple(range(7))
SCRATCH_PATHS = (0, 1000, 100000)
TC_SHAPE = (32, 8, 128)

# The argument lists, one token per argument: P a pointer, H / C / W the shape, D the dtype; every other token a fixed
# value (the rest of a call that every check passes, with n_paths = 0 as N)
VALUES = {"K": _lib.CONTROL_CUBIC, "R": 4, "N": 0, "M": _lib.METHODS["rk4"], "S": 4, "O": 2, "G": 1.0, "T": 4, "I": 1,
          "F": 0.5, "E": 1.0, "Q": 2, "L": 0, "X": None}
ENTRIES = {
    "tcde_cdeint_fixed_mlp": "P K R P P P P P P N C H W M S P P P O P P P G D X",
    "tcde_cdeint_fixed_mlp_stages": "P K R P P P P P P P N C H W M S P P P O P P P G D X",
    "tcde_cdeint_fixed_mlp_backward": "P K R P P P P P P P P N C H W M S P P P O P P P G D X",
    "tcde_mlp_field_param_grads": "P K R P P P P P P P P T P P P P P N C H W G E D X",
    "tcde_vector_field_mlp": "P K R P P P P P P N C H W I F D X",
    "tcde_vector_field_mlp_vjp": "P K R P P P P P P P P P P P P P N C H W I F E E E D X",
    "tcde_cdeint_reversible_heun_mlp": "P K R P P P P P P P Q N C H W S P P P O P P D X",
    "tcde_reversible_heun_mlp_backward_segment": "P K R P P P P P P P P O P P P S P P P L S N C H W P P D X",
    "tcde_dopri5_mlp_backward": "P K R P P P P P P P P P P P P P P P O S N C H W G D X",
}
SCRATCH = {
    "tcde_mlp_field_param_grads_scratch_bytes": "N T C H W",
    "tcde_vector_field_mlp_vjp_scratch_bytes": "N C H W",
}


class Caller:
    def __init__(self):
        self.lib = _lib.load()
        self.buf = ctypes.create_string_buffer(256)
        self.base = (ctypes.addressof(self.buf) + 15) & ~15

    def call(self, name, spec, shape, dtype=None, n_paths=0, skew=-1):
        hidden, channels, width = shape
        args, k = [], 0
        for tok in spec.split():
            if tok == "P":
                args.append(ctypes.c_void_p(self.base + (4 if k == skew else 0)))
                k += 1
            elif tok == "N":
                args.append(n_paths)
            else:
                args.append({"H": hidden, "C": channels, "W": width, "D": dtype}.get(tok, VALUES.get(tok)))
        return getattr(self.lib, name)(*args)

    def variant(self, v):
        assert self.lib.tcde_set_solve_variant(v) == 0


def _edge(admitted):
    """The largest width in [1, 2^20) that admitted(width) accepts, by bisection (0 if width 1 is refused)."""
    lo, hi = 0, 1 << 20
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if admitted(mid) else (lo, mid)
    return lo


def sm_count(lib):
    n = ctypes.c_int(0)
    return n.value if lib.tcde_device_info(ctypes.byref(n), None, None) == 0 else 132


def records():
    """{key: array} of every verdict (see the module docstring); restores solve variant 0"""
    c = Caller()
    out = {"sm_count": np.array(sm_count(c.lib))}
    grid = (len(HIDDEN), len(CHANNELS), len(WIDTH))
    try:
        for name, spec in ENTRIES.items():
            rc = np.zeros(grid + (len(DTYPES), len(VARIANTS)), np.int32)
            edge = np.zeros((len(HIDDEN), len(CHANNELS), len(DTYPES), len(VARIANTS)), np.int64)
            align = np.zeros((spec.split().count("P"), len(VARIANTS)), np.int32)
            for v in VARIANTS:
                c.variant(v)
                for (i, h), (j, ch), (d, dt) in _pairs(HIDDEN, CHANNELS, DTYPES):
                    for w_i, w in enumerate(WIDTH):
                        rc[i, j, w_i, d, v] = c.call(name, spec, (h, ch, w), dt)
                    edge[i, j, d, v] = _edge(lambda w: c.call(name, spec, (h, ch, w), dt) == 0)
                for p in range(align.shape[0]):
                    align[p, v] = c.call(name, spec, TC_SHAPE, _lib.F32, skew=p)
            out["rc/" + name], out["edge/" + name], out["align/" + name] = rc, edge, align
        for name, spec in SCRATCH.items():
            fn = getattr(c.lib, name)
            size = np.zeros((len(SCRATCH_PATHS),) + grid + (len(VARIANTS),), np.int64)
            edge = np.zeros((len(HIDDEN), len(CHANNELS), len(VARIANTS)), np.int64)
            for v in VARIANTS:
                c.variant(v)
                for (i, h), (j, ch), _ in _pairs(HIDDEN, CHANNELS, (None,)):
                    for w_i, w in enumerate(WIDTH):
                        for n_i, n in enumerate(SCRATCH_PATHS):
                            size[n_i, i, j, w_i, v] = c.call(name, spec, (h, ch, w), n_paths=n)
                    edge[i, j, v] = _edge(lambda w: c.call(name, spec, (h, ch, w), n_paths=1000) >= 0)
            out["bytes/" + name], out["edge/" + name] = size, edge
    finally:
        c.variant(0)
    return out


def _pairs(*axes):
    """every combination of the axes, each item as (index, value)"""
    for idx in np.ndindex(*(len(a) for a in axes)):
        yield tuple((k, a[k]) for k, a in zip(idx, axes))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    recs = records()
    np.savez_compressed(sys.argv[1], **recs)
    print("{} arrays, sm_count {}".format(len(recs), int(recs["sm_count"])))
