#!/usr/bin/env python
"""The verdicts of the C dispatch of the MLP and linear fields, for tests/golden/dispatch.npz and
tests/test_dispatch_cpu.py.

    python scripts/dispatch_fixture.py OUT.npz

Every entry point of solve_mlp.cu and of the linear field is called so that it validates its arguments, consults its
route policy and returns before any launch: with no paths where the entry point accepts none, else with no launches
(n_launches = 0) or no steps (n_steps = 0).  No device is needed, and nothing runs on one where there is.  One small
buffer stands in for every pointer.  Recorded for the MLP field, at solve variants 0 to 6:
  * rc/<entry>: the return code over hidden x channels x width x dtype (fp32, fp64, an invalid code) x variant;
  * edge/<entry>: the largest admitted width below 2^20 (0 if none) per hidden x channels x dtype x variant, found by
    bisection as tests/test_gpu_mlp_adjoint.py does: where each shared-memory bound lies;
  * align/<entry>: at the tensor-core shape (32, 8, 128) in fp32, the return code with each pointer argument in turn
    4 bytes off 16-byte alignment, per variant;
  * the two scratch queries' byte counts over n_paths x hidden x channels x width x variant, and their edges.
For the linear field, at solve variants 0 to 6, each return code with the last-error text of a refused call (msg/...):
  * rc/<entry>: over hidden x channels x dtype (fp32, fp64, an invalid code) x variant;
  * args/<entry>: at fp32 32 / 8, over control kind (cubic, linear, invalid) x method (every code and an invalid one;
    entry points without one ignore it) x variant;
  * null/<entry>, align/<entry>: at fp32 32 / 8, each pointer argument in turn null, or 4 bytes off 16-byte
    alignment, per variant;
  * batch/<entry>: the dopri5 entry points at batches of 255, 256 and 512 paths, per variant;
  * the byte counts of the two scratch queries and tcde_dopri5_linear_grid.
A call that needs the device after its checks (the dopri5 attempts set their kernel's shared-memory limit) fails with
TCDE_ERR_CUDA where there is none; it is recorded as admitted.  The scratch sizes and the dopri5 grid scale with the
SM count; sm_count holds the one they were made with (132 without a GPU)."""
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

LINEAR_HIDDEN = (1, 8, 16, 31, 32, 33, 256, 257)
LINEAR_CHANNELS = (1, 4, 7, 8, 9, 32)
LINEAR_SHAPE = (32, 8)
KINDS = (_lib.CONTROL_CUBIC, _lib.CONTROL_LINEAR, 5)
METHOD_CODES = (0, 1, 2, _lib.REVERSIBLE_HEUN, 9)
BATCHES = (255, 256, 512)
CUDA_ERROR = -3
# as VALUES, and B the batch of the dopri5 entry points (which take no empty batch), Z their n_launches / n_steps,
# L / U a backward segment's lo / hi, Y the slots of a dopri5 record
LINEAR_VALUES = dict(VALUES, B=256, Z=0, U=4, Y=4)
LINEAR = {
    "tcde_vector_field_linear": "P K R P P P P N C H I F D X",
    "tcde_vector_field_linear_vjp": "P K R P P P P P P P P P N C H I F E E E D X",
    "tcde_cdeint_fixed_linear": "P K R P P P P N C H M S P P P O P P P G D X",
    "tcde_cdeint_fixed_linear_stages": "P K R P P P P P N C H M S P P P O P P P G D X",
    "tcde_cdeint_fixed_linear_backward": "P K R P P P P P N C H M S P P P O P P P G D X",
    "tcde_cdeint_reversible_heun_linear": "P K R P P P P P Q N C H S P P P O P P D X",
    "tcde_reversible_heun_linear_backward_segment": "P K R P P P P P P P P O P P P P P P L U N C H P P D X",
    "tcde_linear_field_param_grads": "P K R P P P P P T P P P N C H G D X",
    "tcde_dopri5_linear_attempts": "P K R P P P P P P P P O B C H G L Z D X",
    "tcde_dopri5_linear_paired_attempts": "P K R P P P P P P P P P P O B C H G P P P P P Y L Z D X",
    "tcde_dopri5_linear_record_attempts": "P K R P P P P P P P P O B C H G P P P P Y L Z D X",
    "tcde_dopri5_linear_backward": "P K R P P P P P P P P P P P O Z B C H G D X",
}
SCRATCH_STAGES = (0, 1, 7)
GRID_PATHS = (-1, 0, 1, 255, 256, 257, 100000, 10 ** 7)


class Caller:
    def __init__(self):
        self.lib = _lib.load()
        self.buf = ctypes.create_string_buffer(256)
        self.base = (ctypes.addressof(self.buf) + 15) & ~15
        self.has_device = self.lib.tcde_device_info(None, None, None) == 0

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

    def verdict(self, name, spec, shape, dtype=None, n_paths=0, skew=-1, null=-1, **values):
        """(return code, last-error text of a refusal) of a linear entry point; values override fixed tokens"""
        hidden, channels = shape
        args, k = [], 0
        for tok in spec.split():
            if tok == "P":
                args.append(None if k == null else ctypes.c_void_p(self.base + (4 if k == skew else 0)))
                k += 1
            elif tok == "N":
                args.append(n_paths)
            elif tok in values:
                args.append(values[tok])
            else:
                args.append({"H": hidden, "C": channels, "D": dtype}.get(tok, LINEAR_VALUES.get(tok)))
        rc = getattr(self.lib, name)(*args)
        if rc == CUDA_ERROR and not self.has_device:
            rc = 0
        return rc, ("" if rc == 0 else self.lib.tcde_last_error().decode())


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
        out.update(linear_records(c))
    finally:
        c.variant(0)
    return out


def linear_records(c):
    """the linear field's verdicts (see the module docstring) at the solve variant c was left in and 0 to 6"""
    out = {}
    for name, spec in LINEAR.items():
        n_ptr = spec.split().count("P")
        tables = {"rc": (len(LINEAR_HIDDEN), len(LINEAR_CHANNELS), len(DTYPES)), "args": (len(KINDS), len(METHOD_CODES)),
                  "null": (n_ptr,), "align": (n_ptr,)}
        if "B" in spec:
            tables["batch"] = (len(BATCHES),)
        got = {key: (np.zeros(dims + (len(VARIANTS),), np.int32), np.zeros(dims + (len(VARIANTS),), object))
               for key, dims in tables.items()}

        def put(key, idx, verdict):
            got[key][0][idx], got[key][1][idx] = verdict

        for v in VARIANTS:
            c.variant(v)
            for (i, h), (j, ch), (d, dt) in _pairs(LINEAR_HIDDEN, LINEAR_CHANNELS, DTYPES):
                put("rc", (i, j, d, v), c.verdict(name, spec, (h, ch), dt))
            for (i, kind), (j, method) in _pairs(KINDS, METHOD_CODES):
                put("args", (i, j, v), c.verdict(name, spec, LINEAR_SHAPE, _lib.F32, K=kind, M=method))
            for p in range(n_ptr):
                put("null", (p, v), c.verdict(name, spec, LINEAR_SHAPE, _lib.F32, null=p))
                put("align", (p, v), c.verdict(name, spec, LINEAR_SHAPE, _lib.F32, skew=p))
            for i, b in enumerate(BATCHES if "batch" in tables else ()):
                put("batch", (i, v), c.verdict(name, spec, LINEAR_SHAPE, _lib.F32, B=b))
        for key, (rc, msg) in got.items():
            out[key + "/" + name], out[key + "msg/" + name] = rc, msg.astype(str)
    vjp_bytes = np.zeros((len(SCRATCH_PATHS) + 1, len(LINEAR_HIDDEN), len(LINEAR_CHANNELS)), np.int64)
    pg_bytes = np.zeros(vjp_bytes.shape[:1] + (len(SCRATCH_STAGES),) + vjp_bytes.shape[1:], np.int64)
    for (n_i, n), (i, h), (j, ch) in _pairs((-1,) + SCRATCH_PATHS, LINEAR_HIDDEN, LINEAR_CHANNELS):
        vjp_bytes[n_i, i, j] = c.lib.tcde_vector_field_linear_vjp_scratch_bytes(n, ch, h)
        for t_i, t in enumerate(SCRATCH_STAGES):
            pg_bytes[n_i, t_i, i, j] = c.lib.tcde_linear_field_param_grads_scratch_bytes(n, t, ch, h)
    out["bytes/tcde_vector_field_linear_vjp_scratch_bytes"] = vjp_bytes
    out["bytes/tcde_linear_field_param_grads_scratch_bytes"] = pg_bytes
    out["grid/tcde_dopri5_linear_grid"] = np.array([c.lib.tcde_dopri5_linear_grid(n) for n in GRID_PATHS], np.int64)
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
