"""Every coefficient-builder kernel route (hermite.cu, natural.cu, fill.cu) against the oracle, bit for bit, at the tile,
alignment and width edges.

Which kernels ran is observed, not assumed: every case runs under ``torch.profiler`` (CUDA activity) and asserts the
list of ``tcde::`` kernels it launched.  That list is restated from the launchers' selection arithmetic
(``launch_hermite``, ``launch_fill_scan``, ``tcde_linear_fill``, ``launch_natural``) in ``_expected``; a kernel-internal
branch the profiler cannot see (128-bit or scalar loads, bulk or plain stores, packed pairs or scalar sweeps) is forced by
the inputs and named in the case id, and ``_natural_branch`` restates the condition so that the id cannot drift.

Comparators: ``_bits`` compares the int32 / int64 views (so ``-0.0 != +0.0``; a NaN matches any NaN).  The NaN-free
natural cubic multiplies by reciprocals: ``_series_ulps`` measures it in ulps of each (path, channel) series' own largest
coefficient, bar 64 ulp (256 on the "stiff" knots), beside the whole-tensor bar of ``test_gpu_builders``.  The reference
is ``oracle.cde_oracle``; the dense natural routes are also checked against ``natural_missing_kernel``, which runs
NaN-free data in the reference's exact operation order and is itself pinned to the per-series oracle bit for bit.
Every C-ABI call writes into a guard-banded buffer prefilled with a marked NaN: nothing outside the output may change
and nothing inside may keep the mark."""
import contextlib
import json
import os
import tempfile
import time

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import torchcde_b200 as cde
from oracle import cde_oracle as O
from torchcde_b200 import _lib, hostio

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64 = torch.float32, torch.float64
KT = 256                                      # kThreads of builders_common.cuh
INT = {F32: torch.int32, F64: torch.int64}
MARK = {F32: 0x7FC0BEEF, F64: 0x7FF80000DEADBEEF}   # quiet NaNs with a payload no kernel produces
PAD = 64                                      # guard elements on each side of an ABI output

ALL_KERNELS = {
    "hermite_vec4_kernel<true>", "hermite_vec4_kernel<false>",
    *("hermite_kernel<{}, {}>".format(T, U) for T in ("float", "double") for U in ("true", "false")),
    "natural_prep_kernel<float>", "natural_prep_kernel<double>", "natural_warp_kernel",
    "natural_win_kernel<float>", "natural_win_kernel<double>", "natural_kernel<float>", "natural_kernel<double>",
    *("natural_missing_kernel<{}, {}>".format(T, U) for T in ("float", "double") for U in ("true", "false")),
    *("linear_fill_kernel<{}, {}>".format(T, U) for T in ("float", "double") for U in ("true", "false")),
    *("linear_fill_warp_kernel<{}, {}>".format(T, U) for T in ("float", "double") for U in ("true", "false")),
    *("linear_fill_scan_kernel<{}, {}, {}>".format(T, U, o) for T in ("float", "double") for U in ("true", "false")
      for o in (0, 1)),
    *("hold_kernel<{}, {}>".format(T, R) for T in ("float", "double") for R in ("true", "false")),
    "nan_flag_kernel<float>", "nan_flag_kernel<double>",
}
_OBSERVED = set()
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\n[builder routes, worst of each check] " + "; ".join(
        "{}: {} (bar {})".format(k, v, b) for k, (v, b) in sorted(_WORST.items())))


def _report(route, what, value, bar):
    key = "{} {}".format(route, what)
    print("builder {}: {} (bar {})".format(key, value, bar))
    if value > _WORST.get(key, (-1, bar))[0]:
        _WORST[key] = (value, bar)
    assert value <= bar, (key, value, bar)


# ---- comparators -----------------------------------------------------------------------------------------------------
def _bits(got, want):
    """Number of elements whose bit patterns differ (a NaN matches any NaN; -0.0 does not match +0.0)."""
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    both_nan = torch.isnan(got) & torch.isnan(want)
    return int(((got.view(INT[got.dtype]) != want.view(INT[want.dtype])) & ~both_nan).sum())


def _series_ulps(got, want):
    """Worst error in ulps of each (path, channel) series' own scale, max |coefficient| over (interval, part)."""
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype
    assert bool((torch.isnan(got) == torch.isnan(want)).all())
    P, R, C4 = want.shape
    eps = torch.finfo(want.dtype).eps
    g = got.double().nan_to_num(0.0).reshape(P, R, 4, C4 // 4)
    w = want.double().nan_to_num(0.0).reshape(P, R, 4, C4 // 4)
    err = (g - w).abs().amax(dim=(1, 2))
    scale = w.abs().amax(dim=(1, 2))
    ulps = torch.where(err == 0, torch.zeros_like(err), err / (eps * scale))
    return float(ulps.max()) if ulps.numel() else 0.0


def _tensor_ulps(got, want):
    """The whole-tensor measure of test_gpu_builders: ulps of max(1, the tensor's largest |coefficient|)."""
    eps = torch.finfo(want.dtype).eps
    got, want = got.detach().cpu().double().nan_to_num(0.0), want.detach().cpu().double().nan_to_num(0.0)
    if want.numel() == 0:
        return 0.0
    return float((got - want).abs().max()) / (eps * max(1.0, float(want.abs().max())))


# ---- route observer --------------------------------------------------------------------------------------------------
def _kname(name):
    name = name[5:] if name.startswith("void ") else name
    name = name.replace("tcde::", "")
    depth = 0
    for i, ch in enumerate(name):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def _observe(fn, trace=False):
    """(result, names of the tcde kernels fn launched in order[, chrome-trace kernel events])."""
    for attempt in range(5):         # a session now and then returns no records; a builder call is safe to repeat
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA] + ([ProfilerActivity.CPU] if attempt else [])) as prof:
            torch.zeros(1, device=DEV)           # the session's first record is sometimes lost: spend it on a fill
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
        names = [_kname(e.name) for e in prof.events() if "tcde::" in e.name and e.device_type.name == "CUDA"]
        if names:
            break
        time.sleep(0.2)
    assert names, "the profiler recorded no tcde kernel"
    _OBSERVED.update(names)
    if not trace:
        return out, names
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and "tcde::" in e["name"]]
    return out, names, events


@contextlib.contextmanager
def _variant(v):
    _lib.call("tcde_set_natural_variant", v)
    try:
        yield
    finally:
        _lib.call("tcde_set_natural_variant", 0)


# ---- the selection arithmetic of the launchers, restated --------------------------------------------------------------
def _elem(dtype):
    return 4 if dtype == F32 else 8


def _T(dtype):
    return "float" if dtype == F32 else "double"


def _U(unit):
    return "true" if unit else "false"


def _scan_geometry(dtype, L, C, unit):
    """launch_fill_scan: (fits, G, shared bytes)."""
    if C > 32:
        return False, 0, 0
    e = _elem(dtype)
    n_chunks = 32 // C
    lg = 0
    while (1 << lg) * n_chunks < L:
        lg += 1
    G = 1 << lg
    nct = -(-L // G)
    bw = 128 // e
    padw = (C - G * C) % bw
    tile_words = (L * C + nct * padw + 3) & ~3
    smem = (0 if unit else ((L + 3) & ~3) * e) + 8 * tile_words * e
    return smem <= 100 * 1024 and lg < 11, G, smem


def _fill_route(dtype, L, C, unit, variant, flags):
    T, U = _T(dtype), _U(unit)
    if variant == 0 and _scan_geometry(dtype, L, C, unit)[0]:
        return ["linear_fill_scan_kernel<{}, {}, 0>".format(T, U)]
    ks = ["nan_flag_kernel<{}>".format(T)] if flags else []
    Lp = ((L + 31) // 32) * 32 + 1
    if L <= 256 and 8 * C * Lp * _elem(dtype) <= 72 * 1024 and variant != 1:
        return ks + ["linear_fill_warp_kernel<{}, {}>".format(T, U)]
    return ks + ["linear_fill_kernel<{}, {}>".format(T, U)]


def _hermite_route(dtype, C, unit, x_al, o_al):
    if dtype == F32 and C % 4 == 0 and C <= 512 and x_al and o_al:
        return ["hermite_vec4_kernel<{}>".format(_U(unit))]
    return ["hermite_kernel<{}, {}>".format(_T(dtype), _U(unit))]


def _natural_warp_wpc(L, C):
    C2 = C // 2
    n_chunks = 1 if C2 >= 32 else 32 // C2
    lg = 0
    while (1 << lg) * n_chunks < L:
        lg += 1
    G = 1 << lg
    nct = -(-L // G)
    padw = (C - G * C) % 32
    tile_words = L * C + nct * padw
    rows = 2 if C // 4 >= 32 else 64 // (C // 4)
    fixed = 2 * ((L + nct + 2) & ~1) * 8 + ((L + 1) & ~1) * 8
    per_warp = (2 * tile_words + rows * 4 * C) * 4
    wpc = (220 * 1024 - fixed) // per_warp if fixed < 220 * 1024 else 0
    return min(wpc, 12)


def _natural_branch(dtype, L, C, x_al=True, o_al=True, variant=0):
    """launch_natural: 'warp', 'win-{vec4,bulk,plain}-{pairs,scalar}', 'cta-S<n>-{bulk,plain}' or 'refused'."""
    e = _elem(dtype)
    rb = 4 * C * e
    TR = max(1, min(8192 // rb, L - 1))
    if dtype == F32 and C % 4 == 0 and L > 2 and x_al and o_al and variant == 0 and _natural_warp_wpc(L, C) >= 2:
        return "warp"
    Lpw = ((L + 31) // 32) * 32 + 1
    TRw = TR
    while TRw < L - 1 and TRw * max(C // 4, 1) < KT and 2 * TRw * rb <= 16384:
        TRw *= 2
    TRw = min(TRw, L - 1)
    direct = dtype == F32 and C % 4 == 0 and L > 2 and x_al and o_al
    smem_w = 2 * (1 if direct else TRw) * rb + (4 * L + 8) * e + 3 * C * Lpw * e + 16
    if smem_w <= 64 * 1024 and variant != 1:
        sweep = "pairs" if dtype == F32 and C % 2 == 0 else "scalar"
        return "win-{}-{}".format("vec4" if direct else ("bulk" if o_al else "plain"), sweep)
    cp = 1
    while cp < C and cp < 32:
        cp <<= 1
    Lp = ((L + 31) // 32) * 32 + 32 // cp
    per_path = 2 * (C * Lp + 1) * e
    fixed = 2 * TR * rb + 4 * L * e + 16
    S = (32 + C - 1) // C
    while S > 1 and fixed + S * per_path > 100 * 1024:
        S -= 1
    if fixed + S * per_path > 200 * 1024:
        return "refused"
    return "cta-S{}-{}".format(S, "bulk" if o_al else "plain")


def _natural_kernel(dtype, branch):
    if branch == "warp":
        return "natural_warp_kernel"
    return "{}<{}>".format("natural_win_kernel" if branch.startswith("win") else "natural_kernel", _T(dtype))


def _expected(api, dtype, L, C, unit, x_al=True, o_al=True, variant=0, nan=False):
    T, U = _T(dtype), _U(unit)
    if api in ("hermite", "series_abi"):
        if _scan_geometry(dtype, L, C, unit)[0]:
            return ["linear_fill_scan_kernel<{}, {}, 1>".format(T, U)]
        assert api == "hermite"
        return _fill_route(dtype, L, C, unit, variant, False) + _hermite_route(dtype, C, unit, True, True)
    if api == "hermite2":
        return _fill_route(dtype, L, C, unit, variant, False) + _hermite_route(dtype, C, unit, True, o_al)
    if api == "hermite_abi":
        return _hermite_route(dtype, C, unit, x_al, o_al)
    if api in ("fill", "fill_abi"):
        return _fill_route(dtype, L, C, unit, variant, True)
    if api in ("natural", "natural_abi"):
        branch = _natural_branch(dtype, L, C, x_al, o_al, variant)
        ks = ["natural_prep_kernel<{}>".format(T)]
        if branch != "refused":
            ks.append(_natural_kernel(dtype, branch))
        if api == "natural" and (nan or branch == "refused"):
            ks.append("natural_missing_kernel<{}, {}>".format(T, U))
        return ks
    if api == "missing_abi":
        return ["natural_missing_kernel<{}, {}>".format(T, U)]
    if api == "ffill":
        return ["hold_kernel<{}, false>".format(T)]
    if api == "rect_abi":
        return ["hold_kernel<{}, true>".format(T)]
    raise AssertionError(api)


def _last_L(pred, lo, hi):
    """The largest L in [lo, hi) with pred(L) true, pred being true at lo and false at hi (monotone)."""
    assert pred(lo) and not pred(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _knots(kind, L, dtype):
    if kind == "unit":
        return None
    gen = torch.Generator().manual_seed(L)
    if kind == "uneven":
        t = (torch.rand(L, generator=gen, dtype=F64) + 0.1).cumsum(0)
    elif kind == "stiff":                                      # spacings over three decades
        t = (10.0 ** (3 * torch.rand(L, generator=gen, dtype=F64) - 2)).cumsum(0)
    else:                                                      # "f32grid": a float32 grid, widened exactly in fp64
        t = torch.arange(L, dtype=F32) * 0.1
    return t.to(dtype)


def _data(kind, shape, dtype, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=gen, dtype=F64)
    if kind == "zeros":                                        # signed zeros and runs of equal observations
        x = torch.where(torch.rand(shape, generator=gen) < 0.5, torch.full_like(x, -0.0), torch.zeros_like(x))
        x = torch.where(torch.rand(shape, generator=gen) < 0.2, torch.full_like(x, 1.5), x)
    elif kind == "subnormal":
        x = x * (2.0 ** -135 if dtype == F32 else 2.0 ** -1040)
    elif kind == "huge":                                       # near overflow, with room for the knot factors
        x = x * (2.0 ** 80 if dtype == F32 else 2.0 ** 960)
    elif kind == "scales":                                     # series scales 2^-40, 1, 2^40 in one tensor
        x = x * 2.0 ** (40 * torch.randint(-1, 2, (shape[0], 1, shape[-1]), generator=gen)).double()
    return x.to(dtype)


def _holes(x, G):
    """NaN patterns by path: leading run, trailing run (both next to a -0.0 observation), an all-NaN series, a single
    observation, holes on both sides of every chunk boundary, a run longer than two chunks, one hole per chunk, 30 %."""
    x = x.clone()
    P, L, C = x.shape
    nan = float("nan")
    gen = torch.Generator().manual_seed(P * L + C)
    G = max(G, 1)
    run = min(5, L - 1)
    for p in range(P):
        kind = p % 8
        if kind == 0:
            x[p, :run] = nan
            x[p, run, 0] = -0.0
        elif kind == 1:
            x[p, L - run:] = nan
            x[p, L - run - 1, 0] = -0.0
        elif kind == 2:
            x[p, :, 0] = nan
            x[p, torch.rand(L, C, generator=gen) < 0.3] = nan
        elif kind == 3:
            keep = x[p, L // 2].clone()
            x[p] = nan
            x[p, L // 2] = keep
        elif kind == 4:
            for j in range(G, L, G):
                x[p, j - 1:j + 1] = nan
        elif kind == 5:
            x[p, G // 2:G // 2 + 2 * G + 3] = nan
        elif kind == 6:
            for j in range(0, L, G):
                x[p, min(j + (j // G) % G, L - 1)] = nan
        else:
            x[p, torch.rand(L, C, generator=gen) < 0.3] = nan
    return x


def _shifted(x, off):
    """A contiguous view of x's values whose data pointer is ``off`` elements past an allocation (16-byte aligned)."""
    if off == 0:
        return x
    buf = torch.empty(x.numel() + off, dtype=x.dtype, device=x.device)
    buf[off:].copy_(x.flatten())
    return buf[off:].view(x.shape)


def _guarded(n, dtype, off):
    buf = torch.empty(n + 2 * PAD, dtype=dtype, device=DEV)
    buf.view(INT[dtype]).fill_(MARK[dtype])
    return buf, buf[PAD + off:PAD + off + n]


def _check_guard(buf, n, off, what):
    b = buf.view(INT[buf.dtype]).cpu()
    m = MARK[buf.dtype]
    lo, hi = PAD + off, PAD + off + n
    assert bool((b[:lo] == m).all()) and bool((b[hi:] == m).all()), (what, "a write outside the output")
    assert not bool((b[lo:hi] == m).any()), (what, "an output element was not written")


# ---- the calls -------------------------------------------------------------------------------------------------------
def _call(api, x, t, xoff=0, ooff=0, version=1, flags=None, trace=False):
    """Runs one builder on the device copy of x (``xoff`` elements off an aligned allocation).  Returns
    (out on the CPU, kernel names).  ABI calls write into a guard-banded buffer ``ooff`` elements off alignment."""
    P, L, C = x.shape
    xd = _shifted(x.to(DEV), xoff)
    td = None if t is None else t.to(DEV)
    code = _lib.dtype_code(x.dtype)
    stream = _lib.stream_of(xd)
    p = _lib.ptr
    if api == "hermite":
        return _observe(lambda: cde.hermite_cubic_coefficients_with_backward_differences(xd, td), trace)
    if api == "fill":
        return _observe(lambda: cde.linear_interpolation_coeffs(xd, td), trace)
    if api == "natural":
        fn = cde.natural_cubic_coeffs if version == 1 else cde.natural_cubic_spline_coeffs
        return _observe(lambda: fn(xd, td), trace)
    if api == "ffill":
        return _observe(lambda: cde.misc.forward_fill(xd), trace)
    rows = {"fill_abi": L, "rect_abi": 2 * L - 1}.get(api, L - 1)
    width = C if api in ("fill_abi", "rect_abi") else 4 * C
    n = P * rows * width
    buf, out = _guarded(n, x.dtype, ooff)
    fl = torch.zeros(1, dtype=torch.int32, device=DEV) if flags is None else flags
    if api == "hermite_abi":
        fn = lambda: _lib.call("tcde_hermite_bdiff_coeffs", p(xd), p(td), p(out), P, L, C, code, p(fl), stream)
    elif api == "series_abi":
        fn = lambda: _lib.call("tcde_hermite_bdiff_coeffs_series", p(xd), p(td), p(out), P, L, C, code, p(fl), stream)
    elif api == "hermite2":
        filled = torch.empty_like(xd)

        def fn():
            _lib.call("tcde_linear_fill", p(xd), p(td), p(filled), P, L, C, code, None, stream)
            _lib.call("tcde_hermite_bdiff_coeffs", p(filled), p(td), p(out), P, L, C, code, None, stream)
    elif api == "fill_abi":
        fn = lambda: _lib.call("tcde_linear_fill", p(xd), p(td), p(out), P, L, C, code, p(fl), stream)
    elif api == "natural_abi":
        ws = torch.empty(4 * L + 8, dtype=x.dtype, device=DEV)
        fn = lambda: _lib.call("tcde_natural_cubic_coeffs", p(xd), p(td), p(out), p(ws), P, L, C, code, p(fl), stream)
    elif api == "missing_abi":
        scratch = torch.empty(_lib.load().tcde_natural_cubic_missing_scratch_bytes(P, L, C, code), dtype=torch.uint8,
                              device=DEV)
        fn = lambda: _lib.call("tcde_natural_cubic_coeffs_missing", p(xd), p(td), p(out), p(scratch), P, L, C, version,
                               code, stream)
    elif api == "rect_abi":
        fn = lambda: _lib.call("tcde_rectilinear_prepare", p(xd), p(out), P, L, C, 1, code, p(fl), stream)
    else:
        raise AssertionError(api)
    _, *seen = _observe(fn, trace)
    _check_guard(buf, n, ooff, api)
    return (out.view(P, rows, width).cpu(), *seen)


def _oracle_series(x, t, version):
    """natural_cubic_coeffs through the reference's per-series code path even for NaN-free series (the exact operation
    order natural_missing_kernel runs)."""
    tt = O.check_path(x, t)
    xt = x.transpose(-1, -2)
    rows = [O._natural_cubic_series_with_gaps(tt, s, version) for s in xt.reshape(-1, xt.size(-1))]
    parts = [torch.stack([r[j] for r in rows]).reshape(*xt.shape[:-1], -1).transpose(-1, -2) for j in range(4)]
    return torch.cat(parts, dim=-1)


def _check(route, api, x, t, knots, xoff=0, ooff=0, variant=0, version=1, branch=None):
    """Run one case, assert its kernels and compare it with its reference."""
    P, L, C = x.shape
    unit = t is None
    nan = bool(torch.isnan(x).any())
    if branch is not None:
        assert _natural_branch(x.dtype, L, C, xoff == 0, ooff == 0, variant) == branch, (route, branch)
    want_k = _expected(api, x.dtype, L, C, unit, xoff == 0, ooff == 0, variant, nan)
    with _variant(variant):
        got, names = _call(api, x, t, xoff, ooff, version)
        if names != want_k:                          # a lost record, or a real routing change: look once more
            got, names = _call(api, x, t, xoff, ooff, version)
    assert names == want_k, (route, names, want_k)
    if api in ("hermite", "hermite2", "hermite_abi", "series_abi"):
        _report(route, "differing bits", _bits(got, O.hermite_backward_difference_coeffs(x, t)), 0)
    elif api in ("fill", "fill_abi"):
        _report(route, "differing bits", _bits(got, O.linear_knots(x, t)), 0)
    elif api == "ffill":
        _report(route, "differing bits", _bits(got, O.carry_forward(x)), 0)
    elif api == "rect_abi":
        _report(route, "differing bits", _bits(got, O.rectilinear_knots(x, 1)), 0)
    elif api == "missing_abi" or (api == "natural" and (nan or "natural_missing_kernel" in names[-1])):
        _report(route, "differing bits", _bits(got, _oracle_series(x, t, version)), 0)
    else:                                                      # the NaN-free natural routes
        want = O.natural_cubic_coeffs(x, t, 1)
        bar = 256 if knots == "stiff" else 64
        route = route + (" (stiff knots)" if knots == "stiff" else "")
        _report(route, "series ulps", round(_series_ulps(got, want), 2), bar)
        _report(route, "tensor ulps", round(_tensor_ulps(got, want), 2), bar)
    return got, names


# ---- route table -----------------------------------------------------------------------------------------------------
# (id, api, dtypes, (P, L, C), options).  "vec4" / "scalar", "bulk" / "plain", "pairs" / "scalar" name the internal
# branch the shape and offsets force; x+1 / out+1: the input / output one element off a 16-byte boundary.
ROUTES = [
    # Hermite: the fused series kernel, then its fallbacks (C > 32) and the two-launch C-ABI route
    ("hermite/series-vec4", "hermite", [F32], (37, 40, 8), {"holes": True}),
    ("hermite/series-scalar", "hermite", [F32, F64], (37, 40, 3), {"holes": True}),
    ("hermite/series-scalar-x+1", "hermite", [F32], (37, 40, 8), {"holes": True, "xoff": 1}),
    ("hermite/series-scalar-out+1", "series_abi", [F32], (37, 40, 8), {"holes": True, "ooff": 1}),
    ("hermite/ballot-vec4+hvec4", "hermite", [F32], (5, 20, 64), {"holes": True}),
    ("hermite/ballot-scalar+hvec4", "hermite", [F32], (9, 20, 36), {"holes": True}),
    ("hermite/ballot-scalar+hk-bulk", "hermite", [F32, F64], (9, 20, 33), {"holes": True}),
    ("hermite/thread+hk-bulk", "hermite", [F32, F64], (3, 300, 33), {"holes": True}),
    ("hermite/abi-scan+hvec4", "hermite2", [F32], (37, 40, 8), {"holes": True}),
    ("hermite/abi-scan+hk-bulk", "hermite2", [F32, F64], (37, 40, 3), {"holes": True}),
    ("hermite/abi-scan+hk-plain", "hermite2", [F32, F64], (37, 40, 8), {"holes": True, "ooff": 1}),
    ("hermite/abi-ballot+hk-plain", "hermite2", [F32, F64], (37, 40, 3), {"holes": True, "ooff": 1, "variant": 2}),
    ("hermite/abi-thread+hk-plain", "hermite2", [F32, F64], (37, 40, 5), {"holes": True, "ooff": 1, "variant": 1}),
    ("hermite/abi-hk-bulk-x+1", "hermite_abi", [F32, F64], (37, 40, 8), {"xoff": 1}),
    ("hermite/abi-hk-plain-wide", "hermite_abi", [F32], (3, 9, 700), {"ooff": 1}),
    # linear fill
    ("fill/scan-vec4", "fill", [F32], (37, 40, 8), {"holes": True}),
    ("fill/scan-scalar", "fill", [F32, F64], (37, 40, 3), {"holes": True}),
    ("fill/scan-scalar-x+1", "fill", [F32], (37, 40, 8), {"holes": True, "xoff": 1}),
    ("fill/scan-scalar-out+1", "fill_abi", [F32, F64], (37, 40, 8), {"holes": True, "ooff": 1}),
    ("fill/scan-dense", "fill_abi", [F32, F64], (37, 40, 8), {}),
    ("fill/ballot-vec4", "fill", [F32], (37, 40, 8), {"holes": True, "variant": 2}),
    ("fill/ballot-scalar", "fill", [F32, F64], (37, 40, 3), {"holes": True, "variant": 2}),
    ("fill/ballot-scalar-out+1", "fill_abi", [F32], (37, 40, 8), {"holes": True, "variant": 2, "ooff": 1}),
    ("fill/ballot-C33", "fill", [F32, F64], (9, 20, 33), {"holes": True}),
    ("fill/thread", "fill", [F32, F64], (37, 40, 3), {"holes": True, "variant": 1}),
    ("fill/thread-L300", "fill_abi", [F32, F64], (3, 300, 33), {"holes": True, "ooff": 1}),
    # natural cubic, NaN-free
    ("natural/warp", "natural", [F32], (37, 40, 8), {"branch": "warp"}),
    ("natural/win-vec4-pairs", "natural", [F32], (37, 40, 8), {"variant": 2, "branch": "win-vec4-pairs"}),
    ("natural/win-bulk-pairs", "natural", [F32], (37, 40, 6), {"branch": "win-bulk-pairs"}),
    ("natural/win-bulk-pairs-x+1", "natural", [F32], (37, 40, 8), {"xoff": 1, "branch": "win-bulk-pairs"}),
    ("natural/win-bulk-scalar", "natural", [F32], (37, 40, 5), {"branch": "win-bulk-scalar"}),
    ("natural/win-bulk-scalar-f64", "natural", [F64], (37, 40, 8), {"branch": "win-bulk-scalar"}),
    ("natural/win-plain-pairs", "natural_abi", [F32], (37, 40, 6), {"ooff": 1, "branch": "win-plain-pairs"}),
    ("natural/win-plain-scalar", "natural_abi", [F64], (37, 40, 5), {"ooff": 1, "branch": "win-plain-scalar"}),
    ("natural/cta-S3-bulk", "natural", [F64], (7, 1000, 1), {"branch": "cta-S3-bulk"}),
    ("natural/cta-S1-bulk", "natural", [F32, F64], (5, 200, 33), {"branch": "cta-S1-bulk"}),
    ("natural/cta-S1-plain", "natural_abi", [F32, F64], (5, 200, 33), {"ooff": 1, "branch": "cta-S1-plain"}),
    ("natural/cta-S3-plain", "natural_abi", [F64], (7, 1000, 1), {"ooff": 1, "branch": "cta-S3-plain"}),
    ("natural/refused->missing", "natural", [F64], (2, 4000, 1), {"branch": "refused"}),
    # natural cubic with NaNs: natural_missing_kernel after the dense attempt, both versions
    ("natural/missing-v1", "natural", [F32, F64], (9, 30, 3), {"holes": True, "version": 1}),
    ("natural/missing-v0", "natural", [F32, F64], (9, 30, 3), {"holes": True, "version": 0}),
    ("natural/missing-abi-dense", "missing_abi", [F32, F64], (5, 30, 4), {"version": 1}),
    ("natural/missing-abi-out+1", "missing_abi", [F32, F64], (9, 30, 3), {"holes": True, "ooff": 1, "version": 0}),
    # holds
    ("hold/forward-fill", "ffill", [F32, F64], (9, 30, 3), {"holes": True}),
    ("hold/rectilinear", "rect_abi", [F32, F64], (9, 30, 3), {"holes": True, "ooff": 1}),
]


def _route_cases():
    for rid, api, dtypes, shape, opts in ROUTES:
        for dtype in dtypes:
            knot_kinds = ["unit", "uneven"] + (["stiff"] if api.startswith("natural") and not opts.get("holes") else [])
            if api in ("ffill", "rect_abi"):
                knot_kinds = ["unit"]
            for kk in knot_kinds:
                yield pytest.param(rid, api, dtype, shape, opts, kk,
                                   id="{}-{}-{}".format(rid, "f32" if dtype == F32 else "f64", kk))


def _input(api, dtype, shape, opts, data="randn", seed=0):
    x = _data(data, shape, dtype, seed=sum(shape) + seed)
    if opts.get("holes"):
        x = _holes(x, _scan_geometry(dtype, shape[1], shape[2], True)[1])
    if api == "rect_abi":                                      # the time channel (1) has no NaN (an assertion)
        x[:, :, 1] = torch.arange(shape[1], dtype=dtype)
    return x


@pytest.mark.parametrize("rid,api,dtype,shape,opts,knots", list(_route_cases()))
def test_route(rid, api, dtype, shape, opts, knots):
    x = _input(api, dtype, shape, opts)
    t = _knots(knots, shape[1], dtype)
    _check(rid, api, x, t, knots, xoff=opts.get("xoff", 0), ooff=opts.get("ooff", 0), variant=opts.get("variant", 0),
           version=opts.get("version", 1), branch=opts.get("branch"))


# ---- edge table ------------------------------------------------------------------------------------------------------
def _scan_last_L(dtype, C, unit):
    return _last_L(lambda L: _scan_geometry(dtype, L, C, unit)[0], 2, 40000)


def _edge_cases():
    cases = []
    # scan kernel: L = 2, 3 and G * chunks +- 1 (C = 8: 4 chunks), and its 100 KB tile
    for L in (2, 3, 31, 32, 33, 127, 128, 129):
        cases.append(("scan-L{}".format(L), "fill", F32, (11, L, 8), "unit", {"holes": L > 3}))
        cases.append(("series-L{}".format(L), "hermite", F64, (11, L, 8), "uneven", {"holes": L > 3}))
    for dtype, C in ((F32, 32), (F64, 8), (F32, 1)):
        Lm = _scan_last_L(dtype, C, True)
        for L in (Lm, Lm + 1):
            cases.append(("scan-100KB-C{}-L{}".format(C, L), "hermite", dtype, (3, L, C), "unit", {"holes": True}))
    # ballot kernel: 256 positions, 72 KB
    for L in (255, 256, 257):
        cases.append(("ballot-L{}".format(L), "fill", F32, (3, L, 33), "uneven", {"holes": True}))
    # natural_warp_kernel: prefetch switch at n_vec = L C / 4 = 512; two warps per CTA vs one at C = 128
    for C, Ls in ((4, (511, 512, 513)), (8, (255, 256, 257))):
        for L in Ls:
            cases.append(("warp-nvec{}".format(L * C // 4), "natural", F32, (29, L, C), "uneven", {"branch": "warp"}))
    Lw = _last_L(lambda L: _natural_warp_wpc(L, 128) >= 2, 3, 400)
    for L in (Lw, Lw + 1):
        cases.append(("warp-wpc-L{}".format(L), "natural", F32, (5, L, 128), "unit",
                      {"branch": _natural_branch(F32, L, 128)}))
    # natural_win_kernel's 64 KB cap
    for dtype, C in ((F64, 1), (F32, 6), (F64, 4)):
        Lc = _last_L(lambda L: _natural_branch(dtype, L, C).startswith("win"), 3, 20000)
        for L in (Lc, Lc + 1):
            cases.append(("win-64KB-C{}-L{}".format(C, L), "natural", dtype, (3, L, C), "uneven",
                          {"branch": _natural_branch(dtype, L, C)}))
    # widths
    for C in (1, 2, 3, 4, 6, 32, 33, 128, 132):
        for dtype in (F32, F64):
            for api in ("fill", "hermite", "natural"):
                cases.append(("width-{}-C{}".format(api, C), api, dtype, (5, 17, C), "uneven",
                              {"holes": api == "fill" or (api == "hermite" and C % 2 == 1)}))
            cases.append(("width-natural-holes-C{}".format(C), "natural", dtype, (2, 9, C), "unit", {"holes": True}))
    # one path
    for api in ("fill", "hermite", "natural", "hermite_abi", "natural_abi", "ffill"):
        cases.append(("P1-{}".format(api), api, F32, (1, 40, 8), "uneven", {"holes": api in ("fill", "hermite", "ffill")}))
    return [pytest.param(c, id="{}-{}-{}".format(c[0], "f32" if c[2] == F32 else "f64", c[4])) for c in cases]


@pytest.mark.parametrize("case", _edge_cases())
def test_shape_edge(case):
    rid, api, dtype, shape, knots, opts = case
    x = _input(api, dtype, shape, opts)
    t = _knots(knots, shape[1], dtype)
    branch = opts.get("branch")
    _check("edge " + rid.split("-")[0], api, x, t, knots, branch=branch, version=opts.get("version", 1))


DATA = ["randn", "zeros", "subnormal", "huge", "scales"]
KNOTS = ["unit", "uneven", "stiff", "f32grid"]
# (api, variant, (P, L, C)): the gap-filling routes on chunked shapes (G = 8 for the scan kernel at 64 x 4)
DATA_ROUTES = [("fill", 0, (16, 64, 4)), ("fill", 2, (16, 64, 4)), ("fill", 1, (16, 64, 4)), ("hermite", 0, (16, 64, 4)),
               ("hermite", 0, (16, 64, 3)), ("hermite", 0, (16, 40, 33)), ("ffill", 0, (16, 64, 3)),
               ("missing_abi", 0, (8, 40, 3))]


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("knots", KNOTS)
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("api,variant,shape", DATA_ROUTES, ids=["{}-v{}-C{}".format(a, v, s[2]) for a, v, s in DATA_ROUTES])
def test_data_edge(api, variant, shape, data, knots, dtype):
    """Signed zeros (-0.0 next to imputed ends and between equal observations), subnormals, values near overflow and
    series scales 2^+-40 apart, under every NaN pattern of ``_holes`` and four kinds of knots: bit for bit."""
    if api == "ffill" and knots != "unit":
        pytest.skip("forward fill has no knots")
    x = _input(api, dtype, shape, {"holes": True}, data=data)
    t = _knots(knots, shape[1], dtype)
    _check("data " + api, api, x, t, knots, variant=variant, version=0 if data == "zeros" else 1)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("knots", KNOTS)
@pytest.mark.parametrize("data", ["randn", "zeros", "huge", "scales"])
@pytest.mark.parametrize("branch", ["warp", "win-vec4-pairs", "win-bulk-pairs", "win-bulk-scalar", "cta"])
def test_natural_dense_per_series_bar(branch, data, knots, dtype):
    """The NaN-free natural routes within 64 ulp (256 on stiff knots) of each series' own scale -- series 2^40 apart
    in one tensor included -- and within the same bar of natural_missing_kernel.  (Subnormal series are left out: a
    subnormal has fewer significant bits than eps assumes.)"""
    if (branch == "warp" or branch.endswith("pairs")) and dtype == F64:
        pytest.skip("fp32-only branch")
    shape, variant = {"warp": ((12, 48, 8), 0), "win-vec4-pairs": ((12, 48, 8), 2), "win-bulk-pairs": ((12, 48, 6), 0),
                      "win-bulk-scalar": ((12, 48, 5), 0), "cta": ((12, 200, 33), 0)}[branch]
    x = _data(data, shape, dtype, seed=7)
    t = _knots(knots, shape[1], dtype)
    got, _ = _check("dense " + branch, "natural", x, t, knots, variant=variant)
    with _variant(1):
        ref, names = _call("missing_abi", x, t)
    bar = 256 if knots == "stiff" else 64
    _report("dense " + branch + (" (stiff knots)" if knots == "stiff" else ""), "series ulps vs missing kernel",
            round(_series_ulps(got, ref), 2), bar)


@pytest.mark.parametrize("route", ["warp", "win-vec4-pairs", "win-bulk-pairs", "win-bulk-scalar-f64", "cta-S1",
                                   "cta-S3-f64"])
@pytest.mark.parametrize("knots", ["unit", "uneven"])
def test_natural_nan_routing(route, knots):
    """One NaN at the first element of the first path and at the last element of the last path: the dense kernel must
    report it through TCDE_FLAG_NAN_SEEN, and the public builder must then give the per-series oracle's bits."""
    shape, dtype, variant = {"warp": ((9, 40, 8), F32, 0), "win-vec4-pairs": ((9, 40, 8), F32, 2),
                             "win-bulk-pairs": ((9, 40, 6), F32, 0), "win-bulk-scalar-f64": ((9, 40, 5), F64, 0),
                             "cta-S1": ((3, 200, 33), F32, 0), "cta-S3-f64": ((4, 1000, 1), F64, 0)}[route]
    x = _data("randn", shape, dtype, seed=3)
    x[0, 0, 0] = float("nan")
    x[-1, -1, -1] = float("nan")
    t = _knots(knots, shape[1], dtype)
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    with _variant(variant):
        _call("natural_abi", x, t, flags=flags)
    assert int(flags.item()) & _lib.FLAG_NAN_SEEN, route
    for version in (1, 0):
        _check("nan-routing " + route, "natural", x, t, knots, variant=variant, version=version)


# ---- persistent grids: one and two full sweeps -----------------------------------------------------------------------
# (id, api, dtype, (L, C), variant, paths per CTA from its block size)
SWEEPS = [
    ("scan", "fill", F32, (16, 4), 0, lambda blk: blk // 32),
    ("series", "hermite", F64, (16, 3), 0, lambda blk: blk // 32),
    ("ballot", "fill", F32, (16, 4), 2, lambda blk: blk // 32),
    ("hvec4", "hermite_abi", F32, (16, 4), 0, lambda blk: 1),
    ("hk", "hermite_abi", F64, (16, 3), 0, lambda blk: 1),
    ("warp", "natural", F32, (16, 4), 0, lambda blk: blk // 32),
    ("win", "natural", F64, (16, 3), 0, lambda blk: 1),
    ("cta", "natural", F64, (1000, 1), 0, lambda blk: 3),
]


@pytest.mark.parametrize("sid,api,dtype,lc,variant,per_cta", SWEEPS, ids=[s[0] for s in SWEEPS])
def test_grid_sweep_edges(sid, api, dtype, lc, variant, per_cta):
    """P = one sweep of the persistent grid - 1, + 0, + 1 and two sweeps + 1 (the grid is read from the profiler's
    trace of a large launch), against the oracle (and, for the natural routes, natural_missing_kernel)."""
    L, C = lc
    probe = 40000 if sid != "cta" else 2000
    with _variant(variant):
        _, names, events = _call(api, torch.zeros(probe, L, C, dtype=dtype), None, trace=True)
    ev = [e for e in events if _kname(e["name"]) == names[-1]][0]
    sweep = ev["args"]["grid"][0] * per_cta(ev["args"]["block"][0])
    assert sweep < probe, (sid, sweep, probe)
    for P in (sweep - 1, sweep, sweep + 1, 2 * sweep + 1):
        x = _input(api, dtype, (P, L, C), {"holes": api in ("fill", "hermite")}, seed=P)
        if api == "natural" and P * C > 4096:
            with _variant(variant):
                got, _ = _check("sweep " + sid, api, x, None, "unit", variant=variant)
                ref, _ = _call("missing_abi", x, None)
            _report("sweep " + sid, "series ulps vs missing kernel", round(_series_ulps(got, ref), 2), 64)
            pick = torch.arange(0, P, max(1, P // 16))
            _report("sweep " + sid, "missing kernel differing bits", _bits(ref[pick], _oracle_series(x[pick], None, 1)), 0)
        else:
            _check("sweep " + sid, api, x, None, "unit", variant=variant)


# ---- bugs fixed with these tables ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,C", [(F64, 2860), (F32, 7764), (F64, 2327), (F32, 4654)])
@pytest.mark.parametrize("knots", ["unit", "uneven"])
def test_wide_hermite(dtype, C, knots):
    """Rows too wide for one shared-memory tile (logsig_windows at 10 channels / depth 4 gives 2,860 channels, at 8 / 5
    7,764) run hermite_kernel over channel tiles with plain stores; they used to raise NotImplementedError."""
    x = _holes(_data("randn", (2, 6, C), dtype, seed=C), 1)
    t = _knots(knots, 6, dtype)
    _check("wide hermite", "hermite", x, t, knots)
    _check("wide hermite", "hermite2", x, t, knots, ooff=1)


def test_wide_hermite_through_the_host_series_pipeline():
    """cdeint_from_host_series's two-launch builder at 2,860 channels gives the solve of the public builder's bits."""
    P, L, C, H = 3, 6, 2860, 2
    x = _holes(_data("randn", (P, L, C), F64, seed=1), 1).pin_memory()
    z0 = torch.randn(P, H, dtype=F64).pin_memory()
    torch.manual_seed(0)
    func = cde.LinearVectorField(H, C).to(device=DEV, dtype=F64)
    t = torch.tensor([0.0, L - 1.0], dtype=F64)
    got = hostio.cdeint_from_host_series(x, func, z0, t, method="euler", options={"step_size": 1.0})
    torch.cuda.synchronize()
    coeffs = cde.hermite_cubic_coefficients_with_backward_differences(x.to(DEV))
    assert _bits(coeffs, O.hermite_backward_difference_coeffs(x)) == 0
    with torch.no_grad():
        want = cde.cdeint(cde.CubicSpline(coeffs), func, z0.to(DEV), t, adjoint=False, method="euler",
                          options={"step_size": 1.0})
    assert _bits(got, want) == 0


@pytest.mark.parametrize("dtype", [F32, F64])
def test_forward_fill_length_one(dtype):
    """misc.forward_fill has no length limit (misc.py:103-126): a length-1 input is returned as it is."""
    x = torch.tensor([[[1.5, float("nan"), -0.0]], [[float("nan"), 2.0, 3.0]]], dtype=dtype)
    got, names = _call("ffill", x, None)
    assert names == ["hold_kernel<{}, false>".format(_T(dtype))]
    assert _bits(got, O.carry_forward(x)) == 0 and _bits(got, x) == 0
    assert _bits(cde.misc.forward_fill(x.to(DEV).transpose(0, 1), fill_index=0).transpose(0, 1), x) == 0


def test_every_builder_kernel_is_the_observed_kernel_of_a_case():
    """Runs last: the union of the kernels the cases above launched is every builder instantiation of the library."""
    assert _OBSERVED == ALL_KERNELS, (sorted(ALL_KERNELS - _OBSERVED), sorted(_OBSERVED - ALL_KERNELS))
