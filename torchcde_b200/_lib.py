"""ctypes binding of the C-ABI library (include/torchcde_b200.h).

The library is built in-tree (``torchcde_b200/csrc/libtcde_b200.so``, see ``csrc/Makefile``
and ``__graft_entry__.build``).  There is no CPU or PyTorch-eager fallback: if the library is
missing or a call fails, the product path raises.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libtcde_b200.so")

F32, F64 = 0, 1
CONTROL_CUBIC, CONTROL_LINEAR = 0, 1
METHODS = {"euler": 0, "midpoint": 1, "rk4": 2}
REVERSIBLE_HEUN = 3          # tcde_method of torchsde's reversible Heun (tcde_cdeint_reversible_heun_linear)
STAGES = {"euler": 1, "midpoint": 2, "rk4": 4}
FLAG_NAN_SEEN, FLAG_NAN_TIME, FLAG_NAN_FIRST_ROW = 1, 2, 4

_p, _i64, _i32, _int, _dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_int, ctypes.c_double


class SplineMember(ctypes.Structure):
    """``tcde_spline_member``: one member of ``tcde_spline_eval_grouped``."""
    _fields_ = [("control", _p), ("knot_t", _p), ("index", _p), ("frac", _p), ("out", _p), ("n_paths", _i64),
                ("n_rows", _i64), ("channels", _i64), ("n_times", _i64), ("control_kind", _i32), ("reserved", _i32)]


class ContractMember(ctypes.Structure):
    """``tcde_contract_member``: one member of ``tcde_field_contract_grouped``."""
    _fields_ = [("field", _p), ("dx", _p), ("out", _p), ("n_paths", _i64), ("hidden", _i64), ("channels", _i64),
                ("dx_stride", _i64)]

# name -> argtypes; must list every entry point the header declares (tests/test_abi.py checks)
SIGNATURES = {
    "tcde_abi_version": ([], _int),
    "tcde_last_error": ([], ctypes.c_char_p),
    "tcde_device_info": ([_p, _p, _p], _int),
    "tcde_hermite_bdiff_coeffs": ([_p, _p, _p, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_field_contract": ([_p, _p, _p, _i64, _i64, _i64, _i64, ctypes.c_double, _int, _p], _int),
    "tcde_spline_eval_grouped": ([ctypes.POINTER(SplineMember), _int, _int, _int, _p], _int),
    "tcde_field_contract_grouped": ([ctypes.POINTER(ContractMember), _int, _dbl, _int, _p], _int),
    "tcde_hermite_bdiff_coeffs_series": ([_p, _p, _p, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_linear_fill": ([_p, _p, _p, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_nan_flag": ([_p, _i64, _int, _p, _p], _int),
    "tcde_forward_fill": ([_p, _p, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_rectilinear_prepare": ([_p, _p, _i64, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_natural_cubic_coeffs": ([_p, _p, _p, _p, _i64, _i64, _i64, _int, _p, _p], _int),
    "tcde_natural_cubic_missing_scratch_bytes": ([_i64, _i64, _i64, _int], _i64),
    "tcde_natural_cubic_coeffs_missing": ([_p, _p, _p, _p, _i64, _i64, _i64, _int, _int, _p], _int),
    "tcde_spline_eval": ([_p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _int, _int, _int, _p], _int),
    "tcde_vector_field_linear": ([_p, _int, _i64, _p, _p, _p, _p, _i64, _i64, _i64, _i32, _dbl, _int, _p], _int),
    "tcde_vector_field_linear_vjp_scratch_bytes": ([_i64, _i64, _i64], _i64),
    "tcde_vector_field_linear_vjp": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i32, _dbl,
                                      _dbl, _dbl, _dbl, _int, _p], _int),
    "tcde_cdeint_fixed_linear_stages": ([_p, _int, _i64, _p, _p, _p, _p, _p, _i64, _i64, _i64, _int, _i64, _p, _p, _p,
                                         _i64, _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_cdeint_fixed_linear_backward": ([_p, _int, _i64, _p, _p, _p, _p, _p, _i64, _i64, _i64, _int, _i64, _p, _p, _p,
                                           _i64, _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_cdeint_reversible_heun_linear": ([_p, _int, _i64, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64, _p, _p,
                                            _p, _i64, _p, _p, _int, _p], _int),
    "tcde_reversible_heun_linear_backward_segment": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p,
                                                      _p, _p, _i64, _i64, _i64, _i64, _i64, _p, _p, _int, _p], _int),
    "tcde_cdeint_reversible_heun_mlp": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64, _i64,
                                         _p, _p, _p, _i64, _p, _p, _int, _p], _int),
    "tcde_reversible_heun_mlp_backward_segment": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _i64,
                                                   _p, _p, _p, _i64, _i64, _i64, _i64, _i64, _i64, _p, _p, _int, _p], _int),
    "tcde_dopri5_mlp_backward": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64,
                                  _i64, _i64, _i64, _i64, _dbl, _int, _p], _int),
    "tcde_linear_field_param_grads_scratch_bytes": ([_i64, _i64, _i64, _i64], _i64),
    "tcde_linear_field_param_grads": ([_p, _int, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _i64, _i64, _i64, _dbl,
                                       _int, _p], _int),
    "tcde_linear_combination": ([_p, _p, _p, _p, _int, _i64, _int, _p], _int),
    "tcde_error_ratio_partials": ([_i64], _i64),
    "tcde_error_ratio_sumsq": ([_p, _p, _p, _p, _int, _dbl, _dbl, _i64, _int, _p, _p], _int),
    "tcde_cdeint_fixed_linear": ([_p, _int, _i64, _p, _p, _p, _p, _i64, _i64, _i64, _int, _i64, _p, _p, _p, _i64,
                                  _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_cdeint_fixed_mlp": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _int, _i64, _p, _p, _p,
                               _i64, _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_cdeint_fixed_mlp_stages": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _int, _i64, _p,
                                      _p, _p, _i64, _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_cdeint_fixed_mlp_backward": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _int,
                                        _i64, _p, _p, _p, _i64, _p, _p, _p, _dbl, _int, _p], _int),
    "tcde_mlp_field_param_grads_scratch_bytes": ([_i64, _i64, _i64, _i64, _i64], _i64),
    "tcde_mlp_field_param_grads": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64, _i64,
                                    _i64, _i64, _dbl, _dbl, _int, _p], _int),
    "tcde_vector_field_mlp": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _i32, _dbl, _int, _p],
                              _int),
    "tcde_vector_field_mlp_vjp_scratch_bytes": ([_i64, _i64, _i64, _i64], _i64),
    "tcde_vector_field_mlp_vjp": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64,
                                   _i64, _i32, _dbl, _dbl, _dbl, _dbl, _int, _p], _int),
    "tcde_dopri5_linear_grid": ([_i64], _int),
    "tcde_dopri5_linear_paired_attempts": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _dbl,
                                            _p, _p, _p, _p, _p, _i64, _i64, _i64, _int, _p], _int),
    "tcde_dopri5_linear_attempts": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _dbl, _i64, _i64,
                                     _int, _p], _int),
    "tcde_dopri5_linear_record_attempts": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _dbl,
                                            _p, _p, _p, _p, _i64, _i64, _i64, _int, _p], _int),
    "tcde_dopri5_linear_backward": ([_p, _int, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64,
                                     _dbl, _int, _p], _int),
    "tcde_logsignature_max_terms": ([], _i64),
    "tcde_logsignature_windows": ([_p, _i64, _i64, _i64, _p, _i64, _int, _p, _i64, _p, _int, _p], _int),
    "tcde_set_solve_variant": ([_int], _int),
    "tcde_set_natural_variant": ([_int], _int),
}

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes handle; raise loudly if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NativeLibraryError(
            "torchcde_b200: the CUDA library {} is missing. Build it with `make -C torchcde_b200/csrc` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback.".format(LIB_PATH))
    lib = ctypes.CDLL(LIB_PATH)
    for name, (argtypes, restype) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here means header and library disagree
        fn.argtypes = argtypes
        fn.restype = restype
    variant = os.environ.get("TCDE_SOLVE_VARIANT")
    if variant:
        lib.tcde_set_solve_variant(int(variant))
    _lib = lib
    return lib


def dtype_code(dtype):
    if dtype == torch.float32:
        return F32
    if dtype == torch.float64:
        return F64
    raise NotImplementedError("torchcde_b200 kernels are built for float32 and float64; got {}".format(dtype))


def require_cuda(*tensors):
    for x in tensors:
        if x is not None and not x.is_cuda:
            raise RuntimeError(
                "torchcde_b200 runs on CUDA (H100, sm_90a) only and has no CPU path; got a tensor on '{}'. "
                "Move the inputs to the GPU first.".format(x.device))


def ptr(x):
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def stream_of(x):
    return ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.tcde_last_error().decode("utf-8", "replace")
        if rc == -2:
            raise NotImplementedError("{}: {}".format(name, msg))
        if rc == -1:
            raise ValueError("{}: {}".format(name, msg))
        raise RuntimeError("{} failed ({}): {}".format(name, rc, msg))
    return rc
