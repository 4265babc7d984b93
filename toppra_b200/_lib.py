"""ctypes binding of libtoppra_b200.so (include/toppra_b200.h) — the only route from Python to the kernels.

There is NO CPU fallback: if the shared library is missing or a call fails, this module raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtoppra_b200.so")

_c_dp = ctypes.c_void_p  # device (or host) pointer to double
_c_ip = ctypes.c_void_p
_int = ctypes.c_int

_PROTOS = {
    "tb_version": ([], _int),
    "tb_last_error": ([], ctypes.c_char_p),
    "tb_limits": ([ctypes.POINTER(_int), ctypes.POINTER(_int)], _int),
    "tb_record_doubles": ([_int], _int),
    "tb_spline_fit_workspace_doubles": ([_int, _int, _int], _int),
    "tb_spline_fit": ([_c_dp, _int, _c_dp, _int, _int, _int, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, ctypes.c_void_p],
                      _int),
    "tb_ppoly_eval": ([_c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _int, _int, _c_dp, ctypes.c_void_p], _int),
    "tb_coeff_velacc": ([_c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _int, _c_dp, _c_dp, _int, _int, _c_dp,
                         _int, _int, _int, _int, ctypes.c_void_p], _int),
    "tb_xbound_varying": ([_c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _int, _c_dp, _int, _c_dp, _int, _int, _int,
                           ctypes.c_void_p], _int),
    "tb_xbound_velocity": ([_c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _int, _c_dp, _int, _c_dp, _int, _int, _int,
                            ctypes.c_void_p], _int),
    "tb_coeff_second_order": ([_int, _c_dp, _int, _c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _int, _c_dp, _int,
                               _c_dp, _int, _c_dp, _int, _int, _int, ctypes.c_void_p], _int),
    "tb_rows_canlinear": ([_c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _int, _int, _int, _int, _int, _c_dp, _int, _int, _c_dp,
                           _int, _int, _int, ctypes.c_void_p], _int),
    "tb_init_bounds": ([_c_dp, _int, _int, _int, _int, ctypes.c_void_p], _int),
    "tb_scan": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_ip, _c_ip,
                 ctypes.c_void_p], _int),
    "tb_scan_ex": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_dp, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_ip,
                    _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_scan_velacc": ([_c_dp, _c_dp, _int, _int, _int, _c_dp, _int, _int, _int, _c_dp, _int, _int, _c_dp, _c_dp, _c_dp,
                        _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_lp2d_batch": ([_c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _c_ip, _int, _int, _c_ip, _c_dp, _c_dp, _c_ip,
                       ctypes.c_void_p], _int),
    "tb_lp1d_batch": ([_c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _int, _int, _c_ip, _c_dp, _c_dp, _c_ip, ctypes.c_void_p],
                      _int),
    "tb_scan_robust": ([_c_dp, _int, _int, _int, _int, _c_dp, _c_dp, _int, _int, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp,
                        _c_dp, _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_time_grid": ([_c_dp, _c_dp, _int, _int, _int, _c_dp, _c_dp, ctypes.c_void_p], _int),
    "tb_constaccel_eval": ([_c_dp, _c_dp, _int, _int, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _int, _int, _c_dp, _int,
                            _int, _int, _c_dp, ctypes.c_void_p], _int),
    "tb_feasible_sets": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_dp, ctypes.c_void_p], _int),
    "tb_feasible_sets_ex": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _int, _c_dp, ctypes.c_void_p], _int),
    "tb_reachable_sets": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_ip,
                           ctypes.c_void_p], _int),
    "tb_scan_ragged": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp,
                        _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_scan_velacc_ragged": ([_c_dp, _c_dp, _int, _int, _int, _c_dp, _int, _int, _int, _c_ip, _c_dp, _int, _int, _c_dp,
                               _c_dp, _c_dp, _c_dp, _int, _c_dp, _c_dp, _c_dp, _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_feasible_sets_ragged": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_ip, _int, _c_dp, ctypes.c_void_p], _int),
    "tb_reachable_sets_ragged": ([_c_dp, _int, _int, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_dp, _int, _c_dp, _c_dp,
                                  _c_ip, ctypes.c_void_p], _int),
    "tb_scan_robust_ragged": ([_c_dp, _int, _int, _int, _int, _c_dp, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_dp, _int,
                               _c_dp, _c_dp, _c_dp, _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_scan_robust_ex": ([_c_dp, _int, _int, _int, _int, _c_dp, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_dp, _c_dp,
                           _int, _c_dp, _c_dp, _c_dp, _c_ip, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_sd_bisect_ragged": ([_c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _int, _int, _int, _c_ip, _c_dp, ctypes.c_double, _int,
                             _c_ip, _c_dp, _c_dp, _c_dp, _c_ip, ctypes.c_void_p], _int),
    "tb_propose_gridpoints": ([_c_dp, _c_dp, _int, _int, _int, _int, ctypes.c_double, _int, ctypes.c_double, _int, _int,
                               _c_dp, _c_dp, _c_ip, _c_ip, ctypes.c_void_p], _int),
    "tb_sd_bisect": ([_c_dp, _c_dp, _c_dp, _c_dp, _c_dp, _int, _int, _int, _c_dp, ctypes.c_double, _int, _c_ip, _c_dp,
                      _c_dp, _c_dp, _c_ip, ctypes.c_void_p], _int),
    "tb_spline_time_stamps": ([_c_dp, _c_dp, _int, _c_ip, _int, _int, _c_dp, _c_dp, _c_ip, ctypes.c_void_p], _int),
    "tb_solve_velacc_host": ([_int, _c_dp, _c_dp, _int, _int, _int, _c_dp, _int, _c_dp, _c_dp, _int, _int, _c_dp,
                              _c_dp, _c_dp, _c_dp, _c_dp, _c_ip], _int),
}

_lib = None


class ToppraB200Error(RuntimeError):
    """A libtoppra_b200 call failed (argument error < 0, CUDA error > 0)."""


def load():
    """Load libtoppra_b200.so (built by `make -C toppra_b200/csrc` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "toppra_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (argtypes, restype) in _PROTOS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing: loud on purpose
            fn.argtypes = argtypes
            fn.restype = restype
        _lib = lib
    return _lib


def exported_symbols():
    return sorted(_PROTOS)


def check(rc, what):
    if rc != 0:
        msg = load().tb_last_error()
        raise ToppraB200Error("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else ""))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL).  Tensors must be contiguous fp64/int32 on CUDA."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise ValueError("toppra_b200: tensor must be contiguous")
    if str(t.dtype) not in ("torch.float64", "torch.int32"):   # the C-ABI takes `double *` and `int *` only
        raise ValueError("toppra_b200: tensor must be float64 or int32, got %s" % t.dtype)
    return ctypes.c_void_p(t.data_ptr())


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("toppra_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return torch


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
