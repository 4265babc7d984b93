"""ctypes binding of libtoppra_b200_robust.so (include/toppra_b200_robust.h): TOPPRAsd and single stage solves of
problems with a robust (conic) constraint.

The companion library links against libtoppra_b200.so and reports errors through its tb_last_error(), so errors are
read with `_lib.check`.  There is NO CPU fallback: if the library is missing or a call fails, this module raises."""
import ctypes
import os

from . import _lib

LIB_PATH = os.path.join(_lib._HERE, "libtoppra_b200_robust.so")

_c_dp = ctypes.c_void_p
_c_ip = ctypes.c_void_p
_int = ctypes.c_int
_stream = ctypes.c_void_p

_PROTOS = {
    "tbr_version": ([], _int),
    "tbr_sd_forward_robust": ([_c_dp, _int, _int, _int, _int, _c_dp, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_ip, _c_dp,
                               _c_dp, _c_dp, _c_dp, _c_dp, _c_ip, _c_ip, _stream], _int),
    "tbr_socp_stage_batch": ([_c_dp, _c_dp, _c_dp, _c_dp, _int, _int, _int, _c_dp, _c_dp, _c_dp, _int, _c_dp, _stream],
                             _int),
}

_rlib = None


def load():
    """Load libtoppra_b200_robust.so (after libtoppra_b200.so, whose error slot it shares)."""
    global _rlib
    if _rlib is None:
        _lib.load()
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "toppra_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (argtypes, restype) in _PROTOS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing: loud on purpose
            fn.argtypes = argtypes
            fn.restype = restype
        _rlib = lib
    return _rlib


def exported_symbols():
    return sorted(_PROTOS)
