"""ctypes binding of libtoppra_b200_reach.so (include/toppra_b200_reach.h): the reachable sets of problems with a robust
(conic) constraint.

The companion library links against libtoppra_b200.so and reports errors through its tb_last_error(), so errors are
read with `_lib.check`.  There is NO CPU fallback: if the library is missing or a call fails, this module raises."""
import ctypes
import os

from . import _lib

LIB_PATH = os.path.join(_lib._HERE, "libtoppra_b200_reach.so")

_c_dp = ctypes.c_void_p
_c_ip = ctypes.c_void_p
_int = ctypes.c_int
_stream = ctypes.c_void_p

_PROTOS = {
    "tbr_reach_version": ([], _int),
    "tbr_reachable_sets_robust": ([_c_dp, _int, _int, _int, _int, _c_dp, _c_dp, _int, _int, _int, _c_ip, _c_dp, _c_dp,
                                   _c_dp, _c_dp, _c_ip, _stream], _int),
}

_qlib = None


def load():
    """Load libtoppra_b200_reach.so (after libtoppra_b200.so, whose error slot it shares)."""
    global _qlib
    if _qlib is None:
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
        _qlib = lib
    return _qlib


def exported_symbols():
    return sorted(_PROTOS)
