"""ctypes binding of libtoppra_b200_poly.so (include/toppra_b200_poly.h): order-k piecewise-polynomial paths.

The companion library links against libtoppra_b200.so and reports errors through its tb_last_error(), so errors are
read with `_lib.check`.  There is NO CPU fallback: if the library is missing or a call fails, this module raises."""
import ctypes
import os

from . import _lib

LIB_PATH = os.path.join(_lib._HERE, "libtoppra_b200_poly.so")
MAX_COEFFS = 8   # TBP_MAX_COEFFS

_c_dp = ctypes.c_void_p
_c_ip = ctypes.c_void_p
_int = ctypes.c_int
_stream = ctypes.c_void_p

_PROTOS = {
    "tbp_version": ([], _int),
    "tbp_ppoly_eval": ([_c_dp, _c_dp, _int, _int, _int, _int, _int, _c_dp, _int, _int, _int, _c_dp, _stream], _int),
    "tbp_rows_velacc_sampled": ([_c_dp, _c_dp, _int, _int, _c_dp, _int, _int, _c_dp, _c_dp, _int, _int, _c_dp, _int, _int,
                                 _int, _int, _stream], _int),
    "tbp_xbound_varying_sampled": ([_c_dp, _int, _int, _int, _c_dp, _int, _c_dp, _int, _int, _int, _stream], _int),
    "tbp_propose_gridpoints": ([_c_dp, _c_dp, _int, _int, _int, _int, _int, ctypes.c_double, _int, ctypes.c_double, _int,
                                _int, _c_dp, _c_dp, _c_ip, _c_ip, _stream], _int),
    "tbp_constaccel_eval": ([_c_dp, _c_dp, _int, _int, _int, _int, _c_dp, _int, _c_dp, _c_dp, _c_dp, _int, _int, _c_dp,
                             _int, _int, _int, _c_dp, _stream], _int),
}

_plib = None


def load():
    """Load libtoppra_b200_poly.so (after libtoppra_b200.so, whose error slot it shares)."""
    global _plib
    if _plib is None:
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
        _plib = lib
    return _plib


def exported_symbols():
    return sorted(_PROTOS)
