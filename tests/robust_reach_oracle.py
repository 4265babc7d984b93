"""TEST INFRASTRUCTURE ONLY — ctypes front-end of tests/robust_reach_oracle.c, the C restatement of the reachable sets
of robust problems (orc_reachable_sets_robust) and of K2r's backward pass from a velocity range
(orc_controllable_sets_robust).

The library is compiled on first use into a temporary directory (removed at exit), with the flags of oracle/Makefile:
no FMA contraction, no fast math, so that its fp64 results are those of the kernels built with -fmad=false."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "robust_reach_oracle.c")
_LIB = None

_dp = ctypes.POINTER(ctypes.c_double)


def lib():
    global _LIB
    if _LIB is None:
        out = tempfile.mkdtemp(prefix="robust_reach_oracle_")
        atexit.register(shutil.rmtree, out, True)
        so = os.path.join(out, "librobust_reach_oracle.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-o", so, _SRC,
                               "-lm"])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def reachable_sets_robust(rows, xbound, grid, conic_row0, conic_rows, ellipsoid, X, sdmin=0.0, sdmax=None):
    """compute_reachable_sets of one robust path on its feasible sets X [G, 2] (orc_reachable_sets_robust).
    rows [G, 3, R], xbound [G, 2].  Returns (L [G, 2], fail_stage)."""
    rows, rp = _d(rows)
    xb, xp = _d(xbound)
    grid, gp = _d(grid)
    X, Xp = _d(X)
    ell, ep = _d(ellipsoid)
    G, _, R = rows.shape
    L = np.zeros((G, 2))
    fs = lib().orc_reachable_sets_robust(rp, xp, gp, G, R, int(conic_row0), int(conic_rows), ep, Xp,
                                         ctypes.c_double(sdmin), ctypes.c_double(sdmin if sdmax is None else sdmax),
                                         L.ctypes.data_as(_dp))
    return L, int(fs)


def controllable_sets_robust(rows, xbound, grid, conic_row0, conic_rows, ellipsoid, sd_end=0.0, sd_end_hi=None):
    """K2r's backward pass from K[N] = [sd_end^2, sd_end_hi^2] (orc_controllable_sets_robust).  Returns
    (K [G, 2], status, fail_stage)."""
    rows, rp = _d(rows)
    xb, xp = _d(xbound)
    grid, gp = _d(grid)
    ell, ep = _d(ellipsoid)
    G, _, R = rows.shape
    K = np.zeros((G, 2))
    fs = ctypes.c_int()
    st = lib().orc_controllable_sets_robust(rp, xp, gp, G, R, int(conic_row0), int(conic_rows), ep,
                                            ctypes.c_double(sd_end),
                                            ctypes.c_double(sd_end if sd_end_hi is None else sd_end_hi),
                                            K.ctypes.data_as(_dp), ctypes.byref(fs))
    return K, int(st), fs.value
