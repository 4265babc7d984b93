"""TEST INFRASTRUCTURE ONLY — ctypes front-end of tests/robust_sd_oracle.c, the C restatement of
libtoppra_b200_robust.so (robust TOPPRAsd passes and single stage solves).

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
_SRC = os.path.join(_HERE, "robust_sd_oracle.c")
_LIB = None

_dp = ctypes.POINTER(ctypes.c_double)


def lib():
    global _LIB
    if _LIB is None:
        out = tempfile.mkdtemp(prefix="robust_sd_oracle_")
        atexit.register(shutil.rmtree, out, True)
        so = os.path.join(out, "librobust_sd_oracle.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-o", so, _SRC,
                               "-lm"])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def sd_forward_rows_robust(rows, grid, conic_row0, conic_rows, ellipsoid, K, sd_start=0.0, slow=False):
    """One robust TOPPRAsd forward pass (fastest, or slowest with slow=True) over the controllable sets K [G, 2] of the
    backward pass (oracle.solve_rows_robust) — orc_sd_forward_rows_robust.  rows [G, 3, R].  Returns dict(x [G] = sd^2,
    u [G-1], status, fail_stage)."""
    rows, rp = _d(rows)
    grid, gp = _d(grid)
    K, kp = _d(K)
    G, _, R = rows.shape
    ell, ep = _d(ellipsoid)
    x = np.zeros(G)
    u = np.zeros(max(G - 1, 1))
    fs = ctypes.c_int()
    st = lib().orc_sd_forward_rows_robust(rp, gp, G, R, int(conic_row0), int(conic_rows), ep, kp,
                                          ctypes.c_double(sd_start), 1 if slow else 0, x.ctypes.data_as(_dp),
                                          u.ctypes.data_as(_dp), ctypes.byref(fs))
    return dict(x=x, u=u[:G - 1], status=int(st), fail_stage=fs.value)


def socp_stage_robust(g, a, b, c, conic_row0, conic_rows, ellipsoid, xl, xh, xnext=None):
    """One robust stage problem min g0 u + g1 x — orc_socp_stage_robust.  xnext: None or (delta, x_next_lo, x_next_hi).
    Returns [u, x], NaN NaN when infeasible."""
    g, gp_ = _d(g)
    a, ap = _d(a)
    b, bp = _d(b)
    c, cp = _d(c)
    ell, ep = _d(ellipsoid)
    xn, xnp = (None, None) if xnext is None else _d(xnext)
    out = np.zeros(2)
    lib().orc_socp_stage_robust(gp_, ap, bp, cp, int(a.shape[0]), int(conic_row0), int(conic_rows), ep,
                                ctypes.c_double(xl), ctypes.c_double(xh), xnp, out.ctypes.data_as(_dp))
    return out
