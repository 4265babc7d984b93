"""TEST INFRASTRUCTURE ONLY — ctypes front-end of tests/robust_cones_oracle.c, the C restatement of robust problems whose
rows each carry their own ellipsoid (cone table [R, 4] = (flag, ru, rx, rc)) and whose stages may carry a u box.

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
_SRC = os.path.join(_HERE, "robust_cones_oracle.c")
_LIB = None

_dp = ctypes.POINTER(ctypes.c_double)


def lib():
    global _LIB
    if _LIB is None:
        out = tempfile.mkdtemp(prefix="robust_cones_oracle_")
        atexit.register(shutil.rmtree, out, True)
        so = os.path.join(out, "librobust_cones_oracle.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-o", so, _SRC,
                               "-lm"])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _d(a):
    if a is None:
        return None, None
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def table(R, spans):
    """Cone table [R, 4] of robust constraints spans [(row0, nrows, (ru, rx, rc))]."""
    t = np.zeros((R, 4))
    for row0, n, ell in spans:
        t[row0:row0 + n, 0] = 1.0
        t[row0:row0 + n, 1:] = ell
    return t


def scan(rows, xbound, grid, cones, sd_start=0.0, sd_end=0.0, sd_end_hi=None, ubox=None, backward_only=False):
    """K2r of one path (orc_cones_scan).  rows [G, 3, R], xbound [G, 2], ubox [G, 2] or None.  Returns dict(K, sd, u,
    status, fail_stage); sd and u are None when backward_only."""
    rows, rp = _d(rows)
    xb, xp = _d(xbound)
    grid, gp = _d(grid)
    cones, cp = _d(cones)
    ub, up = _d(ubox)
    G, _, R = rows.shape
    K, sd, u = np.zeros((G, 2)), np.zeros(G), np.zeros(max(G - 1, 1))
    fs = ctypes.c_int()
    st = lib().orc_cones_scan(rp, xp, up, gp, G, R, cp, ctypes.c_double(sd_start), ctypes.c_double(sd_end),
                              ctypes.c_double(sd_end if sd_end_hi is None else sd_end_hi), int(backward_only),
                              K.ctypes.data_as(_dp), sd.ctypes.data_as(_dp), u.ctypes.data_as(_dp), ctypes.byref(fs))
    return dict(K=K, sd=None if backward_only else sd, u=None if backward_only else u[:G - 1], status=int(st),
                fail_stage=fs.value)


def feasible(rows, xbound, grid, cones, ubox=None):
    rows, rp = _d(rows)
    xb, xp = _d(xbound)
    grid, gp = _d(grid)
    cones, cp = _d(cones)
    ub, up = _d(ubox)
    G, _, R = rows.shape
    X = np.zeros((G, 2))
    lib().orc_cones_feasible(rp, xp, up, gp, G, R, cp, X.ctypes.data_as(_dp))
    return X


def sd_forward(rows, grid, cones, K, sd_start=0.0, slow=False, ubox=None):
    """One TOPPRAsd pass (orc_cones_sd_forward).  Returns (x [G] = sd^2, u [G-1], status, fail_stage)."""
    rows, rp = _d(rows)
    grid, gp = _d(grid)
    cones, cp = _d(cones)
    K, kp = _d(K)
    ub, up = _d(ubox)
    G, _, R = rows.shape
    x, u = np.zeros(G), np.zeros(max(G - 1, 1))
    fs = ctypes.c_int()
    st = lib().orc_cones_sd_forward(rp, up, gp, G, R, cp, kp, ctypes.c_double(sd_start), int(slow),
                                    x.ctypes.data_as(_dp), u.ctypes.data_as(_dp), ctypes.byref(fs))
    return x, u[:G - 1], int(st), fs.value


def socp(g, a, b, c, cones, xl, xh, xnext=None, ubox=None):
    """One stage problem (orc_cones_socp).  Returns (u, x)."""
    g, gp = _d(g)
    a, ap = _d(a)
    b, bp = _d(b)
    c, cpp = _d(c)
    cones, cp = _d(cones)
    xn, xnp = _d(xnext)
    ub, up = _d(ubox)
    out = np.zeros(2)
    lib().orc_cones_socp(gp, ap, bp, cpp, len(a), cp, ctypes.c_double(xl), ctypes.c_double(xh), xnp, up,
                         out.ctypes.data_as(_dp))
    return out


def reachable(rows, xbound, grid, cones, X, sdmin=0.0, sdmax=None, ubox=None):
    """Reachable sets (orc_cones_reachable).  Returns (L [G, 2], fail_stage)."""
    rows, rp = _d(rows)
    xb, xp = _d(xbound)
    grid, gp = _d(grid)
    cones, cp = _d(cones)
    X, Xp = _d(X)
    ub, up = _d(ubox)
    G, _, R = rows.shape
    L = np.zeros((G, 2))
    fs = lib().orc_cones_reachable(rp, xp, up, gp, G, R, cp, Xp, ctypes.c_double(sdmin),
                                   ctypes.c_double(sdmin if sdmax is None else sdmax), L.ctypes.data_as(_dp))
    return L, int(fs)
