"""Generates tests/golden/long_paths.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh) and scipy on
LONG paths, 16 to 1000 knots, for tests/test_long_paths.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_long.py      # TOPPRA_REFERENCE: default /root/reference

Several kernels change their code path with the number of knots (DESIGN.md section 5, "Long paths"): the fit keeps its
scratch arrays in registers up to 16 knots, the fused scan needs the coefficients in 16 KB, the row builder caches them
in 32 KB.  The cases below sit on both sides of each switch.

  * fits: scipy's CubicSpline(x, y, bc_type).c for n in FIT_N, the three spacings of tests/problems.py (long_breaks) and
    six boundary conditions (not-a-knot, clamped, natural, ((1, d0), (1, d1)), ((2, d0), (1, d1)), periodic), one joint.
    The data are regenerated from seeds (problems.long_spline_data); n <= 116 stores the coefficients ("fit_<n>_<spacing>
    _<bc>"), n = 300 and 1000 the SHA-256 of their bytes ("fitsha_..."), which keeps the file small and is just as exact.
  * solves: TOPPRA(...).compute_parameterization (K, sd, sdd, return code) of the SOLVES table, inputs stored
    ("s<i>_..."), plus the SHA-256 of the reference's spline coefficients.
  * callers, for solves CALLERS: compute_feasible_sets, compute_reachable_sets, propose_gridpoints and TOPPRAsd at
    1.7 x the fastest duration ("s<i>_X", "_L", "_pg", "_sd_*")."""
import hashlib
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings("ignore")

from make_golden import ta  # noqa: E402
import toppra.algorithm as algo  # noqa: E402
import toppra.constraint as constraint  # noqa: E402
import toppra.interpolator as interp  # noqa: E402
from scipy.interpolate import CubicSpline  # noqa: E402

from problems import LONG_SPACINGS, long_breaks, long_spline_data, long_waypoints  # noqa: E402

FIT_N = (16, 17, 18, 33, 48, 49, 50, 114, 115, 116, 300, 1000)
FIT_HASHED = 300                 # n >= this: SHA-256 of the coefficients only
FIT_BC = ("not-a-knot", "clamped", "natural", "first", "mixed", "periodic")
# dof, knots, gridpoints, discretisation (1: interpolation), spacing, velocity-limited, sd_start; the comment names the
# switch the case sits next to (nseg = knots - 1)
SOLVES = (
    (7, 48, 200, 1, "uniform", False, 0.0),      # last fused nseg at dof 7 (47)
    (7, 49, 30, 0, "uneven", False, 0.0),        # first record-route nseg at dof 7, G < nseg
    (7, 114, 500, 1, "decades", False, 0.0),     # last nseg with K1's coefficients in shared memory at dof 7 (113)
    (7, 400, 1000, 1, "uniform", False, 0.0),    # G = 1000 at n = 400
    (6, 56, 40, 1, "uneven", False, 0.375),      # last fused nseg at dof 6 (55), G < nseg, sd_start^2 exact
    (6, 134, 150, 0, "uniform", True, 0.0),      # first K1 global-coefficient nseg at dof 6 (133), velocity-limited
    (3, 108, 60, 1, "decades", False, 0.0),      # last fused nseg at dof 3 (107), G < nseg
    (3, 257, 500, 0, "uneven", False, 0.0),      # first K1 global-coefficient nseg at dof 3 (256)
    (1, 293, 101, 1, "uniform", False, 0.0),     # last fused nseg at dof 1 (292), G < nseg
    (1, 684, 800, 1, "uneven", False, 0.0),      # first K1 global-coefficient nseg at dof 1 (683)
    (7, 115, 300, 1, "uneven", True, 0.0),       # first K1 global-coefficient nseg at dof 7 (114), velocity-limited
)
CALLERS = (0, 4)
SD_FACTOR = 1.7
REACH = (0.0, 0.5)
PROPOSE = dict(max_err_threshold=1e-3, max_seg_length=0.1, min_nb_points=100)


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).digest(), dtype=np.uint8)


def fit_bc(bc, seed, dof):
    """bc name -> scipy bc_type (the derivative values of the tuple forms are drawn from the seed)."""
    d0, d1 = np.random.RandomState(seed + 500000).randn(2, dof)
    return {"first": ((1, d0), (1, d1)), "mixed": ((2, d0), (1, d1))}.get(bc, bc)


def fit_seed(n, spacing):
    return 1000 * n + LONG_SPACINGS.index(spacing)


def fit_input(n, spacing, bc):
    x, y = long_spline_data(n, spacing, fit_seed(n, spacing))
    if bc == "periodic":
        y[-1] = y[0]
    return x, y, fit_bc(bc, fit_seed(n, spacing), y.shape[1])


def solve_input(i):
    dof, n, G, scheme, spacing, vel, sd0 = SOLVES[i]
    rng = np.random.RandomState(77000 + i)
    ss = long_breaks(rng, n, spacing)
    way = long_waypoints(rng, ss, dof)
    vl = (0.5 + rng.rand(dof)) if vel else 10 + 20 * rng.rand(dof)
    al = 10 + 2 * rng.rand(dof)
    return dict(ss=ss, way=way, vlim=np.stack((-vl, vl), 1), alim=np.stack((-al, al), 1), grid=np.linspace(0, ss[-1], G),
                scheme=np.int64(scheme), sd_start=np.float64(sd0))


def main():
    data = {}
    for n in FIT_N:
        for spacing in LONG_SPACINGS:
            for bc in FIT_BC:
                x, y, bct = fit_input(n, spacing, bc)
                c = CubicSpline(x, y, bc_type=bct).c
                key = "%d_%s_%s" % (n, spacing, bc)
                if n >= FIT_HASHED:
                    data["fitsha_" + key] = sha(c)
                else:
                    data["fit_" + key] = c
    codes = list(algo.ParameterizationReturnCode)
    for i in range(len(SOLVES)):
        p = solve_input(i)
        tag = "s%d_" % i
        data.update({tag + k: v for k, v in p.items()})
        path = ta.SplineInterpolator(p["ss"], p["way"])
        mk = lambda: [constraint.JointVelocityConstraint(p["vlim"]),  # noqa: E731
                      constraint.JointAccelerationConstraint(p["alim"], discretization_scheme=int(p["scheme"]))]
        inst = algo.TOPPRA(mk(), path, gridpoints=p["grid"], solver_wrapper="seidel")
        sdd, sd, _, K = inst.compute_parameterization(float(p["sd_start"]), 0.0, return_data=True)
        G = len(p["grid"])
        data[tag + "K"], data[tag + "c_sha"] = K, sha(path.cspl.c)
        data[tag + "sd"] = np.full(G, np.nan) if sd is None else sd
        data[tag + "sdd"] = np.full(G - 1, np.nan) if sdd is None else sdd
        data[tag + "status"] = np.int64(codes.index(inst.problem_data.return_code))
        if i not in CALLERS:
            continue
        data[tag + "X"] = algo.TOPPRA(mk(), path, gridpoints=p["grid"], solver_wrapper="seidel").compute_feasible_sets()
        data[tag + "L"] = algo.TOPPRA(mk(), path, gridpoints=p["grid"],
                                      solver_wrapper="seidel").compute_reachable_sets(*REACH)
        data[tag + "pg"] = np.asarray(interp.propose_gridpoints(path, **PROPOSE))
        assert sd is not None
        fastest = np.sum(2 * np.diff(p["grid"]) / (sd[1:] + sd[:-1]))
        sdi = algo.TOPPRAsd(mk(), path, gridpoints=p["grid"], solver_wrapper="seidel")
        sdi.set_desired_duration(fastest * SD_FACTOR)
        sdd_d, sd_d, _, _ = sdi.compute_parameterization(float(p["sd_start"]), 0.0, return_data=True)
        data[tag + "sd_desired"] = np.float64(fastest * SD_FACTOR)
        data[tag + "sd_sd"], data[tag + "sd_sdd"] = sd_d, sdd_d
        data[tag + "sd_status"] = np.int64(codes.index(sdi.problem_data.return_code))
    np.savez_compressed(os.path.join(HERE, "long_paths.npz"), **data)
    print("long_paths: %d fits, solve statuses %s, proposed grids %s" % (
        sum(k.startswith("fit") for k in data), [int(data["s%d_status" % i]) for i in range(len(SOLVES))],
        [len(data["s%d_pg" % i]) for i in CALLERS]))


if __name__ == "__main__":
    main()
