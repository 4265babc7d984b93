"""Generates tests/golden/poly_paths_k{5,6,7,8}.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving paths given as piecewise polynomials of order k = 5..8 (degree 4..7), for tests/test_piecewise_poly.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_poly.py      # TOPPRA_REFERENCE: default /root/reference

The reference takes any path object.  The one used here (RefPPolyPath) is an AbstractGeometricPath over
scipy.interpolate.PPoly with the convention of the reference's SplineInterpolator (interpolator.py:385-421): orders 1
and 2 are the chained derivative objects cspl.derivative() and cspld.derivative(), never pp(s, nu).

Every file stores the pieces (c, x), the inputs of each case and the reference's outputs under "<case>/<name>" keys."""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

from oracle.ref_loader import load_reference  # noqa: E402
from scipy.interpolate import BPoly, PPoly, make_interp_spline  # noqa: E402

ta = load_reference()
import toppra.algorithm as algo  # noqa: E402
import toppra.constraint as constraint  # noqa: E402
from toppra.interpolator import AbstractGeometricPath  # noqa: E402

DOF = 7


class RefPPolyPath(AbstractGeometricPath):
    """scipy PPoly path with SplineInterpolator's evaluation convention (chained derivative objects)."""

    def __init__(self, c, x):
        self.cspl = PPoly(c, x)
        self.cspld = self.cspl.derivative()
        self.cspldd = self.cspld.derivative()

    def __call__(self, path_positions, order=0):
        return (self.cspl, self.cspld, self.cspldd)[order](path_positions)

    @property
    def dof(self):
        return self.cspl.c.shape[2]

    @property
    def path_interval(self):
        return np.array([self.cspl.x[0], self.cspl.x[-1]])


def quintic_spline():
    """make_interp_spline(k=5) per joint over 9 non-uniform knots -> 4 pieces (the zero-length end pieces dropped)."""
    rng = np.random.RandomState(5)
    x = np.array([0.0, 0.1, 0.25, 0.4, 0.5, 0.62, 0.8, 0.9, 1.0])
    y = rng.randn(9, DOF)
    pps = [PPoly.from_spline(make_interp_spline(x, y[:, j], k=5)) for j in range(DOF)]
    keep = np.nonzero(np.diff(pps[0].x) > 0)[0]
    c = np.stack([p.c[:, keep] for p in pps], axis=-1)
    return c, pps[0].x[np.append(keep, keep[-1] + 1)]


def quintic_hermite():
    """BPoly.from_derivatives through positions, velocities and accelerations at 5 non-uniform knots -> 4 pieces."""
    rng = np.random.RandomState(6)
    xi = np.linspace(0, 1, 5) ** 1.3
    yi = rng.randn(5, 3, DOF) * np.array([1.0, 1.0, 3.0])[None, :, None]
    p = PPoly.from_bernstein_basis(BPoly.from_derivatives(xi, yi))
    return p.c, p.x


def random_pieces(k, nseg, seed):
    """Random order-k pieces on non-uniform breaks; higher powers get smaller coefficients."""
    rng = np.random.RandomState(seed)
    x = np.concatenate(([0.0], np.cumsum(0.5 + rng.rand(nseg))))
    x = x / x[-1]
    scale = 2.0 ** -np.arange(k)[::-1]
    c = rng.randn(k, nseg, DOF) * scale[:, None, None] * 3.0
    return c, x


def limits(seed, vel_active=False):
    rng = np.random.RandomState(seed)
    vl = (0.5 + rng.rand(DOF)) if vel_active else (10 + rng.rand(DOF) * 20)
    al = 10 + rng.rand(DOF) * 2
    return np.vstack((-vl, vl)).T, np.vstack((-al, al)).T


def solve(path, vlim, alim, grid, scheme=1, sd_start=0.0, sd_end=0.0):
    cons = [constraint.JointVelocityConstraint(vlim), constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)]
    inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
    sdd, sd, _, K = inst.compute_parameterization(sd_start, sd_end, return_data=True)
    out = dict(grid=np.asarray(inst.gridpoints, dtype=np.float64), vlim=vlim, alim=alim, scheme=np.int64(scheme),
               sd_start=np.float64(sd_start), sd_end=np.float64(sd_end), K=K, status=np.str_(inst.problem_data.return_code.name))
    out["sd"] = np.full(len(out["grid"]), np.nan) if sd is None else sd
    out["sdd"] = np.full(len(out["grid"]) - 1, np.nan) if sdd is None else sdd
    return inst, cons, out


def cases_for(c, x, seed):
    path = RefPPolyPath(c, x)
    vlim, alim = limits(seed)
    uni = np.linspace(x[0], x[-1], 101)
    rng = np.random.RandomState(seed + 1)
    non = np.concatenate(([x[0]], np.sort(x[0] + (x[-1] - x[0]) * rng.rand(78)), [x[-1]]))
    # path values at breakpoints, inside the pieces, outside the interval and NaN, through the reference's path object
    s = np.concatenate((x, 0.5 * (x[1:] + x[:-1]), np.linspace(x[0], x[-1], 23), [x[0] - 0.3, x[-1] + 0.2, np.nan]))
    out = {"path/c": c, "path/x": x, "path/s": s}
    for order in (0, 1, 2):
        out["path/q%d" % order] = path(s, order)
    cases = {}
    _, cons, cases["uniform_interp"] = solve(path, vlim, alim, uni, 1)
    _, _, cases["uniform_colloc"] = solve(path, vlim, alim, uni, 0)
    _, _, cases["nonuniform_interp"] = solve(path, vlim, alim, non, 1)
    _, _, cases["nonuniform_colloc"] = solve(path, vlim, alim, non, 0)
    vl2, _ = limits(seed, vel_active=True)
    _, _, cases["velocity_limited"] = solve(path, vl2, alim, uni, 1)
    _, _, cases["boundary_speeds"] = solve(path, vlim, alim, uni, 1, sd_start=0.25, sd_end=0.0625)
    _, _, cases["infeasible"] = solve(path, vlim, alim * 1e-3, uni, 1, sd_start=0.25)
    _, _, cases["proposed_grid"] = solve(path, vlim, alim, None, 1)
    for name, d in cases.items():
        for k, v in d.items():
            out["%s/%s" % (name, k)] = np.asarray(v)
    # feasible and reachable sets on the uniform grid, each from a fresh instance: the seidel wrapper warm-starts from
    # the LPs it solved before, which can change the last bits
    out["sets/X"] = algo.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel").compute_feasible_sets()
    out["sets/L"] = np.asarray(algo.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel")
                               .compute_reachable_sets(0.0, 0.0))
    # constraint parameters
    xb = cons[0].compute_constraint_params(path, uni)
    out["params/vel_xbound"] = xb[6]
    a, b, cc, F, g = cons[1].compute_constraint_params(path, uni)[:5]
    out["params/acc_a"], out["params/acc_b"], out["params/acc_c"] = a, b, cc
    out["params/acc_F"], out["params/acc_g"] = F, g
    # trajectories with both parametrizers: durations and evaluations at sample times
    ts = None
    for name in ("ParametrizeSpline", "ParametrizeConstAccel"):
        inst_p = algo.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel", parametrizer=name)
        traj = inst_p.compute_trajectory(0, 0)
        ts = np.linspace(0, traj.duration, 57)
        out["traj_%s/duration" % name] = np.float64(traj.duration)
        out["traj_%s/ts" % name] = ts
        for order in (0, 1, 2):
            out["traj_%s/q%d" % (name, order)] = traj(ts, order)
    # TOPPRAsd below, inside and above the achievable range
    fastest = float(out["traj_ParametrizeConstAccel/duration"])
    for label, want in (("below", 0.5 * fastest), ("inside", 1.5 * fastest), ("above", 1e4)):
        sd_inst = algo.TOPPRAsd(cons, path, gridpoints=uni, solver_wrapper="seidel")
        sd_inst.set_desired_duration(want)
        sdd, sd, _, K = sd_inst.compute_parameterization(0, 0, return_data=True)
        out["sd_%s/desired" % label] = np.float64(want)
        out["sd_%s/sd" % label] = sd
        out["sd_%s/sdd" % label] = sdd
    return out


def main():
    # k counts coefficients: quintic pieces (scipy's k=5 splines, quintic Hermite) have k = 6
    paths = {5: [("random", random_pieces(5, 4, 50))],
             6: [("spline", quintic_spline()), ("hermite", quintic_hermite())],
             7: [("random", random_pieces(7, 3, 70))],
             8: [("random", random_pieces(8, 6, 80))]}
    for k, items in paths.items():
        out = {}
        for label, (c, x) in items:
            assert c.shape[0] == k and c.shape[2] == DOF and np.all(np.diff(x) > 0)
            for key, v in cases_for(c, x, 100 * k + len(out)).items():
                out["%s/%s" % (label, key)] = v
        fn = os.path.join(HERE, "poly_paths_k%d.npz" % k)
        np.savez_compressed(fn, **out)
        print("wrote %s (%d arrays, %d bytes)" % (fn, len(out), os.path.getsize(fn)))


if __name__ == "__main__":
    main()
