"""Generates tests/golden/ragged_batch.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh) with
gridpoints=None, so that it proposes each path's grid itself (algorithm.py:92-106), for tests/test_ragged_and_chunked.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_ragged.py      # TOPPRA_REFERENCE: default /root/reference

The 16 paths of the frows_batch case (seeds 5000 + b, 7 DOF, the first four velocity-limited), each with
  * its proposed grid and length ("grid" padded with NaN, "glen");
  * TOPPRAsd at 0.5, 1.7, 3.0 and 1e6 x the fastest duration on that grid (path b takes factor b % 4); path 2 starts
    at a velocity it cannot leave (uncontrollable);
  * compute_feasible_sets;
  * compute_reachable_sets(sdmin, sdmax) with equal and unequal pairs (the 1-variable branch at stage 0), some of them
    failing;
and the first 8 paths with the frows_batch case's u-bound constraint (a LinearConstraint returning ubound and xbound)
in place of the acceleration constraint: compute_feasible_sets and compute_reachable_sets(0, 0.3) ("ub_*" keys).
Arrays are [16 or 8, Gmax(, 2)], NaN past each path's own grid."""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
warnings.filterwarnings("ignore")

from make_golden import make_path, solve_ref, ta  # noqa: E402
import toppra.algorithm as algo  # noqa: E402
import toppra.constraint as constraint  # noqa: E402

B, DOF = 16, 7
FACTORS = (0.5, 1.7, 3.0, 1e6)
SD_START_FAIL = 2          # this path starts TOPPRAsd at a velocity outside its controllable set
UB_ULIM = np.array([0.3, 0.1, 0.12, 0.08, 0.6, 0.4, 0.5, 0.2])


class UBoundConstraint(constraint.LinearConstraint):
    """frows_batch's constraint: the acceleration rows plus a u-interval that tightens with s and an x-bound."""

    def __init__(self, acc, ulim):
        super(UBoundConstraint, self).__init__()
        self.acc, self.ulim = acc, ulim
        self.discretization_type = acc.discretization_type
        self.identical = True

    def get_dof(self):
        return self.acc.get_dof()

    def compute_constraint_params(self, path, gridpoints, *a):
        pa, pb, pc, F, g, _, _ = self.acc.compute_constraint_params(path, gridpoints)
        n = len(gridpoints)
        ub = np.stack((-self.ulim * (1.0 + gridpoints), self.ulim * (2.0 - gridpoints)), axis=1)
        xb = np.stack((np.zeros(n), 40.0 + 30 * gridpoints), axis=1)
        return pa, pb, pc, F, g, ub, xb


def main():
    ss = np.linspace(0, 1, 5)
    probs = [make_path(5000 + b, dof=DOF) for b in range(B)]
    way = np.stack([p[0] for p in probs])
    vlim = np.stack([p[1] for p in probs])
    alim = np.stack([p[2] for p in probs])
    vlim[:4] *= 0.04
    sdmin = np.where(np.arange(B) % 3 == 0, 0.0, 0.2)
    sdmax = np.where(np.arange(B) % 2 == 0, sdmin, sdmin + 0.5)
    sd_start = np.zeros(B)
    sd_start[SD_START_FAIL] = 50.0
    grids, out = [], {k: [] for k in ("sd", "sdd", "status", "desired", "X", "L")}
    for b in range(B):
        cons = lambda: [constraint.JointVelocityConstraint(vlim[b]), constraint.JointAccelerationConstraint(alim[b])]  # noqa: E731
        path = ta.SplineInterpolator(ss, way[b])
        inst = algo.TOPPRA(cons(), path, solver_wrapper="seidel")
        grid = np.asarray(inst.gridpoints)
        grids.append(grid)
        out["X"].append(inst.compute_feasible_sets())
        out["L"].append(algo.TOPPRA(cons(), path, solver_wrapper="seidel").compute_reachable_sets(sdmin[b], sdmax[b]))
        o, _ = solve_ref(ss, way[b], vlim[b], alim[b], grid)
        fastest = np.sum(2 * np.diff(grid) / (o["sd"][1:] + o["sd"][:-1]))
        out["desired"].append(fastest * FACTORS[b % 4])
        sdi = algo.TOPPRAsd(cons(), path, solver_wrapper="seidel")
        assert np.array_equal(np.asarray(sdi.gridpoints), grid)
        sdi.set_desired_duration(out["desired"][-1])
        sdd, sd, _, _ = sdi.compute_parameterization(sd_start[b], 0, return_data=True)
        n = len(grid)
        out["sd"].append(np.full(n, np.nan) if sd is None else sd)
        out["sdd"].append(np.full(n - 1, np.nan) if sdd is None else sdd)
        out["status"].append(list(algo.ParameterizationReturnCode).index(sdi.problem_data.return_code))
    ub_X, ub_L = [], []
    for b in range(len(UB_ULIM)):
        path = ta.SplineInterpolator(ss, way[b])
        mk = lambda: [constraint.JointVelocityConstraint(vlim[b]),  # noqa: E731
                      UBoundConstraint(constraint.JointAccelerationConstraint(alim[b]), UB_ULIM[b])]
        inst = algo.TOPPRA(mk(), path, solver_wrapper="seidel")
        assert np.array_equal(np.asarray(inst.gridpoints), grids[b])
        ub_X.append(inst.compute_feasible_sets())
        ub_L.append(algo.TOPPRA(mk(), path, solver_wrapper="seidel").compute_reachable_sets(0.0, 0.3))
    glen = np.array([len(g) for g in grids], dtype=np.int32)
    G = int(glen.max())

    def pad(rows, width, tail=()):
        arr = np.full((len(rows), width) + tail, np.nan)
        for b, r in enumerate(rows):
            arr[b, :len(r)] = r
        return arr

    data = dict(ss=ss, way=way, vlim=vlim, alim=alim, sdmin=sdmin, sdmax=sdmax, sd_start=sd_start, glen=glen,
                grid=pad(grids, G), sd_desired=np.array(out["desired"]), sd_sd=pad(out["sd"], G),
                sd_sdd=pad(out["sdd"], G - 1), sd_status=np.array(out["status"], dtype=np.int32),
                X=pad(out["X"], G, (2,)), L=pad(out["L"], G, (2,)), ub_ulim=UB_ULIM, ub_X=pad(ub_X, G, (2,)),
                ub_L=pad(ub_L, G, (2,)))
    np.savez_compressed(os.path.join(HERE, "ragged_batch.npz"), **data)
    print("ragged_batch: glen", glen, "| sd status", data["sd_status"],
          "| u-bound reachable failures", [int(np.isnan(L[:, 0]).any()) for L in ub_L])


if __name__ == "__main__":
    main()
