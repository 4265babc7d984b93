"""Generates tests/golden/cartesian_velocity.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems with a Cartesian speed limit on a frame of the two robot fixtures (tests/golden/robots/*.urdf), for
tests/test_cartesian_velocity.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_cartesian.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 random waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel").  C is a `LinearConstraint`
subclass of the reference returning (0, b, 0, [[1]], [limit]) (collocation; the reference's
canlinear_colloc_to_interpolate for interpolation) with b = v^T S v of the frame velocity v from the 50-digit reference of
tests/kin_ref.py (rnea_ref.MpRobot on the RAW URDF tree, placements differentiated by mpmath.diff), rounded to fp64.
Each path's limit is half the largest v^T S v sd^2 of its solution without C, so that C is active.

Stored per robot `r` under "<r>/...": the inputs (way, vlim, alim, limit), the frame (link, xyz, rpy, ref) and S, b at
the gridpoints, and "<r>/s<s>/" K, sd, sdd, status."""
import multiprocessing
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

import kin_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
# tool-centre points: the flange 0.1 m out (translational speed), and a point of the hand in its own coordinates with a
# weighted, coupled S
FRAMES = {"arm6": ("flange", (0.0, 0.0, 0.1), (0.0, 0.0, 0.0), "local_world_aligned"),
          "arm7": ("hand", (0.02, -0.01, 0.12), (0.1, 0.2, -0.3), "local")}
S_ARM7 = np.diag([1.0, 1.5, 0.8, 0.04, 0.03, 0.05])
S_ARM7[0, 1] = S_ARM7[1, 0] = 0.2
S_ARM7[2, 4] = S_ARM7[4, 2] = 0.01
SMAT = {"arm6": np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]), "arm7": S_ARM7}
NPATH, G = 8, 101
SEED0 = 5200

_robot = None
_name = None


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def problem(seed, nv, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (5, nv)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    alim = np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1)
    return way, vlim, alim


def _init(name):
    global _robot, _name
    _robot = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])
    _name = name


def _b(args):
    """v^T S v at 50 digits, v the frame velocity at (q, qs)."""
    import mpmath
    from toppra_b200.dynamics import rpy_matrix
    q, qs = args
    link, xyz, rpy, ref = FRAMES[_name]
    f = kin_ref.mp_frames(_robot, q, qs, {0: (link, rpy_matrix(rpy), np.asarray(xyz))})[0]
    with mpmath.workdps(kin_ref.DPS):
        v = f["v"][ref]
        S = SMAT[_name]
        return float(mpmath.fsum(v[i] * mpmath.fsum(mpmath.mpf(float(S[i, j])) * v[j] for j in range(6))
                                 for i in range(6)))


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    from toppra.constraint.linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate
    from toppra.constraint.constraint import DiscretizationType
    codes = list(algo.ParameterizationReturnCode)

    class SpeedLimit(LinearConstraint):
        def __init__(self, b, limit, scheme):
            super(SpeedLimit, self).__init__()
            self.b, self.limit, self.identical = b, limit, True
            self.discretization_type = DiscretizationType(scheme)

        def compute_constraint_params(self, path, gridpoints):
            n = len(gridpoints)
            a, b, c = np.zeros((n, 1)), self.b.reshape(n, 1).copy(), np.zeros((n, 1))
            F, g = np.ones((1, 1)), np.full(1, self.limit)
            if self.discretization_type == DiscretizationType.Interpolation:
                return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
            return a, b, c, F, g, None, None

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid}
    for name in ROBOTS:
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits and DOF count only
        probs = [problem(SEED0 + 100 * list(ROBOTS).index(name) + p, model.nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs = path(grid), path(grid, 1)
            jobs += [(q[i], qs[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            bs = np.array(pool.map(_b, jobs, chunksize=8)).reshape(NPATH, G)
        limits = []
        for path, (way, vlim, alim), b in zip(paths, probs, bs):
            free = algo.TOPPRA([constraint.JointVelocityConstraint(vlim), constraint.JointAccelerationConstraint(alim)],
                               path, gridpoints=grid, solver_wrapper="seidel")
            _, sd, _, _ = free.compute_parameterization(0, 0, return_data=True)
            limits.append(0.5 * float(np.max(b * sd ** 2)) if sd is not None else 1.0)
        link, xyz, rpy, ref = FRAMES[name]
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/limit" % name: np.array(limits),
                     "%s/b" % name: bs, "%s/S" % name: SMAT[name], "%s/link" % name: np.array(link),
                     "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy), "%s/ref" % name: np.array(ref)})
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim), b, lim in zip(paths, probs, bs, limits):
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        SpeedLimit(b, lim, scheme)]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
            for k, v in out.items():
                data["%s/s%d/%s" % (name, scheme, k)] = np.stack(v)
            print(name, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "cartesian_velocity.npz"), **data)


if __name__ == "__main__":
    main()
