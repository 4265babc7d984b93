"""Generates tests/golden/rigid_body_torque.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving torque-limited problems of the two robot fixtures (tests/golden/robots/*.urdf), for tests/test_rigid_body.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_rnea.py      # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 random waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, JointTorqueConstraint(inv_dyn, ...)], path, grid, "seidel").
inv_dyn returns the 50-digit Lagrangian reference of tests/rnea_ref.py (MpRobot on the RAW URDF tree, fixed and locked
joints as zero-DOF links) rounded to fp64.  The 7-DOF robot has its gripper fingers locked (LOCKED below).

Stored per robot `r` and scheme `s`, under "<r>/...": the inputs (way, vlim, alim, taulim, fric), the torque terms
(a, b, c) of the reference's JointTorqueConstraint at the gridpoints (collocation), and "<r>/s<s>/" K, sd, sdd, status."""
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

import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None),
          "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013, "finger_right_joint": 0.021})}
NPATH, G = 8, 101
SEED0 = 4100

_robot = None


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def problem(name, seed, nv, effort, velocity):
    """Waypoints and limits of one path: torque limits at 45% of the URDF efforts so that torque rows are active."""
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (5, nv)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    eff = np.where(np.isfinite(effort), effort, 8.0)
    vlim = np.stack([-vel, vel], axis=1)
    alim = np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1)
    taulim = np.stack([-0.45 * eff, 0.45 * eff], axis=1)
    fric = 0.2 + 0.1 * np.arange(nv)
    return way, vlim, alim, taulim, fric


def _init(name):
    global _robot
    _robot = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])


def _three(args):
    q, qs, qss = args
    z = np.zeros_like(q)
    return [_robot.tau64(q, z, z), _robot.tau64(q, z, qs), _robot.tau64(q, qs, qss)]


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    codes = list(algo.ParameterizationReturnCode)
    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid}
    for name in ROBOTS:
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits and DOF count only
        probs = [problem(name, SEED0 + p, model.nv, model.effort_limit, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs, qss = (path(grid, o) for o in (0, 1, 2))
            jobs += [(q[i], qs[i], qss[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            res = pool.map(_three, jobs, chunksize=4)
        cache = {}
        for (q, qs, qss), (t0, t1, t2) in zip(jobs, res):
            z = np.zeros_like(q)
            cache[(q.tobytes(), z.tobytes(), z.tobytes())] = t0
            cache[(q.tobytes(), z.tobytes(), qs.tobytes())] = t1
            cache[(q.tobytes(), qs.tobytes(), qss.tobytes())] = t2

        def inv_dyn(q, qd, qdd):
            return cache[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                           np.asarray(qdd, dtype=np.float64).tobytes())].copy()

        for key, idx in (("way", 0), ("vlim", 1), ("alim", 2), ("taulim", 3), ("fric", 4)):
            data["%s/%s" % (name, key)] = np.stack([pr[idx] for pr in probs])
        terms = {"a": [], "b": [], "c": []}
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim, taulim, fric) in zip(paths, probs):
                pc_tau = constraint.JointTorqueConstraint(inv_dyn, taulim, fric, discretization_scheme=scheme)
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme), pc_tau]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
                if scheme == 0:
                    a, b, c, _, _, _, _ = pc_tau.compute_constraint_params(path, grid)
                    terms["a"].append(a)
                    terms["b"].append(b)
                    terms["c"].append(c)
            for k, v in out.items():
                data["%s/s%d/%s" % (name, scheme, k)] = np.stack(v)
            print(name, "scheme", scheme, "statuses", out["status"])
        for k, v in terms.items():
            data["%s/%s" % (name, k)] = np.stack(v)
    np.savez_compressed(os.path.join(HERE, "rigid_body_torque.npz"), **data)


if __name__ == "__main__":
    main()
