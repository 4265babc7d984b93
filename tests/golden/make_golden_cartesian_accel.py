"""Generates tests/golden/cartesian_acceleration.npz: the UNMODIFIED reference (oracle/_ref, built by
oracle/build_ref.sh) solving problems with a Cartesian acceleration limit on a frame of the two robot fixtures
(tests/golden/robots/*.urdf), for tests/test_cartesian_acceleration.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_cartesian_accel.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 random waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is the reference's own
SecondOrderConstraint(inv_dyn, F, g, dof) in the form of its example examples-old/cartesian_accel.py: F = [I_k; -I_k],
g = [upper; -lower].  inv_dyn returns the selected components of the frame's classical acceleration from the 50-digit
reference of tests/kin_acc_ref.py (rnea_ref.MpRobot on the RAW URDF tree, placements differentiated twice by
mpmath.diff), rounded to fp64.  The values are computed beforehand in a process pool and looked up by the exact bytes of
(q, qd, qdd); acc(q, 0, 0) is exactly 0.  Each path's limits are, per component, half the largest |a u + b x| of its
solution without C, so that C is active.

Stored per robot `r` under "<r>/...": the inputs (way, vlim, alim, climit (B, k, 2)), the frame (link, xyz, rpy, ref)
and components, a and b (B, G, k) at the gridpoints, and "<r>/s<s>/" K, sd, sdd, status."""
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

import kin_acc_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
# the flange 0.1 m out (linear acceleration in world axes), and a point of the hand in its own coordinates (all six)
FRAMES = {"arm6": ("flange", (0.0, 0.0, 0.1), (0.0, 0.0, 0.0), "local_world_aligned", (0, 1, 2)),
          "arm7": ("hand", (0.02, -0.01, 0.12), (0.1, 0.2, -0.3), "local", (0, 1, 2, 3, 4, 5))}
NPATH, G = 8, 101
SEED0 = 6100

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


def _acc(args):
    """The selected components of the 50-digit classical acceleration at (q, qd, qdd), rounded to fp64."""
    from toppra_b200.dynamics import rpy_matrix
    q, qd, qdd = args
    link, xyz, rpy, ref, comps = FRAMES[_name]
    acc = kin_acc_ref.mp_accelerations(_robot, q, qd, qdd, {0: (link, rpy_matrix(rpy), np.asarray(xyz))})[0][ref]
    return np.array([float(acc[j]) for j in comps])


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
        nv = model.nv
        link, xyz, rpy, ref, comps = FRAMES[name]
        k = len(comps)
        probs = [problem(SEED0 + 100 * list(ROBOTS).index(name) + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        zero = np.zeros(nv)
        jobs, evals = [], []
        for path in paths:
            q, qs, qss = path(grid), path(grid, 1), path(grid, 2)
            for i in range(G):
                jobs += [(q[i], zero, qs[i]), (q[i], qs[i], qss[i])]
            evals.append((q, qs, qss))
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            vals = pool.map(_acc, jobs, chunksize=8)
        table = {}
        for (q, qd, qdd), v in zip(jobs, vals):
            table[(q.tobytes(), qd.tobytes(), qdd.tobytes())] = v
        a = np.array(vals[0::2]).reshape(NPATH, G, k)
        b = np.array(vals[1::2]).reshape(NPATH, G, k)

        def inv_dyn(q, qd, qdd):
            if not qd.any() and not qdd.any():
                return np.zeros(k)
            return table[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                          np.asarray(qdd, dtype=np.float64).tobytes())]

        climit = []
        for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
            free = algo.TOPPRA([constraint.JointVelocityConstraint(vlim), constraint.JointAccelerationConstraint(alim)],
                               path, gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, _ = free.compute_parameterization(0, 0, return_data=True)
            if sd is None:
                top = np.ones(k)
            else:
                top = np.max(np.abs(a[i, :-1] * sdd[:, None] + b[i, :-1] * (sd[:-1] ** 2)[:, None]), axis=0)
                top = np.where(top > 0, top, 1.0)
            climit.append(np.stack([-0.5 * top, 0.5 * top], axis=1))
        climit = np.array(climit)
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/climit" % name: climit,
                     "%s/a" % name: a, "%s/b" % name: b, "%s/link" % name: np.array(link),
                     "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy), "%s/ref" % name: np.array(ref),
                     "%s/components" % name: np.array(comps)})
        F = np.vstack((np.eye(k), -np.eye(k)))
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim), lim in zip(paths, probs, climit):
                g = np.concatenate((lim[:, 1], -lim[:, 0]))
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        constraint.SecondOrderConstraint(inv_dyn, lambda _: F, lambda _, g=g: g, nv,
                                                         discretization_scheme=scheme)]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
            for key, v in out.items():
                data["%s/s%d/%s" % (name, scheme, key)] = np.stack(v)
            print(name, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "cartesian_acceleration.npz"), **data)


if __name__ == "__main__":
    main()
