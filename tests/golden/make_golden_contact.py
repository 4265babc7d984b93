"""Generates tests/golden/contact_stability.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems where the robot carries an object on a tray (the contact frame), for tests/test_contact_stability.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_contact.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is the reference's own
SecondOrderConstraint(inv_dyn, F, g, dof) with F the 16 x 6 contact wrench cone of the tray (contact_wrench_cone) and
g = 0.  inv_dyn returns the contact wrench from the 50-digit reference of tests/contact_ref.py (rnea_ref.MpRobot on the
RAW URDF tree, placements differentiated by mpmath.diff), rounded to fp64.  The values are computed beforehand in a
process pool and looked up by the exact bytes of (q, qd, qdd).

How the waypoints are chosen: the object must rest stably on the tray at every gridpoint, or every problem would be
infeasible at rest.  Each robot has a pose UP where the tray's z axis points straight up (found by minimising
1 - R_f[2, 2] from random starts; stored as "<r>/up").  Each path starts at UP and takes four random steps of at most
0.06 rad per joint, so the tray stays within a few degrees of level, well inside the sliding angle atan(mu) and the
tipping angle of the object.

Stored per robot `r` under "<r>/...": the inputs (way, vlim, alim), the frame (link, xyz, rpy), the object (packed:
m, r, Ic), half_lengths and friction, a, b and c (B, G, 6) at the gridpoints, and "<r>/s<s>/" K, sd, sdd, status."""
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

import contact_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
# the tray: on the flange 1 cm out; on the hand 12 cm out and turned 0.3 rad about its normal
FRAMES = {"arm6": ("flange", (0.0, 0.0, 0.01), (0.0, 0.0, 0.0)),
          "arm7": ("hand", (0.0, 0.0, 0.12), (0.0, 0.0, 0.3))}
# a 0.8 kg box, centre of mass 6 cm above the tray and slightly off centre, on a 10 x 8 cm base, mu = 0.5
OBJECT = contact_ref.object_packed(0.8, (0.006, -0.004, 0.06), (0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017))
HALF_LENGTHS, FRICTION = (0.05, 0.04), 0.5
NPATH, G = 8, 101
SEED0 = 7300

_robot = None
_name = None


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def up_pose(model, frame, seed):
    """A configuration where the frame's z axis points up (world +z)."""
    import kin_ref
    from scipy.optimize import minimize
    rng = np.random.RandomState(seed)

    def cost(x):
        return 1.0 - kin_ref.frame_packed(model.packed, frame.packed, x[None], np.zeros((1, model.nv)))[0][0][2, 2]
    best = min((minimize(cost, rng.uniform(-2, 2, model.nv)) for _ in range(20)), key=lambda r: r.fun)
    assert best.fun < 1e-12, best.fun
    return best.x


def problem(seed, up, velocity):
    nv = len(up)
    rng = np.random.RandomState(seed)
    way = up + np.cumsum(np.vstack((np.zeros((1, nv)), rng.uniform(-0.06, 0.06, (4, nv)))), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    alim = np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1)
    return way, vlim, alim


def _init(name):
    global _robot, _name
    _robot = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])
    _name = name


def _wrench(args):
    """The 50-digit contact wrench at (q, qd, qdd), rounded to fp64."""
    from toppra_b200.dynamics import rpy_matrix
    q, qd, qdd = args
    link, xyz, rpy = FRAMES[_name]
    w = contact_ref.mp_wrenches(_robot, q, qd, qdd, {0: (link, rpy_matrix(rpy), np.asarray(xyz))}, OBJECT)[0]
    return np.array([float(x) for x in w])


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.constraint import contact_wrench_cone
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    codes = list(algo.ParameterizationReturnCode)

    F = contact_wrench_cone(HALF_LENGTHS, FRICTION)
    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid, "object": OBJECT, "half_lengths": np.array(HALF_LENGTHS),
            "friction": np.array(FRICTION)}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits, DOF count and the up pose
        nv = model.nv
        link, xyz, rpy = FRAMES[name]
        up = up_pose(model, model.frame(link, xyz=xyz, rpy=rpy), SEED0 + 50 * r)
        probs = [problem(SEED0 + 100 * r + p, up, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        zero = np.zeros(nv)
        jobs = []
        for path in paths:
            q, qs, qss = path(grid), path(grid, 1), path(grid, 2)
            for i in range(G):
                jobs += [(q[i], zero, zero), (q[i], zero, qs[i]), (q[i], qs[i], qss[i])]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            vals = pool.map(_wrench, jobs, chunksize=8)
        table = {}
        for (q, qd, qdd), v in zip(jobs, vals):
            table[(q.tobytes(), qd.tobytes(), qdd.tobytes())] = v
        w0, w1, w2 = (np.array(vals[j::3]).reshape(NPATH, G, 6) for j in range(3))
        assert (np.einsum("kj,bgj->bgk", F, w0) < 0).all(), "the object must rest stably at every gridpoint"

        def inv_dyn(q, qd, qdd):
            return table[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                          np.asarray(qdd, dtype=np.float64).tobytes())]

        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/up" % name: up,
                     "%s/a" % name: w1 - w0, "%s/b" % name: w2 - w0, "%s/c" % name: w0,
                     "%s/link" % name: np.array(link), "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy)})
        zeros = np.zeros(F.shape[0])
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim) in zip(paths, probs):
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        constraint.SecondOrderConstraint(inv_dyn, lambda _: F, lambda _: zeros, nv,
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
    np.savez_compressed(os.path.join(HERE, "contact_stability.npz"), **data)


if __name__ == "__main__":
    main()
