"""Generates tests/golden/support_stability.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems where a robot stands on a support it is not bolted to, for tests/test_support_stability.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_support.py   # TOPPRA_REFERENCE: default /root/reference

Robots: "mobile", tests/golden/robots/mobile_arm.urdf with its four wheels locked (a parked mobile manipulator on its
base_footprint), and "arm6", arm6.urdf on its 4 kg base_link standing on the floor.  Each robot: 8 spline paths
(5 waypoints), G = 101, both discretisation schemes and two footprints, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is the reference's own
SecondOrderConstraint(inv_dyn, F, g, dof) with g = 0 and F either the contact wrench cone of a rectangle with friction
("rect": contact_wrench_cone) or the ZMP rows of a convex polygon ("poly": support_polygon_rows).  inv_dyn returns the
support wrench from the 50-digit reference of tests/support_ref.py (rnea_ref.MpRobot on the RAW URDF tree, link
placements differentiated by mpmath.diff), rounded to fp64.  The values are computed beforehand in a process pool and
looked up by the exact bytes of (q, qd, qdd).

How the waypoints are chosen: the robot must stand stably at every gridpoint, or every problem would be infeasible at
rest.  Each robot has a start pose UP whose centre of mass lies above the middle of both footprints (found by
minimising the squared distance of the static zero-moment point from FOOTPRINT_CENTRE from random starts; stored as
"<r>/up").  Each path starts at UP and takes four random steps of at most STEP per joint; a path whose static
zero-moment point leaves either footprint (with a 10 % margin) anywhere along it is drawn again.

Stored per robot `r` under "<r>/...": the inputs (way, vlim, alim), the support frame (link, xyz, rpy), the base
(packed m_b, c_b), the footprints (half_lengths, friction, polygon), a, b and c (B, G, 6) at the gridpoints, and
"<r>/<form>/s<s>/" K, sd, sdd, status."""
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
import support_ref  # noqa: E402

WHEELS = {"wheel_fl_joint": 0.3, "wheel_fr_joint": -1.2, "wheel_rl_joint": 2.0, "wheel_rr_joint": 0.0}
ROBOTS = {"mobile": ("mobile_arm.urdf", WHEELS), "arm6": ("arm6.urdf", None)}
# the support frame: the footprint of the mobile base; for the arm, its base_link turned 0.4 rad about the floor normal
FRAMES = {"mobile": ("base_footprint", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)),
          "arm6": ("base_link", (0.06, -0.01, 0.0), (0.0, 0.0, 0.4))}
# footprints: a rectangle with friction, and a convex polygon (support axes, counter-clockwise); small enough that
# fast motions move the zero-moment point to their edges
FOOTPRINTS = {
    "mobile": dict(half_lengths=(0.05, 0.04), friction=0.5,
                   polygon=np.array([[-0.04, -0.045], [0.045, -0.04], [0.055, 0.01], [0.02, 0.045], [-0.045, 0.035]])),
    "arm6": dict(half_lengths=(0.04, 0.035), friction=0.6,
                 polygon=np.array([[-0.035, -0.04], [0.04, -0.035], [0.05, 0.015], [0.0, 0.045], [-0.04, 0.03]])),
}
FOOTPRINT_CENTRE = {"mobile": (0.005, -0.002), "arm6": (0.005, 0.0)}
STEP = {"mobile": 0.2, "arm6": 0.15}      # rad per joint and waypoint (m for the torso lift: times PRISMATIC_STEP)
PRISMATIC_STEP = 0.1
ALIM = {"mobile": 20.0, "arm6": 15.0}   # joint acceleration limits, rad/s^2 (m/s^2)
NPATH, G = 8, 101
SEED0 = 8300

_robot = None
_name = None


def urdf_text(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def footprint_rows(name):
    from toppra_b200.constraint import contact_wrench_cone, support_polygon_rows
    fp = FOOTPRINTS[name]
    return {"rect": contact_wrench_cone(fp["half_lengths"], fp["friction"]), "poly": support_polygon_rows(fp["polygon"])}


def static_zmp(model, frame, q):
    z = np.zeros_like(q)
    return support_ref.zmp(support_ref.support_wrench_packed(model.packed, frame.packed, model.packed_base(), q, z, z))


def stable(name, zmp, margin=0.1):
    """Whether the zero-moment points (n, 2) lie inside both footprints shrunk by `margin`."""
    X, Y = FOOTPRINTS[name]["half_lengths"]
    inside = (np.abs(zmp[:, 0]) <= (1 - margin) * X) & (np.abs(zmp[:, 1]) <= (1 - margin) * Y)
    P = FOOTPRINTS[name]["polygon"]
    c = P.mean(axis=0)
    Pm = c + (1 - margin) * (P - c)
    E = np.roll(Pm, -1, axis=0) - Pm
    side = E[None, :, 0] * (zmp[:, None, 1] - Pm[None, :, 1]) - E[None, :, 1] * (zmp[:, None, 0] - Pm[None, :, 0])
    return bool(inside.all() and (side >= 0).all())


def up_pose(name, model, frame, seed):
    """A configuration whose static zero-moment point is FOOTPRINT_CENTRE, near a random pose."""
    from scipy.optimize import minimize
    rng = np.random.RandomState(seed)
    target = np.asarray(FOOTPRINT_CENTRE[name])
    lo = np.where(model.packed[4::27][:model.nv] == 1, 0.05, -2.0)
    hi = np.where(model.packed[4::27][:model.nv] == 1, 0.25, 2.0)

    def cost(x):
        return float(np.sum((static_zmp(model, frame, x[None])[0] - target) ** 2))
    best = min((minimize(cost, rng.uniform(lo, hi)) for _ in range(10)), key=lambda r: r.fun)
    assert best.fun < 1e-8, best.fun
    return best.x


def problem(name, model, frame, up, seed, ss, grid):
    """(way, vlim, alim) of one path from `up`; drawn again until it stands stably everywhere (static ZMP)."""
    from scipy.interpolate import CubicSpline
    nv = len(up)
    step = np.where(model.packed[4::27][:nv] == 1, STEP[name] * PRISMATIC_STEP, STEP[name])
    rng = np.random.RandomState(seed)
    while True:
        way = up + np.cumsum(np.vstack((np.zeros((1, nv)), rng.uniform(-1, 1, (4, nv)) * step)), axis=0)
        q = CubicSpline(ss, way)(np.linspace(0, 1, 4 * len(grid)))
        if stable(name, static_zmp(model, frame, q)):
            break
    vel = np.where(np.isfinite(model.velocity_limit), model.velocity_limit, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    alim = np.stack([-np.full(nv, ALIM[name]), np.full(nv, ALIM[name])], axis=1)
    return way, vlim, alim


def setup(name):
    """(model, support frame) of robot `name`."""
    from toppra_b200.dynamics import RigidBodyModel
    model = RigidBodyModel.from_urdf(urdf_text(name), ROBOTS[name][1])
    link, xyz, rpy = FRAMES[name]
    return model, model.frame(link, xyz=xyz, rpy=rpy)


def _init(name):
    global _robot, _name
    _robot = rnea_ref.MpRobot.from_urdf(urdf_text(name), ROBOTS[name][1])
    _name = name


def _wrench(args):
    """The 50-digit support wrench at (q, qd, qdd), rounded to fp64."""
    from toppra_b200.dynamics import rpy_matrix
    q, qd, qdd = args
    link, xyz, rpy = FRAMES[_name]
    R, p = _robot._kinematics([0.0] * _robot.nv)[0][link]      # the link's placement on the base (fixed)
    R = np.array([[float(R[i, j]) for j in range(3)] for i in range(3)])
    p = np.array([float(x) for x in p])
    w = support_ref.mp_support_wrench(_robot, q, qd, qdd, R @ rpy_matrix(rpy), p + R @ np.asarray(xyz))
    return np.array([float(x) for x in w])


def main():
    from oracle.ref_loader import load_reference
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    codes = list(algo.ParameterizationReturnCode)

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid}
    for r, name in enumerate(ROBOTS):
        model, frame = setup(name)
        nv = model.nv
        up = up_pose(name, model, frame, SEED0 + 50 * r)
        probs = [problem(name, model, frame, up, SEED0 + 100 * r + p, ss, grid) for p in range(NPATH)]
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

        def inv_dyn(q, qd, qdd):
            return table[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                          np.asarray(qdd, dtype=np.float64).tobytes())]

        link, xyz, rpy = FRAMES[name]
        fp = FOOTPRINTS[name]
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/up" % name: up,
                     "%s/a" % name: w1 - w0, "%s/b" % name: w2 - w0, "%s/c" % name: w0,
                     "%s/link" % name: np.array(link), "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy),
                     "%s/base" % name: model.packed_base(), "%s/half_lengths" % name: np.array(fp["half_lengths"]),
                     "%s/friction" % name: np.array(fp["friction"]), "%s/polygon" % name: fp["polygon"]})
        for form, F in footprint_rows(name).items():
            assert (np.einsum("kj,bgj->bgk", F, w0) < 0).all(), "the robot must stand stably at every gridpoint"
            zeros = np.zeros(F.shape[0])
            for scheme in (0, 1):
                out = {"K": [], "sd": [], "sdd": [], "status": []}
                active = 0
                for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
                    cons = [constraint.JointVelocityConstraint(vlim),
                            constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            constraint.SecondOrderConstraint(inv_dyn, lambda _, F=F: F, lambda _, z=zeros: z, nv,
                                                             discretization_scheme=scheme)]
                    inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                    sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                    out["K"].append(K)
                    out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                    out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                    out["status"].append(codes.index(inst.problem_data.return_code))
                    if sd is not None:
                        w = (w1 - w0)[i, :-1] * sdd[:, None] + (w2 - w0)[i, :-1] * (sd[:-1] ** 2)[:, None] + w0[i, :-1]
                        v = w @ F.T
                        active += bool((v >= -1e-6 * np.abs(w).max(axis=1, keepdims=True)).any())
                for key, v in out.items():
                    data["%s/%s/s%d/%s" % (name, form, scheme, key)] = np.stack(v)
                print(name, form, "scheme", scheme, "statuses", out["status"], "support rows active on", active)
    np.savez_compressed(os.path.join(HERE, "support_stability.npz"), **data)


if __name__ == "__main__":
    main()
