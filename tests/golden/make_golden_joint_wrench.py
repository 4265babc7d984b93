"""Generates tests/golden/joint_wrench.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh) solving
problems with limits on the wrench across one joint, for tests/test_joint_wrench.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_joint_wrench.py   # TOPPRA_REFERENCE: default /root/reference

Robots: "arm6", tests/golden/robots/arm6.urdf, the wrench across joint 2 (shoulder_lift, frame upper_arm moved off the
joint), and "arm7", arm7_gripper.urdf with its fingers locked, the wrench across joint 4 (frame link4 moved and turned).
Each robot: 8 spline paths (5 random waypoints), G = 101, both discretisation schemes and two forms, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is the reference's own
SecondOrderConstraint(inv_dyn, F, g, dof) with
  "box":      F = [E; -E], g = [upper; -lower] on the components BOX_COMPONENTS (E selects them; in the frame's axes for
              arm6, world axes for arm7),
  "bearing":  F, g of toppra_b200.constraint.joint_wrench.bearing_rows (axial, radial and tilting limits, 8 sides) on the
              joint axis in the frame's axes.
inv_dyn returns the joint wrench from the 50-digit reference of tests/joint_wrench_ref.py (rnea_ref.MpRobot on the RAW
URDF tree, summed over the joint's subtree, link placements differentiated by mpmath.diff), rounded to fp64.  The values
are computed beforehand in a process pool and looked up by the exact bytes of (q, qd, qdd).

The limits come from the static loads w(q, 0, 0) of the 8 paths: each is 1.25 times the 6th largest of the paths'
largest static loads (at least 0.25 of the largest load of its kind).  So the fast parts of most paths hit the limits,
and the two paths with the largest static loads fail.

Stored per robot `r`: the inputs (way, vlim, alim), the frame (link, xyz, rpy, ref of the box form), the limits (wlim,
box_components, axial, radial, tilting), a, b and c (B, G, 6) of both reference frames' wrenches at the gridpoints
("<r>/local/a", ...; "<r>/world/a", ...), and "<r>/<form>/s<s>/" K, sd, sdd, status."""
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

import joint_wrench_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None),
          "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013, "finger_right_joint": 0.021})}
# (link, xyz, rpy, reference frame of the box form)
FRAMES = {"arm6": ("upper_arm", (0.0, 0.0, 0.04), (0.0, 0.0, 0.0), "local"),
          "arm7": ("link4", (0.01, -0.02, 0.03), (0.2, -0.1, 0.4), "local_world_aligned")}
BOX_COMPONENTS = (4, 0, 2, 3)       # unsorted on purpose: row i of wlim limits BOX_COMPONENTS[i]
SIDES = 8
NPATH, G = 8, 101
SEED0 = 9100

_robot = None


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def problem(seed, nv, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (5, nv)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    al = rng.uniform(6, 10, nv)
    return way, vlim, np.stack([-al, al], axis=1)


def setup(name):
    """(model, frame of the bearing form ("local"), frame of the box form)."""
    from toppra_b200.dynamics import RigidBodyModel
    model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])
    link, xyz, rpy, ref = FRAMES[name]
    return model, model.frame(link, xyz=xyz, rpy=rpy, reference_frame="local"), model.frame(link, xyz=xyz, rpy=rpy,
                                                                                            reference_frame=ref)


def _init(name):
    global _robot
    model, frame, _ = setup(name)
    _robot = (rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1]), frame)


def _wrenches(args):
    """The 50-digit joint wrench at (q, qd, qdd) in the frame's axes and in world axes, rounded to fp64."""
    q, qd, qdd = args
    mp, f = _robot
    return np.stack([joint_wrench_ref.mp_joint_wrench(mp, f.body, q, qd, qdd, f.R, f.p, ref)
                     for ref in (joint_wrench_ref.LOCAL, joint_wrench_ref.LOCAL_WORLD_ALIGNED)])


def _limit(loads, kind_scale):
    """1.25 times the 6th largest of the paths' largest loads, at least a quarter of the largest load of its kind."""
    per_path = np.sort(loads.reshape(NPATH, -1).max(axis=1))
    return max(1.25 * per_path[-6], 0.25 * kind_scale)


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.constraint.joint_wrench import bearing_rows
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    codes = list(algo.ParameterizationReturnCode)

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid, "box_components": np.array(BOX_COMPONENTS), "sides": np.array(SIDES)}
    for r, name in enumerate(ROBOTS):
        model, frame, box_frame = setup(name)
        nv = model.nv
        probs = [problem(SEED0 + 100 * r + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        zero = np.zeros(nv)
        jobs = []
        for path in paths:
            q, qs, qss = path(grid), path(grid, 1), path(grid, 2)
            for i in range(G):
                jobs += [(q[i], zero, zero), (q[i], zero, qs[i]), (q[i], qs[i], qss[i])]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            vals = np.array(pool.map(_wrenches, jobs, chunksize=8))          # (3 NPATH G, 2, 6)
        box_ref = 0 if FRAMES[name][3] == "local" else 1
        table = {}
        for (q, qd, qdd), v in zip(jobs, vals):
            table[(q.tobytes(), qd.tobytes(), qdd.tobytes())] = v
        link, xyz, rpy, ref = FRAMES[name]
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/link" % name: np.array(link),
                     "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy), "%s/ref" % name: np.array(ref)})
        for j, key in enumerate(("local", "world")):
            w0, w1, w2 = (vals[s::3, j].reshape(NPATH, G, 6) for s in range(3))
            data.update({"%s/%s/a" % (name, key): w1 - w0, "%s/%s/b" % (name, key): w2 - w0,
                         "%s/%s/c" % (name, key): w0})

        # limits from the static loads
        w0 = vals[0::3, 0]                                                   # local axes
        a = frame.R.T @ model.body(frame.body)[2:5]
        fa = w0[:, :3] @ a
        fr = np.linalg.norm(w0[:, :3] - fa[:, None] * a, axis=1)
        nt = np.linalg.norm(w0[:, 3:] - (w0[:, 3:] @ a)[:, None] * a, axis=1)
        fscale, nscale = np.abs(w0[:, :3]).max(), np.abs(w0[:, 3:]).max()
        axial, radial, tilting = _limit(np.abs(fa), fscale), _limit(fr, fscale), _limit(nt, nscale)
        wb = vals[0::3, box_ref]
        wlim = []
        for comp in BOX_COMPONENTS:
            scale = np.abs(wb[:, :3] if comp < 3 else wb[:, 3:]).max()
            L = _limit(np.abs(wb[:, comp]), scale)
            wlim.append([-L, L])
        wlim = np.array(wlim)
        data.update({"%s/wlim" % name: wlim, "%s/axial" % name: np.array(axial), "%s/radial" % name: np.array(radial),
                     "%s/tilting" % name: np.array(tilting)})

        E = np.eye(6)[list(BOX_COMPONENTS)]
        forms = {"box": (box_ref, np.vstack((E, -E)), np.concatenate((wlim[:, 1], -wlim[:, 0]))),
                 "bearing": (0,) + bearing_rows(a, axial, radial, tilting, SIDES)}
        for form, (j, F, g) in forms.items():
            def inv_dyn(q, qd, qdd, j=j):
                return table[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                              np.asarray(qdd, dtype=np.float64).tobytes())][j]
            for scheme in (0, 1):
                out = {"K": [], "sd": [], "sdd": [], "status": []}
                for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
                    cons = [constraint.JointVelocityConstraint(vlim),
                            constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            constraint.SecondOrderConstraint(inv_dyn, lambda _, F=F: F, lambda _, g=g: g, nv,
                                                             discretization_scheme=scheme)]
                    inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                    sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                    out["K"].append(K)
                    out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                    out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                    out["status"].append(codes.index(inst.problem_data.return_code))
                for key, v in out.items():
                    data["%s/%s/s%d/%s" % (name, form, scheme, key)] = np.stack(v)
                print(name, form, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "joint_wrench.npz"), **data)


if __name__ == "__main__":
    main()
