"""Generates tests/golden/drive_limits.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh) solving
problems with motor torque and motor speed limits of geared drives, for tests/test_drive_limits.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_drives.py      # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 random waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, SecondOrderConstraint(w, F = [I; -I], g,
custom_term = f o sign(T p'(s))), MotorSpeedRow], path, grid, "seidel").  w is the 50-digit motor torque of
tests/drive_ref.py (rnea_ref.MpRobot on the RAW URDF tree, T^-1 in mpmath) rounded to fp64; MotorSpeedRow is a reference
`LinearConstraint` subclass returning (a, b, c, F, g) = (0, b, -1, [[1]], [0]) with the 50-digit speed row b (lifted by
the reference's own `canlinear_colloc_to_interpolate` under Interpolation).  Both are looked up by the exact bytes of
their arguments.

arm6 has a coupled wrist, T = diag(n) C with C unit lower-triangular on the last three rows; arm7 (gripper fingers
locked) has T = diag(n).  The motor limits are chosen so that motor rows bind: the generator asserts that every solved
path is slower than the solution of the same path under its joint velocity and acceleration limits alone.

Stored per robot `r`: the inputs (way, vlim, alim, drive (packed), taulim (motor torques), omega (motor speeds)), the
motor-torque terms (a, b, c) and the speed row b at the gridpoints (collocation), and "<r>/s<s>/" K, sd, sdd, status."""
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

import drive_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None),
          "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013, "finger_right_joint": 0.021})}
NPATH, G = 8, 101
SEED0 = 7300

_robot = None


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def drive(name, nv):
    """The packed drive: gear ratios from 120 (base) to 50 (tool), rotor inertias from 4e-5 to 1e-5 kg m^2, 0.02 N m of
    motor friction; arm6's wrist motors are coupled."""
    n = np.linspace(120.0, 50.0, nv)
    C = np.eye(nv)
    if name == "arm6":
        C[4, 3], C[5, 3], C[5, 4] = 1.0, 0.5, -1.0
    return drive_ref.pack(np.diag(n) @ C, np.linspace(4e-5, 1e-5, nv), 0.02)


def problem(seed, nv, effort, velocity, n):
    """Waypoints, joint limits and motor limits of one path: motor torques at 45% of the URDF effort over the gear ratio,
    motor speeds at 70% of the URDF joint speed times the gear ratio."""
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (5, nv)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    eff = np.where(np.isfinite(effort), effort, 8.0)
    vlim = np.stack([-vel, vel], axis=1)
    al = rng.uniform(6, 10, nv)
    alim = np.stack([-al, al], axis=1)
    tm = 0.45 * eff / n
    return way, vlim, alim, np.stack([-tm, tm], axis=1), 0.7 * vel * n


def _init(name, packed):
    global _robot
    _robot = (rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1]), packed)


def _three(args):
    q, qs, qss = args
    mp, packed = _robot
    z = np.zeros_like(q)
    return [np.array([float(x) for x in drive_ref.mp_torque(mp, packed, q, a, b)]) for a, b in ((z, z), (z, qs),
                                                                                                 (qs, qss))]


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    from toppra.constraint.linear_constraint import canlinear_colloc_to_interpolate
    codes = list(algo.ParameterizationReturnCode)

    class MotorSpeedRow(constraint.LinearConstraint):
        def __init__(self, table, dof, scheme):
            super(MotorSpeedRow, self).__init__()
            self.table, self.dof, self.identical = table, dof, True
            self.set_discretization_type(scheme)

        def compute_constraint_params(self, path, gridpoints):
            b = np.array([[self.table[x.tobytes()]] for x in path(gridpoints, 1)])
            a, c = np.zeros_like(b), np.full_like(b, -1.0)
            F, g = np.ones((1, 1)), np.zeros(1)
            if self.discretization_type == constraint.DiscretizationType.Interpolation:
                return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
            return a, b, c, F, g, None, None

    def solve(cons, path):
        inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
        sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
        return sdd, sd, K, codes.index(inst.problem_data.return_code)

    def duration(sd):
        return np.sum(2 * np.diff(grid) / (sd[:-1] + sd[1:]))

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits and DOF count only
        nv = model.nv
        packed = drive(name, nv)
        T, _, fric = drive_ref.unpack(packed, nv)
        n = np.diag(T).copy()
        probs = [problem(SEED0 + 100 * r + p, nv, model.effort_limit, model.velocity_limit, n) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs, qss = (path(grid, o) for o in (0, 1, 2))
            jobs += [(q[i], qs[i], qss[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(name, packed)) as pool:
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

        def custom_term(path, s):
            return fric * np.sign(T @ path(s, 1))

        eyes = np.vstack((np.eye(nv), -np.eye(nv)))
        for key, idx in (("way", 0), ("vlim", 1), ("alim", 2), ("taulim", 3), ("omega", 4)):
            data["%s/%s" % (name, key)] = np.stack([pr[idx] for pr in probs])
        data[name + "/drive"] = packed
        terms = {"a": [], "b": [], "c": [], "speed": []}
        tables = []
        for path, pr in zip(paths, probs):
            qs = path(grid, 1)
            tables.append({x.tobytes(): float(drive_ref.mp_speed_row(packed, nv, pr[4], x)) for x in qs})
            terms["speed"].append([tables[-1][x.tobytes()] for x in qs])
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim, taulim, omega), table in zip(paths, probs, tables):
                g_aug = np.concatenate((taulim[:, 1], -taulim[:, 0]))
                pc = constraint.SecondOrderConstraint(inv_dyn, lambda _: eyes, lambda _: g_aug, nv, custom_term,
                                                      discretization_scheme=scheme)
                joint = [constraint.JointVelocityConstraint(vlim),
                         constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)]
                sdd, sd, K, st = solve(joint + [pc, MotorSpeedRow(table, nv, scheme)], path)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(st)
                if st == 0:
                    sd_joint = solve(joint, path)[1]
                    assert duration(sd) > (1 + 1e-3) * duration(sd_joint), (name, scheme, duration(sd),
                                                                             duration(sd_joint))
                if scheme == 0:
                    a, b, c = pc.compute_constraint_params(path, grid)[:3]
                    terms["a"].append(a)
                    terms["b"].append(b)
                    terms["c"].append(c)
            for k, v in out.items():
                data["%s/s%d/%s" % (name, scheme, k)] = np.stack(v)
            print(name, "scheme", scheme, "statuses", out["status"])
        for k, v in terms.items():
            data["%s/%s" % (name, k)] = np.stack(v)
    np.savez_compressed(os.path.join(HERE, "drive_limits.npz"), **data)


if __name__ == "__main__":
    main()
