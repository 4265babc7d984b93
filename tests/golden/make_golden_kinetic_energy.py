"""Generates tests/golden/kinetic_energy.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems with a limit on the kinetic energy or on the linear momentum of the whole robot, for
tests/test_kinetic_energy.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_kinetic_energy.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 waypoints), G = 101, both discretisation schemes, two limits ("energy": T <= E_max,
"momentum": |p| <= p_max), solved by TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid,
"seidel") where C is a reference `LinearConstraint` subclass returning (a, b, c, F, g) = (0, b, 0, [[1]], [limit])
(lifted by the reference's own `canlinear_colloc_to_interpolate` under Interpolation), with b = T(q, q') and limit
E_max, or b = |p(q, q')|^2 and limit p_max^2.  T and p come from the 50-digit reference of tests/momentum_ref.py
(rnea_ref.MpRobot on the RAW URDF tree: its mass matrix, and centre-of-mass Jacobians by mpmath.diff), rounded to fp64;
the values are computed beforehand in a process pool and looked up by the exact bytes of (q, q').

Each limit is 0.3 of the largest value (T, or |p|) on the reference's solution without it (Collocation), so that it
binds.  Per robot and limit, one path starts at a speed s'(0) that the joint limits admit but the limit does not, so
that its failure status is pinned.  Stored per robot `r` and limit `l`: the inputs under "<r>/" (way, vlim, alim),
"<r>/<l>/" limit (E_max or p_max, per path), sd_start (per path) and b (B, G) at the gridpoints, and
"<r>/<l>/s<s>/" K, sd, sdd, status."""
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

import momentum_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
LIMITS = ("energy", "momentum")
NPATH, G = 8, 101
SEED0 = 8700
SHARE = 0.3
START = 1.3           # s'(0) = START sqrt(limit / b(0)): above what the limit admits at s = 0

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


def _init(name):
    global _robot
    _robot = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])


def _b(args):
    """The 50-digit (T, |p|^2) at (q, q'), each rounded to fp64."""
    import mpmath
    q, qs = args
    T, p = momentum_ref.mp_energy_momentum(_robot, q, qs)
    with mpmath.workdps(momentum_ref.DPS):
        return float(T), float(p[0] ** 2 + p[1] ** 2 + p[2] ** 2)


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    from toppra.constraint.linear_constraint import canlinear_colloc_to_interpolate
    codes = list(algo.ParameterizationReturnCode)

    class WholeRobotRow(constraint.LinearConstraint):
        def __init__(self, table, limit, dof, scheme):
            super(WholeRobotRow, self).__init__()
            self.table, self.limit, self.dof = table, limit, dof
            self.identical = True
            self.set_discretization_type(scheme)

        def compute_constraint_params(self, path, gridpoints):
            q, qs = path(gridpoints), path(gridpoints, 1)
            b = np.array([self.table[(x.tobytes(), y.tobytes())] for x, y in zip(q, qs)]).reshape(-1, 1)
            a, c = np.zeros_like(b), np.zeros_like(b)
            F, g = np.ones((1, 1)), np.full(1, self.limit)
            if self.discretization_type == constraint.DiscretizationType.Interpolation:
                return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
            return a, b, c, F, g, None, None

    def solve(path, vlim, alim, extra, scheme, sd_start):
        cons = [constraint.JointVelocityConstraint(vlim),
                constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)] + extra
        inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
        sdd, sd, _, K = inst.compute_parameterization(sd_start, 0, return_data=True)
        return sdd, sd, K, codes.index(inst.problem_data.return_code)

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid, "share": np.array(SHARE)}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits and the DOF count
        nv = model.nv
        probs = [problem(SEED0 + 100 * r + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs = path(grid), path(grid, 1)
            jobs += [(q[i], qs[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            vals = np.array(pool.map(_b, jobs, chunksize=8))
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs])})
        free = [solve(path, vlim, alim, [], 0, 0.0)[1] for path, (way, vlim, alim) in zip(paths, probs)]
        for j, lim_name in enumerate(LIMITS):
            table = {(q.tobytes(), qs.tobytes()): v[j] for (q, qs), v in zip(jobs, vals)}
            b = vals[:, j].reshape(NPATH, G)
            if lim_name == "energy":
                limits = np.array([SHARE * np.max(b[i] * sd ** 2) for i, sd in enumerate(free)])
                rows = limits
            else:
                limits = np.array([SHARE * np.max(np.sqrt(b[i]) * sd) for i, sd in enumerate(free)])
                rows = limits * limits
            # one path whose start speed the joint limits admit and the limit does not
            sd_start = np.zeros(NPATH)
            for i in range(NPATH):
                s0 = START * np.sqrt(rows[i] / b[i, 0])
                if b[i, 0] > 0 and solve(paths[i], probs[i][1], probs[i][2], [], 0, s0)[3] == 0:
                    sd_start[i] = s0
                    break
            assert sd_start.any(), (name, lim_name)
            data.update({"%s/%s/limit" % (name, lim_name): limits, "%s/%s/sd_start" % (name, lim_name): sd_start,
                         "%s/%s/b" % (name, lim_name): b})
            for scheme in (0, 1):
                out = {"K": [], "sd": [], "sdd": [], "status": []}
                for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
                    sdd, sd, K, st = solve(path, vlim, alim, [WholeRobotRow(table, rows[i], nv, scheme)], scheme,
                                           sd_start[i])
                    out["K"].append(K)
                    out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                    out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                    out["status"].append(st)
                for key, v in out.items():
                    data["%s/%s/s%d/%s" % (name, lim_name, scheme, key)] = np.stack(v)
                print(name, lim_name, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "kinetic_energy.npz"), **data)


if __name__ == "__main__":
    main()
