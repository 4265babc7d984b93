"""Generates tests/golden/collision_energy.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems with a collision-energy limit on a robot frame, for tests/test_collision_energy.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_collision_energy.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is a reference
`LinearConstraint` subclass returning (a, b, c, F, g) = (0, b, 0, [[1]], [limit]) (lifted by the reference's own
`canlinear_colloc_to_interpolate` under Interpolation).  b = 1/2 |v|^4 / (|v|^2 / m_H + v^T Lambda_v^-1 v) comes from
the 50-digit reference of tests/energy_ref.py (rnea_ref.MpRobot on the RAW URDF tree: its mass matrix, J_v by
mpmath.diff, mpmath.lu_solve), rounded to fp64; the values are computed beforehand in a process pool and looked up by
the exact bytes of (q, q').

The limit of each path is 0.3 of the largest b sd^2 of the reference's solution without it (Collocation), so that it is
active.  Stored per robot `r` under "<r>/...": the inputs (way, vlim, alim, limit), the frame (link, xyz, rpy), the
human mass, b (B, G) at the gridpoints, and "<r>/s<s>/" K, sd, sdd, status."""
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

import energy_ref  # noqa: E402
import rnea_ref  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
# the contact point: 10 cm past the flange; 12 cm past the hand, turned; human body regions of 0.6 kg (hand) and 40 kg
FRAMES = {"arm6": ("flange", (0.0, 0.0, 0.1), (0.0, 0.0, 0.0)),
          "arm7": ("hand", (0.02, 0.0, 0.12), (0.2, 0.0, 0.3))}
HUMAN_MASS = {"arm6": 0.6, "arm7": 40.0}
NPATH, G = 8, 101
SEED0 = 8100
SHARE = 0.3

_robot = None
_name = None


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
    global _robot, _name
    _robot = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])
    _name = name


def _b(args):
    """The 50-digit b at (q, q'), rounded to fp64."""
    from toppra_b200.dynamics import rpy_matrix
    q, qs = args
    link, xyz, rpy = FRAMES[_name]
    ref = energy_ref.mp_inverse_inertia(_robot, q, {0: (link, rpy_matrix(rpy), np.asarray(xyz))})
    return float(energy_ref.mp_energy_b(ref[(0, "J")], ref[0][0], qs, HUMAN_MASS[_name]))


def main():
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    from toppra.constraint.linear_constraint import canlinear_colloc_to_interpolate
    codes = list(algo.ParameterizationReturnCode)

    class EnergyRow(constraint.LinearConstraint):
        def __init__(self, table, limit, dof, scheme):
            super(EnergyRow, self).__init__()
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

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    data = {"ss": ss, "grid": grid, "share": np.array(SHARE)}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])   # URDF limits and the DOF count
        nv = model.nv
        link, xyz, rpy = FRAMES[name]
        probs = [problem(SEED0 + 100 * r + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs = path(grid), path(grid, 1)
            jobs += [(q[i], qs[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(name,)) as pool:
            vals = pool.map(_b, jobs, chunksize=8)
        table = {(q.tobytes(), qs.tobytes()): v for (q, qs), v in zip(jobs, vals)}
        b = np.array(vals).reshape(NPATH, G)
        limits = []
        for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
            inst = algo.TOPPRA([constraint.JointVelocityConstraint(vlim), constraint.JointAccelerationConstraint(alim)],
                               path, gridpoints=grid, solver_wrapper="seidel")
            sd = inst.compute_parameterization(0, 0, return_data=True)[1]
            limits.append(SHARE * float(np.max(b[i] * sd ** 2)))
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/limit" % name: np.array(limits),
                     "%s/b" % name: b, "%s/human_mass" % name: np.array(HUMAN_MASS[name]),
                     "%s/link" % name: np.array(link), "%s/xyz" % name: np.array(xyz), "%s/rpy" % name: np.array(rpy)})
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim), limit in zip(paths, probs, limits):
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        EnergyRow(table, limit, nv, scheme)]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
            for key, v in out.items():
                data["%s/s%d/%s" % (name, scheme, key)] = np.stack(v)
            print(name, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "collision_energy.npz"), **data)


if __name__ == "__main__":
    main()
