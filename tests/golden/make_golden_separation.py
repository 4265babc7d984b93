"""Generates tests/golden/separation_monitoring.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems with a speed and separation monitoring limit, for tests/test_separation_monitoring.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_separation.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 waypoints), G = 101, both discretisation schemes, solved by
TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is a reference
`LinearConstraint` subclass returning (a, b, c, F, g) = (0, b, c, [[1]], [0]) (lifted by the reference's own
`canlinear_colloc_to_interpolate` under Interpolation).  b and c come from the 50-digit reference of
tests/separation_ref.py (rnea_ref.MpRobot on the RAW URDF tree, kin_ref.mp_frames), rounded to fp64 and looked up by
the exact bytes of (q, q').

Two human spheres per path.  Paths 2..7: one sphere ahead of the tool along its motion, 0.45 to 0.8 m away, so the
limit binds on part of the path, and one 1.5 m away.  Path 0: a small sphere the tool passes at a distance inside the
clearance while moving away from it, and one 2 m behind the motion (the row stays inactive there).  Path 1: the same,
but the tool is still approaching at one gridpoint inside the clearance (x = 0 there).  The gridpoint and the side of
the pass are searched with the numpy double until those rows hold.  Stored per robot `r` under "<r>/...": the inputs
(way, vlim, alim, humans), the points (links, xyz, radii), b and c (B, G) at the gridpoints, the special gridpoints
(inside, (2,)), and "<r>/s<s>/" K, sd, sdd, status; the limit's parameters are shared."""
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
import separation_ref as sr  # noqa: E402

ROBOTS = {"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", {"finger_left_joint": 0.013,
                                                                         "finger_right_joint": 0.021})}
# robot points: (link, xyz, radius); the first is the tool
POINTS = {"arm6": [("flange", (0.0, 0.0, 0.1), 0.05), ("wrist2", (0.0, 0.0, 0.0), 0.06),
                   ("forearm", (0.0, 0.0, 0.0), 0.08)],
          "arm7": [("hand", (0.02, 0.0, 0.12), 0.05), ("link4", (0.0, 0.0, 0.0), 0.07)]}
PARAMS = (0.1, 2.5, 1.6, 0.05)          # reaction time, stopping deceleration, human speed, clearance
NPATH, G = 8, 101
SEED0 = 9100


def _urdf(name):
    return open(os.path.join(HERE, "robots", ROBOTS[name][0])).read()


def problem(seed, nv, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (5, nv)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    al = rng.uniform(6, 10, nv)
    return way, vlim, np.stack([-al, al], axis=1)


def packed_points(model, name):
    from toppra_b200.dynamics import pack_points
    return pack_points([(model.frame(link, xyz=xyz), r) for link, xyz, r in POINTS[name]])[1]


def _perp(u, rng):
    n = np.cross(u, rng.randn(3))
    return n / np.linalg.norm(n)


def pass_by(x, v, grid, g1, before, half, rng):
    """A sphere of radius 0.02 the tool (x, v at s' = 1) passes with its closest approach `before` grid spacings
    before gridpoint g1, the clearance zone reaching `half` grid spacings of arc either side of it."""
    R0 = POINTS_R0
    u = v[g1] / np.linalg.norm(v[g1])
    arc = np.linalg.norm(v[g1]) * (grid[1] - grid[0])
    xc = x[g1] - before * arc * u
    rho = np.sqrt(max(R0 * R0 - (half * arc) ** 2, 0.0))
    return np.concatenate((xc + rho * _perp(u, rng), [0.02]))


def humans_for(i, x, v, grid, rng, rows_at):
    """(2, 4) spheres of path i from the tool's positions x and velocities v (G, 3); rows_at(humans, g) -> (b, c,
    D of the tool's pairs) by the numpy double at gridpoint g."""
    if i >= 2:
        for _ in range(50):
            far = x[int(rng.randint(20, 80))] + 1.5 * _perp(np.array([0.0, 0.0, 1.0]), rng)
            g0 = int(rng.randint(35, 65))
            u = v[g0] / np.linalg.norm(v[g0])
            near = x[g0] + rng.uniform(0.3, 0.6) * u + rng.uniform(0.5, 0.7) * _perp(u, rng)
            hum = np.stack((np.concatenate((near, [0.12])), np.concatenate((far, [0.2]))))
            if all(rows_at(hum, g)[1] < 0 for g in range(len(grid))):    # no stop: vmax > 0 wherever a pair approaches
                return hum, -1
        raise RuntimeError("no sphere placement for path %d" % i)
    for g1 in range(30, 90):
        if np.linalg.norm(v[g1]) < 0.2:
            continue
        u = v[g1] / np.linalg.norm(v[g1])
        far = np.concatenate((x[g1] - 2.0 * u, [0.2]))      # behind the motion
        for _ in range(20):
            # path 0: closest approach 0.2 spacings before g1, zone +-0.35: only g1 inside, moving away;
            # path 1: closest approach 0.3 spacings after g1, zone +-0.55: g1 inside approaching, g1 + 1 moving away
            sph = pass_by(x, v, grid, g1, 0.2 if i == 0 else -0.3, 0.35 if i == 0 else 0.55, rng)
            hum = np.stack((sph, far))
            b, c, D = rows_at(hum, g1)
            if i == 0 and D[0] <= 0 and b == 0.0 and c == -1.0:
                return hum, g1
            if i == 1 and D[0] <= 0 and b > 0.0 and c == 0.0:
                return hum, g1
    raise RuntimeError("no gridpoint for path %d" % i)


POINTS_R0 = None


def main():
    global POINTS_R0
    from oracle.ref_loader import load_reference
    from toppra_b200.dynamics import RigidBodyModel
    import kin_ref
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    from toppra.constraint.linear_constraint import canlinear_colloc_to_interpolate
    codes = list(algo.ParameterizationReturnCode)

    class SeparationRow(constraint.LinearConstraint):
        def __init__(self, table, dof, scheme):
            super(SeparationRow, self).__init__()
            self.table, self.dof = table, dof
            self.identical = True
            self.set_discretization_type(scheme)

        def compute_constraint_params(self, path, gridpoints):
            q, qs = path(gridpoints), path(gridpoints, 1)
            bc = np.array([self.table[(x.tobytes(), y.tobytes())] for x, y in zip(q, qs)])
            b, c = bc[:, :1], bc[:, 1:]
            a = np.zeros_like(b)
            F, g = np.ones((1, 1)), np.zeros(1)
            if self.discretization_type == constraint.DiscretizationType.Interpolation:
                return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
            return a, b, c, F, g, None, None

    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    Tr, a_s, vh, C = PARAMS
    data = {"ss": ss, "grid": grid, "params": np.array(PARAMS)}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])
        mp = rnea_ref.MpRobot.from_urdf(_urdf(name), ROBOTS[name][1])
        nv = model.nv
        pts = packed_points(model, name)
        POINTS_R0 = POINTS[name][0][2] + 0.02 + C + vh * Tr
        rng = np.random.RandomState(SEED0 + r)
        probs = [problem(SEED0 + 100 * r + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        humans, inside, table, bs, cs = [], [], {}, [], []
        spec = {j: (link, np.eye(3), np.asarray(xyz, dtype=float)) for j, (link, xyz, _) in enumerate(POINTS[name])}
        for i, path in enumerate(paths):
            q, qs = path(grid), path(grid, 1)
            _, x, v = kin_ref.frame_packed(model.packed, pts[0, :14], q, qs)
            def rows_at(hum, g):
                d, _ = sr.separation_packed(model.packed, pts, hum, q[g], qs[g])
                b, c = sr.rows_packed(model.packed, pts, hum, PARAMS, q[g], qs[g])
                return b[0], c[0], d[0, 0] - C - vh * Tr

            hum, g1 = humans_for(i, x, v[:, :3], grid, rng, rows_at)
            humans.append(hum)
            inside.append(g1)
            brow, crow = [], []
            for k in range(G):
                st = sr.mp_points(mp, q[k], qs[k], spec)
                pairs = [sr.mp_pair(st[j][0], st[j][1], POINTS[name][j][2], hum[h])
                         for j in range(len(POINTS[name])) for h in range(hum.shape[0])]
                b, c = (float(z) for z in sr.mp_row(pairs, PARAMS))
                table[(q[k].tobytes(), qs[k].tobytes())] = (b, c)
                brow.append(b)
                crow.append(c)
            bs.append(brow)
            cs.append(crow)
        b, c = np.array(bs), np.array(cs)
        # the special gridpoints: path 0 inactive inside the clearance, path 1 approaching there (c == 0, b > 0)
        assert b[0, inside[0]] == 0.0 and c[0, inside[0]] == -1.0, (b[0, inside[0]], c[0, inside[0]])
        assert c[1, inside[1]] == 0.0 and b[1, inside[1]] > 0.0, (b[1, inside[1]], c[1, inside[1]])
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/humans" % name: np.stack(humans),
                     "%s/links" % name: np.array([p[0] for p in POINTS[name]]),
                     "%s/xyz" % name: np.array([p[1] for p in POINTS[name]]),
                     "%s/radii" % name: np.array([p[2] for p in POINTS[name]]),
                     "%s/b" % name: b, "%s/c" % name: c, "%s/inside" % name: np.array(inside[:2])})
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for path, (way, vlim, alim) in zip(paths, probs):
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        SeparationRow(table, nv, scheme)]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
            for key, val in out.items():
                data["%s/s%d/%s" % (name, scheme, key)] = np.stack(val)
            print(name, "scheme", scheme, "statuses", out["status"], "inside", inside[:2])
    np.savez_compressed(os.path.join(HERE, "separation_monitoring.npz"), **data)


if __name__ == "__main__":
    main()
