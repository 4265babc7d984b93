"""Generates tests/golden/capsule_separation.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving problems with a speed and separation monitoring limit on robot and human capsules, for
tests/test_capsule_separation.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_capsules.py   # TOPPRA_REFERENCE: default /root/reference

Each robot: 8 spline paths (5 waypoints, the problems of make_golden_separation.py), G = 101, both discretisation
schemes, solved by TOPPRA([JointVelocityConstraint, JointAccelerationConstraint, C], path, grid, "seidel") where C is a
reference `LinearConstraint` subclass returning (a, b, c, F, g) = (0, b, c, [[1]], [0]) (lifted by the reference's own
`canlinear_colloc_to_interpolate` under Interpolation).  b and c come from the float64 numpy double of
tests/capsule_ref.py, looked up by the exact bytes of (q, q').

The robot: one capsule per link.  The person, per path: a vertical torso capsule (0.5 m, radius 0.12) ahead of the tool
along its motion at a random mid-path gridpoint, 0.55 to 0.8 m to its side, and a forearm capsule (0.3 m, radius 0.05)
reaching from the torso toward the tool's path; placements where an approaching pair would bound s'^2 below X_MIN (a
near-stop, where the solution is ill-conditioned in the rows) are drawn again.  Stored per robot `r` under "<r>/...":
the inputs (way, vlim, alim, humans), the capsules (link_a, xyz_a, link_b, xyz_b, radii), b and c (B, G), and
"<r>/s<s>/" K, sd, sdd, status; the limit's parameters are shared."""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

import capsule_ref as cr  # noqa: E402
from make_golden_separation import ROBOTS, _perp, _urdf, problem  # noqa: E402

# robot capsules: (link_a, xyz_a, link_b, xyz_b, radius)
CAPSULES = {"arm6": [("shoulder", (0, 0, 0), "upper_arm", (0, 0, 0), 0.08),
                     ("upper_arm", (0, 0, 0), "forearm", (0, 0, 0), 0.07),
                     ("forearm", (0, 0, 0), "wrist1", (0, 0, 0), 0.06),
                     ("wrist1", (0, 0, 0), "wrist2", (0, 0, 0), 0.05),
                     ("wrist2", (0, 0, 0), "wrist3", (0, 0, 0), 0.05),
                     ("wrist3", (0, 0, 0), "flange", (0.0, 0.0, 0.1), 0.05)],
            "arm7": [("torso", (0, 0, 0), "link2", (0, 0, 0), 0.08),
                     ("link2", (0, 0, 0), "link3", (0, 0, 0), 0.07),
                     ("link3", (0, 0, 0), "link4", (0, 0, 0), 0.07),
                     ("link4", (0, 0, 0), "link5", (0, 0, 0), 0.06),
                     ("link5", (0, 0, 0), "link6", (0, 0, 0), 0.06),
                     ("link6", (0, 0, 0), "hand", (0.02, 0.0, 0.12), 0.05)]}
PARAMS = (0.1, 2.5, 1.6, 0.05)          # reaction time, stopping deceleration, human speed, clearance
NPATH, G = 8, 101
X_MIN = 1e-2                            # the smallest bound s'^2 <= -c / b the limit may impose on a path
SEED0 = 9200


def packed_capsules(model, name):
    from toppra_b200.dynamics import pack_points
    return pack_points([(model.frame(a, xyz=xa), model.frame(b, xyz=xb), r)
                        for a, xa, b, xb, r in CAPSULES[name]])[1]


def person(x, v, rng):
    """(2, 7): torso and forearm capsules ahead of the tool (x, v: positions and velocities at s' = 1, (G, 3))."""
    g0 = int(rng.randint(35, 65))
    u = v[g0] / np.linalg.norm(v[g0])
    n = _perp(u, rng)
    base = x[g0] + rng.uniform(0.3, 0.5) * u + rng.uniform(0.55, 0.8) * n
    torso = np.r_[base - [0, 0, 0.25], base + [0, 0, 0.25], 0.12]
    arm = np.r_[base + [0, 0, 0.15], base + [0, 0, 0.15] - 0.3 * n, 0.05]
    return np.stack((torso, arm))


def main():
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
    data = {"ss": ss, "grid": grid, "params": np.array(PARAMS)}
    for r, name in enumerate(ROBOTS):
        model = RigidBodyModel.from_urdf(_urdf(name), ROBOTS[name][1])
        nv = model.nv
        caps = packed_capsules(model, name)
        tool = caps[-1, 14:28]
        rng = np.random.RandomState(SEED0 + r)
        probs = [problem(SEED0 + 100 * r + p, nv, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        humans, table, bs, cs = [], {}, [], []
        for path in paths:
            q, qs = path(grid), path(grid, 1)
            _, x, v = kin_ref.frame_packed(model.packed, tool, q, qs)
            for _ in range(50):
                hum = person(x, v[:, :3], rng)
                b, c = cr.capsule_rows_packed(model.packed, caps, hum, PARAMS, q, qs)
                with np.errstate(divide="ignore"):
                    if ((b == 0) | (-c / b >= X_MIN)).all():   # no approaching pair near a stop
                        break
            else:
                raise RuntimeError("no person placement")
            humans.append(hum)
            for k in range(G):
                table[(q[k].tobytes(), qs[k].tobytes())] = (b[k], c[k])
            bs.append(b)
            cs.append(c)
        cs_ = CAPSULES[name]
        data.update({"%s/way" % name: np.stack([p[0] for p in probs]), "%s/vlim" % name: np.stack([p[1] for p in probs]),
                     "%s/alim" % name: np.stack([p[2] for p in probs]), "%s/humans" % name: np.stack(humans),
                     "%s/link_a" % name: np.array([c[0] for c in cs_]), "%s/xyz_a" % name: np.array([c[1] for c in cs_],
                                                                                                   dtype=float),
                     "%s/link_b" % name: np.array([c[2] for c in cs_]), "%s/xyz_b" % name: np.array([c[3] for c in cs_],
                                                                                                   dtype=float),
                     "%s/radii" % name: np.array([c[4] for c in cs_]),
                     "%s/b" % name: np.array(bs), "%s/c" % name: np.array(cs)})
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            n_active = 0
            for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
                cons = [constraint.JointVelocityConstraint(vlim),
                        constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                        SeparationRow(table, nv, scheme)]
                inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(codes.index(inst.problem_data.return_code))
                if sd is not None:
                    b, c = bs[i], cs[i]
                    n_active += bool(((b > 0) & (b * sd ** 2 >= -c * (1 - 1e-6))).any())
            for key, val in out.items():
                data["%s/s%d/%s" % (name, scheme, key)] = np.stack(val)
            print(name, "scheme", scheme, "statuses", out["status"], "limit active on", n_active)
    np.savez_compressed(os.path.join(HERE, "capsule_separation.npz"), **data)


if __name__ == "__main__":
    main()
