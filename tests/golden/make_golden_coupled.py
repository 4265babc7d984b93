"""Generates tests/golden/coupled_joints.npz: the UNMODIFIED reference (oracle/_ref, built by oracle/build_ref.sh)
solving torque-limited problems of a robot with coupled joints, for tests/test_coupled_joints.py:

    bash oracle/build_ref.sh && python tests/golden/make_golden_coupled.py   # TOPPRA_REFERENCE: default /root/reference

Two models of tests/golden/robots/palletizer.urdf with its mimic joints coupled ("free": 6 DOFs, the wrist pitch
free; "level": 5 DOFs, the wrist pitch held at -(shoulder + elbow) by a levelling link, coupled_ref.level_rows).
Each: 6 spline paths (5 waypoints), G = 51, both discretisation schemes, solved by TOPPRA([JointVelocityConstraint,
JointAccelerationConstraint, JointTorqueConstraint(inv_dyn, tau_lim, fs)], path, grid, "seidel").  inv_dyn is the
50-digit reduced Lagrangian of tests/coupled_ref.py (MpCoupled on the RAW URDF tree, mimic joints as DOFs), rounded
to fp64; it is computed beforehand in a process pool at every (q, 0, 0), (q, 0, q') and (q, q', q'') the reference
asks for and looked up by the exact bytes of its arguments.

Per path, tau_lim is symmetric: SHARE of the largest |tau_j| on the reference's solution without it, and at least
1.2 times the largest gravity torque |c_j|, so that the limit binds and the path stays feasible; the last path gets
0.8 times the largest gravity torque on the shoulder, which makes it infeasible.  Stored per model `m`: "<m>/" way,
vlim, alim, taulim (per path), fs, and "<m>/s<s>/" K, sd, sdd, status."""
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

import coupled_ref  # noqa: E402
import rnea_ref  # noqa: E402

NPATH, G = 6, 51
SEED0 = 9300
SHARE = 0.7
MODELS = ("free", "level")

_mp = None


def _urdf():
    return open(os.path.join(HERE, "robots", "palletizer.urdf")).read()


def model_of(which):
    from toppra_b200.dynamics import RigidBodyModel
    m = RigidBodyModel.from_urdf(_urdf(), couple_mimic=True)
    return m if which == "free" else m.with_coupling(coupled_ref.level_rows(m))


def problem(seed, nq, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.5, 0.5, (5, nq)), axis=0)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.stack([-vel, vel], axis=1)
    al = rng.uniform(4, 8, nq)
    return way, vlim, np.stack([-al, al], axis=1)


def _init(which):
    global _mp
    m = model_of(which)
    _mp = coupled_ref.MpCoupled(rnea_ref.MpRobot.from_urdf(_urdf()), *m.coupling)


def _terms(args):
    q, qs, qss = args
    return _mp.tau_terms(q, qs, qss)


def main():
    import mpmath
    from oracle.ref_loader import load_reference
    ta = load_reference()
    import toppra.algorithm as algo
    import toppra.constraint as constraint
    codes = list(algo.ParameterizationReturnCode)
    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)

    def solve(path, vlim, alim, extra, scheme):
        cons = [constraint.JointVelocityConstraint(vlim),
                constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)] + extra
        inst = algo.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
        sdd, sd, _, K = inst.compute_parameterization(0, 0, return_data=True)
        return sdd, sd, K, codes.index(inst.problem_data.return_code)

    data = {"ss": ss, "grid": grid, "share": np.array(SHARE), "level_rows": coupled_ref.level_rows(model_of("free"))}
    for r, which in enumerate(MODELS):
        model = model_of(which)
        nq = model.nq
        probs = [problem(SEED0 + 100 * r + p, nq, model.velocity_limit) for p in range(NPATH)]
        paths = [ta.SplineInterpolator(ss, pr[0]) for pr in probs]
        jobs = []
        for path in paths:
            q, qs, qss = path(grid), path(grid, 1), path(grid, 2)
            jobs += [(q[i], qs[i], qss[i]) for i in range(G)]
        with multiprocessing.Pool(initializer=_init, initargs=(which,)) as pool:
            vals = pool.map(_terms, jobs, chunksize=4)
        table, zero = {}, np.zeros(nq)
        with mpmath.workdps(coupled_ref.DPS):
            for (q, qs, qss), (c, ta_, tb) in zip(jobs, vals):
                f64 = lambda v: np.array([float(x) for x in v])  # noqa: E731
                table[(q.tobytes(), zero.tobytes(), zero.tobytes())] = f64(c)
                table[(q.tobytes(), zero.tobytes(), qs.tobytes())] = f64(ta_)
                table[(q.tobytes(), qs.tobytes(), qss.tobytes())] = f64(tb)

        def inv_dyn(q, qd, qdd):
            return table[(np.asarray(q, dtype=np.float64).tobytes(), np.asarray(qd, dtype=np.float64).tobytes(),
                          np.asarray(qdd, dtype=np.float64).tobytes())]

        fs = np.full(nq, 2.0)
        taulim = []
        for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
            sdd, sd, _, _ = solve(path, vlim, alim, [], 0)
            q, qs, qss = path(grid), path(grid, 1), path(grid, 2)
            c = np.stack([inv_dyn(x, zero, zero) for x in q])
            tau = np.stack([inv_dyn(q[k], zero, zero) + (inv_dyn(q[k], zero, qs[k]) - c[k]) * (sdd[min(k, G - 2)])
                            + (inv_dyn(q[k], qs[k], qss[k]) - c[k]) * sd[k] ** 2 for k in range(G)])
            lim = np.maximum(SHARE * np.abs(tau).max(axis=0), 1.2 * np.abs(c).max(axis=0)) + fs
            if i == NPATH - 1:
                lim[model.joint_names.index("shoulder")] = 0.8 * np.abs(c[:, model.joint_names.index("shoulder")]).max()
            taulim.append(np.stack([-lim, lim], axis=1))
        data.update({"%s/way" % which: np.stack([p[0] for p in probs]), "%s/vlim" % which: np.stack([p[1] for p in probs]),
                     "%s/alim" % which: np.stack([p[2] for p in probs]), "%s/taulim" % which: np.stack(taulim),
                     "%s/fs" % which: fs})
        for scheme in (0, 1):
            out = {"K": [], "sd": [], "sdd": [], "status": []}
            for i, (path, (way, vlim, alim)) in enumerate(zip(paths, probs)):
                jt = constraint.JointTorqueConstraint(inv_dyn, taulim[i], fs, discretization_scheme=scheme)
                sdd, sd, K, st = solve(path, vlim, alim, [jt], scheme)
                out["K"].append(K)
                out["sd"].append(np.full(G, np.nan) if sd is None else sd)
                out["sdd"].append(np.full(G - 1, np.nan) if sdd is None else sdd)
                out["status"].append(st)
            for key, v in out.items():
                data["%s/s%d/%s" % (which, scheme, key)] = np.stack(v)
            print(which, "scheme", scheme, "statuses", out["status"])
    np.savez_compressed(os.path.join(HERE, "coupled_joints.npz"), **data)


if __name__ == "__main__":
    main()
