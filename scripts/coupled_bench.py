"""Torque limits of a robot with coupled joints at the config-3 batch shape: 65 536 paths x 500 gridpoints on the
palletizer of tests/golden/robots/palletizer.urdf (9 bodies: two parallelogram bars and the right finger coupled as
mimic joints, the wrist pitch held by a levelling link at -(shoulder + elbow); 5 path DOFs).

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  coupled_terms   tbd_coupled_torque_terms alone on the B x G points (RigidBodyModel.torque_terms with friction);
  expand_reduce   the same numbers by tbd_coupling_expand, tbd_torque_terms on the 9 bodies and the reduction E^T and
                  the friction term as torch operations (bit-identical, checked once);
  tree_terms      tbd_torque_terms alone on the expanded points: the uncoupled tree's cost;
  torque_solve    the whole BatchTOPPRA solve with joint velocity, acceleration and coupled torque limits (per path);
  base_solve      the same solve without the torque limit.
Also prints the GPU name and power limit read in the same run, and the solved path counts.  Prints one JSON line.

    python scripts/coupled_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import toppra_b200 as ta  # noqa: E402
from toppra_b200 import dynamics  # noqa: E402
from drive_bench import timed  # noqa: E402
from rnea_bench import gpu_info  # noqa: E402
from coupled_ref import level_rows  # noqa: E402


def reduce_(E, t):
    """E^T t in the library's order (nonzero terms, ascending body), as torch operations."""
    cols = []
    for j in range(E.shape[1]):
        s = None
        for k in range(E.shape[0]):
            if E[k, j] != 0:
                u = float(E[k, j]) * t[:, k]
                s = u if s is None else s + u
        cols.append(s)
    return torch.stack(cols, dim=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--grid", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G = args.paths, args.grid
    urdf = os.path.join(ROOT, "tests", "golden", "robots", "palletizer.urdf")
    free = ta.RigidBodyModel.from_urdf(urdf, couple_mimic=True)
    model = free.with_coupling(level_rows(free))
    nv, nq = model.nv, model.nq
    b = model.packed[3:].reshape(nv, 27)
    tree = ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                             gravity=model.gravity)
    E = model.coupling[0]
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.5, 0.5, (B, 5, nq)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(4, 8, (B, nq))
    tl = 0.5 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nq))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    fric = np.full(nq, 2.0)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nq).contiguous() for o in (0, 1, 2))
    dfric = torch.as_tensor(fric, device="cuda")
    lib = ta._lib_dyn.load()
    qb, qsb, qssb = dynamics._expand(torch, lib, model, [q, qs, qss])

    def expand_reduce():
        xb = dynamics._expand(torch, lib, model, [q, qs, qss])
        a, bb, c = tree.torque_terms(*xb)
        return reduce_(E, a), reduce_(E, bb), reduce_(E, c) + torch.sign(qs) * dfric

    got, want = model.torque_terms(q, qs, qss, fric), expand_reduce()
    identical = all(bool(torch.equal(x, y)) for x, y in zip(got, want))
    del got, want

    def solve(cons):
        return lambda: ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0)

    base = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]
    torque = ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)
    legs = {
        "coupled_terms": lambda: model.torque_terms(q, qs, qss, fric),
        "expand_reduce": expand_reduce,
        "tree_terms": lambda: tree.torque_terms(qb, qsb, qssb),
        "torque_solve": solve(base + [torque]),
        "base_solve": solve(base),
    }
    times = {k: [] for k in legs}
    for fn in legs.values():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    ok = {k: int((legs[k]().to_host()["status"] == 0).sum()) for k in ("torque_solve", "base_solve")}
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "bodies": nv, "dofs": nq, "points": B * G, "rounds": args.rounds,
           "fused_bit_identical": identical, "ok_paths": ok}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
