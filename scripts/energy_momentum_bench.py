"""Kinetic-energy limits of the whole robot at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints with
the 6-DOF robot of tests/golden/robots/arm6.urdf and one energy limit per path.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  energy_terms    tbd_energy_momentum_terms alone on the B x G points, b = T(q, q') (RigidBodyModel.energy_momentum_terms);
  velocity_terms  tbd_velocity_norm_terms alone on the same points, the tool speed 10 cm past the flange, for comparison;
  torque_terms    tbd_torque_terms alone on the same points (RigidBodyModel.torque_terms), for comparison;
  energy_solve    the whole BatchTOPPRA solve with vel + acc + joint torque limits + KineticEnergyConstraint;
  base_solve      the whole BatchTOPPRA solve with vel + acc + joint torque limits.
Each path's energy limit is half the largest T on its solution without it, so that it binds.  Also prints the GPU name
and power limit read in the same run and the solved path counts.  Prints one JSON line.

    python scripts/energy_momentum_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import toppra_b200 as ta  # noqa: E402
from drive_bench import timed  # noqa: E402
from rnea_bench import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--grid", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    tcp = model.frame("flange", xyz=(0.0, 0.0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    tl = 0.45 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nv))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    fric = 0.3 + 0.1 * np.arange(nv)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1, 2))

    def solve(cons):
        return lambda: ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0)

    base = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
            ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
    sd = solve(base)().sd
    b = model.energy_momentum_terms(q, qs, "energy").reshape(B, G)
    limit = 0.5 * torch.nan_to_num(b * sd * sd).max(dim=1).values.cpu().numpy()
    del sd, b
    energy = ta.constraint.KineticEnergyConstraint(model, limit)
    legs = {
        "energy_terms": lambda: model.energy_momentum_terms(q, qs, "energy"),
        "velocity_terms": lambda: tcp.velocity_norm_terms(q, qs, S),
        "torque_terms": lambda: model.torque_terms(q, qs, qss, fric),
        "energy_solve": solve(base + [energy]),
        "base_solve": solve(base),
    }
    times = {k: [] for k in legs}
    for fn in legs.values():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    ok = {k: int((legs[k]().to_host()["status"] == 0).sum()) for k in ("energy_solve", "base_solve")}
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "points": B * G, "rounds": args.rounds,
           "energy_limit_J": {"median": float(np.median(limit)), "min": float(limit.min()), "max": float(limit.max())},
           "ok_paths": ok}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
