"""Motor-side torque and speed limits of geared drives at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500
gridpoints with the 6-DOF robot of tests/golden/robots/arm6.urdf and a coupled wrist (T = diag(n) C).

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  drive_terms   tbd_drive_torque_terms alone on the B x G points (Drives.torque_terms);
  joint_terms   tbd_torque_terms alone on the same points (RigidBodyModel.torque_terms), for comparison;
  motor_solve   the whole BatchTOPPRA solve with vel + acc + MotorTorqueConstraint + MotorSpeedConstraint;
  joint_solve   the whole BatchTOPPRA solve with vel + acc + joint-side torque limits (SecondOrderConstraint).
Also prints the GPU name and power limit read in the same run and the solved path counts.  Prints one JSON line.

    python scripts/drive_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
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
from rnea_bench import gpu_info  # noqa: E402


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--grid", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    n = np.linspace(120.0, 50.0, nv)
    C = np.eye(nv)
    C[4, 3], C[5, 3], C[5, 4] = 1.0, 0.5, -1.0
    drives = ta.Drives(model, transmission=np.diag(n) @ C, rotor_inertia=np.linspace(4e-5, 1e-5, nv), friction=0.02)
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    tl = 0.45 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nv))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    motor_lim = taulim / n[:, None]
    omega = 0.7 * model.velocity_limit * n
    fric = 0.3 + 0.1 * np.arange(nv)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1, 2))

    def solve(cons):
        return lambda: ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0)

    joint = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]
    legs = {
        "drive_terms": lambda: drives.torque_terms(q, qs, qss),
        "joint_terms": lambda: model.torque_terms(q, qs, qss, fric),
        "motor_solve": solve(joint + [ta.MotorTorqueConstraint(drives, motor_lim),
                                      ta.MotorSpeedConstraint(drives, omega)]),
        "joint_solve": solve(joint + [ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim,
                                                                                                   fric)]),
    }
    times = {k: [] for k in legs}
    for fn in legs.values():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    ok = {k: int((legs[k]().to_host()["status"] == 0).sum()) for k in ("motor_solve", "joint_solve")}
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "points": B * G, "rounds": args.rounds,
           "ok_paths": ok}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
