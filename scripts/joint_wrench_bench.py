"""Bearing limits on the wrench across a joint at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints
with the 6-DOF robot of tests/golden/robots/arm6.urdf, the bearing of joint 2 (shoulder_lift, frame upper_arm, "local").

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  wrench_terms   tbd_joint_wrench_terms alone on the B x G points, all six components (RigidBodyFrame.joint_wrench_terms);
  torque_terms   tbd_torque_terms alone on the same points (RigidBodyModel.torque_terms), for comparison;
  wrench_solve   the whole BatchTOPPRA solve with vel + acc + joint torque limits + JointWrenchConstraint.bearing
                 (axial, radial and tilting limits, 8 sides: 18 rows, 36 under Interpolation);
  torque_solve   the whole BatchTOPPRA solve with vel + acc + joint torque limits.
The bearing limits are 1.5 times the 90th percentile of the static loads over the batch (the axial one at least half the
radial one), so they bind in the fast parts of the paths.  Also prints the GPU name and power limit read in the same
run and the solved path counts.  Prints one JSON line.

    python scripts/joint_wrench_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
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
    frame = model.frame("upper_arm", reference_frame="local")
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

    # bearing limits from the static loads w(q, 0, 0) of the batch
    c = frame.joint_wrench_terms(q, qs, qss)[2]
    axis = torch.as_tensor(frame.R.T @ model.body(frame.body)[2:5], device="cuda")
    fa = c[:, :3] @ axis
    fr = torch.linalg.norm(c[:, :3] - fa[:, None] * axis, dim=1)
    nt = torch.linalg.norm(c[:, 3:] - (c[:, 3:] @ axis)[:, None] * axis, dim=1)
    axial, radial, tilting = (1.5 * float(torch.quantile(x[::97], 0.9)) for x in (fa.abs(), fr, nt))
    axial = max(axial, 0.5 * radial)   # joint 2's axis stays horizontal: at rest it carries almost no axial force
    del c, fa, fr, nt

    def solve(cons):
        return lambda: ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0)

    base = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
            ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
    bearing = ta.constraint.JointWrenchConstraint.bearing(frame, axial=axial, radial=radial, tilting=tilting)
    legs = {
        "wrench_terms": lambda: frame.joint_wrench_terms(q, qs, qss),
        "torque_terms": lambda: model.torque_terms(q, qs, qss, fric),
        "wrench_solve": solve(base + [bearing]),
        "torque_solve": solve(base),
    }
    times = {k: [] for k in legs}
    for fn in legs.values():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    ok = {k: int((legs[k]().to_host()["status"] == 0).sum()) for k in ("wrench_solve", "torque_solve")}
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "points": B * G, "rounds": args.rounds,
           "bearing_limits": {"axial": axial, "radial": radial, "tilting": tilting}, "ok_paths": ok}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
