"""Robust (conic) problems with two robust constraints on the GPU: 4096 paths x 7 DOF x 200 gridpoints with
JointVelocity, RobustLinearConstraint(JointAcceleration, [1e-3, 5e-2, 9e-3], interpolation) and
RobustLinearConstraint(JointTorqueConstraint(arm7), [2e-3, 1e-1, 0.5]) on tests/golden/robots/arm7_gripper.urdf with the
fingers locked (7 moving joints).

Times, with CUDA events, compute_parameterization, BatchTOPPRAsd.compute_parameterization and
compute_reachable_sets(0, 0) of that problem (libtoppra_b200_cones.so), and the cost of the per-row form on plain
config 4: tbc_scan against tb_scan_robust on the same config-4 records with the table of its one ellipsoid.  The stage
records are built once and reused.  Warm-up first, then `--reps` alternated rounds; medians are reported.  Prints one
JSON line with the card's name and power limit.

    python scripts/robust_cones_bench.py [--reps 7] [--iters 5]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

ELL_ACC = [1e-3, 5e-2, 9e-3]
ELL_TAU = [2e-3, 1e-1, 0.5]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--G", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    import toppra_b200 as ta
    from toppra_b200 import engine
    from problems import make_batch_fast
    from robust_sd_bench import card
    assert torch.cuda.is_available(), "robust_cones_bench needs a GPU"
    B, G = args.B, args.G
    ss, way, vlim, alim = make_batch_fast(B, seed=3000)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    model = ta.dynamics.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm7_gripper.urdf"),
                                                 locked_joints={"finger_left_joint": 0.0, "finger_right_joint": 0.0})
    acc = ta.constraint.RobustLinearConstraint(ta.constraint.JointAccelerationConstraint(alim), ELL_ACC, 1)
    cons = [ta.constraint.JointVelocityConstraint(vlim), acc,
            ta.constraint.RobustLinearConstraint(ta.constraint.JointTorqueConstraint(model, _tau_lim(model),
                                                                                  np.zeros(7)), ELL_TAU, 1)]
    inst = ta.BatchTOPPRA(cons, path, grid)
    inst.setup()
    sd = ta.BatchTOPPRAsd(cons, path, grid)
    sd.set_desired_duration(3.0)
    sd.setup()
    cfg4 = ta.BatchTOPPRA(cons[:2], path, grid)
    cfg4.setup()
    rec, R, conic, d_grid = cfg4.records, cfg4.R, cfg4.conic, cfg4.d_grid
    table = np.zeros((R, 4))
    table[conic[0]:conic[0] + conic[1]] = [1.0] + ELL_ACC
    stages = {
        "parameterization": lambda: inst.compute_parameterization(),
        "toppra_sd": lambda: sd.compute_parameterization(),
        "reachable_sets": lambda: inst.compute_reachable_sets(0.0, 0.0),
        "cfg4_tbc_scan": lambda: engine.scan_cones(rec, R, table, d_grid),
        "cfg4_tb_scan_robust": lambda: engine.scan_robust(rec, R, *conic, d_grid),
    }
    for fn in stages.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in stages}
    for _ in range(args.reps):
        for name, fn in stages.items():   # alternated: every round times every stage once
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                fn()
            t1.record()
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) / args.iters)
    med = {n: float(np.median(v)) for n, v in times.items()}
    spread = {n: float((max(v) - min(v)) / np.median(v)) for n, v in times.items()}
    st = inst.compute_parameterization().status
    a = engine.scan_cones(rec, R, table, d_grid)
    o = engine.scan_robust(rec, R, *conic, d_grid)
    same = all(torch.equal(a[k], o[k]) for k in ("K", "status"))
    name, power = card()
    out = dict(workload="B=%d dof=7 G=%d, JointVelocity + robust JointAcceleration %s + robust JointTorque(arm7) %s, "
                        "records reused" % (B, G, ELL_ACC, ELL_TAU),
               gpu=name, power_limit=power, ms=med, spread=spread, ok=int((st == 0).sum()), cfg4_tbc_equals_tbr=same)
    print(json.dumps(out))


def _tau_lim(model):
    """The model's torque limits, with 30 N m on the joints whose URDF gives none (a robust row needs finite limits)."""
    return np.nan_to_num(model.torque_limits(), posinf=30.0, neginf=-30.0)


if __name__ == "__main__":
    main()
