"""Robust (conic) TOPPRAsd cost on the GPU: 4096 paths x 7 DOF x 200 gridpoints with the config-4 constraints
(JointVelocity + RobustLinearConstraint(JointAcceleration, ellipsoid [1e-3, 5e-2, 9e-3], interpolation)).

Times, with CUDA events, a robust BatchTOPPRAsd.compute_parameterization (desired duration between each path's fastest
and slowest) and a robust BatchTOPPRA.compute_parameterization on the same batch, plus the three launches of the former
alone: the backward-only conic scan, tbr_sd_forward_robust (both forward passes) and tb_sd_bisect.  The stage records
are built once and reused by every call.  Warm-up first, then `--reps` alternated rounds; medians are reported.  Prints
one JSON line with the card's name and power limit.

    python scripts/robust_sd_bench.py [--reps 7] [--iters 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [t.strip() for t in out.split(",")]
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        import torch
        return torch.cuda.get_device_name(), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--G", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    import torch
    import toppra_b200 as ta
    from toppra_b200 import engine
    from problems import make_batch_fast
    assert torch.cuda.is_available(), "robust_sd_bench needs a GPU"
    B, G = args.B, args.G
    ss, way, vlim, alim = make_batch_fast(B, seed=3000)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    cons = [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.RobustLinearConstraint(ta.constraint.JointAccelerationConstraint(alim), [1e-3, 5e-2, 9e-3], 1)]
    sd = ta.BatchTOPPRAsd(cons, path, grid)
    sd.set_desired_duration(0.0)
    r = sd.compute_parameterization()
    fast, slow = r.duration_fast.cpu().numpy(), r.duration_slow.cpu().numpy()
    sd.set_desired_duration(fast + 0.5 * (slow - fast))
    par = ta.BatchTOPPRA(cons, path, grid)
    par.setup()
    rec, R, conic, d_grid = sd.records, sd.R, sd.conic, sd.d_grid
    back = engine.scan_robust(rec, R, *conic, d_grid, backward_only=True)
    fwd = engine.sd_forward_robust(rec, R, *conic, d_grid, back["K"], back["status"])
    want = engine.as_device(np.ascontiguousarray(fast + 0.5 * (slow - fast)), path.device)
    stages = {
        "robust_toppra_sd": lambda: sd.compute_parameterization(),
        "robust_toppra": lambda: par.compute_parameterization(),
        "backward_scan": lambda: engine.scan_robust(rec, R, *conic, d_grid, backward_only=True),
        "sd_forward_robust": lambda: engine.sd_forward_robust(rec, R, *conic, d_grid, back["K"], back["status"]),
        "sd_bisect": lambda: engine.sd_bisect(fwd["x_fast"], fwd["u_fast"], fwd["x_slow"], fwd["u_slow"], d_grid, want,
                                              status_in=fwd["status"]),
    }
    for fn in stages.values():   # warm-up of every shape in the timed window
        for _ in range(3):
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
    res = sd.compute_parameterization()
    name, power = card()
    out = dict(workload="B=%d dof=7 G=%d, JointVelocity + RobustLinearConstraint(JointAcceleration, "
                        "[1e-3, 5e-2, 9e-3], interpolation), records reused" % (B, G),
               gpu=name, power_limit=power, ms=med, spread=spread,
               status_ok=int((res.status == 0).sum()), paths_per_s={n: B / (med[n] * 1e-3) for n in
                                                                    ("robust_toppra_sd", "robust_toppra")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
