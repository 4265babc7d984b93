"""Per-path (ragged) grids against one common grid on the GPU: 4096 paths x 7 DOF, vel+acc.

The batch is solved twice for each method: on the grids the device proposes for each path (`gridpoints=None`, padded
to Gmax with `glen`), and on one common grid of Gmax points, the shape a caller without per-path grids would use.
Methods: BatchTOPPRAsd.compute_parameterization (two scans + the bisection), compute_feasible_sets,
compute_reachable_sets (both on the problem's stage records, built once before timing) and robust
compute_parameterization (RobustLinearConstraint on the acceleration rows).  Timed with CUDA events over `--iters` calls;
warm-up first, then `--reps` alternated rounds (every round times every method on both grids); medians are reported.
Prints one JSON line with the card's name and power limit.

    python scripts/ragged_bench.py [--reps 5] [--iters 5]"""
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    import toppra_b200 as ta
    from problems import make_batch_fast
    assert torch.cuda.is_available(), "ragged_bench needs a GPU"
    B = args.B
    ss, way, vlim, alim = make_batch_fast(B)
    path = ta.BatchSplineInterpolator(ss, way)

    def cons(robust=False):
        acc = ta.constraint.JointAccelerationConstraint(alim)
        if robust:
            acc = ta.constraint.RobustLinearConstraint(acc, [0.02, 0.01, 0.01], 1)
        return [ta.constraint.JointVelocityConstraint(vlim), acc]

    probe = ta.BatchTOPPRA(cons(), path)
    glen = probe.glen.cpu().numpy()
    Gmax = probe.G
    grids = {"ragged": None, "common": np.linspace(0, 1, Gmax)}
    desired = np.full(B, 3.0)
    methods = {}
    for kind, grid in grids.items():
        sd = ta.BatchTOPPRAsd(cons(), path, grid)
        sd.set_desired_duration(desired)
        sets = ta.BatchTOPPRA(cons(), path, grid, fused=False)
        sets.setup()
        rob = ta.BatchTOPPRA(cons(True), path, grid)
        rob.setup()
        methods[("toppra_sd", kind)] = lambda sd=sd: sd.compute_parameterization()
        methods[("feasible_sets", kind)] = lambda i=sets: i.compute_feasible_sets()
        methods[("reachable_sets", kind)] = lambda i=sets: i.compute_reachable_sets(0.0, 0.0)
        methods[("robust", kind)] = lambda i=rob: i.compute_parameterization()
    for fn in methods.values():          # warm-up of every shape in the timed window
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    times = {key: [] for key in methods}
    for _ in range(args.reps):
        for key, fn in methods.items():  # alternated: every round times every method on both grids
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                fn()
            t1.record()
            t1.synchronize()
            times[key].append(t0.elapsed_time(t1) / args.iters)
    name, power = card()
    ms = {"%s/%s" % key: float(np.median(v)) for key, v in times.items()}
    spread = {"%s/%s" % key: float((max(v) - min(v)) / np.median(v)) for key, v in times.items()}
    out = dict(workload="B=%d dof=7 vel+acc, proposed grids: glen %d..%d (mean %.1f), common grid Gmax=%d"
               % (B, glen.min(), glen.max(), glen.mean(), Gmax), gpu=name, power_limit=power, ms=ms, spread=spread,
               paths_per_s={k: B / (v * 1e-3) for k, v in ms.items()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
