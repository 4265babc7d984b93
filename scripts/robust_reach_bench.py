"""Robust (conic) reachable and controllable sets on the GPU: 4096 paths x 7 DOF x 200 gridpoints with the config-4
constraints (JointVelocity + RobustLinearConstraint(JointAcceleration, ellipsoid [1e-3, 5e-2, 9e-3], interpolation)).

Times, with CUDA events, a robust BatchTOPPRA.compute_reachable_sets(0, 0) and its two launches alone (the feasible-set
launch, tb_scan_robust with TB_SCAN_FEASIBLE_SETS, and the forward launch tbr_reachable_sets_robust), a robust
compute_controllable_sets(0, sdmax) (one tb_scan_robust_ex launch) and, for scale, a robust compute_parameterization.
The stage records are built once and reused by every call.  Warm-up first, then `--reps` alternated rounds; medians are
reported.  Prints one JSON line with the card's name and power limit.

    python scripts/robust_reach_bench.py [--reps 7] [--iters 10]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--G", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--sdmax", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    import toppra_b200 as ta
    from toppra_b200 import engine
    from problems import make_batch_fast
    from robust_sd_bench import card
    assert torch.cuda.is_available(), "robust_reach_bench needs a GPU"
    B, G = args.B, args.G
    ss, way, vlim, alim = make_batch_fast(B, seed=3000)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    cons = [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.RobustLinearConstraint(ta.constraint.JointAccelerationConstraint(alim), [1e-3, 5e-2, 9e-3], 1)]
    inst = ta.BatchTOPPRA(cons, path, grid)
    inst.setup()
    rec, R, conic, d_grid = inst.records, inst.R, inst.conic, inst.d_grid
    X = engine.scan_robust(rec, R, *conic, d_grid, feasible_sets=True)["K"]
    zeros = engine.as_device(np.zeros(B), path.device)
    stages = {
        "reachable_sets": lambda: inst.compute_reachable_sets(0.0, 0.0),
        "feasible_set_launch": lambda: engine.scan_robust(rec, R, *conic, d_grid, feasible_sets=True),
        "reachable_forward_launch": lambda: _forward(rec, R, conic, d_grid, X, zeros),
        "controllable_sets_range": lambda: inst.compute_controllable_sets(0.0, args.sdmax),
        "parameterization": lambda: inst.compute_parameterization(),
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
    L, _, fs = inst.compute_reachable_sets(0.0, 0.0)
    K, st = inst.compute_controllable_sets(0.0, args.sdmax)
    name, power = card()
    out = dict(workload="B=%d dof=7 G=%d, JointVelocity + RobustLinearConstraint(JointAcceleration, "
                        "[1e-3, 5e-2, 9e-3], interpolation), records reused; L(0, 0), K(0, %g)" % (B, G, args.sdmax),
               gpu=name, power_limit=power, ms=med, spread=spread, reachable_ok=int((fs == -1).sum()),
               controllable_ok=int((st == 0).sum()))
    print(json.dumps(out))


def _forward(rec, R, conic, grid, X, sdmin):
    """tbr_reachable_sets_robust alone, on the feasible sets X of an earlier launch."""
    import ctypes
    import torch
    from toppra_b200 import _lib, _lib_reach
    B, G, W = rec.shape
    ell = np.ascontiguousarray(conic[2], dtype=np.float64)
    L = torch.empty((B, G, 2), dtype=torch.float64, device=rec.device)
    fs = torch.empty((B,), dtype=torch.int32, device=rec.device)
    rc = _lib_reach.load().tbr_reachable_sets_robust(
        _lib.ptr(rec), W, int(R), int(conic[0]), int(conic[1]), ctypes.c_void_p(ell.ctypes.data), _lib.ptr(grid),
        1 if grid.dim() == 1 else 0, B, G, None, _lib.ptr(X), _lib.ptr(sdmin), None, _lib.ptr(L), _lib.ptr(fs),
        _lib.stream_ptr())
    _lib.check(rc, "tbr_reachable_sets_robust")
    return L


if __name__ == "__main__":
    main()
