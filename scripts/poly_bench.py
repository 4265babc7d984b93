"""Order-k path solve cost on the GPU: 4096 paths x 7 DOF x 200 gridpoints, vel+acc, quintic pieces (k = 6).

Times each stage of the order-k record path with CUDA events (evaluate q' and q'', build the records, record scan) and
the whole solve in paths/s; beside it, the same batch's cubic figures (a cubic spline through the quintic path's
positions at its breaks): the record path (K1 + record scan) and the fused vel+acc scan.  Warm-up first, then
`--reps` alternated rounds; medians are reported.  Prints one JSON line with the card's name and power limit.

    python scripts/poly_bench.py [--reps 7] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    import toppra_b200 as ta
    from toppra_b200 import engine
    assert torch.cuda.is_available(), "poly_bench needs a GPU"
    B, G, dof, nseg, k = args.B, args.G, 7, 4, 6
    rng = np.random.RandomState(2024)
    x = np.linspace(0, 1, nseg + 1)
    c = rng.randn(B, k, nseg, dof) * (2.0 ** -np.arange(k)[::-1])[None, :, None, None] * 3.0
    vl = 10 + rng.rand(B, dof) * 20
    al = 10 + rng.rand(B, dof) * 2
    vlim, alim = np.stack((-vl, vl), -1), np.stack((-al, al), -1)
    grid = np.linspace(0, 1, G)

    def cons():
        return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]

    poly = ta.BatchPiecewisePolyPath(x, c)
    cubic = ta.BatchSplineInterpolator(x, poly.d_wp.cpu().numpy())
    inst = ta.BatchTOPPRA(cons(), poly, grid)
    rec_c = ta.BatchTOPPRA(cons(), cubic, grid, fused=False)
    fus_c = ta.BatchTOPPRA(cons(), cubic, grid)
    assert not inst.fused and not rec_c.fused and fus_c.fused
    d_grid, dev = inst.d_grid, poly.device
    d_vl, d_al = engine.as_device(vlim, dev), engine.as_device(alim, dev)
    R = inst.R
    records, _ = engine.alloc_records(B, G, R, dev)

    def ev():
        return engine.ppoly_eval(poly.d_ppoly, poly.d_ss, d_grid, 1), engine.ppoly_eval(poly.d_ppoly, poly.d_ss, d_grid, 2)

    qd, qdd = ev()
    stages = {
        "poly_eval": lambda: ev(),
        "poly_rows": lambda: engine.rows_velacc_sampled(qd, qdd, d_grid, d_vl, d_al, True, records, R, 0, 1),
        "record_scan": lambda: engine.scan(records, R, d_grid),
        "poly_total": lambda: inst.compute_parameterization(),
        "cubic_records_path": lambda: rec_c.compute_parameterization(),
        "cubic_fused": lambda: fus_c.compute_parameterization(),
    }
    # a full solve rebuilds the records each time, as a caller with new paths would
    full = {"poly_total": inst, "cubic_records_path": rec_c, "cubic_fused": fus_c}

    def run(name):
        if name in full:
            full[name].records = None
            full[name].xbound = None
        stages[name]()

    for name in stages:          # warm-up of every shape in the timed window
        for _ in range(3):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in stages}
    for _ in range(args.reps):
        for name in stages:       # alternated: every round times every stage once
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                run(name)
            t1.record()
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) / args.iters)
    med = {n: float(np.median(v)) for n, v in times.items()}
    spread = {n: float((max(v) - min(v)) / np.median(v)) for n, v in times.items()}
    name, power = card()
    out = dict(workload="B=%d dof=%d G=%d vel+acc, quintic pieces (k=6), %d pieces" % (B, dof, G, nseg), gpu=name,
               power_limit=power, ms=med, spread=spread,
               paths_per_s={n: B / (med[n] * 1e-3) for n in ("poly_total", "cubic_records_path", "cubic_fused")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
