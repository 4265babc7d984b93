"""Cartesian acceleration limits at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints, vel + acc +
torque rows and a tool-acceleration limit on the three linear components of the flange of
tests/golden/robots/arm6.urdf, 0.1 m out along its z axis, with one set of limits per path.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms       tbd_acceleration_terms alone on the B x G points (RigidBodyFrame.acceleration_terms);
  solve_acc   the whole BatchTOPPRA solve with CartesianAccelerationConstraint (one terms launch per record chunk);
  solve       the same solve without it;
  torch       the same a and b computed by a pure-torch frame-acceleration callback, for scale.
Also checks that the kernel and the torch callback agree to 1e-12 of the scale, and prints the GPU name and power limit
read in the same run.  Prints one JSON line.

    python scripts/cartesian_accel_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import toppra_b200 as ta  # noqa: E402


def torch_acceleration_terms(model, frame, q, qs, qss):
    """a = acc(q, 0, qs), b = acc(q, qs, qss), the linear classical acceleration of the frame (local_world_aligned),
    written with torch tensor operations over the M points (a loop over the frame's chain)."""
    dev, M, dt = q.device, q.shape[0], q.dtype
    P = torch.as_tensor(model.packed, device=dev)
    chain, k = [], frame.body
    while k >= 0:
        chain.append(k)
        k = int(model.packed[3 + 27 * k])
    Rw = torch.eye(3, device=dev, dtype=dt).expand(M, 3, 3)
    zero = torch.zeros_like(q)
    states = [[zero, qs], [qs, qss]]                 # (qd, qdd) of a and of b
    w, dw, ao = ([torch.zeros(M, 3, device=dev, dtype=dt) for _ in states] for _ in range(3))
    for k in reversed(chain):
        bd = P[3 + 27 * k:3 + 27 * (k + 1)]
        ax, E, r = bd[2:5], bd[5:14].reshape(3, 3), bd[14:17]
        if float(bd[1]) == 0:
            s, c = torch.sin(q[:, k]), torch.cos(q[:, k])
            K = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], device=dev, dtype=dt)
            J = torch.eye(3, device=dev, dtype=dt) + s[:, None, None] * K + (1 - c)[:, None, None] * (K @ K)
            R, p = E @ J, r.expand(M, 3)
        else:
            R, p = E.expand(M, 3, 3), r + (q[:, k:k + 1] * ax) @ E.T
        d = torch.einsum("mij,mj->mi", Rw, p)
        for i in range(2):
            ao[i] = ao[i] + torch.cross(dw[i], d, dim=1) + torch.cross(w[i], torch.cross(w[i], d, dim=1), dim=1)
        Rw = Rw @ R
        sw = Rw @ ax
        for i, (qd, qdd) in enumerate(states):
            sq = sw * qd[:, k:k + 1]
            c = torch.cross(w[i], sq, dim=1)
            if float(bd[1]) == 0:
                dw[i] = dw[i] + sw * qdd[:, k:k + 1] + c
                w[i] = w[i] + sq
            else:
                ao[i] = ao[i] + sw * qdd[:, k:k + 1] + 2.0 * c
    d = Rw @ torch.as_tensor(frame.p, device=dev)
    return tuple(ao[i] + torch.cross(dw[i], d, dim=1) + torch.cross(w[i], torch.cross(w[i], d, dim=1), dim=1)
                 for i in range(2))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--grid", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    tcp = model.frame("flange", xyz=(0.0, 0.0, 0.1))
    comps = (0, 1, 2)
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    tl = 0.45 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nv))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    fric = 0.3 + 0.1 * np.arange(nv)
    acc = rng.uniform(2.0, 4.0, (B, 1)) * np.ones((1, 3))   # tool acceleration limits, m/s^2, per path and axis
    climit = np.stack([-acc, acc], axis=-1)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)

    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1, 2))
    n = min(B * G, 1 << 20)
    ref = tcp.acceleration_terms(q[:n], qs[:n], qss[:n], comps)
    alt = torch_acceleration_terms(model, tcp, q[:n], qs[:n], qss[:n])
    agree = max(float((x - y).abs().max() / x.abs().max().clamp(min=1.0)) for x, y in zip(ref, alt))
    assert agree <= 1e-12, agree
    del ref, alt

    def cons(cart):
        c = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
             ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
        return c + [ta.constraint.CartesianAccelerationConstraint(tcp, climit, comps)] if cart else c

    legs = {
        "terms": lambda: tcp.acceleration_terms(q, qs, qss, comps),
        "solve_acc": lambda: ta.BatchTOPPRA(cons(True), path, grid).compute_parameterization(0, 0),
        "solve": lambda: ta.BatchTOPPRA(cons(False), path, grid).compute_parameterization(0, 0),
        "torch": lambda: torch_acceleration_terms(model, tcp, q, qs, qss),
    }
    times = {k: [] for k in legs}
    for k, fn in legs.items():   # warm-up of every shape
        try:
            timed(fn)
        except torch.cuda.OutOfMemoryError:
            print("%s: out of memory at %d paths" % (k, B), file=sys.stderr)
            torch.cuda.empty_cache()
    for _ in range(args.rounds):
        for k, fn in legs.items():
            try:
                times[k].append(timed(fn))
            except torch.cuda.OutOfMemoryError:
                times[k].append(float("nan"))
                torch.cuda.empty_cache()
    rc = ta.BatchTOPPRA(cons(True), path, grid).compute_parameterization(0, 0).to_host()
    r0 = ta.BatchTOPPRA(cons(False), path, grid).compute_parameterization(0, 0).to_host()
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "rounds": args.rounds, "kernel_vs_torch": agree,
           "ok_paths": int((rc["status"] == 0).sum()), "ok_paths_without_acc": int((r0["status"] == 0).sum()),
           "slower_paths": int(((rc["status"] == 0) & (r0["status"] == 0)
                                & (rc["sd"] < r0["sd"] * (1 - 1e-9)).any(axis=1)).sum())}
    for k, v in times.items():
        v = [x for x in v if np.isfinite(x)]
        out[k + "_ms"] = ({"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} if v
                          else "out of memory")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
