"""Collision-energy limit at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints, vel + acc + torque rows
of tests/golden/robots/arm6.urdf and CollisionEnergyConstraint on a point 10 cm past its flange, m_H = 0.6 kg (a hand),
one limit per path: 0.3 of the largest collision energy b sd^2 of that path's profile without the limit (so that it is
active on most paths).

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms          tbd_collision_energy_terms alone on the B x G points (RigidBodyFrame.collision_energy_terms);
  solve_energy   the whole BatchTOPPRA solve with CollisionEnergyConstraint (one terms launch per record chunk);
  solve          the same solve without it;
  torch          the same b from a pure-torch route on the first --torch-points points (torch.linalg.cholesky on M
                 built column by column from tbd_torque_terms, J_v from tbd_frame_velocity), for scale.
Also checks that the kernel and the torch route agree to 1e-12 of the scale, and prints the GPU name and power limit read
in the same run, the number of paths that solve with and without the limit and on how many the limit is active.  Prints
one JSON line.

    python scripts/collision_energy_bench.py [--paths 65536] [--grid 500] [--rounds 5] [--torch-points 1048576]"""
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

HUMAN_MASS = 0.6
SHARE = 0.3


def torch_energy_terms(model, frame, q, qs, human_mass):
    """b from M(q) (nv tbd_torque_terms launches with unit q'), torch.linalg.cholesky, torch.cholesky_solve and J_v
    (nv tbd_frame_velocity launches with unit qd)."""
    M, nv = q.shape
    zero = torch.zeros_like(q)
    eye = torch.eye(nv, dtype=q.dtype, device=q.device)
    Mq = torch.stack([model.torque_terms(q, eye[k].expand(M, nv), zero)[0] for k in range(nv)], dim=2)   # M e_k
    J = torch.stack([frame(q, eye[k].expand(M, nv))[:, :3] for k in range(nv)], dim=2)      # (M, 3, nv)
    L = torch.linalg.cholesky(Mq)
    X = torch.cholesky_solve(J.transpose(1, 2), L)                                            # M^-1 J^T
    Linv = J @ X
    v = frame(q, qs)[:, :3]
    vv = (v * v).sum(dim=1)
    w = (v * (Linv @ v[:, :, None])[:, :, 0]).sum(dim=1)
    return torch.where(vv == 0, torch.zeros_like(vv), 0.5 * vv * vv / (vv / human_mass + w))


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
    ap.add_argument("--torch-points", type=int, default=1 << 20)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    tcp = model.frame("flange", xyz=(0.0, 0.0, 0.1))
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
    q, qs = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1))
    n = min(B * G, args.torch_points)
    ref = tcp.collision_energy_terms(q[:n], qs[:n], HUMAN_MASS)
    alt = torch_energy_terms(model, tcp, q[:n], qs[:n], HUMAN_MASS)
    agree = float((ref - alt).abs().max() / ref.abs().max())
    assert agree <= 1e-12, agree
    del ref, alt

    def cons(limit):
        c = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
             ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
        return c + [ta.constraint.CollisionEnergyConstraint(tcp, limit, HUMAN_MASS)] if limit is not None else c

    r0 = ta.BatchTOPPRA(cons(None), path, grid).compute_parameterization(0, 0).to_host()
    b = tcp.collision_energy_terms(q, qs, HUMAN_MASS).reshape(B, G).cpu().numpy()
    limit = SHARE * np.max(b * np.nan_to_num(r0["sd"]) ** 2, axis=1)
    limit = np.where(limit > 0, limit, 1.0)              # paths that do not solve without the limit: any limit

    legs = {
        "terms": lambda: tcp.collision_energy_terms(q, qs, HUMAN_MASS),
        "solve_energy": lambda: ta.BatchTOPPRA(cons(limit), path, grid).compute_parameterization(0, 0),
        "solve": lambda: ta.BatchTOPPRA(cons(None), path, grid).compute_parameterization(0, 0),
        "torch": lambda: torch_energy_terms(model, tcp, q[:n], qs[:n], HUMAN_MASS),
    }
    times = {k: [] for k in legs}
    for k, fn in legs.items():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    rc = ta.BatchTOPPRA(cons(limit), path, grid).compute_parameterization(0, 0).to_host()
    ok = rc["status"] == 0
    E = b * np.nan_to_num(rc["sd"]) ** 2
    active = ok & (E >= limit[:, None] * (1 - 1e-6)).any(axis=1)
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "rounds": args.rounds, "human_mass": HUMAN_MASS,
           "limit_share": SHARE, "limit_J": {"median": float(np.median(limit)), "min": float(limit.min()),
                                             "max": float(limit.max())},
           "torch_points": n, "kernel_vs_torch": agree, "ok_paths": int(ok.sum()),
           "ok_paths_without_energy": int((r0["status"] == 0).sum()), "active_paths": int(active.sum()),
           "energy_within_limit": bool((E[ok] <= limit[ok, None] * (1 + 1e-9)).all())}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
