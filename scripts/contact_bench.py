"""Contact stability at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints, vel + acc + torque rows of
tests/golden/robots/arm6.urdf and a tray on its flange (1 cm out) carrying a 0.8 kg box on a 10 x 8 cm base, mu = 0.5
(the object of tests/test_contact_stability.py).  The paths start at the pose where the tray faces up (stored in
tests/golden/contact_stability.npz) and take four random steps of at most 0.06 rad per joint.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms          tbd_contact_wrench_terms alone on the B x G points (RigidBodyFrame.contact_wrench_terms);
  solve_contact  the whole BatchTOPPRA solve with ContactStabilityConstraint (one terms launch per record chunk);
  solve          the same solve without it;
  torch          the same a, b and c computed by a pure-torch contact-wrench callback, for scale.
Also checks that the kernel and the torch callback agree to 1e-12 of the scale, and prints the GPU name and power limit
read in the same run and the number of paths that solve with and without the constraint.  Prints one JSON line.

    python scripts/contact_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
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

OBJECT = np.array([0.8, 0.006, -0.004, 0.06, 0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017])
HALF_LENGTHS, FRICTION = (0.05, 0.04), 0.5


def torch_contact_terms(model, frame, obj, q, qs, qss):
    """c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c of the contact wrench, written with torch tensor
    operations over the M points (a loop over the frame's chain)."""
    dev, M, dt = q.device, q.shape[0], q.dtype
    P = torch.as_tensor(model.packed, device=dev)
    chain, k = [], frame.body
    while k >= 0:
        chain.append(k)
        k = int(model.packed[3 + 27 * k])
    Rw = torch.eye(3, device=dev, dtype=dt).expand(M, 3, 3)
    zero = torch.zeros_like(q)
    states = [[zero, zero], [zero, qs], [qs, qss]]
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
        for i in range(3):
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
    Rf = Rw @ torch.as_tensor(frame.R, device=dev)
    gl = torch.einsum("mji,j->mi", Rf, P[:3])
    o = torch.as_tensor(obj, device=dev)
    rr = o[1:4].expand(M, 3)
    I = torch.stack([o[[4, 5, 6]], o[[5, 7, 8]], o[[6, 8, 9]]])
    out = []
    for i in range(3):
        af = ao[i] + torch.cross(dw[i], d, dim=1) + torch.cross(w[i], torch.cross(w[i], d, dim=1), dim=1)
        al, dwl, wl = (torch.einsum("mji,mj->mi", Rf, x) for x in (af, dw[i], w[i]))
        f = o[0] * (al + torch.cross(dwl, rr, dim=1) + torch.cross(wl, torch.cross(wl, rr, dim=1), dim=1) - gl)
        tau = dwl @ I.T + torch.cross(wl, wl @ I.T, dim=1) + torch.cross(rr, f, dim=1)
        out.append(torch.cat((f, tau), dim=1))
    return out[1] - out[0], out[2] - out[0], out[0]


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
    tray = model.frame("flange", xyz=(0.0, 0.0, 0.01))
    up = np.load(os.path.join(ROOT, "tests", "golden", "contact_stability.npz"))["arm6/up"]
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    steps = np.concatenate((np.zeros((B, 1, nv)), rng.uniform(-0.06, 0.06, (B, 4, nv))), axis=1)
    way = up + np.cumsum(steps, axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    tl = 0.45 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nv))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    fric = 0.3 + 0.1 * np.arange(nv)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)

    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1, 2))
    n = min(B * G, 1 << 20)
    ref = tray.contact_wrench_terms(OBJECT, q[:n], qs[:n], qss[:n])
    alt = torch_contact_terms(model, tray, OBJECT, q[:n], qs[:n], qss[:n])
    agree = max(float((x - y).abs().max() / x.abs().max().clamp(min=1.0)) for x, y in zip(ref, alt))
    assert agree <= 1e-12, agree
    del ref, alt

    def cons(contact):
        c = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
             ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
        return c + [ta.constraint.ContactStabilityConstraint(tray, OBJECT[0], OBJECT[1:4], OBJECT[4:10], HALF_LENGTHS,
                                                             FRICTION)] if contact else c

    legs = {
        "terms": lambda: tray.contact_wrench_terms(OBJECT, q, qs, qss),
        "solve_contact": lambda: ta.BatchTOPPRA(cons(True), path, grid).compute_parameterization(0, 0),
        "solve": lambda: ta.BatchTOPPRA(cons(False), path, grid).compute_parameterization(0, 0),
        "torch": lambda: torch_contact_terms(model, tray, OBJECT, q, qs, qss),
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
           "ok_paths": int((rc["status"] == 0).sum()), "ok_paths_without_contact": int((r0["status"] == 0).sum()),
           "slower_paths": int(((rc["status"] == 0) & (r0["status"] == 0)
                                & (rc["sd"] < r0["sd"] * (1 - 1e-9)).any(axis=1)).sum())}
    for k, v in times.items():
        v = [x for x in v if np.isfinite(x)]
        out[k + "_ms"] = ({"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} if v
                          else "out of memory")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
