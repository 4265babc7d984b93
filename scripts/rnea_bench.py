"""Rigid-body torque constraints at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints, vel + acc +
torque rows, with the 6-DOF robot of tests/golden/robots/arm6.urdf (RigidBodyModel.from_urdf).

Legs, timed in alternated rounds (one call of each leg per round, CUDA-synchronised wall time), medians and spread:
  terms     tbd_torque_terms alone on the B x G points (model.torque_terms);
  model     the whole BatchTOPPRA solve with the model as inv_dyn (one fused inverse-dynamics launch per record chunk);
  torch     the same solve with a pure-torch batched RNEA passed as batched=True (the route without this library);
  cosine    the config-3 solve with the compiled coupled_cosine device model, for scale;
  model_8k, torch_8k   the model and torch solves on the first 8192 paths (the torch route runs out of memory on the
            full batch: its intermediates are (B G, 3, 3) tensors per body).
Also checks that the model and the torch RNEA agree to 1e-12 of the torque scale, and prints the GPU name and power
limit read in the same run.  Prints one JSON line.

    python scripts/rnea_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import toppra_b200 as ta  # noqa: E402


def torch_rnea(packed, q, qd, qdd):
    """Featherstone RNEA written with torch tensor operations over the M points (a loop over bodies)."""
    nv = q.shape[1]
    dev = q.device
    P = torch.as_tensor(packed, device=dev)
    g = P[:3]
    st, f = [], []
    Rs, ps = [], []
    M = q.shape[0]
    for k in range(nv):
        bd = P[3 + 27 * k:3 + 27 * (k + 1)]
        ax, E, r = bd[2:5], bd[5:14].reshape(3, 3), bd[14:17]
        if float(bd[1]) == 0:
            s, c = torch.sin(q[:, k]), torch.cos(q[:, k])
            K = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], device=dev, dtype=q.dtype)
            J = torch.eye(3, device=dev, dtype=q.dtype) + s[:, None, None] * K + (1 - c)[:, None, None] * (K @ K)
            R = E @ J
            p = r.expand(M, 3)
        else:
            R = E.expand(M, 3, 3)
            p = r + (q[:, k:k + 1] * ax) @ E.T
        Rs.append(R)
        ps.append(p)
        par = int(bd[0])
        if par < 0:
            z = torch.zeros(M, 3, device=dev, dtype=q.dtype)
            wp, vp, dwp, dvp = z, z, z, (-g).expand(M, 3)
        else:
            wp, vp, dwp, dvp = st[par]
        RT = lambda x: torch.einsum("mji,mj->mi", R, x)   # noqa: E731
        w, v = RT(wp), RT(vp + torch.cross(wp, p, dim=1))
        dw, dv = RT(dwp), RT(dvp + torch.cross(dwp, p, dim=1))
        sq, sqq = ax * qd[:, k:k + 1], ax * qdd[:, k:k + 1]
        if float(bd[1]) == 0:
            w = w + sq
            dw = dw + sqq + torch.cross(w, sq, dim=1)
            dv = dv + torch.cross(v, sq, dim=1)
        else:
            v = v + sq
            dv = dv + sqq + torch.cross(w, sq, dim=1)
        st.append((w, v, dw, dv))
        m, c = bd[17], bd[18:21].expand(M, 3)
        Ic = torch.stack([bd[[21, 22, 23]], bd[[22, 24, 25]], bd[[23, 25, 26]]])
        hl = m * (v + torch.cross(w, c, dim=1))
        ha = w @ Ic.T + torch.cross(c, hl, dim=1)
        fl = m * (dv + torch.cross(dw, c, dim=1))
        n = dw @ Ic.T + torch.cross(c, fl, dim=1)
        f.append([n + torch.cross(w, ha, dim=1) + torch.cross(v, hl, dim=1), fl + torch.cross(w, hl, dim=1)])
    tau = torch.empty_like(q)
    for k in range(nv - 1, -1, -1):
        bd = P[3 + 27 * k:3 + 27 * (k + 1)]
        tau[:, k] = (f[k][0] if float(bd[1]) == 0 else f[k][1]) @ bd[2:5]
        par = int(bd[0])
        if par >= 0:
            Rf = torch.einsum("mij,mj->mi", Rs[k], f[k][1])
            f[par][0] = f[par][0] + torch.einsum("mij,mj->mi", Rs[k], f[k][0]) + torch.cross(ps[k], Rf, dim=1)
            f[par][1] = f[par][1] + Rf
    return tau


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=65536)
    ap.add_argument("--grid", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
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
    n = min(B * G, 1 << 20)
    ref = model(q[:n], qs[:n], qss[:n])
    alt = torch_rnea(model.packed, q[:n], qs[:n], qss[:n])
    agree = float((ref - alt).abs().max() / ref.abs().max().clamp(min=1.0))
    assert agree <= 1e-12, agree
    del ref, alt

    small = min(B, 8192)
    path_small = ta.BatchSplineInterpolator(ss, way[:small])

    def solve(inv_dyn, n=B, **kw):
        cons = [ta.constraint.JointVelocityConstraint(vlim[:n]), ta.constraint.JointAccelerationConstraint(alim[:n]),
                ta.constraint.SecondOrderConstraint.joint_torque_constraint(inv_dyn, taulim[:n], fric, **kw)]
        p = path if n == B else path_small
        return lambda: ta.BatchTOPPRA(cons, p, grid).compute_parameterization(0, 0)

    cos_taulim = np.stack([-(40 + 10 * rng.rand(B, nv)), 40 + 10 * rng.rand(B, nv)], axis=-1)
    cos_cons = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
                ta.constraint.SecondOrderConstraint.joint_torque_constraint(
                    None, cos_taulim, np.zeros(nv), device_model=("coupled_cosine", [2.0, 0.3, 0.1, 4.9]))]
    legs = {
        "terms": lambda: model.torque_terms(q, qs, qss, fric),
        "model": solve(model),
        "torch": solve(lambda a, b, c: torch_rnea(model.packed, a, b, c), batched=True),
        "cosine": lambda: ta.BatchTOPPRA(cos_cons, path, grid).compute_parameterization(0, 0),
        "model_8k": solve(model, small),
        "torch_8k": solve(lambda a, b, c: torch_rnea(model.packed, a, b, c), small, batched=True),
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
    res = solve(model)().to_host()
    rm, rt = solve(model, small)().to_host(), solve(lambda a, b, c: torch_rnea(model.packed, a, b, c), small,
                                                   batched=True)().to_host()
    assert (rm["status"] == rt["status"]).all()
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "rounds": args.rounds, "model_vs_torch_rnea": agree,
           "ok_paths": int((res["status"] == 0).sum())}
    for k, v in times.items():
        v = [x for x in v if np.isfinite(x)]
        out[k + "_ms"] = ({"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} if v
                          else "out of memory")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
