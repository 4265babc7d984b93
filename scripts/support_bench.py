"""Support stability at the BASELINE config-3 shape: 65 536 paths x 6 DOF x 500 gridpoints, vel + acc + torque rows of
tests/golden/robots/arm6.urdf standing on a pedestal cart: the arm's base_link is mounted 0.5 m above the floor on a
30 kg cart (centre of mass 0.25 m above the floor) whose small 6 x 5 cm foot, centred 3 cm ahead of the arm's axis,
slides with mu = 0.5 (the 16-row contact wrench cone of SupportStabilityConstraint); the foot is small enough that the
limit binds.  The paths start at the statically stable pose of tests/golden/support_stability.npz and take four random
steps of at most 0.1 rad per joint; joint accelerations are limited to 10..15 rad/s^2.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms          tbd_support_wrench_terms alone on the B x G points (RigidBodyFrame.support_wrench_terms);
  solve_support  the whole BatchTOPPRA solve with SupportStabilityConstraint (one terms launch per record chunk);
  solve          the same solve without it;
  torch          the same a, b and c computed by a pure-torch recursive Newton-Euler route on the first 1 M points,
                 for scale.
Also checks that the kernel and the torch route agree to 1e-12 of the scale, and prints the GPU name and power limit
read in the same run, the number of paths that solve with and without the constraint, and on how many solved paths a
support row is active (within 1e-6 of the wrench's scale at some gridpoint).  Prints one JSON line.

    python scripts/support_bench.py [--paths 65536] [--grid 500] [--rounds 5]"""
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

CART_HEIGHT, CART_MASS, CART_COM = 0.5, 30.0, (0.0, 0.0, -0.25)    # base coordinates: the arm's base_link origin
FOOT = (0.03, 0.0)                                                 # centre of the foot, base coordinates
HALF_LENGTHS, FRICTION = (0.03, 0.025), 0.5


def torch_support_terms(model, frame, base, q, qs, qss):
    """c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c of the support wrench, written with torch tensor
    operations over the M points (three recursive Newton-Euler passes over the tree)."""
    dev, M, dt = q.device, q.shape[0], q.dtype
    P = torch.as_tensor(model.packed, device=dev)
    nv = model.nv
    cross = lambda a, b: torch.cross(a, b, dim=1)  # noqa: E731
    Rs, ps = [], []
    for k in range(nv):
        bd = P[3 + 27 * k:3 + 27 * (k + 1)]
        ax, E, r = bd[2:5], bd[5:14].reshape(3, 3), bd[14:17]
        if float(bd[1]) == 0:
            s, c = torch.sin(q[:, k]), torch.cos(q[:, k])
            K = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], device=dev, dtype=dt)
            J = torch.eye(3, device=dev, dtype=dt) + s[:, None, None] * K + (1 - c)[:, None, None] * (K @ K)
            Rs.append(E @ J)
            ps.append(r.expand(M, 3))
        else:
            Rs.append(E.expand(M, 3, 3))
            ps.append(r + (q[:, k:k + 1] * ax) @ E.T)
    Rsup, psup = torch.as_tensor(frame.R, device=dev), torch.as_tensor(frame.p, device=dev)
    bt = torch.as_tensor(base, device=dev)
    zero = torch.zeros_like(q)
    out = []
    for qd, qdd in ((zero, zero), (zero, qs), (qs, qss)):
        st, f = [], []
        for k in range(nv):
            bd = P[3 + 27 * k:3 + 27 * (k + 1)]
            par = int(model.packed[3 + 27 * k])
            if par < 0:
                wp = vp = dwp = torch.zeros(M, 3, device=dev, dtype=dt)
                dvp = (-P[:3]).expand(M, 3)
            else:
                wp, vp, dwp, dvp = st[par]
            R, p = Rs[k], ps[k]
            RT = lambda x: torch.einsum("mji,mj->mi", R, x)  # noqa: E731
            w, v, dw, dv = RT(wp), RT(vp + cross(wp, p)), RT(dwp), RT(dvp + cross(dwp, p))
            sq, sqq = bd[2:5] * qd[:, k:k + 1], bd[2:5] * qdd[:, k:k + 1]
            if float(bd[1]) == 0:
                w = w + sq
                dw = dw + sqq + cross(w, sq)
                dv = dv + cross(v, sq)
            else:
                v = v + sq
                dv = dv + sqq + cross(w, sq)
            st.append((w, v, dw, dv))
            m, c = bd[17], bd[18:21].expand(M, 3)
            I = torch.stack([bd[[21, 22, 23]], bd[[22, 24, 25]], bd[[23, 25, 26]]])
            hl = m * (v + cross(w, c))
            ha = w @ I.T + cross(c, hl)
            fl = m * (dv + cross(dw, c))
            n = dw @ I.T + cross(c, fl)
            f.append([n + cross(w, ha) + cross(v, hl), fl + cross(w, hl)])
        fb = torch.zeros(M, 3, device=dev, dtype=dt)
        nb = torch.zeros(M, 3, device=dev, dtype=dt)
        for k in range(nv - 1, -1, -1):
            Rf = torch.einsum("mij,mj->mi", Rs[k], f[k][1])
            Rn = torch.einsum("mij,mj->mi", Rs[k], f[k][0]) + cross(ps[k], Rf)
            par = int(model.packed[3 + 27 * k])
            if par >= 0:
                f[par][0] = f[par][0] + Rn
                f[par][1] = f[par][1] + Rf
            else:
                nb, fb = nb + Rn, fb + Rf
        wb = (-(bt[0] * P[:3])).expand(M, 3)
        nb = nb + cross(bt[1:4].expand(M, 3), wb)
        fb = fb + wb
        t = nb - cross(psup.expand(M, 3), fb)
        out.append(torch.cat((fb @ Rsup, t @ Rsup), dim=1))
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
    floor = model.frame("base_link", xyz=(FOOT[0], FOOT[1], -CART_HEIGHT))
    up = np.load(os.path.join(ROOT, "tests", "golden", "support_stability.npz"))["arm6/up"]
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    steps = np.concatenate((np.zeros((B, 1, nv)), rng.uniform(-0.1, 0.1, (B, 4, nv))), axis=1)
    way = up + np.cumsum(steps, axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(10, 15, (B, nv))
    tl = 0.45 * model.effort_limit * rng.uniform(0.8, 1.2, (B, nv))
    vlim, alim, taulim = (np.stack([-x, x], axis=-1) for x in (vl, al, tl))
    fric = 0.3 + 0.1 * np.arange(nv)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    # the cart and the arm's own base_link: one static base
    mb = CART_MASS + model.base_mass
    cb = (CART_MASS * np.asarray(CART_COM) + model.base_mass * model.base_com) / mb
    support = ta.constraint.SupportStabilityConstraint(floor, half_lengths=HALF_LENGTHS, friction=FRICTION,
                                                       base_mass=mb, base_com=cb)
    base = support.base

    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs, qss = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1, 2))
    n = min(B * G, 1 << 20)
    ref = floor.support_wrench_terms(base, q[:n], qs[:n], qss[:n])
    alt = torch_support_terms(model, floor, base, q[:n], qs[:n], qss[:n])
    agree = max(float((x - y).abs().max() / x.abs().max().clamp(min=1.0)) for x, y in zip(ref, alt))
    assert agree <= 1e-12, agree
    del ref, alt
    qn, qsn, qssn = q[:n].clone(), qs[:n].clone(), qss[:n].clone()

    def cons(with_support):
        c = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
             ta.constraint.SecondOrderConstraint.joint_torque_constraint(model, taulim, fric)]
        return c + [support] if with_support else c

    legs = {
        "terms": lambda: floor.support_wrench_terms(base, q, qs, qss),
        "solve_support": lambda: ta.BatchTOPPRA(cons(True), path, grid).compute_parameterization(0, 0),
        "solve": lambda: ta.BatchTOPPRA(cons(False), path, grid).compute_parameterization(0, 0),
        "torch_1M": lambda: torch_support_terms(model, floor, base, qn, qsn, qssn),
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
    rs = ta.BatchTOPPRA(cons(True), path, grid).compute_parameterization(0, 0).to_host()
    r0 = ta.BatchTOPPRA(cons(False), path, grid).compute_parameterization(0, 0).to_host()
    # activity: w = a u + b x + c at the start of every stage of the solved profiles
    a, b, c = floor.support_wrench_terms(base, q, qs, qss)
    Fd = torch.as_tensor(support.F, device="cuda")
    ok = rs["status"] == 0
    sdd = torch.as_tensor(np.nan_to_num(rs["sdd"]), device="cuda")
    x = torch.as_tensor(np.nan_to_num(rs["sd"][:, :-1]) ** 2, device="cuda")
    w = (a.reshape(B, G, 6)[:, :-1] * sdd[..., None] + b.reshape(B, G, 6)[:, :-1] * x[..., None]
         + c.reshape(B, G, 6)[:, :-1])
    v = w @ Fd.T
    scale = w.abs().amax(dim=2, keepdim=True) * max(1.0, float(np.abs(support.F).max()))
    active = ((v >= -1e-6 * scale).any(dim=2).any(dim=1)).cpu().numpy()
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "rounds": args.rounds, "kernel_vs_torch": agree,
           "torch_points": n, "ok_paths": int(ok.sum()), "ok_paths_without_support": int((r0["status"] == 0).sum()),
           "support_active_paths": int((active & ok).sum()),
           "slower_paths": int((ok & (r0["status"] == 0) & (rs["sd"] < r0["sd"] * (1 - 1e-9)).any(axis=1)).sum())}
    for k, v in times.items():
        v = [t for t in v if np.isfinite(t)]
        out[k + "_ms"] = ({"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} if v
                          else "out of memory")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
