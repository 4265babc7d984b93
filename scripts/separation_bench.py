"""Speed and separation monitoring: 4096 paths x 6 DOF x 200 gridpoints of tests/golden/robots/arm6.urdf, velocity and
acceleration limits plus SeparationMonitoringConstraint with P = 6 robot points (one per moving link, the tool 10 cm past
the flange) and H = 4 human spheres per path (one set per path, placed around the tool's workspace), T_r = 0.1 s,
a_s = 2.5 m/s^2, v_h = 1.6 m/s, C = 0.05 m.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms          tbd_separation_terms alone on the B x G points (RigidBodyModel.separation_terms);
  setup          BatchTOPPRA(...) with the separation limit: spline fit and stage records (one terms launch);
  solve_ssm      compute_parameterization of that instance;
  solve_velacc   the whole solve (setup included) with velocity and acceleration limits only;
  solve_energy   the whole solve with CollisionEnergyConstraint (0.6 kg, 2 J) on the tool in place of the separation
                 limit;
  solve_ssm_all  the whole solve with the separation limit (setup included), for comparison with the two above.
Prints the GPU name and power limit read in the same run, the number of paths that solve and on how many the separation
limit is active, as one JSON line.

    python scripts/separation_bench.py [--paths 4096] [--grid 200] [--rounds 5]"""
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

PARAMS = (0.1, 2.5, 1.6, 0.05)


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
    ap.add_argument("--paths", type=int, default=4096)
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    tcp = model.frame("flange", xyz=(0.0, 0.0, 0.1))
    points = [(tcp, 0.06)] + [(model.frame(link), 0.08) for link in ("shoulder", "upper_arm", "forearm", "wrist1",
                                                                    "wrist2")]
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    vlim, alim = (np.stack([-x, x], axis=-1) for x in (vl, al))
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    # four spheres per path: a person 0.8 to 1.6 m from the base, head, torso and two hands
    ang = rng.uniform(0, 2 * np.pi, B)
    dist = rng.uniform(0.8, 1.6, B)
    base = np.stack([dist * np.cos(ang), dist * np.sin(ang), np.zeros(B)], axis=1)
    offs = np.array([[0.0, 0.0, 1.6, 0.12], [0.0, 0.0, 1.2, 0.2], [0.25, 0.2, 1.0, 0.08], [-0.25, 0.2, 1.0, 0.08]])
    humans = np.concatenate((base[:, None, :] + offs[None, :, :3], np.broadcast_to(offs[:, 3:], (B, 4, 1))), axis=2)

    def velacc():
        return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]

    def ssm():
        return velacc() + [ta.constraint.SeparationMonitoringConstraint(points, humans, *PARAMS)]

    def energy():
        return velacc() + [ta.constraint.CollisionEnergyConstraint(tcp, 2.0, 0.6)]

    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1))
    cons = ssm()[2]
    hum_dev = torch.as_tensor(humans, device="cuda")
    inst = {}

    def setup():
        inst["x"] = ta.BatchTOPPRA(ssm(), path, grid)

    legs = {
        "terms": lambda: cons.terms(q, qs, hum_dev, G),
        "setup": setup,
        "solve_ssm": lambda: inst["x"].compute_parameterization(0, 0),
        "solve_velacc": lambda: ta.BatchTOPPRA(velacc(), path, grid).compute_parameterization(0, 0),
        "solve_energy": lambda: ta.BatchTOPPRA(energy(), path, grid).compute_parameterization(0, 0),
        "solve_ssm_all": lambda: ta.BatchTOPPRA(ssm(), path, grid).compute_parameterization(0, 0),
    }
    times = {k: [] for k in legs}
    for k, fn in legs.items():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    rc = ta.BatchTOPPRA(ssm(), path, grid).compute_parameterization(0, 0).to_host()
    r0 = ta.BatchTOPPRA(velacc(), path, grid).compute_parameterization(0, 0).to_host()
    b, c = (x.reshape(B, G).cpu().numpy() for x in cons.terms(q, qs, hum_dev, G))
    ok = rc["status"] == 0
    sd2 = np.nan_to_num(rc["sd"]) ** 2
    active = ok & ((b > 0) & (b * sd2 >= -c * (1 - 1e-6))).any(axis=1)
    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "points": len(points), "humans": humans.shape[1],
           "rounds": args.rounds, "params": dict(zip(("reaction_time", "stopping_deceleration", "human_speed",
                                                      "clearance"), PARAMS)),
           "ok_paths": int(ok.sum()), "ok_paths_velacc": int((r0["status"] == 0).sum()),
           "active_paths": int(active.sum()), "within_limit": bool((b * sd2 + c <= 1e-9)[ok].all())}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
