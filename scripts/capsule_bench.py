"""Speed and separation monitoring with capsules: 4096 paths x 6 DOF x 200 gridpoints of tests/golden/robots/arm6.urdf,
velocity and acceleration limits plus SeparationMonitoringConstraint with one capsule per link (6 robot capsules, the
last one 10 cm past the flange) and 5 human capsules per path (torso, two upper arms, two forearms, one person per path
placed around the workspace), T_r = 0.1 s, a_s = 2.5 m/s^2, v_h = 1.6 m/s, C = 0.05 m.

Legs, timed with CUDA events in alternated rounds (one call of each leg per round), medians and spread:
  terms          tbd_capsule_separation_terms alone on the B x G points;
  setup          BatchTOPPRA(...) with the capsule limit: spline fit and stage records (one terms launch);
  solve          compute_parameterization of that instance;
  solve_all      the whole solve with the capsule limit (setup included);
  solve_spheres  the whole solve with sphere covers instead (tbd_separation_terms): 16 robot spheres that contain
                 the six link capsules, and 15 human spheres, three along each body capsule;
  solve_velacc   the whole solve with velocity and acceleration limits only.
Prints the GPU name and power limit read in the same run, the number of paths that solve and on how many the limit is
active, as one JSON line.

    python scripts/capsule_bench.py [--paths 4096] [--grid 200] [--rounds 5]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import toppra_b200 as ta  # noqa: E402
from separation_bench import PARAMS, gpu_info, timed  # noqa: E402

LINKS = [("shoulder", "upper_arm"), ("upper_arm", "forearm"), ("forearm", "wrist1"), ("wrist1", "wrist2"),
         ("wrist2", "wrist3")]
RADII = (0.08, 0.07, 0.06, 0.05, 0.05, 0.05)
COVER = (2, 4, 4, 2, 1, 3)      # spheres per link in the sphere cover: 16 in all


def capsules_and_cover(model):
    """The six link capsules, and a sphere cover of them: link k cut into COVER[k] equal pieces of length l, one sphere
    on the middle of each piece (on the first frame's body) of radius sqrt(r^2 + (l/2)^2), so the cover contains the
    capsule."""
    tool = model.frame("flange", xyz=(0.0, 0.0, 0.1))
    caps = [(model.frame(a), model.frame(b), r) for (a, b), r in zip(LINKS, RADII)]
    caps.append((model.frame("wrist3"), tool, RADII[-1]))
    body = {name: f[0] for name, f in model.frames.items()}
    cover = []
    for (a, b), r, n in zip(LINKS + [("wrist3", None)], RADII, COVER):
        # the segment's far end in the body coordinates of a: the next joint's origin, or the tool point
        end = tool.p if b is None else model.packed[3 + 27 * body[b] + 14: 3 + 27 * body[b] + 17]
        half = 0.5 * np.linalg.norm(end) / n
        for j in range(n):
            cover.append((model.frame(a, xyz=tuple((j + 0.5) / n * np.asarray(end))), float(np.hypot(r, half))))
    assert len(cover) == 16
    return caps, cover


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=4096)
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    B, G, nv = args.paths, args.grid, 6
    model = ta.RigidBodyModel.from_urdf(os.path.join(ROOT, "tests", "golden", "robots", "arm6.urdf"))
    caps, cover = capsules_and_cover(model)
    rng = np.random.RandomState(1234)
    ss = np.linspace(0, 1, 5)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vl = np.tile(model.velocity_limit, (B, 1))
    al = rng.uniform(6, 10, (B, nv))
    vlim, alim = (np.stack([-x, x], axis=-1) for x in (vl, al))
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    # one person per path, 0.8 to 1.6 m from the base, facing it: torso, upper arms and forearms
    ang = rng.uniform(0, 2 * np.pi, B)
    dist = rng.uniform(0.8, 1.6, B)
    base = np.stack([dist * np.cos(ang), dist * np.sin(ang), np.zeros(B)], axis=1)
    body = np.array([[0.0, 0.0, 0.9, 0.0, 0.0, 1.4, 0.17],
                     [0.2, 0.0, 1.4, 0.25, 0.0, 1.1, 0.05], [-0.2, 0.0, 1.4, -0.25, 0.0, 1.1, 0.05],
                     [0.25, 0.0, 1.1, 0.25, -0.3, 1.05, 0.04], [-0.25, 0.0, 1.1, -0.25, -0.3, 1.05, 0.04]])
    humans = np.concatenate((base[:, None, :] + body[None, :, :3], base[:, None, :] + body[None, :, 3:6],
                             np.broadcast_to(body[:, 6:], (B, 5, 1))), axis=2)
    ts = np.array([0.0, 0.5, 1.0])[None, None, :, None]
    centres = humans[:, :, None, :3] + ts * (humans[:, :, None, 3:6] - humans[:, :, None, :3])
    spheres = np.concatenate((centres, np.broadcast_to(humans[:, :, None, 6:], centres.shape[:3] + (1,))), axis=3)
    spheres = np.ascontiguousarray(spheres.reshape(B, 15, 4))

    def velacc():
        return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]

    def ssm():
        return velacc() + [ta.constraint.SeparationMonitoringConstraint(caps, humans, *PARAMS)]

    def ssm_spheres():
        return velacc() + [ta.constraint.SeparationMonitoringConstraint(cover, spheres, *PARAMS)]

    dgrid = torch.as_tensor(grid, device="cuda")
    q, qs = (path.eval_device(dgrid, o).reshape(B * G, nv) for o in (0, 1))
    cons = ssm()[2]
    assert cons.capsules and not ssm_spheres()[2].capsules
    hum_dev = torch.as_tensor(humans, device="cuda")
    inst = {}

    def setup():
        inst["x"] = ta.BatchTOPPRA(ssm(), path, grid)

    legs = {
        "terms": lambda: cons.terms(q, qs, hum_dev, G),
        "setup": setup,
        "solve": lambda: inst["x"].compute_parameterization(0, 0),
        "solve_all": lambda: ta.BatchTOPPRA(ssm(), path, grid).compute_parameterization(0, 0),
        "solve_spheres": lambda: ta.BatchTOPPRA(ssm_spheres(), path, grid).compute_parameterization(0, 0),
        "solve_velacc": lambda: ta.BatchTOPPRA(velacc(), path, grid).compute_parameterization(0, 0),
    }
    times = {k: [] for k in legs}
    for k, fn in legs.items():   # warm-up of every shape
        timed(fn)
    for _ in range(args.rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    rc = ta.BatchTOPPRA(ssm(), path, grid).compute_parameterization(0, 0).to_host()
    rs = ta.BatchTOPPRA(ssm_spheres(), path, grid).compute_parameterization(0, 0).to_host()
    r0 = ta.BatchTOPPRA(velacc(), path, grid).compute_parameterization(0, 0).to_host()
    b, c = (x.reshape(B, G).cpu().numpy() for x in cons.terms(q, qs, hum_dev, G))
    ok = rc["status"] == 0
    sd2 = np.nan_to_num(rc["sd"]) ** 2
    active = ok & ((b > 0) & (b * sd2 >= -c * (1 - 1e-6))).any(axis=1)

    def duration(h):
        """Median duration of the solved paths that do not stop on the way."""
        with np.errstate(divide="ignore"):
            dur = [np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) for s in h["sd"][h["status"] == 0]]
        return float(np.median([x for x in dur if np.isfinite(x)]))

    out = {"gpu": gpu_info(), "paths": B, "grid": G, "dof": nv, "capsules": len(caps), "humans": humans.shape[1],
           "cover_spheres": len(cover), "human_spheres": spheres.shape[1], "rounds": args.rounds,
           "params": dict(zip(("reaction_time", "stopping_deceleration", "human_speed", "clearance"), PARAMS)),
           "ok_paths": int(ok.sum()), "ok_paths_spheres": int((rs["status"] == 0).sum()),
           "ok_paths_velacc": int((r0["status"] == 0).sum()), "active_paths": int(active.sum()),
           "within_limit": bool((b * sd2 + c <= 1e-9)[ok].all()),
           "median_duration_s": {"capsules": duration(rc), "spheres": duration(rs), "velacc": duration(r0)}}
    for k, v in times.items():
        out[k + "_ms"] = {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
