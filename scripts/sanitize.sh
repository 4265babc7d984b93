#!/usr/bin/env bash
# compute-sanitizer over a small end-to-end solve (K0, K1, K2 record scan + fused scan + ragged, K2r, K3, LP shims, the row-f
# kernels of round 2: propose_gridpoints, reachable sets, TOPPRAsd bisection, spline time stamps, torque rows, ubound
# records): memcheck + racecheck + synccheck.
# usage: bash scripts/sanitize.sh [OUT_DIR]      (summary -> OUT_DIR/sanitizer.txt, default OUT_DIR = sanitizer_out)
set -u
OUT="${1:-sanitizer_out}"
mkdir -p "$OUT"
CASE="$(mktemp /tmp/san_case.XXXXXX.py)"
trap 'rm -f "$CASE"' EXIT
cat > "$CASE" <<'PY'
import sys, numpy as np
sys.path.insert(0, "."); sys.path.insert(0, "tests")
import toppra_b200 as ta
from problems import make_batch
B, G = 24, 40
ss, way, vlim, alim = make_batch(B, 1000)
grid = np.linspace(0, 1, G)
path = ta.BatchSplineInterpolator(ss, way)
vel, acc = ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)
inst = ta.BatchTOPPRA([vel, acc], path, grid)
res = inst.compute_parameterization(0.0, 0.0)
host = inst.solve_to_host(0.0, 0.0)
X = inst.compute_feasible_sets()
rob = ta.BatchTOPPRA([vel, ta.constraint.RobustLinearConstraint(acc, [1e-3, 5e-2, 9e-3], 1)], path, grid).compute_parameterization(0, 0)
bp = ta.BatchParametrizeConstAccel(path, grid, res.sd)
q = bp(np.linspace(0, 1.0, 16), 1)
r = ta.engine.lp2d_batch(np.random.randn(8, 3), np.random.randn(8, 40), np.random.randn(8, 40), -np.random.rand(8, 40),
                         np.tile([-1.0, -1.0], (8, 1)), np.tile([1.0, 1.0], (8, 1)))
rec = ta.BatchTOPPRA([vel, acc], path, grid, fused=False).compute_parameterization(0.0, 0.0)       # record scan (TMA ring)
rag = ta.BatchTOPPRA([vel, acc], path, gridpoints=None)                                           # propose_gridpoints + ragged fused scan
rag_res = rag.compute_parameterization(0.0, 0.0)
rag2 = ta.BatchTOPPRA([vel, acc], path, rag.d_grid, glen=rag.glen, fused=False).compute_parameterization(0.0, 0.0)
L, Xr, fail = inst.compute_reachable_sets(0.0, 0.3)
sdi = ta.BatchTOPPRAsd([vel, acc], path, grid); sdi.set_desired_duration(3.0); sdr = sdi.compute_parameterization(0.0, 0.0)
ps = ta.BatchParametrizeSpline(path, grid, res.sd); pq = ps(np.linspace(0, 1.0, 9), 2)
tl = np.stack((-45 * np.ones((B, 7)), 45 * np.ones((B, 7))), axis=-1)
tq = ta.BatchTOPPRA([vel, acc, ta.constraint.SecondOrderConstraint.joint_torque_constraint(None, tl, np.zeros(7), device_model=("coupled_cosine", [2.0, 0.3, 0.1, 4.9]))], path, grid).compute_parameterization(0, 0)
recs, _ = ta.engine.alloc_records(2, G, 28, path.device, ubound=True); ta.engine.init_bounds(recs, 28)
ta.engine.coeff_velacc(path.d_ppoly[:2].contiguous(), path.d_ss, inst.d_grid, None, acc.device_limits(path.device)[:2].contiguous(), True, recs, 28, 0, 0)
ub = ta.engine.scan(recs, 28, inst.d_grid)
print("ok", int((res.status != 0).sum()), int((rob.status != 0).sum()), float(bp.durations.min()), int(rag.glen.max()),
      int((rag_res.status != 0).sum() + (rag2.status != 0).sum() + (tq.status != 0).sum() + (sdr.status != 0).sum()), float(ps.durations.max()),
      int(ub["status"].sum()), int((rec.status != 0).sum()))
PY
for tool in memcheck racecheck synccheck; do
  echo "== compute-sanitizer --tool $tool"
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 7 python "$CASE" 2>&1 | grep -E "ERROR SUMMARY|RACECHECK SUMMARY|^ok|error|Error" | head -8
done 2>&1 | tee "$OUT/sanitizer.txt"
