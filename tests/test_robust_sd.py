"""Robust (conic) TOPPRAsd and single stage solves (libtoppra_b200_robust.so: tbr_sd_forward_robust,
tbr_socp_stage_batch).  Parity with the reference is unpinned (it solves these problems with ECOS), so the C restatement
(tests/robust_sd_oracle.c, on oracle/toppra_robust_oracle.c's stage primitives) is checked against independent evidence
on the CPU:
  * TOPPRAsd passes: every stage's rows hold at (u, x) in long double, and one step further on the optimising side some
    row is violated; blended durations hit the desired one within atol;
  * stage solves: objective against scipy SLSQP on sampled config-4 stages; the reference's infeasible instances;
  * zero ellipsoid: equal to the linear Seidel restatement (TOPPRAsd passes, stage LPs).
The kernels equal the restatement bit for bit on the GPU (NaN equal to NaN), for 1 to 4 rows per lane, linear and conic
rows, failing paths, ragged and chunked batches.  The host logic (BatchTOPPRAsd, TOPPRAsd, solve_stagewise_optim) runs on
the CPU through tests/cpu_engine.py plus the doubles of the two new engine functions defined here."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import cpu_engine
import robust_sd_oracle as rso
from oracle import oracle as orc
from problems import make_batch, make_path

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROBUST_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_robust.so")
ELL = [1e-3, 5e-2, 9e-3]   # defaults of examples/plot_robust_kinematics.py:26-28
LD = np.longdouble
ECOS_INFTY, ECOS_MAXX = 1000.0, 10000.0


def eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _cfg4(seed, G=200, interp=True):
    """cfg 4 rows: limits of cfg 2, rows/xbound of the acceleration constraint from the linear oracle."""
    ss = np.linspace(0, 1, 5)
    grid = np.linspace(0, 1, G)
    way, vlim, alim = make_path(seed)
    lin = orc.solve_velacc(orc.cubic_spline_fit(ss, way), ss, grid, vlim, alim, interp, 0, 0, want_rows=True)
    return grid, lin["rows"], lin["xbound"]


def _row_values(a, b, c, conic, ell, u, x):
    """a u + b x + c (+ the cone term on conic rows) in long double."""
    u, x = LD(u), LD(x)
    v = a.astype(LD) * u + b.astype(LD) * x + c.astype(LD)
    nrm = np.sqrt((LD(ell[0]) * u) ** 2 + (LD(ell[1]) * x) ** 2 + LD(ell[2]) ** 2)
    return np.where(conic, v + nrm, v)


def _duration(xs, grid):
    sds = np.sqrt(xs)
    t = 0.0
    for i in range(len(grid) - 1):
        t += 2 * (grid[i + 1] - grid[i]) / (sds[i + 1] + sds[i] + 1e-9)
    return t


def _sd_passes(rows, xb, grid, ell, sd_start=0.0, sd_end=0.0, conic=None):
    R = rows.shape[2]
    c0, cn = conic if conic is not None else (0, R)
    K = orc.solve_rows_robust(rows, xb, grid, c0, cn, ell, 0.0, sd_end)["K"]
    f = rso.sd_forward_rows_robust(rows, grid, c0, cn, ell, K, sd_start, slow=False)
    s = rso.sd_forward_rows_robust(rows, grid, c0, cn, ell, K, sd_start, slow=True)
    return K, f, s


# ==== CPU: the restatement against independent evidence =============================================================
@pytest.mark.parametrize("scale", [0.0, 1.0, 3.0])
def test_oracle_sd_passes_feasible_and_extremal(scale):
    ell = [scale * e for e in ELL]
    n_stages = 0
    for seed in range(3000, 3004):
        grid, rows, xb = _cfg4(seed)
        K, f, s = _sd_passes(rows, xb, grid, ell, 0.0, 0.0)
        assert f["status"] == 0 == s["status"] and f["fail_stage"] == -1
        for p, sign in ((f, +1), (s, -1)):
            x, u = p["x"], p["u"]
            assert np.all(x >= K[:, 0] - 1e-12) and np.all(x <= K[:, 1] + 1e-12)
            for i in range(len(grid) - 1):
                td = 2 * (grid[i + 1] - grid[i])
                a, b, c = rows[i]
                cone = np.ones(len(a), bool)
                nxt = np.array([LD(K[i + 1, 0]) - LD(x[i]) - LD(td) * LD(u[i]),
                                LD(x[i]) + LD(td) * LD(u[i]) - LD(K[i + 1, 1])])
                assert _row_values(a, b, c, cone, ell, u[i], x[i]).max() <= 1e-9 and nxt.max() <= 1e-9
                # one step further on the optimising side (fastest: larger u, slowest: smaller u) leaves the set
                v = u[i] + sign * 1e-9 * (1 + abs(u[i]))
                nxt = np.array([LD(K[i + 1, 0]) - LD(x[i]) - LD(td) * LD(v), LD(x[i]) + LD(td) * LD(v) - LD(K[i + 1, 1])])
                assert max(_row_values(a, b, c, cone, ell, v, x[i]).max(), nxt.max()) > 0, (seed, i, sign)
                n_stages += 1
    assert n_stages == 4 * 2 * 199


def test_oracle_sd_blend_hits_the_desired_duration():
    for seed in range(3000, 3004):
        grid, rows, xb = _cfg4(seed)
        _, f, s = _sd_passes(rows, xb, grid, ELL)
        t_fast, t_slow = _duration(f["x"], grid), _duration(s["x"], grid)
        assert t_fast < t_slow
        desired = np.array([t_fast * 0.9, t_fast + 0.3 * (t_slow - t_fast), t_fast + 0.8 * (t_slow - t_fast),
                            t_slow * 1.1])
        out = cpu_engine.sd_bisect(*(torch.from_numpy(np.tile(v, (4, 1))) for v in (f["x"], f["u"], s["x"], s["u"])),
                                   torch.from_numpy(grid), torch.from_numpy(desired), 1e-5)
        for k, want in enumerate(desired):
            T = _duration(out["sd"][k].numpy() ** 2, grid)
            if t_fast <= want <= t_slow:
                assert abs(T - want) <= 1e-5
            else:
                assert T == pytest.approx(t_fast if want < t_fast else t_slow, rel=1e-12)


def test_oracle_sd_start_and_failures():
    grid, rows, xb = _cfg4(3000)
    K, f, _ = _sd_passes(rows, xb, grid, ELL, sd_start=np.sqrt(K0 := 0.0))
    assert f["status"] == 0 and f["x"][0] == K0
    big = np.sqrt(orc.solve_rows_robust(rows, xb, grid, 0, 28, ELL)["K"][0, 1]) + 1.0
    _, f, s = _sd_passes(rows, xb, grid, ELL, sd_start=big)
    assert f["status"] == 3 == s["status"] and f["fail_stage"] == 0 and np.isnan(f["x"]).all() and np.isnan(f["u"]).all()
    bad = rows.copy()
    bad[:, 2, :] = -1e-4            # c = -amax = -1e-4 > -rc: no stage is feasible
    _, f, _ = _sd_passes(bad, xb, grid, ELL)
    assert f["status"] == 3 and f["fail_stage"] == len(grid) - 2 and np.isnan(f["x"]).all()
    # controllable sets that the rows cannot reach: the forward step at stage 9 has an empty u-interval
    Kb = K.copy()
    Kb[10] = [900.0, 901.0]
    for slow in (False, True):
        o = rso.sd_forward_rows_robust(rows, grid, 0, 28, ELL, Kb, 0.0, slow=slow)
        assert o["status"] == 1 and o["fail_stage"] == 9
        assert not np.isnan(o["x"][:10]).any() and np.isnan(o["x"][10:]).all()
        assert not np.isnan(o["u"][:9]).any() and np.isnan(o["u"][9:]).all()


def test_oracle_stage_vs_slsqp():
    """320 stage problems min g.[u, x] of config-4 paths: the restatement's point is feasible in long double, and on the
    >= 120 that scipy SLSQP (on the smooth cone form) solves to convergence the objectives agree to 1e-9 (1 + |obj|)."""
    from scipy.optimize import minimize
    rng = np.random.RandomState(0)
    done = 0
    for seed in range(3000, 3008):
        grid, rows, xb = _cfg4(seed)
        K = orc.solve_rows_robust(rows, xb, grid, 0, 28, ELL)["K"]
        for i in rng.choice(len(grid) - 1, size=10, replace=False):
            a, b, c = rows[i]
            delta = grid[i + 1] - grid[i]
            lo, hi = max(xb[i, 0], -ECOS_INFTY), min(xb[i, 1], ECOS_MAXX, ECOS_INFTY)
            for g in (np.array([-2 * delta, -1.0]), np.array([2 * delta, 1.0]), rng.randn(2), np.array([1.0, -0.3])):
                z = rso.socp_stage_robust(g, a, b, c, 0, 28, ELL, lo, hi, (delta, K[i + 1, 0], K[i + 1, 1]))
                assert not np.isnan(z).any()
                cone = np.ones(len(a), bool)
                assert _row_values(a, b, c, cone, ELL, z[0], z[1]).max() <= 1e-9
                assert lo - 1e-12 <= z[1] <= hi + 1e-12
                assert K[i + 1, 0] - 1e-9 <= z[1] + 2 * delta * z[0] <= K[i + 1, 1] + 1e-9

                def cons(v):
                    u, x = v
                    nrm = np.sqrt((ELL[0] * u) ** 2 + (ELL[1] * x) ** 2 + ELL[2] ** 2)
                    return np.concatenate((-(a * u + b * x + c + nrm),
                                           [x + 2 * delta * u - K[i + 1, 0], K[i + 1, 1] - x - 2 * delta * u]))
                def jac(v):
                    u, x = v
                    nrm = np.sqrt((ELL[0] * u) ** 2 + (ELL[1] * x) ** 2 + ELL[2] ** 2)
                    J = np.empty((len(a) + 2, 2))
                    J[:-2, 0] = -(a + ELL[0] ** 2 * u / nrm)
                    J[:-2, 1] = -(b + ELL[1] ** 2 * x / nrm)
                    J[-2] = [2 * delta, 1.0]
                    J[-1] = [-2 * delta, -1.0]
                    return J
                x0 = 0.5 * (K[i, 0] + K[i, 1])
                u0 = (0.5 * (K[i + 1, 0] + K[i + 1, 1]) - x0) / (2 * delta)
                res = minimize(lambda v: g.dot(v), [u0, x0], jac=lambda v: g, method="SLSQP",
                               constraints=[{"type": "ineq", "fun": cons, "jac": jac}], bounds=[(None, None), (lo, hi)],
                               options={"ftol": 1e-15, "maxiter": 1000})
                if not res.success or np.min(cons(res.x)) < -1e-10:
                    continue
                ours, theirs = g.dot(z), g.dot(res.x)
                assert abs(ours - theirs) <= 1e-9 * (1 + abs(ours)), (seed, i, g, ours, theirs)
                done += 1
    assert done >= 120


def test_oracle_stage_infeasible_instances():
    """The reference's test_infeasible_instance (tests/tests/solverwrapper/test_basic_can_linear.py:168-197) cases."""
    grid, rows, xb = _cfg4(3000)
    a, b, c = rows[0]
    delta = grid[1] - grid[0]
    g = np.array([0.0, 1.0])
    for xl, xh, xn in ((1.1, 1.0, (delta, -ECOS_INFTY, ECOS_INFTY)), (1.1, 1.0, (delta, 0.0, -0.5)),
                       (max(xb[0, 0], -ECOS_INFTY), min(xb[0, 1], ECOS_MAXX, ECOS_INFTY), (delta, 0.0, -0.5))):
        assert np.isnan(rso.socp_stage_robust(g, a, b, c, 0, 28, ELL, xl, xh, xn)).all()


def test_oracle_zero_ellipsoid_equals_linear():
    """Zero ellipsoid: the TOPPRAsd passes equal the linear Seidel restatement's, and stage problems the LP optimum
    (tb_lp2d / tb_lp1d restated), to 1e-9 relative."""
    rng = np.random.RandomState(1)
    for seed in range(3000, 3004):
        grid, rows, xb = _cfg4(seed)
        K, f, s = _sd_passes(rows, xb, grid, [0.0, 0.0, 0.0])
        w = orc.Wrapper(grid, rows, xb, None)
        KL = w.compute_controllable_sets(0.0, 0.0)
        np.testing.assert_allclose(K, KL, rtol=1e-9, atol=1e-12)
        for p, slow in ((f, False), (s, True)):
            xs = np.zeros(len(grid))
            for i in range(len(grid) - 1):
                delta = grid[i + 1] - grid[i]
                obj = [2 * delta, 1.0] if slow else [-2 * delta, -1.0]
                u = w.solve_stagewise_optim(i, None, obj, xs[i], xs[i], KL[i + 1, 0], KL[i + 1, 1])[0]
                np.testing.assert_allclose(p["u"][i], u, rtol=1e-9, atol=1e-9)
                xs[i + 1] = min(KL[i + 1, 1], max(KL[i + 1, 0], xs[i] + 2 * delta * u - 1e-5))
            np.testing.assert_allclose(p["x"], xs, rtol=1e-9, atol=1e-12)
        for i in rng.choice(len(grid) - 1, size=10, replace=False):
            a, b, c = rows[i]
            delta = grid[i + 1] - grid[i]
            for g in (rng.randn(2), np.array([0.0, -1.0]), np.array([0.0, 1.0])):
                z = rso.socp_stage_robust(g, a, b, c, 0, 28, [0.0, 0.0, 0.0], K[i, 0], K[i, 1],
                                          (delta, K[i + 1, 0], K[i + 1, 1]))
                zl = w.solve_stagewise_optim(i, None, g, K[i, 0], K[i, 1], K[i + 1, 0], K[i + 1, 1])
                assert g.dot(z) == pytest.approx(g.dot(zl), rel=1e-9, abs=1e-12)
                if g[0] == 0.0:
                    assert z[1] == pytest.approx(zl[1], rel=1e-9, abs=1e-12)
            # fixed x (x_min == x_max): the 1-D LP
            x = 0.5 * (K[i, 0] + K[i, 1])
            z = rso.socp_stage_robust([-1.0, 0.0], a, b, c, 0, 28, [0.0, 0.0, 0.0], x, x, (delta, K[i + 1, 0], K[i + 1, 1]))
            zl = w.solve_stagewise_optim(i, None, [-1.0, 0.0], x, x, K[i + 1, 0], K[i + 1, 1])
            np.testing.assert_allclose(z, zl, rtol=1e-9, atol=1e-12)


# ==== CPU: host logic through the engine double ======================================================================
def _scan_robust_double(records, R, conic_row0, conic_rows, ellipsoid, grid, sd_start=None, sd_end=None,
                        backward_only=False, counters=False, feasible_sets=False, glen=None):
    """cpu_engine.scan_robust per path on its own gridpoints (ragged batches: the rest is NaN)."""
    if glen is None:
        return cpu_engine.scan_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, sd_start, sd_end,
                                      backward_only, counters, feasible_sets)
    assert backward_only and not feasible_sets
    B, G, _ = records.shape
    K, st = torch.full((B, G, 2), float("nan"), dtype=torch.float64), torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        n = int(glen[b])
        o = cpu_engine.scan_robust(records[b:b + 1, :n], R, conic_row0, conic_rows, ellipsoid, grid[b, :n], None,
                                   None if sd_end is None else sd_end[b:b + 1], True)
        K[b, :n], st[b] = o["K"][0], o["status"][0]
    return dict(K=K, status=st, fail_stage=torch.full((B,), -1, dtype=torch.int32))


def _sd_forward_robust_double(records, R, conic_row0, conic_rows, ellipsoid, grid, K, status_in, sd_start=None,
                              glen=None):
    """tbr_sd_forward_robust through orc_sd_forward_rows_robust, per path on its own gridpoints."""
    B, G, _ = records.shape
    gr, Kn = grid.numpy(), K.numpy()
    out = {k: np.full((B, G), np.nan) for k in ("x_fast", "x_slow")}
    out.update({k: np.full((B, G - 1), np.nan) for k in ("u_fast", "u_slow")})
    status, fail = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
    for b in range(B):
        n = G if glen is None else int(glen[b])
        rows, _ = cpu_engine._rows_of(records, R, b)
        g = gr if gr.ndim == 1 else gr[b]
        s0 = cpu_engine._scalar(sd_start, b)
        for key, slow in (("fast", False), ("slow", True)):
            o = rso.sd_forward_rows_robust(rows[:n], g[:n], conic_row0, conic_rows, ellipsoid, Kn[b, :n], s0, slow)
            out["x_" + key][b, :n], out["u_" + key][b, :n - 1] = o["x"], o["u"]
            if not slow:
                status[b], fail[b] = o["status"], o["fail_stage"]
        assert int(status_in[b]) == 0 or status[b] == int(status_in[b])
    res = {k: torch.from_numpy(v) for k, v in out.items()}
    res.update(status=torch.from_numpy(status), fail_stage=torch.from_numpy(fail))
    return res


def _sd_bisect_double(x_fast, u_fast, x_slow, u_slow, grid, desired, atol=1e-5, status_in=None, max_iter=200,
                      glen=None):
    """cpu_engine.sd_bisect per path on its own gridpoints (ragged batches: the rest is NaN)."""
    if glen is None:
        return cpu_engine.sd_bisect(x_fast, u_fast, x_slow, u_slow, grid, desired, atol, status_in, max_iter)
    B, G = x_fast.shape
    out = dict(sd=torch.full((B, G), float("nan"), dtype=torch.float64),
               u=torch.full((B, G - 1), float("nan"), dtype=torch.float64),
               info=torch.zeros((B, 4), dtype=torch.float64), status=torch.zeros(B, dtype=torch.int32))
    for b in range(B):
        n = int(glen[b])
        o = cpu_engine.sd_bisect(x_fast[b:b + 1, :n], u_fast[b:b + 1, :n - 1], x_slow[b:b + 1, :n],
                                 u_slow[b:b + 1, :n - 1], grid[b, :n], desired[b:b + 1], atol,
                                 None if status_in is None else status_in[b:b + 1], max_iter)
        out["sd"][b, :n], out["u"][b, :n - 1], out["info"][b], out["status"][b] = (o["sd"][0], o["u"][0], o["info"][0],
                                                                                  o["status"][0])
    return out


def _socp_stage_batch_double(g, a, b, c, conic_row0, conic_rows, ellipsoid, xbox, xnext=None):
    g, a, b, c, xbox = (np.asarray(t, dtype=np.float64) for t in (g, a, b, c, xbox))
    B = g.shape[0]
    return np.stack([rso.socp_stage_robust(g[k], a[k], b[k], c[k], conic_row0, conic_rows, ellipsoid, xbox[k, 0],
                                           xbox[k, 1], None if xnext is None else np.asarray(xnext)[k])
                     for k in range(B)])


@pytest.fixture
def cpu_ta(monkeypatch):
    ta = cpu_engine.install(monkeypatch)
    from toppra_b200 import engine
    monkeypatch.setattr(engine, "scan_robust", _scan_robust_double)
    monkeypatch.setattr(engine, "sd_forward_robust", _sd_forward_robust_double)
    monkeypatch.setattr(engine, "socp_stage_batch", _socp_stage_batch_double)
    monkeypatch.setattr(engine, "sd_bisect", _sd_bisect_double)
    return ta


def _robust_sd_problem(ta, B, seed=3000, scale=1.0):
    ss, way, vlim, alim = make_batch(B, seed)
    path = ta.BatchSplineInterpolator(ss, way)
    acc = ta.constraint.JointAccelerationConstraint(alim)
    cons = [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.RobustLinearConstraint(acc, [scale * e for e in ELL], 1)]
    return ss, way, vlim, alim, path, cons


def _fields(r):
    return [np.asarray(v) for v in (r.K, r.sd, r.sdd, r.status, r.fail_stage, r.alpha, r.duration_fast, r.duration_slow)]


def _single_batch(ta, ss, way_b, vlim_b, alim_b, grid_b, desired, sd_start, scale=1.0):
    path = ta.BatchSplineInterpolator(ss, way_b[None])
    acc = ta.constraint.JointAccelerationConstraint(alim_b[None])
    cons = [ta.constraint.JointVelocityConstraint(vlim_b[None]),
            ta.constraint.RobustLinearConstraint(acc, [scale * e for e in ELL], 1)]
    inst = ta.BatchTOPPRAsd(cons, path, grid_b)
    inst.set_desired_duration(desired)
    return _fields(inst.compute_parameterization(sd_start, 0.0))


def test_host_batch_sd_common_and_chunked_equal_per_path(cpu_ta):
    ta = cpu_ta
    B, G = 5, 40
    ss, way, vlim, alim, path, cons = _robust_sd_problem(ta, B)
    grid = np.linspace(0, 1, G)
    desired = np.array([0.5, 2.0, 3.0, 4.0, 50.0])
    sd_start = np.array([0.0, 0.0, 0.5, 100.0, 0.0])   # path 3: inadmissible start
    whole = ta.BatchTOPPRAsd(cons, path, grid)
    whole.set_desired_duration(desired)
    w = _fields(whole.compute_parameterization(sd_start, 0.0))
    per_path = 8 * ta.engine.record_doubles(whole.R) * G
    chunked = ta.BatchTOPPRAsd(cons, path, grid, max_record_bytes=2 * per_path)
    assert chunked.chunk_size() == 2
    chunked.set_desired_duration(desired)
    c = _fields(chunked.compute_parameterization(sd_start, 0.0))
    for x, y in zip(w, c):
        assert eq(x, y)
    assert w[3][3] == 3 and w[4][3] == 0 and w[3][0] == 0
    for b in range(B):
        one = _single_batch(ta, ss, way[b], vlim[b], alim[b], grid, desired[b], sd_start[b])
        for x, y in zip(w, one):
            assert eq(x[b], y[0])


def test_host_batch_sd_ragged_equals_per_path(cpu_ta):
    ta = cpu_ta
    B = 3
    ss, way, vlim, alim, path, cons = _robust_sd_problem(ta, B, seed=3010)
    inst = ta.BatchTOPPRAsd(cons, path, None, gridpt_min_nb_points=30)
    inst.set_desired_duration(2.5)
    r = _fields(inst.compute_parameterization(0.0, 0.0))
    glen = inst.glen.numpy()
    grid = inst.d_grid.numpy()
    assert len(set(glen.tolist())) > 1 or glen.min() < grid.shape[1]
    for b in range(B):
        n = int(glen[b])
        one = _single_batch(ta, ss, way[b], vlim[b], alim[b], grid[b, :n], 2.5, 0.0)
        assert eq(r[0][b, :n], one[0][0]) and np.isnan(r[0][b, n:]).all()
        assert eq(r[1][b, :n], one[1][0]) and np.isnan(r[1][b, n:]).all()
        assert eq(r[2][b, :n - 1], one[2][0])
        for k in range(3, 8):
            assert eq(r[k][b], one[k][0])


def test_host_single_path_toppra_sd_equals_batch_of_one(cpu_ta):
    ta = cpu_ta
    ss, way, vlim, alim, _, _ = _robust_sd_problem(ta, 1, seed=3003)
    grid = np.linspace(0, 1, 60)
    acc = ta.constraint.JointAccelerationConstraint(alim[0])
    cons = [ta.constraint.JointVelocityConstraint(vlim[0]), ta.constraint.RobustLinearConstraint(acc, ELL, 1)]
    inst = ta.algorithm.TOPPRAsd(cons, ta.SplineInterpolator(ss, way[0]), gridpoints=grid, solver_wrapper="ecos")
    inst.set_desired_duration(3.0)
    sdd, sd, v, K = inst.compute_parameterization(0.0, 0.0, return_data=True)
    one = _single_batch(ta, ss, way[0], vlim[0], alim[0], grid, 3.0, 0.0)
    assert eq(K, one[0][0]) and eq(sd, one[1][0]) and eq(sdd, one[2][0]) and inst.alpha == one[5][0]
    assert inst.problem_data.return_code == ta.algorithm.ParameterizationReturnCode.Ok
    T = _duration(sd ** 2, grid)
    assert abs(T - 3.0) <= 1e-5 or not (one[6][0] <= 3.0 <= one[7][0])


def test_host_solve_stagewise_optim_conic(cpu_ta):
    ta = cpu_ta
    ss, way, vlim, alim, _, _ = _robust_sd_problem(ta, 1, seed=3005)
    grid = np.linspace(0, 1, 30)
    acc = ta.constraint.JointAccelerationConstraint(alim[0])
    cons = [ta.constraint.JointVelocityConstraint(vlim[0]), ta.constraint.RobustLinearConstraint(acc, ELL, 1)]
    inst = ta.algorithm.TOPPRA(cons, ta.SplineInterpolator(ss, way[0]), gridpoints=grid, solver_wrapper="ecos")
    sw = inst.solver_wrapper
    rows = sw.rows()
    R = sw.R
    K = inst.compute_controllable_sets(0.0, 0.0)
    for i in (0, 7, 28, 29):
        a, b, c = (rows[k][i, 2:2 + R] for k in ("a", "b", "c"))
        lo, hi = max(-ECOS_INFTY, rows["low"][i, 1]), min(ECOS_INFTY, ECOS_MAXX, rows["high"][i, 1])
        for g in ([-1.0, 0.0], [0.3, -1.0], [0.0, 1.0]):
            got = sw.solve_stagewise_optim(i, None, np.array(g), np.nan, np.nan, K[min(i + 1, 29), 0],
                                           K[min(i + 1, 29), 1])
            xn = (grid[i + 1] - grid[i], K[i + 1, 0], K[i + 1, 1]) if i < 29 else None
            assert eq(got, rso.socp_stage_robust(g, a, b, c, 0, R, ELL, lo, hi, xn)) and not np.isnan(got).any()
        got = sw.solve_stagewise_optim(i, np.zeros((2, 2)), np.array([0.0, 1.0]), 0.2, 0.3, np.nan, np.nan)
        xn = (grid[i + 1] - grid[i], -ECOS_INFTY, ECOS_INFTY) if i < 29 else None
        assert eq(got, rso.socp_stage_robust([0.0, 1.0], a, b, c, 0, R, ELL, max(0.2, rows["low"][i, 1]),
                                             min(0.3, ECOS_MAXX, rows["high"][i, 1]), xn))
    # the reference's infeasible instances give [nan, nan]
    for args in ((1.1, 1.0, np.nan, np.nan), (1.1, 1.0, 0, -0.5), (np.nan, np.nan, 0, -0.5)):
        assert np.isnan(sw.solve_stagewise_optim(0, None, np.r_[0, 1].astype(float), *args)).all()
    with pytest.raises(AssertionError):
        sw.solve_stagewise_optim(0, np.eye(2), np.r_[0, 1].astype(float), np.nan, np.nan, 0, 1)


# ==== CPU: C-ABI and kernel inventory =================================================================================
def _robust_header():
    text = open(os.path.join(ROOT, "include", "toppra_b200_robust.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(tbr_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        kinds = []
        for arg in [a.strip() for a in args.split(",")]:
            if arg in ("", "void"):
                continue
            kinds.append("ptr" if "*" in arg else ("double" if "double" in arg else "int"))
        out[name] = kinds
    return out


def test_robust_header_matches_prototypes():
    from toppra_b200 import _lib_robust
    declared = _robust_header()
    assert set(declared) == set(_lib_robust._PROTOS)
    for name, (argtypes, restype) in _lib_robust._PROTOS.items():
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name], name
        assert restype is ctypes.c_int


def test_companion_exports_every_declared_symbol():
    if not os.path.exists(ROBUST_LIB):
        pytest.skip("libtoppra_b200_robust.so is not built")
    lib = ctypes.CDLL(ROBUST_LIB)
    for name in _robust_header():
        assert hasattr(lib, name), name
    assert lib.tbr_version() == 100


ROBUST_BUILDS = ["sd_forward_robust_kernel<%d>" % r for r in (1, 2, 3, 4)] + \
                ["socp_stage_kernel<%d>" % r for r in (1, 2, 3, 4)]


def test_companion_kernel_inventory():
    from test_piecewise_poly import kernel_key
    cuobjdump = os.path.join("/usr/local/cuda", "bin", "cuobjdump")
    cuobjdump = cuobjdump if os.path.exists(cuobjdump) else shutil.which("cuobjdump")
    if not os.path.exists(ROBUST_LIB):
        pytest.skip("libtoppra_b200_robust.so is not built")
    if not cuobjdump or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not found")
    text = subprocess.run([cuobjdump, "-res-usage", ROBUST_LIB], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", text, re.M)
    names = subprocess.run([shutil.which("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    assert sorted(kernel_key(n) for n in names) == sorted(ROBUST_BUILDS)


# ==== GPU: kernels against the restatement, bit for bit ===============================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _widened_records(ta, rpl, B, G, seed0=3000, ragged=False):
    """cfg-4 records (28 robust acceleration rows) widened to `rpl` rows per lane: R = 28 rpl rows, the first 28 robust,
    the copies (rows scaled by 1.25^k) linear.  Returns (records [B,G,W] on the device, R, grid [G] or [B,G], glen)."""
    ss, way, vlim, alim = make_batch(B, seed0)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    acc = ta.constraint.JointAccelerationConstraint(alim)
    inst = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.RobustLinearConstraint(acc, ELL, 1)],
                          path, grid)
    base = inst.setup()
    R0 = inst.R
    assert R0 == 28 and inst.conic[:2] == (0, 28)
    R = R0 * rpl
    rec, W = ta.engine.alloc_records(B, G, R, base.device)
    rec.fill_(0.0)
    for k in range(rpl):
        s = 1.25 ** k
        for j in range(3):
            rec[:, :, j * R + k * R0:j * R + (k + 1) * R0] = base[:, :, j * R0:(j + 1) * R0] * s
    rec[:, :, 3 * R:3 * R + 2] = base[:, :, 3 * R0:3 * R0 + 2]
    glen = None
    dgrid = torch.as_tensor(grid, device=rec.device)
    if ragged:
        glen = torch.as_tensor(np.random.RandomState(rpl).randint(G // 2, G + 1, size=B), dtype=torch.int32,
                               device=rec.device)
        dgrid = dgrid.expand(B, G).contiguous()
    return rec, R, dgrid, glen


def _failing_inputs(ta, rec, R, grid, glen):
    """Paths 0 (backward pass fails), 1 (inadmissible start), 2 (empty u-interval at stage 9), 3 (admissible start > 0),
    4 (sd_end = 0.1); the others plain."""
    B, G, _ = rec.shape
    rec[0, :, 2 * R:3 * R] = -1e-4      # c = -1e-4 > -rc: every robust row excludes every u
    sd_end = torch.zeros(B, dtype=torch.float64, device=rec.device)
    sd_end[4] = 0.1
    back = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, None, sd_end, backward_only=True,
                                 **({} if glen is None else {"glen": glen}))
    K = back["K"].clone()
    K[2, 10] = torch.tensor([900.0, 901.0], dtype=torch.float64)
    sd_start = torch.zeros(B, dtype=torch.float64, device=rec.device)
    sd_start[1] = 100.0
    sd_start[3] = 0.5 * float(K[3, 0, 1].sqrt())
    return back, K, sd_start, sd_end


@pytest.mark.gpu
@pytest.mark.parametrize("rpl,ragged", [(1, False), (2, False), (3, False), (4, False), (1, True), (3, True)])
def test_gpu_sd_forward_equals_restatement(ta, rpl, ragged):
    B, G = 16, 60
    rec, R, grid, glen = _widened_records(ta, rpl, B, G, ragged=ragged)
    back, K, sd_start, sd_end = _failing_inputs(ta, rec, R, grid, glen)
    out = ta.engine.sd_forward_robust(rec, R, 0, 28, ELL, grid, K, back["status"], sd_start,
                                      **({} if glen is None else {"glen": glen}))
    h = {k: v.cpu().numpy() for k, v in out.items()}
    Kb, Kh, st_in = back["K"].cpu().numpy(), K.cpu().numpy(), back["status"].cpu().numpy()
    hr, gr = rec.cpu().numpy(), grid.cpu().numpy()
    s0, s1 = sd_start.cpu().numpy(), sd_end.cpu().numpy()
    seen = set()
    for b in range(B):
        n = G if glen is None else int(glen[b])
        rows = hr[b, :n, :3 * R].reshape(n, 3, R)
        g = gr if gr.ndim == 1 else gr[b]
        Ko = orc.solve_rows_robust(rows, hr[b, :n, 3 * R:3 * R + 2], g[:n], 0, 28, ELL, 0.0, s1[b])["K"]
        assert eq(Kb[b, :n], Ko) and np.isnan(Kb[b, n:]).all()
        assert st_in[b] == (3 if np.isnan(Ko).any() else 0)
        for key, slow in (("fast", False), ("slow", True)):
            o = rso.sd_forward_rows_robust(rows, g[:n], 0, 28, ELL, Kh[b, :n], s0[b], slow)
            assert eq(h["x_" + key][b, :n], o["x"]) and eq(h["u_" + key][b, :n - 1], o["u"]), (b, key)
            assert np.isnan(h["x_" + key][b, n:]).all() and np.isnan(h["u_" + key][b, n - 1:]).all()
            if not slow:
                assert h["status"][b] == o["status"] and h["fail_stage"][b] == o["fail_stage"], b
        seen.add(int(h["status"][b]))
    assert list(h["status"][:3]) == [3, 3, 1] and h["fail_stage"][1] == 0 and h["fail_stage"][2] == 9
    assert seen == {0, 1, 3} and h["status"][3] == 0 and h["x_fast"][3, 0] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 2, 3, 4])
def test_gpu_socp_stage_equals_restatement(ta, rpl):
    B, G = 8, 60
    rec, R, grid, _ = _widened_records(ta, rpl, B, G)
    K = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, backward_only=True)["K"].cpu().numpy()
    hr, gr = rec.cpu().numpy(), grid.cpu().numpy()
    rng = np.random.RandomState(rpl)
    P = 96
    g, a, b, c = np.zeros((P, 2)), np.zeros((P, R)), np.zeros((P, R)), np.zeros((P, R))
    xbox, xnext = np.zeros((P, 2)), np.full((P, 3), np.nan)
    for k in range(P):
        p, i = k % B, rng.randint(G - 1)
        a[k], b[k], c[k] = hr[p, i, :R], hr[p, i, R:2 * R], hr[p, i, 2 * R:3 * R]
        delta = gr[i + 1] - gr[i]
        g[k] = [(-2 * delta, -1.0), (2 * delta, 1.0), (0.0, 1.0), (0.0, -1.0), tuple(rng.randn(2))][k % 5]
        xbox[k] = [max(hr[p, i, 3 * R], -ECOS_INFTY), min(hr[p, i, 3 * R + 1], ECOS_MAXX, ECOS_INFTY)]
        if k % 7 == 3:
            xbox[k] = [0.2 * K[p, i, 1], 0.3 * K[p, i, 1]]
        if k % 11 == 5:
            xbox[k] = [1.1, 1.0]                       # the reference's infeasible instances
        if k % 6 != 1:
            xnext[k] = [delta, K[p, i + 1, 0], K[p, i + 1, 1]] if k % 13 != 4 else [delta, 0.0, -0.5]
    z = ta.engine.socp_stage_batch(g, a, b, c, 0, 28, ELL, xbox, xnext)
    n_nan = 0
    for k in range(P):
        o = rso.socp_stage_robust(g[k], a[k], b[k], c[k], 0, 28, ELL, xbox[k, 0], xbox[k, 1], xnext[k])
        assert eq(z[k], o), (k, z[k], o)
        n_nan += int(np.isnan(o).all())
    assert 0 < n_nan < P // 2
    # no x_next rows at all (xnext NULL) equals NaN deltas
    z2 = ta.engine.socp_stage_batch(g[:8], a[:8], b[:8], c[:8], 0, 28, ELL, xbox[:8])
    for k in range(8):
        assert eq(z2[k], rso.socp_stage_robust(g[k], a[k], b[k], c[k], 0, 28, ELL, xbox[k, 0], xbox[k, 1]))


@pytest.mark.gpu
def test_gpu_companion_builds_run(ta):
    from test_piecewise_poly import launched
    names = set()
    for _ in range(3):
        with launched() as got:
            for rpl in (1, 2, 3, 4):
                rec, R, grid, _ = _widened_records(ta, rpl, 2, 12)
                back = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, backward_only=True)
                ta.engine.sd_forward_robust(rec, R, 0, 28, ELL, grid, back["K"], back["status"])
                ta.engine.socp_stage_batch(np.array([[1.0, -1.0]]), rec[0, 3, :R], rec[0, 3, R:2 * R],
                                           rec[0, 3, 2 * R:3 * R], 0, 28, ELL, np.array([[0.0, 10.0]]))
        names |= got
        if set(ROBUST_BUILDS) <= names:   # kineto now and then returns a capture without device activity
            break
    assert set(ROBUST_BUILDS) <= names, sorted(names)


# ==== GPU: the public API ============================================================================================
def _robust_cons(ta, vlim, alim, ell):
    acc = ta.constraint.JointAccelerationConstraint(alim)
    return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.RobustLinearConstraint(acc, ell, 1)]


@pytest.mark.gpu
def test_gpu_zero_ellipsoid_sd_equals_linear(ta):
    from toppra_b200.batch import sd_passes_robust
    B, G = 32, 100
    ss, way, vlim, alim = make_batch(B, 3000)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    vel, acc = ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)
    lin = ta.BatchTOPPRA([vel, acc], path, grid, fused=False)
    rob = ta.BatchTOPPRA(_robust_cons(ta, vlim, alim, [0.0, 0.0, 0.0]), path, grid)
    lin.setup()
    rob.setup()
    fl, sl = (ta.engine.scan(lin.records, lin.R, lin.d_grid, None, None, sd_forward=m) for m in ("fast", "slow"))
    fr, sr = sd_passes_robust(rob.records, rob.R, rob.conic, rob.d_grid, None, None)
    assert not fr["status"].any() and not fl["status"].any()
    for x, y in ((fr["K"], fl["K"]), (fr["sd"], fl["sd"]), (sr["sd"], sl["sd"]), (fr["u"], fl["u"]), (sr["u"], sl["u"])):
        np.testing.assert_allclose(x.cpu().numpy(), y.cpu().numpy(), rtol=1e-9, atol=1e-9)
    res = []
    for cons in ([vel, acc], _robust_cons(ta, vlim, alim, [0.0, 0.0, 0.0])):
        inst = ta.BatchTOPPRAsd(cons, path, grid)
        inst.set_desired_duration(1.0)
        r = inst.compute_parameterization(0.0, 0.0)
        t_fast, t_slow = r.duration_fast.cpu().numpy(), r.duration_slow.cpu().numpy()
        want = 1.5 * t_fast
        inst.set_desired_duration(want)
        r = inst.compute_parameterization(0.0, 0.0)
        sd = r.sd.cpu().numpy()
        for b in range(B):
            assert abs(_duration(sd[b] ** 2, grid) - want[b]) <= 1e-5
        res.append((t_fast, t_slow))
    np.testing.assert_allclose(res[1][0], res[0][0], rtol=1e-9)
    # the slowest passes rest at x = 0 over most stages, where 2 delta / (sqrt(x_i) + sqrt(x_i+1) + 1e-9) turns x
    # differences of 1e-18 into O(1) relative changes of the duration: they are compared on x above
    assert np.all(res[1][1] > 1e8) and np.all(res[0][1] > 1e8)


@pytest.mark.gpu
def test_gpu_robust_fastest_durations_grow_with_the_ellipsoid(ta):
    B, G = 32, 100
    ss, way, vlim, alim = make_batch(B, 3000)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    lin = ta.BatchTOPPRAsd([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                           path, grid)
    lin.set_desired_duration(0.0)
    prev = lin.compute_parameterization().duration_fast.cpu().numpy()
    for scale in (0.5, 1.0, 2.0, 4.0):
        inst = ta.BatchTOPPRAsd(_robust_cons(ta, vlim, alim, [scale * e for e in ELL]), path, grid)
        inst.set_desired_duration(0.0)
        r = inst.compute_parameterization()
        assert not r.status.any()
        t = r.duration_fast.cpu().numpy()
        assert np.all(t >= prev * (1 - 1e-12)) and np.any(t > prev)
        prev = t


def _host(r):
    return [v.cpu().numpy() for v in (r.K, r.sd, r.sdd, r.status, r.fail_stage, r.alpha, r.duration_fast,
                                       r.duration_slow)]


@pytest.mark.gpu
def test_gpu_batch_sd_common_chunked_and_single_path(ta):
    B, G = 12, 80
    ss, way, vlim, alim = make_batch(B, 3020)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    cons = _robust_cons(ta, vlim, alim, ELL)
    desired = np.linspace(0.5, 6.0, B)
    sd_start = np.zeros(B)
    sd_start[5] = 100.0
    whole = ta.BatchTOPPRAsd(cons, path, grid)
    whole.set_desired_duration(desired)
    w = _host(whole.compute_parameterization(sd_start, 0.0))
    per_path = 8 * ta.engine.record_doubles(whole.R) * G
    chunked = ta.BatchTOPPRAsd(cons, path, grid, max_record_bytes=5 * per_path)
    chunked.set_desired_duration(desired)
    for x, y in zip(w, _host(chunked.compute_parameterization(sd_start, 0.0))):
        assert eq(x, y)
    assert w[3][5] == 3 and w[4][5] == 0 and (w[3] == 0).sum() == B - 1
    # the blend hits achievable durations; the passes are the restatement's
    rec = whole.records.cpu().numpy()
    R = whole.R
    for b in range(B):
        if b == 5:
            continue
        rows = rec[b, :, :3 * R].reshape(G, 3, R)
        _, f, s = _sd_passes(rows, rec[b, :, 3 * R:3 * R + 2], grid, ELL, conic=(0, R))
        assert w[6][b] == pytest.approx(_duration(f["x"], grid), rel=1e-12)
        assert w[7][b] == pytest.approx(_duration(s["x"], grid), rel=1e-12)
        if w[6][b] <= desired[b] <= w[7][b]:
            assert abs(_duration(w[1][b] ** 2, grid) - desired[b]) <= 1e-5
    # single-path TOPPRAsd (solver_wrapper="ecos" maps to this library) == the batch's row
    for b in (0, 7):
        acc = ta.constraint.JointAccelerationConstraint(alim[b])
        one = ta.algorithm.TOPPRAsd([ta.constraint.JointVelocityConstraint(vlim[b]),
                                     ta.constraint.RobustLinearConstraint(acc, ELL, 1)],
                                    ta.SplineInterpolator(ss, way[b]), gridpoints=grid, solver_wrapper="ecos")
        one.set_desired_duration(desired[b])
        sdd, sd, _, K = one.compute_parameterization(0.0, 0.0, return_data=True)
        assert eq(K, w[0][b]) and eq(sd, w[1][b]) and eq(sdd, w[2][b]) and one.alpha == w[5][b]


@pytest.mark.gpu
def test_gpu_batch_sd_ragged_equals_per_path(ta):
    B = 6
    ss, way, vlim, alim = make_batch(B, 3030)
    path = ta.BatchSplineInterpolator(ss, way)
    inst = ta.BatchTOPPRAsd(_robust_cons(ta, vlim, alim, ELL), path, None)
    inst.set_desired_duration(3.0)
    r = _host(inst.compute_parameterization(0.0, 0.0))
    glen, grid = inst.glen.cpu().numpy(), inst.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for b in range(B):
        n = int(glen[b])
        one = ta.BatchTOPPRAsd(_robust_cons(ta, vlim[b:b + 1], alim[b:b + 1], ELL),
                               ta.BatchSplineInterpolator(ss, way[b:b + 1]), grid[b, :n])
        one.set_desired_duration(3.0)
        o = _host(one.compute_parameterization(0.0, 0.0))
        assert eq(r[0][b, :n], o[0][0]) and np.isnan(r[0][b, n:]).all()
        assert eq(r[1][b, :n], o[1][0]) and eq(r[2][b, :n - 1], o[2][0])
        for k in range(3, 8):
            assert eq(r[k][b], o[k][0])


@pytest.mark.gpu
def test_gpu_solve_stagewise_optim_conic(ta):
    ss, way, vlim, alim = make_batch(1, 3005)
    grid = np.linspace(0, 1, 30)
    acc = ta.constraint.JointAccelerationConstraint(alim[0])
    cons = [ta.constraint.JointVelocityConstraint(vlim[0]), ta.constraint.RobustLinearConstraint(acc, ELL, 1)]
    inst = ta.algorithm.TOPPRA(cons, ta.SplineInterpolator(ss, way[0]), gridpoints=grid, solver_wrapper="ecos")
    sw = inst.solver_wrapper
    rows, R = sw.rows(), sw.R
    K = inst.compute_controllable_sets(0.0, 0.0)
    for i in (0, 11, 29):
        a, b, c = (rows[k][i, 2:2 + R] for k in ("a", "b", "c"))
        lo, hi = max(-ECOS_INFTY, rows["low"][i, 1]), min(ECOS_INFTY, ECOS_MAXX, rows["high"][i, 1])
        for g in ([-1.0, 0.0], [0.3, -1.0], [0.0, 1.0], [0.0, -1.0]):
            j = min(i + 1, 29)
            got = sw.solve_stagewise_optim(i, None, np.array(g), np.nan, np.nan, K[j, 0], K[j, 1])
            xn = (grid[i + 1] - grid[i], K[i + 1, 0], K[i + 1, 1]) if i < 29 else None
            assert eq(got, rso.socp_stage_robust(g, a, b, c, 0, R, ELL, lo, hi, xn)) and not np.isnan(got).any()
    for args in ((1.1, 1.0, np.nan, np.nan), (1.1, 1.0, 0, -0.5), (np.nan, np.nan, 0, -0.5)):
        assert np.isnan(sw.solve_stagewise_optim(0, None, np.r_[0, 1].astype(float), *args)).all()
