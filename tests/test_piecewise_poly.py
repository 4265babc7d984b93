"""Piecewise-polynomial paths of order k <= 8 (PiecewisePolyPath, BatchPiecewisePolyPath, libtoppra_b200_poly.so).

GPU: evaluation against scipy's PPoly and its chained derivative objects; the sampled record builder against K1 on
cubic paths; the single-path API against the unmodified reference (tests/golden/poly_paths_k*.npz, made by
tests/golden/make_golden_poly.py); batched solves against single-path solves and the oracle-backed scan; every
companion kernel build launched under torch.profiler.  Exact comparisons are bit for bit, NaN equal to NaN.
CPU: the companion's C-ABI and kernel inventory, the engine's dispatch on a recording library, and the fixtures'
evaluation convention."""
import contextlib
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy.interpolate import PPoly

import cpu_engine
from conftest import load_golden
from problems import make_batch
from toppra_b200 import _lib, _lib_poly, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLY_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_poly.so")
GOLDEN = ["poly_paths_k5", "poly_paths_k6", "poly_paths_k7", "poly_paths_k8"]
TRAJ_TOL = 1e-9   # compute_trajectory evaluations (spline re-fit / time stamps), as the cubic trajectory tests


def eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def scipy_derivs(c, x):
    p = PPoly(c, x)
    d1 = p.derivative()
    return p, d1, d1.derivative()


def golden_paths(name):
    g = load_golden(name)
    labels = sorted({k.split("/")[0] for k in g})
    return g, labels


# ---- kernel names (as tests/test_kernel_builds.py) ------------------------------------------------------------------
def kernel_key(name):
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    s = s.replace("(anonymous namespace)::", "")
    s = re.sub(r"^(\w+::)+", "", s)
    m = re.match(r"([A-Za-z_]\w*)(<[^<>]*>)?", s)
    return (m.group(1) + (m.group(2) or "")).replace(" ", "") if m else s


@contextlib.contextmanager
def launched():
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    names = set()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield names
        torch.cuda.synchronize()
    names.update(kernel_key(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA)


# ---- inputs ---------------------------------------------------------------------------------------------------------
def random_pieces(B, k, nseg, dof, seed, shared_breaks=True):
    rng = np.random.RandomState(seed)
    def breaks():
        x = np.concatenate(([0.0], np.cumsum(0.5 + rng.rand(nseg))))
        return x / x[-1]
    x = breaks() if shared_breaks else np.stack([breaks() for _ in range(B)])
    scale = 2.0 ** -np.arange(k)[::-1]
    c = rng.randn(B, k, nseg, dof) * scale[None, :, None, None] * 3.0
    c[:, :, 0, 0] = -0.0     # signed zeros must survive the evaluation
    return x, c


def sample_positions(x):
    return np.concatenate((x, 0.5 * (x[1:] + x[:-1]), np.linspace(x[0], x[-1], 17), [x[0] - 0.25, x[-1] + 0.5, np.nan]))


def velacc(vlim, alim, scheme=1):
    import toppra_b200 as ta
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)]


# ==== GPU ===========================================================================================================
# 1. evaluation against scipy
@pytest.mark.gpu
@pytest.mark.parametrize("k", [5, 6, 7, 8])
@pytest.mark.parametrize("shared", [True, False])
def test_eval_equals_scipy_derivative_objects(k, shared):
    B, dof = 3, 4
    x, c = random_pieces(B, k, 5, dof, 10 * k + shared, shared)
    dev = torch.device("cuda")
    d_c, d_x = engine.as_device(c, dev), engine.as_device(x, dev)
    s = np.stack([sample_positions(x if shared else x[b]) for b in range(B)])
    for order in (0, 1, 2):
        got = engine.ppoly_eval(d_c, d_x, engine.as_device(s, dev), order).cpu().numpy()
        for b in range(B):
            want = scipy_derivs(c[b], x if shared else x[b])[order](s[b])
            assert eq(got[b], want), (k, order, b)
            assert eq(np.signbit(got[b]), np.signbit(want)), "signed zeros differ"
    # shared positions too
    s1 = sample_positions(x if shared else x[0])
    got = engine.ppoly_eval(d_c, d_x, engine.as_device(s1, dev), 2).cpu().numpy()
    assert eq(got[0], scipy_derivs(c[0], x if shared else x[0])[2](s1))


# 2. the sampled row builder against K1 on cubic paths
def _cubic_batch(B, G, per_path_grid):
    import toppra_b200 as ta
    ss, way, vlim, alim = make_batch(B, 3000)
    path = ta.BatchSplineInterpolator(ss, way, device="cuda")
    rng = np.random.RandomState(4)
    if per_path_grid:
        grid = np.stack([np.concatenate(([0.0], np.sort(rng.rand(G - 2)), [1.0])) for _ in range(B)])
    else:
        grid = np.linspace(0, 1, G)
    return path, engine.as_device(grid, path.device), vlim, alim


def _rows_pair(path, grid, vlim, alim, interp, R_total, row0, mode, ubound):
    B, G = path.B, grid.shape[-1]
    records, _ = engine.alloc_records(B, G, R_total, path.device, ubound=ubound)
    records.copy_(torch.randn(records.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(7)).cuda())
    k1 = records.clone()
    engine.coeff_velacc(path.d_ppoly, path.d_ss, grid, vlim, alim, interp, k1, R_total, row0, mode)
    qd = engine.ppoly_eval(path.d_ppoly, path.d_ss, grid, 1)
    qdd = engine.ppoly_eval(path.d_ppoly, path.d_ss, grid, 2)
    smp = records.clone()
    engine.rows_velacc_sampled(qd, qdd, grid, vlim, alim, interp, smp, R_total, row0, mode)
    return k1.cpu().numpy(), smp.cpu().numpy()


ROW_CASES = [  # (interp, per-path limits, per-path grid, vel, acc, row0 extra, ubound, write_xbound)
    (1, False, False, True, True, 0, False, 1), (0, False, False, True, True, 0, False, 1),
    (1, True, True, True, True, 0, False, 1), (1, False, False, True, True, 0, False, 0),
    (1, False, False, True, False, 0, False, 2), (1, False, False, True, False, 0, False, 3),
    (0, True, False, True, True, 5, False, 3), (1, False, True, False, True, 3, True, 1),
    (1, True, False, True, True, 0, True, 2), (0, False, False, False, True, 0, False, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ROW_CASES, ids=["-".join(map(str, c)) for c in ROW_CASES])
def test_sampled_rows_equal_k1_on_cubic_paths(case):
    interp, per_lim, per_grid, use_v, use_a, extra, ubound, mode = case
    B, G, dof = 6, 77, 7
    path, grid, vlim, alim = _cubic_batch(B, G, per_grid)
    dev = path.device
    vl = engine.as_device(vlim if per_lim else vlim[0], dev) if use_v else None
    al = engine.as_device(alim if per_lim else alim[0], dev) if use_a else None
    racc = (4 if interp else 2) * dof if use_a else 0
    R_total = racc + extra + (2 if extra else 0)
    k1, smp = _rows_pair(path, grid, vl, al, interp, R_total, extra, mode, ubound)
    assert eq(smp, k1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("shared", [True, False])
def test_sampled_varying_bound_equals_tb_xbound_varying(mode, shared):
    B, G = 5, 64
    path, grid, vlim, _ = _cubic_batch(B, G, False)
    rng = np.random.RandomState(mode)
    vg = np.abs(rng.randn(*((G, 7, 2) if shared else (B, G, 7, 2)))) + 0.5
    vg[..., 0] *= -1
    vg = engine.as_device(vg, path.device)
    R = 4
    records, _ = engine.alloc_records(B, G, R, path.device)
    records.copy_(torch.randn(records.shape, dtype=torch.float64).cuda())
    a, b = records.clone(), records.clone()
    engine.xbound_varying(path.d_ppoly, path.d_ss, grid, vg, a, R, mode)
    engine.xbound_varying_sampled(engine.ppoly_eval(path.d_ppoly, path.d_ss, grid, 1), vg, b, R, mode)
    assert eq(a.cpu().numpy(), b.cpu().numpy())


# 3. the single-path API against the reference
def _golden_cases(g, label):
    return sorted({k.split("/")[1] for k in g if k.startswith(label + "/") and "/" in k[len(label) + 1:]
                   and k.split("/")[1] not in ("path", "sets", "params") and not k.split("/")[1].startswith(("traj_", "sd_"))})


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN)
def test_single_path_api_equals_reference(name):
    import toppra_b200 as ta
    g, labels = golden_paths(name)
    for label in labels:
        P = lambda key: g["%s/%s" % (label, key)]  # noqa: E731
        path = ta.PiecewisePolyPath(P("path/c"), P("path/x"))
        assert path.order == P("path/c").shape[0]
        s = P("path/s")
        for order in (0, 1, 2):
            assert eq(path(s, order), P("path/q%d" % order)), (label, order)
        for case in _golden_cases(g, label):
            C = lambda key: g["%s/%s/%s" % (label, case, key)]  # noqa: E731
            cons = velacc(C("vlim"), C("alim"), int(C("scheme")))
            grid = None if case == "proposed_grid" else C("grid")
            inst = ta.algorithm.TOPPRA(cons, path, gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = inst.compute_parameterization(float(C("sd_start")), float(C("sd_end")), return_data=True)
            assert inst.problem_data.return_code.name == str(C("status")), (label, case)
            assert eq(inst.gridpoints, C("grid")), (label, case)
            assert eq(K, C("K")), (label, case)
            if sd is not None:
                assert eq(sd, C("sd")) and eq(sdd, C("sdd")), (label, case)
            else:
                assert np.isnan(C("sd")).all()
        cons = velacc(P("uniform_interp/vlim"), P("uniform_interp/alim"), 1)
        uni = P("uniform_interp/grid")
        inst = ta.algorithm.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel")
        assert eq(inst.compute_feasible_sets(), P("sets/X"))
        inst = ta.algorithm.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel")
        assert eq(np.asarray(inst.compute_reachable_sets(0.0, 0.0)), P("sets/L"))
        assert eq(cons[0].compute_constraint_params(path, uni)[6], P("params/vel_xbound"))
        prm = cons[1].compute_constraint_params(path, uni)
        for i, key in enumerate(("acc_a", "acc_b", "acc_c", "acc_F", "acc_g")):
            assert eq(prm[i], P("params/" + key)), key
        for pname in ("ParametrizeSpline", "ParametrizeConstAccel"):
            inst_p = ta.algorithm.TOPPRA(cons, path, gridpoints=uni, solver_wrapper="seidel", parametrizer=pname)
            traj = inst_p.compute_trajectory(0, 0)
            T = lambda key: g["%s/traj_%s/%s" % (label, pname, key)]  # noqa: E731
            assert abs(traj.duration - float(T("duration"))) <= TRAJ_TOL
            for order in (0, 1, 2):
                np.testing.assert_allclose(traj(T("ts"), order), T("q%d" % order), rtol=TRAJ_TOL, atol=TRAJ_TOL)
        for which in ("below", "inside", "above"):
            S = lambda key: g["%s/sd_%s/%s" % (label, which, key)]  # noqa: E731
            sd_inst = ta.algorithm.TOPPRAsd(cons, path, gridpoints=uni, solver_wrapper="seidel")
            sd_inst.set_desired_duration(float(S("desired")))
            sdd, sd, _, _ = sd_inst.compute_parameterization(0, 0, return_data=True)
            assert eq(sd, S("sd")) and eq(sdd, S("sdd")), which


# 4. batched solves
def _quintic_batch(B, seed, k=6, nseg=4, shared=True):
    x, c = random_pieces(B, k, nseg, 7, seed, shared)
    rng = np.random.RandomState(seed + 1)
    vl = 10 + rng.rand(B, 7) * 20
    al = 10 + rng.rand(B, 7) * 2
    return x, c, np.stack((-vl, vl), -1), np.stack((-al, al), -1)


def _single(c, x, vlim, alim, grid):
    import toppra_b200 as ta
    inst = ta.algorithm.TOPPRA(velacc(vlim, alim), ta.PiecewisePolyPath(c, x), gridpoints=grid, solver_wrapper="seidel")
    sdd, sd, _, K = inst.compute_parameterization(0.0, 0.0, return_data=True)
    return inst, K, sd, sdd


@pytest.mark.gpu
def test_batch_equals_single_path_and_oracle_scan():
    import toppra_b200 as ta
    B, G = 512, 200
    x, c, vlim, alim = _quintic_batch(B, 500)
    grid = np.linspace(0, 1, G)
    path = ta.BatchPiecewisePolyPath(x, c)
    inst = ta.BatchTOPPRA(velacc(vlim, alim), path, grid)
    assert not inst.fused
    res = inst.compute_parameterization(0.0, 0.0).to_host()
    assert (res["status"] == 0).sum() > B // 2
    recs = inst.records.cpu()
    want = cpu_engine.scan(recs, inst.R, torch.from_numpy(grid))
    for key, wkey in (("K", "K"), ("sd", "sd"), ("sdd", "u"), ("status", "status")):
        assert eq(res[key], want[wkey].numpy()), key
    for b in range(0, B, 37):
        _, K, sd, sdd = _single(c[b], x, vlim[b], alim[b], grid)
        assert eq(res["K"][b], K)
        if sd is not None:
            assert eq(res["sd"][b], sd) and eq(res["sdd"][b], sdd)
    # chunked records, solve_to_host(sync=False), exact=False
    chunked = ta.BatchTOPPRA(velacc(vlim, alim), path, grid, max_record_bytes=8 * engine.record_doubles(inst.R) * G * 100)
    assert chunked.chunk_size() < B
    h = chunked.compute_parameterization(0.0, 0.0).to_host()
    for key in ("K", "sd", "sdd", "status"):
        assert eq(h[key], res[key]), key
    pinned = inst.solve_to_host(0.0, 0.0, sync=False)
    inst.host_ready.synchronize()
    for key in ("K", "sd", "sdd", "status"):
        assert eq(pinned[key].numpy(), res[key]), key
    fast = ta.BatchTOPPRA(velacc(vlim, alim), path, grid, exact=False).compute_parameterization(0.0, 0.0).to_host()
    ok = res["status"] == 0
    assert eq(fast["status"], res["status"])
    assert np.nanmax(np.abs(fast["K"][ok] - res["K"][ok])) <= 1e-15
    assert np.nanmax(np.abs(fast["sd"][ok] - res["sd"][ok])) <= 1e-15


@pytest.mark.gpu
@pytest.mark.parametrize("k", [7, 8])
def test_batch_higher_orders_per_path_breaks_and_limits(k):
    import toppra_b200 as ta
    B, G = 8, 120
    x, c, vlim, alim = _quintic_batch(B, 700 + k, k=k, nseg=5, shared=False)
    grid = np.stack([np.linspace(x[b, 0], x[b, -1], G) for b in range(B)])
    res = ta.BatchTOPPRA(velacc(vlim, alim), ta.BatchPiecewisePolyPath(x, c), grid).compute_parameterization().to_host()
    for b in range(B):
        _, K, sd, sdd = _single(c[b], x[b], vlim[b], alim[b], grid[b])
        assert eq(res["K"][b], K)
        if sd is not None:
            assert eq(res["sd"][b], sd) and eq(res["sdd"][b], sdd)


@pytest.mark.gpu
def test_batch_proposed_ragged_grids_equal_single_path():
    import toppra_b200 as ta
    B = 6
    x, c, vlim, alim = _quintic_batch(B, 900)
    path = ta.BatchPiecewisePolyPath(x, c)
    grid, glen = path.propose_gridpoints(max_err_threshold=1e-3)
    res = ta.BatchTOPPRA(velacc(vlim, alim), path, grid, glen=glen).compute_parameterization().to_host()
    glen = glen.cpu().numpy()
    for b in range(B):
        inst, K, sd, sdd = _single(c[b], x, vlim[b], alim[b], None)
        n = int(glen[b])
        assert eq(grid[b, :n].cpu().numpy(), inst.gridpoints)
        assert eq(res["K"][b, :n], K)
        if sd is not None:
            assert eq(res["sd"][b, :n], sd) and eq(res["sdd"][b, :n - 1], sdd)


@pytest.mark.gpu
def test_batch_sets_robust_and_cubic_equivalence():
    import toppra_b200 as ta
    B, G = 4, 60
    x, c, vlim, alim = _quintic_batch(B, 1100)
    grid = np.linspace(0, 1, G)
    path = ta.BatchPiecewisePolyPath(x, c)
    inst = ta.BatchTOPPRA(velacc(vlim, alim), path, grid)
    X = inst.compute_feasible_sets().cpu().numpy()
    L, _, _ = inst.compute_reachable_sets(0.0, 0.0)
    for b in range(B):
        single = ta.algorithm.TOPPRA(velacc(vlim[b], alim[b]), ta.PiecewisePolyPath(c[b], x), gridpoints=grid)
        assert eq(X[b], single.compute_feasible_sets())
        assert eq(L[b].cpu().numpy(), np.asarray(single.compute_reachable_sets(0.0, 0.0)))
    acc = ta.constraint.JointAccelerationConstraint(alim[0])
    robust = ta.constraint.RobustLinearConstraint(acc, [1e-3, 1e-3, 1e-3])
    rb = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim[0]), robust], path, grid)
    out = rb.compute_parameterization().to_host()
    ok = out["status"] == 0
    assert ok.any()
    K = out["K"][ok]
    assert (K[..., 0] <= K[..., 1]).all() and (K[..., 0] >= 0).all()
    assert (out["sd"][ok] ** 2 <= K[..., 1] * (1 + 1e-9) + 1e-12).all()
    # k <= 4 through BatchPiecewisePolyPath is from_ppoly, bit for bit
    xc, cc = random_pieces(B, 3, 4, 7, 5)
    a = ta.BatchPiecewisePolyPath(xc, cc)
    b = ta.BatchSplineInterpolator.from_ppoly(xc, cc)
    assert eq(a.d_ppoly.cpu().numpy(), b.d_ppoly.cpu().numpy()) and a.order == 3
    ra = ta.BatchTOPPRA(velacc(vlim, alim), a, grid).compute_parameterization().to_host()
    rb_ = ta.BatchTOPPRA(velacc(vlim, alim), b, grid).compute_parameterization().to_host()
    for key in ("K", "sd", "sdd", "status"):
        assert eq(ra[key], rb_[key]), key


# 5. every companion build ran
def _case_eval():
    x, c = random_pieces(2, 7, 4, 3, 1)
    d = torch.device("cuda")
    s = sample_positions(x)
    with launched() as names:
        got = engine.ppoly_eval(engine.as_device(c, d), engine.as_device(x, d), engine.as_device(s, d), 2).cpu().numpy()
    assert eq(got[1], scipy_derivs(c[1], x)[2](s))
    return names


def _case_rows():
    path, grid, vlim, alim = _cubic_batch(3, 40, False)
    x, c, vl, al = _quintic_batch(3, 5)
    p6 = engine.as_device(c, path.device)
    b6 = engine.as_device(x, path.device)
    records, _ = engine.alloc_records(3, 40, 28, path.device)
    with launched() as names:
        engine.coeff_velacc(p6, b6, grid, engine.as_device(vl, path.device), engine.as_device(al, path.device), True,
                            records, 28, 0, 1)
    want = torch.empty_like(records)
    qd, qdd = engine.ppoly_eval(p6, b6, grid, 1), engine.ppoly_eval(p6, b6, grid, 2)
    engine.rows_velacc_sampled(qd, qdd, grid, engine.as_device(vl, path.device), engine.as_device(al, path.device), True,
                               want, 28, 0, 1)
    assert eq(records.cpu().numpy(), want.cpu().numpy())
    assert "coeff_velacc_kernel" not in names
    return names


def _case_varying():
    import toppra_b200 as ta
    x, c, vlim, alim = _quintic_batch(1, 6)
    grid = np.linspace(0, 1, 30)
    path = ta.PiecewisePolyPath(c[0], x)
    cons = ta.constraint.JointVelocityConstraintVarying(lambda s: vlim[0] * (1 + s))
    with launched() as names:
        xb = cons.compute_constraint_params(path, grid)[6]
    qd = scipy_derivs(c[0], x)[1](grid)
    for i, s in enumerate(grid):
        v = vlim[0] * (1 + s)
        hi = np.float32(1e8)
        lo = np.float32(-1e8)
        for j in range(7):
            q = qd[i, j]
            if q > 0:
                hi, lo = np.float32(min(v[j, 1] / q, float(hi))), np.float32(max(v[j, 0] / q, float(lo)))
            elif q < 0:
                hi, lo = np.float32(min(v[j, 0] / q, float(hi))), np.float32(max(v[j, 1] / q, float(lo)))
        assert xb[i, 1] == float(np.float32(hi * hi)) and xb[i, 0] == max(float(lo), 0.0) ** 2
    return names


def _case_propose():
    import toppra_b200 as ta
    x, c, _, _ = _quintic_batch(2, 8, k=8)
    path = ta.BatchPiecewisePolyPath(x, c)
    with launched() as names:
        grid, glen = path.propose_gridpoints(max_err_threshold=1e-3)
    # the reference's rule on the returned grid: every segment is short and its error estimate small
    for b in range(2):
        g = grid[b, :int(glen[b])].cpu().numpy()
        assert g[0] == x[0] and g[-1] == x[-1] and (np.diff(g) > 0).all() and len(g) >= 100
    return names


def _case_constaccel():
    import toppra_b200 as ta
    x, c, vlim, alim = _quintic_batch(1, 9)
    grid = np.linspace(0, 1, 50)
    inst = ta.algorithm.TOPPRA(velacc(vlim[0], alim[0]), ta.PiecewisePolyPath(c[0], x), gridpoints=grid,
                               parametrizer="ParametrizeConstAccel")
    traj = inst.compute_trajectory(0, 0)
    ts = np.linspace(0, traj.duration, 31)
    with launched() as names:
        q1 = traj(ts, 1)
    sd = inst.problem_data.sd_vec
    # parametrizer.py:101-129 restated on the host with scipy's derivative objects
    t_grid = np.concatenate(([0.0], np.cumsum(2 * np.diff(grid) / (sd[:-1] + sd[1:]))))
    us = 0.5 * (sd[1:] ** 2 - sd[:-1] ** 2) / np.diff(grid)
    idx = np.minimum(np.searchsorted(t_grid, ts, side="right") - 1, len(us) - 1)
    dt = ts - t_grid[idx]
    v = sd[idx] + dt * us[idx]
    s = grid[idx] + dt * sd[idx] + 0.5 * dt ** 2 * us[idx]
    np.testing.assert_allclose(q1, scipy_derivs(c[0], x)[1](s) * v[:, None], rtol=1e-12, atol=1e-12)
    return names


POLY_BUILDS = [("poly_eval_kernel", _case_eval), ("rows_velacc_sampled_kernel", _case_rows),
               ("xbound_varying_sampled_kernel", _case_varying), ("propose_gridpoints_poly_kernel", _case_propose),
               ("constaccel_eval_poly_kernel", _case_constaccel)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,case", POLY_BUILDS, ids=[r[0] for r in POLY_BUILDS])
def test_companion_build_runs(name, case):
    for _ in range(3):
        names = case()
        if names:   # kineto now and then returns a capture without device activity; the cases are deterministic
            break
    assert name in names, "%s was not launched; launched: %s" % (name, sorted(names))


# 6. errors
@pytest.mark.gpu
def test_errors():
    import toppra_b200 as ta
    x, c = random_pieces(2, 9, 3, 2, 1)
    with pytest.raises(ValueError):
        ta.BatchPiecewisePolyPath(x, c)
    with pytest.raises(ValueError):
        ta.BatchPiecewisePolyPath(x, c[0, :6])
    with pytest.raises(ValueError):
        ta.BatchPiecewisePolyPath(x[:-1], c[:, :6])
    with pytest.raises(ValueError):
        ta.BatchPiecewisePolyPath(x[::-1].copy(), c[:, :6])
    with pytest.raises(ValueError):
        ta.PiecewisePolyPath(c[0, :6].reshape(6, -1)[:, :0], x)
    xq, cq, vlim, alim = _quintic_batch(2, 3)
    path = ta.BatchPiecewisePolyPath(xq, cq)
    with pytest.raises(ValueError, match="piecewise-cubic"):
        ta.BatchTOPPRA(velacc(vlim, alim), path, np.linspace(0, 1, 20), fused=True)
    tq = ta.constraint.SecondOrderConstraint.joint_torque_constraint(None, np.ones((7, 2)) * [-50, 50], np.zeros(7),
                                                    device_model=("pendulums", np.ones(14)))
    with pytest.raises(NotImplementedError, match="order 6"):
        ta.BatchTOPPRA([tq], path, np.linspace(0, 1, 20)).compute_parameterization()


# ==== CPU ===========================================================================================================
def _poly_header():
    text = open(os.path.join(ROOT, "include", "toppra_b200_poly.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(tbp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        kinds = []
        for arg in [a.strip() for a in args.split(",")]:
            if arg in ("", "void"):
                continue
            kinds.append("ptr" if "*" in arg else ("double" if "double" in arg else "int"))
        out[name] = kinds
    return out


def _kind(t):
    return {ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr")


def test_poly_header_matches_prototypes():
    declared = _poly_header()
    assert set(declared) == set(_lib_poly._PROTOS)
    for name, (argtypes, restype) in _lib_poly._PROTOS.items():
        assert [_kind(t) for t in argtypes] == declared[name], name
        assert restype is ctypes.c_int


def test_companion_exports_every_declared_symbol():
    if not os.path.exists(POLY_LIB):
        pytest.skip("libtoppra_b200_poly.so is not built")
    lib = ctypes.CDLL(POLY_LIB)
    for name in _poly_header():
        assert hasattr(lib, name), name
    assert lib.tbp_version() == 100


def test_companion_kernel_inventory():
    cuobjdump = os.path.join("/usr/local/cuda", "bin", "cuobjdump")
    cuobjdump = cuobjdump if os.path.exists(cuobjdump) else shutil.which("cuobjdump")
    if not os.path.exists(POLY_LIB):
        pytest.skip("libtoppra_b200_poly.so is not built")
    if not cuobjdump or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not found")
    text = subprocess.run([cuobjdump, "-res-usage", POLY_LIB], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", text, re.M)
    names = subprocess.run([shutil.which("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    assert sorted(kernel_key(n) for n in names) == sorted(r[0] for r in POLY_BUILDS)


class _Recorder(object):
    def __init__(self, protos, calls):
        self.protos, self.calls = protos, calls

    def __getattr__(self, name):
        if name not in self.protos:
            raise AttributeError(name)
        argtypes = self.protos[name][0]

        def entry(*args):
            assert len(args) == len(argtypes), name
            self.calls.append(name)
            return {"tb_record_doubles": lambda R: (3 * R + 2 + 1) & ~1}.get(name, lambda *a: 0)(*args)

        return entry


@pytest.fixture
def calls(monkeypatch):
    log = []
    main, poly = _Recorder(_lib._PROTOS, log), _Recorder(_lib_poly._PROTOS, log)
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(_lib, "load", lambda: main)
    monkeypatch.setattr(_lib_poly, "load", lambda: poly)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(engine, "default_device", lambda device=None: torch.device("cpu"))
    return log


def test_dispatch_cubic_keeps_todays_plan(calls):
    import toppra_b200 as ta
    x, c = random_pieces(3, 4, 3, 2, 1)
    lims = np.tile([[-1.0, 1.0]], (2, 1))
    path = ta.BatchPiecewisePolyPath(x, c)
    inst = ta.BatchTOPPRA(velacc(lims, lims), path, np.linspace(0, 1, 9))
    assert inst.fused
    del calls[:]
    inst.compute_parameterization()
    assert calls and all(n.startswith("tb_") for n in calls)
    assert calls == ["tb_xbound_velocity", "tb_scan_velacc_ragged"]


def test_dispatch_order6_takes_the_record_path(calls):
    import toppra_b200 as ta
    x, c = random_pieces(3, 6, 3, 2, 1)
    lims = np.tile([[-1.0, 1.0]], (2, 1))
    path = ta.BatchPiecewisePolyPath(x, c)
    assert calls == ["tbp_ppoly_eval"]        # positions at the breaks
    inst = ta.BatchTOPPRA(velacc(lims, lims), path, np.linspace(0, 1, 9))
    assert not inst.fused
    del calls[:]
    inst.compute_parameterization()
    launches = [n for n in calls if n != "tb_record_doubles"]   # a size query, no kernel
    assert launches == ["tbp_ppoly_eval", "tbp_ppoly_eval", "tbp_rows_velacc_sampled", "tb_scan_ragged"]
    with pytest.raises(NotImplementedError):
        engine.scan_velacc(path.d_ppoly, path.d_ss, inst.d_grid, inst.d_grid, True, inst.d_grid)


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_fixtures_use_scipy_derivative_objects(name):
    g, labels = golden_paths(name)
    for label in labels:
        c, x, s = g[label + "/path/c"], g[label + "/path/x"], g[label + "/path/s"]
        assert c.shape[0] == int(name[-1]) and c.shape[2] == 7 and 3 <= c.shape[1] <= 6 and (np.diff(x) > 0).all()
        for order, p in enumerate(scipy_derivs(c, x)):
            assert eq(g["%s/path/q%d" % (label, order)], p(s)), (label, order)
        statuses = {str(g[k]) for k in g if k.startswith(label + "/") and k.endswith("/status")}
        assert "Ok" in statuses and len(statuses) > 1, statuses
        assert os.path.getsize(os.path.join(ROOT, "tests", "golden", name + ".npz")) < 1 << 20
