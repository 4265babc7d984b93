"""Robust (conic) problems with several robust constraints, each with its own ellipsoid, and with u-bounds beside them:
libtoppra_b200_cones.so (tbc_*), its C restatement (tests/robust_cones_oracle.c) and the routing in toppra_b200.batch.

CPU: the restatement against the 50-digit stage problem (tests/robust_cones_mp.py), bit-identity with the
single-ellipsoid restatements, header prototypes, the library's exports and kernels, refusals before any CUDA call and
launch plans.  GPU: every tbc_* kernel against the restatement bit for bit, against the existing entries, sanity checks
and end-to-end runs on a 7-joint arm."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from mpmath import mpf

import robust_cones_oracle as rco
import robust_reach_oracle as rro
import robust_sd_oracle as rsd
from oracle import oracle as orc
from robust_cones_mp import RowStage
from test_robust_highprec import CASE_IDS, CASES, TOL_X, Worst, _box, check_end, layout
from test_robust_reachability import (ELL, _cfg4_on, _header_protos, _launches, _nonuniform, _ReachRecorder, eq,
                                      same_bits)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONES_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_cones.so")
ARM7 = os.path.join(ROOT, "tests", "golden", "robots", "arm7_gripper.urdf")
TB_ERR_ARG, TB_ERR_UNSUPPORTED, TB_ERR_ALIGN = -1, -2, -3
ELL_B = [4e-3, 2e-2, 3e-2]     # a second, different ellipsoid
ELL_C = [0.0, 1e-1, 2e-3]


def _gpu_present():
    return torch.cuda.is_available()


# ==== CPU: the restatement ===========================================================================================
def _two_cone_problem(seed, G, interp=True, uniform=True):
    """cfg-4 acceleration rows (28 = 2 x 7 x 2) split in two robust constraints with different ellipsoids."""
    grid = np.linspace(0, 1, G) if uniform else _nonuniform(G, seed)
    rows, xb = _cfg4_on(seed, grid, interp)
    R = rows.shape[2]
    return grid, rows, xb, R


def _ubox_of(G, lo, hi):
    return np.tile(np.array([[lo, hi]], dtype=np.float64), (G, 1))


def _row_stage(rows, xb, cones, i, box, xnext, ubox=None):
    return RowStage(rows[i, 0], rows[i, 1], rows[i, 2], cones[:, 0] != 0, cones[:, 1:], box[0], box[1], xnext,
                    None if ubox is None else ubox[i])


def _check_end(st, direction, got, worst, key, clamp0=False, what=""):
    ref = st.extreme_x(direction, None if np.isnan(got) else float(got))
    if ref is None:
        assert np.isnan(got), "%s: infeasible, got %r" % (what, got)
        return
    assert not np.isnan(got), "%s: NaN, the 50-digit reference finds %s" % (what, ref)
    if clamp0 and ref < 0:
        ref = mpf(0)
    err = abs(mpf(float(got)) - ref)
    assert err <= TOL_X * (abs(ref) + mpf("1e-300")), "%s: got %r, 50-digit %s" % (what, got, ref)
    worst.add(key, got, ref)


def _check_K(rows, xb, grid, cones, K, stages, worst, ubox=None, what=""):
    N = len(grid) - 1
    for i in stages:
        if i >= N or np.isnan(K[i + 1]).any() or np.isnan(K[i]).any():
            continue
        st = _row_stage(rows, xb, cones, i, _box(xb, i), (grid[i + 1] - grid[i], K[i + 1, 0], K[i + 1, 1]), ubox)
        _check_end(st, +1, K[i, 1], worst, "K_hi", what="%s stage %d upper" % (what, i))
        _check_end(st, -1, K[i, 0], worst, "K_lo", clamp0=True, what="%s stage %d lower" % (what, i))


@pytest.mark.parametrize("ncones,interp,uniform,ub", [(2, True, True, False), (2, False, False, True),
                                                      (3, True, False, True), (3, False, True, False)])
def test_restatement_cfg4_several_ellipsoids_against_50_digits(ncones, interp, uniform, ub, capsys):
    G = 200
    grid, rows, xb, R = _two_cone_problem(4100 + ncones + (0 if interp else 7), G, interp, uniform)
    spans = [(0, 14, ELL), (14, 14, ELL_B)] if ncones == 2 else [(0, 10, ELL), (10, 8, ELL_B), (18, 10, ELL_C)]
    cones = rco.table(R, spans)
    ubox = _ubox_of(G, -0.5, 0.4) if ub else None
    worst = Worst()
    out = rco.scan(rows, xb, grid, cones, 0.0, 0.0, ubox=ubox)
    assert out["status"] == 0
    N = G - 1
    _check_K(rows, xb, grid, cones, out["K"], [0, 1, N // 2, N - 2, N - 1], worst, ubox, "K")
    X = rco.feasible(rows, xb, grid, cones, ubox)
    for i in (0, N // 3, N):
        xn = (grid[i + 1] - grid[i], -1e4, 1e4) if i < N else None
        st = _row_stage(rows, xb, cones, i, _box(xb, i, True), xn, ubox)
        _check_end(st, -1, X[i, 0], worst, "X_lo", clamp0=True, what="X %d" % i)
        _check_end(st, +1, X[i, 1], worst, "X_hi", what="X %d" % i)
    # TOPPRAsd: u_i = uhi(x_i) of the fastest pass against the 50-digit u-interval
    x, u, st_, fs = rco.sd_forward(rows, grid, cones, out["K"], 0.0, False, ubox)
    assert st_ == 0
    for i in (0, N // 2, N - 1):
        stg = _row_stage(rows, xb, cones, i, (x[i], x[i]), (grid[i + 1] - grid[i], out["K"][i + 1, 0],
                                                           out["K"][i + 1, 1]), ubox)
        lo, hi = stg.u_interval(mpf(float(x[i])))
        assert abs(mpf(float(u[i])) - hi) <= TOL_X * (abs(hi) + 1), (i, u[i], hi)
        worst.add("u", u[i], hi)
        if ub:
            assert ubox[i, 0] <= u[i] <= ubox[i, 1]
    # a stage objective
    i = N // 2
    g = (-2 * (grid[i + 1] - grid[i]), -1.0)
    xn = (grid[i + 1] - grid[i], X[i + 1, 0], X[i + 1, 1])
    z = rco.socp(g, rows[i, 0], rows[i, 1], rows[i, 2], cones, *_box(xb, i), xnext=xn,
                 ubox=None if ubox is None else ubox[i])
    ref = _row_stage(rows, xb, cones, i, _box(xb, i), xn, ubox).socp(g, None)
    obj = g[0] * mpf(float(z[0])) + g[1] * mpf(float(z[1]))
    assert abs(obj - ref["obj"]) <= mpf("1e-12") * (1 + abs(ref["obj"]))
    worst.report(capsys, "%d ellipsoids%s" % (ncones, ", u box" if ub else ""))


def test_restatement_ubound_edges():
    """u box binding at the optimum, emptying a stage, ulo == uhi, and meeting a tangent conic row."""
    G = 40
    grid, rows, xb, R = _two_cone_problem(4200, G)
    cones = rco.table(R, [(0, 14, ELL), (14, 14, ELL_B)])
    free = rco.scan(rows, xb, grid, cones, 0.0, 0.0)
    assert free["status"] == 0
    # binding: a u box inside the free run's u range changes the result and holds on it
    umax = np.nanmax(np.abs(free["u"]))
    box = _ubox_of(G, -0.3 * umax, 0.3 * umax)
    bound = rco.scan(rows, xb, grid, cones, 0.0, 0.0, ubox=box)
    assert bound["status"] == 0 and np.all(bound["u"] <= 0.3 * umax) and np.all(bound["u"] >= -0.3 * umax)
    assert np.any(bound["u"] == 0.3 * umax) and np.all(bound["K"][:, 1] <= free["K"][:, 1] * (1 + 1e-12))
    # emptying stage 7: ulo > uhi
    empty = box.copy()
    empty[7] = (1.0, -1.0)
    out = rco.scan(rows, xb, grid, cones, 0.0, 0.0, ubox=empty)
    assert out["status"] == 3 and out["fail_stage"] == 7 and np.isnan(out["K"][7]).all()
    X = rco.feasible(rows, xb, grid, cones, empty)
    assert np.isnan(X[7]).all() and not np.isnan(X[8]).any()
    # ulo == uhi == 0 from rest: u = 0 throughout, so every x stays 0 -- K is [0, 0] everywhere and the path stands still
    zero = _ubox_of(G, 0.0, 0.0)
    z = rco.scan(rows, xb, grid, cones, 0.0, 0.0, ubox=zero)
    assert z["status"] == 0 and np.all(z["K"] == 0.0) and np.all(z["u"] == 0.0) and np.all(z["sd"] == 0.0)
    # ulo == uhi inside the free u range of one stage: the stage solve returns u = ulo exactly, and it is the 50-digit
    # optimum
    i = 12
    xn = (grid[i + 1] - grid[i], free["K"][i + 1, 0], free["K"][i + 1, 1])
    pin = (0.25 * free["u"][i], 0.25 * free["u"][i])
    zz = rco.socp((-1.0, -0.5), rows[i, 0], rows[i, 1], rows[i, 2], cones, *_box(xb, i), xnext=xn, ubox=pin)
    assert zz[0] == pin[0] and not np.isnan(zz[1])
    ref = _row_stage(rows, xb, cones, i, _box(xb, i), xn, np.array([pin] * G)).socp((-1.0, -0.5), None)
    assert abs(mpf(float(zz[1])) - ref["x"]) <= TOL_X * (abs(ref["x"]) + 1)
    # a tangent conic row: a single robust row a u + c + ||(ru u, 0, rc)|| <= 0 with |a| == ru, and the u box on it
    a, b, c = np.array([0.5]), np.array([0.0]), np.array([-0.25])
    t = np.array([[1.0, 0.5, 0.0, 0.0]])
    for ub in (None, (-1.0, 0.1), (-1.0, 0.25), (0.3, 0.4)):
        zz = rco.socp((-1.0, 0.0), a, b, c, t, 0.0, 1.0, None, ub)
        ref = RowStage(a, b, c, [True], [[0.5, 0.0, 0.0]], 0.0, 1.0, None, ub).socp((-1.0, 0.0), None)
        if ref is None:
            assert np.isnan(zz).all(), ub
        else:
            assert abs(mpf(float(zz[0])) - ref["u"]) <= mpf("1e-13") * (1 + abs(ref["u"])), (ub, zz, ref)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_restatement_edge_catalogue_next_to_a_second_ellipsoid(case, capsys):
    """The hand-built geometries of the edge catalogue on one robust constraint, with a second robust constraint beside
    them whose rows (the case's conic rows, loosened by 1 + |c|) carry other axes; K, the feasible sets and stage optima
    against the 50-digit problem, with the allowance for ill-conditioned ends."""
    _, xb, _, canon, cmask = layout(case)
    G = case["G"]
    grid = np.linspace(0, 1, G)
    ncon = int(cmask.sum())
    second = canon[:, :, cmask].copy()
    second[:, 2] -= 1.0 + np.abs(second[:, 2])
    rows = np.concatenate((canon, second), axis=2)
    R = rows.shape[2]
    nlin = R - 2 * ncon
    cones = rco.table(R, [(nlin, ncon, list(case["ell"])), (nlin + ncon, ncon, [0.3, 0.02, 0.05])])
    worst = Worst()
    e = case["sd_end"]
    out = rco.scan(rows, xb, grid, cones, case["sd_start"], e)
    K = out["K"]
    conic = cones[:, 0] != 0
    fail = [i for i in range(G - 1) if np.isnan(K[i]).any()]
    for i in ([s for s in range(G - 1) if s > fail[0]] + [fail[0]] if fail else range(G - 1)):   # rows below: 0
        if np.isnan(K[i + 1]).any():
            continue
        st = RowStage(rows[i, 0], rows[i, 1], rows[i, 2], conic, cones[:, 1:], *_box(xb, i),
                      (grid[i + 1] - grid[i], K[i + 1, 0], K[i + 1, 1]))
        check_end(st, +1, K[i, 1], worst, "K_hi", what="%s stage %d upper" % (case["name"], i))
        if not np.isnan(K[i, 1]):
            check_end(st, -1, K[i, 0], worst, "K_lo", clamp0=True, what="%s stage %d lower" % (case["name"], i))
    X = rco.feasible(rows, xb, grid, cones)
    for i in range(G):
        xn = (grid[i + 1] - grid[i], -1e4, 1e4) if i < G - 1 else None
        st = RowStage(rows[i, 0], rows[i, 1], rows[i, 2], conic, cones[:, 1:], *_box(xb, i, True), xn)
        check_end(st, -1, X[i, 0], worst, "X_lo", clamp0=True, what="%s X %d" % (case["name"], i))
        check_end(st, +1, X[i, 1], worst, "X_hi", what="%s X %d" % (case["name"], i))
    worst.report(capsys, case["name"] + " + second ellipsoid")


def _arm7_torque_rows(grid, way, ss):
    """Collocation rows of JointTorqueConstraint on the arm7 model (fingers locked, 7 joints), from the float64 double
    of tbd_torque_terms (tests/rnea_ref.py) on a cubic spline: F = [I; -I], g = [tau_hi; -tau_lo]."""
    from scipy.interpolate import CubicSpline
    from rnea_ref import torque_terms_packed
    import toppra_b200 as ta
    model = ta.dynamics.RigidBodyModel.from_urdf(ARM7, locked_joints={"finger_left_joint": 0.0,
                                                                      "finger_right_joint": 0.0})
    sp = CubicSpline(ss, way)
    a, b, c = torque_terms_packed(model.packed, sp(grid), sp(grid, 1), sp(grid, 2))
    lim = _tau_lim(model)
    rows = np.empty((len(grid), 3, 14))
    rows[:, 0] = np.concatenate((a, -a), axis=1)
    rows[:, 1] = np.concatenate((b, -b), axis=1)
    rows[:, 2] = np.concatenate((c - lim[:, 1], -c + lim[:, 0]), axis=1)
    return rows


@pytest.mark.parametrize("interp,uniform,ub", [(True, True, False), (False, False, True), (True, False, True)])
def test_restatement_cfg4_with_arm7_torque_against_50_digits(interp, uniform, ub, capsys):
    """Robust acceleration (config-4 ellipsoid) next to robust torque of the arm7 model (its own ellipsoid), 200
    gridpoints, optionally a u box."""
    from problems import make_path
    G = 200
    seed = 4400 + (0 if interp else 3)
    grid = np.linspace(0, 1, G) if uniform else _nonuniform(G, seed)
    acc, xb = _cfg4_on(seed, grid, interp)
    ss = np.linspace(0, 1, 5)
    way = 0.3 * make_path(seed)[0]            # slower motions: the torque rows bind, the problem stays feasible
    tau = _arm7_torque_rows(grid, way, ss)
    rows = np.concatenate((acc, tau), axis=2)
    R = rows.shape[2]
    Ra = acc.shape[2]
    cones = rco.table(R, [(0, Ra, ELL), (Ra, 14, [2e-3, 1e-1, 0.5])])
    ubox = _ubox_of(G, -2.0, 1.5) if ub else None
    worst = Worst()
    out = rco.scan(rows, xb, grid, cones, 0.0, 0.0, ubox=ubox)
    N = G - 1
    stages = [0, 1, N // 3, N // 2, N - 2, N - 1]
    _check_K(rows, xb, grid, cones, out["K"], stages, worst, ubox, "K")
    checked = [i for i in stages if not np.isnan(out["K"][i:i + 2]).any()]
    assert len(checked) >= 4, (out["status"], out["fail_stage"])
    X = rco.feasible(rows, xb, grid, cones, ubox)
    for i in (0, N // 2, N):
        xn = (grid[i + 1] - grid[i], -1e4, 1e4) if i < N else None
        st = _row_stage(rows, xb, cones, i, _box(xb, i, True), xn, ubox)
        _check_end(st, -1, X[i, 0], worst, "X_lo", clamp0=True, what="X %d" % i)
        _check_end(st, +1, X[i, 1], worst, "X_hi", what="X %d" % i)
    worst.report(capsys, "acceleration + arm7 torque%s" % (", u box" if ub else ""))


def test_restatement_equals_single_ellipsoid_entries_bit_for_bit():
    """One robust constraint, or several sharing one ellipsoid over contiguous rows, without a u box: every entry of the
    per-row restatement equals the single-ellipsoid restatements bit for bit."""
    G = 90
    grid, rows, xb, R = _two_cone_problem(4300, G, uniform=False)
    X1 = orc.feasible_rows_robust(rows, xb, grid, 4, 20, ELL)
    for spans in ([(4, 20, ELL)], [(4, 9, ELL), (13, 11, ELL)]):
        cones = rco.table(R, spans)
        o = orc.solve_rows_robust(rows, xb, grid, 4, 20, ELL, 0.1, 0.05)
        c = rco.scan(rows, xb, grid, cones, 0.1, 0.05)
        assert eq(c["K"], o["K"]) and eq(c["sd"], o["sd"]) and eq(c["u"], o["u"]) and c["status"] == o["status"]
        K, st, fs = rro.controllable_sets_robust(rows, xb, grid, 4, 20, ELL, 0.05, 0.4)
        c = rco.scan(rows, xb, grid, cones, 0.0, 0.05, 0.4, backward_only=True)
        assert eq(c["K"], K) and c["status"] == st and c["fail_stage"] == fs
        assert eq(rco.feasible(rows, xb, grid, cones), X1)
        for slow in (False, True):
            o = rsd.sd_forward_rows_robust(rows, grid, 4, 20, ELL, K, 0.0, slow)
            xo, uo, so, fo = o["x"], o["u"], o["status"], o["fail_stage"]
            xc, uc, sc, fc = rco.sd_forward(rows, grid, cones, K, 0.0, slow)
            assert eq(xc, xo) and eq(uc, uo) and sc == so and fc == fo
        L, f = rro.reachable_sets_robust(rows, xb, grid, 4, 20, ELL, X1, 0.0, 0.2)
        Lc, fc = rco.reachable(rows, xb, grid, cones, X1, 0.0, 0.2)
        assert eq(Lc, L) and fc == f
        i = 30
        xn = (grid[i + 1] - grid[i], X1[i + 1, 0], X1[i + 1, 1])
        for g in ((-1.0, -0.5), (1.0, 0.0), (0.0, -1.0)):
            zo = rsd.socp_stage_robust(g, rows[i, 0], rows[i, 1], rows[i, 2], 4, 20, ELL, *_box(xb, i), xnext=xn)
            zc = rco.socp(g, rows[i, 0], rows[i, 1], rows[i, 2], cones, *_box(xb, i), xnext=xn)
            assert eq(zc, zo), g


# ==== CPU: ABI, refusals and launch plans ============================================================================
def test_prototypes_match_the_header():
    from toppra_b200 import _lib_cones
    kind = {ctypes.c_int: "int", ctypes.c_double: "double"}
    declared = _header_protos("toppra_b200_cones.h", "tbc_")
    assert set(declared) == set(_lib_cones._PROTOS)
    for name, (argtypes, restype) in _lib_cones._PROTOS.items():
        assert [kind.get(t, "ptr") for t in argtypes] == declared[name], name
        assert restype is ctypes.c_int


def test_library_exports_and_kernel_inventory():
    from test_piecewise_poly import kernel_key
    if not os.path.exists(CONES_LIB):
        pytest.skip("libtoppra_b200_cones.so is not built")
    lib = ctypes.CDLL(CONES_LIB)
    for name in _header_protos("toppra_b200_cones.h", "tbc_"):
        assert hasattr(lib, name), name
    assert lib.tbc_version() == 100
    cuobjdump = os.path.join("/usr/local/cuda", "bin", "cuobjdump")
    cuobjdump = cuobjdump if os.path.exists(cuobjdump) else shutil.which("cuobjdump")
    if not cuobjdump or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not found")
    text = subprocess.run([cuobjdump, "-res-usage", CONES_LIB], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", text, re.M)
    names = subprocess.run([shutil.which("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    want = ["%s<%d>" % (k, r) for k in ("tbc_reachable_kernel", "tbc_scan_kernel", "tbc_sd_forward_kernel",
                                        "tbc_socp_stage_kernel") for r in (1, 2, 3, 4)]
    assert sorted(kernel_key(n) for n in names) == sorted(want)


@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_refusals_before_any_cuda_call():
    """Every refusal of the four entries comes before any CUDA call: host addresses stand in for device arrays."""
    from toppra_b200 import _lib, _lib_cones
    lib, clib = _lib.load(), _lib_cones.load()
    mem = np.zeros(1 << 16)
    p = ctypes.c_void_p(mem.ctypes.data)
    good = rco.table(28, [(0, 14, ELL), (14, 14, ELL_B)])
    big = np.zeros((127, 4))

    def tab(t):
        t = np.ascontiguousarray(t)
        tab.keep.append(t)
        return ctypes.c_void_p(t.ctypes.data)
    tab.keep = []
    bad_flag, neg, nan = good.copy(), good.copy(), good.copy()
    bad_flag[3, 0] = 2.0
    neg[5, 2] = -1e-3
    nan[27, 3] = np.nan

    def scan(**kw):
        a = dict(records=p, W=86, R=28, cones=tab(good), grid=p, gs=1, B=2, G=9, glen=None, s0=p, s1=p, s1h=None,
                 flags=1, K=p, sd=p, u=p, st=p, fs=p, cnt=None)
        a.update(kw)
        return clib.tbc_scan(*a.values(), None), lib.tb_last_error().decode()

    for k in ("records", "grid", "cones", "K", "st"):
        rc, msg = scan(**{k: None})
        assert rc == TB_ERR_ARG and "tbc_scan" in msg, k
    assert scan(flags=0, sd=None)[0] == TB_ERR_ARG
    assert scan(W=85)[0] == TB_ERR_ALIGN
    assert scan(flags=1 | 64)[0] == TB_ERR_ARG                      # u box without W >= 3R+4
    assert scan(flags=1 | 4)[0] == TB_ERR_UNSUPPORTED
    for t in (bad_flag, neg, nan):
        rc, msg = scan(cones=tab(t))
        assert rc == TB_ERR_ARG and "cone row" in msg
    assert scan(R=127, W=3 * 127 + 3, cones=tab(big))[0] == TB_ERR_UNSUPPORTED
    assert scan(glen=p)[0] == TB_ERR_ARG

    def sdf(**kw):
        a = dict(records=p, W=86, R=28, cones=tab(good), flags=0, grid=p, gs=1, B=2, G=9, glen=None, K=p, si=p, s0=p,
                 xf=p, uf=p, xs=p, us=p, st=p, fs=p)
        a.update(kw)
        return clib.tbc_sd_forward(*a.values(), None), lib.tb_last_error().decode()

    for k in ("records", "grid", "cones", "K", "si", "xf", "xs", "st"):
        assert sdf(**{k: None})[0] == TB_ERR_ARG, k
    assert sdf(flags=64)[0] == TB_ERR_ARG and sdf(W=85)[0] == TB_ERR_ALIGN and sdf(flags=1)[0] == TB_ERR_UNSUPPORTED
    assert sdf(cones=tab(neg))[0] == TB_ERR_ARG and sdf(R=127, W=400, cones=tab(big))[0] == TB_ERR_UNSUPPORTED

    def socp(**kw):
        a = dict(g=p, a=p, b=p, c=p, n=28, cones=tab(good), xbox=p, xnext=None, ubox=p, B=2, out=p)
        a.update(kw)
        return clib.tbc_socp_stage_batch(*a.values(), None), lib.tb_last_error().decode()

    for k in ("g", "a", "cones", "xbox", "out"):
        assert socp(**{k: None})[0] == TB_ERR_ARG, k
    assert socp(cones=tab(bad_flag))[0] == TB_ERR_ARG and socp(n=127, cones=tab(big))[0] == TB_ERR_UNSUPPORTED

    def reach(**kw):
        a = dict(records=p, W=86, R=28, cones=tab(good), flags=0, grid=p, gs=1, B=2, G=9, glen=None, X=p, lo=p,
                 hi=p, L=p, fs=p)
        a.update(kw)
        return clib.tbc_reachable_sets(*a.values(), None), lib.tb_last_error().decode()

    for k in ("records", "grid", "cones", "X", "L"):
        assert reach(**{k: None})[0] == TB_ERR_ARG, k
    assert reach(flags=64)[0] == TB_ERR_ARG and reach(W=85)[0] == TB_ERR_ALIGN and reach(glen=p)[0] == TB_ERR_ARG
    assert reach(cones=tab(nan))[0] == TB_ERR_ARG and reach(R=127, W=400, cones=tab(big))[0] == TB_ERR_UNSUPPORTED


class _ConesRecorder(_ReachRecorder):
    def __getattr__(self, name):
        from toppra_b200 import _lib_cones
        argtypes, _ = _lib_cones._PROTOS[name]

        def entry(*args):
            assert len(args) == len(argtypes), name
            self.rec.calls.append((name, args))
            return 0
        return entry


@pytest.fixture
def rlib(monkeypatch):
    from test_engine_marshalling import RecordingLib
    import toppra_b200 as ta
    from toppra_b200 import _lib, _lib_cones, _lib_reach, _lib_robust, engine
    rec = RecordingLib()
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(_lib_reach, "load", lambda: _ReachRecorder(rec))
    monkeypatch.setattr(_lib_cones, "load", lambda: _ConesRecorder(rec))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: __import__("contextlib").nullcontext())
    monkeypatch.setattr(engine, "default_device", lambda device=None: torch.device("cpu"))
    return rec, ta


def _problem(ta, kind, B=6, G=40, dof=6, ragged=False):
    rng = np.random.RandomState(0)
    path = ta.BatchSplineInterpolator(np.linspace(0, 1, 5), rng.randn(B, 5, dof))
    lim = np.tile(np.array([[-1.0, 1.0]]), (dof, 1))
    acc = ta.constraint.JointAccelerationConstraint(lim)
    cons = [ta.constraint.JointVelocityConstraint(lim), ta.constraint.RobustLinearConstraint(acc, [0.1, 0.1, 0.1], 1)]
    if kind in ("two", "two+ub"):
        acc2 = ta.constraint.JointAccelerationConstraint(2 * lim)
        cons.append(ta.constraint.RobustLinearConstraint(acc2, [0.2, 0.0, 0.05], 1))
    if kind in ("ub", "two+ub"):
        cons.append(_ubound_constraint(ta, dof, -0.5, 0.5))
    grid = np.linspace(0, 1, G)
    if ragged:
        grid = np.tile(grid, (B, 1))
    return path, cons, grid


def _ubound_constraint(ta, dof, lo, hi):
    """A linear constraint with no rows that bounds only the path acceleration: lo <= u <= hi (its ubound), on every
    path of a batch (the records' u-bound pair)."""
    from toppra_b200.constraint import DiscretizationType, LinearConstraint

    class UBound(LinearConstraint):
        def __init__(self):
            super(UBound, self).__init__()
            self.dof = dof
            self.discretization_type = DiscretizationType.Collocation
            self.identical = True

        def compute_constraint_params(self, path, gridpoints, *args, **kwargs):
            return None, None, None, None, None, np.tile([[lo, hi]], (len(gridpoints), 1)), None

        def num_rows(self, ctx):
            return 0

        def has_ubound(self, ctx):
            return True

        def append_records(self, ctx, records, R_total, row0):
            records[:, :, 3 * R_total + 2].clamp_(min=lo)
            records[:, :, 3 * R_total + 3].clamp_(max=hi)
    return UBound()


def test_launch_plans(rlib):
    rec, ta = rlib
    # one robust constraint, no ubound: today's entries
    path, cons, grid = _problem(ta, "one")
    inst = ta.BatchTOPPRA(cons, path, gridpoints=grid)
    inst.setup()
    assert isinstance(inst.conic, tuple)
    mark = len(rec.calls)
    inst.compute_parameterization(0, 0)
    inst.compute_reachable_sets(0.0, 0.0)
    assert _launches(rec, mark) == ["tb_scan_robust", "tb_scan_robust", "tbr_reachable_sets_robust"]
    # two robust constraints, a ubound, or both: the tbc_* entries
    for kind, ub in (("two", False), ("ub", True), ("two+ub", True)):
        path, cons, grid = _problem(ta, kind)
        inst = ta.BatchTOPPRA(cons, path, gridpoints=grid)
        inst.setup()
        assert isinstance(inst.conic, ta.batch.Cones)
        mark = len(rec.calls)
        inst.compute_parameterization(0, 0)
        inst.compute_controllable_sets(0.0, 0.5)
        inst.compute_reachable_sets(0.0, 0.0)
        inst.compute_feasible_sets()
        assert _launches(rec, mark) == ["tbc_scan", "tbc_scan", "tbc_scan", "tbc_reachable_sets", "tbc_scan"], kind
        args = rec.last("tbc_scan")
        assert args[12] == (2 | (64 if ub else 0)), kind                # TB_SCAN_FEASIBLE_SETS [| TB_SCAN_UBOUND]
        sd = ta.BatchTOPPRAsd(cons, path, gridpoints=grid)
        sd.set_desired_duration(2.0)
        mark = len(rec.calls)
        sd.compute_parameterization(0, 0)
        assert [n for n in _launches(rec, mark) if n.startswith("tbc_")] == ["tbc_scan", "tbc_sd_forward"]
    # record chunks: the same launches per chunk
    path, cons, grid = _problem(ta, "two+ub")
    probe = ta.BatchTOPPRA(cons, path, gridpoints=grid)
    probe.setup()
    per_path = 8 * ta.engine.record_doubles(probe.R) * len(grid)
    small = ta.BatchTOPPRA(cons, path, gridpoints=grid, max_record_bytes=4 * per_path)
    mark = len(rec.calls)
    small.compute_parameterization(0, 0)
    assert [a[6] for n, a in rec.calls[mark:] if n == "tbc_scan"] == [4, 2]


def test_ragged_refusals_still_hold(rlib):
    rec, ta = rlib
    B, G = 4, 30
    path, cons, grid = _problem(ta, "two+ub", B, G, ragged=True)
    glen = np.array([30, 20, 25, 30], dtype=np.int32)
    inst = ta.BatchTOPPRA(cons, path, gridpoints=grid, glen=glen, validate=False)
    inst.setup()
    mark = len(rec.calls)
    with pytest.raises(NotImplementedError):
        inst.compute_reachable_sets(0.0, 0.0)
    with pytest.raises(NotImplementedError):
        inst.compute_controllable_sets(0.0, 0.5)
    assert _launches(rec, mark) == []
    inst.compute_parameterization(0, 0)
    assert [n for n in _launches(rec, mark) if n.startswith("tb")] == ["tbc_scan"]
    assert rec.last("tbc_scan")[8] is not None                                            # glen


def test_still_refused(rlib):
    rec, ta = rlib
    path, cons, grid = _problem(ta, "one")

    base = _ubound_constraint(ta, 6, -1.0, 1.0)
    rob = ta.constraint.RobustLinearConstraint(base, [0.1, 0.1, 0.1], 0)
    inst = ta.BatchTOPPRA(cons[:1] + [rob], path, gridpoints=grid)
    with pytest.raises(NotImplementedError, match="base constraint has a ubound"):
        inst.setup()


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _widened(ta, rpl, B, G, ub=False, ragged=False, seed0=5000):
    """cfg-4 records widened to rpl rows per lane (R = 28 rpl): copy k scaled by 1.25^k; a cone table with a different
    ellipsoid per copy (copy 0 ELL, the others robust with their own axes or linear); optionally the u box."""
    from test_robust_sd import _widened_records
    rec0, R, grid, glen = _widened_records(ta, rpl, B, G, seed0=seed0, ragged=ragged)
    cones = np.zeros((R, 4))
    cones[:28] = [1.0] + ELL
    for k in range(1, rpl):
        if k % 2:
            cones[28 * k:28 * (k + 1)] = [1.0, 2e-3 * k, 3e-2, 5e-3 * k]
    if ub:
        rec, W = ta.engine.alloc_records(B, G, R, rec0.device, ubound=True)
        rec.fill_(0.0)
        rec[:, :, :3 * R + 2] = rec0[:, :, :3 * R + 2]
        rec[:, :, 3 * R] = rec0[:, :, 3 * R]
        lo = -0.4 - 0.1 * torch.rand(B, G, dtype=torch.float64, device=rec.device)
        rec[:, :, 3 * R + 2] = lo
        rec[:, :, 3 * R + 3] = 0.3 + 0.1 * torch.rand(B, G, dtype=torch.float64, device=rec.device)
        return rec, R, grid, glen, cones
    return rec0, R, grid, glen, cones


def _host(rec, R, b, n):
    h = rec[b, :n].cpu().numpy()
    rows = h[:, :3 * R].reshape(n, 3, R)
    ubox = h[:, 3 * R + 2:3 * R + 4] if h.shape[1] >= 3 * R + 4 else None
    return rows, h[:, 3 * R:3 * R + 2], ubox


@pytest.mark.gpu
@pytest.mark.parametrize("rpl,ub,ragged", [(1, False, False), (2, True, False), (3, False, True), (4, True, False),
                                           (1, True, True)])
def test_gpu_kernels_equal_restatement(ta, rpl, ub, ragged):
    B, G = 12, 50
    rec, R, grid, glen, cones = _widened(ta, rpl, B, G, ub, ragged)
    rec[0, :, 2 * R:3 * R] = -1e-4          # path 0: infeasible everywhere
    rec[1, 20:, 2 * R:3 * R] = -1e-4        # path 1: fails at stage 20
    dev = rec.device
    s_end = torch.linspace(0, 0.2, B, dtype=torch.float64, device=dev)
    s_hi = s_end + 0.3
    s_start = torch.zeros(B, dtype=torch.float64, device=dev)
    kw = {} if glen is None else {"glen": glen}
    full = ta.engine.scan_cones(rec, R, cones, grid, s_start, s_end, **kw)
    back = ta.engine.scan_cones(rec, R, cones, grid, None, s_end, backward_only=True, sd_end_hi=s_hi, **kw)
    X = ta.engine.scan_cones(rec, R, cones, grid, feasible_sets=True, **kw)["K"]
    fwd = ta.engine.sd_forward_cones(rec, R, cones, grid, full["K"], full["status"], s_start, **kw)
    reach = ta.engine.reachable_sets_cones(rec, R, cones, grid, s_start, s_end, **kw)
    gr = grid.cpu().numpy()
    h = {k: v.cpu().numpy() for k, v in full.items() if v is not None}
    for b in range(B):
        n = G if glen is None else int(glen[b])
        rows, xb, ubox = _host(rec, R, b, n)
        g = (gr if gr.ndim == 1 else gr[b])[:n]
        o = rco.scan(rows, xb, g, cones, 0.0, float(s_end[b]), ubox=ubox)
        assert eq(h["K"][b, :n], o["K"]) and eq(h["sd"][b, :n], o["sd"]) and eq(h["u"][b, :n - 1], o["u"]), b
        assert h["status"][b] == o["status"] and h["fail_stage"][b] == o["fail_stage"], b
        ob = rco.scan(rows, xb, g, cones, 0.0, float(s_end[b]), float(s_hi[b]), ubox=ubox, backward_only=True)
        assert eq(back["K"][b, :n].cpu().numpy(), ob["K"]) and int(back["status"][b]) == ob["status"], b
        Xo = rco.feasible(rows, xb, g, cones, ubox)
        assert eq(X[b, :n].cpu().numpy(), Xo), b
        for key, slow in (("fast", False), ("slow", True)):
            xo, uo, so, fo = rco.sd_forward(rows, g, cones, h["K"][b, :n], 0.0, slow, ubox)
            assert eq(fwd["x_" + key][b, :n].cpu().numpy(), xo) and eq(fwd["u_" + key][b, :n - 1].cpu().numpy(), uo)
            if not slow:
                assert int(fwd["status"][b]) == so and int(fwd["fail_stage"][b]) == fo
        Lo, fo = rco.reachable(rows, xb, g, cones, Xo, 0.0, float(s_end[b]), ubox)
        assert eq(reach["L"][b, :n].cpu().numpy(), Lo) and int(reach["fail_stage"][b]) == fo, b
    n1 = G if glen is None else int(glen[1])
    assert h["status"][0] == 3 and h["status"][1] == 3 and h["fail_stage"][1] == n1 - 2   # the backward pass meets it first


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 2, 3, 4])
def test_gpu_socp_stage_equals_restatement(ta, rpl):
    rng = np.random.RandomState(rpl)
    n, B = 28 * rpl, 64
    a, b = rng.randn(B, n), rng.randn(B, n) * 0.1
    c = -np.abs(rng.randn(B, n)) - 0.05
    cones = np.zeros((n, 4))
    cones[: n // 2] = [1.0, 0.05, 0.02, 0.01]
    cones[n // 2::3] = [1.0, 0.3, 0.0, 0.04]
    g = rng.randn(B, 2)
    g[::5, 0] = 0.0
    xbox = np.tile([[0.0, 5.0]], (B, 1))
    xnext = np.column_stack((np.full(B, 0.01), np.zeros(B), np.full(B, 3.0)))
    xnext[::7, 0] = np.nan
    ubox = np.column_stack((-1.0 - rng.rand(B), 0.5 + rng.rand(B)))
    ubox[3] = (0.2, 0.2)
    ubox[4] = (0.5, -0.5)
    for ub in (None, ubox):
        out = ta.engine.socp_stage_batch_cones(g, a, b, c, cones, xbox, xnext, ub)
        for p in range(B):
            want = rco.socp(g[p], a[p], b[p], c[p], cones, 0.0, 5.0, xnext[p], None if ub is None else ub[p])
            assert eq(out[p], want), p
    assert np.isnan(out[4]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 2, 4])
def test_gpu_one_ellipsoid_table_equals_existing_entries(ta, rpl):
    B, G = 10, 40
    rec, R, grid, glen, _ = _widened(ta, rpl, B, G, ragged=True)
    dev = rec.device
    s = torch.linspace(0, 0.1, B, dtype=torch.float64, device=dev)
    for spans in ([(0, 28, ELL)], [(0, 11, ELL), (11, 17, ELL)]):
        t = rco.table(R, spans)
        a = ta.engine.scan_cones(rec, R, t, grid, s, s, counters=True, glen=glen)
        o = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, s, s, counters=True, glen=glen)
        for k in ("K", "sd", "u", "status", "fail_stage", "counters"):
            assert same_bits(a[k], o[k]), k
        a = ta.engine.scan_cones(rec, R, t, grid, None, s, backward_only=True, glen=glen, sd_end_hi=s + 0.2)
        o = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, None, s, backward_only=True, glen=glen, sd_end_hi=s + 0.2)
        assert same_bits(a["K"], o["K"]) and same_bits(a["status"], o["status"])
        fa = ta.engine.sd_forward_cones(rec, R, t, grid, o["K"], o["status"], s, glen=glen)
        fo = ta.engine.sd_forward_robust(rec, R, 0, 28, ELL, grid, o["K"], o["status"], s, glen=glen)
        for k in fa:
            assert same_bits(fa[k], fo[k]), k
        ra = ta.engine.reachable_sets_cones(rec, R, t, grid, s, s + 0.1, glen=glen)
        ro = ta.engine.reachable_sets_robust(rec, R, 0, 28, ELL, grid, s, s + 0.1, glen=glen)
        for k in ra:
            assert same_bits(ra[k], ro[k]), k
        # stage solves: stage 7 of every path, g of both signs and g0 = 0, with and without the x_next rows
        h = rec[:, 7].cpu().numpy()
        a, b, c = h[:, :R], h[:, R:2 * R], h[:, 2 * R:3 * R]
        n = a.shape[0]
        g = np.tile([[-1.0, -0.3], [1.0, 0.2], [0.0, -1.0]], (n // 3 + 1, 1))[:n]
        xbox = np.column_stack((np.maximum(h[:, 3 * R], -1e3), np.minimum(h[:, 3 * R + 1], 1e3)))
        Ko = o["K"][:, 8].cpu().numpy()
        xnext = np.column_stack((np.full(n, 0.02), Ko[:, 0], Ko[:, 1]))
        xnext[::4, 0] = np.nan
        for xn in (None, xnext):
            za = ta.engine.socp_stage_batch_cones(g, a, b, c, t, xbox, xn)
            zo = ta.engine.socp_stage_batch(g, a, b, c, 0, 28, ELL, xbox, xn)
            assert eq(za, zo)


def _tau_lim(model):
    """The model's torque limits, with 30 N m on the joints whose URDF gives none (a robust row needs finite limits)."""
    return np.nan_to_num(model.torque_limits(), posinf=30.0, neginf=-30.0)


def _arm7(ta):
    return ta.dynamics.RigidBodyModel.from_urdf(ARM7, locked_joints={"finger_left_joint": 0.0,
                                                                     "finger_right_joint": 0.0})


def _e2e(ta, B=6, G=60, e_acc=ELL, e_tau=(2e-3, 1e-1, 0.5), ub=(-3.0, 2.5), zero=False):
    from problems import make_batch
    model = _arm7(ta)
    ss, way, vlim, alim = make_batch(B, 6100)
    path = ta.BatchSplineInterpolator(ss, way)
    if zero:
        e_acc, e_tau = (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)
    cons = [ta.constraint.JointVelocityConstraint(vlim[0]),
            ta.constraint.RobustLinearConstraint(ta.constraint.JointAccelerationConstraint(alim[0]), list(e_acc), 1),
            ta.constraint.RobustLinearConstraint(ta.constraint.JointTorqueConstraint(model, _tau_lim(model),
                                                                                      np.zeros(7)), list(e_tau), 1)]
    if ub is not None:
        cons.append(_ubound_constraint(ta, 7, *ub))
    return cons, path, np.linspace(0, 1, G), ss, way


def _user_ubound(ta, dof, lo, hi):
    """A user's LinearConstraint with no rows whose only content is a ubound from compute_constraint_params: it takes
    the package's default route (LinearConstraint.has_ubound / append_records), which builds records for one path."""
    from toppra_b200.constraint import DiscretizationType, LinearConstraint

    class UserUBound(LinearConstraint):
        def __init__(self):
            super(UserUBound, self).__init__()
            self.dof = dof
            self.discretization_type = DiscretizationType.Collocation

        def compute_constraint_params(self, path, gridpoints, *args, **kwargs):
            return None, None, None, None, None, np.tile([[lo, hi]], (len(gridpoints), 1)), None
    return UserUBound()


@pytest.mark.gpu
def test_gpu_single_path_user_ubound_default_route(ta):
    """Single-path TOPPRA with two robust constraints and a user constraint whose ubound comes through the default
    route equals the B = 1 batch with the same u box, and keeps u inside it."""
    cons, path, grid, ss, way = _e2e(ta, B=1, ub=None)
    one = ta.SplineInterpolator(ss, way[0])
    algo = ta.algorithm.TOPPRA(cons + [_user_ubound(ta, 7, -3.0, 2.5)], one, gridpoints=grid, solver_wrapper="ecos")
    assert isinstance(algo.solver_wrapper.conic, ta.batch.Cones) and algo.solver_wrapper.conic.ubound
    algo.compute_parameterization(0, 0)
    b1 = ta.BatchTOPPRA(cons + [_ubound_constraint(ta, 7, -3.0, 2.5)], path, grid).compute_parameterization(0, 0)
    h = b1.to_host()
    assert h["status"][0] == 0
    assert eq(algo.problem_data.sd_vec, h["sd"][0]) and eq(algo.problem_data.sdd_vec, h["sdd"][0])
    assert np.all(h["sdd"][0] >= -3.0) and np.all(h["sdd"][0] <= 2.5)
    free = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    if np.nanmax(free["sdd"][0]) > 2.5:        # the u box binds: the fastest pass rides on it somewhere
        assert np.any(h["sdd"][0] == 2.5)
    z = algo.solver_wrapper.solve_stagewise_optim(10, None, np.array([-1.0, 0.0]), np.nan, np.nan, np.nan, np.nan)
    assert -3.0 <= z[0] <= 2.5


@pytest.mark.gpu
def test_gpu_zero_axes_equal_linear_kernels(ta):
    cons, path, grid, _, _ = _e2e(ta, zero=True)
    rob = ta.BatchTOPPRA(cons, path, grid)
    lin = ta.BatchTOPPRA([c.base_constraint if hasattr(c, "base_constraint") else c for c in cons], path, grid)
    r, l_ = rob.compute_parameterization(0, 0).to_host(), lin.compute_parameterization(0, 0).to_host()
    assert np.array_equal(r["status"], l_["status"]) and np.array_equal(r["fail_stage"], l_["fail_stage"])
    for k in ("K", "sd", "sdd"):
        assert np.array_equal(np.isnan(r[k]), np.isnan(l_[k])), k
        np.testing.assert_allclose(r[k], l_[k], rtol=1e-9, atol=1e-9, equal_nan=True)


@pytest.mark.gpu
def test_gpu_bigger_ellipsoid_is_slower_and_rows_hold(ta):
    cons, path, grid, _, _ = _e2e(ta)
    base = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    assert not base["status"].any()
    for which in (1, 2):
        bigger = list(cons)
        ell = 2.0 * np.asarray(cons[which].ellipsoid())
        bigger[which] = ta.constraint.RobustLinearConstraint(cons[which].base_constraint, list(ell), 1)
        h = ta.BatchTOPPRA(bigger, path, grid).compute_parameterization(0, 0).to_host()
        assert not h["status"].any()
        assert np.all(h["K"][:, :, 1] <= base["K"][:, :, 1] * (1 + 1e-12) + 1e-12)
        dur = lambda sd: np.sum(2 * np.diff(grid) / (sd[:, 1:] + sd[:, :-1]), axis=1)   # noqa: E731
        assert np.all(dur(h["sd"]) >= dur(base["sd"]) - 1e-12)
    # every row with its own axes holds at the returned (u, x), in long double; u inside the u box
    inst = ta.BatchTOPPRA(cons, path, grid)
    inst.setup()
    rec = inst.records.cpu().numpy()
    R, t = inst.R, inst.conic.table()
    for b in range(path.B):
        x, u = base["sd"][b] ** 2, base["sdd"][b]
        for i in range(len(grid) - 1):
            a_, b_, c_ = (rec[b, i, k * R:(k + 1) * R].astype(np.longdouble) for k in range(3))
            ui, xi = np.longdouble(u[i]), np.longdouble(x[i])
            norm = np.sqrt((t[:, 1] * ui) ** 2 + (t[:, 2] * xi) ** 2 + t[:, 3] ** 2)
            v = a_ * ui + b_ * xi + c_ + np.where(t[:, 0] != 0, norm, 0)
            assert np.all(v <= 1e-9 * (1 + np.abs(a_ * ui) + np.abs(b_ * xi) + np.abs(c_))), (b, i, v.max())
            assert rec[b, i, 3 * R + 2] <= u[i] <= rec[b, i, 3 * R + 3]


@pytest.mark.gpu
def test_gpu_end_to_end_arm7(ta):
    cons, path, grid, ss, way = _e2e(ta)
    B = path.B
    inst = ta.BatchTOPPRA(cons, path, grid)
    res = inst.compute_parameterization(0, 0)
    h = res.to_host()
    assert not h["status"].any() and np.all(h["sd"] >= 0)
    per_path = 8 * (3 * inst.R + 4) * len(grid)
    small = ta.BatchTOPPRA(cons, path, grid, max_record_bytes=2 * per_path)
    assert small.chunk_size() < B
    hs = small.compute_parameterization(0, 0).to_host()
    for k in h:
        assert eq(h[k], hs[k]), k
    L, X, fs = inst.compute_reachable_sets(0, 0)
    Ls, Xs, fss = small.compute_reachable_sets(0, 0)
    assert same_bits(L, Ls) and same_bits(X, Xs) and same_bits(fs, fss)
    K, st = inst.compute_controllable_sets(0, 1)
    Ks, sts = small.compute_controllable_sets(0, 1)
    assert same_bits(K, Ks) and same_bits(st, sts) and not st.any()
    assert same_bits(inst.compute_feasible_sets(), small.compute_feasible_sets())
    sd = ta.BatchTOPPRAsd(cons, path, grid)
    sd.set_desired_duration(5.0)
    r = sd.compute_parameterization(0, 0)
    sds = ta.BatchTOPPRAsd(cons, path, grid, max_record_bytes=2 * per_path)
    sds.set_desired_duration(5.0)
    rs = sds.compute_parameterization(0, 0)
    for k in ("K", "sd", "sdd", "status"):
        assert same_bits(getattr(r, k), getattr(rs, k)), k
    # single path: TOPPRA / TOPPRAsd with the ecos / cvxpy / b200 wrappers equal the B = 1 batch
    one_path = ta.SplineInterpolator(ss, way[0])
    ones = cons
    b1 = ta.BatchTOPPRA(ones, ta.BatchSplineInterpolator(ss, way[:1]), grid).compute_parameterization(0, 0).to_host()
    for wrapper in ("ecos", "cvxpy", "b200"):
        algo = ta.algorithm.TOPPRA(ones, one_path, gridpoints=grid, solver_wrapper=wrapper)
        algo.compute_parameterization(0, 0)
        assert eq(algo.problem_data.sd_vec, b1["sd"][0]), wrapper
    algo = ta.algorithm.TOPPRA(ones, one_path, gridpoints=grid, solver_wrapper="ecos")
    Kc = algo.compute_controllable_sets(0, 1)
    assert np.all(np.isfinite(Kc))
    Lr = algo.compute_reachable_sets(0, 0)
    assert np.all(np.isfinite(Lr))
    xs = algo.solver_wrapper.solve_stagewise_optim(10, None, np.array([-1.0, -0.01]), np.nan, np.nan, np.nan, np.nan)
    assert np.all(np.isfinite(xs))
    sd1 = ta.algorithm.TOPPRAsd(ones, one_path, gridpoints=grid, solver_wrapper="ecos")
    sd1.set_desired_duration(5.0)
    sd1.compute_parameterization(0, 0)
    b1sd = ta.BatchTOPPRAsd(ones, ta.BatchSplineInterpolator(ss, way[:1]), grid)
    b1sd.set_desired_duration(5.0)
    rr = b1sd.compute_parameterization(0, 0)
    assert eq(sd1.problem_data.sd_vec, rr.sd[0].cpu().numpy())
