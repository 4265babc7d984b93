"""Robust (conic) problems: reachable sets (tbr_reachable_sets_robust, libtoppra_b200_reach.so) and controllable sets
over a velocity range (tb_scan_robust_ex, libtoppra_b200.so: K[N] = [sd_end^2, sd_end_hi^2]).

Parity with the reference is unpinned (it solves these stage problems with ECOS), so the evidence has the shape of
tests/test_robust_sd.py:
  * CPU: the C restatement (tests/robust_sd_oracle.c: orc_reachable_sets_robust, orc_controllable_sets_robust) meets the
    50-digit reference of tests/robust_mp.py at sampled stages: every L end is max / min x + 2 delta' u of its stage
    (Stage.socp), every K end the extreme x of its stage with the interval's own K[i+1] (Stage.extreme_x);
  * GPU: the kernels equal the restatement bit for bit (NaN equal to NaN), for 1 to 4 rows per lane and failing paths;
    ragged batches (engine level), chunked and single-path runs equal their counterparts; sdmin == sdmax and NULL equal
    today's entries;
  * GPU, independent sanity: a zero ellipsoid gives the linear kernels' sets, the sets nest, and parameterisations lie
    inside them;
  * CPU: refusals of the real libraries, the ctypes prototypes, the launch plans on the recording library."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from mpmath import mpf

import robust_reach_oracle as rro
from oracle import oracle as orc
from problems import make_batch, make_path
from test_robust_highprec import CASES, CASE_IDS, TOL_X, Worst, check_K, layout, stage
from test_robust_sd import _widened_records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ELL = [1e-3, 5e-2, 9e-3]   # defaults of examples/plot_robust_kinematics.py:26-28
ECOS_INFTY, ECOS_MAXX = 1000.0, 10000.0
TB_ERR_ARG, TB_ERR_UNSUPPORTED, TB_ERR_ALIGN = -1, -2, -3


def eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def same_bits(a, b):
    """torch.equal on the bit patterns: NaN entries (failed paths) compare equal when their bits are."""
    if a.dtype == torch.float64:
        a, b = a.view(torch.int64), b.view(torch.int64)
    return torch.equal(a, b)


def _cfg4_on(seed, grid, interp=True):
    """cfg 4 rows (the acceleration rows of the linear oracle, all robust) and xbound on the given grid."""
    ss = np.linspace(0, 1, 5)
    way, vlim, alim = make_path(seed)
    lin = orc.solve_velacc(orc.cubic_spline_fit(ss, way), ss, grid, vlim, alim, interp, 0, 0, want_rows=True)
    return lin["rows"], lin["xbound"]


def _nonuniform(G, seed):
    w = 0.3 + np.random.RandomState(seed).rand(G - 1)
    g = np.concatenate(([0.0], np.cumsum(w)))
    g /= g[-1]
    g[-1] = 1.0
    return g


# ==== CPU: the restatement against the 50-digit reference ============================================================
def check_L(rows, xb, grid, conic, ell, X, L, stages, worst, what=""):
    """L [G, 2] of a forward recursion: each sampled end from the result's own L[i] and X[i+1].  The end x + 2 delta' u
    of the 50-digit optimum is met to TOL_X relative; where it is a small difference of large terms, TOL_X of the
    terms' size is allowed (the end moves that much when x or u moves by TOL_X)."""
    N = len(grid) - 1
    nan_rows = [i for i in range(N + 1) if np.isnan(L[i]).any()]
    last = nan_rows[0] if nan_rows else N     # the rows after the first NaN row are not computed (they stay 0)
    for i in stages:
        if i >= last:
            continue
        dq = (grid[i] - grid[i - 1]) if i > 0 else (grid[N] - grid[N - 1])
        box = (max(L[i, 0], xb[i, 0]), min(L[i, 1], ECOS_MAXX, xb[i, 1]))
        xn = (grid[i + 1] - grid[i], -ECOS_INFTY if np.isnan(X[i + 1, 0]) else X[i + 1, 0],
              ECOS_INFTY if np.isnan(X[i + 1, 1]) else X[i + 1, 1])
        st = stage(rows, conic, ell, i, box, xn)
        for end, sign in ((1, -1.0), (0, +1.0)):
            got = L[i + 1, end]
            ref = st.socp((sign * 2 * dq, sign * 1.0), None)
            if ref is None:
                assert np.isnan(got), "%s stage %d: infeasible, got %r" % (what, i, got)
                continue
            assert not np.isnan(got), "%s stage %d: NaN, the reference finds %s" % (what, i, ref)
            val = sign * ref["obj"]
            if end == 0 and val < 0:
                val = mpf(0)
            err = abs(mpf(float(got)) - val)
            tol = TOL_X * (abs(val) + mpf("1e-300"))
            if err > tol:
                tol = TOL_X * (abs(ref["x"]) + abs(2 * mpf(float(dq)) * ref["u"]) + mpf("1e-300"))
            assert err <= tol, "%s stage %d end %d: got %r, 50-digit %s (allowed %.3g)" % (what, i, end, got, val,
                                                                                           float(tol))
            worst.add("L_hi" if end else "L_lo", got, val)


def _cfg4_restatement_case(seed, grid, interp, ell):
    rows, xb = _cfg4_on(seed, grid, interp)
    R = rows.shape[2]
    X = orc.feasible_rows_robust(rows, xb, grid, 0, R, ell)
    return rows, xb, R, X


@pytest.mark.parametrize("scale,interp,uniform", [(0.5, True, True), (1.0, True, False), (3.0, True, True),
                                                  (0.5, False, False), (1.0, False, True), (3.0, False, False)])
def test_restatement_cfg4_against_50_digits(scale, interp, uniform, capsys):
    ell = [scale * e for e in ELL]
    seed = 3100 + int(2 * scale) + (0 if interp else 10)
    G = 120
    grid = np.linspace(0, 1, G) if uniform else _nonuniform(G, seed)
    rows, xb, R, X = _cfg4_restatement_case(seed, grid, interp, ell)
    conic = np.ones(R, bool)
    worst = Worst()
    N = G - 1
    # reachable sets from rest and from a velocity range (the box of stage 0 is then an interval)
    for s0, s1 in ((0.0, 0.0), (0.0, 0.5 * np.sqrt(X[0, 1]))):
        L, fs = rro.reachable_sets_robust(rows, xb, grid, 0, R, ell, X, s0, s1)
        assert fs == -1 and not np.isnan(L).any()
        check_L(rows, xb, grid, conic, ell, X, L, [0, 1, N // 2, N - 1], worst, what="L(%g, %g)" % (s0, s1))
    # controllable sets from a velocity range at the end: both ends, where the upper end of K[N] binds
    K, status, fs = rro.controllable_sets_robust(rows, xb, grid, 0, R, ell, 0.05, 0.6)
    assert status == 0 and fs == -1 and K[N, 0] == 0.05 ** 2 and K[N, 1] == 0.6 ** 2
    check_K(rows, xb, grid, conic, ell, K, [0, N // 2, N - 3, N - 2, N - 1], worst, what="K(0.05, 0.6)")
    worst.report(capsys, "cfg4 scale %g %s %s grid" % (scale, "interpolation" if interp else "collocation",
                                                       "uniform" if uniform else "non-uniform"))


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_restatement_edge_catalogue(case, capsys):
    rows, xb, (c0, cn), canon, cmask = layout(case)
    ell = list(case["ell"])
    grid = np.linspace(0, 1, case["G"])
    X = orc.feasible_rows_robust(rows, xb, grid, c0, cn, ell)
    worst = Worst()
    G = case["G"]
    s = case["sd_start"]
    for s0, s1 in ((s, s), (0.0, max(s, 1.0))):
        L, fs = rro.reachable_sets_robust(rows, xb, grid, c0, cn, ell, X, s0, s1)
        nan_rows = [i for i in range(G) if np.isnan(L[i]).any()]
        assert fs == (nan_rows[0] if nan_rows else -1)
        if nan_rows:
            assert (L[nan_rows[0] + 1:] == 0).all()
        check_L(canon, xb, grid, cmask, ell, X, L, range(G - 1), worst, what="%s L(%g, %g)" % (case["name"], s0, s1))
    e = case["sd_end"]
    K, status, fs = rro.controllable_sets_robust(rows, xb, grid, c0, cn, ell, e, e + 0.5)
    assert status == (3 if fs >= 0 else 0)
    check_K(canon, xb, grid, cmask, ell, K, range(G - 1), worst, what=case["name"] + " K")
    worst.report(capsys, case["name"])


def test_restatement_velocity_range_equals_point_and_nests():
    """sd_end_hi == sd_end is the existing backward pass (orc_solve_rows_robust) bit for bit; K(range) contains K(point)
    and L(range) contains L(point) for a point inside the range."""
    grid = np.linspace(0, 1, 80)
    rows, xb, R, X = _cfg4_restatement_case(3001, grid, True, ELL)
    for e in (0.0, 0.1):
        K = rro.controllable_sets_robust(rows, xb, grid, 0, R, ELL, e, e)[0]
        assert eq(K, orc.solve_rows_robust(rows, xb, grid, 0, R, ELL, 0.0, e)["K"])
    Kr = rro.controllable_sets_robust(rows, xb, grid, 0, R, ELL, 0.0, 0.3)[0]
    Kp = rro.controllable_sets_robust(rows, xb, grid, 0, R, ELL, 0.1, 0.1)[0]
    assert np.all(Kr[:, 0] <= Kp[:, 0] + 1e-12) and np.all(Kr[:, 1] >= Kp[:, 1] - 1e-12)
    Lr, fr = rro.reachable_sets_robust(rows, xb, grid, 0, R, ELL, X, 0.0, 0.3)
    for p in (0.0, 0.1, 0.2):
        Lp, fp = rro.reachable_sets_robust(rows, xb, grid, 0, R, ELL, X, p, p)
        n = len(grid) if fp < 0 else fp      # a point may be unreachable further on; the range reaches on
        assert fr == -1 and np.all(Lr[:n, 0] <= Lp[:n, 0] + 1e-12) and np.all(Lr[:n, 1] >= Lp[:n, 1] - 1e-12)


# ==== CPU: C-ABI, prototypes, launch plans ===========================================================================
def _gpu_present():
    return torch.cuda.is_available()


def _header_protos(path, prefix):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", path)).read(), flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(%s[a-z0-9_]+)\s*\(([^)]*)\)\s*;" % prefix, text):
        out[name] = [("ptr" if "*" in a else ("double" if "double" in a else "int"))
                     for a in (x.strip() for x in args.split(",")) if a not in ("", "void")]
    return out


REACH_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_reach.so")


def test_new_prototypes_match_the_headers():
    from toppra_b200 import _lib, _lib_reach
    kind = {ctypes.c_int: "int", ctypes.c_double: "double"}
    declared = _header_protos("toppra_b200.h", "tb_")["tb_scan_robust_ex"]
    assert [kind.get(t, "ptr") for t in _lib._PROTOS["tb_scan_robust_ex"][0]] == declared
    # the reach library: every declared entry has a prototype and the reverse
    declared = _header_protos("toppra_b200_reach.h", "tbr_")
    assert set(declared) == set(_lib_reach._PROTOS)
    for name, (argtypes, restype) in _lib_reach._PROTOS.items():
        assert [kind.get(t, "ptr") for t in argtypes] == declared[name], name
        assert restype is ctypes.c_int


def test_reach_library_exports_and_kernel_inventory():
    from test_piecewise_poly import kernel_key
    if not os.path.exists(REACH_LIB):
        pytest.skip("libtoppra_b200_reach.so is not built")
    lib = ctypes.CDLL(REACH_LIB)
    for name in _header_protos("toppra_b200_reach.h", "tbr_"):
        assert hasattr(lib, name), name
    assert lib.tbr_reach_version() == 100
    cuobjdump = os.path.join("/usr/local/cuda", "bin", "cuobjdump")
    cuobjdump = cuobjdump if os.path.exists(cuobjdump) else shutil.which("cuobjdump")
    if not cuobjdump or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not found")
    text = subprocess.run([cuobjdump, "-res-usage", REACH_LIB], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", text, re.M)
    names = subprocess.run([shutil.which("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    assert sorted(kernel_key(n) for n in names) == ["reachable_robust_kernel<%d>" % r for r in (1, 2, 3, 4)]


@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_refusals_of_the_real_libraries():
    """Every refusal comes before any CUDA call: host addresses stand in for device arrays."""
    from toppra_b200 import _lib, _lib_reach
    lib, rlib = _lib.load(), _lib_reach.load()
    mem = np.zeros(1 << 16)
    p = ctypes.c_void_p(mem.ctypes.data)
    ell, neg = np.array([0.1, 0.1, 0.1]), np.array([0.1, -0.1, 0.1])
    E, N_ = ctypes.c_void_p(ell.ctypes.data), ctypes.c_void_p(neg.ctypes.data)

    def reach(**kw):
        a = dict(records=p, W=86, R=28, c0=0, cn=28, ell=E, grid=p, gs=1, B=2, G=9, glen=None, X=p, lo=p, hi=p, L=p, fs=p)
        a.update(kw)
        rc = rlib.tbr_reachable_sets_robust(*a.values(), None)
        return rc, lib.tb_last_error().decode()

    for k in ("records", "grid", "ell", "X", "L"):
        rc, msg = reach(**{k: None})
        assert rc == TB_ERR_ARG and "tbr_reachable_sets_robust" in msg, k
    assert reach(B=0)[0] == TB_ERR_ARG and reach(G=0)[0] == TB_ERR_ARG
    rc, msg = reach(glen=p)
    assert rc == TB_ERR_ARG and "glen" in msg
    assert reach(W=85)[0] == TB_ERR_ALIGN
    rc, msg = reach(cn=29)
    assert rc == TB_ERR_ARG and "conic" in msg
    assert reach(c0=-1)[0] == TB_ERR_ARG
    rc, msg = reach(ell=N_)
    assert rc == TB_ERR_ARG and "ellipsoid" in msg
    assert reach(R=127, W=3 * 127 + 3, cn=1)[0] == TB_ERR_UNSUPPORTED

    def ex(**kw):
        a = dict(records=p, W=86, R=28, c0=0, cn=28, ell=E, grid=p, gs=1, B=2, G=9, glen=None, s0=p, s1=p, s1hi=p,
                 flags=1, K=p, sd=p, u=p, status=p, fs=p, counters=None)
        a.update(kw)
        rc = lib.tb_scan_robust_ex(*a.values(), None)
        return rc, lib.tb_last_error().decode()

    for k in ("records", "grid", "ell", "K", "status"):
        assert ex(**{k: None})[0] == TB_ERR_ARG, k
    assert ex(glen=p)[0] == TB_ERR_ARG and ex(B=0)[0] == TB_ERR_ARG
    assert ex(flags=0, sd=None)[0] == TB_ERR_ARG
    assert ex(W=85)[0] == TB_ERR_ALIGN and ex(cn=29)[0] == TB_ERR_ARG and ex(ell=N_)[0] == TB_ERR_ARG
    assert ex(R=127, W=3 * 127 + 3, cn=1)[0] == TB_ERR_UNSUPPORTED


class _ReachRecorder(object):
    """Stands in for libtoppra_b200_reach.so next to the recording libtoppra_b200.so: calls go to the same list."""

    def __init__(self, rec):
        self.rec = rec

    def __getattr__(self, name):
        from toppra_b200 import _lib_reach
        argtypes, _ = _lib_reach._PROTOS[name]

        def entry(*args):
            assert len(args) == len(argtypes), name
            self.rec.calls.append((name, args))
            return 0
        return entry


@pytest.fixture
def rlib(monkeypatch):
    from test_engine_marshalling import RecordingLib
    import toppra_b200 as ta
    from toppra_b200 import _lib, _lib_reach, engine
    rec = RecordingLib()
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(_lib_reach, "load", lambda: _ReachRecorder(rec))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: __import__("contextlib").nullcontext())
    monkeypatch.setattr(engine, "default_device", lambda device=None: torch.device("cpu"))
    return rec, ta


SIZE_QUERIES = ("tb_record_doubles", "tb_spline_fit_workspace_doubles")


def _launches(rec, mark):
    return [n for n, _ in rec.calls[mark:] if n not in SIZE_QUERIES]


def _robust_problem(ta, B=8, G=50, dof=6, ragged=False):
    rng = np.random.RandomState(0)
    path = ta.BatchSplineInterpolator(np.linspace(0, 1, 5), rng.randn(B, 5, dof))
    lim = np.tile(np.array([[-1.0, 1.0]]), (dof, 1))
    acc = ta.constraint.JointAccelerationConstraint(lim)
    cons = [ta.constraint.JointVelocityConstraint(lim), ta.constraint.RobustLinearConstraint(acc, [0.1, 0.1, 0.1], 1)]
    grid = np.linspace(0, 1, G)
    if ragged:
        grid = np.tile(grid, (B, 1))
    return path, cons, grid


def test_launch_plans(rlib):
    rec, ta = rlib
    B, G = 8, 50
    path, cons, grid = _robust_problem(ta, B, G)
    inst = ta.BatchTOPPRA(cons, path, gridpoints=grid)
    inst.setup()
    # reachable sets: one feasible-set launch (TB_SCAN_FEASIBLE_SETS), one forward launch
    mark = len(rec.calls)
    inst.compute_reachable_sets(0.0, np.linspace(0, 1, B))
    assert _launches(rec, mark) == ["tb_scan_robust", "tbr_reachable_sets_robust"]
    assert rec.last("tb_scan_robust")[12] == 2
    args = rec.last("tbr_reachable_sets_robust")
    assert args[8] == B and args[10] is None and args[13] is not None   # B, glen NULL, sdmax
    # controllable sets over a velocity range: one tb_scan_robust_ex launch, backward only
    mark = len(rec.calls)
    inst.compute_controllable_sets(0.0, 0.5)
    assert _launches(rec, mark) == ["tb_scan_robust_ex"]
    ex = rec.last("tb_scan_robust_ex")
    assert ex[13] is not None and ex[14] == 1                          # sd_end_hi, TB_SCAN_BACKWARD_ONLY
    # sdmin == sdmax: today's plan, no sd_end_hi
    mark = len(rec.calls)
    inst.compute_controllable_sets(0.3, 0.3)
    assert _launches(rec, mark) == ["tb_scan_robust"]
    # record chunks of 3, 3, 2 paths: the same launches per chunk
    per_path = 8 * ta.engine.record_doubles(inst.R) * G
    small = ta.BatchTOPPRA(cons, path, gridpoints=grid, max_record_bytes=3 * per_path)
    mark = len(rec.calls)
    small.compute_reachable_sets(0.0, 0.0)
    plan = [n for n in _launches(rec, mark) if n in ("tb_scan_robust", "tbr_reachable_sets_robust")]
    assert plan == ["tb_scan_robust", "tbr_reachable_sets_robust"] * 3
    assert [a[8] for n, a in rec.calls[mark:] if n == "tbr_reachable_sets_robust"] == [3, 3, 2]
    mark = len(rec.calls)
    small.compute_controllable_sets(0.0, 0.5)
    assert [a[8] for n, a in rec.calls[mark:] if n == "tb_scan_robust_ex"] == [3, 3, 2]
    assert "tb_scan_robust" not in _launches(rec, mark)


def test_launch_plans_ragged_refused_and_single_path(rlib):
    rec, ta = rlib
    B, G = 4, 30
    path, cons, grid = _robust_problem(ta, B, G, ragged=True)
    glen = np.array([30, 20, 25, 30], dtype=np.int32)
    inst = ta.BatchTOPPRA(cons, path, gridpoints=grid, glen=glen, validate=False)
    inst.setup()
    # per-path grids: the batched class refuses both before any launch; sdmin == sdmax keeps its ragged scan
    mark = len(rec.calls)
    with pytest.raises(NotImplementedError):
        inst.compute_reachable_sets(0.0, 0.0)
    with pytest.raises(NotImplementedError):
        inst.compute_controllable_sets(0.0, 0.5)
    assert _launches(rec, mark) == []
    inst.compute_controllable_sets(0.5, 0.5)
    assert _launches(rec, mark) == ["tb_scan_robust_ragged"]
    # single-path TOPPRA: the same routes with B = 1
    rng = np.random.RandomState(1)
    lim = np.tile(np.array([[-1.0, 1.0]]), (3, 1))
    acc = ta.constraint.JointAccelerationConstraint(lim)
    one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(lim),
                               ta.constraint.RobustLinearConstraint(acc, [0.1, 0.1, 0.1], 1)],
                              ta.SplineInterpolator(np.linspace(0, 1, 4), rng.randn(4, 3)),
                              gridpoints=np.linspace(0, 1, 20), solver_wrapper="ecos")
    mark = len(rec.calls)
    one.solver_wrapper.reachable_sets(0.0, 0.2)        # (the recorded outputs are not results)
    assert _launches(rec, mark) == ["tb_scan_robust", "tbr_reachable_sets_robust"]
    assert rec.last("tbr_reachable_sets_robust")[8] == 1
    mark = len(rec.calls)
    one.compute_controllable_sets(0.0, 0.2)
    assert _launches(rec, mark) == ["tb_scan_robust_ex"]
    mark = len(rec.calls)
    one.compute_controllable_sets(0.2, 0.2)
    assert _launches(rec, mark) == ["tb_scan_robust"]


# ==== GPU: kernels against the restatement, bit for bit ==============================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _host_rows(rec, R, b, n):
    h = rec[b, :n].cpu().numpy()
    return h[:, :3 * R].reshape(n, 3, R), h[:, 3 * R:3 * R + 2]


def _failing(rec, R):
    """Path 0: no stage feasible; path 1: stages 10.. infeasible (the forward recursion fails there)."""
    rec[0, :, 2 * R:3 * R] = -1e-4
    rec[1, 10:, 2 * R:3 * R] = -1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("rpl,ragged", [(1, False), (2, False), (3, False), (4, False), (1, True), (3, True)])
def test_gpu_reachable_sets_equal_restatement(ta, rpl, ragged):
    B, G = 16, 60
    rec, R, grid, glen = _widened_records(ta, rpl, B, G, ragged=ragged)
    _failing(rec, R)
    dev = rec.device
    sdmin = torch.zeros(B, dtype=torch.float64, device=dev)
    sdmax = torch.linspace(0, 0.3, B, dtype=torch.float64, device=dev)
    sdmin[2], sdmax[2] = 100.0, 100.0          # path 2: the start lies outside every stage's box
    sdmin[3] = 0.05
    kw = {} if glen is None else {"glen": glen}
    out = ta.engine.reachable_sets_robust(rec, R, 0, 28, ELL, grid, sdmin, sdmax, **kw)
    L, X, fs = (out[k].cpu().numpy() for k in ("L", "X", "fail_stage"))
    gr, s0, s1 = grid.cpu().numpy(), sdmin.cpu().numpy(), sdmax.cpu().numpy()
    for b in range(B):
        n = G if glen is None else int(glen[b])
        rows, xb = _host_rows(rec, R, b, n)
        g = gr if gr.ndim == 1 else gr[b]
        Xo = orc.feasible_rows_robust(rows, xb, g[:n], 0, 28, ELL)
        assert eq(X[b, :n], Xo) and np.isnan(X[b, n:]).all()
        Lo, fo = rro.reachable_sets_robust(rows, xb, g[:n], 0, 28, ELL, Xo, s0[b], s1[b])
        assert eq(L[b, :n], Lo), b
        assert np.isnan(L[b, n:]).all() and fs[b] == fo, (b, fs[b], fo)
    assert fs[0] == 1 and fs[1] == 11 and fs[2] == 1 and (fs[3:] == -1).all()
    assert (L[0, 2:(G if glen is None else int(glen[0]))] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rpl,ragged", [(1, False), (2, False), (3, False), (4, False), (2, True)])
def test_gpu_velocity_range_scan_equals_restatement(ta, rpl, ragged):
    B, G = 16, 60
    rec, R, grid, glen = _widened_records(ta, rpl, B, G, ragged=ragged)
    _failing(rec, R)
    dev = rec.device
    lo = torch.linspace(0, 0.1, B, dtype=torch.float64, device=dev)
    hi = lo + torch.linspace(0, 0.8, B, dtype=torch.float64, device=dev)
    kw = {} if glen is None else {"glen": glen}
    out = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, None, lo, backward_only=True, sd_end_hi=hi, **kw)
    K, st, fs = (out[k].cpu().numpy() for k in ("K", "status", "fail_stage"))
    gr, l, h = grid.cpu().numpy(), lo.cpu().numpy(), hi.cpu().numpy()
    for b in range(B):
        n = G if glen is None else int(glen[b])
        rows, xb = _host_rows(rec, R, b, n)
        g = gr if gr.ndim == 1 else gr[b]
        Ko, so, fo = rro.controllable_sets_robust(rows, xb, g[:n], 0, 28, ELL, l[b], h[b])
        assert eq(K[b, :n], Ko) and np.isnan(K[b, n:]).all(), b
        assert st[b] == so and fs[b] == fo, (b, st[b], so, fs[b], fo)
    assert st[0] == 3 and st[1] == 3 and (st[2:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 3])
def test_gpu_scan_robust_ex_with_point_or_null_equals_existing_entries(ta, rpl):
    from toppra_b200 import _lib
    B, G = 12, 50
    rec, R, grid, _ = _widened_records(ta, rpl, B, G)
    _failing(rec, R)
    dev = rec.device
    s0 = torch.linspace(0, 0.05, B, dtype=torch.float64, device=dev)
    s1 = torch.linspace(0, 0.2, B, dtype=torch.float64, device=dev)
    keys = ("K", "sd", "u", "status", "fail_stage", "counters")
    for backward_only in (False, True):
        base = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, s0, s1, backward_only, counters=True)
        same = ta.engine.scan_robust(rec, R, 0, 28, ELL, grid, s0, s1, backward_only, counters=True, sd_end_hi=s1)
        for k in keys:
            if base[k] is not None:
                assert same_bits(base[k], same[k]), (backward_only, k)
        # NULL sd_end_hi through the new entry, with glen = all gridpoints: tb_scan_robust_ragged's results
        gB = grid.expand(B, G).contiguous()
        glen = torch.full((B,), G, dtype=torch.int32, device=dev)
        ragged = ta.engine.scan_robust(rec, R, 0, 28, ELL, gB, s0, s1, backward_only, counters=True, glen=glen)
        out, u_arg = ta.engine._scan_outputs(B, G, dev, backward_only, True)
        ell = np.ascontiguousarray(ELL, dtype=np.float64)
        rc = _lib.load().tb_scan_robust_ex(
            _lib.ptr(rec), rec.shape[2], R, 0, 28, ctypes.c_void_p(ell.ctypes.data), _lib.ptr(gB), 0, B, G,
            _lib.ptr(glen), _lib.ptr(s0), _lib.ptr(s1), None, 1 if backward_only else 0, _lib.ptr(out["K"]),
            _lib.ptr(out["sd"]), _lib.ptr(u_arg), _lib.ptr(out["status"]), _lib.ptr(out["fail_stage"]),
            _lib.ptr(out["counters"]), _lib.stream_ptr())
        _lib.check(rc, "tb_scan_robust_ex")
        for k in keys:
            if base[k] is not None:
                assert same_bits(ragged[k], out[k]) and same_bits(base[k], out[k]), (backward_only, k)


@pytest.mark.gpu
def test_gpu_reachable_builds_run(ta):
    from test_piecewise_poly import launched
    want = {"reachable_robust_kernel<%d>" % r for r in (1, 2, 3, 4)}
    names = set()
    for _ in range(3):
        with launched() as got:
            for rpl in (1, 2, 3, 4):
                rec, R, grid, _ = _widened_records(ta, rpl, 2, 12)
                ta.engine.reachable_sets_robust(rec, R, 0, 28, ELL, grid)
        names |= got
        if want <= names:   # kineto now and then returns a capture without device activity
            break
    assert want <= names, sorted(names)


# ==== GPU: the public API ============================================================================================
def _cons(ta, vlim, alim, ell):
    acc = ta.constraint.JointAccelerationConstraint(alim)
    return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.RobustLinearConstraint(acc, ell, 1)]


def _sets(inst, lo, hi):
    L, X, fs = inst.compute_reachable_sets(lo, hi)
    K, st = inst.compute_controllable_sets(lo, hi)
    return [t.cpu().numpy() for t in (L, X, fs, K, st)]


@pytest.mark.gpu
def test_gpu_chunked_and_single_path_equal(ta):
    B, G = 10, 70
    ss, way, vlim, alim = make_batch(B, 3040)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    cons = _cons(ta, vlim, alim, ELL)
    lo, hi = np.zeros(B), np.linspace(0.0, 0.6, B)
    lo[4] = hi[4] = 1000.0                    # x = 1e6 > ECOS_MAXX: the box of stage 0 is empty, the recursion fails
    whole = ta.BatchTOPPRA(cons, path, grid)
    w = _sets(whole, lo, hi)
    assert w[2][4] == 1 and (np.delete(w[2], 4) == -1).all()
    per_path = 8 * ta.engine.record_doubles(whole.R) * G
    chunked = ta.BatchTOPPRA(cons, path, grid, max_record_bytes=3 * per_path)
    assert chunked.record_chunk_size() == 3
    for x, y in zip(w, _sets(chunked, lo, hi)):
        assert eq(x, y)
    # scalars broadcast to every path
    Ls = whole.compute_reachable_sets(0.0, 0.3)[0].cpu().numpy()
    assert eq(Ls, whole.compute_reachable_sets(np.zeros(B), np.full(B, 0.3))[0].cpu().numpy())
    # single-path TOPPRA (solver_wrapper="ecos" maps to these kernels) == the batch's row
    for b in (0, 4, 7):
        one = ta.algorithm.TOPPRA(_cons(ta, vlim[b], alim[b], ELL), ta.SplineInterpolator(ss, way[b]),
                                  gridpoints=grid, solver_wrapper="ecos")
        L1 = one.compute_reachable_sets(lo[b], hi[b])
        assert eq(L1, w[0][b]) and eq(one.problem_data.X, w[1][b])
        assert eq(one.compute_controllable_sets(lo[b], hi[b]), w[3][b])
    # BatchTOPPRAsd inherits both
    sd = ta.BatchTOPPRAsd(cons, path, grid)
    for x, y in zip(w, _sets(sd, lo, hi)):
        assert eq(x, y)


@pytest.mark.gpu
def test_gpu_zero_ellipsoid_equals_linear(ta):
    """A zero ellipsoid: L and K(sdmin, sdmax) equal the linear kernels' within 1e-9; NaN / zero pattern and fail_stage
    exactly.  Non-uniform per-path grids, so that delta' = deltas[i - 1] differs from deltas[i]."""
    B, G = 24, 90
    ss, way, vlim, alim = make_batch(B, 3050)
    grid = np.stack([_nonuniform(G, 7 + b) for b in range(B)])
    path = ta.BatchSplineInterpolator(ss, way)
    lin = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                         path, grid, fused=False)
    rob = ta.BatchTOPPRA(_cons(ta, vlim, alim, [0.0, 0.0, 0.0]), path, grid)
    rob.setup()
    lo, hi = np.zeros(B), np.linspace(0.0, 0.5, B)
    # path 3 starts above its own velocity bound (and below ECOS_MAXX): both recursions fail at stage 0
    xb_hi = float(rob.records[3, 0, 3 * rob.R + 1])
    assert xb_hi < 4e3
    lo[3] = hi[3] = np.sqrt(2 * xb_hi)
    L, X, fs, _, _ = _sets(rob, lo, hi)
    Ll, Xl, fsl, _, _ = _sets(lin, lo, hi)
    assert eq(fs, fsl) and fs[3] == 1 and (np.delete(fs, 3) == -1).all()
    assert (L[3, 2:] == 0).all() and (Ll[3, 2:] == 0).all()
    for a, b in ((L, Ll), (X, Xl)):
        assert eq(np.isnan(a), np.isnan(b))
        np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-9)
    lo[3], hi[3] = 0.0, 0.2
    for lo_, hi_ in ((lo, hi), (0.0, 0.0)):
        K, st = (t.cpu().numpy() for t in rob.compute_controllable_sets(lo_, hi_))
        Kl, stl = (t.cpu().numpy() for t in lin.compute_controllable_sets(lo_, hi_))
        assert eq(st, stl) and eq(np.isnan(K), np.isnan(Kl))
        np.testing.assert_allclose(K, Kl, rtol=1e-9, atol=1e-9)


@pytest.mark.gpu
def test_gpu_sets_nest(ta):
    B, G = 16, 80
    ss, way, vlim, alim = make_batch(B, 3060)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    tol = lambda v: 1e-9 * (1 + np.abs(v))   # noqa: E731
    prev = None
    for scale in (0.5, 1.0, 3.0):
        inst = ta.BatchTOPPRA(_cons(ta, vlim, alim, [scale * e for e in ELL]), path, grid)
        L, X, fs, K, st = _sets(inst, 0.0, 0.4)
        assert (fs == -1).all() and (st == 0).all()
        # L[1:] lies within X (uniform grid: delta' = delta), the lower end clamped at 0 as X's; L[0] is the given range
        Li, Xi = L[:, 1:], X[:, 1:]
        assert np.all(Li[..., 1] <= Xi[..., 1] + tol(Xi[..., 1])) and np.all(Li[..., 0] >= Xi[..., 0] - tol(Xi[..., 0]))
        if prev is not None:   # a larger ellipsoid: smaller sets
            for now, before in ((L, prev[0]), (K, prev[1])):
                assert np.all(now[..., 1] <= before[..., 1] + tol(before[..., 1]))
                assert np.all(now[..., 0] >= before[..., 0] - tol(before[..., 0]))
            assert np.any(L[..., 1] < prev[0][..., 1]) and np.any(K[..., 1] < prev[1][..., 1])
        prev = (L, K)
        # a range contains a point inside it
        Lp, _, fp, Kp, sp = _sets(inst, 0.2, 0.2)
        rows = np.arange(G)[None, :]
        # a point may become unreachable (or uncontrollable) where the range is not: compare the rows it computed
        live_L = (fp[:, None] < 0) | (rows < fp[:, None])
        live_K = np.repeat((sp == 0)[:, None], G, axis=1)
        assert live_L.sum() > G and live_K.sum() > G
        for rng_, pt, live in ((L, Lp, live_L), (K, Kp, live_K)):
            assert np.all((rng_[..., 0] <= pt[..., 0] + tol(pt[..., 0]))[live])
            assert np.all((rng_[..., 1] >= pt[..., 1] - tol(pt[..., 1]))[live])
        # a parameterisation from a to b lies within L(a, a) and K(b, b)
        K0 = inst.compute_controllable_sets(0.0, 0.0)[0].cpu().numpy()
        for a, b in ((0.0, 0.0), (0.3 * np.sqrt(K0[:, 0, 1]), 0.05)):   # a: a start every path can take
            res = inst.compute_parameterization(a, b)
            assert not res.status.any()
            x = res.sd.cpu().numpy() ** 2
            La, _, fa, _, _ = _sets(inst, a, a)
            Kb, sb = (t.cpu().numpy() for t in inst.compute_controllable_sets(b, b))
            assert (fa == -1).all() and (sb == 0).all()
            for S in (La, Kb):
                assert np.all(x >= S[..., 0] - tol(S[..., 0])) and np.all(x <= S[..., 1] + tol(S[..., 1]))


@pytest.mark.gpu
def test_gpu_reference_robust_example_problem(tmp_path):
    """The problem of the reference's examples/plot_robust_kinematics.py (seed 9, 7 DOF, N = 100, ellipsoid (1e-3, 5e-2,
    9e-3), interpolation), run under `import toppra` as the drop-in suite runs it: compute_reachable_sets(0, 0) and
    compute_controllable_sets(0, 1) return finite, well-formed sets."""
    script = """
import sys, numpy as np
sys.path[:0] = [%r, %r]
import os
os.environ["TB_REF_SUITE_ENGINE"] = "gpu"
import ref_suite_plugin  # noqa: F401
import toppra as ta
import toppra.constraint as constraint
import toppra.algorithm as algo
np.random.seed(9)
way_pts = np.random.randn(5, 7)
vlim_ = np.random.rand(7) * 20
alim_ = np.random.rand(7) * 2
path = ta.SplineInterpolator(np.linspace(0, 1, 5), way_pts)
pc_vel = constraint.JointVelocityConstraint(np.vstack((-vlim_, vlim_)).T)
pc_acc = constraint.JointAccelerationConstraint(np.vstack((-alim_, alim_)).T,
                                                discretization_scheme=constraint.DiscretizationType.Interpolation)
robust = constraint.RobustLinearConstraint(pc_acc, [1e-3, 5e-2, 9e-3], 1)
inst = algo.TOPPRA([pc_vel, robust], path, gridpoints=np.linspace(0, 1, 101), solver_wrapper="ecos")
X = inst.compute_feasible_sets()
L = inst.compute_reachable_sets(0, 0)
K = inst.compute_controllable_sets(0, 1)
np.savez(%r, X=X, L=L, K=K)
""" % (ROOT, os.path.join(ROOT, "tests"), str(tmp_path / "out.npz"))
    proc = subprocess.run([sys.executable, "-c", script], cwd=ROOT, capture_output=True, text=True, timeout=600,
                          env=dict(os.environ, PYTHONDONTWRITEBYTECODE="1"))
    assert proc.returncode == 0, proc.stderr[-3000:]
    o = np.load(str(tmp_path / "out.npz"))
    X, L, K = o["X"], o["L"], o["K"]
    assert L.shape == K.shape == (101, 2)
    for S in (L, K):
        assert np.isfinite(S).all() and np.all(S[:, 0] >= 0) and np.all(S[:, 0] <= S[:, 1])
    assert L[0].tolist() == [0.0, 0.0] and K[-1].tolist() == [0.0, 1.0]
    # L[0] and K[N] are the given ranges; every other row lies within the feasible sets
    assert np.all(L[1:, 1] > 0) and np.all(L[1:, 1] <= X[1:, 1] + 1e-9) and np.all(K[:-1, 1] <= X[:-1, 1] + 1e-9)
