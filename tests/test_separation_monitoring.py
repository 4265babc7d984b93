"""Speed and separation monitoring next to people: surface separations and approach speeds of robot points and human
spheres (RigidBodyModel.separation / separation_terms, SeparationMonitoringConstraint; libtoppra_b200_dyn.so:
tbd_separation, tbd_separation_terms).

CPU:
  * the float64 numpy double of tests/separation_ref.py equals the 50-digit reference (kin_ref.mp_frames on the RAW URDF
    tree) on every link frame of both fixtures: d and w to 1e-13 of the scale, vmax to 1e-13 (1 + vmax) plus
    |dvmax/dD| 1e-15 (|d| + C + v_h T_r);
  * hand cases with closed forms (a prismatic arm moving straight at a sphere, tangent motion, l == 0, D <= 0,
    a_s T_r >> v_h) on the numpy double;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library; the launch plan of the device route on the recording
    libraries (one tbd_separation_terms launch per batch or chunk, per-path spheres sliced, then tb_rows_canlinear).
GPU:
  * both kernels on random trees (1 to 16 bodies) and on the fixtures against the 50-digit reference;
  * the hand cases; tbd_separation_terms equals tbd_separation and the documented torch operations bit for bit; NaN
    isolation; invariances (reference-frame field; moving every sphere away never tightens a row);
  * the reference golden (tests/golden/separation_monitoring.npz, make_golden_separation.py) and 256 paths with per-path
    spheres against the oracle fed with rows from the numpy double, within |dK| <= 1e-9 + 1e-8 |K| (the cfg-3
    tolerance); w sd <= vmax on the solved profiles, and the limit is active;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, host vs device route, path b of a
    batch vs a single-path solve with humans[b]: bit-equal; BatchTOPPRAsd, a quintic BatchPiecewisePolyPath, and the
    constraint next to torque and collision-energy limits against the oracle;
  * one path against 1024 human hypotheses along a ray: durations non-increasing as the person moves away."""
import ctypes
import os

import numpy as np
import pytest

import kin_ref as kr
import rnea_ref as rr
import separation_ref as sr
from dyn_common import (CASES, DYN_LIB, LOCKED, OFFSET, TB_ERR_ARG, TB_ERR_UNSUPPORTED, FakePath, model_of, urdf,
                        _assert_solution, _dev, _dyn_header, _eq, _gpu_present, _model_from_packed, _offset_spec,
                        _oracle_joint_rows, _oracle_rows, _problems)
from test_dyn_calls import H, T, _context, _run, _rows_call, arm, calls  # noqa: F401  (fixtures)

PARAMS = (0.1, 2.5, 1.6, 0.05)            # T_r, a_s, v_h, C


def _pts(m, spec):
    """spec: [(link, offset dict or None, radius)] -> packed points."""
    from toppra_b200.dynamics import pack_points
    return pack_points([(m.frame(link, **(off or {})), r) for link, off, r in spec])[1]


def _humans(rng, H, center=(0.3, 0.0, 0.5), spread=0.8):
    c = np.asarray(center) + rng.uniform(-spread, spread, (H, 3))
    return np.concatenate((c, rng.uniform(0.0, 0.2, (H, 1))), axis=1)


def _mp_pairs(mp, q, qd, spec, humans, packed=False):
    """50-digit (d, w) (P, H) as mp values; `packed`: mp is MpRobot.from_packed, whose link k is "b<k>"."""
    name = (lambda link: "b" + link[4:]) if packed else (lambda link: link)
    st = sr.mp_points(mp, q, qd, {j: (name(link), *_offset_spec(off)) for j, (link, off, _) in enumerate(spec)})
    return [[sr.mp_pair(st[j][0], st[j][1], spec[j][2], h) for h in humans] for j in range(len(spec))]


def _check_vs_mp(d, w, vm, pairs, params, tol=1e-13):
    """Errors of d, w and vmax against the 50-digit pairs; returns the worst scaled error."""
    Tr, a_s, vh, C = params
    dm = np.array([[float(p[0]) for p in row] for row in pairs])
    wm = np.array([[float(p[1]) for p in row] for row in pairs])
    vmm = np.array([[float(sr.mp_vmax(p[0], *params)) for p in row] for row in pairs])
    scale_d = max(1.0, np.abs(dm).max())
    scale_w = max(1.0, np.abs(wm).max())
    worst = max(np.abs(d - dm).max() / scale_d, np.abs(w - wm).max() / scale_w)
    k = a_s * Tr + vh
    D = dm - C - vh * Tr
    dv = np.where(D > 0, a_s / np.sqrt(k * k + 2 * a_s * np.maximum(D, 0)), 0.0)     # |dvmax/dD|
    bound = tol * (1 + vmm) + dv * 1e-15 * (np.abs(dm) + C + vh * Tr)
    assert (np.abs(d - dm) <= tol * scale_d).all() and (np.abs(w - wm) <= tol * scale_w).all(), worst
    assert (np.abs(vm - vmm) <= bound).all(), np.max(np.abs(vm - vmm) - bound)
    return worst


# ==== CPU ============================================================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 301)
    links = list(m.frames)
    spec = [(link, OFFSET if j % 2 else None, 0.01 * j) for j, link in enumerate(links)][:16]
    pts = _pts(m, spec)
    worst = 0.0
    for _ in range(2):
        q, qs = rng.uniform(-2, 2, m.nv), rng.uniform(-1.5, 1.5, m.nv)
        hum = _humans(rng, 3)
        d, w = (x[0] for x in sr.separation_packed(m.packed, pts, hum, q, qs))
        vm = sr.vmax_np(d, *PARAMS)
        worst = max(worst, _check_vs_mp(d, w, vm, _mp_pairs(mp, q, qs, spec, hum), PARAMS))
    print("worst scaled error of the numpy double: %.2e" % worst)


def _prismatic_arm(ta):
    """One prismatic body along x: the point moves at q' along x."""
    return ta.RigidBodyModel([-1], ["prismatic"], [[1.0, 0.0, 0.0]], [np.eye(3)], [[0.0, 0.0, 0.0]], [1.0],
                             [[0.0, 0.0, 0.0]], [[0.01, 0.0, 0.0, 0.01, 0.0, 0.01]])


def _hand_cases(ta, sep, terms):
    """sep(model, points, humans, q, qd) -> (d, w) (M, P, H); terms(model, points, humans, params, q, qs) -> (b, c)."""
    m = _prismatic_arm(ta)
    pts = _pts(m, [("body0", None, 0.1)])
    q = np.array([[0.0], [0.5], [1.0]])
    qs = np.array([[2.0], [2.0], [-1.0]])
    hum = np.array([[3.0, 0.0, 0.0, 0.4]])
    # straight at the sphere: d = 3 - q - 0.5, w = q'
    d, w = sep(m, pts, hum, q, qs)
    np.testing.assert_allclose(d[:, 0, 0], 3.0 - q[:, 0] - 0.5, rtol=0, atol=1e-15)
    np.testing.assert_array_equal(w[:, 0, 0], qs[:, 0])
    b, c = terms(m, pts, hum, PARAMS, q, qs)
    Tr, a_s, vh, C = PARAMS
    D = 3.0 - q[:2, 0] - 0.5 - C - vh * Tr
    vm = a_s * (-(Tr + vh / a_s) + np.sqrt((Tr + vh / a_s) ** 2 + 2 * D / a_s))
    np.testing.assert_allclose(b[:2], 4.0, rtol=0, atol=0)
    np.testing.assert_allclose(-c[:2], vm ** 2, rtol=1e-14)
    assert b[2] == 0.0 and c[2] == -1.0                          # moving away: inactive
    # tangent motion: w = 0, inactive
    hum_t = np.array([[0.5, 1.0, 0.0, 0.1]])
    d, w = sep(m, pts, hum_t, np.array([[0.5]]), np.array([[1.5]]))
    assert w[0, 0, 0] == 0.0
    b, c = terms(m, pts, hum_t, PARAMS, np.array([[0.5]]), np.array([[1.5]]))
    assert b[0] == 0.0 and c[0] == -1.0
    # l == 0: w = |v|, d = -r_p - r_h, D <= 0: vmax = 0, the row stops the point (x = 0)
    hum0 = np.array([[0.25, 0.0, 0.0, 0.05]])
    d, w = sep(m, pts, hum0, np.array([[0.25]]), np.array([[-3.0]]))
    assert w[0, 0, 0] == 3.0 and d[0, 0, 0] == 0.0 - 0.1 - 0.05
    b, c = terms(m, pts, hum0, PARAMS, np.array([[0.25]]), np.array([[-3.0]]))
    assert b[0] == 9.0 and c[0] == 0.0 and not np.signbit(c[0])
    # a_s T_r >> v_h: the difference sqrt(k^2 + 2 a_s D) - k cancels; the rationalised form keeps full precision
    params = (2.0, 50.0, 1e-3, 0.0)
    b, c = terms(m, pts, hum, params, np.array([[0.0]]), np.array([[1.0]]))
    Tr, a_s, vh, C = params
    D = 2.5 - vh * Tr
    k = a_s * Tr + vh
    want = 2 * a_s * D / (np.sqrt(k * k + 2 * a_s * D) + k)
    import mpmath
    with mpmath.workdps(50):
        wmp = sr.mp_vmax(mpmath.mpf(2.5), *params)
    assert abs(want - float(wmp)) <= 2e-16 * float(wmp)
    np.testing.assert_allclose(-c[0], float(wmp) ** 2, rtol=1e-15)


def test_hand_cases_numpy_double():
    import toppra_b200 as ta
    _hand_cases(ta, lambda m, p, h, q, qd: sr.separation_packed(m.packed, p, h, q, qd),
                lambda m, p, h, prm, q, qs: sr.rows_packed(m.packed, p, h, prm, q, qs))


def test_value_errors():
    from toppra_b200.constraint import SeparationMonitoringConstraint as SMC
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    hum = np.array([[0.5, 0.0, 0.5, 0.1]])
    good = [(f, 0.05)]
    for bad in ([f], [(lambda q: q, 0.1)], [(f, (0.1, 0.2))], 3.0, [], [(f, 0.1)] * 17):
        with pytest.raises(ValueError, match="points"):
            SMC(bad, hum, 0.1, 2.0)
    with pytest.raises(ValueError, match="same RigidBodyModel"):
        SMC([(f, 0.1), (model_of("arm6.urdf").frame("flange"), 0.1)], hum, 0.1, 2.0)
    for r in (-0.1, np.nan, np.inf):
        with pytest.raises(ValueError, match="radii"):
            SMC([(f, r)], hum, 0.1, 2.0)
    for h in (np.zeros(4), np.zeros((1, 3)), np.zeros((0, 4)), np.zeros((17, 4)), np.zeros((2, 1, 2, 4)),
              [[0, 0, 0, -0.1]], [[np.nan, 0, 0, 0.1]]):
        with pytest.raises(ValueError, match="humans|human spheres"):
            SMC(good, h, 0.1, 2.0)
    for kw in (dict(reaction_time=-0.1), dict(reaction_time=np.nan), dict(stopping_deceleration=0.0),
               dict(stopping_deceleration=np.inf), dict(human_speed=-1.0), dict(clearance=-0.01),
               dict(clearance=np.inf)):
        args = dict(reaction_time=0.1, stopping_deceleration=2.0)
        args.update(kw)
        with pytest.raises(ValueError, match=list(kw)[0]):
            SMC(good, hum, **args)
    c = SMC(good, hum, 0.0, 2.0, human_speed=0.0)                      # zero reaction time and human speed are fine
    grid = np.linspace(0, 1, 10)
    assert c.dof == 6 and c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    assert SMC(good, hum, 0.1, 2.0, discretization_scheme=1).num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 2
    with pytest.raises(ValueError, match="Wrong dimension"):
        c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
    per_path = SMC(good, np.tile(hum, (3, 1, 1)), 0.1, 2.0)
    assert per_path.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    with pytest.raises(ValueError, match=r"expected \(H, 4\) or \(4, H, 4\)"):
        per_path.num_rows(RecordContext(FakePath(4, 6), grid, grid))
    with pytest.raises(ValueError, match="Wrong dimension"):
        c.compute_constraint_params(type("P", (), {"dof": 7})(), grid)
    with pytest.raises(ValueError, match="single path"):
        per_path.compute_constraint_params(type("P", (), {"dof": 6})(), grid)


def test_dyn_header_prototypes_of_separation_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_separation"] == ["ptr", "int", "ptr", "int", "int", "int", "int", "int", "ptr", "ptr", "ptr",
                                          "ptr", "ptr", "ptr"]
    assert declared["tbd_separation_terms"] == ["ptr", "int", "ptr", "int", "int", "int", "int", "double", "double",
                                                "double", "double", "int", "ptr", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert set(declared) == set(_lib_dyn._PROTOS)
    for name in ("tbd_separation", "tbd_separation_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_separation_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good = _pts(m, [("flange", OFFSET, 0.05), ("wrist2", None, 0.06)])

    def rc(model=m.packed, points=good, nv=6, P=2, H=3, NH=1, ppp=0, M=4, params=PARAMS, null=None, which="both"):
        host = [np.ascontiguousarray(x, dtype=np.float64) for x in (model, points)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        sep = [ptr[0], nv, ptr[1], P, H, NH, ppp, M, d, d, d, d, d]
        ter = [ptr[0], nv, ptr[1], P, H, NH, ppp, *params, M, d, d, d, d, d]
        if null is not None:
            (sep if which == "sep" else ter)[null] = None
        out = []
        if which in ("both", "sep"):
            out.append(lib.tbd_separation(*sep, None))
        if which in ("both", "terms"):
            out.append(lib.tbd_separation_terms(*ter, None))
        assert len(set(out)) == 1, out
        assert out[0] == 0 or _lib.load().tb_last_error()
        return out[0]

    for k in (0, 2, 8, 9, 10, 11, 12):
        assert rc(null=k, which="sep") == TB_ERR_ARG
    for k in (0, 2, 12, 13, 14, 15, 16):
        assert rc(null=k, which="terms") == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    for P in (0, 17):
        assert rc(points=np.zeros((max(P, 1), 15)), P=P) == TB_ERR_UNSUPPORTED
    for H_ in (0, 17):
        assert rc(H=H_) == TB_ERR_UNSUPPORTED
    assert b"human spheres" in _lib.load().tb_last_error()
    assert rc(NH=0) == TB_ERR_ARG and rc(ppp=-1) == TB_ERR_ARG
    assert rc(ppp=2, NH=1) == TB_ERR_ARG and rc(ppp=3, NH=1) == TB_ERR_ARG     # M = 4 points read sets 0..1
    assert rc(ppp=2, NH=2) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)         # passes validation, no device here
    assert rc(ppp=4, NH=1) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model) == TB_ERR_ARG
    for j, value in ((0, 6.0), (0, -2.0), (0, 0.5), (5, np.nan), (11, np.inf), (14, -0.1), (14, np.nan),
                     (14, np.inf), (15 + 14, -1.0), (15 + 0, 9.0)):     # bad frames and radii, in either point
        p = good.copy().reshape(-1)
        p[j] = value
        assert rc(points=p) == TB_ERR_ARG
    for params in ((-0.1, 2.5, 1.6, 0.0), (np.nan, 2.5, 1.6, 0.0), (0.1, 0.0, 1.6, 0.0), (0.1, -1.0, 1.6, 0.0),
                   (0.1, np.inf, 1.6, 0.0), (0.1, 2.5, -1.6, 0.0), (0.1, 2.5, np.nan, 0.0), (0.1, 2.5, 1.6, -0.1),
                   (0.1, 2.5, 1.6, np.inf)):
        assert rc(params=params, which="terms") == TB_ERR_ARG
    assert b"stopping_deceleration" in _lib.load().tb_last_error()
    for ref in (0.0, 1.0, 2.0, 7.0):                            # the reference-frame field is ignored
        p = good.copy()
        p[0, 13] = ref
        assert rc(points=p) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
        assert b"launch failed" in _lib.load().tb_last_error()


@pytest.mark.parametrize("lo,hi,total", [(0, 4, 4), (1, 3, 4)])
@pytest.mark.parametrize("interp", [False, True])
@pytest.mark.parametrize("per_path", [False, True])
def test_launch_plan(calls, arm, monkeypatch, lo, hi, total, interp, per_path):  # noqa: F811
    import test_dyn_calls
    from toppra_b200.constraint import SeparationMonitoringConstraint
    monkeypatch.setitem(test_dyn_calls._OUTPUTS, "tbd_separation_terms", 2)     # label the two output slots
    nv, G = arm.nv, 6
    f = arm.frame(sorted(arm.frames)[-1], xyz=(0.0, 0.0, 0.1))
    g = arm.frame("forearm")
    rng = np.random.RandomState(3)
    hum = _humans(rng, 3)
    if per_path:
        hum = np.stack([hum + 0.1 * i for i in range(total)])
    cons = SeparationMonitoringConstraint([(f, 0.05), (g, 0.08)], hum, *PARAMS, discretization_scheme=int(interp))
    ctx, bp = _context(nv, total, G, lo, hi, total)
    B, n = hi - lo, (hi - lo) * G
    rows, log = _run(calls, cons, ctx)
    assert rows == (2 if interp else 1)
    sets = hum[lo:hi] if per_path else hum[None]
    name = "tbd_separation_terms"
    # the recorder copies the first 14 doubles of the points (one packed frame)
    want = [
        [name, H(arm.packed), nv, H(cons.points.reshape(-1)[:14]), 2, 3, sets.shape[0], G if per_path else 0, *PARAMS,
         n, T("q0", (n, nv)), T("q1", (n, nv)), T(tuple(sets.reshape(-1).tolist()), sets.shape),
         T(name + ".15", (n,)), T(name + ".16", (n,)), None],
        _rows_call(T((0.0,) * (B * G), (B, G, 1)), T(name + ".15", (B, G, 1)), T(name + ".16", (B, G, 1)),
                   T((1.0,), (1, 1)), T((0.0,), (1,)), 0, B, G, 1, 1, interp)]
    assert len(log) == len(want)
    for got_call, want_call in zip(log, want):
        assert len(got_call) == len(want_call), got_call[0]
        for slot, (x, y) in enumerate(zip(got_call, want_call)):
            assert x == y, (got_call[0], slot, x, y)


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _sep_dev(m, p, h, q, qd, ppp=0):
    return tuple(x.cpu().numpy() for x in m.separation(p, _dev(h), _dev(q), _dev(qd), ppp))


def _terms_dev(m, p, h, prm, q, qs, ppp=0):
    return tuple(x.cpu().numpy() for x in m.separation_terms(p, _dev(h), *prm, _dev(q), _dev(qs), ppp))


@pytest.mark.gpu
def test_gpu_vs_mp_random_trees_and_fixtures(ta):
    worst = 0.0
    cases = [(_model_from_packed(ta, rr.random_tree(np.random.RandomState(1300 + nv), nv)), None)
             for nv in (1, 2, 3, 5, 8, 12, 16)]
    cases += [(model_of(n, lk), rr.MpRobot.from_urdf(urdf(n), lk)) for n, lk in CASES]
    for m, mp in cases:
        packed = mp is None
        mp = mp or rr.MpRobot.from_packed(m.packed)
        rng = np.random.RandomState(m.nv + 77)
        links = list(m.frames)
        spec = [(link, OFFSET if j % 2 else None, 0.02 * j) for j, link in enumerate(links)][:16]
        pts = _pts(m, spec)
        hum = _humans(rng, 16 if len(spec) <= 8 else 4)
        q, qs = rng.uniform(-2, 2, (2, m.nv)), rng.uniform(-1.5, 1.5, (2, m.nv))
        d, w = _sep_dev(m, pts, hum, q, qs)
        b, c = _terms_dev(m, pts, hum, PARAMS, q, qs)
        for i in range(2):
            pairs = _mp_pairs(mp, q[i], qs[i], spec, hum, packed)
            worst = max(worst, _check_vs_mp(d[i], w[i], sr.vmax_np(d[i], *PARAMS), pairs, PARAMS))
            bm, cm = sr.mp_row([p for row in pairs for p in row], PARAMS)
            assert abs(b[i] - float(bm)) <= 1e-12 * max(1.0, abs(float(bm)))
            assert abs(c[i] - float(cm)) <= 1e-12 * max(1.0, abs(float(cm)))
        # against the numpy double on many points
        Q, QS = rng.uniform(-3, 3, (512, m.nv)), rng.uniform(-2, 2, (512, m.nv))
        d, w = _sep_dev(m, pts, hum, Q, QS)
        dn, wn = sr.separation_packed(m.packed, pts, hum, Q, QS)
        assert np.max(np.abs(d - dn)) <= 1e-12 and np.max(np.abs(w - wn)) <= 1e-12 * max(1.0, np.abs(wn).max())
    print("kernels vs the 50-digit reference: worst scaled error %.2e" % worst)


@pytest.mark.gpu
def test_gpu_hand_cases(ta):
    _hand_cases(ta, _sep_dev, _terms_dev)


def _torch_terms(d, w, params):
    """tbd_separation_terms from the pairs (M, P, H) of tbd_separation, in the documented operation order."""
    import torch
    Tr, a_s, vh, C = params
    vhTr, twoa, k = vh * Tr, 2.0 * a_s, a_s * Tr + vh
    kk = k * k
    M = d.shape[0]
    d, w = d.reshape(M, -1), w.reshape(M, -1)
    bw2 = torch.zeros(M, dtype=torch.float64, device=d.device)
    bv2 = torch.zeros_like(bw2)
    found = torch.zeros(M, dtype=torch.bool, device=d.device)
    bad = torch.zeros_like(found)
    for j in range(d.shape[1]):
        D = d[:, j] - C
        D = D - vhTr
        num = twoa * D
        vmax = torch.where(D <= 0, torch.zeros_like(D), num / (torch.sqrt(kk + num) + k))
        bad = bad | torch.isnan(w[:, j]) | torch.isnan(vmax)
        w2, v2 = w[:, j] * w[:, j], vmax * vmax
        take = (w[:, j] > 0) & (~found | (v2 * bw2 < bv2 * w2))
        bw2, bv2 = torch.where(take, w2, bw2), torch.where(take, v2, bv2)
        found = found | take
    b = torch.where(found, bw2, torch.zeros_like(bw2))
    c = torch.where(found, 0.0 - bv2, torch.full_like(bv2, -1.0))
    nan = torch.full_like(b, float("nan"))
    return torch.where(bad, nan, b), torch.where(bad, nan, c)


@pytest.mark.gpu
def test_gpu_terms_bit_equal_separation_nan_isolation_and_invariances(ta):
    import torch
    m = model_of("arm7_gripper.urdf")
    rng = np.random.RandomState(11)
    M = 3000
    spec = [("finger_left", OFFSET, 0.02), ("camera", None, 0.05), ("hand", OFFSET, 0.08), ("link3", None, 0.1)]
    pts = _pts(m, spec)
    q, qs = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(2))
    hum = _dev(np.stack([_humans(rng, 5, spread=0.6) for _ in range(M // 100)]))
    for params in (PARAMS, (0.0, 3.0, 0.0, 0.0), (0.5, 40.0, 2.0, 0.3)):
        for ppp, h in ((0, hum[0]), (100, hum)):
            d, w = m.separation(pts, h, q, qs, ppp)
            b, c = m.separation_terms(pts, h, *params, q, qs, ppp)
            want = _torch_terms(d, w, params)
            assert torch.equal(b, want[0]) and torch.equal(c, want[1])
            assert (b > 0).any()
    # the reference-frame field makes no difference
    for ref in ("world", "local"):
        from toppra_b200.dynamics import pack_points
        p2 = pack_points([(m.frame(link, reference_frame=ref, **(off or {})), r) for link, off, r in spec])[1]
        assert torch.equal(m.separation_terms(p2, hum, *PARAMS, q, qs, 100)[1],
                           m.separation_terms(pts, hum, *PARAMS, q, qs, 100)[1])
    # moving every sphere's surface away (same centres, so the same w; smaller radii, so larger d) never tightens a row
    b0, c0 = m.separation_terms(pts, hum[0], *PARAMS, q, qs)
    d0, _ = m.separation(pts, hum[0], q, qs)
    x0 = torch.where(b0 > 0, -c0 / b0, torch.full_like(b0, float("inf")))
    for shrink in (0.5, 0.0):
        away = hum[0].clone()
        away[:, 3] = away[:, 3] * shrink
        b2, c2 = m.separation_terms(pts, away, *PARAMS, q, qs)
        x2 = torch.where(b2 > 0, -c2 / b2, torch.full_like(b2, float("inf")))
        assert torch.equal(b2 > 0, b0 > 0) and (x2 >= x0).all() and (x2 > x0).any()
    # NaN in one point leaves every other point as it was
    q2, qs2 = q.clone(), qs.clone()
    q2[5, 2] = float("nan")
    qs2[9, 0] = float("nan")
    bn, cn = m.separation_terms(pts, hum[0], *PARAMS, q2, qs2)
    assert torch.isnan(bn[[5, 9]]).all() and torch.isnan(cn[[5, 9]]).all()
    keep = torch.ones(M, dtype=torch.bool, device="cuda")
    keep[[5, 9]] = False
    assert torch.equal(bn[keep], b0[keep]) and torch.equal(cn[keep], c0[keep])
    dn, wn = m.separation(pts, hum[0], q2, qs2)
    assert torch.isnan(dn[5]).any() and not torch.isnan(dn[keep]).any() and torch.isnan(wn[9]).any()
    # the constraint's separation(): CUDA and numpy
    cons = ta.constraint.SeparationMonitoringConstraint([(m.frame(l, **(o or {})), r) for l, o, r in spec],
                                                       hum[0].cpu().numpy(), *PARAMS)
    dd, ww = cons.separation(q, qs)
    assert torch.equal(dd, d0)
    dn1, wn1 = cons.separation(q[3].cpu().numpy(), qs[3].cpu().numpy())
    assert np.array_equal(dn1, d0[3].cpu().numpy()) and dn1.shape == (4, 5)


def _golden_points(g, robot, m):
    from toppra_b200.dynamics import pack_points
    return [(m.frame(str(l), xyz=x), float(r)) for l, x, r in zip(g[robot + "/links"], g[robot + "/xyz"],
                                                                     g[robot + "/radii"])], pack_points


def _cons(ta, points, humans, vlim, alim, scheme=0, joint_scheme=None, params=PARAMS):
    joint_scheme = scheme if joint_scheme is None else joint_scheme
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=joint_scheme),
            ta.constraint.SeparationMonitoringConstraint(points, humans, *params, discretization_scheme=scheme)]


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("separation_monitoring")
    m = model_of(name, locked)
    points, pack = _golden_points(g, robot, m)
    pts = pack(points)[1]
    ss, grid, params = g["ss"], g["grid"], tuple(g["params"])
    way, vlim, alim, hum = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "humans"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    d_grid = _dev(grid)
    q, qs = (path.eval_device(d_grid, o).reshape(-1, m.nv) for o in (0, 1))
    b, c = (x.reshape(B, -1).cpu().numpy() for x in m.separation_terms(pts, _dev(hum), *params, q, qs, len(grid)))
    assert np.array_equal(b == 0, g[robot + "/b"] == 0)
    np.testing.assert_allclose(b, g[robot + "/b"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(c, g[robot + "/c"], rtol=1e-12, atol=1e-14)
    ins = g[robot + "/inside"]
    assert b[0, ins[0]] == 0 and c[0, ins[0]] == -1.0               # inside the clearance, moving away: inactive
    assert b[1, ins[1]] > 0 and c[1, ins[1]] == 0.0                 # inside, approaching: x = 0
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (robot, scheme, x)][i]  # noqa: E731
        for i in range(B):
            one = ta.algorithm.TOPPRA(_cons(ta, points, hum[i], vlim[i], alim[i], scheme, params=params),
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA(_cons(ta, points, hum, vlim, alim, scheme, params=params), path, grid)
        h = h.compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


def _sep_rows(b, c, grid, interp):
    """(G, 3, R) rows a = 0, b, c of the constraint for the oracle."""
    G = len(grid)
    return _oracle_rows(np.ones((1, 1)), np.zeros((G, 1)), b.reshape(G, 1), c.reshape(G, 1), grid, interp)


def _arm6_points(m):
    return [(m.frame("flange", xyz=(0, 0, 0.1)), 0.05), (m.frame("wrist2"), 0.06), (m.frame("forearm"), 0.08)]


def _humans_ahead(ta, m, path, grid, rng):
    """(B, 2, 4): per path, one sphere 0.6 m off the tool's motion ahead of a mid-path gridpoint, one 1.5 m away."""
    d = _dev(grid)
    f = m.frame("flange", xyz=(0, 0, 0.1))
    B = path.B
    q, qs = (path.eval_device(d, o).reshape(-1, m.nv).cpu().numpy() for o in (0, 1))
    _, x, v = kr.frame_packed(m.packed, f.packed, q, qs)
    x, v = x.reshape(B, len(grid), 3), v[:, :3].reshape(B, len(grid), 3)
    out = []
    for i in range(B):
        g0 = int(rng.randint(len(grid) // 3, 2 * len(grid) // 3))
        u = v[i, g0] / max(np.linalg.norm(v[i, g0]), 1e-9)
        n = np.cross(u, rng.randn(3))
        n /= np.linalg.norm(n)
        near = x[i, g0] + 0.4 * u + 0.6 * n
        far = x[i, g0] + 1.5 * np.cross(n, u)
        out.append([np.r_[near, 0.1], np.r_[far, 0.2]])
    return np.array(out)


@pytest.mark.gpu
def test_gpu_256_paths_per_path_humans_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    points = _arm6_points(m)
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _problems(B, nv, 61, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    hum = _humans_ahead(ta, m, path, grid, np.random.RandomState(5))
    cons = _cons(ta, points, hum, vlim, alim, 0, 1)
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    pts = cons[2].points
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1))
        b, cc = sr.rows_packed(m.packed, pts, hum[i], PARAMS, q, qs)
        o = orc.solve_rows(np.concatenate((lin["rows"], _sep_rows(b, cc, grid, False)), axis=2), lin["xbound"], grid,
                           0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            d, w = sr.separation_packed(m.packed, pts, hum[i], q, qs)
            vm = sr.vmax_np(d, *PARAMS)
            sd = h["sd"][i][:, None, None]
            assert (w * sd <= vm + 1e-9).all()
            n_active += bool(((b > 0) & (b * h["sd"][i] ** 2 >= -cc * (1 - 1e-6))).any())
    print("separation limit active on %d of %d solved paths" % (n_active, n_ok))
    assert n_ok > 0.8 * B and n_active > 0.5 * n_ok, (n_ok, n_active)


@pytest.mark.gpu
def test_gpu_ragged_chunked_single_path_and_host_route_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    points = [(m.frame("hand", reference_frame="local", **OFFSET), 0.05), (m.frame("link4"), 0.07)]
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, nv, 37, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    rng = np.random.RandomState(9)
    hum = np.stack([_humans(rng, 3, center=(1.0, 0.0, 0.8), spread=0.3) for _ in range(B)])
    rag = ta.BatchTOPPRA(_cons(ta, points, hum, vlim, alim), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, points, hum[i:i + 1], vlim[i:i + 1], alim[i:i + 1]),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, points, hum, vlim, alim, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, points, hum, vlim, alim, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
        assert (hw["status"] == 0).sum() >= B // 4
        from toppra_b200.constraint import LinearConstraint

        class HostRoute(LinearConstraint):
            def __init__(self, inner):
                super(HostRoute, self).__init__()
                self.inner, self.identical = inner, True
                self.discretization_type = inner.discretization_type

            def compute_constraint_params(self, p, gridpoints):
                return self.inner.compute_constraint_params(p, gridpoints)

        for i in range(3):
            sp = ta.SplineInterpolator(ss, way[i])
            # path i of the batch with per-path humans == a single-path solve with humans[i] (shared and (1, H, 4))
            for hi in (hum[i], hum[i:i + 1]):
                one = ta.algorithm.TOPPRA(_cons(ta, points, hi, vlim[i], alim[i], scheme), sp, gridpoints=grid,
                                          solver_wrapper="seidel")
                run_dev = one.compute_parameterization(0, 0, return_data=True)
                assert _eq(run_dev[3], hw["K"][i])
                if hw["status"][i] == 0:
                    assert _eq(run_dev[1], hw["sd"][i]) and _eq(run_dev[0], hw["sdd"][i])
                else:
                    assert run_dev[1] is None
            cons = _cons(ta, points, hum[i], vlim[i], alim[i], scheme)
            cons[2] = HostRoute(cons[2])
            run_host = ta.algorithm.TOPPRA(cons, sp, gridpoints=grid, solver_wrapper="seidel").compute_parameterization(
                0, 0, return_data=True)
            for x, y in zip(run_dev, run_host):
                assert (x is None and y is None) or _eq(x, y)


@pytest.mark.gpu
def test_gpu_toppra_sd_quintic_and_other_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    points = _arm6_points(m)
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(41)
    path = ta.BatchPiecewisePolyPath(np.linspace(0, 1, nseg + 1), rng.uniform(-0.4, 0.4, (B, k, nseg, nv)))
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    hum = _humans_ahead(ta, m, path, grid, rng)
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    f = points[0][0]
    energy = 0.5
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    for extra in (False, True):
        cons = _cons(ta, points, hum, vlim, alim)
        if extra:
            cons += [ta.constraint.JointTorqueConstraint(m, taulim, fric),
                     ta.constraint.CollisionEnergyConstraint(f, energy, 0.6)]
        h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
        assert (h["status"] == 0).sum() >= B // 2
        for i in range(B):
            b, c = sr.rows_packed(m.packed, cons[2].points, hum[i], PARAMS, qs[0][i], qs[1][i])
            rows = [_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]), _sep_rows(b, c, grid, False)]
            if extra:
                import energy_ref as er
                av, bt, cv = rr.torque_terms_packed(m.packed, qs[0][i], qs[1][i], qs[2][i], fric)
                gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
                rows.append(np.stack((av.dot(Fj.T), bt.dot(Fj.T), cv.dot(Fj.T) - gt), axis=1))
                be = er.energy_terms_packed(m.packed, f.packed, qs[0][i], qs[1][i], 0.6)
                rows.append(np.stack((np.zeros(len(grid)), be, np.full(len(grid), 0.0 - energy)), axis=1)[:, :, None])
            o = orc.solve_rows(np.concatenate(rows, axis=2), orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
            _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
    # BatchTOPPRAsd, whole and in record chunks: bit-equal, and the limit holds on the blended profiles
    h = ta.BatchTOPPRA(_cons(ta, points, hum, vlim, alim), path, grid).compute_parameterization(0, 0).to_host()
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        inst = ta.BatchTOPPRAsd(_cons(ta, points, hum, vlim, alim), path, grid)
        if chunk:
            inst = ta.BatchTOPPRAsd(_cons(ta, points, hum, vlim, alim), path, grid,
                                    max_record_bytes=chunk * 8 * ta.engine.record_doubles(inst.R) * inst.G)
            assert inst.chunk_size() == chunk
        inst.set_desired_duration(1.5 * dur)
        r = inst.compute_parameterization(0.0, 0.0)
        runs.append([x.cpu().numpy() for x in (r.status, r.sd, r.sdd, r.duration_slow)])
    for x, y in zip(*runs):
        assert _eq(x, y)
    st, sd = runs[0][0], runs[0][1]
    assert (st[ok] == 0).all()
    for i in np.flatnonzero(ok):
        b, c = sr.rows_packed(m.packed, _cons(ta, points, hum, vlim, alim)[2].points, hum[i], PARAMS, qs[0][i],
                              qs[1][i])
        assert (b * sd[i] ** 2 + c <= 1e-9).all()


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch):
    from dyn_common import _assert_one_terms_launch
    m = model_of("arm6.urdf")
    ss, way, vlim, alim = _problems(10, 6, 47, m.velocity_limit)
    hum = np.stack([_humans(np.random.RandomState(i), 2) for i in range(10)])
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, _arm6_points(m), hum, vlim, alim),
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_separation_terms")


@pytest.mark.gpu
def test_gpu_1024_human_hypotheses_along_a_ray(ta):
    """One path, 1024 hypotheses of where the person stands, along a ray away from the tool's mid-path position: the
    time-optimal duration never grows as the person moves away."""
    m = model_of("arm6.urdf")
    points = _arm6_points(m)
    ss, way, vlim, alim = _problems(1, 6, 71, m.velocity_limit)
    B, G = 1024, 150
    grid = np.linspace(0, 1, G)
    one = ta.BatchSplineInterpolator(ss, way)
    hum0 = _humans_ahead(ta, m, one, grid, np.random.RandomState(2))[0, :1]
    f = points[0][0]
    x = kr.frame_packed(m.packed, f.packed, one.eval_device(_dev(grid), 0).reshape(-1, 6).cpu().numpy(),
                        np.zeros((G, 6)))[1]
    ray = hum0[0, :3] - x[G // 2]
    ray /= np.linalg.norm(ray)
    hum = np.repeat(hum0[None], B, axis=0)
    hum[:, 0, :3] = x[G // 2] + np.linspace(0.0, 3.0, B)[:, None] * ray     # from the tool outward
    path = ta.BatchSplineInterpolator(ss, np.repeat(way, B, axis=0))
    h = ta.BatchTOPPRA(_cons(ta, points, hum, np.repeat(vlim, B, 0), np.repeat(alim, B, 0)), path, grid)
    h = h.compute_parameterization(0, 0).to_host()
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else np.inf for s, o in zip(h["sd"], ok)])
    # near the path a point can be inside the clearance while approaching at one gridpoint, which stops it there
    # (uncontrollable, as for the reference); past the last such hypothesis every one solves
    first = int(np.flatnonzero(~ok).max()) + 1 if (~ok).any() else 0
    assert B - first > B // 2, first
    d = dur[first:]
    assert (np.diff(d) <= 1e-9 * d[1:]).all(), np.max(np.diff(d) / d[1:])
    assert d[0] > 1.05 * d[-1]                                   # the person near the path slows it down
    print("durations: %.3f s at %.2f m to %.3f s at 3 m (%d of %d hypotheses solve)"
          % (d[0], 3.0 * first / (B - 1), d[-1], ok.sum(), B))
