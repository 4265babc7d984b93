"""Every model-taking entry of libtoppra_b200_dyn.so against 50-digit references on hard models.

The fixture tests/golden/dyn_hard_trees.npz (tests/golden/make_golden_dyn_hard.py) holds, for the cases of
tests/dyn_hard.py (16-deep serial chains with a frame on the last body, stars, brooms, badly scaled links with rod-like
inertias, planar, all-prismatic and R/P chains; fast, wound-up and stretched states), the references of the
independent 50-digit code of tests/*_ref.py and a tolerance per output component, 32 (sens + eps mag + spread): sens is
how much the exact result moves when the float64 inputs move by one ulp, mag the output's own magnitude, spread how
much rounding the intermediate quantities of the float64 algorithm moves it (Monte Carlo arithmetic).  None of them is
the scale of the whole state, so a wrong 10 g finger torque does not hide under a 20 kg shoulder.

* CPU: the float64 numpy doubles of tests/*_ref.py meet every tolerance (their worst error / tolerance per entry is
  reported as a warning); one case per family is recomputed at 50 digits and matches the fixture; the generators
  produce what they claim.
* GPU: every entry, called through the C-ABI on every case, meets every tolerance (worst ratio per entry reported as
  a warning); BatchTOPPRA with joint-torque limits on the 16-body badly scaled chain matches the oracle on rows from
  the numpy double.
* A robot capsule whose two ends coincide but move apart, on CPU and GPU (a regression case of the capsule entries)."""
import ctypes
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import capsule_ref as cr  # noqa: E402
import dyn_hard  # noqa: E402
import energy_ref  # noqa: E402
import make_golden_dyn_hard as mg  # noqa: E402
import rnea_ref as rr  # noqa: E402
from dyn_common import OFFSET, _assert_solution, _model_from_packed  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "dyn_hard_trees.npz")
WORLD, LOCAL, LWA = mg.WORLD, mg.LOCAL, mg.LWA


def _model_entries():
    """Every entry of the library that takes a model (all but the version and the two drive / coupling helpers)."""
    from toppra_b200 import _lib_dyn
    return {n[4:] for n in _lib_dyn._PROTOS} - {"version", "drive_speed_terms", "coupling_expand"}


MODEL_ENTRIES = _model_entries()


@pytest.fixture(scope="module")
def fx():
    return np.load(GOLDEN)


def _cases(fx):
    return [str(c) for c in fx["cases"]]


def _setup(fx, name):
    keys = [k for k in fx.files if k.startswith(name + "/") and k.count("/") == 1]
    return {k.split("/", 1)[1]: fx[k] for k in keys}


def _ref(frame, ref):
    f = np.array(frame, dtype=np.float64)
    f[13] = ref
    return f


def _cat(*xs):
    return np.concatenate([np.asarray(x, dtype=np.float64).reshape(x.shape[0], -1) for x in xs], axis=1)


# ==== comparison ======================================================================================================
def ratios(fx, name, got):
    """{entry: worst |got - ref| / tol}; NaN or a missing entry counts as infinite."""
    out = {}
    entries = sorted({k.split("/")[1] for k in fx.files if k.startswith(name + "/") and k.endswith("/ref")})
    for e in entries:
        ref, tol = fx["%s/%s/ref" % (name, e)], fx["%s/%s/tol" % (name, e)]
        if e not in got:
            out[e] = np.inf
            continue
        g = np.asarray(got[e], dtype=np.float64)
        assert g.shape == ref.shape, (e, g.shape, ref.shape)
        err = np.abs(g - ref)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err == 0, 0.0, err / tol)
        out[e] = float(np.max(np.where(np.isnan(r), np.inf, r)))
    return out


def _check(fx, name, got):
    r = ratios(fx, name, got)
    bad = {e: v for e, v in r.items() if not v <= 1.0}
    assert not bad, (name, bad)
    return r


def _report(title, per_case):
    worst = {}
    for r in per_case.values():
        for e, v in r.items():
            worst[e] = max(worst.get(e, 0.0), v)
    lines = ["%-28s %.3g" % (e, worst[e]) for e in sorted(worst)]
    warnings.warn("%s, worst |err| / tol per entry over %d cases:\n  %s" % (title, len(per_case), "\n  ".join(lines)))
    return worst


# ==== CPU =============================================================================================================
def test_fixture_cases_are_the_generators(fx):
    assert _cases(fx) == list(dyn_hard.CASES)
    for name in _cases(fx):
        packed, q, qd, qdd = dyn_hard.case_model(name)
        s = _setup(fx, name)
        for k, v in (("packed", packed), ("q", q), ("qd", qd), ("qdd", qdd)):
            assert np.array_equal(s[k], v), (name, k)
        assert np.array_equal(s["frame"][10:13], OFFSET["xyz"])


@pytest.mark.parametrize("name", list(dyn_hard.CASES))
def test_numpy_doubles_meet_the_fixture(fx, name):
    _check(fx, name, mg.numpy_outputs(_setup(fx, name)))


def test_numpy_doubles_report(fx):
    per_case = {name: _check(fx, name, mg.numpy_outputs(_setup(fx, name))) for name in _cases(fx)}
    worst = _report("numpy float64 doubles", per_case)
    assert set(worst) == MODEL_ENTRIES


@pytest.mark.parametrize("name", dyn_hard.PIN_CASES)
def test_fixture_is_pinned_to_50_digits(fx, name):
    """One small case per family, recomputed at 50 digits (points 0 and 2: fast and stretched)."""
    s = _setup(fx, name)
    for m in (0, 2):
        res = mg.evaluate(s, s["packed"], s["q"][m], s["qd"][m], s["qdd"][m], m)
        for e, (val, _, _) in res.items():
            ref, tol = fx["%s/%s/ref" % (name, e)][m], fx["%s/%s/tol" % (name, e)][m]
            got = np.array([float(x) for x in val])
            assert np.all(np.abs(got - ref) <= 1e-3 * tol + 1e-15 * np.abs(ref)), (name, m, e)


def _world_frames(packed, q):
    """World rotations of every body at q (M, nv, 3, 3)."""
    Rs, _ = rr._transforms(packed, q)
    nv = q.shape[1]
    Rw = []
    for k in range(nv):
        par = int(packed[3 + 27 * k])
        Rw.append(Rs[k] if par < 0 else np.einsum("mij,mjk->mik", Rw[par], Rs[k]))
    return np.stack(Rw, axis=1)


def _principal(bd):
    I = energy_ref._inertia3(bd[21:27])
    return np.linalg.eigvalsh(I)


@pytest.mark.parametrize("name", list(dyn_hard.CASES))
def test_generators_produce_what_they_claim(name):
    import toppra_b200 as ta
    packed, q, qd, qdd = dyn_hard.case_model(name)
    family = dyn_hard.CASES[name][0]
    nv = q.shape[1]
    b = packed[3:].reshape(nv, 27)
    depths = [dyn_hard.depth(packed, k) for k in range(nv)]
    if family == "serial_chain" or family in ("badly_scaled", "planar"):
        assert depths == list(range(1, nv + 1))
        assert dyn_hard.deepest(packed) == nv - 1
    if family == "star":
        assert depths == [1] * nv
    if family == "broom":
        d = int(max(depths)) - 1
        assert depths == list(range(1, d + 1)) + [d + 1] * (nv - d)
    for bd in b:                                             # physical inertias: triangle inequalities
        lam = _principal(bd)
        assert lam[0] > 0 and lam[2] <= (lam[0] + lam[1]) * (1 + 1e-12), (name, lam)
        assert bd[17] > 0
        assert abs(np.linalg.norm(bd[2:5]) - 1) < 1e-15
        E = bd[5:14].reshape(3, 3)
        assert np.allclose(E @ E.T, np.eye(3), atol=1e-15) and np.linalg.det(E) > 0
    if family == "badly_scaled":
        assert b[0, 17] == 1e3 and b[-1, 17] == 1e-3 and np.all(np.diff(b[:, 17]) < 0)
        L = np.linalg.norm(b[:, 14:17], axis=1)
        assert np.all((L >= 1e-3 * (1 - 1e-12)) & (L <= 2 * (1 + 1e-12))) and np.isclose(L.max() / L.min(), 2e3)
        for bd in b:
            lam = _principal(bd)
            assert np.isclose(lam[0] / lam[1], 1e-6, rtol=1e-6), lam       # a rod
    if family == "planar":
        Rw = _world_frames(packed, q)
        rev = b[:, 1] == 0
        axes = np.einsum("mkij,kj->mki", Rw, b[:, 2:5])[:, rev]
        assert rev.any() or name == "planar_p16"
        assert np.allclose(axes, [0.0, 0.0, 1.0], atol=1e-15)           # every revolute axis parallel to z
        if name == "planar_p16":
            assert not rev.any()
    if name == "chain15_zero_g":
        assert not packed[:3].any()
    assert np.abs(qd).max() <= 50 and np.abs(q).max() <= 1e3 and not q[2].any()      # fast, wound, stretched
    if nv >= 15:
        assert np.abs(qd[0]).max() > 40 and np.abs(q[1]).max() > 900
    m = _model_from_packed(ta, packed)
    assert m.nv == nv and np.allclose(m.packed, packed, rtol=0, atol=1e-15)
    assert np.array_equal(m.packed[3:].reshape(nv, 27)[:, :2], b[:, :2])


def test_serial_chain_16_walks_16_bodies():
    for nv in (1, 8, 15, 16):
        packed = dyn_hard.serial_chain(np.random.RandomState(nv), nv)
        assert dyn_hard.depth(packed, dyn_hard.deepest(packed)) == nv
    assert max(dyn_hard.depth(dyn_hard.case_model("chain16")[0], k) for k in range(16)) == 16


# A robot capsule whose two ends coincide but move apart: from the base origin to a slider along z, at q = 0 with the
# slider moving at 2 m/s toward a human sphere (a capsule with c0 == c1) 0.5 m up the z axis.  Every t is a closest
# pair; the end on the slider closes the distance at 2 m/s.  The capsule entries took t = 0 only, the base end, and
# reported an approach speed of 0 (fixed: both ends, as for parallel segments).
SLIDER = np.concatenate(([0.0, 0.0, -9.81], [-1, 1, 0, 0, 1], np.eye(3).reshape(9), [0, 0, 0], [2.0, 0, 0, 0.1],
                         [0.01, 0, 0, 0.01, 0, 0.01]))
SLIDER_CAPSULE = np.concatenate((mg.frame_row(-1, np.eye(3), np.zeros(3), LWA), mg.frame_row(0, np.eye(3), np.zeros(3),
                                                                                                LWA), [0.05]))
SLIDER_HUMAN = np.array([0.0, 0.0, 0.5, 0.0, 0.0, 0.5, 0.1])


def test_capsule_with_coincident_ends_moving_apart():
    xa, va, xb, vb = cr.endpoint_states(SLIDER, SLIDER_CAPSULE[None], [[0.0]], [[2.0]])
    assert np.array_equal(xa, xb) and not np.array_equal(va, vb)
    d, w = cr.capsule_pair_np(xa[0, 0], va[0, 0], xb[0, 0], vb[0, 0], 0.05, SLIDER_HUMAN)
    dm, wm = cr.mp_capsule_pair(xa[0, 0], va[0, 0], xb[0, 0], vb[0, 0], 0.05, SLIDER_HUMAN)
    assert (d, w) == (0.5 - 0.05 - 0.1, 2.0) and abs(float(dm) - d) < 1e-16 and float(wm) == 2.0


@pytest.mark.gpu
def test_gpu_capsule_with_coincident_ends_moving_apart():
    g = _Gpu()
    hum = g.d(SLIDER_HUMAN[None, None])
    Q, QD = g.d([[0.0]]), g.d([[2.0]])
    d, w, b, c = g.out(1, 1, 1), g.out(1, 1, 1), g.out(1), g.out(1)
    g.call("tbd_capsule_separation", g.h(SLIDER), 1, g.h(SLIDER_CAPSULE), 1, 1, 1, 0, 1, Q, QD, hum, d, w)
    params = [ctypes.c_double(x) for x in mg.SEPARATION]
    g.call("tbd_capsule_separation_terms", g.h(SLIDER), 1, g.h(SLIDER_CAPSULE), 1, 1, 1, 0, *params, 1, Q, QD, hum, b,
           c)
    assert float(d) == 0.5 - 0.05 - 0.1 and float(w) == 2.0
    bw, cw = cr.sr.rows_from_pairs(np.array([[[float(d)]]]), np.array([[[2.0]]]), mg.SEPARATION)
    assert float(b) == bw[0] == 4.0 and float(c) == cw[0]


# ==== GPU =============================================================================================================
class _Gpu(object):
    """Direct C-ABI calls of libtoppra_b200_dyn.so: host arrays and device tensors by pointer, the default stream."""

    def __init__(self):
        import torch
        from toppra_b200 import _lib, _lib_dyn
        self.torch, self._lib, self.lib = torch, _lib, _lib_dyn.load()
        self._keep = []

    def h(self, x):
        a = np.ascontiguousarray(x, dtype=np.float64)
        self._keep.append(a)
        return ctypes.c_void_p(a.ctypes.data)

    def d(self, x):
        t = self.torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device="cuda")
        self._keep.append(t)
        return t

    def out(self, *shape):
        t = self.torch.full(shape, np.nan, dtype=self.torch.float64, device="cuda")
        self._keep.append(t)
        return t

    def call(self, name, *args):
        conv = [self._lib.ptr(a) if isinstance(a, self.torch.Tensor) else a for a in args]
        self._lib.check(getattr(self.lib, name)(*conv, None), name)


def gpu_outputs(s):
    g = _Gpu()
    P, q, qd, qdd = s["packed"], s["q"], s["qd"], s["qdd"]
    M, nv = q.shape
    model = g.h(P)
    Q, QD, QDD = g.d(q), g.d(qd), g.d(qdd)
    host = lambda t: t.cpu().numpy()   # noqa: E731
    out = {}
    tau = g.out(M, nv)
    g.call("tbd_rnea", model, nv, M, Q, QD, QDD, tau)
    out["rnea"] = host(tau)
    abc = [g.out(M, nv) for _ in range(3)]
    g.call("tbd_torque_terms", model, nv, M, Q, QD, QDD, g.d(s["friction"]), *abc)
    out["torque_terms"] = _cat(*map(host, abc))
    fr, mid = s["frame"], s["mid_frame"]
    vs = []
    for r in (WORLD, LOCAL, LWA):
        v = g.out(M, 6)
        g.call("tbd_frame_velocity", model, nv, g.h(_ref(fr, r)), M, Q, QD, v)
        vs.append(host(v))
    out["frame_velocity"] = _cat(*vs)
    b = g.out(M)
    g.call("tbd_velocity_norm_terms", model, nv, g.h(fr), g.h(s["S"]), M, Q, QD, b)
    out["velocity_norm_terms"] = _cat(host(b))
    acc, ta_, tb_ = [], [], []
    for r in (LOCAL, LWA):
        x = g.out(M, 6)
        g.call("tbd_frame_acceleration", model, nv, g.h(_ref(fr, r)), M, Q, QD, QDD, x)
        acc.append(host(x))
        a, b = g.out(M, 6), g.out(M, 6)
        g.call("tbd_acceleration_terms", model, nv, g.h(_ref(fr, r)), 63, M, Q, QD, QDD, a, b)
        ta_.append(host(a))
        tb_.append(host(b))
    out["frame_acceleration"] = _cat(*acc)
    out["acceleration_terms"] = _cat(*(ta_ + tb_))
    w = g.out(M, 6)
    g.call("tbd_contact_wrench", model, nv, g.h(fr), g.h(s["object"]), M, Q, QD, QDD, w)
    out["contact_wrench"] = host(w)
    abc = [g.out(M, 6) for _ in range(3)]
    g.call("tbd_contact_wrench_terms", model, nv, g.h(fr), g.h(s["object"]), M, Q, QD, QDD, *abc)
    out["contact_wrench_terms"] = _cat(*map(host, abc))
    Ls = []
    for r in (LOCAL, LWA):
        L = g.out(M, 9)
        g.call("tbd_frame_inverse_inertia", model, nv, g.h(_ref(fr, r)), M, Q, L)
        Ls.append(host(L))
    out["frame_inverse_inertia"] = _cat(*Ls)
    b = g.out(M)
    g.call("tbd_collision_energy_terms", model, nv, g.h(fr), ctypes.c_double(mg.HUMAN_MASS), M, Q, QD, b)
    out["collision_energy_terms"] = _cat(host(b))
    w = g.out(M, 6)
    g.call("tbd_support_wrench", model, nv, g.h(s["support"]), g.h(s["base"]), M, Q, QD, QDD, w)
    out["support_wrench"] = host(w)
    abc = [g.out(M, 6) for _ in range(3)]
    g.call("tbd_support_wrench_terms", model, nv, g.h(s["support"]), g.h(s["base"]), M, Q, QD, QDD, *abc)
    out["support_wrench_terms"] = _cat(*map(host, abc))
    params = [ctypes.c_double(x) for x in mg.SEPARATION]
    for entry, bodies, humans, ppp in (("separation", s["points"], s["humans"][None], 0),
                                       ("capsule_separation", s["capsules"], s["hcaps"], 1)):
        Pn, NH, H = bodies.shape[0], humans.shape[0], humans.shape[1]
        hum = g.d(humans)
        d, w = g.out(M, Pn, H), g.out(M, Pn, H)
        g.call("tbd_" + entry, model, nv, g.h(bodies), Pn, H, NH, ppp, M, Q, QD, hum, d, w)
        out[entry] = _cat(host(d), host(w))
        b, c = g.out(M), g.out(M)
        g.call("tbd_%s_terms" % entry, model, nv, g.h(bodies), Pn, H, NH, ppp, *params, M, Q, QD, hum, b, c)
        out[entry + "_terms"] = _cat(host(b), host(c))
    tau = g.out(M, nv)
    g.call("tbd_drive_torque", model, nv, g.h(s["drive"]), M, Q, QD, QDD, tau)
    out["drive_torque"] = host(tau)
    abc = [g.out(M, nv) for _ in range(3)]
    g.call("tbd_drive_torque_terms", model, nv, g.h(s["drive"]), M, Q, QD, QDD, *abc)
    out["drive_torque_terms"] = _cat(*map(host, abc))
    jw, jt = [], []
    for f in (fr, mid):
        for r in (LOCAL, LWA):
            w = g.out(M, 6)
            g.call("tbd_joint_wrench", model, nv, g.h(_ref(f, r)), M, Q, QD, QDD, w)
            jw.append(host(w))
            abc = [g.out(M, 6) for _ in range(3)]
            g.call("tbd_joint_wrench_terms", model, nv, g.h(_ref(f, r)), 63, M, Q, QD, QDD, *abc)
            jt += list(map(host, abc))
    out["joint_wrench"], out["joint_wrench_terms"] = _cat(*jw), _cat(*jt)
    em = g.out(M, 4)
    g.call("tbd_energy_momentum", model, nv, M, Q, QD, em)
    out["energy_momentum"] = host(em)
    bs = []
    for which in (0, 1):
        b = g.out(M)
        g.call("tbd_energy_momentum_terms", model, nv, which, M, Q, QD, b)
        bs.append(host(b))
    out["energy_momentum_terms"] = _cat(*bs)
    if "E" in s:
        nq = s["E"].shape[1]
        coupling = g.h(np.concatenate((s["E"].reshape(-1), s["o"])))
        Qc, QDc, QDDc = g.d(q[:, :nq]), g.d(qd[:, :nq]), g.d(qdd[:, :nq])
        tau = g.out(M, nq)
        g.call("tbd_coupled_rnea", model, nv, coupling, nq, M, Qc, QDc, QDDc, tau)
        out["coupled_rnea"] = host(tau)
        abc = [g.out(M, nq) for _ in range(3)]
        g.call("tbd_coupled_torque_terms", model, nv, coupling, nq, M, Qc, QDc, QDDc, g.d(s["friction"][:nq]), *abc)
        out["coupled_torque_terms"] = _cat(*map(host, abc))
    g.torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(dyn_hard.CASES))
def test_gpu_entries_meet_the_fixture(fx, name):
    _check(fx, name, gpu_outputs(_setup(fx, name)))


@pytest.mark.gpu
def test_gpu_entries_report(fx):
    per_case = {name: ratios(fx, name, gpu_outputs(_setup(fx, name))) for name in _cases(fx)}
    worst = _report("GPU kernels", per_case)
    assert set(worst) == MODEL_ENTRIES and all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.gpu
def test_gpu_badly_scaled_chain_through_batch_toppra(fx):
    """BatchTOPPRA with joint-torque limits on the 16-body badly scaled chain: statuses, K and sd of the oracle on rows
    from the numpy double of the fixture's model."""
    import toppra_b200 as ta
    from oracle import oracle as orc
    s = _setup(fx, "scaled16")
    m = _model_from_packed(ta, s["packed"])
    B, G, nv = 12, 100, m.nv
    rng = np.random.RandomState(41)
    ss, grid = np.linspace(0, 1, 5), np.linspace(0, 1, G)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vlim = np.tile(np.stack([-np.full(nv, 3.0), np.full(nv, 3.0)], axis=1), (B, 1, 1))
    al = rng.uniform(6, 10, (B, nv))
    alim = np.stack([-al, al], axis=-1)
    fric = s["friction"] * np.abs(s["packed"][3 + 27 * np.arange(nv) + 17]) * 1e-3     # scaled with each body's mass
    taulim = np.empty((B, nv, 2))
    rows_of = []
    for b in range(B):
        c = orc.cubic_spline_fit(ss, way[b])
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        av, bv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        tl = 1.2 * np.abs(cv).max(axis=0) + 0.5 * (np.abs(av) + np.abs(bv)).max(axis=0) * rng.uniform(0.5, 2.0, nv)
        taulim[b] = np.stack([-tl, tl], axis=1)
        rows_of.append((c, av, bv, cv))
    path = ta.BatchSplineInterpolator(ss, way)
    # collocation: 2 nv acceleration and 2 nv torque rows per gridpoint (interpolation would need 8 nv > 126)
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                        ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=0),
                        ta.constraint.SecondOrderConstraint.joint_torque_constraint(m, taulim, fric,
                                                                                    discretization_scheme=0)],
                       path, grid).compute_parameterization(0, 0).to_host()
    F = np.vstack((np.eye(nv), -np.eye(nv)))
    n_ok = 0
    for b in range(B):
        c, av, bv, cv = rows_of[b]
        lin = orc.solve_velacc(c, ss, grid, vlim[b], alim[b], False, 0, 0, want_rows=True)
        g = np.concatenate((taulim[b, :, 1], -taulim[b, :, 0]))
        rows = np.concatenate((lin["rows"], np.stack((av.dot(F.T), bv.dot(F.T), cv.dot(F.T) - g), axis=1)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][b], h["sd"][b]), o["K"], o["sd"], h["status"][b], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok >= B // 2
