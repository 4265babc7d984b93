"""The kinetic energy and the linear momentum of the whole robot, and limits on them (RigidBodyModel.energy_momentum /
energy_momentum_terms, KineticEnergyConstraint, MomentumConstraint; libtoppra_b200_dyn.so: tbd_energy_momentum,
tbd_energy_momentum_terms).

CPU:
  * the float64 numpy double of tests/momentum_ref.py equals the 50-digit T = 1/2 qd^T M qd and p = sum m J_c qd of the
    RAW URDF tree within 1e-13 of the energy and momentum scale: arm6.urdf and arm7_gripper.urdf (fingers locked and
    unlocked), with and without a with_payload payload, and random trees with prismatic joints;
  * every ValueError of both constraints and of the model methods; the ctypes prototypes against the header; each
    refused call of the two entries returns its TB_ERR_* and message from the real library;
  * the calls of both methods and the launch plan of both constraints on the recording library: one terms launch and
    one tb_rows_canlinear call per batch or record chunk, both schemes, shared and per-path limits.
GPU:
  * both kernels on random trees of 1 to 16 bodies against the numpy double within 1e-12 (and the 50-digit reference on
    one point); T against 1/2 qd.(tbd_rnea(q, 0, qd) - tbd_rnea(q, 0, 0)) and p against the force of
    tbd_support_wrench(q, 0, qd) - tbd_support_wrench(q, 0, 0) within 1e-12; the terms kernel bit-equal to the value
    entry's T and to p.p;
  * the reference golden (tests/golden/kinetic_energy.npz, make_golden_kinetic_energy.py): TOPPRA and BatchTOPPRA within
    the cfg-3 tolerance, equal statuses (failing start speeds included), both limits, both schemes;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1: bit-equal; a quintic
    BatchPiecewisePolyPath against the oracle fed with numpy-double rows; BatchTOPPRAsd whole and in record chunks;
    one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import momentum_ref as mr
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, LOCKED, TB_ERR_ARG, TB_ERR_UNSUPPORTED, _assert_one_terms_launch,
                        _assert_solution, _dev, _dyn_header, _eq, _gpu_present, _model_from_packed, _oracle_joint_rows,
                        _problems, model_of, urdf)
from test_collision_energy import PAYLOAD, PAYLOAD_ORIGIN, _urdf_with_payload
from test_dyn_calls import H, T, _OUTPUTS, _context, _flat, _rows_call, _run, arm, calls  # noqa: F401

KINDS = ("energy", "momentum")


def _close(got, want, tol):
    """|got - want| <= tol * max(1, max |want|)."""
    want = np.asarray(want, dtype=np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(np.asarray(got) - want).max())
    assert err <= tol * scale, (err, scale)


def _check_double_vs_mp(packed, mp, rng, n=3):
    nv = (len(packed) - 3) // 27
    for _ in range(n):
        q, qd = rng.uniform(-2, 2, nv), rng.uniform(-2, 2, nv)
        Tm, pm = mr.mp_energy_momentum64(mp, q, qd)
        Td, pd = mr.energy_momentum_packed(packed, q, qd)
        _close(Td, [Tm], 1e-13)
        _close(pd[0], pm, 1e-13)


def _tree(rng, nv):
    """rr.random_tree with a prismatic joint for nv >= 3."""
    packed = rr.random_tree(rng, nv)
    if nv >= 3:
        packed[3:].reshape(nv, 27)[nv // 2, 1] = 1
    return packed


# ==== CPU: numpy double vs the 50-digit reference ===================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    _check_double_vs_mp(m.packed, rr.MpRobot.from_urdf(urdf(name), locked), np.random.RandomState(m.nv + 501))


@pytest.mark.parametrize("name,locked,link", [("arm6.urdf", None, "flange"), ("arm7_gripper.urdf", LOCKED, "hand")])
def test_numpy_double_with_payload_matches_mp_reference(name, locked, link):
    m = model_of(name, locked)
    loaded = m.with_payload(m.frame(link, **PAYLOAD_ORIGIN), *PAYLOAD)
    mp = rr.MpRobot.from_urdf(_urdf_with_payload(name, link), locked)
    rng = np.random.RandomState(7)
    _check_double_vs_mp(loaded.packed, mp, rng)
    q, qd = rng.uniform(-2, 2, (2, m.nv))
    assert not np.isclose(mr.energy_momentum_packed(m.packed, q, qd)[0][0],
                          mr.energy_momentum_packed(loaded.packed, q, qd)[0][0], rtol=1e-6)   # the payload matters


@pytest.mark.parametrize("nv", [1, 2, 3, 7, 16])
def test_numpy_double_random_trees_match_mp_reference(nv):
    rng = np.random.RandomState(600 + nv)
    packed = _tree(rng, nv)
    _check_double_vs_mp(packed, rr.MpRobot.from_packed(packed), rng, n=2)


def test_numpy_double_closed_forms():
    """One prismatic body: T = 1/2 m qd^2, p = m qd axis; one revolute body about z: T = 1/2 I_axis qd^2, p = m w x c."""
    import toppra_b200 as ta
    ax = np.array([0.0, 0.6, 0.8])
    pm = ta.RigidBodyModel([-1], ["prismatic"], [ax], [np.eye(3)], [[0.1, 0.2, 0.3]], [3.5], [[0.05, -0.02, 0.1]],
                           [[0.01, 0.0, 0.0, 0.02, 0.0, 0.03]])
    q, qd = np.array([[0.4], [-0.3]]), np.array([[1.5], [-2.0]])
    Td, pd = mr.energy_momentum_packed(pm.packed, q, qd)
    np.testing.assert_allclose(Td, 0.5 * 3.5 * qd[:, 0] ** 2, rtol=1e-15)
    np.testing.assert_allclose(pd, 3.5 * qd * ax, rtol=1e-15)
    rm = ta.RigidBodyModel([-1], ["revolute"], [[0.0, 0.0, 1.0]], [np.eye(3)], [[0.0, 0.0, 0.5]], [2.0],
                           [[0.2, 0.1, 0.3]], [[0.04, 0.001, 0.002, 0.05, 0.003, 0.06]])
    Td, pd = mr.energy_momentum_packed(rm.packed, np.zeros((1, 1)), np.array([[1.7]]))
    np.testing.assert_allclose(Td, 0.5 * (0.06 + 2.0 * (0.2 ** 2 + 0.1 ** 2)) * 1.7 ** 2, rtol=1e-15)
    np.testing.assert_allclose(pd[0], 2.0 * np.cross([0, 0, 1.7], [0.2, 0.1, 0.3]), rtol=1e-15)


# ==== CPU: errors, header, C-ABI checks ==============================================================================
def test_value_errors():
    from toppra_b200.constraint import KineticEnergyConstraint, MomentumConstraint
    from toppra_b200.constraint.linear_constraint import RecordContext
    from dyn_common import FakePath
    m = model_of("arm6.urdf")
    grid = np.linspace(0, 1, 10)
    for cls in (KineticEnergyConstraint, MomentumConstraint):
        for bad in (m.frame("flange"), None, "arm6.urdf"):
            with pytest.raises(ValueError, match="needs a RigidBodyModel"):
                cls(bad, 1.0)
        for lim in (-1.0, np.nan, [1.0, -0.1], [np.nan, 1.0]):
            with pytest.raises(ValueError, match=">= 0"):
                cls(m, lim)
        with pytest.raises(ValueError, match="float or"):
            cls(m, np.ones((2, 2)))
        c = cls(m, 0.0)                                              # a zero limit is fine
        assert c.dof == 6 and c.get_dof() == 6 and c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
        assert cls(m, 1.0, discretization_scheme=1).num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 2
        with pytest.raises(ValueError, match="Wrong dimension"):
            c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
        per_path = cls(m, [1.0, 2.0, 3.0])
        assert per_path.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
        with pytest.raises(ValueError, match="expected a float or"):
            per_path.num_rows(RecordContext(FakePath(4, 6), grid, grid))
        with pytest.raises(ValueError, match="Wrong dimension"):
            c.compute_constraint_params(type("P", (), {"dof": 7})(), grid)
        with pytest.raises(ValueError, match="single path"):
            per_path.compute_constraint_params(type("P", (), {"dof": 6})(), grid)
    # the row limit: E_max as given, p_max squared once
    assert KineticEnergyConstraint(m, 3.0).limit == 3.0 and MomentumConstraint(m, 3.0).limit == 9.0
    assert np.array_equal(MomentumConstraint(m, [0.5, 3.0])._path_limits, [0.25, 9.0])
    assert KineticEnergyConstraint(m, 3.0).which == "energy" and MomentumConstraint(m, 3.0).which == "momentum"


def test_model_method_calls_and_errors(calls, arm, monkeypatch):  # noqa: F811
    import torch
    from test_dyn_calls import _canon, _dev as _fake_dev
    monkeypatch.setitem(_OUTPUTS, "tbd_energy_momentum", 1)
    nv, M = arm.nv, 5
    rng = np.random.default_rng(3)
    q, qd = (_fake_dev(rng.uniform(-1, 1, (M, nv))) for _ in range(2))
    Tv, p = arm.energy_momentum(q, qd)                           # views of the one (M, 4) output
    assert tuple(Tv.shape) == (M,) and tuple(p.shape) == (M, 3) and p.data_ptr() == Tv.data_ptr() + 8
    assert _canon(calls, {"q": q, "qd": qd}) == [
        ["tbd_energy_momentum", H(arm.packed), nv, M, T("q", (M, nv)), T("qd", (M, nv)),
         T("tbd_energy_momentum.5", (M, 4)), None]]
    for which, code in (("energy", 0), ("momentum", 1)):
        del calls[:]
        b = arm.energy_momentum_terms(q, qd, which)
        assert _canon(calls, {"q": q, "qd": qd, "b": b}) == [
            ["tbd_energy_momentum_terms", H(arm.packed), nv, code, M, T("q", (M, nv)), T("qd", (M, nv)), T("b", (M,)),
             None]]
    del calls[:]
    for which in ("kinetic", 0, None):
        with pytest.raises(ValueError, match="which"):
            arm.energy_momentum_terms(q, qd, which)
    with pytest.raises(ValueError, match=r"expected \(M, 6\)"):
        arm.energy_momentum(q[:, :4], qd[:, :4])
    with pytest.raises(ValueError, match="share shape"):
        arm.energy_momentum(q, qd[:3])
    with pytest.raises(ValueError, match=r"expected \(M, 6\)"):
        arm.energy_momentum_terms(torch.zeros(4, 6, 1).as_subclass(type(q)), qd, "energy")
    assert calls == []


def test_dyn_header_prototypes_of_energy_momentum_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_energy_momentum"] == ["ptr", "int", "int", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_energy_momentum_terms"] == ["ptr", "int", "int", "int", "ptr", "ptr", "ptr", "ptr"]
    for name in ("tbd_energy_momentum", "tbd_energy_momentum_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_energy_momentum_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")

    def err():
        return _lib.load().tb_last_error()

    def rc(model=m.packed, nv=6, M=4, which=0, null=None):
        host = np.array(model, dtype=np.float64)
        mp = ctypes.c_void_p(host.ctypes.data)
        cv = [mp, nv, M, d, d, d]                # model, nv, M, q, qd, out
        ct = [mp, nv, which, M, d, d, d]         # model, nv, which, M, q, qs, b
        if null is not None:                     # index into cv; ct has `which` before M
            cv[null] = None
            ct[null if null < 2 else null + 1] = None
        r1 = lib.tbd_energy_momentum(*cv, None)
        e1 = err()
        r2 = lib.tbd_energy_momentum_terms(*ct, None)
        e2 = err()
        if which in (0, 1):
            assert r1 == r2 and e1.replace(b"tbd_energy_momentum:", b"") == e2.replace(b"tbd_energy_momentum_terms:",
                                                                                         b"")
        assert r2 == 0 or e2.startswith(b"tbd_energy_momentum_terms: ")
        return r2

    for k in (0, 3, 4, 5):
        assert rc(null=k) == TB_ERR_ARG and err() == b"tbd_energy_momentum_terms: null pointer"
    for M in (0, -3):
        assert rc(M=M) == TB_ERR_ARG and b"M=%d must be positive" % M in err()
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and b"nv=0 outside 1..16" in err()
    assert rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED and b"nv=17 outside 1..16" in err()
    for j, value, msg in ((0, 2.0, b"parent"), (17, -1.0, b"mass"), (17, np.nan, b"mass"), (1, 3.0, b"joint type"),
                          (2, 0.0, b"zero joint axis")):
        bad = m.packed.copy()
        k = 2
        bad[3 + 27 * k + j] = value
        if j == 2:
            bad[3 + 27 * k + 2:3 + 27 * k + 5] = 0.0
        assert rc(bad) == TB_ERR_ARG and b"body 2" in err() and msg in err(), (j, err())
    for which in (2, -1, 7):
        assert rc(which=which) == TB_ERR_ARG
        assert err() == (b"tbd_energy_momentum_terms: which=%d must be TBD_KINETIC_ENERGY (0) or TBD_MOMENTUM (1)"
                         % which)
    for which in (0, 1):                         # good calls pass validation and fail only at the launch (no device)
        assert rc(which=which) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
        assert b"launch failed" in err()


# ==== CPU: launch plan on the recording library =======================================================================
@pytest.mark.parametrize("lo,hi,total", [(0, 4, 4), (1, 3, 4)])
@pytest.mark.parametrize("interp", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_launch_plan(calls, arm, monkeypatch, lo, hi, total, interp, kind):  # noqa: F811
    from toppra_b200.constraint import KineticEnergyConstraint, MomentumConstraint
    monkeypatch.setitem(_OUTPUTS, "tbd_energy_momentum_terms", 1)
    cls = KineticEnergyConstraint if kind == "energy" else MomentumConstraint
    name = "tbd_energy_momentum_terms"
    nv, G = arm.nv, 6
    B, n = hi - lo, (hi - lo) * G
    for limit in (2.5, 0.0, np.arange(total) * 0.5 + 1.0):
        cons = cls(arm, limit, discretization_scheme=int(interp))
        ctx, bp = _context(nv, total, G, lo, hi, total)
        rows, log = _run(calls, cons, ctx)
        assert rows == (2 if interp else 1)
        lim = np.broadcast_to(np.asarray(limit, dtype=np.float64).reshape(-1)[lo:hi] if np.ndim(limit) else limit, B)
        c = np.repeat(0.0 - (lim if kind == "energy" else lim * lim), G)
        assert log == [
            [name, H(arm.packed), nv, KINDS.index(kind), n, T("q0", (n, nv)), T("q1", (n, nv)), T(name + ".6", (n,)),
             None],
            _rows_call(T((0.0,) * (B * G), (B, G, 1)), T(name + ".6", (B, G, 1)), T(_flat(c), (B, G, 1)),
                       T((1.0,), (1, 1)), T((0.0,), (1,)), 0, B, G, 1, 1, interp)]


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_random_trees(ta, nv):
    rng = np.random.RandomState(1900 + nv)
    m = _model_from_packed(ta, _tree(rng, nv))
    Q, QD = rng.uniform(-3, 3, (2, 512, nv))
    Tg, pg = (x.cpu().numpy() for x in m.energy_momentum(_dev(Q), _dev(QD)))
    Td, pd = mr.energy_momentum_packed(m.packed, Q, QD)
    _close(Tg, Td, 1e-12)
    _close(pg, pd, 1e-12)
    for which, want in (("energy", Td), ("momentum", mr.momentum_squared(pd))):
        _close(m.energy_momentum_terms(_dev(Q), _dev(QD), which).cpu().numpy(), want, 1e-12)
    Tm, pm = mr.mp_energy_momentum64(rr.MpRobot.from_packed(m.packed), Q[0], QD[0])   # and the 50-digit reference
    _close(Tg[0], [Tm], 1e-12)
    _close(pg[0], pm, 1e-12)
    T3, p3 = m.energy_momentum(Q[3], QD[3])                     # numpy (nv,): a device round trip
    assert isinstance(T3, float) and T3 == Tg[3] and np.array_equal(p3, pg[3])
    T5, p5 = m.energy_momentum(Q[:5], QD[:5])
    assert np.array_equal(T5, Tg[:5]) and np.array_equal(p5, pg[:5])


@pytest.mark.gpu
def test_gpu_identities_with_rnea_and_support_wrench(ta):
    """T = 1/2 qd.(ID(q, 0, qd) - ID(q, 0, 0)) = 1/2 qd.(M qd); at zero velocity the momentum rate is A(q) qdd, so the
    force of the support wrench at (q, 0, qd) less that at (q, 0, 0) is p(q, qd)."""
    import torch
    rng = np.random.RandomState(37)
    for m in (model_of("arm6.urdf"), model_of("arm7_gripper.urdf"), _model_from_packed(ta, _tree(rng, 11))):
        m.frames["origin"] = (-1, np.eye(3), np.zeros(3))
        q, qd = (_dev(rng.uniform(-3, 3, (2000, m.nv))) for _ in range(2))
        zero = torch.zeros_like(q)
        Tg, pg = m.energy_momentum(q, qd)
        Ti = 0.5 * (qd * (m(q, zero, qd) - m(q, zero, zero))).sum(dim=1)
        assert float((Tg - Ti).abs().max()) <= 1e-12 * float(Tg.abs().max())
        f = m.frame("origin")
        pi = (f.support_wrench(None, q, zero, qd) - f.support_wrench(None, q, zero, zero))[:, :3]
        assert float((pg - pi).abs().max()) <= 1e-12 * float(pg.abs().max())
        assert (Tg >= 0).all()


@pytest.mark.gpu
def test_gpu_terms_bit_equal_value_entry(ta):
    import torch
    rng = np.random.RandomState(41)
    for m in (model_of("arm7_gripper.urdf"), model_of("arm6.urdf").with_payload("flange", *PAYLOAD),
              _model_from_packed(ta, _tree(rng, 16))):
        q, qs = (_dev(rng.uniform(-2, 2, (3000, m.nv))) for _ in range(2))
        qs[:7] = 0.0                                             # q' = 0: b = +0
        Tg, p = m.energy_momentum(q, qs)
        bE, bP = (m.energy_momentum_terms(q, qs, w) for w in KINDS)
        assert torch.equal(bE, Tg)
        assert torch.equal(bP, (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
        assert (bE[:7] == 0).all() and not torch.signbit(bE[:7]).any() and not torch.signbit(bP[:7]).any()


def _cons(ta, m, vlim, alim, kind, limit, scheme=0):
    cls = ta.constraint.KineticEnergyConstraint if kind == "energy" else ta.constraint.MomentumConstraint
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
            cls(m, limit, discretization_scheme=scheme)]


def _golden_model(robot):
    return model_of(*{"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf", LOCKED)}[robot])


@pytest.mark.gpu
@pytest.mark.parametrize("robot", ["arm6", "arm7"])
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_reference_golden(ta, golden, robot, kind):
    g = golden("kinetic_energy")
    m = _golden_model(robot)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim = (g[robot + "/" + k] for k in ("way", "vlim", "alim"))
    limit, sd0, bref = (g["%s/%s/%s" % (robot, kind, k)] for k in ("limit", "sd_start", "b"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    d = _dev(grid)
    b = m.energy_momentum_terms(*(path.eval_device(d, o).reshape(-1, m.nv) for o in (0, 1)), kind)
    b = b.reshape(B, len(grid)).cpu().numpy()
    for i in range(B):                                            # against the 50-digit b
        assert np.abs(b[i] - bref[i]).max() <= 1e-12 * np.abs(bref[i]).max()
    statuses = set()
    for scheme in (0, 1):
        key = lambda x, i: g["%s/%s/s%d/%s" % (robot, kind, scheme, x)][i]  # noqa: E731
        for i in range(B):                                        # a shared (float) limit on each path alone
            one = ta.algorithm.TOPPRA(_cons(ta, m, vlim[i], alim[i], kind, float(limit[i]), scheme),
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(float(sd0[i]), 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA(_cons(ta, m, vlim, alim, kind, limit, scheme), path, grid)   # per-path limits
        h = h.compute_parameterization(sd0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))
            statuses.add(int(h["status"][i]))
    assert 0 in statuses and len(statuses) > 1                   # some paths solve, the fast start fails


def _binding_limits(ta, m, kind, path, grid, vlim, alim, share=0.3):
    """Per path: `share` of the largest T (or |p|) on the solution without the limit, so that it binds."""
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                       path, grid).compute_parameterization(0, 0).to_host()
    d = _dev(grid)
    b = m.energy_momentum_terms(*(path.eval_device(d, o).reshape(-1, m.nv) for o in (0, 1)), kind)
    b = b.reshape(path.B, len(grid)).cpu().numpy()
    sd = np.nan_to_num(h["sd"])
    return share * (np.max(b * sd ** 2, axis=1) if kind == "energy" else np.max(np.sqrt(b) * sd, axis=1))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta, kind):
    m = model_of("arm7_gripper.urdf", LOCKED).with_payload("hand", *PAYLOAD)
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, nv, 53, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    limit = _binding_limits(ta, m, kind, path, np.linspace(0, 1, 100), vlim, alim)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cons(ta, m, vlim, alim, kind, limit), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, m, vlim[i:i + 1], alim[i:i + 1], kind, limit[i:i + 1]),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, m, vlim, alim, kind, limit, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, m, vlim, alim, kind, limit, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
        assert (hw["status"] == 0).any()
    # single-path TOPPRA (the reference's 7-tuple from one launch) equals BatchTOPPRA at B = 1
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cons(ta, m, vlim[i], alim[i], kind, float(limit[i]), scheme), sp,
                                      gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cons(ta, m, vlim[i:i + 1], alim[i:i + 1], kind, limit[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0)
            hb = hb.to_host()
            assert sd is not None and _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_quintic_path_vs_oracle_and_toppra_sd(ta, kind):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(59)
    coeffs = rng.uniform(-0.4, 0.4, (B, k, nseg, nv))
    path = ta.BatchPiecewisePolyPath(np.linspace(0, 1, nseg + 1), coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    limit = _binding_limits(ta, m, kind, path, grid, vlim, alim)
    row_limit = limit if kind == "energy" else limit * limit
    h = ta.BatchTOPPRA(_cons(ta, m, vlim, alim, kind, limit), path, grid).compute_parameterization(0, 0).to_host()
    assert (h["status"] == 0).sum() >= B // 2
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    b = np.stack([mr.energy_momentum_terms_packed(m.packed, qs[0][i], qs[1][i], kind) for i in range(B)])
    G = len(grid)
    for i in range(B):
        rows = np.stack((np.zeros(G), b[i], np.full(G, 0.0 - row_limit[i])), axis=1)[:, :, None]
        o = orc.solve_rows(np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]), rows), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
    # BatchTOPPRAsd, whole and in record chunks, at half again the time-optimal duration; the limit holds on the profiles
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        inst = ta.BatchTOPPRAsd(_cons(ta, m, vlim, alim, kind, limit), path, grid)
        if chunk:
            inst = ta.BatchTOPPRAsd(_cons(ta, m, vlim, alim, kind, limit), path, grid,
                                    max_record_bytes=chunk * 8 * ta.engine.record_doubles(inst.R) * inst.G)
            assert inst.chunk_size() == chunk
        inst.set_desired_duration(1.5 * dur)
        r = inst.compute_parameterization(0.0, 0.0)
        runs.append([x.cpu().numpy() for x in (r.status, r.sd, r.sdd, r.duration_slow)])
    for x, y in zip(*runs):
        assert _eq(x, y)
    st, sd, sdd, slow = runs[0]
    assert (st[ok] == 0).all()
    for i in np.flatnonzero(ok):
        assert (b[i] * sd[i] ** 2 <= row_limit[i] * (1 + 1e-9)).all()
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        want = min(1.5 * dur[i], slow[i])
        assert abs(got - want) <= 1e-4 * max(1.0, want), (got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch, kind):
    m = model_of("arm6.urdf")
    ss, way, vlim, alim = _problems(10, 6, 61, m.velocity_limit)
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, m, vlim, alim, kind, np.full(10, 2.0)),
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_energy_momentum_terms")
