"""Robots with coupled joints: URDF mimic joints and linear joint couplings q_b = E q + o in the rigid-body model
(RigidBodyModel(coupling=...), from_urdf(couple_mimic=True), with_coupling; libtoppra_b200_dyn.so: tbd_coupled_rnea,
tbd_coupled_torque_terms, tbd_coupling_expand).

CPU:
  * parsing of tests/golden/robots/palletizer.urdf (E, o, DOF and body names, limits), every refused URDF, the
    unchanged refusal without couple_mimic, composition by with_coupling, and the refusals on coupled models;
  * the float64 numpy double of tests/coupled_ref.py equals the 50-digit reduced Lagrangian (E^T M_b E and mpmath.diff
    in q) within 1e-13 of the torque scale: the palletizer with and without the levelling row and a payload, and random
    trees with random couplings (nq = 1..nv, prismatic joints included);
  * the header prototypes, each refused call of the three entries on the real library, and the calls the host makes on
    the recording library (coupled entries, one expansion before every other entry, a coupled solve's launch plan).
GPU:
  * bit-identity: the coupled entries at E = I against tbd_rnea / tbd_torque_terms; tbd_coupled_torque_terms against
    expansion, tbd_torque_terms and the host reduction; every other quantity of a coupled model against the same entry
    on expanded inputs;
  * the kernels against the numpy double within 1e-12 on random trees of 1 to 16 bodies, and the energy identity
    T = 1/2 qd.(tau_q(q, 0, qd) - tau_q(q, 0, 0)) with T from tbd_energy_momentum;
  * the reference golden (tests/golden/coupled_joints.npz, make_golden_coupled.py): TOPPRA and BatchTOPPRA with equal
    statuses; ragged, chunked and B = 1 runs bit-equal; a quintic path against the oracle fed numpy-double rows;
    KineticEnergyConstraint and CartesianVelocityNorm on the coupled model under BatchTOPPRA."""
import ctypes
import os

import numpy as np
import pytest

import coupled_ref as cr
import rnea_ref as rr
import test_dyn_calls
from dyn_common import (DYN_LIB, TB_ERR_ARG, TB_ERR_UNSUPPORTED, _assert_one_terms_launch, _assert_solution, _dev,
                        _dyn_header, _eq, _gpu_present, _model_from_packed, _oracle_joint_rows, _oracle_rows, close,
                        urdf)
from test_collision_energy import PAYLOAD, PAYLOAD_ORIGIN, _urdf_with_payload
from test_dyn_calls import H, T, _OUTPUTS, _context, _flat, _rows_call, _run, calls  # noqa: F401

PALLETIZER = "palletizer.urdf"
BODIES = ["base_yaw", "shoulder_bar_joint", "shoulder", "elbow", "wrist_pitch", "flange_yaw", "finger_left_joint",
          "finger_right_joint", "elbow_bar_joint"]
DOFS = ["base_yaw", "shoulder", "elbow", "wrist_pitch", "flange_yaw", "finger_left_joint"]


def palletizer(level=False, text=None):
    from toppra_b200 import RigidBodyModel
    m = RigidBodyModel.from_urdf(text or urdf(PALLETIZER), couple_mimic=True)
    return m.with_coupling(cr.level_rows(m)) if level else m


def _mp(model, text=None):
    return cr.MpCoupled(rr.MpRobot.from_urdf(text or urdf(PALLETIZER)), *model.coupling)


# ==== CPU: parsing and the model ======================================================================================
def test_palletizer_parsing():
    m = palletizer()
    assert (m.nv, m.nq, m.dof) == (9, 6, 6)
    assert m.body_joint_names == BODIES and m.joint_names == DOFS
    E, o = m.coupling
    want = np.zeros((9, 6))
    for k, n in enumerate(BODIES):
        src = {"shoulder_bar_joint": "shoulder", "elbow_bar_joint": "elbow",
               "finger_right_joint": "finger_left_joint"}.get(n, n)
        want[k, DOFS.index(src)] = -1.0 if n == "finger_right_joint" else 1.0
    assert np.array_equal(E, want)
    assert np.array_equal(o, np.where(np.array(BODIES) == "finger_right_joint", 0.005, 0.0))
    assert np.array_equal(m.packed_coupling, np.r_[want.reshape(-1), o])
    assert np.array_equal(m.effort_limit, [900, 1200, 800, 300, 120, 200])
    assert np.array_equal(m.velocity_limit, [2.0, 2.0, 2.2, 3.0, 3.5, 0.3])
    assert m.torque_limits().shape == (6, 2)
    # locking every mimic joint gives an uncoupled model of the DOFs; URDFs without mimic joints stay uncoupled
    from toppra_b200 import RigidBodyModel
    locked = RigidBodyModel.from_urdf(urdf(PALLETIZER), locked_joints={"shoulder_bar_joint": 0.1,
                                                                       "elbow_bar_joint": 0.2,
                                                                       "finger_right_joint": 0.01})
    assert locked.coupling is None and locked.joint_names == DOFS and locked.nv == locked.nq == 6
    assert RigidBodyModel.from_urdf(urdf("arm6.urdf"), couple_mimic=True).coupling is None


def _edit(old, new):
    text = urdf(PALLETIZER)
    assert old in text
    return text.replace(old, new)


@pytest.mark.parametrize("text,match", [
    (lambda: _edit('<mimic joint="shoulder"/>', '<mimic joint="nope"/>'), "mimics unknown joint 'nope'"),
    (lambda: _edit('<mimic joint="shoulder"/>', '<mimic joint="hand_fixed"/>'), "mimics the fixed joint"),
    (lambda: _edit('<mimic joint="shoulder"/>', '<mimic joint="elbow_bar_joint"/>'), "mimic chains"),
    (lambda: _edit('<mimic joint="shoulder"/>', '<mimic joint="shoulder" multiplier="nan"/>'), "finite"),
])
def test_refused_urdfs(text, match):
    from toppra_b200 import RigidBodyModel
    with pytest.raises(ValueError, match=match):
        RigidBodyModel.from_urdf(text(), couple_mimic=True)


def test_refused_urdf_locked_source_and_unchanged_default():
    from toppra_b200 import RigidBodyModel
    with pytest.raises(ValueError, match="mimics the locked joint 'shoulder'"):
        RigidBodyModel.from_urdf(urdf(PALLETIZER), locked_joints={"shoulder": 0.3}, couple_mimic=True)
    with pytest.raises(ValueError, match="mimic"):
        RigidBodyModel.from_urdf(urdf(PALLETIZER))


def test_with_coupling_composes_and_keeps_payload():
    m = palletizer()
    lv = palletizer(level=True)
    assert lv.nq == 5 and lv.joint_names == ["base_yaw", "shoulder", "elbow", "flange_yaw", "finger_left_joint"]
    assert np.array_equal(lv.velocity_limit, [2.0, 2.0, 2.2, 3.5, 0.3])
    E1 = lv.coupling[0]
    assert np.array_equal(E1[BODIES.index("wrist_pitch")], [0, -1, -1, 0, 0])
    assert lv.body_joint_names == BODIES and np.array_equal(lv.coupling[1], m.coupling[1])
    # a second coupling on top composes: q_b = E_old (E q + o) + o_old
    E2, o2 = np.array([[1.0, 0.0], [0.0, 2.0], [0.0, -1.0], [0.5, 0.0], [0.0, 1.0]]), np.array([0.1, 0, 0.2, 0, 0.3])
    two = lv.with_coupling(E2, o2, joint_names=["a", "b"])
    assert two.joint_names == ["a", "b"] and np.array_equal(two.velocity_limit, [2.0, 0.3])   # rows e_0 and e_1
    assert np.array_equal(two.coupling[0], E1 @ E2) and np.array_equal(two.coupling[1], E1 @ o2 + lv.coupling[1])
    loaded = lv.with_payload("hand", *PAYLOAD)
    assert loaded.joint_names == lv.joint_names and np.array_equal(loaded.packed_coupling, lv.packed_coupling)
    assert loaded.body_joint_names == BODIES
    for bad, match in (((np.ones((4, 2)),), r"expected \(5, n_new\)"), ((E2, np.zeros(3)), "offset has shape"),
                       ((E2 * np.nan,), "finite"), ((np.zeros((5, 2)),), "move no body"),
                       ((E2, None, ["x"]), "joint_names")):
        with pytest.raises(ValueError, match=match):
            lv.with_coupling(*bad)


def test_coupled_model_refusals():
    import toppra_b200 as ta
    m = palletizer()
    with pytest.raises(ValueError, match="coupled joints"):
        ta.Drives(m, gear_ratio=np.ones(6))
    tcp = m.frame("hand")
    for call in (lambda: tcp.inverse_inertia(np.zeros((1, 6))), lambda: tcp.collision_energy_terms(None, None, 1.0),
                 lambda: ta.constraint.CollisionEnergyConstraint(tcp, 1.0, 2.0)):
        with pytest.raises(ValueError, match="coupled joints"):
            call()
    # a joint whose subtree holds some but not all of the bodies of one DOF
    for link in ("upper_arm", "forearm", "shoulder_bar"):
        with pytest.raises(ValueError, match="both sides of joint"):
            ta.constraint.JointWrenchConstraint(m.frame(link, reference_frame="local"), np.ones((6, 2)) * [-1, 1])
    for link in ("wrist", "flange", "hand", "turret"):              # the whole column inside (or outside) the subtree
        m.frame(link)._check_joint_wrench()
    lv = palletizer(level=True)
    with pytest.raises(ValueError, match="both sides of joint 'wrist_pitch'"):
        lv.frame("wrist")._check_joint_wrench()
    from toppra_b200 import RigidBodyModel
    b = m.packed[3:].reshape(9, 27)
    for coupling, match in ((np.ones((9, 6)), "pair"), ((np.ones((9, 10)), np.zeros(9)), "1 <= nq <= 9"),
                            ((np.ones((9, 3)), np.zeros(8)), "expected"), ((np.full((9, 2), np.inf), np.zeros(9)),
                                                                           "finite"),
                            ((np.c_[np.ones(9), np.zeros(9)], np.zeros(9)), "move no body")):
        with pytest.raises(ValueError, match=match):
            RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                           coupling=coupling)


def test_constraints_take_the_path_dof():
    import toppra_b200 as ta
    from toppra_b200.constraint.linear_constraint import RecordContext
    from dyn_common import FakePath
    lv = palletizer(level=True)
    f = lv.frame("hand", xyz=(0, 0, -0.1))
    grid = np.linspace(0, 1, 10)
    cons = [ta.constraint.KineticEnergyConstraint(lv, 1.0), ta.constraint.CartesianVelocityNorm(f, np.eye(6), 1.0),
            ta.constraint.JointTorqueConstraint(lv, lv.torque_limits(), np.zeros(5)),
            ta.constraint.CartesianAccelerationConstraint(f, np.ones((3, 2)) * [-1, 1]),
            ta.constraint.JointWrenchConstraint(lv.frame("flange"), np.ones((6, 2)) * [-1, 1])]
    for c in cons:
        assert c.get_dof() == 5
        c.num_rows(RecordContext(FakePath(3, 5), grid, grid))
    assert f.dof == 5 and f.nv == 9


# ==== CPU: numpy double vs the 50-digit reference =====================================================================
def _check_double_vs_mp(packed, E, o, mp, rng, n=2):
    nq = E.shape[1]
    for _ in range(n):
        q, qs, qss = rng.uniform(-1.5, 1.5, (3, nq))
        c, a, b = mp.terms64(q, qs, qss)
        ad, bd, cd = cr.coupled_torque_terms_packed(packed, E, o, q, qs, qss)
        scale = max(1.0, np.abs(c).max(), np.abs(a).max(), np.abs(b).max())
        for got, want in ((ad[0], a), (bd[0], b), (cd[0], c)):
            assert np.abs(got - want).max() <= 1e-13 * scale, (np.abs(got - want).max(), scale)
        tau = cr.coupled_rnea_packed(packed, E, o, q, qs, qss)[0]
        assert np.abs(tau - (b + c)).max() <= 1e-13 * scale


@pytest.mark.parametrize("level", [False, True])
@pytest.mark.parametrize("payload", [False, True])
def test_numpy_double_matches_mp_reference(level, payload):
    m = palletizer(level)
    text = None
    if payload:
        m = m.with_payload(m.frame("hand", **PAYLOAD_ORIGIN), *PAYLOAD)
        text = _urdf_with_payload(PALLETIZER, "hand")
    _check_double_vs_mp(m.packed, *m.coupling, _mp(m, text), np.random.RandomState(31 + 2 * level + payload))


@pytest.mark.parametrize("nv,nq", [(1, 1), (2, 1), (3, 2), (4, 4), (5, 3), (6, 1)])
def test_numpy_double_random_trees_match_mp_reference(nv, nq):
    rng = np.random.RandomState(700 + 10 * nv + nq)
    packed = rr.random_tree(rng, nv)
    if nv >= 3:
        packed[3:].reshape(nv, 27)[nv // 2, 1] = 1                     # a prismatic joint
    E, o = cr.random_coupling(rng, nv, nq)
    _check_double_vs_mp(packed, E, o, cr.MpCoupled(rr.MpRobot.from_packed(packed), E, o), rng, n=1)


def test_numpy_double_identity_coupling_is_the_tree():
    rng = np.random.RandomState(5)
    packed = rr.random_tree(rng, 7)
    q, qs, qss = rng.uniform(-2, 2, (3, 40, 7))
    E, o = np.eye(7), np.zeros(7)
    assert np.array_equal(cr.coupled_rnea_packed(packed, E, o, q, qs, qss), rr.rnea_packed(packed, q, qs, qss))
    for x, y in zip(cr.coupled_torque_terms_packed(packed, E, o, q, qs, qss, np.arange(7.0)),
                    rr.torque_terms_packed(packed, q, qs, qss, np.arange(7.0))):
        assert np.array_equal(x, y)


# ==== CPU: header, C-ABI checks ======================================================================================
def test_dyn_header_prototypes_of_coupled_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_coupled_rnea"] == ["ptr", "int", "ptr", "int", "int"] + ["ptr"] * 5
    assert declared["tbd_coupled_torque_terms"] == ["ptr", "int", "ptr", "int", "int"] + ["ptr"] * 8
    assert declared["tbd_coupling_expand"] == ["int", "ptr", "int", "int"] + ["ptr"] * 7
    for name in ("tbd_coupled_rnea", "tbd_coupled_torque_terms", "tbd_coupling_expand"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_coupled_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = palletizer()

    def err():
        return _lib.load().tb_last_error()

    def calls(model=m.packed, nv=9, coupling=m.packed_coupling, nq=6, M=4, null=False):
        host = np.array(model, dtype=np.float64)
        cp = np.array(coupling, dtype=np.float64)
        mp, cpp = ctypes.c_void_p(host.ctypes.data), None if null else ctypes.c_void_p(cp.ctypes.data)
        args = {"tbd_coupled_rnea": [mp, nv, cpp, nq, M] + [d] * 4,
                "tbd_coupled_torque_terms": [mp, nv, cpp, nq, M] + [d] * 7,
                "tbd_coupling_expand": [nv, cpp, nq, M] + [d] * 6}
        out = {}
        for name, a in args.items():
            out[name] = (getattr(lib, name)(*a, None), err())
        return out

    def expect(rc, msg, **kw):
        for name, (got, e) in calls(**kw).items():
            if name == "tbd_coupling_expand" and "model" in kw:
                continue                                            # no model
            assert got == rc and e.startswith(name.encode() + b": ") and msg in e, (name, got, e)

    expect(TB_ERR_ARG, b"null pointer", null=True)                 # the coupling
    for nq in (0, 10, -1):
        expect(TB_ERR_UNSUPPORTED, b"nq=%d outside 1..nv=9" % nq, nq=nq)
    expect(TB_ERR_UNSUPPORTED, b"nq=7 outside 1..nv=6",
           model=m.packed[:3 + 27 * 6], nv=6, coupling=np.r_[np.ones(42), np.zeros(6)], nq=7)
    for M in (0, -2):
        expect(TB_ERR_ARG, b"M=%d must be positive" % M, M=M)
    for j in (0, 17, 54, 57):
        bad = m.packed_coupling.copy()
        bad[j] = np.nan if j % 2 else np.inf
        expect(TB_ERR_ARG, b"coupling E or o is not finite", coupling=bad)
    bad = m.packed_coupling.copy()
    bad[:54].reshape(9, 6)[:, 3] = 0.0
    expect(TB_ERR_ARG, b"DOF 3 moves no body (column 3 of E is zero)", coupling=bad)
    badm = m.packed.copy()
    badm[3 + 27 * 2 + 17] = -1.0
    expect(TB_ERR_ARG, b"body 2: mass", model=badm)
    # the expansion: nv outside 1..16, a rate without its output and the reverse
    cp = ctypes.c_void_p(m.packed_coupling.ctypes.data)
    assert lib.tbd_coupling_expand(0, cp, 1, 4, d, d, d, d, d, d, None) == TB_ERR_UNSUPPORTED
    assert b"nv=0 outside 1..16" in err()
    for args in ((d, None, d, d, d, d), (d, d, d, d, d, None), (d, d, None, d, d, None)):
        rc = lib.tbd_coupling_expand(9, cp, 6, 4, *args, None)
        if args == (d, d, None, d, d, None):                         # both rates of qdd NULL: valid
            assert rc not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED) and b"launch failed" in err()
        else:
            assert rc == TB_ERR_ARG and b"both be given or both be NULL" in err()
    for name, (rc, e) in calls().items():                          # good calls fail only at the launch (no device)
        assert rc not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED) and b"launch failed" in e, name


# ==== CPU: the calls on the recording library ========================================================================
@pytest.fixture
def recorder(calls, monkeypatch):  # noqa: F811
    orig = test_dyn_calls._host_doubles

    def host_doubles(name, slot, args):
        if name in ("tbd_coupled_rnea", "tbd_coupled_torque_terms"):
            return {0: 3 + 27 * args[1], 2: args[1] * args[3] + args[1]}.get(slot)
        if name == "tbd_coupling_expand":
            return args[0] * args[2] + args[0] if slot == 1 else None
        return orig(name, slot, args)

    monkeypatch.setattr(test_dyn_calls, "_host_doubles", host_doubles)
    for name, n in (("tbd_coupled_rnea", 1), ("tbd_coupled_torque_terms", 3), ("tbd_coupling_expand", 3),
                    ("tbd_energy_momentum_terms", 1), ("tbd_energy_momentum", 1)):
        monkeypatch.setitem(_OUTPUTS, name, n)
    return calls


def test_model_and_frame_calls(recorder):
    from test_dyn_calls import _canon, _dev as fake
    m = palletizer(level=True)
    nv, nq, M = 9, 5, 4
    rng = np.random.default_rng(2)
    x = {k: fake(rng.uniform(-1, 1, (M, nq))) for k in ("q", "qd", "qdd")}
    Q, QD, QDD = T("q", (M, nq)), T("qd", (M, nq)), T("qdd", (M, nq))
    tau = m(x["q"], x["qd"], x["qdd"])
    assert _canon(recorder, dict(x, out=tau)) == [
        ["tbd_coupled_rnea", H(m.packed), nv, H(m.packed_coupling), nq, M, Q, QD, QDD, T("out", (M, nq)), None]]
    del recorder[:]
    a, b, c = m.torque_terms(x["q"], x["qd"], x["qdd"], 0.5)
    assert _canon(recorder, dict(x, a=a, b=b, c=c)) == [
        ["tbd_coupled_torque_terms", H(m.packed), nv, H(m.packed_coupling), nq, M, Q, QD, QDD,
         T((0.5,) * nq, (nq,)), T("a", (M, nq)), T("b", (M, nq)), T("c", (M, nq)), None]]
    f = m.frame("hand", xyz=(0, 0, -0.1))
    for run, name, rates, middle, shapes in (
            (lambda: f(x["q"], x["qd"]), "tbd_frame_velocity", 1, [H(f.packed)], [(M, 6)]),
            (lambda: f.acceleration(x["q"], x["qd"], x["qdd"]), "tbd_frame_acceleration", 2, [H(f.packed)], [(M, 6)]),
            (lambda: m.energy_momentum(x["q"], x["qd"])[0], "tbd_energy_momentum", 1, [], [(M, 4)])):
        del recorder[:]
        out = run()
        log = _canon(recorder, dict(x))
        ex = "tbd_coupling_expand"
        outs = [T("%s.%d" % (ex, 7 + i), (M, nv)) if i <= rates else None for i in range(3)]
        assert log[0] == [ex, nv, H(m.packed_coupling), nq, M, Q, QD, QDD if rates == 2 else None] + outs + [None]
        assert log[1] == ([name, H(m.packed), nv] + middle + [M] + [o for o in outs if o is not None]
                          + [T("%s.%d" % (name, 4 + len(middle) + rates + i), s) for i, s in enumerate(shapes)]
                          + [None]), name
        assert len(log) == 2 and out is not None


@pytest.mark.parametrize("lo,hi,total", [(0, 4, 4), (1, 3, 4)])
@pytest.mark.parametrize("interp", [False, True])
def test_launch_plan_of_coupled_solves(recorder, lo, hi, total, interp):
    from toppra_b200.constraint import JointTorqueConstraint, KineticEnergyConstraint
    m = palletizer(level=True)
    nv, nq, G = 9, 5, 6
    B, n = hi - lo, (hi - lo) * G
    fric = np.arange(nq) * 0.1
    lim = m.torque_limits()
    cons = JointTorqueConstraint(m, lim, fric, discretization_scheme=int(interp))
    ctx, bp = _context(nq, total, G, lo, hi, total)
    rows, log = _run(recorder, cons, ctx)
    assert rows == (2 if interp else 1) * 2 * nq
    name = "tbd_coupled_torque_terms"
    g = np.concatenate((lim[:, 1], -lim[:, 0]))
    assert log == [
        [name, H(m.packed), nv, H(m.packed_coupling), nq, n, T("q0", (n, nq)), T("q1", (n, nq)), T("q2", (n, nq)),
         T(_flat(fric), (nq,)), T(name + ".9", (n, nq)), T(name + ".10", (n, nq)), T(name + ".11", (n, nq)), None],
        _rows_call(*[T(name + ".%d" % s, (B, G, nq)) for s in (9, 10, 11)], None, T(_flat(g), g.shape), 2, B, G, nq,
                   2 * nq, interp)]
    cons = KineticEnergyConstraint(m, 2.5, discretization_scheme=int(interp))
    ctx, bp = _context(nq, total, G, lo, hi, total)
    rows, log = _run(recorder, cons, ctx)
    ex, name = "tbd_coupling_expand", "tbd_energy_momentum_terms"
    assert log == [
        [ex, nv, H(m.packed_coupling), nq, n, T("q0", (n, nq)), T("q1", (n, nq)), None, T(ex + ".7", (n, nv)),
         T(ex + ".8", (n, nv)), None, None],
        [name, H(m.packed), nv, 0, n, T(ex + ".7", (n, nv)), T(ex + ".8", (n, nv)), T(name + ".6", (n,)), None],
        _rows_call(T((0.0,) * (B * G), (B, G, 1)), T(name + ".6", (B, G, 1)), T((-2.5,) * (B * G), (B, G, 1)),
                   T((1.0,), (1, 1)), T((0.0,), (1,)), 0, B, G, 1, 1, interp)]


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _uncoupled(ta, m):
    """The same tree without a coupling: the body-space model."""
    b = m.packed[3:].reshape(m.nv, 27)
    return ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                             gravity=m.gravity, frames=m.frames, base_mass=m.base_mass, base_com=m.base_com)


@pytest.mark.gpu
def test_gpu_identity_coupling_bit_equal_tree(ta):
    import torch
    rng = np.random.RandomState(3)
    for packed in (rr.random_tree(rng, 16), rr.random_tree(rng, 5), palletizer().packed):
        tree = _model_from_packed(ta, packed)
        nv = tree.nv
        same = tree.with_coupling(np.eye(nv))
        assert same.coupling is not None
        q, qd, qdd = (_dev(rng.uniform(-2, 2, (3000, nv))) for _ in range(3))
        qd[:5] = 0.0
        assert torch.equal(same(q, qd, qdd), tree(q, qd, qdd))
        for fric in (None, np.linspace(0.1, 1.0, nv)):
            for x, y in zip(same.torque_terms(q, qd, qdd, fric), tree.torque_terms(q, qd, qdd, fric)):
                assert torch.equal(x, y)


def _host_reduce(torch, E, t):
    """E^T t in the fixed order of the library, with torch operations: (M, nv) -> (M, nq)."""
    cols = []
    for j in range(E.shape[1]):
        s = None
        for k in range(E.shape[0]):
            if E[k, j] != 0:
                u = float(E[k, j]) * t[:, k]
                s = u if s is None else s + u
        cols.append(s)
    return torch.stack(cols, dim=1)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [False, True])
def test_gpu_fused_terms_bit_equal_expand_then_tree(ta, level):
    import torch
    from toppra_b200 import dynamics
    m = palletizer(level).with_payload("hand", *PAYLOAD)
    tree = _uncoupled(ta, m)
    E, o = m.coupling
    rng = np.random.RandomState(11)
    q, qs, qss = (_dev(rng.uniform(-2, 2, (4000, m.nq))) for _ in range(3))
    qs[:6] = 0.0
    qb, qsb, qssb = dynamics._expand(torch, ta._lib_dyn.load(), m, [q, qs, qss])
    for got, x, pos in ((qb, q, True), (qsb, qs, False), (qssb, qss, False)):   # the expansion: the numpy double
        assert _eq(got.cpu().numpy(), cr.expand(E, o, x.cpu().numpy(), pos))
    fric = np.linspace(1.0, 3.0, m.nq)
    a, b, c = m.torque_terms(q, qs, qss, fric)
    ab, bb, cb = tree.torque_terms(qb, qsb, qssb)
    assert torch.equal(a, _host_reduce(torch, E, ab)) and torch.equal(b, _host_reduce(torch, E, bb))
    assert torch.equal(c, _host_reduce(torch, E, cb) + torch.sign(qs) * torch.as_tensor(fric, device=q.device))
    assert torch.equal(m(q, qs, qss), _host_reduce(torch, E, tree(qb, qsb, qssb)))


@pytest.mark.gpu
def test_gpu_other_quantities_bit_equal_expanded_tree(ta):
    import torch
    m = palletizer(level=True)
    tree = _uncoupled(ta, m)
    E, o = m.coupling
    rng = np.random.RandomState(17)
    q, qd, qdd = (rng.uniform(-2, 2, (2000, m.nq)) for _ in range(3))
    x = [_dev(v) for v in (q, qd, qdd)]
    xb = [_dev(cr.expand(E, o, v, pos)) for v, pos in ((q, True), (qd, False), (qdd, False))]
    obj = np.array([0.8, 0.006, -0.004, 0.06, 0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017])
    humans = np.array([[0.9, 0.2, 1.0, 0.2], [-0.5, 0.8, 0.6, 0.15]])
    S = np.diag([1.0, 1.0, 1.0, 0.1, 0.1, 0.1])
    for name, kw in (("hand", dict(xyz=(0, 0, -0.1))), ("flange", dict(reference_frame="local"))):
        f, fb = m.frame(name, **kw), tree.frame(name, **kw)
        for get in (lambda f, q, qd, qdd: f(q, qd), lambda f, q, qd, qdd: f.velocity_norm_terms(q, qd, S),
                    lambda f, q, qd, qdd: f.acceleration(q, qd, qdd),
                    lambda f, q, qd, qdd: f.acceleration_terms(q, qd, qdd, (0, 4)),
                    lambda f, q, qd, qdd: f.contact_wrench(obj, q, qd, qdd),
                    lambda f, q, qd, qdd: f.contact_wrench_terms(obj, q, qd, qdd),
                    lambda f, q, qd, qdd: f.joint_wrench(q, qd, qdd),
                    lambda f, q, qd, qdd: f.joint_wrench_terms(q, qd, qdd, (1, 5))):
            got, want = get(f, *x), get(fb, *xb)
            for g_, w_ in zip(got if isinstance(got, tuple) else (got,), want if isinstance(want, tuple) else (want,)):
                assert torch.equal(g_, w_)
    base = m.frame("world")
    for got, want in ((base.support_wrench(None, *x), tree.frame("world").support_wrench(None, *xb)),
                      (m.energy_momentum(x[0], x[1])[1], tree.energy_momentum(xb[0], xb[1])[1]),
                      (m.energy_momentum_terms(x[0], x[1], "energy"), tree.energy_momentum_terms(xb[0], xb[1], "energy"))):
        assert torch.equal(got, want)
    for got, want in zip(base.support_wrench_terms(None, *x), tree.frame("world").support_wrench_terms(None, *xb)):
        assert torch.equal(got, want)
    from toppra_b200.dynamics import pack_points
    pts = pack_points([(m.frame("hand"), 0.05), (m.frame("elbow_bar"), m.frame("forearm"), 0.08)])[1]
    for got, want in zip(m.separation(pts, humans, x[0], x[1]), tree.separation(pts, humans, xb[0], xb[1])):
        assert torch.equal(got, want)
    for got, want in zip(m.separation_terms(pts, humans, 0.1, 2.0, 1.6, 0.05, x[0], x[1]),
                         tree.separation_terms(pts, humans, 0.1, 2.0, 1.6, 0.05, xb[0], xb[1])):
        assert torch.equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_random_trees_vs_numpy_double(ta, nv):
    rng = np.random.RandomState(2100 + nv)
    packed = rr.random_tree(rng, nv)
    if nv >= 3:
        packed[3:].reshape(nv, 27)[nv // 2, 1] = 1
    for nq in sorted({1, max(1, nv // 2), nv}):
        E, o = cr.random_coupling(rng, nv, nq)
        m = _model_from_packed(ta, packed).with_coupling(E, o)
        q, qs, qss = rng.uniform(-2, 2, (3, 500, nq))
        fric = rng.uniform(0, 1, nq)
        got = [t.cpu().numpy() for t in m.torque_terms(_dev(q), _dev(qs), _dev(qss), fric)]
        for g_, w_ in zip(got, cr.coupled_torque_terms_packed(packed, E, o, q, qs, qss, fric)):
            close(g_, w_, 1e-12)
        close(m(_dev(q), _dev(qs), _dev(qss)).cpu().numpy(), cr.coupled_rnea_packed(packed, E, o, q, qs, qss), 1e-12)
        assert np.array_equal(m(q[7], qs[7], qss[7]), m(_dev(q[7:8]), _dev(qs[7:8]), _dev(qss[7:8])).cpu().numpy()[0])


@pytest.mark.gpu
def test_gpu_energy_identity_in_q_space(ta):
    import torch
    rng = np.random.RandomState(23)
    for m in (palletizer(), palletizer(level=True).with_payload("hand", *PAYLOAD),
              _model_from_packed(ta, rr.random_tree(rng, 11)).with_coupling(*cr.random_coupling(rng, 11, 6))):
        q, qd = (_dev(rng.uniform(-2, 2, (2000, m.nq))) for _ in range(2))
        zero = torch.zeros_like(q)
        Tg = m.energy_momentum(q, qd)[0]
        Ti = 0.5 * (qd * (m(q, zero, qd) - m(q, zero, zero))).sum(dim=1)
        assert float((Tg - Ti).abs().max()) <= 1e-12 * float(Tg.abs().max())
        assert (Tg >= 0).all()


def _torque_cons(ta, m, vlim, alim, taulim, fric, scheme=0):
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
            ta.constraint.SecondOrderConstraint.joint_torque_constraint(m, taulim, fric, discretization_scheme=scheme)]


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["free", "level"])
def test_gpu_reference_golden(ta, golden, which):
    g = golden("coupled_joints")
    m = palletizer(which == "level")
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim, taulim, fs = (g["%s/%s" % (which, k)] for k in ("way", "vlim", "alim", "taulim", "fs"))
    B = way.shape[0]
    statuses = set()
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (which, scheme, x)][i]  # noqa: E731
        for i in range(B):                                         # shared limits on each path alone
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                       ta.constraint.JointAccelerationConstraint(alim[i], discretization_scheme=scheme),
                                       ta.constraint.JointTorqueConstraint(m, taulim[i], fs,
                                                                           discretization_scheme=scheme)],
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fs, scheme), ta.BatchSplineInterpolator(ss, way),
                           grid).compute_parameterization(0, 0).to_host()   # per-path limits
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))
            statuses.add(int(h["status"][i]))
    assert 0 in statuses and len(statuses) > 1                    # the last path's torque limit makes it infeasible


def _problems(B, m, seed):
    rng = np.random.RandomState(seed)
    nq = m.nq
    way = np.cumsum(rng.uniform(-0.5, 0.5, (B, 5, nq)), axis=1)
    vlim = np.tile(np.stack([-m.velocity_limit, m.velocity_limit], axis=1), (B, 1, 1))
    al = rng.uniform(4, 8, (B, nq))
    tl = 0.5 * m.effort_limit * rng.uniform(0.8, 1.2, (B, nq))
    return np.linspace(0, 1, 5), way, vlim, np.stack([-al, al], axis=-1), np.stack([-tl, tl], axis=-1)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta):
    m = palletizer(level=True).with_payload("hand", *PAYLOAD)
    B = 12
    ss, way, vlim, alim, taulim = _problems(B, m, 41)
    fric = np.full(m.nq, 1.5)
    path = ta.BatchSplineInterpolator(ss, way)
    rag = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_torque_cons(ta, m, vlim[i:i + 1], alim[i:i + 1], taulim[i:i + 1], fric),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric, scheme), path, grid,
                               max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
        assert (hw["status"] == 0).any()
    for i in range(3):
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                       ta.constraint.JointAccelerationConstraint(alim[i], discretization_scheme=scheme),
                                       ta.constraint.JointTorqueConstraint(m, taulim[i], fric,
                                                                           discretization_scheme=scheme)],
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_torque_cons(ta, m, vlim[i:i + 1], alim[i:i + 1], taulim[i:i + 1], fric, scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0)
            hb = hb.to_host()
            assert sd is not None and _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])


@pytest.mark.gpu
def test_gpu_quintic_path_vs_oracle(ta):
    from oracle import oracle as orc
    m = palletizer(level=True)
    B, nq, nseg, k = 6, m.nq, 3, 6
    rng = np.random.RandomState(43)
    coeffs = rng.uniform(-0.3, 0.3, (B, k, nseg, nq))
    path = ta.BatchPiecewisePolyPath(np.linspace(0, 1, nseg + 1), coeffs)
    grid = np.linspace(0, 1, 120)
    vlim = np.tile(np.stack([-m.velocity_limit, m.velocity_limit], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nq, 6.0), np.full(nq, 6.0)], axis=1), (B, 1, 1))
    taulim = np.tile(0.5 * m.torque_limits(), (B, 1, 1))
    fric = np.full(nq, 2.0)
    h = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, grid).compute_parameterization(0, 0)
    h = h.to_host()
    assert (h["status"] == 0).sum() >= B // 2
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    F = np.vstack((np.eye(nq), -np.eye(nq)))
    E, o_ = m.coupling
    for i in range(B):
        a, b, c = cr.coupled_torque_terms_packed(m.packed, E, o_, qs[0][i], qs[1][i], qs[2][i], fric)
        g = np.concatenate((taulim[i, :, 1], -taulim[i, :, 0]))
        rows = _oracle_rows(F, a, b, c, grid, False)
        rows[:, 2, :] = rows[:, 2, :] - g
        o = orc.solve_rows(np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]), rows), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])


@pytest.mark.gpu
def test_gpu_kinetic_energy_and_tool_speed_on_coupled_model(ta, monkeypatch):
    m = palletizer(level=True)
    ss, way, vlim, alim, taulim = _problems(10, m, 47)
    path = ta.BatchSplineInterpolator(ss, way)
    grid = np.linspace(0, 1, 80)
    tcp = m.frame("hand", xyz=(0, 0, -0.15))
    for extra in (ta.constraint.KineticEnergyConstraint(m, 40.0),
                  ta.constraint.CartesianVelocityNorm(tcp, np.diag([1.0, 1.0, 1.0, 0, 0, 0]), 1.0)):
        base = [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]
        h = ta.BatchTOPPRA(base + [extra], path, grid).compute_parameterization(0, 0).to_host()
        free = ta.BatchTOPPRA(base, path, grid).compute_parameterization(0, 0).to_host()
        assert (h["status"] == 0).all() and (h["sd"] <= free["sd"] * (1 + 1e-12)).all()
        assert (h["sd"] < free["sd"] * (1 - 1e-6)).any()               # the limit binds somewhere
    _assert_one_terms_launch(ta, monkeypatch, lambda: _torque_cons(ta, m, vlim, alim, taulim, np.ones(m.nq)), path,
                             grid, "tbd_coupled_torque_terms")
