"""Collision-energy limits next to people: the inverse operational-space inertia of a robot frame and the energy a
collision at its origin could transfer (RigidBodyFrame.inverse_inertia / collision_energy_terms,
CollisionEnergyConstraint, RigidBodyModel.with_payload; libtoppra_b200_dyn.so: tbd_frame_inverse_inertia,
tbd_collision_energy_terms).

CPU:
  * the float64 numpy double of tests/energy_ref.py equals the 50-digit reference (mass matrix of the RAW URDF tree,
    J_v by mpmath.diff, mpmath.lu_solve) to 1e-13 of the scale: every link frame of both fixtures, locked and
    unlocked, with the usual offset, Lambda_v^-1 in both axes and b;
  * hand cases with closed forms (a prismatic body, a revolute body, a frame on the base, q' = 0) on the numpy double;
  * with_payload against from_urdf of the fixture with an extra fixed child link, and its torques against the 50-digit
    RNEA reference of that URDF;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library.
GPU:
  * both kernels on random trees (1 to 16 bodies) against the 50-digit reference within 1e-14 cond(M) of the scale;
  * the hand cases; b <= 1/2 q'.(M q') (M q' from tbd_torque_terms) with equality where q' = M^-1 J_v^T e;
    invariances (reference-frame field, local vs world axes, monotone in m_H);
  * tbd_collision_energy_terms equals tbd_frame_inverse_inertia, tbd_frame_velocity and the torch operations bit for bit;
    NaN in one point touches no other; a model whose M is singular at some q gives NaN exactly there;
  * the reference golden (tests/golden/collision_energy.npz, make_golden_collision_energy.py) and 256 paths with
    per-path limits against the oracle fed with rows from the numpy double: within |dK| <= 1e-9 + 1e-8 |K| (the cfg-3
    tolerance); the energy of the solved profiles stays within the limit, and the limit is active;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, host route vs device route:
    bit-equal; BatchTOPPRAsd, a quintic BatchPiecewisePolyPath, and the constraint next to torque and tool-speed limits
    against the oracle; one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import energy_ref as er
import kin_ref as kr
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, FakePath, LOCKED, OFFSET, TB_ERR_ARG, TB_ERR_UNSUPPORTED, model_of, urdf,
                        _assert_one_terms_launch, _assert_solution, _dev, _dyn_header, _eq, _gpu_present,
                        _model_from_packed, _problems)

HUMAN_MASS = 0.6


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.max(np.abs(np.asarray(got) - ref)) / max(float(np.max(np.abs(ref))), 1e-300))


def _spec(off):
    from toppra_b200.dynamics import rpy_matrix
    return (rpy_matrix(off["rpy"]) if off else np.eye(3)), (np.asarray(off["xyz"]) if off else np.zeros(3))


def _mpf(x):
    return np.array(x.tolist(), dtype=np.float64)


# ==== CPU: numpy double vs the 50-digit reference, hand cases, payloads, errors, C-ABI ================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 91)
    worst = 0.0
    for _ in range(2):
        q, qs = rng.uniform(-2, 2, m.nv), rng.uniform(-1.5, 1.5, m.nv)
        spec = {}
        for link in m.frames:
            for o, off in enumerate((None, OFFSET)):
                spec[(link, o)] = (link,) + _spec(off)
        ref = er.mp_inverse_inertia(mp, q, spec)
        for (link, o), _ in spec.items():
            off = OFFSET if o else {}
            Wm, Rm = _mpf(ref[(link, o)][0]), _mpf(ref[(link, o)][1])
            J = ref[((link, o), "J")]
            for ref_frame, want in (("local_world_aligned", Wm), ("local", Rm.T @ Wm @ Rm)):
                f = m.frame(link, reference_frame=ref_frame, **off)
                W = er.inverse_inertia_packed(m.packed, f.packed, q)[0]
                if m.frames[link][0] < 0:
                    assert not W.any()                           # a frame on the base: Lambda_v^-1 = 0
                    continue
                worst = max(worst, rel_err(W, want))
            for mh in (HUMAN_MASS, np.inf):
                b = er.energy_terms_packed(m.packed, f.packed, q, qs, mh)[0]
                bm = float(er.mp_energy_b(J, ref[(link, o)][0], qs, mh))
                if m.frames[link][0] < 0 or bm == 0:               # on the base, or on a joint axis
                    assert b == 0.0 and bm == 0.0
                    continue
                worst = max(worst, abs(b - bm) / bm)
    print("worst relative error of the numpy double: %.2e" % worst)
    assert worst <= 1e-13


def _prismatic_model(ta, mass):
    return ta.RigidBodyModel([-1], ["prismatic"], [[0.0, 0.6, 0.8]], [np.eye(3)], [[0.1, 0.2, 0.3]], [mass],
                             [[0.05, -0.02, 0.1]], [[0.01, 0.0, 0.0, 0.02, 0.0, 0.03]])


def _revolute_model(ta):
    """One revolute body about the world z axis: I_axis = Izz + m (cx^2 + cy^2)."""
    return ta.RigidBodyModel([-1], ["revolute"], [[0.0, 0.0, 1.0]], [np.eye(3)], [[0.0, 0.0, 0.5]], [2.0],
                             [[0.2, 0.1, 0.3]], [[0.04, 0.001, 0.002, 0.05, 0.003, 0.06]])


def _hand_cases(ta, L_of, b_of):
    """L_of(frame, q (P, nv)) -> (P, 3, 3); b_of(frame, q, qs, m_H) -> (P,)."""
    rng = np.random.RandomState(3)
    # one prismatic body of mass m: m_R = m along the axis, b = 1/2 m m_H / (m + m_H) q'^2
    m = 3.5
    pm = _prismatic_model(ta, m)
    f = pm.frame("body0", xyz=(0.3, -0.1, 0.2))
    q, qs = rng.uniform(-1, 1, (5, 1)), rng.uniform(-2, 2, (5, 1))
    ax = np.array([0.0, 0.6, 0.8])
    for Lw in L_of(f, q):
        np.testing.assert_allclose(Lw, np.outer(ax, ax) / m, rtol=0, atol=1e-15)
    for mh in (HUMAN_MASS, 75.0, np.inf):
        want = 0.5 * (m if np.isinf(mh) else m * mh / (m + mh)) * qs[:, 0] ** 2
        np.testing.assert_allclose(b_of(f, q, qs, mh), want, rtol=1e-14)
    # one revolute body, the frame at distance d from the axis: Lambda_v^-1 = (d^2 / I_axis) t t^T
    rm = _revolute_model(ta)
    I_axis = 0.06 + 2.0 * (0.2 ** 2 + 0.1 ** 2)
    for xyz in ((0.7, 0.0, 0.1), (0.3, -0.4, -0.2)):
        f = rm.frame("body0", xyz=xyz)
        q = rng.uniform(-3, 3, (4, 1))
        d = np.hypot(xyz[0], xyz[1])
        for qi, Lw in zip(q[:, 0], L_of(f, q)):
            p = np.array([np.cos(qi) * xyz[0] - np.sin(qi) * xyz[1], np.sin(qi) * xyz[0] + np.cos(qi) * xyz[1], 0.0])
            t = np.cross([0.0, 0.0, 1.0], p) / d
            np.testing.assert_allclose(Lw, d * d / I_axis * np.outer(t, t), rtol=0, atol=1e-14)
    # a frame on the base: Lambda_v^-1 = 0 and b = 0
    arm = model_of("arm6.urdf")
    f = arm.frame("base_link", xyz=(0.1, 0.2, 0.3))
    q, qs = rng.uniform(-2, 2, (3, 6)), rng.uniform(-2, 2, (3, 6))
    assert not np.asarray(L_of(f, q)).any()
    b = np.asarray(b_of(f, q, qs, HUMAN_MASS))
    assert (b == 0).all() and not np.signbit(b).any()
    # q' = 0: b = +0
    f = arm.frame("flange", xyz=(0.0, 0.0, 0.1))
    b = np.asarray(b_of(f, q, 0 * qs, HUMAN_MASS))
    assert (b == 0).all() and not np.signbit(b).any()


def test_hand_cases_numpy_double():
    import toppra_b200 as ta
    _hand_cases(ta, lambda f, q: er.inverse_inertia_packed(f.model.packed, f.packed, q),
                lambda f, q, qs, mh: er.energy_terms_packed(f.model.packed, f.packed, q, qs, mh))


PAYLOAD = (1.3, (0.01, -0.02, 0.05), (0.004, 0.0002, -0.0001, 0.005, 0.0003, 0.003))
PAYLOAD_ORIGIN = dict(xyz=(0.02, 0.01, 0.07), rpy=(0.4, -0.3, 0.2))


def _urdf_with_payload(name, parent_link):
    """The fixture with a fixed child link of `parent_link` at PAYLOAD_ORIGIN carrying PAYLOAD's inertial."""
    m, c, I = PAYLOAD
    xyz, rpy = PAYLOAD_ORIGIN["xyz"], PAYLOAD_ORIGIN["rpy"]
    fmt = lambda v: " ".join(repr(float(x)) for x in v)  # noqa: E731
    extra = ('<link name="payload"><inertial><origin xyz="%s" rpy="0 0 0"/><mass value="%r"/>'
             '<inertia ixx="%r" ixy="%r" ixz="%r" iyy="%r" iyz="%r" izz="%r"/></inertial></link>'
             '<joint name="payload_mount" type="fixed"><parent link="%s"/><child link="payload"/>'
             '<origin xyz="%s" rpy="%s"/></joint>' % ((fmt(c), m) + tuple(I) + (parent_link, fmt(xyz), fmt(rpy))))
    text = urdf(name)
    return text.replace("</robot>", extra + "</robot>")


@pytest.mark.parametrize("name,locked,link", [("arm6.urdf", None, "flange"), ("arm7_gripper.urdf", LOCKED, "hand"),
                                              ("arm7_gripper.urdf", None, "finger_left")])
def test_with_payload_matches_urdf(name, locked, link):
    from toppra_b200 import RigidBodyModel
    m = model_of(name, locked)
    text = _urdf_with_payload(name, link)
    want = RigidBodyModel.from_urdf(text, locked_joints=locked)
    for frame in (m.frame(link, **PAYLOAD_ORIGIN), ):
        got = m.with_payload(frame, *PAYLOAD)
        assert rel_err(got.packed, want.packed) <= 1e-14
        assert got.joint_names == m.joint_names and set(got.frames) == set(m.frames)
        assert np.array_equal(got.effort_limit, m.effort_limit) and np.array_equal(got.velocity_limit, m.velocity_limit)
    # by name, without an offset: the payload's frame is the link itself
    got = m.with_payload(link, PAYLOAD[0], PAYLOAD[1], PAYLOAD[2])
    assert np.array_equal(got.packed[:3], m.packed[:3])
    # torques of the loaded model against the 50-digit RNEA reference of the URDF with the payload link
    loaded = m.with_payload(m.frame(link, **PAYLOAD_ORIGIN), *PAYLOAD)
    mp = rr.MpRobot.from_urdf(text, locked)
    rng = np.random.RandomState(5)
    q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
    tau = rr.rnea_packed(loaded.packed, q, qd, qdd)[0]
    want = mp.tau64(q, qd, qdd)
    assert np.max(np.abs(tau - want)) <= 1e-13 * max(1.0, np.max(np.abs(want)))
    assert not np.allclose(rr.rnea_packed(m.packed, q, qd, qdd)[0], want, rtol=1e-6)   # the payload matters


def test_value_errors():
    import toppra_b200 as ta
    from toppra_b200.constraint import CollisionEnergyConstraint
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    with pytest.raises(ValueError, match="RigidBodyFrame"):
        CollisionEnergyConstraint(lambda q, qd: np.zeros(6), 1.0, HUMAN_MASS)
    for lim in (-1.0, np.nan, [1.0, -0.1], [np.nan, 1.0]):
        with pytest.raises(ValueError, match=">= 0"):
            CollisionEnergyConstraint(f, lim, HUMAN_MASS)
    with pytest.raises(ValueError, match="float or"):
        CollisionEnergyConstraint(f, np.ones((2, 2)), HUMAN_MASS)
    for mh in (0.0, -1.0, np.nan, -np.inf):
        with pytest.raises(ValueError, match="human_mass"):
            CollisionEnergyConstraint(f, 1.0, mh)
    c = CollisionEnergyConstraint(f, 0.0, np.inf)                     # zero limit and m_H = inf are fine
    grid = np.linspace(0, 1, 10)
    assert c.dof == 6 and c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    assert CollisionEnergyConstraint(f, 1.0, HUMAN_MASS, discretization_scheme=1).num_rows(
        RecordContext(FakePath(3, 6), grid, grid)) == 2
    with pytest.raises(ValueError, match="Wrong dimension"):
        c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
    per_path = CollisionEnergyConstraint(f, [1.0, 2.0, 3.0], HUMAN_MASS)
    assert per_path.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    with pytest.raises(ValueError, match="expected a float or"):
        per_path.num_rows(RecordContext(FakePath(4, 6), grid, grid))

    class _Path(object):
        dof = 7
    with pytest.raises(ValueError, match="Wrong dimension"):
        c.compute_constraint_params(_Path(), grid)
    with pytest.raises(ValueError, match="single path"):
        per_path.compute_constraint_params(type("P", (), {"dof": 6})(), grid)
    # a joint that moves no inertia: its body and descendants are massless
    b = rr.random_tree(np.random.RandomState(2), 4)[3:].reshape(4, 27).copy()
    b[:, 0] = [-1, 0, 1, 2]
    b[2:, 17] = 0.0
    b[2:, 21:27] = 0.0
    dead = ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                             joint_names=["a", "b", "c", "d"])
    assert dead.inertialess_joints() == ["c", "d"]
    with pytest.raises(ValueError, match="'c', 'd'"):
        CollisionEnergyConstraint(dead.frame("body1"), 1.0, HUMAN_MASS)
    b[3, 17] = 0.5                                                     # now d moves a mass, and so c moves it too
    alive = ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27])
    assert alive.inertialess_joints() == []
    with pytest.raises(ValueError, match="world"):
        m.frame("flange", reference_frame="world").inverse_inertia(np.zeros(6))
    # with_payload
    for bad, match in (((0.0,) + PAYLOAD[1:], "positive"), ((np.nan,) + PAYLOAD[1:], "finite"),
                       ((1.0, (0.0, 0.0), PAYLOAD[2]), "shapes"), ((1.0, PAYLOAD[1], (1, 0, 0, -1, 0, 1)), "semi-definite"),
                       ((1.0, (0.0, np.inf, 0.0), PAYLOAD[2]), "finite")):
        with pytest.raises(ValueError, match=match):
            m.with_payload("flange", *bad)
    with pytest.raises(ValueError, match="no frame"):
        m.with_payload("tool0", *PAYLOAD)
    with pytest.raises(ValueError, match="base"):
        m.with_payload("base_link", *PAYLOAD)
    with pytest.raises(ValueError, match="another model"):
        model_of("arm6.urdf").with_payload(f, *PAYLOAD)


def test_dyn_header_prototypes_of_energy_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_frame_inverse_inertia"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr"]
    assert declared["tbd_collision_energy_terms"] == ["ptr", "int", "ptr", "double", "int", "ptr", "ptr", "ptr", "ptr"]
    for name in ("tbd_frame_inverse_inertia", "tbd_collision_energy_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_energy_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good_frame = m.frame("flange", **OFFSET).packed

    def rc(model=m.packed, frame=good_frame, nv=6, M=4, mh=HUMAN_MASS, null=None, which="both"):
        host = [np.array(x, dtype=np.float64) for x in (model, frame)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        li = [ptr[0], nv, ptr[1], M, d, d]
        ct = [ptr[0], nv, ptr[1], mh, M, d, d, d]
        if null is not None:
            (li if which == "inertia" else ct)[null] = None
        out = []
        if which in ("both", "inertia"):
            out.append(lib.tbd_frame_inverse_inertia(*li, None))
        if which in ("both", "terms"):
            out.append(lib.tbd_collision_energy_terms(*ct, None))
        assert len(set(out)) == 1, out
        assert out[0] == 0 or _lib.load().tb_last_error()
        return out[0]

    for k in (0, 2, 4, 5):
        assert rc(null=k, which="inertia") == TB_ERR_ARG
    for k in (0, 2, 5, 6, 7):
        assert rc(null=k, which="terms") == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model) == TB_ERR_ARG
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 1 + 17] = -1.0                           # negative mass
    assert rc(bad_model) == TB_ERR_ARG
    for j, value in ((0, 6.0), (0, -2.0), (0, 0.5), (5, np.nan), (11, np.inf)):   # bad frames
        f = good_frame.copy()
        f[j] = value
        assert rc(frame=f) == TB_ERR_ARG
    for mh in (0.0, -1.0, np.nan, -np.inf):
        assert rc(mh=mh, which="terms") == TB_ERR_ARG
    assert b"human_mass" in _lib.load().tb_last_error()
    assert rc(mh=np.inf, which="terms") not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)   # inf passes validation
    f = good_frame.copy()
    f[13] = 0.0                                                 # "world"
    assert rc(frame=f, which="inertia") == TB_ERR_UNSUPPORTED
    f[13] = 7.0
    assert rc(frame=f, which="inertia") == TB_ERR_ARG
    for ref in (0.0, 1.0, 2.0, 7.0):                             # the terms entry ignores the reference-frame field:
        f = good_frame.copy()                                    # validation passes, the launch fails (no device here)
        f[13] = ref
        assert rc(frame=f, which="terms") not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
        assert b"launch failed" in _lib.load().tb_last_error()
    for ref in (1.0, 2.0):
        f = good_frame.copy()
        f[13] = ref
        assert rc(frame=f, which="inertia") not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


@pytest.mark.gpu
def test_gpu_random_trees_vs_mp(ta):
    from toppra_b200.dynamics import rpy_matrix
    worst_cond, worst_ratio = 0.0, 0.0
    for nv in (1, 2, 3, 5, 8, 12, 16):
        rng = np.random.RandomState(1100 + nv)
        m = _model_from_packed(ta, rr.random_tree(rng, nv))
        mp = rr.MpRobot.from_packed(m.packed)
        P = 2 if nv <= 8 else 1
        q, qs = rng.uniform(-2, 2, (P, nv)), rng.uniform(-1.5, 1.5, (P, nv))
        for k in sorted({nv - 1, int(rng.randint(nv))}):
            off = dict(xyz=tuple(rng.randn(3) * 0.2), rpy=tuple(rng.uniform(-3, 3, 3)))
            spec = {0: ("b%d" % k,) + _spec(off)}
            for ref_frame in ("local_world_aligned", "local"):
                f = m.frame("body%d" % k, reference_frame=ref_frame, **off)
                L = f.inverse_inertia(_dev(q)).cpu().numpy()
                b = f.collision_energy_terms(_dev(q), _dev(qs), HUMAN_MASS).cpu().numpy()
                for i in range(P):
                    ref = er.mp_inverse_inertia(mp, q[i], spec)
                    Wm, Rm = _mpf(ref[0][0]), _mpf(ref[0][1])
                    want = Wm if ref_frame == "local_world_aligned" else Rm.T @ Wm @ Rm
                    bm = float(er.mp_energy_b(ref[(0, "J")], ref[0][0], qs[i], HUMAN_MASS))
                    cond = np.linalg.cond(_mpf(mp.mass_matrix([float(x) for x in q[i]])))
                    err = max(rel_err(L[i], want), abs(b[i] - bm) / bm)
                    worst_cond = max(worst_cond, cond)
                    worst_ratio = max(worst_ratio, err / cond)
                    assert err <= 1e-14 * cond, (nv, k, err, cond)
            # the kernel against the numpy double on many points
            Q, QS = rng.uniform(-3, 3, (512, nv)), rng.uniform(-2, 2, (512, nv))
            got = f.inverse_inertia(_dev(Q)).cpu().numpy()
            want = er.inverse_inertia_packed(m.packed, f.packed, Q)
            assert np.max(np.abs(got - want)) <= 1e-11 * np.max(np.abs(want))
            assert np.array_equal(f.inverse_inertia(Q[3]), got[3])           # numpy (nv,): a device round trip
    print("random trees: worst cond(M) %.3g, worst error / cond(M) %.3g" % (worst_cond, worst_ratio))


@pytest.mark.gpu
def test_gpu_hand_cases(ta):
    _hand_cases(ta, lambda f, q: f.inverse_inertia(_dev(q)).cpu().numpy(),
                lambda f, q, qs, mh: f.collision_energy_terms(_dev(q), _dev(qs), mh).cpu().numpy())


@pytest.mark.gpu
def test_gpu_energy_below_kinetic_energy_with_equality(ta):
    """m_H = inf: b <= 1/2 q'.(M q') (M q' the a term of tbd_torque_terms), with equality where q' = M^-1 J_v^T e for
    an eigenvector e of Lambda_v^-1 (Cauchy-Schwarz in the M^-1 metric)."""
    import torch
    n_eq = 0
    for seed, nv in ((1, 3), (2, 6), (3, 9), (4, 14)):
        rng = np.random.RandomState(1200 + seed)
        m = _model_from_packed(ta, rr.random_tree(rng, nv))
        f = m.frame("body%d" % (nv - 1), xyz=tuple(rng.randn(3) * 0.2))
        P = 400
        q, qs = _dev(rng.uniform(-2, 2, (P, nv))), _dev(rng.uniform(-2, 2, (P, nv)))
        zero = torch.zeros_like(q)
        b = f.collision_energy_terms(q, qs, np.inf)
        a = m.torque_terms(q, qs, zero)[0]                        # a = ID(q, 0, q') - ID(q, 0, 0) = M q'
        ke = 0.5 * (qs * a).sum(dim=1)
        assert (b <= ke * (1 + 1e-12)).all()
        assert (b < ke * (1 - 1e-6)).any()
        # the equality case on 20 points
        L = f.inverse_inertia(q[:20]).cpu().numpy()
        Mq = np.stack([m.torque_terms(q[:20], _dev(np.tile(np.eye(nv)[k], (20, 1))), zero[:20])[0].cpu().numpy()
                       for k in range(nv)], axis=2)              # M[:, :, k] = M e_k
        J = np.stack([f(q[:20], _dev(np.tile(np.eye(nv)[k], (20, 1))))[:, :3].cpu().numpy() for k in range(nv)], axis=2)
        qs_eq = []
        for i in range(20):
            lam, vec = np.linalg.eigh(L[i])
            nz = np.flatnonzero(lam > 1e-8 * lam[-1])                 # rank(Lambda_v^-1) <= nv: skip its null space
            e = vec[:, nz[int(rng.randint(len(nz)))]]
            qs_eq.append(np.linalg.solve(Mq[i], J[i].T @ e))
        qs_eq = _dev(np.array(qs_eq))
        b = f.collision_energy_terms(q[:20], qs_eq, np.inf).cpu().numpy()
        ke = (0.5 * (qs_eq * m.torque_terms(q[:20], qs_eq, zero[:20])[0]).sum(dim=1)).cpu().numpy()
        np.testing.assert_allclose(b, ke, rtol=1e-12)
        n_eq += 20
    assert n_eq == 80


@pytest.mark.gpu
def test_gpu_invariances(ta):
    m = model_of("arm7_gripper.urdf")                            # fingers unlocked: prismatic bodies on the chain
    rng = np.random.RandomState(13)
    M = 2000
    q, qs = _dev(rng.uniform(-2, 2, (M, m.nv))), _dev(rng.uniform(-2, 2, (M, m.nv)))
    for link in ("finger_left", "camera", "hand", "link3"):
        bs = [m.frame(link, reference_frame=r, **OFFSET).collision_energy_terms(q, qs, HUMAN_MASS)
              for r in ("world", "local", "local_world_aligned")]
        assert _eq(bs[0].cpu().numpy(), bs[1].cpu().numpy()) and _eq(bs[0].cpu().numpy(), bs[2].cpu().numpy())
        fw = m.frame(link, **OFFSET)
        Lw = fw.inverse_inertia(q).cpu().numpy()
        Ll = m.frame(link, reference_frame="local", **OFFSET).inverse_inertia(q).cpu().numpy()
        Rf = kr.frame_packed(m.packed, fw.packed, q.cpu().numpy(), qs.cpu().numpy())[0]
        want = np.einsum("mji,mjk,mkl->mil", Rf, Lw, Rf)
        assert np.max(np.abs(Ll - want)) <= 1e-14 * np.max(np.abs(Lw))
        assert np.array_equal(Lw, np.transpose(Lw, (0, 2, 1)))                  # symmetric by construction
        assert np.linalg.eigvalsh(Lw).min() >= -1e-14 * np.abs(Lw).max()
        prev = None
        for mh in (0.1, 0.6, 4.0, 75.0, np.inf):
            b = fw.collision_energy_terms(q, qs, mh).cpu().numpy()
            if prev is not None:
                assert (b > prev).all()
            prev = b


@pytest.mark.gpu
def test_gpu_terms_bit_equal_inverse_inertia_and_velocity(ta):
    import torch
    m = model_of("arm7_gripper.urdf")
    rng = np.random.RandomState(11)
    M = 3000
    q, qs = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(2))
    qs[:7] = 0.0                                                 # q' = 0: b = +0
    for link, ref in (("finger_left", "local"), ("camera", "world"), ("hand", "local_world_aligned")):
        for mh in (HUMAN_MASS, np.inf):
            f = m.frame(link, reference_frame=ref, **OFFSET)
            fl = m.frame(link, reference_frame="local_world_aligned", **OFFSET)
            W = fl.inverse_inertia(q)
            v = fl(q, qs)[:, :3]
            vv = v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2]
            Wv = [W[:, i, 0] * v[:, 0] + W[:, i, 1] * v[:, 1] + W[:, i, 2] * v[:, 2] for i in range(3)]
            w = v[:, 0] * Wv[0] + v[:, 1] * Wv[1] + v[:, 2] * Wv[2]
            want = torch.where((vv == 0) & ~torch.isnan(w), torch.zeros_like(vv), 0.5 * vv * vv / (vv / mh + w))
            got = f.collision_energy_terms(q, qs, mh)
            assert torch.equal(got, want), link
            assert (got[:7] == 0).all() and not torch.signbit(got[:7]).any()
            cons = ta.constraint.CollisionEnergyConstraint(f, 1.0, mh)
            assert torch.equal(cons.energy(q, qs), got)
            assert cons.energy(q[5].cpu().numpy(), qs[5].cpu().numpy()) == float(got[5].cpu())
    # NaN in one point leaves every other point as it was
    f = model_of("arm6.urdf").frame("flange", **OFFSET)
    q, qs = rng.uniform(-2, 2, (2, 64, 6))
    qn, qsn = q.copy(), qs.copy()
    qn[5, 2] = np.nan
    qsn[9, 0] = np.nan
    ref = f.collision_energy_terms(_dev(q), _dev(qs), HUMAN_MASS).cpu().numpy()
    got = f.collision_energy_terms(_dev(qn), _dev(qsn), HUMAN_MASS).cpu().numpy()
    L = f.inverse_inertia(_dev(qn)).cpu().numpy()
    assert np.isnan(got[[5, 9]]).all() and np.isnan(L[5]).all() and not np.isnan(np.delete(L, 5, axis=0)).any()
    keep = np.ones(64, bool)
    keep[[5, 9]] = False
    assert np.array_equal(got[keep], ref[keep])


@pytest.mark.gpu
def test_gpu_singular_mass_matrix_gives_nan_only_there(ta):
    """A massless revolute body about z carrying a point mass on a prismatic joint along its x axis: M = diag(m q1^2, m),
    singular exactly where q1 = 0.  Built from arrays, so no Python check stands in the way."""
    mass = 2.5
    m = ta.RigidBodyModel([-1, 0], ["revolute", "prismatic"], [[0, 0, 1.0], [1.0, 0, 0]], [np.eye(3)] * 2,
                          [[0, 0, 0.0]] * 2, [0.0, mass], [[0, 0, 0.0]] * 2, [[0.0] * 6] * 2)
    rng = np.random.RandomState(17)
    q = rng.uniform(-1, 1, (50, 2))
    q[[3, 20, 41], 1] = 0.0
    qs = rng.uniform(-1, 1, (50, 2))
    f = m.frame("body1")
    L = f.inverse_inertia(_dev(q)).cpu().numpy()
    b = f.collision_energy_terms(_dev(q), _dev(qs), HUMAN_MASS).cpu().numpy()
    sing = np.zeros(50, bool)
    sing[[3, 20, 41]] = True
    assert np.isnan(L[sing]).all() and np.isnan(b[sing]).all()
    assert np.isfinite(L[~sing]).all() and np.isfinite(b[~sing]).all()
    np.testing.assert_allclose(L[~sing], np.broadcast_to(np.diag([1 / mass, 1 / mass, 0.0]), L[~sing].shape),
                               rtol=0, atol=1e-14)
    zero = np.zeros_like(qs)                                     # NaN beats the q' = 0 rule
    assert np.isnan(f.collision_energy_terms(_dev(q), _dev(zero), HUMAN_MASS).cpu().numpy()[sing]).all()


def _b_dev(f, mh, path, grid):
    d = _dev(grid)
    b = f.collision_energy_terms(*(path.eval_device(d, o).reshape(-1, f.nv) for o in (0, 1)), mh)
    return b.reshape(path.B, len(grid)).cpu().numpy()


def _golden_frame(g, robot, m):
    return m.frame(str(g[robot + "/link"]), xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"])


def _cons(ta, f, vlim, alim, limit, mh, scheme=0, joint_scheme=None):
    joint_scheme = scheme if joint_scheme is None else joint_scheme
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=joint_scheme),
            ta.constraint.CollisionEnergyConstraint(f, limit, mh, discretization_scheme=scheme)]


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("collision_energy")
    m = model_of(name, locked)
    f = _golden_frame(g, robot, m)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim, limit, mh = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "limit", "human_mass"))
    mh = float(mh)
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    b = _b_dev(f, mh, path, grid)
    for i in range(B):                                            # against the 50-digit b
        assert rel_err(b[i], g[robot + "/b"][i]) <= 1e-12
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (robot, scheme, x)][i]  # noqa: E731
        for i in range(B):
            one = ta.algorithm.TOPPRA(_cons(ta, f, vlim[i], alim[i], float(limit[i]), mh, scheme),
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, mh, scheme), path, grid).compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


def _active_limits(ta, f, mh, path, grid, vlim, alim, share=0.3):
    """Per path: `share` of the largest b sd^2 of the solution without the energy limit (so that it is active)."""
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                       path, grid).compute_parameterization(0, 0).to_host()
    b = _b_dev(f, mh, path, grid)
    return share * np.max(b * np.nan_to_num(h["sd"]) ** 2, axis=1)


def _energy_rows(b, limit, grid, interp):
    """(G, 3, R) rows a = 0, b, 0 - limit of the constraint for the oracle."""
    from toppra_b200.constraint.linear_constraint import canlinear_colloc_to_interpolate
    G = len(grid)
    a, c = np.zeros((G, 1)), np.zeros((G, 1))
    F, g = np.ones((1, 1)), np.full(1, limit)
    bb = b.reshape(G, 1)
    if interp:
        a, bb, c, F, g = canlinear_colloc_to_interpolate(a, bb, c, F, g, None, None, grid, identical=True)[:5]
    return np.stack((a.dot(F.T), bb.dot(F.T), c.dot(F.T) - g), axis=1)


@pytest.mark.gpu
def test_gpu_256_paths_per_path_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _problems(B, nv, 31, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    limit = _active_limits(ta, f, HUMAN_MASS, path, grid, vlim, alim)
    # the oracle's joint-acceleration rows (solve_velacc(..., True, ...)) are those of the Interpolation scheme
    h = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, HUMAN_MASS, 0, 1), path, grid).compute_parameterization(0, 0)
    h = h.to_host()
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1))
        b = er.energy_terms_packed(m.packed, f.packed, q, qs, HUMAN_MASS)
        rows = np.concatenate((lin["rows"], _energy_rows(b, limit[i], grid, False)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            E = b * h["sd"][i] ** 2
            assert (E <= limit[i] * (1 + 1e-9)).all(), (i, E.max() / limit[i])
            n_active += bool((E >= limit[i] * (1 - 1e-6)).any())
    print("energy limit active on %d of %d solved paths" % (n_active, n_ok))
    assert n_ok > 0.9 * B and n_active > 0.8 * n_ok, (n_ok, n_active)


@pytest.mark.gpu
def test_gpu_ragged_chunked_single_path_and_host_route_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    f = m.frame("hand", reference_frame="local", **OFFSET)
    B, nv, mh = 12, m.nv, 40.0
    ss, way, vlim, alim = _problems(B, nv, 37, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    limit = _active_limits(ta, f, mh, path, np.linspace(0, 1, 100), vlim, alim)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, mh), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, f, vlim[i:i + 1], alim[i:i + 1], limit[i:i + 1], mh),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, mh, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, mh, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the host route (compute_constraint_params through a user
    # LinearConstraint) equals the device route
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
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cons(ta, f, vlim[i], alim[i], float(limit[i]), mh, scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            run_dev = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cons(ta, f, vlim[i:i + 1], alim[i:i + 1], limit[i:i + 1], mh, scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0).to_host()
            assert _eq(run_dev[3], hb["K"][0]) and _eq(run_dev[1], hb["sd"][0]) and _eq(run_dev[0], hb["sdd"][0])
            cons = _cons(ta, f, vlim[i], alim[i], float(limit[i]), mh, scheme)
            cons[2] = HostRoute(cons[2])
            host = ta.algorithm.TOPPRA(cons, sp, gridpoints=grid, solver_wrapper="seidel")
            run_host = host.compute_parameterization(0, 0, return_data=True)
            for x, y in zip(run_dev, run_host):
                assert _eq(x, y)
            assert run_dev[1] is not None


@pytest.mark.gpu
def test_gpu_toppra_sd_and_quintic_piecewise_poly_path_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(41)
    coeffs = rng.uniform(-0.4, 0.4, (B, k, nseg, nv))
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    limit = _active_limits(ta, f, HUMAN_MASS, path, grid, vlim, alim)
    h = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, limit, HUMAN_MASS), path, grid).compute_parameterization(0, 0).to_host()
    b = _b_dev(f, HUMAN_MASS, path, grid)
    assert (h["status"] == 0).sum() >= B // 2
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    for i in range(B):
        ga = np.concatenate((alim[i][:, 1], -alim[i][:, 0]))
        joint = np.stack((qs[1][i].dot(Fj.T), qs[2][i].dot(Fj.T), np.zeros((len(grid), nv)).dot(Fj.T) - ga), axis=1)
        o = orc.solve_rows(np.concatenate((joint, _energy_rows(b[i], limit[i], grid, False)), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
    # BatchTOPPRAsd, whole and in record chunks: half again the time-optimal duration (or the slowest profile); the
    # energy stays within the limit on the blended profiles
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        inst = ta.BatchTOPPRAsd(_cons(ta, f, vlim, alim, limit, HUMAN_MASS), path, grid)
        if chunk:
            inst = ta.BatchTOPPRAsd(_cons(ta, f, vlim, alim, limit, HUMAN_MASS), path, grid,
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
        assert (b[i] * sd[i] ** 2 <= limit[i] * (1 + 1e-9)).all()
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        want = min(1.5 * dur[i], slow[i])
        assert abs(got - want) <= 1e-4 * max(1.0, want), (got, want)


@pytest.mark.gpu
def test_gpu_with_torque_and_velocity_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 32, 150, 6
    ss, way, vlim, alim = _problems(B, nv, 43, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    limit = _active_limits(ta, f, HUMAN_MASS, path, grid, vlim, alim, share=0.5)
    d = _dev(grid)
    bv = f.velocity_norm_terms(*(path.eval_device(d, o).reshape(-1, nv) for o in (0, 1)), S).reshape(B, G)
    speed = 0.5 * bv.max(dim=1).values.cpu().numpy()
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    cons = _cons(ta, f, vlim, alim, limit, HUMAN_MASS, 1) + [ta.constraint.JointTorqueConstraint(m, taulim, fric),
                                                             ta.constraint.CartesianVelocityNorm(f, S, speed)]
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        b = er.energy_terms_packed(m.packed, f.packed, q, qs, HUMAN_MASS)
        av, btv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        torque = np.stack((av.dot(Fj.T), btv.dot(Fj.T), cv.dot(Fj.T) - gt), axis=1)
        vq = kr.quad_form(S, kr.frame_velocity_packed(m.packed, f.packed, q, qs))
        cart_v = np.stack((np.zeros(G), vq, np.full(G, 0.0 - speed[i])), axis=1)[:, :, None]
        rows = np.concatenate((lin["rows"], _energy_rows(b, limit[i], grid, True), torque, cart_v), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok > 0.8 * B


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch):
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    B = 10
    ss, way, vlim, alim = _problems(B, 6, 47, m.velocity_limit)
    limit = np.full(B, 2.0)
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, f, vlim, alim, limit, HUMAN_MASS),
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_collision_energy_terms")
