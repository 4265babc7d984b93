"""The wrench the support exerts on a whole robot, and its stability on a footprint (RigidBodyFrame.support_wrench /
support_wrench_terms, SupportStabilityConstraint, support_polygon_rows, RigidBodyModel.base_mass / base_com;
libtoppra_b200_dyn.so: tbd_support_wrench, tbd_support_wrench_terms).

CPU:
  * the float64 numpy double of tests/support_ref.py equals the 50-digit wrench of the RAW URDF tree to 1e-13 of the
    scale: mobile_arm.urdf with its wheels locked and unlocked, arm6.urdf, support frames with offsets and rotations,
    random points;
  * the static case: f = -M_total g in support axes, and the zero-moment point is the projection of the total centre of
    mass, computed in closed form from the link masses;
  * support_polygon_rows against a point-in-convex-polygon definition of the centre of pressure on thousands of random
    wrenches; the rectangle's rows equal the tipping rows of contact_wrench_cone; sum_i |e_i| row_i = -2 Area e_fz;
  * from_urdf's base_mass / base_com, array-built models and with_payload;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library.
GPU:
  * tbd_support_wrench on random trees (1 to 16 bodies, several root children, prismatic joints) against the 50-digit
    reference and the numpy double within 1e-12; s_j . (n_b - r_j x f_b) of a tree with one root child equals tbd_rnea's
    tau_j;
  * tbd_support_wrench_terms equals three tbd_support_wrench launches and the two subtractions, bit for bit; NaN in one
    point touches no other;
  * the reference golden (tests/golden/support_stability.npz, make_golden_support.py): TOPPRA and BatchTOPPRA within
    |dK| <= 1e-9 + 1e-8 |K| (the cfg-3 tolerance), equal statuses, both footprint forms and schemes; 256 paths against
    the oracle fed with rows from the numpy double, same tolerance; the zero-moment points of the solved profiles are
    inside the polygon, and the support rows are active;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, the reference-style
    SecondOrderConstraint with cons.wrench as a numpy callback vs SupportStabilityConstraint: bit-equal;
    BatchTOPPRAsd, a quintic BatchPiecewisePolyPath, and the constraint next to JointTorqueConstraint and
    CartesianVelocityNorm against the oracle; one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import rnea_ref as rr
import support_ref as sref
from test_cartesian_velocity import (DYN_LIB, ROOT, TB_ERR_ARG, TB_ERR_UNSUPPORTED, _assert_solution, _dev, _eq,
                                     _gpu_present, _model_from_packed, close, model_of, urdf)
from test_contact_stability import _CountingLib, _oracle_joint_rows, _oracle_rows

WHEELS = {"wheel_fl_joint": 0.3, "wheel_fr_joint": -1.2, "wheel_rl_joint": 2.0, "wheel_rr_joint": 0.0}
CASES = [("mobile_arm.urdf", WHEELS), ("mobile_arm.urdf", None), ("arm6.urdf", None)]
ROOT_LINK = {"mobile_arm.urdf": "base_footprint", "arm6.urdf": "base_link"}
OFFSETS = [dict(), dict(xyz=(0.03, -0.02, 0.0), rpy=(0.0, 0.0, 0.7)), dict(xyz=(-0.1, 0.05, 0.2), rpy=(0.3, -0.2, 0.5))]
G0 = 9.81


class FakePath(object):
    def __init__(self, B, dof):
        self.B, self.dof, self.device = B, dof, "cpu"


def _support(m, name, off=None, ref="local_world_aligned"):
    return m.frame(ROOT_LINK[name], reference_frame=ref, **(off or {}))


# ==== CPU: numpy double vs the 50-digit reference, statics, polygon rows, base inertia, errors, C-ABI ================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 171)
    for _ in range(2):
        q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
        for k, off in enumerate(OFFSETS):
            # the reference frame of a RigidBodyFrame is ignored: the wrench is in the support's own axes
            f = _support(m, name, off, ("local", "world", "local_world_aligned")[k])
            want = [float(x) for x in sref.mp_support_wrench(mp, q, qd, qdd, f.R, f.p)]
            got = sref.support_wrench_packed(m.packed, f.packed, m.packed_base(), q, qd, qdd)[0]
            close(got, want, 1e-13)
        a, b, c = sref.support_terms_packed(m.packed, f.packed, m.packed_base(), q, qd, qdd)
        w0 = sref.support_wrench_packed(m.packed, f.packed, m.packed_base(), q, 0 * q, 0 * q)
        assert np.array_equal(c, w0)
        assert np.array_equal(b, sref.support_wrench_packed(m.packed, f.packed, m.packed_base(), q, qd, qdd) - w0)


@pytest.mark.parametrize("name,locked", CASES)
def test_static_wrench_is_the_weight_and_zmp_the_com(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 5)
    z = np.zeros(m.nv)
    for off in OFFSETS[:2]:                   # support normals along gravity: turned about z only
        f = _support(m, name, off)
        for _ in range(3):
            q = rng.uniform(-2, 2, m.nv)
            w = sref.support_wrench_packed(m.packed, f.packed, m.packed_base(), q, z, z)[0]
            mass, com = sref.mp_total_com(mp, q)
            close(w[:3], f.R.T @ np.array([0.0, 0.0, mass * G0]), 1e-13)
            close(sref.zmp(w), (f.R.T @ (com - f.p))[:2], 1e-13)
            close(w[5], 0.0, 1e-13)


def _inside_polygon(P, p):
    """p (n, 2) inside the convex counter-clockwise polygon P (boundary included): on the left of every edge."""
    E = np.roll(P, -1, axis=0) - P
    side = E[None, :, 0] * (p[:, None, 1] - P[None, :, 1]) - E[None, :, 1] * (p[:, None, 0] - P[None, :, 0])
    return (side >= 0).all(axis=1), np.abs(side).min(axis=1)


POLYGONS = [np.array([[-0.04, -0.045], [0.045, -0.04], [0.055, 0.01], [0.02, 0.045], [-0.045, 0.035]]),
            np.array([[0.1, 0.1], [0.3, 0.12], [0.2, 0.4]]),                   # the origin outside
            np.array([[np.cos(t), np.sin(t)] for t in np.linspace(0, 2 * np.pi, 9)[:-1]]) * 0.2]


def test_polygon_rows_match_the_centre_of_pressure_definition():
    from toppra_b200.constraint import contact_wrench_cone, support_polygon_rows
    rng = np.random.RandomState(3)
    n = inside = 0
    for P in POLYGONS:
        F = support_polygon_rows(P)
        assert F.shape == (len(P), 6)
        lo, hi = P.min(axis=0), P.max(axis=0)
        span = hi - lo
        count = 0
        while count < 1000:
            fz = rng.uniform(0.1, 100.0)
            cop = rng.uniform(lo - 0.3 * span, hi + 0.3 * span)
            w = np.r_[rng.randn(2) * fz, fz, cop[1] * fz, -cop[0] * fz, rng.randn() * fz]
            ins, dist = _inside_polygon(P, cop[None])
            if dist[0] < 1e-9 * span.max() ** 2:
                continue
            v = F @ w
            assert bool((v <= 0).all()) == bool(ins[0]), (P, cop, v)
            # the centre of pressure of the rows' own convention
            close(sref.zmp(w), cop, 1e-14)
            inside += bool(ins[0])
            count += 1
        n += count
        # a wrench that pulls the robot off its support violates a row: sum_i |e_i| row_i = -2 Area e_fz
        E = np.roll(P, -1, axis=0) - P
        area = 0.5 * np.sum(P[:, 0] * np.roll(P[:, 1], -1) - np.roll(P[:, 0], -1) * P[:, 1])
        s = np.hypot(E[:, 0], E[:, 1]) @ F
        close(s, [0.0, 0.0, -2 * area, 0.0, 0.0, 0.0], 1e-15)
        for _ in range(50):
            w = rng.randn(6)
            w[2] = -abs(w[2])
            assert (F @ w > 0).any()
    assert n >= 3000 and 0.2 * n < inside < 0.8 * n, (n, inside)
    # with friction: the four sliding rows of the cone follow
    Fm = support_polygon_rows(POLYGONS[0], 0.4)
    assert Fm.shape == (9, 6) and np.array_equal(Fm[5:], contact_wrench_cone((0.1, 0.1), 0.4)[:4])
    # the rectangle's rows are the cone's tipping rows
    for X, Y in ((0.05, 0.04), (0.3, 0.01)):
        R = support_polygon_rows([[-X, -Y], [X, -Y], [X, Y], [-X, Y]])
        tip = contact_wrench_cone((X, Y), 0.5)[4:8]
        for row in tip:
            assert np.min(np.abs(R - row).max(axis=1)) <= 1e-15, (row, R)


def _raw_base(name, locked):
    """Mass and centre of mass of the root link and the links fixed or locked to it, from the raw URDF tree at q = 0."""
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    fr = mp._kinematics([0] * mp.nv)[0]
    on_base = {mp.root}
    for j in mp.joints:
        if j["parent"] in on_base and j["dof"] is None:
            on_base.add(j["child"])
    mass, mc = 0.0, np.zeros(3)
    for link in on_base:
        if mp.links[link] is None:
            continue
        m, c = float(mp.links[link][0]), np.array([float(x) for x in mp.links[link][1]])
        R, p = (np.array([[float(R[i, j]) for j in range(3)] for i in range(3)]) if k == 0 else
                np.array([float(x) for x in R]) for k, R in enumerate(fr[link]))
        mass += m
        mc += m * (p + R @ c)
    return mass, mc / mass, len(on_base)


def test_base_mass_and_com():
    import toppra_b200 as ta
    for name, locked, n_links in (("mobile_arm.urdf", WHEELS, 6), ("mobile_arm.urdf", None, 2), ("arm6.urdf", None, 1)):
        m = model_of(name, locked)
        mass, com, n = _raw_base(name, locked)
        assert n == n_links
        assert abs(m.base_mass - mass) <= 1e-12 * mass
        close(m.base_com, com, 1e-14)
        assert np.array_equal(m.packed_base(), np.r_[m.base_mass, m.base_com])
        loaded = m.with_payload(m.frame("flange"), 1.5, (0.0, 0.0, 0.05), (0.001, 0, 0, 0.001, 0, 0.001))
        assert loaded.base_mass == m.base_mass and np.array_equal(loaded.base_com, m.base_com)
    assert model_of("mobile_arm.urdf", WHEELS).base_mass == 31.0 and model_of("arm6.urdf").base_mass == 4.0
    arr = _model_from_packed(ta, rr.random_tree(np.random.RandomState(1), 4))
    assert arr.base_mass == 0.0 and np.array_equal(arr.base_com, np.zeros(3))
    b = arr.packed[3:].reshape(4, 27)
    given = ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                              base_mass=2.5, base_com=(0.1, 0.0, 0.3))
    assert given.base_mass == 2.5 and np.array_equal(given.base_com, [0.1, 0.0, 0.3])
    assert np.array_equal(given.packed[3:], arr.packed[3:])
    with pytest.raises(ValueError, match="on the base"):                 # unchanged: no payload on a base frame
        model_of("arm6.urdf").with_payload("base_link", 1.0, (0, 0, 0), (0, 0, 0, 0, 0, 0))


def test_value_errors():
    import toppra_b200 as ta
    from toppra_b200.constraint import SupportStabilityConstraint, support_polygon_rows
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("mobile_arm.urdf", WHEELS)
    s = m.frame("base_footprint")
    P = POLYGONS[0]
    with pytest.raises(ValueError, match="RigidBodyFrame"):
        SupportStabilityConstraint(lambda q, qd, qdd: np.zeros(6), half_lengths=(0.1, 0.1))
    with pytest.raises(ValueError, match="on the base"):
        SupportStabilityConstraint(m.frame("torso"), half_lengths=(0.1, 0.1))
    with pytest.raises(ValueError, match="on the base"):
        m.frame("flange").support_wrench(None, np.zeros(m.nv), np.zeros(m.nv), np.zeros(m.nv))
    for kw in (dict(), dict(half_lengths=(0.1, 0.1), polygon=P)):
        with pytest.raises(ValueError, match="exactly one"):
            SupportStabilityConstraint(s, **kw)
    bad_polygons = {"not convex": [[0, 0], [1, 0], [0.2, 0.2], [0, 1]],
                    "clockwise": P[::-1],
                    "degenerate": [[0, 0], [1, 0], [1, 0], [0, 1]],
                    "collinear": [[0, 0], [0.5, 0], [1, 0], [0, 1]]}
    for what, poly in bad_polygons.items():
        with pytest.raises(ValueError, match="degenerate" if what == "collinear" else what):
            SupportStabilityConstraint(s, polygon=poly)
        with pytest.raises(ValueError):
            support_polygon_rows(poly)
    star = np.array([[np.cos(t), np.sin(t)] for t in np.linspace(0, 4 * np.pi, 6)[:-1]])   # a pentagram: twice round
    with pytest.raises(ValueError, match="not convex"):
        SupportStabilityConstraint(s, polygon=star)
    for poly in ([[0, 0], [1, 0]], np.zeros((4, 3)), [[0, 0], [1, np.nan], [0, 1]]):
        with pytest.raises(ValueError, match="expected|finite"):
            SupportStabilityConstraint(s, polygon=poly)
    for hl in ((0.0, 0.1), (0.1, -0.1)):
        with pytest.raises(ValueError, match="positive"):
            SupportStabilityConstraint(s, half_lengths=hl)
    with pytest.raises(ValueError, match="finite"):
        SupportStabilityConstraint(s, half_lengths=(np.inf, 0.1))
    with pytest.raises(ValueError, match="half_lengths"):
        SupportStabilityConstraint(s, half_lengths=(0.1, 0.1, 0.1))
    for mu in (0.0, -0.3):
        for kw in (dict(half_lengths=(0.1, 0.1)), dict(polygon=P)):
            with pytest.raises(ValueError, match="positive"):
                SupportStabilityConstraint(s, friction=mu, **kw)
    with pytest.raises(ValueError, match="finite"):
        SupportStabilityConstraint(s, polygon=P, friction=np.nan)
    for kw, match in ((dict(base_mass=-1.0), "non-negative"), (dict(base_mass=np.nan), "finite"),
                      (dict(base_com=(0.0, np.inf, 0.0)), "finite"), (dict(base_com=(0.0, 0.0)), "shapes")):
        with pytest.raises(ValueError, match=match):
            SupportStabilityConstraint(s, half_lengths=(0.1, 0.1), **kw)
        with pytest.raises(ValueError, match=match):
            b = m.packed[3:].reshape(m.nv, 27)
            ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21],
                              b[:, 21:27], **kw)
    with pytest.raises(ValueError, match="4 doubles"):
        s.support_wrench(np.zeros(3), np.zeros(m.nv), np.zeros(m.nv), np.zeros(m.nv))
    grid = np.linspace(0, 1, 10)
    ctx = RecordContext(FakePath(3, m.nv), grid, grid)
    c = SupportStabilityConstraint(s, half_lengths=(0.1, 0.08), friction=0.5)
    assert c.dof == m.nv and c.F.shape == (16, 6) and c.num_rows(ctx) == 32
    assert np.array_equal(c.base, m.packed_base())
    c = SupportStabilityConstraint(s, half_lengths=(0.1, 0.08), discretization_scheme=0)
    assert c.F.shape == (4, 6) and c.num_rows(ctx) == 4
    c = SupportStabilityConstraint(s, polygon=P, friction=0.5, base_mass=40.0, base_com=(0.0, 0.0, 0.3))
    assert c.F.shape == (9, 6) and c.num_rows(ctx) == 18 and np.array_equal(c.base, [40.0, 0.0, 0.0, 0.3])
    with pytest.raises(ValueError, match="Wrong dimension"):                                   # a model with another nv
        c.num_rows(RecordContext(FakePath(3, 6), grid, grid))


def test_dyn_header_prototypes_of_support_entries():
    from test_rigid_body import _dyn_header
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_support_wrench"] == ["ptr", "int", "ptr", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_support_wrench_terms"] == ["ptr", "int", "ptr", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr",
                                                    "ptr", "ptr"]
    for name in ("tbd_support_wrench", "tbd_support_wrench_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    assert "#define TBD_BASE_DOUBLES 4" in text and "#define TBD_VERSION 100" in text


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_support_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good_frame = m.frame("base_link", xyz=(0.03, -0.02, 0.0), rpy=(0.0, 0.0, 0.5)).packed
    good_base = m.packed_base()

    def rc(model=m.packed, frame=good_frame, base=good_base, nv=6, M=4, null=None):
        host = [np.array(x, dtype=np.float64) for x in (model, frame, base)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        cw = [ptr[0], nv, ptr[1], ptr[2], M, d, d, d, d]
        ct = [ptr[0], nv, ptr[1], ptr[2], M, d, d, d, d, d, d]
        if null is not None:                   # index into cw; ct has two more outputs
            cw[null] = None
            ct[null] = None
        r1 = lib.tbd_support_wrench(*cw, None)
        r2 = lib.tbd_support_wrench_terms(*ct, None)
        assert r1 == r2, (r1, r2)
        assert r1 == 0 or _lib.load().tb_last_error()
        return r1

    for k in (0, 2, 3, 5, 6, 7, 8):
        assert rc(null=k) == TB_ERR_ARG
    for k in (9, 10):                          # the extra outputs of the terms entry
        host = [np.array(x, dtype=np.float64) for x in (m.packed, good_frame, good_base)]
        ct = [ctypes.c_void_p(h.ctypes.data) for h in host]
        args = [ct[0], 6, ct[1], ct[2], 4, d, d, d, d, d, d]
        args[k] = None
        assert lib.tbd_support_wrench_terms(*args, None) == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model) == TB_ERR_ARG
    for j, value in ((0, 6.0), (0, -2.0), (0, 0.5), (5, np.nan), (11, np.inf)):   # bad frames
        f = good_frame.copy()
        f[j] = value
        assert rc(frame=f) == TB_ERR_ARG
    for body in (0.0, 3.0, 5.0):                                 # a support that is not on the base
        f = good_frame.copy()
        f[0] = body
        assert rc(frame=f) == TB_ERR_ARG
        assert b"support must be on the base" in _lib.load().tb_last_error()
    for j, value in ((0, -1.0), (0, -1e-300), (0, np.nan), (0, np.inf), (1, np.inf), (3, -np.nan)):   # bad bases
        b = good_base.copy()
        b[j] = value
        assert rc(base=b) == TB_ERR_ARG
        assert b"base" in _lib.load().tb_last_error()
    for ok in ([0.0, 0.0, 0.0, 0.0], [0.0, 1.0, -2.0, 3.0], [50.0, 0.1, 0.0, 0.4]):   # a massless base is fine: the
        assert rc(base=ok) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)                 # call passes validation and
        assert b"launch failed" in _lib.load().tb_last_error()                        # fails only at the launch
    for ref in (0.0, 1.0, 2.0, 7.0):                             # the reference-frame field is ignored
        f = good_frame.copy()
        f[13] = ref
        assert rc(frame=f) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
        assert b"launch failed" in _lib.load().tb_last_error()


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _tree_with_root_children(rng, nv, n_roots):
    """rr.random_tree with the first min(n_roots, nv) bodies on the base and at least one prismatic joint for nv >= 3."""
    packed = rr.random_tree(rng, nv)
    b = packed[3:].reshape(nv, 27)
    b[:min(n_roots, nv), 0] = -1
    if nv >= 3:
        b[nv // 2, 1] = 1
    return packed


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_support_wrench_random_trees_vs_mp(ta, nv):
    from toppra_b200.dynamics import rpy_matrix
    rng = np.random.RandomState(1300 + nv)
    m = _model_from_packed(ta, _tree_with_root_children(rng, nv, 3))
    mp = rr.MpRobot.from_packed(m.packed)
    P = 2 if nv <= 8 else 1
    q, qd, qdd = (rng.uniform(-2, 2, (P, nv)) for _ in range(3))
    base = sref.base_packed(rng.uniform(0.0, 20.0), rng.randn(3) * 0.2)
    m.frames["floor"] = (-1, rpy_matrix(rng.uniform(-3, 3, 3)), rng.randn(3) * 0.3)
    for off in (dict(), dict(xyz=tuple(rng.randn(3) * 0.2), rpy=tuple(rng.uniform(-3, 3, 3)))):
        f = m.frame("floor", **off)
        w = f.support_wrench(base, _dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
        for i in range(P):
            want = sref.mp_support_wrench(mp, q[i], qd[i], qdd[i], f.R, f.p, base)
            close(w[i], [float(x) for x in want], 1e-12)
        Q, QD, QDD = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
        got = f.support_wrench(base, _dev(Q), _dev(QD), _dev(QDD)).cpu().numpy()
        want = sref.support_wrench_packed(m.packed, f.packed, base, Q, QD, QDD)
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
        assert np.array_equal(f.support_wrench(base, Q[3], QD[3], QDD[3]), got[3])   # numpy (nv,): a device round trip
        assert np.array_equal(f.support_wrench(base, Q[:5], QD[:5], QDD[:5]), got[:5])


@pytest.mark.gpu
def test_gpu_root_joint_torque_matches_rnea(ta):
    """With one root child (arm6: shoulder_pan), the moment of the moving tree's base wrench about the root joint's
    axis is that joint's torque: s_j . (n_b - r_j x f_b) = tau_j."""
    m = model_of("arm6.urdf")
    bd = m.body(0)
    assert bd[0] == -1 and bd[1] == 0 and all(m.body(k)[0] >= 0 for k in range(1, m.nv))
    s_j, r_j = bd[5:14].reshape(3, 3) @ bd[2:5], bd[14:17]
    rng = np.random.RandomState(21)
    q, qd, qdd = (_dev(rng.uniform(-3, 3, (2000, m.nv))) for _ in range(3))
    w = m.frame("base_link").support_wrench(np.zeros(4), q, qd, qdd).cpu().numpy()   # base origin, base axes, no weight
    got = (w[:, 3:] - np.cross(r_j, w[:, :3])) @ s_j
    tau = m(q, qd, qdd).cpu().numpy()[:, 0]
    assert np.max(np.abs(got - tau)) <= 1e-12 * max(1.0, np.max(np.abs(tau)))


@pytest.mark.gpu
def test_gpu_support_terms_bit_equal_three_launches(ta):
    import torch
    m = model_of("mobile_arm.urdf")                              # wheels unlocked: six root children, a prismatic lift
    rng = np.random.RandomState(11)
    M = 3000
    q, qs, qss = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(3))
    zero = torch.zeros_like(q)
    for off, ref, base in ((OFFSETS[1], "local", None), (OFFSETS[2], "world", [12.0, 0.1, -0.2, 0.5]),
                           (OFFSETS[0], "local_world_aligned", None)):
        f = _support(m, "mobile_arm.urdf", off, ref)
        c = f.support_wrench(base, q, zero, zero)
        a = f.support_wrench(base, q, zero, qs) - c
        b = f.support_wrench(base, q, qs, qss) - c
        got = f.support_wrench_terms(base, q, qs, qss)
        for x, y in zip(got, (a, b, c)):
            assert x.shape == (M, 6) and torch.equal(x, y), off
        # the reference frame is ignored
        same = _support(m, "mobile_arm.urdf", off, "local").support_wrench_terms(base, q, qs, qss)
        assert all(torch.equal(x, y) for x, y in zip(got, same))
    # NaN in one point leaves every other point as it was
    f = model_of("arm6.urdf").frame("base_link", **OFFSETS[1])
    q, qs, qss = rng.uniform(-2, 2, (3, 64, 6))
    qn, qsn, qssn = q.copy(), qs.copy(), qss.copy()
    qn[5, 2] = np.nan
    qsn[9, 0] = np.nan
    qssn[17, 4] = np.nan
    ref = [x.cpu().numpy() for x in f.support_wrench_terms(None, _dev(q), _dev(qs), _dev(qss))]
    got = [x.cpu().numpy() for x in f.support_wrench_terms(None, _dev(qn), _dev(qsn), _dev(qssn))]
    assert np.isnan(got[2][5]).any() and np.isnan(got[0][9]).any() and np.isnan(got[1][17]).any()
    keep = np.ones(64, bool)
    keep[[5, 9, 17]] = False
    for x, y in zip(got, ref):
        assert np.array_equal(x[keep], y[keep])


GOLDEN_ROBOTS = {"mobile": ("mobile_arm.urdf", WHEELS), "arm6": ("arm6.urdf", None)}


def _golden_setup(g, robot):
    name, locked = GOLDEN_ROBOTS[robot]
    m = model_of(name, locked)
    f = m.frame(str(g[robot + "/link"]), xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"])
    assert np.array_equal(g[robot + "/base"], m.packed_base())
    return m, f


def _cons_of(ta, f, g, robot, form, scheme=1):
    if form == "rect":
        return ta.constraint.SupportStabilityConstraint(f, half_lengths=g[robot + "/half_lengths"],
                                                        friction=float(g[robot + "/friction"]),
                                                        discretization_scheme=scheme)
    return ta.constraint.SupportStabilityConstraint(f, polygon=g[robot + "/polygon"], discretization_scheme=scheme)


def _terms(f, path, grid):
    """a, b, c (B, G, 6) of the support wrench on the device path at the grid."""
    d = _dev(grid)
    out = f.support_wrench_terms(None, *(path.eval_device(d, o).reshape(-1, f.nv) for o in (0, 1, 2)))
    return [x.reshape(path.B, len(grid), 6).cpu().numpy() for x in out]


@pytest.mark.gpu
@pytest.mark.parametrize("robot", ["mobile", "arm6"])
def test_gpu_reference_golden(ta, golden, robot):
    g = golden("support_stability")
    m, f = _golden_setup(g, robot)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim = (g[robot + "/" + k] for k in ("way", "vlim", "alim"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    terms = _terms(f, path, grid)
    for i in range(B):                                            # against the 50-digit wrenches
        for x, key in zip(terms, "abc"):
            close(x[i], g[robot + "/" + key][i], 1e-12)
    for form in ("rect", "poly"):
        for scheme in (0, 1):
            key = lambda x, i: g["%s/%s/s%d/%s" % (robot, form, scheme, x)][i]  # noqa: E731
            for i in range(B):                                    # single-path TOPPRA takes the device route too
                one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                           ta.constraint.JointAccelerationConstraint(alim[i],
                                                                                     discretization_scheme=scheme),
                                           _cons_of(ta, f, g, robot, form, scheme)],
                                          ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
                st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
                _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
            h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                                ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                                _cons_of(ta, f, g, robot, form, scheme)], path, grid).compute_parameterization(0, 0)
            h = h.to_host()
            for i in range(B):
                _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


def _problems(B, up, seed, m, alim=15.0, step=0.12):
    """Paths starting at the statically stable pose `up` with four random steps of at most `step` rad per joint (a
    tenth of it for prismatic joints)."""
    nv = len(up)
    rng = np.random.RandomState(seed)
    st = np.where(m.packed[4::27][:nv] == 1, 0.1 * step, step)
    way = up + np.cumsum(np.concatenate((np.zeros((B, 1, nv)), rng.uniform(-1, 1, (B, 4, nv)) * st), axis=1), axis=1)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    al = rng.uniform(0.6 * alim, alim, (B, nv))
    return np.linspace(0, 1, 5), way, vlim, np.stack([-al, al], axis=-1)


def _cons(ta, sup, vlim, alim, scheme=1, joint_scheme=1):
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=joint_scheme), sup(scheme)]


def _zmp_inside(F, P, a, b, c, sd, sdd):
    """The zero-moment points of the solved profile at the start of every stage, w = a u + b x + c, are inside the
    polygon P to 1e-9 of its scale and all rows hold to 1e-9 of the wrench's scale; returns whether a support row is
    active (within 1e-6 of the scale)."""
    w = a[:-1] * sdd[:, None] + b[:-1] * (sd[:-1] ** 2)[:, None] + c[:-1]
    v = w @ F.T
    scale = np.abs(w).max(axis=1, keepdims=True) * max(1.0, np.abs(F).max())
    assert (v <= 1e-9 * scale).all(), np.max(v / scale)
    if P is not None:
        size = np.abs(P).max()
        E = np.roll(P, -1, axis=0) - P
        z = sref.zmp(w)
        side = (E[None, :, 0] * (z[:, None, 1] - P[None, :, 1]) - E[None, :, 1] * (z[:, None, 0] - P[None, :, 0]))
        side = side / np.hypot(E[:, 0], E[:, 1])[None]
        assert (side >= -1e-9 * size).all(), side.min()
    return bool((v >= -1e-6 * scale).any())


@pytest.mark.gpu
def test_gpu_256_paths_vs_oracle(ta, golden):
    from oracle import oracle as orc
    g = golden("support_stability")
    m, f = _golden_setup(g, "arm6")
    P = g["arm6/polygon"]
    F = ta.constraint.support_polygon_rows(P)
    B, G = 256, 200
    ss, way, vlim, alim = _problems(B, g["arm6/up"], 51, m)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    sup = lambda s: _cons_of(ta, f, g, "arm6", "poly", s)  # noqa: E731
    h = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim, scheme=0), path, grid).compute_parameterization(0, 0).to_host()
    a_dev, b_dev, c_dev = _terms(f, path, grid)
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b, cc = sref.support_terms_packed(m.packed, f.packed, m.packed_base(), q, qs, qss)
        rows = np.concatenate((lin["rows"], _oracle_rows(F, a, b, cc, grid, False)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            n_active += _zmp_inside(F, P, a_dev[i], b_dev[i], c_dev[i], h["sd"][i], h["sdd"][i])
    print("support rows active on %d of %d solved paths (%.2f)" % (n_active, n_ok, n_active / max(n_ok, 1)))
    assert n_ok > 0.8 * B and n_active > 0.5 * n_ok, (n_ok, n_active)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta, golden):
    g = golden("support_stability")
    m, f = _golden_setup(g, "mobile")
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, g["mobile/up"], 57, m, alim=20.0)
    path = ta.BatchSplineInterpolator(ss, way)
    sup = lambda s: _cons_of(ta, f, g, "mobile", "rect", s)  # noqa: E731
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, sup, vlim[i:i + 1], alim[i:i + 1]), ta.BatchSplineInterpolator(ss, way[i:i + 1]),
                             grids[i, :n]).compute_parameterization(0, 0).to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the reference-style SecondOrderConstraint with cons.wrench as a
    # numpy callback and the footprint rows as F (F_mode 1 rows) equals SupportStabilityConstraint (F_mode 0 rows)
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cons(ta, sup, vlim[i], alim[i], scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cons(ta, sup, vlim[i:i + 1], alim[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0).to_host()
            assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])
            for form in ("rect", "poly"):
                cons = _cons_of(ta, f, g, "mobile", form, scheme)
                F, zeros = cons.F, np.zeros(cons.F.shape[0])
                ref_c = ta.constraint.SecondOrderConstraint(cons.wrench, lambda _: F, lambda _: zeros, nv,
                                                            discretization_scheme=scheme)
                runs = []
                for c in (ref_c, cons):
                    inst = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                                ta.constraint.JointAccelerationConstraint(alim[i]), c], sp,
                                               gridpoints=grid, solver_wrapper="seidel")
                    runs.append(inst.compute_parameterization(0, 0, return_data=True))
                for x, y in zip(*runs):
                    assert _eq(x, y)
                assert runs[0][1] is not None


@pytest.mark.gpu
def test_gpu_toppra_sd_and_quintic_piecewise_poly_path_vs_oracle(ta, golden):
    from oracle import oracle as orc
    g = golden("support_stability")
    m, f = _golden_setup(g, "arm6")
    P = g["arm6/polygon"]
    F = ta.constraint.support_polygon_rows(P)
    sup = lambda s: _cons_of(ta, f, g, "arm6", "poly", s)  # noqa: E731
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(61)
    coeffs = rng.uniform(-0.05, 0.05, (B, k, nseg, nv))
    coeffs[:, -1] = g["arm6/up"]                       # the constant term: at the stable start pose
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 15.0), np.full(nv, 15.0)], axis=1), (B, 1, 1))
    h = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim, 0, 0), path, grid).compute_parameterization(0, 0).to_host()
    a, b, c = _terms(f, path, grid)
    assert (h["status"] == 0).sum() >= B // 2
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    for i in range(B):
        o = orc.solve_rows(np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]),
                                           _oracle_rows(F, a[i], b[i], c[i], grid, False)), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            _zmp_inside(F, P, a[i], b[i], c[i], h["sd"][i], h["sdd"][i])
    # BatchTOPPRAsd, whole and in record chunks: half again the time-optimal duration (or the slowest profile); the
    # zero-moment points stay inside on the blended profiles (a convex combination of (u, x) of two feasible profiles)
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        sd_inst = ta.BatchTOPPRAsd(_cons(ta, sup, vlim, alim, 0, 0), path, grid)
        if chunk:
            sd_inst = ta.BatchTOPPRAsd(_cons(ta, sup, vlim, alim, 0, 0), path, grid,
                                       max_record_bytes=chunk * 8 * ta.engine.record_doubles(sd_inst.R) * sd_inst.G)
            assert sd_inst.chunk_size() == chunk
        sd_inst.set_desired_duration(1.5 * dur)
        r = sd_inst.compute_parameterization(0.0, 0.0)
        runs.append([x.cpu().numpy() for x in (r.status, r.sd, r.sdd, r.duration_slow)])
    for x, y in zip(*runs):
        assert _eq(x, y)
    st, sd, sdd, slow = runs[0]
    assert (st[ok] == 0).all()
    for i in np.flatnonzero(ok):
        _zmp_inside(F, P, a[i], b[i], c[i], sd[i], sdd[i])
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        want = min(1.5 * dur[i], slow[i])
        assert abs(got - want) <= 1e-4 * max(1.0, want), (got, want)


@pytest.mark.gpu
def test_gpu_with_torque_and_velocity_limits_vs_oracle(ta, golden):
    from oracle import oracle as orc
    import kin_ref as kr
    g = golden("support_stability")
    m, f = _golden_setup(g, "arm6")
    sup = lambda s: _cons_of(ta, f, g, "arm6", "rect", s)  # noqa: E731
    F = sup(1).F
    tcp = m.frame("flange", xyz=(0.0, 0.0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 32, 150, 6
    ss, way, vlim, alim = _problems(B, g["arm6/up"], 63, m)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    d = _dev(grid)
    bv = tcp.velocity_norm_terms(*(path.eval_device(d, o).reshape(-1, nv) for o in (0, 1)), S).reshape(B, G)
    speed = 0.3 * bv.max(dim=1).values.cpu().numpy()
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    cons = _cons(ta, sup, vlim, alim) + [ta.constraint.JointTorqueConstraint(m, taulim, fric),
                                         ta.constraint.CartesianVelocityNorm(tcp, S, speed)]
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b, cc = sref.support_terms_packed(m.packed, f.packed, m.packed_base(), q, qs, qss)
        av, btv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        torque = np.stack((av.dot(Fj.T), btv.dot(Fj.T), cv.dot(Fj.T) - gt), axis=1)   # JointTorqueConstraint: collocation
        vq = kr.quad_form(S, kr.frame_velocity_packed(m.packed, tcp.packed, q, qs))
        cart_v = np.stack((np.zeros(G), vq, np.full(G, 0.0 - speed[i])), axis=1)[:, :, None]
        rows = np.concatenate((lin["rows"], _oracle_rows(F, a, b, cc, grid, True), torque, cart_v), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok >= B // 2, n_ok                       # 45 % torque limits leave some poses infeasible at rest


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, golden, monkeypatch):
    from toppra_b200 import _lib_dyn
    g = golden("support_stability")
    m, f = _golden_setup(g, "mobile")
    sup = lambda s: _cons_of(ta, f, g, "mobile", "poly", s)  # noqa: E731
    B = 10
    ss, way, vlim, alim = _problems(B, g["mobile/up"], 67, m)
    path = ta.BatchSplineInterpolator(ss, way)
    grid = np.linspace(0, 1, 80)
    counting = _CountingLib(_lib_dyn.load())
    monkeypatch.setattr(_lib_dyn, "_dlib", counting)
    whole = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim), path, grid)
    whole.compute_parameterization(0, 0)
    assert counting.calls == {"tbd_support_wrench_terms": 1}, counting.calls
    per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
    counting.calls.clear()
    parts = ta.BatchTOPPRA(_cons(ta, sup, vlim, alim), path, grid, max_record_bytes=4 * per_path)
    assert parts.chunk_size() == 4
    parts.compute_parameterization(0, 0)
    assert counting.calls == {"tbd_support_wrench_terms": 3}, counting.calls          # chunks of 4, 4, 2
