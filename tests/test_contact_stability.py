"""Contact wrenches of an object carried on a robot's tool, and its stability on a rectangular support
(RigidBodyFrame.contact_wrench / contact_wrench_terms, ContactStabilityConstraint, contact_wrench_cone;
libtoppra_b200_dyn.so: tbd_contact_wrench, tbd_contact_wrench_terms).

CPU:
  * the float64 numpy double of tests/contact_ref.py equals the 50-digit wrenches of the RAW URDF tree to 1e-13 of the
    scale: both fixtures, locked and unlocked (prismatic fingers on the chain), with and without tool offsets;
  * contact_wrench_cone against its definition: on 2000 random wrenches away from the boundary, "all 16 rows <= 0" iff
    scipy's linprog finds four corner forces inside their friction pyramids that sum to the wrench;
  * hand cases: an object at rest on a level tray, a static tilt just below and just above atan(mu), a centre of mass
    outside the rectangle;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library.
GPU:
  * tbd_contact_wrench on random trees (1 to 16 bodies) against the 50-digit reference and the numpy double within 1e-12;
  * tbd_contact_wrench_terms equals three tbd_contact_wrench launches and the two subtractions, bit for bit; NaN in one
    point touches no other;
  * the reference golden (tests/golden/contact_stability.npz, make_golden_contact.py): TOPPRA and BatchTOPPRA within
    |dK| <= 1e-9 + 1e-8 |K| (the cfg-3 tolerance), equal statuses; 256 paths against the oracle fed with rows from the
    numpy double, same tolerance; the wrenches of the solved profiles are inside the cone, and the cone is active;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, the reference-style
    SecondOrderConstraint with cons.wrench as a numpy callback vs ContactStabilityConstraint: bit-equal;
    BatchTOPPRAsd, a quintic BatchPiecewisePolyPath, and the constraint next to JointTorqueConstraint and
    CartesianVelocityNorm against the oracle; one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import contact_ref as cref
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, FakePath, LOCKED, OFFSET, ROOT, TB_ERR_ARG, TB_ERR_UNSUPPORTED, close, model_of,
                        urdf, _assert_one_terms_launch, _assert_solution, _dev, _dyn_header, _eq, _gpu_present,
                        _model_from_packed, _offset_spec, _oracle_joint_rows, _oracle_rows)

OBJECT = cref.object_packed(0.8, (0.006, -0.004, 0.06), (0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017))
HALF_LENGTHS, FRICTION = (0.05, 0.04), 0.5
G0 = 9.81


def _cone():
    from toppra_b200.constraint import contact_wrench_cone
    return contact_wrench_cone(HALF_LENGTHS, FRICTION)


def _cons_of(ta, f, scheme=1, obj=OBJECT):
    return ta.constraint.ContactStabilityConstraint(f, obj[0], obj[1:4], obj[4:10], HALF_LENGTHS, FRICTION,
                                                    discretization_scheme=scheme)


# ==== CPU: numpy double vs the 50-digit reference, the cone, hand cases, errors, C-ABI ===============================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 83)
    links = ("flange", "wrist2", "base_link") if "arm6" in name else ("hand", "camera", "finger_left", "link3")
    links = [l for l in links if l in m.frames]
    for _ in range(2):
        q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
        spec, frames = {}, {}
        for link in links:
            for o, off in enumerate((None, OFFSET)):
                # the reference frame of a RigidBodyFrame is ignored: the wrench is in the frame's own axes
                ref = ("local", "world", "local_world_aligned")[o + len(link) % 2]
                spec[(link, o)] = (link,) + _offset_spec(off)
                frames[(link, o)] = m.frame(link, reference_frame=ref, **(off or {}))
        want = cref.mp_wrenches(mp, q, qd, qdd, spec, OBJECT)
        for key, f in frames.items():
            got = cref.contact_wrench_packed(m.packed, f.packed, OBJECT, q, qd, qdd)[0]
            close(got, [float(x) for x in want[key]], 1e-13)
        f = frames[(links[0], 1)]
        a, b, c = cref.contact_terms_packed(m.packed, f.packed, OBJECT, q, qd, qdd)
        w0 = cref.contact_wrench_packed(m.packed, f.packed, OBJECT, q, 0 * q, 0 * q)
        assert np.array_equal(c, w0)
        assert np.array_equal(b, cref.contact_wrench_packed(m.packed, f.packed, OBJECT, q, qd, qdd) - w0)


def _in_cone_by_definition(w, X, Y, mu):
    """w = [f; tau] at the centre is the sum of four corner forces f_i at (+-X, +-Y, 0), each with |f_ix|, |f_iy| <=
    mu f_iz (a feasibility LP)."""
    from scipy.optimize import linprog
    A = np.zeros((6, 12))
    for i, (cx, cy) in enumerate(((X, Y), (X, -Y), (-X, Y), (-X, -Y))):
        A[0:3, 3 * i:3 * i + 3] = np.eye(3)
        A[3:6, 3 * i:3 * i + 3] = [[0.0, 0.0, cy], [0.0, 0.0, -cx], [-cy, cx, 0.0]]   # tau_i = p_i x f_i
    pyramid = np.array([[1, 0, -mu], [-1, 0, -mu], [0, 1, -mu], [0, -1, -mu]], dtype=np.float64)
    A_ub = np.zeros((16, 12))
    for i in range(4):
        A_ub[4 * i:4 * i + 4, 3 * i:3 * i + 3] = pyramid
    res = linprog(np.zeros(12), A_ub=A_ub, b_ub=np.zeros(16), A_eq=A, b_eq=w, bounds=[(None, None)] * 12,
                  method="highs")
    assert res.status in (0, 2), res.message
    return res.status == 0


def test_cone_matches_its_definition():
    from toppra_b200.constraint import contact_wrench_cone
    rng = np.random.RandomState(5)
    n = inside = 0
    for X, Y, mu in ((0.05, 0.04, 0.5), (0.2, 0.03, 0.9), (0.01, 0.12, 0.2)):
        F = contact_wrench_cone((X, Y), mu)
        assert F.shape == (16, 6)
        count = 0
        while count < 700:
            # half the samples are built inside the cone (random corner forces) and then perturbed
            if rng.rand() < 0.5:
                w = rng.randn(6) * np.array([1.0, 1.0, 1.0, X + Y, X + Y, (X + Y) * mu])
                w[2] = abs(w[2]) * 2
            else:
                corners = np.abs(rng.randn(4)) * 3
                w = np.zeros(6)
                for fz, (cx, cy) in zip(corners, ((X, Y), (X, -Y), (-X, Y), (-X, -Y))):
                    fi = np.array([rng.uniform(-mu, mu) * fz, rng.uniform(-mu, mu) * fz, fz])
                    w[:3] += fi
                    w[3:] += np.cross([cx, cy, 0.0], fi)
                w = w + 0.05 * rng.randn(6) * np.abs(w).max() * np.array([1, 1, 1, X + Y, X + Y, X + Y])
            v = F @ w
            # at least 1e-9 from the boundary, relative to the wrench's scale
            if np.min(np.abs(v)) < 1e-9 * np.abs(w).max() * max(1.0, X + Y):
                continue
            closed = bool((v <= 0).all())
            assert closed == _in_cone_by_definition(w, X, Y, mu), (X, Y, mu, w, v)
            inside += closed
            count += 1
        n += count
    assert n >= 2000 and 0.2 * n < inside < 0.8 * n, (n, inside)


def _tilt_model(ta):
    """One revolute joint about the world x axis at the origin, the tray on it: q is the tray's tilt."""
    return ta.RigidBodyModel([-1], ["revolute"], [[1.0, 0.0, 0.0]], [np.eye(3)], [[0.0, 0.0, 0.0]], [1.0],
                             [[0.0, 0.0, 0.0]], [[0.01, 0.0, 0.0, 0.01, 0.0, 0.01]], gravity=(0.0, 0.0, -G0))


def test_hand_cases():
    import toppra_b200 as ta
    m = _tilt_model(ta)
    f = m.frame("body0")
    F = _cone()
    mass, r = OBJECT[0], OBJECT[1:4]
    z = np.zeros(1)
    # at rest on a level tray: f = (0, 0, m g0), the centre of pressure is the projection of the centre of mass
    w = cref.contact_wrench_packed(m.packed, f.packed, OBJECT, z, z, z)[0]
    close(w[:3], [0.0, 0.0, mass * G0], 1e-15)
    assert abs(w[5]) <= 1e-15
    close([-w[4] / w[2], w[3] / w[2]], r[:2], 1e-15)
    assert (F @ w < 0).all()
    # a static tilt just below / just above the sliding angle atan(mu): rows 2, 3 are +-f_y - mu f_z
    obj = OBJECT.copy()
    obj[1:4] = (0.0, 0.0, 0.005)                      # low centre of mass: sliding comes before tipping
    for tilt, ok in ((np.arctan(FRICTION) - 1e-3, True), (np.arctan(FRICTION) + 1e-3, False)):
        for s in (1.0, -1.0):
            w = cref.contact_wrench_packed(m.packed, f.packed, obj, [s * tilt], z, z)[0]
            v = F @ w
            assert (v[2:4].max() <= 0) == ok and (v[[0, 1] + list(range(4, 16))] < 0).all(), (tilt, v)
    # a centre of mass outside the rectangle, level tray: a tipping row is violated, the sliding rows are not
    for k, (dx, dy) in enumerate(((1.2, 0.0), (-1.2, 0.0), (0.0, 1.2), (0.0, -1.2))):
        obj = OBJECT.copy()
        obj[1:3] = (dx * HALF_LENGTHS[0], dy * HALF_LENGTHS[1])
        v = F @ cref.contact_wrench_packed(m.packed, f.packed, obj, z, z, z)[0]
        assert (v[:4] < 0).all() and (v[4:8] > 0).sum() == 1, (dx, dy, v[4:8])


def test_value_errors():
    from toppra_b200.constraint import ContactStabilityConstraint, contact_wrench_cone
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.01))
    args = dict(mass=OBJECT[0], com=OBJECT[1:4], inertia=OBJECT[4:10], half_lengths=HALF_LENGTHS, friction=FRICTION)

    def make(**kw):
        a = dict(args)
        a.update(kw)
        return ContactStabilityConstraint(kw.pop("frame", f), **a)

    with pytest.raises(ValueError, match="RigidBodyFrame"):
        ContactStabilityConstraint(lambda q, qd, qdd: np.zeros(6), **args)
    for mass in (0.0, -1.0):
        with pytest.raises(ValueError, match="positive"):
            make(mass=mass)
    for key, bad in (("mass", np.nan), ("mass", np.inf), ("com", [0.0, np.nan, 0.0]), ("inertia", [1, 0, 0, 1, 0, np.inf])):
        with pytest.raises(ValueError, match="finite"):
            make(**{key: bad})
    with pytest.raises(ValueError, match="semi-definite"):
        make(inertia=[1.0, 0.0, 0.0, -0.1, 0.0, 1.0])
    with pytest.raises(ValueError, match="semi-definite"):
        make(inertia=[1.0, 2.0, 0.0, 1.0, 0.0, 1.0])                    # positive diagonal, indefinite
    make(inertia=[0.0] * 6)                                              # a point mass is fine
    with pytest.raises(ValueError, match="shapes"):
        make(com=[0.0, 0.0])
    with pytest.raises(ValueError, match="shapes"):
        make(inertia=[1.0, 1.0, 1.0])
    for hl, mu in (((0.0, 0.1), 0.5), ((0.1, -0.1), 0.5), ((0.1, 0.1), 0.0), ((0.1, 0.1), -0.3)):
        with pytest.raises(ValueError, match="positive"):
            make(half_lengths=hl, friction=mu)
        with pytest.raises(ValueError, match="positive"):
            contact_wrench_cone(hl, mu)
    for hl, mu in (((np.inf, 0.1), 0.5), ((0.1, 0.1), np.nan)):
        with pytest.raises(ValueError, match="finite"):
            make(half_lengths=hl, friction=mu)
    with pytest.raises(ValueError, match="half_lengths"):
        make(half_lengths=(0.1, 0.1, 0.1))
    grid = np.linspace(0, 1, 10)
    c = make()
    assert c.dof == 6 and c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 32          # interpolation
    assert make().F.shape == (16, 6)
    assert ContactStabilityConstraint(f, discretization_scheme=0, **args).num_rows(
        RecordContext(FakePath(3, 6), grid, grid)) == 16
    with pytest.raises(ValueError, match="Wrong dimension"):                                     # a model with another nv
        c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
    assert np.array_equal(c.object, OBJECT)
    # a user callback with a general F keeps its NotImplementedError on the batched route
    from toppra_b200.constraint import SecondOrderConstraint
    user = SecondOrderConstraint(lambda q, qd, qdd: q, lambda _: np.eye(6), lambda _: np.ones(6), 6, batched=True)
    with pytest.raises(NotImplementedError):
        user.num_rows(RecordContext(FakePath(3, 6), grid, grid))
    with pytest.raises(ValueError, match="10 doubles"):
        f.contact_wrench(OBJECT[:9], np.zeros(6), np.zeros(6), np.zeros(6))


def test_dyn_header_prototypes_of_contact_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_contact_wrench"] == ["ptr", "int", "ptr", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_contact_wrench_terms"] == ["ptr", "int", "ptr", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr",
                                                    "ptr", "ptr"]
    for name in ("tbd_contact_wrench", "tbd_contact_wrench_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    assert "#define TBD_OBJECT_DOUBLES 10" in text


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_contact_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good_frame = m.frame("flange", **OFFSET).packed

    def rc(model=m.packed, frame=good_frame, obj=OBJECT, nv=6, M=4, null=None):
        host = [np.array(x, dtype=np.float64) for x in (model, frame, obj)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        cw = [ptr[0], nv, ptr[1], ptr[2], M, d, d, d, d]
        ct = [ptr[0], nv, ptr[1], ptr[2], M, d, d, d, d, d, d]
        if null is not None:                   # index into cw; ct has two more outputs
            cw[null] = None
            ct[null] = None
        r1 = lib.tbd_contact_wrench(*cw, None)
        r2 = lib.tbd_contact_wrench_terms(*ct, None)
        assert r1 == r2, (r1, r2)
        assert r1 == 0 or _lib.load().tb_last_error()
        return r1

    for k in (0, 2, 3, 5, 6, 7, 8):
        assert rc(null=k) == TB_ERR_ARG
    for k in (9, 10):                          # the extra outputs of the terms entry
        host = [np.array(x, dtype=np.float64) for x in (m.packed, good_frame, OBJECT)]
        ct = [ctypes.c_void_p(h.ctypes.data) for h in host]
        args = [ct[0], 6, ct[1], ct[2], 4, d, d, d, d, d, d]
        args[k] = None
        assert lib.tbd_contact_wrench_terms(*args, None) == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model) == TB_ERR_ARG
    for j, value in ((0, 6.0), (0, -2.0), (0, 0.5), (5, np.nan), (11, np.inf)):   # bad frames
        f = good_frame.copy()
        f[j] = value
        assert rc(frame=f) == TB_ERR_ARG
    for j, value in ((0, 0.0), (0, -1.0), (0, np.nan), (2, np.inf), (7, -np.inf), (9, np.nan)):   # bad objects
        o = OBJECT.copy()
        o[j] = value
        assert rc(obj=o) == TB_ERR_ARG
    assert b"object" in _lib.load().tb_last_error()
    for ref in (0.0, 1.0, 2.0, 7.0):                             # the reference-frame field is ignored: the call
        f = good_frame.copy()                                    # passes validation and fails only at the launch,
        f[13] = ref                                              # as there is no device here
        assert rc(frame=f) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
        assert b"launch failed" in _lib.load().tb_last_error()


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_contact_wrench_random_trees_vs_mp(ta, nv):
    from toppra_b200.dynamics import rpy_matrix
    rng = np.random.RandomState(900 + nv)
    m = _model_from_packed(ta, rr.random_tree(rng, nv))
    mp = rr.MpRobot.from_packed(m.packed)
    P = 2 if nv <= 8 else 1
    q, qd, qdd = (rng.uniform(-2, 2, (P, nv)) for _ in range(3))
    obj = cref.object_packed(rng.uniform(0.2, 3.0), rng.randn(3) * 0.1, (0.01, 0.001, -0.002, 0.02, 0.001, 0.015))
    for k in sorted({nv - 1, int(rng.randint(nv))}):
        off = dict(xyz=tuple(rng.randn(3) * 0.2), rpy=tuple(rng.uniform(-3, 3, 3)))
        f = m.frame("body%d" % k, **off)
        w = f.contact_wrench(obj, _dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
        spec = {0: ("b%d" % k, rpy_matrix(off["rpy"]), np.asarray(off["xyz"]))}
        for i in range(P):
            want = cref.mp_wrenches(mp, q[i], qd[i], qdd[i], spec, obj)[0]
            close(w[i], [float(x) for x in want], 1e-12)
        Q, QD, QDD = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
        got = f.contact_wrench(obj, _dev(Q), _dev(QD), _dev(QDD)).cpu().numpy()
        want = cref.contact_wrench_packed(m.packed, f.packed, obj, Q, QD, QDD)
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
        assert np.array_equal(f.contact_wrench(obj, Q[3], QD[3], QDD[3]), got[3])   # numpy (nv,): a device round trip
        assert np.array_equal(f.contact_wrench(obj, Q[:5], QD[:5], QDD[:5]), got[:5])


@pytest.mark.gpu
def test_gpu_contact_terms_bit_equal_three_launches(ta):
    import torch
    m = model_of("arm7_gripper.urdf")                            # fingers unlocked: prismatic bodies on the chain
    rng = np.random.RandomState(11)
    M = 3000
    q, qs, qss = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(3))
    zero = torch.zeros_like(q)
    for link, ref in (("finger_left", "local"), ("camera", "world"), ("hand", "local_world_aligned")):
        f = m.frame(link, reference_frame=ref, **OFFSET)
        c = f.contact_wrench(OBJECT, q, zero, zero)
        a = f.contact_wrench(OBJECT, q, zero, qs) - c
        b = f.contact_wrench(OBJECT, q, qs, qss) - c
        got = f.contact_wrench_terms(OBJECT, q, qs, qss)
        for x, y in zip(got, (a, b, c)):
            assert x.shape == (M, 6) and torch.equal(x, y), link
        # the reference frame is ignored
        same = m.frame(link, reference_frame="local", **OFFSET).contact_wrench_terms(OBJECT, q, qs, qss)
        assert all(torch.equal(x, y) for x, y in zip(got, same))
    # NaN in one point leaves every other point as it was
    f = model_of("arm6.urdf").frame("flange", **OFFSET)
    q, qs, qss = rng.uniform(-2, 2, (3, 64, 6))
    qn, qsn, qssn = q.copy(), qs.copy(), qss.copy()
    qn[5, 2] = np.nan
    qsn[9, 0] = np.nan
    qssn[17, 4] = np.nan
    ref = [x.cpu().numpy() for x in f.contact_wrench_terms(OBJECT, _dev(q), _dev(qs), _dev(qss))]
    got = [x.cpu().numpy() for x in f.contact_wrench_terms(OBJECT, _dev(qn), _dev(qsn), _dev(qssn))]
    assert np.isnan(got[2][5]).any() and np.isnan(got[0][9]).any() and np.isnan(got[1][17]).any()
    keep = np.ones(64, bool)
    keep[[5, 9, 17]] = False
    for x, y in zip(got, ref):
        assert np.array_equal(x[keep], y[keep])


def _terms(f, obj, path, grid):
    """a, b, c (B, G, 6) of the contact wrench on the device path at the grid."""
    d = _dev(grid)
    out = f.contact_wrench_terms(obj, *(path.eval_device(d, o).reshape(-1, f.nv) for o in (0, 1, 2)))
    return [x.reshape(path.B, len(grid), 6).cpu().numpy() for x in out]


def _in_cone(F, a, b, c, sd, sdd):
    """The wrench of the solved profile at the start of every stage, w = a u + b x + c, is inside the cone to 1e-9 of
    its scale; returns whether a contact row is active (within 1e-6 of the scale)."""
    w = a[:-1] * sdd[:, None] + b[:-1] * (sd[:-1] ** 2)[:, None] + c[:-1]
    v = w @ F.T
    scale = np.abs(w).max(axis=1, keepdims=True) * max(1.0, np.abs(F).max())
    assert (v <= 1e-9 * scale).all(), np.max(v / scale)
    return bool((v >= -1e-6 * scale).any())


def _tray_problems(B, up, seed, velocity, step=0.06):
    """Paths starting at the tray-up pose with four random steps of at most `step` rad per joint (as
    make_golden_contact.py)."""
    nv = len(up)
    rng = np.random.RandomState(seed)
    way = up + np.cumsum(np.concatenate((np.zeros((B, 1, nv)), rng.uniform(-step, step, (B, 4, nv))), axis=1), axis=1)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    al = rng.uniform(6, 10, (B, nv))
    return np.linspace(0, 1, 5), way, vlim, np.stack([-al, al], axis=-1)


def _cons(ta, f, vlim, alim, scheme=1, joint_scheme=1):
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=joint_scheme), _cons_of(ta, f, scheme)]


def _golden_frame(g, robot, m):
    return m.frame(str(g[robot + "/link"]), xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"])


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("contact_stability")
    m = model_of(name, locked)
    f = _golden_frame(g, robot, m)
    assert np.array_equal(g["object"], OBJECT) and tuple(g["half_lengths"]) == HALF_LENGTHS
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim = (g[robot + "/" + k] for k in ("way", "vlim", "alim"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    terms = _terms(f, OBJECT, path, grid)
    for i in range(B):                                            # against the 50-digit wrenches
        for x, key in zip(terms, "abc"):
            close(x[i], g[robot + "/" + key][i], 1e-12)
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (robot, scheme, x)][i]  # noqa: E731
        for i in range(B):                                        # single-path TOPPRA takes the device route too
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                       ta.constraint.JointAccelerationConstraint(alim[i], discretization_scheme=scheme),
                                       _cons_of(ta, f, scheme)],
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            _cons_of(ta, f, scheme)], path, grid).compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


@pytest.mark.gpu
def test_gpu_256_paths_vs_oracle(ta, golden):
    from oracle import oracle as orc
    g = golden("contact_stability")
    m = model_of("arm6.urdf")
    f = _golden_frame(g, "arm6", m)
    F = _cone()
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _tray_problems(B, g["arm6/up"], 51, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    h = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, scheme=0), path, grid).compute_parameterization(0, 0).to_host()
    a_dev, b_dev, c_dev = _terms(f, OBJECT, path, grid)
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b, cc = cref.contact_terms_packed(m.packed, f.packed, OBJECT, q, qs, qss)
        rows = np.concatenate((lin["rows"], _oracle_rows(F, a, b, cc, grid, False)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            n_active += _in_cone(F, a_dev[i], b_dev[i], c_dev[i], h["sd"][i], h["sdd"][i])
    print("contact rows active on %d of %d solved paths (%.2f)" % (n_active, n_ok, n_active / max(n_ok, 1)))
    assert n_ok > 0.9 * B and n_active > 0.5 * n_ok, (n_ok, n_active)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta, golden):
    g = golden("contact_stability")
    m = model_of("arm7_gripper.urdf", LOCKED)
    f = _golden_frame(g, "arm7", m)
    B, nv = 12, m.nv
    ss, way, vlim, alim = _tray_problems(B, g["arm7/up"], 57, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cons(ta, f, vlim, alim), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, f, vlim[i:i + 1], alim[i:i + 1]), ta.BatchSplineInterpolator(ss, way[i:i + 1]),
                             grids[i, :n]).compute_parameterization(0, 0).to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the reference-style SecondOrderConstraint with cons.wrench as a
    # numpy callback and the cone as F (F_mode 1 rows) equals ContactStabilityConstraint (F_mode 0 rows)
    F, zeros = _cone(), np.zeros(16)
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cons(ta, f, vlim[i], alim[i], scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cons(ta, f, vlim[i:i + 1], alim[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0).to_host()
            assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])
            cons = _cons_of(ta, f, scheme)
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
    g = golden("contact_stability")
    m = model_of("arm6.urdf")
    f = _golden_frame(g, "arm6", m)
    F = _cone()
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(61)
    coeffs = rng.uniform(-0.08, 0.08, (B, k, nseg, nv))
    coeffs[:, -1] += g["arm6/up"]                      # the constant term: around the tray-up pose
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    h = ta.BatchTOPPRA(_cons(ta, f, vlim, alim, 0, 0), path, grid).compute_parameterization(0, 0).to_host()
    a, b, c = _terms(f, OBJECT, path, grid)
    assert (h["status"] == 0).sum() >= B // 2
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    for i in range(B):
        o = orc.solve_rows(np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]),
                                           _oracle_rows(F, a[i], b[i], c[i], grid, False)), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            _in_cone(F, a[i], b[i], c[i], h["sd"][i], h["sdd"][i])
    # BatchTOPPRAsd, whole and in record chunks: half again the time-optimal duration (or the slowest profile); the
    # wrenches stay in the cone on the blended profiles (a convex combination of (u, x) of two feasible profiles)
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        sd_inst = ta.BatchTOPPRAsd(_cons(ta, f, vlim, alim, 0, 0), path, grid)
        if chunk:
            sd_inst = ta.BatchTOPPRAsd(_cons(ta, f, vlim, alim, 0, 0), path, grid,
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
        _in_cone(F, a[i], b[i], c[i], sd[i], sdd[i])
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        want = min(1.5 * dur[i], slow[i])
        assert abs(got - want) <= 1e-4 * max(1.0, want), (got, want)


@pytest.mark.gpu
def test_gpu_with_torque_and_velocity_limits_vs_oracle(ta, golden):
    from oracle import oracle as orc
    import kin_ref as kr
    g = golden("contact_stability")
    m = model_of("arm6.urdf")
    f = _golden_frame(g, "arm6", m)
    F = _cone()
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 32, 150, 6
    ss, way, vlim, alim = _tray_problems(B, g["arm6/up"], 63, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    d = _dev(grid)
    bv = f.velocity_norm_terms(*(path.eval_device(d, o).reshape(-1, nv) for o in (0, 1)), S).reshape(B, G)
    speed = 0.3 * bv.max(dim=1).values.cpu().numpy()
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    cons = _cons(ta, f, vlim, alim) + [ta.constraint.JointTorqueConstraint(m, taulim, fric),
                                       ta.constraint.CartesianVelocityNorm(f, S, speed)]
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b, cc = cref.contact_terms_packed(m.packed, f.packed, OBJECT, q, qs, qss)
        av, btv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        torque = np.stack((av.dot(Fj.T), btv.dot(Fj.T), cv.dot(Fj.T) - gt), axis=1)   # JointTorqueConstraint: collocation
        vq = kr.quad_form(S, kr.frame_velocity_packed(m.packed, f.packed, q, qs))
        cart_v = np.stack((np.zeros(G), vq, np.full(G, 0.0 - speed[i])), axis=1)[:, :, None]
        rows = np.concatenate((lin["rows"], _oracle_rows(F, a, b, cc, grid, True), torque, cart_v), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok > 0.8 * B


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, golden, monkeypatch):
    g = golden("contact_stability")
    m = model_of("arm6.urdf")
    f = _golden_frame(g, "arm6", m)
    ss, way, vlim, alim = _tray_problems(10, g["arm6/up"], 67, m.velocity_limit)
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, f, vlim, alim), ta.BatchSplineInterpolator(ss, way),
                             np.linspace(0, 1, 80), "tbd_contact_wrench_terms")
