"""The wrench across a joint, and bearing and reducer limits on it (RigidBodyFrame.joint_wrench / joint_wrench_terms,
JointWrenchConstraint, JointWrenchConstraint.bearing; libtoppra_b200_dyn.so: tbd_joint_wrench, tbd_joint_wrench_terms).

CPU:
  * the float64 numpy double of tests/joint_wrench_ref.py equals the 50-digit wrench summed over the joint's subtree of
    the RAW URDF tree, within 1e-13 of the sample's largest force (forces) and largest moment (moments): arm6.urdf and
    arm7_gripper.urdf (fingers locked and unlocked), frames on every moving body, both reference frames, offset and
    rotated frames;
  * the polygon rows of the bearing form: every wrench within them has a radial force and a tilting moment of at most
    the limit, every wrench within cos(pi / sides) of it satisfies them;
  * every ValueError of both constructors and of the frame methods; the ctypes prototypes against the header; each
    refused call of the two entries returns its TB_ERR_* and message from the real library;
  * the launch plan of both forms on the recording library: one terms launch and one tb_rows_canlinear call per batch
    or record chunk, with the eye form (modes 2 and 3) or the constant F with a shared g (mode 0).
GPU:
  * tbd_joint_wrench on random trees of 1 to 16 bodies, frames on every body, against the numpy double within 1e-12
    (and the 50-digit reference on a few points); the terms entry bit-equal to three launches and the subtractions; at a
    body origin in "local" axes the axis component is tbd_rnea's torque; on arm6 the joint-1 wrench moved to the base
    plus the base's weight is tbd_support_wrench;
  * the reference golden (tests/golden/joint_wrench.npz, make_golden_joint_wrench.py): TOPPRA and BatchTOPPRA within the
    cfg-3 tolerance, equal statuses, box and bearing forms, both schemes;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1 and the reference-style
    SecondOrderConstraint with cons.wrench as a callback: bit-equal; a quintic path against the oracle; BatchTOPPRAsd
    whole and in record chunks; one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import joint_wrench_ref as jr
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, TB_ERR_ARG, TB_ERR_UNSUPPORTED, _assert_one_terms_launch, _assert_solution,
                        _dev, _dyn_header, _eq, _gpu_present, _model_from_packed, _oracle_joint_rows, model_of, urdf)
from test_dyn_calls import H, T, _OUTPUTS, _context, _flat, _rows_call, _run, arm, calls  # noqa: F401

OFFSETS = [dict(), dict(xyz=(0.03, -0.02, 0.1), rpy=(0.3, -0.2, 0.5)), dict(xyz=(-0.1, 0.05, 0.0), rpy=(0.0, 1.2, 0.0))]
REFS = ("local", "local_world_aligned")


def _close_wrench(got, want, tol):
    """Forces within tol of the largest force, moments within tol of the largest moment (at least 1)."""
    got, want = np.atleast_2d(got), np.atleast_2d(want)
    for sl in (slice(0, 3), slice(3, 6)):
        scale = max(1.0, float(np.abs(want[:, sl]).max()))
        err = float(np.abs(got[:, sl] - want[:, sl]).max())
        assert err <= tol * scale, (err, scale, sl)


def _body_frames(m):
    """One frame name per moving body: the first of the frame table on that body."""
    out = {}
    for name, (body, _, _) in sorted(m.frames.items()):
        if body >= 0 and body not in out:
            out[body] = name
    assert sorted(out) == list(range(m.nv))
    return out


# ==== CPU: numpy double vs the 50-digit reference ===================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 411)
    q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
    for body, link in _body_frames(m).items():
        for k, off in enumerate(OFFSETS):
            for ref in REFS:
                f = m.frame(link, reference_frame=ref, **off)
                want = jr.mp_joint_wrench(mp, body, q, qd, qdd, f.R, f.p, jr.LOCAL if ref == "local" else
                                          jr.LOCAL_WORLD_ALIGNED)
                got = jr.joint_wrench_packed(m.packed, f.packed, q, qd, qdd)[0]
                _close_wrench(got, want, 1e-13)
    a, b, c = jr.joint_wrench_terms_packed(m.packed, f.packed, q, qd, qdd)
    w0 = jr.joint_wrench_packed(m.packed, f.packed, q, 0 * q, 0 * q)
    assert np.array_equal(c, w0)
    assert np.array_equal(b, jr.joint_wrench_packed(m.packed, f.packed, q, qd, qdd) - w0)
    a4, b4, c4 = jr.joint_wrench_terms_packed(m.packed, f.packed, q, qd, qdd, (5, 1, 3))
    assert np.array_equal(a4, a[:, [1, 3, 5]]) and np.array_equal(c4, c[:, [1, 3, 5]])


def test_static_wrench_of_the_last_body_is_its_weight():
    """The wrench across the last joint at rest is the weight of what it carries: f = -m g in world axes."""
    m = model_of("arm6.urdf")
    f = m.frame("flange", reference_frame="local_world_aligned")
    z = np.zeros(m.nv)
    for q in np.random.RandomState(2).uniform(-2, 2, (3, m.nv)):
        w = jr.joint_wrench_packed(m.packed, f.packed, q, z, z)[0]
        np.testing.assert_allclose(w[:3], -m.body(5)[17] * m.gravity, rtol=0, atol=1e-13 * 9.81 * m.body(5)[17])


# ==== CPU: polygon rows ==============================================================================================
def _in_plane(rng, a, n, top):
    """n random vectors normal to the unit vector a with norms uniform in [0, top]."""
    v = rng.randn(n, 3)
    v = v - (v @ a)[:, None] * a
    return v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(0, top, (n, 1))


@pytest.mark.parametrize("sides", [4, 5, 8, 13])
def test_bearing_polygon_rows(sides):
    from toppra_b200.constraint.joint_wrench import bearing_rows
    rng = np.random.RandomState(sides)
    c = np.cos(np.pi / sides)
    n = 20000
    for _ in range(5):
        a = rng.randn(3)
        a /= np.linalg.norm(a)
        axial, radial, tilting = rng.uniform(1, 100, 3)
        F, g = bearing_rows(a, axial, radial, tilting, sides)
        assert F.shape == (2 + 2 * sides, 6) and g.shape == (2 + 2 * sides,)
        fa, na = rng.uniform(-1.2 * axial, 1.2 * axial, n), rng.uniform(-1e3, 1e3, n)
        fr, nt = _in_plane(rng, a, n, 1.2 * radial), _in_plane(rng, a, n, 1.2 * tilting)
        w = np.concatenate((fa[:, None] * a + fr, na[:, None] * a + nt), axis=1)
        inside = (w @ F.T <= g).all(axis=1)
        rn, tn = np.linalg.norm(fr, axis=1), np.linalg.norm(nt, axis=1)
        assert 0.05 * n < inside.sum() < 0.95 * n
        # every wrench within the rows is within the limits
        assert (np.abs(fa[inside]) <= axial).all()
        assert (rn[inside] <= radial * (1 + 1e-12)).all() and (tn[inside] <= tilting * (1 + 1e-12)).all()
        # every wrench within cos(pi / sides) of them is within the rows
        sure = (np.abs(fa) <= axial) & (rn <= radial * c) & (tn <= tilting * c)
        assert sure.sum() > 0.05 * n and inside[sure].all()
        only_r, only_t = bearing_rows(a, radial=radial, sides=sides), bearing_rows(a, tilting=tilting, sides=sides)
        assert only_r[0].shape == (sides, 6) and not only_r[0][:, 3:].any() and np.allclose(only_r[1], radial * c)
        assert only_t[0].shape == (sides, 6) and not only_t[0][:, :3].any() and np.allclose(only_t[1], tilting * c)
        # the polygon is inscribed: the vertex between two neighbouring normals lies on the circle
        d = only_r[0][:, :3]
        assert np.allclose(d @ a, 0.0, atol=1e-15) and np.allclose(np.linalg.norm(d, axis=1), 1.0)
        vertex = radial * (d[0] + d[1]) / np.linalg.norm(d[0] + d[1])
        assert np.isclose((d @ vertex).max(), radial * c, rtol=1e-12)


# ==== CPU: errors, header, C-ABI checks ==============================================================================
def test_value_errors():
    from toppra_b200.constraint import JointWrenchConstraint
    m = model_of("arm6.urdf")
    loc = m.frame("forearm", reference_frame="local")
    lwa = m.frame("forearm")
    world = m.frame("forearm", reference_frame="world")
    base = m.frame("base_link", reference_frame="local")
    lim = np.array([[-1.0, 1.0]] * 6)
    with pytest.raises(ValueError, match="needs a RigidBodyFrame"):
        JointWrenchConstraint(m, lim)
    with pytest.raises(ValueError, match="on the base.*SupportStabilityConstraint"):
        JointWrenchConstraint(base, lim)
    with pytest.raises(ValueError, match="world"):
        JointWrenchConstraint(world, lim)
    with pytest.raises(ValueError, match=r"\[fx, fy, fz, nx, ny, nz\]"):
        JointWrenchConstraint(loc, lim[:2], components=(0, 6))
    with pytest.raises(ValueError, match=r"\[fx, fy, fz, nx, ny, nz\]"):
        JointWrenchConstraint(loc, lim[:2], components=(1, 1))
    with pytest.raises(ValueError, match=r"\[fx, fy, fz, nx, ny, nz\]"):
        JointWrenchConstraint(loc, lim[:0], components=())
    with pytest.raises(ValueError, match="wlim has shape"):
        JointWrenchConstraint(loc, lim[:3], components=(0, 1))
    with pytest.raises(ValueError, match="wlim has shape"):
        JointWrenchConstraint(loc, lim.reshape(-1))
    with pytest.raises(ValueError, match="finite"):
        JointWrenchConstraint(lwa, [[-np.inf, 1.0]], components=(2,))
    with pytest.raises(ValueError, match="lower limit exceeds"):
        JointWrenchConstraint(lwa, [[2.0, 1.0]], components=(2,))
    c = JointWrenchConstraint(lwa, np.stack([lim[:2]] * 3), components=(5, 1))
    assert c.limits.shape == (3, 2, 2) and c.components == (1, 5)
    with pytest.raises(ValueError, match="needs a RigidBodyFrame"):
        JointWrenchConstraint.bearing(None, axial=1.0)
    with pytest.raises(ValueError, match="on the base"):
        JointWrenchConstraint.bearing(base, axial=1.0)
    with pytest.raises(ValueError, match="world"):
        JointWrenchConstraint.bearing(world, axial=1.0)
    with pytest.raises(ValueError, match="\"local\""):
        JointWrenchConstraint.bearing(lwa, axial=1.0)
    with pytest.raises(ValueError, match="at least one"):
        JointWrenchConstraint.bearing(loc)
    for kw in (dict(axial=0.0), dict(radial=-1.0), dict(tilting=np.inf), dict(axial=np.nan), dict(radial=[1.0, 2.0])):
        with pytest.raises(ValueError, match="must be a finite number > 0"):
            JointWrenchConstraint.bearing(loc, **kw)
    for sides in (3, 0, 8.0, "8"):
        with pytest.raises(ValueError, match="sides"):
            JointWrenchConstraint.bearing(loc, axial=1.0, sides=sides)
    b = JointWrenchConstraint.bearing(loc, axial=100.0, tilting=20.0, sides=6)
    assert b.F.shape == (8, 6) and b.g.shape == (8,) and b._const_g is b.g
    np.testing.assert_allclose(b.axis, loc.R.T @ m.body(2)[2:5], rtol=0, atol=0)
    np.testing.assert_allclose(b.F[0, :3], b.axis, rtol=0, atol=0)
    for fn in (lambda: base.joint_wrench(np.zeros(6), np.zeros(6), np.zeros(6)),
               lambda: base.joint_wrench_terms(None, None, None)):
        with pytest.raises(ValueError, match="on the base"):
            fn()
    for fn in (lambda: world.joint_wrench(np.zeros(6), np.zeros(6), np.zeros(6)),
               lambda: world.joint_wrench_terms(None, None, None)):
        with pytest.raises(ValueError, match="world"):
            fn()


def test_dyn_header_prototypes_of_joint_wrench_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_joint_wrench"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_joint_wrench_terms"] == ["ptr", "int", "ptr", "int", "int", "ptr", "ptr", "ptr", "ptr", "ptr",
                                                  "ptr", "ptr"]
    for name in ("tbd_joint_wrench", "tbd_joint_wrench_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_joint_wrench_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good = m.frame("forearm", xyz=(0.03, -0.02, 0.0), rpy=(0.0, 0.0, 0.5), reference_frame="local").packed

    def err():
        return _lib.load().tb_last_error()

    def rc(model=m.packed, frame=good, nv=6, M=4, comps=63, null=None):
        host = [np.array(x, dtype=np.float64) for x in (model, frame)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        cw = [ptr[0], nv, ptr[1], M, d, d, d, d]
        ct = [ptr[0], nv, ptr[1], comps, M, d, d, d, d, d, d]
        if null is not None:                   # index into cw; ct has the mask before M and two more outputs
            cw[null] = None
            ct[null if null < 3 else null + 1] = None
        r1 = lib.tbd_joint_wrench(*cw, None)
        e1 = err()
        r2 = lib.tbd_joint_wrench_terms(*ct, None)
        e2 = err()
        if comps == 63:
            assert r1 == r2 and e1.replace(b"tbd_joint_wrench:", b"") == e2.replace(b"tbd_joint_wrench_terms:", b"")
        assert r2 == 0 or e2.startswith(b"tbd_joint_wrench_terms: ")
        return r2

    for k in (0, 2, 4, 5, 6, 7):
        assert rc(null=k) == TB_ERR_ARG and b"null pointer" in err()
    for k in (9, 10):                          # the extra outputs of the terms entry
        host = [np.array(x, dtype=np.float64) for x in (m.packed, good)]
        p = [ctypes.c_void_p(h.ctypes.data) for h in host]
        args = [p[0], 6, p[1], 63, 4, d, d, d, d, d, d]
        args[k] = None
        assert lib.tbd_joint_wrench_terms(*args, None) == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and b"M=0 must be positive" in err()
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and b"nv=0 outside 1..16" in err()
    assert rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED and b"nv=17 outside 1..16" in err()
    for j, value in ((0, 6.0), (0, -2.0), (0, 0.5), (5, np.nan), (11, np.inf)):   # bad frames
        f = good.copy()
        f[j] = value
        assert rc(frame=f) == TB_ERR_ARG
    f = good.copy()
    f[0] = -1.0                                                  # a frame on the base has no joint
    assert rc(frame=f) == TB_ERR_ARG
    assert b"on the base (body -1)" in err() and b"SupportStabilityConstraint" in err()
    f = good.copy()
    f[13] = 0.0                                                  # TBD_WORLD
    assert rc(frame=f) == TB_ERR_UNSUPPORTED
    assert b"the world reference frame is not supported for joint wrenches" in err()
    for comps in (0, -1, 64, 1 << 20):
        assert rc(comps=comps) == TB_ERR_ARG
        assert b"tbd_joint_wrench_terms: components=%d must be a bit mask in 1..63" % comps in err()
    for ref in (1.0, 2.0):                                       # good calls pass validation and fail only at the launch
        for comps in (1, 21, 63):
            f = good.copy()
            f[13] = ref
            assert rc(frame=f, comps=comps) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)
            assert b"launch failed" in err()


# ==== CPU: launch plan on the recording library =======================================================================
@pytest.mark.parametrize("lo,hi,total", [(0, 4, 4), (1, 3, 4)])
@pytest.mark.parametrize("interp", [False, True])
def test_launch_plan(calls, arm, monkeypatch, lo, hi, total, interp):  # noqa: F811
    from toppra_b200.constraint import JointWrenchConstraint
    monkeypatch.setitem(_OUTPUTS, "tbd_joint_wrench_terms", 3)
    nv, G = arm.nv, 6
    f = arm.frame("forearm", xyz=(0.0, 0.0, 0.05), reference_frame="local")
    B, n = hi - lo, (hi - lo) * G
    name = "tbd_joint_wrench_terms"
    wlim = np.array([[-3.0, 4.0], [-5.0, 6.0]])                  # components (5, 1): row 0 limits nz, row 1 fy
    for lim in (wlim, np.stack([wlim * (1 + i) for i in range(total)])):
        cons = JointWrenchConstraint(f, lim, components=(5, 1), discretization_scheme=int(interp))
        ctx, bp = _context(nv, total, G, lo, hi, total)
        rows, log = _run(calls, cons, ctx)
        assert rows == (2 if interp else 1) * 4
        srt = lim[..., ::-1, :]                                  # the kernel's columns: fy, nz
        g = np.concatenate((srt[..., 1], -srt[..., 0]), axis=-1)
        g = g if g.ndim == 1 else g[lo:hi]
        out = [T(name + ".%d" % s, (n, 2)) for s in (8, 9, 10)]
        assert log == [
            [name, H(arm.packed), nv, H(f.packed), 2 + 32, n, T("q0", (n, nv)), T("q1", (n, nv)), T("q2", (n, nv))]
            + out + [None],
            _rows_call(*[T(name + ".%d" % s, (B, G, 2)) for s in (8, 9, 10)], None, T(_flat(g), g.shape),
                       2 if g.ndim == 1 else 3, B, G, 2, 4, interp)]
    cons = JointWrenchConstraint.bearing(f, axial=300.0, radial=500.0, tilting=80.0, discretization_scheme=int(interp))
    k = cons.F.shape[0]
    assert k == 18
    ctx, bp = _context(nv, total, G, lo, hi, total)
    rows, log = _run(calls, cons, ctx)
    assert rows == (2 if interp else 1) * k
    assert log == [
        [name, H(arm.packed), nv, H(f.packed), 63, n, T("q0", (n, nv)), T("q1", (n, nv)), T("q2", (n, nv))]
        + [T(name + ".%d" % s, (n, 6)) for s in (8, 9, 10)] + [None],
        _rows_call(*[T(name + ".%d" % s, (B, G, 6)) for s in (8, 9, 10)], T(_flat(cons.F), (k, 6)),
                   T(_flat(cons.g), (k,)), 0, B, G, 6, k, interp)]
    assert (cons.g > 0).all()


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _tree(rng, nv):
    """rr.random_tree with a prismatic joint for nv >= 3 and at most two root children."""
    packed = rr.random_tree(rng, nv)
    b = packed[3:].reshape(nv, 27)
    b[2:, 0] = np.maximum(b[2:, 0], 0)
    if nv >= 3:
        b[nv // 2, 1] = 1
    return packed


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_joint_wrench_random_trees(ta, nv):
    from toppra_b200.dynamics import rpy_matrix
    rng = np.random.RandomState(1700 + nv)
    m = _model_from_packed(ta, _tree(rng, nv))
    mp = rr.MpRobot.from_packed(m.packed)
    Q, QD, QDD = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
    for body in range(nv):
        m.frames["f%d" % body] = (body, rpy_matrix(rng.uniform(-3, 3, 3)), rng.randn(3) * 0.2)
        for ref in REFS:
            f = m.frame("f%d" % body, reference_frame=ref)
            got = f.joint_wrench(_dev(Q), _dev(QD), _dev(QDD)).cpu().numpy()
            want = jr.joint_wrench_packed(m.packed, f.packed, Q, QD, QDD)
            _close_wrench(got, want, 1e-12)
            if body in (0, nv - 1):                              # and the 50-digit reference on one point
                w = jr.mp_joint_wrench(mp, body, Q[0], QD[0], QDD[0], f.R, f.p,
                                       jr.LOCAL if ref == "local" else jr.LOCAL_WORLD_ALIGNED)
                _close_wrench(got[0], w, 1e-12)
            assert np.array_equal(f.joint_wrench(Q[3], QD[3], QDD[3]), got[3])   # numpy (nv,): a device round trip


@pytest.mark.gpu
def test_gpu_terms_bit_equal_three_launches(ta):
    import torch
    rng = np.random.RandomState(23)
    for m in (model_of("arm7_gripper.urdf"), _model_from_packed(ta, _tree(rng, 9))):
        M = 3000
        q, qs, qss = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(3))
        zero = torch.zeros_like(q)
        for body in (0, m.nv // 2, m.nv - 1):
            m.frames["t%d" % body] = (body, np.eye(3), np.array([0.01, -0.03, 0.05]))
            for ref in REFS:
                f = m.frame("t%d" % body, rpy=(0.3, -0.2, 0.5), reference_frame=ref)
                c = f.joint_wrench(q, zero, zero)
                a = f.joint_wrench(q, zero, qs) - c
                b = f.joint_wrench(q, qs, qss) - c
                for comps in ((0, 1, 2, 3, 4, 5), (4, 0), (3,)):
                    cols = sorted(comps)
                    got = f.joint_wrench_terms(q, qs, qss, comps)
                    for x, y in zip(got, (a, b, c)):
                        assert x.shape == (M, len(cols)) and torch.equal(x, y[:, cols]), (body, ref, comps)


@pytest.mark.gpu
def test_gpu_axis_component_is_the_joint_torque(ta):
    rng = np.random.RandomState(29)
    for m in (model_of("arm6.urdf"), _model_from_packed(ta, _tree(rng, 11))):
        q, qd, qdd = (_dev(rng.uniform(-3, 3, (2000, m.nv))) for _ in range(3))
        tau = m(q, qd, qdd).cpu().numpy()
        scale = max(1.0, np.abs(tau).max())
        for k in range(m.nv):
            m.frames["o%d" % k] = (k, np.eye(3), np.zeros(3))
            w = m.frame("o%d" % k, reference_frame="local").joint_wrench(q, qd, qdd).cpu().numpy()
            bd = m.body(k)
            got = (w[:, 3:] if bd[1] == 0 else w[:, :3]) @ bd[2:5]
            assert np.abs(got - tau[:, k]).max() <= 1e-14 * scale, k


@pytest.mark.gpu
def test_gpu_root_joint_wrench_plus_base_weight_is_the_support_wrench(ta):
    m = model_of("arm6.urdf")
    assert m.body(0)[0] == -1 and all(m.body(k)[0] >= 0 for k in range(1, m.nv))
    rng = np.random.RandomState(31)
    q, qd, qdd = (_dev(rng.uniform(-3, 3, (2000, m.nv))) for _ in range(3))
    w = m.frame("shoulder", reference_frame="local_world_aligned").joint_wrench(q, qd, qdd).cpu().numpy()
    p0 = m.body(0)[14:17]                                         # body 0's origin on the base (revolute)
    wb = -m.base_mass * m.gravity
    f = w[:, :3] + wb
    n = w[:, 3:] + np.cross(p0, w[:, :3]) + np.cross(m.base_com, wb)
    s = m.frame("base_link").support_wrench(None, q, qd, qdd).cpu().numpy()
    _close_wrench(np.concatenate((f, n), axis=1), s, 1e-12)


def _golden_setup(g, robot):
    from toppra_b200.constraint import JointWrenchConstraint
    m = model_of(*{"arm6": ("arm6.urdf", None), "arm7": ("arm7_gripper.urdf",
                                                         {"finger_left_joint": 0.013, "finger_right_joint": 0.021})}[robot])
    link, xyz, rpy = str(g[robot + "/link"]), g[robot + "/xyz"], g[robot + "/rpy"]
    loc = m.frame(link, xyz=xyz, rpy=rpy, reference_frame="local")
    box = m.frame(link, xyz=xyz, rpy=rpy, reference_frame=str(g[robot + "/ref"]))

    def cons(form, scheme=1, wlim=None):
        if form == "box":
            return JointWrenchConstraint(box, g[robot + "/wlim"] if wlim is None else wlim,
                                         components=tuple(g["box_components"]), discretization_scheme=scheme)
        return JointWrenchConstraint.bearing(loc, axial=float(g[robot + "/axial"]), radial=float(g[robot + "/radial"]),
                                             tilting=float(g[robot + "/tilting"]), sides=int(g["sides"]),
                                             discretization_scheme=scheme)
    return m, loc, box, cons


def _joint_cons(ta, vlim, alim, scheme=1):
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme)]


@pytest.mark.gpu
@pytest.mark.parametrize("robot", ["arm6", "arm7"])
def test_gpu_reference_golden(ta, golden, robot):
    g = golden("joint_wrench")
    m, loc, box, cons = _golden_setup(g, robot)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim = (g[robot + "/" + k] for k in ("way", "vlim", "alim"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    d = _dev(grid)
    x = [path.eval_device(d, o).reshape(-1, m.nv) for o in (0, 1, 2)]
    for f, key in ((loc, "local"), (m.frame(loc.name, xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"]), "world")):
        terms = [t.reshape(B, len(grid), 6).cpu().numpy() for t in f.joint_wrench_terms(*x)]
        for i in range(B):                                       # against the 50-digit wrenches
            for t, k in zip(terms, "abc"):
                _close_wrench(t[i], g["%s/%s/%s" % (robot, key, k)][i], 1e-12)
    statuses = set()
    for form in ("box", "bearing"):
        for scheme in (0, 1):
            key = lambda x, i: g["%s/%s/s%d/%s" % (robot, form, scheme, x)][i]  # noqa: E731
            for i in range(B):                                   # single-path TOPPRA takes the device route too
                one = ta.algorithm.TOPPRA(_joint_cons(ta, vlim[i], alim[i], scheme) + [cons(form, scheme)],
                                          ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
                sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
                st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
                _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
            h = ta.BatchTOPPRA(_joint_cons(ta, vlim, alim, scheme) + [cons(form, scheme)], path,
                               grid).compute_parameterization(0, 0).to_host()
            for i in range(B):
                _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))
                statuses.add(int(h["status"][i]))
    assert 0 in statuses and len(statuses) > 1                   # some paths solve, some fail


def _problems(g, robot, B, seed):
    rng = np.random.RandomState(seed)
    way0, vlim, alim = (g[robot + "/" + k] for k in ("way", "vlim", "alim"))
    way = way0[rng.randint(0, way0.shape[0], B)] + rng.uniform(-0.1, 0.1, (B,) + way0.shape[1:])
    idx = rng.randint(0, way0.shape[0], B)
    return g["ss"], way, vlim[idx], alim[idx]


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta, golden):
    g = golden("joint_wrench")
    m, loc, box, cons = _golden_setup(g, "arm6")
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(g, "arm6", B, 71)
    path = ta.BatchSplineInterpolator(ss, way)
    per_path = np.stack([g["arm6/wlim"] * (1.0 + 0.05 * i) for i in range(B)])
    for form, mk in (("bearing", lambda s, sl=slice(None): cons("bearing", s)),
                     ("box", lambda s, sl=slice(None): cons("box", s, per_path[sl]))):
        # ragged (proposed per-path grids) against each path solved alone on its own grid
        rag = ta.BatchTOPPRA(_joint_cons(ta, vlim, alim) + [mk(1)], path, None)
        hr = rag.compute_parameterization(0, 0).to_host()
        glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
        assert len(set(glen.tolist())) > 1
        for i in range(B):
            n = int(glen[i])
            one = ta.BatchTOPPRA(_joint_cons(ta, vlim[i:i + 1], alim[i:i + 1]) + [mk(1, slice(i, i + 1))],
                                 ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n])
            one = one.compute_parameterization(0, 0).to_host()
            assert hr["status"][i] == one["status"][0]
            assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
        # chunked against unchunked on a common grid
        grid = np.linspace(0, 1, 150)
        for scheme in (0, 1):
            whole = ta.BatchTOPPRA(_joint_cons(ta, vlim, alim, scheme) + [mk(scheme)], path, grid)
            rec = 8 * ta.engine.record_doubles(whole.R) * whole.G
            parts = ta.BatchTOPPRA(_joint_cons(ta, vlim, alim, scheme) + [mk(scheme)], path, grid,
                                   max_record_bytes=5 * rec)
            assert parts.chunk_size() == 5
            hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
            for k in ("K", "sd", "sdd", "status"):
                assert _eq(hw[k], hp[k]), (form, k)
            assert (hw["status"] == 0).any()
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the reference-style SecondOrderConstraint with cons.wrench as a
    # numpy callback (F_mode 1 rows) equals the constraint's own rows
    grid = np.linspace(0, 1, 150)
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            for form in ("box", "bearing"):
                c = cons(form, scheme)
                one = ta.algorithm.TOPPRA(_joint_cons(ta, vlim[i], alim[i], scheme) + [c], sp, gridpoints=grid,
                                          solver_wrapper="seidel")
                sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
                hb = ta.BatchTOPPRA(_joint_cons(ta, vlim[i:i + 1], alim[i:i + 1], scheme) + [cons(form, scheme)],
                                    ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid)
                hb = hb.compute_parameterization(0, 0).to_host()
                if sd is None:                                   # a path that fails: NaN profiles in the batch
                    assert hb["status"][0] != 0 and np.isnan(hb["sd"][0]).all()
                else:
                    assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])
                if form == "bearing":
                    F, gg = c.F, c.g
                else:
                    E = np.eye(6)[list(c.components)]
                    F, gg = np.vstack((E, -E)), c._eye_form[0]
                ref_c = ta.constraint.SecondOrderConstraint(c.wrench, lambda _, F=F: F, lambda _, gg=gg: gg, nv,
                                                            discretization_scheme=scheme)
                runs = []
                for x in (ref_c, c):
                    inst = ta.algorithm.TOPPRA(_joint_cons(ta, vlim[i], alim[i], scheme) + [x], sp, gridpoints=grid,
                                               solver_wrapper="seidel")
                    runs.append(inst.compute_parameterization(0, 0, return_data=True))
                for x, y in zip(*runs):
                    assert (x is None and y is None) or _eq(x, y), (form, scheme)


def _oracle_rows_g(F, g, a, b, c):
    """(G, 3, R) collocation rows a F^T, b F^T, c F^T - g for the oracle."""
    return np.stack((a.dot(F.T), b.dot(F.T), c.dot(F.T) - g), axis=1)


@pytest.mark.gpu
def test_gpu_quintic_path_vs_oracle_and_toppra_sd(ta, golden):
    from oracle import oracle as orc
    g = golden("joint_wrench")
    m, loc, box, cons = _golden_setup(g, "arm6")
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(73)
    coeffs = rng.uniform(-0.6, 0.6, (B, k, nseg, nv))
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = m.velocity_limit
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    c = cons("bearing", 0)
    h = ta.BatchTOPPRA(_joint_cons(ta, vlim, alim, 0) + [c], path, grid).compute_parameterization(0, 0).to_host()
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    terms = [t.reshape(B, len(grid), 6).cpu().numpy() for t in
             loc.joint_wrench_terms(*(_dev(x.reshape(-1, nv)) for x in qs))]
    assert (h["status"] == 0).sum() >= B // 2
    for i in range(B):
        o = orc.solve_rows(np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]),
                                           _oracle_rows_g(c.F, c.g, terms[0][i], terms[1][i], terms[2][i])), axis=2),
                           orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
    # BatchTOPPRAsd, whole and in record chunks, at half again the time-optimal duration
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        inst = ta.BatchTOPPRAsd(_joint_cons(ta, vlim, alim, 0) + [cons("bearing", 0)], path, grid)
        if chunk:
            inst = ta.BatchTOPPRAsd(_joint_cons(ta, vlim, alim, 0) + [cons("bearing", 0)], path, grid,
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
        w = terms[0][i, :-1] * sdd[i][:, None] + terms[1][i, :-1] * (sd[i, :-1] ** 2)[:, None] + terms[2][i, :-1]
        assert (w @ c.F.T <= c.g + 1e-9 * np.abs(w).max()).all()
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        assert abs(got - min(1.5 * dur[i], slow[i])) <= 1e-4 * max(1.0, got)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["box", "bearing"])
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, golden, monkeypatch, form):
    g = golden("joint_wrench")
    m, loc, box, cons = _golden_setup(g, "arm7")
    ss, way, vlim, alim = _problems(g, "arm7", 10, 79)
    _assert_one_terms_launch(ta, monkeypatch, lambda: _joint_cons(ta, vlim, alim) + [cons(form)],
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_joint_wrench_terms")
