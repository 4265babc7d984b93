"""Speed and separation monitoring with capsules: robot links (segments between two frame origins) and human body parts
as capsules (RigidBodyModel.separation / separation_terms with packed capsules, SeparationMonitoringConstraint with
(frame_a, frame_b, radius) points or (H, 7) humans; libtoppra_b200_dyn.so: tbd_capsule_separation,
tbd_capsule_separation_terms).

CPU:
  * the independent 50-digit reference of tests/capsule_ref.py against the closed forms of the hand cases, its
    one-sided finite difference of the distance equal to -w (the parallel case included), and the float64 numpy double
    against the reference on every link capsule of both fixtures;
  * the header prototypes against _lib_dyn._PROTOS and the exported symbols; every refused call of the two entries,
    message for message; every Python ValueError; the launch plan on the recording libraries (one
    tbd_capsule_separation_terms launch per batch or chunk, while a problem of spheres only still records
    tbd_separation_terms).
GPU:
  * both kernels against the 50-digit reference on every link of both fixtures and on random trees of 1 to 16 bodies,
    and on the hand cases (bit-equal to the numpy double there); the terms bit-equal to tbd_capsule_separation plus the
    documented operations; degenerate capsules equal to the sphere entries; a sphere cover of a link never closer than
    its capsule; endpoint swaps; the reference golden (tests/golden/capsule_separation.npz); 256 paths with per-path
    human capsules, ragged, chunked, B = 1, shared-vs-per-path, BatchTOPPRAsd, a quintic path and torque limits alongside
    against the oracle; 1024 hypotheses of a person's pose; a profiler capture with both kernels."""
import ctypes
import os
import subprocess
import sys

import mpmath
import numpy as np
import pytest

import capsule_ref as cr
import rnea_ref as rr
import separation_ref as sr
from dyn_common import (CASES, DYN_LIB, LOCKED, TB_ERR_ARG, TB_ERR_UNSUPPORTED, FakePath, model_of, urdf,
                        _assert_solution, _dev, _dyn_header, _eq, _gpu_present, _model_from_packed, _oracle_rows,
                        _oracle_joint_rows, _problems)
from test_dyn_calls import H, T, _context, _run, _rows_call, arm, calls  # noqa: F401  (fixtures)

PARAMS = (0.1, 2.5, 1.6, 0.05)            # T_r, a_s, v_h, C
EYE = np.eye(3)


def _link_spec(m, radius=0.05):
    """One capsule per pair of consecutive frames of the model (every link and the tool), at most 16:
    [((link_a, xyz_a), (link_b, xyz_b), r)]."""
    names = list(m.frames)
    spec = [((names[k], (0.0, 0.0, 0.0)), (names[k + 1], (0.0, 0.0, 0.0)), radius + 0.01 * k)
            for k in range(len(names) - 1)]
    return spec[:16]


def _caps(m, spec):
    from toppra_b200.dynamics import pack_points
    return pack_points([(m.frame(a[0], xyz=a[1]), m.frame(b[0], xyz=b[1]), r) for a, b, r in spec])[1]


def _mp_spec(spec, packed=False):
    name = (lambda link: "b" + link[4:]) if packed else (lambda link: link)
    return [((name(a[0]), EYE, np.asarray(a[1], float)), (name(b[0]), EYE, np.asarray(b[1], float)), r)
            for a, b, r in spec]


def _human_capsules(rng, H, center=(0.4, 0.0, 0.5), spread=0.7):
    c0 = np.asarray(center) + rng.uniform(-spread, spread, (H, 3))
    c1 = c0 + rng.uniform(-0.4, 0.4, (H, 3))
    return np.concatenate((c0, c1, rng.uniform(0.0, 0.15, (H, 1))), axis=1)


def _check(d, w, pairs, tol=4e-15):
    dm = np.array([[float(p[0]) for p in row] for row in pairs])
    wm = np.array([[float(p[1]) for p in row] for row in pairs])
    sd, sw = max(1.0, np.abs(dm).max()), max(1.0, np.abs(wm).max())
    err = max(np.abs(d - dm).max() / sd, np.abs(w - wm).max() / sw)
    assert err <= tol, err
    return err


# ---- hand cases: a vertical link of one revolute body (axis y) against human capsules --------------------------------
def _pendulum(ta):
    """One revolute body about y at the origin: at q = 0, qd = 1 the point (0, 0, z) moves at (z, 0, 0)."""
    return ta.RigidBodyModel([-1], ["revolute"], [[0.0, 1.0, 0.0]], [np.eye(3)], [[0.0, 0.0, 0.0]], [1.0],
                             [[0.0, 0.0, 0.3]], [[0.01, 0.0, 0.0, 0.01, 0.0, 0.01]])


def _tilted(theta):
    """A human capsule from (0.375, 0, 0), 0.75 long, tilted by theta toward +x in the xz plane (coplanar)."""
    return [0.375, 0.0, 0.0, 0.375 + 0.75 * np.sin(theta), 0.0, 0.75 * np.cos(theta), 0.125]


# name, robot capsule (z_a, z_b) on the link, human capsule, the closed form (d, w) or None
HAND = [
    ("crossing", (0.125, 0.625), [0.375, -0.5, 0.375, 0.375, 0.5, 0.375, 0.125], (0.375 - 0.0625 - 0.125, 0.375)),
    ("end_to_end", (0.125, 0.625), [0.25, 0.0, 0.875, 0.75, 0.0, 1.25, 0.125], None),
    ("end_to_interior", (0.125, 0.625), [-0.5, 0.0, 0.875, 0.5, 0.0, 0.875, 0.125], (0.25 - 0.0625 - 0.125, 0.0)),
    ("parallel_overlap", (0.125, 0.625), [0.375, 0.0, 0.0, 0.375, 0.0, 0.75, 0.125],
     (0.375 - 0.0625 - 0.125, 0.625)),
    ("parallel_overlap_reversed", (0.625, 0.125), [0.375, 0.0, 0.75, 0.375, 0.0, 0.0, 0.125],
     (0.375 - 0.0625 - 0.125, 0.625)),
    ("parallel_apart", (0.125, 0.625), [0.375, 0.0, 1.0, 0.375, 0.0, 1.5, 0.125], None),
    ("angle_1e-5", (0.125, 0.625), _tilted(1e-5), None),
    ("angle_1e-7", (0.125, 0.625), _tilted(1e-7), None),
    ("robot_zero_length", (0.375, 0.375), [0.375, 0.0, 0.0, 0.375, 0.0, 0.75, 0.125], (0.375 - 0.0625 - 0.125, 0.375)),
    ("human_zero_length", (0.125, 0.625), [0.375, 0.0, 0.5, 0.375, 0.0, 0.5, 0.125], (0.375 - 0.0625 - 0.125, 0.5)),
    ("both_zero_length", (0.25, 0.25), [0.375, 0.0, 0.25, 0.375, 0.0, 0.25, 0.125], (0.375 - 0.0625 - 0.125, 0.25)),
    ("l_zero", (0.125, 0.625), [0.0, -0.5, 0.375, 0.0, 0.5, 0.375, 0.125], (0.0 - 0.0625 - 0.125, 0.375)),
]


def _hand_states(za, zb):
    """Endpoint states of the pendulum's capsule at q = 0, qd = 1."""
    return [0.0, 0.0, za], [za, 0.0, 0.0], [0.0, 0.0, zb], [zb, 0.0, 0.0]


def test_reference_hand_cases_and_finite_difference():
    for name, (za, zb), hc, closed in HAND:
        xa, va, xb, vb = _hand_states(za, zb)
        d, w = cr.mp_capsule_pair(xa, va, xb, vb, 0.0625, hc)
        if closed is not None:
            assert abs(float(d) - closed[0]) <= 1e-16 and abs(float(w) - closed[1]) <= 1e-16, name
        if name != "l_zero":                  # |E| is not differentiable at l == 0
            fd = cr.mp_fd_speed(xa, va, xb, vb, hc)
            with mpmath.workdps(cr.DPS):
                assert abs(fd - w) <= mpmath.mpf(10) ** -20, (name, fd, w)
        dn, wn = cr.capsule_pair_np(xa, va, xb, vb, 0.0625, hc)
        assert abs(dn - float(d)) <= 4e-16, name
        if name == "angle_1e-7":
            # under the parallel threshold the segments count as parallel: w is the larger of the two ends (the top,
            # 0.625), not the unique closest pair's (the bottom, 0.125), which the top overtakes within ~1e-7 s
            assert abs(wn - 0.625) <= 1e-14 and float(w) < 0.13, (wn, float(w))
        elif name == "angle_1e-5":
            assert abs(wn - float(w)) <= 4e-16 and abs(wn - 0.125) <= 1e-10, wn   # above it: the unique pair
        else:
            assert abs(wn - float(w)) <= 4e-16, (name, wn, float(w))
    # the parallel rule's w is the Danskin maximum, not an arbitrary member of the set
    xa, va, xb, vb = _hand_states(0.125, 0.625)
    assert cr.capsule_pair_np(xa, va, xb, vb, 0.0625, HAND[3][2])[1] == 0.625


@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 511)
    spec = _link_spec(m)
    caps = _caps(m, spec)
    q, qs = rng.uniform(-2, 2, m.nv), rng.uniform(-1.5, 1.5, m.nv)
    hum = _human_capsules(rng, 3)
    d, w = (x[0] for x in cr.capsule_separation_packed(m.packed, caps, hum, q, qs))
    _check(d, w, cr.mp_capsule_pairs(mp, q, qs, _mp_spec(spec), hum), tol=1e-13)


def test_pack_points_and_value_errors():
    from toppra_b200.constraint import SeparationMonitoringConstraint as SMC
    from toppra_b200.constraint.linear_constraint import RecordContext
    from toppra_b200.dynamics import CAPSULE_DOUBLES, POINT_DOUBLES, pack_points
    m = model_of("arm6.urdf")
    f, g = m.frame("flange", xyz=(0, 0, 0.1)), m.frame("forearm")
    _, sph = pack_points([(f, 0.05), (g, 0.06)])
    _, cap = pack_points([(f, 0.05), (g, f, 0.06)])
    assert sph.shape == (2, POINT_DOUBLES) and cap.shape == (2, CAPSULE_DOUBLES) and cap.flags.c_contiguous
    assert _eq(cap[0], np.r_[f.packed, f.packed, 0.05]) and _eq(cap[1], np.r_[g.packed, f.packed, 0.06])
    hum = np.array([[0.5, 0.0, 0.5, 0.5, 0.0, 1.0, 0.1]])
    for bad in ([(f, g)], [(f, g, 0.1, 0.2)], [(f, lambda q: q, 0.1)], [(f, g, (0.1, 0.2))], [(f, 0.1)] * 17):
        with pytest.raises(ValueError, match="points"):
            SMC(bad, hum, 0.1, 2.0)
    with pytest.raises(ValueError, match="same RigidBodyModel"):
        SMC([(f, model_of("arm6.urdf").frame("flange"), 0.1)], hum, 0.1, 2.0)
    for r in (-0.1, np.nan, np.inf):
        with pytest.raises(ValueError, match="radii"):
            SMC([(f, g, r)], hum, 0.1, 2.0)
    for h in (np.zeros(7), np.zeros((1, 5)), np.zeros((0, 7)), np.zeros((17, 7)), np.zeros((2, 1, 2, 7)),
              [[0, 0, 0, 0, 0, 0, -0.1]], [[0, np.inf, 0, 0, 0, 0, 0.1]]):
        with pytest.raises(ValueError, match="humans|human spheres and capsules"):
            SMC([(f, g, 0.05)], h, 0.1, 2.0)
    for kw in (dict(reaction_time=-0.1), dict(stopping_deceleration=0.0), dict(clearance=np.nan)):
        args = dict(reaction_time=0.1, stopping_deceleration=2.0)
        args.update(kw)
        with pytest.raises(ValueError, match=list(kw)[0]):
            SMC([(f, g, 0.05)], hum, **args)
    # a capsule on either side widens the other side to capsules of zero length
    c1 = SMC([(f, 0.05)], hum, 0.1, 2.0)
    assert c1.capsules and _eq(c1.points, np.r_[f.packed, f.packed, 0.05][None]) and _eq(c1.humans, hum)
    c2 = SMC([(f, g, 0.05)], hum[:, [0, 1, 2, 6]], 0.1, 2.0)
    assert c2.capsules and _eq(c2.humans, np.array([[0.5, 0.0, 0.5, 0.5, 0.0, 0.5, 0.1]]))
    c3 = SMC([(f, 0.05)], hum[:, [0, 1, 2, 6]], 0.1, 2.0)
    assert not c3.capsules and c3.points.shape == (1, POINT_DOUBLES) and c3.humans.shape == (1, 4)
    grid = np.linspace(0, 1, 10)
    assert c1.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    per_path = SMC([(f, g, 0.05)], np.tile(hum, (3, 1, 1)), 0.1, 2.0, discretization_scheme=1)
    assert per_path.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 2
    with pytest.raises(ValueError, match=r"expected \(H, 7\) or \(4, H, 7\)"):
        per_path.num_rows(RecordContext(FakePath(4, 6), grid, grid))
    with pytest.raises(ValueError, match="single path"):
        per_path.compute_constraint_params(type("P", (), {"dof": 6})(), grid)


def test_dyn_header_prototypes_and_symbols_of_capsule_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_capsule_separation"] == declared["tbd_separation"]
    assert declared["tbd_capsule_separation_terms"] == declared["tbd_separation_terms"]
    assert set(declared) == set(_lib_dyn._PROTOS)
    for name in ("tbd_capsule_separation", "tbd_capsule_separation_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int
        assert name in _lib_dyn.exported_symbols()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "toppra_b200_dyn.h")).read()
    assert "#define TBD_CAPSULE_DOUBLES (2 * TBD_FRAME_DOUBLES + 1)" in text
    assert "#define TBD_HUMAN_CAPSULE_DOUBLES 7" in text
    assert "#define TBD_CAPSULE_PARALLEL %r" % cr.PARALLEL in text
    if os.path.exists(DYN_LIB):
        lib = _lib_dyn.load()
        for name in ("tbd_capsule_separation", "tbd_capsule_separation_terms"):
            assert getattr(lib, name).argtypes == _lib_dyn._PROTOS[name][0]


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_capsule_argument_checks_message_for_message():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good = _caps(m, [(("flange", (0.0, 0.0, 0.1)), ("wrist2", (0.0, 0.0, 0.0)), 0.05),
                     (("forearm", (0.0, 0.0, 0.0)), ("upper_arm", (0.0, 0.0, 0.0)), 0.06)])
    sph = np.ascontiguousarray(np.concatenate((good[:, :14], good[:, 28:]), axis=1))

    def call(entry, model, points, nv, P, H, NH, ppp, M, params, null):
        host = [np.ascontiguousarray(x, dtype=np.float64) for x in (model, points)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        if entry.endswith("_terms"):
            args = [ptr[0], nv, ptr[1], P, H, NH, ppp, *params, M, d, d, d, d, d]
        else:
            args = [ptr[0], nv, ptr[1], P, H, NH, ppp, M, d, d, d, d, d]
        if null is not None:
            args[null] = None
        rc = getattr(lib, entry)(*args, None)
        msg = _lib.load().tb_last_error().decode()
        return rc, msg.split(": ", 1)[1] if ": " in msg else msg

    def both(model=m.packed, caps=good, nv=6, P=2, H=3, NH=1, ppp=0, M=4, params=PARAMS, null=None, terms=(0, 1)):
        """(rc, message) of the capsule entries, each equal to the sphere entry's with the nouns swapped."""
        out = set()
        for t in terms:
            entry = ("tbd_separation", "tbd_separation_terms")[t]
            n = null if null is None or t == 0 or null < 7 else null + 4
            rc_c, msg_c = call("tbd_capsule" + entry[3:], model, caps, nv, P, H, NH, ppp, M, params, n)
            spheres = sph if caps is good else np.zeros((max(P, 1), 15))
            rc_s, msg_s = call(entry, model, spheres, nv, P, H, NH, ppp, M, params, n)
            assert rc_c == rc_s, (entry, rc_c, rc_s, msg_c, msg_s)
            if rc_c in (TB_ERR_ARG, TB_ERR_UNSUPPORTED):
                want = msg_s.replace("human spheres", "human capsules").replace("human-sphere", "human-capsule")
                want = want.replace(" points outside", " capsules outside")
                assert msg_c == want, (msg_c, want)
            out.add(rc_c)
        assert len(out) == 1
        return out.pop()

    for k in (0, 2, 8, 9, 10, 11, 12):
        assert both(null=k, terms=(0,)) == TB_ERR_ARG
    for k in (0, 2, 8, 9, 10, 11, 12):                         # + 4 in the terms entries (the four scalars)
        assert both(null=k, terms=(1,)) == TB_ERR_ARG
    assert both(M=0) == TB_ERR_ARG and both(M=-3) == TB_ERR_ARG
    assert both(nv=0) == TB_ERR_UNSUPPORTED
    for P in (0, 17):
        assert both(caps=np.zeros((max(P, 1), 29)), P=P) == TB_ERR_UNSUPPORTED
    for H_ in (0, 17):
        assert both(H=H_) == TB_ERR_UNSUPPORTED
    assert both(NH=0) == TB_ERR_ARG and both(ppp=-1) == TB_ERR_ARG
    assert both(ppp=2, NH=1) == TB_ERR_ARG and both(ppp=3, NH=1) == TB_ERR_ARG
    assert both(ppp=2, NH=2) not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED)       # passes validation, no device here
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0
    assert both(bad_model) == TB_ERR_ARG
    for params in ((-0.1, 2.5, 1.6, 0.0), (0.1, 0.0, 1.6, 0.0), (0.1, 2.5, np.nan, 0.0), (0.1, 2.5, 1.6, np.inf)):
        assert both(params=params, terms=(1,)) == TB_ERR_ARG
    # bad frames (frame a, then frame b) and radii, in either capsule, each refused with the message of its check
    for j, value, what in ((0, 6.0, "body"), (0, 0.5, "body"), (5, np.nan, "finite"), (14, 6.0, "body"),
                           (14 + 11, np.inf, "finite"), (28, -0.1, "capsule 0: radius"),
                           (28, np.nan, "capsule 0: radius"), (29 + 28, np.inf, "capsule 1: radius"),
                           (29 + 14, 9.0, "body")):
        p = good.copy().reshape(-1)
        p[j] = value
        for entry, args in (("tbd_capsule_separation", (0,)), ("tbd_capsule_separation_terms", (1,))):
            rc, msg = call(entry, m.packed, p, 6, 2, 3, 1, 0, 4, PARAMS, None)
            assert rc == TB_ERR_ARG and (what in msg or what == "body"), (j, msg)


@pytest.mark.parametrize("lo,hi,total", [(0, 4, 4), (1, 3, 4)])
@pytest.mark.parametrize("interp", [False, True])
@pytest.mark.parametrize("kind", ["robot", "human", "both", "spheres"])
def test_launch_plan(calls, arm, monkeypatch, lo, hi, total, interp, kind):  # noqa: F811
    import test_dyn_calls
    from toppra_b200.constraint import SeparationMonitoringConstraint
    nv, G = arm.nv, 6
    f = arm.frame(sorted(arm.frames)[-1], xyz=(0.0, 0.0, 0.1))
    g = arm.frame("forearm")
    rng = np.random.RandomState(3)
    hum7 = np.stack([_human_capsules(rng, 3) + 0.1 * i for i in range(total)])
    hum4 = hum7[..., [0, 1, 2, 6]]
    points = [(f, g, 0.05), (g, 0.08)] if kind in ("robot", "both") else [(f, 0.05), (g, 0.08)]
    hum = hum7 if kind in ("human", "both") else hum4
    cons = SeparationMonitoringConstraint(points, hum, *PARAMS, discretization_scheme=int(interp))
    name = "tbd_separation_terms" if kind == "spheres" else "tbd_capsule_separation_terms"
    monkeypatch.setitem(test_dyn_calls._OUTPUTS, name, 2)
    ctx, bp = _context(nv, total, G, lo, hi, total)
    B, n = hi - lo, (hi - lo) * G
    rows, log = _run(calls, cons, ctx)
    assert rows == (2 if interp else 1)
    sets = cons.humans[lo:hi]
    assert sets.shape[-1] == (4 if kind == "spheres" else 7)
    if kind == "human":
        assert _eq(cons.points, np.concatenate((np.stack([f.packed, g.packed]),) * 2 + (np.array([[0.05], [0.08]]),),
                                               axis=1))
    if kind == "robot":
        assert _eq(sets, np.concatenate((hum4[lo:hi, :, :3], hum4[lo:hi]), axis=2))
    want = [
        [name, H(arm.packed), nv, H(cons.points.reshape(-1)[:14]), 2, 3, sets.shape[0], G, *PARAMS,
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
def test_gpu_vs_mp_every_link_and_random_trees(ta):
    worst = 0.0
    cases = [(_model_from_packed(ta, rr.random_tree(np.random.RandomState(1700 + nv), nv)), None)
             for nv in (1, 2, 3, 5, 8, 12, 16)]
    cases += [(model_of(n, lk), rr.MpRobot.from_urdf(urdf(n), lk)) for n, lk in CASES]
    for m, mp in cases:
        packed = mp is None
        mp = mp or rr.MpRobot.from_packed(m.packed)
        rng = np.random.RandomState(m.nv + 91)
        spec = _link_spec(m)
        if packed:        # frames on bodies and offsets off them: segments across joints and within one body
            names = list(m.frames)
            spec = [((names[k], tuple(rng.uniform(-0.2, 0.2, 3))), (names[rng.randint(len(names))],
                     tuple(rng.uniform(-0.2, 0.2, 3))), 0.03 * k) for k in range(min(len(names), 16))]
        caps = _caps(m, spec)
        hum = _human_capsules(rng, 5)
        q, qs = rng.uniform(-2, 2, (2, m.nv)), rng.uniform(-1.5, 1.5, (2, m.nv))
        d, w = _sep_dev(m, caps, hum, q, qs)
        b, c = _terms_dev(m, caps, hum, PARAMS, q, qs)
        for i in range(2):
            pairs = cr.mp_capsule_pairs(mp, q[i], qs[i], _mp_spec(spec, packed), hum)
            worst = max(worst, _check(d[i], w[i], pairs, tol=1e-13))
            bm, cm = sr.mp_row([p for row in pairs for p in row], PARAMS)
            assert abs(b[i] - float(bm)) <= 1e-12 * max(1.0, abs(float(bm)))
            assert abs(c[i] - float(cm)) <= 1e-12 * max(1.0, abs(float(cm)))
        Q, QS = rng.uniform(-3, 3, (64, m.nv)), rng.uniform(-2, 2, (64, m.nv))
        d, w = _sep_dev(m, caps, hum, Q, QS)
        dn, wn = cr.capsule_separation_packed(m.packed, caps, hum, Q, QS)
        assert np.max(np.abs(d - dn)) <= 1e-12 and np.max(np.abs(w - wn)) <= 1e-12 * max(1.0, np.abs(wn).max())
    print("capsule kernels vs the 50-digit reference: worst scaled error %.2e" % worst)


@pytest.mark.gpu
def test_gpu_hand_cases(ta):
    m = _pendulum(ta)
    for name, (za, zb), hc, closed in HAND:
        caps = _caps(m, [(("body0", (0.0, 0.0, za)), ("body0", (0.0, 0.0, zb)), 0.0625)])
        hum = np.array([hc])
        d, w = _sep_dev(m, caps, hum, np.zeros((1, 1)), np.ones((1, 1)))
        b, c = _terms_dev(m, caps, hum, PARAMS, np.zeros((1, 1)), np.ones((1, 1)))
        xa, va, xb, vb = _hand_states(za, zb)
        dn, wn = cr.capsule_pair_np(xa, va, xb, vb, 0.0625, hc)
        assert d[0, 0, 0] == dn and w[0, 0, 0] == wn, (name, d, w, dn, wn)
        bn, cn = sr.rows_from_pairs(np.array([[[dn]]]), np.array([[[wn]]]), PARAMS)
        assert _eq(b, bn) and _eq(c, cn), name
        dm, wm = cr.mp_capsule_pair(xa, va, xb, vb, 0.0625, hc)
        assert abs(d[0, 0, 0] - float(dm)) <= 4e-16, name
        if name != "angle_1e-7":
            assert abs(w[0, 0, 0] - float(wm)) <= 4e-16, name
        else:
            assert w[0, 0, 0] > float(wm)            # the parallel rule is conservative
        if closed is not None:
            assert abs(d[0, 0, 0] - closed[0]) <= 1e-16 and abs(w[0, 0, 0] - closed[1]) <= 1e-16, name


def _torch_terms(d, w, params):
    from test_separation_monitoring import _torch_terms as tt
    return tt(d, w, params)


@pytest.mark.gpu
def test_gpu_terms_bit_equal_degenerate_cover_and_swaps(ta):
    import torch
    from toppra_b200.dynamics import pack_points
    m = model_of("arm7_gripper.urdf")
    rng = np.random.RandomState(12)
    M = 2000
    spec = _link_spec(m)
    caps = _caps(m, spec)
    q, qs = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(2))
    hum = _dev(np.stack([_human_capsules(rng, 5, spread=0.5) for _ in range(M // 100)]))
    for params in (PARAMS, (0.0, 3.0, 0.0, 0.0), (0.5, 40.0, 2.0, 0.3)):
        for ppp, h in ((0, hum[0]), (100, hum)):
            d, w = m.separation(caps, h, q, qs, ppp)
            b, c = m.separation_terms(caps, h, *params, q, qs, ppp)
            want = _torch_terms(d, w, params)
            assert torch.equal(b, want[0]) and torch.equal(c, want[1])
            assert (b > 0).any()
    # degenerate capsules give the sphere entries' numbers
    frames = [(m.frame(a[0], xyz=a[1]), r) for a, _, r in spec]
    sph = pack_points(frames)[1]
    hs = _dev(np.stack([_human_capsules(rng, 4)[:, [0, 1, 2, 6]] for _ in range(M // 100)]))
    d0, w0 = m.separation(sph, hs, q, qs, 100)
    b0, c0 = m.separation_terms(sph, hs, *PARAMS, q, qs, 100)
    from toppra_b200.dynamics import _launch, sphere_humans_as_capsules, sphere_points_as_capsules
    P, H_ = sph.shape[0], hs.shape[1]
    dc, wc = _launch(m, "tbd_capsule_separation", (sphere_points_as_capsules(sph), P, H_, hs.shape[0], 100), (q, qs),
                     [(P, H_)] * 2, extra=(sphere_humans_as_capsules(hs),))
    bc, cc = _launch(m, "tbd_capsule_separation_terms",
                     (sphere_points_as_capsules(sph), P, H_, hs.shape[0], 100, *PARAMS), (q, qs), [(), ()],
                     extra=(sphere_humans_as_capsules(hs),))
    for x, y in ((d0, dc), (w0, wc), (b0, bc), (c0, cc)):
        assert np.array_equal(x.cpu().numpy(), y.cpu().numpy())
    # a sphere cover of a link lies inside the capsule of the same radius: the capsule is never farther, and the
    # nearest sphere approaches it as the spacing shrinks (nested covers, so the gap never grows)
    mm = model_of("arm6.urdf")
    Q, QS = (_dev(rng.uniform(-2, 2, (512, 6))) for _ in range(2))
    hum1 = _dev(_human_capsules(rng, 3, center=(0.3, 0.0, 0.6), spread=0.4))
    r_b = mm.packed[3 + 27 * 3 + 14: 3 + 27 * 3 + 17]       # wrist1's joint origin in forearm coordinates
    capsule = _caps(mm, [(("forearm", (0.0, 0.0, 0.0)), ("forearm", tuple(r_b)), 0.06)])
    dcap = mm.separation(capsule, hum1, Q, QS)[0][:, 0, :]
    across = _caps(mm, [(("forearm", (0.0, 0.0, 0.0)), ("wrist1", (0.0, 0.0, 0.0)), 0.06)])
    assert torch.allclose(mm.separation(across, hum1, Q, QS)[0][:, 0, :], dcap, rtol=0, atol=1e-15)
    gaps = []
    for n in (2, 5, 17, 65):
        ts = np.linspace(0, 1, n)
        ds = torch.cat([mm.separation(pack_points([(mm.frame("forearm", xyz=tuple(t * r_b)), 0.06)
                                                   for t in ts[i:i + 16]])[1], hum1, Q, QS)[0]
                        for i in range(0, n, 16)], dim=1)
        dmin = ds.min(dim=1).values
        assert (dcap <= dmin + 1e-15).all()
        gaps.append(float((dmin - dcap).max()))
        assert gaps[-1] <= 0.5 * np.linalg.norm(r_b) / (n - 1) + 1e-15, (n, gaps)
    assert gaps == sorted(gaps, reverse=True), gaps
    # swapping a capsule's endpoints, or a human capsule's, leaves d and w unchanged to rounding
    swapped = _caps(m, [(b, a, r) for a, b, r in spec])
    hsw = hum[:, :, [3, 4, 5, 0, 1, 2, 6]].contiguous()
    d, w = m.separation(caps, hum, q, qs, 100)
    radii = torch.as_tensor(caps[:, 28], device="cuda")
    l = d + radii[None, :, None] + hum[:, :, 6].repeat_interleave(100, dim=0)[:, None, :]
    # E = h - p cancels where the pair is close: its direction, so w, carries rounding of order |x| / l
    tol_w = 1e-14 * (1 + w.abs().max()) * (1 + 1 / l)
    for cp, hh in ((swapped, hum), (caps, hsw), (swapped, hsw)):
        d2, w2 = m.separation(cp, hh, q, qs, 100)
        assert torch.allclose(d2, d, rtol=0, atol=1e-14)
        assert ((w2 - w).abs() <= tol_w).all(), float(((w2 - w).abs() / tol_w).max())


def _cons(ta, points, humans, vlim, alim, scheme=0, joint_scheme=None, params=PARAMS):
    joint_scheme = scheme if joint_scheme is None else joint_scheme
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=joint_scheme),
            ta.constraint.SeparationMonitoringConstraint(points, humans, *params, discretization_scheme=scheme)]


def _golden_capsules(g, robot, m):
    return [(m.frame(str(a), xyz=xa), m.frame(str(b), xyz=xb), float(r))
            for a, xa, b, xb, r in zip(g[robot + "/link_a"], g[robot + "/xyz_a"], g[robot + "/link_b"],
                                       g[robot + "/xyz_b"], g[robot + "/radii"])]


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    from toppra_b200.dynamics import pack_points
    g = golden("capsule_separation")
    m = model_of(name, locked)
    points = _golden_capsules(g, robot, m)
    caps = pack_points(points)[1]
    ss, grid, params = g["ss"], g["grid"], tuple(g["params"])
    way, vlim, alim, hum = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "humans"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    d_grid = _dev(grid)
    q, qs = (path.eval_device(d_grid, o).reshape(-1, m.nv) for o in (0, 1))
    b, c = (x.reshape(B, -1).cpu().numpy() for x in m.separation_terms(caps, _dev(hum), *params, q, qs, len(grid)))
    assert np.array_equal(b == 0, g[robot + "/b"] == 0)
    np.testing.assert_allclose(b, g[robot + "/b"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(c, g[robot + "/c"], rtol=1e-12, atol=1e-14)
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


def _arm6_capsules(m):
    return [(m.frame("upper_arm"), m.frame("forearm"), 0.07), (m.frame("forearm"), m.frame("wrist1"), 0.06),
            (m.frame("wrist2"), m.frame("flange", xyz=(0, 0, 0.1)), 0.05)]


def _torsos_ahead(ta, m, path, grid, rng):
    """(B, 2, 7): per path, a vertical torso 0.5 m long, 0.85 m off the tool's motion ahead of a mid-path gridpoint,
    and an arm reaching 0.25 m toward it."""
    import kin_ref as kr
    f = m.frame("flange", xyz=(0, 0, 0.1))
    B = path.B
    q, qs = (path.eval_device(_dev(grid), o).reshape(-1, m.nv).cpu().numpy() for o in (0, 1))
    _, x, v = kr.frame_packed(m.packed, f.packed, q, qs)
    x, v = x.reshape(B, len(grid), 3), v[:, :3].reshape(B, len(grid), 3)
    out = []
    for i in range(B):
        g0 = int(rng.randint(len(grid) // 3, 2 * len(grid) // 3))
        u = v[i, g0] / max(np.linalg.norm(v[i, g0]), 1e-9)
        n = np.cross(u, rng.randn(3))
        n /= np.linalg.norm(n)
        base = x[i, g0] + 0.4 * u + 0.85 * n
        torso = np.r_[base - [0, 0, 0.25], base + [0, 0, 0.25], 0.12]
        arm_ = np.r_[base + [0, 0, 0.2], base + [0, 0, 0.2] - 0.25 * n, 0.05]
        out.append([torso, arm_])
    return np.array(out)


def _sep_rows(b, c, grid, interp):
    G = len(grid)
    return _oracle_rows(np.ones((1, 1)), np.zeros((G, 1)), b.reshape(G, 1), c.reshape(G, 1), grid, interp)


@pytest.mark.gpu
def test_gpu_256_paths_per_path_human_capsules_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    points = _arm6_capsules(m)
    B, G = 256, 200
    ss, way, vlim, alim = _problems(B, 6, 63, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    hum = _torsos_ahead(ta, m, path, grid, np.random.RandomState(5))
    cons = _cons(ta, points, hum, vlim, alim, 0, 1)
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    caps = cons[2].points
    n_ok = n_active = n_stop = 0
    for i in range(0, B, 4):          # every fourth path against the oracle (the numpy double is a Python loop)
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1))
        b, cc = cr.capsule_rows_packed(m.packed, caps, hum[i], PARAMS, q, qs)
        if ((b > 0) & (cc == 0)).any():
            # a link approaches inside the clearance: x = 0 there, and whether the profile can still reach that
            # stop depends on the last bits of the neighbouring rows; only the outcome class is pinned
            n_stop += 1
            assert h["status"][i] in (0, 3)
            continue
        o = orc.solve_rows(np.concatenate((lin["rows"], _sep_rows(b, cc, grid, False)), axis=2), lin["xbound"], grid,
                           0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            n_active += bool(((b > 0) & (b * h["sd"][i] ** 2 >= -cc * (1 - 1e-6))).any())
    print("capsule limit active on %d of %d solved paths; %d paths stop next to the person" % (n_active, n_ok, n_stop))
    compared = B // 4 - n_stop
    assert compared >= B // 8 and n_ok > 0.8 * compared and n_active > 0.3 * n_ok, (n_ok, n_active, n_stop)


@pytest.mark.gpu
def test_gpu_ragged_chunked_single_and_shared_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    points = [(m.frame("link4"), m.frame("hand", xyz=(0.02, 0.0, 0.12)), 0.06), (m.frame("link3"), 0.07)]
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, nv, 39, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    rng = np.random.RandomState(9)
    hum = np.stack([_human_capsules(rng, 3, center=(1.0, 0.0, 0.8), spread=0.3) for _ in range(B)])
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
        # shared humans == per-path copies
        shared = ta.BatchTOPPRA(_cons(ta, points, hum[0], vlim, alim, scheme), path, grid)
        copies = ta.BatchTOPPRA(_cons(ta, points, np.repeat(hum[:1], B, 0), vlim, alim, scheme), path, grid)
        hs, hc = shared.compute_parameterization(0, 0).to_host(), copies.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hs[k], hc[k]), k
        for i in range(3):
            sp = ta.SplineInterpolator(ss, way[i])
            for hi in (hum[i], hum[i:i + 1]):       # a single path == path i of the batch == a batch of one
                one = ta.algorithm.TOPPRA(_cons(ta, points, hi, vlim[i], alim[i], scheme), sp, gridpoints=grid,
                                          solver_wrapper="seidel")
                run = one.compute_parameterization(0, 0, return_data=True)
                assert _eq(run[3], hw["K"][i])
                if hw["status"][i] == 0:
                    assert _eq(run[1], hw["sd"][i]) and _eq(run[0], hw["sdd"][i])
            b1 = ta.BatchTOPPRA(_cons(ta, points, hum[i:i + 1], vlim[i:i + 1], alim[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0)
            b1 = b1.to_host()
            for k in ("K", "sd", "status"):
                assert _eq(b1[k][0], hw[k][i]), k


@pytest.mark.gpu
def test_gpu_toppra_sd_quintic_and_torque_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    points = _arm6_capsules(m)
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(43)
    path = ta.BatchPiecewisePolyPath(np.linspace(0, 1, nseg + 1), rng.uniform(-0.4, 0.4, (B, k, nseg, nv)))
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    hum = _torsos_ahead(ta, m, path, grid, rng)
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    Fj = np.vstack((np.eye(nv), -np.eye(nv)))
    for extra in (False, True):
        cons = _cons(ta, points, hum, vlim, alim)
        if extra:
            cons += [ta.constraint.JointTorqueConstraint(m, taulim, fric)]
        h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
        assert (h["status"] == 0).sum() >= B // 2
        for i in range(B):
            b, c = cr.capsule_rows_packed(m.packed, cons[2].points, hum[i], PARAMS, qs[0][i], qs[1][i])
            rows = [_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]), _sep_rows(b, c, grid, False)]
            if extra:
                av, bt, cv = rr.torque_terms_packed(m.packed, qs[0][i], qs[1][i], qs[2][i], fric)
                gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
                rows.append(np.stack((av.dot(Fj.T), bt.dot(Fj.T), cv.dot(Fj.T) - gt), axis=1))
            o = orc.solve_rows(np.concatenate(rows, axis=2), orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
            _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
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
    caps = _cons(ta, points, hum, vlim, alim)[2].points
    for i in np.flatnonzero(ok):
        b, c = cr.capsule_rows_packed(m.packed, caps, hum[i], PARAMS, qs[0][i], qs[1][i])
        assert (b * sd[i] ** 2 + c <= 1e-9).all()


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch):
    from dyn_common import _assert_one_terms_launch
    m = model_of("arm6.urdf")
    ss, way, vlim, alim = _problems(10, 6, 49, m.velocity_limit)
    hum = np.stack([_human_capsules(np.random.RandomState(i), 2) for i in range(10)])
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, _arm6_capsules(m), hum, vlim, alim),
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_capsule_separation_terms")


_PROFILE = """
import sys
import numpy as np
from test_piecewise_poly import launched
from test_capsule_separation import PARAMS, _arm6_capsules, _human_capsules
from dyn_common import _dev, model_of
from toppra_b200.dynamics import pack_points
m = model_of("arm6.urdf")
caps = pack_points(_arm6_capsules(m))[1]
hum = _dev(_human_capsules(np.random.RandomState(1), 2))
q = _dev(np.random.RandomState(1).uniform(-1, 1, (300, 6)))
want = {"capsule_separation_kernel", "capsule_separation_terms_kernel"}
names = set()
for _ in range(3):
    with launched() as got:
        m.separation(caps, hum, q, q)
        m.separation_terms(caps, hum, *PARAMS, q, q)
    names |= got
    if want <= names:          # kineto now and then returns a capture without device activity
        break
print(sorted(names))
sys.exit(0 if want <= names else 1)
"""


@pytest.mark.gpu
def test_gpu_profiler_capture_shows_both_kernels():
    """torch.profiler sees both capsule kernels run.  The capture runs in a process of its own, so that no profiler
    state is left behind in the test process for the kernel-inventory tests that profile later."""
    tests = os.path.dirname(os.path.abspath(__file__))
    paths = [os.path.dirname(tests), tests] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(paths))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _PROFILE]
    out = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr[-2000:]


@pytest.mark.gpu
def test_gpu_1024_human_pose_hypotheses_along_a_ray(ta):
    """One path, 1024 hypotheses of where a person (torso and arm capsules) stands, along a ray away from the tool's
    mid-path position: the time-optimal duration never grows as the person moves away."""
    import kin_ref as kr
    m = model_of("arm6.urdf")
    points = _arm6_capsules(m)
    ss, way, vlim, alim = _problems(1, 6, 73, m.velocity_limit)
    B, G = 1024, 150
    grid = np.linspace(0, 1, G)
    one = ta.BatchSplineInterpolator(ss, way)
    hum0 = _torsos_ahead(ta, m, one, grid, np.random.RandomState(2))[0]
    f = m.frame("flange", xyz=(0, 0, 0.1))
    x = kr.frame_packed(m.packed, f.packed, one.eval_device(_dev(grid), 0).reshape(-1, 6).cpu().numpy(),
                        np.zeros((G, 6)))[1]
    mid = 0.5 * (hum0[0, :3] + hum0[0, 3:6])
    ray = mid - x[G // 2]
    ray /= np.linalg.norm(ray)
    shift = (x[G // 2] + np.linspace(0.0, 3.0, B)[:, None] * ray) - mid
    hum = np.repeat(hum0[None], B, axis=0)
    for j in (0, 3):
        hum[:, :, j:j + 3] += shift[:, None, :]
    path = ta.BatchSplineInterpolator(ss, np.repeat(way, B, axis=0))
    h = ta.BatchTOPPRA(_cons(ta, points, hum, np.repeat(vlim, B, 0), np.repeat(alim, B, 0)), path, grid)
    h = h.compute_parameterization(0, 0).to_host()
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else np.inf for s, o in zip(h["sd"], ok)])
    first = int(np.flatnonzero(~ok).max()) + 1 if (~ok).any() else 0
    assert B - first > B // 2, first
    d = dur[first:]
    assert (np.diff(d) <= 1e-9 * d[1:]).all(), np.max(np.diff(d) / d[1:])
    assert d[0] > 1.05 * d[-1]
    print("durations: %.3f s near the path to %.3f s at 3 m (%d of %d poses solve)" % (d[0], d[-1], ok.sum(), B))
