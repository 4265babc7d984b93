"""Torque and speed limits of geared robots on the motor side (toppra_b200.Drives, MotorTorqueConstraint,
MotorSpeedConstraint; libtoppra_b200_dyn.so: tbd_drive_torque, tbd_drive_torque_terms, tbd_drive_speed_terms).

CPU:
  * the float64 numpy doubles of tests/drive_ref.py equal the 50-digit reference (rnea_ref.MpRobot on the RAW URDF tree,
    T^-1 in mpmath) on both fixtures, locked and unlocked, with a coupled transmission: to 1e-13 of the scale;
  * every refused call of the three entries on the real library, message for message; the ctypes prototypes against
    include/toppra_b200_dyn.h; every ValueError of the Python layer.
GPU:
  * tbd_drive_torque on random trees of 1 to 16 bodies (random T of condition number <= 100, random I_r) against the
    50-digit reference, to 1e-12 of the scale;
  * tbd_drive_torque_terms is three tbd_drive_torque launches plus the torch operations (torch.equal); with T = I,
    I_r = 0 and the joint friction it is tbd_torque_terms (torch.equal); a diagonal T is (tau + n^2 I_r qdd) / n;
  * tbd_drive_speed_terms equals the numpy restatement bit for bit, and NaN in q' gives NaN;
  * the reference golden (tests/golden/drive_limits.npz, make_golden_drives.py) through TOPPRA and BatchTOPPRA, and 256
    paths with per-path torque limits against the oracle fed with rows from the numpy double;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1: bit-equal; BatchTOPPRAsd and a
    quintic path against the oracle; one terms launch per batch or record chunk."""
import ctypes
import os

import numpy as np
import pytest

import drive_ref as dr
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, LOCKED, ROOT, TB_ERR_ARG, TB_ERR_UNSUPPORTED, FakePath, model_of, urdf,
                        _assert_solution, _dev, _dyn_header, _eq, _gpu_present, _model_from_packed, _oracle_joint_rows,
                        _oracle_rows, _problems)


def _transmission(rng, nv, cond=100.0):
    """A random T = U diag(s) V^T with singular values in [1, cond], times a gear-ratio scale."""
    U, _ = np.linalg.qr(rng.randn(nv, nv))
    V, _ = np.linalg.qr(rng.randn(nv, nv))
    s = np.exp(rng.uniform(0, np.log(cond), nv))
    s[0], s[-1] = 1.0, cond if nv > 1 else 1.0
    return rng.uniform(20, 120) * (U * s) @ V.T


def _coupled(nv):
    """Gear ratios with a coupled wrist on the last three motors (as in the golden's arm6)."""
    C = np.eye(nv)
    if nv >= 3:
        C[-2, -3], C[-1, -3], C[-1, -2] = 1.0, 0.5, -1.0
    return np.diag(np.linspace(120.0, 50.0, nv)) @ C


def _scale(x):
    return max(1.0, float(np.max(np.abs(np.asarray(x, dtype=np.float64)))))


# ==== CPU ============================================================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 500)
    packed = dr.pack(_coupled(m.nv), rng.uniform(1e-5, 5e-5, m.nv), 0.0)
    omega = rng.uniform(100, 400, m.nv)
    omega[1] = np.inf
    worst = 0.0
    for _ in range(2):
        q, qd, qdd = rng.uniform(-2, 2, m.nv), rng.uniform(-1.5, 1.5, m.nv), rng.uniform(-3, 3, m.nv)
        want = np.array([float(x) for x in dr.mp_torque(mp, packed, q, qd, qdd)])
        got = dr.torque_packed(m.packed, packed, q, qd, qdd)[0]
        err = np.max(np.abs(got - want)) / _scale(want)
        assert err <= 1e-13, err
        worst = max(worst, err)
        bm = float(dr.mp_speed_row(packed, m.nv, omega, qd))
        assert abs(dr.speed_terms_packed(packed, omega, qd)[0] - bm) <= 1e-13 * max(1.0, bm)
    print("worst scaled error of the numpy double: %.2e" % worst)


def test_dyn_header_prototypes_of_drive_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_drive_torque"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_drive_torque_terms"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr", "ptr",
                                                  "ptr"]
    assert declared["tbd_drive_speed_terms"] == ["int", "ptr", "ptr", "int", "ptr", "ptr", "ptr"]
    assert set(declared) == set(_lib_dyn._PROTOS)
    for name in ("tbd_drive_torque", "tbd_drive_torque_terms", "tbd_drive_speed_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    assert "#define TBD_DRIVE_DOUBLES(nv) ((nv) * (nv) + 2 * (nv))" in text
    assert "#define TBD_VERSION 100" in text


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_drive_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good = dr.pack(_coupled(6), 2e-5, 0.01)
    omega = np.full(6, 300.0)

    def err():
        return _lib.load().tb_last_error().decode()

    def rc(model=m.packed, drive=good, nv=6, M=4, om=omega, null=None, which="torque"):
        """(return code, tb_last_error()) of one call of entry `which` ("torque", "terms" or "speed")."""
        host = [np.ascontiguousarray(x, dtype=np.float64) for x in (model, drive, om)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        args = {"torque": [ptr[0], nv, ptr[1], M, d, d, d, d],
                "terms": [ptr[0], nv, ptr[1], M, d, d, d, d, d, d],
                "speed": [nv, ptr[1], ptr[2], M, d, d]}[which]
        if null is not None:
            args[null] = None
        entry = {"torque": lib.tbd_drive_torque, "terms": lib.tbd_drive_torque_terms,
                 "speed": lib.tbd_drive_speed_terms}[which]
        out = entry(*args, None)
        return out, (err() if out else "")

    for k in (0, 2, 4, 5, 6, 7):
        assert rc(null=k, which="torque") == (TB_ERR_ARG, "tbd_drive_torque: null pointer")
    for k in (0, 2, 4, 5, 6, 7, 8, 9):
        assert rc(null=k, which="terms") == (TB_ERR_ARG, "tbd_drive_torque_terms: null pointer")
    for k in (1, 2, 4, 5):
        assert rc(null=k, which="speed") == (TB_ERR_ARG, "tbd_drive_speed_terms: null pointer")
    assert rc(M=0, which="torque") == (TB_ERR_ARG, "tbd_drive_torque: M=0 must be positive")
    assert rc(M=-3, which="speed") == (TB_ERR_ARG, "tbd_drive_speed_terms: M=-3 must be positive")
    for nv in (0, 17):
        big = np.zeros(17 * 17 + 34)
        assert rc(nv=nv, drive=big, om=np.ones(17), which="speed") == (
            TB_ERR_UNSUPPORTED, "tbd_drive_speed_terms: nv=%d outside 1..16" % nv)
        assert rc(np.r_[m.packed, np.zeros(27 * 11)], nv=nv, drive=big, which="terms") == (
            TB_ERR_UNSUPPORTED, "tbd_drive_torque_terms: nv=%d outside 1..16" % nv)
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model, which="torque")[0] == TB_ERR_ARG
    # the drive: every entry refuses it with the same message
    for j, value, msg in ((0, np.nan, "transmission T is not finite"), (7, np.inf, "transmission T is not finite"),
                          (36 + 2, -1e-9, "motor 2: rotor inertia -1e-09 must be finite and >= 0"),
                          (36 + 5, np.nan, "motor 5: rotor inertia nan must be finite and >= 0"),
                          (42 + 0, -0.5, "motor 0: friction -0.5 must be finite and >= 0"),
                          (42 + 4, np.inf, "motor 4: friction inf must be finite and >= 0")):
        bad = good.copy()
        bad[j] = value
        for which, entry in (("torque", "tbd_drive_torque"), ("terms", "tbd_drive_torque_terms"),
                             ("speed", "tbd_drive_speed_terms")):
            assert rc(drive=bad, which=which) == (TB_ERR_ARG, "%s: %s" % (entry, msg))
    singular = _coupled(6)
    singular[3] = 2.0 * singular[1]                            # two equal rows up to scale
    for T in (singular, np.zeros((6, 6))):
        for which, entry in (("torque", "tbd_drive_torque"), ("terms", "tbd_drive_torque_terms"),
                             ("speed", "tbd_drive_speed_terms")):
            r, msg = rc(drive=dr.pack(T, 0.0, 0.0), which=which)
            assert r == TB_ERR_ARG and msg.startswith("%s: transmission T is singular (zero pivot in column" % entry)
    assert rc(drive=dr.pack(np.diag([1.0, 2.0, 0.0, 4.0, 5.0, 6.0]), 0.0, 0.0), which="speed") == (
        TB_ERR_ARG, "tbd_drive_speed_terms: transmission T is singular (zero pivot in column 2)")
    # a non-finite inverse: T finite, pivots finite, T^-1 overflows
    huge = np.diag([1e-310, 1.0, 1.0, 1.0, 1.0, 1.0])
    assert rc(drive=dr.pack(huge, 0.0, 0.0), which="torque") == (
        TB_ERR_ARG, "tbd_drive_torque: the inverse of transmission T is not finite")
    for i, value in ((0, 0.0), (3, -1.0), (5, np.nan), (2, -np.inf)):
        om = omega.copy()
        om[i] = value
        assert rc(om=om, which="speed") == (
            TB_ERR_ARG, "tbd_drive_speed_terms: motor %d: speed limit %g must be > 0 (inf allowed)" % (i, value))
    # valid calls pass validation and fail only at the launch (no device here)
    om = omega.copy()
    om[1] = np.inf
    for which in ("torque", "terms", "speed"):
        r, msg = rc(om=om, which=which)
        assert r not in (0, TB_ERR_ARG, TB_ERR_UNSUPPORTED) and "launch failed" in msg


def test_value_errors():
    import toppra_b200 as ta
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    n = np.full(6, 100.0)
    with pytest.raises(ValueError, match="exactly one"):
        ta.Drives(m)
    with pytest.raises(ValueError, match="exactly one"):
        ta.Drives(m, gear_ratio=n, transmission=np.diag(n))
    with pytest.raises(ValueError, match="RigidBodyModel"):
        ta.Drives(None, gear_ratio=n)
    for kw in (dict(gear_ratio=np.ones(5)), dict(gear_ratio=np.ones((6, 1))), dict(transmission=np.eye(5)),
               dict(transmission=np.ones(36)), dict(gear_ratio=n, rotor_inertia=np.ones(3)),
               dict(gear_ratio=n, friction=np.ones((6, 6)))):
        with pytest.raises(ValueError, match="shape"):
            ta.Drives(m, **kw)
    drv = ta.Drives(m, gear_ratio=n, rotor_inertia=1e-5, friction=0.01)
    assert drv.packed.shape == (6 * 6 + 12,) and np.array_equal(drv.packed[:36], np.diag(n).reshape(-1))
    assert np.array_equal(ta.Drives(m, transmission=_coupled(6)).packed[:36], _coupled(6).reshape(-1))
    lim = np.stack([-np.ones(6), np.ones(6)], axis=1)
    for bad in (np.ones((6, 3)), np.ones((7, 2)), np.ones((2, 5, 2)), np.ones(12)):       # dof mismatch, wrong shapes
        with pytest.raises(ValueError, match="torque_limits has shape"):
            ta.MotorTorqueConstraint(drv, bad)
    for bad in (np.ones(5), np.ones((6, 1)), 300.0):
        with pytest.raises(ValueError, match="speed_limit has shape"):
            ta.MotorSpeedConstraint(drv, bad)
    for cls, arg in ((ta.MotorTorqueConstraint, lim), (ta.MotorSpeedConstraint, np.full(6, 300.0))):
        with pytest.raises(ValueError, match="Drives"):
            cls(m, arg)
    grid = np.linspace(0, 1, 10)
    tc = ta.MotorTorqueConstraint(drv, lim)
    assert tc.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 24           # Interpolation: 4 nv
    assert ta.MotorTorqueConstraint(drv, lim, 0).num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 12
    per_path = ta.MotorTorqueConstraint(drv, np.tile(lim, (3, 1, 1)))
    assert per_path.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 24
    with pytest.raises(ValueError, match=r"torque_limits has shape \(3, 6, 2\); expected \(6, 2\) or \(4, 6, 2\)"):
        per_path.num_rows(RecordContext(FakePath(4, 6), grid, grid))
    sc = ta.MotorSpeedConstraint(drv, np.full(6, 300.0))
    assert sc.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    assert ta.MotorSpeedConstraint(drv, np.full(6, 300.0), 1).num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 2
    for c in (tc, sc):
        with pytest.raises(ValueError, match="Wrong dimension"):
            c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
        with pytest.raises(NotImplementedError):
            c.compute_constraint_params(type("P", (), {"dof": 6})(), grid)
    assert ta.constraint.Drives is ta.Drives and ta.constraint.MotorSpeedConstraint is ta.MotorSpeedConstraint
    with pytest.raises(ValueError, match="speed_limit has shape"):
        drv.speed_terms(np.zeros((2, 6)), np.ones(5))


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


@pytest.mark.gpu
def test_gpu_vs_mp_random_trees_and_fixtures(ta):
    worst = 0.0
    for nv in (1, 2, 3, 5, 8, 12, 16):
        rng = np.random.RandomState(2300 + nv)
        m = _model_from_packed(ta, rr.random_tree(rng, nv))
        mp = rr.MpRobot.from_packed(m.packed)
        T = _transmission(rng, nv)
        assert np.linalg.cond(T) <= 100.0 * (1 + 1e-9)
        drv = ta.Drives(m, transmission=T, rotor_inertia=rng.uniform(0, 1e-3, nv))
        npts = 2 if nv <= 8 else 1
        q, qd, qdd = (rng.uniform(-2, 2, (npts, nv)) for _ in range(3))
        got = drv.torque(_dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
        for i in range(npts):
            want = np.array([float(x) for x in dr.mp_torque(mp, drv.packed, q[i], qd[i], qdd[i])])
            err = np.max(np.abs(got[i] - want)) / _scale(want)
            assert err <= 1e-12, (nv, err)
            worst = max(worst, err)
        Q, QD, QDD = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
        np.testing.assert_allclose(drv.torque(Q, QD, QDD), dr.torque_packed(m.packed, drv.packed, Q, QD, QDD),
                                   rtol=0, atol=1e-11 * _scale(dr.torque_packed(m.packed, drv.packed, Q, QD, QDD)))
    for name, locked in CASES:
        m = model_of(name, locked)
        mp = rr.MpRobot.from_urdf(urdf(name), locked)
        rng = np.random.RandomState(m.nv)
        drv = ta.Drives(m, transmission=_coupled(m.nv), rotor_inertia=rng.uniform(1e-5, 5e-5, m.nv))
        q, qd, qdd = (rng.uniform(-2, 2, m.nv) for _ in range(3))
        got = drv.torque(q, qd, qdd)                                      # numpy round trip
        want = np.array([float(x) for x in dr.mp_torque(mp, drv.packed, q, qd, qdd)])
        worst = max(worst, np.max(np.abs(got - want)) / _scale(want))
        assert got.shape == (m.nv,) and worst <= 1e-12
    print("tbd_drive_torque vs the 50-digit reference: worst scaled error %.2e" % worst)


@pytest.mark.gpu
def test_gpu_terms_three_launch_identity_joint_side_reduction_and_diagonal(ta):
    import torch
    m = model_of("arm7_gripper.urdf")
    nv, M = m.nv, 4000
    rng = np.random.RandomState(17)
    q, qs, qss = (_dev(rng.uniform(-2, 2, (M, nv))) for _ in range(3))
    qs[::7, 1] = 0.0
    zero = torch.zeros_like(q)
    # three launches plus the torch operations, f = 0
    drv = ta.Drives(m, transmission=_transmission(rng, nv), rotor_inertia=rng.uniform(0, 1e-4, nv))
    a, b, c = drv.torque_terms(q, qs, qss)
    w0 = drv.torque(q, zero, zero)
    assert torch.equal(c, w0)
    assert torch.equal(a, drv.torque(q, zero, qs) - w0) and torch.equal(b, drv.torque(q, qs, qss) - w0)
    # T = I, I_r = 0, f = the joint friction: the joint-side terms of tbd_torque_terms
    fric = 0.1 + 0.05 * np.arange(nv)
    eye = ta.Drives(m, gear_ratio=np.ones(nv), friction=fric)
    for x, y in zip(eye.torque_terms(q, qs, qss), m.torque_terms(q, qs, qss, fric)):
        assert torch.equal(x, y)
    # T = diag(n): (tau + n^2 I_r qdd) / n
    n, Ir = rng.uniform(30, 160, nv), rng.uniform(1e-5, 1e-4, nv)
    diag = ta.Drives(m, gear_ratio=n, rotor_inertia=Ir)
    tau = m(q, qs, qss).cpu().numpy()
    want = (tau + n * n * Ir * qss.cpu().numpy()) / n
    np.testing.assert_allclose(diag.torque(q, qs, qss).cpu().numpy(), want, rtol=1e-14, atol=1e-14 * _scale(want))
    # friction: c += f o sign(T q')
    fr = ta.Drives(m, transmission=_coupled(nv), friction=0.03)
    c1 = fr.torque_terms(q, qs, qss)[2]
    c0 = ta.Drives(m, transmission=_coupled(nv)).torque_terms(q, qs, qss)[2]
    want = c0.cpu().numpy() + 0.03 * np.sign(qs.cpu().numpy() @ _coupled(nv).T)
    np.testing.assert_allclose(c1.cpu().numpy(), want, rtol=0, atol=1e-15 * _scale(want))


@pytest.mark.gpu
def test_gpu_speed_row_bit_equal_and_nan(ta):
    m = model_of("arm6.urdf")
    rng = np.random.RandomState(5)
    M = 5000
    qs = rng.uniform(-3, 3, (M, 6))
    qs[::11] = 0.0
    for T in (_coupled(6), _transmission(rng, 6), np.diag(np.full(6, 80.0))):
        drv = ta.Drives(m, transmission=T)
        for omega in (rng.uniform(100, 500, 6), np.array([np.inf, 200, np.inf, 300, 100, np.inf])):
            b = drv.speed_terms(_dev(qs), omega).cpu().numpy()
            assert np.array_equal(b, dr.speed_terms_packed(drv.packed, omega, qs))
            assert (b[::11] == 0).all() and (b > 0).any()
    bad = qs[:20].copy()
    bad[3, 2], bad[7, 0] = np.nan, np.nan
    b = ta.Drives(m, transmission=_coupled(6)).speed_terms(_dev(bad), np.full(6, 300.0)).cpu().numpy()
    assert np.isnan(b[[3, 7]]).all() and not np.isnan(np.delete(b, [3, 7])).any()
    b = ta.Drives(m, gear_ratio=np.full(6, 50.0)).speed_terms(_dev(bad), np.array([np.inf] * 5 + [300.0])).cpu().numpy()
    assert np.isnan(b[[3, 7]]).all()                                 # NaN * 0 / inf: the row is NaN, not 0


def _drives_of(ta, g, robot, m):
    T, Ir, f = dr.unpack(g[robot + "/drive"], m.nv)
    return ta.Drives(m, transmission=T, rotor_inertia=Ir, friction=f)


def _cons(ta, drv, vlim, alim, taulim, omega, scheme=0):
    return [ta.constraint.JointVelocityConstraint(vlim),
            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
            ta.MotorTorqueConstraint(drv, taulim, discretization_scheme=scheme),
            ta.MotorSpeedConstraint(drv, omega, discretization_scheme=scheme)]


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("drive_limits")
    m = model_of(name, locked)
    drv = _drives_of(ta, g, robot, m)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim, taulim, omega = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "taulim", "omega"))
    B, G = way.shape[0], len(grid)
    assert (omega == omega[0]).all()
    path = ta.BatchSplineInterpolator(ss, way)
    q, qs, qss = (path.eval_device(_dev(grid), o).reshape(-1, m.nv) for o in (0, 1, 2))
    terms = [x.cpu().numpy().reshape(B, G, m.nv) for x in drv.torque_terms(q, qs, qss)]
    for got, key in zip(terms, ("a", "b", "c")):
        assert np.max(np.abs(got - g[robot + "/" + key])) <= 1e-12 * _scale(g[robot + "/" + key])
    sp = drv.speed_terms(qs, omega[0]).cpu().numpy().reshape(B, G)
    np.testing.assert_allclose(sp, g[robot + "/speed"], rtol=1e-12, atol=0)
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (robot, scheme, x)][i]  # noqa: E731
        for i in range(B):
            one = ta.algorithm.TOPPRA(_cons(ta, drv, vlim[i], alim[i], taulim[i], omega[i], scheme),
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega[0], scheme), path, grid)
        h = h.compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


def _motor_rows(m, drv, taulim, omega, q, qs, qss, grid):
    """(G, 3, 2 nv + 1) collocation rows of the two motor limits for the oracle, from the numpy doubles."""
    nv = m.nv
    a, b, c = dr.torque_terms_packed(m.packed, drv.packed, q, qs, qss)
    F = np.vstack((np.eye(nv), -np.eye(nv)))
    g = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    tor = np.stack((a.dot(F.T), b.dot(F.T), c.dot(F.T) - g), axis=1)
    G = len(grid)
    sp = dr.speed_terms_packed(drv.packed, omega, qs).reshape(G, 1)
    speed = _oracle_rows(np.ones((1, 1)), np.zeros((G, 1)), sp, np.full((G, 1), -1.0), grid, False)
    return np.concatenate((tor, speed), axis=2)


def _limits(m, drv, B, seed, frac=0.45):
    rng = np.random.RandomState(seed)
    n = np.abs(np.diag(dr.unpack(drv.packed, m.nv)[0]))
    eff = np.where(np.isfinite(m.effort_limit), m.effort_limit, 8.0)
    tm = frac * eff / n * rng.uniform(0.8, 1.2, (B, m.nv))
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    return np.stack([-tm, tm], axis=-1), 0.7 * vel * n


@pytest.mark.gpu
def test_gpu_256_paths_per_path_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    drv = ta.Drives(m, transmission=_coupled(6), rotor_inertia=np.linspace(4e-5, 1e-5, 6), friction=0.02)
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _problems(B, nv, 83, m.velocity_limit)
    taulim, omega = _limits(m, drv, B, 3)
    grid = np.linspace(0, 1, G)
    h = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega), ta.BatchSplineInterpolator(ss, way), grid)
    h = h.compute_parameterization(0, 0).to_host()
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        rows = np.concatenate((_oracle_joint_rows(qs, qss, vlim[i], alim[i]),
                               _motor_rows(m, drv, taulim[i], omega, q, qs, qss, grid)), axis=2)
        o = orc.solve_rows(rows, orc.velocity_xbound(qs, vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += h["status"][i] == 0
    assert n_ok > 0.8 * B, n_ok


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    nv, B = m.nv, 12
    drv = ta.Drives(m, transmission=_coupled(nv), rotor_inertia=3e-5, friction=0.02)
    ss, way, vlim, alim = _problems(B, nv, 29, m.velocity_limit)
    taulim, omega = _limits(m, drv, B, 4)
    path = ta.BatchSplineInterpolator(ss, way)
    rag = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, drv, vlim[i:i + 1], alim[i:i + 1], taulim[i:i + 1], omega),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega, scheme), path, grid,
                               max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
        assert (hw["status"] == 0).sum() >= B // 2
        for i in range(3):
            one = ta.algorithm.TOPPRA(_cons(ta, drv, vlim[i], alim[i], taulim[i], omega, scheme),
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            run = one.compute_parameterization(0, 0, return_data=True)
            assert _eq(run[3], hw["K"][i])
            if hw["status"][i] == 0:
                assert _eq(run[1], hw["sd"][i]) and _eq(run[0], hw["sdd"][i])
            b1 = ta.BatchTOPPRA(_cons(ta, drv, vlim[i:i + 1], alim[i:i + 1], taulim[i:i + 1], omega, scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0)
            b1 = b1.to_host()
            assert _eq(b1["K"][0], hw["K"][i]) and _eq(b1["sd"][0], hw["sd"][i]) and b1["status"][0] == hw["status"][i]


@pytest.mark.gpu
def test_gpu_toppra_sd_and_quintic_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    drv = ta.Drives(m, transmission=_coupled(6), rotor_inertia=np.linspace(4e-5, 1e-5, 6), friction=0.02)
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(43)
    path = ta.BatchPiecewisePolyPath(np.linspace(0, 1, nseg + 1), rng.uniform(-0.4, 0.4, (B, k, nseg, nv)))
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    taulim, omega = _limits(m, drv, B, 6)
    d = _dev(grid)
    qs = [path.eval_device(d, o).cpu().numpy() for o in (0, 1, 2)]
    h = ta.BatchTOPPRA(_cons(ta, drv, vlim, alim, taulim, omega), path, grid).compute_parameterization(0, 0).to_host()
    ok = h["status"] == 0
    assert ok.sum() >= B // 2
    for i in range(B):
        rows = np.concatenate((_oracle_joint_rows(qs[1][i], qs[2][i], vlim[i], alim[i]),
                               _motor_rows(m, drv, taulim[i], omega, qs[0][i], qs[1][i], qs[2][i], grid)), axis=2)
        o = orc.solve_rows(rows, orc.velocity_xbound(qs[1][i], vlim[i]), grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
    # BatchTOPPRAsd, whole and in record chunks: bit-equal, and the motor speeds hold on the blended profiles
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        inst = ta.BatchTOPPRAsd(_cons(ta, drv, vlim, alim, taulim, omega), path, grid)
        if chunk:
            inst = ta.BatchTOPPRAsd(_cons(ta, drv, vlim, alim, taulim, omega), path, grid,
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
        b = dr.speed_terms_packed(drv.packed, omega, qs[1][i])
        assert (b * sd[i] ** 2 <= 1 + 1e-9).all()


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch):
    from dyn_common import _assert_one_terms_launch
    m = model_of("arm6.urdf")
    drv = ta.Drives(m, transmission=_coupled(6), rotor_inertia=2e-5)
    ss, way, vlim, alim = _problems(10, 6, 47, m.velocity_limit)
    taulim, omega = _limits(m, drv, 10, 8)
    path, grid = ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80)
    joint = lambda: [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)]  # noqa: E731
    _assert_one_terms_launch(ta, monkeypatch, lambda: joint() + [ta.MotorTorqueConstraint(drv, taulim)], path, grid,
                             "tbd_drive_torque_terms")
    _assert_one_terms_launch(ta, monkeypatch, lambda: joint() + [ta.MotorSpeedConstraint(drv, omega)], path, grid,
                             "tbd_drive_speed_terms")
