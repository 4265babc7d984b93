"""Rigid-body models and their inverse dynamics on the GPU (toppra_b200.RigidBodyModel, libtoppra_b200_dyn.so).

CPU:
  * URDF parsing and folding: the packed model of RigidBodyModel.from_urdf, evaluated by the float64 numpy double of
    tests/rnea_ref.py, equals the 50-digit Lagrangian reference on the RAW URDF tree (fixed and locked joints as zero-DOF
    links) to 1e-13 of the torque scale max|tau| of each state;
  * every ValueError of from_urdf; the ctypes prototypes against include/toppra_b200_dyn.h; each argument check of the
    C-ABI returns its TB_ERR_* from the real library.
GPU:
  * tbd_rnea on random trees (1 to 16 bodies) against the 50-digit reference within 1e-12 of max|tau|; the mass matrix
    from unit accelerations is symmetric and equals the Jacobian form;
  * tbd_torque_terms equals three model(...) calls plus the torch operations of SecondOrderConstraint bit for bit;
  * the reference golden (tests/golden/rigid_body_torque.npz, make_golden_rnea.py): torque terms within 1e-12,
    TOPPRA and BatchTOPPRA K and sd within |dK| <= 1e-9 + 1e-8 |K| (the cfg-3 tolerance), equal statuses;
  * 256 paths against the oracle fed with rows from the numpy double, same tolerance;
  * ragged vs per-path common grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1: bit-equal; a quintic
    BatchPiecewisePolyPath."""
import ctypes
import os
import re

import numpy as np
import pytest

import rnea_ref as rr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROBOTS = os.path.join(ROOT, "tests", "golden", "robots")
DYN_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_dyn.so")
LOCKED = {"finger_left_joint": 0.013, "finger_right_joint": 0.021}
TB_ERR_ARG, TB_ERR_UNSUPPORTED = -1, -2
CASES = [("arm6.urdf", None), ("arm7_gripper.urdf", LOCKED), ("arm7_gripper.urdf", None)]


def urdf(name):
    return open(os.path.join(ROBOTS, name)).read()


def model_of(name, locked=None):
    from toppra_b200 import RigidBodyModel
    return RigidBodyModel.from_urdf(urdf(name), locked_joints=locked)


def close(got, ref, tol):
    """|got - ref| <= tol * max(1, max|ref|) (the torque scale of the state)."""
    ref = np.asarray(ref, dtype=np.float64)
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(np.asarray(got) - ref)))
    assert err <= tol * scale, (err, scale)
    return err / scale


# ==== CPU: parsing, folding, errors ==================================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_urdf_folding_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    assert m.nv == mp.nv and m.joint_names == [j["name"] for j in mp.joints if j["dof"] is not None]
    rng = np.random.RandomState(m.nv)
    for _ in range(2):
        q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
        close(rr.rnea_packed(m.packed, q, qd, qdd)[0], mp.tau64(q, qd, qdd), 1e-13)


def test_urdf_joint_order_and_limits():
    m = model_of("arm7_gripper.urdf")
    # depth first, children in file order: the camera joint (listed before upper_roll) comes after the arm subtree
    assert m.joint_names == ["torso_yaw", "shoulder", "upper_roll", "elbow", "forearm_roll", "wrist_pitch",
                             "finger_left_joint", "finger_right_joint", "camera_pan"]
    assert [int(m.body(k)[1]) for k in range(m.nv)] == [0] * 6 + [1, 1, 0]
    assert [int(m.body(k)[0]) for k in range(m.nv)] == [-1, 0, 1, 2, 3, 4, 5, 5, 0]
    tl = m.torque_limits()
    assert tl.shape == (9, 2) and tl[0, 1] == 180 and tl[0, 0] == -180 and np.isinf(tl[8]).all()
    assert m.velocity_limit[6] == 0.2 and np.isinf(m.velocity_limit[8])
    m6 = model_of("arm6.urdf")
    assert m6.nv == 6 and m6.body(5)[17] == pytest.approx(0.25 + 0.9)     # flange folded into wrist3
    assert np.allclose(m6.gravity, [0, 0, -9.81])


def _chain(n, extra=""):
    links = "".join('<link name="l%d"><inertial><mass value="1"/><inertia ixx="1" iyy="1" izz="1"/></inertial></link>'
                    % k for k in range(n + 1))
    joints = "".join('<joint name="j%d" type="revolute"><parent link="l%d"/><child link="l%d"/><axis xyz="0 0 1"/></joint>'
                     % (k, k, k + 1) for k in range(n))
    return '<robot name="t">%s%s%s</robot>' % (links, joints, extra)


@pytest.mark.parametrize("text,match", [
    (_chain(2).replace('name="j1" type="revolute"', 'name="j1" type="floating"'), "floating"),
    (_chain(2).replace('name="j1" type="revolute"', 'name="j1" type="planar"'), "planar"),
    (_chain(2).replace('<axis xyz="0 0 1"/></joint></robot>', '<axis xyz="0 0 1"/><mimic joint="j0"/></joint></robot>'),
     "mimic"),
    (_chain(2) .replace("</robot>", '<link name="stray"/></robot>'), "root"),
    (_chain(2).replace("</robot>", '<joint name="loop" type="fixed"><parent link="l2"/><child link="l0"/></joint></robot>'),
     "root"),
    (_chain(17), "more than 16"),
    (_chain(2).replace('name="j1" type="revolute"', 'name="j1" type="screw"'), "unknown type"),
])
def test_urdf_value_errors(text, match):
    from toppra_b200 import RigidBodyModel
    with pytest.raises(ValueError, match=match):
        RigidBodyModel.from_urdf(text)


def test_urdf_locking_removes_mimic_and_counts():
    from toppra_b200 import RigidBodyModel
    text = _chain(2).replace('<axis xyz="0 0 1"/></joint></robot>', '<axis xyz="0 0 1"/><mimic joint="j0"/></joint></robot>')
    assert RigidBodyModel.from_urdf(text, locked_joints={"j1": 0.3}).nv == 1
    assert RigidBodyModel.from_urdf(_chain(17), locked_joints={"j16": 0.0}).nv == 16
    with pytest.raises(ValueError, match="unknown"):
        RigidBodyModel.from_urdf(_chain(2), locked_joints={"nope": 0.0})


def test_rigid_body_model_routes_torque_constraints_to_the_device():
    import toppra_b200 as ta
    m = model_of("arm6.urdf")
    so = ta.constraint.SecondOrderConstraint.joint_torque_constraint(m, m.torque_limits(), np.zeros(6))
    assert so.batched
    jt = ta.constraint.JointTorqueConstraint(m, m.torque_limits(), np.ones(6))
    assert jt._second_order().batched and jt._second_order().inv_dyn is m


def _dyn_header():
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(tbd_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        out[name] = ["ptr" if "*" in a else ("double" if "double" in a else "int")
                     for a in (x.strip() for x in args.split(",")) if a not in ("", "void")]
    return out


def test_dyn_header_matches_prototypes():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert set(declared) == set(_lib_dyn._PROTOS)
    for name, (argtypes, restype) in _lib_dyn._PROTOS.items():
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name], name
        assert restype is ctypes.c_int


def _gpu_present():
    import torch
    return torch.cuda.is_available()


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_dyn_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    assert lib.tbd_version() == 100
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    good = model_of("arm6.urdf").packed

    def rc(packed, nv=6, M=4, null=None):
        host = np.array(packed, dtype=np.float64)
        args = [ctypes.c_void_p(host.ctypes.data), nv, M, d, d, d, d]
        targs = [ctypes.c_void_p(host.ctypes.data), nv, M, d, d, d, None, d, d, d]
        if null is not None:
            args[null] = None
            targs[null if null < 6 else null + 1] = None
        r1 = lib.tbd_rnea(*args, None)
        r2 = lib.tbd_torque_terms(*targs, None)
        assert r1 == r2, (r1, r2)
        assert r1 == 0 or _lib.load().tb_last_error()
        return r1

    for k in (0, 3, 4, 5, 6):
        assert rc(good, null=k) == TB_ERR_ARG
    assert rc(good, M=0) == TB_ERR_ARG and rc(good, M=-3) == TB_ERR_ARG
    assert rc(good, nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[good, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED

    def bad(k, j, value):
        p = good.copy()
        p[3 + 27 * k + j] = value
        return rc(p)
    assert bad(2, 0, 2.0) == TB_ERR_ARG                 # parent[k] >= k
    assert bad(2, 0, 1.5) == TB_ERR_ARG and bad(0, 0, -2.0) == TB_ERR_ARG
    assert bad(3, 1, 2.0) == TB_ERR_ARG                 # unknown joint type
    assert bad(1, 17, -1.0) == TB_ERR_ARG and bad(1, 17, np.nan) == TB_ERR_ARG and bad(1, 17, np.inf) == TB_ERR_ARG
    p = good.copy()
    p[3 + 27 * 4 + 2:3 + 27 * 4 + 5] = 0.0              # zero axis
    assert rc(p) == TB_ERR_ARG
    # the torque-terms entry additionally takes a nullable friction: its NULL is not an error, the outputs' are
    host = good.copy()
    for k in (7, 8, 9):
        targs = [ctypes.c_void_p(host.ctypes.data), 6, 4, d, d, d, None, d, d, d, None]
        targs[k] = None
        assert lib.tbd_torque_terms(*targs) == TB_ERR_ARG


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _dev(x):
    import torch
    return torch.as_tensor(np.asarray(x, dtype=np.float64), device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_rnea_random_trees_vs_mp(ta, nv):
    rng = np.random.RandomState(100 + nv)
    packed = rr.random_tree(rng, nv)
    m = ta.RigidBodyModel(packed[3::27][:nv], packed[4::27][:nv], packed[3:].reshape(nv, 27)[:, 2:5],
                          packed[3:].reshape(nv, 27)[:, 5:14], packed[3:].reshape(nv, 27)[:, 14:17],
                          packed[3:].reshape(nv, 27)[:, 17], packed[3:].reshape(nv, 27)[:, 18:21],
                          packed[3:].reshape(nv, 27)[:, 21:27], gravity=packed[:3])
    assert np.allclose(m.packed, packed, rtol=1e-15, atol=0)      # the constructor re-normalises the unit axes
    packed = m.packed
    mp = rr.MpRobot.from_packed(packed)
    P = 2 if nv <= 8 else 1
    q, qd, qdd = (rng.uniform(-2, 2, (P, nv)) for _ in range(3))
    tau = m(_dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
    for i in range(P):
        close(tau[i], mp.tau64(q[i], qd[i], qdd[i]), 1e-12)
    # many more states against the numpy double (itself pinned to the mp reference on the CPU)
    q, qd, qdd = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
    tau = m(_dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
    ref = rr.rnea_packed(packed, q, qd, qdd)
    assert np.max(np.abs(tau - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref)))
    # numpy (nv,) input: the same launch through a device round trip
    assert np.array_equal(m(q[0], qd[0], qdd[0]), tau[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name,locked", CASES)
def test_gpu_mass_matrix_symmetric_and_jacobian_form(ta, name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(7)
    q = rng.uniform(-2, 2, m.nv)
    eye = np.eye(m.nv)
    Q = np.tile(q, (m.nv + 1, 1))
    acc = np.vstack([np.zeros(m.nv), eye])
    tau = m(_dev(Q), _dev(np.zeros_like(Q)), _dev(acc)).cpu().numpy()
    Mg = (tau[1:] - tau[0]).T
    with __import__("mpmath").workdps(rr.DPS):
        Mref = np.array(mp.mass_matrix([__import__("mpmath").mpf(float(x)) for x in q]).tolist(), dtype=np.float64)
    assert np.max(np.abs(Mg - Mg.T)) <= 1e-12 * np.max(np.abs(Mref))
    close(Mg, Mref, 1e-12)


@pytest.mark.gpu
def test_gpu_builds_run(ta):
    from test_piecewise_poly import launched
    m = model_of("arm6.urdf")
    x = _dev(np.random.RandomState(1).randn(64, 6))
    names = set()
    for _ in range(3):
        with launched() as got:
            m(x, x, x)
            m.torque_terms(x, x, x, np.ones(6))
        names |= got
        if {"rnea_kernel", "torque_terms_kernel"} <= names:   # kineto now and then returns a capture without device activity
            break
    assert {"rnea_kernel", "torque_terms_kernel"} <= names, sorted(names)


@pytest.mark.gpu
@pytest.mark.parametrize("fric", [None, "ones", "mixed"])
def test_gpu_torque_terms_bit_equal_three_calls(ta, fric):
    import torch
    m = model_of("arm7_gripper.urdf")
    rng = np.random.RandomState(3)
    M = 1000
    q, qs, qss = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(3))
    qs[::7, 2] = 0.0                                            # sign(0) = 0
    f = {None: None, "ones": np.ones(m.nv), "mixed": np.r_[0.0, 0.5, 0.0, 1.5, 2.0, 0.1, 0.0, 0.3, 0.7]}[fric]
    a, b, c = m.torque_terms(q, qs, qss, f)
    zero = torch.zeros_like(q)
    c0 = m(q, zero, zero)
    a0 = m(q, zero, qs) - c0
    b0 = m(q, qs, qss) - c0
    if f is not None:
        c0 = c0 + torch.sign(qs) * _dev(f)
    assert torch.equal(a, a0) and torch.equal(b, b0) and torch.equal(c, c0)


def _golden_problem(g, robot, b):
    return (g[robot + "/way"][b], g[robot + "/vlim"][b], g[robot + "/alim"][b], g[robot + "/taulim"][b],
            g[robot + "/fric"][b])


def _assert_solution(got, ref_K, ref_sd, st, ref_st):
    assert st == ref_st
    if ref_st == 0:
        np.testing.assert_allclose(got[0], ref_K, rtol=1e-8, atol=1e-9)
        np.testing.assert_allclose(got[1], ref_sd, rtol=1e-8, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("rigid_body_torque")
    m = model_of(name, locked)
    ss, grid = g["ss"], g["grid"]
    B = g[robot + "/way"].shape[0]
    path = ta.BatchSplineInterpolator(ss, g[robot + "/way"])
    # torque terms at the gridpoints, collocation form, against the reference's JointTorqueConstraint on the mp model
    q, qs, qss = (path.eval_device(_dev(grid), o).reshape(-1, m.nv) for o in (0, 1, 2))
    for b in range(B):
        a, bb, c = m.torque_terms(q, qs, qss, g[robot + "/fric"][b])
        G = len(grid)
        sl = slice(b * G, (b + 1) * G)
        for got, key in ((a, "a"), (bb, "b"), (c, "c")):
            close(got[sl].cpu().numpy(), g[robot + "/" + key][b], 1e-12)
    for scheme in (0, 1):
        way, vlim, alim, taulim, fric = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "taulim", "fric"))
        for b in range(B):                     # single-path TOPPRA (JointTorqueConstraint takes the device route)
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[b]),
                                       ta.constraint.JointAccelerationConstraint(alim[b], discretization_scheme=scheme),
                                       ta.constraint.JointTorqueConstraint(m, taulim[b], fric[b],
                                                                           discretization_scheme=scheme)],
                                      ta.SplineInterpolator(ss, way[b]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), g["%s/s%d/K" % (robot, scheme)][b], g["%s/s%d/sd" % (robot, scheme)][b], st,
                             g["%s/s%d/status" % (robot, scheme)][b])
        # BatchTOPPRA: friction per batch is one vector, so solve the paths that share fric[0] (all of them here)
        assert (fric == fric[0]).all()
        h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            ta.constraint.SecondOrderConstraint.joint_torque_constraint(
                                m, taulim, fric[0], discretization_scheme=scheme)],
                           path, grid).compute_parameterization(0, 0).to_host()
        for b in range(B):
            _assert_solution((h["K"][b], h["sd"][b]), g["%s/s%d/K" % (robot, scheme)][b],
                             g["%s/s%d/sd" % (robot, scheme)][b], h["status"][b], g["%s/s%d/status" % (robot, scheme)][b])


def _random_problems(B, nv, seed, effort, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    al = rng.uniform(6, 10, (B, nv))
    alim = np.stack([-al, al], axis=-1)
    tl = 0.45 * effort * rng.uniform(0.8, 1.2, (B, nv))
    taulim = np.stack([-tl, tl], axis=-1)
    return np.linspace(0, 1, 5), way, vlim, alim, taulim


@pytest.mark.gpu
def test_gpu_256_paths_vs_oracle_with_numpy_double_rows(ta):
    from oracle import oracle as orc
    from toppra_b200.constraint.linear_constraint import canlinear_colloc_to_interpolate
    m = model_of("arm6.urdf")
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim, taulim = _random_problems(B, nv, 5, m.effort_limit, m.velocity_limit)
    fric = 0.3 + 0.1 * np.arange(nv)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
                        ta.constraint.SecondOrderConstraint.joint_torque_constraint(m, taulim, fric)],
                       path, grid).compute_parameterization(0, 0).to_host()
    F = np.vstack((np.eye(nv), -np.eye(nv)))
    n_ok = 0
    for b in range(B):
        c = orc.cubic_spline_fit(ss, way[b])
        lin = orc.solve_velacc(c, ss, grid, vlim[b], alim[b], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        av, bv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        g = np.concatenate((taulim[b, :, 1], -taulim[b, :, 0]))
        a2, b2, c2, F2, g2, _, _ = canlinear_colloc_to_interpolate(av, bv, cv, F, g, None, None, grid, identical=True)
        rows = np.concatenate((lin["rows"], np.stack((a2.dot(F2.T), b2.dot(F2.T), c2.dot(F2.T) - g2), axis=1)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][b], h["sd"][b]), o["K"], o["sd"], h["status"][b], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok > 0.9 * B


def _torque_cons(ta, m, vlim, alim, taulim, fric):
    return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
            ta.constraint.SecondOrderConstraint.joint_torque_constraint(m, taulim, fric)]


def _eq(x, y):
    return np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    B, nv = 12, m.nv
    ss, way, vlim, alim, taulim = _random_problems(B, nv, 11, np.where(np.isfinite(m.effort_limit), m.effort_limit, 8.0),
                                                   m.velocity_limit)
    fric = 0.2 * np.ones(nv)
    path = ta.BatchSplineInterpolator(ss, way)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for b in range(B):
        n = int(glen[b])
        gb = grids[b, :n]
        one = ta.BatchTOPPRA(_torque_cons(ta, m, vlim[b:b + 1], alim[b:b + 1], taulim[b:b + 1], fric),
                             ta.BatchSplineInterpolator(ss, way[b:b + 1]), gb).compute_parameterization(0, 0).to_host()
        assert hr["status"][b] == one["status"][0]
        assert _eq(hr["K"][b, :n], one["K"][0]) and _eq(hr["sd"][b, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    whole = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, grid)
    per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
    parts = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, grid, max_record_bytes=5 * per_path)
    assert parts.chunk_size() == 5
    hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
    for k in ("K", "sd", "sdd", "status"):
        assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA with JointTorqueConstraint equals BatchTOPPRA at B = 1
    for b in range(3):
        one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[b]),
                                   ta.constraint.JointAccelerationConstraint(alim[b]),
                                   ta.constraint.JointTorqueConstraint(m, taulim[b], fric,
                                                                       discretization_scheme=1)],
                                  ta.SplineInterpolator(ss, way[b]), gridpoints=grid, solver_wrapper="seidel")
        sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
        hb = ta.BatchTOPPRA(_torque_cons(ta, m, vlim[b:b + 1], alim[b:b + 1], taulim[b:b + 1], fric),
                            ta.BatchSplineInterpolator(ss, way[b:b + 1]), grid).compute_parameterization(0, 0).to_host()
        assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])


@pytest.mark.gpu
def test_gpu_quintic_piecewise_poly_path(ta):
    import torch
    m = model_of("arm6.urdf")
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(21)
    coeffs = rng.uniform(-0.4, 0.4, (B, k, nseg, nv))
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    taulim = np.tile(0.45 * m.torque_limits(), (B, 1, 1))
    fric = 0.25 * np.ones(nv)
    h = ta.BatchTOPPRA(_torque_cons(ta, m, vlim, alim, taulim, fric), path, grid).compute_parameterization(0, 0).to_host()
    # the same problem through the general batched callback (three model calls plus torch operations)
    so = ta.constraint.SecondOrderConstraint.joint_torque_constraint(lambda q, qd, qdd: m(q, qd, qdd), taulim, fric,
                                                                     batched=True)
    ht = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim), so],
                        path, grid).compute_parameterization(0, 0).to_host()
    for key in ("K", "sd", "sdd", "status"):
        assert _eq(h[key], ht[key]), key
    assert (h["status"] == 0).sum() >= B // 2
    assert isinstance(path.eval_device(torch.as_tensor(grid, device="cuda"), 2), torch.Tensor)
