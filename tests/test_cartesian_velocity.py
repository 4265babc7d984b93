"""Frame velocities of a rigid-body model on the GPU and the Cartesian speed limit of a frame (RigidBodyModel.frame,
RigidBodyFrame, CartesianVelocityNorm's device route; libtoppra_b200_dyn.so: tbd_frame_velocity, tbd_velocity_norm_terms).

CPU:
  * the frame table of from_urdf (every link: the root, links folded by fixed and locked joints, with offsets), through
    the float64 numpy double of tests/kin_ref.py, equals the 50-digit placements and velocities of the RAW URDF tree to
    1e-13 of the state's scale, in all three reference frames;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library.
GPU:
  * tbd_frame_velocity on random trees (1 to 16 bodies) against the 50-digit reference within 1e-12; a frame on the base
    gives exact zeros;
  * tbd_velocity_norm_terms equals tbd_frame_velocity plus the fixed-order quadratic form bit for bit; NaN in, NaN out;
  * the reference golden (tests/golden/cartesian_velocity.npz, make_golden_cartesian.py): TOPPRA and BatchTOPPRA within
    |dK| <= 1e-9 + 1e-8 |K| (the cfg-3 tolerance), equal statuses; 256 paths with per-path limits against the oracle fed
    with rows from the numpy double, same tolerance; b sd^2 <= limit on the solved profiles, active somewhere;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, host route vs device route:
    bit-equal; a quintic BatchPiecewisePolyPath; the constraint next to JointTorqueConstraint on the same model."""
import ctypes
import os

import numpy as np
import pytest

import kin_ref as kr
import rnea_ref as rr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROBOTS = os.path.join(ROOT, "tests", "golden", "robots")
DYN_LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200_dyn.so")
LOCKED = {"finger_left_joint": 0.013, "finger_right_joint": 0.021}
TB_ERR_ARG, TB_ERR_UNSUPPORTED = -1, -2
CASES = [("arm6.urdf", None), ("arm7_gripper.urdf", LOCKED), ("arm7_gripper.urdf", None)]
OFFSET = dict(xyz=(0.03, -0.02, 0.1), rpy=(0.3, -0.2, 0.5))


def urdf(name):
    return open(os.path.join(ROBOTS, name)).read()


def model_of(name, locked=None):
    from toppra_b200 import RigidBodyModel
    return RigidBodyModel.from_urdf(urdf(name), locked_joints=locked)


def close(got, ref, tol):
    """|got - ref| <= tol * max(1, max|ref|) (the scale of the state)."""
    ref = np.asarray(ref, dtype=np.float64)
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(np.asarray(got) - ref)))
    assert err <= tol * scale, (err, scale)
    return err / scale


def _mp_check(m, mp, frames, q, qd, tol):
    """Every RigidBodyFrame of `frames` {key: (frame, link, offset or None)} at (q, qd): placement and velocity of the
    numpy double against the 50-digit reference."""
    from toppra_b200.dynamics import rpy_matrix
    spec = {}
    for key, (f, link, off) in frames.items():
        spec[key] = (link, rpy_matrix(off["rpy"]) if off else np.eye(3), np.asarray(off["xyz"]) if off else np.zeros(3))
    ref = kr.mp_frames(mp, q, qd, spec)
    for key, (f, _, _) in frames.items():
        Rf, pf, v = kr.frame_packed(m.packed, f.packed, q, qd)
        r = ref[key]
        close(Rf[0], np.array(r["R"].tolist(), dtype=np.float64), tol)
        close(pf[0], [float(x) for x in r["p"]], tol)
        close(v[0], [float(x) for x in r["v"][f.reference_frame]], tol)


# ==== CPU: frame table, errors, C-ABI ================================================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_frame_table_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    assert set(m.frames) == set(mp.links)                       # every link, the root and folded ones included
    for link in ("world", "hand", "camera", "finger_left", "finger_right") if "arm7" in name else ("base_link", "flange"):
        assert link in m.frames
    assert m.frames[mp.root][0] == -1
    rng = np.random.RandomState(m.nv + 31)
    for _ in range(2):
        q, qd = rng.uniform(-2, 2, (2, m.nv))
        frames = {}
        for link in m.frames:
            for ref in kr.REFERENCE_FRAMES:
                frames[(link, ref, 0)] = (m.frame(link, reference_frame=ref), link, None)
                frames[(link, ref, 1)] = (m.frame(link, reference_frame=ref, **OFFSET), link, OFFSET)
        _mp_check(m, mp, frames, q, qd, 1e-13)


def test_frames_of_array_models():
    from toppra_b200 import RigidBodyModel
    packed = rr.random_tree(np.random.RandomState(4), 3)
    b = packed[3:].reshape(3, 27)
    m = RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27])
    assert sorted(m.frames) == ["body0", "body1", "body2"]
    f = m.frame("body2", reference_frame="world")
    assert f.body == 2 and np.array_equal(f.R, np.eye(3)) and np.array_equal(f.p, np.zeros(3))
    assert np.array_equal(f.packed, np.r_[2.0, np.eye(3).reshape(9), np.zeros(3), 0.0])
    assert m.frame("body0", xyz=(1, 2, 3)).packed[10:14].tolist() == [1.0, 2.0, 3.0, 2.0]


def test_value_errors():
    import toppra_b200 as ta
    from toppra_b200.constraint import CartesianVelocityNorm
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    with pytest.raises(ValueError, match="no frame"):
        m.frame("tool0")
    with pytest.raises(ValueError, match="reference_frame"):
        m.frame("flange", reference_frame="LOCAL")
    f = m.frame("flange")
    S = np.eye(6)
    with pytest.raises(ValueError, match="6x6"):
        CartesianVelocityNorm(f, np.eye(3), 0.25)
    with pytest.raises(ValueError, match="6x6"):
        CartesianVelocityNorm(f, np.eye(6)[:5], 0.25)
    with pytest.raises(ValueError, match="positive"):
        CartesianVelocityNorm(f, S, -0.1)
    with pytest.raises(ValueError, match="positive"):
        CartesianVelocityNorm(f, S, [0.2, -0.1, 0.3])
    with pytest.raises(ValueError, match="dof"):
        CartesianVelocityNorm(f, S, 0.25, dof=7)

    class FakePath(object):
        def __init__(self, B, dof):
            self.B, self.dof, self.device = B, dof, "cpu"
    grid = np.linspace(0, 1, 10)
    c = CartesianVelocityNorm(f, S, [0.2, 0.3, 0.4])
    assert c.get_dof() == 6 and c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 1
    assert CartesianVelocityNorm(f, S, 0.2, discretization_scheme=1).num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 2
    with pytest.raises(ValueError, match=r"expected a float or \(4,\)"):
        c.num_rows(RecordContext(FakePath(4, 6), grid, grid))
    with pytest.raises(ValueError, match=r"expected a float or \(5,\)"):            # a chunk of a 5-path batch
        c.num_rows(RecordContext(FakePath(2, 6), grid, grid, None, 0, 2, 5))
    with pytest.raises(ValueError, match="Wrong dimension"):
        c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
    # the varying form and user callbacks keep the host route and its messages
    v = CartesianVelocityNorm(f, velocity_limit=lambda s: (S, 0.2))
    with pytest.raises(NotImplementedError, match="no batched device implementation"):
        v.num_rows(RecordContext(FakePath(3, 6), grid, grid))
    assert not ta.constraint.CartesianVelocityNorm(lambda q, qd: np.zeros(6), S, 0.2, dof=6)._device()


def test_dyn_header_prototypes_of_frame_entries():
    from test_rigid_body import _dyn_header
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_frame_velocity"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_velocity_norm_terms"] == ["ptr", "int", "ptr", "ptr", "int", "ptr", "ptr", "ptr", "ptr"]
    for name in ("tbd_frame_velocity", "tbd_velocity_norm_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int
    text = open(os.path.join(ROOT, "include", "toppra_b200_dyn.h")).read()
    from toppra_b200.dynamics import REFERENCE_FRAMES
    for key, code in (("WORLD", 0), ("LOCAL", 1), ("LOCAL_WORLD_ALIGNED", 2)):
        assert "#define TBD_%s %d" % (key, code) in text and REFERENCE_FRAMES[key.lower()] == code
    assert "#define TBD_FRAME_DOUBLES 14" in text and model_of("arm6.urdf").frame("flange").packed.shape == (14,)


def _gpu_present():
    import torch
    return torch.cuda.is_available()


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_frame_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good_frame = m.frame("flange", **OFFSET).packed
    good_S = np.eye(6)

    def rc(model=m.packed, frame=good_frame, S=good_S, nv=6, M=4, null=None):
        host = [np.array(x, dtype=np.float64) for x in (model, frame, S)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        fv = [ptr[0], nv, ptr[1], M, d, d, d]
        nt = [ptr[0], nv, ptr[1], ptr[2], M, d, d, d]
        if null is not None:
            if null != "S":
                fv[null] = None
                nt[null if null < 3 else null + 1] = None
            else:
                nt[3] = None
        r2 = lib.tbd_velocity_norm_terms(*nt, None)
        if null == "S":
            assert r2 == TB_ERR_ARG and _lib.load().tb_last_error()
            return r2
        r1 = lib.tbd_frame_velocity(*fv, None)
        assert r1 == r2, (r1, r2)
        assert r1 == 0 or _lib.load().tb_last_error()
        return r1

    for k in (0, 2, 4, 5, 6, "S"):
        assert rc(null=k) == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k: the model checks come first
    assert rc(bad_model) == TB_ERR_ARG

    def frame_with(j, value):
        f = good_frame.copy()
        f[j] = value
        return rc(frame=f)
    for body in (6.0, -2.0, 1.5, np.nan):                     # body outside [-1, nv) or not an integer
        assert frame_with(0, body) == TB_ERR_ARG
    for ref in (3.0, -1.0, 0.5, np.nan):                       # unknown reference frame
        assert frame_with(13, ref) == TB_ERR_ARG
    for j in (1, 5, 9, 10, 12):                                # non-finite R or p
        assert frame_with(j, np.nan) == TB_ERR_ARG and frame_with(j, np.inf) == TB_ERR_ARG
    for j in (0, 17, 35):                                      # non-finite S (the norm entry only)
        S = good_S.copy().reshape(36)
        S[j] = np.inf
        host = np.array(S)
        args = [ctypes.c_void_p(m.packed.ctypes.data), 6, ctypes.c_void_p(good_frame.ctypes.data),
                ctypes.c_void_p(host.ctypes.data), 4, d, d, d, None]
        assert lib.tbd_velocity_norm_terms(*args) == TB_ERR_ARG


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


def _dev(x):
    import torch
    return torch.as_tensor(np.asarray(x, dtype=np.float64), device="cuda")


def _model_from_packed(ta, packed):
    nv = (len(packed) - 3) // 27
    b = packed[3:].reshape(nv, 27)
    return ta.RigidBodyModel(b[:, 0], b[:, 1], b[:, 2:5], b[:, 5:14], b[:, 14:17], b[:, 17], b[:, 18:21], b[:, 21:27],
                             gravity=packed[:3])


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_frame_velocity_random_trees_vs_mp(ta, nv):
    from toppra_b200.dynamics import rpy_matrix
    rng = np.random.RandomState(300 + nv)
    m = _model_from_packed(ta, rr.random_tree(rng, nv))
    mp = rr.MpRobot.from_packed(m.packed)
    P = 2 if nv <= 8 else 1
    q, qd = (rng.uniform(-2, 2, (P, nv)) for _ in range(2))
    frames = {}
    for ref in kr.REFERENCE_FRAMES:
        for k in sorted({nv - 1, int(rng.randint(nv))}):
            off = dict(xyz=tuple(rng.randn(3) * 0.2), rpy=tuple(rng.uniform(-3, 3, 3)))
            frames[(k, ref)] = (m.frame("body%d" % k, reference_frame=ref, **off), "b%d" % k, off)
    for (k, ref), (f, link, off) in frames.items():
        v = f(_dev(q), _dev(qd)).cpu().numpy()
        spec = {0: (link, rpy_matrix(off["rpy"]), np.asarray(off["xyz"]))}
        for i in range(P):
            r = kr.mp_frames(mp, q[i], qd[i], spec)[0]
            close(v[i], [float(x) for x in r["v"][ref]], 1e-12)
        # many more states against the numpy double (itself pinned to the mp reference on the CPU)
        Q, QD = (rng.uniform(-3, 3, (512, nv)) for _ in range(2))
        got = f(_dev(Q), _dev(QD)).cpu().numpy()
        want = kr.frame_velocity_packed(m.packed, f.packed, Q, QD)
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
        assert np.array_equal(f(Q[3], QD[3]), got[3])              # numpy (nv,): the same launch via a round trip
    # a frame on the base does not move
    for ref in kr.REFERENCE_FRAMES:
        base = ta.RigidBodyFrame(m, "base", -1, rpy_matrix((0.2, 0.1, -0.4)), (0.3, -0.1, 0.5), ref)
        z = base(_dev(rng.uniform(-3, 3, (64, nv))), _dev(rng.uniform(-3, 3, (64, nv)))).cpu().numpy()
        assert (z == 0).all()


@pytest.mark.gpu
def test_gpu_velocity_norm_terms_bit_equal_frame_velocity(ta):
    m = model_of("arm7_gripper.urdf")                            # fingers unlocked: prismatic bodies on the chain
    rng = np.random.RandomState(8)
    M = 3000
    q, qs = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(2))
    A = rng.randn(6, 6)
    for S in (A @ A.T, A, np.diag(rng.uniform(0, 2, 6))):          # symmetric, general, diagonal
        for link, ref in (("finger_left", "local"), ("camera", "world"), ("hand", "local_world_aligned")):
            f = m.frame(link, reference_frame=ref, **OFFSET)
            v = f(q, qs).cpu().numpy()
            b = f.velocity_norm_terms(q, qs, S).cpu().numpy()
            assert np.array_equal(b, kr.quad_form(S, v)), (link, ref)
    # NaN in, NaN out, nothing else touched
    m6 = model_of("arm6.urdf")
    f = m6.frame("flange", **OFFSET)
    q, qs = rng.uniform(-2, 2, (2, 64, 6))
    qn, qsn = q.copy(), qs.copy()
    qn[5, 2] = np.nan
    qsn[9, 0] = np.nan
    v, vn = f(q, qs), f(qn, qsn)
    bn = f.velocity_norm_terms(_dev(qn), _dev(qsn), np.eye(6)).cpu().numpy()
    assert np.isnan(vn[[5, 9]]).all() and np.isnan(bn[[5, 9]]).all()
    keep = np.ones(64, bool)
    keep[[5, 9]] = False
    assert np.array_equal(vn[keep], v[keep]) and np.isfinite(bn[keep]).all()


def _assert_solution(got, ref_K, ref_sd, st, ref_st):
    assert st == ref_st
    if ref_st == 0:
        np.testing.assert_allclose(got[0], ref_K, rtol=1e-8, atol=1e-9)
        np.testing.assert_allclose(got[1], ref_sd, rtol=1e-8, atol=1e-9)


def _golden_frame(g, robot, m):
    return m.frame(str(g[robot + "/link"]), xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"],
                   reference_frame=str(g[robot + "/ref"]))


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("cartesian_velocity")
    m = model_of(name, locked)
    f = _golden_frame(g, robot, m)
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim, limit, S = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "limit", "S"))
    B, G = way.shape[0], len(grid)
    path = ta.BatchSplineInterpolator(ss, way)
    q, qs = (path.eval_device(_dev(grid), o).reshape(-1, m.nv) for o in (0, 1))
    b = f.velocity_norm_terms(q, qs, S).cpu().numpy().reshape(B, G)
    for i in range(B):                                            # b against v^T S v of the 50-digit velocities
        close(b[i], g[robot + "/b"][i], 1e-12)
    for scheme in (0, 1):
        for i in range(B):                                        # single-path TOPPRA takes the device route too
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                       ta.constraint.JointAccelerationConstraint(alim[i], discretization_scheme=scheme),
                                       ta.constraint.CartesianVelocityNorm(f, S, limit[i], discretization_scheme=scheme)],
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), g["%s/s%d/K" % (robot, scheme)][i], g["%s/s%d/sd" % (robot, scheme)][i], st,
                             g["%s/s%d/status" % (robot, scheme)][i])
        h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            ta.constraint.CartesianVelocityNorm(f, S, limit, discretization_scheme=scheme)],
                           path, grid).compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), g["%s/s%d/K" % (robot, scheme)][i],
                             g["%s/s%d/sd" % (robot, scheme)][i], h["status"][i], g["%s/s%d/status" % (robot, scheme)][i])


def _problems(B, nv, seed, velocity):
    rng = np.random.RandomState(seed)
    way = np.cumsum(rng.uniform(-0.7, 0.7, (B, 5, nv)), axis=1)
    vel = np.where(np.isfinite(velocity), velocity, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    al = rng.uniform(6, 10, (B, nv))
    return np.linspace(0, 1, 5), way, vlim, np.stack([-al, al], axis=-1)


def _active_limits(ta, f, S, path, grid, vlim, alim, share=0.5):
    """Per path: `share` of the largest b sd^2 of the solution without the speed limit (so that it is active), and b."""
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                       path, grid).compute_parameterization(0, 0).to_host()
    d = _dev(grid)
    b = f.velocity_norm_terms(*(path.eval_device(d, o).reshape(-1, f.nv) for o in (0, 1)), S)
    b = b.reshape(path.B, -1).cpu().numpy()
    top = np.max(np.where(np.isfinite(h["sd"]), b * h["sd"] ** 2, -np.inf), axis=1)
    return share * np.where(np.isfinite(top) & (top > 0), top, 1.0), b


@pytest.mark.gpu
def test_gpu_256_paths_per_path_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _problems(B, nv, 17, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    limit, b_dev = _active_limits(ta, f, S, path, grid, vlim, alim)
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
                        ta.constraint.CartesianVelocityNorm(f, S, limit)], path, grid).compute_parameterization(0, 0).to_host()
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1))
        bv = kr.quad_form(S, kr.frame_velocity_packed(m.packed, f.packed, q, qs))
        row = np.stack((np.zeros(G), bv, np.full(G, 0.0 - limit[i])), axis=1)[:, :, None]
        o = orc.solve_rows(np.concatenate((lin["rows"], row), axis=2), lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            speed = b_dev[i] * h["sd"][i] ** 2                   # the constraint's meaning on the solved profile
            assert (speed <= limit[i] * (1 + 1e-9)).all()
            n_active += int(speed.max() >= limit[i] * (1 - 1e-6))
    assert n_ok > 0.9 * B and n_active > 0.9 * n_ok


def _cart_cons(ta, f, S, vlim, alim, limit, scheme=0):
    return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
            ta.constraint.CartesianVelocityNorm(f, S, limit, discretization_scheme=scheme)]


def _eq(x, y):
    return np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    f = m.frame("hand", reference_frame="local", **OFFSET)
    A = np.random.RandomState(2).randn(6, 6)
    S = A @ A.T / 6
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, nv, 23, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    limit, _ = _active_limits(ta, f, S, path, np.linspace(0, 1, 100), vlim, alim)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim, alim, limit), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim[i:i + 1], alim[i:i + 1], limit[i:i + 1]),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim, alim, limit, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim, alim, limit, scheme), path, grid, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the host route (the frame as a plain numpy callback) equals the
    # device route.  v^T S v with one non-zero entry of S is exact in any summation order, so numpy's dot on the host
    # and the kernel's fixed order agree bit for bit there.
    S1 = np.zeros((6, 6))
    S1[1, 1] = 1.0
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cart_cons(ta, f, S, vlim[i], alim[i], limit[i], scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim[i:i + 1], alim[i:i + 1], limit[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0).to_host()
            assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])
            lim1 = 0.3 * limit[i]
            dev = ta.algorithm.TOPPRA(_cart_cons(ta, f, S1, vlim[i], alim[i], lim1, scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            host_c = ta.constraint.CartesianVelocityNorm(lambda q, qd: f(q, qd), S1, lim1, dof=nv,
                                                         discretization_scheme=scheme)
            host = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                        ta.constraint.JointAccelerationConstraint(alim[i]), host_c], sp,
                                       gridpoints=grid, solver_wrapper="seidel")
            rd, rh = (x.compute_parameterization(0, 0, return_data=True) for x in (dev, host))
            for a, b in zip(rd, rh):
                assert _eq(a, b)
            assert rd[1] is not None
    # the varying form with a frame keeps the single-path host route
    vary = ta.constraint.CartesianVelocityNorm(f, velocity_limit=lambda s: (S, limit[0]))
    with pytest.raises(NotImplementedError, match="no batched device implementation"):
        ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), vary], path, grid).compute_parameterization(0, 0)


@pytest.mark.gpu
def test_gpu_quintic_piecewise_poly_path(ta):
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1), reference_frame="world")
    S = np.diag([1.0, 1.0, 1.0, 0.01, 0.01, 0.01])
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(21)
    coeffs = rng.uniform(-0.4, 0.4, (B, k, nseg, nv))
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    limit, b = _active_limits(ta, f, S, path, grid, vlim, alim)
    h = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim, alim, limit), path, grid).compute_parameterization(0, 0).to_host()
    assert (h["status"] == 0).sum() >= B // 2
    for i in range(B):
        one = ta.BatchTOPPRA(_cart_cons(ta, f, S, vlim[i:i + 1], alim[i:i + 1], limit[i:i + 1]),
                             ta.BatchPiecewisePolyPath(breaks, coeffs[i:i + 1]), grid).compute_parameterization(0, 0)
        one = one.to_host()
        for key in ("K", "sd", "sdd", "status"):
            assert _eq(h[key][i], one[key][0]), key
        if h["status"][i] == 0:
            speed = b[i] * h["sd"][i] ** 2
            assert (speed <= limit[i] * (1 + 1e-9)).all() and speed.max() >= limit[i] * (1 - 1e-6)


@pytest.mark.gpu
def test_gpu_with_joint_torque_constraint_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 32, 150, 6
    ss, way, vlim, alim = _problems(B, nv, 29, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    limit, _ = _active_limits(ta, f, S, path, grid, vlim, alim, share=0.7)
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    cons = _cart_cons(ta, f, S, vlim, alim, limit) + [ta.constraint.JointTorqueConstraint(m, taulim, fric)]
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    F = np.vstack((np.eye(nv), -np.eye(nv)))
    gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        bv = kr.quad_form(S, kr.frame_velocity_packed(m.packed, f.packed, q, qs))
        cart = np.stack((np.zeros(G), bv, np.full(G, 0.0 - limit[i])), axis=1)[:, :, None]
        av, btv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        torque = np.stack((av.dot(F.T), btv.dot(F.T), cv.dot(F.T) - gt), axis=1)   # JointTorqueConstraint: collocation
        rows = np.concatenate((lin["rows"], cart, torque), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok > 0.8 * B
