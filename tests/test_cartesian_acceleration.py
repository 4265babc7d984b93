"""Frame accelerations of a rigid-body model on the GPU and the Cartesian acceleration limit of a frame
(RigidBodyFrame.acceleration / acceleration_terms, CartesianAccelerationConstraint; libtoppra_b200_dyn.so:
tbd_frame_acceleration, tbd_acceleration_terms).

CPU:
  * the float64 numpy double of tests/kin_acc_ref.py equals the 50-digit classical accelerations of the RAW URDF tree to
    1e-13 of the state's scale: every link of both fixtures, locked and unlocked (prismatic fingers on the chain), both
    allowed reference frames, with and without a tool offset;
  * every ValueError; the ctypes prototypes of the new entries against include/toppra_b200_dyn.h; each argument check of
    the two entries returns its TB_ERR_* from the real library.
GPU:
  * tbd_frame_acceleration on random trees (1 to 16 bodies) against the 50-digit reference and the numpy double within
    1e-12; a frame on the base gives exact zeros;
  * tbd_acceleration_terms equals tbd_frame_acceleration at (q, 0, q') and (q, q', q'') after the column selection, bit
    for bit; NaN in one point touches no other;
  * the reference golden (tests/golden/cartesian_acceleration.npz, make_golden_cartesian_accel.py): TOPPRA and
    BatchTOPPRA within |dK| <= 1e-9 + 1e-8 |K| (the cfg-3 tolerance), equal statuses; 256 paths with per-path limits
    against the oracle fed with rows from the numpy double, same tolerance; the frame accelerations of the solved
    profiles are within the limits, which are active;
  * ragged vs per-path grids, chunked vs unchunked, TOPPRA vs BatchTOPPRA at B = 1, the reference-style
    SecondOrderConstraint with the frame as a numpy callback vs CartesianAccelerationConstraint: bit-equal;
    BatchTOPPRAsd, a quintic BatchPiecewisePolyPath, and the constraint next to JointTorqueConstraint and
    CartesianVelocityNorm against the oracle."""
import ctypes
import os

import numpy as np
import pytest

import kin_acc_ref as kar
import kin_ref as kr
import rnea_ref as rr
from dyn_common import (CASES, DYN_LIB, FakePath, LOCKED, OFFSET, TB_ERR_ARG, TB_ERR_UNSUPPORTED, close, model_of, urdf,
                        _assert_one_terms_launch, _assert_solution, _dev, _dyn_header, _eq, _gpu_present,
                        _model_from_packed, _offset_spec, _problems)


# ==== CPU: numpy double vs the 50-digit reference, errors, C-ABI =====================================================
@pytest.mark.parametrize("name,locked", CASES)
def test_numpy_double_matches_mp_reference(name, locked):
    m = model_of(name, locked)
    mp = rr.MpRobot.from_urdf(urdf(name), locked)
    rng = np.random.RandomState(m.nv + 57)
    for _ in range(2):
        q, qd, qdd = rng.uniform(-2, 2, (3, m.nv))
        spec, frames = {}, {}
        for link in m.frames:
            for ref in kar.REFERENCE_FRAMES:
                for o, off in enumerate((None, OFFSET)):
                    spec[(link, ref, o)] = (link,) + _offset_spec(off)
                    frames[(link, ref, o)] = m.frame(link, reference_frame=ref, **(off or {}))
        want = kar.mp_accelerations(mp, q, qd, qdd, spec)
        for key, f in frames.items():
            got = kar.frame_acceleration_packed(m.packed, f.packed, q, qd, qdd)[0]
            close(got, [float(x) for x in want[key][key[1]]], 1e-13)
        # the terms double: a = acc(q, 0, q'), b = acc(q, q', q''), columns in increasing order
        f = frames[(sorted(m.frames)[-1], "local", 1)]
        a, b = kar.acceleration_terms_packed(m.packed, f.packed, q, qd, qdd, (4, 0, 2))
        assert np.array_equal(a[0], kar.frame_acceleration_packed(m.packed, f.packed, q, 0 * qd, qd)[0][[0, 2, 4]])
        assert np.array_equal(b[0], kar.frame_acceleration_packed(m.packed, f.packed, q, qd, qdd)[0][[0, 2, 4]])


def test_value_errors():
    from toppra_b200.constraint import CartesianAccelerationConstraint
    from toppra_b200.constraint.linear_constraint import RecordContext
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    lim = np.array([[-1.0, 1.0]] * 3)
    with pytest.raises(ValueError, match="world"):
        CartesianAccelerationConstraint(m.frame("flange", reference_frame="world"), lim)
    with pytest.raises(ValueError, match="world"):
        m.frame("flange", reference_frame="world").acceleration(np.zeros(6), np.zeros(6), np.zeros(6))
    with pytest.raises(ValueError, match="RigidBodyFrame"):
        CartesianAccelerationConstraint(lambda q, qd, qdd: np.zeros(3), lim)
    for comps in ((), (0, 0, 1), (0, 6), (-1, 2), (0.0, 1.0), (0.5,)):
        with pytest.raises(ValueError, match="components"):
            CartesianAccelerationConstraint(f, np.zeros((max(len(comps), 1), 2)), components=comps)
    with pytest.raises(ValueError, match=r"expected \(3, 2\) or \(B, 3, 2\)"):
        CartesianAccelerationConstraint(f, lim[:2])
    with pytest.raises(ValueError, match=r"expected \(2, 2\)"):
        CartesianAccelerationConstraint(f, lim, components=(3, 5))
    with pytest.raises(ValueError, match="alim has shape"):
        CartesianAccelerationConstraint(f, lim.T)
    with pytest.raises(ValueError, match="alim has shape"):
        CartesianAccelerationConstraint(f, [1.0, 2.0])
    for bad in (np.nan, np.inf, -np.inf):
        x = lim.copy()
        x[1, 0] = bad
        with pytest.raises(ValueError, match="finite"):
            CartesianAccelerationConstraint(f, x)
    with pytest.raises(ValueError, match="lower limit exceeds"):
        CartesianAccelerationConstraint(f, [[-1.0, 1.0], [0.5, 0.4], [-1.0, 1.0]])
    with pytest.raises(ValueError, match="lower limit exceeds"):
        CartesianAccelerationConstraint(f, np.tile(lim, (4, 1, 1)) * np.array([1, 1, 1, -1])[:, None, None])
    grid = np.linspace(0, 1, 10)
    c = CartesianAccelerationConstraint(f, np.tile(lim, (3, 1, 1)))
    assert c.dof == 6 and c.components == (0, 1, 2)
    assert c.num_rows(RecordContext(FakePath(3, 6), grid, grid)) == 12                 # interpolation: 2 x 2k
    assert CartesianAccelerationConstraint(f, lim[:1], components=(5,), discretization_scheme=0).num_rows(
        RecordContext(FakePath(7, 6), grid, grid)) == 2
    with pytest.raises(ValueError, match=r"expected \(3, 2\) or \(4, 3, 2\)"):
        c.num_rows(RecordContext(FakePath(4, 6), grid, grid))
    with pytest.raises(ValueError, match=r"\(5, 3, 2\)"):                              # a chunk of a 5-path batch
        c.num_rows(RecordContext(FakePath(2, 6), grid, grid, None, 0, 2, 5))
    with pytest.raises(ValueError, match="Wrong dimension"):                           # a model with another nv
        c.num_rows(RecordContext(FakePath(3, 7), grid, grid))
    # alim rows follow `components` as given; the rows of the constraint come in increasing component order
    u = CartesianAccelerationConstraint(f, [[-5.0, 5.0], [-1.0, 2.0]], components=(4, 1))
    assert u.components == (1, 4)
    assert np.array_equal(u._eye_form[0], [2.0, 5.0, 1.0, 5.0])


def test_dyn_header_prototypes_of_acceleration_entries():
    from toppra_b200 import _lib_dyn
    declared = _dyn_header()
    assert declared["tbd_frame_acceleration"] == ["ptr", "int", "ptr", "int", "ptr", "ptr", "ptr", "ptr", "ptr"]
    assert declared["tbd_acceleration_terms"] == ["ptr", "int", "ptr", "int", "int", "ptr", "ptr", "ptr", "ptr", "ptr",
                                                  "ptr"]
    for name in ("tbd_frame_acceleration", "tbd_acceleration_terms"):
        argtypes, restype = _lib_dyn._PROTOS[name]
        assert [{ctypes.c_int: "int", ctypes.c_double: "double"}.get(t, "ptr") for t in argtypes] == declared[name]
        assert restype is ctypes.c_int


# host addresses stand in for device arrays: a case that slipped through the validation would launch a kernel on them
@pytest.mark.skipif(_gpu_present(), reason="validation-only calls with host addresses: run without a GPU")
def test_acceleration_argument_checks():
    if not os.path.exists(DYN_LIB):
        pytest.skip("libtoppra_b200_dyn.so is not built")
    from toppra_b200 import _lib, _lib_dyn
    lib = _lib_dyn.load()
    mem = np.zeros(1 << 12)
    d = ctypes.c_void_p(mem.ctypes.data)
    m = model_of("arm6.urdf")
    good_frame = m.frame("flange", **OFFSET).packed

    def rc(model=m.packed, frame=good_frame, nv=6, M=4, null=None, components=7):
        host = [np.array(x, dtype=np.float64) for x in (model, frame)]
        ptr = [ctypes.c_void_p(h.ctypes.data) for h in host]
        fa = [ptr[0], nv, ptr[1], M, d, d, d, d]
        at = [ptr[0], nv, ptr[1], components, M, d, d, d, d, d]
        if null is not None:                   # index into fa; at has `components` inserted before M
            fa[null] = None
            at[null if null < 3 else null + 1] = None
        r2 = lib.tbd_acceleration_terms(*at, None)
        if components != 7:
            assert r2 == 0 or _lib.load().tb_last_error()
            return r2
        r1 = lib.tbd_frame_acceleration(*fa, None)
        assert r1 == r2, (r1, r2)
        assert r1 == 0 or _lib.load().tb_last_error()
        return r1

    for k in (0, 2, 4, 5, 6, 7):
        assert rc(null=k) == TB_ERR_ARG
    assert rc(null=None, components=0) == TB_ERR_ARG and rc(components=64) == TB_ERR_ARG
    assert rc(components=-1) == TB_ERR_ARG
    assert rc(M=0) == TB_ERR_ARG and rc(M=-3) == TB_ERR_ARG
    assert rc(nv=0) == TB_ERR_UNSUPPORTED and rc(np.r_[m.packed, np.zeros(27 * 11)], nv=17) == TB_ERR_UNSUPPORTED
    bad_model = m.packed.copy()
    bad_model[3 + 27 * 2] = 2.0                                 # parent[k] >= k
    assert rc(bad_model) == TB_ERR_ARG
    for j, value in ((0, 6.0), (0, -2.0), (13, 3.0), (5, np.nan), (11, np.inf)):   # bad frames
        f = good_frame.copy()
        f[j] = value
        assert rc(frame=f) == TB_ERR_ARG
    world = m.frame("flange", reference_frame="world").packed
    assert rc(frame=world) == TB_ERR_UNSUPPORTED
    assert b"world" in _lib.load().tb_last_error()


# ==== GPU ============================================================================================================
@pytest.fixture(scope="module")
def ta():
    import toppra_b200
    return toppra_b200


@pytest.mark.gpu
@pytest.mark.parametrize("nv", [1, 2, 3, 5, 8, 12, 16])
def test_gpu_frame_acceleration_random_trees_vs_mp(ta, nv):
    from toppra_b200.dynamics import rpy_matrix
    rng = np.random.RandomState(700 + nv)
    m = _model_from_packed(ta, rr.random_tree(rng, nv))
    mp = rr.MpRobot.from_packed(m.packed)
    P = 2 if nv <= 8 else 1
    q, qd, qdd = (rng.uniform(-2, 2, (P, nv)) for _ in range(3))
    for ref in kar.REFERENCE_FRAMES:
        for k in sorted({nv - 1, int(rng.randint(nv))}):
            off = dict(xyz=tuple(rng.randn(3) * 0.2), rpy=tuple(rng.uniform(-3, 3, 3)))
            f = m.frame("body%d" % k, reference_frame=ref, **off)
            acc = f.acceleration(_dev(q), _dev(qd), _dev(qdd)).cpu().numpy()
            spec = {0: ("b%d" % k, rpy_matrix(off["rpy"]), np.asarray(off["xyz"]))}
            for i in range(P):
                want = kar.mp_accelerations(mp, q[i], qd[i], qdd[i], spec)[0][ref]
                close(acc[i], [float(x) for x in want], 1e-12)
            Q, QD, QDD = (rng.uniform(-3, 3, (512, nv)) for _ in range(3))
            got = f.acceleration(_dev(Q), _dev(QD), _dev(QDD)).cpu().numpy()
            want = kar.frame_acceleration_packed(m.packed, f.packed, Q, QD, QDD)
            assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
            assert np.array_equal(f.acceleration(Q[3], QD[3], QDD[3]), got[3])   # numpy (nv,): a device round trip
            assert np.array_equal(f.acceleration(Q[:5], QD[:5], QDD[:5]), got[:5])
    for ref in kar.REFERENCE_FRAMES:                                              # a frame on the base does not move
        base = ta.RigidBodyFrame(m, "base", -1, rpy_matrix((0.2, 0.1, -0.4)), (0.3, -0.1, 0.5), ref)
        z = base.acceleration(*(_dev(rng.uniform(-3, 3, (64, nv))) for _ in range(3))).cpu().numpy()
        assert (z == 0).all()


@pytest.mark.gpu
def test_gpu_acceleration_terms_bit_equal_frame_acceleration(ta):
    import torch
    m = model_of("arm7_gripper.urdf")                            # fingers unlocked: prismatic bodies on the chain
    rng = np.random.RandomState(9)
    M = 3000
    q, qs, qss = (_dev(rng.uniform(-2, 2, (M, m.nv))) for _ in range(3))
    zero = torch.zeros_like(q)
    for link, ref in (("finger_left", "local"), ("camera", "local_world_aligned"), ("hand", "local")):
        f = m.frame(link, reference_frame=ref, **OFFSET)
        acc0 = f.acceleration(q, zero, qs).cpu().numpy()
        acc1 = f.acceleration(q, qs, qss).cpu().numpy()
        for comps in ((0, 1, 2), (0, 1, 2, 3, 4, 5), (5,), (1, 3), (4, 0, 2)):
            a, b = f.acceleration_terms(q, qs, qss, comps)
            cols = sorted(comps)
            assert a.shape == (M, len(cols)) and b.shape == (M, len(cols))
            assert np.array_equal(a.cpu().numpy(), acc0[:, cols]), (link, comps)
            assert np.array_equal(b.cpu().numpy(), acc1[:, cols]), (link, comps)
    # NaN in one point leaves every other point as it was
    f = model_of("arm6.urdf").frame("flange", **OFFSET)
    q, qs, qss = rng.uniform(-2, 2, (3, 64, 6))
    qn, qsn, qssn = q.copy(), qs.copy(), qss.copy()
    qn[5, 2] = np.nan
    qsn[9, 0] = np.nan
    qssn[17, 4] = np.nan
    acc, accn = f.acceleration(q, qs, qss), f.acceleration(qn, qsn, qssn)
    a, b = f.acceleration_terms(_dev(q), _dev(qs), _dev(qss), range(6))
    an, bn = (x.cpu().numpy() for x in f.acceleration_terms(_dev(qn), _dev(qsn), _dev(qssn), range(6)))
    assert np.isnan(accn[[5, 9, 17]]).any(axis=1).all() and np.isnan(bn[[5, 9, 17]]).any(axis=1).all()
    assert np.isnan(an[[5, 9]]).any(axis=1).all()
    keep = np.ones(64, bool)
    keep[[5, 9, 17]] = False
    assert np.array_equal(accn[keep], acc[keep])
    assert np.array_equal(an[keep], a.cpu().numpy()[keep]) and np.array_equal(bn[keep], b.cpu().numpy()[keep])


def _cons(ta, f, climit, comps, vlim, alim, scheme=1):
    return [ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim),
            ta.constraint.CartesianAccelerationConstraint(f, climit, comps, discretization_scheme=scheme)]


def _terms(f, comps, path, grid):
    """a, b (B, G, k) of the frame on the device path at the grid."""
    d = _dev(grid)
    a, b = f.acceleration_terms(*(path.eval_device(d, o).reshape(-1, f.nv) for o in (0, 1, 2)), comps)
    return a.reshape(path.B, len(grid), -1).cpu().numpy(), b.reshape(path.B, len(grid), -1).cpu().numpy()


def _active_limits(ta, f, comps, path, grid, vlim, alim, share=0.5):
    """Per path and component: `share` of the largest |a u + b x| of the solution without the acceleration limit (so
    that the limit is active), as (B, k, 2) [lower, upper]; and a, b."""
    h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim), ta.constraint.JointAccelerationConstraint(alim)],
                       path, grid).compute_parameterization(0, 0).to_host()
    a, b = _terms(f, comps, path, grid)
    val = np.abs(a[:, :-1] * h["sdd"][:, :, None] + b[:, :-1] * (h["sd"][:, :-1] ** 2)[:, :, None])
    top = np.max(np.where(np.isfinite(val), val, -np.inf), axis=1)
    top = share * np.where(np.isfinite(top) & (top > 0), top, 1.0)
    return np.stack([-top, top], axis=-1), a, b


def _meaning(a, b, sd, sdd, lim, grid, interp=True):
    """The frame acceleration of the solved profile at the gridpoints, acc = a u + b x: at the start of every stage
    (u_i, x_i) and, under interpolation, at its end (u_i, x_i + 2 ds u_i; the forward pass may store x_{i+1} up
    to 1e-8 below that).  Within the limits; returns whether a limit is reached."""
    x = sd[:-1] ** 2
    vals = [a[:-1] * sdd[:, None] + b[:-1] * x[:, None]]
    if interp:
        vals.append(a[1:] * sdd[:, None] + b[1:] * (x + 2 * np.diff(grid) * sdd)[:, None])
    scale = np.abs(lim).max(axis=1)
    active = False
    for v in vals:
        assert (v <= lim[:, 1] + 1e-9 * scale).all() and (v >= lim[:, 0] - 1e-9 * scale).all()
        active |= bool(((v >= lim[:, 1] - 1e-6 * scale) | (v <= lim[:, 0] + 1e-6 * scale)).any())
    return active


def _oracle_rows(a, b, lim, grid, interp):
    """(G, 3, R) rows a F^T, b F^T, c F^T - g of the constraint (F = [I; -I], c = 0) for the oracle."""
    from toppra_b200.constraint.linear_constraint import canlinear_colloc_to_interpolate
    k = a.shape[1]
    F = np.vstack((np.eye(k), -np.eye(k)))
    g = np.concatenate((lim[:, 1], -lim[:, 0]))
    c = np.zeros_like(a)
    if interp:
        a, b, c, F, g = canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, grid, identical=True)[:5]
    return np.stack((a.dot(F.T), b.dot(F.T), c.dot(F.T) - g), axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("robot,name,locked", [("arm6", "arm6.urdf", None), ("arm7", "arm7_gripper.urdf", LOCKED)])
def test_gpu_reference_golden(ta, golden, robot, name, locked):
    g = golden("cartesian_acceleration")
    m = model_of(name, locked)
    f = m.frame(str(g[robot + "/link"]), xyz=g[robot + "/xyz"], rpy=g[robot + "/rpy"],
                reference_frame=str(g[robot + "/ref"]))
    comps = tuple(int(j) for j in g[robot + "/components"])
    ss, grid = g["ss"], g["grid"]
    way, vlim, alim, climit = (g[robot + "/" + k] for k in ("way", "vlim", "alim", "climit"))
    B = way.shape[0]
    path = ta.BatchSplineInterpolator(ss, way)
    a, b = _terms(f, comps, path, grid)
    for i in range(B):                                            # against the 50-digit accelerations
        close(a[i], g[robot + "/a"][i], 1e-12)
        close(b[i], g[robot + "/b"][i], 1e-12)
    for scheme in (0, 1):
        key = lambda x, i: g["%s/s%d/%s" % (robot, scheme, x)][i]  # noqa: E731
        for i in range(B):                                        # single-path TOPPRA takes the device route too
            one = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                       ta.constraint.JointAccelerationConstraint(alim[i], discretization_scheme=scheme),
                                       ta.constraint.CartesianAccelerationConstraint(f, climit[i], comps,
                                                                                     discretization_scheme=scheme)],
                                      ta.SplineInterpolator(ss, way[i]), gridpoints=grid, solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            st = list(ta.algorithm.ParameterizationReturnCode).index(one.problem_data.return_code)
            _assert_solution((K, sd), key("K", i), key("sd", i), st, key("status", i))
        h = ta.BatchTOPPRA([ta.constraint.JointVelocityConstraint(vlim),
                            ta.constraint.JointAccelerationConstraint(alim, discretization_scheme=scheme),
                            ta.constraint.CartesianAccelerationConstraint(f, climit, comps, discretization_scheme=scheme)],
                           path, grid).compute_parameterization(0, 0).to_host()
        for i in range(B):
            _assert_solution((h["K"][i], h["sd"][i]), key("K", i), key("sd", i), h["status"][i], key("status", i))


@pytest.mark.gpu
def test_gpu_256_paths_per_path_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    comps = (0, 1, 2)
    B, G, nv = 256, 200, 6
    ss, way, vlim, alim = _problems(B, nv, 31, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    climit, a_dev, b_dev = _active_limits(ta, f, comps, path, grid, vlim, alim)
    h = ta.BatchTOPPRA(_cons(ta, f, climit, comps, vlim, alim), path, grid).compute_parameterization(0, 0).to_host()
    n_ok = n_active = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b = kar.acceleration_terms_packed(m.packed, f.packed, q, qs, qss, comps)
        rows = np.concatenate((lin["rows"], _oracle_rows(a, b, climit[i], grid, True)), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        if h["status"][i] == 0:
            n_ok += 1
            n_active += _meaning(a_dev[i], b_dev[i], h["sd"][i], h["sdd"][i], climit[i], grid)
    assert n_ok > 0.9 * B and n_active > 0.9 * n_ok, (n_ok, n_active)


@pytest.mark.gpu
def test_gpu_ragged_chunked_and_single_path_bit_equal(ta):
    m = model_of("arm7_gripper.urdf", LOCKED)
    f = m.frame("hand", reference_frame="local", **OFFSET)
    comps = (0, 1, 2, 3, 4, 5)
    B, nv = 12, m.nv
    ss, way, vlim, alim = _problems(B, nv, 37, m.velocity_limit)
    path = ta.BatchSplineInterpolator(ss, way)
    climit, _, _ = _active_limits(ta, f, comps, path, np.linspace(0, 1, 100), vlim, alim)
    # ragged (proposed per-path grids) against each path solved alone on its own grid
    rag = ta.BatchTOPPRA(_cons(ta, f, climit, comps, vlim, alim), path, None)
    hr = rag.compute_parameterization(0, 0).to_host()
    glen, grids = rag.glen.cpu().numpy(), rag.d_grid.cpu().numpy()
    assert len(set(glen.tolist())) > 1
    for i in range(B):
        n = int(glen[i])
        one = ta.BatchTOPPRA(_cons(ta, f, climit[i:i + 1], comps, vlim[i:i + 1], alim[i:i + 1]),
                             ta.BatchSplineInterpolator(ss, way[i:i + 1]), grids[i, :n]).compute_parameterization(0, 0)
        one = one.to_host()
        assert hr["status"][i] == one["status"][0]
        assert _eq(hr["K"][i, :n], one["K"][0]) and _eq(hr["sd"][i, :n], one["sd"][0])
    # chunked against unchunked on a common grid
    grid = np.linspace(0, 1, 150)
    for scheme in (0, 1):
        whole = ta.BatchTOPPRA(_cons(ta, f, climit, comps, vlim, alim, scheme), path, grid)
        per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
        parts = ta.BatchTOPPRA(_cons(ta, f, climit, comps, vlim, alim, scheme), path, grid,
                               max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5
        hw, hp = whole.compute_parameterization(0, 0).to_host(), parts.compute_parameterization(0, 0).to_host()
        for k in ("K", "sd", "sdd", "status"):
            assert _eq(hw[k], hp[k]), k
    # single-path TOPPRA equals BatchTOPPRA at B = 1; the reference-style SecondOrderConstraint with the frame as a
    # numpy callback (examples-old/cartesian_accel.py) equals CartesianAccelerationConstraint: the general-F rows of
    # [I; -I] and the eye-form rows are the same numbers
    lin3 = (0, 1, 2)
    F = np.vstack((np.eye(3), -np.eye(3)))
    for i in range(3):
        sp = ta.SplineInterpolator(ss, way[i])
        for scheme in (0, 1):
            one = ta.algorithm.TOPPRA(_cons(ta, f, climit[i], comps, vlim[i], alim[i], scheme), sp, gridpoints=grid,
                                      solver_wrapper="seidel")
            sdd, sd, _, K = one.compute_parameterization(0, 0, return_data=True)
            hb = ta.BatchTOPPRA(_cons(ta, f, climit[i:i + 1], comps, vlim[i:i + 1], alim[i:i + 1], scheme),
                                ta.BatchSplineInterpolator(ss, way[i:i + 1]), grid).compute_parameterization(0, 0).to_host()
            assert _eq(K, hb["K"][0]) and _eq(sd, hb["sd"][0]) and _eq(sdd, hb["sdd"][0])
            lim3 = climit[i, :3]
            gv = np.concatenate((lim3[:, 1], -lim3[:, 0]))
            ref_c = ta.constraint.SecondOrderConstraint(lambda q, qd, qdd: f.acceleration(q, qd, qdd)[:3],
                                                        lambda _: F, lambda _: gv, nv, discretization_scheme=scheme)
            runs = []
            for c in (ref_c, ta.constraint.CartesianAccelerationConstraint(f, lim3, lin3, discretization_scheme=scheme)):
                inst = ta.algorithm.TOPPRA([ta.constraint.JointVelocityConstraint(vlim[i]),
                                            ta.constraint.JointAccelerationConstraint(alim[i]), c], sp,
                                           gridpoints=grid, solver_wrapper="seidel")
                runs.append(inst.compute_parameterization(0, 0, return_data=True))
            for x, y in zip(*runs):
                assert _eq(x, y)
            assert runs[0][1] is not None


@pytest.mark.gpu
def test_gpu_toppra_sd_and_quintic_piecewise_poly_path(ta):
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    comps = (0, 1, 2)
    B, nv, nseg, k = 6, 6, 3, 6
    rng = np.random.RandomState(41)
    coeffs = rng.uniform(-0.4, 0.4, (B, k, nseg, nv))
    breaks = np.linspace(0, 1, nseg + 1)
    path = ta.BatchPiecewisePolyPath(breaks, coeffs)
    grid = np.linspace(0, 1, 120)
    vel = np.where(np.isfinite(m.velocity_limit), m.velocity_limit, 3.0)
    vlim = np.tile(np.stack([-vel, vel], axis=1), (B, 1, 1))
    alim = np.tile(np.stack([-np.full(nv, 8.0), np.full(nv, 8.0)], axis=1), (B, 1, 1))
    climit, a, b = _active_limits(ta, f, comps, path, grid, vlim, alim)
    h = ta.BatchTOPPRA(_cons(ta, f, climit, comps, vlim, alim), path, grid).compute_parameterization(0, 0).to_host()
    assert (h["status"] == 0).sum() >= B // 2
    for i in range(B):
        one = ta.BatchTOPPRA(_cons(ta, f, climit[i:i + 1], comps, vlim[i:i + 1], alim[i:i + 1]),
                             ta.BatchPiecewisePolyPath(breaks, coeffs[i:i + 1]), grid).compute_parameterization(0, 0)
        one = one.to_host()
        for key in ("K", "sd", "sdd", "status"):
            assert _eq(h[key][i], one[key][0]), key
        if h["status"][i] == 0:
            assert _meaning(a[i], b[i], h["sd"][i], h["sdd"][i], climit[i], grid)
    # BatchTOPPRAsd, whole and in record chunks: half again the time-optimal duration (or the slowest profile), and the
    # acceleration limit holds on the blended profiles (a convex combination of (u, x) of two feasible profiles)
    ok = h["status"] == 0
    dur = np.array([np.sum(2 * np.diff(grid) / (s[:-1] + s[1:])) if o else 1.0 for s, o in zip(h["sd"], ok)])
    runs = []
    for chunk in (None, 2):
        sd_inst = ta.BatchTOPPRAsd(_cons(ta, f, climit, comps, vlim, alim), path, grid)
        if chunk:
            sd_inst = ta.BatchTOPPRAsd(_cons(ta, f, climit, comps, vlim, alim), path, grid,
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
        assert _meaning(a[i], b[i], sd[i], sdd[i], climit[i], grid) is not None
        got = np.sum(2 * np.diff(grid) / (sd[i, :-1] + sd[i, 1:]))
        want = min(1.5 * dur[i], slow[i])
        assert abs(got - want) <= 1e-4 * max(1.0, want), (got, want)


@pytest.mark.gpu
def test_gpu_with_torque_and_velocity_limits_vs_oracle(ta):
    from oracle import oracle as orc
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    comps = (0, 1, 2)
    S = np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    B, G, nv = 32, 150, 6
    ss, way, vlim, alim = _problems(B, nv, 43, m.velocity_limit)
    grid = np.linspace(0, 1, G)
    path = ta.BatchSplineInterpolator(ss, way)
    climit, _, _ = _active_limits(ta, f, comps, path, grid, vlim, alim, share=0.7)
    d = _dev(grid)
    bv = f.velocity_norm_terms(*(path.eval_device(d, o).reshape(-1, nv) for o in (0, 1)), S).reshape(B, G)
    speed = 0.8 * bv.max(dim=1).values.cpu().numpy()
    taulim = 0.45 * m.torque_limits()
    fric = 0.3 + 0.1 * np.arange(nv)
    cons = _cons(ta, f, climit, comps, vlim, alim) + [ta.constraint.JointTorqueConstraint(m, taulim, fric),
                                                      ta.constraint.CartesianVelocityNorm(f, S, speed)]
    h = ta.BatchTOPPRA(cons, path, grid).compute_parameterization(0, 0).to_host()
    F = np.vstack((np.eye(nv), -np.eye(nv)))
    gt = np.concatenate((taulim[:, 1], -taulim[:, 0]))
    n_ok = 0
    for i in range(B):
        c = orc.cubic_spline_fit(ss, way[i])
        lin = orc.solve_velacc(c, ss, grid, vlim[i], alim[i], True, 0, 0, want_rows=True)
        q, qs, qss = (orc.ppoly_eval(c, ss, grid, o) for o in (0, 1, 2))
        a, b = kar.acceleration_terms_packed(m.packed, f.packed, q, qs, qss, comps)
        av, btv, cv = rr.torque_terms_packed(m.packed, q, qs, qss, fric)
        torque = np.stack((av.dot(F.T), btv.dot(F.T), cv.dot(F.T) - gt), axis=1)   # JointTorqueConstraint: collocation
        vq = kr.quad_form(S, kr.frame_velocity_packed(m.packed, f.packed, q, qs))
        cart_v = np.stack((np.zeros(G), vq, np.full(G, 0.0 - speed[i])), axis=1)[:, :, None]
        rows = np.concatenate((lin["rows"], _oracle_rows(a, b, climit[i], grid, True), torque, cart_v), axis=2)
        o = orc.solve_rows(rows, lin["xbound"], grid, 0.0, 0.0)
        _assert_solution((h["K"][i], h["sd"][i]), o["K"], o["sd"], h["status"][i], o["status"])
        n_ok += int(o["status"] == 0)
    assert n_ok > 0.8 * B


@pytest.mark.gpu
def test_gpu_one_terms_launch_per_batch_or_chunk(ta, monkeypatch):
    m = model_of("arm6.urdf")
    f = m.frame("flange", xyz=(0, 0, 0.1))
    ss, way, vlim, alim = _problems(10, 6, 31, m.velocity_limit)
    climit = np.tile([[-4.0, 4.0]], (3, 1))
    _assert_one_terms_launch(ta, monkeypatch, lambda: _cons(ta, f, climit, (0, 1, 2), vlim, alim),
                             ta.BatchSplineInterpolator(ss, way), np.linspace(0, 1, 80), "tbd_acceleration_terms")
