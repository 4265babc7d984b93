"""Long paths: 15 to 1000 knots through every kernel branch that depends on the path length.

Planners hand TOPP-RA dense waypoint lists, and several kernels switch code paths once a path gets long:
  K0 spline_fit_kernel          scratch in thread-local arrays up to LOCAL_KNOTS = 16 knots, in the caller's workspace
                                [B*dof][7][n] above that (csrc/tb_spline.cu:18, 84-91)
  fused scan tb_scan_velacc     the derivative coefficients must fit in 16 KB, else BatchTOPPRA takes the record route
                                (csrc/tb_scan.cu:1157-1161, csrc/tb_api.cu:70, engine.velacc_fused_supported)
  fused row / forward threads   the segment index is carried from stage to stage, never searched: several breakpoints per
                                stage happen only when G < nseg (csrc/tb_scan.cu:529-549, csrc/tb_scan_fwd.cu:92-99)
  K1 coeff_velacc_kernel        derivative coefficients cached in shared memory while (nseg+1 + 5 nseg dof) * 8 <= 32 KB,
                                re-derived from global memory above (csrc/tb_coeff.cu:45-48, 65-67, 105-112, 492-495)
  find_interval                 binary search depth grows with nseg (csrc/tb_common.cuh)

CPU (no marker): the oracle against tests/golden/long_paths.npz (the unmodified reference and scipy, written by
tests/golden/make_golden_long.py) bit for bit; the switch formulas restated and the cases checked to straddle them; the
route choice of BatchTOPPRA on the engine double; the K0 workspace size query of the real library.
GPU (-m gpu): every kernel branch against the oracle or the oracle-backed engine double (tests/cpu_engine.py), bit for bit
with NaN equal to NaN.  The only tolerance is the one test_kernel_builds.case_second_order states for the trigonometric
rows of the device torque model (TRIG_ULPS).  The batched callers on long paths are in
tests/test_zzz_long_path_callers.py, which sorts after every test that reads torch.profiler."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import cpu_engine
from oracle import oracle as orc
from problems import LONG_SPACINGS, long_breaks, long_spline_data, long_waypoints

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "long_paths.npz")
TB_ERR_UNSUPPORTED = -2
LOCAL_KNOTS = 16                                   # csrc/tb_spline.cu:18
# the golden's cases (tests/golden/make_golden_long.py; restated: that script imports the reference)
FIT_N = (16, 17, 18, 33, 48, 49, 50, 114, 115, 116, 300, 1000)
FIT_HASHED = 300
FIT_BC = ("not-a-knot", "clamped", "natural", "first", "mixed", "periodic")
N_SOLVES = 11
CALLERS = (0, 4)
SD_FACTOR = 1.7
REACH = (0.0, 0.5)
PROPOSE = dict(max_err_threshold=1e-3, max_seg_length=0.1, min_nb_points=100)


# ---- the switches, restated from the C sources ---------------------------------------------------------------------------
def fused_fits(nseg, dof, interp):
    """csrc/tb_scan.cu:1157-1161 (and tb_api.cu:70): one LP row per lane (R + 2 <= 32) and the record of 6 derivative
    coefficients per (segment, joint) + breakpoints, rounded to an even count, within 16 KB."""
    R = (4 if interp else 2) * dof
    Wc = (nseg * dof * 6 + nseg + 2) & ~1
    return R + 2 <= 32 and Wc * 8 <= 16 * 1024


def k1_smem(nseg, dof):
    """csrc/tb_coeff.cu:492-493: K1 caches breakpoints + 5 derivative coefficients per (segment, joint) in shared memory."""
    return (nseg + 1 + nseg * dof * 5) * 8 <= 32 * 1024


def last_true(pred):
    n = 1
    while pred(n + 1):
        n += 1
    return n


FUSED_LAST = {dof: last_true(lambda n, d=dof: fused_fits(n, d, dof != 14)) for dof in (1, 3, 6, 7, 14)}
K1_LAST = {dof: last_true(lambda n, d=dof: k1_smem(n, d)) for dof in (1, 3, 6, 7, 14)}


# ---- helpers --------------------------------------------------------------------------------------------------------------
def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def first_diff(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    if a.shape != b.shape:
        return "shapes %s vs %s" % (a.shape, b.shape)
    bad = np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))))
    return "%d differ, first at %s: %r vs %r" % (len(bad), tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])]) if len(bad) \
        else "equal"


def assert_same(got, want, what):
    assert same(got, want), "%s: %s" % (what, first_diff(got, want))


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).digest(), dtype=np.uint8)


def host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def golden():
    return np.load(GOLDEN)


def fit_bc(bc, seed, dof):
    d0, d1 = np.random.RandomState(seed + 500000).randn(2, dof)
    return {"first": ((1, d0), (1, d1)), "mixed": ((2, d0), (1, d1))}.get(bc, bc)


def fit_input(n, spacing, bc):
    seed = 1000 * n + LONG_SPACINGS.index(spacing)
    x, y = long_spline_data(n, spacing, seed)
    if bc == "periodic":
        y[-1] = y[0]
    return x, y, fit_bc(bc, seed, y.shape[1])


def solve_input(g, i):
    t = "s%d_" % i
    return {k: g[t + k] for k in ("ss", "way", "vlim", "alim", "grid", "scheme", "sd_start")}


def velacc(pkg, vlim, alim, scheme):
    return [pkg.constraint.JointVelocityConstraint(vlim),
            pkg.constraint.JointAccelerationConstraint(alim, discretization_scheme=int(scheme))]


# ==== CPU: the oracle against the reference ================================================================================
def test_golden_covers_the_switches():
    g = golden()
    nseg = [len(g["s%d_ss" % i]) - 1 for i in range(N_SOLVES)]
    dofs = [g["s%d_way" % i].shape[1] for i in range(N_SOLVES)]
    G = [len(g["s%d_grid" % i]) for i in range(N_SOLVES)]
    for dof in (1, 3, 6, 7):
        have = {n for n, d in zip(nseg, dofs) if d == dof}
        assert FUSED_LAST[dof] in have or FUSED_LAST[dof] + 1 in have, dof
        assert K1_LAST[dof] in have or K1_LAST[dof] + 1 in have, dof
    assert any(gg < n for gg, n in zip(G, nseg)), "a solve with G < nseg"
    assert any(gg == 1000 and n == 399 for gg, n in zip(G, nseg)), "G = 1000 at n = 400"
    assert {int(g["s%d_scheme" % i]) for i in range(N_SOLVES)} == {0, 1}
    sd0 = [float(g["s%d_sd_start" % i]) for i in range(N_SOLVES)]
    assert any(v > 0 and v ** 2 == v * v for v in sd0)
    assert all(int(g["s%d_status" % i]) == 0 for i in range(N_SOLVES))


@pytest.mark.parametrize("n", FIT_N)
def test_oracle_fits_equal_scipy_golden(n):
    g = golden()
    for spacing in LONG_SPACINGS:
        for bc in FIT_BC:
            x, y, bct = fit_input(n, spacing, bc)
            c = orc.cubic_spline_fit(x, y, "periodic" if bc == "periodic" else bct)
            key = "%d_%s_%s" % (n, spacing, bc)
            if n >= FIT_HASHED:
                assert np.array_equal(sha(c), g["fitsha_" + key]), key
            else:
                assert_same(c, g["fit_" + key], key)


@pytest.mark.parametrize("i", range(N_SOLVES))
def test_oracle_solves_equal_reference_golden(i):
    g = golden()
    p = solve_input(g, i)
    t = "s%d_" % i
    c = orc.cubic_spline_fit(p["ss"], p["way"])
    assert np.array_equal(sha(c), g[t + "c_sha"]), "spline coefficients"
    o = orc.solve_velacc(c, p["ss"], p["grid"], p["vlim"], p["alim"], bool(p["scheme"]), float(p["sd_start"]), 0.0)
    assert o["status"] == int(g[t + "status"])
    for k, w in (("K", "K"), ("sd", "sd"), ("u", "sdd")):
        assert_same(o[k], g[t + w], "solve %d %s" % (i, k))


@pytest.mark.parametrize("i", CALLERS)
def test_callers_on_the_double_equal_reference_golden(i, monkeypatch):
    """Feasible and reachable sets, proposed grid and TOPPRAsd of the package's single-path API on the engine double."""
    ta = cpu_engine.install(monkeypatch)
    g = golden()
    p = solve_input(g, i)
    t = "s%d_" % i
    path = ta.SplineInterpolator(p["ss"], p["way"])
    mk = lambda: ta.algorithm.TOPPRA(velacc(ta, p["vlim"], p["alim"], p["scheme"]), path, gridpoints=p["grid"],  # noqa
                                     solver_wrapper="seidel")
    assert_same(mk().compute_feasible_sets(), g[t + "X"], "feasible sets")
    assert_same(mk().compute_reachable_sets(*REACH), g[t + "L"], "reachable sets")
    assert_same(np.asarray(ta.propose_gridpoints(path, **PROPOSE)), g[t + "pg"], "propose_gridpoints")
    sdi = ta.algorithm.TOPPRAsd(velacc(ta, p["vlim"], p["alim"], p["scheme"]), path, gridpoints=p["grid"],
                                solver_wrapper="seidel")
    sdi.set_desired_duration(float(g[t + "sd_desired"]))
    sdd, sd, _, _ = sdi.compute_parameterization(float(p["sd_start"]), 0.0, return_data=True)
    assert_same(sd, g[t + "sd_sd"], "TOPPRAsd sd")
    assert_same(sdd, g[t + "sd_sdd"], "TOPPRAsd sdd")
    sd_f = g[t + "sd"]
    assert float(g[t + "sd_desired"]) == np.sum(2 * np.diff(p["grid"]) / (sd_f[1:] + sd_f[:-1])) * SD_FACTOR


# ==== CPU: the switches ======================================================================================================
def test_switch_formulas_match_the_engine_and_the_issue_table():
    assert FUSED_LAST == {1: 292, 3: 107, 6: 55, 7: 47, 14: 24}
    assert K1_LAST == {1: 682, 3: 255, 6: 132, 7: 113, 14: 57}
    from toppra_b200 import engine
    for dof in (1, 2, 3, 6, 7, 8, 10, 14, 15):
        for interp in (True, False):
            for nseg in list(range(1, 80)) + [100, 106, 107, 108, 255, 291, 292, 293, 500]:
                assert engine.velacc_fused_supported(nseg, dof, interp) == fused_fits(nseg, dof, interp), (nseg, dof)


def gpu_cases():
    """(dof, nseg) pairs the GPU part of this file runs, by switch: each switch is met at its last value on one side and
    the first on the other."""
    fused = {(d, FUSED_LAST[d] + e) for d in (6, 7, 14) for e in (0, 1)}
    k1 = {(d, K1_LAST[d] + e) for d in (1, 7, 14) for e in (-1, 0, 1)}
    return fused, k1


def test_gpu_cases_straddle_the_switches():
    fused, k1 = gpu_cases()
    for dof in (6, 7, 14):
        interp = dof != 14
        sides = {fused_fits(n, dof, interp) for d, n in fused if d == dof}
        assert sides == {True, False}, dof
        assert fused_fits(FUSED_LAST[dof], dof, interp) and not fused_fits(FUSED_LAST[dof] + 1, dof, interp)
    for dof in (1, 7, 14):
        sides = [k1_smem(n, dof) for d, n in sorted(k1) if d == dof]
        assert sides == [True, True, False], dof
    assert LOCAL_KNOTS in K0_KNOTS and LOCAL_KNOTS + 1 in K0_KNOTS


def _lib():
    from toppra_b200 import _lib as L
    return L.load()


@pytest.mark.skipif(torch.cuda.is_available(), reason="the C-ABI size query, run on the library without a GPU")
def test_spline_workspace_size_query():
    lib = _lib()
    f = lib.tb_spline_fit_workspace_doubles
    f.restype = ctypes.c_int
    assert f(3, LOCAL_KNOTS, 7) == 0
    assert f(3, LOCAL_KNOTS + 1, 7) == 7 * 3 * (LOCAL_KNOTS + 1) * 7
    assert f(4096, 1000, 7) == 7 * 4096 * 1000 * 7
    assert f(4096, 11000, 7) == TB_ERR_UNSUPPORTED                     # more than 2^31 doubles
    assert f(16384 + 37, 48, 7) == 7 * (16384 + 37) * 48 * 7          # the forward-threads case below


def _route_problem(dof, nseg, B=4, seed=0):
    rng = np.random.RandomState(seed)
    ss = long_breaks(rng, nseg + 1, "uneven")
    way = np.stack([long_waypoints(rng, ss, dof) for _ in range(B)])
    vl, al = 10 + 20 * rng.rand(B, dof), 10 + 2 * rng.rand(B, dof)
    return ss, way, np.stack((-vl, vl), -1), np.stack((-al, al), -1)


@pytest.mark.parametrize("dof", [6, 7, 14])
def test_route_choice_at_the_fused_limit_on_the_double(dof, monkeypatch):
    ta = cpu_engine.install(monkeypatch)
    scheme = 0 if dof == 14 else 1
    for nseg, fused in ((FUSED_LAST[dof], True), (FUSED_LAST[dof] + 1, False)):
        ss, way, vlim, alim = _route_problem(dof, nseg)
        path = ta.BatchSplineInterpolator(ss, way)
        grid = np.linspace(0, ss[-1], 20)
        inst = ta.BatchTOPPRA(velacc(ta, vlim, alim, scheme), path, grid)
        assert inst.fused is fused, (dof, nseg)
        if not fused:
            with pytest.raises(ValueError):
                ta.BatchTOPPRA(velacc(ta, vlim, alim, scheme), path, grid, fused=True)
        h = inst.compute_parameterization(0.0, 0.0).to_host()
        o = orc.solve_velacc_batch(host(path.d_ppoly), np.tile(ss, (len(way), 1)), grid, vlim, alim, bool(scheme))
        for k, w in (("K", "K"), ("sd", "sd"), ("sdd", "u"), ("status", "status")):
            assert_same(h[k], o[w], "%s nseg %d" % (k, nseg))


@pytest.mark.parametrize("i", range(N_SOLVES))
def test_batch_on_the_double_equals_reference_golden(i, monkeypatch):
    ta = cpu_engine.install(monkeypatch)
    g = golden()
    p = solve_input(g, i)
    t = "s%d_" % i
    path = ta.BatchSplineInterpolator(p["ss"], p["way"][None])
    inst = ta.BatchTOPPRA(velacc(ta, p["vlim"], p["alim"], p["scheme"]), path, p["grid"])
    dof, nseg = p["way"].shape[1], len(p["ss"]) - 1
    assert inst.fused == fused_fits(nseg, dof, bool(p["scheme"]))
    h = inst.compute_parameterization(float(p["sd_start"]), 0.0).to_host()
    assert int(h["status"][0]) == int(g[t + "status"])
    for k in ("K", "sd", "sdd"):
        assert_same(h[k][0], g[t + k], k)


# ==== GPU ====================================================================================================================
K0_KNOTS = (15, 16, 17, 18, 33, 100, 1000)
K0_BCS = ("not-a-knot", "clamped", "natural", "first", "mixed", "periodic")


def _nthreads():
    return min(16, os.cpu_count() or 1)


def _gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import toppra_b200
    return toppra_b200


def _t(x, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("n", K0_KNOTS)
def test_k0_spline_fit_every_boundary_condition(n):
    """B * dof = 133 (two CTAs of 128, the last one partly idle), one motionless joint, shared and per-path breakpoints."""
    ta = _gpu()
    E = ta.engine
    B, dof = 19, 7
    rng = np.random.RandomState(n)
    ss_shared = long_breaks(rng, n, "decades" if n % 2 else "uneven")
    ss_path = np.stack([long_breaks(rng, n, LONG_SPACINGS[b % 3]) for b in range(B)])
    for ss in (ss_shared, ss_path):
        way = np.stack([long_waypoints(rng, ss if ss.ndim == 1 else ss[b], dof) for b in range(B)])
        way[4, :, 2] = way[4, 0, 2]                                                    # a motionless joint
        d0, d1 = rng.randn(2, B, dof)
        for bc in K0_BCS:
            w = way.copy()
            if bc == "periodic":
                w[:, -1] = w[:, 0]
            bct = {"first": ((1, d0), (1, d1)), "mixed": ((2, d0), (1, d1))}.get(bc, bc)
            got = host(E.spline_fit(_t(ss), _t(w), E.parse_bc(bct, B, dof, torch.device("cuda"))))
            for b in range(B):
                x = ss if ss.ndim == 1 else ss[b]
                bcb = bct if isinstance(bct, str) else ((bct[0][0], bct[0][1][b]), (bct[1][0], bct[1][1][b]))
                assert_same(got[b], orc.cubic_spline_fit(x, w[b], bcb),
                            "n %d bc %s %s breakpoints, path %d" % (n, bc, "shared" if ss.ndim == 1 else "per-path", b))


@pytest.mark.gpu
def test_ppoly_eval_on_1000_knots():
    ta = _gpu()
    B, dof, n = 3, 7, 1000
    rng = np.random.RandomState(11)
    ss = long_breaks(rng, n, "uneven")
    c = np.stack([orc.cubic_spline_fit(ss, long_waypoints(rng, ss, dof)) for _ in range(B)])
    s = np.r_[ss, 0.5 * (ss[1:] + ss[:-1]), ss[:-1] + 0.999 * np.diff(ss), ss[-1], ss[0] - 0.25, ss[-1] + 0.5,
              np.nextafter(ss[-1], np.inf), np.nextafter(ss[0], -np.inf)]
    for order in (0, 1, 2):
        got = host(ta.engine.ppoly_eval(_t(c), _t(ss), _t(s), order))
        for b in range(B):
            assert_same(got[b], orc.ppoly_eval(c[b], ss, s, order), "order %d path %d" % (order, b))


def _k1_paths(dof, nseg, B=3, seed=0):
    rng = np.random.RandomState(1000 * dof + nseg + seed)
    ss = long_breaks(rng, nseg + 1, "uneven")
    way = np.stack([long_waypoints(rng, ss, dof) for _ in range(B)])
    way[1, :, dof - 1] = way[1, 0, dof - 1]
    c = np.stack([orc.cubic_spline_fit(ss, way[b]) for b in range(B)])
    vl, al = 10 + 20 * rng.rand(dof), 10 + 2 * rng.rand(dof)
    return ss, c, np.stack((-vl, vl), -1), np.stack((-al, al), -1)


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [1, 7, 14])
def test_k1_records_around_the_shared_memory_switch(dof):
    ta = _gpu()
    E = ta.engine
    for nseg in (K1_LAST[dof] - 1, K1_LAST[dof], K1_LAST[dof] + 1):
        ss, c, vlim, alim = _k1_paths(dof, nseg)
        B = len(c)
        for G in (max(2, nseg // 7), 3 * nseg + 1):
            grid = np.linspace(0, ss[-1], G)
            for interp in (True, False):
                R = (4 if interp else 2) * dof
                rec, W = E.alloc_records(B, G, R, torch.device("cuda"))
                E.init_bounds(rec, R)
                want = torch.full((B, G, W), 7.0, dtype=torch.float64)
                torch.cuda.synchronize()
                want.copy_(rec.cpu())
                E.coeff_velacc(_t(c), _t(ss), _t(grid), _t(vlim), _t(alim), interp, rec, R)
                cpu_engine.coeff_velacc(torch.from_numpy(c), torch.from_numpy(ss), torch.from_numpy(grid),
                                        torch.from_numpy(vlim), torch.from_numpy(alim), interp, want, R)
                assert_same(host(rec), want.numpy(), "dof %d nseg %d G %d interp %d (shared memory: %s)"
                            % (dof, nseg, G, interp, k1_smem(nseg, dof)))


def _batch_inputs(dof, nseg, B, seed, vel_every=8):
    rng = np.random.RandomState(seed)
    ss = long_breaks(rng, nseg + 1, "uneven")
    way = np.stack([long_waypoints(rng, ss, dof) for _ in range(B)])
    way[np.arange(B) % 11 == 3, :, dof - 1] = way[np.arange(B) % 11 == 3, :1, dof - 1]
    vl, al = 10 + 20 * rng.rand(B, dof), 10 + 2 * rng.rand(B, dof)
    vl[::vel_every] = 0.02 + 0.05 * rng.rand(len(vl[::vel_every]), dof)           # velocity-limited paths
    return ss, way, np.stack((-vl, vl), -1), np.stack((-al, al), -1)


def _check_batch(h, o, what):
    assert_same(h["status"], o["status"], what + " status")
    for k, w in (("K", "K"), ("sd", "sd"), ("sdd", "u")):
        assert_same(h[k], o[w], what + " " + k)


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [6, 7, 14])
def test_fused_scan_around_its_limit(dof):
    ta = _gpu()
    scheme = 0 if dof == 14 else 1
    B = 64
    for nseg, fused in ((FUSED_LAST[dof], True), (FUSED_LAST[dof] + 1, False)):
        ss, way, vlim, alim = _batch_inputs(dof, nseg, B, 31 * dof + nseg)
        path = ta.BatchSplineInterpolator(ss, way)
        sd0 = np.where(np.arange(B) % 5 == 0, 0.0625, 0.0)
        for G in (nseg // 3, 4 * nseg):
            grid = np.linspace(0, ss[-1], G)
            inst = ta.BatchTOPPRA(velacc(ta, vlim, alim, scheme), path, grid)
            assert inst.fused is fused
            h = inst.compute_parameterization(sd0, 0.0).to_host()
            o = orc.solve_velacc_batch(host(path.d_ppoly), np.tile(ss, (B, 1)), grid, vlim, alim, bool(scheme), sd0, None,
                                       nthreads=_nthreads())
            what = "dof %d nseg %d G %d fused %s" % (dof, nseg, G, fused)
            _check_batch(h, o, what)
            assert (o["status"] == 0).any()
            if fused:
                r = ta.BatchTOPPRA(velacc(ta, vlim, alim, scheme), path, grid, fused=False)
                assert not r.fused
                hr = r.compute_parameterization(sd0, 0.0).to_host()
                for k in ("K", "sd", "sdd", "status"):
                    assert_same(hr[k], h[k], what + " record route " + k)


@pytest.mark.gpu
def test_forward_threads_at_the_fused_limit():
    from test_kernel_builds import launched
    ta = _gpu()
    dof, nseg, B = 7, FUSED_LAST[7], 16384 + 37
    ss, way, vlim, alim = _batch_inputs(dof, nseg, B, 4242)
    path = ta.BatchSplineInterpolator(ss, way)
    idx = np.arange(B)
    sd0 = np.where(idx % 13 == 0, 30.0, np.where(idx % 6 == 1, 0.0625, 0.0))      # inadmissible starts mixed in
    c = host(path.d_ppoly)
    for G in (48, 20):
        grid = np.linspace(0, ss[-1], G)
        inst = ta.BatchTOPPRA(velacc(ta, vlim, alim, 1), path, grid)
        assert inst.fused
        with launched() as k:
            h = inst.compute_parameterization(sd0, 0.0).to_host()
        assert "forward_threads_kernel<7>" in k, sorted(k)
        o = orc.solve_velacc_batch(c, np.tile(ss, (B, 1)), grid, vlim, alim, True, sd0, None, nthreads=_nthreads())
        _check_batch(h, o, "G %d" % G)
        st = np.bincount(o["status"], minlength=5)
        assert st[0] > B // 2 and st[3] > 0, st
        pinned = inst.solve_to_host(sd0, 0.0)
        for k_ in ("K", "sd", "sdd", "status"):
            assert_same(pinned[k_].numpy(), h[k_], "solve_to_host G %d %s" % (G, k_))


@pytest.mark.gpu
def test_order_k_paths_with_200_quintic_pieces():
    from scipy.interpolate import PPoly
    ta = _gpu()
    B, k, nseg, dof, G = 16, 6, 200, 7, 300
    rng = np.random.RandomState(200)
    x = np.r_[0.0, np.cumsum(0.5 + rng.rand(nseg))]
    x /= x[-1]
    c = rng.randn(B, k, nseg, dof) * (2.0 ** -np.arange(k)[::-1])[None, :, None, None] * 3.0
    s = np.r_[x, 0.5 * (x[1:] + x[:-1]), x[0] - 0.25, x[-1] + 0.5]
    path = ta.BatchPiecewisePolyPath(x, c)
    for b in range(0, B, 5):
        p = PPoly(c[b], x)
        d1 = p.derivative()
        for order, f in enumerate((p, d1, d1.derivative())):
            assert_same(path(s, order)[b], f(s), "eval order %d path %d" % (order, b))
    vl, al = 10 + 20 * rng.rand(B, dof), 10 + 2 * rng.rand(B, dof)
    vlim, alim = np.stack((-vl, vl), -1), np.stack((-al, al), -1)
    grid = np.linspace(0, 1, G)
    inst = ta.BatchTOPPRA(velacc(ta, vlim, alim, 1), path, grid)
    assert not inst.fused
    res = inst.compute_parameterization(0.0, 0.0).to_host()
    want = cpu_engine.scan(inst.records.cpu(), inst.R, torch.from_numpy(grid))
    for key, wkey in (("K", "K"), ("sd", "sd"), ("sdd", "u"), ("status", "status")):
        assert_same(res[key], want[wkey].numpy(), key)
    assert (res["status"] == 0).any()
    # the records' rows from scipy's derivative objects at the gridpoints, restated by the engine double
    qd = np.stack([PPoly(c[b], x).derivative()(grid) for b in range(B)])
    qdd = np.stack([PPoly(c[b], x).derivative().derivative()(grid) for b in range(B)])
    assert_same(host(inst.path.eval_device(_t(grid), 1)), qd, "q' at the gridpoints")
    assert_same(host(inst.path.eval_device(_t(grid), 2)), qdd, "q'' at the gridpoints")


@pytest.mark.gpu
def test_device_torque_model_rows_on_200_knots():
    """tb_coeff_second_order (pendulums) as test_kernel_builds.case_second_order checks it: a and b rows and the bounds
    bit for bit, the c rows (p_k sin q_k + ...) within TRIG_ULPS of their sin terms."""
    from test_kernel_builds import TRIG_ULPS, _rows_tol
    ta = _gpu()
    E = ta.engine
    B, dof, nseg, G = 12, 6, 199, 300
    ss, way, vlim, alim = _batch_inputs(dof, nseg, B, 4711)
    c = np.stack([orc.cubic_spline_fit(ss, way[b]) for b in range(B)])
    grid = np.linspace(0, ss[-1], G)
    rng = np.random.RandomState(1)
    prm = list((np.stack((1 + rng.rand(dof), 5 + 3 * rng.rand(dof)), 1)).reshape(-1))
    taulim = np.stack((-(40 + 10 * rng.rand(dof)), 40 + 10 * rng.rand(dof)), 1)
    fric = 0.5 * rng.rand(dof)
    eps = np.finfo(float).eps
    for interp in (True, False):
        R = (4 if interp else 2) * dof
        rec, W = E.alloc_records(B, G, R, torch.device("cuda"))
        E.init_bounds(rec, R)
        host_rec = torch.from_numpy(host(rec).copy())
        E.coeff_second_order("pendulums", prm, _t(c), _t(ss), _t(grid), _t(taulim), _t(fric), interp, rec, R, 0)
        got = host(rec)
        cpu_engine.coeff_second_order("pendulums", prm, torch.from_numpy(c), torch.from_numpy(ss), torch.from_numpy(grid),
                                      torch.from_numpy(taulim), torch.from_numpy(fric), interp, host_rec, R, 0)
        want = host_rec.numpy()
        what = "interp %d" % interp
        assert_same(got[..., 3 * R:], want[..., 3 * R:], what + " bounds")
        assert_same(got[..., :R], want[..., :R], what + " a")
        assert_same(got[..., R:2 * R], want[..., R:2 * R], what + " b")
        sin_scale = np.abs(np.asarray(prm)[1::2]) * np.ones((B, G, dof))
        gc, wc = got[..., 2 * R:3 * R], want[..., 2 * R:3 * R]
        tol = TRIG_ULPS * _rows_tol(eps * sin_scale, R, dof) + 2 * np.spacing(np.abs(wc))
        assert np.all(np.abs(gc - wc) <= tol), what + " c"


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SOLVES))
def test_golden_replay_single_and_batch(i):
    ta = _gpu()
    g = golden()
    p = solve_input(g, i)
    t = "s%d_" % i
    scheme, sd0 = int(p["scheme"]), float(p["sd_start"])
    one = ta.algorithm.TOPPRA(velacc(ta, p["vlim"], p["alim"], scheme), ta.SplineInterpolator(p["ss"], p["way"]),
                              gridpoints=p["grid"], solver_wrapper="seidel")
    sdd, sd, _, K = one.compute_parameterization(sd0, 0.0, return_data=True)
    assert_same(K, g[t + "K"], "TOPPRA K")
    assert_same(sd, g[t + "sd"], "TOPPRA sd")
    assert_same(sdd, g[t + "sdd"], "TOPPRA sdd")
    path = ta.BatchSplineInterpolator(p["ss"], np.stack([p["way"]] * 3))
    assert np.array_equal(sha(host(path.d_ppoly)[0]), g[t + "c_sha"]), "spline coefficients"
    routes = (None, False) if fused_fits(len(p["ss"]) - 1, p["way"].shape[1], bool(scheme)) else (None,)
    for fused in routes:
        inst = ta.BatchTOPPRA(velacc(ta, p["vlim"], p["alim"], scheme), path, p["grid"], fused=fused)
        h = inst.compute_parameterization(sd0, 0.0).to_host()
        assert (h["status"] == int(g[t + "status"])).all()
        for k in ("K", "sd", "sdd"):
            for b in range(3):
                assert_same(h[k][b], g[t + k], "BatchTOPPRA fused=%s %s" % (inst.fused, k))
