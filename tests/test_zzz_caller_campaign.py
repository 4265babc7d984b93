"""GPU (-m gpu; the harness itself is replayed on the engine double under -m "not gpu"): the batched CALLERS around the
scan against the oracle on RANDOMLY SHAPED problems (tests/problems.py: random_shaped_problem, the draw of
scripts/fuzz_oracle_vs_reference.py, whose CPU campaign pins the oracle to the unmodified reference for these families).

Families, each with the edge values where its kernel's control flow turns:
  propose_gridpoints (tb_propose.cuh)      path lengths != 1, max_seg_length = length / 2**k exactly, 33+ and 65+
                                           segments in a pass, max_iteration 1..3 and convergence on the last allowed
                                           pass, max_points at / one below the needed count and a cap only the doubling
                                           crosses, motionless joints, NaN coefficients
  BatchTOPPRA                               fused and record scan on common, per-path and proposed (ragged) grids,
                                           per-path limits and start speeds, batch sizes 1 / 31 / 33 / 129 and ~2000
  TOPPRAsd / sd_bisect                      durations k * t_fast and exactly d_fast / d_slow, atol 0, tiny max_iter,
                                           status_in, NaN profiles, a ragged batch with Gmax > 3072 (dynamic shared
                                           memory above 48 KB)
  reachable / controllable sets             sdmin == sdmax (1-variable stage LPs), sdmin = 0, paths that fail mid-way
  parametrizers                             spline time stamps (5 s rule at exactly TINY, dropped knots, ragged glen),
                                           BatchParametrizeSpline, ConstAccel time grid and evaluation
  constraint producers                      a user constraint with ubound / xbound, JointVelocityConstraintVarying,
                                           JointTorqueConstraint with dry friction and a motionless joint

The GPU results are copied to the host first; then the oracle-backed engine double (tests/cpu_engine.py) is installed and
the same calls are made again.  Engine arguments the public API cannot set (max_points, status_in, atol, max_iter, the
info row) are compared through toppra_b200.engine against cpu_engine on the same inputs.  A path of a ragged batch is
compared with a single-path solve on its own grid[b, :glen[b]].  Bit for bit, NaN equal to NaN, except the ConstAccel
evaluation (rounding of a time lookup, fuzz-script tolerances).  scripts/caller_campaign.py runs the same checks for
as long as wanted."""
import time

import numpy as np
import pytest
import torch

import cpu_engine
from oracle import oracle as orc
from problems import inv_dyn_numpy, random_shaped_problem

SEED0 = 700000
N_PROBLEMS = {"gpu": 48, "cpu_double": 10}
# seeds that once exposed a mismatch, replayed first
REGRESSION_SEEDS = []


class Side(object):
    """The package under test: on the GPU the real kernels (and the double on demand), else the double throughout."""

    def __init__(self, gpu, monkeypatch):
        import toppra_b200
        self.gpu, self.pkg, self.mp = gpu, toppra_b200, monkeypatch
    
    def t(self, x, dtype=None):
        x = torch.as_tensor(np.ascontiguousarray(x), dtype=dtype)
        return x.cuda() if self.gpu else x

    def both(self, fn):
        """fn(pkg) -> host results, run on the kernels and then on the double (once when the double is all there is)."""
        first = fn(self.pkg)
        if not self.gpu:
            return first, first
        with self.mp.context() as m:
            cpu_engine.install(m)
            return first, fn(self.pkg)


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "cpu_double"])
def ta(request, monkeypatch):
    if request.param == "cpu_double":
        cpu_engine.install(monkeypatch)
        return Side(False, monkeypatch)
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return Side(True, monkeypatch)


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x


def square_exact(v):
    """The next float >= v whose square the reference's pow(v, 2.0) rounds like v * v (problems.py)."""
    v = float(v)
    while v ** 2 != v * v:
        v = float(np.nextafter(v, np.inf))
    return v


def hit(hist, key, n=1):
    hist[key] = hist.get(key, 0) + n


def spline(p):
    return np.ascontiguousarray(orc.cubic_spline_fit(p["ss"], p["way"]))


def durations(x, grid):
    return cpu_engine._duration(x, np.diff(grid))


# ---- propose_gridpoints ------------------------------------------------------------------------------------------------
def _propose_double(c, ss, **kw):
    g, n, s = cpu_engine.propose_gridpoints(torch.from_numpy(c[None]), torch.from_numpy(ss), **kw)
    return g[0].numpy(), int(n[0]), int(s[0])


def _segments_target(c, ss, target, kw):
    """A max_err_threshold at which the converged pass list has exactly `target` segments (None if bisection misses)."""
    lo, hi = -12.0, 2.0      # log10 of the threshold: more segments below
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        _, n, st = _propose_double(c, ss, **dict(kw, max_err_threshold=10 ** mid))
        if st == 0 and n - 1 == target:
            return 10 ** mid
        if st != 0 or n - 1 > target:
            lo = mid
        else:
            hi = mid
    return None


def check_propose(ta, p, rng, hist):
    ss = p["ss"] * (10 ** rng.uniform(-1, 1) if rng.rand() < 0.7 else 1.0)      # path lengths other than 1
    ss = ss if ss[-1] > ss[0] else np.linspace(0, 1, len(ss))
    c = np.ascontiguousarray(orc.cubic_spline_fit(ss, p["way"]))
    nseg, dof = c.shape[1], c.shape[2]
    if rng.rand() < 0.2:
        c[:3, :, rng.randint(dof)] = 0.0                                        # a joint that does not move
    if rng.rand() < 0.1:
        c[rng.randint(4), rng.randint(nseg), rng.randint(dof)] = np.nan         # np.max's NaN rule
    span = ss[-1] - ss[0]
    kw = dict(max_err_threshold=10 ** rng.uniform(-5, -1), max_iteration=100, max_seg_length=rng.uniform(0.02, 0.6) * span,
              min_nb_points=int(rng.randint(2, 200)), max_points=8192)
    kind = rng.randint(6)
    if kind == 1:                                                               # lengths land exactly on the > test
        kw["max_seg_length"] = span / 2 ** rng.randint(0, 8)
        kw["max_err_threshold"] = 10 ** rng.uniform(-3, 2)
    elif kind == 2:
        kw["max_iteration"] = int(rng.choice([1, 2, 3]))
    elif kind == 3:                                                             # converge on the last allowed pass
        kw["min_nb_points"] = 2
        for m in range(1, 16):
            if _propose_double(c, ss, **dict(kw, max_iteration=m))[2] == 0:
                kw["max_iteration"] = m - 1 if (m > 1 and rng.rand() < 0.7) else m
                break
    elif kind == 4:                                                             # caps around the needed count
        _, need, st = _propose_double(c, ss, **dict(kw, min_nb_points=2))
        _, full, st2 = _propose_double(c, ss, **kw)
        if st == 0 and st2 == 0:                                            # need: after the passes, full: doubled
            r = rng.randint(3) if full > need + 1 else rng.randint(2)
            kw["max_points"] = max(2, [full, full - 1, (need + full) // 2][r])
            hit(hist, "propose cap " + ["= needed", "= needed - 1", "crossed by the doubling"][r])
    elif kind == 5:                                                             # 31 / 32 / 33 / 65 segments in a pass
        kw.update(min_nb_points=2, max_seg_length=2 * span)
        target = int(rng.choice([31, 32, 33, 65]))
        thr = _segments_target(c, ss, target, kw)
        if thr is not None:
            kw["max_err_threshold"] = thr
            hit(hist, "propose %d segments" % target)
    cc = np.stack((c, 0.5 * c, 3.0 * c))
    got = [host(x) for x in ta.pkg.engine.propose_gridpoints(ta.t(cc), ta.t(ss), **kw)]
    want = [x.numpy() for x in cpu_engine.propose_gridpoints(torch.from_numpy(cc), torch.from_numpy(ss), **kw)]
    for what, g, w in zip(("grid", "glen", "status"), got, want):
        assert same(g, w), "propose_gridpoints %s (kind %d, %s)" % (what, kind, kw)
    for s in want[2]:
        hit(hist, "propose status %s" % ("<0" if s < 0 else s))
    if kw["max_iteration"] > 1 and want[2][0] == 1 and kind == 3:
        hit(hist, "propose converged on the last pass")
    hit(hist, "propose >32 segments", int(np.sum(want[1] > 33)))
    hit(hist, "propose >64 segments", int(np.sum(want[1] > 65)))
    if kind in (1, 2) and not np.isnan(c).any():                               # the public API, raise and all
        def run(pkg):
            path = pkg.SplineInterpolator(ss, p["way"])
            try:
                return np.asarray(pkg.propose_gridpoints(path, **kw))
            except ValueError as e:
                return str(e)
        a, b = ta.both(run)
        assert (isinstance(a, str) and a == b) or same(a, b), "public propose_gridpoints (%s)" % kw


# ---- BatchTOPPRA on common, per-path and proposed grids -------------------------------------------------------------------
def _batch_problem(p, rng, B):
    n, dof = len(p["ss"]), min(p["way"].shape[1], 7)
    way = rng.randn(B, n, dof) * (10 ** rng.uniform(-1, 0.5))
    vl, al = 1 + 20 * rng.rand(B, dof), 5 + 10 * rng.rand(B, dof)
    vlim, alim = np.stack((-vl, vl), axis=-1), np.stack((-al, al), axis=-1)
    sd0 = np.array([square_exact(v) for v in np.where(rng.rand(B) < 0.5, 0.0, 10 ** rng.uniform(-3, 0.3, B))])
    sd1 = np.array([square_exact(v) for v in np.where(rng.rand(B) < 0.7, 0.0, 10 ** rng.uniform(-3, -1, B))])
    c = np.stack([orc.cubic_spline_fit(p["ss"], way[b]) for b in range(B)])
    return dict(ss=p["ss"], c=np.ascontiguousarray(c), vlim=vlim, alim=alim, sd0=sd0, sd1=sd1, interp=p["interp"], B=B)


def _cmp_solution(h, b, o, G, tag):
    assert h["status"][b] == o["status"] and same(h["K"][b, :G], o["K"]), "K / status, " + tag
    if o["status"] == 0:
        assert same(h["sd"][b, :G], o["sd"]) and same(h["sdd"][b, :G - 1], o["u"]), "sd / u, " + tag


def check_batch(ta, p, rng, hist, B):
    q = _batch_problem(p, rng, B)
    pkg, G = ta.pkg, len(p["grid"])
    bpath = pkg.BatchSplineInterpolator.from_ppoly(q["ss"], q["c"])
    cons = [pkg.constraint.JointVelocityConstraint(q["vlim"]),
            pkg.constraint.JointAccelerationConstraint(q["alim"], discretization_scheme=q["interp"])]
    o = orc.solve_velacc_batch(q["c"], np.tile(q["ss"], (B, 1)), p["grid"], q["vlim"], q["alim"], bool(q["interp"]),
                               q["sd0"], q["sd1"], nthreads=8)
    per_path = np.stack([p["grid"]] + [np.r_[0.0, np.sort(rng.uniform(0, p["ss"][-1], G - 2)), p["ss"][-1]]
                                       for _ in range(B - 1)]) if G > 3 else np.tile(p["grid"], (B, 1))
    for fused in (None, False):
        inst = pkg.BatchTOPPRA(cons, bpath, gridpoints=p["grid"], fused=fused)
        h = inst.compute_parameterization(q["sd0"], q["sd1"]).to_host()
        hit(hist, "batch fused" if inst.fused else "batch records")
        for b in range(B):
            _cmp_solution(h, b, dict(K=o["K"][b], sd=o["sd"][b], u=o["u"][b], status=o["status"][b]), G,
                          "common grid, B %d, path %d, fused %s" % (B, b, inst.fused))
            hit(hist, "batch status %d" % o["status"][b])
    if B > 200 or np.any(np.diff(per_path, axis=1) <= 0):
        return
    grids = {"per-path grid": (per_path, None)}
    try:
        inst = pkg.BatchTOPPRA(cons, bpath, gridpoints=None, gridpt_max_err_threshold=10 ** rng.uniform(-4, -2),
                               gridpt_min_nb_points=int(rng.randint(2, 120)))
        grids["proposed grid"] = (host(inst.d_grid), host(inst.glen))
    except ValueError:          # no good grid within the passes / more than max_points: propose_gridpoints' own checks
        hit(hist, "batch proposal raised")
    for tag, (grid, glen) in grids.items():
        for fused in (None, False):
            inst = pkg.BatchTOPPRA(cons, bpath, gridpoints=grid, glen=glen, fused=fused)
            h = inst.compute_parameterization(q["sd0"], q["sd1"]).to_host()
            for b in range(B):
                n = grid.shape[1] if glen is None else int(glen[b])
                o = orc.solve_velacc(q["c"][b], q["ss"], grid[b, :n], q["vlim"][b], q["alim"][b], bool(q["interp"]),
                                     q["sd0"][b], q["sd1"][b])
                _cmp_solution(h, b, o, n, "%s, B %d, path %d, fused %s" % (tag, B, b, inst.fused))
            hit(hist, "batch " + tag)


# ---- TOPPRAsd -------------------------------------------------------------------------------------------------------------
def _sd_inputs(rng, B, G, grid_shared):
    """Fastest / slowest pass outputs as sd_bisect sees them (x = sd^2 >= 0, slower below faster), a few NaN profiles."""
    xf = np.abs(rng.randn(B, G)) * 10 ** rng.uniform(-2, 2, (B, 1)) + 1e-4
    xf[:, 0] = np.where(rng.rand(B) < 0.6, 0.0, xf[:, 0])
    xf[:, -1] = np.where(rng.rand(B) < 0.6, 0.0, xf[:, -1])
    xs = xf * rng.uniform(0.01, 1.0, (B, G))
    nan = rng.rand(B) < 0.08
    xf[nan, rng.randint(G)] = np.nan
    uf, us = rng.randn(B, G - 1), rng.randn(B, G - 1)
    g = np.r_[0.0, np.cumsum(0.01 + rng.rand(G - 1))] * 10 ** rng.uniform(-2, 1)
    grid = g if grid_shared else np.stack([np.r_[0.0, np.cumsum(0.01 + rng.rand(G - 1))] for _ in range(B)])
    return xf, uf, xs, us, grid


def _wants(rng, xf, xs, grid, glen=None):
    B = xf.shape[0]
    want, kinds = np.empty(B), []
    for b in range(B):
        n = xf.shape[1] if glen is None else int(glen[b])
        g = grid if grid.ndim == 1 else grid[b]
        d_fast, d_slow = durations(xf[b, :n], g[:n]), durations(xs[b, :n], g[:n])
        k = rng.randint(4)
        kinds.append(["factor", "= d_fast", "= d_slow", "between"][k])
        want[b] = [d_fast * rng.choice([0.5, 1.0, 1.2, 2.0, 7.0, 1e3]), d_fast, d_slow, 0.5 * (d_fast + d_slow)][k]
    return want, kinds


def _sd_hist(hist, info, want, kinds, status_in=None):
    for b in range(len(want)):
        if status_in is not None and status_in[b] == 3:
            hit(hist, "sd status_in 3")
            continue
        a, d_fast, d_slow = info[b, :3]
        branch = "fast" if d_fast > want[b] else ("slow" if d_slow < want[b] else "bisect")
        hit(hist, "sd " + branch)
        if kinds[b] in ("= d_fast", "= d_slow") and branch == "bisect":
            hit(hist, "sd want " + kinds[b])


def check_sd_bisect(ta, rng, hist, B, G, ragged=False):
    ragged = ragged and ta.gpu                      # the double has no ragged forms: ragged runs compare path by path
    xf, uf, xs, us, grid = _sd_inputs(rng, B, G, grid_shared=not ragged and rng.rand() < 0.5)
    glen = np.where(rng.rand(B) < 0.3, G, rng.randint(2, G + 1, B)).astype(np.int32) if ragged else None
    want, kinds = _wants(rng, xf, xs, grid, glen)
    atol = float(rng.choice([1e-5, 0.0, 1e-9]))
    max_iter = int(rng.choice([1, 2, 3, 200, 200]))
    st_in = np.where(rng.rand(B) < 0.15, 3, 0).astype(np.int32) if rng.rand() < 0.7 else None
    args = [xf, uf, xs, us, grid, want]
    got = ta.pkg.engine.sd_bisect(*[ta.t(x) for x in args], atol=atol, max_iter=max_iter,
                                  status_in=None if st_in is None else ta.t(st_in, torch.int32),
                                  **({} if glen is None else dict(glen=ta.t(glen, torch.int32))))
    got = {k: host(v) for k, v in got.items()}
    tag = "sd_bisect B %d G %d atol %g max_iter %d ragged %s" % (B, G, atol, max_iter, ragged)
    if glen is None:
        w = cpu_engine.sd_bisect(*[torch.from_numpy(np.ascontiguousarray(x)) for x in args], atol=atol,
                                 status_in=None if st_in is None else torch.from_numpy(st_in), max_iter=max_iter)
        for k in ("sd", "u", "info", "status"):
            assert same(got[k], w[k].numpy()), "%s: %s" % (k, tag)
        info = w["info"].numpy()
    else:
        info = np.empty((B, 4))
        for b in range(B):
            n = int(glen[b])
            one = [x[b:b + 1, :n] for x in (xf, uf[:, :n - 1], xs, us[:, :n - 1], grid)]
            w = cpu_engine.sd_bisect(*[torch.from_numpy(np.ascontiguousarray(x)) for x in one],
                                     torch.from_numpy(want[b:b + 1]), atol=atol, max_iter=max_iter,
                                     status_in=None if st_in is None else torch.from_numpy(st_in[b:b + 1]))
            msg = "path %d (glen %d): %s" % (b, n, tag)
            assert same(got["sd"][b, :n], w["sd"][0].numpy()) and same(got["u"][b, :n - 1], w["u"][0].numpy()), msg
            assert same(got["info"][b], w["info"][0].numpy()) and got["status"][b] == int(w["status"][0]), "info, " + msg
            if st_in is None or st_in[b] != 3:
                assert np.isnan(got["sd"][b, n:]).all() and np.isnan(got["u"][b, n - 1:]).all(), "padding, " + msg
            info[b] = w["info"][0].numpy()
        hit(hist, "sd Gmax > 3072" if G > 3072 else "sd ragged")
    _sd_hist(hist, info, want, kinds, st_in)
    for s in got["status"]:
        hit(hist, "sd status %d" % s)
    hit(hist, "sd atol 0" if atol == 0 else "sd atol > 0")
    if max_iter < 4:
        hit(hist, "sd tiny max_iter")


def check_toppra_sd(ta, p, rng, hist):
    """The public BatchTOPPRAsd: both passes, the bisection, status_in from the fastest pass (uncontrollable paths)."""
    B = 5
    q = _batch_problem(p, rng, B)
    q["sd0"][rng.rand(B) < 0.3] = 50.0                                   # inadmissible start: FailUncontrollable
    t_fast = np.empty(B)
    for b in range(B):
        o = orc.solve_velacc(q["c"][b], q["ss"], p["grid"], q["vlim"][b], q["alim"][b], bool(q["interp"]), 0.0, 0.0)
        s = o["sd"]
        with np.errstate(divide="ignore"):
            t_fast[b] = np.sum(2 * np.diff(p["grid"]) / (s[1:] + s[:-1])) if o["status"] == 0 else 1.0
    want = t_fast * rng.choice([0.5, 1.0, 1.2, 2.0, 7.0, 1e3], B)
    atol = float(rng.choice([1e-5, 0.0]))

    def run(pkg):
        bpath = pkg.BatchSplineInterpolator.from_ppoly(q["ss"], q["c"])
        cons = [pkg.constraint.JointVelocityConstraint(q["vlim"]),
                pkg.constraint.JointAccelerationConstraint(q["alim"], discretization_scheme=q["interp"])]
        inst = pkg.BatchTOPPRAsd(cons, bpath, gridpoints=p["grid"])
        inst.set_desired_duration(want)
        r = inst.compute_parameterization(q["sd0"], q["sd1"], atol=atol)
        info = np.stack([host(x) for x in (r.alpha, r.duration_fast, r.duration_slow)], axis=1)
        return {k: host(getattr(r, k)) for k in ("K", "sd", "sdd", "status", "fail_stage")} | {"info": info}
    a, b = ta.both(run)
    for k in a:
        assert same(a[k], b[k]), "BatchTOPPRAsd %s (atol %g)" % (k, atol)
    for s in a["status"]:
        hit(hist, "TOPPRAsd status %d" % s)


# ---- reachable and controllable sets ----------------------------------------------------------------------------------------
def _sd_limits(rng, B):
    lo, hi = np.empty(B), np.empty(B)
    for b in range(B):
        k = rng.randint(4)
        lo[b] = [0.0, square_exact(10 ** rng.uniform(-3, -0.5)), square_exact(10 ** rng.uniform(-2, 0)), 7.0][k]
        hi[b] = lo[b] if (k == 2 or rng.rand() < 0.3) else square_exact(lo[b] + 10 ** rng.uniform(-3, 0.5))
    return lo, hi


def check_reachable(ta, p, rng, hist):
    B = 4
    q = _batch_problem(p, rng, B)
    lo, hi = _sd_limits(rng, B)
    tight = rng.rand() < 0.4                                        # velocity bounds that make forward passes fail

    def run(pkg, grid=None, glen=None, rows=slice(None)):
        bpath = pkg.BatchSplineInterpolator.from_ppoly(q["ss"], q["c"][rows])
        vl = q["vlim"][rows] * (0.05 if tight else 1.0)
        cons = [pkg.constraint.JointVelocityConstraint(vl),
                pkg.constraint.JointAccelerationConstraint(q["alim"][rows], discretization_scheme=q["interp"])]
        inst = pkg.BatchTOPPRA(cons, bpath, gridpoints=p["grid"] if grid is None else grid, glen=glen, fused=False)
        L, X, fs = inst.compute_reachable_sets(lo[rows], hi[rows])
        K, st = inst.compute_controllable_sets(lo[rows], hi[rows])
        return dict(L=host(L), X=host(X), fs=host(fs), K=host(K), st=host(st))
    a, b = ta.both(run)
    for k in a:
        assert same(a[k], b[k]), "reachable / controllable sets, common grid: " + k
    hit(hist, "reach 1-variable", int(np.sum(lo == hi)))
    hit(hist, "reach sdmin = 0", int(np.sum(lo == 0)))
    hit(hist, "reach fail_stage > 0", int(np.sum(a["fs"] > 0)))
    hit(hist, "controllable status 3", int(np.sum(a["st"] == 3)))
    # ragged: the proposed grids of the batch against single-path solves on each grid
    bpath = ta.pkg.BatchSplineInterpolator.from_ppoly(q["ss"], q["c"])
    try:
        grid, glen = (host(x) for x in bpath.propose_gridpoints(10 ** rng.uniform(-3, -1), 100, 0.2 * q["ss"][-1], 2))
    except ValueError:
        return
    if grid.shape[1] > 160:
        return
    if not ta.gpu:
        return
    a = run(ta.pkg, grid, glen)
    for i in range(B):
        n = int(glen[i])
        one = ta.both(lambda pkg: run(pkg, grid[i:i + 1, :n], None, slice(i, i + 1)))[1]
        tag = "ragged path %d (glen %d)" % (i, n)
        assert same(a["L"][i, :n], one["L"][0]) and same(a["X"][i, :n], one["X"][0]), "L / X, " + tag
        assert a["fs"][i] == one["fs"][0], "fail_stage, " + tag
        assert same(a["K"][i, :n], one["K"][0]) and a["st"][i] == one["st"][0], "controllable sets, " + tag
        assert np.isnan(a["L"][i, n:]).all() and np.isnan(a["X"][i, n:]).all(), "padding, " + tag
    hit(hist, "reach ragged")


# ---- output parametrizers ----------------------------------------------------------------------------------------------
def _velocity_profiles(rng, B, G):
    v = np.abs(rng.randn(B, G)) * 10 ** rng.uniform(-2, 1, (B, 1)) + 1e-3
    for b in range(B):
        k = rng.randint(5)
        i = rng.randint(1, G)
        if k == 0:
            v[b, rng.randint(0, G, 2)] = 0.0                       # stops: 5 s rule
        elif k == 1:
            v[b, G // 3:G // 3 + 3] = 1e10                         # increments below TINY: knots dropped
        elif k == 2:
            v[b, i - 1:i + 1] = 1e-8                               # average exactly TINY: 5 s rule (not >)
        elif k == 3:
            v[b, i - 1:i + 1] = 1e-10                              # average exactly 1e-10
    return v


def check_time_stamps(ta, rng, hist, B):
    G = int(rng.choice([2, 3, 17, 60, 200]))
    v = _velocity_profiles(rng, B, G)
    grid = np.cumsum(np.c_[np.zeros(B), 1e-3 + rng.rand(B, G - 1)], axis=1) * 10 ** rng.uniform(-3, 1, (B, 1))
    glen = rng.randint(1, G + 1, B).astype(np.int32)
    got = [host(x) for x in ta.pkg.engine.spline_time_stamps(ta.t(v), ta.t(grid), ta.t(glen, torch.int32))]
    want = [x.numpy() for x in cpu_engine.spline_time_stamps(torch.from_numpy(v), torch.from_numpy(grid),
                                                             torch.from_numpy(glen))]
    for what, g, w in zip(("t", "s", "nkeep"), got, want):
        assert same(g, w), "spline_time_stamps %s (B %d, G %d)" % (what, B, G)
    for b in range(B):
        n = int(glen[b])
        avg = (v[b, :n - 1] + v[b, 1:n]) / 2
        hit(hist, "stamps 5 s rule at TINY", int(np.sum(avg == 1e-8)))
        hit(hist, "stamps 5 s rule", int(np.sum(~(avg > 1e-8))))
    hit(hist, "stamps dropped knot", int(np.sum(want[2] < glen)))


def check_param_outputs(ta, p, rng, hist):
    """time_grid bit for bit, ConstAccel evaluation at and around the knot times, BatchParametrizeSpline knots and re-fit."""
    B = 3
    q = _batch_problem(p, rng, B)
    G = len(p["grid"])
    if G < 3:
        return
    sd = np.abs(rng.randn(B, G)) + 0.05
    sd[:, 0] = 0.0 if rng.rand() < 0.5 else sd[:, 0]
    c, ss, grid = q["c"], q["ss"], p["grid"]
    E = ta.pkg.engine
    t, us = E.time_grid(ta.t(sd), ta.t(grid))
    tw, uw = cpu_engine.time_grid(torch.from_numpy(sd), torch.from_numpy(grid))
    assert same(host(t), tw.numpy()) and same(host(us), uw.numpy()), "time_grid"
    tw = tw.numpy()
    ts = np.stack([np.r_[0.0, tw[b], tw[b, -1] * (1 + 1e-3), tw[b, -1] + 1.0, -1e-3, rng.uniform(0, tw[b, -1], 20)]
                   for b in range(B)])
    scale = max(1.0, np.abs(c).max() * max(1.0, ss[-1]) ** 3)
    for order, tol in ((0, 1e-11), (1, 1e-9), (2, 1e-7)):
        got = host(E.constaccel_eval(ta.t(c), ta.t(ss), ta.t(grid), ta.t(sd), t, us, ta.t(ts), order))
        want = cpu_engine.constaccel_eval(torch.from_numpy(c), torch.from_numpy(ss), torch.from_numpy(grid),
                                          torch.from_numpy(sd), torch.from_numpy(tw), uw, torch.from_numpy(ts), order).numpy()
        np.testing.assert_allclose(got, want, rtol=tol, atol=tol * max(scale, np.abs(want).max()),
                                   err_msg="constaccel_eval order %d" % order)
        worst = np.max(np.abs(got - want) / (tol * max(scale, np.abs(want).max())))
        hist["constaccel worst / tol"] = max(hist.get("constaccel worst / tol", 0.0), float(worst))
    v = _velocity_profiles(rng, B, G)
    if (cpu_engine.spline_time_stamps(torch.from_numpy(v), torch.from_numpy(grid))[2] < 2).any():
        v = sd                                     # a single knot has no spline (the reference raises too)

    def run(pkg):
        bpath = pkg.BatchSplineInterpolator.from_ppoly(ss, c)
        f = pkg.BatchParametrizeSpline(bpath, grid, v)
        return dict(t=host(f.t_knots), s=host(f.s_knots), n=host(f.nkeep), d=host(f.durations),
                    coeff=[(idx, host(fit.d_ppoly)) for idx, fit in f.groups])
    a, b = ta.both(run)
    for k in ("t", "s", "n", "d"):
        assert same(a[k], b[k]), "BatchParametrizeSpline " + k
    for (ia, ca), (ib, cb) in zip(a["coeff"], b["coeff"]):
        assert same(ia, ib)
        if same(ca, cb):
            hit(hist, "spline refit bit-equal")
        else:                         # the clamped re-fit: test_zzz_shape_campaign's bound
            np.testing.assert_allclose(ca, cb, rtol=1e-11, atol=1e-12 * max(1.0, np.abs(cb).max()), err_msg="re-fit")
            hit(hist, "spline refit within 1e-11")


# ---- constraint producers -------------------------------------------------------------------------------------------------
def _ub_class(cons):
    class UB(cons.LinearConstraint):
        """Acceleration rows + a u-interval and an x-interval per gridpoint."""

        def __init__(self, acc, ub, xb):
            super(UB, self).__init__()
            self.acc, self.ub, self.xb = acc, ub, xb
            self.discretization_type = acc.discretization_type
            self.identical = True

        def get_dof(self):
            return self.acc.get_dof()

        def compute_constraint_params(self, path, gridpoints, *a):
            pa, pb, pc, F, g, _, _ = self.acc.compute_constraint_params(path, gridpoints)
            return pa, pb, pc, F, g, self.ub, self.xb
    return UB


def check_constraints(ta, p, rng, hist):
    if len(p["grid"]) < 3 or len(p["grid"]) > 200:
        return
    dof, G = p["way"].shape[1], len(p["grid"])
    way = p["way"].copy()
    if rng.rand() < 0.4:
        way[:, rng.randint(dof)] = way[0, 0]                        # sign(q') = 0 in the friction term
    width = 10 ** rng.uniform(-1.5, 1.0) * max(1e-3, np.abs(p["alim"]).max())
    ub = np.stack((-width * (0.5 + rng.rand(G)), width * (0.5 + rng.rand(G))), axis=1)
    xb = np.stack((np.zeros(G), 10 ** rng.uniform(-2, 3) * (0.5 + rng.rand(G))), axis=1)
    k0, k1 = 0.05 + rng.rand(), rng.rand() / p["ss"][-1]
    sdmax = square_exact(10 ** rng.uniform(-2, 0))
    taulim = np.stack((-(20 + 30 * rng.rand(dof)), 20 + 30 * rng.rand(dof)), axis=1)
    fric = 0.5 * rng.rand(dof)
    scheme = int(rng.rand() < 0.5)

    def run(pkg):
        C = pkg.constraint
        path = pkg.SplineInterpolator(p["ss"], way)
        acc = lambda: C.JointAccelerationConstraint(p["alim"], p["interp"])  # noqa: E731
        mk = lambda: [C.JointVelocityConstraint(p["vlim"]), _ub_class(C)(acc(), ub, xb)]  # noqa: E731
        alg = lambda cons: pkg.algorithm.TOPPRA(cons, path, gridpoints=p["grid"], solver_wrapper="seidel")  # noqa: E731
        out = dict(ub=alg(mk()).compute_parameterization(0, 0, return_data=True),
                   ub_X=alg(mk()).compute_feasible_sets(), ub_L=alg(mk()).compute_reachable_sets(0.0, sdmax))
        var = C.JointVelocityConstraintVarying(lambda s: p["vlim"] * (k0 + k1 * s))
        out["var_xbound"] = var.compute_constraint_params(path, p["grid"])[-1]
        out["var"] = alg([var, acc()]).compute_parameterization(0, 0, return_data=True)
        if dof <= 7:
            tau = C.JointTorqueConstraint(inv_dyn_numpy, taulim, fric, discretization_scheme=scheme)
            inst = alg([C.JointVelocityConstraint(p["vlim"]), tau])
            out["torque"] = inst.compute_parameterization(p["sd0"], p["sd1"], return_data=True)
            out["torque code"] = inst.problem_data.return_code.name
        return out
    a, b = ta.both(run)
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, tuple):
            assert all(same(u, w) for u, w in zip(x, y)), "constraint producers: " + k
        elif isinstance(x, str):
            assert x == y, k
        else:
            assert same(x, y), "constraint producers: " + k
    hit(hist, "ubound")
    hit(hist, "varying velocity")
    if "torque" in a:
        hit(hist, "torque scheme %d" % scheme)


# ---- the campaign ---------------------------------------------------------------------------------------------------------
BATCH_SIZES = {"gpu": (1, 31, 33, 129), "cpu_double": (1, 3)}


def check_problem(ta, seed, hist, k):
    """Every family on the problem of `seed`; k picks the batch size and the rarer (larger) draws."""
    rng = np.random.RandomState(seed)
    p = random_shaped_problem(rng)
    if len(p["ss"]) < 3:
        p = random_shaped_problem(np.random.RandomState(seed + 10 ** 6))
    mode = "gpu" if ta.gpu else "cpu_double"
    check_propose(ta, p, rng, hist)
    sizes = BATCH_SIZES[mode]
    check_batch(ta, p, rng, hist, sizes[k % len(sizes)])
    check_sd_bisect(ta, rng, hist, int(rng.randint(1, 40)), int(rng.choice([2, 3, 17, 100, 500])), ragged=bool(k % 2))
    if len(p["grid"]) <= 100:
        check_toppra_sd(ta, p, rng, hist)
        check_reachable(ta, p, rng, hist)
    check_time_stamps(ta, rng, hist, (129, 257)[k % 2] if ta.gpu else 9)
    check_param_outputs(ta, p, rng, hist)
    check_constraints(ta, p, rng, hist)
    hit(hist, "problems")


def check_large(ta, seed, hist):
    """The rare sizes: a batch of about 2000 paths and a ragged sd_bisect batch beyond 3072 gridpoints."""
    rng = np.random.RandomState(seed)
    p = random_shaped_problem(rng)
    while len(p["ss"]) < 3 or len(p["grid"]) > 200:
        p = random_shaped_problem(rng)
    check_batch(ta, p, rng, hist, 2000 if ta.gpu else 40)
    check_sd_bisect(ta, rng, hist, 6, 3500, ragged=True)


FLOORS = ("propose status 0", "propose status 1", "propose status <0", "propose converged on the last pass",
          "propose >32 segments", "propose >64 segments", "sd fast", "sd slow", "sd bisect", "sd want = d_fast",
          "sd want = d_slow", "sd status_in 3", "sd status 1", "sd Gmax > 3072", "reach 1-variable", "reach fail_stage > 0",
          "stamps 5 s rule", "stamps 5 s rule at TINY", "stamps dropped knot", "batch fused", "batch records",
          "batch proposed grid", "reach ragged", "ubound", "torque scheme 0", "torque scheme 1")


GPU_ONLY = ("sd Gmax > 3072", "reach ragged")


def campaign(ta, seeds):
    hist, t0 = {}, time.time()
    for k, seed in enumerate(seeds):
        check_problem(ta, seed, hist, k)
    check_large(ta, seeds[0], hist)
    return hist, time.time() - t0


def test_callers_equal_the_oracle_on_randomly_shaped_problems(ta):
    n = N_PROBLEMS["gpu" if ta.gpu else "cpu_double"]
    hist, wall = campaign(ta, REGRESSION_SEEDS + list(range(SEED0, SEED0 + n)))
    print("\ncaller campaign (%s): %d problems in %.1f s; %s" % ("gpu" if ta.gpu else "cpu_double", hist["problems"], wall,
                                                               sorted(hist.items())))
    missing = [k for k in FLOORS if not hist.get(k) and (ta.gpu or k not in GPU_ONLY)]
    assert not missing, "branches never reached: %s" % missing
