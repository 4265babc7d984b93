"""BatchTOPPRAsd, feasible sets, reachable sets and robust solves on per-path (ragged) grids and in record chunks.

  * GPU, against tests/golden/ragged_batch.npz (the UNMODIFIED reference with gridpoints=None, make_golden_ragged.py):
    BatchTOPPRAsd, compute_feasible_sets and compute_reachable_sets on proposed grids, bit for bit, NaN past glen.
  * GPU, against the common-grid entries: every path of a ragged batch equals the same path solved alone at B = 1 on its
    unpadded grid, for every ragged method (robust ones included: they have no reference) and an order-6 path.
  * GPU: each kernel build launched with a non-null glen (torch.profiler); padding poisoned with NaN / +-1e300 changes
    nothing; chunked results equal unchunked ones bit for bit.
  * CPU: the launch plans through the recording library, the new entries' argument errors through the real library,
    and the host logic replayed against the fixture on oracle-backed doubles of the ragged engine forms."""
import ctypes

import numpy as np
import pytest

import cpu_engine
from test_kernel_builds import launched

GOLD = "ragged_batch"


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _h(t):
    return t.detach().cpu().numpy()


def _cons(ta, g, sl=slice(None)):
    return [ta.constraint.JointVelocityConstraint(g["vlim"][sl]), ta.constraint.JointAccelerationConstraint(g["alim"][sl])]


def _check_reference(ta, g, fused):
    path = ta.BatchSplineInterpolator(g["ss"], g["way"])
    glen = g["glen"]
    sd = ta.BatchTOPPRAsd(_cons(ta, g), path, fused=fused)
    assert np.array_equal(_h(sd.glen), glen)
    grid = _h(sd.d_grid)
    for b, n in enumerate(glen):
        assert np.array_equal(grid[b, :n], g["grid"][b, :n])
    sd.set_desired_duration(g["sd_desired"])
    res = sd.compute_parameterization(g["sd_start"], 0.0)
    h = res.to_host()
    assert np.array_equal(h["status"], g["sd_status"]) and h["status"].any()          # path 2 is uncontrollable
    assert _same(h["sd"], g["sd_sd"]) and _same(h["sdd"], g["sd_sdd"])
    inst = ta.BatchTOPPRA(_cons(ta, g), path, fused=fused)
    assert _same(_h(inst.compute_feasible_sets()), g["X"])
    L, X, fail = inst.compute_reachable_sets(g["sdmin"], g["sdmax"])
    assert _same(_h(X), g["X"]) and _same(_h(L), g["L"])
    real = np.arange(g["L"].shape[1])[None, :] < glen[:, None]
    nan_rows = np.isnan(g["L"]).any(axis=2) & real
    first = np.where(nan_rows.any(axis=1), nan_rows.argmax(axis=1), -1)
    assert np.array_equal(_h(fail), first) and (first >= 0).sum() >= 1
    _check_ubound_reference(ta, g, path)


def _check_ubound_reference(ta, g, path):
    """The u-bound case: records with a u-bound pair (TB_SCAN_UBOUND) on the proposed grids of the first 8 paths.
    The batched API takes that user constraint for one path at a time only, so the records are assembled here as the
    single-path API does: vel + acc rows (K1, interpolation), then the constraint's x-bound and u-bound intersected in."""
    torch, eng = ta.engine.torch_mod(), ta.engine
    nb = len(g["ub_ulim"])
    sub = path.chunk(0, nb)
    glen = g["glen"][:nb]
    G = g["grid"].shape[1]
    dev = path.device
    grid_h = np.where(np.isnan(g["grid"][:nb]), 1.0, g["grid"][:nb])
    grid, d_glen = eng.as_device(grid_h, dev), eng.as_device(glen, dev, torch.int32)
    R = 4 * g["way"].shape[2]
    rec, _ = eng.alloc_records(nb, G, R, dev, ubound=True)
    eng.init_bounds(rec, R)
    eng.coeff_velacc(sub.d_ppoly, sub.d_ss, grid, eng.as_device(g["vlim"][:nb], dev), eng.as_device(g["alim"][:nb], dev),
                     True, rec, R)
    ulim = g["ub_ulim"][:, None]
    ub = eng.as_device(np.stack((-ulim * (1.0 + grid_h), ulim * (2.0 - grid_h)), axis=-1), dev)
    xb = eng.as_device(np.stack((np.zeros_like(grid_h), 40.0 + 30 * grid_h), axis=-1), dev)
    rec[:, :, 3 * R + 2] = torch.maximum(rec[:, :, 3 * R + 2], ub[..., 0])
    rec[:, :, 3 * R + 3] = torch.minimum(rec[:, :, 3 * R + 3], ub[..., 1])
    rec[:, :, 3 * R] = torch.maximum(rec[:, :, 3 * R], xb[..., 0])
    rec[:, :, 3 * R + 1] = torch.minimum(rec[:, :, 3 * R + 1], xb[..., 1])
    assert eng.has_ubound(rec, R)
    assert _same(_h(eng.feasible_sets(rec, R, grid, glen=d_glen)), g["ub_X"])
    zero, top = eng.as_device(np.zeros(nb), dev), eng.as_device(np.full(nb, 0.3), dev)
    out = eng.reachable_sets(rec, R, grid, zero, top, glen=d_glen)
    assert _same(_h(out["X"]), g["ub_X"]) and _same(_h(out["L"]), g["ub_L"])


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [None, False])
def test_ragged_methods_equal_the_reference(golden, fused):
    import toppra_b200 as ta
    _check_reference(ta, golden(GOLD), fused)


# ---- GPU: ragged = each path alone on its own grid ------------------------------------------------------------------
def _robust(ta, g, sl):
    acc = ta.constraint.JointAccelerationConstraint(g["alim"][sl])
    return [ta.constraint.JointVelocityConstraint(g["vlim"][sl]), ta.constraint.RobustLinearConstraint(acc, [0.02, 0.01, 0.01], 1)]


def _solve_all(ta, cons, path, grid, glen, sdmin, sdmax, desired, robust):
    """Every ragged method of one problem -> {name: host array}."""
    out = {}
    inst = ta.BatchTOPPRA(cons, path, grid, glen=glen, fused=False)
    out["X"] = _h(inst.compute_feasible_sets())
    if robust:
        r = inst.compute_parameterization(0.0, 0.0)
        out.update(K=_h(r.K), sd=_h(r.sd), sdd=_h(r.sdd), status=_h(r.status))
        K, st = inst.compute_controllable_sets(sdmin, sdmin)
        out.update(Kc=_h(K), stc=_h(st))
        return out
    L, X, fail = inst.compute_reachable_sets(sdmin, sdmax)
    out.update(L=_h(L), X2=_h(X), fail=_h(fail))
    K, st = inst.compute_controllable_sets(sdmin, sdmax)
    out.update(Kc=_h(K), stc=_h(st))
    sd = ta.BatchTOPPRAsd(cons, path, grid, glen=glen, fused=False)
    sd.set_desired_duration(desired)
    r = sd.compute_parameterization(0.0, 0.0)
    out.update(sd=_h(r.sd), sdd=_h(r.sdd), status=_h(r.status), alpha=_h(r.alpha))
    return out


def _ragged_vs_single(ta, g, robust, make_path):
    B = 6
    sl = slice(0, B)
    glen = g["glen"][sl].copy()
    glen[1] = 40                                                      # a short path: most of its row is padding
    G = int(glen.max())
    grid = np.ones((B, G))
    for b in range(B):
        n = glen[b]
        grid[b, :n] = g["grid"][b, :n] if b != 1 else np.linspace(0, 1, n)
    sdmin, sdmax = g["sdmin"][sl], g["sdmax"][sl]
    desired = g["sd_desired"][sl]
    ragged = _solve_all(ta, (_robust if robust else _cons)(ta, g, sl), make_path(sl), grid, glen, sdmin, sdmax, desired,
                        robust)
    for b in range(B):
        n = glen[b]
        one = _solve_all(ta, (_robust if robust else _cons)(ta, g, slice(b, b + 1)), make_path(slice(b, b + 1)),
                         grid[b, :n], None, sdmin[b:b + 1], sdmax[b:b + 1], desired[b:b + 1], robust)
        for key, want in one.items():
            got = ragged[key][b]
            if got.ndim >= 1 and got.shape[0] in (G, G - 1) and key not in ("alpha",):
                m = want.shape[1]
                assert _same(got[:m], want[0]), (key, b)
                assert np.isnan(got[m:]).all(), (key, b)
            else:
                assert _same(got, want[0]), (key, b)


@pytest.mark.gpu
@pytest.mark.parametrize("robust", [False, True])
def test_ragged_batch_equals_each_path_alone(golden, robust):
    import toppra_b200 as ta
    g = golden(GOLD)
    _ragged_vs_single(ta, g, robust, lambda sl: ta.BatchSplineInterpolator(g["ss"], g["way"][sl]))


@pytest.mark.gpu
def test_ragged_order6_path_equals_each_path_alone(golden):
    import toppra_b200 as ta
    from scipy.interpolate import make_interp_spline
    g = golden(GOLD)
    from scipy.interpolate import PPoly
    knots = np.linspace(0, 1, 8)
    c = []
    for b in range(6):                      # quintic interpolating splines per joint, the zero-length end pieces dropped
        y = np.random.RandomState(b).randn(8, 7)
        pps = [PPoly.from_spline(make_interp_spline(knots, y[:, j], k=5)) for j in range(7)]
        keep = np.nonzero(np.diff(pps[0].x) > 0)[0]
        c.append(np.stack([p.c[:, keep] for p in pps], axis=-1))
        x = pps[0].x[np.append(keep, keep[-1] + 1)]
    c = np.stack(c)
    assert c.shape[1] == 6
    _ragged_vs_single(ta, g, False, lambda sl: ta.BatchPiecewisePolyPath(x, c[sl]))


# ---- GPU: raw records at the rows-per-lane edges, under the profiler -------------------------------------------------
ROW_COUNTS = {1: 29, 2: 61, 3: 93, 4: 124}           # nC = R + 2: 31, 63, 95, 126 -> RPL 1..4


def _raw(R, ub=False, B=5, G=23, seed=0):
    """Random stage records (feasible at u = 0, x small) on ragged grids: (records, grid, glen) on the device."""
    import torch
    ta = __import__("toppra_b200")
    rng = np.random.RandomState(seed + R)
    dev = ta.engine.default_device()
    rec, W = ta.engine.alloc_records(B, G, R, dev, ubound=ub)
    host = np.zeros((B, G, W))
    host[..., :R] = rng.randn(B, G, R)
    host[..., R:2 * R] = 0.3 * rng.randn(B, G, R)
    host[..., 2 * R:3 * R] = -0.5 - rng.rand(B, G, R)
    host[..., 3 * R], host[..., 3 * R + 1] = 0.0, 2.0 + rng.rand(B, G)
    if ub:
        host[..., 3 * R + 2], host[..., 3 * R + 3] = -1.0 - rng.rand(B, G), 1.0 + rng.rand(B, G)
    rec.copy_(torch.from_numpy(host))
    glen = np.array([G, 3, 1, G - 5, 11][:B], dtype=np.int32)
    grid = np.ones((B, G))
    for b, n in enumerate(glen):
        grid[b, :n] = np.linspace(0, 1, n) if n > 1 else [0.0]
    return rec, ta.engine.as_device(grid, dev), ta.engine.as_device(glen, dev, torch.int32), glen


def _single(rec, grid, b, n):
    return rec[b:b + 1, :n].contiguous(), grid[b, :n].contiguous()


def _compare_rows(got, want, what):
    m = want.shape[1]
    assert _same(got[:m], want[0]), ("differs from the path alone", what)
    assert np.isnan(got[m:]).all(), ("padding not NaN", what)


def _profiled(fn):
    """(fn(), kernel keys launched) under torch.profiler.  Kineto (torch 2.11, H100) now and then returns a capture with
    no device activity at all, not even the result copies (tests/test_kernel_builds.py meets the same); the calls here
    are deterministic, so such a capture is taken again, at most twice."""
    import torch
    for _ in range(3):
        with launched() as k:
            out = fn()
            torch.cuda.synchronize()
        if k:
            break
    assert k, "torch.profiler captured no device activity in three attempts"
    return out, k


def _assert_launched(key, k):
    assert key in k, "%s was not launched; launched: %s" % (key, sorted(k))


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 2, 3, 4])
def test_ragged_kernel_builds(rpl):
    ta = __import__("toppra_b200")
    eng = ta.engine
    R = ROW_COUNTS[rpl]
    dev = eng.default_device()
    for ub in (False, True):
        rec, grid, glen, gl = _raw(R, ub)
        B = len(gl)
        lo = eng.as_device(np.full(B, 0.1), dev)
        hi = eng.as_device(np.full(B, 0.3), dev)
        (X, out), k = _profiled(lambda: (_h(eng.feasible_sets(rec, R, grid, glen=glen)),
                                         eng.reachable_sets(rec, R, grid, lo, hi, glen=glen)))
        _assert_launched("feasible_kernel<%d>" % rpl, k)
        _assert_launched("reachable_kernel<%d,%s>" % (rpl, "true" if ub else "false"), k)
        for b, n in enumerate(gl):
            r1, g1 = _single(rec, grid, b, n)
            _compare_rows(X[b], _h(eng.feasible_sets(r1, R, g1)), ("feasible X", ub, b))
            one = eng.reachable_sets(r1, R, g1, lo[b:b + 1], hi[b:b + 1])
            for key in ("X", "L"):
                _compare_rows(_h(out[key])[b], _h(one[key]), ("reachable " + key, ub, b))
            assert _h(out["fail_stage"])[b] == _h(one["fail_stage"])[0], ("reachable fail_stage", ub, b)
    rec, grid, glen, gl = _raw(R)
    ell = np.array([0.02, 0.01, 0.01])
    (rob, feas), k = _profiled(lambda: (eng.scan_robust(rec, R, 0, R // 2, ell, grid, glen=glen),
                                        eng.scan_robust(rec, R, 0, R // 2, ell, grid, feasible_sets=True, glen=glen)))
    _assert_launched("scan_robust_kernel<%d>" % rpl, k)
    for b, n in enumerate(gl):
        r1, g1 = _single(rec, grid, b, n)
        one = eng.scan_robust(r1, R, 0, R // 2, ell, g1)
        for key in ("K", "sd", "u"):
            _compare_rows(_h(rob[key])[b], _h(one[key]), ("robust " + key, b))
        assert _h(rob["status"])[b] == _h(one["status"])[0], ("robust status", b)
        _compare_rows(_h(feas["K"])[b], _h(eng.scan_robust(r1, R, 0, R // 2, ell, g1, feasible_sets=True)["K"]),
                      ("robust feasible", b))


SENTINEL = 0x7FF4DEAD0000BEEF      # a NaN payload no kernel writes: an entry still holding it was never written


def _sentinel(shape, dtype="f8"):
    import torch
    if dtype == "i4":
        return torch.full(shape, -12345, dtype=torch.int32, device="cuda")
    return torch.full(shape, SENTINEL, dtype=torch.int64, device="cuda").view(torch.float64)


def _unwritten(t):
    import torch
    if t.dtype == torch.int32:
        return int((t == -12345).sum())
    return int((t.view(torch.int64) == SENTINEL).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("rpl", [1, 2, 3, 4])
def test_ragged_entries_write_every_output_entry(rpl):
    """The four ragged entries called directly with outputs pre-filled with a sentinel: every entry, real or padding,
    of every output is written, in every mode (feasible / reachable with and without u-bounds, robust full scan,
    backward only and feasible sets, sd_bisect)."""
    import torch
    from toppra_b200 import _lib
    ta = __import__("toppra_b200")
    lib, P, S = _lib.load(), _lib.ptr, _lib.stream_ptr()
    R = ROW_COUNTS[rpl]
    for ub in (False, True):
        rec, grid, glen, gl = _raw(R, ub)
        B, G, W = rec.shape
        flags = 64 if ub else 0
        X = _sentinel((B, G, 2))
        _lib.check(lib.tb_feasible_sets_ragged(P(rec), W, R, P(grid), 0, B, G, P(glen), flags, P(X), S), "feasible")
        lo = ta.engine.as_device(np.full(B, 0.1), rec.device)
        X2, L, fs = _sentinel((B, G, 2)), _sentinel((B, G, 2)), _sentinel((B,), "i4")
        _lib.check(lib.tb_reachable_sets_ragged(P(rec), W, R, P(grid), 0, B, G, P(glen), P(lo), None, flags, P(X2),
                                                P(L), P(fs), S), "reachable")
        torch.cuda.synchronize()
        for name, t in (("X", X), ("X2", X2), ("L", L), ("fail_stage", fs)):
            assert _unwritten(t) == 0, (name, ub, _unwritten(t))
    rec, grid, glen, gl = _raw(R)
    B, G, W = rec.shape
    ell = np.array([0.02, 0.01, 0.01])
    for mode in (0, 1, 2):
        K, st, fs = _sentinel((B, G, 2)), _sentinel((B,), "i4"), _sentinel((B,), "i4")
        sd, u = (_sentinel((B, G)), _sentinel((B, G - 1))) if mode == 0 else (None, None)
        _lib.check(lib.tb_scan_robust_ragged(P(rec), W, R, 0, R // 2, ctypes.c_void_p(ell.ctypes.data), P(grid), 0, B, G,
                                             P(glen), None, None, mode, P(K), P(sd), P(u), P(st), P(fs), None, S),
                   "robust")
        torch.cuda.synchronize()
        for name, t in (("K", K), ("sd", sd), ("u", u), ("status", st), ("fail_stage", fs)):
            if t is not None:
                assert _unwritten(t) == 0, (name, mode, _unwritten(t))
    rng = np.random.RandomState(rpl)
    xs = ta.engine.as_device(rng.rand(B, G) + 0.1, rec.device)
    xf = xs + 1.0
    uf, us = (ta.engine.as_device(rng.randn(B, G - 1), rec.device) for _ in range(2))
    want = ta.engine.as_device(np.array([1.5, 0.8, 1.2, 100.0, 0.01]), rec.device)
    sd, sdd, info, st = _sentinel((B, G)), _sentinel((B, G - 1)), _sentinel((B, 4)), _sentinel((B,), "i4")
    _lib.check(lib.tb_sd_bisect_ragged(P(xf), P(uf), P(xs), P(us), P(grid), 0, B, G, P(glen), P(want), 1e-5, 200, None,
                                       P(sd), P(sdd), P(info), P(st), S), "sd_bisect")
    torch.cuda.synchronize()
    for name, t in (("sd", sd), ("sdd", sdd), ("info", info), ("status", st)):
        assert _unwritten(t) == 0, (name, _unwritten(t))


@pytest.mark.gpu
def test_ragged_sd_bisect_build():
    import torch
    eng = __import__("toppra_b200").engine
    dev = eng.default_device()
    rng = np.random.RandomState(3)
    B, G = 5, 30
    gl = np.array([30, 2, 17, 9, 25], dtype=np.int32)
    grid = np.ones((B, G))
    for b, n in enumerate(gl):
        grid[b, :n] = np.linspace(0, 1, n)
    xs = rng.rand(B, G) + 0.1
    xf = xs + rng.rand(B, G)
    uf, us = rng.randn(B, G - 1), rng.randn(B, G - 1)
    t = lambda a: eng.as_device(a, dev)  # noqa: E731
    want = np.array([1.5, 0.8, 1.2, 100.0, 0.01])
    out, k = _profiled(lambda: eng.sd_bisect(t(xf), t(uf), t(xs), t(us), t(grid), t(want),
                                             glen=eng.as_device(gl, dev, torch.int32)))
    _assert_launched("sd_bisect_kernel", k)
    for b, n in enumerate(gl):
        one = eng.sd_bisect(t(xf[b:b + 1, :n]), t(uf[b:b + 1, :n - 1]), t(xs[b:b + 1, :n]), t(us[b:b + 1, :n - 1]),
                            t(grid[b, :n]), t(want[b:b + 1]))
        _compare_rows(_h(out["sd"])[b], _h(one["sd"]), ("sd", b))
        _compare_rows(_h(out["u"])[b], _h(one["u"]), ("u", b))
        assert _same(_h(out["info"])[b], _h(one["info"])[0]) and _h(out["status"])[b] == _h(one["status"])[0], b


@pytest.mark.gpu
def test_poisoned_padding_changes_nothing():
    import torch
    eng = __import__("toppra_b200").engine
    dev = eng.default_device()
    R = 29
    rec, grid, glen, gl = _raw(R)
    B = len(gl)
    lo = eng.as_device(np.full(B, 0.1), dev)
    ell = np.array([0.02, 0.01, 0.01])

    def run(rec, grid):
        return dict(X=_h(eng.feasible_sets(rec, R, grid, glen=glen)),
                    L=_h(eng.reachable_sets(rec, R, grid, lo, lo, glen=glen)["L"]),
                    K=_h(eng.scan_robust(rec, R, 0, R // 2, ell, grid, glen=glen)["sd"]),
                    F=_h(eng.scan_robust(rec, R, 0, R // 2, ell, grid, feasible_sets=True, glen=glen)["K"]))

    rng = np.random.RandomState(7)
    G = grid.shape[1]
    xs = eng.as_device(rng.rand(B, G) + 0.1, dev)
    xf = xs + 1.0
    uf, us = (eng.as_device(rng.randn(B, G - 1), dev) for _ in range(2))
    want = eng.as_device(np.array([1.5, 0.8, 1.2, 100.0, 0.01]), dev)

    def run_sd(xf, uf, xs, us, grid):
        out = eng.sd_bisect(xf, uf, xs, us, grid, want, glen=glen)
        return {"sd_" + key: _h(v) for key, v in out.items()}

    clean = dict(run(rec, grid), **run_sd(xf, uf, xs, us, grid))
    for value in (float("nan"), 1e300, -1e300):
        r2, g2 = rec.clone(), grid.clone()
        xf2, uf2, xs2, us2 = xf.clone(), uf.clone(), xs.clone(), us.clone()
        for b, n in enumerate(gl):
            r2[b, n:] = value
            g2[b, n:] = value
            xf2[b, n:], xs2[b, n:] = value, value
            uf2[b, max(n - 1, 0):], us2[b, max(n - 1, 0):] = value, value
        torch.cuda.synchronize()
        dirty = dict(run(r2, g2), **run_sd(xf2, uf2, xs2, us2, g2))
        for key in clean:
            assert _same(dirty[key], clean[key]), (key, value)


# ---- GPU: chunks ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ragged", [False, True])
def test_chunked_equals_unchunked(golden, ragged):
    import toppra_b200 as ta
    g = golden(GOLD)
    path = ta.BatchSplineInterpolator(g["ss"], g["way"])
    grid = None if ragged else np.linspace(0, 1, 150)
    whole = ta.BatchTOPPRA(_cons(ta, g), path, grid, fused=False)
    per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
    for kind in ("linear", "robust"):
        cons = (lambda: _cons(ta, g)) if kind == "linear" else (lambda: _robust(ta, g, slice(None)))
        one = ta.BatchTOPPRA(cons(), path, grid, fused=False)
        parts = ta.BatchTOPPRA(cons(), path, grid, fused=False, max_record_bytes=5 * per_path)
        assert parts.chunk_size() == 5 and one.chunk_size() == 16                     # chunks of 5, 5, 5, 1
        assert _same(_h(parts.compute_feasible_sets()), _h(one.compute_feasible_sets()))
        a, b = parts.compute_controllable_sets(0.0, 0.0), one.compute_controllable_sets(0.0, 0.0)
        assert _same(_h(a[0]), _h(b[0])) and _same(_h(a[1]), _h(b[1]))
        if kind == "robust":
            ra, rb = parts.compute_parameterization(), one.compute_parameterization()
            assert _same(_h(ra.sd), _h(rb.sd)) and _same(_h(ra.K), _h(rb.K))
            continue
        a, b = parts.compute_reachable_sets(g["sdmin"], g["sdmax"]), one.compute_reachable_sets(g["sdmin"], g["sdmax"])
        for x, y in zip(a, b):
            assert _same(_h(x), _h(y))
        a, b = parts.compute_controllable_sets(0.0, 0.2), one.compute_controllable_sets(0.0, 0.2)
        assert _same(_h(a[0]), _h(b[0]))
        res = []
        for inst in (ta.BatchTOPPRAsd(cons(), path, grid, fused=False, max_record_bytes=5 * per_path),
                     ta.BatchTOPPRAsd(cons(), path, grid, fused=False)):
            inst.set_desired_duration(g["sd_desired"])
            r = inst.compute_parameterization(g["sd_start"], 0.0)
            res.append([_h(r.sd), _h(r.sdd), _h(r.status), _h(r.alpha), _h(r.duration_fast), _h(r.K)])
        for x, y in zip(*res):
            assert _same(x, y)


# ---- CPU: launch plans ------------------------------------------------------------------------------------------------
from test_engine_marshalling import lib, named_args  # noqa: E402,F401  (lib: fixture)


def _calls(lib, start, name):  # noqa: F811
    return [named_args(n, a) for n, a in lib.calls[start:] if n == name]


def _plan(lib, start):  # noqa: F811
    return [n for n, _ in lib.calls[start:] if n not in ("tb_record_doubles", "tb_spline_fit_workspace_doubles")]


def _poke(pointer, array):
    ctypes.memmove(pointer.value, array.ctypes.data, array.nbytes)


LENS = np.array([20, 35, 35, 28, 50, 31, 22, 47], dtype=np.int32)


@pytest.fixture
def proposing(lib, monkeypatch):  # noqa: F811
    def propose(*args):
        grid = np.ones((len(LENS), args[10]))
        for b, n in enumerate(LENS):
            grid[b, :n] = np.linspace(0, 1, n)
        _poke(args[11], grid)
        _poke(args[13], LENS)
        _poke(args[14], np.zeros(len(LENS), dtype=np.int32))
        return 0
    monkeypatch.setitem(lib.RESULTS, "tb_propose_gridpoints", propose)
    return lib


def _problem(dof=6):
    import toppra_b200 as ta
    rng = np.random.RandomState(0)
    path = ta.BatchSplineInterpolator(np.linspace(0, 1, 5), rng.randn(len(LENS), 5, dof))
    lim = np.tile(np.array([[-1.0, 1.0]]), (dof, 1))
    return ta, path, ta.constraint.JointVelocityConstraint(lim), ta.constraint.JointAccelerationConstraint(lim)


def test_ragged_plans_call_the_ragged_entries(proposing):
    lib = proposing
    ta, path, vel, acc = _problem()
    Gmax = int(LENS.max())
    mark = len(lib.calls)
    inst = ta.BatchTOPPRA([vel, acc], path)
    inst.compute_feasible_sets()
    inst.compute_reachable_sets(0.0, 0.1)
    assert _plan(lib, mark) == ["tb_propose_gridpoints", "tb_coeff_velacc", "tb_feasible_sets_ragged",
                                "tb_reachable_sets_ragged"]
    mark = len(lib.calls)
    sd = ta.BatchTOPPRAsd([vel, acc], path)
    sd.set_desired_duration(3.0)
    sd.compute_parameterization()
    assert _plan(lib, mark) == ["tb_propose_gridpoints", "tb_xbound_velocity", "tb_scan_velacc_ragged",
                                "tb_scan_velacc_ragged", "tb_sd_bisect_ragged"]
    mark = len(lib.calls)
    robust = ta.constraint.RobustLinearConstraint(acc, [0.1, 0.1, 0.1], 1)
    rob = ta.BatchTOPPRA([vel, robust], path)
    rob.compute_parameterization()
    rob.compute_feasible_sets()
    assert _plan(lib, mark)[-2:] == ["tb_scan_robust_ragged", "tb_scan_robust_ragged"]
    for name in ("tb_feasible_sets_ragged", "tb_reachable_sets_ragged", "tb_sd_bisect_ragged", "tb_scan_robust_ragged"):
        for args in _calls(lib, 0, name):
            assert args["G"] == Gmax and args["glen"] is not None and args["grid_shared"] == 0, name
    with pytest.raises(NotImplementedError):
        rob.compute_reachable_sets(0.0, 0.0)
    with pytest.raises(NotImplementedError):
        rob.compute_controllable_sets(0.0, 0.1)


@pytest.mark.parametrize("ragged", [False, True])
def test_chunk_plans(proposing, ragged):
    lib = proposing
    ta, path, vel, acc = _problem()
    grid = None if ragged else np.linspace(0, 1, 50)
    whole = ta.BatchTOPPRA([vel, acc], path, grid, fused=False)
    per_path = 8 * ta.engine.record_doubles(whole.R) * whole.G
    sfx = "_ragged" if ragged else ""
    cases = [("feasible", "tb_feasible_sets" + (sfx or "_ex"), lambda i: i.compute_feasible_sets()),
             ("reachable", "tb_reachable_sets" + sfx, lambda i: i.compute_reachable_sets(0.0, 0.1)),
             ("controllable", "tb_scan_ragged", lambda i: i.compute_controllable_sets(0.0, 0.1))]
    for what, entry, call in cases:
        # the set methods chunk their records even when the scan is fused; the controllable sets of a fused problem
        # need no records, so that case takes the record scan
        inst = ta.BatchTOPPRA([vel, acc], path, grid, max_record_bytes=3 * per_path,
                              fused=False if what == "controllable" else None)
        mark = len(lib.calls)
        call(inst)
        k1 = _calls(lib, mark, "tb_coeff_velacc")
        runs = _calls(lib, mark, entry)
        assert [a["B"] for a in runs] == [3, 3, 2] and [a["B"] for a in k1] == [3, 3, 2], what
        assert len({a["records"].value for a in runs}) == 1, what                 # one record buffer, reused
        stride = 8 * 4 * 4 * 6
        assert [a["ppoly"].value - k1[0]["ppoly"].value for a in k1] == [0, 3 * stride, 6 * stride], what
        if ragged:
            g0 = runs[0]["grid"].value
            assert [a["grid"].value - g0 for a in runs] == [0, 3 * 8 * whole.G, 6 * 8 * whole.G], what
    sd = ta.BatchTOPPRAsd([vel, acc], path, grid, fused=False, max_record_bytes=3 * per_path)
    sd.set_desired_duration(np.arange(1.0, 9.0))
    mark = len(lib.calls)
    sd.compute_parameterization()
    plan = _plan(lib, mark)
    assert plan == ["tb_coeff_velacc", "tb_scan_ragged", "tb_scan_ragged", "tb_sd_bisect" + sfx] * 3
    bis = _calls(lib, mark, "tb_sd_bisect" + sfx)
    assert [a["B"] for a in bis] == [3, 3, 2]
    d0 = bis[0]["desired_duration"].value
    assert [a["desired_duration"].value - d0 for a in bis] == [0, 24, 48]


# ---- CPU: argument errors of the new entries (real library) ----------------------------------------------------------
def test_ragged_entries_reject_glen_with_a_shared_grid():
    import torch
    if torch.cuda.is_available():
        pytest.skip("validation-only calls with host addresses: run without a GPU")
    from toppra_b200 import _lib
    from test_cabi_errors import _call
    lib = _lib.load()
    mem = np.zeros(1 << 16)
    buf = (mem, ctypes.c_void_p(mem.ctypes.data))
    ell = np.zeros(3)
    cases = {"tb_feasible_sets_ragged": dict(W=86, R=28, B=4, G=10, flags=0),
             "tb_reachable_sets_ragged": dict(W=86, R=28, B=4, G=10, flags=0),
             "tb_scan_robust_ragged": dict(W=86, R=28, conic_row0=0, conic_rows=28, B=4, G=10, flags=0,
                                           ellipsoid_host3=ctypes.c_void_p(ell.ctypes.data)),
             "tb_sd_bisect_ragged": dict(B=4, G=10, atol=1e-5, max_iter=10)}
    for name, kw in cases.items():
        rc, msg = _call(lib, name, buf, grid_shared=1, **kw)
        assert rc == -1 and "ragged" in msg, (name, rc, msg)


# ---- CPU: host logic on oracle-backed doubles of the ragged engine forms ----------------------------------------------
def _ragged_double(fn):
    """A double of an engine function's ragged form: each path sliced to its own gridpoints (n, or n - 1 for per-stage
    arrays) and solved by the common-grid double `fn`; results padded with NaN to the batch's width."""
    import torch

    def call(*args, glen=None, **kw):
        if glen is None:
            return fn(*args, **kw)
        gl = cpu_engine._np(glen)
        B = len(gl)
        G = max(a.shape[1] for a in args if isinstance(a, torch.Tensor) and a.dim() >= 2 and a.shape[0] == B)
        parts = []
        for n in gl:
            b, n = len(parts), int(n)
            sub = []
            for a in args:
                if isinstance(a, torch.Tensor) and a.dim() >= 1 and a.shape[0] == B:
                    a = a[b:b + 1]
                    if a.dim() >= 2:
                        a = a[:, :n if a.shape[1] == G else n - 1]
                    a = a.contiguous()
                sub.append(a)
            kw2 = {key: (v[b:b + 1] if isinstance(v, torch.Tensor) and v.dim() >= 1 and v.shape[0] == B else v)
                   for key, v in kw.items()}
            parts.append(fn(*sub, **kw2))
        return _pad_parts(parts, G, B)
    return call


def _pad_parts(parts, G, B):
    import torch
    single = isinstance(parts[0], torch.Tensor)
    keys = ["_"] if single else list(parts[0])
    out = {}
    for key in keys:
        vals = [p if single else p[key] for p in parts]
        if vals[0] is None:
            out[key] = None
            continue
        v0 = vals[0]
        if v0.dim() >= 2 and key != "info" and key != "counters":
            width = G - 1 if key == "u" else G
            full = torch.full((B, width) + tuple(v0.shape[2:]), float("nan"), dtype=v0.dtype)
            for b, v in enumerate(vals):
                full[b, :v.shape[1]] = v[0]
        else:
            full = torch.cat([v.reshape((1,) + tuple(v.shape[1:])) for v in vals])
        out[key] = full
    return out["_"] if single else out


def _install_ragged(monkeypatch):
    ta = cpu_engine.install(monkeypatch)
    from toppra_b200 import engine
    for name in ("feasible_sets", "reachable_sets", "scan", "sd_bisect"):
        monkeypatch.setattr(engine, name, _ragged_double(getattr(cpu_engine, name)))
    return ta


def test_host_logic_against_the_fixture_on_the_oracle_double(monkeypatch, golden):
    ta = _install_ragged(monkeypatch)
    _check_reference(ta, golden(GOLD), False)
