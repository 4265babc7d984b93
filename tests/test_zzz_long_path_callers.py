"""GPU (-m gpu): the batched callers around the scan on long paths (115 and 300 knots), the part of
tests/test_long_paths.py that runs the package twice, on the kernels and on the oracle-backed engine double
(tests/cpu_engine.py), through the public API.  Like tests/test_zzz_caller_campaign.py it sorts after every test that
reads torch.profiler: in the same process, profiled captures that follow it have lost device activity (the first
kernels of a capture) on an H100 with torch 2.11, while the suite without it captured everything.

propose_gridpoints, feasible and reachable sets, BatchTOPPRAsd, the ConstAccel time grid and evaluation and
BatchParametrizeSpline are compared bit for bit, NaN equal to NaN, except the ConstAccel evaluation and the clamped re-fit
of BatchParametrizeSpline, which keep test_zzz_caller_campaign's tolerances."""
import numpy as np
import pytest
import torch

import cpu_engine
from oracle import oracle as orc
from test_long_paths import _batch_inputs, _gpu, _t, assert_same, host, same, velacc


class _Both(object):
    """Runs fn(pkg) on the kernels, then again with the oracle-backed engine double installed."""

    def __init__(self, monkeypatch):
        self.mp = monkeypatch
        self.pkg = _gpu()

    def __call__(self, fn):
        first = fn(self.pkg)
        with self.mp.context() as m:
            cpu_engine.install(m)
            return first, fn(self.pkg)


@pytest.mark.gpu
@pytest.mark.parametrize("nseg", [114, 299])
def test_callers_on_long_paths(nseg, monkeypatch):
    both = _Both(monkeypatch)
    B, dof, G = 32, 7, 150
    ss, way, vlim, alim = _batch_inputs(dof, nseg, B, 900 + nseg)
    c = np.stack([orc.cubic_spline_fit(ss, way[b]) for b in range(B)])
    grid = np.linspace(0, ss[-1], G)
    rng = np.random.RandomState(nseg)
    E = both.pkg.engine
    kw = dict(max_err_threshold=1e-2, max_iteration=100, max_seg_length=0.5, min_nb_points=100, max_points=8192)
    got = [host(x) for x in E.propose_gridpoints(_t(c), _t(ss), **kw)]
    want = [host(x) for x in cpu_engine.propose_gridpoints(torch.from_numpy(c), torch.from_numpy(ss), **kw)]
    for what, a, b in zip(("grid", "glen", "status"), got, want):
        assert_same(a, b, "propose_gridpoints " + what)
    assert (want[2] == 0).all() and want[1].min() > nseg

    sdmin = np.where(np.arange(B) % 3 == 0, 0.0, 0.25)
    sdmax = np.where(np.arange(B) % 2 == 0, sdmin, sdmin + 0.5)
    desired = 10 ** rng.uniform(-0.5, 1.5, B)
    frac = rng.rand(B, 8)                      # drawn once: both sides evaluate the same sample times

    def run(pkg):
        path = pkg.BatchSplineInterpolator.from_ppoly(ss, c)
        cons = velacc(pkg, vlim, alim, 1)
        inst = pkg.BatchTOPPRA(cons, path, grid)
        X = host(inst.compute_feasible_sets())
        L, _, fs = (host(x) for x in inst.compute_reachable_sets(sdmin, sdmax))
        sdi = pkg.BatchTOPPRAsd(cons, path, grid)
        sdi.set_desired_duration(desired)
        r = sdi.compute_parameterization(0.0, 0.0)
        fast = inst.compute_parameterization(0.0, 0.0).to_host()
        sd = np.maximum(np.nan_to_num(fast["sd"]), 1e-3)
        ca = pkg.BatchParametrizeConstAccel(path, grid, sd)
        t = host(ca.t_grid)
        ts = np.stack([np.r_[t[b, :: max(1, G // 20)], t[b, -1], t[b, -1] * frac[b]] for b in range(B)])
        q = [host(ca(ts, order)) for order in (0, 1, 2)]
        ps = pkg.BatchParametrizeSpline(path, grid, sd)
        return dict(X=X, L=L, fs=fs, sd=host(r.sd), sdd=host(r.sdd), st=host(r.status), alpha=host(r.alpha), t=t,
                    us=host(ca.us), q=q, ps_t=host(ps.t_knots), ps_n=host(ps.nkeep), ps_d=host(ps.durations),
                    ps_c=[(i, host(f.d_ppoly)) for i, f in ps.groups])

    a, b = both(run)
    for k in ("X", "L", "fs", "sd", "sdd", "st", "alpha", "t", "us", "ps_t", "ps_n", "ps_d"):
        assert_same(a[k], b[k], k)
    assert (a["st"] == 0).any() and np.isfinite(a["L"]).all(axis=(1, 2)).any()     # some paths solve, some sets reach
    scale = max(1.0, np.abs(c).max() * max(1.0, ss[-1]) ** 3)
    for order, tol in ((0, 1e-11), (1, 1e-9), (2, 1e-7)):     # test_zzz_caller_campaign's ConstAccel tolerances
        np.testing.assert_allclose(a["q"][order], b["q"][order], rtol=tol,
                                   atol=tol * max(scale, np.abs(b["q"][order]).max()), err_msg="ConstAccel %d" % order)
    for (ia, ca_), (ib, cb) in zip(a["ps_c"], b["ps_c"]):
        assert same(ia, ib)
        if not same(ca_, cb):                                 # the clamped re-fit: test_zzz_caller_campaign's bound
            np.testing.assert_allclose(ca_, cb, rtol=1e-11, atol=1e-12 * max(1.0, np.abs(cb).max()))
