"""CPU (-m "not gpu"): the scalar model of the scan kernel's min-x closure (tests/closure_model.c, same rule and margin
as toppra_b200/csrc/tb_scan.cu lp2d_impl) reproduces the sequential restatement bit for bit, closes most min-x LPs
of the benchmark, and needs its margin: with the margin at 0 it disagrees on near-degenerate and badly scaled rows.
The kernel itself is checked against the oracle by the -m gpu tests."""
import numpy as np

from closure_model import closure_model
from oracle import oracle as orc
from test_shortcut_model import _degenerate_rows, _paths


def _near_degenerate(rng, n):
    for it in range(n):
        G, R0 = rng.randint(5, 40), rng.randint(2, 10)
        rows = _degenerate_rows(rng, G, R0, it % 4, 10 ** rng.uniform(-14, -6))
        xb = np.stack((np.zeros(G), np.full(G, 10 ** rng.uniform(-2, 3))), axis=1)
        orc.solve_rows(rows, xb, np.linspace(0, 1, G), 0, 0)


def _badly_scaled(rng, n):
    """the row sets of test_shortcut_model.test_model_on_badly_scaled_problems"""
    for it in range(n):
        G, R = rng.randint(5, 40), rng.randint(2, 20)
        sa, sb, sc = 10 ** rng.uniform(-8, 1), 10 ** rng.uniform(-8, 1), 10 ** rng.uniform(-3, 5)
        if it % 3 == 0:
            a = np.cumsum(rng.randn(G, R) * 0.05, 0) * sa + rng.randn(1, R) * sa
            b = np.cumsum(rng.randn(G, R) * 0.05, 0) * sb + rng.randn(1, R) * sb
        else:
            a, b = rng.randn(G, R) * sa, rng.randn(G, R) * sb
        rows = np.stack((a, b, -rng.rand(G, R) * sc), axis=1)
        xb = np.stack((np.zeros(G), np.full(G, 1e8 if it % 2 else 10 ** rng.uniform(-2, 9))), axis=1)
        orc.solve_rows(rows, xb, np.linspace(0, 1, G), 0, 0)


def test_closure_on_benchmark_like_paths():
    """cfg 2 of bench.py (4096 paths x 7 DOF x 200 gridpoints, vel + acc): the closure ends most min-x LPs, and the
    re-solve count is the shortcut model's (the closure is the one re-solve it replaces)."""
    grid = np.linspace(0, 1, 200)
    with closure_model() as cm:
        for vel_active, B in ((False, 3072), (True, 1024)):
            c, x, vlim, alim = _paths(B, vel_active, 4321)
            r = orc.solve_velacc_batch(c, x, grid, vlim, alim, nthreads=1)
            assert not r["status"].any()
        st = cm.stats()
    with orc.shortcut_model() as sm:
        for vel_active, B in ((False, 3072), (True, 1024)):
            c, x, vlim, alim = _paths(B, vel_active, 4321)
            orc.solve_velacc_batch(c, x, grid, vlim, alim, nthreads=1)
        ref = sm.stats()
    assert st["mismatches"] == 0 and st["lps"] == 4096 * 398
    min_x_lps = 4096 * 199
    assert st["closed"] > 0.9 * min_x_lps
    assert st["resolves_model"] == ref["resolves_model"]


def test_closure_on_hard_rows():
    rng = np.random.RandomState(7)
    with closure_model() as cm:
        _near_degenerate(rng, 6000)
        _badly_scaled(rng, 6000)
        st = cm.stats()
    assert st["mismatches"] == 0 and st["closed"] > 10000 and st["close_declined"] > 500


def _mixed_sign(rng, n):
    """rows half of which have c of either sign, x boxes away from 0: rows after shortcut A's row m can fail at the
    closed point, so the closure has something to decline"""
    for it in range(n):
        G, R = rng.randint(5, 40), rng.randint(2, 20)
        sa, sb, sc = 10 ** rng.uniform(-8, 1), 10 ** rng.uniform(-8, 1), 10 ** rng.uniform(-3, 5)
        a, b = rng.randn(G, R) * sa, rng.randn(G, R) * sb
        c = -rng.rand(G, R) * sc
        c[:, R // 2:] = rng.randn(G, R - R // 2) * sc * 1e-3
        xb = np.stack((np.full(G, 10 ** rng.uniform(-3, 1) if it % 2 else 0.0), np.full(G, 10 ** rng.uniform(1, 3))), 1)
        orc.solve_rows(np.stack((a, b, c), axis=1), xb, np.linspace(0, 1, G), 0, 0)


def test_closure_certificate_matters():
    """The certificate declines closures the reference does not take; with it switched off (margin -inf: every row
    passes) the model disagrees with the reference."""
    for gap, ok in ((1e-7, True), (-np.inf, False)):
        with closure_model() as cm:
            cm.margin(gap)
            _mixed_sign(np.random.RandomState(8), 3000)
            st = cm.stats()
        assert st["closed"] > 50
        if ok:
            assert st["mismatches"] == 0 and st["close_declined"] > 10
        else:
            assert st["mismatches"] > 10
