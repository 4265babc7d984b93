"""One row per compiled kernel of libtoppra_b200.so: each row names a kernel build (template arguments included) and a
case that routes to it through the public `toppra_b200.engine` functions.  The GPU test runs the case under
torch.profiler, asserts that the row's build is among the launched kernels, and compares the outputs with a plain
reference: the oracle-backed engine double (tests/cpu_engine.py) fed the same records, or the oracle's batch solver on
the GPU's spline coefficients.  Without the profiler check a launcher change could silently turn a row into a duplicate
of another row.  The CPU test checks that the table lists exactly the kernels of the built library.

Exact builds are compared bit for bit (NaN equal to NaN).  The fast builds (TB_SCAN_FAST_LOWER) skip the reference's
projected re-solves of the min-x LP and are compared within FAST_ATOL (K, sd) and FAST_RTOL (sdd)."""
import contextlib
import functools
import os
import re
import shutil
import subprocess
from collections import namedtuple

import numpy as np
import pytest

from problems import degenerate_rows_batch, make_batch_fast

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "toppra_b200", "libtoppra_b200.so")

# K and sd of a fast build against the exact reference.  Measured on an H100: at most 2.2e-16 (K), 2.8e-17 (sd)
FAST_ATOL = 1e-15
FAST_RTOL = 1e-9       # sdd of a fast build, relative to max(1, max |sdd|)
FWD_THREADS_MIN = 16384
FUSED_WARPS_PER_SM = 28


# ---- kernel names -------------------------------------------------------------------------------------------------------
def kernel_key(name):
    """Demangled kernel name -> 'name<args>' without spaces, namespaces or parameter list.  Accepts the c++filt /
    kineto style ('1, 28, false') and the cu++filt style ('(int)1, (int)28, (bool)0')."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    s = s.replace("(anonymous namespace)::", "")
    s = re.sub(r"^(\w+::)+", "", s)
    s = s.replace("(bool)0", "false").replace("(bool)1", "true")
    s = re.sub(r"\((?:unsigned )?(?:int|long|short|char)\)", "", s)
    m = re.match(r"([A-Za-z_]\w*)(<[^<>]*>)?", s)
    return (m.group(1) + (m.group(2) or "")).replace(" ", "") if m else s


def build_key(name, args):
    if not args:
        return name
    return "%s<%s>" % (name, ",".join(("true" if a else "false") if isinstance(a, bool) else str(a) for a in args))


@contextlib.contextmanager
def launched():
    """Collects the keys of the kernels (and copies) the device ran inside the block (torch.profiler, CUDA
    activities).  Work queued before the block is finished first, so that none of it is counted."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    names = set()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield names
        torch.cuda.synchronize()
    names.update(kernel_key(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA)


# ---- a case's result ----------------------------------------------------------------------------------------------------
Check = namedtuple("Check", "label got want atol rtol")   # atol = rtol = None: bit for bit, NaN equal to NaN
Run = namedtuple("Run", "label kernels checks absent")    # one profiled launch sequence of a case


def exact(label, got, want):
    return Check(label, np.asarray(got), np.asarray(want), None, None)


def fast_checks(label, got, want, keys=("K", "sd", "sdd"), status=True):
    """A fast build: statuses equal, K / sd within FAST_ATOL, sdd within FAST_RTOL of the largest |sdd|."""
    out = [exact(label + " status", got["status"], want["status"])] if status else []
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        if k == "sdd":
            fin = np.abs(w[np.isfinite(w)])
            out.append(Check(label + " " + k, g, w, FAST_RTOL * max(1.0, fin.max() if fin.size else 0.0), 0.0))
        else:
            out.append(Check(label + " " + k, g, w, FAST_ATOL, 0.0))
    return out


def _h(t):
    return None if t is None else t.detach().cpu().numpy()


def _exact_square(v):
    """The next speed >= v whose square the reference's pow(v, 2) rounds like v * v (DESIGN.md section 2)."""
    v = float(v)
    while v ** 2 != v * v:
        v = float(np.nextafter(v, np.inf))
    return v


def _nthreads():
    return min(16, os.cpu_count() or 1)


@functools.lru_cache(maxsize=None)
def _ta():
    import toppra_b200
    return toppra_b200


def _eng():
    return _ta().engine


def _dev():
    return _eng().default_device()


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _t(x, dtype=None):
    return _eng().as_device(x, _dev(), dtype)


# ---- fused vel + acc problems (scan_velacc) -----------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def fused_problem(B, dof, interp, G=24, seed=0):
    """B random paths, 1/8 velocity-limited, one motionless joint on every 11th path (its rows have a = 0 exactly),
    mixed start speeds (zero, small, inadmissible 30, and, where the velocity bound does not set it, just above K[0]'s
    upper end, which makes the forward pass retry), mixed end speeds.  Returns device inputs, host copies and the
    oracle's solution on the GPU's spline."""
    import torch
    from oracle import oracle as orc
    eng = _eng()
    ss, way, vlim, alim = make_batch_fast(B, seed=1000 * dof + 7 * B % 1000 + seed, dof=dof)
    vlim[:B // 8] *= 0.03
    idx = np.arange(B)
    way[idx % 11 == 3, :, dof - 1] = way[idx % 11 == 3, :1, dof - 1]
    grid = np.linspace(0, 1, G)
    s1 = np.where(idx % 7 == 0, _exact_square(0.04), 0.0)
    d_ss, d_grid = _t(ss), _t(grid)
    ppoly = eng.spline_fit(d_ss, _t(way))
    d_vlim, d_alim = _t(vlim), _t(alim)
    xbound = eng.xbound_velocity(ppoly, d_ss, d_grid, d_vlim)
    K = _h(eng.scan_velacc(ppoly, d_ss, d_grid, d_alim, interp, xbound, None, _t(s1), backward_only=True)["K"])
    s0 = np.where(idx % 13 == 0, 30.0, np.where(idx % 5 == 0, _exact_square(0.05), 0.0))
    xb0 = _h(xbound)[:, 0, 1]
    retry = (idx % 9 == 4) & (idx >= B // 8) & np.isfinite(K[:, 0, 1]) & (K[:, 0, 1] < xb0 * (1 - 1e-9))
    for b in np.nonzero(retry)[0]:
        s0[b] = _exact_square(np.sqrt(K[b, 0, 1] + 5e-6))
    torch.cuda.synchronize()
    o = orc.solve_velacc_batch(_h(ppoly), np.tile(ss, (B, 1)), grid, vlim, alim, interp, sd_start=s0, sd_end=s1,
                               nthreads=_nthreads())
    ref = dict(K=o["K"], sd=o["sd"], sdd=o["u"], status=o["status"])
    bad = np.isnan(o["K"]).any(axis=(1, 2))
    back = dict(K=o["K"], status=np.where(bad, 3, 0).astype(np.int32))
    return dict(B=B, dof=dof, interp=interp, G=G, ss=ss, way=way, vlim=vlim, alim=alim, grid=grid, s0=s0, s1=s1,
                retry=retry, ppoly=ppoly, d_ss=d_ss, d_grid=d_grid, d_alim=d_alim, xbound=xbound, d_s0=_t(s0),
                d_s1=_t(s1), ref=ref, back=back)


def _velacc(p, **kw):
    eng = _eng()
    return eng.scan_velacc(p["ppoly"], p["d_ss"], p["d_grid"], p["d_alim"], p["interp"], p["xbound"], p["d_s0"],
                           p["d_s1"], **kw)


def _host(out):
    h = {k: _h(out[k]) for k in ("K", "sd", "u", "status", "fail_stage", "counters") if out.get(k) is not None}
    if "u" in h:
        h["sdd"] = h.pop("u")
    return h


def _solution_checks(label, got, want, fast):
    if fast:
        return fast_checks(label, got, want)
    return [exact(label + " " + k, got[k], want[k]) for k in ("status", "K", "sd", "sdd")]


def _backward_checks(label, got, want, fast):
    if fast:
        return fast_checks(label, got, want, keys=("K",))
    return [exact(label + " status", got["status"], want["status"]), exact(label + " K", got["K"], want["K"])]


def _fused_b(which):
    """'28': the largest batch of the 72-register build (28 CTAs per SM, one wave); '32': one path more."""
    B28 = FUSED_WARPS_PER_SM * _num_sms()
    return B28 if which == "28" else B28 + 1


def _other_minb(minb):
    return "32" if minb == "28" else "28"


def case_fused(minb, fast, mode):
    """scan_velacc at the fused register-budget edge: B = 28 SMs (MINB 28) or 28 SMs + 1 (MINB 32), 7-DOF."""
    p = fused_problem(_fused_b(minb), 7, True)
    ref, back, label = p["ref"], p["back"], "B=%d" % p["B"]
    absent = {"forward_threads_kernel<7>"} | {build_key("scan_kernel", (1, int(_other_minb(minb)), f, m, True, False))
                                              for f in (False, True) for m in (0, 1, 16, -1)}
    runs = []
    if mode == 0:
        with launched() as k:
            out = _host(_velacc(p, fast_lower=fast))
        runs.append(Run(label, k, _solution_checks(label, out, ref, fast), absent))
        if minb == "32" and not fast:
            # the forward-thread threshold: one path below it the warp kernel still runs the whole scan
            q = fused_problem(FWD_THREADS_MIN - 1, 7, True)
            with launched() as k2:
                out2 = _host(_velacc(q))
            runs.append(Run("B=%d" % q["B"], k2, _solution_checks("B=16383", out2, q["ref"], False),
                            {"forward_threads_kernel<7>"}))
    elif mode == 1:
        with launched() as k:
            out = _host(_velacc(p, fast_lower=fast, backward_only=True))
        runs.append(Run(label, k, _backward_checks(label, out, back, fast), absent))
    elif mode == 16:
        with launched() as k:
            b = _velacc(p, fast_lower=fast, backward_only=True)
            out = _host(_velacc(p, fast_lower=fast, forward_from=b))
        runs.append(Run(label, k, _solution_checks(label, out, ref, fast), absent))
    else:
        with launched() as k:
            out = _host(_velacc(p, fast_lower=fast, counters=True))
        checks = _solution_checks(label + " counters", out, ref, fast)
        checks.append(exact(label + " retries fired", bool((out["counters"][p["retry"], 3] > 0).all()), True))
        runs.append(Run(label + " counters", k, checks, absent))
        runs.append(_fused_ragged(p, fast, label, absent))
    return runs


@functools.lru_cache(maxsize=None)
def fused_ragged(B):
    """glen: path b keeps its first G - b % 5 gridpoints (its own uniform grid), the rest of the row is padding.
    Returns the device inputs and the oracle's solution path by path."""
    from oracle import oracle as orc
    p = fused_problem(B, 7, True)
    G = p["G"]
    glen = G - np.arange(B) % 5
    grids = np.ones((B, G))
    for b in range(B):
        grids[b, :glen[b]] = np.linspace(0, 1, glen[b])
    d_grid = _t(grids)
    xb = _eng().xbound_velocity(p["ppoly"], p["d_ss"], d_grid, _t(p["vlim"]))
    ref = dict(K=np.full((B, G, 2), np.nan), sd=np.full((B, G), np.nan), sdd=np.full((B, G - 1), np.nan),
               status=np.zeros(B, np.int32))
    pp = _h(p["ppoly"])
    for b in range(B):
        n = int(glen[b])
        o = orc.solve_velacc(pp[b], p["ss"], grids[b, :n], p["vlim"][b], p["alim"][b], p["interp"], p["s0"][b],
                             p["s1"][b])
        ref["K"][b, :n], ref["status"][b] = o["K"], o["status"]
        if o["status"] != 3:
            ref["sd"][b, :n], ref["sdd"][b, :n - 1] = o["sd"], o["u"]
    return dict(d_grid=d_grid, xbound=xb, glen=_t(glen.astype(np.int32), _int32()), ref=ref)


def _fused_ragged(p, fast, label, absent):
    r = fused_ragged(p["B"])
    with launched() as k:
        out = _host(_eng().scan_velacc(p["ppoly"], p["d_ss"], r["d_grid"], p["d_alim"], p["interp"], r["xbound"],
                                       p["d_s0"], p["d_s1"], fast_lower=fast, glen=r["glen"]))
    return Run(label + " ragged", k, _solution_checks(label + " ragged", out, r["ref"], fast), absent)


def _int32():
    import torch
    return torch.int32


def case_forward_threads(dof):
    """B = 16384 (the first batch of the thread-per-path forward pass): both discretisations the fused scan takes
    (dof 8 only with collocation: 4 * 8 + 2 rows do not fit one warp), the single launch and the split launch
    (backward only, then forward from it) of solve_to_host.  A counters launch of the same batch (the warp kernel)
    shows that the retry rule fires on the paths that start just above K[0]."""
    runs = []
    for interp in ((False,) if dof == 8 else (True, False)):
        p = fused_problem(FWD_THREADS_MIN, dof, interp)
        label = "dof=%d interp=%d" % (dof, interp)
        with launched() as k:
            out = _host(_velacc(p))
        runs.append(Run(label, k, _solution_checks(label, out, p["ref"], False), ()))
        with launched() as k:
            b = _velacc(p, backward_only=True)
            out = _host(_velacc(p, forward_from=b))
        runs.append(Run(label + " split", k, _solution_checks(label + " split", out, p["ref"], False), ()))
        cnt = _h(_velacc(p, counters=True)["counters"])
        assert p["retry"].sum() > 0 and (cnt[p["retry"], 3] > 0).all(), "the retry rule did not fire (%s)" % label
    return runs


# ---- raw stage records (engine.scan, feasible / reachable sets, robust scan) --------------------------------------------
RPL_R = {1: (29, 30), 2: (31, 62), 3: (63, 94), 4: (95, 125, 126)}   # R -> nC = R + 2 at both ends of each RPL range


@functools.lru_cache(maxsize=None)
def stage_records(R, ubound=False, B=48, G=16, seed=0):
    """Random stage records with R rows (scaled and near-duplicate row pairs, problems.degenerate_rows_batch).  Every
    fourth path has an infeasible stage (row 0 u + 1 x + 1 <= 0 with x >= 0), every fourth a stage with the flat row
    0 u - x + 0.01 <= 0, which lifts that stage's lowest x.  Start speeds 0 or 0.5.  Returns the device records and
    their host copy."""
    import torch
    rows, xb = degenerate_rows_batch((R + 1) // 2, G, B, 1000 + R + seed)
    rows = rows[..., :R].copy()
    for b in range(1, B, 4):
        rows[b, (5 * b) % (G - 1), :, b % R] = (0.0, 1.0, 1.0)
        rows[b + 1, (3 * b) % (G - 1), :, (b + 1) % R] = (0.0, -1.0, 0.01)
    rec, W = _eng().alloc_records(B, G, R, _dev(), ubound=ubound)
    host = np.zeros((B, G, W))
    host[:, :, 0:R], host[:, :, R:2 * R], host[:, :, 2 * R:3 * R] = rows[:, :, 0], rows[:, :, 1], rows[:, :, 2]
    host[:, :, 3 * R] = np.maximum(xb[:, :, 0], -1e8)
    host[:, :, 3 * R + 1] = np.minimum(xb[:, :, 1], 1e8)
    if ubound:
        rng = np.random.RandomState(R)
        host[:, :, 3 * R + 2] = -(0.2 + 2 * rng.rand(B, G))
        host[:, :, 3 * R + 3] = 0.2 + 2 * rng.rand(B, G)
    rec.copy_(torch.from_numpy(host))
    s0 = np.where(np.arange(B) % 3 == 1, 0.5, 0.0)
    return dict(R=R, B=B, G=G, rec=rec, host=torch.from_numpy(host), grid=np.linspace(0, 1, G), s0=s0)


@functools.lru_cache(maxsize=None)
def records_ref(R, ubound=False, backward_only=False):
    import torch
    import cpu_engine
    r = stage_records(R, ubound)
    out = cpu_engine.scan(r["host"], R, torch.from_numpy(r["grid"]), torch.from_numpy(r["s0"]), None,
                          backward_only=backward_only)
    return _host(out)


def _scan_records(r, **kw):
    eng = _eng()
    return _host(eng.scan(r["rec"], r["R"], _t(r["grid"]), _t(r["s0"]), None, **kw))


def _record_checks(label, got, want, fast, backward_only=False):
    checks = (_backward_checks if backward_only else _solution_checks)(label, got, want, fast)
    if not fast:
        checks.append(exact(label + " fail_stage", got["fail_stage"], want["fail_stage"]))
    return checks


def case_record_scan(rpl, fast, mode, ubound=False):
    """engine.scan over raw stage records at both ends of a rows-per-lane range.  mode 0: plain; 1: backward only;
    16: forward from an earlier backward-only result; -1: counters, and a ragged glen batch."""
    runs = []
    for R in RPL_R[rpl]:
        r = stage_records(R, ubound)
        label = "R=%d" % R
        if mode == 1:
            with launched() as k:
                out = _scan_records(r, fast_lower=fast, backward_only=True)
            runs.append(Run(label, k, _record_checks(label, out, records_ref(R, ubound, True), fast, True), ()))
            continue
        if mode == 16:
            with launched() as k:
                b = _eng().scan(r["rec"], R, _t(r["grid"]), _t(r["s0"]), None, fast_lower=fast, backward_only=True)
                out = _host(_eng().scan(r["rec"], R, _t(r["grid"]), _t(r["s0"]), None, fast_lower=fast, forward_from=b))
        else:
            with launched() as k:
                out = _scan_records(r, fast_lower=fast, counters=(mode == -1))
        absent = ()
        if rpl == 2 and not fast and not ubound:
            # two rows per lane, exact: the register-capped build, unless counters are asked for
            absent = {build_key("scan_kernel", (2, 24, False, -1, False, False) if mode == -1
                                else (2, 1, False, -1, False, False))}
        runs.append(Run(label, k, _record_checks(label, out, records_ref(R, ubound), fast), absent))
        if mode == -1 and rpl == 1:
            runs.append(_records_ragged(r, fast, label))
    return runs


def _records_ragged(r, fast, label):
    import torch
    import cpu_engine
    B, G, R = r["B"], r["G"], r["R"]
    glen = (G - np.arange(B) % 4).astype(np.int32)
    grids = np.ones((B, G))
    for b in range(B):
        grids[b, :glen[b]] = np.linspace(0, 1, glen[b])
    with launched() as k:
        out = _host(_eng().scan(r["rec"], R, _t(grids), _t(r["s0"]), None, fast_lower=fast,
                                glen=_t(glen, _int32())))
    want = _host(cpu_engine.scan(r["host"], R, torch.from_numpy(grids), torch.from_numpy(r["s0"]), None,
                                 glen=torch.from_numpy(glen)))
    return Run(label + " ragged", k, _solution_checks(label + " ragged", out, want, fast), ())


def case_feasible(rpl):
    import torch
    import cpu_engine
    runs = []
    for R in RPL_R[rpl]:
        for ub in (False, True):
            r = stage_records(R, ub)
            with launched() as k:
                X = _h(_eng().feasible_sets(r["rec"], R, _t(r["grid"])))
            want = _h(cpu_engine.feasible_sets(r["host"], R, torch.from_numpy(r["grid"])))
            runs.append(Run("R=%d ub=%d" % (R, ub), k, [exact("X", X, want)], ()))
    return runs


def case_reachable(rpl, ub):
    import torch
    import cpu_engine
    runs = []
    for R in RPL_R[rpl]:
        r = stage_records(R, ub)
        B = r["B"]
        smax = np.where(np.arange(B) % 2 == 0, 0.5, 0.0)
        with launched() as k:
            out = _eng().reachable_sets(r["rec"], R, _t(r["grid"]), None, _t(smax))
        out = {key: _h(v) for key, v in out.items()}
        want = cpu_engine.reachable_sets(r["host"], R, torch.from_numpy(r["grid"]), None, torch.from_numpy(smax))
        want = {key: _h(v) for key, v in want.items()}
        label = "R=%d" % R
        runs.append(Run(label, k, [exact(label + " " + key, out[key], want[key]) for key in ("X", "L", "fail_stage")],
                        ()))
    return runs


ELLIPSOID = (0.05, 0.02, 0.01)


def case_robust(rpl):
    """Robust scan with the conic rows [3, R - 2): a sub-range that starts past row 0 and stops before the last row."""
    import torch
    import cpu_engine
    runs = []
    for R in RPL_R[rpl]:
        r = stage_records(R)
        c0, cn = 3, R - 5
        for fs in (False, True):
            with launched() as k:
                out = _host(_eng().scan_robust(r["rec"], R, c0, cn, ELLIPSOID, _t(r["grid"]), _t(r["s0"]), None,
                                               feasible_sets=fs))
            want = _host(cpu_engine.scan_robust(r["host"], R, c0, cn, ELLIPSOID, torch.from_numpy(r["grid"]),
                                                torch.from_numpy(r["s0"]), None, feasible_sets=fs))
            label = "R=%d%s" % (R, " feasible sets" if fs else "")
            keys = ("status", "K") if fs else ("status", "K", "sd", "sdd")
            runs.append(Run(label, k, [exact(label + " " + key, out[key], want[key]) for key in keys], ()))
    return runs


# ---- stand-alone LPs ----------------------------------------------------------------------------------------------------
LP2D_N = {1: (1, 32), 2: (33, 64), 3: (65, 96), 4: (97, 128)}


def case_lp2d(rpl):
    import cpu_engine
    rng = np.random.RandomState(70 + rpl)
    runs = []
    for n in LP2D_N[rpl]:
        B = 64
        v = rng.randn(B, 3)
        a, b = rng.randn(2, B, n)
        c = np.where(rng.rand(B, 1) < 0.5, -rng.rand(B, n), rng.randn(B, n) * 0.3 - 0.6)
        low, high = np.tile([-1.0, -2.0], (B, 1)), np.tile([1.5, 0.7], (B, 1))
        act = rng.randint(-4, n + 2, size=(B, 2))
        with launched() as k:
            got = _eng().lp2d_batch(v, a, b, c, low, high, act)
        want = cpu_engine.lp2d_batch(v, a, b, c, low, high, act)
        ok = want[0] == 1
        label = "n=%d" % n
        checks = [exact(label + " result", got[0], want[0]), exact(label + " optval", got[1][ok], want[1][ok]),
                  exact(label + " optvar", got[2][ok], want[2][ok]), exact(label + " active", got[3][ok], want[3][ok])]
        if n > 1:
            checks.append(exact(label + " feasible and infeasible LPs", bool((~ok).any() and ok.any()), True))
        runs.append(Run(label, k, checks, ()))
    return runs


def case_lp1d():
    import cpu_engine
    rng = np.random.RandomState(71)
    runs = []
    for n in (0, 1, 31, 32, 33, 100):
        B = 64
        v = rng.randn(B, 2)
        a, b = rng.randn(B, n), rng.randn(B, n) - 2.5
        a[:, ::7] *= 1e-11          # rows below the 1e-10 threshold are ignored
        low, high = -1 - rng.rand(B), 1 + rng.rand(B)
        low[::5] = 2.0 + rng.rand(B)[::5]   # an empty box
        with launched() as k:
            got = _eng().lp1d_batch(v, a, b, low, high)
        want = cpu_engine.lp1d_batch(v, a, b, low, high)
        ok = want[0] == 1
        label = "n=%d" % n
        checks = [exact(label + " result", got[0], want[0])]
        checks += [exact(label + " " + w, g[ok], h[ok]) for w, g, h in zip(("optval", "optvar", "active"), got[1:], want[1:])]
        if n > 1:
            checks.append(exact(label + " feasible and infeasible LPs", bool((~ok).any() and ok.any()), True))
        runs.append(Run(label, k, checks, ()))
    return runs


# ---- spline, rows, bounds, parametrisation ------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def small_paths(B=16, dof=6, G=40, seed=3):
    ss, way, vlim, alim = make_batch_fast(B, seed=seed, dof=dof)
    way[5, :, 2] = way[5, 0, 2]        # a motionless joint
    return dict(B=B, dof=dof, G=G, ss=ss, way=way, vlim=vlim, alim=alim, grid=np.linspace(0, 1, G))


def _spline(p):
    return _eng().spline_fit(_t(p["ss"]), _t(p["way"]))


def _cpu(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x))


def case_spline_fit():
    import cpu_engine
    p = small_paths()
    with launched() as k:
        c = _h(_spline(p))
    want = _h(cpu_engine.spline_fit(_cpu(p["ss"]), _cpu(p["way"])))
    return [Run("", k, [exact("ppoly", c, want)], ())]


def case_ppoly_eval():
    import cpu_engine
    p = small_paths()
    pp = _spline(p)
    s = np.linspace(-0.1, 1.1, 57)
    runs = []
    for order in (0, 1, 2):
        with launched() as k:
            got = _h(_eng().ppoly_eval(pp, _t(p["ss"]), _t(s), order))
        want = _h(cpu_engine.ppoly_eval(_cpu(_h(pp)), _cpu(p["ss"]), _cpu(s), order))
        runs.append(Run("order %d" % order, k, [exact("order %d" % order, got, want)], ()))
    return runs


def _records_pair(p, R):
    import torch
    rec, W = _eng().alloc_records(p["B"], p["G"], R, _dev())
    _eng().init_bounds(rec, R)
    torch.cuda.synchronize()
    return rec, torch.full((p["B"], p["G"], W), 7.0, dtype=torch.float64)


def case_coeff_velacc():
    import cpu_engine
    p = small_paths()
    pp = _spline(p)
    R = 4 * p["dof"]
    rec, host = _records_pair(p, R)
    cpu_engine.init_bounds(host, R)
    with launched() as k:
        _eng().coeff_velacc(pp, _t(p["ss"]), _t(p["grid"]), _t(p["vlim"]), _t(p["alim"]), True, rec, R)
    cpu_engine.coeff_velacc(_cpu(_h(pp)), _cpu(p["ss"]), _cpu(p["grid"]), _cpu(p["vlim"]), _cpu(p["alim"]), True,
                            host, R)
    return [Run("", k, [exact("records", _h(rec), _h(host))], ())]


def case_init_bounds():
    import cpu_engine
    p = small_paths()
    runs = []
    for ub in (False, True):
        rec, W = _eng().alloc_records(p["B"], p["G"], 5, _dev(), ubound=ub)
        rec.fill_(7.0)
        host = _cpu(_h(rec))
        with launched() as k:
            _eng().init_bounds(rec, 5)
        cpu_engine.init_bounds(host, 5)
        runs.append(Run("ub=%d" % ub, k, [exact("records", _h(rec)[..., 15:], _h(host)[..., 15:])], ()))
    return runs


def case_rows_canlinear():
    import cpu_engine
    rng = np.random.RandomState(5)
    B, G, m, kk = 6, 37, 3, 5
    a, b, c = rng.randn(3, B, G, m)
    F, g = rng.randn(kk, m), rng.rand(kk)
    grid = np.r_[0.0, np.sort(rng.rand(G - 2)), 1.0]
    R = 2 * kk + 1
    p = dict(B=B, G=G)
    runs = []
    for interp in (False, True):
        rec, host = _records_pair(p, R)
        host.copy_(_cpu(_h(rec)))
        with launched() as k:
            _eng().rows_canlinear(_t(a), _t(b), _t(c), _t(F), _t(g), 0, _t(grid), interp, rec, R, 1)
        cpu_engine.rows_canlinear(_cpu(a), _cpu(b), _cpu(c), _cpu(F), _cpu(g), 0, _cpu(grid), interp, host, R, 1)
        runs.append(Run("interp=%d" % interp, k, [exact("records", _h(rec), _h(host))], ()))
    return runs


def case_xbound_varying():
    import cpu_engine
    p = small_paths()
    pp = _spline(p)
    vg = p["vlim"][0][None] * (0.05 + 0.5 * p["grid"])[:, None, None]
    rec, host = _records_pair(p, 0)
    host.copy_(_cpu(_h(rec)))
    with launched() as k:
        _eng().xbound_varying(pp, _t(p["ss"]), _t(p["grid"]), _t(vg), rec, 0, 1)
    cpu_engine.xbound_varying(_cpu(_h(pp)), _cpu(p["ss"]), _cpu(p["grid"]), _cpu(vg), host, 0, 1)
    return [Run("", k, [exact("xbound", _h(rec), _h(host))], ())]


def case_propose_gridpoints():
    import cpu_engine
    p = small_paths()
    pp = _spline(p)
    with launched() as k:
        got = [_h(x) for x in _eng().propose_gridpoints(pp, _t(p["ss"]), 1e-3, 100, 0.05, 20, 512)]
    want = [_h(x) for x in cpu_engine.propose_gridpoints(_cpu(_h(pp)), _cpu(p["ss"]), 1e-3, 100, 0.05, 20, 512)]
    return [Run("", k, [exact(w, g, h) for w, g, h in zip(("grid", "glen", "status"), got, want)], ())]


@functools.lru_cache(maxsize=None)
def _sd_passes():
    """Fastest and slowest TOPPRAsd passes (x = sd^2) of small_paths(), computed by the double on host records."""
    import cpu_engine
    p = small_paths()
    R = 4 * p["dof"]
    host = _cpu(np.zeros((p["B"], p["G"], _eng().record_doubles(R))))
    cpu_engine.init_bounds(host, R)
    pp = _cpu(_h(_spline(p)))
    cpu_engine.coeff_velacc(pp, _cpu(p["ss"]), _cpu(p["grid"]), _cpu(p["vlim"]), _cpu(p["alim"]), True, host, R)
    f = cpu_engine.scan(host, R, _cpu(p["grid"]), None, None, sd_forward="fast")
    s = cpu_engine.scan(host, R, _cpu(p["grid"]), None, None, sd_forward="slow")
    return {k: _h(v) for k, v in (("xf", f["sd"]), ("uf", f["u"]), ("xs", s["sd"]), ("us", s["u"]))}


def case_sd_bisect():
    import cpu_engine
    p = small_paths()
    s = _sd_passes()
    B = p["B"]
    want_d = np.linspace(0.5, 6.0, B)
    args = [s["xf"], s["uf"], s["xs"], s["us"], p["grid"], want_d]
    with launched() as k:
        got = _host_dict(_eng().sd_bisect(*[_t(x) for x in args], atol=1e-5))
    want = _host_dict(cpu_engine.sd_bisect(*[_cpu(x) for x in args], atol=1e-5))
    return [Run("", k, [exact(key, got[key], want[key]) for key in ("sd", "u", "info", "status")], ())]


def _host_dict(d):
    return {k: _h(v) for k, v in d.items()}


def _param_input():
    p = small_paths()
    x = np.maximum(_sd_passes()["xf"], 0.0)
    sd = np.sqrt(x)
    sd[:, 1:-1] = np.maximum(sd[:, 1:-1], 1e-3)
    sd[3, 7] = 0.0                     # a stop inside the path: its knot is dropped
    return p, sd


def case_spline_time_stamps():
    import cpu_engine
    p, sd = _param_input()
    B, G = sd.shape
    grid = np.tile(p["grid"], (B, 1))
    glen = (G - np.arange(B) % 3).astype(np.int32)
    with launched() as k:
        got = [_h(x) for x in _eng().spline_time_stamps(_t(sd), _t(grid), _t(glen, _int32()))]
    want = [_h(x) for x in cpu_engine.spline_time_stamps(_cpu(sd), _cpu(grid), _cpu(glen))]
    return [Run("", k, [exact(w, g, h) for w, g, h in zip(("t", "s", "nkeep"), got, want)], ())]


def case_time_grid():
    import cpu_engine
    p, sd = _param_input()
    sd = np.maximum(sd, 1e-3)
    with launched() as k:
        got = [_h(x) for x in _eng().time_grid(_t(sd), _t(p["grid"]))]
    want = [_h(x) for x in cpu_engine.time_grid(_cpu(sd), _cpu(p["grid"]))]
    return [Run("", k, [exact(w, g, h) for w, g, h in zip(("t", "us"), got, want)], ())]


def case_constaccel_eval():
    """Same tolerances as the const-accel parametrizer test of tests/test_gpu_parity.py."""
    import cpu_engine
    p, sd = _param_input()
    sd = np.maximum(sd, 1e-3)
    pp = _spline(p)
    t, us = _eng().time_grid(_t(sd), _t(p["grid"]))
    ts = np.stack([np.linspace(0, float(d), 31) for d in _h(t)[:, -1]])
    runs = []
    for order, (rtol, atol) in enumerate(((1e-12, 1e-13), (1e-11, 1e-12), (1e-10, 1e-10))):
        with launched() as k:
            got = _h(_eng().constaccel_eval(pp, _t(p["ss"]), _t(p["grid"]), _t(sd), t, us, _t(ts), order))
        want = _h(cpu_engine.constaccel_eval(_cpu(_h(pp)), _cpu(p["ss"]), _cpu(p["grid"]), _cpu(sd), _cpu(_h(t)),
                                             _cpu(_h(us)), _cpu(ts), order))
        runs.append(Run("order %d" % order, k, [Check("order %d" % order, got, want, atol, rtol)], ()))
    return runs


# ---- joint-torque rows of a device model ----------------------------------------------------------------------------------
SO_MODELS = {0: ("coupled_cosine", [2.0, 0.3, 0.1, 4.9]), 1: ("pendulums", None)}
# CUDA's fp64 sin and cos are within 2 ulp (CUDA C Programming Guide, mathematical functions), numpy's within 1
TRIG_ULPS = 3


def case_second_order(model):
    """tb_coeff_second_order's records against the double (cpu_engine.coeff_second_order).  Rows without a sin or cos
    term match bit for bit; the others within TRIG_ULPS of their sin / cos terms' magnitude, plus rounding of the sums
    around them.  For the pendulums, the scan of the GPU's own records then matches the double's scan bit for bit."""
    import cpu_engine
    from oracle import oracle as orc
    p = small_paths(B=12, dof=6, G=45, seed=8)
    name, prm = SO_MODELS[model]
    dof, B, G = p["dof"], p["B"], p["G"]
    rng = np.random.RandomState(model)
    if prm is None:
        prm = list((np.stack((1 + rng.rand(dof), 5 + 3 * rng.rand(dof)), 1)).reshape(-1))
    taulim = np.stack((-(40 + 10 * rng.rand(dof)), 40 + 10 * rng.rand(dof)), 1)
    fric = 0.5 * rng.rand(dof)
    pp = _spline(p)
    eps = np.finfo(float).eps
    qd, qdd = (np.stack([orc.ppoly_eval(_h(pp)[b], p["ss"], p["grid"], o) for b in range(B)]) for o in (1, 2))
    runs = []
    for interp in (True, False):
        R = (4 if interp else 2) * dof
        rec, host = _records_pair(p, R)
        cpu_engine.init_bounds(host, R)
        with launched() as k:
            _eng().coeff_second_order(name, prm, pp, _t(p["ss"]), _t(p["grid"]), _t(taulim), _t(fric), interp, rec, R, 0)
            got = _h(rec)
            if name == "pendulums":   # then the scan of the GPU's own records
                out = _host(_eng().scan(rec, R, _t(p["grid"]), _t(np.zeros(B)), None))
        cpu_engine.coeff_second_order(name, prm, _cpu(_h(pp)), _cpu(p["ss"]), _cpu(p["grid"]), _cpu(taulim),
                                      _cpu(fric), interp, host, R, 0)
        want = _h(host)
        label = "interp=%d" % interp
        ga, gb, gc = (got[..., j * R:(j + 1) * R] for j in range(3))
        wa, wb, wc = (want[..., j * R:(j + 1) * R] for j in range(3))
        checks = [exact(label + " xbound", got[..., 3 * R:], want[..., 3 * R:])]
        if name == "pendulums":
            sin_scale = np.abs(np.asarray(prm)[1::2]) * np.ones((B, G, dof))       # c = p_k sin q_k + ...
            checks += [exact(label + " a", ga, wa), exact(label + " b", gb, wb)]
        else:
            m0, m1, h, g0 = prm
            sin_scale = abs(g0) * np.ones((B, G, dof))
            # a = m0 q' + m1 (cos q_k sum_j cos q_j q'_j + sin q_k sum_j sin q_j q'_j): each of the two products is
            # off by at most 2 trig errors times sum_j |q'_j|; b likewise with q'', plus h sin q_k |q'|^2
            ta = 2 * TRIG_ULPS * eps * 2 * abs(m1) * np.abs(qd).sum(-1, keepdims=True) * np.ones((1, 1, dof))
            tb = TRIG_ULPS * eps * (4 * abs(m1) * np.abs(qdd).sum(-1, keepdims=True)
                                    + abs(h) * (qd * qd).sum(-1, keepdims=True)) * np.ones((1, 1, dof))
            two_delta = np.r_[2 * np.diff(p["grid"]), 0.0][None, :, None]
            ta_lift = ta.copy()
            ta_lift[:, :-1] = ta[:, 1:] + two_delta[:, :-1] * tb[:, 1:]
            checks += [Check(label + " a", ga, wa, _rows_tol(ta, R, dof, ta_lift) + 2 * np.spacing(np.abs(wa)), 0.0),
                       Check(label + " b", gb, wb, _rows_tol(tb, R, dof) + 2 * np.spacing(np.abs(wb)), 0.0)]
        unit = _rows_tol(eps * sin_scale, R, dof)
        checks.append(Check(label + " c", gc, wc, TRIG_ULPS * unit + 2 * np.spacing(np.abs(wc)), 0.0))
        _report("second-order rows %s %s: max |c - c_ref| = %.3g eps * |sin coefficient|; a, b equal: %s %s" % (
            name, label, np.max(np.abs(gc - wc) / unit), np.array_equal(ga, wa), np.array_equal(gb, wb)))
        if name == "pendulums":
            ref = _host(cpu_engine.scan(_cpu(got), R, _cpu(p["grid"]), _cpu(np.zeros(B)), None))
            checks += _record_checks(label + " scan", out, ref, False)
            checks.append(exact("some paths solved", bool((out["status"] == 0).any()), True))
        runs.append(Run(label, k, checks, ()))
    return runs


def _rows_tol(per_joint, nr, dof, lifted=None):
    """[B, G, dof] bound -> [B, G, nr] in the record's row order (blocks of dof rows: +, -, lifted +, lifted -)."""
    t = np.concatenate([per_joint] * (nr // dof), axis=-1)
    if lifted is not None and nr == 4 * dof:
        t[..., 2 * dof:] = np.concatenate([lifted] * 2, axis=-1)
    return t


def _report(line):
    print(line)


# ---- the table ----------------------------------------------------------------------------------------------------------------
def _builds():
    rows = []
    for minb in ("28", "32"):
        for fast in (False, True):
            for mode in (0, 1, 16, -1):
                rows.append(("scan_kernel", (1, int(minb), fast, mode, True, False), case_fused, (minb, fast, mode)))
    for fast in (False, True):
        for mode in (0, 1, 16, -1):
            rows.append(("scan_kernel", (1, 32, fast, mode, False, False), case_record_scan, (1, fast, mode)))
    rows.append(("scan_kernel", (1, 1, False, -1, False, True), case_record_scan, (1, False, 0, True)))
    for rpl in (2, 3, 4):
        rows.append(("scan_kernel", (rpl, 1, False, -1, False, False), case_record_scan, (rpl, False, -1 if rpl == 2 else 0)))
        rows.append(("scan_kernel", (rpl, 1, True, -1, False, False), case_record_scan, (rpl, True, 0)))
        rows.append(("scan_kernel", (rpl, 1, False, -1, False, True), case_record_scan, (rpl, False, 0, True)))
    rows.append(("scan_kernel", (2, 24, False, -1, False, False), case_record_scan, (2, False, 0)))
    for d in range(1, 9):
        rows.append(("forward_threads_kernel", (d,), case_forward_threads, (d,)))
    for rpl in (1, 2, 3, 4):
        rows.append(("feasible_kernel", (rpl,), case_feasible, (rpl,)))
        rows.append(("reachable_kernel", (rpl, False), case_reachable, (rpl, False)))
        rows.append(("reachable_kernel", (rpl, True), case_reachable, (rpl, True)))
        rows.append(("scan_robust_kernel", (rpl,), case_robust, (rpl,)))
        rows.append(("lp2d_batch_kernel", (rpl,), case_lp2d, (rpl,)))
    for model in (0, 1):
        rows.append(("second_order_rows_tiled_kernel", (model,), case_second_order, (model,)))
    for name, case in (("spline_fit_kernel", case_spline_fit), ("ppoly_eval_kernel", case_ppoly_eval),
                       ("coeff_velacc_kernel", case_coeff_velacc), ("rows_canlinear_kernel", case_rows_canlinear),
                       ("xbound_varying_kernel", case_xbound_varying), ("init_bounds_kernel", case_init_bounds),
                       ("propose_gridpoints_kernel", case_propose_gridpoints), ("sd_bisect_kernel", case_sd_bisect),
                       ("spline_time_stamps_kernel", case_spline_time_stamps), ("time_grid_kernel", case_time_grid),
                       ("constaccel_eval_kernel", case_constaccel_eval), ("lp1d_batch_kernel", case_lp1d)):
        rows.append((name, (), case, ()))
    return rows


BUILDS = _builds()


def _compare(c):
    if c.atol is None:
        assert np.array_equal(c.got, c.want, equal_nan=True), "%s differs: max |diff| %s" % (c.label, _maxdiff(c))
        return
    assert c.got.shape == c.want.shape, c.label
    nan_g, nan_w = np.isnan(c.got), np.isnan(c.want)
    assert np.array_equal(nan_g, nan_w), "%s: NaN at different places" % c.label
    err = np.abs(np.where(nan_g, 0.0, c.got - c.want))
    tol = c.atol + c.rtol * np.abs(np.where(nan_w, 0.0, c.want))
    assert (err <= tol).all(), "%s: max |diff| %.3g, max |diff| / tolerance %.3g" % (c.label, err.max(), (err / tol).max())


def _maxdiff(c):
    try:
        d = np.abs(np.asarray(c.got, float) - np.asarray(c.want, float))
        return np.nanmax(d) if d.size else 0.0
    except (TypeError, ValueError):
        return "n/a"


@pytest.mark.gpu
@pytest.mark.parametrize("name,args,case,case_args", BUILDS, ids=[build_key(r[0], r[1]) for r in BUILDS])
def test_build_runs_and_matches_reference(name, args, case, case_args):
    key = build_key(name, args)
    for _ in range(3):
        # kineto (torch 2.11, H100) now and then returns a capture without any device activity, not even the copies
        # of the results; the cases are deterministic, so such a case is simply run again
        runs = case(*case_args)
        if all(run.kernels for run in runs):
            break
    assert runs
    for run in runs:
        assert key in run.kernels, "%s [%s]: %s was not launched; launched: %s" % (key, run.label, key, sorted(run.kernels))
        for other in run.absent:
            assert other not in run.kernels, "%s [%s]: %s was launched too" % (key, run.label, other)
        for c in run.checks:
            _compare(c)
        dev = [float(np.nanmax(np.abs(c.got - c.want))) for c in run.checks
               if c.atol is not None and c.got.size and np.isfinite(c.got).any()]
        if len(args) > 2 and args[2] is True and name == "scan_kernel":
            print("fast-deviation %s [%s]: %s" % (key, run.label, " ".join("%.3g" % d for d in dev)))


# ---- the inventory ------------------------------------------------------------------------------------------------------------
def _cuda_tool(name):
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", name)):
            return os.path.join(d, "bin", name)
    return shutil.which(name)


def library_kernels(so=LIB):
    """Kernel keys of the built library: cuobjdump -res-usage lists one 'Function <mangled>:' per kernel."""
    text = subprocess.run([_cuda_tool("cuobjdump"), "-res-usage", so], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", text, re.M)
    names = subprocess.run([shutil.which("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    return [kernel_key(n) for n in names]


def test_kernel_key_accepts_both_demangler_styles():
    assert kernel_key("void tb::(anonymous namespace)::scan_kernel<1, 28, false, -1, true, false>(double const*, int)") \
        == "scan_kernel<1,28,false,-1,true,false>"
    assert kernel_key("void tb::<unnamed>::scan_kernel<(int)1, (int)28, (bool)0, (int)-1, (bool)1, (bool)0>"
                      "(const double *, int)".replace("<unnamed>::", "")) == "scan_kernel<1,28,false,-1,true,false>"
    assert kernel_key("tb::(anonymous namespace)::lp1d_batch_kernel(double const*, int)") == "lp1d_batch_kernel"
    assert build_key("reachable_kernel", (4, True)) == "reachable_kernel<4,true>"


def test_builds_table_lists_every_kernel_of_the_library():
    """Adding or removing a template instantiation without a row in BUILDS fails here, without a GPU."""
    if not os.path.exists(LIB):
        pytest.skip("libtoppra_b200.so is not built")
    if not _cuda_tool("cuobjdump") or not shutil.which("c++filt"):
        pytest.skip("cuobjdump / c++filt not found")
    lib = library_kernels()
    table = [build_key(r[0], r[1]) for r in BUILDS]
    assert len(set(table)) == len(table), "duplicate rows in BUILDS"
    assert len(set(lib)) == len(lib)
    assert set(lib) == set(table), "kernels without a row: %s; rows without a kernel: %s" % (
        sorted(set(lib) - set(table)), sorted(set(table) - set(lib)))
    print("%d kernel builds in %s, one row each" % (len(lib), os.path.basename(LIB)))
