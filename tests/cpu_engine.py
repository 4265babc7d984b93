"""TEST DOUBLE (tests/ only, never imported by the product): a CPU stand-in of `toppra_b200.engine` built on the oracle.

`install(monkeypatch)` replaces the tensor-level kernel wrappers of toppra_b200/engine.py by functions that do the same
job on CPU torch tensors through the plain-C restatement (oracle/), and lets `_lib.require_cuda()` pass.  With it the
whole Python host side — SplineInterpolator, constraints, record assembly, solver wrapper, TOPPRA, BatchTOPPRA chunking,
parametrizers, error paths — runs under `-m "not gpu"` (tests/test_host_pipeline_cpu.py replays the GPU parity tests
through it).  It checks HOST LOGIC only: the numbers are the oracle's, the CUDA kernels are checked by the `-m gpu`
tests.  The product has no CPU path; this module lives outside the package on purpose."""
import ctypes

import numpy as np
import torch

from oracle import oracle as orc

VAR_MIN, VAR_MAX = -1e8, 1e8


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _per_path(arr, b):
    """arr is shared ([n]) or per path ([B, n])."""
    return arr if arr.ndim == 1 else arr[b]


# ---- K0 ---------------------------------------------------------------------------------------------------------------
def spline_fit(ss, wp, bc=((0, None), (0, None))):
    ssn, wpn = _np(ss), _np(wp)
    B, n, dof = wpn.shape
    (k0, v0), (k1, v1) = bc
    out = np.empty((B, 4, n - 1, dof))
    for b in range(B):
        vb0 = np.zeros(dof) if v0 is None else _np(v0)[b]
        vb1 = np.zeros(dof) if v1 is None else _np(v1)[b]
        out[b] = orc.cubic_spline_fit(_per_path(ssn, b), wpn[b], ((k0, vb0), (k1, vb1)))
    return torch.from_numpy(out)


def ppoly_eval(ppoly, breaks, s, order):
    pp, br, sn = _np(ppoly), _np(breaks), _np(s)
    B = pp.shape[0]
    return torch.from_numpy(np.stack([orc.ppoly_eval(pp[b], _per_path(br, b), _per_path(sn, b), order) for b in range(B)]))


# ---- records ------------------------------------------------------------------------------------------------------------
def record_doubles(R):
    return (3 * int(R) + 2 + 1) & ~1


def alloc_records(B, G, R, device, ubound=False):
    W = ((3 * int(R) + 4 + 1) & ~1) if ubound else record_doubles(R)
    return torch.full((B, G, W), float("nan"), dtype=torch.float64), W


def has_ubound(records, R):
    return records.shape[-1] >= 3 * int(R) + 4


def init_bounds(records, R):
    records[:, :, 3 * R] = VAR_MIN
    records[:, :, 3 * R + 1] = VAR_MAX
    records[:, :, 3 * R + 2:] = 0.0
    if has_ubound(records, R):
        records[:, :, 3 * R + 2] = VAR_MIN
        records[:, :, 3 * R + 3] = VAR_MAX


def _write_xbound(rec, R_total, xb, mode):
    lo, hi = rec[:, :, 3 * R_total], rec[:, :, 3 * R_total + 1]
    xb = torch.from_numpy(np.ascontiguousarray(xb))
    if mode == 1:
        lo.copy_(torch.clamp(xb[..., 0], min=VAR_MIN))
        hi.copy_(torch.clamp(xb[..., 1], max=VAR_MAX))
    elif mode == 2:
        lo.copy_(xb[..., 0])
        hi.copy_(xb[..., 1])
    elif mode == 3:
        lo.copy_(torch.maximum(lo, xb[..., 0]))
        hi.copy_(torch.minimum(hi, xb[..., 1]))


def coeff_velacc(ppoly, breaks, grid, vlim, alim, interp, records, R_total, row0=0, write_xbound=1):
    pp, br, gr = _np(ppoly), _np(breaks), _np(grid)
    vl, al = _np(vlim), _np(alim)
    B, _, nseg, dof = pp.shape
    G = gr.shape[-1]
    rec = records
    xb = np.empty((B, G, 2))
    L = orc.lib()
    for b in range(B):
        g = np.ascontiguousarray(_per_path(gr, b))
        qs = orc.ppoly_eval(pp[b], _per_path(br, b), g, 1)
        qss = orc.ppoly_eval(pp[b], _per_path(br, b), g, 2)
        if vl is None:
            xb[b, :, 0], xb[b, :, 1] = VAR_MIN, VAR_MAX
        else:
            xb[b] = orc.velocity_xbound(qs, vl if vl.ndim == 2 else vl[b])
        if al is not None:
            R = (4 if interp else 2) * dof
            a, bb, c = (np.zeros((G, R)) for _ in range(3))
            alb = np.ascontiguousarray(al if al.ndim == 2 else al[b])
            dp = ctypes.POINTER(ctypes.c_double)
            L.orc_accel_rows(np.ascontiguousarray(qs).ctypes.data_as(dp), np.ascontiguousarray(qss).ctypes.data_as(dp),
                             alb.ctypes.data_as(dp), g.ctypes.data_as(dp), G, dof, 1 if interp else 0, R, 0,
                             a.ctypes.data_as(dp), bb.ctypes.data_as(dp), c.ctypes.data_as(dp))
            rec[b, :, row0:row0 + R] = torch.from_numpy(a)
            rec[b, :, R_total + row0:R_total + row0 + R] = torch.from_numpy(bb)
            rec[b, :, 2 * R_total + row0:2 * R_total + row0 + R] = torch.from_numpy(c)
    if write_xbound:
        _write_xbound(rec, R_total, xb, write_xbound)
        rec[:, :, 3 * R_total + (4 if has_ubound(rec, R_total) else 2):] = 0.0   # padding; a u-bound pair is kept


def rows_canlinear(a, b, c, F, g, F_mode, grid, interp, records, R_total, row0):
    """Port of rows_canlinear_kernel (csrc/tb_coeff.cu): same term order (sum over q = 0..m-1, left to right)."""
    an, bn, cn, Fn, gn, gr = _np(a), _np(b), _np(c), _np(F), _np(g), _np(grid)
    B, G, m = an.shape
    k = Fn.shape[0] if F_mode == 0 else (Fn.shape[2] if F_mode == 1 else 2 * m)
    nrows = 2 * k if interp else k
    N = G - 1
    out = np.zeros((B, G, 3, nrows))
    for p in range(B):
        gp = _per_path(gr, p)
        for gi in range(G):
            for r in range(nrows):
                second = r >= k
                j = r - k if second else r
                src = gi + 1 if (second and gi < N) else gi
                lift = second and gi < N
                two_delta = 2 * (gp[gi + 1] - gp[gi]) if lift else 0.0
                av = an[p, src] + two_delta * bn[p, src] if lift else an[p, src]
                if F_mode >= 2:
                    col, sgn = (j, 1.0) if j < m else (j - m, -1.0)
                    ta, tb, tc = sgn * av[col], sgn * bn[p, src, col], sgn * cn[p, src, col]
                    gv = gn[p, j] if F_mode == 3 else gn[j]
                else:
                    Fr = Fn[j] if F_mode == 0 else Fn[p, src, j]
                    ta = tb = tc = 0.0
                    for q in range(m):
                        ta = ta + Fr[q] * av[q]
                        tb = tb + Fr[q] * bn[p, src, q]
                        tc = tc + Fr[q] * cn[p, src, q]
                    gv = gn[j] if F_mode == 0 else gn[p, src, j]
                out[p, gi, :, r] = (ta, tb, tc - gv)
    t = torch.from_numpy(out)
    records[:, :, row0:row0 + nrows] = t[:, :, 0]
    records[:, :, R_total + row0:R_total + row0 + nrows] = t[:, :, 1]
    records[:, :, 2 * R_total + row0:2 * R_total + row0 + nrows] = t[:, :, 2]
    return nrows


def xbound_varying(ppoly, breaks, grid, vlim_grid, records, R_total, write_xbound):
    """_create_velocity_constraint_varying (_CythonUtils.pyx:61-101): the constant-limit formula with vlim_grid[i]."""
    pp, br, gr, vg = _np(ppoly), _np(breaks), _np(grid), _np(vlim_grid)
    B, G = pp.shape[0], gr.shape[-1]
    xb = np.empty((B, G, 2))
    for b in range(B):
        qs = orc.ppoly_eval(pp[b], _per_path(br, b), _per_path(gr, b), 1)
        lim = vg if vg.ndim == 3 else vg[b]
        for i in range(G):
            xb[b, i] = orc.velocity_xbound(qs[i:i + 1], lim[i])[0]
    _write_xbound(records, R_total, xb, write_xbound)


# ---- K2 -----------------------------------------------------------------------------------------------------------------
def _rows_of(records, R, b):
    rec = _np(records[b])
    rows = np.stack((rec[:, 0:R], rec[:, R:2 * R], rec[:, 2 * R:3 * R]), axis=1)
    return rows, rec[:, 3 * R:3 * R + 2]


def _wrapper(records, R, b, grid, n=None):
    """The oracle's stateful seidelWrapper restatement over path b's records (first n gridpoints of a ragged batch)."""
    rows, xb = _rows_of(records, R, b)
    ub = _np(records[b])[:, 3 * R + 2:3 * R + 4] if has_ubound(records, R) else None
    if n is not None:
        rows, xb, grid = rows[:n], xb[:n], grid[:n]
        ub = None if ub is None else ub[:n]
    return orc.Wrapper(np.ascontiguousarray(grid), np.ascontiguousarray(rows), np.ascontiguousarray(xb),
                       None if ub is None else np.ascontiguousarray(ub))


def _scalar(t, b, default=0.0):
    return default if t is None else float(_np(t).reshape(-1)[b])


def check_glen(glen, B, grid):
    if glen is not None and (tuple(glen.shape) != (B,) or grid.dim() != 2):
        raise ValueError("glen must have shape (B,) and the grid (B, G)")


def scan(records, R, grid, sd_start=None, sd_end=None, sd_end_hi=None, backward_only=False, counters=False,
         sd_forward=None, forward_from=None, fast_lower=False, glen=None):
    B, G, W = records.shape
    if sd_forward is not None:
        return _scan_sd(records, R, grid, sd_start, sd_end, sd_forward == "slow")
    if glen is not None:
        return _scan_ragged(records, R, grid, sd_start, sd_end, _np(glen))
    gr = _np(grid)
    K = np.zeros((B, G, 2))
    sd = np.full((B, G), np.nan)
    u = np.full((B, max(G - 1, 0)), np.nan)
    status = np.zeros(B, dtype=np.int32)
    fail = np.full(B, -1, dtype=np.int32)
    cnt = np.zeros((B, 4), dtype=np.int32)
    for b in range(B):
        w = _wrapper(records, R, b, _per_path(gr, b))
        s0, s1 = _scalar(sd_start, b), _scalar(sd_end, b)
        if backward_only:
            K[b] = w.compute_controllable_sets(s1, _scalar(sd_end_hi, b, s1))
            bad = np.isnan(K[b]).any(axis=1)
            if bad.any():
                status[b], fail[b] = 3, int(np.nonzero(bad)[0].max())
            continue
        o = w.compute_parameterization(s0, s1)
        K[b], status[b] = o["K"], o["status"]
        if o["status"] == 3:
            bad = np.isnan(K[b]).any(axis=1)
            fail[b] = int(np.nonzero(bad)[0].max()) if bad.any() else 0
        else:
            sd[b], u[b] = o["sd"], o["u"]
            if o["status"] != 0:
                fail[b] = int(np.nonzero(np.isnan(o["sd"]))[0].min()) - 1
        c = w.counters() if hasattr(w, "counters") else None
        if c is not None:
            cnt[b, :3] = [c.get("lp2d", 0), c.get("lp1d", 0), c.get("resolves", 0)]
            cnt[b, 3] = o.get("retries", 0)
    out = dict(K=torch.from_numpy(K), status=torch.from_numpy(status), fail_stage=torch.from_numpy(fail),
               sd=None if backward_only else torch.from_numpy(sd), u=None if backward_only else torch.from_numpy(u))
    if counters:
        out["counters"] = torch.from_numpy(cnt)
    return out


def _scan_ragged(records, R, grid, sd_start, sd_end, glen):
    """Ragged batch: path b uses its first glen[b] gridpoints; everything past them is NaN (tb_scan_ragged)."""
    B, G, W = records.shape
    gr = _np(grid)
    K, sd, u = np.full((B, G, 2), np.nan), np.full((B, G), np.nan), np.full((B, G - 1), np.nan)
    status, fail = np.zeros(B, dtype=np.int32), np.full(B, -1, dtype=np.int32)
    for b in range(B):
        n = int(glen[b])
        o = _wrapper(records, R, b, gr[b], n).compute_parameterization(_scalar(sd_start, b), _scalar(sd_end, b))
        K[b, :n], status[b] = o["K"], o["status"]
        if o["status"] != 3:
            sd[b, :n], u[b, :n - 1] = o["sd"], o["u"]
    return dict(K=torch.from_numpy(K), sd=torch.from_numpy(sd), u=torch.from_numpy(u), status=torch.from_numpy(status),
                fail_stage=torch.from_numpy(fail))


def coeff_second_order(model, params, ppoly, breaks, grid, taulim, friction, interp, records, R_total, row0):
    """Double of tb_coeff_second_order: the registry's models in numpy, rows assembled by the rows_canlinear double."""
    pp, br, gr = _np(ppoly), _np(breaks), _np(grid)
    B, _, nseg, dof = pp.shape
    G = gr.shape[-1]
    prm = np.asarray(params, dtype=np.float64).reshape(-1)
    a, b, c = np.empty((B, G, dof)), np.empty((B, G, dof)), np.empty((B, G, dof))
    for p_ in range(B):
        g = np.ascontiguousarray(_per_path(gr, p_))
        q, qd, qdd = (orc.ppoly_eval(pp[p_], _per_path(br, p_), g, o) for o in (0, 1, 2))
        sq, cq = np.sin(q), np.cos(q)
        if model == "coupled_cosine":
            m0, m1, h, g0 = prm
            c[p_] = g0 * sq
            a[p_] = m0 * qd + m1 * (cq * (cq * qd).sum(-1, keepdims=True) + sq * (sq * qd).sum(-1, keepdims=True))
            b[p_] = (m0 * qdd + m1 * (cq * (cq * qdd).sum(-1, keepdims=True) + sq * (sq * qdd).sum(-1, keepdims=True))
                     + h * sq * (qd * qd).sum(-1, keepdims=True))
        else:
            c[p_] = prm[1::2] * sq
            a[p_] = prm[0::2] * qd
            b[p_] = prm[0::2] * qdd
        if friction is not None:
            c[p_] = c[p_] + np.sign(qd) * _np(friction)
    tl = _np(taulim)
    gaug = np.concatenate((tl[..., 1], -tl[..., 0]), axis=-1)
    return rows_canlinear(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c), None, torch.from_numpy(gaug),
                          2 if gaug.ndim == 1 else 3, grid, interp, records, R_total, row0)


def xbound_constant(ppoly, breaks, grid, vlim, records, R_total, write_xbound):
    coeff_velacc(ppoly, breaks, grid, vlim, None, False, records, R_total, 0, write_xbound)


def scan_velacc(ppoly, breaks, grid, alim, interp, xbound, sd_start=None, sd_end=None, sd_end_hi=None,
                backward_only=False, counters=False, sd_forward=None, forward_from=None, fast_lower=False, glen=None):
    """Double of the fused vel+acc scan: materialise the acceleration rows with the K1 double, take the velocity bound
    from `xbound`, run the record scan."""
    B, _, nseg, dof = ppoly.shape
    G = grid.shape[-1]
    R = (4 if interp else 2) * dof
    rec, _ = alloc_records(B, G, R, None)
    coeff_velacc(ppoly, breaks, grid, None, alim, interp, rec, R, 0, 0)
    rec[:, :, 3 * R:3 * R + 2] = xbound
    return scan(rec, R, grid, sd_start, sd_end, sd_end_hi, backward_only, counters, sd_forward, forward_from, fast_lower,
                glen)


def _scan_sd(records, R, grid, sd_start, sd_end, slow):
    """TOPPRAsd passes (desired_duration_algorithm.py:42-121, 207-234): controllable sets, then a forward pass with no
    retry rule and x_next = clip(x + 2 delta u - 1e-5, K[i+1]); fastest: g = (-2 delta, -1), slowest: g = (2 delta, 1).
    The `sd` output holds x = sd^2 like the kernel's TB_SCAN_SD_FORWARD mode."""
    B, G, W = records.shape
    gr = _np(grid)
    K = np.zeros((B, G, 2))
    xs, us = np.full((B, G), np.nan), np.full((B, G - 1), np.nan)
    status, fail = np.zeros(B, dtype=np.int32), np.full(B, -1, dtype=np.int32)
    for b in range(B):
        g = _per_path(gr, b)
        w = _wrapper(records, R, b, g)
        s0, s1 = _scalar(sd_start, b), _scalar(sd_end, b)
        K[b] = w.compute_controllable_sets(s1, s1)
        x0 = s0 * s0
        if np.isnan(K[b]).any() or x0 + 1e-5 < K[b, 0, 0] or K[b, 0, 1] + 1e-5 < x0:
            status[b] = 3
            fail[b] = int(np.nonzero(np.isnan(K[b]).any(axis=1))[0].max()) if np.isnan(K[b]).any() else 0
            continue
        xs[b, 0] = x0
        for i in range(G - 1):
            delta = g[i + 1] - g[i]
            obj = [2 * delta, 1.0] if slow else [-2 * delta, -1.0]
            u = w.solve_stagewise_optim(i, None, obj, xs[b, i], xs[b, i], K[b, i + 1, 0], K[b, i + 1, 1])[0]
            if np.isnan(u):
                status[b], fail[b] = 1, i
                break
            us[b, i] = u
            xs[b, i + 1] = min(K[b, i + 1, 1], max(K[b, i + 1, 0], xs[b, i] + 2 * delta * u - 1e-5))
    return dict(K=torch.from_numpy(K), sd=torch.from_numpy(xs), u=torch.from_numpy(us), status=torch.from_numpy(status),
                fail_stage=torch.from_numpy(fail))


def scan_robust(records, R, conic_row0, conic_rows, ellipsoid, grid, sd_start=None, sd_end=None, backward_only=False,
                counters=False, feasible_sets=False):
    B, G, W = records.shape
    gr = _np(grid)
    if feasible_sets:
        X = np.empty((B, G, 2))
        for b in range(B):
            rows, xb = _rows_of(records, R, b)
            X[b] = orc.feasible_rows_robust(rows, xb, _per_path(gr, b), conic_row0, conic_rows, ellipsoid)
        return dict(K=torch.from_numpy(X), status=torch.zeros(B, dtype=torch.int32),
                    fail_stage=torch.full((B,), -1, dtype=torch.int32))
    K, sd, u = np.zeros((B, G, 2)), np.full((B, G), np.nan), np.full((B, max(G - 1, 1)), np.nan)
    status = np.zeros(B, dtype=np.int32)
    for b in range(B):
        rows, xb = _rows_of(records, R, b)
        o = orc.solve_rows_robust(rows, xb, _per_path(gr, b), conic_row0, conic_rows, ellipsoid, _scalar(sd_start, b),
                                  _scalar(sd_end, b))
        K[b], status[b] = o["K"], o["status"]
        if backward_only:     # no start-velocity check: uncontrollable iff a stage of the backward pass was infeasible
            status[b] = 3 if np.isnan(o["K"]).any() else 0
        elif o["status"] == 0:
            sd[b], u[b, :G - 1] = o["sd"], o["u"]
    if backward_only:
        return dict(K=torch.from_numpy(K), status=torch.from_numpy(status),
                    fail_stage=torch.full((B,), -1, dtype=torch.int32))
    out = dict(K=torch.from_numpy(K), sd=torch.from_numpy(sd), u=torch.from_numpy(u[:, :max(G - 1, 0)]),
               status=torch.from_numpy(status), fail_stage=torch.full((B,), -1, dtype=torch.int32))
    if counters:
        out["counters"] = torch.zeros((B, 4), dtype=torch.int32)
    return out


def feasible_sets(records, R, grid):
    B, G, W = records.shape
    gr = _np(grid)
    X = np.empty((B, G, 2))
    for b in range(B):
        X[b] = _wrapper(records, R, b, _per_path(gr, b)).compute_feasible_sets()
    return torch.from_numpy(X)


def reachable_sets(records, R, grid, sdmin=None, sdmax=None):
    """compute_reachable_sets (reachability_algorithm.py:378-431) on the oracle's STATEFUL wrapper: the feasible-set pass
    first, then the forward recursion through solve_stagewise_optim with the warm-start slots it left behind."""
    B, G, W = records.shape
    gr = _np(grid)
    X, L, fs = np.empty((B, G, 2)), np.zeros((B, G, 2)), np.full(B, -1, dtype=np.int32)
    for b in range(B):
        g = _per_path(gr, b)
        w = _wrapper(records, R, b, g)
        X[b] = w.compute_feasible_sets()
        s0 = _scalar(sdmin, b)
        L[b, 0] = [s0 ** 2, _scalar(sdmax, b, s0) ** 2]
        deltas = np.diff(g)
        for i in range(G - 1):
            dq = deltas[i - 1]
            obj = np.array([-2 * dq, -1.0])
            o1 = w.solve_stagewise_optim(i, None, obj, L[b, i, 0], L[b, i, 1], X[b, i + 1, 0], X[b, i + 1, 1])
            o0 = w.solve_stagewise_optim(i, None, -obj, L[b, i, 0], L[b, i, 1], X[b, i + 1, 0], X[b, i + 1, 1])
            L[b, i + 1] = [o0[1] + 2 * dq * o0[0], o1[1] + 2 * dq * o1[0]]
            if L[b, i + 1, 0] < 0:
                L[b, i + 1, 0] = 0
            if np.isnan(L[b, i + 1]).any():
                fs[b] = i + 1
                break
    return dict(X=torch.from_numpy(X), L=torch.from_numpy(L), fail_stage=torch.from_numpy(fs))


def propose_gridpoints(ppoly, breaks, max_err_threshold=1e-4, max_iteration=100, max_seg_length=0.05, min_nb_points=100,
                       max_points=2048):
    """interpolator.py:49-122 per path on the oracle's PPoly evaluation.  Failures as in tb_propose_gridpoints: status 1
    (the last allowed pass ran; the reference raises) skips the doubling, and status -2 (a pass or the doubling would
    exceed max_points) returns the last list that fitted."""
    pp, br = _np(ppoly), _np(breaks)
    B = pp.shape[0]
    grid = np.zeros((B, max_points))
    glen, status = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
    for b in range(B):
        x = _per_path(br, b)
        pts = [x[0], x[-1]]
        it, st, converged = 0, 0, False
        for it in range(max_iteration):
            arr = np.asarray(pts)
            mids, dist = 0.5 * (arr[:-1] + arr[1:]), arr[1:] - arr[:-1]
            qss = orc.ppoly_eval(pp[b], x, mids, 2)
            new = [mids[j] for j in range(len(mids))
                   if dist[j] > max_seg_length or np.max(np.abs(0.5 * qss[j] * dist[j] ** 2)) > max_err_threshold]
            if len(pts) + len(new) > max_points:
                st = -2
                break
            if not new:
                converged = True
                break
            pts = sorted(pts + new)
        if st == 0 and (not converged or it == max_iteration - 1):
            st = 1
        while st == 0 and len(pts) < min_nb_points:
            if 2 * len(pts) - 1 > max_points:
                st = -2
                break
            arr = np.asarray(pts)
            pts = sorted(pts + list(0.5 * (arr[:-1] + arr[1:])))
        n = len(pts)
        grid[b, :n], grid[b, n:], glen[b], status[b] = pts, pts[-1], n, st
    return torch.from_numpy(grid), torch.from_numpy(glen), torch.from_numpy(status)


def _duration(xs, deltas):
    sds = np.sqrt(xs)
    t = 0
    for i in range(len(deltas)):
        t += 2 * deltas[i] / (sds[i + 1] + sds[i] + 1e-9)
    return t


def sd_bisect(x_fast, u_fast, x_slow, u_slow, grid, desired, atol=1e-5, status_in=None, max_iter=200):
    """desired_duration_algorithm.py:139-191 per path."""
    xf, uf, xs, us, gr, want = (_np(t) for t in (x_fast, u_fast, x_slow, u_slow, grid, desired))
    B, G = xf.shape
    sd, u = np.full((B, G), np.nan), np.full((B, G - 1), np.nan)
    info, status = np.zeros((B, 4)), np.zeros(B, dtype=np.int32)
    st_in = None if status_in is None else _np(status_in)
    for b in range(B):
        if st_in is not None and st_in[b] == 3:
            status[b], info[b, :3] = 3, np.nan
            continue
        deltas = np.diff(_per_path(gr, b))
        with np.errstate(invalid="ignore"):
            d_fast, d_slow = _duration(xf[b], deltas), _duration(xs[b], deltas)
            its = 0
            if d_fast > want[b]:
                alpha = 1.0
            elif d_slow < want[b]:
                alpha = 0.0
            else:
                lo, hi, diff, alpha = 1.0, 0.0, 10, 0.5
                while diff > atol and its < max_iter:
                    its += 1
                    alpha = 0.5 * (lo + hi)
                    d = _duration(alpha * xf[b] + (1 - alpha) * xs[b], deltas)
                    if d < want[b]:
                        lo, diff = alpha, want[b] - d
                    else:
                        hi, diff = alpha, d - want[b]
            sd[b] = np.sqrt(alpha * xf[b] + (1 - alpha) * xs[b])
        u[b] = alpha * uf[b] + (1 - alpha) * us[b]
        status[b] = 1 if np.isnan(sd[b]).any() else 0
        info[b] = [alpha, d_fast, d_slow, its]
    return dict(sd=torch.from_numpy(sd), u=torch.from_numpy(u), info=torch.from_numpy(info), status=torch.from_numpy(status))


def spline_time_stamps(sd, grid, glen=None):
    """parametrizer.py:171-186 per path (compacted, tail padded with the last kept entry)."""
    v, gr = _np(sd), _np(grid)
    B, G = v.shape
    t, s, nk = np.zeros((B, G)), np.zeros((B, G)), np.zeros(B, dtype=np.int32)
    for b in range(B):
        g = _per_path(gr, b)
        n = G if glen is None else int(_np(glen)[b])
        acc, keep_t, keep_s = 0.0, [0.0], [g[0]]
        for i in range(1, n):
            avg = (v[b, i - 1] + v[b, i]) / 2
            ds = g[i] - g[i - 1]
            dt = ds / avg if avg > 1e-8 else 5
            acc = acc + dt
            if not dt < 1e-8:
                keep_t.append(acc)
                keep_s.append(g[i])
        k = len(keep_t)
        t[b, :k], s[b, :k], t[b, k:], s[b, k:], nk[b] = keep_t, keep_s, keep_t[-1], keep_s[-1], k
    return torch.from_numpy(t), torch.from_numpy(s), torch.from_numpy(nk)


# ---- LP shims -------------------------------------------------------------------------------------------------------------
def lp2d_batch(v, a, b, c, low, high, active_c=None):
    v, low, high = (np.asarray(_np(t) if isinstance(t, torch.Tensor) else t, dtype=np.float64) for t in (v, low, high))
    B = v.shape[0]
    a, b, c = (np.asarray(_np(t) if isinstance(t, torch.Tensor) else t, dtype=np.float64).reshape(B, -1) for t in (a, b, c))
    act = np.zeros((B, 2), dtype=np.int64) if active_c is None else np.asarray(active_c, dtype=np.int64).reshape(B, 2)
    res, val, var, out_act = np.zeros(B, np.int32), np.zeros(B), np.zeros((B, 2)), np.zeros((B, 2), np.int32)
    for i in range(B):
        res[i], val[i], var[i], out_act[i] = orc.lp2d(v[i], a[i], b[i], c[i], low[i], high[i], act[i])
    return res, val, var, out_act


def lp1d_batch(v, a, b, low, high):
    v, low, high = (np.asarray(_np(t) if isinstance(t, torch.Tensor) else t, dtype=np.float64) for t in (v, low, high))
    B = v.shape[0]
    a, b = (np.asarray(_np(t) if isinstance(t, torch.Tensor) else t, dtype=np.float64).reshape(B, -1) for t in (a, b))
    res, val, var, act = np.zeros(B, np.int32), np.zeros(B), np.zeros(B), np.zeros(B, np.int32)
    for i in range(B):
        res[i], val[i], var[i], act[i] = orc.lp1d(v[i], a[i], b[i], float(low[i]), float(high[i]))
    return res, val, var, act


# ---- K3: ParametrizeConstAccel (parametrizer.py:52-129) -------------------------------------------------------------------
def time_grid(sd, grid):
    sdn, gr = _np(sd), _np(grid)
    B, G = sdn.shape
    t, us = np.zeros((B, G)), np.zeros((B, G - 1))
    for b in range(B):
        s, v = _per_path(gr, b), sdn[b]
        x = v ** 2
        for i in range(G - 1):
            us[b, i] = 0.5 * (x[i + 1] - x[i]) / (s[i + 1] - s[i])
            t[b, i + 1] = t[b, i] + 2 * (s[i + 1] - s[i]) / (v[i] + v[i + 1])
    return torch.from_numpy(t), torch.from_numpy(us)


def constaccel_eval(ppoly, breaks, grid, sd, t_grid, us, ts, order):
    pp, br, gr, sdn, tg, un, tn = (_np(t) for t in (ppoly, breaks, grid, sd, t_grid, us, ts))
    B, dof = pp.shape[0], pp.shape[3]
    M = tn.shape[-1]
    out = np.zeros((B, M, dof))
    for b in range(B):
        s, t = _per_path(gr, b), _per_path(tn, b)
        idx = np.searchsorted(tg[b], t, side="right") - 1
        idx = np.where(idx == un.shape[1], idx - 1, idx)
        dt = t - tg[b][idx]
        u = un[b][idx]
        v = sdn[b][idx] + dt * u
        pos = s[idx] + dt * sdn[b][idx] + 0.5 * dt ** 2 * u
        ev = lambda k: orc.ppoly_eval(pp[b], _per_path(br, b), pos, k)  # noqa: E731
        if order == 0:
            out[b] = ev(0)
        elif order == 1:
            out[b] = ev(1) * v[:, None]
        else:
            out[b] = ev(2) * v[:, None] ** 2 + ev(1) * u[:, None]
    return torch.from_numpy(out)


class _NoStream(object):
    def synchronize(self):
        pass


PATCHED = ("spline_fit", "ppoly_eval", "record_doubles", "alloc_records", "init_bounds", "coeff_velacc",
           "rows_canlinear", "coeff_second_order", "xbound_varying", "xbound_constant", "scan", "scan_velacc", "scan_robust", "feasible_sets", "lp2d_batch", "lp1d_batch",
           "time_grid", "constaccel_eval", "has_ubound", "check_glen", "reachable_sets", "propose_gridpoints", "sd_bisect",
           "spline_time_stamps")


def install(monkeypatch):
    """Route toppra_b200 through this module for the duration of one test."""
    import toppra_b200  # noqa: F401
    from toppra_b200 import _lib, engine
    monkeypatch.setattr(_lib, "require_cuda", lambda: torch)
    monkeypatch.setattr(engine, "default_device", lambda device=None: torch.device("cpu"))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _NoStream())
    for name in PATCHED:
        assert hasattr(engine, name), name
        monkeypatch.setattr(engine, name, globals()[name])
    return toppra_b200


def install_plain():
    """The same routing without pytest's monkeypatch: for spawned worker processes (tests/test_distributed_gloo.py),
    which end with the test anyway."""
    class _Setter(object):
        @staticmethod
        def setattr(obj, name, value):
            setattr(obj, name, value)
    return install(_Setter)
