"""Solver-wrapper strategy interface — same surface as the reference
`toppra/solverwrapper/solverwrapper.py:9-166` + `cy_seidel_solverwrapper.pyx:392-697` (seidelWrapper).

`B200SolverWrapper` holds the stage records on the device (built once at construction, like
seidelWrapper.__init__) and exposes
  * the reference per-stage method `solve_stagewise_optim(i, H, g, x_min, x_max, x_next_min, x_next_max)`
    (one tiny launch per call — for API parity and stage-level tests, not for speed);
  * whole-pass methods used by the algorithms: `parameterize`, `controllable_sets`, `feasible_sets`
    (one launch each, csrc/tb_scan.cu)."""
import numpy as np

from .. import engine
from ..constants import ECOS_INFTY, ECOS_MAXX
from ..constraint import RecordContext


def available_solvers(output_msg=True):
    """Solver availability in the reference's format; only the Seidel path exists here."""
    solver_availability = (("seidel", True), ("b200", True), ("hotqpoases", False), ("qpoases", False),
                           ("ecos", False), ("cvxpy", False))
    if output_msg:
        print(solver_availability)
    return solver_availability


def check_solver_availability(solver):
    return any(sname == solver and avail for sname, avail in available_solvers(False))


class SolverWrapper(object):
    """Base class of solver wrappers (reference solverwrapper.py:49-166)."""

    def __init__(self, constraint_list, path, path_discretization):
        self.constraints = constraint_list
        self.path = path
        self.path_discretization = np.array(path_discretization)
        self.N = len(path_discretization) - 1
        self.deltas = self.path_discretization[1:] - self.path_discretization[:-1]
        assert path.path_interval[0] == path_discretization[0]
        assert path.path_interval[1] == path_discretization[-1]
        for i in range(self.N):
            assert path_discretization[i + 1] > path_discretization[i]
        self.nV = 2 + sum([c.get_no_extra_vars() for c in constraint_list])

    def get_no_stages(self):
        return self.N

    def get_no_vars(self):
        return self.nV

    def get_deltas(self):
        return self.deltas

    def solve_stagewise_optim(self, i, H, g, x_min, x_max, x_next_min, x_next_max):
        raise NotImplementedError

    def setup_solver(self):
        pass

    def close_solver(self):
        pass


class B200SolverWrapper(SolverWrapper):
    """GPU implementation of the reference `seidelWrapper` (Seidel's LP, solve_lp1d=True)."""

    def __init__(self, constraint_list, path, path_discretization, solve_lp1d=True):
        from ..batch import build_records, conic_info
        super(B200SolverWrapper, self).__init__(constraint_list, path, path_discretization)
        if not hasattr(path, "as_batch"):
            raise TypeError("toppra_b200 needs a path with a piecewise-polynomial device form (SplineInterpolator, PPolyPath, "
                            "PiecewisePolyPath, SimplePath, PolynomialPath up to degree 3); got %s" % type(path).__name__)
        bpath = path.as_batch()
        grid = np.ascontiguousarray(self.path_discretization, dtype=np.float64)
        self.ctx = RecordContext(bpath, engine.as_device(grid, bpath.device), grid, path)
        self.records, self.R = build_records(self.ctx, constraint_list)
        self.conic = conic_info(self.ctx, constraint_list)
        self.nC = self.R + 2
        self._solve_lp1d = solve_lp1d
        self._params = None
        self._rows_host = None
        self.active_c_up = np.zeros(2, dtype=np.int32)    # warm-start slots, pyx:526-527
        self.active_c_down = np.zeros(2, dtype=np.int32)

    def _no_conic(self, what):
        if self.conic is not None:
            raise NotImplementedError("%s is not available for problems with a robust (conic) constraint" % what)

    @property
    def params(self):
        """Per-constraint 7-tuples (a, b, c, F, g, ubound, xbound), like seidelWrapper.params."""
        if self._params is None:
            self._params = []
            for c in self.constraints:
                cached = getattr(c, "_hp_cache", None)
                if cached is not None and cached[0] is self.ctx:
                    # the very tuple the stage records were built from (the reference stores the tuples of its
                    # constructor, pyx:440-442; matters for a constraint whose parameters are not reproducible)
                    self._params.append(cached[1])
                else:
                    self._params.append(c.compute_constraint_params(self.path, self.path_discretization))
        return self._params

    def rows(self):
        """LP row arrays like seidelWrapper's a_arr, b_arr, c_arr [(N+1), nC] (rows 0,1 zero) and low/high."""
        rec = self.records[0].cpu().numpy()
        R, G = self.R, rec.shape[0]
        out = {}
        for idx, key in enumerate(("a", "b", "c")):
            arr = np.zeros((G, self.nC))
            arr[:, 2:] = rec[:, idx * R:(idx + 1) * R]
            out[key] = arr
        ub = engine.has_ubound(self.records, R)   # u-bound pair behind the x-bound pair (pyx:512-515)
        out["low"] = np.stack((rec[:, 3 * R + 2] if ub else np.full(G, -1e8), rec[:, 3 * R]), axis=1)
        out["high"] = np.stack((rec[:, 3 * R + 3] if ub else np.full(G, 1e8), rec[:, 3 * R + 1]), axis=1)
        return out

    def solve_stagewise_optim(self, i, H, g, x_min, x_max, x_next_min, x_next_max):
        """One stage LP, reference semantics (cy_seidel_solverwrapper.pyx:549-697): min g.[u,x] subject to the
        stage-i rows, x_min <= x <= x_max, x_next_min <= x + 2 delta_i u <= x_next_max (NaN = bound absent).
        Returns [u, x] or [nan, nan] when infeasible.  One small launch per call (tb_lp1d_batch / tb_lp2d_batch).
        Problems with a robust (conic) constraint: the second-order-cone program of ecosWrapper.solve_stagewise_optim
        (ecos_solverwrapper.py:90-207), one tbr_socp_stage_batch launch."""
        assert 0 <= i <= self.N
        if self.conic is not None:
            return self._solve_stage_conic(i, H, g, x_min, x_max, x_next_min, x_next_max)
        if self._rows_host is None:
            self._rows_host = self.rows()
        rows = self._rows_host
        a, b, c = rows["a"][i].copy(), rows["b"][i].copy(), rows["c"][i].copy()
        low, high = rows["low"][i].copy(), rows["high"][i].copy()
        if not np.isnan(x_min):
            low[1] = max(low[1], x_min)
        if not np.isnan(x_max):
            high[1] = min(high[1], x_max)
        a[0:2], b[0:2], c[0:2] = 0.0, 0.0, -1.0
        if i < self.N:
            if not np.isnan(x_next_min):
                a[0], b[0], c[0] = -2 * self.deltas[i], -1.0, x_next_min
            if not np.isnan(x_next_max):
                a[1], b[1], c[1] = 2 * self.deltas[i], 1.0, -x_next_max
        g = np.asarray(g, dtype=np.float64)
        if x_min == x_max and self._solve_lp1d:
            v = np.array([[-g[0], -g[1] * x_min]])
            res, _, optvar, act = engine.lp1d_batch(v, a[None], (b * x_min + c)[None], low[0:1], high[0:1])
            if res[0] == 0:
                return np.array([np.nan, np.nan])
            (self.active_c_up if g[1] > 0 else self.active_c_down)[0] = act[0]
            return np.array([optvar[0], x_min])
        slot = self.active_c_up if g[1] > 0 else self.active_c_down
        v = np.array([[-g[0], -g[1], 0.0]])
        res, _, optvar, act = engine.lp2d_batch(v, a[None], b[None], c[None], low[None], high[None], slot[None])
        if res[0] == 0:
            return np.array([np.nan, np.nan])
        slot[:] = act[0]
        return optvar[0].copy()

    def _solve_stage_conic(self, i, H, g, x_min, x_max, x_next_min, x_next_max):
        """ecos_solverwrapper.py:90-207: absent x / x_next bounds are -/+ECOS_INFTY, the xbound rows give
        x >= xbound_lo and x <= min(ECOS_MAXX, xbound_hi); no x_next rows at the last stage."""
        assert H is None or np.allclose(H, np.zeros(2))
        if self._rows_host is None:
            self._rows_host = self.rows()
        rows, R = self._rows_host, self.R
        xlo = -ECOS_INFTY if np.isnan(x_min) else x_min
        xhi = ECOS_INFTY if np.isnan(x_max) else x_max
        xbox = [max(xlo, rows["low"][i][1]), min(xhi, min(ECOS_MAXX, rows["high"][i][1]))]
        xnext = None
        if i < self.N:
            xnext = [[self.deltas[i], -ECOS_INFTY if np.isnan(x_next_min) else x_next_min,
                      ECOS_INFTY if np.isnan(x_next_max) else x_next_max]]
        g = np.asarray(g, dtype=np.float64)[:2]
        return engine.socp_stage_batch(g[None], rows["a"][i][None, 2:2 + R], rows["b"][i][None, 2:2 + R],
                                       rows["c"][i][None, 2:2 + R], self.conic[0], self.conic[1], self.conic[2],
                                       np.array([xbox]), xnext)[0]

    # ---- whole-pass entry points ---------------------------------------------------------------------
    def _scalar(self, v):
        return engine.as_device(np.array([float(v)]), self.ctx.device)

    def parameterize(self, sd_start, sd_end, counters=False, sd_forward=None):
        from ..batch import scan_any
        if sd_forward is not None:
            self._no_conic("TOPPRAsd")
            out = engine.scan(self.records, self.R, self.ctx.d_grid, self._scalar(sd_start), self._scalar(sd_end),
                              counters=counters, sd_forward=sd_forward)
        else:
            out = scan_any(self.records, self.R, self.ctx.d_grid, self.conic, self._scalar(sd_start),
                           self._scalar(sd_end), counters=counters)
        res = dict(K=out["K"][0].cpu().numpy(), sd=out["sd"][0].cpu().numpy(), u=out["u"][0].cpu().numpy(),
                   status=int(out["status"][0].item()), fail_stage=int(out["fail_stage"][0].item()))
        if counters:
            res["counters"] = out["counters"][0].cpu().numpy()
        return res

    def parameterize_sd(self, sd_start, sd_end, desired_duration, atol=1e-5):
        """TOPPRAsd on the device: two scans (fastest / slowest forward rules) + tb_sd_bisect; host arrays out.  Robust
        problems: one backward-only conic scan, both forward passes in one tbr_sd_forward_robust launch, tb_sd_bisect."""
        from ..batch import sd_passes_robust
        s0, s1 = self._scalar(sd_start), self._scalar(sd_end)
        if self.conic is not None:
            fast, slow = sd_passes_robust(self.records, self.R, self.conic, self.ctx.d_grid, s0, s1)
        else:
            fast = engine.scan(self.records, self.R, self.ctx.d_grid, s0, s1, sd_forward="fast")
            slow = engine.scan(self.records, self.R, self.ctx.d_grid, s0, s1, sd_forward="slow")
        out = engine.sd_bisect(fast["sd"], fast["u"], slow["sd"], slow["u"], self.ctx.d_grid,
                               self._scalar(desired_duration), atol, status_in=fast["status"])
        info = out["info"][0].cpu().numpy()
        return dict(K=fast["K"][0].cpu().numpy(), status=int(fast["status"][0].item()),
                    blend_status=int(out["status"][0].item()), sd=out["sd"][0].cpu().numpy(),
                    u=out["u"][0].cpu().numpy(), alpha=float(info[0]), duration_fast=float(info[1]),
                    duration_slow=float(info[2]))

    def controllable_sets(self, sdmin, sdmax):
        from ..batch import scan_any
        out = scan_any(self.records, self.R, self.ctx.d_grid, self.conic, None, self._scalar(sdmin),
                       None if sdmin == sdmax else self._scalar(sdmax), backward_only=True)
        return out["K"][0].cpu().numpy(), int(out["status"][0].item())

    def reachable_sets(self, sdmin, sdmax):
        """(X, L, fail_stage) of compute_reachable_sets: one launch (tb_reachable_sets)."""
        self._no_conic("compute_reachable_sets")
        out = engine.reachable_sets(self.records, self.R, self.ctx.d_grid, self._scalar(sdmin), self._scalar(sdmax))
        return out["X"][0].cpu().numpy(), out["L"][0].cpu().numpy(), int(out["fail_stage"][0].item())

    def feasible_sets(self):
        if self.conic is not None:
            return engine.scan_robust(self.records, self.R, self.conic[0], self.conic[1], self.conic[2],
                                      self.ctx.d_grid, feasible_sets=True)["K"][0].cpu().numpy()
        return engine.feasible_sets(self.records, self.R, self.ctx.d_grid)[0].cpu().numpy()
