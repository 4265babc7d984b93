"""CanonicalLinear constraints — same surface as the reference `toppra/constraint/linear_constraint.py`.

`compute_constraint_params` keeps the reference's 7-tuple contract (a, b, c, F, g, ubound, xbound) with numpy
arrays; the numbers come from the GPU (csrc/tb_coeff.cu).  Solvers do not go through that host round trip:
they call `append_records` which writes the LP rows of this constraint straight into the device stage records."""
import numpy as np

from .constraint import Constraint, ConstraintType, DiscretizationType
from .. import engine


class LinearConstraint(Constraint):
    """A Canonical Linear Constraint:  a_i u + b_i x + c_i = v,  F_i v <= g_i,  xbound, ubound
    (reference linear_constraint.py:7-81)."""

    def __init__(self):
        self.constraint_type = ConstraintType.CanonicalLinear
        self.discretization_type = DiscretizationType.Collocation
        self.n_extra_vars = 0
        self.identical = False
        self._format_string = ""

    def compute_constraint_params(self, path, gridpoints, *args, **kwargs):
        raise NotImplementedError

    # ---- device protocol used by toppra_b200.algorithm / BatchTOPPRA -------------------------------------
    def num_rows(self, ctx):
        """Number of static LP rows this constraint contributes per stage."""
        a, _, _, F = self._host_params(ctx)[:4]
        if a is None:
            return 0
        return F.shape[0] if self.identical else F.shape[1]

    def has_ubound(self, ctx):
        """True if this constraint returns a `ubound` (then the stage records carry a u-bound pair, TB_SCAN_UBOUND).
        Constraints with their own device implementation never do; user-defined subclasses are asked through their
        host 7-tuple."""
        if type(self).append_records is not LinearConstraint.append_records:
            return False
        return self._host_params(ctx)[5] is not None

    def append_records(self, ctx, records, R_total, row0):
        """Write this constraint's rows [row0, row0+num_rows) and intersect its x / u bounds into `records`.

        Default implementation for user-defined subclasses: take the host 7-tuple from
        `compute_constraint_params` (single path only) and assemble F.a, F.b, F.c - g on the device
        (seidelWrapper.__init__, cy_seidel_solverwrapper.pyx:474-520)."""
        torch = engine.torch_mod()
        a, b, c, F, g, ubound, xbound = self._host_params(ctx)
        dev = records.device
        if ubound is not None:
            # seidelWrapper.__init__ (pyx:512-515): low[i, 0] = max(low, ubound[i, 0]), high[i, 0] = min(high, ubound[i, 1])
            if not engine.has_ubound(records, R_total):
                raise ValueError("stage records without a u-bound pair: allocate them with alloc_records(..., ubound=True)")
            ub = engine.as_device(np.asarray(ubound, dtype=np.float64)[None], dev)
            records[:, :, 3 * R_total + 2] = torch.maximum(records[:, :, 3 * R_total + 2], ub[:, :, 0])
            records[:, :, 3 * R_total + 3] = torch.minimum(records[:, :, 3 * R_total + 3], ub[:, :, 1])
        if a is not None:
            d = lambda x: engine.as_device(np.asarray(x, dtype=np.float64)[None], dev)  # noqa: E731
            if self.identical:
                Fd, gd, mode = engine.as_device(F, dev), engine.as_device(g, dev), 0
            else:
                Fd, gd, mode = d(F), d(g), 1
            engine.rows_canlinear(d(a), d(b), d(c), Fd, gd, mode, ctx.d_grid, False, records, R_total, row0)
        if xbound is not None:
            xb = engine.as_device(np.asarray(xbound, dtype=np.float64)[None], dev)
            records[:, :, 3 * R_total] = torch.maximum(records[:, :, 3 * R_total], xb[:, :, 0])
            records[:, :, 3 * R_total + 1] = torch.minimum(records[:, :, 3 * R_total + 1], xb[:, :, 1])

    def _host_params(self, ctx):
        cache = getattr(self, "_hp_cache", None)
        if cache is None or cache[0] is not ctx:
            if ctx.B != 1 or ctx.path is None:
                raise NotImplementedError(
                    "toppra_b200: %s has no batched device implementation" % type(self).__name__)
            self._hp_cache = (ctx, self.compute_constraint_params(ctx.path, ctx.grid_host))
        return self._hp_cache[1]


class RecordContext(object):
    """What a constraint needs to write its rows: the (batched) device path, the gridpoints on device and host."""

    def __init__(self, bpath, d_grid, grid_host, path=None, lo=0, hi=None, total=None):
        self.bpath = bpath          # BatchSplineInterpolator (or a chunk view of one)
        self.d_grid = d_grid        # CUDA tensor [G] (shared) or [B, G]
        self.grid_host = grid_host  # numpy [G] (shared grids only) or None
        self.path = path            # the user's single path object (B == 1) or None
        self.B = bpath.B
        self.G = d_grid.shape[-1]
        self.device = bpath.device
        self.lo = lo                # this context covers paths [lo, hi) of the full batch (chunked solves)
        self.hi = self.B if hi is None else hi
        self.total = self.hi if total is None else total   # paths of the full batch (per-path limit arrays)

    def limits(self, t):
        """Per-path limit tensors [Bfull, dof, 2] are sliced to this chunk; shared ones pass through."""
        return t[self.lo:self.hi] if (t is not None and t.dim() == 3) else t


def canlinear_colloc_to_interpolate(a, b, c, F, g, xbound, ubound, gridpoints, identical=False):
    """Convert collocation parameters to the interpolation scheme (reference linear_constraint.py:84-192):
    the second block evaluates the constraint at s_{i+1} in stage-i variables,
    a+ = a_{i+1} + 2 delta_i b_{i+1}, b+ = b_{i+1}, c+ = c_{i+1}; the last stage duplicates itself.

    Host (numpy) utility kept for API compatibility; the solvers use the device version in
    csrc/tb_coeff.cu (tb_coeff_velacc / tb_rows_canlinear with interp=1)."""
    if a is None:
        return None, None, None, None, None, xbound, ubound
    a, b, c = np.asarray(a), np.asarray(b), np.asarray(c)
    N = a.shape[0] - 1
    deltas = np.diff(gridpoints)

    def lift(first, nxt):
        out = np.zeros((N + 1, 2 * first.shape[1]))
        d = first.shape[1]
        out[:, :d] = first
        out[:-1, d:] = nxt
        out[-1, d:] = out[-1, :d]
        return out

    a_intp = lift(a, a[1:] + 2 * deltas.reshape(-1, 1) * b[1:])
    b_intp = lift(b, b[1:])
    c_intp = lift(c, c[1:])
    if identical:
        m, d = F.shape
        g_intp = np.zeros(2 * m)
        g_intp[:m] = g
        g_intp[m:] = g
        F_intp = np.zeros((2 * m, 2 * d))
        F_intp[:m, :d] = F
        F_intp[m:, d:] = F
    else:
        d = a.shape[1]
        m = g.shape[1]
        g_intp = np.zeros((N + 1, 2 * m))
        g_intp[:, :m] = g
        g_intp[:-1, m:] = g[1:]
        g_intp[-1, m:] = g_intp[-1, :m]
        F_intp = np.zeros((N + 1, 2 * m, 2 * d))
        F_intp[:, :m, :d] = F
        F_intp[:-1, m:, d:] = F[1:]
        F_intp[-1, m:, d:] = F[-1]
    return a_intp, b_intp, c_intp, F_intp, g_intp, xbound, ubound
