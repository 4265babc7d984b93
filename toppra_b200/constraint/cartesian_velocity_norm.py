"""Cartesian velocity-norm constraint — the C++-only constraint of the reference
(`cpp/src/toppra/constraint/cartesian_velocity_norm.hpp:10-95`, `.cpp:23-54`; SURVEY §8 f4) with a Python surface.

    v = J(p(s)) p'(s) sd  is the 6-D velocity of a frame;   ||v||_S^2 = v^T S v <= limit
    =>  one CanonicalLinear row per gridpoint:  a = 0,  b = v1^T S v1  (v1 = the frame velocity for sd = 1),  c = 0,
        F = [1],  g = [limit]                                                                 (.cpp:36-52)

`compute_velocity(q, qd) -> v[6]` is USER code (the C++ class leaves `computeVelocity` pure virtual), called once per
gridpoint on the host with q = p(s), qd = p'(s).  Constant (S, limit) gives an identical F/g like the C++ constant
constructor; `velocity_limit(s) -> (S, limit)` gives the varying form (`computeVelocityLimit`, .hpp:73-80).

A `toppra_b200.RigidBodyFrame` (`RigidBodyModel.frame(...)`) as `compute_velocity` with a constant limit takes the device
route: every b of the batch (or record chunk) comes from ONE `tbd_velocity_norm_terms` launch on q, q' evaluated on the
device, and the rows go through `tb_rows_canlinear` as a = 0, b, c = -limit with F = [1], g = [0] — the reference's
F.c - g bit for bit.  There `limit` may also be (B,), one limit per path of the batch.  The varying form keeps the
single-path host route."""
import numpy as np

from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .. import engine
from ..dynamics import RigidBodyFrame


class CartesianVelocityNorm(LinearConstraint):
    """compute_velocity: (q, qd) -> v[6] or a RigidBodyFrame; S (6, 6); limit: float, or (B,) per path with a
    RigidBodyFrame; velocity_limit(s) -> (S, limit) instead of (S, limit); discretization_scheme: Collocation (default)
    or Interpolation."""

    def __init__(self, compute_velocity, S=None, limit=None, velocity_limit=None, dof=None,
                 discretization_scheme=DiscretizationType.Collocation):
        super(CartesianVelocityNorm, self).__init__()
        self.set_discretization_type(discretization_scheme)
        self.compute_velocity = compute_velocity
        self.velocity_limit = velocity_limit
        frame = isinstance(compute_velocity, RigidBodyFrame)
        if frame and dof is not None and dof != compute_velocity.dof:
            raise ValueError("Wrong dimension: constraint dof ({:d}) not equal to the frame's model dof ({:d})".format(
                dof, compute_velocity.dof))
        self.dof = compute_velocity.dof if frame and dof is None else dof
        self._path_limits = None   # (B,) limits of the device route
        if velocity_limit is None:
            if S is None or limit is None:
                raise ValueError("CartesianVelocityNorm needs (S, limit) or velocity_limit(s) -> (S, limit)")
            if np.ndim(limit) == 1 and frame:
                lim = np.array(limit, dtype=float)
                self._check(S, lim.min() if lim.size else 0.0)
                self.S, self.limit, self._path_limits = np.array(S, dtype=float), None, lim
            else:
                self.S, self.limit = np.array(S, dtype=float), float(limit)
                self._check(self.S, self.limit)
        else:
            self.S, self.limit = np.zeros((6, 6)), 1.0  # like the C++ varying constructor: set per gridpoint
        self.identical = velocity_limit is None
        self._format_string = "    Velocity norm limit: {:}\n".format(
            ("per path" if self._path_limits is not None else self.limit) if self.identical else "varying")

    @staticmethod
    def _check(S, limit):  # .cpp:16-21
        if limit < 0:
            raise ValueError("Velocity limit should be positive.")
        if np.shape(S) != (6, 6):
            raise ValueError("S matrix should be of size 6x6.")

    def get_dof(self):
        return self.dof

    def compute_constraint_params(self, path, gridpoints):
        if self.dof is not None:
            check_dof(self.dof, path.dof)
        gridpoints = np.asarray(gridpoints, dtype=float)
        G = gridpoints.shape[0]
        q, qd = path(gridpoints), path(gridpoints, 1)
        limit = single_path_limit(self)
        a, b, c = np.zeros((G, 1)), np.zeros((G, 1)), np.zeros((G, 1))
        F = np.ones((1, 1)) if self.identical else np.ones((G, 1, 1))
        g = np.full(1, limit) if self.identical else np.zeros((G, 1))
        S = self.S
        # a RigidBodyFrame evaluates every gridpoint in one launch; a user callback runs point by point
        vs = self.compute_velocity(q, qd) if isinstance(self.compute_velocity, RigidBodyFrame) else None
        for i in range(G):
            if not self.identical:
                S, limit = self.velocity_limit(gridpoints[i])
                S, limit = np.asarray(S, dtype=float), float(limit)
                self._check(S, limit)
                g[i, 0] = limit
            v = vs[i] if vs is not None else np.asarray(self.compute_velocity(q[i], qd[i]), dtype=float)
            if v.shape != (6,):
                raise ValueError("compute_velocity must return the 6-D frame velocity")
            b[i, 0] = v.dot(S.dot(v))  # v^T (S v), .cpp:43-46
        if self.discretization_type == DiscretizationType.Interpolation:
            return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=self.identical)
        return a, b, c, F, g, None, None

    # ---- device route: a RigidBodyFrame with a constant limit ------------------------------------------------
    def _device(self):
        return isinstance(self.compute_velocity, RigidBodyFrame) and self.identical

    def _interp(self):
        return self.discretization_type == DiscretizationType.Interpolation

    def num_rows(self, ctx):
        if not self._device():
            return super(CartesianVelocityNorm, self).num_rows(ctx)
        return sd2_num_rows(self, ctx)

    def append_records(self, ctx, records, R_total, row0):
        """One tbd_velocity_norm_terms launch for the B x G gridpoints of this context, then the rows a = 0, b,
        c = -limit (F = [1], g = [0]) through tb_rows_canlinear (with the interpolation lift if selected)."""
        if not self._device():
            return super(CartesianVelocityNorm, self).append_records(ctx, records, R_total, row0)
        append_sd2_rows(self, ctx, lambda q, qs: self.compute_velocity.velocity_norm_terms(q, qs, self.S), records,
                        R_total, row0)


# ---- a limit b(q, q') s'^2 <= limit: the parts shared by CartesianVelocityNorm, CollisionEnergyConstraint,
# KineticEnergyConstraint and MomentumConstraint, whose `cons` has dof, limit (a float, or None) and _path_limits
# ((Bfull,) or None) and _interp() ----------------------------------------------------------------------------------
def single_path_limit(cons):
    """The limit of the single-path route: the float, or the only per-path limit."""
    if cons._path_limits is None:
        return cons.limit
    if cons._path_limits.shape != (1,):
        raise ValueError("a single path takes one limit; got %d" % cons._path_limits.shape[0])
    return float(cons._path_limits[0])


def sd2_num_rows(cons, ctx):
    """Rows per stage of the device route, after checking the batch: the path's dof, and one limit per path of the
    full batch when the limits are per path."""
    check_dof(cons.dof, ctx.bpath.dof)
    if cons._path_limits is not None and cons._path_limits.shape[0] != ctx.total:
        raise ValueError("%s: limit has shape %s; expected a float or (%d,)"
                         % (type(cons).__name__, cons._path_limits.shape, ctx.total))
    return 2 if cons._interp() else 1


def append_sd2_rows(cons, ctx, terms, records, R_total, row0):
    """The device rows: ONE `terms(q, qs) -> b (B G,)` call on q, q' of the B x G gridpoints of `ctx`, then a = 0, b,
    c = 0 - limit (the float, or the per-path limits sliced to the context) with F = [1], g = [0] through
    tb_rows_canlinear, with the interpolation lift if selected."""
    sd2_num_rows(cons, ctx)
    limit, path_limits = cons.limit, cons._path_limits
    torch = engine.torch_mod()
    bp = ctx.bpath
    B, G, dof = ctx.B, ctx.G, bp.dof
    q = bp.eval_device(ctx.d_grid, 0).reshape(B * G, dof)
    qs = bp.eval_device(ctx.d_grid, 1).reshape(B * G, dof)
    b = terms(q, qs).reshape(B, G, 1)
    # c = 0 - limit, not -limit: a zero limit gives +0 like the reference's F.c - g = 1 * 0 - 0
    if path_limits is None:
        c = torch.full((B, G, 1), 0.0 - limit, dtype=torch.float64, device=ctx.device)
    else:
        lim = engine.as_device(0.0 - path_limits[ctx.lo:ctx.hi], ctx.device)
        c = lim.reshape(B, 1, 1).expand(B, G, 1).contiguous()
    a = torch.zeros_like(b)
    F = engine.as_device(np.ones((1, 1)), ctx.device)
    g = engine.as_device(np.zeros(1), ctx.device)
    engine.rows_canlinear(a, b, c, F, g, 0, ctx.d_grid, cons._interp(), records, R_total, row0)
