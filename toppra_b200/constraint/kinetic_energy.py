"""Limits on the kinetic energy and the linear momentum of the whole robot in motion.

    T = 1/2 qd^T M(q) qd <= E_max          (KineticEnergyConstraint)
    |p| = |sum_k m_k v_ck| <= p_max       (MomentumConstraint)

Energy-based safety schemes for human-robot collaboration cap T, because no contact can take more energy out of the arm
than it carries; collaborative arms commonly cap the momentum next to the tool speed and the energy, and the momentum
bounds how hard the arm pushes a light base or cart when it starts and stops.  Both sums run over every moving body of a
`toppra_b200.RigidBodyModel` (with its folded links and payloads); the static base does not move.

Along a path qd = q' s', so with x = s'^2 both limits are exact and linear in x:

    T = T(q, q') x <= E_max,    |p|^2 = |p(q, q')|^2 x <= p_max^2

one CanonicalLinear row per gridpoint: a = 0, b, c = -limit (F = [1], g = [0]), the shape of CartesianVelocityNorm's and
CollisionEnergyConstraint's device rows; p_max is squared once on the host.  No mass-matrix inverse is involved, so
joints that move no inertia are fine.  Every b of the batch (or record chunk) comes from ONE
`tbd_energy_momentum_terms` launch, one forward velocity walk of the tree per gridpoint.  So TOPPRA, BatchTOPPRA,
BatchTOPPRAsd, feasible, reachable and controllable sets, ragged grids, record chunks and order-k paths take them
unchanged."""
import numpy as np

from .cartesian_velocity_norm import append_sd2_rows, sd2_num_rows, single_path_limit
from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .. import _lib
from ..dynamics import RigidBodyModel


class _WholeRobotLimit(LinearConstraint):
    """b(q, q') s'^2 <= limit with b = model.energy_momentum_terms(q, q', which): the parts both constraints share."""

    which = None

    def __init__(self, model, limit, unit, discretization_scheme):
        super(_WholeRobotLimit, self).__init__()
        name = type(self).__name__
        if not isinstance(model, RigidBodyModel):
            raise ValueError("%s needs a RigidBodyModel (RigidBodyModel.from_urdf(...)); got %s"
                             % (name, type(model).__name__))
        self.set_discretization_type(discretization_scheme)
        lim = np.array(limit, dtype=np.float64)
        if lim.ndim > 1:
            raise ValueError("%s: limit must be a float or (B,); got shape %s" % (name, lim.shape))
        if np.isnan(lim).any() or (lim < 0).any():
            raise ValueError("%s: the limit must be >= 0 (not NaN); got %s" % (name, limit))
        self.model = model
        self.dof = model.dof
        rows = self._row_limit(lim)
        self.limit, self._path_limits = (float(rows), None) if lim.ndim == 0 else (None, rows)
        self.identical = True
        self._format_string = "    {:}: {:} {:}\n".format(
            name, "per path" if lim.ndim else float(lim), unit)

    @staticmethod
    def _row_limit(lim):
        """The limit of the row b x <= limit from the user's limit."""
        return lim

    def get_dof(self):
        return self.dof

    def _interp(self):
        return self.discretization_type == DiscretizationType.Interpolation

    def terms(self, q, qs):
        """b of the constraint at (q, qs = q'): CUDA tensors (M, nv) -> (M,), one tbd_energy_momentum_terms launch."""
        return self.model.energy_momentum_terms(q, qs, self.which)

    def compute_constraint_params(self, path, gridpoints):
        """The reference's 7-tuple for one path: a = 0, b from one launch on q, q' at the gridpoints, c = 0,
        F = [1], g = [limit]."""
        check_dof(self.dof, path.dof)
        limit = single_path_limit(self)
        gridpoints = np.asarray(gridpoints, dtype=float)
        G = gridpoints.shape[0]
        torch = _lib.require_cuda()
        q, qs = (torch.as_tensor(np.atleast_2d(path(gridpoints, o)), device="cuda") for o in (0, 1))
        b = self.terms(q, qs).cpu().numpy().reshape(G, 1)
        a, c = np.zeros((G, 1)), np.zeros((G, 1))
        F, g = np.ones((1, 1)), np.full(1, limit)
        if self._interp():
            return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
        return a, b, c, F, g, None, None

    # ---- device route ------------------------------------------------------------------------------------------
    def num_rows(self, ctx):
        return sd2_num_rows(self, ctx)

    def append_records(self, ctx, records, R_total, row0):
        """One tbd_energy_momentum_terms launch for the B x G gridpoints of this context, then the rows a = 0, b,
        c = 0 - limit (F = [1], g = [0]) through tb_rows_canlinear (with the interpolation lift if selected)."""
        append_sd2_rows(self, ctx, self.terms, records, R_total, row0)


class KineticEnergyConstraint(_WholeRobotLimit):
    """model: a RigidBodyModel; limit: E_max >= 0 in J, a float or (B,) with one limit per path of the batch;
    discretization_scheme: Collocation (default) or Interpolation.  Row: b = T(q, q'), limit E_max.  1 row per stage,
    2 with Interpolation."""

    which = "energy"

    def __init__(self, model, limit, discretization_scheme=DiscretizationType.Collocation):
        super(KineticEnergyConstraint, self).__init__(model, limit, "J", discretization_scheme)


class MomentumConstraint(_WholeRobotLimit):
    """model: a RigidBodyModel; limit: p_max >= 0 in kg m/s, a float or (B,) with one limit per path of the batch;
    discretization_scheme: Collocation (default) or Interpolation.  Row: b = |p(q, q')|^2, limit p_max^2 (the
    constraint's `limit`).  1 row per stage, 2 with Interpolation."""

    which = "momentum"

    def __init__(self, model, limit, discretization_scheme=DiscretizationType.Collocation):
        super(MomentumConstraint, self).__init__(model, limit, "kg m/s", discretization_scheme)

    @staticmethod
    def _row_limit(lim):
        return lim * lim
