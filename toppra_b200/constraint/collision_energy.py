"""Collision-energy limit of a robot point working next to people (power and force limiting, ISO/TS 15066, Annex A).
The energy a moving robot point could transfer to a human body region it hits is bounded:

    E = 1/2 mu |v|^2 <= E_max,    mu = (1/m_H + 1/m_R)^-1,    m_R = 1 / (u^T Lambda_v^-1 u),  u = v / |v|

with v the velocity of the contact point (a `toppra_b200.RigidBodyFrame`'s origin), m_H the effective mass of the body
region and m_R the robot's effective (reflected) mass at that point in the direction it moves: Khatib's operational-space
inertia, Lambda_v^-1 = J_v M(q)^-1 J_v^T ("Inertial properties in robotic manipulation", IJRR 1995).  m_R depends on the
pose, so the limit is fast where the arm reflects little mass along its motion and slow where it reflects much.

Along a path v = J_v(q) q' s' and u does not depend on s', so E = b(q, q') s'^2 with

    b = 1/2 |v1|^4 / (|v1|^2 / m_H + v1^T Lambda_v^-1 v1),    v1 = J_v q'  (the frame velocity at s' = 1)

one CanonicalLinear row per gridpoint: a = 0, b, c = -E_max (F = [1], g = [0]), the shape of CartesianVelocityNorm's
device row.  Every b of the batch (or record chunk) comes from ONE `tbd_collision_energy_terms` launch, which forms M(q)
(composite-rigid-body algorithm), its Cholesky factor and Lambda_v^-1 at every gridpoint.  So TOPPRA, BatchTOPPRA,
BatchTOPPRAsd, feasible, reachable and controllable sets, ragged grids, record chunks and order-k paths take it
unchanged."""
import numpy as np

from .cartesian_velocity_norm import append_sd2_rows, sd2_num_rows, single_path_limit
from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .. import _lib
from ..dynamics import RigidBodyFrame, _is_cuda, _round_trip


class CollisionEnergyConstraint(LinearConstraint):
    """frame: the contact point, a RigidBodyFrame (model.frame(...); its reference frame is ignored); limit: E_max >= 0
    in J, a float or (B,) with one limit per path of the batch; human_mass: m_H > 0 in kg (inf: the robot-only energy
    1/2 m_R |v|^2); discretization_scheme: Collocation (default) or Interpolation.  1 row per stage, 2 with
    Interpolation."""

    def __init__(self, frame, limit, human_mass, discretization_scheme=DiscretizationType.Collocation):
        super(CollisionEnergyConstraint, self).__init__()
        if not isinstance(frame, RigidBodyFrame):
            raise ValueError("CollisionEnergyConstraint needs a RigidBodyFrame (RigidBodyModel.frame(...)) as the "
                             "contact point")
        frame.model._refuse_coupled("CollisionEnergyConstraint")
        self.set_discretization_type(discretization_scheme)
        lim = np.array(limit, dtype=np.float64)
        if lim.ndim > 1:
            raise ValueError("CollisionEnergyConstraint: limit must be a float or (B,); got shape %s" % (lim.shape,))
        if np.isnan(lim).any() or (lim < 0).any():
            raise ValueError("CollisionEnergyConstraint: the energy limit must be >= 0 (not NaN); got %s" % (limit,))
        human_mass = float(human_mass)
        if not human_mass > 0:
            raise ValueError("CollisionEnergyConstraint: human_mass %r must be positive (inf allowed)" % human_mass)
        dead = frame.model.inertialess_joints()
        if dead:
            raise ValueError("CollisionEnergyConstraint: joint(s) %s move no inertia (their bodies and descendants have "
                             "zero mass and inertia), so the mass matrix is singular" % ", ".join(map(repr, dead)))
        self.frame = frame
        self.dof = frame.dof
        self.human_mass = human_mass
        self.limit, self._path_limits = (float(lim), None) if lim.ndim == 0 else (None, lim)
        self.identical = True
        self._format_string = "    Collision energy limit: {:} J, human mass {:} kg\n".format(
            "per path" if self._path_limits is not None else self.limit, human_mass)

    def get_dof(self):
        return self.dof

    def _interp(self):
        return self.discretization_type == DiscretizationType.Interpolation

    def terms(self, q, qs):
        """b of the constraint at (q, qs = q'): CUDA tensors (M, nv) -> (M,), one tbd_collision_energy_terms launch."""
        return self.frame.collision_energy_terms(q, qs, self.human_mass)

    def energy(self, q, qd):
        """E = 1/2 mu |v|^2 at the state (q, qd): CUDA tensors (M, nv) -> (M,), one launch; numpy (nv,) -> float or
        (M, nv) -> (M,), through a device round trip."""
        if _is_cuda(q):
            return self.terms(q, qd)
        E = _round_trip(self.terms, q, qd)
        return float(E) if np.ndim(q) == 1 else E

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
        """One tbd_collision_energy_terms launch for the B x G gridpoints of this context, then the rows a = 0, b,
        c = 0 - limit (F = [1], g = [0]) through tb_rows_canlinear (with the interpolation lift if selected)."""
        append_sd2_rows(self, ctx, self.terms, records, R_total, row0)
