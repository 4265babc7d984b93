"""Cartesian acceleration limits of a robot frame: the tool must not exceed an acceleration, e.g. so that a payload does
not slip, liquid does not spill or a camera does not blur.  The reference expresses it as a `SecondOrderConstraint`
whose user callback returns the frame's acceleration (`examples-old/cartesian_accel.py`); here the frame comes from a
`toppra_b200.RigidBodyModel` and the accelerations are computed on the GPU.

    acc(q, qd, qdd) = J(q) qdd + dJ(q, qd) qd        (the classical acceleration, no gravity)
    along the path:  acc = acc(q, 0, q') u + acc(q, q', q'') x,   u = s'', x = s'^2,   acc(q, 0, 0) = 0
    lower <= acc[components] <= upper   =>   F = [I_k; -I_k],  g = [upper; -lower],  a, b as above,  c = 0

It is `SecondOrderConstraint`'s eye form with the frame's acceleration as `inv_dyn`: every a and b of the batch (or
record chunk) come from ONE `tbd_acceleration_terms` launch (RigidBodyFrame.acceleration_terms, its `device_terms`),
and the rows go through the same `tb_rows_canlinear` call as joint torque limits.  So TOPPRA, BatchTOPPRA, BatchTOPPRAsd, feasible, reachable and
controllable sets, ragged grids, record chunks and order-k paths take it unchanged."""
import numpy as np

from .constraint import DiscretizationType
from .linear_second_order import SecondOrderConstraint
from .. import engine
from ..dynamics import RigidBodyFrame, component_indices


class CartesianAccelerationConstraint(SecondOrderConstraint):
    """frame: a RigidBodyFrame (model.frame(...), reference frame "local" or "local_world_aligned"); components: indices
    into [ax, ay, az, wx, wy, wz] (default: the linear part); alim: (k, 2) [lower, upper] with row i limiting
    components[i], or (B, k, 2) with one set per path of the batch; discretization_scheme: Interpolation (default, like
    SecondOrderConstraint) or Collocation."""

    def __init__(self, frame, alim, components=(0, 1, 2), discretization_scheme=DiscretizationType.Interpolation):
        if not isinstance(frame, RigidBodyFrame):
            raise ValueError("CartesianAccelerationConstraint needs a RigidBodyFrame (RigidBodyModel.frame(...)); "
                             "for a user callback use SecondOrderConstraint")
        frame._check_acceleration()
        comps = component_indices(components)
        k = len(comps)
        alim = np.array(alim, dtype=np.float64)
        if alim.ndim not in (2, 3) or alim.shape[-2:] != (k, 2):
            raise ValueError("CartesianAccelerationConstraint: alim has shape %s; expected (%d, 2) or (B, %d, 2) for "
                             "components %s" % (alim.shape, k, k, tuple(components)))
        if not np.isfinite(alim).all():
            raise ValueError("CartesianAccelerationConstraint: limits must be finite")
        if (alim[..., 0] > alim[..., 1]).any():
            raise ValueError("CartesianAccelerationConstraint: a lower limit exceeds its upper limit")
        # row i of alim belongs to components[i]; the kernel's columns come in increasing component order
        alim = alim[..., np.argsort(np.asarray(components).reshape(-1), kind="stable"), :]
        eyes = np.vstack((np.eye(k), -np.eye(k)))
        g_aug = np.concatenate((alim[..., 1], -alim[..., 0]), axis=-1)
        g_single = g_aug if g_aug.ndim == 1 else g_aug[0]
        super(CartesianAccelerationConstraint, self).__init__(frame.acceleration, lambda _: eyes, lambda _: g_single,
                                                              frame.dof, discretization_scheme=discretization_scheme,
                                                              batched=True)
        self._eye_form = (g_aug, np.zeros(k))
        self.device_terms = self._terms
        self.frame = frame
        self.components = tuple(comps)
        self.limits = alim          # not `alim`: BatchTOPPRA checks attributes of that name against the path's dof
        self._format_string = "    Kind: Cartesian acceleration limit of frame %r, components %s\n" % (
            frame.name, self.components)

    def _terms(self, q, qs, qss):
        """acc(q, 0, 0) = 0: c = 0, and a, b need no subtraction."""
        a, b = self.frame.acceleration_terms(q, qs, qss, self.components)
        return a, b, engine.torch_mod().zeros_like(a)

    def _check_batch(self, ctx):
        super(CartesianAccelerationConstraint, self)._check_batch(ctx)
        if self.limits.ndim == 3 and self.limits.shape[0] != ctx.total:
            raise ValueError("CartesianAccelerationConstraint: alim has shape %s; expected (%d, 2) or (%d, %d, 2)"
                             % (self.limits.shape, len(self.components), ctx.total, len(self.components)))
