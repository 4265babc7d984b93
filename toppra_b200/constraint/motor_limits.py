"""Torque and speed limits of geared robots on the motor side.  A data sheet gives a peak torque and a maximum speed per
motor; each motor drives its joint through a gear ratio, and coupled wrist motors turn several joints.  With the
transmission theta = T q of `toppra_b200.Drives`:

    motor torques   w(q, qd, qdd) = T^-T ID(q, qd, qdd) + I_r o (T qdd),   c += f o sign(T q')
    motor speeds    |(T q')_i s'| <= omega_i  <=>  x ((T q')_i / omega_i)^2 <= 1   (x = s'^2)

Both are linear in (u, x), so they are exact TOPP-RA rows.  `MotorTorqueConstraint` is `SecondOrderConstraint`'s eye
form with the motor torques as `inv_dyn`: the three terms of every gridpoint of the batch (or record chunk) come from
ONE `tbd_drive_torque_terms` launch.  `MotorSpeedConstraint` is one row per gridpoint, a = 0, b = max_i ((T q')_i /
omega_i)^2, c = -1, with the feasible set of the nv rows, from ONE `tbd_drive_speed_terms` launch.  So TOPPRA,
BatchTOPPRA, BatchTOPPRAsd, ragged grids, record chunks and order-k paths take them unchanged."""
import numpy as np

from .cartesian_velocity_norm import append_sd2_rows, sd2_num_rows
from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint
from .linear_second_order import SecondOrderConstraint
from ..dynamics import Drives


def _check_drives(what, drives):
    if not isinstance(drives, Drives):
        raise ValueError("%s needs a toppra_b200.Drives" % what)


class MotorTorqueConstraint(SecondOrderConstraint):
    """drives: a Drives; torque_limits: (nv, 2) [lower, upper] motor torques, or (B, nv, 2) with one set per path of the
    batch; discretization_scheme: Interpolation (default, like SecondOrderConstraint) or Collocation."""

    def __init__(self, drives, torque_limits, discretization_scheme=DiscretizationType.Interpolation):
        _check_drives("MotorTorqueConstraint", drives)
        nv = drives.nv
        tl = np.array(torque_limits, dtype=np.float64)
        if tl.ndim not in (2, 3) or tl.shape[-2:] != (nv, 2):
            raise ValueError("MotorTorqueConstraint: torque_limits has shape %s; expected (%d, 2) or (B, %d, 2)"
                             % (tl.shape, nv, nv))
        eyes = np.vstack((np.eye(nv), -np.eye(nv)))
        g_aug = np.concatenate((tl[..., 1], -tl[..., 0]), axis=-1)
        g_single = g_aug if g_aug.ndim == 1 else g_aug[0]
        super(MotorTorqueConstraint, self).__init__(drives.torque, lambda _: eyes, lambda _: g_single, nv,
                                                    discretization_scheme=discretization_scheme, batched=True)
        self._eye_form = (g_aug, np.zeros(nv))    # the motor friction is in the terms: f o sign(T q')
        self.device_terms = drives.torque_terms
        self.drives = drives
        self.torque_limits = tl
        self._format_string = "    Kind: Motor torque limit\n"

    def _check_batch(self, ctx):
        super(MotorTorqueConstraint, self)._check_batch(ctx)
        if self.torque_limits.ndim == 3 and self.torque_limits.shape[0] != ctx.total:
            raise ValueError("MotorTorqueConstraint: torque_limits has shape %s; expected (%d, 2) or (%d, %d, 2)"
                             % (self.torque_limits.shape, self.dof, ctx.total, self.dof))


class MotorSpeedConstraint(LinearConstraint):
    """drives: a Drives; speed_limit: (nv,) motor speeds omega_i > 0 in rad/s (inf: no limit); discretization_scheme:
    Collocation (default) or Interpolation.  1 row per stage, 2 with Interpolation."""

    def __init__(self, drives, speed_limit, discretization_scheme=DiscretizationType.Collocation):
        super(MotorSpeedConstraint, self).__init__()
        _check_drives("MotorSpeedConstraint", drives)
        omega = np.array(speed_limit, dtype=np.float64)
        if omega.shape != (drives.nv,):
            raise ValueError("MotorSpeedConstraint: speed_limit has shape %s; expected (%d,)"
                             % (omega.shape, drives.nv))
        self.set_discretization_type(discretization_scheme)
        self.drives = drives
        self.dof = drives.nv
        self.speed_limit = omega
        self.limit, self._path_limits = 1.0, None     # the row b x <= 1 of append_sd2_rows
        self.identical = True
        self._format_string = "    Motor speed limit: {:}\n".format(omega)

    def get_dof(self):
        return self.dof

    def _interp(self):
        return self.discretization_type == DiscretizationType.Interpolation

    def terms(self, q, qs):
        """b of the constraint at qs = q': CUDA tensors (M, nv) -> (M,), one tbd_drive_speed_terms launch."""
        return self.drives.speed_terms(qs, self.speed_limit)

    def num_rows(self, ctx):
        return sd2_num_rows(self, ctx)

    def append_records(self, ctx, records, R_total, row0):
        """One tbd_drive_speed_terms launch for the B x G gridpoints of this context, then the rows a = 0, b, c = -1
        (F = [1], g = [0]) through tb_rows_canlinear (with the interpolation lift if selected)."""
        append_sd2_rows(self, ctx, self.terms, records, R_total, row0)
