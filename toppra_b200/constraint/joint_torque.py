"""Joint torque constraint — same surface as the reference `toppra/constraint/joint_torque.py:7-116`.

    A(q) qdd + qd^T B(q) qd + C(q) + D(qd) = w,   tau_min <= w <= tau_max
    c = w(q,0,0);  a = w(q,0,q') - c;  b = w(q,q',q'') - c;  c += fs_coef * sign(q')          (:98-108)
    F = [I; -I],  g = [tau_max; -tau_min]  (identical for all gridpoints, :90-96)

`inv_dyn(q, qd, qdd)` is USER code on 1-D numpy arrays, called 3 x (N+1) times on the host exactly like the
reference does; the rows F.a, F.b, F.c - g (and the interpolation lift, linear_constraint.py:84-192) are assembled on
the GPU by the same kernel path as `SecondOrderConstraint.joint_torque_constraint` (csrc/tb_coeff.cu:
tb_rows_canlinear), which produces the same numbers for the same model.

With a `toppra_b200.RigidBodyModel` as `inv_dyn` the device protocol takes the batched route of that delegate: one
fused inverse-dynamics launch for the whole batch (libtoppra_b200_dyn.so), so BatchTOPPRA accepts the constraint."""
import numpy as np

from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .linear_second_order import SecondOrderConstraint


class JointTorqueConstraint(LinearConstraint):
    """inv_dyn: (q, qd, qdd) -> torque; tau_lim (dof, 2); fs_coef (dof,) dry-friction coefficients;
    discretization_scheme: Collocation (default, like the reference) or Interpolation."""

    def __init__(self, inv_dyn, tau_lim, fs_coef, discretization_scheme=DiscretizationType.Collocation):
        super(JointTorqueConstraint, self).__init__()
        self.inv_dyn = inv_dyn
        self.tau_lim = np.array(tau_lim, dtype=float)
        self.fs_coef = np.array(fs_coef)
        self.dof = self.tau_lim.shape[0]
        self.set_discretization_type(discretization_scheme)
        assert self.tau_lim.shape[1] == 2, "Wrong input shape."
        self._format_string = "    Torque limit: \n"
        for i in range(self.tau_lim.shape[0]):
            self._format_string += "      J{:d}: {:}".format(i + 1, self.tau_lim[i]) + "\n"
        self.identical = True
        self._delegate = None

    def compute_constraint_params(self, path, gridpoints):
        """Host 7-tuple (a, b, c, F, g, None, None) with the reference's shapes: collocation (G, dof) / F (2 dof, dof),
        interpolation (G, 2 dof) / F (4 dof, 2 dof); F and g are the same for every gridpoint (`identical`)."""
        n = self.get_dof()
        check_dof(n, path.dof)
        grid = np.asarray(gridpoints)
        q, dq, ddq = (path(grid, order) for order in (0, 1, 2))
        rest = np.zeros(n)
        tau = self.inv_dyn
        gravity = np.array([tau(qi, rest, rest) for qi in q])                    # w(q, 0, 0)
        a = np.array([tau(qi, rest, dqi) for qi, dqi in zip(q, dq)]) - gravity      # A(q) p'
        b = np.array([tau(qi, dqi, ddqi) for qi, dqi, ddqi in zip(q, dq, ddq)]) - gravity
        c = gravity
        for j in range(n):  # dry friction D(qd) = fs * sign(qd), joint by joint like the reference (:106-108)
            c[:, j] += self.fs_coef[j] * np.sign(dq[:, j])
        F = np.concatenate((np.identity(n), -np.identity(n)))
        g = np.concatenate((self.tau_lim[:, 1], -self.tau_lim[:, 0]))
        if self.discretization_type == DiscretizationType.Interpolation:
            return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, grid, identical=True)
        if self.discretization_type == DiscretizationType.Collocation:
            return a, b, c, F, g, None, None
        raise NotImplementedError("Other form of discretization not supported!")

    # ---- device protocol: the rows are those of SecondOrderConstraint.joint_torque_constraint -------------
    def _second_order(self):
        if self._delegate is None or self._delegate.discretization_type != self.discretization_type:
            self._delegate = SecondOrderConstraint.joint_torque_constraint(
                self.inv_dyn, self.tau_lim, self.fs_coef, discretization_scheme=self.discretization_type)
        return self._delegate

    def num_rows(self, ctx):
        return self._second_order().num_rows(ctx)

    def append_records(self, ctx, records, R_total, row0):
        self._second_order().append_records(ctx, records, R_total, row0)
