"""Contact stability of an object carried on a robot's tool without being gripped ("waiter motion"): a box on a tray, a
glass on a plate.  The object must not slide, tip over or twist on its rectangular support.  The reference expresses it
as a `SecondOrderConstraint` whose user callback returns the contact wrench; here the contact frame comes from a
`toppra_b200.RigidBodyModel` and the wrenches are computed on the GPU.

The contact frame (a RigidBodyFrame) has its origin at the centre of the contact rectangle, of half-lengths X, Y along
its x and y axes, and its z axis along the support normal, pointing into the object.  The object has mass m, centre of
mass r and rotational inertia Ic about it, in contact-frame coordinates.  In contact-frame axes, with g_l = R_f^T g:

    f = m (a_r - g_l),   tau = Ic dw + w x (Ic w) + r x f,   w(q, qd, qdd) = [f; tau]    (at the contact origin)
    along the path:  c = w(q, 0, 0),  a = w(q, 0, q') - c,  b = w(q, q', q'') - c,   F (a u + b x + c) <= 0

F (16 x 6) is the contact wrench cone of the rectangle with friction coefficient mu (Caron, Pham, Nakamura, "Stability
of surface contacts for humanoid robots: closed-form formulae of the contact wrench cone for rectangular support
areas", ICRA 2015): the wrenches that are the sum, taken at the centre, of four corner forces each inside its friction
pyramid.  Every a, b and c of the batch (or record chunk) come from ONE `tbd_contact_wrench_terms` launch (the
constraint's `device_terms`), and the rows go through `tb_rows_canlinear` with the shared F and g = 0 (the constant-F
form of `SecondOrderConstraint`).  So TOPPRA, BatchTOPPRA, BatchTOPPRAsd, feasible, reachable
and controllable sets, ragged grids, record chunks and order-k paths take it unchanged."""
import numpy as np

from .constraint import DiscretizationType
from .linear_second_order import SecondOrderConstraint
from ..dynamics import RigidBodyFrame, _packed_object, _rigid_inertia

NUM_ROWS = 16


def contact_wrench_cone(half_lengths, friction):
    """F (16, 6): the wrench w = [f; tau] at the centre of a rectangle of half-lengths (X, Y) with friction coefficient
    mu is the sum of four corner forces inside their friction pyramids iff F w <= 0.  Rows, in order:
      sliding   +-f_x - mu f_z,  +-f_y - mu f_z;
      tipping   +-tau_x - Y f_z,  +-tau_y - X f_z  (the centre of pressure inside the rectangle);
      twisting  s1 (Y f_x - mu tau_x) + s2 (X f_y - mu tau_y) - mu (X + Y) f_z - tau_z  (lower bound on tau_z) and
                s1 (Y f_x + mu tau_x) + s2 (X f_y + mu tau_y) - mu (X + Y) f_z + tau_z  (upper bound), each for
                (s1, s2) = (+, +), (+, -), (-, +), (-, -)."""
    X, Y = half_lengths_of(half_lengths)
    mu = friction_of(friction)
    F = []
    for s in (1.0, -1.0):
        F.append([s, 0.0, -mu, 0.0, 0.0, 0.0])
    for s in (1.0, -1.0):
        F.append([0.0, s, -mu, 0.0, 0.0, 0.0])
    for s in (1.0, -1.0):
        F.append([0.0, 0.0, -Y, s, 0.0, 0.0])
    for s in (1.0, -1.0):
        F.append([0.0, 0.0, -X, 0.0, s, 0.0])
    signs = ((1.0, 1.0), (1.0, -1.0), (-1.0, 1.0), (-1.0, -1.0))
    for t in (-1.0, 1.0):                       # lower bound on tau_z (t = -1), then upper bound (t = +1)
        for s1, s2 in signs:
            F.append([s1 * Y, s2 * X, -mu * (X + Y), t * s1 * mu, t * s2 * mu, t])
    return np.array(F, dtype=np.float64)


def half_lengths_of(half_lengths):
    """(X, Y) of a rectangle around the origin, or ValueError: both finite and positive."""
    hl = np.asarray(half_lengths, dtype=np.float64)
    if hl.shape != (2,):
        raise ValueError("half_lengths must be (X, Y); got shape %s" % (hl.shape,))
    if not np.isfinite(hl).all():
        raise ValueError("half_lengths must be finite")
    if not (hl > 0).all():
        raise ValueError("half_lengths must be positive; got %s" % hl)
    return float(hl[0]), float(hl[1])


def friction_of(friction):
    """A friction coefficient, or ValueError: a finite, positive scalar."""
    mu = np.asarray(friction, dtype=np.float64)
    if mu.shape != ():
        raise ValueError("friction must be a scalar; got shape %s" % (mu.shape,))
    if not np.isfinite(mu):
        raise ValueError("friction must be finite")
    if not mu > 0:
        raise ValueError("friction %r must be positive" % float(mu))
    return float(mu)


class ContactStabilityConstraint(SecondOrderConstraint):
    """frame: the contact frame, a RigidBodyFrame (model.frame(...); its reference frame is ignored, the wrench is in
    the frame's own axes); mass > 0; com (3,) and inertia (6,) = Ixx, Ixy, Ixz, Iyy, Iyz, Izz about the centre of mass
    (positive semi-definite), both in contact-frame coordinates; half_lengths (X, Y) > 0 of the contact rectangle;
    friction mu > 0; discretization_scheme: Interpolation (default, like SecondOrderConstraint) or Collocation.
    16 rows per stage, 32 with Interpolation."""

    def __init__(self, frame, mass, com, inertia, half_lengths, friction,
                 discretization_scheme=DiscretizationType.Interpolation):
        if not isinstance(frame, RigidBodyFrame):
            raise ValueError("ContactStabilityConstraint needs a RigidBodyFrame (RigidBodyModel.frame(...)) as the "
                             "contact frame; for a user callback use SecondOrderConstraint")
        mass, com, _ = _rigid_inertia("ContactStabilityConstraint", mass, com, inertia)
        F = contact_wrench_cone(half_lengths, friction)
        zeros = np.zeros(NUM_ROWS)
        super(ContactStabilityConstraint, self).__init__(self.wrench, lambda _: F, lambda _: zeros, frame.dof,
                                                         discretization_scheme=discretization_scheme, batched=True)
        self.frame = frame
        self.F = self._const_F = F
        self.object = _packed_object(np.concatenate(([mass], com, np.asarray(inertia, dtype=np.float64))))
        self.device_terms = lambda q, qs, qss: frame.contact_wrench_terms(self.object, q, qs, qss)
        self.half_lengths = tuple(float(x) for x in np.asarray(half_lengths, dtype=np.float64))
        self.friction = float(friction)
        self._format_string = "    Kind: contact stability of an object on frame %r, %d rows\n" % (frame.name, NUM_ROWS)

    def wrench(self, q, qd, qdd):
        """The contact wrench [f; tau] (frame axes, at the contact origin).  CUDA tensors (M, nv) -> (M, 6), one
        tbd_contact_wrench launch; numpy (nv,) -> (6,) through a device round trip: a reference-style `inv_dyn`."""
        return self.frame.contact_wrench(self.object, q, qd, qdd)
