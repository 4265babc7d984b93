"""Support stability of the whole robot: a robot standing on a support it is not bolted to (an arm on a parked mobile
base or a light cart, on a table that is not fixed, a legged robot rooted at its stance foot) must not tip over, slide
or twist on it.  Fast arm motions move the zero-moment point (ZMP, the centre of pressure on the ground) out of the
footprint.  The reference expresses it as a `SecondOrderConstraint` whose user callback returns the ground reaction
wrench; here the robot is a `toppra_b200.RigidBodyModel` and the wrenches are computed on the GPU.

The support frame (a RigidBodyFrame on the base) has its origin on the support plane and its z axis along the support
normal, pointing into the robot.  In support axes, at the support origin, the support exerts on the robot

    w(q, qd, qdd) = [f; tau]:  the recursive Newton-Euler wrench of the whole moving tree (gravity included) plus the
                              weight of the static base (base_mass, base_com)
    along the path:  c = w(q, 0, 0),  a = w(q, 0, q') - c,  b = w(q, q', q'') - c,   F (a u + b x + c) <= 0

and the ZMP is (-tau_y / f_z, tau_x / f_z).  F is either the contact wrench cone of a rectangular footprint with
friction (`contact_wrench_cone`: sliding, tipping and twisting; Caron, Pham, Nakamura, ICRA 2015) or the rows of a
convex footprint polygon (`support_polygon_rows`: one ZMP row per edge, plus four sliding rows with friction).  Every
a, b and c of the batch (or record chunk) come from ONE `tbd_support_wrench_terms` launch (the constraint's
`device_terms`), and the rows go through `tb_rows_canlinear` with the shared F and g = 0 (the constant-F form of
`SecondOrderConstraint`).  So TOPPRA, BatchTOPPRA, BatchTOPPRAsd, feasible, reachable and
controllable sets, ragged grids, record chunks and order-k paths take it unchanged."""
import numpy as np

from .constraint import DiscretizationType
from .contact_stability import contact_wrench_cone, friction_of, half_lengths_of
from .linear_second_order import SecondOrderConstraint
from ..dynamics import RigidBodyFrame, _base_inertia


def _polygon(vertices):
    """(n, 2) float64 vertices of a convex, counter-clockwise polygon (seen from +z), or ValueError."""
    v = np.asarray(vertices, dtype=np.float64)
    if v.ndim != 2 or v.shape[1] != 2 or v.shape[0] < 3:
        raise ValueError("support polygon: expected (n, 2) vertices with n >= 3; got shape %s" % (v.shape,))
    if not np.isfinite(v).all():
        raise ValueError("support polygon: the vertices must be finite")
    e = np.roll(v, -1, axis=0) - v
    length = np.hypot(e[:, 0], e[:, 1])
    scale = np.abs(v - v.mean(axis=0)).max()
    if not scale > 0 or (length <= 1e-12 * scale).any():
        raise ValueError("support polygon: degenerate (repeated vertices or zero size)")
    en = np.roll(e, -1, axis=0)
    turn = e[:, 0] * en[:, 1] - e[:, 1] * en[:, 0]                       # |e_i| |e_i+1| sin(angle at vertex i + 1)
    if (np.abs(turn) <= 1e-12 * length * np.roll(length, -1)).any():
        raise ValueError("support polygon: degenerate (three collinear vertices)")
    if (turn < 0).all():
        raise ValueError("support polygon: the vertices are clockwise; give them counter-clockwise seen from +z")
    angles = np.arctan2(turn, (e * en).sum(axis=1))
    if (turn < 0).any() or abs(angles.sum() - 2 * np.pi) > 1e-6:
        raise ValueError("support polygon: not convex")
    return v


def support_polygon_rows(vertices, friction=None):
    """F (n or n + 4, 6): rows on the wrench w = [f; tau] at the support origin (support axes) that keep the centre of
    pressure (-tau_y / f_z, tau_x / f_z) inside the convex polygon `vertices` ((n, 2), counter-clockwise seen from +z,
    the origin need not be inside) iff F w <= 0.  For edge e = v[i+1] - v[i] the row is
    [0, 0, -(e_y v_ix - e_x v_iy), -e_x, -e_y, 0] / |e|: the centre of pressure on the inner side of that edge.  No
    separate f_z >= 0 row is needed: sum_i |e_i| row_i = [0, 0, -2 Area, 0, 0, 0].  With `friction` mu the four sliding
    rows +-f_x - mu f_z, +-f_y - mu f_z follow; a polygon gets no twisting rows (contact_wrench_cone has them for a
    rectangle)."""
    v = _polygon(vertices)
    e = np.roll(v, -1, axis=0) - v
    F = np.zeros((v.shape[0], 6))
    F[:, 2] = -(e[:, 1] * v[:, 0] - e[:, 0] * v[:, 1])
    F[:, 3] = -e[:, 0]
    F[:, 4] = -e[:, 1]
    F = F / np.hypot(e[:, 0], e[:, 1])[:, None]
    if friction is not None:
        mu = friction_of(friction)
        F = np.vstack((F, [[1.0, 0.0, -mu, 0.0, 0.0, 0.0], [-1.0, 0.0, -mu, 0.0, 0.0, 0.0],
                           [0.0, 1.0, -mu, 0.0, 0.0, 0.0], [0.0, -1.0, -mu, 0.0, 0.0, 0.0]]))
    return F


class SupportStabilityConstraint(SecondOrderConstraint):
    """support: the support frame, a RigidBodyFrame on the base (model.frame("base_footprint"), body -1; its reference
    frame is ignored, the wrench is in the frame's own axes).  The footprint is exactly one of
      half_lengths (X, Y) > 0: the rectangle [-X, X] x [-Y, Y] around the support origin; with `friction` its contact
                               wrench cone (16 rows: sliding, tipping, twisting), without it its four ZMP rows;
      polygon (n, 2), n >= 3:  a convex polygon in support axes, counter-clockwise seen from +z (support_polygon_rows:
                               one ZMP row per edge, and with `friction` four sliding rows; no twisting rows).
    friction mu > 0 or None; base_mass >= 0 and base_com (3,) (base coordinates) of the static base, by default the
    model's (RigidBodyModel.base_mass / base_com, which from_urdf takes from the root link and the links fixed or locked
    to it); discretization_scheme: Interpolation (default, like SecondOrderConstraint) or Collocation."""

    def __init__(self, support, half_lengths=None, polygon=None, friction=None, base_mass=None, base_com=None,
                 discretization_scheme=DiscretizationType.Interpolation):
        if not isinstance(support, RigidBodyFrame):
            raise ValueError("SupportStabilityConstraint needs a RigidBodyFrame on the base (RigidBodyModel.frame(...)) "
                             "as the support frame; for a user callback use SecondOrderConstraint")
        if support.body != -1:
            raise ValueError("SupportStabilityConstraint: the support must be on the base; frame %r is on body %d"
                             % (support.name, support.body))
        if (half_lengths is None) == (polygon is None):
            raise ValueError("SupportStabilityConstraint: give exactly one of half_lengths and polygon")
        model = support.model
        mass, com = _base_inertia("SupportStabilityConstraint",
                                  model.base_mass if base_mass is None else base_mass,
                                  model.base_com if base_com is None else base_com)
        if half_lengths is not None:
            X, Y = half_lengths_of(half_lengths)
            if friction is not None:
                F = contact_wrench_cone((X, Y), friction)
            else:
                F = support_polygon_rows([[-X, -Y], [X, -Y], [X, Y], [-X, Y]])
            self.half_lengths, self.polygon = (X, Y), None
        else:
            F = support_polygon_rows(polygon, friction)
            self.half_lengths, self.polygon = None, _polygon(polygon).copy()
        zeros = np.zeros(F.shape[0])
        super(SupportStabilityConstraint, self).__init__(self.wrench, lambda _: F, lambda _: zeros, support.dof,
                                                         discretization_scheme=discretization_scheme, batched=True)
        self.support = support
        self.F = self._const_F = F
        self.friction = None if friction is None else float(friction)
        self.base = np.concatenate(([mass], com))
        self.device_terms = lambda q, qs, qss: support.support_wrench_terms(self.base, q, qs, qss)
        self._format_string = "    Kind: support stability on frame %r, %d rows\n" % (support.name, F.shape[0])

    def wrench(self, q, qd, qdd):
        """The support wrench [f; tau] (support axes, at the support origin).  CUDA tensors (M, nv) -> (M, 6), one
        tbd_support_wrench launch; numpy (nv,) -> (6,) through a device round trip: a reference-style `inv_dyn`."""
        return self.support.support_wrench(self.base, q, qd, qdd)

    def zmp(self, q, qd, qdd):
        """The zero-moment point (centre of pressure) (-tau_y / f_z, tau_x / f_z) in support axes: (..., 2), like
        `wrench`."""
        w = self.wrench(q, qd, qdd)
        x, y = -w[..., 4] / w[..., 2], w[..., 3] / w[..., 2]
        if isinstance(w, np.ndarray):
            return np.stack((x, y), axis=-1)
        import torch
        return torch.stack((x, y), dim=-1)
