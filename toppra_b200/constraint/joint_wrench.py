"""Bearing and reducer loads of a robot joint: the force and moment that a joint passes from its parent to everything
beyond it must stay within what its bearing, reducer or actuator module is rated for.  Data sheets rate more than the
torque about the joint axis: cross-roller bearings and reducers give an allowable axial force, radial force and
tilting moment, actuator modules a maximum axial force and bending moment, heavy-payload wrists permitted load moments.
Fast motions with a heavy tool break these limits well before they break the torque limits.  The reference expresses
such a limit as a `SecondOrderConstraint` whose user callback returns the wrench; here the robot is a
`toppra_b200.RigidBodyModel` and the wrenches are computed on the GPU.

For a frame on body k (a RigidBodyFrame), the joint wrench w = [f; n] is the wrench the parent side of joint k exerts
on k's subtree (body k, the bodies below it, the links folded into them and a payload from `with_payload`), gravity
included, the moment about the frame origin, in the frame's axes ("local") or world axes ("local_world_aligned"):

    w(q, qd, qdd) = the recursive Newton-Euler force of body k, moved to the frame    (RigidBodyFrame.joint_wrench)
    along the path:  c = w(q, 0, 0),  a = w(q, 0, q') - c,  b = w(q, q', q'') - c,   F (a u + b x + c) <= g

Two forms:
  JointWrenchConstraint(frame, wlim, components)  lower <= w[components] <= upper: `SecondOrderConstraint`'s eye form
                                                  (F = [I; -I]), limits shared or one set per path;
  JointWrenchConstraint.bearing(frame, axial, radial, tilting)
                                                  |f.a| <= axial, |f - (f.a) a| <= radial, |n - (n.a) a| <= tilting
                                                  with a the joint axis: constant rows on all six components.
Every a, b and c of the batch (or record chunk) come from ONE `tbd_joint_wrench_terms` launch (the constraint's
`device_terms`) and the rows go through `tb_rows_canlinear`.  So TOPPRA, BatchTOPPRA, BatchTOPPRAsd, feasible,
reachable and controllable sets, ragged grids, record chunks and order-k paths take it unchanged.

Row budget: a problem holds at most 126 rows (R <= 126).  The box form costs 2 k rows (4 k under Interpolation), a
bearing constraint 2 + sides per radial or tilting limit (with sides = 8 and all three limits: 18 rows, 36 under
Interpolation)."""
import numpy as np

from .constraint import DiscretizationType
from .linear_second_order import SecondOrderConstraint
from ..dynamics import WRENCH_COMPONENTS, RigidBodyFrame, component_indices

ALL_COMPONENTS = (0, 1, 2, 3, 4, 5)


def _check_frame(what, frame):
    if not isinstance(frame, RigidBodyFrame):
        raise ValueError("%s needs a RigidBodyFrame (RigidBodyModel.frame(...)) on the joint's body; for a user "
                         "callback use SecondOrderConstraint" % what)
    frame._check_joint_wrench()


def polygon_rows(axis, sides):
    """(sides, 3) unit normals d_j of the regular polygon inscribed in the unit circle of the plane normal to the unit
    vector `axis`: x . d_j <= cos(pi / sides) for every j keeps the component of x in that plane inside the polygon,
    so within the circle, and every x whose component there is within cos(pi / sides) satisfies them."""
    a = np.asarray(axis, dtype=np.float64)
    e = np.eye(3)[int(np.argmin(np.abs(a)))]          # the basis vector least aligned with the axis
    u = e - np.dot(e, a) * a
    u = u / np.linalg.norm(u)
    v = np.cross(a, u)
    t = 2.0 * np.pi * np.arange(sides) / sides
    return np.cos(t)[:, None] * u[None] + np.sin(t)[:, None] * v[None]


def bearing_rows(axis, axial=None, radial=None, tilting=None, sides=8):
    """(F (r, 6), g (r,)) on w = [f; n] with the unit joint axis `axis` in the same axes:
      axial    2 rows      [+-a, 0] w <= axial
      radial   sides rows  [d_j, 0] w <= radial cos(pi / sides)
      tilting  sides rows  [0, d_j] w <= tilting cos(pi / sides)
    d_j from polygon_rows.  Each norm limit L uses the regular polygon inscribed in the circle of radius L: every
    wrench within the rows has a radial force (tilting moment) of at most L, and every one of at most L cos(pi / sides)
    is within them."""
    a = np.asarray(axis, dtype=np.float64)
    F, g = [], []
    if axial is not None:
        F += [np.r_[a, 0.0, 0.0, 0.0], np.r_[-a, 0.0, 0.0, 0.0]]
        g += [axial, axial]
    d = polygon_rows(a, sides)
    inner = np.cos(np.pi / sides)
    if radial is not None:
        F += [np.r_[dj, 0.0, 0.0, 0.0] for dj in d]
        g += [radial * inner] * sides
    if tilting is not None:
        F += [np.r_[0.0, 0.0, 0.0, dj] for dj in d]
        g += [tilting * inner] * sides
    return np.array(F), np.array(g, dtype=np.float64)


class JointWrenchConstraint(SecondOrderConstraint):
    """frame: a RigidBodyFrame on the joint's body (model.frame(...), reference frame "local" or
    "local_world_aligned"; not on the base); components: indices into [fx, fy, fz, nx, ny, nz] (default: all six);
    wlim: (k, 2) [lower, upper] with row i limiting components[i], or (B, k, 2) with one set per path of the batch;
    discretization_scheme: Interpolation (default, like SecondOrderConstraint) or Collocation.  See `bearing` for the
    data-sheet limits of a bearing."""

    def __init__(self, frame, wlim, components=ALL_COMPONENTS, discretization_scheme=DiscretizationType.Interpolation):
        _check_frame("JointWrenchConstraint", frame)
        comps = component_indices(components, WRENCH_COMPONENTS)
        k = len(comps)
        wlim = np.array(wlim, dtype=np.float64)
        if wlim.ndim not in (2, 3) or wlim.shape[-2:] != (k, 2):
            raise ValueError("JointWrenchConstraint: wlim has shape %s; expected (%d, 2) or (B, %d, 2) for components "
                             "%s" % (wlim.shape, k, k, tuple(components)))
        if not np.isfinite(wlim).all():
            raise ValueError("JointWrenchConstraint: limits must be finite")
        if (wlim[..., 0] > wlim[..., 1]).any():
            raise ValueError("JointWrenchConstraint: a lower limit exceeds its upper limit")
        # row i of wlim belongs to components[i]; the kernel's columns come in increasing component order
        wlim = wlim[..., np.argsort(np.asarray(components).reshape(-1), kind="stable"), :]
        eyes = np.vstack((np.eye(k), -np.eye(k)))
        g_aug = np.concatenate((wlim[..., 1], -wlim[..., 0]), axis=-1)
        g_single = g_aug if g_aug.ndim == 1 else g_aug[0]
        super(JointWrenchConstraint, self).__init__(self._selected, lambda _: eyes, lambda _: g_single, frame.dof,
                                                    discretization_scheme=discretization_scheme, batched=True)
        self._eye_form = (g_aug, np.zeros(k))
        self.frame = frame
        self.components = tuple(comps)
        self.limits = wlim          # not `alim`: BatchTOPPRA checks attributes of that name against the path's dof
        self.device_terms = lambda q, qs, qss: frame.joint_wrench_terms(q, qs, qss, self.components)
        self._format_string = "    Kind: joint wrench limit of frame %r, components %s\n" % (frame.name,
                                                                                               self.components)

    @classmethod
    def bearing(cls, frame, axial=None, radial=None, tilting=None, sides=8,
                discretization_scheme=DiscretizationType.Interpolation):
        """Data-sheet limits of the bearing (reducer, actuator module) of the joint of `frame`'s body, relative to that
        joint's axis a: |f.a| <= axial, |f - (f.a) a| <= radial and |n - (n.a) a| <= tilting (the tilting or bending
        moment about the frame origin, which should lie at the bearing's rating point).  Give at least one limit, each
        finite and > 0; sides >= 4 is the number of half-planes per norm limit (bearing_rows: conservative by at most a
        factor cos(pi / sides)).  The frame must be "local": the rows are constant in its axes."""
        _check_frame("JointWrenchConstraint.bearing", frame)
        if frame.reference_frame != "local":
            raise ValueError("JointWrenchConstraint.bearing: frame %r has reference frame %r; the bearing rows are "
                             "constant only in the frame's own axes (\"local\")" % (frame.name, frame.reference_frame))
        limits = {"axial": axial, "radial": radial, "tilting": tilting}
        if all(v is None for v in limits.values()):
            raise ValueError("JointWrenchConstraint.bearing: give at least one of axial, radial and tilting")
        for name, v in limits.items():
            if v is not None and not (np.ndim(v) == 0 and np.isfinite(v) and v > 0):
                raise ValueError("JointWrenchConstraint.bearing: %s limit %r must be a finite number > 0" % (name, v))
        if not (isinstance(sides, (int, np.integer)) and sides >= 4):
            raise ValueError("JointWrenchConstraint.bearing: sides %r must be an integer >= 4" % (sides,))
        axis = frame.R.T @ frame.model.body(frame.body)[2:5]  # the joint axis in body k's coordinates, in frame axes
        F, g = bearing_rows(axis, *(None if v is None else float(v) for v in limits.values()), sides=int(sides))
        obj = cls.__new__(cls)
        SecondOrderConstraint.__init__(obj, frame.joint_wrench, lambda _: F, lambda _: g, frame.dof,
                                       discretization_scheme=discretization_scheme, batched=True)
        obj._const_F, obj._const_g = F, g
        obj.F, obj.g = F, g
        obj.frame = frame
        obj.components = ALL_COMPONENTS
        obj.limits = None
        obj.axis = axis
        obj.bearing_limits = {k: None if v is None else float(v) for k, v in limits.items()}
        obj.sides = int(sides)
        obj.device_terms = lambda q, qs, qss: frame.joint_wrench_terms(q, qs, qss)
        obj._format_string = "    Kind: bearing limits of the joint of frame %r, %d rows\n" % (frame.name, F.shape[0])
        return obj

    def wrench(self, q, qd, qdd):
        """The joint wrench [fx, fy, fz, nx, ny, nz] (RigidBodyFrame.joint_wrench): CUDA tensors (M, nv) -> (M, 6), one
        tbd_joint_wrench launch; numpy (nv,) -> (6,) through a device round trip: a reference-style `inv_dyn`."""
        return self.frame.joint_wrench(q, qd, qdd)

    def _selected(self, q, qd, qdd):
        """The limited components of the joint wrench, in increasing index order: the `inv_dyn` of the box form."""
        return self.wrench(q, qd, qdd)[..., list(self.components)]

    def _check_batch(self, ctx):
        super(JointWrenchConstraint, self)._check_batch(ctx)
        if self.limits is not None and self.limits.ndim == 3 and self.limits.shape[0] != ctx.total:
            raise ValueError("JointWrenchConstraint: wlim has shape %s; expected (%d, 2) or (%d, %d, 2)"
                             % (self.limits.shape, len(self.components), ctx.total, len(self.components)))
