"""Speed and separation monitoring next to people (ISO/TS 15066, 5.5.4): a robot point may move toward a person only
as fast as lets it still stop before contact.  With P robot points (a `toppra_b200.RigidBodyFrame`'s origin and a
radius r_p) and H human spheres (c_h, r_h) in base coordinates, per pair at a gridpoint:

    e = c_h - x_p,  l = |e|,  d = l - r_p - r_h               (surface separation)
    w = e.v1 / l    (the speed toward the sphere at s' = 1, v1 = J_v(q) q'; w = |v1| where l == 0)
    D = d - C - v_h T_r,  k = a_s T_r + v_h
    vmax = 0 if D <= 0 else 2 a_s D / (sqrt(k^2 + 2 a_s D) + k)

vmax is the robot speed v_r that solves the standard's protective separation distance
S_p = v_h (T_r + T_s) + v_r T_r + v_r^2 / (2 a_s) + C = d with the stopping time T_s = v_r / a_s, in a rationalised form
that has no cancellation when a_s T_r is large.  The limit w s' <= vmax only binds where w > 0, as w^2 x <= vmax^2
(x = s'^2), one linear row per pair.  Of those, the pair that minimises vmax^2 / w^2 gives the single row a = 0,
b = w*^2, c = 0 - vmax*^2 (F = [1], g = [0]) of the gridpoint; where no pair approaches, the row is inactive (b = 0,
c = -1).

Every row of the batch (or record chunk) comes from ONE `tbd_separation_terms` launch: one walk of the tree per
gridpoint gives every point, and all P x H pairs are evaluated from it.  The human spheres are shared by the batch,
(H, 4), or given per path, (B, H, 4): one hypothesis of where the person stands for each path, so one path checked
against thousands of hypotheses is one launch.  TOPPRA, BatchTOPPRA, BatchTOPPRAsd, feasible, reachable and
controllable sets, ragged grids, record chunks and order-k paths take it unchanged.

Capsules: a robot entry (frame_a, frame_b, r_p) is the capsule of radius r_p about the segment between the two frame
origins (a link), and human capsules (c0, c1, r_h), (H, 7) or (B, H, 7), are body parts (torso, arms, legs).  Then d
and w are those of the closest pair of every two capsules, the largest w over the pairs where parallel segments have
many (include/toppra_b200_dyn.h).  A problem with a capsule on either side makes one `tbd_capsule_separation_terms`
launch per batch or record chunk, with the spheres of the other side as capsules of zero length (frame_b = frame_a,
c1 = c0); a problem of spheres only keeps `tbd_separation_terms`."""
import numpy as np

from .constraint import DiscretizationType
from .linear_constraint import LinearConstraint, canlinear_colloc_to_interpolate, check_dof
from .. import _lib, engine
from ..dynamics import (CAPSULE_DOUBLES, HUMAN_CAPSULE_DOUBLES, HUMAN_SPHERE_DOUBLES, MAX_HUMANS, _is_cuda,
                        _round_trip, pack_points, sphere_humans_as_capsules, sphere_points_as_capsules)


class SeparationMonitoringConstraint(LinearConstraint):
    """points: a sequence of (RigidBodyFrame, radius >= 0), spheres, or (RigidBodyFrame, RigidBodyFrame, radius >= 0),
    capsules, of one model (1 to 16; the frames' reference frames are ignored); humans: (H, 4) spheres (centre x, y, z,
    radius >= 0) or (H, 7) capsules (c0, c1, radius >= 0) in the model's base coordinates, shared by the batch, or
    (B, H, 4) / (B, H, 7), one set per path (1 <= H <= 16); reaction_time T_r >= 0 (s); stopping_deceleration
    a_s > 0 (m/s^2); human_speed v_h >= 0 (m/s, 1.6 by ISO 13855); clearance C >= 0 (m), the standard's C + Z_d + Z_r;
    discretization_scheme: Collocation (default) or Interpolation.  1 row per stage, 2 with Interpolation."""

    def __init__(self, points, humans, reaction_time, stopping_deceleration, human_speed=1.6, clearance=0.0,
                 discretization_scheme=DiscretizationType.Collocation):
        super(SeparationMonitoringConstraint, self).__init__()
        self.model, self.points = pack_points(points)
        self.set_discretization_type(discretization_scheme)
        hum = np.array(humans, dtype=np.float64)
        if (hum.ndim not in (2, 3) or hum.shape[-1] not in (HUMAN_SPHERE_DOUBLES, HUMAN_CAPSULE_DOUBLES)
                or not 1 <= hum.shape[-2] <= MAX_HUMANS or hum.shape[0] < 1):
            raise ValueError("SeparationMonitoringConstraint: humans must be (H, 4) or (B, H, 4) spheres, or (H, 7) or "
                             "(B, H, 7) capsules, with 1 <= H <= %d; got shape %s" % (MAX_HUMANS, hum.shape))
        if not np.isfinite(hum).all() or (hum[..., -1] < 0).any():
            raise ValueError("SeparationMonitoringConstraint: human spheres and capsules must be finite with radii >= 0")
        params = dict(reaction_time=reaction_time, stopping_deceleration=stopping_deceleration,
                      human_speed=human_speed, clearance=clearance)
        for name, value in params.items():
            value = float(value)
            ok = np.isfinite(value) and (value > 0 if name == "stopping_deceleration" else value >= 0)
            if not ok:
                raise ValueError("SeparationMonitoringConstraint: %s %r must be finite and %s"
                                 % (name, value, "> 0" if name == "stopping_deceleration" else ">= 0"))
            setattr(self, name, value)
        self.capsules = self.points.shape[1] == CAPSULE_DOUBLES or hum.shape[-1] == HUMAN_CAPSULE_DOUBLES
        if self.capsules and self.points.shape[1] != CAPSULE_DOUBLES:
            self.points = sphere_points_as_capsules(self.points)
        if self.capsules and hum.shape[-1] != HUMAN_CAPSULE_DOUBLES:
            hum = sphere_humans_as_capsules(hum)
        self.humans = hum
        self.per_path = hum.ndim == 3
        self.dof = self.model.dof
        self.identical = True
        self._dev_humans = None
        self._format_string = "    Speed and separation monitoring: {:d} {:}, {:d} human {:}{:}\n".format(
            self.points.shape[0], "capsules" if self.capsules else "points", hum.shape[-2],
            "capsules" if self.capsules else "spheres", " per path" if self.per_path else "")

    def get_dof(self):
        return self.dof

    def _interp(self):
        return self.discretization_type == DiscretizationType.Interpolation

    def _humans_on(self, device):
        """The human spheres or capsules as a CUDA tensor (NH, H, 4 or 7) on `device`, copied once per device."""
        torch = _lib.require_cuda()
        if self._dev_humans is None or self._dev_humans.device != torch.device(device):
            self._dev_humans = torch.as_tensor(self.humans.reshape(-1, *self.humans.shape[-2:]), device=device)
        return self._dev_humans

    def terms(self, q, qs, humans=None, points_per_path=0):
        """(b, c) of the constraint at (q, qs = q'): CUDA tensors (M, nv) -> (M,) each, one tbd_separation_terms (or
        tbd_capsule_separation_terms) launch.  humans: a CUDA tensor (NH, H, 4 or 7) read as in
        RigidBodyModel.separation (default: the constraint's)."""
        hum = self._humans_on(q.device) if humans is None else humans
        return self.model.separation_terms(self.points, hum, self.reaction_time, self.stopping_deceleration,
                                           self.human_speed, self.clearance, q, qs, points_per_path)

    def separation(self, q, qd):
        """(d, w): surface separation and approach speed of every point and human sphere at the state (q, qd), each
        (M, P, H).  Shared spheres are read by every point; per-path spheres (B, H, 4) take M = B n points, path-major
        (n points per path).  CUDA tensors (M, nv), one launch; numpy (nv,) -> (P, H) each or (M, nv) -> (M, P, H)
        each, through a device round trip."""
        if not _is_cuda(q):
            out = _round_trip(lambda *x: _stack(self.separation(*x)), q, qd)
            return out[..., 0, :, :], out[..., 1, :, :]
        ppp = 0
        if self.per_path:
            B = self.humans.shape[0]
            if q.shape[0] % B:
                raise ValueError("SeparationMonitoringConstraint.separation: %d points do not split into the %d paths of "
                                 "the per-path human spheres" % (q.shape[0], B))
            ppp = q.shape[0] // B
        return self.model.separation(self.points, self._humans_on(q.device), q, qd, ppp)

    def compute_constraint_params(self, path, gridpoints):
        """The reference's 7-tuple for one path: a = 0, b and c from one launch on q, q' at the gridpoints, F = [1],
        g = [0]."""
        check_dof(self.dof, path.dof)
        if self.per_path and self.humans.shape[0] != 1:
            raise ValueError("SeparationMonitoringConstraint: a single path takes one set of human spheres; got %d"
                             % self.humans.shape[0])
        gridpoints = np.asarray(gridpoints, dtype=float)
        G = gridpoints.shape[0]
        torch = _lib.require_cuda()
        q, qs = (torch.as_tensor(np.atleast_2d(path(gridpoints, o)), device="cuda") for o in (0, 1))
        b, c = (x.cpu().numpy().reshape(G, 1) for x in self.terms(q, qs))
        a = np.zeros((G, 1))
        F, g = np.ones((1, 1)), np.zeros(1)
        if self._interp():
            return canlinear_colloc_to_interpolate(a, b, c, F, g, None, None, gridpoints, identical=True)
        return a, b, c, F, g, None, None

    # ---- device route ------------------------------------------------------------------------------------------
    def num_rows(self, ctx):
        check_dof(self.dof, ctx.bpath.dof)
        if self.per_path and self.humans.shape[0] != ctx.total:
            w = self.humans.shape[-1]
            raise ValueError("SeparationMonitoringConstraint: humans has shape %s; expected (H, %d) or (%d, H, %d)"
                             % (self.humans.shape, w, ctx.total, w))
        return 2 if self._interp() else 1

    def append_records(self, ctx, records, R_total, row0):
        """One tbd_separation_terms (or tbd_capsule_separation_terms) launch for the B x G gridpoints of this context
        (per-path humans sliced to it), then the rows a = 0, b, c (F = [1], g = [0]) through tb_rows_canlinear (with
        the interpolation lift if selected)."""
        self.num_rows(ctx)
        torch = engine.torch_mod()
        bp = ctx.bpath
        B, G, dof = ctx.B, ctx.G, bp.dof
        q = bp.eval_device(ctx.d_grid, 0).reshape(B * G, dof)
        qs = bp.eval_device(ctx.d_grid, 1).reshape(B * G, dof)
        hum = self._humans_on(ctx.device)
        if self.per_path:
            b, c = self.terms(q, qs, hum[ctx.lo:ctx.hi].contiguous(), G)
        else:
            b, c = self.terms(q, qs, hum, 0)
        b, c = b.reshape(B, G, 1), c.reshape(B, G, 1)
        a = torch.zeros_like(b)
        F = engine.as_device(np.ones((1, 1)), ctx.device)
        g = engine.as_device(np.zeros(1), ctx.device)
        engine.rows_canlinear(a, b, c, F, g, 0, ctx.d_grid, self._interp(), records, R_total, row0)


def _stack(dw):
    torch = _lib.require_cuda()
    return torch.stack(dw, dim=1)
