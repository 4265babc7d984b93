"""Rigid-body models of fixed-base robots for joint-torque constraints: `RigidBodyModel` (per-body arrays or a URDF file)
whose inverse dynamics run on the GPU (libtoppra_b200_dyn.so, Featherstone's recursive Newton-Euler algorithm).

    model = RigidBodyModel.from_urdf("arm.urdf")
    tau = model(q, qd, qdd)                                  # CUDA tensors (M, nv): one kernel launch
    pc = JointTorqueConstraint(model, model.torque_limits(), friction)

A `RigidBodyModel` is a valid `inv_dyn` for `JointTorqueConstraint` and `SecondOrderConstraint.joint_torque_constraint`;
there it takes the device route: the three inverse-dynamics terms of every gridpoint of the batch come from ONE fused
launch (`torque_terms`).  The packed layout the library takes is documented in include/toppra_b200_dyn.h.

    tcp = model.frame("flange", xyz=(0, 0, 0.1))              # a RigidBodyFrame: the tool-centre point
    v = tcp(q, qd)                                            # (M, 6) frame velocities, one kernel launch
    pc = CartesianVelocityNorm(tcp, S, limit)                 # tool-speed limit, batched on the device
    acc = tcp.acceleration(q, qd, qdd)                        # (M, 6) classical frame accelerations, one launch
    pc = CartesianAccelerationConstraint(tcp, alim)           # tool-acceleration limit, batched on the device
    pc = ContactStabilityConstraint(tray, m, com, I, (X, Y), mu)  # an object carried on a tray must not slide or tip
    Linv = tcp.inverse_inertia(q)                             # (M, 3, 3) J_v M(q)^-1 J_v^T, one launch
    pc = CollisionEnergyConstraint(tcp, E_max, m_H)           # collision energy next to people (ISO/TS 15066)
    loaded = model.with_payload("flange", m, com, I)          # a rigidly held payload folded into the flange's body
    floor = model.frame("base_footprint")                     # a support frame on the base (z: the support normal)
    w = floor.support_wrench(None, q, qd, qdd)                # (M, 6) the support's wrench on the whole robot, one launch
    pc = SupportStabilityConstraint(floor, half_lengths=(X, Y), friction=mu)  # the robot must not tip over or slide"""
import ctypes
import xml.etree.ElementTree as ET

import numpy as np

from . import _lib, _lib_dyn

MAX_BODIES = 16
BODY_DOUBLES = 27
REVOLUTE, PRISMATIC = 0, 1
_JOINT_TYPES = {"revolute": REVOLUTE, "continuous": REVOLUTE, "prismatic": PRISMATIC}
# pinocchio's ReferenceFrame values (include/toppra_b200_dyn.h TBD_WORLD, TBD_LOCAL, TBD_LOCAL_WORLD_ALIGNED)
REFERENCE_FRAMES = {"world": 0, "local": 1, "local_world_aligned": 2}


def rpy_matrix(rpy):
    """URDF `origin rpy`: fixed-axis roll-pitch-yaw, R = Rz(y) Ry(p) Rx(r)."""
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def axis_rotation(axis, angle):
    """Rotation by `angle` about the unit vector `axis` (Rodrigues)."""
    a = np.asarray(axis, dtype=np.float64)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * (K @ K)


class RigidBodyModel(object):
    """Fixed-base kinematic tree of nv <= 16 moving bodies, one joint DOF each (DOF index = body index), bodies in
    topological order (parent[k] < k, -1 = base).

    parent (nv,); joint_type (nv,) of "revolute" / "prismatic" (or 0 / 1); axis (nv, 3) in the joint frame;
    E (nv, 3, 3), r (nv, 3): placement of the joint frame in the parent frame at q = 0 (E maps body to parent
    coordinates); mass (nv,); com (nv, 3) in the body frame; inertia (nv, 6) = Ixx, Ixy, Ixz, Iyy, Iyz, Izz about the
    centre of mass in the body frame; gravity (3,) in the base frame; base_mass >= 0 and base_com (3,), in base
    coordinates, of the static base itself, which moves no joint and enters only the support wrench
    (RigidBodyFrame.support_wrench)."""

    def __init__(self, parent, joint_type, axis, E, r, mass, com, inertia, gravity=(0.0, 0.0, -9.81), joint_names=None,
                 effort_limit=None, velocity_limit=None, frames=None, base_mass=0.0, base_com=(0.0, 0.0, 0.0)):
        parent = np.asarray(parent, dtype=np.float64).reshape(-1)
        nv = parent.shape[0]
        if not 1 <= nv <= MAX_BODIES:
            raise ValueError("RigidBodyModel: %d moving bodies, supported 1..%d" % (nv, MAX_BODIES))
        jt = np.array([_JOINT_TYPES.get(t, t) if isinstance(t, str) else t for t in np.atleast_1d(joint_type)],
                      dtype=np.float64)
        axis = np.asarray(axis, dtype=np.float64).reshape(nv, 3)
        norm = np.linalg.norm(axis, axis=1, keepdims=True)
        axis = np.where(norm > 0, axis / np.where(norm > 0, norm, 1.0), axis)   # a zero axis is rejected by the library
        packed = np.zeros(3 + BODY_DOUBLES * nv)
        packed[:3] = np.asarray(gravity, dtype=np.float64).reshape(3)
        body = packed[3:].reshape(nv, BODY_DOUBLES)
        body[:, 0] = parent
        body[:, 1] = jt.reshape(nv)
        body[:, 2:5] = axis
        body[:, 5:14] = np.asarray(E, dtype=np.float64).reshape(nv, 9)
        body[:, 14:17] = np.asarray(r, dtype=np.float64).reshape(nv, 3)
        body[:, 17] = np.asarray(mass, dtype=np.float64).reshape(nv)
        body[:, 18:21] = np.asarray(com, dtype=np.float64).reshape(nv, 3)
        body[:, 21:27] = np.asarray(inertia, dtype=np.float64).reshape(nv, 6)
        self.packed = packed
        self.nv = nv
        self.joint_names = list(joint_names) if joint_names is not None else ["joint%d" % k for k in range(nv)]
        inf = np.full(nv, np.inf)
        self.effort_limit = inf.copy() if effort_limit is None else np.asarray(effort_limit, dtype=np.float64)
        self.velocity_limit = inf.copy() if velocity_limit is None else np.asarray(velocity_limit, dtype=np.float64)
        # name -> (body index, R, p): frames rigidly attached to a body (-1 = the base), in that body's coordinates
        self.frames = dict(frames) if frames is not None else {"body%d" % k: (k, np.eye(3), np.zeros(3))
                                                               for k in range(nv)}
        self.base_mass, self.base_com = _base_inertia("RigidBodyModel", base_mass, base_com)

    @property
    def dof(self):
        return self.nv

    @property
    def gravity(self):
        return self.packed[:3].copy()

    def body(self, k):
        """The 27 packed doubles of body k (include/toppra_b200_dyn.h)."""
        return self.packed[3 + BODY_DOUBLES * k:3 + BODY_DOUBLES * (k + 1)].copy()

    def frame(self, name, xyz=(0.0, 0.0, 0.0), rpy=(0.0, 0.0, 0.0), reference_frame="local_world_aligned"):
        """The frame `name` of the frame table (every URDF link, or "body<k>"), moved by the offset `xyz` / `rpy` in
        its own coordinates (URDF origin convention; e.g. a tool-centre point), whose velocities are expressed in
        `reference_frame`: "local", "world" or "local_world_aligned" (pinocchio's ReferenceFrame)."""
        if name not in self.frames:
            raise ValueError("RigidBodyModel has no frame %r (frames: %s)" % (name, sorted(self.frames)))
        if reference_frame not in REFERENCE_FRAMES:
            raise ValueError("unknown reference_frame %r (known: %s)" % (reference_frame, sorted(REFERENCE_FRAMES)))
        body, R, p = self.frames[name]
        Ro = rpy_matrix(np.asarray(rpy, dtype=np.float64).reshape(3))
        return RigidBodyFrame(self, name, body, R @ Ro, p + R @ np.asarray(xyz, dtype=np.float64).reshape(3),
                              reference_frame)

    def packed_base(self):
        """The packed base of include/toppra_b200_dyn.h: (base_mass, base_com)."""
        return np.concatenate(([self.base_mass], self.base_com))

    def torque_limits(self):
        """(nv, 2) [-effort, effort] per joint, the tau_lim of JointTorqueConstraint (+-inf where the URDF has none)."""
        return np.stack([-self.effort_limit, self.effort_limit], axis=1)

    def with_payload(self, frame, mass, com, inertia):
        """A new model with a payload rigidly held by `frame` (a frame name or a RigidBodyFrame of this model) folded
        into the frame's body by the parallel-axis theorem: mass > 0, centre of mass com (3,) and rotational inertia
        (6,) = Ixx, Ixy, Ixz, Iyy, Iyz, Izz about it (positive semi-definite), both in the frame's axes.  Joint names,
        limits, gravity, the frame table and the base's mass and centre of mass are kept."""
        if isinstance(frame, RigidBodyFrame):
            if frame.model is not self:
                raise ValueError("with_payload: the frame %r belongs to another model" % frame.name)
            body, R, p = frame.body, frame.R, frame.p
        else:
            if frame not in self.frames:
                raise ValueError("RigidBodyModel has no frame %r (frames: %s)" % (frame, sorted(self.frames)))
            body, R, p = self.frames[frame]
        mass, com, I = _rigid_inertia("with_payload", mass, com, inertia)
        if body < 0:
            raise ValueError("with_payload: frame %r is on the base, where a payload moves no joint" % (frame,))
        bodies = self.packed[3:].reshape(self.nv, BODY_DOUBLES).copy()
        bd = bodies[body]
        mb, cb = bd[17], bd[18:21].copy()
        Ib = _inertia3(bd[21:27])
        cp, Ip = R @ com + p, R @ I @ R.T                      # the payload in body coordinates
        m = mb + mass
        c = (mb * cb + mass * cp) / m
        Ic = np.zeros((3, 3))
        for pm, pc, pI in ((mb, cb, Ib), (mass, cp, Ip)):
            d = pc - c
            Ic = Ic + pI + pm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
        bd[17], bd[18:21] = m, c
        bd[21:27] = [Ic[0, 0], Ic[0, 1], Ic[0, 2], Ic[1, 1], Ic[1, 2], Ic[2, 2]]
        return RigidBodyModel(bodies[:, 0], bodies[:, 1], bodies[:, 2:5], bodies[:, 5:14].reshape(-1, 3, 3),
                              bodies[:, 14:17], bodies[:, 17], bodies[:, 18:21], bodies[:, 21:27], self.gravity,
                              joint_names=self.joint_names, effort_limit=self.effort_limit.copy(),
                              velocity_limit=self.velocity_limit.copy(), frames=self.frames, base_mass=self.base_mass,
                              base_com=self.base_com)

    def inertialess_joints(self):
        """Names of the moving joints that move no inertia: the joint's body and all its descendants have zero mass and
        zero rotational inertia, so the mass matrix M(q) is singular at every q."""
        bodies = self.packed[3:].reshape(self.nv, BODY_DOUBLES)
        empty = [bool(bd[17] == 0 and not np.any(bd[21:27])) for bd in bodies]
        for k in range(self.nv - 1, -1, -1):                   # children come after their parent
            par = int(bodies[k, 0])
            if par >= 0 and not empty[k]:
                empty[par] = False
        return [self.joint_names[k] for k in range(self.nv) if empty[k]]

    # ---- evaluation on the GPU ----------------------------------------------------------------------------------
    def _prepare(self, torch, *xs):
        out = []
        for x in xs:
            if x.dim() != 2 or x.shape[1] != self.nv:
                raise ValueError("RigidBodyModel: expected (M, %d) tensors, got %s" % (self.nv, tuple(x.shape)))
            out.append(x.to(dtype=torch.float64).contiguous())
        if any(x.shape != out[0].shape or x.device != out[0].device for x in out):
            raise ValueError("RigidBodyModel: q, qd, qdd must share shape and device")
        return out

    def __call__(self, q, qd, qdd):
        """Joint torques tau = M(q) qdd + h(q, qd) + g(q).  CUDA tensors (M, nv) -> (M, nv), one tbd_rnea launch on the
        current stream; numpy (nv,) or (M, nv) -> numpy, through a device round trip."""
        if not _is_cuda(q):
            return _round_trip(self, q, qd, qdd)
        return _launch(self, "tbd_rnea", (), (q, qd, qdd), [(self.nv,)])

    def torque_terms(self, q, qs, qss, friction=None):
        """The terms of SecondOrderConstraint for CUDA tensors (M, nv), one tbd_torque_terms launch:
        c = ID(q, 0, 0), a = ID(q, 0, qs) - c, b = ID(q, qs, qss) - c, c += sign(qs) * friction (friction (nv,) or
        None).  Returns (a, b, c)."""
        fric = None
        if friction is not None and np.any(np.asarray(friction) != 0):
            fric = np.broadcast_to(np.asarray(friction, dtype=np.float64), (self.nv,)).copy()
        return _launch(self, "tbd_torque_terms", (), (q, qs, qss), [(self.nv,)] * 3, extra=(fric,))

    # ---- URDF ---------------------------------------------------------------------------------------------------
    @classmethod
    def from_urdf(cls, urdf, locked_joints=None, gravity=(0.0, 0.0, -9.81)):
        """Build the model from a URDF file name or XML string (xml.etree only).

        revolute / continuous joints become revolute bodies, prismatic ones prismatic; fixed joints and the joints named
        in `locked_joints` (name -> position) fold their child link into the parent body (mass, centre of mass, inertia
        by the parallel-axis theorem).  DOF order is depth-first with children in file order; `joint_names` lists it.
        The root link and the links folded into it (e.g. locked wheels) make the static base: `base_mass` and
        `base_com` (base coordinates).  floating, planar and unlocked mimic joints, a missing or ambiguous root and more
        than 16 moving bodies raise ValueError."""
        text = urdf if urdf.lstrip().startswith("<") else open(urdf).read()
        robot = ET.fromstring(text)
        locked = dict(locked_joints or {})
        links = {}
        for el in robot.findall("link"):
            links[el.get("name")] = el
        joints, parent_of, children = [], {}, {name: [] for name in links}
        for el in robot.findall("joint"):
            name, jtype = el.get("name"), el.get("type")
            par, chi = el.find("parent").get("link"), el.find("child").get("link")
            if par not in links or chi not in links:
                raise ValueError("URDF joint %r connects unknown links %r -> %r" % (name, par, chi))
            if chi in parent_of:
                raise ValueError("URDF link %r has two parent joints" % chi)
            if jtype in ("floating", "planar"):
                raise ValueError("URDF joint %r: %s joints are not supported (fixed base, one DOF per joint)"
                                 % (name, jtype))
            if jtype not in _JOINT_TYPES and jtype != "fixed":
                raise ValueError("URDF joint %r: unknown type %r" % (name, jtype))
            if el.find("mimic") is not None and name not in locked:
                raise ValueError("URDF joint %r mimics another joint; lock it (locked_joints)" % name)
            parent_of[chi] = name
            joints.append(el)
            children[par].append(el)
        unknown = set(locked) - {j.get("name") for j in joints}
        if unknown:
            raise ValueError("locked_joints names unknown joints: %s" % sorted(unknown))
        roots = [name for name in links if name not in parent_of]
        if len(roots) != 1:
            raise ValueError("URDF needs exactly one root link, found %s" % (roots or "none"))

        bodies = []          # dicts of one moving body each, in DOF order
        parts = {-1: []}     # body index -> [(mass, com, inertia about com)] in the body frame
        frames = {}          # link name -> (body index, R, p) of the link frame in the body frame

        def origin(el):
            o = el.find("origin") if el is not None else None
            xyz = np.array(o.get("xyz", "0 0 0").split(), dtype=np.float64) if o is not None else np.zeros(3)
            rpy = np.array(o.get("rpy", "0 0 0").split(), dtype=np.float64) if o is not None else np.zeros(3)
            return rpy_matrix(rpy), xyz

        def add_inertial(body, link, R, p):
            inert = links[link].find("inertial")
            if inert is None:
                return
            Ri, pi = origin(inert)
            m = float(inert.find("mass").get("value")) if inert.find("mass") is not None else 0.0
            el = inert.find("inertia")
            v = {k: float(el.get(k, 0.0)) if el is not None else 0.0
                 for k in ("ixx", "ixy", "ixz", "iyy", "iyz", "izz")}
            I = np.array([[v["ixx"], v["ixy"], v["ixz"]], [v["ixy"], v["iyy"], v["iyz"]], [v["ixz"], v["iyz"], v["izz"]]])
            Rb = R @ Ri
            parts[body].append((m, R @ pi + p, Rb @ I @ Rb.T))

        def visit(link, body, R, p):
            frames[link] = (body, R, p)
            add_inertial(body, link, R, p)
            for el in children[link]:
                name, jtype = el.get("name"), el.get("type")
                Ro, po = origin(el)
                Rj, pj = R @ Ro, R @ po + p
                ax_el = el.find("axis")
                axis = np.array(ax_el.get("xyz").split(), dtype=np.float64) if ax_el is not None else np.array([1.0, 0.0, 0.0])
                if np.linalg.norm(axis) == 0 and jtype != "fixed":
                    raise ValueError("URDF joint %r has a zero axis" % name)
                axis = axis / np.linalg.norm(axis) if jtype != "fixed" else axis
                child = el.find("child").get("link")
                if jtype == "fixed" or name in locked:
                    if jtype != "fixed":
                        pos = float(locked[name])
                        if _JOINT_TYPES[jtype] == REVOLUTE:
                            Rj = Rj @ axis_rotation(axis, pos)
                        else:
                            pj = pj + Rj @ (axis * pos)
                    visit(child, body, Rj, pj)
                    continue
                if len(bodies) == MAX_BODIES:
                    raise ValueError("URDF has more than %d moving joints" % MAX_BODIES)
                lim = el.find("limit")
                bodies.append(dict(parent=body, type=_JOINT_TYPES[jtype], axis=axis, E=Rj, r=pj, name=name,
                                   effort=float(lim.get("effort", np.inf)) if lim is not None else np.inf,
                                   velocity=float(lim.get("velocity", np.inf)) if lim is not None else np.inf))
                k = len(bodies) - 1
                parts[k] = []
                visit(child, k, np.eye(3), np.zeros(3))

        visit(roots[0], -1, np.eye(3), np.zeros(3))
        if not bodies:
            raise ValueError("URDF has no moving joint")
        mass, com, inertia = [], [], []
        for k in range(len(bodies)):
            m = sum(pm for pm, _, _ in parts[k])
            c = sum(pm * pc for pm, pc, _ in parts[k]) / m if m > 0 else np.zeros(3)
            Ic = np.zeros((3, 3))
            for pm, pc, pI in parts[k]:
                d = pc - c
                Ic = Ic + pI + pm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
            mass.append(m)
            com.append(c)
            inertia.append([Ic[0, 0], Ic[0, 1], Ic[0, 2], Ic[1, 1], Ic[1, 2], Ic[2, 2]])
        base_mass = sum(pm for pm, _, _ in parts[-1])
        base_com = sum(pm * pc for pm, pc, _ in parts[-1]) / base_mass if base_mass > 0 else np.zeros(3)
        return cls([b["parent"] for b in bodies], [b["type"] for b in bodies], [b["axis"] for b in bodies],
                   [b["E"] for b in bodies], [b["r"] for b in bodies], mass, com, inertia, gravity,
                   joint_names=[b["name"] for b in bodies], effort_limit=[b["effort"] for b in bodies],
                   velocity_limit=[b["velocity"] for b in bodies], frames=frames, base_mass=base_mass,
                   base_com=base_com)


class RigidBodyFrame(object):
    """A frame rigidly attached to a body of a RigidBodyModel (model.frame(...)): body index (-1 = the base), its
    placement (R, p) in the body frame and the reference frame of its velocities.  `packed` is the host array of
    include/toppra_b200_dyn.h.

    A velocity is [linear(3); angular(3)] (pinocchio's Motion::toVector()).  With p_f, R_f the frame's world placement
    and w the world angular velocity: "local_world_aligned" (dp_f, w), "local" (R_f^T dp_f, R_f^T w), "world"
    (dp_f - w x p_f, w), the spatial velocity at the world origin.  Calling the frame like `compute_velocity(q, qd)` makes
    it the frame-velocity callback of CartesianVelocityNorm, which then takes its device route."""

    def __init__(self, model, name, body, R, p, reference_frame="local_world_aligned"):
        self.model = model
        self.name = name
        self.body = int(body)
        self.R = np.array(R, dtype=np.float64).reshape(3, 3)
        self.p = np.array(p, dtype=np.float64).reshape(3)
        self.reference_frame = reference_frame
        self.packed = np.concatenate(([float(self.body)], self.R.reshape(9), self.p,
                                      [float(REFERENCE_FRAMES[reference_frame])]))

    @property
    def nv(self):
        return self.model.nv

    def __call__(self, q, qd):
        """Frame velocities.  CUDA tensors (M, nv) -> (M, 6), one tbd_frame_velocity launch on the current stream;
        numpy (nv,) -> (6,) or (M, nv) -> (M, 6), through a device round trip."""
        if not _is_cuda(q):
            return _round_trip(self, q, qd)
        return _launch(self.model, "tbd_frame_velocity", (self.packed,), (q, qd), [(6,)])

    def velocity_norm_terms(self, q, qs, S):
        """b = v^T (S v), v the frame velocity at (q, qs = q'), for CUDA tensors (M, nv) -> (M,): one
        tbd_velocity_norm_terms launch.  S: (6, 6)."""
        S = np.ascontiguousarray(S, dtype=np.float64)
        if S.shape != (6, 6):
            raise ValueError("S matrix should be of size 6x6.")
        return _launch(self.model, "tbd_velocity_norm_terms", (self.packed, S), (q, qs), [()])

    def _refuse_world(self, quantity):
        """ValueError for a "world" frame where `quantity` is one of the frame origin."""
        if self.reference_frame == "world":
            raise ValueError("RigidBodyFrame %r: %s; the \"world\" reference frame is not supported (use \"local\" or "
                             "\"local_world_aligned\")" % (self.name, quantity))

    def _check_acceleration(self):
        self._refuse_world("frame accelerations are classical accelerations of the frame origin")

    def acceleration(self, q, qd, qdd):
        """Classical frame accelerations [linear(3); angular(3)] (pinocchio's getFrameClassicalAcceleration, no
        gravity): "local_world_aligned" (d2p_f/dt2, dw/dt), "local" (R_f^T d2p_f/dt2, R_f^T dw/dt).  CUDA tensors
        (M, nv) -> (M, 6), one tbd_frame_acceleration launch on the current stream; numpy (nv,) -> (6,) or (M, nv) ->
        (M, 6), through a device round trip.  On one numpy point it is an `inv_dyn` of SecondOrderConstraint."""
        self._check_acceleration()
        if not _is_cuda(q):
            return _round_trip(self.acceleration, q, qd, qdd)
        return _launch(self.model, "tbd_frame_acceleration", (self.packed,), (q, qd, qdd), [(6,)])

    def acceleration_terms(self, q, qs, qss, components):
        """a = acc(q, 0, qs), b = acc(q, qs, qss) for CUDA tensors (M, nv), restricted to `components` (indices into
        [ax, ay, az, wx, wy, wz]; the columns come in increasing index order): one tbd_acceleration_terms launch.
        Returns (a, b), each (M, k)."""
        self._check_acceleration()
        comps = component_indices(components)
        mask = sum(1 << j for j in comps)
        return _launch(self.model, "tbd_acceleration_terms", (self.packed, mask), (q, qs, qss), [(len(comps),)] * 2)

    def contact_wrench(self, obj, q, qd, qdd):
        """The wrench [f; tau] this frame, as a contact frame, exerts on an object it carries, at its origin in its own
        axes (the reference frame is ignored); `obj` is the packed object of include/toppra_b200_dyn.h (m, r, Ic; see
        ContactStabilityConstraint).  CUDA tensors (M, nv) -> (M, 6), one tbd_contact_wrench launch on the current
        stream; numpy (nv,) -> (6,) or (M, nv) -> (M, 6), through a device round trip."""
        obj = _packed_object(obj)
        if not _is_cuda(q):
            return _round_trip(lambda *x: self.contact_wrench(obj, *x), q, qd, qdd)
        return _launch(self.model, "tbd_contact_wrench", (self.packed, obj), (q, qd, qdd), [(6,)])

    def contact_wrench_terms(self, obj, q, qs, qss):
        """c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c of the contact wrench (contact_wrench) for CUDA
        tensors (M, nv): one tbd_contact_wrench_terms launch.  Returns (a, b, c), each (M, 6)."""
        obj = _packed_object(obj)
        return _launch(self.model, "tbd_contact_wrench_terms", (self.packed, obj), (q, qs, qss), [(6,)] * 3)

    def inverse_inertia(self, q):
        """Lambda_v^-1 = J_v M(q)^-1 J_v^T of the frame origin: the inverse operational-space inertia for linear motion
        (Khatib), whose quadratic form u^T Lambda_v^-1 u = 1 / m_R(u) gives the robot's effective mass in the unit
        direction u.  "local_world_aligned": world axes; "local": R_f^T Lambda_v^-1 R_f; "world" raises ValueError.
        NaN where M(q) is singular.  CUDA tensors (M, nv) -> (M, 3, 3), one tbd_frame_inverse_inertia launch on the
        current stream; numpy (nv,) -> (3, 3) or (M, nv) -> (M, 3, 3), through a device round trip."""
        self._refuse_world("the inverse inertia is that of the frame origin")
        if not _is_cuda(q):
            return _round_trip(self.inverse_inertia, q)
        return _launch(self.model, "tbd_frame_inverse_inertia", (self.packed,), (q,), [(3, 3)])

    def collision_energy_terms(self, q, qs, human_mass):
        """b = 1/2 |v|^4 / (|v|^2 / m_H + v^T Lambda_v^-1 v), v the world linear velocity of the frame origin at
        (q, qs = q'), m_H = human_mass (> 0, inf allowed): the collision energy E = b s'^2 of
        CollisionEnergyConstraint, for CUDA tensors (M, nv) -> (M,): one tbd_collision_energy_terms launch.  The
        reference frame is ignored."""
        return _launch(self.model, "tbd_collision_energy_terms", (self.packed, float(human_mass)), (q, qs), [()])

    def _support_base(self, base):
        """The packed base of a support frame, which must be on the base: the model's when `base` is None."""
        if self.body != -1:
            raise ValueError("RigidBodyFrame %r: the support must be on the base (frame body %d, expected -1)"
                             % (self.name, self.body))
        return self.model.packed_base() if base is None else _packed_base(base)

    def support_wrench(self, base, q, qd, qdd):
        """The wrench [f; tau] the support exerts on the whole robot, at this frame's origin in its axes (the reference
        frame is ignored); this frame must be on the base, its z axis the support normal pointing into the robot.
        `base` is the packed base of include/toppra_b200_dyn.h (m_b, c_b), or None for the model's (base_mass,
        base_com).  CUDA tensors (M, nv) -> (M, 6), one tbd_support_wrench launch on the current stream; numpy (nv,) ->
        (6,) or (M, nv) -> (M, 6), through a device round trip: on one numpy point an `inv_dyn` of
        SecondOrderConstraint."""
        base = self._support_base(base)
        if not _is_cuda(q):
            return _round_trip(lambda *x: self.support_wrench(base, *x), q, qd, qdd)
        return _launch(self.model, "tbd_support_wrench", (self.packed, base), (q, qd, qdd), [(6,)])

    def support_wrench_terms(self, base, q, qs, qss):
        """c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c of the support wrench (support_wrench) for CUDA
        tensors (M, nv): one tbd_support_wrench_terms launch.  Returns (a, b, c), each (M, 6)."""
        base = self._support_base(base)
        return _launch(self.model, "tbd_support_wrench_terms", (self.packed, base), (q, qs, qss), [(6,)] * 3)


def _is_cuda(x):
    """Whether x is a CUDA tensor; there is no CPU route, so a CUDA device is required either way."""
    torch = _lib.require_cuda()
    return isinstance(x, torch.Tensor) and x.is_cuda


def _round_trip(fn, *xs):
    """fn, which takes CUDA tensors (M, nv), on numpy inputs: (nv,) -> one point, (M, nv) -> (M, ...)."""
    torch = _lib.require_cuda()
    arrs = [np.asarray(x, dtype=np.float64) for x in xs]
    out = fn(*[torch.as_tensor(np.atleast_2d(x), device="cuda") for x in arrs]).cpu().numpy()
    return out[0] if arrs[0].ndim == 1 else out


def _launch(model, name, params, inputs, out_shapes, extra=()):
    """One launch of the dyn entry `name` on the current stream; every entry takes (model, nv, *params, M, *inputs,
    *extra, *outputs, stream).  params: host numpy arrays (passed by pointer) and scalars; inputs: (M, nv) CUDA tensors;
    extra: host vectors copied to their device, or None for a null pointer; outputs: new float64 tensors (M,) + shape
    for each of `out_shapes`.  Returns the output, or the tuple of outputs."""
    torch = _lib.require_cuda()
    inputs = model._prepare(torch, *inputs)
    q = inputs[0]
    extra = [None if x is None else torch.as_tensor(x, device=q.device) for x in extra]
    outs = [torch.empty((q.shape[0],) + tuple(s), dtype=torch.float64, device=q.device) for s in out_shapes]
    host = [ctypes.c_void_p(p.ctypes.data) if isinstance(p, np.ndarray) else p for p in params]
    with torch.cuda.device(q.device):
        _lib.check(getattr(_lib_dyn.load(), name)(ctypes.c_void_p(model.packed.ctypes.data), model.nv, *host,
                                                  q.shape[0], *[_lib.ptr(x) for x in inputs + extra],
                                                  *[_lib.ptr(o) for o in outs], _lib.stream_ptr()), name)
    return outs[0] if len(outs) == 1 else tuple(outs)


def _inertia3(I6):
    Ixx, Ixy, Ixz, Iyy, Iyz, Izz = I6
    return np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]], dtype=np.float64)


def _rigid_inertia(what, mass, com, inertia):
    """(mass, com (3,), inertia 3x3) of a rigid body, or ValueError: finite, mass > 0, inertia positive semi-definite."""
    mass = np.asarray(mass, dtype=np.float64)
    com = np.asarray(com, dtype=np.float64)
    inertia = np.asarray(inertia, dtype=np.float64)
    if mass.shape != () or com.shape != (3,) or inertia.shape != (6,):
        raise ValueError("%s: expected a scalar mass, com (3,) and inertia (6,); got shapes %s, %s, %s"
                         % (what, mass.shape, com.shape, inertia.shape))
    if not (np.isfinite(mass) and np.isfinite(com).all() and np.isfinite(inertia).all()):
        raise ValueError("%s: mass, com and inertia must be finite" % what)
    if not mass > 0:
        raise ValueError("%s: mass %r must be positive" % (what, float(mass)))
    I = _inertia3(inertia)
    if np.linalg.eigvalsh(I).min() < -1e-12 * max(1e-300, np.abs(I).max()):
        raise ValueError("%s: the inertia matrix is not positive semi-definite" % what)
    return float(mass), com, I


OBJECT_DOUBLES = 10


def _packed_object(obj):
    """The packed object of include/toppra_b200_dyn.h (TBD_OBJECT_DOUBLES = 10 doubles: m, r, Ic) as a contiguous
    float64 array; the library reads exactly 10 doubles from it."""
    obj = np.ascontiguousarray(obj, dtype=np.float64)
    if obj.shape != (OBJECT_DOUBLES,):
        raise ValueError("packed object: expected %d doubles (m, r, Ic), got shape %s" % (OBJECT_DOUBLES, obj.shape))
    return obj


BASE_DOUBLES = 4


def _base_inertia(what, mass, com):
    """(mass, com (3,)) of a static base, or ValueError: finite, mass >= 0."""
    mass = np.asarray(mass, dtype=np.float64)
    com = np.asarray(com, dtype=np.float64)
    if mass.shape != () or com.shape != (3,):
        raise ValueError("%s: expected a scalar base mass and a base com (3,); got shapes %s, %s"
                         % (what, mass.shape, com.shape))
    if not (np.isfinite(mass) and np.isfinite(com).all()):
        raise ValueError("%s: the base mass and base com must be finite" % what)
    if not mass >= 0:
        raise ValueError("%s: the base mass %r must be non-negative" % (what, float(mass)))
    return float(mass), com.copy()


def _packed_base(base):
    """The packed base of include/toppra_b200_dyn.h (TBD_BASE_DOUBLES = 4 doubles: m_b, c_b) as a contiguous float64
    array; the library reads exactly 4 doubles from it."""
    base = np.ascontiguousarray(base, dtype=np.float64)
    if base.shape != (BASE_DOUBLES,):
        raise ValueError("packed base: expected %d doubles (m_b, c_b), got shape %s" % (BASE_DOUBLES, base.shape))
    return base


def component_indices(components):
    """Sorted indices into [ax, ay, az, wx, wy, wz] of a frame acceleration; ValueError when `components` is empty,
    repeats an index or has one outside 0..5."""
    comps = np.asarray(components).reshape(-1)
    if (comps.size == 0 or comps.dtype.kind not in "iu" or len(set(comps.tolist())) != comps.size
            or comps.min() < 0 or comps.max() > 5):
        raise ValueError("components %r: expected distinct indices in 0..5 of [ax, ay, az, wx, wy, wz]"
                         % (components,))
    return sorted(comps.tolist())
