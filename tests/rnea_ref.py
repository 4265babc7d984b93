"""TEST INFRASTRUCTURE — references for rigid-body inverse dynamics (toppra_b200.RigidBodyModel, libtoppra_b200_dyn.so).

* `MpRobot`: 50-digit mpmath inverse dynamics of the RAW URDF tree (fixed and locked joints stay zero-DOF links, so the
  folding of RigidBodyModel.from_urdf is checked too), or of a packed model.  It does not use the recursive
  Newton-Euler algorithm of the kernels: it takes the Lagrangian form
      M(q) = sum_links m Jv^T Jv + Jw^T (R I R^T) Jw,     g(q) = -sum_links Jv^T m g,
      h_k  = sum_ij (d_i M_kj - 1/2 d_k M_ij) qd_i qd_j   (d_i M by mpmath.diff),
      tau  = M qdd + h + g,
  with Jacobians from world-frame joint axes and origins.
* `rnea_packed`, `torque_terms_packed`: a float64 numpy double of tbd_rnea / tbd_torque_terms on the packed layout of
  include/toppra_b200_dyn.h, vectorised over points: the CPU double of the two entries for host-side tests."""
import xml.etree.ElementTree as ET

import mpmath
import numpy as np

DPS = 50


# ==== 50-digit Lagrangian reference ==================================================================================
def _mpv(text, default="0 0 0"):
    return [mpmath.mpf(x) for x in (text if text is not None else default).split()]


def _rot_rpy(rpy):
    r, p, y = rpy
    Rx = mpmath.matrix([[1, 0, 0], [0, mpmath.cos(r), -mpmath.sin(r)], [0, mpmath.sin(r), mpmath.cos(r)]])
    Ry = mpmath.matrix([[mpmath.cos(p), 0, mpmath.sin(p)], [0, 1, 0], [-mpmath.sin(p), 0, mpmath.cos(p)]])
    Rz = mpmath.matrix([[mpmath.cos(y), -mpmath.sin(y), 0], [mpmath.sin(y), mpmath.cos(y), 0], [0, 0, 1]])
    return Rz * Ry * Rx


def _rot_axis(a, t):
    K = mpmath.matrix([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return mpmath.eye(3) + mpmath.sin(t) * K + (1 - mpmath.cos(t)) * (K * K)


def _unit(v):
    n = mpmath.sqrt(sum(x * x for x in v))
    return mpmath.matrix([x / n for x in v])


def _cross(a, b):
    return mpmath.matrix([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


class MpRobot(object):
    """A fixed-base tree of links joined by joints: ("revolute" | "prismatic" | "fixed", parent link, child link,
    origin (R, p), unit axis, locked position or None).  Moving joints get DOF indices in depth-first order."""

    def __init__(self, links, joints, root, gravity):
        self.links = links          # name -> (mass, com, R_inertial, I 3x3) in the link frame
        self.joints = joints        # list of dicts, topological (depth-first) order
        self.root = root
        self.g = mpmath.matrix([mpmath.mpf(x) for x in gravity])
        self.nv = sum(1 for j in joints if j["dof"] is not None)

    @classmethod
    def from_urdf(cls, text, locked_joints=None, gravity=("0", "0", "-9.81")):
        locked = {k: mpmath.mpf(v) for k, v in (locked_joints or {}).items()}
        robot = ET.fromstring(text)
        links = {}
        for el in robot.findall("link"):
            inert = el.find("inertial")
            if inert is None:
                links[el.get("name")] = None
                continue
            o = inert.find("origin")
            m = mpmath.mpf(inert.find("mass").get("value"))
            i = inert.find("inertia")
            v = {k: mpmath.mpf(i.get(k, "0")) for k in ("ixx", "ixy", "ixz", "iyy", "iyz", "izz")}
            I = mpmath.matrix([[v["ixx"], v["ixy"], v["ixz"]], [v["ixy"], v["iyy"], v["iyz"]],
                               [v["ixz"], v["iyz"], v["izz"]]])
            links[el.get("name")] = (m, mpmath.matrix(_mpv(o.get("xyz") if o is not None else None)),
                                     _rot_rpy(_mpv(o.get("rpy") if o is not None else None)), I)
        raw, children, has_parent = [], {}, set()
        for el in robot.findall("joint"):
            o, ax = el.find("origin"), el.find("axis")
            jt = {"continuous": "revolute"}.get(el.get("type"), el.get("type"))
            j = dict(name=el.get("name"), type=jt, parent=el.find("parent").get("link"),
                     child=el.find("child").get("link"),
                     R=_rot_rpy(_mpv(o.get("rpy") if o is not None else None)),
                     p=mpmath.matrix(_mpv(o.get("xyz") if o is not None else None)),
                     axis=_unit(_mpv(ax.get("xyz") if ax is not None else None, "1 0 0")),
                     locked=locked.get(el.get("name")), dof=None)
            raw.append(j)
            children.setdefault(j["parent"], []).append(j)
            has_parent.add(j["child"])
        root = [n for n in links if n not in has_parent][0]
        order = []

        def visit(link):
            for j in children.get(link, []):
                if j["type"] != "fixed" and j["locked"] is None:
                    j["dof"] = sum(1 for x in order if x["dof"] is not None)
                order.append(j)
                visit(j["child"])
        visit(root)
        return cls(links, order, root, gravity)

    @classmethod
    def from_packed(cls, packed):
        """The same reference on a packed model (include/toppra_b200_dyn.h): body k = link "b<k>" on joint k."""
        packed = np.asarray(packed, dtype=np.float64)
        nv = (len(packed) - 3) // 27
        links, joints = {"base": None}, []
        for k in range(nv):
            bd = [mpmath.mpf(float(x)) for x in packed[3 + 27 * k:3 + 27 * (k + 1)]]
            Ixx, Ixy, Ixz, Iyy, Iyz, Izz = bd[21:27]
            links["b%d" % k] = (bd[17], mpmath.matrix(bd[18:21]), mpmath.eye(3),
                                mpmath.matrix([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]]))
            par = int(bd[0])
            joints.append(dict(name="j%d" % k, type="revolute" if bd[1] == 0 else "prismatic",
                               parent="base" if par < 0 else "b%d" % par, child="b%d" % k,
                               R=mpmath.matrix([bd[5:8], bd[8:11], bd[11:14]]), p=mpmath.matrix(bd[14:17]),
                               axis=mpmath.matrix(bd[2:5]), locked=None, dof=k))
        return cls(links, joints, "base", [mpmath.mpf(float(x)) for x in packed[:3]])

    def _kinematics(self, q):
        """World frames of every link and (axis, origin, type) of every DOF's joint."""
        frames = {self.root: (mpmath.eye(3), mpmath.matrix([0, 0, 0]))}
        path = {self.root: []}           # DOFs from the root to the link
        axes = {}
        for j in self.joints:
            Rp, pp = frames[j["parent"]]
            R0 = Rp * j["R"]
            p0 = pp + Rp * j["p"]
            t = q[j["dof"]] if j["dof"] is not None else j["locked"]
            if j["type"] == "revolute" and t is not None:
                R, p = R0 * _rot_axis(j["axis"], t), p0
            elif j["type"] == "prismatic" and t is not None:
                R, p = R0, p0 + R0 * (j["axis"] * t)
            else:
                R, p = R0, p0
            frames[j["child"]] = (R, p)
            path[j["child"]] = path[j["parent"]] + ([j["dof"]] if j["dof"] is not None else [])
            if j["dof"] is not None:
                axes[j["dof"]] = (R0 * j["axis"], p0, j["type"])
        return frames, path, axes

    def _link_terms(self, q):
        """Per massive link: (m, Jv 3 x nv, Jw 3 x nv, world inertia)."""
        frames, path, axes = self._kinematics(q)
        out = []
        for name, inert in self.links.items():
            if inert is None or name not in frames:
                continue
            m, c, Ri, I = inert
            R, p = frames[name]
            pc = p + R * c
            Rw = R * Ri
            Jv, Jw = mpmath.zeros(3, self.nv), mpmath.zeros(3, self.nv)
            for d in path[name]:
                z, o, kind = axes[d]
                col = _cross(z, pc - o) if kind == "revolute" else z
                for r in range(3):
                    Jv[r, d] = col[r]
                    Jw[r, d] = z[r] if kind == "revolute" else 0
            out.append((m, Jv, Jw, Rw * I * Rw.T))
        return out

    def mass_matrix(self, q):
        M = mpmath.zeros(self.nv, self.nv)
        for m, Jv, Jw, Iw in self._link_terms(q):
            M += m * (Jv.T * Jv) + Jw.T * Iw * Jw
        return M

    def gravity_torque(self, q):
        g = mpmath.zeros(self.nv, 1)
        for m, Jv, _, _ in self._link_terms(q):
            g -= Jv.T * (m * self.g)
        return g

    def velocity_torque(self, q, qd):
        nv = self.nv
        if all(x == 0 for x in qd):
            return mpmath.zeros(nv, 1)
        dM = []
        for i in range(nv):
            def Mi(t, i=i):
                return self.mass_matrix([q[k] + (t if k == i else 0) for k in range(nv)])
            dM.append(mpmath.diff(Mi, mpmath.mpf(0)))
        h = mpmath.zeros(nv, 1)
        for k in range(nv):
            h[k] = mpmath.fsum((dM[i][k, j] - dM[k][i, j] / 2) * qd[i] * qd[j] for i in range(nv) for j in range(nv))
        return h

    def tau(self, q, qd, qdd):
        """ID(q, qd, qdd) at DPS digits (inputs: floats or mpf)."""
        with mpmath.workdps(DPS):
            q, qd, qdd = ([mpmath.mpf(float(x)) if not isinstance(x, mpmath.mpf) else x for x in v] for v in (q, qd, qdd))
            t = self.mass_matrix(q) * mpmath.matrix(qdd) + self.velocity_torque(q, qd) + self.gravity_torque(q)
            return [t[k] for k in range(self.nv)]

    def tau64(self, q, qd, qdd):
        return np.array([float(x) for x in self.tau(q, qd, qdd)])


# ==== float64 numpy double of the two entries (packed layout) ========================================================
def _cross_np(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def _transforms(packed, q):
    nv = q.shape[1]
    Rs, ps = [], []
    for k in range(nv):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        ax, E, r = bd[2:5], bd[5:14].reshape(3, 3), bd[14:17]
        if bd[1] == 0:
            s, c = np.sin(q[:, k]), np.cos(q[:, k])
            K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
            J = np.eye(3)[None] + s[:, None, None] * K[None] + (1 - c)[:, None, None] * (K @ K)[None]
            Rs.append(np.einsum("ij,mjk->mik", E, J))
            ps.append(np.broadcast_to(r, (q.shape[0], 3)))
        else:
            Rs.append(np.broadcast_to(E, (q.shape[0], 3, 3)))
            ps.append(r[None] + (q[:, k:k + 1] * ax[None]) @ E.T)
    return Rs, ps


def _pass(packed, Rs, ps, qd, qdd):
    """The recursive Newton-Euler pass of the device's rnea_pass: (tau (M, nv), f), f[k] = [n, f] the force of body k
    plus those its children carried up (root children keep theirs)."""
    M, nv = qd.shape
    g = packed[:3]
    st, f = [], []
    for k in range(nv):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        par = int(bd[0])
        if par < 0:
            wp, vp, dwp = np.zeros((M, 3)), np.zeros((M, 3)), np.zeros((M, 3))
            dvp = np.broadcast_to(-g, (M, 3))
        else:
            wp, vp, dwp, dvp = st[par]
        R, p = Rs[k], ps[k]
        RT = lambda x: np.einsum("mji,mj->mi", R, x)   # noqa: E731
        w, v = RT(wp), RT(vp + _cross_np(wp, p))
        dw, dv = RT(dwp), RT(dvp + _cross_np(dwp, p))
        ax = bd[2:5][None]
        sq, sqq = ax * qd[:, k:k + 1], ax * qdd[:, k:k + 1]
        if bd[1] == 0:
            w = w + sq
            dw = dw + sqq + _cross_np(w, sq)
            dv = dv + _cross_np(v, sq)
        else:
            v = v + sq
            dv = dv + sqq + _cross_np(w, sq)
        st.append((w, v, dw, dv))
        m, c = bd[17], np.broadcast_to(bd[18:21], (M, 3))
        Ixx, Ixy, Ixz, Iyy, Iyz, Izz = bd[21:27]
        Ic = np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]])
        hl = m * (v + _cross_np(w, c))
        ha = w @ Ic.T + _cross_np(c, hl)
        fl = m * (dv + _cross_np(dw, c))
        n = dw @ Ic.T + _cross_np(c, fl)
        f.append([n + _cross_np(w, ha) + _cross_np(v, hl), fl + _cross_np(w, hl)])
    tau = np.zeros((M, nv))
    for k in range(nv - 1, -1, -1):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        tau[:, k] = (f[k][0] if bd[1] == 0 else f[k][1]) @ bd[2:5]
        par = int(bd[0])
        if par >= 0:
            Rf = np.einsum("mij,mj->mi", Rs[k], f[k][1])
            f[par][0] = f[par][0] + np.einsum("mij,mj->mi", Rs[k], f[k][0]) + _cross_np(ps[k], Rf)
            f[par][1] = f[par][1] + Rf
    return tau, f


def rnea_packed(packed, q, qd, qdd):
    """float64 double of tbd_rnea: (M, nv) arrays -> tau (M, nv)."""
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    Rs, ps = _transforms(np.asarray(packed, dtype=np.float64), q)
    return _pass(packed, Rs, ps, qd, qdd)[0]


def torque_terms_packed(packed, q, qs, qss, friction=None):
    """float64 double of tbd_torque_terms: (a, b, c)."""
    q, qs, qss = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qs, qss))
    Rs, ps = _transforms(np.asarray(packed, dtype=np.float64), q)
    zero = np.zeros_like(q)
    c = _pass(packed, Rs, ps, zero, zero)[0]
    a = _pass(packed, Rs, ps, zero, qs)[0] - c
    b = _pass(packed, Rs, ps, qs, qss)[0] - c
    if friction is not None and np.any(np.asarray(friction) != 0):
        c = c + np.sign(qs) * np.asarray(friction, dtype=np.float64)
    return a, b, c


def random_tree(rng, nv):
    """Random packed model: nv bodies, random parents, joint types, axes, placements and physical inertias."""
    packed = np.zeros(3 + 27 * nv)
    packed[:3] = rng.randn(3) * 4
    for k in range(nv):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        bd[0] = rng.randint(-1, k)
        bd[1] = 1 if rng.rand() < 0.25 else 0
        ax = rng.randn(3)
        bd[2:5] = ax / np.linalg.norm(ax)
        Q, _ = np.linalg.qr(rng.randn(3, 3))
        bd[5:14] = (Q * np.sign(np.linalg.det(Q))).reshape(9)
        bd[14:17] = rng.randn(3) * 0.3
        bd[17] = rng.uniform(0.1, 5.0)
        bd[18:21] = rng.randn(3) * 0.1
        P, _ = np.linalg.qr(rng.randn(3, 3))
        mom = rng.uniform(0.01, 0.1, 3)
        mom[2] = rng.uniform(abs(mom[0] - mom[1]) + 1e-3, mom[0] + mom[1] - 1e-3)   # triangle inequalities
        I = P @ np.diag(mom) @ P.T
        bd[21:27] = [I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2]]
    return packed
