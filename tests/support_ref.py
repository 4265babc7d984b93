"""TEST INFRASTRUCTURE — references for support wrenches (SupportStabilityConstraint, RigidBodyFrame.support_wrench /
support_wrench_terms, libtoppra_b200_dyn.so: tbd_support_wrench / tbd_support_wrench_terms).

* `mp_support_wrench`: the 50-digit wrench the support exerts on a whole `rnea_ref.MpRobot` (its `_kinematics` on the
  RAW URDF tree: fixed and locked joints stay zero-DOF links, nothing is folded, so the root link and everything fixed
  or locked to it count as links like the others) along t -> q + t qd + t^2/2 qdd.  For every link with an inertial,
  its centre-of-mass position p_i(t) and the world orientation R_i(t) of its inertia are differentiated with
  `mpmath.diff`; then, in base coordinates,
      f_i = m_i (p_i'' - g),   n_i = (p_i - o) x f_i + R_i' Ic_i R_i^T w_i + R_i Ic_i R_i'^T w_i + R_i Ic_i R_i^T w_i'
  with w = vee(R' R^T), w' = vee(R'' R^T) (as contact_ref.py): the rate of change of the link's momentum and of its
  angular momentum about the support origin o.  The sums over links are rotated into support axes.  It uses neither
  the recursion of the kernel nor a Jacobian.
* `support_wrench_packed`, `support_terms_packed`: a float64 numpy double of the device algorithm of the two entries
  (include/toppra_b200_dyn.h), vectorised over points."""
import mpmath
import numpy as np

import kin_ref
import rnea_ref

DPS = rnea_ref.DPS


def base_packed(mass, com):
    """The packed base of include/toppra_b200_dyn.h: m_b, c_b (3)."""
    return np.concatenate(([float(mass)], np.asarray(com, dtype=np.float64)))


# ==== 50-digit reference ==============================================================================================
def mp_support_wrench(robot, q, qd, qdd, R_s, p_s, base=None):
    """[f; tau] (6 mp) at the support origin p_s (base coordinates) in support axes R_s (float arrays).  `base`: an
    extra static point mass (packed m_b, c_b) on top of the robot's own links, for packed models whose base has none."""
    with mpmath.workdps(DPS):
        q, qd, qdd = ([mpmath.mpf(float(x)) for x in v] for v in (q, qd, qdd))
        Rs = mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(R_s)])
        o = mpmath.matrix([mpmath.mpf(float(x)) for x in np.asarray(p_s)])
        links = [(name, inert) for name, inert in robot.links.items() if inert is not None]
        cache = {}

        def placements(t):
            # (R of the inertia, centre-of-mass position) of every link; keyed by the working precision too, as in
            # contact_ref (mpmath.diff evaluates t = 0 at a raised precision)
            key_t = (t, mpmath.mp.prec)
            if key_t not in cache:
                fr = robot._kinematics([q[i] + t * qd[i] + t * t / 2 * qdd[i] for i in range(len(q))])[0]
                cache[key_t] = {name: (fr[name][0] * Ri, fr[name][1] + fr[name][0] * c)
                                for name, (_, c, Ri, _) in links}
            return cache[key_t]

        zero = mpmath.mpf(0)
        f, n = mpmath.matrix([0, 0, 0]), mpmath.matrix([0, 0, 0])
        for name, (m, _, _, Ic) in links:
            R, p = placements(zero)[name]
            ddp = mpmath.matrix([mpmath.diff(lambda t, i=i: placements(t)[name][1][i], zero, 2) for i in range(3)])
            dR, ddR = mpmath.matrix(3, 3), mpmath.matrix(3, 3)
            for i in range(3):
                for j in range(3):
                    dR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[name][0][i, j], zero, 1)
                    ddR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[name][0][i, j], zero, 2)
            w = mpmath.matrix(kin_ref._skew_vec(dR * R.T))
            dw = mpmath.matrix(kin_ref._skew_vec(ddR * R.T))
            fi = m * (ddp - robot.g)
            f += fi
            n += rnea_ref._cross(p - o, fi) + dR * Ic * R.T * w + R * Ic * dR.T * w + R * Ic * R.T * dw
        if base is not None:
            mb = mpmath.mpf(float(base[0]))
            cb = mpmath.matrix([mpmath.mpf(float(x)) for x in base[1:4]])
            fi = -mb * robot.g
            f += fi
            n += rnea_ref._cross(cb - o, fi)
        return list(Rs.T * f) + list(Rs.T * n)


def mp_total_com(robot, q):
    """(total mass, world centre of mass) of the raw tree's links at q, in closed form from the link masses (floats)."""
    with mpmath.workdps(DPS):
        fr = robot._kinematics([mpmath.mpf(float(x)) for x in q])[0]
        mass, mc = mpmath.mpf(0), mpmath.matrix([0, 0, 0])
        for name, inert in robot.links.items():
            if inert is None:
                continue
            m, c = inert[0], inert[1]
            mass += m
            mc += m * (fr[name][1] + fr[name][0] * c)
        return float(mass), np.array([float(x / mass) for x in mc])


# ==== float64 numpy double of the device algorithm ====================================================================
def _forces(packed, Rs, ps, qd, qdd):
    """The forces f[k] = (n, f) of every body after the recursive Newton-Euler pass of rnea_ref._pass (the device's
    rnea_pass): each body's own force plus those its children carried up; root children keep theirs."""
    M, nv = qd.shape
    g = packed[:3]
    cross = rnea_ref._cross_np
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
        w, v = RT(wp), RT(vp + cross(wp, p))
        dw, dv = RT(dwp), RT(dvp + cross(dwp, p))
        ax = bd[2:5][None]
        sq, sqq = ax * qd[:, k:k + 1], ax * qdd[:, k:k + 1]
        if bd[1] == 0:
            w = w + sq
            dw = dw + sqq + cross(w, sq)
            dv = dv + cross(v, sq)
        else:
            v = v + sq
            dv = dv + sqq + cross(w, sq)
        st.append((w, v, dw, dv))
        m, c = bd[17], np.broadcast_to(bd[18:21], (M, 3))
        Ixx, Ixy, Ixz, Iyy, Iyz, Izz = bd[21:27]
        Ic = np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]])
        hl = m * (v + cross(w, c))
        ha = w @ Ic.T + cross(c, hl)
        fl = m * (dv + cross(dw, c))
        n = dw @ Ic.T + cross(c, fl)
        f.append([n + cross(w, ha) + cross(v, hl), fl + cross(w, hl)])
    for k in range(nv - 1, -1, -1):
        par = int(packed[3 + 27 * k])
        if par >= 0:
            Rf = np.einsum("mij,mj->mi", Rs[k], f[k][1])
            f[par][0] = f[par][0] + np.einsum("mij,mj->mi", Rs[k], f[k][0]) + cross(ps[k], Rf)
            f[par][1] = f[par][1] + Rf
    return f


def _wrench(packed, frame, base, Rs, ps, f, M):
    cross = rnea_ref._cross_np
    nv = len(Rs)
    fb, nb = np.zeros((M, 3)), np.zeros((M, 3))
    for k in range(nv):
        if int(packed[3 + 27 * k]) >= 0:
            continue
        Rf = np.einsum("mij,mj->mi", Rs[k], f[k][1])
        nb = nb + np.einsum("mij,mj->mi", Rs[k], f[k][0]) + cross(ps[k], Rf)
        fb = fb + Rf
    wb = np.broadcast_to(-(base[0] * packed[:3]), (M, 3))
    nb = nb + cross(np.broadcast_to(base[1:4], (M, 3)), wb)
    fb = fb + wb
    R_s, p_s = np.asarray(frame[1:10]).reshape(3, 3), np.asarray(frame[10:13])
    t = nb - cross(np.broadcast_to(p_s, (M, 3)), fb)
    return np.concatenate((fb @ R_s, t @ R_s), axis=1)


def support_wrench_packed(packed, frame, base, q, qd, qdd):
    """Double of tbd_support_wrench: (M, nv) arrays -> w (M, 6) = [f; tau] in support axes at the support origin."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    Rs, ps = rnea_ref._transforms(packed, q)
    return _wrench(packed, frame, np.asarray(base, dtype=np.float64), Rs, ps, _forces(packed, Rs, ps, qd, qdd),
                   q.shape[0])


def support_terms_packed(packed, frame, base, q, qs, qss):
    """Double of tbd_support_wrench_terms: c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    zero = np.zeros_like(q)
    c = support_wrench_packed(packed, frame, base, q, zero, zero)
    a = support_wrench_packed(packed, frame, base, q, zero, qs) - c
    b = support_wrench_packed(packed, frame, base, q, qs, qss) - c
    return a, b, c


def zmp(w):
    """The centre of pressure (-tau_y / f_z, tau_x / f_z) of wrenches (..., 6)."""
    w = np.asarray(w)
    return np.stack((-w[..., 4] / w[..., 2], w[..., 3] / w[..., 2]), axis=-1)
