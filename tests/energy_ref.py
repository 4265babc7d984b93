"""TEST INFRASTRUCTURE — references for the inverse operational-space inertia and the collision energy
(RigidBodyFrame.inverse_inertia / collision_energy_terms, CollisionEnergyConstraint; libtoppra_b200_dyn.so:
tbd_frame_inverse_inertia / tbd_collision_energy_terms).

* `mp_inverse_inertia`, `mp_energy_b`: 50 digits on the RAW URDF tree of an `rnea_ref.MpRobot` (fixed and locked joints
  stay zero-DOF links, nothing is folded).  M(q) is `MpRobot.mass_matrix` (the Jacobian form, sum of m Jv^T Jv +
  Jw^T I Jw over the links), J_v is `mpmath.diff` of the frame origin's world position (the placements `kin_ref` uses)
  in each joint coordinate, and Lambda_v^-1 = J_v X with X = `mpmath.lu_solve(M, J_v^T)`.  Neither the
  composite-rigid-body algorithm nor a Cholesky factor of the kernels is used.
* `inverse_inertia_packed`, `energy_terms_packed`: a float64 numpy double of the device algorithm (J_v from the chain
  walk, M by the composite-rigid-body algorithm, M = L L^T, Y = L^-1 J_v^T, Lambda_v^-1 = Y^T Y), vectorised over
  points; NaN where a pivot is not positive."""
import mpmath
import numpy as np

import kin_ref
import rnea_ref

DPS = rnea_ref.DPS


# ==== 50-digit reference ==============================================================================================
def mp_inverse_inertia(robot, q, frames):
    """frames: {key: (link, R_off, p_off)} with offsets as float arrays.  Returns {key: (Linv, R)} as mp matrices:
    Lambda_v^-1 in world axes and the frame's world orientation R at q.  Also returns J_v under key (key, "J")."""
    with mpmath.workdps(DPS):
        q = [mpmath.mpf(float(x)) for x in q]
        nv = len(q)
        M = robot.mass_matrix(q)
        offs = {key: (link, mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(Ro)]),
                      mpmath.matrix([mpmath.mpf(float(x)) for x in np.asarray(po)]))
                for key, (link, Ro, po) in frames.items()}
        cache = {}

        def placement(i, t):
            key_t = (i, t, mpmath.mp.prec)
            if key_t not in cache:
                fr = robot._kinematics([q[k] + (t if k == i else 0) for k in range(nv)])[0]
                cache[key_t] = {key: (fr[link][0] * Ro, fr[link][1] + fr[link][0] * po)
                                for key, (link, Ro, po) in offs.items()}
            return cache[key_t]

        out = {}
        zero = mpmath.mpf(0)
        for key in offs:
            J = mpmath.zeros(3, nv)
            for i in range(nv):
                for r in range(3):
                    J[r, i] = mpmath.diff(lambda t, i=i, r=r: placement(i, t)[key][1][r], zero)
            X = mpmath.zeros(nv, 3)
            for c in range(3):
                x = mpmath.lu_solve(M, mpmath.matrix([J[c, i] for i in range(nv)]))
                for i in range(nv):
                    X[i, c] = x[i]
            out[key] = (J * X, placement(0, zero)[key][0])
            out[(key, "J")] = J
        return out


def mp_energy_b(J, Linv, qs, human_mass):
    """b = 1/2 |v|^4 / (|v|^2 / m_H + v^T Linv v), v = J qs, at 50 digits (m_H may be inf)."""
    with mpmath.workdps(DPS):
        v = J * mpmath.matrix([mpmath.mpf(float(x)) for x in qs])
        vv = sum(v[i] ** 2 for i in range(3))
        if vv == 0:
            return mpmath.mpf(0)
        w = (v.T * Linv * v)[0, 0]
        mh = mpmath.inf if np.isinf(human_mass) else mpmath.mpf(float(human_mass))
        return vv * vv / 2 / (vv / mh + w)


# ==== float64 numpy double of the device algorithm =====================================================================
def _inertia3(I6):
    Ixx, Ixy, Ixz, Iyy, Iyz, Izz = I6
    return np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]])


def mass_matrix_packed(packed, q):
    """M(q) (P, nv, nv) by the composite-rigid-body algorithm in body coordinates."""
    packed = np.asarray(packed, dtype=np.float64)
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    P, nv = q.shape
    Rs, ps = rnea_ref._transforms(packed, q)
    body = [packed[3 + 27 * k:3 + 27 * (k + 1)] for k in range(nv)]
    mass, h, Io = [], [], []
    for bd in body:
        c = bd[18:21]
        mass.append(np.full(P, bd[17]))
        h.append(np.broadcast_to(bd[17] * c, (P, 3)).copy())
        Io.append(np.broadcast_to(_inertia3(bd[21:27]) + bd[17] * (c @ c * np.eye(3) - np.outer(c, c)), (P, 3, 3)).copy())
    for k in range(nv - 1, -1, -1):
        par = int(body[k][0])
        if par < 0:
            continue
        R, p = Rs[k], ps[k]
        hr = np.einsum("mij,mj->mi", R, h[k])
        B = np.einsum("mij,mjk,mlk->mil", R, Io[k], R)
        pp = np.einsum("mi,mi->m", p, p)
        ph = np.einsum("mi,mi->m", p, hr)
        m = mass[k][:, None, None]
        Io[par] = Io[par] + B - (m * np.einsum("mi,mj->mij", p, p) + np.einsum("mi,mj->mij", p, hr)
                                 + np.einsum("mi,mj->mij", hr, p)) + (mass[k] * pp + 2 * ph)[:, None, None] * np.eye(3)
        h[par] = h[par] + hr + mass[k][:, None] * p
        mass[par] = mass[par] + mass[k]
    M = np.zeros((P, nv, nv))
    for k in range(nv):
        ax = body[k][2:5]
        if body[k][1] == 0:
            n, f = Io[k] @ ax, rnea_ref._cross_np(np.broadcast_to(ax, (P, 3)), h[k])
        else:
            n, f = rnea_ref._cross_np(h[k], np.broadcast_to(ax, (P, 3))), mass[k][:, None] * ax
        j = k
        while True:
            aj = body[j][2:5]
            M[:, k, j] = M[:, j, k] = (n if body[j][1] == 0 else f) @ aj
            par = int(body[j][0])
            if par < 0:
                break
            Rf = np.einsum("mij,mj->mi", Rs[j], f)
            n = np.einsum("mij,mj->mi", Rs[j], n) + rnea_ref._cross_np(ps[j], Rf)
            f = Rf
            j = par
    return M


def jacobian_packed(packed, frame, q):
    """J_v (P, 3, nv) of the frame origin in world axes, and the frame's world orientation R_f (P, 3, 3)."""
    packed = np.asarray(packed, dtype=np.float64)
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    P, nv = q.shape
    Rs, ps = rnea_ref._transforms(packed, q)
    Rw, pw = np.broadcast_to(np.eye(3), (P, 3, 3)), np.zeros((P, 3))
    cols = []
    for k in kin_ref._chain(packed, frame[0]):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        pw = pw + np.einsum("mij,mj->mi", Rw, ps[k])
        Rw = np.einsum("mij,mjk->mik", Rw, Rs[k])
        cols.append((k, bd[1], Rw @ bd[2:5], pw))
    pf = pw + Rw @ np.asarray(frame[10:13])
    J = np.zeros((P, 3, nv))
    for k, kind, s, o in cols:
        J[:, :, k] = rnea_ref._cross_np(s, pf - o) if kind == 0 else s
    return J, Rw @ np.asarray(frame[1:10]).reshape(3, 3)


def inverse_inertia_packed(packed, frame, q):
    """Double of tbd_frame_inverse_inertia: (P, nv) -> Linv (P, 3, 3) in the frame's reference axes (world for
    TBD_LOCAL_WORLD_ALIGNED, R_f^T (.) R_f for TBD_LOCAL); NaN where a Cholesky pivot is not positive."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    P, nv = q.shape
    M = mass_matrix_packed(packed, q)
    J, Rf = jacobian_packed(packed, frame, q)
    L = np.zeros_like(M)
    bad = np.zeros(P, bool)
    for j in range(nv):
        d = M[:, j, j] - np.sum(L[:, j, :j] ** 2, axis=1)
        bad |= ~(d > 0)
        L[:, j, j] = np.sqrt(np.where(d > 0, d, 1.0))
        for i in range(j + 1, nv):
            L[:, i, j] = (M[:, i, j] - np.sum(L[:, i, :j] * L[:, j, :j], axis=1)) / L[:, j, j]
    Y = np.transpose(J, (0, 2, 1)).copy()
    for i in range(nv):
        Y[:, i] = (Y[:, i] - np.einsum("mk,mkc->mc", L[:, i, :i], Y[:, :i])) / L[:, i, i][:, None]
    W = np.einsum("mir,mic->mrc", Y, Y)
    if int(frame[13]) == 1:
        W = np.einsum("mji,mjk,mkl->mil", Rf, W, Rf)
    W[bad] = np.nan
    return W


def energy_terms_packed(packed, frame, q, qs, human_mass):
    """Double of tbd_collision_energy_terms: b (P,) = 1/2 vv^2 / (vv / m_H + w) with v the world linear velocity of the
    frame origin at (q, qs), vv = v.v, w = v.(Linv v); +0 where vv == 0 and w is not NaN."""
    lwa = np.array(frame, dtype=np.float64)
    lwa[13] = 2.0
    W = inverse_inertia_packed(packed, lwa, q)
    v = kin_ref.frame_velocity_packed(packed, lwa, q, qs)[:, :3]
    vv = v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2]
    Wv = [W[:, i, 0] * v[:, 0] + W[:, i, 1] * v[:, 1] + W[:, i, 2] * v[:, 2] for i in range(3)]
    w = v[:, 0] * Wv[0] + v[:, 1] * Wv[1] + v[:, 2] * Wv[2]
    with np.errstate(invalid="ignore", divide="ignore"):
        b = 0.5 * vv * vv / (vv / human_mass + w)
    return np.where((vv == 0) & ~np.isnan(w), 0.0, b)
