"""TEST INFRASTRUCTURE — references for the kinetic energy and the linear momentum of the whole robot
(RigidBodyModel.energy_momentum / energy_momentum_terms, KineticEnergyConstraint, MomentumConstraint;
libtoppra_b200_dyn.so: tbd_energy_momentum / tbd_energy_momentum_terms).

* `mp_energy_momentum`: 50 digits on the RAW URDF tree of an `rnea_ref.MpRobot` (fixed and locked joints stay zero-DOF
  links, nothing is folded), independent of the kernels' recursion: T = 1/2 qd^T M(q) qd with M from
  `MpRobot.mass_matrix` (the Jacobian form), and p = sum_l m_l J_cl qd with each link's centre-of-mass Jacobian J_cl
  taken by `mpmath.diff` of its centre-of-mass world position in each joint coordinate.
* `energy_momentum_packed`, `energy_momentum_terms_packed`: a float64 numpy double of the device algorithm (one forward
  walk of the bodies in order, each body's centre-of-mass velocity and body-axis angular velocity, every sum in body
  order and left to right), vectorised over points."""
import mpmath
import numpy as np

import rnea_ref

DPS = rnea_ref.DPS


# ==== 50-digit reference ==============================================================================================
def mp_energy_momentum(robot, q, qd):
    """(T, p (3,)) of the robot at (q, qd) as mpf values; p in base axes."""
    with mpmath.workdps(DPS):
        q = [mpmath.mpf(float(x)) for x in q]
        qd = mpmath.matrix([mpmath.mpf(float(x)) for x in qd])
        nv = len(q)
        T = (qd.T * robot.mass_matrix(q) * qd)[0, 0] / 2
        cache = {}

        def com_positions(i, t):
            key = (i, t, mpmath.mp.prec)
            if key not in cache:
                frames = robot._kinematics([q[k] + (t if k == i else 0) for k in range(nv)])[0]
                cache[key] = {name: frames[name][1] + frames[name][0] * inert[1]
                              for name, inert in robot.links.items() if inert is not None and name in frames}
            return cache[key]

        zero = mpmath.mpf(0)
        p = [mpmath.mpf(0)] * 3
        for name, inert in robot.links.items():
            if inert is None or name not in com_positions(0, zero):
                continue
            for i in range(nv):
                if qd[i] == 0:
                    continue
                for r in range(3):
                    dr = mpmath.diff(lambda t, i=i, r=r: com_positions(i, t)[name][r], zero)
                    p[r] += inert[0] * dr * qd[i]
        return T, p


def mp_energy_momentum64(robot, q, qd):
    """mp_energy_momentum rounded to float64: (T, p (3,))."""
    T, p = mp_energy_momentum(robot, q, qd)
    return float(T), np.array([float(x) for x in p])


# ==== float64 numpy double of the device algorithm =====================================================================
def _inertia3(I6):
    Ixx, Ixy, Ixz, Iyy, Iyz, Izz = I6
    return np.array([[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]])


def energy_momentum_packed(packed, q, qd):
    """Double of tbd_energy_momentum: (P, nv) arrays -> (T (P,), p (P, 3))."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd))
    P, nv = q.shape
    Rs, ps = rnea_ref._transforms(packed, q)
    Rw, w, vo = [], [], []
    e, p = np.zeros(P), np.zeros((P, 3))
    for k in range(nv):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        par = int(bd[0])
        if par < 0:
            Rp, wp, vp = np.broadcast_to(np.eye(3), (P, 3, 3)), np.zeros((P, 3)), np.zeros((P, 3))
        else:
            Rp, wp, vp = Rw[par], w[par], vo[par]
        d = np.einsum("mij,mj->mi", Rp, ps[k])
        v = vp + rnea_ref._cross_np(wp, d)
        R = np.einsum("mij,mjk->mik", Rp, Rs[k])
        s = np.einsum("mij,j->mi", R, bd[2:5])
        if bd[1] == 0:
            wk = wp + s * qd[:, k:k + 1]
        else:
            wk, v = wp, v + s * qd[:, k:k + 1]
        Rw.append(R)
        w.append(wk)
        vo.append(v)
        vc = v + rnea_ref._cross_np(wk, np.einsum("mij,j->mi", R, bd[18:21]))
        wb = np.einsum("mji,mj->mi", R, wk)
        Iwb = wb @ _inertia3(bd[21:27]).T
        vv = vc[:, 0] * vc[:, 0] + vc[:, 1] * vc[:, 1] + vc[:, 2] * vc[:, 2]
        ww = wb[:, 0] * Iwb[:, 0] + wb[:, 1] * Iwb[:, 1] + wb[:, 2] * Iwb[:, 2]
        e = e + (bd[17] * vv + ww)
        p = p + bd[17] * vc
    return 0.5 * e, p


def momentum_squared(p):
    """(px px + py py) + pz pz of p (P, 3), the b of MomentumConstraint."""
    return p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]


def energy_momentum_terms_packed(packed, q, qs, which):
    """Double of tbd_energy_momentum_terms: b (P,) = T(q, qs) (which "energy") or |p(q, qs)|^2 ("momentum")."""
    T, p = energy_momentum_packed(packed, q, qs)
    return T if which == "energy" else momentum_squared(p)
