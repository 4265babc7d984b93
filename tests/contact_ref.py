"""TEST INFRASTRUCTURE — references for contact wrenches (ContactStabilityConstraint, RigidBodyFrame.contact_wrench /
contact_wrench_terms, libtoppra_b200_dyn.so: tbd_contact_wrench / tbd_contact_wrench_terms).

* `mp_wrenches`: 50-digit wrenches that contact frames of an `rnea_ref.MpRobot` (its `_kinematics` on the RAW URDF tree:
  fixed and locked joints stay zero-DOF links, nothing is folded), moved by a frame offset, exert on a carried object,
  along t -> q + t qd + t^2/2 qdd.  The frame's world orientation R(t) and the object's centre-of-mass position p(t) are
  differentiated with `mpmath.diff`; then, in world axes,
      f = m (p'' - g),   tau_com = d/dt (R Ic R^T w) = R' Ic R^T w + R Ic R'^T w + R Ic R^T w',
  with w = vee(R' R^T) and w' = vee(R'' R^T) (R' R'^T is symmetric), the rate of change of the angular momentum about
  the centre of mass, written out from R, R', R'' (not Euler's equation).  Both are rotated into contact axes (R^T)
  and the moment is moved to the contact origin: tau = tau_com + r x f.  It uses neither the chain recursion of the
  kernel nor a Jacobian formula.
* `contact_wrench_packed`, `contact_terms_packed`: a float64 numpy double of the device recursion of the two entries
  (include/toppra_b200_dyn.h), vectorised over points."""
import mpmath
import numpy as np

import kin_acc_ref
import kin_ref
import rnea_ref

DPS = rnea_ref.DPS


def object_packed(mass, com, inertia):
    """The packed object of include/toppra_b200_dyn.h: m, r (3), Ic (6) = Ixx, Ixy, Ixz, Iyy, Iyz, Izz."""
    return np.concatenate(([float(mass)], np.asarray(com, dtype=np.float64), np.asarray(inertia, dtype=np.float64)))


def _inertia_matrix(I6):
    Ixx, Ixy, Ixz, Iyy, Iyz, Izz = I6
    return [[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]]


# ==== 50-digit reference ==============================================================================================
def mp_wrenches(robot, q, qd, qdd, frames, obj):
    """frames: {key: (link, R_off, p_off)} with offsets as float arrays (the contact frame in link coordinates); obj the
    packed object.  Returns {key: [6] mp}: [f; tau] in contact axes at the contact origin."""
    with mpmath.workdps(DPS):
        q, qd, qdd = ([mpmath.mpf(float(x)) for x in v] for v in (q, qd, qdd))
        m = mpmath.mpf(float(obj[0]))
        r = mpmath.matrix([mpmath.mpf(float(x)) for x in obj[1:4]])
        Ic = mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in _inertia_matrix(obj[4:10])])
        offs = {key: (link, mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(Ro)]),
                      mpmath.matrix([mpmath.mpf(float(x)) for x in np.asarray(po)]))
                for key, (link, Ro, po) in frames.items()}
        cache = {}

        def placements(t):
            # (R, centre-of-mass position) of every contact frame; keyed by the working precision too, as in
            # kin_acc_ref (mpmath.diff evaluates t = 0 at a raised precision)
            key_t = (t, mpmath.mp.prec)
            if key_t not in cache:
                fr = robot._kinematics([q[i] + t * qd[i] + t * t / 2 * qdd[i] for i in range(len(q))])[0]
                out = {}
                for key, (link, Ro, po) in offs.items():
                    R = fr[link][0] * Ro
                    out[key] = (R, fr[link][1] + fr[link][0] * po + R * r)
                cache[key_t] = out
            return cache[key_t]

        out = {}
        zero = mpmath.mpf(0)
        for key in offs:
            R, _ = placements(zero)[key]
            ddp = mpmath.matrix([mpmath.diff(lambda t, i=i: placements(t)[key][1][i], zero, 2) for i in range(3)])
            dR, ddR = mpmath.matrix(3, 3), mpmath.matrix(3, 3)
            for i in range(3):
                for j in range(3):
                    dR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[key][0][i, j], zero, 1)
                    ddR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[key][0][i, j], zero, 2)
            w = mpmath.matrix(kin_ref._skew_vec(dR * R.T))
            dw = mpmath.matrix(kin_ref._skew_vec(ddR * R.T))
            f = m * (ddp - robot.g)
            tau_com = dR * Ic * R.T * w + R * Ic * dR.T * w + R * Ic * R.T * dw
            fl, tl = R.T * f, R.T * tau_com
            out[key] = list(fl) + list(tl + rnea_ref._cross(r, fl))
        return out


# ==== float64 numpy double of the device recursion ====================================================================
def _local(frame):
    f = np.array(frame, dtype=np.float64)
    f[13] = 1.0                                  # the wrench is in the frame's own axes, whatever its reference frame
    return f


def contact_wrench_packed(packed, frame, obj, q, qd, qdd):
    """Double of tbd_contact_wrench: (M, nv) arrays -> w (M, 6) = [f; tau] in contact axes at the contact origin."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    fl = _local(frame)
    acc = kin_acc_ref.frame_acceleration_packed(packed, fl, q, qd, qdd)    # [a_f; dw], frame axes
    Rf, _, v = kin_ref.frame_packed(packed, fl, q, qd)                     # v[:, 3:] = Rf^T w
    wl = v[:, 3:]
    gl = np.einsum("mji,j->mi", Rf, packed[:3])
    cross = rnea_ref._cross_np
    M = q.shape[0]
    r = np.broadcast_to(np.asarray(obj[1:4], dtype=np.float64), (M, 3))
    I = np.asarray(_inertia_matrix(obj[4:10]), dtype=np.float64)
    a_f, dw = acc[:, :3], acc[:, 3:]
    f = obj[0] * (a_f + cross(dw, r) + cross(wl, cross(wl, r)) - gl)
    tau = dw @ I.T + cross(wl, wl @ I.T) + cross(r, f)
    return np.concatenate((f, tau), axis=1)


def contact_terms_packed(packed, frame, obj, q, qs, qss):
    """Double of tbd_contact_wrench_terms: c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    zero = np.zeros_like(q)
    c = contact_wrench_packed(packed, frame, obj, q, zero, zero)
    a = contact_wrench_packed(packed, frame, obj, q, zero, qs) - c
    b = contact_wrench_packed(packed, frame, obj, q, qs, qss) - c
    return a, b, c
