"""TEST INFRASTRUCTURE — references for frame accelerations (RigidBodyFrame.acceleration / acceleration_terms,
libtoppra_b200_dyn.so: tbd_frame_acceleration / tbd_acceleration_terms).

* `mp_accelerations`: 50-digit classical accelerations of frames of an `rnea_ref.MpRobot` (its `_kinematics` on the RAW
  URDF tree: fixed and locked joints stay zero-DOF links, nothing is folded), moved by a frame offset, along
  t -> q + t qd + t^2/2 qdd: the origin's acceleration is `mpmath.diff(p, 0, 2)`, the angular acceleration the vector of
  R'' R^T (R' R'^T is symmetric, so the skew part of R'' R^T is that of d/dt (R' R^T)), and "local" multiplies both by
  R^T.  It uses neither the chain recursion of the kernel nor a Jacobian formula.
* `frame_acceleration_packed`, `acceleration_terms_packed`: a float64 numpy double of the packed-frame recursion of the
  two entries (include/toppra_b200_dyn.h), vectorised over points."""
import mpmath
import numpy as np

import kin_ref
import rnea_ref

DPS = rnea_ref.DPS
REFERENCE_FRAMES = ("local", "local_world_aligned")


# ==== 50-digit reference ==============================================================================================
def mp_accelerations(robot, q, qd, qdd, frames):
    """frames: {key: (link, R_off, p_off)} with offsets as float arrays (the frame in link coordinates).  Returns
    {key: {reference frame: [6] mp}}: [linear; angular] classical accelerations at (q, qd, qdd)."""
    with mpmath.workdps(DPS):
        q, qd, qdd = ([mpmath.mpf(float(x)) for x in v] for v in (q, qd, qdd))
        offs = {key: (link, mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(Ro)]),
                      mpmath.matrix([mpmath.mpf(float(x)) for x in np.asarray(po)]))
                for key, (link, Ro, po) in frames.items()}
        cache = {}

        def placements(t):
            # keyed by the working precision too: the central second difference evaluates t = 0 at a raised precision,
            # where the placement at DPS digits would be divided by h^2
            key_t = (t, mpmath.mp.prec)
            if key_t not in cache:
                fr = robot._kinematics([q[i] + t * qd[i] + t * t / 2 * qdd[i] for i in range(len(q))])[0]
                cache[key_t] = {key: (fr[link][0] * Ro, fr[link][1] + fr[link][0] * po)
                                for key, (link, Ro, po) in offs.items()}
            return cache[key_t]

        out = {}
        zero = mpmath.mpf(0)
        for key in offs:
            R, _ = placements(zero)[key]
            ddp = mpmath.matrix([mpmath.diff(lambda t, i=i: placements(t)[key][1][i], zero, 2) for i in range(3)])
            ddR = mpmath.matrix(3, 3)
            for i in range(3):
                for j in range(3):
                    ddR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[key][0][i, j], zero, 2)
            dw = mpmath.matrix(kin_ref._skew_vec(ddR * R.T))
            out[key] = {"local_world_aligned": list(ddp) + list(dw), "local": list(R.T * ddp) + list(R.T * dw)}
        return out


# ==== float64 numpy double of the packed-frame recursion ==============================================================
def frame_acceleration_packed(packed, frame, q, qd, qdd):
    """Double of tbd_frame_acceleration: (M, nv) arrays -> acc (M, 6) in the frame's reference frame (frame =
    RigidBodyFrame.packed, reference frame "local" or "local_world_aligned")."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    M = q.shape[0]
    Rs, ps = rnea_ref._transforms(packed, q)
    cross = rnea_ref._cross_np
    Rw = np.broadcast_to(np.eye(3), (M, 3, 3))
    w, dw, ao = np.zeros((M, 3)), np.zeros((M, 3)), np.zeros((M, 3))
    for k in kin_ref._chain(packed, frame[0]):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        d = np.einsum("mij,mj->mi", Rw, ps[k])
        ao = ao + cross(dw, d) + cross(w, cross(w, d))
        Rw = np.einsum("mij,mjk->mik", Rw, Rs[k])
        s = Rw @ bd[2:5]
        sq = s * qd[:, k:k + 1]
        c = cross(w, sq)
        if bd[1] == 0:
            dw = dw + s * qdd[:, k:k + 1] + c
            w = w + sq
        else:
            ao = ao + s * qdd[:, k:k + 1] + 2.0 * c
    Rfb, pfb = np.asarray(frame[1:10]).reshape(3, 3), np.asarray(frame[10:13])
    d = Rw @ pfb
    af = ao + cross(dw, d) + cross(w, cross(w, d))
    ref = kin_ref.REFERENCE_FRAMES[int(frame[13])]
    if ref == "local":
        Rf = Rw @ Rfb
        return np.concatenate((np.einsum("mji,mj->mi", Rf, af), np.einsum("mji,mj->mi", Rf, dw)), axis=1)
    assert ref == "local_world_aligned", ref
    return np.concatenate((af, dw), axis=1)


def acceleration_terms_packed(packed, frame, q, qs, qss, components):
    """Double of tbd_acceleration_terms: a = acc(q, 0, qs), b = acc(q, qs, qss), columns `components` (sorted)."""
    cols = sorted(components)
    a = frame_acceleration_packed(packed, frame, q, np.zeros_like(np.atleast_2d(q)), qs)
    b = frame_acceleration_packed(packed, frame, q, qs, qss)
    return a[:, cols], b[:, cols]
