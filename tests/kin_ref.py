"""TEST INFRASTRUCTURE — references for frame velocities (RigidBodyModel.frame, RigidBodyFrame, libtoppra_b200_dyn.so:
tbd_frame_velocity / tbd_velocity_norm_terms).

* `mp_frames`: 50-digit world placements of every link of an `rnea_ref.MpRobot` (its `_kinematics` on the RAW URDF tree:
  fixed and locked joints stay zero-DOF links, nothing is folded), moved by a frame offset, and their time derivatives
  along t -> q + t qd by `mpmath.diff` of the placement.  w comes from dR R^T.  It uses neither the chain recursion of the
  kernel nor a Jacobian formula.
* `frame_packed`, `frame_velocity_packed`, `quad_form`: a float64 numpy double of the packed-frame recursion of the two
  entries (include/toppra_b200_dyn.h), vectorised over points, and the fixed-order quadratic form v^T (S v)."""
import mpmath
import numpy as np

import rnea_ref

DPS = rnea_ref.DPS
REFERENCE_FRAMES = ("world", "local", "local_world_aligned")


# ==== 50-digit reference ==============================================================================================
def _skew_vec(W):
    """The vector of the skew-symmetric part of W."""
    return [(W[2, 1] - W[1, 2]) / 2, (W[0, 2] - W[2, 0]) / 2, (W[1, 0] - W[0, 1]) / 2]


def velocities_mp(R, p, dp, w):
    """[linear; angular] in the three reference frames, from the world placement (R, p), the origin velocity dp and the
    angular velocity w (all mp)."""
    Rt = R.T
    local = list(Rt * mpmath.matrix(dp)) + list(Rt * mpmath.matrix(w))
    wxp = rnea_ref._cross(mpmath.matrix(w), p)
    world = [dp[i] - wxp[i] for i in range(3)] + list(w)
    return {"local_world_aligned": list(dp) + list(w), "local": local, "world": world}


def mp_frames(robot, q, qd, frames):
    """frames: {key: (link, R_off, p_off)} with offsets as float arrays (the frame in link coordinates).  Returns
    {key: dict(R, p, v={reference frame: [6]})} as mp values (R, p the world placement at q)."""
    with mpmath.workdps(DPS):
        q = [mpmath.mpf(float(x)) for x in q]
        qd = [mpmath.mpf(float(x)) for x in qd]
        offs = {key: (link, mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(Ro)]),
                      mpmath.matrix([mpmath.mpf(float(x)) for x in np.asarray(po)]))
                for key, (link, Ro, po) in frames.items()}
        cache = {}

        def placements(t):
            if t not in cache:
                fr = robot._kinematics([q[i] + t * qd[i] for i in range(len(q))])[0]
                cache[t] = {key: (fr[link][0] * Ro, fr[link][1] + fr[link][0] * po) for key, (link, Ro, po) in offs.items()}
            return cache[t]

        out = {}
        zero = mpmath.mpf(0)
        for key in offs:
            R, p = placements(zero)[key]
            dp = [mpmath.diff(lambda t, i=i: placements(t)[key][1][i], zero) for i in range(3)]
            dR = mpmath.matrix(3, 3)
            for i in range(3):
                for j in range(3):
                    dR[i, j] = mpmath.diff(lambda t, i=i, j=j: placements(t)[key][0][i, j], zero)
            w = _skew_vec(dR * R.T)
            out[key] = dict(R=R, p=p, v=velocities_mp(R, p, dp, w))
        return out


# ==== float64 numpy double of the packed-frame recursion ==============================================================
def _chain(packed, body):
    chain, k = [], int(body)
    while k >= 0:
        chain.append(k)
        k = int(packed[3 + 27 * k])
    return chain[::-1]


def frame_packed(packed, frame, q, qd):
    """Double of tbd_frame_velocity: (M, nv) arrays -> (R_f (M, 3, 3), p_f (M, 3), v (M, 6)) with v in the frame's
    reference frame (frame = RigidBodyFrame.packed)."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd))
    M = q.shape[0]
    Rs, ps = rnea_ref._transforms(packed, q)
    Rw, pw = np.broadcast_to(np.eye(3), (M, 3, 3)), np.zeros((M, 3))
    w, vo = np.zeros((M, 3)), np.zeros((M, 3))
    for k in _chain(packed, frame[0]):
        bd = packed[3 + 27 * k:3 + 27 * (k + 1)]
        d = np.einsum("mij,mj->mi", Rw, ps[k])
        vo = vo + rnea_ref._cross_np(w, d)
        pw = pw + d
        Rw = np.einsum("mij,mjk->mik", Rw, Rs[k])
        s = Rw @ bd[2:5]
        if bd[1] == 0:
            w = w + s * qd[:, k:k + 1]
        else:
            vo = vo + s * qd[:, k:k + 1]
    Rfb, pfb = np.asarray(frame[1:10]).reshape(3, 3), np.asarray(frame[10:13])
    d = Rw @ pfb
    pd = vo + rnea_ref._cross_np(w, d)
    pf = pw + d
    Rf = Rw @ Rfb
    ref = REFERENCE_FRAMES[int(frame[13])]
    if ref == "local":
        v = np.concatenate((np.einsum("mji,mj->mi", Rf, pd), np.einsum("mji,mj->mi", Rf, w)), axis=1)
    elif ref == "world":
        v = np.concatenate((pd - rnea_ref._cross_np(w, pf), w), axis=1)
    else:
        v = np.concatenate((pd, w), axis=1)
    return Rf, pf, v


def frame_velocity_packed(packed, frame, q, qd):
    return frame_packed(packed, frame, q, qd)[2]


def quad_form(S, v):
    """v^T (S v) for v (M, 6): S v row by row, then v . (S v), each sum left to right (tbd_velocity_norm_terms)."""
    S = np.asarray(S, dtype=np.float64)
    acc = None
    for i in range(6):
        sv = S[i, 0] * v[:, 0]
        for j in range(1, 6):
            sv = sv + S[i, j] * v[:, j]
        acc = v[:, 0] * sv if i == 0 else acc + v[:, i] * sv
    return acc
