"""TEST INFRASTRUCTURE — references for speed and separation monitoring (SeparationMonitoringConstraint,
RigidBodyModel.separation / separation_terms; libtoppra_b200_dyn.so: tbd_separation / tbd_separation_terms).

* `mp_pairs`, `mp_vmax`, `mp_row`: 50-digit reference on the RAW URDF tree.  Point positions x_p and velocities v1 come
  from `kin_ref.mp_frames` (world placements by `rnea_ref.MpRobot._kinematics`, derivatives by `mpmath.diff`); the
  separation, the approach speed, the stopping speed and the binding pair follow the definitions, with exact square
  roots and divisions at 50 digits.
* `separation_packed`, `vmax_np`, `rows_packed`: a float64 numpy double of the two entries, vectorised over points, in
  the operation order include/toppra_b200_dyn.h documents (the point states from `kin_ref.frame_packed`)."""
import mpmath
import numpy as np

import kin_ref
import rnea_ref

DPS = rnea_ref.DPS


# ==== 50-digit reference ==============================================================================================
def mp_points(robot, q, qd, spec):
    """spec: {key: (link, R_off, p_off)}.  {key: (x (3 mp), v (3 mp))}: world position and linear velocity of the
    frame origin at (q, qd)."""
    fr = kin_ref.mp_frames(robot, q, qd, spec)
    return {key: (list(fr[key]["p"]), fr[key]["v"]["local_world_aligned"][:3]) for key in spec}


def mp_pair(x, v, rp, hs):
    """(d, w) of the point (x, v, radius rp) and the sphere hs = (c, r), 50 digits."""
    with mpmath.workdps(DPS):
        e = [mpmath.mpf(float(hs[j])) - x[j] for j in range(3)]
        l = mpmath.sqrt(sum(ej * ej for ej in e))
        d = l - mpmath.mpf(float(rp)) - mpmath.mpf(float(hs[3]))
        w = mpmath.sqrt(sum(vj * vj for vj in v)) if l == 0 else sum(e[j] * v[j] for j in range(3)) / l
        return d, w


def mp_vmax(d, reaction_time, stopping_deceleration, human_speed, clearance):
    """The largest v_r with v_h (T_r + v_r / a_s) + v_r T_r + v_r^2 / (2 a_s) + C <= d: the positive root of
    v_r^2 / (2 a_s) + (T_r + v_h / a_s) v_r - D = 0, D = d - C - v_h T_r, by the quadratic formula; 0 where D <= 0."""
    with mpmath.workdps(DPS):
        Tr, a, vh, C = (mpmath.mpf(float(x)) for x in (reaction_time, stopping_deceleration, human_speed, clearance))
        D = d - C - vh * Tr
        if D <= 0:
            return mpmath.mpf(0)
        p = Tr + vh / a
        return a * (-p + mpmath.sqrt(p * p + 2 * D / a))


def mp_row(pairs, params):
    """(b, c) of the constraint from [(d, w)] in pair order: the pair with w > 0 minimising vmax^2 / w^2 (the first on
    ties); (0, -1) where none approaches."""
    best = None
    with mpmath.workdps(DPS):
        for d, w in pairs:
            if w > 0:
                vm = mp_vmax(d, *params)
                ratio = vm * vm / (w * w)
                if best is None or ratio < best[0]:
                    best = (ratio, w * w, vm * vm)
        if best is None:
            return mpmath.mpf(0), mpmath.mpf(-1)
        return best[1], -best[2]


# ==== float64 numpy double =============================================================================================
def point_states_packed(packed, points, q, qd):
    """x, v (M, P, 3): world position and linear velocity of every packed point (P, 15) at (M, nv) states."""
    xs, vs = [], []
    for row in np.asarray(points, dtype=np.float64):
        frame = row[:14].copy()
        frame[13] = 2.0                                   # local_world_aligned: the linear part is dp_f
        _, pf, v = kin_ref.frame_packed(packed, frame, q, qd)
        xs.append(pf)
        vs.append(v[:, :3])
    return np.stack(xs, axis=1), np.stack(vs, axis=1)


def separation_packed(packed, points, humans, q, qd, points_per_path=0):
    """Double of tbd_separation: (d, w), each (M, P, H).  humans (NH, H, 4) or (H, 4)."""
    q, qd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd))
    M = q.shape[0]
    hum = np.asarray(humans, dtype=np.float64)
    hum = hum[None] if hum.ndim == 2 else hum
    sets = np.arange(M) // points_per_path if points_per_path > 0 else np.zeros(M, int)
    hs = hum[sets]                                        # (M, H, 4)
    x, v = point_states_packed(packed, points, q, qd)     # (M, P, 3)
    rp = np.asarray(points, dtype=np.float64)[:, 14]
    e = hs[:, None, :, :3] - x[:, :, None, :]             # (M, P, H, 3)
    l = np.sqrt(e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1] + e[..., 2] * e[..., 2])
    d = l - rp[None, :, None] - hs[:, None, :, 3]
    vv = v[:, :, None, :]
    speed = np.sqrt(vv[..., 0] * vv[..., 0] + vv[..., 1] * vv[..., 1] + vv[..., 2] * vv[..., 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.where(l == 0, speed, (e[..., 0] * vv[..., 0] + e[..., 1] * vv[..., 1] + e[..., 2] * vv[..., 2]) / l)
    return d, w


def vmax_np(d, reaction_time, stopping_deceleration, human_speed, clearance):
    """vmax of every separation d, in the documented operation order."""
    vhTr, twoa = human_speed * reaction_time, 2.0 * stopping_deceleration
    k = stopping_deceleration * reaction_time + human_speed
    kk = k * k
    D = d - clearance
    D = D - vhTr
    num = twoa * D
    with np.errstate(invalid="ignore"):
        return np.where(D <= 0, 0.0, num / (np.sqrt(kk + num) + k))


def rows_from_pairs(d, w, params):
    """(b, c) (M,) from the pairs (M, P, H), in the documented order of tbd_separation_terms."""
    M = d.shape[0]
    d, w = d.reshape(M, -1), w.reshape(M, -1)
    vm = vmax_np(d, *params)
    bw2, bv2 = np.zeros(M), np.zeros(M)
    found, bad = np.zeros(M, bool), np.zeros(M, bool)
    for j in range(d.shape[1]):
        bad |= np.isnan(w[:, j]) | np.isnan(vm[:, j])
        w2, v2 = w[:, j] * w[:, j], vm[:, j] * vm[:, j]
        with np.errstate(invalid="ignore"):
            take = (w[:, j] > 0) & (~found | (v2 * bw2 < bv2 * w2))
        bw2, bv2 = np.where(take, w2, bw2), np.where(take, v2, bv2)
        found |= take
    b = np.where(found, bw2, 0.0)
    c = np.where(found, 0.0 - bv2, -1.0)
    return np.where(bad, np.nan, b), np.where(bad, np.nan, c)


def rows_packed(packed, points, humans, params, q, qs, points_per_path=0):
    """Double of tbd_separation_terms: (b, c), each (M,).  params = (T_r, a_s, v_h, C)."""
    d, w = separation_packed(packed, points, humans, q, qs, points_per_path)
    return rows_from_pairs(d, w, params)
