"""TEST INFRASTRUCTURE — references for speed and separation monitoring with capsules (SeparationMonitoringConstraint
with capsules, RigidBodyModel.separation / separation_terms; libtoppra_b200_dyn.so: tbd_capsule_separation /
tbd_capsule_separation_terms).

* `mp_capsule_pair`: 50-digit reference.  The endpoint positions and velocities come from `separation_ref.mp_points`
  (`kin_ref.mp_frames` on the RAW URDF tree).  The closest pair is found by an algorithm independent of the kernels':
  the squared distance |r0 + t d1 - tau d2|^2 is a convex quadratic on the unit square, minimised by checking the
  interior stationary point, the minimum on each of the four edges and the corners.  Where the minimum is not unique
  (parallel segments), d is the minimum and w the largest approach speed over the set of minimisers (Danskin).
  `mp_fd_speed` is a one-sided finite difference of that distance at 50 digits, with the endpoints moved along their
  velocities: it must equal -w, which checks the envelope argument itself.
* `capsule_pair_np`, `capsule_separation_packed`, `capsule_rows_packed`: a float64 double of the two entries in the
  operation order of include/toppra_b200_dyn.h (Python floats are IEEE doubles; math.sqrt is correctly rounded), the
  endpoint states from `kin_ref.frame_packed`."""
import math

import mpmath
import numpy as np

import separation_ref as sr

DPS = sr.DPS
PARALLEL = 1e-12              # TBD_CAPSULE_PARALLEL
FRAME = 14


# ==== 50-digit reference ==============================================================================================
def _mp(x):
    return [mpmath.mpf(float(v)) if not isinstance(v, mpmath.mpf) else v for v in x]


def _dot(a, b):
    return sum(x * y for x, y in zip(a, b))


def _minimisers(xa, xb, c0, c1):
    """[(t, tau)] minimising |h(tau) - p(t)|^2 on the unit square (all of them, up to 1e-40 of the scale), and the
    minimum."""
    d1 = [xb[j] - xa[j] for j in range(3)]
    d2 = [c1[j] - c0[j] for j in range(3)]
    r0 = [xa[j] - c0[j] for j in range(3)]

    def F(t, tau):
        r = [r0[j] + t * d1[j] - tau * d2[j] for j in range(3)]
        return _dot(r, r)

    a, e, b = _dot(d1, d1), _dot(d2, d2), _dot(d1, d2)
    c, f = _dot(d1, r0), _dot(d2, r0)
    clamp = lambda x: min(max(x, mpmath.mpf(0)), mpmath.mpf(1))  # noqa: E731
    cands = [(mpmath.mpf(t), mpmath.mpf(u)) for t in (0, 1) for u in (0, 1)]
    det = a * e - b * b
    if det > 0:                               # interior stationary point of the quadratic
        t = (b * f - c * e) / det
        u = (a * f - b * c) / det
        if 0 <= t <= 1 and 0 <= u <= 1:
            cands.append((t, u))
    for t in (mpmath.mpf(0), mpmath.mpf(1)):  # edges t = 0, 1: the best tau
        if e > 0:
            cands.append((t, clamp((b * t + f) / e)))
    for u in (mpmath.mpf(0), mpmath.mpf(1)):  # edges tau = 0, 1: the best t
        if a > 0:
            cands.append((clamp((b * u - c) / a), u))
    vals = [F(t, u) for t, u in cands]
    fmin = min(vals)
    scale = 1 + _dot(r0, r0) + a + e
    return [cu for cu, v in zip(cands, vals) if v - fmin <= mpmath.mpf(10) ** -40 * scale], fmin


def mp_capsule_pair(xa, va, xb, vb, rp, hc):
    """(d, w) of the robot capsule (endpoints xa, xb with velocities va, vb, radius rp) and the human capsule
    hc = (c0, c1, r_h), 50 digits."""
    with mpmath.workdps(DPS):
        xa, va, xb, vb = (_mp(x) for x in (xa, va, xb, vb))
        c0, c1 = _mp(hc[:3]), _mp(hc[3:6])
        sets, fmin = _minimisers(xa, xb, c0, c1)
        l = mpmath.sqrt(fmin)
        d = l - mpmath.mpf(float(rp)) - mpmath.mpf(float(hc[6]))
        ws = []
        for t, u in sets:
            E = [c0[j] + u * (c1[j] - c0[j]) - xa[j] - t * (xb[j] - xa[j]) for j in range(3)]
            v = [va[j] + t * (vb[j] - va[j]) for j in range(3)]
            ws.append(mpmath.sqrt(_dot(v, v)) if l == 0 else _dot(E, v) / l)
        return d, max(ws)


def mp_fd_speed(xa, va, xb, vb, hc, h=mpmath.mpf(10) ** -25):
    """-(dist(s = h) - dist(0)) / h with the endpoints at x + s v: the one-sided rate at which the distance closes."""
    with mpmath.workdps(DPS):
        xa, va, xb, vb = (_mp(x) for x in (xa, va, xb, vb))
        c0, c1 = _mp(hc[:3]), _mp(hc[3:6])
        l0 = mpmath.sqrt(_minimisers(xa, xb, c0, c1)[1])
        xa1 = [xa[j] + h * va[j] for j in range(3)]
        xb1 = [xb[j] + h * vb[j] for j in range(3)]
        l1 = mpmath.sqrt(_minimisers(xa1, xb1, c0, c1)[1])
        return -(l1 - l0) / h


def mp_capsule_pairs(robot, q, qd, spec, humans):
    """spec: [((link_a, R_a, p_a), (link_b, R_b, p_b), r_p)].  [[(d, w)] per human] per capsule, 50 digits."""
    frames = {}
    for i, (fa, fb, _) in enumerate(spec):
        frames[2 * i], frames[2 * i + 1] = fa, fb
    st = sr.mp_points(robot, q, qd, frames)
    return [[mp_capsule_pair(st[2 * i][0], st[2 * i][1], st[2 * i + 1][0], st[2 * i + 1][1], spec[i][2], h)
             for h in humans] for i in range(len(spec))]


# ==== float64 numpy double =============================================================================================
def _clamp(x):
    return 0.0 if x < 0.0 else (1.0 if x > 1.0 else x)


def _sep(p, v, rp, hs):
    """separation_pair of include/toppra_b200_dyn.h (tbd_separation)."""
    e = [hs[0] - p[0], hs[1] - p[1], hs[2] - p[2]]
    l = math.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
    d = l - rp - hs[3]
    if l == 0.0:
        w = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    else:
        w = (e[0] * v[0] + e[1] * v[1] + e[2] * v[2]) / l
    return d, w


def capsule_pair_np(xa, va, xb, vb, rp, hc):
    """(d, w) of one pair in the documented float64 operation order."""
    xa, va, xb, vb, hc = ([float(z) for z in x] for x in (xa, va, xb, vb, hc))
    rp = float(rp)
    if any(math.isnan(z) for z in xa + va + xb + vb):
        return math.nan, math.nan
    d1 = [xb[j] - xa[j] for j in range(3)]
    d2 = [hc[3 + j] - hc[j] for j in range(3)]
    r0 = [xa[j] - hc[j] for j in range(3)]
    a = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]
    e = d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2]
    f = d2[0] * r0[0] + d2[1] * r0[1] + d2[2] * r0[2]
    t = tau = 0.0
    pairs = None
    if a == 0.0:
        if e != 0.0:
            tau = _clamp(f / e)
    else:
        c = d1[0] * r0[0] + d1[1] * r0[1] + d1[2] * r0[2]
        if e == 0.0:
            t = _clamp(-c / a)
        else:
            b = d1[0] * d2[0] + d1[1] * d2[1] + d1[2] * d2[2]
            denom = a * e - b * b
            general = True
            if denom <= PARALLEL * a * e:
                t0, t1 = -c / a, (b - c) / a
                lo, hi = max(min(t0, t1), 0.0), min(max(t0, t1), 1.0)
                if lo <= hi:
                    pairs = [(lo, _clamp((b * lo + f) / e)), (hi, _clamp((b * hi + f) / e))]
                    general = False
            else:
                t = _clamp((b * f - c * e) / denom)
            if general:
                tau = (b * t + f) / e
                if tau < 0.0:
                    tau, t = 0.0, _clamp(-c / a)
                elif tau > 1.0:
                    tau, t = 1.0, _clamp((b - c) / a)
    out = []
    for t, tau in (pairs or [(t, tau)]):
        p = [xa[j] + t * d1[j] for j in range(3)]
        v = [va[j] + t * (vb[j] - va[j]) for j in range(3)]
        hs = [hc[j] + tau * d2[j] for j in range(3)] + [hc[6]]
        out.append(_sep(p, v, rp, hs))
    d, w = out[0]
    for d2_, w2_ in out[1:]:
        d = d2_ if d2_ < d else d
        w = w2_ if w2_ > w else w
    return d, w


def endpoint_states(packed, capsules, q, qd):
    """xa, va, xb, vb (M, P, 3) of packed capsules (P, 29) at (M, nv) states."""
    caps = np.asarray(capsules, dtype=np.float64)
    ends = [np.r_[row[:FRAME], 0.0] for row in caps] + [np.r_[row[FRAME:2 * FRAME], 0.0] for row in caps]
    x, v = sr.point_states_packed(packed, np.array(ends), q, qd)
    P = caps.shape[0]
    return x[:, :P], v[:, :P], x[:, P:], v[:, P:]


def capsule_separation_packed(packed, capsules, humans, q, qd, points_per_path=0):
    """Double of tbd_capsule_separation: (d, w), each (M, P, H).  humans (NH, H, 7) or (H, 7)."""
    q, qd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd))
    M = q.shape[0]
    hum = np.asarray(humans, dtype=np.float64)
    hum = hum[None] if hum.ndim == 2 else hum
    sets = np.arange(M) // points_per_path if points_per_path > 0 else np.zeros(M, int)
    caps = np.asarray(capsules, dtype=np.float64)
    xa, va, xb, vb = endpoint_states(packed, caps, q, qd)
    P, H = caps.shape[0], hum.shape[1]
    d, w = np.empty((M, P, H)), np.empty((M, P, H))
    for m in range(M):
        for i in range(P):
            for h in range(H):
                d[m, i, h], w[m, i, h] = capsule_pair_np(xa[m, i], va[m, i], xb[m, i], vb[m, i], caps[i, 2 * FRAME],
                                                         hum[sets[m], h])
    return d, w


def capsule_rows_packed(packed, capsules, humans, params, q, qs, points_per_path=0):
    """Double of tbd_capsule_separation_terms: (b, c), each (M,).  params = (T_r, a_s, v_h, C)."""
    d, w = capsule_separation_packed(packed, capsules, humans, q, qs, points_per_path)
    return sr.rows_from_pairs(d, w, params)
