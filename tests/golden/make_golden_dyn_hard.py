"""Regenerate tests/golden/dyn_hard_trees.npz: 50-digit references of every model-taking entry of libtoppra_b200_dyn.so
on the hard model families of tests/dyn_hard.py (16-deep chains, stars, brooms, badly scaled links, planar, prismatic
and R/P chains) at fast, wound-up and stretched states, with a tolerance per output component.

    python tests/golden/make_golden_dyn_hard.py        (a few minutes on 8 cores; the output is byte-identical)

The references are the existing independent 50-digit code of tests/*_ref.py on `MpRobot.from_packed` (Lagrangian
inverse dynamics, mpmath.diff of world placements, the reduced Lagrangian of a coupling); the difference entries
(a = w(q, 0, q') - w(q, 0, 0) and the others) are formed at 50 digits before rounding.

Tolerance of output component i:  tol_i = 32 (sens_i + eps mag_i + spread_i), eps = 2^-52, where
* sens_i is the largest change of the 50-digit result when the float64 inputs (the model's real parameters, q, qd and
  qdd) move by one ulp, in four seeded random sign patterns (`perturbed`): what the output owes to the conditioning
  of the problem itself (a wound-up q of 1e3 rad, a torque next to a 1e6 times heavier link, a near-singular M(q)).
  For a difference entry it is the sum of the changes of its two terms, which the kernels compute and round apart.
* mag_i is the output's own magnitude: the length of the 3-vector it is a component of (a linear or angular velocity
  or acceleration, a force, a moment, a momentum; rotations mix their components), the Frobenius norm of Lambda_v^-1,
  |x| of a joint torque or a scalar, |w1| + |w0| for a difference w1 - w0, |v|^T |S| |v| for a quadratic form; for a
  separation l + r_p + r_h plus, for capsules, the endpoints' distances from the origin (the closest points are
  interpolated between them); |v| for an approach speed (times 1 + those distances / l for capsules).  Never the
  scale of the whole state.
* spread_i is how far Monte Carlo arithmetic (every floating-point result of the numpy double multiplied by
  1 + u, |u| <= 2^-53, six seeded runs; `_MC`) moves the output: the rounding of the large intermediate quantities
  an output can be a small remainder of (the 1e4 m/s^2 acceleration of a 1 g link whose torque is 1e-5 N m).
The constant 32 leaves room over the float64 numpy doubles of tests/*_ref.py, whose worst error on this fixture is
a small fraction of the tolerance (test_dyn_hard_trees.py reports it per entry)."""
import io
import multiprocessing
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import capsule_ref as cr  # noqa: E402
import contact_ref  # noqa: E402
import coupled_ref  # noqa: E402
import drive_ref  # noqa: E402
import dyn_hard  # noqa: E402
import energy_ref  # noqa: E402
import joint_wrench_ref as jr  # noqa: E402
import kin_acc_ref  # noqa: E402
import kin_ref  # noqa: E402
import momentum_ref  # noqa: E402
import rnea_ref as rr  # noqa: E402
import separation_ref as sr  # noqa: E402
import support_ref  # noqa: E402

OUT = os.path.join(HERE, "dyn_hard_trees.npz")
DIRECTIONS = 4
C_TOL = 32.0
EPS = 2.0 ** -52
OFFSET_XYZ, OFFSET_RPY = (0.03, -0.02, 0.1), (0.3, -0.2, 0.5)        # dyn_common.OFFSET
OBJECT = np.array([0.8, 0.006, -0.004, 0.06, 0.0021, 0.0001, -0.0002, 0.0026, 0.0001, 0.0017])
BASE = np.array([12.0, 0.01, -0.02, 0.1])
SUPPORT = (-1, (0.1, -0.05, 0.2), (0.01, 0.02, 0.0))
HUMAN_MASS = 40.0
SEPARATION = (0.1, 2.5, 1.6, 0.05)            # T_r, a_s, v_h, C
P_POINTS, H_HUMANS, P_CAPSULES, H_CAPSULES = 16, 16, 6, 16
COUPLED = ("chain8", "chain16")                # a mimic joint: the last body follows the one before it
WORLD, LOCAL, LWA = 0, 1, 2


def rpy(v):
    from toppra_b200.dynamics import rpy_matrix
    return rpy_matrix(np.asarray(v, dtype=np.float64))


def frame_row(body, R, p, ref):
    return np.concatenate(([float(body)], np.asarray(R, dtype=np.float64).reshape(9), np.asarray(p, dtype=np.float64),
                           [float(ref)]))


def chain_of(packed, body):
    out = []
    while body >= 0:
        out.insert(0, body)
        body = int(packed[3 + 27 * body])
    return out


def setup(name):
    """Everything a case feeds the entries besides the model and the states, from the case's seed."""
    packed, q, qd, qdd = dyn_hard.case_model(name)
    nv = q.shape[1]
    rng = np.random.RandomState(dyn_hard.CASES[name][1] + 7000)
    deep = dyn_hard.deepest(packed)
    chain = chain_of(packed, deep)
    mid = chain[(len(chain) - 1) // 2]
    s = {"packed": packed, "q": q, "qd": qd, "qdd": qdd, "deep": np.array(deep), "mid": np.array(mid)}
    Roff = rpy(OFFSET_RPY)
    s["frame"] = frame_row(deep, Roff, OFFSET_XYZ, LOCAL)               # reference-frame field set per call
    s["mid_frame"] = frame_row(mid, Roff, OFFSET_XYZ, LOCAL)
    s["support"] = frame_row(SUPPORT[0], rpy(SUPPORT[1]), SUPPORT[2], LOCAL)
    s["object"], s["base"] = OBJECT.copy(), BASE.copy()
    A = rng.randn(6, 6)
    s["S"] = A @ A.T / 6
    s["friction"] = rng.uniform(0.0, 2.0, nv)
    T = np.diag(rng.uniform(5.0, 100.0, nv))
    if nv > 1:
        T[nv - 1, nv - 2] = rng.uniform(-20.0, 20.0)                        # a coupled wrist
    s["drive"] = np.concatenate((T.reshape(-1), rng.uniform(1e-5, 1e-3, nv), rng.uniform(0.0, 0.5, nv)))
    # robot points on the deepest bodies, humans around the robot
    pts = []
    for i in range(P_POINTS):
        body = chain[-1 - (i % len(chain))]
        pts.append(np.concatenate((frame_row(body, dyn_hard._rotation(rng), rng.randn(3) * 0.1, LWA),
                                   [rng.uniform(0.0, 0.05)])))
    s["points"] = np.array(pts)
    s["humans"] = np.concatenate((rng.randn(H_HUMANS, 3) * 0.8 + (0.0, 0.0, 0.5),
                                  rng.uniform(0.05, 0.3, (H_HUMANS, 1))), axis=1)
    caps = []
    for i in range(P_CAPSULES):
        a, b = chain[-1 - (i % len(chain))], chain[-1 - ((i + 1) % len(chain))] if len(chain) > 1 else -1
        caps.append(np.concatenate((frame_row(a, np.eye(3), rng.randn(3) * 0.1, LWA),
                                    frame_row(b, np.eye(3), rng.randn(3) * 0.1, LWA), [rng.uniform(0.0, 0.05)])))
    s["capsules"] = np.array(caps)
    # one human set per state (points_per_path = 1); capsule 1 is a sphere (c0 == c1).  On a star, bodies 0 and 1 are
    # sliders along the base's x and z axes (dyn_hard.star): robot capsule 0 runs from x_a = (0, 0, q1) to
    # x_b = (q0, 0, 0), and human capsule 0 is that segment moved by o = (q0, 0.25, q1), c0 = (q0, 0.25, 2 q1),
    # c1 = (2 q0, 0.25, q1), every sum exact.  The two are parallel in exact arithmetic, so the 50-digit reference and
    # the kernels' parallel-segment branch see the same segment of closest pairs, along which the approach speed
    # changes (the ends move along x and z).
    star = dyn_hard.CASES[name][0] == "star"
    if star:
        s["capsules"][0, :28] = np.concatenate((frame_row(1, np.eye(3), np.zeros(3), LWA),
                                                frame_row(0, np.eye(3), np.zeros(3), LWA)))
    sets = []
    for m in range(q.shape[0]):
        hc = np.concatenate((rng.randn(H_CAPSULES, 3) * 0.8, rng.randn(H_CAPSULES, 3) * 0.8,
                             rng.uniform(0.05, 0.2, (H_CAPSULES, 1))), axis=1)
        hc[1, 3:6] = hc[1, :3]
        if star:
            hc[0, :6] = (q[m, 0], 0.25, 2 * q[m, 1], 2 * q[m, 0], 0.25, q[m, 1])
        sets.append(hc)
    s["hcaps"] = np.array(sets)
    if name in COUPLED:
        E = np.zeros((nv, nv - 1))
        E[:nv - 1, :nv - 1] = np.eye(nv - 1)
        E[nv - 1, nv - 2] = -0.7
        s["E"], s["o"] = E, np.concatenate((np.zeros(nv - 1), [0.1]))
    return s


def _ref(frame, ref):
    f = np.array(frame, dtype=np.float64)
    f[13] = ref
    return f


def _cat(*xs):
    return np.concatenate([np.asarray(x, dtype=np.float64).reshape(x.shape[0], -1) for x in xs], axis=1)


# ==== the float64 numpy doubles of tests/*_ref.py, in the fixture's layout ============================================
def numpy_outputs(s):
    P, q, qd, qdd = s["packed"], s["q"], s["qd"], s["qdd"]
    M = q.shape[0]
    fr, mid = s["frame"], s["mid_frame"]
    out = {"rnea": rr.rnea_packed(P, q, qd, qdd),
           "torque_terms": _cat(*rr.torque_terms_packed(P, q, qd, qdd, s["friction"])),
           "frame_velocity": _cat(*(kin_ref.frame_velocity_packed(P, _ref(fr, r), q, qd) for r in (WORLD, LOCAL, LWA))),
           "velocity_norm_terms": _cat(kin_ref.quad_form(s["S"], kin_ref.frame_velocity_packed(P, fr, q, qd))),
           "frame_acceleration": _cat(*(kin_acc_ref.frame_acceleration_packed(P, _ref(fr, r), q, qd, qdd)
                                        for r in (LOCAL, LWA)))}
    at = [kin_acc_ref.acceleration_terms_packed(P, _ref(fr, r), q, qd, qdd, range(6)) for r in (LOCAL, LWA)]
    out["acceleration_terms"] = _cat(at[0][0], at[1][0], at[0][1], at[1][1])
    out["contact_wrench"] = contact_ref.contact_wrench_packed(P, fr, s["object"], q, qd, qdd)
    out["contact_wrench_terms"] = _cat(*contact_ref.contact_terms_packed(P, fr, s["object"], q, qd, qdd))
    out["frame_inverse_inertia"] = _cat(*(energy_ref.inverse_inertia_packed(P, _ref(fr, r), q) for r in (LOCAL, LWA)))
    out["collision_energy_terms"] = _cat(energy_ref.energy_terms_packed(P, fr, q, qd, HUMAN_MASS))
    out["support_wrench"] = support_ref.support_wrench_packed(P, s["support"], s["base"], q, qd, qdd)
    out["support_wrench_terms"] = _cat(*support_ref.support_terms_packed(P, s["support"], s["base"], q, qd, qdd))
    out["separation"] = _cat(*sr.separation_packed(P, s["points"], s["humans"], q, qd))
    out["separation_terms"] = _cat(*sr.rows_packed(P, s["points"], s["humans"], SEPARATION, q, qd))
    out["capsule_separation"] = _cat(*cr.capsule_separation_packed(P, s["capsules"], s["hcaps"], q, qd, 1))
    out["capsule_separation_terms"] = _cat(*cr.capsule_rows_packed(P, s["capsules"], s["hcaps"], SEPARATION, q, qd, 1))
    out["drive_torque"] = drive_ref.torque_packed(P, s["drive"], q, qd, qdd)
    out["drive_torque_terms"] = _cat(*drive_ref.torque_terms_packed(P, s["drive"], q, qd, qdd))
    jw, jt = [], []
    for f in (fr, mid):
        for r in (LOCAL, LWA):
            jw.append(jr.joint_wrench_packed(P, _ref(f, r), q, qd, qdd))
            jt += list(jr.joint_wrench_terms_packed(P, _ref(f, r), q, qd, qdd))
    out["joint_wrench"], out["joint_wrench_terms"] = _cat(*jw), _cat(*jt)
    T, p = momentum_ref.energy_momentum_packed(P, q, qd)
    out["energy_momentum"] = _cat(T, p)
    out["energy_momentum_terms"] = _cat(T, momentum_ref.momentum_squared(p))
    if "E" in s:
        nq = s["E"].shape[1]
        x = (q[:, :nq], qd[:, :nq], qdd[:, :nq])
        out["coupled_rnea"] = coupled_ref.coupled_rnea_packed(P, s["E"], s["o"], *x)
        out["coupled_torque_terms"] = _cat(*coupled_ref.coupled_torque_terms_packed(P, s["E"], s["o"], *x,
                                                                                     friction=s["friction"][:nq]))
    assert all(v.shape[0] == M for v in out.values())
    return out



# ==== Monte Carlo arithmetic on the numpy doubles =====================================================================
class _MC(np.ndarray):
    """An array whose every floating-point operation result is multiplied by (1 + u), u uniform in +-2^-53 (Monte Carlo
    arithmetic, D. S. Parker 1997): the spread of the results over a few runs measures how much rounding of the
    intermediate quantities of an algorithm moves its output, the eps-sized part of its magnitude-sum."""
    rng = None

    @classmethod
    def _perturb(cls, out):
        if isinstance(out, np.ndarray) and out.dtype == np.float64:
            out = out * (1.0 + cls.rng.uniform(-1.0, 1.0, out.shape) * 2.0 ** -53)
            return out.view(cls)
        if isinstance(out, (float, np.floating)):
            return np.asarray(float(out) * (1.0 + cls.rng.uniform(-1.0, 1.0) * 2.0 ** -53)).view(cls)
        return out

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        args = [x.view(np.ndarray) if isinstance(x, _MC) else x for x in inputs]
        out = getattr(ufunc, method)(*args, **kwargs)
        return self._perturb(out) if ufunc.types[-1][-1] == "d" or np.asarray(out).dtype == np.float64 else out

    def __array_function__(self, func, types, args, kwargs):
        def plain(x):
            if isinstance(x, _MC):
                return x.view(np.ndarray)
            if isinstance(x, (list, tuple)):
                return type(x)(plain(y) for y in x)
            return x
        out = func(*plain(args), **plain(kwargs))
        if func in (np.einsum, np.dot, np.matmul, np.sum, np.cross):
            return self._perturb(out)
        if isinstance(out, np.ndarray) and out.dtype == np.float64:
            return out.view(_MC)
        return out


def rounding_spread(s, runs=6, seed=0):
    """{entry: (M, n) the largest |MC run - plain run| of the numpy doubles over `runs` runs} (see _MC)."""
    plain = numpy_outputs(s)
    _MC.rng = np.random.RandomState(seed)
    mc = dict(s)
    for k in ("packed", "q", "qd", "qdd"):
        mc[k] = np.array(s[k], dtype=np.float64).view(_MC)
    spread = {k: np.zeros_like(v) for k, v in plain.items()}
    asarray = np.asarray
    np.asarray = np.asanyarray               # the doubles take their inputs through np.asarray: keep them _MC
    try:
        runs_out = [numpy_outputs(mc) for _ in range(runs)]
    finally:
        np.asarray = asarray
    for out in runs_out:
        for k, v in out.items():
            spread[k] = np.maximum(spread[k], np.abs(np.array(v, dtype=np.float64).view(np.ndarray) - plain[k]))
    return spread


# ==== 50-digit evaluation of every entry at one point =================================================================
def _offset(frame):
    return int(frame[0]), np.asarray(frame[1:10]).reshape(3, 3), np.asarray(frame[10:13])


def evaluate(s, packed, q, qd, qdd, m):
    """{entry: [(value, mag, parts)]} at 50 digits for point m of case setup s, with the model and state given (possibly
    perturbed).  value and mag are flat lists of mpf; parts the list of flat lists whose changes make up sens."""
    import mpmath

    import capsule_ref
    import contact_ref
    import coupled_ref
    import drive_ref
    import energy_ref
    import kin_acc_ref
    import kin_ref
    import momentum_ref
    import rnea_ref
    import separation_ref
    import support_ref
    mpmath.mp.dps = rnea_ref.DPS
    robot = rnea_ref.MpRobot.from_packed(packed)
    tau_cache = {}
    raw_tau = robot.tau

    def tau(a, b, c):                         # the Lagrangian torques, shared by the torque and drive entries
        key = tuple(float(x) for x in np.concatenate((a, b, c)))
        if key not in tau_cache:
            tau_cache[key] = raw_tau(a, b, c)
        return tau_cache[key]
    robot.tau = tau
    nv = len(q)
    zero = np.zeros(nv)
    out = {}
    A = lambda v: [abs(x) for x in v]         # noqa: E731
    sub = lambda x, y: [a - b for a, b in zip(x, y)]   # noqa: E731
    add = lambda x, y: [a + b for a, b in zip(x, y)]   # noqa: E731

    def G(v, g):                              # |x| of each component's group of g: a 3-vector, a 3x3 matrix
        return [mpmath.sqrt(mpmath.fsum(x * x for x in v[i - i % g:i - i % g + g])) for i in range(len(v))]

    def direct(v, g=1):
        return (list(v), G(v, g), [list(v)])

    def diff(w1, w0, g=1):
        return (sub(w1, w0), add(G(w1, g), G(w0, g)), [list(w1), list(w0)])

    # joint torques
    t1, ta, t0 = tau(q, qd, qdd), tau(q, zero, qd), tau(q, zero, zero)
    out["rnea"] = direct(t1)
    fr = [mpmath.mpf(float(x)) * (1 if v > 0 else (-1 if v < 0 else 0)) for x, v in zip(s["friction"], qd)]
    out["torque_terms"] = _stack([diff(ta, t0), diff(t1, t0), (add(t0, fr), add(A(t0), A(fr)), [list(t0)])])
    # frame velocities and accelerations (frame on the deepest body)
    body, Ro, po = _offset(s["frame"])
    spec = {0: (_link(body), Ro, po)}
    v = kin_ref.mp_frames(robot, q, qd, spec)[0]["v"]
    out["frame_velocity"] = _stack([direct(v[k], 3) for k in ("world", "local", "local_world_aligned")])
    S = [[mpmath.mpf(float(x)) for x in row] for row in s["S"]]
    vl = v["local"]
    qf = mpmath.fsum(vl[i] * S[i][j] * vl[j] for i in range(6) for j in range(6))
    qm = mpmath.fsum(abs(vl[i] * S[i][j] * vl[j]) for i in range(6) for j in range(6))
    out["velocity_norm_terms"] = ([qf], [qm], [[qf]])
    acc_b = kin_acc_ref.mp_accelerations(robot, q, qd, qdd, spec)[0]
    acc_a = kin_acc_ref.mp_accelerations(robot, q, zero, qd, spec)[0]
    out["frame_acceleration"] = _stack([direct(acc_b[k], 3) for k in ("local", "local_world_aligned")])
    out["acceleration_terms"] = _stack([direct(acc_a[k], 3) for k in ("local", "local_world_aligned")]
                                       + [direct(acc_b[k], 3) for k in ("local", "local_world_aligned")])
    # contact wrench of a carried object
    obj = s["object"]
    w1, wa, w0 = (contact_ref.mp_wrenches(robot, q, x, y, spec, obj)[0]
                  for x, y in ((qd, qdd), (zero, qd), (zero, zero)))
    out["contact_wrench"] = direct(w1, 3)
    out["contact_wrench_terms"] = _stack([diff(wa, w0, 3), diff(w1, w0, 3), direct(w0, 3)])
    # inverse operational-space inertia and collision energy
    ii = energy_ref.mp_inverse_inertia(robot, q, spec)
    Linv, Rf = ii[0]
    loc = Rf.T * Linv * Rf
    out["frame_inverse_inertia"] = _stack([direct([loc[i, j] for i in range(3) for j in range(3)], 9),
                                           direct([Linv[i, j] for i in range(3) for j in range(3)], 9)])
    eb = energy_ref.mp_energy_b(ii[(0, "J")], Linv, qd, HUMAN_MASS)
    out["collision_energy_terms"] = ([eb], [abs(eb)], [[eb]])
    # support wrench of the whole tree
    _, Rs, ps = _offset(s["support"])
    w1, wa, w0 = (support_ref.mp_support_wrench(robot, q, x, y, Rs, ps, s["base"])
                  for x, y in ((qd, qdd), (zero, qd), (zero, zero)))
    out["support_wrench"] = direct(w1, 3)
    out["support_wrench_terms"] = _stack([diff(wa, w0, 3), diff(w1, w0, 3), direct(w0, 3)])
    # separation of points and spheres
    pts = s["points"]
    st = separation_ref.mp_points(robot, q, qd, {i: (_link(int(r[0])), r[1:10].reshape(3, 3), r[10:13])
                                                  for i, r in enumerate(pts)})
    pairs, dmag, wmag = [], [], []
    for i, r in enumerate(pts):
        x, vel = st[i]
        speed = mpmath.sqrt(sum(c * c for c in vel))
        for h in s["humans"]:
            d, w = separation_ref.mp_pair(x, vel, r[14], h)
            pairs.append((d, w))
            dmag.append(abs(d) + 2 * (mpmath.mpf(float(r[14])) + mpmath.mpf(float(h[3]))))
            wmag.append(speed)
    ds, ws = [p[0] for p in pairs], [p[1] for p in pairs]
    out["separation"] = _stack([(ds, dmag, [ds]), (ws, wmag, [ws])])
    b, c = separation_ref.mp_row(pairs, SEPARATION)
    out["separation_terms"] = ([b, c], [abs(b), abs(c)], [[b, c]])
    # capsules
    caps = s["capsules"]
    spec_c = [((_link(int(r[0])), r[1:10].reshape(3, 3), r[10:13]), (_link(int(r[14])), r[15:24].reshape(3, 3),
                                                                     r[24:27]), r[28]) for r in caps]
    hset = s["hcaps"][m]
    cp = capsule_ref.mp_capsule_pairs(robot, q, qd, spec_c, hset)
    ends = separation_ref.mp_points(robot, q, qd, {2 * i + j: spec_c[i][j] for i in range(len(caps)) for j in (0, 1)})
    flat, dmag, wmag = [], [], []
    norm = lambda v: mpmath.sqrt(sum(mpmath.mpf(float(x)) ** 2 if not isinstance(x, mpmath.mpf) else x * x
                                     for x in v))  # noqa: E731
    for i in range(len(caps)):
        sp = norm(ends[2 * i][1]) + norm(ends[2 * i + 1][1])
        for h in range(len(hset)):
            d, w = cp[i][h]
            flat.append((d, w))
            radii = mpmath.mpf(float(caps[i][28])) + mpmath.mpf(float(hset[h][6]))
            # the closest points are interpolated between the endpoints: their rounding is relative to the endpoints'
            pos = norm(ends[2 * i][0]) + norm(ends[2 * i + 1][0]) + norm(hset[h][:3]) + norm(hset[h][3:6])
            dmag.append(abs(d) + 2 * radii + pos)
            wmag.append(sp * (1 + pos / max(abs(d) + radii, mpmath.mpf(10) ** -30)))
    ds, ws = [p[0] for p in flat], [p[1] for p in flat]
    out["capsule_separation"] = _stack([(ds, dmag, [ds]), (ws, wmag, [ws])])
    b, c = separation_ref.mp_row(flat, SEPARATION)
    out["capsule_separation_terms"] = ([b, c], [abs(b), abs(c)], [[b, c]])
    # geared drives
    drive = s["drive"]
    d1, da, d0 = (drive_ref.mp_torque(robot, drive, q, x, y) for x, y in ((qd, qdd), (zero, qd), (zero, zero)))
    Tm, _, fm = drive_ref.unpack(drive, nv)
    sg = np.sign(Tm @ qd)
    fr = [mpmath.mpf(float(x)) * int(y) for x, y in zip(fm, sg)]
    out["drive_torque"] = direct(d1)
    out["drive_torque_terms"] = _stack([diff(da, d0), diff(d1, d0), (add(d0, fr), add(A(d0), A(fr)), [list(d0)])])
    # wrench across the joint of the deepest and of a mid-chain body
    jw, jt = [], []
    for key in ("frame", "mid_frame"):
        body, Rf_, pf_ = _offset(s[key])
        for ref in (LOCAL, LWA):
            w1, wa, w0 = (_mp_joint_wrench(robot, body, q, x, y, Rf_, pf_, ref)
                          for x, y in ((qd, qdd), (zero, qd), (zero, zero)))
            jw.append(direct(w1, 3))
            jt += [diff(wa, w0, 3), diff(w1, w0, 3), direct(w0, 3)]
    out["joint_wrench"] = _stack(jw)
    out["joint_wrench_terms"] = _stack(jt)
    # kinetic energy and momentum
    T, p = momentum_ref.mp_energy_momentum(robot, q, qd)
    out["energy_momentum"] = ([T] + list(p), [abs(T)] + G(p, 3), [[T] + list(p)])
    pp = p[0] * p[0] + p[1] * p[1] + p[2] * p[2]
    out["energy_momentum_terms"] = ([T, pp], [abs(T), pp], [[T, pp]])
    # coupled joints
    if "E" in s:
        nq = s["E"].shape[1]
        cr = coupled_ref.MpCoupled(robot, s["E"], s["o"])
        c0, ca, c1 = cr.tau_terms(q[:nq], qd[:nq], qdd[:nq])
        fr = [mpmath.mpf(float(x)) * (1 if y > 0 else (-1 if y < 0 else 0))
              for x, y in zip(s["friction"][:nq], qd[:nq])]
        out["coupled_rnea"] = direct(c1)
        out["coupled_torque_terms"] = _stack([diff(ca, c0), diff(c1, c0), (add(c0, fr), add(A(c0), A(fr)), [list(c0)])])
    # every entry as blocks: parts[block][term][component]
    return {k: v if isinstance(v[2][0][0], list) else _stack([v]) for k, v in out.items()}


def _link(body):
    return "base" if body < 0 else "b%d" % body


def _stack(items):
    """Concatenate several (value, mag, parts) blocks into one (the entry's outputs are laid out block after block)."""
    val, mag, parts = [], [], []
    for v, m_, p in items:
        val += list(v)
        mag += list(m_)
        parts.append(p)
    return val, mag, parts


def _mp_joint_wrench(robot, body, q, qd, qdd, R_f, p_f, ref):
    """joint_wrench_ref.mp_joint_wrench kept at 50 digits: the subtree's wrench about the world origin in world axes
    (support_ref.mp_support_wrench with an identity support frame at the origin, exact inputs), then moved to the
    frame origin and rotated at 50 digits."""
    import copy

    import mpmath

    import joint_wrench_ref
    import rnea_ref
    import support_ref
    child, below = joint_wrench_ref.subtree_links(robot, body)
    sub = copy.copy(robot)
    sub.links = {name: (inert if name in below else None) for name, inert in robot.links.items()}
    w = support_ref.mp_support_wrench(sub, q, qd, qdd, np.eye(3), np.zeros(3))
    with mpmath.workdps(rnea_ref.DPS):
        Rb, pb = robot._kinematics([mpmath.mpf(float(x)) for x in q])[0][child]
        Rf = mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in R_f])
        o = pb + Rb * mpmath.matrix([mpmath.mpf(float(x)) for x in p_f])
        f, n = mpmath.matrix(w[:3]), mpmath.matrix(w[3:])
        n = n - rnea_ref._cross(o, f)
        R = Rb * Rf if ref == LOCAL else mpmath.eye(3)
        return list(R.T * f) + list(R.T * n)


# ==== sensitivity and the fixture =====================================================================================
def perturbed(s, d):
    """(packed, q, qd, qdd) with every real input moved by one ulp in sign pattern d (d < 0: the inputs as they are).
    A nonzero model parameter that is part of a vector or matrix (gravity, axis, E, r, com, inertia) moves by one ulp
    of that group's largest entry, the size of a rounding error of float64 arithmetic on the group.  Zeros stay: they
    are exact (an axis along z, an offset in a plane), and what a float64 algorithm rounds next to them is covered by
    mag, the size of the output's own vector.  Joint positions, speeds and accelerations move by one ulp of their
    own."""
    packed, q, qd, qdd = (np.array(s[k], dtype=np.float64) for k in ("packed", "q", "qd", "qdd"))
    if d < 0:
        return packed, q, qd, qdd
    rng = np.random.RandomState(1000 + d)
    nv = q.shape[1]
    groups = [(0, 3)] + [(3 + 27 * k + a, 3 + 27 * k + b) for k in range(nv)
                         for a, b in ((2, 5), (5, 14), (14, 17), (17, 18), (18, 21), (21, 27))]
    out = packed.copy()                       # parent index and joint type (+0, +1) are codes and stay
    for a, b in groups:
        step = np.spacing(np.max(np.abs(packed[a:b])))
        out[a:b] = packed[a:b] + rng.choice([-1.0, 1.0], b - a) * np.where(packed[a:b] != 0, step, 0.0)
    rest = [np.nextafter(x, rng.choice([-1.0, 1.0], x.shape) * np.inf) for x in (q, qd, qdd)]
    return (out,) + tuple(rest)


def _task(args):
    name, m, d = args
    s = setup(name)
    packed, q, qd, qdd = perturbed(s, d)
    return evaluate(s, packed, q[m], qd[m], qdd[m], m)


def main():
    import mpmath
    names = list(dyn_hard.CASES)
    setups = {n: setup(n) for n in names}
    jobs = [(n, m, d) for n in names for m in range(setups[n]["q"].shape[0]) for d in range(-1, DIRECTIONS)]
    jobs.sort(key=lambda j: -len(setups[j[0]]["q"][0]))                    # the big models first
    with multiprocessing.Pool() as pool:
        results = dict(zip(jobs, pool.map(_task, jobs, chunksize=1)))
    data = {"cases": np.array(names), "directions": np.array(DIRECTIONS), "c_tol": np.array(C_TOL)}
    with mpmath.workdps(60):
        for n in names:
            s = setups[n]
            for k, v in s.items():
                data["%s/%s" % (n, k)] = np.asarray(v)
            M = s["q"].shape[0]
            spread = rounding_spread(s)
            for entry in results[(n, 0, -1)]:
                refs, tols = [], []
                for m in range(M):
                    val, mag, parts = results[(n, m, -1)][entry]
                    sens = [mpmath.mpf(0)] * len(val)
                    for d in range(DIRECTIONS):
                        pd = results[(n, m, d)][entry][2]
                        ch = [mpmath.mpf(0)] * len(val)
                        i = 0
                        for blk, blk_d in zip(parts, pd):
                            width = len(blk[0])
                            for term, term_d in zip(blk, blk_d):
                                for j in range(width):
                                    ch[i + j] += abs(term_d[j] - term[j])
                            i += width
                        sens = [max(a, b) for a, b in zip(sens, ch)]
                    refs.append([float(x) for x in val])
                    tols.append([float(C_TOL * (a + EPS * b + mpmath.mpf(float(c))))
                                 for a, b, c in zip(sens, mag, spread[entry][m])])
                data["%s/%s/ref" % (n, entry)] = np.array(refs)
                data["%s/%s/tol" % (n, entry)] = np.array(tols)
    save(OUT, data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def save(path, data):
    """np.savez_compressed with fixed member timestamps, so that the file is byte-identical on every run."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


if __name__ == "__main__":
    main()
