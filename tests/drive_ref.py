"""TEST INFRASTRUCTURE — references for geared drives (toppra_b200.Drives, MotorTorqueConstraint, MotorSpeedConstraint;
libtoppra_b200_dyn.so: tbd_drive_torque, tbd_drive_torque_terms, tbd_drive_speed_terms).

* `mp_torque`, `mp_speed_row`: 50 digits.  The joint torques come from `rnea_ref.MpRobot` (the Lagrangian form on the
  RAW URDF tree, or on a packed model), T^-1 from mpmath's own inverse:  w = T^-T tau + I_r o (T qdd),
  b = max_i ((T q')_i / omega_i)^2.
* `torque_packed`, `torque_terms_packed`, `speed_terms_packed`: float64 numpy doubles on the packed layouts of
  include/toppra_b200_dyn.h, vectorised over points.  The torque doubles sit on `rnea_ref.rnea_packed` and invert T with
  numpy; the speed row restates the kernel's order exactly (each (T q')_i summed left to right, then / omega_i, squared,
  and a NaN-propagating maximum), so it is bit-comparable."""
import mpmath
import numpy as np

import rnea_ref as rr


def unpack(drive, nv):
    """(T (nv, nv), I_r (nv,), f (nv,)) of a packed drive."""
    drive = np.asarray(drive, dtype=np.float64)
    return drive[:nv * nv].reshape(nv, nv), drive[nv * nv:nv * nv + nv], drive[nv * nv + nv:nv * nv + 2 * nv]


def pack(T, rotor_inertia, friction):
    nv = T.shape[0]
    return np.concatenate((np.asarray(T, dtype=np.float64).reshape(-1),
                           np.broadcast_to(np.asarray(rotor_inertia, dtype=np.float64), (nv,)),
                           np.broadcast_to(np.asarray(friction, dtype=np.float64), (nv,))))


# ==== 50 digits ======================================================================================================
def _mp_matrix(T):
    return mpmath.matrix([[mpmath.mpf(float(x)) for x in row] for row in np.asarray(T)])


def mp_torque(mp, drive, q, qd, qdd):
    """w(q, qd, qdd) at rr.DPS digits as mp values: mp is an rr.MpRobot."""
    T, Ir, _ = unpack(drive, mp.nv)
    with mpmath.workdps(rr.DPS):
        tau = mpmath.matrix(mp.tau(q, qd, qdd))
        Tm = _mp_matrix(T)
        Tmt_inv = mpmath.inverse(Tm).T
        load = Tmt_inv * tau
        acc = Tm * mpmath.matrix([mpmath.mpf(float(x)) for x in qdd])
        return [load[i] + mpmath.mpf(float(Ir[i])) * acc[i] for i in range(mp.nv)]


def mp_speed_row(drive, nv, omega, qs):
    """b = max_i ((T q')_i / omega_i)^2 at rr.DPS digits (omega_i = inf contributes 0)."""
    T, _, _ = unpack(drive, nv)
    with mpmath.workdps(rr.DPS):
        v = _mp_matrix(T) * mpmath.matrix([mpmath.mpf(float(x)) for x in qs])
        return max((v[i] / mpmath.mpf(float(omega[i]))) ** 2 if np.isfinite(omega[i]) else mpmath.mpf(0)
                   for i in range(nv))


# ==== float64 numpy doubles ==========================================================================================
def torque_packed(model, drive, q, qd, qdd):
    """float64 double of tbd_drive_torque: (M, nv) arrays -> w (M, nv)."""
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    T, Ir, _ = unpack(drive, q.shape[1])
    tau = rr.rnea_packed(model, q, qd, qdd)
    return tau @ np.linalg.inv(T) + Ir * (qdd @ T.T)


def torque_terms_packed(model, drive, q, qs, qss):
    """float64 double of tbd_drive_torque_terms: (a, b, c)."""
    q, qs, qss = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qs, qss))
    T, _, f = unpack(drive, q.shape[1])
    zero = np.zeros_like(q)
    c = torque_packed(model, drive, q, zero, zero)
    a = torque_packed(model, drive, q, zero, qs) - c
    b = torque_packed(model, drive, q, qs, qss) - c
    return a, b, c + f * np.sign(qs @ T.T)


def speed_terms_packed(drive, omega, qs):
    """tbd_drive_speed_terms in its order of operations: (M, nv) -> b (M,)."""
    qs = np.atleast_2d(np.asarray(qs, dtype=np.float64))
    nv = qs.shape[1]
    T, _, _ = unpack(drive, nv)
    r2 = []
    for i in range(nv):
        v = T[i, 0] * qs[:, 0]
        for j in range(1, nv):
            v = v + T[i, j] * qs[:, j]
        r = v / omega[i]
        r2.append(r * r)
    return np.max(np.stack(r2, axis=1), axis=1)
