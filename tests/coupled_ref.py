"""TEST INFRASTRUCTURE — references for robots with coupled joints (RigidBodyModel with a coupling, from_urdf with
couple_mimic=True, with_coupling; libtoppra_b200_dyn.so: tbd_coupled_rnea, tbd_coupled_torque_terms,
tbd_coupling_expand).

* `MpCoupled`: 50 digits on the RAW URDF tree of an `rnea_ref.MpRobot` (mimic joints are DOFs there, nothing is
  folded) or on a packed model, with the body joint positions q_b = E q + o.  It does not take the kernels' route
  E^T ID(q_b, ...): it forms the reduced Lagrangian in q,
      M_q(q) = E^T M_b(E q + o) E,     g_q = dV/dq,     h_q,k = sum_ij (d_i M_q,kj - 1/2 d_k M_q,ij) qd_i qd_j,
      tau_q  = M_q qdd + h_q + g_q,
  with V the potential energy of every link and each derivative in q by `mpmath.diff`.
* `expand`, `reduce_`, `coupled_rnea_packed`, `coupled_torque_terms_packed`: a float64 numpy double of the device
  algorithm (include/toppra_b200_dyn.h): the expansion and reduction in their fixed operation order around
  `rnea_ref.rnea_packed` / `rnea_ref.torque_terms_packed`, vectorised over points."""
import mpmath
import numpy as np

import rnea_ref

DPS = rnea_ref.DPS


# ==== 50-digit reduced Lagrangian ======================================================================================
class MpCoupled(object):
    """tau_q of `robot` (an rnea_ref.MpRobot whose DOF k is body k) under the coupling q_b = E q + o."""

    def __init__(self, robot, E, o):
        self.robot = robot
        self.E = [[mpmath.mpf(float(x)) for x in row] for row in np.asarray(E, dtype=np.float64)]
        self.o = [mpmath.mpf(float(x)) for x in np.asarray(o, dtype=np.float64)]
        self.nv, self.nq = len(self.E), len(self.E[0])
        assert self.nv == robot.nv

    def _qb(self, q):
        return [mpmath.fsum(self.E[k][j] * q[j] for j in range(self.nq)) + self.o[k] for k in range(self.nv)]

    def mass_matrix(self, q):
        Mb = self.robot.mass_matrix(self._qb(q))
        Em = mpmath.matrix(self.E)
        return Em.T * Mb * Em

    def potential(self, q):
        frames = self.robot._kinematics(self._qb(q))[0]
        V = mpmath.mpf(0)
        for name, inert in self.robot.links.items():
            if inert is None or name not in frames:
                continue
            R, p = frames[name]
            pc = p + R * inert[1]
            V -= inert[0] * sum(self.robot.g[r] * pc[r] for r in range(3))
        return V

    def tau_terms(self, q, qs, qss):
        """(ID_q(q, 0, 0), ID_q(q, 0, qs), ID_q(q, qs, qss)) at DPS digits, each a list of nq mpf."""
        nq = self.nq
        with mpmath.workdps(DPS):
            q, qs, qss = ([mpmath.mpf(float(x)) for x in v] for v in (q, qs, qss))
            shift = lambda i, t: [q[k] + (t if k == i else 0) for k in range(nq)]  # noqa: E731
            zero = mpmath.mpf(0)
            g = [mpmath.diff(lambda t, i=i: self.potential(shift(i, t)), zero) for i in range(nq)]
            M = self.mass_matrix(q)
            h = [zero] * nq
            if any(x != 0 for x in qs):
                dM = [mpmath.diff(lambda t, i=i: self.mass_matrix(shift(i, t)), zero) for i in range(nq)]
                h = [mpmath.fsum((dM[i][k, j] - dM[k][i, j] / 2) * qs[i] * qs[j] for i in range(nq) for j in range(nq))
                     for k in range(nq)]
            Ma = [mpmath.fsum(M[k, j] * qs[j] for j in range(nq)) for k in range(nq)]
            Mb = [mpmath.fsum(M[k, j] * qss[j] for j in range(nq)) for k in range(nq)]
            return g, [Ma[k] + g[k] for k in range(nq)], [Mb[k] + h[k] + g[k] for k in range(nq)]

    def tau(self, q, qd, qdd):
        """ID_q(q, qd, qdd) at DPS digits."""
        return self.tau_terms(q, qd, qdd)[2]

    def tau64(self, q, qd, qdd):
        return np.array([float(x) for x in self.tau(q, qd, qdd)])

    def terms64(self, q, qs, qss):
        """(c, a, b) of the torque rows, c = ID_q(q, 0, 0), a = ID_q(q, 0, qs) - c, b = ID_q(q, qs, qss) - c, each
        difference taken at DPS digits and rounded to fp64."""
        with mpmath.workdps(DPS):
            c, ta, tb = self.tau_terms(q, qs, qss)
            return (np.array([float(x) for x in c]), np.array([float(x - y) for x, y in zip(ta, c)]),
                    np.array([float(x - y) for x, y in zip(tb, c)]))


# ==== float64 numpy double of the device algorithm =====================================================================
def expand(E, o, x, pos):
    """E x (+ o where pos) for x (P, nq) -> (P, nv): per row the nonzero terms in ascending j from the first term, then
    + o[k] where o[k] != 0 (positions)."""
    E = np.asarray(E, dtype=np.float64)
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    out = np.zeros((x.shape[0], E.shape[0]))
    for k in range(E.shape[0]):
        s = None
        for j in range(E.shape[1]):
            if E[k, j] != 0:
                t = E[k, j] * x[:, j]
                s = t if s is None else s + t
        s = np.zeros(x.shape[0]) if s is None else s
        if pos and o[k] != 0:
            s = s + o[k]
        out[:, k] = s
    return out


def reduce_(E, t):
    """E^T t for t (P, nv) -> (P, nq): per DOF the nonzero terms in ascending k from the first term."""
    E = np.asarray(E, dtype=np.float64)
    out = np.zeros((t.shape[0], E.shape[1]))
    for j in range(E.shape[1]):
        s = None
        for k in range(E.shape[0]):
            if E[k, j] != 0:
                u = E[k, j] * t[:, k]
                s = u if s is None else s + u
        out[:, j] = s
    return out


def coupled_rnea_packed(packed, E, o, q, qd, qdd):
    """Double of tbd_coupled_rnea: (P, nq) arrays -> tau (P, nq)."""
    return reduce_(E, rnea_ref.rnea_packed(packed, expand(E, o, q, True), expand(E, o, qd, False),
                                           expand(E, o, qdd, False)))


def coupled_torque_terms_packed(packed, E, o, q, qs, qss, friction=None):
    """Double of tbd_coupled_torque_terms: (a, b, c), each (P, nq)."""
    a, b, c = rnea_ref.torque_terms_packed(packed, expand(E, o, q, True), expand(E, o, qs, False),
                                           expand(E, o, qss, False))
    a, b, c = reduce_(E, a), reduce_(E, b), reduce_(E, c)
    if friction is not None and np.any(np.asarray(friction) != 0):
        c = c + np.sign(np.atleast_2d(qs)) * np.asarray(friction, dtype=np.float64)
    return a, b, c


def level_rows(model):
    """The levelling link of the palletizer fixture: the coupling (nq, nq - 1) of RigidBodyModel.with_coupling that
    holds wrist_pitch at -(shoulder + elbow), every other DOF kept."""
    names = model.joint_names
    keep = [n for n in names if n != "wrist_pitch"]
    L = np.zeros((len(names), len(keep)))
    for i, n in enumerate(names):
        if n == "wrist_pitch":
            L[i, keep.index("shoulder")] = L[i, keep.index("elbow")] = -1.0
        else:
            L[i, keep.index(n)] = 1.0
    return L


def random_coupling(rng, nv, nq):
    """E (nv, nq) with every column nonzero: DOF j drives body perm[j] with a random ratio, the other bodies are
    coupled to one or two random DOFs or to none (a body held at its offset); o random, some zero."""
    perm = rng.permutation(nv)
    E = np.zeros((nv, nq))
    for j in range(nq):
        E[perm[j], j] = rng.choice([1.0, -1.0, rng.uniform(-2, 2)])
    for k in perm[nq:]:
        for j in rng.choice(nq, size=rng.randint(0, min(2, nq) + 1), replace=False):
            E[k, j] = rng.uniform(-1.5, 1.5)
    o = np.where(rng.rand(nv) < 0.5, 0.0, rng.uniform(-0.5, 0.5, nv))
    return E, o
