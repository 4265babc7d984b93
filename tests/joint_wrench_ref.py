"""TEST INFRASTRUCTURE — references for the wrench across a joint (JointWrenchConstraint, RigidBodyFrame.joint_wrench /
joint_wrench_terms, libtoppra_b200_dyn.so: tbd_joint_wrench / tbd_joint_wrench_terms).

* `mp_joint_wrench`: the 50-digit wrench the parent side of a joint exerts on the joint's subtree of a
  `rnea_ref.MpRobot`, along t -> q + t qd + t^2/2 qdd.  The subtree is taken on the RAW URDF tree (fixed and locked
  joints stay zero-DOF links, nothing is folded): the joint's child link and every link below it.  Over those links
  only, it is `support_ref.mp_support_wrench`'s sum of the rate of change of each link's momentum and angular momentum
  minus its weight, f_i = m_i (p_i'' - g), n_i = (p_i - o) x f_i + d/dt (R_i Ic_i R_i^T w_i), about the frame origin o
  (both differentiated with mpmath.diff), in the frame's axes or in world axes.  It uses neither the recursion of the
  kernels nor a Jacobian.
* `joint_wrench_packed`, `joint_wrench_terms_packed`: a float64 numpy double of the device algorithm of the two entries
  (include/toppra_b200_dyn.h), vectorised over points."""
import copy

import mpmath
import numpy as np

import rnea_ref
import support_ref

DPS = rnea_ref.DPS
LOCAL, LOCAL_WORLD_ALIGNED = 1, 2


def subtree_links(robot, dof):
    """(child link of the joint of DOF `dof`, the names of that link and of every link below it) on the raw tree."""
    child = [j["child"] for j in robot.joints if j["dof"] == dof][0]
    below, grew = {child}, True
    while grew:
        grew = False
        for j in robot.joints:
            if j["parent"] in below and j["child"] not in below:
                below.add(j["child"])
                grew = True
    return child, below


# ==== 50-digit reference ==============================================================================================
def mp_joint_wrench(robot, dof, q, qd, qdd, R_f, p_f, ref=LOCAL):
    """[f; n] (6 floats) across the joint of DOF `dof`, at the origin of the frame (R_f, p_f) given in the joint's child
    link frame (the body frame of RigidBodyModel), in the frame's axes (ref LOCAL) or world axes (LOCAL_WORLD_ALIGNED)."""
    child, below = subtree_links(robot, dof)
    sub = copy.copy(robot)
    sub.links = {name: (inert if name in below else None) for name, inert in robot.links.items()}
    with mpmath.workdps(DPS):
        R, p = robot._kinematics([mpmath.mpf(float(x)) for x in q])[0][child]
        Rb = np.array([[float(R[i, j]) for j in range(3)] for i in range(3)])
        pb = np.array([float(x) for x in p])
    Rw = Rb @ np.asarray(R_f, dtype=np.float64)
    o = pb + Rb @ np.asarray(p_f, dtype=np.float64)
    w = support_ref.mp_support_wrench(sub, q, qd, qdd, Rw if ref == LOCAL else np.eye(3), o)
    return np.array([float(x) for x in w])


# ==== float64 numpy double of the device algorithm ====================================================================
def _chain(packed, body):
    chain = []
    while body >= 0:
        chain.insert(0, body)
        body = int(packed[3 + 27 * body])
    return chain


def _wrench(packed, frame, Rs, f, M):
    body = int(frame[0])
    R_f, p_f, ref = np.asarray(frame[1:10]).reshape(3, 3), np.asarray(frame[10:13]), int(frame[13])
    n, fl = f[body]
    t = n - rnea_ref._cross_np(np.broadcast_to(p_f, (M, 3)), fl)
    if ref == LOCAL:
        return np.concatenate((fl @ R_f, t @ R_f), axis=1)
    chain = _chain(packed, body)
    Rw = Rs[chain[0]]
    for k in chain[1:]:
        Rw = np.einsum("mij,mjk->mik", Rw, Rs[k])
    return np.concatenate((np.einsum("mij,mj->mi", Rw, fl), np.einsum("mij,mj->mi", Rw, t)), axis=1)


def joint_wrench_packed(packed, frame, q, qd, qdd):
    """Double of tbd_joint_wrench: (M, nv) arrays -> w (M, 6) = [f; n] at the frame origin."""
    packed = np.asarray(packed, dtype=np.float64)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    Rs, ps = rnea_ref._transforms(packed, q)
    return _wrench(packed, frame, Rs, rnea_ref._pass(packed, Rs, ps, qd, qdd)[1], q.shape[0])


def joint_wrench_terms_packed(packed, frame, q, qs, qss, components=(0, 1, 2, 3, 4, 5)):
    """Double of tbd_joint_wrench_terms: c = w(q, 0, 0), a = w(q, 0, qs) - c, b = w(q, qs, qss) - c, the columns of
    `components` in increasing order."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    zero = np.zeros_like(q)
    cols = sorted(components)
    c = joint_wrench_packed(packed, frame, q, zero, zero)
    a = joint_wrench_packed(packed, frame, q, zero, qs) - c
    b = joint_wrench_packed(packed, frame, q, qs, qss) - c
    return a[:, cols], b[:, cols], c[:, cols]
