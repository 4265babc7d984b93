/*
 * toppra_b200_dyn.h — C-ABI of libtoppra_b200_dyn.so: rigid-body inverse dynamics (recursive Newton-Euler) of a
 * fixed-base kinematic tree on the GPU, the hot path of joint-torque constraints on real robots
 * (toppra_b200.RigidBodyModel; the reference drives JointTorqueConstraint with pinocchio.rnea for the same purpose).
 *
 * Conventions are those of include/toppra_b200.h: device pointers (except model_host), caller-owned memory,
 * asynchronous on `stream`, 0 / TB_ERR_* / cudaError_t returns, fp64 with -fmad=false.  This library links against
 * libtoppra_b200.so and reports errors through its tb_last_error().
 *
 * Model: a fixed-base tree of nv <= TBD_MAX_BODIES moving bodies, one joint DOF per body, DOF index = body index,
 * bodies in topological order (parent[k] < k, -1 = the base).  model_host is a HOST array of 3 + 27 nv doubles:
 *
 *   [0, 3)            gravity g in the base frame (e.g. 0, 0, -9.81); it enters the recursion as base acceleration -g
 *   body k at 3 + 27 k:
 *     +0              parent body index (-1 = base), an integer stored as a double
 *     +1              joint type: TBD_REVOLUTE or TBD_PRISMATIC
 *     +2  .. +4       joint axis (unit, joint frame = body frame)
 *     +5  .. +13      E, row-major 3x3: rotation of the joint frame at q = 0 relative to the parent frame
 *                     (maps body-frame coordinates to parent-frame coordinates)
 *     +14 .. +16      r: origin of the joint frame in the parent frame
 *     +17             mass m
 *     +18 .. +20      centre of mass c in the body frame
 *     +21 .. +26      rotational inertia about the centre of mass in the body frame: Ixx, Ixy, Ixz, Iyy, Iyz, Izz
 *
 * The body frame at q is the joint frame moved by the joint: rotated by q about the axis (revolute) or translated by
 * q along it (prismatic).  The model travels to the kernel by value as a __grid_constant__ parameter (no device copy,
 * no __constant__ symbol shared between streams).
 *
 * Frame: a frame rigidly attached to one body (toppra_b200.RigidBodyFrame).  frame_host is a HOST array of
 * TBD_FRAME_DOUBLES doubles:
 *
 *   +0              body index (-1 = the base), an integer stored as a double
 *   +1  .. +9       R, row-major 3x3: orientation of the frame in the body frame (maps frame to body coordinates)
 *   +10 .. +12      p: origin of the frame in the body frame
 *   +13             reference frame of the velocity: TBD_WORLD, TBD_LOCAL or TBD_LOCAL_WORLD_ALIGNED
 *
 * A frame velocity is [linear(3); angular(3)] (pinocchio's Motion::toVector()).  With p_f, R_f the frame's world
 * placement, dp_f the velocity of its origin and w the angular velocity in world coordinates:
 *   TBD_LOCAL_WORLD_ALIGNED   (dp_f, w)
 *   TBD_LOCAL                 (R_f^T dp_f, R_f^T w)
 *   TBD_WORLD                 (dp_f - w x p_f, w): the spatial velocity at the world origin
 * The reference-frame codes are pinocchio's ReferenceFrame values.
 */
#ifndef TOPPRA_B200_DYN_H_
#define TOPPRA_B200_DYN_H_

#ifdef __cplusplus
extern "C" {
#endif

#define TBD_VERSION 100
#define TBD_MAX_BODIES 16
#define TBD_BODY_DOUBLES 27
#define TBD_REVOLUTE 0
#define TBD_PRISMATIC 1
#define TBD_FRAME_DOUBLES 14
#define TBD_WORLD 0
#define TBD_LOCAL 1
#define TBD_LOCAL_WORLD_ALIGNED 2
#define TBD_OBJECT_DOUBLES 10
#define TBD_BASE_DOUBLES 4
#define TBD_POINT_DOUBLES (TBD_FRAME_DOUBLES + 1)
#define TBD_MAX_POINTS 16
#define TBD_MAX_HUMANS 16
#define TBD_CAPSULE_DOUBLES (2 * TBD_FRAME_DOUBLES + 1)
#define TBD_HUMAN_CAPSULE_DOUBLES 7
#define TBD_CAPSULE_PARALLEL 1e-12
#define TBD_DRIVE_DOUBLES(nv) ((nv) * (nv) + 2 * (nv))
#define TBD_KINETIC_ENERGY 0
#define TBD_MOMENTUM 1
#define TBD_COUPLING_DOUBLES(nv, nq) ((nv) * (nq) + (nv))

int tbd_version(void);

/* tau = ID(q, qd, qdd) for M points, one thread per point: Featherstone's spatial RNEA in body coordinates.
 *   q, qd, qdd, tau [M][nv] row-major. */
int tbd_rnea(const double *model_host, int nv, int M, const double *q, const double *qd, const double *qdd, double *tau,
             void *stream);

/* The three inverse-dynamics terms of SecondOrderConstraint (linear_second_order.py) in one launch; the joint transforms
 * are computed once per point and shared by the three passes:
 *   c = ID(q, 0, 0);  a = ID(q, 0, qs) - c;  b = ID(q, qs, qss) - c;  c = c + sign(qs) * friction  (friction != NULL)
 * qs = q', qss = q'' of the path.  Bit-identical to three tbd_rnea launches followed by those element-wise operations.
 *   q, qs, qss, a, b, c [M][nv]; friction (nullable) [nv]. */
int tbd_torque_terms(const double *model_host, int nv, int M, const double *q, const double *qs, const double *qss,
                     const double *friction, double *a, double *b, double *c, void *stream);

/* v = the velocity of the frame frame_host at (q, qd) for M points, one thread per point.
 *   q, qd [M][nv]; v [M][6].  TB_ERR_ARG for a frame body outside [-1, nv) or not an integer, an unknown reference
 *   frame or a non-finite R or p. */
int tbd_frame_velocity(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                       const double *qd, double *v, void *stream);

/* The row of CartesianVelocityNorm: b = v^T (S v) with v the velocity of frame_host at (q, qs = q'), S v row by row,
 * then v . (S v), each sum left to right.  Bit-identical to tbd_frame_velocity followed by that quadratic form.
 *   S_host: HOST array of 36 doubles (6x6 row-major, finite); q, qs [M][nv]; b [M]. */
int tbd_velocity_norm_terms(const double *model_host, int nv, const double *frame_host, const double *S_host, int M,
                            const double *q, const double *qs, double *b, void *stream);

/* acc = the classical acceleration of the frame frame_host at (q, qd, qdd) for M points, one thread per point
 * (pinocchio's getFrameClassicalAcceleration; no gravity, purely kinematic).  [linear(3); angular(3)]: the second time
 * derivative of the frame origin's world position p_f and dw/dt, expressed as
 *   TBD_LOCAL_WORLD_ALIGNED   (d2p_f/dt2, dw/dt)
 *   TBD_LOCAL                 (R_f^T d2p_f/dt2, R_f^T dw/dt)
 * acc = J(q) qdd + dJ(q, qd) qd is affine in (s'', s'^2) along a path: with qd = q' s', qdd = q' s'' + q'' s'^2,
 * acc = acc(q, 0, q') s'' + acc(q, q', q'') s'^2.
 *   q, qd, qdd [M][nv]; acc [M][6].  TB_ERR_UNSUPPORTED for a TBD_WORLD frame; otherwise the checks of
 *   tbd_frame_velocity. */
int tbd_frame_acceleration(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                           const double *qd, const double *qdd, double *acc, void *stream);

/* The rows of CartesianAccelerationConstraint in one launch, one chain walk per point (the joint transforms and their
 * sincos are shared by both states):
 *   a = acc(q, 0, qs);  b = acc(q, qs, qss)
 * restricted to the components of the bit mask `components`: bit j selects component j of [ax, ay, az, wx, wy, wz];
 * the k = popcount(components) columns come in increasing j.  Bit-identical to two tbd_frame_acceleration launches
 * (with qd = 0 and qd = qs) followed by that column selection.
 *   q, qs, qss [M][nv]; a, b [M][k].  TB_ERR_ARG for components outside 1..63; otherwise the checks of
 *   tbd_frame_acceleration. */
int tbd_acceleration_terms(const double *model_host, int nv, const double *frame_host, int components, int M,
                           const double *q, const double *qs, const double *qss, double *a, double *b, void *stream);

/* w = the wrench [f(3); tau(3)] the contact frame frame_host exerts on an object it carries, at (q, qd, qdd) for M
 * points, one thread per point (toppra_b200.constraint.ContactStabilityConstraint).  The frame's origin is the centre
 * of the contact area and its z axis the support normal, pointing into the object.  object_host is a HOST array of
 * TBD_OBJECT_DOUBLES doubles, all in contact-frame coordinates:
 *
 *   +0              mass m
 *   +1  .. +3       r: centre of mass
 *   +4  .. +9       rotational inertia Ic about the centre of mass: Ixx, Ixy, Ixz, Iyy, Iyz, Izz
 *
 * With R_f the frame's world orientation, g_l = R_f^T g (g the model's gravity), a_r the classical acceleration of
 * the centre of mass, w and dw the frame's angular velocity and acceleration, all in frame axes:
 *   f = m (a_r - g_l);  tau = Ic dw + w x (Ic w) + r x f      (tau about the frame origin)
 * The wrench is always in the frame's own axes: the reference-frame field of frame_host (+13) is ignored.
 *   q, qd, qdd [M][nv]; w [M][6].  TB_ERR_ARG for a null or non-finite object or m <= 0; otherwise the model and frame
 *   checks of tbd_frame_acceleration. */
int tbd_contact_wrench(const double *model_host, int nv, const double *frame_host, const double *object_host, int M,
                       const double *q, const double *qd, const double *qdd, double *w, void *stream);

/* The three terms of SecondOrderConstraint with the contact wrench as inverse dynamics, in one launch and one chain
 * walk per point:
 *   c = w(q, 0, 0);  a = w(q, 0, qs) - c;  b = w(q, qs, qss) - c
 * Bit-identical to three tbd_contact_wrench launches followed by the two subtractions.
 *   q, qs, qss [M][nv]; a, b, c [M][6].  The checks of tbd_contact_wrench. */
int tbd_contact_wrench_terms(const double *model_host, int nv, const double *frame_host, const double *object_host,
                             int M, const double *q, const double *qs, const double *qss, double *a, double *b,
                             double *c, void *stream);

/* Lambda_v^-1 = J_v M(q)^-1 J_v^T: the inverse of the operational-space (Khatib) inertia of the origin of frame_host
 * for linear motion, 3x3 row-major, for M points, one thread per point.  J_v (3 x nv) maps qd to the world velocity
 * of the frame origin, M(q) is the joint-space mass matrix of the whole tree.  The robot's effective mass at the
 * origin in the unit direction u is m_R(u) = 1 / (u^T Lambda_v^-1 u).  Expressed in the frame's reference axes:
 *   TBD_LOCAL_WORLD_ALIGNED   Lambda_v^-1 as is (world axes)
 *   TBD_LOCAL                 R_f^T Lambda_v^-1 R_f
 * Computed as M = L L^T (Cholesky, M from the composite-rigid-body algorithm), Y = L^-1 J_v^T, Lambda_v^-1 = Y^T Y:
 * symmetric and positive semi-definite by construction; 0 for a frame on the base.  Where a Cholesky pivot is not
 * positive (M singular or not finite at that q), all nine entries of that point are NaN.
 *   q [M][nv]; Linv [M][9].  TB_ERR_UNSUPPORTED for a TBD_WORLD frame; otherwise the checks of tbd_frame_velocity. */
int tbd_frame_inverse_inertia(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                              double *Linv, void *stream);

/* The row of CollisionEnergyConstraint: the energy a collision at the frame origin could transfer to a human body
 * region of effective mass m_H = human_mass (ISO/TS 15066, Annex A), E = 1/2 mu |v|^2 with
 * mu = (1/m_H + 1/m_R)^-1 and m_R the robot's effective mass in the direction of v, is b s'^2 along a path, with
 *   v = the world linear velocity of the frame origin at (q, qs = q')   (tbd_frame_velocity, first three entries)
 *   vv = v.v;  w = v.(Lambda_v^-1 v), Lambda_v^-1 v row by row;  b = 0.5 * vv * vv / (vv / m_H + w)
 * each sum left to right, and b = +0 where vv == 0 and w is not NaN.  m_H = +inf gives the robot-only energy
 * 1/2 m_R |v|^2.  Bit-identical to tbd_frame_inverse_inertia and tbd_frame_velocity with the frame's reference-frame
 * field set to TBD_LOCAL_WORLD_ALIGNED, followed by those operations; the field of frame_host (+13) is ignored.  NaN
 * where Lambda_v^-1 is NaN.
 *   q, qs [M][nv]; b [M].  TB_ERR_ARG for human_mass not > 0 (NaN included); otherwise the checks of
 *   tbd_frame_velocity. */
int tbd_collision_energy_terms(const double *model_host, int nv, const double *frame_host, double human_mass, int M,
                               const double *q, const double *qs, double *b, void *stream);

/* w = the wrench [f(3); tau(3)] the support exerts on the whole robot, at (q, qd, qdd) for M points, one thread per
 * point (toppra_b200.constraint.SupportStabilityConstraint).  The support frame frame_host is a frame on the base
 * (body -1): its origin lies on the support plane and its z axis is the support normal, pointing into the robot.
 * base_host is a HOST array of TBD_BASE_DOUBLES doubles describing the static base, which the model's bodies leave
 * out:
 *
 *   +0              mass m_b >= 0
 *   +1  .. +3       c_b: centre of mass, base coordinates
 *
 * With R_s, p_s the support frame's placement in base coordinates, g the model's gravity and (f_k, n_k) the force of
 * the recursive Newton-Euler pass (gravity as base acceleration -g) that each root child k would hand to the base:
 *   f_b = sum_k R_k f_k;  n_b = sum_k (R_k n_k + p_k x R_k f_k);  f_b += -m_b g;  n_b += c_b x (-m_b g)
 *   w = [R_s^T f_b; R_s^T (n_b - p_s x f_b)]
 * The wrench is always in support axes: the reference-frame field of frame_host (+13) is ignored.  The zero-moment
 * point (centre of pressure) is (-tau_y / f_z, tau_x / f_z) in support axes.
 *   q, qd, qdd [M][nv]; w [M][6].  TB_ERR_ARG for a frame whose body is not -1, a null or non-finite base or m_b < 0;
 *   otherwise the model and frame checks of tbd_frame_velocity. */
int tbd_support_wrench(const double *model_host, int nv, const double *frame_host, const double *base_host, int M,
                       const double *q, const double *qd, const double *qdd, double *w, void *stream);

/* The three terms of SecondOrderConstraint with the support wrench as inverse dynamics, in one launch; the joint
 * transforms are computed once per point and shared by the three passes:
 *   c = w(q, 0, 0);  a = w(q, 0, qs) - c;  b = w(q, qs, qss) - c
 * Bit-identical to three tbd_support_wrench launches followed by the two subtractions.
 *   q, qs, qss [M][nv]; a, b, c [M][6].  The checks of tbd_support_wrench. */
int tbd_support_wrench_terms(const double *model_host, int nv, const double *frame_host, const double *base_host,
                             int M, const double *q, const double *qs, const double *qss, double *a, double *b,
                             double *c, void *stream);

/* Speed and separation monitoring (ISO/TS 15066 5.5.4; toppra_b200.constraint.SeparationMonitoringConstraint): the
 * surface separation and the approach speed of P robot points and H human spheres, for M points, one thread per point.
 * points_host is a HOST array of P x TBD_POINT_DOUBLES doubles: a packed frame (TBD_FRAME_DOUBLES) followed by the
 * point's radius r_p >= 0.  The point is the sphere about the frame's origin; the frame's reference-frame field (+13)
 * is ignored.  humans is a DEVICE array [NH][H][4] of spheres (c_h(3), r_h) in base coordinates; point m reads set
 * m / points_per_path, or set 0 when points_per_path is 0.  One walk of the tree gives every point's world position x_p
 * and linear velocity v (the linear part of tbd_frame_velocity for a TBD_LOCAL_WORLD_ALIGNED frame at the point), then
 * for each pair, p-major then h, each sum left to right:
 *   e = c_h - x_p;  l = sqrt(e.e);  d = l - r_p - r_h;  w = (e.v) / l, or sqrt(v.v) where l == 0
 * d is the surface separation and w the speed at which the point approaches the sphere's centre.
 *   q, qd [M][nv]; d, w [M][P][H].  TB_ERR_UNSUPPORTED for P or H outside 1..16 (TBD_MAX_POINTS, TBD_MAX_HUMANS);
 *   TB_ERR_ARG for a null pointer, a radius r_p that is not finite or is negative, NH < 1, points_per_path < 0 or a
 *   points_per_path that reads past set NH - 1, and the model and frame checks of tbd_frame_velocity.  The human spheres
 *   are device data and are not checked. */
int tbd_separation(const double *model_host, int nv, const double *points_host, int P, int H, int NH,
                   int points_per_path, int M, const double *q, const double *qd, const double *humans, double *d,
                   double *w, void *stream);

/* The row of SeparationMonitoringConstraint at (q, qs = q'): with the reaction time T_r >= 0, the stopping deceleration
 * a_s > 0, the human speed v_h >= 0 and the clearance C >= 0 (all finite), the separation distance of the standard,
 * S_p = v_h (T_r + T_s) + v_r T_r + v_r^2 / (2 a_s) + C with T_s = v_r / a_s, stays below d for robot speeds up to
 *   vmax = 0 where D <= 0, else 2 a_s D / (sqrt(k^2 + 2 a_s D) + k),   D = d - C - v_h T_r,  k = a_s T_r + v_h
 * and the limit w s' <= vmax binds where w > 0 as w^2 s'^2 <= vmax^2.  Per point, one row a = 0, b, c:
 *   b = w*^2, c = 0 - vmax*^2     for the pair * among those with w > 0 that minimises vmax^2 / w^2 (the first in
 *                                 pair order on ties);
 *   b = 0, c = -1                 where no pair has w > 0 (an inactive row);
 *   b = c = NaN                   where any pair's d or w is NaN.
 * Bit-identical to tbd_separation with qd = qs followed by these float64 operations, in this order, on host scalars
 * vhTr = v_h * T_r, twoa = 2 * a_s, k = a_s * T_r + v_h, kk = k * k:
 *   per pair:  D = d - C;  D = D - vhTr;  num = twoa * D;  vmax = D <= 0 ? 0 : num / (sqrt(kk + num) + k);
 *              w2 = w * w;  v2 = vmax * vmax;
 *              the pair replaces the best (bw2, bv2) when w > 0 and (no best yet or v2 * bw2 < bv2 * w2)
 *   per point: b = bw2, c = 0 - bv2.
 *   q, qs [M][nv]; b, c [M].  TB_ERR_ARG for a parameter out of range (NaN included); otherwise the checks of
 *   tbd_separation. */
int tbd_separation_terms(const double *model_host, int nv, const double *points_host, int P, int H, int NH,
                         int points_per_path, double reaction_time, double stopping_deceleration, double human_speed,
                         double clearance, int M, const double *q, const double *qs, const double *humans, double *b,
                         double *c, void *stream);

/* Speed and separation monitoring with capsules: P robot capsules and H human capsules, for M points, one thread per
 * point.  capsules_host is a HOST array of P x TBD_CAPSULE_DOUBLES doubles: packed frame a, packed frame b (each
 * TBD_FRAME_DOUBLES, reference-frame fields ignored) and the radius r_p >= 0.  The robot capsule is the set of points
 * within r_p of the segment between the two frame origins; the frames may lie on different bodies.  With x_a, v_a and
 * x_b, v_b the world positions and linear velocities of the two origins (the walk of tbd_separation), the point at
 * parameter t is p(t) = x_a + t (x_b - x_a) and its velocity v(t) = v_a + t (v_b - v_a), exact for two moving points.
 * humans is a DEVICE array [NH][H][TBD_HUMAN_CAPSULE_DOUBLES] of capsules (c0(3), c1(3), r_h) in base coordinates, the
 * points within r_h of the segment c0 -> c1, h(tau) = c0 + tau (c1 - c0); sets are read as in tbd_separation.
 *
 * Per pair, capsule-major then h, the closest pair (t, tau) of the two segments (Ericson, Real-Time Collision
 * Detection 5.1.9), each dot product summed left to right, clamp(x) = x < 0 ? 0 : (x > 1 ? 1 : x) (NaN passes):
 *   d1 = x_b - x_a;  d2 = c1 - c0;  r0 = x_a - c0;  a = d1.d1;  e = d2.d2;  f = d2.r0
 *   a == 0:             tau = 0 where e == 0, else clamp(f / e); the pairs (0, tau) and (1, tau) (below): the ends
 *                       coincide, every t is a closest pair, and the ends may move apart (frames on different bodies)
 *   otherwise c = d1.r0, and
 *   e == 0:             tau = 0;  t = clamp(-c / a)            (-c: the negation of c)
 *   otherwise b = d1.d2;  denom = a * e - b * b;
 *     parallel, denom <= TBD_CAPSULE_PARALLEL * a * e (evaluated left to right; an angle below about 1e-6 rad):
 *       t0 = -c / a;  t1 = (b - c) / a;  lo = max(min(t0, t1), 0);  hi = min(max(t0, t1), 1)
 *       lo <= hi:  the pairs (lo, clamp((b * lo + f) / e)) and (hi, clamp((b * hi + f) / e)) (below)
 *       lo > hi:   t = 0, then the re-clamp
 *     not parallel:  t = clamp((b * f - c * e) / denom), then the re-clamp
 *     re-clamp:  tau = (b * t + f) / e;  tau < 0: tau = 0, t = clamp(-c / a);  tau > 1: tau = 1, t = clamp((b - c) / a)
 * then with p = x_a + t * d1, v = v_a + t * (v_b - v_a), h = c0 + tau * d2 (per component) the operations of
 * tbd_separation:  E = h - p;  l = sqrt(E.E);  d = l - r_p - r_h;  w = (E.v) / l, or sqrt(v.v) where l == 0.
 * Parallel segments whose projections overlap, and a robot capsule whose ends coincide, have a segment of closest
 * pairs, along which w is affine in t; the rate at which the distance closes is the largest w over that set (Danskin's
 * theorem), so both ends are evaluated and d = the smaller d, w = the larger w of the two.  A capsule with frame a == frame b and a human capsule with
 * c0 == c1 give the numbers of tbd_separation (signed zeros aside).
 *   q, qd [M][nv]; d, w [M][P][H].  TB_ERR_UNSUPPORTED for P or H outside 1..16; TB_ERR_ARG for a null pointer, a
 *   radius r_p that is not finite or is negative, NH < 1, points_per_path < 0 or a points_per_path that reads past set
 *   NH - 1, and the model and frame checks of tbd_frame_velocity for both frames.  The human capsules are device data
 *   and are not checked.  The capsules travel by value next to the model (32 endpoints, 1160 bytes), which makes the
 *   kernel parameters 4696 bytes here and 4744 bytes in tbd_capsule_separation_terms: above the classic 4 KB, within
 *   the 32 KB that CUDA 12.1+ allows on sm_90a. */
int tbd_capsule_separation(const double *model_host, int nv, const double *capsules_host, int P, int H, int NH,
                           int points_per_path, int M, const double *q, const double *qd, const double *humans,
                           double *d, double *w, void *stream);

/* The row of SeparationMonitoringConstraint at (q, qs = q') with capsules: bit-identical to tbd_capsule_separation
 * with qd = qs followed by the float64 operations of tbd_separation_terms (the same vmax, binding pair in pair order,
 * inactive row and NaN rule).
 *   q, qs [M][nv]; b, c [M].  TB_ERR_ARG for a parameter out of range (NaN included); otherwise the checks of
 *   tbd_capsule_separation. */
int tbd_capsule_separation_terms(const double *model_host, int nv, const double *capsules_host, int P, int H, int NH,
                                 int points_per_path, double reaction_time, double stopping_deceleration,
                                 double human_speed, double clearance, int M, const double *q, const double *qs,
                                 const double *humans, double *b, double *c, void *stream);

/* Geared drives (toppra_b200.Drives; MotorTorqueConstraint, MotorSpeedConstraint): each joint is driven by motors
 * through a constant transmission.  Motor positions are theta = T q with T an invertible nv x nv matrix (a gear
 * ratio n_k on the diagonal; off-diagonal entries couple joints, as in a coupled wrist).  Both sides exchange the same
 * power, so the joint torques tau_j load the motors with T^-T tau_j, and each motor also accelerates its rotor of
 * inertia I_r (rotor gyroscopic terms neglected, as in pinocchio's armature).  drive_host is a HOST array of
 * TBD_DRIVE_DOUBLES(nv) doubles:
 *
 *   [0, nv*nv)            T, row-major
 *   [nv*nv, nv*nv + nv)   I_r: rotor inertia of each motor, finite and >= 0
 *   [nv*nv + nv, ...)     f: Coulomb friction torque of each motor, finite and >= 0
 *
 * Every entry refuses (TB_ERR_ARG) a T with a non-finite entry and a singular T: the entry inverts T on the host in fp64
 * by Gauss-Jordan elimination with partial pivoting and refuses a zero pivot or a non-finite inverse.  T and T^-T travel
 * to the kernel by value next to the model.  Every matrix-vector sum below is taken left to right.
 *
 * tau_m = w(q, qd, qdd) = T^-T ID(q, qd, qdd) + I_r o (T qdd): the motor torques at M points, one thread per point
 * (the RNEA of tbd_rnea, then the motor map, in that order: (T^-T tau)_i + I_r,i (T qdd)_i).
 *   q, qd, qdd, tau_m [M][nv].  TB_ERR_ARG for a null pointer, a bad drive and the model checks of tbd_rnea. */
int tbd_drive_torque(const double *model_host, int nv, const double *drive_host, int M, const double *q,
                     const double *qd, const double *qdd, double *tau_m, void *stream);

/* The three terms of SecondOrderConstraint with the motor torques as inverse dynamics, in one launch; the joint
 * transforms are computed once per point and shared by the three passes:
 *   c = w(q, 0, 0);  a = w(q, 0, qs) - c;  b = w(q, qs, qss) - c;  c = c + f o sign(T qs)
 * Bit-identical to three tbd_drive_torque launches followed by those element-wise operations (sign: 0 at +-0 and NaN).
 * With T = I, I_r = 0 and f the joint friction it equals tbd_torque_terms.
 *   q, qs, qss, a, b, c [M][nv].  The checks of tbd_drive_torque. */
int tbd_drive_torque_terms(const double *model_host, int nv, const double *drive_host, int M, const double *q,
                           const double *qs, const double *qss, double *a, double *b, double *c, void *stream);

/* The motor-speed row at qs = q': |theta'_i| s' <= omega_i for every motor i is x = s'^2 times
 *   b = max_i ((T qs)_i / omega_i)^2 <= 1
 * one row a = 0, b, c = -1 per point with the feasible set of the nv rows.  Per motor: v = (T qs)_i, r = v / omega_i,
 * r * r; the maximum propagates NaN (a NaN in qs gives a NaN b).  omega_i = inf contributes 0 (for a finite v).
 *   speed_limit: HOST array of nv doubles omega_i > 0 (inf allowed); qs [M][nv]; b [M].  TB_ERR_UNSUPPORTED for nv
 *   outside 1..16; TB_ERR_ARG for a null pointer, M <= 0, an omega_i that is not > 0 (NaN included) and a bad drive. */
int tbd_drive_speed_terms(int nv, const double *drive_host, const double *speed_limit, int M, const double *qs,
                          double *b, void *stream);

/* w = the wrench [f(3); n(3)] across joint k, for M points, one thread per point (toppra_b200.constraint.
 * JointWrenchConstraint): the force and moment the parent side of joint k exerts on everything beyond it, with k the
 * moving joint of the body frame_host is attached to.  That subtree is body k and every body below it (with the links
 * folded into them and a payload folded in by the model), and gravity is included: w is the subtree's rate of change of
 * momentum minus its weight, the moment taken about the frame origin.  Bearings and reducers rate the axial force, the
 * radial force and the tilting moment of this wrench; tbd_rnea's tau_k is only its component along the joint axis.
 * With (f_k, n_k) the force of the recursive Newton-Euler pass of tbd_rnea at body k (about body k's origin, body-k
 * coordinates; gravity as base acceleration -g) and (R_f, p_f) the frame's placement in body k:
 *   TBD_LOCAL                 w = [R_f^T f_k; R_f^T (n_k - p_f x f_k)]                   (the frame's own axes)
 *   TBD_LOCAL_WORLD_ALIGNED   w = [R_k f_k; R_k (n_k - p_f x f_k)]                       (world axes)
 * where R_k = R_c0 R_c1 ... R_k is body k's world orientation, the product of the joint rotations along its root chain.
 * The order [f; n] is that of tbd_contact_wrench (tbd_rnea's pass stores [n; f]).
 *   q, qd, qdd [M][nv]; w [M][6].  TB_ERR_UNSUPPORTED for a TBD_WORLD frame; TB_ERR_ARG for a frame on the base
 *   (body -1: its load is the support wrench of tbd_support_wrench); otherwise the checks of tbd_frame_velocity. */
int tbd_joint_wrench(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                     const double *qd, const double *qdd, double *w, void *stream);

/* The three terms of SecondOrderConstraint with the joint wrench as inverse dynamics, in one launch; the joint
 * transforms and the axes are computed once per point and shared by the three passes:
 *   c = w(q, 0, 0);  a = w(q, 0, qs) - c;  b = w(q, qs, qss) - c
 * restricted to the components of the bit mask `components`: bit j selects component j of [fx, fy, fz, nx, ny, nz];
 * the k = popcount(components) columns come in increasing j.  Bit-identical to three tbd_joint_wrench launches
 * followed by the two subtractions and that column selection.
 *   q, qs, qss [M][nv]; a, b, c [M][k].  TB_ERR_ARG for components outside 1..63; otherwise the checks of
 *   tbd_joint_wrench. */
int tbd_joint_wrench_terms(const double *model_host, int nv, const double *frame_host, int components, int M,
                           const double *q, const double *qs, const double *qss, double *a, double *b, double *c,
                           void *stream);

/* The kinetic energy T and the linear momentum p of the whole robot at (q, qd), for M points, one thread per point
 * (toppra_b200.constraint.KineticEnergyConstraint, MomentumConstraint):
 *   T = 1/2 qd^T M(q) qd = 1/2 sum_k (m_k |v_ck|^2 + w_k^T I_ck w_k);   p = sum_k m_k v_ck = m_total v_com
 * summed over the moving bodies (with the links folded into them and a payload folded in by the model; the static base
 * does not move), v_ck the velocity of body k's centre of mass, w_k its angular velocity and I_ck its rotational inertia
 * about the centre of mass.  p is in base axes.  One forward walk of bodies 0..nv-1 gives each body's world rotation
 * Rw_k, angular velocity w_k and origin velocity vo_k (as the walk of tbd_separation); then for each body, in body
 * order, with d = Rw_k c_k, every sum left to right:
 *   v_c = vo_k + w_k x d;  w_b = Rw_k^T w_k;  e += m_k (v_c . v_c) + w_b . (Ic_k w_b);  p += m_k v_c;  T = 0.5 e
 * No mass-matrix inverse is involved: a model whose joints move no inertia is fine.
 *   q, qd [M][nv]; out [M][4] = T, px, py, pz.  TB_ERR_UNSUPPORTED for nv outside 1..16; TB_ERR_ARG for a null pointer,
 *   M <= 0 and the model checks of tbd_rnea. */
int tbd_energy_momentum(const double *model_host, int nv, int M, const double *q, const double *qd, double *out,
                        void *stream);

/* The row of KineticEnergyConstraint or MomentumConstraint at (q, qs = q'): along a path qd = q' s', so T = b s'^2 and
 * |p|^2 = b s'^2 with
 *   which = TBD_KINETIC_ENERGY   b = T(q, qs)
 *   which = TBD_MOMENTUM         b = (px px + py py) + pz pz,  p = p(q, qs)
 * Bit-identical to tbd_energy_momentum followed by that choice.
 *   q, qs [M][nv]; b [M].  TB_ERR_ARG for any other `which`; otherwise the checks of tbd_energy_momentum. */
int tbd_energy_momentum_terms(const double *model_host, int nv, int which, int M, const double *q, const double *qs,
                              double *b, void *stream);

/* Coupled joints (toppra_b200.RigidBodyModel with a coupling: URDF mimic joints, RigidBodyModel.with_coupling): the nv
 * body joint positions are affine in nq <= nv independent path DOFs, q_b = E q + o, so qd_b = E qd and qdd_b = E qdd.
 * A URDF mimic joint is a row of E with one nonzero entry, q_k = multiplier q_src + offset; an uncoupled model is
 * E = I, o = 0.  coupling_host is a HOST array of TBD_COUPLING_DOUBLES(nv, nq) doubles:
 *
 *   [0, nv*nq)            E (nv x nq), row-major
 *   [nv*nq, nv*nq + nv)   o
 *
 * The generalized forces on the DOFs follow from virtual work, tau_q = E^T ID(q_b, qd_b, qdd_b), exact for the
 * holonomic constraint q_b = E q + o: forces inside the mechanism that realises the coupling do no virtual work.
 * Operation order, fixed with __dmul_rn / __dadd_rn whatever the contraction flags:
 *   expansion   (E x)_k: the nonzero terms E[k][j] x[j] in ascending j, starting from the first term (0 for a row
 *               without one); positions then add o[k] where o[k] != 0
 *   reduction   (E^T t)_j: the nonzero terms E[k][j] t[k] in ascending k, starting from the first term
 * With E = I and o = 0 both dynamics entries are bit-identical to tbd_rnea and tbd_torque_terms.  Every entry refuses
 * nq outside 1..nv (TB_ERR_UNSUPPORTED), a non-finite E or o and a zero column of E, a DOF that moves no body
 * (TB_ERR_ARG).  The coupling travels to the kernel by value next to the model (2176 bytes): the kernel parameters are
 * above the classic 4 KB, within the 32 KB that CUDA 12.1+ allows on sm_90a.
 *
 * tau_q = E^T ID(E q + o, E qd, E qdd) for M points, one thread per point: the expansion, the RNEA of tbd_rnea on the
 * nv bodies, then the reduction.
 *   q, qd, qdd, tau [M][nq].  TB_ERR_ARG for a null pointer and the model checks of tbd_rnea, then the coupling's. */
int tbd_coupled_rnea(const double *model_host, int nv, const double *coupling_host, int nq, int M, const double *q,
                     const double *qd, const double *qdd, double *tau, void *stream);

/* The terms of tbd_torque_terms on the nq DOFs, one thread per point, with q_b = E q + o, qs_b = E qs, qss_b = E qss:
 *   c = E^T ID(q_b, 0, 0);  a = E^T (ID(q_b, 0, qs_b) - ID(q_b, 0, 0));  b = E^T (ID(q_b, qs_b, qss_b) - ID(q_b, 0, 0));
 *   c = c + sign(qs) * friction  (friction != NULL, per DOF)
 * the subtractions in body space as in tbd_torque_terms, then the reduction.  Bit-identical to tbd_coupling_expand,
 * tbd_torque_terms without friction on the expanded points, the reduction of a, b and c, then the friction term.
 *   q, qs, qss, a, b, c [M][nq]; friction (nullable) [nq].  The checks of tbd_coupled_rnea. */
int tbd_coupled_torque_terms(const double *model_host, int nv, const double *coupling_host, int nq, int M,
                             const double *q, const double *qs, const double *qss, const double *friction, double *a,
                             double *b, double *c, void *stream);

/* q_out = E q + o, qd_out = E qd, qdd_out = E qdd for M points, one thread per point: the body-space inputs of every
 * other entry on a coupled model.  qd and qd_out (qdd and qdd_out) are both given or both NULL.
 *   q, qd, qdd [M][nq]; q_out, qd_out, qdd_out [M][nv].  TB_ERR_UNSUPPORTED for nv outside 1..16; TB_ERR_ARG for a
 *   null q, q_out or coupling, a rate without its output (or the reverse) and M <= 0; then the coupling's checks. */
int tbd_coupling_expand(int nv, const double *coupling_host, int nq, int M, const double *q, const double *qd,
                        const double *qdd, double *q_out, double *qd_out, double *qdd_out, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* TOPPRA_B200_DYN_H_ */
