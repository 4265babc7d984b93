// tb_dyn.cu — libtoppra_b200_dyn.so: inverse dynamics of a fixed-base rigid-body tree (recursive Newton-Euler), the
// hot path of joint-torque constraints on real robots.  C-ABI and model layout in include/toppra_b200_dyn.h.
//
//   rnea_kernel          tau = ID(q, qd, qdd), one thread per point;
//   torque_terms_kernel  c = ID(q, 0, 0), a = ID(q, 0, q') - c, b = ID(q, q', q'') - c, c += sign(q') friction, one
//                        thread per point; the joint transforms (and their sincos) are computed once per point.
//
// Both kernels run the same two device functions, joint_transforms and rnea_pass, so torque_terms_kernel is bit-identical
// to three rnea_kernel launches followed by the element-wise operations of SecondOrderConstraint (-fmad=false).
//
//   frame_velocity_kernel       v = the 6-D velocity of a frame at (q, qd), one thread per point;
//   velocity_norm_terms_kernel  b = v^T S v at (q, q'), the row of CartesianVelocityNorm, one thread per point.
// Both run frame_velocity, which walks only the frame's root-to-body chain with its state in registers (no local
// arrays); the per-body placement is TB_BODY_TRANSFORM, shared with joint_transforms.
//
//   frame_acceleration_kernel   acc = the classical 6-D acceleration of a frame at (q, qd, qdd), one thread per point;
//   acceleration_terms_kernel   a = acc(q, 0, q'), b = acc(q, q', q''), selected components: the rows of
//                               CartesianAccelerationConstraint, one thread and one chain walk per point.
// Both run frame_acceleration, the same register walk with the angular acceleration and the origin acceleration.
//
//   contact_wrench_kernel        w = the wrench a contact frame exerts on an object it carries, at (q, qd, qdd);
//   contact_wrench_terms_kernel  c = w(q, 0, 0), a = w(q, 0, q') - c, b = w(q, q', q'') - c: the terms of
//                                ContactStabilityConstraint, one thread and one chain walk per point.
// Both run frame_acceleration<NS, true>, which also hands out the frame's orientation and angular velocity, and then
// contact_wrench.
//
//   frame_inverse_inertia_kernel   Lambda_v^-1 = J_v M(q)^-1 J_v^T of a frame origin (3x3), one thread per point;
//   collision_energy_terms_kernel  b = 1/2 |v|^4 / (|v|^2 / m_H + v^T Lambda_v^-1 v) at (q, q'): the row of
//                                  CollisionEnergyConstraint, one thread per point.
// Both run frame_inverse_inertia: the composite-rigid-body mass matrix of the whole tree in per-thread local arrays,
// its Cholesky factor and a forward substitution; the terms kernel adds frame_velocity.
//
//   separation_kernel        d, w = surface separation and approach speed of P robot points and H human spheres at
//                            (q, qd), one thread per point;
//   separation_terms_kernel  the row b, c of SeparationMonitoringConstraint at (q, q') from the same pairs.
// Both run point_states, one walk of the tree's bodies with their world placements and velocities in per-thread local
// arrays, then separation_pair for every pair.
//
//   capsule_separation_kernel        d, w of P robot capsules (segments between two frame origins) and H human
//                                    capsules at (q, qd), one thread per point;
//   capsule_separation_terms_kernel  the row b, c from the same pairs.
// Both run point_states on the 2 P endpoints, then capsule_pair (the closest pair of two segments, then
// separation_pair).  Both terms kernels select the binding pair in separation_row.
//
//   drive_torque_kernel        tau_m = T^-T ID(q, qd, qdd) + I_r o (T qdd), the motor torques of geared drives;
//   drive_torque_terms_kernel  the terms of MotorTorqueConstraint from the same motor map after each of the three passes;
//   drive_speed_terms_kernel   b = max_i ((T q')_i / omega_i)^2, the row of MotorSpeedConstraint (no model).
// The torque kernels run joint_transforms and rnea_pass as rnea_kernel does, then motor_torque.
//
//   joint_wrench_kernel        w = the wrench across the joint of a frame's body (on its whole subtree) at (q, qd, qdd);
//   joint_wrench_terms_kernel  the terms of JointWrenchConstraint, the selected components, from the three passes.
// Both run joint_transforms and rnea_pass as rnea_kernel does, then joint_wrench on the body's force f[k].
//
//   energy_momentum_kernel        T, p = the kinetic energy and the linear momentum of the whole tree at (q, qd);
//   energy_momentum_terms_kernel  b = T or p.p at (q, q'): the row of KineticEnergyConstraint or MomentumConstraint.
// Both run energy_momentum, one forward velocity walk of the tree (no force pass), one thread per point.
//
//   coupled_rnea_kernel          tau_q = E^T ID(E q + o, E qd, E qdd): the torques on the nq independent DOFs of a
//                                linearly coupled model (URDF mimic joints), one thread per point;
//   coupled_torque_terms_kernel  the terms of torque_terms_kernel on the expanded state, reduced by E^T;
//   coupling_expand_kernel       q_b = E q + o and the rates E qd, E qdd: the expanded inputs of every other entry.
// The two dynamics kernels expand into per-thread arrays and run joint_transforms and rnea_pass unchanged;
// coupling_expand and coupling_reduce fix their operation order with __dmul_rn / __dadd_rn.
//
// Featherstone's spatial RNEA in body coordinates: motion vectors (w, v) and forces (n, f) about the body origin.
// X[k] = (R, p): R maps body-k coordinates to parent coordinates, p is the body origin in the parent frame.
//   forward   w = R^T wp,  v = R^T (vp + wp x p),  dw = R^T dwp,  dv = R^T (dvp + dwp x p)  (base: 0, 0, 0, -g),
//             plus the joint's S qd, S qdd and crm(v) S qd;
//             f_k = I a + v x* I v with I the spatial inertia of mass m, COM c and rotational inertia Ic about c;
//   backward  tau_k = S^T f_k;  parent: n += R n_k + p x (R f_k),  f += R f_k.
// The per-body state (12 doubles of motion, 6 of force, 12 of transform) lives in per-thread local arrays indexed by
// body: the tree is walked with a runtime trip count and runtime parents, so the arrays are not register-promoted.
// DESIGN.md ("Rigid-body inverse dynamics") lists the registers and stack of both builds.
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error).  Each library
// carries its own static CUDA runtime, so launch errors are read here (launch_status).
#include <cmath>
#include <cuda_runtime.h>

#include "tb_common.cuh"
#include "../../include/toppra_b200_dyn.h"

namespace tb {
namespace {

constexpr int NB = TBD_MAX_BODIES;
constexpr int THREADS = 128;

// The whole model, passed by value (__grid_constant__): every thread reads the same parameter address (a broadcast).
struct DynModel {
  double body[NB][TBD_BODY_DOUBLES];
  double g[3];
};

__device__ __forceinline__ void cross3(const double *a, const double *b, double *o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// o = R x (R row-major 3x3)
__device__ __forceinline__ void mul3(const double *R, const double *x, double *o) {
  o[0] = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  o[1] = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  o[2] = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
}

// o = R^T x
__device__ __forceinline__ void mul3t(const double *R, const double *x, double *o) {
  o[0] = R[0] * x[0] + R[3] * x[1] + R[6] * x[2];
  o[1] = R[1] * x[0] + R[4] * x[1] + R[7] * x[2];
  o[2] = R[2] * x[0] + R[5] * x[1] + R[8] * x[2];
}

// O = A B (row-major 3x3), each entry summed left to right
__device__ __forceinline__ void mul33(const double *A, const double *B, double *O) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) O[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}

// o = I x with I = (Ixx, Ixy, Ixz, Iyy, Iyz, Izz)
__device__ __forceinline__ void mul_inertia(const double *I, const double *x, double *o) {
  o[0] = I[0] * x[0] + I[1] * x[1] + I[2] * x[2];
  o[1] = I[1] * x[0] + I[3] * x[1] + I[4] * x[2];
  o[2] = I[2] * x[0] + I[4] * x[1] + I[5] * x[2];
}

// Placement (R row-major, p) of body bd in its parent frame at joint position qk: the joint frame (E, r) rotated by qk
// about the axis (sincos, Rodrigues) or translated by qk along it.  Shared by joint_transforms and frame_velocity.  A
// macro, not a function: as a separate function it changes the instruction schedule nvcc gives joint_transforms, and
// rnea_kernel and torque_terms_kernel keep their machine code byte for byte this way.
#define TB_BODY_TRANSFORM(bd, qk, R, p)                                                                                  \
  do {                                                                                                                 \
    const double *ax = (bd) + 2, *E = (bd) + 5, *r = (bd) + 14;                                                        \
    if ((bd)[1] == TBD_REVOLUTE) {                                                                                     \
      double s, c;                                                                                                     \
      sincos((qk), &s, &c);                                                                                            \
      const double t = 1.0 - c;                                                                                        \
      const double J[9] = {t * ax[0] * ax[0] + c,         t * ax[0] * ax[1] - s * ax[2], t * ax[0] * ax[2] + s * ax[1], \
                           t * ax[0] * ax[1] + s * ax[2], t * ax[1] * ax[1] + c,         t * ax[1] * ax[2] - s * ax[0], \
                           t * ax[0] * ax[2] - s * ax[1], t * ax[1] * ax[2] + s * ax[0], t * ax[2] * ax[2] + c};        \
      for (int i = 0; i < 3; ++i)                                                                                      \
        for (int j = 0; j < 3; ++j) (R)[3 * i + j] = E[3 * i] * J[j] + E[3 * i + 1] * J[3 + j] + E[3 * i + 2] * J[6 + j]; \
      (p)[0] = r[0]; (p)[1] = r[1]; (p)[2] = r[2];                                                                     \
    } else {                                                                                                           \
      const double d[3] = {ax[0] * (qk), ax[1] * (qk), ax[2] * (qk)};                                                  \
      double Ed[3];                                                                                                    \
      mul3(E, d, Ed);                                                                                                  \
      for (int i = 0; i < 9; ++i) (R)[i] = E[i];                                                                       \
      (p)[0] = r[0] + Ed[0]; (p)[1] = r[1] + Ed[1]; (p)[2] = r[2] + Ed[2];                                             \
    }                                                                                                                  \
  } while (0)

// X[k] = (R row-major [0, 9), p [9, 12)) of every body at configuration q (one point, nv entries).
__device__ void joint_transforms(const DynModel &m, const int nv, const double *__restrict__ q, double (*X)[12]) {
  for (int k = 0; k < nv; ++k) {
    const double *bd = m.body[k];
    double *R = X[k], *p = X[k] + 9;
    const double qk = q[k];
    TB_BODY_TRANSFORM(bd, qk, R, p);
  }
}

// tau = ID(q, qd, qdd) on the transforms X of q.  st, f: scratch [nv][12], [nv][6].
__device__ void rnea_pass(const DynModel &m, const int nv, const double (*X)[12], const double *qd, const double *qdd,
                          double (*st)[12], double (*f)[6], double *tau) {
  for (int k = 0; k < nv; ++k) {
    const double *bd = m.body[k];
    const int par = (int)bd[0];
    const double *R = X[k], *p = X[k] + 9, *ax = bd + 2;
    double wp[3], vp[3], dwp[3], dvp[3];
    if (par < 0) {
      for (int i = 0; i < 3; ++i) { wp[i] = 0.0; vp[i] = 0.0; dwp[i] = 0.0; dvp[i] = -m.g[i]; }
    } else {
      for (int i = 0; i < 3; ++i) { wp[i] = st[par][i]; vp[i] = st[par][3 + i]; dwp[i] = st[par][6 + i]; dvp[i] = st[par][9 + i]; }
    }
    double t[3], w[3], v[3], dw[3], dv[3];
    cross3(wp, p, t);
    t[0] = vp[0] + t[0]; t[1] = vp[1] + t[1]; t[2] = vp[2] + t[2];
    mul3t(R, t, v);
    mul3t(R, wp, w);
    mul3t(R, dwp, dw);
    cross3(dwp, p, t);
    t[0] = dvp[0] + t[0]; t[1] = dvp[1] + t[1]; t[2] = dvp[2] + t[2];
    mul3t(R, t, dv);
    const double sq[3] = {ax[0] * qd[k], ax[1] * qd[k], ax[2] * qd[k]};
    const double sqq[3] = {ax[0] * qdd[k], ax[1] * qdd[k], ax[2] * qdd[k]};
    const bool revolute = bd[1] == TBD_REVOLUTE;
    if (revolute) {
      for (int i = 0; i < 3; ++i) w[i] = w[i] + sq[i];
      double c1[3], c2[3];
      cross3(w, sq, c1);
      cross3(v, sq, c2);
      for (int i = 0; i < 3; ++i) { dw[i] = dw[i] + sqq[i] + c1[i]; dv[i] = dv[i] + c2[i]; }
    } else {
      for (int i = 0; i < 3; ++i) v[i] = v[i] + sq[i];
      double c1[3];
      cross3(w, sq, c1);
      for (int i = 0; i < 3; ++i) dv[i] = dv[i] + sqq[i] + c1[i];
    }
    for (int i = 0; i < 3; ++i) { st[k][i] = w[i]; st[k][3 + i] = v[i]; st[k][6 + i] = dw[i]; st[k][9 + i] = dv[i]; }
    // f = I a + v x* I v about the body origin
    const double mass = bd[17], *c = bd + 18, *Ic = bd + 21;
    double hl[3], ha[3], fl[3], n[3], u[3];
    cross3(w, c, u);
    for (int i = 0; i < 3; ++i) hl[i] = mass * (v[i] + u[i]);
    mul_inertia(Ic, w, ha);
    cross3(c, hl, u);
    for (int i = 0; i < 3; ++i) ha[i] = ha[i] + u[i];
    cross3(dw, c, u);
    for (int i = 0; i < 3; ++i) fl[i] = mass * (dv[i] + u[i]);
    mul_inertia(Ic, dw, n);
    cross3(c, fl, u);
    for (int i = 0; i < 3; ++i) n[i] = n[i] + u[i];
    double u2[3];
    cross3(w, ha, u);
    cross3(v, hl, u2);
    for (int i = 0; i < 3; ++i) n[i] = n[i] + u[i] + u2[i];
    cross3(w, hl, u);
    for (int i = 0; i < 3; ++i) { fl[i] = fl[i] + u[i]; f[k][i] = n[i]; f[k][3 + i] = fl[i]; }
  }
  for (int k = nv - 1; k >= 0; --k) {
    const double *bd = m.body[k];
    const double *ax = bd + 2;
    const double *fk = bd[1] == TBD_REVOLUTE ? f[k] : f[k] + 3;
    tau[k] = ax[0] * fk[0] + ax[1] * fk[1] + ax[2] * fk[2];
    const int par = (int)bd[0];
    if (par >= 0) {
      const double *R = X[k], *p = X[k] + 9;
      double Rf[3], Rn[3], u[3];
      mul3(R, f[k] + 3, Rf);
      mul3(R, f[k], Rn);
      cross3(p, Rf, u);
      for (int i = 0; i < 3; ++i) { f[par][i] = f[par][i] + Rn[i] + u[i]; f[par][3 + i] = f[par][3 + i] + Rf[i]; }
    }
  }
}

__global__ void __launch_bounds__(THREADS)
rnea_kernel(const __grid_constant__ DynModel m, const int nv, const int M, const double *__restrict__ q,
            const double *__restrict__ qd, const double *__restrict__ qdd, double *__restrict__ tau) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], t[NB];
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, qd + o, qdd + o, st, f, t);
  for (int k = 0; k < nv; ++k) tau[o + k] = t[k];
}

__global__ void __launch_bounds__(THREADS)
torque_terms_kernel(const __grid_constant__ DynModel m, const int nv, const int M, const double *__restrict__ q,
                    const double *__restrict__ qs, const double *__restrict__ qss, const double *__restrict__ friction,
                    double *__restrict__ a, double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], zero[NB], tc[NB], t[NB];
  for (int k = 0; k < nv; ++k) zero[k] = 0.0;
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, zero, zero, st, f, tc);
  rnea_pass(m, nv, X, zero, qs + o, st, f, t);
  for (int k = 0; k < nv; ++k) a[o + k] = t[k] - tc[k];
  rnea_pass(m, nv, X, qs + o, qss + o, st, f, t);
  for (int k = 0; k < nv; ++k) b[o + k] = t[k] - tc[k];
  for (int k = 0; k < nv; ++k) {
    double ck = tc[k];
    if (friction) {
      const double x = qs[o + k];
      const double sgn = (double)((0.0 < x) - (x < 0.0));   // torch.sign: 0 at +-0 and NaN
      ck = ck + sgn * friction[k];
    }
    c[o + k] = ck;
  }
}

// A frame rigidly attached to one body, passed by value next to the model: its placement (R, p) in the body frame, the
// bodies from the root to that body (chain[0, n); n = 0 for a frame on the base), the reference frame of the result and,
// for tbd_velocity_norm_terms, the 6x6 weight S.
struct DynFrame {
  double R[9], p[3], S[36];
  int chain[NB];
  int n, ref;
};

// v = [linear(3); angular(3)] velocity of frame f at (q, qd), in f's reference frame.  Walks f's chain from the root
// with the world placement (Rw, pw), the angular velocity w and the body-origin velocity vo in registers; the only
// runtime indices are the model's body indices of the chain, never a function of q.
__device__ __forceinline__ void frame_velocity(const DynModel &m, const DynFrame &f, const double *__restrict__ q,
                                               const double *__restrict__ qd, double *v) {
  double Rw[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, pw[3] = {0.0, 0.0, 0.0};
  double w[3] = {0.0, 0.0, 0.0}, vo[3] = {0.0, 0.0, 0.0};
  for (int i = 0; i < f.n; ++i) {
    const int k = f.chain[i];
    const double *bd = m.body[k];
    double R[9], p[3], d[3], t[3], Rn[9];
    const double qk = q[k];
    TB_BODY_TRANSFORM(bd, qk, R, p);
    mul3(Rw, p, d);                     // origin of body k relative to its parent's, world coordinates
    cross3(w, d, t);
    for (int j = 0; j < 3; ++j) { pw[j] = pw[j] + d[j]; vo[j] = vo[j] + t[j]; }
    mul33(Rw, R, Rn);
    for (int j = 0; j < 9; ++j) Rw[j] = Rn[j];
    double s[3];
    mul3(Rw, bd + 2, s);                // joint axis, world coordinates
    const double qdk = qd[k];
    if (bd[1] == TBD_REVOLUTE) {
      for (int j = 0; j < 3; ++j) w[j] = w[j] + s[j] * qdk;
    } else {
      for (int j = 0; j < 3; ++j) vo[j] = vo[j] + s[j] * qdk;
    }
  }
  double d[3], t[3], pd[3];
  mul3(Rw, f.p, d);                     // frame origin relative to the body origin, world coordinates
  cross3(w, d, t);
  for (int j = 0; j < 3; ++j) pd[j] = vo[j] + t[j];
  if (f.ref == TBD_LOCAL) {
    double Rf[9];
    mul33(Rw, f.R, Rf);
    mul3t(Rf, pd, v);
    mul3t(Rf, w, v + 3);
  } else if (f.ref == TBD_WORLD) {
    double pf[3];
    for (int j = 0; j < 3; ++j) pf[j] = pw[j] + d[j];
    cross3(w, pf, t);
    for (int j = 0; j < 3; ++j) { v[j] = pd[j] - t[j]; v[3 + j] = w[j]; }
  } else {                              // TBD_LOCAL_WORLD_ALIGNED
    for (int j = 0; j < 3; ++j) { v[j] = pd[j]; v[3 + j] = w[j]; }
  }
}

__global__ void __launch_bounds__(THREADS)
frame_velocity_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv, const int M,
                      const double *__restrict__ q, const double *__restrict__ qd, double *__restrict__ v) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[6];
  frame_velocity(m, f, q + o, qd + o, x);
  for (int j = 0; j < 6; ++j) v[(size_t)pt * 6 + j] = x[j];
}

// b = v^T (S v) at (q, q'): S v row by row, then v . (S v), each sum left to right (cartesian_velocity_norm.cpp).
__global__ void __launch_bounds__(THREADS)
velocity_norm_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv,
                           const int M, const double *__restrict__ q, const double *__restrict__ qs,
                           double *__restrict__ b) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[6];
  frame_velocity(m, f, q + o, qs + o, x);
  double acc = 0.0;
  for (int i = 0; i < 6; ++i) {
    double sv = f.S[6 * i] * x[0];
    for (int j = 1; j < 6; ++j) sv = sv + f.S[6 * i + j] * x[j];
    acc = i == 0 ? x[0] * sv : acc + x[i] * sv;
  }
  b[pt] = acc;
}

// The classical acceleration [linear(3); angular(3)] of frame f at NS states (qd[s], qdd[s]) of one configuration q,
// in f's reference frame (TBD_LOCAL or TBD_LOCAL_WORLD_ALIGNED; TBD_WORLD is refused on the host).  One walk of f's
// chain from the root: the world rotation Rw and the joint transforms (with their sincos) are shared by the states,
// each of which keeps w, dw and the body-origin acceleration ao in registers, in world coordinates.  For body k with
// d = Rw p_k from the parent's Rw:
//   ao += dw x d + w x (w x d);  Rw = Rw R_k;  s = Rw axis_k;
//   revolute   dw += s qdd_k + w x (s qd_k);  w += s qd_k
//   prismatic  ao += s qdd_k + 2 w x (s qd_k)
// and at the frame origin, d = Rw p_f:  a_f = ao + dw x d + w x (w x d).  A null qd[s] stands for qd = 0: the state
// then runs the same operations on a literal 0.0, so its result is bit-identical to a call with a zero array.
// ROT (the contact wrench; f.ref is TBD_LOCAL): also hands out the frame's world orientation Rf_out = Rw R_f and each
// state's angular velocity in frame axes, wl[s] = Rf^T w; a null qdd[s] then stands for qdd = 0 like a null qd[s].
template <int NS, bool ROT = false>
__device__ __forceinline__ void frame_acceleration(const DynModel &m, const DynFrame &f, const double *__restrict__ q,
                                                   const double *const (&qd)[NS], const double *const (&qdd)[NS],
                                                   double (&acc)[NS][6], double (*wl)[3] = nullptr,
                                                   double *Rf_out = nullptr) {
  double Rw[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
  double w[NS][3], dw[NS][3], ao[NS][3];
  for (int s = 0; s < NS; ++s)
    for (int j = 0; j < 3; ++j) { w[s][j] = 0.0; dw[s][j] = 0.0; ao[s][j] = 0.0; }
  for (int i = 0; i < f.n; ++i) {
    const int k = f.chain[i];
    const double *bd = m.body[k];
    double R[9], p[3], d[3], Rn[9];
    const double qk = q[k];
    TB_BODY_TRANSFORM(bd, qk, R, p);
    mul3(Rw, p, d);                     // origin of body k relative to its parent's, world coordinates
    for (int s = 0; s < NS; ++s) {
      double t1[3], t2[3], t3[3];
      cross3(dw[s], d, t1);
      cross3(w[s], d, t2);
      cross3(w[s], t2, t3);
      for (int j = 0; j < 3; ++j) ao[s][j] = ao[s][j] + t1[j] + t3[j];
    }
    mul33(Rw, R, Rn);
    for (int j = 0; j < 9; ++j) Rw[j] = Rn[j];
    double sx[3];
    mul3(Rw, bd + 2, sx);               // joint axis, world coordinates
    const bool revolute = bd[1] == TBD_REVOLUTE;
    for (int s = 0; s < NS; ++s) {
      const double qdk = qd[s] ? qd[s][k] : 0.0, qddk = (ROT && !qdd[s]) ? 0.0 : qdd[s][k];
      double sq[3], c[3];
      for (int j = 0; j < 3; ++j) sq[j] = sx[j] * qdk;
      cross3(w[s], sq, c);
      if (revolute) {
        for (int j = 0; j < 3; ++j) { dw[s][j] = dw[s][j] + sx[j] * qddk + c[j]; w[s][j] = w[s][j] + sq[j]; }
      } else {
        for (int j = 0; j < 3; ++j) ao[s][j] = ao[s][j] + sx[j] * qddk + 2.0 * c[j];
      }
    }
  }
  double d[3], Rf[9];
  mul3(Rw, f.p, d);                     // frame origin relative to the body origin, world coordinates
  if (ROT || f.ref == TBD_LOCAL) mul33(Rw, f.R, Rf);
  for (int s = 0; s < NS; ++s) {
    double t1[3], t2[3], t3[3], af[3];
    cross3(dw[s], d, t1);
    cross3(w[s], d, t2);
    cross3(w[s], t2, t3);
    for (int j = 0; j < 3; ++j) af[j] = ao[s][j] + t1[j] + t3[j];
    if (ROT || f.ref == TBD_LOCAL) {
      mul3t(Rf, af, acc[s]);
      mul3t(Rf, dw[s], acc[s] + 3);
      if constexpr (ROT) mul3t(Rf, w[s], wl[s]);
    } else {                            // TBD_LOCAL_WORLD_ALIGNED
      for (int j = 0; j < 3; ++j) { acc[s][j] = af[j]; acc[s][3 + j] = dw[s][j]; }
    }
  }
  if constexpr (ROT)
    for (int j = 0; j < 9; ++j) Rf_out[j] = Rf[j];
}

__global__ void __launch_bounds__(THREADS)
frame_acceleration_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv,
                          const int M, const double *__restrict__ q, const double *__restrict__ qd,
                          const double *__restrict__ qdd, double *__restrict__ acc) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  const double *const qds[1] = {qd + o}, *const qdds[1] = {qdd + o};
  double x[1][6];
  frame_acceleration<1>(m, f, q + o, qds, qdds, x);
  for (int j = 0; j < 6; ++j) acc[(size_t)pt * 6 + j] = x[0][j];
}

// a = acc(q, 0, q'), b = acc(q, q', q''): the rows of CartesianAccelerationConstraint, the components of bit mask
// `components` in increasing order (k = popcount columns).  One chain walk for both states.
__global__ void __launch_bounds__(THREADS)
acceleration_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv,
                          const int components, const int k, const int M, const double *__restrict__ q,
                          const double *__restrict__ qs, const double *__restrict__ qss, double *__restrict__ a,
                          double *__restrict__ b) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  const double *const qds[2] = {nullptr, qs + o}, *const qdds[2] = {qs + o, qss + o};
  double x[2][6];
  frame_acceleration<2>(m, f, q + o, qds, qdds, x);
  double *ao = a + (size_t)pt * k, *bo = b + (size_t)pt * k;
  int c = 0;
  for (int j = 0; j < 6; ++j)
    if ((components >> j) & 1) { ao[c] = x[0][j]; bo[c] = x[1][j]; ++c; }
}

// An object rigidly held by a contact frame (include/toppra_b200_dyn.h): mass, centre of mass r and rotational inertia
// Ic about it, both in contact-frame axes.
struct DynObject {
  double mass, r[3], Ic[6];
};

// The wrench [f; tau] the contact frame exerts on the object, at the frame origin in frame axes, from the frame's
// classical acceleration acc = [a_f; dw] and angular velocity wl (frame axes, frame_acceleration<NS, true>) and
// gl = Rf^T g:
//   a_r = a_f + dw x r + w x (w x r);  f = m (a_r - gl);  tau = Ic dw + w x (Ic w) + r x f.
__device__ __forceinline__ void contact_wrench(const DynObject &o, const double *gl, const double *acc, const double *wl,
                                               double *out) {
  double t1[3], t2[3], t3[3], f[3], n[3], Iw[3];
  cross3(acc + 3, o.r, t1);
  cross3(wl, o.r, t2);
  cross3(wl, t2, t3);
  for (int j = 0; j < 3; ++j) f[j] = o.mass * (acc[j] + t1[j] + t3[j] - gl[j]);
  mul_inertia(o.Ic, acc + 3, n);
  mul_inertia(o.Ic, wl, Iw);
  cross3(wl, Iw, t1);
  cross3(o.r, f, t2);
  for (int j = 0; j < 3; ++j) { out[j] = f[j]; out[3 + j] = n[j] + t1[j] + t2[j]; }
}

__global__ void __launch_bounds__(THREADS)
contact_wrench_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f,
                      const __grid_constant__ DynObject obj, const int nv, const int M, const double *__restrict__ q,
                      const double *__restrict__ qd, const double *__restrict__ qdd, double *__restrict__ w) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  const double *const qds[1] = {qd + o}, *const qdds[1] = {qdd + o};
  double x[1][6], wl[1][3], Rf[9], gl[3], y[6];
  frame_acceleration<1, true>(m, f, q + o, qds, qdds, x, wl, Rf);
  mul3t(Rf, m.g, gl);
  contact_wrench(obj, gl, x[0], wl[0], y);
  for (int j = 0; j < 6; ++j) w[(size_t)pt * 6 + j] = y[j];
}

// c = w(q, 0, 0), a = w(q, 0, q') - c, b = w(q, q', q'') - c: the terms of ContactStabilityConstraint, one chain walk
// for the three states.
__global__ void __launch_bounds__(THREADS)
contact_wrench_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f,
                            const __grid_constant__ DynObject obj, const int nv, const int M,
                            const double *__restrict__ q, const double *__restrict__ qs, const double *__restrict__ qss,
                            double *__restrict__ a, double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  const double *const qds[3] = {nullptr, nullptr, qs + o}, *const qdds[3] = {nullptr, qs + o, qss + o};
  double x[3][6], wl[3][3], Rf[9], gl[3], y[3][6];
  frame_acceleration<3, true>(m, f, q + o, qds, qdds, x, wl, Rf);
  mul3t(Rf, m.g, gl);
  for (int s = 0; s < 3; ++s) contact_wrench(obj, gl, x[s], wl[s], y[s]);
  const size_t r = (size_t)pt * 6;
  for (int j = 0; j < 6; ++j) { c[r + j] = y[0][j]; a[r + j] = y[1][j] - y[0][j]; b[r + j] = y[2][j] - y[0][j]; }
}

// Lambda_v^-1 = J_v M(q)^-1 J_v^T (3x3 row-major) of the origin of frame f at q, in world axes, or in frame axes
// R_f^T (.) R_f when f.ref is TBD_LOCAL.  False, with every entry NaN, where a Cholesky pivot of M is not positive.
//   J_v     the chain walk of frame_velocity on the transforms X: column k is s_k x (p_f - o_k) (revolute) or s_k
//           (prismatic) for the bodies on f's chain, 0 elsewhere (s_k the world joint axis, o_k the body origin);
//   M(q)    the composite-rigid-body algorithm in body coordinates: every body's inertia (m, h = m c, Io about the
//           body origin) is folded into its parent's, then F = Ic_k S_k is carried up to the root, M_kj = S_j^T F;
//   M = L L^T in place (packed lower triangle), Y = L^-1 J_v^T by forward substitution, Lambda_v^-1 = Y^T Y.
// Every sum is taken left to right.  M couples all bodies, so the whole tree is walked, not only f's chain.
__device__ bool frame_inverse_inertia(const DynModel &m, const DynFrame &f, const int nv, const double *__restrict__ q,
                                      double *Linv) {
  double X[NB][12], ic[NB][10], L[NB * (NB + 1) / 2], Y[NB][3];
  joint_transforms(m, nv, q, X);
  // J_v^T into Y: world placement of f's chain, joint axes and origins
  double Rw[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, pw[3] = {0.0, 0.0, 0.0};
  double s[NB][3], o[NB][3];
  for (int k = 0; k < nv; ++k)
    for (int j = 0; j < 3; ++j) Y[k][j] = 0.0;
  for (int i = 0; i < f.n; ++i) {
    const int k = f.chain[i];
    const double *R = X[k], *p = X[k] + 9;
    double d[3], Rn[9];
    mul3(Rw, p, d);
    for (int j = 0; j < 3; ++j) pw[j] = pw[j] + d[j];
    mul33(Rw, R, Rn);
    for (int j = 0; j < 9; ++j) Rw[j] = Rn[j];
    mul3(Rw, m.body[k] + 2, s[i]);
    for (int j = 0; j < 3; ++j) o[i][j] = pw[j];
  }
  double pf[3], d[3];
  mul3(Rw, f.p, d);
  for (int j = 0; j < 3; ++j) pf[j] = pw[j] + d[j];
  for (int i = 0; i < f.n; ++i) {
    const int k = f.chain[i];
    if (m.body[k][1] == TBD_REVOLUTE) {
      const double r[3] = {pf[0] - o[i][0], pf[1] - o[i][1], pf[2] - o[i][2]};
      cross3(s[i], r, Y[k]);
    } else {
      for (int j = 0; j < 3; ++j) Y[k][j] = s[i][j];
    }
  }
  // composite inertias: (m, h, Io = Ixx, Ixy, Ixz, Iyy, Iyz, Izz about the body origin), body coordinates
  for (int k = 0; k < nv; ++k) {
    const double *bd = m.body[k];
    const double mass = bd[17], *c = bd + 18, *Ic = bd + 21;
    double *e = ic[k];
    e[0] = mass;
    for (int j = 0; j < 3; ++j) e[1 + j] = mass * c[j];
    // Io = Ic + m (|c|^2 I - c c^T)
    const double cc = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
    e[4] = Ic[0] + mass * (cc - c[0] * c[0]);
    e[5] = Ic[1] - mass * (c[0] * c[1]);
    e[6] = Ic[2] - mass * (c[0] * c[2]);
    e[7] = Ic[3] + mass * (cc - c[1] * c[1]);
    e[8] = Ic[4] - mass * (c[1] * c[2]);
    e[9] = Ic[5] + mass * (cc - c[2] * c[2]);
  }
  for (int k = nv - 1; k >= 0; --k) {
    const int par = (int)m.body[k][0];
    if (par < 0) continue;
    // parent coordinates: h' = R h + m p;  Io' = R Io R^T + m (|p|^2 I - p p^T) + 2 (p.hr) I - p hr^T - hr p^T
    const double *R = X[k], *p = X[k] + 9, *e = ic[k];
    double hr[3], A[9], B[9];
    mul3(R, e + 1, hr);
    const double I3[9] = {e[4], e[5], e[6], e[5], e[7], e[8], e[6], e[8], e[9]};
    const double Rt[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]};
    mul33(R, I3, A);
    mul33(A, Rt, B);
    const double pp = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
    const double ph = p[0] * hr[0] + p[1] * hr[1] + p[2] * hr[2];
    const double diag = e[0] * pp + 2.0 * ph;
    double *t = ic[par];
    t[0] = t[0] + e[0];
    for (int j = 0; j < 3; ++j) t[1 + j] = t[1 + j] + (hr[j] + e[0] * p[j]);
    const int rr[6] = {0, 0, 0, 1, 1, 2}, cc[6] = {0, 1, 2, 1, 2, 2};
    for (int j = 0; j < 6; ++j) {
      const int r = rr[j], c = cc[j];
      double v = B[3 * r + c] - (e[0] * p[r] * p[c] + p[r] * hr[c] + hr[r] * p[c]);
      if (r == c) v = v + diag;
      t[4 + j] = t[4 + j] + v;
    }
  }
  // M: F = Ic_k S_k = (n, f) about body k's origin, carried up the tree
  for (int k = 0; k < nv; ++k) {
    const double *bd = m.body[k], *ax = bd + 2, *e = ic[k];
    double n[3], fl[3];
    if (bd[1] == TBD_REVOLUTE) {
      mul_inertia(e + 4, ax, n);
      cross3(ax, e + 1, fl);
    } else {
      cross3(e + 1, ax, n);
      for (int j = 0; j < 3; ++j) fl[j] = e[0] * ax[j];
    }
    int j = k;
    for (;;) {
      const double *bj = m.body[j], *aj = bj + 2;
      const double *g = bj[1] == TBD_REVOLUTE ? n : fl;
      L[k * (k + 1) / 2 + j] = aj[0] * g[0] + aj[1] * g[1] + aj[2] * g[2];
      const int par = (int)bj[0];
      if (par < 0) break;
      const double *R = X[j], *p = X[j] + 9;
      double Rf[3], Rn[3], u[3];
      mul3(R, fl, Rf);
      mul3(R, n, Rn);
      cross3(p, Rf, u);
      for (int i = 0; i < 3; ++i) { n[i] = Rn[i] + u[i]; fl[i] = Rf[i]; }
      for (int i = par + 1; i < j; ++i) L[k * (k + 1) / 2 + i] = 0.0;   // bodies off k's chain to the root
      j = par;
    }
    for (int i = 0; i < j; ++i) L[k * (k + 1) / 2 + i] = 0.0;
  }
  // M = L L^T (packed lower triangle, row k at k (k + 1) / 2), then Y = L^-1 J_v^T
  bool ok = true;
  for (int j = 0; j < nv && ok; ++j) {
    double *Lj = L + j * (j + 1) / 2;
    double dd = Lj[j];
    for (int k = 0; k < j; ++k) dd = dd - Lj[k] * Lj[k];
    if (!(dd > 0.0)) { ok = false; break; }
    Lj[j] = sqrt(dd);
    for (int i = j + 1; i < nv; ++i) {
      double *Li = L + i * (i + 1) / 2;
      double v = Li[j];
      for (int k = 0; k < j; ++k) v = v - Li[k] * Lj[k];
      Li[j] = v / Lj[j];
    }
  }
  if (!ok) {
    for (int j = 0; j < 9; ++j) Linv[j] = nan("");
    return false;
  }
  for (int i = 0; i < nv; ++i) {
    const double *Li = L + i * (i + 1) / 2;
    for (int c = 0; c < 3; ++c) {
      double v = Y[i][c];
      for (int k = 0; k < i; ++k) v = v - Li[k] * Y[k][c];
      Y[i][c] = v / Li[i];
    }
  }
  double W[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double v = Y[0][r] * Y[0][c];
      for (int i = 1; i < nv; ++i) v = v + Y[i][r] * Y[i][c];
      W[3 * r + c] = v;
    }
  if (f.ref == TBD_LOCAL) {
    double Rf[9], T[9];
    mul33(Rw, f.R, Rf);
    mul33(W, Rf, T);
    const double Rft[9] = {Rf[0], Rf[3], Rf[6], Rf[1], Rf[4], Rf[7], Rf[2], Rf[5], Rf[8]};
    mul33(Rft, T, Linv);                                               // R_f^T W R_f
  } else {
    for (int j = 0; j < 9; ++j) Linv[j] = W[j];
  }
  return true;
}

__global__ void __launch_bounds__(THREADS)
frame_inverse_inertia_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv,
                             const int M, const double *__restrict__ q, double *__restrict__ Linv) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  double W[9];
  frame_inverse_inertia(m, f, nv, q + (size_t)pt * nv, W);
  for (int j = 0; j < 9; ++j) Linv[(size_t)pt * 9 + j] = W[j];
}

// b = 1/2 vv^2 / (vv / m_H + w) with v the world linear velocity of f at (q, q'), vv = v.v, w = v.(Lambda_v^-1 v)
// (Lambda_v^-1 v row by row), each sum left to right; b = +0 where vv == 0 and w is not NaN.  f.ref is
// TBD_LOCAL_WORLD_ALIGNED (set on the host).
__global__ void __launch_bounds__(THREADS)
collision_energy_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame f, const int nv,
                              const double human_mass, const int M, const double *__restrict__ q,
                              const double *__restrict__ qs, double *__restrict__ b) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double W[9], x[6];
  frame_inverse_inertia(m, f, nv, q + o, W);
  frame_velocity(m, f, q + o, qs + o, x);
  const double vv = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
  double Wv[3];
  for (int i = 0; i < 3; ++i) Wv[i] = W[3 * i] * x[0] + W[3 * i + 1] * x[1] + W[3 * i + 2] * x[2];
  const double w = x[0] * Wv[0] + x[1] * Wv[1] + x[2] * Wv[2];
  b[pt] = (vv == 0.0 && !isnan(w)) ? 0.0 : 0.5 * vv * vv / (vv / human_mass + w);
}

// The static base under the moving tree (include/toppra_b200_dyn.h): mass and centre of mass in base coordinates.
struct DynBase {
  double mass, c[3];
};

// The wrench [f; tau] the support exerts on the whole robot, at the origin of the support frame s (a frame on the base)
// in its axes, from the forces f of a finished rnea_pass.  rnea_pass carries each body's force up to its parent and
// drops it at the base, so f[k] of a root child k is then the wrench of k's whole subtree about k's origin, in k's
// coordinates:
//   f_b = sum_k R_k f_k,  n_b = sum_k R_k n_k + p_k x R_k f_k   (root children k, in base coordinates)
//   f_b += -m_b g;  n_b += c_b x (-m_b g)                       (the static base's weight)
//   w = [R_s^T f_b; R_s^T (n_b - p_s x f_b)]
// Every sum is taken in body order, left to right.
__device__ __forceinline__ void support_wrench(const DynModel &m, const DynFrame &s, const DynBase &base, const int nv,
                                               const double (*X)[12], const double (*f)[6], double *out) {
  double fb[3] = {0.0, 0.0, 0.0}, nb[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < nv; ++k) {
    if ((int)m.body[k][0] >= 0) continue;
    const double *R = X[k], *p = X[k] + 9;
    double Rf[3], Rn[3], u[3];
    mul3(R, f[k] + 3, Rf);
    mul3(R, f[k], Rn);
    cross3(p, Rf, u);
    for (int i = 0; i < 3; ++i) { nb[i] = nb[i] + Rn[i] + u[i]; fb[i] = fb[i] + Rf[i]; }
  }
  double wb[3], u[3], t[3];
  for (int i = 0; i < 3; ++i) wb[i] = -(base.mass * m.g[i]);
  cross3(base.c, wb, u);
  for (int i = 0; i < 3; ++i) { nb[i] = nb[i] + u[i]; fb[i] = fb[i] + wb[i]; }
  cross3(s.p, fb, u);
  for (int i = 0; i < 3; ++i) t[i] = nb[i] - u[i];
  mul3t(s.R, fb, out);
  mul3t(s.R, t, out + 3);
}

__global__ void __launch_bounds__(THREADS)
support_wrench_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame s,
                      const __grid_constant__ DynBase base, const int nv, const int M, const double *__restrict__ q,
                      const double *__restrict__ qd, const double *__restrict__ qdd, double *__restrict__ w) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], t[NB], y[6];
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, qd + o, qdd + o, st, f, t);
  support_wrench(m, s, base, nv, X, f, y);
  for (int j = 0; j < 6; ++j) w[(size_t)pt * 6 + j] = y[j];
}

// c = w(q, 0, 0), a = w(q, 0, q') - c, b = w(q, q', q'') - c: the terms of SupportStabilityConstraint; the joint
// transforms (and their sincos) are computed once per point and shared by the three passes.
__global__ void __launch_bounds__(THREADS)
support_wrench_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame s,
                            const __grid_constant__ DynBase base, const int nv, const int M,
                            const double *__restrict__ q, const double *__restrict__ qs, const double *__restrict__ qss,
                            double *__restrict__ a, double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], zero[NB], t[NB], y0[6], y[6];
  for (int k = 0; k < nv; ++k) zero[k] = 0.0;
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, zero, zero, st, f, t);
  support_wrench(m, s, base, nv, X, f, y0);
  const size_t r = (size_t)pt * 6;
  for (int j = 0; j < 6; ++j) c[r + j] = y0[j];
  rnea_pass(m, nv, X, zero, qs + o, st, f, t);
  support_wrench(m, s, base, nv, X, f, y);
  for (int j = 0; j < 6; ++j) a[r + j] = y[j] - y0[j];
  rnea_pass(m, nv, X, qs + o, qss + o, st, f, t);
  support_wrench(m, s, base, nv, X, f, y);
  for (int j = 0; j < 6; ++j) b[r + j] = y[j] - y0[j];
}

// The robot points of speed and separation monitoring (include/toppra_b200_dyn.h), passed by value: each point's body
// (-1 = the base), the origin p of its frame in body coordinates and its radius.  Bodies [0, top) cover every point's
// chain (parents come first), so the walk stops there.  NP points at most: the P spheres of tbd_separation, or the 2 P
// endpoints of tbd_capsule_separation (capsule i = points 2 i and 2 i + 1, its radius in r[2 i]).
template <int NP>
struct DynPointSet {
  double p[NP][3], r[NP];
  int body[NP];
  int n, top;
};
struct DynPoints : DynPointSet<TBD_MAX_POINTS> {};
struct DynCapsules : DynPointSet<2 * TBD_MAX_POINTS> {};

// World position x and linear velocity v of every point at (q, qd): one walk of the tree's bodies [0, top) with each
// body's world placement (Rw, pw), angular velocity w and origin velocity vo in per-thread local arrays.  The per-body
// operations are those of frame_velocity on a chain, so v is bit-identical to the linear part of tbd_frame_velocity
// for a TBD_LOCAL_WORLD_ALIGNED frame at the point.
template <int NP>
__device__ __forceinline__ void point_states(const DynModel &m, const DynPointSet<NP> &pts, const double *__restrict__ q,
                                             const double *__restrict__ qd, double (*x)[3], double (*v)[3]) {
  double Rw[NB][9], pw[NB][3], w[NB][3], vo[NB][3];
  for (int k = 0; k < pts.top; ++k) {
    const double *bd = m.body[k];
    const int par = (int)bd[0];
    double Rp[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, pp[3] = {0.0, 0.0, 0.0};
    double wp[3] = {0.0, 0.0, 0.0}, vp[3] = {0.0, 0.0, 0.0};
    if (par >= 0) {
      for (int j = 0; j < 9; ++j) Rp[j] = Rw[par][j];
      for (int j = 0; j < 3; ++j) { pp[j] = pw[par][j]; wp[j] = w[par][j]; vp[j] = vo[par][j]; }
    }
    double R[9], p[3], d[3], t[3];
    const double qk = q[k];
    TB_BODY_TRANSFORM(bd, qk, R, p);
    mul3(Rp, p, d);                     // origin of body k relative to its parent's, world coordinates
    cross3(wp, d, t);
    for (int j = 0; j < 3; ++j) { pw[k][j] = pp[j] + d[j]; vo[k][j] = vp[j] + t[j]; }
    mul33(Rp, R, Rw[k]);
    double s[3];
    mul3(Rw[k], bd + 2, s);             // joint axis, world coordinates
    const double qdk = qd[k];
    if (bd[1] == TBD_REVOLUTE) {
      for (int j = 0; j < 3; ++j) { w[k][j] = wp[j] + s[j] * qdk; }
    } else {
      for (int j = 0; j < 3; ++j) { w[k][j] = wp[j]; vo[k][j] = vo[k][j] + s[j] * qdk; }
    }
  }
  for (int i = 0; i < pts.n; ++i) {
    const int k = pts.body[i];
    if (k < 0) {
      for (int j = 0; j < 3; ++j) { x[i][j] = pts.p[i][j]; v[i][j] = 0.0; }
      continue;
    }
    double d[3], t[3];
    mul3(Rw[k], pts.p[i], d);           // point relative to the body origin, world coordinates
    cross3(w[k], d, t);
    for (int j = 0; j < 3; ++j) { x[i][j] = pw[k][j] + d[j]; v[i][j] = vo[k][j] + t[j]; }
  }
}

// Surface separation dd and approach speed ww of the point (x, v, radius rp) and the human sphere hs = (c, r):
//   e = c - x;  l = sqrt(e.e);  dd = l - rp - r;  ww = (e.v) / l, or |v| where l == 0
// each sum left to right.
__device__ __forceinline__ void separation_pair(const double *x, const double *v, const double rp, const double *hs,
                                                double &dd, double &ww) {
  const double e[3] = {hs[0] - x[0], hs[1] - x[1], hs[2] - x[2]};
  const double l = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
  dd = l - rp - hs[3];
  ww = l == 0.0 ? sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) : (e[0] * v[0] + e[1] * v[1] + e[2] * v[2]) / l;
}

__device__ __forceinline__ double clamp01(const double x) { return x < 0.0 ? 0.0 : (x > 1.0 ? 1.0 : x); }

// Surface separation dd and approach speed ww of the robot capsule (segment xa -> xb, endpoint velocities va, vb,
// radius rp) and the human capsule hc = (c0, c1, r_h): the closest pair (t, tau) of the two segments (Ericson, Real-Time
// Collision Detection 5.1.9), then separation_pair of p(t) = xa + t (xb - xa), v(t) = va + t (vb - va) and the sphere
// (c0 + tau (c1 - c0), r_h).  Parallel segments (denom <= TBD_CAPSULE_PARALLEL a e) whose projections overlap on
// [t_lo, t_hi] have a segment of closest pairs: both ends are evaluated, dd is the smaller and ww the larger (Danskin).
// Operation order in include/toppra_b200_dyn.h.
__device__ __forceinline__ void capsule_pair(const double *xa, const double *va, const double *xb, const double *vb,
                                             const double rp, const double *hc, double &dd, double &ww) {
  double d1[3], d2[3], r0[3];
  for (int j = 0; j < 3; ++j) { d1[j] = xb[j] - xa[j]; d2[j] = hc[3 + j] - hc[j]; r0[j] = xa[j] - hc[j]; }
  const double a = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2];
  const double e = d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2];
  const double f = d2[0] * r0[0] + d2[1] * r0[1] + d2[2] * r0[2];
  double t = 0.0, tau = 0.0, t2 = 0.0, tau2 = 0.0;
  bool two = false;
  if (a == 0.0) {
    if (e != 0.0) tau = clamp01(f / e);
  } else {
    const double c = d1[0] * r0[0] + d1[1] * r0[1] + d1[2] * r0[2];
    if (e == 0.0) {
      t = clamp01(-c / a);
    } else {
      const double b = d1[0] * d2[0] + d1[1] * d2[1] + d1[2] * d2[2];
      const double denom = a * e - b * b;
      bool general = true;
      if (denom <= TBD_CAPSULE_PARALLEL * a * e) {
        const double t0 = -c / a, t1 = (b - c) / a;
        const double lo = fmax(fmin(t0, t1), 0.0), hi = fmin(fmax(t0, t1), 1.0);
        if (lo <= hi) {
          t = lo;
          tau = clamp01((b * lo + f) / e);
          t2 = hi;
          tau2 = clamp01((b * hi + f) / e);
          two = true;
          general = false;
        }
      } else {
        t = clamp01((b * f - c * e) / denom);
      }
      if (general) {
        tau = (b * t + f) / e;
        if (tau < 0.0) {
          tau = 0.0;
          t = clamp01(-c / a);
        } else if (tau > 1.0) {
          tau = 1.0;
          t = clamp01((b - c) / a);
        }
      }
    }
  }
  double p[3], v[3], hs[4];
  for (int j = 0; j < 3; ++j) {
    p[j] = xa[j] + t * d1[j];
    v[j] = va[j] + t * (vb[j] - va[j]);
    hs[j] = hc[j] + tau * d2[j];
  }
  hs[3] = hc[6];
  separation_pair(p, v, rp, hs, dd, ww);
  if (two) {
    for (int j = 0; j < 3; ++j) {
      p[j] = xa[j] + t2 * d1[j];
      v[j] = va[j] + t2 * (vb[j] - va[j]);
      hs[j] = hc[j] + tau2 * d2[j];
    }
    double d2_, w2_;
    separation_pair(p, v, rp, hs, d2_, w2_);
    if (d2_ < dd) dd = d2_;
    if (w2_ > ww) ww = w2_;
  }
}

// The human set of point pt: [H][HD] doubles of set pt / points_per_path (set 0 when points_per_path is 0); HD = 4 for
// spheres, TBD_HUMAN_CAPSULE_DOUBLES for capsules.
template <int HD = 4>
__device__ __forceinline__ const double *human_set(const double *humans, const int H, const int points_per_path,
                                                   const long pt) {
  const long set = points_per_path > 0 ? pt / points_per_path : 0;
  return humans + (size_t)set * H * HD;
}

// The row of SeparationMonitoringConstraint at point pt from the pairs pair(i, h, dd, ww), i < n, h < H, i-major: per
// pair
//   D = dd - C - vhTr;  num = twoa * D;  vmax = D <= 0 ? 0 : num / (sqrt(kk + num) + k)
// with twoa = 2 a_s, vhTr = v_h T_r, k = a_s T_r + v_h, kk = k k; among the pairs with ww > 0 the first one minimising
// vmax^2 / ww^2 by cross-multiplication (v2 * bw2 < bv2 * w2, v2 = vmax vmax, w2 = ww ww) gives b = bw2, c = 0 - bv2;
// no such pair gives b = 0, c = -1; a NaN dd or ww of any pair gives b = c = NaN.
template <class Pair>
__device__ __forceinline__ void separation_row(const Pair &pair, const int n, const int H, const double clearance,
                                               const double vhTr, const double twoa, const double k, const double kk,
                                               const long pt, double *__restrict__ b, double *__restrict__ c) {
  double bw2 = 0.0, bv2 = 0.0;
  bool found = false, bad = false;
  for (int i = 0; i < n; ++i)
    for (int h = 0; h < H; ++h) {
      double dd, ww;
      pair(i, h, dd, ww);
      const double D = dd - clearance - vhTr;
      const double num = twoa * D;
      const double vmax = D <= 0.0 ? 0.0 : num / (sqrt(kk + num) + k);
      bad = bad || isnan(ww) || isnan(vmax);
      if (ww > 0.0) {
        const double w2 = ww * ww, v2 = vmax * vmax;
        if (!found || v2 * bw2 < bv2 * w2) { bw2 = w2; bv2 = v2; found = true; }
      }
    }
  if (bad) {
    b[pt] = nan("");
    c[pt] = nan("");
  } else {
    b[pt] = found ? bw2 : 0.0;
    c[pt] = found ? 0.0 - bv2 : -1.0;
  }
}

__global__ void __launch_bounds__(THREADS)
separation_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynPoints pts, const int nv, const int H,
                  const int points_per_path, const int M, const double *__restrict__ q, const double *__restrict__ qd,
                  const double *__restrict__ humans, double *__restrict__ dist, double *__restrict__ speed) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[TBD_MAX_POINTS][3], v[TBD_MAX_POINTS][3];
  point_states(m, pts, q + o, qd + o, x, v);
  const double *hs = human_set(humans, H, points_per_path, pt);
  for (int i = 0; i < pts.n; ++i)
    for (int h = 0; h < H; ++h) {
      double dd, ww;
      separation_pair(x[i], v[i], pts.r[i], hs + 4 * h, dd, ww);
      const size_t r = ((size_t)pt * pts.n + i) * H + h;
      dist[r] = dd;
      speed[r] = ww;
    }
}

// The row of SeparationMonitoringConstraint at (q, qs = q'), from the pairs of separation_kernel at qd = qs
// (separation_row).
__global__ void __launch_bounds__(THREADS)
separation_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynPoints pts, const int nv,
                        const int H, const int points_per_path, const double clearance, const double vhTr,
                        const double twoa, const double k, const double kk, const int M, const double *__restrict__ q,
                        const double *__restrict__ qs, const double *__restrict__ humans, double *__restrict__ b,
                        double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[TBD_MAX_POINTS][3], v[TBD_MAX_POINTS][3];
  point_states(m, pts, q + o, qs + o, x, v);
  const double *hs = human_set(humans, H, points_per_path, pt);
  separation_row([&](const int i, const int h, double &dd, double &ww) {
    separation_pair(x[i], v[i], pts.r[i], hs + 4 * h, dd, ww);
  }, pts.n, H, clearance, vhTr, twoa, k, kk, pt, b, c);
}

// d, w of P robot capsules (the 2 P endpoints of caps) and H human capsules at (q, qd), capsule-major, then h.
__global__ void __launch_bounds__(THREADS)
capsule_separation_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynCapsules caps, const int nv,
                          const int H, const int points_per_path, const int M, const double *__restrict__ q,
                          const double *__restrict__ qd, const double *__restrict__ humans, double *__restrict__ dist,
                          double *__restrict__ speed) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[2 * TBD_MAX_POINTS][3], v[2 * TBD_MAX_POINTS][3];
  point_states(m, caps, q + o, qd + o, x, v);
  const double *hc = human_set<TBD_HUMAN_CAPSULE_DOUBLES>(humans, H, points_per_path, pt);
  const int P = caps.n / 2;
  for (int i = 0; i < P; ++i)
    for (int h = 0; h < H; ++h) {
      double dd, ww;
      capsule_pair(x[2 * i], v[2 * i], x[2 * i + 1], v[2 * i + 1], caps.r[2 * i], hc + TBD_HUMAN_CAPSULE_DOUBLES * h,
                   dd, ww);
      const size_t r = ((size_t)pt * P + i) * H + h;
      dist[r] = dd;
      speed[r] = ww;
    }
}

// The row of SeparationMonitoringConstraint at (q, qs = q') from the pairs of capsule_separation_kernel at qd = qs.
__global__ void __launch_bounds__(THREADS)
capsule_separation_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynCapsules caps,
                                const int nv, const int H, const int points_per_path, const double clearance,
                                const double vhTr, const double twoa, const double k, const double kk, const int M,
                                const double *__restrict__ q, const double *__restrict__ qs,
                                const double *__restrict__ humans, double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double x[2 * TBD_MAX_POINTS][3], v[2 * TBD_MAX_POINTS][3];
  point_states(m, caps, q + o, qs + o, x, v);
  const double *hc = human_set<TBD_HUMAN_CAPSULE_DOUBLES>(humans, H, points_per_path, pt);
  separation_row([&](const int i, const int h, double &dd, double &ww) {
    capsule_pair(x[2 * i], v[2 * i], x[2 * i + 1], v[2 * i + 1], caps.r[2 * i], hc + TBD_HUMAN_CAPSULE_DOUBLES * h,
                 dd, ww);
  }, caps.n / 2, H, clearance, vhTr, twoa, k, kk, pt, b, c);
}

// Geared drives (include/toppra_b200_dyn.h), passed by value next to the model: the transmission T and T^-T (row-major,
// entries [0, nv) of each), the rotor inertias, the motor friction and, for tbd_drive_speed_terms, the speed limits.
struct DynDrive {
  double T[NB][NB], Tit[NB][NB], Ir[NB], f[NB], omega[NB];
};

// tm = T^-T tau + I_r o (T qdd): per motor i, both sums left to right, then (T^-T tau)_i + I_r,i (T qdd)_i.
__device__ __forceinline__ void motor_torque(const DynDrive &d, const int nv, const double *tau, const double *qdd,
                                             double *tm) {
  for (int i = 0; i < nv; ++i) {
    double s = d.Tit[i][0] * tau[0], t = d.T[i][0] * qdd[0];
    for (int j = 1; j < nv; ++j) { s = s + d.Tit[i][j] * tau[j]; t = t + d.T[i][j] * qdd[j]; }
    tm[i] = s + d.Ir[i] * t;
  }
}

// (T x)_i, summed left to right.
__device__ __forceinline__ double motor_row(const DynDrive &d, const int nv, const int i, const double *x) {
  double v = d.T[i][0] * x[0];
  for (int j = 1; j < nv; ++j) v = v + d.T[i][j] * x[j];
  return v;
}

__global__ void __launch_bounds__(THREADS)
drive_torque_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynDrive d, const int nv, const int M,
                    const double *__restrict__ q, const double *__restrict__ qd, const double *__restrict__ qdd,
                    double *__restrict__ tau_m) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], t[NB];
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, qd + o, qdd + o, st, f, t);
  motor_torque(d, nv, t, qdd + o, tau_m + o);
}

// c = w(q, 0, 0), a = w(q, 0, q') - c, b = w(q, q', q'') - c, c += f o sign(T q'): the terms of MotorTorqueConstraint;
// the joint transforms (and their sincos) are computed once per point and shared by the three passes.
__global__ void __launch_bounds__(THREADS)
drive_torque_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynDrive d, const int nv,
                          const int M, const double *__restrict__ q, const double *__restrict__ qs,
                          const double *__restrict__ qss, double *__restrict__ a, double *__restrict__ b,
                          double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], zero[NB], t[NB], wc[NB], w[NB];
  for (int k = 0; k < nv; ++k) zero[k] = 0.0;
  joint_transforms(m, nv, q + o, X);
  rnea_pass(m, nv, X, zero, zero, st, f, t);
  motor_torque(d, nv, t, zero, wc);
  rnea_pass(m, nv, X, zero, qs + o, st, f, t);
  motor_torque(d, nv, t, qs + o, w);
  for (int k = 0; k < nv; ++k) a[o + k] = w[k] - wc[k];
  rnea_pass(m, nv, X, qs + o, qss + o, st, f, t);
  motor_torque(d, nv, t, qss + o, w);
  for (int k = 0; k < nv; ++k) b[o + k] = w[k] - wc[k];
  for (int k = 0; k < nv; ++k) {
    const double x = motor_row(d, nv, k, qs + o);
    const double sgn = (double)((0.0 < x) - (x < 0.0));   // torch.sign: 0 at +-0 and NaN
    c[o + k] = wc[k] + sgn * d.f[k];
  }
}

// b = max_i ((T q')_i / omega_i)^2, the maximum propagating NaN: the motor-speed row of MotorSpeedConstraint.
__global__ void __launch_bounds__(THREADS)
drive_speed_terms_kernel(const __grid_constant__ DynDrive d, const int nv, const int M, const double *__restrict__ qs,
                         double *__restrict__ b) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const double *x = qs + (size_t)pt * nv;
  double mx = 0.0;
  for (int i = 0; i < nv; ++i) {
    const double r = motor_row(d, nv, i, x) / d.omega[i];
    const double r2 = r * r;
    if (!isnan(mx) && (i == 0 || r2 > mx || isnan(r2))) mx = r2;
  }
  b[pt] = mx;
}

// The axes A of a joint wrench, out = A^T x: R_f for a TBD_LOCAL frame f on body k; for TBD_LOCAL_WORLD_ALIGNED the
// transpose of body k's world orientation Rw = R_c0 R_c1 ... R_k, the rotations of X along f's chain from the root.
__device__ __forceinline__ void joint_wrench_axes(const DynFrame &fr, const double (*X)[12], double *A) {
  if (fr.ref == TBD_LOCAL) {
    for (int j = 0; j < 9; ++j) A[j] = fr.R[j];
    return;
  }
  double Rw[9], Rn[9];
  for (int j = 0; j < 9; ++j) Rw[j] = X[fr.chain[0]][j];
  for (int i = 1; i < fr.n; ++i) {
    mul33(Rw, X[fr.chain[i]], Rn);
    for (int j = 0; j < 9; ++j) Rw[j] = Rn[j];
  }
  const double Rt[9] = {Rw[0], Rw[3], Rw[6], Rw[1], Rw[4], Rw[7], Rw[2], Rw[5], Rw[8]};
  for (int j = 0; j < 9; ++j) A[j] = Rt[j];
}

// The wrench [f; n] the parent side of joint k exerts on k's subtree, at the origin p_f of frame fr (on body k), from
// the forces of a finished rnea_pass: f[k] = [n_k; f_k] about body k's origin in body-k coordinates, the momentum rate
// of the subtree minus its weight (gravity enters as base acceleration -g).
//   out = [A^T f_k; A^T (n_k - p_f x f_k)]   (A: joint_wrench_axes)
__device__ __forceinline__ void joint_wrench(const DynFrame &fr, const double *A, const double (*f)[6], double *out) {
  const double *fk = f[fr.chain[fr.n - 1]];
  double u[3], t[3];
  cross3(fr.p, fk + 3, u);
  for (int j = 0; j < 3; ++j) t[j] = fk[j] - u[j];
  mul3t(A, fk + 3, out);
  mul3t(A, t, out + 3);
}

__global__ void __launch_bounds__(THREADS)
joint_wrench_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame fr, const int nv, const int M,
                    const double *__restrict__ q, const double *__restrict__ qd, const double *__restrict__ qdd,
                    double *__restrict__ w) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], t[NB], A[9], y[6];
  joint_transforms(m, nv, q + o, X);
  joint_wrench_axes(fr, X, A);
  rnea_pass(m, nv, X, qd + o, qdd + o, st, f, t);
  joint_wrench(fr, A, f, y);
  for (int j = 0; j < 6; ++j) w[(size_t)pt * 6 + j] = y[j];
}

// c = w(q, 0, 0), a = w(q, 0, q') - c, b = w(q, q', q'') - c: the terms of JointWrenchConstraint, the components of bit
// mask `components` in increasing order (k = popcount columns); the joint transforms and the axes are computed once per
// point and shared by the three passes.
__global__ void __launch_bounds__(THREADS)
joint_wrench_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynFrame fr, const int nv,
                          const int components, const int k, const int M, const double *__restrict__ q,
                          const double *__restrict__ qs, const double *__restrict__ qss, double *__restrict__ a,
                          double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double X[NB][12], st[NB][12], f[NB][6], zero[NB], t[NB], A[9], y0[6], y[6];
  for (int j = 0; j < nv; ++j) zero[j] = 0.0;
  joint_transforms(m, nv, q + o, X);
  joint_wrench_axes(fr, X, A);
  rnea_pass(m, nv, X, zero, zero, st, f, t);
  joint_wrench(fr, A, f, y0);
  double *ao = a + (size_t)pt * k, *bo = b + (size_t)pt * k, *co = c + (size_t)pt * k;
  for (int j = 0, i = 0; j < 6; ++j)
    if ((components >> j) & 1) co[i++] = y0[j];
  rnea_pass(m, nv, X, zero, qs + o, st, f, t);
  joint_wrench(fr, A, f, y);
  for (int j = 0, i = 0; j < 6; ++j)
    if ((components >> j) & 1) ao[i++] = y[j] - y0[j];
  rnea_pass(m, nv, X, qs + o, qss + o, st, f, t);
  joint_wrench(fr, A, f, y);
  for (int j = 0, i = 0; j < 6; ++j)
    if ((components >> j) & 1) bo[i++] = y[j] - y0[j];
}

// The kinetic energy T and the linear momentum p (base axes) of the whole tree at (q, qd): one walk of bodies [0, nv)
// with each body's world rotation Rw, angular velocity w and origin velocity vo in per-thread local arrays (the per-body
// operations of point_states), and for each body, in body order, with d = Rw c:
//   vc = vo + w x d;  wb = Rw^T w;  e += m ((vc0 vc0 + vc1 vc1) + vc2 vc2) + ((wb0 Iwb0 + wb1 Iwb1) + wb2 Iwb2);
//   p += m vc;        (Iwb = Ic wb)
// and T = 0.5 e.  No world origin is kept: neither sum depends on where a body is.
__device__ __forceinline__ void energy_momentum(const DynModel &m, const int nv, const double *__restrict__ q,
                                                const double *__restrict__ qd, double &T, double *p) {
  double Rw[NB][9], w[NB][3], vo[NB][3];
  double e = 0.0;
  for (int j = 0; j < 3; ++j) p[j] = 0.0;
  for (int k = 0; k < nv; ++k) {
    const double *bd = m.body[k];
    const int par = (int)bd[0];
    double Rp[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    double wp[3] = {0.0, 0.0, 0.0}, vp[3] = {0.0, 0.0, 0.0};
    if (par >= 0) {
      for (int j = 0; j < 9; ++j) Rp[j] = Rw[par][j];
      for (int j = 0; j < 3; ++j) { wp[j] = w[par][j]; vp[j] = vo[par][j]; }
    }
    double R[9], po[3], d[3], t[3];
    const double qk = q[k];
    TB_BODY_TRANSFORM(bd, qk, R, po);
    mul3(Rp, po, d);                    // origin of body k relative to its parent's, world coordinates
    cross3(wp, d, t);
    for (int j = 0; j < 3; ++j) vo[k][j] = vp[j] + t[j];
    mul33(Rp, R, Rw[k]);
    double s[3];
    mul3(Rw[k], bd + 2, s);             // joint axis, world coordinates
    const double qdk = qd[k];
    if (bd[1] == TBD_REVOLUTE) {
      for (int j = 0; j < 3; ++j) { w[k][j] = wp[j] + s[j] * qdk; }
    } else {
      for (int j = 0; j < 3; ++j) { w[k][j] = wp[j]; vo[k][j] = vo[k][j] + s[j] * qdk; }
    }
    const double mass = bd[17], *c = bd + 18, *Ic = bd + 21;
    double vc[3], wb[3], Iwb[3];
    mul3(Rw[k], c, d);                  // centre of mass relative to the body origin, world coordinates
    cross3(w[k], d, t);
    for (int j = 0; j < 3; ++j) vc[j] = vo[k][j] + t[j];
    mul3t(Rw[k], w[k], wb);             // angular velocity, body coordinates
    mul_inertia(Ic, wb, Iwb);
    const double vv = vc[0] * vc[0] + vc[1] * vc[1] + vc[2] * vc[2];
    const double ww = wb[0] * Iwb[0] + wb[1] * Iwb[1] + wb[2] * Iwb[2];
    e = e + (mass * vv + ww);
    for (int j = 0; j < 3; ++j) p[j] = p[j] + mass * vc[j];
  }
  T = 0.5 * e;
}

__global__ void __launch_bounds__(THREADS)
energy_momentum_kernel(const __grid_constant__ DynModel m, const int nv, const int M, const double *__restrict__ q,
                       const double *__restrict__ qd, double *__restrict__ out) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double T, p[3];
  energy_momentum(m, nv, q + o, qd + o, T, p);
  double *y = out + (size_t)pt * 4;
  y[0] = T;
  for (int j = 0; j < 3; ++j) y[1 + j] = p[j];
}

// b = T(q, q') (which = TBD_KINETIC_ENERGY) or (px px + py py) + pz pz (TBD_MOMENTUM): the row of KineticEnergyConstraint
// or MomentumConstraint.
__global__ void __launch_bounds__(THREADS)
energy_momentum_terms_kernel(const __grid_constant__ DynModel m, const int nv, const int which, const int M,
                             const double *__restrict__ q, const double *__restrict__ qs, double *__restrict__ b) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nv;
  double T, p[3];
  energy_momentum(m, nv, q + o, qs + o, T, p);
  b[pt] = which == TBD_KINETIC_ENERGY ? T : p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
}

// A linear joint coupling (include/toppra_b200_dyn.h), passed by value next to the model: body joint positions
// q_b = E q + o, E (nv x nq) in entries [0, nv) x [0, nq) of E.
struct DynCoupling {
  double E[NB][NB], o[NB];
};

// xb = E x, plus o where `pos` (positions): per body k the nonzero terms E[k][j] x[j] in ascending j, starting from the
// first term, then + o[k] where o[k] != 0.  __dmul_rn / __dadd_rn keep that order whatever the contraction flags.
__device__ __forceinline__ void coupling_expand(const DynCoupling &cp, const int nv, const int nq,
                                                const double *__restrict__ x, const bool pos, double *xb) {
  for (int k = 0; k < nv; ++k) {
    double s = 0.0;
    bool first = true;
    for (int j = 0; j < nq; ++j) {
      const double e = cp.E[k][j];
      if (e == 0.0) continue;
      const double t = __dmul_rn(e, x[j]);
      s = first ? t : __dadd_rn(s, t);
      first = false;
    }
    if (pos && cp.o[k] != 0.0) s = __dadd_rn(s, cp.o[k]);
    xb[k] = s;
  }
}

// y = E^T t: per DOF j the nonzero terms E[k][j] t[k] in ascending k, starting from the first term (every column of E
// has one: load_coupling).
__device__ __forceinline__ void coupling_reduce(const DynCoupling &cp, const int nv, const int nq, const double *t,
                                                double *y) {
  for (int j = 0; j < nq; ++j) {
    double s = 0.0;
    bool first = true;
    for (int k = 0; k < nv; ++k) {
      const double e = cp.E[k][j];
      if (e == 0.0) continue;
      const double u = __dmul_rn(e, t[k]);
      s = first ? u : __dadd_rn(s, u);
      first = false;
    }
    y[j] = s;
  }
}

// tau_q = E^T ID(E q + o, E qd, E qdd): joint_transforms and rnea_pass of rnea_kernel on the expanded state.
__global__ void __launch_bounds__(THREADS)
coupled_rnea_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynCoupling cp, const int nv,
                    const int nq, const int M, const double *__restrict__ q, const double *__restrict__ qd,
                    const double *__restrict__ qdd, double *__restrict__ tau) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nq;
  double X[NB][12], st[NB][12], f[NB][6], qb[NB], qdb[NB], qddb[NB], t[NB];
  coupling_expand(cp, nv, nq, q + o, true, qb);
  coupling_expand(cp, nv, nq, qd + o, false, qdb);
  coupling_expand(cp, nv, nq, qdd + o, false, qddb);
  joint_transforms(m, nv, qb, X);
  rnea_pass(m, nv, X, qdb, qddb, st, f, t);
  coupling_reduce(cp, nv, nq, t, tau + o);
}

// The terms of torque_terms_kernel on the expanded state, each subtracted in body space and then reduced by E^T;
// c += sign(q') friction on the nq DOFs.
__global__ void __launch_bounds__(THREADS)
coupled_torque_terms_kernel(const __grid_constant__ DynModel m, const __grid_constant__ DynCoupling cp, const int nv,
                            const int nq, const int M, const double *__restrict__ q, const double *__restrict__ qs,
                            const double *__restrict__ qss, const double *__restrict__ friction,
                            double *__restrict__ a, double *__restrict__ b, double *__restrict__ c) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nq;
  double X[NB][12], st[NB][12], f[NB][6], zero[NB], qb[NB], qsb[NB], qssb[NB], tc[NB], t[NB];
  for (int k = 0; k < nv; ++k) zero[k] = 0.0;
  coupling_expand(cp, nv, nq, q + o, true, qb);
  coupling_expand(cp, nv, nq, qs + o, false, qsb);
  coupling_expand(cp, nv, nq, qss + o, false, qssb);
  joint_transforms(m, nv, qb, X);
  rnea_pass(m, nv, X, zero, zero, st, f, tc);
  rnea_pass(m, nv, X, zero, qsb, st, f, t);
  for (int k = 0; k < nv; ++k) t[k] = t[k] - tc[k];
  coupling_reduce(cp, nv, nq, t, a + o);
  rnea_pass(m, nv, X, qsb, qssb, st, f, t);
  for (int k = 0; k < nv; ++k) t[k] = t[k] - tc[k];
  coupling_reduce(cp, nv, nq, t, b + o);
  coupling_reduce(cp, nv, nq, tc, t);
  for (int j = 0; j < nq; ++j) {
    double cj = t[j];
    if (friction) {
      const double x = qs[o + j];
      const double sgn = (double)((0.0 < x) - (x < 0.0));   // torch.sign: 0 at +-0 and NaN
      cj = __dadd_rn(cj, __dmul_rn(sgn, friction[j]));
    }
    c[o + j] = cj;
  }
}

// q_b = E q + o and, where given, the rates E qd, E qdd.
__global__ void __launch_bounds__(THREADS)
coupling_expand_kernel(const __grid_constant__ DynCoupling cp, const int nv, const int nq, const int M,
                       const double *__restrict__ q, const double *__restrict__ qd, const double *__restrict__ qdd,
                       double *__restrict__ q_out, double *__restrict__ qd_out, double *__restrict__ qdd_out) {
  const long pt = (long)blockIdx.x * THREADS + threadIdx.x;
  if (pt >= M) return;
  const size_t o = (size_t)pt * nq, ob = (size_t)pt * nv;
  coupling_expand(cp, nv, nq, q + o, true, q_out + ob);
  if (qd) coupling_expand(cp, nv, nq, qd + o, false, qd_out + ob);
  if (qdd) coupling_expand(cp, nv, nq, qdd + o, false, qdd_out + ob);
}

// The point count and the number of bodies (or motors): 0, or the TB_ERR_* code (message set).
int check_sizes(const int nv, const int M, const char *what) {
  if (M <= 0) { set_error("%s: M=%d must be positive", what, M); return TB_ERR_ARG; }
  if (nv < 1 || nv > NB) { set_error("%s: nv=%d outside 1..%d", what, nv, NB); return TB_ERR_UNSUPPORTED; }
  return 0;
}

// Validates the packed model and copies it into the by-value launch parameter: 0, or the TB_ERR_* code (message set).
int load_model(const double *host, const int nv, const int M, DynModel *m, const char *what) {
  if (const int rc = check_sizes(nv, M, what)) return rc;
  for (int i = 0; i < 3; ++i) m->g[i] = host[i];
  for (int k = 0; k < NB; ++k)
    for (int j = 0; j < TBD_BODY_DOUBLES; ++j) m->body[k][j] = k < nv ? host[3 + TBD_BODY_DOUBLES * k + j] : 0.0;
  for (int k = 0; k < nv; ++k) {
    const double *bd = m->body[k];
    if (!(bd[0] >= -1.0 && bd[0] < (double)k && bd[0] == std::floor(bd[0]))) {
      set_error("%s: body %d: parent %g must be an integer in [-1, %d)", what, k, bd[0], k);
      return TB_ERR_ARG;
    }
    if (bd[1] != TBD_REVOLUTE && bd[1] != TBD_PRISMATIC) {
      set_error("%s: body %d: unknown joint type %g", what, k, bd[1]);
      return TB_ERR_ARG;
    }
    if (!std::isfinite(bd[17]) || bd[17] < 0.0) {
      set_error("%s: body %d: mass %g must be finite and non-negative", what, k, bd[17]);
      return TB_ERR_ARG;
    }
    if (bd[2] == 0.0 && bd[3] == 0.0 && bd[4] == 0.0) {
      set_error("%s: body %d: zero joint axis", what, k);
      return TB_ERR_ARG;
    }
  }
  return 0;
}

// Validates the packed frame (include/toppra_b200_dyn.h) of a model already loaded by load_model and copies it, the
// root-to-body chain and S (nullable) into the by-value launch parameter: 0, or the TB_ERR_* code (message set).  `ref`
// replaces the frame's reference-frame field (-1: as given), for entries whose result is always in one frame's axes.
int load_frame(const double *host, const DynModel &m, const int nv, const double *S, const int ref, DynFrame *f,
               const char *what) {
  const double body = host[0];
  if (!(body >= -1.0 && body < (double)nv && body == std::floor(body))) {
    set_error("%s: frame body %g must be an integer in [-1, %d)", what, body, nv);
    return TB_ERR_ARG;
  }
  const double r = ref >= 0 ? (double)ref : host[13];
  if (r != TBD_WORLD && r != TBD_LOCAL && r != TBD_LOCAL_WORLD_ALIGNED) {
    set_error("%s: unknown reference frame %g", what, r);
    return TB_ERR_ARG;
  }
  for (int j = 0; j < 12; ++j)
    if (!std::isfinite(host[1 + j])) { set_error("%s: frame placement is not finite", what); return TB_ERR_ARG; }
  for (int j = 0; j < 9; ++j) f->R[j] = host[1 + j];
  for (int j = 0; j < 3; ++j) f->p[j] = host[10 + j];
  for (int j = 0; j < 36; ++j) {
    f->S[j] = S ? S[j] : 0.0;
    if (!std::isfinite(f->S[j])) { set_error("%s: S is not finite", what); return TB_ERR_ARG; }
  }
  f->ref = (int)r;
  int n = 0;
  for (int k = (int)body; k >= 0; k = (int)m.body[k][0]) ++n;   // parents are validated: parent[k] < k
  f->n = n;
  for (int k = (int)body, i = n - 1; k >= 0; k = (int)m.body[k][0], --i) f->chain[i] = k;
  for (int i = n; i < NB; ++i) f->chain[i] = 0;
  return 0;
}

// Frame accelerations and the inverse inertia are those of the frame origin: a quantity "at the world origin" is no
// limit a user means, so TBD_WORLD is TB_ERR_UNSUPPORTED.
int refuse_world(const DynFrame &f, const char *what, const char *quantity) {
  if (f.ref != TBD_WORLD) return 0;
  set_error("%s: the world reference frame is not supported%s (use local or local_world_aligned)", what, quantity);
  return TB_ERR_UNSUPPORTED;
}

// The packed object (TBD_OBJECT_DOUBLES): finite, with a positive mass.
int load_object(const double *host, DynObject *o, const char *what) {
  for (int j = 0; j < TBD_OBJECT_DOUBLES; ++j)
    if (!std::isfinite(host[j])) { set_error("%s: object parameters are not finite", what); return TB_ERR_ARG; }
  if (!(host[0] > 0.0)) { set_error("%s: object mass %g must be positive", what, host[0]); return TB_ERR_ARG; }
  o->mass = host[0];
  for (int j = 0; j < 3; ++j) o->r[j] = host[1 + j];
  for (int j = 0; j < 6; ++j) o->Ic[j] = host[4 + j];
  return 0;
}

// The packed base (TBD_BASE_DOUBLES): finite, with a non-negative mass.
int load_base(const double *host, DynBase *base, const char *what) {
  for (int j = 0; j < TBD_BASE_DOUBLES; ++j)
    if (!std::isfinite(host[j])) { set_error("%s: base parameters are not finite", what); return TB_ERR_ARG; }
  if (!(host[0] >= 0.0)) { set_error("%s: base mass %g must be non-negative", what, host[0]); return TB_ERR_ARG; }
  base->mass = host[0];
  for (int j = 0; j < 3; ++j) base->c[j] = host[1 + j];
  return 0;
}

// The support wrench is that of a support frame on the base, in its own axes.
int load_support(const double *host, const DynModel &m, const int nv, DynFrame *s, const char *what) {
  if (const int rc = load_frame(host, m, nv, nullptr, TBD_LOCAL, s, what)) return rc;
  if (host[0] != -1.0) {
    set_error("%s: the support must be on the base (frame body %g, expected -1)", what, host[0]);
    return TB_ERR_ARG;
  }
  return 0;
}

// The wrench across a joint is that of the moving joint of the frame's body, at the frame origin: TBD_WORLD is
// TB_ERR_UNSUPPORTED (refuse_world), and a frame on the base has no joint (TB_ERR_ARG).
int load_joint_frame(const double *host, const DynModel &m, const int nv, DynFrame *f, const char *what) {
  if (const int rc = load_frame(host, m, nv, nullptr, -1, f, what)) return rc;
  if (const int rc = refuse_world(*f, what, " for joint wrenches")) return rc;
  if (f->n == 0) {
    set_error("%s: the frame is on the base (body -1), which has no joint; the base's load is the support wrench "
              "(SupportStabilityConstraint)", what);
    return TB_ERR_ARG;
  }
  return 0;
}

// The packed points (P x TBD_POINT_DOUBLES: a packed frame and a radius), the human-sphere sets and their assignment to
// points, for a model already loaded by load_model: 0, or the TB_ERR_* code (message set).  The frames' reference-frame
// field is ignored.
// The counts and the assignment of human sets shared by both separation forms: robot and human name the two sides in
// the messages ("points" and "sphere", or "capsules" and "capsule").
int check_separation_sets(const int P, const int H, const int NH, const int points_per_path, const int M,
                          const char *robot, const char *human, const char *what) {
  if (P < 1 || P > TBD_MAX_POINTS) { set_error("%s: P=%d %s outside 1..%d", what, P, robot, TBD_MAX_POINTS); return TB_ERR_UNSUPPORTED; }
  if (H < 1 || H > TBD_MAX_HUMANS) { set_error("%s: H=%d human %ss outside 1..%d", what, H, human, TBD_MAX_HUMANS); return TB_ERR_UNSUPPORTED; }
  if (NH < 1) { set_error("%s: NH=%d human-%s sets must be positive", what, NH, human); return TB_ERR_ARG; }
  if (points_per_path < 0 || (points_per_path > 0 && (M - 1) / points_per_path >= NH)) {
    set_error("%s: points_per_path=%d with M=%d reads past the NH=%d human-%s sets", what, points_per_path, M, NH, human);
    return TB_ERR_ARG;
  }
  return 0;
}

// An empty point set with n points.
template <int NP>
void clear_points(DynPointSet<NP> *pts, const int n) {
  pts->n = n;
  pts->top = 0;
  for (int i = 0; i < NP; ++i) {
    pts->body[i] = -1;
    pts->r[i] = 0.0;
    for (int j = 0; j < 3; ++j) pts->p[i][j] = 0.0;
  }
}

// Point i of the set: the origin of the packed frame fh (checked by load_frame), radius r.
template <int NP>
int put_point(const double *fh, const double r, const DynModel &m, const int nv, const int i, DynPointSet<NP> *pts,
              const char *what) {
  DynFrame f;
  if (const int rc = load_frame(fh, m, nv, nullptr, TBD_LOCAL_WORLD_ALIGNED, &f, what)) return rc;
  pts->body[i] = (int)fh[0];
  pts->r[i] = r;
  for (int j = 0; j < 3; ++j) pts->p[i][j] = f.p[j];
  if (pts->body[i] + 1 > pts->top) pts->top = pts->body[i] + 1;
  return 0;
}

int load_points(const double *host, const int P, const int H, const int NH, const int points_per_path, const int M,
                const DynModel &m, const int nv, DynPoints *pts, const char *what) {
  if (const int rc = check_separation_sets(P, H, NH, points_per_path, M, "points", "sphere", what)) return rc;
  clear_points(pts, P);
  for (int i = 0; i < P; ++i) {
    const double *ph = host + (size_t)TBD_POINT_DOUBLES * i;
    const double r = ph[TBD_FRAME_DOUBLES];
    if (const int rc = put_point(ph, r, m, nv, i, pts, what)) return rc;
    if (!std::isfinite(r) || r < 0.0) { set_error("%s: point %d: radius %g must be finite and >= 0", what, i, r); return TB_ERR_ARG; }
  }
  return 0;
}

// The packed capsules (P x TBD_CAPSULE_DOUBLES: packed frames a and b and a radius) as the 2 P endpoints of caps, the
// human-capsule sets and their assignment to points; the checks of load_points, frame a, frame b, then the radius.
int load_capsules(const double *host, const int P, const int H, const int NH, const int points_per_path, const int M,
                  const DynModel &m, const int nv, DynCapsules *caps, const char *what) {
  if (const int rc = check_separation_sets(P, H, NH, points_per_path, M, "capsules", "capsule", what)) return rc;
  clear_points(caps, 2 * P);
  for (int i = 0; i < P; ++i) {
    const double *ch = host + (size_t)TBD_CAPSULE_DOUBLES * i;
    const double r = ch[2 * TBD_FRAME_DOUBLES];
    if (const int rc = put_point(ch, r, m, nv, 2 * i, caps, what)) return rc;
    if (const int rc = put_point(ch + TBD_FRAME_DOUBLES, r, m, nv, 2 * i + 1, caps, what)) return rc;
    if (!std::isfinite(r) || r < 0.0) { set_error("%s: capsule %d: radius %g must be finite and >= 0", what, i, r); return TB_ERR_ARG; }
  }
  return 0;
}

// The four scalars of the limit (include/toppra_b200_dyn.h, tbd_separation_terms) and the host values the terms
// kernels take: 0, or TB_ERR_ARG (message set).
int load_limit(const double reaction_time, const double stopping_deceleration, const double human_speed,
               const double clearance, double *vhTr, double *twoa, double *k, double *kk, const char *what) {
  if (!(std::isfinite(reaction_time) && reaction_time >= 0.0 && std::isfinite(stopping_deceleration) &&
        stopping_deceleration > 0.0 && std::isfinite(human_speed) && human_speed >= 0.0 && std::isfinite(clearance) &&
        clearance >= 0.0)) {
    set_error("%s: reaction_time %g, human_speed %g and clearance %g must be finite and >= 0, "
              "stopping_deceleration %g finite and > 0", what, reaction_time, human_speed, clearance,
              stopping_deceleration);
    return TB_ERR_ARG;
  }
  *vhTr = human_speed * reaction_time;
  *twoa = 2.0 * stopping_deceleration;
  *k = stopping_deceleration * reaction_time + human_speed;
  *kk = *k * *k;
  return 0;
}

// Validates the packed drive (TBD_DRIVE_DOUBLES(nv)) of nv motors, already checked to be in 1..NB, and copies T, T^-T,
// I_r, f and the speed limits omega (nullable: entries without them) into the by-value launch parameter: 0, or
// TB_ERR_ARG (message set).  T^-1 by Gauss-Jordan elimination with partial pivoting on [T | I], in fp64.
int load_drive(const double *host, const int nv, const double *omega, DynDrive *d, const char *what) {
  *d = DynDrive{};
  const double *Ir = host + nv * nv, *fr = Ir + nv;
  for (int j = 0; j < nv * nv; ++j)
    if (!std::isfinite(host[j])) { set_error("%s: transmission T is not finite", what); return TB_ERR_ARG; }
  for (int i = 0; i < nv; ++i) {
    if (!(std::isfinite(Ir[i]) && Ir[i] >= 0.0)) {
      set_error("%s: motor %d: rotor inertia %g must be finite and >= 0", what, i, Ir[i]);
      return TB_ERR_ARG;
    }
    if (!(std::isfinite(fr[i]) && fr[i] >= 0.0)) {
      set_error("%s: motor %d: friction %g must be finite and >= 0", what, i, fr[i]);
      return TB_ERR_ARG;
    }
    if (omega && !(omega[i] > 0.0)) {
      set_error("%s: motor %d: speed limit %g must be > 0 (inf allowed)", what, i, omega[i]);
      return TB_ERR_ARG;
    }
    d->Ir[i] = Ir[i];
    d->f[i] = fr[i];
    d->omega[i] = omega ? omega[i] : 0.0;
  }
  double A[NB][2 * NB];
  for (int i = 0; i < nv; ++i)
    for (int j = 0; j < nv; ++j) {
      d->T[i][j] = A[i][j] = host[nv * i + j];
      A[i][nv + j] = i == j ? 1.0 : 0.0;
    }
  for (int c = 0; c < nv; ++c) {
    int p = c;
    for (int r = c + 1; r < nv; ++r)
      if (std::fabs(A[r][c]) > std::fabs(A[p][c])) p = r;
    if (!(A[p][c] != 0.0)) { set_error("%s: transmission T is singular (zero pivot in column %d)", what, c); return TB_ERR_ARG; }
    for (int j = 0; j < 2 * nv; ++j) { const double x = A[c][j]; A[c][j] = A[p][j]; A[p][j] = x; }
    const double piv = A[c][c];
    for (int j = 0; j < 2 * nv; ++j) A[c][j] = A[c][j] / piv;
    for (int r = 0; r < nv; ++r) {
      if (r == c) continue;
      const double e = A[r][c];
      for (int j = 0; j < 2 * nv; ++j) A[r][j] = A[r][j] - e * A[c][j];
    }
  }
  for (int i = 0; i < nv; ++i)
    for (int j = 0; j < nv; ++j) {
      if (!std::isfinite(A[i][nv + j])) { set_error("%s: the inverse of transmission T is not finite", what); return TB_ERR_ARG; }
      d->Tit[j][i] = A[i][nv + j];
    }
  return 0;
}

// Validates the packed coupling (TBD_COUPLING_DOUBLES(nv, nq): E row-major, then o) of nv bodies, already checked to
// be in 1..NB, and copies it into the by-value launch parameter: 0, or the TB_ERR_* code (message set).
int load_coupling(const double *host, const int nv, const int nq, DynCoupling *cp, const char *what) {
  if (nq < 1 || nq > nv) { set_error("%s: nq=%d outside 1..nv=%d", what, nq, nv); return TB_ERR_UNSUPPORTED; }
  *cp = DynCoupling{};
  for (int j = 0; j < nv * nq + nv; ++j)
    if (!std::isfinite(host[j])) { set_error("%s: coupling E or o is not finite", what); return TB_ERR_ARG; }
  for (int k = 0; k < nv; ++k) {
    for (int j = 0; j < nq; ++j) cp->E[k][j] = host[nq * k + j];
    cp->o[k] = host[nv * nq + k];
  }
  for (int j = 0; j < nq; ++j) {
    bool moves = false;
    for (int k = 0; k < nv; ++k) moves = moves || cp->E[k][j] != 0.0;
    if (!moves) { set_error("%s: DOF %d moves no body (column %d of E is zero)", what, j, j); return TB_ERR_ARG; }
  }
  return 0;
}

unsigned blocks(const int M) { return (unsigned)((M + THREADS - 1) / THREADS); }

// 0 if no pointer is null, else "<what>: null pointer" and TB_ERR_ARG.
template <class... P>
int nonnull(const char *what, const P *...ptrs) {
  if ((... && ptrs)) return 0;
  set_error("%s: null pointer", what);
  return TB_ERR_ARG;
}

// One thread per point on `stream`, then the launch status of entry `what`.
template <class... K, class... A>
int launch(const char *what, void (*kernel)(K...), const int M, void *stream, const A &...args) {
  kernel<<<blocks(M), THREADS, 0, (cudaStream_t)stream>>>(args...);
  return launch_status(what);
}

}  // namespace
}  // namespace tb

// Each entry checks its pointers, its scalars and the packed model and parameters (loaders), in that order, and
// launches; __func__ names the entry in every error message.

extern "C" int tbd_version(void) { return TBD_VERSION; }

extern "C" int tbd_rnea(const double *model_host, int nv, int M, const double *q, const double *qd, const double *qdd,
                        double *tau, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, q, qd, qdd, tau)) return rc;
  DynModel m;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  return launch(__func__, rnea_kernel, M, stream, m, nv, M, q, qd, qdd, tau);
}

// friction may be null (no friction).
extern "C" int tbd_torque_terms(const double *model_host, int nv, int M, const double *q, const double *qs,
                                const double *qss, const double *friction, double *a, double *b, double *c,
                                void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  return launch(__func__, torque_terms_kernel, M, stream, m, nv, M, q, qs, qss, friction, a, b, c);
}

extern "C" int tbd_frame_velocity(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                                  const double *qd, double *v, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qd, v)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, -1, &f, __func__)) return rc;
  return launch(__func__, frame_velocity_kernel, M, stream, m, f, nv, M, q, qd, v);
}

extern "C" int tbd_velocity_norm_terms(const double *model_host, int nv, const double *frame_host, const double *S_host,
                                       int M, const double *q, const double *qs, double *b, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, S_host, q, qs, b)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, S_host, -1, &f, __func__)) return rc;
  return launch(__func__, velocity_norm_terms_kernel, M, stream, m, f, nv, M, q, qs, b);
}

extern "C" int tbd_frame_acceleration(const double *model_host, int nv, const double *frame_host, int M,
                                      const double *q, const double *qd, const double *qdd, double *acc, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qd, qdd, acc)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, -1, &f, __func__)) return rc;
  if (const int rc = refuse_world(f, __func__, " for accelerations")) return rc;
  return launch(__func__, frame_acceleration_kernel, M, stream, m, f, nv, M, q, qd, qdd, acc);
}

extern "C" int tbd_acceleration_terms(const double *model_host, int nv, const double *frame_host, int components, int M,
                                      const double *q, const double *qs, const double *qss, double *a, double *b,
                                      void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qs, qss, a, b)) return rc;
  if (components < 1 || components > 63) {
    set_error("%s: components=%d must be a bit mask in 1..63", __func__, components);
    return TB_ERR_ARG;
  }
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, -1, &f, __func__)) return rc;
  if (const int rc = refuse_world(f, __func__, " for accelerations")) return rc;
  const int k = __builtin_popcount((unsigned)components);
  return launch(__func__, acceleration_terms_kernel, M, stream, m, f, nv, components, k, M, q, qs, qss, a, b);
}

// The contact wrench is always in the contact frame's own axes: its reference-frame field is ignored.
extern "C" int tbd_contact_wrench(const double *model_host, int nv, const double *frame_host, const double *object_host,
                                  int M, const double *q, const double *qd, const double *qdd, double *w,
                                  void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, object_host, q, qd, qdd, w)) return rc;
  DynModel m;
  DynFrame f;
  DynObject o;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, TBD_LOCAL, &f, __func__)) return rc;
  if (const int rc = load_object(object_host, &o, __func__)) return rc;
  return launch(__func__, contact_wrench_kernel, M, stream, m, f, o, nv, M, q, qd, qdd, w);
}

extern "C" int tbd_contact_wrench_terms(const double *model_host, int nv, const double *frame_host,
                                        const double *object_host, int M, const double *q, const double *qs,
                                        const double *qss, double *a, double *b, double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, object_host, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  DynFrame f;
  DynObject o;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, TBD_LOCAL, &f, __func__)) return rc;
  if (const int rc = load_object(object_host, &o, __func__)) return rc;
  return launch(__func__, contact_wrench_terms_kernel, M, stream, m, f, o, nv, M, q, qs, qss, a, b, c);
}

extern "C" int tbd_frame_inverse_inertia(const double *model_host, int nv, const double *frame_host, int M,
                                         const double *q, double *Linv, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, Linv)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, -1, &f, __func__)) return rc;
  if (const int rc = refuse_world(f, __func__, "")) return rc;
  return launch(__func__, frame_inverse_inertia_kernel, M, stream, m, f, nv, M, q, Linv);
}

// The collision energy needs the world linear velocity: the frame is read as TBD_LOCAL_WORLD_ALIGNED.
extern "C" int tbd_collision_energy_terms(const double *model_host, int nv, const double *frame_host, double human_mass,
                                          int M, const double *q, const double *qs, double *b, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qs, b)) return rc;
  if (!(human_mass > 0.0)) {
    set_error("%s: human_mass %g must be positive (inf allowed)", __func__, human_mass);
    return TB_ERR_ARG;
  }
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_frame(frame_host, m, nv, nullptr, TBD_LOCAL_WORLD_ALIGNED, &f, __func__)) return rc;
  return launch(__func__, collision_energy_terms_kernel, M, stream, m, f, nv, human_mass, M, q, qs, b);
}

extern "C" int tbd_support_wrench(const double *model_host, int nv, const double *frame_host, const double *base_host,
                                  int M, const double *q, const double *qd, const double *qdd, double *w,
                                  void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, base_host, q, qd, qdd, w)) return rc;
  DynModel m;
  DynFrame s;
  DynBase base;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_support(frame_host, m, nv, &s, __func__)) return rc;
  if (const int rc = load_base(base_host, &base, __func__)) return rc;
  return launch(__func__, support_wrench_kernel, M, stream, m, s, base, nv, M, q, qd, qdd, w);
}

extern "C" int tbd_support_wrench_terms(const double *model_host, int nv, const double *frame_host,
                                        const double *base_host, int M, const double *q, const double *qs,
                                        const double *qss, double *a, double *b, double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, base_host, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  DynFrame s;
  DynBase base;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_support(frame_host, m, nv, &s, __func__)) return rc;
  if (const int rc = load_base(base_host, &base, __func__)) return rc;
  return launch(__func__, support_wrench_terms_kernel, M, stream, m, s, base, nv, M, q, qs, qss, a, b, c);
}

extern "C" int tbd_separation(const double *model_host, int nv, const double *points_host, int P, int H, int NH,
                              int points_per_path, int M, const double *q, const double *qd, const double *humans,
                              double *d, double *w, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, points_host, q, qd, humans, d, w)) return rc;
  DynModel m;
  DynPoints pts;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_points(points_host, P, H, NH, points_per_path, M, m, nv, &pts, __func__)) return rc;
  return launch(__func__, separation_kernel, M, stream, m, pts, nv, H, points_per_path, M, q, qd, humans, d, w);
}

extern "C" int tbd_separation_terms(const double *model_host, int nv, const double *points_host, int P, int H, int NH,
                                    int points_per_path, double reaction_time, double stopping_deceleration,
                                    double human_speed, double clearance, int M, const double *q, const double *qs,
                                    const double *humans, double *b, double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, points_host, q, qs, humans, b, c)) return rc;
  double vhTr, twoa, k, kk;
  if (const int rc = load_limit(reaction_time, stopping_deceleration, human_speed, clearance, &vhTr, &twoa, &k, &kk,
                                __func__))
    return rc;
  DynModel m;
  DynPoints pts;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_points(points_host, P, H, NH, points_per_path, M, m, nv, &pts, __func__)) return rc;
  return launch(__func__, separation_terms_kernel, M, stream, m, pts, nv, H, points_per_path, clearance, vhTr, twoa, k,
                kk, M, q, qs, humans, b, c);
}

extern "C" int tbd_capsule_separation(const double *model_host, int nv, const double *capsules_host, int P, int H,
                                      int NH, int points_per_path, int M, const double *q, const double *qd,
                                      const double *humans, double *d, double *w, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, capsules_host, q, qd, humans, d, w)) return rc;
  DynModel m;
  DynCapsules caps;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_capsules(capsules_host, P, H, NH, points_per_path, M, m, nv, &caps, __func__)) return rc;
  return launch(__func__, capsule_separation_kernel, M, stream, m, caps, nv, H, points_per_path, M, q, qd, humans, d,
                w);
}

extern "C" int tbd_capsule_separation_terms(const double *model_host, int nv, const double *capsules_host, int P,
                                            int H, int NH, int points_per_path, double reaction_time,
                                            double stopping_deceleration, double human_speed, double clearance, int M,
                                            const double *q, const double *qs, const double *humans, double *b,
                                            double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, capsules_host, q, qs, humans, b, c)) return rc;
  double vhTr, twoa, k, kk;
  if (const int rc = load_limit(reaction_time, stopping_deceleration, human_speed, clearance, &vhTr, &twoa, &k, &kk,
                                __func__))
    return rc;
  DynModel m;
  DynCapsules caps;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_capsules(capsules_host, P, H, NH, points_per_path, M, m, nv, &caps, __func__)) return rc;
  return launch(__func__, capsule_separation_terms_kernel, M, stream, m, caps, nv, H, points_per_path, clearance, vhTr,
                twoa, k, kk, M, q, qs, humans, b, c);
}

extern "C" int tbd_drive_torque(const double *model_host, int nv, const double *drive_host, int M, const double *q,
                                const double *qd, const double *qdd, double *tau_m, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, drive_host, q, qd, qdd, tau_m)) return rc;
  DynModel m;
  DynDrive d;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_drive(drive_host, nv, nullptr, &d, __func__)) return rc;
  return launch(__func__, drive_torque_kernel, M, stream, m, d, nv, M, q, qd, qdd, tau_m);
}

extern "C" int tbd_drive_torque_terms(const double *model_host, int nv, const double *drive_host, int M,
                                      const double *q, const double *qs, const double *qss, double *a, double *b,
                                      double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, drive_host, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  DynDrive d;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_drive(drive_host, nv, nullptr, &d, __func__)) return rc;
  return launch(__func__, drive_torque_terms_kernel, M, stream, m, d, nv, M, q, qs, qss, a, b, c);
}

// No model: the speed row needs only the transmission.
extern "C" int tbd_drive_speed_terms(int nv, const double *drive_host, const double *speed_limit, int M,
                                     const double *qs, double *b, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, drive_host, speed_limit, qs, b)) return rc;
  if (const int rc = check_sizes(nv, M, __func__)) return rc;
  DynDrive d;
  if (const int rc = load_drive(drive_host, nv, speed_limit, &d, __func__)) return rc;
  return launch(__func__, drive_speed_terms_kernel, M, stream, d, nv, M, qs, b);
}

extern "C" int tbd_joint_wrench(const double *model_host, int nv, const double *frame_host, int M, const double *q,
                                const double *qd, const double *qdd, double *w, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qd, qdd, w)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_joint_frame(frame_host, m, nv, &f, __func__)) return rc;
  return launch(__func__, joint_wrench_kernel, M, stream, m, f, nv, M, q, qd, qdd, w);
}

extern "C" int tbd_joint_wrench_terms(const double *model_host, int nv, const double *frame_host, int components,
                                      int M, const double *q, const double *qs, const double *qss, double *a, double *b,
                                      double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, frame_host, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  DynFrame f;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_joint_frame(frame_host, m, nv, &f, __func__)) return rc;
  if (components < 1 || components > 63) {
    set_error("%s: components=%d must be a bit mask in 1..63", __func__, components);
    return TB_ERR_ARG;
  }
  const int k = __builtin_popcount((unsigned)components);
  return launch(__func__, joint_wrench_terms_kernel, M, stream, m, f, nv, components, k, M, q, qs, qss, a, b, c);
}

extern "C" int tbd_energy_momentum(const double *model_host, int nv, int M, const double *q, const double *qd,
                                   double *out, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, q, qd, out)) return rc;
  DynModel m;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  return launch(__func__, energy_momentum_kernel, M, stream, m, nv, M, q, qd, out);
}

extern "C" int tbd_energy_momentum_terms(const double *model_host, int nv, int which, int M, const double *q,
                                         const double *qs, double *b, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, q, qs, b)) return rc;
  if (which != TBD_KINETIC_ENERGY && which != TBD_MOMENTUM) {
    set_error("%s: which=%d must be TBD_KINETIC_ENERGY (0) or TBD_MOMENTUM (1)", __func__, which);
    return TB_ERR_ARG;
  }
  DynModel m;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  return launch(__func__, energy_momentum_terms_kernel, M, stream, m, nv, which, M, q, qs, b);
}

extern "C" int tbd_coupled_rnea(const double *model_host, int nv, const double *coupling, int nq, int M,
                                const double *q, const double *qd, const double *qdd, double *tau, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, coupling, q, qd, qdd, tau)) return rc;
  DynModel m;
  DynCoupling cp;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_coupling(coupling, nv, nq, &cp, __func__)) return rc;
  return launch(__func__, coupled_rnea_kernel, M, stream, m, cp, nv, nq, M, q, qd, qdd, tau);
}

// friction may be null (no friction).
extern "C" int tbd_coupled_torque_terms(const double *model_host, int nv, const double *coupling, int nq, int M,
                                        const double *q, const double *qs, const double *qss, const double *friction,
                                        double *a, double *b, double *c, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, model_host, coupling, q, qs, qss, a, b, c)) return rc;
  DynModel m;
  DynCoupling cp;
  if (const int rc = load_model(model_host, nv, M, &m, __func__)) return rc;
  if (const int rc = load_coupling(coupling, nv, nq, &cp, __func__)) return rc;
  return launch(__func__, coupled_torque_terms_kernel, M, stream, m, cp, nv, nq, M, q, qs, qss, friction, a, b, c);
}

// No model: the expansion needs only the coupling.  qd and qd_out, and qdd and qdd_out, are both given or both NULL.
extern "C" int tbd_coupling_expand(int nv, const double *coupling, int nq, int M, const double *q, const double *qd,
                                   const double *qdd, double *q_out, double *qd_out, double *qdd_out, void *stream) {
  using namespace tb;
  if (const int rc = nonnull(__func__, coupling, q, q_out)) return rc;
  if (!qd != !qd_out || !qdd != !qdd_out) {
    set_error("%s: qd and qd_out (and qdd and qdd_out) must both be given or both be NULL", __func__);
    return TB_ERR_ARG;
  }
  if (const int rc = check_sizes(nv, M, __func__)) return rc;
  DynCoupling cp;
  if (const int rc = load_coupling(coupling, nv, nq, &cp, __func__)) return rc;
  return launch(__func__, coupling_expand_kernel, M, stream, cp, nv, nq, M, q, qd, qdd, q_out, qd_out, qdd_out);
}
