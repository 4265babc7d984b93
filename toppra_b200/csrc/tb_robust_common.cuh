// tb_robust_common.cuh — the conic stage-problem primitives of one warp, shared by tb_robust.cu (K2r, libtoppra_b200.so)
// and tb_conic.cu (robust TOPPRAsd passes and single stage solves, libtoppra_b200_robust.so).
//
// A stage problem has two variables (u, x) and rows  a u + b x + c (+ ||diag(ru, rx, rc) [u, x, 1]||_2) <= 0, the cone
// term on the rows of the robust constraint only (conic_constraint.py:95-124, ecos_solverwrapper.py:175-188):
//   * for a fixed x every row bounds u from one quadratic: with beta = b x + c, gamma^2 = rx^2 x^2 + rc^2,
//     A = a^2 - ru^2, D = a^2 gamma^2 + ru^2 (beta^2 - gamma^2):
//       |a| > ru : one bound   u <= / >= (-a beta - sign(a) sqrt(D)) / A
//       |a| < ru : an interval between the two roots (feasible iff D >= 0 and beta <= 0)
//     so the feasible u-interval [ulo(x), uhi(x)] is a max / min over the lanes (redux.sync reductions);
//   * the feasible x form an interval (the feasible set is convex), w(x) = uhi(x) - ulo(x) is concave: max x / min x
//     are found by a bracketed secant/bisection on w(x) >= 0 (extreme_x).
// Lane `lane` holds rows lane + 32 s, s < RPL; rows 0 and 1 are the x_next rows, the records' rows start at row 2.
#pragma once
#include "tb_common.cuh"

namespace tb {
namespace {

constexpr double ECOS_INFTY = 1000.0;   // toppra/constants.py:47
constexpr double ECOS_MAXX = 10000.0;   // toppra/constants.py:46

// Bounds on u implied by one row at a fixed x.  lo/hi are only tightened; bad = the row excludes every u.
__device__ __forceinline__ void row_u_bounds(const bool conic, const double a, const double b, const double c,
                                             const double ru, const double rx, const double rc, const double x,
                                             double &lo, double &hi, bool &bad) {
  double beta = b * x + c;
  double gamma2 = 0.0;
  if (conic) gamma2 = rx * rx * (x * x) + rc * rc;
  if (!conic || ru == 0.0) {
    // linear in u: a u + (beta + gamma) <= 0
    if (conic) beta = beta + sqrt(gamma2);
    if (a > LP_TINY) { const double t = -beta / a; hi = (t < hi) ? t : hi; }
    else if (a < -LP_TINY) { const double t = -beta / a; lo = (t > lo) ? t : lo; }
    else if (beta > LP_SMALL) bad = true;
    return;
  }
  const double A = a * a - ru * ru;
  const double D = a * a * gamma2 + ru * ru * (beta * beta - gamma2);
  const double p = -a * beta;
  if (A > 0.0) {
    // f(u) = a u + beta + sqrt(ru^2 u^2 + gamma^2) is monotone: one root, on the side where a u + beta <= 0
    const double sq = sqrt(D > 0.0 ? D : 0.0);
    const double s = (a > 0.0) ? 1.0 : -1.0;
    // root = (p - s sq) / A = (beta^2 - gamma^2) / (p + s sq): take the form without cancellation
    const double root = (s * p <= 0.0) ? (p - s * sq) / A : (beta * beta - gamma2) / (p + s * sq);
    if (a > 0.0) hi = (root < hi) ? root : hi; else lo = (root > lo) ? root : lo;
  } else if (A < 0.0) {
    // f is convex with f -> +inf on both sides: feasible between the two roots, iff D >= 0 and beta <= 0
    if (D < 0.0 || beta > 0.0) { bad = true; return; }
    const double sq = sqrt(D);
    const double q = p + ((p >= 0.0) ? sq : -sq);
    double r1, r2;
    if (q != 0.0) { r1 = q / A; r2 = (beta * beta - gamma2) / q; } else { r1 = 0.0; r2 = 0.0; }
    const double rl = (r1 < r2) ? r1 : r2, rh = (r1 < r2) ? r2 : r1;
    lo = (rl > lo) ? rl : lo;
    hi = (rh < hi) ? rh : hi;
  } else {
    // |a| == ru > 0: 2 a beta u + beta^2 - gamma^2 = 0, feasible side exists only for beta < 0
    if (beta >= 0.0) { bad = true; return; }
    const double root = (gamma2 - beta * beta) / (2 * a * beta);
    if (a > 0.0) hi = (root < hi) ? root : hi; else lo = (root > lo) ? root : lo;
  }
}

// Feasible u-interval at x over all rows of the stage (lane = row; RPL rows per lane).  Returns the width
// w = uhi - ulo (negative or -inf if infeasible) and uhi.
template <int RPL>
__device__ __forceinline__ double u_interval(const double x, const double (&a)[RPL], const double (&b)[RPL],
                                             const double (&c)[RPL], const unsigned (&cmask)[RPL], const int lane,
                                             const double ru, const double rx, const double rc, double &uhi) {
  double lo = VAR_MIN, hi = VAR_MAX;
  bool bad = false;
#pragma unroll
  for (int s = 0; s < RPL; ++s) row_u_bounds(cmask[s] != 0, a[s], b[s], c[s], ru, rx, rc, x, lo, hi, bad);
  const double ulo = -warp_min(-lo);
  uhi = warp_min(hi);
  if (__any_sync(FULL, bad)) return -__longlong_as_double(0x7ff0000000000000LL);
  return uhi - ulo;
}

// Both ends of the feasible u-interval at x, each the warp-reduced bound itself (ulo is not uhi - w).  Returns whether
// the interval is non-empty, by the rule of u_interval (w >= 0, no row excluding every u).
template <int RPL>
__device__ __forceinline__ bool u_bounds(const double x, const double (&a)[RPL], const double (&b)[RPL],
                                         const double (&c)[RPL], const unsigned (&cmask)[RPL], const double ru,
                                         const double rx, const double rc, double &ulo, double &uhi) {
  double lo = VAR_MIN, hi = VAR_MAX;
  bool bad = false;
#pragma unroll
  for (int s = 0; s < RPL; ++s) row_u_bounds(cmask[s] != 0, a[s], b[s], c[s], ru, rx, rc, x, lo, hi, bad);
  ulo = -warp_min(-lo);
  uhi = warp_min(hi);
  if (__any_sync(FULL, bad)) return false;
  return uhi - ulo >= 0.0;
}

// Largest (dir = +1) or smallest (dir = -1) x in [xl, xh] with a non-empty u-interval.  false = infeasible.
template <int RPL>
__device__ __forceinline__ bool extreme_x(const int dir, const double xl, const double xh, const double (&a)[RPL],
                                          const double (&b)[RPL], const double (&c)[RPL],
                                          const unsigned (&cmask)[RPL], const int lane, const double ru,
                                          const double rx, const double rc, double &xout, int &n_eval,
                                          const double hint /* NaN = none */) {
  if (xl > xh) return false;
  double uh;
  const double xgoal = (dir > 0) ? xh : xl, xother = (dir > 0) ? xl : xh;
  double wg = u_interval<RPL>(xgoal, a, b, c, cmask, lane, ru, rx, rc, uh);
  ++n_eval;
  if (wg >= 0.0) { xout = xgoal; return true; }
  double wo = u_interval<RPL>(xother, a, b, c, cmask, lane, ru, rx, rc, uh);
  ++n_eval;
  double xf = xother, wf = wo;
  double xb0 = xgoal, wb0 = wg;
  if (wo >= 0.0 && hint > xl && hint < xh) {
    // the answer of the neighbouring stage is usually close: two probes around it shrink the bracket at once
    const double h1 = hint, h2 = (dir > 0) ? fmin(xh, hint * 1.25 + 1e-9) : fmax(xl, hint * 0.8 - 1e-9);
    const double w1 = u_interval<RPL>(h1, a, b, c, cmask, lane, ru, rx, rc, uh);
    ++n_eval;
    if (w1 >= 0.0) {
      xf = h1; wf = w1;
      if (h2 != xgoal) {
        const double w2 = u_interval<RPL>(h2, a, b, c, cmask, lane, ru, rx, rc, uh);
        ++n_eval;
        if (w2 >= 0.0) { xf = h2; wf = w2; } else { xb0 = h2; wb0 = w2; }
      }
    } else {
      xb0 = h1; wb0 = w1;
    }
  }
  if (!(wo >= 0.0)) {
    // both ends infeasible: golden-section search for the maximum of the concave width
    const double invphi = 0.6180339887498949;
    double lo = xl, hi = xh;
    double x1 = hi - invphi * (hi - lo), x2 = lo + invphi * (hi - lo);
    double w1 = u_interval<RPL>(x1, a, b, c, cmask, lane, ru, rx, rc, uh);
    double w2 = u_interval<RPL>(x2, a, b, c, cmask, lane, ru, rx, rc, uh);
    n_eval += 2;
    bool found = false;
    for (int it = 0; it < 80; ++it) {
      if (w1 >= 0.0) { xf = x1; wf = w1; found = true; break; }
      if (w2 >= 0.0) { xf = x2; wf = w2; found = true; break; }
      if (!(hi - lo > 1e-15 * (fabs(hi) + fabs(lo)) + 1e-300)) break;
      if (w1 > w2) { hi = x2; x2 = x1; w2 = w1; x1 = hi - invphi * (hi - lo); w1 = u_interval<RPL>(x1, a, b, c, cmask, lane, ru, rx, rc, uh); }
      else { lo = x1; x1 = x2; w1 = w2; x2 = lo + invphi * (hi - lo); w2 = u_interval<RPL>(x2, a, b, c, cmask, lane, ru, rx, rc, uh); }
      ++n_eval;
    }
    if (!found) return false;
  }
  // bracket: xf feasible (wf >= 0), xb infeasible (w < 0, possibly -inf)
  double xb = xb0, wb = wb0;
  for (int it = 0; it < 200; ++it) {
    const double width = fabs(xb - xf);
    if (!(width > 2.3e-16 * (fabs(xb) + fabs(xf)) + 1e-300)) break;
    double t;
    const bool finite = wb > -1e300;
    if (finite && (it % 3) != 2) {
      double frac = wf / (wf - wb);  // secant step from the feasible end
      frac = (frac < 0.02) ? 0.02 : ((frac > 0.98) ? 0.98 : frac);
      t = xf + (xb - xf) * frac;
    } else {
      t = 0.5 * (xf + xb);
    }
    if (t == xf || t == xb) break;
    const double wt = u_interval<RPL>(t, a, b, c, cmask, lane, ru, rx, rc, uh);
    ++n_eval;
    if (wt >= 0.0) { xf = t; wf = wt; } else { xb = t; wb = wt; }
  }
  xout = xf;
  return true;
}

template <int RPL>
__device__ __forceinline__ void rload_rows(const double *__restrict__ rec, const int R, const int nC, const int lane,
                                           const int conic0, const int conicn, double (&a)[RPL], double (&b)[RPL],
                                           double (&c)[RPL], unsigned (&cmask)[RPL]) {
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r >= 2 && r < nC) {
      a[s] = rec[r - 2]; b[s] = rec[R + r - 2]; c[s] = rec[2 * R + r - 2];
      cmask[s] = (r - 2 >= conic0 && r - 2 < conic0 + conicn) ? 1u : 0u;
    } else {
      a[s] = 0.0; b[s] = 0.0; c[s] = -1.0; cmask[s] = 0u;
    }
  }
}

}  // namespace
}  // namespace tb
