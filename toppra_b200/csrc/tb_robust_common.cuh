// tb_robust_common.cuh — the conic stage-problem primitives of one warp, shared through tb_robust_kernels.cuh by
// tb_robust.cu (K2r, libtoppra_b200.so), tb_conic.cu (robust TOPPRAsd passes and single stage solves,
// libtoppra_b200_robust.so), tb_reach.cu (reachable sets, libtoppra_b200_reach.so) and tb_cones.cu (the same with an
// ellipsoid per row and a u box, libtoppra_b200_cones.so).
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
//   * min g0 u + g1 x over one stage: the feasible x-interval, then golden-section search on a convex phi(x)
//     (socp_stage_solve, shared by the stage solves and the reachable sets of the companion libraries).
// Lane `lane` holds rows lane + 32 s, s < RPL; rows 0 and 1 are the x_next rows, the records' rows start at row 2.
#pragma once
#include <type_traits>

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
    // |a| == ru > 0: 2 a beta u + beta^2 - gamma^2 = 0, feasible side exists only for beta < 0 -- or for
    // beta == gamma == 0 (rc = 0 at x = 0), where a u + ru |u| <= 0 holds for every u <= 0 (a > 0) / u >= 0 (a < 0)
    if (beta >= 0.0) {
      if (beta != 0.0 || gamma2 != 0.0) { bad = true; return; }
      if (a > 0.0) hi = (0.0 < hi) ? 0.0 : hi; else lo = (0.0 > lo) ? 0.0 : lo;
      return;
    }
    const double root = (gamma2 - beta * beta) / (2 * a * beta);
    if (a > 0.0) hi = (root < hi) ? root : hi; else lo = (root > lo) ? root : lo;
  }
}

// The axes of a lane's rows come in one of two forms: one value for every row (one ellipsoid, `double`), or one value
// per lane slot (Slots<RPL>, read from a cone table by load_cones).  axis() reads the value of slot s.  Every primitive
// below takes the axes ru, rx, rc in either form (Ax) and the u box [ulo_box, uhi_box] the u-interval starts from
// ([VAR_MIN, VAR_MAX] when the stage has none).
template <int RPL>
struct Slots {
  double v[RPL];
};
__device__ __forceinline__ double axis(const double v, const int) { return v; }
template <int RPL>
__device__ __forceinline__ double axis(const Slots<RPL> &v, const int s) { return v.v[s]; }

// Feasible u-interval at x over all rows of the stage (lane = row; RPL rows per lane).  Returns the width
// w = uhi - ulo (negative or -inf if infeasible) and uhi.
template <int RPL, class Ax>
__device__ __forceinline__ double u_interval(const double x, const double (&a)[RPL], const double (&b)[RPL],
                                             const double (&c)[RPL], const unsigned (&cmask)[RPL], const int lane,
                                             const Ax ru, const Ax rx, const Ax rc, const double ulo_box,
                                             const double uhi_box, double &uhi) {
  double lo = ulo_box, hi = uhi_box;
  bool bad = false;
#pragma unroll
  for (int s = 0; s < RPL; ++s)
    row_u_bounds(cmask[s] != 0, a[s], b[s], c[s], axis(ru, s), axis(rx, s), axis(rc, s), x, lo, hi, bad);
  const double ulo = -warp_min(-lo);
  uhi = warp_min(hi);
  if (__any_sync(FULL, bad)) return -__longlong_as_double(0x7ff0000000000000LL);
  return uhi - ulo;
}

// Both ends of the feasible u-interval at x, each the warp-reduced bound itself (ulo is not uhi - w).  Returns whether
// the interval is non-empty, by the rule of u_interval (w >= 0, no row excluding every u).
template <int RPL, class Ax>
__device__ __forceinline__ bool u_bounds(const double x, const double (&a)[RPL], const double (&b)[RPL],
                                         const double (&c)[RPL], const unsigned (&cmask)[RPL], const Ax ru,
                                         const Ax rx, const Ax rc, const double ulo_box, const double uhi_box,
                                         double &ulo, double &uhi) {
  double lo = ulo_box, hi = uhi_box;
  bool bad = false;
#pragma unroll
  for (int s = 0; s < RPL; ++s)
    row_u_bounds(cmask[s] != 0, a[s], b[s], c[s], axis(ru, s), axis(rx, s), axis(rc, s), x, lo, hi, bad);
  ulo = -warp_min(-lo);
  uhi = warp_min(hi);
  if (__any_sync(FULL, bad)) return false;
  return uhi - ulo >= 0.0;
}

// Largest (dir = +1) or smallest (dir = -1) x in [xl, xh] with a non-empty u-interval.  false = infeasible.
template <int RPL, class Ax>
__device__ __forceinline__ bool extreme_x(const int dir, const double xl, const double xh, const double (&a)[RPL],
                                          const double (&b)[RPL], const double (&c)[RPL],
                                          const unsigned (&cmask)[RPL], const int lane, const Ax ru, const Ax rx,
                                          const Ax rc, const double ulo_box, const double uhi_box, double &xout,
                                          int &n_eval, const double hint /* NaN = none */) {
  if (xl > xh) return false;
  double uh;
  const double xgoal = (dir > 0) ? xh : xl, xother = (dir > 0) ? xl : xh;
  double wg = u_interval<RPL, Ax>(xgoal, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
  ++n_eval;
  if (wg >= 0.0) { xout = xgoal; return true; }
  double wo = u_interval<RPL, Ax>(xother, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
  ++n_eval;
  double xf = xother, wf = wo;
  double xb0 = xgoal, wb0 = wg;
  if (wo >= 0.0 && hint > xl && hint < xh) {
    // the answer of the neighbouring stage is usually close: two probes around it shrink the bracket at once
    const double h1 = hint, h2 = (dir > 0) ? fmin(xh, hint * 1.25 + 1e-9) : fmax(xl, hint * 0.8 - 1e-9);
    const double w1 = u_interval<RPL, Ax>(h1, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
    ++n_eval;
    if (w1 >= 0.0) {
      xf = h1; wf = w1;
      if (h2 != xgoal) {
        const double w2 = u_interval<RPL, Ax>(h2, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
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
    double w1 = u_interval<RPL, Ax>(x1, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
    double w2 = u_interval<RPL, Ax>(x2, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
    n_eval += 2;
    bool found = false;
    for (int it = 0; it < 80; ++it) {
      if (w1 >= 0.0) { xf = x1; wf = w1; found = true; break; }
      if (w2 >= 0.0) { xf = x2; wf = w2; found = true; break; }
      if (!(hi - lo > 1e-15 * (fabs(hi) + fabs(lo)) + 1e-300)) break;
      if (w1 > w2) { hi = x2; x2 = x1; w2 = w1; x1 = hi - invphi * (hi - lo); w1 = u_interval<RPL, Ax>(x1, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh); }
      else { lo = x1; x1 = x2; w1 = w2; x2 = lo + invphi * (hi - lo); w2 = u_interval<RPL, Ax>(x2, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh); }
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
    const double wt = u_interval<RPL, Ax>(t, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, uh);
    ++n_eval;
    if (wt >= 0.0) { xf = t; wf = wt; } else { xb = t; wb = wt; }
  }
  xout = xf;
  return true;
}

// One stage's rows from its record; rows 0 and 1 (the x_next rows) and the padding past nC are 0 u + 0 x - 1 <= 0.
// PER_ROW = false: the conic mask of the rows [conic0, conic0 + conicn), set here per stage.  PER_ROW = true: the mask
// came from the cone table (load_cones) and stays; with ub the stage's u box is the record's u-bound pair.
template <int RPL, bool PER_ROW>
__device__ __forceinline__ void rload_rows(const double *__restrict__ rec, const int R, const int nC, const int lane,
                                           const int conic0, const int conicn, double (&a)[RPL], double (&b)[RPL],
                                           double (&c)[RPL], unsigned (&cmask)[RPL], const bool ub, double &ulo,
                                           double &uhi) {
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r >= 2 && r < nC) {
      a[s] = rec[r - 2]; b[s] = rec[R + r - 2]; c[s] = rec[2 * R + r - 2];
      if constexpr (!PER_ROW) cmask[s] = (r - 2 >= conic0 && r - 2 < conic0 + conicn) ? 1u : 0u;
    } else {
      a[s] = 0.0; b[s] = 0.0; c[s] = -1.0;
      if constexpr (!PER_ROW) cmask[s] = 0u;
    }
  }
  if constexpr (PER_ROW) {
    if (ub) { ulo = rec[3 * R + 2]; uhi = rec[3 * R + 3]; }
  }
}

// The cone table of libtoppra_b200_cones.so, one row (robust flag 0/1, ru, rx, rc) per record row, handed to the
// kernels by value as a __grid_constant__ parameter (4032 bytes; rows past R are zero) and read in place.
struct ConeTable {
  double v[MAX_ROWS][4];
};

// The conic mask and the axes of the lane's rows from the cone table, once per path: row k = lane + 32 s - 2 of the
// table for 0 <= k < n, linear rows (the x_next rows, the padding) elsewhere.
template <int RPL>
__device__ __forceinline__ void load_cones(const ConeTable *__restrict__ t, const int n, const int lane,
                                           unsigned (&cmask)[RPL], Slots<RPL> &ru, Slots<RPL> &rx, Slots<RPL> &rc) {
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int k = lane + 32 * s - 2;
    const bool in = k >= 0 && k < n;
    cmask[s] = (in && t->v[k][0] != 0.0) ? 1u : 0u;
    ru.v[s] = in ? t->v[k][1] : 0.0;
    rx.v[s] = in ? t->v[k][2] : 0.0;
    rc.v[s] = in ? t->v[k][3] : 0.0;
  }
}

// The axes of a row form: double (one ellipsoid) or Slots<RPL> (a cone table).
template <int RPL, bool PER_ROW>
using Axes = typename std::conditional<PER_ROW, Slots<RPL>, double>::type;

// min g0 u + g1 x over one stage whose rows (x_next rows included) the warp holds, on xl <= x <= xh: the feasible
// x-interval [xmin, xmax] by extreme_x, then (g0 != 0) the convex phi(x) by golden-section search on it.  us / xs out,
// NaN NaN when infeasible.
template <int RPL, class Ax>
__device__ __forceinline__ void socp_stage_solve(const double g0, const double g1, const double xl, const double xh,
                                                 const double (&a)[RPL], const double (&b)[RPL],
                                                 const double (&c)[RPL], const unsigned (&cmask)[RPL], const int lane,
                                                 const Ax ru, const Ax rx, const Ax rc, const double ulo_box,
                                                 const double uhi_box, double &us, double &xs) {
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  int n_eval = 0;
  double xmin = nan_d, xmax = nan_d;
  xs = nan_d;
  us = nan_d;
  const bool feasible = extreme_x<RPL, Ax>(-1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, xmin, n_eval, nan_d) &&
                        extreme_x<RPL, Ax>(+1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ulo_box, uhi_box, xmax, n_eval, nan_d);
  if (feasible && g0 == 0.0) {
    // the objective does not depend on u: the x end g1 points to (xmin for g1 == 0), u the middle of the u-interval
    // there.  An interior-point solver returns some u of that face; which one is solver-dependent.
    xs = (g1 < 0.0) ? xmax : xmin;
    double ulo, uhi;
    if (u_bounds<RPL, Ax>(xs, a, b, c, cmask, ru, rx, rc, ulo_box, uhi_box, ulo, uhi)) us = 0.5 * (ulo + uhi);
    else xs = nan_d;
  } else if (feasible) {
    // phi(x) = g1 x + g0 u*(x), u*(x) = uhi(x) (g0 < 0) or ulo(x) (g0 > 0): convex on [xmin, xmax] (uhi is concave and
    // ulo convex on the convex feasible set).  Golden-section search down to a few-ulp bracket; the best point
    // evaluated, the two ends included, wins (the first one on ties).
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    const auto phi = [&](const double x, double &u) {
      double ulo, uhi;
      const bool ok = u_bounds<RPL, Ax>(x, a, b, c, cmask, ru, rx, rc, ulo_box, uhi_box, ulo, uhi);
      u = (g0 < 0.0) ? uhi : ulo;
      return ok ? g1 * x + g0 * u : inf;
    };
    double ua, ub;
    const double fa = phi(xmin, ua), fb = phi(xmax, ub);
    double fbest;
    if (fa <= fb) { xs = xmin; us = ua; fbest = fa; } else { xs = xmax; us = ub; fbest = fb; }
    const double invphi = 0.6180339887498949;
    double lo = xmin, hi = xmax;
    double x1 = hi - invphi * (hi - lo), x2 = lo + invphi * (hi - lo);
    double u1, u2;
    double f1 = phi(x1, u1), f2 = phi(x2, u2);
    if (f1 < fbest) { xs = x1; us = u1; fbest = f1; }
    if (f2 < fbest) { xs = x2; us = u2; fbest = f2; }
    for (int it = 0; it < 200; ++it) {
      if (!(hi - lo > 2.3e-16 * (fabs(hi) + fabs(lo)) + 1e-300)) break;
      if (f1 <= f2) {
        hi = x2; x2 = x1; f2 = f1; u2 = u1;
        x1 = hi - invphi * (hi - lo);
        f1 = phi(x1, u1);
        if (f1 < fbest) { xs = x1; us = u1; fbest = f1; }
      } else {
        lo = x1; x1 = x2; f1 = f2; u1 = u2;
        x2 = lo + invphi * (hi - lo);
        f2 = phi(x2, u2);
        if (f2 < fbest) { xs = x2; us = u2; fbest = f2; }
      }
    }
    if (!(fbest < inf)) { xs = nan_d; us = nan_d; }
  }
}

// Host checks of the robust libraries' entries: 0, or the TB_ERR_* code (message set).
inline int check_conic(const int R, const int conic_row0, const int conic_rows, const double *ell, const char *what) {
  if (R > MAX_ROWS) { set_error("%s: R=%d > %d rows", what, R, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (conic_row0 < 0 || conic_rows < 0 || conic_row0 + conic_rows > R) { set_error("%s: bad conic row range", what); return TB_ERR_ARG; }
  if (!(ell[0] >= 0) || !(ell[1] >= 0) || !(ell[2] >= 0)) { set_error("%s: negative ellipsoid axis", what); return TB_ERR_ARG; }
  return 0;
}

}  // namespace
}  // namespace tb
