// tb_robust.cu — K2r: TOPP-RA with a robustified (ellipsoidal) CanonicalLinear constraint, one warp per path.
//
// Problem definition (reference):
//   RobustLinearConstraint.compute_constraint_params   toppra/constraint/conic_constraint.py:95-124
//       rows a = F a0, b = F b0, c = F c0 - g; perturbation ellipsoid diag(ru, rx, rc)
//   ecosWrapper.solve_stagewise_optim                   toppra/solverwrapper/ecos_solverwrapper.py:90-207
//       min g.[u,x]  s.t.  x_min <= x <= x_max (NaN -> -/+ECOS_INFTY = 1000), x_next bounds likewise,
//       linear rows, x <= min(ECOS_MAXX = 1e4, xbound_hi), x >= xbound_lo, and per robust row the cone
//       a u + b x + c + || diag(ru, rx, rc) [u, x, 1] ||_2 <= 0                      (:175-188)
//   driver: reachability_algorithm.py:166-376 (same backward / forward passes and retry rule as K2).
//
// The reference hands every stage problem to ECOS (a third-party interior-point solver, absent here): parity is
// UNPINNED for this kernel.  It solves the same 2-variable second-order-cone programs exactly instead:
//   * for a fixed x every row bounds u from one quadratic: with beta = b x + c, gamma^2 = rx^2 x^2 + rc^2,
//     A = a^2 - ru^2, D = a^2 gamma^2 + ru^2 (beta^2 - gamma^2):
//       |a| > ru : one bound   u <= / >= (-a beta - sign(a) sqrt(D)) / A
//       |a| < ru : an interval between the two roots (feasible iff D >= 0 and beta <= 0)
//     so the feasible u-interval [ulo(x), uhi(x)] is a max / min over the lanes (redux.sync reductions);
//   * the feasible x form an interval (the feasible set is convex), w(x) = uhi(x) - ulo(x) is concave: max x / min x
//     are found by a bracketed secant/bisection on w(x) >= 0, the forward step is u = uhi(x).
// With a zero ellipsoid the rows are linear and the results agree with the LP path (tests: 1e-9).
#include <limits.h>

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

// One warp per CTA, like the record scan: a finished path frees its slot at once.
template <int RPL>
__global__ void __launch_bounds__(32, (RPL == 1) ? 28 : 1)
scan_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
                   const double ru, const double rx, const double rc, const double *__restrict__ grid,
                   const int grid_shared, const int B, const int G, const double *__restrict__ sd_start,
                   const double *__restrict__ sd_end, const int flags, double *__restrict__ Kout,
                   double *__restrict__ sdout, double *__restrict__ uout, int *__restrict__ status,
                   int *__restrict__ fail_stage, int *__restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  const int N = G - 1, nC = R + 2;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  double *Kp = Kout + (size_t)path * G * 2;
  const bool backward_only = (flags & 1) != 0;
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  double a[RPL], b[RPL], c[RPL];
  unsigned cmask[RPL];
  int n_eval = 0, n_retry = 0;

  if (flags & 2) {
    // compute_feasible_sets (reachability_algorithm.py:131-164): x, x_next in [-1e4, 1e4], every stage on its own
    for (int i = 0; i <= N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask);
      const double xl = fmax(-CVXPY_MAXX, rec[3 * R]);
      const double xh = fmin(CVXPY_MAXX, fmin(ECOS_MAXX, rec[3 * R + 1]));
      if (i < N) {
        const double delta = gp[i + 1] - gp[i];
        if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = -CVXPY_MAXX; }
        if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -CVXPY_MAXX; }
      }
      double x0 = nan_d, x1 = nan_d;
      if (!extreme_x<RPL>(-1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, x0, n_eval, nan_d)) x0 = nan_d;
      if (!extreme_x<RPL>(+1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, x1, n_eval, nan_d)) x1 = nan_d;
      if (x0 < 0) x0 = 0;
      if (lane == 0) { Kp[2 * i] = x0; Kp[2 * i + 1] = x1; }
    }
    if (lane == 0) { status[path] = TB_STATUS_OK; if (fail_stage) fail_stage[path] = -1; }
    return;
  }
  const double sde = sd_end ? sd_end[path] : 0.0;
  const double sds = sd_start ? sd_start[path] : 0.0;
  double kn0 = sde * sde, kn1 = sde * sde;
  if (lane == 0) { Kp[2 * N] = kn0; Kp[2 * N + 1] = kn1; }
  int st = TB_STATUS_OK, fstage = -1;
  for (int i = N - 1; i >= 0; --i) {
    const double *rec = rec_path + (size_t)i * W;
    rload_rows<RPL>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask);
    if (i > 0 && lane * 16 < W)  // pull the next stage's record towards L1 while this stage is solved
      asm volatile("prefetch.global.L1 [%0];" ::"l"(rec - W + lane * 16));
    // x box: NaN x_min/x_max -> -/+ECOS_INFTY; xbound: x <= min(ECOS_MAXX, hi), x >= lo  (ecos_solverwrapper.py:112-172)
    const double xl = fmax(-ECOS_INFTY, rec[3 * R]);
    const double xh = fmin(ECOS_INFTY, fmin(ECOS_MAXX, rec[3 * R + 1]));
    const double delta = gp[i + 1] - gp[i];
    if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = kn0; }
    if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -kn1; }
    double x_upper = nan_d, x_lower = nan_d;
    const bool ok_hi = extreme_x<RPL>(+1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, x_upper, n_eval, kn1);
    const bool ok_lo = ok_hi && extreme_x<RPL>(-1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, x_lower, n_eval, kn0);
    if (!ok_hi) x_upper = nan_d;
    if (!ok_lo) x_lower = nan_d;
    if (x_lower < 0) x_lower = 0;
    if (lane == 0) { Kp[2 * i] = x_lower; Kp[2 * i + 1] = x_upper; }
    if (!(ok_hi && ok_lo)) {
      st = TB_STATUS_FAIL_UNCONTROLLABLE;
      fstage = i;
      for (int j = lane; j < 2 * i; j += 32) Kp[j] = 0.0;
      break;
    }
    kn0 = x_lower;
    kn1 = x_upper;
  }
  __syncwarp();
  const double x_start = sds * sds;
  if (st == TB_STATUS_OK && !backward_only) {
    if (x_start + ALG_SMALL < kn0 || kn1 + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  if (backward_only) {
    if (lane == 0) { status[path] = st; if (fail_stage) fail_stage[path] = fstage; }
    return;
  }
  if (st != TB_STATUS_OK) {
    for (int j = lane; j < G; j += 32) sdp[j] = nan_d;
    for (int j = lane; j < N; j += 32) up[j] = nan_d;
  } else {
    double x = x_start;
    if (lane == 0) sdp[0] = x;
    for (int i = 0; i < N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask);
      if (i + 2 < N && lane * 16 < W) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 2 * W + lane * 16));
      const double delta = gp[i + 1] - gp[i];
      const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
      if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = k0; }
      if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -k1; }
      int tries = 0;
      bool ok;
      double uopt = 0.0;
      while (true) {
        double uh;
        const double w = u_interval<RPL>(x, a, b, c, cmask, lane, ru, rx, rc, uh);
        ++n_eval;
        ok = w >= 0.0;
        uopt = uh;
        if (ok || tries >= MAX_TRIES) break;
        x = fmax(x - ALG_TINY, 0.999 * x);
        ++tries;
        ++n_retry;
      }
      if (!ok) {
        st = TB_STATUS_ERR_UNKNOWN;
        fstage = i;
        if (lane == 0) sdp[i] = x;
        for (int j = i + 1 + lane; j < G; j += 32) sdp[j] = nan_d;
        for (int j = i + lane; j < N; j += 32) up[j] = 0.0;
        break;
      }
      double x_next = x + 2 * delta * uopt;
      x_next = fmax(x_next - ALG_TINY, 0.9999 * x_next);
      x_next = fmin(k1, fmax(k0, x_next));
      if (lane == 0) {
        up[i] = uopt;
        if (tries) sdp[i] = x;
        sdp[i + 1] = x_next;
      }
      x = x_next;
    }
    __syncwarp();
    for (int j = lane; j < G; j += 32) sdp[j] = sqrt(sdp[j]);
  }
  if (lane == 0) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
    if (counters) {
      counters[path * 4 + 0] = n_eval;
      counters[path * 4 + 1] = 0;
      counters[path * 4 + 2] = 0;
      counters[path * 4 + 3] = n_retry;
    }
  }
}

}  // namespace
}  // namespace tb

extern "C" int tb_scan_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                              const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                              const double *sd_start, const double *sd_end, int flags, double *K, double *sd, double *u,
                              int *status, int *fail_stage, int *counters, void *stream) {
  using namespace tb;
  if (!records || !grid || !ellipsoid_host3 || !K || !status || B <= 0 || G <= 0 || R < 0) {
    set_error("tb_scan_robust: bad argument");
    return TB_ERR_ARG;
  }
  const bool backward_only = (flags & (TB_SCAN_BACKWARD_ONLY | TB_SCAN_FEASIBLE_SETS)) != 0;
  if (!backward_only && (!sd || (G > 1 && !u))) { set_error("tb_scan_robust: null output"); return TB_ERR_ARG; }
  if (R > MAX_ROWS) { set_error("tb_scan_robust: R=%d > %d rows", R, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2) { set_error("tb_scan_robust: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  if (conic_row0 < 0 || conic_rows < 0 || conic_row0 + conic_rows > R) { set_error("tb_scan_robust: bad conic row range"); return TB_ERR_ARG; }
  if (ellipsoid_host3[0] < 0 || ellipsoid_host3[1] < 0 || ellipsoid_host3[2] < 0) { set_error("tb_scan_robust: negative ellipsoid axis"); return TB_ERR_ARG; }
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(R + 2, [&](auto rpl) {
    scan_robust_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(records, W, R, conic_row0, conic_rows, ru, rx, rc,
                                                                      grid, grid_shared, B, G, sd_start, sd_end, flags,
                                                                      K, sd, u, status, fail_stage, counters);
  });
  return check_launch("tb_scan_robust");
}
