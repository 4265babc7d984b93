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
// UNPINNED for this kernel.  It solves the same 2-variable second-order-cone programs exactly instead, with the
// primitives of tb_robust_common.cuh: the feasible u-interval [ulo(x), uhi(x)] in closed form per x, max x / min x by a
// bracketed secant/bisection on its width (extreme_x); the forward step is u = uhi(x).
// With a zero ellipsoid the rows are linear and the results agree with the LP path (tests: 1e-9).
#include <limits.h>

#include "tb_robust_common.cuh"

namespace tb {
namespace {

// One warp per CTA, like the record scan: a finished path frees its slot at once.
template <int RPL>
__global__ void __launch_bounds__(32, (RPL == 1) ? 28 : 1)
scan_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
                   const double ru, const double rx, const double rc, const double *__restrict__ grid,
                   const int grid_shared, const int B, const int G, const double *__restrict__ sd_start,
                   const double *__restrict__ sd_end, const int flags, double *__restrict__ Kout,
                   double *__restrict__ sdout, double *__restrict__ uout, int *__restrict__ status,
                   int *__restrict__ fail_stage, int *__restrict__ counters, const int *__restrict__ glen,
                   const double *__restrict__ sd_end_hi /* last: the other parameters keep their offsets */) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  // glen (optional): ragged batches, as in scan_kernel; K / sd / u past this path's gridpoints are NaN
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int nC = R + 2;
  // The stage count lives in shared memory (one warp per CTA) and is re-read where it is used.  Held in a register
  // across the passes it raises the RPL 1 build's spills under its 72-register cap (-Xptxas -v: 192/368 bytes of spill
  // stores/loads with a compile-time G - 1, 264/608 with a register-held count, 152/224 like this).
  volatile __shared__ int s_n;
  if (lane == 0) s_n = Gp - 1;
  __syncwarp();
  const volatile int &N = s_n;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  double *Kp = Kout + (size_t)path * G * 2;
  const bool backward_only = (flags & 1) != 0;
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  // the padding is written up front: no pass below touches it, and the registers that hold Gp and the output pointers
  // are free here (written at the end, it adds spill traffic to the RPL 1 build)
  for (int j = 2 * Gp + lane; j < 2 * G; j += 32) Kp[j] = nan_d;
  if (!(flags & 3)) {
    for (int j = Gp + lane; j < G; j += 32) sdp[j] = nan_d;
    for (int j = N + lane; j < G - 1; j += 32) up[j] = nan_d;
  }
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
  const double sdeh = sd_end_hi ? sd_end_hi[path] : sde;   // K[N] = [sd_end^2, sd_end_hi^2]
  const double sds = sd_start ? sd_start[path] : 0.0;
  double kn0 = sde * sde, kn1 = sdeh * sdeh;
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
    for (int j = lane; j < Gp; j += 32) sdp[j] = nan_d;
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
        for (int j = i + 1 + lane; j < Gp; j += 32) sdp[j] = nan_d;
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
    for (int j = lane; j < Gp; j += 32) sdp[j] = sqrt(sdp[j]);
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

extern "C" int tb_scan_robust_ex(const double *records, int W, int R, int conic_row0, int conic_rows,
                                 const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                                 const int *glen, const double *sd_start, const double *sd_end, const double *sd_end_hi,
                                 int flags, double *K, double *sd, double *u, int *status, int *fail_stage, int *counters,
                                 void *stream) {
  using namespace tb;
  if (!records || !grid || !ellipsoid_host3 || !K || !status || B <= 0 || G <= 0 || R < 0) {
    set_error("tb_scan_robust: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tb_scan_robust: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  const bool backward_only = (flags & (TB_SCAN_BACKWARD_ONLY | TB_SCAN_FEASIBLE_SETS)) != 0;
  if (!backward_only && (!sd || (G > 1 && !u))) { set_error("tb_scan_robust: null output"); return TB_ERR_ARG; }
  if (R > MAX_ROWS) { set_error("tb_scan_robust: R=%d > %d rows", R, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2) { set_error("tb_scan_robust: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  if (conic_row0 < 0 || conic_rows < 0 || conic_row0 + conic_rows > R) { set_error("tb_scan_robust: bad conic row range"); return TB_ERR_ARG; }
  if (ellipsoid_host3[0] < 0 || ellipsoid_host3[1] < 0 || ellipsoid_host3[2] < 0) { set_error("tb_scan_robust: negative ellipsoid axis"); return TB_ERR_ARG; }
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(R + 2, [&](auto rpl) {
    scan_robust_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(records, W, R, conic_row0, conic_rows, ru, rx, rc,
                                                                      grid, grid_shared, B, G, sd_start, sd_end,
                                                                      flags, K, sd, u, status, fail_stage, counters,
                                                                      glen, sd_end_hi);
  });
  return check_launch("tb_scan_robust");
}

extern "C" int tb_scan_robust_ragged(const double *records, int W, int R, int conic_row0, int conic_rows,
                                     const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                                     const int *glen, const double *sd_start, const double *sd_end, int flags, double *K,
                                     double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream) {
  return tb_scan_robust_ex(records, W, R, conic_row0, conic_rows, ellipsoid_host3, grid, grid_shared, B, G, glen,
                           sd_start, sd_end, nullptr, flags, K, sd, u, status, fail_stage, counters, stream);
}

extern "C" int tb_scan_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                              const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                              const double *sd_start, const double *sd_end, int flags, double *K, double *sd, double *u,
                              int *status, int *fail_stage, int *counters, void *stream) {
  return tb_scan_robust_ex(records, W, R, conic_row0, conic_rows, ellipsoid_host3, grid, grid_shared, B, G, nullptr,
                           sd_start, sd_end, nullptr, flags, K, sd, u, status, fail_stage, counters, stream);
}
