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
#include "tb_robust_kernels.cuh"

namespace tb {
namespace {

// One warp per CTA, like the record scan: a finished path frees its slot at once.  The body is scan_robust_body
// (tb_robust_kernels.cuh) on one ellipsoid.
template <int RPL>
__global__ void __launch_bounds__(32, (RPL == 1) ? 28 : 1)
scan_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
                   const double ru, const double rx, const double rc, const double *__restrict__ grid,
                   const int grid_shared, const int B, const int G, const double *__restrict__ sd_start,
                   const double *__restrict__ sd_end, const int flags, double *__restrict__ Kout,
                   double *__restrict__ sdout, double *__restrict__ uout, int *__restrict__ status,
                   int *__restrict__ fail_stage, int *__restrict__ counters, const int *__restrict__ glen,
                   const double *__restrict__ sd_end_hi /* last: the other parameters keep their offsets */) {
  scan_robust_body<RPL, false>(records, W, R, conic0, conicn, ru, rx, rc, grid, grid_shared, B, G, sd_start, sd_end,
                               flags, Kout, sdout, uout, status, fail_stage, counters, glen, sd_end_hi, nullptr, false);
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
