// tb_conic.cu — libtoppra_b200_robust.so: the TOPPRAsd forward passes and single stage solves of robust (conic)
// problems.  C-ABI in include/toppra_b200_robust.h.
//
// The reference runs TOPPRAsd (desired_duration_algorithm.py:42-234) and solve_stagewise_optim on a conic problem
// through ecosWrapper.solve_stagewise_optim (ecos_solverwrapper.py:90-207).  Both solve the same two-variable stage
// problems as K2r (tb_robust.cu), with the primitives of tb_robust_common.cuh:
//   sd_forward_robust_kernel  the fastest and the slowest forward pass on the controllable sets K of a backward-only
//                             tb_scan_robust_ragged launch: at stage i x is fixed, so the stage problem is the
//                             u-interval at x, and the fastest pass takes u = uhi(x), the slowest u = ulo(x);
//   socp_stage_kernel         min g0 u + g1 x over one stage: the feasible x-interval by extreme_x, then the convex
//                             phi(x) = g1 x + g0 (g0 < 0 ? uhi(x) : ulo(x)) by golden-section search on it
//                             (socp_stage_solve, tb_robust_common.cuh).
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error).  Each library
// carries its own static CUDA runtime, so launch errors are read here (launch_status).
#include "tb_robust_kernels.cuh"
#include "../../include/toppra_b200_robust.h"

namespace tb {
namespace {

// One warp per (path, pass), one warp per CTA: blockIdx.x = 2 path + (0 fastest, 1 slowest).  The rules are those of
// desired_duration_algorithm.py:87-121 (the slowest pass :207-234), on the conventions of tb_scan_ex with
// TB_SCAN_SD_FORWARD: x out holds x = sd^2, status / fail_stage are the fastest pass's.  Body: sd_forward_robust_body
// (tb_robust_kernels.cuh) on one ellipsoid.
template <int RPL>
__global__ void __launch_bounds__(32)
sd_forward_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0,
                         const int conicn, const double ru, const double rx, const double rc,
                         const double *__restrict__ grid, const int grid_shared, const int B, const int G,
                         const int *__restrict__ glen, const double *__restrict__ K, const int *__restrict__ status_in,
                         const double *__restrict__ sd_start, double *__restrict__ x_fast, double *__restrict__ u_fast,
                         double *__restrict__ x_slow, double *__restrict__ u_slow, int *__restrict__ status,
                         int *__restrict__ fail_stage) {
  sd_forward_robust_body<RPL, false>(records, W, R, conic0, conicn, ru, rx, rc, grid, grid_shared, B, G, glen, K,
                                     status_in, sd_start, x_fast, u_fast, x_slow, u_slow, status, fail_stage, nullptr,
                                     false);
}

// One stage problem per warp (one warp per CTA): rows 0 / 1 are the optional x_next rows, rows 2.. the caller's n rows.
// Body: socp_stage_body (tb_robust_kernels.cuh) on one ellipsoid.
template <int RPL>
__global__ void __launch_bounds__(32)
socp_stage_kernel(const double *__restrict__ g, const double *__restrict__ ra, const double *__restrict__ rb,
                  const double *__restrict__ rcst, const int n, const int conic0, const int conicn, const double ru,
                  const double rx, const double rc, const double *__restrict__ xbox, const double *__restrict__ xnext,
                  const int B, double *__restrict__ out) {
  socp_stage_body<RPL, false>(g, ra, rb, rcst, n, conic0, conicn, ru, rx, rc, xbox, xnext, B, out, nullptr, nullptr);
}

}  // namespace
}  // namespace tb

extern "C" int tbr_version(void) { return TBR_VERSION; }

extern "C" int tbr_sd_forward_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                                     const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                                     const int *glen, const double *K, const int *status_in, const double *sd_start,
                                     double *x_fast, double *u_fast, double *x_slow, double *u_slow, int *status,
                                     int *fail_stage, void *stream) {
  using namespace tb;
  if (!records || !grid || !ellipsoid_host3 || !K || !status_in || !x_fast || !x_slow || !status || B <= 0 || G <= 0 ||
      R < 0 || (G > 1 && (!u_fast || !u_slow))) {
    set_error("tbr_sd_forward_robust: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tbr_sd_forward_robust: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (W < 3 * R + 2) { set_error("tbr_sd_forward_robust: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  if (const int rc = check_conic(R, conic_row0, conic_rows, ellipsoid_host3, "tbr_sd_forward_robust")) return rc;
  if (B > 0x3fffffff) { set_error("tbr_sd_forward_robust: batch too large for one launch"); return TB_ERR_UNSUPPORTED; }
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(R + 2, [&](auto rpl) {
    sd_forward_robust_kernel<rpl.value><<<2 * B, 32, 0, (cudaStream_t)stream>>>(
        records, W, R, conic_row0, conic_rows, ru, rx, rc, grid, grid_shared, B, G, glen, K, status_in, sd_start, x_fast,
        u_fast, x_slow, u_slow, status, fail_stage);
  });
  return launch_status("tbr_sd_forward_robust");
}

extern "C" int tbr_socp_stage_batch(const double *g, const double *a, const double *b, const double *c, int n,
                                    int conic_row0, int conic_rows, const double *ellipsoid_host3, const double *xbox,
                                    const double *xnext, int B, double *optvar, void *stream) {
  using namespace tb;
  if (!g || !ellipsoid_host3 || !xbox || !optvar || B <= 0 || n < 0 || (n > 0 && (!a || !b || !c))) {
    set_error("tbr_socp_stage_batch: bad argument");
    return TB_ERR_ARG;
  }
  if (const int rc = check_conic(n, conic_row0, conic_rows, ellipsoid_host3, "tbr_socp_stage_batch")) return rc;
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(n + 2, [&](auto rpl) {
    socp_stage_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(g, a, b, c, n, conic_row0, conic_rows, ru, rx, rc,
                                                                     xbox, xnext, B, optvar);
  });
  return launch_status("tbr_socp_stage_batch");
}
