// tb_cones.cu — libtoppra_b200_cones.so: robust (conic) problems with several robust constraints, each with its own
// ellipsoid, and with a u box beside them.  C-ABI in include/toppra_b200_cones.h.
//
// The reference (ecosWrapper, ecos_solverwrapper.py:56-79, 138-188) accepts any number of CanonicalConic constraints,
// each with its own diag(ru, rx, rc), and adds ulo <= u <= uhi for every linear constraint with a ubound.  Its stage
// rows are those of K2r row by row:
//   a u + b x + c + ||diag(ru_k, rx_k, rc_k) [u, x, 1]||_2 <= 0     on the rows of robust constraint k,
// linear rows elsewhere, and the u box is the records' u-bound pair (TB_SCAN_UBOUND), the intersection over the
// constraints that seidelWrapper builds.  The four kernels below run the bodies of tb_robust_kernels.cuh with PER_ROW = true:
// each lane reads the flag and axes of its rows from the cone table once per path (load_cones).
// Their stage loops are those of tb_scan_robust_ex, tbr_sd_forward_robust, tbr_socp_stage_batch and
// tbr_reachable_sets_robust; with the table of one ellipsoid and no u box the results are bit-identical to theirs.
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error).  Each library
// carries its own static CUDA runtime, so launch errors are read here (launch_status).
#include "tb_robust_kernels.cuh"
#include "../../include/toppra_b200_cones.h"

namespace tb {
namespace {

// K2r on the cone table, one warp per CTA (scan_robust_body).  ub: the records carry a u-bound pair.
template <int RPL>
__global__ void __launch_bounds__(32)
tbc_scan_kernel(const double *__restrict__ records, const int W, const int R, const __grid_constant__ ConeTable cones,
                const int ub, const double *__restrict__ grid, const int grid_shared, const int B, const int G,
                const double *__restrict__ sd_start, const double *__restrict__ sd_end, const int flags,
                double *__restrict__ Kout, double *__restrict__ sdout, double *__restrict__ uout,
                int *__restrict__ status, int *__restrict__ fail_stage, int *__restrict__ counters,
                const int *__restrict__ glen, const double *__restrict__ sd_end_hi) {
  scan_robust_body<RPL, true>(records, W, R, 0, 0, Slots<RPL>{}, Slots<RPL>{}, Slots<RPL>{}, grid, grid_shared, B, G,
                              sd_start, sd_end, flags, Kout, sdout, uout, status, fail_stage, counters, glen, sd_end_hi,
                              &cones, ub != 0);
}

// TOPPRAsd's fastest and slowest forward pass on the cone table, one warp per (path, pass) (sd_forward_robust_body).
template <int RPL>
__global__ void __launch_bounds__(32)
tbc_sd_forward_kernel(const double *__restrict__ records, const int W, const int R,
                      const __grid_constant__ ConeTable cones, const int ub, const double *__restrict__ grid,
                      const int grid_shared, const int B, const int G, const int *__restrict__ glen,
                      const double *__restrict__ K, const int *__restrict__ status_in,
                      const double *__restrict__ sd_start, double *__restrict__ x_fast, double *__restrict__ u_fast,
                      double *__restrict__ x_slow, double *__restrict__ u_slow, int *__restrict__ status,
                      int *__restrict__ fail_stage) {
  sd_forward_robust_body<RPL, true>(records, W, R, 0, 0, Slots<RPL>{}, Slots<RPL>{}, Slots<RPL>{}, grid, grid_shared, B,
                                    G, glen, K, status_in, sd_start, x_fast, u_fast, x_slow, u_slow, status, fail_stage,
                                    &cones, ub != 0);
}

// One stage problem per warp on the cone table (socp_stage_body); ubox (nullable) [B][2] is each problem's u box.
template <int RPL>
__global__ void __launch_bounds__(32)
tbc_socp_stage_kernel(const double *__restrict__ g, const double *__restrict__ ra, const double *__restrict__ rb,
                      const double *__restrict__ rcst, const int n, const __grid_constant__ ConeTable cones,
                      const double *__restrict__ xbox, const double *__restrict__ xnext,
                      const double *__restrict__ ubox, const int B, double *__restrict__ out) {
  socp_stage_body<RPL, true>(g, ra, rb, rcst, n, 0, 0, Slots<RPL>{}, Slots<RPL>{}, Slots<RPL>{}, xbox, xnext, B, out,
                             &cones, ubox);
}

// compute_reachable_sets' forward recursion on the cone table, one warp per path (reachable_robust_body).
template <int RPL>
__global__ void __launch_bounds__(32)
tbc_reachable_kernel(const double *__restrict__ records, const int W, const int R,
                     const __grid_constant__ ConeTable cones, const int ub, const double *__restrict__ grid,
                     const int grid_shared, const int B, const int G, const int *__restrict__ glen,
                     const double *__restrict__ X, const double *__restrict__ sdmin, const double *__restrict__ sdmax,
                     double *__restrict__ Lout, int *__restrict__ fail_stage) {
  reachable_robust_body<RPL, true>(records, W, R, 0, 0, Slots<RPL>{}, Slots<RPL>{}, Slots<RPL>{}, grid, grid_shared, B,
                                   G, glen, X, sdmin, sdmax, Lout, fail_stage, &cones, ub != 0);
}

// The cone table of an entry: 0 and `t` filled (rows past R zero), or the TB_ERR_* code (message set).  Validated on the
// host before any CUDA call.
int cone_table(const int R, const double *cones_host, ConeTable &t, const char *what) {
  if (R > MAX_ROWS) { set_error("%s: R=%d > %d rows", what, R, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  for (int k = 0; k < MAX_ROWS; ++k)
    for (int j = 0; j < 4; ++j) t.v[k][j] = 0.0;
  for (int k = 0; k < R; ++k) {
    const double *row = cones_host + 4 * k;
    if (!(row[0] == 0.0 || row[0] == 1.0)) { set_error("%s: cone row %d: robust flag %g is not 0 or 1", what, k, row[0]); return TB_ERR_ARG; }
    for (int j = 1; j < 4; ++j)
      if (!(row[j] >= 0.0)) { set_error("%s: cone row %d: axis %d is negative or NaN", what, k, j - 1); return TB_ERR_ARG; }
    for (int j = 0; j < 4; ++j) t.v[k][j] = row[j];
  }
  return 0;
}

}  // namespace
}  // namespace tb

extern "C" int tbc_version(void) { return TBC_VERSION; }

extern "C" int tbc_scan(const double *records, int W, int R, const double *cones_host, const double *grid,
                        int grid_shared, int B, int G, const int *glen, const double *sd_start, const double *sd_end,
                        const double *sd_end_hi, int flags, double *K, double *sd, double *u, int *status,
                        int *fail_stage, int *counters, void *stream) {
  using namespace tb;
  if (!records || !grid || !cones_host || !K || !status || B <= 0 || G <= 0 || R < 0) {
    set_error("tbc_scan: bad argument");
    return TB_ERR_ARG;
  }
  ConeTable t;
  if (const int rc = cone_table(R, cones_host, t, "tbc_scan")) return rc;
  if (glen && grid_shared) { set_error("tbc_scan: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  const bool backward_only = (flags & (TB_SCAN_BACKWARD_ONLY | TB_SCAN_FEASIBLE_SETS)) != 0;
  if (!backward_only && (!sd || (G > 1 && !u))) { set_error("tbc_scan: null output"); return TB_ERR_ARG; }
  if (flags & ~(TB_SCAN_BACKWARD_ONLY | TB_SCAN_FEASIBLE_SETS | TB_SCAN_UBOUND)) { set_error("tbc_scan: unsupported flags %d", flags); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2) { set_error("tbc_scan: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  const int ub = (flags & TB_SCAN_UBOUND) ? 1 : 0;
  if (ub && W < 3 * R + 4) { set_error("tbc_scan: TB_SCAN_UBOUND needs records of W >= 3R+4 doubles"); return TB_ERR_ARG; }
  with_rows_per_lane(R + 2, [&](auto rpl) {
    tbc_scan_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(records, W, R, t, ub, grid, grid_shared, B, G,
                                                                   sd_start, sd_end, flags & ~TB_SCAN_UBOUND, K, sd, u,
                                                                   status, fail_stage, counters, glen, sd_end_hi);
  });
  return launch_status("tbc_scan");
}

extern "C" int tbc_sd_forward(const double *records, int W, int R, const double *cones_host, int flags,
                              const double *grid, int grid_shared, int B, int G, const int *glen, const double *K,
                              const int *status_in, const double *sd_start, double *x_fast, double *u_fast,
                              double *x_slow, double *u_slow, int *status, int *fail_stage, void *stream) {
  using namespace tb;
  if (!records || !grid || !cones_host || !K || !status_in || !x_fast || !x_slow || !status || B <= 0 || G <= 0 ||
      R < 0 || (G > 1 && (!u_fast || !u_slow))) {
    set_error("tbc_sd_forward: bad argument");
    return TB_ERR_ARG;
  }
  ConeTable t;
  if (const int rc = cone_table(R, cones_host, t, "tbc_sd_forward")) return rc;
  if (glen && grid_shared) { set_error("tbc_sd_forward: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (flags & ~TB_SCAN_UBOUND) { set_error("tbc_sd_forward: unsupported flags %d", flags); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2) { set_error("tbc_sd_forward: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  const int ub = (flags & TB_SCAN_UBOUND) ? 1 : 0;
  if (ub && W < 3 * R + 4) { set_error("tbc_sd_forward: TB_SCAN_UBOUND needs records of W >= 3R+4 doubles"); return TB_ERR_ARG; }
  if (B > 0x3fffffff) { set_error("tbc_sd_forward: batch too large for one launch"); return TB_ERR_UNSUPPORTED; }
  with_rows_per_lane(R + 2, [&](auto rpl) {
    tbc_sd_forward_kernel<rpl.value><<<2 * B, 32, 0, (cudaStream_t)stream>>>(
        records, W, R, t, ub, grid, grid_shared, B, G, glen, K, status_in, sd_start, x_fast, u_fast, x_slow, u_slow,
        status, fail_stage);
  });
  return launch_status("tbc_sd_forward");
}

extern "C" int tbc_socp_stage_batch(const double *g, const double *a, const double *b, const double *c, int n,
                                    const double *cones_host, const double *xbox, const double *xnext,
                                    const double *ubox, int B, double *optvar, void *stream) {
  using namespace tb;
  if (!g || !cones_host || !xbox || !optvar || B <= 0 || n < 0 || (n > 0 && (!a || !b || !c))) {
    set_error("tbc_socp_stage_batch: bad argument");
    return TB_ERR_ARG;
  }
  ConeTable t;
  if (const int rc = cone_table(n, cones_host, t, "tbc_socp_stage_batch")) return rc;
  with_rows_per_lane(n + 2, [&](auto rpl) {
    tbc_socp_stage_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(g, a, b, c, n, t, xbox, xnext, ubox, B,
                                                                         optvar);
  });
  return launch_status("tbc_socp_stage_batch");
}

extern "C" int tbc_reachable_sets(const double *records, int W, int R, const double *cones_host, int flags,
                                  const double *grid, int grid_shared, int B, int G, const int *glen, const double *X,
                                  const double *sdmin, const double *sdmax, double *L, int *fail_stage, void *stream) {
  using namespace tb;
  if (!records || !grid || !cones_host || !X || !L || B <= 0 || G <= 0 || R < 0) {
    set_error("tbc_reachable_sets: bad argument");
    return TB_ERR_ARG;
  }
  ConeTable t;
  if (const int rc = cone_table(R, cones_host, t, "tbc_reachable_sets")) return rc;
  if (glen && grid_shared) { set_error("tbc_reachable_sets: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (flags & ~TB_SCAN_UBOUND) { set_error("tbc_reachable_sets: unsupported flags %d", flags); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2) { set_error("tbc_reachable_sets: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  const int ub = (flags & TB_SCAN_UBOUND) ? 1 : 0;
  if (ub && W < 3 * R + 4) { set_error("tbc_reachable_sets: TB_SCAN_UBOUND needs records of W >= 3R+4 doubles"); return TB_ERR_ARG; }
  with_rows_per_lane(R + 2, [&](auto rpl) {
    tbc_reachable_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(records, W, R, t, ub, grid, grid_shared, B, G,
                                                                        glen, X, sdmin, sdmax, L, fail_stage);
  });
  return launch_status("tbc_reachable_sets");
}
