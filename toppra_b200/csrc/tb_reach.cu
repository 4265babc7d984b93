// tb_reach.cu — libtoppra_b200_reach.so: the reachable sets of robust (conic) problems.  C-ABI in
// include/toppra_b200_reach.h.
//
// The reference computes compute_reachable_sets (reachability_algorithm.py:378-431) of a conic problem through
// ecosWrapper.solve_stagewise_optim (ecos_solverwrapper.py:90-207).  reachable_robust_kernel solves the same stage
// problems with the primitives of tb_robust_common.cuh, two socp_stage_solve problems per stage; its input, the feasible
// sets X, comes from a tb_scan_robust_ragged (TB_SCAN_FEASIBLE_SETS) launch of libtoppra_b200.so.
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error).  Each library
// carries its own static CUDA runtime, so launch errors are read here (launch_status).
#include "tb_robust_kernels.cuh"
#include "../../include/toppra_b200_reach.h"

namespace tb {
namespace {

// compute_reachable_sets of a robust problem (reachability_algorithm.py:378-431), one warp per path: the forward
// recursion L[i+1] = _one_step_forward(i, L[i], X[i+1]) on the feasible sets X of a tb_scan_robust_ragged
// (TB_SCAN_FEASIBLE_SETS) launch.  Body: reachable_robust_body (tb_robust_kernels.cuh) on one ellipsoid.
template <int RPL>
__global__ void __launch_bounds__(32)
reachable_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0,
                        const int conicn, const double ru, const double rx, const double rc,
                        const double *__restrict__ grid, const int grid_shared, const int B, const int G,
                        const int *__restrict__ glen, const double *__restrict__ X, const double *__restrict__ sdmin,
                        const double *__restrict__ sdmax, double *__restrict__ Lout, int *__restrict__ fail_stage) {
  reachable_robust_body<RPL, false>(records, W, R, conic0, conicn, ru, rx, rc, grid, grid_shared, B, G, glen, X, sdmin,
                                    sdmax, Lout, fail_stage, nullptr, false);
}

}  // namespace
}  // namespace tb

extern "C" int tbr_reach_version(void) { return TBR_REACH_VERSION; }

extern "C" int tbr_reachable_sets_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                                         const double *ellipsoid_host3, const double *grid, int grid_shared, int B,
                                         int G, const int *glen, const double *X, const double *sdmin,
                                         const double *sdmax, double *L, int *fail_stage, void *stream) {
  using namespace tb;
  if (!records || !grid || !ellipsoid_host3 || !X || !L || B <= 0 || G <= 0 || R < 0) {
    set_error("tbr_reachable_sets_robust: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tbr_reachable_sets_robust: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (W < 3 * R + 2) { set_error("tbr_reachable_sets_robust: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  if (const int rc = check_conic(R, conic_row0, conic_rows, ellipsoid_host3, "tbr_reachable_sets_robust")) return rc;
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(R + 2, [&](auto rpl) {
    reachable_robust_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(
        records, W, R, conic_row0, conic_rows, ru, rx, rc, grid, grid_shared, B, G, glen, X, sdmin, sdmax, L,
        fail_stage);
  });
  return launch_status("tbr_reachable_sets_robust");
}
