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
#include "tb_robust_common.cuh"
#include "../../include/toppra_b200_reach.h"

namespace tb {
namespace {

// compute_reachable_sets of a robust problem (reachability_algorithm.py:378-431), one warp per path: the forward
// recursion L[i+1] = _one_step_forward(i, L[i], X[i+1]) on the feasible sets X of a tb_scan_robust_ragged
// (TB_SCAN_FEASIBLE_SETS) launch.  Each end of L[i+1] is one socp_stage_solve: max / min x + 2 delta' u over stage i
// with L[i] in the x box and X[i+1] on the x_next rows (ecos_solverwrapper.py:90-207).  The reference's objective uses
// delta' = deltas[i - 1] (deltas[N - 1] at i = 0, Python's negative index) while the x_next rows use deltas[i], as in
// reachable_kernel (tb_scan.cu).  After a NaN end the remaining rows of L stay 0 (np.zeros).
template <int RPL>
__global__ void __launch_bounds__(32)
reachable_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0,
                        const int conicn, const double ru, const double rx, const double rc,
                        const double *__restrict__ grid, const int grid_shared, const int B, const int G,
                        const int *__restrict__ glen, const double *__restrict__ X, const double *__restrict__ sdmin,
                        const double *__restrict__ sdmax, double *__restrict__ Lout, int *__restrict__ fail_stage) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int N = Gp - 1, nC = R + 2;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  const double *Xp = X + (size_t)path * G * 2;
  double *Lp = Lout + (size_t)path * G * 2;
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  for (int j = 2 * Gp + lane; j < 2 * G; j += 32) Lp[j] = nan_d;   // ragged padding
  const double s0 = sdmin ? sdmin[path] : 0.0, s1 = sdmax ? sdmax[path] : s0;
  double l0 = s0 * s0, l1 = s1 * s1;
  for (int j = 2 * lane; j < 2 * Gp; j += 64) { Lp[j] = 0.0; Lp[j + 1] = 0.0; }
  __syncwarp();
  if (lane == 0) { Lp[0] = l0; Lp[1] = l1; }
  int fs = -1;
  double a[RPL], b[RPL], c[RPL];
  unsigned cmask[RPL];
  for (int i = 0; i < N; ++i) {
    const double *rec = rec_path + (size_t)i * W;
    rload_rows<RPL>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask);
    if (i + 2 < N && lane * 16 < W) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 2 * W + lane * 16));
    // x box: x_min / x_max = L[i] and the xbound rows x >= lo, x <= min(ECOS_MAXX, hi) (ecos_solverwrapper.py:110-172)
    const double xl = fmax(l0, rec[3 * R]), xh = fmin(l1, fmin(ECOS_MAXX, rec[3 * R + 1]));
    // x_next rows from X[i+1]: a NaN end is an absent bound, -/+ECOS_INFTY
    const double delta = gp[i + 1] - gp[i];
    double xn0 = Xp[2 * (i + 1)], xn1 = Xp[2 * (i + 1) + 1];
    xn0 = (xn0 == xn0) ? xn0 : -ECOS_INFTY;
    xn1 = (xn1 == xn1) ? xn1 : ECOS_INFTY;
    if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = xn0; }
    if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -xn1; }
    const double dq = (i > 0) ? (gp[i] - gp[i - 1]) : (gp[N] - gp[N - 1]);   // deltas[i - 1]
    double u1, x1v, u0, x0v;
    socp_stage_solve<RPL>(-2 * dq, -1.0, xl, xh, a, b, c, cmask, lane, ru, rx, rc, u1, x1v);
    socp_stage_solve<RPL>(2 * dq, 1.0, xl, xh, a, b, c, cmask, lane, ru, rx, rc, u0, x0v);
    const double x_upper = x1v + 2 * dq * u1;   // NaN when the stage is infeasible
    double x_lower = x0v + 2 * dq * u0;
    if (x_lower < 0) x_lower = 0;
    if (lane == 0) { Lp[2 * (i + 1)] = x_lower; Lp[2 * (i + 1) + 1] = x_upper; }
    if (!(x_lower == x_lower && x_upper == x_upper)) { fs = i + 1; break; }   // "Path not parametrizable"
    l0 = x_lower;
    l1 = x_upper;
  }
  if (lane == 0 && fail_stage) fail_stage[path] = fs;
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
