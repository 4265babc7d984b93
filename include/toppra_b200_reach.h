/*
 * toppra_b200_reach.h — C-ABI of libtoppra_b200_reach.so: the reachable sets of problems with one robust (conic)
 * constraint, the companion of tb_scan_robust_ragged in libtoppra_b200.so (include/toppra_b200.h), whose
 * TB_SCAN_FEASIBLE_SETS launch provides the feasible sets it starts from.
 *
 * The reference computes them in ReachabilityAlgorithm.compute_reachable_sets
 * (toppra/algorithm/reachabilitybased/reachability_algorithm.py:378-431) through ecosWrapper.solve_stagewise_optim
 * (toppra/solverwrapper/ecos_solverwrapper.py:90-207).  Rows and ellipsoid are those of tb_scan_robust; each stage
 * problem is solved by the method of tbr_socp_stage_batch (include/toppra_b200_robust.h).  The reference solves them with
 * ECOS (an interior-point solver): results agree with it to solver tolerance only; parity is unpinned, as for
 * tb_scan_robust (see DESIGN.md).
 *
 * Conventions are those of include/toppra_b200.h: device pointers (except ellipsoid_host3), caller-owned memory,
 * asynchronous on `stream`, 0 / TB_ERR_* / cudaError_t returns, fp64 with -fmad=false.  This library links against
 * libtoppra_b200.so and reports errors through its tb_last_error().
 */
#ifndef TOPPRA_B200_REACH_H_
#define TOPPRA_B200_REACH_H_

#ifdef __cplusplus
extern "C" {
#endif

#define TBR_REACH_VERSION 100

int tbr_reach_version(void);

/* Reachable sets L of B robust problems (compute_reachable_sets(sdmin, sdmax)), one warp per path.
 *   records, R, conic_row0, conic_rows, ellipsoid_host3, grid, grid_shared, glen: as tb_scan_robust_ragged;
 *   X [B][G][2]: the feasible sets of a tb_scan_robust_ragged(..., TB_SCAN_FEASIBLE_SETS) launch on the same records;
 *   sdmin, sdmax (nullable) [B]: sdmax NULL = sdmin, sdmin NULL = zeros.
 * Outputs, with the conventions of tb_reachable_sets[_ragged]:
 *   L [B][G][2], L[0] = [sdmin^2, sdmax^2]; the rows after the first row with a NaN end stay 0;
 *   fail_stage (nullable) [B]: index of the first NaN row of L, -1 if none.  Entries past a path's own end are NaN.
 * Stage i, with delta = grid[i+1] - grid[i] and delta' = deltas[i - 1] (deltas[N - 1] for i = 0, the reference's
 * negative index, kept as tb_reachable_sets keeps it):
 *   x box [max(L[i][0], xbound_lo), min(L[i][1], ECOS_MAXX, xbound_hi)];
 *   x_next rows X[i+1][0] <= x + 2 delta u <= X[i+1][1], a NaN end of X[i+1] being -/+ECOS_INFTY;
 *   L[i+1] = [x0 + 2 delta' u0, x1 + 2 delta' u1]: (u0, x0) minimises and (u1, x1) maximises x + 2 delta' u, each by the
 *   method of tbr_socp_stage_batch; the lower end is clamped at 0. */
int tbr_reachable_sets_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                              const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                              const int *glen, const double *X, const double *sdmin, const double *sdmax, double *L,
                              int *fail_stage, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* TOPPRA_B200_REACH_H_ */
