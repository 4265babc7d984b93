/*
 * toppra_b200_robust.h — C-ABI of libtoppra_b200_robust.so: TOPPRAsd and single stage solves for problems with one
 * robust (conic) constraint, the companions of tb_scan_robust[_ragged] in libtoppra_b200.so (include/toppra_b200.h).
 *
 * The reference runs these through ecosWrapper.solve_stagewise_optim (toppra/solverwrapper/ecos_solverwrapper.py:90-207):
 *
 *   tbr_sd_forward_robust <-> the two forward passes of TOPPRAsd.compute_parameterization
 *                             (toppra/algorithm/reachabilitybased/desired_duration_algorithm.py:42-121, 207-234)
 *   tbr_socp_stage_batch  <-> ecosWrapper.solve_stagewise_optim(i, None, g, x_min, x_max, x_next_min, x_next_max)
 *
 * Rows and ellipsoid are those of tb_scan_robust: rows [conic_row0, conic_row0 + conic_rows) are robust rows
 * a u + b x + c + ||diag(ru, rx, rc) [u, x, 1]||_2 <= 0 with ellipsoid_host3 = (ru, rx, rc) (HOST pointer, 3 doubles),
 * the other rows are linear.  The reference solves the stage problems with ECOS (an interior-point solver): results agree
 * with it to solver tolerance only; parity is unpinned, as for tb_scan_robust (see DESIGN.md).
 *
 * Conventions are those of include/toppra_b200.h: device pointers (except ellipsoid_host3), caller-owned memory,
 * asynchronous on `stream`, 0 / TB_ERR_* / cudaError_t returns, fp64 with -fmad=false.  This library links against
 * libtoppra_b200.so and reports errors through its tb_last_error().
 */
#ifndef TOPPRA_B200_ROBUST_H_
#define TOPPRA_B200_ROBUST_H_

#ifdef __cplusplus
extern "C" {
#endif

#define TBR_VERSION 100

int tbr_version(void);

/* The fastest and the slowest TOPPRAsd forward pass of B robust problems in one launch, one warp per (path, pass).
 *   records [B][G][W], R, conic_row0, conic_rows, ellipsoid_host3, grid [G] (grid_shared = 1) or [B][G], glen (nullable,
 *   ragged batches, needs grid_shared = 0): as tb_scan_robust_ragged;
 *   K [B][G][2], status_in [B]: controllable sets and status of a tb_scan_robust_ragged(..., TB_SCAN_BACKWARD_ONLY)
 *   launch on the same records (K[N] = sd_end^2), so the conic backward pass runs once for both passes;
 *   sd_start (nullable = zeros) [B].
 * Outputs, with the layout and conventions of tb_scan_ex(TB_SCAN_SD_FORWARD [| TB_SCAN_SD_SLOW]):
 *   x_fast, x_slow [B][G]: x = sd^2 of the two passes; u_fast, u_slow [B][G-1] (may be NULL when G = 1);
 *   status [B], fail_stage (nullable) [B]: those of the fastest pass.  A failure of the slowest pass shows as NaN in
 *   x_slow / u_slow, which tb_sd_bisect turns into ErrUnknown.
 * Rules (desired_duration_algorithm.py:83-121):
 *   status_in != Ok: status_in is kept, fail_stage is the last row of K with a NaN end, x / u are NaN;
 *   x0 = sd_start^2 with x0 + 1e-5 < K[0][0] or K[0][1] + 1e-5 < x0: FailUncontrollable, fail_stage 0, x / u NaN;
 *   stage i: x = x[i] is fixed, the rows are the stage's linear and cone rows plus K[i+1][0] <= x + 2 delta u <= K[i+1][1];
 *   the fastest pass takes u = uhi(x), the slowest u = ulo(x) (the ends of the feasible u-interval); no retry rule;
 *   x[i+1] = min(K[i+1][1], max(K[i+1][0], x + 2 delta u - 1e-5));
 *   an empty u-interval: ErrUnknown, fail_stage i, u[i:] and x[i+1:] NaN.
 *   The x box (xbound, -/+1000) is not checked at a forward stage, as in the forward step of tb_scan_robust: x comes
 *   from K[i] (x[0] from the start check), which lies in the box up to the 1e-5 of these rules.
 *   Entries at and past a path's own end (glen) are NaN. */
int tbr_sd_forward_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                          const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                          const int *glen, const double *K, const int *status_in, const double *sd_start, double *x_fast,
                          double *u_fast, double *x_slow, double *u_slow, int *status, int *fail_stage, void *stream);

/* B independent stage problems, one warp each — the conic counterpart of tb_lp2d_batch:
 *   minimise g0 u + g1 x  s.t.  a u + b x + c (+ ||diag(ru, rx, rc) [u, x, 1]||_2) <= 0 (n rows, robust on
 *   [conic_row0, conic_row0 + conic_rows)),  xbox[0] <= x <= xbox[1],
 *   and, when xnext is given and its delta is not NaN, xnext[1] <= x + 2 delta u <= xnext[2].
 *   g [B][2]; a, b, c [B][n] (n <= 126); xbox [B][2]; xnext (nullable) [B][3] = (delta, x_next_lo, x_next_hi).
 *   The bounds are final: the caller fills absent ones (ECOS_INFTY = 1000) and caps xbox[1] at ECOS_MAXX = 1e4, as
 *   ecos_solverwrapper.py:110-172 does.
 *   optvar out [B][2] = (u, x), NaN NaN when infeasible.
 * Method: the feasible x-interval [xmin, xmax] (the bracketed search of tb_scan_robust); g0 == 0: x = xmax if g1 < 0 else
 * xmin, u = the middle of the u-interval there (which u of that face ECOS returns is solver-dependent); g0 != 0: the
 * convex phi(x) = g1 x + g0 u*(x), u*(x) = uhi(x) (g0 < 0) or ulo(x) (g0 > 0), minimised by golden-section search down to
 * a bracket of a few ulps, ends included. */
int tbr_socp_stage_batch(const double *g, const double *a, const double *b, const double *c, int n, int conic_row0,
                         int conic_rows, const double *ellipsoid_host3, const double *xbox, const double *xnext, int B,
                         double *optvar, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* TOPPRA_B200_ROBUST_H_ */
