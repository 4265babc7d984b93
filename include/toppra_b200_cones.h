/*
 * toppra_b200_cones.h — C-ABI of libtoppra_b200_cones.so: robust (conic) problems with any number of robust
 * constraints, each with its own ellipsoid, and with the u box of linear constraints that have a ubound.
 *
 * The reference solves such problems through ecosWrapper.solve_stagewise_optim
 * (toppra/solverwrapper/ecos_solverwrapper.py:56-79, 138-188).  Each entry is the counterpart of an entry for one robust
 * constraint, with the same conventions, output layouts and failure rules:
 *
 *   tbc_scan              <-> tb_scan_robust_ex (include/toppra_b200.h)
 *   tbc_sd_forward        <-> tbr_sd_forward_robust (include/toppra_b200_robust.h)
 *   tbc_socp_stage_batch  <-> tbr_socp_stage_batch (include/toppra_b200_robust.h), plus an optional u box
 *   tbc_reachable_sets    <-> tbr_reachable_sets_robust (include/toppra_b200_reach.h)
 *
 * The triple (conic_row0, conic_rows, ellipsoid_host3) of those entries becomes one HOST table cones_host [R][4]
 * (cones_host [n][4] for the stage solves): row k holds (robust flag 0 / 1, ru, rx, rc), and a robust row k reads
 *   a u + b x + c + ||diag(ru, rx, rc) [u, x, 1]||_2 <= 0,
 * a row with flag 0 is linear (its axes are not used).  A flag other than 0 or 1, or a negative or NaN axis, is
 * TB_ERR_ARG; R > 126 (n > 126) is TB_ERR_UNSUPPORTED.  Both are found before any CUDA call.
 *
 * flags may hold TB_SCAN_UBOUND: the records carry the u-bound pair (ulo, uhi) behind the x-bound pair (W >= 3R+4,
 * TB_ERR_ARG otherwise, as for tb_scan), and every stage also has ulo <= u <= uhi.  Without it the u box is
 * [-1e8, 1e8], where every u-interval starts.  The robust entries of the other libraries have no u box.
 *
 * Conventions are those of include/toppra_b200.h: device pointers (except cones_host), caller-owned memory,
 * asynchronous on `stream`, 0 / TB_ERR_* / cudaError_t returns, fp64 with -fmad=false.  This library links against
 * libtoppra_b200.so and reports errors through its tb_last_error().  It allocates nothing: the table travels as a kernel
 * parameter.
 */
#ifndef TOPPRA_B200_CONES_H_
#define TOPPRA_B200_CONES_H_

#ifdef __cplusplus
extern "C" {
#endif

#define TBC_VERSION 100

int tbc_version(void);

/* K2r on the cone table (tb_scan_robust_ex): backward and forward pass, or with TB_SCAN_BACKWARD_ONLY the backward pass
 * alone, or with TB_SCAN_FEASIBLE_SETS the feasible sets in K.  glen (nullable) [B]: ragged batches on per-path grids;
 * sd_end_hi (nullable) [B]: K[N] = [sd_end^2, sd_end_hi^2].  flags: those three bits only. */
int tbc_scan(const double *records, int W, int R, const double *cones_host, const double *grid, int grid_shared, int B,
             int G, const int *glen, const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags,
             double *K, double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream);

/* TOPPRAsd's fastest and slowest forward pass (tbr_sd_forward_robust) on K and status of a backward-only tbc_scan over
 * the same records and table.  flags: 0 or TB_SCAN_UBOUND. */
int tbc_sd_forward(const double *records, int W, int R, const double *cones_host, int flags, const double *grid,
                   int grid_shared, int B, int G, const int *glen, const double *K, const int *status_in,
                   const double *sd_start, double *x_fast, double *u_fast, double *x_slow, double *u_slow, int *status,
                   int *fail_stage, void *stream);

/* B stage problems (tbr_socp_stage_batch) over the rows a, b, c [B][n] with the table cones_host [n][4]; ubox (nullable)
 * [B][2]: ubox[p][0] <= u <= ubox[p][1] (NULL: [-1e8, 1e8]).  optvar [B][2] = (u, x), NaN NaN when infeasible. */
int tbc_socp_stage_batch(const double *g, const double *a, const double *b, const double *c, int n,
                         const double *cones_host, const double *xbox, const double *xnext, const double *ubox, int B,
                         double *optvar, void *stream);

/* Reachable sets (tbr_reachable_sets_robust) on the feasible sets X of a tbc_scan(..., TB_SCAN_FEASIBLE_SETS) launch
 * over the same records and table.  flags: 0 or TB_SCAN_UBOUND. */
int tbc_reachable_sets(const double *records, int W, int R, const double *cones_host, int flags, const double *grid,
                       int grid_shared, int B, int G, const int *glen, const double *X, const double *sdmin,
                       const double *sdmax, double *L, int *fail_stage, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* TOPPRA_B200_CONES_H_ */
