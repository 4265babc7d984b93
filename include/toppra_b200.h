/*
 * toppra_b200.h — C-ABI of libtoppra_b200.so: batched TOPP-RA (time-optimal path
 * parameterisation by reachability analysis) on NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for the hot path of hungpham2511/toppra v0.6.2
 * (paths below are relative to the reference tree):
 *
 *   tb_spline_fit        <-> SplineInterpolator.__init__            toppra/interpolator.py:385-421 (scipy CubicSpline)
 *   tb_ppoly_eval        <-> SplineInterpolator.__call__(s, order)  toppra/interpolator.py:423-430 (scipy PPoly)
 *   tb_coeff_velacc      <-> JointVelocityConstraint.compute_constraint_params      toppra/constraint/linear_joint_velocity.py:43-53
 *                            + _create_velocity_constraint                          toppra/_CythonUtils.pyx:16-59
 *                            + JointAccelerationConstraint.compute_constraint_params toppra/constraint/linear_joint_acceleration.py:63-104
 *                            + canlinear_colloc_to_interpolate                      toppra/constraint/linear_constraint.py:84-192
 *                            + seidelWrapper.__init__ row assembly                  toppra/solverwrapper/cy_seidel_solverwrapper.pyx:425-531
 *   tb_rows_canlinear    <-> the same row assembly for a generic CanonicalLinear constraint
 *                            (a, b, c, F, g), e.g. SecondOrderConstraint            toppra/constraint/linear_second_order.py:142-173
 *   tb_scan              <-> ReachabilityAlgorithm.compute_parameterization         toppra/algorithm/reachabilitybased/reachability_algorithm.py:240-376
 *                            = compute_controllable_sets (:166-238) + forward pass (TOPPRA._forward_step,
 *                            time_optimal_algorithm.py:55-92), every stage LP solved like
 *                            seidelWrapper.solve_stagewise_optim (cy_seidel_solverwrapper.pyx:549-697,
 *                            cy_solve_lp2d :149-390, cy_solve_lp1d :93-144)
 *   tb_feasible_sets     <-> ReachabilityAlgorithm.compute_feasible_sets            reachability_algorithm.py:131-164
 *   tb_solve_velacc_host <-> the whole `TOPPRA([vel, acc], SplineInterpolator(ss, wp), gridpoints,
 *                            solver_wrapper="seidel").compute_parameterization(sd_start, sd_end)` for a batch of
 *                            paths with HOST buffers (copies included).
 *
 * Conventions
 *   - C linkage, plain pointers and sizes, no C++/torch types, no exceptions cross the boundary.
 *   - Every function returns 0 on success, a negative TB_ERR_* for argument errors, or a positive
 *     cudaError_t value; tb_last_error() returns a thread-local message.
 *   - Unless a name ends in _host, every pointer is a DEVICE pointer owned by the caller
 *     (e.g. torch.Tensor.data_ptr()); nothing is allocated or freed inside; `stream` is a
 *     cudaStream_t passed as void* (NULL = default stream); calls are asynchronous.
 *   - All reals are IEEE fp64; arithmetic order follows the reference so that results are
 *     bit-identical to its Cython seidelWrapper (kernels are compiled with -fmad=false).
 *   - "shared" flags: 1 = one array shared by all B paths, 0 = one array per path ([B][...]).
 *
 * Stage record layout (one per path and gridpoint, `W` doubles, W even so that W*8 % 16 == 0):
 *      rec[0      .. R)   a-coefficients of the R static LP rows  (u multiplier)
 *      rec[R      .. 2R)  b-coefficients                          (x multiplier)
 *      rec[2R     .. 3R)  c-coefficients
 *      rec[3R], rec[3R+1] x lower / upper bound: the constraints' xbound INTERSECTED with the solver box [-1e8, 1e8]
 *                         (seidelWrapper low/high, pyx:477-478,517-520; +-1e8 when absent) - the producers below
 *                         clip, tb_scan does not
 *      rec[3R+2 .. W)     padding (R odd only)
 *   i.e. row r is  a*u + b*x + c <= 0, exactly a_arr/b_arr/c_arr[i, 2+r] of the reference's
 *   seidelWrapper; rows 0,1 of the reference (the x_next rows it rewrites per call) are synthesised
 *   inside tb_scan.
 */
#ifndef TOPPRA_B200_H_
#define TOPPRA_B200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB_VERSION 100

/* argument errors */
#define TB_ERR_ARG (-1)          /* null pointer / non-positive size */
#define TB_ERR_UNSUPPORTED (-2)  /* size outside the compiled limits (see tb_limits) */
#define TB_ERR_ALIGN (-3)        /* pointer or record stride not 16-byte aligned */

/* per-path status written by tb_scan; values follow the order of the reference enum
 * ParameterizationReturnCode (toppra/algorithm/algorithm.py:49-56) */
#define TB_STATUS_OK 0
#define TB_STATUS_ERR_UNKNOWN 1          /* NaN in the forward pass (retry budget exhausted) */
#define TB_STATUS_ERR_SHORT_PATH 2       /* (unused by this path, kept for code parity) */
#define TB_STATUS_FAIL_UNCONTROLLABLE 3  /* NaN in K, or sd_start^2 outside K[0] +- 1e-5 */
#define TB_STATUS_ERR_FORWARD_PASS_FAIL 4

/* boundary-condition kinds of tb_spline_fit (scipy CubicSpline bc_type) */
#define TB_BC_NOT_A_KNOT 0
#define TB_BC_FIRST_DERIV 1   /* 'clamped' = first derivative 0 */
#define TB_BC_SECOND_DERIV 2  /* 'natural' = second derivative 0 */
#define TB_BC_PERIODIC 3      /* both ends; the caller guarantees wp[.][0] == wp[.][n-1] (scipy checks allclose 1e-15) */

int tb_version(void);
const char *tb_last_error(void);

/* Compiled limits: max_rows = largest R (static LP rows per stage), max_knots = largest n of tb_spline_fit. */
int tb_limits(int *max_rows, int *max_knots);

/* Record stride in doubles for R static rows: 3R+2 rounded up to even. */
int tb_record_doubles(int R);

/* K0 — not-a-knot / clamped / natural / periodic cubic spline through wp[B][n][dof] at ss.
 *   ss: [n] (ss_shared=1) or [B][n]; bc0/bc1: boundary values [B][dof] or NULL (= zeros);
 *   ppoly out: [B][4][n-1][dof] (scipy PPoly.c layout per path, highest power first);
 *   workspace: device scratch of tb_spline_fit_workspace_doubles(B, n, dof) doubles (0 for short splines:
 *   NULL allowed then). */
int tb_spline_fit_workspace_doubles(int B, int n, int dof);
int tb_spline_fit(const double *ss, int ss_shared, const double *wp, int B, int n, int dof, int bc0_kind,
                  const double *bc0, int bc1_kind, const double *bc1, double *ppoly, double *workspace, void *stream);

/* path(s, order), order in {0,1,2}.  breaks: [nseg+1] or [B][nseg+1]; s: [G] or [B][G];
 *   out: [B][G][dof]. */
int tb_ppoly_eval(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                  const double *s, int s_shared, int G, int order, double *out, void *stream);

/* K1 — stage records for JointVelocityConstraint (vlim, may be NULL) + JointAccelerationConstraint (alim).
 *   vlim/alim: [dof][2] (lim_shared=1) or [B][dof][2], (lower, upper);
 *   interp: 1 = DiscretizationType.Interpolation (R = 4*dof), 0 = Collocation (R = 2*dof);
 *   records out: [B][G][W] with the accel rows at row offset `row0` of R_total rows
 *   (row0=0, R_total=R for vel+acc only; other constraints append with tb_rows_canlinear);
 *   write_xbound: 0 = leave the xbound slots alone; 1 = overwrite them with the velocity bound intersected
 *   with [-1e8, 1e8] (the seidelWrapper low/high init, pyx:477-478,517-520), or +-1e8 when vlim==NULL;
 *   2 = overwrite with the raw xbound of compute_constraint_params (no clipping);
 *   3 = intersect with what the slots already hold (several velocity constraints). */
int tb_coeff_velacc(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                    const double *grid, int grid_shared, int G, const double *vlim, const double *alim,
                    int lim_shared, int interp, double *records, int W, int R_total, int row0, int write_xbound,
                    void *stream);

/* JointVelocityConstraintVarying (toppra/constraint/linear_joint_velocity.py:56-87): velocity limits per gridpoint,
 * vlim_grid [G][dof][2] (vlim_shared=1) or [B][G][dof][2]; write_xbound 1/2/3 as in tb_coeff_velacc. */
int tb_xbound_varying(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                      const double *grid, int grid_shared, int G, const double *vlim_grid, int vlim_shared,
                      double *records, int W, int R_total, int write_xbound, void *stream);

/* JointVelocityConstraint alone (linear_joint_velocity.py:43-53, _CythonUtils.pyx:16-59): the velocity bound of every
 * gridpoint into the xbound slots, one thread per (path, gridpoint), no acceleration rows.  vlim [dof][2] (lim_shared=1)
 * or [B][dof][2]; write_xbound 1/2/3 as in tb_coeff_velacc.  With W = 2, R_total = 0 the output is the plain
 * xbound [B][G][2] array that tb_scan_velacc reads. */
int tb_xbound_velocity(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                       const double *grid, int grid_shared, int G, const double *vlim, int lim_shared, double *records,
                       int W, int R_total, int write_xbound, void *stream);

/* Row assembly for a generic CanonicalLinear constraint given its collocation parameters:
 *   a, b, c: [B][G][m];  F: [k][m] (F_mode=0, identical) or [B][G][k][m] (F_mode=1);
 *   g: [k] / [B][G][k];  F_mode=2: F = [I; -I] (k = 2m) with g: [k] shared (torque-limit form);
 *   F_mode=3: same with g per path [B][k];
 *   interp: 1 = lift with canlinear_colloc_to_interpolate (2k rows), 0 = k rows.
 *   Writes rows [row0, row0 + (interp?2k:k)) of every record. */
int tb_rows_canlinear(const double *a, const double *b, const double *c, const double *F, const double *g, int F_mode,
                      int B, int G, int m, int k, const double *grid, int grid_shared, int interp, double *records,
                      int W, int R_total, int row0, void *stream);

/* SecondOrderConstraint on device (toppra/constraint/linear_second_order.py:114-173, BASELINE cfg 3): the reference
 * calls a user Python inv_dyn 3 (N+1) times per path; here the inverse dynamics is a DEVICE MODEL from a small
 * registry, evaluated from the spline by one thread per (path, gridpoint), and the joint-torque rows
 * (F = [I; -I], g = [tau_max; -tau_min], + sign(q') * friction, Interpolation lift) go straight into the records.
 *   model / params (device pointer, nparams doubles):
 *     TB_INVDYN_COUPLED_COSINE  tau_i = p0 qdd_i + p1 sum_j cos(q_i - q_j) qdd_j + p2 sin(q_i) |qd|^2 + p3 sin(q_i)   (4)
 *     TB_INVDYN_PENDULUMS       tau_i = p[2i] qdd_i + p[2i+1] sin(q_i)                                               (2 dof)
 *   taulim [dof][2] (lim_shared=1) or [B][dof][2]; friction [dof] or NULL; writes rows [row0, row0 + (interp?4:2)*dof).
 *   Models outside the registry use the host/tensor callback + tb_rows_canlinear.  fp64, not bit-identical to a numpy
 *   inv_dyn (libm sin/cos, BLAS dot order): parity tolerance 1e-9 relative on K / sd (SURVEY.md section 8d). */
#define TB_INVDYN_COUPLED_COSINE 0
#define TB_INVDYN_PENDULUMS 1
int tb_coeff_second_order(int model, const double *params, int nparams, const double *ppoly, const double *breaks,
                          int breaks_shared, int B, int nseg, int dof, const double *grid, int grid_shared, int G,
                          const double *taulim, int lim_shared, const double *friction, int interp, double *records, int W,
                          int R_total, int row0, void *stream);

/* Fill the xbound slots of every record with the defaults (-1e8, +1e8) (no velocity constraint). */
int tb_init_bounds(double *records, int B, int G, int W, int R_total, void *stream);

/* K2 — backward controllable sets + forward parameterisation, one warp per path.
 *   records: [B][G][W]; grid: [G] or [B][G]; sd_start, sd_end: [B] (NULL = zeros);
 *   K out: [B][G][2]; sd out: [B][G]; u out: [B][G-1]; status out: [B] (TB_STATUS_*);
 *   fail_stage out (nullable): [B], stage index where the pass failed, -1 if Ok. */
int tb_scan(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
            const double *sd_start, const double *sd_end, double *K, double *sd, double *u, int *status,
            int *fail_stage, void *stream);

/* K2r — the same passes for a problem with ONE robustified constraint (RobustLinearConstraint,
 * toppra/constraint/conic_constraint.py:47-124): rows [conic_row0, conic_row0 + conic_rows) of every record are
 * robust rows  a u + b x + c + ||diag(ru, rx, rc) [u, x, 1]||_2 <= 0  with the ellipsoid axes
 * ellipsoid_host3 = (ru, rx, rc) (HOST pointer, 3 doubles); the other rows are linear.  Stage problems follow
 * ecosWrapper.solve_stagewise_optim (toppra/solverwrapper/ecos_solverwrapper.py:90-207): absent x / x_next bounds are
 * -/+1000, x <= min(1e4, xbound_hi).  The reference solves them with ECOS (third party, interior point): results
 * agree with it only to solver tolerance — parity for this entry is unpinned (see DESIGN.md).
 * flags / outputs as tb_scan_ex; counters[.][0] = evaluations of the feasible-u interval, [3] = forward retries. */
int tb_scan_robust(const double *records, int W, int R, int conic_row0, int conic_rows, const double *ellipsoid_host3,
                   const double *grid, int grid_shared, int B, int G, const double *sd_start, const double *sd_end,
                   int flags, double *K, double *sd, double *u, int *status, int *fail_stage, int *counters,
                   void *stream);

/* Feasible sets X[B][G][2] (compute_feasible_sets, reachability_algorithm.py:131-164).
 * tb_feasible_sets_ex: flags = TB_SCAN_UBOUND for records that carry a u-bound pair (see tb_scan_ex). */
int tb_feasible_sets(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                     double *X, void *stream);
int tb_feasible_sets_ex(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                        int flags, double *X, void *stream);

/* Reachable sets (compute_reachable_sets(sdmin, sdmax), reachability_algorithm.py:378-431) of B paths in one launch:
 * the feasible-set pass followed by the forward recursion L[i+1] = _one_step_forward(i, L[i], X[i+1]) — one kernel
 * because the reference's solver wrapper carries its warm-start slots from the first pass into the second.
 *   sdmin, sdmax: [B] (sdmax NULL = sdmin; sdmin NULL = zeros);  X out, L out: [B][G][2];
 *   L rows after a failed stage stay 0 like the reference's np.zeros; fail_stage (nullable) [B]: index of the first
 *   NaN row of L, -1 if none.  flags: 0 or TB_SCAN_UBOUND. */
int tb_reachable_sets(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                      const double *sdmin, const double *sdmax, int flags, double *X, double *L, int *fail_stage,
                      void *stream);

/* Extended K2 entry:
 *   sd_end_hi (nullable): [B] upper terminal velocity, K[N] = [sd_end^2, sd_end_hi^2]
 *                         (compute_controllable_sets(sdmin, sdmax), reachability_algorithm.py:166-202);
 *   flags: TB_SCAN_BACKWARD_ONLY = stop after the backward pass (K and status only; sd/u may be NULL);
 *   counters (nullable): device [B][4] int32 = (2-D LP solves, 1-D LP solves, projected re-solves,
 *                        forward retries) — instrumentation for profiling. */
#define TB_SCAN_BACKWARD_ONLY 1
#define TB_SCAN_SD_FORWARD 4     /* forward-pass rules of TOPPRAsd (desired_duration_algorithm.py:103-121): no retry, x_next - 1e-5; the sd output then holds x = sd^2 */
#define TB_SCAN_SD_SLOW 8        /* with TB_SCAN_SD_FORWARD: the slowest pass (minimise the next velocity), :218-223 */
#define TB_SCAN_FORWARD_ONLY 16  /* forward pass alone: K, status (and fail_stage) hold the results of an earlier
                                   TB_SCAN_BACKWARD_ONLY launch on the same buffers (lets the D2H copy of K overlap) */
#define TB_SCAN_FAST_LOWER 32   /* OPT-IN, not bit-identical: K[i][0] = xbound_lo whenever some u is feasible there (the exact LP
                                   optimum) instead of replaying the reference's ~4 Seidel re-solves, whose projection
                                   arithmetic returns xbound_lo +- ~1e-16; falls back to the Seidel LP otherwise.
                                   Deviation from the reference: <= ~1e-15 on K and sd (tests: 1e-12). */
#define TB_SCAN_FEASIBLE_SETS 2 /* tb_scan_robust only: K receives the feasible sets X (compute_feasible_sets) */
#define TB_SCAN_UBOUND 64       /* the records carry a u-bound pair behind the x-bound pair: record = a[R] | b[R] | c[R] | xlo |
                                   xhi | ulo | uhi (W >= 3R+4): `ubound` of a constraint intersected into low/high[:, 0]
                                   (seidelWrapper.__init__, cy_seidel_solverwrapper.pyx:512-515).  Not with TB_SCAN_FAST_LOWER. */
int tb_scan_ex(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
               const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K, double *sd,
               double *u, int *status, int *fail_stage, int *counters, void *stream);

/* Ragged batches (per-path gridpoint counts, e.g. from tb_propose_gridpoints): grid is [B][G] (grid_shared = 0) padded to
 * the longest path, glen [B] (device int32, nullable = all G) holds each path's count 1 <= glen[p] <= G.  Strides stay G;
 * K / sd / u entries at and past a path's own end are NaN.  Everything else as tb_scan_ex / tb_scan_velacc. */
int tb_scan_ragged(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                   const int *glen, const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags,
                   double *K, double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream);
int tb_scan_velacc_ragged(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof,
                          const double *grid, int grid_shared, int B, int G, const int *glen, const double *alim,
                          int lim_shared, int interp, const double *xbound, const double *sd_start, const double *sd_end,
                          const double *sd_end_hi, int flags, double *K, double *sd, double *u, int *status,
                          int *fail_stage, int *counters, void *stream);
/* The other per-path solves on ragged batches, with the same glen convention (nullable; glen with grid_shared = 1 is
 * TB_ERR_ARG).  Each path reads only its own glen[p] gridpoints and records; every output entry at or past its own end
 * is NaN (X, L, K: rows >= glen[p]; sd: >= glen[p]; u / sdd: >= glen[p] - 1).  Everything else as the entry without the
 * suffix:
 *   tb_feasible_sets_ragged   = tb_feasible_sets_ex;
 *   tb_reachable_sets_ragged  = tb_reachable_sets (L is 0 up to glen[p] after a failed stage, as there);
 *   tb_scan_robust_ragged     = tb_scan_robust (also with TB_SCAN_FEASIBLE_SETS);
 *   tb_sd_bisect_ragged       = tb_sd_bisect: the durations sum each path's own glen[p] - 1 stages. */
int tb_feasible_sets_ragged(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                            const int *glen, int flags, double *X, void *stream);
int tb_reachable_sets_ragged(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                             const int *glen, const double *sdmin, const double *sdmax, int flags, double *X, double *L,
                             int *fail_stage, void *stream);
int tb_scan_robust_ragged(const double *records, int W, int R, int conic_row0, int conic_rows,
                          const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                          const int *glen, const double *sd_start, const double *sd_end, int flags, double *K,
                          double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream);
int tb_sd_bisect_ragged(const double *x_fast, const double *u_fast, const double *x_slow, const double *u_slow,
                        const double *grid, int grid_shared, int B, int G, const int *glen,
                        const double *desired_duration, double atol, int max_iter, const int *status_in, double *sd,
                        double *sdd, double *info, int *status, void *stream);

/* K2 fused with K1 for the JointVelocity + JointAcceleration problem (the headline case): no stage records at all.
 * Every lane of the path's warp builds its own LP row in the stage prologue from the spline (same arithmetic as
 * tb_coeff_velacc, so the rows are bit-identical to the materialised records); only the velocity bound comes from
 * memory:  xbound [B][G][2] = tb_coeff_velacc(..., alim = NULL, records = xbound, W = 2, R_total = 0, row0 = 0,
 * write_xbound = 1).  Same passes, flags and outputs as tb_scan_ex.  Returns TB_ERR_UNSUPPORTED when the problem does
 * not fit one row per lane ((interp ? 4 : 2) * dof + 2 > 32) or the spline has too many segments; the caller then
 * uses tb_coeff_velacc + tb_scan.  Replaces the same reference functions as tb_coeff_velacc + tb_scan. */
int tb_scan_velacc(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof, const double *grid,
                   int grid_shared, int B, int G, const double *alim, int lim_shared, int interp, const double *xbound,
                   const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                   double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream);

/* propose_gridpoints (toppra/interpolator.py:49-122) for B paths, one warp per path: adaptive bisection of the path
 * interval until every segment is at most max_seg_length long and its estimated interpolation error
 * 0.5 max_k |q_k''(mid)| len^2 is at most max_err_threshold, then doubling up to min_nb_points.  The grids are RAGGED:
 *   grid_out [B][Gmax] (tail padded with the path end), glen out [B] = gridpoints per path, scratch [B][Gmax];
 *   status out [B]: 0 ok, 1 = the reference would raise "Unable to find a good gridpoint for this path"
 *   (max_iteration passes used up), TB_ERR_UNSUPPORTED = more than Gmax points needed.
 * Feed grid_out / glen to tb_scan_ragged / tb_scan_velacc_ragged. */
int tb_propose_gridpoints(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                          double max_err_threshold, int max_iteration, double max_seg_length, int min_nb_points,
                          int Gmax, double *grid_out, double *scratch, int *glen, int *status, void *stream);

/* TOPPRAsd (desired_duration_algorithm.py:139-191): bisection on alpha so that the blend alpha * fastest +
 * (1 - alpha) * slowest parameterisation has the desired duration (_compute_duration :10-17, running sum in stage order).
 *   x_fast / x_slow [B][G], u_fast / u_slow [B][G-1]: squared velocities and accelerations of the two forward passes
 *   (tb_scan_ex with TB_SCAN_SD_FORWARD [| TB_SCAN_SD_SLOW]); desired_duration [B]; status_in (nullable) [B]: paths
 *   with TB_STATUS_FAIL_UNCONTROLLABLE get NaN outputs and keep that status;
 *   sd out [B][G] = sqrt(blend), sdd out [B][G-1]; info out [B][4] = (alpha, fastest duration, slowest duration,
 *   bisection steps); status out [B]: Ok or ErrUnknown (NaN in sd).  max_iter <= 0: 200 (the reference has no cap). */
int tb_sd_bisect(const double *x_fast, const double *u_fast, const double *x_slow, const double *u_slow,
                 const double *grid, int grid_shared, int B, int G, const double *desired_duration, double atol,
                 int max_iter, const int *status_in, double *sd, double *sdd, double *info, int *status, void *stream);

/* ParametrizeSpline time stamps (toppra/parametrizer.py:171-186): t_i = t_{i-1} + ds / mean(sd) with the two
 * data-dependent rules (mean speed <= 1e-8 -> 5 s; increments < 1e-8 are dropped from the knot list).
 *   sd, grid [B][G] (grid [G] if grid_shared); glen nullable (ragged); t_out, s_out [B][G]: kept time stamps and
 *   gridpoints, compacted, tail padded with the last kept entry; nkeep out [B]. */
int tb_spline_time_stamps(const double *sd, const double *grid, int grid_shared, const int *glen, int B, int G,
                          double *t_out, double *s_out, int *nkeep, void *stream);

/* Stand-alone batched LPs, one warp per LP — device counterparts of the reference's Python shims
 * solve_lp2d / solve_lp1d (cy_seidel_solverwrapper.pyx:42-87).
 *   tb_lp2d_batch: max v0 u + v1 x + v2  s.t. a u + b x + c <= 0 (n rows), low <= (u,x) <= high.
 *     v [B][3]; a,b,c [B][n]; low, high [B][2]; active_in [B][2] warm-start pair (nullable = zeros);
 *     result [B] (1 feasible / 0 infeasible); optval [B]; optvar [B][2] (NaN if infeasible);
 *     active_out [B][2] (row indices, or -1..-4 for the box bounds low0, high0, low1, high1).
 *   tb_lp1d_batch: max v0 x + v1  s.t. a x + b <= 0, low <= x <= high.   v [B][2]; a,b [B][n]; low, high [B];
 *     active_out [B] (row index, -1 = low, -2 = high). */
int tb_lp2d_batch(const double *v, const double *a, const double *b, const double *c, const double *low,
                  const double *high, const int *active_in, int B, int n, int *result, double *optval, double *optvar,
                  int *active_out, void *stream);
int tb_lp1d_batch(const double *v, const double *a, const double *b, const double *low, const double *high, int B,
                  int n, int *result, double *optval, double *optvar, int *active_out, void *stream);

/* K3 — output trajectory under the constant-acceleration assumption (ParametrizeConstAccel,
 * toppra/parametrizer.py:23-158).
 *   tb_time_grid: t_grid [B][G] time stamps of the gridpoints (t_0 = 0), us (nullable) [B][G-1] path accelerations,
 *                 from sd [B][G]; the duration of path b is t_grid[b][G-1].
 *   tb_constaccel_eval: out [B][M][dof] = q(t) (order 0), qd(t) (1), qdd(t) (2) at times ts [M] (ts_shared=1) or [B][M]. */
int tb_time_grid(const double *sd, const double *grid, int grid_shared, int B, int G, double *t_grid, double *us,
                 void *stream);
int tb_constaccel_eval(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof, const double *grid,
                       int grid_shared, const double *sd, const double *t_grid, const double *us, int B, int G,
                       const double *ts, int ts_shared, int M, int order, double *out, void *stream);

/* Whole pipeline with HOST buffers (K0 -> K1 -> K2, H2D/D2H inside, synchronous):
 *   ss [n] shared; wp [B][n][dof]; grid [G] shared; vlim (nullable) / alim: [dof][2] shared or [B][dof][2];
 *   outputs (host): K [B][G][2], sd [B][G], u [B][G-1], status [B].  device: CUDA device ordinal. */
int tb_solve_velacc_host(int device, const double *ss, const double *wp, int B, int n, int dof, const double *grid,
                         int G, const double *vlim, const double *alim, int lim_shared, int interp,
                         const double *sd_start, const double *sd_end, double *K, double *sd, double *u,
                         int *status);

#ifdef __cplusplus
}
#endif
#endif /* TOPPRA_B200_H_ */
