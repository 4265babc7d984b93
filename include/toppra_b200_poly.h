/*
 * toppra_b200_poly.h — C-ABI of libtoppra_b200_poly.so: piecewise-polynomial paths of order k <= 8 (degree <= 7)
 * for the batched TOPP-RA of libtoppra_b200.so (include/toppra_b200.h).
 *
 * The reference (hungpham2511/toppra v0.6.2) accepts any path object: its algorithm samples the path at the
 * gridpoints only (path(gridpoints, 1), path(gridpoints, 2): toppra/constraint/linear_joint_velocity.py:48,
 * linear_joint_acceleration.py:72-73; path(mid, 2): toppra/interpolator.py:102; path(...): toppra/parametrizer.py:87-92).
 * This library gives the solver those samples for paths in scipy's PPoly layout with up to 8 coefficients per piece:
 *
 *   tbp_ppoly_eval            <-> PPoly(c, x)(s), .derivative()(s), .derivative().derivative()(s)
 *   tbp_rows_velacc_sampled   <-> JointVelocity / JointAcceleration records from sampled q'(grid), q''(grid)
 *                                 (the contract of tb_coeff_velacc)
 *   tbp_xbound_varying_sampled<-> JointVelocityConstraintVarying from sampled q'(grid) (the contract of tb_xbound_varying)
 *   tbp_propose_gridpoints    <-> propose_gridpoints, toppra/interpolator.py:49-122 (the contract of tb_propose_gridpoints)
 *   tbp_constaccel_eval       <-> ParametrizeConstAccel.__call__, toppra/parametrizer.py:82-129 (the contract of
 *                                 tb_constaccel_eval)
 * The records these functions write go to the record kernels of libtoppra_b200.so unchanged (tb_scan_ragged,
 * tb_feasible_sets_ex, tb_reachable_sets, tb_scan_robust).
 *
 * Conventions are those of include/toppra_b200.h: device pointers, caller-owned memory, asynchronous on `stream`,
 * 0 / TB_ERR_* / cudaError_t returns, fp64 with -fmad=false.  This library links against libtoppra_b200.so and reports
 * errors through its tb_last_error().
 *
 * Path layout: ppoly [B][k][nseg][dof] (scipy PPoly.c per path: highest power first, local basis (s - x[i])),
 * 1 <= k <= TBP_MAX_COEFFS; breaks [nseg+1] (breaks_shared=1) or [B][nseg+1].  Derivatives follow scipy's derivative
 * objects: order 1 has the coefficients c[j] * (k-1-j), order 2 the chained (c[j] * (k-1-j)) * (k-2-j); each is
 * evaluated with scipy's evaluate_poly1 power accumulation over exactly its own coefficients.
 */
#ifndef TOPPRA_B200_POLY_H_
#define TOPPRA_B200_POLY_H_

#ifdef __cplusplus
extern "C" {
#endif

#define TBP_VERSION 100
#define TBP_MAX_COEFFS 8

int tbp_version(void);

/* q^(order)(s), order 0..2: s [G] (s_shared=1) or [B][G] -> out [B][G][dof].  NaN s gives NaN; s outside the
 * breakpoints extrapolates the end pieces (scipy find_interval). */
int tbp_ppoly_eval(const double *ppoly, const double *breaks, int breaks_shared, int B, int k, int nseg, int dof,
                   const double *s, int s_shared, int G, int order, double *out, void *stream);

/* Stage records from sampled path derivatives: qd = q'(grid), qdd = q''(grid), both [B][G][dof] (e.g. two calls of
 * tbp_ppoly_eval).  Every other argument, and the records written, as tb_coeff_velacc. */
int tbp_rows_velacc_sampled(const double *qd, const double *qdd, int B, int dof, const double *grid, int grid_shared,
                            int G, const double *vlim, const double *alim, int lim_shared, int interp, double *records,
                            int W, int R_total, int row0, int write_xbound, void *stream);

/* JointVelocityConstraintVarying from sampled qd = q'(grid) [B][G][dof]; vlim_grid and the rest as tb_xbound_varying. */
int tbp_xbound_varying_sampled(const double *qd, int B, int dof, int G, const double *vlim_grid, int vlim_shared,
                               double *records, int W, int R_total, int write_xbound, void *stream);

/* tb_propose_gridpoints on order-k paths. */
int tbp_propose_gridpoints(const double *ppoly, const double *breaks, int breaks_shared, int B, int k, int nseg, int dof,
                           double max_err_threshold, int max_iteration, double max_seg_length, int min_nb_points,
                           int Gmax, double *grid_out, double *scratch, int *glen, int *status, void *stream);

/* tb_constaccel_eval on order-k paths (t_grid / us from tb_time_grid). */
int tbp_constaccel_eval(const double *ppoly, const double *breaks, int breaks_shared, int k, int nseg, int dof,
                        const double *grid, int grid_shared, const double *sd, const double *t_grid, const double *us,
                        int B, int G, const double *ts, int ts_shared, int M, int order, double *out, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* TOPPRA_B200_POLY_H_ */
