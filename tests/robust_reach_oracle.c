/*
 * tests/robust_reach_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * Scalar CPU restatement of the reachable sets of robust problems (tbr_reachable_sets_robust, libtoppra_b200_reach.so,
 * toppra_b200/csrc/tb_reach.cu) and of K2r's backward pass from a velocity range (tb_scan_robust_ex with
 * TB_SCAN_BACKWARD_ONLY, toppra_b200/csrc/tb_robust.cu), with the same operation order, so that the kernels can be
 * compared with it bit for bit.  It builds on tests/robust_sd_oracle.c (each stage end is one orc_socp_stage_robust) and
 * on the stage primitives of oracle/toppra_robust_oracle.c, both included unchanged.  Compile with -ffp-contract=off
 * -fno-fast-math; tests/robust_reach_oracle.py does this into a temporary directory.  Parity with the reference is
 * unpinned (it solves these problems with ECOS); tests/test_robust_reachability.py checks this restatement against the
 * 50-digit reference of tests/robust_mp.py.
 */
#include "robust_sd_oracle.c"

/* Controllable sets with a velocity range at the end: K2r's backward pass as orc_solve_rows_robust runs it, from
 * K[N] = [sd_end^2, sd_end_hi^2].  rows [G][3][R], xbound [G][2], K out [G][2] (the rows before a failed stage 0).
 * Returns the status (0 or 3); *fail_stage = the failed stage or -1. */
int orc_controllable_sets_robust(const double *rows, const double *xbound, const double *grid, int G, int R, int conic0,
                                 int conicn, const double *ell, double sd_end, double sd_end_hi, double *K,
                                 int *fail_stage) {
  int N = G - 1, nC = R + 2, status = 0, fstage = -1;
  double *a = (double *)malloc(sizeof(double) * nC), *b = (double *)malloc(sizeof(double) * nC);
  double *c = (double *)malloc(sizeof(double) * nC);
  unsigned char *conic = (unsigned char *)calloc(nC, 1);
  for (int r = 0; r < R; ++r) conic[2 + r] = (r >= conic0 && r < conic0 + conicn);
  stage_t st = {nC, a, b, c, conic, ell[0], ell[1], ell[2], 0};
  for (int i = 0; i < 2 * G; ++i) K[i] = 0.0;
  K[2 * N] = sd_end * sd_end; K[2 * N + 1] = sd_end_hi * sd_end_hi;
  for (int i = N - 1; i >= 0; --i) {
    for (int r = 0; r < R; ++r) {
      a[2 + r] = rows[((size_t)i * 3 + 0) * R + r]; b[2 + r] = rows[((size_t)i * 3 + 1) * R + r];
      c[2 + r] = rows[((size_t)i * 3 + 2) * R + r];
    }
    double xl = fmax(-ECOS_INFTY, xbound[i * 2]), xh = fmin(ECOS_INFTY, fmin(ECOS_MAXX, xbound[i * 2 + 1]));
    double delta = grid[i + 1] - grid[i];
    a[0] = -2 * delta; b[0] = -1.0; c[0] = K[2 * (i + 1)];
    a[1] = 2 * delta; b[1] = 1.0; c[1] = -K[2 * (i + 1) + 1];
    double x_upper = NAN, x_lower = NAN;
    int ok_hi = extreme_x(&st, +1, xl, xh, &x_upper, K[2 * (i + 1) + 1]);
    int ok_lo = ok_hi && extreme_x(&st, -1, xl, xh, &x_lower, K[2 * (i + 1)]);
    if (!ok_hi) x_upper = NAN;
    if (!ok_lo) x_lower = NAN;
    if (x_lower < 0) x_lower = 0;
    K[2 * i] = x_lower; K[2 * i + 1] = x_upper;
    if (!(ok_hi && ok_lo)) { status = 3; fstage = i; break; }
  }
  free(a); free(b); free(c); free(conic);
  if (fail_stage) *fail_stage = fstage;
  return status;
}

/* Reachable sets (tbr_reachable_sets_robust, include/toppra_b200_reach.h, whose rules this restates) on the feasible
 * sets X [G][2] (orc_feasible_rows_robust).  rows [G][3][R], xbound [G][2], L out [G][2].  Returns fail_stage: the index
 * of the first NaN row of L, or -1. */
int orc_reachable_sets_robust(const double *rows, const double *xbound, const double *grid, int G, int R, int conic0,
                              int conicn, const double *ell, const double *X, double sdmin, double sdmax, double *L) {
  int N = G - 1, fs = -1;
  double *ra = (double *)malloc(sizeof(double) * (R > 0 ? R : 1)), *rb = (double *)malloc(sizeof(double) * (R > 0 ? R : 1));
  double *rc = (double *)malloc(sizeof(double) * (R > 0 ? R : 1));
  for (int i = 0; i < 2 * G; ++i) L[i] = 0.0;
  double l0 = sdmin * sdmin, l1 = sdmax * sdmax;
  L[0] = l0; L[1] = l1;
  for (int i = 0; i < N; ++i) {
    for (int r = 0; r < R; ++r) {
      ra[r] = rows[((size_t)i * 3 + 0) * R + r]; rb[r] = rows[((size_t)i * 3 + 1) * R + r];
      rc[r] = rows[((size_t)i * 3 + 2) * R + r];
    }
    double xl = fmax(l0, xbound[2 * i]), xh = fmin(l1, fmin(ECOS_MAXX, xbound[2 * i + 1]));
    double xnext[3] = {grid[i + 1] - grid[i], isnan(X[2 * (i + 1)]) ? -ECOS_INFTY : X[2 * (i + 1)],
                       isnan(X[2 * (i + 1) + 1]) ? ECOS_INFTY : X[2 * (i + 1) + 1]};
    double dq = (i > 0) ? (grid[i] - grid[i - 1]) : (grid[N] - grid[N - 1]);
    double g1[2] = {-2 * dq, -1.0}, g0[2] = {2 * dq, 1.0}, z1[2], z0[2];
    orc_socp_stage_robust(g1, ra, rb, rc, R, conic0, conicn, ell, xl, xh, xnext, z1);
    orc_socp_stage_robust(g0, ra, rb, rc, R, conic0, conicn, ell, xl, xh, xnext, z0);
    double x_upper = z1[1] + 2 * dq * z1[0], x_lower = z0[1] + 2 * dq * z0[0];
    if (x_lower < 0) x_lower = 0;
    L[2 * (i + 1)] = x_lower; L[2 * (i + 1) + 1] = x_upper;
    if (isnan(x_lower) || isnan(x_upper)) { fs = i + 1; break; }
    l0 = x_lower;
    l1 = x_upper;
  }
  free(ra); free(rb); free(rc);
  return fs;
}
