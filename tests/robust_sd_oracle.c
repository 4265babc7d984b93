/*
 * tests/robust_sd_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * Scalar CPU restatement of libtoppra_b200_robust.so (toppra_b200/csrc/tb_conic.cu): the robust TOPPRAsd forward passes
 * (tbr_sd_forward_robust) and single stage problems (tbr_socp_stage_batch), with the same operation order, so that the
 * kernels can be compared with it bit for bit.  It builds on the restatement of K2r's stage primitives in
 * oracle/toppra_robust_oracle.c (row_u_bounds, u_interval, extreme_x), which it includes unchanged, as
 * oracle/shortcut_model.c includes oracle/toppra_oracle.c.  Compile with -ffp-contract=off -fno-fast-math (no FMA
 * contraction, like the kernels' -fmad=false); tests/robust_sd_oracle.py does this into a temporary directory.
 * Parity with the reference is unpinned (it solves these problems with ECOS); tests/test_robust_sd.py checks this
 * restatement against independent evidence.
 */
#include "../oracle/toppra_robust_oracle.c"

/* Both ends of the feasible u-interval at x; 1 = non-empty (the rule of u_interval). */
static int u_bounds(stage_t *st, double x, double *ulo, double *uhi) {
  double lo = VAR_MIN, hi = VAR_MAX;
  int bad = 0;
  for (int r = 0; r < st->nC; ++r)
    row_u_bounds(st->conic[r], st->a[r], st->b[r], st->c[r], st->ru, st->rx, st->rc, x, &lo, &hi, &bad);
  st->n_eval++;
  *ulo = lo;
  *uhi = hi;
  if (bad) return 0;
  return hi - lo >= 0.0;
}

/* One TOPPRAsd forward pass (desired_duration_algorithm.py:83-121; slow = the slowest pass, :207-234) over the controllable
 * sets K [G][2] of the backward pass (orc_solve_rows_robust).  rows [G][3][R]; x out [G] holds x = sd^2, u out [G-1].
 * Returns the status; *fail_stage as tbr_sd_forward_robust (include/toppra_b200_robust.h), whose rules this restates. */
int orc_sd_forward_rows_robust(const double *rows, const double *grid, int G, int R, int conic0, int conicn,
                               const double *ell, const double *K, double sd_start, int slow, double *x, double *u,
                               int *fail_stage) {
  int N = G - 1, nC = R + 2, status = 0, fstage = -1;
  for (int i = 0; i < G; ++i) x[i] = NAN;
  for (int i = 0; i < N; ++i) u[i] = NAN;
  for (int i = 0; i < G; ++i)
    if (isnan(K[2 * i]) || isnan(K[2 * i + 1])) { status = 3; fstage = i; }
  double x0 = sd_start * sd_start;
  if (status == 0 && (x0 + ALG_SMALL < K[0] || K[1] + ALG_SMALL < x0)) { status = 3; fstage = 0; }
  if (status == 0) {
    double *a = (double *)malloc(sizeof(double) * nC), *b = (double *)malloc(sizeof(double) * nC);
    double *c = (double *)malloc(sizeof(double) * nC);
    unsigned char *conic = (unsigned char *)calloc(nC, 1);
    for (int r = 0; r < R; ++r) conic[2 + r] = (r >= conic0 && r < conic0 + conicn);
    stage_t st = {nC, a, b, c, conic, ell[0], ell[1], ell[2], 0};
    x[0] = x0;
    for (int i = 0; i < N; ++i) {
      for (int r = 0; r < R; ++r) {
        a[2 + r] = rows[((size_t)i * 3 + 0) * R + r]; b[2 + r] = rows[((size_t)i * 3 + 1) * R + r];
        c[2 + r] = rows[((size_t)i * 3 + 2) * R + r];
      }
      double delta = grid[i + 1] - grid[i];
      double k0 = K[2 * (i + 1)], k1 = K[2 * (i + 1) + 1];
      a[0] = -2 * delta; b[0] = -1.0; c[0] = k0;
      a[1] = 2 * delta; b[1] = 1.0; c[1] = -k1;
      double ulo, uhi;
      if (!u_bounds(&st, x[i], &ulo, &uhi)) { status = 1; fstage = i; break; }
      u[i] = slow ? ulo : uhi;
      double xn = x[i] + 2 * delta * u[i] - ALG_SMALL;
      xn = (xn > k0) ? xn : k0;
      x[i + 1] = (xn < k1) ? xn : k1;
    }
    free(a); free(b); free(c); free(conic);
  }
  if (fail_stage) *fail_stage = fstage;
  return status;
}

/* One stage problem (tbr_socp_stage_batch, include/toppra_b200_robust.h): min g0 u + g1 x over n rows a, b, c (robust on
 * [conic0, conic0 + conicn)), xl <= x <= xh and, when xnext is not NULL and xnext[0] (delta) is not NaN,
 * xnext[1] <= x + 2 delta u <= xnext[2].  out = (u, x), NaN NaN when infeasible; returns 1 when feasible. */
int orc_socp_stage_robust(const double *g, const double *ra, const double *rb, const double *rcst, int n, int conic0,
                          int conicn, const double *ell, double xl, double xh, const double *xnext, double *out) {
  int nC = n + 2;
  double *a = (double *)malloc(sizeof(double) * nC), *b = (double *)malloc(sizeof(double) * nC);
  double *c = (double *)malloc(sizeof(double) * nC);
  unsigned char *conic = (unsigned char *)calloc(nC, 1);
  for (int r = 0; r < n; ++r) {
    a[2 + r] = ra[r]; b[2 + r] = rb[r]; c[2 + r] = rcst[r];
    conic[2 + r] = (r >= conic0 && r < conic0 + conicn);
  }
  a[0] = 0.0; b[0] = 0.0; c[0] = -1.0;
  a[1] = 0.0; b[1] = 0.0; c[1] = -1.0;
  if (xnext && !isnan(xnext[0])) {
    a[0] = -2 * xnext[0]; b[0] = -1.0; c[0] = xnext[1];
    a[1] = 2 * xnext[0]; b[1] = 1.0; c[1] = -xnext[2];
  }
  stage_t st = {nC, a, b, c, conic, ell[0], ell[1], ell[2], 0};
  double g0 = g[0], g1 = g[1];
  double xmin = NAN, xmax = NAN, xs = NAN, us = NAN;
  int feasible = extreme_x(&st, -1, xl, xh, &xmin, NAN) && extreme_x(&st, +1, xl, xh, &xmax, NAN);
  if (feasible && g0 == 0.0) {
    double ulo, uhi;
    xs = (g1 < 0.0) ? xmax : xmin;
    if (u_bounds(&st, xs, &ulo, &uhi)) us = 0.5 * (ulo + uhi);
    else xs = NAN;
  } else if (feasible) {
    double ua, ub, u1, u2, ulo, uhi, fbest;
#define PHI(xv, uout) (u_bounds(&st, (xv), &ulo, &uhi) ? ((uout) = (g0 < 0.0) ? uhi : ulo, g1 * (xv) + g0 * (uout)) \
                                                        : ((uout) = (g0 < 0.0) ? uhi : ulo, INFINITY))
    double fa = PHI(xmin, ua), fb = PHI(xmax, ub);
    if (fa <= fb) { xs = xmin; us = ua; fbest = fa; } else { xs = xmax; us = ub; fbest = fb; }
    const double invphi = 0.6180339887498949;
    double lo = xmin, hi = xmax;
    double x1 = hi - invphi * (hi - lo), x2 = lo + invphi * (hi - lo);
    double f1 = PHI(x1, u1), f2 = PHI(x2, u2);
    if (f1 < fbest) { xs = x1; us = u1; fbest = f1; }
    if (f2 < fbest) { xs = x2; us = u2; fbest = f2; }
    for (int it = 0; it < 200; ++it) {
      if (!(hi - lo > 2.3e-16 * (fabs(hi) + fabs(lo)) + 1e-300)) break;
      if (f1 <= f2) {
        hi = x2; x2 = x1; f2 = f1; u2 = u1;
        x1 = hi - invphi * (hi - lo);
        f1 = PHI(x1, u1);
        if (f1 < fbest) { xs = x1; us = u1; fbest = f1; }
      } else {
        lo = x1; x1 = x2; f1 = f2; u1 = u2;
        x2 = lo + invphi * (hi - lo);
        f2 = PHI(x2, u2);
        if (f2 < fbest) { xs = x2; us = u2; fbest = f2; }
      }
    }
#undef PHI
    if (!(fbest < INFINITY)) { xs = NAN; us = NAN; }
  }
  out[0] = us;
  out[1] = xs;
  free(a); free(b); free(c); free(conic);
  return !isnan(xs);
}
