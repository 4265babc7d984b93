/*
 * tests/robust_cones_oracle.c — TEST INFRASTRUCTURE ONLY.
 *
 * Scalar CPU restatement of libtoppra_b200_cones.so (toppra_b200/csrc/tb_cones.cu): robust problems whose rows each
 * carry their own robust flag and ellipsoid axes, cones [R][4] = (flag, ru, rx, rc), and whose stages may carry a u box
 * ubox [G][2] (ulo <= u <= uhi; NULL = [VAR_MIN, VAR_MAX]).  The stage loops are those of oracle/toppra_robust_oracle.c,
 * tests/robust_sd_oracle.c and tests/robust_reach_oracle.c, in the same operation order, row by row: so that
 *   * with the table of one ellipsoid and no u box, every entry here equals its single-ellipsoid counterpart bit for bit
 *     (tests/test_robust_cones.py checks this), and
 *   * the kernels can be compared with it bit for bit.
 * The closed form of one row, row_u_bounds, is the one of oracle/toppra_robust_oracle.c, included unchanged.  Compile
 * with -ffp-contract=off -fno-fast-math; tests/robust_cones_oracle.py does this into a temporary directory.
 */
#include "../oracle/toppra_robust_oracle.c"

typedef struct {
  int nC;                  /* rows incl. the two x_next rows at index 0, 1 */
  const double *a, *b, *c;
  const unsigned char *conic;
  const double *ru, *rx, *rc;  /* per row */
  double ulo, uhi;         /* the stage's u box */
} cstage_t;

static double cu_interval(const cstage_t *st, double x, double *uhi) {
  double lo = st->ulo, hi = st->uhi;
  int bad = 0;
  for (int r = 0; r < st->nC; ++r)
    row_u_bounds(st->conic[r], st->a[r], st->b[r], st->c[r], st->ru[r], st->rx[r], st->rc[r], x, &lo, &hi, &bad);
  *uhi = hi;
  if (bad) return -INFINITY;
  return hi - lo;
}

static int cu_bounds(const cstage_t *st, double x, double *ulo, double *uhi) {
  double lo = st->ulo, hi = st->uhi;
  int bad = 0;
  for (int r = 0; r < st->nC; ++r)
    row_u_bounds(st->conic[r], st->a[r], st->b[r], st->c[r], st->ru[r], st->rx[r], st->rc[r], x, &lo, &hi, &bad);
  *ulo = lo;
  *uhi = hi;
  if (bad) return 0;
  return hi - lo >= 0.0;
}

/* extreme_x of oracle/toppra_robust_oracle.c on the per-row stage */
static int cextreme_x(const cstage_t *st, int dir, double xl, double xh, double *xout, double hint) {
  if (xl > xh) return 0;
  double uh;
  double xgoal = (dir > 0) ? xh : xl, xother = (dir > 0) ? xl : xh;
  double wg = cu_interval(st, xgoal, &uh);
  if (wg >= 0.0) { *xout = xgoal; return 1; }
  double wo = cu_interval(st, xother, &uh);
  double xf = xother, wf = wo;
  double xb0 = xgoal, wb0 = wg;
  if (wo >= 0.0 && hint > xl && hint < xh) {
    double h1 = hint, h2 = (dir > 0) ? fmin(xh, hint * 1.25 + 1e-9) : fmax(xl, hint * 0.8 - 1e-9);
    double w1 = cu_interval(st, h1, &uh);
    if (w1 >= 0.0) {
      xf = h1; wf = w1;
      if (h2 != xgoal) {
        double w2 = cu_interval(st, h2, &uh);
        if (w2 >= 0.0) { xf = h2; wf = w2; } else { xb0 = h2; wb0 = w2; }
      }
    } else {
      xb0 = h1; wb0 = w1;
    }
  }
  if (!(wo >= 0.0)) {
    const double invphi = 0.6180339887498949;
    double lo = xl, hi = xh;
    double x1 = hi - invphi * (hi - lo), x2 = lo + invphi * (hi - lo);
    double w1 = cu_interval(st, x1, &uh);
    double w2 = cu_interval(st, x2, &uh);
    int found = 0;
    for (int it = 0; it < 80; ++it) {
      if (w1 >= 0.0) { xf = x1; wf = w1; found = 1; break; }
      if (w2 >= 0.0) { xf = x2; wf = w2; found = 1; break; }
      if (!(hi - lo > 1e-15 * (fabs(hi) + fabs(lo)) + 1e-300)) break;
      if (w1 > w2) { hi = x2; x2 = x1; w2 = w1; x1 = hi - invphi * (hi - lo); w1 = cu_interval(st, x1, &uh); }
      else { lo = x1; x1 = x2; w1 = w2; x2 = lo + invphi * (hi - lo); w2 = cu_interval(st, x2, &uh); }
    }
    if (!found) return 0;
  }
  double xb = xb0, wb = wb0;
  for (int it = 0; it < 200; ++it) {
    double width = fabs(xb - xf);
    if (!(width > 2.3e-16 * (fabs(xb) + fabs(xf)) + 1e-300)) break;
    double t;
    int finite = wb > -1e300;
    if (finite && (it % 3) != 2) {
      double frac = wf / (wf - wb);
      frac = (frac < 0.02) ? 0.02 : ((frac > 0.98) ? 0.98 : frac);
      t = xf + (xb - xf) * frac;
    } else {
      t = 0.5 * (xf + xb);
    }
    if (t == xf || t == xb) break;
    double wt = cu_interval(st, t, &uh);
    if (wt >= 0.0) { xf = t; wf = wt; } else { xb = t; wb = wt; }
  }
  *xout = xf;
  return 1;
}

/* Row arrays of nC = R + 2 rows with the table's flags and axes on rows 2.. (rows 0, 1 linear). */
typedef struct {
  double *a, *b, *c, *ru, *rx, *rc;
  unsigned char *conic;
} rowbuf_t;

static rowbuf_t rows_alloc(int R, const double *cones) {
  int nC = R + 2;
  rowbuf_t w;
  w.a = (double *)calloc(nC, sizeof(double)); w.b = (double *)calloc(nC, sizeof(double));
  w.c = (double *)calloc(nC, sizeof(double)); w.ru = (double *)calloc(nC, sizeof(double));
  w.rx = (double *)calloc(nC, sizeof(double)); w.rc = (double *)calloc(nC, sizeof(double));
  w.conic = (unsigned char *)calloc(nC, 1);
  for (int r = 0; r < R; ++r) {
    w.conic[2 + r] = cones[4 * r] != 0.0;
    w.ru[2 + r] = cones[4 * r + 1]; w.rx[2 + r] = cones[4 * r + 2]; w.rc[2 + r] = cones[4 * r + 3];
  }
  return w;
}

static void rows_free(rowbuf_t *w) { free(w->a); free(w->b); free(w->c); free(w->ru); free(w->rx); free(w->rc); free(w->conic); }

static cstage_t stage_of(const rowbuf_t *w, int nC) {
  cstage_t st = {nC, w->a, w->b, w->c, w->conic, w->ru, w->rx, w->rc, VAR_MIN, VAR_MAX};
  return st;
}

/* the records' rows of stage i, and its u box */
static void load_stage(rowbuf_t *w, cstage_t *st, const double *rows, const double *ubox, int R, int i) {
  for (int r = 0; r < R; ++r) {
    w->a[2 + r] = rows[((size_t)i * 3 + 0) * R + r]; w->b[2 + r] = rows[((size_t)i * 3 + 1) * R + r];
    w->c[2 + r] = rows[((size_t)i * 3 + 2) * R + r];
  }
  st->ulo = ubox ? ubox[2 * i] : VAR_MIN;
  st->uhi = ubox ? ubox[2 * i + 1] : VAR_MAX;
}

/* K2r (tbc_scan): rows [G][3][R], xbound [G][2] (as in the records), ubox [G][2] or NULL, K[N] = [sd_end^2,
 * sd_end_hi^2].  backward_only: the backward pass alone.  Outputs K [G][2], sd [G], u [G-1] (untouched when
 * backward_only), *fail_stage; returns the status.  The rules are those of orc_solve_rows_robust and
 * orc_controllable_sets_robust. */
int orc_cones_scan(const double *rows, const double *xbound, const double *ubox, const double *grid, int G, int R,
                   const double *cones, double sd_start, double sd_end, double sd_end_hi, int backward_only, double *K,
                   double *sd, double *u, int *fail_stage) {
  int N = G - 1, nC = R + 2, status = 0, fstage = -1;
  rowbuf_t w = rows_alloc(R, cones);
  cstage_t st = stage_of(&w, nC);
  for (int i = 0; i < 2 * G; ++i) K[i] = 0.0;
  K[2 * N] = sd_end * sd_end; K[2 * N + 1] = sd_end_hi * sd_end_hi;
  for (int i = N - 1; i >= 0; --i) {
    load_stage(&w, &st, rows, ubox, R, i);
    double xl = fmax(-ECOS_INFTY, xbound[i * 2]), xh = fmin(ECOS_INFTY, fmin(ECOS_MAXX, xbound[i * 2 + 1]));
    double delta = grid[i + 1] - grid[i];
    w.a[0] = -2 * delta; w.b[0] = -1.0; w.c[0] = K[2 * (i + 1)];
    w.a[1] = 2 * delta; w.b[1] = 1.0; w.c[1] = -K[2 * (i + 1) + 1];
    double x_upper = NAN, x_lower = NAN;
    int ok_hi = cextreme_x(&st, +1, xl, xh, &x_upper, K[2 * (i + 1) + 1]);
    int ok_lo = ok_hi && cextreme_x(&st, -1, xl, xh, &x_lower, K[2 * (i + 1)]);
    if (!ok_hi) x_upper = NAN;
    if (!ok_lo) x_lower = NAN;
    if (x_lower < 0) x_lower = 0;
    K[2 * i] = x_lower; K[2 * i + 1] = x_upper;
    if (!(ok_hi && ok_lo)) { status = 3; fstage = i; break; }
  }
  if (!backward_only) {
    double x_start = sd_start * sd_start;
    if (status == 0 && (x_start + ALG_SMALL < K[0] || K[1] + ALG_SMALL < x_start)) { status = 3; fstage = 0; }
    for (int i = 0; i < G; ++i) sd[i] = NAN;
    for (int i = 0; i < N; ++i) u[i] = NAN;
    if (status == 0) {
      double *xs = (double *)calloc(G, sizeof(double));
      for (int i = 0; i < N; ++i) u[i] = 0.0;
      xs[0] = x_start;
      for (int i = 0; i < N; ++i) {
        load_stage(&w, &st, rows, ubox, R, i);
        double delta = grid[i + 1] - grid[i];
        double k0 = K[2 * (i + 1)], k1 = K[2 * (i + 1) + 1];
        w.a[0] = -2 * delta; w.b[0] = -1.0; w.c[0] = k0;
        w.a[1] = 2 * delta; w.b[1] = 1.0; w.c[1] = -k1;
        int tries = 0, ok;
        double uh = 0.0, x = xs[i];
        while (1) {
          double wd = cu_interval(&st, x, &uh);
          ok = wd >= 0.0;
          if (ok || tries >= MAX_TRIES) break;
          x = fmax(x - ALG_TINY, 0.999 * x);
          ++tries;
        }
        xs[i] = x;
        if (!ok) { for (int j = i + 1; j < G; ++j) xs[j] = NAN; status = 1; fstage = i; break; }
        u[i] = uh;
        double x_next = x + 2 * delta * uh;
        x_next = fmax(x_next - ALG_TINY, 0.9999 * x_next);
        xs[i + 1] = fmin(k1, fmax(k0, x_next));
      }
      for (int j = 0; j < G; ++j) sd[j] = sqrt(xs[j]);
      free(xs);
    }
  }
  rows_free(&w);
  if (fail_stage) *fail_stage = fstage;
  return status;
}

/* Feasible sets (tbc_scan with TB_SCAN_FEASIBLE_SETS), the rules of orc_feasible_rows_robust. */
void orc_cones_feasible(const double *rows, const double *xbound, const double *ubox, const double *grid, int G, int R,
                        const double *cones, double *X) {
  int N = G - 1, nC = R + 2;
  rowbuf_t w = rows_alloc(R, cones);
  cstage_t st = stage_of(&w, nC);
  for (int i = 0; i <= N; ++i) {
    load_stage(&w, &st, rows, ubox, R, i);
    double xl = fmax(-CVXPY_MAXX, xbound[i * 2]), xh = fmin(CVXPY_MAXX, fmin(ECOS_MAXX, xbound[i * 2 + 1]));
    w.a[0] = 0.0; w.b[0] = 0.0; w.c[0] = -1.0;
    w.a[1] = 0.0; w.b[1] = 0.0; w.c[1] = -1.0;
    if (i < N) {
      double delta = grid[i + 1] - grid[i];
      w.a[0] = -2 * delta; w.b[0] = -1.0; w.c[0] = -CVXPY_MAXX;
      w.a[1] = 2 * delta; w.b[1] = 1.0; w.c[1] = -CVXPY_MAXX;
    }
    double x0 = NAN, x1 = NAN;
    if (!cextreme_x(&st, -1, xl, xh, &x0, NAN)) x0 = NAN;
    if (!cextreme_x(&st, +1, xl, xh, &x1, NAN)) x1 = NAN;
    if (x0 < 0) x0 = 0;
    X[2 * i] = x0; X[2 * i + 1] = x1;
  }
  rows_free(&w);
}

/* One TOPPRAsd forward pass (tbc_sd_forward), the rules of orc_sd_forward_rows_robust. */
int orc_cones_sd_forward(const double *rows, const double *ubox, const double *grid, int G, int R, const double *cones,
                         const double *K, double sd_start, int slow, double *x, double *u, int *fail_stage) {
  int N = G - 1, nC = R + 2, status = 0, fstage = -1;
  for (int i = 0; i < G; ++i) x[i] = NAN;
  for (int i = 0; i < N; ++i) u[i] = NAN;
  for (int i = 0; i < G; ++i)
    if (isnan(K[2 * i]) || isnan(K[2 * i + 1])) { status = 3; fstage = i; }
  double x0 = sd_start * sd_start;
  if (status == 0 && (x0 + ALG_SMALL < K[0] || K[1] + ALG_SMALL < x0)) { status = 3; fstage = 0; }
  if (status == 0) {
    rowbuf_t w = rows_alloc(R, cones);
    cstage_t st = stage_of(&w, nC);
    x[0] = x0;
    for (int i = 0; i < N; ++i) {
      load_stage(&w, &st, rows, ubox, R, i);
      double delta = grid[i + 1] - grid[i];
      double k0 = K[2 * (i + 1)], k1 = K[2 * (i + 1) + 1];
      w.a[0] = -2 * delta; w.b[0] = -1.0; w.c[0] = k0;
      w.a[1] = 2 * delta; w.b[1] = 1.0; w.c[1] = -k1;
      double ulo, uhi;
      if (!cu_bounds(&st, x[i], &ulo, &uhi)) { status = 1; fstage = i; break; }
      u[i] = slow ? ulo : uhi;
      double xn = x[i] + 2 * delta * u[i] - ALG_SMALL;
      xn = (xn > k0) ? xn : k0;
      x[i + 1] = (xn < k1) ? xn : k1;
    }
    rows_free(&w);
  }
  if (fail_stage) *fail_stage = fstage;
  return status;
}

/* One stage problem (tbc_socp_stage_batch), the rules of orc_socp_stage_robust; ubox2 (nullable) = (ulo, uhi). */
int orc_cones_socp(const double *g, const double *ra, const double *rb, const double *rcst, int n, const double *cones,
                   double xl, double xh, const double *xnext, const double *ubox2, double *out) {
  int nC = n + 2;
  rowbuf_t w = rows_alloc(n, cones);
  cstage_t st = stage_of(&w, nC);
  for (int r = 0; r < n; ++r) { w.a[2 + r] = ra[r]; w.b[2 + r] = rb[r]; w.c[2 + r] = rcst[r]; }
  w.a[0] = 0.0; w.b[0] = 0.0; w.c[0] = -1.0;
  w.a[1] = 0.0; w.b[1] = 0.0; w.c[1] = -1.0;
  if (xnext && !isnan(xnext[0])) {
    w.a[0] = -2 * xnext[0]; w.b[0] = -1.0; w.c[0] = xnext[1];
    w.a[1] = 2 * xnext[0]; w.b[1] = 1.0; w.c[1] = -xnext[2];
  }
  if (ubox2) { st.ulo = ubox2[0]; st.uhi = ubox2[1]; }
  double g0 = g[0], g1 = g[1];
  double xmin = NAN, xmax = NAN, xs = NAN, us = NAN;
  int feasible = cextreme_x(&st, -1, xl, xh, &xmin, NAN) && cextreme_x(&st, +1, xl, xh, &xmax, NAN);
  if (feasible && g0 == 0.0) {
    double ulo, uhi;
    xs = (g1 < 0.0) ? xmax : xmin;
    if (cu_bounds(&st, xs, &ulo, &uhi)) us = 0.5 * (ulo + uhi);
    else xs = NAN;
  } else if (feasible) {
    double ua, ub, u1, u2, ulo, uhi, fbest;
#define PHI(xv, uout) (cu_bounds(&st, (xv), &ulo, &uhi) ? ((uout) = (g0 < 0.0) ? uhi : ulo, g1 * (xv) + g0 * (uout)) \
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
  rows_free(&w);
  return !isnan(xs);
}

/* Reachable sets (tbc_reachable_sets), the rules of orc_reachable_sets_robust.  Returns fail_stage. */
int orc_cones_reachable(const double *rows, const double *xbound, const double *ubox, const double *grid, int G, int R,
                        const double *cones, const double *X, double sdmin, double sdmax, double *L) {
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
    orc_cones_socp(g1, ra, rb, rc, R, cones, xl, xh, xnext, ubox ? ubox + 2 * i : NULL, z1);
    orc_cones_socp(g0, ra, rb, rc, R, cones, xl, xh, xnext, ubox ? ubox + 2 * i : NULL, z0);
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
