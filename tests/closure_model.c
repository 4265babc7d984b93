/*
 * tests/closure_model.c — TEST INFRASTRUCTURE ONLY.
 *
 * Scalar model of the min-x closure of the CUDA scan kernel (toppra_b200/csrc/tb_scan.cu, lp2d_impl: "Closure"), on top
 * of the unchanged model of shortcuts A and B (oracle/shortcut_model.c), checked the same way: beside the sequential
 * restatement on every 2-variable LP, counting results that differ in any bit.
 *
 * The closure: once shortcut A has named the last row m the reference visits in a min-x LP (objective (+, -)), the
 * re-solve on m ends on the x-box item x >= low1 unless another item binds.  The model computes that outcome with the
 * kernel's arithmetic (three divisions) and takes it when every other row, the u box and x <= high1 hold at the closed
 * point with a relative margin; otherwise it re-solves exactly.  See the kernel for why the margin is sufficient.
 * The closure counts as the one re-solve it replaces.
 */
#include "../oracle/shortcut_model.c"

static long cm_taken = 0, cm_declined = 0;
static double cm_gap = 1e-7; /* tb_scan.cu: SKIP_GAP */

/* row (aj, bj, cj) holds at (p0, p1) with margin */
static int cm_holds(double aj, double bj, double cj, double p0, double p1) {
  const double val = aj * p0 + bj * p1 + cj;
  return val <= -cm_gap * (1.0 + fabs(cj) + (fabs(aj) + fabs(bj)) * (fabs(p0) + fabs(p1)));
}

/* Closure of the re-solve on row m (natural order): 1 and (cur, act) = the reference's final state, or 0 */
static int cm_close(int nrows, const double *a, const double *b, const double *c, const double low[2],
                    const double high[2], int m, double cur[2], int act[2]) {
  const double nrm = a[m] * a[m] + b[m] * b[m];
  const double z0 = -a[m] * c[m] / nrm, z1 = -b[m] * c[m] / nrm;
  const double dt0 = -b[m], dt1 = a[m];
  /* box row (0, -1, low1) projected onto line m, in the operand order of the kernel's project_item */
  const double num = low[1] + z1 * -1.0 + z0 * 0.0;
  const double denom = dt0 * 0.0 + dt1 * -1.0;
  const double t = -num / denom;
  const double p0 = z0 + t * dt0, p1 = z1 + t * dt1;
  if (!(fabs(t) < sm_tmax)) return 0;
  for (int j = 0; j < nrows; ++j)
    if (j != m && !cm_holds(a[j], b[j], c[j], p0, p1)) return 0;
  if (!cm_holds(-1.0, 0.0, low[0], p0, p1) || !cm_holds(1.0, 0.0, -high[0], p0, p1) ||
      !cm_holds(0.0, 1.0, -high[1], p0, p1))
    return 0;
  cur[0] = p0;
  cur[1] = p1;
  act[0] = m;
  act[1] = -3;
  return 1;
}

/* sm_lp2d (oracle/shortcut_model.c) with the closure after shortcut A */
static LpSol cm_lp2d(const double v[3], int nrows, const double *a, const double *b, const double *c,
                     const double low[2], const double high[2], const long active_c[2], long *order, double *a_1d,
                     double *b_1d, long *nres) {
  LpSol sol;
  memset(&sol, 0, sizeof(sol));
  double cur[2];
  int act[2];
  for (int i = 0; i < 2; ++i) {
    if (low[i] > high[i]) return sol;
    if (v[i] > LP_TINY) { cur[i] = high[i]; act[i] = (i == 0) ? -2 : -4; }
    else { cur[i] = low[i]; act[i] = (i == 0) ? -1 : -3; }
  }
  const int valid = active_c[0] >= 0 && active_c[0] < nrows && active_c[1] >= 0 && active_c[1] < nrows &&
                    active_c[0] != active_c[1];
  if (valid) {
    int n = 2;
    order[0] = active_c[1];
    order[1] = active_c[0];
    for (int i = 0; i < nrows; ++i) if (i != active_c[0] && i != active_c[1]) order[n++] = i;
  } else {
    for (int i = 0; i < nrows; ++i) order[i] = i;
  }
  const int objective_ok = (v[0] > LP_TINY && v[1] < 0) || (v[0] < -LP_TINY && v[1] > 0);
  int k = 0, first = 1;
  while (k < nrows) {
    int kk = -1;
    for (int j = k; j < nrows; ++j) {
      const long i = order[j];
      if (!(a[i] * cur[0] + b[i] * cur[1] + c[i] < LP_TINY)) { kk = j; break; }
    }
    if (kk < 0) break;
    int target = kk;
    if (first && objective_ok) {
      if (!valid) {
        const int m = sm_shortcut_a(v, nrows, a, b, c, low, high, cur);
        if (m >= 0) {
          target = m;
          ++sm_a_used;
          if (v[0] > 0) {
            if (cm_close(nrows, a, b, c, low, high, m, cur, act)) {
              ++cm_taken;
              ++*nres;
              break;
            }
            ++cm_declined;
          }
        } else ++sm_a_abort;
      } else if (kk == 0) {
        if (sm_shortcut_b(v, a, b, c, low, high, order[0], order[1])) { target = 1; ++sm_b_used; } else ++sm_b_abort;
      }
    }
    first = 0;
    ++*nres;
    if (!sm_resolve(v, target, order, a, b, c, low, high, a_1d, b_1d, cur, act)) return sol;
    k = target + 1;
  }
  sol.result = 1;
  sol.optvar[0] = cur[0];
  sol.optvar[1] = cur[1];
  sol.active_c[0] = act[0];
  sol.active_c[1] = act[1];
  return sol;
}

static void cm_hook(const double v[3], int nrows, const double *a, const double *b, const double *c,
                    const double low[2], const double high[2], const long active_in[2], int result,
                    const double optvar[2], const int active_out[2]) {
  long *order = (long *)malloc(sizeof(long) * (nrows + 1));
  double *a1 = (double *)malloc(sizeof(double) * (nrows + 4)), *b1 = (double *)malloc(sizeof(double) * (nrows + 4));
  long nref = 0, nmodel = 0;
  {
    long *im = (long *)malloc(sizeof(long) * (nrows + 1));
    (void)lp2d(v, nrows, a, b, c, low, high, active_in, im, a1, b1, &nref);
    free(im);
  }
  const LpSol t = cm_lp2d(v, nrows, a, b, c, low, high, active_in, order, a1, b1, &nmodel);
  free(order); free(a1); free(b1);
  ++sm_lp;
  sm_resolve_ref += nref;
  sm_resolve_model += nmodel;
  if (t.result != result ||
      (result && (memcmp(t.optvar, optvar, 2 * sizeof(double)) || t.active_c[0] != active_out[0] ||
                  t.active_c[1] != active_out[1])))
    ++sm_mismatch;
}

void orc_closure_model_enable(int on) { orc_lp2d_hook = on ? cm_hook : NULL; }
void orc_closure_model_margin(double gap) { cm_gap = gap; }
/* out: the eight counters of orc_shortcut_model_stats, then closures taken, closures declined */
void orc_closure_model_stats(long *out, int reset) {
  orc_shortcut_model_stats(out, reset);
  out[8] = cm_taken; out[9] = cm_declined;
  if (reset) cm_taken = cm_declined = 0;
}
