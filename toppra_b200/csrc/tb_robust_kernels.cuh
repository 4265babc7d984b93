// tb_robust_kernels.cuh — the stage loops of the four conic kernels, one body each, templated on the row form:
//   PER_ROW = false  one ellipsoid (ru, rx, rc: double) on the rows [conic0, conic0 + conicn), the conic mask set per
//                    stage, no u box (table, ub / ubox unused);
//   PER_ROW = true   the robust flag and the axes (ru, rx, rc: Slots<RPL>) of each row from the cone table, loaded once
//                    per path (conic0 / conicn unused), and the u box: the records' u-bound pair when ub
//                    (TB_SCAN_UBOUND), ubox[p] for the stage solves.
// Each library wraps a body in its own __global__ kernel:
//   scan_robust_body        K2r: backward / forward pass, feasible sets      scan_robust_kernel (tb_robust.cu),
//                                                                             tbc_scan_kernel (tb_cones.cu)
//   sd_forward_robust_body  TOPPRAsd's fastest and slowest forward pass      sd_forward_robust_kernel (tb_conic.cu),
//                                                                             tbc_sd_forward_kernel
//   socp_stage_body         one stage problem min g0 u + g1 x               socp_stage_kernel (tb_conic.cu),
//                                                                             tbc_socp_stage_kernel
//   reachable_robust_body   compute_reachable_sets' forward recursion        reachable_robust_kernel (tb_reach.cu),
//                                                                             tbc_reachable_kernel
// With PER_ROW = false the single-ellipsoid kernels compile to the machine code they had as kernels of their own
// (DESIGN.md, section 4).
#pragma once
#include <limits.h>

#include "tb_robust_common.cuh"

namespace tb {
namespace {

// One warp per CTA, like the record scan: a finished path frees its slot at once.
template <int RPL, bool PER_ROW>
__device__ __forceinline__ void scan_robust_body(
    const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
    Axes<RPL, PER_ROW> ru, Axes<RPL, PER_ROW> rx, Axes<RPL, PER_ROW> rc, const double *__restrict__ grid,
    const int grid_shared, const int B, const int G, const double *__restrict__ sd_start,
    const double *__restrict__ sd_end, const int flags, double *__restrict__ Kout, double *__restrict__ sdout,
    double *__restrict__ uout, int *__restrict__ status, int *__restrict__ fail_stage, int *__restrict__ counters,
    const int *__restrict__ glen, const double *__restrict__ sd_end_hi, const ConeTable *__restrict__ table,
    const bool ub) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  // glen (optional): ragged batches, as in scan_kernel; K / sd / u past this path's gridpoints are NaN
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int nC = R + 2;
  // The stage count lives in shared memory (one warp per CTA) and is re-read where it is used.  Held in a register
  // across the passes it raises the RPL 1 build's spills under its 72-register cap (-Xptxas -v: 192/368 bytes of spill
  // stores/loads with a compile-time G - 1, 264/608 with a register-held count, 152/224 like this).
  volatile __shared__ int s_n;
  if (lane == 0) s_n = Gp - 1;
  __syncwarp();
  const volatile int &N = s_n;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  double *Kp = Kout + (size_t)path * G * 2;
  const bool backward_only = (flags & 1) != 0;
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  // the padding is written up front: no pass below touches it, and the registers that hold Gp and the output pointers
  // are free here (written at the end, it adds spill traffic to the RPL 1 build)
  for (int j = 2 * Gp + lane; j < 2 * G; j += 32) Kp[j] = nan_d;
  if (!(flags & 3)) {
    for (int j = Gp + lane; j < G; j += 32) sdp[j] = nan_d;
    for (int j = N + lane; j < G - 1; j += 32) up[j] = nan_d;
  }
  double a[RPL], b[RPL], c[RPL];
  unsigned cmask[RPL];
  double ubox_lo = VAR_MIN, ubox_hi = VAR_MAX;   // the u box: the records' u-bound pair with ub (PER_ROW)
  if constexpr (PER_ROW) load_cones<RPL>(table, R, lane, cmask, ru, rx, rc);
  int n_eval = 0, n_retry = 0;

  if (flags & 2) {
    // compute_feasible_sets (reachability_algorithm.py:131-164): x, x_next in [-1e4, 1e4], every stage on its own
    for (int i = 0; i <= N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL, PER_ROW>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask, ub, ubox_lo, ubox_hi);
      const double xl = fmax(-CVXPY_MAXX, rec[3 * R]);
      const double xh = fmin(CVXPY_MAXX, fmin(ECOS_MAXX, rec[3 * R + 1]));
      if (i < N) {
        const double delta = gp[i + 1] - gp[i];
        if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = -CVXPY_MAXX; }
        if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -CVXPY_MAXX; }
      }
      double x0 = nan_d, x1 = nan_d;
      if (!extreme_x<RPL>(-1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, x0, n_eval, nan_d)) x0 = nan_d;
      if (!extreme_x<RPL>(+1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, x1, n_eval, nan_d)) x1 = nan_d;
      if (x0 < 0) x0 = 0;
      if (lane == 0) { Kp[2 * i] = x0; Kp[2 * i + 1] = x1; }
    }
    if (lane == 0) { status[path] = TB_STATUS_OK; if (fail_stage) fail_stage[path] = -1; }
    return;
  }
  const double sde = sd_end ? sd_end[path] : 0.0;
  const double sdeh = sd_end_hi ? sd_end_hi[path] : sde;   // K[N] = [sd_end^2, sd_end_hi^2]
  const double sds = sd_start ? sd_start[path] : 0.0;
  double kn0 = sde * sde, kn1 = sdeh * sdeh;
  if (lane == 0) { Kp[2 * N] = kn0; Kp[2 * N + 1] = kn1; }
  int st = TB_STATUS_OK, fstage = -1;
  for (int i = N - 1; i >= 0; --i) {
    const double *rec = rec_path + (size_t)i * W;
    rload_rows<RPL, PER_ROW>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask, ub, ubox_lo, ubox_hi);
    if (i > 0 && lane * 16 < W)  // pull the next stage's record towards L1 while this stage is solved
      asm volatile("prefetch.global.L1 [%0];" ::"l"(rec - W + lane * 16));
    // x box: NaN x_min/x_max -> -/+ECOS_INFTY; xbound: x <= min(ECOS_MAXX, hi), x >= lo  (ecos_solverwrapper.py:112-172)
    const double xl = fmax(-ECOS_INFTY, rec[3 * R]);
    const double xh = fmin(ECOS_INFTY, fmin(ECOS_MAXX, rec[3 * R + 1]));
    const double delta = gp[i + 1] - gp[i];
    if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = kn0; }
    if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -kn1; }
    double x_upper = nan_d, x_lower = nan_d;
    const bool ok_hi = extreme_x<RPL>(+1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, x_upper, n_eval, kn1);
    const bool ok_lo = ok_hi && extreme_x<RPL>(-1, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, x_lower, n_eval, kn0);
    if (!ok_hi) x_upper = nan_d;
    if (!ok_lo) x_lower = nan_d;
    if (x_lower < 0) x_lower = 0;
    if (lane == 0) { Kp[2 * i] = x_lower; Kp[2 * i + 1] = x_upper; }
    if (!(ok_hi && ok_lo)) {
      st = TB_STATUS_FAIL_UNCONTROLLABLE;
      fstage = i;
      for (int j = lane; j < 2 * i; j += 32) Kp[j] = 0.0;
      break;
    }
    kn0 = x_lower;
    kn1 = x_upper;
  }
  __syncwarp();
  const double x_start = sds * sds;
  if (st == TB_STATUS_OK && !backward_only) {
    if (x_start + ALG_SMALL < kn0 || kn1 + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  if (backward_only) {
    if (lane == 0) { status[path] = st; if (fail_stage) fail_stage[path] = fstage; }
    return;
  }
  if (st != TB_STATUS_OK) {
    for (int j = lane; j < Gp; j += 32) sdp[j] = nan_d;
    for (int j = lane; j < N; j += 32) up[j] = nan_d;
  } else {
    double x = x_start;
    if (lane == 0) sdp[0] = x;
    for (int i = 0; i < N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL, PER_ROW>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask, ub, ubox_lo, ubox_hi);
      if (i + 2 < N && lane * 16 < W) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 2 * W + lane * 16));
      const double delta = gp[i + 1] - gp[i];
      const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
      if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = k0; }
      if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -k1; }
      int tries = 0;
      bool ok;
      double uopt = 0.0;
      while (true) {
        double uh;
        const double w = u_interval<RPL>(x, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, uh);
        ++n_eval;
        ok = w >= 0.0;
        uopt = uh;
        if (ok || tries >= MAX_TRIES) break;
        x = fmax(x - ALG_TINY, 0.999 * x);
        ++tries;
        ++n_retry;
      }
      if (!ok) {
        st = TB_STATUS_ERR_UNKNOWN;
        fstage = i;
        if (lane == 0) sdp[i] = x;
        for (int j = i + 1 + lane; j < Gp; j += 32) sdp[j] = nan_d;
        for (int j = i + lane; j < N; j += 32) up[j] = 0.0;
        break;
      }
      double x_next = x + 2 * delta * uopt;
      x_next = fmax(x_next - ALG_TINY, 0.9999 * x_next);
      x_next = fmin(k1, fmax(k0, x_next));
      if (lane == 0) {
        up[i] = uopt;
        if (tries) sdp[i] = x;
        sdp[i + 1] = x_next;
      }
      x = x_next;
    }
    __syncwarp();
    for (int j = lane; j < Gp; j += 32) sdp[j] = sqrt(sdp[j]);
  }
  if (lane == 0) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
    if (counters) {
      counters[path * 4 + 0] = n_eval;
      counters[path * 4 + 1] = 0;
      counters[path * 4 + 2] = 0;
      counters[path * 4 + 3] = n_retry;
    }
  }
}

// One warp per (path, pass), one warp per CTA: blockIdx.x = 2 path + (0 fastest, 1 slowest).  The rules are those of
// desired_duration_algorithm.py:87-121 (the slowest pass :207-234), on the conventions of tb_scan_ex with
// TB_SCAN_SD_FORWARD: x out holds x = sd^2, status / fail_stage are the fastest pass's.
template <int RPL, bool PER_ROW>
__device__ __forceinline__ void sd_forward_robust_body(
    const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
    Axes<RPL, PER_ROW> ru, Axes<RPL, PER_ROW> rx, Axes<RPL, PER_ROW> rc, const double *__restrict__ grid,
    const int grid_shared, const int B, const int G, const int *__restrict__ glen, const double *__restrict__ K,
    const int *__restrict__ status_in, const double *__restrict__ sd_start, double *__restrict__ x_fast,
    double *__restrict__ u_fast, double *__restrict__ x_slow, double *__restrict__ u_slow, int *__restrict__ status,
    int *__restrict__ fail_stage, const ConeTable *__restrict__ table, const bool ub) {
  const int lane = threadIdx.x & 31;
  const long warp = warp_path();
  const long path = warp >> 1;
  const bool slow = (warp & 1) != 0;
  if (path >= B) return;
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int N = Gp - 1, nC = R + 2;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  const double *Kp = K + (size_t)path * G * 2;
  double *xp = (slow ? x_slow : x_fast) + (size_t)path * G;
  double *up = (slow ? u_slow : u_fast) + (size_t)path * (G > 1 ? G - 1 : 0);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  for (int j = Gp + lane; j < G; j += 32) xp[j] = nan_d;       // ragged padding
  for (int j = N + lane; j < G - 1; j += 32) up[j] = nan_d;

  int st = status_in[path], fstage = -1;
  if (st != TB_STATUS_OK) {
    // the backward pass failed: its stage is the last row of K with a NaN end (the rows before it are 0)
    int last = -1;
    for (int j = lane; j < Gp; j += 32)
      if (!(Kp[2 * j] == Kp[2 * j]) || !(Kp[2 * j + 1] == Kp[2 * j + 1])) last = j;
    fstage = __reduce_max_sync(FULL, last);
  } else {
    // admissibility of sd_start, desired_duration_algorithm.py:83-84
    const double sds = sd_start ? sd_start[path] : 0.0;
    const double x0 = sds * sds;
    if (x0 + ALG_SMALL < Kp[0] || Kp[1] + ALG_SMALL < x0) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  if (st != TB_STATUS_OK) {
    for (int j = lane; j < Gp; j += 32) xp[j] = nan_d;
    for (int j = lane; j < N; j += 32) up[j] = nan_d;
  } else {
    const double sds = sd_start ? sd_start[path] : 0.0;
    double x = sds * sds;
    if (lane == 0) xp[0] = x;
    double a[RPL], b[RPL], c[RPL];
    unsigned cmask[RPL];
    double ubox_lo = VAR_MIN, ubox_hi = VAR_MAX;
    if constexpr (PER_ROW) load_cones<RPL>(table, R, lane, cmask, ru, rx, rc);
    for (int i = 0; i < N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL, PER_ROW>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask, ub, ubox_lo, ubox_hi);
      if (i + 2 < N && lane * 16 < W) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 2 * W + lane * 16));
      const double delta = gp[i + 1] - gp[i];
      const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
      // x_next rows K[i+1][0] <= x + 2 delta u <= K[i+1][1]; x itself is not re-checked against the x box (below)
      if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = k0; }
      if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -k1; }
      double ulo, uhi;
      if (!u_bounds<RPL>(x, a, b, c, cmask, ru, rx, rc, ubox_lo, ubox_hi, ulo, uhi)) {
        // :99-104: the stage fails, us[i:] and xs[i+1:] are NaN; no retry rule in TOPPRAsd
        st = TB_STATUS_ERR_UNKNOWN;
        fstage = i;
        for (int j = i + 1 + lane; j < Gp; j += 32) xp[j] = nan_d;
        for (int j = i + lane; j < N; j += 32) up[j] = nan_d;
        break;
      }
      const double u = slow ? ulo : uhi;
      // :117 xs[i+1] = min(K[i+1,1], max(K[i+1,0], xs[i] + 2 deltas[i] us[i] - SMALL)), Python's min / max
      double x_next = x + 2 * delta * u - ALG_SMALL;
      x_next = (x_next > k0) ? x_next : k0;
      x_next = (x_next < k1) ? x_next : k1;
      if (lane == 0) { up[i] = u; xp[i + 1] = x_next; }
      x = x_next;
    }
  }
  if (!slow && lane == 0) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
  }
}

// One stage problem per warp (one warp per CTA): rows 0 / 1 are the optional x_next rows, rows 2.. the caller's n rows.
template <int RPL, bool PER_ROW>
__device__ __forceinline__ void socp_stage_body(
    const double *__restrict__ g, const double *__restrict__ ra, const double *__restrict__ rb,
    const double *__restrict__ rcst, const int n, const int conic0, const int conicn, Axes<RPL, PER_ROW> ru,
    Axes<RPL, PER_ROW> rx, Axes<RPL, PER_ROW> rc, const double *__restrict__ xbox, const double *__restrict__ xnext,
    const int B, double *__restrict__ out, const ConeTable *__restrict__ table, const double *__restrict__ ubox) {
  const int lane = threadIdx.x & 31;
  const long p = warp_path();
  if (p >= B) return;
  double a[RPL], b[RPL], c[RPL];
  unsigned cmask[RPL];
  double ubox_lo = VAR_MIN, ubox_hi = VAR_MAX;   // the u box ubox[p] (PER_ROW)
  if constexpr (PER_ROW) {
    load_cones<RPL>(table, n, lane, cmask, ru, rx, rc);
    if (ubox) { ubox_lo = ubox[2 * p]; ubox_hi = ubox[2 * p + 1]; }
  }
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r >= 2 && r < n + 2) {
      a[s] = ra[p * n + r - 2]; b[s] = rb[p * n + r - 2]; c[s] = rcst[p * n + r - 2];
      if constexpr (!PER_ROW) cmask[s] = (r - 2 >= conic0 && r - 2 < conic0 + conicn) ? 1u : 0u;
    } else {
      a[s] = 0.0; b[s] = 0.0; c[s] = -1.0;
      if constexpr (!PER_ROW) cmask[s] = 0u;
    }
  }
  const double delta = xnext ? xnext[3 * p] : __longlong_as_double(0x7ff8000000000000LL);
  if (delta == delta) {
    if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = xnext[3 * p + 1]; }
    if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -xnext[3 * p + 2]; }
  }
  double us, xs;
  socp_stage_solve<RPL>(g[2 * p], g[2 * p + 1], xbox[2 * p], xbox[2 * p + 1], a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, us, xs);
  if (lane == 0) { out[2 * p] = us; out[2 * p + 1] = xs; }
}

// compute_reachable_sets of a robust problem (reachability_algorithm.py:378-431), one warp per path: the forward
// recursion L[i+1] = _one_step_forward(i, L[i], X[i+1]) on the feasible sets X of a tb_scan_robust_ragged
// (TB_SCAN_FEASIBLE_SETS) launch.  Each end of L[i+1] is one socp_stage_solve: max / min x + 2 delta' u over stage i
// with L[i] in the x box and X[i+1] on the x_next rows (ecos_solverwrapper.py:90-207).  The reference's objective uses
// delta' = deltas[i - 1] (deltas[N - 1] at i = 0, Python's negative index) while the x_next rows use deltas[i], as in
// reachable_kernel (tb_scan.cu).  After a NaN end the remaining rows of L stay 0 (np.zeros).
template <int RPL, bool PER_ROW>
__device__ __forceinline__ void reachable_robust_body(
    const double *__restrict__ records, const int W, const int R, const int conic0, const int conicn,
    Axes<RPL, PER_ROW> ru, Axes<RPL, PER_ROW> rx, Axes<RPL, PER_ROW> rc, const double *__restrict__ grid,
    const int grid_shared, const int B, const int G, const int *__restrict__ glen, const double *__restrict__ X,
    const double *__restrict__ sdmin, const double *__restrict__ sdmax, double *__restrict__ Lout,
    int *__restrict__ fail_stage, const ConeTable *__restrict__ table, const bool ub) {
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
  double ubox_lo = VAR_MIN, ubox_hi = VAR_MAX;
  if constexpr (PER_ROW) load_cones<RPL>(table, R, lane, cmask, ru, rx, rc);
  for (int i = 0; i < N; ++i) {
    const double *rec = rec_path + (size_t)i * W;
    rload_rows<RPL, PER_ROW>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask, ub, ubox_lo, ubox_hi);
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
    socp_stage_solve<RPL>(-2 * dq, -1.0, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, u1, x1v);
    socp_stage_solve<RPL>(2 * dq, 1.0, xl, xh, a, b, c, cmask, lane, ru, rx, rc, ubox_lo, ubox_hi, u0, x0v);
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
