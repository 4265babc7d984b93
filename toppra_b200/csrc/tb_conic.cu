// tb_conic.cu — libtoppra_b200_robust.so: the TOPPRAsd forward passes and single stage solves of robust (conic)
// problems.  C-ABI in include/toppra_b200_robust.h.
//
// The reference runs TOPPRAsd (desired_duration_algorithm.py:42-234) and solve_stagewise_optim on a conic problem
// through ecosWrapper.solve_stagewise_optim (ecos_solverwrapper.py:90-207).  Both solve the same two-variable stage
// problems as K2r (tb_robust.cu), with the primitives of tb_robust_common.cuh:
//   sd_forward_robust_kernel  the fastest and the slowest forward pass on the controllable sets K of a backward-only
//                             tb_scan_robust_ragged launch: at stage i x is fixed, so the stage problem is the
//                             u-interval at x, and the fastest pass takes u = uhi(x), the slowest u = ulo(x);
//   socp_stage_kernel         min g0 u + g1 x over one stage: the feasible x-interval by extreme_x, then the convex
//                             phi(x) = g1 x + g0 (g0 < 0 ? uhi(x) : ulo(x)) by golden-section search on it
//                             (socp_stage_solve, tb_robust_common.cuh).
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error).  Each library
// carries its own static CUDA runtime, so launch errors are read here (launch_status).
#include "tb_robust_common.cuh"
#include "../../include/toppra_b200_robust.h"

namespace tb {
namespace {

// One warp per (path, pass), one warp per CTA: blockIdx.x = 2 path + (0 fastest, 1 slowest).  The rules are those of
// desired_duration_algorithm.py:87-121 (the slowest pass :207-234), on the conventions of tb_scan_ex with
// TB_SCAN_SD_FORWARD: x out holds x = sd^2, status / fail_stage are the fastest pass's.
template <int RPL>
__global__ void __launch_bounds__(32)
sd_forward_robust_kernel(const double *__restrict__ records, const int W, const int R, const int conic0,
                         const int conicn, const double ru, const double rx, const double rc,
                         const double *__restrict__ grid, const int grid_shared, const int B, const int G,
                         const int *__restrict__ glen, const double *__restrict__ K, const int *__restrict__ status_in,
                         const double *__restrict__ sd_start, double *__restrict__ x_fast, double *__restrict__ u_fast,
                         double *__restrict__ x_slow, double *__restrict__ u_slow, int *__restrict__ status,
                         int *__restrict__ fail_stage) {
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
    for (int i = 0; i < N; ++i) {
      const double *rec = rec_path + (size_t)i * W;
      rload_rows<RPL>(rec, R, nC, lane, conic0, conicn, a, b, c, cmask);
      if (i + 2 < N && lane * 16 < W) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec + 2 * W + lane * 16));
      const double delta = gp[i + 1] - gp[i];
      const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
      // x_next rows K[i+1][0] <= x + 2 delta u <= K[i+1][1]; x itself is not re-checked against the x box (below)
      if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = k0; }
      if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -k1; }
      double ulo, uhi;
      if (!u_bounds<RPL>(x, a, b, c, cmask, ru, rx, rc, ulo, uhi)) {
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
template <int RPL>
__global__ void __launch_bounds__(32)
socp_stage_kernel(const double *__restrict__ g, const double *__restrict__ ra, const double *__restrict__ rb,
                  const double *__restrict__ rcst, const int n, const int conic0, const int conicn, const double ru,
                  const double rx, const double rc, const double *__restrict__ xbox, const double *__restrict__ xnext,
                  const int B, double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long p = warp_path();
  if (p >= B) return;
  double a[RPL], b[RPL], c[RPL];
  unsigned cmask[RPL];
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r >= 2 && r < n + 2) {
      a[s] = ra[p * n + r - 2]; b[s] = rb[p * n + r - 2]; c[s] = rcst[p * n + r - 2];
      cmask[s] = (r - 2 >= conic0 && r - 2 < conic0 + conicn) ? 1u : 0u;
    } else {
      a[s] = 0.0; b[s] = 0.0; c[s] = -1.0; cmask[s] = 0u;
    }
  }
  const double delta = xnext ? xnext[3 * p] : __longlong_as_double(0x7ff8000000000000LL);
  if (delta == delta) {
    if (lane == 0) { a[0] = -2 * delta; b[0] = -1.0; c[0] = xnext[3 * p + 1]; }
    if (lane == 1) { a[0] = 2 * delta; b[0] = 1.0; c[0] = -xnext[3 * p + 2]; }
  }
  double us, xs;
  socp_stage_solve<RPL>(g[2 * p], g[2 * p + 1], xbox[2 * p], xbox[2 * p + 1], a, b, c, cmask, lane, ru, rx, rc, us, xs);
  if (lane == 0) { out[2 * p] = us; out[2 * p + 1] = xs; }
}

}  // namespace
}  // namespace tb

extern "C" int tbr_version(void) { return TBR_VERSION; }

extern "C" int tbr_sd_forward_robust(const double *records, int W, int R, int conic_row0, int conic_rows,
                                     const double *ellipsoid_host3, const double *grid, int grid_shared, int B, int G,
                                     const int *glen, const double *K, const int *status_in, const double *sd_start,
                                     double *x_fast, double *u_fast, double *x_slow, double *u_slow, int *status,
                                     int *fail_stage, void *stream) {
  using namespace tb;
  if (!records || !grid || !ellipsoid_host3 || !K || !status_in || !x_fast || !x_slow || !status || B <= 0 || G <= 0 ||
      R < 0 || (G > 1 && (!u_fast || !u_slow))) {
    set_error("tbr_sd_forward_robust: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tbr_sd_forward_robust: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (W < 3 * R + 2) { set_error("tbr_sd_forward_robust: record stride W=%d < 3R+2", W); return TB_ERR_ALIGN; }
  if (const int rc = check_conic(R, conic_row0, conic_rows, ellipsoid_host3, "tbr_sd_forward_robust")) return rc;
  if (B > 0x3fffffff) { set_error("tbr_sd_forward_robust: batch too large for one launch"); return TB_ERR_UNSUPPORTED; }
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(R + 2, [&](auto rpl) {
    sd_forward_robust_kernel<rpl.value><<<2 * B, 32, 0, (cudaStream_t)stream>>>(
        records, W, R, conic_row0, conic_rows, ru, rx, rc, grid, grid_shared, B, G, glen, K, status_in, sd_start, x_fast,
        u_fast, x_slow, u_slow, status, fail_stage);
  });
  return launch_status("tbr_sd_forward_robust");
}

extern "C" int tbr_socp_stage_batch(const double *g, const double *a, const double *b, const double *c, int n,
                                    int conic_row0, int conic_rows, const double *ellipsoid_host3, const double *xbox,
                                    const double *xnext, int B, double *optvar, void *stream) {
  using namespace tb;
  if (!g || !ellipsoid_host3 || !xbox || !optvar || B <= 0 || n < 0 || (n > 0 && (!a || !b || !c))) {
    set_error("tbr_socp_stage_batch: bad argument");
    return TB_ERR_ARG;
  }
  if (const int rc = check_conic(n, conic_row0, conic_rows, ellipsoid_host3, "tbr_socp_stage_batch")) return rc;
  const double ru = ellipsoid_host3[0], rx = ellipsoid_host3[1], rc = ellipsoid_host3[2];
  with_rows_per_lane(n + 2, [&](auto rpl) {
    socp_stage_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(g, a, b, c, n, conic_row0, conic_rows, ru, rx, rc,
                                                                     xbox, xnext, B, optvar);
  });
  return launch_status("tbr_socp_stage_batch");
}
