// tb_scan_fwd.cu — forward pass of the fused vel+acc scan with ONE THREAD PER PATH, for large batches.
//
// Replaces (reference): ReachabilityAlgorithm.compute_parameterization's forward loop (reachability_algorithm.py:303-365),
// TOPPRA._forward_step (time_optimal_algorithm.py:55-92) and the 1-variable branch of
// seidelWrapper.solve_stagewise_optim / cy_solve_lp1d (cy_seidel_solverwrapper.pyx:631-650, 93-144) — the same functions as
// the forward half of scan_kernel in tb_scan.cu, with identical results.
//
// Why a second form: a large batch (BASELINE cfg 5) is bound by instruction issue, and the forward stage is one 1-variable
// LP: its only collective is a min / max over the rows.  One warp per path spends ~200 issue slots per stage on it
// (row prologue, one division, two redux, vote); a thread that walks its path's 30 rows alone needs ~1000 instructions
// per stage, but a warp then serves 32 paths: ~30 issue slots per path and stage.  Small batches stay on the warp kernel
// (a 4096-path batch would be 128 warps of pure latency).  Launched after a TB_SCAN_BACKWARD_ONLY launch of scan_kernel,
// whose K / status / fail_stage it reads.
//
// Exactness: the rows are K1's arithmetic (scipy evaluate_poly1 on the derivative coefficients, interpolation lift); the
// values at s_{i+1} of stage i are carried into stage i+1 (the warp kernel recomputes the same numbers); the negated copies
// use exact IEEE negation: (-b) x + c = -(b x) + c and -bxc / (-a) = bxc / a; min / max over the rows is order-independent.
#include "tb_scan_common.cuh"

namespace tb {
namespace {

constexpr int FWD_THREADS = 128;

// one +- slab of the 1-variable LP at fixed x: row P: a u + (b x + cP) <= 0, row N: -a u + (-(b x) + cN) <= 0 (pyx:633-641)
__device__ __forceinline__ void fwd_slab(const double a, const double b, const double cP, const double cN, const double x,
                                         double &hi, double &lo) {
  const double bx = b * x;
  const double bxcP = bx + cP, bxcN = -bx + cN;
  if (a > LP_TINY) {            // P bounds u from above, N (coefficient -a) from below
    const double tP = -bxcP / a, tN = bxcN / a;
    hi = (tP < hi) ? tP : hi;
    lo = (tN > lo) ? tN : lo;
  } else if (a < -LP_TINY) {    // the other way round
    const double tP = -bxcP / a, tN = bxcN / a;
    lo = (tP > lo) ? tP : lo;
    hi = (tN < hi) ? tN : hi;
  }
}

template <int DOF>
__global__ void __launch_bounds__(FWD_THREADS)
forward_threads_kernel(const VelAccSrc src, const int interp, const double *__restrict__ grid, const int grid_shared,
                       const int B, const int G, const double *__restrict__ sd_start, const double *__restrict__ Kin,
                       double *__restrict__ sdout, double *__restrict__ uout, int *__restrict__ status,
                       int *__restrict__ fail_stage) {
  const long p = (long)blockIdx.x * FWD_THREADS + threadIdx.x;
  if (p >= B) return;
  const int N = G - 1, nseg = src.nseg;
  const double *gp = grid + (grid_shared ? 0 : (size_t)p * G);
  const double *Kp = Kin + (size_t)p * G * 2;
  double *sdp = sdout + (size_t)p * G;
  double *up = uout + (size_t)p * (G > 1 ? G - 1 : 0);
  const double *cpp = src.ppoly + (size_t)p * 4 * nseg * DOF;
  const double *xb = src.breaks + (src.breaks_shared ? 0 : (size_t)p * (nseg + 1));
  const double *al = src.alim + (src.lim_shared ? 0 : (size_t)p * DOF * 2);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  int st = status[p], fs = fail_stage ? fail_stage[p] : -1;
  const double sds = sd_start ? sd_start[p] : 0.0;
  const double x_start = sds * sds;
  if (st == TB_STATUS_OK) {
    // admissibility of the start velocity, reachability_algorithm.py:290-301
    if (x_start + ALG_SMALL < Kp[0] || Kp[1] + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fs = 0; }
  }
  if (st != TB_STATUS_OK) {
    for (int j = 0; j < G; ++j) sdp[j] = nan_d;
    for (int j = 0; j < N; ++j) up[j] = nan_d;
    status[p] = st;
    if (fail_stage) fail_stage[p] = fs;
    return;
  }
  double cP[DOF], cN[DOF];
#pragma unroll
  for (int k = 0; k < DOF; ++k) {
    cP[k] = 0.0 - al[k * 2 + 1];          // F c - g with c = 0, g = [amax; -amin]
    cN[k] = 0.0 - (-al[k * 2 + 0]);
  }
  // derivative coefficients of the current segment (scipy PPoly.derivative: c'[j] = c[j] (k - j))
  double d0[DOF], d1[DOF], d2[DOF], e0[DOF], e1[DOF];
  int seg = 0;
  double seg_x0 = xb[0], seg_x1 = xb[1];     // breakpoints of the current segment [x0, x1)
  auto load_seg = [&]() {
#pragma unroll
    for (int k = 0; k < DOF; ++k) {
      const double c0 = cpp[(0 * nseg + seg) * DOF + k], c1 = cpp[(1 * nseg + seg) * DOF + k];
      const double c2 = cpp[(2 * nseg + seg) * DOF + k];
      d0[k] = c0 * 3.0; d1[k] = c1 * 2.0; d2[k] = c2 * 1.0;
      e0[k] = d0[k] * 2.0; e1[k] = d1[k] * 1.0;
    }
    seg_x0 = xb[seg];
    seg_x1 = xb[seg + 1];
  };
  // q'(s), q''(s): find_interval's index is monotone in s, so it is carried (a NaN gridpoint leaves it alone)
  auto eval_at = [&](const double s, double (&v1)[DOF], double (&v2)[DOF]) {
    if (seg < nseg - 1 && s >= seg_x1) {
      while (seg < nseg - 1 && s >= xb[seg + 1]) ++seg;
      load_seg();
    }
    const double ds = s - seg_x0;
#pragma unroll
    for (int k = 0; k < DOF; ++k) {
      double z = ds;
      double a1 = 0.0 + d2[k];
      a1 = a1 + d1[k] * z;
      z = z * ds;
      a1 = a1 + d0[k] * z;
      double a2 = 0.0 + e1[k];
      a2 = a2 + e0[k] * ds;
      v1[k] = a1;
      v2[k] = a2;
    }
  };
  load_seg();
  double c1v[DOF], c2v[DOF], n1v[DOF], n2v[DOF];   // q', q'' at s_i and at s_{i+1}
  eval_at(gp[0], c1v, c2v);
  double x = x_start;
  int i = 0;
  for (; i < N; ++i) {
    const double g0 = gp[i], g1 = gp[i + 1];
    const double delta = g1 - g0;
    eval_at(g1, n1v, n2v);
    const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
    const double v0 = -(-2 * delta);          // _forward_step: g = (-2 delta, -1) -> v0 = 2 delta (pyx:628-636)
    const bool pick_min = (fabs(v0) < LP_TINY) || (v0 < 0);
    int tries = 0;
    bool ok;
    double uopt = 0.0;
    while (true) {
      double hi = VAR_MAX, lo = VAR_MIN;
      // rows 0 / 1 (pyx:604-620): (-2 delta, -1, x_next_min), (2 delta, 1, -x_next_max)
      fwd_slab(2 * delta, 1.0, -k1, k0, x, hi, lo);
#pragma unroll
      for (int k = 0; k < DOF; ++k) {
        fwd_slab(c1v[k], c2v[k], cP[k], cN[k], x, hi, lo);
        if (interp) fwd_slab(n1v[k] + (2 * delta) * n2v[k], n2v[k], cP[k], cN[k], x, hi, lo);  // lift, linear_constraint.py:170
      }
      ok = !(lo > hi);                          // cy_solve_lp1d: infeasible iff cur_min > cur_max (pyx:126-128)
      uopt = pick_min ? lo : hi;
      if (ok || tries >= MAX_TRIES) break;
      x = py_max(x - ALG_TINY, 0.999 * x);    // reachability_algorithm.py:324-327
      ++tries;
    }
    sdp[i] = sqrt(x);                           // x_i is final now (the retry rule may have shrunk it)
    if (!ok) {
      // :337-342: xs[i+1:] = nan -> sd NaN -> ErrUnknown; us stay 0
      st = TB_STATUS_ERR_UNKNOWN;
      fs = i;
      for (int j = i + 1; j < G; ++j) sdp[j] = nan_d;
      for (int j = i; j < N; ++j) up[j] = 0.0;
      break;
    }
    double x_next = x + 2 * delta * uopt;                        // :352
    x_next = py_max(x_next - ALG_TINY, 0.9999 * x_next);         // :353
    x_next = py_min(k1, py_max(k0, x_next));                     // :354
    up[i] = uopt;
    x = x_next;
#pragma unroll
    for (int k = 0; k < DOF; ++k) { c1v[k] = n1v[k]; c2v[k] = n2v[k]; }
  }
  if (st == TB_STATUS_OK) sdp[N] = sqrt(x);
  status[p] = st;
  if (fail_stage) fail_stage[p] = fs;
}

}  // namespace

bool forward_threads_supported(int dof, int B) { return dof >= 1 && dof <= 8 && B >= FWD_THREADS_MIN; }

int launch_forward_threads(const VelAccSrc &src, int interp, const double *grid, int grid_shared, int B, int G,
                           const double *sd_start, const double *K, double *sd, double *u, int *status, int *fail_stage,
                           cudaStream_t stream) {
  const int blocks = (B + FWD_THREADS - 1) / FWD_THREADS;
#define TB_FWD(D) \
  case D: forward_threads_kernel<D><<<blocks, FWD_THREADS, 0, stream>>>(src, interp, grid, grid_shared, B, G, sd_start, K, sd, u, \
                                                                       status, fail_stage); break
  switch (src.dof) {
    TB_FWD(1); TB_FWD(2); TB_FWD(3); TB_FWD(4); TB_FWD(5); TB_FWD(6); TB_FWD(7); TB_FWD(8);
    default: set_error("tb_scan_velacc: forward_threads_kernel supports dof <= 8"); return TB_ERR_UNSUPPORTED;
  }
#undef TB_FWD
  return check_launch("tb_scan_velacc");
}

}  // namespace tb
