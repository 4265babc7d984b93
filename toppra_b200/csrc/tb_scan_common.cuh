// tb_scan_common.cuh — helpers shared by the scan kernels (tb_scan.cu: one warp per path; tb_scan_pair.cu: two paths per
// warp): Seidel's row order (cy_seidel_solverwrapper.pyx:252-264), the shortcut thresholds, Python's min/max.
#pragma once
#include <limits.h>

#include "tb_common.cuh"

namespace tb {

// Position of LP row r in Seidel's processing order, cy_seidel_solverwrapper.pyx:252-264:
// a valid warm-start pair puts active_c[1] first, active_c[0] second, then the remaining rows ascending.
static __device__ __forceinline__ int row_pos(int r, bool valid, int ac0, int ac1) {
  if (!valid) return r;
  if (r == ac1) return 0;
  if (r == ac0) return 1;
  return 2 + r - (r > ac0 ? 1 : 0) - (r > ac1 ? 1 : 0);
}
static __device__ __forceinline__ int pos_row(int p, bool valid, int ac0, int ac1) {
  if (!valid) return p;
  if (p == 0) return ac1;
  if (p == 1) return ac0;
  const int lo = min(ac0, ac1), hi = max(ac0, ac1);
  int r = p - 2;
  if (r >= lo) ++r;
  if (r >= hi) ++r;
  return r;
}

// Identity the optimiser cannot see through: keeps a sanitised division operand from being folded back into the
// original one when the quotient is later replaced by a select (the compiler would divide the raw value again).
static __device__ __forceinline__ double opaque(double v) {
  asm volatile("" : "+d"(v));
  return v;
}

// Python's builtin max(a, b) / min(a, b) on floats (reachability_algorithm.py:324-354): a unless b compares beyond it
static __device__ __forceinline__ double py_max(const double a, const double b) { return (b > a) ? b : a; }
static __device__ __forceinline__ double py_min(const double a, const double b) { return (b < a) ? b : a; }

constexpr int BOXBASE = 1 << 20;
constexpr double SKIP_GAP = 1e-7;   // shortcuts A/B: required violation, relative to the terms' magnitudes (TINY = 1e-10)
constexpr double SKIP_BIG = 1e300;
constexpr double SKIP_TMAX = 90.0;  // shortcut A: largest line parameter of a skipped visit (see lp2d_impl)

// Row source of the fused vel+acc scans (tb_scan_velacc): the path's spline, the acceleration limits and the velocity bound.
struct VelAccSrc {
  const double *ppoly;   // [B][4][nseg][dof]
  const double *breaks;  // [nseg+1] or [B][nseg+1]
  const double *alim;    // [dof][2] or [B][dof][2]
  const double *xbound;  // [B][G][2]
  int breaks_shared, nseg, dof, lim_shared;
};


// launcher of the two-paths-per-warp build (tb_scan_pair.cu); returns TB_ERR_UNSUPPORTED when the problem does not fit
int launch_scan_velacc_pair(const VelAccSrc &src, int interp, const double *grid, int grid_shared, int B, int G,
                            const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                            double *sd, double *u, int *status, int *fail_stage, cudaStream_t stream);
bool scan_velacc_pair_supported(int dof, int interp, int nseg, int flags);

// forward pass with one thread per path (tb_scan_fwd.cu), for large batches: reads K / status / fail_stage of a
// TB_SCAN_BACKWARD_ONLY launch
#ifndef TB_SCAN_FWD_THREADS_MIN_DEFAULT
// smallest batch (paths) that takes the thread-per-path forward pass.  H100 80GB (400 W), 7-DOF, 200 gridpoints, fused
// scan: 16384 paths 5.17 vs 5.36 ms (warp form), 24576: 7.33 vs 7.95 ms, 32768: 9.40 vs 10.96 ms
#define TB_SCAN_FWD_THREADS_MIN_DEFAULT 16384
#endif
bool forward_threads_supported(int dof, int B);
int launch_forward_threads(const VelAccSrc &src, int interp, const double *grid, int grid_shared, int B, int G,
                           const double *sd_start, const double *K, double *sd, double *u, int *status, int *fail_stage,
                           cudaStream_t stream);

}  // namespace tb
