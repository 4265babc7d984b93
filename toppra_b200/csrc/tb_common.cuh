// tb_common.cuh — shared constants and helpers of libtoppra_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/toppra_b200.h"

namespace tb {

// LP layer constants: toppra/solverwrapper/cy_seidel_solverwrapper.pyx:17-29
constexpr double LP_TINY = 1e-10;
constexpr double LP_SMALL = 1e-8;
constexpr double VAR_MIN = -100000000.0;
constexpr double VAR_MAX = 100000000.0;
constexpr double LP_INF = 10000000000.0;
// algorithm layer constants: toppra/constants.py:16-17,24,32,42
constexpr double ALG_TINY = 1e-8;
constexpr double ALG_SMALL = 1e-5;
constexpr int MAX_TRIES = 10;
constexpr double JVEL_MAXSD = 1e8;
constexpr double CVXPY_MAXX = 10000.0;

constexpr int MAX_ROWS = 126;   // R <= 126 -> nC = R + 2 <= 128 = 4 rows per lane

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ int find_interval(const double *__restrict__ x, const int nseg, const double s) {
  // scipy _ppoly.pyx find_interval: x[j] <= s < x[j+1]; s == x[-1] -> last interval; out of range -> end intervals
  if (!(s == s)) return -1;
  if (s < x[0]) return 0;
  if (s >= x[nseg]) return nseg - 1;
  int lo = 0, hi = nseg;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (s >= x[mid]) lo = mid; else hi = mid;
  }
  return lo;
}

// q^(order)(s) for one (segment, dof): derivative coefficients then res += c*z, z *= ds  (scipy evaluate_poly1)
__device__ __forceinline__ double ppoly_eval1(const double *__restrict__ c, const int nseg, const int dof,
                                              const int seg, const int k, const double ds, const int order) {
  const double c0 = c[(0 * nseg + seg) * dof + k], c1 = c[(1 * nseg + seg) * dof + k];
  const double c2 = c[(2 * nseg + seg) * dof + k];
  double res, z;
  if (order == 0) {
    const double c3 = c[(3 * nseg + seg) * dof + k];
    res = 0.0 + c3; z = ds;
    res = res + c2 * z; z = z * ds;
    res = res + c1 * z; z = z * ds;
    res = res + c0 * z;
  } else if (order == 1) {
    const double d0 = c0 * 3.0, d1 = c1 * 2.0, d2 = c2 * 1.0;
    res = 0.0 + d2; z = ds;
    res = res + d1 * z; z = z * ds;
    res = res + d0 * z;
  } else {
    const double e0 = (c0 * 3.0) * 2.0, e1 = (c1 * 2.0) * 1.0;
    res = 0.0 + e1; z = ds;
    res = res + e0 * z;
  }
  return res;
}

void set_error(const char *fmt, ...);
int check_launch(const char *what);
// multiprocessor count of the current device (132 on an H100 SXM): sizes grid-stride launches and one-wave batches
int num_sms();

}  // namespace tb
