// tb_common.cuh — shared constants and helpers of libtoppra_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

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

// Calls f(std::integral_constant<int, RPL>{}) with the LP rows per lane of a one-warp kernel for nC rows: RPL = 1..4,
// lane `lane` holds rows lane + 32 * s, s < RPL.  nC <= MAX_ROWS + 2 (checked by the caller).
template <class F>
auto with_rows_per_lane(const int nC, F &&f) {
  if (nC <= 32) return f(std::integral_constant<int, 1>{});
  if (nC <= 64) return f(std::integral_constant<int, 2>{});
  if (nC <= 96) return f(std::integral_constant<int, 3>{});
  return f(std::integral_constant<int, 4>{});
}

constexpr unsigned FULL = 0xffffffffu;

// Warp-wide min / max of doubles (no NaNs) with two 32-bit redux.sync each instead of five shuffle rounds.
// Order-preserving map double -> (khi, klo): flip all bits of negative numbers, the sign bit of the others; then
// reduce the high words, and the low words among the lanes that tie on the high word.
__device__ __forceinline__ double warp_min(double v) {
  const int hi = __double2hiint(v), lo = __double2loint(v);
  const int m = hi >> 31;  // 0 or -1
  const unsigned khi = (unsigned)(hi ^ (m | (int)0x80000000)), klo = (unsigned)(lo ^ m);
  const unsigned mh = __reduce_min_sync(FULL, khi);
  const unsigned ml = __reduce_min_sync(FULL, khi == mh ? klo : 0xffffffffu);
  const int m2 = ((int)~mh) >> 31;  // -1 if the winner is negative
  return __hiloint2double((int)(mh ^ (unsigned)(m2 | (int)0x80000000)), (int)(ml ^ (unsigned)m2));
}
__device__ __forceinline__ double warp_max(double v) {
  const int hi = __double2hiint(v), lo = __double2loint(v);
  const int m = hi >> 31;
  const unsigned khi = (unsigned)(hi ^ (m | (int)0x80000000)), klo = (unsigned)(lo ^ m);
  const unsigned mh = __reduce_max_sync(FULL, khi);
  const unsigned ml = __reduce_max_sync(FULL, khi == mh ? klo : 0u);
  const int m2 = ((int)~mh) >> 31;
  return __hiloint2double((int)(mh ^ (unsigned)(m2 | (int)0x80000000)), (int)(ml ^ (unsigned)m2));
}

// Path (or LP) of a one-warp CTA of feasible_kernel, reachable_kernel, lp2d_batch_kernel and scan_robust_kernel:
// blockIdx.x.  The term threadIdx.x >> 5 is 0, but it keeps the index per-thread for the compiler: as a uniform value,
// ptxas moves the per-path addressing to the uniform datapath, and the machine code of these kernels changes
// (reachable_kernel<4> then spills 20-32 bytes).
__device__ __forceinline__ long warp_path() { return (long)blockIdx.x + (int)(threadIdx.x >> 5); }

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

// CTAs of a grid-stride launch over `total` items: one item per thread, at most per_sm CTAs per multiprocessor.
inline long grid_stride_blocks(const long total, const int threads, const int per_sm) {
  const long blocks = (total + threads - 1) / threads;
  return blocks > (long)num_sms() * per_sm ? (long)num_sms() * per_sm : blocks;
}

// check_launch for the companion libraries.  Each library carries its own static CUDA runtime, and cudaGetLastError
// sees only the launches made through it, so each companion reads its launch errors here, through the copy compiled
// into it (static: a call is never bound to another library's copy), not through libtoppra_b200.so's check_launch.
static inline int launch_status(const char *what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

}  // namespace tb
