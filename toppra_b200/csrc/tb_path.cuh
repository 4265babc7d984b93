// tb_path.cuh — sampling a batch of paths in scipy's PPoly layout ([kc][nseg][dof] coefficients per path), shared by
// the cubic kernels of libtoppra_b200.so and the order-k kernels of libtoppra_b200_poly.so.
//
// A path evaluator has kc(): the coefficients per piece, and eval(c, nseg, dof, seg, k, ds, order):
// q_k^(order)(x[seg] + ds) of one path's coefficients c, order 0..2.  CubicPath is the spline's (ppoly_eval1);
// tb_poly.cu has PolyPath for k <= TBP_MAX_COEFFS.  The bodies below are templates over it; every kernel that runs
// one is a plain __global__ wrapper that passes its own evaluator.
#pragma once
#include "tb_common.cuh"

namespace tb {

struct CubicPath {
  __device__ __forceinline__ int kc() const { return 4; }
  __device__ __forceinline__ double eval(const double *c, const int nseg, const int dof, const int seg, const int k,
                                         const double ds, const int order) const {
    return ppoly_eval1(c, nseg, dof, seg, k, ds, order);
  }
};

// path(s, order) (interpolator.py:423-430 for the cubic; the same scipy calls for any order): one thread per
// (path, position, joint), NaN where s has no piece.
template <class Path>
__device__ __forceinline__ void path_eval(const Path path, const double *__restrict__ ppoly,
                                          const double *__restrict__ breaks, const int breaks_shared, const long B,
                                          const int nseg, const int dof, const double *__restrict__ s,
                                          const int s_shared, const int G, const int order, double *__restrict__ out) {
  const long total = B * G * dof;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % dof);
    const long pg = idx / dof;
    const int gi = (int)(pg % G);
    const long p = pg / G;
    const double *x = breaks + (breaks_shared ? 0 : p * (nseg + 1));
    const double sv = s[(s_shared ? 0 : p * G) + gi];
    const int seg = find_interval(x, nseg, sv);
    double r;
    if (seg < 0) r = __longlong_as_double(0x7ff8000000000000LL);
    else r = path.eval(ppoly + p * path.kc() * nseg * dof, nseg, dof, seg, k, sv - x[seg], order);
    out[idx] = r;
  }
}

// ParametrizeConstAccel output (parametrizer.py:82-129): q | q'v | q''v^2 + q'u at the times ts, one thread per
// (path, sample, joint).  t_grid, sd, us are tb_time_grid's knot times, speeds and stage accelerations.
template <class Path>
__device__ __forceinline__ void constaccel_eval(const Path path, const double *__restrict__ ppoly,
                                               const double *__restrict__ breaks, const int breaks_shared,
                                               const int nseg, const int dof, const double *__restrict__ grid,
                                               const int grid_shared, const double *__restrict__ sd,
                                               const double *__restrict__ t_grid, const double *__restrict__ us,
                                               const long B, const int G, const double *__restrict__ ts,
                                               const int ts_shared, const int M, const int order,
                                               double *__restrict__ out) {
  const long total = B * M * dof;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % dof);
    const long pm = idx / dof;
    const int m = (int)(pm % M);
    const long p = pm / M;
    const double t = ts[(ts_shared ? 0 : p * M) + m];
    const double *tg = t_grid + p * G;
    // np.searchsorted(tg, t, side="right") - 1, then idx == len(us) -> idx - 1   (parametrizer.py:117-121)
    int lo = 0, hi = G;  // first index with tg[j] > t
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (tg[mid] <= t) lo = mid + 1; else hi = mid;
    }
    int i = lo - 1;
    if (i == G - 1) i = G - 2;
    // t before the start: the reference indexes with -1, i.e. the LAST entry of each array (knot time, speed and
    // position at the end, the last stage's acceleration: parametrizer.py:115-128)
    const int it = i < 0 ? G - 1 : i, iu = i < 0 ? G - 2 : i;
    const double *sg = grid + (grid_shared ? 0 : p * G);
    const double dt = t - tg[it];
    const double u = us[p * (G - 1) + iu];
    const double v0 = sd[p * G + it];
    const double v = v0 + dt * u;
    const double s = sg[it] + dt * v0 + 0.5 * (dt * dt) * u;
    const double *x = breaks + (breaks_shared ? 0 : p * (nseg + 1));
    const double *c = ppoly + p * path.kc() * nseg * dof;
    const int seg = find_interval(x, nseg, s);
    double r;
    if (seg < 0) {
      r = __longlong_as_double(0x7ff8000000000000LL);
    } else {
      const double ds = s - x[seg];
      if (order == 0) r = path.eval(c, nseg, dof, seg, k, ds, 0);
      else if (order == 1) r = path.eval(c, nseg, dof, seg, k, ds, 1) * v;
      else r = path.eval(c, nseg, dof, seg, k, ds, 2) * (v * v) + path.eval(c, nseg, dof, seg, k, ds, 1) * u;
    }
    out[idx] = r;
  }
}

}  // namespace tb
