// tb_propose.cuh — the propose_gridpoints passes of one path on one warp, shared by tb_frows.cu (cubic paths) and
// tb_poly.cu (order-k paths).  The two callers differ only in how they evaluate q''.
//
// Replaces (reference) propose_gridpoints, toppra/interpolator.py:49-122.  A pass visits every segment of the current
// (sorted) list; a segment longer than max_seg_length, or whose estimated interpolation error
// 0.5 * max_k |q_k''(mid)| * len^2 exceeds the threshold, gets its midpoint inserted (the reference appends and sorts:
// the same list).  Lanes take segments 32 at a time; the output position of a segment is its index plus the number of
// insertions before it (ballot + popc prefix).
#pragma once
#include "tb_common.cuh"

namespace tb {

// `qdd` has kc(): the coefficients per piece, and qdd(c, nseg, dof, seg, k, ds): q_k''(x[seg] + ds) of the piece
// coefficients c of one path.  The parameters are those of the kernels, which call this with blockIdx.x / threadIdx.x.
template <class Qdd>
__device__ __forceinline__ void propose_gridpoints_warp(const double *__restrict__ ppoly,
                                                        const double *__restrict__ breaks, const int breaks_shared,
                                                        const int B, const int nseg, const int dof, const double max_err,
                                                        const int max_iter, const double max_seg, const int min_pts,
                                                        const int Gmax, double *__restrict__ grid_out,
                                                        double *__restrict__ scratch, int *__restrict__ glen,
                                                        int *__restrict__ status, const Qdd qdd) {
  const int p = blockIdx.x, lane = threadIdx.x;
  if (p >= B) return;
  const double *x = breaks + (breaks_shared ? 0 : (size_t)p * (nseg + 1));
  const double *c = ppoly + (size_t)p * qdd.kc() * nseg * dof;
  double *cur = grid_out + (size_t)p * Gmax, *nxt = scratch + (size_t)p * Gmax;
  int n = 2, st = 0;
  if (lane == 0) { cur[0] = x[0]; cur[1] = x[nseg]; }   // path.path_interval
  __syncwarp();
  bool converged = false;
  int it = 0;
  for (; it < max_iter; ++it) {
    int base = 0;      // insertions before the current block of 32 segments
    bool any = false;
    const int nsegs = n - 1;
    for (int s0 = 0; s0 < nsegs; s0 += 32) {
      const int idx = s0 + lane;
      bool add = false;
      double lo = 0.0, mid = 0.0;
      if (idx < nsegs) {
        lo = cur[idx];
        const double hi = cur[idx + 1];
        mid = 0.5 * (lo + hi);
        const double dist = hi - lo;
        if (dist > max_seg) {
          add = true;
        } else {
          const int seg = find_interval(x, nseg, mid);
          const double d2 = dist * dist;
          double worst = -1.0;
          bool isnan_any = false;
          for (int k = 0; k < dof; ++k) {
            const double e = fabs((0.5 * qdd(c, nseg, dof, seg < 0 ? 0 : seg, k, mid - x[seg < 0 ? 0 : seg])) * d2);
            isnan_any = isnan_any || (e != e);
            worst = (e > worst) ? e : worst;
          }
          // np.max propagates NaN, and NaN > threshold is False
          add = !isnan_any && (worst > max_err);
        }
      }
      const unsigned m = __ballot_sync(FULL, add);
      const int pos = idx + base + __popc(m & ((1u << lane) - 1u));
      if (idx < nsegs) {
        if (pos < Gmax) nxt[pos] = lo;
        if (add && pos + 1 < Gmax) nxt[pos + 1] = mid;
      }
      base += __popc(m);
      any = any || (m != 0u);
    }
    const int n_new = n + base;
    if (n_new > Gmax) { st = TB_ERR_UNSUPPORTED; break; }
    if (lane == 0) nxt[n_new - 1] = cur[n - 1];
    __syncwarp();
    if (!any) { converged = true; break; }
    { double *t = cur; cur = nxt; nxt = t; }
    n = n_new;
  }
  // interpolator.py:119-120: `iteration == max_iteration - 1` after the loop means the last allowed pass ran — whether
  // or not it still inserted points — and raises "Unable to find a good gridpoint for this path."
  if (st == 0 && (!converged || it == max_iter - 1)) st = 1;
  // interpolator.py:111-117: double the resolution until there are at least min_nb_points
  while (st == 0 && n < min_pts) {
    const int n_new = 2 * n - 1;
    if (n_new > Gmax) { st = TB_ERR_UNSUPPORTED; break; }
    for (int idx = lane; idx < n - 1; idx += 32) {
      const double lo = cur[idx], hi = cur[idx + 1];
      nxt[2 * idx] = lo;
      nxt[2 * idx + 1] = 0.5 * (lo + hi);
    }
    if (lane == 0) nxt[n_new - 1] = cur[n - 1];
    __syncwarp();
    { double *t = cur; cur = nxt; nxt = t; }
    n = n_new;
  }
  // result into grid_out, tail padded with the end of the path (finite values for the padded coefficient columns)
  double *out = grid_out + (size_t)p * Gmax;
  const double last = cur[n - 1];
  if (cur != out)
    for (int j = lane; j < n; j += 32) out[j] = cur[j];
  for (int j = n + lane; j < Gmax; j += 32) out[j] = last;
  if (lane == 0) { glen[p] = n; status[p] = st; }
}

}  // namespace tb
