// tb_param.cu — K3: output trajectory under the piecewise-constant path-acceleration assumption (SURVEY §8 f1).
//
// Replaces (reference) ParametrizeConstAccel, toppra/parametrizer.py:23-158:
//   _process_parametrization (:52-65)  u_i = 0.5 (x_{i+1} - x_i) / (s_{i+1} - s_i),
//                                      t_{i+1} = t_i + 2 (s_{i+1} - s_i) / (sd_i + sd_{i+1})
//   _eval_params (:101-129)            idx = searchsorted(ts, t, side="right") - 1 (last index clamped),
//                                      dt = t - t_idx, v = sd_idx + dt u_idx, s = s_idx + dt sd_idx + 0.5 dt^2 u_idx
//   __call__ (:82-99)                  q(s) | q'(s) v | q''(s) v^2 + q'(s) u
// tb_time_grid: one thread per path walks its grid sequentially (the running sum keeps the reference's rounding
// order).  tb_constaccel_eval: one thread per (path, sample, joint).
#include "tb_common.cuh"

namespace tb {
namespace {

__global__ void time_grid_kernel(const double *__restrict__ sd, const double *__restrict__ grid, const int grid_shared,
                                 const long B, const int G, double *__restrict__ t_out, double *__restrict__ us_out) {
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= B) return;
  const double *v = sd + p * G;
  const double *s = grid + (grid_shared ? 0 : p * G);
  double *t = t_out + p * G;
  double *us = us_out ? us_out + p * (G - 1) : nullptr;
  double acc = 0.0;
  t[0] = 0.0;
  for (int i = 0; i < G - 1; ++i) {
    const double ds = s[i + 1] - s[i];
    if (us) us[i] = 0.5 * (v[i + 1] * v[i + 1] - v[i] * v[i]) / ds;
    acc = acc + 2 * ds / (v[i] + v[i + 1]);
    t[i + 1] = acc;
  }
}

__global__ void constaccel_eval_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                       const int breaks_shared, const int nseg, const int dof,
                                       const double *__restrict__ grid, const int grid_shared,
                                       const double *__restrict__ sd, const double *__restrict__ t_grid,
                                       const double *__restrict__ us, const long B, const int G,
                                       const double *__restrict__ ts, const int ts_shared, const int M, const int order,
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
    const double *c = ppoly + p * 4 * nseg * dof;
    const int seg = find_interval(x, nseg, s);
    double r;
    if (seg < 0) {
      r = __longlong_as_double(0x7ff8000000000000LL);
    } else {
      const double ds = s - x[seg];
      if (order == 0) r = ppoly_eval1(c, nseg, dof, seg, k, ds, 0);
      else if (order == 1) r = ppoly_eval1(c, nseg, dof, seg, k, ds, 1) * v;
      else r = ppoly_eval1(c, nseg, dof, seg, k, ds, 2) * (v * v) + ppoly_eval1(c, nseg, dof, seg, k, ds, 1) * u;
    }
    out[idx] = r;
  }
}

}  // namespace
}  // namespace tb

extern "C" int tb_time_grid(const double *sd, const double *grid, int grid_shared, int B, int G, double *t_grid,
                            double *us, void *stream) {
  using namespace tb;
  if (!sd || !grid || !t_grid || B <= 0 || G < 2) { set_error("tb_time_grid: bad argument"); return TB_ERR_ARG; }
  const int threads = 128;
  const long blocks = ((long)B + threads - 1) / threads;
  time_grid_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(sd, grid, grid_shared, B, G, t_grid, us);
  return check_launch("tb_time_grid");
}

extern "C" int tb_constaccel_eval(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof,
                                  const double *grid, int grid_shared, const double *sd, const double *t_grid,
                                  const double *us, int B, int G, const double *ts, int ts_shared, int M, int order,
                                  double *out, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !grid || !sd || !t_grid || !us || !ts || !out || B <= 0 || G < 2 || M <= 0 || nseg <= 0 ||
      dof <= 0) {
    set_error("tb_constaccel_eval: bad argument");
    return TB_ERR_ARG;
  }
  if (order < 0 || order > 2) { set_error("tb_constaccel_eval: order %d not in {0,1,2}", order); return TB_ERR_ARG; }
  const long total = (long)B * M * dof;
  const int threads = 256;
  long blocks = (total + threads - 1) / threads;
  if (blocks > (long)num_sms() * 64) blocks = (long)num_sms() * 64;
  constaccel_eval_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      ppoly, breaks, breaks_shared, nseg, dof, grid, grid_shared, sd, t_grid, us, B, G, ts, ts_shared, M, order, out);
  return check_launch("tb_constaccel_eval");
}
