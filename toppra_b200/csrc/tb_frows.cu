// tb_frows.cu — batched device forms of the callers on either side of the scan (SURVEY.md section 8, rows f1-f3).
//
// Replaces (reference, hungpham2511/toppra v0.6.2):
//   propose_gridpoints                       toppra/interpolator.py:49-122        -> tb_propose_gridpoints (ragged grids)
//   TOPPRAsd.compute_parameterization        toppra/algorithm/reachabilitybased/desired_duration_algorithm.py:139-191
//     (bisection on the convex combination of the fastest and slowest passes) + _compute_duration :10-17
//                                                                                   -> tb_sd_bisect
//   ParametrizeSpline.__init__ time stamps   toppra/parametrizer.py:171-186      -> tb_spline_time_stamps
// All three are per-path sequential recurrences whose rounding order is the reference's; the batch supplies the
// parallelism (one warp or one thread per path).  fp64, -fmad=false.
#include "tb_common.cuh"
#include "tb_propose.cuh"

namespace tb {
namespace {

constexpr double PARAM_TINY = 1e-8;  // toppra/constants.py:15 (TINY), used by parametrizer.py:178,182

// ---------------------------------------------------------------------------------------------------------------
// propose_gridpoints: one warp per path, the passes of tb_propose.cuh on the cubic pieces.
// ---------------------------------------------------------------------------------------------------------------
struct CubicQdd {
  __device__ __forceinline__ int kc() const { return 4; }
  __device__ __forceinline__ double operator()(const double *c, const int nseg, const int dof, const int seg, const int k,
                                               const double ds) const {
    return ppoly_eval1(c, nseg, dof, seg, k, ds, 2);
  }
};

__global__ void __launch_bounds__(32)
propose_gridpoints_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks, const int breaks_shared,
                          const int B, const int nseg, const int dof, const double max_err, const int max_iter,
                          const double max_seg, const int min_pts, const int Gmax, double *__restrict__ grid_out,
                          double *__restrict__ scratch, int *__restrict__ glen, int *__restrict__ status) {
  propose_gridpoints_warp(ppoly, breaks, breaks_shared, B, nseg, dof, max_err, max_iter, max_seg, min_pts, Gmax, grid_out,
                          scratch, glen, status, CubicQdd{});
}

// ---------------------------------------------------------------------------------------------------------------
// TOPPRAsd: duration of a blend and the bisection on alpha.  One warp per path; the lanes fill sqrt(x) and the
// per-stage terms in shared memory, lane 0 adds them up in stage order (the reference's running sum).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double blend_duration(const double *xf, const double *xs, const double *g, const int G,
                                                 const double alpha, const bool blend, double *sds, double *term,
                                                 const int lane) {
  for (int j = lane; j < G; j += 32) {
    const double xv = blend ? (alpha * xf[j] + (1 - alpha) * xs[j]) : xf[j];
    sds[j] = sqrt(xv);
  }
  __syncwarp();
  for (int j = lane; j < G - 1; j += 32) term[j] = 2 * (g[j + 1] - g[j]) / (sds[j + 1] + sds[j] + 1e-9);
  __syncwarp();
  double t = 0.0;
  if (lane == 0)
    for (int j = 0; j < G - 1; ++j) t = t + term[j];
  t = __shfl_sync(FULL, t, 0);
  __syncwarp();
  return t;
}

__global__ void __launch_bounds__(32)
sd_bisect_kernel(const double *__restrict__ x_fast, const double *__restrict__ u_fast, const double *__restrict__ x_slow,
                 const double *__restrict__ u_slow, const double *__restrict__ grid, const int grid_shared, const int B,
                 const int G, const double *__restrict__ desired, const double atol, const int max_iter,
                 const int *__restrict__ status_in, double *__restrict__ sd, double *__restrict__ sdd,
                 double *__restrict__ info, int *__restrict__ status, const int *__restrict__ glen) {
  extern __shared__ double sm[];
  const int p = blockIdx.x, lane = threadIdx.x;
  if (p >= B) return;
  // ragged batches: this path's own gridpoints; strides stay G, entries past them are NaN
  const int Gp = glen ? min(max(glen[p], 1), G) : G;
  double *sds = sm, *term = sm + G;
  const double *xf = x_fast + (size_t)p * G, *xs = x_slow + (size_t)p * G;
  const double *uf = u_fast + (size_t)p * (G - 1), *us = u_slow + (size_t)p * (G - 1);
  const double *g = grid + (grid_shared ? 0 : (size_t)p * G);
  double *sdp = sd + (size_t)p * G, *up = sdd + (size_t)p * (G - 1);
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  const int st_in = status_in ? status_in[p] : TB_STATUS_OK;
  if (st_in == TB_STATUS_FAIL_UNCONTROLLABLE) {   // the reference returns None(s): :74-91
    for (int j = lane; j < G; j += 32) sdp[j] = nan_d;
    for (int j = lane; j < G - 1; j += 32) up[j] = nan_d;
    if (lane == 0) { status[p] = st_in; info[p * 4] = nan_d; info[p * 4 + 1] = nan_d; info[p * 4 + 2] = nan_d; info[p * 4 + 3] = 0.0; }
    return;
  }
  const double want = desired[p];
  const double d_fast = blend_duration(xf, xs, g, Gp, 1.0, false, sds, term, lane);
  const double d_slow = blend_duration(xs, xs, g, Gp, 0.0, false, sds, term, lane);
  double alpha;
  int iters = 0;
  if (d_fast > want) {
    alpha = 1.0;           // not achievable: the fastest parameterisation (:143-147)
  } else if (d_slow < want) {
    alpha = 0.0;           // the slowest (:148-152)
  } else {
    double a_low = 1.0, a_high = 0.0, diff = 10.0;
    alpha = 0.5;
    while (diff > atol && iters < max_iter) {
      ++iters;
      alpha = 0.5 * (a_low + a_high);
      const double d_alpha = blend_duration(xf, xs, g, Gp, alpha, true, sds, term, lane);
      if (d_alpha < want) { a_low = alpha; diff = want - d_alpha; }
      else { a_high = alpha; diff = d_alpha - want; }
    }
  }
  bool bad = false;
  for (int j = lane; j < Gp; j += 32) {
    const double v = sqrt(alpha * xf[j] + (1 - alpha) * xs[j]);
    sdp[j] = v;
    bad = bad || (v != v);
  }
  for (int j = lane; j < Gp - 1; j += 32) up[j] = alpha * uf[j] + (1 - alpha) * us[j];
  for (int j = Gp + lane; j < G; j += 32) sdp[j] = nan_d;
  for (int j = Gp - 1 + lane; j < G - 1; j += 32) up[j] = nan_d;
  bad = __any_sync(FULL, bad);
  if (lane == 0) {
    status[p] = bad ? TB_STATUS_ERR_UNKNOWN : TB_STATUS_OK;
    info[p * 4] = alpha; info[p * 4 + 1] = d_fast; info[p * 4 + 2] = d_slow; info[p * 4 + 3] = (double)iters;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ParametrizeSpline time stamps: thread per path, the reference's recurrence with its two data-dependent rules
// (average speed <= TINY -> 5 s; increments below TINY are dropped from the knot list, np.delete).
// ---------------------------------------------------------------------------------------------------------------
__global__ void spline_time_stamps_kernel(const double *__restrict__ sd, const double *__restrict__ grid,
                                          const int grid_shared, const int *__restrict__ glen, const long B, const int G,
                                          double *__restrict__ t_out, double *__restrict__ s_out,
                                          int *__restrict__ nkeep) {
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= B) return;
  const double *v = sd + p * G;
  const double *s = grid + (grid_shared ? 0 : p * G);
  double *t = t_out + p * G, *so = s_out + p * G;
  const int n = glen ? glen[p] : G;
  double acc = 0.0;
  int k = 1;
  t[0] = 0.0;
  so[0] = s[0];
  for (int i = 1; i < n; ++i) {
    const double sd_average = (v[i - 1] + v[i]) / 2;
    const double delta_s = s[i] - s[i - 1];
    const double delta_t = (sd_average > PARAM_TINY) ? (delta_s / sd_average) : 5.0;
    acc = acc + delta_t;
    if (!(delta_t < PARAM_TINY)) { t[k] = acc; so[k] = s[i]; ++k; }
  }
  const double tl = t[k - 1], sl = so[k - 1];
  for (int i = k; i < G; ++i) { t[i] = tl; so[i] = sl; }
  nkeep[p] = k;
}

}  // namespace
}  // namespace tb

extern "C" int tb_propose_gridpoints(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                                     double max_err_threshold, int max_iteration, double max_seg_length,
                                     int min_nb_points, int Gmax, double *grid_out, double *scratch, int *glen,
                                     int *status, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !grid_out || !scratch || !glen || !status || B <= 0 || nseg <= 0 || dof <= 0 || Gmax < 2 ||
      max_iteration <= 0) {
    set_error("tb_propose_gridpoints: bad argument");
    return TB_ERR_ARG;
  }
  propose_gridpoints_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(ppoly, breaks, breaks_shared, B, nseg, dof,
                                                              max_err_threshold, max_iteration, max_seg_length,
                                                              min_nb_points, Gmax, grid_out, scratch, glen, status);
  return check_launch("tb_propose_gridpoints");
}

extern "C" int tb_sd_bisect_ragged(const double *x_fast, const double *u_fast, const double *x_slow,
                                   const double *u_slow, const double *grid, int grid_shared, int B, int G,
                                   const int *glen, const double *desired_duration, double atol, int max_iter,
                                   const int *status_in, double *sd, double *sdd, double *info, int *status,
                                   void *stream) {
  using namespace tb;
  if (!x_fast || !u_fast || !x_slow || !u_slow || !grid || !desired_duration || !sd || !sdd || !info || !status || B <= 0 ||
      G < 2) {
    set_error("tb_sd_bisect: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tb_sd_bisect: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  const size_t smem = (size_t)2 * G * sizeof(double);
  if (smem > 200 * 1024) { set_error("tb_sd_bisect: G=%d too large", G); return TB_ERR_UNSUPPORTED; }
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(sd_bisect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("tb_sd_bisect: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  }
  sd_bisect_kernel<<<B, 32, smem, (cudaStream_t)stream>>>(x_fast, u_fast, x_slow, u_slow, grid, grid_shared, B, G,
                                                         desired_duration, atol, max_iter > 0 ? max_iter : 200, status_in,
                                                         sd, sdd, info, status, glen);
  return check_launch("tb_sd_bisect");
}

extern "C" int tb_sd_bisect(const double *x_fast, const double *u_fast, const double *x_slow, const double *u_slow,
                            const double *grid, int grid_shared, int B, int G, const double *desired_duration, double atol,
                            int max_iter, const int *status_in, double *sd, double *sdd, double *info, int *status,
                            void *stream) {
  return tb_sd_bisect_ragged(x_fast, u_fast, x_slow, u_slow, grid, grid_shared, B, G, nullptr, desired_duration, atol,
                             max_iter, status_in, sd, sdd, info, status, stream);
}

extern "C" int tb_spline_time_stamps(const double *sd, const double *grid, int grid_shared, const int *glen, int B, int G,
                                     double *t_out, double *s_out, int *nkeep, void *stream) {
  using namespace tb;
  if (!sd || !grid || !t_out || !s_out || !nkeep || B <= 0 || G < 1) {
    set_error("tb_spline_time_stamps: bad argument");
    return TB_ERR_ARG;
  }
  if (glen && grid_shared) { set_error("tb_spline_time_stamps: ragged batches need per-path grids"); return TB_ERR_ARG; }
  const int threads = 128;
  const long blocks = ((long)B + threads - 1) / threads;
  spline_time_stamps_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(sd, grid, grid_shared, glen, B, G,
                                                                                   t_out, s_out, nkeep);
  return check_launch("tb_spline_time_stamps");
}
