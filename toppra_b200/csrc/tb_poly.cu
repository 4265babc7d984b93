// tb_poly.cu — libtoppra_b200_poly.so: piecewise-polynomial paths with up to TBP_MAX_COEFFS = 8 coefficients per piece
// (degree <= 7).  C-ABI in include/toppra_b200_poly.h.
//
// The reference accepts any path object, because its algorithm only samples the path at the gridpoints:
//   path(gridpoints, 1), path(gridpoints, 2)   toppra/constraint/linear_joint_velocity.py:48,
//                                              linear_joint_acceleration.py:72-73, linear_second_order.py:148-150
//   path(mid, 2)                               toppra/interpolator.py:102 (propose_gridpoints)
//   path(...)                                  toppra/parametrizer.py:87-92, 187-194
// For a path in scipy's PPoly layout those samples are PPoly(c, x)(s) and the chained derivative objects
// .derivative()(s), .derivative().derivative()(s) (the convention of SplineInterpolator, interpolator.py:385-421).
// An order-k solve is: evaluate q', q'' at the gridpoints (poly_eval_kernel), build the stage records from the samples
// (rows_velacc_sampled_kernel), then the record scan of libtoppra_b200.so.  Every kernel here is a cubic kernel's body
// with the order-k path evaluator PolyPath or with loaded samples of q', q'':
//   poly_eval_kernel, constaccel_eval_poly_kernel   tb_path.cuh        (ppoly_eval_kernel, constaccel_eval_kernel)
//   propose_gridpoints_poly_kernel                  tb_propose.cuh     (propose_gridpoints_kernel)
//   rows_velacc_sampled_kernel                      tb_records.cuh     (coeff_velacc_kernel, K1)
//   xbound_varying_sampled_kernel                   tb_records.cuh     (xbound_varying_kernel)
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error) and num_sms();
// launch errors are read with launch_status (tb_common.cuh).
#include "tb_path.cuh"
#include "tb_propose.cuh"
#include "tb_records.cuh"
#include "../../include/toppra_b200_poly.h"

namespace tb {
namespace {

constexpr int MAXC = TBP_MAX_COEFFS;

// q_j^(order)(x[seg] + ds) for one (piece, joint) of an order-kc path, c = the path's [kc][nseg][dof] coefficients.
// The derivative's coefficient of power t is e_t = c[kc-1-order-t] * f (order 1: f = t+1; order 2 chained:
// (c * (t+2)) * (t+1), as PPoly.derivative().derivative() rounds), and the sum is scipy evaluate_poly1's:
// res = 0.0 + e_0; z = ds; res = res + e_t * z; z = z * ds; ... over exactly the n = kc - order coefficients (no
// zero padding, which could turn -0.0 into +0.0).  The loop is unrolled to MAXC so that e_t stays in registers.
__device__ __forceinline__ double poly_eval1(const double *__restrict__ c, const int kc, const int nseg, const int dof,
                                             const int seg, const int j, const double ds, const int order) {
  const int n = kc - order;
  const double *cj = c + (long)seg * dof + j;
  const long stride = (long)nseg * dof;
  double res = 0.0, z = ds;
#pragma unroll
  for (int t = 0; t < MAXC; ++t) {
    if (t < n) {
      const double ct = cj[(n - 1 - t) * stride];
      const double e = order == 0 ? ct : (order == 1 ? ct * (double)(t + 1) : (ct * (double)(t + 2)) * (double)(t + 1));
      if (t == 0) {
        res = 0.0 + e;
      } else {
        res = res + e * z;
        z = z * ds;
      }
    }
  }
  return res;
}

// The order-k path evaluator (tb_path.cuh).
struct PolyPath {
  int k;
  __device__ __forceinline__ int kc() const { return k; }
  __device__ __forceinline__ double eval(const double *c, const int nseg, const int dof, const int seg, const int j,
                                         const double ds, const int order) const {
    return poly_eval1(c, k, nseg, dof, seg, j, ds, order);
  }
};

constexpr int EVAL_THREADS = 256;

// tbp_ppoly_eval: one thread per (path, position, joint).
__global__ void poly_eval_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                 const int breaks_shared, const long B, const int kc, const int nseg, const int dof,
                                 const double *__restrict__ s, const int s_shared, const int G, const int order,
                                 double *__restrict__ out) {
  path_eval(PolyPath{kc}, ppoly, breaks, breaks_shared, B, nseg, dof, s, s_shared, G, order, out);
}

// The stage records from sampled q'(grid), q''(grid) [B][G][dof]: K1's record builder (tb_records.cuh) with the samples
// loaded where K1 evaluates the spline.  Fed samples of a cubic path it writes what K1 writes.
__global__ void __launch_bounds__(VELACC_THREADS)
rows_velacc_sampled_kernel(const double *__restrict__ qd, const double *__restrict__ qdd, const int dof,
                           const double *__restrict__ grid, const int grid_shared, const int G,
                           const double *__restrict__ vlim, const double *__restrict__ alim, const int lim_shared,
                           const int interp, double *__restrict__ records, const int W, const int R_total,
                           const int row0, const int write_xbound, const int nchunks) {
  extern __shared__ double sm[];
  const int VS = 6 * dof + 3;
  double *raw = sm;
  double *cand = raw + (VELACC_CH + 1) * 2 * dof;
  double *vec = cand + VELACC_CH * 2 * dof;
  double *sgrid = vec + VELACC_CH * VS;
  unsigned short *tab = reinterpret_cast<unsigned short *>(sgrid + VELACC_CH + 1);
  const long path = blockIdx.x / nchunks;
  const int chunk = blockIdx.x % nchunks;
  const int i0 = chunk * VELACC_CH;
  const int N = G - 1;
  const int npts = min(VELACC_CH, G - i0);
  const int nev = min(VELACC_CH + 1, G - i0);
  const double *q1 = qd + (path * G + i0) * (long)dof;
  const double *q2 = qdd + (path * G + i0) * (long)dof;
  const double *gp = grid + (grid_shared ? 0 : path * G);
  const double *al = alim ? alim + (lim_shared ? 0 : path * dof * 2) : nullptr;
  const double *vl = vlim ? vlim + (lim_shared ? 0 : path * dof * 2) : nullptr;
  const int tid = threadIdx.x;
  const int Racc = al ? (interp ? 4 : 2) * dof : 0;

  for (int ci = tid; ci < nev; ci += VELACC_THREADS) sgrid[ci] = gp[i0 + ci];
  velacc_column_table(tab, tid, W, R_total, row0, Racc, dof, write_xbound);
  for (int idx = tid; idx < nev * dof; idx += VELACC_THREADS) {
    const int ci = idx / dof, k = idx - ci * dof;
    velacc_store_sample(raw, cand, vl, ci, k, dof, npts, q1[idx], q2[idx], write_xbound);
  }
  __syncthreads();
  VELACC_WRITE_RECORDS(raw, cand, vec, sgrid, tab, al, vl, records, path, G, i0, N, npts, dof, VS, W, R_total,
                       write_xbound, tid);
}

// xbound_varying_kernel's bound from sampled q'(grid) [B][G][dof]: a NaN sample updates nothing, as a NaN gridpoint (no
// piece) does there.  One thread per (path, gridpoint).
__global__ void xbound_varying_sampled_kernel(const double *__restrict__ qd, const long B, const int dof, const int G,
                                              const double *__restrict__ vlim_grid, const int vlim_shared,
                                              double *__restrict__ records, const int W, const int R_total,
                                              const int mode) {
  const long total = B * G;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int gi = (int)(idx % G);
    const long p = idx / G;
    const double *vl = vlim_grid + ((vlim_shared ? 0 : p * G) + gi) * (long)dof * 2;
    const double *q1 = qd + idx * dof;
    velocity_xbound([&](const int k) { return q1[k]; }, true, dof, vl, records + idx * W, R_total, mode);
  }
}

// ---- propose_gridpoints (interpolator.py:49-122): the passes of tb_propose.cuh on the order-k pieces ----
__global__ void __launch_bounds__(32)
propose_gridpoints_poly_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                               const int breaks_shared, const int B, const int kc, const int nseg, const int dof,
                               const double max_err, const int max_iter, const double max_seg, const int min_pts,
                               const int Gmax, double *__restrict__ grid_out, double *__restrict__ scratch,
                               int *__restrict__ glen, int *__restrict__ status) {
  propose_gridpoints_warp(ppoly, breaks, breaks_shared, B, nseg, dof, max_err, max_iter, max_seg, min_pts, Gmax, grid_out,
                          scratch, glen, status, PolyPath{kc});
}

// ParametrizeConstAccel output (parametrizer.py:82-129) on order-k paths: one thread per (path, sample, joint).
__global__ void constaccel_eval_poly_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                            const int breaks_shared, const int kc, const int nseg, const int dof,
                                            const double *__restrict__ grid, const int grid_shared,
                                            const double *__restrict__ sd, const double *__restrict__ t_grid,
                                            const double *__restrict__ us, const long B, const int G,
                                            const double *__restrict__ ts, const int ts_shared, const int M,
                                            const int order, double *__restrict__ out) {
  constaccel_eval(PolyPath{kc}, ppoly, breaks, breaks_shared, nseg, dof, grid, grid_shared, sd, t_grid, us, B, G, ts,
                  ts_shared, M, order, out);
}

bool bad_order(const int k, const char *what) {
  if (k >= 1 && k <= MAXC) return false;
  set_error("%s: k=%d coefficients per piece; 1 <= k <= %d", what, k, MAXC);
  return true;
}

}  // namespace
}  // namespace tb

extern "C" int tbp_version(void) { return TBP_VERSION; }

extern "C" int tbp_ppoly_eval(const double *ppoly, const double *breaks, int breaks_shared, int B, int k, int nseg,
                              int dof, const double *s, int s_shared, int G, int order, double *out, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !s || !out || B <= 0 || nseg <= 0 || dof <= 0 || G <= 0) {
    set_error("tbp_ppoly_eval: bad argument");
    return TB_ERR_ARG;
  }
  if (bad_order(k, "tbp_ppoly_eval")) return TB_ERR_ARG;
  if (order < 0 || order > 2) { set_error("tbp_ppoly_eval: order %d not in {0,1,2}", order); return TB_ERR_ARG; }
  const long total = (long)B * G * dof;
  const long blocks = grid_stride_blocks(total, EVAL_THREADS, 64);
  poly_eval_kernel<<<(unsigned)blocks, EVAL_THREADS, 0, (cudaStream_t)stream>>>(ppoly, breaks, breaks_shared, B, k, nseg,
                                                                               dof, s, s_shared, G, order, out);
  return launch_status("tbp_ppoly_eval");
}

extern "C" int tbp_rows_velacc_sampled(const double *qd, const double *qdd, int B, int dof, const double *grid,
                                       int grid_shared, int G, const double *vlim, const double *alim, int lim_shared,
                                       int interp, double *records, int W, int R_total, int row0, int write_xbound,
                                       void *stream) {
  using namespace tb;
  if (!qd || !qdd || !grid || (!alim && !vlim) || !records || B <= 0 || dof <= 0 || G <= 0) {
    set_error("tbp_rows_velacc_sampled: bad argument");
    return TB_ERR_ARG;
  }
  const int nchunks = (G + VELACC_CH - 1) / VELACC_CH;
  const long blocks = (long)B * nchunks;
  if (const int rc = velacc_check("tbp_rows_velacc_sampled", alim ? (interp ? 4 : 2) * dof : 0, dof, W, R_total, row0,
                                  blocks))
    return rc;
  const size_t smem = velacc_smem("tbp_rows_velacc_sampled", rows_velacc_sampled_kernel, dof, W, 0);
  if (!smem) return TB_ERR_UNSUPPORTED;
  rows_velacc_sampled_kernel<<<(unsigned)blocks, VELACC_THREADS, smem, (cudaStream_t)stream>>>(
      qd, qdd, dof, grid, grid_shared, G, vlim, alim, lim_shared, interp, records, W, R_total, row0, write_xbound, nchunks);
  return launch_status("tbp_rows_velacc_sampled");
}

extern "C" int tbp_xbound_varying_sampled(const double *qd, int B, int dof, int G, const double *vlim_grid,
                                          int vlim_shared, double *records, int W, int R_total, int write_xbound,
                                          void *stream) {
  using namespace tb;
  if (!qd || !vlim_grid || !records || B <= 0 || dof <= 0 || G <= 0 || R_total < 0 || write_xbound < 1 ||
      write_xbound > 3 || W < 3 * R_total + 2) {
    set_error("tbp_xbound_varying_sampled: bad argument");
    return TB_ERR_ARG;
  }
  const long total = (long)B * G;
  const int threads = 128;
  const long blocks = grid_stride_blocks(total, threads, 64);
  xbound_varying_sampled_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(qd, B, dof, G, vlim_grid,
                                                                                       vlim_shared, records, W, R_total,
                                                                                       write_xbound);
  return launch_status("tbp_xbound_varying_sampled");
}

extern "C" int tbp_propose_gridpoints(const double *ppoly, const double *breaks, int breaks_shared, int B, int k,
                                      int nseg, int dof, double max_err_threshold, int max_iteration,
                                      double max_seg_length, int min_nb_points, int Gmax, double *grid_out,
                                      double *scratch, int *glen, int *status, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !grid_out || !scratch || !glen || !status || B <= 0 || nseg <= 0 || dof <= 0 || Gmax < 2 ||
      max_iteration <= 0) {
    set_error("tbp_propose_gridpoints: bad argument");
    return TB_ERR_ARG;
  }
  if (bad_order(k, "tbp_propose_gridpoints")) return TB_ERR_ARG;
  propose_gridpoints_poly_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(ppoly, breaks, breaks_shared, B, k, nseg, dof,
                                                                   max_err_threshold, max_iteration, max_seg_length,
                                                                   min_nb_points, Gmax, grid_out, scratch, glen, status);
  return launch_status("tbp_propose_gridpoints");
}

extern "C" int tbp_constaccel_eval(const double *ppoly, const double *breaks, int breaks_shared, int k, int nseg, int dof,
                                   const double *grid, int grid_shared, const double *sd, const double *t_grid,
                                   const double *us, int B, int G, const double *ts, int ts_shared, int M, int order,
                                   double *out, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !grid || !sd || !t_grid || !us || !ts || !out || B <= 0 || G < 2 || M <= 0 || nseg <= 0 ||
      dof <= 0) {
    set_error("tbp_constaccel_eval: bad argument");
    return TB_ERR_ARG;
  }
  if (bad_order(k, "tbp_constaccel_eval")) return TB_ERR_ARG;
  if (order < 0 || order > 2) { set_error("tbp_constaccel_eval: order %d not in {0,1,2}", order); return TB_ERR_ARG; }
  const long total = (long)B * M * dof;
  const int threads = 256;
  const long blocks = grid_stride_blocks(total, threads, 64);
  constaccel_eval_poly_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      ppoly, breaks, breaks_shared, k, nseg, dof, grid, grid_shared, sd, t_grid, us, B, G, ts, ts_shared, M, order, out);
  return launch_status("tbp_constaccel_eval");
}
