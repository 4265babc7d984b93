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
// (rows_velacc_sampled_kernel), then the record scan of libtoppra_b200.so.  The record builder does not depend on the
// path's degree: fed samples of a cubic path it writes what K1 (coeff_velacc_kernel, tb_coeff.cu) writes.
//
// This library is linked against libtoppra_b200.so and uses its error slot (set_error / tb_last_error) and num_sms().
// Each library carries its own static CUDA runtime, so launch errors are read here (launch_status), not with the main
// library's check_launch, whose cudaGetLastError sees only launches made by that library.
#include "tb_common.cuh"
#include "tb_propose.cuh"
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

constexpr int EVAL_THREADS = 256;

// tbp_ppoly_eval: one thread per (path, position, joint).  Replaces path(s, order) of the reference
// (interpolator.py:423-430 for its cubic; the same scipy calls for any order).
__global__ void poly_eval_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                 const int breaks_shared, const long B, const int kc, const int nseg, const int dof,
                                 const double *__restrict__ s, const int s_shared, const int G, const int order,
                                 double *__restrict__ out) {
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
    else r = poly_eval1(ppoly + p * kc * nseg * dof, kc, nseg, dof, seg, k, sv - x[seg], order);
    out[idx] = r;
  }
}

// ---- stage records from sampled q'(grid), q''(grid) ------------------------------------------------------------------
// Restates K1 (coeff_velacc_kernel, tb_coeff.cu) with phase 0's coefficient table and phase 1's spline evaluation
// replaced by loads of the samples; the record arithmetic below is K1's, operation for operation:
//   _create_velocity_constraint (fp32 running min/max)   toppra/_CythonUtils.pyx:16-59
//   JointAccelerationConstraint.compute_constraint_params toppra/constraint/linear_joint_acceleration.py:63-104
//   canlinear_colloc_to_interpolate                      toppra/constraint/linear_constraint.py:84-192
//   seidelWrapper.__init__ row assembly                  toppra/solverwrapper/cy_seidel_solverwrapper.pyx:474-520
// tests/test_piecewise_poly.py feeds both builders samples of cubic paths and requires identical records; that test
// pins this copy to K1.
constexpr int ROWS_THREADS = 128;
constexpr int CH = 32;  // gridpoints per CTA

__device__ __forceinline__ int R_total_or1(int R_total) { return R_total > 0 ? R_total : 1; }

// Shared memory of one CTA (dof = d, VS = 6d + 3): raw [(CH+1)][2d] | cand [CH][2d] | vec [CH][VS] | sgrid [CH+1] |
// tab [W] (offset into vec per record column; bit 15 = negate, 0x7fff = column not owned).  Layout as in K1.
__global__ void __launch_bounds__(ROWS_THREADS)
rows_velacc_sampled_kernel(const double *__restrict__ qd, const double *__restrict__ qdd, const int dof,
                           const double *__restrict__ grid, const int grid_shared, const int G,
                           const double *__restrict__ vlim, const double *__restrict__ alim, const int lim_shared,
                           const int interp, double *__restrict__ records, const int W, const int R_total,
                           const int row0, const int write_xbound, const int nchunks) {
  extern __shared__ double sm[];
  const int VS = 6 * dof + 3;
  double *raw = sm;
  double *cand = raw + (CH + 1) * 2 * dof;
  double *vec = cand + CH * 2 * dof;
  double *sgrid = vec + CH * VS;
  unsigned short *tab = reinterpret_cast<unsigned short *>(sgrid + CH + 1);
  const long path = blockIdx.x / nchunks;
  const int chunk = blockIdx.x % nchunks;
  const int i0 = chunk * CH;
  const int N = G - 1;
  const int npts = min(CH, G - i0);
  const int nev = min(CH + 1, G - i0);
  const double *q1 = qd + (path * G + i0) * (long)dof;
  const double *q2 = qdd + (path * G + i0) * (long)dof;
  const double *gp = grid + (grid_shared ? 0 : path * G);
  const double *al = alim ? alim + (lim_shared ? 0 : path * dof * 2) : nullptr;
  const double *vl = vlim ? vlim + (lim_shared ? 0 : path * dof * 2) : nullptr;
  const int tid = threadIdx.x;
  const int Racc = al ? (interp ? 4 : 2) * dof : 0;

  // ---- phase 0: gridpoints, column table ----
  for (int ci = tid; ci < nev; ci += ROWS_THREADS) sgrid[ci] = gp[i0 + ci];
  for (int w = tid; w < W; w += ROWS_THREADS) {
    unsigned short code = 0x7fff;
    const int kind = w / R_total_or1(R_total), r = w - kind * R_total - row0;
    if (kind < 3 && R_total > 0 && r >= 0 && r < Racc) {
      const int blk = r / dof, k = r - blk * dof;
      const int neg = blk & 1, second = blk >> 1;
      if (kind == 0) code = (unsigned short)((second ? dof + k : k) | (neg << 15));
      else if (kind == 1) code = (unsigned short)((second ? 3 * dof + k : 2 * dof + k) | (neg << 15));
      else code = (unsigned short)(neg ? 5 * dof + k : 4 * dof + k);
    } else if (w >= 3 * R_total) {
      const bool ub_slot = (W >= 3 * R_total + 4) && (w == 3 * R_total + 2 || w == 3 * R_total + 3);
      if (write_xbound && !ub_slot)
        code = (unsigned short)(w == 3 * R_total ? 6 * dof : (w == 3 * R_total + 1 ? 6 * dof + 1 : 6 * dof + 2));
    }
    tab[w] = code;
  }

  // ---- phase 1: the samples of the chunk (+1 gridpoint for the lift), velocity-bound candidates ----
  const double inf_d = __longlong_as_double(0x7ff0000000000000LL);
  for (int idx = tid; idx < nev * dof; idx += ROWS_THREADS) {
    const int ci = idx / dof, k = idx - ci * dof;
    const double v1 = q1[idx], v2 = q2[idx];
    raw[ci * 2 * dof + k] = v1;
    raw[ci * 2 * dof + dof + k] = v2;
    if (vl && write_xbound && ci < npts) {
      // _CythonUtils.pyx:44-50: q' > 0: (vmax/q', vmin/q'); q' < 0: (vmin/q', vmax/q'); q' == 0 (or NaN): no update
      const bool posq = v1 > 0, negq = v1 < 0;
      const double qdv = (posq || negq) ? v1 : 1.0;
      const double r1 = vl[k * 2 + 1] / qdv, r0 = vl[k * 2 + 0] / qdv;
      cand[ci * 2 * dof + k] = posq ? r1 : (negq ? r0 : inf_d);
      cand[ci * 2 * dof + dof + k] = posq ? r0 : (negq ? r1 : -inf_d);
    }
  }
  __syncthreads();

  // ---- phase 1b: per-gridpoint value vectors q' | a+ | q'' | b+ | -amax | +amin | xlo | xhi | 0 ----
  double *rec0 = records + (path * G + i0) * (long)W;
  for (int idx = tid; idx < npts * dof; idx += ROWS_THREADS) {
    const int ci = idx / dof, k = idx - ci * dof;
    const int gi = i0 + ci;
    double *v = vec + ci * VS;
    const double a = raw[ci * 2 * dof + k], b = raw[ci * 2 * dof + dof + k];
    double ap = a, bp = b;  // last gridpoint duplicates itself, linear_constraint.py:171,175
    if (gi < N) {
      const double delta = sgrid[ci + 1] - sgrid[ci];
      ap = raw[(ci + 1) * 2 * dof + k] + (2 * delta) * raw[(ci + 1) * 2 * dof + dof + k];  // linear_constraint.py:170
      bp = raw[(ci + 1) * 2 * dof + dof + k];
    }
    v[k] = a; v[dof + k] = ap; v[2 * dof + k] = b; v[3 * dof + k] = bp;
    if (al) {
      v[4 * dof + k] = 0.0 - al[k * 2 + 1];       // F.c - g with c = 0, g = [amax; -amin]
      v[5 * dof + k] = 0.0 - (-al[k * 2 + 0]);
    }
    if (k == 0 && write_xbound) {
      double xlo = VAR_MIN, xhi = VAR_MAX;  // seidelWrapper low_arr/high_arr init, pyx:477-478
      if (vl) {
        // the reference's fp32 running min/max s <- (float)min(cand_k, (double)s), s_0 = 1e8f, equals
        // (float)min(1e8, min_k cand_k): round-to-nearest is monotone and idempotent (likewise for the max)
        double mhi = JVEL_MAXSD, mlo = -JVEL_MAXSD;
        for (int kk = 0; kk < dof; ++kk) {
          const double hi = cand[ci * 2 * dof + kk], lo = cand[ci * 2 * dof + dof + kk];
          mhi = (hi <= mhi) ? hi : mhi;
          mlo = (lo >= mlo) ? lo : mlo;
        }
        const float sdmax = __double2float_rn(mhi), sdmin = __double2float_rn(mlo);
        const float up = __fmul_rn(sdmax, sdmax);                          // powf(sdmax, 2) in fp32
        const double lo_d = ((double)sdmin >= 0.0) ? (double)sdmin : 0.0;  // float64_max(sdmin, 0.)
        xlo = lo_d * lo_d;
        xhi = (double)up;
        if (write_xbound != 2) {
          xlo = fmax(VAR_MIN, xlo);  // pyx:517-520
          xhi = fmin(VAR_MAX, xhi);
        }
      }
      if (write_xbound == 3) {  // intersect with what the record already holds
        const double *rec = rec0 + (long)ci * W;
        xlo = fmax(rec[3 * R_total], xlo);
        xhi = fmin(rec[3 * R_total + 1], xhi);
      }
      v[6 * dof] = xlo; v[6 * dof + 1] = xhi; v[6 * dof + 2] = 0.0;
    }
  }
  __syncthreads();

  // ---- phase 2: stream the records out; thread -> fixed 16-byte column pair, loop over gridpoints ----
  const int Wh = W >> 1;
  const int ngrp = ROWS_THREADS / Wh;
  const int g = tid / Wh, j = tid - g * Wh;
  if (ngrp > 0 && g < ngrp) {
    const unsigned short c0 = tab[2 * j], c1 = tab[2 * j + 1];
    const int o0 = c0 & 0x7fff, o1 = c1 & 0x7fff;
    const bool n0 = (c0 & 0x8000) != 0, n1 = (c1 & 0x8000) != 0;
    const bool own0 = c0 != 0x7fff, own1 = c1 != 0x7fff;
    double *dst = rec0 + (long)g * W + 2 * j;
    const double *v = vec + g * VS;
    if (own0 && own1) {
      for (int ci = g; ci < npts; ci += ngrp, dst += (long)ngrp * W, v += ngrp * VS) {
        double2 o;
        o.x = n0 ? -v[o0] : v[o0];
        o.y = n1 ? -v[o1] : v[o1];
        __stcs(reinterpret_cast<double2 *>(dst), o);
      }
    } else if (own0 || own1) {
      for (int ci = g; ci < npts; ci += ngrp, dst += (long)ngrp * W, v += ngrp * VS) {
        if (own0) dst[0] = n0 ? -v[o0] : v[o0];
        if (own1) dst[1] = n1 ? -v[o1] : v[o1];
      }
    }
  } else if (ngrp == 0) {  // records wider than 2 * ROWS_THREADS columns: column loop per gridpoint
    for (int ci = 0; ci < npts; ++ci)
      for (int w = tid; w < W; w += ROWS_THREADS) {
        const unsigned short cw = tab[w];
        if (cw != 0x7fff) {
          const double t = vec[ci * VS + (cw & 0x7fff)];
          rec0[(long)ci * W + w] = (cw & 0x8000) ? -t : t;
        }
      }
  }
}

// JointVelocityConstraintVarying (linear_joint_velocity.py:56-87, _CythonUtils.pyx:61-101) from sampled q'(grid).
// Restates the per-gridpoint branch of xbound_varying_kernel (tb_coeff.cu) with q' loaded instead of evaluated; a NaN
// sample updates nothing, as a NaN gridpoint (no piece) does there.  One thread per (path, gridpoint).
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
    float sdmin = -(float)JVEL_MAXSD, sdmax = (float)JVEL_MAXSD;
    for (int k = 0; k < dof; ++k) {
      const double q = q1[k];
      if (q > 0) {
        const double hi = vl[k * 2 + 1] / q, lo = vl[k * 2 + 0] / q;
        sdmax = __double2float_rn(hi <= (double)sdmax ? hi : (double)sdmax);
        sdmin = __double2float_rn(lo >= (double)sdmin ? lo : (double)sdmin);
      } else if (q < 0) {
        const double hi = vl[k * 2 + 0] / q, lo = vl[k * 2 + 1] / q;
        sdmax = __double2float_rn(hi <= (double)sdmax ? hi : (double)sdmax);
        sdmin = __double2float_rn(lo >= (double)sdmin ? lo : (double)sdmin);
      }
    }
    const float up = __fmul_rn(sdmax, sdmax);
    const double lo_d = ((double)sdmin >= 0.0) ? (double)sdmin : 0.0;
    double xlo = lo_d * lo_d, xhi = (double)up;
    double *rec = records + idx * W;
    if (mode != 2) { xlo = fmax(VAR_MIN, xlo); xhi = fmin(VAR_MAX, xhi); }
    if (mode == 3) { xlo = fmax(rec[3 * R_total], xlo); xhi = fmin(rec[3 * R_total + 1], xhi); }
    rec[3 * R_total] = xlo;
    rec[3 * R_total + 1] = xhi;
  }
}

// ---- propose_gridpoints (interpolator.py:49-122): the passes of tb_propose.cuh with the order-k q'' ----
struct PolyQdd {
  int k;
  __device__ __forceinline__ int kc() const { return k; }
  __device__ __forceinline__ double operator()(const double *c, const int nseg, const int dof, const int seg, const int j,
                                               const double ds) const {
    return poly_eval1(c, k, nseg, dof, seg, j, ds, 2);
  }
};

__global__ void __launch_bounds__(32)
propose_gridpoints_poly_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                               const int breaks_shared, const int B, const int kc, const int nseg, const int dof,
                               const double max_err, const int max_iter, const double max_seg, const int min_pts,
                               const int Gmax, double *__restrict__ grid_out, double *__restrict__ scratch,
                               int *__restrict__ glen, int *__restrict__ status) {
  propose_gridpoints_warp(ppoly, breaks, breaks_shared, B, nseg, dof, max_err, max_iter, max_seg, min_pts, Gmax, grid_out,
                          scratch, glen, status, PolyQdd{kc});
}

// ---- ParametrizeConstAccel output (parametrizer.py:82-129) on order-k paths ----
// Restates constaccel_eval_kernel (tb_param.cu) with the order-k evaluation: idx = searchsorted(ts, t, "right") - 1
// (last index clamped), dt = t - t_idx, v = sd_idx + dt u_idx, s = s_idx + dt sd_idx + 0.5 dt^2 u_idx, then
// q(s) | q'(s) v | q''(s) v^2 + q'(s) u.  One thread per (path, sample, joint).
__global__ void constaccel_eval_poly_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                            const int breaks_shared, const int kc, const int nseg, const int dof,
                                            const double *__restrict__ grid, const int grid_shared,
                                            const double *__restrict__ sd, const double *__restrict__ t_grid,
                                            const double *__restrict__ us, const long B, const int G,
                                            const double *__restrict__ ts, const int ts_shared, const int M,
                                            const int order, double *__restrict__ out) {
  const long total = B * M * dof;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % dof);
    const long pm = idx / dof;
    const int m = (int)(pm % M);
    const long p = pm / M;
    const double t = ts[(ts_shared ? 0 : p * M) + m];
    const double *tg = t_grid + p * G;
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
    const double *c = ppoly + p * kc * nseg * dof;
    const int seg = find_interval(x, nseg, s);
    double r;
    if (seg < 0) {
      r = __longlong_as_double(0x7ff8000000000000LL);
    } else {
      const double ds = s - x[seg];
      if (order == 0) r = poly_eval1(c, kc, nseg, dof, seg, k, ds, 0);
      else if (order == 1) r = poly_eval1(c, kc, nseg, dof, seg, k, ds, 1) * v;
      else r = poly_eval1(c, kc, nseg, dof, seg, k, ds, 2) * (v * v) + poly_eval1(c, kc, nseg, dof, seg, k, ds, 1) * u;
    }
    out[idx] = r;
  }
}

int launch_status(const char *what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

long grid_stride_blocks(const long total, const int threads, const int per_sm) {
  const long blocks = (total + threads - 1) / threads;
  return blocks > (long)num_sms() * per_sm ? (long)num_sms() * per_sm : blocks;
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
  const int Racc = alim ? (interp ? 4 : 2) * dof : 0;
  if (row0 < 0 || row0 + Racc > R_total || W < 3 * R_total + 2) {
    set_error("tbp_rows_velacc_sampled: rows [%d,%d) do not fit R_total=%d / W=%d", row0, row0 + Racc, R_total, W);
    return TB_ERR_ARG;
  }
  if (R_total > MAX_ROWS) { set_error("tbp_rows_velacc_sampled: R=%d > %d", R_total, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (6 * dof + 3 >= 0x7fff) { set_error("tbp_rows_velacc_sampled: dof=%d too large", dof); return TB_ERR_UNSUPPORTED; }
  const int nchunks = (G + CH - 1) / CH;
  const long blocks = (long)B * nchunks;
  if (blocks > 0x7fffffffL) { set_error("tbp_rows_velacc_sampled: batch too large for one launch"); return TB_ERR_UNSUPPORTED; }
  const size_t smem = (size_t)((CH + 1) * dof * 2 + CH * dof * 2 + CH * (6 * dof + 3) + CH + 1) * sizeof(double) +
                      (size_t)W * sizeof(unsigned short) + 16;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(rows_velacc_sampled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("tbp_rows_velacc_sampled: dof=%d too large for shared memory", dof); return TB_ERR_UNSUPPORTED; }
  }
  rows_velacc_sampled_kernel<<<(unsigned)blocks, ROWS_THREADS, smem, (cudaStream_t)stream>>>(
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
