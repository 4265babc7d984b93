// tb_spline.cu — K0: batched cubic-spline fit, and piecewise-polynomial evaluation.
//
// Replaces (reference): SplineInterpolator.__init__ / __call__, toppra/interpolator.py:385-430, which wrap
// scipy.interpolate.CubicSpline / PPoly (third-party, scipy/_cubic.py + _ppoly.pyx; restated here):
//   * slopes s at the knots from the tridiagonal system of CubicSpline.__init__ (not-a-knot, first- or
//     second-derivative boundary conditions; n == 2 and n == 3 special cases), solved with the LAPACK
//     dgtsv elimination order (partial pivoting) that scipy.linalg.solve_banded((1,1),..) uses;
//   * coefficients of CubicHermiteSpline.__init__: t=(s_i+s_{i+1}-2m)/h; c0=t/h; c1=(m-s_i)/h-t; c2=s_i; c3=y_i;
//   * evaluation = PPoly.derivative(nu) coefficients (c*3, c*2, ...) + power accumulation of evaluate_poly1.
// One thread per (path, dof) for the fit (n is small: 5 knots in the BASELINE configs), one thread per
// output element for the evaluation.  fp64, -fmad=false: bit-identical to scipy on x86-64.
#include "tb_common.cuh"

namespace tb {

namespace {

constexpr int LOCAL_KNOTS = 16;  // splines up to this many knots are fitted entirely in thread-local storage

__global__ void ppoly_eval_kernel(const double *__restrict__ ppoly, const double *__restrict__ breaks,
                                  const int breaks_shared, const long B, const int nseg, const int dof,
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
    else r = ppoly_eval1(ppoly + p * 4 * nseg * dof, nseg, dof, seg, k, sv - x[seg], order);
    out[idx] = r;
  }
}

// LAPACK dgtsv elimination (partial pivoting) + back substitution, single right-hand side.
__device__ void dgtsv_like(const int n, double *dl, double *d, double *du, double *b) {
  for (int i = 0; i < n - 1; ++i) {
    if (fabs(d[i]) >= fabs(dl[i])) {
      if (d[i] != 0.0) {
        const double fact = dl[i] / d[i];
        d[i + 1] = d[i + 1] - fact * du[i];
        b[i + 1] = b[i + 1] - fact * b[i];
      }
      if (i < n - 2) dl[i] = 0.0;
    } else {
      const double fact = d[i] / dl[i];
      d[i] = dl[i];
      double temp = d[i + 1];
      d[i + 1] = du[i] - fact * temp;
      if (i < n - 2) {
        dl[i] = du[i + 1];
        du[i + 1] = -fact * dl[i];
      }
      du[i] = temp;
      temp = b[i];
      b[i] = b[i + 1];
      b[i + 1] = temp - fact * b[i + 1];
    }
  }
  b[n - 1] = b[n - 1] / d[n - 1];
  if (n > 1) b[n - 2] = (b[n - 2] - du[n - 2] * b[n - 1]) / d[n - 2];
  for (int i = n - 3; i >= 0; --i) b[i] = (b[i] - du[i] * b[i + 1] - dl[i] * b[i + 2]) / d[i];
}

__global__ void spline_fit_kernel(const double *__restrict__ ss, const int ss_shared, const double *__restrict__ wp,
                                  const long B, const int n, const int dof, const int bc0_kind,
                                  const double *__restrict__ bc0, const int bc1_kind,
                                  const double *__restrict__ bc1, double *__restrict__ ppoly,
                                  double *__restrict__ workspace) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * dof) return;
  const int k = (int)(idx % dof);
  const long p = idx / dof;
  const double *x = ss + (ss_shared ? 0 : p * n);
  const double *y = wp + p * n * dof;
  double *c = ppoly + p * 4 * (n - 1) * dof;
  const int nseg = n - 1;
  // scratch: thread-local arrays for short splines, caller workspace [B*dof][7][n] for long ones
  double l_dx[LOCAL_KNOTS], l_slope[LOCAL_KNOTS], l_s[LOCAL_KNOTS], l_dl[LOCAL_KNOTS], l_dd[LOCAL_KNOTS],
      l_du[LOCAL_KNOTS], l_t2[LOCAL_KNOTS];
  double *dx = l_dx, *slope = l_slope, *s = l_s, *dl = l_dl, *dd = l_dd, *du = l_du, *t2 = l_t2;
  if (n > LOCAL_KNOTS) {
    double *w = workspace + idx * 7 * (long)n;
    dx = w; slope = w + n; s = w + 2 * (long)n; dl = w + 3 * (long)n; dd = w + 4 * (long)n; du = w + 5 * (long)n;
    t2 = w + 6 * (long)n;
  }
  for (int i = 0; i < nseg; ++i) {
    dx[i] = x[i + 1] - x[i];
    slope[i] = (y[(i + 1) * dof + k] - y[i * dof + k]) / dx[i];
  }
  int k0 = bc0_kind, k1 = bc1_kind;
  double v0 = bc0 ? bc0[p * dof + k] : 0.0, v1 = bc1 ? bc1[p * dof + k] : 0.0;
  if (n == 2) {  // _cubic.py: not-a-knot / periodic on 2 points -> first derivative = slope (0 for periodic data)
    if (k0 == TB_BC_NOT_A_KNOT || k0 == TB_BC_PERIODIC) { k0 = TB_BC_FIRST_DERIV; v0 = slope[0]; }
    if (k1 == TB_BC_NOT_A_KNOT || k1 == TB_BC_PERIODIC) { k1 = TB_BC_FIRST_DERIV; v1 = slope[0]; }
  }
  if (k0 == TB_BC_PERIODIC && n == 3) {
    // _cubic.py: t = (slope / dx).sum(0) / (1 / dx).sum(0); every knot gets this derivative
    const double t = (slope[0] / dx[0] + slope[1] / dx[1]) / (1.0 / dx[0] + 1.0 / dx[1]);
    s[0] = t; s[1] = t; s[2] = t;
  } else if (k0 == TB_BC_PERIODIC) {
    // _cubic.py, periodic branch: s[n-1] = s[0]; the cyclic (n-1) x (n-1) system is condensed to a tridiagonal
    // (n-2) x (n-2) matrix Ac solved for two right-hand sides (b1, and b2 = minus the removed column), then
    // s[n-2] = (b[-1] - a_m1_0 s1[0] - a_m1_m2 s1[-1]) / (a_m1_m1 + a_m1_0 s2[0] + a_m1_m2 s2[-1]), s[:n-2] = s1 + s[n-2] s2
    const int m = n - 2;
    const double a_m1_0 = dx[n - 3], a_m1_m2 = dx[n - 2], a_m1_m1 = 2 * (dx[n - 2] + dx[n - 3]);
    const double b_last = 3 * (dx[n - 2] * slope[n - 3] + dx[n - 3] * slope[n - 2]);
    for (int pass = 0; pass < 2; ++pass) {   // dgtsv overwrites the matrix: it is built once per right-hand side
      dd[0] = 2 * (dx[n - 2] + dx[0]);
      for (int j = 1; j < m; ++j) dd[j] = 2 * (dx[j - 1] + dx[j]);
      du[0] = dx[n - 2];
      for (int j = 1; j < m - 1; ++j) du[j] = dx[j - 1];
      for (int j = 0; j < m - 1; ++j) dl[j] = dx[j + 1];
      if (pass == 0) {
        s[0] = 3 * (dx[0] * slope[n - 2] + dx[n - 2] * slope[0]);
        for (int i = 1; i < m; ++i) s[i] = 3 * (dx[i] * slope[i - 1] + dx[i - 1] * slope[i]);
        dgtsv_like(m, dl, dd, du, s);
      } else {
        for (int i = 0; i < m; ++i) t2[i] = 0.0;
        t2[0] = -dx[0];
        t2[m - 1] = -dx[n - 4];
        dgtsv_like(m, dl, dd, du, t2);
      }
    }
    const double s_m1 = ((b_last - a_m1_0 * s[0]) - a_m1_m2 * s[m - 1]) / ((a_m1_m1 + a_m1_0 * t2[0]) + a_m1_m2 * t2[m - 1]);
    for (int i = 0; i < m; ++i) s[i] = s[i] + s_m1 * t2[i];
    s[n - 2] = s_m1;
    s[n - 1] = s[0];
  } else if (n == 3 && k0 == TB_BC_NOT_A_KNOT && k1 == TB_BC_NOT_A_KNOT) {
    // parabola through the 3 points: dense 3x3 system, LU with partial pivoting (scipy.linalg.solve)
    double A[3][3] = {{1, 1, 0}, {dx[1], 2 * (dx[0] + dx[1]), dx[0]}, {0, 1, 1}};
    double b[3] = {2 * slope[0], 3 * (dx[0] * slope[1] + dx[1] * slope[0]), 2 * slope[1]};
    int pv[3] = {0, 1, 2};
    for (int col = 0; col < 3; ++col) {
      int piv = col;
      for (int r = col + 1; r < 3; ++r)
        if (fabs(A[pv[r]][col]) > fabs(A[pv[piv]][col])) piv = r;
      const int t = pv[col]; pv[col] = pv[piv]; pv[piv] = t;
      for (int r = col + 1; r < 3; ++r) {
        const double f = A[pv[r]][col] / A[pv[col]][col];
        A[pv[r]][col] = 0;
        for (int cc = col + 1; cc < 3; ++cc) A[pv[r]][cc] -= f * A[pv[col]][cc];
        b[pv[r]] -= f * b[pv[col]];
      }
    }
    s[2] = b[pv[2]] / A[pv[2]][2];
    s[1] = (b[pv[1]] - A[pv[1]][2] * s[2]) / A[pv[1]][1];
    s[0] = (b[pv[0]] - A[pv[0]][1] * s[1] - A[pv[0]][2] * s[2]) / A[pv[0]][0];
  } else {
    for (int i = 1; i < n - 1; ++i) {
      dd[i] = 2 * (dx[i - 1] + dx[i]);
      du[i] = dx[i - 1];
      dl[i - 1] = dx[i];
      s[i] = 3 * (dx[i] * slope[i - 1] + dx[i - 1] * slope[i]);
    }
    if (k0 == TB_BC_NOT_A_KNOT) {
      dd[0] = dx[1];
      du[0] = x[2] - x[0];
      const double d = x[2] - x[0];
      s[0] = ((dx[0] + 2 * d) * dx[1] * slope[0] + dx[0] * dx[0] * slope[1]) / d;
    } else if (k0 == TB_BC_FIRST_DERIV) {
      dd[0] = 1; du[0] = 0; s[0] = v0;
    } else {
      dd[0] = 2 * dx[0]; du[0] = dx[0];
      s[0] = -0.5 * v0 * (dx[0] * dx[0]) + 3 * (y[1 * dof + k] - y[0 * dof + k]);
    }
    if (k1 == TB_BC_NOT_A_KNOT) {
      dd[n - 1] = dx[n - 3];
      dl[n - 2] = x[n - 1] - x[n - 3];
      const double d = x[n - 1] - x[n - 3];
      s[n - 1] = ((dx[n - 2] * dx[n - 2]) * slope[n - 3] + (2 * d + dx[n - 2]) * dx[n - 3] * slope[n - 2]) / d;
    } else if (k1 == TB_BC_FIRST_DERIV) {
      dd[n - 1] = 1; dl[n - 2] = 0; s[n - 1] = v1;
    } else {
      dd[n - 1] = 2 * dx[n - 2]; dl[n - 2] = dx[n - 2];
      s[n - 1] = 0.5 * v1 * (dx[n - 2] * dx[n - 2]) + 3 * (y[(n - 1) * dof + k] - y[(n - 2) * dof + k]);
    }
    dgtsv_like(n, dl, dd, du, s);
  }
  for (int i = 0; i < nseg; ++i) {
    const double t = (s[i] + s[i + 1] - 2 * slope[i]) / dx[i];
    c[(0 * nseg + i) * dof + k] = t / dx[i];
    c[(1 * nseg + i) * dof + k] = (slope[i] - s[i]) / dx[i] - t;
    c[(2 * nseg + i) * dof + k] = s[i];
    c[(3 * nseg + i) * dof + k] = y[i * dof + k];
  }
}

}  // namespace
}  // namespace tb

extern "C" int tb_spline_fit_workspace_doubles(int B, int n, int dof) {
  if (B <= 0 || n < 2 || dof <= 0) return TB_ERR_ARG;
  if (n <= tb::LOCAL_KNOTS) return 0;
  const long need = (long)B * dof * 7 * n;
  return need > 0x7fffffffL ? TB_ERR_UNSUPPORTED : (int)need;
}

extern "C" int tb_spline_fit(const double *ss, int ss_shared, const double *wp, int B, int n, int dof, int bc0_kind,
                             const double *bc0, int bc1_kind, const double *bc1, double *ppoly, double *workspace,
                             void *stream) {
  using namespace tb;
  if (!ss || !wp || !ppoly || B <= 0 || dof <= 0) { set_error("tb_spline_fit: bad argument"); return TB_ERR_ARG; }
  if (n < 2) { set_error("tb_spline_fit: n=%d < 2", n); return TB_ERR_ARG; }
  if (n > LOCAL_KNOTS && !workspace) {
    set_error("tb_spline_fit: n=%d > %d needs a workspace of tb_spline_fit_workspace_doubles() doubles", n, LOCAL_KNOTS);
    return TB_ERR_ARG;
  }
  if (bc0_kind < 0 || bc0_kind > 3 || bc1_kind < 0 || bc1_kind > 3) { set_error("tb_spline_fit: bad bc kind"); return TB_ERR_ARG; }
  if ((bc0_kind == TB_BC_PERIODIC) != (bc1_kind == TB_BC_PERIODIC)) {
    set_error("tb_spline_fit: 'periodic' is defined for both ends of the curve");   // scipy _validate_bc
    return TB_ERR_ARG;
  }
  const long total = (long)B * dof;
  const int threads = 128;
  const long blocks = (total + threads - 1) / threads;
  spline_fit_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(ss, ss_shared, wp, B, n, dof, bc0_kind, bc0,
                                                                           bc1_kind, bc1, ppoly, workspace);
  return check_launch("tb_spline_fit");
}

extern "C" int tb_ppoly_eval(const double *ppoly, const double *breaks, int breaks_shared, int B, int nseg, int dof,
                             const double *s, int s_shared, int G, int order, double *out, void *stream) {
  using namespace tb;
  if (!ppoly || !breaks || !s || !out || B <= 0 || nseg <= 0 || dof <= 0 || G <= 0) {
    set_error("tb_ppoly_eval: bad argument");
    return TB_ERR_ARG;
  }
  if (order < 0 || order > 2) { set_error("tb_ppoly_eval: order %d not in {0,1,2}", order); return TB_ERR_ARG; }
  const long total = (long)B * G * dof;
  const int threads = 256;
  long blocks = (total + threads - 1) / threads;
  if (blocks > (long)num_sms() * 64) blocks = (long)num_sms() * 64;
  ppoly_eval_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(ppoly, breaks, breaks_shared, B, nseg, dof, s,
                                                                           s_shared, G, order, out);
  return check_launch("tb_ppoly_eval");
}
