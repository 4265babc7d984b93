// tb_api.cu — host side of the C-ABI: error reporting, limits, and the host-buffer convenience entry
// tb_solve_velacc_host (K0 -> K1 -> K2 with the H2D / D2H copies inside).
#include <stdarg.h>
#include <string.h>

#include "tb_common.cuh"

namespace tb {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char *what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      n <= 0)
    return 132;
  return n;
}

}  // namespace tb

extern "C" int tb_version(void) { return TB_VERSION; }
extern "C" const char *tb_last_error(void) { return tb::g_err; }
extern "C" int tb_limits(int *max_rows, int *max_knots) {
  if (max_rows) *max_rows = tb::MAX_ROWS;
  if (max_knots) *max_knots = 1 << 20;  // limited by the caller-provided workspace only
  return 0;
}

#define TB_CUDA(call)                                                            \
  do {                                                                           \
    cudaError_t e_ = (call);                                                     \
    if (e_ != cudaSuccess) {                                                     \
      tb::set_error("%s: %s", #call, cudaGetErrorString(e_));                    \
      rc = (int)e_;                                                              \
      goto done;                                                                 \
    }                                                                            \
  } while (0)

extern "C" int tb_solve_velacc_host(int device, const double *ss, const double *wp, int B, int n, int dof,
                                    const double *grid, int G, const double *vlim, const double *alim,
                                    int lim_shared, int interp, const double *sd_start, const double *sd_end,
                                    double *K, double *sd, double *u, int *status) {
  using namespace tb;
  if (!ss || !wp || !grid || !alim || !K || !sd || !status || (G > 1 && !u) || B <= 0 || n < 2 || dof <= 0 || G <= 0) {
    set_error("tb_solve_velacc_host: bad argument");
    return TB_ERR_ARG;
  }
  int rc = 0;
  const int nseg = n - 1;
  const int R = (interp ? 4 : 2) * dof;
  // vel+acc problems that fit one LP row per lane take the fused scan (no stage records): K1 shrinks to the velocity
  // bound [B][G][2]; larger ones materialise the records (K1 -> K2)
  const bool fused = (R + 2 <= 32) && (((size_t)nseg * dof * 6 + nseg + 2) * sizeof(double) <= 16 * 1024);
  const int W = fused ? 2 : tb_record_doubles(R);
  const size_t nlim = (size_t)(lim_shared ? 1 : B) * dof * 2;
  // one device arena
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_ss = take(sizeof(double) * n), o_wp = take(sizeof(double) * (size_t)B * n * dof);
  const size_t o_grid = take(sizeof(double) * G), o_vl = take(sizeof(double) * nlim), o_al = take(sizeof(double) * nlim);
  const size_t o_s0 = take(sizeof(double) * B), o_s1 = take(sizeof(double) * B);
  const size_t o_pp = take(sizeof(double) * (size_t)B * 4 * nseg * dof);
  const size_t o_rec = take(sizeof(double) * (size_t)B * G * W);
  const int ws_doubles = tb_spline_fit_workspace_doubles(B, n, dof);
  if (ws_doubles < 0) { set_error("tb_solve_velacc_host: spline too large"); return ws_doubles; }
  const size_t o_ws = take(sizeof(double) * (size_t)(ws_doubles > 0 ? ws_doubles : 1));
  const size_t o_K = take(sizeof(double) * (size_t)B * G * 2), o_sd = take(sizeof(double) * (size_t)B * G);
  const size_t o_u = take(sizeof(double) * (size_t)B * (G > 1 ? G - 1 : 1)), o_st = take(sizeof(int) * (size_t)B);
  char *d = nullptr;
  cudaStream_t st = nullptr;
  TB_CUDA(cudaSetDevice(device));
  TB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  TB_CUDA(cudaMalloc(&d, off));
  TB_CUDA(cudaMemcpyAsync(d + o_ss, ss, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaMemcpyAsync(d + o_wp, wp, sizeof(double) * (size_t)B * n * dof, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaMemcpyAsync(d + o_grid, grid, sizeof(double) * G, cudaMemcpyHostToDevice, st));
  if (vlim) TB_CUDA(cudaMemcpyAsync(d + o_vl, vlim, sizeof(double) * nlim, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaMemcpyAsync(d + o_al, alim, sizeof(double) * nlim, cudaMemcpyHostToDevice, st));
  if (sd_start) TB_CUDA(cudaMemcpyAsync(d + o_s0, sd_start, sizeof(double) * B, cudaMemcpyHostToDevice, st));
  if (sd_end) TB_CUDA(cudaMemcpyAsync(d + o_s1, sd_end, sizeof(double) * B, cudaMemcpyHostToDevice, st));
  rc = tb_spline_fit((double *)(d + o_ss), 1, (double *)(d + o_wp), B, n, dof, TB_BC_NOT_A_KNOT, nullptr,
                     TB_BC_NOT_A_KNOT, nullptr, (double *)(d + o_pp), ws_doubles > 0 ? (double *)(d + o_ws) : nullptr, st);
  if (rc) goto done;
  if (fused) {
    rc = vlim ? tb_xbound_velocity((double *)(d + o_pp), (double *)(d + o_ss), 1, B, nseg, dof, (double *)(d + o_grid), 1,
                                   G, (double *)(d + o_vl), lim_shared, (double *)(d + o_rec), 2, 0, 1, st)
              : tb_init_bounds((double *)(d + o_rec), B, G, 2, 0, st);
    if (rc) goto done;
    rc = tb_scan_velacc((double *)(d + o_pp), (double *)(d + o_ss), 1, nseg, dof, (double *)(d + o_grid), 1, B, G,
                        (double *)(d + o_al), lim_shared, interp, (double *)(d + o_rec),
                        sd_start ? (double *)(d + o_s0) : nullptr, sd_end ? (double *)(d + o_s1) : nullptr, nullptr, 0,
                        (double *)(d + o_K), (double *)(d + o_sd), (double *)(d + o_u), (int *)(d + o_st), nullptr,
                        nullptr, st);
    if (rc) goto done;
  } else {
    rc = tb_coeff_velacc((double *)(d + o_pp), (double *)(d + o_ss), 1, B, nseg, dof, (double *)(d + o_grid), 1, G,
                         vlim ? (double *)(d + o_vl) : nullptr, (double *)(d + o_al), lim_shared, interp,
                         (double *)(d + o_rec), W, R, 0, 1, st);
    if (rc) goto done;
    rc = tb_scan((double *)(d + o_rec), W, R, (double *)(d + o_grid), 1, B, G, sd_start ? (double *)(d + o_s0) : nullptr,
                 sd_end ? (double *)(d + o_s1) : nullptr, (double *)(d + o_K), (double *)(d + o_sd), (double *)(d + o_u),
                 (int *)(d + o_st), nullptr, st);
    if (rc) goto done;
  }
  TB_CUDA(cudaMemcpyAsync(K, d + o_K, sizeof(double) * (size_t)B * G * 2, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaMemcpyAsync(sd, d + o_sd, sizeof(double) * (size_t)B * G, cudaMemcpyDeviceToHost, st));
  if (G > 1) TB_CUDA(cudaMemcpyAsync(u, d + o_u, sizeof(double) * (size_t)B * (G - 1), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaMemcpyAsync(status, d + o_st, sizeof(int) * (size_t)B, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
done:
  if (d) cudaFree(d);
  if (st) cudaStreamDestroy(st);
  return rc;
}
