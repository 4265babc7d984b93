// tb_records.cuh — stage records of joint velocity and acceleration limits, shared by K1 (coeff_velacc_kernel,
// tb_coeff.cu), which evaluates q'(s_i), q''(s_i) from the cubic spline, and rows_velacc_sampled_kernel (tb_poly.cu),
// which loads them from samples of an order-k path; and the velocity bound of JointVelocityConstraintVarying, shared by
// xbound_varying_kernel (tb_coeff.cu) and xbound_varying_sampled_kernel (tb_poly.cu).  The reference functions these
// replace are listed in tb_coeff.cu.
//
// One CTA of VELACC_THREADS threads per (path, chunk of VELACC_CH gridpoints).  Shared memory of one CTA (dof = d,
// VS = 6d + 3 doubles per gridpoint), carved up by each kernel in this order:
//   raw   [(CH+1)][2d]   q'(s_i), q''(s_i) of the chunk (+1 gridpoint for the interpolation lift)
//   cand  [CH][2d]       velocity-bound candidates vlim/q' per joint (upper, lower)
//   vec   [CH][VS]       per gridpoint: q' | a+ | q'' | b+ | -amax | +amin | xlo | xhi | 0
//   sgrid [CH+1]         the chunk's gridpoints
//   the kernel's own doubles (K1: breakpoints and derivative coefficients)
//   tab   [W]            per record column: offset into vec (bit 15 = negate, 0x7fff = column not owned)
// A record kernel runs:
//   phase 0   the chunk's gridpoints into sgrid, velacc_column_table (and the kernel's own loads)
//   phase 1   q', q'' of the chunk's nev gridpoints, each stored by velacc_store_sample
//   __syncthreads()
//   VELACC_WRITE_RECORDS: phase 1b, the per-gridpoint value vectors; phase 2, the records: every thread owns one
//             16-byte column pair and walks down the gridpoints, rec[ci][col] = +-vec[ci][tab[col]] -> two shared
//             loads + one coalesced 16-byte store per iteration.
#pragma once
#include "tb_common.cuh"

namespace tb {

constexpr int VELACC_THREADS = 128;
constexpr int VELACC_CH = 32;  // gridpoints per CTA

__device__ __forceinline__ int R_total_or1(int R_total) { return R_total > 0 ? R_total : 1; }

// Phase 0: the column table of a record of W doubles, where this call owns rows [row0, row0 + Racc) of the R_total
// rows and, when write_xbound, the xbound pair and the padding.
__device__ __forceinline__ void velacc_column_table(unsigned short *tab, const int tid, const int W, const int R_total,
                                                    const int row0, const int Racc, const int dof,
                                                    const int write_xbound) {
  for (int w = tid; w < W; w += VELACC_THREADS) {
    unsigned short code = 0x7fff;  // not owned by this call: leave untouched
    const int kind = w / R_total_or1(R_total), r = w - kind * R_total - row0;
    if (kind < 3 && R_total > 0 && r >= 0 && r < Racc) {
      const int blk = r / dof, k = r - blk * dof;
      const int neg = blk & 1, second = blk >> 1;
      if (kind == 0) code = (unsigned short)((second ? dof + k : k) | (neg << 15));
      else if (kind == 1) code = (unsigned short)((second ? 3 * dof + k : 2 * dof + k) | (neg << 15));
      else code = (unsigned short)(neg ? 5 * dof + k : 4 * dof + k);
    } else if (w >= 3 * R_total) {
      // xlo | xhi | padding zeros; records with a u-bound pair (W >= 3R+4, TB_SCAN_UBOUND) keep those two slots
      const bool ub_slot = (W >= 3 * R_total + 4) && (w == 3 * R_total + 2 || w == 3 * R_total + 3);
      if (write_xbound && !ub_slot)
        code = (unsigned short)(w == 3 * R_total ? 6 * dof : (w == 3 * R_total + 1 ? 6 * dof + 1 : 6 * dof + 2));
    }
    tab[w] = code;
  }
}

// Phase 1: q'(s_ci) = v1 and q''(s_ci) = v2 of joint k, and the joint's velocity-bound candidates.
__device__ __forceinline__ void velacc_store_sample(double *raw, double *cand, const double *vl, const int ci,
                                                    const int k, const int dof, const int npts, const double v1,
                                                    const double v2, const int write_xbound) {
  const double inf_d = __longlong_as_double(0x7ff0000000000000LL);
  raw[ci * 2 * dof + k] = v1;
  raw[ci * 2 * dof + dof + k] = v2;
  if (vl && write_xbound && ci < npts) {
    // _CythonUtils.pyx:44-50: q' > 0: (vmax/q', vmin/q'); q' < 0: (vmin/q', vmax/q'); q' == 0 (or NaN): no update
    const bool posq = v1 > 0, negq = v1 < 0;
    const double qd = (posq || negq) ? v1 : 1.0;
    const double r1 = vl[k * 2 + 1] / qd, r0 = vl[k * 2 + 0] / qd;
    cand[ci * 2 * dof + k] = posq ? r1 : (negq ? r0 : inf_d);          // candidate for sdmax
    cand[ci * 2 * dof + dof + k] = posq ? r0 : (negq ? r1 : -inf_d);   // candidate for sdmin
  }
}

// Phases 1b and 2 of the CTA, after the __syncthreads() that ends phase 1.  The arguments are the kernel's locals of the
// same names: path / i0 / npts the CTA's path, first gridpoint and gridpoints written, N = G - 1, al / vl the path's
// limits or null.  A macro, not a function: nvcc optimises a called function before it inlines it, and as a function
// these phases change the machine code of K1.
#define VELACC_WRITE_RECORDS(raw, cand, vec, sgrid, tab, al, vl, records, path, G, i0, N, npts, dof, VS, W, R_total,    \
                             write_xbound, tid)                                                                         \
  do {                                                                                                                      \
    /* ---- phase 1b: per-gridpoint value vectors ---- */                                                                   \
    double *rec0 = records + (path * G + i0) * (long)W;                                                                     \
    for (int idx = tid; idx < npts * dof; idx += VELACC_THREADS) {                                                          \
      const int ci = idx / dof, k = idx - ci * dof;                                                                         \
      const int gi = i0 + ci;                                                                                               \
      double *v = vec + ci * VS;                                                                                            \
      const double a = raw[ci * 2 * dof + k], b = raw[ci * 2 * dof + dof + k];                                              \
      double ap = a, bp = b;  /* last gridpoint duplicates itself, linear_constraint.py:171,175 */                          \
      if (gi < N) {                                                                                                         \
        const double delta = sgrid[ci + 1] - sgrid[ci];                                                                     \
        ap = raw[(ci + 1) * 2 * dof + k] + (2 * delta) * raw[(ci + 1) * 2 * dof + dof + k];  /* linear_constraint.py:170 */ \
        bp = raw[(ci + 1) * 2 * dof + dof + k];                                                                             \
      }                                                                                                                     \
      v[k] = a; v[dof + k] = ap; v[2 * dof + k] = b; v[3 * dof + k] = bp;                                                   \
      if (al) {                                                                                                             \
        v[4 * dof + k] = 0.0 - al[k * 2 + 1];       /* F.c - g with c = 0, g = [amax; -amin] */                             \
        v[5 * dof + k] = 0.0 - (-al[k * 2 + 0]);                                                                            \
      }                                                                                                                     \
      if (k == 0 && write_xbound) {                                                                                         \
        /* velocity bound of this gridpoint: fp32 running min/max over the joints exactly like _CythonUtils.pyx:41-58 */    \
        double xlo = VAR_MIN, xhi = VAR_MAX;  /* seidelWrapper low_arr/high_arr init, pyx:477-478 */                        \
        if (vl) {                                                                                                           \
          /* The reference keeps the running min/max in C floats: s <- (float)min(cand_k, (double)s), k = 0..dof-1, */      \
          /* s_0 = 1e8f (_CythonUtils.pyx:41-50).  Round-to-nearest is monotone and idempotent, so that chain equals */     \
          /* (float)min(1e8, min_k cand_k) (likewise for the max): reduce in fp64, round once. */                           \
          double mhi = JVEL_MAXSD, mlo = -JVEL_MAXSD;                                                                       \
          for (int kk = 0; kk < dof; ++kk) {                                                                                \
            const double hi = cand[ci * 2 * dof + kk], lo = cand[ci * 2 * dof + dof + kk];                                  \
            mhi = (hi <= mhi) ? hi : mhi;                                                                                   \
            mlo = (lo >= mlo) ? lo : mlo;                                                                                   \
          }                                                                                                                 \
          const float sdmax = __double2float_rn(mhi), sdmin = __double2float_rn(mlo);                                       \
          const float up = __fmul_rn(sdmax, sdmax);                          /* powf(sdmax, 2) in fp32 */                   \
          const double lo_d = ((double)sdmin >= 0.0) ? (double)sdmin : 0.0;  /* float64_max(sdmin, 0.) */                   \
          xlo = lo_d * lo_d;                                                                                                \
          xhi = (double)up;                                                                                                 \
          if (write_xbound != 2) {                                                                                          \
            /* pyx:517-520: low = max(VAR_MIN, xbound_lo), high = min(VAR_MAX, xbound_hi) */                                \
            xlo = fmax(VAR_MIN, xlo);                                                                                       \
            xhi = fmin(VAR_MAX, xhi);                                                                                       \
          }                                                                                                                 \
        }                                                                                                                   \
        if (write_xbound == 3) {  /* intersect with what the record already holds */                                        \
          const double *rec = rec0 + (long)ci * W;                                                                          \
          xlo = fmax(rec[3 * R_total], xlo);                                                                                \
          xhi = fmin(rec[3 * R_total + 1], xhi);                                                                            \
        }                                                                                                                   \
        v[6 * dof] = xlo; v[6 * dof + 1] = xhi; v[6 * dof + 2] = 0.0;                                                       \
      }                                                                                                                     \
    }                                                                                                                       \
    __syncthreads();                                                                                                        \
                                                                                                                            \
    /* ---- phase 2: stream the records out; thread -> fixed 16-byte column pair, loop over gridpoints ---- */              \
    const int Wh = W >> 1;                                                                                                  \
    const int ngrp = VELACC_THREADS / Wh;  /* gridpoints written per sweep (threads beyond ngrp * Wh idle) */               \
    const int g = tid / Wh, j = tid - g * Wh;                                                                               \
    if (ngrp > 0 && g < ngrp) {                                                                                             \
      const unsigned short c0 = tab[2 * j], c1 = tab[2 * j + 1];                                                            \
      const int o0 = c0 & 0x7fff, o1 = c1 & 0x7fff;                                                                         \
      const bool n0 = (c0 & 0x8000) != 0, n1 = (c1 & 0x8000) != 0;                                                          \
      const bool own0 = c0 != 0x7fff, own1 = c1 != 0x7fff;                                                                  \
      double *dst = rec0 + (long)g * W + 2 * j;                                                                             \
      const double *v = vec + g * VS;                                                                                       \
      if (own0 && own1) {                                                                                                   \
        for (int ci = g; ci < npts; ci += ngrp, dst += (long)ngrp * W, v += ngrp * VS) {                                    \
          double2 o;                                                                                                        \
          o.x = n0 ? -v[o0] : v[o0];                                                                                        \
          o.y = n1 ? -v[o1] : v[o1];                                                                                        \
          __stcs(reinterpret_cast<double2 *>(dst), o);  /* streaming store: written once, read later by K2 */               \
        }                                                                                                                   \
      } else if (own0 || own1) {                                                                                            \
        for (int ci = g; ci < npts; ci += ngrp, dst += (long)ngrp * W, v += ngrp * VS) {                                    \
          if (own0) dst[0] = n0 ? -v[o0] : v[o0];                                                                           \
          if (own1) dst[1] = n1 ? -v[o1] : v[o1];                                                                           \
        }                                                                                                                   \
      }                                                                                                                     \
    } else if (ngrp == 0) {  /* records wider than 2 * VELACC_THREADS columns: column loop per gridpoint */                 \
      for (int ci = 0; ci < npts; ++ci)                                                                                     \
        for (int w = tid; w < W; w += VELACC_THREADS) {                                                                     \
          const unsigned short cw = tab[w];                                                                                 \
          if (cw != 0x7fff) {                                                                                               \
            const double t = vec[ci * VS + (cw & 0x7fff)];                                                                  \
            rec0[(long)ci * W + w] = (cw & 0x8000) ? -t : t;                                                                \
          }                                                                                                                 \
        }                                                                                                                   \
    }                                                                                                                       \
  } while (0)

// JointVelocityConstraintVarying at one gridpoint (linear_joint_velocity.py:56-87, _CythonUtils.pyx:61-101): the fp32
// running min/max of vlim/q' over the joints, then x in [max(sdmin, 0)^2, sdmax^2] into rec's xbound pair.  qd(k) is
// q'_k of joint k; q'_k == 0 or NaN updates nothing, and so does every joint when `valid` is false.  mode 1 clamps to
// [VAR_MIN, VAR_MAX], 2 writes the bound as it is, 3 clamps and intersects with what rec holds.
template <class Qd>
__device__ __forceinline__ void velocity_xbound(const Qd &qd, const bool valid, const int dof, const double *vl,
                                                double *rec, const int R_total, const int mode) {
  float sdmin = -(float)JVEL_MAXSD, sdmax = (float)JVEL_MAXSD;
  for (int k = 0; k < dof && valid; ++k) {
    const double q = qd(k);
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
  if (mode != 2) { xlo = fmax(VAR_MIN, xlo); xhi = fmin(VAR_MAX, xhi); }
  if (mode == 3) { xlo = fmax(rec[3 * R_total], xlo); xhi = fmin(rec[3 * R_total + 1], xhi); }
  rec[3 * R_total] = xlo;
  rec[3 * R_total + 1] = xhi;
}

// ---- host side of both record entries ----

// The record-shape checks after the pointer checks: 0, or the TB_ERR_* code (message set, prefixed with `what`).
inline int velacc_check(const char *what, const int Racc, const int dof, const int W, const int R_total,
                        const int row0, const long blocks) {
  if (row0 < 0 || row0 + Racc > R_total || W < 3 * R_total + 2) {
    set_error("%s: rows [%d,%d) do not fit R_total=%d / W=%d", what, row0, row0 + Racc, R_total, W);
    return TB_ERR_ARG;
  }
  if (R_total > MAX_ROWS) { set_error("%s: R=%d > %d", what, R_total, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (6 * dof + 3 >= 0x7fff) { set_error("%s: dof=%d too large", what, dof); return TB_ERR_UNSUPPORTED; }
  if (blocks > 0x7fffffffL) { set_error("%s: batch too large for one launch", what); return TB_ERR_UNSUPPORTED; }
  return 0;
}

// Dynamic shared memory of one CTA of `kernel`, with `extra` doubles of the kernel's own, opted in above 48 KB: the
// size in bytes, or 0 when the device cannot give it (message set).
template <class Kernel>
size_t velacc_smem(const char *what, Kernel kernel, const int dof, const int W, const size_t extra) {
  const size_t smem = (size_t)((VELACC_CH + 1) * dof * 2 + VELACC_CH * dof * 2 + VELACC_CH * (6 * dof + 3) +
                               VELACC_CH + 1 + extra) * sizeof(double) + (size_t)W * sizeof(unsigned short) + 16;
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("%s: dof=%d too large for shared memory", what, dof);
    return 0;
  }
  return smem;
}

}  // namespace tb
