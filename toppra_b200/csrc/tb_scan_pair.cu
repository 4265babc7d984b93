// tb_scan_pair.cu — K2 for JointVelocity + JointAcceleration problems, TWO PATHS PER WARP.  EXPERIMENT, opt-in
// (TB_SCAN_PAIR=1: divergent half-warps, TB_SCAN_PAIR=2: lockstep): both forms are bit-identical to the one-warp-per-path
// kernel on the whole GPU test suite and both were measured slower than it (DESIGN.md section 10).  The default launch
// path does not use this file.
//
// Replaces the same reference functions as tb_scan.cu (reachability_algorithm.py:166-376, time_optimal_algorithm.py:55-92,
// cy_seidel_solverwrapper.pyx:93-144, 149-390, 549-697); results are bit-identical to it and to the one-warp-per-path
// kernel (same tests).
//
// Why: the one-warp-per-path scan is bound by instruction issue and by the dependent chain of each path; most of its
// instructions are warp-uniform control (row search, broadcasts, reductions, shortcut tests) paid once per path although
// only 30 of 32 lanes hold a row.  The acceleration rows come in +- PAIRS by construction (F = [I; -I]:
// amin <= a u + b x <= amax), and so do the two x_next rows (xn_min <= 2 delta u + x <= xn_max) and the box rows.  A lane
// therefore holds a SLAB — base (a, b) with row P = (a, b, cP) and row N = (-a, -b, cN) — a path needs 2 dof + 1 <= 15
// lanes, and a warp carries two paths in its two half-warps.  Every collective (shuffle, redux, vote) names only the
// half-warp's 16 lanes, so the halves are free to diverge (different numbers of re-solves) and run converged otherwise.
// Per pair the shared products are computed once:  val_N = -(a p0 + b p1) + cN,  denom_N = -denom_P,
// num_N = (cN - z1 b) - z0 a, and both quotients share the divisor — all exact consequences of IEEE negation, so every
// number equals the reference's row-by-row arithmetic bit for bit.
//
// Lane map of a half-warp (l = 0..15):  l = 0: x_next slab, P = row 1 (2 delta, 1, -xn_max), N = row 0;
// l = 1 + s dof + k: joint k of block pair s (s = 1: the lifted block of the interpolation scheme), P = row 2 + 2 s dof + k,
// N = row P + dof;  remaining lanes: padding (0, 0, -1).  The four box rows of a re-solve ride as two slabs
// (u: (1, 0, -high0 | low0), x: (0, 1, -high1 | low1)) on lanes whose rows do not take part (the padding lane is always
// one), with a fallback slot when fewer than two such lanes exist.
#include <stdlib.h>

#include "tb_scan_common.cuh"

namespace tb {
namespace {

constexpr int GL = 16;  // lanes per path

// min over the lanes of `gmask` (a half-warp) of doubles without NaNs: two 32-bit redux.sync on order-preserving keys
__device__ __forceinline__ double grp_min(const double v, const unsigned gmask) {
  const int hi = __double2hiint(v), lo = __double2loint(v);
  const int m = hi >> 31;
  const unsigned khi = (unsigned)(hi ^ (m | (int)0x80000000)), klo = (unsigned)(lo ^ m);
  const unsigned mh = __reduce_min_sync(gmask, khi);
  const unsigned ml = __reduce_min_sync(gmask, khi == mh ? klo : 0xffffffffu);
  const int m2 = ((int)~mh) >> 31;
  return __hiloint2double((int)(mh ^ (unsigned)(m2 | (int)0x80000000)), (int)(ml ^ (unsigned)m2));
}

// One slab (both rows) projected onto the line of a re-solve (pyx:298-347).  partP / partN: the row takes part.
// Row P: denom = dP, num = (cP + z1 b) + z0 a;  row N: denom = -dP, num = (cN - z1 b) - z0 a  (exact negations), so
// t_P = -numP / dP and t_N = -numN / (-dP) = numN / dP.  dP > TINY: P bounds t from above and N from below; dP < -TINY:
// the other way round; otherwise parallel (infeasible if num > SMALL).  Outputs: this lane's upper / lower limit with
// the order keys of the rows they come from (+-LP_INF / INT_MAX when absent).
__device__ __forceinline__ void project_slab(const bool partP, const bool partN, const double a, const double b,
                                             const double cP, const double cN, const int keyP, const int keyN,
                                             const double dt0, const double dt1, const double z0, const double z1,
                                             double &thi, double &tlo, int &khi, int &klo, bool &bad) {
  const double dP = dt0 * a + dt1 * b;
  const double zb = z1 * b, za = z0 * a;
  const double numP = (cP + zb) + za;
  const double numN = (cN - zb) - za;
  const bool dpos = dP > LP_TINY, dneg = dP < -LP_TINY;
  const double dsafe = (dpos || dneg) ? dP : 1.0;   // the IEEE division never leaves its fast path for discarded values
  const double qP = -numP / dsafe;
  const double qN = numN / dsafe;
  const bool upP = partP && dpos, upN = partN && dneg, dnP = partP && dneg, dnN = partN && dpos;
  const double tu = upP ? qP : qN, tl = dnP ? qP : qN;
  // `cur_x < cur_max` / `cur_x > cur_min` (pyx:115-124): a limit at or beyond the sentinel, or NaN, never wins
  const bool hu = (upP || upN) && (tu < LP_INF), hl = (dnP || dnN) && (tl > -LP_INF);
  thi = hu ? tu : LP_INF;
  tlo = hl ? tl : -LP_INF;
  khi = upP ? keyP : keyN;
  klo = dnP ? keyP : keyN;
  bad = bad || (!(dpos || dneg) && ((partP && numP > LP_SMALL) || (partN && numN > LP_SMALL)));
}

// cy_solve_lp2d (pyx:149-390) on one half-warp; see lp2d_impl in tb_scan.cu for the row-per-lane form this mirrors
// statement by statement (start vertex, row order incl. the warm-start permutation, shortcuts A / B, projected
// re-solves, active pair).  rP / rN: LP row indices of this lane's slab (-1: padding).
template <bool PERM, bool SKIP>
__device__ __forceinline__ bool lp2d_pair_impl(const double v0, const double v1, const double a, const double b,
                                               const double cP, const double cN, const int rP, const int rN,
                                               const double low0, const double high0, const double low1,
                                               const double high1, int &ac0, int &ac1, double &out_u, double &out_x,
                                               const int l, const unsigned gmask, const int gbase) {
  double p0 = (v0 > LP_TINY) ? high0 : low0;       // pyx:236-247
  double p1 = (v1 > LP_TINY) ? high1 : low1;
  int nac0 = (v0 > LP_TINY) ? -2 : -1;
  int nac1 = (v1 > LP_TINY) ? -4 : -3;
  constexpr bool valid = PERM;
  const int posP = (rP >= 0) ? row_pos(rP, valid, ac0, ac1) : INT_MAX;
  const int posN = (rN >= 0) ? row_pos(rN, valid, ac0, ac1) : INT_MAX;
  const unsigned lt_mask = (1u << l) - 1u;
  int kpos = -1;
  const bool skip_ok = SKIP && (((v0 > LP_TINY) && (v1 < 0)) || ((v0 < -LP_TINY) && (v1 > 0)));
  while (true) {
    int knew = INT_MAX;
    if constexpr (SKIP && !PERM) {
      if (kpos < 0 && skip_ok) {
        // Shortcut A (natural order; DESIGN.md section 4 K2, lp2d_impl in tb_scan.cu): the last row the reference's walk
        // visits is the row m with the smallest own bound on ua = sg u at x = its box bound; one exact re-solve on m.
        const double sg = (v0 > 0) ? 1.0 : -1.0;
        const double x = p1, u0m = sg * p0;
        const double sa = sg * a;                                   // row P; row N: -sa
        const bool aup = sa > LP_TINY, adn = sa < -LP_TINY, any = aup || adn;
        const bool realP = posP != INT_MAX, realN = posN != INT_MAX;
        const bool uprP = realP && aup, uprN = realN && adn, lorP = realP && adn, lorN = realN && aup;
        const double bx = b * x;
        const double bxcP = bx + cP, bxcN = -bx + cN;
        const double den = any ? a : 1.0;
        // own bounds u_j = -(b_j x + c_j) / a_j; a zero numerator would take the division's slow path: these values only
        // feed the margin tests, 0 is substituted directly
        const bool znP = (bxcP == 0.0), znN = (bxcN == 0.0);
        const double qdP = -opaque(znP ? 1.0 : bxcP) / den;
        const double qdN = opaque(znN ? 1.0 : bxcN) / den;           // -bxcN / (-a)
        const double uoP = znP ? 0.0 : sg * qdP, uoN = znN ? 0.0 : sg * qdN;
        // the upper row of this slab (if any) and its data; the other row is the lower one
        const bool hasU = uprP || uprN;
        const double uoU = uprP ? uoP : uoN;
        const int posU = uprP ? posP : posN;
        const double v1dP = (-b) * v0 + a * v1;                      // the exact path's v1d if row P were visited; row N: -v1dP
        const double v1dU = uprP ? v1dP : -v1dP;
        bool bad = hasU && !((fabs(v1dU) < LP_TINY) || (v1dU < 0));
        // line parameter of the landing point of the upper row: |x a_j - (sg uo) b_j| < TMAX (a^2 + b^2)
        const double aU = uprP ? a : -a, bU = uprP ? b : -b;
        bad = bad || (hasU && !(fabs(x * aU - (sg * uoU) * bU) < SKIP_TMAX * (aU * aU + bU * bU)));
        const double um = grp_min(hasU ? uoU : SKIP_BIG, gmask);
        const int m = __reduce_min_sync(gmask, (hasU && uoU == um) ? posU : INT_MAX);
        if (m != INT_MAX) {
          double second = grp_min((hasU && posU != m) ? uoU : SKIP_BIG, gmask);
          second = (u0m < second) ? u0m : second;
          // row m itself (an upper row): violated at the second-smallest bound by the margin
          if (hasU && posU == m) {
            const double cU = uprP ? cP : cN, bxcU = uprP ? bxcP : bxcN;
            const double au = aU * (sg * second);
            const double val = au + bxcU;
            bad = bad || !(val >= SKIP_GAP * (1.0 + fabs(au) + fabs(bU * x) + fabs(cU)));
          }
          // rows before m: lower rows must hold at the final u with a margin, rows with a ~ 0 must be clearly satisfied
          if (posP < m && !(uprP && posP == m))
            bad = bad || (lorP && (uoP > um - 1e-9 * (1.0 + fabs(um)))) || (!uprP && !lorP && ((bxcP > -1e-9) || (a != 0.0)));
          if (posN < m && !(uprN && posN == m))
            bad = bad || (lorN && (uoN > um - 1e-9 * (1.0 + fabs(um)))) || (!uprN && !lorN && ((bxcN > -1e-9) || (a != 0.0)));
          const double ur = sg * um;
          bad = bad || (ur < low0 + 1.0) || (ur > high0 - 1.0);
          if (!__any_sync(gmask, bad)) knew = m;
        }
      }
    }
    if (knew == INT_MAX) {
      // first row (in order) violated at the current point, pyx:269-275.  NaN counts as violated (not `< TINY`).
      const double s = a * p0 + b * p1;
      const double valP = s + cP, valN = -s + cN;
      const bool candP = !(valP < LP_TINY) && (posP > kpos) && (posP != INT_MAX);
      const bool candN = !(valN < LP_TINY) && (posN > kpos) && (posN != INT_MAX);
      const int mypos = min(candP ? posP : INT_MAX, candN ? posN : INT_MAX);
      knew = __reduce_min_sync(gmask, mypos);
      if (knew == INT_MAX) break;
      if constexpr (SKIP && PERM) {
        if (kpos < 0 && skip_ok && knew == 0) {
          // Shortcut B (valid warm-start pair: order = row p = ac1, row k = ac0, the rest): see lp2d_impl
          const bool mineP = (rP == ac1), mineN = (rN == ac1);
          const unsigned holder = __ballot_sync(gmask, mineP || mineN);
          const int src = __ffs(holder) - 1;
          const double ap = __shfl_sync(gmask, mineN ? -a : a, src);
          const double bp = __shfl_sync(gmask, mineN ? -b : b, src);
          const double cp = __shfl_sync(gmask, mineN ? cN : cP, src);
          bool okb = fabs(ap) > 1e-6;
          const double ia = 1.0 / (okb ? ap : 1.0);
          okb = okb && (low1 <= high1 - 1e-7 * (1.0 + fabs(low1) + fabs(high1)));
          const double slp = v1 - v0 * bp * ia;
          okb = okb && !(fabs(slp) < 1e-6);
          const double sx = (slp > 0) ? high1 : low1;
          const double su = -(bp * sx + cp) * ia;
          okb = okb && (su >= low0 + 1.0) && (su <= high0 - 1.0);
          okb = okb && (fabs(sx * ap - su * bp) < 1e9 * (ap * ap + bp * bp));
          // row k = the row at position 1: violated at (su, sx) by the margin?
          const double t1P = a * su, t2P = b * sx;                   // row N: -t1P, -t2P
          const double vP = t1P + t2P + cP, vN = -t1P + -t2P + cN;
          const double mag = fabs(t1P) + fabs(t2P);
          const bool kviol = ((posP == 1) && (vP >= SKIP_GAP * (1.0 + mag + fabs(cP)))) ||
                             ((posN == 1) && (vN >= SKIP_GAP * (1.0 + mag + fabs(cN))));
          if (__any_sync(gmask, kviol) && okb) knew = 1;
        }
      }
    }
    kpos = knew;
    const int krow = pos_row(kpos, valid, ac0, ac1);
    nac0 = krow;
    // broadcast row k from the lane that holds it (as row P or as row N)
    const bool kN = (rN == krow);
    const unsigned holder = __ballot_sync(gmask, (rP == krow) || kN);
    const int src = __ffs(holder) - 1;
    const double ak = __shfl_sync(gmask, kN ? -a : a, src);
    const double bk = __shfl_sync(gmask, kN ? -b : b, src);
    const double ck = __shfl_sync(gmask, kN ? cN : cP, src);
    // project the origin onto line k, pyx:290-295; one division sequence for both components (odd lanes: the second)
    const double nrm = ak * ak + bk * bk;
    const double zq = ((l & 1) ? (-bk * ck) : (-ak * ck)) / nrm;
    const double z0 = __shfl_sync(gmask, zq, gbase);
    const double z1 = __shfl_sync(gmask, zq, gbase + 1);
    const double dt0 = -bk, dt1 = ak;
    const double v1d = dt0 * v0 + dt1 * v1;
    // earlier rows and the four box rows onto the line, pyx:298-347
    const bool partP = posP < kpos, partN = posN < kpos;
    const bool idle = !(partP || partN);
    const unsigned idleb = (__ballot_sync(gmask, idle) >> gbase) & 0xffffu;
    const int inl = min(__popc(idleb), 2);                           // box slabs that ride on idle lanes (half-warp-uniform)
    const int rank = __popc(idleb & lt_mask);
    const bool isbox = idle && rank < inl;                           // slab `rank`: 0 = the u box, 1 = the x box
    double thi, tlo;
    int khi, klo;
    bool bad = false;
    {
      const bool bu = rank == 0;
      const double ba = isbox ? (bu ? 1.0 : 0.0) : a, bb = isbox ? (bu ? 0.0 : 1.0) : b;
      const double bcP = isbox ? (bu ? -high0 : -high1) : cP, bcN = isbox ? (bu ? low0 : low1) : cN;
      // keys: box row m = 0: low0 <= u, 1: u <= high0, 2: low1 <= x, 3: x <= high1  (P = the upper bound of the slab)
      const int kP = isbox ? BOXBASE + (bu ? 1 : 3) : posP, kN2 = isbox ? BOXBASE + (bu ? 0 : 2) : posN;
      project_slab(isbox || partP, isbox || partN, ba, bb, bcP, bcN, kP, kN2, dt0, dt1, z0, z1, thi, tlo, khi, klo, bad);
    }
    double my_hi = thi, my_lo = tlo;
    double fhi = LP_INF, flo = -LP_INF;
    int fkhi = INT_MAX, fklo = INT_MAX;
    if (inl < 2) {  // fewer than two idle lanes: the remaining box slab(s) take an extra item on lanes 0.. of the half-warp
      const int slab = inl + l;                                      // lane l handles box slab inl + l (< 2)
      const bool bu = slab == 0;
      project_slab(slab < 2, slab < 2, bu ? 1.0 : 0.0, bu ? 0.0 : 1.0, bu ? -high0 : -high1, bu ? low0 : low1,
                   BOXBASE + (bu ? 1 : 3), BOXBASE + (bu ? 0 : 2), dt0, dt1, z0, z1, fhi, flo, fkhi, fklo, bad);
      my_hi = (fhi < my_hi) ? fhi : my_hi;
      my_lo = (flo > my_lo) ? flo : my_lo;
    }
    // 1-D LP on the line with bounds +-INF, pyx:350 -> cy_solve_lp1d pyx:93-144: only the optimal end is reduced
    // exactly; "cur_min > cur_max" is a vote against the other side
    const bool pick_min = (fabs(v1d) < LP_TINY) || (v1d < 0);
    const double red = grp_min(pick_min ? -my_lo : my_hi, gmask);
    const double tstar = pick_min ? -red : red;
    const bool cross = pick_min ? (my_hi < tstar) : (my_lo > tstar);
    if (__any_sync(gmask, bad || cross)) return false;
    if (tstar == (pick_min ? -LP_INF : LP_INF)) return false;       // optimum on the sentinel: infeasible, pyx:376-383
    // active item = lowest key among the items that attain the optimum (sentinels never match a finite tstar)
    int mykey = ((pick_min ? tlo : thi) == tstar) ? (pick_min ? klo : khi) : INT_MAX;
    if (inl < 2) mykey = ((pick_min ? flo : fhi) == tstar) ? min(mykey, pick_min ? fklo : fkhi) : mykey;
    const int akey = __reduce_min_sync(gmask, mykey);
    nac1 = (akey >= BOXBASE) ? (-1 - (akey - BOXBASE)) : pos_row(akey, valid, ac0, ac1);
    p0 = z0 + tstar * dt0;  // pyx:362-363
    p1 = z1 + tstar * dt1;
  }
  ac0 = nac0;
  ac1 = nac1;
  out_u = p0;
  out_x = p1;
  return true;
}

template <bool SKIP>
__device__ __forceinline__ bool lp2d_pair(const double v0, const double v1, const double a, const double b,
                                          const double cP, const double cN, const int rP, const int rN, const int nC,
                                          const double low0, const double high0, const double low1, const double high1,
                                          int &ac0, int &ac1, double &out_u, double &out_x, const int l,
                                          const unsigned gmask, const int gbase) {
  if (low0 > high0 || low1 > high1) return false;  // pyx:233-235
  const bool valid = ac0 >= 0 && ac0 < nC && ac1 >= 0 && ac1 < nC && ac0 != ac1;  // uniform over the half-warp
  if (valid)
    return lp2d_pair_impl<true, SKIP>(v0, v1, a, b, cP, cN, rP, rN, low0, high0, low1, high1, ac0, ac1, out_u, out_x, l,
                                      gmask, gbase);
  return lp2d_pair_impl<false, SKIP>(v0, v1, a, b, cP, cN, rP, rN, low0, high0, low1, high1, ac0, ac1, out_u, out_x, l,
                                     gmask, gbase);
}

// cy_solve_lp1d (pyx:93-144) in the x_min == x_max branch of solve_stagewise_optim (pyx:631-650) on slabs:
// row P: a u + (b x + cP) <= 0, row N: -a u + (-b x + cN) <= 0.  a > TINY: P bounds u from above, N from below.
__device__ __forceinline__ bool lp1d_pair(const double v0, const double x, const double a, const double b,
                                          const double cP, const double cN, const double low0, const double high0,
                                          double &out_u, const unsigned gmask) {
  const double bx = b * x;
  const double bxcP = bx + cP, bxcN = -bx + cN;
  const bool ap = a > LP_TINY, an = a < -LP_TINY;
  const double den = (ap || an) ? a : 1.0;
  // a zero numerator is not divided (the IEEE division's slow path): (-bxc) * den is the quotient's correctly signed zero
  const bool znP = (bxcP == 0.0), znN = (bxcN == 0.0);
  const double qP0 = -opaque(znP ? 1.0 : bxcP) / den;
  const double qN0 = opaque(znN ? 1.0 : bxcN) / den;                 // -bxcN / (-a)
  const double tP = znP ? (-bxcP) * den : qP0;
  const double tN = znN ? (-bxcN) * (-den) : qN0;
  // a > TINY: t_P is an upper limit, t_N a lower one; a < -TINY: the other way round
  const double tu = ap ? tP : tN, tl = ap ? tN : tP;
  double my_hi = high0, my_lo = low0;
  my_hi = ((ap || an) && tu < my_hi) ? tu : my_hi;
  my_lo = ((ap || an) && tl > my_lo) ? tl : my_lo;
  const bool pick_min = (fabs(v0) < LP_TINY) || (v0 < 0);
  const double red = grp_min(pick_min ? -my_lo : my_hi, gmask);
  const double ustar = pick_min ? -red : red;
  if (__any_sync(gmask, pick_min ? (my_hi < ustar) : (my_lo > ustar))) return false;
  out_u = ustar;
  return true;
}

// CFLAGS: compile-time scan mode (0 full scan, TB_SCAN_BACKWARD_ONLY, TB_SCAN_FORWARD_ONLY).  FAST: TB_SCAN_FAST_LOWER.
template <bool FAST, int CFLAGS, int MINB>
__global__ void __launch_bounds__(32, MINB)
scan_pair_kernel(const VelAccSrc src, const int interp, const int Wc, const double *__restrict__ grid, const int grid_shared,
                 const int B, const int G, const double *__restrict__ sd_start, const double *__restrict__ sd_end,
                 const double *__restrict__ sd_end_hi, double *__restrict__ Kout, double *__restrict__ sdout,
                 double *__restrict__ uout, int *__restrict__ status, int *__restrict__ fail_stage) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = (int)threadIdx.x;
  const int grp = lane >> 4, l = lane & 15, gbase = grp * GL;
  const unsigned gmask = 0xffffu << gbase;
  const long path = (long)blockIdx.x * 2 + grp;
  if (path >= B) return;   // an odd batch: the second half-warp of the last warp has no path (it is in no mask)
  constexpr bool backward_only = (CFLAGS & TB_SCAN_BACKWARD_ONLY) != 0;
  constexpr bool forward_only = (CFLAGS & TB_SCAN_FORWARD_ONLY) != 0;
  const int N = G - 1, nseg = src.nseg, dof = src.dof;
  const int nblk = interp ? 2 : 1;                 // block pairs: plain, lifted
  const int nC = 2 * nblk * dof + 2;
  // shared memory per half-warp: derivative coefficients of the PPoly dco [nseg][dof][6] + breakpoints [nseg + 1]
  double *bufs = reinterpret_cast<double *>(smem_raw) + (size_t)grp * Wc;
  const double *dco = bufs, *sx = bufs + nseg * dof * 6;
  {
    const double *cpp = src.ppoly + (size_t)path * 4 * nseg * dof;
    const double *xb = src.breaks + (src.breaks_shared ? 0 : (size_t)path * (nseg + 1));
    double *dco_w = bufs, *sx_w = bufs + nseg * dof * 6;
    for (int q = l; q < nseg * dof; q += GL) {
      // scipy PPoly.derivative: c'[j] = c[j] * (k - j); cspldd = cspld.derivative() (interpolator.py:419-421)
      const double c0 = cpp[q], c1 = cpp[nseg * dof + q], c2 = cpp[2 * nseg * dof + q];
      const double d0 = c0 * 3.0, d1 = c1 * 2.0, d2 = c2 * 1.0;
      double *o = dco_w + q * 6;
      o[0] = d0; o[1] = d1; o[2] = d2; o[3] = d0 * 2.0; o[4] = d1 * 1.0; o[5] = 0.0;
    }
    for (int q = l; q <= nseg; q += GL) sx_w[q] = xb[q];
  }
  // this lane's slab: l = 0: x_next rows (P = row 1, N = row 0); l = 1 + s dof + k: joint k of block pair s
  const bool isj = (l >= 1) && (l - 1 < nblk * dof);
  const int f_second = isj ? (l - 1) / dof : 0;
  const int f_k = isj ? (l - 1) - f_second * dof : 0;
  const int rP = (l == 0) ? 1 : (isj ? 2 + 2 * f_second * dof + f_k : -1);
  const int rN = (l == 0) ? 0 : (isj ? rP + dof : -1);
  double cP = -1.0, cN = -1.0;
  if (isj) {
    const double *al = src.alim + (src.lim_shared ? 0 : (size_t)path * dof * 2);
    cP = 0.0 - al[f_k * 2 + 1];          // F c - g with c = 0, g = [amax; -amin] (tb_coeff.cu phase 1b)
    cN = 0.0 - (-al[f_k * 2 + 0]);
  }
  int f_seg = 0;
  __syncwarp(gmask);
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  const double *xbp = src.xbound + (size_t)path * G * 2;
  double *Kp = Kout + (size_t)path * G * 2;
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);
  // base (a, b) of this lane's joint slab at stage i: K1's arithmetic (scipy evaluate_poly1 on the derivative coefficients,
  // interpolation lift a+ = q'(s_{i+1}) + 2 delta q''(s_{i+1})); the segment index is carried from stage to stage
  auto slab_ab = [&](const double s0, const double s1, const bool down, const double delta, double &ra, double &rb) {
    const double s = f_second ? s1 : s0;
    if (down) { while (f_seg > 0 && s < sx[f_seg]) --f_seg; }
    else { while (f_seg < nseg - 1 && s >= sx[f_seg + 1]) ++f_seg; }
    const double ds = s - sx[f_seg];
    const double2 *o = reinterpret_cast<const double2 *>(dco + (f_seg * dof + f_k) * 6);
    const double2 o01 = o[0], o23 = o[1], o45 = o[2];
    double z = ds;
    double v1 = 0.0 + o23.x;
    v1 = v1 + o01.y * z;
    z = z * ds;
    v1 = v1 + o01.x * z;
    double v2 = 0.0 + o45.x;
    v2 = v2 + o23.y * ds;
    const double va = f_second ? (v1 + (2 * delta) * v2) : v1;  // lift, linear_constraint.py:170
    ra = isj ? va : 0.0;
    rb = isj ? v2 : 0.0;
  };

  // ---------------- backward pass: controllable sets, reachability_algorithm.py:166-238 ----------------
  const double sde = sd_end ? sd_end[path] : 0.0;
  const double sds = sd_start ? sd_start[path] : 0.0;
  const double sdeh = sd_end_hi ? sd_end_hi[path] : sde;
  double kn0 = sde * sde, kn1 = sdeh * sdeh;  // K[N] = [sdmin^2, sdmax^2]
  if (l == 0 && !forward_only) { Kp[2 * N] = kn0; Kp[2 * N + 1] = kn1; }
  int st = TB_STATUS_OK, fstage = -1;
  int up0 = 0, up1 = 0, dn0 = 0, dn1 = 0;  // active_c_up / active_c_down (pyx:526-527)
  if (forward_only) {
    st = status[path];
    fstage = fail_stage ? fail_stage[path] : -1;
    kn0 = Kp[0];
    kn1 = Kp[1];
  }
  double2 xb_ahead = make_double2(0.0, 0.0);
  f_seg = nseg - 1;
  if (!forward_only && N > 0) xb_ahead = reinterpret_cast<const double2 *>(xbp)[N - 1];
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  double a, b;
  for (int i = forward_only ? -1 : N - 1; i >= 0; --i) {
    const double g0 = gp[i], g1 = gp[i + 1];
    const double delta = g1 - g0;
    slab_ab(g0, g1, true, delta, a, b);
    const double xlo = xb_ahead.x, xhi = xb_ahead.y;
    if (i > 0) xb_ahead = reinterpret_cast<const double2 *>(xbp)[i - 1];
    // x_next slab on lane 0 (pyx:604-620): row 0 = (-2 delta, -1, x_next_min), row 1 = (2 delta, 1, -x_next_max)
    const double sa = (l == 0) ? 2 * delta : a, sb = (l == 0) ? 1.0 : b;
    const double scP = (l == 0) ? -kn1 : cP, scN = (l == 0) ? kn0 : cN;
    double uu, xx;
    // x_upper: g = (1e-9, -1) -> v = (-1e-9, 1), slot active_c_down, reachability_algorithm.py:229-233
    const bool ok_hi = lp2d_pair<true>(-1e-9, 1.0, sa, sb, scP, scN, rP, rN, nC, VAR_MIN, VAR_MAX, xlo, xhi, dn0, dn1, uu,
                                       xx, l, gmask, gbase);
    const double x_upper = ok_hi ? xx : nan_d;
    // x_lower: g = (-1e-9, 1) -> v = (1e-9, -1), slot active_c_up, :234-236
    bool ok_lo;
    double x_lower, ufeas;
    if (FAST && xlo <= xhi && lp1d_pair(1.0, xlo, sa, sb, scP, scN, VAR_MIN, VAR_MAX, ufeas, gmask)) {
      ok_lo = true;      // TB_SCAN_FAST_LOWER: some u is feasible at x = xlo, so min x IS xlo (not the reference's rounding noise)
      x_lower = xlo;
    } else {
      ok_lo = lp2d_pair<true>(1e-9, -1.0, sa, sb, scP, scN, rP, rN, nC, VAR_MIN, VAR_MAX, xlo, xhi, up0, up1, uu, xx, l,
                              gmask, gbase);
      x_lower = ok_lo ? xx : nan_d;
    }
    if (x_lower < 0) x_lower = 0;  // reachability_algorithm.py:190-191
    if (l == 0) { Kp[2 * i] = x_lower; Kp[2 * i + 1] = x_upper; }
    if (!(ok_hi && ok_lo)) {
      // :192-197: stop; the remaining K entries stay 0 (np.zeros)
      st = TB_STATUS_FAIL_UNCONTROLLABLE;
      fstage = i;
      for (int j = l; j < 2 * i; j += GL) Kp[j] = 0.0;
      break;
    }
    kn0 = x_lower;
    kn1 = x_upper;
  }
  __syncwarp(gmask);
  const double x_start = sds * sds;
  if (backward_only) {
    if (l == 0) {
      status[path] = st;
      if (fail_stage) fail_stage[path] = fstage;
    }
    return;
  }
  if (st == TB_STATUS_OK) {
    // kn0, kn1 == K[0]; admissibility check reachability_algorithm.py:290-301
    if (x_start + ALG_SMALL < kn0 || kn1 + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  if (st != TB_STATUS_OK) {
    for (int j = l; j < G; j += GL) sdp[j] = nan_d;
    for (int j = l; j < N; j += GL) up[j] = nan_d;
  } else {
    // ---------------- forward pass, reachability_algorithm.py:303-364; sd = sqrt(x) in one sweep afterwards ----------------
    double x = x_start;
    if (l == 0) sdp[0] = x;
    f_seg = 0;
    for (int i = 0; i < N; ++i) {
      const double g0 = gp[i], g1 = gp[i + 1];
      const double delta = g1 - g0;
      slab_ab(g0, g1, false, delta, a, b);
      const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
      const double sa = (l == 0) ? 2 * delta : a, sb = (l == 0) ? 1.0 : b;
      const double scP = (l == 0) ? -k1 : cP, scN = (l == 0) ? k0 : cN;
      int tries = 0;
      bool ok;
      double uopt = 0.0;
      while (true) {
        // _forward_step: g = (-2 delta, -1), x_min = x_max = x -> 1-variable branch, v0 = 2 delta (pyx:628-636)
        ok = lp1d_pair(-(-2 * delta), x, sa, sb, scP, scN, VAR_MIN, VAR_MAX, uopt, gmask);
        if (ok || tries >= MAX_TRIES) break;
        x = py_max(x - ALG_TINY, 0.999 * x);  // reachability_algorithm.py:324-327
        ++tries;
      }
      if (!ok) {
        // :337-342: xs[i+1:] = nan -> sd NaN -> ErrUnknown; us stay 0
        st = TB_STATUS_ERR_UNKNOWN;
        fstage = i;
        if (l == 0) sdp[i] = x;
        for (int j = i + 1 + l; j < G; j += GL) sdp[j] = nan_d;
        for (int j = i + l; j < N; j += GL) up[j] = 0.0;
        break;
      }
      double x_next = x + 2 * delta * uopt;                        // :352
      x_next = py_max(x_next - ALG_TINY, 0.9999 * x_next);         // :353
      x_next = py_min(k1, py_max(k0, x_next));                     // :354
      if (l == 0) {
        up[i] = uopt;
        if (tries) sdp[i] = x;  // x was shrunk by the retry rule
        sdp[i + 1] = x_next;
      }
      x = x_next;
    }
    __syncwarp(gmask);
    for (int j = l; j < G; j += GL) sdp[j] = sqrt(sdp[j]);  // reachability_algorithm.py:365
  }
  if (l == 0) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
  }
}

// ======================================================================================================================
// LOCKSTEP form.  redux.sync and vote.sync deliver ONE result per warp, so with half-warp masks every collective of the
// kernel above is executed once per half plus a convergence branch.  Here both half-warps run ONE instruction stream: reductions are xor-butterflies of full-mask
// shuffles (offsets 8, 4, 2, 1 stay inside a half), votes are one full-mask ballot from which each half reads its 16 bits,
// and what differs between the two paths — number of re-solves, shortcut taken or not, failure — is predication on
// per-half flags instead of branches.  Same arithmetic, same results.
// ======================================================================================================================
__device__ __forceinline__ double half_min(double v) {
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) {
    const double o = __shfl_xor_sync(FULL, v, off);
    v = (o < v) ? o : v;
  }
  return v;
}
__device__ __forceinline__ int half_min_int(int v) {
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) v = min(v, __shfl_xor_sync(FULL, v, off));
  return v;
}
__device__ __forceinline__ bool half_any(const bool pred, const int gbase) {
  return ((__ballot_sync(FULL, pred) >> gbase) & 0xffffu) != 0u;
}

// lp2d for both halves at once.  `en`: this half has a problem to solve.  Returns feasibility per half; outputs (ac0, ac1,
// out_u, out_x) are written only for a feasible, enabled half.
template <bool SKIP>
__device__ __forceinline__ bool lp2d_lock(const double v0, const double v1, const double a, const double b, const double cP,
                                          const double cN, const int rP, const int rN, const int nC, const double low0,
                                          const double high0, const double low1, const double high1, int &ac0, int &ac1,
                                          double &out_u, double &out_x, const int l, const int gbase, const bool en) {
  bool act = en && !(low0 > high0 || low1 > high1);  // pyx:233-235
  bool ok = act;
  const bool valid = ac0 >= 0 && ac0 < nC && ac1 >= 0 && ac1 < nC && ac0 != ac1;  // uniform over the half-warp
  double p0 = (v0 > LP_TINY) ? high0 : low0;       // pyx:236-247
  double p1 = (v1 > LP_TINY) ? high1 : low1;
  int nac0 = (v0 > LP_TINY) ? -2 : -1;
  int nac1 = (v1 > LP_TINY) ? -4 : -3;
  const int posP = (rP >= 0) ? row_pos(rP, valid, ac0, ac1) : INT_MAX;
  const int posN = (rN >= 0) ? row_pos(rN, valid, ac0, ac1) : INT_MAX;
  const unsigned lt_mask = (1u << l) - 1u;
  int kpos = -1;
  const bool skip_ok = SKIP && (((v0 > LP_TINY) && (v1 < 0)) || ((v0 < -LP_TINY) && (v1 > 0)));
  while (true) {
    int knew = INT_MAX;
    // ---- shortcut A (natural order), for the halves that are at their first visit without a valid warm-start pair
    const bool needA = SKIP && act && kpos < 0 && !valid && skip_ok;
    if (SKIP && __any_sync(FULL, needA)) {
      const double sg = (v0 > 0) ? 1.0 : -1.0;
      const double x = p1, u0m = sg * p0;
      const double sa = sg * a;
      const bool aup = sa > LP_TINY, adn = sa < -LP_TINY, any = aup || adn;
      const bool realP = posP != INT_MAX, realN = posN != INT_MAX;
      const bool uprP = realP && aup, uprN = realN && adn, lorP = realP && adn, lorN = realN && aup;
      const double bx = b * x;
      const double bxcP = bx + cP, bxcN = -bx + cN;
      const double den = any ? a : 1.0;
      const bool znP = (bxcP == 0.0), znN = (bxcN == 0.0);
      const double qdP = -opaque(znP ? 1.0 : bxcP) / den;
      const double qdN = opaque(znN ? 1.0 : bxcN) / den;
      const double uoP = znP ? 0.0 : sg * qdP, uoN = znN ? 0.0 : sg * qdN;
      const bool hasU = uprP || uprN;
      const double uoU = uprP ? uoP : uoN;
      const int posU = uprP ? posP : posN;
      const double v1dP = (-b) * v0 + a * v1;
      const double v1dU = uprP ? v1dP : -v1dP;
      bool bad = hasU && !((fabs(v1dU) < LP_TINY) || (v1dU < 0));
      const double aU = uprP ? a : -a, bU = uprP ? b : -b;
      bad = bad || (hasU && !(fabs(x * aU - (sg * uoU) * bU) < SKIP_TMAX * (aU * aU + bU * bU)));
      const double um = half_min(hasU ? uoU : SKIP_BIG);
      const int m = half_min_int((hasU && uoU == um) ? posU : INT_MAX);
      double second = half_min((hasU && posU != m) ? uoU : SKIP_BIG);
      second = (u0m < second) ? u0m : second;
      if (hasU && posU == m) {
        const double cU = uprP ? cP : cN, bxcU = uprP ? bxcP : bxcN;
        const double au = aU * (sg * second);
        const double val = au + bxcU;
        bad = bad || !(val >= SKIP_GAP * (1.0 + fabs(au) + fabs(bU * x) + fabs(cU)));
      }
      if (posP < m)
        bad = bad || (lorP && (uoP > um - 1e-9 * (1.0 + fabs(um)))) || (!uprP && !lorP && ((bxcP > -1e-9) || (a != 0.0)));
      if (posN < m)
        bad = bad || (lorN && (uoN > um - 1e-9 * (1.0 + fabs(um)))) || (!uprN && !lorN && ((bxcN > -1e-9) || (a != 0.0)));
      const double ur = sg * um;
      bad = bad || (ur < low0 + 1.0) || (ur > high0 - 1.0);
      const bool anybad = half_any(bad, gbase);
      if (needA && m != INT_MAX && !anybad) knew = m;
    }
    // ---- first row (in order) violated at the current point, pyx:269-275 (NaN counts as violated)
    const bool searched = (knew == INT_MAX);
    {
      const double s = a * p0 + b * p1;
      const double valP = s + cP, valN = -s + cN;
      const bool candP = !(valP < LP_TINY) && (posP > kpos) && (posP != INT_MAX);
      const bool candN = !(valN < LP_TINY) && (posN > kpos) && (posN != INT_MAX);
      const int found = half_min_int(min(candP ? posP : INT_MAX, candN ? posN : INT_MAX));
      if (searched) knew = found;
    }
    // ---- shortcut B (valid warm-start pair, row p = ac1 violated at the start vertex)
    const bool needB = SKIP && act && searched && kpos < 0 && valid && skip_ok && knew == 0;
    if (SKIP && __any_sync(FULL, needB)) {
      const bool mineN = (rN == ac1);
      const unsigned holder = (__ballot_sync(FULL, (rP == ac1) || mineN) >> gbase) & 0xffffu;
      const int src = gbase + __ffs(holder) - 1;
      const double ap = __shfl_sync(FULL, mineN ? -a : a, src);
      const double bp = __shfl_sync(FULL, mineN ? -b : b, src);
      const double cp = __shfl_sync(FULL, mineN ? cN : cP, src);
      bool okb = fabs(ap) > 1e-6;
      const double ia = 1.0 / (okb ? ap : 1.0);
      okb = okb && (low1 <= high1 - 1e-7 * (1.0 + fabs(low1) + fabs(high1)));
      const double slp = v1 - v0 * bp * ia;
      okb = okb && !(fabs(slp) < 1e-6);
      const double sx = (slp > 0) ? high1 : low1;
      const double su = -(bp * sx + cp) * ia;
      okb = okb && (su >= low0 + 1.0) && (su <= high0 - 1.0);
      okb = okb && (fabs(sx * ap - su * bp) < 1e9 * (ap * ap + bp * bp));
      const double t1P = a * su, t2P = b * sx;
      const double vP = t1P + t2P + cP, vN = -t1P + -t2P + cN;
      const double mag = fabs(t1P) + fabs(t2P);
      const bool kviol = ((posP == 1) && (vP >= SKIP_GAP * (1.0 + mag + fabs(cP)))) ||
                         ((posN == 1) && (vN >= SKIP_GAP * (1.0 + mag + fabs(cN))));
      const bool anyk = half_any(kviol, gbase);
      if (needB && anyk && okb) knew = 1;
    }
    if (act && knew == INT_MAX) act = false;           // no violated row left: this half holds its optimum
    if (!__any_sync(FULL, act)) break;
    // ---- projected re-solve on row `knew` (halves that are done run along; their results are discarded)
    const int kp = knew;
    const int krow = pos_row(kp, valid, ac0, ac1);
    const bool kN = (rN == krow);
    const unsigned holder = (__ballot_sync(FULL, (rP == krow) || kN) >> gbase) & 0xffffu;
    const int src = gbase + __ffs(holder) - 1;
    const double ak = __shfl_sync(FULL, kN ? -a : a, src);
    const double bk = __shfl_sync(FULL, kN ? -b : b, src);
    const double ck = __shfl_sync(FULL, kN ? cN : cP, src);
    const double nrm = ak * ak + bk * bk;
    const double zq = ((l & 1) ? (-bk * ck) : (-ak * ck)) / (act ? nrm : 1.0);
    const double z0 = __shfl_sync(FULL, zq, gbase);
    const double z1 = __shfl_sync(FULL, zq, gbase + 1);
    const double dt0 = -bk, dt1 = ak;
    const double v1d = dt0 * v0 + dt1 * v1;
    const bool partP = posP < kp, partN = posN < kp;
    const bool idle = !(partP || partN);
    const unsigned idleb = (__ballot_sync(FULL, idle) >> gbase) & 0xffffu;
    const int inl = min(__popc(idleb), 2);
    const int rank = __popc(idleb & lt_mask);
    const bool isbox = idle && rank < inl;
    double thi, tlo;
    int khi, klo;
    bool bad = false;
    {
      const bool bu = rank == 0;
      const double ba = isbox ? (bu ? 1.0 : 0.0) : a, bb = isbox ? (bu ? 0.0 : 1.0) : b;
      const double bcP = isbox ? (bu ? -high0 : -high1) : cP, bcN = isbox ? (bu ? low0 : low1) : cN;
      const int kP = isbox ? BOXBASE + (bu ? 1 : 3) : posP, kN2 = isbox ? BOXBASE + (bu ? 0 : 2) : posN;
      project_slab(isbox || partP, isbox || partN, ba, bb, bcP, bcN, kP, kN2, dt0, dt1, z0, z1, thi, tlo, khi, klo, bad);
    }
    double my_hi = thi, my_lo = tlo;
    double fhi = LP_INF, flo = -LP_INF;
    int fkhi = INT_MAX, fklo = INT_MAX;
    if (__any_sync(FULL, act && inl < 2)) {  // some half has fewer than two idle lanes: extra box item on its lanes 0..
      const int slab = inl + l;
      const bool bu = slab == 0, on = (inl < 2) && (slab < 2);
      project_slab(on, on, bu ? 1.0 : 0.0, bu ? 0.0 : 1.0, bu ? -high0 : -high1, bu ? low0 : low1,
                   BOXBASE + (bu ? 1 : 3), BOXBASE + (bu ? 0 : 2), dt0, dt1, z0, z1, fhi, flo, fkhi, fklo, bad);
      my_hi = (fhi < my_hi) ? fhi : my_hi;
      my_lo = (flo > my_lo) ? flo : my_lo;
    }
    const bool pick_min = (fabs(v1d) < LP_TINY) || (v1d < 0);
    const double red = half_min(pick_min ? -my_lo : my_hi);
    const double tstar = pick_min ? -red : red;
    const bool cross = pick_min ? (my_hi < tstar) : (my_lo > tstar);
    const bool infeas = half_any(bad || cross, gbase) || (tstar == (pick_min ? -LP_INF : LP_INF));  // pyx:376-383
    int mykey = ((pick_min ? tlo : thi) == tstar) ? (pick_min ? klo : khi) : INT_MAX;
    mykey = ((pick_min ? flo : fhi) == tstar) ? min(mykey, pick_min ? fklo : fkhi) : mykey;
    const int akey = half_min_int(mykey);
    if (act) {
      if (infeas) {
        ok = false;
        act = false;
      } else {
        kpos = kp;
        nac0 = krow;
        nac1 = (akey >= BOXBASE) ? (-1 - (akey - BOXBASE)) : pos_row(akey, valid, ac0, ac1);
        p0 = z0 + tstar * dt0;  // pyx:362-363
        p1 = z1 + tstar * dt1;
      }
    }
  }
  if (ok) {
    ac0 = nac0;
    ac1 = nac1;
    out_u = p0;
    out_x = p1;
  }
  return ok;
}

__device__ __forceinline__ bool lp1d_lock(const double v0, const double x, const double a, const double b, const double cP,
                                          const double cN, const double low0, const double high0, double &out_u,
                                          const int gbase) {
  const double bx = b * x;
  const double bxcP = bx + cP, bxcN = -bx + cN;
  const bool ap = a > LP_TINY, an = a < -LP_TINY;
  const double den = (ap || an) ? a : 1.0;
  const bool znP = (bxcP == 0.0), znN = (bxcN == 0.0);
  const double qP0 = -opaque(znP ? 1.0 : bxcP) / den;
  const double qN0 = opaque(znN ? 1.0 : bxcN) / den;
  const double tP = znP ? (-bxcP) * den : qP0;
  const double tN = znN ? (-bxcN) * (-den) : qN0;
  const double tu = ap ? tP : tN, tl = ap ? tN : tP;
  double my_hi = high0, my_lo = low0;
  my_hi = ((ap || an) && tu < my_hi) ? tu : my_hi;
  my_lo = ((ap || an) && tl > my_lo) ? tl : my_lo;
  const bool pick_min = (fabs(v0) < LP_TINY) || (v0 < 0);
  const double red = half_min(pick_min ? -my_lo : my_hi);
  const double ustar = pick_min ? -red : red;
  const bool infeas = half_any(pick_min ? (my_hi < ustar) : (my_lo > ustar), gbase);
  out_u = ustar;
  return !infeas;
}

template <bool FAST, int CFLAGS, int MINB>
__global__ void __launch_bounds__(32, MINB)
scan_lock_kernel(const VelAccSrc src, const int interp, const int Wc, const double *__restrict__ grid, const int grid_shared,
                 const int B, const int G, const double *__restrict__ sd_start, const double *__restrict__ sd_end,
                 const double *__restrict__ sd_end_hi, double *__restrict__ Kout, double *__restrict__ sdout,
                 double *__restrict__ uout, int *__restrict__ status, int *__restrict__ fail_stage) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = (int)threadIdx.x;
  const int grp = lane >> 4, l = lane & 15, gbase = grp * GL;
  const long path_raw = (long)blockIdx.x * 2 + grp;
  const bool en = path_raw < B;                     // an odd batch: the last half-warp runs along on the last path, muted
  const long path = en ? path_raw : (long)B - 1;
  constexpr bool backward_only = (CFLAGS & TB_SCAN_BACKWARD_ONLY) != 0;
  constexpr bool forward_only = (CFLAGS & TB_SCAN_FORWARD_ONLY) != 0;
  const int N = G - 1, nseg = src.nseg, dof = src.dof;
  const int nblk = interp ? 2 : 1;
  const int nC = 2 * nblk * dof + 2;
  double *bufs = reinterpret_cast<double *>(smem_raw) + (size_t)grp * Wc;
  const double *dco = bufs, *sx = bufs + nseg * dof * 6;
  {
    const double *cpp = src.ppoly + (size_t)path * 4 * nseg * dof;
    const double *xb = src.breaks + (src.breaks_shared ? 0 : (size_t)path * (nseg + 1));
    double *dco_w = bufs, *sx_w = bufs + nseg * dof * 6;
    for (int q = l; q < nseg * dof; q += GL) {
      const double c0 = cpp[q], c1 = cpp[nseg * dof + q], c2 = cpp[2 * nseg * dof + q];
      const double d0 = c0 * 3.0, d1 = c1 * 2.0, d2 = c2 * 1.0;
      double *o = dco_w + q * 6;
      o[0] = d0; o[1] = d1; o[2] = d2; o[3] = d0 * 2.0; o[4] = d1 * 1.0; o[5] = 0.0;
    }
    for (int q = l; q <= nseg; q += GL) sx_w[q] = xb[q];
  }
  const bool isj = (l >= 1) && (l - 1 < nblk * dof);
  const int f_second = isj ? (l - 1) / dof : 0;
  const int f_k = isj ? (l - 1) - f_second * dof : 0;
  const int rP = (l == 0) ? 1 : (isj ? 2 + 2 * f_second * dof + f_k : -1);
  const int rN = (l == 0) ? 0 : (isj ? rP + dof : -1);
  double cP = -1.0, cN = -1.0;
  if (isj) {
    const double *al = src.alim + (src.lim_shared ? 0 : (size_t)path * dof * 2);
    cP = 0.0 - al[f_k * 2 + 1];
    cN = 0.0 - (-al[f_k * 2 + 0]);
  }
  int f_seg = 0;
  __syncwarp();
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  const double *xbp = src.xbound + (size_t)path * G * 2;
  double *Kp = Kout + (size_t)path * G * 2;
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);
  auto slab_ab = [&](const double s0, const double s1, const bool down, const double delta, double &ra, double &rb) {
    const double s = f_second ? s1 : s0;
    if (down) { while (f_seg > 0 && s < sx[f_seg]) --f_seg; }
    else { while (f_seg < nseg - 1 && s >= sx[f_seg + 1]) ++f_seg; }
    const double ds = s - sx[f_seg];
    const double2 *o = reinterpret_cast<const double2 *>(dco + (f_seg * dof + f_k) * 6);
    const double2 o01 = o[0], o23 = o[1], o45 = o[2];
    double z = ds;
    double v1 = 0.0 + o23.x;
    v1 = v1 + o01.y * z;
    z = z * ds;
    v1 = v1 + o01.x * z;
    double v2 = 0.0 + o45.x;
    v2 = v2 + o23.y * ds;
    const double va = f_second ? (v1 + (2 * delta) * v2) : v1;
    ra = isj ? va : 0.0;
    rb = isj ? v2 : 0.0;
  };
  const bool lead = en && (l == 0);               // the lane that writes this path's scalars

  // ---------------- backward pass ----------------
  const double sde = sd_end ? sd_end[path] : 0.0;
  const double sds = sd_start ? sd_start[path] : 0.0;
  const double sdeh = sd_end_hi ? sd_end_hi[path] : sde;
  double kn0 = sde * sde, kn1 = sdeh * sdeh;
  if (lead && !forward_only) { Kp[2 * N] = kn0; Kp[2 * N + 1] = kn1; }
  int st = TB_STATUS_OK, fstage = -1;
  int up0 = 0, up1 = 0, dn0 = 0, dn1 = 0;
  if (forward_only) {
    st = status[path];
    fstage = fail_stage ? fail_stage[path] : -1;
    kn0 = Kp[0];
    kn1 = Kp[1];
  }
  double2 xb_ahead = make_double2(0.0, 0.0);
  f_seg = nseg - 1;
  if (!forward_only && N > 0) xb_ahead = reinterpret_cast<const double2 *>(xbp)[N - 1];
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  double a, b;
  bool alive = en;                                 // this half is still scanning
  for (int i = forward_only ? -1 : N - 1; i >= 0; --i) {
    if (!__any_sync(FULL, alive)) break;
    const double g0 = gp[i], g1 = gp[i + 1];
    const double delta = g1 - g0;
    slab_ab(g0, g1, true, delta, a, b);
    const double xlo = xb_ahead.x, xhi = xb_ahead.y;
    if (i > 0) xb_ahead = reinterpret_cast<const double2 *>(xbp)[i - 1];
    const double sa = (l == 0) ? 2 * delta : a, sb = (l == 0) ? 1.0 : b;
    const double scP = (l == 0) ? -kn1 : cP, scN = (l == 0) ? kn0 : cN;
    double uu = 0.0, xx = 0.0;
    const bool ok_hi = lp2d_lock<true>(-1e-9, 1.0, sa, sb, scP, scN, rP, rN, nC, VAR_MIN, VAR_MAX, xlo, xhi, dn0, dn1, uu,
                                       xx, l, gbase, alive);
    const double x_upper = ok_hi ? xx : nan_d;
    bool ok_lo;
    double x_lower, ufeas;
    bool fastok = false;
    if (FAST) fastok = (xlo <= xhi) && lp1d_lock(1.0, xlo, sa, sb, scP, scN, VAR_MIN, VAR_MAX, ufeas, gbase);
    {
      // TB_SCAN_FAST_LOWER: a half with some feasible u at x = xlo takes min x = xlo and sits the exact LP out
      const bool ok2 = lp2d_lock<true>(1e-9, -1.0, sa, sb, scP, scN, rP, rN, nC, VAR_MIN, VAR_MAX, xlo, xhi, up0, up1, uu,
                                       xx, l, gbase, alive && !fastok);
      ok_lo = fastok || ok2;
      x_lower = fastok ? xlo : (ok2 ? xx : nan_d);
    }
    if (x_lower < 0) x_lower = 0;
    if (alive && l == 0) { Kp[2 * i] = x_lower; Kp[2 * i + 1] = x_upper; }
    const bool failnow = alive && !(ok_hi && ok_lo);
    if (__any_sync(FULL, failnow)) {
      for (int j = l; j < 2 * i; j += GL)
        if (failnow) Kp[j] = 0.0;
    }
    if (failnow) {
      st = TB_STATUS_FAIL_UNCONTROLLABLE;
      fstage = i;
      alive = false;
    }
    if (alive) {
      kn0 = x_lower;
      kn1 = x_upper;
    }
  }
  __syncwarp();
  const double x_start = sds * sds;
  if (backward_only) {
    if (lead) {
      status[path] = st;
      if (fail_stage) fail_stage[path] = fstage;
    }
    return;
  }
  if (st == TB_STATUS_OK) {
    if (x_start + ALG_SMALL < kn0 || kn1 + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  alive = en && (st == TB_STATUS_OK);
  if (en && !alive) {
    for (int j = l; j < G; j += GL) sdp[j] = nan_d;
    for (int j = l; j < N; j += GL) up[j] = nan_d;
  }
  // ---------------- forward pass ----------------
  double x = x_start;
  if (alive && l == 0) sdp[0] = x;
  f_seg = 0;
  for (int i = 0; i < N; ++i) {
    if (!__any_sync(FULL, alive)) break;
    const double g0 = gp[i], g1 = gp[i + 1];
    const double delta = g1 - g0;
    slab_ab(g0, g1, false, delta, a, b);
    const double k0 = Kp[2 * (i + 1)], k1 = Kp[2 * (i + 1) + 1];
    const double sa = (l == 0) ? 2 * delta : a, sb = (l == 0) ? 1.0 : b;
    const double scP = (l == 0) ? -k1 : cP, scN = (l == 0) ? k0 : cN;
    int tries = 0;
    bool ok = false, pending = alive;
    double uopt = 0.0;
    while (true) {
      double ucand;
      const bool okc = lp1d_lock(-(-2 * delta), x, sa, sb, scP, scN, VAR_MIN, VAR_MAX, ucand, gbase);
      if (pending) {
        ok = okc;
        uopt = ucand;
        if (ok || tries >= MAX_TRIES) {
          pending = false;
        } else {
          x = py_max(x - ALG_TINY, 0.999 * x);  // reachability_algorithm.py:324-327
          ++tries;
        }
      }
      if (!__any_sync(FULL, pending)) break;
    }
    const bool failnow = alive && !ok;
    if (__any_sync(FULL, failnow)) {
      if (failnow && l == 0) sdp[i] = x;
      for (int j = i + 1 + l; j < G; j += GL)
        if (failnow) sdp[j] = nan_d;
      for (int j = i + l; j < N; j += GL)
        if (failnow) up[j] = 0.0;
    }
    if (failnow) {
      st = TB_STATUS_ERR_UNKNOWN;
      fstage = i;
      alive = false;
    }
    double x_next = x + 2 * delta * uopt;
    x_next = py_max(x_next - ALG_TINY, 0.9999 * x_next);
    x_next = py_min(k1, py_max(k0, x_next));
    if (alive && l == 0) {
      up[i] = uopt;
      if (tries) sdp[i] = x;
      sdp[i + 1] = x_next;
    }
    if (alive) x = x_next;
  }
  __syncwarp();
  // sd = sqrt(x) for the paths that ran the forward pass (to the end or until ErrUnknown: sqrt(NaN) = NaN)
  if (en && (st == TB_STATUS_OK || st == TB_STATUS_ERR_UNKNOWN))
    for (int j = l; j < G; j += GL) sdp[j] = sqrt(sdp[j]);
  if (lead) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
  }
}

#ifndef TB_SCAN_PAIR_MINB
#define TB_SCAN_PAIR_MINB 16  // resident warps per SM the register budget is sized for (128 registers)
#endif

template <bool FAST, int CFLAGS>
int launch_pair(const VelAccSrc &src, int interp, int Wc, const double *grid, int grid_shared, int B, int G,
                const double *sd_start, const double *sd_end, const double *sd_end_hi, double *K, double *sd, double *u,
                int *status, int *fail_stage, cudaStream_t stream) {
  const size_t smem = (size_t)2 * Wc * sizeof(double);
  const int blocks = (B + 1) / 2;
  static const char *env = getenv("TB_SCAN_PAIR");
  if (env && env[0] == '1')   // the divergent half-warp experiment (slower; kept for A/B)
    scan_pair_kernel<FAST, CFLAGS, TB_SCAN_PAIR_MINB><<<blocks, 32, smem, stream>>>(src, interp, Wc, grid, grid_shared, B, G,
                                                                                   sd_start, sd_end, sd_end_hi, K, sd, u,
                                                                                   status, fail_stage);
  else
    scan_lock_kernel<FAST, CFLAGS, TB_SCAN_PAIR_MINB><<<blocks, 32, smem, stream>>>(src, interp, Wc, grid, grid_shared, B, G,
                                                                                   sd_start, sd_end, sd_end_hi, K, sd, u,
                                                                                   status, fail_stage);
  return check_launch("tb_scan_velacc");
}

}  // namespace

bool scan_velacc_pair_supported(int dof, int interp, int nseg, int flags) {
  // Measured: both forms are slower than the one-warp-per-path kernel (file header); opt-in for A/B only.
  static const char *env = getenv("TB_SCAN_PAIR");   // 2: lockstep build, 1: divergent half-warp build, else off
  if (!(env && (env[0] == '1' || env[0] == '2'))) return false;
  const int mode = flags & ~TB_SCAN_FAST_LOWER;
  if (mode != 0 && mode != TB_SCAN_BACKWARD_ONLY && mode != TB_SCAN_FORWARD_ONLY) return false;  // TOPPRAsd rules etc.
  const int Wc = (nseg * dof * 6 + nseg + 1 + 1) & ~1;
  return (interp ? 2 : 1) * dof + 1 <= GL && (size_t)2 * Wc * 8 <= 40 * 1024;
}

int launch_scan_velacc_pair(const VelAccSrc &src, int interp, const double *grid, int grid_shared, int B, int G,
                            const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                            double *sd, double *u, int *status, int *fail_stage, cudaStream_t stream) {
  const int Wc = (src.nseg * src.dof * 6 + src.nseg + 1 + 1) & ~1;
  const bool fast = (flags & TB_SCAN_FAST_LOWER) != 0;
  const int mode = flags & ~TB_SCAN_FAST_LOWER;
#define TB_PAIR(FASTV, MODE) \
  return launch_pair<FASTV, MODE>(src, interp, Wc, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, K, sd, u, status, \
                                  fail_stage, stream)
  if (mode == 0) { if (fast) TB_PAIR(true, 0); TB_PAIR(false, 0); }
  if (mode == TB_SCAN_BACKWARD_ONLY) { if (fast) TB_PAIR(true, TB_SCAN_BACKWARD_ONLY); TB_PAIR(false, TB_SCAN_BACKWARD_ONLY); }
  if (mode == TB_SCAN_FORWARD_ONLY) { if (fast) TB_PAIR(true, TB_SCAN_FORWARD_ONLY); TB_PAIR(false, TB_SCAN_FORWARD_ONLY); }
#undef TB_PAIR
  set_error("tb_scan_velacc: scan mode %d not available in the two-paths-per-warp build", mode);
  return TB_ERR_UNSUPPORTED;
}

}  // namespace tb
