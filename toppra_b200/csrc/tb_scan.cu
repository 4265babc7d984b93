// tb_scan.cu — K2: backward controllable sets + forward parameterisation (TOPP-RA), one warp per path.
//
// Replaces (reference, hungpham2511/toppra v0.6.2):
//   ReachabilityAlgorithm.compute_controllable_sets / _one_step   reachability_algorithm.py:166-238
//   ReachabilityAlgorithm.compute_parameterization                reachability_algorithm.py:240-376
//   TOPPRA._forward_step                                          time_optimal_algorithm.py:55-92
//   seidelWrapper.solve_stagewise_optim                           cy_seidel_solverwrapper.pyx:549-697
//   cy_solve_lp2d / cy_solve_lp1d                                 cy_seidel_solverwrapper.pyx:149-390 / 93-144
//
// Design: the stages of one path are strictly sequential (K[i] <- K[i+1], x[i+1] <- x[i]), so the
// parallelism is (i) across paths: one warp per path, and (ii) across the LP rows of a stage: one row per lane
// (RPL rows per lane when nC > 32).  Seidel's incremental 2-variable LP keeps its exact row order (including
// the reference's warm-start permutation) so results are bit-identical to the Cython solver:
//   * "first violated row in order"      -> per-lane position + redux.sync min
//   * projection of earlier rows + box   -> one fp64 division per lane
//   * 1-D LP (min of upper / max of lower limits) -> redux.sync min / max on a two-word order-preserving key
// The per-stage record (3R+2 doubles) is streamed HBM -> shared memory with cp.async.bulk (TMA bulk copy,
// mbarrier complete_tx) into a ring of SCAN_NBUF = 4 buffers, three stages ahead of the solve.
// Compiled with -fmad=false: no FMA contraction, same roundings as the x86-64 reference.
#include <limits.h>

#include "tb_common.cuh"
#include "tb_scan_common.cuh"

namespace tb {
namespace {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// Arrive/copy/wait take 32-bit shared-window addresses (computed once per kernel): no generic->shared conversion and
// no 64-bit pointer arithmetic in the stage loops.
__device__ __forceinline__ void mbar_expect_tx_s(uint32_t bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s_s(uint32_t dst, const void *src, unsigned bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_wait_s(const uint32_t addr, unsigned parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        " .reg .pred p;\n"
        " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        " selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    if (!ok) __nanosleep(64);  // the copy is still in flight: do not burn issue slots other warps could use
  } while (!ok);
}

constexpr int SCAN_NBUF = 4;  // record buffers per warp (NBUF-1 stages of look-ahead)

// One projected constraint of the 1-D sub-problem (pyx:326-347): its limit on t as an upper bound `thi` (denom >
// TINY) or a lower bound `tlo` (denom < -TINY); +-LP_INF = no limit of that kind (the 1-D LP's own bounds);
// bad: parallel & infeasible.  The divisor of unused lanes is replaced by 1 so that the IEEE division never
// leaves its fast path for a value that is thrown away (x/0 would take the slow-path subroutine).
__device__ __forceinline__ void project_item(const bool part, const double aj, const double bj, const double cj,
                                             const double dt0, const double dt1, const double z0, const double z1,
                                             double &thi, double &tlo, bool &bad) {
  const double denom = dt0 * aj + dt1 * bj;
  const double num = cj + z1 * bj + z0 * aj;
  const bool up = part && (denom > LP_TINY), dn = part && (denom < -LP_TINY);
  const double t = -num / ((up || dn) ? denom : 1.0);
  // `cur_x < cur_max` / `cur_x > cur_min` (pyx:115-124): a limit at or beyond the sentinel, or NaN, never wins
  thi = (up && t < LP_INF) ? t : LP_INF;
  tlo = (dn && t > -LP_INF) ? t : -LP_INF;
  bad = bad || (part && !(up || dn) && (num > LP_SMALL));
}

// (aj, bj, cj) of box row m: 0: low0 <= u, 1: u <= high0, 2: low1 <= x, 3: x <= high1   (pyx:300-318)
__device__ __forceinline__ void box_row(const int m, const double low0, const double high0, const double low1,
                                        const double high1, double &aj, double &bj, double &cj) {
  aj = __hiloint2double((m == 0) ? (int)0xBFF00000 : ((m == 1) ? 0x3FF00000 : 0), 0);
  bj = __hiloint2double((m == 2) ? (int)0xBFF00000 : ((m == 3) ? 0x3FF00000 : 0), 0);
  cj = (m < 2) ? ((m == 0) ? low0 : -high0) : ((m == 2) ? low1 : -high1);
}

// cy_solve_lp2d (pyx:149-390) on one warp.  Lane `lane` holds LP rows r = lane + 32*s, s < RPL
// (padding rows must be (0, 0, -1)).  maximise v0*u + v1*x  s.t.  a u + b x + c <= 0, low <= (u,x) <= high.
// ac0/ac1: in = warm-start pair (active_c of the previous solve of this slot), out = new active pair
// (updated only when feasible, like pyx:673-676,690-691).  Returns false when infeasible.
//
// Per violated row k (one "re-solve"): the earlier rows and the four box rows are projected onto line k, one item
// per lane.  The box rows ride on lanes whose own row does not take part in this re-solve (rows at or after k,
// padding lanes); only if fewer than four such lanes exist they fall back to an extra item slot.
// PERM = a valid warm-start pair permutes the row order (pyx:252-264); PERM = false is the natural order, for which
// position == row index and the bookkeeping folds away (in the TOPP-RA backward pass: always for the min-x LP, whose
// optimum sits on the x box bound and invalidates the pair; the max-x LP usually has a valid pair).
// SKIP = the caller is the backward pass of the scan: the shortcuts A / B below may name the first row to re-solve on
// (bit-identical; a scalar model of the rules is checked by tests/test_shortcut_model.py); all else walks the rows in order.
template <int RPL, bool PERM, bool SKIP>
__device__ __forceinline__ bool lp2d_impl(const double v0, const double v1, const double (&a)[RPL],
                                          const double (&b)[RPL], const double (&c)[RPL], const int nC,
                                          const double low0, const double high0, const double low1,
                                          const double high1, int &ac0, int &ac1, double &out_u, double &out_x,
                                          const int lane, int &n_resolve) {
  double p0 = (v0 > LP_TINY) ? high0 : low0;       // pyx:236-247
  double p1 = (v1 > LP_TINY) ? high1 : low1;
  int nac0 = (v0 > LP_TINY) ? -2 : -1;
  int nac1 = (v1 > LP_TINY) ? -4 : -3;
  constexpr bool valid = PERM;
  int pos[RPL];
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    pos[s] = (r < nC) ? row_pos(r, valid, ac0, ac1) : INT_MAX;
  }
  const unsigned lt_mask = (1u << lane) - 1u;
  int kpos = -1;
  // shortcuts A/B below: only for the two objectives of the backward pass (min x, max x)
  const bool skip_ok = SKIP && (((v0 > LP_TINY) && (v1 < 0)) || ((v0 < -LP_TINY) && (v1 > 0)));
  while (true) {
    int knew = INT_MAX;
    if constexpr (SKIP && !PERM) {
      if (kpos < 0 && skip_ok) {
        // Shortcut A (natural order; DESIGN.md §4 K2).  Start vertex = (high0, low1) for the min-x LP, (low0,
        // high1) for the max-x LP.  In mirrored variables (ua = sg*u) every visit of the reference's walk sits on a
        // row that bounds ua from above, lands on x = its box bound and only lowers ua; each visit recomputes the
        // point from scratch over ALL earlier rows, so the final state depends only on the LAST visited row, and
        // that is the row m with the smallest own bound at this x.  The reference is certain to visit m when the
        // smallest bound among the OTHER rows (and the start value) violates row m far above the TINY threshold;
        // one exact re-solve on m then reproduces the reference's state bit for bit, and the exact walk goes on
        // from there.  Rows before m that bound ua from below (or not at all) must hold at the final point with
        // a margin, and every upper row must pick the low end of its line (the exact path's v1d test).  Any doubt
        // -> ordinary walk.  A scalar model of these rules is checked by tests/test_shortcut_model.py.
        const double sg = (v0 > 0) ? 1.0 : -1.0;
        const double x = p1, u0m = sg * p0;
        double uo[RPL], bxc[RPL];
        bool upr[RPL], lor[RPL];
        double lmin = SKIP_BIG;
        bool bad = false;
#pragma unroll
        for (int s = 0; s < RPL; ++s) {
          const bool real = pos[s] != INT_MAX;
          const double sa = sg * a[s];
          bxc[s] = b[s] * x + c[s];
          upr[s] = real && (sa > LP_TINY);
          lor[s] = real && (sa < -LP_TINY);
          // a zero numerator (row 0 at x = 0 with K_lo = 0: every stage) would send the IEEE division through its
          // slow-path subroutine; this value only feeds the margin tests, so 0 is substituted directly
          const bool zn = (bxc[s] == 0.0);
          const double qd = -opaque(zn ? 1.0 : bxc[s]) / ((upr[s] || lor[s]) ? a[s] : 1.0);
          uo[s] = zn ? 0.0 : sg * qd;
          const double v1d_own = (-b[s]) * v0 + a[s] * v1;  // the exact path's v1d if this row were visited
          bad = bad || (upr[s] && !((fabs(v1d_own) < LP_TINY) || (v1d_own < 0)));
          // line parameter t of this row's landing point (own bound, x): a skipped visit must neither end on the
          // +-1e10 sentinel of the 1-D LP nor be far enough from the foot point for a "parallel" row (|denom| <=
          // TINY although the lines cross) to fail the LP_SMALL test there: |t| * TINY stays far below LP_SMALL
          bad = bad || (upr[s] && !(fabs(x * a[s] - (sg * uo[s]) * b[s]) < SKIP_TMAX * (a[s] * a[s] + b[s] * b[s])));
          lmin = (upr[s] && uo[s] < lmin) ? uo[s] : lmin;
        }
        const double um = warp_min(lmin);
        int mp = INT_MAX;
#pragma unroll
        for (int s = 0; s < RPL; ++s) mp = (upr[s] && uo[s] == um) ? min(mp, pos[s]) : mp;
        const int m = __reduce_min_sync(FULL, mp);
        if (m != INT_MAX) {
          double l2 = SKIP_BIG;
#pragma unroll
          for (int s = 0; s < RPL; ++s) l2 = (upr[s] && pos[s] != m && uo[s] < l2) ? uo[s] : l2;
          double second = warp_min(l2);
          second = (u0m < second) ? u0m : second;
#pragma unroll
          for (int s = 0; s < RPL; ++s) {
            if (pos[s] == m) {
              const double au = a[s] * (sg * second);
              const double val = au + bxc[s];
              bad = bad || !(val >= SKIP_GAP * (1.0 + fabs(au) + fabs(b[s] * x) + fabs(c[s])));
            } else if (pos[s] < m) {
              bad = bad || (lor[s] && (uo[s] > um - 1e-9 * (1.0 + fabs(um)))) ||
                    (!upr[s] && !lor[s] && ((bxc[s] > -1e-9) || (a[s] != 0.0)));
            }
          }
          const double ur = sg * um;
          bad = bad || (ur < low0 + 1.0) || (ur > high0 - 1.0);
          if (!__any_sync(FULL, bad)) knew = m;
          if (knew == m && v0 > 0.0) {
            // Closure (min-x LP; DESIGN.md §4 K2).  The re-solve on m ends on the x-box item x >= low1 unless another
            // item binds: compute that outcome with the re-solve's own arithmetic (z, then t of box row (0, -1, low1)
            // as project_item forms it) and take it if every other row, the u box and x <= high1 hold at the closed
            // point q with a relative margin.  Then every earlier row's item lies strictly on the far side of t (no
            // tie, cross or parallel-infeasible item, |t| * TINY < SMALL), and the search after the re-solve finds no
            // violated row.  The closure is the one re-solve it replaces.  Scalar model: tests/closure_model.c.
            double am = a[0], bm = b[0], cm = c[0];
#pragma unroll
            for (int s = 1; s < RPL; ++s)
              if ((m >> 5) == s) { am = a[s]; bm = b[s]; cm = c[s]; }
            am = __shfl_sync(FULL, am, m & 31);
            bm = __shfl_sync(FULL, bm, m & 31);
            cm = __shfl_sync(FULL, cm, m & 31);
            const double nrm = am * am + bm * bm;
            const double zq = ((lane & 1) ? (-bm * cm) : (-am * cm)) / nrm;
            const double z0 = __shfl_sync(FULL, zq, 0);
            const double z1 = __shfl_sync(FULL, zq, 1);
            const double dt0 = -bm, dt1 = am;
            const double num = low1 + z1 * -1.0 + z0 * 0.0;
            const double den = dt0 * 0.0 + dt1 * -1.0;
            const double t = -num / den;
            const double q0 = z0 + t * dt0, q1 = z1 + t * dt1;
            const double qs = fabs(q0) + fabs(q1);
            bool miss = !(fabs(t) < SKIP_TMAX);
#pragma unroll
            for (int s = 0; s < RPL; ++s) {
              const double val = a[s] * q0 + b[s] * q1 + c[s];
              miss = miss || ((pos[s] != INT_MAX) && (pos[s] != m) &&
                              !(val <= -SKIP_GAP * (1.0 + fabs(c[s]) + (fabs(a[s]) + fabs(b[s])) * qs)));
            }
            {  // box rows u >= low0, u <= high0, x <= high1 on lanes 0..2
              double ba, bb, bc;
              box_row((lane == 2) ? 3 : lane, low0, high0, low1, high1, ba, bb, bc);
              const double val = ba * q0 + bb * q1 + bc;
              miss = miss || ((lane < 3) && !(val <= -SKIP_GAP * (1.0 + fabs(bc) + (fabs(ba) + fabs(bb)) * qs)));
            }
            if (!__any_sync(FULL, miss)) {
              ++n_resolve;
              ac0 = m;
              ac1 = -3;
              out_u = q0;
              out_x = q1;
              return true;
            }
          }
        }
      }
    }
    if (knew == INT_MAX) {
      // first row (in order) violated at the current point, pyx:269-275.  NaN counts as violated (not `< TINY`).
      int mypos = INT_MAX;
#pragma unroll
      for (int s = 0; s < RPL; ++s) {
        const double val = a[s] * p0 + b[s] * p1 + c[s];
        const bool cand = !(val < LP_TINY) && (pos[s] > kpos) && (pos[s] != INT_MAX);
        mypos = cand ? min(mypos, pos[s]) : mypos;
      }
      knew = __reduce_min_sync(FULL, mypos);
      if (knew == INT_MAX) break;
      if constexpr (SKIP && PERM) {
        if (kpos < 0 && skip_ok && knew == 0) {
          // Shortcut B (valid warm-start pair; order = row p = ac1, row k = ac0, the rest).  Row p is violated at
          // the start vertex, so the reference re-solves on it against the box only and holds the optimum of line p
          // inside the box next.  That point is cheap to compute with plain arithmetic; if row k is violated there
          // far above the TINY threshold the reference is certain to re-solve on position 1 next, and that re-solve
          // (row p + the box, recomputed from scratch) does not depend on the skipped one.
          const int lp = ac1 & 31;
          double ap = a[0], bp = b[0], cp = c[0];
#pragma unroll
          for (int s = 1; s < RPL; ++s)
            if ((ac1 >> 5) == s) { ap = a[s]; bp = b[s]; cp = c[s]; }
          ap = __shfl_sync(FULL, ap, lp);
          bp = __shfl_sync(FULL, bp, lp);
          cp = __shfl_sync(FULL, cp, lp);
          bool okb = fabs(ap) > 1e-6;
          const double ia = 1.0 / (okb ? ap : 1.0);
          okb = okb && (low1 <= high1 - 1e-7 * (1.0 + fabs(low1) + fabs(high1)));
          const double slp = v1 - v0 * bp * ia;  // d objective / dx along line p
          okb = okb && !(fabs(slp) < 1e-6);
          // optimum of line p inside the box: the x bound the objective points to, provided u stays well inside its
          // own bounds there (otherwise the u bounds clip the line first: left to the exact path)
          const double sx = (slp > 0) ? high1 : low1;
          const double su = -(bp * sx + cp) * ia;
          okb = okb && (su >= low0 + 1.0) && (su <= high0 - 1.0);
          // the skipped 1-D optimum must stay clear of the +-1e10 sentinel (pyx:376-383 would report infeasible)
          okb = okb && (fabs(sx * ap - su * bp) < 1e9 * (ap * ap + bp * bp));
          bool kviol = false;
#pragma unroll
          for (int s = 0; s < RPL; ++s) {
            const double t1 = a[s] * su, t2 = b[s] * sx;
            const double val = t1 + t2 + c[s];
            kviol = kviol || ((pos[s] == 1) && (val >= SKIP_GAP * (1.0 + fabs(t1) + fabs(t2) + fabs(c[s]))));
          }
          if (__any_sync(FULL, kviol) && okb) knew = 1;
        }
      }
    }
    kpos = knew;
    const int krow = pos_row(kpos, valid, ac0, ac1);
    ++n_resolve;
    nac0 = krow;
    // broadcast row k
    double ak = a[0], bk = b[0], ck = c[0];
#pragma unroll
    for (int s = 1; s < RPL; ++s)
      if ((krow >> 5) == s) { ak = a[s]; bk = b[s]; ck = c[s]; }
    ak = __shfl_sync(FULL, ak, krow & 31);
    bk = __shfl_sync(FULL, bk, krow & 31);
    ck = __shfl_sync(FULL, ck, krow & 31);
    // project the origin onto line k, pyx:290-295: z = (-a c, -b c) / (a^2 + b^2).  One division sequence for
    // both components: odd lanes divide the second numerator.
    const double nrm = ak * ak + bk * bk;
    const double zq = ((lane & 1) ? (-bk * ck) : (-ak * ck)) / nrm;
    const double z0 = __shfl_sync(FULL, zq, 0);
    const double z1 = __shfl_sync(FULL, zq, 1);
    const double dt0 = -bk, dt1 = ak;
    const double v1d = dt0 * v0 + dt1 * v1;
    // project the earlier rows and the four box rows onto the line, pyx:298-347
    double thi[RPL], tlo[RPL];
    int key[RPL];
    bool bad = false;
    const bool idle0 = !(pos[0] < kpos);  // this lane's slot-0 row does not take part (row k, later rows, padding)
    const unsigned idle = __ballot_sync(FULL, idle0);
    const bool box_inline = __popc(idle) >= 4;  // warp-uniform
    {
      // slot 0: own row, or (on the first four idle lanes) box row m = rank
      const int m = __popc(idle & lt_mask);
      const bool isbox = box_inline && idle0 && m < 4;
      double ba, bb, bc;
      box_row(m, low0, high0, low1, high1, ba, bb, bc);
      key[0] = isbox ? BOXBASE + m : pos[0];
      project_item(isbox || !idle0, isbox ? ba : a[0], isbox ? bb : b[0], isbox ? bc : c[0], dt0, dt1, z0, z1, thi[0],
                   tlo[0], bad);
    }
#pragma unroll
    for (int s = 1; s < RPL; ++s) {
      key[s] = pos[s];
      project_item(pos[s] < kpos, a[s], b[s], c[s], dt0, dt1, z0, z1, thi[s], tlo[s], bad);
    }
    // 1-D LP on the line with bounds +-INF, pyx:350 -> cy_solve_lp1d pyx:93-144
    double my_hi = thi[0], my_lo = tlo[0];
#pragma unroll
    for (int s = 1; s < RPL; ++s) {
      my_hi = (thi[s] < my_hi) ? thi[s] : my_hi;
      my_lo = (tlo[s] > my_lo) ? tlo[s] : my_lo;
    }
    double xhi_t = LP_INF, xlo_t = -LP_INF;  // extra item slot, only when the box rows could not ride inline
    if (!box_inline) {  // rare: (almost) every row takes part -> box rows on lanes 0..3
      double ba, bb, bc;
      box_row(lane, low0, high0, low1, high1, ba, bb, bc);
      project_item(lane < 4, ba, bb, bc, dt0, dt1, z0, z1, xhi_t, xlo_t, bad);
      my_hi = (xhi_t < my_hi) ? xhi_t : my_hi;
      my_lo = (xlo_t > my_lo) ? xlo_t : my_lo;
    }
    // The objective's sign decides which end of [cur_min, cur_max] is the optimum (pyx:130-143); only that end is
    // reduced exactly (max lo = -min(-lo)); "cur_min > cur_max" (pyx:126-128) is a vote against the other side.
    const bool pick_min = (fabs(v1d) < LP_TINY) || (v1d < 0);
    const double red = warp_min(pick_min ? -my_lo : my_hi);
    const double tstar = pick_min ? -red : red;
    const bool cross = pick_min ? (my_hi < tstar) : (my_lo > tstar);
    if (__any_sync(FULL, bad || cross)) return false;
    // optimum on the +-INF sentinel (1-D active index -1/-2) counts as infeasible, pyx:376-383
    if (tstar == (pick_min ? -LP_INF : LP_INF)) return false;
    // active item = first (lowest key) item that attains the optimum; tstar is finite here, sentinels never match
    int mykey = INT_MAX;
#pragma unroll
    for (int s = 0; s < RPL; ++s) mykey = ((pick_min ? tlo[s] : thi[s]) == tstar) ? min(mykey, key[s]) : mykey;
    if (!box_inline) mykey = ((pick_min ? xlo_t : xhi_t) == tstar) ? min(mykey, BOXBASE + lane) : mykey;
    const int akey = __reduce_min_sync(FULL, mykey);
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

template <int RPL, bool SKIP = false>
__device__ __forceinline__ bool lp2d_warp(const double v0, const double v1, const double (&a)[RPL],
                                          const double (&b)[RPL], const double (&c)[RPL], const int nC,
                                          const double low0, const double high0, const double low1,
                                          const double high1, int &ac0, int &ac1, double &out_u, double &out_x,
                                          const int lane, int &n_resolve) {
  if (low0 > high0 || low1 > high1) return false;  // pyx:233-235
  const bool valid = ac0 >= 0 && ac0 < nC && ac1 >= 0 && ac1 < nC && ac0 != ac1;  // warp-uniform
  if (valid)
    return lp2d_impl<RPL, true, SKIP>(v0, v1, a, b, c, nC, low0, high0, low1, high1, ac0, ac1, out_u, out_x, lane,
                                       n_resolve);
  return lp2d_impl<RPL, false, SKIP>(v0, v1, a, b, c, nC, low0, high0, low1, high1, ac0, ac1, out_u, out_x, lane,
                                     n_resolve);
}

// cy_solve_lp1d (pyx:93-144) as used by the x_min == x_max branch of solve_stagewise_optim (pyx:631-650):
// rows a*u + (b*x + c) <= 0 over ALL nC rows, u in [low0, high0]; objective v0*u.  Returns false if infeasible.
template <int RPL>
__device__ __forceinline__ bool lp1d_fixed_x_warp(const double v0, const double x, const double (&a)[RPL],
                                                  const double (&b)[RPL], const double (&c)[RPL],
                                                  const double low0, const double high0, double &out_u) {
  double my_hi = high0, my_lo = low0;
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const double bxc = b[s] * x + c[s];
    const bool up = a[s] > LP_TINY, dn = a[s] < -LP_TINY;
    // unused lanes divide by 1 and a zero numerator (row 0 at x = 0 with K_lo = 0) is not divided at all: both would
    // leave the IEEE division's fast path.  (-bxc) * a is the quotient's correctly signed zero.
    const double den = (up || dn) ? a[s] : 1.0;
    const bool zn = (bxc == 0.0);
    const double q = -opaque(zn ? 1.0 : bxc) / den;
    const double t = zn ? (-bxc) * den : q;
    my_hi = (up && t < my_hi) ? t : my_hi;
    my_lo = (dn && t > my_lo) ? t : my_lo;
  }
  // exact reduction of the optimal end only; infeasibility (cur_min > cur_max) as a vote against the other side
  const bool pick_min = (fabs(v0) < LP_TINY) || (v0 < 0);
  const double red = warp_min(pick_min ? -my_lo : my_hi);
  const double ustar = pick_min ? -red : red;
  if (__any_sync(FULL, pick_min ? (my_hi < ustar) : (my_lo > ustar))) return false;
  out_u = ustar;
  return true;
}

// The rows lp1d_fixed_x_warp skips (|a| <= LP_TINY, as cy_solve_lp1d does) hold at (u, x).  The fast min-x shortcut
// needs this: the 2-D LP it stands in for keeps those rows, and a flat row such as x >= 0.5 or x <= -1 moves or
// removes the optimum at x = xlo although the 1-D LP there is feasible.
template <int RPL>
__device__ __forceinline__ bool flat_rows_hold(const double u, const double x, const double (&a)[RPL],
                                               const double (&b)[RPL], const double (&c)[RPL]) {
  bool bad = false;
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const bool flat = !(a[s] > LP_TINY) && !(a[s] < -LP_TINY);
    bad |= flat && (a[s] * u + (b[s] * x + c[s]) > 0.0);
  }
  return !__any_sync(FULL, bad);
}

// Load this lane's rows of one stage record (shared memory) into registers.  LP row r: r = 0,1 are the
// x_next rows (filled by the caller), r >= 2 is static row r-2; padding rows are (0,0,-1).
template <int RPL>
__device__ __forceinline__ void load_rows(const double *rec, const int R, const int nC, const int lane,
                                          double (&a)[RPL], double (&b)[RPL], double (&c)[RPL]) {
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    const bool in = (r >= 2) && (r < nC);
    const int j = in ? r - 2 : 0;  // always a valid slot of the record: load, then select
    const double va = rec[j], vb = rec[R + j], vc = rec[2 * R + j];
    a[s] = in ? va : 0.0;
    b[s] = in ? vb : 0.0;
    c[s] = in ? vc : -1.0;
  }
}

template <int RPL>
__device__ __forceinline__ void set_xnext_rows(const int lane, const double delta, const double xn_min,
                                               const double xn_max, double (&a)[RPL], double (&b)[RPL],
                                               double (&c)[RPL]) {
  // pyx:604-620: row0 = (-2 delta, -1, x_next_min), row1 = (2 delta, 1, -x_next_max); selects, no branches
  const bool xr = lane < 2, first = lane == 0;
  const double sgn = first ? -1.0 : 1.0;
  a[0] = xr ? sgn * (2 * delta) : a[0];  // -(2 delta) == -2 * delta bit for bit
  b[0] = xr ? sgn : b[0];
  c[0] = xr ? (first ? xn_min : -xn_max) : c[0];
}

// CFLAGS >= 0: the scan-mode bits of `flags` (backward-only, forward-only, TOPPRAsd rules) are this compile-time
// constant (the argument is ignored), so the unused passes and rules and their bookkeeping fold away; -1: run time.
// Row source of the FUSED scan (tb_scan_velacc): JointVelocity + JointAcceleration problems need no stage records at
// all — lane r builds its own LP row from the path's spline in the stage prologue, with the arithmetic of K1
// (tb_coeff.cu: PPoly derivative evaluation like scipy, interpolation lift a+ = q'(s_{i+1}) + 2 delta q''(s_{i+1}),
// c = -amax / +amin), so the rows are bit-identical to the materialised records; only the velocity bound
// (xbound [B][G][2], 16 B per gridpoint instead of 8 (3R+2)) still comes from memory.
// UB: the stage records carry a u-bound pair (ulo, uhi) behind the x-bound pair (TB_SCAN_UBOUND: `ubound` of a
// constraint, intersected into low/high[:, 0] by seidelWrapper.__init__, pyx:512-515); otherwise u in [-1e8, 1e8].
// glen (optional): ragged batches, path p has glen[p] <= G gridpoints (strides stay G; outputs past glen[p] are NaN).
// One warp per CTA (block = path): a finished path frees its slot at once (measured best: 1 < 2 < 4 warps per CTA).
// MINB = resident one-warp CTAs per SM the register budget is sized for.
template <int RPL, int MINB, bool FAST, int CFLAGS = -1, bool FUSED = false, bool UB = false>
__global__ void __launch_bounds__(32, MINB)
scan_kernel(const double *__restrict__ records, const int W, const int R, const double *__restrict__ grid,
            const int grid_shared, const int B, const int G, const double *__restrict__ sd_start,
            const double *__restrict__ sd_end, const double *__restrict__ sd_end_hi, const int flags_arg,
            double *__restrict__ Kout, double *__restrict__ sdout, double *__restrict__ uout,
            int *__restrict__ status, int *__restrict__ fail_stage, int *__restrict__ counters,
            const int *__restrict__ glen, const VelAccSrc src) {
  static_assert(!FUSED || RPL == 1, "the fused row source holds one row per lane");
  static_assert(!(FUSED && UB), "velocity + acceleration problems have no u-bound");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // the lane is read once and kept: the optimiser otherwise re-reads the special register (S2R, ~20 cycles) at every use
  // when it runs short of registers
  int lane;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(lane));
  const long path = blockIdx.x;
  if (path >= B) return;
  // shared-memory plan.  records: ring of SCAN_NBUF stage records + mbarriers; FUSED: derivative coefficients
  // of the path's PPoly dco [nseg][dof][5] + breakpoints [nseg+1] (in W doubles; W = that size rounded up to even)
  double *bufs = reinterpret_cast<double *>(smem_raw);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)(FUSED ? 1 : SCAN_NBUF) * W * sizeof(double));
  // ragged batches run on the run-time-flag build (CFLAGS < 0); the specialised builds keep G as the loop bound
  const int Gp = (CFLAGS < 0 && glen) ? min(max(glen[path], 1), G) : G;  // this path's gridpoints
  const int N = Gp - 1, nC = R + 2;
  const unsigned rec_bytes = (unsigned)(W * sizeof(double));
  // Per-path base pointers live in shared memory: under the 64-register cap the compiler otherwise rebuilds them
  // from blockIdx and the kernel parameters (a chain of 64-bit multiplies) at every use inside the stage loops.
  const void *volatile *sptr = reinterpret_cast<const void *volatile *>(
      smem_raw + (size_t)(FUSED ? 1 : SCAN_NBUF) * W * sizeof(double) + SCAN_NBUF * sizeof(uint64_t));
  if (lane == 0) {
    sptr[0] = FUSED ? static_cast<const void *>(src.xbound + (size_t)path * G * 2)
                    : static_cast<const void *>(records + (size_t)path * G * W);
    sptr[1] = grid + (grid_shared ? 0 : (size_t)path * G);
    sptr[2] = Kout + (size_t)path * G * 2;
  }
  // FUSED: this lane's row.  LP row r = lane: r - 2 = blk * dof + k; blk & 1: the negated copy (F = [I; -I]);
  // blk >> 1: the lifted block evaluated at s_{i+1} (canlinear_colloc_to_interpolate, linear_constraint.py:84-192)
  const double *dco = bufs, *sx = bufs + (FUSED ? src.nseg * src.dof * 6 : 0);
  bool f_isrow = false, f_neg = false;
  int f_second = 0, f_k = 0, f_seg = 0;
  double f_c = -1.0;
  if constexpr (FUSED) {
    const int nseg = src.nseg, dof = src.dof;
    const double *cpp = src.ppoly + (size_t)path * 4 * nseg * dof;
    const double *xb = src.breaks + (src.breaks_shared ? 0 : (size_t)path * (nseg + 1));
    double *dco_w = bufs, *sx_w = bufs + nseg * dof * 6;
    for (int q = lane; q < nseg * dof; q += 32) {
      // scipy PPoly.derivative: c'[j] = c[j] * (k - j); cspldd = cspld.derivative() (interpolator.py:419-421)
      const double c0 = cpp[q], c1 = cpp[nseg * dof + q], c2 = cpp[2 * nseg * dof + q];
      const double d0 = c0 * 3.0, d1 = c1 * 2.0, d2 = c2 * 1.0;
      double *o = dco_w + q * 6;  // 48-byte entries: three 16-byte shared loads per evaluation
      o[0] = d0; o[1] = d1; o[2] = d2; o[3] = d0 * 2.0; o[4] = d1 * 1.0; o[5] = 0.0;
    }
    for (int q = lane; q <= nseg; q += 32) sx_w[q] = xb[q];
    const int rr = lane - 2;
    f_isrow = (lane >= 2) && (lane < nC);
    const int blk = f_isrow ? rr / dof : 0;
    f_k = f_isrow ? rr - blk * dof : 0;
    f_neg = (blk & 1) != 0;
    f_second = blk >> 1;
    const double *al = src.alim + (src.lim_shared ? 0 : (size_t)path * dof * 2);
    // F.c - g with c = 0, g = [amax; -amin] (tb_coeff.cu phase 1b)
    f_c = f_isrow ? (f_neg ? (0.0 - (-al[f_k * 2 + 0])) : (0.0 - al[f_k * 2 + 1])) : -1.0;
  }
  __syncwarp();
  auto rec_path = [&]() { return static_cast<const double *>(sptr[0]); };
  auto gp = [&]() { return static_cast<const double *>(sptr[1]); };
  auto Kp = [&]() { return static_cast<double *>(const_cast<void *>(sptr[2])); };
  const int flags = (CFLAGS >= 0) ? CFLAGS : flags_arg;
  const bool backward_only = (flags & 1) != 0;  // compute_controllable_sets(sdmin, sdmax) alone
  const bool forward_only = (flags & 16) != 0;  // K and status come from an earlier TB_SCAN_BACKWARD_ONLY launch
  constexpr bool fast_lower = FAST;             // opt-in shortcut for the min-x LP (TB_SCAN_FAST_LOWER, not bit-identical)
  const bool sd_mode = (flags & 4) != 0;        // TOPPRAsd forward-pass rules (no retry, x_next - 1e-5 clip)
  const bool sd_slow = (flags & 8) != 0;        // TOPPRAsd slowest pass: minimise the next velocity
  double *sdp = backward_only ? nullptr : sdout + (size_t)path * G;
  double *up = backward_only ? nullptr : uout + (size_t)path * (G > 1 ? G - 1 : 0);

  if (!FUSED && lane == 0) {
#pragma unroll
    for (int q = 0; q < SCAN_NBUF; ++q) mbar_init(&bars[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();

  // Ring of SCAN_NBUF record buffers: up to SCAN_NBUF-1 bulk copies in flight per warp.  The forward pass solves a
  // stage in well under the HBM round trip, so one stage of look-ahead is not enough there.
  unsigned n_issued = 0, n_waited = 0;
  const uint32_t bufs_s = smem_u32(bufs), bars_s = smem_u32(bars);
  auto issue = [&](int stage) {
    if (!FUSED && lane == 0) {
      const unsigned q = n_issued % SCAN_NBUF;
      mbar_expect_tx_s(bars_s + q * 8u, rec_bytes);
      bulk_g2s_s(bufs_s + q * rec_bytes, rec_path() + (size_t)stage * W, rec_bytes, bars_s + q * 8u);
    }
    ++n_issued;
  };
  auto acquire = [&]() -> const double * {
    const unsigned q = n_waited % SCAN_NBUF;
    if (!FUSED) mbar_wait_s(bars_s + q * 8u, (n_waited / SCAN_NBUF) & 1);
    ++n_waited;
    return bufs + (size_t)q * W;
  };
  constexpr int AHEAD = SCAN_NBUF - 1;
  // FUSED: this lane's row of stage i = K1's arithmetic (tb_coeff.cu phases 1, 1b) at the lane's own gridpoint
  // `s0`, `s1` = gridpoints i, i+1 (already loaded for delta).  The segment index of scipy's find_interval —
  // max{j <= nseg-1 : x[j] <= s}, 0 below the first breakpoint — is monotone in s, so it is carried from stage to
  // stage (DOWN in the backward pass, up in the forward pass) instead of searched: one comparison per stage.  A NaN
  // gridpoint leaves the index alone and poisons ds, so the row is NaN like K1's.
  auto fused_row = [&](const double s0, const double s1, const bool down, const double delta, double &ra, double &rb,
                       double &rc) {
    const double s = f_second ? s1 : s0;
    if (down) { while (f_seg > 0 && s < sx[f_seg]) --f_seg; }
    else { while (f_seg < src.nseg - 1 && s >= sx[f_seg + 1]) ++f_seg; }
    // scipy evaluate_poly1: res = 0; z = 1; for each power: res += c * z; z *= ds
    const double ds = s - sx[f_seg];
    const double2 *o = reinterpret_cast<const double2 *>(dco + (f_seg * src.dof + f_k) * 6);
    const double2 o01 = o[0], o23 = o[1], o45 = o[2];
    double z = ds;
    double v1 = 0.0 + o23.x;
    v1 = v1 + o01.y * z;
    z = z * ds;
    v1 = v1 + o01.x * z;
    double v2 = 0.0 + o45.x;
    v2 = v2 + o23.y * ds;
    const double va = f_second ? (v1 + (2 * delta) * v2) : v1;  // lift, linear_constraint.py:170
    ra = f_isrow ? (f_neg ? -va : va) : 0.0;
    rb = f_isrow ? (f_neg ? -v2 : v2) : 0.0;
    rc = f_c;
  };

  // instrumentation: projected re-solves, retries, fast-mode stages; the LP counts are derived from the stage counts.
  // Only the run-time-flag build (CFLAGS < 0) carries the counters: the launchers route instrumented launches there, so
  // the specialised builds do not spend three registers on them.
  constexpr bool COUNT = (CFLAGS < 0);
  int n_resolve = 0, n_retry = 0, n_fast = 0;
  double a[RPL], b[RPL], c[RPL];

  // ---------------- backward pass: controllable sets, reachability_algorithm.py:166-238 ----------------
  const double sde = sd_end ? sd_end[path] : 0.0;
  const double sds = sd_start ? sd_start[path] : 0.0;
  const double sdeh = sd_end_hi ? sd_end_hi[path] : sde;
  double kn0 = sde * sde, kn1 = sdeh * sdeh;  // K[N] = [sdmin^2, sdmax^2], reachability_algorithm.py:185
  if (lane == 0 && !forward_only) { double *kq = Kp(); kq[2 * N] = kn0; kq[2 * N + 1] = kn1; }
  int st = TB_STATUS_OK, fstage = -1;
  int up0 = 0, up1 = 0, dn0 = 0, dn1 = 0;  // active_c_up / active_c_down, initialised to zeros (pyx:526-527)
  if (forward_only) {
    st = status[path];
    fstage = fail_stage ? fail_stage[path] : -1;
    { const double *kq = Kp(); kn0 = kq[0]; kn1 = kq[1]; }
  }
  for (int q = 0; !FUSED && !forward_only && q < AHEAD && N - 1 - q >= 0; ++q) issue(N - 1 - q);
  // FUSED: the velocity bound of the NEXT stage is loaded one stage ahead (its L2 latency hides behind this stage)
  double2 xb_ahead = make_double2(0.0, 0.0);
  if constexpr (FUSED) {
    f_seg = src.nseg - 1;
    if (!forward_only && N > 0) xb_ahead = reinterpret_cast<const double2 *>(rec_path())[N - 1];
  }
  for (int i = forward_only ? -1 : N - 1; i >= 0; --i) {
    const double *gq = gp();
    const double g0 = gq[i], g1 = gq[i + 1];
    const double delta = g1 - g0;
    double xlo, xhi;
    double ulo = VAR_MIN, uhi = VAR_MAX;
    if constexpr (FUSED) {
      fused_row(g0, g1, true, delta, a[0], b[0], c[0]);
      xlo = xb_ahead.x;
      xhi = xb_ahead.y;
      if (i > 0) xb_ahead = reinterpret_cast<const double2 *>(rec_path())[i - 1];  // xbound [G][2] of this path
    } else {
      const double *rec = acquire();
      load_rows<RPL>(rec, R, nC, lane, a, b, c);
      xlo = rec[3 * R];
      xhi = rec[3 * R + 1];
      if constexpr (UB) { ulo = rec[3 * R + 2]; uhi = rec[3 * R + 3]; }
      __syncwarp();
      if (i - AHEAD >= 0) issue(i - AHEAD);
    }
    set_xnext_rows<RPL>(lane, delta, kn0, kn1, a, b, c);
    // low/high: pyx:587-601 with x_min = x_max = NaN
    double uu, xx;
    // x_upper: g = (1e-9, -1) -> v = (-1e-9, 1), slot active_c_down (g[1] <= 0), reachability_algorithm.py:229-233
    const bool ok_hi = lp2d_warp<RPL, true>(-1e-9, 1.0, a, b, c, nC, ulo, uhi, xlo, xhi, dn0, dn1, uu, xx, lane,
                                      n_resolve);
    const double x_upper = ok_hi ? xx : __longlong_as_double(0x7ff8000000000000LL);
    // x_lower: g = (-1e-9, 1) -> v = (1e-9, -1), slot active_c_up, reachability_algorithm.py:234-236
    bool ok_lo;
    double x_lower;
    double ufeas;
    if (fast_lower && xlo <= xhi && lp1d_fixed_x_warp<RPL>(1.0, xlo, a, b, c, ulo, uhi, ufeas) &&
        flat_rows_hold<RPL>(ufeas, xlo, a, b, c)) {
      // TB_SCAN_FAST_LOWER: some u is feasible at x = xlo, so min x IS xlo.  The reference reaches the same vertex
      // through ~4 projected re-solves and returns xlo plus rounding noise of its projection arithmetic
      // (|noise| <= ~1e-16, 5 % of the stages): this shortcut is exact for the LP, not bit-identical to that noise.
      ok_lo = true;
      x_lower = xlo;
      ++n_fast;
    } else {
        ok_lo = lp2d_warp<RPL, true>(1e-9, -1.0, a, b, c, nC, ulo, uhi, xlo, xhi, up0, up1, uu, xx, lane,
                                   n_resolve);
      x_lower = ok_lo ? xx : __longlong_as_double(0x7ff8000000000000LL);
    }
    if (x_lower < 0) x_lower = 0;  // reachability_algorithm.py:190-191
    if (lane == 0) { double *kq = Kp(); kq[2 * i] = x_lower; kq[2 * i + 1] = x_upper; }
    if (!(ok_hi && ok_lo)) {
      // reachability_algorithm.py:192-197: stop; the remaining K entries stay 0 (np.zeros)
      st = TB_STATUS_FAIL_UNCONTROLLABLE;
      fstage = i;
      { double *kq = Kp(); for (int j = lane; j < 2 * i; j += 32) kq[j] = 0.0; }
      break;
    }
    kn0 = x_lower;
    kn1 = x_upper;
  }
  if (COUNT && counters && lane == 0 && !forward_only) {
    // backward stages entered: N, or N - fstage when stage fstage failed; 2 LPs each (fast mode: n_fast of them 1-variable)
    const int nb = (st == TB_STATUS_OK) ? N : N - fstage;
    counters[path * 4 + 0] = 2 * nb - n_fast;
    counters[path * 4 + 1] = n_fast;
  }
  // drain a prefetch that was issued but not consumed (failure path), so the buffers can be reused
  while (n_waited < n_issued) (void)acquire();
  __syncwarp();

  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  const double x_start = sds * sds;
  if (Gp < G && !forward_only) {  // ragged batch: K entries past this path's grid are NaN
    double *kq = Kp();
    for (int j = 2 * Gp + lane; j < 2 * G; j += 32) kq[j] = nan_d;
  }
  if (backward_only) {
    if (lane == 0) {
      status[path] = st;
      if (fail_stage) fail_stage[path] = fstage;
    }
    return;
  }
  if (st == TB_STATUS_OK) {
    // kn0,kn1 == K[0]; admissibility check reachability_algorithm.py:290-301
    if (x_start + ALG_SMALL < kn0 || kn1 + ALG_SMALL < x_start) { st = TB_STATUS_FAIL_UNCONTROLLABLE; fstage = 0; }
  }
  if (st != TB_STATUS_OK) {
    for (int j = lane; j < Gp; j += 32) sdp[j] = nan_d;
    for (int j = lane; j < N; j += 32) up[j] = nan_d;
  } else {
    // ---------------- forward pass, reachability_algorithm.py:303-364 ----------------
    // sd = sqrt(x) is applied in one coalesced sweep after the pass; until then sd[] holds x
    double x = x_start;
    if (lane == 0) sdp[0] = x;
    for (int q = 0; !FUSED && q < AHEAD && q < N; ++q) issue(q);
    int i = 0;
    if constexpr (FUSED) f_seg = 0;
    for (; i < N; ++i) {
      const double *gq = gp();
      const double g0 = gq[i], g1 = gq[i + 1];
      const double delta = g1 - g0;
      double f_ulo = VAR_MIN, f_uhi = VAR_MAX;
      if constexpr (FUSED) {
        fused_row(g0, g1, false, delta, a[0], b[0], c[0]);
      } else {
        const double *rec = acquire();
        load_rows<RPL>(rec, R, nC, lane, a, b, c);
        if constexpr (UB) { f_ulo = rec[3 * R + 2]; f_uhi = rec[3 * R + 3]; }
        __syncwarp();
        if (i + AHEAD < N) issue(i + AHEAD);
      }
      const double *kq = Kp();
      const double k0 = kq[2 * (i + 1)], k1 = kq[2 * (i + 1) + 1];
      set_xnext_rows<RPL>(lane, delta, k0, k1, a, b, c);
      int tries = 0;
      bool ok;
      double uopt = 0.0;
      while (true) {
        // _forward_step: g = (-2 delta, -1), x_min = x_max = x -> 1-D branch, v0 = 2 delta (pyx:628-636);
        // TOPPRAsd's slowest pass uses g = (2 delta, 1) (desired_duration_algorithm.py:218-223)
          ok = lp1d_fixed_x_warp<RPL>(sd_slow ? -(2 * delta) : -(-2 * delta), x, a, b, c, f_ulo, f_uhi, uopt);
        if (ok || sd_mode || tries >= MAX_TRIES) break;  // TOPPRAsd has no retry rule
        x = py_max(x - ALG_TINY, 0.999 * x);  // reachability_algorithm.py:324-327
        ++tries;
        ++n_retry;
      }
      if (!ok) {
        // reachability_algorithm.py:337-342: xs[i+1:] = nan -> sd NaN -> ErrUnknown; us stay 0
        // (TOPPRAsd: us[i:] and xs[i+1:] become NaN, desired_duration_algorithm.py:106-111)
        st = TB_STATUS_ERR_UNKNOWN;
        fstage = i;
        if (lane == 0) sdp[i] = x;
        for (int j = i + 1 + lane; j < Gp; j += 32) sdp[j] = nan_d;
        for (int j = i + lane; j < N; j += 32) up[j] = sd_mode ? nan_d : 0.0;
        break;
      }
      double x_next = x + 2 * delta * uopt;                       // reachability_algorithm.py:352
      if (sd_mode) {
        x_next = py_min(k1, py_max(k0, x_next - ALG_SMALL));          // desired_duration_algorithm.py:117
      } else {
        x_next = py_max(x_next - ALG_TINY, 0.9999 * x_next);        // :353
        x_next = py_min(k1, py_max(k0, x_next));                      // :354
      }
      if (lane == 0) {
        up[i] = uopt;
        if (tries) sdp[i] = x;  // x was shrunk by the retry rule
        sdp[i + 1] = x_next;
      }
      x = x_next;
    }
    while (n_waited < n_issued) (void)acquire();
    __syncwarp();
    if (!sd_mode)  // TOPPRAsd combines the squared velocities: its passes return x = sd^2
      for (int j = lane; j < Gp; j += 32) sdp[j] = sqrt(sdp[j]);  // reachability_algorithm.py:365
  }
  if (Gp < G) {  // ragged batch: entries past this path's grid are NaN
    for (int j = Gp + lane; j < G; j += 32) sdp[j] = nan_d;
    for (int j = max(Gp - 1, 0) + lane; j < G - 1; j += 32) up[j] = nan_d;
  }
  if (lane == 0) {
    status[path] = st;
    if (fail_stage) fail_stage[path] = fstage;
    if (COUNT && counters) {
      // forward: one 1-variable LP per stage entered (N, or fstage + 1 when stage fstage failed) + one per retry;
      // none when the path failed before the forward pass
      const int n_fwd_stages = (st == TB_STATUS_OK) ? N : ((st == TB_STATUS_ERR_UNKNOWN) ? fstage + 1 : -1);
      if (forward_only) { counters[path * 4 + 0] = 0; counters[path * 4 + 1] = 0; }
      if (n_fwd_stages >= 0) counters[path * 4 + 1] += n_fwd_stages + n_retry;
      counters[path * 4 + 2] = n_resolve;
      counters[path * 4 + 3] = n_retry;
    }
  }
}

// compute_feasible_sets, reachability_algorithm.py:131-164: X[i] = [min x, max x] over stage i alone
// (x in [-1e4, 1e4], x_next in [-1e4, 1e4]); warm-start slots up/dn chained over i like the reference.
// ub: the records carry a u-bound pair (TB_SCAN_UBOUND).  The caller owns the row arrays, the warm-start slots and
// n_resolve: declared here, the row arrays double the spills of reachable_kernel<4, *>.  The record address is formed
// here from (records, path) rather than passed in as the path's base pointer: that way ptxas keeps
// feasible_kernel<3> at 112 registers instead of 114.
template <int RPL>
__device__ __forceinline__ void feasible_pass(const double *records, const long path, const int G, const int W,
                                              const int R, const int nC, const double *gp, const int N, const bool ub,
                                              const int lane, double *Xp, double (&a)[RPL], double (&b)[RPL],
                                              double (&c)[RPL],
                                              int &up0, int &up1, int &dn0, int &dn1, int &n_resolve) {
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  for (int i = 0; i <= N; ++i) {
    const double *rec = records + (size_t)path * G * W + (size_t)i * W;
    load_rows<RPL>(rec, R, nC, lane, a, b, c);
    const double xlo = fmax(rec[3 * R], -CVXPY_MAXX), xhi = fmin(rec[3 * R + 1], CVXPY_MAXX);  // pyx:598-601
    const double ulo = ub ? rec[3 * R + 2] : VAR_MIN, uhi = ub ? rec[3 * R + 3] : VAR_MAX;
    if (i < N) {
      const double delta = gp[i + 1] - gp[i];
      set_xnext_rows<RPL>(lane, delta, -CVXPY_MAXX, CVXPY_MAXX, a, b, c);
    }  // i == N: rows 0,1 stay (0,0,-1), pyx:621-625
    double uu, xx;
    // g_lower = (1e-9, 1): g[1] > 0 -> slot up; v = (-1e-9, -1)
    const bool ok0 = lp2d_warp<RPL>(-1e-9, -1.0, a, b, c, nC, ulo, uhi, xlo, xhi, up0, up1, uu, xx, lane,
                                    n_resolve);
    double x0 = ok0 ? xx : nan_d;
    const bool ok1 = lp2d_warp<RPL>(1e-9, 1.0, a, b, c, nC, ulo, uhi, xlo, xhi, dn0, dn1, uu, xx, lane,
                                    n_resolve);
    const double x1 = ok1 ? xx : nan_d;
    if (x0 < 0) x0 = 0;  // reachability_algorithm.py:160-162
    if (lane == 0) { Xp[2 * i] = x0; Xp[2 * i + 1] = x1; }
  }
}

template <int RPL>
__global__ void __launch_bounds__(32)
feasible_kernel(const double *__restrict__ records, const int W, const int R, const double *__restrict__ grid,
                const int grid_shared, const int B, const int G, const int ub, double *__restrict__ Xout,
                const int *__restrict__ glen) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  // glen (optional): ragged batches, as in scan_kernel; X past this path's gridpoints is NaN
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int N = Gp - 1, nC = R + 2;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  double *Xp = Xout + (size_t)path * G * 2;
  double a[RPL], b[RPL], c[RPL];
  int up0 = 0, up1 = 0, dn0 = 0, dn1 = 0, n_resolve = 0;
  for (int j = 2 * Gp + lane; j < 2 * G; j += 32) Xp[j] = __longlong_as_double(0x7ff8000000000000LL);
  feasible_pass<RPL>(records, path, G, W, R, nC, gp, N, ub != 0, lane, Xp, a, b, c, up0, up1, dn0, dn1, n_resolve);
}

// End of cy_solve_lp1d with the active index (pyx:93-144): the lanes' bounds my_hi / my_lo, each with the first of the
// lane's rows that set it (hi_idx / lo_idx, INT_MAX = none: strict improvement only), reduced over the warp.  Sequential
// semantics: the first row (lowest index) that reaches the final value wins; -1 = low, -2 = high if no row improved
// the bound.  Returns false if infeasible (cur_min > cur_max); else the optimum of max v0 * t and its active index.
__device__ __forceinline__ bool lp1d_active_reduce(const double v0, const double my_hi, const int hi_idx,
                                                   const double my_lo, const int lo_idx, double &out, int &active) {
  const double cur_max = warp_min(my_hi), cur_min = warp_max(my_lo);
  int hk = (hi_idx != INT_MAX && my_hi == cur_max) ? hi_idx : INT_MAX;
  int lk = (lo_idx != INT_MAX && my_lo == cur_min) ? lo_idx : INT_MAX;
  hk = __reduce_min_sync(FULL, hk);
  lk = __reduce_min_sync(FULL, lk);
  if (cur_min > cur_max) return false;
  if (fabs(v0) < LP_TINY || v0 < 0) { out = cur_min; active = (lk == INT_MAX) ? -1 : lk; }
  else { out = cur_max; active = (hk == INT_MAX) ? -2 : hk; }
  return true;
}

// cy_solve_lp1d (pyx:93-144) over the rows a*u + (b*x + c) <= 0 of one stage, WITH the active index the reference stores
// in active_c[0] of the chosen warm-start slot (pyx:645-650): the first row that set the final bound, -1 = low,
// -2 = high.  (The scan's forward pass uses the leaner lp1d_fixed_x_warp: nothing reads that index there.)
template <int RPL>
__device__ __forceinline__ bool lp1d_fixed_x_active_warp(const double v0, const double x, const double (&a)[RPL],
                                                         const double (&b)[RPL], const double (&c)[RPL], const int nC,
                                                         const double low0, const double high0, const int lane,
                                                         double &out_u, int &active) {
  double my_hi = high0, my_lo = low0;
  int hi_idx = INT_MAX, lo_idx = INT_MAX;
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r >= nC) continue;
    const double bxc = b[s] * x + c[s];
    if (a[s] > LP_TINY) {
      const double t = -bxc / a[s];
      if (t < my_hi) { my_hi = t; hi_idx = r; }
    } else if (a[s] < -LP_TINY) {
      const double t = -bxc / a[s];
      if (t > my_lo) { my_lo = t; lo_idx = r; }
    }
  }
  return lp1d_active_reduce(v0, my_hi, hi_idx, my_lo, lo_idx, out_u, active);
}

// compute_reachable_sets (reachability_algorithm.py:378-431), one warp per path, ONE launch: the feasible-set pass
// (compute_feasible_sets, :131-164) followed by the forward recursion L[i+1] = _one_step_forward(i, L[i], X[i+1]).
// Both passes run in the same kernel because the reference's seidelWrapper is stateful: the warm-start slots
// active_c_up / active_c_down left behind by the feasible-set pass are the ones the reachable pass starts from.
// Reference quirks kept: the objective and the x_next formula use deltas[i - 1] (deltas[N - 1] for i = 0, Python's
// negative index, :389-404) while rows 0/1 of the stage use deltas[i]; a stage with L[i,0] == L[i,1] takes the 1-variable
// branch of solve_stagewise_optim and stores its active index in slot [0] only; after a NaN the remaining L stay 0.
template <int RPL, bool UB>
__global__ void __launch_bounds__(32)
reachable_kernel(const double *__restrict__ records, const int W, const int R, const double *__restrict__ grid,
                 const int grid_shared, const int B, const int G, const double *__restrict__ sdmin,
                 const double *__restrict__ sdmax, double *__restrict__ Xout, double *__restrict__ Lout,
                 int *__restrict__ fail_stage, const int *__restrict__ glen) {
  const int lane = threadIdx.x & 31;
  const long path = warp_path();
  if (path >= B) return;
  // glen (optional): ragged batches, as in scan_kernel; X and L past this path's gridpoints are NaN
  const int Gp = glen ? min(max(glen[path], 1), G) : G;
  const int N = Gp - 1, nC = R + 2;
  const double *rec_path = records + (size_t)path * G * W;
  const double *gp = grid + (grid_shared ? 0 : (size_t)path * G);
  double *Xp = Xout + (size_t)path * G * 2;
  double *Lp = Lout + (size_t)path * G * 2;
  double a[RPL], b[RPL], c[RPL];
  int up0 = 0, up1 = 0, dn0 = 0, dn1 = 0, n_resolve = 0;
  const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
  for (int j = 2 * Gp + lane; j < 2 * G; j += 32) { Xp[j] = nan_d; Lp[j] = nan_d; }   // no pass below writes these
  feasible_pass<RPL>(records, path, G, W, R, nC, gp, N, UB, lane, Xp, a, b, c, up0, up1, dn0, dn1, n_resolve);
  __syncwarp();
  // ---- reachable sets ----
  const double s0 = sdmin ? sdmin[path] : 0.0, s1 = sdmax ? sdmax[path] : s0;
  double l0 = s0 * s0, l1 = s1 * s1;
  for (int j = 2 * lane; j < 2 * Gp; j += 64) { Lp[j] = 0.0; Lp[j + 1] = 0.0; }   // np.zeros((N + 1, 2))
  __syncwarp();
  if (lane == 0) { Lp[0] = l0; Lp[1] = l1; }
  int fs = -1;
  for (int i = 0; i < N; ++i) {
    const double *rec = rec_path + (size_t)i * W;
    load_rows<RPL>(rec, R, nC, lane, a, b, c);
    // low/high of solve_stagewise_optim (pyx:592-601): xbound of the stage intersected with [x_min, x_max] = L[i]
    const double r_lo = rec[3 * R], r_hi = rec[3 * R + 1];
    const double xlo = (r_lo > l0) ? r_lo : l0, xhi = (r_hi < l1) ? r_hi : l1;   // dbl_max / dbl_min (pyx:13-14)
    const double ulo = UB ? rec[3 * R + 2] : VAR_MIN, uhi = UB ? rec[3 * R + 3] : VAR_MAX;
    const double xn0 = Xp[2 * (i + 1)], xn1 = Xp[2 * (i + 1) + 1];
    // rows 0/1: NaN bound = absent = (0, 0, -1) (pyx:604-620)
    set_xnext_rows<RPL>(lane, gp[i + 1] - gp[i], xn0, xn1, a, b, c);
    if ((lane == 0 && xn0 != xn0) || (lane == 1 && xn1 != xn1)) { a[0] = 0.0; b[0] = 0.0; c[0] = -1.0; }
    const double dq = (i > 0) ? (gp[i] - gp[i - 1]) : (gp[N] - gp[N - 1]);   // deltas[i - 1]
    double u1 = nan_d, x1v = nan_d, u0 = nan_d, x0v = nan_d;
    bool ok_a, ok_b;
    if (l0 == l1) {
      // 1-variable branch (pyx:631-650): both objectives
      int act = 0;
      ok_a = lp1d_fixed_x_active_warp<RPL>(-(-2 * dq), l0, a, b, c, nC, ulo, uhi, lane, u1, act);
      if (ok_a) { x1v = l0; dn0 = act; }                 // g[1] = -1: active_c_down[0]
      ok_b = lp1d_fixed_x_active_warp<RPL>(-(2 * dq), l0, a, b, c, nC, ulo, uhi, lane, u0, act);
      if (ok_b) { x0v = l0; up0 = act; }                 // g[1] = +1: active_c_up[0]
    } else {
      ok_a = lp2d_warp<RPL>(-(-2 * dq), 1.0, a, b, c, nC, ulo, uhi, xlo, xhi, dn0, dn1, u1, x1v, lane, n_resolve);
      ok_b = lp2d_warp<RPL>(-(2 * dq), -1.0, a, b, c, nC, ulo, uhi, xlo, xhi, up0, up1, u0, x0v, lane, n_resolve);
    }
    double x_upper = ok_a ? (x1v + 2 * dq * u1) : nan_d;
    double x_lower = ok_b ? (x0v + 2 * dq * u0) : nan_d;
    if (x_lower < 0) x_lower = 0;
    if (lane == 0) { Lp[2 * (i + 1)] = x_lower; Lp[2 * (i + 1) + 1] = x_upper; }
    if (!(ok_a && ok_b)) { fs = i + 1; break; }   // "Path not parametrizable": return L (rest zeros)
    l0 = x_lower;
    l1 = x_upper;
  }
  if (lane == 0 && fail_stage) fail_stage[path] = fs;
}

// Batched stand-alone LPs (one warp per LP): the device counterparts of the reference's Python shims
// solve_lp2d / solve_lp1d (cy_seidel_solverwrapper.pyx:42-87).  Used by B200SolverWrapper.solve_stagewise_optim
// and by the LP-level known-answer / differential tests.
template <int RPL>
__global__ void __launch_bounds__(32)
lp2d_batch_kernel(const double *__restrict__ v, const double *__restrict__ a, const double *__restrict__ b,
                  const double *__restrict__ c, const double *__restrict__ low, const double *__restrict__ high,
                  const int *__restrict__ active_in, const int B, const int n, int *__restrict__ result,
                  double *__restrict__ optval, double *__restrict__ optvar, int *__restrict__ active_out) {
  const int lane = threadIdx.x & 31;
  const long p = warp_path();
  if (p >= B) return;
  double ra[RPL], rb[RPL], rc[RPL];
#pragma unroll
  for (int s = 0; s < RPL; ++s) {
    const int r = lane + 32 * s;
    if (r < n) { ra[s] = a[p * n + r]; rb[s] = b[p * n + r]; rc[s] = c[p * n + r]; }
    else { ra[s] = 0.0; rb[s] = 0.0; rc[s] = -1.0; }
  }
  int ac0 = active_in ? active_in[p * 2] : 0, ac1 = active_in ? active_in[p * 2 + 1] : 0;
  int n_resolve = 0;
  double uu = 0.0, xx = 0.0;
  const double v0 = v[p * 3], v1 = v[p * 3 + 1], v2 = v[p * 3 + 2];
  const bool ok = lp2d_warp<RPL>(v0, v1, ra, rb, rc, n, low[p * 2], high[p * 2], low[p * 2 + 1], high[p * 2 + 1], ac0,
                                 ac1, uu, xx, lane, n_resolve);
  if (lane == 0) {
    result[p] = ok ? 1 : 0;
    const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
    optvar[p * 2] = ok ? uu : nan_d;
    optvar[p * 2 + 1] = ok ? xx : nan_d;
    optval[p] = ok ? (uu * v0 + xx * v1 + v2) : nan_d;  // pyx:389
    active_out[p * 2] = ac0;
    active_out[p * 2 + 1] = ac1;
  }
}

// cy_solve_lp1d with the active index (pyx:93-144): max v0 x + v1, a x + b <= 0, low <= x <= high.
__global__ void lp1d_batch_kernel(const double *__restrict__ v, const double *__restrict__ a,
                                  const double *__restrict__ b, const double *__restrict__ low,
                                  const double *__restrict__ high, const int B, const int n,
                                  int *__restrict__ result, double *__restrict__ optval,
                                  double *__restrict__ optvar, int *__restrict__ active_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long p = (long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (p >= B) return;
  double my_hi = high[p], my_lo = low[p];
  int hi_idx = INT_MAX, lo_idx = INT_MAX;
  for (int r = lane; r < n; r += 32) {
    const double ar = a[p * n + r], br = b[p * n + r];
    if (ar > LP_TINY) {
      const double cx = -br / ar;
      if (cx < my_hi) { my_hi = cx; hi_idx = r; }
    } else if (ar < -LP_TINY) {
      const double cx = -br / ar;
      if (cx > my_lo) { my_lo = cx; lo_idx = r; }
    }
  }
  const double v0 = v[p * 2];
  double x = 0.0;
  int active = 0;
  const bool ok = lp1d_active_reduce(v0, my_hi, hi_idx, my_lo, lo_idx, x, active);
  if (lane == 0) {
    const double nan_d = __longlong_as_double(0x7ff8000000000000LL);
    result[p] = ok ? 1 : 0;
    optvar[p] = ok ? x : nan_d;
    optval[p] = ok ? (v0 * x + v[p * 2 + 1]) : nan_d;
    active_out[p] = ok ? active : 0;
  }
}

// Register budget of the record scan for nC <= 32: 65536 / (32 * 32) -> 64 registers/thread (measured: 32 > 28 > 24);
// the 4096-path batch of BASELINE cfg 2 is then a single wave on 132 SMs
constexpr int SCAN_WARPS_PER_SM = 32;
// resident warps per SM for nC in (32, 64].  H100 80GB (400 W), cfg 3 scan (16384 x 500, nC = 50), two runs:
// 16 -> 24.1 / 23.6 ms, 20 -> 23.1 / 22.9 ms, 24 (80 registers) -> 22.6 / 22.4 ms
constexpr int SCAN_RPL2_WARPS_PER_SM = 24;
constexpr int SCAN_FUSED_WARPS_PER_SM = 28;  // 72 registers: 28 resident one-warp CTAs per SM

using ScanKernel = decltype(&scan_kernel<1, SCAN_WARPS_PER_SM, false>);  // every build has this signature

// The one-row-per-lane scan_kernel build of a launch.  The three launch kinds of the batched solver (full scan, backward
// only, forward only) get their own build with the mode folded in; instrumented (counters) and ragged (glen) launches and
// the TOPPRAsd modes run on the run-time-flag build.
template <int MINB, bool FUSED>
ScanKernel scan_build(const int flags, const bool counters_or_glen) {
  const bool fast = (flags & TB_SCAN_FAST_LOWER) != 0;
  const int mode = flags & (TB_SCAN_BACKWARD_ONLY | TB_SCAN_SD_FORWARD | TB_SCAN_SD_SLOW | TB_SCAN_FORWARD_ONLY);
  if (!counters_or_glen) {
    if (mode == 0) return fast ? scan_kernel<1, MINB, true, 0, FUSED> : scan_kernel<1, MINB, false, 0, FUSED>;
    if (mode == TB_SCAN_BACKWARD_ONLY)
      return fast ? scan_kernel<1, MINB, true, TB_SCAN_BACKWARD_ONLY, FUSED>
                  : scan_kernel<1, MINB, false, TB_SCAN_BACKWARD_ONLY, FUSED>;
    if (mode == TB_SCAN_FORWARD_ONLY)
      return fast ? scan_kernel<1, MINB, true, TB_SCAN_FORWARD_ONLY, FUSED>
                  : scan_kernel<1, MINB, false, TB_SCAN_FORWARD_ONLY, FUSED>;
  }
  return fast ? scan_kernel<1, MINB, true, -1, FUSED> : scan_kernel<1, MINB, false, -1, FUSED>;
}

template <int RPL>
int launch_scan(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                double *sd, double *u, int *status, int *fail_stage, int *counters, const int *glen,
                cudaStream_t stream) {
  const size_t smem = (size_t)SCAN_NBUF * W * sizeof(double) + SCAN_NBUF * sizeof(uint64_t) + 4 * sizeof(void *);
  const bool fast = (flags & TB_SCAN_FAST_LOWER) != 0;
  ScanKernel kern;
  if constexpr (RPL == 1) {
    kern = scan_build<SCAN_WARPS_PER_SM, false>(flags, counters || glen);
  } else {
    kern = fast ? scan_kernel<RPL, 1, true> : scan_kernel<RPL, 1, false>;
  }
  if constexpr (RPL == 2) {
    // nC in (32, 64] (BASELINE cfg 3: 50 rows).  Left alone the compiler takes about 150 registers (13 resident warps
    // per SM); the capped build trades a few spills for residency.
    if (!fast && !counters) kern = scan_kernel<RPL, SCAN_RPL2_WARPS_PER_SM, false>;
  }
  if (flags & TB_SCAN_UBOUND)  // records with a u-bound pair: the generic build (exact mode only)
    kern = scan_kernel<RPL, 1, false, -1, false, true>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("tb_scan: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  }
  kern<<<B, 32, smem, stream>>>(records, W, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, flags, K, sd, u,
                                status, fail_stage, counters, glen, VelAccSrc{});
  return check_launch("tb_scan");
}

// Fused vel+acc scan (one row per lane).  MINB = resident one-warp CTAs per SM the register budget is sized for.
template <int MINB>
int launch_scan_velacc_occ(const VelAccSrc &src, int W, int R, const double *grid, int grid_shared, int B, int G,
                           const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                           double *sd, double *u, int *status, int *fail_stage, int *counters, const int *glen,
                           cudaStream_t stream) {
  const size_t smem = (size_t)W * sizeof(double) + SCAN_NBUF * sizeof(uint64_t) + 4 * sizeof(void *);
  const ScanKernel kern = scan_build<MINB, true>(flags, counters || glen);
  kern<<<B, 32, smem, stream>>>(nullptr, W, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, flags, K, sd, u,
                                status, fail_stage, counters, glen, src);
  return check_launch("tb_scan_velacc");
}

int launch_scan_velacc(const VelAccSrc &src, int W, int R, const double *grid, int grid_shared, int B, int G,
                       const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                       double *sd, double *u, int *status, int *fail_stage, int *counters, const int *glen,
                       cudaStream_t stream) {
  // Register budget by batch size: while 28 resident one-warp CTAs per SM cover the whole batch in one wave, the
  // 72-register build is used; larger batches are issue-bound and want the 32 resident warps per SM of the 64-register
  // build.
  const auto launch = ((long)B <= (long)num_sms() * SCAN_FUSED_WARPS_PER_SM)
                          ? launch_scan_velacc_occ<SCAN_FUSED_WARPS_PER_SM>
                          : launch_scan_velacc_occ<SCAN_WARPS_PER_SM>;
  const int mode = flags & (TB_SCAN_BACKWARD_ONLY | TB_SCAN_SD_FORWARD | TB_SCAN_SD_SLOW | TB_SCAN_FORWARD_ONLY);
  if ((mode == 0 || mode == TB_SCAN_FORWARD_ONLY) && !counters && !glen && forward_threads_supported(src.dof, B)) {
    // large batches (issue-bound): the forward pass runs with one thread per path (tb_scan_fwd.cu) after a backward-only
    // launch of this kernel
    if (mode == 0) {
      const int bflags = (flags & TB_SCAN_FAST_LOWER) | TB_SCAN_BACKWARD_ONLY;
      const int rc = launch(src, W, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, bflags, K, nullptr, nullptr,
                            status, fail_stage, nullptr, nullptr, stream);
      if (rc) return rc;
    }
    return launch_forward_threads(src, R == 4 * src.dof, grid, grid_shared, B, G, sd_start, K, sd, u, status, fail_stage, stream);
  }
  return launch(src, W, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, flags, K, sd, u, status, fail_stage,
                counters, glen, stream);
}

template <int RPL>
int launch_feasible(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                    const int *glen, int ub, double *X, cudaStream_t stream) {
  feasible_kernel<RPL><<<B, 32, 0, stream>>>(records, W, R, grid, grid_shared, B, G, ub, X, glen);
  return check_launch("tb_feasible_sets");
}

template <int RPL>
int launch_reachable(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                     const int *glen, const double *sdmin, const double *sdmax, int flags, double *X, double *L,
                     int *fail_stage, cudaStream_t stream) {
  if (flags & TB_SCAN_UBOUND)
    reachable_kernel<RPL, true><<<B, 32, 0, stream>>>(records, W, R, grid, grid_shared, B, G, sdmin, sdmax, X, L,
                                                      fail_stage, glen);
  else
    reachable_kernel<RPL, false><<<B, 32, 0, stream>>>(records, W, R, grid, grid_shared, B, G, sdmin, sdmax, X, L,
                                                       fail_stage, glen);
  return check_launch("tb_reachable_sets");
}

int check_scan_args(const char *fn, const void *records, int W, int R, const void *grid, int B, int G) {
  if (!records || !grid || B <= 0 || G <= 0 || R < 0) { set_error("%s: bad argument", fn); return TB_ERR_ARG; }
  if (R > MAX_ROWS) { set_error("%s: R=%d > %d rows", fn, R, MAX_ROWS); return TB_ERR_UNSUPPORTED; }
  if (W < 3 * R + 2 || (W & 1)) { set_error("%s: record stride W=%d must be even and >= 3R+2", fn, W); return TB_ERR_ALIGN; }
  if (((uintptr_t)records & 15) != 0) { set_error("%s: records not 16-byte aligned", fn); return TB_ERR_ALIGN; }
  return 0;
}

}  // namespace
}  // namespace tb

extern "C" int tb_scan_ragged(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                              const int *glen, const double *sd_start, const double *sd_end, const double *sd_end_hi,
                              int flags, double *K, double *sd, double *u, int *status, int *fail_stage, int *counters,
                              void *stream) {
  using namespace tb;
  int rc = check_scan_args("tb_scan", records, W, R, grid, B, G);
  if (rc) return rc;
  if ((flags & TB_SCAN_UBOUND) && W < 3 * R + 4) { set_error("tb_scan: TB_SCAN_UBOUND needs records of W >= 3R+4 doubles"); return TB_ERR_ARG; }
  if ((flags & TB_SCAN_UBOUND) && (flags & TB_SCAN_FAST_LOWER)) { set_error("tb_scan: TB_SCAN_UBOUND excludes TB_SCAN_FAST_LOWER"); return TB_ERR_UNSUPPORTED; }
  if (glen && grid_shared) { set_error("tb_scan: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  const bool backward_only = (flags & TB_SCAN_BACKWARD_ONLY) != 0;
  if (!K || !status || (!backward_only && (!sd || (G > 1 && !u)))) { set_error("tb_scan: null output"); return TB_ERR_ARG; }
  return with_rows_per_lane(R + 2, [&](auto rpl) {
    return launch_scan<rpl.value>(records, W, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, flags, K, sd, u,
                                  status, fail_stage, counters, glen, (cudaStream_t)stream);
  });
}

extern "C" int tb_scan_ex(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                          const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags, double *K,
                          double *sd, double *u, int *status, int *fail_stage, int *counters, void *stream) {
  return tb_scan_ragged(records, W, R, grid, grid_shared, B, G, nullptr, sd_start, sd_end, sd_end_hi, flags, K, sd, u,
                        status, fail_stage, counters, stream);
}

extern "C" int tb_scan_velacc_ragged(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof,
                                     const double *grid, int grid_shared, int B, int G, const int *glen,
                                     const double *alim, int lim_shared, int interp, const double *xbound,
                                     const double *sd_start, const double *sd_end, const double *sd_end_hi, int flags,
                                     double *K, double *sd, double *u, int *status, int *fail_stage, int *counters,
                                     void *stream) {
  using namespace tb;
  if (glen && grid_shared) { set_error("tb_scan_velacc: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if (!ppoly || !breaks || !grid || !alim || !xbound || B <= 0 || G <= 0 || nseg <= 0 || dof <= 0) {
    set_error("tb_scan_velacc: bad argument");
    return TB_ERR_ARG;
  }
  const bool backward_only = (flags & TB_SCAN_BACKWARD_ONLY) != 0;
  if (!K || !status || (!backward_only && (!sd || (G > 1 && !u)))) { set_error("tb_scan_velacc: null output"); return TB_ERR_ARG; }
  if (((uintptr_t)xbound & 15) != 0) { set_error("tb_scan_velacc: xbound not 16-byte aligned"); return TB_ERR_ALIGN; }
  const int R = (interp ? 4 : 2) * dof;
  const int Wc = (nseg * dof * 6 + nseg + 1 + 1) & ~1;  // per-warp coefficient block (48-byte entries), doubles
  if (R + 2 > 32 || Wc * 8 > 16 * 1024) {
    set_error("tb_scan_velacc: %d rows / %d segments exceed the fused kernel (one row per lane, 16 KB of coefficients): "
              "use tb_coeff_velacc + tb_scan", R, nseg);
    return TB_ERR_UNSUPPORTED;
  }
  const VelAccSrc src{ppoly, breaks, alim, xbound, breaks_shared, nseg, dof, lim_shared};
  return launch_scan_velacc(src, Wc, R, grid, grid_shared, B, G, sd_start, sd_end, sd_end_hi, flags, K, sd, u, status,
                            fail_stage, counters, glen, (cudaStream_t)stream);
}

extern "C" int tb_scan_velacc(const double *ppoly, const double *breaks, int breaks_shared, int nseg, int dof,
                              const double *grid, int grid_shared, int B, int G, const double *alim, int lim_shared,
                              int interp, const double *xbound, const double *sd_start, const double *sd_end,
                              const double *sd_end_hi, int flags, double *K, double *sd, double *u, int *status,
                              int *fail_stage, int *counters, void *stream) {
  return tb_scan_velacc_ragged(ppoly, breaks, breaks_shared, nseg, dof, grid, grid_shared, B, G, nullptr, alim,
                               lim_shared, interp, xbound, sd_start, sd_end, sd_end_hi, flags, K, sd, u, status,
                               fail_stage, counters, stream);
}

extern "C" int tb_scan(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                       const double *sd_start, const double *sd_end, double *K, double *sd, double *u, int *status,
                       int *fail_stage, void *stream) {
  return tb_scan_ex(records, W, R, grid, grid_shared, B, G, sd_start, sd_end, nullptr, 0, K, sd, u, status, fail_stage,
                    nullptr, stream);
}

extern "C" int tb_feasible_sets_ragged(const double *records, int W, int R, const double *grid, int grid_shared, int B,
                                       int G, const int *glen, int flags, double *X, void *stream) {
  using namespace tb;
  int rc = check_scan_args("tb_feasible_sets", records, W, R, grid, B, G);
  if (rc) return rc;
  if (!X) { set_error("tb_feasible_sets: null output"); return TB_ERR_ARG; }
  if (glen && grid_shared) { set_error("tb_feasible_sets: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  const int ub = (flags & TB_SCAN_UBOUND) ? 1 : 0;
  if (ub && W < 3 * R + 4) { set_error("tb_feasible_sets: TB_SCAN_UBOUND needs W >= 3R+4"); return TB_ERR_ARG; }
  return with_rows_per_lane(R + 2, [&](auto rpl) {
    return launch_feasible<rpl.value>(records, W, R, grid, grid_shared, B, G, glen, ub, X, (cudaStream_t)stream);
  });
}

extern "C" int tb_feasible_sets_ex(const double *records, int W, int R, const double *grid, int grid_shared, int B,
                                   int G, int flags, double *X, void *stream) {
  return tb_feasible_sets_ragged(records, W, R, grid, grid_shared, B, G, nullptr, flags, X, stream);
}

extern "C" int tb_feasible_sets(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                                double *X, void *stream) {
  return tb_feasible_sets_ex(records, W, R, grid, grid_shared, B, G, 0, X, stream);
}

extern "C" int tb_reachable_sets_ragged(const double *records, int W, int R, const double *grid, int grid_shared,
                                        int B, int G, const int *glen, const double *sdmin, const double *sdmax,
                                        int flags, double *X, double *L, int *fail_stage, void *stream) {
  using namespace tb;
  int rc = check_scan_args("tb_reachable_sets", records, W, R, grid, B, G);
  if (rc) return rc;
  if (!X || !L) { set_error("tb_reachable_sets: null output"); return TB_ERR_ARG; }
  if (glen && grid_shared) { set_error("tb_reachable_sets: ragged batches (glen) need per-path grids [B][G]"); return TB_ERR_ARG; }
  if ((flags & TB_SCAN_UBOUND) && W < 3 * R + 4) { set_error("tb_reachable_sets: TB_SCAN_UBOUND needs W >= 3R+4"); return TB_ERR_ARG; }
  return with_rows_per_lane(R + 2, [&](auto rpl) {
    return launch_reachable<rpl.value>(records, W, R, grid, grid_shared, B, G, glen, sdmin, sdmax, flags, X, L,
                                       fail_stage, (cudaStream_t)stream);
  });
}

extern "C" int tb_reachable_sets(const double *records, int W, int R, const double *grid, int grid_shared, int B, int G,
                                 const double *sdmin, const double *sdmax, int flags, double *X, double *L,
                                 int *fail_stage, void *stream) {
  return tb_reachable_sets_ragged(records, W, R, grid, grid_shared, B, G, nullptr, sdmin, sdmax, flags, X, L, fail_stage,
                                  stream);
}

extern "C" int tb_lp2d_batch(const double *v, const double *a, const double *b, const double *c, const double *low,
                             const double *high, const int *active_in, int B, int n, int *result, double *optval,
                             double *optvar, int *active_out, void *stream) {
  using namespace tb;
  if (!v || !low || !high || !result || !optval || !optvar || !active_out || B <= 0 || n < 0 || (n > 0 && (!a || !b || !c))) {
    set_error("tb_lp2d_batch: bad argument");
    return TB_ERR_ARG;
  }
  if (n > MAX_ROWS + 2) { set_error("tb_lp2d_batch: n=%d > %d rows", n, MAX_ROWS + 2); return TB_ERR_UNSUPPORTED; }
  with_rows_per_lane(n, [&](auto rpl) {
    lp2d_batch_kernel<rpl.value><<<B, 32, 0, (cudaStream_t)stream>>>(v, a, b, c, low, high, active_in, B, n, result,
                                                                     optval, optvar, active_out);
  });
  return check_launch("tb_lp2d_batch");
}

extern "C" int tb_lp1d_batch(const double *v, const double *a, const double *b, const double *low, const double *high,
                             int B, int n, int *result, double *optval, double *optvar, int *active_out,
                             void *stream) {
  using namespace tb;
  if (!v || !low || !high || !result || !optval || !optvar || !active_out || B <= 0 || n < 0 || (n > 0 && (!a || !b))) {
    set_error("tb_lp1d_batch: bad argument");
    return TB_ERR_ARG;
  }
  lp1d_batch_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(v, a, b, low, high, B, n, result, optval, optvar, active_out);
  return check_launch("tb_lp1d_batch");
}
