// Likelihood pass of the Vecchia factor with TWO observations per warp (one per half-warp) — the dominant kernel of
// GPB_EvalNegLogLikelihood at the headline configuration (n = 1e6, m = 30, d = 2).
//
// Same mathematics as vecchia_factor_kernel<COV, MODE_NLL, 2, 30> (vecchia_factor.cuh: augmented (q+2) x (q+2) matrix, one
// right-looking Cholesky with look-ahead, D_i = pivot q, (By)_i^2 / D_i = L[q+1][q]^2; reference: CalcCovFactorGradientVecchia,
// src/GPBoost/Vecchia_utils.cpp:1461-1684 + re_model_template.h:9957-9964, :2947), different mapping:
//   * a half-warp owns one observation; lane hl of the half owns matrix rows hl ("lo", columns 0..15 matter) and hl + 16 ("hi"),
//     48 register doubles per lane instead of 32 for twice the observations;
//   * a rank-1 update step costs (30 - k) DFMA for the hi rows plus (15 - k) for the lo rows per TWO observations (616 warp
//     instructions per pair instead of 2 x 496), the pivot chain (shuffle, rsqrt, scale) is issued once for both, and every
//     LDS.128 that broadcasts two entries of L's column serves both halves (the two matrices are offset by 16 bytes modulo 128, so
//     the two 16-byte addresses of an instruction fall into different banks: one wavefront). ncu of the one-observation kernel
//     has the LSU pipe at 78 % and the FP64 pipe at 54 %: both counts drop here;
//   * the 465 pair covariances of an observation take 30 circulant rounds of 16 lanes (both halves in the same instruction).
// Partial sums are kept per half-warp (partials row = 2 * warp + half) and reduced in fixed order as before.
#pragma once
#include "vecchia_factor.cuh"

namespace gpb {

constexpr int kNll2Half = 32 * kLd + 2;  // doubles per half: 32 x 33 matrix + 2 pad -> halves 16 bytes apart modulo 128 bytes
constexpr int kNll2Pts = 96;             // doubles per half: points 0..30 and a copy of points 0..15 behind them (47 x 2, padded)
// ---- covariance evaluation of this kernel. ncu of the first version had 52 % of
// the stall samples in the pair-covariance rounds: every round a serial chain of ~33 dependent FP64 instructions (the shared-memory
// store of round r ordered the load of round r + 1 behind it), issued at the DFMA latency. Here
//   * the rounds run in groups whose values stay in registers until the group is done (no store between the point loads of a
//     group: its chains interleave);
//   * the points are pre-scaled by the range parameter (distance in units of the range comes out of the square root directly);
//   * sqrt(x) = x * rsqrt(x) with the correction applied to x * y (one multiply less);
//   * exp() reduces the argument to |r| <= ln2 / 64 with a 32-entry table of 2^(j/32) held one entry per lane: degree-6 instead of
//     degree-13 polynomial (truncation 3.5e-18 relative); underflow is caught on the integer pipe.
// Matern-1.5 pair: 22 FP64 instructions instead of 33.
__constant__ double kExp2Tab32[32] = {
    1.0, 1.0218971486541166, 1.0442737824274138, 1.0671404006768237, 1.0905077326652577, 1.1143867425958924, 1.1387886347566916,
    1.1637248587775775, 1.189207115002721, 1.215247359980469, 1.241857812073484, 1.2690509571917332, 1.2968395546510096,
    1.3252366431597413, 1.3542555469368927, 1.383909881963832, 1.4142135623730951, 1.4451808069770467, 1.4768261459394993,
    1.5091644275934228, 1.5422108254079407, 1.5759808451078865, 1.6104903319492543, 1.645755478153965, 1.681792830507429,
    1.718619298122478, 1.7562521603732995, 1.7947090750031072, 1.8340080864093424, 1.8741676341103, 1.9152065613971474,
    1.9571441241754002};

// exp(ax) for |ax| <= 700 (the caller zeroes the result below -700): n = rint(ax * 32 / ln2), r = ax - n ln2 / 32 (two-step,
// n * hi exact), e^r by Taylor to r^6, 2^(n/32) = 2^(n >> 5) * tab[n & 31] with the power of two added into the exponent field.
// tab_lane: lane l of the warp holds 2^(l/32) — the lookup is a register shuffle (a shared-memory table would order every lookup
// behind the preceding stores of covariance values: same address space, run-time indices). All 32 lanes must call this together.
__device__ __forceinline__ double exp_tab32(double ax, double tab_lane) {
  const double t = fma(ax, 46.16624130844683, 6755399441055744.0);
  const double n = t - 6755399441055744.0;
  double r = fma(n, -6.93147180369123816490e-01 / 32., ax);
  r = fma(n, -1.90821492927058770002e-10 / 32., r);
  const int ni = __double2loint(t);
  double pl = 1. / 720.;
  pl = fma(pl, r, 1. / 120.);
  pl = fma(pl, r, 1. / 24.);
  pl = fma(pl, r, 1. / 6.);
  pl = fma(pl, r, 0.5);
  pl = fma(pl, r, 1.0);
  pl = fma(pl, r, 1.0);
  const double v = pl * __shfl_sync(0xffffffffu, tab_lane, ni & 31);
  return __hiloint2double(__double2hiint(v) + ((ni >> 5) << 20), __double2loint(v));
}
// ax < -700 by the high word alone (sign-magnitude order of negative doubles; -700 = 0xC085E000_00000000)
__device__ __forceinline__ bool below_m700(double ax) { return (unsigned)__double2hiint(ax) > 0xC085E000u; }

// covariance (and d / d log range) from the SCALED squared distance d2s = (range * dist)^2 (Gaussian: range * dist^2), guarded
// away from 0 by the caller; logvar = log(var). Same closed forms as cov_eval (cov_fcts.h:2100-2118, :2154, :2535-2563).
template <int COV, bool GRAD>
__device__ __forceinline__ double cov_eval_scaled(double d2s, double var, double logvar, double tab, double& grad) {
  double val;
  if (COV == COV_GAUSSIAN) {
    const double ax = logvar - d2s;
    val = exp_tab32(ax, tab);
    if (below_m700(ax)) val = 0.;
    if (GRAD) grad = -d2s * val;
    return val;
  }
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d2s));
  const double g = d2s * y;
  const double e = fma(-g, y, 1.0);
  const double rd = fma(g * e, fma(0.375, e, 0.5), g);  // sqrt(d2s)
  if (COV == COV_EXPONENTIAL) {
    const double ax = logvar - rd;
    val = exp_tab32(ax, tab);
    if (below_m700(ax)) val = 0.;
    if (GRAD) grad = -rd * val;
  } else {
    double ex = exp_tab32(-rd, tab);
    if (below_m700(-rd)) ex = 0.;
    if (COV == COV_MATERN15) {
      val = fma(var, rd, var) * ex;
      if (GRAD) grad = -(var * d2s) * ex;
    } else {
      const double q1 = 1. + rd;
      val = (var * fma(d2s, 1. / 3., q1)) * ex;
      if (GRAD) grad = -(var * (1. / 3.)) * d2s * q1 * ex;
    }
  }
  return val;
}

#ifndef GPB_NLL2_BLOCKS
#define GPB_NLL2_BLOCKS 3
#endif
// gradient pass: the range-derivative pair values are parked in the strict upper triangle of the shared matrix buffer (the
// factorisation only uses column c, rows >= c) instead of 60 registers per lane held across the elimination: the pass fits the
// register budget of three resident CTAs per SM like the likelihood pass. GPB_NLL2_GRAD_SMEM=0: registers, two CTAs (first version).
#ifndef GPB_NLL2_GRAD_SMEM
#define GPB_NLL2_GRAD_SMEM 1
#endif
#ifndef GPB_NLL2_GRAD_BLOCKS
#define GPB_NLL2_GRAD_BLOCKS (GPB_NLL2_GRAD_SMEM ? 3 : 2)
#endif

// GRAD = true: the gradient pass (MODE_GRAD of vecchia_factor_kernel: adjoint identities dD_k = b^T dSigma~_k b,
// (dB_k y)_i = -b^T dSigma~_k w~ with b = [-A_i, 1], w~ = [S^-1 y_N, 0]; re_model_template.h:1988-2010, Vecchia_utils.cpp:1636-1652) in
// the same layout: the range-derivative pair values stay in the registers of the lane that computed them (30 per lane), the two
// back substitutions (A_i and S^-1 y_N) run with lane hl owning unknowns hl and hl + 16, b and w~ are exchanged through the
// (by then free) point buffer. 4 warps x 2 CTAs per SM = 16 observations in flight (one-observation kernel: 12).
// MODE = MODE_STORE: one back substitution, A_i / D_i^-1 / u_i written like vecchia_factor_kernel<MODE_STORE>.
template <int COV, int MODE>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, MODE == MODE_GRAD ? GPB_NLL2_GRAD_BLOCKS : GPB_NLL2_BLOCKS) vecchia_nll2_kernel(const FactorArgs p) {
  constexpr bool GP_SMEM = GPB_NLL2_GRAD_SMEM != 0;
  constexpr bool GRAD = MODE == MODE_GRAD;
  constexpr bool SOLVE = MODE != MODE_NLL;
  static_assert(MODE == MODE_NLL || MODE == MODE_STORE || MODE == MODE_GRAD, "modes: NLL, STORE, GRAD");
  constexpr int MT = 30, P = 31;
  extern __shared__ __align__(16) double smem_raw[];
  const int lane = threadIdx.x & 31, hl = lane & 15, hh = lane >> 4, wib = threadIdx.x >> 5;
  const int hbase = lane & 16;  // first lane of my half
  // per-warp shared layout: two matrices of 32 x kLd + 2, then two point buffers of kNll2Pts
  double* S = smem_raw + (size_t)wib * (2 * (kNll2Half + kNll2Pts)) + (size_t)hh * kNll2Half;
  double* pts = smem_raw + (size_t)wib * (2 * (kNll2Half + kNll2Pts)) + 2 * kNll2Half + (size_t)hh * kNll2Pts;
  const int64_t gwarp = (int64_t)blockIdx.x * kWarpsPerBlock + wib, nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  const int m = p.m;
  const double var = p.var;
  const double sc = COV == COV_GAUSSIAN ? sqrt(p.range) : p.range;  // points are kept scaled: pair distances in units of the range
  const double logvar = log(var);
  const double tab = kExp2Tab32[lane];
  double acc0 = 0., acc1 = 0., acc2 = 0.;
  double accg[GRAD ? 6 : 1];
#pragma unroll
  for (int k = 0; k < (GRAD ? 6 : 1); ++k) accg[k] = 0.;

  // source observation of point slot s of row ii (-1: dummy slot)
  auto slot_src = [&](int64_t ii, int s) -> int {  // observation indices fit 32 bits (the neighbour table is int32)
    const int qq = ii < m ? (int)ii : m;
    if (s < qq) return p.nn[ii * m + s];
    return s == MT ? (int)ii : -1;
  };
  auto row_of = [&](int64_t it) -> int64_t { return p.row_begin + 2 * it + hh; };
  // software pipeline, two deep: the neighbour indices of the pair after the next one and the responses / coordinates of the next
  // pair (addressed by indices that were loaded one iteration earlier) are in flight while this pair is computed — a gather whose
  // data loads wait for its own index load stalls the warp for a full memory latency (12 % of the samples of the first version)
  int64_t it = gwarp;
  int64_t i = row_of(it);
  bool active = i < p.row_end;
  int s_lo = -1, s_hi = -1, sn_lo = -1, sn_hi = -1;
  double2 c_lo = make_double2(0., 0.), c_hi = c_lo;
  double y_lo = 0., y_hi = 0.;
  auto fetch_idx = [&](int64_t ii, bool act, int& a_lo, int& a_hi) {
    a_lo = -1; a_hi = -1;
    if (act) {
      a_lo = slot_src(ii, hl);
      a_hi = hl + 16 <= MT ? slot_src(ii, hl + 16) : -1;  // slot 31 does not exist (row 31 = responses)
    }
  };
  auto fetch_data = [&]() {  // of the slots named by s_lo / s_hi
    y_lo = 0.; y_hi = 0.;
    if (s_lo >= 0) { y_lo = p.y[s_lo]; c_lo = *reinterpret_cast<const double2*>(p.coords + (int64_t)s_lo * 2); }
    if (s_hi >= 0) { y_hi = p.y[s_hi]; c_hi = *reinterpret_cast<const double2*>(p.coords + (int64_t)s_hi * 2); }
  };
  fetch_idx(i, active, s_lo, s_hi);
  fetch_data();
  fetch_idx(row_of(it + nwarps), row_of(it + nwarps) < p.row_end, sn_lo, sn_hi);

  // ---- pair covariances: round r -> offset t = r / 2 + 1, own point pi = hl + 16 (r & 1), partner o = (pi + t) mod P.
  // Every address of a round is a per-lane base plus a compile-time offset (the lane-dependent addresses of the 30 rounds, kept
  // across the pair loop, were what spilled): point s sits at pts2[s] and, for s < 16, again at pts2[s + P], so the partner is
  // read at pts2[pi + t] without a wrap; pair (min, max) sits at S[min * kLd + max], i.e. at pi (kLd + 1) + t when pi + t < P and
  // at pi (kLd + 1) + (t - P) kLd when the partner wraps (only hi rounds wrap: hl + t <= 30). The padded pair (lane 15, odd
  // rounds, pi = 31) is computed on a copied point and not stored.
  double2* pts2 = reinterpret_cast<double2*>(pts);
  auto Sd = [&]() { return S + hl * (kLd + 1); };         // S[hl][hl]: base of the lo rounds
  auto Sh = [&]() { return S + (hl + 16) * (kLd + 1); };  // S[hl + 16][hl + 16]: base of the hi rounds
  const bool pad_lane = hl + 16 >= P;

  for (; __any_sync(0xffffffffu, active); ) {
    const int q = i < m ? (int)i : m;
    const bool real_lo = s_lo >= 0, real_hi = s_hi >= 0;
    const double yl = y_lo, yh = y_hi;
    const double2 my_lo = make_double2(c_lo.x * sc, c_lo.y * sc), my_hi = make_double2(c_hi.x * sc, c_hi.y * sc);
    if (real_lo) { pts2[hl] = my_lo; pts2[hl + P] = my_lo; }
    if (real_hi) pts2[hl + 16] = my_hi;
    // which point slots of my half are real (bit s): slots 0..q-1 and slot MT
    const unsigned blo = __ballot_sync(0xffffffffu, real_lo), bhi = __ballot_sync(0xffffffffu, real_hi);
    const unsigned real_mask = ((blo >> hbase) & 0xffffu) | (((bhi >> hbase) & 0xffffu) << 16);
    // no dummy slots anywhere in the warp (supplied neighbour sets may pad rows i >= m with -1 too)
    const bool full = (__all_sync(0xffffffffu, real_mask == (1u << P) - 1u || !active)) != 0;
    // bit t: the pair of round t (lo / hi) is kept; dummy slots are zeroed unless the whole warp is free of them
    const unsigned long long real2 = (unsigned long long)real_mask | ((unsigned long long)real_mask << P);
    const unsigned keep_lo = full ? ~0u : (real_lo ? real_mask >> hl : 0u);
    const unsigned keep_hi = full ? ~0u : (real_hi ? (unsigned)(real2 >> (hl + 16)) : 0u);
    const bool was_active = active;
    // next pair
    const int64_t it_n = it + nwarps;
    const int64_t i_n = row_of(it_n);
    const bool active_n = i_n < p.row_end;
    __syncwarp();

    // The rounds run in groups of G: the G values stay in registers until the group's rounds are done, then they are stored — a
    // store between two point loads would order the second load behind it (same address space, run-time indices) and serialise the
    // rounds' dependent FP64 chains (the state of the first version of this kernel).
    constexpr int NR = 2 * (MT / 2);
    constexpr int G = 6;
    static_assert(NR % G == 0, "group size must divide the number of rounds");
    double gp[(GRAD && !GP_SMEM) ? NR : 1];
#pragma unroll
    for (int r0 = 0; r0 < NR; r0 += G) {
      double val[G], gval[(GRAD && GP_SMEM) ? G : 1];
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int r = r0 + j;
        const int t = (r >> 1) + 1;
        const bool odd = (r & 1) != 0;
        const double2 po = pts2[hl + (odd ? 16 : 0) + t];
        const double2 me = odd ? my_hi : my_lo;
        const double dx = me.x - po.x, dy = me.y - po.y;
        const double d2s = fma(dy, dy, fma(dx, dx, 1e-300));
        double g = 0.;
        val[j] = cov_eval_scaled<COV, GRAD>(d2s, var, logvar, tab, g);
        if (GRAD) { if (GP_SMEM) gval[j] = g; else gp[r] = g; }
      }
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const int r = r0 + j;
        const int t = (r >> 1) + 1;
        const bool odd = (r & 1) != 0;
        const bool keep = (((odd ? keep_hi : keep_lo) >> t) & 1u) != 0u;  // no branches
        const double v = keep ? val[j] : 0.;
        // derivative value: 0 for padded / dummy pairs; pair (a, b), a < b -> column b, row a
        if (!odd) {
          Sd()[t] = v;
          if (GRAD) { if (GP_SMEM) Sd()[t * kLd] = keep ? gval[j] : 0.; else gp[r] = keep ? gp[r] : 0.; }
        } else {
          const bool wrap = hl + 16 + t >= P;
          if (!pad_lane) {
            if (wrap) Sh()[(t - P) * kLd] = v; else Sh()[t] = v;
            if (GRAD && GP_SMEM) { if (wrap) Sh()[t - P] = keep ? gval[j] : 0.; else Sh()[t * kLd] = keep ? gval[j] : 0.; }
          }
          if (GRAD && !GP_SMEM) gp[r] = (keep && !pad_lane) ? gp[r] : 0.;
        }
      }
    }
    // prefetch: data of the next pair (its indices arrived during the previous iteration), indices of the pair after it
    s_lo = sn_lo; s_hi = sn_hi;
    fetch_data();
    {
      const int64_t i_n2 = row_of(it_n + nwarps);
      fetch_idx(i_n2, i_n2 < p.row_end, sn_lo, sn_hi);
    }
    // diagonal and response row (row 31): S[c][c], S[c][31] = y_c for c <= 30
    S[hl * kLd + hl] = real_lo ? p.diag_nb : 1.;
    S[hl * kLd + (MT + 1)] = yl;
    if (hl + 16 <= MT) {
      S[(hl + 16) * kLd + (hl + 16)] = real_hi ? (hl + 16 == MT ? p.diag_obs : p.diag_nb) : 1.;
      S[(hl + 16) * kLd + (MT + 1)] = yh;
    }
    __syncwarp();

    // ---- my two rows of the lower triangle -> registers (entries above the diagonal: don't-care values)
    double lo[16], hi[MT + 1];
#pragma unroll
    for (int c = 0; c < 16; ++c) lo[c] = S[c * kLd + hl];
#pragma unroll
    for (int c = 0; c <= MT; ++c) hi[c] = S[c * kLd + hl + 16];
    __syncwarp();

    // ---- right-looking Cholesky with look-ahead, pivots 0..MT
    double Di, lk_lo, lk_hi;
    double dg_lo = S[hl * kLd + hl], dg_hi = S[(hl + 16) * kLd + hl + 16];  // my diagonals (row 31 has none: never a pivot)
    {
      const double d0 = __shfl_sync(0xffffffffu, lo[0], hbase);
      const double r0 = rsqrt_fast(d0);
      lk_lo = lo[0] * r0; lk_hi = hi[0] * r0;
      S[hl] = lk_lo; S[hl + 16] = lk_hi;
      Di = d0;
    }
    __syncwarp();
#pragma unroll
    for (int k = 0; k < MT; ++k) {
      // column k of L is visible in shared memory; lk_* = L[my rows][k].
      // Pivot chain of column k+1 first, from registers only: every lane keeps the diagonal entries of its own two rows up to date
      // with its own column values (a[r][r] -= L[r][k]^2 needs nothing from the other lanes), so the next pivot is one DFMA and a
      // shuffle away from lk — no shared-memory round trip on the chain that serialises the 31 steps
      dg_lo = fma(-lk_lo, lk_lo, dg_lo);
      dg_hi = fma(-lk_hi, lk_hi, dg_hi);
      const double dn = (k + 1 < 16) ? __shfl_sync(0xffffffffu, dg_lo, hbase + k + 1) : __shfl_sync(0xffffffffu, dg_hi, hbase + k + 1 - 16);
      {
        const double m1 = S[k * kLd + k + 1];
        hi[k + 1] -= lk_hi * m1;
        if (k + 1 < 16) lo[k + 1] -= lk_lo * m1;
      }
      if (k + 1 == MT) Di = dn;
      const double rn = rsqrt_fast(dn);
      const double lk1_lo = (k + 1 < 16) ? lo[k + 1] * rn : 0.;
      const double lk1_hi = hi[k + 1] * rn;
      // remaining rank-1 updates of step k: columns k+2..MT (pairs; the pair load may touch column MT+1: harmless)
#pragma unroll
      for (int c = k + 2; c <= MT; c += 2) {
        const double2 l2 = *reinterpret_cast<const double2*>(&S[k * kLd + c]);
        hi[c] -= lk_hi * l2.x;
        if (c + 1 <= MT) hi[c + 1] -= lk_hi * l2.y;
        if (c < 16) lo[c] -= lk_lo * l2.x;
        if (c + 1 < 16) lo[c + 1] -= lk_lo * l2.y;
      }
      // column k+1 goes out LAST: a store in front of the loads above would order them behind it (run-time row index: the compiler
      // cannot tell the two columns apart), i.e. behind the whole pivot chain — with it the next step's pivot would wait for
      // store -> load -> update of column k+2 instead of running from registers
      // (rows above the diagonal are not stored: in the gradient pass those slots hold the derivative values)
      if (k + 1 < 16 && (!(GRAD && GP_SMEM) || hl >= k + 1)) S[(k + 1) * kLd + hl] = lk1_lo;
      if (!(GRAD && GP_SMEM) || k + 1 <= 16 || hl + 16 >= k + 1) S[(k + 1) * kLd + hl + 16] = lk1_hi;
      __syncwarp();
      lk_lo = lk1_lo; lk_hi = lk1_hi;
    }
    // lane hl = 15 (row 31) wrote L[31][30] = (By)_i / sqrt(D_i) into column 30
    const double r_over_sd = S[MT * kLd + (MT + 1)];
    if (hl == 0 && was_active) {
      acc0 += r_over_sd * r_over_sd;
      acc1 += log(Di);
      acc2 += !(Di > 0.) ? 1. : 0.;
    }
    if (SOLVE) {
      // ---- back substitution L_NN^T x = L[30][.] (-> A_i) and L_NN^T x = L[31][.] (-> w = S^-1 y_N): lane hl owns unknowns hl, hl + 16
      const bool has_hi = hl + 16 < MT;
      double xa_lo = S[hl * kLd + MT], xw_lo = GRAD ? S[hl * kLd + (MT + 1)] : 0.;
      double xa_hi = has_hi ? S[(hl + 16) * kLd + MT] : 0., xw_hi = (GRAD && has_hi) ? S[(hl + 16) * kLd + (MT + 1)] : 0.;
      const double dinv_lo = 1. / S[hl * kLd + hl];
      const double dinv_hi = has_hi ? 1. / S[(hl + 16) * kLd + hl + 16] : 0.;
#pragma unroll
      for (int r = MT - 1; r >= 0; --r) {
        double fa, fw = 0.;
        if (r < 16) {
          fa = __shfl_sync(0xffffffffu, xa_lo * dinv_lo, hbase + r);
          if (GRAD) fw = __shfl_sync(0xffffffffu, xw_lo * dinv_lo, hbase + r);
          if (hl == r) { xa_lo = fa; xw_lo = fw; }
        } else {
          fa = __shfl_sync(0xffffffffu, xa_hi * dinv_hi, hbase + r - 16);
          if (GRAD) fw = __shfl_sync(0xffffffffu, xw_hi * dinv_hi, hbase + r - 16);
          if (hl + 16 == r) { xa_hi = fa; xw_hi = fw; }
        }
        const double l_lo = hl < r ? S[hl * kLd + r] : 0.;             // L[r][hl]
        xa_lo -= l_lo * fa; xw_lo -= l_lo * fw;
        if (r > 16) {  // unknowns hl + 16 only couple to rows r > hl + 16 >= 16
          const double l_hi = (has_hi && hl + 16 < r) ? S[(hl + 16) * kLd + r] : 0.;  // L[r][hl+16]
          xa_hi -= l_hi * fa; xw_hi -= l_hi * fw;
        }
      }
      // (the gradient pass writes the factor as well when the store buffers exist: the GPBoost iteration asks for it right after)
      if ((MODE == MODE_STORE || (GRAD && p.A != nullptr)) && was_active) {
        if (hl < m) p.A[i * m + hl] = hl < q ? xa_lo : 0.;
        if (hl + 16 < m) p.A[i * m + hl + 16] = hl + 16 < q ? xa_hi : 0.;
        if (hl == 0) { const double Dinv_i = 1. / Di; p.Dinv[i] = Dinv_i; p.w[i] = r_over_sd * sqrt(Di) * Dinv_i; }
      }
      if (GRAD) {
      // b = [-A, 1], w~ = [w, 0] over the 31 points, exchanged through the point buffer (free after the pair phase)
      __syncwarp();
      double* xb = pts;
      double* xwt = pts + 32;
      xb[hl] = -xa_lo; xwt[hl] = xw_lo;
      if (hl + 16 <= MT) { xb[hl + 16] = has_hi ? -xa_hi : 1.; xwt[hl + 16] = has_hi ? xw_hi : 0.; }
      __syncwarp();
      const double b_lo = xb[hl], w_lo = xwt[hl];
      const double b_hi = hl + 16 <= MT ? xb[hl + 16] : 0., w_hi = hl + 16 <= MT ? xwt[hl + 16] : 0.;
      double bgb = 0., bgw = 0.;
#pragma unroll
      for (int r = 0; r < 2 * (MT / 2); ++r) {
        const int t = (r >> 1) + 1;
        const bool odd = (r & 1) != 0;
        const int pi = hl + (odd ? 16 : 0);
        int o = pi + t;
        if (o >= P) o -= P;
        if (pi >= P) o = 0;
        const double g = GP_SMEM ? ((pi < P) ? S[max(pi, o) * kLd + min(pi, o)] : 0.) : gp[r];  // 0 for padded / inactive pairs
        const double bo = xb[o], wo = xwt[o];
        const double bm = odd ? b_hi : b_lo, wm = odd ? w_hi : w_lo;
        bgb += g * (bm * bo);
        bgw += g * (bm * wo + bo * wm);
      }
      double aa = xa_lo * xa_lo + xa_hi * xa_hi, aw = xa_lo * xw_lo + xa_hi * xw_hi;  // dummy unknowns are exactly 0
#pragma unroll
      for (int ofs = 8; ofs > 0; ofs >>= 1) {
        bgb += __shfl_xor_sync(0xffffffffu, bgb, ofs);
        bgw += __shfl_xor_sync(0xffffffffu, bgw, ofs);
        aa += __shfl_xor_sync(0xffffffffu, aa, ofs);
        aw += __shfl_xor_sync(0xffffffffu, aw, ofs);
      }
      if (hl == 0 && was_active) {
        const double Dinv_i = 1. / Di;
        const double u = r_over_sd * sqrt(Di) * Dinv_i;  // (D^-1 B y)_i
        const double dD0 = var - aa - (1. + var - Di);   // Vecchia_utils.cpp:1623
        const double dD1 = 2. * bgb;
        accg[0] += -aw * u;
        accg[1] += -bgw * u;
        accg[2] += u * u * dD0;
        accg[3] += u * u * dD1;
        accg[4] += dD0 * Dinv_i;
        accg[5] += dD1 * Dinv_i;
      }
      }  // GRAD
    }    // SOLVE
    __syncwarp();
    it = it_n; i = i_n; active = active_n;
  }
  if (hl == 0) {
    double* out = p.partials + (size_t)(gwarp * 2 + hh) * kNumAcc;
    out[0] = acc0; out[1] = acc1; out[2] = acc2;
#pragma unroll
    for (int k = 3; k < kNumAcc; ++k) out[k] = GRAD ? accg[k - 3] : 0.;
  }
}

}  // namespace gpb
