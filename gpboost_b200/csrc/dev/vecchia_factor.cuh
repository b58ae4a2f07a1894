// Vecchia factor kernel for sm_90a — one warp per observation, matrix rows in registers.
//
// Replaces the reference's per-observation loop in CalcCovFactorGradientVecchia
// (src/GPBoost/Vecchia_utils.cpp:1461-1684) together with the covariance-block construction it calls
// (include/GPBoost/re_comp.h:1476-1503 -> cov_fcts.h:635-755, gradients cov_fcts.h:1073-1218) and, fused
// behind it, the reductions the Gaussian likelihood and its gradient need
// (re_model_template.h:9957-9964 quad form, :2947 log-det, :1988-2010 gradient).
//
// Formulation (not a translation of the reference's Eigen code):
//   * points 0..q-1 = neighbours N(i), point q = observation i itself. The (q+2) x (q+2) matrix
//         [ S     s     y_N ]      S = Sigma_NN + I (nugget 1 on the transformed scale)
//         [ s^T   1+v   y_i ]      s = Sigma_iN,  v = sigma_1^2 / sigma^2
//         [ y_N^T y_i    *  ]
//     is factorised by ONE right-looking Cholesky with lane j owning row j (registers a[0..31]).
//     Then  D_i = pivot q before the square root,  z = L[q][0..q) = L_NN^-1 s,
//           L[q+1][q] = (B y)_i / sqrt(D_i)   =>  (By)_i^2 / D_i = L[q+1][q]^2 :
//     the likelihood needs NO triangular solve and B is never materialised.
//   * distances are recomputed from gathered coordinates (the reference keeps 7.2 GB of saved
//     neighbour distances at n=1e6); the 465 pair covariances are evaluated with a balanced circulant
//     schedule (lane l handles pairs (l, l+t mod P)) and staged through shared memory, which then
//     doubles as the column store of L (stride 33 doubles: conflict-free row loads, broadcasts and
//     transposed reads).
//   * A_i = L_NN^-T z (and w = S^-1 y_N in gradient mode) by a lane-per-unknown back substitution
//     reading L by columns from shared memory.
//   * the kernel is specialised on a compile-time neighbour capacity MT in {10, 20, 30}: a model with m <= MT
//     neighbours (and the first rows, which have fewer than m predecessors) is padded with "dummy" points that
//     are uncorrelated with everything (unit diagonal, zero off-diagonal, zero response); the padded
//     factorisation reproduces the un-padded one exactly. All loops are then fully unrolled without runtime
//     predicates and the Cholesky is software-pipelined (look-ahead): the pivot chain of column k+1
//     (shuffle -> rsqrt -> scale -> shared store) is issued right after column k+1 received its update and
//     overlaps with the remaining rank-1 updates of step k.
//   * gradient mode uses the adjoint identities  dD_k = b^T dSigma~_k b,  (dB_k y)_i = -b^T dSigma~_k w~
//     with b = [-A_i, 1], w~ = [w, 0]: no derivative matrix is factorised or stored; the range-derivative
//     pair values stay in the registers of the lane that computed them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gpb {

enum CovType : int { COV_EXPONENTIAL = 0, COV_MATERN15 = 1, COV_MATERN25 = 2, COV_GAUSSIAN = 3 };
// MODE_STORE_GRAD: MODE_STORE plus the derivative of the factor w.r.t. log(range): dA_i (= -B_grad row) and dD_i, what
// CalcCovFactorGradientVecchia leaves in B_grad[1], D_grad[1] (Vecchia_utils.cpp:1636-1652) — needed where the derivative of
// Sigma^-1 is applied to many vectors (Laplace-approximated likelihoods, likelihoods.h:6615-6690).
// MODE_STORE_GRAD2: the Gaussian (nugget) model's MODE_STORE plus the derivatives of the factor w.r.t. log(var) AND log(range)
// on the transformed scale, what CalcCovFactorGradientVecchia leaves in B_grad[0..1], D_grad[0..1] — the Fisher information of
// the covariance parameters (re_model_template.h:10145-10230) applies them to a block of probe vectors.
// MODE_GRAD_ANISO: the gradient of an anisotropic kernel (ARD / space-time) evaluated on scaled coordinates at range 1: one
// log-range derivative per coordinate group c instead of one in total. With r^2 the squared scaled distance of a pair and S_c the
// part of r^2 from the coordinates of group c, dk/dlog(lambda_c) = (dk/dlog(lambda))_iso(r) * S_c / r^2 (0 at r = 0): every pair's
// isotropic derivative is computed once, as in MODE_GRAD, and split by coordinate share inside the adjoint contractions.
// Sums go to a kAnisoAcc-wide partial row (see there); the coordinate groups are g_aniso_ngroups / g_aniso_mask.
enum FactorMode : int { MODE_NLL = 0, MODE_STORE = 1, MODE_GRAD = 2, MODE_STORE_GRAD = 3, MODE_STORE_GRAD2 = 4, MODE_GRAD_ANISO = 5 };

#ifndef GPB_NLL_BLOCKS
#define GPB_NLL_BLOCKS 5
#endif
#ifndef GPB_GRAD_BLOCKS
#define GPB_GRAD_BLOCKS 3
#endif
constexpr int kWarpsPerBlock = 4;
constexpr int kLd = 33;            // column stride (doubles) of the shared matrix
constexpr int kMaxNeighbors = 30;  // q + 2 rows must fit one warp
// per-warp accumulators: 0 sum (By)^2/D  1 sum log D  2 #non-positive D
//   gradient mode: 3,4 sum u_k u   5,6 sum u^2 dD_k   7,8 sum dD_k / D   (k = 0 variance, 1 range)
constexpr int kNumAcc = 9;
// MODE_GRAD_ANISO per-warp sums: 0..2 as above, then for k = 0 (variance) and k = 1..C (range of coordinate group k - 1)
// 3 + 3k: sum u_k u   4 + 3k: sum u^2 dD_k   5 + 3k: sum dD_k / D. Lane k of the warp owns the three sums of parameter k.
constexpr int kMaxAnisoGroups = 16;
constexpr int kAnisoAcc = 3 + 3 * (1 + kMaxAnisoGroups);

struct FactorArgs {
  const double* coords;   // n x d row-major, Vecchia order
  const int32_t* nn;      // n x m, -1 padded
  const double* y;        // n, Vecchia order
  double* A;              // n x m  (MODE_STORE): A_i, i.e. -B[i, nn]
  double* Dinv;           // n      (MODE_STORE)
  double* w;              // n      (MODE_STORE): D^-1 (B y)
  double* partials;       // num_warps_total x kNumAcc
  int64_t n;
  int64_t row_begin, row_end;  // shard of observations handled by this launch
  int m;
  int d;
  double var;     // sigma_1^2 / sigma^2
  double range;   // transformed range (cov_fcts.h:485-552)
  // diagonal of the covariance block: Gaussian likelihood (transformed scale) var + 1 for both; latent GP of a
  // non-Gaussian likelihood: neighbours var * JITTER_MULT_VECCHIA, the observation itself var
  // (Vecchia_utils.cpp:1411-1417, 1555-1563, 1599-1609)
  double diag_nb;
  double diag_obs;
};
// Outputs of MODE_STORE_GRAD (d A_i / d log(range): n x m, d D_i / d log(range): n). Kept out of FactorArgs so that the
// parameter block — and with it the generated code — of the other modes is exactly what the committed ncu captures describe;
// set with cudaMemcpyToSymbolAsync on the engine's stream right before the launch (one engine per device at a time).
__device__ double* g_factor_dA = nullptr;
__device__ double* g_factor_dD = nullptr;
// MODE_STORE_GRAD2 only: d A_i / d log(var) (n x m) and d D_i / d log(var) (n); the range pair goes to g_factor_dA / g_factor_dD
__device__ double* g_factor_dA0 = nullptr;
__device__ double* g_factor_dD0 = nullptr;
// MODE_GRAD_ANISO (and BIG_GRAD_ANISO): number of coordinate groups and, per group, the bit mask of its coordinates
__constant__ int g_aniso_ngroups;
__constant__ unsigned g_aniso_mask[kMaxAnisoGroups];

// squared distance of points a and b (rows of pts, stride dim) restricted to the coordinates in mask
__device__ __forceinline__ double masked_d2(const double* pa, const double* pb, int dim, unsigned mask) {
  double s = 0.;
  for (int k = 0; k < dim; ++k) {
    if ((mask >> k) & 1u) {
      const double df = pa[k] - pb[k];
      s = fma(df, df, s);
    }
  }
  return s;
}

// exp(ax) for ax <= 0 (clamped at -700): round-to-nearest range reduction by the 1.5*2^52 trick, degree-13 Taylor
// polynomial on |r| <= ln2/2 (truncation error 4e-18), scaling by an exponent-field add. No special-case paths and the
// coefficients are constant-bank operands of the DFMAs — about half the instructions of the library exp().
__constant__ double kExpC[12] = {1. / 6227020800., 1. / 479001600., 1. / 39916800., 1. / 3628800., 1. / 362880., 1. / 40320.,
                                 1. / 5040.,       1. / 720.,       1. / 120.,      1. / 24.,      1. / 6.,      0.5};
__device__ __forceinline__ double exp_neg(double ax) {
  ax = ax < -700. ? -700. : ax;
  const double t = fma(ax, 1.4426950408889634074, 6755399441055744.0);
  const double n = t - 6755399441055744.0;
  double r = fma(n, -6.93147180369123816490e-01, ax);
  r = fma(n, -1.90821492927058770002e-10, r);
  double pl = kExpC[0];
#pragma unroll
  for (int k = 1; k < 12; ++k) pl = fma(pl, r, kExpC[k]);
  pl = fma(pl, r, 1.0);
  pl = fma(pl, r, 1.0);
  const int hi = __double2hiint(pl) + (__double2loint(t) << 20);
  return __hiloint2double(hi, __double2loint(pl));
}

// covariance value and d/dlog(range) on the transformed scale — closed forms cov_fcts.h:2100-2118,2154;
// gradient constants cov_fcts.h:2183-2206, element formulas :2535-2563.
template <int COV, bool GRAD>
__device__ __forceinline__ double cov_eval(double dist, double var, double range, double& grad) {
  double val;
  if (COV == COV_EXPONENTIAL) {
    val = var * exp_neg(-range * dist);
    if (GRAD) grad = -range * dist * val;
  } else if (COV == COV_MATERN15) {
    const double rd = range * dist;
    const double e = exp_neg(-rd);
    val = var * (1. + rd) * e;
    if (GRAD) grad = -var * range * range * dist * dist * e;
  } else if (COV == COV_MATERN25) {
    const double rd = range * dist;
    const double e = exp_neg(-rd);
    val = var * (1. + rd + rd * rd / 3.) * e;
    if (GRAD) grad = -var * range * range / 3. * dist * dist * (1. + rd) * e;
  } else {
    val = var * exp_neg(-range * dist * dist);
    if (GRAD) grad = -range * dist * dist * val;
  }
  return val;
}

// 1/sqrt(x) for x > 0: MUFU.RSQ64H seed + one third-order correction (relative error ~1e-16); no special-case
// handling (pivots are >= the nugget, squared distances are guarded by the caller).
__device__ __forceinline__ double rsqrt_fast(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double e = fma(-x * y, y, 1.0);                // 1 - x y^2
  return fma(y * e, fma(0.375, e, 0.5), y);            // y (1 + e/2 + 3 e^2 / 8)
}

__device__ __forceinline__ double shfl_d(double x, int src) { return __shfl_sync(0xffffffffu, x, src); }
__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

template <int COV, int MODE, int DIM, int MT>
__global__ void __launch_bounds__(kWarpsPerBlock * 32,
                                  MODE == MODE_GRAD_ANISO ? 2  // the per-group contractions need more registers than three CTAs leave
                                  : (MODE == MODE_GRAD || MODE == MODE_STORE_GRAD || MODE == MODE_STORE_GRAD2) ? GPB_GRAD_BLOCKS
                                                                                                               : GPB_NLL_BLOCKS)
vecchia_factor_kernel(const FactorArgs p) {
  constexpr bool ANISO = (MODE == MODE_GRAD_ANISO);
  constexpr bool GRAD = (MODE == MODE_GRAD) || ANISO;
  constexpr bool DSTORE = (MODE == MODE_STORE_GRAD) || (MODE == MODE_STORE_GRAD2);  // the range derivative is stored
  constexpr bool GPAIR = GRAD || DSTORE;  // the range-derivative pair values are kept
  constexpr bool SOLVE = (MODE != MODE_NLL);
  constexpr int P = MT + 1;      // point slots: 0..MT-1 neighbours (real or dummy), MT = the observation
  constexpr int NT = MT / 2;     // circulant rounds (P is odd)
  static_assert(MT % 2 == 0 && MT >= 2 && MT <= kMaxNeighbors, "MT must be even and <= 30");
  extern __shared__ __align__(16) double smem_raw[];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int dim = DIM > 0 ? DIM : p.d;
  // per-warp shared layout: L/S matrix 32 x kLd | points 32 x dim | xb 32 | xw 32
  const int per_warp = 32 * kLd + 32 * dim + 64;
  double* S = smem_raw + (size_t)wib * per_warp;
  double* pts = S + 32 * kLd;
  double* xb = pts + 32 * dim;
  double* xw = xb + 32;

  const int64_t gwarp = (int64_t)blockIdx.x * kWarpsPerBlock + wib;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  const int m = p.m;
  const double var = p.var, range = p.range;

  double acc[kNumAcc];
#pragma unroll
  for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.;
  double acc_an[3] = {0., 0., 0.};  // MODE_GRAD_ANISO: the sums of parameter `lane`

  // slot -> source observation of row ii (or -1 for a dummy slot)
  auto slot_src = [&](int64_t ii) -> int64_t {
    const int qq = ii < m ? (int)ii : m;  // Vecchia_utils.cpp:788-813: the first m+1 points condition on all predecessors
    if (lane < qq) return (int64_t)p.nn[ii * m + lane];
    return lane == MT ? ii : (int64_t)-1;
  };
  // software pipeline over observations (DIM == 2): the gather of row i + nwarps is issued while row i is computed
  int64_t src_pre = -1;
  double2 c_pre = make_double2(0., 0.);
  double y_pre = 0.;
  if (DIM == 2 && p.row_begin + gwarp < p.row_end) {
    src_pre = slot_src(p.row_begin + gwarp);
    if (src_pre >= 0) {
      y_pre = p.y[src_pre];
      c_pre = *reinterpret_cast<const double2*>(p.coords + src_pre * 2);
    }
  }

  for (int64_t i = p.row_begin + gwarp; i < p.row_end; i += nwarps) {
    // ---- gather: neighbour ids, coordinates, responses
    const int q = i < m ? (int)i : m;
    int64_t src;
    double yv = 0.;
    if (DIM == 2) {
      src = src_pre;
      yv = y_pre;
      if (src >= 0) *reinterpret_cast<double2*>(pts + lane * 2) = c_pre;
    } else {
      src = slot_src(i);
      if (src >= 0) {
        yv = p.y[src];
        for (int k = 0; k < dim; ++k) pts[lane * dim + k] = p.coords[src * dim + k];
      }
    }
    const bool real = src >= 0;  // slots q..MT-1 are dummies
    int64_t src_next = -1;
    if (DIM == 2 && i + nwarps < p.row_end) src_next = slot_src(i + nwarps);  // consumed after the pair phase
    const unsigned real_mask = __ballot_sync(0xffffffffu, real);
    __syncwarp();

    // ---- pair covariances, circulant schedule: lane l <-> point (l + t) mod P, t = 1..NT
    double gpair[GPAIR ? NT : 1];
    double my[DIM > 0 ? DIM : 1];
    if (DIM > 0) {
#pragma unroll
      for (int k = 0; k < (DIM > 0 ? DIM : 1); ++k) my[k] = pts[lane * dim + k];
    }
    // warp-uniform: no dummy slots (rows i >= m of a model with m == MT, unless supplied neighbour sets pad them with -1)
    const bool full = real_mask == (1u << P) - 1u;
#pragma unroll
    for (int t = 1; t <= NT; ++t) {
      int o = lane + t;
      if (o >= P) o -= P;
      if (lane >= P) o = 0;  // lane 31 computes a throw-away pair
      double d2 = 0.;
      if (DIM > 0) {
#pragma unroll
        for (int k = 0; k < (DIM > 0 ? DIM : 1); ++k) {
          const double df = my[k] - pts[o * dim + k];
          d2 = k == 0 ? df * df : fma(df, df, d2);
        }
      } else {
        for (int k = 0; k < dim; ++k) {
          const double df = pts[lane * dim + k] - pts[o * dim + k];
          d2 = fma(df, df, d2);
        }
      }
      // dist = d2 / sqrt(d2); the tiny offset makes coincident points come out as exactly 0 without a branch
      const double dist = d2 * rsqrt_fast(d2 + 1e-300);
      double g = 0.;
      double val = cov_eval<COV, GPAIR>(dist, var, range, g);
      if (ANISO) g = d2 > 0. ? g / d2 : 0.;  // split later by coordinate share: g_c = g S_c / r^2
      if (!full) {
        const bool both = real && ((real_mask >> o) & 1u);
        val = both ? val : 0.;
        g = both ? g : 0.;
      }
      if (lane < P) S[min(lane, o) * kLd + max(lane, o)] = val;
      if (GPAIR) gpair[t - 1] = (lane < P) ? g : 0.;
    }
    if (DIM == 2) {  // dependent gather of the next row; lands during the factorisation
      src_pre = src_next;
      y_pre = 0.;
      if (src_next >= 0) {
        y_pre = p.y[src_next];
        c_pre = *reinterpret_cast<const double2*>(p.coords + src_next * 2);
      }
    }
    // diagonal: variance + nugget 1 (Vecchia_utils.cpp:1601 / :1411,1563), 1 for dummies; response row MT+1
    if (lane < P) {
      S[lane * kLd + lane] = real ? (lane == MT ? p.diag_obs : p.diag_nb) : 1.;
      S[lane * kLd + (MT + 1)] = yv;
    }
    __syncwarp();

    // ---- row j of the lower triangle -> registers of lane j
    double a[MT + 2];
#pragma unroll
    for (int c = 0; c <= MT; ++c) a[c] = S[c * kLd + lane];
    a[MT + 1] = 0.;
    __syncwarp();

    // ---- right-looking Cholesky with look-ahead, pivots 0..MT (row MT+1 is eliminated but never a pivot)
    double Di;
    double lk;
    {
      const double d0 = shfl_d(a[0], 0);
      lk = a[0] * rsqrt_fast(d0);
      S[lane] = lk;  // column 0 of L (rows above the diagonal hold don't-care values)
      Di = d0;
    }
    __syncwarp();
#pragma unroll
    for (int k = 0; k < MT; ++k) {
      // column k of L is visible in shared memory; lk = L[lane][k]
      a[k + 1] -= lk * S[k * kLd + k + 1];
      // look-ahead: pivot chain of column k+1
      const double dn = shfl_d(a[k + 1], k + 1);
      if (k + 1 == MT) Di = dn;
      const double lk1 = a[k + 1] * rsqrt_fast(dn);
      S[(k + 1) * kLd + lane] = lk1;
      // remaining rank-1 updates of step k (columns k+2..MT; the pair load may touch column MT+1: harmless)
#pragma unroll
      for (int c = k + 2; c <= MT; c += 2) {
        const double2 l2 = *reinterpret_cast<const double2*>(&S[k * kLd + c]);
        a[c] -= lk * l2.x;
        a[c + 1] -= lk * l2.y;
      }
      __syncwarp();
      lk = lk1;
    }
    // lane MT+1 wrote L[MT+1][MT] = (By)_i / sqrt(D_i) into column MT
    const double r_over_sd = S[MT * kLd + (MT + 1)];
    const double quad = r_over_sd * r_over_sd;  // (By)_i^2 / D_i
    const bool bad = !(Di > 0.);
    if (lane == 0) {
      acc[0] += quad;
      acc[1] += log(Di);
      acc[2] += bad ? 1. : 0.;
    }

    if (SOLVE) {
      // ---- back substitution L_NN^T x = z for z = L[MT][.] (-> A_i) and, in gradient mode, L[MT+1][.] (-> w)
      // lane c owns unknown c; L[r][c] is read by columns: S[c*kLd + r]. Dummy unknowns come out as 0.
      double xa = (lane < MT) ? S[lane * kLd + MT] : 0.;
      double xwv = (GRAD && lane < MT) ? S[lane * kLd + (MT + 1)] : 0.;
      const double dinv = (lane < MT) ? 1. / S[lane * kLd + lane] : 0.;
#pragma unroll
      for (int r = MT - 1; r >= 0; --r) {
        const double fa = shfl_d(xa * dinv, r);
        double fw = 0.;
        if (GRAD) fw = shfl_d(xwv * dinv, r);
        const double lrc = (lane < r) ? S[lane * kLd + r] : 0.;
        if (lane == r) { xa = fa; if (GRAD) xwv = fw; }
        xa -= lrc * fa;
        if (GRAD) xwv -= lrc * fw;
      }
      // xa = A_i[lane] for lane < q
      const double Dinv_i = 1. / Di;
      const double By = r_over_sd * sqrt(Di);
      if (MODE == MODE_STORE || DSTORE) {
        if (lane < m) p.A[i * m + lane] = (lane < q) ? xa : 0.;
        if (lane == 0) { p.Dinv[i] = Dinv_i; p.w[i] = By * Dinv_i; }
      }
      if (DSTORE) {
        // r = dSigma~ b over the P points (b = [-A, 1]): rows 0..MT-1 of r are dSigma_iN - dSigma_NN A, and b.r = dD
        __syncwarp();
        xb[lane] = (lane < MT) ? -xa : (lane == MT ? 1. : 0.);
        __syncwarp();
        const double bl = xb[lane];
        double racc = 0.;
#pragma unroll
        for (int t = 1; t <= NT; ++t) {
          int o = lane + t;
          if (o >= P) o -= P;
          o = lane < P ? o : 0;
          const double g = gpair[t - 1];  // pair (lane, o); 0 for padded / inactive pairs
          racc += g * xb[o];
          int src = lane - t;             // the lane whose partner of round t is this lane
          if (src < 0) src += P;
          const double sent = shfl_d(g * bl, src);
          if (lane < P) racc += sent;
        }
        const double dDv = warp_sum(lane < P ? bl * racc : 0.);
        // dA = S^-1 r = L^-T L^-1 r: forward substitution with lane = row (L[row][c] = S[c * kLd + row]), then the same
        // back substitution as for A
        double xg = (lane < MT) ? racc : 0.;
#pragma unroll
        for (int j = 0; j < MT; ++j) {
          const double wj = shfl_d(xg * dinv, j);
          const double lij = (lane > j && lane < MT) ? S[j * kLd + lane] : 0.;
          if (lane == j) xg = wj;
          xg -= lij * wj;
        }
#pragma unroll
        for (int r = MT - 1; r >= 0; --r) {
          const double fa = shfl_d(xg * dinv, r);
          const double lrc = (lane < r) ? S[lane * kLd + r] : 0.;
          if (lane == r) xg = fa;
          xg -= lrc * fa;
        }
        if (lane < m) g_factor_dA[i * m + lane] = (lane < q) ? xg : 0.;
        if (lane == 0) g_factor_dD[i] = dDv;
      }
      if (MODE == MODE_STORE_GRAD2) {
        // log(var): dSigma~ = Sigma~ - I (the nugget does not move), so dA = S^-1 (s - (S - I) A) = S^-1 A and
        // dD = var - dA.s - A.s = D - 1 - A.A  (A.s = 1 + var - D; Vecchia_utils.cpp:1571, :1623, :1636-1652)
        double xv = (lane < MT) ? xa : 0.;
#pragma unroll
        for (int j = 0; j < MT; ++j) {
          const double wj = shfl_d(xv * dinv, j);
          const double lij = (lane > j && lane < MT) ? S[j * kLd + lane] : 0.;
          if (lane == j) xv = wj;
          xv -= lij * wj;
        }
#pragma unroll
        for (int r = MT - 1; r >= 0; --r) {
          const double fa = shfl_d(xv * dinv, r);
          const double lrc = (lane < r) ? S[lane * kLd + r] : 0.;
          if (lane == r) xv = fa;
          xv -= lrc * fa;
        }
        const double aa = warp_sum((lane < q) ? xa * xa : 0.);
        if (lane < m) g_factor_dA0[i * m + lane] = (lane < q) ? xv : 0.;
        if (lane == 0) g_factor_dD0[i] = Di - 1. - aa;
      }
      if (GRAD) {
        // b = [-A, 1], w~ = [w, 0] over the P points
        __syncwarp();
        xb[lane] = (lane < MT) ? -xa : (lane == MT ? 1. : 0.);
        xw[lane] = (lane < MT) ? xwv : 0.;
        __syncwarp();
        // adjoint contractions over this lane's pairs: b^T G b and b^T G w~ (G symmetric, zero diagonal)
        double bgb = 0., bgw = 0.;
        const double bl = xb[lane], wl = xw[lane];
        if (ANISO) {
          // per coordinate group c: the same contractions with g_c = (g / r^2) S_c; lane c + 1 keeps group c's results
          const int ng = g_aniso_ngroups;
          for (int c = 0; c < ng; ++c) {
            const unsigned mask = g_aniso_mask[c];
            double cgb = 0., cgw = 0.;
#pragma unroll
            for (int t = 1; t <= NT; ++t) {
              int o = lane + t;
              if (o >= P) o -= P;
              o = lane < P ? o : 0;
              const double gq = gpair[t - 1];  // g / r^2; 0 for padded / inactive / coincident pairs
              const double gc = gq != 0. ? gq * masked_d2(pts + lane * dim, pts + o * dim, dim, mask) : 0.;
              const double bo = xb[o], wo = xw[o];
              cgb += gc * (bl * bo);
              cgw += gc * (bl * wo + bo * wl);
            }
            cgb = 2. * warp_sum(cgb);
            cgw = warp_sum(cgw);
            if (lane == c + 1) { bgb = cgb; bgw = cgw; }
          }
        } else {
#pragma unroll
          for (int t = 1; t <= NT; ++t) {
            int o = lane + t;
            if (o >= P) o -= P;
            o = lane < P ? o : 0;
            const double g = gpair[t - 1];  // 0 for padded / inactive pairs
            const double bo = xb[o], wo = xw[o];
            bgb += g * (bl * bo);
            bgw += g * (bl * wo + bo * wl);
          }
          bgb = 2. * warp_sum(bgb);
          bgw = warp_sum(bgw);
        }
        // variance parameter (dSigma~ = Sigma~ without nugget): dD_0 = v - A.A - A.s ; (dB_0 y)_i = -A.w
        // A.s = 1 + v - D  (Vecchia_utils.cpp:1623)
        double aa = (lane < q) ? xa * xa : 0.;
        double aw = (lane < q) ? xa * xwv : 0.;
        aa = warp_sum(aa);
        aw = warp_sum(aw);
        if (ANISO) {
          const double u = By * Dinv_i;
          const double dDk = lane == 0 ? var - aa - (1. + var - Di) : bgb;
          const double ukk = lane == 0 ? -aw : -bgw;
          acc_an[0] += ukk * u;
          acc_an[1] += u * u * dDk;
          acc_an[2] += dDk * Dinv_i;
        } else if (lane == 0) {
          const double u = By * Dinv_i;  // (D^-1 B y)_i
          const double dD0 = var - aa - (1. + var - Di);
          const double dD1 = bgb;
          const double uk0 = -aw;
          const double uk1 = -bgw;
          acc[3] += uk0 * u;
          acc[4] += uk1 * u;
          acc[5] += u * u * dD0;
          acc[6] += u * u * dD1;
          acc[7] += dD0 * Dinv_i;
          acc[8] += dD1 * Dinv_i;
        }
      }
    }
    __syncwarp();
  }
  if (ANISO) {
    double* row = p.partials + gwarp * kAnisoAcc;
    if (lane == 0)
      for (int k = 0; k < 3; ++k) row[k] = acc[k];
    if (lane <= kMaxAnisoGroups)
      for (int k = 0; k < 3; ++k) row[3 + 3 * lane + k] = acc_an[k];
  } else if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kNumAcc; ++k) p.partials[gwarp * kNumAcc + k] = acc[k];
  }
}

}  // namespace gpb
