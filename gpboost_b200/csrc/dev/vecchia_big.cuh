// Vecchia factor kernel for neighbour sets of up to 60 points, and Vecchia prediction.
//
// vecchia_factor.cuh keeps one matrix row per lane in registers and is specialised on <= 30 neighbours (the headline
// configuration). This kernel serves what does not fit that layout, with the matrix in shared memory and runtime sizes:
//   * models with 30 < num_neighbors <= 60 (same modes NLL / STORE / GRAD, same 9 sums, same stored factor layout; BIG_GRAD_ANISO is
//     MODE_GRAD_ANISO of vecchia_factor.cuh with its kAnisoAcc sums);
//   * prediction (MODE_PRED): CalcPredVecchiaObservedFirstOrder with CondObsOnly = true (src/GPBoost/Vecchia_utils.cpp:1701-2100;
//     the reference predicts with 2 x num_neighbors neighbours, re_model_template.h:299): for a prediction point p with observed
//     neighbours N(p):  A_p = Sigma_NN^-1 Sigma_pN (:1960),  D_p = v - A_p . Sigma_pN (:1925-1931, :1969),  mean_p = A_p y_N (:2061),
//     var_p = D_p (:2074) on the transformed scale.
//
// Formulation (the same augmented matrix as the register kernel): points 0..q-1 = neighbours, point q = the row's own location,
// row q+1 = the responses. ONE right-looking Cholesky over pivots 0..q of
//       [ S     s     y_N ]
//       [ s^T   d_o   y_i ]        S = Sigma_NN + nugget,  s = Sigma_iN
//       [ y_N^T y_i    *  ]
// leaves D_i in pivot q, (B y)_i = y_i - A_i . y_N in entry (q+1, q) before its scaling, z = L_NN^-1 s in row q and L_NN^-1 y_N in
// row q+1. With y_i = 0 that entry is -A_p . y_N: the predictive mean needs no triangular solve at all.
// One warp per row; lane-strided loops over rows/columns, runtime q, no padding with dummy points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vecchia_factor.cuh"

namespace gpb {

constexpr int kBigMaxNeighbors = 60;
constexpr int kBigLd = 65;  // row stride (doubles) of the shared matrices: 64 + 1, conflict-free for lane = row and lane = column
enum BigMode : int { BIG_NLL = 0, BIG_STORE = 1, BIG_GRAD = 2, BIG_PRED = 3, BIG_GRAD_ANISO = 4 };

struct BigArgs {
  const double* coords;   // observed points, n_obs x d row-major, Vecchia order
  const double* y;        // n_obs, Vecchia order
  const int32_t* nn;      // rows x m neighbour ids (observed points), -1 padded
  const double* qcoords;  // BIG_PRED: query coordinates, rows x d; otherwise null (row i is observed point i)
  double* A;              // BIG_STORE: rows x m
  double* Dinv;           // BIG_STORE: rows
  double* w;              // BIG_STORE: rows, D^-1 (B y)
  double* pred_mean;      // BIG_PRED: rows
  double* pred_var;       // BIG_PRED: rows (D_p, transformed scale)
  double* partials;       // warps x kNumAcc
  int64_t row_begin, row_end;
  int m, d;
  double var, range, diag_nb, diag_obs;
};

static inline size_t big_smem_bytes(int mode, int warps, int d) {
  const size_t per_warp = (size_t)(mode == BIG_GRAD || mode == BIG_GRAD_ANISO ? 2 : 1) * 64 * kBigLd + 64 * d + 4 * 64;
  return per_warp * warps * sizeof(double);
}

template <int COV, int MODE>
__global__ void __launch_bounds__(128) vecchia_big_kernel(const BigArgs p) {
  constexpr bool ANISO = MODE == BIG_GRAD_ANISO;
  constexpr bool GRAD = MODE == BIG_GRAD || ANISO;
  extern __shared__ __align__(16) double big_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nwib = blockDim.x >> 5;
  const int d = p.d, m = p.m;
  const size_t per_warp = (size_t)(GRAD ? 2 : 1) * 64 * kBigLd + 64 * d + 4 * 64;
  double* S = big_smem + (size_t)wib * per_warp;     // (q+2) x (q+2) lower triangle, row-major stride kBigLd
  double* G = S + 64 * kBigLd;                       // GRAD: range derivative of the covariances, rows 0..q
  double* pts = S + (size_t)(GRAD ? 2 : 1) * 64 * kBigLd;
  double* xa = pts + 64 * d;                         // A (back substitution), then b = [-A, 1]
  double* xw = xa + 64;                              // S^-1 y_N, then w~ = [w, 0]
  double* dg = xw + 64;                              // 1 / L[r][r]
  const int64_t gwarp = (int64_t)blockIdx.x * nwib + wib, nwarps = (int64_t)gridDim.x * nwib;
  const double var = p.var, range = p.range;
  double acc[kNumAcc];
#pragma unroll
  for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.;
  double acc_an[3] = {0., 0., 0.};  // BIG_GRAD_ANISO: the sums of parameter `lane` (vecchia_factor.cuh, kAnisoAcc)

  for (int64_t i = p.row_begin + gwarp; i < p.row_end; i += nwarps) {
    // ---- gather: neighbours (valid entries of a row are a prefix), own location, responses into row q+1
    int q = 0;
    for (int k = lane; k < m; k += 32) {
      const int32_t src = p.nn[i * m + k];
      if (src >= 0) {
        for (int c = 0; c < d; ++c) pts[k * d + c] = p.coords[(int64_t)src * d + c];
        xw[k] = p.y[src];
      }
      q += src >= 0 ? 1 : 0;
    }
    q = (int)warp_sum((double)q);
    if (lane == 0) {
      const double* own = MODE == BIG_PRED ? p.qcoords + i * d : p.coords + i * d;
      for (int c = 0; c < d; ++c) pts[q * d + c] = own[c];
    }
    const double yi = MODE == BIG_PRED ? 0. : p.y[i];
    __syncwarp();
    // ---- covariances: rows r = 0..q (row q = the row's own point), columns c < r; diagonal; response row
    for (int r = 1; r <= q; ++r) {
      for (int c = lane; c < r; c += 32) {
        double d2 = 0.;
        for (int e = 0; e < d; ++e) { const double df = pts[r * d + e] - pts[c * d + e]; d2 = fma(df, df, d2); }
        double g = 0.;
        const double val = cov_eval<COV, GRAD>(sqrt(d2), var, range, g);
        S[r * kBigLd + c] = val;
        if (GRAD) G[r * kBigLd + c] = ANISO ? (d2 > 0. ? g / d2 : 0.) : g;  // ANISO: g / r^2, split by coordinate share below
      }
    }
    for (int r = lane; r <= q; r += 32) {
      S[r * kBigLd + r] = r == q ? p.diag_obs : p.diag_nb;
      S[(q + 1) * kBigLd + r] = r == q ? yi : xw[r];
    }
    __syncwarp();
    // ---- right-looking Cholesky, pivots 0..q over rows 0..q+1
    const int R = q + 2;
    double Di = 0., By = 0.;
    for (int k = 0; k <= q; ++k) {
      const double piv = S[k * kBigLd + k];
      if (k == q) { Di = piv; By = S[(q + 1) * kBigLd + q]; }
      const double rinv = 1. / sqrt(piv);
      __syncwarp();  // every lane holds the pivot (and, at k = q, the unscaled response entry) before the column is scaled
      if (lane == 0) dg[k] = rinv;  // L[k][k] itself is never read again
      for (int r = k + 1 + lane; r < R; r += 32) S[r * kBigLd + k] *= rinv;
      __syncwarp();
      // trailing update: lane owns rows r = k+1+lane, k+33+lane; columns k+1..min(r, q)
      for (int r = k + 1 + lane; r < R; r += 32) {
        const double lrk = S[r * kBigLd + k];
        const int cend = min(r, q);
        for (int c = k + 1; c <= cend; ++c) S[r * kBigLd + c] -= lrk * S[c * kBigLd + k];
      }
      __syncwarp();
    }
    const double Dinv_i = 1. / Di;
    const bool bad = !(Di > 0.);
    if (MODE == BIG_PRED) {
      if (lane == 0) { p.pred_mean[i] = -By; p.pred_var[i] = Di; }
      __syncwarp();
      continue;
    }
    if (lane == 0) {
      acc[0] += By * By * Dinv_i;
      acc[1] += log(Di);
      acc[2] += bad ? 1. : 0.;
    }
    if (MODE == BIG_NLL) { __syncwarp(); continue; }
    // ---- back substitution L_NN^T x = z (row q -> A_i) and, for the gradient, L_NN^T x = L_NN^-1 y_N (row q+1 -> w = S^-1 y_N)
    for (int c = lane; c < q; c += 32) { xa[c] = S[q * kBigLd + c]; xw[c] = S[(q + 1) * kBigLd + c]; }
    __syncwarp();
    for (int r = q - 1; r >= 0; --r) {
      const double fa = xa[r] * dg[r], fw = xw[r] * dg[r];
      __syncwarp();
      if (lane == 0) { xa[r] = fa; xw[r] = fw; }
      for (int c = lane; c < r; c += 32) {
        const double lrc = S[r * kBigLd + c];
        xa[c] -= lrc * fa;
        xw[c] -= lrc * fw;
      }
      __syncwarp();
    }
    if (MODE == BIG_STORE) {
      for (int k = lane; k < m; k += 32) p.A[i * m + k] = k < q ? xa[k] : 0.;
      if (lane == 0) { p.Dinv[i] = Dinv_i; p.w[i] = By * Dinv_i; }
    }
    if (GRAD) {
      // adjoint contractions (vecchia_factor.cuh): dD_k = b^T dSigma~_k b, (dB_k y)_i = -b^T dSigma~_k w~, b = [-A, 1], w~ = [w, 0]
      double aa = 0., aw = 0.;
      for (int c = lane; c < q; c += 32) { aa += xa[c] * xa[c]; aw += xa[c] * xw[c]; }
      aa = warp_sum(aa); aw = warp_sum(aw);
      __syncwarp();
      for (int c = lane; c <= q; c += 32) { xa[c] = c < q ? -xa[c] : 1.; if (c == q) xw[c] = 0.; }
      __syncwarp();
      double bgb = 0., bgw = 0.;
      if (ANISO) {
        const int ng = g_aniso_ngroups;
        for (int cg = 0; cg < ng; ++cg) {
          const unsigned mask = g_aniso_mask[cg];
          double cgb = 0., cgw = 0.;
          for (int r = 1; r <= q; ++r) {
            const double br = xa[r], wr = xw[r];
            for (int c = lane; c < r; c += 32) {
              const double gq = G[r * kBigLd + c];
              const double g = gq != 0. ? gq * masked_d2(pts + r * d, pts + c * d, d, mask) : 0.;
              cgb += g * (br * xa[c]);
              cgw += g * (br * xw[c] + xa[c] * wr);
            }
          }
          cgb = 2. * warp_sum(cgb);
          cgw = warp_sum(cgw);
          if (lane == cg + 1) { bgb = cgb; bgw = cgw; }
        }
        const double u = By * Dinv_i;
        const double dDk = lane == 0 ? var - aa - (p.diag_obs - Di) : bgb;
        const double ukk = lane == 0 ? -aw : -bgw;
        acc_an[0] += ukk * u;
        acc_an[1] += u * u * dDk;
        acc_an[2] += dDk * Dinv_i;
      } else {
        for (int r = 1; r <= q; ++r) {
          const double br = xa[r], wr = xw[r];
          for (int c = lane; c < r; c += 32) {
            const double g = G[r * kBigLd + c];
            bgb += g * (br * xa[c]);
            bgw += g * (br * xw[c] + xa[c] * wr);
          }
        }
        bgb = 2. * warp_sum(bgb);
        bgw = warp_sum(bgw);
      }
      if (!ANISO && lane == 0) {
        const double u = By * Dinv_i;
        const double dD0 = var - aa - (p.diag_obs - Di);  // A.s = diag_obs - D (Vecchia_utils.cpp:1623)
        const double dD1 = bgb;
        acc[3] += -aw * u;
        acc[4] += -bgw * u;
        acc[5] += u * u * dD0;
        acc[6] += u * u * dD1;
        acc[7] += dD0 * Dinv_i;
        acc[8] += dD1 * Dinv_i;
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
  } else if (MODE != BIG_PRED && lane == 0) {
#pragma unroll
    for (int k = 0; k < kNumAcc; ++k) p.partials[gwarp * kNumAcc + k] = acc[k];
  }
}

}  // namespace gpb
