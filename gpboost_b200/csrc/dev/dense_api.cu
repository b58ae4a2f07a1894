// Device engine for the exact (dense) Gaussian-process likelihood — SURVEY §8 row a6, BASELINE config 1.
//
// Replaces RECompGP::CalcSigma (include/GPBoost/re_comp.h:1273 -> CovFunction::CalculateCovMat cov_fcts.h:635-755),
// CalcZSigmaZt (re_model_template.h:9273: Psi = I + Sigma), CalcChol (:6492, Eigen::LLT), the two triangular solves of
// CalcYAux (:9894) / CalcYTPsiIInvY (:10002) and the log-determinant (:3127).
//
// Formulation: the (n+1) x (n+1) matrix [[Psi, y],[y^T, *]] (lower triangle, row-major, 64 x 64 tiles) is factorised by a
// right-looking blocked Cholesky; the response rides along as row n, so after the factorisation
//     log|Psi| = 2 sum_{i<n} log L_ii      and      y^T Psi^-1 y = sum_{c<n} L[n][c]^2
// without a separate forward solve. Per block column k: (1) POTRF of the diagonal tile in shared memory, (2) TRSM of
// the tiles below it, (3) trailing update A_ij -= L_ik L_jk^T on the FP64 tensor cores (mma.sync m8n8k4 f64 = DMMA; tcgen05
// has no FP64 kind), operands staged in shared memory. Psi^-1 y = L^-T z by a blocked back substitution.
// Bound: tensor/FP64 pipe for the trailing update (n^3/3 flop), HBM for the Gram build (8 n^2 bytes written once).
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "vecchia_factor.cuh"  // cov_eval, rsqrt_fast

namespace {
thread_local std::string g_dense_err;
int dfail(const std::string& m) { g_dense_err = m; return -1; }
#define DCUDA(expr)                                                                                          \
  do {                                                                                                       \
    cudaError_t e__ = (expr);                                                                                \
    if (e__ != cudaSuccess)                                                                                  \
      return dfail(std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) + ": " + cudaGetErrorString(e__)); \
  } while (0)

constexpr int NB = 64;

// ---- Gram build: lower-triangular tiles of Psi = I + Sigma, plus the response row n
template <int COV>
__global__ void gram_kernel(const double* __restrict__ coords, int n, int d, const double* __restrict__ y, double var, double range,
                            double* __restrict__ A, int ld) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (tj > ti) return;
  const int N = n + 1;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = ti * NB + e / NB, c = tj * NB + e % NB;
    if (r >= ld || c >= ld) continue;
    double v = 0.;
    if (r < n && c < n) {
      if (r == c) v = var + 1.;
      else if (c < r) {
        double d2 = 0.;
        for (int k = 0; k < d; ++k) { const double df = coords[(size_t)r * d + k] - coords[(size_t)c * d + k]; d2 = fma(df, df, d2); }
        const double dist = d2 * gpb::rsqrt_fast(d2 + 1e-300);
        double g;
        v = gpb::cov_eval<COV, false>(dist, var, range, g);
      }
    } else if (r == n && c < n) {
      v = y[c];
    } else if (r == c) {
      v = 1.;  // padding rows/cols (and the response row's own diagonal): identity, never used as pivots that matter
    }
    A[(size_t)r * ld + c] = v;
    (void)N;
  }
}

// ---- POTRF of the diagonal tile k (one CTA, tile in shared memory). Rows >= npiv of the tile are eliminated but not pivoted.
__global__ void potrf_tile_kernel(double* __restrict__ A, int ld, int k, int npiv, int* __restrict__ info) {
  __shared__ double T[NB][NB + 1];
  double* base = A + (size_t)k * NB * ld + (size_t)k * NB;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) T[e / NB][e % NB] = base[(size_t)(e / NB) * ld + e % NB];
  __syncthreads();
  for (int p = 0; p < npiv; ++p) {
    const double dpp = T[p][p];
    if (threadIdx.x == 0 && !(dpp > 0.)) atomicAdd(info, 1);
    const double rs = gpb::rsqrt_fast(dpp);
    __syncthreads();
    for (int r = p + threadIdx.x; r < NB; r += blockDim.x) T[r][p] *= rs;  // column p (incl. the diagonal: sqrt)
    __syncthreads();
    for (int e = threadIdx.x; e < (NB - p - 1) * (NB - p - 1); e += blockDim.x) {
      const int r = p + 1 + e / (NB - p - 1), c = p + 1 + e % (NB - p - 1);
      if (c <= r) T[r][c] -= T[r][p] * T[c][p];
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = e / NB, c = e % NB;
    if (c <= r) base[(size_t)r * ld + c] = T[r][c];
  }
}

// ---- TRSM: tiles (i, k), i > k:  X = A_ik L_kk^-T  (each thread owns one row of the tile; L_kk in shared memory)
__global__ void trsm_tile_kernel(double* __restrict__ A, int ld, int k, int npiv) {
  __shared__ double L[NB][NB + 1];
  const double* lkk = A + (size_t)k * NB * ld + (size_t)k * NB;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) L[e / NB][e % NB] = lkk[(size_t)(e / NB) * ld + e % NB];
  __syncthreads();
  const int i = k + 1 + blockIdx.x;
  const int r = threadIdx.x;
  if (r >= NB) return;
  double* row = A + ((size_t)i * NB + r) * ld + (size_t)k * NB;
  double x[NB];
#pragma unroll
  for (int c = 0; c < NB; ++c) x[c] = row[c];
#pragma unroll
  for (int c = 0; c < NB; ++c) {
    if (c < npiv) {
      double s = x[c];
#pragma unroll
      for (int t = 0; t < c; ++t) s -= x[t] * L[c][t];
      x[c] = s / L[c][c];
    }
  }
#pragma unroll
  for (int c = 0; c < NB; ++c) row[c] = x[c];
}

// ---- trailing update on the FP64 tensor cores: A_ij -= L_ik L_jk^T for i >= j > k. One CTA (8 warps) per tile; warp w owns
// the 8-row band w of the tile and sweeps its 8 column blocks with mma.sync.m8n8k4.f64.
__device__ __forceinline__ void dmma8x8x4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__global__ void __launch_bounds__(256) syrk_tile_kernel(double* __restrict__ A, int ld, int k, int nt) {
  // map the linear block index to a lower-triangular tile (i, j) of the trailing matrix, i >= j > k
  const int m = nt - k - 1;
  int t = blockIdx.x;
  int bi = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  while (bi * (bi + 1) / 2 > t) --bi;
  const int bj = t - bi * (bi + 1) / 2;
  if (bi >= m) return;
  const int i = k + 1 + bi, j = k + 1 + bj;
  extern __shared__ __align__(16) double syrk_sm[];
  double (*Li)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(syrk_sm);
  double (*Lj)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(syrk_sm + NB * (NB + 1));
  const double* pi = A + (size_t)i * NB * ld + (size_t)k * NB;
  const double* pj = A + (size_t)j * NB * ld + (size_t)k * NB;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    Li[e / NB][e % NB] = pi[(size_t)(e / NB) * ld + e % NB];
    Lj[e / NB][e % NB] = pj[(size_t)(e / NB) * ld + e % NB];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ar = warp * 8 + (lane >> 2);   // A fragment: row lane/4 of the band, k-column lane%4
  const int kc = lane & 3;
  double acc[8][2];
#pragma unroll
  for (int cb = 0; cb < 8; ++cb) { acc[cb][0] = 0.; acc[cb][1] = 0.; }
#pragma unroll 4
  for (int k0 = 0; k0 < NB; k0 += 4) {
    const double a = Li[ar][k0 + kc];
#pragma unroll
    for (int cb = 0; cb < 8; ++cb) {
      const double b = Lj[cb * 8 + (lane >> 2)][k0 + kc];  // B[k][c] = L_j[c][k], column c = lane/4 of block cb
      dmma8x8x4(acc[cb][0], acc[cb][1], a, b);
    }
  }
  double* out = A + (size_t)i * NB * ld + (size_t)j * NB;
  const int orow = warp * 8 + (lane >> 2);
#pragma unroll
  for (int cb = 0; cb < 8; ++cb) {
    const int oc = cb * 8 + (lane & 3) * 2;
    double* o = out + (size_t)orow * ld + oc;
    o[0] -= acc[cb][0];
    o[1] -= acc[cb][1];
  }
}

// ---- log-det and quadratic form from the factor: out[0] = sum_{c<n} L[n][c]^2, out[1] = 2 sum_{i<n} log L_ii
__global__ void dense_sums_kernel(const double* __restrict__ A, int ld, int n, double* __restrict__ out) {
  __shared__ double s0[256], s1[256];
  double q = 0., l = 0.;
  const int per = (n + blockDim.x - 1) / blockDim.x;
  const int b = threadIdx.x * per, e = min(b + per, n);
  for (int c = b; c < e; ++c) { const double z = A[(size_t)n * ld + c]; q += z * z; l += log(A[(size_t)c * ld + c]); }
  s0[threadIdx.x] = q; s1[threadIdx.x] = l;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) { s0[threadIdx.x] += s0[threadIdx.x + o]; s1[threadIdx.x] += s1[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[0] = s0[0]; out[1] = 2. * s1[0]; }
}

// ---- Psi^-1 y = L^-T z, z = L[n][0..n): one CTA; x lives in shared memory; columns are swept from the last to the first
__global__ void dense_backsolve_kernel(const double* __restrict__ A, int ld, int n, double scale, double* x_out) {
  double* xs = x_out;  // global (L2-resident) work vector: one CTA, ordered by __syncthreads
  for (int c = threadIdx.x; c < n; c += blockDim.x) xs[c] = A[(size_t)n * ld + c];
  __syncthreads();
  for (int r = n - 1; r >= 0; --r) {
    if (threadIdx.x == 0) xs[r] /= A[(size_t)r * ld + r];
    __syncthreads();
    const double xr = xs[r];
    const double* lrow = A + (size_t)r * ld;  // row r of L holds L[r][c] for c < r: contiguous, coalesced
    for (int c = threadIdx.x; c < r; c += blockDim.x) xs[c] -= lrow[c] * xr;
    __syncthreads();
  }
  for (int c = threadIdx.x; c < n; c += blockDim.x) xs[c] *= scale;
}

// ---- gradient pieces (REModelTemplate::CalcPsiInv re_model_template.h:6586-6617 + the dense branch of CalcGradPars :2018-2039): W = L^-1 by blocked forward
// substitution, Psi^-1 = W^T W, then  tr(Psi^-1 dPsi_k)  and  alpha^T dPsi_k alpha  (alpha = Psi^-1 y) as tile reductions with dPsi
// recomputed from the coordinates. Rows >= n of the factor buffer (response row, padding) are treated as identity rows.
__device__ __forceinline__ double load_L(const double* __restrict__ A, int ld, int n, int r, int c) {
  if (r >= n || c >= n) return r == c ? 1. : 0.;
  return c <= r ? A[(size_t)r * ld + c] : 0.;
}
// C[4][4] (thread (ty,tx) of a 16 x 16 layout owns rows 4ty.., cols 4tx..) += As (64 x 64, [r][k]) * Bs (64 x 64, [k][c])
__device__ __forceinline__ void tile_fma(double (&C)[4][4], const double (*As)[NB + 1], const double (*Bs)[NB + 1], int ty, int tx) {
#pragma unroll 8
  for (int k = 0; k < NB; ++k) {
    double a[4], b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) { a[u] = As[ty * 4 + u][k]; b[u] = Bs[k][tx * 4 + u]; }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) C[u][v] = fma(a[u], b[v], C[u][v]);
  }
}
// W_ii = L_ii^-1 for every diagonal tile (thread c solves column c of the tile by forward substitution)
__global__ void trinv_diag_kernel(const double* __restrict__ A, int ld, int n, double* __restrict__ W) {
  __shared__ double Ls[NB][NB + 1];
  const int i = blockIdx.x;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) Ls[e / NB][e % NB] = load_L(A, ld, n, i * NB + e / NB, i * NB + e % NB);
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= NB) return;
  double x[NB];
#pragma unroll
  for (int r = 0; r < NB; ++r) {
    double s = r == c ? 1. : 0.;
#pragma unroll
    for (int t = 0; t < r; ++t) s -= Ls[r][t] * x[t];
    x[r] = r < c ? 0. : s / Ls[r][r];
  }
  double* out = W + (size_t)i * NB * ld + (size_t)i * NB;
#pragma unroll
  for (int r = 0; r < NB; ++r) out[(size_t)r * ld + c] = x[r];
}
// block row i of W, tiles j < i:  W_ij = -W_ii * sum_{k=j}^{i-1} L_ik W_kj
__global__ void __launch_bounds__(256) trinv_row_kernel(const double* __restrict__ A, int ld, int n, double* __restrict__ W, int i) {
  extern __shared__ __align__(16) double tsm[];
  double (*As)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(tsm);
  double (*Bs)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(tsm + NB * (NB + 1));
  const int j = blockIdx.x;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  double C[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) C[u][v] = 0.;
  for (int k = j; k < i; ++k) {
    __syncthreads();
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
      const int r = e / NB, c = e % NB;
      As[r][c] = load_L(A, ld, n, i * NB + r, k * NB + c);
      Bs[r][c] = W[(size_t)(k * NB + r) * ld + (size_t)j * NB + c];
    }
    __syncthreads();
    tile_fma(C, As, Bs, ty, tx);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) As[e / NB][e % NB] = W[(size_t)(i * NB + e / NB) * ld + (size_t)i * NB + e % NB];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) Bs[ty * 4 + u][tx * 4 + v] = C[u][v];
  __syncthreads();
  double D[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) D[u][v] = 0.;
  tile_fma(D, As, Bs, ty, tx);
  double* out = W + (size_t)i * NB * ld + (size_t)j * NB;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) out[(size_t)(ty * 4 + u) * ld + tx * 4 + v] = -D[u][v];
}
// P_IJ = sum_{K >= I} W_KI^T W_KJ for the lower tiles I >= J (P = Psi^-1)
__global__ void __launch_bounds__(256) wtw_kernel(const double* __restrict__ W, int ld, int nt, double* __restrict__ P) {
  int t = blockIdx.x;
  int bi = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  while (bi * (bi + 1) / 2 > t) --bi;
  const int bj = t - bi * (bi + 1) / 2;
  extern __shared__ __align__(16) double tsm[];
  double (*As)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(tsm);
  double (*Bs)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(tsm + NB * (NB + 1));
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  double C[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) C[u][v] = 0.;
  for (int k = bi; k < nt; ++k) {
    __syncthreads();
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
      const int r = e / NB, c = e % NB;  // element (r, c) of W_K. : row r of block row K
      As[c][r] = W[(size_t)(k * NB + r) * ld + (size_t)bi * NB + c];  // transposed: As[row of P tile][k]
      Bs[r][c] = W[(size_t)(k * NB + r) * ld + (size_t)bj * NB + c];
    }
    __syncthreads();
    tile_fma(C, As, Bs, ty, tx);
  }
  double* out = P + (size_t)bi * NB * ld + (size_t)bj * NB;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) out[(size_t)(ty * 4 + u) * ld + tx * 4 + v] = C[u][v];
}
// per lower tile: 0 sum_{i != j} P_ij G_ij   1 sum_{i != j} alpha_i alpha_j G_ij   2 tr P   (G = dSigma / dlog range, zero diagonal)
template <int COV>
__global__ void dense_grad_sums_kernel(const double* __restrict__ coords, int n, int d, double var, double range,
                                       const double* __restrict__ P, int ld, const double* __restrict__ alpha, double* __restrict__ part) {
  int t = blockIdx.x;
  int bi = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  while (bi * (bi + 1) / 2 > t) --bi;
  const int bj = t - bi * (bi + 1) / 2;
  double s0 = 0., s1 = 0., s2 = 0.;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = bi * NB + e / NB, c = bj * NB + e % NB;
    if (r >= n || c > r) continue;
    const double p = P[(size_t)r * ld + c];
    if (r == c) { s2 += p; continue; }
    double d2 = 0.;
    for (int k = 0; k < d; ++k) { const double df = coords[(size_t)r * d + k] - coords[(size_t)c * d + k]; d2 = fma(df, df, d2); }
    const double dist = d2 * gpb::rsqrt_fast(d2 + 1e-300);
    double g;
    gpb::cov_eval<COV, true>(dist, var, range, g);
    s0 += 2. * p * g;
    s1 += 2. * alpha[r] * alpha[c] * g;
  }
  __shared__ double sh[3][256];
  sh[0][threadIdx.x] = s0; sh[1][threadIdx.x] = s1; sh[2][threadIdx.x] = s2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int q = 0; q < 3; ++q) sh[q][threadIdx.x] += sh[q][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 3) part[(size_t)blockIdx.x * 3 + threadIdx.x] = sh[threadIdx.x][0];
}
// fixed-order sum of the tile partials + alpha^T alpha
__global__ void dense_grad_final_kernel(const double* __restrict__ part, int nblk, const double* __restrict__ alpha, int n, double* __restrict__ out) {
  __shared__ double sh[4][256];
  double a[4] = {0., 0., 0., 0.};
  const int per = (nblk + 255) / 256;
  for (int b = threadIdx.x * per; b < min((threadIdx.x + 1) * per, nblk); ++b)
    for (int q = 0; q < 3; ++q) a[q] += part[(size_t)b * 3 + q];
  const int pern = (n + 255) / 256;
  for (int i = threadIdx.x * pern; i < min((threadIdx.x + 1) * pern, n); ++i) a[3] += alpha[i] * alpha[i];
  for (int q = 0; q < 4; ++q) sh[q][threadIdx.x] = a[q];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int q = 0; q < 4; ++q) sh[q][threadIdx.x] += sh[q][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 4) out[threadIdx.x] = sh[threadIdx.x][0];
}
using GradSumsKernel = void (*)(const double*, int, int, double, double, const double*, int, const double*, double*);
GradSumsKernel pick_grad_sums(int cov) {
  switch (cov) {
    case 0: return dense_grad_sums_kernel<0>;
    case 1: return dense_grad_sums_kernel<1>;
    case 2: return dense_grad_sums_kernel<2>;
    default: return dense_grad_sums_kernel<3>;
  }
}

using GramKernel = void (*)(const double*, int, int, const double*, double, double, double*, int);
GramKernel pick_gram(int cov) {
  switch (cov) {
    case 0: return gram_kernel<0>;
    case 1: return gram_kernel<1>;
    case 2: return gram_kernel<2>;
    default: return gram_kernel<3>;
  }
}
}  // namespace

struct gpbdev_dense {
  int device = 0;
  int n = 0, d = 0, ld = 0, nt = 0;
  cudaStream_t stream = nullptr;
  double *coords = nullptr, *y = nullptr, *A = nullptr, *out = nullptr, *x = nullptr;
  double *W = nullptr, *P = nullptr, *gpart = nullptr;  // gradient pass: L^-1, Psi^-1, tile partials (lazy)
  int last_cov = -1; double last_var = 0., last_range = 0.;
  int* info = nullptr;
  double* out_host = nullptr;
  int64_t launches = 0;
  bool factored = false;
  bool psi_inv_ready = false;  // P holds Psi^-1 of the current factor
};

extern "C" {

const char* gpbdev_dense_last_error(void) { return g_dense_err.c_str(); }

int gpbdev_dense_create(gpbdev_dense_t* out, int device, int n, int d, const double* coords_rowmajor) {
  if (!out || !coords_rowmajor) return dfail("gpbdev_dense_create: null argument");
  if (n <= 0 || d <= 0) return dfail("gpbdev_dense_create: need n > 0 and dim > 0");
  if (n > 46000) return dfail("gpbdev_dense_create: the dense engine keeps an n x n fp64 matrix; n is limited to 46000 (use gp_approx = 'vecchia')");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) {
    cudaGetLastError();
    return dfail("gpbdev_dense_create: no CUDA device " + std::to_string(device) + " — the CUDA engine has no CPU fallback");
  }
  DCUDA(cudaSetDevice(device));
  gpbdev_dense* h = new gpbdev_dense();
  h->device = device; h->n = n; h->d = d;
  h->nt = (n + 1 + NB - 1) / NB;
  h->ld = h->nt * NB;
  DCUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  DCUDA(cudaMalloc(&h->coords, sizeof(double) * (size_t)n * d));
  DCUDA(cudaMalloc(&h->y, sizeof(double) * n));
  DCUDA(cudaMalloc(&h->x, sizeof(double) * n));
  DCUDA(cudaMalloc(&h->A, sizeof(double) * (size_t)h->ld * h->ld));
  DCUDA(cudaMalloc(&h->out, sizeof(double) * 4));
  DCUDA(cudaMalloc(&h->info, sizeof(int)));
  DCUDA(cudaMallocHost(&h->out_host, sizeof(double) * 4));
  // on the engine's stream: it does not wait for the legacy default stream, so a cudaMemset there could land after the
  // first set_y and zero the response
  DCUDA(cudaMemcpyAsync(h->coords, coords_rowmajor, sizeof(double) * (size_t)n * d, cudaMemcpyHostToDevice, h->stream));
  DCUDA(cudaMemsetAsync(h->y, 0, sizeof(double) * n, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  DCUDA(cudaFuncSetAttribute(syrk_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * 2 * NB * (NB + 1))));
  *out = h;
  return 0;
}

int gpbdev_dense_free(gpbdev_dense_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaFree(h->coords); cudaFree(h->y); cudaFree(h->x); cudaFree(h->A); cudaFree(h->out); cudaFree(h->info);
  cudaFree(h->W); cudaFree(h->P); cudaFree(h->gpart);
  cudaFreeHost(h->out_host);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int gpbdev_dense_set_y(gpbdev_dense_t h, const double* y_host) {
  if (!h || !y_host) return dfail("gpbdev_dense_set_y: null argument");
  DCUDA(cudaSetDevice(h->device));
  DCUDA(cudaMemcpyAsync(h->y, y_host, sizeof(double) * h->n, cudaMemcpyHostToDevice, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  h->factored = false;
  h->psi_inv_ready = false;
  return 0;
}

int gpbdev_dense_eval(gpbdev_dense_t h, int cov_type, double var, double range, double* out3) {
  if (!h || !out3) return dfail("gpbdev_dense_eval: null argument");
  if (cov_type < 0 || cov_type > 3) return dfail("gpbdev_dense_eval: unknown covariance id");
  if (!(var > 0.) || !(range > 0.)) return dfail("gpbdev_dense_eval: covariance parameters must be positive");
  DCUDA(cudaSetDevice(h->device));
  const int n = h->n, nt = h->nt, ld = h->ld;
  h->psi_inv_ready = false;
  DCUDA(cudaMemsetAsync(h->info, 0, sizeof(int), h->stream));
  pick_gram(cov_type)<<<dim3(nt, nt), 256, 0, h->stream>>>(h->coords, n, h->d, h->y, var, range, h->A, ld);
  DCUDA(cudaGetLastError());
  h->launches += 1;
  for (int k = 0; k < nt; ++k) {
    // pivots of this tile that belong to Psi (the response row n and the padding are eliminated, never pivoted)
    const int npiv = std::max(0, std::min(NB, n - k * NB));
    if (npiv == 0) break;
    potrf_tile_kernel<<<1, 256, 0, h->stream>>>(h->A, ld, k, npiv, h->info);
    if (k + 1 < nt) {
      trsm_tile_kernel<<<nt - k - 1, NB, 0, h->stream>>>(h->A, ld, k, npiv);
      const int m = nt - k - 1;
      syrk_tile_kernel<<<m * (m + 1) / 2, 256, sizeof(double) * 2 * NB * (NB + 1), h->stream>>>(h->A, ld, k, nt);
      h->launches += 2;
    }
    h->launches += 1;
    DCUDA(cudaGetLastError());
  }
  dense_sums_kernel<<<1, 256, 0, h->stream>>>(h->A, ld, n, h->out);
  h->launches += 1;
  int info = 0;
  DCUDA(cudaMemcpyAsync(h->out_host, h->out, sizeof(double) * 2, cudaMemcpyDeviceToHost, h->stream));
  DCUDA(cudaMemcpyAsync(&info, h->info, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  out3[0] = h->out_host[0];
  out3[1] = h->out_host[1];
  out3[2] = (double)info;  // non-positive pivots (matrix not positive definite)
  h->factored = true;
  h->last_cov = cov_type; h->last_var = var; h->last_range = range;
  return 0;
}

// Gradient sums at the parameters of the last gpbdev_dense_eval: out4 = {tr(Psi^-1 Sigma), tr(Psi^-1 dSigma/dlog range),
// alpha^T Sigma alpha, alpha^T dSigma/dlog range alpha} with alpha = Psi^-1 y (transformed scale, Psi = I + Sigma).
int gpbdev_dense_grad(gpbdev_dense_t h, double* out4) {
  if (!h || !out4) return dfail("gpbdev_dense_grad: null argument");
  if (!h->factored) return dfail("gpbdev_dense_grad: call gpbdev_dense_eval first");
  DCUDA(cudaSetDevice(h->device));
  const int n = h->n, nt = h->nt, ld = h->ld;
  const int ntiles = nt * (nt + 1) / 2;
  if (!h->W) {
    DCUDA(cudaMalloc(&h->W, sizeof(double) * (size_t)ld * ld));
    DCUDA(cudaMalloc(&h->P, sizeof(double) * (size_t)ld * ld));
    DCUDA(cudaMalloc(&h->gpart, sizeof(double) * (size_t)ntiles * 3));
    const int smem = (int)(sizeof(double) * 2 * NB * (NB + 1));
    DCUDA(cudaFuncSetAttribute(trinv_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DCUDA(cudaFuncSetAttribute(wtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  const size_t smem = sizeof(double) * 2 * NB * (NB + 1);
  const double quad = h->out_host[0];  // y^T Psi^-1 y = alpha^T y
  dense_backsolve_kernel<<<1, 1024, 0, h->stream>>>(h->A, ld, n, 1.0, h->x);
  trinv_diag_kernel<<<nt, NB, 0, h->stream>>>(h->A, ld, n, h->W);
  DCUDA(cudaGetLastError());
  for (int i = 1; i < nt; ++i) trinv_row_kernel<<<i, 256, smem, h->stream>>>(h->A, ld, n, h->W, i);
  DCUDA(cudaGetLastError());
  wtw_kernel<<<ntiles, 256, smem, h->stream>>>(h->W, ld, nt, h->P);
  pick_grad_sums(h->last_cov)<<<ntiles, 256, 0, h->stream>>>(h->coords, n, h->d, h->last_var, h->last_range, h->P, ld, h->x, h->gpart);
  dense_grad_final_kernel<<<1, 256, 0, h->stream>>>(h->gpart, ntiles, h->x, n, h->out + 0);
  DCUDA(cudaGetLastError());
  h->launches += 4 + nt;
  DCUDA(cudaMemcpyAsync(h->out_host, h->out, sizeof(double) * 4, cudaMemcpyDeviceToHost, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  const double s_pg = h->out_host[0], s_aga = h->out_host[1], tr_p = h->out_host[2], aa = h->out_host[3];
  out4[0] = (double)n - tr_p;   // tr(Psi^-1 (Psi - I))
  out4[1] = s_pg;
  out4[2] = quad - aa;          // alpha^T (Psi - I) alpha = alpha^T y - alpha^T alpha
  out4[3] = s_aga;
  h->out_host[0] = quad;
  h->psi_inv_ready = true;
  return 0;
}

int gpbdev_dense_yaux(gpbdev_dense_t h, double scale, double* yaux_host) {
  if (!h || !yaux_host) return dfail("gpbdev_dense_yaux: null argument");
  if (!h->factored) return dfail("gpbdev_dense_yaux: call gpbdev_dense_eval first");
  DCUDA(cudaSetDevice(h->device));
  dense_backsolve_kernel<<<1, 1024, 0, h->stream>>>(h->A, h->ld, h->n, scale, h->x);
  DCUDA(cudaGetLastError());
  h->launches += 1;
  DCUDA(cudaMemcpyAsync(yaux_host, h->x, sizeof(double) * h->n, cudaMemcpyDeviceToHost, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

// Read-back of the factor for tests. Only the lower triangle of the diagonal tiles is the factor (the trailing update
// writes whole diagonal tiles, and tiles above the diagonal are never written), so the upper triangle is zeroed here.
int gpbdev_dense_get_factor(gpbdev_dense_t h, double* L_host, double* z_host) {
  if (!h || !L_host) return dfail("gpbdev_dense_get_factor: null argument");
  if (!h->factored) return dfail("gpbdev_dense_get_factor: no current factor (call gpbdev_dense_eval after gpbdev_dense_set_y)");
  DCUDA(cudaSetDevice(h->device));
  const size_t n = (size_t)h->n, ld = (size_t)h->ld;
  DCUDA(cudaMemcpy2DAsync(L_host, sizeof(double) * n, h->A, sizeof(double) * ld, sizeof(double) * n, n, cudaMemcpyDeviceToHost,
                          h->stream));
  if (z_host) DCUDA(cudaMemcpyAsync(z_host, h->A + n * ld, sizeof(double) * n, cudaMemcpyDeviceToHost, h->stream));
  DCUDA(cudaStreamSynchronize(h->stream));
  for (size_t r = 0; r < n; ++r) std::fill(L_host + r * n + r + 1, L_host + (r + 1) * n, 0.);
  return 0;
}

// Read-back of Psi^-1 for tests: block row I of P is copied up to its diagonal tile (the upper tiles are never written),
// then the strict lower triangle is mirrored.
int gpbdev_dense_get_psi_inv(gpbdev_dense_t h, double* P_host) {
  if (!h || !P_host) return dfail("gpbdev_dense_get_psi_inv: null argument");
  if (!h->factored || !h->psi_inv_ready) return dfail("gpbdev_dense_get_psi_inv: no current Psi^-1 (call gpbdev_dense_grad after gpbdev_dense_eval)");
  DCUDA(cudaSetDevice(h->device));
  const size_t n = (size_t)h->n, ld = (size_t)h->ld;
  for (size_t r0 = 0; r0 < n; r0 += NB) {
    const size_t rows = std::min<size_t>(NB, n - r0), cols = std::min(r0 + NB, n);
    DCUDA(cudaMemcpy2DAsync(P_host + r0 * n, sizeof(double) * n, h->P + r0 * ld, sizeof(double) * ld, sizeof(double) * cols, rows,
                            cudaMemcpyDeviceToHost, h->stream));
  }
  DCUDA(cudaStreamSynchronize(h->stream));
  for (size_t r = 0; r < n; ++r)
    for (size_t c = r + 1; c < n; ++c) P_host[r * n + c] = P_host[c * n + r];
  return 0;
}

int64_t gpbdev_dense_launch_count(gpbdev_dense_t h) { return h ? h->launches : 0; }

}  // extern "C"
