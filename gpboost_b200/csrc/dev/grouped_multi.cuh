// Device engine for K >= 2 grouped random effects (crossed or nested) with a Gaussian likelihood. Included at the end of
// grouped_api.cu (shares its error channel and the per-level segmented sum kernel).
//
// Replaces, for num_re_group_total_ >= 2, no GP, matrix_inversion_method = "iterative", cg_preconditioner_type = "ssor", the
// reference's Woodbury path on the random-effect scale, M = Sigma^-1 + Z^T Z (size G = sum_k G_k, components in
// cum_num_rand_eff order):
//   CalcCovFactor iterative / SSOR branch    re_model_template.h:9422-9438   (D = diag(M), L = lower(M), P = L D^-1 L^T)
//   CalcYAux iterative branch                :9850-9891, CGRandomEffectsVec   CG_utils.cpp:1147-1281 (M x = Z^T y, warm start)
//   log-det, iterative branch                :3033-3124, CGTridiagRandomEffects CG_utils.cpp:1283-1473, LogDetStochTridiag
//   CalcGradPars_..._Woodbury_Gauss, iterative :2530-2619 (stochastic trace with SSOR variance reduction, CalcOptimalC)
//
// Design. Only diag(M) depends on the covariance parameters: the off-diagonal entries are co-occurrence counts of the levels
// of two factors, fixed by the data. Every observation has one level per factor, so each diagonal block of Z^T Z is diagonal
// and L is block lower-triangular with diagonal blocks: a triangular solve is K block steps, each a sparse row product over the
// earlier (forward) or later (backward) blocks followed by a diagonal scaling, one launch per block. M's off-diagonal part is
// held once as CSR (columns ascending, `split[i]` = first entry right of the diagonal), so the same arrays serve M X, the lower
// and the upper triangle. Multi-vectors are G x t row-major: a warp owns a row, lanes own columns, so a gathered row is one
// contiguous 8t-byte read. The CG scalars (per-column dots) come to the host every iteration, as in the Laplace engine.
// The sparsity pattern is built on the host at creation (sort of the K (K - 1) n level pairs).
#include <numeric>

#include "slq.h"

namespace gmk {

constexpr int kMaxCols = 128;
constexpr int kPer = kMaxCols / 32;
constexpr int kBlock = 256;

struct Coef { double v[kMaxCols]; };

// Y = diag .* X + Off X (diag may be null: off-diagonal part only)
__global__ void __launch_bounds__(kBlock) spmm_kernel(int G, int t, const int64_t* __restrict__ rp, const int32_t* __restrict__ col,
                                                      const double* __restrict__ val, const double* __restrict__ diag,
                                                      const double* __restrict__ X, double* __restrict__ Y) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int i = gw; i < G; i += nw) {
    double acc[kPer];
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int c = q * 32 + lane;
      acc[q] = (c < t && diag) ? diag[i] * X[(size_t)i * t + c] : 0.;
    }
    for (int64_t e = rp[i]; e < rp[i + 1]; ++e) {
      const size_t j = (size_t)col[e];
      const double v = val[e];
#pragma unroll
      for (int q = 0; q < kPer; ++q) {
        const int c = q * 32 + lane;
        if (c < t) acc[q] += v * X[j * t + c];
      }
    }
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int c = q * 32 + lane;
      if (c < t) Y[(size_t)i * t + c] = acc[q];
    }
  }
}

// rows [r0, r1) of one block.  mode 0 (forward solve with L D^-1/2):  W_i = (R_i - sum_{j < i} M_ij dis_j W_j) / ld_i
//                              mode 1 (backward solve with its transpose): W_i = (R_i - sum_{j > i} M_ji dis_i W_j) / ld_i
//                              mode 2 (probe map u = L D^-1/2 r):     W_i = ld_i R_i + sum_{j < i} M_ij dis_j R_j
//                              mode 3 (D^-1 upper(M) X):              W_i = Dinv_i (Mdiag_i R_i + sum_{j > i} M_ij R_j)
// ld = diag(L D^-1/2) = Mdiag .* dis, dis = D^-1/2. Modes 0 / 1 read W of the other blocks (written by earlier launches).
template <int kMode>
__global__ void __launch_bounds__(kBlock) tri_kernel(int r0, int r1, int t, const int64_t* __restrict__ rp, const int64_t* __restrict__ split,
                                                     const int32_t* __restrict__ col, const double* __restrict__ val,
                                                     const double* __restrict__ dis, const double* __restrict__ ld,
                                                     const double* __restrict__ Mdiag, const double* __restrict__ Dinv,
                                                     const double* __restrict__ R, double* W) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int i = r0 + gw; i < r1; i += nw) {
    const bool lower = kMode == 0 || kMode == 2;
    const int64_t eb = lower ? rp[i] : split[i], ee = lower ? split[i] : rp[i + 1];
    const double* src = (kMode == 0 || kMode == 1) ? W : R;
    double acc[kPer];
#pragma unroll
    for (int q = 0; q < kPer; ++q) acc[q] = 0.;
    for (int64_t e = eb; e < ee; ++e) {
      const size_t j = (size_t)col[e];
      double v = val[e];
      if (kMode == 0 || kMode == 2) v *= dis[j];
      else if (kMode == 1) v *= dis[i];
#pragma unroll
      for (int q = 0; q < kPer; ++q) {
        const int c = q * 32 + lane;
        if (c < t) acc[q] += v * src[j * t + c];
      }
    }
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int c = q * 32 + lane;
      if (c >= t) continue;
      const double r = R[(size_t)i * t + c];
      double w;
      if (kMode == 0 || kMode == 1) w = (r - acc[q]) / ld[i];
      else if (kMode == 2) w = ld[i] * r + acc[q];
      else w = Dinv[i] * (Mdiag[i] * r + acc[q]);
      W[(size_t)i * t + c] = w;
    }
  }
}

// diag(M) at variance ratios v_k (inv_v = 1 / v_k per component, comp = component of each row), D^-1, D^-1/2, diag(L D^-1/2)
// and log diag(L D^-1/2)
__global__ void diag_kernel(int G, const int32_t* __restrict__ comp, const double* __restrict__ cnt, Coef inv_v, double* __restrict__ Mdiag,
                            double* __restrict__ Dinv, double* __restrict__ dis, double* __restrict__ ld, double* __restrict__ logld) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < G; i += gridDim.x * blockDim.x) {
    const double m = inv_v.v[comp[i]] + cnt[i];
    const double di = 1. / m;
    const double s = sqrt(di);
    Mdiag[i] = m; Dinv[i] = di; dis[i] = s; ld[i] = m * s; logld[i] = log(m * s);
  }
}

// out[c] = sum_{i in [r0, r1)} A[i t + c] B[i t + c] (kAbs: sum of |A[i t + c]|, B unused): one block per column, contiguous slice
// per thread, fixed-order tree
template <bool kAbs>
__global__ void __launch_bounds__(kBlock) coldot_kernel(int r0, int r1, int t, const double* __restrict__ A, const double* __restrict__ B,
                                                        double* __restrict__ out) {
  __shared__ double sh[kBlock];
  const int c = blockIdx.x;
  const int len = r1 - r0;
  const int per = (len + kBlock - 1) / kBlock;
  const int b = r0 + threadIdx.x * per, e = min(b + per, r1);
  double a = 0.;
  for (int i = b; i < e; ++i) a += kAbs ? fabs(A[(size_t)i * t + c]) : A[(size_t)i * t + c] * B[(size_t)i * t + c];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int o = kBlock / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[c] = sh[0];
}

// U += a H (U may be null), R -= a V  (a per column)
__global__ void axpy_kernel(int64_t len, int t, Coef a, const double* __restrict__ H, const double* __restrict__ V, double* __restrict__ R,
                            double* __restrict__ U) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < len; e += (int64_t)gridDim.x * blockDim.x) {
    const double ac = a.v[e % t];
    if (U) U[e] += ac * H[e];
    R[e] -= ac * V[e];
  }
}

// H = Z + b H
__global__ void hupd_kernel(int64_t len, int t, Coef b, const double* __restrict__ Z, double* __restrict__ H) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < len; e += (int64_t)gridDim.x * blockDim.x) H[e] = Z[e] + b.v[e % t] * H[e];
}

// out_i = (y_i - sum_k x[cum_k + idx_k(i)]) * scale, original observation order
__global__ void yaux_kernel(int64_t n, int K, const int32_t* __restrict__ idx, Coef cum, const double* __restrict__ x, const double* __restrict__ y,
                            double scale, double* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double zx = 0.;
    for (int k = 0; k < K; ++k) zx += x[(int64_t)cum.v[k] + idx[(int64_t)k * n + i]];
    out[i] = (y[i] - zx) * scale;
  }
}

}  // namespace gmk

struct gpbdev_grouped_multi {
  int device = 0, num_sms = 0, K = 0, G = 0, tmax = 0, t = 0;
  int64_t n = 0, nnz = 0;
  cudaStream_t stream = nullptr;
  std::vector<int> cum;                  // K + 1 component offsets
  std::vector<int64_t> rp_host;          // for tests / nnz
  int64_t *rp = nullptr, *split = nullptr;
  int32_t *col = nullptr, *comp = nullptr, *idx = nullptr, *perm = nullptr, *offs = nullptr;
  double *val = nullptr, *cnt = nullptr, *ones = nullptr;
  double *Mdiag = nullptr, *Dinv = nullptr, *dis = nullptr, *ld = nullptr, *logld = nullptr;
  double *y = nullptr, *yaux = nullptr, *Zty = nullptr, *yy = nullptr, *x = nullptr, *g1 = nullptr, *g2 = nullptr;
  double *R = nullptr, *Z = nullptr, *H = nullptr, *V = nullptr, *W = nullptr, *U = nullptr, *probes = nullptr, *UP = nullptr;
  double *dots = nullptr, *dots_host = nullptr, *stage = nullptr;
  std::vector<double> v;                 // variance ratios of the last evaluation
  double yTy = 0.;
  bool has_y = false, has_x = false, state_valid = false;
  int64_t launches = 0;
};

namespace {

int gm_grid(const gpbdev_grouped_multi* h, int64_t rows_or_len, int per) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((rows_or_len * per + gmk::kBlock - 1) / gmk::kBlock, (int64_t)h->num_sms * 16));
}

// column dots over rows [r0, r1) -> out (host); B = nullptr: column sums of |A| (L1 norms)
int gm_dots(gpbdev_grouped_multi* h, int r0, int r1, int t, const double* A, const double* B, double* out) {
  if (B) gmk::coldot_kernel<false><<<t, gmk::kBlock, 0, h->stream>>>(r0, r1, t, A, B, h->dots);
  else gmk::coldot_kernel<true><<<t, gmk::kBlock, 0, h->stream>>>(r0, r1, t, A, nullptr, h->dots);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  GCUDA(cudaMemcpyAsync(h->dots_host, h->dots, sizeof(double) * t, cudaMemcpyDeviceToHost, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  std::memcpy(out, h->dots_host, sizeof(double) * t);
  return 0;
}

int gm_spmm(gpbdev_grouped_multi* h, int t, const double* diag, const double* X, double* Y) {
  gmk::spmm_kernel<<<gm_grid(h, h->G, 32), gmk::kBlock, 0, h->stream>>>(h->G, t, h->rp, h->col, h->val, diag, X, Y);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

template <int kMode>
int gm_tri(gpbdev_grouped_multi* h, int r0, int r1, int t, const double* R, double* W) {
  gmk::tri_kernel<kMode><<<gm_grid(h, r1 - r0, 32), gmk::kBlock, 0, h->stream>>>(r0, r1, t, h->rp, h->split, h->col, h->val, h->dis, h->ld,
                                                                                  h->Mdiag, h->Dinv, R, W);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

// Z = P^-1 R = (L D^-1/2)^-T (L D^-1/2)^-1 R (W: scratch); column dots R.Z -> rz
int gm_precond(gpbdev_grouped_multi* h, int t, const double* R, double* Z, double* W, double* rz) {
  for (int k = 0; k < h->K; ++k)
    if (gm_tri<0>(h, h->cum[k], h->cum[k + 1], t, R, W)) return -1;
  for (int k = h->K - 1; k >= 0; --k)
    if (gm_tri<1>(h, h->cum[k], h->cum[k + 1], t, W, Z)) return -1;
  return rz ? gm_dots(h, 0, h->G, t, R, Z, rz) : 0;
}

// G x t work blocks for up to t columns (t = 1 serves the single-vector solve of M x = Z^T y)
int gm_reserve(gpbdev_grouped_multi* h, int t) {
  if (t <= h->tmax) return 0;
  double** mv[] = {&h->R, &h->Z, &h->H, &h->V, &h->W, &h->U, &h->probes, &h->UP};
  for (double** p : mv) { cudaFree(*p); *p = nullptr; GCUDA(cudaMalloc(p, sizeof(double) * h->G * t)); }
  h->tmax = t;
  return 0;
}

int gm_set_diag(gpbdev_grouped_multi* h, const double* v) {
  gmk::Coef iv;
  for (int k = 0; k < h->K; ++k) {
    if (!(v[k] > 0.)) return gfail("gpbdev_grouped_multi: the variance ratios must be positive");
    iv.v[k] = 1. / v[k];
  }
  gmk::diag_kernel<<<gm_grid(h, h->G, 1), gmk::kBlock, 0, h->stream>>>(h->G, h->comp, h->cnt, iv, h->Mdiag, h->Dinv, h->dis, h->ld, h->logld);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  h->v.assign(v, v + h->K);
  return 0;
}

// Preconditioned CG on M X = B over t columns (B, X: G x t row-major). lanczos = false: CGRandomEffectsVec (t = 1, stop on the
// residual norm, X warm-started when `warm`); lanczos = true: CGTridiagRandomEffects (X from zero, stop on the mean column
// residual norm, Lanczos tridiagonals of every column in Td / Ts). Returns the iteration count in *its.
int gm_pcg(gpbdev_grouped_multi* h, int t, const double* B, double* X, bool warm, int maxit, double delta, bool lanczos,
           std::vector<std::vector<double>>* Td, std::vector<std::vector<double>>* Ts, int* its) {
  const int64_t len = (int64_t)h->G * t;
  const int lb = gm_grid(h, len, 1);
  const int p = std::min(maxit, h->G);
  GCUDA(cudaMemcpyAsync(h->R, B, sizeof(double) * len, cudaMemcpyDeviceToDevice, h->stream));
  std::vector<double> rz(t), rz_new(t), hv(t), rr(t), a(t, 1.), a_old(t, 1.), b(t, 0.), b_old(t, 0.);
  if (!lanczos) {
    double b1;  // the reference returns zero when |B|_1 < 1e-100 (THRESHOLD_ZERO_RHS_CG_)
    if (gm_dots(h, 0, h->G, 1, B, nullptr, &b1)) return -1;
    if (b1 < 1e-100) {
      GCUDA(cudaMemsetAsync(X, 0, sizeof(double) * len, h->stream));
      return 0;
    }
    if (warm) {
      if (gm_spmm(h, 1, h->Mdiag, X, h->V)) return -1;
      gmk::Coef one; one.v[0] = 1.;
      gmk::axpy_kernel<<<lb, gmk::kBlock, 0, h->stream>>>(len, 1, one, nullptr, h->V, h->R, nullptr);
      GCUDA(cudaGetLastError());
      h->launches += 1;
    }
  }
  if (!warm || lanczos) GCUDA(cudaMemsetAsync(X, 0, sizeof(double) * len, h->stream));
  if (gm_precond(h, t, h->R, h->Z, h->W, rz.data())) return -1;
  GCUDA(cudaMemcpyAsync(h->H, h->Z, sizeof(double) * len, cudaMemcpyDeviceToDevice, h->stream));
  if (lanczos) { Td->assign(t, {}); Ts->assign(t, {}); }
  for (int j = 0; j < p; ++j) {
    if (gm_spmm(h, t, h->Mdiag, h->H, h->V)) return -1;
    if (gm_dots(h, 0, h->G, t, h->H, h->V, hv.data())) return -1;
    a_old = a;
    gmk::Coef ac;
    for (int c = 0; c < t; ++c) { a[c] = rz[c] / hv[c]; ac.v[c] = a[c]; }
    gmk::axpy_kernel<<<lb, gmk::kBlock, 0, h->stream>>>(len, t, ac, h->H, h->V, h->R, X);
    GCUDA(cudaGetLastError());
    h->launches += 1;
    if (gm_dots(h, 0, h->G, t, h->R, h->R, rr.data())) return -1;
    bool early = false;
    if (!lanczos) {
      const double rn = std::sqrt(rr[0]);
      if (!std::isfinite(rn)) return gfail("There was Nan or Inf value generated in the Conjugate Gradient Method!");
      if (rn < delta) { *its = j + 1; return 0; }
    } else {
      double mean_norm = 0.;
      for (int c = 0; c < t; ++c) mean_norm += std::sqrt(rr[c]);
      mean_norm /= t;
      if (!std::isfinite(mean_norm)) return gfail("There was Nan or Inf value generated in the Conjugate Gradient Method!");
      early = mean_norm < delta;
    }
    if (gm_precond(h, t, h->R, h->Z, h->W, rz_new.data())) return -1;
    b_old = b;
    gmk::Coef bc;
    for (int c = 0; c < t; ++c) { b[c] = rz_new[c] / rz[c]; bc.v[c] = b[c]; rz[c] = rz_new[c]; }
    gmk::hupd_kernel<<<lb, gmk::kBlock, 0, h->stream>>>(len, t, bc, h->Z, h->H);
    GCUDA(cudaGetLastError());
    h->launches += 1;
    if (lanczos) {
      for (int c = 0; c < t; ++c) {
        (*Td)[c].push_back(1. / a[c] + b_old[c] / a_old[c]);
        if (j > 0) (*Ts)[c].push_back(std::sqrt(b_old[c]) / a_old[c]);
      }
      if (early) { *its = j + 1; return 0; }
    }
  }
  *its = p;
  return 0;
}

// CalcYAux (iterative): x = M^-1 Z^T y, warm-started from the previous solution when asked and one exists
int gm_solve_x(gpbdev_grouped_multi* h, int maxit, double delta, bool warm, int* its) {
  if (gm_pcg(h, 1, h->Zty, h->x, warm && h->has_x, maxit, delta, false, nullptr, nullptr, its)) return -1;
  h->has_x = true;
  return 0;
}

}  // namespace

extern "C" {

int gpbdev_grouped_multi_create(gpbdev_grouped_multi_t* out, int device, int64_t n, int K, const int32_t* level_index, const int* num_levels) {
  if (!out || !level_index || !num_levels) return gfail("gpbdev_grouped_multi_create: null argument");
  if (n <= 0 || K < 2 || K > gmk::kMaxCols) return gfail("gpbdev_grouped_multi_create: need n > 0 and 2 <= K <= 128 grouping factors");
  if (n > INT32_MAX) return gfail("gpbdev_grouped_multi_create: at most 2^31 - 1 observations");
  std::vector<int> cum(K + 1, 0);
  for (int k = 0; k < K; ++k) {
    if (num_levels[k] <= 0) return gfail("gpbdev_grouped_multi_create: every factor needs at least one level");
    if ((int64_t)cum[k] + num_levels[k] > INT32_MAX) return gfail("gpbdev_grouped_multi_create: too many levels");
    cum[k + 1] = cum[k] + num_levels[k];
  }
  const int G = cum[K];
  for (int k = 0; k < K; ++k)
    for (int64_t i = 0; i < n; ++i)
      if (level_index[(size_t)k * n + i] < 0 || level_index[(size_t)k * n + i] >= num_levels[k])
        return gfail("gpbdev_grouped_multi_create: level index out of range");
  // ---- host set-up: level counts, per-factor counting sort (segmented sums of Z_k^T y), pattern of the off-diagonal blocks of
  // Z^T Z with their co-occurrence counts (keys row * G + col of every ordered pair of factors, sorted, run-length counted)
  std::vector<double> cnt(G, 0.);
  std::vector<int32_t> comp(G), offs((size_t)G + K, 0), perm((size_t)K * n);
  for (int k = 0; k < K; ++k) {
    for (int g = cum[k]; g < cum[k + 1]; ++g) comp[g] = k;
    int32_t* o = offs.data() + cum[k] + k;  // factor k: num_levels[k] + 1 offsets
    const int32_t* li = level_index + (size_t)k * n;
    for (int64_t i = 0; i < n; ++i) ++o[li[i] + 1];
    for (int g = 0; g < num_levels[k]; ++g) { cnt[cum[k] + g] = o[g + 1]; o[g + 1] += o[g]; }
    std::vector<int32_t> fill(o, o + num_levels[k]);
    int32_t* pk = perm.data() + (size_t)k * n;
    for (int64_t i = 0; i < n; ++i) pk[fill[li[i]]++] = (int32_t)i;
  }
  std::vector<uint64_t> keys;
  keys.reserve((size_t)K * (K - 1) * n);
  for (int k = 0; k < K; ++k)
    for (int l = 0; l < K; ++l) {
      if (k == l) continue;
      const int32_t* lk = level_index + (size_t)k * n;
      const int32_t* ll = level_index + (size_t)l * n;
      for (int64_t i = 0; i < n; ++i) keys.push_back((uint64_t)(cum[k] + lk[i]) * (uint64_t)G + (uint64_t)(cum[l] + ll[i]));
    }
  std::sort(keys.begin(), keys.end());
  std::vector<int64_t> rp((size_t)G + 1, 0), split(G);
  std::vector<int32_t> col;
  std::vector<double> val;
  for (size_t e = 0; e < keys.size();) {
    size_t f = e;
    while (f < keys.size() && keys[f] == keys[e]) ++f;
    const int r = (int)(keys[e] / (uint64_t)G);
    col.push_back((int32_t)(keys[e] % (uint64_t)G));
    val.push_back((double)(f - e));
    ++rp[r + 1];
    e = f;
  }
  keys.clear(); keys.shrink_to_fit();
  for (int g = 0; g < G; ++g) rp[g + 1] += rp[g];
  for (int g = 0; g < G; ++g) {
    int64_t s = rp[g];
    while (s < rp[g + 1] && col[s] < g) ++s;
    split[g] = s;
  }
  const int64_t nnz = rp[G];
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) {
    cudaGetLastError();
    return gfail("gpbdev_grouped_multi_create: no CUDA device " + std::to_string(device) + " — the CUDA engine has no CPU fallback");
  }
  GCUDA(cudaSetDevice(device));
  gpbdev_grouped_multi* h = new gpbdev_grouped_multi();
  *out = h;  // freed by gpbdev_grouped_multi_free also when a later step fails
  h->device = device; h->n = n; h->K = K; h->G = G; h->cum = cum; h->nnz = nnz; h->rp_host = rp;
  cudaDeviceProp prop;
  GCUDA(cudaGetDeviceProperties(&prop, device));
  h->num_sms = prop.multiProcessorCount;
  GCUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  GCUDA(cudaMalloc(&h->rp, sizeof(int64_t) * (G + 1)));
  GCUDA(cudaMalloc(&h->split, sizeof(int64_t) * G));
  GCUDA(cudaMalloc(&h->col, sizeof(int32_t) * std::max<int64_t>(nnz, 1)));
  GCUDA(cudaMalloc(&h->val, sizeof(double) * std::max<int64_t>(nnz, 1)));
  GCUDA(cudaMalloc(&h->comp, sizeof(int32_t) * G));
  GCUDA(cudaMalloc(&h->idx, sizeof(int32_t) * K * n));
  GCUDA(cudaMalloc(&h->perm, sizeof(int32_t) * K * n));
  GCUDA(cudaMalloc(&h->offs, sizeof(int32_t) * (G + K)));
  double** gvecs[] = {&h->cnt, &h->ones, &h->Mdiag, &h->Dinv, &h->dis, &h->ld, &h->logld, &h->Zty, &h->yy, &h->x, &h->g1, &h->g2};
  for (double** p : gvecs) GCUDA(cudaMalloc(p, sizeof(double) * G));
  GCUDA(cudaMalloc(&h->y, sizeof(double) * n));
  GCUDA(cudaMalloc(&h->yaux, sizeof(double) * n));
  GCUDA(cudaMalloc(&h->dots, sizeof(double) * gmk::kMaxCols));
  GCUDA(cudaMallocHost(&h->dots_host, sizeof(double) * gmk::kMaxCols));
  GCUDA(cudaMallocHost(&h->stage, sizeof(double) * std::max<int64_t>(n, G)));
  if (gm_reserve(h, 1)) return -1;
  std::vector<double> ones(G, 1.);
  GCUDA(cudaMemcpyAsync(h->rp, rp.data(), sizeof(int64_t) * (G + 1), cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->split, split.data(), sizeof(int64_t) * G, cudaMemcpyHostToDevice, h->stream));
  if (nnz > 0) {
    GCUDA(cudaMemcpyAsync(h->col, col.data(), sizeof(int32_t) * nnz, cudaMemcpyHostToDevice, h->stream));
    GCUDA(cudaMemcpyAsync(h->val, val.data(), sizeof(double) * nnz, cudaMemcpyHostToDevice, h->stream));
  }
  GCUDA(cudaMemcpyAsync(h->comp, comp.data(), sizeof(int32_t) * G, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->idx, level_index, sizeof(int32_t) * K * n, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->perm, perm.data(), sizeof(int32_t) * K * n, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->offs, offs.data(), sizeof(int32_t) * (G + K), cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->cnt, cnt.data(), sizeof(double) * G, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->ones, ones.data(), sizeof(double) * G, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

int gpbdev_grouped_multi_free(gpbdev_grouped_multi_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  int64_t* i64[] = {h->rp, h->split};
  for (int64_t* p : i64) cudaFree(p);
  int32_t* i32[] = {h->col, h->comp, h->idx, h->perm, h->offs};
  for (int32_t* p : i32) cudaFree(p);
  double* dv[] = {h->val, h->cnt, h->ones, h->Mdiag, h->Dinv, h->dis, h->ld, h->logld, h->y, h->yaux, h->Zty, h->yy, h->x, h->g1, h->g2,
                  h->R, h->Z, h->H, h->V, h->W, h->U, h->probes, h->UP, h->dots};
  for (double* p : dv) cudaFree(p);
  cudaFreeHost(h->dots_host); cudaFreeHost(h->stage);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

// size of the structure: out[0] = G, out[1] = nnz of the off-diagonal part of Z^T Z
int gpbdev_grouped_multi_info(gpbdev_grouped_multi_t h, int64_t* out2) {
  if (!h || !out2) return gfail("gpbdev_grouped_multi_info: null argument");
  out2[0] = h->G; out2[1] = h->nnz;
  return 0;
}

// Z_k^T y of every factor (segmented sums in the order of the observations inside a level) and y^T y
static int gm_after_y(gpbdev_grouped_multi_t h) {
  for (int k = 0; k < h->K; ++k) {
    group_sums_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->y, h->perm + (size_t)k * h->n, h->offs + h->cum[k] + k, h->cum[k + 1] - h->cum[k],
                                                             h->Zty + h->cum[k], h->yy + h->cum[k]);
    GCUDA(cudaGetLastError());
    h->launches += 1;
  }
  if (gm_dots(h, 0, h->cum[1], 1, h->yy, h->ones, &h->yTy)) return -1;
  h->has_y = true;
  h->state_valid = false;
  return 0;
}

int gpbdev_grouped_multi_set_y(gpbdev_grouped_multi_t h, const double* y_host) {
  if (!h || !y_host) return gfail("gpbdev_grouped_multi_set_y: null argument");
  GCUDA(cudaSetDevice(h->device));
  GCUDA(cudaStreamSynchronize(h->stream));
  std::memcpy(h->stage, y_host, sizeof(double) * h->n);
  GCUDA(cudaMemcpyAsync(h->y, h->stage, sizeof(double) * h->n, cudaMemcpyHostToDevice, h->stream));
  return gm_after_y(h);
}

int gpbdev_grouped_multi_set_y_device(gpbdev_grouped_multi_t h, const double* y_dev) {
  if (!h || !y_dev) return gfail("gpbdev_grouped_multi_set_y_device: null argument");
  GCUDA(cudaSetDevice(h->device));
  GCUDA(cudaMemcpyAsync(h->y, y_dev, sizeof(double) * h->n, cudaMemcpyDeviceToDevice, h->stream));
  return gm_after_y(h);
}

int gpbdev_grouped_multi_set_probes(gpbdev_grouped_multi_t h, const double* probes, int t) {
  if (!h || !probes) return gfail("gpbdev_grouped_multi_set_probes: null argument");
  if (t < 1 || t > gmk::kMaxCols) return gfail("gpbdev_grouped_multi_set_probes: the number of probe vectors must be in [1, 128]");
  GCUDA(cudaSetDevice(h->device));
  GCUDA(cudaStreamSynchronize(h->stream));
  if (gm_reserve(h, t)) return -1;
  std::vector<double> rm((size_t)h->G * t);  // column-major (the reference's probe matrix) -> row-major
  for (int c = 0; c < t; ++c)
    for (int i = 0; i < h->G; ++i) rm[(size_t)i * t + c] = probes[(size_t)c * h->G + i];
  GCUDA(cudaMemcpy(h->probes, rm.data(), sizeof(double) * rm.size(), cudaMemcpyHostToDevice));
  h->t = t;
  h->state_valid = false;
  return 0;
}

// Negative log-likelihood pieces at variance ratios v (K values, sigma_k^2 / sigma^2).
// cfg: 0 cg_max_num_it, 1 cg_max_num_it_tridiag, 2 cg_delta_conv, 3 warm start of M x = Z^T y from the previous solution (0/1).
// out: 0 y^T Psi^-1 y, 1 log|Psi| (SLQ estimate + preconditioner correction + sum_k G_k log v_k), 2 CG iterations of M x = Z^T y,
//      3 CG iterations of the Lanczos block, 4 the SLQ estimate of log|P^-1 M| alone.
int gpbdev_grouped_multi_eval(gpbdev_grouped_multi_t h, const double* v, const double* cfg, double* out) {
  if (!h || !v || !cfg || !out) return gfail("gpbdev_grouped_multi_eval: null argument");
  if (!h->has_y) return gfail("gpbdev_grouped_multi_eval: no response installed (call gpbdev_grouped_multi_set_y first)");
  if (h->t == 0) return gfail("gpbdev_grouped_multi_eval: no probe vectors (call gpbdev_grouped_multi_set_probes first)");
  GCUDA(cudaSetDevice(h->device));
  h->state_valid = false;
  if (gm_set_diag(h, v)) return -1;
  int its = 0, its_tri = 0;
  if (gm_solve_x(h, (int)cfg[0], cfg[2], cfg[3] != 0., &its)) return -1;
  double ztyx;
  if (gm_dots(h, 0, h->G, 1, h->Zty, h->x, &ztyx)) return -1;
  const int t = h->t;
  // u = L D^-1/2 r (N(0, P) probes), then CG with Lanczos from zero: U = M^-1 u (solution_for_trace)
  if (gm_tri<2>(h, 0, h->G, t, h->probes, h->UP)) return -1;
  std::vector<std::vector<double>> Td, Ts;
  if (gm_pcg(h, t, h->UP, h->U, false, (int)cfg[1], cfg[2], true, &Td, &Ts, &its_tri)) return -1;
  double ldet = 0.;
  for (int c = 0; c < t; ++c) ldet += slq::tridiag_e1_log_e1(Td[c], Ts[c]);
  ldet = ldet * (double)h->G / t;
  double sl;
  if (gm_dots(h, 0, h->G, 1, h->logld, h->ones, &sl)) return -1;
  double logdet = ldet + 2. * sl;
  for (int k = 0; k < h->K; ++k) logdet += (double)(h->cum[k + 1] - h->cum[k]) * std::log(v[k]);
  out[0] = h->yTy - ztyx;
  out[1] = logdet;
  out[2] = its;
  out[3] = its_tri;
  out[4] = ldet;
  h->state_valid = true;
  return 0;
}

// Gradient of the negative log-likelihood w.r.t. log v_k at the parameters of the preceding gpbdev_grouped_multi_eval, the error
// variance at sigma2 (CalcGradPars_Only_Grouped_REs_Woodbury_GaussLikelihood_Cluster_i, iterative / SSOR branch):
//   grad_k = -v_k |Z_k^T (y - Z x)|^2 / (2 sigma2) + tr_k / 2, tr_k = stochastic tr(M^-1 dSigma^-1/dlog v_k) with the SSOR control
//   variate + G_k.
int gpbdev_grouped_multi_grad(gpbdev_grouped_multi_t h, double sigma2, double* grad) {
  if (!h || !grad) return gfail("gpbdev_grouped_multi_grad: null argument");
  if (!h->state_valid) return gfail("gpbdev_grouped_multi_grad: run gpbdev_grouped_multi_eval first");
  GCUDA(cudaSetDevice(h->device));
  const int t = h->t, K = h->K, G = h->G;
  // PI = P^-1 u -> Z,  Wd = D^-1 upper(M) PI -> V
  if (gm_precond(h, t, h->UP, h->Z, h->W, nullptr)) return -1;
  if (gm_tri<3>(h, 0, G, t, h->Z, h->V)) return -1;
  // Z^T (y - Z x) = Z^T y - Z^T Z x -> g2
  if (gm_spmm(h, 1, h->cnt, h->x, h->g1)) return -1;
  GCUDA(cudaMemcpyAsync(h->g2, h->Zty, sizeof(double) * G, cudaMemcpyDeviceToDevice, h->stream));
  gmk::Coef one; one.v[0] = 1.;
  gmk::axpy_kernel<<<gm_grid(h, G, 1), gmk::kBlock, 0, h->stream>>>(G, 1, one, nullptr, h->g1, h->g2, nullptr);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  std::vector<double> sUP(t), sPW(t), sWW(t), zA(t), zP(t);
  for (int k = 0; k < K; ++k) {
    const int r0 = h->cum[k], r1 = h->cum[k + 1];
    const double vk = h->v[k], iv = 1. / vk;
    double q, sD;
    if (gm_dots(h, r0, r1, 1, h->g2, h->g2, &q)) return -1;
    if (gm_dots(h, r0, r1, 1, h->Dinv, h->ones, &sD)) return -1;
    if (gm_dots(h, r0, r1, t, h->U, h->Z, sUP.data())) return -1;
    if (gm_dots(h, r0, r1, t, h->Z, h->V, sPW.data())) return -1;
    if (gm_dots(h, r0, r1, t, h->V, h->V, sWW.data())) return -1;
    for (int c = 0; c < t; ++c) {
      zA[c] = -iv * sUP[c];
      zP[c] = -2. * iv * sPW[c] + iv * sWW[c];
    }
    double tr = slq::mean(zA);
    const double trP = slq::mean(zP);
    const double trD = -iv * sD;
    const double copt = slq::optimal_c(zA, zP, tr, trP);
    tr += copt * (trD - trP);
    tr += (double)(r1 - r0);
    grad[k] = -(q * vk) / sigma2 / 2. + tr / 2.;
  }
  return 0;
}

// Psi^-1 y * scale = (y - Z M^-1 Z^T y) * scale at variance ratios v (CalcYAux: one more CG solve, warm-started as cfg[3] says)
// into out (device pointer when out_is_device, else host); cfg as for gpbdev_grouped_multi_eval. *its = CG iterations.
int gpbdev_grouped_multi_yaux(gpbdev_grouped_multi_t h, const double* v, const double* cfg, double scale, double* out, int out_is_device,
                              int* its) {
  if (!h || !v || !cfg || !out) return gfail("gpbdev_grouped_multi_yaux: null argument");
  if (!h->has_y) return gfail("gpbdev_grouped_multi_yaux: no response installed (call gpbdev_grouped_multi_set_y first)");
  GCUDA(cudaSetDevice(h->device));
  h->state_valid = false;
  if (gm_set_diag(h, v)) return -1;
  int it = 0;
  if (gm_solve_x(h, (int)cfg[0], cfg[2], cfg[3] != 0., &it)) return -1;
  if (its) *its = it;
  gmk::Coef cum;
  for (int k = 0; k < h->K; ++k) cum.v[k] = h->cum[k];
  double* dst = out_is_device ? out : h->yaux;
  gmk::yaux_kernel<<<gm_grid(h, h->n, 1), gmk::kBlock, 0, h->stream>>>(h->n, h->K, h->idx, cum, h->x, h->y, scale, dst);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  if (!out_is_device) {
    GCUDA(cudaMemcpyAsync(h->stage, h->yaux, sizeof(double) * h->n, cudaMemcpyDeviceToHost, h->stream));
    GCUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(out, h->stage, sizeof(double) * h->n);
  }
  GCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

// Test hook: one operator at variance ratios v on a host G x t row-major X -> Y:
//   0 M X,  1 P^-1 X (SSOR),  2 L D^-1/2 X (probe map),  3 D^-1 upper(M) X.  Also gives x = M^-1 Z^T y of the last solve (which 4,
//   t = 1, X ignored).
int gpbdev_grouped_multi_apply(gpbdev_grouped_multi_t h, const double* v, int which, const double* X, int t, double* Y) {
  if (!h || !v || !Y || (which != 4 && !X)) return gfail("gpbdev_grouped_multi_apply: null argument");
  if (t < 1 || t > gmk::kMaxCols) return gfail("gpbdev_grouped_multi_apply: t must be in [1, 128]");
  if (t > h->tmax) return gfail("gpbdev_grouped_multi_apply: t exceeds the probe count (call gpbdev_grouped_multi_set_probes first)");
  GCUDA(cudaSetDevice(h->device));
  const size_t len = (size_t)h->G * t;
  if (which == 4) {
    if (!h->has_x) return gfail("gpbdev_grouped_multi_apply: no solve has run");
    GCUDA(cudaMemcpy(Y, h->x, sizeof(double) * h->G, cudaMemcpyDeviceToHost));
    return 0;
  }
  h->state_valid = false;
  if (gm_set_diag(h, v)) return -1;
  GCUDA(cudaMemcpyAsync(h->R, X, sizeof(double) * len, cudaMemcpyHostToDevice, h->stream));
  int rc = 0;
  if (which == 0) rc = gm_spmm(h, t, h->Mdiag, h->R, h->Z);
  else if (which == 1) rc = gm_precond(h, t, h->R, h->Z, h->W, nullptr);
  else if (which == 2) rc = gm_tri<2>(h, 0, h->G, t, h->R, h->Z);
  else if (which == 3) rc = gm_tri<3>(h, 0, h->G, t, h->R, h->Z);
  else return gfail("gpbdev_grouped_multi_apply: unknown operator");
  if (rc) return -1;
  GCUDA(cudaMemcpyAsync(Y, h->Z, sizeof(double) * len, cudaMemcpyDeviceToHost, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

// Bench hook: device time (CUDA events, mean over reps after one warm-up) of one M X and one P^-1 X on the probe block, after an eval.
int gpbdev_grouped_multi_time_ops(gpbdev_grouped_multi_t h, int reps, float* out_ms) {
  if (!h || !out_ms || reps < 1) return gfail("gpbdev_grouped_multi_time_ops: bad argument");
  if (!h->state_valid) return gfail("gpbdev_grouped_multi_time_ops: run gpbdev_grouped_multi_eval first");
  GCUDA(cudaSetDevice(h->device));
  cudaEvent_t e0, e1;
  GCUDA(cudaEventCreate(&e0));
  GCUDA(cudaEventCreate(&e1));
  float acc[2] = {0.f, 0.f};
  for (int r = 0; r < reps + 1; ++r)
    for (int which = 0; which < 2; ++which) {
      GCUDA(cudaEventRecord(e0, h->stream));
      const int rc = which == 0 ? gm_spmm(h, h->t, h->Mdiag, h->UP, h->V) : gm_precond(h, h->t, h->UP, h->Z, h->W, nullptr);
      if (rc) { cudaEventDestroy(e0); cudaEventDestroy(e1); return -1; }
      GCUDA(cudaEventRecord(e1, h->stream));
      GCUDA(cudaEventSynchronize(e1));
      float ms = 0.f;
      GCUDA(cudaEventElapsedTime(&ms, e0, e1));
      if (r > 0) acc[which] += ms;
    }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  h->state_valid = false;  // V, Z and W were overwritten
  out_ms[0] = acc[0] / reps; out_ms[1] = acc[1] / reps;
  return 0;
}

int64_t gpbdev_grouped_multi_launch_count(gpbdev_grouped_multi_t h) { return h ? h->launches : 0; }

}  // extern "C"
