// Device engine for the Vecchia-approximated Gaussian process: C ABI of include/gpboost_b200_dev.h.
// sm_90a (H100) only; there is no CPU fallback (every entry fails loudly without a CUDA device).
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <numeric>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "knn.cuh"
#include "vecchia_factor.cuh"
#include "vecchia_big.cuh"
#include "vecchia_nll2.cuh"

namespace {

thread_local std::string g_last_error;

int fail(const std::string& msg) {
  g_last_error = msg;
  return -1;
}

#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t err__ = (expr);                                                                     \
    if (err__ != cudaSuccess) {                                                                     \
      return fail(std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) + ": " +    \
                  cudaGetErrorString(err__));                                                       \
    }                                                                                               \
  } while (0)

// ---- small kernels around the factor kernel -------------------------------------------------------

// y_ord[i] = y_orig[perm[i]]  (the per-cluster re-ordering SetY does, re_model_template.h:6185-6200)
__global__ void gather_perm_kernel(const double* __restrict__ src, const int32_t* __restrict__ perm,
                                   double* __restrict__ dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = src[perm[i]];
}

// fixed-order reduction of the per-warp partial sums (NACC per row): deterministic for a given grid
template <int NACC = gpb::kNumAcc>
__global__ void reduce_partials_kernel(const double* __restrict__ partials, int64_t nrows, double* __restrict__ out) {
  __shared__ double sh[256];
  for (int k = 0; k < NACC; ++k) {
    double s = 0.;
    for (int64_t r = threadIdx.x; r < nrows; r += blockDim.x) s += partials[r * NACC + k];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[k] = sh[0];
    __syncthreads();
  }
}

// y_aux = B^T u with u = D^-1 B y (CalcYAux, re_model_template.h:9772), gather form over the CSC view of
// B's pattern: one warp per column, deterministic; result scattered back to the original observation order.
__global__ void bt_apply_kernel(const double* __restrict__ A, const double* __restrict__ u,
                                const int32_t* __restrict__ colptr, const int32_t* __restrict__ csc_pos,
                                const int32_t* __restrict__ perm, double* __restrict__ out_orig, int64_t n, int m,
                                int64_t row_begin, int64_t row_end, double scale) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j = warp; j < n; j += nwarps) {
    const int32_t b = colptr[j], e = colptr[j + 1];
    double s = 0.;
    for (int32_t p = b + lane; p < e; p += 32) {
      const int32_t pos = csc_pos[p];
      s -= A[pos] * u[pos / m];
    }
    s = gpb::warp_sum(s);
    if (lane == 0) {
      if (j >= row_begin && j < row_end) s += u[j];  // unit diagonal of B
      out_orig[perm[j]] = s * scale;
    }
  }
}

// dst[order[k]] = src[k]: results of a clustered prediction set (computed cluster by cluster) back to the caller's point order
__global__ void scatter_order_kernel(const double* __restrict__ src, const int32_t* __restrict__ order, double* __restrict__ dst, int64_t n) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) dst[order[k]] = src[k];
}

__global__ void fill_kernel(double* p, int64_t n, double v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// FP64 FMA throughput probe: 8 independent dependent-chains per thread, no memory traffic. Gives the measured
// DFMA peak of this chip that the factor kernel (FP64-pipe bound) is compared against in bench.py.
__global__ void fp64_peak_kernel(double* out, int iters, double a, double b) {
  double x0 = threadIdx.x, x1 = x0 + 1., x2 = x0 + 2., x3 = x0 + 3., x4 = x0 + 4., x5 = x0 + 5., x6 = x0 + 6., x7 = x0 + 7.;
  for (int i = 0; i < iters; ++i) {
    x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b);
    x4 = fma(x4, a, b); x5 = fma(x5, a, b); x6 = fma(x6, a, b); x7 = fma(x7, a, b);
  }
  if (x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7 == 12345.678) out[0] = x0;
}

using FactorKernel = void (*)(const gpb::FactorArgs);

template <int COV, int MODE, int DIM>
FactorKernel pick_cap(int m) {
  if (m <= 10) return gpb::vecchia_factor_kernel<COV, MODE, DIM, 10>;
  if (m <= 20) return gpb::vecchia_factor_kernel<COV, MODE, DIM, 20>;
  // d = 2, 20 < m <= 30: NLL / STORE / GRAD run the two-observation kernel (vecchia_nll2.cuh), so only the factor-derivative
  // modes and the anisotropic gradient are instantiated at this cap
  if constexpr (DIM == 2 && MODE != gpb::MODE_STORE_GRAD && MODE != gpb::MODE_STORE_GRAD2 && MODE != gpb::MODE_GRAD_ANISO) return nullptr;
  else return gpb::vecchia_factor_kernel<COV, MODE, DIM, 30>;
}
template <int COV, int MODE>
FactorKernel pick_dim(int d, int m) {
  return d == 2 ? pick_cap<COV, MODE, 2>(m) : pick_cap<COV, MODE, 0>(m);
}
template <int COV>
FactorKernel pick_mode(int mode, int d, int m) {
  switch (mode) {
    case gpb::MODE_NLL: return pick_dim<COV, gpb::MODE_NLL>(d, m);
    case gpb::MODE_STORE: return pick_dim<COV, gpb::MODE_STORE>(d, m);
    case gpb::MODE_GRAD: return pick_dim<COV, gpb::MODE_GRAD>(d, m);
    case gpb::MODE_STORE_GRAD2: return pick_dim<COV, gpb::MODE_STORE_GRAD2>(d, m);
    case gpb::MODE_GRAD_ANISO: return pick_dim<COV, gpb::MODE_GRAD_ANISO>(d, m);
    default: return pick_dim<COV, gpb::MODE_STORE_GRAD>(d, m);
  }
}
FactorKernel pick_kernel(int cov, int mode, int d, int m) {
  switch (cov) {
    case gpb::COV_EXPONENTIAL: return pick_mode<gpb::COV_EXPONENTIAL>(mode, d, m);
    case gpb::COV_MATERN15: return pick_mode<gpb::COV_MATERN15>(mode, d, m);
    case gpb::COV_MATERN25: return pick_mode<gpb::COV_MATERN25>(mode, d, m);
    default: return pick_mode<gpb::COV_GAUSSIAN>(mode, d, m);
  }
}

using BigKernel = void (*)(const gpb::BigArgs);
template <int COV>
BigKernel pick_big_mode(int mode) {
  switch (mode) {
    case gpb::BIG_NLL: return gpb::vecchia_big_kernel<COV, gpb::BIG_NLL>;
    case gpb::BIG_STORE: return gpb::vecchia_big_kernel<COV, gpb::BIG_STORE>;
    case gpb::BIG_GRAD: return gpb::vecchia_big_kernel<COV, gpb::BIG_GRAD>;
    case gpb::BIG_GRAD_ANISO: return gpb::vecchia_big_kernel<COV, gpb::BIG_GRAD_ANISO>;
    default: return gpb::vecchia_big_kernel<COV, gpb::BIG_PRED>;
  }
}
BigKernel pick_big_kernel(int cov, int mode) {
  switch (cov) {
    case gpb::COV_EXPONENTIAL: return pick_big_mode<gpb::COV_EXPONENTIAL>(mode);
    case gpb::COV_MATERN15: return pick_big_mode<gpb::COV_MATERN15>(mode);
    case gpb::COV_MATERN25: return pick_big_mode<gpb::COV_MATERN25>(mode);
    default: return pick_big_mode<gpb::COV_GAUSSIAN>(mode);
  }
}

}  // namespace

struct gpb_laplace_state;

struct gpbdev_vecchia {
  gpb_laplace_state* lap = nullptr;  // Laplace-Vecchia buffers (laplace.cuh), lazy
  gpbdev_allreduce_fn allreduce = nullptr;  // device collective hook (row-sharded engines)
  void* allreduce_ctx = nullptr;
  int device = 0;
  int64_t n = 0;
  int d = 0, m = 0;
  int64_t row_begin = 0, row_end = 0;
  int num_sms = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  double* coords = nullptr;   // n x d; for anisotropic kernels the coordinates scaled by gpbdev_vecchia_set_coord_scale
  double* coords_orig = nullptr;  // n x d unscaled copy (lazy, first gpbdev_vecchia_set_coord_scale)
  double* partials_aniso = nullptr;  // grid_cap * kWarpsPerBlock x kAnisoAcc (lazy, gpbdev_vecchia_eval_grad_aniso)
  bool nn_searched = true;    // false from gpbdev_vecchia_create_unsearched until the first gpbdev_vecchia_search_neighbors
  int32_t* nn = nullptr;      // n x m
  int32_t* perm = nullptr;    // n
  double* y_in = nullptr;     // n staging (original order)
  double* y = nullptr;        // n ordered
  double* A = nullptr;        // n x m   (lazy)
  double* Dinv = nullptr;     // n       (lazy)
  double* u = nullptr;        // n       (lazy)
  double* dA = nullptr;       // n x m   (lazy, MODE_STORE_GRAD)
  double* dD = nullptr;       // n       (lazy, MODE_STORE_GRAD)
  double* yaux = nullptr;     // n       (lazy, original order)
  int32_t* colptr = nullptr;  // n + 1   (lazy)
  int32_t* csc_pos = nullptr; // nnz     (lazy)
  int32_t* csc_row = nullptr; // nnz     (lazy, Laplace): row of every CSC entry (= csc_pos / m)
  double* A_csc = nullptr;    // nnz     (lazy, Laplace): A in CSC order, refreshed after every latent factorisation
  double* partials = nullptr;
  double* sums = nullptr;     // kNumAcc (device)
  double* sums_host = nullptr;  // pinned
  double* stage_host = nullptr; // pinned n doubles
  double* flush = nullptr;
  int64_t flush_n = 0;
  int grid_cap = 0;
  int64_t partial_rows = 0;   // rows of kNumAcc sums that `partials` holds
  int64_t launches = 0;
  bool factor_stored = false;
  // parameters of the stored factor and of the last pass (whose sums sit in `sums`): a STORE request for exactly this state is
  // already satisfied — the gradient pass of the two-observation kernel writes A, D^-1, u as well once the buffers exist
  int stored_cov = -1, last_cov = -1;
  bool stored_latent = false, last_latent = false;
  double stored_var = 0., stored_range = 0., last_var = 0., last_range = 0.;
  int knn_replayed = 0;  // queries whose neighbour set was re-derived by the exact replay of the reference walk
  std::vector<int32_t> nn_host;  // kept for the lazy CSC build
  // independent realizations (gpbdev_vecchia_create_clusters): cluster c holds the ordered rows [clu_start[c], clu_start[c + 1]);
  // empty for an engine of one realization
  std::vector<int64_t> clu_start;
  // linear regression covariates (covariates.cuh), lazy
  int p = 0;                       // number of covariates
  double* X = nullptr;             // n x p ROW-major, Vecchia order
  double* y0 = nullptr;            // n: y - offset, Vecchia order (the response is the residual y0 - X beta)
  double* gram_partial = nullptr;  // gram_chunks x (p^2 + p)
  double* gram_out = nullptr;      // p^2 + p
  double* quad_partial = nullptr;  // per-warp sums of the residual pass
  int gram_chunks = 0;
};

namespace {

void laplace_release(gpbdev_vecchia* h);  // laplace.cuh

int ensure_store_buffers(gpbdev_vecchia* h) {
  if (h->A) return 0;
  CUDA_TRY(cudaMalloc(&h->A, sizeof(double) * h->n * h->m));
  CUDA_TRY(cudaMalloc(&h->Dinv, sizeof(double) * h->n));
  CUDA_TRY(cudaMalloc(&h->u, sizeof(double) * h->n));
  CUDA_TRY(cudaMemsetAsync(h->A, 0, sizeof(double) * h->n * h->m, h->stream));
  CUDA_TRY(cudaMemsetAsync(h->u, 0, sizeof(double) * h->n, h->stream));
  CUDA_TRY(cudaMemsetAsync(h->Dinv, 0, sizeof(double) * h->n, h->stream));
  return 0;
}

// CSC view of the pattern of B restricted to this shard's rows: for column j the positions i*m+k with nn[i,k]==j
int ensure_csc(gpbdev_vecchia* h) {
  if (h->colptr) return 0;
  const int64_t n = h->n;
  const int m = h->m;
  if (h->nn_host.empty()) {
    h->nn_host.resize((size_t)n * m);
    CUDA_TRY(cudaMemcpy(h->nn_host.data(), h->nn, sizeof(int32_t) * n * m, cudaMemcpyDeviceToHost));
  }
  std::vector<int32_t> colptr(n + 1, 0);
  for (int64_t i = h->row_begin; i < h->row_end; ++i)
    for (int k = 0; k < m; ++k) {
      const int32_t j = h->nn_host[(size_t)i * m + k];
      if (j >= 0) ++colptr[j + 1];
    }
  for (int64_t j = 0; j < n; ++j) colptr[j + 1] += colptr[j];
  std::vector<int32_t> pos((size_t)colptr[n]);
  std::vector<int32_t> fill(colptr.begin(), colptr.end() - 1);
  for (int64_t i = h->row_begin; i < h->row_end; ++i)
    for (int k = 0; k < m; ++k) {
      const int32_t j = h->nn_host[(size_t)i * m + k];
      if (j >= 0) pos[fill[j]++] = (int32_t)(i * m + k);
    }
  CUDA_TRY(cudaMalloc(&h->colptr, sizeof(int32_t) * (n + 1)));
  CUDA_TRY(cudaMalloc(&h->csc_pos, sizeof(int32_t) * std::max<size_t>(pos.size(), 1)));
  CUDA_TRY(cudaMemcpy(h->colptr, colptr.data(), sizeof(int32_t) * (n + 1), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(h->csc_pos, pos.data(), sizeof(int32_t) * pos.size(), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMalloc(&h->yaux, sizeof(double) * n));
  return 0;
}

int launch_eval(gpbdev_vecchia* h, int cov_type, double var, double range, int mode, bool latent = false) {
  if (cov_type < 0 || cov_type > 3) return fail("gpbdev_vecchia_eval: unknown covariance id");
  if (mode < 0 || mode > 3) return fail("gpbdev_vecchia_eval: unknown mode");
  if (!h->nn_searched) return fail("gpbdev_vecchia_eval: the neighbour sets have not been searched (gpbdev_vecchia_search_neighbors)");
  if (!(var > 0.) || !(range > 0.)) return fail("gpbdev_vecchia_eval: covariance parameters must be positive");
  CUDA_TRY(cudaSetDevice(h->device));
  // GPBoost iteration: OptimCovPar's last accepted trial was a gradient pass at the final parameters on this response, and
  // CalcGradient asks for the factor at the same state right after (regression_objective.hpp:164-165): nothing to recompute.
  if (mode == gpb::MODE_STORE && !latent && h->factor_stored && h->stored_cov == cov_type && h->stored_latent == latent &&
      h->stored_var == var && h->stored_range == range && h->last_cov == cov_type && h->last_latent == latent && h->last_var == var &&
      h->last_range == range)
    return 0;
  if (mode == gpb::MODE_STORE || mode == gpb::MODE_STORE_GRAD) {
    if (ensure_store_buffers(h)) return -1;
  }
  h->last_cov = cov_type; h->last_latent = latent; h->last_var = var; h->last_range = range;
  if (mode == gpb::MODE_STORE || mode == gpb::MODE_STORE_GRAD) { h->stored_cov = cov_type; h->stored_latent = latent; h->stored_var = var; h->stored_range = range; }
  if (mode == gpb::MODE_STORE_GRAD && !h->dA) {
    CUDA_TRY(cudaMalloc(&h->dA, sizeof(double) * h->n * h->m));
    CUDA_TRY(cudaMalloc(&h->dD, sizeof(double) * h->n));
    CUDA_TRY(cudaMemsetAsync(h->dA, 0, sizeof(double) * h->n * h->m, h->stream));
    CUDA_TRY(cudaMemsetAsync(h->dD, 0, sizeof(double) * h->n, h->stream));
  }
  gpb::FactorArgs a;
  a.coords = h->coords; a.nn = h->nn; a.y = h->y;
  a.A = h->A; a.Dinv = h->Dinv; a.w = h->u;
  a.partials = h->partials;
  a.n = h->n; a.row_begin = h->row_begin; a.row_end = h->row_end;
  a.m = h->m; a.d = h->d; a.var = var; a.range = range;
  a.diag_nb = latent ? var * (1. + 1e-10) : var + 1.;
  a.diag_obs = latent ? var : var + 1.;
  if (mode == gpb::MODE_STORE_GRAD) {
    CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dA, &h->dA, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dD, &h->dD, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
  }
  if (latent && mode == gpb::MODE_GRAD) return fail("gpbdev_vecchia_eval: the gradient pass assumes a Gaussian likelihood");
  // every pass ends alike: the fixed-order reduction of its `rows` per-warp partial rows into the sums, on row shards the
  // all-reduce of the sums over the ranks on this stream (NCCL kernel), and the record of a stored factor
  auto finish = [&](int64_t rows) -> int {
    CUDA_TRY(cudaGetLastError());
    if (rows > h->partial_rows)
      return fail("gpbdev_vecchia_eval: " + std::to_string(rows) + " partial rows launched, " + std::to_string(h->partial_rows) + " allocated");
    reduce_partials_kernel<<<1, 256, 0, h->stream>>>(h->partials, rows, h->sums);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    if (h->allreduce && !latent) {
      if (h->allreduce(h->allreduce_ctx, h->sums, gpb::kNumAcc, (void*)h->stream)) return fail("gpbdev_vecchia_eval: device all-reduce failed");
    }
    if (mode == gpb::MODE_STORE || mode == gpb::MODE_STORE_GRAD) h->factor_stored = true;
    return 0;
  };
  if (h->m > gpb::kMaxNeighbors) {  // 30 < num_neighbors <= 60: shared-memory kernel (vecchia_big.cuh), same sums and factor layout
    if (mode == gpb::MODE_STORE_GRAD) return fail("gpbdev_vecchia_eval: the factor derivative (non-Gaussian likelihoods) supports num_neighbors <= 30");
    gpb::BigArgs b;
    b.coords = h->coords; b.y = h->y; b.nn = h->nn; b.qcoords = nullptr;
    b.A = h->A; b.Dinv = h->Dinv; b.w = h->u; b.pred_mean = nullptr; b.pred_var = nullptr; b.partials = h->partials;
    b.row_begin = h->row_begin; b.row_end = h->row_end; b.m = h->m; b.d = h->d;
    b.var = var; b.range = range; b.diag_nb = a.diag_nb; b.diag_obs = a.diag_obs;
    const int bmode = mode == gpb::MODE_NLL ? gpb::BIG_NLL : (mode == gpb::MODE_STORE ? gpb::BIG_STORE : gpb::BIG_GRAD);
    const int warps = bmode == gpb::BIG_GRAD ? 2 : 4;
    BigKernel bk = pick_big_kernel(cov_type, bmode);
    const size_t bsmem = gpb::big_smem_bytes(bmode, warps, h->d);
    CUDA_TRY(cudaFuncSetAttribute(bk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
    int grid = std::min(h->num_sms, (int)((h->grid_cap * gpb::kWarpsPerBlock) / warps));  // one CTA per SM; partials has grid_cap * 4 rows
    grid = std::max(grid, 1);
    bk<<<grid, warps * 32, bsmem, h->stream>>>(b);
    return finish((int64_t)grid * warps);
  }
  // likelihood and gradient passes at the headline shape (d = 2, 20 < m <= 30): two observations per warp (vecchia_nll2.cuh)
  if ((mode == gpb::MODE_NLL || mode == gpb::MODE_STORE || (mode == gpb::MODE_GRAD && !latent)) && h->d == 2 && h->m > 20) {
    FactorKernel k2 = nullptr;
#define GPB_PICK2(COVID)                                                                                                              \
    k2 = mode == gpb::MODE_NLL ? gpb::vecchia_nll2_kernel<COVID, gpb::MODE_NLL>                                                      \
         : (mode == gpb::MODE_STORE ? gpb::vecchia_nll2_kernel<COVID, gpb::MODE_STORE> : gpb::vecchia_nll2_kernel<COVID, gpb::MODE_GRAD>)
    switch (cov_type) {
      case gpb::COV_EXPONENTIAL: GPB_PICK2(gpb::COV_EXPONENTIAL); break;
      case gpb::COV_MATERN15: GPB_PICK2(gpb::COV_MATERN15); break;
      case gpb::COV_MATERN25: GPB_PICK2(gpb::COV_MATERN25); break;
      default: GPB_PICK2(gpb::COV_GAUSSIAN); break;
    }
#undef GPB_PICK2
    const size_t smem2 = sizeof(double) * gpb::kWarpsPerBlock * 2 * (gpb::kNll2Half + gpb::kNll2Pts);
    CUDA_TRY(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    CUDA_TRY(cudaFuncSetAttribute(k2, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int per_sm2 = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, k2, gpb::kWarpsPerBlock * 32, smem2));
    int grid2 = std::max(per_sm2, 1) * h->num_sms;
    grid2 = std::max(1, std::min(grid2, h->grid_cap / 2));  // two partial rows per warp
    k2<<<grid2, gpb::kWarpsPerBlock * 32, smem2, h->stream>>>(a);
    if (finish((int64_t)grid2 * gpb::kWarpsPerBlock * 2)) return -1;
    if (mode == gpb::MODE_GRAD && a.A != nullptr) {  // the pass also wrote A, D^-1, u (vecchia_nll2_kernel<GRAD>)
      h->factor_stored = true;
      h->stored_cov = cov_type; h->stored_latent = false; h->stored_var = var; h->stored_range = range;
    }
    return 0;
  }
  FactorKernel k = pick_kernel(cov_type, mode, h->d, h->m);
  if (!k) return fail("gpbdev_vecchia_eval: no one-observation factor kernel for this mode at d = 2, num_neighbors > 20");
  const size_t smem = sizeof(double) * gpb::kWarpsPerBlock * (32 * gpb::kLd + 32 * h->d + 64);
  CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  // persistent grid = resident CTAs per SM (registers / shared memory of this instantiation) x SM count
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, gpb::kWarpsPerBlock * 32, smem));
  int grid = std::max(per_sm, 1) * h->num_sms;
  if (grid > h->grid_cap) grid = h->grid_cap;
  k<<<grid, gpb::kWarpsPerBlock * 32, smem, h->stream>>>(a);
  return finish((int64_t)grid * gpb::kWarpsPerBlock);
}

}  // namespace

extern "C" {

const char* gpbdev_last_error(void) { return g_last_error.c_str(); }

int gpbdev_vecchia_set_allreduce(gpbdev_vecchia_t h, gpbdev_allreduce_fn fn, void* ctx) {
  if (!h) return fail("gpbdev_vecchia_set_allreduce: null argument");
  h->allreduce = fn;
  h->allreduce_ctx = ctx;
  return 0;
}

int gpbdev_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) { cudaGetLastError(); return 0; }
  return c;
}

}  // extern "C"

namespace {

int vecchia_create(gpbdev_vecchia_t* out, int device, int64_t n, int d, int m, const double* coords_ordered, const int32_t* perm,
                   const int32_t* nn, int64_t row_begin, int64_t row_end, bool search, int num_clusters = 0,
                   const int64_t* cluster_start = nullptr) {
  if (!out || !coords_ordered || !perm) return fail("gpbdev_vecchia_create: null argument");
  if (num_clusters > 0) {
    if (!cluster_start || cluster_start[0] != 0 || cluster_start[num_clusters] != n)
      return fail("gpbdev_vecchia_create_clusters: cluster_start must run from 0 to n");
    for (int c = 0; c < num_clusters; ++c)
      if (cluster_start[c + 1] <= cluster_start[c]) return fail("gpbdev_vecchia_create_clusters: every cluster needs at least one row");
  }
  if (n <= 0 || d <= 0 || d > 16) return fail("gpbdev_vecchia_create: need n > 0 and 1 <= dim <= 16");
  if (m < 1 || m > gpb::kBigMaxNeighbors)
    return fail("gpbdev_vecchia_create: num_neighbors must be in [1, " + std::to_string(gpb::kBigMaxNeighbors) +
                "] for the CUDA Vecchia engine");
  if ((int64_t)n * m >= (int64_t)2147483647) return fail("gpbdev_vecchia_create: n * num_neighbors exceeds int32 positions");
  if (row_begin < 0 || row_end > n || row_begin > row_end) return fail("gpbdev_vecchia_create: bad row shard");
  if (nn) {
    // Supplied neighbour sets. The Laplace triangular solves poll the rows a row depends on until they are written, which only
    // ends if every dependency comes earlier in the order: each entry must be -1 (padding) or an earlier row, at most once per row.
    std::vector<int64_t> seen((size_t)n, -1);
    for (int64_t i = 0; i < n; ++i)
      for (int k = 0; k < m; ++k) {
        const int32_t j = nn[i * m + k];
        if (j == -1) continue;
        if (j < -1 || j >= i)
          return fail("gpbdev_vecchia_create: neighbour " + std::to_string(j) + " of row " + std::to_string(i) +
                      " is neither -1 nor an earlier row");
        if (seen[(size_t)j] == i)
          return fail("gpbdev_vecchia_create: neighbour " + std::to_string(j) + " appears twice in row " + std::to_string(i));
        seen[(size_t)j] = i;
      }
  }
  if (gpbdev_device_count() <= device)
    return fail("gpbdev_vecchia_create: no CUDA device " + std::to_string(device) + " — the CUDA engine has no CPU fallback");
  CUDA_TRY(cudaSetDevice(device));
  gpbdev_vecchia* h = new gpbdev_vecchia();
  h->device = device; h->n = n; h->d = d; h->m = m; h->row_begin = row_begin; h->row_end = row_end;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  h->num_sms = prop.multiProcessorCount;
  CUDA_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreate(&h->ev0));
  CUDA_TRY(cudaEventCreate(&h->ev1));
  CUDA_TRY(cudaMalloc(&h->coords, sizeof(double) * n * d));
  CUDA_TRY(cudaMalloc(&h->nn, sizeof(int32_t) * n * m));
  CUDA_TRY(cudaMalloc(&h->perm, sizeof(int32_t) * n));
  CUDA_TRY(cudaMalloc(&h->y_in, sizeof(double) * n));
  CUDA_TRY(cudaMalloc(&h->y, sizeof(double) * n));
  CUDA_TRY(cudaMemset(h->y, 0, sizeof(double) * n));
  // upper bound of the persistent grid (the launch picks resident-CTAs-per-SM x SM count, see launch_eval)
  h->grid_cap = h->num_sms * 8;
  const int64_t rows = row_end - row_begin;
  const int64_t max_blocks = (rows + gpb::kWarpsPerBlock - 1) / gpb::kWarpsPerBlock;
  if (h->grid_cap > max_blocks) h->grid_cap = (int)std::max<int64_t>(max_blocks, 1);
  // the two-observation kernel launches at least one CTA of kWarpsPerBlock warps with two partial rows each, even on a shard of
  // at most kWarpsPerBlock rows (grid_cap = 1)
  h->partial_rows = (int64_t)std::max(h->grid_cap, 2) * gpb::kWarpsPerBlock;
  CUDA_TRY(cudaMalloc(&h->partials, sizeof(double) * h->partial_rows * gpb::kNumAcc));
  CUDA_TRY(cudaMalloc(&h->sums, sizeof(double) * gpb::kNumAcc));
  CUDA_TRY(cudaMallocHost(&h->sums_host, sizeof(double) * gpb::kNumAcc));
  CUDA_TRY(cudaMallocHost(&h->stage_host, sizeof(double) * n));
  CUDA_TRY(cudaMemcpy(h->coords, coords_ordered, sizeof(double) * n * d, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(h->perm, perm, sizeof(int32_t) * n, cudaMemcpyHostToDevice));
  if (nn) {
    CUDA_TRY(cudaMemcpy(h->nn, nn, sizeof(int32_t) * n * m, cudaMemcpyHostToDevice));
    h->nn_host.assign(nn, nn + (size_t)n * m);
  } else if (!search) {
    CUDA_TRY(cudaMemset(h->nn, 0xff, sizeof(int32_t) * n * m));
    h->nn_searched = false;
  } else if (num_clusters > 0) {
    h->clu_start.assign(cluster_start, cluster_start + num_clusters + 1);
    std::string err;
    gpb::KnnInfo info;
    const int nl = gpb::knn_cluster_search(h->coords, coords_ordered, n, n, d, m, m, num_clusters, cluster_start, nullptr, h->nn, h->stream,
                                           h->num_sms, &info, &err);
    if (nl < 0) { gpbdev_vecchia_free(h); return fail("gpbdev_vecchia_create_clusters: device neighbour search failed: " + err); }
    h->launches += nl;
    h->knn_replayed = (int)info.replayed;
  } else {
    std::string err;
    gpb::KnnInfo info;
    const int nl = gpb::knn_vecchia_search(h->coords, coords_ordered, n, d, m, h->nn, h->stream, h->num_sms, &info, &err,
                                           /*q_begin=*/0, /*end_search_at=*/n - 2);
    if (nl < 0) { gpbdev_vecchia_free(h); return fail("gpbdev_vecchia_create: device neighbour search failed: " + err); }
    h->launches += nl;
    h->knn_replayed = (int)info.replayed;
  }
  *out = h;
  return 0;
}

}  // namespace

extern "C" {

int gpbdev_vecchia_create(gpbdev_vecchia_t* out, int device, int64_t n, int d, int m, const double* coords_ordered,
                          const int32_t* perm, const int32_t* nn, int64_t row_begin, int64_t row_end) {
  return vecchia_create(out, device, n, d, m, coords_ordered, perm, nn, row_begin, row_end, true);
}

int gpbdev_vecchia_create_clusters(gpbdev_vecchia_t* out, int device, int64_t n, int d, int m, const double* coords_ordered,
                                   const int32_t* perm, int num_clusters, const int64_t* cluster_start) {
  if (num_clusters < 1) return fail("gpbdev_vecchia_create_clusters: num_clusters must be positive");
  return vecchia_create(out, device, n, d, m, coords_ordered, perm, nullptr, 0, n, true, num_clusters, cluster_start);
}

int gpbdev_vecchia_create_unsearched(gpbdev_vecchia_t* out, int device, int64_t n, int d, int m, const double* coords_ordered,
                                     const int32_t* perm, int64_t row_begin, int64_t row_end) {
  return vecchia_create(out, device, n, d, m, coords_ordered, perm, nullptr, row_begin, row_end, false);
}

int gpbdev_vecchia_free(gpbdev_vecchia_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  laplace_release(h);
  cudaFree(h->coords); cudaFree(h->nn); cudaFree(h->perm); cudaFree(h->y_in); cudaFree(h->y);
  cudaFree(h->dA); cudaFree(h->dD);
  cudaFree(h->A); cudaFree(h->Dinv); cudaFree(h->u); cudaFree(h->yaux); cudaFree(h->colptr); cudaFree(h->csc_pos);
  cudaFree(h->csc_row); cudaFree(h->A_csc);
  cudaFree(h->X); cudaFree(h->y0); cudaFree(h->gram_partial); cudaFree(h->gram_out); cudaFree(h->quad_partial);
  cudaFree(h->partials); cudaFree(h->sums); cudaFree(h->flush);
  cudaFree(h->coords_orig); cudaFree(h->partials_aniso);
  cudaFreeHost(h->sums_host); cudaFreeHost(h->stage_host);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int gpbdev_vecchia_get_nn(gpbdev_vecchia_t h, int32_t* nn_host) {
  if (!h || !nn_host) return fail("gpbdev_vecchia_get_nn: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy(nn_host, h->nn, sizeof(int32_t) * h->n * h->m, cudaMemcpyDeviceToHost));
  return 0;
}

int gpbdev_vecchia_get_perm(gpbdev_vecchia_t h, int32_t* perm_host) {
  if (!h || !perm_host) return fail("gpbdev_vecchia_get_perm: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy(perm_host, h->perm, sizeof(int32_t) * h->n, cudaMemcpyDeviceToHost));
  return 0;
}

int gpbdev_vecchia_set_y_device(gpbdev_vecchia_t h, const double* y_dev) {
  if (!h || !y_dev) return fail("gpbdev_vecchia_set_y_device: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  gather_perm_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(y_dev, h->perm, h->y, h->n);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  h->factor_stored = false;
  return 0;
}

// zero x outside [b, e)
__global__ void zero_outside_range_kernel(double* __restrict__ x, int64_t n, int64_t b, int64_t e) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (i < b || i >= e) x[i] = 0.;
}

int gpbdev_vecchia_set_y(gpbdev_vecchia_t h, const double* y_host) {
  if (!h || !y_host) return fail("gpbdev_vecchia_set_y: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  // Row-sharded engine with the device collective: every rank uploads only ITS slice of the response (the same index range as its
  // row shard, taken over the original order) and the slices are exchanged over NVLink (zero elsewhere + sum all-reduce) instead
  // of N full host-to-device copies of the same vector.
  const bool sliced = h->allreduce != nullptr && (h->row_begin != 0 || h->row_end != h->n);
  const int64_t b = sliced ? h->row_begin : 0, e = sliced ? h->row_end : h->n;
  cudaPointerAttributes attr;
  const bool pinned = cudaPointerGetAttributes(&attr, y_host) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  if (pinned) {  // page-locked caller buffer: DMA straight from it
    CUDA_TRY(cudaMemcpyAsync(h->y_in + b, y_host + b, sizeof(double) * (e - b), cudaMemcpyHostToDevice, h->stream));
  } else {
    // pageable caller memory: stage through the engine's pinned buffer (parallel copy) so the H2D runs at link speed
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    const int64_t len = e - b;
    const int64_t chunk = 1 << 16;
#pragma omp parallel for schedule(static) num_threads(8)
    for (int64_t c = 0; c < (len + chunk - 1) / chunk; ++c) {
      const int64_t lo = b + c * chunk, cl = std::min(chunk, e - lo);
      std::memcpy(h->stage_host + lo, y_host + lo, sizeof(double) * cl);
    }
    CUDA_TRY(cudaMemcpyAsync(h->y_in + b, h->stage_host + b, sizeof(double) * len, cudaMemcpyHostToDevice, h->stream));
  }
  if (sliced) {
    zero_outside_range_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(h->y_in, h->n, b, e);
    CUDA_TRY(cudaGetLastError());
    if (h->allreduce(h->allreduce_ctx, h->y_in, h->n, (void*)h->stream)) return fail("gpbdev_vecchia_set_y: device all-reduce failed");
    h->launches += 1;
  }
  return gpbdev_vecchia_set_y_device(h, h->y_in);
}

int gpbdev_vecchia_eval_async(gpbdev_vecchia_t h, int cov_type, double var, double range, int mode) {
  if (!h) return fail("gpbdev_vecchia_eval: null handle");
  return launch_eval(h, cov_type, var, range, mode);
}

int gpbdev_vecchia_eval(gpbdev_vecchia_t h, int cov_type, double var, double range, int mode, double* out) {
  if (!h || !out) return fail("gpbdev_vecchia_eval: null argument");
  if (launch_eval(h, cov_type, var, range, mode)) return -1;
  return gpbdev_vecchia_last_sums(h, out);
}

int gpbdev_vecchia_last_sums(gpbdev_vecchia_t h, double* out) {
  if (!h || !out) return fail("gpbdev_vecchia_last_sums: null argument");
  CUDA_TRY(cudaMemcpyAsync(h->sums_host, h->sums, sizeof(double) * gpb::kNumAcc, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::memcpy(out, h->sums_host, sizeof(double) * gpb::kNumAcc);
  return 0;
}

int gpbdev_vecchia_yaux(gpbdev_vecchia_t h, double* yaux_host) {
  if (!h || !yaux_host) return fail("gpbdev_vecchia_yaux: null argument");
  if (!h->factor_stored) return fail("gpbdev_vecchia_yaux: call gpbdev_vecchia_eval(mode=STORE) first");
  CUDA_TRY(cudaSetDevice(h->device));
  if (ensure_csc(h)) return -1;
  bt_apply_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->A, h->u, h->colptr, h->csc_pos, h->perm, h->yaux, h->n,
                                                         h->m, h->row_begin, h->row_end, 1.0);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (h->allreduce && h->allreduce(h->allreduce_ctx, h->yaux, h->n, (void*)h->stream)) return fail("gpbdev_vecchia_yaux: device all-reduce failed");
  CUDA_TRY(cudaMemcpyAsync(h->stage_host, h->yaux, sizeof(double) * h->n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::memcpy(yaux_host, h->stage_host, sizeof(double) * h->n);
  return 0;
}

int gpbdev_vecchia_yaux_device(gpbdev_vecchia_t h, double* out_dev, double scale) {
  if (!h || !out_dev) return fail("gpbdev_vecchia_yaux_device: null argument");
  if (!h->factor_stored) return fail("gpbdev_vecchia_yaux_device: call gpbdev_vecchia_eval(mode=STORE) first");
  CUDA_TRY(cudaSetDevice(h->device));
  if (ensure_csc(h)) return -1;
  bt_apply_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->A, h->u, h->colptr, h->csc_pos, h->perm, out_dev, h->n, h->m,
                                                         h->row_begin, h->row_end, scale);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (h->allreduce && h->allreduce(h->allreduce_ctx, out_dev, h->n, (void*)h->stream)) return fail("gpbdev_vecchia_yaux_device: device all-reduce failed");
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

// Vecchia prediction at new locations (SURVEY §8 f1), observed data ordered first, neighbours among the observed points only
// (CalcPredVecchiaObservedFirstOrder, CondObsOnly = true: src/GPBoost/Vecchia_utils.cpp:1701-2100), split into a prediction set
// that is built once per set of locations (coordinates and neighbour sets in HBM) and an evaluation at given parameters.
}  // extern "C"

struct gpbdev_vecchia_predset {
  gpbdev_vecchia_t h = nullptr;
  int64_t np = 0;
  int mp = 0;
  double* qcoords = nullptr;  // np x d row-major
  int32_t* nn = nullptr;      // np x mp, indices into the observed points (Vecchia order)
  double* mean = nullptr;     // np: A_p y_N(p) of the last evaluation
  double* dvar = nullptr;     // np: D_p (transformed scale) of the last evaluation
  // clustered set: the points are searched and evaluated cluster by cluster; order[k] = caller's index of point k, and the kernel
  // writes mean_k / dvar_k before they are scattered to mean / dvar
  int32_t* order = nullptr;
  double* mean_k = nullptr;
  double* dvar_k = nullptr;
};

extern "C" {

int gpbdev_vecchia_predset_create(gpbdev_vecchia_t h, const double* coords_pred_host, int64_t np, int num_neighbors_pred,
                                  gpbdev_vecchia_predset_t* out) {
  if (!h || !coords_pred_host || !out) return fail("gpbdev_vecchia_predict: null argument");
  *out = nullptr;
  if (np <= 0) return fail("gpbdev_vecchia_predict: no prediction points");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_predict: prediction needs the whole model on this device (row-sharded engine)");
  if (!h->clu_start.empty()) return fail("gpbdev_vecchia_predict: an engine of several clusters predicts through gpbdev_vecchia_predset_create_clusters");
  const int64_t n = h->n;
  const int d = h->d;
  int mp = (int)std::min<int64_t>(num_neighbors_pred, n);  // Vecchia_utils.cpp:752-755
  if (mp < 1 || mp > gpb::kBigMaxNeighbors)
    return fail("gpbdev_vecchia_predict: num_neighbors_pred must be in [1, " + std::to_string(gpb::kBigMaxNeighbors) + "] for the CUDA Vecchia engine");
  if ((n + np) >= (int64_t)2147483647 || np * (int64_t)mp >= (int64_t)2147483647) return fail("gpbdev_vecchia_predict: too many points for int32 indices");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  const int64_t na = n + np;
  // all points = observed (Vecchia order) followed by the prediction points; ranks in the sorted coordinate sums decide distance ties
  std::vector<double> call((size_t)na * d);
  CUDA_TRY(cudaMemcpy(call.data(), h->coords, sizeof(double) * n * d, cudaMemcpyDeviceToHost));
  std::memcpy(call.data() + (size_t)n * d, coords_pred_host, sizeof(double) * np * d);
  auto* ps = new gpbdev_vecchia_predset();
  ps->h = h; ps->np = np; ps->mp = mp;
  double* call_dev = nullptr;
  auto release = [&]() { cudaFree(call_dev); gpbdev_vecchia_predset_free(ps); };
  cudaError_t e = cudaMalloc(&call_dev, sizeof(double) * na * d);
  if (e == cudaSuccess) e = cudaMalloc(&ps->nn, sizeof(int32_t) * np * mp);
  if (e == cudaSuccess) e = cudaMalloc(&ps->qcoords, sizeof(double) * np * d);
  if (e == cudaSuccess) e = cudaMalloc(&ps->mean, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMalloc(&ps->dvar, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMemcpy(call_dev, call.data(), sizeof(double) * na * d, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { release(); return fail(std::string("gpbdev_vecchia_predict: ") + cudaGetErrorString(e)); }
  std::string err;
  gpb::KnnInfo info;
  const int nl = gpb::knn_vecchia_search(call_dev, call.data(), na, d, mp, ps->nn, h->stream, h->num_sms, &info, &err,
                                         /*q_begin=*/n, /*end_search_at=*/n - 1);
  if (nl < 0) { release(); return fail("gpbdev_vecchia_predict: device neighbour search failed: " + err); }
  h->launches += nl;
  e = cudaMemcpyAsync(ps->qcoords, call_dev + (size_t)n * d, sizeof(double) * np * d, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(call_dev);
  call_dev = nullptr;
  if (e != cudaSuccess) { release(); return fail(std::string("gpbdev_vecchia_predict: ") + cudaGetErrorString(e)); }
  *out = ps;
  return 0;
}

int gpbdev_vecchia_predset_create_clusters(gpbdev_vecchia_t h, const double* coords_pred_host, int64_t np, int num_neighbors_pred,
                                           const int32_t* cluster_of_pred, gpbdev_vecchia_predset_t* out) {
  if (!h || !coords_pred_host || !cluster_of_pred || !out) return fail("gpbdev_vecchia_predict: null argument");
  *out = nullptr;
  if (np <= 0) return fail("gpbdev_vecchia_predict: no prediction points");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_predict: prediction needs the whole model on this device (row-sharded engine)");
  const int64_t n = h->n;
  const int d = h->d;
  const std::vector<int64_t> obs_start = h->clu_start.empty() ? std::vector<int64_t>{0, n} : h->clu_start;
  const int K = (int)obs_start.size() - 1;
  int64_t max_obs = 0;
  for (int c = 0; c < K; ++c) max_obs = std::max(max_obs, obs_start[c + 1] - obs_start[c]);
  const int mp = (int)std::min<int64_t>(num_neighbors_pred, max_obs);  // Vecchia_utils.cpp:752-755, per cluster in the search
  if (mp < 1 || mp > gpb::kBigMaxNeighbors)
    return fail("gpbdev_vecchia_predict: num_neighbors_pred must be in [1, " + std::to_string(gpb::kBigMaxNeighbors) + "] for the CUDA Vecchia engine");
  if ((n + np) >= (int64_t)2147483647 || np * (int64_t)mp >= (int64_t)2147483647) return fail("gpbdev_vecchia_predict: too many points for int32 indices");
  // points grouped by cluster (cluster order, each cluster's points in the caller's order), points of no cluster (-1) last
  std::vector<int64_t> cnt((size_t)K + 2, 0);
  for (int64_t p = 0; p < np; ++p) {
    const int32_t c = cluster_of_pred[p];
    if (c < -1 || c >= K) return fail("gpbdev_vecchia_predict: cluster index " + std::to_string(c) + " of prediction point " + std::to_string(p) + " outside [-1, " + std::to_string(K) + ")");
    ++cnt[(size_t)(c < 0 ? K : c) + 1];
  }
  for (int c = 0; c <= K; ++c) cnt[(size_t)c + 1] += cnt[(size_t)c];
  std::vector<int64_t> pred_start((size_t)K + 1);
  for (int c = 0; c <= K; ++c) pred_start[(size_t)c] = n + cnt[(size_t)c];
  std::vector<int32_t> order((size_t)np);
  {
    std::vector<int64_t> fill(cnt.begin(), cnt.end() - 1);
    for (int64_t p = 0; p < np; ++p) {
      const int32_t c = cluster_of_pred[p];
      order[(size_t)fill[(size_t)(c < 0 ? K : c)]++] = (int32_t)p;
    }
  }
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  const int64_t na = n + np;
  std::vector<double> call((size_t)na * d);
  CUDA_TRY(cudaMemcpy(call.data(), h->coords, sizeof(double) * n * d, cudaMemcpyDeviceToHost));
  for (int64_t k = 0; k < np; ++k)
    std::memcpy(call.data() + (size_t)(n + k) * d, coords_pred_host + (size_t)order[(size_t)k] * d, sizeof(double) * d);
  auto* ps = new gpbdev_vecchia_predset();
  ps->h = h; ps->np = np; ps->mp = mp;
  double* call_dev = nullptr;
  auto release = [&]() { cudaFree(call_dev); gpbdev_vecchia_predset_free(ps); };
  cudaError_t e = cudaMalloc(&call_dev, sizeof(double) * na * d);
  if (e == cudaSuccess) e = cudaMalloc(&ps->nn, sizeof(int32_t) * np * mp);
  if (e == cudaSuccess) e = cudaMalloc(&ps->qcoords, sizeof(double) * np * d);
  if (e == cudaSuccess) e = cudaMalloc(&ps->mean, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMalloc(&ps->dvar, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMalloc(&ps->mean_k, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMalloc(&ps->dvar_k, sizeof(double) * np);
  if (e == cudaSuccess) e = cudaMalloc(&ps->order, sizeof(int32_t) * np);
  if (e == cudaSuccess) e = cudaMemcpy(ps->order, order.data(), sizeof(int32_t) * np, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(call_dev, call.data(), sizeof(double) * na * d, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { release(); return fail(std::string("gpbdev_vecchia_predict: ") + cudaGetErrorString(e)); }
  std::string err;
  gpb::KnnInfo info;
  const int nl = gpb::knn_cluster_search(call_dev, call.data(), na, n, d, mp, num_neighbors_pred, K, obs_start.data(), pred_start.data(),
                                         ps->nn, h->stream, h->num_sms, &info, &err);
  if (nl < 0) { release(); return fail("gpbdev_vecchia_predict: device neighbour search failed: " + err); }
  h->launches += nl;
  e = cudaMemcpyAsync(ps->qcoords, call_dev + (size_t)n * d, sizeof(double) * np * d, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(call_dev);
  call_dev = nullptr;
  if (e != cudaSuccess) { release(); return fail(std::string("gpbdev_vecchia_predict: ") + cudaGetErrorString(e)); }
  *out = ps;
  return 0;
}

int gpbdev_vecchia_predset_eval(gpbdev_vecchia_predset_t ps, int cov_type, double var, double range, const double** mean_dev,
                                const double** var_dev) {
  if (!ps || !ps->h) return fail("gpbdev_vecchia_predset_eval: null argument");
  if (cov_type < 0 || cov_type > 3) return fail("gpbdev_vecchia_predict: unknown covariance id");
  if (!(var > 0.) || !(range > 0.)) return fail("gpbdev_vecchia_predict: covariance parameters must be positive");
  gpbdev_vecchia_t h = ps->h;
  const int d = h->d;
  CUDA_TRY(cudaSetDevice(h->device));
  gpb::BigArgs b;
  b.coords = h->coords; b.y = h->y; b.nn = ps->nn; b.qcoords = ps->qcoords;
  b.A = nullptr; b.Dinv = nullptr; b.w = nullptr; b.partials = nullptr;
  b.pred_mean = ps->order ? ps->mean_k : ps->mean; b.pred_var = ps->order ? ps->dvar_k : ps->dvar;
  b.row_begin = 0; b.row_end = ps->np; b.m = ps->mp; b.d = d;
  b.var = var; b.range = range; b.diag_nb = var + 1.; b.diag_obs = var;  // Vecchia_utils.cpp:1940-1952 (nugget on the neighbour block), :1925-1931
  BigKernel bk = pick_big_kernel(cov_type, gpb::BIG_PRED);
  const size_t bsmem = gpb::big_smem_bytes(gpb::BIG_PRED, 4, d);
  CUDA_TRY(cudaFuncSetAttribute(bk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(h->num_sms, (ps->np + 3) / 4));
  bk<<<grid, 128, bsmem, h->stream>>>(b);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (ps->order) {  // rows of a point without observed neighbours are all -1: mean 0 and D_p = var, the prior
    const int sg = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)h->num_sms * 4, (ps->np + 255) / 256));
    scatter_order_kernel<<<sg, 256, 0, h->stream>>>(ps->mean_k, ps->order, ps->mean, ps->np);
    scatter_order_kernel<<<sg, 256, 0, h->stream>>>(ps->dvar_k, ps->order, ps->dvar, ps->np);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
  }
  CUDA_TRY(cudaStreamSynchronize(h->stream));  // the results are read on other streams (the booster's metric kernel) or copied out
  if (mean_dev) *mean_dev = ps->mean;
  if (var_dev) *var_dev = ps->dvar;
  return 0;
}

int gpbdev_vecchia_predset_free(gpbdev_vecchia_predset_t ps) {
  if (!ps) return 0;
  if (ps->h) cudaSetDevice(ps->h->device);
  cudaFree(ps->qcoords); cudaFree(ps->nn); cudaFree(ps->mean); cudaFree(ps->dvar);
  cudaFree(ps->order); cudaFree(ps->mean_k); cudaFree(ps->dvar_k);
  delete ps;
  return 0;
}

int gpbdev_vecchia_predict(gpbdev_vecchia_t h, int cov_type, double var, double range, const double* coords_pred_host, int64_t np,
                           int num_neighbors_pred, double* mean_out_host, double* var_out_host) {
  return gpbdev_vecchia_predict_clusters(h, cov_type, var, range, coords_pred_host, np, num_neighbors_pred, nullptr, mean_out_host,
                                         var_out_host);
}

int gpbdev_vecchia_predict_clusters(gpbdev_vecchia_t h, int cov_type, double var, double range, const double* coords_pred_host, int64_t np,
                                    int num_neighbors_pred, const int32_t* cluster_of_pred, double* mean_out_host, double* var_out_host) {
  if (!h || !coords_pred_host || !mean_out_host || !var_out_host) return fail("gpbdev_vecchia_predict: null argument");
  if (np <= 0) return fail("gpbdev_vecchia_predict: no prediction points");
  if (cov_type < 0 || cov_type > 3) return fail("gpbdev_vecchia_predict: unknown covariance id");
  if (!(var > 0.) || !(range > 0.)) return fail("gpbdev_vecchia_predict: covariance parameters must be positive");
  gpbdev_vecchia_predset_t ps = nullptr;
  if (cluster_of_pred ? gpbdev_vecchia_predset_create_clusters(h, coords_pred_host, np, num_neighbors_pred, cluster_of_pred, &ps)
                      : gpbdev_vecchia_predset_create(h, coords_pred_host, np, num_neighbors_pred, &ps)) return -1;
  const double *mean_dev = nullptr, *var_dev = nullptr;
  if (gpbdev_vecchia_predset_eval(ps, cov_type, var, range, &mean_dev, &var_dev)) { gpbdev_vecchia_predset_free(ps); return -1; }
  cudaError_t e = cudaMemcpy(mean_out_host, mean_dev, sizeof(double) * np, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(var_out_host, var_dev, sizeof(double) * np, cudaMemcpyDeviceToHost);
  gpbdev_vecchia_predset_free(ps);
  if (e != cudaSuccess) return fail(std::string("gpbdev_vecchia_predict: ") + cudaGetErrorString(e));
  return 0;
}

// latent factor (non-Gaussian likelihood: no nugget, jitter on the neighbour blocks) with its range derivative, to host buffers:
// A, dA n x m row-major; Dinv, dD n. Test / diagnostics entry of MODE_STORE_GRAD.

int gpbdev_vecchia_latent_factor_grad(gpbdev_vecchia_t h, int cov_type, double var, double range, double* A_host, double* Dinv_host,
                                      double* dA_host, double* dD_host) {
  if (!h || !A_host || !Dinv_host || !dA_host || !dD_host) return fail("gpbdev_vecchia_latent_factor_grad: null argument");
  if (launch_eval(h, cov_type, var, range, gpb::MODE_STORE_GRAD, true)) return -1;
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy(A_host, h->A, sizeof(double) * h->n * h->m, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(Dinv_host, h->Dinv, sizeof(double) * h->n, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(dA_host, h->dA, sizeof(double) * h->n * h->m, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(dD_host, h->dD, sizeof(double) * h->n, cudaMemcpyDeviceToHost));
  return 0;
}

int gpbdev_vecchia_get_factor(gpbdev_vecchia_t h, double* A_host, double* Dinv_host) {
  if (!h || !A_host || !Dinv_host) return fail("gpbdev_vecchia_get_factor: null argument");
  if (!h->factor_stored) return fail("gpbdev_vecchia_get_factor: call gpbdev_vecchia_eval(mode=STORE) first");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy(A_host, h->A, sizeof(double) * h->n * h->m, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(Dinv_host, h->Dinv, sizeof(double) * h->n, cudaMemcpyDeviceToHost));
  return 0;
}

int gpbdev_vecchia_timer_start(gpbdev_vecchia_t h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
  return 0;
}
int gpbdev_vecchia_timer_stop(gpbdev_vecchia_t h, float* ms) {
  if (!h || !ms) return fail("null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(cudaEventSynchronize(h->ev1));
  CUDA_TRY(cudaEventElapsedTime(ms, h->ev0, h->ev1));
  return 0;
}
int gpbdev_vecchia_sync(gpbdev_vecchia_t h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}
// ---- anisotropic kernels (ARD / space-time): scaled coordinates, neighbour sets searched in the scaled space, per-group gradient

}  // extern "C"

namespace {

struct CoordScale {
  double s[16];
};

// dst = src * s[column], one rounded multiply per entry: the same single operation as the host's scaling, so both agree bitwise
__global__ void scale_coords_kernel(const double* __restrict__ src, double* __restrict__ dst, int64_t n, int d, CoordScale s) {
  const int64_t nd = n * d;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nd; e += (int64_t)gridDim.x * blockDim.x)
    dst[e] = __dmul_rn(src[e], s.s[e % d]);
}

// every view derived from the parameters or the neighbour sets is stale: the STORE shortcut, the stored factor, the CSC pattern
void drop_factor_state(gpbdev_vecchia* h) {
  h->factor_stored = false;
  h->stored_cov = -1; h->last_cov = -1;
}

}  // namespace

extern "C" {

int gpbdev_vecchia_set_coord_scale(gpbdev_vecchia_t h, const double* scale) {
  if (!h || !scale) return fail("gpbdev_vecchia_set_coord_scale: null argument");
  CoordScale cs;
  for (int k = 0; k < 16; ++k) cs.s[k] = k < h->d ? scale[k] : 0.;
  for (int k = 0; k < h->d; ++k)
    if (!(cs.s[k] > 0.) || !std::isfinite(cs.s[k])) return fail("gpbdev_vecchia_set_coord_scale: scale factors must be positive and finite");
  CUDA_TRY(cudaSetDevice(h->device));
  if (!h->coords_orig) {
    CUDA_TRY(cudaMalloc(&h->coords_orig, sizeof(double) * h->n * h->d));
    CUDA_TRY(cudaMemcpyAsync(h->coords_orig, h->coords, sizeof(double) * h->n * h->d, cudaMemcpyDeviceToDevice, h->stream));
  }
  scale_coords_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->coords_orig, h->coords, h->n, h->d, cs);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  drop_factor_state(h);
  return 0;
}

int gpbdev_vecchia_search_neighbors(gpbdev_vecchia_t h) {
  if (!h) return fail("gpbdev_vecchia_search_neighbors: null handle");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_search_neighbors: needs the whole model on this device");
  if (!h->clu_start.empty()) return fail("gpbdev_vecchia_search_neighbors: not supported for an engine of several clusters");
  CUDA_TRY(cudaSetDevice(h->device));
  std::vector<double> ch((size_t)h->n * h->d);  // the search replays ties on the host copy of the same coordinates
  CUDA_TRY(cudaMemcpyAsync(ch.data(), h->coords, sizeof(double) * h->n * h->d, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::string err;
  gpb::KnnInfo info;
  const int nl = gpb::knn_vecchia_search(h->coords, ch.data(), h->n, h->d, h->m, h->nn, h->stream, h->num_sms, &info, &err,
                                         /*q_begin=*/0, /*end_search_at=*/h->n - 2);
  if (nl < 0) return fail("gpbdev_vecchia_search_neighbors: device neighbour search failed: " + err);
  h->launches += nl;
  h->knn_replayed = (int)info.replayed;
  h->nn_searched = true;
  // views of the old sets: host copy, CSC pattern (and the buffers built with it), Laplace state
  h->nn_host.clear();
  cudaFree(h->colptr); cudaFree(h->csc_pos); cudaFree(h->yaux); cudaFree(h->csc_row); cudaFree(h->A_csc);
  h->colptr = nullptr; h->csc_pos = nullptr; h->yaux = nullptr; h->csc_row = nullptr; h->A_csc = nullptr;
  laplace_release(h);
  drop_factor_state(h);
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int gpbdev_vecchia_eval_grad_aniso(gpbdev_vecchia_t h, int cov_type, double var, const int32_t* group_of_coord, int ngroups,
                                   double* out) {
  if (!h || !group_of_coord || !out) return fail("gpbdev_vecchia_eval_grad_aniso: null argument");
  if (cov_type < 0 || cov_type > 3) return fail("gpbdev_vecchia_eval_grad_aniso: unknown covariance id");
  if (!(var > 0.)) return fail("gpbdev_vecchia_eval_grad_aniso: covariance parameters must be positive");
  if (ngroups < 1 || ngroups > gpb::kMaxAnisoGroups) return fail("gpbdev_vecchia_eval_grad_aniso: need 1 <= number of groups <= 16");
  if (!h->nn_searched) return fail("gpbdev_vecchia_eval_grad_aniso: the neighbour sets have not been searched (gpbdev_vecchia_search_neighbors)");
  unsigned mask[gpb::kMaxAnisoGroups] = {0u};
  for (int k = 0; k < h->d; ++k) {
    if (group_of_coord[k] < 0 || group_of_coord[k] >= ngroups) return fail("gpbdev_vecchia_eval_grad_aniso: coordinate group out of range");
    mask[group_of_coord[k]] |= 1u << k;
  }
  CUDA_TRY(cudaSetDevice(h->device));
  const int64_t rows_cap = (int64_t)h->grid_cap * gpb::kWarpsPerBlock;
  if (!h->partials_aniso)  // partial rows, then the reduced sums
    CUDA_TRY(cudaMalloc(&h->partials_aniso, sizeof(double) * (rows_cap + 1) * gpb::kAnisoAcc));
  double* sums = h->partials_aniso + rows_cap * gpb::kAnisoAcc;
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_aniso_ngroups, &ngroups, sizeof(int), 0, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_aniso_mask, mask, sizeof(mask), 0, cudaMemcpyHostToDevice, h->stream));
  const double range = 1.;  // the isotropic closed form at unit range on the scaled coordinates
  int64_t rows = 0;
  if (h->m > gpb::kMaxNeighbors) {
    gpb::BigArgs b;
    b.coords = h->coords; b.y = h->y; b.nn = h->nn; b.qcoords = nullptr;
    b.A = nullptr; b.Dinv = nullptr; b.w = nullptr; b.pred_mean = nullptr; b.pred_var = nullptr; b.partials = h->partials_aniso;
    b.row_begin = h->row_begin; b.row_end = h->row_end; b.m = h->m; b.d = h->d;
    b.var = var; b.range = range; b.diag_nb = var + 1.; b.diag_obs = var + 1.;
    const int warps = 2;
    BigKernel bk = pick_big_kernel(cov_type, gpb::BIG_GRAD_ANISO);
    const size_t bsmem = gpb::big_smem_bytes(gpb::BIG_GRAD_ANISO, warps, h->d);
    CUDA_TRY(cudaFuncSetAttribute(bk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
    int grid = std::max(1, std::min(h->num_sms, (int)(rows_cap / warps)));
    bk<<<grid, warps * 32, bsmem, h->stream>>>(b);
    rows = (int64_t)grid * warps;
  } else {
    gpb::FactorArgs a;
    a.coords = h->coords; a.nn = h->nn; a.y = h->y;
    a.A = nullptr; a.Dinv = nullptr; a.w = nullptr;
    a.partials = h->partials_aniso;
    a.n = h->n; a.row_begin = h->row_begin; a.row_end = h->row_end;
    a.m = h->m; a.d = h->d; a.var = var; a.range = range;
    a.diag_nb = var + 1.; a.diag_obs = var + 1.;
    FactorKernel k = pick_kernel(cov_type, gpb::MODE_GRAD_ANISO, h->d, h->m);
    if (!k) return fail("gpbdev_vecchia_eval_grad_aniso: no factor kernel for this shape");
    const size_t smem = sizeof(double) * gpb::kWarpsPerBlock * (32 * gpb::kLd + 32 * h->d + 64);
    CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, gpb::kWarpsPerBlock * 32, smem));
    int grid = std::min(std::max(per_sm, 1) * h->num_sms, h->grid_cap);
    k<<<grid, gpb::kWarpsPerBlock * 32, smem, h->stream>>>(a);
    rows = (int64_t)grid * gpb::kWarpsPerBlock;
  }
  CUDA_TRY(cudaGetLastError());
  reduce_partials_kernel<gpb::kAnisoAcc><<<1, 256, 0, h->stream>>>(h->partials_aniso, rows, sums);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  const int nout = 3 + 3 * (1 + ngroups);
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  CUDA_TRY(cudaMemcpy(out, sums, sizeof(double) * nout, cudaMemcpyDeviceToHost));
  return 0;
}

int64_t gpbdev_vecchia_launch_count(gpbdev_vecchia_t h) { return h ? h->launches : 0; }
int gpbdev_vecchia_knn_replayed(gpbdev_vecchia_t h) { return h ? h->knn_replayed : 0; }

int gpbdev_knn_search(int device, const double* coords_host, int64_t n, int d, int m, int64_t q_begin, int64_t end_search_at,
                      int32_t* nn_host, int64_t* info_out) {
  if (!coords_host || !nn_host || !info_out) return fail("gpbdev_knn_search: null argument");
  if (d < 1) return fail("gpbdev_knn_search: need dim >= 1");
  if (m < 1 || m > gpb::kBigMaxNeighbors)
    return fail("gpbdev_knn_search: num_neighbors must be in [1, " + std::to_string(gpb::kBigMaxNeighbors) + "]");
  if (n < 1 || n >= (int64_t)2147483647) return fail("gpbdev_knn_search: need 1 <= n < 2^31");
  if (q_begin < 0 || q_begin >= n) return fail("gpbdev_knn_search: q_begin must be in [0, n)");
  if (end_search_at != (q_begin == 0 ? n - 2 : q_begin - 1))
    return fail("gpbdev_knn_search: end_search_at must be n - 2 for model queries (q_begin = 0) and q_begin - 1 for prediction");
  m = (int)std::min<int64_t>(m, end_search_at + 1);  // Vecchia_utils.cpp:752-755
  if (m < 1) return fail("gpbdev_knn_search: model queries need n >= 2");
  const int64_t nq = n - q_begin;
  if (nq * m >= (int64_t)2147483647) return fail("gpbdev_knn_search: n * num_neighbors exceeds int32 positions");
  if (gpbdev_device_count() <= device) return fail("gpbdev_knn_search: no CUDA device " + std::to_string(device));
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  cudaStream_t stream = nullptr;
  double* coords_dev = nullptr;
  int32_t* nn_dev = nullptr;
  CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  auto release = [&]() { cudaFree(coords_dev); cudaFree(nn_dev); cudaStreamDestroy(stream); };
  cudaError_t e = cudaMalloc(&coords_dev, sizeof(double) * n * d);
  if (e == cudaSuccess) e = cudaMalloc(&nn_dev, sizeof(int32_t) * nq * m);
  if (e == cudaSuccess) e = cudaMemcpy(coords_dev, coords_host, sizeof(double) * n * d, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { release(); return fail(std::string("gpbdev_knn_search: ") + cudaGetErrorString(e)); }
  std::string err;
  gpb::KnnInfo info;
  if (gpb::knn_vecchia_search(coords_dev, coords_host, n, d, m, nn_dev, stream, prop.multiProcessorCount, &info, &err, q_begin,
                              end_search_at) < 0) {
    release();
    return fail("gpbdev_knn_search: " + err);
  }
  e = cudaMemcpy(nn_host, nn_dev, sizeof(int32_t) * nq * m, cudaMemcpyDeviceToHost);
  release();
  if (e != cudaSuccess) return fail(std::string("gpbdev_knn_search: ") + cudaGetErrorString(e));
  const int64_t vals[7] = {info.replayed, info.launches, info.brute_end, info.ncell, info.g[0], info.g[1], info.g[2]};
  std::memcpy(info_out, vals, sizeof(vals));
  return 0;
}

int gpbdev_fp64_peak(int device, double* tflops) {
  if (!tflops) return fail("null argument");
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  double* out = nullptr;
  CUDA_TRY(cudaMalloc(&out, 8));
  cudaEvent_t e0, e1;
  CUDA_TRY(cudaEventCreate(&e0));
  CUDA_TRY(cudaEventCreate(&e1));
  const int blocks = prop.multiProcessorCount * 8, threads = 256, iters = 1 << 14;
  fp64_peak_kernel<<<blocks, threads>>>(out, 1 << 10, 1.0000001, 1e-9);
  double best = 0.;
  for (int rep = 0; rep < 5; ++rep) {
    CUDA_TRY(cudaEventRecord(e0));
    fp64_peak_kernel<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9);
    CUDA_TRY(cudaEventRecord(e1));
    CUDA_TRY(cudaEventSynchronize(e1));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
    const double flops = 2.0 * 8 * (double)iters * blocks * threads;
    best = std::max(best, flops / (ms * 1e-3) / 1e12);
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  *tflops = best;
  return 0;
}

int gpbdev_vecchia_flush_l2(gpbdev_vecchia_t h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  if (!h->flush) {
    h->flush_n = (int64_t)(256 << 20) / sizeof(double);  // 256 MiB > the 50 MB L2 of an H100
    CUDA_TRY(cudaMalloc(&h->flush, sizeof(double) * h->flush_n));
  }
  fill_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->flush, h->flush_n, 1.0);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // extern "C"

#include "newton.cuh"
#include "covariates.cuh"
#include "laplace.cuh"
#include "fisher.cuh"
