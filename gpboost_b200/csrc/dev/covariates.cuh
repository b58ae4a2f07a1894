// Linear regression coefficients (covariates X, n x p) of the Gaussian Vecchia model, profiled out by GLS in every likelihood
// evaluation. Included at the end of dev_api.cu (shares the engine struct and the stored factor).
//
// Replaces ProfileOutCoef / UpdateCoefGLS (include/GPBoost/re_model_template.h:2665-2683, :10012-10019) for a Vecchia factor
// Psi^-1 = B^T D^-1 B (transformed scale):
//   * Gram pass, after a STORE pass at theta: per ordered row i, w_i = (B X)_i = X_i - sum_k A_ik X_nn(i,k) (p values) and
//     b_i = (B y0)_i with y0 = y - offset; G = sum D^-1_i w_i w_i^T (= X^T Psi^-1 X), r = sum D^-1_i w_i b_i (= X^T Psi^-1 y0).
//     One CTA per chunk of consecutive rows keeps its share of G in registers (a T x T tile of the lower triangle per thread);
//     chunk partials are summed in chunk order, so two calls give bitwise the same G and r. Only G and r leave the device.
//     B y0 is formed here from the resident y0 with the same gathers as B X, so the pass does not depend on which response the
//     STORE pass saw (between evaluations the engine's response is the residual of the previous coefficients).
//   * Residual pass, given beta: y_r = y0 - X beta becomes the engine's response (Vecchia order), then u = D^-1 B y_r,
//     y_r^T Psi^-1 y_r and log|Psi| from the resident A, D^-1. No covariance evaluation, no factorisation. The quadratic form is
//     summed from y_r directly, not assembled from an augmented Gram of [y0 X] (that cancels catastrophically when the mean is
//     large against the noise).
// HBM traffic of the Gram pass per row: A and nn (12 m B), D^-1 and y0 (16 B), the row's own X (8 p B), and the neighbours' X rows
// and y0 values (8 (p + 1) m B when none of them is reused from L2).
namespace gpc {

constexpr int kThreads = 256;   // 16 x 16 threads own the register tiles of G
constexpr int kWarps = kThreads / 32;
constexpr int kRows = 32;       // rows per batch: each warp forms the w rows of kRows / kWarps observations
constexpr int kRowsPerWarp = kRows / kWarps;
constexpr int kMaxP = 64;

struct ResidualArgs {
  double beta[kMaxP];
};

// partial[chunk][p*p + p]: lower triangle of G (row-major, a >= b) then r
template <int T>
__global__ void __launch_bounds__(kThreads, 2) gls_gram_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn,
                                                            const double* __restrict__ Dinv, const double* __restrict__ X,
                                                            const double* __restrict__ y0, int64_t n, int m, int p, int P,
                                                            int64_t rows_per_chunk, double* __restrict__ partial) {
  extern __shared__ double sm[];
  double* ws = sm;                          // kRows x p : w
  double* wds = sm + kRows * p;             // kRows x p : D^-1 w
  double* us = sm + 2 * kRows * p;          // kRows     : D^-1 b
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const int ty = tid / 16, tx = tid % 16;
  const bool tile_live = tx * T <= ty * T + T - 1 && ty * T < p;  // tile touches the lower triangle
  double acc[T][T];
#pragma unroll
  for (int a = 0; a < T; ++a)
#pragma unroll
    for (int b = 0; b < T; ++b) acc[a][b] = 0.;
  double racc = 0.;
  // lane = s * P + c: column c (and c + 32 when p > 32), neighbour slice s of S = 32 / P
  const int S = 32 / P, s = lane / P, c = lane % P;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_chunk, r1 = min(r0 + rows_per_chunk, n);
  for (int64_t base = r0; base < r1; base += kRows) {
    // the warp's kRowsPerWarp rows are gathered together: their neighbour loads are independent, so several rows' gathers are in
    // flight at once. Padding (-1) and rows past the chunk gather row r0 (always valid) with weight 0.
    int64_t ir[kRowsPerWarp];
    bool live[kRowsPerWarp];
    double x0[kRowsPerWarp], x1[kRowsPerWarp], xb[kRowsPerWarp];
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
      const int64_t i = base + wp + q * kWarps;
      live[q] = i < r1;
      ir[q] = live[q] ? i : r0;
      x0[q] = 0.; x1[q] = 0.; xb[q] = 0.;
    }
#pragma unroll 1
    for (int k = s; k < m; k += S) {
      int32_t j[kRowsPerWarp];
      double a[kRowsPerWarp];
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q) {
        const int32_t jq = nn[ir[q] * m + k];
        a[q] = (live[q] && jq >= 0) ? A[ir[q] * m + k] : 0.;
        j[q] = jq >= 0 ? jq : 0;
      }
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q) {
        const double* Xj = X + (int64_t)j[q] * p;
        if (c < p) x0[q] = fma(a[q], Xj[c], x0[q]);
        if (c + 32 < p) x1[q] = fma(a[q], Xj[c + 32], x1[q]);
        xb[q] = fma(a[q], y0[j[q]], xb[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
      // sum over the neighbour slices (fixed butterfly: the same on every call)
      for (int o = P; o < 32; o <<= 1) {
        x0[q] += __shfl_xor_sync(0xffffffffu, x0[q], o);
        x1[q] += __shfl_xor_sync(0xffffffffu, x1[q], o);
        xb[q] += __shfl_xor_sync(0xffffffffu, xb[q], o);
      }
      const int rr = wp + q * kWarps;
      const int64_t i = ir[q];
      if (s == 0) {
        const double di = live[q] ? Dinv[i] : 0.;
        const double* Xi = X + i * p;
        if (c < p) {
          const double w = live[q] ? Xi[c] - x0[q] : 0.;
          ws[rr * p + c] = w;
          wds[rr * p + c] = di * w;
        }
        if (c + 32 < p) {
          const double w = live[q] ? Xi[c + 32] - x1[q] : 0.;
          ws[rr * p + c + 32] = w;
          wds[rr * p + c + 32] = di * w;
        }
        if (c == 0) us[rr] = live[q] ? di * (y0[i] - xb[q]) : 0.;
      }
    }
    __syncthreads();
    if (tile_live) {
#pragma unroll 4
      for (int rr = 0; rr < kRows; ++rr) {
        double va[T], vb[T];
#pragma unroll
        for (int t = 0; t < T; ++t) {
          const int a = ty * T + t, b = tx * T + t;
          va[t] = a < p ? wds[rr * p + a] : 0.;
          vb[t] = b < p ? ws[rr * p + b] : 0.;
        }
#pragma unroll
        for (int ta = 0; ta < T; ++ta)
#pragma unroll
          for (int tb = 0; tb < T; ++tb) acc[ta][tb] = fma(va[ta], vb[tb], acc[ta][tb]);
      }
    }
    if (tid < p)
#pragma unroll 4
      for (int rr = 0; rr < kRows; ++rr) racc = fma(ws[rr * p + tid], us[rr], racc);
    __syncthreads();
  }
  double* out = partial + (size_t)blockIdx.x * (p * p + p);
  if (tile_live) {
#pragma unroll
    for (int ta = 0; ta < T; ++ta)
#pragma unroll
      for (int tb = 0; tb < T; ++tb) {
        const int a = ty * T + ta, b = tx * T + tb;
        if (a < p && b <= a) out[a * p + b] = acc[ta][tb];
      }
  }
  if (tid < p) out[p * p + tid] = racc;
}

// G (p x p, both triangles from the lower one) and r = sums over the chunks in chunk order
__global__ void gls_gram_reduce_kernel(const double* __restrict__ partial, int nchunks, int p, double* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= p * p + p) return;
  int src = e;
  if (e < p * p) {
    const int a = e / p, b = e % p;
    src = a >= b ? a * p + b : b * p + a;
  }
  double s = 0.;
  for (int ch = 0; ch < nchunks; ++ch) s += partial[(size_t)ch * (p * p + p) + src];
  out[e] = s;
}

// y_r = y0 - X beta (Vecchia order), the engine's new response
__global__ void gls_residual_kernel(const double* __restrict__ X, const double* __restrict__ y0, int64_t n, int p,
                                    const ResidualArgs args, double* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double* Xi = X + i * p;
    double xb = 0.;
    for (int c = 0; c < p; ++c) xb = fma(Xi[c], args.beta[c], xb);
    y[i] = y0[i] - xb;
  }
}

// u = D^-1 B y from the resident factor; one warp per row (lanes over the neighbours), per-warp sums of
// {(By)_i^2 D^-1_i, -log D^-1_i, #(D_i <= 0)} in a fixed order, written to partial[warp][3]
__global__ void gls_quad_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, const double* __restrict__ Dinv,
                                const double* __restrict__ y, int64_t n, int m, double* __restrict__ u, double* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double q = 0., ld = 0., bad = 0.;
  for (int64_t i = warp; i < n; i += nwarps) {
    double s = 0.;
    for (int k = lane; k < m; k += 32) {
      const int32_t j = nn[i * m + k];
      if (j >= 0) s = fma(A[i * m + k], y[j], s);
    }
    s = gpb::warp_sum(s);
    if (lane == 0) {
      const double di = Dinv[i];
      const double by = y[i] - s;
      u[i] = di * by;
      q += by * by * di;
      ld -= log(di);
      bad += di > 0. ? 0. : 1.;
    }
  }
  if (lane == 0) {
    partial[warp * 3 + 0] = q;
    partial[warp * 3 + 1] = ld;
    partial[warp * 3 + 2] = bad;
  }
}

__global__ void gls_quad_reduce_kernel(const double* __restrict__ partial, int64_t nwarps, double* __restrict__ sums) {
  __shared__ double sh[256];
  for (int k = 0; k < 3; ++k) {
    double s = 0.;
    for (int64_t r = threadIdx.x; r < nwarps; r += blockDim.x) s += partial[r * 3 + k];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) sums[k] = sh[0];  // GPBDEV_SUM_QUAD, _LOGDET, _NBAD
    __syncthreads();
  }
}

// Xo[i*p + c] = X_colmajor[c*n + perm[i]]
__global__ void gather_covariates_kernel(const double* __restrict__ Xcm, const int32_t* __restrict__ perm, int64_t n, int p,
                                         double* __restrict__ Xo) {
  const int64_t total = n * p;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / p;
    const int c = (int)(e % p);
    Xo[e] = Xcm[(int64_t)c * n + perm[i]];
  }
}

using GramKernel = void (*)(const double*, const int32_t*, const double*, const double*, const double*, int64_t, int, int, int,
                            int64_t, double*);
inline GramKernel pick_gram(int T) {
  switch (T) {
    case 1: return gls_gram_kernel<1>;
    case 2: return gls_gram_kernel<2>;
    case 3: return gls_gram_kernel<3>;
    default: return gls_gram_kernel<4>;
  }
}

}  // namespace gpc

extern "C" {

int gpbdev_vecchia_set_covariates(gpbdev_vecchia_t h, const double* X_colmajor_host, int p) {
  if (!h || !X_colmajor_host) return fail("gpbdev_vecchia_set_covariates: null argument");
  if (p < 1 || p > gpc::kMaxP)
    return fail("gpbdev_vecchia_set_covariates: the number of covariates must be in [1, " + std::to_string(gpc::kMaxP) + "] (got " +
                std::to_string(p) + ")");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_set_covariates: row-sharded engines are not supported");
  CUDA_TRY(cudaSetDevice(h->device));
  const int64_t n = h->n;
  if (h->X == nullptr || h->p != p) {
    cudaFree(h->X); cudaFree(h->gram_partial); cudaFree(h->gram_out);
    h->X = nullptr; h->gram_partial = nullptr; h->gram_out = nullptr;
    h->p = 0;
    CUDA_TRY(cudaMalloc(&h->X, sizeof(double) * n * p));
    // one chunk per resident CTA (registers of this tile width): the chunk count, and with it the summation order, is fixed for
    // the engine and p
    int per_sm = 0;
    const size_t smem = sizeof(double) * (2 * gpc::kRows * p + gpc::kRows);
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gpc::pick_gram((p + 15) / 16), gpc::kThreads, smem));
    h->gram_chunks = (int)std::max<int64_t>(1, std::min<int64_t>((n + gpc::kRows - 1) / gpc::kRows, (int64_t)h->num_sms * std::max(per_sm, 1)));
    CUDA_TRY(cudaMalloc(&h->gram_partial, sizeof(double) * (size_t)h->gram_chunks * (p * p + p)));
    CUDA_TRY(cudaMalloc(&h->gram_out, sizeof(double) * (p * p + p)));
    h->p = p;
  }
  if (h->y0 == nullptr) {
    CUDA_TRY(cudaMalloc(&h->y0, sizeof(double) * n));
    const int64_t nw = (int64_t)h->num_sms * 8 * 8;  // warps of gls_quad_kernel
    CUDA_TRY(cudaMalloc(&h->quad_partial, sizeof(double) * nw * 3));
  }
  double* Xcm = nullptr;
  CUDA_TRY(cudaMalloc(&Xcm, sizeof(double) * n * p));
  cudaError_t e = cudaMemcpyAsync(Xcm, X_colmajor_host, sizeof(double) * n * p, cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) {
    gpc::gather_covariates_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(Xcm, h->perm, n, p, h->X);
    e = cudaGetLastError();
  }
  // the installed response (y - offset, Vecchia order) is the fixed part of every residual
  if (e == cudaSuccess) e = cudaMemcpyAsync(h->y0, h->y, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(Xcm);
  h->launches += 1;
  if (e != cudaSuccess) return fail(std::string("gpbdev_vecchia_set_covariates: ") + cudaGetErrorString(e));
  return 0;
}

int gpbdev_vecchia_gls_gram(gpbdev_vecchia_t h, double* G_host, double* r_host) {
  if (!h || !G_host || !r_host) return fail("gpbdev_vecchia_gls_gram: null argument");
  if (h->X == nullptr) return fail("gpbdev_vecchia_gls_gram: no covariates (gpbdev_vecchia_set_covariates first)");
  if (!h->factor_stored) return fail("gpbdev_vecchia_gls_gram: the factor is not resident (gpbdev_vecchia_eval with mode = STORE first)");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_gls_gram: row-sharded engines are not supported");
  CUDA_TRY(cudaSetDevice(h->device));
  const int64_t n = h->n;
  const int p = h->p, m = h->m;
  const int T = (p + 15) / 16;
  int P = 1;
  while (P < p && P < 32) P <<= 1;
  const int nchunks = h->gram_chunks;
  const int64_t rpc = (n + nchunks - 1) / nchunks;
  const size_t smem = sizeof(double) * (2 * gpc::kRows * p + gpc::kRows);
  gpc::pick_gram(T)<<<nchunks, gpc::kThreads, smem, h->stream>>>(h->A, h->nn, h->Dinv, h->X, h->y0, n, m, p, P, rpc, h->gram_partial);
  CUDA_TRY(cudaGetLastError());
  gpc::gls_gram_reduce_kernel<<<(p * p + p + 255) / 256, 256, 0, h->stream>>>(h->gram_partial, nchunks, p, h->gram_out);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  CUDA_TRY(cudaMemcpyAsync(G_host, h->gram_out, sizeof(double) * p * p, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaMemcpyAsync(r_host, h->gram_out + p * p, sizeof(double) * p, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int gpbdev_vecchia_gls_residual(gpbdev_vecchia_t h, const double* beta_host, double* out3) {
  if (!h || !beta_host || !out3) return fail("gpbdev_vecchia_gls_residual: null argument");
  if (h->X == nullptr) return fail("gpbdev_vecchia_gls_residual: no covariates (gpbdev_vecchia_set_covariates first)");
  if (!h->factor_stored) return fail("gpbdev_vecchia_gls_residual: the factor is not resident (gpbdev_vecchia_eval with mode = STORE first)");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_gls_residual: row-sharded engines are not supported");
  CUDA_TRY(cudaSetDevice(h->device));
  gpc::ResidualArgs args;
  for (int c = 0; c < gpc::kMaxP; ++c) args.beta[c] = c < h->p ? beta_host[c] : 0.;
  gpc::gls_residual_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->X, h->y0, h->n, h->p, args, h->y);
  CUDA_TRY(cudaGetLastError());
  const int blocks = h->num_sms * 8;
  gpc::gls_quad_kernel<<<blocks, 256, 0, h->stream>>>(h->A, h->nn, h->Dinv, h->y, h->n, h->m, h->u, h->quad_partial);
  CUDA_TRY(cudaGetLastError());
  gpc::gls_quad_reduce_kernel<<<1, 256, 0, h->stream>>>(h->quad_partial, (int64_t)blocks * 8, h->sums);
  CUDA_TRY(cudaGetLastError());
  h->launches += 3;
  // the response changed; the factor did not: A, D^-1 stay valid and u now belongs to y_r
  CUDA_TRY(cudaMemcpyAsync(h->sums_host, h->sums, sizeof(double) * 3, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::memcpy(out3, h->sums_host, sizeof(double) * 3);
  return 0;
}

}  // extern "C"
