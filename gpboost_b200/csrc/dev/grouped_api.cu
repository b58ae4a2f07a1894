// Device engine for a single-level grouped random effect with a Gaussian likelihood (SURVEY §8 row a7, BASELINE config 3).
//
// Replaces, for num_re_group_total_ == 1 && num_comps_total_ == 1, the reference's Woodbury path:
//   InitializeMatricesForUseWoodburyIdentity   re_model_template.h:7174-7308 (Zt_, ZtZ_ = diag(n_g))
//   SetY / CalcZtY                             :6185-6200, :6326                (Z^T y = per-group sums)
//   CalcCovFactor single-RE branch             :9417-9420  (diag(Sigma^-1 + Z^T Z) = 1/v + n_g)
//   CalcYtilde / CalcYTPsiIInvY / log-det      :9907-9918, :9938-10007, :3029-3031
//   CalcYAux single-RE branch                  :9843-9844, :9874-9891 (y_aux = y - Z (1/v + n_g)^-1 Z^T y)
//   CalcGradPars_Only_Grouped_REs_Woodbury...  :2462-2529
// Everything reduces to the fixed group counts n_g and the per-group sums s_g = sum_{i in g} y_i:
//   y^T Psi^-1 y = y^T y - sum_g s_g^2 / (1/v + n_g),  log|Psi| = sum_g log(1 + v n_g),  v = sigma_1^2 / sigma^2.
// Design: observations are sorted by group once (counting sort on the host at creation), so s_g is a segmented
// sum over contiguous memory (one warp per group, deterministic); one evaluation = one pass over G groups (16 B/group),
// the response is touched only when it changes (12 B/observation). HBM-bound; at n = 1e6, G = 1e4 an evaluation is
// launch-latency sized.
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace {
thread_local std::string g_grp_err;
int gfail(const std::string& m) { g_grp_err = m; return -1; }
#define GCUDA(expr)                                                                                          \
  do {                                                                                                       \
    cudaError_t e__ = (expr);                                                                                \
    if (e__ != cudaSuccess)                                                                                  \
      return gfail(std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) + ": " + cudaGetErrorString(e__)); \
  } while (0)

__device__ __forceinline__ double wsum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// y_sorted[p] = y[perm[p]]; per-group sum s_g and the group's contribution to y^T y (one warp per group, fixed order)
__global__ void group_sums_kernel(const double* __restrict__ y, const int32_t* __restrict__ perm, const int32_t* __restrict__ offs,
                                  int G, double* __restrict__ s, double* __restrict__ yy) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int g = warp; g < G; g += nw) {
    double a = 0., b = 0.;
    for (int p = offs[g] + lane; p < offs[g + 1]; p += 32) { const double v = y[perm[p]]; a += v; b += v * v; }
    a = wsum(a); b = wsum(b);
    if (lane == 0) { s[g] = a; yy[g] = b; }
  }
}

// sums over groups at variance ratio v: 0 y^T y   1 sum s_g^2/(1/v+n_g)   2 sum log(1+v n_g)
//   3 sum s_g^2 v/(1+v n_g)^2  (= -d(yPy)/dlog v)   4 sum v n_g/(1+v n_g)  (= d log|Psi|/dlog v)
__global__ void group_eval_kernel(const double* __restrict__ s, const double* __restrict__ yy, const int32_t* __restrict__ offs, int G,
                                  double v, double* __restrict__ out) {
  __shared__ double sh[5][256];
  double acc[5] = {0., 0., 0., 0., 0.};
  const int per = (G + blockDim.x - 1) / blockDim.x;  // contiguous slice per thread: fixed summation order
  const int b = threadIdx.x * per, e = min(b + per, G);
  for (int g = b; g < e; ++g) {
    const double ng = (double)(offs[g + 1] - offs[g]);
    const double sg = s[g];
    const double d = 1. / v + ng;
    const double opn = 1. + v * ng;
    acc[0] += yy[g];
    acc[1] += sg * sg / d;
    acc[2] += log(opn);
    acc[3] += sg * sg * v / (opn * opn);
    acc[4] += v * ng / opn;
  }
  for (int k = 0; k < 5; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int k = 0; k < 5; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 5) out[threadIdx.x] = sh[threadIdx.x][0];
}

// y_aux[i] = (y_i - s_g / (1/v + n_g)) * scale, original order
__global__ void group_yaux_kernel(const double* __restrict__ y, const int32_t* __restrict__ perm, const int32_t* __restrict__ offs,
                                  const double* __restrict__ s, int G, double v, double scale, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int g = warp; g < G; g += nw) {
    const double m = s[g] / (1. / v + (double)(offs[g + 1] - offs[g]));
    for (int p = offs[g] + lane; p < offs[g + 1]; p += 32) { const int i = perm[p]; out[i] = (y[i] - m) * scale; }
  }
}
}  // namespace

struct gpbdev_grouped {
  int device = 0, num_sms = 0;
  int64_t n = 0;
  int G = 0;
  cudaStream_t stream = nullptr;
  int32_t *perm = nullptr, *offs = nullptr;
  double *y = nullptr, *s = nullptr, *yy = nullptr, *out = nullptr, *yaux = nullptr;
  double* out_host = nullptr;
  double* stage = nullptr;
  int64_t launches = 0;
  bool has_y = false;  // s / yy hold the sums of an installed response
};

extern "C" {

const char* gpbdev_grouped_last_error(void) { return g_grp_err.c_str(); }

int gpbdev_grouped_create(gpbdev_grouped_t* out, int device, int64_t n, const int32_t* group_index, int num_groups) {
  if (!out || !group_index) return gfail("gpbdev_grouped_create: null argument");
  if (n <= 0 || num_groups <= 0) return gfail("gpbdev_grouped_create: need n > 0 and at least one group");
  // the host-side grouping is validated before any device resource exists
  std::vector<int32_t> offs(num_groups + 1, 0), perm(n);
  for (int64_t i = 0; i < n; ++i) {
    if (group_index[i] < 0 || group_index[i] >= num_groups) return gfail("gpbdev_grouped_create: group index out of range");
    ++offs[group_index[i] + 1];
  }
  for (int g = 0; g < num_groups; ++g) offs[g + 1] += offs[g];
  std::vector<int32_t> fill(offs.begin(), offs.end() - 1);
  for (int64_t i = 0; i < n; ++i) perm[fill[group_index[i]]++] = (int32_t)i;  // stable: ascending i inside a group
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) {
    cudaGetLastError();
    return gfail("gpbdev_grouped_create: no CUDA device " + std::to_string(device) + " — the CUDA engine has no CPU fallback");
  }
  GCUDA(cudaSetDevice(device));
  gpbdev_grouped* h = new gpbdev_grouped();
  h->device = device; h->n = n; h->G = num_groups;
  cudaDeviceProp prop;
  GCUDA(cudaGetDeviceProperties(&prop, device));
  h->num_sms = prop.multiProcessorCount;
  GCUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  GCUDA(cudaMalloc(&h->perm, sizeof(int32_t) * n));
  GCUDA(cudaMalloc(&h->offs, sizeof(int32_t) * (num_groups + 1)));
  GCUDA(cudaMalloc(&h->y, sizeof(double) * n));
  GCUDA(cudaMalloc(&h->yaux, sizeof(double) * n));
  GCUDA(cudaMalloc(&h->s, sizeof(double) * num_groups));
  GCUDA(cudaMalloc(&h->yy, sizeof(double) * num_groups));
  GCUDA(cudaMalloc(&h->out, sizeof(double) * 8));
  GCUDA(cudaMallocHost(&h->out_host, sizeof(double) * 8));
  GCUDA(cudaMallocHost(&h->stage, sizeof(double) * n));
  // on the engine's stream (it does not wait for the legacy default stream), complete before the first set_y
  GCUDA(cudaMemcpyAsync(h->perm, perm.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaMemcpyAsync(h->offs, offs.data(), sizeof(int32_t) * (num_groups + 1), cudaMemcpyHostToDevice, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  *out = h;
  return 0;
}

int gpbdev_grouped_free(gpbdev_grouped_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaFree(h->perm); cudaFree(h->offs); cudaFree(h->y); cudaFree(h->yaux); cudaFree(h->s); cudaFree(h->yy); cudaFree(h->out);
  cudaFreeHost(h->out_host); cudaFreeHost(h->stage);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int gpbdev_grouped_set_y(gpbdev_grouped_t h, const double* y_host) {
  if (!h || !y_host) return gfail("gpbdev_grouped_set_y: null argument");
  GCUDA(cudaSetDevice(h->device));
  GCUDA(cudaStreamSynchronize(h->stream));
  std::memcpy(h->stage, y_host, sizeof(double) * h->n);
  GCUDA(cudaMemcpyAsync(h->y, h->stage, sizeof(double) * h->n, cudaMemcpyHostToDevice, h->stream));
  group_sums_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->y, h->perm, h->offs, h->G, h->s, h->yy);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  h->has_y = true;
  return 0;
}

int gpbdev_grouped_set_y_device(gpbdev_grouped_t h, const double* y_dev) {
  if (!h || !y_dev) return gfail("gpbdev_grouped_set_y_device: null argument");
  GCUDA(cudaSetDevice(h->device));
  GCUDA(cudaMemcpyAsync(h->y, y_dev, sizeof(double) * h->n, cudaMemcpyDeviceToDevice, h->stream));
  group_sums_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->y, h->perm, h->offs, h->G, h->s, h->yy);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  h->has_y = true;
  return 0;
}

int gpbdev_grouped_eval(gpbdev_grouped_t h, double var_ratio, double* out5) {
  if (!h || !out5) return gfail("gpbdev_grouped_eval: null argument");
  if (!(var_ratio > 0.)) return gfail("gpbdev_grouped_eval: the variance ratio must be positive");
  if (!h->has_y) return gfail("gpbdev_grouped_eval: no response installed (call gpbdev_grouped_set_y first)");
  GCUDA(cudaSetDevice(h->device));
  group_eval_kernel<<<1, 256, 0, h->stream>>>(h->s, h->yy, h->offs, h->G, var_ratio, h->out);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  GCUDA(cudaMemcpyAsync(h->out_host, h->out, sizeof(double) * 5, cudaMemcpyDeviceToHost, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  std::memcpy(out5, h->out_host, sizeof(double) * 5);
  return 0;
}

int gpbdev_grouped_yaux(gpbdev_grouped_t h, double var_ratio, double scale, double* yaux_host) {
  if (!h || !yaux_host) return gfail("gpbdev_grouped_yaux: null argument");
  if (!h->has_y) return gfail("gpbdev_grouped_yaux: no response installed (call gpbdev_grouped_set_y first)");
  GCUDA(cudaSetDevice(h->device));
  group_yaux_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->y, h->perm, h->offs, h->s, h->G, var_ratio, scale, h->yaux);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  GCUDA(cudaMemcpyAsync(h->stage, h->yaux, sizeof(double) * h->n, cudaMemcpyDeviceToHost, h->stream));
  GCUDA(cudaStreamSynchronize(h->stream));
  std::memcpy(yaux_host, h->stage, sizeof(double) * h->n);
  return 0;
}

int gpbdev_grouped_yaux_device(gpbdev_grouped_t h, double var_ratio, double scale, double* out_dev) {
  if (!h || !out_dev) return gfail("gpbdev_grouped_yaux_device: null argument");
  if (!h->has_y) return gfail("gpbdev_grouped_yaux_device: no response installed (call gpbdev_grouped_set_y first)");
  GCUDA(cudaSetDevice(h->device));
  group_yaux_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->y, h->perm, h->offs, h->s, h->G, var_ratio, scale, out_dev);
  GCUDA(cudaGetLastError());
  h->launches += 1;
  GCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

int64_t gpbdev_grouped_launch_count(gpbdev_grouped_t h) { return h ? h->launches : 0; }

}  // extern "C"

#include "grouped_multi.cuh"
