// Laplace approximation for a latent Vecchia GP with a bernoulli_logit likelihood (SURVEY §8 row a12, BASELINE config 5).
// Included at the end of dev_api.cu (shares the engine struct, the factor launch and the CSC view of B).
//
// Replaces, for likelihood = "bernoulli_logit", gp_approx = "vecchia", matrix_inversion_method = "iterative",
// cg_preconditioner_type = "vadu":
//   FindModePostRandEffCalcMLLVecchia      include/GPBoost/likelihoods.h:3773-4059   (Newton mode finding + objective)
//   CheckConvergenceModeFinding            include/GPBoost/likelihoods.h:16079-16125
//   Inv_SigmaI_plus_ZtWZ_Vecchia_iterative include/GPBoost/likelihoods.h:16264-16348 (VADU branch)
//   CGVecchiaLaplaceVec                    src/GPBoost/CG_utils.cpp:21-108
//   CalcLogDetStochVecchia                 include/GPBoost/likelihoods.h:16376-16521 (VADU branch)
//   CGTridiagVecchiaLaplace                src/GPBoost/CG_utils.cpp:110-229
//   LogDetStochTridiag                     src/GPBoost/CG_utils.cpp:1035-1052
//   bernoulli_logit log-likelihood / derivatives likelihoods.h:11401, 12477, 13307; DF_utils.h:37-60
//
// Design. All vectors live in the Vecchia order. "Multi-vectors" are n x t row-major (t = 1 for the Newton
// system, t = 50 probe vectors for the stochastic Lanczos quadrature), so one gathered neighbour row is one
// contiguous 8t-byte read. Every operator is a warp-per-row pass over B's fixed pattern:
//   mv_B    T = D^-1 (B X)                         row-dense A, gather of m neighbour rows
//   mv_Bt   V = B^T T + W X  (+ column dots X.V)   CSC gather (deterministic, no atomics)
//   trs_bwd Y = B^-T R                             sparse triangular solve, see below
//   trs_fwd Z = B^-1 (Y / (D^-1 + W))  (+ dots R.Z)
// The two triangular solves of the VADU preconditioner P = B^T (D^-1 + W) B are the serial part of the reference
// (Eigen triangularView solve). Here they are *synchronisation-free*: the solution buffer is pre-filled with a
// sentinel NaN payload, a persistent cooperative grid assigns rows to warps in topological (index) order, and a warp
// simply polls the entries it depends on (ld.relaxed.gpu from L2) until they stop being the sentinel. The dependency
// depth of B at n = 1e6, m = 30 is ~500 rows, so a solve costs ~500 dependency hops of a few L2 round trips each instead
// of 500 kernel launches or grid barriers. All of these kernels are HBM/L2 gather bound: algorithmic bytes per row and column = 8(m+1) gathered
// + 8 written, plus 12m for the pattern and A, amortised over the t columns.
#include <cooperative_groups.h>

#include "slq.h"

namespace gpl {

constexpr unsigned long long kSentinel = 0x7ff8dead0badf00dULL;  // quiet-NaN payload no computation produces
constexpr int kMaxCols = 128;
constexpr int kBlock = 256;
constexpr int kSpinLimit = 1 << 22;
constexpr int kSleepNs = 100;  // back-off between polls of a dependency that is still in flight

struct Coef { double v[kMaxCols]; };

__device__ __forceinline__ bool is_sent(double v) { return (unsigned long long)__double_as_longlong(v) == kSentinel; }
__device__ __forceinline__ double ld_gpu(const double* p) {
  double v;
  asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_gpu(double* p, double v) {
  asm volatile("st.relaxed.gpu.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double wsum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
// polls until the value at p is no longer the sentinel (bounded; a timeout raises *err and yields 0)
__device__ __forceinline__ double poll(const double* p, int* err) {
  double v = ld_gpu(p);
  int spins = 0;
  while (is_sent(v)) {
    if (++spins > kSpinLimit) { atomicExch(err, 1); return 0.; }
    __nanosleep(kSleepNs);
    v = ld_gpu(p);
  }
  return v;
}

__global__ void fill_sentinel_kernel(double* __restrict__ x, int64_t len) {
  const double s = __longlong_as_double((long long)kSentinel);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < len; e += (int64_t)gridDim.x * blockDim.x) x[e] = s;
}

// per-warp column partials -> column sums, fixed order (one block per column and quantity)
__global__ void col_reduce_kernel(const double* __restrict__ partials, int nwarps, int stride, double* __restrict__ out) {
  __shared__ double sh[kBlock];
  const int c = blockIdx.x;
  double a = 0.;
  const int per = (nwarps + kBlock - 1) / kBlock;
  const int b = threadIdx.x * per, e = min(b + per, nwarps);
  for (int w = b; w < e; ++w) a += partials[(size_t)w * stride + c];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int o = kBlock / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[c] = sh[0];
}

// ---- multi-vector kernels ----------------------------------------------------------------------------------------
// Work unit = (row, column group): a warp owns 32 consecutive columns of a row (lane = column), so a row of t = 50 probe
// columns is two independent units. Warp gw works on column group gw % G and on rows gw / G, gw / G + W / G, ... .
// All m gathers of a unit are issued before the first use (m loads in flight per lane); per-warp column partials are
// laid out [row sequence gw / G][column], so every column of a partial row is written by exactly one warp.
constexpr int kM = 30;  // neighbour capacity of the engine (gpb::kMaxNeighbors)

struct Unit {
  int lane, c, cc;     // lane, column, clamped column
  bool active;
  int64_t r0, rstep;   // first row and row stride of this warp
  size_t pslot;        // row of the partial buffer
};
__device__ __forceinline__ Unit make_unit(int t, int G) {
  Unit u;
  u.lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int cg = (int)(gw % G);
  u.c = cg * 32 + u.lane;
  u.active = u.c < t;
  u.cc = u.active ? u.c : t - 1;
  u.r0 = gw / G;
  u.rstep = nw / G;
  u.pslot = (size_t)(gw / G);
  return u;
}

// T[i,:] = s_i * (X[i,:] - sum_k A[i,k] X[nn[i,k],:]),  s_i = Dinv[i] (or 1 when Dinv == nullptr)
// `order` (optional): rows are taken in this order instead of by index — a space-filling-curve order of the locations, so that
// the rows in flight across the grid at any moment are spatial neighbours and share their (spatially near) gathered rows in L2; the
// multi-vector itself stays in Vecchia order, only the time at which a row is processed changes.
__global__ void __launch_bounds__(kBlock) mv_B_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, int m, int64_t n, int t, int G,
                                                      const double* __restrict__ Dinv, const double* __restrict__ X, double* __restrict__ T,
                                                      const int32_t* __restrict__ order) {
  const Unit u = make_unit(t, G);
  for (int64_t p = u.r0; p < n; p += u.rstep) {
    const int64_t i = order ? (int64_t)order[p] : p;
    int32_t jk = u.lane < m ? nn[i * m + u.lane] : -1;
    const double ak = jk >= 0 ? A[i * m + u.lane] : 0.;
    jk = max(jk, 0);
    double acc = X[i * t + u.cc];
    double v[kM];
#pragma unroll
    for (int k = 0; k < kM; ++k) v[k] = X[(int64_t)__shfl_sync(0xffffffffu, jk, k) * t + u.cc];
#pragma unroll
    for (int k = 0; k < kM; ++k) acc -= __shfl_sync(0xffffffffu, ak, k) * v[k];
    if (u.active) T[i * t + u.c] = (Dinv ? Dinv[i] : 1.) * acc;
  }
}

// single-vector form: lane k owns neighbour k
__global__ void v_mv_B_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, int m, int64_t n,
                              const double* __restrict__ Dinv, const double* __restrict__ x, double* __restrict__ T) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = gw; i < n; i += nw) {
    double v = 0.;
    if (lane < m) {
      const int32_t j = nn[i * m + lane];
      if (j >= 0) v = A[i * m + lane] * x[j];
    }
    v = wsum(v);
    if (lane == 0) T[i] = (Dinv ? Dinv[i] : 1.) * (x[i] - v);
  }
}

// V[j,:] = T[j,:] - sum_{(i,k): nn[i,k]=j} A[i,k] T[i,:] + W[j] X[j,:];  partial[.][c] += X[j,c] V[j,c]
__global__ void __launch_bounds__(kBlock) mv_Bt_kernel(const double* __restrict__ A, const int32_t* __restrict__ colptr,
                                                       const int32_t* __restrict__ csc_pos, int m, int64_t n, int t, int G,
                                                       const double* __restrict__ T, const double* __restrict__ W,
                                                       const double* __restrict__ X, double* __restrict__ V, double* __restrict__ partial,
                                                       const int32_t* __restrict__ order) {
  const Unit u = make_unit(t, G);
  double dot = 0.;
  for (int64_t p = u.r0; p < n; p += u.rstep) {
    const int64_t j = order ? (int64_t)order[p] : p;
    double acc = T[j * t + u.cc];
    const double xj = X[j * t + u.cc];
    const int e0 = colptr[j], e1 = colptr[j + 1];
    for (int eb = e0; eb < e1; eb += 32) {
      const int e = eb + u.lane;
      const int32_t pos = e < e1 ? csc_pos[e] : 0;
      const double ap = e < e1 ? A[pos] : 0.;
      const int64_t rowp = e < e1 ? pos / m : j;
      const int cnt = min(32, e1 - eb);
#pragma unroll
      for (int hb = 0; hb < 32; hb += 16) {
        if (hb < cnt) {
          double v[16];
#pragma unroll
          for (int q = 0; q < 16; ++q) v[q] = T[__shfl_sync(0xffffffffu, rowp, hb + q) * t + u.cc];
#pragma unroll
          for (int q = 0; q < 16; ++q) acc -= __shfl_sync(0xffffffffu, ap, hb + q) * v[q];
        }
      }
    }
    const double v = acc + (W ? W[j] : 0.) * xj;
    if (u.active) { V[j * t + u.c] = v; dot += xj * v; }
  }
  if (u.active) partial[u.pslot * kMaxCols + u.c] = dot;
}

__global__ void v_mv_Bt_kernel(const double* __restrict__ A_csc, const int32_t* __restrict__ colptr, const int32_t* __restrict__ csc_row,
                               int64_t n, const double* __restrict__ T, const double* __restrict__ W,
                               const double* __restrict__ x, double* __restrict__ V, double* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double dot = 0.;
  for (int64_t j = gw; j < n; j += nw) {
    const int e0 = colptr[j], e1 = colptr[j + 1];
    double s = 0.;
    for (int e = e0 + lane; e < e1; e += 32) s += A_csc[e] * T[csc_row[e]];  // coefficients and rows stream, T is gathered (L2)
    s = wsum(s);
    if (lane == 0) {
      const double xj = x[j];
      const double v = T[j] - s + (W ? W[j] : 0.) * xj;
      V[j] = v;
      dot += xj * v;
    }
  }
  if (lane == 0) partial[(size_t)gw * kMaxCols] = dot;
}

// R -= V * a[c]  (and U += H * a[c] when U != nullptr);  partial[.][c] += R[i,c]^2
__global__ void axpy_norm_kernel(int64_t n, int t, int G, Coef a, const double* __restrict__ V, double* __restrict__ R,
                                 const double* __restrict__ H, double* __restrict__ U, double* __restrict__ partial) {
  const Unit u = make_unit(t, G);
  double rr = 0.;
  if (u.active) {
    const double ac = a.v[u.c];
    for (int64_t i = u.r0; i < n; i += u.rstep) {
      const double r = R[i * t + u.c] - V[i * t + u.c] * ac;
      R[i * t + u.c] = r;
      rr += r * r;
      if (U) U[i * t + u.c] += H[i * t + u.c] * ac;
    }
    partial[u.pslot * kMaxCols + u.c] = rr;
  }
}

// single-vector form of axpy_norm_kernel (the lane = column layout leaves 31 of 32 lanes idle at t = 1): r -= a v, u += a h,
// per-warp partial of sum r^2 in row 0 of the warp's partial slot; grid-stride with a fixed assignment, so deterministic
__global__ void v_axpy_norm_kernel(int64_t n, double a, const double* __restrict__ v, double* __restrict__ r, const double* __restrict__ hh,
                                   double* __restrict__ u, double* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  double rr = 0.;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double ri = r[i] - v[i] * a;
    r[i] = ri;
    rr += ri * ri;
    if (u) u[i] += hh[i] * a;
  }
  rr = wsum(rr);
  if (lane == 0) partial[(size_t)gw * kMaxCols] = rr;
}

// H = Z + H * b[c]
__global__ void h_update_kernel(int64_t len, int t, Coef b, const double* __restrict__ Z, double* __restrict__ H) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < len; e += (int64_t)gridDim.x * blockDim.x)
    H[e] = Z[e] + H[e] * b.v[(int)(e % t)];
}

// ---- synchronisation-free sparse triangular solves --------------------------------------------------------------
// Units are assigned to the warps of a persistent cooperative grid in topological (index) order: within a column group,
// warp w handles rows w, w + W', w + 2W', ... . A unit only ever waits for units of the same column group with a
// smaller position in that order, which belong to co-resident warps at an earlier or equal step of their own
// sequence, so the wait always ends.
// The value itself is the flag: the solution buffer is pre-filled with a sentinel NaN payload. A consumer issues the L2
// loads (ld.cg) of ALL its dependencies at once; for a dependency that still carries the payload ONE lane polls (so a
// waiting warp costs one L2 request per back-off period, not 32) and the warp then re-reads that row. No fences and no
// separate flags: a dependency that finished long ago costs exactly the load the product needs anyway, and a hop of
// the critical path costs about two L2 round trips.
// Resolves the dependencies of one unit. On entry v[k] holds a first (weak, L2) load of dependency k's value at this
// lane's column, dep = this LANE's own dependency row (lane k <-> dependency k), coef != 0 marks real dependencies.
// Dependencies whose value still carries the payload are polled IN PARALLEL (lane k polls the first column of
// dependency k), then the rows that became ready are re-read with all loads in flight: a hop of the critical path
// costs about two L2 round trips no matter how many dependencies were still in flight at the first load.
__device__ __forceinline__ double ld_gpu_nc(const double* p) {  // strong L2 load without a compiler barrier: loads overlap
  double v;
  asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
template <int N>
__device__ __forceinline__ void resolve_deps(double (&v)[N], const double* base, int64_t dep, bool real, int t, int cg0, int cc, int lane,
                                             int* err) {
  unsigned pend = 0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const bool rk = __shfl_sync(0xffffffffu, (int)real, k) != 0;
    if (rk && __any_sync(0xffffffffu, is_sent(v[k]))) pend |= 1u << k;
  }
  int spins = 0;
  while (pend) {
    const bool mine = lane < N && ((pend >> lane) & 1u);
    double w = 0.;
    if (mine) w = ld_gpu(base + dep * t + cg0);
    unsigned still = __ballot_sync(0xffffffffu, mine && is_sent(w));
    const unsigned ready = pend & ~still;
    if (ready) {
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const int64_t row = __shfl_sync(0xffffffffu, dep, k);
        if ((ready >> k) & 1u) v[k] = ld_gpu_nc(base + row * t + cc);
      }
#pragma unroll
      for (int k = 0; k < N; ++k)
        if (((ready >> k) & 1u) && __any_sync(0xffffffffu, is_sent(v[k]))) still |= 1u << k;  // row only partly visible yet
    } else {
      if (++spins > kSpinLimit) { if (lane == 0) atomicExch(err, 1); return; }
      __nanosleep(kSleepNs);
    }
    pend = still;
  }
}

// Y = B^-T R, rows in descending order
__global__ void __launch_bounds__(kBlock) trs_bwd_kernel(const double* __restrict__ A, const int32_t* __restrict__ colptr,
                                                         const int32_t* __restrict__ csc_pos, int m, int64_t n, int t, int G,
                                                         const double* __restrict__ R, double* Y, int* err) {
  const Unit u = make_unit(t, G);
  const int cg0 = u.c - u.lane;
  for (int64_t jj = u.r0; jj < n; jj += u.rstep) {
    const int64_t j = n - 1 - jj;
    double acc = R[j * t + u.cc];
    const int e0 = colptr[j], e1 = colptr[j + 1];
    // A column's entries are sorted by row. Rows far above j finished long ago, the rows just above j may still be in
    // flight: batches are taken from the END of the list, so everything that is already there is consumed while the
    // recent rows complete and only the last batch sits on the dependency chain (early columns have hundreds of entries).
    constexpr int kBatch = 16;  // entries resolved together (16 values + coefficients per lane keep two CTAs per SM resident)
    for (int eb = e0 + ((e1 - e0 - 1) / kBatch) * kBatch; eb >= e0 && e1 > e0; eb -= kBatch) {
      const int e = eb + (u.lane & (kBatch - 1));
      const bool real = e < e1 && u.lane < kBatch;
      const int32_t pos = e < e1 ? csc_pos[e] : 0;
      const double ap = e < e1 ? A[pos] : 0.;
      const int64_t rowp = e < e1 ? pos / m : j;  // idle slots: coefficient 0, value never used
      double v[kBatch];
#pragma unroll
      for (int q = 0; q < kBatch; ++q) v[q] = __ldcg(Y + __shfl_sync(0xffffffffu, rowp, q) * t + u.cc);
      resolve_deps<kBatch>(v, Y, rowp, real, t, cg0, u.cc, u.lane, err);
#pragma unroll
      for (int q = 0; q < kBatch; ++q) {
        const double a = __shfl_sync(0xffffffffu, ap, q);
        if (a != 0.) acc += a * v[q];
      }
    }
    if (u.active) st_gpu(Y + j * t + u.c, acc);
  }
}

// Z = B^-1 (Y / dw), rows ascending; partial[.][c] += R[i,c] Z[i,c]
__global__ void __launch_bounds__(kBlock) trs_fwd_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, int m, int64_t n, int t, int G,
                                                         const double* __restrict__ dw, const double* __restrict__ Y,
                                                         const double* __restrict__ R, double* Z, double* __restrict__ partial, int* err) {
  const Unit u = make_unit(t, G);
  const int cg0 = u.c - u.lane;
  double dot = 0.;
  for (int64_t i = u.r0; i < n; i += u.rstep) {
    int32_t jk = u.lane < m ? nn[i * m + u.lane] : -1;
    const bool real = jk >= 0;
    const double ak = real ? A[i * m + u.lane] : 0.;
    const int64_t dep = real ? jk : (i > 0 ? i - 1 : 0);  // padded slots: coefficient 0, value never used
    double acc = Y[i * t + u.cc] / dw[i];
    const double ri = R[i * t + u.cc];
    double v[kM];
#pragma unroll
    for (int k = 0; k < kM; ++k) v[k] = __ldcg(Z + __shfl_sync(0xffffffffu, dep, k) * t + u.cc);
    resolve_deps<kM>(v, Z, dep, real, t, cg0, u.cc, u.lane, err);
#pragma unroll
    for (int k = 0; k < kM; ++k) {
      const double a = __shfl_sync(0xffffffffu, ak, k);
      if (a != 0.) acc += a * v[k];
    }
    if (u.active) { st_gpu(Z + i * t + u.c, acc); dot += ri * acc; }
  }
  if (u.active) partial[u.pslot * kMaxCols + u.c] = dot;
}

// Single-vector forms (lane = dependency): every lane polls its own dependency (ld.relaxed.gpu, L2) until the payload
// is gone — one L2 round trip per hop of the critical path. The next row's pattern is fetched before the wait.
__global__ void v_trs_bwd_kernel(const double* __restrict__ A, const int32_t* __restrict__ colptr, const int32_t* __restrict__ csc_pos,
                                 int m, int64_t n, const double* __restrict__ r, double* y, int* err) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t jj = gw; jj < n; jj += nw) {
    const int64_t j = n - 1 - jj;
    const int e0 = colptr[j], e1 = colptr[j + 1];
    const double rj = r[j];
    double s = 0.;
    int e = e1 - 1 - lane;  // far rows first (long finished), the rows just above j last
    for (; e - 96 >= e0; e -= 128) {  // four entries per lane in flight
      int32_t pos[4]; double a[4], v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { pos[q] = csc_pos[e - 32 * q]; }
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = A[pos[q]]; v[q] = ld_gpu_nc(y + pos[q] / m); }
#pragma unroll
      for (int q = 0; q < 4; ++q) s += a[q] * (is_sent(v[q]) ? poll(y + pos[q] / m, err) : v[q]);
    }
    for (; e >= e0; e -= 32) {
      const int32_t pos = csc_pos[e];
      s += A[pos] * poll(y + pos / m, err);
    }
    s = wsum(s);
    if (lane == 0) st_gpu(y + j, rj + s);
  }
}

__global__ void v_trs_fwd_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, int m, int64_t n,
                                 const double* __restrict__ dw, const double* __restrict__ y, const double* __restrict__ r,
                                 double* z, double* __restrict__ partial, int* err) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double dot = 0.;
  int32_t jn = -1; double an = 0., yn = 0., rn = 0.;
  if (gw < n) {
    if (lane < m) { jn = nn[gw * m + lane]; an = A[gw * m + lane]; }
    yn = y[gw] / dw[gw]; rn = r[gw];
  }
  for (int64_t i = gw; i < n; i += nw) {
    const int32_t j = jn; const double a = an, yi = yn, ri = rn;
    const int64_t ni = i + nw;
    if (ni < n) {  // next row's pattern and right-hand side: in flight while this row waits
      jn = lane < m ? nn[ni * m + lane] : -1;
      an = lane < m ? A[ni * m + lane] : 0.;
      yn = y[ni] / dw[ni]; rn = r[ni];
    }
    double s = 0.;
    if (j >= 0) s = a * poll(z + j, err);
    s = wsum(s);
    if (lane == 0) {
      const double zi = yi + s;
      st_gpu(z + i, zi);
      dot += ri * zi;
    }
  }
  if (lane == 0) partial[(size_t)gw * kMaxCols] = dot;
}

__global__ void csc_gather_kernel(const double* __restrict__ A, const int32_t* __restrict__ csc_pos, int m, int64_t cnt,
                                  double* __restrict__ A_csc, int32_t* __restrict__ csc_row) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < cnt; e += (int64_t)gridDim.x * blockDim.x) {
    const int32_t pos = csc_pos[e];
    A_csc[e] = A[pos];
    csc_row[e] = pos / m;
  }
}

// ---- likelihood pieces: the three per-row kernels (prep_kernel, row_stats_kernel, grad_coef_kernel) are templated on
// the likelihood; everything else (operators, solves, SLQ, trace estimation) is likelihood-free. loc = mode + fixed effect.
//   bernoulli_logit (DF_utils.h:37-60, likelihoods.h:11401, 12477, 13307): log-lik y loc - softplus(loc), first derivative
//     y - p, information W = p (1 - p) <= 1/4, its derivative dW = p (1 - p) (1 - 2p), p = sigmoid(loc)
//   poisson, log link: log-lik y loc - exp(loc) (LogLikPoisson with incl_norm_const = false, likelihoods.h:11121-11126, 11407-11415),
//     first derivative y - exp(loc) (likelihoods.h:12176-12182, 12385-12386, 12481-12483), information W = exp(loc), unbounded
//     (likelihoods.h:12881-12886, 13061-13066, 13183-13184, 13255-13256, 13315-13317), dW = exp(loc) (likelihoods.h:13822-13827,
//     14110-14115). The normalising constant -sum_i log(y_i!) (likelihoods.h:10750-10757, 10985-10996) does not depend on
//     loc: the host computes it once per response and the evaluation adds it to every log-likelihood sum, as LogLikelihood does
//     (likelihoods.h:11290). No overflow guard on exp(loc): the reference has none.
enum : int { kLikBernoulliLogit = 0, kLikPoisson = 1 };

__device__ __forceinline__ double sigmoid_stable(double x) {
  if (x >= 0.) { const double e = exp(-x); return 1. / (1. + e); }
  const double e = exp(x);
  return e / (1. + e);
}
__device__ __forceinline__ double softplus(double x) { return log1p(exp(-fabs(x))) + fmax(x, 0.); }

// first derivative, information W, Newton right-hand side W mode + first derivative, dw = D^-1 + W
template <int kLik>
__global__ void prep_kernel(int64_t n, const double* __restrict__ y, const double* __restrict__ mode, const double* __restrict__ fe,
                            const double* __restrict__ Dinv, double* __restrict__ W, double* __restrict__ rhs, double* __restrict__ dw) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double loc = mode[i] + (fe ? fe[i] : 0.);
    if constexpr (kLik == kLikBernoulliLogit) {
      const double p = sigmoid_stable(loc);
      const double w = p * (1. - p);
      W[i] = w;
      if (rhs) rhs[i] = w * mode[i] + (y[i] - p);
      dw[i] = Dinv[i] + w;
    } else {
      const double mu = exp(loc);
      W[i] = mu;
      if (rhs) rhs[i] = mu * mode[i] + (y[i] - mu);
      dw[i] = Dinv[i] + mu;
    }
  }
}

// x = (1 - lr) * a + lr * b  (lr = 1 copies b);  d = b - a when d != nullptr
__global__ void lincomb_kernel(int64_t n, double lr, const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ x,
                               double* __restrict__ d) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (x) x[i] = lr == 1. ? b[i] : (1. - lr) * a[i] + lr * b[i];
    if (d) d[i] = b[i] - a[i];
  }
}

// per-warp partials of: 0 sum_i Dinv_i (B x)_i^2   1 sum_i W_i x_i^2   2 sum_i loglik(y_i, x_i + fe_i) (without the constant)
//                       3 sum_i log Dinv_i          4 sum_i log dw_i
template <int kLik>
__global__ void row_stats_kernel(const double* __restrict__ A, const int32_t* __restrict__ nn, int m, int64_t n,
                                 const double* __restrict__ Dinv, const double* __restrict__ x, const double* __restrict__ W,
                                 const double* __restrict__ y, const double* __restrict__ fe, const double* __restrict__ dw,
                                 double* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double s0 = 0., s1 = 0., s2 = 0., s3 = 0., s4 = 0.;
  for (int64_t i = gw; i < n; i += nw) {
    double v = 0.;
    if (lane < m) {
      const int32_t j = nn[i * m + lane];
      if (j >= 0) v = A[i * m + lane] * x[j];
    }
    v = wsum(v);
    if (lane == 0) {
      const double xi = x[i];
      const double bx = xi - v;
      s0 += Dinv[i] * bx * bx;
      if (W) s1 += W[i] * xi * xi;
      if (y) {
        const double loc = xi + (fe ? fe[i] : 0.);
        if constexpr (kLik == kLikBernoulliLogit) s2 += y[i] * loc - softplus(loc);
        else s2 += y[i] * loc - exp(loc);
      }
      s3 += log(Dinv[i]);
      if (dw) s4 += log(dw[i]);
    }
  }
  if (lane == 0) {
    double* o = partial + (size_t)gw * kMaxCols;
    o[0] = s0; o[1] = s1; o[2] = s2; o[3] = s3; o[4] = s4;
  }
}

// probes (n x t column-major, as the reference draws them) -> Zp = B^T (sqrt(dw) .* probes), row-major n x t
__global__ void scale_transpose_kernel(int64_t n, int t, const double* __restrict__ probes_cm, const double* __restrict__ dw,
                                       double* __restrict__ out_rm) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n * t; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / t;
    const int c = (int)(e % t);
    out_rm[e] = sqrt(dw[i]) * probes_cm[(int64_t)c * n + i];
  }
}

// out[perm[i]] = x[i]
__global__ void scatter_perm_kernel(int64_t n, const double* __restrict__ x, const int32_t* __restrict__ perm, double* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[perm[i]] = x[i];
}

// ---- gradient of the Laplace-approximated likelihood (likelihoods.h:6521-7044, iterative branch) ----
// T[i,:] = -sum_k dA[i,k] X[nn[i,k],:]  = (B_grad X)[i,:]  (B_grad = -dA has no diagonal); same unit scheme as mv_B_kernel
__global__ void __launch_bounds__(kBlock) mv_Bg_kernel(const double* __restrict__ dA, const int32_t* __restrict__ nn, int m, int64_t n, int t, int G,
                                                       const double* __restrict__ X, double* __restrict__ T) {
  const Unit u = make_unit(t, G);
  for (int64_t i = u.r0; i < n; i += u.rstep) {
    int32_t jk = u.lane < m ? nn[i * m + u.lane] : -1;
    const double ak = jk >= 0 ? dA[i * m + u.lane] : 0.;
    jk = max(jk, 0);
    double acc = 0.;
    double v[kM];
#pragma unroll
    for (int k = 0; k < kM; ++k) v[k] = X[(int64_t)__shfl_sync(0xffffffffu, jk, k) * t + u.cc];
#pragma unroll
    for (int k = 0; k < kM; ++k) acc -= __shfl_sync(0xffffffffu, ak, k) * v[k];
    if (u.active) T[i * t + u.c] = acc;
  }
}
// V[j,:] (+)= -sum_{(i,k): nn[i,k]=j} dA[i,k] T[i,:]  = (B_grad^T T)[j,:]; accumulate != 0 adds to what V holds
__global__ void __launch_bounds__(kBlock) mv_Bgt_kernel(const double* __restrict__ dA, const int32_t* __restrict__ colptr,
                                                        const int32_t* __restrict__ csc_pos, int m, int64_t n, int t, int G,
                                                        const double* __restrict__ T, double* __restrict__ V, int accumulate) {
  const Unit u = make_unit(t, G);
  for (int64_t j = u.r0; j < n; j += u.rstep) {
    double acc = accumulate ? V[j * t + u.cc] : 0.;
    const int e0 = colptr[j], e1 = colptr[j + 1];
    for (int eb = e0; eb < e1; eb += 32) {
      const int e = eb + u.lane;
      const int32_t pos = e < e1 ? csc_pos[e] : 0;
      const double ap = e < e1 ? dA[pos] : 0.;
      const int64_t rowp = e < e1 ? pos / m : j;
      const int cnt = min(32, e1 - eb);
      for (int q = 0; q < cnt; ++q) acc -= __shfl_sync(0xffffffffu, ap, q) * T[__shfl_sync(0xffffffffu, rowp, q) * t + u.cc];
    }
    if (u.active) V[j * t + u.c] = acc;
  }
}
// partial[.][c] = sum_i X[i,c] Y[i,c]
__global__ void __launch_bounds__(kBlock) coldot_kernel(int64_t n, int t, int G, const double* __restrict__ X, const double* __restrict__ Y,
                                                        double* __restrict__ partial) {
  const Unit u = make_unit(t, G);
  double d = 0.;
  if (u.active) {
    for (int64_t i = u.r0; i < n; i += u.rstep) d += X[i * t + u.c] * Y[i * t + u.c];
    partial[u.pslot * kMaxCols + u.c] = d;
  }
}
// elementwise row scalings of multi-vectors:  out[i,:] = a_i * X[i,:] + b_i * Y[i,:]  with
//   mode 0: a = Dinv, b = -Dinv * dD          (T3 = D^-1 T2 - D^-1 dD T1,            X = T2, Y = T1)
//   mode 1: a = Dinv, b = -Dinv * dD + W/Dinv.. see below
// kept general: a_i = ca[i], b_i = cb[i] are precomputed n-vectors
__global__ void rowscale2_kernel(int64_t n, int t, const double* __restrict__ ca, const double* __restrict__ X, const double* __restrict__ cb,
                                 const double* __restrict__ Y, double* __restrict__ out) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n * t; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / t;
    out[e] = ca[i] * X[e] + cb[i] * Y[e];
  }
}
__global__ void rowscale1_kernel(int64_t n, int t, const double* __restrict__ ca, const double* __restrict__ X, double* __restrict__ out) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n * t; e += (int64_t)gridDim.x * blockDim.x) out[e] = ca[e / t] * X[e];
}
// coefficient vectors of the range derivative:  c0 = Dinv, c1 = -Dinv dD,  c2 = Dinv + W  (= T3 + W T2 coefficient of T2),
// c3 = 1 + W / Dinv (coefficient of T1 in T1 + W (B X));  dW = dW/dloc of the likelihood (CalcFirstDerivInformationLocPar)
// per-warp partials: 0 sum Dinv dD   1 sum Dinv / dw   2 sum Dinv^2 dD / dw
template <int kLik>
__global__ void grad_coef_kernel(int64_t n, const double* __restrict__ Dinv, const double* __restrict__ dD, const double* __restrict__ W,
                                 const double* __restrict__ dw, const double* __restrict__ mode, const double* __restrict__ fe,
                                 double* __restrict__ c1, double* __restrict__ c2, double* __restrict__ c3, double* __restrict__ dWout,
                                 double* __restrict__ partial) {
  const int lane = threadIdx.x & 31;
  const int64_t gt = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
  double s0 = 0., s1 = 0., s2 = 0.;
  for (int64_t i = gt; i < n; i += nt) {
    const double di = Dinv[i], dd = dD[i], w = W[i];
    c1[i] = -di * dd;
    c2[i] = di + w;
    c3[i] = 1. + w / di;
    if constexpr (kLik == kLikBernoulliLogit) {
      const double p = sigmoid_stable(mode[i] + (fe ? fe[i] : 0.));
      dWout[i] = p * (1. - p) * (1. - 2. * p);
    } else {
      dWout[i] = exp(mode[i] + (fe ? fe[i] : 0.));
    }
    s0 += di * dd; s1 += di / dw[i]; s2 += di * di * dd / dw[i];
  }
  s0 = wsum(s0); s1 = wsum(s1); s2 = wsum(s2);
  if (lane == 0) {
    double* o = partial + (size_t)(gt >> 5) * kMaxCols;
    o[0] = s0; o[1] = s1; o[2] = s2;
  }
}
// d mll / d mode (CalcLogDetStochDerivModeVecchia, VADU branch, + the factor 1/2 of likelihoods.h:6601): one warp per row,
//   ZA = U dW Z (stochastic tr((Sigma^-1 + W)^-1 dW/db_i)), ZP = T dW T (tr(P^-1 dP/db_i), T = B P^-1 Z),
//   c = cov(ZA, ZP) / var(ZP) over the probe columns (CalcOptimalCVectorized), out = (mean ZA + c (dW / dw - mean ZP)) / 2
__global__ void stoch_dmode_kernel(int64_t n, int t, const double* __restrict__ U, const double* __restrict__ Z, const double* __restrict__ T,
                                   const double* __restrict__ dW, const double* __restrict__ dw, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  constexpr int kPer = kMaxCols / 32;
  for (int64_t i = gw; i < n; i += nw) {
    const double dwi = dW[i];
    double za[kPer], zp[kPer];
    double sa = 0., sp = 0.;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int c = q * 32 + lane;
      if (c < t) {
        const double tv = T[i * t + c];
        za[q] = U[i * t + c] * dwi * Z[i * t + c];
        zp[q] = tv * dwi * tv;
        sa += za[q]; sp += zp[q];
      } else { za[q] = 0.; zp[q] = 0.; }
    }
    const double ma = wsum(sa) / t, mp = wsum(sp) / t;
    double cc = 0., cv = 0.;
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int c = q * 32 + lane;
      if (c < t) { const double a = za[q] - ma, b = zp[q] - mp; cc += a * b; cv += b * b; }
    }
    cc = wsum(cc) / t; cv = wsum(cv) / t;
    const double copt = cv == 0. ? 1. : cc / cv;
    if (lane == 0) out[i] = 0.5 * (ma + copt * (dwi / dw[i]) - copt * mp);
  }
}

}  // namespace gpl

struct gpb_laplace_state {
  int t = 0;              // probe columns held by this process
  int t_total = 0;        // probe columns of the whole job (columns are sharded over ranks, see set_collective)
  void (*allreduce)(double*, int) = nullptr;
  int grid = 0;           // persistent cooperative grid (blocks): what is co-resident for the polling kernels
  int grid_mv = 0;        // grid of the ordinary (non-polling) row kernels
  int grid_v = 0;         // cooperative grid of the single-vector polling kernels (few registers: more resident warps)
  int32_t* order = nullptr;  // n: processing order of the order-free row kernels (Morton order of the locations); null = by index
  int nwarps = 0;
  double *mode = nullptr, *mode_new = nullptr, *upd = nullptr, *dir = nullptr, *rhs = nullptr, *W = nullptr, *dw = nullptr, *fe = nullptr;
  double *r = nullptr, *z = nullptr, *hv = nullptr, *v = nullptr, *tt = nullptr, *yy = nullptr;  // n-vectors of the Newton CG
  double *probes = nullptr;  // n x t column-major (reference layout), ordered rows
  double *R = nullptr, *Z = nullptr, *H = nullptr, *V = nullptr, *T = nullptr, *Y = nullptr;  // n x t row-major
  // gradient (gpbdev_vecchia_laplace_grad): the SLQ's CG solutions (Sigma^-1 + W)^-1 Z are kept when `keep` is set
  bool keep = false, fe_set = false, solutions_valid = false;
  int lik = gpl::kLikBernoulliLogit;  // instance of the per-row kernels (gpbdev_vecchia_laplace_set_likelihood)
  double log_norm_const = 0.;         // added to every log-likelihood sum (0 for bernoulli_logit)
  double* U = nullptr;        // n x t
  int U_t = 0;
  double *c1 = nullptr, *c2 = nullptr, *c3 = nullptr, *dWv = nullptr;  // n
  double* partial = nullptr;  // nwarps x kMaxCols
  double* colsum = nullptr;   // kMaxCols (device)
  double* colsum_host = nullptr;  // pinned
  int* err = nullptr;
  double* stage = nullptr;    // pinned n
};

namespace {

void laplace_release(gpbdev_vecchia* h) {
  gpb_laplace_state* L = h->lap;
  if (!L) return;
  double* bufs[] = {L->mode, L->mode_new, L->upd, L->dir, L->rhs, L->W, L->dw, L->fe, L->r, L->z, L->hv, L->v, L->tt, L->yy,
                    L->probes, L->R, L->Z, L->H, L->V, L->T, L->Y, L->partial, L->colsum, L->U, L->c1, L->c2, L->c3, L->dWv};
  for (double* b : bufs) cudaFree(b);
  cudaFree(L->err);
  cudaFree(L->order);
  cudaFreeHost(L->colsum_host);
  cudaFreeHost(L->stage);
  delete L;
  h->lap = nullptr;
}

int laplace_ensure(gpbdev_vecchia* h) {
  if (h->lap) return 0;
  if (h->row_begin != 0 || h->row_end != h->n) return fail("Laplace-Vecchia: row-sharded engines are not supported yet");
  if (h->m > gpl::kM) return fail("Laplace-Vecchia: num_neighbors must be <= 30 for non-Gaussian likelihoods in the CUDA engine");
  int coop = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device));
  if (!coop) return fail("Laplace-Vecchia: the device does not support cooperative launches");
  gpb_laplace_state* L = new gpb_laplace_state();
  h->lap = L;
  const int64_t n = h->n;
  // persistent grid: what is co-resident for the polling kernels (the most register-hungry instantiation bounds all)
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gpl::trs_bwd_kernel, gpl::kBlock, 0));
  int per_sm2 = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, gpl::trs_fwd_kernel, gpl::kBlock, 0));
  per_sm = std::max(1, std::min(std::min(per_sm, per_sm2), 4));
  L->grid = per_sm * h->num_sms;
  L->grid_mv = 6 * h->num_sms;
  int per_v = 0, per_v2 = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_v, gpl::v_trs_bwd_kernel, gpl::kBlock, 0));
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_v2, gpl::v_trs_fwd_kernel, gpl::kBlock, 0));
  L->grid_v = std::max(1, std::min(std::min(per_v, per_v2), 4)) * h->num_sms;
  L->nwarps = std::max(std::max(L->grid, L->grid_mv), L->grid_v) * (gpl::kBlock / 32) + 1;
  double** vecs[] = {&L->mode, &L->mode_new, &L->upd, &L->dir, &L->rhs, &L->W, &L->dw, &L->fe, &L->r, &L->z, &L->hv, &L->v, &L->tt, &L->yy};
  for (double** p : vecs) {
    CUDA_TRY(cudaMalloc(p, sizeof(double) * n));
    CUDA_TRY(cudaMemsetAsync(*p, 0, sizeof(double) * n, h->stream));
  }
  CUDA_TRY(cudaMalloc(&L->partial, sizeof(double) * (size_t)L->nwarps * gpl::kMaxCols));
  CUDA_TRY(cudaMemsetAsync(L->partial, 0, sizeof(double) * (size_t)L->nwarps * gpl::kMaxCols, h->stream));
  CUDA_TRY(cudaMalloc(&L->colsum, sizeof(double) * gpl::kMaxCols));
  CUDA_TRY(cudaMallocHost(&L->colsum_host, sizeof(double) * gpl::kMaxCols));
  CUDA_TRY(cudaMalloc(&L->err, sizeof(int)));
  CUDA_TRY(cudaMemsetAsync(L->err, 0, sizeof(int), h->stream));
  CUDA_TRY(cudaMallocHost(&L->stage, sizeof(double) * n));
  // processing order of mv_B / mv_Bt: Morton (Z-order) curve over the bounding box of the locations (d = 2: 2 x 16 bits, d = 3: 3 x 10 bits),
  // index order at every other d
  if (h->d == 2 || h->d == 3) {
    const int d = h->d;
    std::vector<double> c((size_t)n * d);
    CUDA_TRY(cudaMemcpy(c.data(), h->coords, sizeof(double) * n * d, cudaMemcpyDeviceToHost));
    double lo[3] = {c[0], c[1], d > 2 ? c[2] : 0.}, hi[3] = {c[0], c[1], d > 2 ? c[2] : 0.};
    for (int64_t i = 0; i < n; ++i)
      for (int k = 0; k < d; ++k) { lo[k] = std::min(lo[k], c[(size_t)i * d + k]); hi[k] = std::max(hi[k], c[(size_t)i * d + k]); }
    const int bits = d == 2 ? 16 : 10;
    std::vector<std::pair<uint32_t, int32_t>> key((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      uint32_t code = 0;
      uint32_t q[3] = {0, 0, 0};
      for (int k = 0; k < d; ++k) {
        const double w = hi[k] > lo[k] ? (c[(size_t)i * d + k] - lo[k]) / (hi[k] - lo[k]) : 0.;
        q[k] = (uint32_t)std::min<double>((double)((1u << bits) - 1), w * (double)(1u << bits));
      }
      for (int b = bits - 1; b >= 0; --b)
        for (int k = 0; k < d; ++k) code = (code << 1) | ((q[k] >> b) & 1u);
      key[(size_t)i] = std::make_pair(code, (int32_t)i);
    }
    std::sort(key.begin(), key.end());
    std::vector<int32_t> ord((size_t)n);
    for (int64_t p = 0; p < n; ++p) ord[(size_t)p] = key[(size_t)p].second;
    CUDA_TRY(cudaMalloc(&L->order, sizeof(int32_t) * n));
    CUDA_TRY(cudaMemcpy(L->order, ord.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice));
  }
  return 0;
}

// column sums of the per-warp partials -> pinned host (synchronises the stream)
int laplace_colsums(gpbdev_vecchia* h, int ncols, double* out, int nrows) {
  gpb_laplace_state* L = h->lap;
  gpl::col_reduce_kernel<<<ncols, gpl::kBlock, 0, h->stream>>>(L->partial, nrows, gpl::kMaxCols, L->colsum);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(L->colsum_host, L->colsum, sizeof(double) * ncols, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  for (int c = 0; c < ncols; ++c) out[c] = L->colsum_host[c];
  h->launches += 1;
  return 0;
}

template <typename K, typename... Args>
int coop_launch(gpbdev_vecchia* h, int grid, K kernel, Args... args) {
  void* params[] = {(void*)&args...};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)kernel, dim3(grid), dim3(gpl::kBlock), params, 0, h->stream));
  h->launches += 1;
  return 0;
}

// column groups of a t-column multi-vector and the grid that keeps (warps % groups) == 0
inline int lap_groups(int t) { return (t + 31) / 32; }
inline int lap_grid(int grid, int G) { return std::max(G, grid - grid % G); }

// Coefficients in CSC order: the B^T products and the backward solves walk columns, and A[csc_pos[e]] is a random 8-byte read
// (one 32-byte sector each) where A_csc[e] streams. Rebuilt after every latent factorisation (one gather over nnz entries).
int lap_refresh_csc_coefs(gpbdev_vecchia* h) {
  const int64_t nnz = (int64_t)h->n * h->m;  // upper bound of the CSC length (padded slots are not in it)
  int32_t cnt = 0;
  CUDA_TRY(cudaMemcpyAsync(&cnt, h->colptr + h->n, sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (!h->A_csc) {
    CUDA_TRY(cudaMalloc(&h->A_csc, sizeof(double) * std::max<int64_t>(nnz, 1)));
    CUDA_TRY(cudaMalloc(&h->csc_row, sizeof(int32_t) * std::max<int64_t>(nnz, 1)));
  }
  const int gb = (int)std::min<int64_t>(((int64_t)cnt + 255) / 256 + 1, (int64_t)h->num_sms * 16);
  gpl::csc_gather_kernel<<<gb, 256, 0, h->stream>>>(h->A, h->csc_pos, h->m, cnt, h->A_csc, h->csc_row);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return 0;
}

// multi-vector products with B and B^T: gather kernels over G = ceil(t / 32) column groups, rows in the engine's order.
// *prow = rows of the per-warp partial dots the B^T product leaves behind.
int lap_mv_B(gpbdev_vecchia* h, int t, const double* Dinv, const double* X, double* T) {
  gpb_laplace_state* L = h->lap;
  const int G = lap_groups(t), grid = lap_grid(L->grid_mv, G);
  gpl::mv_B_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, h->n, t, G, Dinv, X, T, L->order);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return 0;
}
int lap_mv_Bt(gpbdev_vecchia* h, int t, const double* Tin, const double* W, const double* X, double* V, int* prow) {
  gpb_laplace_state* L = h->lap;
  const int G = lap_groups(t), grid = lap_grid(L->grid_mv, G);
  gpl::mv_Bt_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, h->n, t, G, Tin, W, X, V, L->partial, L->order);
  *prow = grid * (gpl::kBlock / 32) / G;
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return 0;
}

// V = (B^T D^-1 B + W) X, dots[c] = X[:,c] . V[:,c]
int lap_apply_op(gpbdev_vecchia* h, int t, const double* X, double* V, double* Tbuf, double* dots) {
  gpb_laplace_state* L = h->lap;
  const int64_t n = h->n;
  const int G = lap_groups(t), grid = lap_grid(L->grid_mv, G);
  if (t == 1) {
    gpl::v_mv_B_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, n, h->Dinv, X, Tbuf);
    gpl::v_mv_Bt_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->A_csc, h->colptr, h->csc_row, n, Tbuf, L->W, X, V, L->partial);
  } else {
    int prow = 0;
    if (lap_mv_B(h, t, h->Dinv, X, Tbuf)) return -1;
    if (lap_mv_Bt(h, t, Tbuf, L->W, X, V, &prow)) return -1;
    return laplace_colsums(h, t, dots, prow);
  }
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  return laplace_colsums(h, t, dots, grid * (gpl::kBlock / 32) / G);
}

// Z = P^-1 R with P = B^T (D^-1 + W) B;  dots[c] = R[:,c] . Z[:,c]
int lap_precond(gpbdev_vecchia* h, int t, const double* R, double* Z, double* Ybuf, double* dots) {
  gpb_laplace_state* L = h->lap;
  const int64_t n = h->n;
  const double* A = h->A; const int32_t* colptr = h->colptr; const int32_t* csc = h->csc_pos; const int32_t* nn = h->nn;
  int m = h->m; int64_t nn_ = n; int tt = t; const double* dw = L->dw; double* partial = L->partial; int* err = L->err;
  const double* Yc = Ybuf;
  if (t == 1) {
    const int fb = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->num_sms * 16);
    gpl::fill_sentinel_kernel<<<fb, 256, 0, h->stream>>>(Ybuf, n);
    gpl::fill_sentinel_kernel<<<fb, 256, 0, h->stream>>>(Z, n);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    if (coop_launch(h, L->grid_v, gpl::v_trs_bwd_kernel, A, colptr, csc, m, nn_, R, Ybuf, err)) return -1;
    if (coop_launch(h, L->grid_v, gpl::v_trs_fwd_kernel, A, nn, m, nn_, dw, Yc, R, Z, partial, err)) return -1;
  } else {
    const int64_t len = n * t;
    const int fb = (int)std::min<int64_t>((len + 255) / 256, (int64_t)h->num_sms * 16);
    gpl::fill_sentinel_kernel<<<fb, 256, 0, h->stream>>>(Ybuf, len);
    gpl::fill_sentinel_kernel<<<fb, 256, 0, h->stream>>>(Z, len);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    int G = lap_groups(t);
    const int grid = lap_grid(L->grid, G);
    if (coop_launch(h, grid, gpl::trs_bwd_kernel, A, colptr, csc, m, nn_, tt, G, R, Ybuf, err)) return -1;
    if (coop_launch(h, grid, gpl::trs_fwd_kernel, A, nn, m, nn_, tt, G, dw, Yc, R, Z, partial, err)) return -1;
    return laplace_colsums(h, t, dots, grid * (gpl::kBlock / 32) / G);
  }
  return laplace_colsums(h, t, dots, L->grid_v * (gpl::kBlock / 32));
}

int lap_row_stats(gpbdev_vecchia* h, const double* x, const double* W, const double* y, const double* fe, const double* dw, double* out5) {
  gpb_laplace_state* L = h->lap;
  if (L->lik == gpl::kLikPoisson)
    gpl::row_stats_kernel<gpl::kLikPoisson><<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, h->n, h->Dinv, x, W, y, fe, dw, L->partial);
  else
    gpl::row_stats_kernel<gpl::kLikBernoulliLogit><<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, h->n, h->Dinv, x, W, y, fe, dw, L->partial);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (laplace_colsums(h, 5, out5, L->grid_mv * (gpl::kBlock / 32))) return -1;
  if (y && L->lik == gpl::kLikPoisson) out5[2] += L->log_norm_const;  // ll += log_normalizing_constant_ (likelihoods.h:11290)
  return 0;
}

// W, dw = D^-1 + W and (rhs != nullptr) the Newton right-hand side at the current mode
int lap_prep(gpbdev_vecchia* h, const double* fe, double* rhs) {
  gpb_laplace_state* L = h->lap;
  const int eb = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 16);
  if (L->lik == gpl::kLikPoisson)
    gpl::prep_kernel<gpl::kLikPoisson><<<eb, 256, 0, h->stream>>>(h->n, h->y, L->mode, fe, h->Dinv, L->W, rhs, L->dw);
  else
    gpl::prep_kernel<gpl::kLikBernoulliLogit><<<eb, 256, 0, h->stream>>>(h->n, h->y, L->mode, fe, h->Dinv, L->W, rhs, L->dw);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return 0;
}

int lap_check_err(gpbdev_vecchia* h) {
  int e = 0;
  CUDA_TRY(cudaMemcpyAsync(&e, h->lap->err, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (e) return fail("Laplace-Vecchia: a sparse triangular solve timed out waiting for a dependency");
  return 0;
}

// one operator of gpbdev_vecchia_laplace_apply on device multi-vectors X, X2 (n x t); out receives the result, scr is scratch
int lap_apply_run(gpbdev_vecchia* h, int op, int t, const double* X, const double* X2, double* out, double* scr, double* dots) {
  gpb_laplace_state* L = h->lap;
  const int64_t n = h->n;
  const int G = lap_groups(t), grid = lap_grid(L->grid_mv, G);
  double scratch_dots[gpl::kMaxCols];
  CUDA_TRY(cudaMemsetAsync(L->err, 0, sizeof(int), h->stream));
  switch (op) {
    case 0: if (lap_mv_B(h, t, h->Dinv, X, out)) return -1; break;
    case 1: {
      int prow = 0;
      if (lap_mv_Bt(h, t, X, L->W, X2, out, &prow)) return -1;
      if (laplace_colsums(h, t, dots, prow)) return -1;
      break;
    }
    case 2: if (lap_apply_op(h, t, X, out, scr, dots)) return -1; break;
    case 3: if (lap_precond(h, t, X, out, scr, dots)) return -1; break;
    case 4: if (lap_precond(h, t, X, scr, out, scratch_dots)) return -1; break;  // out = the Y buffer: B^-T X
    case 5:
      gpl::mv_Bg_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->dA, h->nn, h->m, n, t, G, X, out);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      break;
    default:
      CUDA_TRY(cudaMemcpyAsync(out, X2, sizeof(double) * (size_t)n * t, cudaMemcpyDeviceToDevice, h->stream));
      gpl::mv_Bgt_kernel<<<grid, gpl::kBlock, 0, h->stream>>>(h->dA, h->colptr, h->csc_pos, h->m, n, t, G, X, out, 1);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      break;
  }
  return lap_check_err(h);
}

}  // namespace

extern "C" {

int gpbdev_vecchia_laplace_set_probes(gpbdev_vecchia_t h, const double* probes_colmajor, int t) {
  if (!h || !probes_colmajor) return fail("gpbdev_vecchia_laplace_set_probes: null argument");
  if (t < 1 || t > gpl::kMaxCols) return fail("gpbdev_vecchia_laplace_set_probes: num_rand_vec_trace must be in [1, 128]");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  gpb_laplace_state* L = h->lap;
  const size_t bytes = sizeof(double) * (size_t)h->n * t;
  if (L->t != t) {
    double** bufs[] = {&L->probes, &L->R, &L->Z, &L->H, &L->V, &L->T, &L->Y};
    for (double** b : bufs) { cudaFree(*b); *b = nullptr; CUDA_TRY(cudaMalloc(b, bytes)); }
    L->t = t;
  }
  if (L->t_total < t || L->allreduce == nullptr) L->t_total = t;
  CUDA_TRY(cudaMemcpy(L->probes, probes_colmajor, bytes, cudaMemcpyHostToDevice));
  return 0;
}

// Multi-GPU: the probe columns of the stochastic Lanczos quadrature are sharded over the ranks (each rank holds the whole
// factor and runs its own columns' PCGs; SURVEY §8e). The only exchanges are one scalar per SLQ iteration (the mean
// residual norm that decides the common early stop, CG_utils.cpp:175-188) and one scalar at the end (the quadrature sum).
int gpbdev_vecchia_laplace_set_collective(gpbdev_vecchia_t h, void (*allreduce_sum)(double*, int), int t_total) {
  if (!h) return fail("gpbdev_vecchia_laplace_set_collective: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  h->lap->allreduce = allreduce_sum;
  h->lap->t_total = t_total;
  return 0;
}

// Laplace-approximated marginal log-likelihood at (var, range): labels come from gpbdev_vecchia_set_y, the optional
// fixed effects in the ORIGINAL data order. cfg: 0 maxit_mode_newton, 1 delta_conv_mode_finding, 2 max lr halvings,
// 3 cg_max_num_it, 4 cg_max_num_it_tridiag, 5 cg_delta_conv, 6 calc log-det (0/1), 7 c_armijo.
// out: 0 approximate NEGATIVE marginal log-likelihood, 1 Newton iterations, 2 CG iterations (total), 3 SLQ iterations,
//      4 log det(Sigma W + I), 5 objective at the mode (log-lik - 0.5 b^T Sigma^-1 b)
int gpbdev_vecchia_laplace_eval(gpbdev_vecchia_t h, int cov_type, double var, double range, const double* fixed_effects_host,
                                const double* cfg, double* out) {
  if (!h || !cfg || !out) return fail("gpbdev_vecchia_laplace_eval: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  gpb_laplace_state* L = h->lap;
  const int64_t n = h->n;
  const int maxit = (int)cfg[0];
  const double delta_mode = cfg[1];
  const int max_shrink = (int)cfg[2];
  const int cg_max = (int)std::min<double>(cfg[3], (double)n);
  const int cg_max_tri = (int)std::min<double>(cfg[4], (double)n);
  const double cg_delta = cfg[5];
  const bool calc_logdet = cfg[6] != 0.;
  const double c_armijo = cfg[7];
  if (calc_logdet && L->t == 0) return fail("gpbdev_vecchia_laplace_eval: call gpbdev_vecchia_laplace_set_probes first");
  // latent factor B, D^-1 (Vecchia_utils.cpp:1367-1699 with gauss_likelihood = false)
  if (launch_eval(h, cov_type, var, range, gpb::MODE_STORE, true)) return -1;
  if (ensure_csc(h)) return -1;
  if (lap_refresh_csc_coefs(h)) return -1;
  const int eb = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->num_sms * 16);
  if (fixed_effects_host) {
    std::memcpy(L->stage, fixed_effects_host, sizeof(double) * n);
    CUDA_TRY(cudaMemcpyAsync(h->y_in, L->stage, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
    gather_perm_kernel<<<eb, 256, 0, h->stream>>>(h->y_in, h->perm, L->fe, n);
    CUDA_TRY(cudaGetLastError());
  }
  const double* fe = fixed_effects_host ? L->fe : nullptr;
  L->fe_set = fixed_effects_host != nullptr;
  L->solutions_valid = false;
  CUDA_TRY(cudaMemsetAsync(L->mode, 0, sizeof(double) * n, h->stream));   // InitializeModeAvec (re_model_template.h:3199-3202)
  CUDA_TRY(cudaMemsetAsync(L->upd, 0, sizeof(double) * n, h->stream));
  CUDA_TRY(cudaMemsetAsync(L->err, 0, sizeof(int), h->stream));
  double st[5];
  if (lap_row_stats(h, L->mode, nullptr, h->y, fe, nullptr, st)) return -1;
  double mll = st[2] - 0.5 * st[0];
  const double sum_log_dinv = st[3];
  double mll_new = mll;
  int it = 0, cg_total = 0;
  bool upd_is_zero = true;
  bool na = false;
  for (it = 0; it < maxit; ++it) {
    if (lap_prep(h, fe, L->rhs)) return -1;
    // ---- CGVecchiaLaplaceVec: (Sigma^-1 + W) upd = rhs, VADU preconditioner, warm start from the previous update
    {
      double dot;
      CUDA_TRY(cudaMemcpyAsync(L->r, L->rhs, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
      if (it == 0 || upd_is_zero) {
        CUDA_TRY(cudaMemsetAsync(L->upd, 0, sizeof(double) * n, h->stream));
      } else {
        if (lap_apply_op(h, 1, L->upd, L->v, L->tt, &dot)) return -1;
        gpl::Coef one; one.v[0] = 1.;
        gpl::v_axpy_norm_kernel<<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, one.v[0], L->v, L->r, nullptr, nullptr, L->partial);
        CUDA_TRY(cudaGetLastError());
        h->launches += 1;
      }
      double rz = 0., rz_new = 0., hv = 0., rr = 0.;
      if (lap_precond(h, 1, L->r, L->z, L->yy, &rz)) return -1;
      CUDA_TRY(cudaMemcpyAsync(L->hv, L->z, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
      int j = 0;
      for (j = 0; j < cg_max; ++j) {
        if (lap_apply_op(h, 1, L->hv, L->v, L->tt, &hv)) return -1;
        gpl::Coef a; a.v[0] = rz / hv;
        gpl::v_axpy_norm_kernel<<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, a.v[0], L->v, L->r, L->hv, L->upd, L->partial);
        CUDA_TRY(cudaGetLastError());
        h->launches += 1;
        if (laplace_colsums(h, 1, &rr, L->grid_mv * (gpl::kBlock / 32))) return -1;
        ++cg_total;
        const double rn = std::sqrt(rr);
        if (!std::isfinite(rn)) { na = true; break; }
        if (rn < cg_delta) break;
        if (lap_precond(h, 1, L->r, L->z, L->yy, &rz_new)) return -1;
        gpl::Coef b; b.v[0] = rz_new / rz;
        rz = rz_new;
        gpl::h_update_kernel<<<eb, 256, 0, h->stream>>>(n, 1, b, L->z, L->hv);
        CUDA_TRY(cudaGetLastError());
        h->launches += 1;
      }
      upd_is_zero = false;
    }
    if (na) { mll_new = std::nan(""); break; }
    // ---- backtracking line search on the Laplace objective (likelihoods.h:3929-3968)
    gpl::lincomb_kernel<<<eb, 256, 0, h->stream>>>(n, 1., L->mode, L->upd, nullptr, L->dir);
    CUDA_TRY(cudaGetLastError());
    h->launches += 1;
    if (lap_row_stats(h, L->dir, L->W, nullptr, nullptr, nullptr, st)) return -1;
    const double grad_dot_dir = st[0] + st[1];
    double lr = 1.;
    for (int ih = 0; ih < max_shrink; ++ih) {
      gpl::lincomb_kernel<<<eb, 256, 0, h->stream>>>(n, lr, L->mode, L->upd, L->mode_new, nullptr);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      if (lap_row_stats(h, L->mode_new, nullptr, h->y, fe, nullptr, st)) return -1;
      mll_new = st[2] - 0.5 * st[0];
      if (mll_new < mll + c_armijo * lr * grad_dot_dir || std::isnan(mll_new) || std::isinf(mll_new)) lr *= 0.5;
      else break;
    }
    std::swap(L->mode, L->mode_new);
    // ---- CheckConvergenceModeFinding (likelihoods.h:16079-16125)
    if (std::isnan(mll_new) || std::isinf(mll_new)) { na = true; mll = mll_new; break; }
    bool stop;
    if (it == 0) stop = std::fabs(mll_new - mll) < delta_mode * std::fabs(mll);
    else stop = (mll_new - mll) < delta_mode * std::fabs(mll);
    mll = mll_new;
    if (stop) break;
  }
  if (lap_check_err(h)) return -1;
  out[1] = it; out[2] = cg_total; out[3] = 0.; out[4] = 0.; out[5] = mll;
  if (na) { out[0] = std::nan(""); return 0; }
  // information at the mode (information_changes_after_mode_finding_)
  if (lap_prep(h, fe, nullptr)) return -1;
  double logdet = 0.;
  if (calc_logdet) {
    const int t = L->t;
    const int64_t len = n * t;
    const int lb = (int)std::min<int64_t>((len + 255) / 256, (int64_t)h->num_sms * 16);
    // z_i = B^T (D^-1 + W)^0.5 r_i  (likelihoods.h:16480-16490)
    gpl::scale_transpose_kernel<<<lb, 256, 0, h->stream>>>(n, t, L->probes, L->dw, L->T);
    CUDA_TRY(cudaGetLastError());
    const int G = lap_groups(t), gridg = lap_grid(L->grid_mv, G), prow = gridg * (gpl::kBlock / 32) / G;
    gpl::mv_Bt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, t, G, L->T, nullptr, L->T, L->R, L->partial, L->order);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    // ---- CGTridiagVecchiaLaplace
    std::vector<double> rz(t), rz_new(t), hvd(t), rr(t), a(t, 1.), a_old(t, 1.), b(t, 0.), b_old(t, 0.);
    std::vector<std::vector<double>> Td(t), Ts(t);
    if (lap_precond(h, t, L->R, L->Z, L->Y, rz.data())) return -1;
    CUDA_TRY(cudaMemcpyAsync(L->H, L->Z, sizeof(double) * len, cudaMemcpyDeviceToDevice, h->stream));
    double* Uacc = nullptr;  // solutions U = (Sigma^-1 + W)^-1 Z of the t systems (CG_utils.cpp:171), for the gradient
    if (L->keep) {
      if (L->U_t != t) { cudaFree(L->U); L->U = nullptr; CUDA_TRY(cudaMalloc(&L->U, sizeof(double) * len)); L->U_t = t; }
      CUDA_TRY(cudaMemsetAsync(L->U, 0, sizeof(double) * len, h->stream));
      Uacc = L->U;
    }
    int j = 0;
    bool early = false;
    for (j = 0; j < cg_max_tri; ++j) {
      if (lap_apply_op(h, t, L->H, L->V, L->T, hvd.data())) return -1;
      a_old = a;
      gpl::Coef ac;
      for (int c = 0; c < t; ++c) { a[c] = rz[c] / hvd[c]; ac.v[c] = a[c]; }
      gpl::axpy_norm_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(n, t, G, ac, L->V, L->R, Uacc ? L->H : nullptr, Uacc, L->partial);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      if (laplace_colsums(h, t, rr.data(), prow)) return -1;
      double mean_norm = 0.;
      for (int c = 0; c < t; ++c) mean_norm += std::sqrt(rr[c]);
      if (L->allreduce) L->allreduce(&mean_norm, 1);
      mean_norm /= L->t_total;
      if (!std::isfinite(mean_norm)) { na = true; break; }
      if (mean_norm < cg_delta) early = true;
      if (lap_precond(h, t, L->R, L->Z, L->Y, rz_new.data())) return -1;
      b_old = b;
      gpl::Coef bc;
      for (int c = 0; c < t; ++c) { b[c] = rz_new[c] / rz[c]; bc.v[c] = b[c]; rz[c] = rz_new[c]; }
      gpl::h_update_kernel<<<lb, 256, 0, h->stream>>>(len, t, bc, L->Z, L->H);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      for (int c = 0; c < t; ++c) {
        Td[c].push_back(1. / a[c] + b_old[c] / a_old[c]);
        if (j > 0) Ts[c].push_back(std::sqrt(b_old[c]) / a_old[c]);
      }
      if (early) { ++j; break; }
    }
    if (lap_check_err(h)) return -1;
    out[3] = j;
    if (na) { out[0] = std::nan(""); return 0; }
    double ldet = 0.;
    for (int c = 0; c < t; ++c) ldet += slq::tridiag_e1_log_e1(Td[c], Ts[c]);
    if (L->allreduce) L->allreduce(&ldet, 1);
    ldet = ldet * (double)n / L->t_total;
    // log|Sigma W + I| = log|P^-1 (Sigma^-1 + W)| + log|P| + log|Sigma|   (likelihoods.h:16505-16511)
    if (lap_row_stats(h, L->mode, nullptr, nullptr, nullptr, L->dw, st)) return -1;
    logdet = ldet - sum_log_dinv + st[4];
    L->solutions_valid = L->keep;
  }
  out[4] = logdet;
  out[0] = -(mll - 0.5 * logdet);
  return 0;
}

// bench hook: device time of one operator application (B^T D^-1 B + W) X and of one preconditioner application B^-1 (D^-1 + W)^-1 B^-T R
// on t columns (t = 1: the Newton system's vectors, t = the probe count: the SLQ block), after gpbdev_vecchia_laplace_eval. CUDA events
// on the engine's stream; mean over `reps` applications after one warm-up. out_ms = {operator, preconditioner}.
int gpbdev_vecchia_laplace_time_ops(gpbdev_vecchia_t h, int t, int reps, float* out_ms) {
  if (!h || !out_ms || reps < 1) return fail("gpbdev_vecchia_laplace_time_ops: bad argument");
  CUDA_TRY(cudaSetDevice(h->device));
  gpb_laplace_state* L = h->lap;
  if (!L || !h->A_csc) return fail("gpbdev_vecchia_laplace_time_ops: run gpbdev_vecchia_laplace_eval first");
  if (t != 1 && t != L->t) return fail("gpbdev_vecchia_laplace_time_ops: t must be 1 or the number of probe columns");
  double dots[gpl::kMaxCols];
  float acc[2] = {0.f, 0.f};
  for (int r = 0; r < reps + 1; ++r) {
    for (int which = 0; which < 2; ++which) {
      CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
      int rc;
      if (which == 0) rc = t == 1 ? lap_apply_op(h, 1, L->hv, L->v, L->tt, dots) : lap_apply_op(h, t, L->H, L->V, L->T, dots);
      else rc = t == 1 ? lap_precond(h, 1, L->r, L->z, L->yy, dots) : lap_precond(h, t, L->R, L->Z, L->Y, dots);
      if (rc) return -1;
      CUDA_TRY(cudaEventRecord(h->ev1, h->stream));
      CUDA_TRY(cudaEventSynchronize(h->ev1));
      float ms = 0.f;
      CUDA_TRY(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
      if (r > 0) acc[which] += ms;
    }
  }
  if (lap_check_err(h)) return -1;
  out_ms[0] = acc[0] / reps; out_ms[1] = acc[1] / reps;
  return 0;
}

// The next evaluation keeps what the gradient needs (the SLQ's CG solutions); costs one more n x t buffer.
int gpbdev_vecchia_laplace_keep_solutions(gpbdev_vecchia_t h, int keep) {
  if (!h) return fail("gpbdev_vecchia_laplace_keep_solutions: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  h->lap->keep = keep != 0;
  return 0;
}

// Gradient of the Laplace-approximated negative log-likelihood w.r.t. (log variance, log range) at the parameters of the
// preceding gpbdev_vecchia_laplace_eval (which must have run with keep_solutions): the reference's
// CalcGradNegMargLikelihoodLaplaceApproxVecchia, iterative branch with the VADU preconditioner (likelihoods.h:6567-6690):
//   explicit part 1/2 (mode^T dSigma^-1 mode + d log|Sigma W + I|), the log-determinant derivative by stochastic trace
//   estimation with the SLQ's probe vectors z and solutions (Sigma^-1 + W)^-1 z, variance-reduced with the preconditioner
//   (CalcLogDetStochDerivCovParVecchia :16706-16781, optimal c CG_utils.cpp:1053-1069), and the implicit part through
//   d mll / d mode (CalcLogDetStochDerivModeVecchia :16651-16692) and one more PCG solve.
// dSigma^-1/dlog(var) = -Sigma^-1 (one GP); dSigma^-1/dlog(range) = Bg^T D^-1 B + B^T D^-1 Bg - B^T D^-1 dD D^-1 B with
// Bg = -dA, dD from the factor kernel's MODE_STORE_GRAD. out[0..1] = gradient on the scale the reference's optimiser uses
// (log of the ORIGINAL range: factor -1, Gaussian kernel -1/2 as in the reference), out[2] = CG iterations of the implicit solve.
// Verified on the H100 against the reference goldens (tests/test_laplace_gpu.py).
int gpbdev_vecchia_laplace_grad(gpbdev_vecchia_t h, int cov_type, double var, double range, const double* cfg, double* out) {
  if (!h || !cfg || !out) return fail("gpbdev_vecchia_laplace_grad: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  gpb_laplace_state* L = h->lap;
  if (!L || !L->solutions_valid) return fail("gpbdev_vecchia_laplace_grad: run gpbdev_vecchia_laplace_eval with keep_solutions first");
  if (L->t != L->t_total) return fail("gpbdev_vecchia_laplace_grad: probe columns sharded over ranks are not supported yet");
  const int64_t n = h->n;
  const int t = L->t;
  const int cg_max = (int)std::min<double>(cfg[3], (double)n);
  const double cg_delta = cfg[5];
  if (!L->c1) {
    double** vecs[] = {&L->c1, &L->c2, &L->c3, &L->dWv};
    for (double** p : vecs) CUDA_TRY(cudaMalloc(p, sizeof(double) * n));
  }
  const double* fe = L->fe_set ? L->fe : nullptr;
  // factor with its range derivative (A, D^-1 are rewritten with the same values)
  if (launch_eval(h, cov_type, var, range, gpb::MODE_STORE_GRAD, true)) return -1;
  const int64_t len = n * t;
  const int lb = (int)std::min<int64_t>((len + 255) / 256, (int64_t)h->num_sms * 16);
  const int eb = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->num_sms * 16);
  const int G = lap_groups(t), gridg = lap_grid(L->grid_mv, G), prow = gridg * (gpl::kBlock / 32) / G;
  const int grid1 = lap_grid(L->grid_mv, 1), prow1 = grid1 * (gpl::kBlock / 32);
  // coefficient vectors, dW, deterministic sums
  double sdet[3];
  if (L->lik == gpl::kLikPoisson)
    gpl::grad_coef_kernel<gpl::kLikPoisson><<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, h->Dinv, h->dD, L->W, L->dw, L->mode, fe, L->c1, L->c2, L->c3, L->dWv, L->partial);
  else
    gpl::grad_coef_kernel<gpl::kLikBernoulliLogit><<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, h->Dinv, h->dD, L->W, L->dw, L->mode, fe, L->c1, L->c2, L->c3, L->dWv, L->partial);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (laplace_colsums(h, 3, sdet, L->grid_mv * (gpl::kBlock / 32))) return -1;
  // Zp = B^T (sqrt(dw) probes) -> R;  PI_Z = P^-1 Zp -> Z
  std::vector<double> dots(t), zA(t), zP(t);
  gpl::scale_transpose_kernel<<<lb, 256, 0, h->stream>>>(n, t, L->probes, L->dw, L->T);
  gpl::mv_Bt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, t, G, L->T, nullptr, L->T, L->R, L->partial, L->order);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  CUDA_TRY(cudaMemsetAsync(L->err, 0, sizeof(int), h->stream));
  if (lap_precond(h, t, L->R, L->Z, L->Y, dots.data())) return -1;
  // d mll / d mode -> rhs;  x = (Sigma^-1 + W)^-1 rhs -> upd (PCG from zero, Inv_SigmaI_plus_ZtWZ_Vecchia_iterative_given_PC)
  gpl::mv_B_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, n, t, G, nullptr, L->Z, L->T, L->order);
  gpl::stoch_dmode_kernel<<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, t, L->U, L->Z, L->T, L->dWv, L->dw, L->rhs);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  int cg_its = 0;
  {
    CUDA_TRY(cudaMemcpyAsync(L->r, L->rhs, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    CUDA_TRY(cudaMemsetAsync(L->upd, 0, sizeof(double) * n, h->stream));
    double rz = 0., rz_new = 0., hv = 0., rr = 0.;
    if (lap_precond(h, 1, L->r, L->z, L->yy, &rz)) return -1;
    CUDA_TRY(cudaMemcpyAsync(L->hv, L->z, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    for (int j = 0; j < cg_max; ++j) {
      if (lap_apply_op(h, 1, L->hv, L->v, L->tt, &hv)) return -1;
      gpl::Coef a; a.v[0] = rz / hv;
      gpl::v_axpy_norm_kernel<<<L->grid_mv, gpl::kBlock, 0, h->stream>>>(n, a.v[0], L->v, L->r, L->hv, L->upd, L->partial);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
      if (laplace_colsums(h, 1, &rr, L->grid_mv * (gpl::kBlock / 32))) return -1;
      ++cg_its;
      const double rn = std::sqrt(rr);
      if (!std::isfinite(rn)) return fail("gpbdev_vecchia_laplace_grad: NaN or Inf in the conjugate gradient solve");
      if (rn < cg_delta) break;
      if (lap_precond(h, 1, L->r, L->z, L->yy, &rz_new)) return -1;
      gpl::Coef b; b.v[0] = rz_new / rz;
      rz = rz_new;
      gpl::h_update_kernel<<<eb, 256, 0, h->stream>>>(n, 1, b, L->z, L->hv);
      CUDA_TRY(cudaGetLastError());
      h->launches += 1;
    }
  }
  using slq::mean;
  using slq::optimal_c;
  double grad[2];
  // ---- j = 0, marginal variance: dSigma^-1 = -Sigma^-1
  double m_v = 0., x_v = 0.;
  {
    gpl::mv_B_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, n, t, G, h->Dinv, L->Z, L->T, L->order);     // T1 = D^-1 B PI_Z
    gpl::mv_Bt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, t, G, L->T, nullptr, L->Z, L->V, L->partial, L->order);  // V = Sigma^-1 PI_Z
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    if (laplace_colsums(h, t, zP.data(), prow)) return -1;  // PI_Z . V
    gpl::coldot_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(n, t, G, L->U, L->V, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 1;
    if (laplace_colsums(h, t, zA.data(), prow)) return -1;
    for (int c = 0; c < t; ++c) { zA[c] = -zA[c]; zP[c] = -zP[c]; }
    // single vector: Sigma^-1 mode -> v
    gpl::mv_B_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(h->A, h->nn, h->m, n, 1, 1, h->Dinv, L->mode, L->tt, L->order);
    gpl::mv_Bt_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, 1, 1, L->tt, nullptr, L->mode, L->v, L->partial, L->order);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    if (laplace_colsums(h, 1, &m_v, prow1)) return -1;
    gpl::coldot_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(n, 1, 1, L->upd, L->v, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 1;
    if (laplace_colsums(h, 1, &x_v, prow1)) return -1;
    const double tr1 = mean(zA), trP = mean(zP);
    const double c = optimal_c(zA, zP, tr1, trP);
    const double d = tr1 + (double)n + c * (-sdet[1]) - c * trP;
    grad[0] = 0.5 * (-m_v + d) + x_v;  // mode^T dSigma^-1 mode = -m_v, implicit term -(x . dSigma^-1 mode) = +x_v
  }
  // ---- j = 1, range
  {
    // T = D^-1 B PI_Z (still valid), Y = Bg PI_Z, H = D^-1 Y - D^-1 dD T, V = B^T H + Bg^T T
    gpl::mv_Bg_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->dA, h->nn, h->m, n, t, G, L->Z, L->Y);
    gpl::rowscale2_kernel<<<lb, 256, 0, h->stream>>>(n, t, h->Dinv, L->Y, L->c1, L->T, L->H);
    gpl::mv_Bt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, t, G, L->H, nullptr, L->Z, L->V, L->partial, L->order);
    gpl::mv_Bgt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->dA, h->colptr, h->csc_pos, h->m, n, t, G, L->T, L->V, 1);
    gpl::coldot_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(n, t, G, L->U, L->V, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 5;
    if (laplace_colsums(h, t, zA.data(), prow)) return -1;
    // dP = dSigma^-1 + B^T W Bg + Bg^T W B:  R = B^T ((D^-1 + W) Y - D^-1 dD T) + Bg^T ((1 + W / D^-1) T)
    gpl::rowscale2_kernel<<<lb, 256, 0, h->stream>>>(n, t, L->c2, L->Y, L->c1, L->T, L->H);
    gpl::mv_Bt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, t, G, L->H, nullptr, L->Z, L->R, L->partial, L->order);
    gpl::rowscale1_kernel<<<lb, 256, 0, h->stream>>>(n, t, L->c3, L->T, L->H);
    gpl::mv_Bgt_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(h->dA, h->colptr, h->csc_pos, h->m, n, t, G, L->H, L->R, 1);
    gpl::coldot_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(n, t, G, L->Z, L->R, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 5;
    if (laplace_colsums(h, t, zP.data(), prow)) return -1;
    // single vector: tt = D^-1 B mode (still valid), yy = Bg mode, z = D^-1 yy - D^-1 dD tt, v = B^T z + Bg^T tt
    gpl::mv_Bg_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(h->dA, h->nn, h->m, n, 1, 1, L->mode, L->yy);
    gpl::rowscale2_kernel<<<eb, 256, 0, h->stream>>>(n, 1, h->Dinv, L->yy, L->c1, L->tt, L->z);
    gpl::mv_Bt_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(h->A, h->colptr, h->csc_pos, h->m, n, 1, 1, L->z, nullptr, L->mode, L->v, L->partial, L->order);
    gpl::mv_Bgt_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(h->dA, h->colptr, h->csc_pos, h->m, n, 1, 1, L->tt, L->v, 1);
    gpl::coldot_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(n, 1, 1, L->mode, L->v, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 5;
    if (laplace_colsums(h, 1, &m_v, prow1)) return -1;
    gpl::coldot_kernel<<<grid1, gpl::kBlock, 0, h->stream>>>(n, 1, 1, L->upd, L->v, L->partial);
    CUDA_TRY(cudaGetLastError());
    h->launches += 1;
    if (laplace_colsums(h, 1, &x_v, prow1)) return -1;
    const double tr1 = mean(zA), trP = mean(zP);
    const double c = optimal_c(zA, zP, tr1, trP);
    const double d = tr1 + sdet[0] + c * (-sdet[2]) - c * trP;
    grad[1] = 0.5 * (m_v + d) - x_v;
  }
  if (lap_check_err(h)) return -1;
  out[0] = grad[0];
  out[1] = grad[1] * (cov_type == gpb::COV_GAUSSIAN ? -0.5 : -1.);
  out[2] = cg_its;
  return 0;
}

// posterior mode of the latent process in the ORIGINAL data order (after gpbdev_vecchia_laplace_eval)
int gpbdev_vecchia_laplace_get_mode(gpbdev_vecchia_t h, double* mode_host) {
  if (!h || !mode_host) return fail("gpbdev_vecchia_laplace_get_mode: null argument");
  if (!h->lap) return fail("gpbdev_vecchia_laplace_get_mode: no Laplace evaluation has been run");
  CUDA_TRY(cudaSetDevice(h->device));
  gpb_laplace_state* L = h->lap;
  const int eb = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 16);
  gpl::scatter_perm_kernel<<<eb, 256, 0, h->stream>>>(h->n, L->mode, h->perm, L->dir);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(L->stage, L->dir, sizeof(double) * h->n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  std::memcpy(mode_host, L->stage, sizeof(double) * h->n);
  return 0;
}

// Test read-back of one operator (include/gpboost_b200_dev.h). Leaves W, dw and the factor as an evaluation would overwrite them
// anyway; the kept SLQ solutions are invalidated, so a gradient needs a new evaluation first.
int gpbdev_vecchia_laplace_apply(gpbdev_vecchia_t h, int cov_type, double var, double range, int op, int t, const double* W_host,
                                 const double* X_host, const double* X2_host, double* out_host, double* dots_host) {
  if (!h) return fail("gpbdev_vecchia_laplace_apply: null handle");
  if (op < 0 || op > 6) return fail("gpbdev_vecchia_laplace_apply: unknown operator " + std::to_string(op));
  if (t < 1 || t > gpl::kMaxCols) return fail("gpbdev_vecchia_laplace_apply: t must be in [1, 128]");
  if (h->m > gpl::kM) return fail("gpbdev_vecchia_laplace_apply: num_neighbors must be <= 30");
  const bool need_x2 = op == 1 || op == 6, need_dots = op >= 1 && op <= 3;
  if (!W_host || !X_host || !out_host || (need_x2 && !X2_host) || (need_dots && !dots_host))
    return fail("gpbdev_vecchia_laplace_apply: null buffer");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  gpb_laplace_state* L = h->lap;
  L->solutions_valid = false;
  if (launch_eval(h, cov_type, var, range, gpb::MODE_STORE_GRAD, true)) return -1;
  if (ensure_csc(h)) return -1;
  if (lap_refresh_csc_coefs(h)) return -1;
  const int64_t n = h->n;
  std::vector<double> dw((size_t)n);
  CUDA_TRY(cudaMemcpyAsync(dw.data(), h->Dinv, sizeof(double) * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  for (int64_t i = 0; i < n; ++i) dw[(size_t)i] += W_host[i];
  CUDA_TRY(cudaMemcpyAsync(L->W, W_host, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyAsync(L->dw, dw.data(), sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  const size_t bytes = sizeof(double) * (size_t)n * t;
  double *X = nullptr, *X2 = nullptr, *out = nullptr, *scr = nullptr;
  cudaError_t e = cudaMalloc(&X, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&X2, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&out, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&scr, bytes);
  if (e == cudaSuccess) e = cudaMemcpyAsync(X, X_host, bytes, cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess && need_x2) e = cudaMemcpyAsync(X2, X2_host, bytes, cudaMemcpyHostToDevice, h->stream);
  int rc = e == cudaSuccess ? 0 : fail(std::string("gpbdev_vecchia_laplace_apply: ") + cudaGetErrorString(e));
  double dots[gpl::kMaxCols];
  if (rc == 0) rc = lap_apply_run(h, op, t, X, X2, out, scr, dots);
  if (rc == 0) {
    e = cudaMemcpyAsync(out_host, out, bytes, cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) rc = fail(std::string("gpbdev_vecchia_laplace_apply: ") + cudaGetErrorString(e));
    else if (need_dots) std::memcpy(dots_host, dots, sizeof(double) * t);
  }
  cudaStreamSynchronize(h->stream);
  cudaFree(X); cudaFree(X2); cudaFree(out); cudaFree(scr);
  return rc;
}

int gpbdev_vecchia_laplace_set_likelihood(gpbdev_vecchia_t h, int likelihood, double log_norm_const) {
  if (!h) return fail("gpbdev_vecchia_laplace_set_likelihood: null handle");
  if (likelihood != GPBDEV_LIK_BERNOULLI_LOGIT && likelihood != GPBDEV_LIK_POISSON)
    return fail("gpbdev_vecchia_laplace_set_likelihood: unknown likelihood " + std::to_string(likelihood));
  if (!std::isfinite(log_norm_const)) return fail("gpbdev_vecchia_laplace_set_likelihood: the normalising constant must be finite");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  gpb_laplace_state* L = h->lap;
  if (L->lik != likelihood) L->solutions_valid = false;
  L->lik = likelihood;
  L->log_norm_const = likelihood == GPBDEV_LIK_POISSON ? log_norm_const : 0.;
  return 0;
}

// Test read-back of the three per-row kernels of one likelihood (include/gpboost_b200_dev.h): stateless, off the hot path.
int gpbdev_laplace_rows(int device, int likelihood, int64_t n, const double* y_host, const double* mode_host, const double* fe_host,
                        const double* Dinv_host, double* out_host) {
  if (likelihood != GPBDEV_LIK_BERNOULLI_LOGIT && likelihood != GPBDEV_LIK_POISSON)
    return fail("gpbdev_laplace_rows: unknown likelihood " + std::to_string(likelihood));
  if (n < 1 || n > (1 << 20)) return fail("gpbdev_laplace_rows: n must be in [1, 2^20]");
  if (!y_host || !mode_host || !Dinv_host || !out_host) return fail("gpbdev_laplace_rows: null buffer");
  CUDA_TRY(cudaSetDevice(device));
  const int rows_per_block = gpl::kBlock / 32;
  const int grid = (int)((n + rows_per_block - 1) / rows_per_block);  // one warp per row in row_stats_kernel
  const size_t nb = sizeof(double) * (size_t)n;
  const size_t pb = sizeof(double) * (size_t)grid * rows_per_block * gpl::kMaxCols;
  double *y = nullptr, *mode = nullptr, *fe = nullptr, *Dinv = nullptr, *dD = nullptr, *W = nullptr, *rhs = nullptr, *dw = nullptr;
  double *c1 = nullptr, *c2 = nullptr, *c3 = nullptr, *dW = nullptr, *partial = nullptr;
  double** bufs[] = {&y, &mode, &fe, &Dinv, &dD, &W, &rhs, &dw, &c1, &c2, &c3, &dW};
  cudaError_t e = cudaSuccess;
  for (double** b : bufs)
    if (e == cudaSuccess) e = cudaMalloc(b, nb);
  if (e == cudaSuccess) e = cudaMalloc(&partial, pb);
  if (e == cudaSuccess) e = cudaMemcpy(y, y_host, nb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(mode, mode_host, nb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && fe_host) e = cudaMemcpy(fe, fe_host, nb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(Dinv, Dinv_host, nb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(dD, 0, nb);
  if (e == cudaSuccess) e = cudaMemset(partial, 0, pb);
  const double* fep = fe_host ? fe : nullptr;
  if (e == cudaSuccess) {
    if (likelihood == GPBDEV_LIK_POISSON) {
      gpl::prep_kernel<gpl::kLikPoisson><<<grid, gpl::kBlock>>>(n, y, mode, fep, Dinv, W, rhs, dw);
      gpl::grad_coef_kernel<gpl::kLikPoisson><<<grid, gpl::kBlock>>>(n, Dinv, dD, W, dw, mode, fep, c1, c2, c3, dW, partial);
      gpl::row_stats_kernel<gpl::kLikPoisson><<<grid, gpl::kBlock>>>(nullptr, nullptr, 0, n, Dinv, mode, nullptr, y, fep, nullptr, partial);
    } else {
      gpl::prep_kernel<gpl::kLikBernoulliLogit><<<grid, gpl::kBlock>>>(n, y, mode, fep, Dinv, W, rhs, dw);
      gpl::grad_coef_kernel<gpl::kLikBernoulliLogit><<<grid, gpl::kBlock>>>(n, Dinv, dD, W, dw, mode, fep, c1, c2, c3, dW, partial);
      gpl::row_stats_kernel<gpl::kLikBernoulliLogit><<<grid, gpl::kBlock>>>(nullptr, nullptr, 0, n, Dinv, mode, nullptr, y, fep, nullptr, partial);
    }
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  // out: 5 x n rows: W, rhs, dw, log-likelihood term of row i (row_stats_kernel, warp i's partial 2), dW
  double* outs[] = {W, rhs, dw, nullptr, dW};
  for (int k = 0; k < 5 && e == cudaSuccess; ++k)
    if (outs[k]) e = cudaMemcpy(out_host + (size_t)k * n, outs[k], nb, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess)
    e = cudaMemcpy2D(out_host + 3 * (size_t)n, sizeof(double), partial + 2, sizeof(double) * gpl::kMaxCols, sizeof(double), (size_t)n,
                     cudaMemcpyDeviceToHost);
  for (double** b : bufs) cudaFree(*b);
  cudaFree(partial);
  if (e != cudaSuccess) return fail(std::string("gpbdev_laplace_rows: ") + cudaGetErrorString(e));
  return 0;
}

}  // extern "C"
