// Vecchia neighbour search on the device: for every ordered point i, the m nearest among points j < i.
//
// Replaces find_nearest_neighbors_Vecchia_fast / find_nearest_neighbors_fast_internal
// (src/GPBoost/Vecchia_utils.cpp:733-985, :1029-1093) and the reference's own CUDA variant
// find_neighbors_kernel (src/GPBoost/cuda_kernel.cu:440-494: one THREAD per query walking the sorted
// coordinate sums, serial insertion sort). The result must be the same int32 sets in the same order:
//   * squared distances use the reference's arithmetic: sequential sum of unfused products
//     (Eigen row redux, x86-64 baseline has no FMA)  -> __dmul_rn / __dadd_rn here;
//   * ties in squared distance are resolved like the reference's walk: candidates are visited alternately
//     below/above the query in the order of the sorted coordinate sums, a later candidate only displaces on
//     strictly smaller distance (:1066) and the insertion sort is stable (utils.h:250-262). That is the
//     lexicographic order (sed, visit_rank) with visit_rank = 2*|pos_j - pos_i| + (pos_j > pos_i), where pos
//     is the rank in the sorted sums (computed by the caller with the same std::sort the reference uses).
//
// Design: a uniform cell list (counting/radix sort by cell, stable so that every cell lists its points
// by increasing index => the "j < i" constraint is a prefix of each cell), one WARP per query scanning
// Chebyshev rings of cells outward until the m-th best distance is inside the scanned radius; the running
// top-m lives one-entry-per-lane and is updated by ballot/shuffle insertion. Early points (few candidates,
// huge search radius) are done by a warp-cooperative brute force.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include <numeric>
#include <string>
#include <vector>

namespace gpb {

struct KnnGrid {
  double lo[3];
  double inv_h[3];
  double hmin;
  int g[3];
  int dim;
};

// What one search did (test read-back gpbdev_knn_search): queries re-derived by the exact replay, kernels launched, first query
// of the cell-list search (= n when every query is brute force) and the cell grid (ncell = 0, g = 0 without one).
struct KnnInfo {
  int64_t replayed = 0;
  int64_t launches = 0;
  int64_t brute_end = 0;
  int64_t ncell = 0;
  int g[3] = {0, 0, 0};
};

__device__ __forceinline__ double knn_sqdist(const double* __restrict__ a, const double* __restrict__ b, int d) {
  double s = 0.;
  for (int k = 0; k < d; ++k) {
    const double t = __dsub_rn(a[k], b[k]);
    s = __dadd_rn(s, __dmul_rn(t, t));
  }
  return s;
}

// lexicographic (sed, rank) "a before b"
__device__ __forceinline__ bool knn_before(double sa, int ra, double sb, int rb) {
  return sa < sb || (sa == sb && ra < rb);
}

// Running top-m of a query, m <= 32 * KS: KS entries per lane, entry (slot, lane) holds position slot * 32 + lane of the list,
// ascending by (sed, rank). KS = 1 is the Vecchia search (m <= 30 neighbours ... 32), KS = 2 serves up to 64 (prediction uses
// 2 m neighbours, re_model_template.h:299; models with 30 < num_neighbors <= 60).
template <int KS>
struct KnnTop {
  double s[KS];
  int r[KS];
  int id[KS];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < KS; ++k) { s[k] = INFINITY; r[k] = 0x7fffffff; id[k] = -1; }
  }
  // entry at list position p (warp-uniform p)
  __device__ __forceinline__ double s_at(int p) const {
    double v = 0.;
#pragma unroll
    for (int k = 0; k < KS; ++k) { const double t = __shfl_sync(0xffffffffu, s[k], p & 31); if ((p >> 5) == k) v = t; }
    return v;
  }
  __device__ __forceinline__ int r_at(int p) const {
    int v = 0;
#pragma unroll
    for (int k = 0; k < KS; ++k) { const int t = __shfl_sync(0xffffffffu, r[k], p & 31); if ((p >> 5) == k) v = t; }
    return v;
  }
};

// insert (cs, cr, cid) if it sorts before the entry at position m-1
template <int KS>
__device__ __forceinline__ void knn_insert(KnnTop<KS>& t, double cs, int cr, int cid, int lane, int m) {
  int posn = 0;  // entries that stay in front of the candidate (the list is sorted: they form a prefix)
#pragma unroll
  for (int k = 0; k < KS; ++k)
    posn += __popc(__ballot_sync(0xffffffffu, knn_before(t.s[k], t.r[k], cs, cr) || (t.s[k] == cs && t.r[k] == cr)));
  if (posn >= m) return;
  // shift positions > posn up by one (the last entry of slot k-1 moves into lane 0 of slot k), then place the candidate
#pragma unroll
  for (int k = KS - 1; k >= 0; --k) {
    double us = __shfl_up_sync(0xffffffffu, t.s[k], 1);
    int ur = __shfl_up_sync(0xffffffffu, t.r[k], 1);
    int ui = __shfl_up_sync(0xffffffffu, t.id[k], 1);
    if (k > 0) {
      const double ps = __shfl_sync(0xffffffffu, t.s[k - 1], 31);
      const int pr = __shfl_sync(0xffffffffu, t.r[k - 1], 31);
      const int pi = __shfl_sync(0xffffffffu, t.id[k - 1], 31);
      if (lane == 0) { us = ps; ur = pr; ui = pi; }
    }
    const int p = k * 32 + lane;
    if (p > posn) { t.s[k] = us; t.r[k] = ur; t.id[k] = ui; }
    else if (p == posn) { t.s[k] = cs; t.r[k] = cr; t.id[k] = cid; }
  }
}

__device__ __forceinline__ int knn_rank(int pj, int pi) {
  const int dlt = pj - pi;
  return dlt < 0 ? (-2 * dlt) : (2 * dlt + 1);
}

// offer one candidate per lane (valid flag), serialised through the warp in lane order
template <int KS>
__device__ __forceinline__ void knn_offer(KnnTop<KS>& t, bool valid, double s, int r, int id, int lane, int m) {
  const double ts = t.s_at(m - 1);  // threshold = entry at position m-1
  const int tr = t.r_at(m - 1);
  unsigned mask = __ballot_sync(0xffffffffu, valid && knn_before(s, r, ts, tr));
  while (mask) {
    const int src = __ffs(mask) - 1;
    mask &= mask - 1;
    const double cs = __shfl_sync(0xffffffffu, s, src);
    const int cr = __shfl_sync(0xffffffffu, r, src);
    const int ci = __shfl_sync(0xffffffffu, id, src);
    knn_insert<KS>(t, cs, cr, ci, lane, m);
  }
}

// The reference's walk prunes a direction as soon as a visited candidate has (sum_j - sum_i)^2 > d * (current m-th
// squared distance) (Vecchia_utils.cpp:1060-1063). In exact arithmetic that never removes a true neighbour; in
// floating point it can when the comparison is decided by rounding (equidistant points on lattices). If every
// neighbour found here satisfies smd <= d * T_final the reference provably visited all of them and the results are
// identical; otherwise the query is queued for knn_walk_kernel, which replays the reference's walk exactly.
template <int KS>
__device__ __forceinline__ void knn_finish(int64_t i, int lane, int m, int d, const KnnTop<KS>& t, const double* __restrict__ csum,
                                           int32_t* __restrict__ nn_row, int32_t* __restrict__ flagged, int* __restrict__ nflag) {
  const double tfin = t.s_at(m - 1);
  bool risky = false;
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    const int p = k * 32 + lane;
    if (p < m) {
      nn_row[p] = t.id[k];
      if (t.id[k] >= 0) {
        const double dd = __dsub_rn(csum[t.id[k]], csum[i]);
        const double smd = __dmul_rn(dd, dd);
        risky = risky || smd > __dmul_rn((double)d, tfin);
      }
    }
  }
  const unsigned any = __ballot_sync(0xffffffffu, risky);
  if (any && lane == 0) flagged[atomicAdd(nflag, 1)] = (int32_t)i;
}

// Exact replay of find_nearest_neighbors_fast_internal (Vecchia_utils.cpp:1029-1093) for the queued queries:
// one thread per query walks the sorted coordinate sums down/up alternately with the reference's pruning rule,
// strict-'<' replacement and stable insertion (utils.h:250-262).
// Candidates of query i are the points c < i with c <= end_search_at (training: end_search_at = n - 1; prediction points are
// appended behind the observed ones and search the observed ones only, Vecchia_utils.cpp:1784-1800). nn row of query i = i - row0.
template <int KS>
__global__ void knn_walk_kernel(const double* __restrict__ coords, const double* __restrict__ csum,
                                const int32_t* __restrict__ sort_sum, const int32_t* __restrict__ pos, int64_t n, int d, int m,
                                int64_t end_search_at, int64_t row0,
                                const int32_t* __restrict__ flagged, const int* __restrict__ nflag, int32_t* __restrict__ nn) {
  const int nf = *nflag;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += gridDim.x * blockDim.x) {
    const int64_t i = flagged[f];
    double sq[32 * KS];
    int id[32 * KS];
    for (int j = 0; j < m; ++j) { sq[j] = INFINITY; id[j] = -1; }
    bool down = true, up = true;
    int64_t up_i = pos[i], down_i = pos[i];
    while (up || down) {
      if (down_i == 0) down = false;
      if (up_i == n - 1) up = false;
      for (int dir = 0; dir < 2; ++dir) {
        if (dir == 0 ? !down : !up) continue;
        const int64_t p = dir == 0 ? --down_i : ++up_i;
        const int c = sort_sum[p];
        if (c < i && c <= end_search_at) {
          const double dd = __dsub_rn(csum[c], csum[i]);
          const double smd = __dmul_rn(dd, dd);
          if (smd > __dmul_rn((double)d, sq[m - 1])) {
            if (dir == 0) down = false; else up = false;
          } else {
            const double sed = knn_sqdist(coords + (int64_t)c * d, coords + i * d, d);
            if (sed < sq[m - 1]) {
              int k = m - 1;
              sq[k] = sed; id[k] = c;
              while (k > 0 && sq[k] < sq[k - 1]) {
                const double v = sq[k]; const int l = id[k];
                sq[k] = sq[k - 1]; id[k] = id[k - 1];
                sq[k - 1] = v; id[k - 1] = l;
                --k;
              }
            }
          }
        }
      }
    }
    for (int j = 0; j < m; ++j) nn[(i - row0) * m + j] = id[j];
  }
}

__global__ void knn_cell_id_kernel(const double* __restrict__ coords, int64_t n, KnnGrid gr, uint32_t* __restrict__ cell,
                                   int32_t* __restrict__ idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t c = 0;
    for (int k = gr.dim - 1; k >= 0; --k) {
      int ck = (int)floor((coords[i * gr.dim + k] - gr.lo[k]) * gr.inv_h[k]);
      ck = min(max(ck, 0), gr.g[k] - 1);
      c = c * (uint32_t)gr.g[k] + (uint32_t)ck;
    }
    cell[i] = c;
    idx[i] = (int32_t)i;
  }
}

__global__ void knn_cell_start_kernel(const uint32_t* __restrict__ sorted_cell, int64_t n, int64_t ncell,
                                      int32_t* __restrict__ cell_start) {
  // cell_start[c] = first position p with sorted_cell[p] >= c ; cell_start[ncell] = n
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p <= n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t cur = p < n ? (int64_t)sorted_cell[p] : ncell;
    const int64_t prev = p > 0 ? (int64_t)sorted_cell[p - 1] : -1;
    for (int64_t c = prev + 1; c <= cur; ++c) cell_start[c] = (int32_t)p;
  }
}

// queries i in [q_begin, q_end): brute force over all j < min(i, end_search_at + 1) — warp per query
template <int KS>
__global__ void knn_brute_kernel(const double* __restrict__ coords, const int32_t* __restrict__ pos,
                                 const double* __restrict__ csum, int d, int m, int64_t q_begin, int64_t q_end, int64_t end_search_at,
                                 int64_t row0, int32_t* __restrict__ nn, int32_t* __restrict__ flagged, int* __restrict__ nflag) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = q_begin + warp; i < q_end; i += nwarps) {
    const int64_t ncand = min(i, end_search_at + 1);
    int32_t* row = nn + (i - row0) * m;
    // Vecchia_utils.cpp:788-813: rows i <= m take all predecessors, in index order. Later rows go through the walk even when
    // they have exactly m candidates (prediction with m = the number of observed points): distance order.
    if (i <= m) {
      for (int p = lane; p < m; p += 32) row[p] = p < ncand ? p : -1;
      continue;
    }
    KnnTop<KS> top; top.init();
    const int pi = pos[i];
    for (int64_t j0 = 0; j0 < ncand; j0 += 32) {
      const int64_t j = j0 + lane;
      const bool valid = j < ncand;
      double s = 0.; int r = 0;
      if (valid) { s = knn_sqdist(coords + j * d, coords + i * d, d); r = knn_rank(pos[j], pi); }
      knn_offer<KS>(top, valid, s, r, (int)j, lane, m);
    }
    knn_finish<KS>(i, lane, m, d, top, csum, row, flagged, nflag);
  }
}

// queries i in [q_begin, n): cell-list search — warp per query, DIM in {1,2,3}
template <int KS>
__global__ void knn_grid_kernel(const double* __restrict__ coords, const int32_t* __restrict__ pos,
                                const double* __restrict__ csum, const int32_t* __restrict__ cell_start,
                                const int32_t* __restrict__ sorted_idx, KnnGrid gr, int m, int64_t q_begin, int64_t n,
                                int64_t end_search_at, int64_t row0,
                                int32_t* __restrict__ nn, int32_t* __restrict__ flagged, int* __restrict__ nflag) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int d = gr.dim;
  for (int64_t i = q_begin + warp; i < n; i += nwarps) {
    KnnTop<KS> top; top.init();
    const int pi = pos[i];
    const int64_t id_end = min(i, end_search_at + 1);  // candidates: ids below this
    int qc[3] = {0, 0, 0};
    for (int k = 0; k < d; ++k) {
      int ck = (int)floor((coords[i * d + k] - gr.lo[k]) * gr.inv_h[k]);
      qc[k] = min(max(ck, 0), gr.g[k] - 1);
    }
    const int rmax = max(max(gr.g[0], gr.g[1]), gr.g[2]);
    for (int r = 0; r <= rmax; ++r) {
      // cells at Chebyshev distance exactly r: enumerate the (2r+1)^d cube, keep the shell
      const int w = 2 * r + 1;
      const int64_t ncube = d == 1 ? w : (d == 2 ? (int64_t)w * w : (int64_t)w * w * w);
      // 2-D shortcut: walk only the 8r ring cells
      const int64_t ncand = (d == 2 && r > 0) ? 8 * (int64_t)r : ncube;
      for (int64_t t0 = 0; t0 < ncand; t0 += 32) {
        const int64_t t = t0 + lane;
        int32_t pb = 0, pe = 0;
        if (t < ncand) {
          int dx = 0, dy = 0, dz = 0;
          if (d == 2 && r > 0) {
            const int side = (int)(t / (2 * r)), off = (int)(t % (2 * r));
            if (side == 0) { dx = -r + off; dy = -r; }
            else if (side == 1) { dx = r; dy = -r + off; }
            else if (side == 2) { dx = r - off; dy = r; }
            else { dx = -r; dy = r - off; }
          } else {
            dx = (int)(t % w) - r;
            dy = d > 1 ? (int)((t / w) % w) - r : 0;
            dz = d > 2 ? (int)(t / ((int64_t)w * w)) - r : 0;
          }
          const bool shell = max(max(abs(dx), abs(dy)), abs(dz)) == r;
          const int cx = qc[0] + dx, cy = qc[1] + dy, cz = qc[2] + dz;
          if (shell && cx >= 0 && cx < gr.g[0] && cy >= 0 && cy < gr.g[1] && cz >= 0 && cz < gr.g[2]) {
            const int64_t c = ((int64_t)cz * gr.g[1] + cy) * gr.g[0] + cx;
            pb = cell_start[c];
            pe = cell_start[c + 1];
          }
        }
        // lock-step scan of each lane's cell; the valid part of a cell is a prefix (indices ascending)
        while (__any_sync(0xffffffffu, pb < pe)) {
          bool valid = false;
          double s = 0.; int rk = 0; int id = -1;
          if (pb < pe) {
            id = sorted_idx[pb];
            if (id < id_end) {
              valid = true;
              s = knn_sqdist(coords + (int64_t)id * d, coords + i * d, d);
              rk = knn_rank(pos[id], pi);
              ++pb;
            } else {
              pb = pe;
            }
          }
          knn_offer<KS>(top, valid, s, rk, id, lane, m);
        }
      }
      // every unscanned point is farther than r*hmin in some coordinate (safety margin for the cell rounding)
      const double ts = top.s_at(m - 1);
      const double reach = (double)r * gr.hmin * (1. - 1e-9);
      if (ts < reach * reach) break;
    }
    knn_finish<KS>(i, lane, m, d, top, csum, nn + (i - row0) * m, flagged, nflag);
  }
}

// First query of the cell-list search: queries with few candidates (the first points of the ordering; every query when there are
// few observed points, or in more than three dimensions) are done by brute force.
inline int64_t knn_brute_end(int64_t n, int d, int64_t end_search_at) {
  if (d > 3 || end_search_at + 1 <= 4096) return n;
  return std::min<int64_t>(n, 4096);
}

// Cell grid over the bounding box of all n points (d <= 3), about n / 8 cells of edge h. Only axes at least as wide as a cell are
// sliced: h is computed from the product of the sliced extents, every axis thinner than h becomes a single slab (g = 1,
// inv_h = 0, like an axis of zero extent), and h is recomputed until no axis is dropped. Otherwise a thin but non-zero axis (a
// nearly flat cloud) would shrink the cells along every axis: billions of cells, and neighbours hundreds of rings apart. The
// widest axis is never dropped, every sliced axis has g <= 2 extent / h, so there are at most 2^d n / 8 cells. Unscanned cells
// differ from the query's cell along a sliced axis, so the ring stop test of knn_grid_kernel stays valid. Returns the cell count.
inline int64_t knn_grid_setup(const double* coords_host, int64_t n, int d, KnnGrid* gr) {
  gr->dim = d;
  double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  for (int k = 0; k < d; ++k) { lo[k] = coords_host[k]; hi[k] = coords_host[k]; }
  for (int64_t i = 0; i < n; ++i)
    for (int k = 0; k < d; ++k) {
      const double v = coords_host[i * d + k];
      lo[k] = std::min(lo[k], v); hi[k] = std::max(hi[k], v);
    }
  bool sliced[3] = {false, false, false};
  for (int k = 0; k < d; ++k) sliced[k] = hi[k] > lo[k];
  const double target_cells = std::max(1.0, (double)n / 8.0);
  double h = 1.0;
  for (bool dropped = true; dropped;) {
    double vol = 1.;
    int active = 0;
    for (int k = 0; k < d; ++k) { if (sliced[k]) { vol *= (hi[k] - lo[k]); ++active; } }
    h = active > 0 ? std::pow(vol / target_cells, 1.0 / active) : 1.0;
    if (!(h > 0.)) h = 1.0;
    dropped = false;
    for (int k = 0; k < d; ++k)
      if (sliced[k] && hi[k] - lo[k] < h) { sliced[k] = false; dropped = true; }
  }
  int64_t ncell = 1;
  gr->hmin = h;
  for (int k = 0; k < 3; ++k) {
    if (k < d && sliced[k]) {
      int gk = (int)std::min<double>(std::ceil((hi[k] - lo[k]) / h), 1 << 20);
      gk = std::max(gk, 1);
      gr->g[k] = gk; gr->lo[k] = lo[k]; gr->inv_h[k] = 1.0 / h;
    } else {
      gr->g[k] = 1; gr->lo[k] = k < d ? lo[k] : 0.; gr->inv_h[k] = 0.;  // thin or degenerate axis: one slab
    }
    ncell *= gr->g[k];
  }
  return ncell;
}

// Returns the number of kernels launched, or -1 with *err set. coords: device n x d row-major (Vecchia order; prediction: the
// observed points followed by the prediction points). Queries are the points [q_begin, n); the candidates of query i are the
// points below min(i, end_search_at + 1); nn_dev holds the rows of the queries only (row of query i = i - q_begin).
// Training: q_begin = 0, end_search_at = n - 2. KS = entries per lane of the running top-m (m <= 32 KS).
template <int KS>
inline int knn_vecchia_device_ks(const double* coords_dev, const double* coords_host, int64_t n, int d, int m,
                                 const int32_t* pos_dev, const int32_t* sort_sum_dev, const double* csum_dev, int32_t* nn_dev,
                                 cudaStream_t stream, int num_sms, KnnInfo* info, std::string* err, int64_t q_begin,
                                 int64_t end_search_at) {
  const int64_t row0 = q_begin;
  auto ck = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess) { *err = std::string(what) + ": " + cudaGetErrorString(e); return false; }
    return true;
  };
  int launches = 0;
  int32_t* flagged = nullptr;
  int* nflag = nullptr;
  if (!ck(cudaMalloc(&flagged, sizeof(int32_t) * n), "cudaMalloc") || !ck(cudaMalloc(&nflag, sizeof(int)), "cudaMalloc") ||
      !ck(cudaMemsetAsync(nflag, 0, sizeof(int), stream), "memset")) return -1;
  auto finish = [&](bool ok) -> int {
    if (ok) {
      knn_walk_kernel<KS><<<num_sms * 4, 128, 0, stream>>>(coords_dev, csum_dev, sort_sum_dev, pos_dev, n, d, m, end_search_at, row0, flagged, nflag, nn_dev);
      ok = ck(cudaGetLastError(), "knn_walk_kernel");
      ++launches;
      int nf = 0;
      if (ok) ok = ck(cudaMemcpyAsync(&nf, nflag, sizeof(int), cudaMemcpyDeviceToHost, stream), "memcpy");
      if (ok) ok = ck(cudaStreamSynchronize(stream), "knn sync");
      info->replayed = nf;
    }
    info->launches = launches;
    cudaFree(flagged); cudaFree(nflag);
    return ok ? launches : -1;
  };
  const int64_t brute_end = knn_brute_end(n, d, end_search_at);
  info->brute_end = brute_end;
  if (brute_end > q_begin) {
    const int blocks = (int)std::min<int64_t>((brute_end - q_begin + 7) / 8, (int64_t)num_sms * 8);
    knn_brute_kernel<KS><<<std::max(blocks, 1), 256, 0, stream>>>(coords_dev, pos_dev, csum_dev, d, m, q_begin, brute_end, end_search_at, row0,
                                                                  nn_dev, flagged, nflag);
    if (!ck(cudaGetLastError(), "knn_brute_kernel")) return finish(false);
    ++launches;
  }
  if (brute_end >= n) return finish(true);
  // ---- cell list over all points (host computes the bounding box: one pass over n x d doubles)
  KnnGrid gr;
  const int64_t ncell = knn_grid_setup(coords_host, n, d, &gr);
  info->ncell = ncell;
  for (int k = 0; k < 3; ++k) info->g[k] = gr.g[k];
  if (ncell >= ((int64_t)1 << 31)) { *err = "cell grid too large"; return finish(false); }
  uint32_t *cell = nullptr, *cell_sorted = nullptr;
  int32_t *idx = nullptr, *idx_sorted = nullptr, *cell_start = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  bool ok = ck(cudaMalloc(&cell, sizeof(uint32_t) * n), "cudaMalloc") && ck(cudaMalloc(&cell_sorted, sizeof(uint32_t) * n), "cudaMalloc") &&
            ck(cudaMalloc(&idx, sizeof(int32_t) * n), "cudaMalloc") && ck(cudaMalloc(&idx_sorted, sizeof(int32_t) * n), "cudaMalloc") &&
            ck(cudaMalloc(&cell_start, sizeof(int32_t) * (ncell + 1)), "cudaMalloc");
  if (ok) {
    knn_cell_id_kernel<<<num_sms * 8, 256, 0, stream>>>(coords_dev, n, gr, cell, idx);
    ok = ck(cudaGetLastError(), "knn_cell_id_kernel");
    ++launches;
  }
  int bits = 1;
  while (((int64_t)1 << bits) < ncell) ++bits;
  if (ok) ok = ck(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, cell, cell_sorted, idx, idx_sorted, (int)n, 0, bits, stream), "cub size");
  if (ok) ok = ck(cudaMalloc(&tmp, tmp_bytes), "cudaMalloc");
  if (ok) {
    ok = ck(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, cell, cell_sorted, idx, idx_sorted, (int)n, 0, bits, stream), "cub sort");
    launches += 4;
  }
  if (ok) {
    knn_cell_start_kernel<<<num_sms * 8, 256, 0, stream>>>(cell_sorted, n, ncell, cell_start);
    ok = ck(cudaGetLastError(), "knn_cell_start_kernel");
    ++launches;
  }
  if (ok) {
    knn_grid_kernel<KS><<<num_sms * 16, 128, 0, stream>>>(coords_dev, pos_dev, csum_dev, cell_start, idx_sorted, gr, m, std::max(brute_end, q_begin), n,
                                                          end_search_at, row0, nn_dev, flagged, nflag);
    ok = ck(cudaGetLastError(), "knn_grid_kernel");
    ++launches;
  }
  if (ok) ok = ck(cudaStreamSynchronize(stream), "knn sync");
  const int rc = finish(ok);
  cudaFree(cell); cudaFree(cell_sorted); cudaFree(idx); cudaFree(idx_sorted); cudaFree(cell_start); cudaFree(tmp);
  return rc;
}

// The whole search from host coordinates: coordinate sums and their ranks on the host, then the device kernels. coords_dev and
// coords_host hold the same n x d row-major points. Model queries: q_begin = 0, end_search_at = n - 2; prediction: q_begin =
// end_search_at + 1 = the number of observed points. m must not exceed end_search_at + 1 (the caller clips it, :752-755).
// Returns the number of kernels launched, or -1 with *err set; synchronises `stream`.
inline int knn_vecchia_search(const double* coords_dev, const double* coords_host, int64_t n, int d, int m, int32_t* nn_dev,
                              cudaStream_t stream, int num_sms, KnnInfo* info, std::string* err, int64_t q_begin,
                              int64_t end_search_at) {
  // rank of every point in the sorted coordinate sums (Vecchia_utils.cpp:775-786). The permutation of equal sums is whatever
  // std::sort yields, so the same library call is made on the same input.
  std::vector<double> csum((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    double sacc = 0.;
    for (int k = 0; k < d; ++k) sacc += coords_host[i * d + k];
    csum[(size_t)i] = sacc;
  }
  std::vector<int> sort_sum((size_t)n);
  std::iota(sort_sum.begin(), sort_sum.end(), 0);
  std::sort(sort_sum.begin(), sort_sum.end(), [&csum](int i1, int i2) { return csum[i1] < csum[i2]; });
  std::vector<int32_t> pos((size_t)n);
  for (int64_t r = 0; r < n; ++r) pos[(size_t)sort_sum[(size_t)r]] = (int32_t)r;
  int32_t *pos_dev = nullptr, *sort_sum_dev = nullptr;
  double* csum_dev = nullptr;
  cudaError_t e = cudaMalloc(&pos_dev, sizeof(int32_t) * n);
  if (e == cudaSuccess) e = cudaMalloc(&sort_sum_dev, sizeof(int32_t) * n);
  if (e == cudaSuccess) e = cudaMalloc(&csum_dev, sizeof(double) * n);
  if (e == cudaSuccess) e = cudaMemcpy(pos_dev, pos.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(sort_sum_dev, sort_sum.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(csum_dev, csum.data(), sizeof(double) * n, cudaMemcpyHostToDevice);
  int rc = -1;
  if (e != cudaSuccess) {
    *err = std::string("upload: ") + cudaGetErrorString(e);
  } else if (m <= 32) {
    rc = knn_vecchia_device_ks<1>(coords_dev, coords_host, n, d, m, pos_dev, sort_sum_dev, csum_dev, nn_dev, stream, num_sms, info, err,
                                  q_begin, end_search_at);
  } else {
    rc = knn_vecchia_device_ks<2>(coords_dev, coords_host, n, d, m, pos_dev, sort_sum_dev, csum_dev, nn_dev, stream, num_sms, info, err,
                                  q_begin, end_search_at);
  }
  if (rc >= 0) {
    e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) { *err = std::string("knn sync: ") + cudaGetErrorString(e); rc = -1; }
  }
  cudaFree(pos_dev); cudaFree(sort_sum_dev); cudaFree(csum_dev);
  return rc;
}

}  // namespace gpb
