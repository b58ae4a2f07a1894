// Device tree learner: histogram construction, split search and data partition for one leaf-wise tree on dense
// uint8 bins (numerical features, no missing values, constant hessian). C ABI in include/gpboost_b200_dev.h.
//
// Replaces, for that configuration, the reference's SerialTreeLearner::Train loop
// (src/LightGBM/treelearner/serial_tree_learner.cpp:159-209) and what it calls:
//   ConstructHistograms :351 -> Dataset::ConstructHistogramsInner (io/dataset.cpp:1143-1245),
//                               DenseBin::ConstructHistogramInner (io/dense_bin.hpp:98-141)
//   FindBestSplitsFromHistograms :375 -> FeatureHistogram::FindBestThreshold / FindBestThresholdSequentially
//                               (feature_histogram.hpp:85-113, 858-960, 1057-1083), Subtract :79, SplitInfo::operator> split_info.hpp:126
//   SplitInner :565 -> DataPartition::Split (data_partition.hpp:101-120), LeafSplits::Init (leaf_splits.hpp:70-110)
// and the reference's own device kernels histogram16/64/256 (treelearner/kernels/histogram_16_64_256.cu: float2 atomics in
// shared memory, sm_60-75 only, split search on the CPU).
//
// Design:
//  * bins live row-major n x Fpad (Fpad = 32-multiple) so one warp reads one 32-byte sector per row: lane = feature;
//  * histogram kernel: one warp per (row chunk, 32-feature group); every lane owns the private shared-memory histogram
//    of ITS feature (grad fp64 + count u32, 96 KB per warp) and walks the chunk's rows in order: no atomics, no
//    inter-lane conflicts by construction, deterministic, and the same accumulation order per feature as the reference's
//    column-wise pass inside a chunk; chunk partials are merged in chunk order by a second kernel;
//  * split kernel: one thread per feature replays the reference's right-to-left scan with identical arithmetic
//    (child sums are the scan's running sums, as in the reference), block arg-max with SplitInfo's tie rule;
//  * partition: flag + exclusive scan (CUB) + scatter = stable, like the reference's ordered partition.
// The leaf loop runs on the host (one small D2H per split); HBM traffic per split = rows_in_smaller_leaf * (Fpad + 12) bytes.
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cub/device/device_scan.cuh>
#include <string>
#include <vector>

namespace {

thread_local std::string g_tree_err;
int tfail(const std::string& m) { g_tree_err = m; return -1; }
#define TCUDA(expr)                                                                                          \
  do {                                                                                                       \
    cudaError_t e__ = (expr);                                                                                \
    if (e__ != cudaSuccess)                                                                                  \
      return tfail(std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) + ": " + cudaGetErrorString(e__)); \
  } while (0)

constexpr int kBins = 256;
constexpr double kEps = (double)1e-15f;  // kEpsilon, include/LightGBM/meta.h:54

struct SplitOut {  // mirrors the fields of SplitInfo the learner consumes (split_info.hpp:22-60)
  double gain;
  double left_output, right_output;
  double left_sum_gradient, left_sum_hessian, right_sum_gradient, right_sum_hessian;
  int feature, threshold, left_count, right_count;
};

struct LeafArgs {
  int leaf;            // -1: inactive; also the row of the per-leaf "splittable" flags
  int hist_slot;
  int inherit;         // 1: features flagged unsplittable in the parent (snapshot in parent_flags) are skipped
  int num_data;
  double sum_gradients, sum_hessians;
};

// Work description for the device-resident leaf loop (tree_*_kernel below): written by one thread between the data-parallel
// kernels of a split, read by every CTA of the next kernel in the stream. Kernels that take a `const DevJob*` use their
// by-value launch parameters when it is null (host-driven loop) and these fields otherwise.
struct DevJob {
  int done, error;
  int do_find;
  int hist_begin, hist_cnt, hist_use_idx, hist_rpc, hist_nchunks;
  LeafArgs a0, a1;
  int parent_row;
  int part_on, part_begin, part_cnt, part_feature, part_threshold, part_seg, part_nseg;
  // ping-pong row-index buffers of the device-resident leaf loop: a split reads its leaf's rows from one buffer and writes the two
  // children (same positions) into the other — no copy back. hist_buf / part_buf: which buffer holds the leaf in question.
  int hist_buf, part_buf;
};

// ---- histogram: lane = feature, private shared histograms, rows of the chunk in order
__global__ void __launch_bounds__(32) hist_kernel(const uint8_t* __restrict__ bins, int Fpad, const int32_t* __restrict__ idx,
                                                   int64_t begin, int64_t count, int64_t rows_per_chunk,
                                                   const double* __restrict__ grad, double* __restrict__ part_g,
                                                   uint32_t* __restrict__ part_c) {
  extern __shared__ __align__(16) unsigned char sm[];
  double* hg = reinterpret_cast<double*>(sm);                        // [32][257]
  uint32_t* hc = reinterpret_cast<uint32_t*>(sm + 32 * 257 * 8);     // [32][257]
  const int lane = threadIdx.x;
  const int chunk = blockIdx.x, fg = blockIdx.y;
  for (int b = 0; b < 257; ++b) { hg[lane * 257 + b] = 0.; hc[lane * 257 + b] = 0u; }
  __syncwarp();
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(r0 + rows_per_chunk, count);
  const uint8_t* bcol = bins + fg * 32 + lane;
  double* mg = hg + lane * 257;
  uint32_t* mc = hc + lane * 257;
  // batches of 32 rows, software-pipelined: the gather of batch k+1 (row ids -> one 32-byte bin sector + one gradient per
  // row) is in flight while the read-modify-writes of batch k run in row order
  constexpr int KB = 32;
  int bcur[KB];
  double gcur[KB];
  auto load_batch = [&](int64_t j0, int* bb, double* gg) {
    const int64_t jl = j0 + lane;
    int64_t rid = 0;
    if (jl < r1) rid = idx ? (int64_t)idx[begin + jl] : (begin + jl);
#pragma unroll
    for (int u = 0; u < KB; ++u) {
      const int64_t r = __shfl_sync(0xffffffffu, rid, u);
      const bool ok = j0 + u < r1;
      bb[u] = ok ? (int)bcol[r * Fpad] : 256;   // slot 256 = scratch for the tail
      gg[u] = ok ? grad[r] : 0.;
    }
  };
  if (r0 < r1) load_batch(r0, bcur, gcur);
  for (int64_t j = r0; j < r1; j += KB) {
    int bnext[KB];
    double gnext[KB];
    const bool more = j + KB < r1;
    if (more) load_batch(j + KB, bnext, gnext);
    // read-modify-write of 4 rows at a time: the four loads are in flight together and equal bins are forwarded in
    // registers, so the result is the one of the row-by-row loop (same additions, same order) at a quarter of the
    // shared-memory round trips on the dependent chain
#pragma unroll
    for (int u = 0; u < KB; u += 4) {
      const int b0 = bcur[u], b1 = bcur[u + 1], b2 = bcur[u + 2], b3 = bcur[u + 3];
      const double h0 = mg[b0], h1 = mg[b1], h2 = mg[b2], h3 = mg[b3];
      const uint32_t c0 = mc[b0], c1 = mc[b1], c2 = mc[b2], c3 = mc[b3];
      const bool e10 = b1 == b0, e20 = b2 == b0, e21 = b2 == b1, e30 = b3 == b0, e31 = b3 == b1, e32 = b3 == b2;
      const double n0 = h0 + gcur[u];
      const double n1 = (e10 ? n0 : h1) + gcur[u + 1];
      const double n2 = (e21 ? n1 : (e20 ? n0 : h2)) + gcur[u + 2];
      const double n3 = (e32 ? n2 : (e31 ? n1 : (e30 ? n0 : h3))) + gcur[u + 3];
      const uint32_t m0 = c0 + 1u;
      const uint32_t m1 = (e10 ? m0 : c1) + 1u;
      const uint32_t m2 = (e21 ? m1 : (e20 ? m0 : c2)) + 1u;
      const uint32_t m3 = (e32 ? m2 : (e31 ? m1 : (e30 ? m0 : c3))) + 1u;
      mg[b0] = n0; mg[b1] = n1; mg[b2] = n2; mg[b3] = n3;
      mc[b0] = m0; mc[b1] = m1; mc[b2] = m2; mc[b3] = m3;
    }
    if (more) {
#pragma unroll
      for (int u = 0; u < KB; ++u) { bcur[u] = bnext[u]; gcur[u] = gnext[u]; }
    }
  }
  __syncwarp();
  // partial[chunk][feature][bin], coalesced over bins
  const int64_t base = ((int64_t)chunk * Fpad + fg * 32) * kBins;
  for (int f = 0; f < 32; ++f)
    for (int b = lane; b < kBins; b += 32) {
      part_g[base + f * kBins + b] = hg[f * 257 + b];
      part_c[base + f * kBins + b] = hc[f * 257 + b];
    }
}

// ---- histogram, multi-warp: one CTA = one row chunk x up to 64 features (all of them at F <= 64), one CTA per SM.
// Warp w owns the four features 4w..4w+3 of the CTA's feature group and a private histogram for them
// (4 x 256 x (f64 + u32) = 12 KB): thirteen accumulation chains per SM at F = 50 instead of the two of the single-warp
// kernel above. Rows of the chunk are staged tile by tile (256 rows, one row per thread: row id -> the row's bins + one
// gradient, through registers one tile ahead) into shared memory TRANSPOSED, tb[feature][row], so that the bins of one
// feature for eight consecutive rows are one aligned 8-byte word. Lane = (row slot 0..7, feature 0..3): eight rows advance
// per step, branch-free:
//   * every lane loads the 8-byte word of its feature and finds the slots holding its own bin with byte-parallel
//     arithmetic (exact zero-byte test of word ^ bin * 0x01010101);
//   * the FIRST slot of every (feature, bin) group is the group's leader: it alone touches the counter — one shared-memory
//     load, its own gradient and then the gradients of the later members in slot order (predicated additions from the
//     step's eight gradients, which every lane holds in registers), one store, one integer RED for the count.
// No atomics on the fp64 sums, no votes, no divergence: the additions on a counter follow a fixed schedule (row order
// inside a step, steps in row order), so the result is deterministic, and a low-cardinality feature (all eight rows in one
// bin) costs the same as a high-cardinality one. (Two earlier versions: groups found with match.any — MATCH.ANY costs
// ~750 cycles when last measured; groups resolved by rank rounds — divergent, and a constant padding feature made its warp 8x slower
// than the others, which then waited at the tile barrier.)
constexpr int kHistTile = 256;
constexpr int kHistMaxWarps = 16;
static inline int hist2_warps(int F) { return std::max(8, std::min(kHistMaxWarps, (std::min(F, 64) + 3) / 4)); }
static inline size_t hist2_smem(int nw) { return (size_t)nw * 4 * kBins * 12 + 64 * kHistTile + kHistTile * 8; }
// bit 7 of every byte of the result is set iff that byte of x is zero (exact: the 7-bit partial sums cannot carry)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu); }
__global__ void __launch_bounds__(kHistMaxWarps * 32, 1) hist2_kernel(const uint8_t* __restrict__ bins, int Fpad, int F,
                                                                      const int32_t* __restrict__ idx, int64_t begin, int64_t count,
                                                                      int64_t rows_per_chunk, const double* __restrict__ grad,
                                                                      double* __restrict__ part_g, uint32_t* __restrict__ part_c,
                                                                      const DevJob* __restrict__ job, const int32_t* __restrict__ idx_alt) {
  if (job) {  // device-resident leaf loop: the leaf's row range comes from the planner kernel
    if (job->done || !job->do_find || (int)blockIdx.x >= job->hist_nchunks) return;
    begin = job->hist_begin; count = job->hist_cnt; rows_per_chunk = job->hist_rpc;
    if (job->hist_buf && idx_alt) idx = idx_alt;
    if (!job->hist_use_idx) idx = nullptr;
  }
  extern __shared__ __align__(16) unsigned char sm[];
  const int nw = blockDim.x >> 5;
  double* hg = reinterpret_cast<double*>(sm);                                   // [nw * 4 features][256]
  uint32_t* hc = reinterpret_cast<uint32_t*>(sm + (size_t)nw * 4 * kBins * 8);  // [nw * 4 features][256]
  uint8_t* tb = reinterpret_cast<uint8_t*>(hc + nw * 4 * kBins);                // [64 features][256 rows]
  double* tg = reinterpret_cast<double*>(tb + 64 * kHistTile);                  // [256 rows]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int chunk = blockIdx.x;
  const int f0 = blockIdx.y * 64;                 // first feature of this CTA's group
  const int gwords = min(16, (Fpad - f0) >> 2);   // 32-bit bin words per row in the group (Fpad is a multiple of 32)
  for (int e = tid; e < nw * 4 * kBins; e += blockDim.x) { hg[e] = 0.; hc[e] = 0u; }
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(r0 + rows_per_chunk, count);
  const bool warp_active = f0 + w * 4 < F;  // a warp of padding features has nothing to accumulate
  const int slot = lane >> 2, fsub = lane & 3;
  const bool feat_ok = f0 + w * 4 + fsub < F;
  double* myg = hg + (w * 4 + fsub) * kBins;
  uint32_t* myc = hc + (w * 4 + fsub) * kBins;
  const uint8_t* mytb = tb + (w * 4 + fsub) * kHistTile;  // this lane's feature: one byte per tile row
  // byte masks (bit 7 of a byte = a row slot of the step): slots in front of / behind this lane's slot
  const unsigned long long all80 = 0x8080808080808080ull;
  const unsigned long long below64 = slot == 0 ? 0ull : (all80 >> (8 * (8 - slot)));
  const unsigned long long above64 = slot == 7 ? 0ull : (all80 << (8 * (slot + 1)));
  const uint32_t blo = (uint32_t)below64, bhi = (uint32_t)(below64 >> 32), alo = (uint32_t)above64, ahi = (uint32_t)(above64 >> 32);
  uint4 s0 = make_uint4(0u, 0u, 0u, 0u), s1 = s0, s2 = s0, s3 = s0;
  double sg = 0.;
  auto load_row = [&](int64_t j) {
    if (tid < kHistTile && j < r1) {
      const int64_t rid = idx ? (int64_t)idx[begin + j] : (begin + j);
      const uint4* src = reinterpret_cast<const uint4*>(bins + rid * Fpad + f0);
      s0 = src[0]; s1 = src[1];
      if (gwords > 8) { s2 = src[2]; s3 = src[3]; }
      sg = grad[rid];
    }
  };
  auto put_word = [&](int c, uint32_t v) {  // bins 4c..4c+3 of row tid -> tb[4c + k][tid]
    tb[(4 * c + 0) * kHistTile + tid] = (uint8_t)(v & 0xffu);
    tb[(4 * c + 1) * kHistTile + tid] = (uint8_t)((v >> 8) & 0xffu);
    tb[(4 * c + 2) * kHistTile + tid] = (uint8_t)((v >> 16) & 0xffu);
    tb[(4 * c + 3) * kHistTile + tid] = (uint8_t)(v >> 24);
  };
  load_row(r0 + tid);
  for (int64_t t0 = r0; t0 < r1; t0 += kHistTile) {
    __syncthreads();  // the previous tile has been consumed (first pass: the zero fill is complete)
    if (tid < kHistTile) {
      put_word(0, s0.x); put_word(1, s0.y); put_word(2, s0.z); put_word(3, s0.w);
      put_word(4, s1.x); put_word(5, s1.y); put_word(6, s1.z); put_word(7, s1.w);
      if (gwords > 8) {
        put_word(8, s2.x); put_word(9, s2.y); put_word(10, s2.z); put_word(11, s2.w);
        put_word(12, s3.x); put_word(13, s3.y); put_word(14, s3.z); put_word(15, s3.w);
      }
      tg[tid] = sg;
    }
    __syncthreads();
    load_row(t0 + kHistTile + tid);  // next tile: in flight while this one is accumulated
    if (!warp_active) continue;
    const int rows = (int)min((int64_t)kHistTile, r1 - t0);
#pragma unroll 2
    for (int b = 0; b < rows; b += 8) {
      // rows b .. b+7 of the tile; nv of them exist
      const int nv = rows - b;
      const unsigned long long vm64 = nv >= 8 ? all80 : (all80 >> (8 * (8 - nv)));
      const uint2 bw = *reinterpret_cast<const uint2*>(mytb + b);  // the 8 bins of my feature
      const double2 ga = *reinterpret_cast<const double2*>(tg + b), gb = *reinterpret_cast<const double2*>(tg + b + 2),
                    gc = *reinterpret_cast<const double2*>(tg + b + 4), gd = *reinterpret_cast<const double2*>(tg + b + 6);
      const double gown = tg[b + slot];
      const uint32_t mybin = (uint32_t)(((((unsigned long long)bw.y << 32) | bw.x) >> (8 * slot)) & 0xffull);
      const uint32_t rep = mybin * 0x01010101u;
      const uint32_t eq_lo = zero_bytes(bw.x ^ rep) & (uint32_t)vm64, eq_hi = zero_bytes(bw.y ^ rep) & (uint32_t)(vm64 >> 32);
      const bool leader = feat_ok && slot < nv && ((eq_lo & blo) | (eq_hi & bhi)) == 0u;
      const uint32_t pa_lo = eq_lo & alo, pa_hi = eq_hi & ahi;  // later members of my group
      if (leader) {
        double v = myg[mybin] + gown;
        if (pa_lo & 0x00008000u) v += ga.y;
        if (pa_lo & 0x00800000u) v += gb.x;
        if (pa_lo & 0x80000000u) v += gb.y;
        if (pa_hi & 0x00000080u) v += gc.x;
        if (pa_hi & 0x00008000u) v += gc.y;
        if (pa_hi & 0x00800000u) v += gd.x;
        if (pa_hi & 0x80000000u) v += gd.y;
        myg[mybin] = v;
        atomicAdd(&myc[mybin], 1u + (uint32_t)__popc(pa_lo) + (uint32_t)__popc(pa_hi));
      }
      __syncwarp();  // the next step's leaders may read counters written by other lanes in this one
    }
  }
  __syncthreads();
  // partial[chunk][feature][bin], coalesced
  const int nfl = min(nw * 4, Fpad - f0);
  const int64_t base = ((int64_t)chunk * Fpad + f0) * kBins;
  for (int e = tid; e < nfl * kBins; e += blockDim.x) {
    part_g[base + e] = hg[e];
    part_c[base + e] = hc[e];
  }
}

// hist3_kernel = hist2_kernel with the two shared-memory savings its ncu capture asks for:
// tile rows padded by 8 bytes (the four 8-byte bin words of a warp fall into different banks: 2 wavefronts instead of 8) and the
// step's gradients loaded only by leaders whose group has later members. The default (GPB200_HIST_KERNEL=3; 4 = the PLAIN_COUNT
// form); tests/test_tree_kernels_gpu.py runs both in every leaf loop.
constexpr int kHist3Stride = kHistTile + 8;
static inline size_t hist3_smem(int nw) { return (size_t)nw * 4 * kBins * 12 + 64 * kHist3Stride + kHistTile * 8; }
// PLAIN_COUNT: the leader updates the integer counter with an ordinary load / add / store like the gradient sum (it is the only lane
// that touches the counter in a step, and steps are separated by __syncwarp) instead of a shared-memory RED: a spread-address
// ATOMS costs ~2 cycles per lane on this part (B300_MICROARCH.md), more than everything else in the step together.
template <bool PLAIN_COUNT>
__global__ void __launch_bounds__(kHistMaxWarps * 32, 1) hist3_kernel(const uint8_t* __restrict__ bins, int Fpad, int F,
                                                                      const int32_t* __restrict__ idx, int64_t begin, int64_t count,
                                                                      int64_t rows_per_chunk, const double* __restrict__ grad,
                                                                      double* __restrict__ part_g, uint32_t* __restrict__ part_c,
                                                                      const DevJob* __restrict__ job, const int32_t* __restrict__ idx_alt) {
  if (job) {  // device-resident leaf loop: the leaf's row range comes from the planner kernel
    if (job->done || !job->do_find || (int)blockIdx.x >= job->hist_nchunks) return;
    begin = job->hist_begin; count = job->hist_cnt; rows_per_chunk = job->hist_rpc;
    if (job->hist_buf && idx_alt) idx = idx_alt;
    if (!job->hist_use_idx) idx = nullptr;
  }
  extern __shared__ __align__(16) unsigned char sm[];
  const int nw = blockDim.x >> 5;
  double* hg = reinterpret_cast<double*>(sm);                                   // [nw * 4 features][256]
  uint32_t* hc = reinterpret_cast<uint32_t*>(sm + (size_t)nw * 4 * kBins * 8);  // [nw * 4 features][256]
  uint8_t* tb = reinterpret_cast<uint8_t*>(hc + nw * 4 * kBins);                // [64 features][kHist3Stride]: rows of the four features of a warp in different banks
  double* tg = reinterpret_cast<double*>(tb + 64 * kHist3Stride);                  // [256 rows]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int chunk = blockIdx.x;
  const int f0 = blockIdx.y * 64;                 // first feature of this CTA's group
  const int gwords = min(16, (Fpad - f0) >> 2);   // 32-bit bin words per row in the group (Fpad is a multiple of 32)
  for (int e = tid; e < nw * 4 * kBins; e += blockDim.x) { hg[e] = 0.; hc[e] = 0u; }
  const int64_t r0 = (int64_t)chunk * rows_per_chunk;
  const int64_t r1 = min(r0 + rows_per_chunk, count);
  const bool warp_active = f0 + w * 4 < F;  // a warp of padding features has nothing to accumulate
  const int slot = lane >> 2, fsub = lane & 3;
  const bool feat_ok = f0 + w * 4 + fsub < F;
  double* myg = hg + (w * 4 + fsub) * kBins;
  uint32_t* myc = hc + (w * 4 + fsub) * kBins;
  const uint8_t* mytb = tb + (w * 4 + fsub) * kHist3Stride;  // this lane's feature: one byte per tile row
  // byte masks (bit 7 of a byte = a row slot of the step): slots in front of / behind this lane's slot
  const unsigned long long all80 = 0x8080808080808080ull;
  const unsigned long long below64 = slot == 0 ? 0ull : (all80 >> (8 * (8 - slot)));
  const unsigned long long above64 = slot == 7 ? 0ull : (all80 << (8 * (slot + 1)));
  const uint32_t blo = (uint32_t)below64, bhi = (uint32_t)(below64 >> 32), alo = (uint32_t)above64, ahi = (uint32_t)(above64 >> 32);
  uint4 s0 = make_uint4(0u, 0u, 0u, 0u), s1 = s0, s2 = s0, s3 = s0;
  double sg = 0.;
  auto load_row = [&](int64_t j) {
    if (tid < kHistTile && j < r1) {
      const int64_t rid = idx ? (int64_t)idx[begin + j] : (begin + j);
      const uint4* src = reinterpret_cast<const uint4*>(bins + rid * Fpad + f0);
      s0 = src[0]; s1 = src[1];
      if (gwords > 8) { s2 = src[2]; s3 = src[3]; }
      sg = grad[rid];
    }
  };
  auto put_word = [&](int c, uint32_t v) {  // bins 4c..4c+3 of row tid -> tb[4c + k][tid]
    tb[(4 * c + 0) * kHist3Stride + tid] = (uint8_t)(v & 0xffu);
    tb[(4 * c + 1) * kHist3Stride + tid] = (uint8_t)((v >> 8) & 0xffu);
    tb[(4 * c + 2) * kHist3Stride + tid] = (uint8_t)((v >> 16) & 0xffu);
    tb[(4 * c + 3) * kHist3Stride + tid] = (uint8_t)(v >> 24);
  };
  load_row(r0 + tid);
  for (int64_t t0 = r0; t0 < r1; t0 += kHistTile) {
    __syncthreads();  // the previous tile has been consumed (first pass: the zero fill is complete)
    if (tid < kHistTile) {
      put_word(0, s0.x); put_word(1, s0.y); put_word(2, s0.z); put_word(3, s0.w);
      put_word(4, s1.x); put_word(5, s1.y); put_word(6, s1.z); put_word(7, s1.w);
      if (gwords > 8) {
        put_word(8, s2.x); put_word(9, s2.y); put_word(10, s2.z); put_word(11, s2.w);
        put_word(12, s3.x); put_word(13, s3.y); put_word(14, s3.z); put_word(15, s3.w);
      }
      tg[tid] = sg;
    }
    __syncthreads();
    load_row(t0 + kHistTile + tid);  // next tile: in flight while this one is accumulated
    if (!warp_active) continue;
    const int rows = (int)min((int64_t)kHistTile, r1 - t0);
#pragma unroll 2
    for (int b = 0; b < rows; b += 8) {
      // rows b .. b+7 of the tile; nv of them exist
      const int nv = rows - b;
      const unsigned long long vm64 = nv >= 8 ? all80 : (all80 >> (8 * (8 - nv)));
      const uint2 bw = *reinterpret_cast<const uint2*>(mytb + b);  // the 8 bins of my feature
      const double gown = tg[b + slot];
      const uint32_t mybin = (uint32_t)(((((unsigned long long)bw.y << 32) | bw.x) >> (8 * slot)) & 0xffull);
      const uint32_t rep = mybin * 0x01010101u;
      const uint32_t eq_lo = zero_bytes(bw.x ^ rep) & (uint32_t)vm64, eq_hi = zero_bytes(bw.y ^ rep) & (uint32_t)(vm64 >> 32);
      const bool leader = feat_ok && slot < nv && ((eq_lo & blo) | (eq_hi & bhi)) == 0u;
      const uint32_t pa_lo = eq_lo & alo, pa_hi = eq_hi & ahi;  // later members of my group
      if (leader) {
        double v = myg[mybin] + gown;
        if (pa_lo | pa_hi) {  // the group has later members (a minority of the leaders): only they load the step's gradients
          const double2 ga = *reinterpret_cast<const double2*>(tg + b), gb = *reinterpret_cast<const double2*>(tg + b + 2),
                        gc = *reinterpret_cast<const double2*>(tg + b + 4), gd = *reinterpret_cast<const double2*>(tg + b + 6);
          if (pa_lo & 0x00008000u) v += ga.y;
          if (pa_lo & 0x00800000u) v += gb.x;
          if (pa_lo & 0x80000000u) v += gb.y;
          if (pa_hi & 0x00000080u) v += gc.x;
          if (pa_hi & 0x00008000u) v += gc.y;
          if (pa_hi & 0x00800000u) v += gd.x;
          if (pa_hi & 0x80000000u) v += gd.y;
        }
        myg[mybin] = v;
        const uint32_t members = 1u + (uint32_t)__popc(pa_lo) + (uint32_t)__popc(pa_hi);
        if (PLAIN_COUNT) myc[mybin] += members;
        else atomicAdd(&myc[mybin], members);
      }
      __syncwarp();  // the next step's leaders may read counters written by other lanes in this one
    }
  }
  __syncthreads();
  // partial[chunk][feature][bin], coalesced
  const int nfl = min(nw * 4, Fpad - f0);
  const int64_t base = ((int64_t)chunk * Fpad + f0) * kBins;
  for (int e = tid; e < nfl * kBins; e += blockDim.x) {
    part_g[base + e] = hg[e];
    part_c[base + e] = hc[e];
  }
}

// merge chunk partials -> hist[slot][f][bin] = (sum grad, count * hess_const)   (dataset.cpp:1223-1226).
// Block = (feature, 32 bins) x 8 warps; warp s sums a contiguous eighth of the chunks in chunk order, then the eight slice
// sums are added in slice order: a fixed summation tree (deterministic), 8 x 32 threads per 32 counters in flight.
constexpr int kReduceSlices = 8;
__global__ void __launch_bounds__(kReduceSlices * 32) hist_reduce_kernel(const double* __restrict__ part_g, const uint32_t* __restrict__ part_c,
                                                                         int nchunks, int Fpad, int F, double hess_const,
                                                                         double* __restrict__ hist, double* __restrict__ parent,
                                                                         const DevJob* __restrict__ job) {
  if (job) {  // device-resident leaf loop of a data-parallel learner: local chunk partials -> the staging histogram that is all-reduced
    if (job->done || !job->do_find) return;
    nchunks = job->hist_nchunks;
  }
  __shared__ double sg[kReduceSlices][32];
  __shared__ unsigned long long sc[kReduceSlices][32];
  const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int f = blockIdx.x / (kBins / 32), b = (blockIdx.x % (kBins / 32)) * 32 + lane;
  const int per = (nchunks + kReduceSlices - 1) / kReduceSlices;
  const int c0 = sl * per, c1 = min(c0 + per, nchunks);
  const int64_t cs = (int64_t)Fpad * kBins, o0 = (int64_t)f * kBins + b;
  double g = 0.;
  unsigned long long c = 0;
  int ch = c0;
  for (; ch + 8 <= c1; ch += 8) {  // eight chunks' loads are issued together
    double gv[8];
    uint32_t cv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { gv[u] = part_g[(ch + u) * cs + o0]; cv[u] = part_c[(ch + u) * cs + o0]; }
#pragma unroll
    for (int u = 0; u < 8; ++u) { g += gv[u]; c += cv[u]; }
  }
  for (; ch < c1; ++ch) {
    g += part_g[ch * cs + o0];
    c += part_c[ch * cs + o0];
  }
  sg[sl][lane] = g;
  sc[sl][lane] = c;
  __syncthreads();
  if (sl != 0) return;
#pragma unroll
  for (int k = 1; k < kReduceSlices; ++k) { g += sg[k][lane]; c += sc[k][lane]; }
  const double hs = (double)c * hess_const;
  const int t = f * kBins + b;
  hist[2 * t] = g;
  hist[2 * t + 1] = hs;
  if (parent) {  // larger = parent - smaller (feature_histogram.hpp:79-83), in place on the parent's slot
    parent[2 * t] -= g;
    parent[2 * t + 1] -= hs;
  }
}

// larger = parent - smaller (feature_histogram.hpp:79-83), in place on the parent's slot
__global__ void hist_subtract_kernel(double* __restrict__ parent, const double* __restrict__ smaller, int n2) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n2) parent[t] -= smaller[t];
}

__device__ __forceinline__ bool split_better(double ga, int fa, double gb, int fb) {  // SplitInfo::operator>
  if (fa == -1) fa = 2147483647;
  if (fb == -1) fb = 2147483647;
  if (ga != gb) return ga > gb;
  return fa < fb;
}

struct ScanScratch {  // per scanning warp
  double rsg[kBins], rsh[kBins];
  int rcn[kBins];
};
// One warp examines one feature of one leaf: h = the feature's histogram in shared memory (16-byte aligned, 2 * nb doubles).
// Replays the reference's right-to-left scan (feature_histogram.hpp:858-960, result :1057-1083); writes the feature's
// candidate to *out and the leaf's "splittable" flag of the feature.
__device__ __forceinline__ void scan_feature(const double* h, int nb, const LeafArgs& a, int f, int lane, int min_data_in_leaf,
                                             double min_sum_hessian, double lambda_l2, double min_gain_to_split,
                                             unsigned char* flags, ScanScratch* scr, SplitOut* out) {
  double* rsg = scr->rsg;
  double* rsh = scr->rsh;
  int* rcn = scr->rcn;
  SplitOut s;
  s.gain = -INFINITY; s.feature = -1; s.threshold = 0; s.left_count = s.right_count = 0;
  s.left_output = s.right_output = 0.;
  s.left_sum_gradient = s.left_sum_hessian = s.right_sum_gradient = s.right_sum_hessian = 0.;
  // The reference walks t = nb-1 .. 1 accumulating the right-hand sums in that order and keeps the FIRST strictly larger
  // gain. Its `continue` / `break` tests are monotone in t (counts and hessian sums only grow), so a threshold is admissible
  // iff it passes all tests itself: lane 0 reproduces the running sums sequentially (fp64 order matters), then all lanes
  // evaluate the gains of their thresholds and the warp picks the maximum, ties to the larger t (= the first one met).
  const double sum_gradient = a.sum_gradients;
  const double sum_hessian = a.sum_hessians + 2 * kEps;
  const double min_gain_shift = (sum_gradient * sum_gradient) / (sum_hessian + lambda_l2) + min_gain_to_split;
  const double cnt_factor = a.num_data / sum_hessian;
  // per-bin counts RoundInt(hess * cnt_factor) (feature_histogram.hpp:899) are independent of the scan: all lanes compute
  // them, then an integer suffix sum (exact in any order) gives the running right-hand count of every threshold
  {
    int cl[kBins / 32];  // lane owns bins 8*lane .. 8*lane+7
    int loc = 0;
#pragma unroll
    for (int u = kBins / 32 - 1; u >= 0; --u) {
      const int t = (kBins / 32) * lane + u;
      const int c = (t >= 1 && t < nb) ? (int)(h[2 * t + 1] * cnt_factor + 0.5f) : 0;
      loc += c;
      cl[u] = loc;  // suffix sum inside the lane's block
    }
    int above = loc;  // inclusive suffix scan over lanes, then make it exclusive
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_down_sync(0xffffffffu, above, o);
      if ((int)lane + o < 32) above += v;
    }
    above -= loc;
#pragma unroll
    for (int u = 0; u < kBins / 32; ++u) rcn[(kBins / 32) * lane + u] = cl[u] + above;
  }
  // the fp64 running sums follow the reference's order (t = nb-1 .. 1, one addition after the other): lane 0, with the
  // loads of eight bins issued together ahead of their dependent additions
  if (lane == 0) {
    double srg = 0., srh = kEps;
    int t = nb - 1;
    while (t >= 1) {
      double gg[8], hh[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = t - u >= 1 ? t - u : 1;
        const double2 v = *reinterpret_cast<const double2*>(&h[2 * tt]);
        gg[u] = v.x; hh[u] = v.y;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (t - u >= 1) { srg += gg[u]; srh += hh[u]; rsg[t - u] = srg; rsh[t - u] = srh; }
      }
      t -= 8;
    }
  }
  __syncwarp();
  double best_gain = -INFINITY;
  int best_t = -1;
  for (int t = nb - 1 - (int)lane; t >= 1; t -= 32) {
    const double srg = rsg[t], srh = rsh[t];
    const int rc = rcn[t];
    if (rc < min_data_in_leaf || srh < min_sum_hessian) continue;
    const int lc = a.num_data - rc;
    if (lc < min_data_in_leaf) continue;
    const double slh = sum_hessian - srh;
    if (slh < min_sum_hessian) continue;
    const double slg = sum_gradient - srg;
    const double gain = (slg * slg) / (slh + lambda_l2) + (srg * srg) / (srh + lambda_l2);
    if (gain <= min_gain_shift) continue;
    if (gain > best_gain) { best_gain = gain; best_t = t; }  // this lane visits its t in descending order
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, best_gain, o);
    const int ot = __shfl_xor_sync(0xffffffffu, best_t, o);
    if (og > best_gain || (og == best_gain && ot > best_t)) { best_gain = og; best_t = ot; }
  }
  if (lane != 0) return;
  const bool spl = best_t >= 1;
  flags[f] = spl ? 1 : 0;
  if (spl) {
    const double srg = rsg[best_t], srh = rsh[best_t];
    const double best_lg = sum_gradient - srg, best_lh = sum_hessian - srh;
    const int best_lc = a.num_data - rcn[best_t];
    s.feature = f; s.threshold = best_t - 1;
    s.left_output = -best_lg / (best_lh + lambda_l2);
    s.left_count = best_lc;
    s.left_sum_gradient = best_lg; s.left_sum_hessian = best_lh - kEps;
    s.right_output = -(sum_gradient - best_lg) / (sum_hessian - best_lh + lambda_l2);
    s.right_count = a.num_data - best_lc;
    s.right_sum_gradient = sum_gradient - best_lg; s.right_sum_hessian = sum_hessian - best_lh - kEps;
    s.gain = best_gain - min_gain_shift;
  }
  *out = s;
}

// block (feature f, leaf slot s): the warp stages the 4 KB histogram row in shared memory, lane 0 replays the reference's
// right-to-left scan (feature_histogram.hpp:858-960, result :1057-1083); per-feature candidates go to cand[s][f]
__global__ void __launch_bounds__(32) split_scan_kernel(const double* __restrict__ hist_base, int64_t slot_stride,
                                                        const int32_t* __restrict__ num_bin, int F, LeafArgs a0, LeafArgs a1,
                                                        int min_data_in_leaf, double min_sum_hessian, double lambda_l2,
                                                        double min_gain_to_split, unsigned char* __restrict__ splittable,
                                                        const unsigned char* __restrict__ parent_flags, SplitOut* __restrict__ cand) {
  const LeafArgs a = blockIdx.y == 0 ? a0 : a1;
  if (a.leaf < 0) return;
  const int f = blockIdx.x;
  __shared__ __align__(16) double h[kBins * 2];
  unsigned char* flags = splittable + (int64_t)a.leaf * F;
  SplitOut s;
  s.gain = -INFINITY; s.feature = -1; s.threshold = 0; s.left_count = s.right_count = 0;
  s.left_output = s.right_output = 0.;
  s.left_sum_gradient = s.left_sum_hessian = s.right_sum_gradient = s.right_sum_hessian = 0.;
  // a feature that had no admissible threshold in the parent is not examined (serial_tree_learner.cpp:329-336)
  const bool skip = a.inherit && !parent_flags[f];
  const int nb = num_bin[f];
  if (!skip) {
    const double* src = hist_base + (int64_t)a.hist_slot * slot_stride + (int64_t)f * kBins * 2;
    double v[kBins * 2 / 32];  // all loads of the 4 KB row in flight before the first store
#pragma unroll
    for (int u = 0; u < kBins * 2 / 32; ++u) { const int t = threadIdx.x + 32 * u; v[u] = t < nb * 2 ? src[t] : 0.; }
#pragma unroll
    for (int u = 0; u < kBins * 2 / 32; ++u) { const int t = threadIdx.x + 32 * u; if (t < nb * 2) h[t] = v[u]; }
  }
  __syncwarp();
  if (skip) {
    if (threadIdx.x == 0) { flags[f] = 0; cand[blockIdx.y * F + f] = s; }
    return;
  }
  __shared__ ScanScratch scr;
  scan_feature(h, nb, a, f, (int)threadIdx.x, min_data_in_leaf, min_sum_hessian, lambda_l2, min_gain_to_split, flags, &scr,
               cand + blockIdx.y * F + f);
}

// ---- merge + subtraction + split scan in one launch (single GPU): block = one feature. 32 warps merge the feature's chunk
// partials (warp = (slice of the chunks, 32 bins), slices added in slice order), 256 threads write the smaller child's
// histogram, take larger = parent - smaller in place (feature_histogram.hpp:79-83) and keep both in shared memory, then
// warp 0 scans the smaller child and warp 1 the larger one straight from there. Replaces hist_reduce_kernel, the snapshot
// of the parent's flags and split_scan_kernel (two launches, one copy and one histogram round trip through L2 per split).
constexpr int kFusedSlices = 4;
__global__ void __launch_bounds__(kFusedSlices * kBins) reduce_scan_kernel(
    const double* __restrict__ part_g, const uint32_t* __restrict__ part_c, int nchunks, int Fpad, int F, double hess_const,
    double* __restrict__ hist_base, int64_t slot_stride, const int32_t* __restrict__ num_bin, LeafArgs a0, LeafArgs a1, int parent_row,
    int min_data_in_leaf, double min_sum_hessian, double lambda_l2, double min_gain_to_split, unsigned char* __restrict__ splittable,
    SplitOut* __restrict__ cand, const DevJob* __restrict__ job) {
  if (job) {
    if (job->done || !job->do_find) return;
    nchunks = job->hist_nchunks; a0 = job->a0; a1 = job->a1; parent_row = job->parent_row;
  }
  __shared__ __align__(16) double hs[2][kBins * 2];
  __shared__ double sg[kFusedSlices][kBins];
  __shared__ unsigned long long sc[kFusedSlices][kBins];
  __shared__ ScanScratch scr[2];
  __shared__ int pflag;
  const int f = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bin = tid & (kBins - 1), sl = tid / kBins;
  // both children inherit the parent's flag of this feature; the left child overwrites it below (same row)
  if (tid == 0) pflag = a0.inherit ? (int)splittable[(int64_t)parent_row * F + f] : 1;
  {
    const int per = (nchunks + kFusedSlices - 1) / kFusedSlices;
    const int c0 = sl * per, c1 = min(c0 + per, nchunks);
    const int64_t cs = (int64_t)Fpad * kBins, o0 = (int64_t)f * kBins + bin;
    double g = 0.;
    unsigned long long c = 0;
    int ch = c0;
    for (; ch + 8 <= c1; ch += 8) {
      double gv[8];
      uint32_t cv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) { gv[u] = part_g[(ch + u) * cs + o0]; cv[u] = part_c[(ch + u) * cs + o0]; }
#pragma unroll
      for (int u = 0; u < 8; ++u) { g += gv[u]; c += cv[u]; }
    }
    for (; ch < c1; ++ch) {
      g += part_g[ch * cs + o0];
      c += part_c[ch * cs + o0];
    }
    sg[sl][bin] = g;
    sc[sl][bin] = c;
  }
  __syncthreads();
  if (tid < kBins) {
    double g = sg[0][bin];
    unsigned long long c = sc[0][bin];
#pragma unroll
    for (int k = 1; k < kFusedSlices; ++k) { g += sg[k][bin]; c += sc[k][bin]; }
    const double hsv = (double)c * hess_const;  // dataset.cpp:1223-1226
    double* dst = hist_base + (int64_t)a0.hist_slot * slot_stride + ((int64_t)f * kBins + bin) * 2;
    dst[0] = g; dst[1] = hsv;
    hs[0][2 * bin] = g; hs[0][2 * bin + 1] = hsv;
    if (a1.leaf >= 0) {
      double* par = hist_base + (int64_t)a1.hist_slot * slot_stride + ((int64_t)f * kBins + bin) * 2;
      const double pg = par[0] - g, ph = par[1] - hsv;
      par[0] = pg; par[1] = ph;
      hs[1][2 * bin] = pg; hs[1][2 * bin + 1] = ph;
    }
  }
  __syncthreads();
  if (warp >= 2) return;
  const LeafArgs a = warp == 0 ? a0 : a1;
  if (a.leaf < 0) return;
  unsigned char* flags = splittable + (int64_t)a.leaf * F;
  SplitOut* out = cand + warp * F + f;
  if (a.inherit && !pflag) {  // no admissible threshold in the parent: not examined (serial_tree_learner.cpp:329-336)
    if (lane == 0) {
      SplitOut s;
      s.gain = -INFINITY; s.feature = -1; s.threshold = 0; s.left_count = s.right_count = 0;
      s.left_output = s.right_output = 0.;
      s.left_sum_gradient = s.left_sum_hessian = s.right_sum_gradient = s.right_sum_hessian = 0.;
      flags[f] = 0;
      *out = s;
    }
    return;
  }
  scan_feature(hs[warp], num_bin[f], a, f, lane, min_data_in_leaf, min_sum_hessian, lambda_l2, min_gain_to_split, flags, &scr[warp], out);
}

// reduce_scan2_kernel = reduce_scan_kernel with the gains of the thresholds evaluated by one thread each (the two fp64 divisions
// per threshold are paid once instead of eight times per lane). The default (GPB200_FUSED_SCAN=2).
// counts + sequential running sums of one child: the first half of scan_feature
__device__ __forceinline__ void scan_sums(const double* h, int nb, const LeafArgs& a, int lane, ScanScratch* scr) {
  double* rsg = scr->rsg;
  double* rsh = scr->rsh;
  int* rcn = scr->rcn;
  const double sum_hessian = a.sum_hessians + 2 * kEps;
  const double cnt_factor = a.num_data / sum_hessian;
  {
    int cl[kBins / 32];
    int loc = 0;
#pragma unroll
    for (int u = kBins / 32 - 1; u >= 0; --u) {
      const int t = (kBins / 32) * lane + u;
      const int c = (t >= 1 && t < nb) ? (int)(h[2 * t + 1] * cnt_factor + 0.5f) : 0;
      loc += c;
      cl[u] = loc;
    }
    int above = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_down_sync(0xffffffffu, above, o);
      if ((int)lane + o < 32) above += v;
    }
    above -= loc;
#pragma unroll
    for (int u = 0; u < kBins / 32; ++u) rcn[(kBins / 32) * lane + u] = cl[u] + above;
  }
  if (lane == 0) {
    double srg = 0., srh = kEps;
    int t = nb - 1;
    while (t >= 1) {
      double gg[8], hh[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = t - u >= 1 ? t - u : 1;
        const double2 v = *reinterpret_cast<const double2*>(&h[2 * tt]);
        gg[u] = v.x; hh[u] = v.y;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (t - u >= 1) { srg += gg[u]; srh += hh[u]; rsg[t - u] = srg; rsh[t - u] = srh; }
      }
      t -= 8;
    }
  }
  __syncwarp();
}
// stage != nullptr (data-parallel learner): the smaller child's histogram has already been merged and summed over the ranks
// (hist_reduce_kernel -> all-reduce); it is taken from there instead of from the chunk partials.
__global__ void __launch_bounds__(kFusedSlices * kBins) reduce_scan2_kernel(
    const double* __restrict__ part_g, const uint32_t* __restrict__ part_c, int nchunks, int Fpad, int F, double hess_const,
    double* __restrict__ hist_base, int64_t slot_stride, const int32_t* __restrict__ num_bin, LeafArgs a0, LeafArgs a1, int parent_row,
    int min_data_in_leaf, double min_sum_hessian, double lambda_l2, double min_gain_to_split, unsigned char* __restrict__ splittable,
    SplitOut* __restrict__ cand, const DevJob* __restrict__ job, const double* __restrict__ stage) {
  if (job) {
    if (job->done || !job->do_find) return;
    nchunks = job->hist_nchunks; a0 = job->a0; a1 = job->a1; parent_row = job->parent_row;
  }
  if (stage) nchunks = 0;
  __shared__ __align__(16) double hs[2][kBins * 2];
  __shared__ double sg[kFusedSlices][kBins];
  __shared__ unsigned long long sc[kFusedSlices][kBins];
  __shared__ ScanScratch scr[2];
  __shared__ int pflag;
  const int f = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bin = tid & (kBins - 1), sl = tid / kBins;
  // both children inherit the parent's flag of this feature; the left child overwrites it below (same row)
  if (tid == 0) pflag = a0.inherit ? (int)splittable[(int64_t)parent_row * F + f] : 1;
  {
    const int per = (nchunks + kFusedSlices - 1) / kFusedSlices;
    const int c0 = sl * per, c1 = min(c0 + per, nchunks);
    const int64_t cs = (int64_t)Fpad * kBins, o0 = (int64_t)f * kBins + bin;
    double g = 0.;
    unsigned long long c = 0;
    int ch = c0;
    for (; ch + 8 <= c1; ch += 8) {
      double gv[8];
      uint32_t cv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) { gv[u] = part_g[(ch + u) * cs + o0]; cv[u] = part_c[(ch + u) * cs + o0]; }
#pragma unroll
      for (int u = 0; u < 8; ++u) { g += gv[u]; c += cv[u]; }
    }
    for (; ch < c1; ++ch) {
      g += part_g[ch * cs + o0];
      c += part_c[ch * cs + o0];
    }
    sg[sl][bin] = g;
    sc[sl][bin] = c;
  }
  __syncthreads();
  if (tid < kBins) {
    double g = sg[0][bin];
    unsigned long long c = sc[0][bin];
#pragma unroll
    for (int k = 1; k < kFusedSlices; ++k) { g += sg[k][bin]; c += sc[k][bin]; }
    double hsv = (double)c * hess_const;  // dataset.cpp:1223-1226
    if (stage) { g = stage[((int64_t)f * kBins + bin) * 2]; hsv = stage[((int64_t)f * kBins + bin) * 2 + 1]; }
    double* dst = hist_base + (int64_t)a0.hist_slot * slot_stride + ((int64_t)f * kBins + bin) * 2;
    dst[0] = g; dst[1] = hsv;
    hs[0][2 * bin] = g; hs[0][2 * bin + 1] = hsv;
    if (a1.leaf >= 0) {
      double* par = hist_base + (int64_t)a1.hist_slot * slot_stride + ((int64_t)f * kBins + bin) * 2;
      const double pg = par[0] - g, ph = par[1] - hsv;
      par[0] = pg; par[1] = ph;
      hs[1][2 * bin] = pg; hs[1][2 * bin + 1] = ph;
    }
  }
  __syncthreads();
  // ---- scan, phase A: per-bin counts and the sequential running sums of both children (warp 0: smaller, warp 1: larger)
  const int nb = num_bin[f];
  if (warp < 2) {
    const LeafArgs a = warp == 0 ? a0 : a1;
    if (a.leaf >= 0 && !(a.inherit && !pflag)) scan_sums(hs[warp], nb, a, lane, &scr[warp]);
  }
  __syncthreads();
  // ---- phase B: one threshold per thread (two fp64 divisions each, once), arg-max with the reference's tie rule
  __shared__ double wbest_g[2][kBins / 32];
  __shared__ int wbest_t[2][kBins / 32];
  if (tid < 2 * kBins) {
    const int child = tid / kBins, t = tid & (kBins - 1);
    const LeafArgs a = child == 0 ? a0 : a1;
    const bool act = a.leaf >= 0 && !(a.inherit && !pflag);
    double gain = -INFINITY;
    int bt = -1;
    if (act && t >= 1 && t <= nb - 1) {
      const double sum_gradient = a.sum_gradients;
      const double sum_hessian = a.sum_hessians + 2 * kEps;
      const double min_gain_shift = (sum_gradient * sum_gradient) / (sum_hessian + lambda_l2) + min_gain_to_split;
      const double srg = scr[child].rsg[t], srh = scr[child].rsh[t];
      const int rc = scr[child].rcn[t];
      const int lc = a.num_data - rc;
      const double slh = sum_hessian - srh;
      if (!(rc < min_data_in_leaf || srh < min_sum_hessian || lc < min_data_in_leaf || slh < min_sum_hessian)) {
        const double slg = sum_gradient - srg;
        const double gv = (slg * slg) / (slh + lambda_l2) + (srg * srg) / (srh + lambda_l2);
        if (!(gv <= min_gain_shift)) { gain = gv; bt = t; }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double og = __shfl_xor_sync(0xffffffffu, gain, o);
      const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
      if (og > gain || (og == gain && ot > bt)) { gain = og; bt = ot; }
    }
    if (lane == 0) { wbest_g[child][t >> 5] = gain; wbest_t[child][t >> 5] = bt; }
  }
  __syncthreads();
  if (tid != 0 && tid != kBins) return;
  const int child = tid / kBins;
  const LeafArgs a = child == 0 ? a0 : a1;
  if (a.leaf < 0) return;
  unsigned char* flags = splittable + (int64_t)a.leaf * F;
  SplitOut s;
  s.gain = -INFINITY; s.feature = -1; s.threshold = 0; s.left_count = s.right_count = 0;
  s.left_output = s.right_output = 0.;
  s.left_sum_gradient = s.left_sum_hessian = s.right_sum_gradient = s.right_sum_hessian = 0.;
  double best_gain = -INFINITY;
  int best_t = -1;
  if (!(a.inherit && !pflag)) {
    for (int k = 0; k < kBins / 32; ++k) {
      const double og = wbest_g[child][k];
      const int ot = wbest_t[child][k];
      if (og > best_gain || (og == best_gain && ot > best_t)) { best_gain = og; best_t = ot; }
    }
  }
  const bool spl = best_t >= 1;
  flags[f] = spl ? 1 : 0;
  if (spl) {
    const double sum_gradient = a.sum_gradients;
    const double sum_hessian = a.sum_hessians + 2 * kEps;
    const double min_gain_shift = (sum_gradient * sum_gradient) / (sum_hessian + lambda_l2) + min_gain_to_split;
    const double srg = scr[child].rsg[best_t], srh = scr[child].rsh[best_t];
    const double best_lg = sum_gradient - srg, best_lh = sum_hessian - srh;
    const int best_lc = a.num_data - scr[child].rcn[best_t];
    s.feature = f; s.threshold = best_t - 1;
    s.left_output = -best_lg / (best_lh + lambda_l2);
    s.left_count = best_lc;
    s.left_sum_gradient = best_lg; s.left_sum_hessian = best_lh - kEps;
    s.right_output = -(sum_gradient - best_lg) / (sum_hessian - best_lh + lambda_l2);
    s.right_count = a.num_data - best_lc;
    s.right_sum_gradient = sum_gradient - best_lg; s.right_sum_hessian = sum_hessian - best_lh - kEps;
    s.gain = best_gain - min_gain_shift;
  }
  cand[child * F + f] = s;
}

// best candidate per leaf with SplitInfo::operator> (gain, then the smaller feature index)
__global__ void split_argmax_kernel(const SplitOut* __restrict__ cand, int F, SplitOut* __restrict__ out) {
  __shared__ SplitOut sh[256];
  SplitOut best;
  best.gain = -INFINITY; best.feature = -1; best.threshold = 0; best.left_count = best.right_count = 0;
  best.left_output = best.right_output = 0.;
  best.left_sum_gradient = best.left_sum_hessian = best.right_sum_gradient = best.right_sum_hessian = 0.;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const SplitOut c = cand[blockIdx.x * F + f];
    if (split_better(c.gain, c.feature, best.gain, best.feature)) best = c;
  }
  sh[threadIdx.x] = best;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const SplitOut& c = sh[threadIdx.x + o];
      if (split_better(c.gain, c.feature, sh[threadIdx.x].gain, sh[threadIdx.x].feature)) sh[threadIdx.x] = c;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = sh[0];
}

__global__ void mark_kernel(const uint8_t* __restrict__ bins, int Fpad, int feature, int threshold, const int32_t* __restrict__ idx,
                            int64_t begin, int64_t count, int32_t* __restrict__ flag) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += (int64_t)gridDim.x * blockDim.x)
    flag[j] = bins[(int64_t)idx[begin + j] * Fpad + feature] <= threshold ? 1 : 0;
}
// stable scatter: lefts keep their order at the front, rights theirs behind (data_partition.hpp:101-120)
__global__ void scatter_kernel(const int32_t* __restrict__ idx, int64_t begin, int64_t count, const int32_t* __restrict__ flag,
                               const int32_t* __restrict__ pos, int32_t nleft, int32_t* __restrict__ out) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t p = pos[j];
    const int64_t dst = flag[j] ? p : (nleft + (j - p));
    out[dst] = idx[begin + j];
  }
}
// ---- stable partition in two kernels (replaces flag + device-wide scan + scatter). Every CTA owns one contiguous segment
// of the leaf's rows. part_count_kernel: go-left flags (one byte per row) + lefts per segment. part_scatter_kernel: every
// CTA sums the segment counts in front of it (<= a few hundred values), then walks its segment tile by tile in row order
// with ballot / popc ranks, so lefts keep their order at the front and rights theirs behind (data_partition.hpp:101-120).
constexpr int kPartThreads = 256;
__global__ void __launch_bounds__(kPartThreads) part_count_kernel(const uint8_t* __restrict__ bins, int Fpad, int feature, int threshold,
                                                                  const int32_t* __restrict__ idx, int64_t begin, int64_t count,
                                                                  int64_t seg, uint8_t* __restrict__ flag, int32_t* __restrict__ seg_left,
                                                                  const DevJob* __restrict__ job, const int32_t* __restrict__ idx_alt) {
  if (job) {
    if (job->done || !job->part_on || (int)blockIdx.x >= job->part_nseg) return;
    feature = job->part_feature; threshold = job->part_threshold; begin = job->part_begin; count = job->part_cnt; seg = job->part_seg;
    if (job->part_buf && idx_alt) idx = idx_alt;
  }
  __shared__ int wsum[kPartThreads / 32];
  const int64_t j0 = (int64_t)blockIdx.x * seg, j1 = min(j0 + seg, count);
  int c = 0;
  for (int64_t j = j0 + threadIdx.x; j < j1; j += kPartThreads) {
    const uint8_t f = bins[(int64_t)idx[begin + j] * Fpad + feature] <= threshold ? 1 : 0;
    flag[j] = f;
    c += f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int k = 0; k < kPartThreads / 32; ++k) t += wsum[k];
    seg_left[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(kPartThreads) part_scatter_kernel(const int32_t* __restrict__ idx, int64_t begin, int64_t count, int64_t seg,
                                                                    const uint8_t* __restrict__ flag, const int32_t* __restrict__ seg_left,
                                                                    int nseg, int32_t* __restrict__ out, int32_t* __restrict__ nleft_out,
                                                                    const DevJob* __restrict__ job, int32_t* __restrict__ idx_alt) {
  // host-driven loop: out = a scratch buffer holding the leaf from position 0. Device-resident loop (idx_alt != null): the two row
  // index buffers alternate — read the leaf from the buffer that holds it, write the children at the same positions of the other one.
  int64_t out_off = 0;
  if (job) {
    if (job->done || !job->part_on || (int)blockIdx.x >= job->part_nseg) return;
    begin = job->part_begin; count = job->part_cnt; seg = job->part_seg; nseg = job->part_nseg;
    if (idx_alt) {
      int32_t* a = const_cast<int32_t*>(idx);
      if (job->part_buf) { idx = idx_alt; out = a; } else { out = idx_alt; }
      out_off = begin;
    }
  }
  __shared__ int red[2][kPartThreads / 32];
  __shared__ int woff[kPartThreads / 32];
  __shared__ int base_s[2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // lefts in the segments before this one, and in all segments
  int before = 0, total = 0;
  for (int k = threadIdx.x; k < nseg; k += kPartThreads) {
    const int v = seg_left[k];
    total += v;
    if (k < (int)blockIdx.x) before += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { before += __shfl_xor_sync(0xffffffffu, before, o); total += __shfl_xor_sync(0xffffffffu, total, o); }
  if (lane == 0) { red[0][wid] = before; red[1][wid] = total; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int b = 0, t = 0;
    for (int k = 0; k < kPartThreads / 32; ++k) { b += red[0][k]; t += red[1][k]; }
    base_s[0] = b; base_s[1] = t;
    if (blockIdx.x == 0 && nleft_out) *nleft_out = t;
  }
  __syncthreads();
  int lefts_before = base_s[0];  // lefts in front of the current tile
  const int nleft = base_s[1];
  const int64_t j0 = (int64_t)blockIdx.x * seg, j1 = min(j0 + seg, count);
  for (int64_t t0 = j0; t0 < j1; t0 += kPartThreads) {
    const int64_t j = t0 + threadIdx.x;
    const bool in = j < j1;
    const bool left = in && flag[j] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, left);
    if (lane == 0) woff[wid] = __popc(bal);
    __syncthreads();
    int wbefore = 0, tile_left = 0;
#pragma unroll
    for (int k = 0; k < kPartThreads / 32; ++k) { const int v = woff[k]; tile_left += v; if (k < wid) wbefore += v; }
    if (in) {
      const int lb = lefts_before + wbefore + __popc(bal & ((1u << lane) - 1u));  // lefts in front of row j
      const int64_t dst = left ? (int64_t)lb : (int64_t)nleft + (j - lb);
      out[out_off + dst] = idx[begin + j];
    }
    lefts_before += tile_left;
    __syncthreads();  // woff is rewritten by the next tile
  }
}
__global__ void iota_kernel(int32_t* p, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = (int32_t)i;
}
// deterministic sum: fixed block partials, then one block
__global__ void sum_stage1_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ part) {
  __shared__ double sh[256];
  double s = 0.;
  const int64_t per = (n + gridDim.x - 1) / gridDim.x;
  const int64_t b = (int64_t)blockIdx.x * per, e = min(b + per, n);
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) s += x[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
// deterministic dot product: fixed block partials (sum_stage2_kernel finishes it)
__global__ void dot_stage1_kernel(const double* __restrict__ x, const double* __restrict__ y, int64_t n, double* __restrict__ part) {
  __shared__ double sh[256];
  double s = 0.;
  const int64_t per = (n + gridDim.x - 1) / gridDim.x;
  const int64_t b = (int64_t)blockIdx.x * per, e = min(b + per, n);
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) s = fma(x[i], y[i], s);
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
__global__ void sum_stage2_kernel(const double* __restrict__ part, int np, double* __restrict__ out) {
  __shared__ double sh[256];
  double s = 0.;
  for (int i = threadIdx.x; i < np; i += blockDim.x) s += part[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) out[0] = sh[0];
}
// score[row] += value[leaf] for the rows of every leaf of the last tree (Tree::AddPredictionToScore via the data partition)
__global__ void add_score_kernel(const int32_t* __restrict__ idx0, const int32_t* __restrict__ idx1, const int32_t* __restrict__ leaf_buf,
                                 const int32_t* __restrict__ leaf_begin,
                                 const int32_t* __restrict__ leaf_cnt, const double* __restrict__ value, double* __restrict__ score,
                                 int32_t* __restrict__ leaf_of_row) {
  const int l = blockIdx.y;
  const int64_t b = leaf_begin[l], c = leaf_cnt[l];
  const double v = value[l];
  const int32_t* __restrict__ idx = leaf_buf[l] ? idx1 : idx0;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < c; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t r = idx[b + j];
    if (score) score[r] += v;
    if (leaf_of_row) leaf_of_row[r] = l;
  }
}

__global__ void sub_kernel(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = a[i] - b[i];
}
__global__ void add_const_kernel(double* __restrict__ a, double c, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] += c;
}


// ---- device-resident leaf loop (single GPU): the state SerialTreeLearner::Train keeps on the host (leaf ranges and sums,
// best split per leaf, the growing tree; serial_tree_learner.cpp:159-209, tree.h:533-575) lives in HBM, one thread advances
// it between the data-parallel kernels, and the host enqueues the kernels of all num_leaves - 1 splits without reading
// anything back: one device-to-host copy per TREE instead of one per split.
constexpr int kMaxLeavesDev = 256;
struct TreeDevState {
  DevJob job;
  int num_leaves, left_leaf, right_leaf, next_slot;
  // leaf_begin / leaf_cnt: this rank's rows of the leaf (partition and histogram ranges); leaf_cnt_g: rows over all ranks — every
  // decision uses the global counts so that all ranks of a data-parallel learner grow the same tree (equal on one GPU)
  int leaf_begin[kMaxLeavesDev], leaf_cnt[kMaxLeavesDev], leaf_cnt_g[kMaxLeavesDev], leaf_depth[kMaxLeavesDev], leaf_parent[kMaxLeavesDev], slot_of[kMaxLeavesDev];
  int leaf_buf[kMaxLeavesDev];  // which of the two row-index buffers holds the leaf's rows
  double leaf_sg[kMaxLeavesDev], leaf_sh[kMaxLeavesDev];
  SplitOut best[kMaxLeavesDev];
  int split_feature[kMaxLeavesDev], threshold_bin[kMaxLeavesDev], left_child[kMaxLeavesDev], right_child[kMaxLeavesDev];
  float split_gain[kMaxLeavesDev];
  double leaf_value[kMaxLeavesDev];
  int leaf_count[kMaxLeavesDev];
};

// BeforeTrain (leaf_splits.hpp:70-83): all rows in leaf 0
__global__ void tree_init_kernel(TreeDevState* __restrict__ st, const double* __restrict__ root_sum_gradient, int n, int n_global, double hess_const, int L) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  st->job.done = 0; st->job.error = 0; st->job.do_find = 0; st->job.part_on = 0;
  st->num_leaves = 1; st->left_leaf = 0; st->right_leaf = -1; st->next_slot = 0;
  for (int l = 0; l < L; ++l) {
    st->leaf_begin[l] = 0; st->leaf_cnt[l] = 0; st->leaf_cnt_g[l] = 0; st->leaf_buf[l] = 0; st->leaf_depth[l] = 0; st->leaf_parent[l] = -1; st->slot_of[l] = -1;
    st->leaf_sg[l] = 0.; st->leaf_sh[l] = 0.;
    st->best[l].gain = -INFINITY; st->best[l].feature = -1;
    st->split_feature[l] = 0; st->threshold_bin[l] = 0; st->left_child[l] = 0; st->right_child[l] = 0; st->split_gain[l] = 0.f;
    st->leaf_value[l] = 0.; st->leaf_count[l] = 0;
  }
  st->leaf_cnt[0] = n;
  st->leaf_cnt_g[0] = n_global;
  st->leaf_sg[0] = root_sum_gradient[0];
  st->leaf_sh[0] = hess_const * (double)n_global;
  st->leaf_count[0] = n_global;
}

// BeforeFindBestSplit (serial_tree_learner.cpp:283-322): may the two newest leaves be examined, which one gets a histogram pass
// keep_part: called from tree_advance_kernel BEFORE the partition of the split that was just selected ran — its job must stay armed
__device__ void tree_plan_body(TreeDevState* __restrict__ st, int max_depth, int min_data_in_leaf, int num_chunk_ctas, bool keep_part) {
  DevJob& job = st->job;
  job.do_find = 0;
  if (!keep_part) job.part_on = 0;
  if (job.done) return;
  const int left_leaf = st->left_leaf, right_leaf = st->right_leaf;
  bool do_find = true;
  if (max_depth > 0 && st->leaf_depth[left_leaf] >= max_depth) do_find = false;
  if (do_find) {
    const int nl = st->leaf_cnt_g[left_leaf], nr = right_leaf >= 0 ? st->leaf_cnt_g[right_leaf] : 0;
    if (nr < min_data_in_leaf * 2 && nl < min_data_in_leaf * 2) do_find = false;
  }
  if (!do_find) {
    st->best[left_leaf].gain = -INFINITY;
    if (right_leaf >= 0) st->best[right_leaf].gain = -INFINITY;
    return;
  }
  int smaller, larger = -1, parent_slot = -1;
  if (right_leaf < 0) smaller = left_leaf;
  else if (st->leaf_cnt_g[left_leaf] < st->leaf_cnt_g[right_leaf]) { smaller = left_leaf; larger = right_leaf; }
  else { smaller = right_leaf; larger = left_leaf; }
  if (right_leaf >= 0) parent_slot = st->slot_of[left_leaf];  // the parent's histograms sit under the left (= parent) id
  const int new_slot = st->next_slot++;
  if (larger >= 0) st->slot_of[larger] = parent_slot;  // larger = parent - smaller, in place
  st->slot_of[smaller] = new_slot;
  LeafArgs a0, a1;
  a0.leaf = smaller; a0.hist_slot = new_slot; a0.inherit = right_leaf >= 0 ? 1 : 0; a0.num_data = st->leaf_cnt_g[smaller];
  a0.sum_gradients = st->leaf_sg[smaller]; a0.sum_hessians = st->leaf_sh[smaller];
  a1.leaf = larger; a1.hist_slot = larger >= 0 ? parent_slot : 0; a1.inherit = 1; a1.num_data = larger >= 0 ? st->leaf_cnt_g[larger] : 0;
  a1.sum_gradients = larger >= 0 ? st->leaf_sg[larger] : 0.; a1.sum_hessians = larger >= 0 ? st->leaf_sh[larger] : 0.;
  job.a0 = a0; job.a1 = a1;
  job.parent_row = left_leaf;
  const int cnt = st->leaf_cnt[smaller];
  job.hist_begin = st->leaf_begin[smaller]; job.hist_cnt = cnt; job.hist_use_idx = st->num_leaves > 1 ? 1 : 0;
  job.hist_buf = st->leaf_buf[smaller];
  int rpc = ((cnt + num_chunk_ctas - 1) / num_chunk_ctas + 7) / 8 * 8;  // same chunking as the host-driven loop
  if (rpc < 128) rpc = 128;
  job.hist_rpc = rpc; job.hist_nchunks = (cnt + rpc - 1) / rpc;
  job.do_find = 1;
}

__global__ void tree_plan_kernel(TreeDevState* __restrict__ st, int max_depth, int min_data_in_leaf, int num_chunk_ctas) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  tree_plan_body(st, max_depth, min_data_in_leaf, num_chunk_ctas, false);
}

// best leaf (ArrayArgs::ArgMax with SplitInfo::operator>), Tree::Split (tree.h:533-575), the partition job
// sharded != 0: the children's LOCAL row ranges are not known before the partition ran (tree_local_ranges_kernel sets them)
__device__ void tree_select_body(TreeDevState* __restrict__ st, const SplitOut* split_dev, double min_gain_to_split, int max_seg, int sharded) {
  DevJob& job = st->job;
  job.part_on = 0;
  if (job.done) return;
  if (job.do_find) {
    st->best[job.a0.leaf] = split_dev[0];
    if (job.a1.leaf >= 0) st->best[job.a1.leaf] = split_dev[1];
  }
  const int num_leaves = st->num_leaves;
  int best_leaf = 0;
  for (int l = 1; l < num_leaves; ++l)
    if (split_better(st->best[l].gain, st->best[l].feature, st->best[best_leaf].gain, st->best[best_leaf].feature)) best_leaf = l;
  const SplitOut bs = st->best[best_leaf];
  if (!(bs.gain > 0.0)) { job.done = 1; return; }
  const int b = st->leaf_begin[best_leaf], c = st->leaf_cnt[best_leaf];
  // constant hessian: the scan's RoundInt counts are the partition's counts (see the host-driven loop)
  const int nleft = bs.left_count, nright = st->leaf_cnt_g[best_leaf] - nleft;
  if (nleft <= 0 || nright <= 0) { job.error = 1; job.done = 1; return; }
  job.part_on = 1; job.part_begin = b; job.part_cnt = c; job.part_feature = bs.feature; job.part_threshold = bs.threshold;
  job.part_buf = st->leaf_buf[best_leaf];
  int seg = ((c + max_seg - 1) / max_seg + kPartThreads - 1) / kPartThreads * kPartThreads;
  if (seg < 4 * kPartThreads) seg = 4 * kPartThreads;
  job.part_seg = seg; job.part_nseg = (c + seg - 1) / seg;
  const int new_leaf = num_leaves;
  st->leaf_buf[best_leaf] = st->leaf_buf[new_leaf] = 1 - job.part_buf;  // the children are written into the other buffer
  st->leaf_cnt_g[best_leaf] = nleft; st->leaf_cnt_g[new_leaf] = nright;
  if (!sharded) { st->leaf_cnt[best_leaf] = nleft; st->leaf_begin[new_leaf] = b + nleft; st->leaf_cnt[new_leaf] = nright; }
  const int node = num_leaves - 1;
  const int parent = st->leaf_parent[best_leaf];
  if (parent >= 0) { if (st->left_child[parent] == ~best_leaf) st->left_child[parent] = node; else st->right_child[parent] = node; }
  st->split_feature[node] = bs.feature; st->threshold_bin[node] = bs.threshold;
  st->split_gain[node] = (float)(bs.gain + min_gain_to_split);
  st->left_child[node] = ~best_leaf; st->right_child[node] = ~new_leaf;
  st->leaf_parent[best_leaf] = node; st->leaf_parent[new_leaf] = node;
  st->leaf_value[best_leaf] = isnan(bs.left_output) ? 0. : bs.left_output; st->leaf_count[best_leaf] = nleft;
  st->leaf_value[new_leaf] = isnan(bs.right_output) ? 0. : bs.right_output; st->leaf_count[new_leaf] = nright;
  st->leaf_depth[new_leaf] = st->leaf_depth[best_leaf] + 1; st->leaf_depth[best_leaf]++;
  st->leaf_sg[best_leaf] = bs.left_sum_gradient; st->leaf_sh[best_leaf] = bs.left_sum_hessian;
  st->leaf_sg[new_leaf] = bs.right_sum_gradient; st->leaf_sh[new_leaf] = bs.right_sum_hessian;
  st->best[best_leaf].gain = -INFINITY; st->best[best_leaf].feature = -1;
  st->best[new_leaf].gain = -INFINITY; st->best[new_leaf].feature = -1;
  st->num_leaves = num_leaves + 1;
  st->left_leaf = best_leaf; st->right_leaf = new_leaf;
}

__global__ void tree_select_kernel(TreeDevState* __restrict__ st, const SplitOut* __restrict__ split_dev, double min_gain_to_split, int max_seg,
                                   int sharded) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  tree_select_body(st, split_dev, min_gain_to_split, max_seg, sharded);
}

// One launch instead of three between the split scan and the partition (single GPU): arg-max over the per-feature candidates of both
// children (split_argmax_kernel), the selector (tree_select_kernel) and the planner of the NEXT split (tree_plan_kernel — on one GPU it
// needs nothing the partition produces: the children's ranges follow from the split's counts).
__global__ void __launch_bounds__(128) tree_advance_kernel(TreeDevState* __restrict__ st, const SplitOut* __restrict__ cand, int F, double min_gain_to_split,
                                                           int max_seg, int max_depth, int min_data_in_leaf, int num_chunk_ctas, int plan_next) {
  __shared__ SplitOut sh[128];
  __shared__ SplitOut best2[2];
  const int child = threadIdx.x >> 6, t = threadIdx.x & 63;
  SplitOut best;
  best.gain = -INFINITY; best.feature = -1; best.threshold = 0; best.left_count = best.right_count = 0;
  best.left_output = best.right_output = 0.;
  best.left_sum_gradient = best.left_sum_hessian = best.right_sum_gradient = best.right_sum_hessian = 0.;
  const bool find = !st->job.done && st->job.do_find;
  if (find) {
    for (int f = t; f < F; f += 64) {
      const SplitOut c = cand[child * F + f];
      if (split_better(c.gain, c.feature, best.gain, best.feature)) best = c;
    }
  }
  sh[threadIdx.x] = best;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) {
    if (t < o) {
      const SplitOut& c = sh[threadIdx.x + o];
      if (split_better(c.gain, c.feature, sh[threadIdx.x].gain, sh[threadIdx.x].feature)) sh[threadIdx.x] = c;
    }
    __syncthreads();
  }
  if (t == 0) best2[child] = sh[threadIdx.x];
  __syncthreads();
  if (threadIdx.x != 0) return;
  tree_select_body(st, best2, min_gain_to_split, max_seg, 0);
  if (plan_next) tree_plan_body(st, max_depth, min_data_in_leaf, num_chunk_ctas, true);
}

// data-parallel learner: after the local partition, the children's ranges on THIS rank (lefts counted by part_count_kernel)
__global__ void tree_local_ranges_kernel(TreeDevState* __restrict__ st, const int32_t* __restrict__ seg_left) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const DevJob& job = st->job;
  if (job.done || !job.part_on) return;
  int nl = 0;
  for (int k = 0; k < job.part_nseg; ++k) nl += seg_left[k];
  const int best_leaf = st->left_leaf, new_leaf = st->right_leaf;
  st->leaf_cnt[best_leaf] = nl;
  st->leaf_begin[new_leaf] = job.part_begin + nl;
  st->leaf_cnt[new_leaf] = job.part_cnt - nl;
}

}  // namespace

struct gpbdev_tree {
  int device = 0, num_sms = 0;
  int64_t n = 0;
  int F = 0, Fpad = 0, L = 0;
  gpbdev_tree_config cfg;
  cudaStream_t stream = nullptr;
  const uint8_t* bins = nullptr;  // n x Fpad row-major (bins_owned, or a Dataset's device matrix read in place)
  uint8_t* bins_owned = nullptr;
  int32_t* leaf_of_row = nullptr;  // n, lazy (gpbdev_tree_leaf_indices)
  double* stage = nullptr;         // F x 256 x 2: the smaller child's merged histogram on its way through the all-reduce (data-parallel)
  int32_t* num_bin = nullptr;     // F
  int32_t *idx = nullptr, *idx_tmp = nullptr, *flag = nullptr, *pos = nullptr;
  double* grad = nullptr;         // n (device copy when the caller passes host gradients)
  double* hist = nullptr;         // (L + 1) slots x F x 256 x 2
  unsigned char* splittable = nullptr;  // L x F, row = leaf id (FeatureHistogram::is_splittable_)
  unsigned char* parent_flags = nullptr; // F: snapshot of the parent's flags while its two children are examined
  double* part_g = nullptr;
  uint32_t* part_c = nullptr;
  int max_chunks = 0;
  uint8_t* flag8 = nullptr;        // n go-left flags of the leaf being split
  int32_t* seg_left = nullptr;     // lefts per partition segment
  int32_t* nleft_dev = nullptr;
  int32_t* nleft_host = nullptr;   // pinned
  int max_seg = 0;
  cudaGraphExec_t graph_exec = nullptr;  // GPB200_TREE_LOOP=graph
  const double* graph_grad = nullptr;
  double graph_hess = 0.;
  // Implementation switches (environment, read at creation; every combination below passes the same parity tests,
  // tests/test_tree_kernels_gpu.py runs every combination against the oracle). Defaults = the fastest verified set.
  int device_loop = 2;             // GPB200_TREE_LOOP = graph (2, default) | device (1) | host (0). Row-sharded learners use the host loop.
  TreeDevState* state_dev = nullptr;
  TreeDevState* state_host = nullptr;  // pinned
  int fused_scan = 2;              // GPB200_FUSED_SCAN = 2 (default): reduce_scan2_kernel | 1: reduce_scan_kernel | 0: hist_reduce_kernel + split_scan_kernel
  int fused_advance = 1;           // GPB200_FUSED_ADVANCE = 1 (default): arg-max + selector + next planner in one launch (single GPU) | 0: three launches
  int sharded_graph = 0;           // GPB200_SHARDED_LOOP = graph: capture the data-parallel leaf loop (NCCL kernels included) in a CUDA graph
  int sharded_host_loop = 0;       // GPB200_SHARDED_LOOP = host: data-parallel learners use the host-driven leaf loop (one blocking all-reduce and one
                                   // D2H per split, CUB partition) instead of the device-resident / graph loop with in-stream all-reduces
  int partition_version = 2;       // GPB200_PARTITION = 2 (default): part_count_kernel + part_scatter_kernel | 1: flag + CUB scan + scatter
  int hist_kernel_version = 3;     // GPB200_HIST_KERNEL = 3 (default): hist3_kernel, RED counters | 4: hist3_kernel with plain counter updates (measured 7 % slower)
                                   // | 2: hist2_kernel | 1: single-warp hist_kernel
  double* sum_part = nullptr;
  SplitOut* split_dev = nullptr;
  SplitOut* cand_dev = nullptr;    // 2 x F per-feature candidates
  SplitOut* split_host = nullptr;  // pinned
  double* scalar_host = nullptr;   // pinned
  void* scan_tmp = nullptr;
  size_t scan_tmp_bytes = 0;
  int32_t *leaf_begin_dev = nullptr, *leaf_cnt_dev = nullptr, *leaf_buf_dev = nullptr;
  std::vector<int> leaf_buf;  // per leaf of the last tree: which row-index buffer holds its rows
  double* leaf_val_dev = nullptr;
  std::vector<int> leaf_begin, leaf_cnt;
  int last_num_leaves = 0;
  int64_t launches = 0;
  std::vector<uint8_t> bins_rm_host;
  // data-parallel mode (rows sharded over ranks, SURVEY §8e): histograms of the smaller child and the root gradient sum are
  // all-reduced on this stream; split decisions are then identical on every rank, the partition stays local
  gpbdev_allreduce_fn allreduce = nullptr;
  void* allreduce_ctx = nullptr;
  int64_t n_global = 0;
};

namespace {
__global__ void zero_outside_kernel(double* __restrict__ x, int64_t n, int64_t b, int64_t e) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (i < b || i >= e) x[i] = 0.;
}
}  // namespace

extern "C" {

const char* gpbdev_tree_last_error(void) { return g_tree_err.c_str(); }

int gpbdev_tree_set_allreduce(gpbdev_tree_t h, gpbdev_allreduce_fn fn, void* ctx, int64_t n_global) {
  if (!h) return tfail("gpbdev_tree_set_allreduce: null argument");
  if (fn != nullptr && n_global < h->n) return tfail("gpbdev_tree_set_allreduce: n_global is smaller than the local row count");
  h->allreduce = fn; h->allreduce_ctx = ctx; h->n_global = fn ? n_global : 0;
  return 0;
}

// every rank holds rows [b, e) of a replicated n-vector up to date: make the whole vector current everywhere
int gpbdev_vec_allgather_rows(gpbdev_tree_t h, double* vec_dev, int64_t n, int64_t b, int64_t e) {
  if (!h || !vec_dev) return tfail("gpbdev_vec_allgather_rows: null argument");
  if (!h->allreduce) return tfail("gpbdev_vec_allgather_rows: no collective installed (gpbdev_tree_set_allreduce)");
  TCUDA(cudaSetDevice(h->device));
  zero_outside_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(vec_dev, n, b, e);
  TCUDA(cudaGetLastError());
  if (h->allreduce(h->allreduce_ctx, vec_dev, n, (void*)h->stream)) return tfail("gpbdev_vec_allgather_rows: device all-reduce failed");
  TCUDA(cudaStreamSynchronize(h->stream));
  h->launches += 1;
  return 0;
}

// bins_feature_major != nullptr: host bins, transposed and uploaded (owned); else bins_dev: row-major n x Fpad_in already in HBM (adopted)
static int tree_create_common(gpbdev_tree_t* out, int device, int64_t n, int F, const uint8_t* bins_feature_major, const uint8_t* bins_dev,
                              int Fpad_in, const int32_t* num_bin, const gpbdev_tree_config* cfg) {
  if (!out || (!bins_feature_major && !bins_dev) || !num_bin || !cfg) return tfail("gpbdev_tree_create: null argument");
  if (n <= 0 || F <= 0) return tfail("gpbdev_tree_create: need n > 0 and F > 0");
  if (cfg->num_leaves < 2) return tfail("gpbdev_tree_create: num_leaves must be >= 2");
  if (cfg->min_data_in_leaf < 0) return tfail("gpbdev_tree_create: min_data_in_leaf must be >= 0");
  for (int f = 0; f < F; ++f)
    if (num_bin[f] < 1 || num_bin[f] > kBins) return tfail("gpbdev_tree_create: num_bin must be in [1, 256]");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) {
    cudaGetLastError();
    return tfail("gpbdev_tree_create: no CUDA device " + std::to_string(device) + " — the CUDA tree learner has no CPU fallback");
  }
  TCUDA(cudaSetDevice(device));
  gpbdev_tree* h = new gpbdev_tree();
  h->device = device; h->n = n; h->F = F; h->Fpad = (F + 31) / 32 * 32; h->L = cfg->num_leaves; h->cfg = *cfg;
  // With both limits at 0 a threshold past a leaf's last occupied bin is admissible and gains (sum g)^2 (1/(H + eps) - 1/(H + 2 eps))
  // > 0 when the hessian sum H is small: a split with an empty child, which the partition cannot produce. The reference raises
  // min_data_in_leaf to 1 in that case (Config::CheckParamConflict, io/config.cpp:400-405).
  if (h->cfg.min_data_in_leaf <= 0 && h->cfg.min_sum_hessian_in_leaf <= kEps) h->cfg.min_data_in_leaf = 1;
  cudaDeviceProp prop;
  TCUDA(cudaGetDeviceProperties(&prop, device));
  h->num_sms = prop.multiProcessorCount;
  TCUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  // feature-major (the reference's dense-bin layout) -> row-major padded (one 32-byte sector per row and feature group)
  if (bins_feature_major) {
    h->bins_rm_host.assign((size_t)n * h->Fpad, 0);
    for (int f = 0; f < F; ++f)
      for (int64_t i = 0; i < n; ++i) h->bins_rm_host[(size_t)i * h->Fpad + f] = bins_feature_major[(size_t)f * n + i];
    TCUDA(cudaMalloc(&h->bins_owned, (size_t)n * h->Fpad));
    TCUDA(cudaMemcpy(h->bins_owned, h->bins_rm_host.data(), (size_t)n * h->Fpad, cudaMemcpyHostToDevice));
    h->bins_rm_host.clear(); h->bins_rm_host.shrink_to_fit();
    h->bins = h->bins_owned;
  } else {
    if (Fpad_in != h->Fpad) { delete h; return tfail("gpbdev_tree_create_on_device_bins: Fpad must be F rounded up to a multiple of 32"); }
    h->bins = bins_dev;  // read in place; the Dataset owns it
  }
  TCUDA(cudaMalloc(&h->num_bin, sizeof(int32_t) * F));
  TCUDA(cudaMemcpy(h->num_bin, num_bin, sizeof(int32_t) * F, cudaMemcpyHostToDevice));
  TCUDA(cudaMalloc(&h->idx, sizeof(int32_t) * n));
  TCUDA(cudaMalloc(&h->idx_tmp, sizeof(int32_t) * n));
  TCUDA(cudaMalloc(&h->flag, sizeof(int32_t) * n));
  TCUDA(cudaMalloc(&h->pos, sizeof(int32_t) * n));
  TCUDA(cudaMalloc(&h->grad, sizeof(double) * n));
  const size_t slot = (size_t)F * kBins * 2;
  TCUDA(cudaMalloc(&h->hist, sizeof(double) * slot * (h->L + 1)));
  TCUDA(cudaMalloc(&h->splittable, (size_t)h->L * F));
  TCUDA(cudaMalloc(&h->parent_flags, (size_t)F));
  h->max_chunks = h->num_sms * 2;
  TCUDA(cudaMalloc(&h->part_g, sizeof(double) * (size_t)h->max_chunks * h->Fpad * kBins));
  TCUDA(cudaMalloc(&h->part_c, sizeof(uint32_t) * (size_t)h->max_chunks * h->Fpad * kBins));
  TCUDA(cudaMalloc(&h->sum_part, sizeof(double) * 1024));
  TCUDA(cudaMalloc(&h->split_dev, sizeof(SplitOut) * 2));
  TCUDA(cudaMalloc(&h->cand_dev, sizeof(SplitOut) * 2 * F));
  TCUDA(cudaMallocHost(&h->split_host, sizeof(SplitOut) * 2));
  TCUDA(cudaMallocHost(&h->scalar_host, sizeof(double) * 4));
  TCUDA(cub::DeviceScan::ExclusiveSum(nullptr, h->scan_tmp_bytes, h->flag, h->pos, (int)n, h->stream));
  TCUDA(cudaMalloc(&h->scan_tmp, h->scan_tmp_bytes));
  TCUDA(cudaMalloc(&h->leaf_begin_dev, sizeof(int32_t) * h->L));
  TCUDA(cudaMalloc(&h->leaf_cnt_dev, sizeof(int32_t) * h->L));
  TCUDA(cudaMalloc(&h->leaf_buf_dev, sizeof(int32_t) * h->L));
  h->leaf_buf.assign(h->L, 0);
  TCUDA(cudaMalloc(&h->leaf_val_dev, sizeof(double) * h->L));
  TCUDA(cudaFuncSetAttribute(hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 257 * 12));
  TCUDA(cudaFuncSetAttribute(hist2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist2_smem(hist2_warps(F))));
  TCUDA(cudaFuncSetAttribute(hist3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist3_smem(hist2_warps(F))));
  TCUDA(cudaFuncSetAttribute(hist3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist3_smem(hist2_warps(F))));
  h->max_seg = h->num_sms * 4;
  TCUDA(cudaMalloc(&h->flag8, (size_t)n));
  TCUDA(cudaMalloc(&h->seg_left, sizeof(int32_t) * h->max_seg));
  TCUDA(cudaMalloc(&h->nleft_dev, sizeof(int32_t)));
  TCUDA(cudaMallocHost(&h->nleft_host, sizeof(int32_t)));
  TCUDA(cudaMalloc(&h->state_dev, sizeof(TreeDevState)));
  TCUDA(cudaMallocHost(&h->state_host, sizeof(TreeDevState)));
  if (const char* e = std::getenv("GPB200_TREE_LOOP")) h->device_loop = std::string(e) == "device" ? 1 : (std::string(e) == "host" ? 0 : 2);
  if (const char* e = std::getenv("GPB200_FUSED_SCAN")) h->fused_scan = std::atoi(e) == 0 ? 0 : (std::atoi(e) == 1 ? 1 : 2);
  if (const char* e = std::getenv("GPB200_FUSED_ADVANCE")) h->fused_advance = std::atoi(e) == 0 ? 0 : 1;
  if (const char* e = std::getenv("GPB200_SHARDED_LOOP")) { h->sharded_host_loop = std::string(e) == "host" ? 1 : 0; h->sharded_graph = std::string(e) == "graph" ? 1 : 0; }
  if (const char* e = std::getenv("GPB200_PARTITION")) h->partition_version = std::atoi(e) == 1 ? 1 : 2;
  if (const char* e = std::getenv("GPB200_HIST_KERNEL")) h->hist_kernel_version = std::atoi(e) >= 1 && std::atoi(e) <= 4 ? std::atoi(e) : 3;
  *out = h;
  return 0;
}

int gpbdev_tree_create(gpbdev_tree_t* out, int device, int64_t n, int F, const uint8_t* bins_feature_major, const int32_t* num_bin,
                       const gpbdev_tree_config* cfg) {
  if (!bins_feature_major) return tfail("gpbdev_tree_create: null argument");
  return tree_create_common(out, device, n, F, bins_feature_major, nullptr, 0, num_bin, cfg);
}

int gpbdev_tree_create_on_device_bins(gpbdev_tree_t* out, int device, int64_t n, int F, int Fpad, const uint8_t* bins_dev,
                                      const int32_t* num_bin, const gpbdev_tree_config* cfg) {
  if (!bins_dev) return tfail("gpbdev_tree_create_on_device_bins: null argument");
  return tree_create_common(out, device, n, F, nullptr, bins_dev, Fpad, num_bin, cfg);
}

int gpbdev_tree_free(gpbdev_tree_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaFree(h->bins_owned); cudaFree(h->leaf_of_row); cudaFree(h->stage); cudaFree(h->num_bin); cudaFree(h->idx); cudaFree(h->idx_tmp); cudaFree(h->flag); cudaFree(h->pos);
  cudaFree(h->grad); cudaFree(h->hist); cudaFree(h->splittable); cudaFree(h->parent_flags); cudaFree(h->part_g); cudaFree(h->part_c); cudaFree(h->sum_part);
  cudaFree(h->split_dev); cudaFree(h->cand_dev); cudaFree(h->scan_tmp); cudaFree(h->leaf_begin_dev); cudaFree(h->leaf_cnt_dev); cudaFree(h->leaf_buf_dev); cudaFree(h->leaf_val_dev);
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  cudaFree(h->state_dev); cudaFreeHost(h->state_host);
  cudaFree(h->flag8); cudaFree(h->seg_left); cudaFree(h->nleft_dev); cudaFreeHost(h->nleft_host);
  cudaFreeHost(h->split_host); cudaFreeHost(h->scalar_host);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int64_t gpbdev_tree_launch_count(gpbdev_tree_t h) { return h ? h->launches : 0; }
void* gpbdev_tree_stream(gpbdev_tree_t h) { return h ? (void*)h->stream : nullptr; }

// device-resident leaf loop: every kernel of every split is enqueued up front; the planner / selector kernels steer them
static int tree_train_device_loop(gpbdev_tree_t h, const double* grad, double hess_const, int* num_leaves_out, int* split_feature,
                                  int* threshold_bin, int* left_child, int* right_child, float* split_gain, double* leaf_value,
                                  int* leaf_count) {
  const int64_t n = h->n;
  const int F = h->F, Fpad = h->Fpad, L = h->L;
  const gpbdev_tree_config& cfg = h->cfg;
  const size_t slot_stride = (size_t)F * kBins * 2;
  TreeDevState* st = h->state_dev;
  const DevJob* job = &st->job;
  // GPB200_TREE_LOOP=graph: the whole tree (root sums included) is one CUDA graph, captured once per (gradient buffer,
  // hessian) and replayed every boosting iteration — one graph launch instead of ~8 launches per split
  // Data-parallel learners enqueue the same sequence eagerly (kernels and NCCL all-reduces, no host round trip per split); replaying
  // NCCL collectives from a captured graph is opt-in (GPB200_SHARDED_LOOP=graph) — the first two-GPU run of that combination did
  // not complete.
  const bool use_graph = h->device_loop == 2 && (h->allreduce == nullptr || h->sharded_graph);
  if (use_graph && h->graph_exec && (h->graph_grad != grad || h->graph_hess != hess_const)) {
    cudaGraphExecDestroy(h->graph_exec);
    h->graph_exec = nullptr;
  }
  const bool replay = use_graph && h->graph_exec != nullptr;
  // data-parallel learner (row shards over ranks): the same enqueued sequence with three additions — the root gradient sum and the
  // smaller child's merged histogram are summed over the ranks ON THIS STREAM (NCCL kernels, captured into the graph like everything
  // else; DataParallelTreeLearner, data_parallel_tree_learner.cpp:155-175, :244), and the children's local row ranges are set after
  // the local partition. Every rank replays the same number of collectives whatever the tree does (finished trees skip the work,
  // not the exchange). The whole 2 F x 256 block is all-reduced and scanned on every rank: at F = 50..100 it is a 0.2..0.4 MB
  // message, latency-bound on NVSwitch — a reduce-scatter by feature block (the reference's choice for Ethernet clusters) would add
  // a second latency-bound collective per split for the best-split exchange and scan no faster (one CTA per feature either way).
  const bool sharded = h->allreduce != nullptr;
  const int n_glob = sharded ? (int)h->n_global : (int)n;
  if (sharded && !h->stage) {
    TCUDA(cudaMalloc(&h->stage, sizeof(double) * slot_stride));
    TCUDA(cudaMemsetAsync(h->stage, 0, sizeof(double) * slot_stride, h->stream));
    // one eager exchange of each message size before anything is captured: the communicator sets up its channels / buffers for a
    // (size, algorithm) at the first call, which must not happen inside a stream capture
    if (h->allreduce(h->allreduce_ctx, h->stage, (int64_t)slot_stride, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
    if (h->allreduce(h->allreduce_ctx, h->stage, 1, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
    TCUDA(cudaStreamSynchronize(h->stream));
  }
  if (use_graph && !replay) TCUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
  bool coll_failed = false;
  if (!replay) {
  if (use_graph) {  // the eager path ran these before the call
    iota_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(h->idx, n);
    const int nb1 = (int)std::min<int64_t>(1024, (n + 4095) / 4096);
    sum_stage1_kernel<<<nb1, 256, 0, h->stream>>>(grad, n, h->sum_part);
    sum_stage2_kernel<<<1, 256, 0, h->stream>>>(h->sum_part, nb1, h->sum_part + 1023);
    if (sharded && h->allreduce(h->allreduce_ctx, h->sum_part + 1023, 1, (void*)h->stream)) coll_failed = true;
  }
  tree_init_kernel<<<1, 32, 0, h->stream>>>(st, h->sum_part + 1023, (int)n, n_glob, hess_const, L);
  const int nw = hist2_warps(F);
  const dim3 hgrid(h->num_sms, (Fpad + 63) / 64);
  const bool fused_advance = !sharded && h->fused_advance;
  if (fused_advance) tree_plan_kernel<<<1, 32, 0, h->stream>>>(st, cfg.max_depth, cfg.min_data_in_leaf, h->num_sms);  // first split; later ones: tree_advance_kernel
  for (int split = 0; split < L - 1 && !coll_failed; ++split) {
    if (!fused_advance) tree_plan_kernel<<<1, 32, 0, h->stream>>>(st, cfg.max_depth, cfg.min_data_in_leaf, h->num_sms);
    if (h->hist_kernel_version == 4)
      hist3_kernel<true><<<hgrid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, h->idx, 0, 0, 0, grad, h->part_g, h->part_c, job, h->idx_tmp);
    else if (h->hist_kernel_version == 3)
      hist3_kernel<false><<<hgrid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, h->idx, 0, 0, 0, grad, h->part_g, h->part_c, job, h->idx_tmp);
    else
      hist2_kernel<<<hgrid, nw * 32, hist2_smem(nw), h->stream>>>(h->bins, Fpad, F, h->idx, 0, 0, 0, grad, h->part_g, h->part_c, job, h->idx_tmp);
    LeafArgs dummy;
    dummy.leaf = -1; dummy.hist_slot = 0; dummy.inherit = 0; dummy.num_data = 0; dummy.sum_gradients = 0.; dummy.sum_hessians = 0.;
    if (sharded) {
      hist_reduce_kernel<<<F * (kBins / 32), kReduceSlices * 32, 0, h->stream>>>(h->part_g, h->part_c, 0, Fpad, F, hess_const, h->stage, nullptr, job);
      if (h->allreduce(h->allreduce_ctx, h->stage, (int64_t)slot_stride, (void*)h->stream)) { coll_failed = true; break; }
    }
    if (h->fused_scan == 2 || sharded)
      reduce_scan2_kernel<<<F, kFusedSlices * kBins, 0, h->stream>>>(h->part_g, h->part_c, 0, Fpad, F, hess_const, h->hist, (int64_t)slot_stride,
                                                                    h->num_bin, dummy, dummy, 0, cfg.min_data_in_leaf,
                                                                    cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                                                    h->splittable, h->cand_dev, job, sharded ? h->stage : nullptr);
    else
    reduce_scan_kernel<<<F, kFusedSlices * kBins, 0, h->stream>>>(h->part_g, h->part_c, 0, Fpad, F, hess_const, h->hist, (int64_t)slot_stride,
                                                                 h->num_bin, dummy, dummy, 0, cfg.min_data_in_leaf,
                                                                 cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                                                 h->splittable, h->cand_dev, job);
    if (fused_advance) {
      tree_advance_kernel<<<1, 128, 0, h->stream>>>(st, h->cand_dev, F, cfg.min_gain_to_split, h->max_seg, cfg.max_depth, cfg.min_data_in_leaf, h->num_sms,
                                                    split + 1 < L - 1 ? 1 : 0);
    } else {
      split_argmax_kernel<<<2, 64, 0, h->stream>>>(h->cand_dev, F, h->split_dev);
      tree_select_kernel<<<1, 32, 0, h->stream>>>(st, h->split_dev, cfg.min_gain_to_split, h->max_seg, sharded ? 1 : 0);
    }
    part_count_kernel<<<h->max_seg, kPartThreads, 0, h->stream>>>(h->bins, Fpad, 0, 0, h->idx, 0, 0, 0, h->flag8, h->seg_left, job, h->idx_tmp);
    part_scatter_kernel<<<h->max_seg, kPartThreads, 0, h->stream>>>(h->idx, 0, 0, 0, h->flag8, h->seg_left, 0, nullptr, nullptr, job, h->idx_tmp);
    if (sharded) tree_local_ranges_kernel<<<1, 32, 0, h->stream>>>(st, h->seg_left);
  }
  TCUDA(cudaMemcpyAsync(h->state_host, st, sizeof(TreeDevState), cudaMemcpyDeviceToHost, h->stream));
  }  // !replay
  if (use_graph && !replay) {
    cudaGraph_t g = nullptr;
    TCUDA(cudaStreamEndCapture(h->stream, &g));
    if (coll_failed) { if (g) cudaGraphDestroy(g); return tfail("gpbdev_tree_train: device all-reduce failed"); }
    const cudaError_t ie = cudaGraphInstantiate(&h->graph_exec, g, 0);
    cudaGraphDestroy(g);
    if (ie != cudaSuccess) { h->graph_exec = nullptr; return tfail(std::string("gpbdev_tree_train: cudaGraphInstantiate: ") + cudaGetErrorString(ie)); }
    h->graph_grad = grad; h->graph_hess = hess_const;
  }
  if (!use_graph && coll_failed) return tfail("gpbdev_tree_train: device all-reduce failed");
  if (!replay) TCUDA(cudaGetLastError());
  if (use_graph) TCUDA(cudaGraphLaunch(h->graph_exec, h->stream));
  const bool one_advance = !sharded && h->fused_advance;
  h->launches += (sharded ? 10 : (one_advance ? 5 : 7)) * (L - 1) + (use_graph ? (sharded ? 4 : 3) : 0) + (one_advance ? 1 : 0);
  TCUDA(cudaStreamSynchronize(h->stream));
  const TreeDevState& r = *h->state_host;
  if (r.job.error) return tfail("gpbdev_tree_train: inconsistent split counts");
  const int num_leaves = r.num_leaves;
  for (int i = 0; i < num_leaves - 1; ++i) {
    split_feature[i] = r.split_feature[i]; threshold_bin[i] = r.threshold_bin[i]; left_child[i] = r.left_child[i];
    right_child[i] = r.right_child[i]; split_gain[i] = r.split_gain[i];
  }
  for (int i = 0; i < num_leaves; ++i) { leaf_value[i] = r.leaf_value[i]; leaf_count[i] = r.leaf_count[i]; }
  h->leaf_begin.assign(r.leaf_begin, r.leaf_begin + L);
  h->leaf_cnt.assign(r.leaf_cnt, r.leaf_cnt + L);
  h->leaf_buf.assign(r.leaf_buf, r.leaf_buf + L);
  h->last_num_leaves = num_leaves;
  *num_leaves_out = num_leaves;
  return 0;
}

int gpbdev_tree_train(gpbdev_tree_t h, const double* grad_in, int grad_on_device, double hess_const, int* num_leaves_out,
                      int* split_feature, int* threshold_bin, int* left_child, int* right_child, float* split_gain,
                      double* leaf_value, int* leaf_count) {
  if (!h || !grad_in || !num_leaves_out) return tfail("gpbdev_tree_train: null argument");
  TCUDA(cudaSetDevice(h->device));
  const int64_t n = h->n;
  const int F = h->F, Fpad = h->Fpad, L = h->L;
  const gpbdev_tree_config& cfg = h->cfg;
  const double* grad = grad_in;
  if (!grad_on_device) {
    TCUDA(cudaMemcpyAsync(h->grad, grad_in, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
    grad = h->grad;
  }
  const size_t slot_stride = (size_t)F * kBins * 2;
  // ---- BeforeTrain: partition = all rows in leaf 0, root sums (leaf_splits.hpp:70-83)
  const bool sharded = h->allreduce != nullptr;
  const int64_t n_glob = sharded ? h->n_global : n;
  const bool dev_loop_sharded = !sharded || !h->sharded_host_loop;
  if (h->device_loop == 2 && (!sharded || (dev_loop_sharded && h->sharded_graph)) && L <= kMaxLeavesDev && grad_on_device)  // everything, root sums included, is in the graph
    return tree_train_device_loop(h, grad, hess_const, num_leaves_out, split_feature, threshold_bin, left_child, right_child, split_gain,
                                  leaf_value, leaf_count);
  iota_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(h->idx, n);
  const int nb1 = (int)std::min<int64_t>(1024, (n + 4095) / 4096);
  sum_stage1_kernel<<<nb1, 256, 0, h->stream>>>(grad, n, h->sum_part);
  sum_stage2_kernel<<<1, 256, 0, h->stream>>>(h->sum_part, nb1, h->sum_part + 1023);
  if (sharded && h->allreduce(h->allreduce_ctx, h->sum_part + 1023, 1, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
  if (h->device_loop && dev_loop_sharded && L <= kMaxLeavesDev) {
    h->launches += 3;
    const int keep = h->device_loop;
    h->device_loop = 1;  // eager enqueue (host gradients are staged per call: no graph)
    const int rc = tree_train_device_loop(h, grad, hess_const, num_leaves_out, split_feature, threshold_bin, left_child, right_child, split_gain,
                                          leaf_value, leaf_count);
    h->device_loop = keep;
    return rc;
  }
  TCUDA(cudaMemcpyAsync(h->scalar_host, h->sum_part + 1023, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  h->launches += 3;
  // leaf_cnt: rows of the leaf on THIS rank (partition, histogram ranges); leaf_cnt_g: rows over all ranks (every decision)
  std::vector<int> leaf_begin(L, 0), leaf_cnt(L, 0), leaf_cnt_g(L, 0), leaf_depth(L, 0), leaf_parent(L, -1), slot_of(L, -1);
  std::vector<double> leaf_sg(L, 0.), leaf_sh(L, 0.);
  std::vector<SplitOut> best(L);
  for (auto& b : best) { b.gain = -INFINITY; b.feature = -1; }
  std::vector<int> free_slots;
  for (int s = L; s >= 0; --s) free_slots.push_back(s);
  leaf_cnt[0] = (int)n;
  leaf_cnt_g[0] = (int)n_glob;
  leaf_sg[0] = h->scalar_host[0];
  leaf_sh[0] = hess_const * (double)n_glob;
  leaf_value[0] = 0.; leaf_count[0] = (int)n_glob;
  int num_leaves = 1, left_leaf = 0, right_leaf = -1;

  // nchunks_out != nullptr: only the chunk partials are produced (the merge is fused into the split scan, reduce_scan_kernel)
  auto build_hist = [&](int leaf, int slot, int parent_slot_sub, int* nchunks_out) -> int {
    const int64_t cnt = leaf_cnt[leaf];
    double* dst = h->hist + (size_t)slot * slot_stride;
    double* par = parent_slot_sub >= 0 ? h->hist + (size_t)parent_slot_sub * slot_stride : nullptr;
    if (cnt > 0) {
      int64_t rpc = std::max<int64_t>(256, (cnt + h->max_chunks - 1) / h->max_chunks);
      int nchunks = (int)((cnt + rpc - 1) / rpc);
      dim3 grid(nchunks, Fpad / 32);
      if (h->hist_kernel_version >= 2) {
        // one CTA per SM and chunk; grid.y = groups of 64 features
        rpc = std::max<int64_t>(128, ((cnt + h->num_sms - 1) / h->num_sms + 7) / 8 * 8);  // whole 8-row steps per chunk
        nchunks = (int)((cnt + rpc - 1) / rpc);
        const int nw = hist2_warps(F);
        if (h->hist_kernel_version == 4)
          hist3_kernel<true><<<dim3(nchunks, (Fpad + 63) / 64), nw * 32, hist3_smem(nw), h->stream>>>(
              h->bins, Fpad, F, (num_leaves == 1) ? nullptr : h->idx, leaf_begin[leaf], cnt, rpc, grad, h->part_g, h->part_c, nullptr, nullptr);
        else if (h->hist_kernel_version == 3)
          hist3_kernel<false><<<dim3(nchunks, (Fpad + 63) / 64), nw * 32, hist3_smem(nw), h->stream>>>(
              h->bins, Fpad, F, (num_leaves == 1) ? nullptr : h->idx, leaf_begin[leaf], cnt, rpc, grad, h->part_g, h->part_c, nullptr, nullptr);
        else
        hist2_kernel<<<dim3(nchunks, (Fpad + 63) / 64), nw * 32, hist2_smem(nw), h->stream>>>(
            h->bins, Fpad, F, (num_leaves == 1) ? nullptr : h->idx, leaf_begin[leaf], cnt, rpc, grad, h->part_g, h->part_c, nullptr, nullptr);
      }
      else
        hist_kernel<<<grid, 32, 32 * 257 * 12, h->stream>>>(h->bins, Fpad, (num_leaves == 1) ? nullptr : h->idx, leaf_begin[leaf], cnt,
                                                           rpc, grad, h->part_g, h->part_c);
      TCUDA(cudaGetLastError());
      if (nchunks_out) { *nchunks_out = nchunks; h->launches += 1; return 0; }
      // single GPU: larger = parent - smaller is fused into the merge of the chunk partials
      hist_reduce_kernel<<<F * (kBins / 32), kReduceSlices * 32, 0, h->stream>>>(h->part_g, h->part_c, nchunks, Fpad, F, hess_const, dst,
                                                                        sharded ? nullptr : par, nullptr);
      TCUDA(cudaGetLastError());
      h->launches += 2;
    } else {
      TCUDA(cudaMemsetAsync(dst, 0, sizeof(double) * slot_stride, h->stream));  // this rank holds no row of the leaf
    }
    if (sharded) {
      // data-parallel learner (the reference's DataParallelTreeLearner reduce-scatters the smaller child's histograms,
      // src/LightGBM/treelearner/data_parallel_tree_learner.cpp:155-175): sum over ranks on this stream, then the subtraction
      if (h->allreduce(h->allreduce_ctx, dst, (int64_t)slot_stride, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
      if (par) {
        hist_subtract_kernel<<<((int)slot_stride + 255) / 256, 256, 0, h->stream>>>(par, dst, (int)slot_stride);
        TCUDA(cudaGetLastError());
        h->launches += 1;
      }
    }
    return 0;
  };

  for (int split = 0; split < L - 1; ++split) {
    // ---- BeforeFindBestSplit (serial_tree_learner.cpp:283-322)
    bool do_find = true;
    if (cfg.max_depth > 0 && leaf_depth[left_leaf] >= cfg.max_depth) do_find = false;
    if (do_find) {
      const int nl = leaf_cnt_g[left_leaf], nr = right_leaf >= 0 ? leaf_cnt_g[right_leaf] : 0;
      if (nr < cfg.min_data_in_leaf * 2 && nl < cfg.min_data_in_leaf * 2) do_find = false;
    }
    if (!do_find) {
      best[left_leaf].gain = -INFINITY;
      if (right_leaf >= 0) best[right_leaf].gain = -INFINITY;
    } else {
      int smaller, larger = -1, parent_slot = -1;
      if (right_leaf < 0) smaller = left_leaf;
      else if (leaf_cnt_g[left_leaf] < leaf_cnt_g[right_leaf]) { smaller = left_leaf; larger = right_leaf; }
      else { smaller = right_leaf; larger = left_leaf; }
      if (right_leaf >= 0) parent_slot = slot_of[left_leaf];  // the parent's histograms sit under the left (= parent) id
      const int new_slot = free_slots.back();
      free_slots.pop_back();
      // larger = parent - smaller, in place (fused into the merge of the chunk partials): the parent's slot becomes the larger leaf's
      const bool fused = h->fused_scan && !sharded && leaf_cnt[smaller] > 0;
      int nchunks_f = 0;
      if (build_hist(smaller, new_slot, larger >= 0 ? parent_slot : -1, fused ? &nchunks_f : nullptr)) return -1;
      if (larger >= 0) slot_of[larger] = parent_slot;
      slot_of[smaller] = new_slot;
      // both children inherit the parent's flags (the parent's id is the left child's id): snapshot them first
      if (right_leaf >= 0 && !fused)
        TCUDA(cudaMemcpyAsync(h->parent_flags, h->splittable + (size_t)left_leaf * F, F, cudaMemcpyDeviceToDevice, h->stream));
      LeafArgs a0, a1;
      a0.leaf = smaller; a0.hist_slot = new_slot; a0.inherit = right_leaf >= 0 ? 1 : 0; a0.num_data = leaf_cnt_g[smaller];
      a0.sum_gradients = leaf_sg[smaller]; a0.sum_hessians = leaf_sh[smaller];
      a1.leaf = larger; a1.hist_slot = larger >= 0 ? parent_slot : 0; a1.inherit = 1; a1.num_data = larger >= 0 ? leaf_cnt_g[larger] : 0;
      a1.sum_gradients = larger >= 0 ? leaf_sg[larger] : 0.; a1.sum_hessians = larger >= 0 ? leaf_sh[larger] : 0.;
      if (fused && h->fused_scan == 2)
        reduce_scan2_kernel<<<F, kFusedSlices * kBins, 0, h->stream>>>(h->part_g, h->part_c, nchunks_f, Fpad, F, hess_const, h->hist,
                                                                      (int64_t)slot_stride, h->num_bin, a0, a1, left_leaf, cfg.min_data_in_leaf,
                                                                      cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                                                      h->splittable, h->cand_dev, nullptr, nullptr);
      else if (fused)
        reduce_scan_kernel<<<F, kFusedSlices * kBins, 0, h->stream>>>(h->part_g, h->part_c, nchunks_f, Fpad, F, hess_const, h->hist,
                                                                     (int64_t)slot_stride, h->num_bin, a0, a1, left_leaf, cfg.min_data_in_leaf,
                                                                     cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                                                     h->splittable, h->cand_dev, nullptr);
      else
        split_scan_kernel<<<dim3(F, 2), 32, 0, h->stream>>>(h->hist, (int64_t)slot_stride, h->num_bin, F, a0, a1, cfg.min_data_in_leaf,
                                                            cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                                            h->splittable, h->parent_flags, h->cand_dev);
      TCUDA(cudaGetLastError());
      if (larger < 0) TCUDA(cudaMemsetAsync(h->split_dev + 1, 0, sizeof(SplitOut), h->stream));
      split_argmax_kernel<<<larger >= 0 ? 2 : 1, 64, 0, h->stream>>>(h->cand_dev, F, h->split_dev);
      TCUDA(cudaGetLastError());
      h->launches += 2;
      TCUDA(cudaMemcpyAsync(h->split_host, h->split_dev, sizeof(SplitOut) * 2, cudaMemcpyDeviceToHost, h->stream));
      TCUDA(cudaStreamSynchronize(h->stream));
      best[smaller] = h->split_host[0];
      if (larger >= 0) best[larger] = h->split_host[1];
    }
    // ---- leaf with the best split (ArrayArgs::ArgMax with SplitInfo::operator>)
    int best_leaf = 0;
    for (int l = 1; l < num_leaves; ++l) {
      int fa = best[l].feature == -1 ? 2147483647 : best[l].feature, fb = best[best_leaf].feature == -1 ? 2147483647 : best[best_leaf].feature;
      const bool better = best[l].gain != best[best_leaf].gain ? best[l].gain > best[best_leaf].gain : fa < fb;
      if (better) best_leaf = l;
    }
    const SplitOut bs = best[best_leaf];
    if (!(bs.gain > 0.0)) break;
    // ---- DataPartition::Split (stable) on this rank's rows of the leaf
    const int64_t b = leaf_begin[best_leaf], c = leaf_cnt[best_leaf];
    // With a constant hessian the histogram's hessian entries are exact multiples of it, so the split scan's
    // RoundInt(hess * cnt_factor) counts ARE the partition's counts (the reference overwrites them with the
    // partition's, serial_tree_learner.cpp:589-593 — same numbers). On one GPU no device round trip is needed for them;
    // with row shards the LOCAL left count comes back from the scan.
    const int nleft_g = bs.left_count, nright_g = leaf_cnt_g[best_leaf] - nleft_g;
    if (nleft_g <= 0 || nright_g <= 0) return tfail("gpbdev_tree_train: inconsistent split counts");
    int nleft = nleft_g;
    if (c > 0 && h->partition_version == 2 && !sharded) {  // the host loop of a data-parallel learner keeps the CUB path
      const int64_t seg = std::max<int64_t>(4 * kPartThreads, ((c + h->max_seg - 1) / h->max_seg + kPartThreads - 1) / kPartThreads * kPartThreads);
      const int nseg = (int)((c + seg - 1) / seg);
      part_count_kernel<<<nseg, kPartThreads, 0, h->stream>>>(h->bins, Fpad, bs.feature, bs.threshold, h->idx, b, c, seg, h->flag8, h->seg_left, nullptr, nullptr);
      part_scatter_kernel<<<nseg, kPartThreads, 0, h->stream>>>(h->idx, b, c, seg, h->flag8, h->seg_left, nseg, h->idx_tmp,
                                                                sharded ? h->nleft_dev : nullptr, nullptr, nullptr);
      TCUDA(cudaGetLastError());
      TCUDA(cudaMemcpyAsync(h->idx + b, h->idx_tmp, sizeof(int32_t) * c, cudaMemcpyDeviceToDevice, h->stream));
      if (sharded) {  // this rank's share of the left child
        TCUDA(cudaMemcpyAsync(h->nleft_host, h->nleft_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        TCUDA(cudaStreamSynchronize(h->stream));
        nleft = *h->nleft_host;
      }
      h->launches += 2;
    } else if (c > 0) {
      const int gridp = (int)std::min<int64_t>((c + 255) / 256, (int64_t)h->num_sms * 8);
      mark_kernel<<<gridp, 256, 0, h->stream>>>(h->bins, Fpad, bs.feature, bs.threshold, h->idx, b, c, h->flag);
      TCUDA(cub::DeviceScan::ExclusiveSum(h->scan_tmp, h->scan_tmp_bytes, h->flag, h->pos, (int)c, h->stream));
      if (sharded) {
        int32_t last[2];
        TCUDA(cudaMemcpyAsync(&last[0], h->pos + (c - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        TCUDA(cudaMemcpyAsync(&last[1], h->flag + (c - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        TCUDA(cudaStreamSynchronize(h->stream));
        nleft = last[0] + last[1];
      }
      scatter_kernel<<<gridp, 256, 0, h->stream>>>(h->idx, b, c, h->flag, h->pos, nleft, h->idx_tmp);
      TCUDA(cudaMemcpyAsync(h->idx + b, h->idx_tmp, sizeof(int32_t) * c, cudaMemcpyDeviceToDevice, h->stream));
      h->launches += 4;
    } else {
      nleft = 0;
    }
    const int nright = (int)c - nleft;
    const int new_leaf = num_leaves;
    leaf_cnt[best_leaf] = nleft; leaf_begin[new_leaf] = (int)(b + nleft); leaf_cnt[new_leaf] = nright;
    leaf_cnt_g[best_leaf] = nleft_g; leaf_cnt_g[new_leaf] = nright_g;
    // ---- Tree::Split (tree.h:533-575)
    const int node = num_leaves - 1;
    const int parent = leaf_parent[best_leaf];
    if (parent >= 0) { if (left_child[parent] == ~best_leaf) left_child[parent] = node; else right_child[parent] = node; }
    split_feature[node] = bs.feature; threshold_bin[node] = bs.threshold;
    split_gain[node] = (float)(bs.gain + cfg.min_gain_to_split);
    left_child[node] = ~best_leaf; right_child[node] = ~new_leaf;
    leaf_parent[best_leaf] = node; leaf_parent[new_leaf] = node;
    leaf_value[best_leaf] = std::isnan(bs.left_output) ? 0. : bs.left_output; leaf_count[best_leaf] = nleft_g;
    leaf_value[new_leaf] = std::isnan(bs.right_output) ? 0. : bs.right_output; leaf_count[new_leaf] = nright_g;
    leaf_depth[new_leaf] = leaf_depth[best_leaf] + 1; leaf_depth[best_leaf]++;
    leaf_sg[best_leaf] = bs.left_sum_gradient; leaf_sh[best_leaf] = bs.left_sum_hessian;
    leaf_sg[new_leaf] = bs.right_sum_gradient; leaf_sh[new_leaf] = bs.right_sum_hessian;
    best[best_leaf].gain = -INFINITY; best[best_leaf].feature = -1;
    best[new_leaf].gain = -INFINITY; best[new_leaf].feature = -1;
    ++num_leaves;
    left_leaf = best_leaf; right_leaf = new_leaf;
  }
  h->leaf_begin = leaf_begin; h->leaf_cnt = leaf_cnt; h->last_num_leaves = num_leaves;
  h->leaf_buf.assign(L, 0);  // the host-driven loop copies every partition back into the first buffer
  *num_leaves_out = num_leaves;
  return 0;
}

int gpbdev_tree_add_score(gpbdev_tree_t h, const double* leaf_values, int num_leaves, double* score_dev, int32_t* leaf_of_row_dev) {
  if (!h || !leaf_values) return tfail("gpbdev_tree_add_score: null argument");
  if (num_leaves != h->last_num_leaves) return tfail("gpbdev_tree_add_score: num_leaves does not match the last trained tree");
  TCUDA(cudaSetDevice(h->device));
  std::vector<int32_t> lb(h->leaf_begin.begin(), h->leaf_begin.begin() + num_leaves), lc(h->leaf_cnt.begin(), h->leaf_cnt.begin() + num_leaves);
  TCUDA(cudaMemcpyAsync(h->leaf_begin_dev, lb.data(), sizeof(int32_t) * num_leaves, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaMemcpyAsync(h->leaf_cnt_dev, lc.data(), sizeof(int32_t) * num_leaves, cudaMemcpyHostToDevice, h->stream));
  std::vector<int32_t> lbuf(h->leaf_buf.begin(), h->leaf_buf.begin() + num_leaves);
  TCUDA(cudaMemcpyAsync(h->leaf_buf_dev, lbuf.data(), sizeof(int32_t) * num_leaves, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaMemcpyAsync(h->leaf_val_dev, leaf_values, sizeof(double) * num_leaves, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));  // the host vectors above are temporaries
  dim3 grid((unsigned)std::min<int64_t>((h->n / num_leaves + 255) / 256 + 1, 1024), num_leaves);
  add_score_kernel<<<grid, 256, 0, h->stream>>>(h->idx, h->idx_tmp, h->leaf_buf_dev, h->leaf_begin_dev, h->leaf_cnt_dev, h->leaf_val_dev, score_dev, leaf_of_row_dev);
  TCUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

// bench hook: device time of the root-pass histogram kernel alone (all n rows, the learner's default kernel), L2 flushed before each
// of `reps` launches; CUDA events on the learner's stream. Algorithmic bytes per launch: n * (Fpad + 8) (SURVEY §8d).
int gpbdev_tree_time_root_hist(gpbdev_tree_t h, const double* grad_dev, int reps, float* mean_ms) {
  if (!h || !grad_dev || !mean_ms || reps < 1) return tfail("gpbdev_tree_time_root_hist: bad argument");
  TCUDA(cudaSetDevice(h->device));
  const int F = h->F, Fpad = h->Fpad;
  const int64_t n = h->n;
  cudaEvent_t e0, e1;
  TCUDA(cudaEventCreate(&e0)); TCUDA(cudaEventCreate(&e1));
  double* flush = nullptr;
  const size_t flush_bytes = (size_t)256 << 20;
  TCUDA(cudaMalloc(&flush, flush_bytes));
  const int nw = hist2_warps(F);
  const int64_t rpc = std::max<int64_t>(128, ((n + h->num_sms - 1) / h->num_sms + 7) / 8 * 8);
  const int nchunks = (int)((n + rpc - 1) / rpc);
  const dim3 grid(nchunks, (Fpad + 63) / 64);
  double total = 0.;
  for (int r = 0; r < reps + 1; ++r) {
    TCUDA(cudaMemsetAsync(flush, r, flush_bytes, h->stream));
    TCUDA(cudaEventRecord(e0, h->stream));
    if (h->hist_kernel_version == 4)
      hist3_kernel<true><<<grid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, nullptr, 0, n, rpc, grad_dev, h->part_g, h->part_c, nullptr, nullptr);
    else if (h->hist_kernel_version == 3)
      hist3_kernel<false><<<grid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, nullptr, 0, n, rpc, grad_dev, h->part_g, h->part_c, nullptr, nullptr);
    else
      hist2_kernel<<<grid, nw * 32, hist2_smem(nw), h->stream>>>(h->bins, Fpad, F, nullptr, 0, n, rpc, grad_dev, h->part_g, h->part_c, nullptr, nullptr);
    TCUDA(cudaEventRecord(e1, h->stream));
    TCUDA(cudaEventSynchronize(e1));
    float ms = 0.f;
    TCUDA(cudaEventElapsedTime(&ms, e0, e1));
    if (r > 0) total += ms;  // first launch = warm-up
  }
  h->launches += reps + 1;
  cudaFree(flush); cudaEventDestroy(e0); cudaEventDestroy(e1);
  *mean_ms = (float)(total / reps);
  return 0;
}

int gpbdev_tree_leaf_indices(gpbdev_tree_t h, const int32_t** leaf_of_row_dev) {
  if (!h || !leaf_of_row_dev) return tfail("gpbdev_tree_leaf_indices: null argument");
  if (h->last_num_leaves < 1) return tfail("gpbdev_tree_leaf_indices: no tree has been trained");
  TCUDA(cudaSetDevice(h->device));
  if (!h->leaf_of_row) TCUDA(cudaMalloc(&h->leaf_of_row, sizeof(int32_t) * h->n));
  const int nl = h->last_num_leaves;
  std::vector<int32_t> lb(h->leaf_begin.begin(), h->leaf_begin.begin() + nl), lc(h->leaf_cnt.begin(), h->leaf_cnt.begin() + nl);
  TCUDA(cudaMemcpyAsync(h->leaf_begin_dev, lb.data(), sizeof(int32_t) * nl, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaMemcpyAsync(h->leaf_cnt_dev, lc.data(), sizeof(int32_t) * nl, cudaMemcpyHostToDevice, h->stream));
  std::vector<int32_t> lbuf(h->leaf_buf.begin(), h->leaf_buf.begin() + nl);
  TCUDA(cudaMemcpyAsync(h->leaf_buf_dev, lbuf.data(), sizeof(int32_t) * nl, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  dim3 grid((unsigned)std::min<int64_t>((h->n / nl + 255) / 256 + 1, 1024), nl);
  add_score_kernel<<<grid, 256, 0, h->stream>>>(h->idx, h->idx_tmp, h->leaf_buf_dev, h->leaf_begin_dev, h->leaf_cnt_dev, h->leaf_val_dev, nullptr, h->leaf_of_row);
  TCUDA(cudaGetLastError());
  TCUDA(cudaStreamSynchronize(h->stream));
  h->launches += 1;
  *leaf_of_row_dev = h->leaf_of_row;
  return 0;
}

// ---- device vectors owned by the host-side Booster (training score, label, gradient)
int gpbdev_vec_alloc(gpbdev_tree_t h, double** out, int64_t n) {
  if (!h || !out) return tfail("gpbdev_vec_alloc: null argument");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaMalloc(out, sizeof(double) * n));
  TCUDA(cudaMemsetAsync(*out, 0, sizeof(double) * n, h->stream));
  return 0;
}
int gpbdev_vec_free(gpbdev_tree_t h, double* p) {
  if (h) cudaSetDevice(h->device);
  cudaFree(p);
  return 0;
}
int gpbdev_vec_upload(gpbdev_tree_t h, double* dst_dev, const double* src_host, int64_t n) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaMemcpyAsync(dst_dev, src_host, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}
int gpbdev_vec_download(gpbdev_tree_t h, double* dst_host, const double* src_dev, int64_t n) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaMemcpyAsync(dst_host, src_dev, sizeof(double) * n, cudaMemcpyDeviceToHost, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}
// out = a - b   (RegressionL2loss::GetGradients: grad = score - label, regression_objective.hpp:158-162)
int gpbdev_vec_sub(gpbdev_tree_t h, const double* a_dev, const double* b_dev, double* out_dev, int64_t n) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  sub_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(a_dev, b_dev, out_dev, n);
  TCUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}
int gpbdev_vec_add_const(gpbdev_tree_t h, double* a_dev, double c, int64_t n) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  add_const_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(a_dev, c, n);
  TCUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

int gpbdev_vec_dot(gpbdev_tree_t h, const double* a_dev, const double* b_dev, int64_t n, double* out_host) {
  if (!h || !a_dev || !b_dev || !out_host) return tfail("gpbdev_vec_dot: null argument");
  TCUDA(cudaSetDevice(h->device));
  const int nb1 = (int)std::min<int64_t>(1023, (n + 4095) / 4096);
  dot_stage1_kernel<<<nb1, 256, 0, h->stream>>>(a_dev, b_dev, n, h->sum_part);
  sum_stage2_kernel<<<1, 256, 0, h->stream>>>(h->sum_part, nb1, h->sum_part + 1023);
  TCUDA(cudaGetLastError());
  TCUDA(cudaMemcpyAsync(h->scalar_host, h->sum_part + 1023, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  *out_host = h->scalar_host[0];
  h->launches += 2;
  return 0;
}
int gpbdev_vec_zero(gpbdev_tree_t h, double* a_dev, int64_t n) {
  if (!h || !a_dev) return tfail("gpbdev_vec_zero: null argument");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaMemsetAsync(a_dev, 0, sizeof(double) * n, h->stream));
  return 0;
}
int gpbdev_vec_copy(gpbdev_tree_t h, double* dst_dev, const double* src_dev, int64_t n) {
  if (!h || !dst_dev || !src_dev) return tfail("gpbdev_vec_copy: null argument");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaMemcpyAsync(dst_dev, src_dev, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

int gpbdev_tree_sync(gpbdev_tree_t h) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // extern "C"
