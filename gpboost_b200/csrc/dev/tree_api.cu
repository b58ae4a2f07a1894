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
// Design (one split = five launches on one GPU):
//  * bins live row-major n x Fpad (Fpad = 32-multiple), so the bins of one row and 32 features are one 32-byte sector;
//  * hist3_kernel: chunk partial histograms of the smaller child, one CTA per SM and row chunk, deterministic (no fp64 atomics);
//  * reduce_scan2_kernel: one CTA per feature merges the chunk partials in a fixed order, takes larger = parent - smaller and
//    replays the reference's right-to-left scan for both children with identical arithmetic;
//  * tree_advance_kernel: best split per child and best leaf with SplitInfo's tie rule, Tree::Split, the plan of the next split;
//  * part_count_kernel + part_scatter_kernel: stable partition, like the reference's ordered partition.
// The leaf loop itself runs on the device (tree_grow); HBM traffic per split = rows_in_smaller_leaf * (Fpad + 12) bytes.
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
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
  int inherit;         // 1: features flagged unsplittable in the parent (row parent_row of the flags) are skipped
  int num_data;
  double sum_gradients, sum_hessians;
};

// Work description for the leaf loop (tree_*_kernel below): written by one thread between the data-parallel kernels of a split,
// read by every CTA of the next kernel in the stream.
struct DevJob {
  int done, error;
  int do_find;
  int hist_begin, hist_cnt, hist_use_idx, hist_rpc, hist_nchunks;
  LeafArgs a0, a1;
  int parent_row;
  int part_on, part_begin, part_cnt, part_feature, part_threshold, part_seg, part_nseg;
  // ping-pong row-index buffers: a split reads its leaf's rows from one buffer and writes the two
  // children (same positions) into the other — no copy back. hist_buf / part_buf: which buffer holds the leaf in question.
  int hist_buf, part_buf;
};

// ---- histogram: one CTA = one row chunk x up to 64 features (all of them at F <= 64), one CTA per SM.
// Warp w owns the four features 4w..4w+3 of the CTA's feature group and a private histogram for them
// (4 x 256 x (f64 + u32) = 12 KB): thirteen accumulation chains per SM at F = 50. Rows of the chunk are staged tile by tile
// (256 rows, one row per thread: row id -> the row's bins + one gradient, through registers one tile ahead) into shared memory
// TRANSPOSED, tb[feature][row], so that the bins of one feature for eight consecutive rows are one aligned 8-byte word; tile rows
// are padded by 8 bytes, so the four 8-byte bin words of a warp fall into different banks. Lane = (row slot 0..7, feature 0..3):
// eight rows advance per step, branch-free:
//   * every lane loads the 8-byte word of its feature and finds the slots holding its own bin with byte-parallel
//     arithmetic (exact zero-byte test of word ^ bin * 0x01010101);
//   * the FIRST slot of every (feature, bin) group is the group's leader: it alone touches the counter — one shared-memory
//     load, its own gradient and then the gradients of the later members in slot order (predicated additions, the step's
//     gradients loaded only by leaders whose group has later members), one store, one integer RED for the count.
// No atomics on the fp64 sums, no votes, no divergence: the additions on a counter follow a fixed schedule (row order
// inside a step, steps in row order), so the result is deterministic, and a low-cardinality feature (all eight rows in one
// bin) costs the same as a high-cardinality one. (Groups found with match.any — MATCH.ANY costs ~750 cycles when last
// measured — or resolved by rank rounds — divergent: a constant padding feature made its warp 8x slower than the others, which
// then waited at the tile barrier — were slower. A plain load / add / store of the counter instead of the RED measured 7 % slower.)
constexpr int kHistTile = 256;
constexpr int kHistMaxWarps = 16;
constexpr int kHist3Stride = kHistTile + 8;
static inline int hist_warps(int F) { return std::max(8, std::min(kHistMaxWarps, (std::min(F, 64) + 3) / 4)); }
static inline size_t hist3_smem(int nw) { return (size_t)nw * 4 * kBins * 12 + 64 * kHist3Stride + kHistTile * 8; }
// bit 7 of every byte of the result is set iff that byte of x is zero (exact: the 7-bit partial sums cannot carry)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu); }
__global__ void __launch_bounds__(kHistMaxWarps * 32, 1) hist3_kernel(const uint8_t* __restrict__ bins, int Fpad, int F,
                                                                      const int32_t* __restrict__ idx, int64_t begin, int64_t count,
                                                                      int64_t rows_per_chunk, const double* __restrict__ grad,
                                                                      double* __restrict__ part_g, uint32_t* __restrict__ part_c,
                                                                      const DevJob* __restrict__ job, const int32_t* __restrict__ idx_alt) {
  if (job) {  // leaf loop: the leaf's row range comes from the planner (no job: gpbdev_tree_time_root_hist's root pass)
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
        atomicAdd(&myc[mybin], members);
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

// data-parallel learner: this rank's chunk partials -> stage[f][bin] = (sum grad, count * hess_const) (dataset.cpp:1223-1226), the
// histogram of the smaller child that is then all-reduced. Block = (feature, 32 bins) x 8 warps; warp s sums a contiguous eighth
// of the chunks in chunk order, then the eight slice sums are added in slice order: a fixed summation tree (deterministic),
// 8 x 32 threads per 32 counters in flight.
constexpr int kReduceSlices = 8;
__global__ void __launch_bounds__(kReduceSlices * 32) hist_reduce_kernel(const double* __restrict__ part_g, const uint32_t* __restrict__ part_c,
                                                                         int Fpad, double hess_const, double* __restrict__ stage,
                                                                         const DevJob* __restrict__ job) {
  if (job->done || !job->do_find) return;
  const int nchunks = job->hist_nchunks;
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
  const int t = f * kBins + b;
  stage[2 * t] = g;
  stage[2 * t + 1] = (double)c * hess_const;
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
// ---- merge + subtraction + split scan of the two newest leaves in one launch: block = one feature. 32 warps merge the feature's
// chunk partials (warp = (slice of the chunks, 32 bins), slices added in slice order), 256 threads write the smaller child's
// histogram, take larger = parent - smaller in place (feature_histogram.hpp:79-83) and keep both in shared memory; then each
// child's right-to-left scan (feature_histogram.hpp:858-960, result :1057-1083) runs straight from there.
// The reference walks t = nb-1 .. 1 accumulating the right-hand sums in that order and keeps the FIRST strictly larger gain. Its
// `continue` / `break` tests are monotone in t (counts and hessian sums only grow), so a threshold is admissible iff it passes all
// tests itself: one lane per child reproduces the running sums sequentially (fp64 order matters), then one thread per threshold
// evaluates its gain (two fp64 divisions, once) and the block picks the maximum, ties to the larger t (= the first one met).
// scan_sums: the per-bin counts and the sequential running sums of one child, one warp
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
constexpr int kFusedSlices = 4;
__global__ void __launch_bounds__(kFusedSlices * kBins) reduce_scan2_kernel(
    const double* __restrict__ part_g, const uint32_t* __restrict__ part_c, int Fpad, int F, double hess_const,
    double* __restrict__ hist_base, int64_t slot_stride, const int32_t* __restrict__ num_bin,
    int min_data_in_leaf, double min_sum_hessian, double lambda_l2, double min_gain_to_split, unsigned char* __restrict__ splittable,
    SplitOut* __restrict__ cand, const DevJob* __restrict__ job, const double* __restrict__ stage) {
  if (job->done || !job->do_find) return;
  const int nchunks = stage ? 0 : job->hist_nchunks;
  const LeafArgs a0 = job->a0, a1 = job->a1;
  const int parent_row = job->parent_row;
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

// ---- stable partition of the leaf the selector picked, in two kernels. Every CTA owns one contiguous segment of the leaf's
// rows. part_count_kernel: go-left flags (one byte per row) + lefts per segment. part_scatter_kernel: every CTA sums the segment
// counts in front of it (<= a few hundred values), then walks its segment tile by tile in row order with ballot / popc ranks,
// so lefts keep their order at the front and rights theirs behind (data_partition.hpp:101-120). The two row-index buffers
// alternate: the leaf is read from the buffer that holds it and the children are written at the same positions of the other one.
constexpr int kPartThreads = 256;
__global__ void __launch_bounds__(kPartThreads) part_count_kernel(const uint8_t* __restrict__ bins, int Fpad, const int32_t* __restrict__ idx0,
                                                                  const int32_t* __restrict__ idx1, uint8_t* __restrict__ flag,
                                                                  int32_t* __restrict__ seg_left, const DevJob* __restrict__ job) {
  if (job->done || !job->part_on || (int)blockIdx.x >= job->part_nseg) return;
  const int feature = job->part_feature, threshold = job->part_threshold;
  const int64_t begin = job->part_begin, count = job->part_cnt, seg = job->part_seg;
  const int32_t* __restrict__ idx = job->part_buf ? idx1 : idx0;
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
__global__ void __launch_bounds__(kPartThreads) part_scatter_kernel(int32_t* __restrict__ idx0, int32_t* __restrict__ idx1,
                                                                    const uint8_t* __restrict__ flag, const int32_t* __restrict__ seg_left,
                                                                    const DevJob* __restrict__ job) {
  if (job->done || !job->part_on || (int)blockIdx.x >= job->part_nseg) return;
  const int64_t begin = job->part_begin, count = job->part_cnt, seg = job->part_seg;
  const int nseg = job->part_nseg;
  const int32_t* __restrict__ idx = job->part_buf ? idx1 : idx0;
  int32_t* __restrict__ out = (job->part_buf ? idx0 : idx1) + begin;
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
      out[dst] = idx[begin + j];
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

// ---- validation data ----------------------------------------------------------------------------------------------------------
// score[i] += leaf_value[leaf(i)] (Tree::AddPredictionToScore, tree.h:104-120): one thread per row walks the tree on the row's bins,
// bin <= threshold_bin -> left (the bin form of NumericalDecision for bins made by the training data's bin mappers). Nodes are one
// int4 each, read through the read-only cache; every row touches one byte per level of its own row.
__global__ void __launch_bounds__(256) valid_tree_score_kernel(const uint8_t* __restrict__ bins, int Fpad, int64_t n,
                                                               const int4* __restrict__ nodes, const double* __restrict__ leaf_value,
                                                               double* __restrict__ score) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* __restrict__ row = bins + i * Fpad;
    int node = 0;
    while (node >= 0) {
      const int4 nd = __ldg(nodes + node);
      node = (int)row[nd.x] <= nd.y ? nd.z : nd.w;
    }
    score[i] += __ldg(leaf_value + ~node);
  }
}

// Metric sums (RegressionMetric / TestNegLogLikelihood, regression_metric.hpp): kMetricAcc accumulators per row, fixed contiguous
// block ranges and a fixed shared-memory tree, then one block per accumulator sums the block partials in block order.
constexpr int kMetricAcc = 4;
constexpr int kMetricMaxBlocks = 1024;
__global__ void __launch_bounds__(256) metric_stage1_kernel(const double* __restrict__ score, const double* __restrict__ label, int64_t n,
                                                            const double* __restrict__ gp_mean, const double* __restrict__ gp_dvar,
                                                            double sigma2, double shift, double* __restrict__ part) {
  __shared__ double sh[kMetricAcc][256];
  double s_sq = 0., s_abs = 0., s_lin = 0., s_nll = 0.;
  const int64_t per = (n + gridDim.x - 1) / gridDim.x;
  const int64_t b = (int64_t)blockIdx.x * per, e = min(b + per, n);
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
    double p = score[i];
    if (gp_mean) p -= gp_mean[i];  // score - (mean of F - y): the GP's prediction of y - F added to F (regression_metric.hpp:102)
    const double r = p - label[i];
    const double rs = r + shift;
    s_sq += rs * rs;
    s_abs += fabs(r);
    s_lin += r;
    if (gp_dvar) {
      const double v = sigma2 * (gp_dvar[i] + 1.);  // response variance: sigma^2 D_p plus the nugget sigma^2 (REModel::Predict)
      s_nll += r * r / v + log(v);
    }
  }
  sh[0][threadIdx.x] = s_sq; sh[1][threadIdx.x] = s_abs; sh[2][threadIdx.x] = s_lin; sh[3][threadIdx.x] = s_nll;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int k = 0; k < kMetricAcc; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < kMetricAcc) part[(size_t)threadIdx.x * kMetricMaxBlocks + blockIdx.x] = sh[threadIdx.x][0];
}
__global__ void __launch_bounds__(256) metric_stage2_kernel(const double* __restrict__ part, int nb, double* __restrict__ out) {
  __shared__ double sh[256];
  const double* __restrict__ p = part + (size_t)blockIdx.x * kMetricMaxBlocks;
  double s = 0.;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s += p[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) out[blockIdx.x] = sh[0];
}

// ---- the leaf loop on the device: the state SerialTreeLearner::Train keeps on the host (leaf ranges and sums, best split per leaf,
// the growing tree; serial_tree_learner.cpp:159-209, tree.h:533-575) lives in HBM, one thread advances it between the data-parallel
// kernels, and the host enqueues the kernels of the splits without reading anything back per split.
// Per-leaf arrays hold num_leaves entries and are allocated with the learner. The records the host reads after a tree (LeafOut)
// follow the TreeDevState in one allocation, so the state and the records of the leaves grown come back in one copy.
struct LeafOut {  // internal node i (i < num_leaves - 1) and leaf i of the tree
  double leaf_value;
  float split_gain;
  int split_feature, threshold_bin, left_child, right_child, leaf_count;
  // this rank's rows of the leaf (partition and histogram ranges) and which of the two row-index buffers holds them
  int leaf_begin, leaf_cnt, leaf_buf;
};
struct LeafWork {  // per-leaf state that stays on the device
  SplitOut best;
  double sg, sh;  // gradient and hessian sums
  // cnt_g: rows over all ranks — every decision uses the global counts so that all ranks of a data-parallel learner grow the same
  // tree (equal to leaf_cnt on one GPU); slot: the histogram slot of the leaf
  int cnt_g, depth, parent, slot;
};
struct alignas(16) TreeDevState {
  DevJob job;
  int num_leaves, left_leaf, right_leaf, next_slot;
  LeafWork* work;  // [num_leaves]
  LeafOut* out;    // [num_leaves], right behind this struct
};

// BeforeFindBestSplit (serial_tree_learner.cpp:283-322): may the two newest leaves be examined, which one gets a histogram pass
// keep_part: called from tree_advance_kernel BEFORE the partition of the split that was just selected ran — its job must stay armed
__device__ void tree_plan_body(TreeDevState* __restrict__ st, int max_depth, int min_data_in_leaf, int num_chunk_ctas, bool keep_part) {
  DevJob& job = st->job;
  LeafWork* w = st->work;
  const LeafOut* o = st->out;
  job.do_find = 0;
  if (!keep_part) job.part_on = 0;
  if (job.done) return;
  const int left_leaf = st->left_leaf, right_leaf = st->right_leaf;
  bool do_find = true;
  if (max_depth > 0 && w[left_leaf].depth >= max_depth) do_find = false;
  if (do_find) {
    const int nl = w[left_leaf].cnt_g, nr = right_leaf >= 0 ? w[right_leaf].cnt_g : 0;
    if (nr < min_data_in_leaf * 2 && nl < min_data_in_leaf * 2) do_find = false;
  }
  if (!do_find) {
    w[left_leaf].best.gain = -INFINITY;
    if (right_leaf >= 0) w[right_leaf].best.gain = -INFINITY;
    return;
  }
  int smaller, larger = -1, parent_slot = -1;
  if (right_leaf < 0) smaller = left_leaf;
  else if (w[left_leaf].cnt_g < w[right_leaf].cnt_g) { smaller = left_leaf; larger = right_leaf; }
  else { smaller = right_leaf; larger = left_leaf; }
  if (right_leaf >= 0) parent_slot = w[left_leaf].slot;  // the parent's histograms sit under the left (= parent) id
  const int new_slot = st->next_slot++;
  if (larger >= 0) w[larger].slot = parent_slot;  // larger = parent - smaller, in place
  w[smaller].slot = new_slot;
  LeafArgs a0, a1;
  a0.leaf = smaller; a0.hist_slot = new_slot; a0.inherit = right_leaf >= 0 ? 1 : 0; a0.num_data = w[smaller].cnt_g;
  a0.sum_gradients = w[smaller].sg; a0.sum_hessians = w[smaller].sh;
  a1.leaf = larger; a1.hist_slot = larger >= 0 ? parent_slot : 0; a1.inherit = 1; a1.num_data = larger >= 0 ? w[larger].cnt_g : 0;
  a1.sum_gradients = larger >= 0 ? w[larger].sg : 0.; a1.sum_hessians = larger >= 0 ? w[larger].sh : 0.;
  job.a0 = a0; job.a1 = a1;
  job.parent_row = left_leaf;
  const int cnt = o[smaller].leaf_cnt;
  job.hist_begin = o[smaller].leaf_begin; job.hist_cnt = cnt; job.hist_use_idx = st->num_leaves > 1 ? 1 : 0;
  job.hist_buf = o[smaller].leaf_buf;
  int rpc = ((cnt + num_chunk_ctas - 1) / num_chunk_ctas + 7) / 8 * 8;  // one CTA per SM and chunk, whole 8-row steps per chunk
  if (rpc < 128) rpc = 128;
  job.hist_rpc = rpc; job.hist_nchunks = (cnt + rpc - 1) / rpc;
  job.do_find = 1;
}

// BeforeTrain (leaf_splits.hpp:70-83): all rows in leaf 0; then the plan of the first split
__global__ void tree_init_kernel(TreeDevState* __restrict__ st, const double* __restrict__ root_sum_gradient, int n, int n_global,
                                 double hess_const, int L, int max_depth, int min_data_in_leaf, int num_chunk_ctas) {
  LeafWork* w = st->work;
  LeafOut* o = st->out;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    w[l].best.gain = -INFINITY; w[l].best.feature = -1;
    w[l].sg = 0.; w[l].sh = 0.; w[l].cnt_g = 0; w[l].depth = 0; w[l].parent = -1; w[l].slot = -1;
    o[l].leaf_value = 0.; o[l].split_gain = 0.f; o[l].split_feature = 0; o[l].threshold_bin = 0; o[l].left_child = 0; o[l].right_child = 0;
    o[l].leaf_count = 0; o[l].leaf_begin = 0; o[l].leaf_cnt = 0; o[l].leaf_buf = 0;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  st->job.done = 0; st->job.error = 0; st->job.do_find = 0; st->job.part_on = 0;
  st->num_leaves = 1; st->left_leaf = 0; st->right_leaf = -1; st->next_slot = 0;
  o[0].leaf_cnt = n;
  w[0].cnt_g = n_global;
  w[0].sg = root_sum_gradient[0];
  w[0].sh = hess_const * (double)n_global;
  o[0].leaf_count = n_global;
  tree_plan_body(st, max_depth, min_data_in_leaf, num_chunk_ctas, false);
}

// Tree::Split (tree.h:533-575) of best_leaf and the partition job
// sharded != 0: the children's LOCAL row ranges are not known before the partition ran (tree_local_ranges_kernel sets them)
__device__ void tree_select_body(TreeDevState* __restrict__ st, int best_leaf, double min_gain_to_split, int max_seg, int sharded) {
  DevJob& job = st->job;
  LeafWork* w = st->work;
  LeafOut* o = st->out;
  job.part_on = 0;
  const int num_leaves = st->num_leaves;
  const SplitOut bs = w[best_leaf].best;
  if (!(bs.gain > 0.0)) { job.done = 1; return; }
  const int b = o[best_leaf].leaf_begin, c = o[best_leaf].leaf_cnt;
  // With a constant hessian the histogram's hessian entries are exact multiples of it, so the split scan's RoundInt(hess * cnt_factor)
  // counts ARE the partition's counts (the reference overwrites them with the partition's, serial_tree_learner.cpp:589-593 — same numbers)
  const int nleft = bs.left_count, nright = w[best_leaf].cnt_g - nleft;
  if (nleft <= 0 || nright <= 0) { job.error = 1; job.done = 1; return; }
  job.part_on = 1; job.part_begin = b; job.part_cnt = c; job.part_feature = bs.feature; job.part_threshold = bs.threshold;
  job.part_buf = o[best_leaf].leaf_buf;
  int seg = ((c + max_seg - 1) / max_seg + kPartThreads - 1) / kPartThreads * kPartThreads;
  if (seg < 4 * kPartThreads) seg = 4 * kPartThreads;
  job.part_seg = seg; job.part_nseg = (c + seg - 1) / seg;
  const int new_leaf = num_leaves;
  o[best_leaf].leaf_buf = o[new_leaf].leaf_buf = 1 - job.part_buf;  // the children are written into the other buffer
  w[best_leaf].cnt_g = nleft; w[new_leaf].cnt_g = nright;
  if (!sharded) { o[best_leaf].leaf_cnt = nleft; o[new_leaf].leaf_begin = b + nleft; o[new_leaf].leaf_cnt = nright; }
  const int node = num_leaves - 1;
  const int parent = w[best_leaf].parent;
  if (parent >= 0) { if (o[parent].left_child == ~best_leaf) o[parent].left_child = node; else o[parent].right_child = node; }
  o[node].split_feature = bs.feature; o[node].threshold_bin = bs.threshold;
  o[node].split_gain = (float)(bs.gain + min_gain_to_split);
  o[node].left_child = ~best_leaf; o[node].right_child = ~new_leaf;
  w[best_leaf].parent = node; w[new_leaf].parent = node;
  o[best_leaf].leaf_value = isnan(bs.left_output) ? 0. : bs.left_output; o[best_leaf].leaf_count = nleft;
  o[new_leaf].leaf_value = isnan(bs.right_output) ? 0. : bs.right_output; o[new_leaf].leaf_count = nright;
  w[new_leaf].depth = w[best_leaf].depth + 1; w[best_leaf].depth++;
  w[best_leaf].sg = bs.left_sum_gradient; w[best_leaf].sh = bs.left_sum_hessian;
  w[new_leaf].sg = bs.right_sum_gradient; w[new_leaf].sh = bs.right_sum_hessian;
  w[best_leaf].best.gain = -INFINITY; w[best_leaf].best.feature = -1;
  w[new_leaf].best.gain = -INFINITY; w[new_leaf].best.feature = -1;
  st->num_leaves = num_leaves + 1;
  st->left_leaf = best_leaf; st->right_leaf = new_leaf;
}

// SplitInfo::operator>, then the smaller leaf index: ArrayArgs::ArgMax keeps the first of equal maxima
__device__ __forceinline__ bool leaf_better(double ga, int fa, int la, double gb, int fb, int lb) {
  return split_better(ga, fa, gb, fb) || (!split_better(gb, fb, ga, fa) && la < lb);
}

// One launch between the split scan and the partition: the arg-max over the per-feature candidates of both children, the best leaf
// over all leaves, the selector, and on one GPU the planner of the NEXT split (plan_next: it needs nothing the partition produces there,
// the children's ranges follow from the split's counts). Row shards run the planner after the partition (tree_local_ranges_kernel).
constexpr int kAdvanceThreads = 128;
__global__ void __launch_bounds__(kAdvanceThreads) tree_advance_kernel(TreeDevState* __restrict__ st, const SplitOut* __restrict__ cand, int F,
                                                                      double min_gain_to_split, int max_seg, int max_depth, int min_data_in_leaf,
                                                                      int num_chunk_ctas, int plan_next, int sharded) {
  __shared__ SplitOut sh[kAdvanceThreads];
  __shared__ double lg[kAdvanceThreads];
  __shared__ int lf[kAdvanceThreads], ll[kAdvanceThreads];
  const DevJob& job = st->job;
  if (job.done) return;
  const int tid = threadIdx.x, child = tid >> 6, t = tid & 63;
  SplitOut best;
  best.gain = -INFINITY; best.feature = -1; best.threshold = 0; best.left_count = best.right_count = 0;
  best.left_output = best.right_output = 0.;
  best.left_sum_gradient = best.left_sum_hessian = best.right_sum_gradient = best.right_sum_hessian = 0.;
  if (job.do_find) {
    for (int f = t; f < F; f += 64) {
      const SplitOut c = cand[child * F + f];
      if (split_better(c.gain, c.feature, best.gain, best.feature)) best = c;
    }
  }
  sh[tid] = best;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) {
    if (t < o) {
      const SplitOut& c = sh[tid + o];
      if (split_better(c.gain, c.feature, sh[tid].gain, sh[tid].feature)) sh[tid] = c;
    }
    __syncthreads();
  }
  if (job.do_find && t == 0) {
    const int leaf = child == 0 ? job.a0.leaf : job.a1.leaf;
    if (leaf >= 0) st->work[leaf].best = sh[tid];
  }
  __syncthreads();
  // the leaf with the best split: strided over the leaves, then a tree reduction (the order is total: any reduction order agrees)
  const LeafWork* w = st->work;
  const int num_leaves = st->num_leaves;
  double bg = -INFINITY;
  int bf = -1, bl = 0x7fffffff;
  for (int l = tid; l < num_leaves; l += kAdvanceThreads)
    if (leaf_better(w[l].best.gain, w[l].best.feature, l, bg, bf, bl)) { bg = w[l].best.gain; bf = w[l].best.feature; bl = l; }
  lg[tid] = bg; lf[tid] = bf; ll[tid] = bl;
  __syncthreads();
  for (int o = kAdvanceThreads / 2; o > 0; o >>= 1) {
    if (tid < o && leaf_better(lg[tid + o], lf[tid + o], ll[tid + o], lg[tid], lf[tid], ll[tid])) {
      lg[tid] = lg[tid + o]; lf[tid] = lf[tid + o]; ll[tid] = ll[tid + o];
    }
    __syncthreads();
  }
  if (tid != 0) return;
  tree_select_body(st, ll[0], min_gain_to_split, max_seg, sharded);
  if (plan_next) tree_plan_body(st, max_depth, min_data_in_leaf, num_chunk_ctas, true);
}

// data-parallel learner: after the local partition, the children's ranges on THIS rank (lefts counted by part_count_kernel); then the
// plan of the next split
__global__ void tree_local_ranges_kernel(TreeDevState* __restrict__ st, const int32_t* __restrict__ seg_left, int max_depth,
                                         int min_data_in_leaf, int num_chunk_ctas, int plan_next) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const DevJob& job = st->job;
  if (!job.done && job.part_on) {
    int nl = 0;
    for (int k = 0; k < job.part_nseg; ++k) nl += seg_left[k];
    LeafOut* o = st->out;
    const int best_leaf = st->left_leaf, new_leaf = st->right_leaf;
    o[best_leaf].leaf_cnt = nl;
    o[new_leaf].leaf_begin = job.part_begin + nl;
    o[new_leaf].leaf_cnt = job.part_cnt - nl;
  }
  if (plan_next) tree_plan_body(st, max_depth, min_data_in_leaf, num_chunk_ctas, false);
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
  int32_t *idx = nullptr, *idx_tmp = nullptr;  // the two row-index buffers of the leaf loop
  double* grad = nullptr;         // n (device copy when the caller passes host gradients)
  double* hist = nullptr;         // (L + 1) slots x F x 256 x 2
  unsigned char* splittable = nullptr;  // L x F, row = leaf id (FeatureHistogram::is_splittable_)
  double* part_g = nullptr;
  uint32_t* part_c = nullptr;
  int max_chunks = 0;
  uint8_t* flag8 = nullptr;        // n go-left flags of the leaf being split
  int32_t* seg_left = nullptr;     // lefts per partition segment
  int max_seg = 0;
  cudaGraphExec_t graph_exec = nullptr;  // the whole tree, captured for (graph_grad, graph_hess)
  const double* graph_grad = nullptr;
  double graph_hess = 0.;
  TreeDevState* state_dev = nullptr;   // followed by L LeafOut records
  TreeDevState* state_host = nullptr;  // pinned, same layout: the records of the last tree
  LeafWork* work_dev = nullptr;        // L
  double* sum_part = nullptr;
  SplitOut* cand_dev = nullptr;    // 2 x F per-feature candidates
  double* scalar_host = nullptr;   // pinned
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
  // validation data (lazy): one tree's nodes (L int4 {feature, threshold bin, left, right}) followed by its L leaf values; the metric
  // kernel's block partials (kMetricAcc x kMetricMaxBlocks, then kMetricAcc results)
  int4* vnodes_dev = nullptr;
  double* metric_part = nullptr;
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
  TCUDA(cudaMalloc(&h->grad, sizeof(double) * n));
  const size_t slot = (size_t)F * kBins * 2;
  TCUDA(cudaMalloc(&h->hist, sizeof(double) * slot * (h->L + 1)));
  TCUDA(cudaMalloc(&h->splittable, (size_t)h->L * F));
  h->max_chunks = h->num_sms * 2;
  TCUDA(cudaMalloc(&h->part_g, sizeof(double) * (size_t)h->max_chunks * h->Fpad * kBins));
  TCUDA(cudaMalloc(&h->part_c, sizeof(uint32_t) * (size_t)h->max_chunks * h->Fpad * kBins));
  TCUDA(cudaMalloc(&h->sum_part, sizeof(double) * 1024));
  TCUDA(cudaMalloc(&h->cand_dev, sizeof(SplitOut) * 2 * F));
  TCUDA(cudaMallocHost(&h->scalar_host, sizeof(double) * 4));
  TCUDA(cudaMalloc(&h->leaf_begin_dev, sizeof(int32_t) * h->L));
  TCUDA(cudaMalloc(&h->leaf_cnt_dev, sizeof(int32_t) * h->L));
  TCUDA(cudaMalloc(&h->leaf_buf_dev, sizeof(int32_t) * h->L));
  TCUDA(cudaMalloc(&h->leaf_val_dev, sizeof(double) * h->L));
  TCUDA(cudaFuncSetAttribute(hist3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist3_smem(hist_warps(F))));
  h->max_seg = h->num_sms * 4;
  TCUDA(cudaMalloc(&h->flag8, (size_t)n));
  TCUDA(cudaMalloc(&h->seg_left, sizeof(int32_t) * h->max_seg));
  const size_t state_bytes = sizeof(TreeDevState) + sizeof(LeafOut) * h->L;
  TCUDA(cudaMalloc(&h->state_dev, state_bytes));
  TCUDA(cudaMallocHost(&h->state_host, state_bytes));
  TCUDA(cudaMalloc(&h->work_dev, sizeof(LeafWork) * h->L));
  std::memset(h->state_host, 0, sizeof(TreeDevState));
  h->state_host->work = h->work_dev;
  h->state_host->out = reinterpret_cast<LeafOut*>(h->state_dev + 1);
  TCUDA(cudaMemcpy(h->state_dev, h->state_host, sizeof(TreeDevState), cudaMemcpyHostToDevice));
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
  cudaFree(h->bins_owned); cudaFree(h->leaf_of_row); cudaFree(h->stage); cudaFree(h->num_bin); cudaFree(h->idx); cudaFree(h->idx_tmp);
  cudaFree(h->grad); cudaFree(h->hist); cudaFree(h->splittable); cudaFree(h->part_g); cudaFree(h->part_c); cudaFree(h->sum_part);
  cudaFree(h->cand_dev); cudaFree(h->leaf_begin_dev); cudaFree(h->leaf_cnt_dev); cudaFree(h->leaf_buf_dev); cudaFree(h->leaf_val_dev);
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  cudaFree(h->state_dev); cudaFreeHost(h->state_host); cudaFree(h->work_dev);
  cudaFree(h->flag8); cudaFree(h->seg_left);
  cudaFreeHost(h->scalar_host);
  cudaFree(h->vnodes_dev); cudaFree(h->metric_part);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int64_t gpbdev_tree_launch_count(gpbdev_tree_t h) { return h ? h->launches : 0; }
void* gpbdev_tree_stream(gpbdev_tree_t h) { return h ? (void*)h->stream : nullptr; }

// A tree of up to kSplitBatch + 1 leaves is one batch of splits.
constexpr int kSplitBatch = 255;

// Grows one tree: the kernels of every split are enqueued without a host round trip per split; the planner / selector steer them
// through the job, and once the tree is finished the remaining launches return at once.
//  * device gradients on one GPU with num_leaves <= kSplitBatch + 1: the whole tree (root sums and the read-back included) is one CUDA
//    graph, captured once per (gradient buffer, hessian) and replayed every boosting iteration: one graph launch instead of ~5 per split;
//  * otherwise the same sequence is enqueued eagerly, kSplitBatch splits at a time; between batches the host reads job.done (one word)
//    and stops when it is set, so a tree that stops early costs at most one batch of no-op launches.
// Data-parallel learner (row shards over ranks): the root gradient sum and the smaller child's merged histogram are summed over the
// ranks ON THIS STREAM (NCCL kernels; DataParallelTreeLearner, data_parallel_tree_learner.cpp:155-175, :244), and the children's local
// row ranges are set after the local partition. Every rank enqueues the same number of collectives whatever the tree does (finished
// trees skip the work, not the exchange). The whole 2 F x 256 block is all-reduced and scanned on every rank: at F = 50..100 it is a
// 0.2..0.4 MB message, latency-bound on NVSwitch — a reduce-scatter by feature block (the reference's choice for Ethernet clusters)
// would add a second latency-bound collective per split for the best-split exchange and scan no faster (one CTA per feature either way).
static int tree_grow(gpbdev_tree_t h, const double* grad, double hess_const, bool graph_ok) {
  const int64_t n = h->n;
  const int F = h->F, Fpad = h->Fpad, L = h->L;
  const gpbdev_tree_config& cfg = h->cfg;
  const size_t slot_stride = (size_t)F * kBins * 2;
  TreeDevState* st = h->state_dev;
  const DevJob* job = &st->job;
  const bool sharded = h->allreduce != nullptr;
  const int n_glob = sharded ? (int)h->n_global : (int)n;
  if (sharded && !h->stage) {
    TCUDA(cudaMalloc(&h->stage, sizeof(double) * slot_stride));
    TCUDA(cudaMemsetAsync(h->stage, 0, sizeof(double) * slot_stride, h->stream));
    // one exchange of each message size before the first tree: the communicator sets up its channels / buffers for a
    // (size, algorithm) at the first call
    if (h->allreduce(h->allreduce_ctx, h->stage, (int64_t)slot_stride, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
    if (h->allreduce(h->allreduce_ctx, h->stage, 1, (void*)h->stream)) return tfail("gpbdev_tree_train: device all-reduce failed");
    TCUDA(cudaStreamSynchronize(h->stream));
  }
  bool coll_failed = false;
  auto enqueue_root = [&]() {
    iota_kernel<<<h->num_sms * 4, 256, 0, h->stream>>>(h->idx, n);
    const int nb1 = (int)std::min<int64_t>(1024, (n + 4095) / 4096);
    sum_stage1_kernel<<<nb1, 256, 0, h->stream>>>(grad, n, h->sum_part);
    sum_stage2_kernel<<<1, 256, 0, h->stream>>>(h->sum_part, nb1, h->sum_part + 1023);
    if (sharded && h->allreduce(h->allreduce_ctx, h->sum_part + 1023, 1, (void*)h->stream)) coll_failed = true;
    tree_init_kernel<<<1, 256, 0, h->stream>>>(st, h->sum_part + 1023, (int)n, n_glob, hess_const, L, cfg.max_depth, cfg.min_data_in_leaf,
                                               h->num_sms);
  };
  const int nw = hist_warps(F);
  const dim3 hgrid(h->num_sms, (Fpad + 63) / 64);
  auto enqueue_splits = [&](int s0, int s1) {
    for (int split = s0; split < s1 && !coll_failed; ++split) {
      const int plan_next = split + 1 < L - 1 ? 1 : 0;
      hist3_kernel<<<hgrid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, h->idx, 0, 0, 0, grad, h->part_g, h->part_c, job, h->idx_tmp);
      if (sharded) {
        hist_reduce_kernel<<<F * (kBins / 32), kReduceSlices * 32, 0, h->stream>>>(h->part_g, h->part_c, Fpad, hess_const, h->stage, job);
        if (h->allreduce(h->allreduce_ctx, h->stage, (int64_t)slot_stride, (void*)h->stream)) { coll_failed = true; break; }
      }
      reduce_scan2_kernel<<<F, kFusedSlices * kBins, 0, h->stream>>>(h->part_g, h->part_c, Fpad, F, hess_const, h->hist, (int64_t)slot_stride,
                                                                    h->num_bin, cfg.min_data_in_leaf, cfg.min_sum_hessian_in_leaf, cfg.lambda_l2,
                                                                    cfg.min_gain_to_split, h->splittable, h->cand_dev, job,
                                                                    sharded ? h->stage : nullptr);
      tree_advance_kernel<<<1, kAdvanceThreads, 0, h->stream>>>(st, h->cand_dev, F, cfg.min_gain_to_split, h->max_seg, cfg.max_depth,
                                                                cfg.min_data_in_leaf, h->num_sms, sharded ? 0 : plan_next, sharded ? 1 : 0);
      part_count_kernel<<<h->max_seg, kPartThreads, 0, h->stream>>>(h->bins, Fpad, h->idx, h->idx_tmp, h->flag8, h->seg_left, job);
      part_scatter_kernel<<<h->max_seg, kPartThreads, 0, h->stream>>>(h->idx, h->idx_tmp, h->flag8, h->seg_left, job);
      if (sharded)
        tree_local_ranges_kernel<<<1, 32, 0, h->stream>>>(st, h->seg_left, cfg.max_depth, cfg.min_data_in_leaf, h->num_sms, plan_next);
    }
  };
  auto read_back = [&](int records) {
    return cudaMemcpyAsync(h->state_host, st, sizeof(TreeDevState) + sizeof(LeafOut) * records, cudaMemcpyDeviceToHost, h->stream);
  };
  int splits = L - 1;  // enqueued
  if (graph_ok && !sharded && L - 1 <= kSplitBatch) {
    if (h->graph_exec && (h->graph_grad != grad || h->graph_hess != hess_const)) {
      cudaGraphExecDestroy(h->graph_exec);
      h->graph_exec = nullptr;
    }
    if (!h->graph_exec) {
      TCUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
      enqueue_root();
      enqueue_splits(0, L - 1);
      TCUDA(read_back(L));
      cudaGraph_t g = nullptr;
      TCUDA(cudaStreamEndCapture(h->stream, &g));
      TCUDA(cudaGetLastError());
      const cudaError_t ie = cudaGraphInstantiate(&h->graph_exec, g, 0);
      cudaGraphDestroy(g);
      if (ie != cudaSuccess) { h->graph_exec = nullptr; return tfail(std::string("gpbdev_tree_train: cudaGraphInstantiate: ") + cudaGetErrorString(ie)); }
      h->graph_grad = grad; h->graph_hess = hess_const;
    }
    TCUDA(cudaGraphLaunch(h->graph_exec, h->stream));
  } else {
    enqueue_root();
    for (splits = 0; splits < L - 1 && !coll_failed;) {
      const int end = std::min(L - 1, splits + kSplitBatch);
      enqueue_splits(splits, end);
      splits = end;
      if (coll_failed || splits == L - 1) break;
      TCUDA(cudaMemcpyAsync(&h->state_host->job.done, &st->job.done, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      TCUDA(cudaStreamSynchronize(h->stream));
      if (h->state_host->job.done) break;
    }
    if (coll_failed) return tfail("gpbdev_tree_train: device all-reduce failed");
    TCUDA(cudaGetLastError());
    TCUDA(read_back(std::min(L, splits + 1)));
  }
  h->launches += (sharded ? 5 : 4) + (int64_t)splits * (sharded ? 8 : 5);
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

int gpbdev_tree_train(gpbdev_tree_t h, const double* grad_in, int grad_on_device, double hess_const, int* num_leaves_out,
                      int* split_feature, int* threshold_bin, int* left_child, int* right_child, float* split_gain,
                      double* leaf_value, int* leaf_count) {
  if (!h || !grad_in || !num_leaves_out) return tfail("gpbdev_tree_train: null argument");
  TCUDA(cudaSetDevice(h->device));
  const double* grad = grad_in;
  if (!grad_on_device) {  // staged into the learner's buffer on every call, and enqueued eagerly
    TCUDA(cudaMemcpyAsync(h->grad, grad_in, sizeof(double) * h->n, cudaMemcpyHostToDevice, h->stream));
    grad = h->grad;
  }
  if (tree_grow(h, grad, hess_const, grad_on_device != 0)) return -1;
  const TreeDevState& r = *h->state_host;
  if (r.job.error) return tfail("gpbdev_tree_train: inconsistent split counts");
  const LeafOut* o = reinterpret_cast<const LeafOut*>(h->state_host + 1);
  const int num_leaves = r.num_leaves;
  for (int i = 0; i < num_leaves - 1; ++i) {
    split_feature[i] = o[i].split_feature; threshold_bin[i] = o[i].threshold_bin; left_child[i] = o[i].left_child;
    right_child[i] = o[i].right_child; split_gain[i] = o[i].split_gain;
  }
  h->leaf_begin.resize(num_leaves); h->leaf_cnt.resize(num_leaves); h->leaf_buf.resize(num_leaves);
  for (int i = 0; i < num_leaves; ++i) {
    leaf_value[i] = o[i].leaf_value; leaf_count[i] = o[i].leaf_count;
    h->leaf_begin[i] = o[i].leaf_begin; h->leaf_cnt[i] = o[i].leaf_cnt; h->leaf_buf[i] = o[i].leaf_buf;
  }
  h->last_num_leaves = num_leaves;
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

// bench hook: device time of the root-pass histogram kernel alone (all n rows), L2 flushed before each
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
  const int nw = hist_warps(F);
  const int64_t rpc = std::max<int64_t>(128, ((n + h->num_sms - 1) / h->num_sms + 7) / 8 * 8);
  const int nchunks = (int)((n + rpc - 1) / rpc);
  const dim3 grid(nchunks, (Fpad + 63) / 64);
  double total = 0.;
  for (int r = 0; r < reps + 1; ++r) {
    TCUDA(cudaMemsetAsync(flush, r, flush_bytes, h->stream));
    TCUDA(cudaEventRecord(e0, h->stream));
    hist3_kernel<<<grid, nw * 32, hist3_smem(nw), h->stream>>>(h->bins, Fpad, F, nullptr, 0, n, rpc, grad_dev, h->part_g, h->part_c, nullptr, nullptr);
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

int gpbdev_tree_valid_add_score(gpbdev_tree_t h, const uint8_t* bins_dev, int Fpad, int64_t nrow, int num_leaves,
                                const int32_t* split_feature_inner, const int32_t* threshold_bin, const int32_t* left_child,
                                const int32_t* right_child, const double* leaf_value, double* score_dev) {
  if (!h || !leaf_value || !score_dev) return tfail("gpbdev_tree_valid_add_score: null argument");
  if (nrow <= 0) return 0;
  TCUDA(cudaSetDevice(h->device));
  const int grid = (int)std::min<int64_t>((nrow + 255) / 256, (int64_t)h->num_sms * 16);
  if (num_leaves <= 1) {  // constant tree (Tree::AddPredictionToScore with one leaf: the leaf value on every row)
    add_const_kernel<<<grid, 256, 0, h->stream>>>(score_dev, leaf_value[0], nrow);
    TCUDA(cudaGetLastError());
    h->launches += 1;
    return 0;
  }
  if (!bins_dev || !split_feature_inner || !threshold_bin || !left_child || !right_child) return tfail("gpbdev_tree_valid_add_score: null argument");
  if (num_leaves > h->L) return tfail("gpbdev_tree_valid_add_score: the tree has more leaves than the learner's num_leaves");
  if (Fpad < h->F) return tfail("gpbdev_tree_valid_add_score: the bin matrix has fewer features than the learner");
  if (!h->vnodes_dev) TCUDA(cudaMalloc(&h->vnodes_dev, (size_t)h->L * (sizeof(int4) + sizeof(double))));
  std::vector<int4> nodes(num_leaves - 1);
  for (int i = 0; i < num_leaves - 1; ++i) {
    if (split_feature_inner[i] < 0 || split_feature_inner[i] >= h->F) return tfail("gpbdev_tree_valid_add_score: split feature out of range");
    for (int c : {left_child[i], right_child[i]})
      if (c >= 0 ? (c <= i || c >= num_leaves - 1) : (~c >= num_leaves)) return tfail("gpbdev_tree_valid_add_score: child index out of range");
    nodes[i] = make_int4(split_feature_inner[i], threshold_bin[i], left_child[i], right_child[i]);
  }
  double* leaf_dev = reinterpret_cast<double*>(h->vnodes_dev + h->L);
  TCUDA(cudaMemcpyAsync(h->vnodes_dev, nodes.data(), sizeof(int4) * (num_leaves - 1), cudaMemcpyHostToDevice, h->stream));
  TCUDA(cudaMemcpyAsync(leaf_dev, leaf_value, sizeof(double) * num_leaves, cudaMemcpyHostToDevice, h->stream));
  valid_tree_score_kernel<<<grid, 256, 0, h->stream>>>(bins_dev, Fpad, nrow, h->vnodes_dev, leaf_dev, score_dev);
  TCUDA(cudaGetLastError());
  h->launches += 1;
  TCUDA(cudaStreamSynchronize(h->stream));  // `nodes` is a temporary; the next tree reuses the node buffer
  return 0;
}

int gpbdev_metric_sums(gpbdev_tree_t h, const double* score_dev, const double* label_dev, int64_t n, const double* gp_mean_dev,
                       const double* gp_dvar_dev, double sigma2, double shift, double* out4) {
  if (!h || !score_dev || !label_dev || !out4) return tfail("gpbdev_metric_sums: null argument");
  if (n <= 0) return tfail("gpbdev_metric_sums: no rows");
  TCUDA(cudaSetDevice(h->device));
  if (!h->metric_part) TCUDA(cudaMalloc(&h->metric_part, sizeof(double) * (kMetricAcc * kMetricMaxBlocks + kMetricAcc)));
  const int nb = (int)std::min<int64_t>(kMetricMaxBlocks, (n + 4095) / 4096);
  double* res = h->metric_part + kMetricAcc * kMetricMaxBlocks;
  metric_stage1_kernel<<<nb, 256, 0, h->stream>>>(score_dev, label_dev, n, gp_mean_dev, gp_dvar_dev, sigma2, shift, h->metric_part);
  metric_stage2_kernel<<<kMetricAcc, 256, 0, h->stream>>>(h->metric_part, nb, res);
  TCUDA(cudaGetLastError());
  h->launches += 2;
  TCUDA(cudaMemcpyAsync(out4, res, sizeof(double) * kMetricAcc, cudaMemcpyDeviceToHost, h->stream));
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

int gpbdev_tree_sync(gpbdev_tree_t h) {
  if (!h) return tfail("null handle");
  TCUDA(cudaSetDevice(h->device));
  TCUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // extern "C"
