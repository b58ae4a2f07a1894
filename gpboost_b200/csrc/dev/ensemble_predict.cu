// Device ensemble prediction on a raw feature matrix: the sum of the leaf values (or the leaf index per tree) of every row of a dense
// host matrix, for the trees of a boosted ensemble. C ABI in include/gpboost_b200_dev.h (gpbdev_ensemble_*).
//
// Replaces the row loop of GBDT::PredictRaw / PredictLeafIndex (src/LightGBM/boosting/gbdt_prediction.cpp) over Tree::Predict /
// NumericalDecision (include/LightGBM/tree.h:329-347). The result is bitwise the host loop's: the walk compares the same doubles, and
// a row's score is s = 0; s += leaf_k in ensemble order, one fp64 add per tree (no partial sums over trees, nothing to contract).
//
// Kernel: one thread per row, a block owns a tile of rows. The tile's feature values are staged into shared memory (coalesced loads
// for both input layouts, float32 widened there) with an odd row stride, so that the data-dependent row[split_feature] reads hit
// shared memory without a systematic bank conflict. Trees are packed once into 24-byte nodes + leaf values and kept in HBM; a block
// stages them into shared memory: the whole iteration range when it fits beside the tile (then once per block, for all its tiles),
// else in chunks of consecutive trees that every thread walks before the next chunk is staged (the per-row sum lives in a register
// across chunks, so chunk boundaries do not change the add order). When ncol is too wide for a 32-row tile the features are read from
// global memory instead.
//
// Host side: the matrix arrives in pageable host memory. It is streamed in row chunks through two pinned staging buffers (parallel
// host copy -> cudaMemcpyAsync -> kernel -> result copy, one stream), so that the host copy of chunk i+1 overlaps the transfer and the
// walk of chunk i. Buffers grow to the largest call and are released with the handle.
#include "../../../include/gpboost_b200_dev.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace {

thread_local std::string g_ens_err;
int efail(const std::string& m) { g_ens_err = m; return -1; }
#define ECUDA(expr)                                                                                          \
  do {                                                                                                       \
    cudaError_t e__ = (expr);                                                                                \
    if (e__ != cudaSuccess)                                                                                  \
      return efail(std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) + ": " + cudaGetErrorString(e__)); \
  } while (0)

// children: >= 0 index into the ensemble's node array, < 0 ~(index into the ensemble's leaf array)
struct PackedNode {
  double threshold;
  int32_t left, right;
  int32_t feature;
  int32_t decision_type;  // bit 1 default-left, bits 2-3 missing type (0 None, 1 Zero, 2 NaN)
};
static_assert(sizeof(PackedNode) == 24, "PackedNode is three 8-byte words");

constexpr int kMaxTile = 256;             // rows (= threads) of the largest tile
constexpr int kMinTile = 32;
constexpr int64_t kStageBytes = 64ll << 20;  // one staging chunk of the input (and at most of the output)

// NumericalDecision (tree.h:329-347)
__device__ __forceinline__ int next_node(const PackedNode& n, double fval) {
  const double kZero = (double)1e-35f;
  const int missing = (n.decision_type >> 2) & 3;
  const bool is_nan = fval != fval;
  if (is_nan && missing != 2) fval = 0.0;
  if ((missing == 1 && fval >= -kZero && fval <= kZero) || (missing == 2 && is_nan)) return (n.decision_type & 2) ? n.left : n.right;
  return fval <= n.threshold ? n.left : n.right;
}

// stage: rows of one staging chunk. ROWMAJOR: stage[r * ncol + c]; else stage[c * ld_in + r]. blockDim.x = tile rows.
// Dynamic shared memory: [tile: blockDim.x * ld doubles when FEAT_SMEM][tree stage: leaf values, then nodes].
// tree_chunk[0 .. nchunks]: boundaries (tree indices) of the runs of consecutive trees that fit the tree stage.
template <typename T, bool ROWMAJOR, bool FEAT_SMEM>
__global__ void __launch_bounds__(kMaxTile) ensemble_predict_kernel(const T* __restrict__ stage, int64_t rows, int ncol, int64_t ld_in,
                                                                    const PackedNode* __restrict__ nodes,
                                                                    const double* __restrict__ leaf_value,
                                                                    const int32_t* __restrict__ root,
                                                                    const int32_t* __restrict__ node_offset,
                                                                    const int32_t* __restrict__ leaf_offset,
                                                                    const int32_t* __restrict__ tree_chunk, int nchunks, int first_tree,
                                                                    int count, int what, double* __restrict__ out) {
  extern __shared__ double smem[];
  const int tile_rows = blockDim.x;
  const int ld = ncol | 1;
  double* tile = smem;
  double* tstage = smem + (FEAT_SMEM ? (size_t)tile_rows * ld : 0);
  const int tid = threadIdx.x;
  bool staged = false;
  for (int64_t t0 = (int64_t)blockIdx.x * tile_rows; t0 < rows; t0 += (int64_t)gridDim.x * tile_rows) {
    const int tr = (int)min((int64_t)tile_rows, rows - t0);
    __syncthreads();  // the previous tile (and tree chunk) is no longer read
    if (FEAT_SMEM) {
      if (ROWMAJOR) {
        const T* src = stage + t0 * ncol;
        const int total = tr * ncol;
        for (int e = tid; e < total; e += tile_rows) {
          const int r = e / ncol;
          tile[r * ld + (e - r * ncol)] = (double)src[e];
        }
      } else {
        const int total = tile_rows * ncol;
        for (int e = tid; e < total; e += tile_rows) {
          const int c = e / tile_rows, r = e - c * tile_rows;
          if (r < tr) tile[r * ld + c] = (double)stage[(int64_t)c * ld_in + t0 + r];
        }
      }
    }
    const int64_t row = t0 + tid;
    const bool active = tid < tr;
    double s = 0.0;
    for (int ch = 0; ch < nchunks; ++ch) {
      const int ta = tree_chunk[ch], tb = tree_chunk[ch + 1];
      const int nbase = node_offset[ta], nn = node_offset[tb] - nbase;
      const int lbase = leaf_offset[ta], nl = leaf_offset[tb] - lbase;
      double* sleaf = tstage;
      const PackedNode* snode = reinterpret_cast<const PackedNode*>(tstage + nl);
      if (nchunks > 1 || !staged) {
        if (ch > 0) __syncthreads();  // every thread has walked the previous chunk
        for (int i = tid; i < nl; i += tile_rows) sleaf[i] = leaf_value[lbase + i];
        const unsigned long long* gsrc = reinterpret_cast<const unsigned long long*>(nodes + nbase);
        unsigned long long* sdst = reinterpret_cast<unsigned long long*>(tstage + nl);
        for (int i = tid; i < 3 * nn; i += tile_rows) sdst[i] = gsrc[i];
        staged = true;
        __syncthreads();
      } else if (ch == 0) {
        __syncthreads();  // resident ensemble: only the tile was rewritten
      }
      if (active) {
        for (int k = ta; k < tb; ++k) {
          int node = root[k];
          while (node >= 0) {
            const PackedNode n = snode[node - nbase];
            double fval;
            if (FEAT_SMEM) fval = tile[tid * ld + n.feature];
            else fval = (double)(ROWMAJOR ? stage[row * ncol + n.feature] : stage[(int64_t)n.feature * ld_in + row]);
            node = next_node(n, fval);
          }
          if (what == 0) s += sleaf[~node - lbase];
          else out[row * count + (k - first_tree)] = (double)(~node - leaf_offset[k]);
        }
      }
    }
    if (what == 0 && active) out[row] = s;
  }
}

struct Buffer {
  void* p = nullptr;
  size_t cap = 0;
};

}  // namespace

struct gpbdev_ensemble {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t done[2] = {nullptr, nullptr};
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  int num_sms = 0;
  size_t smem_block_max = 0, smem_sm = 0;
  // packed ensemble (device) and its offsets (host copy for planning)
  int num_trees = 0, max_feature = -1;
  PackedNode* nodes = nullptr;
  double* leaf_value = nullptr;
  int32_t *root = nullptr, *node_offset = nullptr, *leaf_offset = nullptr, *tree_chunk = nullptr;
  std::vector<int32_t> node_off_h, leaf_off_h;
  // staging: pinned host input / output and device input / output, two of each
  Buffer pin_in[2], pin_out[2], dev_in[2], dev_out[2];
};

namespace {

struct Plan {
  int tile_rows = kMaxTile;
  bool feat_smem = true;
  size_t smem_bytes = 0;
  std::vector<int32_t> tree_chunk;  // boundaries
  int64_t chunk_rows = 1;
};

size_t tree_bytes(const gpbdev_ensemble* h, int a, int b) {
  return (size_t)(h->node_off_h[b] - h->node_off_h[a]) * sizeof(PackedNode) + (size_t)(h->leaf_off_h[b] - h->leaf_off_h[a]) * sizeof(double);
}

int make_plan(const gpbdev_ensemble* h, int data_type, int ncol, int first, int count, int what, Plan* p) {
  const size_t total = tree_bytes(h, first, first + count);
  size_t largest = 0;
  for (int k = first; k < first + count; ++k) largest = std::max(largest, tree_bytes(h, k, k + 1));
  const size_t ld = (size_t)(ncol | 1);
  const size_t cap = h->smem_block_max;
  int tile = 0;
  for (int t = kMaxTile; t >= kMinTile && tile == 0; t >>= 1)  // the largest tile beside which the whole range stays resident
    if (t * ld * 8 + total <= cap) tile = t;
  for (int t = kMaxTile; t >= kMinTile && tile == 0; t >>= 1)  // else the largest tile that leaves half of the memory, and one tree, to the trees
    if (t * ld * 8 <= cap / 2 && t * ld * 8 + largest <= cap) tile = t;
  p->feat_smem = tile != 0;
  p->tile_rows = tile != 0 ? tile : kMaxTile;
  const size_t tile_bytes = p->feat_smem ? p->tile_rows * ld * 8 : 0;
  if (largest > cap - tile_bytes)
    return efail("gpbdev_ensemble_predict: a tree of the ensemble needs " + std::to_string(largest) + " bytes, more than the " +
                 std::to_string(cap) + " bytes of shared memory of a block");
  const size_t stage_cap = cap - tile_bytes;
  p->tree_chunk.assign(1, first);
  size_t used = 0, stage_used = 0;
  for (int k = first; k < first + count; ++k) {
    const size_t b = tree_bytes(h, k, k + 1);
    if (used + b > stage_cap) { p->tree_chunk.push_back(k); used = 0; }
    used += b;
    stage_used = std::max(stage_used, used);
  }
  p->tree_chunk.push_back(first + count);
  p->smem_bytes = tile_bytes + stage_used;
  const int64_t row_bytes = (int64_t)ncol * (data_type == 0 ? 4 : 8);
  const int64_t out_bytes = what == 0 ? 8 : (int64_t)8 * std::max(count, 1);
  p->chunk_rows = std::max<int64_t>(1, std::min(kStageBytes / row_bytes, kStageBytes / out_bytes));
  return 0;
}

template <typename T, bool RM, bool FS>
int launch_one(gpbdev_ensemble* h, const Plan& p, int nchunks, const void* stage, int64_t rows, int ncol, int64_t ld_in, int first, int count,
               int what, double* out) {
  auto kern = ensemble_predict_kernel<T, RM, FS>;
  ECUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_block_max));
  const int64_t tiles = (rows + p.tile_rows - 1) / p.tile_rows;
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(h->smem_sm / (p.smem_bytes + 1024), 2048 / p.tile_rows));
  const int grid = (int)std::min<int64_t>(tiles, (int64_t)h->num_sms * per_sm);
  kern<<<grid, p.tile_rows, p.smem_bytes, h->stream>>>(static_cast<const T*>(stage), rows, ncol, ld_in, h->nodes, h->leaf_value, h->root,
                                                        h->node_offset, h->leaf_offset, h->tree_chunk, nchunks, first, count, what, out);
  ECUDA(cudaGetLastError());
  return 0;
}

int launch(gpbdev_ensemble* h, const Plan& p, const void* stage, int data_type, int64_t rows, int ncol, int is_row_major, int first, int count,
           int what, double* out) {
  const int nchunks = (int)p.tree_chunk.size() - 1;
  const int64_t ld_in = rows;
#define GPB_ENS_CASE(T, RM, FS) return launch_one<T, RM, FS>(h, p, nchunks, stage, rows, ncol, ld_in, first, count, what, out)
  if (data_type == 0) {
    if (is_row_major) { if (p.feat_smem) GPB_ENS_CASE(float, true, true); else GPB_ENS_CASE(float, true, false); }
    else { if (p.feat_smem) GPB_ENS_CASE(float, false, true); else GPB_ENS_CASE(float, false, false); }
  } else {
    if (is_row_major) { if (p.feat_smem) GPB_ENS_CASE(double, true, true); else GPB_ENS_CASE(double, true, false); }
    else { if (p.feat_smem) GPB_ENS_CASE(double, false, true); else GPB_ENS_CASE(double, false, false); }
  }
#undef GPB_ENS_CASE
}

int ensure(Buffer* b, size_t bytes, bool pinned) {
  if (b->cap >= bytes) return 0;
  if (b->p) { if (pinned) cudaFreeHost(b->p); else cudaFree(b->p); }
  b->p = nullptr; b->cap = 0;
  ECUDA(pinned ? cudaMallocHost(&b->p, bytes) : cudaMalloc(&b->p, bytes));
  b->cap = bytes;
  return 0;
}

// rows [r0, r0 + rows) of the caller's matrix into a pinned chunk: row-major rows are contiguous, a column-major chunk is ncol strips
// (kept column-major with leading dimension `rows`)
void gather_chunk(char* dst, const char* src, size_t elem, int64_t nrow, int ncol, int is_row_major, int64_t r0, int64_t rows) {
  if (is_row_major) {
    const size_t bytes = (size_t)rows * ncol * elem, block = 1 << 20;
    const int64_t nblock = (int64_t)((bytes + block - 1) / block);
    const char* s = src + (size_t)r0 * ncol * elem;
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < nblock; ++b) std::memcpy(dst + b * block, s + b * block, std::min(block, bytes - (size_t)b * block));
  } else {
#pragma omp parallel for schedule(static)
    for (int c = 0; c < ncol; ++c) std::memcpy(dst + (size_t)c * rows * elem, src + ((size_t)c * nrow + r0) * elem, (size_t)rows * elem);
  }
}

int check_range(const gpbdev_ensemble* h, const void* data, int data_type, int64_t nrow, int ncol, int first, int count, int what, const char* who) {
  if (!h) return efail(std::string(who) + ": null handle");
  if (!data) return efail(std::string(who) + ": null argument");
  if (data_type != 0 && data_type != 1) return efail(std::string(who) + ": data_type must be 0 (float32) or 1 (float64)");
  if (nrow <= 0 || ncol <= 0) return efail(std::string(who) + ": bad shape");
  if (what != 0 && what != 1) return efail(std::string(who) + ": what must be 0 (sum of leaf values) or 1 (leaf index)");
  if (first < 0 || count < 0 || first + count > h->num_trees) return efail(std::string(who) + ": tree range outside the ensemble");
  if (h->max_feature >= ncol) return efail(std::string(who) + ": the ensemble splits on feature " + std::to_string(h->max_feature) +
                                           " but the matrix has " + std::to_string(ncol) + " columns");
  return 0;
}

void free_trees(gpbdev_ensemble* h) {
  cudaFree(h->nodes); cudaFree(h->leaf_value); cudaFree(h->root); cudaFree(h->node_offset); cudaFree(h->leaf_offset); cudaFree(h->tree_chunk);
  h->nodes = nullptr; h->leaf_value = nullptr; h->root = h->node_offset = h->leaf_offset = h->tree_chunk = nullptr;
  h->num_trees = 0; h->max_feature = -1;
  h->node_off_h.assign(1, 0); h->leaf_off_h.assign(1, 0);
}

}  // namespace

extern "C" {

const char* gpbdev_ensemble_last_error(void) { return g_ens_err.c_str(); }

int gpbdev_ensemble_create(gpbdev_ensemble_t* out, int device) {
  if (!out) return efail("gpbdev_ensemble_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device || device < 0) {
    cudaGetLastError();
    return efail("gpbdev_ensemble_create: no CUDA device " + std::to_string(device) + " — device prediction has no CPU fallback");
  }
  ECUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  ECUDA(cudaGetDeviceProperties(&prop, device));
  auto* h = new gpbdev_ensemble();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  h->smem_block_max = prop.sharedMemPerBlockOptin;
  h->smem_sm = prop.sharedMemPerMultiprocessor;
  h->node_off_h.assign(1, 0); h->leaf_off_h.assign(1, 0);
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = cudaEventCreateWithFlags(&h->done[i], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreate(&h->t0);
  if (e == cudaSuccess) e = cudaEventCreate(&h->t1);
  if (e != cudaSuccess) {
    gpbdev_ensemble_free(h);
    return efail(std::string("gpbdev_ensemble_create: ") + cudaGetErrorString(e));
  }
  *out = h;
  return 0;
}

int gpbdev_ensemble_free(gpbdev_ensemble_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  free_trees(h);
  for (int i = 0; i < 2; ++i) {
    cudaFreeHost(h->pin_in[i].p); cudaFreeHost(h->pin_out[i].p); cudaFree(h->dev_in[i].p); cudaFree(h->dev_out[i].p);
    if (h->done[i]) cudaEventDestroy(h->done[i]);
  }
  if (h->t0) cudaEventDestroy(h->t0);
  if (h->t1) cudaEventDestroy(h->t1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int gpbdev_ensemble_set_trees(gpbdev_ensemble_t h, int num_trees, const int32_t* node_offset, const int32_t* leaf_offset,
                              const int32_t* split_feature, const double* threshold, const int8_t* decision_type, const int32_t* left_child,
                              const int32_t* right_child, const double* leaf_value) {
  if (!h) return efail("gpbdev_ensemble_set_trees: null handle");
  if (num_trees < 0 || !node_offset || !leaf_offset) return efail("gpbdev_ensemble_set_trees: null argument");
  const int NN = node_offset[num_trees], NL = leaf_offset[num_trees];
  if (node_offset[0] != 0 || leaf_offset[0] != 0) return efail("gpbdev_ensemble_set_trees: offsets must start at 0");
  if ((NN > 0 && (!split_feature || !threshold || !decision_type || !left_child || !right_child)) || (NL > 0 && !leaf_value))
    return efail("gpbdev_ensemble_set_trees: null argument");
  std::vector<PackedNode> packed((size_t)NN);
  std::vector<int32_t> root((size_t)num_trees);
  int max_feature = -1;
  for (int k = 0; k < num_trees; ++k) {
    const int nb = node_offset[k], nn = node_offset[k + 1] - nb, lb = leaf_offset[k], nl = leaf_offset[k + 1] - lb;
    // a tree has nl >= 1 leaves and nl - 1 internal nodes; children of node i are leaves (~leaf in [0, nl)) or internal nodes with a
    // larger index (Tree::Split appends nodes), so every walk terminates
    if (nl < 1 || nn != nl - 1) return efail("gpbdev_ensemble_set_trees: tree " + std::to_string(k) + " needs num_leaves - 1 internal nodes");
    root[k] = nn > 0 ? nb : ~lb;
    for (int i = 0; i < nn; ++i) {
      PackedNode& n = packed[(size_t)nb + i];
      n.threshold = threshold[nb + i];
      n.feature = split_feature[nb + i];
      n.decision_type = decision_type[nb + i];
      if (n.feature < 0) return efail("gpbdev_ensemble_set_trees: split_feature out of range");
      if (n.decision_type & 1) return efail("gpbdev_ensemble_set_trees: categorical splits are not supported");
      max_feature = std::max(max_feature, n.feature);
      int32_t* dst[2] = {&n.left, &n.right};
      const int32_t src[2] = {left_child[nb + i], right_child[nb + i]};
      for (int s = 0; s < 2; ++s) {
        const int c = src[s];
        if (!(c >= 0 ? (c > i && c < nn) : (~c < nl))) return efail("gpbdev_ensemble_set_trees: child index out of range");
        *dst[s] = c >= 0 ? nb + c : ~(lb + ~c);
      }
    }
  }
  ECUDA(cudaSetDevice(h->device));
  ECUDA(cudaStreamSynchronize(h->stream));
  free_trees(h);
  cudaError_t e = cudaMalloc(&h->nodes, std::max<size_t>(1, packed.size()) * sizeof(PackedNode));
  if (e == cudaSuccess) e = cudaMalloc(&h->leaf_value, std::max<size_t>(1, (size_t)NL) * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&h->root, std::max<size_t>(1, (size_t)num_trees) * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->node_offset, ((size_t)num_trees + 1) * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->leaf_offset, ((size_t)num_trees + 1) * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->tree_chunk, ((size_t)num_trees + 2) * sizeof(int32_t));
  if (e == cudaSuccess && NN > 0) e = cudaMemcpy(h->nodes, packed.data(), packed.size() * sizeof(PackedNode), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && NL > 0) e = cudaMemcpy(h->leaf_value, leaf_value, (size_t)NL * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && num_trees > 0) e = cudaMemcpy(h->root, root.data(), (size_t)num_trees * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->node_offset, node_offset, ((size_t)num_trees + 1) * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->leaf_offset, leaf_offset, ((size_t)num_trees + 1) * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    free_trees(h);
    return efail(std::string("gpbdev_ensemble_set_trees: ") + cudaGetErrorString(e));
  }
  h->num_trees = num_trees;
  h->max_feature = max_feature;
  h->node_off_h.assign(node_offset, node_offset + num_trees + 1);
  h->leaf_off_h.assign(leaf_offset, leaf_offset + num_trees + 1);
  return 0;
}

int gpbdev_ensemble_plan(gpbdev_ensemble_t h, int data_type, int ncol, int first_tree, int num_trees, int what, int64_t* out4) {
  static const double dummy = 0.;
  if (!out4) return efail("gpbdev_ensemble_plan: null argument");
  if (int rc = check_range(h, &dummy, data_type, 1, ncol, first_tree, num_trees, what, "gpbdev_ensemble_plan")) return rc;
  Plan p;
  if (int rc = make_plan(h, data_type, ncol, first_tree, num_trees, what, &p)) return rc;
  out4[0] = p.tile_rows; out4[1] = p.chunk_rows; out4[2] = p.feat_smem ? 1 : 0; out4[3] = (int64_t)p.tree_chunk.size() - 1;
  return 0;
}

int gpbdev_ensemble_predict(gpbdev_ensemble_t h, const void* data_host, int data_type, int64_t nrow, int ncol, int is_row_major,
                            int first_tree, int num_trees, int what, double* out_host) {
  if (int rc = check_range(h, data_host, data_type, nrow, ncol, first_tree, num_trees, what, "gpbdev_ensemble_predict")) return rc;
  if (!out_host) return efail("gpbdev_ensemble_predict: null argument");
  if (num_trees == 0) {  // an empty range: the score is the empty sum, and there is no leaf index to write
    if (what == 0) std::fill(out_host, out_host + nrow, 0.0);
    return 0;
  }
  Plan p;
  if (int rc = make_plan(h, data_type, ncol, first_tree, num_trees, what, &p)) return rc;
  ECUDA(cudaSetDevice(h->device));
  const size_t elem = data_type == 0 ? 4 : 8;
  const int64_t chunk = std::min(p.chunk_rows, nrow);
  const size_t out_per_row = what == 0 ? 1 : (size_t)num_trees;
  for (int b = 0; b < 2; ++b) {
    if (b == 1 && nrow <= chunk) break;  // a single chunk needs one set of buffers
    if (int rc = ensure(&h->pin_in[b], (size_t)chunk * ncol * elem, true)) return rc;
    if (int rc = ensure(&h->dev_in[b], (size_t)chunk * ncol * elem, false)) return rc;
    if (int rc = ensure(&h->pin_out[b], (size_t)chunk * out_per_row * 8, true)) return rc;
    if (int rc = ensure(&h->dev_out[b], (size_t)chunk * out_per_row * 8, false)) return rc;
  }
  int rc = 0;
  cudaError_t e = cudaMemcpyAsync(h->tree_chunk, p.tree_chunk.data(), p.tree_chunk.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream);
  auto collect = [&](int64_t i) {  // chunk i is complete: its results leave the pinned buffer
    const int b = (int)(i & 1);
    cudaError_t ce = cudaEventSynchronize(h->done[b]);
    if (ce != cudaSuccess) return ce;
    const int64_t r0 = i * chunk, rows = std::min(chunk, nrow - r0);
    std::memcpy(out_host + (size_t)r0 * out_per_row, h->pin_out[b].p, (size_t)rows * out_per_row * 8);
    return cudaSuccess;
  };
  const int64_t nchunk = (nrow + chunk - 1) / chunk;
  int64_t collected = 0;
  for (int64_t i = 0; i < nchunk && e == cudaSuccess && rc == 0; ++i) {
    const int b = (int)(i & 1);
    if (i >= 2) { e = collect(i - 2); ++collected; if (e != cudaSuccess) break; }
    const int64_t r0 = i * chunk, rows = std::min(chunk, nrow - r0);
    gather_chunk(static_cast<char*>(h->pin_in[b].p), static_cast<const char*>(data_host), elem, nrow, ncol, is_row_major, r0, rows);
    e = cudaMemcpyAsync(h->dev_in[b].p, h->pin_in[b].p, (size_t)rows * ncol * elem, cudaMemcpyHostToDevice, h->stream);
    if (e != cudaSuccess) break;
    rc = launch(h, p, h->dev_in[b].p, data_type, rows, ncol, is_row_major, first_tree, num_trees, what, static_cast<double*>(h->dev_out[b].p));
    if (rc != 0) break;
    e = cudaMemcpyAsync(h->pin_out[b].p, h->dev_out[b].p, (size_t)rows * out_per_row * 8, cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaEventRecord(h->done[b], h->stream);
  }
  for (; collected < nchunk && e == cudaSuccess && rc == 0; ++collected) e = collect(collected);
  const cudaError_t es = cudaStreamSynchronize(h->stream);  // nothing of this call stays in flight, also after an error
  if (rc != 0) return rc;
  if (e == cudaSuccess) e = es;
  if (e != cudaSuccess) return efail(std::string("gpbdev_ensemble_predict: ") + cudaGetErrorString(e));
  return 0;
}

int gpbdev_ensemble_time_kernel(gpbdev_ensemble_t h, const void* data_host, int data_type, int64_t nrow, int ncol, int is_row_major,
                                int first_tree, int num_trees, int reps, float* mean_ms) {
  if (int rc = check_range(h, data_host, data_type, nrow, ncol, first_tree, num_trees, 0, "gpbdev_ensemble_time_kernel")) return rc;
  if (!mean_ms || reps < 1 || num_trees < 1) return efail("gpbdev_ensemble_time_kernel: bad argument");
  Plan p;
  if (int rc = make_plan(h, data_type, ncol, first_tree, num_trees, 0, &p)) return rc;
  ECUDA(cudaSetDevice(h->device));
  const size_t bytes = (size_t)nrow * ncol * (data_type == 0 ? 4 : 8);
  if (int rc = ensure(&h->dev_in[0], bytes, false)) return rc;
  if (int rc = ensure(&h->dev_out[0], (size_t)nrow * 8, false)) return rc;
  ECUDA(cudaMemcpyAsync(h->tree_chunk, p.tree_chunk.data(), p.tree_chunk.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  ECUDA(cudaMemcpyAsync(h->dev_in[0].p, data_host, bytes, cudaMemcpyHostToDevice, h->stream));
  double* out = static_cast<double*>(h->dev_out[0].p);
  if (int rc = launch(h, p, h->dev_in[0].p, data_type, nrow, ncol, is_row_major, first_tree, num_trees, 0, out)) return rc;  // warm-up
  ECUDA(cudaEventRecord(h->t0, h->stream));
  for (int r = 0; r < reps; ++r)
    if (int rc = launch(h, p, h->dev_in[0].p, data_type, nrow, ncol, is_row_major, first_tree, num_trees, 0, out)) return rc;
  ECUDA(cudaEventRecord(h->t1, h->stream));
  ECUDA(cudaStreamSynchronize(h->stream));
  float ms = 0.f;
  ECUDA(cudaEventElapsedTime(&ms, h->t0, h->t1));
  *mean_ms = ms / (float)reps;
  return 0;
}

}  // extern "C"
