// See collective.h. NCCL entry points are resolved at run time (dlopen("libnccl.so.2")).
#include "collective.h"

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>

#include "runtime.h"

namespace gpb200 {
namespace {
// the part of nccl.h this file needs (NCCL 2.x ABI)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[kNcclIdBytes]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclFloat64 = 8 };  // ncclDataType_t: ncclDouble
enum { ncclSum = 0 };      // ncclRedOp_t

struct Nccl {
  void* so = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  ncclComm_t comm = nullptr;
  cudaStream_t stream = nullptr;  // for the host-buffer convenience path
  double* scratch = nullptr;
  size_t scratch_count = 0;
};
Nccl g;

void Load() {
  if (g.so) return;
  for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
    g.so = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (g.so) break;
  }
  if (!g.so) throw std::runtime_error(std::string("cannot load NCCL (libnccl.so.2): ") + dlerror());
  auto sym = [&](const char* n) {
    void* p = dlsym(g.so, n);
    if (!p) throw std::runtime_error(std::string("NCCL symbol missing: ") + n);
    return p;
  };
  g.GetUniqueId = reinterpret_cast<decltype(g.GetUniqueId)>(sym("ncclGetUniqueId"));
  g.CommInitRank = reinterpret_cast<decltype(g.CommInitRank)>(sym("ncclCommInitRank"));
  g.CommDestroy = reinterpret_cast<decltype(g.CommDestroy)>(sym("ncclCommDestroy"));
  g.AllReduce = reinterpret_cast<decltype(g.AllReduce)>(sym("ncclAllReduce"));
  g.GetErrorString = reinterpret_cast<decltype(g.GetErrorString)>(sym("ncclGetErrorString"));
}
void Check(int rc, const char* what) {
  if (rc != ncclSuccess) throw std::runtime_error(std::string(what) + ": " + (g.GetErrorString ? g.GetErrorString(rc) : "NCCL error"));
}
void CudaCheck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void NcclGetUniqueId(char* id) {
  Load();
  ncclUniqueId u;
  Check(g.GetUniqueId(&u), "ncclGetUniqueId");
  std::memcpy(id, u.internal, kNcclIdBytes);
}

void NcclInit(int rank, int world_size, const char* id) {
  if (world_size < 1 || rank < 0 || rank >= world_size) throw std::runtime_error("GPB200_NcclInit: bad rank / world_size");
  Load();
  Runtime& rt = GetRuntime();
  CudaCheck(cudaSetDevice(rt.device), "cudaSetDevice");
  if (g.comm) NcclFinalize();
  ncclUniqueId u;
  std::memcpy(u.internal, id, kNcclIdBytes);
  Check(g.CommInitRank(&g.comm, world_size, u, rank), "ncclCommInitRank");
  CudaCheck(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking), "cudaStreamCreate");
  rt.rank = rank;
  rt.world_size = world_size;
}

void NcclFinalize() {
  if (!g.comm) return;
  g.CommDestroy(g.comm);
  g.comm = nullptr;
  if (g.stream) { cudaStreamDestroy(g.stream); g.stream = nullptr; }
  if (g.scratch) { cudaFree(g.scratch); g.scratch = nullptr; g.scratch_count = 0; }
  Runtime& rt = GetRuntime();
  rt.rank = 0; rt.world_size = 1;
}

int NcclAllReduceSumDevice(void* /*ctx*/, double* buf, int64_t count, void* stream) {
  if (!g.comm) return -1;
  return g.AllReduce(buf, buf, (size_t)count, ncclFloat64, ncclSum, g.comm, reinterpret_cast<cudaStream_t>(stream)) == ncclSuccess ? 0 : -1;
}

void NcclAllReduceSumHost(double* buf, int count) {
  if ((size_t)count > g.scratch_count) {
    if (g.scratch) cudaFree(g.scratch);
    g.scratch_count = std::max<size_t>(1024, (size_t)count);
    CudaCheck(cudaMalloc(&g.scratch, sizeof(double) * g.scratch_count), "cudaMalloc");
  }
  CudaCheck(cudaMemcpyAsync(g.scratch, buf, sizeof(double) * count, cudaMemcpyHostToDevice, g.stream), "H2D");
  Check(g.AllReduce(g.scratch, g.scratch, (size_t)count, ncclFloat64, ncclSum, g.comm, g.stream), "ncclAllReduce");
  CudaCheck(cudaMemcpyAsync(buf, g.scratch, sizeof(double) * count, cudaMemcpyDeviceToHost, g.stream), "D2H");
  CudaCheck(cudaStreamSynchronize(g.stream), "sync");
}

void RowShard(int64_t n, int64_t* begin, int64_t* end) {
  const Runtime& rt = GetRuntime();
  const int64_t chunk = (n + rt.world_size - 1) / rt.world_size;
  *begin = std::min<int64_t>(n, chunk * rt.rank);
  *end = std::min<int64_t>(n, *begin + chunk);
}

}  // namespace gpb200
