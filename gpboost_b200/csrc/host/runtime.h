// Process-wide runtime configuration of this build: which device this process drives and, when the
// observations are row-sharded over several processes (one per GPU), this process' rank and the collective used
// on shard boundaries. The collective is injected by the caller exactly like the reference lets callers inject
// theirs (LGBM_NetworkInitWithFunctions, include/LightGBM/c_api.h:1306-1317): the host frontend passes a function
// that sums a small fp64 buffer over all ranks (torch.distributed over NCCL/NVLink in bench.py, gloo in CPU tests).
#ifndef GPB200_RUNTIME_H_
#define GPB200_RUNTIME_H_
#include <cstdint>
namespace gpb200 {
typedef void (*AllReduceSumFn)(double* buf, int count);
// in-place sum-all-reduce of a DEVICE buffer, enqueued on `stream` (cudaStream_t); same type as gpbdev_allreduce_fn
typedef int (*AllReduceDevFn)(void* ctx, double* dev_buf, int64_t count, void* stream);
struct Runtime {
  int device = 0;
  int rank = 0;
  int world_size = 1;
  AllReduceSumFn allreduce_sum = nullptr;   // host buffers: injected (GPB200_SetCollective) or NCCL-backed (GPB200_NcclInit)
  AllReduceDevFn allreduce_dev = nullptr;   // device buffers: NCCL on the engines' streams (collective.h); null with an injected collective
  void* allreduce_ctx = nullptr;
};
Runtime& GetRuntime();
// a warning through the log callback the bindings registered (LGBM_RegisterLogCallback), formatted like Log::REWarning
void LogWarning(const char* msg);
}  // namespace gpb200
#endif
