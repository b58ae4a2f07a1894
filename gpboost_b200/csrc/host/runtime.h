// Process-wide runtime configuration of this build: which device this process drives and, when the observations are
// row-sharded over several processes (one per GPU), this process' rank. rank and world_size are set by NcclInit
// (collective.h), which also provides the all-reduces used on shard boundaries.
#ifndef GPB200_RUNTIME_H_
#define GPB200_RUNTIME_H_
namespace gpb200 {
struct Runtime {
  int device = 0;
  int rank = 0;
  int world_size = 1;
};
Runtime& GetRuntime();
// a warning through the log callback the bindings registered (LGBM_RegisterLogCallback), formatted like Log::REWarning
void LogWarning(const char* msg);
}  // namespace gpb200
#endif
