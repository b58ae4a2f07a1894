// Native collective of the CUDA runtime: NCCL over NVLink / NVSwitch, driven from C++ on the engines' own CUDA streams.
//
// The reference's distributed learners exchange histograms and split information through LightGBM's Network layer
// (src/LightGBM/network/*, Network::Allreduce / ReduceScatter, include/LightGBM/network.h:86-170) over sockets or MPI; the
// GP part has no distributed path at all. Here one process drives one GPU; the only exchanges on the hot path are
// sum-all-reduces of device buffers (9 likelihood sums, an n-vector of Psi^-1 y, one histogram per split) and they run as
// NCCL kernels on the stream that produced the buffer — no host staging, no Python in the loop.
// NCCL is opened with dlopen at initialisation, so the library itself has no link-time dependency on it.
#ifndef GPB200_COLLECTIVE_H_
#define GPB200_COLLECTIVE_H_
#include <cstddef>
#include <cstdint>

namespace gpb200 {
constexpr int kNcclIdBytes = 128;
// fills `id` (kNcclIdBytes) on the calling rank: to be broadcast to all ranks by the launcher (torch.distributed, MPI, a file)
void NcclGetUniqueId(char* id);
// joins the communicator on the runtime's device and sets Runtime::{rank, world_size}; NcclFinalize resets them to {0, 1},
// so world_size > 1 only while a communicator is open
void NcclInit(int rank, int world_size, const char* id);
void NcclFinalize();
// in-place sum over all ranks of `count` fp64 values at device pointer `buf`, enqueued on `stream` (cudaStream_t);
// the gpbdev_allreduce_fn hook of the engines (`ctx` unused)
int NcclAllReduceSumDevice(void* ctx, double* buf, int64_t count, void* stream);
// in-place sum over all ranks of `count` fp64 values in host memory, staged through a device scratch buffer; for the handful of
// scalars the host logic itself owns (e.g. the common SLQ stopping test)
void NcclAllReduceSumHost(double* buf, int count);
// this rank's contiguous share [begin, end) of n ordered rows: chunks of ceil(n / world_size), the last ones short or empty
void RowShard(int64_t n, int64_t* begin, int64_t* end);
}  // namespace gpb200
#endif  // GPB200_COLLECTIVE_H_
