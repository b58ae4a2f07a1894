"""Multi-GPU plumbing: one process per GPU (torchrun), observations row-sharded, NCCL only on shard boundaries.

The C++ runtime owns the collective: it opens its own NCCL communicator (csrc/host/collective.cpp) and all-reduces device
buffers on the engines' streams. torch.distributed only carries the communicator's 128-byte id from rank 0 to the others.
What crosses ranks per likelihood evaluation is 9 fp64 sums (SURVEY §8e)."""
import ctypes


def init_nccl(lib, dist, device_index):
    """Open the C++ runtime's NCCL communicator on `device_index` for this rank of `dist`'s process group. Call it before creating
    models or boosters: they shard their rows over the ranks when they are created."""
    import torch
    rank, world = dist.get_rank(), dist.get_world_size()
    if lib.GPB200_SetDevice(int(device_index)) != 0:
        raise RuntimeError(lib.LGBM_GetLastError().decode())
    buf = ctypes.create_string_buffer(128)
    if rank == 0 and lib.GPB200_NcclGetUniqueId(buf) != 0:
        raise RuntimeError(lib.LGBM_GetLastError().decode())
    t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
    if dist.get_backend() == "nccl":
        t = t.to(torch.device("cuda", int(device_index)))
    dist.broadcast(t, src=0)
    ident = bytes(t.cpu().numpy().tobytes())
    if lib.GPB200_NcclInit(rank, world, ctypes.c_char_p(ident)) != 0:
        raise RuntimeError(lib.LGBM_GetLastError().decode())
