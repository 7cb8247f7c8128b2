"""Peer-mapped assignment vectors for one-process-per-GPU runs (torchrun): every rank allocates its
full-length ``best[P]`` through ``rpk_ipc_alloc``, the 64-byte CUDA IPC handles travel over
``torch.distributed``, and every rank maps its peers' vectors.  The select kernel's epilogue then stores each
result into all N vectors over NVLink (``rpk_select_device_gather``) -- the all-gather is part of the
kernel, only a barrier follows it."""
from __future__ import annotations


class _RawCudaBuffer:
    """Minimal ``__cuda_array_interface__`` carrier so torch can view a raw device pointer."""

    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def as_int32_tensor(ptr: int, n: int, device):
    import torch

    return torch.as_tensor(_RawCudaBuffer(ptr, n, "<i4"), device=device)


def exchange_peer_buffer(engine, nbytes: int, rank: int, world: int):
    """-> (own device pointer, [device pointer of rank r's zero-initialised buffer for r in range(world)])."""
    import torch.distributed as dist

    own_ptr, handle = engine.ipc_alloc(nbytes)
    handles = [None] * world
    dist.all_gather_object(handles, handle)
    return own_ptr, [own_ptr if r == rank else engine.ipc_open(handles[r]) for r in range(world)]


def exchange_peer_vectors(engine, n_elems: int, rank: int, world: int, device):
    """-> (own vector as an int32 torch view, [device pointer of rank r's vector for r in range(world)])."""
    own_ptr, ptrs = exchange_peer_buffer(engine, n_elems * 4, rank, world)
    return as_int32_tensor(own_ptr, n_elems, device), ptrs


def exchange_peer_flags(engine, rank: int, world: int):
    """-> [device pointer of rank r's zero-initialised 64-word flag array for r in range(world)] (rpk_peer_fence)."""
    return exchange_peer_buffer(engine, 64 * 4, rank, world)[1]
