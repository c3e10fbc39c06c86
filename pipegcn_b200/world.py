"""Who the peers are and how their memory is reached.

`DistWorld`: one process per GPU under torch.distributed (the reference's process
model, PipeGCN/main.py:51-57); peers' symmetric heaps are mapped with CUDA
IPC and written over NVLink/NVSwitch from inside the exchange kernels.

`LocalWorld`: all ranks of a world live in this process on ONE GPU (peer pointers
are plain local pointers).  It runs the very same kernels and descriptors and is
what the single-GPU parity tests and `--gpus 1` multi-partition runs use.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, List

import torch

from . import _C


class _CudaMem:
    """A raw device allocation exposed to torch through __cuda_array_interface__ (zero copy)."""

    def __init__(self, ptr: int, nbytes: int, owner=None):
        self.ptr, self.nbytes, self._owner = int(ptr), int(nbytes), owner
        self.__cuda_array_interface__ = {"shape": (self.nbytes,), "typestr": "|u1", "data": (self.ptr, False),
                                         "version": 2, "strides": None}


def tensor_from_ptr(ptr: int, nbytes: int, device) -> torch.Tensor:
    mem = _CudaMem(ptr, nbytes)
    t = torch.as_tensor(mem, device=device)
    t._pg_owner = mem   # keep the descriptor alive
    return t


class Heap:
    """cudaMalloc'ed, zero-initialised region carved into aligned blocks."""

    def __init__(self, nbytes: int, device):
        self.nbytes = int(nbytes)
        self.device = torch.device(device)
        p = C.c_void_p()
        with torch.cuda.device(self.device):
            _C.check(_C.lib.pg_heap_alloc(self.nbytes, C.byref(p)), "pg_heap_alloc")
        self.ptr = int(p.value)
        self.bytes = tensor_from_ptr(self.ptr, self.nbytes, self.device)

    def view(self, offset: int, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        nb = n * torch.empty(0, dtype=dtype).element_size()
        return self.bytes[offset: offset + nb].view(dtype).view(*shape)

    def export_handle(self) -> bytes:
        buf = C.create_string_buffer(_C.IPC_HANDLE_BYTES)
        _C.check(_C.lib.pg_ipc_export(C.c_void_p(self.ptr), buf), "pg_ipc_export")
        return bytes(buf.raw)

    def free(self):
        if self.ptr:
            self.bytes = None
            _C.lib.pg_heap_free(C.c_void_p(self.ptr))
            self.ptr = 0


class LocalWorld:
    """P simulated ranks in one process on one device."""

    def __init__(self, size: int, device="cuda"):
        self.size = int(size)
        self.device = torch.device(device)
        self._pub: Dict[str, Dict[int, Any]] = {}

    def view(self, rank: int) -> "LocalRank":
        return LocalRank(self, rank)


class LocalRank:
    def __init__(self, world: LocalWorld, rank: int):
        self.world, self.rank, self.size, self.device = world, int(rank), world.size, world.device
        self.is_local = True

    def publish(self, key: str, obj):
        self.world._pub.setdefault(key, {})[self.rank] = obj

    def collect(self, key: str) -> List[Any]:
        got = self.world._pub.get(key, {})
        if len(got) != self.size:
            missing = [r for r in range(self.size) if r not in got]
            raise RuntimeError(f"LocalWorld: ranks {missing} have not published '{key}' yet "
                               f"(initialise every rank's Buffer before the first update)")
        return [got[r] for r in range(self.size)]

    def heap_token(self, heap: Heap):
        return ("ptr", heap.ptr)

    def map_peer(self, token) -> int:
        return int(token[1])

    def unmap_peer(self, token):
        pass

    def barrier(self):
        pass

    def all_reduce_sum_(self, tensor):
        raise RuntimeError("LocalWorld ranks reduce through LocalReducerGroup, not a collective")


class DistWorld:
    """This process is one rank of an initialised torch.distributed group; one GPU per process."""

    def __init__(self, device=None, group=None):
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.rank, self.size = dist.get_rank(group), dist.get_world_size(group)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.is_local = False
        self._cache: Dict[str, List[Any]] = {}
        self._mapped: Dict[bytes, int] = {}

    def publish(self, key: str, obj):
        out = [None] * self.size
        self.dist.all_gather_object(out, obj, group=self.group)
        self._cache[key] = out

    def collect(self, key: str) -> List[Any]:
        return self._cache[key]

    def heap_token(self, heap: Heap):
        return ("ipc", heap.export_handle(), self.rank, heap.ptr)

    def map_peer(self, token) -> int:
        kind, handle, owner, ptr = token
        if owner == self.rank:
            return int(ptr)
        if handle not in self._mapped:
            p = C.c_void_p()
            _C.check(_C.lib.pg_ipc_import(handle, C.byref(p)), f"pg_ipc_import(rank {owner})")
            self._mapped[handle] = int(p.value)
        return self._mapped[handle]

    def unmap_peer(self, token):
        kind, handle, owner, ptr = token
        p = self._mapped.pop(handle, None)
        if p is not None:
            _C.check(_C.lib.pg_ipc_close(C.c_void_p(p)), f"pg_ipc_close(rank {owner})")

    def barrier(self):
        torch.cuda.synchronize(self.device)
        self.dist.barrier(group=self.group)

    def all_reduce_sum_(self, tensor):
        self.dist.all_reduce(tensor, op=self.dist.ReduceOp.SUM, group=self.group)
        return tensor


def default_world():
    """World of the calling process: torch.distributed if initialised, else a single local rank."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return DistWorld()
    return LocalWorld(1).view(0)
