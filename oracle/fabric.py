"""Oracle transports: tagged point-to-point + all-reduce between simulated ranks.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Stands in for the reference's
`torch.distributed` gloo calls (`dist.isend/irecv` with tags at
PipeGCN/helper/feature_buffer.py:173,179 and `dist.all_reduce` at
PipeGCN/helper/reducer.py:30).  `ThreadFabric` runs a whole world inside
one process (one Python thread per rank); `GlooFabric` uses a real gloo process
group, one process per rank, like the reference's launcher
(PipeGCN/main.py:51-57).
"""
from __future__ import annotations

import queue
import threading
from collections import defaultdict

import torch


class ThreadFabric:
    def __init__(self, size: int):
        self.size = size
        self._lock = threading.Lock()
        self._boxes = defaultdict(queue.Queue)
        self._bar = threading.Barrier(size)
        self._red = {}

    def _box(self, key):
        with self._lock:
            return self._boxes[key]

    def send(self, tensor, src, dst, tag):
        self._box((src, dst, tag)).put(tensor.detach().clone())

    def recv(self, src, dst, tag, shape=None, dtype=None, timeout=600.0):
        return self._box((src, dst, tag)).get(timeout=timeout)

    def all_reduce_sum(self, rank, tensor, key):
        """In-place sum over ranks, accumulated in rank order (deterministic)."""
        if self.size == 1:
            return tensor
        with self._lock:
            self._red.setdefault(key, {})[rank] = tensor.detach().clone()
        self._bar.wait()
        parts = self._red[key]
        total = parts[0].clone()
        for r in range(1, self.size):
            total += parts[r]
        self._bar.wait()
        if rank == 0:
            with self._lock:
                del self._red[key]
        tensor.copy_(total)
        return tensor

    def barrier(self):
        if self.size > 1:
            self._bar.wait()


class GlooFabric:
    """Same interface over an initialised torch.distributed (gloo) group; `src`/`dst` are global ranks."""

    def __init__(self):
        import torch.distributed as dist
        self.dist = dist
        self.size = dist.get_world_size()
        self._pending = []

    def send(self, tensor, src, dst, tag):
        t = tensor.detach().clone().contiguous()
        self._pending = [(r, b) for r, b in self._pending if not r.is_completed()]
        self._pending.append((self.dist.isend(t, dst=dst, tag=tag), t))

    def recv(self, src, dst, tag, shape=None, dtype=torch.float32, timeout=None):
        buf = torch.empty(shape, dtype=dtype)
        self.dist.recv(buf, src=src, tag=tag)
        return buf

    def flush(self):
        for req, _ in self._pending:
            req.wait()
        self._pending.clear()

    def all_reduce_sum(self, rank, tensor, key):
        self.dist.all_reduce(tensor, op=self.dist.ReduceOp.SUM)
        return tensor

    def barrier(self):
        self.dist.barrier()
