"""The graph object handed to the layers: CSR + CSC of one partition on the GPU.

Takes the place of the DGL heterograph `('_U','_E','_V')` that
PipeGCN/train.py:`construct` builds (train.py:206-229) and
PipeGCN/module/layer.py:38-51 consumes; only `num_nodes('_U' | '_V')`
and the adjacency survive.
"""
from __future__ import annotations

import copy
import ctypes as C
import os
from typing import Optional

import torch

from . import _C


class CsrPlan:
    """Device CSR + the split of its long rows, packaged as a `pg_csr` for the C ABI."""

    def __init__(self, indptr: torch.Tensor, indices: torch.Tensor, seg_len: Optional[int] = None,
                 sort_rows: bool = True, row_bytes_hint: int = 512):
        assert indptr.dtype == torch.int32 and indices.dtype == torch.int32
        self.indptr, self.indices = indptr.contiguous(), indices.contiguous()
        self.n_rows = int(indptr.numel() - 1)
        self.nnz = int(indices.numel())
        dev = indptr.device
        deg = (self.indptr[1:] - self.indptr[:-1]).to(torch.int64)
        if seg_len is None:
            # segments of a few average rows: long enough to amortise the partial write,
            # short enough that the heaviest hub is spread over hundreds of warps
            mean = self.nnz / max(self.n_rows, 1)
            seg_len = int(os.environ.get("PG_SEG_LEN", 0)) or int(min(4096, max(512, 16 * mean)))
        self.seg_len = int(seg_len)
        # rows are handed to the warps by falling length: the warps of a CTA get similar amounts of work
        # (no CTA waits for one heavy row) and the heaviest rows start first
        order = torch.argsort(deg, descending=True, stable=True)
        ldeg = deg[order]
        self.row_order = order.to(torch.int32).contiguous() if (self.n_rows and sort_rows) else None
        n_long = int((ldeg > self.seg_len).sum().item()) if self.n_rows else 0
        self.long_row = order[:n_long].to(torch.int32).contiguous()        # long rows, longest first
        nseg = (ldeg[:n_long] + self.seg_len - 1) // self.seg_len
        self.long_seg_ptr = torch.zeros(n_long + 1, dtype=torch.int32, device=dev)
        if n_long:
            self.long_seg_ptr[1:] = torch.cumsum(nseg, 0).to(torch.int32)
        self.n_seg = int(self.long_seg_ptr[-1].item()) if n_long else 0
        self.seg_long = torch.repeat_interleave(torch.arange(n_long, dtype=torch.int32, device=dev), nseg) \
            if n_long else torch.zeros(0, dtype=torch.int32, device=dev)
        self.n_long = n_long
        self.max_deg = int(deg.max().item()) if self.n_rows else 0
        self._scratch = None
        self.chunks = self.pidx = self.prow = None
        self.n_chunks = self.n_chunks_long = self.n_hot = 0
        self.row_bytes_hint = int(row_bytes_hint)
        if self.n_rows and sort_rows and int(os.environ.get("PG_AGG_CHUNKS", "1")):
            self._build_chunks(order, ldeg, n_long, nseg)
        self.c = _C.pg_csr(self.indptr.data_ptr(), self.indices.data_ptr(), self.n_rows, self.seg_len, n_long,
                           self.n_seg, self.long_row.data_ptr(), self.long_seg_ptr.data_ptr(),
                           self.seg_long.data_ptr(),
                           self.row_order.data_ptr() if self.row_order is not None else None, self.nnz,
                           self.chunks.data_ptr() if self.chunks is not None else None, self.n_chunks,
                           self.n_chunks_long, self.pidx.data_ptr() if self.pidx is not None else None,
                           self.prow.data_ptr() if self.prow is not None else None)

    def _build_chunks(self, order, ldeg, n_long, nseg):
        """Permuted CSR + chunk table of the chunked aggregate kernel (include/pipegcn_b200.h: pg_csr::chunks)."""
        dev = self.indptr.device
        i64 = dict(dtype=torch.int64, device=dev)
        pptr = torch.zeros(self.n_rows + 1, **i64)
        pptr[1:] = torch.cumsum(ldeg, 0)
        if self.nnz:
            start = self.indptr.to(torch.int64)[order]
            pos = torch.repeat_interleave(start - pptr[:-1], ldeg) + torch.arange(self.nnz, **i64)
            pidx = self.indices[pos]
            # "hot" source rows: the most referenced ones, as many as fit a byte budget of about half the 50 MB L2; the
            # kernel loads them with an evict_last policy and everything else with evict_first (bit 31 of the column id).
            # The hints are off by default (agg_l2_hint) and have not been measured on H100.
            budget_rows = int(float(os.environ.get("PG_HOT_MB", "24")) * 2 ** 20) // max(self.row_bytes_hint, 1)
            refs = torch.bincount(self.indices.to(torch.int64))
            if budget_rows > 0:
                if refs.numel() > budget_rows:
                    kth = torch.topk(refs, budget_rows, sorted=True).values[-1]
                    hot = refs >= torch.clamp(kth, min=2)
                else:
                    hot = refs >= 2
                self.n_hot = int(hot.sum().item())
                flag = torch.tensor(-2 ** 31, dtype=torch.int32, device=dev)
                pidx = torch.where(hot[pidx.to(torch.int64)], pidx | flag, pidx)
            self.pidx = pidx.contiguous()
        else:
            self.pidx = torch.zeros(1, dtype=torch.int32, device=dev)
        self.prow = order.to(torch.int32).contiguous()
        parts = []
        if n_long:        # kind 2: segments of the long rows, in segment order (= scratch slot)
            seg_of = self.seg_long.to(torch.int64)
            k = torch.arange(self.n_seg, **i64) - self.long_seg_ptr.to(torch.int64)[seg_of]
            e_beg = pptr[seg_of] + k * self.seg_len
            n = torch.minimum(torch.full_like(k, self.seg_len), ldeg[seg_of] - k * self.seg_len)
            parts.append(torch.stack([e_beg, n, torch.arange(self.n_seg, **i64), torch.full_like(k, 2)], 1))
        n_mid_end = max(n_long, int((ldeg > 32).sum().item()))
        if n_mid_end > n_long:      # kind 1: one row per chunk
            it = torch.arange(n_long, n_mid_end, **i64)
            parts.append(torch.stack([pptr[it], ldeg[it], it, torch.full_like(it, 1 | (1 << 2))], 1))
        # kind 0: rows of equal length len <= 32, floor(32 / len) of them per chunk (32 empty rows per chunk)
        small = ldeg[n_mid_end:]
        if small.numel():
            cnt = torch.bincount(small, minlength=33)                  # rows per length, lengths 0..32
            a = n_mid_end
            for length in range(32, -1, -1):
                m = int(cnt[length].item())
                if m == 0:
                    continue
                per = 32 // length if length > 0 else 32
                first = a + torch.arange(0, m, per, **i64)
                rows = torch.clamp(a + m - first, max=per)
                parts.append(torch.stack([pptr[first], torch.full_like(first, length), first, rows << 2], 1))
                a += m
        self.n_chunks_long = self.n_seg + max(0, n_mid_end - n_long)
        tab = torch.cat(parts, 0) if parts else torch.zeros(0, 4, **i64)
        self.chunks = tab.to(torch.int32).contiguous()
        self.n_chunks = int(tab.shape[0])

    def scratch(self, d: int) -> Optional[torch.Tensor]:
        if self.n_seg == 0:
            return None
        need = self.n_seg * ((d + 7) // 8 * 8)
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.float32, device=self.indptr.device)
        return self._scratch


class PartGraph:
    """Bipartite `_U` -> `_V` graph of one partition (forward CSR by `_V`, backward CSC by `_U`)."""

    def __init__(self, num_in: int, num_all: int, indptr, indices, t_indptr, t_indices, in_deg,
                 device="cuda", seg_len: Optional[int] = None):
        self.num_in, self.num_all = int(num_in), int(num_all)
        dev = torch.device(device)
        self.fwd = CsrPlan(indptr.to(dev), indices.to(dev), seg_len)
        self.bwd = CsrPlan(t_indptr.to(dev), t_indices.to(dev), seg_len)
        self.in_deg = in_deg.to(dev)
        self.in_deg_f = self.in_deg.to(torch.float32).contiguous()       # `/ degs` operand (layer.py:45,50)
        self.device = dev

    @classmethod
    def from_layout(cls, lay, device="cuda", seg_len=None) -> "PartGraph":
        return cls(lay.num_in, lay.num_all, lay.indptr, lay.indices, lay.t_indptr, lay.t_indices, lay.in_deg,
                   device=device, seg_len=seg_len)

    def scratch_view(self) -> "PartGraph":
        """The same graph (shared index arrays) with scratch space of its own.  A user that runs between replays of
        CUDA graphs captured on this graph (the partitioned evaluation, whose eval branch aggregates wider rows than
        the training step) must not grow the scratch those graphs hold: growing frees the captured address."""
        view = copy.copy(self)
        for name in ("fwd", "bwd"):
            plan = copy.copy(getattr(self, name))
            plan._scratch = None
            setattr(view, name, plan)
        return view

    def deg_as_float(self, in_deg) -> torch.Tensor:
        """fp32 view of the `in_deg` argument of GraphSAGELayer.forward (cached for the graph's own tensor)."""
        if in_deg is None or in_deg is self.in_deg:
            return self.in_deg_f
        if in_deg.dtype == torch.float32 and in_deg.is_contiguous():
            return in_deg
        return in_deg.to(device=self.device, dtype=torch.float32).contiguous()

    def row_degrees(self) -> torch.Tensor:
        """`graph.in_degrees()` of the eval branch (layer.py:54): row lengths of the forward CSR."""
        if not hasattr(self, "_row_deg_f"):
            self._row_deg_f = (self.fwd.indptr[1:] - self.fwd.indptr[:-1]).to(torch.float32).contiguous()
        return self._row_deg_f

    def num_nodes(self, ntype: str = "_U") -> int:
        if ntype == "_U":
            return self.num_all
        if ntype == "_V":
            return self.num_in
        raise KeyError(ntype)

    @property
    def nnz(self) -> int:
        return self.fwd.nnz


def alloc_rows(n_rows: int, d: int, dtype, device, zero: bool = False) -> torch.Tensor:
    """[n_rows, d] view of storage whose row stride is padded to 8 elements (16-byte vectors)."""
    ld = (d + 7) // 8 * 8
    base = (torch.zeros if zero else torch.empty)(max(n_rows, 1), ld, dtype=dtype, device=device)
    return base[:n_rows, :d]
