"""torch-facing wrappers of the C-ABI kernels (PyTorch tensors in, PyTorch tensors out).

Each autograd Function mirrors one step of the reference's module/layer.py:44-51 and
its autograd; nothing here computes on the host or falls back to torch kernels for
the aggregate / exchange path.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch

from . import _C
from .graph import CsrPlan, PartGraph, alloc_rows


def _rows(t: torch.Tensor):
    if t.dim() != 2 or (t.shape[1] > 1 and t.stride(1) != 1):
        raise _C.PgError(f"expected a row-major 2-D tensor, got shape {tuple(t.shape)} strides {t.stride()}")
    if not t.is_cuda:
        raise _C.PgError("the hot path runs on CUDA tensors only (no CPU fall-back)")
    return t


class DropSpec:
    """Key of a dropout mask (include/pipegcn_b200.h: pg_drop): probability, 64-bit seed, device-side step counter +
    offset.  The same key evaluated by different kernels gives the same mask, so the mask is never stored."""

    def __init__(self, p: float, seed: int, step: torch.Tensor = None, step_off: int = 0):
        self.p, self.seed, self.step, self.step_off = float(p), int(seed) & 0xFFFFFFFFFFFFFFFF, step, int(step_off)

    def shifted(self, off: int) -> "DropSpec":
        return DropSpec(self.p, self.seed, self.step, self.step_off + off)

    def c(self):
        return _C.pg_drop(self.p, self.seed, self.step.data_ptr() if self.step is not None else None, self.step_off)


DROP_MUL = (0x9E3779B1, 0x85EBCA6B, 0xC2B2AE35, 0x27D4EB2F)


def dropout_keep_host(spec: DropSpec, step, row0: int, n_rows: int, d: int, elem_size: int):
    """Host port of csrc/common.cuh's drop_seed_hi / drop_base / drop_bits: numpy bool [n_rows, d], True where the mask
    of `spec` keeps element (row0 + r, c) of a tensor of d columns of `elem_size`-byte elements.  `step` is the value
    of the device counter spec.step points at, or None for a key without a counter (spec.step is None)."""
    import numpy as np
    M = 0xFFFFFFFF
    u64 = np.uint64
    thresh16 = int(np.float32(spec.p) * np.float32(65536.0) + np.float32(0.5))   # make_drop: fp32 arithmetic
    seed_lo, seed_hi = spec.seed & M, spec.seed >> 32
    key = seed_hi if step is None else (seed_hi + 0x632BE5AB * ((int(step) + spec.step_off + 1) & M)) & M
    key = int(_mix32(key))
    v = 16 // int(elem_size)
    nvec = (int(d) + v - 1) // v
    col = np.arange(d, dtype=np.uint64)
    i = (np.arange(n_rows, dtype=np.uint64)[:, None] + u64(row0)) * u64(nvec) + col[None, :] // u64(v)
    lo, hi = i & u64(M), i >> u64(32)
    base = _mix32(((lo ^ u64(seed_lo)) + ((u64(key) + hi * u64(0x9E3779B9)) & u64(M))) & u64(M))
    pair = (col % u64(v)) // u64(2)
    mul = np.asarray(DROP_MUL, dtype=np.uint64)[(pair & u64(3)).astype(np.int64)]
    h = (base * mul[None, :]) & u64(M)
    h ^= h >> u64(16)
    bits = np.where((col % u64(2)) == 0, h & u64(0xFFFF), h >> u64(16))
    return bits >= u64(thresh16)


def layer_seed(layer: int) -> int:
    """Dropout seed of graph layer `layer`: the same on every rank (all ranks seed torch identically, train.py:298)."""
    return (torch.initial_seed() * 0x9E3779B97F4A7C15 + (layer + 1) * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF


class BnsSpec:
    """Key of a boundary-node sample (include/pipegcn_b200.h: pg_bns): sampling rate p, 64-bit seed, and the epoch,
    a host value or the device counter `epoch_dev` (CUDA-graph replay)."""

    def __init__(self, p: float, seed: int, epoch: int = 0, epoch_dev: torch.Tensor = None):
        self.p, self.seed = float(p), int(seed) & 0xFFFFFFFFFFFFFFFF
        self.thresh = bns_threshold(p)
        self.epoch, self.epoch_dev = int(epoch) & 0xFFFFFFFF, epoch_dev

    def c(self):
        return _C.pg_bns(self.seed, self.thresh, self.epoch,
                         self.epoch_dev.data_ptr() if self.epoch_dev is not None else None)


def bns_threshold(p: float) -> int:
    """round(p * 2^32) as the uint32 bound of the keep test (hash < thresh); p < 1."""
    if not 0.0 < p < 1.0:
        raise ValueError(f"sampling rate {p}: the sampled path needs 0 < p < 1")
    return min(int(round(p * 2.0 ** 32)), 0xFFFFFFFF)


def bns_seed(seed: int) -> int:
    """Seed of the boundary sample from the run's --seed (the same on every rank)."""
    return (int(seed) * 0x9E3779B97F4A7C15 + 0xB5AD4ECEDA1CE2A9) & 0xFFFFFFFFFFFFFFFF


def _mix32(x):
    x = x & 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def bns_keep_host(seed: int, epoch: int, rank: int, rows, thresh: int):
    """Host port of csrc/common.cuh's bns_key / bns_keep: numpy bool array, True where rank `rank` keeps `_U` row
    `rows` in epoch `epoch`."""
    import numpy as np
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    k = _mix32(((seed >> 32) + 0x632BE5AB * ((epoch + 1) & 0xFFFFFFFF)) & 0xFFFFFFFF)
    key = _mix32((((seed & 0xFFFFFFFF) ^ k) + 0x85EBCA6B * ((rank + 1) & 0xFFFFFFFF)) & 0xFFFFFFFF)
    h = np.asarray(rows, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
    hv = _mix32((_mix32(h ^ np.uint64(key)) + np.uint64(key)) & np.uint64(0xFFFFFFFF))
    return hv < np.uint64(thresh)


def bns_sample(spec: BnsSpec, rank: int, plan: CsrPlan, num_in: int, num_all: int, mask: torch.Tensor,
               deg: torch.Tensor):
    """mask[:num_all - num_in] <- keep bytes of this rank's halo rows, deg[:num_in] <- sampled in-degrees (fp32)."""
    assert mask.dtype == torch.uint8 and deg.dtype == torch.float32 and plan.n_rows == num_in
    _C.count()
    _C.check(_C.lib.pg_bns_sample(C.byref(spec.c()), int(rank), plan.indptr.data_ptr(), plan.indices.data_ptr(),
                                  int(num_in), int(num_all), mask.data_ptr(), deg.data_ptr(), _C.stream_ptr()),
             "pg_bns_sample")


def bns_mask_rows(mask: torch.Tensor, dst: torch.Tensor, src: torch.Tensor = None):
    """dst = mask ? src : 0 row by row; without `src` only the unkept rows of dst are zeroed."""
    n, d = dst.shape
    if n == 0:
        return dst
    _C.count()
    _C.check(_C.lib.pg_bns_mask_rows(src.data_ptr() if src is not None else None, src.stride(0) if src is not None else 0,
                                     dst.data_ptr(), dst.stride(0), n, d, _C.dtype_code(dst.dtype), mask.data_ptr(),
                                     _C.stream_ptr()), "pg_bns_mask_rows")
    return dst


class QuantSpec:
    """Key of one quantised message stream (include/pipegcn_b200.h: pg_quant): bits, 64-bit run seed, graph layer and
    direction (0 = features, 1 = gradients)."""

    def __init__(self, bits: int, seed: int, layer: int = 0, direction: int = 0):
        if bits not in (8, 4):
            raise ValueError(f"halo bits {bits}: expected 8 or 4")
        self.bits, self.seed = int(bits), int(seed) & 0xFFFFFFFFFFFFFFFF
        self.layer, self.direction = int(layer), int(direction)

    def c(self):
        return _C.pg_quant(self.seed, self.bits, 2 * self.layer + self.direction)


def quant_seed(seed: int) -> int:
    """Seed of the rounding noise of quantised halo messages from the run's --seed (the same on every rank)."""
    return (int(seed) * 0x9E3779B97F4A7C15 + 0x7A3B1D5E0C9F4821) & 0xFFFFFFFFFFFFFFFF


def quant_row_bytes(d: int, bits: int) -> int:
    """Bytes of one code row: ceil(d * bits / 8) padded to 16."""
    return ((int(d) * int(bits) + 7) // 8 + 15) // 16 * 16


def quant_link_bytes(rows: int, d: int, bits, elem_size: int = 4) -> int:
    """Bytes a message of `rows` rows moves: code rows plus the (lo, scale) pairs, or rows * d * elem_size exact."""
    if bits is None:
        return int(rows) * int(d) * int(elem_size)
    return int(rows) * (quant_row_bytes(d, bits) + 8)


def quant_noise_host(seed: int, layer: int, direction: int, step: int, rank: int, rows, d: int):
    """Host port of csrc/common.cuh's quant_key / quant_row_key / quant_u: float32 [len(rows), d] noise u in [0, 1) of
    the message rows that fill receiver rows `rows` of rank `rank`, in the message whose flag value is `step`."""
    import numpy as np
    M = 0xFFFFFFFF
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    k = _mix32(((seed >> 32) + 0x27D4EB2F * ((step + 1) & M)) & M)
    k2 = _mix32((((seed & M) ^ k) + 0x165667B1 * ((rank + 1) & M)) & M)
    key = _mix32((k2 + 0xD3A2646B * ((2 * layer + direction + 1) & M)) & M)
    r = np.asarray(rows, dtype=np.uint64).reshape(-1) & np.uint64(M)
    rk = _mix32((_mix32(r ^ np.uint64(key)) + np.uint64(key)) & np.uint64(M))
    e = np.arange(d, dtype=np.uint64)
    h = _mix32((rk[:, None] + np.uint64(0x9E3779B9) * (e[None, :] + np.uint64(1))) & np.uint64(M))
    return (h >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def quantise_host(x, bits: int, seed: int, layer: int, direction: int, step: int, rank: int, row0: int):
    """Host port of pg_halo_push_q for the rows x [n, d] (float32 values) of one message filling receiver rows
    row0.. of rank `rank`: (codes uint8 [n, quant_row_bytes(d, bits)], lo float32 [n], scale float32 [n])."""
    import numpy as np
    x = np.asarray(x, dtype=np.float32)
    n, d = x.shape
    qmax = np.float32(2 ** bits - 1)
    with np.errstate(all='ignore'):
        bad = ~np.isfinite(x).all(axis=1)
        lo = x.min(axis=1) if d else np.zeros(n, np.float32)
        rng = (x.max(axis=1) - lo).astype(np.float32)
        scale = (rng / qmax).astype(np.float32)
        inv = (qmax / rng).astype(np.float32)
        bad |= ~np.isfinite(scale)
        lo = np.where(bad, np.float32(np.nan), lo).astype(np.float32)
        scale = np.where(bad, np.float32(np.nan), scale).astype(np.float32)
        coded = (scale > 0) & np.isfinite(inv)
        u = quant_noise_host(seed, layer, direction, step, rank, row0 + np.arange(n), d)
        t = np.floor(((x - lo[:, None]).astype(np.float32) * inv[:, None]).astype(np.float32) + u)
        q = np.where(coded[:, None], np.clip(t, 0, qmax), 0).astype(np.uint8)
    codes = np.zeros((n, quant_row_bytes(d, bits)), dtype=np.uint8)
    if bits == 8:
        codes[:, :d] = q
    else:
        qe = np.zeros((n, d + d % 2), dtype=np.uint8)
        qe[:, :d] = q
        codes[:, :(d + 1) // 2] = qe[:, 0::2] | (qe[:, 1::2] << 4)
    return codes, lo, scale


def dequantise_host(codes, lo, scale, bits: int, d: int):
    """Host port of the decode: float32 [n, d] = lo + q * scale (a multiply, then an add, each rounded)."""
    import numpy as np
    codes = np.asarray(codes, dtype=np.uint8)
    if bits == 8:
        q = codes[:, :d]
    else:
        b = codes[:, :(d + 1) // 2]
        q = np.stack([b & 15, b >> 4], axis=2).reshape(codes.shape[0], -1)[:, :d]
    lo = np.asarray(lo, dtype=np.float32)[:, None]
    scale = np.asarray(scale, dtype=np.float32)[:, None]
    return (lo + (q.astype(np.float32) * scale).astype(np.float32)).astype(np.float32)


def qmsg_array(entries, device) -> torch.Tensor:
    """Device array of pg_qmsg for one quantised push: `entries` = [(pairs pointer, receiving rank)] per message."""
    arr = (_C.pg_qmsg * len(entries))(*[_C.pg_qmsg(p, int(r), 0) for p, r in entries])
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device)


def halo_push_q(ms, qmsgs: torch.Tensor, src: torch.Tensor, d: int, spec: QuantSpec, value: int, value_dev=None):
    """Quantise the rows of `src` the messages of the `_MsgSet` ms name into their code rows and pairs, publish
    `value` (+ *value_dev) in their flag words (pg_halo_push_q)."""
    _C.count()
    _C.check(_C.lib.pg_halo_push_q(ms.ptr, ms.n_msgs, ms.n_ctas, qmsgs.data_ptr(), src.data_ptr(), src.stride(0), d,
                                   _C.dtype_code(src.dtype), int(value) & 0xFFFFFFFF, value_dev, C.byref(spec.c()),
                                   _C.stream_ptr()), "pg_halo_push_q")


def halo_dequant(codes: torch.Tensor, pairs: torch.Tensor, d: int, bits: int, out: torch.Tensor,
                 mirror: torch.Tensor = None, momentum: float = 0.0, drop: DropSpec = None, drop_row0: int = 0):
    """out[r, :d] = decode(codes[r], pairs[r]) (through the EMA `mirror` when given, then the dropout `drop`)."""
    n = codes.shape[0]
    if n == 0:
        return out
    _C.count()
    _C.check(_C.lib.pg_halo_dequant(codes.data_ptr(), codes.stride(0), pairs.data_ptr(), n, d, bits, out.data_ptr(),
                                    out.stride(0), _C.dtype_code(out.dtype),
                                    mirror.data_ptr() if mirror is not None else None,
                                    mirror.stride(0) if mirror is not None else 0, momentum, 1 - momentum,
                                    C.byref(drop.c()) if drop is not None and drop.p > 0 else None, int(drop_row0),
                                    _C.stream_ptr()), "pg_halo_dequant")
    return out


def boundary_add_q(grad: torch.Tensor, d: int, codes: torch.Tensor, pairs: torch.Tensor, bits: int, urow, uptr, usrc,
                   mirror: torch.Tensor = None, momentum: float = 0.0):
    """grad[urow[i], :d] += the decoded slots usrc[uptr[i]:uptr[i+1]] in that order (pg_boundary_add_q)."""
    if urow is None or urow.numel() == 0:
        return grad
    _C.count()
    _C.check(_C.lib.pg_boundary_add_q(grad.data_ptr(), grad.stride(0), d, _C.dtype_code(grad.dtype), codes.data_ptr(),
                                      codes.stride(0), pairs.data_ptr(), bits, urow.data_ptr(), uptr.data_ptr(),
                                      usrc.data_ptr(), int(urow.numel()),
                                      mirror.data_ptr() if mirror is not None else None,
                                      mirror.stride(0) if mirror is not None else 0, momentum, 1 - momentum,
                                      _C.stream_ptr()), "pg_boundary_add_q")
    return grad


def _drop_ok(t: torch.Tensor) -> bool:
    """The mask is defined on 16-byte vectors of padded, aligned rows."""
    return t.dim() == 2 and t.is_cuda and t.stride(1) == 1 and (t.stride(0) * t.element_size()) % 16 == 0 \
        and t.data_ptr() % 16 == 0 and t.stride(0) >= (t.shape[1] + 7) // 8 * 8 and t.dtype in (torch.float32, torch.bfloat16)


def dropout_rows(x: torch.Tensor, spec: DropSpec, out: torch.Tensor = None, row0: int = 0) -> torch.Tensor:
    """out = dropout(x) under the key `spec`; rows are numbered from row0 (x may be a row slice of a larger tensor)."""
    if out is None:
        out = alloc_rows(x.shape[0], x.shape[1], x.dtype, x.device)
    _C.count()
    _C.check(_C.lib.pg_dropout_rows(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), int(row0), x.shape[0],
                                    x.shape[1], _C.dtype_code(x.dtype), C.byref(spec.c()), _C.stream_ptr()),
             "pg_dropout_rows")
    return out


def aggregate(plan: CsrPlan, x: torch.Tensor, out: torch.Tensor = None, row_div: torch.Tensor = None,
              acc_rows: int = 0, drop: DropSpec = None) -> torch.Tensor:
    """out[r] = sum_{e in row r} x[indices[e]] (/ row_div[r]) (+ out[r] for r < acc_rows); with `drop` the mask of that
    key is applied to every row as it is written."""
    _rows(x)
    d = x.shape[1]
    if out is None:
        out = alloc_rows(plan.n_rows, d, x.dtype, x.device)
    _rows(out)
    assert out.shape[0] == plan.n_rows and out.shape[1] == d and out.dtype == x.dtype
    scratch = plan.scratch(d)
    prof = PROFILE
    if prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _C.count(2 if plan.n_long else 1)
    if drop is not None and drop.p > 0:
        _C.check(_C.lib.pg_aggregate_drop(C.byref(plan.c), x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), d,
                                          _C.dtype_code(x.dtype), row_div.data_ptr() if row_div is not None else None,
                                          int(acc_rows), scratch.data_ptr() if scratch is not None else None,
                                          C.byref(drop.c()), _C.stream_ptr()), "pg_aggregate_drop")
    else:
        _C.check(_C.lib.pg_aggregate(C.byref(plan.c), x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), d,
                                     _C.dtype_code(x.dtype), row_div.data_ptr() if row_div is not None else None,
                                     int(acc_rows), scratch.data_ptr() if scratch is not None else None,
                                     _C.stream_ptr()), "pg_aggregate")
    if prof is not None:
        e1.record()
        prof.append((e0, e1, aggregate_bytes(plan, x, row_div is not None)))
    return out


# when a list, every aggregate launch appends (start event, end event, algorithmic bytes)
PROFILE = None


def aggregate_bytes(plan: CsrPlan, x: torch.Tensor, has_div: bool) -> int:
    """ALGORITHMIC bytes of one launch (SURVEY.md §8d): column ids + row pointers + divisor +
    every source row once + every output row once."""
    s, d = x.element_size(), x.shape[1]
    return 4 * plan.nnz + 4 * (plan.n_rows + 1) + (4 * plan.n_rows if has_div else 0) \
        + s * d * x.shape[0] + s * d * plan.n_rows


def row_div(x: torch.Tensor, div: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    _rows(x)
    if out is None:
        out = alloc_rows(x.shape[0], x.shape[1], x.dtype, x.device)
    _C.count()
    _C.check(_C.lib.pg_row_div(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), x.shape[0], x.shape[1],
                               _C.dtype_code(x.dtype), div.data_ptr(), _C.stream_ptr()), "pg_row_div")
    return out


class SageAggregate(torch.autograd.Function):
    """ah = (A @ feat) / in_deg   (layer.py:47-50) and its gradient  g_feat = A^T @ (g_ah / in_deg)."""

    @staticmethod
    def forward(ctx, feat, graph: PartGraph, deg_f):
        ctx.graph, ctx.deg_f = graph, deg_f
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        return aggregate(graph.fwd, feat, row_div=deg_f)

    @staticmethod
    def backward(ctx, g_ah):
        graph = ctx.graph
        if g_ah.stride(1) != 1:
            g_ah = g_ah.contiguous()
        gs = row_div(g_ah, ctx.deg_f)
        return aggregate(graph.bwd, gs), None, None


def sage_aggregate(feat: torch.Tensor, graph: PartGraph, deg_f: torch.Tensor = None) -> torch.Tensor:
    return SageAggregate.apply(feat, graph, graph.in_deg_f if deg_f is None else deg_f)


# ---- dense part: hand-written wgmma GEMMs (csrc/linear_wgmma.cu, csrc/wgrad_wgmma.cu) -----------
LINEAR_IMPL = "wgmma (pg_linear / pg_wgrad: TMA + wgmma.mma_async bf16 / 3xTF32, register accumulators; dW MN-major bf16 split-K)"


def _tma_ready(t: torch.Tensor) -> torch.Tensor:
    """Row-major view whose rows start on 16-byte boundaries (what a TMA descriptor needs)."""
    if t.dim() == 2 and t.stride(1) == 1 and (t.stride(0) * t.element_size()) % 16 == 0 \
            and t.data_ptr() % 16 == 0 and t.stride(0) >= t.shape[1]:
        return t
    out = alloc_rows(t.shape[0], t.shape[1], t.dtype, t.device)
    out.copy_(t)
    return out


def padded_weight(w: torch.Tensor, dtype, transpose: bool = False) -> torch.Tensor:
    """[n, k] copy of a weight (or of its transpose) in the activation dtype with 16-byte aligned rows."""
    src = w.detach().t() if transpose else w.detach()
    out = alloc_rows(src.shape[0], src.shape[1], dtype, w.device)
    out.copy_(src)
    return out


def split_tf32(x: torch.Tensor):
    """(hi, lo) with hi = x truncated to tf32 and lo = x - hi, both padded row-major fp32 (pg_split_tf32)."""
    _rows(x)
    hi = alloc_rows(x.shape[0], x.shape[1], torch.float32, x.device)
    lo = alloc_rows(x.shape[0], x.shape[1], torch.float32, x.device)
    if x.shape[0]:
        _C.count()
        _C.check(_C.lib.pg_split_tf32(x.data_ptr(), x.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0),
                                      x.shape[0], x.shape[1], _C.stream_ptr()), "pg_split_tf32")
    return hi, lo


# fp32 activations: "3xtf32" = hi*hi + hi*lo + lo*hi on the tf32 tensor cores (fp32-grade accuracy, the
# parity mode); "tf32" = one pass (rel. error ~1e-3).  bf16 activations always use one bf16 pass.
FP32_GEMM = os.environ.get("PG_FP32_GEMM", "3xtf32")


class Split:
    """An fp32 operand together with its tf32 (hi, lo) halves, so that one split serves every product that uses the
    operand (a gradient feeds two dX GEMMs and two weight-gradient GEMMs)."""

    def __init__(self, x: torch.Tensor):
        self.x = _rows(x)
        self.hi, self.lo = split_tf32(x)

    def rows(self, lo: int, hi: int = None) -> "Split":
        out = Split.__new__(Split)
        out.x, out.hi, out.lo = self.x[lo:hi], self.hi[lo:hi], self.lo[lo:hi]
        return out


def presplit(x: torch.Tensor):
    """`Split(x)` when x is an fp32 operand of the 3xTF32 product, else x itself."""
    if isinstance(x, torch.Tensor) and x.dtype == torch.float32 and FP32_GEMM == "3xtf32":
        return Split(x)
    return x


def _plain(t):
    return t.x if isinstance(t, Split) else t


def _halves(t):
    return (t.hi, t.lo) if isinstance(t, Split) else split_tf32(t)


def gemm_nt(a0, b0, a1=None, b1=None, bias=None, row_div=None, out=None, out_dtype=None, drop=None,
            drop_row0: int = 0) -> torch.Tensor:
    """out[m, n] = a0 @ b0^T (+ a1 @ b1^T) (+ bias) (/ row_div[:, None]) on the tensor cores.  Operands may be
    `Split` objects (fp32 operands split once by the caller).  `drop`: dropout mask applied to `out` as it is written
    (out's first row is row `drop_row0` of the tensor the mask is defined on)."""
    a, b = ([a0, a1], [b0, b1]) if a1 is not None else ([a0], [b0])
    return _gemm(a, [dict(b=b, bias=bias, row_div=row_div, out=out, drop=drop, drop_row0=drop_row0)], out_dtype)[0]


def gemm_nt_group(a, bs, row_divs=None, outs=None, out_dtype=None) -> list:
    """[a @ b^T (/ row_div[:, None]) for b in bs] (at most four products of the same width) in ONE launch: the
    products share their A operand, and the CTAs that multiply the same rows of it run together, so `a` is read from
    HBM once for all of them.  Each output has the bits of its own `gemm_nt` call."""
    row_divs = row_divs or [None] * len(bs)
    outs = outs or [None] * len(bs)
    return _gemm([a], [dict(b=[b], bias=None, row_div=r, out=o, drop=None, drop_row0=0)
                       for b, r, o in zip(bs, row_divs, outs)], out_dtype)


def _gemm(raw_a, probs, out_dtype):
    """pg_linear_group: every problem (dict of b, bias, row_div, out, drop, drop_row0) multiplies the A operands
    `raw_a` by its own B operands."""
    a0 = _plain(raw_a[0])
    m, n = a0.shape[0], _plain(probs[0]["b"][0]).shape[0]
    for pr in probs:
        for a, b in zip(raw_a, pr["b"]):
            a, b = _rows(_plain(a)), _rows(_plain(b))
            assert a.shape[0] == m and b.shape[0] == n and a.shape[1] == b.shape[1] and a.dtype == b.dtype == a0.dtype
    outs = []
    for pr in probs:
        out = pr["out"]
        if out is None:
            out = alloc_rows(m, n, out_dtype or a0.dtype, a0.device)
        assert out.shape == (m, n) and out.stride(1) == 1 and out.dtype == (outs[0].dtype if outs else out.dtype)
        outs.append(out)
    if n > 256:
        # one N tile holds at most 256 columns: split the weight rows, each product writing its 256-column slice of
        # one output (padded rows like every other output: 16-byte aligned, usable by the row kernels and TMA)
        assert all(pr["drop"] is None or pr["drop"].p == 0 for pr in probs), "fused dropout with n > 256 is not supported"
        for i in range(0, n, 256):
            _gemm(raw_a, [dict(pr, b=[_plain(b)[i:i + 256] for b in pr["b"]], out=out[:, i:i + 256], drop=None,
                               bias=None if pr["bias"] is None else pr["bias"][i:i + 256])
                          for pr, out in zip(probs, outs)], out_dtype)
        return outs
    if m == 0:
        return outs
    if a0.dtype == torch.float32 and FP32_GEMM == "3xtf32":
        a_halves = [_halves(a) for a in raw_a]
        pairs = []
        for pr in probs:
            for (ah, al), b in zip(a_halves, pr["b"]):
                bh, bl = _halves(b)
                pairs += [(ah, bh), (ah, bl), (al, bh)]
    else:
        a_ready = [_tma_ready(_rows(_plain(a))) for a in raw_a]
        pairs = [(a, _tma_ready(_rows(_plain(b)))) for pr in probs for a, b in zip(a_ready, pr["b"])]
    srcs = (_C.pg_gemm_src * len(pairs))(*[_C.pg_gemm_src(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                                                            a.shape[1]) for a, b in pairs])
    keep, couts = [], []
    for pr, out in zip(probs, outs):
        bias, drop = pr["bias"], pr["drop"]
        if bias is not None:
            bias = bias.detach().to(torch.float32).contiguous()
            keep.append(bias)
        dc = None
        if drop is not None and drop.p > 0:
            dc = drop.c()
            keep.append(dc)
        couts.append(_C.pg_gemm_out(bias.data_ptr() if bias is not None else None,
                                    pr["row_div"].data_ptr() if pr["row_div"] is not None else None,
                                    out.data_ptr(), out.stride(0), C.addressof(dc) if dc is not None else None,
                                    int(pr["drop_row0"])))
    _C.count()
    _C.check(_C.lib.pg_linear_group(_C.dtype_code(a0.dtype), _C.dtype_code(outs[0].dtype), srcs,
                                    len(pairs) // len(probs), len(probs), (_C.pg_gemm_out * len(couts))(*couts), m, n,
                                    _C.stream_ptr()), "pg_linear_group")
    return outs


def _split_bf16(x: torch.Tensor, terms: int):
    """x = b0 + b1 + ... in bf16 (three terms carry every bit of an fp32 value)."""
    out, r = [], x.float()
    for _ in range(terms):
        b = alloc_rows(x.shape[0], x.shape[1], torch.bfloat16, x.device)
        b.copy_(r)
        out.append(b)
        r = r - b.float()
    return out



def wgrad(g: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """g^T @ x  -> fp32 [n, k]: the weight gradient of `x @ W^T` on the tensor cores (pg_wgrad: MN-major bf16
    operands straight from the row-major activations, split-K over the rows, fixed-order reduction).  The tensor core
    transposes 16-bit operands only, so fp32 activations go in as sums of bf16 terms."""
    return wgrad_group([(g, x)])[0]


def wgrad_group(pairs) -> list:
    """[g^T @ x for g, x in pairs] (one or two products of the same n and k; the rows may differ) with the products
    in ONE launch per 256 x 256 block of the output (pg_wgrad_group): the CTAs of both products over the same rows run
    together, so an operand they share is read from HBM once.  Each output has the bits of its own `wgrad` call."""
    assert 1 <= len(pairs) <= 2
    ps = [(_rows(_plain(g)), _rows(_plain(x))) for g, x in pairs]
    n, k, dt = ps[0][0].shape[1], ps[0][1].shape[1], ps[0][0].dtype
    for g, x in ps:
        assert x.shape[0] == g.shape[0] and g.shape[1] == n and x.shape[1] == k and g.dtype == x.dtype == dt
    outs = [torch.empty(n, k, dtype=torch.float32, device=g.device) for g, _ in ps]
    live = []
    for out, (g, x) in zip(outs, ps):
        if g.shape[0] == 0:
            out.zero_()
        else:
            live.append((out, g, x))
    if not live:
        return outs
    terms = {}

    def split(t, n_terms):      # one split of an operand the products share
        key = (t.data_ptr(), tuple(t.shape), t.stride(0))
        if key not in terms:
            terms[key] = _split_bf16(t, n_terms)
        return terms[key]

    prob_pairs = []
    for _, g, x in live:
        if dt == torch.float32 and FP32_GEMM == "3xtf32":
            # fp32 = b0 + b1 + b2 exactly (three bf16 terms): six bf16 products carry the product to ~2^-24
            g3, x3 = split(g, 3), split(x, 3)
            prob_pairs.append([(g3[0], x3[0]), (g3[0], x3[1]), (g3[1], x3[0]), (g3[0], x3[2]), (g3[2], x3[0]),
                               (g3[1], x3[1])])
        elif dt == torch.float32:
            # one-pass mode: two bf16 terms, three products (~2^-16, finer than one tf32 pass)
            g2, x2 = split(g, 2), split(x, 2)
            prob_pairs.append([(g2[0], x2[0]), (g2[0], x2[1]), (g2[1], x2[0])])
        else:
            prob_pairs.append([(_tma_ready(g), _tma_ready(x))])
    code = _C.dtype_code(prob_pairs[0][0][0].dtype)
    es = prob_pairs[0][0][0].element_size()
    n_src = len(prob_pairs[0])
    for n0 in range(0, n, 256):
        for k0 in range(0, k, 256):
            nn, kk = min(256, n - n0), min(256, k - k0)
            srcs = (_C.pg_gemm_src * (n_src * len(live)))(*[
                _C.pg_gemm_src(a.data_ptr() + n0 * es, a.stride(0), b.data_ptr() + k0 * es, b.stride(0), a.shape[0])
                for pp in prob_pairs for a, b in pp])
            wss, couts = [], []
            for out, g, _ in live:
                m = g.shape[0]
                # split-K partials: a fresh block per call (the caching allocator is stream-aware; several simulated
                # ranks run on their own streams in one process and must not share scratch)
                ws = torch.empty(int(_C.lib.pg_wgrad_workspace(m, nn, kk, code)), dtype=torch.float32, device=g.device)
                wss.append(ws)
                o = out[n0:n0 + nn, k0:k0 + kk]
                couts.append(_C.pg_wgrad_out(o.data_ptr(), o.stride(0), m, ws.data_ptr(), ws.numel()))
            _C.count(2)
            _C.check(_C.lib.pg_wgrad_group(code, srcs, n_src, len(live), (_C.pg_wgrad_out * len(couts))(*couts), nn,
                                           kk, _C.stream_ptr()), "pg_wgrad_group")
    return outs


class _Linear(torch.autograd.Function):
    """y = x @ W^T + b   (plain `nn.Linear` layers: use_pp layer 0 and the trailing n_linear layers)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        wp = padded_weight(weight, x.dtype)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return gemm_nt(x, wp, bias=bias)

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == x.dtype else g.to(x.dtype))
        gsp = presplit(g)
        gx = gemm_nt(gsp, padded_weight(weight, x.dtype, transpose=True)) if ctx.needs_input_grad[0] else None
        gw = wgrad(gsp, x).to(weight.dtype)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        return gx, gw, gb


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor = None) -> torch.Tensor:
    return _Linear.apply(x, weight, bias)


class SageLayerFn(torch.autograd.Function):
    """The whole training branch of GraphSAGELayer.forward (layer.py:44-51) and its gradient:

        ah  = (A @ feat) / in_deg                         pg_aggregate
        out = feat[:N_in] @ W1^T + ah @ W2^T + (b1 + b2)  pg_linear, two sources, one kernel

        g_feat[:N_in] = g @ W1                            pg_linear_group: one launch for both, g read once,
        gs            = (g @ W2) / in_deg                 the row scale fused into the second product
        g_feat       += A^T @ gs                          pg_aggregate accumulating into rows < N_in
        gW1 = g^T feat[:N_in], gW2 = g^T ah               pg_wgrad_group: one launch for both, g read once
        gb = sum g                                        column sums of the LayerNorm backward
    """

    @staticmethod
    def forward(ctx, feat, graph, deg_f, w1, b1, w2, b2, drop_bwd=None):
        # drop_bwd: `feat` already IS dropout(F) (written that way by its producers); the gradient returned is the one
        # with respect to F, i.e. the dropout backward is applied to g_feat as the transposed aggregate writes it
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        ah = aggregate(graph.fwd, feat, row_div=deg_f)
        x = feat[:n_in]
        bias = None
        if b1 is not None:
            bias = b1.detach().float() + b2.detach().float()
        out = gemm_nt(x, padded_weight(w1, feat.dtype), ah, padded_weight(w2, feat.dtype), bias=bias)
        ctx.graph, ctx.deg_f = graph, deg_f
        ctx.has_bias = b1 is not None
        ctx.save_for_backward(x, ah, w1, w2)
        ctx.num_all = feat.shape[0]
        return out

    @staticmethod
    def backward(ctx, g):
        x, ah, w1, w2 = ctx.saved_tensors
        graph, deg_f = ctx.graph, ctx.deg_f
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == x.dtype else g.to(x.dtype))
        gsp = presplit(g)                      # fp32: one split of g serves the two dX and the two dW products
        g_feat = None
        if ctx.needs_input_grad[0]:
            d_in = x.shape[1]
            g_feat = alloc_rows(ctx.num_all, d_in, x.dtype, x.device)
            _, gs = gemm_nt_group(gsp, [padded_weight(w1, x.dtype, transpose=True),
                                        padded_weight(w2, x.dtype, transpose=True)],
                                  row_divs=[None, deg_f], outs=[g_feat[:graph.num_in], None])
            aggregate(graph.bwd, gs, out=g_feat, acc_rows=graph.num_in, drop=ctx.drop_bwd)
        gw1, gw2 = wgrad_group([(gsp, x), (gsp, ah)])
        gw1, gw2 = gw1.to(w1.dtype), gw2.to(w2.dtype)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        return g_feat, None, None, gw1, gb, gw2, gb, None


class SageLayerNarrowFn(torch.autograd.Function):
    """The same function as `SageLayerFn`, evaluated TRANSFORM-FIRST when the layer narrows (d_out < d_in):

        z   = feat @ W2^T                          [num_all, d_out]   pg_linear over all rows (inner + halo)
        out = feat[:N_in] @ W1^T + (b1 + b2)       [N_in, d_out]      pg_linear
        out += (A @ z) / in_deg                                       pg_aggregate, accumulating, division fused

    (A F) W = A (F W): the aggregate -- the HBM/L2-bound part of PipeGCN/module/layer.py:47-51 -- moves
    d_out-wide rows instead of d_in-wide ones (4x fewer bytes for the 256 -> 64 output layer of the headline config).
    Backward: dz = A^T (g / in_deg) [num_all, d_out], g_feat = dz @ W2 (+ g @ W1 on the inner rows),
    gW2 = dz^T feat, gW1 = g^T feat[:N_in].  Same sums, different association: fp32 results agree with the
    aggregate-first form to rounding (parity tests compare against the oracle, which aggregates first).
    """

    @staticmethod
    def forward(ctx, feat, graph, deg_f, w1, b1, w2, b2, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        fsp = presplit(feat)                   # fp32: one split of feat for both products
        bias = None
        if b1 is not None:
            bias = b1.detach().float() + b2.detach().float()
        na, nb = w2.shape[0], w1.shape[0]
        v = 16 // feat.element_size()
        na_pad = -(-na // v) * v
        if MERGE_NARROW and na_pad + nb <= 256:
            # ONE product reads feat once: [z | self part] = feat @ [W2 ; W1]^T (+ [0 | b1 + b2]); the self part of
            # the halo rows is computed and never read.  W1 starts at a 16-byte aligned column.
            wc = alloc_rows(na_pad + nb, feat.shape[1], feat.dtype, feat.device)
            if na_pad != na:
                wc[na:na_pad].zero_()
            wc[:na].copy_(w2.detach())
            wc[na_pad:].copy_(w1.detach())
            bias_c = None
            if bias is not None:
                bias_c = torch.zeros(na_pad + nb, dtype=torch.float32, device=feat.device)
                bias_c[na_pad:].copy_(bias)
            zc = gemm_nt(fsp, wc, bias=bias_c)
            z, out = zc[:, :na], zc[:n_in, na_pad:]
        else:
            z = gemm_nt(fsp, padded_weight(w2, feat.dtype))
            out = gemm_nt(fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in], padded_weight(w1, feat.dtype),
                          bias=bias)
        aggregate(graph.fwd, z, out=out, row_div=deg_f, acc_rows=n_in)
        ctx.graph, ctx.deg_f = graph, deg_f
        ctx.has_bias = b1 is not None
        ctx.save_for_backward(feat, w1, w2)
        return out

    @staticmethod
    def backward(ctx, g):
        feat, w1, w2 = ctx.saved_tensors
        graph, deg_f = ctx.graph, ctx.deg_f
        n_in = graph.num_in
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        gs = row_div(g, deg_f)
        dz = aggregate(graph.bwd, gs)                                   # [num_all, d_out]
        gsp, dzsp, fsp = presplit(g), presplit(dz), presplit(feat)
        is_split = isinstance(fsp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(feat.shape[0], feat.shape[1], feat.dtype, feat.device)
            w1t, w2t = padded_weight(w1, feat.dtype, transpose=True), padded_weight(w2, feat.dtype, transpose=True)
            db = ctx.drop_bwd if (ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 and feat.shape[1] <= 256
                                  and _drop_ok(g_feat)) else None   # dropout backward in the GEMM's epilogue
            gemm_nt(dzsp.rows(0, n_in) if is_split else dz[:n_in], w2t, gsp, w1t, out=g_feat[:n_in], drop=db)
            if feat.shape[0] > n_in:
                gemm_nt(dzsp.rows(n_in) if is_split else dz[n_in:], w2t, out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if db is None and ctx.drop_bwd is not None and ctx.drop_bwd.p > 0:
                dropout_rows(g_feat, ctx.drop_bwd, out=g_feat)
        # one launch for both: feat is read from HBM once
        gw1, gw2 = wgrad_group([(gsp, fsp.rows(0, n_in) if is_split else feat[:n_in]), (dzsp, fsp)])
        gw1, gw2 = gw1.to(w1.dtype), gw2.to(w2.dtype)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        return g_feat, None, None, gw1, gb, gw2, gb, None


# transform-first when the layer narrows (PG_NARROW=0 keeps the reference's aggregate-first association everywhere)
NARROW = os.environ.get("PG_NARROW", "1") != "0"
# ... with the neighbour and self products of its forward in one GEMM (PG_MERGE_NARROW=0: two GEMMs)
MERGE_NARROW = os.environ.get("PG_MERGE_NARROW", "1") != "0"


def sage_layer(feat, graph, deg_f, w1, b1, w2, b2, drop_bwd=None) -> torch.Tensor:
    if NARROW and w1.shape[0] < feat.shape[1]:
        return SageLayerNarrowFn.apply(feat, graph, deg_f, w1, b1, w2, b2, drop_bwd)
    return SageLayerFn.apply(feat, graph, deg_f, w1, b1, w2, b2, drop_bwd)


def sage_linear(x, ah, w1, b1, w2, b2) -> torch.Tensor:
    """x @ W1^T + b1 + ah @ W2^T + b2   (layer.py:51) -- un-fused composition (eval branch)."""
    return linear(x, w1, b1) + linear(ah, w2, b2)


# ---- graph convolution (GraphConv, norm='both'): the scaled aggregate of csrc/aggregate.cu --------------------------
def sym_norm(deg: torch.Tensor) -> torch.Tensor:
    """c = clamp(deg, min=1)^(-1/2) in fp32 as 1 / sqrt(deg): two correctly rounded operations, so every device and
    the host give the same bits."""
    d = torch.clamp(deg.to(torch.float32), min=1.0)
    return torch.div(1.0, torch.sqrt(d)).contiguous()


def graphconv_preload():
    """Load every scaled-aggregate kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_aggregate_scaled_preload(), "pg_aggregate_scaled_preload")


def aggregate_scaled(plan: CsrPlan, x: torch.Tensor, src: torch.Tensor, dst: torch.Tensor, bias: torch.Tensor = None,
                     drop: DropSpec = None, out: torch.Tensor = None) -> torch.Tensor:
    """out[r] = dst[r] * sum_{e in row r} src[indices[e]] * x[indices[e]] (+ bias); with `drop` the mask of that key is
    applied to every row as it is written (pg_aggregate_scaled)."""
    _rows(x)
    d = x.shape[1]
    if out is None:
        out = alloc_rows(plan.n_rows, d, x.dtype, x.device)
    _rows(out)
    assert out.shape[0] == plan.n_rows and out.shape[1] == d and out.dtype == x.dtype
    assert src.dtype == dst.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous()
    assert src.numel() >= x.shape[0] and dst.numel() >= plan.n_rows
    if bias is not None:
        bias = bias.detach()
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == d and bias.is_cuda
    scratch = plan.scratch(d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_aggregate_scaled(C.byref(plan.c), x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), d,
                                        _C.dtype_code(x.dtype), src.data_ptr(), dst.data_ptr(),
                                        bias.data_ptr() if bias is not None else None,
                                        scratch.data_ptr() if scratch is not None else None,
                                        C.byref(drop.c()) if drop is not None and drop.p > 0 else None,
                                        _C.stream_ptr()), "pg_aggregate_scaled")
    return out


def _graphconv_wgrad(g, x, weight):
    """dW [in, out] of `x @ W` from wgrad's [out, in]."""
    return wgrad(g, x).t().contiguous().to(weight.dtype)


class GraphConvLayerFn(torch.autograd.Function):
    """GraphConv (norm='both') aggregating first, d_in <= d_out; c = deg^-1/2 over the [inner | halo] rows:

        ah  = c[:N_in] * (A @ (c * feat))           pg_aggregate_scaled over the CSR
        out = ah @ W + b                            pg_linear

        g_ah = g @ W^T                              pg_linear
        g_feat = c * (A^T @ (c[:N_in] * g_ah))      pg_aggregate_scaled over the CSC, dropout backward in its store
        gW = ah^T g, gb = sum g
    """

    @staticmethod
    def forward(ctx, feat, graph, c, weight, bias, drop_bwd=None):
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        ah = aggregate_scaled(graph.fwd, feat, c, c[:n_in])
        out = gemm_nt(ah, padded_weight(weight, feat.dtype, transpose=True), bias=bias)
        ctx.graph, ctx.c, ctx.drop_bwd = graph, c, drop_bwd
        ctx.has_bias = bias is not None
        ctx.save_for_backward(ah, weight)
        return out

    @staticmethod
    def backward(ctx, g):
        ah, weight = ctx.saved_tensors
        graph, c = ctx.graph, ctx.c
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == ah.dtype else g.to(ah.dtype))
        gsp = presplit(g)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_ah = gemm_nt(gsp, padded_weight(weight, ah.dtype))
            g_feat = aggregate_scaled(graph.bwd, g_ah, c, c, drop=ctx.drop_bwd)
        gw = _graphconv_wgrad(gsp, ah, weight)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        return g_feat, None, None, gw, gb, None


class GraphConvLayerNarrowFn(torch.autograd.Function):
    """The same function transform-first when the layer narrows (d_out < d_in), as `SageLayerNarrowFn`:

        z   = feat @ W                              [num_all, d_out]   pg_linear over the inner and halo rows
        out = c[:N_in] * (A @ (c * z)) + b                             pg_aggregate_scaled, bias in its store

        dz = c * (A^T @ (c[:N_in] * g))            [num_all, d_out]   pg_aggregate_scaled over the CSC
        g_feat = dz @ W^T                                              pg_linear, dropout backward in its epilogue
        gW = feat^T dz, gb = sum g
    """

    @staticmethod
    def forward(ctx, feat, graph, c, weight, bias, drop_bwd=None):
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        z = gemm_nt(feat, padded_weight(weight, feat.dtype, transpose=True))
        out = aggregate_scaled(graph.fwd, z, c, c[:graph.num_in], bias=bias)
        ctx.graph, ctx.c, ctx.drop_bwd = graph, c, drop_bwd
        ctx.has_bias = bias is not None
        ctx.save_for_backward(feat, weight)
        return out

    @staticmethod
    def backward(ctx, g):
        feat, weight = ctx.saved_tensors
        graph, c = ctx.graph, ctx.c
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        dz = aggregate_scaled(graph.bwd, g, c, c)                       # [num_all, d_out]
        dzsp = presplit(dz)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(feat.shape[0], feat.shape[1], feat.dtype, feat.device)
            db = ctx.drop_bwd if (ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 and feat.shape[1] <= 256
                                  and _drop_ok(g_feat)) else None   # dropout backward in the GEMM's epilogue
            gemm_nt(dzsp, padded_weight(weight, feat.dtype), out=g_feat, drop=db)
            if db is None and ctx.drop_bwd is not None and ctx.drop_bwd.p > 0:
                dropout_rows(g_feat, ctx.drop_bwd, out=g_feat)
        gw = _graphconv_wgrad(dzsp, feat, weight)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        return g_feat, None, None, gw, gb, None


def graphconv_layer(feat, graph, c, weight, bias, drop_bwd=None) -> torch.Tensor:
    """GraphConv(norm='both') over the [num_all, d_in] rows `feat` of `graph` with the norm vector c [num_all];
    weight [d_in, d_out] (DGL's layout), bias [d_out] or None.  Returns the [N_in, d_out] inner rows."""
    if NARROW and weight.shape[1] < feat.shape[1]:
        return GraphConvLayerNarrowFn.apply(feat, graph, c, weight, bias, drop_bwd)
    return GraphConvLayerFn.apply(feat, graph, c, weight, bias, drop_bwd)


# ---- GCNII (--model gcnii): the residual aggregate of csrc/aggregate.cu and the row kernels of csrc/gcnii.cu ------
def gcnii_preload():
    """Load every residual-aggregate kernel (and the column sum of fc_in's bias gradient) now (see gat_preload)."""
    _C.check(_C.lib.pg_aggregate_scaled_res_preload(), "pg_aggregate_scaled_res_preload")
    graphconv_preload()
    gat_preload()


def gcnii_beta(lam: float, layer: int) -> float:
    """beta_l = ln(lambda / l + 1) of convolution l (1-based)."""
    import math
    return math.log(lam / layer + 1.0)


def gcnii_h0_seed() -> int:
    """Dropout seed of h0 on its way into the first convolution (distinct from every layer_seed)."""
    return (layer_seed(0) * 0x9E3779B97F4A7C15 + 0x5851F42D4C957F2D) & 0xFFFFFFFFFFFFFFFF


def aggregate_scaled_res(plan: CsrPlan, x: torch.Tensor, src: torch.Tensor, dst: torch.Tensor,
                         res: torch.Tensor = None, alpha: float = 0.0, bias: torch.Tensor = None,
                         drop: DropSpec = None, out: torch.Tensor = None) -> torch.Tensor:
    """out[r] = dst[r] * sum_{e in row r} src[indices[e]] * x[indices[e]] + alpha * res[r] (+ bias), one rounding
    (pg_aggregate_scaled_res); res None is `aggregate_scaled`."""
    _rows(x)
    d = x.shape[1]
    if out is None:
        out = alloc_rows(plan.n_rows, d, x.dtype, x.device)
    _rows(out)
    assert out.shape[0] == plan.n_rows and out.shape[1] == d and out.dtype == x.dtype
    assert src.dtype == dst.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous()
    assert src.numel() >= x.shape[0] and dst.numel() >= plan.n_rows
    if res is not None:
        _rows(res)
        assert res.shape[0] >= plan.n_rows and res.shape[1] == d and res.dtype == x.dtype
    if bias is not None:
        bias = bias.detach()
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == d and bias.is_cuda
    scratch = plan.scratch(d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_aggregate_scaled_res(C.byref(plan.c), x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0),
                                            d, _C.dtype_code(x.dtype), src.data_ptr(), dst.data_ptr(),
                                            res.data_ptr() if res is not None else None,
                                            res.stride(0) if res is not None else 0, float(alpha),
                                            bias.data_ptr() if bias is not None else None,
                                            scratch.data_ptr() if scratch is not None else None,
                                            C.byref(drop.c()) if drop is not None and drop.p > 0 else None,
                                            _C.stream_ptr()), "pg_aggregate_scaled_res")
    return out


def gcnii_relu_drop(z: torch.Tensor, drop: DropSpec = None):
    """(h0, hd): h0 = ReLU(z) and hd = dropout(h0) under the key `drop` in one pass (pg_gcnii_relu_drop); without a
    dropout hd is h0."""
    _rows(z)
    n, d = z.shape
    h0 = alloc_rows(n, d, z.dtype, z.device)
    hd = alloc_rows(n, d, z.dtype, z.device) if drop is not None and drop.p > 0 else None
    _C.count()
    _C.check(_C.lib.pg_gcnii_relu_drop(z.data_ptr(), z.stride(0), h0.data_ptr(), h0.stride(0),
                                       hd.data_ptr() if hd is not None else None, hd.stride(0) if hd is not None else 0,
                                       n, d, _C.dtype_code(z.dtype), C.byref(drop.c()) if hd is not None else None,
                                       _C.stream_ptr()), "pg_gcnii_relu_drop")
    return h0, (hd if hd is not None else h0)


def gcnii_teleport(ds: torch.Tensor, acc: torch.Tensor, alpha: float, accumulate: bool):
    """acc = alpha * ds, or acc = fma(alpha, ds, acc) when `accumulate`, in fp32 (pg_gcnii_teleport)."""
    _rows(ds)
    assert acc.dtype == torch.float32 and acc.shape == ds.shape and acc.stride(1) == 1
    _C.count()
    _C.check(_C.lib.pg_gcnii_teleport(ds.data_ptr(), ds.stride(0), acc.data_ptr(), acc.stride(0), ds.shape[0],
                                      ds.shape[1], _C.dtype_code(ds.dtype), float(alpha), int(bool(accumulate)),
                                      _C.stream_ptr()), "pg_gcnii_teleport")


def gcnii_relu_bwd(g: torch.Tensor, h0: torch.Tensor, acc: torch.Tensor = None) -> torch.Tensor:
    """dz = (h0 > 0) ? g + acc : 0 in fp32, acc on its first acc.shape[0] rows only (pg_gcnii_relu_bwd)."""
    _rows(g)
    _rows(h0)
    n, d = g.shape
    assert h0.shape == g.shape and h0.dtype == g.dtype
    n_acc = 0
    if acc is not None:
        assert acc.dtype == torch.float32 and acc.shape[1] == d and acc.shape[0] <= n and acc.stride(1) == 1
        n_acc = acc.shape[0]
    dz = alloc_rows(n, d, g.dtype, g.device)
    _C.count()
    _C.check(_C.lib.pg_gcnii_relu_bwd(g.data_ptr(), g.stride(0), h0.data_ptr(), h0.stride(0),
                                      acc.data_ptr() if acc is not None else None,
                                      acc.stride(0) if acc is not None else 0, n_acc, dz.data_ptr(), dz.stride(0), n, d,
                                      _C.dtype_code(g.dtype), _C.stream_ptr()), "pg_gcnii_relu_bwd")
    return dz


class GCNIIState:
    """What the convolutions of one GCNII forward share: the clean initial representation h0 [num_all, d] (layer 0
    writes it, every convolution reads its inner rows), the dropout key of h0 on its way into convolution 0, and the
    fp32 [N_in, d] sum of the gradients the convolutions send to h0 (the first backward writes it, the later ones add
    to it: layer L-1 down to 0, the order autograd runs them in)."""

    def __init__(self, drop_h0: DropSpec = None):
        self.drop_h0 = drop_h0
        self.h0 = None
        self.acc = None
        self.written = False


def gcnii_weight(w1: torch.Tensor, beta: float) -> torch.Tensor:
    """W_eff = (1 - beta) I + beta W1 in fp32 from the master weight ([d, d], in x out)."""
    w = w1.detach().float() * beta
    w.diagonal().add_(1.0 - beta)
    return w


def _gcnii_conv_fwd(feat, graph, c, cs, h0_in, alpha, w_eff, bias):
    """S = (1-a) c[:N_in] * (A @ (c * feat)) + a h0 (the residual aggregate), out = S @ W_eff + b (pg_linear)."""
    s = aggregate_scaled_res(graph.fwd, feat, c, cs, res=h0_in, alpha=alpha)
    return s, gemm_nt(s, padded_weight(w_eff, feat.dtype, transpose=True), bias=bias)


def _gcnii_conv_bwd(ctx, g, s, w_eff, need_feat, drop_bwd):
    """Gradients of one convolution: dS = g W_eff^T (pg_linear), alpha dS into the teleport sum, the input gradient
    c * (A^T @ ((1-a) c[:N_in] * dS)) with the dropout backward in its store, dW1 = beta S^T g (pg_wgrad), db."""
    graph, c, cs, state = ctx.graph, ctx.c, ctx.cs, ctx.state
    colsum = _take_colsum(g)
    g = _tma_ready(g if g.dtype == s.dtype else g.to(s.dtype))
    gsp = presplit(g)
    ds = gemm_nt(gsp, padded_weight(w_eff, s.dtype))
    if state.acc is None:
        state.acc = alloc_rows(s.shape[0], s.shape[1], torch.float32, s.device)
    gcnii_teleport(ds, state.acc, ctx.alpha, accumulate=state.written)
    state.written = True
    g_feat = aggregate_scaled(graph.bwd, ds, cs, c, drop=drop_bwd) if need_feat else None
    gw = (wgrad(gsp, s).t() * ctx.beta).contiguous()
    gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
    return g_feat, gw, gb


class GCNIIConvFn(torch.autograd.Function):
    """GCNII convolution l >= 1 (DGL GCN2Conv, project_initial_features=True, no activation) over the [inner | halo]
    rows `feat`, with h0 the inner rows of state.h0:

        S   = (1-a) c[:N_in] * (A @ (c * feat)) + a h0      pg_aggregate_scaled_res over the CSR
        out = S @ ((1-b) I + b W1) + bias                   pg_linear

        dS = g W_eff^T                                      pg_linear
        h0 += a dS                                          pg_gcnii_teleport (fp32 sum, GCNIIState)
        g_feat = c * (A^T @ ((1-a) c[:N_in] * dS))          pg_aggregate_scaled over the CSC, dropout backward in its store
        dW1 = b S^T g, d bias = sum g
    """

    @staticmethod
    def forward(ctx, feat, weight1, bias, graph, c, cs, alpha, beta, state, drop_bwd=None):
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        w_eff = gcnii_weight(weight1, beta)
        s, out = _gcnii_conv_fwd(feat, graph, c, cs, state.h0[:graph.num_in], alpha, w_eff, bias)
        ctx.graph, ctx.c, ctx.cs, ctx.state, ctx.drop_bwd = graph, c, cs, state, drop_bwd
        ctx.alpha, ctx.beta, ctx.has_bias = alpha, beta, bias is not None
        ctx.save_for_backward(s, w_eff)
        return out

    @staticmethod
    def backward(ctx, g):
        s, w_eff = ctx.saved_tensors
        g_feat, gw, gb = _gcnii_conv_bwd(ctx, g, s, w_eff, ctx.needs_input_grad[0], ctx.drop_bwd)
        return g_feat, gw, gb, None, None, None, None, None, None, None


class GCNIIFirstFn(torch.autograd.Function):
    """Graph layer 0 of GCNII: fc_in over every [inner | halo] row of the (dropped) input features, then convolution 0:

        z = x W_in^T + b_in                                 pg_linear over num_all rows
        h0 = ReLU(z), hd = dropout(h0)                      pg_gcnii_relu_drop (state.h0 = h0)
        out = convolution 0 of hd with the residual h0[:N_in]     as GCNIIConvFn

    Backward: convolution 0's gradients (its teleport term last in the sum), then
        dz = ReLU'(z) * (g_hd + teleport sum on the inner rows)    pg_gcnii_relu_bwd
        dW_in = dz^T x (pg_wgrad), d b_in = column sum of dz (pg_gat_colsum); no gradient to x.
    Every rank's dW_in covers the halo rows it used: the all-reduce adds them up to the whole graph's gradient.
    """

    @staticmethod
    def forward(ctx, x, fc_weight, fc_bias, weight1, bias, graph, c, cs, alpha, beta, state):
        if x.stride(1) != 1:
            x = x.contiguous()
        z = gemm_nt(x, padded_weight(fc_weight, x.dtype), bias=fc_bias)
        h0, hd = gcnii_relu_drop(z, state.drop_h0)
        del z
        state.h0, state.acc, state.written = h0, None, False
        w_eff = gcnii_weight(weight1, beta)
        s, out = _gcnii_conv_fwd(hd, graph, c, cs, h0[:graph.num_in], alpha, w_eff, bias)
        ctx.graph, ctx.c, ctx.cs, ctx.state = graph, c, cs, state
        ctx.alpha, ctx.beta, ctx.has_bias = alpha, beta, bias is not None
        ctx.has_fc_bias = fc_bias is not None
        ctx.save_for_backward(x, h0, s, w_eff)
        return out

    @staticmethod
    def backward(ctx, g):
        x, h0, s, w_eff = ctx.saved_tensors
        state = ctx.state
        g_hd, gw, gb = _gcnii_conv_bwd(ctx, g, s, w_eff, True, state.drop_h0)
        dz = gcnii_relu_bwd(g_hd, h0, state.acc)
        dzsp = presplit(dz)
        g_fc_w = wgrad(dzsp, x)
        g_fc_b = gat_colsum(dz) if ctx.has_fc_bias else None
        return None, g_fc_w, g_fc_b, gw, gb, None, None, None, None, None, None


def gcnii_first(x, graph, c, cs, fc_weight, fc_bias, weight1, bias, alpha, beta, state) -> torch.Tensor:
    """Graph layer 0 of GCNII (GCNIIFirstFn): fc_in, ReLU and convolution 0; fills state.h0."""
    return GCNIIFirstFn.apply(x, fc_weight, fc_bias, weight1, bias, graph, c, cs, alpha, beta, state)


def gcnii_conv(feat, graph, c, cs, weight1, bias, alpha, beta, state, drop_bwd=None) -> torch.Tensor:
    """GCNII convolution l >= 1 (GCNIIConvFn) over the [num_all, d] rows `feat`; returns the [N_in, d] inner rows."""
    return GCNIIConvFn.apply(feat, weight1, bias, graph, c, cs, alpha, beta, state, drop_bwd)


# ---- graph attention (csrc/attention.cu) -------------------------------------------------------------------
def gat_preload():
    """Load every attention kernel now: a first launch may wait for the device, so it must not happen while a halo
    wait of a simulated rank spins."""
    _C.check(_C.lib.pg_gat_preload(), "pg_gat_preload")


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).reshape(-1).contiguous()


def gat_scores(z: torch.Tensor, attn_l: torch.Tensor, attn_r: torch.Tensor, heads: int, n_er: int):
    """(el [rows, H], er [n_er, H]) fp32: the per-head dot products of z with attn_l (every row) and attn_r (the
    first n_er rows)."""
    _rows(z)
    n, hd = z.shape
    el = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    er = torch.empty(n_er, heads, dtype=torch.float32, device=z.device)
    _C.count()
    _C.check(_C.lib.pg_gat_scores(z.data_ptr(), z.stride(0), n, int(n_er), heads, hd // heads, _C.dtype_code(z.dtype),
                                  attn_l.data_ptr(), attn_r.data_ptr(), el.data_ptr(), er.data_ptr(), _C.stream_ptr()),
             "pg_gat_scores")
    return el, er


def _gat_scratch(plan: CsrPlan, heads: int, d: int):
    return plan.scratch(heads * (d + 2))


def gat_aggregate(graph: PartGraph, z, el, er, bias, heads: int, keep=None):
    """out [N_in, H*D] = per-head edge softmax of LeakyReLU(el[u] + er[v]) over the forward CSR applied to z, + bias;
    with the softmax statistics m, s [N_in, H] fp32."""
    plan = graph.fwd
    n, hd = plan.n_rows, z.shape[1]
    d = hd // heads
    out = alloc_rows(n, hd, z.dtype, z.device)
    m = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    s = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    scratch = _gat_scratch(plan, heads, d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gat_aggregate(C.byref(plan.c), z.data_ptr(), z.stride(0), heads, d, _C.dtype_code(z.dtype),
                                     el.data_ptr(), er.data_ptr(), _ptr(bias), _ptr(keep), graph.num_in,
                                     out.data_ptr(), out.stride(0), m.data_ptr(), s.data_ptr(), _ptr(scratch),
                                     _C.stream_ptr()), "pg_gat_aggregate")
    return out, m, s


def gat_bwd_dst(graph: PartGraph, z, g, el, er, m, s, heads: int, keep=None):
    """(der, dv) [N_in, H] fp32: the gradient of er, and <g, out - bias> per row and head."""
    plan = graph.fwd
    n, hd = plan.n_rows, z.shape[1]
    d = hd // heads
    der = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    dv = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    scratch = _gat_scratch(plan, heads, d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gat_bwd_dst(C.byref(plan.c), z.data_ptr(), z.stride(0), g.data_ptr(), g.stride(0), heads, d,
                                   _C.dtype_code(z.dtype), el.data_ptr(), er.data_ptr(), m.data_ptr(), s.data_ptr(),
                                   _ptr(keep), graph.num_in, der.data_ptr(), dv.data_ptr(), _ptr(scratch),
                                   _C.stream_ptr()), "pg_gat_bwd_dst")
    return der, dv


def gat_bwd_src(graph: PartGraph, z, g, el, er, m, s, dv, der, attn_l, attn_r, heads: int, keep=None):
    """(dz [num_all, H*D] in z's dtype, del [num_all, H] fp32) over the CSC of the graph."""
    plan = graph.bwd
    n, hd = plan.n_rows, z.shape[1]
    d = hd // heads
    dz = alloc_rows(n, hd, z.dtype, z.device)
    dl = torch.empty(n, heads, dtype=torch.float32, device=z.device)
    scratch = _gat_scratch(plan, heads, d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gat_bwd_src(C.byref(plan.c), z.data_ptr(), z.stride(0), g.data_ptr(), g.stride(0), heads, d,
                                   _C.dtype_code(z.dtype), el.data_ptr(), er.data_ptr(), m.data_ptr(), s.data_ptr(),
                                   dv.data_ptr(), der.data_ptr(), attn_l.data_ptr(), attn_r.data_ptr(), _ptr(keep),
                                   graph.num_in, dz.data_ptr(), dz.stride(0), dl.data_ptr(), _ptr(scratch),
                                   _C.stream_ptr()), "pg_gat_bwd_src")
    return dz, dl


def gat_colsum(x: torch.Tensor, heads: int = 1, coef: torch.Tensor = None) -> torch.Tensor:
    """fp32 [H*D]: sum_r coef[r, k] * x[r, k*D + c] (coef None: plain column sums), in a fixed order."""
    _rows(x)
    n, hd = x.shape
    nb = int(_C.lib.pg_gat_colsum_blocks(n))
    partial = torch.empty(nb * hd, dtype=torch.float32, device=x.device)
    out = torch.empty(hd, dtype=torch.float32, device=x.device)
    _C.count(2)
    _C.check(_C.lib.pg_gat_colsum(x.data_ptr(), x.stride(0), n, heads, hd // heads, _C.dtype_code(x.dtype),
                                  _ptr(coef), out.data_ptr(), partial.data_ptr(), _C.stream_ptr()), "pg_gat_colsum")
    return out


class GatLayerFn(torch.autograd.Function):
    """One GAT layer (DGL GATConv, no attention dropout, no residual) over the [inner | halo] rows `feat` of a
    partition, returning the inner rows:

        z  = feat @ W^T                    [num_all, H*D]   pg_linear over all rows
        el, er                             [num_all, H]     pg_gat_scores (er of the inner rows only)
        out = softmax-aggregate(z) + bias  [N_in, H*D]      pg_gat_aggregate (+ softmax statistics m, s)

    Backward: der, D (pg_gat_bwd_dst over the CSR), dz and del (pg_gat_bwd_src over the CSC), d attn_l / d attn_r
    and the bias gradient as fixed-order column sums, dW = dz^T feat (pg_wgrad), g_feat = dz @ W (pg_linear, with the
    dropout backward of `drop_bwd` in its epilogue).  `keep`: the boundary-node sample of the halo rows (uint8), or
    None."""

    @staticmethod
    def forward(ctx, feat, graph, keep, heads, weight, attn_l, attn_r, bias, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        z = gemm_nt(presplit(feat), padded_weight(weight, feat.dtype))
        al, ar = _f32(attn_l), _f32(attn_r)
        el, er = gat_scores(z, al, ar, heads, n_in)
        b32 = _f32(bias) if bias is not None else None
        out, m, s = gat_aggregate(graph, z, el, er, b32, heads, keep)
        ctx.save_for_backward(feat, z, el, er, m, s, weight)
        ctx.graph, ctx.keep, ctx.heads, ctx.al, ctx.ar, ctx.b32 = graph, keep, heads, al, ar, b32
        ctx.attn_shape, ctx.attn_dtype = tuple(attn_l.shape), attn_l.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        feat, z, el, er, m, s, weight = ctx.saved_tensors
        graph, heads, keep = ctx.graph, ctx.heads, ctx.keep
        n_in = graph.num_in
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        der, dv = gat_bwd_dst(graph, z, g, el, er, m, s, heads, keep)
        dz, dl = gat_bwd_src(graph, z, g, el, er, m, s, dv, der, ctx.al, ctx.ar, heads, keep)
        g_al = gat_colsum(z, heads, dl).view(ctx.attn_shape).to(ctx.attn_dtype)
        g_ar = gat_colsum(z[:n_in], heads, der).view(ctx.attn_shape).to(ctx.attn_dtype)
        gb = None
        if ctx.b32 is not None:
            gb = colsum if colsum is not None else gat_colsum(g)
        dzsp = presplit(dz)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(feat.shape[0], feat.shape[1], feat.dtype, feat.device)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
            gemm_nt(dzsp, padded_weight(weight, feat.dtype, transpose=True), out=g_feat, drop=db)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        gw = wgrad(dzsp, presplit(feat)).to(weight.dtype)
        return g_feat, None, None, None, gw, g_al, g_ar, gb, None


def gat_layer(feat, graph, keep, heads, weight, attn_l, attn_r, bias, drop_bwd=None) -> torch.Tensor:
    return GatLayerFn.apply(feat, graph, keep, int(heads), weight, attn_l, attn_r, bias, drop_bwd)


# ---- dynamic graph attention, GATv2 (csrc/attention.cu) ----------------------------------------------------
def gatv2_preload():
    """Load every GATv2 kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_gatv2_preload(), "pg_gatv2_preload")


def gatv2_aggregate(graph: PartGraph, zs, zd, attn, heads: int, keep=None):
    """out [N_in, H*D] = per-head edge softmax of <attn, LeakyReLU(zs[u] + zd[v])> over the forward CSR applied to zs;
    with the softmax statistics m, s [N_in, H] fp32.  attn: fp32 [H*D]."""
    plan = graph.fwd
    n, hd = plan.n_rows, zs.shape[1]
    d = hd // heads
    out = alloc_rows(n, hd, zs.dtype, zs.device)
    m = torch.empty(n, heads, dtype=torch.float32, device=zs.device)
    s = torch.empty(n, heads, dtype=torch.float32, device=zs.device)
    scratch = plan.scratch(heads * (d + 2))
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gatv2_aggregate(C.byref(plan.c), zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), heads,
                                       d, _C.dtype_code(zs.dtype), attn.data_ptr(), _ptr(keep), graph.num_in,
                                       out.data_ptr(), out.stride(0), m.data_ptr(), s.data_ptr(), _ptr(scratch),
                                       _C.stream_ptr()), "pg_gatv2_aggregate")
    return out, m, s


def gatv2_bwd_dst(graph: PartGraph, zs, zd, g, attn, m, s, heads: int, keep=None):
    """(dzd [N_in, H*D] in zs's dtype, dv [N_in, H] fp32, pattn [N_in, H*D] fp32) over the forward CSR: the gradient
    of zd, D_v = <g_v, out_v>, and the per-row terms of the attn gradient (its column sum)."""
    plan = graph.fwd
    n, hd = plan.n_rows, zs.shape[1]
    d = hd // heads
    dzd = alloc_rows(n, hd, zs.dtype, zs.device)
    dv = torch.empty(n, heads, dtype=torch.float32, device=zs.device)
    pattn = alloc_rows(n, hd, torch.float32, zs.device)
    scratch = plan.scratch(heads * (4 * d + 1))
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gatv2_bwd_dst(C.byref(plan.c), zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0),
                                     g.data_ptr(), g.stride(0), heads, d, _C.dtype_code(zs.dtype), attn.data_ptr(),
                                     m.data_ptr(), s.data_ptr(), _ptr(keep), graph.num_in, dzd.data_ptr(),
                                     dzd.stride(0), dv.data_ptr(), pattn.data_ptr(), pattn.stride(0), _ptr(scratch),
                                     _C.stream_ptr()), "pg_gatv2_bwd_dst")
    return dzd, dv, pattn


def gatv2_bwd_src(graph: PartGraph, zs, zd, g, attn, m, s, dv, heads: int, keep=None):
    """dzs [num_all, H*D] in zs's dtype over the CSC of the graph (0 on unkept halo rows)."""
    plan = graph.bwd
    n, hd = plan.n_rows, zs.shape[1]
    d = hd // heads
    dzs = alloc_rows(n, hd, zs.dtype, zs.device)
    scratch = plan.scratch(heads * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_gatv2_bwd_src(C.byref(plan.c), zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0),
                                     g.data_ptr(), g.stride(0), heads, d, _C.dtype_code(zs.dtype), attn.data_ptr(),
                                     m.data_ptr(), s.data_ptr(), dv.data_ptr(), _ptr(keep), graph.num_in,
                                     dzs.data_ptr(), dzs.stride(0), _ptr(scratch), _C.stream_ptr()), "pg_gatv2_bwd_src")
    return dzs


class GatV2LayerFn(torch.autograd.Function):
    """One GATv2 layer (DGL GATv2Conv, share_weights=False, no attention dropout, no residual) over the [inner | halo]
    rows `feat` of a partition, returning the inner rows:

        zs  = feat @ W_s^T + b_s           [num_all, H*D]   pg_linear over all rows
        zd  = feat[:N_in] @ W_d^T + b_d    [N_in, H*D]      pg_linear over the inner rows
        out = softmax-aggregate(zs)        [N_in, H*D]      pg_gatv2_aggregate (+ softmax statistics m, s)

    Backward: dzd, D_v and the attn terms (pg_gatv2_bwd_dst over the CSR), dzs (pg_gatv2_bwd_src over the CSC), d attn
    and the bias gradients as fixed-order column sums, dW_s = dzs^T feat, dW_d = dzd^T feat[:N_in] (pg_wgrad),
    g_feat = dzs @ W_s (+ dzd @ W_d on the inner rows, one two-source pg_linear), with the dropout backward of
    `drop_bwd` in its epilogue.  `keep`: the boundary-node sample of the halo rows (uint8), or None."""

    @staticmethod
    def forward(ctx, feat, graph, keep, heads, w_s, b_s, w_d, b_d, attn, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        fsp = presplit(feat)                   # fp32: one split of feat for both products
        zs = gemm_nt(fsp, padded_weight(w_s, feat.dtype), bias=b_s)
        zd = gemm_nt(fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in], padded_weight(w_d, feat.dtype),
                     bias=b_d)
        a32 = _f32(attn)
        out, m, s = gatv2_aggregate(graph, zs, zd, a32, heads, keep)
        ctx.save_for_backward(feat, zs, zd, m, s, w_s, w_d)
        ctx.graph, ctx.keep, ctx.heads, ctx.a32 = graph, keep, heads, a32
        ctx.attn_shape, ctx.attn_dtype = tuple(attn.shape), attn.dtype
        ctx.has_bias = b_s is not None, b_d is not None
        return out

    @staticmethod
    def backward(ctx, g):
        feat, zs, zd, m, s, w_s, w_d = ctx.saved_tensors
        graph, heads, keep = ctx.graph, ctx.heads, ctx.keep
        n_in = graph.num_in
        _take_colsum(g)                        # no output bias: the by-product is not needed
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        dzd, dv, pattn = gatv2_bwd_dst(graph, zs, zd, g, ctx.a32, m, s, heads, keep)
        dzs = gatv2_bwd_src(graph, zs, zd, g, ctx.a32, m, s, dv, heads, keep)
        g_attn = gat_colsum(pattn).view(ctx.attn_shape).to(ctx.attn_dtype)
        gbs = gat_colsum(dzs) if ctx.has_bias[0] else None
        gbd = gat_colsum(dzd) if ctx.has_bias[1] else None
        dzsp, dzdp = presplit(dzs), presplit(dzd)
        is_split = isinstance(dzsp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(feat.shape[0], feat.shape[1], feat.dtype, feat.device)
            wst = padded_weight(w_s, feat.dtype, transpose=True)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
            gemm_nt(dzsp.rows(0, n_in) if is_split else dzs[:n_in], wst, dzdp,
                    padded_weight(w_d, feat.dtype, transpose=True), out=g_feat[:n_in], drop=db)
            if feat.shape[0] > n_in:
                gemm_nt(dzsp.rows(n_in) if is_split else dzs[n_in:], wst, out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        fsp = presplit(feat)
        gws = wgrad(dzsp, fsp).to(w_s.dtype)
        gwd = wgrad(dzdp, fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in]).to(w_d.dtype)
        return g_feat, None, None, None, gws, gbs, gwd, gbd, g_attn, None


def gatv2_layer(feat, graph, keep, heads, w_s, b_s, w_d, b_d, attn, drop_bwd=None) -> torch.Tensor:
    return GatV2LayerFn.apply(feat, graph, keep, int(heads), w_s, b_s, w_d, b_d, attn, drop_bwd)


# ---- graph transformer, TransformerConv (csrc/attention.cu) -------------------------------------------------
def transformer_preload():
    """Load every graph-transformer kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_tconv_preload(), "pg_tconv_preload")


def transformer_width(hd: int, dtype) -> int:
    """Columns of each half of the paired [k | v] and [q | skip] operands: H*D, rounded up to a multiple of 8 when
    H*D elements are not a multiple of 16 bytes, so that the second half starts 16-byte aligned like every GEMM
    operand (a misaligned view would be copied by _tma_ready)."""
    es = torch.empty((), dtype=dtype).element_size()
    return hd if (hd * es) % 16 == 0 else (hd + 7) // 8 * 8


def _tconv_scale(d: int) -> float:
    return 1.0 / math.sqrt(d)


def transformer_aggregate(graph: PartGraph, q, k, v, skip, heads: int, keep=None):
    """out [N_in, H*D] = per-head edge softmax of <q[v], k[u]> / sqrt(D) over the forward CSR applied to v, + skip;
    with the softmax statistics m, s [N_in, H] fp32."""
    plan = graph.fwd
    n, hd = plan.n_rows, q.shape[1]
    d = hd // heads
    out = alloc_rows(n, hd, q.dtype, q.device)
    m = torch.empty(n, heads, dtype=torch.float32, device=q.device)
    s = torch.empty(n, heads, dtype=torch.float32, device=q.device)
    scratch = plan.scratch(heads * (d + 2))
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_tconv_aggregate(C.byref(plan.c), q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0),
                                       v.data_ptr(), v.stride(0), skip.data_ptr(), skip.stride(0), heads, d,
                                       _C.dtype_code(q.dtype), _tconv_scale(d), _ptr(keep), graph.num_in,
                                       out.data_ptr(), out.stride(0), m.data_ptr(), s.data_ptr(), _ptr(scratch),
                                       _C.stream_ptr()), "pg_tconv_aggregate")
    return out, m, s


def transformer_bwd_dst(graph: PartGraph, q, k, v, g, m, s, heads: int, keep=None, dq=None, gc=None):
    """(dq [N_in, H*D], gc = a copy of g, both in q's dtype, delta [N_in, H] fp32) over the forward CSR, with
    delta_v = sum_u a_uv <g_v, v_u>.  `dq` / `gc`: the views to write (allocated when None)."""
    plan = graph.fwd
    n, hd = plan.n_rows, q.shape[1]
    d = hd // heads
    dq = alloc_rows(n, hd, q.dtype, q.device) if dq is None else dq
    gc = alloc_rows(n, hd, q.dtype, q.device) if gc is None else gc
    delta = torch.empty(n, heads, dtype=torch.float32, device=q.device)
    scratch = plan.scratch(heads * (2 * d + 1))
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_tconv_bwd_dst(C.byref(plan.c), q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0),
                                     v.data_ptr(), v.stride(0), g.data_ptr(), g.stride(0), heads, d,
                                     _C.dtype_code(q.dtype), _tconv_scale(d), m.data_ptr(), s.data_ptr(), _ptr(keep),
                                     graph.num_in, dq.data_ptr(), dq.stride(0), gc.data_ptr(), gc.stride(0),
                                     delta.data_ptr(), _ptr(scratch), _C.stream_ptr()), "pg_tconv_bwd_dst")
    return dq, gc, delta


def transformer_bwd_src(graph: PartGraph, q, k, v, g, m, s, delta, heads: int, keep=None, dk=None, dv=None):
    """(dk, dv) [num_all, H*D] in k's dtype over the CSC of the graph (0 on unkept halo rows).  `dk` / `dv`: the
    views to write (allocated when None)."""
    plan = graph.bwd
    n, hd = plan.n_rows, k.shape[1]
    d = hd // heads
    dk = alloc_rows(n, hd, k.dtype, k.device) if dk is None else dk
    dv = alloc_rows(n, hd, k.dtype, k.device) if dv is None else dv
    scratch = plan.scratch(heads * 2 * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_tconv_bwd_src(C.byref(plan.c), q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0),
                                     v.data_ptr(), v.stride(0), g.data_ptr(), g.stride(0), heads, d,
                                     _C.dtype_code(k.dtype), _tconv_scale(d), m.data_ptr(), s.data_ptr(),
                                     delta.data_ptr(), _ptr(keep), graph.num_in, dk.data_ptr(), dk.stride(0),
                                     dv.data_ptr(), dv.stride(0), _ptr(scratch), _C.stream_ptr()), "pg_tconv_bwd_src")
    return dk, dv


def _pair_weight(wa, wb, width: int, dtype, transpose: bool = False) -> torch.Tensor:
    """[2 width, d_in] in the activation dtype with wa in rows [0, H*D) and wb in rows [width, width + H*D), zero
    rows between (transpose: its [d_in, 2 width] transpose), built from the fp32 masters."""
    hd, d_in = wa.shape
    pad = width != hd
    if transpose:
        out = alloc_rows(d_in, 2 * width, dtype, wa.device, zero=pad)
        out[:, :hd].copy_(wa.detach().t())
        out[:, width:width + hd].copy_(wb.detach().t())
    else:
        out = alloc_rows(2 * width, d_in, dtype, wa.device, zero=pad)
        out[:hd].copy_(wa.detach())
        out[width:width + hd].copy_(wb.detach())
    return out


def _pair_bias(ba, bb, hd: int, width: int) -> torch.Tensor:
    out = torch.zeros(2 * width, dtype=torch.float32, device=ba.device)
    out[:hd].copy_(ba.detach())
    out[width:width + hd].copy_(bb.detach())
    return out


class TransformerLayerFn(torch.autograd.Function):
    """One graph-transformer layer (PyG TransformerConv, concat=True, beta=False, root_weight=True, no edge features,
    no attention dropout) over the [inner | halo] rows `feat` of a partition, returning the inner rows.  With W the
    half width of transformer_width:

        [k | v]    = feat @ [W_k; W_v]^T + [b_k; b_v]          [num_all, 2W]   one pg_linear over all rows
        [q | skip] = feat[:N_in] @ [W_q; W_s]^T + [b_q; b_s]   [N_in, 2W]      one pg_linear over the inner rows
        out = softmax-aggregate(v) + skip                      [N_in, H*D]     pg_tconv_aggregate (+ statistics m, s)

    Backward: dq next to a copy of g (pg_tconv_bwd_dst over the CSR, which also writes delta_v), [dk | dv]
    (pg_tconv_bwd_src over the CSC), the bias gradients as fixed-order column sums (b_s from the column sum the
    LayerNorm backward stashed, when there is one; b_k's is exactly 0, the softmax being shift-invariant), the weight gradients as one pg_wgrad per row set, and
    g_feat = [dk | dv] @ [W_k; W_v] (+ [dq | g] @ [W_q; W_s] on the inner rows, one two-source pg_linear), with the
    dropout backward of `drop_bwd` in its epilogue.  `keep`: the boundary-node sample of the halo rows (uint8), or
    None."""

    @staticmethod
    def forward(ctx, feat, graph, keep, heads, w_q, b_q, w_k, b_k, w_v, b_v, w_s, b_s, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in, hd = graph.num_in, w_q.shape[0]
        w = transformer_width(hd, feat.dtype)
        fsp = presplit(feat)                   # fp32: one split of feat for both products
        kv = gemm_nt(fsp, _pair_weight(w_k, w_v, w, feat.dtype), bias=_pair_bias(b_k, b_v, hd, w))
        qs = gemm_nt(fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in],
                     _pair_weight(w_q, w_s, w, feat.dtype), bias=_pair_bias(b_q, b_s, hd, w))
        out, m, s = transformer_aggregate(graph, qs[:, :hd], kv[:, :hd], kv[:, w:w + hd], qs[:, w:w + hd], heads,
                                          keep)
        ctx.save_for_backward(feat, kv, qs, m, s, w_q, w_k, w_v, w_s)
        ctx.graph, ctx.keep, ctx.heads, ctx.width = graph, keep, heads, w
        return out

    @staticmethod
    def backward(ctx, g):
        feat, kv, qs, m, s, w_q, w_k, w_v, w_s = ctx.saved_tensors
        graph, heads, keep, w = ctx.graph, ctx.heads, ctx.keep, ctx.width
        n_in, n_all, hd = graph.num_in, feat.shape[0], w_q.shape[0]
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        q, k, v = qs[:, :hd], kv[:, :hd], kv[:, w:w + hd]
        dqg = alloc_rows(n_in, 2 * w, feat.dtype, feat.device, zero=w != hd)
        dkv = alloc_rows(n_all, 2 * w, feat.dtype, feat.device, zero=w != hd)
        _, _, delta = transformer_bwd_dst(graph, q, k, v, g, m, s, heads, keep, dq=dqg[:, :hd], gc=dqg[:, w:w + hd])
        transformer_bwd_src(graph, q, k, v, g, m, s, delta, heads, keep, dk=dkv[:, :hd], dv=dkv[:, w:w + hd])
        # b_k shifts every score of a destination row by the same <q_v, b_k>, which the softmax cancels: its gradient
        # sum_u dk_u = scale sum_v q_v sum_u a_uv (gd_uv - delta_v) is exactly 0, so it is not summed from rounded dk
        gbk = torch.zeros(hd, dtype=torch.float32, device=feat.device)
        gbv = gat_colsum(dkv[:, w:w + hd])
        if colsum is not None:
            gbq, gbs = gat_colsum(dqg[:, :hd]), colsum
        else:
            gb_qs = gat_colsum(dqg)
            gbq, gbs = gb_qs[:hd], gb_qs[w:w + hd]
        dkvp, dqgp = presplit(dkv), presplit(dqg)
        is_split = isinstance(dkvp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(n_all, feat.shape[1], feat.dtype, feat.device)
            wkv = _pair_weight(w_k, w_v, w, feat.dtype, transpose=True)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
            gemm_nt(dkvp.rows(0, n_in) if is_split else dkv[:n_in], wkv, dqgp,
                    _pair_weight(w_q, w_s, w, feat.dtype, transpose=True), out=g_feat[:n_in], drop=db)
            if n_all > n_in:
                gemm_nt(dkvp.rows(n_in) if is_split else dkv[n_in:], wkv, out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        fsp = presplit(feat)
        gw_kv = wgrad(dkvp, fsp)
        gw_qs = wgrad(dqgp, fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in])
        gwq, gwk, gwv, gws = [t.contiguous() for t in (gw_qs[:hd], gw_kv[:hd], gw_kv[w:w + hd], gw_qs[w:w + hd])]
        return (g_feat, None, None, None, gwq.to(w_q.dtype), gbq.contiguous(), gwk.to(w_k.dtype), gbk,
                gwv.to(w_v.dtype), gbv, gws.to(w_s.dtype), gbs.contiguous(), None)


def transformer_layer(feat, graph, keep, heads, w_q, b_q, w_k, b_k, w_v, b_v, w_s, b_s,
                      drop_bwd=None) -> torch.Tensor:
    return TransformerLayerFn.apply(feat, graph, keep, int(heads), w_q, b_q, w_k, b_k, w_v, b_v, w_s, b_s, drop_bwd)


# ---- max-pool GraphSAGE (csrc/pool.cu) ---------------------------------------------------------------------
def pool_preload():
    """Load every pool kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_pool_preload(), "pg_pool_preload")


def _scratch_ld(d: int) -> int:
    return (int(d) + 7) // 8 * 8


def max_aggregate(plan: CsrPlan, q: torch.Tensor):
    """(hn, A) over the forward CSR `plan`: hn [n_rows, d] = ReLU(max over the in-edges u -> v of q[u]) in q's dtype
    (0 for a row without in-edges), A [n_rows, d] int32 = the u of that maximum (the first in CSR order on a tie, -1
    for a row without in-edges)."""
    _rows(q)
    d = q.shape[1]
    hn = alloc_rows(plan.n_rows, d, q.dtype, q.device)
    arg = alloc_rows(plan.n_rows, d, torch.int32, q.device)
    ld_s = _scratch_ld(2 * d)
    scratch = plan.scratch(2 * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_max_aggregate(C.byref(plan.c), q.data_ptr(), q.stride(0), d, _C.dtype_code(q.dtype),
                                     hn.data_ptr(), hn.stride(0), arg.data_ptr(), arg.stride(0), _ptr(scratch), ld_s,
                                     _C.stream_ptr()), "pg_max_aggregate")
    return hn, arg


def max_aggregate_bwd(plan_t: CsrPlan, q: torch.Tensor, arg: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """gq [plan_t.n_rows, d] in q's dtype: gq[u, c] = [q[u, c] > 0] * sum over the CSC row u of `plan_t` of g[v, c]
    where arg[v, c] == u, accumulated in fp32 in CSC order."""
    _rows(q), _rows(arg), _rows(g)
    d = q.shape[1]
    assert g.dtype == q.dtype and arg.dtype == torch.int32 and g.shape[1] == d and arg.shape == g.shape
    gq = alloc_rows(plan_t.n_rows, d, q.dtype, q.device)
    scratch = plan_t.scratch(d)
    _C.count(2 if plan_t.n_long else 1)
    _C.check(_C.lib.pg_max_aggregate_bwd(C.byref(plan_t.c), q.data_ptr(), q.stride(0), arg.data_ptr(), arg.stride(0),
                                         g.data_ptr(), g.stride(0), d, _C.dtype_code(q.dtype), gq.data_ptr(),
                                         gq.stride(0), _ptr(scratch), _scratch_ld(d), _C.stream_ptr()),
             "pg_max_aggregate_bwd")
    return gq


class SagePoolLayerFn(torch.autograd.Function):
    """One max-pool GraphSAGE layer (DGL SAGEConv(aggregator_type='pool')) over the [inner | halo] rows `feat` of a
    partition, returning the inner rows:

        Q   = feat @ Wp^T + bp                           [num_all, d_in]  pg_linear over all rows
        hn  = ReLU(max_{u -> v} Q[u]), A = its argmax    [N_in, d_in]     pg_max_aggregate
        out = feat[:N_in] @ W1^T + hn @ W2^T + (b1 + b2) [N_in, d_out]    pg_linear, two sources

    ReLU(max Q) = max ReLU(Q) exactly, so the ReLU is the aggregate's store.  Backward: g_neigh = g @ W2 (pg_linear),
    gQ = [Q > 0] * the g_neigh of the destinations whose argmax is u (pg_max_aggregate_bwd over the CSC),
    g_feat = g @ W1 + gQ @ Wp (one two-source pg_linear on the inner rows, gQ @ Wp on the halo rows, the dropout
    backward of `drop_bwd` in their epilogues), dW1 = g^T feat[:N_in], dW2 = g^T hn, dWp = gQ^T feat (pg_wgrad),
    dbp = colsum(gQ).  `keep`: the boundary-node sample of the halo rows (uint8) or None; an unkept halo row's Q is
    zeroed, so it can win only where the output is 0, and gets no gradient."""

    @staticmethod
    def forward(ctx, feat, graph, keep, w1, b1, w2, b2, wp, bp, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in = graph.num_in
        fsp = presplit(feat)                   # fp32: one split of feat for both products
        q = gemm_nt(fsp, padded_weight(wp, feat.dtype), bias=bp)
        if keep is not None and feat.shape[0] > n_in:
            bns_mask_rows(keep, q[n_in:])
        hn, arg = max_aggregate(graph.fwd, q)
        bias = None
        if b1 is not None:
            bias = b1.detach().float() + b2.detach().float()
        out = gemm_nt(fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in], padded_weight(w1, feat.dtype),
                      hn, padded_weight(w2, feat.dtype), bias=bias)
        ctx.graph = graph
        ctx.has_bias, ctx.has_pbias = b1 is not None, bp is not None
        ctx.save_for_backward(feat, q, arg, hn, w1, w2, wp)
        return out

    @staticmethod
    def backward(ctx, g):
        feat, q, arg, hn, w1, w2, wp = ctx.saved_tensors
        graph = ctx.graph
        n_in = graph.num_in
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        gsp = presplit(g)                      # fp32: one split of g serves g_neigh, the g_feat product and dW1 / dW2
        g_neigh = gemm_nt(gsp, padded_weight(w2, feat.dtype, transpose=True))
        gq = max_aggregate_bwd(graph.bwd, q, arg, g_neigh)
        gqsp = presplit(gq)
        is_split = isinstance(gqsp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(feat.shape[0], feat.shape[1], feat.dtype, feat.device)
            wpt = padded_weight(wp, feat.dtype, transpose=True)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
            gemm_nt(gsp, padded_weight(w1, feat.dtype, transpose=True), gqsp.rows(0, n_in) if is_split else gq[:n_in],
                    wpt, out=g_feat[:n_in], drop=db)
            if feat.shape[0] > n_in:
                gemm_nt(gqsp.rows(n_in) if is_split else gq[n_in:], wpt, out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        gw1 = wgrad(gsp, feat[:n_in]).to(w1.dtype)
        gw2 = wgrad(gsp, hn).to(w2.dtype)
        gwp = wgrad(gqsp, feat).to(wp.dtype)
        gb = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias else None
        gbp = gat_colsum(gq) if ctx.has_pbias else None
        return g_feat, None, None, gw1, gb, gw2, gb, gwp, gbp, None


def sage_pool_layer(feat, graph, keep, w1, b1, w2, b2, wp, bp, drop_bwd=None) -> torch.Tensor:
    return SagePoolLayerFn.apply(feat, graph, keep, w1, b1, w2, b2, wp, bp, drop_bwd)


# ---- principal neighbourhood aggregation, PNAConv (csrc/pna.cu) --------------------------------------------
def pna_preload():
    """Load every PNA kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_pna_preload(), "pg_pna_preload")


def pna_width(d: int) -> int:
    """Stride of the parts of the concatenated PNA operands ([mu | max | min | std], [g | a g | t g], [g_zs | g_zd]):
    d rounded up to a multiple of 8, so that every part starts on a 16-byte boundary.  The columns between the parts
    are zero."""
    return (int(d) + 7) // 8 * 8


def pna_degree_histogram(indptr: torch.Tensor) -> list:
    """Counts of the row lengths 0, 1, ... of a CSR (a partition's inner rows): the integer input of pna_delta."""
    deg = (indptr[1:] - indptr[:-1]).to(device="cpu", dtype=torch.int64)
    return torch.bincount(deg).tolist() if deg.numel() else []


def pna_delta(histograms) -> float:
    """PNA's delta, the mean of log(D + 1) over the nodes, from the degree histograms of all partitions: merged as
    integers, then sum_k count_k log1p(k) / N in fp64 in ascending k -- the same bits on every rank, for any
    partitioning of the same graph."""
    merged = [0] * max((len(h) for h in histograms), default=0)
    for h in histograms:
        for k, c in enumerate(h):
            merged[k] += int(c)
    n = sum(merged)
    if n == 0:
        raise ValueError("PNA: delta of an empty graph")
    s = 0.0
    for k, c in enumerate(merged):
        if c:
            s += c * math.log1p(k)
    delta = s / n
    if not delta > 0:
        raise ValueError(f"PNA: delta {delta} (every node without in-edges)")
    return delta


def pna_scalers_host(deg: torch.Tensor, delta: float):
    """(a, t) fp32: the amplification log(D + 1) / delta and attenuation delta / log(D + 1) of rows with D in-edges,
    computed in fp64 and rounded once (t = 0 for D = 0: such a row aggregates to 0)."""
    lg = torch.log1p(deg.to(torch.float64))
    a = lg / float(delta)
    t = torch.where(deg > 0, float(delta) / torch.where(deg > 0, lg, torch.ones_like(lg)), torch.zeros_like(lg))
    return a.to(torch.float32), t.to(torch.float32)


def pna_aggregate(plan: CsrPlan, zs: torch.Tensor, zd: torch.Tensor, stats: bool = True):
    """(agg, mu, var, amax, amin) over the forward CSR `plan` (pg_pna_aggregate): agg [n_rows, 4 W] in zs's dtype
    ([mu + zd | max + zd | min + zd | std], parts W = pna_width(d) apart, zero between), mu / var [n_rows, d] fp32 and
    the sources of the extremes amax / amin [n_rows, d] int32.  `stats` False: only agg (the others are None)."""
    _rows(zs), _rows(zd)
    n, d = plan.n_rows, zs.shape[1]
    w = pna_width(d)
    assert zd.dtype == torch.float32 and zd.shape == (n, d)
    dev = zs.device
    agg = alloc_rows(n, 4 * w, zs.dtype, dev, zero=w != d)
    mu = var = amax = amin = None
    if stats:
        mv = alloc_rows(n, 2 * w, torch.float32, dev)
        ar = alloc_rows(n, 2 * w, torch.int32, dev)
        mu, var, amax, amin = mv[:, :d], mv[:, w:w + d], ar[:, :d], ar[:, w:w + d]
    scratch = plan.scratch(6 * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_pna_aggregate(C.byref(plan.c), zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), d,
                                     _C.dtype_code(zs.dtype), agg.data_ptr(), agg.stride(0), w, _ptr(mu), _ptr(var),
                                     mu.stride(0) if stats else 0, _ptr(amax), _ptr(amin),
                                     amax.stride(0) if stats else 0, _ptr(scratch), _scratch_ld(6 * d),
                                     _C.stream_ptr()), "pg_pna_aggregate")
    return agg, mu, var, amax, amin


def pna_combine(y: torch.Tensor, z: torch.Tensor, a: torch.Tensor, t: torch.Tensor, dtype) -> torch.Tensor:
    """out [n, d_out] = y + a * z[:, :d_out] + t * z[:, d_out:] in fp32, rounded once to `dtype` (pg_pna_combine)."""
    n, d_out = y.shape
    out = alloc_rows(n, d_out, dtype, y.device)
    _C.count()
    _C.check(_C.lib.pg_pna_combine(y.data_ptr(), y.stride(0), z.data_ptr(), z.stride(0), a.data_ptr(), t.data_ptr(),
                                   n, d_out, _C.dtype_code(dtype), out.data_ptr(), out.stride(0), _C.stream_ptr()),
             "pg_pna_combine")
    return out


def pna_grad_scale(g: torch.Tensor, a: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """G3 = [g | a g | t g] in g's dtype, parts pna_width(d_out) apart, zero between (pg_pna_grad_scale)."""
    _rows(g)
    n, d_out = g.shape
    wo = pna_width(d_out)
    out = alloc_rows(n, 3 * wo, g.dtype, g.device, zero=wo != d_out)
    _C.count()
    _C.check(_C.lib.pg_pna_grad_scale(g.data_ptr(), g.stride(0), a.data_ptr(), t.data_ptr(), n, d_out,
                                      _C.dtype_code(g.dtype), out.data_ptr(), out.stride(0), wo, _C.stream_ptr()),
             "pg_pna_grad_scale")
    return out


def pna_bwd_dst(indptr: torch.Tensor, gagg: torch.Tensor, mu: torch.Tensor, var: torch.Tensor, gzd: torch.Tensor):
    """(alpha, beta [n, d] fp32, g_mx, g_mn [n, d] in gzd's dtype) from g_agg [n, 4 W] fp32 (pg_pna_bwd_dst); writes
    g_zd into `gzd`."""
    n, d = mu.shape
    w = pna_width(d)
    dev = mu.device
    ab = alloc_rows(n, 2 * w, torch.float32, dev)
    gm = alloc_rows(n, 2 * w, gzd.dtype, dev)
    alpha, beta, gmx, gmn = ab[:, :d], ab[:, w:w + d], gm[:, :d], gm[:, w:w + d]
    _C.count()
    _C.check(_C.lib.pg_pna_bwd_dst(indptr.data_ptr(), gagg.data_ptr(), gagg.stride(0), w, mu.data_ptr(),
                                   var.data_ptr(), mu.stride(0), n, d, _C.dtype_code(gzd.dtype), gzd.data_ptr(),
                                   gzd.stride(0), alpha.data_ptr(), beta.data_ptr(), alpha.stride(0), gmx.data_ptr(),
                                   gmn.data_ptr(), gmx.stride(0), _C.stream_ptr()), "pg_pna_bwd_dst")
    return alpha, beta, gmx, gmn


def pna_bwd_src(plan_t: CsrPlan, zs, alpha, beta, amax, amin, gmx, gmn, gzs: torch.Tensor) -> torch.Tensor:
    """g_zs over the CSC `plan_t` into `gzs` [plan_t.n_rows, d] (pg_pna_bwd_src)."""
    d = zs.shape[1]
    scratch = plan_t.scratch(2 * d)
    _C.count(2 if plan_t.n_long else 1)
    _C.check(_C.lib.pg_pna_bwd_src(C.byref(plan_t.c), zs.data_ptr(), zs.stride(0), alpha.data_ptr(), beta.data_ptr(),
                                   alpha.stride(0), amax.data_ptr(), amin.data_ptr(), amax.stride(0), gmx.data_ptr(),
                                   gmn.data_ptr(), gmx.stride(0), d, _C.dtype_code(zs.dtype), gzs.data_ptr(),
                                   gzs.stride(0), _ptr(scratch), _scratch_ld(2 * d), _C.stream_ptr()),
             "pg_pna_bwd_src")
    return gzs


def pna_u_operands(w_u: torch.Tensor, d: int, dtype, transposed: bool = False):
    """U's scaled-aggregate columns [W_1 | W_2 | W_3] ([d_out, 12 d]) as the padded GEMM operands of a PNA layer, each
    written once from the master weights in the activation dtype, zero in the columns between the parts (pna_width):
    W_1 [d_out, 4 W] and [W_2; W_3] [2 d_out, 4 W] for the forward, and with `transposed` also the backward's
    [W_1; W_2; W_3]^T [4 W, 3 Wo] (element (k W + c, s Wo + o) = W_{s+1}[o, k d + c]).  None in place of the last one
    otherwise."""
    d_out = w_u.shape[0]
    w, wo = pna_width(d), pna_width(d_out)
    pad = w != d
    src = w_u.detach()[:, d:].view(d_out, 3, 4, d)
    w1 = alloc_rows(d_out, 4 * w, dtype, w_u.device, zero=pad)
    w1.view(d_out, 4, w)[:, :, :d].copy_(src[:, 0])
    w23 = alloc_rows(2 * d_out, 4 * w, dtype, w_u.device, zero=pad)
    w23.view(2, d_out, 4, w)[:, :, :, :d].copy_(src[:, 1:].permute(1, 0, 2, 3))
    w123t = None
    if transposed:
        w123t = alloc_rows(4 * w, 3 * wo, dtype, w_u.device, zero=pad or wo != d_out)
        w123t.view(4, w, 3, wo)[:, :d, :, :d_out].copy_(src.permute(2, 3, 1, 0))
    return w1, w23, w123t


def _col_split(sp, lo: int, hi: int):
    """Columns [lo, hi) of an fp32 `Split` (or of a plain tensor)."""
    if not isinstance(sp, Split):
        return sp[:, lo:hi]
    out = Split.__new__(Split)
    out.x, out.hi, out.lo = sp.x[:, lo:hi], sp.hi[:, lo:hi], sp.lo[:, lo:hi]
    return out


class PnaLayerFn(torch.autograd.Function):
    """One PNA layer (DGL PNAConvTower: aggregators mean, max, min, std; scalers identity, amplification,
    attenuation; one tower, no edge features) over the [inner | halo] rows `feat` of a partition, returning the inner
    rows.  With M.weight = [W_s | W_d], U.weight = [W_x | W_1 | W_2 | W_3], W = pna_width(d):

        zs  = feat @ W_s^T                                  [num_all, d]    pg_linear over all rows
        zd  = feat[:N_in] @ W_d^T + b_M                     [N_in, d] fp32  pg_linear over the inner rows
        agg = [mu + zd | max + zd | min + zd | std]         [N_in, 4W]      pg_pna_aggregate (+ mu, var, A+, A-)
        y   = feat[:N_in] @ W_x^T + agg @ W_1^T + b_U       [N_in, d_out]   fp32, one two-source pg_linear
        z   = agg @ [W_2; W_3]^T                            [N_in, 2 d_out] fp32, pg_linear
        out = y + a * z[:, :d_out] + t * z[:, d_out:]                       pg_pna_combine

    The per-row scalers a, t are applied to d_out-wide outputs, so the 12d-wide scaled aggregate is never formed.
    Backward: G3 = [g | a g | t g] (pg_pna_grad_scale), g_agg = G3 @ [W_1; W_2; W_3] (fp32, pg_linear), g_zd, alpha,
    beta, g_mx, g_mn (pg_pna_bwd_dst), g_zs (pg_pna_bwd_src over the CSC), written side by side as [g_zs | g_zd];
    g_feat = g @ W_x + [g_zs | g_zd] @ [W_s; W_d] on the inner rows and g_zs @ W_s on the halo rows with the dropout
    backward of `drop_bwd` in their epilogues; dW_x = g^T feat[:N_in], [dW_1; dW_2; dW_3] = G3^T agg,
    dW_s = g_zs^T feat, dW_d = g_zd^T feat[:N_in] (pg_wgrad), db_U = colsum(g), db_M = colsum(g_zd)."""

    @staticmethod
    def forward(ctx, feat, graph, delta, w_m, b_m, w_u, b_u, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in, d = graph.num_in, feat.shape[1]
        sa, st = graph.pna_scalers(delta)
        fsp = presplit(feat)                   # fp32: one split of feat for every product
        finner = fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in]
        zs = gemm_nt(fsp, padded_weight(w_m[:, :d], feat.dtype))
        zd = gemm_nt(finner, padded_weight(w_m[:, d:], feat.dtype), bias=b_m, out_dtype=torch.float32)
        keep = any(ctx.needs_input_grad)
        agg, mu, var, amax, amin = pna_aggregate(graph.fwd, zs, zd, stats=keep)
        del zd
        w1, w23, w123t = pna_u_operands(w_u, d, feat.dtype, transposed=keep)
        aggsp = presplit(agg)
        y = gemm_nt(finner, padded_weight(w_u[:, :d], feat.dtype), aggsp, w1, bias=b_u, out_dtype=torch.float32)
        z = gemm_nt(aggsp, w23, out_dtype=torch.float32)
        out = pna_combine(y, z, sa, st, feat.dtype)
        if keep:
            ctx.save_for_backward(feat, zs, agg, mu, var, amax, amin, w_m, w_u)
            ctx.graph, ctx.sa, ctx.st, ctx.has_bias = graph, sa, st, (b_m is not None, b_u is not None)
            ctx.w123t = w123t                  # the step's weights: the backward uses the forward's operand
        return out

    @staticmethod
    def backward(ctx, g):
        feat, zs, agg, mu, var, amax, amin, w_m, w_u = ctx.saved_tensors
        graph = ctx.graph
        n_in, n_all, d, d_out = graph.num_in, feat.shape[0], feat.shape[1], w_u.shape[0]
        w, wo = pna_width(d), pna_width(d_out)
        dt = feat.dtype
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == dt else g.to(dt))
        g3 = pna_grad_scale(g, ctx.sa, ctx.st)
        g3sp = presplit(g3)
        gagg = gemm_nt(g3sp, ctx.w123t, out_dtype=torch.float32)
        ctx.w123t = None
        pz = alloc_rows(n_all, 2 * w, dt, feat.device, zero=w != d)      # [g_zs | g_zd]
        gzd = pz[:n_in, w:w + d]
        alpha, beta, gmx, gmn = pna_bwd_dst(graph.fwd.indptr, gagg, mu, var, gzd)
        del gagg
        pna_bwd_src(graph.bwd, zs, alpha, beta, amax, amin, gmx, gmn, pz[:, :d])
        del alpha, beta, gmx, gmn
        gsp, pzsp = presplit(g), presplit(pz)
        is_split = isinstance(pzsp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(n_all, d, dt, feat.device)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and d <= 256 and _drop_ok(g_feat) else None
            gemm_nt(gsp, padded_weight(w_u[:, :d], dt, transpose=True), pzsp.rows(0, n_in) if is_split else pz[:n_in],
                    _pair_weight(w_m[:, :d], w_m[:, d:], w, dt, transpose=True), out=g_feat[:n_in], drop=db)
            if n_all > n_in:
                gemm_nt(_col_split(pzsp.rows(n_in) if is_split else pz[n_in:], 0, d),
                        padded_weight(w_m[:, :d], dt, transpose=True), out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        fsp = presplit(feat)
        finner = fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in]
        gws = wgrad(_col_split(pzsp, 0, d), fsp)
        gwd = wgrad(_col_split(pzsp.rows(0, n_in) if is_split else pz[:n_in], w, w + d), finner)
        gwx = wgrad(gsp, finner)
        gr = wgrad(g3sp, presplit(agg)).view(3, wo, 4, w)[:, :d_out, :, :d]
        gw_u = torch.cat([gwx, gr.permute(1, 0, 2, 3).reshape(d_out, 12 * d)], 1)
        gw_m = torch.cat([gws, gwd], 1)
        gbm = gat_colsum(gzd) if ctx.has_bias[0] else None
        gbu = (colsum if colsum is not None else g.float().sum(0)) if ctx.has_bias[1] else None
        return g_feat, None, None, gw_m.to(w_m.dtype), gbm, gw_u.to(w_u.dtype), gbu, None


def pna_layer(feat, graph, delta, w_m, b_m, w_u, b_u, drop_bwd=None) -> torch.Tensor:
    return PnaLayerFn.apply(feat, graph, float(delta), w_m, b_m, w_u, b_u, drop_bwd)


# ---- softmax-aggregation graph convolution, GENConv (csrc/genconv.cu) ---------------------------------------
GENCONV_DT_PARTIALS = 264          # PG_GENCONV_DT_PARTIALS of include/pipegcn_b200.h


def genconv_preload():
    """Load every GENConv kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_genconv_preload(), "pg_genconv_preload")


def genconv_aggregate(plan: CsrPlan, xs: torch.Tensor, xd: torch.Tensor, t: torch.Tensor, keep=None, num_in: int = 0,
                      stats: bool = True, learn_t: bool = False):
    """(S, agg, lse, var) over the forward CSR `plan` (pg_genconv_aggregate): S [n_rows, d] in xs's dtype = the
    per-channel softmax aggregate of ReLU(xs) + 1e-7 with temperature t (fp32 [1] on the device) plus xd; agg and
    lse = log sum exp(t m) [n_rows, d] fp32 when `stats`, var [n_rows, d] fp32 when `stats` and `learn_t` (None
    otherwise).  `keep`: uint8 keep mask of the halo rows (rows >= num_in of xs), or None."""
    _rows(xs), _rows(xd)
    n, d = plan.n_rows, xs.shape[1]
    assert xd.dtype == xs.dtype and xd.shape == (n, d) and t.dtype == torch.float32 and t.is_cuda
    dev = xs.device
    s = alloc_rows(n, d, xs.dtype, dev)
    agg = lse = var = None
    if stats:
        agg, lse = alloc_rows(n, d, torch.float32, dev), alloc_rows(n, d, torch.float32, dev)
        if learn_t:
            var = alloc_rows(n, d, torch.float32, dev)
    parts = 4 if var is not None else 3
    scratch = plan.scratch(parts * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_genconv_aggregate(C.byref(plan.c), xs.data_ptr(), xs.stride(0), xd.data_ptr(), xd.stride(0), d,
                                         _C.dtype_code(xs.dtype), t.data_ptr(), _ptr(keep), int(num_in), s.data_ptr(),
                                         s.stride(0), _ptr(agg), agg.stride(0) if stats else 0, _ptr(lse),
                                         lse.stride(0) if stats else 0, _ptr(var),
                                         var.stride(0) if var is not None else 0, _ptr(scratch),
                                         _scratch_ld(parts * d), _C.stream_ptr()), "pg_genconv_aggregate")
    return s, agg, lse, var


def genconv_bwd_dst(gs: torch.Tensor, agg: torch.Tensor, t: torch.Tensor, var: torch.Tensor = None, dtype=None):
    """(Q, gst, dt) from g_S [n, d] fp32 (pg_genconv_bwd_dst): Q = t g_S agg fp32; gst = g_S rounded to `dtype` (None
    when dtype is None); dt = sum g_S var as an fp32 [1] device tensor when var is given, else None."""
    n, d = gs.shape
    dev = gs.device
    q = alloc_rows(n, d, torch.float32, dev)
    gst = alloc_rows(n, d, dtype, dev) if dtype is not None else None
    dt = partial = None
    if var is not None:
        dt = torch.empty(1, dtype=torch.float32, device=dev)
        partial = torch.empty(GENCONV_DT_PARTIALS, dtype=torch.float64, device=dev)
    _C.count(2 if var is not None else 1)
    _C.check(_C.lib.pg_genconv_bwd_dst(gs.data_ptr(), gs.stride(0), agg.data_ptr(), agg.stride(0), _ptr(var),
                                       var.stride(0) if var is not None else 0, t.data_ptr(), n, d,
                                       _C.dtype_code(dtype if dtype is not None else torch.float32), q.data_ptr(),
                                       q.stride(0), _ptr(gst), gst.stride(0) if gst is not None else 0, _ptr(partial),
                                       _ptr(dt), _C.stream_ptr()), "pg_genconv_bwd_dst")
    return q, gst, dt


def genconv_bwd_src(plan_t: CsrPlan, xs: torch.Tensor, t: torch.Tensor, lse, gs, q, keep=None, num_in: int = 0,
                    add: torch.Tensor = None, drop: DropSpec = None) -> torch.Tensor:
    """dx [plan_t.n_rows, d] in xs's dtype over the CSC `plan_t` (pg_genconv_bwd_src): the gradient of x_src, plus
    `add` (fp32) on its first add.shape[0] rows, through the dropout backward of `drop` when given."""
    _rows(xs)
    d = xs.shape[1]
    dx = alloc_rows(plan_t.n_rows, d, xs.dtype, xs.device)
    scratch = plan_t.scratch(d)
    drop = drop if drop is not None and drop.p > 0 else None
    _C.count(2 if plan_t.n_long else 1)
    _C.check(_C.lib.pg_genconv_bwd_src(C.byref(plan_t.c), xs.data_ptr(), xs.stride(0), t.data_ptr(), _ptr(keep),
                                       int(num_in), lse.data_ptr(), lse.stride(0), gs.data_ptr(), gs.stride(0),
                                       q.data_ptr(), q.stride(0), _ptr(add), add.stride(0) if add is not None else 0,
                                       add.shape[0] if add is not None else 0,
                                       C.byref(drop.c()) if drop is not None else None, d, _C.dtype_code(xs.dtype),
                                       dx.data_ptr(), dx.stride(0), _ptr(scratch), _scratch_ld(d), _C.stream_ptr()),
             "pg_genconv_bwd_src")
    return dx


class GenConvLayerFn(torch.autograd.Function):
    """One GENConv layer (PyG GENConv, aggr='softmax', scalar temperature t, no edge features, no message norm, MLP
    [d, 2d, d] without norm or bias) over the [inner | halo] rows `feat` of a partition, returning the inner rows:

        x_src = feat @ W_src^T   (or feat when d_in == d)   [num_all, d]    pg_linear over all rows
        x_dst = feat[:N_in] @ W_dst^T  (or feat[:N_in])     [N_in, d]       pg_linear over the inner rows
        S = softmax_aggregate(ReLU(x_src) + 1e-7) + x_dst   [N_in, d]       pg_genconv_aggregate (+ agg, L, var)
        R = ReLU(S @ W1^T)                                  [N_in, 2d]      pg_linear, pg_gcnii_relu_drop
        out = R @ W2^T                                      [N_in, d]       pg_linear

    Backward: g_R = g @ W2 (pg_linear), g_H = ReLU'(R) g_R (pg_gcnii_relu_bwd), g_S = g_H @ W1 (fp32, pg_linear);
    Q, g_S in the activation dtype and dt (pg_genconv_bwd_dst); dx_src over the CSC (pg_genconv_bwd_src); then
    g_feat = dx_src @ W_src (+ g_S @ W_dst on the inner rows) as one two-source pg_linear with the dropout backward of
    `drop_bwd` in its epilogue, or, when d_in == d, dx_src + g_S on the inner rows written by the source pass itself,
    dropout backward included; dW2 = g^T R, dW1 = g_H^T S, dW_src = dx_src^T feat, dW_dst = g_S^T feat[:N_in]
    (pg_wgrad).  `t` is an fp32 [1] device tensor read by the kernels (a CUDA graph sees its updates); its gradient dt
    is returned when it requires one.  `keep`: the boundary-node sample of the halo rows (uint8), or None."""

    @staticmethod
    def forward(ctx, feat, graph, keep, t, w_src, w_dst, w1, w2, drop_bwd=None, train=True):
        ctx.drop_bwd = drop_bwd
        proj = w_src is not None
        if not proj:
            # feat is x_src itself: the kernels read whole 16-byte vectors of 16-byte aligned rows (a contiguous [N, d]
            # tensor of an unaligned width, as whole-graph evaluation passes between layers, is copied to padded rows)
            feat = _tma_ready(feat)
        elif feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in, dt_ = graph.num_in, feat.dtype
        fsp = presplit(feat) if proj else feat
        finner = fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in]
        xs = gemm_nt(fsp, padded_weight(w_src, dt_)) if proj else feat
        xd = gemm_nt(finner, padded_weight(w_dst, dt_)) if proj else feat[:n_in]
        keep_stats = train and any(ctx.needs_input_grad)
        learn_t = keep_stats and ctx.needs_input_grad[3]
        s, agg, lse, var = genconv_aggregate(graph.fwd, xs, xd, t, keep, n_in, stats=keep_stats, learn_t=learn_t)
        del xd
        r, _ = gcnii_relu_drop(gemm_nt(s, padded_weight(w1, dt_)))
        out = gemm_nt(r, padded_weight(w2, dt_))
        if keep_stats:
            ctx.save_for_backward(feat, xs, s, agg, lse, var, r, t, w_src, w_dst, w1, w2)
            ctx.graph, ctx.keep, ctx.proj = graph, keep, proj
        return out

    @staticmethod
    def backward(ctx, g):
        feat, xs, s, agg, lse, var, r, t, w_src, w_dst, w1, w2 = ctx.saved_tensors
        graph, keep, proj = ctx.graph, ctx.keep, ctx.proj
        n_in, n_all, d = graph.num_in, feat.shape[0], xs.shape[1]
        dt_ = feat.dtype
        g = _tma_ready(g if g.dtype == dt_ else g.to(dt_))
        gsp = presplit(g)
        gh = gcnii_relu_bwd(gemm_nt(gsp, padded_weight(w2, dt_, transpose=True)), r)
        ghsp = presplit(gh)
        gs = gemm_nt(ghsp, padded_weight(w1, dt_, transpose=True), out_dtype=torch.float32)
        gw2 = wgrad(gsp, presplit(r)).to(w2.dtype)
        gw1 = wgrad(ghsp, presplit(s)).to(w1.dtype)
        del gh, ghsp
        q, gst, d_t = genconv_bwd_dst(gs, agg, t, var if ctx.needs_input_grad[3] else None,
                                      dtype=dt_ if proj and dt_ != torch.float32 else None)
        need_feat = ctx.needs_input_grad[0]
        drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
        g_feat = gw_src = gw_dst = None
        if not proj:
            # x_src = feat: the source pass adds g_S on the inner rows and applies the dropout backward itself
            g_feat = genconv_bwd_src(graph.bwd, xs, t, lse, gs, q, keep, n_in, add=gs, drop=drop) if need_feat else None
        else:
            dxs = genconv_bwd_src(graph.bwd, xs, t, lse, gs, q, keep, n_in)
            gst = gst if gst is not None else gs
            dxsp, gstsp = presplit(dxs), presplit(gst)
            if need_feat:
                g_feat = alloc_rows(n_all, feat.shape[1], dt_, feat.device)
                db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
                gemm_nt(dxsp.rows(0, n_in) if isinstance(dxsp, Split) else dxs[:n_in],
                        padded_weight(w_src, dt_, transpose=True), gstsp, padded_weight(w_dst, dt_, transpose=True),
                        out=g_feat[:n_in], drop=db)
                if n_all > n_in:
                    gemm_nt(dxsp.rows(n_in) if isinstance(dxsp, Split) else dxs[n_in:],
                            padded_weight(w_src, dt_, transpose=True), out=g_feat[n_in:], drop=db, drop_row0=n_in)
                if drop is not None and db is None:
                    dropout_rows(g_feat, drop, out=g_feat)
            fsp = presplit(feat)
            gw_src = wgrad(dxsp, fsp).to(w_src.dtype)
            gw_dst = wgrad(gstsp, fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in]).to(w_dst.dtype)
        return g_feat, None, None, d_t, gw_src, gw_dst, gw1, gw2, None, None


def genconv_layer(feat, graph, keep, t, w_src, w_dst, w1, w2, drop_bwd=None) -> torch.Tensor:
    """GENConv layer (GenConvLayerFn); w_src and w_dst None when d_in == d.  `t`: fp32 [1] on the device."""
    return GenConvLayerFn.apply(feat, graph, keep, t, w_src, w_dst, w1, w2, drop_bwd, torch.is_grad_enabled())


# ---- residual gated graph convolution, ResGatedGraphConv (csrc/resgated.cu) --------------------------------
def resgated_preload():
    """Load every ResGatedGCN kernel now (see gat_preload)."""
    _C.check(_C.lib.pg_resgated_preload(), "pg_resgated_preload")


def resgated_aggregate(graph: PartGraph, qv, ks, d: int, half: int, keep=None):
    """out [N_in, d] in qv's dtype = skip[v] + sum_u sigmoid(k[v] + q[u]) val[u] over the forward CSR
    (pg_resgated_aggregate); qv = [q | val] [num_all, >= half + d] and ks = [k | skip] [N_in, >= half + d] with the
    second halves at column `half`."""
    plan = graph.fwd
    out = alloc_rows(plan.n_rows, d, qv.dtype, qv.device)
    scratch = plan.scratch(d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_resgated_aggregate(C.byref(plan.c), qv.data_ptr(), qv.stride(0), ks.data_ptr(), ks.stride(0),
                                          int(half), int(d), _C.dtype_code(qv.dtype), _ptr(keep), graph.num_in,
                                          out.data_ptr(), out.stride(0), _ptr(scratch), _scratch_ld(d),
                                          _C.stream_ptr()), "pg_resgated_aggregate")
    return out


def resgated_bwd_dst(graph: PartGraph, qv, ks, g, d: int, half: int, keep=None, dkg=None):
    """[dk | g] [N_in, 2 half] in qv's dtype over the forward CSR (pg_resgated_bwd_dst): dk[v] = g[v] sum_u
    sigmoid'(k[v] + q[u]) val[u] at [0, d), a copy of g at [half, half + d).  `dkg`: the tensor to write (allocated
    when None, with zero pad columns)."""
    plan = graph.fwd
    if dkg is None:
        dkg = alloc_rows(plan.n_rows, 2 * half, qv.dtype, qv.device, zero=half != d)
    scratch = plan.scratch(d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_resgated_bwd_dst(C.byref(plan.c), qv.data_ptr(), qv.stride(0), ks.data_ptr(), ks.stride(0),
                                        int(half), g.data_ptr(), g.stride(0), int(d), _C.dtype_code(qv.dtype),
                                        _ptr(keep), graph.num_in, dkg.data_ptr(), dkg.stride(0), _ptr(scratch),
                                        _scratch_ld(d), _C.stream_ptr()), "pg_resgated_bwd_dst")
    return dkg


def resgated_bwd_src(graph: PartGraph, qv, ks, g, d: int, half: int, keep=None, dqv=None):
    """[dq | dval] [num_all, 2 half] in qv's dtype over the CSC of the graph (pg_resgated_bwd_src): dq[u] = val[u]
    sum_v g[v] sigmoid'(k[v] + q[u]) at [0, d), dval[u] = sum_v g[v] sigmoid(k[v] + q[u]) at [half, half + d); 0 on
    unkept halo rows.  `dqv`: the tensor to write (allocated when None, with zero pad columns)."""
    plan = graph.bwd
    if dqv is None:
        dqv = alloc_rows(plan.n_rows, 2 * half, qv.dtype, qv.device, zero=half != d)
    scratch = plan.scratch(2 * d)
    _C.count(2 if plan.n_long else 1)
    _C.check(_C.lib.pg_resgated_bwd_src(C.byref(plan.c), qv.data_ptr(), qv.stride(0), ks.data_ptr(), ks.stride(0),
                                        int(half), g.data_ptr(), g.stride(0), int(d), _C.dtype_code(qv.dtype),
                                        _ptr(keep), graph.num_in, dqv.data_ptr(), dqv.stride(0), _ptr(scratch),
                                        _scratch_ld(2 * d), _C.stream_ptr()), "pg_resgated_bwd_src")
    return dqv


class ResGatedLayerFn(torch.autograd.Function):
    """One residual gated graph convolution (PyG ResGatedGraphConv, act=Sigmoid, root_weight=True, bias=True, no edge
    features) over the [inner | halo] rows `feat` of a partition, returning the inner rows.  With W the half width of
    transformer_width:

        [q | val]  = feat @ [W_q; W_v]^T + [b_q; b_v]          [num_all, 2W]   one pg_linear over all rows
        [k | skip] = feat[:N_in] @ [W_k; W_s]^T + [b_k; b]     [N_in, 2W]      one pg_linear over the inner rows
        out[v] = skip[v] + sum_u sigmoid(k[v] + q[u]) val[u]   [N_in, d]       pg_resgated_aggregate

    Backward: [dk | g] (pg_resgated_bwd_dst over the CSR), [dq | dval] (pg_resgated_bwd_src over the CSC), the bias
    gradients as fixed-order column sums (b from the column sum the LayerNorm backward stashed, when there is one), the
    weight gradients as one pg_wgrad per row set, and g_feat = [dq | dval] @ [W_q; W_v] (+ [dk | g] @ [W_k; W_s] on the
    inner rows, one two-source pg_linear), with the dropout backward of `drop_bwd` in its epilogue.  `keep`: the
    boundary-node sample of the halo rows (uint8), or None."""

    @staticmethod
    def forward(ctx, feat, graph, keep, w_k, b_k, w_q, b_q, w_v, b_v, w_s, bias, drop_bwd=None):
        ctx.drop_bwd = drop_bwd
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        n_in, d = graph.num_in, w_q.shape[0]
        w = transformer_width(d, feat.dtype)
        fsp = presplit(feat)                   # fp32: one split of feat for both products
        qv = gemm_nt(fsp, _pair_weight(w_q, w_v, w, feat.dtype), bias=_pair_bias(b_q, b_v, d, w))
        ks = gemm_nt(fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in],
                     _pair_weight(w_k, w_s, w, feat.dtype), bias=_pair_bias(b_k, bias, d, w))
        out = resgated_aggregate(graph, qv, ks, d, w, keep)
        ctx.save_for_backward(feat, qv, ks, w_k, w_q, w_v, w_s)
        ctx.graph, ctx.keep, ctx.width = graph, keep, w
        return out

    @staticmethod
    def backward(ctx, g):
        feat, qv, ks, w_k, w_q, w_v, w_s = ctx.saved_tensors
        graph, keep, w = ctx.graph, ctx.keep, ctx.width
        n_in, n_all, d = graph.num_in, feat.shape[0], w_q.shape[0]
        colsum = _take_colsum(g)
        g = _tma_ready(g if g.dtype == feat.dtype else g.to(feat.dtype))
        dkg = resgated_bwd_dst(graph, qv, ks, g, d, w, keep)
        dqv = resgated_bwd_src(graph, qv, ks, g, d, w, keep)
        gb_qv = gat_colsum(dqv)
        if colsum is not None:
            gbk, gb = gat_colsum(dkg[:, :d]), colsum
        else:
            gb_ks = gat_colsum(dkg)
            gbk, gb = gb_ks[:d], gb_ks[w:w + d]
        dqvp, dkgp = presplit(dqv), presplit(dkg)
        is_split = isinstance(dqvp, Split)
        g_feat = None
        if ctx.needs_input_grad[0]:
            g_feat = alloc_rows(n_all, feat.shape[1], feat.dtype, feat.device)
            wqv = _pair_weight(w_q, w_v, w, feat.dtype, transpose=True)
            drop = ctx.drop_bwd if ctx.drop_bwd is not None and ctx.drop_bwd.p > 0 else None
            db = drop if drop is not None and feat.shape[1] <= 256 and _drop_ok(g_feat) else None
            gemm_nt(dqvp.rows(0, n_in) if is_split else dqv[:n_in], wqv, dkgp,
                    _pair_weight(w_k, w_s, w, feat.dtype, transpose=True), out=g_feat[:n_in], drop=db)
            if n_all > n_in:
                gemm_nt(dqvp.rows(n_in) if is_split else dqv[n_in:], wqv, out=g_feat[n_in:], drop=db, drop_row0=n_in)
            if drop is not None and db is None:
                dropout_rows(g_feat, drop, out=g_feat)
        fsp = presplit(feat)
        gw_qv = wgrad(dqvp, fsp)
        gw_ks = wgrad(dkgp, fsp.rows(0, n_in) if isinstance(fsp, Split) else feat[:n_in])
        gwk, gwq, gwv, gws = [t.contiguous() for t in (gw_ks[:d], gw_qv[:d], gw_qv[w:w + d], gw_ks[w:w + d])]
        return (g_feat, None, None, gwk.to(w_k.dtype), gbk.contiguous(), gwq.to(w_q.dtype), gb_qv[:d].contiguous(),
                gwv.to(w_v.dtype), gb_qv[w:w + d].contiguous(), gws.to(w_s.dtype), gb.contiguous(), None)


def resgated_layer(feat, graph, keep, w_k, b_k, w_q, b_q, w_v, b_v, w_s, bias, drop_bwd=None) -> torch.Tensor:
    return ResGatedLayerFn.apply(feat, graph, keep, w_k, b_k, w_q, b_q, w_v, b_v, w_s, bias, drop_bwd)


# ---- row-wise epilogues (csrc/rowops.cu) -------------------------------------------------------------------
# column sums of a gradient tensor computed as a by-product by the kernel that produced it, keyed by the
# tensor's address: the bias gradient of the linear upstream (saves a full pass over [N, d])
_COLSUM = {}


def _stash_colsum(t: torch.Tensor, colsum: torch.Tensor):
    if len(_COLSUM) > 64:
        _COLSUM.clear()
    _COLSUM[(t.data_ptr(), tuple(t.shape))] = colsum


def reset_colsum():
    """Drop by-products of an earlier backward (called at the start of every backward pass): an entry that was
    never consumed must not be picked up by a later gradient that happens to reuse the address."""
    _COLSUM.clear()


def _take_colsum(t: torch.Tensor):
    return _COLSUM.pop((t.data_ptr(), tuple(t.shape)), None)


def ln_relu_supported(y: torch.Tensor) -> bool:
    v = 16 // y.element_size()
    d = y.shape[1]
    return y.is_cuda and y.dim() == 2 and d % v == 0 and d // v <= 128 and y.stride(1) == 1 \
        and (y.stride(0) * y.element_size()) % 16 == 0 and y.data_ptr() % 16 == 0


class LayerNormReLU(torch.autograd.Function):
    """relu(LayerNorm(y)) in one pass (model.py:53-56); the backward also yields d gamma, d beta and the column
    sums of g_y, which is the bias gradient of the linear that produced y."""

    @staticmethod
    def forward(ctx, y, gamma, beta, eps, relu, out, clean=None, drop=None):
        # clean / drop: `out` receives dropout(result) under the key `drop` (the next layer's dropout, fused), `clean`
        # the result itself (source of the halo push, ReLU mask of the backward)
        n, d = y.shape
        if out is None:
            out = alloc_rows(n, d, y.dtype, y.device)
        mean = torch.empty(n, dtype=torch.float32, device=y.device)
        rstd = torch.empty(n, dtype=torch.float32, device=y.device)
        g32, b32 = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
        _C.count()
        if clean is not None or drop is not None:
            _C.check(_C.lib.pg_ln_relu_drop_fwd(y.data_ptr(), y.stride(0), g32.data_ptr(), b32.data_ptr(), float(eps),
                                                int(relu), out.data_ptr(), out.stride(0),
                                                clean.data_ptr() if clean is not None else None,
                                                clean.stride(0) if clean is not None else 0,
                                                mean.data_ptr(), rstd.data_ptr(), n, d, _C.dtype_code(y.dtype),
                                                C.byref(drop.c()) if drop is not None else None, _C.stream_ptr()),
                     "pg_ln_relu_drop_fwd")
        else:
            _C.check(_C.lib.pg_ln_relu_fwd(y.data_ptr(), y.stride(0), g32.data_ptr(), b32.data_ptr(), float(eps), int(relu),
                                           out.data_ptr(), out.stride(0), mean.data_ptr(), rstd.data_ptr(), n, d,
                                           _C.dtype_code(y.dtype), _C.stream_ptr()), "pg_ln_relu_fwd")
        ctx.save_for_backward(y, mean, rstd, g32, b32)
        ctx.relu = bool(relu)
        ctx.param_dtype = gamma.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        y, mean, rstd, g32, b32 = ctx.saved_tensors
        n, d = y.shape
        if g.dtype != y.dtype or g.stride(1) != 1 or (g.stride(0) * g.element_size()) % 16 or g.data_ptr() % 16:
            g = _tma_ready(g.to(y.dtype))
        g_y = alloc_rows(n, d, y.dtype, y.device)
        grid = _C.lib.pg_row_grid(n)
        partial = torch.empty(grid * 3 * d, dtype=torch.float32, device=y.device)
        red = torch.empty(3, d, dtype=torch.float32, device=y.device)
        _C.count(2)
        # the ReLU mask is recomputed from y (beta given): the forward output is neither kept nor read
        _C.check(_C.lib.pg_ln_relu_bwd2(g.data_ptr(), g.stride(0), None, 0, y.data_ptr(), y.stride(0),
                                        mean.data_ptr(), rstd.data_ptr(), g32.data_ptr(), b32.data_ptr(), int(ctx.relu),
                                        g_y.data_ptr(), g_y.stride(0), red[0].data_ptr(), red[1].data_ptr(),
                                        red[2].data_ptr(), partial.data_ptr(), n, d, _C.dtype_code(y.dtype),
                                        _C.stream_ptr()), "pg_ln_relu_bwd")
        _stash_colsum(g_y, red[2])
        return g_y, red[0].to(ctx.param_dtype), red[1].to(ctx.param_dtype), None, None, None, None, None


def layer_norm_relu(y, gamma, beta, eps=1e-5, relu=True, out=None, clean=None, drop=None):
    return LayerNormReLU.apply(y, gamma, beta, eps, relu, out, clean, drop)


class KeyedDropout(torch.autograd.Function):
    """dropout(x) under an explicit key, forward and backward (the un-fused form of what the fused producers do:
    PG_FUSED_DROPOUT=0, and the reference the fused kernels are tested against)."""

    @staticmethod
    def forward(ctx, x, spec):
        ctx.spec = spec
        return dropout_rows(x, spec)

    @staticmethod
    def backward(ctx, g):
        if not _drop_ok(g):
            gp = alloc_rows(g.shape[0], g.shape[1], g.dtype, g.device)
            gp.copy_(g)
            g = gp
        return dropout_rows(g, ctx.spec, out=g), None


def keyed_dropout(x, spec: DropSpec):
    return KeyedDropout.apply(x, spec) if spec.p > 0 else x


# dropout of graph layers >= 1 applied by the producers of the dropped tensor (LayerNorm epilogue, halo push,
# transposed aggregate) instead of by [num_all, d] passes; PG_FUSED_DROPOUT=0: the same masks by separate passes
FUSED_DROPOUT = os.environ.get("PG_FUSED_DROPOUT", "1") != "0"


class CrossEntropySum(torch.autograd.Function):
    """CrossEntropyLoss(reduction='sum') over the first n_train rows of the logits (train.py:320,351); the gradient
    is zero on the remaining rows (train rows come first after move_train_first)."""

    @staticmethod
    def forward(ctx, logits, labels, n_train):
        n, c = logits.shape
        dev = logits.device
        lse = torch.empty(max(n_train, 1), dtype=torch.float32, device=dev)
        grid = _C.lib.pg_row_grid(max(n, 1))
        partial = torch.empty(grid * max(c, 1), dtype=torch.float32, device=dev)
        loss = torch.zeros(1, dtype=torch.float32, device=dev)
        if n_train:
            _C.count(2)
            _C.check(_C.lib.pg_ce_fwd(logits.data_ptr(), logits.stride(0), labels.data_ptr(), n_train, c,
                                      _C.dtype_code(logits.dtype), lse.data_ptr(), partial.data_ptr(), loss.data_ptr(),
                                      _C.stream_ptr()), "pg_ce_fwd")
        ctx.save_for_backward(logits, labels, lse, partial)
        ctx.n_train = n_train
        return loss[0]

    @staticmethod
    def backward(ctx, up):
        logits, labels, lse, partial = ctx.saved_tensors
        n, c = logits.shape
        g = alloc_rows(n, c, logits.dtype, logits.device)
        colsum = torch.empty(c, dtype=torch.float32, device=logits.device)
        up = up.detach().float().reshape(1).contiguous()
        _C.count(2)
        _C.check(_C.lib.pg_ce_bwd(logits.data_ptr(), logits.stride(0), labels.data_ptr(), lse.data_ptr(), up.data_ptr(),
                                  ctx.n_train, n, c, _C.dtype_code(logits.dtype), g.data_ptr(), g.stride(0),
                                  colsum.data_ptr(), partial.data_ptr(), _C.stream_ptr()), "pg_ce_bwd")
        _stash_colsum(g, colsum)
        return g, None, None


def cross_entropy_sum(logits, labels, n_train):
    if logits.stride(1) != 1:
        logits = logits.contiguous()
    return CrossEntropySum.apply(logits, labels, int(n_train))


def eval_count(logits: torch.Tensor, labels: torch.Tensor = None, tag: torch.Tensor = None, n_tags: int = 0,
               want_pred: bool = False):
    """(counts, pred): counts [n_tags, 2] int64 = (correct, total) of every mask k (rows whose `tag` has bit k), with
    torch.argmax(logits, 1) as the prediction; pred [N] int32 (or None).  One kernel, the logits stay on the device."""
    if n_tags and labels.dim() != 1:
        # as calc_acc: the multi-label (yelp) F1 evaluation is not implemented
        raise NotImplementedError("multi-label (yelp) evaluation is out of scope")
    if logits.dim() != 2 or (logits.shape[1] > 1 and logits.stride(1) != 1) or not logits.is_cuda:
        raise _C.PgError(f"eval_count: expected row-major CUDA logits, got {tuple(logits.shape)} {logits.stride()}")
    n, c = logits.shape
    dev = logits.device
    counts = torch.empty(max(n_tags, 1), 2, dtype=torch.int64, device=dev)
    pred = torch.empty(n, dtype=torch.int32, device=dev) if want_pred else None
    if n_tags:
        labels, tag = labels.contiguous(), tag.contiguous()
        assert labels.dtype == torch.int64 and tag.dtype == torch.uint8 and labels.numel() == n and tag.numel() == n
    _C.count()
    _C.check(_C.lib.pg_eval_count(logits.data_ptr(), logits.stride(0), n, c, _C.dtype_code(logits.dtype),
                                  labels.data_ptr() if n_tags else None, tag.data_ptr() if n_tags else None,
                                  int(n_tags), pred.data_ptr() if pred is not None else None,
                                  counts.data_ptr() if n_tags else None, _C.stream_ptr()), "pg_eval_count")
    return counts[:n_tags], pred


class Dropout(torch.autograd.Function):
    """Dropout whose mask is regenerated from (seed, element index) in the backward (csrc/rowops.cu)."""

    @staticmethod
    def forward(ctx, x, p, seed):
        out = alloc_rows(x.shape[0], x.shape[1], x.dtype, x.device)
        _C.count()
        step = STEP_DEV.data_ptr() if STEP_DEV is not None else None
        _C.check(_C.lib.pg_dropout(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), x.shape[0], x.shape[1],
                                   _C.dtype_code(x.dtype), float(p), int(seed), step, _C.stream_ptr()), "pg_dropout")
        ctx.p, ctx.seed, ctx.step = p, seed, step
        return out

    @staticmethod
    def backward(ctx, g):
        if g.stride(1) != 1 or (g.stride(0) * g.element_size()) % 16 or g.data_ptr() % 16 \
                or g.stride(0) < (g.shape[1] + 7) // 8 * 8:
            gp = alloc_rows(g.shape[0], g.shape[1], g.dtype, g.device)
            gp.copy_(g)
            g = gp
        _C.count()
        _C.check(_C.lib.pg_dropout(g.data_ptr(), g.stride(0), g.data_ptr(), g.stride(0), g.shape[0], g.shape[1],
                                   _C.dtype_code(g.dtype), float(ctx.p), int(ctx.seed), ctx.step, _C.stream_ptr()),
                 "pg_dropout")
        return g, None, None


_dropout_calls = 0
# device int32 step counter mixed into every dropout seed (set while epochs are replayed from a CUDA graph, where
# the host-side call counter is frozen at capture time)
STEP_DEV = None


def dropout(x: torch.Tensor, p: float, training: bool = True) -> torch.Tensor:
    """model.py:47.  Padded, 16-byte aligned rows go through the mask-free kernel; anything else through torch."""
    global _dropout_calls
    if not training or p == 0.0:
        return x
    ld_ok = x.dim() == 2 and x.is_cuda and x.stride(1) == 1 and (x.stride(0) * x.element_size()) % 16 == 0 \
        and x.data_ptr() % 16 == 0 and x.stride(0) >= (x.shape[1] + 7) // 8 * 8 and x.dtype in (torch.float32, torch.bfloat16)
    if not ld_ok:
        return torch.nn.functional.dropout(x, p, True)
    _dropout_calls += 1
    seed = (torch.initial_seed() * 0x9E3779B97F4A7C15 + _dropout_calls * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF
    return Dropout.apply(x, p, seed)
