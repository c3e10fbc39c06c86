"""torch-facing wrappers of the C-ABI kernels (PyTorch tensors in, PyTorch tensors out).

Each autograd Function mirrors one step of the reference's module/layer.py:44-51 and
its autograd; nothing here computes on the host or falls back to torch kernels for
the aggregate / exchange path.
"""
from __future__ import annotations

import ctypes as C
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
    raw = [(a0, b0)] + ([(a1, b1)] if a1 is not None else [])
    a0, b0 = _plain(a0), _plain(b0)
    pairs = [(_rows(_plain(a)), _rows(_plain(b))) for a, b in raw]
    m, n = a0.shape[0], b0.shape[0]
    for a, b in pairs:
        assert a.shape[0] == m and b.shape[0] == n and a.shape[1] == b.shape[1] and a.dtype == b.dtype == a0.dtype
    if n > 256:
        # one N tile holds at most 256 columns: split the weight rows, each product writing its 256-column slice of
        # one output (padded rows like every other output: 16-byte aligned, usable by the row kernels and TMA)
        assert drop is None or drop.p == 0, "fused dropout with n > 256 is not supported"
        if out is None:
            out = alloc_rows(m, n, out_dtype or a0.dtype, a0.device)
        assert out.shape == (m, n) and out.stride(1) == 1
        for i in range(0, n, 256):
            gemm_nt(raw[0][0], b0[i:i + 256], raw[1][0] if len(raw) > 1 else None,
                    None if len(raw) == 1 else _plain(raw[1][1])[i:i + 256],
                    None if bias is None else bias[i:i + 256], row_div, out[:, i:i + 256], out_dtype)
        return out
    if out is None:
        out = alloc_rows(m, n, out_dtype or a0.dtype, a0.device)
    assert out.shape == (m, n) and out.stride(1) == 1
    if m == 0:
        return out
    if a0.dtype == torch.float32 and FP32_GEMM == "3xtf32":
        split = []
        for a, b in raw:
            (ah, al), (bh, bl) = _halves(a), _halves(b)
            split += [(ah, bh), (ah, bl), (al, bh)]
        pairs = split
    else:
        pairs = [(_tma_ready(a), _tma_ready(b)) for a, b in pairs]
    srcs = (_C.pg_gemm_src * len(pairs))(*[_C.pg_gemm_src(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                                                            a.shape[1]) for a, b in pairs])
    if bias is not None:
        bias = bias.detach().to(torch.float32).contiguous()
    _C.count()
    if drop is not None and drop.p > 0:
        _C.check(_C.lib.pg_linear_drop(_C.dtype_code(a0.dtype), _C.dtype_code(out.dtype), srcs, len(pairs),
                                       bias.data_ptr() if bias is not None else None,
                                       row_div.data_ptr() if row_div is not None else None,
                                       out.data_ptr(), out.stride(0), m, n, C.byref(drop.c()), int(drop_row0),
                                       _C.stream_ptr()), "pg_linear_drop")
        return out
    _C.check(_C.lib.pg_linear(_C.dtype_code(a0.dtype), _C.dtype_code(out.dtype), srcs, len(pairs),
                              bias.data_ptr() if bias is not None else None,
                              row_div.data_ptr() if row_div is not None else None,
                              out.data_ptr(), out.stride(0), m, n, _C.stream_ptr()), "pg_linear")
    return out


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
    g, x = _rows(_plain(g)), _rows(_plain(x))
    m, n, k = g.shape[0], g.shape[1], x.shape[1]
    assert x.shape[0] == m and g.dtype == x.dtype
    out = torch.empty(n, k, dtype=torch.float32, device=g.device)
    if m == 0:
        return out.zero_()
    if g.dtype == torch.float32 and FP32_GEMM == "3xtf32":
        # fp32 = b0 + b1 + b2 exactly (three bf16 terms): six bf16 products carry the product to ~2^-24
        g3, x3 = _split_bf16(g, 3), _split_bf16(x, 3)
        pairs = [(g3[0], x3[0]), (g3[0], x3[1]), (g3[1], x3[0]), (g3[0], x3[2]), (g3[2], x3[0]), (g3[1], x3[1])]
    elif g.dtype == torch.float32:
        # one-pass mode: two bf16 terms, three products (~2^-16, finer than one tf32 pass)
        g2, x2 = _split_bf16(g, 2), _split_bf16(x, 2)
        pairs = [(g2[0], x2[0]), (g2[0], x2[1]), (g2[1], x2[0])]
    else:
        pairs = [(_tma_ready(g), _tma_ready(x))]
    code = _C.dtype_code(pairs[0][0].dtype)
    for n0 in range(0, n, 256):
        for k0 in range(0, k, 256):
            nn, kk = min(256, n - n0), min(256, k - k0)
            # split-K partials: a fresh block per call (the caching allocator is stream-aware; several simulated
            # ranks run on their own streams in one process and must not share scratch)
            ws = torch.empty(int(_C.lib.pg_wgrad_workspace(m, nn, kk, code)), dtype=torch.float32, device=g.device)
            es = pairs[0][0].element_size()
            srcs = (_C.pg_gemm_src * len(pairs))(*[
                _C.pg_gemm_src(a.data_ptr() + n0 * es, a.stride(0), b.data_ptr() + k0 * es, b.stride(0), m)
                for a, b in pairs])
            o = out[n0:n0 + nn, k0:k0 + kk]
            _C.count(2)
            _C.check(_C.lib.pg_wgrad(code, srcs, len(pairs), o.data_ptr(), o.stride(0), m, nn, kk, ws.data_ptr(),
                                     ws.numel(), _C.stream_ptr()), "pg_wgrad")
    return out


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

        g_feat[:N_in] = g @ W1                            pg_linear
        gs            = (g @ W2) / in_deg                 pg_linear with the row scale fused
        g_feat       += A^T @ gs                          pg_aggregate accumulating into rows < N_in
        gW1 = g^T feat[:N_in], gW2 = g^T ah, gb = sum g   library GEMM / reduction
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
            gemm_nt(gsp, padded_weight(w1, x.dtype, transpose=True), out=g_feat[:graph.num_in])
            gs = gemm_nt(gsp, padded_weight(w2, x.dtype, transpose=True), row_div=deg_f)
            aggregate(graph.bwd, gs, out=g_feat, acc_rows=graph.num_in, drop=ctx.drop_bwd)
        gw1 = wgrad(gsp, x).to(w1.dtype)
        gw2 = wgrad(gsp, ah).to(w2.dtype)
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
        gw1 = wgrad(gsp, fsp.rows(0, n_in) if is_split else feat[:n_in]).to(w1.dtype)
        gw2 = wgrad(dzsp, fsp).to(w2.dtype)
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
