"""`Buffer`: the halo feature / gradient exchange of one rank, NVLink-native.

Same public surface as PipeGCN/helper/feature_buffer.py (`init_buffer`
:45-46, `update` :143, `next_epoch` :129) with the data path replaced:

reference                                             here
---------------------------------------------------   ------------------------------------------
gather rows -> pinned host -> gloo isend/irecv ->     one kernel gathers the boundary rows and
pinned host -> H2D copy, one peer at a time           stores them straight into every peer's
(:165-194), ThreadPool + side streams + events        `f_buf` halo rows over NVLink, then
                                                      publishes a flag (pg_halo_push)
torch.cat([feat] + recv buffers) (:132-141)           the peers write into rows [N_in:] of the
                                                      [num_all, d] tensor `update` returns; only
                                                      the inner rows are copied
EMA on the receiver after the H2D copy (:186-191)     sender-side fp32 mirror, fused in the push
                                                      kernel (same value sequence, same rounding)
per-peer grad[boundary[i]] += recv (:208-217)         one ordered scatter-add kernel
blocking r.wait() / event waits (:144-148,154-158)    a flag-wait kernel on the compute stream,
                                                      bracketed by CUDA events (= exposed comm)

Staleness (`pipeline=True`): the message produced at (epoch t, layer l) is consumed
at (t+1, l); epoch 0 consumes zeros.  Two buffer versions (epoch parity) make this safe:
the per-epoch gradient all-reduce separates a version's last read from its next write
(SURVEY.md Appendix A.6).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import torch

from .. import _C
from ..world import Heap, default_world
from .timer.timer import comm_timer

_ALIGN = 256


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class _MsgSet:
    """Device array of pg_msg for one launch."""

    def __init__(self, msgs: List[_C.pg_msg], device):
        rows_per_cta = _C.lib.pg_push_rows_per_cta()
        cta = 0
        for m in msgs:
            m.cta_begin = cta
            cta += (m.n_rows + rows_per_cta - 1) // rows_per_cta
        self.n_msgs, self.n_ctas = len(msgs), cta
        arr = (_C.pg_msg * len(msgs))(*msgs)
        raw = bytes(arr)
        self.dev = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)
        self.ptr = self.dev.data_ptr()


class _HaloUpdate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, buf, layer, push_src, drop):
        ctx.buf, ctx.layer, ctx.epoch = buf, layer, buf._epoch
        return buf._forward(layer, feat, push_src, drop)

    @staticmethod
    def backward(ctx, grad):
        return ctx.buf._backward(ctx.layer, ctx.epoch, grad), None, None, None, None


class Buffer(object):

    def __init__(self, world=None):
        super().__init__()
        self._world = world
        self._epoch = 0
        self._ready = False
        self._connected = False
        self._pipeline = False
        self.timeout_ms = 20000
        self.timer = comm_timer
        self.graph_mode = False      # True while an epoch is captured into / replayed from a CUDA graph

    # ------------------------------------------------------------------ set-up
    def init_buffer(self, num_in, num_all, boundary, f_recv_shape, layer_size, use_pp=False, backend='nccl',
                    pipeline=False, corr_feat=False, corr_grad=False, corr_momentum=0,
                    dtype=torch.float32, world=None, key='pipegcn.buffer', static_layer0=False):
        if backend not in ('nccl', 'nvlink'):
            # the reference implements gloo only and raises for the rest (feature_buffer.py:204-205);
            # this engine implements the NVLink path only
            raise NotImplementedError(f"backend '{backend}': only the NVLink/NCCL path exists in this engine")
        if world is not None:
            self._world = world
        if self._world is None:
            self._world = default_world()
        w = self._world
        rank, size = w.rank, w.size
        dev = w.device
        self._num_in, self._num_all = int(num_in), int(num_all)
        self._boundary = boundary
        self._n_layers = len(layer_size)
        self._layer_size = list(layer_size)
        self._pipeline = bool(pipeline)
        self._epoch = 0
        self._recv_shape = list(f_recv_shape)
        self._corr_feat, self._corr_grad = bool(corr_feat), bool(corr_grad)
        self._corr_momentum = float(corr_momentum)
        self._use_pp = bool(use_pp)
        self._dtype = dtype
        self._es = torch.empty(0, dtype=dtype).element_size()
        self._nver = 2 if pipeline else 1
        self._peers = [j for j in range(size) if j != rank]
        L = self._n_layers
        # static-layer-0 shortcut (SURVEY.md §8f-2): the input features never change, so their halo rows are
        # exchanged ONCE (`static0_begin/_end`) into `x0`; what `update(0, .)` returns at epoch t is c_t * x0 with
        # c_t = [t > 0] (pipelined) / 1 (synchronous), or 1 - m^k after k EMA updates with feat-corr -- the
        # closed form of feature_buffer.py:186-191 applied to a constant message
        self._static0 = bool(static_layer0) and not use_pp and size > 1 and L > 0
        self._static0_gen = 0
        self._static0_ready = False
        self._l0_one = set()

        # rows [pl[j], pr[j]) of the [num_all] space hold peer j's halo (feature_buffer.py:33-43)
        self._pl, self._pr = [None] * size, [None] * size
        tot = self._num_in
        for j in range(size):
            if j == rank:
                continue
            self._pl[j] = tot
            tot += int(f_recv_shape[j])
            self._pr[j] = tot
        assert tot == self._num_all, f"recv shapes {f_recv_shape} do not add up to num_all={num_all}"

        # concatenated boundary space: rows [boff[j], boff[j]+B_j) of b_recv belong to peer j
        self._bidx = [None] * size
        self._boff = [0] * size
        btot = 0
        for j in range(size):
            if j == rank:
                continue
            self._boff[j] = btot
            self._bidx[j] = boundary[j].to(device=dev, dtype=torch.int32).contiguous()
            btot += int(boundary[j].numel())
        self._btot = btot

        # ---- carve the symmetric heap
        self._ld = [_round_up(d, 8) for d in layer_size]
        off = 0
        self._flag_off = off
        off = _round_up(off + 4 * L * 2 * size, _ALIGN)
        self._f_off, self._b_off = {}, {}
        for l in range(L):
            if l == 0 and use_pp:
                continue
            for v in range(self._nver):
                self._f_off[(l, v)] = off
                off = _round_up(off + self._num_all * self._ld[l] * self._es, _ALIGN)
                if l > 0:
                    self._b_off[(l, v)] = off
                    off = _round_up(off + max(btot, 1) * self._ld[l] * self._es, _ALIGN)
        self._x0_off = None
        if self._static0:
            self._x0_off = off
            off = _round_up(off + max(self._num_all - self._num_in, 1) * self._ld[0] * self._es, _ALIGN)
        self._heap = Heap(max(off, _ALIGN), dev)
        self._x0 = None if self._x0_off is None else self._heap.view(
            self._x0_off, (max(self._num_all - self._num_in, 1), self._ld[0]), dtype)
        self._flags = self._heap.view(self._flag_off, (L, 2, size), torch.int32)
        self._f_buf = {k: self._heap.view(o, (self._num_all, self._ld[k[0]]), dtype) for k, o in self._f_off.items()}
        self._b_recv = {k: self._heap.view(o, (max(btot, 1), self._ld[k[0]]), dtype) for k, o in self._b_off.items()}

        # ---- sender-side EMA mirrors (fp32), one per (layer, peer)
        self._f_ema = [None] * L
        self._b_ema = [None] * L
        for l in range(L):
            if l == 0 and use_pp:
                continue
            if corr_feat:
                self._f_ema[l] = {j: torch.zeros(int(boundary[j].numel()), self._ld[l], device=dev) for j in self._peers}
            if corr_grad and l > 0:
                self._b_ema[l] = {j: torch.zeros(int(f_recv_shape[j]), self._ld[l], device=dev) for j in self._peers}

        # ---- ordered boundary add: for every inner row that is a boundary row of some peer, the
        #      rows of b_recv to add, peers ascending (feature_buffer.py:210-217)
        if btot > 0:
            rows = torch.cat([self._bidx[j].to(torch.int64) for j in self._peers])
            slot = torch.arange(btot, device=dev, dtype=torch.int64)
            order = torch.argsort(rows * btot + slot)          # by row, then by concatenated slot (= peer order)
            rows_s = rows[order]
            urow, counts = torch.unique_consecutive(rows_s, return_counts=True)
            self._urow = urow.to(torch.int32).contiguous()
            uptr = torch.zeros(urow.numel() + 1, dtype=torch.int64, device=dev)
            uptr[1:] = torch.cumsum(counts, 0)
            self._uptr = uptr.to(torch.int32).contiguous()
            self._usrc = slot[order].to(torch.int32).contiguous()
        else:
            self._urow = self._uptr = self._usrc = None

        self._counters = torch.zeros(max(1, (4 * L * self._nver + 1) * size), dtype=torch.int32, device=dev)
        self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        # nanoseconds the compute stream spent blocked in flag waits, accumulated by the wait kernel itself
        # (comm_timer.py:17-27's exposed-comm metric where host events cannot be used: CUDA-graph replays)
        self._wait_ns = torch.zeros(1, dtype=torch.int64, device=dev)
        self._epoch_dev = torch.zeros(1, dtype=torch.int32, device=dev)    # == self._epoch, readable by kernels
        self._comm_stream = torch.cuda.Stream(device=dev) if dev.type == 'cuda' else None
        self._push_done = {}
        self._comm_forked = False
        self._keep = []

        self._key = key
        w.publish(key, {
            'heap': w.heap_token(self._heap), 'f_off': dict(self._f_off), 'b_off': dict(self._b_off),
            'flag_off': self._flag_off, 'pl': list(self._pl), 'boff': list(self._boff), 'ld': list(self._ld),
            'n_layers': L, 'nver': self._nver, 'es': self._es, 'x0_off': self._x0_off, 'num_in': self._num_in,
        })
        self._ready, self._connected = True, False

    def _connect(self):
        """Map the peers' heaps and build the message descriptors (needs every rank's table)."""
        w = self._world
        rank, size, dev = w.rank, w.size, w.device
        tables = w.collect(self._key)
        base = {j: w.map_peer(tables[j]['heap']) for j in range(size)}
        L, es = self._n_layers, self._es
        for j in self._peers:
            t = tables[j]
            if t['ld'] != self._ld or t['nver'] != self._nver or t['es'] != es:
                raise RuntimeError(f"rank {j} was initialised with a different layer/dtype/pipeline configuration")
        cnt = iter(range(self._counters.numel()))

        def counter_ptr():
            return self._counters.data_ptr() + 4 * next(cnt)

        def flag_ptr(j, l, direction):
            # word (l, direction, source=rank) of rank j's flag array
            return base[j] + tables[j]['flag_off'] + 4 * ((l * 2 + direction) * size + rank)

        self._self_msgs, self._fwd_msgs, self._bwd_msgs = {}, {}, {}
        for (l, v) in self._f_off:
            ld = self._ld[l]
            m = _C.pg_msg(None, 0, self._num_in, 0, self._f_buf[(l, v)].data_ptr(), ld, None, 0, None, None, 0)
            self._self_msgs[(l, v)] = _MsgSet([m], dev)
            msgs = []
            for j in self._peers:
                dst = base[j] + tables[j]['f_off'][(l, v)] + tables[j]['pl'][rank] * ld * es
                ema = self._f_ema[l][j] if self._f_ema[l] is not None else None
                msgs.append(_C.pg_msg(self._bidx[j].data_ptr(), 0, int(self._bidx[j].numel()), 0, dst, ld,
                                      ema.data_ptr() if ema is not None else None, ld,
                                      flag_ptr(j, l, 0), counter_ptr(), int(tables[j]['pl'][rank])))
            self._fwd_msgs[(l, v)] = _MsgSet(msgs, dev) if msgs else None
        for (l, v) in self._b_off:
            ld = self._ld[l]
            msgs = []
            for j in self._peers:
                dst = base[j] + tables[j]['b_off'][(l, v)] + tables[j]['boff'][rank] * ld * es
                ema = self._b_ema[l][j] if self._b_ema[l] is not None else None
                msgs.append(_C.pg_msg(None, self._pl[j], int(self._recv_shape[j]), 0, dst, ld,
                                      ema.data_ptr() if ema is not None else None, ld,
                                      flag_ptr(j, l, 1), counter_ptr(), int(tables[j]['boff'][rank])))
            self._bwd_msgs[(l, v)] = _MsgSet(msgs, dev) if msgs else None
        self._x0_msgs = None
        if self._static0:
            ld = self._ld[0]
            msgs = []
            for j in self._peers:
                if tables[j]['x0_off'] is None:
                    raise RuntimeError(f"rank {j} was initialised without static_layer0")
                dst = base[j] + tables[j]['x0_off'] + (tables[j]['pl'][rank] - tables[j]['num_in']) * ld * es
                # the backward flag word of layer 0 is free (layer 0 has no gradient exchange): it carries the
                # generation of the one-shot push
                msgs.append(_C.pg_msg(self._bidx[j].data_ptr(), 0, int(self._bidx[j].numel()), 0, dst, ld,
                                      None, 0, flag_ptr(j, 0, 1), counter_ptr(),
                                      int(tables[j]['pl'][rank] - tables[j]['num_in'])))
            self._x0_msgs = _MsgSet(msgs, dev) if msgs else None
        # device arrays of the flag words this rank waits on, per (layer, direction)
        self._wait = {}
        for l in range(L):
            for direction in (0, 1):
                ptrs = [self._heap.ptr + self._flag_off + 4 * ((l * 2 + direction) * size + j) for j in self._peers]
                self._wait[(l, direction)] = torch.tensor(ptrs, dtype=torch.int64, device=dev) if ptrs else None
        self._connected = True

    # ------------------------------------------------------------------ zero-copy producer interface
    def _use_version(self) -> int:
        return (self._epoch + 1) % 2 if self._pipeline else 0

    def inner_view(self, layer):
        """[N_in, d] view of the rows `update(layer, .)` will return first in this epoch.  A producer that writes
        its output here (the LayerNorm/ReLU epilogue of the previous layer, the input features) saves `update`
        the copy of the inner rows: the `torch.cat` of feature_buffer.py:132-141 costs nothing at all."""
        if not self._ready or (layer, 0) not in self._f_off:
            return None
        v = self._use_version()
        ev = self._push_done.get((layer, v))
        if ev is not None:                       # the side-stream push of two epochs ago read these rows
            torch.cuda.current_stream().wait_event(ev)
        return self._f_buf[(layer, v)][:self._num_in, :self._layer_size[layer]]

    def has_peers(self) -> bool:
        return bool(self._ready and self._peers)

    def clean_view(self, layer):
        """[N_in, d] buffer for the CLEAN (not dropped-out) rows of layer `layer` in this epoch's version: with the
        dropout fused into the producers, `inner_view(layer)` holds dropout(h) for the local aggregate / GEMM and this
        holds h itself -- what the halo push sends and what the LayerNorm backward needs."""
        if not self._ready or (layer, 0) not in self._f_off:
            return None
        v = self._use_version()
        if not hasattr(self, '_clean'):
            self._clean = {}
        if (layer, v) not in self._clean:
            from ..graph import alloc_rows
            self._clean[(layer, v)] = alloc_rows(self._num_in, self._layer_size[layer], self._dtype, self._world.device)
        return self._clean[(layer, v)]

    def load_inner(self, layer, feat):
        """Write `feat` into the inner rows of every version of layer `layer` (static input features)."""
        d = self._layer_size[layer]
        for v in range(self._nver):
            dst = self._f_buf[(layer, v)][:self._num_in, :d]
            if feat.is_cuda and feat.dtype == dst.dtype:
                # an SM kernel, not a copy-engine memcpy: a device-to-device memcpy can queue behind a host-to-device
                # transfer in flight on the same engine (the input pipeline of the end-to-end arm), a kernel cannot
                torch.mul(feat, 1, out=dst)
            else:
                dst.copy_(feat)

    # ------------------------------------------------------------------ epoch control
    def next_epoch(self):
        if self.graph_mode and self._comm_forked:
            # a captured epoch must re-join the side stream it forked (the pushes of this epoch); a stream that
            # was not forked into the capture must not be waited on (cudaErrorStreamCaptureIsolation)
            torch.cuda.current_stream().wait_stream(self._comm_stream)
        self._comm_forked = False
        self._epoch += 1
        self._epoch_dev.add_(1)
        self._keep.clear()

    def _val(self, offset: int):
        """(value, value_dev) of a flag publish / wait for epoch + offset: a host constant when running eagerly,
        an offset to the device-side epoch counter when the epoch is captured into a CUDA graph."""
        if self.graph_mode:
            return offset & 0xffffffff, self._epoch_dev.data_ptr()
        return (self._epoch + offset) & 0xffffffff, None

    def take_wait_ns(self) -> int:
        """Exposed communication (ns blocked in flag waits) since the last call; host sync."""
        ns = int(self._wait_ns.item())
        self._wait_ns.zero_()
        return ns

    def check_status(self):
        """Raises if a flag wait timed out since the last check (host sync)."""
        if int(self._status.item()) != 0:
            self._status.zero_()
            raise _C.PgError("halo exchange: a peer's flag did not arrive within "
                             f"{self.timeout_ms} ms (PG_ERR_TIMEOUT); rank {self._world.rank} epoch {self._epoch} "
                             f"pipeline={self._pipeline} static0={self._static0_ready} received flags "
                             f"[layer][fwd,bwd][source rank] = {self._flags.tolist()}")

    # ------------------------------------------------------------------ kernels
    def _push(self, ms: Optional[_MsgSet], src: torch.Tensor, d: int, offset: int, drop=None):
        """`offset`: the flag carries epoch + offset (1 for a message of this epoch).  `drop`: the RECEIVER's dropout
        key, applied to the rows as they are stored into its buffer."""
        if ms is None:
            return
        value, value_dev = self._val(offset)
        _C.count()
        if drop is not None and drop.p > 0:
            _C.check(_C.lib.pg_halo_push_drop(ms.ptr, ms.n_msgs, ms.n_ctas, src.data_ptr(), src.stride(0), d,
                                              _C.dtype_code(src.dtype), self._corr_momentum, 1 - self._corr_momentum,
                                              value, value_dev, C.byref(drop.c()), _C.stream_ptr()), "pg_halo_push_drop")
            return
        _C.check(_C.lib.pg_halo_push(ms.ptr, ms.n_msgs, ms.n_ctas, src.data_ptr(), src.stride(0), d,
                                     _C.dtype_code(src.dtype), self._corr_momentum, 1 - self._corr_momentum,
                                     value, value_dev, _C.stream_ptr()), "pg_halo_push")

    def _wait_flags(self, layer: int, direction: int, offset: int, name: str):
        ptrs = self._wait[(layer, direction)]
        if ptrs is None:
            return
        value, value_dev = self._val(offset)
        timed = not self.graph_mode                   # timing events cannot be queried inside a captured graph
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _C.count()
        _C.check(_C.lib.pg_halo_wait(ptrs.data_ptr(), ptrs.numel(), value, value_dev, self.timeout_ms,
                                     self._status.data_ptr(), self._wait_ns.data_ptr(), _C.stream_ptr()),
                 "pg_halo_wait")
        if timed:
            e1.record()
            self.timer.add_events(name, e0, e1)

    def _check_feat(self, layer, feat):
        if not self._ready:
            raise RuntimeError("Buffer.update before init_buffer")
        if feat.dim() != 2 or feat.shape[0] != self._num_in or feat.shape[1] != self._layer_size[layer]:
            raise ValueError(f"update(layer={layer}): expected [{self._num_in}, {self._layer_size[layer]}], "
                             f"got {tuple(feat.shape)}")
        if feat.dtype != self._dtype:
            raise TypeError(f"update(layer={layer}): buffer dtype is {self._dtype}, feat is {feat.dtype}")
        if not feat.is_cuda:
            raise _C.PgError("Buffer.update needs a CUDA tensor (no CPU fall-back)")

    # ------------------------------------------------------------------ static layer 0
    def static0_begin(self, feat):
        """Push this rank's boundary rows of the (static) input features into every peer's `x0` store.  Every rank
        calls `static0_begin` and then `static0_end` once, before the first epoch and again whenever the input
        features change."""
        if not self._static0:
            return
        if not self._connected:
            self._connect()
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        self._static0_gen += 1
        ms = self._x0_msgs
        if ms is not None:
            _C.count()
            _C.check(_C.lib.pg_halo_push(ms.ptr, ms.n_msgs, ms.n_ctas, feat.data_ptr(), feat.stride(0),
                                         self._layer_size[0], _C.dtype_code(feat.dtype), 0.0, 1.0,
                                         self._static0_gen, None, _C.stream_ptr()), "pg_halo_push")

    def static0_end(self):
        if not self._static0:
            return
        ptrs = self._wait[(0, 1)]
        if ptrs is not None:
            _C.count()
            _C.check(_C.lib.pg_halo_wait(ptrs.data_ptr(), ptrs.numel(), self._static0_gen, None, self.timeout_ms,
                                         self._status.data_ptr(), None, _C.stream_ptr()), "pg_halo_wait")
        self._static0_ready = True
        self._l0_one.clear()
        if self.graph_mode and not self._corr_feat:
            # captured epochs contain no layer-0 kernel (halo rows already hold x0): refresh them here
            for v in range(self._nver):
                self._scale_x0(v, 1, None)
                self._l0_one.add(v)

    def _scale_x0(self, v, k, k_dev):
        d = self._layer_size[0]
        dst = self._f_buf[(0, v)][self._num_in:]
        n = self._num_all - self._num_in
        if n == 0:
            return
        _C.count()
        _C.check(_C.lib.pg_scale_rows(self._x0.data_ptr(), self._x0.stride(0), dst.data_ptr(), dst.stride(0), n, d,
                                      _C.dtype_code(self._dtype), float(self._corr_momentum), int(self._corr_feat),
                                      int(k), k_dev, _C.stream_ptr()), "pg_scale_rows")

    def _forward_static0(self, feat):
        d = self._layer_size[0]
        v = self._use_version()
        if not (feat.data_ptr() == self._f_buf[(0, v)].data_ptr() and feat.stride(0) == self._ld[0]):
            if feat.stride(1) != 1:
                feat = feat.contiguous()
            self._push(self._self_msgs[(0, v)], feat, d, 0)
        # k = EMA updates the consumed message has seen: epoch t consumes message t-1 (pipelined) or t
        off = 0 if self._pipeline else 1
        if self._corr_feat:
            if self.graph_mode:
                self._scale_x0(v, off, self._epoch_dev.data_ptr())
            else:
                self._scale_x0(v, self._epoch + off, None)
        elif v not in self._l0_one and self._epoch + off > 0:
            self._scale_x0(v, 1, None)              # c = 1 from now on: nothing left to do for this version
            self._l0_one.add(v)
        return self._f_buf[(0, v)][:, :d]

    # ------------------------------------------------------------------ forward
    def update(self, layer, feat, push_src=None, drop=None):
        """[N_in, d] -> [num_all, d] = cat(feat, halo rows of every peer); differentiable wrt feat.
        Fused dropout (not in the reference): `feat` already holds dropout(h) under the key `drop`, `push_src` holds h;
        the peers receive h with THEIR dropout of the same key applied by the push, so that the returned tensor is
        dropout(cat(h, halo)) as model.py:47 would compute it -- without a pass over [num_all, d]."""
        self._check_feat(layer, feat)
        if not self._connected:
            self._connect()
        return _HaloUpdate.apply(feat, self, layer, push_src, drop)

    def _forward(self, layer, feat, push_src=None, drop=None):
        if layer == 0 and self._static0_ready:
            return self._forward_static0(feat)
        d = self._layer_size[layer]
        t = self._epoch
        if feat.stride(1) != 1:
            feat = feat.contiguous()
        src = push_src if push_src is not None else feat      # what the peers receive (clean rows)
        def aliased(v):
            return feat.data_ptr() == self._f_buf[(layer, v)].data_ptr() and feat.stride(0) == self._ld[layer]
        if not self._pipeline:
            v = 0
            if not aliased(v):
                self._push(self._self_msgs[(layer, v)], feat, d, 0)
            self._push(self._fwd_msgs[(layer, v)], src, d, 1, drop)          # consumed in this epoch: same step
            self._wait_flags(layer, 0, 1, f'forward_{layer}')
        else:
            v_use, v_send = (t + 1) % 2, t % 2
            v = v_use
            zero_copy = aliased(v_use)
            if not zero_copy:
                self._push(self._self_msgs[(layer, v_use)], feat, d, 0)
            if t > 0:
                self._wait_flags(layer, 0, 0, f'forward_{layer}')
            ms = self._fwd_msgs[(layer, v_send)]
            if ms is not None:
                cur = torch.cuda.current_stream()
                self._comm_stream.wait_stream(cur)
                self._comm_forked = True
                if not self.graph_mode:
                    src.record_stream(self._comm_stream)
                self._keep.append(src)
                with torch.cuda.stream(self._comm_stream):
                    # consumed by the peers in the NEXT epoch: their mask of step + 1
                    self._push(ms, src, d, 1, drop.shifted(1) if drop is not None else None)
                    if zero_copy and not self.graph_mode:
                        ev = torch.cuda.Event()
                        ev.record()
                        self._push_done[(layer, v_use)] = ev
        return self._f_buf[(layer, v)][:, :d]

    # ------------------------------------------------------------------ backward
    def _backward(self, layer, epoch, grad):
        d = self._layer_size[layer]
        t = epoch
        if grad.stride(1) != 1:
            grad = grad.contiguous()
        if not self._pipeline:
            v = 0
            self._push(self._bwd_msgs[(layer, v)], grad, d, epoch - self._epoch + 1)
            self._wait_flags(layer, 1, epoch - self._epoch + 1, f'backward_{layer}')
            self._boundary_add(layer, v, grad)
        else:
            v_use, v_send = (t + 1) % 2, t % 2
            if t > 0:
                self._wait_flags(layer, 1, epoch - self._epoch, f'backward_{layer}')
            self._boundary_add(layer, v_use, grad)
            ms = self._bwd_msgs[(layer, v_send)]
            if ms is not None:
                cur = torch.cuda.current_stream()
                self._comm_stream.wait_stream(cur)
                self._comm_forked = True
                if not self.graph_mode:
                    grad.record_stream(self._comm_stream)
                self._keep.append(grad)
                with torch.cuda.stream(self._comm_stream):
                    self._push(ms, grad, d, epoch - self._epoch + 1)
        return grad[:self._num_in]

    def _boundary_add(self, layer, v, grad):
        if self._urow is None:
            return
        recv = self._b_recv[(layer, v)]
        _C.count()
        _C.check(_C.lib.pg_boundary_add(grad.data_ptr(), grad.stride(0), recv.data_ptr(), recv.stride(0),
                                        self._layer_size[layer], _C.dtype_code(grad.dtype),
                                        self._urow.data_ptr(), self._uptr.data_ptr(), self._usrc.data_ptr(),
                                        int(self._urow.numel()), _C.stream_ptr()), "pg_boundary_add")

    def release(self):
        """Give the symmetric heap back: close the peers' mappings, wait for every rank (they close theirs of this
        heap), free.  Collective over the world; the buffer is unusable afterwards."""
        w = self._world
        if self._connected:
            for j, t in enumerate(w.collect(self._key)):
                if j != w.rank:
                    w.unmap_peer(t['heap'])
        w.barrier()
        self._heap.free()
        self._ready = self._connected = False

    def synchronize(self):
        """Join the side stream (end of training / before reading buffers on the host)."""
        if self._comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self._comm_stream)
