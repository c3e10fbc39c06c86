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


class _Exchange:
    """The protocol every halo exchange here shares: the row map of the [num_all] space, the per-peer boundary index,
    a symmetric heap whose flag words come first (word [row][j] = the last value peer j published for flag row `row`),
    the peers' mappings, and the push / flag-wait launches with their timeout status."""

    def _init_rows(self, world, num_in, num_all, boundary, recv_shape, dtype):
        self._world = world
        rank, size, dev = world.rank, world.size, world.device
        self._num_in, self._num_all = int(num_in), int(num_all)
        self._dtype, self._es = dtype, torch.empty(0, dtype=dtype).element_size()
        self._recv_shape = list(recv_shape)
        self._peers = [j for j in range(size) if j != rank]
        # rows [pl[j], pl[j] + recv_shape[j]) of the [num_all] space hold peer j's halo (feature_buffer.py:33-43)
        self._pl, self._bidx = [None] * size, [None] * size
        tot = self._num_in
        for j in self._peers:
            self._pl[j] = tot
            tot += int(recv_shape[j])
            self._bidx[j] = boundary[j].to(device=dev, dtype=torch.int32).contiguous()
        assert tot == self._num_all, f"recv shapes {recv_shape} do not add up to num_all={num_all}"
        self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._mapped = []
        self._connected = False

    def _publish(self, key, nbytes, table, flag_shape):
        """Allocate the heap (flags of `flag_shape` first) and publish its token with `table` under `key`."""
        w = self._world
        self._key = key
        self._heap = Heap(nbytes, w.device)
        self._flags = self._heap.view(0, flag_shape, torch.int32)
        w.publish(key, dict(heap=w.heap_token(self._heap), **table))

    def _map_peers(self):
        """Every rank's table and the base address of each peer's heap (needs every rank's table)."""
        w = self._world
        tables = w.collect(self._key)
        self._mapped = [tables[j]['heap'] for j in self._peers]
        base = {j: w.map_peer(t) for j, t in zip(self._peers, self._mapped)}
        self._connected = True
        return tables, base

    def _flag_ptr(self, base, row):          # word [row][this rank] of the flags of the peer heap at `base`
        return base + 4 * (row * self._world.size + self._world.rank)

    def _wait_ptrs(self, row):
        """Device array of this rank's flag words [row][j] for every peer j (None without peers)."""
        size = self._world.size
        ptrs = [self._heap.ptr + 4 * (row * size + j) for j in self._peers]
        return torch.tensor(ptrs, dtype=torch.int64, device=self._world.device) if ptrs else None

    def _msg_set(self, msgs):
        return _MsgSet(msgs, self._world.device) if msgs else None

    def _halo_push(self, ms: Optional[_MsgSet], src, d, value, value_dev=None, momentum=0.0, drop=None):
        """Send the rows of `src` the messages name, publish `value` (+ *value_dev) in their flag words.  `drop`: the
        RECEIVER's dropout key, applied to the rows as they are stored into its buffer."""
        if ms is None:
            return
        _C.count()
        if drop is not None and drop.p > 0:
            _C.check(_C.lib.pg_halo_push_drop(ms.ptr, ms.n_msgs, ms.n_ctas, src.data_ptr(), src.stride(0), d,
                                              _C.dtype_code(src.dtype), momentum, 1 - momentum,
                                              value, value_dev, C.byref(drop.c()), _C.stream_ptr()), "pg_halo_push_drop")
            return
        _C.check(_C.lib.pg_halo_push(ms.ptr, ms.n_msgs, ms.n_ctas, src.data_ptr(), src.stride(0), d,
                                     _C.dtype_code(src.dtype), momentum, 1 - momentum,
                                     value, value_dev, _C.stream_ptr()), "pg_halo_push")

    def _halo_wait(self, ptrs, value, value_dev=None, wait_ns=None):
        """Block the stream until the flag words `ptrs` hold `value` (+ *value_dev), for at most `timeout_ms` (a
        timeout is reported by `check_status`); the kernel adds its blocked time to the device int64 `wait_ns`."""
        if ptrs is None:
            return
        _C.count()
        _C.check(_C.lib.pg_halo_wait(ptrs.data_ptr(), ptrs.numel(), value, value_dev, self.timeout_ms,
                                     self._status.data_ptr(), wait_ns, _C.stream_ptr()), "pg_halo_wait")

    def check_status(self):
        """Raises if a flag wait timed out since the last check (host sync)."""
        if int(self._status.item()) != 0:
            self._status.zero_()
            raise _C.PgError(self._timeout_text())

    def release(self):
        """Give the symmetric heap back: close the peers' mappings, wait for every rank (they close theirs of this
        heap), free.  Collective over the world; the exchange is unusable afterwards."""
        w = self._world
        for t in self._mapped:
            w.unmap_peer(t)
        self._mapped = []
        w.barrier()
        self._heap.free()
        self._connected = False


def check_sampling(sampling_rate, pipeline=False, corr_feat=False, corr_grad=False) -> float:
    """The boundary-node sampling rate as a float; raises for a rate outside (0, 1] and for the combinations that are
    not implemented (before anything is allocated)."""
    p = float(sampling_rate)
    if not 0.0 < p <= 1.0:
        raise ValueError(f"--sampling-rate {sampling_rate}: expected 0 < p <= 1")
    if p < 1.0:
        other = [name for name, on in (('--enable-pipeline', pipeline), ('--feat-corr', corr_feat),
                                       ('--grad-corr', corr_grad)) if on]
        if other:
            raise NotImplementedError(f"--sampling-rate {p} together with {' '.join(other)}: boundary-node sampling "
                                      "is implemented for synchronous training without corrections only")
    return p


class _HaloUpdate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, buf, layer, push_src, drop):
        ctx.buf, ctx.layer, ctx.epoch = buf, layer, buf._epoch
        return buf._forward(layer, feat, push_src, drop)

    @staticmethod
    def backward(ctx, grad):
        return ctx.buf._backward(ctx.layer, ctx.epoch, grad), None, None, None, None


class Buffer(_Exchange):

    def __init__(self, world=None):
        self._world = world
        self._epoch = 0
        self._ready = False
        self._pipeline = False
        self.timeout_ms = 20000
        self.timer = comm_timer
        self.graph_mode = False      # True while an epoch is captured into / replayed from a CUDA graph
        self._bns = False            # boundary-node sampling (init_buffer's sampling_rate < 1)

    # ------------------------------------------------------------------ set-up
    def init_buffer(self, num_in, num_all, boundary, f_recv_shape, layer_size, use_pp=False, backend='nccl',
                    pipeline=False, corr_feat=False, corr_grad=False, corr_momentum=0,
                    dtype=torch.float32, world=None, key='pipegcn.buffer', static_layer0=False, sampling_rate=1.0,
                    sampling_seed=0):
        """`sampling_rate` p < 1: boundary-node sampling (synchronous, no corrections): every epoch this rank keeps a
        random fraction p of its halo rows (`sample`), the peers push only those, the others read as zero rows."""
        rate = check_sampling(sampling_rate, pipeline, corr_feat, corr_grad)
        if backend not in ('nccl', 'nvlink'):
            # the reference implements gloo only and raises for the rest (feature_buffer.py:204-205);
            # this engine implements the NVLink path only
            raise NotImplementedError(f"backend '{backend}': only the NVLink/NCCL path exists in this engine")
        if world is not None:
            self._world = world
        if self._world is None:
            self._world = default_world()
        w = self._world
        size, dev = w.size, w.device
        self._init_rows(w, num_in, num_all, boundary, f_recv_shape, dtype)
        self._n_layers = len(layer_size)
        self._layer_size = list(layer_size)
        self._pipeline = bool(pipeline)
        self._epoch = 0
        self._corr_feat, self._corr_grad = bool(corr_feat), bool(corr_grad)
        self._corr_momentum = float(corr_momentum)
        self._use_pp = bool(use_pp)
        self._nver = 2 if pipeline else 1
        L = self._n_layers
        # static-layer-0 shortcut (SURVEY.md §8f-2): the input features never change, so their halo rows are
        # exchanged ONCE (`static0_begin/_end`) into `x0`; what `update(0, .)` returns at epoch t is c_t * x0 with
        # c_t = [t > 0] (pipelined) / 1 (synchronous), or 1 - m^k after k EMA updates with feat-corr -- the
        # closed form of feature_buffer.py:186-191 applied to a constant message
        self._static0 = bool(static_layer0) and not use_pp and size > 1 and L > 0
        self._static0_gen = 0
        self._static0_ready = False
        self._l0_one = set()

        # concatenated boundary space: rows [boff[j], boff[j]+B_j) of b_recv belong to peer j
        self._boff = [0] * size
        btot = 0
        for j in self._peers:
            self._boff[j] = btot
            btot += int(boundary[j].numel())

        # ---- carve the symmetric heap: flags [L][2][P] (row l * 2 + direction), then the row blocks
        self._ld = [_round_up(d, 8) for d in layer_size]
        off = _round_up(4 * L * 2 * size, _ALIGN)
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
        self._publish(key, max(off, _ALIGN), {
            'f_off': dict(self._f_off), 'b_off': dict(self._b_off), 'pl': list(self._pl), 'boff': list(self._boff),
            'ld': list(self._ld), 'nver': self._nver, 'es': self._es, 'x0_off': self._x0_off, 'num_in': self._num_in,
        }, (L, 2, size))
        self._x0 = None if self._x0_off is None else self._heap.view(
            self._x0_off, (max(self._num_all - self._num_in, 1), self._ld[0]), dtype)
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
        # nanoseconds the compute stream spent blocked in flag waits, accumulated by the wait kernel itself
        # (comm_timer.py:17-27's exposed-comm metric where host events cannot be used: CUDA-graph replays)
        self._wait_ns = torch.zeros(1, dtype=torch.int64, device=dev)
        self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=dev)    # == self._epoch, readable by kernels
        self._comm_stream = torch.cuda.Stream(device=dev) if dev.type == 'cuda' else None
        # boundary-node sampling: this epoch's keep mask of the halo rows and the sampled in-degree (`sample`)
        self._bns = rate < 1.0 and bool(self._peers)
        self._bns_rate, self._bns_seed = rate, int(sampling_seed)
        self._bns_mask = self._bns_deg = None
        if self._bns:
            self._bns_mask = torch.zeros(max(self._num_all - self._num_in, 1), dtype=torch.uint8, device=dev)
            self._bns_deg = torch.zeros(self._num_in, dtype=torch.float32, device=dev)
        self._push_done = {}
        self._comm_forked = False
        self._keep = []
        self._ready = True

    def _connect(self):
        """Map the peers' heaps and build the message descriptors (needs every rank's table)."""
        rank = self._world.rank
        tables, base = self._map_peers()
        L, es = self._n_layers, self._es
        for j in self._peers:
            t = tables[j]
            if t['ld'] != self._ld or t['nver'] != self._nver or t['es'] != es:
                raise RuntimeError(f"rank {j} was initialised with a different layer/dtype/pipeline configuration")
        cnt = iter(range(self._counters.numel()))

        def counter_ptr():
            return self._counters.data_ptr() + 4 * next(cnt)

        self._self_msgs, self._fwd_msgs, self._bwd_msgs = {}, {}, {}
        for (l, v) in self._f_off:
            ld = self._ld[l]
            m = _C.pg_msg(None, 0, self._num_in, 0, self._f_buf[(l, v)].data_ptr(), ld, None, 0, None, None, 0)
            self._self_msgs[(l, v)] = self._msg_set([m])
            msgs = []
            for j in self._peers:
                dst = base[j] + tables[j]['f_off'][(l, v)] + tables[j]['pl'][rank] * ld * es
                ema = self._f_ema[l][j] if self._f_ema[l] is not None else None
                msgs.append(_C.pg_msg(self._bidx[j].data_ptr(), 0, int(self._bidx[j].numel()), 0, dst, ld,
                                      ema.data_ptr() if ema is not None else None, ld,
                                      self._flag_ptr(base[j], l * 2), counter_ptr(), int(tables[j]['pl'][rank])))
            self._fwd_msgs[(l, v)] = self._msg_set(msgs)
        for (l, v) in self._b_off:
            ld = self._ld[l]
            msgs = []
            for j in self._peers:
                dst = base[j] + tables[j]['b_off'][(l, v)] + tables[j]['boff'][rank] * ld * es
                ema = self._b_ema[l][j] if self._b_ema[l] is not None else None
                msgs.append(_C.pg_msg(None, self._pl[j], int(self._recv_shape[j]), 0, dst, ld,
                                      ema.data_ptr() if ema is not None else None, ld,
                                      self._flag_ptr(base[j], l * 2 + 1), counter_ptr(), int(tables[j]['boff'][rank])))
            self._bwd_msgs[(l, v)] = self._msg_set(msgs)
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
                                      None, 0, self._flag_ptr(base[j], 1), counter_ptr(),
                                      int(tables[j]['pl'][rank] - tables[j]['num_in'])))
            self._x0_msgs = self._msg_set(msgs)
        if self._bns:
            # sample keys (rank, `_U` row of row 0) per message: a feature push is keyed in the receiver's space, a
            # gradient push in this rank's; slot k of b_recv by the peer that filled it and the row it filled there
            self._bns_fwd_keys = self._keys([(j, tables[j]['pl'][rank]) for j in self._peers])
            self._bns_bwd_keys = self._keys([(rank, self._pl[j]) for j in self._peers])
            slots = [torch.stack([torch.full((n,), j, dtype=torch.int64), tables[j]['pl'][rank] + torch.arange(n)], 1)
                     for j in self._peers for n in [int(self._bidx[j].numel())]]
            self._bns_slot_keys = torch.cat(slots).to(device=self._world.device, dtype=torch.int32).contiguous()
        # device arrays of the flag words this rank waits on, per (layer, direction)
        self._wait = {(l, direction): self._wait_ptrs(l * 2 + direction) for l in range(L) for direction in (0, 1)}

    def _keys(self, pairs):
        return torch.tensor(pairs, dtype=torch.int32, device=self._world.device).reshape(-1, 2).contiguous()

    # ------------------------------------------------------------------ boundary-node sampling
    @property
    def sampling(self) -> bool:
        """True when epochs exchange a sample of the halo rows (rate < 1 and peers to exchange with)."""
        return self._bns

    def _bns_spec(self):
        from ..ops import BnsSpec
        if self.graph_mode:
            return BnsSpec(self._bns_rate, self._bns_seed, 0, self.epoch_dev)
        return BnsSpec(self._bns_rate, self._bns_seed, self._epoch)

    def sample(self, plan):
        """Draw this epoch's sample (one launch): the keep mask of this rank's halo rows and the sampled in-degree of
        its inner rows over the forward CSR `plan`.  Returns the degree [N_in] fp32, the `in_deg` of this epoch."""
        from ..ops import bns_sample
        bns_sample(self._bns_spec(), self._world.rank, plan, self._num_in, self._num_all, self._bns_mask, self._bns_deg)
        return self._bns_deg

    def sample_mask(self):
        """[num_all - N_in] bool copy of the current keep mask of the halo rows (None without sampling)."""
        if not self._bns:
            return None
        return self._bns_mask[:self._num_all - self._num_in].bool()

    def _push_bns(self, ms, keys, src, d, offset, drop=None):
        if ms is None:
            return
        _C.count()
        spec = self._bns_spec()
        _C.check(_C.lib.pg_halo_push_bns(ms.ptr, ms.n_msgs, ms.n_ctas, keys.data_ptr(), src.data_ptr(), src.stride(0),
                                         d, _C.dtype_code(src.dtype), *self._val(offset),
                                         C.byref(drop.c()) if drop is not None and drop.p > 0 else None,
                                         C.byref(spec.c()), _C.stream_ptr()), "pg_halo_push_bns")

    def _halo_rows(self, layer, v):
        return self._f_buf[(layer, v)][self._num_in:, :self._layer_size[layer]]

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
        # the side-stream push of two epochs ago read these rows (an eager epoch's event: not inside a capture)
        if ev is not None and not self.graph_mode:
            torch.cuda.current_stream().wait_event(ev)
        return self._f_buf[(layer, v)][:self._num_in, :self._layer_size[layer]]

    def has_peers(self) -> bool:
        return bool(self._ready and self._peers)

    @property
    def static0_ready(self) -> bool:                # True once `static0_end` has run
        return self._static0_ready

    def input_rows(self):
        """[N_in, d_0] inner rows of layer 0, version 0 (the input features), or None with --use-pp."""
        if not self._ready or (0, 0) not in self._f_off:
            return None
        return self._f_buf[(0, 0)][:self._num_in, :self._layer_size[0]]

    def static_halo(self):
        """[num_all - N_in, d_0] raw halo rows of the static layer-0 store once exchanged, else None."""
        if not self._static0_ready or self._x0 is None:
            return None
        return self._x0[:self._num_all - self._num_in, :self._layer_size[0]]

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
        self.epoch_dev.add_(1)
        self._keep.clear()

    def _val(self, offset: int):
        """(value, value_dev) of a flag publish / wait for epoch + offset: a host constant when running eagerly,
        an offset to the device-side epoch counter when the epoch is captured into a CUDA graph."""
        if self.graph_mode:
            return offset & 0xffffffff, self.epoch_dev.data_ptr()
        return (self._epoch + offset) & 0xffffffff, None

    def take_wait_ns(self) -> int:
        """Exposed communication (ns blocked in flag waits) since the last call; host sync."""
        ns = int(self._wait_ns.item())
        self._wait_ns.zero_()
        return ns

    def _timeout_text(self):
        return ("halo exchange: a peer's flag did not arrive within "
                f"{self.timeout_ms} ms (PG_ERR_TIMEOUT); rank {self._world.rank} epoch {self._epoch} "
                f"pipeline={self._pipeline} static0={self._static0_ready} received flags "
                f"[layer][fwd,bwd][source rank] = {self._flags.tolist()}")

    # ------------------------------------------------------------------ kernels
    def _push(self, ms: Optional[_MsgSet], src: torch.Tensor, d: int, offset: int, drop=None):
        """`offset`: the flag carries epoch + offset (1 for a message of this epoch)."""
        self._halo_push(ms, src, d, *self._val(offset), self._corr_momentum, drop)

    def _wait_flags(self, layer: int, direction: int, offset: int, name: str):
        ptrs = self._wait[(layer, direction)]
        if ptrs is None:
            return
        timed = not self.graph_mode                   # timing events cannot be queried inside a captured graph
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        self._halo_wait(ptrs, *self._val(offset), self._wait_ns.data_ptr())
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
        self._halo_push(self._x0_msgs, feat, self._layer_size[0], self._static0_gen)

    def static0_end(self):
        if not self._static0:
            return
        self._halo_wait(self._wait[(0, 1)], self._static0_gen)
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
        if self._bns:
            from ..ops import bns_mask_rows          # this epoch's sample of x0: keep * x0, rebuilt every epoch
            bns_mask_rows(self._bns_mask, self._halo_rows(0, v), self._x0[:self._num_all - self._num_in, :d])
        elif self._corr_feat:
            if self.graph_mode:
                self._scale_x0(v, off, self.epoch_dev.data_ptr())
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
            if self._bns:
                from ..ops import bns_mask_rows
                self._push_bns(self._fwd_msgs[(layer, v)], self._bns_fwd_keys, src, d, 1, drop)
                bns_mask_rows(self._bns_mask, self._halo_rows(layer, v))      # unkept halo rows read as zero
            else:
                self._push(self._fwd_msgs[(layer, v)], src, d, 1, drop)      # consumed in this epoch: same step
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
            if self._bns:                             # gradients of the kept halo rows only
                self._push_bns(self._bwd_msgs[(layer, v)], self._bns_bwd_keys, grad, d, epoch - self._epoch + 1)
            else:
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
        if self._bns:                                 # the slots the receiving peers kept
            _C.check(_C.lib.pg_boundary_add_bns(grad.data_ptr(), grad.stride(0), recv.data_ptr(), recv.stride(0),
                                                self._layer_size[layer], _C.dtype_code(grad.dtype),
                                                self._urow.data_ptr(), self._uptr.data_ptr(), self._usrc.data_ptr(),
                                                int(self._urow.numel()), self._bns_slot_keys.data_ptr(),
                                                C.byref(self._bns_spec().c()), _C.stream_ptr()), "pg_boundary_add_bns")
            return
        _C.check(_C.lib.pg_boundary_add(grad.data_ptr(), grad.stride(0), recv.data_ptr(), recv.stride(0),
                                        self._layer_size[layer], _C.dtype_code(grad.dtype),
                                        self._urow.data_ptr(), self._uptr.data_ptr(), self._usrc.data_ptr(),
                                        int(self._urow.numel()), _C.stream_ptr()), "pg_boundary_add")

    def release(self):
        super().release()
        self._ready = False

    def synchronize(self):
        """Join the side stream (end of training / before reading buffers on the host)."""
        if self._comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self._comm_stream)


class EvalExchange(_Exchange):
    """Forward-only, synchronous halo exchange of the partitioned evaluation, on a symmetric heap of its own.

    Evaluation never writes the training `Buffer`: with --enable-pipeline the version the next epoch reads already
    holds halo rows the peers have pushed, and overwriting them would silently change training.  Rows are exact: the
    current eval-mode activations, no EMA, no dropout, no staleness.

    Heap: flags [2][P] (uint32, word [b][j] = the last value peer j published into buffer b), then two row buffers
    [num_all, ld] with ld = the padded widest graph-layer input.  Graph layer l reads buffer l % 2; the norm / ReLU
    epilogue of layer l writes the inner rows of buffer (l + 1) % 2; a push sends this rank's boundary rows of buffer
    l % 2 into the peers' halo rows of their buffer l % 2 and publishes seq * L + l + 1 (`seq` counts the eval calls).

    Two buffers are enough.  Peer j pushes its layer l + 2 rows into my buffer l % 2 only after its wait on my layer
    l + 1 flag, and my layer l + 1 push is stream-ordered after my layer-l aggregate, the last read of those halo rows.
    My own inner rows of buffer l % 2 are rewritten by my layer l + 1 epilogue, stream-ordered after my layer-l push
    (their only remote consumer: pushes write the peer's memory, nobody reads mine).  Across eval calls something
    collective has to separate the last read of a call from the first push of the next, which waits on nothing:
    `RankEngine.evaluate` sums its accuracy counts with an all-reduce, `RankEngine.predict` ends with a one-element
    all-reduce, and `LocalTrainer` joins every rank's stream into the current stream at the end of a call and starts
    the next call's streams after it.
    """

    def __init__(self, world, num_in, num_all, boundary, recv_shape, widths, n_layers, dtype,
                 key='pipegcn.eval', timeout_ms=20000):
        self._init_rows(world, num_in, num_all, boundary, recv_shape, dtype)
        self._L = max(int(n_layers), 1)
        self._ld = _round_up(max(list(widths) + [1]), 8)
        size = world.size
        # heap = flags + 2 * num_all * ld * s: independent of the number of layers
        self.flag_bytes = _round_up(4 * 2 * size, _ALIGN)
        buf_bytes = self._num_all * self._ld * self._es
        self._buf_off = [self.flag_bytes, self.flag_bytes + buf_bytes]
        self.heap_bytes = self.flag_bytes + 2 * buf_bytes
        self._publish(key, self.heap_bytes, {'buf_off': list(self._buf_off), 'pl': list(self._pl), 'ld': self._ld,
                                             'es': self._es}, (2, size))
        self._buf = [self._heap.view(o, (self._num_all, self._ld), dtype) for o in self._buf_off]
        self._counters = torch.zeros(2 * size, dtype=torch.int32, device=world.device)
        self.timeout_ms = int(timeout_ms)
        self.seq = 0

    def _connect(self):
        rank, size, ld, es = self._world.rank, self._world.size, self._ld, self._es
        tables, base = self._map_peers()
        self._msgs, self._wait = [None, None], [None, None]
        for b in (0, 1):
            msgs = []
            for j in self._peers:
                t = tables[j]
                if t['ld'] != ld or t['es'] != es:
                    raise RuntimeError(f"rank {j} set up its eval exchange with another width / dtype")
                dst = base[j] + t['buf_off'][b] + t['pl'][rank] * ld * es
                counter = self._counters.data_ptr() + 4 * (b * size + j)
                msgs.append(_C.pg_msg(self._bidx[j].data_ptr(), 0, int(self._bidx[j].numel()), 0, dst, ld, None, 0,
                                      self._flag_ptr(base[j], b), counter, int(t['pl'][rank])))
            self._msgs[b] = self._msg_set(msgs)
            self._wait[b] = self._wait_ptrs(b)

    def begin(self):
        """Start an eval call (every rank, in the same order)."""
        if not self._connected:
            self._connect()
        self.seq += 1

    def rows(self, layer, d):
        """[num_all, d]: the input of graph layer `layer`, inner rows then halo rows."""
        return self._buf[layer % 2][:, :d]

    def inner(self, layer, d):
        return self._buf[layer % 2][:self._num_in, :d]

    def halo(self, layer, d):
        return self._buf[layer % 2][self._num_in:, :d]

    def _value(self, layer):
        return (self.seq * self._L + layer + 1) & 0xffffffff

    def push(self, layer, d):
        """Send this rank's boundary rows of layer `layer`'s input to every peer and publish the flag (zero-row
        messages too: every peer waits for every other)."""
        self._halo_push(self._msgs[layer % 2], self.inner(layer, d), d, self._value(layer))

    def wait(self, layer):
        """Block the stream until every peer's layer-`layer` rows have arrived (bounded: a timeout is reported by
        `check_status`, it does not hang)."""
        self._halo_wait(self._wait[layer % 2], self._value(layer))

    def _timeout_text(self):
        return (f"eval halo exchange: a peer's flag did not arrive within {self.timeout_ms} ms "
                f"(PG_ERR_TIMEOUT); rank {self._world.rank} eval call {self.seq} received flags "
                f"[buffer][source rank] = {self._flags.tolist()}")

    def release(self):
        super().release()
        self._buf = None


class OneShotExchange(_Exchange):
    """One exchange of the halo rows of a static [N_in, d] tensor (the raw input features): the first half of
    --use-pp's precompute (PipeGCN/train.py:169-189) and the layer-0 halo rows of an evaluation layout.  `push`, then
    `wait` (every rank pushes before any rank waits), then `release` once every rank has waited.  Heap: flags [1][2][P],
    then rows [num_all, round_up(d, 8)] -- the layout of a one-layer, non-pipelined `Buffer`."""

    def __init__(self, world, lay, d, dtype, key, timeout_ms=20000):
        self._init_rows(world, lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, dtype)
        self.timeout_ms = int(timeout_ms)
        self._d, self._ld = int(d), _round_up(int(d), 8)
        size = world.size
        row_off = _round_up(4 * 2 * size, _ALIGN)
        self._publish(key, _round_up(row_off + self._num_all * self._ld * self._es, _ALIGN),
                      {'row_off': row_off, 'pl': list(self._pl)}, (1, 2, size))
        self._rows = self._heap.view(row_off, (self._num_all, self._ld), dtype)
        self._counters = torch.zeros(size, dtype=torch.int32, device=world.device)

    def _connect(self):
        rank, ld, es = self._world.rank, self._ld, self._es
        tables, base = self._map_peers()
        self._self_msgs = self._msg_set([_C.pg_msg(None, 0, self._num_in, 0, self._rows.data_ptr(), ld, None, 0,
                                                   None, None, 0)])
        msgs = []
        for k, j in enumerate(self._peers):
            t = tables[j]
            dst = base[j] + t['row_off'] + t['pl'][rank] * ld * es
            msgs.append(_C.pg_msg(self._bidx[j].data_ptr(), 0, int(self._bidx[j].numel()), 0, dst, ld, None, 0,
                                  self._flag_ptr(base[j], 0), self._counters.data_ptr() + 4 * k, int(t['pl'][rank])))
        self._msgs = self._msg_set(msgs)
        self._wait = self._wait_ptrs(0)

    def push(self, feat):
        """Copy `feat` into the inner rows and send its boundary rows to every peer."""
        if not self._connected:
            self._connect()
        feat = feat if feat.stride(1) == 1 else feat.contiguous()
        self._halo_push(self._self_msgs, feat, self._d, 0)
        self._halo_push(self._msgs, feat, self._d, 1)

    def wait(self) -> torch.Tensor:
        """Block the stream until the peers' rows have arrived; [num_all, d]: inner rows, then halo rows."""
        self._halo_wait(self._wait, 1)
        return self._rows[:, :self._d]

    def _timeout_text(self):
        return (f"one-shot halo exchange '{self._key}': a peer's flag did not arrive within {self.timeout_ms} ms "
                f"(PG_ERR_TIMEOUT); rank {self._world.rank} received flags [source rank] = {self._flags[0, 0].tolist()}")
