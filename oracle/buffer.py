"""Oracle: the halo exchange buffer (SURVEY.md §8a rows A1-A9), CPU fp32.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates
PipeGCN/helper/feature_buffer.py for one rank, on host tensors, with the
gloo transfer replaced by an oracle fabric.  What the reference does with
threads, side streams and events is stated here as the value semantics those
mechanisms implement (SURVEY.md Appendix A.3/A.4):

* non-pipelined: the message of (epoch t, layer l) is received and used at
  (t, l) (feature_buffer.py:145-152, 222-227);
* pipelined: it is received at (t+1, l); epoch 0 uses the zero-initialised
  buffers (feature_buffer.py:153-163, 228-236, zeros from :109-112);
* feat-corr / grad-corr: every received message updates
  `avg <- m*avg + (1-m)*recv` (feature_buffer.py:186-191) and the concat / the
  boundary add read `avg` instead of `recv` (:137-140, 214-217).
"""
from __future__ import annotations

import time
from typing import List, Optional

import torch


class OracleBuffer:
    def __init__(self, fabric, rank: int, size: int, timer=None):
        self.fabric, self.rank, self.size = fabric, rank, size
        self.timer = timer
        self._epoch = 0
        self.grad_trace = None     # when a dict: (epoch, layer) -> (grad handed to the hook, grad it returns)

    # feature_buffer.py:33-43
    def _init_pl_pr(self):
        self._pl, self._pr = [], []
        tot = self._num_in
        for s in self._recv_shape:
            if s is None:
                self._pl.append(None)
                self._pr.append(None)
            else:
                self._pl.append(tot)
                tot += s
                self._pr.append(tot)

    # feature_buffer.py:45-127 (host staging, streams, events and pools have no value semantics)
    def init_buffer(self, num_in, num_all, boundary, f_recv_shape, layer_size, use_pp=False, backend="gloo",
                    pipeline=False, corr_feat=False, corr_grad=False, corr_momentum=0):
        self._num_in, self._num_all = num_in, num_all
        self._boundary = boundary
        self._n_layers = len(layer_size)
        self._layer_size = layer_size
        self._pipeline = pipeline
        self._epoch = 0
        self._recv_shape = f_recv_shape
        self._corr_feat, self._corr_grad, self._corr_momentum = corr_feat, corr_grad, corr_momentum
        L = self._n_layers
        self._f_buf = [None] * L
        self._f_recv, self._b_recv = [None] * L, [None] * L
        self._f_avg, self._b_avg = [None] * L, [None] * L
        self._f_pending, self._b_pending = [False] * L, [False] * L
        for i in range(L):
            if i == 0 and use_pp:
                continue
            d = layer_size[i]
            z = lambda n: torch.zeros(n, d)
            self._f_recv[i] = [None if j == self.rank else z(f_recv_shape[j]) for j in range(self.size)]
            if i > 0:
                self._b_recv[i] = [None if j == self.rank else z(boundary[j].shape[0]) for j in range(self.size)]
            if corr_feat:
                self._f_avg[i] = [None if j == self.rank else z(f_recv_shape[j]) for j in range(self.size)]
            if corr_grad and i > 0:
                self._b_avg[i] = [None if j == self.rank else z(boundary[j].shape[0]) for j in range(self.size)]
        self._init_pl_pr()

    def next_epoch(self):                                  # feature_buffer.py:129-130
        self._epoch += 1

    # ---- transfers (feature_buffer.py:165-206, 239-249): ring-offset posting order, tags as the reference
    def _send_all(self, tensor, tag, forward):
        for i in range(1, self.size):
            right = (self.rank + i) % self.size
            if forward:
                msg = tensor[self._boundary[right]]                          # :176
            else:
                msg = tensor[self._pl[right]:self._pr[right]]                # :178
            self.fabric.send(msg, self.rank, right, tag)

    def _recv_all(self, recv, tag, corr, avg):
        for i in range(1, self.size):
            left = (self.rank - i + self.size) % self.size
            got = self.fabric.recv(left, self.rank, tag, shape=tuple(recv[left].shape))
            recv[left].copy_(got)                                            # :185
            if corr:                                                         # :186-191
                t = avg[left]
                t *= self._corr_momentum
                t += (1 - self._corr_momentum) * recv[left]

    def _timed(self, name):
        return self.timer.timer(name) if self.timer is not None else _Null()

    def _feat_concat(self, layer, feat):                   # feature_buffer.py:132-141
        src = self._f_avg[layer] if self._corr_feat else self._f_recv[layer]
        return torch.cat([feat] + [src[i] for i in range(self.size) if i != self.rank])

    def update(self, layer, feat):                         # feature_buffer.py:143-163
        L = self._n_layers
        if not self._pipeline:
            with self._timed(f"forward_{layer}"):
                tag = self._epoch * 2 * L + layer                            # :197
                self._send_all(feat, tag, True)
                self._recv_all(self._f_recv[layer], tag, self._corr_feat, self._f_avg[layer])
        else:
            if self._epoch > 0:
                with self._timed(f"forward_{layer}"):
                    tag = (self._epoch - 1) * 2 * L + layer
                    self._recv_all(self._f_recv[layer], tag, self._corr_feat, self._f_avg[layer])
        buf = self._feat_concat(layer, feat)
        if self._pipeline:
            self._send_all(feat, self._epoch * 2 * L + layer, True)          # :160 (async in the reference)
        self._f_buf[layer] = buf
        if buf.requires_grad:
            buf.register_hook(self._grad_hook(self._epoch, layer))
        return buf

    def _update_grad(self, layer, grad):                   # feature_buffer.py:208-217
        src = self._b_avg[layer] if self._corr_grad else self._b_recv[layer]
        for i in range(self.size):
            if i != self.rank:
                grad[self._boundary[i]] += src[i]

    def _grad_hook(self, epoch, layer):                    # feature_buffer.py:219-237
        L = self._n_layers

        def fn(grad):
            g_in = grad.clone() if self.grad_trace is not None else None
            grad = grad.clone()       # autograd may hand out a shared buffer; the reference mutates in place
            if g_in is not None:
                self.grad_trace[(epoch, layer)] = (g_in, grad)   # `grad` is updated in place below
            if not self._pipeline:
                with self._timed(f"backward_{layer}"):
                    tag = epoch * 2 * L + layer + L                          # :240
                    self._send_all(grad, tag, False)
                    self._recv_all(self._b_recv[layer], tag, self._corr_grad, self._b_avg[layer])
                self._update_grad(layer, grad)
                return grad
            if self._epoch > 0:
                with self._timed(f"backward_{layer}"):
                    tag = (epoch - 1) * 2 * L + layer + L
                    self._recv_all(self._b_recv[layer], tag, self._corr_grad, self._b_avg[layer])
            self._update_grad(layer, grad)
            self._send_all(grad, epoch * 2 * L + layer + L, False)           # :235
            return grad
        return fn


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class OracleCommTimer:
    """PipeGCN/helper/timer/comm_timer.py:6-33."""

    def __init__(self):
        self._time = {}

    def timer(self, name):
        outer = self

        class _T:
            def __enter__(self_inner):
                if name in outer._time:
                    raise Exception(name + " already exists")               # comm_timer.py:14-15
                self_inner.t0 = time.time()

            def __exit__(self_inner, *a):
                outer._time[name] = (self_inner.t0, time.time())
                return False
        return _T()

    def tot_time(self):
        return sum(t1 - t0 for t0, t1 in self._time.values())

    def clear(self):
        self._time = {}
