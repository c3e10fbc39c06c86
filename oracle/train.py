"""Oracle: the per-process training loop (SURVEY.md §8a rows R1, S6; §3.3), CPU fp32.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates the part of
PipeGCN/train.py:`run` that the hot path lives in:

  model creation from `torch.manual_seed(args.seed)`   train.py:298-300
  reducer: grad <- sum_ranks(grad / n_train)          helper/reducer.py:23-33, train.py:200-203,304-305
  loss: CrossEntropyLoss(reduction='sum') on train rows   train.py:317-320, 348-351
  Adam(lr, weight_decay), zero_grad(set_to_none=True)  train.py:321-323, 353
  epoch order: forward, loss, backward, next_epoch, reducer.synchronize, step   train.py:341-362
  timing rule: epochs < 5 and every log_every-th epoch excluded   train.py:364-367

A world of P ranks runs as P threads over a ThreadFabric (or P gloo processes
over a GlooFabric); traces of per-layer tensors, losses and gradients are what
the parity tests and the golden fixtures compare.
"""
from __future__ import annotations

import threading
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from .buffer import OracleBuffer, OracleCommTimer
from .fabric import ThreadFabric
from .model import OracleGraph, OracleGraphSAGE
from .setup import RankSetup


@dataclass
class OracleArgs:
    n_layers: int = 2
    n_hidden: int = 16
    n_linear: int = 0
    n_feat: int = 0
    n_class: int = 0
    n_train: int = 0
    dropout: float = 0.0
    norm: Optional[str] = "layer"
    lr: float = 1e-2
    weight_decay: float = 0.0
    use_pp: bool = False
    enable_pipeline: bool = False
    feat_corr: bool = False
    grad_corr: bool = False
    corr_momentum: float = 0.95
    seed: int = 0
    n_epochs: int = 4
    log_every: int = 10


def get_layer_size(n_feat, n_hidden, n_class, n_layers):           # helper/utils.py:147-151
    layer_size = [n_feat]
    layer_size.extend([n_hidden] * (n_layers - 1))
    layer_size.append(n_class)
    return layer_size


@dataclass
class RankTrace:
    losses: List[float] = field(default_factory=list)             # loss.item() (sum over local train rows)
    layers: List[Dict[int, Dict[str, torch.Tensor]]] = field(default_factory=list)   # per epoch
    logits: List[torch.Tensor] = field(default_factory=list)
    grads: List[Dict[str, torch.Tensor]] = field(default_factory=list)               # after the reducer
    local_grads: List[Dict[str, torch.Tensor]] = field(default_factory=list)         # before the reducer
    state_dict: Optional[Dict[str, torch.Tensor]] = None
    epoch_time: List[float] = field(default_factory=list)
    comm_time: List[float] = field(default_factory=list)
    reduce_time: List[float] = field(default_factory=list)
    wall: List[float] = field(default_factory=list)                 # every epoch, no exclusions
    states: List[Dict[str, torch.Tensor]] = field(default_factory=list)   # weights at the START of every epoch
    hook_grads: Dict = field(default_factory=dict)                  # (epoch, layer) -> (grad in, grad out) of the halo hook


def run_rank(rs: RankSetup, args: OracleArgs, fabric, init_state=None, keep_trace=True, feat=None,
             forced_states=None) -> RankTrace:
    rank, size = rs.rank, rs.size
    timer = OracleCommTimer()
    buf = OracleBuffer(fabric, rank, size, timer)
    layer_size = get_layer_size(args.n_feat, args.n_hidden, args.n_class, args.n_layers)
    graph = OracleGraph(rs.u, rs.v, rs.num_in, rs.num_all)
    in_deg = rs.in_deg
    buf.init_buffer(rs.num_in, rs.num_all, rs.boundary, rs.recv_shape,
                    layer_size[:args.n_layers - args.n_linear], use_pp=args.use_pp, backend="gloo",
                    pipeline=args.enable_pipeline, corr_feat=args.feat_corr, corr_grad=args.grad_corr,
                    corr_momentum=args.corr_momentum)                      # train.py:283-285
    feat = rs.node_dict["feat"] if feat is None else feat
    train_mask = rs.node_dict["train_mask"]
    labels = rs.node_dict["label"][train_mask]                            # train.py:290
    torch.manual_seed(args.seed)                                          # train.py:298
    model = OracleGraphSAGE(layer_size, F.relu, args.use_pp, norm=args.norm, dropout=args.dropout,
                            n_linear=args.n_linear, train_size=args.n_train)
    if init_state is not None:
        model.load_state_dict(init_state)
    loss_fcn = torch.nn.CrossEntropyLoss(reduction="sum")                 # train.py:320
    opt = torch.optim.Adam(model.parameters(), lr=args.lr, weight_decay=args.weight_decay)
    tr = RankTrace()
    if keep_trace:
        buf.grad_trace = tr.hook_grads
    for epoch in range(args.n_epochs):
        t0 = time.time()
        model.train()
        if forced_states is not None:           # teacher forcing: start every epoch from given weights
            model.load_state_dict(forced_states[epoch])
        if keep_trace:
            tr.states.append({k: v.detach().clone() for k, v in model.state_dict().items()})
        ltrace = {} if keep_trace else None
        logits = model(graph, feat, in_deg, buf, trace=ltrace)
        loss = loss_fcn(logits[train_mask], labels)                       # train.py:351
        opt.zero_grad(set_to_none=True)
        loss.backward()
        buf.next_epoch()                                                  # train.py:357
        t_red = time.time()
        local = {n: p.grad.detach().clone() for n, p in model.named_parameters()} if keep_trace else None
        for name, p in model.named_parameters():                          # reducer.py:27-31
            p.grad.div_(args.n_train)
            fabric.all_reduce_sum(rank, p.grad, ("grad", epoch, name))
        reduce_time = time.time() - t_red
        opt.step()                                                        # train.py:362
        if epoch >= 5 and epoch % args.log_every != 0:                    # train.py:364-367
            tr.epoch_time.append(time.time() - t0)
            tr.comm_time.append(timer.tot_time())
            tr.reduce_time.append(reduce_time)
        tr.wall.append(time.time() - t0)
        timer.clear()
        tr.losses.append(float(loss.item()))
        if keep_trace:
            tr.layers.append(ltrace)
            tr.logits.append(logits.detach().clone())
            tr.local_grads.append(local)
            tr.grads.append({n: p.grad.detach().clone() for n, p in model.named_parameters()})
    tr.state_dict = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return tr


def run_world(setups: List[RankSetup], args: OracleArgs, init_state=None, keep_trace=True,
              forced_states=None) -> List[RankTrace]:
    """All ranks of a world as threads in this process."""
    size = len(setups)
    fabric = ThreadFabric(size)
    out: List[Optional[RankTrace]] = [None] * size
    err: List[Optional[BaseException]] = [None] * size
    feats = [None] * size
    if args.use_pp:                                                        # train.py:287-288
        from .setup import precompute
        feats = precompute(setups)
    if size == 1:
        return [run_rank(setups[0], args, fabric, init_state, keep_trace, feat=feats[0], forced_states=forced_states)]
    torch.set_num_threads(max(1, torch.get_num_threads() // size))

    # every rank seeds the global RNG identically before building its model (train.py:298); with threads the
    # global RNG is shared, so models are built serially under a lock by passing an explicit initial state.
    if init_state is None:
        layer_size = get_layer_size(args.n_feat, args.n_hidden, args.n_class, args.n_layers)
        torch.manual_seed(args.seed)
        m = OracleGraphSAGE(layer_size, F.relu, args.use_pp, norm=args.norm, dropout=args.dropout,
                            n_linear=args.n_linear, train_size=args.n_train)
        init_state = {k: v.detach().clone() for k, v in m.state_dict().items()}

    def work(r):
        try:
            out[r] = run_rank(setups[r], args, fabric, init_state, keep_trace, feat=feats[r],
                              forced_states=forced_states)
        except BaseException as e:   # noqa: BLE001
            err[r] = e
            try:
                fabric._bar.abort()
            except Exception:
                pass

    ths = [threading.Thread(target=work, args=(r,), daemon=True) for r in range(size)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return out  # type: ignore[return-value]


def initial_state(args: OracleArgs) -> Dict[str, torch.Tensor]:
    layer_size = get_layer_size(args.n_feat, args.n_hidden, args.n_class, args.n_layers)
    torch.manual_seed(args.seed)
    m = OracleGraphSAGE(layer_size, F.relu, args.use_pp, norm=args.norm, dropout=args.dropout,
                        n_linear=args.n_linear, train_size=args.n_train)
    return {k: v.detach().clone() for k, v in m.state_dict().items()}
