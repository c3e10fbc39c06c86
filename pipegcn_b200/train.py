"""Per-rank trainer: the epoch loop around the hot path.

Keeps the entry points of PipeGCN/train.py -- `init_processes(rank, size, args)`
(:408-416) and `run(...)` (:242-400) -- and the order of an epoch (:341-362):
forward, summed cross-entropy on the local train rows, backward (which runs the
gradient halo exchange), `buffer.next_epoch()`, `reducer.synchronize()`, Adam step.
The DGL partition arguments of the reference's `run(graph, node_dict, gpb, args)` are
replaced by a `PartitionLayout` (pipegcn_b200/partition.py); evaluation and
checkpointing (train.py:20-61,377-400) run on the GPU with the same kernels (pipegcn_b200/evaluate.py).

`RankEngine` is one rank; `LocalTrainer` steps several simulated ranks of a
`LocalWorld` in lock-step on one GPU (each on its own stream).

With `--eval --eval-partitioned` evaluation is collective: every rank evaluates its own inner rows
(`RankEngine.predict` / `evaluate`, `LocalTrainer.predict` / `evaluate`) over an exact halo exchange of its own heap
(`helper.feature_buffer.EvalExchange`), and no rank needs the global graph.
"""
from __future__ import annotations

import contextlib
import os
import time
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from .graph import PartGraph
from .helper import context as ctx
from .helper.feature_buffer import Buffer, EvalExchange, OneShotExchange, check_sampling
from .helper.reducer import Reducer
from .helper.timer.comm_timer import CommTimer
from .module.model import GraphSAGE
from .partition import PartitionLayout, get_layer_size


def _bns_seed(args):
    from .ops import bns_seed
    return bns_seed(getattr(args, 'seed', 0))


def create_model(layer_size, args, buffer=None, dtype=torch.float32):
    if args.model in ('graphsage', 'gcn'):
        return GraphSAGE(layer_size, F.relu, args.use_pp, norm=args.norm, dropout=args.dropout,
                         n_linear=args.n_linear, train_size=args.n_train, buffer=buffer, dtype=dtype)
    raise NotImplementedError(args.model)


def pp_input(graph, feat, rows):
    """--use-pp layer-0 input of the inner rows: cat(feat, neighbour mean) (second half of `precompute`,
    PipeGCN/train.py:169-189); `rows` [num_all, d] holds the raw features of the inner and the halo rows."""
    from . import ops
    from .graph import alloc_rows
    d = feat.shape[1]
    mean = ops.aggregate(graph.fwd, rows, row_div=graph.in_deg_f)
    both = alloc_rows(graph.num_in, 2 * d, feat.dtype, feat.device)
    both[:, :d].copy_(feat)
    both[:, d:].copy_(mean)
    return both


@contextlib.contextmanager
def _eval_mode(models):
    """Every model in eval mode for the duration, each restored to its own mode afterwards (set once around the
    whole, possibly lock-stepped, forward: the ranks of a LocalWorld may share one model)."""
    uniq = list({id(m): m for m in models}.values())
    modes = [m.training for m in uniq]
    for m in uniq:
        m.eval()
    try:
        yield
    finally:
        for m, was in zip(uniq, modes):
            m.train(was)


def reduce_hook(reducer, param, name, n_train):
    def fn(grad):
        reducer.reduce(param, name, grad, n_train)
    return fn


def act_dtype(args):
    return torch.bfloat16 if getattr(args, 'dtype', 'fp32') in ('bf16', 'bfloat16') else torch.float32


class RankEngine:
    """Everything one rank owns: graph, exchange buffer, model replica, reducer, optimiser."""

    def __init__(self, layout: PartitionLayout, args, world, buffer: Optional[Buffer] = None,
                 reducer: Optional[Reducer] = None, init_state=None, seg_len=None):
        sampling_rate = check_sampling(getattr(args, 'sampling_rate', 1.0), args.enable_pipeline, args.feat_corr,
                                       args.grad_corr)
        self.args, self.world, self.rank = args, world, world.rank
        dev = world.device
        self.device = dev
        self.dtype = act_dtype(args)
        self.graph = PartGraph.from_layout(layout, device=dev, seg_len=seg_len)
        self.in_deg = self.graph.in_deg
        self.layer_size = get_layer_size(args.n_feat, args.n_hidden, args.n_class, args.n_layers)
        self.buffer = buffer if buffer is not None else Buffer(world)
        if buffer is None:
            self.buffer.timer = CommTimer()
        self.buffer.init_buffer(layout.num_in, layout.num_all, layout.boundary, layout.recv_shape,
                                self.layer_size[:args.n_layers - args.n_linear], use_pp=args.use_pp,
                                backend=args.backend, pipeline=args.enable_pipeline, corr_feat=args.feat_corr,
                                corr_grad=args.grad_corr, corr_momentum=args.corr_momentum,
                                dtype=self.dtype, world=world,
                                static_layer0=bool(getattr(args, 'static_layer0', True)),
                                sampling_rate=sampling_rate, sampling_seed=_bns_seed(args))
        self.feat = layout.feat.to(dev).to(self.dtype)
        # the collective set-up; its first step (allocate and publish this rank's heaps) runs here.  The ranks of a
        # LocalWorld run the rest together (`LocalTrainer`), every other rank runs it now
        self.setup_steps = self._setup_steps(layout)
        next(self.setup_steps)
        if not self._local_peers():
            _lockstep([self.setup_steps])
        tm = layout.train_mask.to(dev)
        self.part_train = int(tm.sum().item())
        prefix = bool(tm[:self.part_train].all().item()) if self.part_train else True
        self.train_sel = slice(0, self.part_train) if prefix else tm
        self.labels = layout.label.to(dev)[tm]
        torch.manual_seed(args.seed)                                      # train.py:298
        self.model = create_model(self.layer_size, args, buffer=self.buffer, dtype=self.dtype)
        if init_state is not None:
            self.model.load_state_dict(init_state)
        self.model.to(dev)
        self.reducer = reducer if reducer is not None else Reducer(world)
        self.reducer.init(self.model, world)
        for name, p in self.model.named_parameters():
            p.register_hook(reduce_hook(self.reducer, p, name, args.n_train))
        self.loss_fcn = torch.nn.CrossEntropyLoss(reduction='sum')        # train.py:320
        self.use_graph = bool(getattr(args, 'cuda_graph', False))
        # the reference's optimiser (train.py:321-323); `fused`: torch's single-kernel implementation of the same update
        # (one launch instead of seven foreach kernels per step)
        self.optimizer = torch.optim.Adam(self.model.parameters(), lr=args.lr, weight_decay=args.weight_decay,
                                          capturable=self.use_graph, fused=bool(getattr(args, 'fused_adam', True)))
        self.graphs = None
        self.epoch = 0
        self.last_logits = None
        self.keep_logits = False
        # what the partitioned evaluation of the training layout needs (index spaces, labels and masks of the inner
        # rows); its exchange heap is allocated at the first evaluation
        self._own_eval = SimpleNamespace(num_in=layout.num_in, num_all=layout.num_all, boundary=layout.boundary,
                                         recv_shape=layout.recv_shape, label=layout.label,
                                         val_mask=layout.val_mask, test_mask=layout.test_mask, feat=None)
        self._evals = {}

    def _local_peers(self) -> bool:
        """True for a rank of a LocalWorld with peers: its collective steps need the other ranks' steps in between."""
        return getattr(self.world, 'is_local', False) and self.world.size > 1

    def _setup_steps(self, layout):
        """Collective set-up (generator): the --use-pp precompute (train.py:169-189), cat(feat, neighbour mean) over
        the raw features' halo rows, or else the one-shot exchange of the static layer-0 halo rows (SURVEY.md §8f-2)."""
        if self.args.use_pp:
            self.feat = yield from _raw_halo_steps(self.world, layout, self.feat, self.args.n_feat, 'pipegcn.buffer.pp',
                                                   self.buffer.timeout_ms,
                                                   lambda rows: pp_input(self.graph, self.feat, rows))
            return
        # the static input features live in the exchange buffer of layer 0 (all versions): update(0, .) copies nothing
        self.buffer.load_inner(0, self.feat)
        yield 'publish'
        yield from self._static0_steps()

    def _static0_steps(self):
        self.buffer.static0_begin(self.buffer.input_rows())
        yield 'push'
        self.buffer.static0_end()

    def forward_backward(self, keep_logits=False):
        """train.py:343-355; returns the summed loss (device tensor, no host sync)."""
        self.model.train()
        # boundary-node sampling: this epoch's sample, and its in-degrees for every graph layer
        in_deg = self.buffer.sample(self.graph.fwd) if self.buffer.sampling else self.in_deg
        feat = self.buffer.inner_view(0)
        logits = self.model(self.graph, feat if feat is not None else self.feat, in_deg)
        if isinstance(self.train_sel, slice) and logits.dtype in (torch.float32, torch.bfloat16):
            from . import ops
            loss = ops.cross_entropy_sum(logits, self.labels, self.part_train)      # fused softmax-CE (sum)
        else:
            loss = self.loss_fcn(logits[self.train_sel].float(), self.labels)
        if keep_logits or self.keep_logits:
            self.last_logits = logits.detach()
        self.optimizer.zero_grad(set_to_none=True)
        from . import ops as _ops
        _ops.reset_colsum()
        loss.backward()
        return loss.detach()

    def set_features(self, feat):
        """New input features for the coming epoch (host or device tensor, [N_in, n_feat])."""
        if self.buffer.inner_view(0) is not None:
            static0 = self.buffer.static0_ready          # new features: their halo rows have to be exchanged again
            if static0 and self._local_peers():
                raise RuntimeError("set_features on one rank of a LocalWorld cannot re-exchange the static layer-0 "
                                   "halo rows (its peers would have to push at the same time): set static_layer0=False")
            # layer 0 lives in the exchange buffer, one copy per version (epoch parity): refresh all of them
            self.buffer.load_inner(0, feat.to(self.device, non_blocking=True) if not feat.is_cuda else feat)
            if static0:
                _lockstep([self._static0_steps()])
            return
        # --use-pp: `self.feat` is cat(feat, neighbour mean) (train.py:169-189); the raw half is refreshed, the mean is
        # set-up work of the reference (precompute runs once, train.py:287-288) and is not recomputed per step
        dst = self.feat[:, :feat.shape[1]]
        if feat.is_cuda and feat.dtype == dst.dtype:
            torch.mul(feat, 1, out=dst)
        else:
            dst.copy_(feat, non_blocking=True)

    # ---- input pipeline: the next epoch's features travel host -> device while this epoch computes
    def prefetch_features(self, feat_host, label_host=None) -> int:
        """Start the asynchronous copy of a [N_in, n_feat] pinned host tensor (and optionally the train labels) into one
        of two staging buffers on a copy stream; returns the slot to hand to `commit_features`."""
        if not hasattr(self, '_stage'):
            self._stage_lab = [torch.empty_like(self.labels) for _ in range(2)]
            n_feat = feat_host.shape[1]
            self._stage = [torch.empty(feat_host.shape[0], n_feat, dtype=self.dtype, device=self.device) for _ in range(2)]
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._staged = [torch.cuda.Event(), torch.cuda.Event()]
            self._consumed = [torch.cuda.Event(), torch.cuda.Event()]
            self._stage_n = 0
        slot = self._stage_n % 2
        self._stage_n += 1
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._consumed[slot])        # the epoch that last read this slot has taken it
            self._stage[slot].copy_(feat_host, non_blocking=True)
            if label_host is not None:
                self._stage_lab[slot].copy_(label_host, non_blocking=True)
            self._stage_has_lab = label_host is not None
            self._staged[slot].record()
        return slot

    def commit_features(self, slot: int):
        """Make the staged features of `slot` the input of the coming epoch (device-to-device, on the compute stream)."""
        cur = torch.cuda.current_stream()
        cur.wait_event(self._staged[slot])
        self.set_features(self._stage[slot])
        if getattr(self, '_stage_has_lab', False):
            torch.add(self._stage_lab[slot], 0, out=self.labels)     # SM kernel (see Buffer.load_inner)
        self._consumed[slot].record(cur)

    def finish_epoch(self, reduce=True):
        """train.py:357-362."""
        self.buffer.next_epoch()
        if reduce:
            self.reducer.synchronize()
        self.optimizer.step()
        self.epoch += 1

    def run_epoch(self):
        if self.graphs is not None:
            return self.replay()
        self.buffer.timer.clear()            # sections are per epoch (comm_timer.py:14-15 raises on duplicates)
        loss = self.forward_backward()
        self.finish_epoch()
        return loss

    # ------------------------------------------------------------------ CUDA graphs
    def capture(self):
        """Capture one whole epoch (forward, loss, backward with both halo exchanges, gradient all-reduce, Adam
        step) into a CUDA graph -- two graphs with --enable-pipeline, one per epoch parity, because the exchange
        buffers alternate.  Everything that changes from epoch to epoch is read from the device: the epoch counter
        behind the flag values (`Buffer.epoch_dev`) and the dropout step.  Call after >= 3 eager epochs."""
        from . import ops
        assert self.epoch >= 3, "run a few eager epochs first (allocator, lazy handles, steady-state control flow)"
        assert self.use_graph, "create the engine with args.cuda_graph=True (capturable optimizer)"
        self.buffer.graph_mode = True
        ops.STEP_DEV = self.buffer.epoch_dev
        torch.cuda.synchronize()
        graphs = []
        pool = None
        for _ in range(2 if self.args.enable_pipeline else 1):
            g = torch.cuda.CUDAGraph()
            self.optimizer.zero_grad(set_to_none=True)
            with torch.cuda.graph(g, pool=pool):
                loss = self.forward_backward()
                self.finish_epoch()
            pool = g.pool()
            graphs.append((g, loss, self.last_logits, [p.grad for p in self.model.parameters()]))
        torch.cuda.synchronize()
        self.graphs, self._replays = graphs, 0
        return self

    def replay(self):
        g, loss, logits, grads = self.graphs[self._replays % len(self.graphs)]
        g.replay()
        self._replays += 1
        self.last_logits = logits
        for p, gr in zip(self.model.parameters(), grads):     # each graph owns its gradient tensors
            p.grad = gr
        return loss

    # ------------------------------------------------------------------ partitioned evaluation (--eval-partitioned)
    # Every rank evaluates its own inner rows over an exact, synchronous halo exchange of the eval-mode activations
    # (`EvalExchange`, a heap of its own).  The collective steps are generators that yield after every halo push,
    # driven by `_lockstep` (all ranks of a LocalWorld together, so that every rank has pushed before any rank waits).
    # Callers run them under torch.no_grad().
    def _eval_open_steps(self, eval_layout=None):
        """Set up the partitioned evaluation of `eval_layout` (None: the training layout, transductive).  Collective."""
        args, dev = self.args, self.device
        own = eval_layout is None
        lay = self._own_eval if own else eval_layout
        if lay.val_mask is None or lay.test_mask is None:
            raise ValueError("partitioned evaluation needs the layout's val_mask / test_mask")
        n_graph = args.n_layers - args.n_linear
        widths = self.layer_size[(1 if args.use_pp else 0):n_graph]
        tag = lay.val_mask.to(dev).to(torch.uint8) | (lay.test_mask.to(dev).to(torch.uint8) << 1)
        st = SimpleNamespace(label=lay.label.to(dev), tag=tag, pp_feat=None, x0=None, feat=None, push0=False,
                             n_rows=lay.num_in, layout=eval_layout)
        if own:
            st.graph = self.graph.scratch_view()           # captured training epochs keep their scratch address
            # the eval branch divides by the row lengths of the CSR: a partition holds every in-edge of its inner rows,
            # so these are the global in-degrees the training path divides by
            if not torch.equal(self.graph.row_degrees(), self.graph.in_deg_f):
                raise RuntimeError("partition layout: the CSR row lengths differ from the global in-degrees")
            key = 'pipegcn.eval'
        else:
            st.graph = PartGraph.from_layout(eval_layout, device=dev)
            # one key per evaluation layout (every rank opens them in the same order): several may be alive at once
            self._n_eval_layouts = getattr(self, '_n_eval_layouts', 0) + 1
            key = 'pipegcn.eval.layout%d' % self._n_eval_layouts
        st.xch = EvalExchange(self.world, lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, widths, n_graph,
                              self.dtype, key=key, timeout_ms=self.buffer.timeout_ms)
        self.last_eval_exchange = st.xch
        yield 'publish'
        if own:
            if args.use_pp:
                st.pp_feat = self.feat                     # cat(feat, neighbour mean), computed at set-up
            else:
                # the raw halo rows of the static layer-0 shortcut (not the c_t-scaled copy update(0, .) returns);
                # a view: `set_features` refreshes them.  Without that store every evaluation exchanges the current
                # features' halo rows
                st.x0 = self.buffer.static_halo()
                st.push0 = st.x0 is None and self.world.size > 1
            return st
        # an evaluation layout: its features are those of the graph it was built from, static for the run
        feat = eval_layout.feat.to(dev).to(self.dtype)

        def use(rows):
            if args.use_pp:
                st.pp_feat = pp_input(st.graph, feat, rows)    # recomputed over this layout's graph
            else:
                st.feat = feat
                st.x0 = rows[lay.num_in:].clone()
        yield from _raw_halo_steps(self.world, lay, feat, args.n_feat, key + '.raw', self.buffer.timeout_ms, use)
        return st

    def _predict_steps(self, st, model):
        """One rank's eval forward (generator); `model` is in eval mode for the whole call (`_eval_mode`)."""
        xch = st.xch
        xch.begin()
        if not self.args.use_pp:
            d = self.args.n_feat
            xch.inner(0, d).copy_(st.feat if st.feat is not None else self.buffer.input_rows())
            n_halo = xch.halo(0, d).shape[0]
            if st.x0 is not None and n_halo:
                xch.halo(0, d).copy_(st.x0[:n_halo])
        logits = yield from model.forward_partitioned(st.graph, xch, st.pp_feat, push0=st.push0)
        return logits

    @staticmethod
    def _eval_key(eval_layout):
        return None if eval_layout is None else id(eval_layout)

    def _count(self, eval_layout, logits) -> torch.Tensor:
        """[2, 2] int64 (correct, total) of this rank's validation and test rows (pg_eval_count)."""
        from . import ops
        st = self._evals[self._eval_key(eval_layout)]
        counts, _ = ops.eval_count(logits, st.label, st.tag, 2)
        return counts

    def _predict(self, eval_layout, model):
        if self._local_peers():
            raise RuntimeError("the ranks of a LocalWorld evaluate together: use LocalTrainer.predict / evaluate")
        return _predict([self], [eval_layout], [self.model if model is None else model])[0]

    def predict(self, eval_layout=None, model=None) -> torch.Tensor:
        """Eval-mode logits [N_in, C] of this rank's inner rows of `eval_layout` (None: the training layout), over an
        exact halo exchange with the peers (collective: every rank calls it; the ranks of a LocalWorld go through
        `LocalTrainer.predict`).  `model`: another model of the same shape (default: this rank's replica); it keeps
        its train / eval mode."""
        logits = self._predict(eval_layout, model)
        if self.world.size > 1:
            # the exchange's two buffers are reused by the next call: its first push into a peer's buffers must not
            # overtake that peer's last read of this call (`evaluate` gets the same separation from its count sum)
            self.world.all_reduce_sum_(torch.zeros(1, device=self.device))
        return logits

    def evaluate(self, eval_layout=None, model=None):
        """(validation accuracy, test accuracy) over the inner rows of every rank: per-rank counts summed across the
        world with `all_reduce_sum_` -- what `calc_acc` returns on the whole graph (nan for an empty mask).
        Collective."""
        counts = self._count(eval_layout, self._predict(eval_layout, model))
        if self.world.size > 1:
            self.world.all_reduce_sum_(counts)
        return accuracies(counts)

    def release_eval(self, eval_layout=None):
        """Free the eval exchange heap of `eval_layout` (collective)."""
        st = self._evals.pop(self._eval_key(eval_layout), None)
        if st is not None:
            st.xch.release()

    @property
    def eval_heap_bytes(self) -> int:
        return sum(st.xch.heap_bytes for st in self._evals.values())


def _raw_halo_steps(world, lay, feat, d, key, timeout_ms, use):
    """One-shot exchange of the raw features' halo rows (generator): publish, push, wait, hand the [num_all, d] rows
    (inner, then halo) to `use`, then -- once every rank has used its rows -- free the heap.  Returns `use`'s result."""
    one = OneShotExchange(world, lay, d, feat.dtype, key, timeout_ms)
    yield 'publish'
    one.push(feat)
    yield 'push'
    out = use(one.wait())
    yield 'copied'                                     # every rank has its rows: the one-shot heap may go
    torch.cuda.synchronize()
    one.check_status()
    one.release()
    return out


def _lockstep(gens, streams=None):
    """Step the collective step generators of one or more ranks round by round (each on its rank's stream, or all on
    the current stream when `streams` is None): every rank reaches its next yield (after its halo push) before any
    rank goes on to its wait.  Their return values."""
    cur = torch.cuda.current_stream()
    for s in streams or ():
        s.wait_stream(cur)
    out = [None] * len(gens)
    live = list(range(len(gens)))
    while live:
        nxt = []
        for i in live:
            with torch.cuda.stream(streams[i] if streams else None):
                try:
                    next(gens[i])
                    nxt.append(i)
                except StopIteration as stop:
                    out[i] = stop.value
        live = nxt
    for s in streams or ():
        cur.wait_stream(s)
    return out


def _predict(engines, lays, models, streams=None):
    """Eval-mode logits of every engine's inner rows of its layout (None: the training layout) under its model: sets
    up the evaluation states it is missing, runs the forward steps in lock-step, checks the exchanges."""
    with torch.no_grad(), _eval_mode(models):
        missing = [i for i, (e, l) in enumerate(zip(engines, lays)) if e._eval_key(l) not in e._evals]
        if missing:
            assert len(missing) == len(engines), "every rank sets up its eval exchange at the same time"
            states = _lockstep([e._eval_open_steps(l) for e, l in zip(engines, lays)], streams)
            for e, l, st in zip(engines, lays, states):
                e._evals[e._eval_key(l)] = st
        logits = _lockstep([e._predict_steps(e._evals[e._eval_key(l)], m) for e, l, m in zip(engines, lays, models)],
                           streams)
    for e, l in zip(engines, lays):
        e._evals[e._eval_key(l)].xch.check_status()
    return logits


def accuracies(counts: torch.Tensor):
    """[k, 2] (correct, total) -> k accuracies (calc_acc: nan for an empty mask)."""
    c = counts.cpu().tolist()
    return tuple(float(a) / b if b else float('nan') for a, b in c)


class LocalTrainer:
    """Lock-step driver of all ranks of a LocalWorld on one GPU (one stream per rank)."""

    def __init__(self, layouts: List[PartitionLayout], args, local_world, init_state=None, seg_len=None):
        self.streams = [torch.cuda.Stream(device=local_world.device) for _ in layouts]
        if len(layouts) > 1 and not args.enable_pipeline:
            self._dry_run(layouts, args, local_world, seg_len)
        self.world = local_world
        self.engines = [RankEngine(l, args, local_world.view(r), init_state=init_state, seg_len=seg_len)
                        for r, l in enumerate(layouts)]
        if len(layouts) > 1:
            _lockstep([e.setup_steps for e in self.engines], self.streams)
            torch.cuda.synchronize()
        for e in self.engines:
            e.buffer.timeout_ms = 5000

    def _dry_run(self, layouts, args, local_world, seg_len):
        """One GPU, one process, non-pipelined exchange: a rank's flag-wait kernel spins until its peers'
        pushes are LAUNCHED by this same host thread, so nothing on the host may synchronise with the
        device in between (lazy module loading, first-use handle creation, allocator growth).  Two
        throw-away pipelined epochs (which never wait on unlaunched work) on the same streams trigger
        all of that first.  Real multi-GPU runs (one process per GPU) do not need this."""
        import copy
        from .world import LocalWorld
        dry_args = copy.copy(args)
        dry_args.enable_pipeline = True
        dry_args.sampling_rate = 1.0
        dry = LocalTrainer.__new__(LocalTrainer)
        dry.world = LocalWorld(local_world.size, local_world.device)
        dry.streams = self.streams
        dry.engines = [RankEngine(l, dry_args, dry.world.view(r), seg_len=seg_len) for r, l in enumerate(layouts)]
        _lockstep([e.setup_steps for e in dry.engines], self.streams)     # --use-pp: the precompute
        rng = torch.cuda.get_rng_state(local_world.device)
        for _ in range(2):
            dry.run_epoch()
        torch.cuda.synchronize()
        for e in dry.engines:
            e.buffer.release()
        torch.cuda.set_rng_state(rng, local_world.device)
        del dry

    def run_epoch(self, keep_logits=False):
        cur = torch.cuda.current_stream()
        losses = []
        for e in self.engines:
            e.buffer.timer.clear()
        for e, s in zip(self.engines, self.streams):
            s.wait_stream(cur)
            with torch.cuda.stream(s):
                losses.append(e.forward_backward(keep_logits))
        for e, s in zip(self.engines, self.streams):
            with torch.cuda.stream(s):
                e.buffer.next_epoch()
                e.reducer.pack()
        for s in self.streams:
            cur.wait_stream(s)
        total = self.engines[0].reducer.flat.clone()
        for e in self.engines[1:]:
            total += e.reducer.flat
        for e in self.engines:
            e.reducer.flat.copy_(total)
            e.reducer.unpack()
            e.optimizer.step()
            e.epoch += 1
        for e in self.engines:
            e.buffer.check_status()
        return losses

    # ---- partitioned evaluation, all ranks in lock-step (each rank pushes a layer before any rank waits on it)
    def predict(self, eval_layouts=None, model=None) -> List[torch.Tensor]:
        """Eval-mode logits of every rank's inner rows (`RankEngine.predict`); `eval_layouts`: one layout per rank, or
        None for the training layouts; `model`: one model all ranks evaluate (default: each rank's replica), which
        keeps its train / eval mode.  Consecutive calls are separated by the host: a call's streams join the current
        stream at its end, and the next call's streams start after it."""
        lays = eval_layouts if eval_layouts is not None else [None] * len(self.engines)
        models = [model] * len(self.engines) if model is not None else [e.model for e in self.engines]
        return _predict(self.engines, lays, models, self.streams)

    def evaluate(self, eval_layouts=None, model=None):
        """(validation accuracy, test accuracy) over all ranks: per-rank device counts, summed on the host."""
        lays = eval_layouts if eval_layouts is not None else [None] * len(self.engines)
        logits = self.predict(eval_layouts, model)
        total = sum(e._count(l, z).cpu() for e, l, z in zip(self.engines, lays, logits))
        return accuracies(total)

    def release_eval(self, eval_layouts=None):
        lays = eval_layouts if eval_layouts is not None else [None] * len(self.engines)
        torch.cuda.synchronize()
        for e, l in zip(self.engines, lays):
            e.release_eval(l)


def run(layout: PartitionLayout, args, world=None, eval_graph=None, eval_layouts=None):
    """One rank's training loop with the reference's log line, evaluation and checkpoint (train.py:341-400).
    `eval_graph`: the global graph rank 0 evaluates on every `log_every` epochs when `args.eval` is set.
    With `args.eval_partitioned` every rank evaluates its own inner rows instead (no global graph anywhere); for
    --inductive `eval_layouts` (helper.utils.InductiveEvalLayouts) builds the validation and test layouts."""
    if world is None:
        from .world import default_world
        world = default_world()
    rank = world.rank
    engine = RankEngine(layout, args, world, buffer=ctx.buffer, reducer=ctx.reducer)
    timer = engine.buffer.timer
    part_eval = bool(getattr(args, 'eval', False)) and bool(getattr(args, 'eval_partitioned', False))
    do_eval = bool(getattr(args, 'eval', False)) and (rank == 0 or part_eval)
    inductive = bool(getattr(args, 'inductive', False))
    best = result_file_name = val_layout = None
    if part_eval:
        if inductive:
            if eval_layouts is None:
                raise ValueError("run(..., eval_layouts=None) with --inductive --eval-partitioned: pass "
                                 "load_partition(..., return_eval_layouts=True)[1]")
            val_layout = eval_layouts.val_layout()

        def val_accs():                          # collective: every rank evaluates
            return engine.evaluate(val_layout)

        def test_acc(model):
            nonlocal val_layout
            test_layout = val_layout
            if inductive:                        # the test graph (all nodes) is built once the val heap is gone
                engine.release_eval(val_layout)
                val_layout = None
                test_layout = eval_layouts.test_layout()
            acc = engine.evaluate(test_layout, model=model)[1]
            engine.release_eval(test_layout)
            return acc
    elif do_eval:
        if eval_graph is None:
            raise ValueError("run(..., eval_graph=None) with args.eval set: rank 0 needs the global graph "
                             "(load_partition(..., return_graph=True)) or pass --no-eval")
        from .evaluate import EvalSet, accuracies as full_graph_accuracies
        eval_set = EvalSet(eval_graph, engine.device, inductive=inductive, dtype=engine.dtype)

        def val_accs():
            masks = ('val_mask',) if inductive else ('val_mask', 'test_mask')
            return full_graph_accuracies(engine.model, eval_set.val, masks)

        def test_acc(model):
            return full_graph_accuracies(model, eval_set.test, ('test_mask',))[0]
    if do_eval:
        from .evaluate import BestModel, _emit, result_file
        best = BestModel()                       # every rank that evaluates: the replicas make the same choices
        if rank == 0:
            os.makedirs('checkpoint/', exist_ok=True)                     # train.py:258-260
            os.makedirs('results/', exist_ok=True)
            result_file_name = result_file(args)
    del eval_graph
    train_dur, comm_dur, reduce_dur = [], [], []
    for epoch in range(args.n_epochs):
        torch.cuda.synchronize()
        t0 = time.time()
        loss = engine.forward_backward()
        engine.buffer.next_epoch()
        torch.cuda.synchronize()
        pre_reduce = time.time()
        engine.reducer.synchronize()
        torch.cuda.synchronize()
        reduce_time = time.time() - pre_reduce
        engine.optimizer.step()
        torch.cuda.synchronize()
        if epoch >= 5 and epoch % args.log_every != 0:                    # train.py:364-367
            train_dur.append(time.time() - t0)
            comm_dur.append(timer.tot_time())
            reduce_dur.append(reduce_time)
        if (epoch + 1) % 10 == 0:
            print("Process {:03d} | Epoch {:05d} | Time(s) {:.4f} | Comm(s) {:.4f} | Reduce(s) {:.4f} | Loss {:.4f}".format(
                rank, epoch, np.mean(train_dur) if train_dur else float('nan'),
                np.mean(comm_dur) if comm_dur else float('nan'),
                np.mean(reduce_dur) if reduce_dur else float('nan'), loss.item() / max(engine.part_train, 1)))
        timer.clear()
        engine.buffer.check_status()
        if do_eval and (epoch + 1) % args.log_every == 0:                 # train.py:377-390
            name = 'Epoch %05d' % epoch
            accs = val_accs()
            if rank == 0:
                if not inductive:
                    _emit("{:s} | Validation Accuracy {:.2%} | Test Accuracy {:.2%}".format(name, *accs[:2]),
                          result_file_name)
                else:
                    _emit("{:s} | Accuracy {:.2%}".format(name, accs[0]), result_file_name)
            best.offer(accs[0], engine.model)
    engine.buffer.synchronize()
    if do_eval and best.state is not None:                                # train.py:392-400
        path = best.save(args) if rank == 0 else None
        if rank == 0:
            print('model saved')
            print("Validation accuracy {:.2%}".format(best.acc))
        final = create_model(engine.layer_size, args, buffer=engine.buffer, dtype=engine.dtype).to(engine.device)
        final.load_state_dict(best.state)
        engine.test_acc = test_acc(final)
        if rank == 0:
            _emit("{:s} | Accuracy {:.2%}".format('Test Result', engine.test_acc), None)
        engine.best_val_acc, engine.checkpoint_path = best.acc, path
    if part_eval:
        engine.release_eval(val_layout)
    return engine


def check_parser(args):
    if args.norm == 'none':
        args.norm = None


def init_processes(rank, size, args):
    """Initialise the distributed environment and train this rank (train.py:408-416)."""
    check_sampling(getattr(args, 'sampling_rate', 1.0), args.enable_pipeline, args.feat_corr, args.grad_corr)
    os.environ['MASTER_ADDR'] = args.master_addr
    os.environ['MASTER_PORT'] = '%d' % args.port
    import torch.distributed as dist
    if args.backend not in ('nccl', 'nvlink'):
        raise NotImplementedError("backend '%s': this engine implements the NVLink/NCCL path only" % args.backend)
    if size > torch.cuda.device_count() or getattr(args, 'node_rank', 0) > 0 \
            or size > getattr(args, 'parts_per_node', size):
        # peer heaps are mapped with CUDA IPC, which does not cross nodes
        raise NotImplementedError(f"single-node only: {size} partitions need {size} GPUs of ONE node "
                                  f"({torch.cuda.device_count()} visible, --parts-per-node "
                                  f"{getattr(args, 'parts_per_node', size)}, --node-rank {getattr(args, 'node_rank', 0)})")
    torch.cuda.set_device(rank)
    # 'nvlink' names the halo path; the process group (gradient all-reduce, handle exchange) is always NCCL
    dist.init_process_group('nccl', rank=rank, world_size=size, device_id=torch.device('cuda', rank))
    check_parser(args)
    from .helper.utils import load_partition
    part_eval = bool(getattr(args, 'eval', False)) and bool(getattr(args, 'eval_partitioned', False))
    want_graph = bool(getattr(args, 'eval', False)) and rank == 0 and not part_eval
    want_layouts = part_eval and bool(getattr(args, 'inductive', False))
    g_full = eval_layouts = None
    if want_graph:
        layout, g_full = load_partition(args, rank, return_graph=True)
    elif want_layouts:
        layout, eval_layouts = load_partition(args, rank, return_eval_layouts=True)
    else:
        layout = load_partition(args, rank)
    try:
        return run(layout, args, eval_graph=g_full, eval_layouts=eval_layouts)
    finally:
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()
