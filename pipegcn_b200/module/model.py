"""`GraphSAGE` (alias `GCN`): the layer loop of PipeGCN/module/model.py:25-58.

Per graph layer: `buffer.update` (halo exchange) -> dropout -> GraphSAGELayer -> norm ->
activation; trailing `n_linear` plain linears.  The reference defines no `GCN` class
(SURVEY.md §0.2): the north-star's `module.model.GCN` is this class under a second name.
state_dict keys match the reference (`layers.{i}.linear1.weight`, `norm.{i}.weight`, ...).

Extra keyword arguments (not in the reference): `buffer` -- the exchange object to use
instead of the process-global `helper.context.buffer` (several simulated ranks in one
process); `dtype` -- activation storage type, float32 (reference) or bfloat16 (fp32
accumulate, fp32 master weights).

`aggregator='pool'` (not in the reference) builds max-pool GraphSAGE layers (DGL SAGEConv(aggregator_type='pool'),
module/layer.py); with boundary-node sampling they take the buffer's keep mask of the halo rows in place of the
in-degrees, and zero the pooled transform of the unkept rows before the maximum.

`GAT` (not in the reference) is the same layer loop with `GATLayer`s: every graph layer whose output feeds another
layer concatenates `n_heads` heads of d_out / n_heads columns, a graph layer that produces the logits has one head.  The
exchange moves the layer input h, so pipelining, the corrections, the static layer-0 store and the fused dropout apply
unchanged; with boundary-node sampling the layers take the buffer's keep mask of the halo rows (`Buffer.keep_mask`),
and unkept rows are absent from every softmax.

`GATv2(GAT)` (not in the reference) is `GAT` with `GATv2Layer`s (DGL's GATv2Conv): the same heads, keep mask and
partitioned evaluation; only the graph layers and the kernels they load differ.

`GraphTransformer(GAT)` (not in the reference) is `GAT` with `TransformerLayer`s (PyG's TransformerConv): the same
heads, keep mask and partitioned evaluation; only the graph layers and the kernels they load differ.

`GraphConv(GraphSAGE)` (not in the reference) is the same layer loop with `GraphConvLayer`s (DGL's GraphConv,
norm='both'): the layers read the symmetric norm from the graph (`PartGraph.sym_norm`) instead of the in-degrees.
`GCN` stays the reference's name for GraphSAGE.

`GCNII(GraphSAGE)` (not in the reference) is the same layer loop with `GCNIILayer`s (DGL's GCN2Conv): graph layer 0 is
fc_in + ReLU + convolution 1 over the exchanged input features, every later graph layer one square convolution, and
the trailing `n_linear` (>= 1) linears produce the logits.  Every layer reads h0 = ReLU(fc_in(dropout(x))) through
the `ops.GCNIIState` of the forward; h0 enters convolution 1 through its own keyed dropout and the residuals clean.
Between the graph layers the loop applies norm, ReLU and dropout as for every other model; the paper has ReLU only.

`PNA(GraphSAGE)` (not in the reference) is the same layer loop with `PNALayer`s (DGL's PNAConvTower, module/layer.py).
Its degree scalers need delta, the mean of log(D + 1) over the training graph's nodes: the trainer computes it from the
merged integer degree histograms of all partitions (`train.RankEngine`) and sets it with `set_delta`.  delta is model
state: the state dict carries it as the fp64 scalar `pna_delta`, so a loaded checkpoint evaluates with the delta it
was trained with.  Every graph (partition, whole graph, evaluation layout) computes its own rows' scalers from its row
degrees and this delta (`PartGraph.pna_scalers`).

`GENConv(GraphSAGE)` (not in the reference) is the same layer loop with `GENConvLayer`s (PyG's GENConv with the softmax
aggregator, module/layer.py); a last graph layer that produces the logits is a GENConvLayer(d_in, n_class).  Like
`GAT`, with boundary-node sampling its layers take the buffer's keep mask of the halo rows, and unkept rows are absent
from every softmax.  The temperature `t` (constant, or learnt with `learn_t`) is read by the kernels from device
memory, so a captured CUDA graph sees the optimizer's updates of it.

`ResGatedGCN(GraphSAGE)` (not in the reference) is the same layer loop with `ResGatedLayer`s (PyG's ResGatedGraphConv,
module/layer.py); a last graph layer that produces the logits is a ResGatedLayer(d_in, n_class).  Like `GENConv`, with
boundary-node sampling its layers take the buffer's keep mask of the halo rows, and unkept rows are absent from every
sum.

`MoNet(GraphSAGE)` (not in the reference) is the same layer loop with `MoNetLayer`s (DGL's GMMConv with the mean
aggregator on the degree pseudo-coordinates, module/layer.py); a last graph layer that produces the logits is a
MoNetLayer(d_in, n_class).  Like `GraphConv`, the layers read c = deg^-1/2 from the graph (`PartGraph.sym_norm`,
the halo rows' values from their owners).  mu and inv_sigma are read by the kernels from device memory, so a captured
CUDA graph sees the optimizer's updates of them.
"""
import torch
from torch import nn
import torch.nn.functional as F

from ..helper import context as ctx
from .layer import (GATLayer, GATv2Layer, GCNIILayer, GENConvLayer, GraphConvLayer, GraphSAGELayer, MoNetLayer,
                    PNALayer, ResGatedLayer, TransformerLayer)


class GNNBase(nn.Module):

    def __init__(self, layer_size, activation, use_pp=False, dropout=0.5, norm='layer', n_linear=0):
        super().__init__()
        self.n_layers = len(layer_size) - 1
        self.n_linear = n_linear
        self.n_graph_layers = self.n_layers - n_linear
        self.activation = activation
        self.use_pp = use_pp
        self.use_norm = norm is not None
        self.layers = nn.ModuleList()
        if self.use_norm:
            self.norm = nn.ModuleList()
        self.dropout = nn.Dropout(p=dropout)


class GraphSAGE(GNNBase):

    def __init__(self, layer_size, activation, use_pp, dropout=0.5, norm='layer', train_size=None, n_linear=0,
                 buffer=None, dtype=torch.float32, aggregator='mean'):
        super().__init__(layer_size, activation, use_pp, dropout, norm, n_linear)
        if aggregator not in ('mean', 'pool'):
            raise ValueError(f"aggregator '{aggregator}': expected 'mean' or 'pool'")
        if aggregator == 'pool' and use_pp:
            raise NotImplementedError("the pool aggregator with use_pp: the precompute is a neighbour mean")
        self.aggregator = aggregator
        self.buffer = buffer
        self.act_dtype = dtype
        for i, (d_in, d_out) in enumerate(zip(layer_size[:-1], layer_size[1:])):
            if i < self.n_graph_layers:
                self.layers.append(self._graph_layer(i, d_in, d_out))
            else:
                self.layers.append(nn.Linear(d_in, d_out))
            if self.use_norm and i < self.n_layers - 1:
                if norm == 'layer':
                    self.norm.append(nn.LayerNorm(d_out, elementwise_affine=True))
                elif norm == 'batch':
                    from .sync_bn import SyncBatchNorm
                    self.norm.append(SyncBatchNorm(d_out, train_size))
                else:
                    raise ValueError(f"unknown norm '{norm}'")

    def _graph_layer(self, i, d_in, d_out):
        if self.aggregator == 'pool':
            return GraphSAGELayer(d_in, d_out, aggregator='pool')
        return GraphSAGELayer(d_in, d_out, use_pp=(self.use_pp and i == 0))

    def _layer_arg(self, in_deg):
        """The third argument of every graph layer in training: the in-degrees, or for pool layers the keep mask of
        this epoch's boundary-node sample (training with sampling), else None."""
        if self.aggregator == 'pool':
            buf = self._buffer() if self.training else None
            return getattr(buf, 'keep_mask', None) if buf is not None else None
        return in_deg

    def _drop(self, h):
        from .. import ops
        return ops.dropout(h, self.dropout.p, self.training)

    def _drop_input(self, i, h):
        """Dropout of graph layer i's input rows where no fused or keyed path applies."""
        return self._drop(h)

    def _buffer(self):
        return self.buffer if self.buffer is not None else ctx.buffer

    def _drop_spec(self, i):
        """Dropout key of graph layer i in this epoch (same on every rank; the step is the buffer's device-side epoch)."""
        from .. import ops
        return ops.DropSpec(self.dropout.p, ops.layer_seed(i), getattr(self._buffer(), 'epoch_dev', None), 0)

    def _norm_act(self, i, h, dest=None, fuse_drop=False):
        if self.use_norm:
            n = self.norm[i]
            from .. import ops
            if isinstance(n, nn.LayerNorm) and self.activation in (F.relu, torch.relu) and ops.ln_relu_supported(h):
                # LayerNorm + ReLU in one pass, written straight into the next layer's exchange buffer
                if fuse_drop and dest is not None:
                    buf = self._buffer()
                    # the clean rows are only needed as the source of the halo push: no peers, no copy
                    clean = buf.clean_view(i + 1) if buf.has_peers() else None
                    if ops._drop_ok(dest) and (clean is None or ops._drop_ok(clean)):
                        # ... together with the NEXT layer's dropout: dest <- dropout(h), clean <- h
                        self._fused = (i + 1, clean)
                        return ops.layer_norm_relu(h, n.weight, n.bias, n.eps, relu=True, out=dest, clean=clean,
                                                   drop=self._drop_spec(i + 1))
                return ops.layer_norm_relu(h, n.weight, n.bias, n.eps, relu=True, out=dest)
            if isinstance(n, nn.LayerNorm) and h.dtype != n.weight.dtype:
                h = F.layer_norm(h, n.normalized_shape, n.weight.to(h.dtype), n.bias.to(h.dtype), n.eps)
            else:
                h = n(h)
        return self.activation(h)

    def forward(self, g, feat, in_deg=None):
        from .. import ops
        if self.aggregator == 'pool':
            ops.pool_preload()
        h = feat if feat.dtype == self.act_dtype else feat.to(self.act_dtype)
        p = self.dropout.p if self.training else 0.0
        in_deg = self._layer_arg(in_deg)
        self._fused = None
        for i, layer in enumerate(self.layers):
            if i < self.n_graph_layers:
                fused = self._fused is not None and self._fused[0] == i
                if self.training and (i > 0 or not self.use_pp):
                    if fused:       # h = dropout(LayerNorm output), written by the epilogue; the peers get the clean rows
                        h = self._buffer().update(i, h, push_src=self._fused[1], drop=self._drop_spec(i))
                    else:
                        h = self._buffer().update(i, h)
                if fused:
                    h = layer(g, h, in_deg, drop_bwd=self._drop_spec(i))
                elif self.training and p > 0 and i > 0 and ops._drop_ok(h):
                    # same mask as the fused path, as separate passes (PG_FUSED_DROPOUT=0 / unsupported shapes)
                    h = layer(g, ops.keyed_dropout(h, self._drop_spec(i)), in_deg)
                else:
                    h = layer(g, self._drop_input(i, h), in_deg)
            else:
                h = ops.linear(self._drop(h), layer.weight, layer.bias)
            if i < self.n_layers - 1:
                dest = None
                if self.training and i + 1 < self.n_graph_layers:
                    dest = self._buffer().inner_view(i + 1)
                h = self._norm_act(i, h, dest, fuse_drop=ops.FUSED_DROPOUT and p > 0 and dest is not None)
        return h

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        """Eval-mode forward of the inner rows of one partition (partitioned evaluation), as a generator that yields
        after every halo push: with several ranks driven by one host thread every rank pushes before any rank waits.
        `xch` is an `EvalExchange` whose buffer 0 holds the layer-0 input: the inner rows, and the halo rows too
        unless `push0` (then they are exchanged like every later layer's); every norm / ReLU epilogue writes the next
        graph layer's inner rows straight into the exchange buffer.  `pp_feat`: the --use-pp layer-0 input
        cat(feat, neighbour mean) of the inner rows.  Returns the logits [N_in, C]."""
        from .. import ops
        assert not self.training
        if self.aggregator == 'pool':
            ops.pool_preload()
        h = None
        arg = self._layer_arg(None)
        for i, layer in enumerate(self.layers):
            if i < self.n_graph_layers:
                if i == 0 and self.use_pp:
                    h = self._pp_layer0(layer, pp_feat)
                else:
                    d = layer.in_feats
                    if i > 0 or push0:
                        xch.push(i, d)
                        yield i
                        xch.wait(i)
                    h = layer(g, xch.rows(i, d), arg)
            else:
                h = ops.linear(h, layer.weight, layer.bias)
            if i < self.n_layers - 1:
                dest = xch.inner(i + 1, h.shape[1]) if i + 1 < self.n_graph_layers else None
                out = self._norm_act(i, h, dest)
                if dest is not None and out.data_ptr() != dest.data_ptr():
                    dest.copy_(out)
                h = out
        return h

    def _pp_layer0(self, layer, pp_feat):
        """--use-pp layer 0 on its precomputed input rows (partitioned evaluation)."""
        from .. import ops
        return ops.linear(pp_feat, layer.linear.weight, layer.linear.bias)


GCN = GraphSAGE


class GraphConv(GraphSAGE):

    def _graph_layer(self, i, d_in, d_out):
        return GraphConvLayer(d_in, d_out, use_pp=(self.use_pp and i == 0))

    def _layer_arg(self, in_deg):
        """GraphConv layers take no degrees: the norm lives on the graph."""
        return None

    def _pp_layer0(self, layer, pp_feat):
        return layer.pp_linear(pp_feat)

    def _preload(self):
        from .. import ops
        ops.graphconv_preload()

    def forward(self, g, feat, in_deg=None):
        self._preload()
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._preload()
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))


class GCNII(GraphSAGE):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=1, buffer=None,
                 dtype=torch.float32, alpha=0.1, lam=0.5):
        n_graph = len(layer_size) - 1 - n_linear
        if n_linear < 1:
            raise ValueError("GCNII needs n_linear >= 1: its last convolution is square, the logits come from a linear")
        if n_graph < 1:
            raise ValueError("GCNII needs at least one graph layer")
        if len(set(layer_size[1:n_graph + 1])) != 1:
            raise ValueError(f"GCNII: every convolution is square, got widths {layer_size[1:n_graph + 1]}")
        self.alpha, self.lam = float(alpha), float(lam)
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)

    def _graph_layer(self, i, d_in, d_out):
        return GCNIILayer(d_in, d_out, i, alpha=self.alpha, lam=self.lam)

    def _layer_arg(self, in_deg):
        """A fresh `ops.GCNIIState` per forward, with the dropout key of h0 in training."""
        from .. import ops
        drop = None
        if self.training and self.dropout.p > 0:
            drop = ops.DropSpec(self.dropout.p, ops.gcnii_h0_seed(), getattr(self._buffer(), 'epoch_dev', None), 0)
        return ops.GCNIIState(drop)

    def _drop_input(self, i, h):
        """Layer 0's input features take a keyed mask too (CUDA-graph replays draw fresh ones)."""
        from .. import ops
        if i > 0 or not self.training or self.dropout.p == 0:
            return super()._drop_input(i, h)
        if not ops._drop_ok(h):
            from ..graph import alloc_rows
            hp = alloc_rows(h.shape[0], h.shape[1], h.dtype, h.device)
            hp.copy_(h)
            h = hp
        return ops.keyed_dropout(h, self._drop_spec(0))

    def _preload(self):
        from .. import ops
        ops.gcnii_preload()

    def forward(self, g, feat, in_deg=None):
        self._preload()
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._preload()
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))


class GAT(GraphSAGE):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=0, buffer=None,
                 dtype=torch.float32, n_heads=4):
        n_graph = len(layer_size) - 1 - n_linear
        for i in range(n_graph):
            if i < len(layer_size) - 2 and layer_size[i + 1] % n_heads:
                raise ValueError(f"GAT: {layer_size[i + 1]} hidden units do not split into {n_heads} heads")
        self.n_heads = n_heads
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)

    def _graph_layer(self, i, d_in, d_out):
        if i < self.n_layers - 1:
            return GATLayer(d_in, d_out // self.n_heads, self.n_heads)
        return GATLayer(d_in, d_out, 1)                  # the logits: one head of n_class

    def _layer_arg(self, in_deg):
        """The keep mask of this epoch's boundary-node sample (training with sampling), else None."""
        buf = self._buffer() if self.training else None
        return getattr(buf, 'keep_mask', None) if buf is not None else None

    def _preload(self):
        from .. import ops
        ops.gat_preload()

    def forward(self, g, feat, in_deg=None):
        self._preload()
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._preload()
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))


class GATv2(GAT):

    def _graph_layer(self, i, d_in, d_out):
        if i < self.n_layers - 1:
            return GATv2Layer(d_in, d_out // self.n_heads, self.n_heads)
        return GATv2Layer(d_in, d_out, 1)                # the logits: one head of n_class

    def _preload(self):
        from .. import ops
        ops.gatv2_preload()


class GraphTransformer(GAT):

    def _graph_layer(self, i, d_in, d_out):
        if i < self.n_layers - 1:
            return TransformerLayer(d_in, d_out // self.n_heads, self.n_heads)
        return TransformerLayer(d_in, d_out, 1)          # the logits: one head of n_class, and so does the skip

    def _preload(self):
        from .. import ops
        ops.transformer_preload()


class PNA(GraphSAGE):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=0, buffer=None,
                 dtype=torch.float32):
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)
        self.register_buffer('pna_delta', torch.tensor(float('nan'), dtype=torch.float64))
        self.delta = None

    def _graph_layer(self, i, d_in, d_out):
        return PNALayer(d_in, d_out)

    def _layer_arg(self, in_deg):
        """PNA layers take no degrees: the scalers live on the graph."""
        return None

    def set_delta(self, delta: float):
        """delta of the degree scalers (the mean of log(D + 1) over the training graph), for every graph layer."""
        self.delta = float(delta)
        self.pna_delta.fill_(self.delta)
        for i in range(self.n_graph_layers):
            self.layers[i].delta = self.delta

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        d = state_dict.get(prefix + 'pna_delta')
        if d is not None and bool(torch.isfinite(d)):
            self.set_delta(float(d))

    def _prepare(self, g):
        """Loads the kernels and the graph's scalers before any halo wait can spin (both may wait for the device)."""
        from .. import ops
        ops.pna_preload()
        if self.delta is None:
            raise RuntimeError("PNA: delta is not set (train through RankEngine, or load a checkpoint)")
        g.pna_scalers(self.delta)

    def forward(self, g, feat, in_deg=None):
        self._prepare(g)
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._prepare(g)
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))


class _KeepMaskLayers(GraphSAGE):
    """The layer loop of a model whose graph layers take the keep mask of this epoch's boundary-node sample as their
    third argument (`GENConv`, `ResGatedGCN`) and whose kernels `_preload` loads before any halo wait can spin."""

    def _layer_arg(self, in_deg):
        """The keep mask of this epoch's boundary-node sample (training with sampling), else None."""
        buf = self._buffer() if self.training else None
        return getattr(buf, 'keep_mask', None) if buf is not None else None

    def _preload(self):
        raise NotImplementedError

    def forward(self, g, feat, in_deg=None):
        self._preload()
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._preload()
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))


class GENConv(_KeepMaskLayers):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=0, buffer=None,
                 dtype=torch.float32, t=1.0, learn_t=False):
        self.t, self.learn_t = float(t), bool(learn_t)
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)

    def _graph_layer(self, i, d_in, d_out):
        return GENConvLayer(d_in, d_out, t=self.t, learn_t=self.learn_t)

    def _preload(self):
        from .. import ops
        ops.genconv_preload()


class ResGatedGCN(_KeepMaskLayers):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=0, buffer=None,
                 dtype=torch.float32):
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)

    def _graph_layer(self, i, d_in, d_out):
        return ResGatedLayer(d_in, d_out)

    def _preload(self):
        from .. import ops
        ops.resgated_preload()


class MoNet(GraphSAGE):

    def __init__(self, layer_size, activation, dropout=0.5, norm='layer', train_size=None, n_linear=0, buffer=None,
                 dtype=torch.float32, n_kernels=3):
        self.n_kernels = int(n_kernels)
        super().__init__(layer_size, activation, False, dropout=dropout, norm=norm, train_size=train_size,
                         n_linear=n_linear, buffer=buffer, dtype=dtype)

    def _graph_layer(self, i, d_in, d_out):
        return MoNetLayer(d_in, d_out, self.n_kernels)

    def _layer_arg(self, in_deg):
        """MoNet layers take no degrees: the pseudo-coordinates and the row lengths live on the graph."""
        return None

    def _prepare(self, g):
        """Loads the kernels and the graph's reciprocal row lengths before any halo wait can spin (both may wait for
        the device)."""
        from .. import ops
        ops.monet_preload()
        g.inv_row_degrees()

    def forward(self, g, feat, in_deg=None):
        self._prepare(g)
        return super().forward(g, feat, in_deg)

    def forward_partitioned(self, g, xch, pp_feat=None, push0=False):
        self._prepare(g)
        return (yield from super().forward_partitioned(g, xch, pp_feat, push0))
