"""`GraphSAGE` (alias `GCN`): the layer loop of PipeGCN/module/model.py:25-58.

Per graph layer: `buffer.update` (halo exchange) -> dropout -> GraphSAGELayer -> norm ->
activation; trailing `n_linear` plain linears.  The reference defines no `GCN` class
(SURVEY.md §0.2): the north-star's `module.model.GCN` is this class under a second name.
state_dict keys match the reference (`layers.{i}.linear1.weight`, `norm.{i}.weight`, ...).

Extra keyword arguments (not in the reference): `buffer` -- the exchange object to use
instead of the process-global `helper.context.buffer` (several simulated ranks in one
process); `dtype` -- activation storage type, float32 (reference) or bfloat16 (fp32
accumulate, fp32 master weights).
"""
import torch
from torch import nn
import torch.nn.functional as F

from ..helper import context as ctx
from .layer import GraphSAGELayer


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
                 buffer=None, dtype=torch.float32):
        super().__init__(layer_size, activation, use_pp, dropout, norm, n_linear)
        self.buffer = buffer
        self.act_dtype = dtype
        for i, (d_in, d_out) in enumerate(zip(layer_size[:-1], layer_size[1:])):
            if i < self.n_graph_layers:
                self.layers.append(GraphSAGELayer(d_in, d_out, use_pp=(use_pp and i == 0)))
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

    def _drop(self, h):
        from .. import ops
        return ops.dropout(h, self.dropout.p, self.training)

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
        h = feat if feat.dtype == self.act_dtype else feat.to(self.act_dtype)
        p = self.dropout.p if self.training else 0.0
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
                    h = layer(g, self._drop(h), in_deg)
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
        h = None
        for i, layer in enumerate(self.layers):
            if i < self.n_graph_layers:
                if i == 0 and self.use_pp:
                    h = ops.linear(pp_feat, layer.linear.weight, layer.linear.bias)
                else:
                    d = layer.in_feats
                    if i > 0 or push0:
                        xch.push(i, d)
                        yield i
                        xch.wait(i)
                    h = layer(g, xch.rows(i, d), None)
            else:
                h = ops.linear(h, layer.weight, layer.bias)
            if i < self.n_layers - 1:
                dest = xch.inner(i + 1, h.shape[1]) if i + 1 < self.n_graph_layers else None
                out = self._norm_act(i, h, dest)
                if dest is not None and out.data_ptr() != dest.data_ptr():
                    dest.copy_(out)
                h = out
        return h


GCN = GraphSAGE
