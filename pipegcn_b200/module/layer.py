"""`GraphSAGELayer`: neighbour mean + two linears, on the sm_90a kernels.

API and parameters of PipeGCN/module/layer.py:8-63 (state_dict keys
`linear1.*`, `linear2.*`, or `linear.*` with use_pp; init U(-1/sqrt(in), 1/sqrt(in))
for weights and biases drawn in the reference's order so that equal seeds give equal
weights).  `graph` is a `pipegcn_b200.graph.PartGraph` instead of a DGL heterograph.

    training:  out = feat[:N_in] @ W1^T + b1 + ((A @ feat) / in_deg) @ W2^T + b2      (layer.py:44-51)
    eval:      same on a homogeneous graph, degrees taken from the graph               (layer.py:52-62)

`aggregator='pool'` (not in the reference): the max-pool aggregator of DGL's `SAGEConv(aggregator_type='pool')`, with
a third linear `pool` [d_in, d_in] (state-dict keys `pool.weight` / `pool.bias`, drawn after linear1 and linear2):

    out = feat[:N_in] @ W1^T + b1 + ReLU(max_{u -> v} (feat[u] @ Wp^T + bp)) @ W2^T + b2

the same in training and evaluation (a row without in-edges aggregates to 0).

`GATLayer` (not in the reference): DGL's `GATConv` with feat_drop = attn_drop = 0, no residual, negative_slope 0.2,
over the `[inner | halo]` rows h the halo exchange returns (inner rows v, in-edges u -> v, per head):

    z = h @ W^T,  el = <z, attn_l>,  er = <z, attn_r>,
    out[v] = sum_u softmax_u(LeakyReLU(el[u] + er[v])) z[u] + bias

State-dict keys are GATConv's: `fc.weight` [H*D, d_in], `attn_l` / `attn_r` [1, H, D], `bias` [H*D].

`GATv2Layer` (not in the reference): DGL's `GATv2Conv` with share_weights=False, bias=True, feat_drop = attn_drop = 0,
no residual, negative_slope 0.2 (Brody et al., "How Attentive are Graph Attention Networks?", ICLR 2022), over the
same rows, per head k:

    zs = h @ W_s^T + b_s  (every row),  zd = h[:N_in] @ W_d^T + b_d  (destination rows),
    e_uv = <attn[k], LeakyReLU(zs[u, k] + zd[v, k])>,
    out[v, k] = sum_u softmax_u(e_uv) zs[u, k]                    (no output bias; 0 for a row without in-edges)

State-dict keys are GATv2Conv's: `fc_src.weight` / `fc_dst.weight` [H*D, d_in], `fc_src.bias` / `fc_dst.bias` [H*D],
`attn` [1, H, D].  Initialisation is GATv2Conv.reset_parameters, in this draw order, with
gain = calculate_gain('relu'): xavier_normal_(fc_src.weight), fc_src.bias = 0, xavier_normal_(fc_dst.weight),
fc_dst.bias = 0, xavier_normal_(attn).

`TransformerLayer` (not in the reference): PyG's `TransformerConv` with concat=True, beta=False, dropout=0,
edge_dim=None, bias=True, root_weight=True (Shi et al., "Masked Label Prediction: Unified Message Passing Model for
Semi-Supervised Classification", IJCAI 2021), over the same rows, per head k:

    q = h[:N_in] @ W_q^T + b_q,  k = h @ W_k^T + b_k,  v = h @ W_v^T + b_v,  skip = h[:N_in] @ W_s^T + b_s,
    e_uv = <q[v, k], k[u, k]> / sqrt(D),
    out[v, k] = sum_u softmax_u(e_uv) v[u, k] + skip[v, k]       (attention part 0 for a row without in-edges)

State-dict keys are TransformerConv's: `lin_query.*`, `lin_key.*`, `lin_value.*`, `lin_skip.*`, weights [H*D, d_in]
and biases [H*D].  Initialisation is TransformerConv.reset_parameters, in this draw order, each PyG `Linear` drawing
as `nn.Linear` does (weight kaiming_uniform_(a=sqrt(5)), then bias U(-1/sqrt(d_in), 1/sqrt(d_in))): lin_key,
lin_query, lin_value, lin_skip.

`GraphConvLayer` (not in the reference): DGL's `GraphConv(in, out, norm='both', weight=True, bias=True)` (Kipf & Welling,
"Semi-Supervised Classification with Graph Convolutional Networks", ICLR 2017), no activation inside, over the same
rows, with c = clamp(deg, min=1)^(-1/2) of every [inner | halo] row (deg: in-degree with the self loop in the whole
graph; the halo rows' values come from their owners, `PartGraph.sym_norm`):

    out[v] = c[v] * sum_{u -> v} c[u] h[u] @ W + b

aggregating first when d_in <= d_out, transforming first otherwise (DGL's rule; PG_NARROW=0 always aggregates first).
State-dict keys are GraphConv's: `weight` [d_in, d_out] (not transposed like nn.Linear), `bias` [d_out].
Initialisation is GraphConv.reset_parameters, in this draw order: xavier_uniform_(weight), then bias = 0.
With --use-pp layer 0 multiplies the precomputed rows c[v] * sum_u c[u] x[u] by the same weight.

`GCNIILayer` (not in the reference): one convolution of GCNII (Chen et al., "Simple and Deep Graph Convolutional
Networks", ICML 2020), DGL's `GCN2Conv(d, layer=l, alpha, lambda_, project_initial_features=True, bias=True)`, no
activation inside, over the same rows and with the same c as GraphConvLayer.  Convolution l = i + 1 of graph layer i:

    S   = (1 - alpha) * c[v] * sum_{u -> v} c[u] h[u] + alpha * h0[v]
    out = (1 - beta_l) * S + beta_l * S @ W1 + b,      beta_l = ln(lambda / l + 1)

h0 = ReLU(fc_in(dropout(x))) is the model's initial representation; graph layer 0 holds `fc_in` (an nn.Linear
[d, n_feat], default initialisation, drawn first) in front of its convolution and computes it over every [inner | halo]
row of x.  State-dict keys: `fc_in.weight` / `fc_in.bias` (layer 0 only), `weight1` [d, d] (in x out, DGL's layout),
`bias` [d].  Initialisation is the GCNII authors': weight1 ~ U(-1/sqrt(d), 1/sqrt(d)), then bias = 0.

`PNALayer` (not in the reference): principal neighbourhood aggregation (Corso et al., "Principal Neighbourhood
Aggregation for Graph Nets", NeurIPS 2020), DGL's `PNAConvTower` with aggregators mean, max, min, std, scalers
identity, amplification, attenuation, one tower and no edge features, over the same rows.  With D_v the in-degree of v
(its CSR row length, self loop included) and delta the mean of log(D + 1) over the training graph:

    m_uv    = M(cat(h[u], h[v])) = zs[u] + zd[v],   zs = h @ W_s^T,  zd = h[:N_in] @ W_d^T + b_M   (M.weight = [W_s | W_d])
    agg_v   = [mean_u m_uv | max_u m_uv | min_u m_uv | std_u m_uv]                                 (4 d_in)
    h_neigh = [agg_v | a_v agg_v | t_v agg_v],   a_v = log(D_v + 1) / delta,  t_v = delta / log(D_v + 1)
    out[v]  = U(cat(h[v], h_neigh))                                                                   (13 d_in -> d_out)

The std is sqrt(max(var, 0) + 1e-30) of the messages; it equals that of zs (the shift zd[v] cancels), so it is computed
over zs alone (DGL takes relu(E[m^2] - E[m]^2) over the messages).  A row without in-edges gets h_neigh = 0, as DGL does
not reduce a node without messages.  Left out of DGL's tower: the graph-size norm, the tower's batch norm and dropout
(the model's loop supplies LayerNorm, ReLU and dropout between layers); there is no mixing layer and no residual.
State-dict keys: `M.weight` [d_in, 2 d_in], `M.bias`, `U.weight` [d_out, 13 d_in], `U.bias`, both `nn.Linear` with
the default initialisation, M drawn before U.  delta is not a layer parameter: the model sets it (`PNA.set_delta`).

`GENConvLayer` (not in the reference): the softmax-aggregation graph convolution of DeeperGCN (Li et al., "DeeperGCN:
All You Need to Train Deeper GCNs", 2020), PyG's `GENConv(d_in, d, aggr='softmax', t=T, learn_t=L, norm=None,
num_layers=2, expansion=2, eps=1e-7, bias=False)` without edge features or message norm, over the same rows:

    x_src = h @ W_src^T  (h itself when d_in == d),   x_dst = h[:N_in] @ W_dst^T  (h[:N_in] when d_in == d)
    m_u   = ReLU(x_src[u]) + 1e-7
    agg_v = sum_{u -> v} softmax_u(t m_u) * m_u       (per channel; 0 for a row without in-edges)
    out   = ReLU((agg + x_dst) @ W1^T) @ W2^T         (W1 [2d, d], W2 [d, 2d]: PyG's MLP with norm=None)

With boundary-node sampling the sums cover the inner and the kept halo sources only.  t is a scalar: with `learn_t`
a `Parameter` of shape [1] initialised to T (key `aggr_module.t`), else a constant outside the state dict, as in PyG.
State-dict keys: `lin_src.weight` and `lin_dst.weight` [d, d_in] (only when d_in != d), `mlp.lins.0.weight`
[2d, d], `mlp.lins.1.weight` [d, 2d] and `aggr_module.t`.  Every weight is drawn as `nn.Linear` draws it
(kaiming_uniform_(a=sqrt(5))), in the order lin_src, lin_dst, mlp.lins.0, mlp.lins.1.  PyG draws some of them twice
(at construction and in reset_parameters), so equal seeds do not give PyG's initial weights.

`ResGatedLayer` (not in the reference): the residual gated graph convolution of Bresson & Laurent ("Residual Gated
Graph ConvNets", 2017), PyG's `ResGatedGraphConv(d_in, d_out, act=Sigmoid(), edge_dim=None, root_weight=True,
bias=True)` with aggr='add', over the same rows, per channel:

    k = h[:N_in] @ W_k^T + b_k,  q = h @ W_q^T + b_q,  val = h @ W_v^T + b_v,  skip = h[:N_in] @ W_s^T
    out[v] = skip[v] + b + sum_{u -> v} sigmoid(k[v] + q[u]) * val[u]      (skip + b for a row without in-edges)

Each edge has its own gate and nothing normalises the gates over the in-edges: with boundary-node sampling the unkept
halo sources are absent from every sum, which is exactly the layer over the sampled graph (no rescaling).  State-dict
keys are ResGatedGraphConv's: `lin_key.*`, `lin_query.*`, `lin_value.*` (weights [d_out, d_in] and biases [d_out]),
`lin_skip.weight` [d_out, d_in] (no bias) and `bias` [d_out].  Each linear is drawn as `nn.Linear` draws it
(kaiming_uniform_(a=sqrt(5)), then its bias U(-1/sqrt(d_in), 1/sqrt(d_in))), in the order lin_key, lin_query,
lin_value, lin_skip, then bias = 0.  PyG draws the linears twice (at construction and in reset_parameters), so equal
seeds do not give PyG's initial weights.

`MoNetLayer` (not in the reference): the Gaussian mixture model convolution of MoNet (Monti et al., "Geometric deep
learning on graphs and manifolds using mixture model CNNs", CVPR 2017), DGL's `GMMConv(d_in, d_out, dim=2,
n_kernels=K, aggregator_type='mean', residual=False, bias=True)` with the degree pseudo-coordinates of DGL's MoNet
citation example (without its per-layer `pseudo_proj`), over the same rows.  c = clamp(deg, min=1)^(-1/2) of every
[inner | halo] row (deg: in-degree with the self loop in the whole graph; the halo rows' values come from their
owners, `PartGraph.sym_norm`), deg_v the CSR row length of v:

    e_uv   = (c[u], c[v])                                                 pseudo-coordinates of u -> v
    w_k(e) = exp(-1/2 sum_j (e_j - mu[k, j])^2 inv_sigma[k, j]^2)         k = 0..K-1, j = 0, 1
    z_u[k] = h[u] @ W_k^T,   W_k = fc.weight[k d_out:(k + 1) d_out]       (fc has no bias)
    out[v] = (1/deg_v) sum_{u -> v} sum_k w_k(e_uv) z_u[k] + bias

It aggregates first when d_in <= K d_out (A_v[k] = (1/deg_v) sum_u w_k(e_uv) h[u], then one GEMM of A [N_in, K d_in]
with the k-major B[k d_in + i, m] = W_k[m, i]), and transforms first otherwise (z over every row, then the
mixture-weighted mean of its K slices); the rule follows from the shapes alone.  The gradients, with G = dL/d out and
s_k(e_uv) = dL/dw_k(e_uv):

    aggregate first:  dA_v[k] = G_v @ W_k,  s_k(e_uv) = <dA_v[k], h[u]> / deg_v,
                      dh[u] = sum_{v: u -> v} (1/deg_v) sum_k w_k(e_uv) dA_v[k],  dfc = G^T A (permuted back)
    transform first:  dz_u[k] = sum_{v: u -> v} (w_k(e_uv) / deg_v) G_v,  s_k(e_uv) = <G_v, z_u[k]> / deg_v,
                      dh = dz @ fc.weight,  dfc = dz^T h
    both:             dmu[k, j] = sum_e s_k w_k (e_j - mu[k, j]) inv_sigma[k, j]^2
                      dinv_sigma[k, j] = -sum_e s_k w_k (e_j - mu[k, j])^2 inv_sigma[k, j],  dbias = sum_v G_v

Every edge lives in the CSR of its destination's rank, so each rank's mu / inv_sigma gradient covers its own edges and
the all-reduce of the gradients sums them.  State-dict keys are GMMConv's: `mu` [K, 2], `inv_sigma` [K, 2],
`fc.weight` [K d_out, d_in], `bias` [d_out].  Initialisation follows GMMConv's constructor and draw order: fc is built
as `nn.Linear(bias=False)` (drawing its default initialisation), then reset_parameters draws
xavier_normal_(fc.weight, gain=calculate_gain('relu')), then normal_(mu, 0, 0.1), then inv_sigma = 1 and bias = 0.
"""
import math

import torch
from torch import nn

from .. import ops


class GraphSAGELayer(nn.Module):

    def __init__(self, in_feats, out_feats, bias=True, use_pp=False, aggregator='mean'):
        super().__init__()
        self.in_feats, self.out_feats, self.use_pp = in_feats, out_feats, use_pp
        if aggregator not in ('mean', 'pool'):
            raise ValueError(f"aggregator '{aggregator}': expected 'mean' or 'pool'")
        if aggregator == 'pool' and use_pp:
            raise NotImplementedError("the pool aggregator with use_pp: the precompute is a neighbour mean")
        self.aggregator = aggregator
        if use_pp:
            self.linear = nn.Linear(2 * in_feats, out_feats, bias=bias)
        else:
            self.linear1 = nn.Linear(in_feats, out_feats, bias=bias)
            self.linear2 = nn.Linear(in_feats, out_feats, bias=bias)
        if aggregator == 'pool':
            self.pool = nn.Linear(in_feats, in_feats, bias=bias)
        self.reset_parameters()

    def _linears(self):
        if self.use_pp:
            return [self.linear]
        return [self.linear1, self.linear2] + ([self.pool] if self.aggregator == 'pool' else [])

    def reset_parameters(self):
        lins = self._linears()
        bound = 1. / math.sqrt(lins[0].weight.size(1))
        # weights first, then biases -- the draw order of layer.py:24-36
        for lin in lins:
            lin.weight.data.uniform_(-bound, bound)
        for lin in lins:
            if lin.bias is not None:
                lin.bias.data.uniform_(-bound, bound)

    def forward(self, graph, feat, in_deg, drop_bwd=None):
        """`drop_bwd` (not in the reference): `feat` is already dropout(F) under that key -- the layer's gradient with
        respect to F then includes the dropout backward (fused into the transposed aggregate's store).  A pool layer
        takes the keep mask of the halo rows (boundary-node sampling, uint8) or None in place of `in_deg`."""
        if self.aggregator == 'pool':
            return ops.sage_pool_layer(feat, graph, in_deg if self.training else None, self.linear1.weight,
                                       self.linear1.bias, self.linear2.weight, self.linear2.bias, self.pool.weight,
                                       self.pool.bias, drop_bwd)
        if self.training:
            if self.use_pp:
                return ops.linear(feat, self.linear.weight, self.linear.bias)
            return ops.sage_layer(feat, graph, graph.deg_as_float(in_deg), self.linear1.weight, self.linear1.bias,
                                  self.linear2.weight, self.linear2.bias, drop_bwd)
        assert in_deg is None
        ah = ops.sage_aggregate(feat, graph, graph.row_degrees())
        # a partition's graph (partitioned evaluation): feat holds [inner | halo] rows, the outputs are the inner rows
        x = feat[:graph.num_in] if feat.shape[0] != graph.num_in else feat
        if self.use_pp:
            return ops.linear(torch.cat((x, ah), dim=1), self.linear.weight, self.linear.bias)
        return ops.sage_linear(x, ah, self.linear1.weight, self.linear1.bias,
                               self.linear2.weight, self.linear2.bias)


class GraphConvLayer(nn.Module):
    """GraphConv(in_feats, out_feats, norm='both', weight=True, bias=True), no activation inside: module docstring."""

    def __init__(self, in_feats, out_feats, use_pp=False):
        super().__init__()
        self.in_feats, self.out_feats, self.use_pp = in_feats, out_feats, use_pp
        self.weight = nn.Parameter(torch.empty(in_feats, out_feats))
        self.bias = nn.Parameter(torch.empty(out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        """GraphConv.reset_parameters."""
        nn.init.xavier_uniform_(self.weight)
        nn.init.zeros_(self.bias)

    def pp_linear(self, pp_feat):
        """--use-pp layer 0: the precomputed c_v sum_u c_u x_u rows times W, plus b."""
        return ops.linear(pp_feat, self.weight.t(), self.bias)

    def forward(self, graph, feat, in_deg=None, drop_bwd=None):
        """`feat`: the [num_all, d_in] rows of `graph`, or with --use-pp (layer 0, training) the precomputed rows;
        returns the [N_in, d_out] inner rows.  `in_deg` is unused: the norm is `graph.sym_norm()`.  `drop_bwd` as
        GraphSAGELayer.forward."""
        if self.use_pp and self.training:
            return self.pp_linear(feat)
        return ops.graphconv_layer(feat, graph, graph.sym_norm(), self.weight, self.bias, drop_bwd)


class GCNIILayer(nn.Module):
    """GCN2Conv(d, layer=i+1, alpha, lambda_, project_initial_features=True, bias=True), no activation inside, with
    fc_in in front of it in graph layer 0: module docstring."""

    def __init__(self, in_feats, out_feats, layer, alpha=0.1, lam=0.5):
        super().__init__()
        if layer > 0 and in_feats != out_feats:
            raise ValueError(f"GCNII convolution {layer + 1}: {in_feats} -> {out_feats} is not square")
        self.in_feats, self.out_feats, self.layer = in_feats, out_feats, layer
        self.alpha, self.lam = float(alpha), float(lam)
        self.beta = ops.gcnii_beta(self.lam, layer + 1)
        if layer == 0:
            self.fc_in = nn.Linear(in_feats, out_feats)
        self.weight1 = nn.Parameter(torch.empty(out_feats, out_feats))
        self.bias = nn.Parameter(torch.empty(out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        """The GCNII authors' initialisation of the convolution (fc_in keeps nn.Linear's, drawn at construction)."""
        stdv = 1.0 / math.sqrt(self.out_feats)
        nn.init.uniform_(self.weight1, -stdv, stdv)
        nn.init.zeros_(self.bias)

    def forward(self, graph, feat, state, drop_bwd=None):
        """`feat`: the [num_all, d_in] rows of `graph` (layer 0: the dropped input features); `state`: the
        `ops.GCNIIState` of this forward (layer 0 fills its h0).  Returns the [N_in, d] inner rows.  `drop_bwd` as
        GraphSAGELayer.forward."""
        c, cs = graph.sym_norm(), graph.gcnii_norm(self.alpha)
        if self.layer == 0:
            return ops.gcnii_first(feat, graph, c, cs, self.fc_in.weight, self.fc_in.bias, self.weight1, self.bias,
                                   self.alpha, self.beta, state)
        return ops.gcnii_conv(feat, graph, c, cs, self.weight1, self.bias, self.alpha, self.beta, state, drop_bwd)


class GATLayer(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads):
        super().__init__()
        self.in_feats, self.out_feats, self.num_heads = in_feats, out_feats, num_heads
        self.fc = nn.Linear(in_feats, out_feats * num_heads, bias=False)
        self.attn_l = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.attn_r = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.bias = nn.Parameter(torch.empty(num_heads * out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        """GATConv.reset_parameters."""
        gain = nn.init.calculate_gain('relu')
        nn.init.xavier_normal_(self.fc.weight, gain=gain)
        nn.init.xavier_normal_(self.attn_l, gain=gain)
        nn.init.xavier_normal_(self.attn_r, gain=gain)
        nn.init.constant_(self.bias, 0)

    def forward(self, graph, feat, keep=None, drop_bwd=None):
        """`feat`: the [num_all, d_in] rows of `graph` (a partition's `[inner | halo]`, or a whole graph); returns the
        [N_in, H*D] inner rows.  `keep`: uint8 keep mask of the halo rows (boundary-node sampling) or None.
        `drop_bwd`: `feat` already is dropout(F) under that key; the gradient returned is the one with respect to F."""
        return ops.gat_layer(feat, graph, keep, self.num_heads, self.fc.weight, self.attn_l, self.attn_r, self.bias,
                             drop_bwd)


class GATv2Layer(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads):
        super().__init__()
        self.in_feats, self.out_feats, self.num_heads = in_feats, out_feats, num_heads
        self.fc_src = nn.Linear(in_feats, out_feats * num_heads, bias=True)
        self.fc_dst = nn.Linear(in_feats, out_feats * num_heads, bias=True)
        self.attn = nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        """GATv2Conv.reset_parameters (share_weights=False)."""
        gain = nn.init.calculate_gain('relu')
        nn.init.xavier_normal_(self.fc_src.weight, gain=gain)
        nn.init.constant_(self.fc_src.bias, 0)
        nn.init.xavier_normal_(self.fc_dst.weight, gain=gain)
        nn.init.constant_(self.fc_dst.bias, 0)
        nn.init.xavier_normal_(self.attn, gain=gain)

    def forward(self, graph, feat, keep=None, drop_bwd=None):
        """As GATLayer.forward."""
        return ops.gatv2_layer(feat, graph, keep, self.num_heads, self.fc_src.weight, self.fc_src.bias,
                               self.fc_dst.weight, self.fc_dst.bias, self.attn, drop_bwd)


class TransformerLayer(nn.Module):

    def __init__(self, in_feats, out_feats, num_heads):
        super().__init__()
        self.in_feats, self.out_feats, self.num_heads = in_feats, out_feats, num_heads
        self.lin_key = nn.Linear(in_feats, out_feats * num_heads)
        self.lin_query = nn.Linear(in_feats, out_feats * num_heads)
        self.lin_value = nn.Linear(in_feats, out_feats * num_heads)
        self.lin_skip = nn.Linear(in_feats, out_feats * num_heads)
        self.reset_parameters()

    def reset_parameters(self):
        """TransformerConv.reset_parameters (beta=False, root_weight=True)."""
        for lin in (self.lin_key, self.lin_query, self.lin_value, self.lin_skip):
            lin.reset_parameters()

    def forward(self, graph, feat, keep=None, drop_bwd=None):
        """As GATLayer.forward."""
        return ops.transformer_layer(feat, graph, keep, self.num_heads, self.lin_query.weight, self.lin_query.bias,
                                     self.lin_key.weight, self.lin_key.bias, self.lin_value.weight,
                                     self.lin_value.bias, self.lin_skip.weight, self.lin_skip.bias, drop_bwd)


class PNALayer(nn.Module):

    def __init__(self, in_feats, out_feats):
        super().__init__()
        self.in_feats, self.out_feats = in_feats, out_feats
        self.M = nn.Linear(2 * in_feats, in_feats)
        self.U = nn.Linear(13 * in_feats, out_feats)
        self.delta = None

    def forward(self, graph, feat, arg=None, drop_bwd=None):
        """As GraphSAGELayer.forward; `arg` is unused (the scalers live on the graph, `PartGraph.pna_scalers`)."""
        if self.delta is None:
            raise RuntimeError("PNALayer: delta is not set (PNA.set_delta, set by the trainer or a loaded checkpoint)")
        return ops.pna_layer(feat, graph, self.delta, self.M.weight, self.M.bias, self.U.weight, self.U.bias, drop_bwd)


class _GenConvMLP(nn.Module):
    """PyG's MLP([d, 2d, d], norm=None, bias=False) as a container of its two linears (keys `lins.0`, `lins.1`)."""

    def __init__(self, d):
        super().__init__()
        self.lins = nn.ModuleList([nn.Linear(d, 2 * d, bias=False), nn.Linear(2 * d, d, bias=False)])


class _SoftmaxAggr(nn.Module):
    """PyG's SoftmaxAggregation(learn=True, channels=1): the learnable temperature `t` [1]."""

    def __init__(self, t):
        super().__init__()
        self.t = nn.Parameter(torch.tensor([float(t)], dtype=torch.float32))


class GENConvLayer(nn.Module):

    def __init__(self, in_feats, out_feats, t=1.0, learn_t=False):
        super().__init__()
        if not math.isfinite(float(t)):
            raise ValueError(f"GENConv: temperature {t} is not finite")
        self.in_feats, self.out_feats, self.learn_t = in_feats, out_feats, bool(learn_t)
        if in_feats != out_feats:
            self.lin_src = nn.Linear(in_feats, out_feats, bias=False)
            self.lin_dst = nn.Linear(in_feats, out_feats, bias=False)
        else:
            self.lin_src = self.lin_dst = None
        self.mlp = _GenConvMLP(out_feats)
        if self.learn_t:
            self.aggr_module = _SoftmaxAggr(t)
        else:
            # a constant the kernels read from device memory; not part of the state dict
            self.register_buffer('t_const', torch.tensor([float(t)], dtype=torch.float32), persistent=False)

    def temperature(self) -> torch.Tensor:
        return self.aggr_module.t if self.learn_t else self.t_const

    def forward(self, graph, feat, keep=None, drop_bwd=None):
        """As GATLayer.forward: `feat` [num_all, d_in] rows of `graph`, `keep` the keep mask of the halo rows
        (boundary-node sampling, uint8) or None; returns the [N_in, d] inner rows."""
        return ops.genconv_layer(feat, graph, keep, self.temperature(),
                                 self.lin_src.weight if self.lin_src is not None else None,
                                 self.lin_dst.weight if self.lin_dst is not None else None,
                                 self.mlp.lins[0].weight, self.mlp.lins[1].weight, drop_bwd)


class ResGatedLayer(nn.Module):
    """ResGatedGraphConv(in_feats, out_feats), sigmoid gate, root weight and bias: module docstring."""

    def __init__(self, in_feats, out_feats):
        super().__init__()
        self.in_feats, self.out_feats = in_feats, out_feats
        self.lin_key = nn.Linear(in_feats, out_feats)
        self.lin_query = nn.Linear(in_feats, out_feats)
        self.lin_value = nn.Linear(in_feats, out_feats)
        self.lin_skip = nn.Linear(in_feats, out_feats, bias=False)
        self.bias = nn.Parameter(torch.zeros(out_feats))

    def forward(self, graph, feat, keep=None, drop_bwd=None):
        """As GATLayer.forward: `feat` [num_all, d_in] rows of `graph`, `keep` the keep mask of the halo rows
        (boundary-node sampling, uint8) or None; returns the [N_in, d_out] inner rows."""
        return ops.resgated_layer(feat, graph, keep, self.lin_key.weight, self.lin_key.bias, self.lin_query.weight,
                                  self.lin_query.bias, self.lin_value.weight, self.lin_value.bias,
                                  self.lin_skip.weight, self.bias, drop_bwd)


class MoNetLayer(nn.Module):
    """GMMConv(in_feats, out_feats, dim=2, n_kernels, aggregator_type='mean') on the degree pseudo-coordinates: module
    docstring."""

    def __init__(self, in_feats, out_feats, n_kernels=3):
        super().__init__()
        self.in_feats, self.out_feats, self.n_kernels = in_feats, out_feats, n_kernels
        self.mu = nn.Parameter(torch.empty(n_kernels, 2))
        self.inv_sigma = nn.Parameter(torch.empty(n_kernels, 2))
        self.fc = nn.Linear(in_feats, n_kernels * out_feats, bias=False)
        self.bias = nn.Parameter(torch.empty(out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        """GMMConv.reset_parameters."""
        nn.init.xavier_normal_(self.fc.weight, gain=nn.init.calculate_gain('relu'))
        nn.init.normal_(self.mu.data, 0, 0.1)
        nn.init.constant_(self.inv_sigma.data, 1)
        nn.init.zeros_(self.bias.data)

    def forward(self, graph, feat, in_deg=None, drop_bwd=None):
        """`feat`: the [num_all, d_in] rows of `graph`; returns the [N_in, d_out] inner rows.  `in_deg` is unused: the
        pseudo-coordinates are `graph.sym_norm()` and the mean divides by the CSR row lengths.  `drop_bwd` as
        GraphSAGELayer.forward."""
        return ops.monet_layer(feat, graph, self.fc.weight, self.mu, self.inv_sigma, self.bias, drop_bwd)
