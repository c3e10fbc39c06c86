"""`GraphSAGELayer`: neighbour mean + two linears, on the sm_90a kernels.

API and parameters of PipeGCN/module/layer.py:8-63 (state_dict keys
`linear1.*`, `linear2.*`, or `linear.*` with use_pp; init U(-1/sqrt(in), 1/sqrt(in))
for weights and biases drawn in the reference's order so that equal seeds give equal
weights).  `graph` is a `pipegcn_b200.graph.PartGraph` instead of a DGL heterograph.

    training:  out = feat[:N_in] @ W1^T + b1 + ((A @ feat) / in_deg) @ W2^T + b2      (layer.py:44-51)
    eval:      same on a homogeneous graph, degrees taken from the graph               (layer.py:52-62)
"""
import math

import torch
from torch import nn

from .. import ops


class GraphSAGELayer(nn.Module):

    def __init__(self, in_feats, out_feats, bias=True, use_pp=False):
        super().__init__()
        self.in_feats, self.out_feats, self.use_pp = in_feats, out_feats, use_pp
        if use_pp:
            self.linear = nn.Linear(2 * in_feats, out_feats, bias=bias)
        else:
            self.linear1 = nn.Linear(in_feats, out_feats, bias=bias)
            self.linear2 = nn.Linear(in_feats, out_feats, bias=bias)
        self.reset_parameters()

    def _linears(self):
        return [self.linear] if self.use_pp else [self.linear1, self.linear2]

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
        respect to F then includes the dropout backward (fused into the transposed aggregate's store)."""
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
