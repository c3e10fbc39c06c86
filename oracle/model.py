"""Oracle: GraphSAGE-mean layer and model (SURVEY.md §8a rows B1-B6), CPU fp32.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates
PipeGCN/module/layer.py and PipeGCN/module/model.py with DGL's
`update_all(fn.copy_src, fn.sum)` (layer.py:47-49) written as the 0/1 CSR product
`A @ X` and its autograd as `A^T @ g`.
"""
from __future__ import annotations

import math

import torch
from torch import nn


class OracleGraph:
    """Bipartite `_U` -> `_V` graph of one rank: 0/1 CSR `A [N_in, num_all]` and its transpose (int64)."""

    def __init__(self, u: torch.Tensor, v: torch.Tensor, num_in: int, num_all: int):
        self.num_in, self.num_all = int(num_in), int(num_all)
        self.A = _csr(v, u, self.num_in)
        self.At = _csr(u, v, self.num_all)

    def num_nodes(self, ntype):
        return self.num_all if ntype == "_U" else self.num_in


def _csr(rows, cols, n_rows):
    order = torch.argsort(rows, stable=True)          # edge order inside a row = edge-list order
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n_rows), 0)
    return indptr.contiguous(), cols[order].to(torch.int64).contiguous()


def spmm_sum(csr, x: torch.Tensor) -> torch.Tensor:
    """out[r] = sum_{e in row r} x[indices[e]]  -- oracle/csrc/spmm.c (layer.py:47-49)."""
    from .cbuild import lib
    indptr, indices = csr
    x = x.detach().contiguous().float()
    out = torch.empty(indptr.numel() - 1, x.shape[1], dtype=torch.float32)
    lib().oracle_spmm_sum_f32(indptr.data_ptr(), indices.data_ptr(), x.data_ptr(), out.data_ptr(),
                              indptr.numel() - 1, x.shape[1])
    return out


class _CopySrcSum(torch.autograd.Function):
    """h_v = sum over edges u->v of h_u   (DGL gspmm copy_lhs/sum and its backward on the reversed graph)."""

    @staticmethod
    def forward(ctx, graph, feat):
        ctx.graph = graph
        return spmm_sum(graph.A, feat)

    @staticmethod
    def backward(ctx, g):
        return None, spmm_sum(ctx.graph.At, g)


class OracleSageLayer(nn.Module):
    def __init__(self, in_feats, out_feats, bias=True, use_pp=False):    # layer.py:10-22
        super().__init__()
        self.use_pp = use_pp
        if use_pp:
            self.linear = nn.Linear(2 * in_feats, out_feats, bias=bias)
        else:
            self.linear1 = nn.Linear(in_feats, out_feats, bias=bias)
            self.linear2 = nn.Linear(in_feats, out_feats, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):                                          # layer.py:24-36
        if self.use_pp:
            stdv = 1.0 / math.sqrt(self.linear.weight.size(1))
            self.linear.weight.data.uniform_(-stdv, stdv)
            if self.linear.bias is not None:
                self.linear.bias.data.uniform_(-stdv, stdv)
        else:
            stdv = 1.0 / math.sqrt(self.linear1.weight.size(1))
            self.linear1.weight.data.uniform_(-stdv, stdv)
            self.linear2.weight.data.uniform_(-stdv, stdv)
            if self.linear1.bias is not None:
                self.linear1.bias.data.uniform_(-stdv, stdv)
                self.linear2.bias.data.uniform_(-stdv, stdv)

    def forward(self, graph, feat, in_deg, trace=None):                  # layer.py:38-51 (train branch)
        if self.use_pp:
            return self.linear(feat)
        degs = in_deg.unsqueeze(1)
        num_dst = graph.num_nodes("_V")
        ah = _CopySrcSum.apply(graph, feat) / degs
        if trace is not None:
            trace["ah"] = ah.detach().clone()
        return self.linear1(feat[0:num_dst]) + self.linear2(ah)


class OracleGraphSAGE(nn.Module):
    def __init__(self, layer_size, activation, use_pp, dropout=0.5, norm="layer", train_size=None, n_linear=0):
        super().__init__()                                               # model.py:9-39
        self.n_layers = len(layer_size) - 1
        self.layers = nn.ModuleList()
        self.activation = activation
        self.use_pp = use_pp
        self.n_linear = n_linear
        self.use_norm = norm is not None
        if self.use_norm:
            self.norm = nn.ModuleList()
        self.dropout = nn.Dropout(p=dropout)
        for i in range(self.n_layers):
            if i < self.n_layers - self.n_linear:
                self.layers.append(OracleSageLayer(layer_size[i], layer_size[i + 1], use_pp=use_pp))
            else:
                self.layers.append(nn.Linear(layer_size[i], layer_size[i + 1]))
            if i < self.n_layers - 1 and self.use_norm:
                if norm == "layer":
                    self.norm.append(nn.LayerNorm(layer_size[i + 1], elementwise_affine=True))
                else:
                    raise NotImplementedError("SyncBatchNorm is out of scope (SURVEY.md §2.1 #4)")
            use_pp = False

    def forward(self, g, feat, in_deg, buffer, trace=None):             # model.py:41-58
        h = feat
        for i in range(self.n_layers):
            tr = None if trace is None else trace.setdefault(i, {})
            if i < self.n_layers - self.n_linear:
                if self.training and (i > 0 or not self.use_pp):
                    h = buffer.update(i, h)
                if tr is not None:
                    tr["f_buf"] = h.detach().clone()           # what the layer consumes (before dropout)
                h = self.dropout(h)
                h = self.layers[i](g, h, in_deg, trace=tr)
            else:
                h = self.dropout(h)
                h = self.layers[i](h)
            if tr is not None:
                tr["layer_out"] = h.detach().clone()
            if i < self.n_layers - 1:
                if self.use_norm:
                    h = self.norm[i](h)
                h = self.activation(h)
        return h
