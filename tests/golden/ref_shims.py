"""Shims that let the UNMODIFIED reference modules run on a host without GPU, DGL or ogb.

Used only by tests/golden/make_golden.py (which needs a PipeGCN checkout;
its outputs are the committed fixtures).  Two things are stood in for:

1. CUDA: the reference needs a GPU even on its gloo path (`torch.cuda.Stream()`, `device='cuda'` buffers,
   `.cuda()`, pinned host memory: PipeGCN/helper/feature_buffer.py:72-75,84,98,109-112;
   PipeGCN/helper/reducer.py:19-21; PipeGCN/train.py:74-81,300).  Streams and events carry
   no values, so they become no-ops and every 'cuda' tensor lives on the host: the arithmetic the reference
   performs is unchanged.
2. DGL (absent, unpinned fork): only the graph CONTAINER the reference's set-up helpers and layer use --
   `dgl.graph`, `dgl.heterograph`, `edges/out_edges/out_degrees/num_nodes/add_nodes`, `update_all(copy_src,
   sum)` written as `index_add_` -- none of the reference's own logic.
"""
from __future__ import annotations

import contextlib
import sys
import types

import torch


# ------------------------------------------------------------------------------------------------ CUDA -> host
class _Stream:
    def wait_stream(self, other):
        pass

    def wait_event(self, ev):
        pass

    def synchronize(self):
        pass


class _Event:
    def __init__(self, *a, **k):
        pass

    def record(self, stream=None):
        pass

    def synchronize(self):
        pass


def _strip_cuda(kwargs):
    dev = kwargs.get("device", None)
    if dev is not None and "cuda" in str(dev):
        kwargs["device"] = "cpu"
    kwargs.pop("pin_memory", None)
    return kwargs


def install_cuda_shims():
    torch.cuda.Stream = lambda *a, **k: _Stream()
    torch.cuda.Event = _Event
    torch.cuda.current_stream = lambda *a, **k: _Stream()
    torch.cuda.stream = lambda s: contextlib.nullcontext()
    torch.cuda.reset_peak_memory_stats = lambda *a, **k: None
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.pin_memory = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    for name in ("zeros", "ones", "empty", "arange", "tensor", "zeros_like", "full"):
        orig = getattr(torch, name)

        def make(orig):
            def f(*a, **k):
                return orig(*a, **_strip_cuda(k))
            return f
        setattr(torch, name, make(orig))
    orig_device = torch.device

    class _Dev:
        def __new__(cls, *a, **k):
            if a and "cuda" in str(a[0]):
                return orig_device("cpu")
            return orig_device(*a, **k)
    torch.device = _Dev


# ------------------------------------------------------------------------------------------------ DGL container
NID = "_ID"


class _Data(dict):
    pass


class _NodeView:
    def __init__(self, g):
        self.g = g

    def __getitem__(self, ntype):
        return types.SimpleNamespace(data=self.g._ndata.setdefault(ntype, _Data()))


class FakeGraph:
    """Homogeneous (`ntypes=None`) or bipartite `_U -> _V` graph holding an edge list."""

    def __init__(self, u, v, n_u=None, n_v=None, bipartite=False):
        self.u, self.v = u, v
        self.bipartite = bipartite
        if bipartite:
            self._n = {"_U": int(n_u if n_u is not None else (int(u.max()) + 1 if u.numel() else 0)),
                       "_V": int(n_v if n_v is not None else (int(v.max()) + 1 if v.numel() else 0))}
        else:
            n = max(int(u.max()) + 1 if u.numel() else 0, int(v.max()) + 1 if v.numel() else 0)
            self._n = {None: int(n_u) if n_u is not None else n}
        self._ndata = {}
        self.ndata, self.edata = _Data(), _Data()
        self.nodes = _NodeView(self)

    # container API used by PipeGCN/train.py and module/layer.py
    def edges(self):
        return self.u.clone(), self.v.clone()

    def num_nodes(self, ntype=None):
        return self._n[ntype]

    def num_edges(self):
        return int(self.u.numel())

    def clone(self):
        g = FakeGraph(self.u.clone(), self.v.clone(), bipartite=self.bipartite)
        g._n = dict(self._n)
        return g

    def int(self):
        g = self.clone()
        g.u, g.v = g.u.int(), g.v.int()
        return g

    def to(self, device):
        return self

    def add_nodes(self, n, ntype=None):
        self._n[ntype] += int(n)

    def out_degrees(self, nodes):
        return torch.bincount(self.u.long(), minlength=self.num_nodes())[nodes.long()]

    def out_edges(self, nodes):
        """(src, dst) of the out-edges of `nodes`, grouped by node in the given order, edge-id order inside."""
        n = self.num_nodes()
        order = torch.argsort(self.u.long(), stable=True)
        counts = torch.bincount(self.u.long(), minlength=n)
        ptr = torch.zeros(n + 1, dtype=torch.int64)
        ptr[1:] = torch.cumsum(counts, 0)
        nodes = nodes.long()
        deg = counts[nodes]
        rep = torch.repeat_interleave(torch.arange(nodes.numel()), deg)
        offs = torch.arange(int(deg.sum())) - torch.repeat_interleave(torch.cumsum(deg, 0) - deg, deg)
        eids = order[ptr[nodes][rep] + offs]
        return self.u[eids], self.v[eids]

    def in_degrees(self):
        return torch.bincount(self.v.long(), minlength=self.num_nodes())

    @contextlib.contextmanager
    def local_scope(self):
        saved = {k: _Data(v) for k, v in self._ndata.items()}
        try:
            yield
        finally:
            self._ndata = saved

    def __getitem__(self, etype):
        return self

    def update_all(self, msg, red, etype=None):
        """update_all(fn.copy_src(src, out), fn.sum(msg, out)): h_v = sum over edges u->v of h_u."""
        assert msg[0] == "copy_src" and red[0] == "sum"
        if self.bipartite:
            h = self._ndata["_U"][msg[1]]
            out = torch.zeros(self._n["_V"], h.shape[1], dtype=h.dtype).index_add_(0, self.v.long(), h[self.u.long()])
            self._ndata.setdefault("_V", _Data())[red[2]] = out
        else:
            h = self.ndata[msg[1]]
            self.ndata[red[2]] = torch.zeros(self.num_nodes(), h.shape[1], dtype=h.dtype).index_add_(
                0, self.v.long(), h[self.u.long()])


def install_dgl_shim():
    dgl = types.ModuleType("dgl")
    dgl.NID = NID
    dgl.graph = lambda uv, **k: FakeGraph(uv[0], uv[1])
    dgl.heterograph = lambda d, **k: FakeGraph(*list(d.values())[0], bipartite=True)
    fn = types.ModuleType("dgl.function")
    fn.copy_src = lambda src, out: ("copy_src", src, out)
    fn.sum = lambda msg, out: ("sum", msg, out)
    dgl.function = fn
    data = types.ModuleType("dgl.data")
    data.RedditDataset = None
    distm = types.ModuleType("dgl.distributed")
    distm.partition_graph = None
    distm.load_partition = None
    dgl.data, dgl.distributed = data, distm
    ogb = types.ModuleType("ogb")
    ogbn = types.ModuleType("ogb.nodeproppred")
    ogbn.DglNodePropPredDataset = None
    ogb.nodeproppred = ogbn
    for name, mod in (("dgl", dgl), ("dgl.function", fn), ("dgl.data", data), ("dgl.distributed", distm),
                      ("ogb", ogb), ("ogb.nodeproppred", ogbn)):
        sys.modules[name] = mod
