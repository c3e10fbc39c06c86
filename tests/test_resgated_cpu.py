"""Residual gated graph convolution (`--model resgatedgcn`) without a GPU: the hand-written forward and the two backward
passes the kernels implement (the saturating-safe gate, the destination pass's dk and the source pass's dq and dval)
against fp64 autograd through a plain-torch restatement of PyG's ResGatedGraphConv, the gate's accuracy where it
saturates, the partitioned layer over [inner | halo] rows against the whole graph, the sampled form against the sampled
graph, the parser, the refused configurations, and the keys, shapes and draw order.

`pyg_forward` and `handwritten_forward` / `handwritten_backward` are the fp64 restatements the GPU tests compare
against."""
import argparse
import math

import pytest
import torch

from tests.test_genconv_cpu import _kept_edges
from tests.test_pna_cpu import graph_case

# the state-dict order of ResGatedGraphConv: the module's own parameter first, then its linears
KEYS = ("bias", "lin_key.weight", "lin_key.bias", "lin_query.weight", "lin_query.bias", "lin_value.weight",
        "lin_value.bias", "lin_skip.weight")


# ------------------------------------------------------------------------------------------------ restatement
def pyg_forward(h, rows, cols, num_in, wk, bk, wq, bq, wv, bv, ws, b, store=None):
    """PyG's ResGatedGraphConv (act=Sigmoid, root_weight, bias, aggr='add') without edge features: k from the
    destination rows, q and v from the sources, message sigmoid(k_i + q_j) * v_j summed over the edges cols -> rows,
    plus lin_skip of the destination rows and the bias.  `store` rounds (with a straight-through gradient) where the
    engine stores values: [q | v] and [k | skip + b]."""
    store = store or (lambda x: x)
    k = store(h[:num_in] @ wk.T + bk)
    q, v = store(h @ wq.T + bq), store(h @ wv.T + bv)
    skip = store(h[:num_in] @ ws.T + b)
    msg = torch.sigmoid(k[rows] + q[cols]) * v[cols]
    return torch.zeros_like(skip).index_add(0, rows, msg) + skip


def gate(x):
    """(sigmoid(x), sigmoid'(x)) in x's dtype from one exp, as the kernels evaluate them."""
    e = torch.exp(-x.abs())
    r = 1 / (1 + e)
    er = e * r
    return torch.where(x >= 0, r, er), er * r


def handwritten_forward(h, rows, cols, num_in, wk, bk, wq, bq, wv, bv, ws, b, keep=None):
    """The layer as the kernels compute it, with the sources of unkept halo rows (keep: uint8 mask of rows >= num_in)
    left out.  Returns out and the intermediates."""
    rows, cols = _kept_edges(rows, cols, num_in, keep)
    k, skip = h[:num_in] @ wk.T + bk, h[:num_in] @ ws.T + b
    q, v = h @ wq.T + bq, h @ wv.T + bv
    s, ds = gate(k[rows] + q[cols])
    out = skip + torch.zeros_like(skip).index_add(0, rows, s * v[cols])
    return out, dict(k=k, q=q, v=v, s=s, ds=ds, rows=rows, cols=cols)


def handwritten_backward(g, h, num_in, wk, wq, wv, ws, st):
    """The kernels' backward from G = dL/d out: the destination pass dk[v] = G[v] sum_u sigmoid'(x) val[u], the
    source pass dval[u] = sum_v G[v] sigmoid(x) and dq[u] = val[u] sum_v G[v] sigmoid'(x), then the weight, bias and
    input gradients."""
    rows, cols, v = st["rows"], st["cols"], st["v"]
    num_all, d = h.shape[0], g.shape[1]
    z = lambda n: torch.zeros(n, d, dtype=h.dtype, device=h.device)
    dk = g * z(num_in).index_add(0, rows, st["ds"] * v[cols])
    dval = z(num_all).index_add(0, cols, g[rows] * st["s"])
    dq = v * z(num_all).index_add(0, cols, g[rows] * st["ds"])
    gh = dq @ wq + dval @ wv
    gh[:num_in] += dk @ wk + g @ ws
    hi = h[:num_in]
    return dict(dk=dk, dq=dq, dval=dval, h=gh, wk=dk.T @ hi, bk=dk.sum(0), wq=dq.T @ h, bq=dq.sum(0),
                wv=dval.T @ h, bv=dval.sum(0), ws=g.T @ hi, b=g.sum(0))


def weights(d_in, d, seed, scale=1.0):
    """(wk, bk, wq, bq, wv, bv, ws, b) fp64; `scale` multiplies the gate's weights and biases."""
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    w = lambda: r(d, d_in) / math.sqrt(d_in)
    return scale * w(), scale * r(d), scale * w(), scale * r(d), w(), r(d), w(), r(d)


NAMES = ("wk", "bk", "wq", "bq", "wv", "bv", "ws", "b")


# ------------------------------------------------------------------------------------------------ formulas
@pytest.mark.parametrize("scale", [1.0, 8.0, 40.0])
@pytest.mark.parametrize("d_in,d", [(6, 6), (6, 5), (3, 9)])
def test_handwritten_layer_matches_pyg_autograd(scale, d_in, d):
    """At scale 40 the gate arguments |k + q| reach past 100: every gate is 0 or 1 to the last bit, and sigmoid'
    underflows on some edges; the formulas stay finite and equal autograd of torch.sigmoid."""
    h, rows, cols, num_in = graph_case(seed=3, d=d_in)
    ws_ = weights(d_in, d, seed=11, scale=scale)
    out, st = handwritten_forward(h, rows, cols, num_in, *ws_)
    x = st["k"][rows] + st["q"][cols]
    if scale == 40.0:
        assert float(x.abs().max()) > 100
    assert torch.isfinite(out).all()
    leaves = [h.clone().requires_grad_(True)] + [w.clone().requires_grad_(True) for w in ws_]
    ref = pyg_forward(leaves[0], rows, cols, num_in, *leaves[1:])
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)
    # no in-edges (row 0): skip + b; a self loop only (rows 1, 2): one gate of its own q
    torch.testing.assert_close(out[0], h[0] @ ws_[6].T + ws_[7], rtol=1e-14, atol=1e-14)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    ref.backward(g)
    got = handwritten_backward(g, h, num_in, ws_[0], ws_[2], ws_[4], ws_[6], st)
    for name, leaf in zip(("h",) + NAMES, leaves):
        assert torch.isfinite(got[name]).all(), name
        torch.testing.assert_close(got[name], leaf.grad, rtol=1e-9, atol=1e-9 * (1 + float(leaf.grad.abs().max())),
                                   msg=name)


def test_gate_saturates_without_cancellation():
    """fp32, as the kernels evaluate it: sigmoid within 2 ulp and sigmoid' within 4 ulp of fp64 for |x| up to 100,
    relative to their own size, until sigmoid' leaves the normal range; never Inf or NaN.  1 - sigmoid would lose
    sigmoid' entirely past |x| = 17."""
    x = torch.cat([torch.linspace(-100, 100, 20001), torch.tensor([0.0, -0.0, 1e-30, -1e-30, 85.0, -85.0, 88.8,
                                                                   -88.8, 103.9, -103.9])])
    s, ds = gate(x.float())
    assert torch.isfinite(s).all() and torch.isfinite(ds).all()
    x64 = x.double()
    rs, rds = torch.sigmoid(x64), torch.sigmoid(x64) * torch.sigmoid(-x64)
    ulp = 2.0 ** -23
    assert torch.all(((s.double() - rs).abs() <= 2 * ulp * rs)[rs >= 2.0 ** -126])
    assert torch.all(((s.double() - rs).abs() <= 2.0 ** -148)[rs < 2.0 ** -126])   # subnormal: absolute
    normal = rds >= 2.0 ** -126
    assert torch.all(((ds.double() - rds).abs() <= 4 * ulp * rds)[normal])
    assert torch.all(ds.double()[~normal] <= 2.0 ** -126)            # underflowed: subnormal or 0, never more
    assert bool(normal[x.abs() == 85.0].all())                       # accurate well past where 1 - s is 0
    naive = s * (1 - s)
    assert torch.all(naive[x > 17] == 0) and torch.all(ds[(x > 17) & (x < 80)] > 0)
    assert torch.all(s[x >= 17] == 1) and torch.all(s[x <= -100] > 0)


def test_rows_without_in_edges_and_self_loops():
    h, rows, cols, num_in = graph_case(seed=1, d=4)
    ws_ = weights(4, 4, 2)
    out, st = handwritten_forward(h, rows, cols, num_in, *ws_)
    k, q, v = st["k"], st["q"], st["v"]
    skip = h[:num_in] @ ws_[6].T + ws_[7]
    torch.testing.assert_close(out[0], skip[0], rtol=0, atol=0)
    for r in (1, 2):                 # self loop only: skip + sigmoid(k_v + q_v) v_v
        torch.testing.assert_close(out[r], skip[r] + torch.sigmoid(k[r] + q[r]) * v[r], rtol=1e-15, atol=1e-15)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got = handwritten_backward(g, h, num_in, ws_[0], ws_[2], ws_[4], ws_[6], st)
    assert torch.all(got["dk"][0] == 0)                              # no in-edges: no gate, dk = 0


def test_sampled_form_equals_the_sampled_graph():
    """Unkept halo rows leave every sum: the masked formulas equal autograd on the graph without their edges (no
    rescaling), and unkept rows get exactly zero gradient."""
    h, rows, cols, num_in = graph_case(seed=4, d=6)
    num_all = h.shape[0]
    keep = (torch.arange(num_all - num_in) % 3 != 0).to(torch.uint8)
    ws_ = weights(6, 5, seed=9)
    out, st = handwritten_forward(h, rows, cols, num_in, *ws_, keep=keep)
    kr, kc = _kept_edges(rows, cols, num_in, keep)
    assert len(kr) < len(rows)
    leaves = [h.clone().requires_grad_(True)] + [w.clone().requires_grad_(True) for w in ws_]
    ref = pyg_forward(leaves[0], kr, kc, num_in, *leaves[1:])
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    ref.backward(g)
    got = handwritten_backward(g, h, num_in, ws_[0], ws_[2], ws_[4], ws_[6], st)
    for name, leaf in zip(("h",) + NAMES, leaves):
        torch.testing.assert_close(got[name], leaf.grad, rtol=1e-9, atol=1e-9, msg=name)
    unkept = num_in + torch.nonzero(keep == 0)[:, 0]
    assert torch.all(got["dq"][unkept] == 0) and torch.all(got["dval"][unkept] == 0)
    assert torch.all(got["h"][unkept] == 0)


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_partitioned_layer_equals_whole_graph(n_parts, metis):
    """fp64: every partition's layer over its [inner | halo] rows gives the whole graph's rows, and the partitions'
    weight, bias and input gradients add up to the whole graph's."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    part = random_partition(g.n_nodes, n_parts)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    lays = build_layouts(g, part, n_parts)
    n, d_in, d = g.n_nodes, 7, 5
    gen = torch.Generator().manual_seed(n_parts)
    x = torch.randn(n, d_in, generator=gen, dtype=torch.float64)
    ws_ = weights(d_in, d, seed=n_parts, scale=2.0)
    wmat = (ws_[0], ws_[2], ws_[4], ws_[6])
    gout = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lay_edges = []
    for lay in lays:
        r = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
        lay_edges.append((r, lay.indices.long()))
    grows, gcols = [], []
    for lay, (r, c) in zip(lays, lay_edges):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        grows.append(gid[r])
        gcols.append(gid[c])
    grows, gcols = torch.cat(grows), torch.cat(gcols)
    order = torch.argsort(grows, stable=True)
    whole, st = handwritten_forward(x, grows[order], gcols[order], n, *ws_)
    ref = handwritten_backward(gout, x, n, *wmat, st)
    acc = {k: torch.zeros_like(ref[k]) for k in NAMES + ("h",)}
    for lay, (r, c) in zip(lays, lay_edges):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        inner = lay.inner_gid.long()
        out, pst = handwritten_forward(x[gid], r, c, lay.num_in, *ws_)
        torch.testing.assert_close(out, whole[inner], rtol=1e-12, atol=1e-12)
        got = handwritten_backward(gout[inner], x[gid], lay.num_in, *wmat, pst)
        for k in NAMES:
            acc[k] = acc[k] + got[k]
        acc["h"].index_add_(0, gid, got["h"])
    for k, v in acc.items():
        torch.testing.assert_close(v, ref[k], rtol=1e-10, atol=1e-10, msg=k)


# ------------------------------------------------------------------------------------------------ parser / model
def test_parser_and_an_unchanged_namespace():
    from pipegcn_b200.helper.parser import create_parser
    a = create_parser(["--model", "resgatedgcn", "--n-heads", "8"])
    assert a.model == "resgatedgcn"
    base = vars(create_parser([]))
    with_model = vars(create_parser(["--model", "resgatedgcn"]))
    assert with_model.pop("model") == "resgatedgcn"
    base.pop("model")
    assert with_model == base


def _args(**kw):
    base = dict(model="resgatedgcn", use_pp=False, n_hidden=16, enable_pipeline=False, feat_corr=False,
                grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(aggregator="pool"), ValueError, "--model resgatedgcn has its own"),
    (dict(use_pp=True), NotImplementedError, "precompute is a neighbour mean"),
])
def test_refused_before_allocation(kw, exc, match):
    """RankEngine and init_processes refuse before touching the layout, the world or a device."""
    from pipegcn_b200 import train
    args = _args(**kw)
    with pytest.raises(exc, match=match):
        train.RankEngine(None, args, None)
    with pytest.raises(exc, match=match):
        train.init_processes(0, 2, args)
    with pytest.raises(exc, match=match):
        train.create_model([20, 16, 5], argparse.Namespace(norm='layer', dropout=0.5, n_linear=0, n_train=1,
                                                            **vars(args)))


def test_sampling_and_heads_are_accepted():
    from pipegcn_b200.train import check_model
    check_model(_args(sampling_rate=0.5))
    check_model(_args(n_heads=3))                   # --n-heads is ignored: 16 does not split into 3


def _model(n_linear, seed=0):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    argv = ["--model", "resgatedgcn", "--n-hidden", "16", "--n-layers", "3", "--n-linear", str(n_linear)]
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], create_parser(argv))


@pytest.mark.parametrize("n_linear", [0, 1])
def test_keys_shapes_and_draw_order(n_linear):
    from torch import nn
    from pipegcn_b200.module.model import ResGatedGCN
    model = _model(n_linear, seed=3)
    assert isinstance(model, ResGatedGCN)
    sd = model.state_dict()
    sizes = [20, 16, 16, 5]
    torch.manual_seed(3)
    expect = {}
    for i, (d_in, d) in enumerate(zip(sizes[:-1], sizes[1:])):
        p = f"layers.{i}."
        if i < 3 - n_linear:                     # lin_key, lin_query, lin_value, lin_skip, then bias = 0
            for name in ("lin_key", "lin_query", "lin_value"):
                lin = nn.Linear(d_in, d)
                expect.update({p + name + ".weight": lin.weight, p + name + ".bias": lin.bias})
            expect[p + "lin_skip.weight"] = nn.Linear(d_in, d, bias=False).weight
            expect[p + "bias"] = torch.zeros(d)
        else:
            lin = nn.Linear(d_in, d)
            expect.update({p + "weight": lin.weight, p + "bias": lin.bias})
        if i < 2:
            expect.update({f"norm.{i}.weight": torch.ones(d), f"norm.{i}.bias": torch.zeros(d)})
    assert set(sd) == set(expect)
    for k, v in expect.items():
        assert torch.equal(sd[k], v.detach()), k
    assert [k for k in sd if k.startswith("layers.0.")] == [f"layers.0.{k}" for k in KEYS]
    if n_linear == 0:                            # the logits come from a ResGatedLayer(d_in, n_class)
        assert sd["layers.2.lin_skip.weight"].shape == (5, 16) and sd["layers.2.bias"].shape == (5,)
