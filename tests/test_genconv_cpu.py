"""Softmax-aggregation graph convolution (`--model genconv`) without a GPU: the hand-written forward and backward the
kernels implement (log-sum-exp L, agg, var, Q = t g_S agg, the source pass and dt) against fp64 autograd through a
plain-torch restatement of PyG's GENConv, the partitioned layer over [inner | halo] rows against the whole graph, the
sampled form against the sampled graph, the parser, the refused configurations, and the keys, shapes and draw order.

`handwritten_forward` / `handwritten_backward` are the fp64 restatement the GPU tests compare against."""
import argparse
import math

import pytest
import torch

from tests.test_pna_cpu import graph_case

EPS_MSG = 1e-7
TEMPS = [-0.5, 0.0, 0.1, 1.0, 20.0]


# ------------------------------------------------------------------------------------------------ restatement
def pyg_forward(h, rows, cols, num_in, t, w_src, w_dst, w1, w2, store=None):
    """PyG's GENConv(aggr='softmax', norm=None, bias=False, num_layers=2) without edge features: lin_src / lin_dst
    (None when d_in == d), messages ReLU(x_src[u]) + eps, a scatter softmax of t * m with max subtraction, a scatter
    sum, then the MLP on agg + x_dst.  `t` may be a tensor that requires grad.  `store` rounds (with a straight-through
    gradient) where the engine stores values: x_src, x_dst, S and the MLP hidden layer."""
    store = store or (lambda x: x)
    xs = store(h @ w_src.T) if w_src is not None else h
    xd = store(h[:num_in] @ w_dst.T) if w_dst is not None else h[:num_in]
    d = xs.shape[1]
    m = torch.relu(xs[cols]) + EPS_MSG
    s = t * m
    idx = rows[:, None].expand(-1, d)
    mx = torch.full((num_in, d), float("-inf"), dtype=h.dtype, device=h.device).scatter_reduce(0, idx, s.detach(), "amax",
                                                                           include_self=True)
    e = torch.exp(s - mx[rows])
    den = torch.zeros(num_in, d, dtype=h.dtype, device=h.device).index_add(0, rows, e)
    a = e / den[rows]
    agg = torch.zeros(num_in, d, dtype=h.dtype, device=h.device).index_add(0, rows, a * m)
    return store(torch.relu(store(agg + xd) @ w1.T)) @ w2.T


def _kept_edges(rows, cols, num_in, keep):
    if keep is None:
        return rows, cols
    ok = (cols < num_in) | keep[(cols - num_in).clamp(min=0)].bool()
    return rows[ok], cols[ok]


def handwritten_forward(h, rows, cols, num_in, t, w_src, w_dst, w1, w2, keep=None, store=None):
    """The layer as the kernels compute it, in h's dtype, with the sources of unkept halo rows (keep: uint8 mask of
    rows >= num_in) left out.  Returns out and the intermediates.  `store` rounds where the engine stores values
    (x_src, S, the MLP hidden layer)."""
    store = store or (lambda x: x)
    rows, cols = _kept_edges(rows, cols, num_in, keep)
    xs = store(h @ w_src.T) if w_src is not None else h
    xd = store(h[:num_in] @ w_dst.T) if w_dst is not None else h[:num_in]
    d = xs.shape[1]
    m = torch.relu(xs) + EPS_MSG
    tm = t * m
    idx = rows[:, None].expand(-1, d)
    mx = torch.full((num_in, d), float("-inf"), dtype=h.dtype, device=h.device).scatter_reduce(0, idx, tm[cols], "amax")
    has = torch.bincount(rows, minlength=num_in)[:, None] > 0
    msafe = torch.where(has, mx, torch.zeros_like(mx))
    w = torch.zeros(num_in, d, dtype=h.dtype, device=h.device).index_add(0, rows, torch.exp(tm[cols] - msafe[rows]))
    lse = torch.where(has, msafe + torch.log(torch.where(has, w, torch.ones_like(w))), torch.full_like(w, -math.inf))
    a = torch.exp(tm[cols] - lse[rows])                 # per edge: exp(t m_u - L_v), never exp(t m_u) exp(-L_v)
    agg = torch.zeros(num_in, d, dtype=h.dtype, device=h.device).index_add(0, rows, a * m[cols])
    sq = torch.zeros(num_in, d, dtype=h.dtype, device=h.device).index_add(0, rows, a * m[cols] ** 2)
    var = torch.clamp(sq - agg ** 2, min=0)
    s = store(agg + xd)
    hid = torch.relu(s @ w1.T)
    r = store(hid)
    out = r @ w2.T
    return out, dict(xs=xs, m=m, tm=tm, lse=lse, agg=agg, var=var, s=s, r=r, rows=rows, cols=cols)


def handwritten_backward(g, h, num_in, t, w_src, w_dst, w1, w2, st, keep=None):
    """The kernels' backward from the forward's intermediates: g_S through the MLP, Q = t g_S agg, the source pass
    dm_u = sum_v exp(t m_u - L_v) (G_v (1 + t m_u) - Q_v), dx_src = [x_src > 0] dm, dt = sum g_S var, and the
    weight and input gradients."""
    rows, cols = st["rows"], st["cols"]
    num_all = h.shape[0]
    g_r = g @ w2
    g_h = g_r * (st["r"] > 0)
    gs = g_h @ w1
    q = t * gs * st["agg"]
    e = torch.exp(st["tm"][cols] - st["lse"][rows])
    term = e * (gs[rows] * (1 + st["tm"][cols]) - q[rows])
    dm = torch.zeros(num_all, gs.shape[1], dtype=h.dtype, device=h.device).index_add(0, cols, term)
    dxs = torch.where(st["xs"] > 0, dm, torch.zeros_like(dm))
    dt = (gs * st["var"]).sum()
    out = dict(gs=gs, q=q, dxs=dxs, dt=dt, w2=g.T @ st["r"], w1=g_h.T @ st["s"])
    if w_src is not None:
        gh = dxs @ w_src
        gh[:num_in] += gs @ w_dst
        out.update(w_src=dxs.T @ h, w_dst=gs.T @ h[:num_in])
    else:
        gh = dxs.clone()
        gh[:num_in] += gs
    out["h"] = gh
    return out


def weights(d_in, d, seed, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    ws = (scale * r(d, d_in) / math.sqrt(d_in)) if d_in != d else None
    wd = (r(d, d_in) / math.sqrt(d_in)) if d_in != d else None
    return ws, wd, r(2 * d, d) / math.sqrt(d), r(d, 2 * d) / math.sqrt(2 * d)


# ------------------------------------------------------------------------------------------------ formulas
@pytest.mark.parametrize("t", TEMPS)
@pytest.mark.parametrize("d_in,d", [(6, 6), (6, 5)])
def test_handwritten_layer_matches_pyg_autograd(t, d_in, d):
    h, rows, cols, num_in = graph_case(seed=3, d=d_in)
    h = 6.0 * h                                  # |t m| up to > 100 at t = 20: the softmax saturates to one-hot
    ws, wd, w1, w2 = weights(d_in, d, seed=11)
    out, st = handwritten_forward(h, rows, cols, num_in, t, ws, wd, w1, w2)
    assert torch.all(st["agg"][0] == 0) and torch.all(torch.isinf(st["lse"][0]))       # no in-edges
    if ws is None:
        assert (t * (torch.relu(h) + EPS_MSG)).abs().max() > 100 or t != 20.0
    leaves = [x.clone().requires_grad_(True) if x is not None else None for x in (h, ws, wd, w1, w2)]
    tt = torch.tensor(t, dtype=torch.float64, requires_grad=True)
    ref = pyg_forward(leaves[0], rows, cols, num_in, tt, *leaves[1:])
    assert torch.allclose(out, ref, rtol=1e-10, atol=1e-10)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    ref.backward(g)
    got = handwritten_backward(g, h, num_in, t, ws, wd, w1, w2, st)
    names = ["h", "w_src", "w_dst", "w1", "w2"]
    for name, leaf in zip(names, leaves):
        if leaf is not None:
            assert torch.allclose(got[name], leaf.grad, rtol=1e-9, atol=1e-9), name
    assert math.isclose(float(got["dt"]), float(tt.grad), rel_tol=1e-9, abs_tol=1e-9)


def test_all_equal_and_self_loop_rows():
    h, rows, cols, num_in = graph_case(seed=1, d=4)
    _, st = handwritten_forward(h, rows, cols, num_in, 1.5, None, None, *weights(4, 4, 2)[2:])
    m = torch.relu(h) + EPS_MSG
    for v in (1, 2, 5):             # one source, or sources with equal rows: agg = m, var = 0
        assert torch.allclose(st["agg"][v], m[v], rtol=1e-15, atol=0)
        assert torch.all(st["var"][v] <= 1e-15)


def test_sampled_form_equals_the_sampled_graph():
    """Unkept halo rows leave every softmax: the masked formulas equal autograd on the graph without their edges, and
    unkept rows get exactly zero gradient."""
    h, rows, cols, num_in = graph_case(seed=4, d=6)
    num_all = h.shape[0]
    keep = (torch.arange(num_all - num_in) % 3 != 0).to(torch.uint8)
    t = 0.7
    ws, wd, w1, w2 = weights(6, 5, seed=9)
    out, st = handwritten_forward(h, rows, cols, num_in, t, ws, wd, w1, w2, keep=keep)
    kr, kc = _kept_edges(rows, cols, num_in, keep)
    leaves = [x.clone().requires_grad_(True) for x in (h, ws, wd, w1, w2)]
    tt = torch.tensor(t, dtype=torch.float64, requires_grad=True)
    ref = pyg_forward(leaves[0], kr, kc, num_in, tt, *leaves[1:])
    assert torch.allclose(out, ref, rtol=1e-10, atol=1e-10)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    ref.backward(g)
    got = handwritten_backward(g, h, num_in, t, ws, wd, w1, w2, st, keep=keep)
    assert torch.allclose(got["h"], leaves[0].grad, rtol=1e-9, atol=1e-9)
    unkept = num_in + torch.nonzero(keep == 0)[:, 0]
    assert torch.all(got["dxs"][unkept] == 0)
    assert math.isclose(float(got["dt"]), float(tt.grad), rel_tol=1e-9, abs_tol=1e-9)


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_partitioned_layer_equals_whole_graph(n_parts, metis):
    """fp64: every partition's layer over its [inner | halo] rows gives the whole graph's rows, and the partitions'
    weight, temperature and input gradients add up to the whole graph's."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    part = random_partition(g.n_nodes, n_parts)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    lays = build_layouts(g, part, n_parts)
    n, d_in, d, t = g.n_nodes, 7, 5, 0.8
    gen = torch.Generator().manual_seed(n_parts)
    x = torch.randn(n, d_in, generator=gen, dtype=torch.float64)
    ws, wd, w1, w2 = weights(d_in, d, seed=n_parts)
    gout = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lay_edges = []
    for lay in lays:
        r = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
        lay_edges.append((r, lay.indices.long()))
    # whole graph, from the layouts' edges in global ids
    grows, gcols = [], []
    for lay, (r, c) in zip(lays, lay_edges):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        grows.append(gid[r])
        gcols.append(gid[c])
    grows, gcols = torch.cat(grows), torch.cat(gcols)
    order = torch.argsort(grows, stable=True)
    whole, st = handwritten_forward(x, grows[order], gcols[order], n, t, ws, wd, w1, w2)
    ref = handwritten_backward(gout, x, n, t, ws, wd, w1, w2, st)
    acc = {k: torch.zeros_like(ref[k]) for k in ("w_src", "w_dst", "w1", "w2", "dt", "h")}
    for lay, (r, c) in zip(lays, lay_edges):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        inner = lay.inner_gid.long()
        out, pst = handwritten_forward(x[gid], r, c, lay.num_in, t, ws, wd, w1, w2)
        assert torch.allclose(out, whole[inner], rtol=1e-12, atol=1e-12)
        got = handwritten_backward(gout[inner], x[gid], lay.num_in, t, ws, wd, w1, w2, pst)
        for k in ("w_src", "w_dst", "w1", "w2", "dt"):
            acc[k] = acc[k] + got[k]
        acc["h"].index_add_(0, gid, got["h"])
    for k, v in acc.items():
        assert torch.allclose(v, ref[k], rtol=1e-10, atol=1e-10), k


# ------------------------------------------------------------------------------------------------ parser / model
def test_parser_flags_and_an_unchanged_namespace():
    from pipegcn_b200.helper.parser import create_parser
    a = create_parser(["--model", "genconv", "--genconv-t", "-0.5", "--genconv-learn-t"])
    assert a.model == "genconv" and a.genconv_t == -0.5 and a.genconv_learn_t is True
    assert create_parser(["--genconv_t", "0"]).genconv_t == 0.0
    base = vars(create_parser([]))
    with_model = vars(create_parser(["--model", "genconv"]))
    assert "genconv_t" not in with_model and "genconv_learn_t" not in with_model
    assert with_model.pop("model") == "genconv"
    base.pop("model")
    assert with_model == base
    for bad in ("nan", "inf", "-inf", "x"):
        with pytest.raises(SystemExit):
            create_parser(["--model", "genconv", "--genconv-t", bad])


def _args(**kw):
    base = dict(model="genconv", use_pp=False, n_hidden=16, enable_pipeline=False, feat_corr=False, grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(aggregator="pool"), ValueError, "--model genconv has its own"),
    (dict(use_pp=True), NotImplementedError, "precompute is a neighbour mean"),
    (dict(genconv_t=float("nan")), ValueError, "finite temperature"),
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


def test_sampling_is_accepted():
    from pipegcn_b200.train import check_model
    check_model(_args(sampling_rate=0.5))


def _model(n_linear, learn_t, seed=0, t=None):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    argv = ["--model", "genconv", "--n-hidden", "16", "--n-layers", "3", "--n-linear", str(n_linear)]
    argv += (["--genconv-learn-t"] if learn_t else []) + (["--genconv-t", str(t)] if t is not None else [])
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], create_parser(argv))


@pytest.mark.parametrize("learn_t", [False, True])
@pytest.mark.parametrize("n_linear", [0, 1])
def test_keys_shapes_and_draw_order(n_linear, learn_t):
    from torch import nn
    model = _model(n_linear, learn_t, seed=3, t=0.25)
    sd = model.state_dict()
    sizes = [20, 16, 16, 5]
    torch.manual_seed(3)
    expect = {}
    for i, (d_in, d) in enumerate(zip(sizes[:-1], sizes[1:])):
        if i < 3 - n_linear:
            p = f"layers.{i}."
            if d_in != d:                        # lin_src, lin_dst, mlp.lins.0, mlp.lins.1
                expect[p + "lin_src.weight"] = nn.Linear(d_in, d, bias=False).weight
                expect[p + "lin_dst.weight"] = nn.Linear(d_in, d, bias=False).weight
            expect[p + "mlp.lins.0.weight"] = nn.Linear(d, 2 * d, bias=False).weight
            expect[p + "mlp.lins.1.weight"] = nn.Linear(2 * d, d, bias=False).weight
            if learn_t:
                expect[p + "aggr_module.t"] = torch.tensor([0.25])
            assert model.layers[i].temperature().tolist() == [0.25]
        else:
            lin = nn.Linear(d_in, d)
            expect.update({f"layers.{i}.weight": lin.weight, f"layers.{i}.bias": lin.bias})
        if i < 2:
            expect.update({f"norm.{i}.weight": torch.ones(d), f"norm.{i}.bias": torch.zeros(d)})
    assert set(sd) == set(expect)
    for k, v in expect.items():
        assert torch.equal(sd[k], v.detach()), k
    names = {n for n, _ in model.named_parameters()}
    assert all((f"layers.{i}.aggr_module.t" in names) == learn_t for i in range(3 - n_linear))
    if n_linear == 0:                            # the logits come from a GENConv(d_in, n_class)
        assert sd["layers.2.mlp.lins.1.weight"].shape == (5, 10)
