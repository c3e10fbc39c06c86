"""Gaussian mixture model convolution (`--model monet`) without a GPU: the parser and the refused configurations, the
parameters and their draw order, the factorised forward and backward of both evaluation orders against fp64 autograd
through DGL's unfactorised per-edge definition, the order rule, and the partitioned layer against the whole graph.

`dgl_forward` is the fp64 restatement the GPU tests compare against."""
import argparse

import pytest
import torch


# ------------------------------------------------------------------------------------------------ restatement
def pseudo_coords(c, rows, cols):
    """e_uv = (c[u], c[v]) of every edge cols[e] = u -> rows[e] = v."""
    return torch.stack([c[cols], c[rows]], 1)


def mixture_weights(e, mu, inv_sigma):
    """w [E, K] = exp(-1/2 sum_j (e_j - mu[k, j])^2 inv_sigma[k, j]^2), DGL's GMMConv."""
    g = -0.5 * (e[:, None, :] - mu[None]) ** 2 * inv_sigma[None] ** 2
    return torch.exp(g.sum(-1))


def dgl_forward(h, rows, cols, num_in, c, fc_w, mu, inv_sigma, bias):
    """DGL's GMMConv(aggregator_type='mean') over the edge list, unfactorised: every edge carries its K transformed
    messages w_k(e) z_u[k], the mean over the in-edges per kernel, then the sum over the kernels and the bias."""
    k = mu.shape[0]
    z = (h @ fc_w.T).view(h.shape[0], k, -1)
    w = mixture_weights(pseudo_coords(c, rows, cols), mu, inv_sigma)
    m = z[cols] * w[:, :, None]
    deg = torch.bincount(rows, minlength=num_in).clamp(min=1).to(h.dtype)
    agg = torch.zeros(num_in, k, z.shape[2], dtype=h.dtype, device=h.device).index_add(0, rows, m) / deg[:, None, None]
    return agg.sum(1) + bias


def handwritten(h, rows, cols, num_in, c, fc_w, mu, inv_sigma, bias, G, aggregate_first):
    """The factorised forward and backward the kernels and GEMMs compute (module/layer.py), in either order."""
    n_all, d_in = h.shape
    k = mu.shape[0]
    d_out = fc_w.shape[0] // k
    W = fc_w.view(k, d_out, d_in)
    e = pseudo_coords(c, rows, cols)
    w = mixture_weights(e, mu, inv_sigma)
    deg = torch.bincount(rows, minlength=num_in).clamp(min=1).to(h.dtype)
    rd = 1.0 / deg[rows]
    if aggregate_first:
        A = torch.zeros(num_in, k, d_in, dtype=h.dtype).index_add(0, rows, w[:, :, None] * h[cols][:, None, :])
        A = A / deg[:, None, None]
        out = torch.einsum('vki,kmi->vm', A, W) + bias
        dA = torch.einsum('vm,kmi->vki', G, W)
        s = (dA[rows] * h[cols][:, None, :]).sum(-1) * rd[:, None]
        dh = torch.zeros(n_all, d_in, dtype=h.dtype).index_add(
            0, cols, ((w * rd[:, None])[:, :, None] * dA[rows]).sum(1))
        dfc = torch.einsum('vm,vki->kmi', G, A).reshape(k * d_out, d_in)
    else:
        z = (h @ fc_w.T).view(n_all, k, d_out)
        out = torch.zeros(num_in, d_out, dtype=h.dtype).index_add(0, rows, (w[:, :, None] * z[cols]).sum(1))
        out = out / deg[:, None] + bias
        dz = torch.zeros(n_all, k, d_out, dtype=h.dtype).index_add(
            0, cols, (w * rd[:, None])[:, :, None] * G[rows][:, None, :])
        s = (G[rows][:, None, :] * z[cols]).sum(-1) * rd[:, None]
        dh = dz.reshape(n_all, k * d_out) @ fc_w
        dfc = dz.reshape(n_all, k * d_out).T @ h
    diff = e[:, None, :] - mu[None]
    sw = (s * w)[:, :, None]
    dmu = (sw * diff).sum(0) * inv_sigma ** 2
    dinv = -(sw * diff ** 2).sum(0) * inv_sigma
    return dict(out=out, h=dh, fc=dfc, mu=dmu, inv_sigma=dinv, bias=G.sum(0))


def graph_case(seed=0, num_in=30, num_halo=12, d_in=6):
    """(h, rows, cols, num_in, c): a partition-shaped graph in which every inner row has its self loop, degrees vary
    from 1 to 8, and c = deg^-1/2 of every row (the halo rows' degrees drawn as their owners would know them)."""
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    h = torch.randn(num_all, d_in, generator=gen, dtype=torch.float64)
    rows, cols = [], []
    for v in range(num_in):
        n = int(torch.randint(0, 8, (1,), generator=gen))
        src = list(dict.fromkeys([v] + torch.randperm(num_all, generator=gen)[:n].tolist()))
        rows += [v] * len(src)
        cols += src
    rows, cols = torch.tensor(rows), torch.tensor(cols)
    deg = torch.cat([torch.bincount(rows, minlength=num_in),
                     torch.randint(1, 12, (num_halo,), generator=gen)]).double()
    return h, rows, cols, num_in, deg.clamp(min=1) ** -0.5


def params(d_in, d_out, k, seed, isg=1.0, mu_scale=0.3):
    gen = torch.Generator().manual_seed(seed + 100)
    fc_w = torch.randn(k * d_out, d_in, generator=gen, dtype=torch.float64) * 0.5
    mu = 0.5 + mu_scale * torch.randn(k, 2, generator=gen, dtype=torch.float64)
    inv_sigma = isg * (0.5 + torch.rand(k, 2, generator=gen, dtype=torch.float64))
    bias = torch.randn(d_out, generator=gen, dtype=torch.float64)
    return fc_w, mu, inv_sigma, bias


def autograd_reference(h, rows, cols, num_in, c, fc_w, mu, inv_sigma, bias, G):
    leaves = [t.clone().requires_grad_(True) for t in (h, fc_w, mu, inv_sigma, bias)]
    out = dgl_forward(leaves[0], rows, cols, num_in, c, *leaves[1:])
    out.backward(G)
    return dict(out=out.detach(), **{n: t.grad for n, t in zip(("h", "fc", "mu", "inv_sigma", "bias"), leaves)})


# ------------------------------------------------------------------------------------------------ formulas
@pytest.mark.parametrize("aggregate_first", [True, False])
@pytest.mark.parametrize("k,d_out", [(1, 4), (3, 5), (8, 2)])
@pytest.mark.parametrize("isg", [1.0, 2000.0])
def test_handwritten_layer_matches_dgl_autograd(aggregate_first, k, d_out, isg):
    """isg = 2000: most weights underflow to exactly 0, and some rows have no edge with a nonzero weight."""
    h, rows, cols, num_in, c = graph_case(seed=k)
    fc_w, mu, inv_sigma, bias = params(h.shape[1], d_out, k, seed=k, isg=isg)
    if isg > 1:
        mu[:, 0], mu[:, 1] = c[cols[:k]], c[rows[:k]]      # centred on real edges, so not every weight is 0
        w = mixture_weights(pseudo_coords(c, rows, cols), mu, inv_sigma)
        assert (w == 0).any() and (w > 0).any()
        row_w = torch.zeros(num_in, dtype=torch.float64).index_add(0, rows, w.sum(1))
        assert (row_w == 0).any()
    G = torch.randn(num_in, d_out, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    ref = autograd_reference(h, rows, cols, num_in, c, fc_w, mu, inv_sigma, bias, G)
    got = handwritten(h, rows, cols, num_in, c, fc_w, mu, inv_sigma, bias, G, aggregate_first)
    for name, v in ref.items():
        torch.testing.assert_close(got[name], v, rtol=1e-11, atol=1e-11, msg=name)


def test_order_rule_on_both_sides():
    from pipegcn_b200.ops import monet_aggregate_first
    assert monet_aggregate_first(768, 256, 3) and not monet_aggregate_first(769, 256, 3)
    assert monet_aggregate_first(256, 256, 3) and monet_aggregate_first(602, 256, 3)
    assert not monet_aggregate_first(256, 64, 3) and not monet_aggregate_first(256, 41, 3)
    assert monet_aggregate_first(8, 8, 1) and not monet_aggregate_first(9, 8, 1)


def test_slices_are_whole_vectors():
    from pipegcn_b200.ops import monet_slice
    assert [monet_slice(d, torch.float32) for d in (1, 4, 5, 602)] == [4, 4, 8, 604]
    assert [monet_slice(d, torch.bfloat16) for d in (1, 8, 9, 41)] == [8, 8, 16, 48]


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
@pytest.mark.parametrize("aggregate_first", [True, False])
def test_partitioned_layer_equals_whole_graph(n_parts, metis, aggregate_first):
    """fp64: every partition's layer over its [inner | halo] rows, with c of the halo rows from their owners (the
    global degrees), gives the whole graph's rows; the partitions' fc, mu, inv_sigma, bias and input gradients add up
    to the whole graph's."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    part = random_partition(g.n_nodes, n_parts)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    lays = build_layouts(g, part, n_parts)
    n, d_in, d_out, k = g.n_nodes, 7, 5, 3
    gen = torch.Generator().manual_seed(n_parts)
    x = torch.randn(n, d_in, generator=gen, dtype=torch.float64)
    fc_w, mu, inv_sigma, bias = params(d_in, d_out, k, seed=n_parts)
    gout = torch.randn(n, d_out, generator=gen, dtype=torch.float64)
    lay_edges, grows, gcols = [], [], []
    for lay in lays:
        r = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
        lay_edges.append((r, lay.indices.long()))
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        grows.append(gid[r])
        gcols.append(gid[lay.indices.long()])
    grows, gcols = torch.cat(grows), torch.cat(gcols)
    order = torch.argsort(grows, stable=True)
    c = torch.bincount(grows, minlength=n).clamp(min=1).double() ** -0.5
    ref = handwritten(x, grows[order], gcols[order], n, c, fc_w, mu, inv_sigma, bias, gout, aggregate_first)
    acc = {key: torch.zeros_like(v) for key, v in ref.items() if key != "out"}
    for lay, (r, cc) in zip(lays, lay_edges):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        inner = lay.inner_gid.long()
        got = handwritten(x[gid], r, cc, lay.num_in, c[gid], fc_w, mu, inv_sigma, bias, gout[inner], aggregate_first)
        torch.testing.assert_close(got["out"], ref["out"][inner], rtol=1e-12, atol=1e-12)
        for key in ("fc", "mu", "inv_sigma", "bias"):
            acc[key] = acc[key] + got[key]
        acc["h"].index_add_(0, gid, got["h"])
    for key, v in acc.items():
        torch.testing.assert_close(v, ref[key], rtol=1e-10, atol=1e-10, msg=key)


# ------------------------------------------------------------------------------------------------ parser / model
def test_parser_kernel_range_and_an_unchanged_namespace():
    from pipegcn_b200.helper.parser import create_parser
    a = create_parser(["--model", "monet", "--n-heads", "8"])
    assert a.model == "monet" and not hasattr(a, "monet_kernels")
    assert getattr(a, "monet_kernels", 3) == 3
    for k in (1, 5, 8):
        assert create_parser(["--model", "monet", "--monet-kernels", str(k)]).monet_kernels == k
    assert create_parser(["--monet_kernels", "2"]).monet_kernels == 2
    for bad in ("0", "9", "-1", "2.5", "x"):
        with pytest.raises(SystemExit):
            create_parser(["--model", "monet", "--monet-kernels", bad])
    base = vars(create_parser([]))
    with_model = vars(create_parser(["--model", "monet"]))
    assert with_model.pop("model") == "monet"
    base.pop("model")
    assert with_model == base


def _args(**kw):
    base = dict(model="monet", use_pp=False, n_hidden=16, enable_pipeline=False, feat_corr=False, grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(aggregator="pool"), ValueError, "--model monet has its own"),
    (dict(use_pp=True), NotImplementedError, "precompute is a neighbour mean"),
    (dict(sampling_rate=0.5), NotImplementedError, "defined on the full graph's degrees"),
    (dict(monet_kernels=9), ValueError, "expected 1 to 8"),
    (dict(monet_kernels=0), ValueError, "expected 1 to 8"),
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


def test_heads_are_ignored():
    from pipegcn_b200.train import check_model
    check_model(_args(n_heads=3))                   # 16 does not split into 3 heads: --n-heads is not read


def dgl_gmmconv_params(d_in, d_out, k):
    """The parameters of DGL's GMMConv(d_in, d_out, dim=2, n_kernels=k, aggregator_type='mean', residual=False,
    bias=True), restated: the constructor registers mu, inv_sigma, fc (nn.Linear without bias, drawing its default
    initialisation) and bias, then reset_parameters draws xavier_normal_(fc.weight, relu gain), normal_(mu, 0, 0.1),
    and sets inv_sigma = 1 and bias = 0."""
    from torch import nn
    mu = torch.empty(k, 2)
    inv_sigma = torch.empty(k, 2)
    fc = nn.Linear(d_in, k * d_out, bias=False)
    bias = torch.empty(d_out)
    nn.init.xavier_normal_(fc.weight, gain=nn.init.calculate_gain('relu'))
    nn.init.normal_(mu, 0, 0.1)
    nn.init.constant_(inv_sigma, 1)
    nn.init.zeros_(bias)
    return {"mu": mu, "inv_sigma": inv_sigma, "fc.weight": fc.weight.detach(), "bias": bias}


@pytest.mark.parametrize("n_linear,k", [(0, 3), (1, 3), (0, 1), (1, 8)])
def test_keys_shapes_and_draw_order(n_linear, k):
    from torch import nn
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.module.model import MoNet
    from pipegcn_b200.train import create_model
    argv = ["--model", "monet", "--n-hidden", "16", "--n-layers", "3", "--n-linear", str(n_linear)]
    if k != 3:
        argv += ["--monet-kernels", str(k)]
    torch.manual_seed(5)
    model = create_model([20, 16, 16, 5], create_parser(argv))
    assert isinstance(model, MoNet)
    sd = model.state_dict()
    sizes = [20, 16, 16, 5]
    torch.manual_seed(5)
    expect = {}
    for i, (d_in, d) in enumerate(zip(sizes[:-1], sizes[1:])):
        p = f"layers.{i}."
        if i < 3 - n_linear:
            expect.update({p + key: v for key, v in dgl_gmmconv_params(d_in, d, k).items()})
        else:
            lin = nn.Linear(d_in, d)
            expect.update({p + "weight": lin.weight, p + "bias": lin.bias})
        if i < 2:
            expect.update({f"norm.{i}.weight": torch.ones(d), f"norm.{i}.bias": torch.zeros(d)})
    assert set(sd) == set(expect)
    for key, v in expect.items():
        assert torch.equal(sd[key], v.detach()), key
    assert [key for key in sd if key.startswith("layers.0.")] == \
        ["layers.0.mu", "layers.0.inv_sigma", "layers.0.bias", "layers.0.fc.weight"]
    assert sd["layers.0.fc.weight"].shape == (k * 16, 20) and sd["layers.0.mu"].shape == (k, 2)
    if n_linear == 0:                            # the logits come from a MoNetLayer(d_in, n_class)
        assert sd["layers.2.fc.weight"].shape == (k * 5, 16) and sd["layers.2.bias"].shape == (5,)
