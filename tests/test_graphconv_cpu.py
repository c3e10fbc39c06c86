"""Graph convolution (`--model graphconv`) without a GPU: the parser, the refused configurations, DGL GraphConv's
parameters and seeded initialisation, the layer's forward and backward formulas for both associations in fp64, and
the symmetry of the partitions that lets a halo row's owner supply its degree."""
import argparse

import pytest
import torch


def test_parser_accepts_graphconv_and_keeps_gcn():
    from pipegcn_b200.helper.parser import create_parser
    assert create_parser(["--model", "graphconv"]).model == "graphconv"
    assert create_parser(["--model", "gcn"]).model == "gcn"
    base = vars(create_parser([]))
    with_model = vars(create_parser(["--model", "graphconv"]))
    assert with_model.pop("model") == "graphconv"
    base.pop("model")
    assert with_model == base


def test_gcn_stays_graphsage():
    from pipegcn_b200.module.model import GCN, GraphConv, GraphSAGE
    assert GCN is GraphSAGE and GraphConv is not GraphSAGE


def _args(**kw):
    base = dict(model="graphconv", use_pp=False, n_hidden=16, enable_pipeline=False, feat_corr=False, grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(aggregator="pool"), ValueError, "--model graphconv has none"),
    (dict(sampling_rate=0.5), NotImplementedError, "sampled out-degree"),
])
def test_refused_before_allocation(kw, exc, match):
    """RankEngine and init_processes refuse before touching the layout, the world or a device."""
    from pipegcn_b200 import train
    args = _args(**kw)
    with pytest.raises(exc, match=match):
        train.RankEngine(None, args, None)
    with pytest.raises(exc, match=match):
        train.init_processes(0, 2, args)


def _model(n_linear, seed=0, use_pp=False):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    argv = ["--model", "graphconv", "--n-hidden", "16", "--n-layers", "3", "--n-linear", str(n_linear)]
    args = create_parser(argv + (["--use-pp"] if use_pp else []))
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], args)


@pytest.mark.parametrize("n_linear", [0, 1])
@pytest.mark.parametrize("use_pp", [False, True])
def test_keys_and_shapes_are_graphconv(n_linear, use_pp):
    sd = _model(n_linear, use_pp=use_pp).state_dict()
    n_graph = 3 - n_linear
    for i, (d_in, d_out) in enumerate(zip([20, 16, 16], [16, 16, 5])):
        if i < n_graph:
            assert sd[f"layers.{i}.weight"].shape == (d_in, d_out)         # [in, out], not nn.Linear's [out, in]
            assert sd[f"layers.{i}.bias"].shape == (d_out,)
        else:
            assert sd[f"layers.{i}.weight"].shape == (d_out, d_in)         # the trailing nn.Linear
    assert {k for k in sd if k.startswith("norm.")} == {f"norm.{i}.{p}" for i in (0, 1) for p in ("weight", "bias")}


def test_initialisation_is_graphconv_reset_parameters():
    """xavier_uniform_(weight) then zeros_(bias), layer by layer in construction order, under the seed; then the
    trailing nn.Linear's own draws."""
    model = _model(1, seed=7)
    torch.manual_seed(7)
    expect = {}
    for i, (d_in, d_out) in enumerate([(20, 16), (16, 16)]):
        w = torch.empty(d_in, d_out)
        torch.nn.init.xavier_uniform_(w)
        expect[f"layers.{i}.weight"] = w
        expect[f"layers.{i}.bias"] = torch.zeros(d_out)
    tail = torch.nn.Linear(16, 5)
    expect["layers.2.weight"], expect["layers.2.bias"] = tail.weight.detach(), tail.bias.detach()
    sd = model.state_dict()
    for k, v in expect.items():
        assert torch.equal(sd[k], v), k


# ------------------------------------------------------------------------------------------------ formulas
def _graph(num_in=40, num_halo=15, seed=0):
    """Edges (rows = destinations < num_in, cols = sources < num_all) with self loops, a hub, and rows whose only
    edge is the self loop; c of every row from a made-up global degree >= its local in-degree."""
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    rows, cols = [], []
    for v in range(num_in):
        k = 0 if v % 7 == 3 else (30 if v == 0 else int(torch.randint(1, 6, (1,), generator=gen)))
        srcs = [v] + torch.randint(0, num_all, (k,), generator=gen).tolist()
        rows += [v] * len(srcs)
        cols += srcs
    deg = torch.randint(1, 9, (num_all,), generator=gen).double()
    return torch.tensor(rows), torch.tensor(cols), num_in, num_all, deg.rsqrt()


def _adj(rows, cols, num_in, num_all):
    a = torch.zeros(num_in, num_all, dtype=torch.float64)
    return a.index_put_((rows, cols), torch.ones(rows.numel(), dtype=torch.float64), accumulate=True)


def _drop_mask(shape, p, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=gen, dtype=torch.float64) >= p).double() / (1 - p)


@pytest.mark.parametrize("d_in,d_out", [(12, 20), (20, 6)])      # aggregate first, transform first
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_layer_formulas_match_autograd(d_in, d_out, p):
    """The association GraphConvLayerFn / GraphConvLayerNarrowFn compute, forward and backward, written out with the
    scaled aggregate as a gather (fp64), equals torch.autograd of the dense restatement c_v sum_u c_u (m * F)_u W + b,
    where m is the dropout mask of the key the backward store applies (drop_bwd)."""
    rows, cols, num_in, num_all, c = _graph()
    gen = torch.Generator().manual_seed(1)
    f = torch.randn(num_all, d_in, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(d_in, d_out, generator=gen, dtype=torch.float64, requires_grad=True)
    b = torch.randn(d_out, generator=gen, dtype=torch.float64, requires_grad=True)
    g = torch.randn(num_in, d_out, generator=gen, dtype=torch.float64)
    m = _drop_mask((num_all, d_in), p, 2) if p else torch.ones(num_all, d_in, dtype=torch.float64)
    a_hat = c[:num_in, None] * _adj(rows, cols, num_in, num_all) * c[None, :]
    out = a_hat @ (m * f) @ w + b
    out.backward(g)

    def scaled(dst_rows, src_cols, x, src, dst, n):      # out[r] = dst[r] sum_{e in row r} src[idx] x[idx]
        return dst[:, None] * torch.zeros(n, x.shape[1], dtype=x.dtype).index_add(0, dst_rows, src[src_cols, None] * x[src_cols])

    h = m * f.detach()
    if d_in <= d_out:
        ah = scaled(rows, cols, h, c, c[:num_in], num_in)
        o = ah @ w.detach() + b.detach()
        g_ah = g @ w.detach().t()
        g_f = m * scaled(cols, rows, g_ah, c, c, num_all)      # CSC: rows of sources, entries are destinations
        gw = (g.t() @ ah).t()
    else:
        z = h @ w.detach()
        o = scaled(rows, cols, z, c, c[:num_in], num_in) + b.detach()
        dz = scaled(cols, rows, g, c, c, num_all)
        g_f = m * (dz @ w.detach().t())
        gw = (dz.t() @ h).t()
    torch.testing.assert_close(o, out.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(g_f, f.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(gw, w.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(g.sum(0), b.grad, rtol=1e-12, atol=1e-12)
    lonely = [v for v in range(num_in) if (rows == v).sum() == 1]
    assert lonely, "the graph has nodes with only a self loop"


def test_sym_norm_is_correctly_rounded():
    from pipegcn_b200.ops import sym_norm
    deg = torch.tensor([0, 1, 2, 3, 4, 7, 1000, 123457])
    c = sym_norm(deg)
    ref = (1.0 / torch.clamp(deg, min=1).double().sqrt())
    assert c.dtype == torch.float32 and torch.equal(c[:2], torch.ones(2))
    assert torch.all((c.double() - ref).abs() <= ref * 2 ** -23)


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_csc_row_lengths_sum_to_the_degree(n_parts, metis):
    """Summed over the partitions, a node's CSC row lengths (the edges it sends into each partition) equal its in-degree:
    the graphs are symmetric with one self loop per node, so a source's out-degree -- DGL's source-side norm -- is its
    in-degree, and the owner's in-degree is the degree every partition must use for its halo copy."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    else:
        part = random_partition(g.n_nodes, n_parts)
    lays = build_layouts(g, part, n_parts)
    total = torch.zeros(g.n_nodes, dtype=torch.int64)
    for lay in lays:
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long()
        total.index_add_(0, gid, (lay.t_indptr[1:] - lay.t_indptr[:-1]).long())
    assert torch.equal(total, g.in_degrees().long())
    assert torch.equal(torch.bincount(g.src.long(), minlength=g.n_nodes), g.in_degrees().long())
