"""GCNII (`--model gcnii`) without a GPU: the parser, the refused configurations, GCN2Conv's parameters, initialisation
and beta schedule, the layer stack's forward and its hand-written backward (teleport sum over the layers, dropout
keys) against torch autograd in fp64, and a restatement of partitioned training (fc_in over the halo rows, per-rank
weight gradients summed) against whole-graph training."""
import argparse
import math

import pytest
import torch


# ------------------------------------------------------------------------------------------------ parser
def test_parser_flags_and_unchanged_namespace():
    from pipegcn_b200.helper.parser import create_parser
    a = create_parser(["--model", "gcnii", "--gcnii-alpha", "0.2", "--gcnii_lambda", "1.5"])
    assert a.model == "gcnii" and a.gcnii_alpha == 0.2 and a.gcnii_lambda == 1.5
    assert create_parser(["--gcnii-alpha", "0"]).gcnii_alpha == 0.0
    assert create_parser(["--gcnii-alpha", "1"]).gcnii_alpha == 1.0
    base = vars(create_parser([]))
    assert "gcnii_alpha" not in base and "gcnii_lambda" not in base
    with_model = vars(create_parser(["--model", "gcnii"]))
    assert with_model.pop("model") == "gcnii"
    base.pop("model")
    assert with_model == base


@pytest.mark.parametrize("flag,value", [("--gcnii-alpha", "-0.1"), ("--gcnii-alpha", "1.5"), ("--gcnii-alpha", "nan"),
                                        ("--gcnii-alpha", "x"), ("--gcnii-lambda", "0"), ("--gcnii-lambda", "-1"),
                                        ("--gcnii-lambda", "nan"), ("--gcnii-lambda", "inf")])
def test_parser_refuses_bad_values(flag, value):
    from pipegcn_b200.helper.parser import create_parser
    with pytest.raises(SystemExit):
        create_parser(["--model", "gcnii", flag, value])


# ------------------------------------------------------------------------------------------------ refusals
def _args(**kw):
    base = dict(model="gcnii", use_pp=False, n_hidden=16, n_layers=3, n_linear=1, enable_pipeline=False,
                feat_corr=False, grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(n_linear=0), ValueError, "--n-linear >= 1"),
    (dict(n_layers=2, n_linear=2), ValueError, "at least one convolution"),
    (dict(use_pp=True), NotImplementedError, "fc_in"),
    (dict(aggregator="pool"), ValueError, "--model gcnii has none"),
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


# ------------------------------------------------------------------------------------------------ parameters
def _model(n_layers=4, n_linear=1, seed=0, extra=()):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.partition import get_layer_size
    from pipegcn_b200.train import create_model
    args = create_parser(["--model", "gcnii", "--n-hidden", "16", "--n-layers", str(n_layers), "--n-linear",
                          str(n_linear)] + list(extra))
    torch.manual_seed(seed)
    return create_model(get_layer_size(20, 16, 5, n_layers), args)


@pytest.mark.parametrize("n_layers,n_linear", [(2, 1), (4, 1), (5, 2)])
def test_keys_and_shapes(n_layers, n_linear):
    sd = _model(n_layers, n_linear).state_dict()
    n_graph = n_layers - n_linear
    expect = {"layers.0.fc_in.weight": (16, 20), "layers.0.fc_in.bias": (16,)}
    for i in range(n_graph):
        expect[f"layers.{i}.weight1"] = (16, 16)
        expect[f"layers.{i}.bias"] = (16,)
    for i in range(n_graph, n_layers):
        expect[f"layers.{i}.weight"] = (5 if i == n_layers - 1 else 16, 16)
        expect[f"layers.{i}.bias"] = (5 if i == n_layers - 1 else 16,)
    for i in range(n_layers - 1):
        expect[f"norm.{i}.weight"] = expect[f"norm.{i}.bias"] = (16,)
    assert {k: tuple(v.shape) for k, v in sd.items()} == expect


def test_initialisation_and_draw_order():
    """fc_in (nn.Linear's default) first, then every convolution's weight1 ~ U(-1/sqrt(d), 1/sqrt(d)) with bias 0, in
    layer order, then the trailing linear."""
    model = _model(4, 1, seed=7)
    torch.manual_seed(7)
    fc = torch.nn.Linear(20, 16)
    expect = {"layers.0.fc_in.weight": fc.weight.detach(), "layers.0.fc_in.bias": fc.bias.detach()}
    for i in range(3):
        w = torch.empty(16, 16)
        torch.nn.init.uniform_(w, -0.25, 0.25)
        expect[f"layers.{i}.weight1"], expect[f"layers.{i}.bias"] = w, torch.zeros(16)
    tail = torch.nn.Linear(16, 5)
    expect["layers.3.weight"], expect["layers.3.bias"] = tail.weight.detach(), tail.bias.detach()
    sd = model.state_dict()
    for k, v in expect.items():
        assert torch.equal(sd[k], v), k


def test_beta_schedule_is_one_based():
    model = _model(6, 1, extra=["--gcnii-lambda", "0.7", "--gcnii-alpha", "0.3"])
    for i in range(5):
        layer = model.layers[i]
        assert layer.beta == math.log(0.7 / (i + 1) + 1) and layer.alpha == 0.3
    assert model.layers[0].beta == math.log(1.7)


# ------------------------------------------------------------------------------------------------ formulas (fp64)
def _graph(num_in=40, num_halo=15, seed=0):
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


def _scaled(dst_rows, src_cols, x, src, dst, n):
    """out[r] = dst[r] sum_{e in row r} src[idx] x[idx]: the scaled aggregate as a gather."""
    return dst[:, None] * torch.zeros(n, x.shape[1], dtype=x.dtype).index_add(0, dst_rows, src[src_cols, None] * x[src_cols])


def _mask(shape, p, seed):
    if p == 0:
        return torch.ones(shape, dtype=torch.float64)
    gen = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=gen, dtype=torch.float64) >= p).double() / (1 - p)


@pytest.mark.parametrize("p", [0.0, 0.4])
@pytest.mark.parametrize("n_conv", [1, 4])
def test_layer_stack_backward_matches_autograd(p, n_conv):
    """The forward of GCNIIFirstFn / GCNIIConvFn and their backward as written in ops.py -- dS = g W_eff^T, the fp32
    teleport sum alpha dS over layers L-1 .. 0, the input gradient through the transposed scaled aggregate with the
    dropout mask of its key, dz = ReLU'(z) (g_hd + teleport), dW1 = beta S^T g, dW_in = dz^T x -- equal torch.autograd
    of DGL GCN2Conv's formula, with ReLU and dropout between the layers (fp64)."""
    rows, cols, num_in, num_all, c = _graph()
    alpha, lam, F, d = 0.2, 0.6, 12, 10
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(num_all, F, generator=gen, dtype=torch.float64)
    w_in = torch.randn(d, F, generator=gen, dtype=torch.float64, requires_grad=True)
    b_in = torch.randn(d, generator=gen, dtype=torch.float64, requires_grad=True)
    w1 = [(0.3 * torch.randn(d, d, generator=gen, dtype=torch.float64)).requires_grad_() for _ in range(n_conv)]
    b1 = [torch.randn(d, generator=gen, dtype=torch.float64, requires_grad=True) for _ in range(n_conv)]
    g_out = torch.randn(num_in, d, generator=gen, dtype=torch.float64)
    betas = [math.log(lam / (i + 1) + 1) for i in range(n_conv)]
    m_h0 = _mask((num_all, d), p, 10)
    # later layers' inputs: [inner | halo] rows; the halo rows are fixed data here (the exchange is not under test)
    halo = [torch.randn(num_all - num_in, d, generator=gen, dtype=torch.float64) for _ in range(n_conv)]
    m = [_mask((num_all, d), p, 20 + i) for i in range(n_conv)]
    a_hat = torch.zeros(num_in, num_all, dtype=torch.float64).index_put_((rows, cols), torch.ones(rows.numel(), dtype=torch.float64),
                                                                         accumulate=True)
    a_hat = c[:num_in, None] * a_hat * c[None, :]
    eye = torch.eye(d, dtype=torch.float64)

    # GCN2Conv, literally: h = ((1-a) A_hat h + a h0) ((1-b) I + b W1) + bias
    h0 = torch.relu(x @ w_in.t() + b_in)
    h = m_h0 * h0
    for i in range(n_conv):
        if i > 0:
            h = m[i] * torch.cat([torch.relu(h), halo[i]])
        s = (1 - alpha) * (a_hat @ h) + alpha * h0[:num_in]
        h = (1 - betas[i]) * s + betas[i] * (s @ w1[i]) + b1[i]
    h.backward(g_out)

    # ops.py, step by step
    cs = (1 - alpha) * c[:num_in]
    z = x @ w_in.detach().t() + b_in.detach()
    h0_ = torch.relu(z)
    ins, ss, pres = [m_h0 * h0_], [], []
    for i in range(n_conv):
        if i > 0:
            ins.append(m[i] * torch.cat([torch.relu(pres[-1]), halo[i]]))
        w_eff = (1 - betas[i]) * eye + betas[i] * w1[i].detach()
        s = _scaled(rows, cols, ins[i], c, cs, num_in) + alpha * h0_[:num_in]
        ss.append(s)
        pres.append(s @ w_eff + b1[i].detach())
    torch.testing.assert_close(pres[-1], h.detach(), rtol=1e-12, atol=1e-12)
    g, acc = g_out, None
    for i in reversed(range(n_conv)):
        w_eff = (1 - betas[i]) * eye + betas[i] * w1[i].detach()
        ds = g @ w_eff.t()
        acc = alpha * ds if acc is None else acc + alpha * ds          # L-1 down to 0
        torch.testing.assert_close(betas[i] * (g.t() @ ss[i]).t(), w1[i].grad, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(g.sum(0), b1[i].grad, rtol=1e-12, atol=1e-12)
        g_in = (m[i] if i > 0 else m_h0) * _scaled(cols, rows, ds, cs, c, num_all)   # dropout backward in the store
        if i > 0:
            g = g_in[:num_in] * (pres[i - 1] > 0).double()
    teleport = torch.zeros(num_all, d, dtype=torch.float64)
    teleport[:num_in] = acc
    dz = (z > 0).double() * (g_in + teleport)
    torch.testing.assert_close(dz.t() @ x, w_in.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dz.sum(0), b_in.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ partitioned
def _gcnii_full(x, src, dst, c, params, alpha, betas, n):
    """Whole-graph GCNII, fp64: fc_in, ReLU, convolutions with ReLU between, logits linear."""
    w_in, b_in, w1, b1, w_out, b_out = params
    a = torch.zeros(n, n, dtype=torch.float64).index_put_((dst, src), torch.ones(src.numel(), dtype=torch.float64),
                                                          accumulate=True)
    a_hat = c[:, None] * a * c[None, :]
    h0 = torch.relu(x @ w_in.t() + b_in)
    h = h0
    for i in range(len(w1)):
        if i > 0:
            h = torch.relu(h)
        s = (1 - alpha) * (a_hat @ h) + alpha * h0
        h = s @ ((1 - betas[i]) * torch.eye(h.shape[1], dtype=torch.float64) + betas[i] * w1[i]) + b1[i]
    return torch.relu(h) @ w_out.t() + b_out


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_partitioned_restatement_equals_full_graph(n_parts, metis):
    """Synchronous partitioned training restated in torch: every rank runs fc_in over its inner AND halo rows of x
    (layer 0 exchanges x, not h0), later layers read their halo rows from the owners' outputs, every rank holds its
    own copy of the parameters; the per-rank gradients summed (the all-reduce) equal whole-graph training's, fc_in's
    included."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    part = random_partition(g.n_nodes, n_parts)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    lays = build_layouts(g, part, n_parts)
    n, F, d, C, n_conv, alpha, lam = g.n_nodes, g.n_feat, 8, 3, 3, 0.15, 0.5
    betas = [math.log(lam / (i + 1) + 1) for i in range(n_conv)]
    gen = torch.Generator().manual_seed(5)
    x = g.feat.double()
    c = torch.clamp(g.in_degrees().double(), min=1).rsqrt()
    base = [torch.randn(d, F, generator=gen, dtype=torch.float64) * 0.3, torch.randn(d, generator=gen, dtype=torch.float64),
            [torch.randn(d, d, generator=gen, dtype=torch.float64) * 0.3 for _ in range(n_conv)],
            [torch.randn(d, generator=gen, dtype=torch.float64) for _ in range(n_conv)],
            torch.randn(C, d, generator=gen, dtype=torch.float64), torch.randn(C, generator=gen, dtype=torch.float64)]
    probe = torch.randn(n, C, generator=gen, dtype=torch.float64)

    def clone():
        p = [t.clone().requires_grad_() for t in base[:2]] + [[t.clone().requires_grad_() for t in base[2]],
                                                              [t.clone().requires_grad_() for t in base[3]]] \
            + [t.clone().requires_grad_() for t in base[4:]]
        return p

    def flat(p):
        return [p[0], p[1]] + p[2] + p[3] + [p[4], p[5]]

    full = clone()
    (_gcnii_full(x, g.src, g.dst, c, full, alpha, betas, n) * probe).sum().backward()

    ranks = [clone() for _ in lays]
    gids = [torch.cat([lay.inner_gid, lay.halo_gid]).long() for lay in lays]
    h0s, hs = [], []
    for lay, p, gid in zip(lays, ranks, gids):                 # layer 0: fc_in over [inner | halo] rows of x
        h0 = torch.relu(x[gid] @ p[0].t() + p[1])
        h0s.append(h0)
        hs.append(h0)
    outs = None
    for i in range(n_conv):
        if i > 0:                                              # exchange: halo rows from their owners' outputs
            owner_rows = torch.zeros(n, d, dtype=torch.float64)
            for lay, o in zip(lays, outs):
                owner_rows = owner_rows.index_put((lay.inner_gid.long(),), torch.relu(o))
            hs = [owner_rows[gid] for gid in gids]
        outs = []
        for lay, p, gid, h, h0 in zip(lays, ranks, gids, hs, h0s):
            rows = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
            cl = c[gid]
            s = (1 - alpha) * _scaled(rows, lay.indices.long(), h, cl, cl[:lay.num_in], lay.num_in) + alpha * h0[:lay.num_in]
            outs.append(s @ ((1 - betas[i]) * torch.eye(d, dtype=torch.float64) + betas[i] * p[2][i]) + p[3][i])
    loss = 0
    for lay, p, o in zip(lays, ranks, outs):
        loss = loss + ((torch.relu(o) @ p[4].t() + p[5]) * probe[lay.inner_gid.long()]).sum()
    loss.backward()
    for k, ref in enumerate(flat(full)):
        got = sum(flat(p)[k].grad for p in ranks)
        torch.testing.assert_close(got, ref.grad, rtol=1e-10, atol=1e-10)
    halo_rows = sum(int(lay.halo_gid.numel()) for lay in lays)
    assert halo_rows > 0
