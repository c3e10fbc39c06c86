"""Principal neighbourhood aggregation (`--model pna`) without a GPU: the parser, the refused configurations, the
parameters and their draw order, the factorised forward and backward the kernels implement against autograd through
DGL's unfactorised definition in fp64, delta from merged degree histograms, and the scalers' rounding.

`graph_case` and `factorised_forward` / `factorised_backward` are the fp64 restatement the GPU tests compare against."""
import argparse
import math

import numpy as np
import pytest
import torch

# ------------------------------------------------------------------------------------------------ restatement
def graph_case(seed=0, num_in=30, num_halo=12, d=6):
    """(h [num_all, d] fp64, rows, cols (CSR order: edge e is cols[e] -> rows[e]), num_in) of a partition-shaped graph
    with a row without in-edges (0), self-loop-only rows (1, 2), a row whose sources are all equal (5: rows 5, 31,
    32 hold the same features) and a row whose every column has a tie for its maximum or minimum (8: h[8] = -h[5])."""
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    h = torch.randn(num_all, d, generator=gen, dtype=torch.float64)
    h[31] = h[32] = h[5]
    h[8] = -h[5]
    rows, cols = [], []
    for v in range(num_in):
        if v == 0:
            src = []
        elif v in (1, 2):
            src = [v]
        elif v == 5:
            src = [5, 31, 32]
        elif v == 8:
            src = [8, 31, 32]
        else:
            k = int(torch.randint(1, 7, (1,), generator=gen))
            src = [v] + torch.randperm(num_all, generator=gen)[:k].tolist()
            src = list(dict.fromkeys(src))
        rows += [v] * len(src)
        cols += src
    return h, torch.tensor(rows), torch.tensor(cols), num_in


def csr_of(rows, cols, n_rows):
    """(indptr, indices) of the edges in the order given (CSR order within a row)."""
    counts = torch.bincount(rows, minlength=n_rows)
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(counts, 0)
    order = torch.argsort(rows, stable=True)
    return indptr, cols[order]


def scalers64(deg, delta):
    lg = torch.log1p(deg.double())
    a = lg / delta
    t = torch.where(deg > 0, delta / torch.where(deg > 0, lg, torch.ones_like(lg)), torch.zeros_like(lg))
    return a, t


def extremes(zs, srcs):
    """(max, argmax, min, argmin) over the rows `srcs` of zs, per column: the first source in order wins a tie, the
    first NaN source is taken and kept."""
    d = zs.shape[1]
    mx, ax = torch.zeros(d, dtype=zs.dtype), torch.full((d,), -1)
    mn, an = torch.zeros(d, dtype=zs.dtype), torch.full((d,), -1)
    for u in srcs:
        x = zs[u]
        for c in range(d):
            xc = x[c]
            if ax[c] < 0 or xc > mx[c] or (xc != xc and mx[c] == mx[c]):
                mx[c], ax[c] = xc, u
            if an[c] < 0 or xc < mn[c] or (xc != xc and mn[c] == mn[c]):
                mn[c], an[c] = xc, u
    return mx, ax, mn, an


def factorised_forward(h, indptr, indices, num_in, delta, wm, bm, wu, bu, store=None):
    """The layer as the kernels compute it, in h's dtype.  Returns out and a dict of the intermediates.  `store`:
    rounds zs and agg where the engine stores them (bf16), so that the extremes pick the sources the kernels see."""
    store = store or (lambda t: t)
    d = h.shape[1]
    zs = store(h @ wm[:, :d].T)
    zd = h[:num_in] @ wm[:, d:].T + bm
    deg = indptr[1:] - indptr[:-1]
    mu = torch.zeros(num_in, d, dtype=h.dtype)
    var = torch.zeros_like(mu)
    agg = torch.zeros(num_in, 4 * d, dtype=h.dtype)
    amax = torch.full((num_in, d), -1)
    amin = torch.full((num_in, d), -1)
    for v in range(num_in):
        srcs = indices[indptr[v]:indptr[v + 1]].tolist()
        if not srcs:
            continue
        m, m2 = torch.zeros(d, dtype=h.dtype), torch.zeros(d, dtype=h.dtype)
        for k, u in enumerate(srcs, 1):                 # Welford, as the kernel: all-equal sources give var = 0
            delta_ = zs[u] - m
            m = m + delta_ / k
            m2 = m2 + delta_ * (zs[u] - m)
        mu[v], var[v] = m, m2 / len(srcs)
        mx, amax[v], mn, amin[v] = extremes(zs, srcs)
        sig = torch.sqrt(torch.clamp(var[v], min=0) + 1e-30)
        agg[v] = torch.cat([mu[v] + zd[v], mx + zd[v], mn + zd[v], sig])
    agg = store(agg)
    a, t = scalers64(deg, delta)
    a, t = a.to(h.dtype), t.to(h.dtype)
    wx, w1, w2, w3 = wu[:, :d], wu[:, d:5 * d], wu[:, 5 * d:9 * d], wu[:, 9 * d:]
    out = h[:num_in] @ wx.T + agg @ w1.T + bu + a[:, None] * (agg @ w2.T) + t[:, None] * (agg @ w3.T)
    return out, dict(zs=zs, zd=zd, mu=mu, var=var, agg=agg, amax=amax, amin=amin, a=a, t=t, deg=deg)


def factorised_backward(g, h, indptr, indices, num_in, wm, wu, st):
    """The hand-written backward of the layer (the kernels' formulas) from the forward's intermediates `st`."""
    d, d_out = h.shape[1], wu.shape[0]
    num_all = h.shape[0]
    a, t, deg = st["a"], st["t"], st["deg"]
    g3 = torch.cat([g, a[:, None] * g, t[:, None] * g], 1)
    w123 = torch.cat([wu[:, d:5 * d], wu[:, 5 * d:9 * d], wu[:, 9 * d:]], 0)          # [3 d_out, 4d]
    gagg = g3 @ w123
    gm, gx, gn, gs = gagg[:, :d], gagg[:, d:2 * d], gagg[:, 2 * d:3 * d], gagg[:, 3 * d:]
    has = (deg > 0)[:, None]
    df = deg.clamp(min=1).to(h.dtype)[:, None]
    sig = torch.sqrt(torch.clamp(st["var"], min=0) + 1e-30)
    gzd = torch.where(has, gm + gx + gn, torch.zeros_like(gm))
    beta = torch.where(has & (st["var"] > 0), gs / (df * sig), torch.zeros_like(gs))
    alpha = torch.where(has, gm / df - beta * st["mu"], torch.zeros_like(gm))
    gmx, gmn = torch.where(has, gx, 0 * gx), torch.where(has, gn, 0 * gn)
    s1 = torch.zeros(num_all, d, dtype=h.dtype)
    s2 = torch.zeros(num_all, d, dtype=h.dtype)
    for v in range(num_in):
        for u in indices[indptr[v]:indptr[v + 1]].tolist():
            s1[u] += alpha[v]
            s2[u] += beta[v]
            s1[u] += torch.where(st["amax"][v] == u, gmx[v], torch.zeros_like(gmx[v]))
            s1[u] += torch.where(st["amin"][v] == u, gmn[v], torch.zeros_like(gmn[v]))
    gzs = s1 + st["zs"] * s2
    ws, wd, wx = wm[:, :d], wm[:, d:], wu[:, :d]
    gh = gzs @ ws
    gh[:num_in] += g @ wx + gzd @ wd
    gwu = torch.cat([g.T @ h[:num_in], (g3.T @ st["agg"]).view(3, d_out, 4 * d).permute(1, 0, 2).reshape(d_out, 12 * d)],
                    1)
    gwm = torch.cat([gzs.T @ h, gzd.T @ h[:num_in]], 1)
    return dict(h=gh, wm=gwm, bm=gzd.sum(0), wu=gwu, bu=g.sum(0), gzs=gzs, gzd=gzd, alpha=alpha, beta=beta,
                gmx=gmx, gmn=gmn, gagg=gagg, g3=g3)


def dgl_forward(h, rows, cols, num_in, delta, wm, bm, wu, bu):
    """DGL's PNAConvTower, unfactorised: per-edge messages M(cat(h_u, h_v)), the mailbox reductions (std as
    sqrt(relu(E[m^2] - E[m]^2) + 1e-30)), the scalers and U(cat(h_v, h_neigh)); a node without messages gets
    h_neigh = 0."""
    d = h.shape[1]
    m = torch.cat([h[cols], h[rows]], 1) @ wm.T + bm
    deg = torch.bincount(rows, minlength=num_in)
    a, t = scalers64(deg, delta)
    neigh = []
    for v in range(num_in):
        box = m[rows == v]
        if box.shape[0] == 0:
            neigh.append(torch.zeros(12 * d, dtype=h.dtype))
            continue
        mean = box.mean(0)
        var = torch.relu((box * box).mean(0) - mean * mean)
        agg = torch.cat([mean, box.max(0).values, box.min(0).values, torch.sqrt(var + 1e-30)])
        neigh.append(torch.cat([agg, a[v] * agg, t[v] * agg]))
    return torch.cat([h[:num_in], torch.stack(neigh)], 1) @ wu.T + bu


def _params(d, d_out, seed):
    gen = torch.Generator().manual_seed(seed)
    wm = torch.randn(d, 2 * d, generator=gen, dtype=torch.float64) / math.sqrt(2 * d)
    bm = torch.randn(d, generator=gen, dtype=torch.float64) * 0.1
    wu = torch.randn(d_out, 13 * d, generator=gen, dtype=torch.float64) / math.sqrt(13 * d)
    bu = torch.randn(d_out, generator=gen, dtype=torch.float64) * 0.1
    return wm, bm, wu, bu


# ------------------------------------------------------------------------------------------------ formulas
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_factorised_layer_matches_dgl_autograd(seed):
    h, rows, cols, num_in = graph_case(seed)
    d, d_out, delta = h.shape[1], 5, 1.37
    wm, bm, wu, bu = _params(d, d_out, seed + 10)
    indptr, indices = csr_of(rows, cols, num_in)
    out, st = factorised_forward(h, indptr, indices, num_in, delta, wm, bm, wu, bu)
    assert torch.equal(st["var"][5], torch.zeros(d)) and torch.equal(st["var"][1], torch.zeros(d))
    assert torch.all(st["amax"][0] == -1) and torch.all(st["amin"][0] == -1)
    # row 8: every column's extreme among the two equal sources 31, 32 goes to the first, 31
    assert torch.all((st["amax"][8] == 31) | (st["amin"][8] == 31))
    assert not torch.any(st["amax"][8] == 32) and not torch.any(st["amin"][8] == 32)

    leaves = [x.clone().requires_grad_(True) for x in (h, wm, bm, wu, bu)]
    ref = dgl_forward(leaves[0], rows, cols, num_in, delta, *leaves[1:])
    # DGL's E[m^2] - E[m]^2 cancels against the message's zd part: its std carries errors of about
    # sqrt(2^-52 E[m^2]), which the factorised Welford form over zs does not have
    assert torch.allclose(out, ref, rtol=1e-7, atol=1e-7)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 20), dtype=torch.float64)
    ref.backward(g)
    got = factorised_backward(g, h, indptr, indices, num_in, wm, wu, st)
    # all-equal rows: DGL's E[m^2] - E[m]^2 may round to a tiny positive variance whose std gradient is O(1e-8 |g|);
    # the factorised form has var = 0 exactly there
    for name, leaf in zip(("h", "wm", "bm", "wu", "bu"), leaves):
        assert torch.allclose(got[name], leaf.grad, rtol=1e-6, atol=1e-6), name


# ------------------------------------------------------------------------------------------------ delta / scalers
def _whole_delta(deg):
    lg = torch.log1p(deg.double())
    return float(lg.mean())


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_delta_is_the_same_bits_for_every_partition(n_parts, metis):
    from pipegcn_b200.ops import pna_degree_histogram, pna_delta
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny", seed_graph=0)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    else:
        part = random_partition(g.n_nodes, n_parts)
    lays = build_layouts(g, part, n_parts)
    whole = torch.bincount(g.in_degrees().long()).tolist()
    ref = pna_delta([whole])
    got = pna_delta([pna_degree_histogram(lay.indptr) for lay in lays])
    assert got == ref                                       # bit for bit
    assert math.isclose(got, _whole_delta(g.in_degrees()), rel_tol=1e-14)
    # every rank merges the same list: any order of the ranks gives the same bits
    assert pna_delta([pna_degree_histogram(lay.indptr) for lay in reversed(lays)]) == ref


@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_delta_of_distgraph_layouts_equals_whole_graph(n_parts):
    from pipegcn_b200.distgraph import build_rank_layout
    from pipegcn_b200.ops import pna_degree_histogram, pna_delta
    spec = dict(n_nodes=3000, n_edges=40_000, n_feat=12, n_class=5, train_frac=0.3)
    lays = [build_rank_layout(spec, r, n_parts, "cpu", pair_chunk=7000)[0] for r in range(n_parts)]
    deg = torch.zeros(spec["n_nodes"], dtype=torch.int64)
    for lay in lays:
        deg[lay.inner_gid.long()] = (lay.indptr[1:] - lay.indptr[:-1]).long()
    assert pna_delta([pna_degree_histogram(lay.indptr) for lay in lays]) == pna_delta([torch.bincount(deg).tolist()])
    assert math.isclose(pna_delta([torch.bincount(deg).tolist()]), _whole_delta(deg), rel_tol=1e-14)


def test_scalers_are_correctly_rounded():
    from pipegcn_b200.ops import pna_scalers_host
    deg = torch.tensor([0, 1, 2, 3, 7, 100, 1000, 123457])
    delta = 2.718281828459045 / 1.7
    a, t = pna_scalers_host(deg, delta)
    lg = torch.log1p(deg.double())
    assert a.dtype == t.dtype == torch.float32
    assert torch.equal(a, (lg / delta).float())
    assert torch.equal(t[1:], (delta / lg[1:]).float()) and t[0] == 0 and a[0] == 0
    for k in range(1, deg.numel()):                       # fp64 within half an fp32 ulp: correctly rounded
        exact = math.log1p(int(deg[k])) / delta
        assert abs(float(a[k]) - exact) <= float(np.spacing(np.float32(a[k]))) / 2 * (1 + 1e-9)


# ------------------------------------------------------------------------------------------------ parser / model
def test_parser_accepts_pna_and_changes_nothing_else():
    from pipegcn_b200.helper.parser import create_parser
    assert create_parser(["--model", "pna"]).model == "pna"
    base = vars(create_parser([]))
    with_model = vars(create_parser(["--model", "pna"]))
    assert with_model.pop("model") == "pna"
    base.pop("model")
    assert with_model == base


def _args(**kw):
    base = dict(model="pna", use_pp=False, n_hidden=16, enable_pipeline=False, feat_corr=False, grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(aggregator="pool"), ValueError, "--model pna has its own"),
    (dict(use_pp=True), NotImplementedError, "precompute is a neighbour mean"),
    (dict(sampling_rate=0.5), NotImplementedError, "sampling changes the degrees"),
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


def _model(n_linear, seed=0):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    args = create_parser(["--model", "pna", "--n-hidden", "16", "--n-layers", "3", "--n-linear", str(n_linear)])
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], args)


@pytest.mark.parametrize("n_linear", [0, 1])
def test_keys_shapes_and_draw_order(n_linear):
    from torch import nn
    model = _model(n_linear, seed=3)
    sd = model.state_dict()
    sizes = [20, 16, 16, 5]
    torch.manual_seed(3)
    expect = {}
    for i, (d_in, d_out) in enumerate(zip(sizes[:-1], sizes[1:])):
        if i < 3 - n_linear:
            m, u = nn.Linear(2 * d_in, d_in), nn.Linear(13 * d_in, d_out)        # M drawn before U
            expect.update({f"layers.{i}.M.weight": m.weight, f"layers.{i}.M.bias": m.bias,
                           f"layers.{i}.U.weight": u.weight, f"layers.{i}.U.bias": u.bias})
            assert sd[f"layers.{i}.M.weight"].shape == (d_in, 2 * d_in)
            assert sd[f"layers.{i}.U.weight"].shape == (d_out, 13 * d_in)
        else:
            lin = nn.Linear(d_in, d_out)
            expect.update({f"layers.{i}.weight": lin.weight, f"layers.{i}.bias": lin.bias})
        if i < 2:
            expect.update({f"norm.{i}.weight": torch.ones(d_out), f"norm.{i}.bias": torch.zeros(d_out)})
    assert set(sd) == set(expect) | {"pna_delta"}
    for k, v in expect.items():
        assert torch.equal(sd[k], v.detach()), k
    assert sd["pna_delta"].dtype == torch.float64 and torch.isnan(sd["pna_delta"])


def test_delta_travels_with_the_state_dict():
    model = _model(0)
    model.set_delta(1.25)
    assert all(model.layers[i].delta == 1.25 for i in range(model.n_graph_layers))
    other = _model(0, seed=1)
    assert other.delta is None
    other.load_state_dict(model.state_dict())
    assert other.delta == 1.25 and all(other.layers[i].delta == 1.25 for i in range(other.n_graph_layers))
