"""Dynamic graph attention (`--model gatv2`) without a GPU: the parser, the refused configurations, the parameters
(DGL GATv2Conv's keys and shapes, share_weights=False) and their seeded initialisation, and the backward formulas the
kernels implement, written out in fp64 and checked against torch.autograd of the forward restatement."""
import argparse

import pytest
import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------ restatement
def ref_gatv2(zs, zd, attn, rows, cols, num_in):
    """fp64 GATv2Conv aggregate over the edges cols -> rows: zs [num_all, H, D], zd [num_in, H, D], attn [1, H, D] ->
    out [num_in, H*D] (no output bias) and the softmax statistics (m, s) [num_in, H]."""
    heads = zs.shape[1]
    t = zs[cols] + zd[rows]                                        # [E, H, D]
    e = (F.leaky_relu(t, 0.2) * attn.view(1, heads, -1)).sum(-1)   # [E, H]
    m = torch.full((num_in, heads), float("-inf"), dtype=zs.dtype, device=zs.device)
    m = m.scatter_reduce(0, rows[:, None].expand(-1, heads), e, "amax")
    p = torch.exp(e - m[rows])
    s = torch.zeros(num_in, heads, dtype=zs.dtype, device=zs.device).index_add(0, rows, p)
    a = p / s[rows]
    out = torch.zeros(num_in, heads, zs.shape[2], dtype=zs.dtype, device=zs.device)
    out = out.index_add(0, rows, a[..., None] * zs[cols])
    return out.reshape(num_in, -1), m.detach(), s.detach()


def ref_gatv2_backward(zs, zd, attn, rows, cols, num_in, g):
    """The backward of ref_gatv2 as the kernels compute it, g = dL/d out [num_in, H*D]:
        dot_uv = <g_v, zs_u>,  D_v = sum_u a_uv dot_uv,  de_uv = a_uv (dot_uv - D_v),  σ'(t) = 1 if t > 0 else 0.2
        d zs_u = sum_v a_uv g_v + de_uv attn ⊙ σ'(t_uv),  d zd_v = sum_u de_uv attn ⊙ σ'(t_uv),
        d attn = sum over edges de_uv LeakyReLU(t_uv)
    Returns (d zs, d zd, d attn, D)."""
    heads, d = zs.shape[1], zs.shape[2]
    gv = g.view(num_in, heads, d)
    t = zs[cols] + zd[rows]
    e = (F.leaky_relu(t, 0.2) * attn.view(1, heads, d)).sum(-1)
    m = torch.full((num_in, heads), float("-inf"), dtype=zs.dtype).scatter_reduce(
        0, rows[:, None].expand(-1, heads), e, "amax")
    p = torch.exp(e - m[rows])
    s = torch.zeros(num_in, heads, dtype=zs.dtype).index_add(0, rows, p)
    a = p / s[rows]                                                # [E, H]
    dot = (gv[rows] * zs[cols]).sum(-1)                            # [E, H]
    dv = torch.zeros(num_in, heads, dtype=zs.dtype).index_add(0, rows, a * dot)
    de = a * (dot - dv[rows])
    slope = torch.where(t > 0, torch.ones_like(t), torch.full_like(t, 0.2))
    term = de[..., None] * attn.view(1, heads, d) * slope          # [E, H, D]
    dzs = torch.zeros_like(zs).index_add(0, cols, a[..., None] * gv[rows] + term)
    dzd = torch.zeros_like(zd).index_add(0, rows, term)
    dattn = (de[..., None] * F.leaky_relu(t, 0.2)).sum(0).view(1, heads, d)
    return dzs, dzd, dattn, dv


def _graph(num_in=60, num_halo=25, seed=0):
    """Edges (rows = destinations, cols = sources) with self loops, hub rows, rows whose only edge is the self loop,
    and a halo source with many destinations."""
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    deg = torch.randint(1, 6, (num_in,), generator=gen)
    deg[:3] = torch.tensor([70, 45, 33])
    deg[3:8] = 0
    dst = torch.repeat_interleave(torch.arange(num_in), deg)
    src = torch.randint(0, num_all, (int(deg.sum()),), generator=gen)
    src[torch.randperm(src.numel(), generator=gen)[:30]] = num_in + 2
    pairs = torch.unique(torch.stack([dst, src], 1), dim=0)
    pairs = pairs[pairs[:, 0] != pairs[:, 1]]
    loops = torch.arange(num_in)
    return torch.cat([pairs[:, 0], loops]), torch.cat([pairs[:, 1], loops]), num_in, num_all


@pytest.mark.parametrize("heads,d", [(1, 5), (2, 3), (4, 8)])
@pytest.mark.parametrize("masked", [False, True])
def test_backward_formulas_equal_autograd(heads, d, masked):
    rows, cols, num_in, num_all = _graph()
    gen = torch.Generator().manual_seed(heads * 10 + d)
    zs = torch.randn(num_all, heads, d, generator=gen, dtype=torch.float64)
    zd = torch.randn(num_in, heads, d, generator=gen, dtype=torch.float64)
    # t_uv exactly 0 in some columns: zd of a destination is minus zs of one of its sources there
    for v in range(10, 30):
        u = int(cols[rows == v][0])
        zd[v, :, 0] = -zs[u, :, 0]
        if v % 2:
            zd[v] = -zs[u]                                         # the whole edge: every column of t is 0
    attn = torch.randn(1, heads, d, generator=gen, dtype=torch.float64)
    if masked:
        keep = torch.ones(num_all, dtype=torch.bool)
        keep[num_in:] = torch.rand(num_all - num_in, generator=gen) < 0.5
        keep[num_in + 2] = True
        ek = keep[cols]
        rows, cols = rows[ek], cols[ek]
    t = zs[cols] + zd[rows]
    assert int((t == 0).sum()) >= 20
    g = torch.randn(num_in, heads * d, generator=gen, dtype=torch.float64)

    leaves = [x.clone().requires_grad_(True) for x in (zs, zd, attn)]
    out, _, _ = ref_gatv2(*leaves, rows, cols, num_in)
    out.backward(g)
    dzs, dzd, dattn, dv = ref_gatv2_backward(zs, zd, attn, rows, cols, num_in, g)
    for name, got, ref in (("d zs", dzs, leaves[0].grad), ("d zd", dzd, leaves[1].grad), ("d attn", dattn, leaves[2].grad)):
        torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-12, msg=name)
    torch.testing.assert_close(dv, (out.detach() * g).view(num_in, heads, d).sum(-1), rtol=1e-10, atol=1e-12)
    if masked:
        unkept = ~keep
        assert torch.count_nonzero(dzs[unkept]) == 0


# ------------------------------------------------------------------------------------------------ flags, model
def test_parser_accepts_gatv2_and_heads():
    from pipegcn_b200.helper.parser import create_parser
    args = create_parser(["--model", "gatv2", "--n-heads", "8"])
    assert args.model == "gatv2" and args.n_heads == 8
    base = vars(create_parser([]))
    assert "n_heads" not in base
    with_model = vars(create_parser(["--model", "gatv2"]))
    assert with_model.pop("model") == "gatv2"
    base.pop("model")
    assert with_model == base


def _args(**kw):
    base = dict(model="gatv2", use_pp=False, n_hidden=16, n_heads=4, enable_pipeline=False, feat_corr=False,
                grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(use_pp=True), NotImplementedError, "gatv2 with --use-pp"),
    (dict(aggregator="pool"), ValueError, "--model gatv2 has none"),
    (dict(n_hidden=16, n_heads=3), ValueError, "--n-heads"),
    (dict(n_hidden=10, n_heads=4), ValueError, "--n-heads"),
])
def test_refused_before_allocation(kw, exc, match):
    """RankEngine and init_processes refuse before touching the layout, the world or a device."""
    from pipegcn_b200 import train
    args = _args(**kw)
    with pytest.raises(exc, match=match):
        train.RankEngine(None, args, None)
    with pytest.raises(exc, match=match):
        train.init_processes(0, 2, args)


def test_other_models_still_raise():
    from pipegcn_b200.train import create_model
    args = argparse.Namespace(model="gatv3", use_pp=False, norm="layer", dropout=0.5, n_linear=0, n_train=1)
    with pytest.raises(NotImplementedError):
        create_model([4, 4, 2], args)


def _model(n_linear, seed=0, heads=4):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    args = create_parser(["--model", "gatv2", "--n-heads", str(heads), "--n-hidden", "16", "--n-layers", "3",
                          "--n-linear", str(n_linear)])
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], args)


@pytest.mark.parametrize("n_linear", [0, 1])
def test_state_dict_keys_and_shapes(n_linear):
    from pipegcn_b200.module.model import GATv2
    m = _model(n_linear)
    assert isinstance(m, GATv2)
    want = {}
    for i in range(3 - n_linear):
        d_in, (H, D) = [20, 16, 16][i], ((4, 4) if i < 2 else (1, 5))
        for fc in ("fc_src", "fc_dst"):
            want.update({f"layers.{i}.{fc}.weight": (H * D, d_in), f"layers.{i}.{fc}.bias": (H * D,)})
        want[f"layers.{i}.attn"] = (1, H, D)
    if n_linear:
        want.update({"layers.2.weight": (5, 16), "layers.2.bias": (5,)})
    for i in range(2):
        want.update({f"norm.{i}.weight": (16,), f"norm.{i}.bias": (16,)})
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == want


def test_initialisation_is_gatv2conv_and_seeded():
    a, b, c = _model(0, seed=3), _model(0, seed=3), _model(0, seed=4)
    for (k, x), (_, y), (_, z) in zip(a.state_dict().items(), b.state_dict().items(), c.state_dict().items()):
        assert torch.equal(x, y), k
        if k.endswith("bias") and k.startswith("layers."):
            assert torch.count_nonzero(x) == 0, k          # fc_src / fc_dst biases start at 0
        elif not k.startswith("norm."):
            assert not torch.equal(x, z), k
    # xavier_normal_ with gain calculate_gain('relu'): std = gain * sqrt(2 / (fan_in + fan_out))
    gain = torch.nn.init.calculate_gain("relu")
    layer = _model(0, seed=5).layers[0]
    for w in (layer.fc_src.weight, layer.fc_dst.weight):
        std = gain * (2.0 / (20 + 16)) ** 0.5
        assert 0.7 * std < float(w.detach().std()) < 1.3 * std
    # attn [1, 4, 4]: fan_in = 4 * 4, fan_out = 1 * 4
    attn = torch.cat([_model(0, seed=s).layers[0].attn.detach().reshape(-1) for s in range(20)])
    std = gain * (2.0 / (16 + 4)) ** 0.5
    assert 0.8 * std < float(attn.std()) < 1.2 * std


def test_draw_order_is_src_dst_attn():
    from pipegcn_b200.module.layer import GATv2Layer
    torch.manual_seed(11)
    layer = GATv2Layer(20, 4, 4)
    torch.manual_seed(11)
    gain = torch.nn.init.calculate_gain("relu")
    w_s, w_d, attn = torch.empty(16, 20), torch.empty(16, 20), torch.empty(1, 4, 4)
    torch.nn.Linear(20, 16), torch.nn.Linear(20, 16)               # the construction draws of fc_src and fc_dst
    torch.nn.init.xavier_normal_(w_s, gain=gain)
    torch.nn.init.xavier_normal_(w_d, gain=gain)
    torch.nn.init.xavier_normal_(attn, gain=gain)
    assert torch.equal(layer.fc_src.weight.detach(), w_s)
    assert torch.equal(layer.fc_dst.weight.detach(), w_d)
    assert torch.equal(layer.attn.detach(), attn)
