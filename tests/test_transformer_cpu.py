"""Graph transformer (`--model transformer`) without a GPU: the parser, the refused configurations, the parameters
(PyG TransformerConv's keys and shapes) and their seeded initialisation, the paired operand layout, and the backward
formulas the kernels implement, written out in fp64 and checked against torch.autograd of the forward restatement."""
import argparse
import math

import pytest
import torch

from tests.test_gatv2_cpu import _graph


# ------------------------------------------------------------------------------------------------ restatement
def _softmax_weights(q, k, rows, cols, num_in):
    """a_uv [E, H] and the statistics (m, s) [num_in, H] of e_uv = <q_v, k_u> / sqrt(D) over the edges cols -> rows."""
    heads, d = q.shape[1], q.shape[2]
    e = (q[rows] * k[cols]).sum(-1) / math.sqrt(d)                 # [E, H]
    m = torch.full((num_in, heads), float("-inf"), dtype=q.dtype, device=q.device)
    m = m.scatter_reduce(0, rows[:, None].expand(-1, heads), e.detach(), "amax")
    p = torch.exp(e - m[rows])
    s = torch.zeros(num_in, heads, dtype=q.dtype, device=q.device).index_add(0, rows, p)
    return p / s[rows], m, s.detach()


def ref_transformer(q, k, v, skip, rows, cols, num_in):
    """fp64 TransformerConv aggregate over the edges cols -> rows: q [num_in, H, D], k and v [num_all, H, D], skip
    [num_in, H*D] -> out [num_in, H*D] and the softmax statistics (m, s) [num_in, H]."""
    a, m, s = _softmax_weights(q, k, rows, cols, num_in)
    out = torch.zeros(num_in, q.shape[1], q.shape[2], dtype=q.dtype, device=q.device)
    out = out.index_add(0, rows, a[..., None] * v[cols])
    return out.reshape(num_in, -1) + skip, m, s


def ref_transformer_backward(q, k, v, rows, cols, num_in, g):
    """The backward of ref_transformer as the kernels compute it, g = dL/d out [num_in, H*D], scale = 1/sqrt(D):
        gd_uv = <g_v, v_u>,  delta_v = sum_u a_uv gd_uv,  c_uv = a_uv (gd_uv - delta_v)
        dq_v = scale (A_v - delta_v B_v) with A_v = sum_u a_uv gd_uv k_u, B_v = sum_u a_uv k_u  (the destination pass)
        dk_u = scale sum_v c_uv q_v,  dv_u = sum_v a_uv g_v  (the source pass),  d skip = g
    Returns (dq, dk, dv, delta)."""
    heads, d = q.shape[1], q.shape[2]
    scale = 1.0 / math.sqrt(d)
    gv = g.view(num_in, heads, d)
    a, _, _ = _softmax_weights(q, k, rows, cols, num_in)
    gd = (gv[rows] * v[cols]).sum(-1)                              # [E, H]
    delta = torch.zeros(num_in, heads, dtype=q.dtype).index_add(0, rows, a * gd)
    A = torch.zeros_like(q).index_add(0, rows, (a * gd)[..., None] * k[cols])
    B = torch.zeros_like(q).index_add(0, rows, a[..., None] * k[cols])
    dq = scale * (A - delta[..., None] * B)
    c = a * (gd - delta[rows])
    dk = scale * torch.zeros_like(k).index_add(0, cols, c[..., None] * q[rows])
    dv = torch.zeros_like(v).index_add(0, cols, a[..., None] * gv[rows])
    return dq, dk, dv, delta


@pytest.mark.parametrize("heads,d", [(1, 5), (2, 3), (4, 8)])
@pytest.mark.parametrize("masked", [False, True])
def test_backward_formulas_equal_autograd(heads, d, masked):
    """Rows 3-7 have only their self loop; rows 10-29 have scores near 1e3, where exp without the max subtraction
    overflows even in fp64."""
    rows, cols, num_in, num_all = _graph()
    gen = torch.Generator().manual_seed(heads * 10 + d)
    q = torch.randn(num_in, heads, d, generator=gen, dtype=torch.float64)
    k = torch.randn(num_all, heads, d, generator=gen, dtype=torch.float64)
    v = torch.randn(num_all, heads, d, generator=gen, dtype=torch.float64)
    skip = torch.randn(num_in, heads * d, generator=gen, dtype=torch.float64)
    q[10:30] *= 40 * math.sqrt(d)
    k[:num_in] *= 5
    if masked:
        keep = torch.ones(num_all, dtype=torch.bool)
        keep[num_in:] = torch.rand(num_all - num_in, generator=gen) < 0.5
        keep[num_in + 2] = True
        ek = keep[cols]
        rows, cols = rows[ek], cols[ek]
    e = (q[rows] * k[cols]).sum(-1) / math.sqrt(d)
    assert float(e.abs().max()) > 710                               # exp(710) overflows fp64
    g = torch.randn(num_in, heads * d, generator=gen, dtype=torch.float64)

    leaves = [x.clone().requires_grad_(True) for x in (q, k, v, skip)]
    out, m, s = ref_transformer(*leaves, rows, cols, num_in)
    assert torch.isfinite(out).all() and bool((s[:num_in] >= 1).all())
    out.backward(g)
    dq, dk, dv, delta = ref_transformer_backward(q, k, v, rows, cols, num_in, g)
    for name, got, ref in (("dq", dq, leaves[0].grad), ("dk", dk, leaves[1].grad), ("dv", dv, leaves[2].grad)):
        torch.testing.assert_close(got, ref, rtol=1e-10, atol=1e-10, msg=name)
    torch.testing.assert_close(leaves[3].grad, g)                  # d skip = g
    attn = (out.detach() - skip).view(num_in, heads, d)
    torch.testing.assert_close(delta, (attn * g.view(num_in, heads, d)).sum(-1), rtol=1e-10, atol=1e-10)
    for r in range(3, 8):                                          # only the self loop: a_vv = 1, dq_v = 0
        torch.testing.assert_close(attn[r], v[r])
        assert torch.count_nonzero(dq[r]) == 0
    # the gradient of b_k, sum_u dk_u, is 0: every score of a row moves by the same <q_v, b_k>
    torch.testing.assert_close(dk.sum(0), torch.zeros_like(dk[0]), rtol=0, atol=1e-12 * float(dk.abs().sum()))
    if masked:
        unkept = ~keep
        assert torch.count_nonzero(dk[unkept]) == 0 and torch.count_nonzero(dv[unkept]) == 0


# ------------------------------------------------------------------------------------------------ operand layout
@pytest.mark.parametrize("dtype,hd,want", [(torch.float32, 4, 4), (torch.float32, 6, 8), (torch.float32, 64, 64),
                                           (torch.bfloat16, 8, 8), (torch.bfloat16, 12, 16), (torch.bfloat16, 5, 8),
                                           (torch.bfloat16, 256, 256)])
def test_half_width_starts_16_byte_aligned(dtype, hd, want):
    from pipegcn_b200.ops import transformer_width
    w = transformer_width(hd, dtype)
    assert w == want and (w * torch.empty((), dtype=dtype).element_size()) % 16 == 0


@pytest.mark.parametrize("transpose", [False, True])
def test_paired_weight_layout(transpose):
    """[W_a; 0; W_b; 0] with each half at a multiple of 8 rows, and the concatenated bias to match."""
    from pipegcn_b200.ops import _pair_bias, _pair_weight, transformer_width
    gen = torch.Generator().manual_seed(0)
    wa, wb = torch.randn(6, 10, generator=gen), torch.randn(6, 10, generator=gen)
    w = transformer_width(6, torch.bfloat16)
    p = _pair_weight(wa, wb, w, torch.bfloat16, transpose=transpose)
    p = p.t() if transpose else p
    assert p.shape == (16, 10)
    assert torch.equal(p[:6], wa.to(torch.bfloat16)) and torch.equal(p[8:14], wb.to(torch.bfloat16))
    assert torch.count_nonzero(p[6:8]) == 0 and torch.count_nonzero(p[14:]) == 0
    b = _pair_bias(wa[:, 0], wb[:, 0], 6, w)
    assert torch.equal(b[:6], wa[:, 0]) and torch.equal(b[8:14], wb[:, 0]) and torch.count_nonzero(b[6:8]) == 0


# ------------------------------------------------------------------------------------------------ flags, model
def test_parser_accepts_transformer_and_heads():
    from pipegcn_b200.helper.parser import create_parser
    args = create_parser(["--model", "transformer", "--n-heads", "8"])
    assert args.model == "transformer" and args.n_heads == 8
    base = vars(create_parser([]))
    assert "n_heads" not in base
    with_model = vars(create_parser(["--model", "transformer"]))
    assert with_model.pop("model") == "transformer"
    base.pop("model")
    assert with_model == base


def _args(**kw):
    base = dict(model="transformer", use_pp=False, n_hidden=16, n_heads=4, enable_pipeline=False, feat_corr=False,
                grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(use_pp=True), NotImplementedError, "transformer with --use-pp"),
    (dict(aggregator="pool"), ValueError, "--model transformer has none"),
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


def _model(n_linear, seed=0, heads=4):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    args = create_parser(["--model", "transformer", "--n-heads", str(heads), "--n-hidden", "16", "--n-layers", "3",
                          "--n-linear", str(n_linear)])
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], args)


@pytest.mark.parametrize("n_linear", [0, 1])
def test_state_dict_keys_and_shapes(n_linear):
    """PyG's keys; hidden layers have 4 heads of 4, a layer that produces the logits one head of n_class."""
    from pipegcn_b200.module.model import GraphTransformer
    m = _model(n_linear)
    assert isinstance(m, GraphTransformer)
    want = {}
    for i in range(3 - n_linear):
        d_in, (H, D) = [20, 16, 16][i], ((4, 4) if i < 2 else (1, 5))
        for lin in ("lin_key", "lin_query", "lin_value", "lin_skip"):
            want.update({f"layers.{i}.{lin}.weight": (H * D, d_in), f"layers.{i}.{lin}.bias": (H * D,)})
    if n_linear:
        want.update({"layers.2.weight": (5, 16), "layers.2.bias": (5,)})
    for i in range(2):
        want.update({f"norm.{i}.weight": (16,), f"norm.{i}.bias": (16,)})
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == want
    assert [k for k in m.state_dict() if k.startswith("layers.0.")] == [
        f"layers.0.{lin}.{p}" for lin in ("lin_key", "lin_query", "lin_value", "lin_skip") for p in ("weight", "bias")]


def test_initialisation_is_linear_default_and_seeded():
    a, b, c = _model(0, seed=3), _model(0, seed=3), _model(0, seed=4)
    for (k, x), (_, y), (_, z) in zip(a.state_dict().items(), b.state_dict().items(), c.state_dict().items()):
        assert torch.equal(x, y), k
        if not k.startswith("norm."):
            assert not torch.equal(x, z), k
    # nn.Linear's default: weight and bias U(-1/sqrt(d_in), 1/sqrt(d_in)), std = bound / sqrt(3)
    layers = [_model(0, seed=s).layers[0] for s in range(8)]
    bound = 1.0 / math.sqrt(20)
    for name in ("lin_key", "lin_query", "lin_value", "lin_skip"):
        w = torch.cat([getattr(l, name).weight.detach().reshape(-1) for l in layers])
        bias = torch.cat([getattr(l, name).bias.detach() for l in layers])
        for t in (w, bias):
            assert float(t.abs().max()) <= bound, name
        assert 0.9 * bound / math.sqrt(3) < float(w.std()) < 1.1 * bound / math.sqrt(3), name


def test_draw_order_is_key_query_value_skip():
    from pipegcn_b200.module.layer import TransformerLayer
    torch.manual_seed(11)
    layer = TransformerLayer(20, 4, 4)
    torch.manual_seed(11)
    lins = [torch.nn.Linear(20, 16) for _ in range(4)]             # the construction draws
    for lin in lins:                                               # reset_parameters: key, query, value, skip
        lin.reset_parameters()
    for name, lin in zip(("lin_key", "lin_query", "lin_value", "lin_skip"), lins):
        assert torch.equal(getattr(layer, name).weight.detach(), lin.weight.detach()), name
        assert torch.equal(getattr(layer, name).bias.detach(), lin.bias.detach()), name
