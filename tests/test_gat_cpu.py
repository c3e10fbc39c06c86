"""Graph attention (`--model gat`) without a GPU: the parser flags, the refused configurations, the parameters
(DGL GATConv's keys and shapes) and their seeded initialisation."""
import argparse

import pytest
import torch


def test_parser_accepts_gat_and_heads():
    from pipegcn_b200.helper.parser import create_parser
    args = create_parser(["--model", "gat", "--n-heads", "8"])
    assert args.model == "gat" and args.n_heads == 8
    assert create_parser(["--model", "gat", "--n_heads", "2"]).n_heads == 2
    for bad in ("0", "-1", "two"):
        with pytest.raises(SystemExit):
            create_parser(["--n-heads", bad])


def test_flag_absent_keeps_todays_namespace():
    from pipegcn_b200.helper.parser import create_parser
    base = vars(create_parser([]))
    assert "n_heads" not in base
    with_flag = vars(create_parser(["--n-heads", "4"]))
    assert with_flag.pop("n_heads") == 4
    assert with_flag == base


def _args(**kw):
    base = dict(model="gat", use_pp=False, n_hidden=16, n_heads=4, enable_pipeline=False, feat_corr=False,
                grad_corr=False)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(use_pp=True), NotImplementedError, "--use-pp"),
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


def test_graphsage_configurations_pass_the_gat_check():
    from pipegcn_b200 import train
    train.check_model(argparse.Namespace(model="graphsage", use_pp=True, n_hidden=10))
    train.check_model(_args(n_hidden=12, n_heads=3))


def _model(n_linear, seed=0, heads=4):
    from pipegcn_b200.helper.parser import create_parser
    from pipegcn_b200.train import create_model
    args = create_parser(["--model", "gat", "--n-heads", str(heads), "--n-hidden", "16", "--n-layers", "3",
                          "--n-linear", str(n_linear)])
    torch.manual_seed(seed)
    return create_model([20, 16, 16, 5], args)


@pytest.mark.parametrize("n_linear", [0, 1])
def test_state_dict_keys_and_shapes(n_linear):
    from pipegcn_b200.module.model import GAT
    m = _model(n_linear)
    assert isinstance(m, GAT)
    want = {}
    for i in range(3 - n_linear):
        d_in, (H, D) = [20, 16, 16][i], ((4, 4) if i < 2 else (1, 5))
        want.update({f"layers.{i}.fc.weight": (H * D, d_in), f"layers.{i}.attn_l": (1, H, D),
                     f"layers.{i}.attn_r": (1, H, D), f"layers.{i}.bias": (H * D,)})
    if n_linear:
        want.update({"layers.2.weight": (5, 16), "layers.2.bias": (5,)})
    for i in range(2):
        want.update({f"norm.{i}.weight": (16,), f"norm.{i}.bias": (16,)})
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == want


def test_initialisation_is_gatconv_and_seeded():
    a, b, c = _model(0, seed=3), _model(0, seed=3), _model(0, seed=4)
    for (k, x), (_, y), (_, z) in zip(a.state_dict().items(), b.state_dict().items(), c.state_dict().items()):
        assert torch.equal(x, y), k
        if k.endswith("bias") and k.startswith("layers."):
            assert torch.count_nonzero(x) == 0, k          # GATConv: zero bias
        elif not k.startswith("norm."):
            assert not torch.equal(x, z), k
    # xavier_normal_ with gain calculate_gain('relu'): std = gain * sqrt(2 / (fan_in + fan_out))
    w = _model(0, seed=5).layers[0].fc.weight
    std = torch.nn.init.calculate_gain("relu") * (2.0 / (20 + 16)) ** 0.5
    assert 0.7 * std < float(w.detach().std()) < 1.3 * std


def test_non_graphsage_models_other_than_gat_still_raise():
    from pipegcn_b200.train import create_model
    args = argparse.Namespace(model="gin", use_pp=False, norm="layer", dropout=0.5, n_linear=0, n_train=1)
    with pytest.raises(NotImplementedError):
        create_model([4, 4, 2], args)
