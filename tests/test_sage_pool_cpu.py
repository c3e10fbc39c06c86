"""Max-pool GraphSAGE (`--aggregator pool`) without a GPU: the flag, the refusals, the parameters and their draws."""
import argparse

import pytest
import torch
import torch.nn.functional as F

from pipegcn_b200.helper.parser import create_parser
from pipegcn_b200.module.layer import GraphSAGELayer
from pipegcn_b200.module.model import GraphSAGE


@pytest.mark.parametrize("value", ["mean", "pool"])
def test_flag_parses(value):
    assert create_parser(["--aggregator", value]).aggregator == value
    assert create_parser([f"--aggregator={value}"]).aggregator == value


@pytest.mark.parametrize("value", ["max", "lstm", "gcn", "Pool", ""])
def test_bad_values_are_refused(value):
    with pytest.raises(SystemExit):
        create_parser(["--aggregator", value])


def test_absent_flag_leaves_the_namespace_unchanged():
    a = create_parser([])
    assert not hasattr(a, "aggregator")
    assert getattr(a, "aggregator", "mean") == "mean"
    # the namespace with the flag differs from today's by that attribute alone
    b = create_parser(["--aggregator", "mean"])
    assert set(vars(b)) - set(vars(a)) == {"aggregator"}
    assert {k: v for k, v in vars(b).items() if k != "aggregator"} == vars(a)


def _args(**kw):
    base = dict(model="graphsage", use_pp=False, n_hidden=16, n_feat=8, n_class=4, n_layers=2, n_linear=0,
                norm="layer", dropout=0.5, n_train=10)
    base.update(kw)
    return argparse.Namespace(**base)


class _Boom:
    """A world whose first use fails the test: the refusals must come before anything is allocated."""

    def __getattr__(self, name):
        raise AssertionError(f"world.{name} used before the configuration was refused")


@pytest.mark.parametrize("kw,exc", [(dict(model="gat", aggregator="pool"), ValueError),
                                    (dict(use_pp=True, aggregator="pool"), NotImplementedError)])
def test_refused_configurations_raise_before_allocation(kw, exc):
    from pipegcn_b200.train import RankEngine, check_model, create_model
    a = _args(**kw)
    with pytest.raises(exc):
        check_model(a)
    with pytest.raises(exc):
        create_model([8, 16, 4], a)
    a.sampling_rate, a.enable_pipeline, a.feat_corr, a.grad_corr = 1.0, False, False, False
    with pytest.raises(exc):
        RankEngine(None, a, _Boom())


def test_mean_and_gat_configurations_still_pass_the_check():
    from pipegcn_b200.train import check_model
    check_model(_args())
    check_model(_args(aggregator="mean", use_pp=True))
    check_model(_args(aggregator="pool"))
    check_model(_args(model="gat", n_heads=4))


def test_pool_parameters_keys_shapes_and_draw_order():
    torch.manual_seed(3)
    m = GraphSAGE([8, 16, 16, 4], F.relu, False, aggregator="pool", n_linear=1)
    sd = m.state_dict()
    for i, (d_in, d_out) in enumerate([(8, 16), (16, 16)]):
        assert tuple(sd[f"layers.{i}.pool.weight"].shape) == (d_in, d_in)
        assert tuple(sd[f"layers.{i}.pool.bias"].shape) == (d_in,)
        assert tuple(sd[f"layers.{i}.linear1.weight"].shape) == (d_out, d_in)
        assert tuple(sd[f"layers.{i}.linear2.weight"].shape) == (d_out, d_in)
    assert "layers.2.pool.weight" not in sd and tuple(sd["layers.2.weight"].shape) == (4, 16)

    # the draws: construct the three linears, then weights (linear1, linear2, pool), then biases, all U(+-1/sqrt(d_in))
    torch.manual_seed(11)
    layer = GraphSAGELayer(24, 10, aggregator="pool")
    torch.manual_seed(11)
    lins = [torch.nn.Linear(24, 10), torch.nn.Linear(24, 10), torch.nn.Linear(24, 24)]
    bound = 1 / 24 ** 0.5
    ws = [torch.empty_like(l.weight).uniform_(-bound, bound) for l in lins]
    bs = [torch.empty_like(l.bias).uniform_(-bound, bound) for l in lins]
    for lin, w, b in zip((layer.linear1, layer.linear2, layer.pool), ws, bs):
        assert torch.equal(lin.weight, w) and torch.equal(lin.bias, b)


def test_mean_model_weights_are_unchanged():
    """The default and an explicit 'mean' draw exactly the weights of a model built without the argument, which are
    the draws of two linears per layer."""
    torch.manual_seed(5)
    a = GraphSAGE([8, 16, 4], F.relu, False).state_dict()
    torch.manual_seed(5)
    b = GraphSAGE([8, 16, 4], F.relu, False, aggregator="mean").state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert not any(".pool." in k for k in a)
    torch.manual_seed(5)
    lins = [torch.nn.Linear(8, 16), torch.nn.Linear(8, 16)]
    bound = 1 / 8 ** 0.5
    ws = [torch.empty_like(l.weight).uniform_(-bound, bound) for l in lins]
    assert torch.equal(a["layers.0.linear1.weight"], ws[0]) and torch.equal(a["layers.0.linear2.weight"], ws[1])


def test_layer_refuses_bad_aggregators():
    with pytest.raises(ValueError):
        GraphSAGELayer(4, 4, aggregator="lstm")
    with pytest.raises(NotImplementedError):
        GraphSAGELayer(4, 4, use_pp=True, aggregator="pool")
    with pytest.raises(NotImplementedError):
        GraphSAGE([8, 16, 4], F.relu, True, aggregator="pool")
