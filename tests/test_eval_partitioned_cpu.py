"""Host-side pieces of the partition-parallel evaluation (--eval-partitioned): the evaluation masks of the layouts,
the partition of the inductive evaluation graphs, the partitioned forward restated in torch on the oracle model, and
the command-line default."""
import argparse

import pytest
import torch


def test_layout_masks_follow_global_graph_rule():
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny")
    for lay in build_layouts(g, random_partition(g.n_nodes, 3), 3):
        assert torch.equal(lay.val_mask, g.val_mask[lay.inner_gid])
        assert torch.equal(lay.test_mask, g.test_mask[lay.inner_gid])
        assert not (lay.val_mask & lay.test_mask).any() and not (lay.val_mask & lay.train_mask).any()


def test_distgraph_masks_follow_global_graph_rule():
    from pipegcn_b200.distgraph import build_rank_layout
    spec = dict(n_nodes=2_000, n_edges=20_000, n_feat=8, n_class=4, train_frac=0.5)
    for r in range(2):
        lay, _ = build_rank_layout(spec, r, 2, "cpu")
        ids = lay.inner_gid
        assert torch.equal(lay.val_mask, ~lay.train_mask & (ids % 2 == 0))
        assert torch.equal(lay.test_mask, ~lay.train_mask & (ids % 2 == 1))


def test_inductive_eval_partition_extends_training_partition():
    from pipegcn_b200.partition import build_eval_layout, extend_partition
    from pipegcn_b200.synthetic import induced_subgraph, make_graph, random_partition, train_subgraph
    g = make_graph("tiny")
    gt = train_subgraph(g)
    tpart = random_partition(gt.n_nodes, 3)
    a = extend_partition(g.train_mask, tpart, 3)
    b = extend_partition(g.train_mask, tpart, 3)
    assert torch.equal(a, b)                                   # deterministic: the same on every rank
    assert torch.equal(a[g.train_mask], tpart)                 # every training node keeps its part
    assert set(a[~g.train_mask].tolist()) == {0, 1, 2}
    keep = g.train_mask | g.val_mask
    sub, ids = induced_subgraph(g, keep)
    lays = [build_eval_layout(g, keep, a, 3, r) for r in range(3)]
    assert sorted(torch.cat([l.inner_gid for l in lays]).tolist()) == list(range(sub.n_nodes))
    for lay in lays:
        assert torch.equal(lay.val_mask, g.val_mask[ids[lay.inner_gid]])
        assert not lay.test_mask.any()                         # the validation graph holds no test node
        assert torch.equal(lay.label, g.label[ids[lay.inner_gid]])
    full = [build_eval_layout(g, None, a, 3, r) for r in range(3)]
    assert int(sum(l.test_mask.sum() for l in full)) == int(g.test_mask.sum())


def _edges(lay):
    v = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
    return lay.indices.long(), v


@pytest.mark.parametrize("n_parts", [1, 2, 3])
def test_partitioned_forward_restated_in_torch_matches_oracle(n_parts):
    """Every rank computes its inner rows of each layer from [its inner rows | halo rows gathered by halo_gid] of the
    previous layer's output: the oracle model gives the logits of its full-graph evaluation."""
    import torch.nn.functional as F
    from oracle.model import OracleGraph, OracleGraphSAGE
    from pipegcn_b200.partition import build_layouts, get_layer_size
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("tiny")
    torch.manual_seed(0)
    model = OracleGraphSAGE(get_layer_size(g.n_feat, 16, 5, 4), F.relu, False, norm="layer", n_linear=1).eval()
    deg = g.in_degrees().float()
    with torch.no_grad():
        ref = model(OracleGraph(g.src, g.dst, g.n_nodes, g.n_nodes), g.feat, deg, None)
        lays = build_layouts(g, random_partition(g.n_nodes, n_parts), n_parts)
        graphs = [OracleGraph(*_edges(l), l.num_in, l.num_all) for l in lays]
        n_graph = model.n_layers - model.n_linear
        h = g.feat.clone()                                     # the current layer's input, all nodes (global ids)
        for i in range(model.n_layers):
            out = torch.empty(g.n_nodes, model.layers[i].out_features if i >= n_graph else
                              model.layers[i].linear1.out_features)
            for lay, og in zip(lays, graphs):
                if i < n_graph:
                    x = torch.cat([h[lay.inner_gid], h[lay.halo_gid]])          # inner rows, then halo rows
                    y = model.layers[i](og, x, lay.in_deg.float())
                else:
                    y = model.layers[i](h[lay.inner_gid])
                if i < model.n_layers - 1:
                    y = F.relu(model.norm[i](y))
                out[lay.inner_gid] = y
            h = out
    torch.testing.assert_close(h, ref, rtol=1e-5, atol=1e-5)


def test_parser_flag_is_off_by_default():
    from pipegcn_b200.helper.parser import create_parser
    assert getattr(create_parser([]), "eval_partitioned", False) is False
    assert create_parser(["--eval-partitioned"]).eval_partitioned is True
    assert create_parser(["--eval_partitioned"]).eval_partitioned is True


class _StubEngine:
    def __init__(self, layout, args, world, buffer=None, reducer=None):
        self.buffer = argparse.Namespace(timer=None)


def test_run_takes_todays_eval_path_without_the_flag(monkeypatch):
    """Without --eval-partitioned rank 0 needs the global graph (today's path); with it no rank does, and an inductive
    run asks for the evaluation layouts instead."""
    from pipegcn_b200 import train
    monkeypatch.setattr(train, "RankEngine", _StubEngine)
    world = argparse.Namespace(rank=0, size=2)
    args = argparse.Namespace(eval=True, inductive=True, n_epochs=0)
    with pytest.raises(ValueError, match="global graph"):
        train.run(None, args, world, eval_graph=None)
    args.eval_partitioned = True
    with pytest.raises(ValueError, match="eval_layouts"):
        train.run(None, args, world, eval_graph=None)


def test_multilabel_evaluation_is_refused():
    """As calc_acc: multi-label (yelp) accuracy is not implemented, whichever path evaluates."""
    from pipegcn_b200 import ops
    from pipegcn_b200.evaluate import calc_acc
    labels = torch.zeros(4, 3, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        calc_acc(torch.zeros(4, 3), labels)
    with pytest.raises(NotImplementedError):
        ops.eval_count(torch.zeros(4, 3), labels, torch.zeros(4, dtype=torch.uint8), 1)
