"""The oracle and the layout builder against the golden fixtures, i.e. against outputs of the UNMODIFIED
reference code (tests/golden/make_golden.py ran PipeGCN's Buffer, GraphSAGE, Reducer and set-up helpers
over gloo on the host).  This is what pins the oracle: fp32, same inputs, same initial weights."""
from pathlib import Path

import pytest
import torch

from oracle import dglpart
from oracle import setup as osetup
from oracle.train import OracleArgs, run_world
from pipegcn_b200.partition import build_layouts
from pipegcn_b200.synthetic import GlobalGraph

GOLDEN = Path(__file__).resolve().parent / "golden"
FIXTURES = sorted(p.name for p in GOLDEN.glob("ref_*.pt"))


def load(name):
    fx = torch.load(GOLDEN / name, weights_only=False)
    gr = fx["graph"]
    g = GlobalGraph(gr["n_nodes"], gr["src"], gr["dst"], gr["feat"], gr["label"], gr["train_mask"])
    return fx, g, gr["part"]


def oracle_args(fx, g):
    c = fx["config"]
    return OracleArgs(n_layers=c["n_layers"], n_hidden=c["n_hidden"], n_feat=g.n_feat, n_class=c["n_class"],
                      n_train=int(g.train_mask.sum()), dropout=0.0, lr=c["lr"], n_epochs=c["n_epochs"], seed=c["seed"],
                      enable_pipeline=c.get("enable_pipeline", False), feat_corr=c.get("feat_corr", False),
                      grad_corr=c.get("grad_corr", False), corr_momentum=c.get("corr_momentum", 0.95),
                      use_pp=c.get("use_pp", False))


def test_fixtures_exist():
    assert len(FIXTURES) >= 4


@pytest.mark.parametrize("name", FIXTURES)
def test_layouts_equal_reference_setup(name):
    """Index spaces: reference helpers (train.py:84-155,206-229, utils.py:154-188) == oracle == product, exactly."""
    fx, g, part = load(name)
    P = fx["config"]["n_parts"]
    setups = osetup.setup_world(dglpart.partition_graph(g.n_nodes, g.src, g.dst, part, P, g.feat, g.label, g.train_mask))
    layouts = build_layouts(g, part, P)
    for r in range(P):
        ref, S, L = fx["ranks"][r]["layout"], setups[r], layouts[r]
        assert (ref["num_in"], ref["num_all"]) == (S.num_in, S.num_all) == (L.num_in, L.num_all)
        key_ref = torch.sort(ref["v"] * ref["num_all"] + ref["u"]).values
        assert torch.equal(key_ref, torch.sort(S.v * S.num_all + S.u).values)
        rows = torch.repeat_interleave(torch.arange(L.num_in), (L.indptr[1:] - L.indptr[:-1]).long())
        assert torch.equal(key_ref, torch.sort(rows * L.num_all + L.indices.long()).values)
        assert ref["recv_shape"] == S.recv_shape == L.recv_shape
        for a, b, c in zip(ref["boundary"], S.boundary, L.boundary):
            assert (a is None and b is None and c is None) or (torch.equal(a, b) and torch.equal(a, c))
        assert torch.equal(ref["in_deg"][: S.num_in], S.in_deg) and torch.equal(S.in_deg, L.in_deg)
        n_feat = S.node_dict["feat"].shape[1]            # with --use-pp the reference's feat is cat(feat, mean)
        assert torch.equal(ref["feat"][: S.num_in, :n_feat], S.node_dict["feat"]) and torch.equal(S.node_dict["feat"], L.feat)
        assert torch.equal(ref["label"], L.label) and torch.equal(ref["train_mask"], L.train_mask)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_run(name):
    """Per-layer concatenated features, layer outputs, logits, loss and reduced gradients of every epoch.
    fp32 tolerance: rtol 1e-5 / atol 1e-6 (only the neighbour-sum order differs)."""
    fx, g, part = load(name)
    P = fx["config"]["n_parts"]
    setups = osetup.setup_world(dglpart.partition_graph(g.n_nodes, g.src, g.dst, part, P, g.feat, g.label, g.train_mask))
    oargs = oracle_args(fx, g)
    init = fx["ranks"][0]["init_state"]
    forced = [ep["state"] for ep in fx["ranks"][0]["epochs"]]
    traces = run_world(setups, oargs, init_state=init, forced_states=forced)
    tol = dict(rtol=1e-5, atol=1e-6)
    for r in range(P):
        for e, ep in enumerate(fx["ranks"][r]["epochs"]):
            for l, rec in ep["layers"].items():
                torch.testing.assert_close(traces[r].layers[e][l]["f_buf"], rec["f_buf"], **tol)
                torch.testing.assert_close(traces[r].layers[e][l]["layer_out"], rec["layer_out"], **tol)
            torch.testing.assert_close(traces[r].logits[e], ep["logits"], **tol)
            assert abs(traces[r].losses[e] - ep["loss"]) <= 1e-5 * abs(ep["loss"])
            for n, gref in ep["grads"].items():
                torch.testing.assert_close(traces[r].grads[e][n], gref, rtol=1e-4, atol=1e-7)


def test_oracle_free_running_matches_reference_weights():
    """Without teacher forcing the oracle's own Adam trajectory stays on the reference's (same torch optimizer)."""
    fx, g, part = load("ref_sync_p2.pt")
    setups = osetup.setup_world(dglpart.partition_graph(g.n_nodes, g.src, g.dst, part, 2, g.feat, g.label, g.train_mask))
    traces = run_world(setups, oracle_args(fx, g), init_state=fx["ranks"][0]["init_state"])
    for e, ep in enumerate(fx["ranks"][0]["epochs"]):
        assert abs(traces[0].losses[e] - ep["loss"]) <= 2e-3 * abs(ep["loss"])


def test_seeded_initial_weights_equal_reference():
    """`torch.manual_seed(seed)` + model construction draws the reference's initial weights (layer.py:24-36)."""
    from oracle.train import initial_state
    fx, g, _ = load("ref_sync_p2.pt")
    init = initial_state(oracle_args(fx, g))
    ref = fx["ranks"][0]["init_state"]
    assert set(init) == set(ref)
    for k in ref:
        assert torch.equal(init[k], ref[k]), k
    import torch.nn.functional as F
    from pipegcn_b200.module.model import GraphSAGE
    from pipegcn_b200.partition import get_layer_size
    c = fx["config"]
    torch.manual_seed(c["seed"])
    m = GraphSAGE(get_layer_size(g.n_feat, c["n_hidden"], c["n_class"], c["n_layers"]), F.relu, False, dropout=0.0)
    for k in ref:
        assert torch.equal(m.state_dict()[k], ref[k]), k
