"""Partition-parallel evaluation (--eval-partitioned) on the GPU: the accuracy-count kernel against torch, the
partitioned logits and accuracies against rank 0's full-graph evaluation, training left bit-identical by evaluations
in between, the inductive evaluation graphs, the trainer end to end, and two real ranks under torchrun."""
import argparse
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


# ---------------------------------------------------------------------------------------------------- pg_eval_count
@pytest.mark.parametrize("n_rows", [0, 1, 33, 100_003])
@pytest.mark.parametrize("c", [1, 2, 5, 41, 64, 172, 1000])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_eval_count_matches_torch(dtype, c, n_rows):
    from pipegcn_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(c * 7 + n_rows)
    ld = c + 3                                               # padded, unaligned rows
    base = torch.randn(n_rows, ld, generator=gen, device="cuda").to(dtype)
    z = base[:, :c]
    if n_rows > 8 and c > 1:
        z[1, :] = 1.5                                        # all equal: index 0
        z[2, c // 2:] = z[2].max() + 1                       # a tie of several maxima: the first
        z[3, c - 1] = float("nan")                           # NaN is the maximum
        z[4, 0] = float("nan")
        z[4, c - 1] = float("nan")                           # two NaNs: the first
        z[5, :] = float("-inf")
    labels = torch.randint(0, c, (n_rows,), generator=gen, device="cuda")
    if n_rows > 8:
        labels[:6] = torch.argmax(z[:6].float(), dim=1)      # the special rows are hits (when torch agrees)
    tag = torch.randint(0, 4, (n_rows,), generator=gen, device="cuda").to(torch.uint8)   # overlapping: bits 0 and 1
    n_tags = 3                                               # mask 2 is empty
    counts, pred = ops.eval_count(z, labels, tag, n_tags, want_pred=True)
    want_pred = torch.argmax(z, dim=1)
    assert torch.equal(pred.long(), want_pred)
    hit = want_pred == labels
    for k in range(n_tags):
        m = (tag.long() >> k) & 1 == 1
        assert counts[k].tolist() == [int((hit & m).sum()), int(m.sum())], k
    # no masks: pred only
    counts0, pred0 = ops.eval_count(z, want_pred=True)
    assert counts0.numel() == 0 and torch.equal(pred0, pred)


# ---------------------------------------------------------------------------------------------------- helpers
def _reference_logits(g, model, dtype):
    """Rank 0's evaluation today: the model's eval branch on the whole graph."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    es = EvalSet(g, "cuda", inductive=False, dtype=dtype)
    return _logits(model, es.val), es


def _scatter(layouts, logits, n):
    out = torch.full((n, logits[0].shape[1]), float("nan"), device="cuda")
    for lay, z in zip(layouts, logits):
        out[lay.inner_gid.to("cuda")] = z.float()
    return out


def _near_ties(ref, tol):
    top = torch.topk(ref, min(2, ref.shape[1]), dim=1).values
    if ref.shape[1] == 1:
        return torch.zeros(ref.shape[0], dtype=torch.bool, device=ref.device)
    return (top[:, 0] - top[:, 1]) < tol


def _check_acc(got_acc, ref, label, mask, tol):
    """The partitioned accuracy equals calc_acc on the reference logits except for rows whose top-2 margin is within
    the tolerance: at most that many rows may flip."""
    n = int(mask.sum())
    if n == 0:
        assert got_acc != got_acc
        return
    ref_correct = int((ref[mask].argmax(1) == label[mask]).sum())
    slack = int((_near_ties(ref, tol) & mask).sum())
    assert abs(round(got_acc * n) - ref_correct) <= slack, (got_acc * n, ref_correct, slack)


def _bf16_close(got, ref):
    scale = ref.abs().max().item()
    torch.testing.assert_close(got, ref, rtol=2e-2, atol=1e-2 * scale)


def _train(trainer, n):
    for _ in range(n):
        trainer.run_epoch()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("use_pp", [False, True])
@pytest.mark.parametrize("method", ["random", "metis"])
@pytest.mark.parametrize("n_parts", [1, 2, 3, 4])
def test_partitioned_logits_match_full_graph(n_parts, method, use_pp, dtype):
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args
    g = make_graph("small")
    if method == "random":
        part = random_partition(g.n_nodes, n_parts)
    else:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    layouts = build_layouts(g, part, n_parts)
    _, args = make_args(g, 16, n_layers=3, n_hidden=32, n_linear=1, use_pp=use_pp, dropout=0.3,
                        enable_pipeline=True, feat_corr=True)
    args.dtype = dtype
    trainer = LocalTrainer(layouts, args, LocalWorld(n_parts, "cuda"))
    _train(trainer, 3)
    logits = trainer.predict()
    model = trainer.engines[0].model
    assert model.training                                    # predict leaves the mode as it found it
    ref, es = _reference_logits(g, model, trainer.engines[0].dtype)
    got = _scatter(layouts, logits, g.n_nodes)
    assert not torch.isnan(got).any()
    if dtype == "fp32":
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
        tol = 4e-4
    else:
        _bf16_close(got, ref)
        tol = 2e-2 * ref.abs().max().item()
    val_acc, test_acc = trainer.evaluate()
    label = es.val["label"]
    _check_acc(val_acc, ref, label, es.val["val_mask"], tol)
    _check_acc(test_acc, ref, label, es.val["test_mask"], tol)
    for e in trainer.engines:
        e.buffer.check_status()
    trainer.release_eval()


def test_shared_model_keeps_its_mode_and_evaluates_in_eval_mode():
    """One model shared by all ranks of a LocalWorld (P = 3, --norm batch, in train mode): the logits are those of
    each rank's own identical replica, and the model comes back in train mode."""
    from pipegcn_b200.train import LocalTrainer, create_model
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, _ = small_world("small", 3)
    _, args = make_args(g, 16, n_layers=3, n_hidden=32, norm="batch", enable_pipeline=True)
    trainer = LocalTrainer(layouts, args, LocalWorld(3, "cuda"))
    state = trainer.engines[0].model.state_dict()
    gen = torch.Generator(device="cuda").manual_seed(5)
    for k in state:                                          # running statistics far from (0, 1)
        if k.endswith("running_mean"):
            state[k] = torch.randn(state[k].shape, generator=gen, device="cuda")
        elif k.endswith("running_var"):
            state[k] = torch.rand(state[k].shape, generator=gen, device="cuda") * 4 + 0.5
    for e in trainer.engines:
        e.model.load_state_dict(state)
    shared = create_model(trainer.engines[0].layer_size, args, buffer=trainer.engines[0].buffer).cuda()
    shared.load_state_dict(state)
    shared.train()
    own = trainer.predict()
    assert all(e.model.training for e in trainer.engines)
    got = trainer.predict(model=shared)
    assert shared.training
    for a, b in zip(own, got):
        assert torch.equal(a, b)
    trainer.release_eval()


def test_layer0_halo_follows_new_features_without_static_layer0():
    """Without the static layer-0 store the training heap keeps no raw halo rows: every evaluation exchanges the
    current features' halo rows, so new features (set_features) are evaluated as they are."""
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, _ = small_world("small", 3)
    _, args = make_args(g, 16, n_hidden=32, enable_pipeline=True)
    args.static_layer0 = False
    trainer = LocalTrainer(layouts, args, LocalWorld(3, "cuda"))
    model = trainer.engines[0].model
    for step in range(2):
        if step:
            g.feat = torch.randn(g.feat.shape, generator=torch.Generator().manual_seed(9))
            for e, lay in zip(trainer.engines, layouts):
                e.set_features(g.feat[lay.inner_gid].cuda())
        got = _scatter(layouts, trainer.predict(), g.n_nodes)
        ref, _ = _reference_logits(g, model, torch.float32)
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
    trainer.release_eval()


# ---------------------------------------------------------------------------------------------------- no interference
def _six_epochs(layouts, args, evals, graph=False):
    from pipegcn_b200 import ops
    from pipegcn_b200.train import LocalTrainer, RankEngine
    from pipegcn_b200.world import LocalWorld
    ops._dropout_calls = 0
    ops.STEP_DEV = None                                      # left behind by an earlier capture
    torch.manual_seed(7)
    out = []
    if graph:
        args.cuda_graph = True
        eng = RankEngine(layouts[0], args, LocalWorld(1, "cuda").view(0), seg_len=32)
        eng.keep_logits = True
        for e in range(6):
            if e == 3:
                eng.capture()
            loss = eng.run_epoch()
            out.append(([float(loss.item())], [eng.last_logits.float().clone()]))
            if e in evals:
                eng.evaluate()
        params = [p.detach().clone() for p in eng.model.parameters()]
        eng.release_eval()
        return out, [params]
    trainer = LocalTrainer(layouts, args, LocalWorld(len(layouts), "cuda"))
    for e in range(6):
        losses = trainer.run_epoch(keep_logits=True)
        out.append(([float(l.item()) for l in losses], [en.last_logits.float().clone() for en in trainer.engines]))
        if e in evals:
            trainer.evaluate()
    params = [[p.detach().clone() for p in en.model.parameters()] for en in trainer.engines]
    trainer.release_eval()
    return out, params


@pytest.mark.parametrize("graph", [False, True])
def test_evaluation_does_not_disturb_training(graph):
    """Pipeline + feat-corr + grad-corr, dropout 0.5: six epochs with evaluations in between give the losses, logits
    and parameters of six epochs without, bit for bit.  Eager: P = 3, evaluations after epochs 2 and 4.  CUDA graphs:
    one rank (`LocalTrainer` does not capture), captured after the three eager epochs capture() needs and before the
    first evaluation, evaluations after epochs 4 and 5."""
    from tests.helpers import make_args, small_world
    n_parts = 1 if graph else 3
    g, _, layouts, _ = small_world("small", n_parts)
    runs = []
    for evals in ((), (3, 4) if graph else (1, 3)):
        _, args = make_args(g, 16, n_hidden=32, dropout=0.5, enable_pipeline=True, feat_corr=True, grad_corr=True)
        runs.append(_six_epochs(layouts, args, evals, graph))
    (a, pa), (b, pb) = runs
    for e, ((la, za), (lb, zb)) in enumerate(zip(a, b)):
        assert la == lb, e
        for x, y in zip(za, zb):
            assert torch.equal(x, y), e
    for ra, rb in zip(pa, pb):
        for x, y in zip(ra, rb):
            assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------- inductive
@pytest.mark.parametrize("use_pp", [False, True])
def test_inductive_matches_rank0(use_pp):
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.partition import build_eval_layout, build_layouts, extend_partition
    from pipegcn_b200.synthetic import make_graph, random_partition, train_subgraph
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args
    P = 3
    g = make_graph("small")
    gt = train_subgraph(g)
    tpart = random_partition(gt.n_nodes, P)
    layouts = build_layouts(gt, tpart, P)
    _, args = make_args(gt, 16, n_hidden=32, use_pp=use_pp, enable_pipeline=True)
    trainer = LocalTrainer(layouts, args, LocalWorld(P, "cuda"))
    _train(trainer, 3)
    part = extend_partition(g.train_mask, tpart, P)
    es = EvalSet(g, "cuda", inductive=True)
    model = trainer.engines[0].model
    for mode in ("val", "test"):
        keep = (g.train_mask | g.val_mask) if mode == "val" else None
        lays = [build_eval_layout(g, keep, part, P, r) for r in range(P)]
        val_acc, test_acc = trainer.evaluate(lays)
        ref = _logits(model, getattr(es, mode))
        got = _scatter(lays, trainer.predict(lays), ref.shape[0])
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
        part_ = getattr(es, mode)
        _check_acc(val_acc if mode == "val" else test_acc, ref, part_["label"], part_[mode + "_mask"], 4e-4)
        trainer.release_eval(lays)


# ---------------------------------------------------------------------------------------------------- trainer
def _roundtrip_args(**kw):
    base = dict(model="graphsage", backend="nccl", dtype="fp32", n_layers=2, n_hidden=32, n_linear=0, n_feat=24,
                n_class=4, n_train=0, dropout=0.1, norm="layer", lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=False,
                feat_corr=False, grad_corr=False, corr_momentum=0.95, seed=0, n_epochs=60, log_every=10,
                n_partitions=1, eval=True, inductive=False, dataset="synthetic:test", graph_name="roundtrip")
    base.update(kw)
    return argparse.Namespace(**base)


def test_trainer_eval_partitioned_roundtrip(tmp_path, monkeypatch, capsys):
    """train.run with --eval --eval-partitioned on planted labels: the result-file lines of today's rank-0 path, a
    checkpoint that loads strictly into the oracle's module tree, best validation accuracy above 0.6, and an eval
    heap of 2 * num_all * ld_max * s bytes + the flags."""
    import torch.nn.functional as F
    from oracle.model import OracleGraphSAGE
    from pipegcn_b200 import train
    from pipegcn_b200.helper import context as ctx
    from pipegcn_b200.helper.feature_buffer import Buffer
    from pipegcn_b200.helper.reducer import Reducer
    from pipegcn_b200.partition import build_layouts, get_layer_size
    from pipegcn_b200.synthetic import make_graph
    from pipegcn_b200.world import LocalWorld
    spec = dict(n_nodes=3_000, n_edges=30_000, n_feat=24, n_class=4, train_frac=0.6)
    g = make_graph(spec, planted_labels=True)
    layout = build_layouts(g, torch.zeros(g.n_nodes, dtype=torch.int64), 1)[0]
    texts = {}
    seen = []                                                # rank 0's logits at every evaluation
    from pipegcn_b200 import evaluate as evmod
    real_logits = evmod._logits

    def spy(model, part):
        z = real_logits(model, part)
        seen.append(z.clone())
        return z
    monkeypatch.setattr(evmod, "_logits", spy)
    for mode in ("rank0", "partitioned"):
        d = tmp_path / mode
        d.mkdir()
        monkeypatch.chdir(d)
        args = _roundtrip_args(n_train=int(g.train_mask.sum()))
        if mode == "partitioned":
            args.eval_partitioned = True
        world = LocalWorld(1, "cuda").view(0)
        ctx.buffer, ctx.reducer = Buffer(world), Reducer(world)
        from pipegcn_b200 import ops
        ops._dropout_calls, ops.STEP_DEV = 0, None                # both runs train the same weights
        eng = train.run(layout, args, world, eval_graph=g if mode == "rank0" else None)
        if mode == "rank0":
            seen.pop()                                       # the final test of the best model
        assert eng.checkpoint_path == "model/roundtrip_final.pth.tar"
        state = torch.load(d / eng.checkpoint_path)
        ref_model = OracleGraphSAGE(get_layer_size(24, 32, 4, 2), F.relu, False, norm="layer", dropout=0.1)
        ref_model.load_state_dict(state, strict=True)
        assert eng.best_val_acc > 0.6, eng.best_val_acc
        texts[mode] = (next((d / "results").iterdir()).name, next((d / "results").iterdir()).read_text())
        if mode == "partitioned":
            x = eng.last_eval_exchange
            ld_max = (max(24, 32) + 7) // 8 * 8                  # graph-layer inputs: 24 features, 32 hidden
            assert x.heap_bytes == 2 * layout.num_all * ld_max * 4 + x.flag_bytes
            assert x.flag_bytes == 256                           # [2][P] uint32 words, one 256-byte block
            assert eng._evals == {}                           # freed at the end of the run
    assert texts["rank0"][0] == texts["partitioned"][0]
    pat = re.compile(r"^Epoch (\d{5}) \| Validation Accuracy ([\d.]+)% \| Test Accuracy ([\d.]+)%$")
    la, lb = texts["rank0"][1].splitlines(), texts["partitioned"][1].splitlines()
    assert len(la) == len(lb) == len(seen) == 6
    masks = (g.val_mask.cuda(), g.test_mask.cuda())
    for x, y, ref in zip(la, lb, seen):
        mx, my = pat.match(x), pat.match(y)
        assert mx and my, (x, y)
        assert mx.group(1) == my.group(1)
        # one graph, one partition, the same weights: only the sum order of the aggregate differs (rows relabelled).
        # The near-tie rule of the parity tests: the correct counts may differ by at most the number of rows whose
        # top-2 margin in rank 0's logits is below the tolerance
        for k, m in enumerate(masks):
            n = int(m.sum())
            diff = round(abs(float(mx.group(2 + k)) - float(my.group(2 + k))) / 100 * n)
            assert diff <= int((_near_ties(ref, 4e-4) & m).sum()), (x, y)
    out = capsys.readouterr().out
    assert "Test Result | Accuracy" in out


# ---------------------------------------------------------------------------------------------------- two ranks
def _dist_main():
    """torchrun entry: both ranks evaluate the `tiny` graph partitioned; rank 0 compares with its full-graph eval."""
    import torch.distributed as dist
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import DistWorld
    from tests.helpers import make_args
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    g = make_graph("tiny")
    P = dist.get_world_size()
    layouts = build_layouts(g, random_partition(g.n_nodes, P), P)
    _, args = make_args(g, 5)
    eng = RankEngine(layouts[rank], args, DistWorld())
    # two back-to-back predictions with different weights: the second call's pushes must not overtake a peer's
    # reads of the first call
    from pipegcn_b200.train import create_model
    other = create_model(eng.layer_size, args, buffer=eng.buffer, dtype=eng.dtype).to(eng.device)
    other.load_state_dict(eng.model.state_dict())
    with torch.no_grad():
        for p in other.parameters():
            p.mul_(-0.5)
    logits_other = eng.predict(model=other)
    logits = eng.predict()
    val_acc, test_acc = eng.evaluate()
    got_other = [None] * P
    dist.all_gather_object(got_other, (layouts[rank].inner_gid, logits_other.cpu()))
    got = [None] * P
    dist.all_gather_object(got, (layouts[rank].inner_gid, logits.cpu()))
    ok = True
    if rank == 0:
        ref, es = _reference_logits(g, eng.model, torch.float32)
        full = torch.empty_like(ref)
        for gid, z in got:
            full[gid.cuda()] = z.cuda()
        ok = torch.allclose(full, ref, rtol=2e-4, atol=2e-4)
        ref_other, _ = _reference_logits(g, other, torch.float32)
        for gid, z in got_other:
            full[gid.cuda()] = z.cuda()
        ok = ok and torch.allclose(full, ref_other, rtol=2e-4, atol=2e-4)
        _check_acc(val_acc, ref, es.val["label"], es.val["val_mask"], 4e-4)
        _check_acc(test_acc, ref, es.val["label"], es.val["test_mask"], 4e-4)
    eng.release_eval()
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("ALL OK" if ok else "MISMATCH")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_ranks_match_rank0_eval():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29534", str(Path(__file__).resolve())]
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ALL OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]


if __name__ == "__main__":
    sys.path.insert(0, str(ROOT))
    _dist_main()
