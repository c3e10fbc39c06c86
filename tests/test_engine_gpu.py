"""GPU end-to-end parity: the CUDA engine (exchange + aggregate kernels through the C ABI) against the
CPU oracle on the same seeded graph, partition, weights and flags -- logits, loss, reduced gradients
and weights after every epoch, for the four exchange modes of the reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = {
    "sync": dict(),
    "sync_corr": dict(feat_corr=True, grad_corr=True, corr_momentum=0.9),
    "pipeline": dict(enable_pipeline=True),
    "pipeline_corr": dict(enable_pipeline=True, feat_corr=True, grad_corr=True, corr_momentum=0.95),
}


def _run_pair(n_parts, mode, n_epochs=4, shape="tiny", n_class=5, dtype="fp32", **extra):
    from oracle.train import initial_state, run_world
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, setups = small_world(shape, n_parts)
    oargs, eargs = make_args(g, n_class, n_epochs=n_epochs, **MODES[mode], **extra)
    eargs.dtype = dtype
    init = initial_state(oargs)
    traces = run_world(setups, oargs, init_state=init)
    trainer = LocalTrainer(layouts, eargs, LocalWorld(n_parts, "cuda"), init_state=init, seg_len=32)
    got = []
    for e in range(n_epochs):
        # teacher forcing: every epoch starts from the oracle's weights of that epoch.  Adam's first steps are
        # lr * sign(grad), so a gradient entry that is zero up to rounding sends free-running replicas apart by
        # 2 * lr; with forced weights every epoch compares the same function and the exchange history
        # (stale halo rows, EMA state) is still the engine's own.
        for eng in trainer.engines:
            eng.model.load_state_dict(traces[0].states[e])
        losses = trainer.run_epoch(keep_logits=True)
        got.append(dict(
            loss=[float(l.item()) for l in losses],
            logits=[e.last_logits.float().cpu() for e in trainer.engines],
            grads=[{n: p.grad.detach().float().cpu().clone() for n, p in e.model.named_parameters()}
                   for e in trainer.engines]))
    state = [{k: v.detach().float().cpu() for k, v in e.model.state_dict().items()} for e in trainer.engines]
    return traces, got, state


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n_parts", [1, 2, 3])
def test_engine_matches_oracle_fp32(n_parts, mode):
    # fp32 tolerance: per-layer outputs/logits rtol 2e-4 (sum order + cuBLAS vs MKL), loss rel 1e-4
    traces, got, state = _run_pair(n_parts, mode)
    for e, ep in enumerate(got):
        for r in range(n_parts):
            torch.testing.assert_close(ep["logits"][r], traces[r].logits[e], rtol=2e-4, atol=2e-4)
            assert abs(ep["loss"][r] - traces[r].losses[e]) <= 1e-4 * abs(traces[r].losses[e]) + 1e-4
            for n, gref in traces[r].grads[e].items():
                torch.testing.assert_close(ep["grads"][r][n], gref, rtol=2e-3, atol=2e-5)
    # weights after the last step, started from the same weights one epoch earlier (the optimizer state is the
    # engine's own): entries whose gradient is zero up to rounding may differ by the Adam step, 2 * lr
    for r in range(n_parts):
        for k, v in traces[r].state_dict.items():
            diff = (state[r][k] - v).abs()
            assert diff.max().item() <= 2.5e-2 and diff.mean().item() <= 2e-3, (k, diff.max(), diff.mean())


@pytest.mark.parametrize("mode", ["sync", "pipeline_corr"])
def test_engine_matches_oracle_bf16(mode):
    # bf16 storage (inputs, activations, gradients) with fp32 accumulation against the fp32 oracle:
    # logits within 2 % of their range on average (25 % at the worst element: LayerNorm over 16 channels
    # amplifies bf16 rounding on low-variance rows), loss within 2 %
    traces, got, _ = _run_pair(2, mode, n_epochs=3, dtype="bf16")
    for e, ep in enumerate(got):
        for r in range(2):
            diff = (ep["logits"][r] - traces[r].logits[e]).abs()
            scale = traces[r].logits[e].abs().max().item()
            assert diff.max().item() <= 0.25 * scale and diff.mean().item() <= 2e-2 * scale, (diff.max(), diff.mean())
            assert abs(ep["loss"][r] - traces[r].losses[e]) <= 2e-2 * abs(traces[r].losses[e])


@pytest.mark.parametrize("n_parts,mode", [(4, "pipeline_corr"), (2, "sync"), (3, "sync_corr"), (2, "pipeline")])
def test_engine_larger_graph(n_parts, mode):
    """20k-node RMAT, hubs above the segment length, messages of many CTAs."""
    traces, got, _ = _run_pair(n_parts, mode, n_epochs=3, shape="small", n_class=16, n_hidden=32)
    for e, ep in enumerate(got):
        for r in range(n_parts):
            torch.testing.assert_close(ep["logits"][r], traces[r].logits[e], rtol=1e-3, atol=1e-3)


def test_exposed_comm_timer_sections():
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, _ = small_world("tiny", 2)
    _, eargs = make_args(g, 5)
    eargs.static_layer0 = False
    trainer = LocalTrainer(layouts, eargs, LocalWorld(2, "cuda"))
    trainer.run_epoch()
    torch.cuda.synchronize()
    sec = trainer.engines[0].buffer.timer.sections()
    assert set(sec) == {"forward_0", "forward_1", "forward_2", "backward_1", "backward_2"}
    # with the static-layer-0 shortcut (default) layer 0 is exchanged once at set-up: no per-epoch wait
    _, eargs = make_args(g, 5)
    trainer2 = LocalTrainer(layouts, eargs, LocalWorld(2, "cuda"))
    trainer2.run_epoch()
    torch.cuda.synchronize()
    assert set(trainer2.engines[0].buffer.timer.sections()) == {"forward_1", "forward_2", "backward_1", "backward_2"}
    assert all(v >= 0 for v in sec.values())
    with pytest.raises(Exception):
        trainer.engines[0].buffer.timer.add_events("forward_0", None, None)   # duplicate name, as the reference


@pytest.mark.parametrize("static0", [True, False])
@pytest.mark.parametrize("name", ["ref_sync_p2.pt", "ref_sync_corr_p2.pt", "ref_pipeline_p2.pt", "ref_pipeline_corr_p3.pt",
                                  "ref_pipeline_pp_p2.pt"])
def test_engine_matches_reference_golden(name, static0):
    """The CUDA engine against the committed outputs of the unmodified reference (tests/golden): per-layer inputs
    and outputs, logits, loss, reduced gradients; fp32, teacher-forced weights.  Tolerances: exchange/aggregate
    outputs rtol 1e-5 (sum order), layer outputs/logits 2e-4 (3xTF32 tensor-core product), gradients 2e-3."""
    from tests.test_golden_cpu import load
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args
    fx, g, part = load(name)
    c = fx["config"]
    P = c["n_parts"]
    layouts = build_layouts(g, part, P)
    _, eargs = make_args(g, c["n_class"], n_epochs=c["n_epochs"], n_layers=c["n_layers"], n_hidden=c["n_hidden"],
                         enable_pipeline=c.get("enable_pipeline", False), feat_corr=c.get("feat_corr", False),
                         grad_corr=c.get("grad_corr", False), corr_momentum=c.get("corr_momentum", 0.95),
                         use_pp=c.get("use_pp", False))
    eargs.static_layer0 = static0
    trainer = LocalTrainer(layouts, eargs, LocalWorld(P, "cuda"), init_state=fx["ranks"][0]["init_state"], seg_len=32)
    assert all(e.buffer.static0_ready == (static0 and not c.get("use_pp", False)) for e in trainer.engines)
    caps = [dict() for _ in range(P)]
    for r, eng in enumerate(trainer.engines):
        for i, layer in enumerate(eng.model.layers):
            def hook(mod, inp, out, r=r, i=i):
                caps[r][i] = ((inp[1] if len(inp) > 1 else inp[0]).detach(), out.detach())
            layer.register_forward_hook(hook)
    for e in range(c["n_epochs"]):
        for eng in trainer.engines:
            eng.model.load_state_dict(fx["ranks"][0]["epochs"][e]["state"])
        losses = trainer.run_epoch(keep_logits=True)
        for r, eng in enumerate(trainer.engines):
            ep = fx["ranks"][r]["epochs"][e]
            for i, rec in ep["layers"].items():
                if i == 0:        # pure exchange (+ EMA): no GEMM upstream
                    torch.testing.assert_close(caps[r][i][0].cpu(), rec["f_buf"], rtol=1e-5, atol=1e-6)
                torch.testing.assert_close(caps[r][i][0].cpu(), rec["f_buf"], rtol=2e-4, atol=2e-5)
                torch.testing.assert_close(caps[r][i][1].cpu(), rec["layer_out"], rtol=2e-4, atol=2e-4)
            torch.testing.assert_close(eng.last_logits.cpu(), ep["logits"], rtol=2e-4, atol=2e-4)
            assert abs(float(losses[r].item()) - ep["loss"]) <= 1e-4 * abs(ep["loss"])
            for n, p in eng.model.named_parameters():
                torch.testing.assert_close(p.grad.cpu(), ep["grads"][n], rtol=2e-3, atol=2e-5)


@pytest.mark.parametrize("mode", ["sync", "pipeline_corr"])
def test_cuda_graph_replay_equals_eager(mode):
    """Epochs replayed from captured CUDA graphs (device-side epoch counter, one graph per parity) produce what
    eagerly launched epochs produce: same oracle-forced weights, same logits and gradients."""
    from oracle.train import initial_state, run_world
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, setups = small_world("tiny", 1)
    n_epochs = 7
    oargs, eargs = make_args(g, 5, n_epochs=n_epochs, **MODES[mode])
    init = initial_state(oargs)
    traces = run_world(setups, oargs, init_state=init)
    eargs.cuda_graph = True
    eng = RankEngine(layouts[0], eargs, LocalWorld(1, "cuda").view(0), init_state=init, seg_len=32)
    eng.keep_logits = True
    for e in range(n_epochs):
        if e == 3:
            eng.capture()
            assert len(eng.graphs) == (2 if eargs.enable_pipeline else 1)
        eng.model.load_state_dict(traces[0].states[e])
        loss = eng.run_epoch()
        torch.testing.assert_close(eng.last_logits.float().cpu(), traces[0].logits[e], rtol=2e-4, atol=2e-4)
        assert abs(float(loss.item()) - traces[0].losses[e]) <= 1e-4 * abs(traces[0].losses[e])
        for n, p in eng.model.named_parameters():
            torch.testing.assert_close(p.grad.cpu(), traces[0].grads[e][n], rtol=2e-3, atol=2e-5)


@pytest.mark.parametrize("mode", ["sync", "pipeline_corr"])
def test_engine_with_empty_messages(mode):
    """A chain graph cut into three runs: ranks 0 and 2 share no edge, so their messages have zero rows (the flag
    is still published) and rank 1 borrows exactly one row from each neighbour."""
    from oracle import dglpart
    from oracle import setup as osetup
    from oracle.train import initial_state, run_world
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import GlobalGraph
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args
    n, P = 90, 3
    a = torch.arange(n - 1)
    loops = torch.arange(n)
    src, dst = torch.cat([a, a + 1, loops]), torch.cat([a + 1, a, loops])
    gen = torch.Generator().manual_seed(0)
    g = GlobalGraph(n, src, dst, torch.randn(n, 12, generator=gen), torch.randint(0, 4, (n,), generator=gen),
                    torch.rand(n, generator=gen) < 0.7)
    part = torch.arange(n) // (n // P)
    layouts = build_layouts(g, part, P)
    assert layouts[0].recv_shape[2] == 0 and layouts[0].boundary[2].numel() == 0 and layouts[1].recv_shape == [1, None, 1]
    setups = osetup.setup_world(dglpart.partition_graph(n, g.src, g.dst, part, P, g.feat, g.label, g.train_mask))
    oargs, eargs = make_args(g, 4, n_epochs=3, n_hidden=8, **MODES[mode])
    init = initial_state(oargs)
    traces = run_world(setups, oargs, init_state=init)
    trainer = LocalTrainer(layouts, eargs, LocalWorld(P, "cuda"), init_state=init)
    for e in range(3):
        for eng in trainer.engines:
            eng.model.load_state_dict(traces[0].states[e])
        losses = trainer.run_epoch(keep_logits=True)
        for r, eng in enumerate(trainer.engines):
            torch.testing.assert_close(eng.last_logits.cpu(), traces[r].logits[e], rtol=2e-4, atol=2e-4)
            assert abs(float(losses[r].item()) - traces[r].losses[e]) <= 1e-4 * abs(traces[r].losses[e]) + 1e-5


@pytest.mark.parametrize("p", [0.5, 0.3])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["sync_corr", "pipeline_corr"])
def test_fused_dropout_equals_separate_passes(mode, dtype, p):
    """--dropout 0.5 / 0.3 (1 / (1 - p) exact or not): the masks applied by the producers (LayerNorm epilogue, halo push with the receiver's key, transposed
    aggregate / GEMM output) are the masks separate [num_all, d] passes would apply under the same keys: logits and
    losses are bit-identical, gradients identical in fp32 (bf16: the fused store rounds once instead of twice)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, _ = small_world("small", 3)
    outs = []
    saved = ops.FUSED_DROPOUT
    try:
        for fused in (True, False):
            ops.FUSED_DROPOUT = fused
            ops._dropout_calls = 0          # layer 0 (static features) keeps the stand-alone pass, keyed by a call counter
            torch.manual_seed(123)
            _, eargs = make_args(g, 16, n_epochs=3, n_hidden=64, dropout=p, **MODES[mode])
            eargs.dtype = dtype
            trainer = LocalTrainer(layouts, eargs, LocalWorld(3, "cuda"))
            ep = []
            for _ in range(3):
                losses = trainer.run_epoch(keep_logits=True)
                ep.append(([float(l.item()) for l in losses], [e.last_logits.float().clone() for e in trainer.engines],
                           [[p.grad.detach().float().clone() for p in e.model.parameters()] for e in trainer.engines]))
            outs.append(ep)
    finally:
        ops.FUSED_DROPOUT = saved
    # epoch 0 starts from the same weights: the forward must agree BIT FOR BIT (same masks, same rounding points)
    (la, za, ga), (lb, zb, gb) = outs[0][0], outs[1][0]
    assert la == lb
    for r, (a, b) in enumerate(zip(za, zb)):
        assert torch.equal(a, b), f"epoch 0 rank {r}: logits differ by {(a - b).abs().max().item():.3e}"
    # gradients (and with them the later epochs of the free-running replicas): the fused stores round once where the
    # separate passes round twice (bf16), and agree to the last few ulps in fp32
    gtol = dict(rtol=1e-5, atol=1e-8) if dtype == "fp32" else None
    for e, ((la, za, ga), (lb, zb, gb)) in enumerate(zip(*outs)):
        for r, (ra, rb) in enumerate(zip(ga, gb)):
            for i, (a, b) in enumerate(zip(ra, rb)):
                if dtype == "fp32":
                    # epoch 0: last-ulp agreement; the free-running replicas then drift apart at the 1e-4 level
                    tol = (1e-4, 1e-6) if e == 0 else (1e-2, 1e-3)
                    assert torch.allclose(a, b, rtol=tol[0], atol=tol[1] * max(b.abs().max().item(), 1e-12)), \
                        f"epoch {e} rank {r} grad {i}: max diff {(a - b).abs().max().item():.3e} of {b.abs().max().item():.3e}"
                elif e == 0 or p == 0.5:
                    # 1 / (1 - p) = 2 commutes with the rounding: identical; otherwise one rounding against two
                    torch.testing.assert_close(a, b, rtol=5e-2, atol=2e-2 * max(b.abs().max().item(), 1e-6),
                                               msg=lambda m: f"epoch {e} rank {r} grad {i}: {m}")
                else:
                    # later epochs of free-running bf16 replicas: Adam turns last-bit gradient differences into
                    # lr-sized weight differences; only the scale is comparable
                    assert (a - b).abs().max().item() <= 0.5 * max(b.abs().max().item(), 1e-6), f"epoch {e} rank {r} grad {i}"
        for r, (a, b) in enumerate(zip(za, zb)):
            tol = 1e-4 if dtype == "fp32" else (5e-2 if (e == 0 or p == 0.5) else 0.25)
            assert (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1.0), f"epoch {e} rank {r} logits"


def test_keyed_dropout_statistics_and_row_offset():
    """pg_dropout_rows: the kept fraction is 1 - p, kept values are scaled by 1 / (1 - p), the mask of a row slice equals
    the slice of the mask (row0), and it changes with the step counter."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    x = alloc_rows(4096, 256, torch.float32, "cuda")
    x.fill_(1.0)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    spec = ops.DropSpec(0.3, 12345, step, 0)
    y = ops.dropout_rows(x, spec)
    kept = (y != 0).float().mean().item()
    assert abs(kept - 0.7) < 0.01 and torch.allclose(y[y != 0], torch.tensor(1 / 0.7, device="cuda"))
    part = ops.dropout_rows(x[1000:1500], spec, row0=1000)
    assert torch.equal(part, y[1000:1500])
    step.add_(1)
    assert not torch.equal(ops.dropout_rows(x, spec), y)
    assert torch.equal(ops.dropout_rows(x, spec.shifted(-1)), y)


def test_set_features_on_one_local_rank_with_static_layer0_raises():
    """One rank of a LocalWorld with P > 1 cannot re-exchange the static layer-0 halo rows on its own (its peers
    would never push): `set_features` raises before launching anything instead of waiting for the flag timeout."""
    from pipegcn_b200 import _C
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world
    g, _, layouts, _ = small_world("tiny", 2)
    _, eargs = make_args(g, 5)
    trainer = LocalTrainer(layouts, eargs, LocalWorld(2, "cuda"))
    eng = trainer.engines[0]
    assert eng.buffer.static0_ready
    launches = _C.LAUNCHES
    with pytest.raises(RuntimeError, match="static_layer0=False"):
        eng.set_features(layouts[0].feat.cuda())
    assert _C.LAUNCHES == launches
    eng.buffer.check_status()
