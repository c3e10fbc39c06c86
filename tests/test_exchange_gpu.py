"""GPU parity of the halo exchange alone (no GEMM in the loop): `Buffer.update` and its backward replayed on
the oracle's own per-epoch inputs must reproduce the oracle's concatenated features and hooked gradients
BIT FOR BIT in fp32 -- same values, same EMA rounding (two roundings, no FMA), same peer order of the
boundary add -- in all four modes of PipeGCN/helper/feature_buffer.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = {
    "sync": dict(),
    "sync_corr": dict(feat_corr=True, grad_corr=True, corr_momentum=0.9),
    "pipeline": dict(enable_pipeline=True),
    "pipeline_corr": dict(enable_pipeline=True, feat_corr=True, grad_corr=True, corr_momentum=0.95),
}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n_parts,n_hidden", [(2, 16), (3, 16), (4, 16), (8, 16), (4, 37), (8, 37)],
                         ids=["2", "3", "4", "8", "4-h37", "8-h37"])
def test_buffer_replay_bit_exact(n_parts, n_hidden, mode):
    """P = 8 is the partition count the project is measured at (seven peers per push); a hidden width of 37 leaves
    a ragged last 16-byte vector in every row of the hidden layers."""
    from oracle.train import run_world
    from pipegcn_b200.helper.feature_buffer import Buffer
    from pipegcn_b200.helper.timer.comm_timer import CommTimer
    from pipegcn_b200.partition import get_layer_size
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import make_args, small_world

    g, _, layouts, setups = small_world("tiny", n_parts)
    n_epochs, n_layers = 4, 3
    oargs, _ = make_args(g, 5, n_epochs=n_epochs, n_layers=n_layers, n_hidden=n_hidden, **MODES[mode])
    traces = run_world(setups, oargs)
    layer_size = get_layer_size(g.n_feat, oargs.n_hidden, 5, n_layers)[:n_layers]

    streams = [torch.cuda.Stream() for _ in layouts]

    def make_bufs(pipeline):
        world = LocalWorld(n_parts, "cuda")
        out = []
        for r, lay in enumerate(layouts):
            b = Buffer(world.view(r))
            b.timer = CommTimer()
            b.timeout_ms = 5000
            b.init_buffer(lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, layer_size, pipeline=pipeline,
                          corr_feat=oargs.feat_corr, corr_grad=oargs.grad_corr, corr_momentum=oargs.corr_momentum)
            out.append(b)
        return out

    # host-side warm-up with throw-away pipelined buffers (never waits on unlaunched work): loads every
    # kernel and warms the allocator so that nothing synchronises the host while a flag-wait kernel spins
    dry = make_bufs(True)
    for e in range(2):
        keep = []
        for l in range(n_layers):
            for r, b in enumerate(dry):
                with torch.cuda.stream(streams[r]):
                    f = torch.zeros(layouts[r].num_in, layer_size[l], device="cuda", requires_grad=l > 0)
                    keep.append(b.update(l, f))
        for o in keep:
            if o.requires_grad:
                o.backward(torch.zeros_like(o))
        for b in dry:
            b.timer.clear()
            b.next_epoch()
    torch.cuda.synchronize()
    del dry, keep

    bufs = make_bufs(oargs.enable_pipeline)
    feats = {(e, r, l): traces[r].layers[e][l]["f_buf"][: layouts[r].num_in].to("cuda")
             for e in range(n_epochs) for r in range(n_parts) for l in range(n_layers)}
    gins = {(e, r, l): traces[r].hook_grads[(e, l)][0].to("cuda")
            for e in range(n_epochs) for r in range(n_parts) for l in range(1, n_layers)}
    torch.cuda.synchronize()

    for e in range(n_epochs):
        outs = {}
        for b in bufs:
            b.timer.clear()
        for l in range(n_layers):                      # forward, layer-major like the model loop
            for r, b in enumerate(bufs):
                with torch.cuda.stream(streams[r]):
                    feat = feats[(e, r, l)].requires_grad_(l > 0)
                    outs[(r, l)] = (feat, b.update(l, feat))
        torch.cuda.synchronize()
        for (r, l), (feat, out) in outs.items():
            assert torch.equal(out.detach().cpu(), traces[r].layers[e][l]["f_buf"]), (e, r, l)
        for l in range(n_layers - 1, 0, -1):           # backward, reversed layers like autograd
            for r, b in enumerate(bufs):
                with torch.cuda.stream(streams[r]):
                    outs[(r, l)][1].backward(gins[(e, r, l)])
        torch.cuda.synchronize()
        for r in range(n_parts):
            for l in range(1, n_layers):
                _, g_out = traces[r].hook_grads[(e, l)]
                got = outs[(r, l)][0].grad.cpu()
                assert torch.equal(got, g_out[: layouts[r].num_in]), (e, r, l)
        for b in bufs:
            b.next_epoch()
            b.check_status()


def test_update_rejects_wrong_shape_and_backend():
    from pipegcn_b200.helper.feature_buffer import Buffer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import small_world
    _, _, layouts, _ = small_world("tiny", 1)
    lay = layouts[0]
    b = Buffer(LocalWorld(1, "cuda").view(0))
    with pytest.raises(NotImplementedError):
        b.init_buffer(lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, [20, 16], backend="gloo")
    b.init_buffer(lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, [20, 16])
    with pytest.raises(ValueError):
        b.update(0, torch.zeros(lay.num_in, 7, device="cuda"))
    with pytest.raises(TypeError):
        b.update(0, torch.zeros(lay.num_in, 20, device="cuda", dtype=torch.bfloat16))
    out = b.update(0, torch.ones(lay.num_in, 20, device="cuda"))      # P=1: identity (feature_buffer.py:135)
    assert out.shape == (lay.num_all, 20) and bool((out == 1).all())
