"""Boundary-node sampling (`--sampling-rate p`) on the GPU: the sample kernel against its host port, the sampled
exchange (kept rows bit for bit, unkept rows contribute nothing), the engine against a torch restatement of the sampled
graph, p = 1 as today's path, determinism, CUDA-graph replay of the sampled kernels, partitioned evaluation after
sampled training, and a two-rank torchrun run."""
import argparse
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def _layouts(shape, P, method="random"):
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph(shape)
    if method == "metis":
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, P)
    else:
        part = random_partition(g.n_nodes, P)
    return g, build_layouts(g, part, P)


def _trainer(layouts, args):
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    return LocalTrainer(layouts, args, LocalWorld(len(layouts), "cuda"), seg_len=32)


def _args(g, n_class=5, **kw):
    from tests.helpers import make_args
    static0 = kw.pop("static_layer0", True)
    rate = kw.pop("sampling_rate", None)
    _, a = make_args(g, n_class, **kw)
    a.static_layer0 = static0
    if rate is not None:
        a.sampling_rate = rate
    return a


# ------------------------------------------------------------------------------------------------ sample kernel
def test_sample_kernel_matches_host_port_and_recount():
    from pipegcn_b200 import ops
    g, layouts = _layouts("tiny", 3)
    tr = _trainer(layouts, _args(g, sampling_rate=0.5))
    for e in range(3):
        tr.run_epoch()
        torch.cuda.synchronize()
        for eng, lay in zip(tr.engines, layouts):
            buf = eng.buffer
            mask = buf.sample_mask().cpu().numpy()
            want = ops.bns_keep_host(ops.bns_seed(0), e, eng.rank, np.arange(lay.num_in, lay.num_all),
                                     ops.bns_threshold(0.5))
            assert np.array_equal(mask, want), (e, eng.rank)
            keep_u = torch.cat([torch.ones(lay.num_in, dtype=torch.bool), torch.from_numpy(mask)])
            rows = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
            deg = torch.zeros(lay.num_in).index_add_(0, rows, keep_u[lay.indices.long()].float())
            assert torch.equal(buf._bns_deg.cpu(), deg)
            assert 0.3 < mask.mean() < 0.7


# ------------------------------------------------------------------------------------------------ restatement
def _restate(layouts, masks, state, a, dtype):
    """Sampled-graph forward / loss / reduced gradients in float64 torch: rank r's graph is its partition without the
    edges whose source is an unkept halo row, the mean divides by the sampled in-degree.  Returns per-rank
    (per-graph-layer outputs, logits, loss) and the reduced gradients."""
    dev = "cuda"
    n = sum(l.num_in for l in layouts)
    params = {k: v.detach().to(dev, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=dev)
    for lay in layouts:
        H[lay.inner_gid.to(dev)] = lay.feat.to(dev).to(dtype).double()
    g = []
    for lay, m in zip(layouts, masks):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).to(dev)
        keep = torch.cat([torch.ones(lay.num_in, dtype=torch.bool, device=dev), m.to(dev)])
        rows = torch.repeat_interleave(torch.arange(lay.num_in, device=dev),
                                       (lay.indptr[1:] - lay.indptr[:-1]).long().to(dev))
        cols = lay.indices.long().to(dev)
        ek = keep[cols]
        deg = torch.zeros(lay.num_in, dtype=torch.float64, device=dev).index_add_(0, rows[ek], ek[ek].double())
        g.append(dict(gid=gid, keep=keep, rows=rows, cols=cols, ek=ek, deg=deg,
                      full_deg=lay.in_deg.to(dev).double(), inner=lay.inner_gid.to(dev)))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=dev)
        for r, gr in enumerate(g):
            if i < n_graph:
                if i == 0 and a.use_pp:
                    xu = H[gr["gid"]]          # the precompute: full graph, full degrees
                    agg = torch.zeros(len(gr["inner"]), xu.shape[1], dtype=torch.float64, device=dev)
                    agg = agg.index_add_(0, gr["rows"], xu[gr["cols"]]) / gr["full_deg"][:, None]
                    x = torch.cat([xu[:len(gr["inner"])], agg], 1)
                    if dtype == torch.bfloat16:
                        x = x.to(dtype).double()
                    out = x @ params[f"layers.{i}.linear.weight"].T + params[f"layers.{i}.linear.bias"]
                else:
                    xu = H[gr["gid"]] * gr["keep"][:, None]
                    e = gr["ek"]
                    agg = torch.zeros(len(gr["inner"]), xu.shape[1], dtype=torch.float64, device=dev)
                    agg = agg.index_add_(0, gr["rows"][e], xu[gr["cols"][e]]) / gr["deg"][:, None]
                    out = (xu[:len(gr["inner"])] @ params[f"layers.{i}.linear1.weight"].T
                           + params[f"layers.{i}.linear1.bias"]
                           + agg @ params[f"layers.{i}.linear2.weight"].T + params[f"layers.{i}.linear2.bias"])
                outs[r][i] = out
            else:
                out = H[gr["inner"]] @ params[f"layers.{i}.weight"].T + params[f"layers.{i}.bias"]
            if i < n_layers - 1:
                out = F.relu(F.layer_norm(out, (out.shape[1],), params[f"norm.{i}.weight"], params[f"norm.{i}.bias"]))
            Hn = Hn.index_put((gr["inner"],), out)
        H = Hn
    total, losses, logits = 0.0, [], []
    for r, (lay, gr) in enumerate(zip(layouts, g)):
        z = H[gr["inner"]]
        logits.append(z)
        tm = lay.train_mask.to(dev)
        loss = F.cross_entropy(z[tm], lay.label.to(dev)[tm], reduction="sum")
        losses.append(loss)
        total = total + loss
    (total / a.n_train).backward()
    grads = {k: p.grad for k, p in params.items()}
    return outs, logits, losses, grads


CASES = [  # (P, partition, static layer 0, use_pp, n_linear, dtype)
    (2, "random", True, False, 0, "fp32"),
    (3, "metis", False, False, 0, "fp32"),
    (4, "random", True, True, 0, "fp32"),
    (3, "random", True, False, 1, "fp32"),
    (4, "metis", False, False, 0, "fp32"),
    (2, "metis", False, True, 1, "bf16"),
    (4, "random", True, False, 0, "bf16"),
]


@pytest.mark.parametrize("p", [0.5, 0.1])
@pytest.mark.parametrize("P,method,static0,use_pp,n_linear,dtype", CASES)
def test_engine_matches_sampled_graph_restatement(P, method, static0, use_pp, n_linear, dtype, p):
    """Per graph layer, logits, loss and reduced gradients of the engine against the restatement, with the engine's
    masks, dropout 0 and the engine's weights of every epoch.  Layer 0 (20 -> 16 features) and the output layer
    (16 -> 5) narrow (transform-first), layer 1 (16 -> 16) does not.  Every halo row is poisoned with NaN before each
    epoch: an unkept row that leaked into a sum would show."""
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, sampling_rate=p, static_layer0=static0, use_pp=use_pp, n_linear=n_linear)
    a.dtype = dtype
    tr = _trainer(layouts, a)
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    caps = [dict() for _ in range(P)]
    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:a.n_layers - n_linear]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: caps[r].__setitem__(i, out.detach()))
    for epoch in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        for eng in tr.engines:
            buf = eng.buffer
            for (layer, v), rows in buf._f_buf.items():
                rows[buf._num_in:, :buf._layer_size[layer]] = float("nan")
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        masks = [eng.buffer.sample_mask() for eng in tr.engines]
        assert all(m is not None for m in masks)
        outs, logits, ref_losses, grads = _restate(layouts, masks, state, a, tdt)
        for r, eng in enumerate(tr.engines):
            got_logits = eng.last_logits.double()
            assert torch.isfinite(got_logits).all()
            if dtype == "fp32":
                for i, ref in outs[r].items():
                    torch.testing.assert_close(caps[r][i].double(), ref.detach(), rtol=2e-4, atol=2e-4)
                torch.testing.assert_close(got_logits, logits[r].detach(), rtol=2e-4, atol=2e-4)
                ref_l = float(ref_losses[r].detach())
                assert abs(float(losses[r]) - ref_l) <= 1e-4 * abs(ref_l) + 1e-4
                for name, prm in eng.model.named_parameters():
                    torch.testing.assert_close(prm.grad.double(), grads[name], rtol=2e-3, atol=2e-5)
            else:   # bf16 storage against fp64: the tolerances of test_engine_matches_oracle_bf16 (25 % at the worst)
                for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
                    got = got_logits if i == "logits" else caps[r][i].double()
                    diff, scale = (got - ref.detach()).abs(), ref.detach().abs().max().item()
                    assert diff.max().item() <= 0.25 * scale and diff.mean().item() <= 2e-2 * scale, (i, diff.max())
                ref_l = float(ref_losses[r].detach())
                assert abs(float(losses[r]) - ref_l) <= 2e-2 * abs(ref_l)
                for name, prm in eng.model.named_parameters():
                    gr = grads[name]
                    assert (prm.grad.double() - gr).norm() <= 0.25 * gr.norm() + 1e-6, name


def test_kept_rows_bit_exact_unkept_zero_and_owner_gradient():
    """P = 3, one sampled epoch: the kept halo rows of layer 1 are the owners' rows bit for bit, the unkept rows are
    zero; the owners' boundary add summed exactly the gradient rows of the kept copies."""
    g, layouts = _layouts("tiny", 3)
    tr = _trainer(layouts, _args(g, sampling_rate=0.5, static_layer0=False))
    for eng in tr.engines:
        buf = eng.buffer
        buf._f_buf[(1, 0)][buf._num_in:] = float("nan")
    tr.run_epoch()
    torch.cuda.synchronize()
    engs = tr.engines
    n_rows = 0
    for r, eng in enumerate(engs):
        buf, mask = eng.buffer, eng.buffer.sample_mask()
        d = buf._layer_size[1]
        halo = buf._f_buf[(1, 0)][buf._num_in:, :d]
        assert torch.equal(halo[~mask], torch.zeros_like(halo[~mask]))
        for j in buf._peers:
            owner = engs[j].buffer
            lo, hi = buf._pl[j] - buf._num_in, buf._pl[j] - buf._num_in + buf._recv_shape[j]
            sent = owner._f_buf[(1, 0)][owner._bidx[r].long(), :d]
            m = mask[lo:hi]
            assert torch.equal(halo[lo:hi][m].view(torch.int32 if halo.dtype == torch.float32 else torch.int16),
                               sent[m].view(torch.int32 if halo.dtype == torch.float32 else torch.int16))
            n_rows += int(m.sum())
    assert n_rows > 0


def test_owner_boundary_add_sums_kept_rows_only():
    """The gradient exchange of one layer by hand at P = 3: every rank pushes known gradient rows for its halo rows;
    each owner's gradient gains exactly the rows of the copies its peers kept."""
    from pipegcn_b200.helper.feature_buffer import Buffer
    from pipegcn_b200.helper.timer.comm_timer import CommTimer
    from pipegcn_b200.train import _lockstep
    from pipegcn_b200.world import LocalWorld
    g, layouts = _layouts("tiny", 3)
    P = 3
    world = LocalWorld(P, "cuda")
    bufs, streams = [], [torch.cuda.Stream() for _ in range(P)]
    for r, lay in enumerate(layouts):
        b = Buffer(world.view(r))
        b.timer = CommTimer()
        b.init_buffer(lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, [8, 8], sampling_rate=0.5,
                      sampling_seed=7)
        bufs.append(b)
    plans = []
    for lay in layouts:
        from pipegcn_b200.graph import PartGraph
        plans.append(PartGraph.from_layout(lay, device="cuda"))
    for b in bufs:
        b._connect()
    grads = [torch.randn(lay.num_all, 8, device="cuda") for lay in layouts]
    for b, pg in zip(bufs, plans):
        b.sample(pg.fwd)
    outs = [None] * P

    def step(r):
        b = bufs[r]
        b._push_bns(b._bwd_msgs[(1, 0)], b._bns_bwd_keys, grads[r], 8, 1)
        yield "push"
        out = grads[r].clone()
        b._wait_flags(1, 1, 1, "backward_1")
        b._boundary_add(1, 0, out)
        outs[r] = out
    _lockstep([step(r) for r in range(P)], streams)
    torch.cuda.synchronize()
    for r, lay in enumerate(layouts):
        want = grads[r].clone()
        for j in bufs[r]._peers:
            mj = bufs[j].sample_mask()
            lo = bufs[j]._pl[r] - layouts[j].num_in
            rows = mj[lo:lo + layouts[j].recv_shape[r]]
            src = grads[j][bufs[j]._pl[r]:bufs[j]._pl[r] + layouts[j].recv_shape[r]]
            want.index_add_(0, lay.boundary[j].cuda()[rows], src[rows])
        torch.testing.assert_close(outs[r][:lay.num_in], want[:lay.num_in], rtol=1e-5, atol=1e-5)
    for b in bufs:
        b.check_status()
        b.release()


# ------------------------------------------------------------------------------------------------ today's path
def _fresh_dropout_counter():
    """Layer 0's dropout seeds count the calls of the process (`ops.dropout`): two trainers in one process see the
    same masks only from the same count."""
    from pipegcn_b200 import ops
    ops._dropout_calls = 0


def test_rate_one_is_todays_path():
    from pipegcn_b200 import _C
    g, layouts = _layouts("tiny", 3)
    runs = []
    for rate in (None, 1.0):
        _fresh_dropout_counter()
        tr = _trainer(layouts, _args(g, sampling_rate=rate, dropout=0.5))
        assert not any(e.buffer.sampling for e in tr.engines)
        n0 = _C.LAUNCHES
        losses = [[l.clone() for l in tr.run_epoch(keep_logits=True)] for _ in range(3)]
        logits = [e.last_logits.clone() for e in tr.engines]
        torch.cuda.synchronize()
        runs.append((_C.LAUNCHES - n0, losses, logits))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(runs[0][2], runs[1][2]))


def test_free_running_sampled_training_is_deterministic():
    g, layouts = _layouts("tiny", 3)
    runs = []
    for _ in range(2):
        _fresh_dropout_counter()
        tr = _trainer(layouts, _args(g, sampling_rate=0.3, dropout=0.5))
        runs.append([float(l) for _ in range(10) for l in tr.run_epoch()])
    assert runs[0] == runs[1]
    assert all(math.isfinite(x) for x in runs[0])


# ------------------------------------------------------------------------------------------------ CUDA graphs
def test_captured_sampled_kernels_replay_like_eager_launches():
    """pg_bns_sample, pg_halo_push_bns and pg_boundary_add_bns captured once with the device epoch counter and replayed
    for epochs 0..4 equal eager launches with host epochs."""
    import ctypes as C
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.graph import CsrPlan
    from pipegcn_b200.helper.feature_buffer import _MsgSet
    torch.manual_seed(3)
    dev = "cuda"
    num_in, num_all, d = 300, 700, 24
    deg = torch.randint(1, 9, (num_in,))
    indptr = torch.zeros(num_in + 1, dtype=torch.int32)
    indptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    indices = torch.randint(0, num_all, (int(indptr[-1]),), dtype=torch.int32)
    plan = CsrPlan(indptr.to(dev), indices.to(dev))
    src = torch.randn(num_all, 32, device=dev)
    idx = torch.randint(0, num_all, (200,), dtype=torch.int32, device=dev)
    keys = torch.tensor([[2, 500], [1, num_in]], dtype=torch.int32, device=dev)
    n_urow = 150
    urow = torch.randperm(num_in, device=dev)[:n_urow].to(torch.int32)
    uptr = torch.arange(0, 2 * n_urow + 1, 2, dtype=torch.int32, device=dev)
    usrc = torch.randperm(2 * n_urow, device=dev).to(torch.int32)
    slot_keys = torch.stack([torch.randint(0, 4, (2 * n_urow,)), torch.randint(0, 10000, (2 * n_urow,))], 1)
    slot_keys = slot_keys.to(torch.int32).to(dev).contiguous()
    recv = torch.randn(2 * n_urow, 32, device=dev)
    mask = torch.zeros(num_all - num_in, dtype=torch.uint8, device=dev)
    sdeg = torch.zeros(num_in, device=dev)
    dst = torch.zeros(400, 32, device=dev)
    grad = torch.zeros(num_in, 32, device=dev)
    base = torch.randn(num_in, 32, device=dev)
    ms = _MsgSet([_C.pg_msg(idx.data_ptr(), 0, 200, 0, dst.data_ptr(), 32, None, 0, None, None, 500),
                  _C.pg_msg(None, num_in, 200, 0, dst[200:].data_ptr(), 32, None, 0, None, None, 0)], dev)
    epoch_dev = torch.zeros(1, dtype=torch.int32, device=dev)

    def launch(spec):
        ops.bns_sample(spec, 1, plan, num_in, num_all, mask, sdeg)
        dst.fill_(-1.0)
        _C.check(_C.lib.pg_halo_push_bns(ms.ptr, ms.n_msgs, ms.n_ctas, keys.data_ptr(), src.data_ptr(), 32, d,
                                         _C.PG_F32, 1, None, None, C.byref(spec.c()), _C.stream_ptr()))
        grad.copy_(base)
        _C.check(_C.lib.pg_boundary_add_bns(grad.data_ptr(), 32, recv.data_ptr(), 32, d, _C.PG_F32, urow.data_ptr(),
                                            uptr.data_ptr(), usrc.data_ptr(), n_urow, slot_keys.data_ptr(),
                                            C.byref(spec.c()), _C.stream_ptr()))
        return [t.clone() for t in (mask, sdeg, dst, grad)]

    eager = []
    for t in range(5):
        eager.append(launch(ops.BnsSpec(0.4, 99, t)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        launch(ops.BnsSpec(0.4, 99, 0, epoch_dev))         # warm-up outside the capture
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):
            outs = launch(ops.BnsSpec(0.4, 99, 0, epoch_dev))
    torch.cuda.synchronize()
    for t in range(5):
        epoch_dev.fill_(t)
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(outs, eager[t]):
            assert torch.equal(a, b), t
    # the eager results themselves: the sample varies with the epoch, unkept pushed rows are not written
    assert not torch.equal(eager[0][0], eager[1][0])
    want = ops.bns_keep_host(99, 2, 2, 500 + np.arange(200), ops.bns_threshold(0.4))
    kept = torch.from_numpy(want).to(dev)
    assert torch.equal(eager[2][2][:200][kept][:, :d], src[idx.long()][kept][:, :d])
    assert bool((eager[2][2][:200][~kept] == -1).all())


# ------------------------------------------------------------------------------------------------ evaluation
def test_partitioned_evaluation_after_sampled_training():
    """Evaluation is never sampled: after sampled epochs the partitioned logits equal rank 0's full-graph ones."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    g, layouts = _layouts("tiny", 3)
    tr = _trainer(layouts, _args(g, sampling_rate=0.3, dropout=0.5))
    for _ in range(3):
        tr.run_epoch()
    got = tr.predict()
    model = tr.engines[0].model
    ref = _logits(model, EvalSet(g, "cuda", inductive=False, dtype=torch.float32).val)
    for lay, z in zip(layouts, got):
        torch.testing.assert_close(z.float(), ref[lay.inner_gid.to("cuda")].float(), rtol=2e-4, atol=2e-4)
    tr.release_eval()


# ------------------------------------------------------------------------------------------------ torchrun
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_ranks_sampled_training_runs():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29537", str(ROOT / "tools" / "bns_bench.py"),
           "--shapes", "tiny", "--rates", "1", "0.5", "--epochs", "3", "--warmup", "1", "--check"]
    p = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "BNS CHECK OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
