"""Graph convolution (`--model graphconv`) on the GPU: `pg_aggregate_scaled` against fp64 on every dispatch path and
bit for bit against `pg_aggregate` where the scales reduce it to a mean, the halo rows' degrees from their owners, the
layer's autograd, full-graph equivalence of partitioned training, evaluation, checkpoints and CUDA-graph replay."""
import argparse

import pytest
import torch
import torch.nn.functional as F

from tests.test_kernel_conformance_gpu import AGG_IMPLS, DEV, _graph, _normal, knobs, x_with_nans

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24


def _scales(n, gen, lo=0.05, hi=1.0):
    return (lo + (hi - lo) * torch.rand(n, generator=gen)).to(DEV).contiguous()


def scaled_ref(indptr, indices, x, src, dst, bias=None):
    """fp64 dst[r] sum src[u] x[u] (+ bias) and the magnitude of its terms."""
    n_rows = indptr.numel() - 1
    lens = (indptr[1:] - indptr[:-1]).long()
    rows = torch.repeat_interleave(torch.arange(n_rows, device=DEV), lens)
    idx = indices.long()
    terms = src.double()[idx, None] * x.double()[idx]
    ref = torch.zeros(n_rows, x.shape[1], dtype=torch.float64, device=DEV).index_add_(0, rows, terms)
    mag = torch.zeros_like(ref).index_add_(0, rows, terms.abs())
    ref, mag = ref * dst.double()[:, None], mag * dst.double()[:, None]
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    return ref, mag, lens


def _guarded_out(n_rows, d, dtype):
    """An output view inside storage of sentinel bits: a guard row above and below, and the columns past the 16-byte
    vector that holds column d-1.  Returns the view and a check that the guard is untouched."""
    from tests.test_kernel_conformance_gpu import SENTINEL
    vec = 16 // torch.tensor([], dtype=dtype).element_size()
    dv = -(-d // vec) * vec
    ld = dv + 2 * vec
    itype = torch.int32 if dtype == torch.float32 else torch.int16
    base = torch.full(((n_rows + 2) * ld,), SENTINEL[dtype], dtype=itype, device=DEV)
    full = base.view(dtype)[ld:ld + n_rows * ld].view(n_rows, ld)
    out = full[:, :d]

    def check():
        rows = base.view(n_rows + 2, ld)
        assert torch.all(rows[0] == SENTINEL[dtype]) and torch.all(rows[-1] == SENTINEL[dtype])
        assert torch.all(rows[1:-1, dv:] == SENTINEL[dtype])
    return out, check


def _widths():
    return [(torch.float32, d) for d in (5, 8, 64, 256, 602)] + [(torch.bfloat16, d) for d in (8, 64, 256, 602)]


@pytest.mark.parametrize("impl,narrow", AGG_IMPLS)
@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("dtype,d", _widths())
@pytest.mark.parametrize("seg_len", [32, 512])
def test_aggregate_scaled_vs_fp64(impl, narrow, overlap, dtype, d, seg_len):
    """Empty rows, full 32-entry chunks, rows around seg_len, hubs and repeated ids (structured_csr), with and without
    a bias; NaN in row 0, the unreferenced rows and every pad column of x; a guard around the output."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(seg_len)
    gen = torch.Generator().manual_seed(d + seg_len)
    n_ref = 6000
    x = x_with_nans(n_ref + 50, n_ref, d, dtype, gen)
    src = _scales(n_ref + 50, gen)
    dst = _scales(plan.n_rows, gen)
    bias = _normal((d,), gen).to(DEV)
    with knobs(agg_impl=impl, agg_narrow=narrow, agg_overlap=overlap):
        for b in (None, bias):
            out, check_guard = _guarded_out(plan.n_rows, d, dtype)
            ops.aggregate_scaled(plan, x, src, dst, bias=b, out=out)
            check_guard()
            ref, mag, lens = scaled_ref(indptr, indices, x, src, dst, b)
            c = ((lens.double() + 13) * U24)[:, None]
            err = (out.double() - ref).abs()
            bound = c * mag + (ref.abs() * 2.0 ** -8 if dtype == torch.bfloat16 else 0)
            assert torch.all(err <= bound), f"max excess {float((err - bound).max())}"
            again = ops.aggregate_scaled(plan, x, src, dst, bias=b)
            assert torch.equal(out.view(torch.int32 if dtype == torch.float32 else torch.int16),
                               again.view(torch.int32 if dtype == torch.float32 else torch.int16))


@pytest.mark.parametrize("opts", [dict(agg_impl=2, agg_l2_hint=1), dict(agg_impl=3, agg_l2_hint=1),
                                  dict(agg_impl=1, agg_unroll=4), dict(agg_impl=2, agg_occ=5)])
@pytest.mark.parametrize("dtype,d", [(torch.float32, 64), (torch.float32, 602), (torch.bfloat16, 64),
                                     (torch.bfloat16, 256), (torch.bfloat16, 602)])
def test_aggregate_scaled_other_knobs(opts, dtype, d):
    """The L2-hint walkers, four rows in flight in the row-per-group kernel, and agg_occ 5 (which the scaled kernels
    do not use) against fp64, with a bias."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(32)
    gen = torch.Generator().manual_seed(d + 1)
    x = x_with_nans(6050, 6000, d, dtype, gen)
    src, dst = _scales(6050, gen), _scales(plan.n_rows, gen)
    bias = _normal((d,), gen).to(DEV)
    with knobs(**opts):
        out, check_guard = _guarded_out(plan.n_rows, d, dtype)
        ops.aggregate_scaled(plan, x, src, dst, bias=bias, out=out)
        check_guard()
    ref, mag, lens = scaled_ref(indptr, indices, x, src, dst, bias)
    err = (out.double() - ref).abs()
    bound = ((lens.double() + 13) * U24)[:, None] * mag + (ref.abs() * 2.0 ** -8 if dtype == torch.bfloat16 else 0)
    assert torch.all(err <= bound), f"max excess {float((err - bound).max())}"


@pytest.mark.parametrize("impl,narrow", AGG_IMPLS)
@pytest.mark.parametrize("dtype,d", [(torch.float32, 5), (torch.float32, 64), (torch.float32, 602),
                                     (torch.bfloat16, 8), (torch.bfloat16, 256)])
@pytest.mark.parametrize("seg_len", [32, 512])
def test_identity_with_pg_aggregate(impl, narrow, dtype, d, seg_len):
    """src = 1, dst = 1 / deg (IEEE division on the device), no bias: the bits of pg_aggregate(row_div=deg), and of
    pg_aggregate_drop under the same dropout key."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(seg_len)
    gen = torch.Generator().manual_seed(d)
    n_ref = 6000
    x = x_with_nans(n_ref + 50, n_ref, d, dtype, gen)
    deg = torch.clamp(indptr[1:] - indptr[:-1], min=1).float().contiguous()
    ones = torch.ones(n_ref + 50, device=DEV)
    inv = (1.0 / deg).contiguous()
    w = torch.int32 if dtype == torch.float32 else torch.int16
    with knobs(agg_impl=impl, agg_narrow=narrow):
        a = ops.aggregate(plan, x, row_div=deg)
        b = ops.aggregate_scaled(plan, x, ones, inv)
        assert torch.equal(a.view(w), b.view(w))
        spec = ops.DropSpec(0.5, 1234)
        a = ops.aggregate(plan, x, row_div=deg, drop=spec)
        b = ops.aggregate_scaled(plan, x, ones, inv, drop=spec)
        assert torch.equal(a.view(w), b.view(w))


def _small(n_parts, metis=False, shape="tiny"):
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph(shape, seed_graph=0)
    if metis:
        from pipegcn_b200.metis import metis_partition
        part = metis_partition(g, n_parts)
    else:
        part = random_partition(g.n_nodes, n_parts)
    return g, build_layouts(g, part, n_parts)


def _args(g, n_class, **kw):
    base = dict(model="graphconv", backend="nccl", dtype="fp32", n_layers=3, n_hidden=16, n_linear=0,
                n_feat=g.n_feat, n_class=n_class, n_train=int(g.train_mask.sum()), dropout=0.0, norm="layer",
                lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=False, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=4, log_every=10)
    base.update(kw)
    return argparse.Namespace(**base)


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_halo_norm_from_owners(n_parts, metis):
    """After set-up every rank's c holds deg^-1/2 of the global graph at inner_gid and halo_gid, bit for bit."""
    from pipegcn_b200 import ops
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(n_parts, metis)
    n_class = int(g.label.max()) + 1
    tr = LocalTrainer(lays, _args(g, n_class), LocalWorld(n_parts, DEV))
    c_glob = ops.sym_norm(g.in_degrees().to(DEV))
    for e, lay in zip(tr.engines, lays):
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long().to(DEV)
        assert torch.equal(e.graph.sym_norm(), c_glob[gid])


def _dense_gcn_logits(g, state, n_graph=3):
    """fp64 full-graph GraphConv forward with LayerNorm + ReLU between layers (eval, no dropout)."""
    n = g.n_nodes
    a = torch.zeros(n, n, dtype=torch.float64)
    a.index_put_((g.dst.long(), g.src.long()), torch.ones(g.src.numel(), dtype=torch.float64), accumulate=True)
    c = 1.0 / torch.clamp(g.in_degrees().double(), min=1).sqrt()
    a_hat = c[:, None] * a * c[None, :]
    h = g.feat.double()
    for i in range(n_graph):
        h = a_hat @ h @ state[f"layers.{i}.weight"].double().cpu() + state[f"layers.{i}.bias"].double().cpu()
        if i < n_graph - 1:
            h = torch.nn.functional.layer_norm(h, h.shape[1:], state[f"norm.{i}.weight"].double().cpu(),
                                               state[f"norm.{i}.bias"].double().cpu())
            h = torch.relu(h)
    return h


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [1, 2, 3, 4])
def test_full_graph_equivalence(n_parts, metis):
    """Synchronous training without dropout or corrections: every rank's logits and loss, and the reduced gradients,
    equal those of an fp64 full-graph GraphConv.  Halo rows scaled by their partition's CSC row lengths would not."""
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(n_parts, metis)
    n_class = int(g.label.max()) + 1
    tr = LocalTrainer(lays, _args(g, n_class), LocalWorld(n_parts, DEV))
    state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
    ref = _dense_gcn_logits(g, state)
    losses = tr.run_epoch(keep_logits=True)
    label = g.label.long()
    tm = g.train_mask
    total = 0.0
    for e, lay in zip(tr.engines, lays):
        gid = lay.inner_gid.long()
        torch.testing.assert_close(e.last_logits.double().cpu(), ref[gid], rtol=2e-4, atol=2e-4)
    ref_loss = torch.nn.functional.cross_entropy(ref[tm], label[tm], reduction="sum")
    total = sum(float(l.item()) for l in losses)
    assert abs(total - float(ref_loss)) <= 1e-4 * abs(float(ref_loss)) + 1e-3
    # reduced gradients: autograd of the fp64 restatement, one step of the same loss
    st = {k: v.double().cpu().requires_grad_(True) for k, v in state.items()}
    loss = torch.nn.functional.cross_entropy(_dense_gcn_logits(g, st)[tm], label[tm], reduction="sum") / tm.sum()
    loss.backward()
    got = tr.engines[0].model
    for name, p in got.named_parameters():
        if p.grad is not None and name in st and st[name].grad is not None:
            torch.testing.assert_close(p.grad.double().cpu(), st[name].grad, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize("mode", ["sync", "pipeline", "pipeline_corr"])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("extra", [dict(), dict(n_linear=1), dict(use_pp=True), dict(static_layer0=False),
                                   dict(halo_bits=8)])
def test_engine_trains(mode, dtype, extra):
    """The engine runs every exchange mode with GraphConv: finite losses that fall over a few epochs on 3 ranks."""
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(3)
    n_class = int(g.label.max()) + 1
    kw = dict(dtype=dtype, dropout=0.5, enable_pipeline=mode != "sync", feat_corr=mode == "pipeline_corr",
              grad_corr=mode == "pipeline_corr")
    kw.update(extra)
    tr = LocalTrainer(lays, _args(g, n_class, **kw), LocalWorld(3, DEV))
    first = None
    for _ in range(12):
        loss = sum(float(l.item()) for l in tr.run_epoch())
        assert loss == loss
        first = loss if first is None else first
    assert loss < first


def test_eval_paths_and_checkpoint(tmp_path):
    """Whole-graph and partitioned evaluation agree; a checkpoint loads strictly into a fresh GraphConv."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(2)
    n_class = int(g.label.max()) + 1
    tr = LocalTrainer(lays, _args(g, n_class, dropout=0.5), LocalWorld(2, DEV))
    for _ in range(3):
        tr.run_epoch()
    torch.cuda.synchronize()
    whole = _logits(tr.engines[0].model, EvalSet(g, DEV).val)
    parts = tr.predict()
    for z, lay in zip(parts, lays):
        torch.testing.assert_close(z.float(), whole[lay.inner_gid.long().to(DEV)], rtol=2e-4, atol=2e-4)
    tr.release_eval()
    path = tmp_path / "gc.pt"
    torch.save(tr.engines[0].model.state_dict(), path)
    from pipegcn_b200.train import create_model
    fresh = create_model(tr.engines[0].layer_size, _args(g, n_class))
    fresh.load_state_dict(torch.load(path), strict=True)


def _replay_runs(a, lay, capture_at=3, epochs=6):
    from pipegcn_b200 import ops
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    ops.STEP_DEV = None
    torch.manual_seed(0)
    eng = RankEngine(lay, a, LocalWorld(1, DEV).view(0), seg_len=32)
    eng.keep_logits = True
    rec = []
    for e in range(epochs):
        if capture_at is not None and e == capture_at:
            eng.capture()
        loss = eng.run_epoch()
        if e >= 3:
            rec.append((loss.clone(), eng.last_logits.clone(), [p.detach().clone() for p in eng.model.parameters()]))
    torch.cuda.synchronize()
    ops.STEP_DEV = None
    return rec


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_cuda_graph_replay_equals_eager_bit_for_bit(dtype):
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit.  No dropout:
    eager dropout keys its masks with a host call counter, a replayed epoch with the device epoch counter."""
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def test_learns_planted_labels():
    """16 planted classes (chance 1/16): validation accuracy after 60 pipelined epochs on 2 partitions."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g = make_graph("small", planted_labels=True)
    lays = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    tr = LocalTrainer(lays, _args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True), LocalWorld(2, DEV))
    for _ in range(60):
        tr.run_epoch()
    val, _ = tr.evaluate()
    tr.release_eval()
    print(f"graphconv planted-label validation accuracy {val:.4f}")
    assert val > 0.3, val


# ------------------------------------------------------------------------------------------------ layer autograd
def ref_gc_layer(x, w, b, rows, cols, num_in, c):
    """fp64 GraphConv over the edges cols -> rows: c_v sum_u c_u x_u @ W + b."""
    terms = c[cols, None] * x[cols]
    agg = torch.zeros(num_in, x.shape[1], dtype=x.dtype, device=x.device).index_add(0, rows, terms)
    return (c[:num_in, None] * agg) @ w + b


@pytest.mark.parametrize("drop", [0.0, 0.3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d_in,d_out", [(24, 40), (64, 64), (300, 40), (40, 300)])
def test_layer_autograd_matches_restatement(d_in, d_out, dtype, drop):
    """Both associations (d_in <= d_out aggregates first), hubs longer than seg_len in the CSR and the CSC, rows without
    in-edges; with drop_bwd the input gradient carries that key's mask (the CSC store, the GEMM epilogue, or for
    d_in > 256 the separate pass)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    from tests.test_gat_gpu import _edges
    from tests.test_sage_pool_gpu import _graph as _pool_graph
    g = _pool_graph()
    deg = torch.bincount(g.bwd.indices.long(), minlength=g.num_in)            # any positive per-row degrees
    c = ops.sym_norm(torch.cat([deg + 1, (g.bwd.indptr[1:] - g.bwd.indptr[:-1])[g.num_in:] + 3]))
    g.set_sym_norm(c)
    gen = torch.Generator(device=DEV).manual_seed(7)
    x = alloc_rows(g.num_all, d_in, dtype, DEV)
    x.copy_(torch.randn(g.num_all, d_in, generator=gen, device=DEV))
    w = torch.randn(d_in, d_out, generator=gen, device=DEV) * d_in ** -0.5
    b = torch.randn(d_out, generator=gen, device=DEV)
    up = torch.randn(g.num_in, d_out, generator=gen, device=DEV)
    spec = ops.DropSpec(drop, 1234) if drop > 0 else None

    def run():
        xs = x.detach().clone().requires_grad_(True)
        ws, bs = w.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
        o = ops.graphconv_layer(xs, g, g.sym_norm(), ws, bs, drop_bwd=spec)
        o.backward(up.to(dtype))
        return o.detach(), xs.grad, ws.grad, bs.grad

    r1, r2 = run(), run()
    assert all(torch.equal(p, q) for p, q in zip(r1, r2))
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    xr = x.double().requires_grad_(True)
    wr = w.to(dtype).double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    o_r = ref_gc_layer(xr, wr, br, rows, cols, g.num_in, c.double())
    o_r.backward(up.to(dtype).double())
    gx_ref = xr.grad
    if spec is not None:
        keep = ops.dropout_keep_host(spec, None, 0, g.num_all, d_in, x.element_size())
        gx_ref = gx_ref * torch.from_numpy(keep).to(DEV) / (1 - drop)
    tol = 1e-4 if dtype == torch.float32 else 3e-2

    def close(got, ref, what):
        err, scale = (got.double() - ref).abs().max().item(), ref.abs().max().item()
        assert err <= tol * scale + 1e-6, (what, err, scale)

    close(r1[0], o_r.detach(), "out")
    close(r1[1], gx_ref, "g_feat")
    close(r1[2], wr.grad, "dW")
    close(r1[3], br.grad, "db")


# ------------------------------------------------------------------------------------------------ engine restatement
def restate_training(g, layouts, state, a, dtype):
    """Partitioned GraphConv training in fp64: per rank the forward over its partition with the global graph's
    c = deg^-1/2 (with --use-pp, layer 0 on the precomputed c_v sum_u c_u x_u), loss and reduced gradients.  With bf16
    storage the weights, the transform-first product and the layer inputs are rounded where the engine stores them."""
    from tests.test_gat_gpu import _edges, _stored
    n = g.n_nodes
    c_glob = 1.0 / torch.clamp(g.in_degrees().to(DEV).double(), min=1).sqrt()
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=DEV)
    for lay in layouts:
        H[lay.inner_gid.to(DEV)] = lay.feat.to(DEV).to(dtype).double()
    gr = []
    for lay in layouts:
        rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long().to(DEV)
        gr.append(dict(gid=gid, rows=rows, cols=cols, inner=lay.inner_gid.long().to(DEV), num_in=lay.num_in,
                       c=c_glob[gid]))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                w, b = _stored(params[f"layers.{i}.weight"], dtype), params[f"layers.{i}.bias"]
                xu = _stored(H[q["gid"]], dtype)
                if i == 0 and a.use_pp:
                    terms = q["c"][q["cols"], None] * xu[q["cols"]]
                    agg = torch.zeros(q["num_in"], xu.shape[1], dtype=torch.float64, device=DEV).index_add(
                        0, q["rows"], terms)
                    out = _stored(q["c"][:q["num_in"], None] * agg, dtype) @ w + b
                elif w.shape[1] < w.shape[0]:                 # transform first: z is stored
                    z = _stored(xu @ w, dtype)
                    agg = torch.zeros(q["num_in"], z.shape[1], dtype=torch.float64, device=DEV).index_add(
                        0, q["rows"], q["c"][q["cols"], None] * z[q["cols"]])
                    out = q["c"][:q["num_in"], None] * agg + b
                else:
                    out = ref_gc_layer(xu, w, b, q["rows"], q["cols"], q["num_in"], q["c"])
                outs[r][i] = out
            else:
                out = H[q["inner"]] @ params[f"layers.{i}.weight"].T + params[f"layers.{i}.bias"]
            if i < n_layers - 1:
                out = F.relu(F.layer_norm(out, (out.shape[1],), params[f"norm.{i}.weight"], params[f"norm.{i}.bias"]))
            Hn = Hn.index_put((q["inner"],), out)
        H = Hn
    total, losses, logits = 0.0, [], []
    for lay, q in zip(layouts, gr):
        z = H[q["inner"]]
        logits.append(z)
        tm = lay.train_mask.to(DEV)
        loss = F.cross_entropy(z[tm], lay.label.to(DEV)[tm], reduction="sum")
        losses.append(loss)
        total = total + loss
    (total / a.n_train).backward()
    return outs, logits, losses, {k: p.grad for k, p in params.items()}


def _check_engine(g, tr, layouts, a, caps, state, losses, dtype):
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    outs, logits, ref_losses, grads = restate_training(g, layouts, state, a, tdt)
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
        else:
            for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
                got = got_logits if i == "logits" else caps[r][i].double()
                diff, scale = (got - ref.detach()).abs(), ref.detach().abs().max().item()
                assert diff.max().item() <= 0.25 * scale and diff.mean().item() <= 2e-2 * scale, (i, diff.max())
            ref_l = float(ref_losses[r].detach())
            assert abs(float(losses[r]) - ref_l) <= 2e-2 * abs(ref_l)
            for name, prm in eng.model.named_parameters():
                gref = grads[name]
                assert (prm.grad.double() - gref).norm() <= 0.25 * gref.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype, use_pp)
    (1, "random", True, 0, "fp32", False),
    (1, "random", False, 1, "bf16", True),
    (2, "random", True, 0, "fp32", True),
    (2, "metis", False, 1, "bf16", False),
    (3, "metis", False, 0, "fp32", False),
    (3, "random", True, 1, "fp32", True),
    (4, "metis", False, 1, "fp32", False),
    (4, "random", True, 0, "bf16", False),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype,use_pp", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype, use_pp):
    """Synchronous training, dropout 0, 3 epochs with the engine's weights; every halo row poisoned with NaN before
    each epoch.  Per-layer outputs, logits, losses and reduced gradients against the fp64 restatement (hidden 16 ->
    the last graph layer narrows 16 -> 5 and transforms first; with n_linear 1 both graph layers aggregate first)."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, 5, static_layer0=static0, n_linear=n_linear, dtype=dtype, use_pp=use_pp)
    tr = _trainer(layouts, a)
    caps = _hook_outputs(tr, a)
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        _check_engine(g, tr, layouts, a, caps, state, losses, dtype)


@pytest.mark.parametrize("mode", [dict(feat_corr=True, grad_corr=True), dict(enable_pipeline=True),
                                  dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8)])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_exchange_modes_layer_parity(mode, dtype):
    """P = 3, every exchange mode (--halo-bits 8 included): every graph layer's output and input gradient equal the
    fp64 layer applied to the rows the layer read (its own f_buf rows, the decoded messages where quantised) and the
    upstream gradient it received, with the global graph's c."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _edges
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _args(g, 5, static_layer0=False, dtype=dtype, **mode)
    if bits is not None:
        a.halo_bits = bits
    tr = _trainer(layouts, a)
    recs = [dict() for _ in tr.engines]

    def hook(mod, inp, out, r, i):
        rec = recs[r].setdefault(i, {})
        rec["x"], rec["out"] = inp[1].detach().clone(), out.detach().clone()
        rec.pop("gx", None)
        out.register_hook(lambda gr: rec.__setitem__("gout", gr.detach().clone()))
        if inp[1].requires_grad:
            inp[1].register_hook(lambda gr: rec.__setitem__("gx", gr.detach().clone()))

    n_graph = a.n_layers - a.n_linear
    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:n_graph]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: hook(mod, inp, out, r, i))
    c_glob = 1.0 / torch.clamp(g.in_degrees().to(DEV).double(), min=1).sqrt()
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    tol = 2e-4 if dtype == "fp32" else 3e-2
    n_checked = 0
    for _ in range(4):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        tr.run_epoch()
        torch.cuda.synchronize()
        for r, (eng, lay) in enumerate(zip(tr.engines, layouts)):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            c = c_glob[torch.cat([lay.inner_gid, lay.halo_gid]).long().to(DEV)]
            for i in range(n_graph):
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                w = state[f"layers.{i}.weight"].to(tdt).double()
                out = ref_gc_layer(x, w, state[f"layers.{i}.bias"], rows, cols, lay.num_in, c)
                scale = out.abs().max().item()
                assert (rec["out"].double() - out.detach()).abs().max().item() <= tol * scale + 1e-6, (r, i)
                out.backward(rec["gout"].double())
                if "gx" in rec:
                    gs = x.grad.abs().max().item()
                    assert (rec["gx"].double() - x.grad).abs().max().item() <= tol * gs + 1e-6, (r, i)
                    n_checked += 1
    assert n_checked > 0


# ------------------------------------------------------------------------------------------------ other layouts
@pytest.mark.parametrize("use_pp", [False, True])
def test_inductive_matches_rank0(use_pp):
    """--inductive evaluation layouts exchange their own graph's degrees: partitioned evaluation of the validation and
    the test graph equals whole-graph evaluation, whose norm comes from that graph's row degrees."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.partition import build_eval_layout, build_layouts, extend_partition
    from pipegcn_b200.synthetic import make_graph, random_partition, train_subgraph
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    from tests.test_gat_gpu import _scatter
    P = 3
    g = make_graph("small")
    gt = train_subgraph(g)
    tpart = random_partition(gt.n_nodes, P)
    layouts = build_layouts(gt, tpart, P)
    trainer = LocalTrainer(layouts, _args(gt, 16, n_hidden=32, use_pp=use_pp, enable_pipeline=True),
                           LocalWorld(P, DEV))
    for _ in range(3):
        trainer.run_epoch()
    torch.cuda.synchronize()
    part = extend_partition(g.train_mask, tpart, P)
    es = EvalSet(g, DEV, inductive=True)
    model = trainer.engines[0].model
    for mode in ("val", "test"):
        keep = (g.train_mask | g.val_mask) if mode == "val" else None
        lays = [build_eval_layout(g, keep, part, P, r) for r in range(P)]
        ref = _logits(model, getattr(es, mode))
        got = _scatter(lays, trainer.predict(lays), ref.shape[0])
        assert not torch.isnan(got).any()
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
        trainer.release_eval(lays)


def test_halo_norm_distgraph_layouts():
    """The per-rank distgraph layouts carry no global degrees: after set-up every halo row's c has the bits its owner
    computed for the same node, and every inner row's c is deg^-1/2 of its in-degree."""
    from pipegcn_b200 import ops
    from pipegcn_b200.distgraph import build_rank_layout
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    P = 3
    spec = dict(n_nodes=3_000, n_edges=30_000, n_feat=8, n_class=4, train_frac=0.5)
    lays = [build_rank_layout(spec, r, P, DEV)[0] for r in range(P)]
    a = _args(argparse.Namespace(n_feat=spec["n_feat"], train_mask=torch.cat([l.train_mask for l in lays])),
              spec["n_class"])
    tr = LocalTrainer(lays, a, LocalWorld(P, DEV))
    owner = torch.full((spec["n_nodes"],), float("nan"), device=DEV)
    for e, lay in zip(tr.engines, lays):
        c = e.graph.sym_norm()
        assert torch.equal(c[:lay.num_in], ops.sym_norm(lay.in_deg.to(DEV)))
        owner[lay.inner_gid.long().to(DEV)] = c[:lay.num_in]
    for e, lay in zip(tr.engines, lays):
        assert torch.equal(e.graph.sym_norm()[lay.num_in:], owner[lay.halo_gid.long().to(DEV)])
    assert all(lay.num_all > lay.num_in for lay in lays)
