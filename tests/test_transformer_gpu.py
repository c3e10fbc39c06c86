"""Graph transformer (`--model transformer`) on the GPU: the TransformerConv kernels and the layer against the fp64
restatement of tests/test_transformer_cpu.py (whose backward formulas are pinned to torch.autograd there), the engine
against a restatement of partitioned training (partitions, exchange modes, boundary-node sampling, quantised halos),
evaluation, checkpoints, CUDA-graph replay and free-running training."""

import pytest
import torch
import torch.nn.functional as F

from tests.test_boundary_sampling_gpu import _layouts, _trainer
from tests.test_gat_gpu import (_close, _edges, _full_logits, _hook_outputs, _keep, _poison, _scatter, _stored,
                                _test_graph)
from tests.test_sage_pool_gpu import _graph as _pool_graph
from tests.test_transformer_cpu import ref_transformer

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ("lin_query.weight", "lin_query.bias", "lin_key.weight", "lin_key.bias", "lin_value.weight", "lin_value.bias",
        "lin_skip.weight", "lin_skip.bias")


def ref_layer(x, wq, bq, wk, bk, wv, bv, ws, bs, rows, cols, num_in, heads, keep=None, dtype=torch.float32):
    """fp64 TransformerConv over the edges cols -> rows of x [num_all, d_in]; an unkept source is absent.  With bf16
    storage the four projections are rounded where the engine stores them."""
    if keep is not None:
        ek = keep[cols]
        rows, cols = rows[ek], cols[ek]
    q = _stored(x[:num_in] @ wq.T + bq, dtype).view(num_in, heads, -1)
    k = _stored(x @ wk.T + bk, dtype).view(x.shape[0], heads, -1)
    v = _stored(x @ wv.T + bv, dtype).view(x.shape[0], heads, -1)
    skip = _stored(x[:num_in] @ ws.T + bs, dtype)
    return ref_transformer(q, k, v, skip, rows, cols, num_in)[0]


def _tensors(g, d_in, heads, d, dtype, seed=1):
    from pipegcn_b200.graph import alloc_rows
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = alloc_rows(g.num_all, d_in, dtype, DEV)
    x.copy_(torch.randn(g.num_all, d_in, generator=gen, device=DEV))
    params = []
    for _ in range(4):                                  # query, key, value, skip
        params += [torch.randn(heads * d, d_in, generator=gen, device=DEV) / d_in ** 0.5,
                   torch.randn(heads * d, generator=gen, device=DEV) * 0.1]
    up = torch.randn(g.num_in, heads * d, generator=gen, device=DEV)
    return x, params, up


def _nan_rows(n, hd, dtype):
    from pipegcn_b200.graph import alloc_rows
    return alloc_rows(n, hd, dtype, DEV).fill_(float("nan"))


def _check_kernels(g, heads, d, dtype, keep, keep_u, d_in=24):
    """The three passes on the engine's own projections (unkept k / v rows poisoned with NaN, every output buffer
    NaN-filled first) against the restatement and its autograd; returns the tensors for the layer check."""
    from pipegcn_b200 import ops
    x, params, up = _tensors(g, d_in, heads, d, dtype)
    wq, bq, wk, bk, wv, bv, ws, bs = params
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    x[~keep_u] = 0                      # the exchange leaves unkept halo rows zero
    n_in, hd = g.num_in, heads * d
    xs, xi = ops.presplit(x), ops.presplit(x[:g.num_in])
    q = ops.gemm_nt(xi, ops.padded_weight(wq, dtype), bias=bq)
    k = ops.gemm_nt(xs, ops.padded_weight(wk, dtype), bias=bk)
    v = ops.gemm_nt(xs, ops.padded_weight(wv, dtype), bias=bv)
    skip = ops.gemm_nt(xi, ops.padded_weight(ws, dtype), bias=bs)
    k[~keep_u] = float("nan")
    v[~keep_u] = float("nan")
    out, m, s = ops.transformer_aggregate(g, q, k, v, skip, heads, keep)
    out2, m2, s2 = ops.transformer_aggregate(g, q, k, v, skip, heads, keep)
    assert torch.equal(out, out2) and torch.equal(m, m2) and torch.equal(s, s2)
    ek = keep_u[cols]
    ql = q.double().view(n_in, heads, d).clone().requires_grad_(True)
    kl, vl = [t.double().view(g.num_all, heads, d).clone() for t in (k, v)]
    kl[~keep_u] = 0
    vl[~keep_u] = 0
    kl.requires_grad_(True)
    vl.requires_grad_(True)
    o_ref, m_ref, s_ref = ref_transformer(ql, kl, vl, skip.double(), rows[ek], cols[ek], n_in)
    torch.testing.assert_close(m.double(), m_ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(s.double(), s_ref, rtol=1e-5, atol=1e-5)
    _close(out, o_ref, dtype, "out", rel=1e-4 if dtype == torch.float32 else 1e-2)
    gu = up.to(dtype)
    dq, gc = _nan_rows(n_in, hd, dtype), _nan_rows(n_in, hd, dtype)
    dk, dv = _nan_rows(g.num_all, hd, dtype), _nan_rows(g.num_all, hd, dtype)
    _, _, delta = ops.transformer_bwd_dst(g, q, k, v, gu, m, s, heads, keep, dq=dq, gc=gc)
    ops.transformer_bwd_src(g, q, k, v, gu, m, s, delta, heads, keep, dk=dk, dv=dv)
    assert torch.equal(gc, gu)
    dk2, dv2 = ops.transformer_bwd_src(g, q, k, v, gu, m, s, delta, heads, keep)
    assert torch.equal(dk, dk2) and torch.equal(dv, dv2)
    o_ref.backward(gu.double())
    attn = (o_ref.detach() - skip.double()).view(n_in, heads, d)
    torch.testing.assert_close(delta.double(), (attn * gu.double().view(n_in, heads, d)).sum(-1),
                               rtol=1e-4, atol=1e-4 * max(1.0, float(delta.abs().max())))
    rel = 1e-4 if dtype == torch.float32 else 2e-2
    _close(dq, ql.grad.reshape(n_in, -1), dtype, "dq", rel=rel)
    for name, got, ref in (("dk", dk, kl.grad), ("dv", dv, vl.grad)):
        ref = ref.reshape(g.num_all, -1)
        _close(got[:n_in], ref[:n_in], dtype, name + " inner", rel=rel)
        _close(got[n_in:][keep_u[n_in:]], ref[n_in:][keep_u[n_in:]], dtype, name + " halo", rel=rel)
        assert torch.isfinite(got.float()).all(), name
        if keep is not None:
            assert torch.count_nonzero(got[~keep_u].float()) == 0, name
    return x, params, up


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 256])
@pytest.mark.parametrize("heads", [1, 2, 4, 8])
def test_kernels_and_layer_match_fp64_restatement(heads, d, dtype, masked):
    """Hub rows past seg_len (fix-ups), rows whose only edge is the self loop, a halo row with a long CSC row; at
    d = 5 the paired operands' halves are padded to 8 columns."""
    from pipegcn_b200 import ops
    g = _test_graph()
    keep, keep_u = _keep(g, masked)
    x, params, up = _check_kernels(g, heads, d, dtype, keep, keep_u)
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))

    def layer_run():
        xs = x.detach().clone().requires_grad_(True)
        ps = [t.detach().clone().requires_grad_(True) for t in params]
        o = ops.transformer_layer(xs, g, keep, heads, *ps)
        o.backward(up.to(dtype))
        return o.detach(), xs.grad, [p.grad for p in ps]

    o1, gx1, gp1 = layer_run()
    o2, gx2, gp2 = layer_run()
    assert torch.equal(o1, o2) and torch.equal(gx1, gx2) and all(torch.equal(a, b) for a, b in zip(gp1, gp2))

    xr = torch.where(keep_u[:, None], x.double(), torch.zeros((), dtype=torch.float64, device=DEV))
    xr = xr.requires_grad_(True)
    pr = [((t.to(dtype) if dtype == torch.bfloat16 and t.dim() == 2 else t).double()).requires_grad_(True)
          for t in params]
    o_r = ref_layer(xr, *pr, rows, cols, g.num_in, heads, keep_u, dtype)
    o_r.backward(up.double())
    _close(o1, o_r, dtype, "layer out", rel=2e-4 if dtype == torch.float32 else 3e-2)
    _close(gx1[keep_u], xr.grad[keep_u], dtype, "dh", rel=2e-4 if dtype == torch.float32 else 5e-2)
    if masked:
        assert torch.count_nonzero(gx1[~keep_u].float()) == 0
    for name, got, ref in zip(KEYS, gp1, [p.grad for p in pr]):
        _close(got, ref, dtype, name, rel=2e-4 if dtype == torch.float32 else 5e-2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernels_past_the_first_wave(dtype):
    """More CTAs than one wave can hold at any occupancy (16 resident 128-thread CTAs per SM), with long rows."""
    g = _pool_graph(num_in=120000, num_halo=20000, seed=1, max_deg=8)
    waves = 16 * torch.cuda.get_device_properties(0).multi_processor_count
    assert g.fwd.n_chunks // 4 > waves and g.bwd.n_chunks // 4 > waves
    keep, keep_u = _keep(g, True)
    _check_kernels(g, 4, 64, dtype, keep, keep_u)


def test_head_width_past_512_is_refused():
    from pipegcn_b200 import _C, ops
    g = _test_graph()
    q = torch.zeros(g.num_in, 513, device=DEV)
    k = torch.zeros(g.num_all, 513, device=DEV)
    with pytest.raises(_C.PgError, match="D must be in 1..512"):
        ops.transformer_aggregate(g, q, k, k, q, 1)


# ------------------------------------------------------------------------------------------------ engine
def _tc_args(g, n_class=5, **kw):
    from tests.test_boundary_sampling_gpu import _args
    heads = kw.pop("n_heads", 4)
    bits = kw.pop("halo_bits", None)
    a = _args(g, n_class, **kw)
    a.model, a.n_heads = "transformer", heads
    if bits is not None:
        a.halo_bits = bits
    return a


def restate_training(layouts, masks, state, a, dtype):
    """Partitioned graph-transformer training in fp64 (see test_gat_gpu.restate_training)."""
    n = sum(l.num_in for l in layouts)
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=DEV)
    for lay in layouts:
        H[lay.inner_gid.to(DEV)] = lay.feat.to(DEV).to(dtype).double()
    gr = []
    for r, lay in enumerate(layouts):
        keep = torch.ones(lay.num_all, dtype=torch.bool, device=DEV)
        if masks is not None:
            keep[lay.num_in:] = masks[r].to(DEV)
        rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
        gr.append(dict(gid=torch.cat([lay.inner_gid, lay.halo_gid]).to(DEV), keep=keep, rows=rows, cols=cols,
                       inner=lay.inner_gid.to(DEV), num_in=lay.num_in))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                p = [params[f"layers.{i}.{k}"] for k in KEYS]
                for j in (0, 2, 4, 6):
                    p[j] = _stored(p[j], dtype)
                heads = a.n_heads if i < n_layers - 1 else 1
                xu = _stored(H[q["gid"]], dtype) * q["keep"][:, None]
                out = ref_layer(xu, *p, q["rows"], q["cols"], q["num_in"], heads, q["keep"], dtype)
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


def _check_engine(tr, layouts, a, caps, masks, state, losses, dtype):
    """GATv2's tolerances (test_gatv2_gpu._check_engine)."""
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    outs, logits, ref_losses, grads = restate_training(layouts, masks, state, a, tdt)
    for r, eng in enumerate(tr.engines):
        got_logits = eng.last_logits.double()
        assert torch.isfinite(got_logits).all()
        ref_l = float(ref_losses[r].detach())
        if dtype == "fp32":
            for i, ref in outs[r].items():
                torch.testing.assert_close(caps[r][i].double(), ref.detach(), rtol=2e-4, atol=2e-4)
            torch.testing.assert_close(got_logits, logits[r].detach(), rtol=2e-4, atol=2e-4)
            assert abs(float(losses[r]) - ref_l) <= 1e-4 * abs(ref_l) + 1e-4
            for name, prm in eng.model.named_parameters():
                torch.testing.assert_close(prm.grad.double(), grads[name], rtol=2e-3, atol=2e-5, msg=name)
        else:
            for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
                got = got_logits if i == "logits" else caps[r][i].double()
                diff, scale = (got - ref.detach()).abs(), ref.detach().abs().max().item()
                assert diff.max().item() <= 0.25 * scale and diff.mean().item() <= 2e-2 * scale, (i, diff.max())
            assert abs(float(losses[r]) - ref_l) <= 2e-2 * abs(ref_l)
            for name, prm in eng.model.named_parameters():
                gr = grads[name]
                assert (prm.grad.double() - gr).norm() <= 0.25 * gr.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype)
    (1, "random", True, 0, "fp32"),
    (2, "random", True, 0, "fp32"),
    (3, "metis", False, 0, "fp32"),
    (3, "random", True, 1, "fp32"),
    (4, "metis", False, 0, "fp32"),
    (4, "random", True, 1, "fp32"),
    (2, "metis", False, 1, "bf16"),
    (4, "random", True, 0, "bf16"),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype):
    """Synchronous training, dropout 0, 3 epochs; every halo row poisoned with NaN before each epoch."""
    g, layouts = _layouts("tiny", P, method)
    a = _tc_args(g, static_layer0=static0, n_linear=n_linear)
    a.dtype = dtype
    tr = _trainer(layouts, a)
    caps = _hook_outputs(tr, a)
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        _check_engine(tr, layouts, a, caps, None, state, losses, dtype)


@pytest.mark.parametrize("p", [0.5, 0.1])
@pytest.mark.parametrize("P,method,static0,dtype", [(3, "random", True, "fp32"), (4, "metis", False, "fp32"),
                                                    (2, "random", True, "bf16")])
def test_sampled_engine_matches_restatement(P, method, static0, dtype, p):
    """Boundary-node sampling: unkept halo sources are absent from every softmax; unkept rows are NaN-poisoned."""
    g, layouts = _layouts("tiny", P, method)
    a = _tc_args(g, static_layer0=static0, sampling_rate=p)
    a.dtype = dtype
    tr = _trainer(layouts, a)
    caps = _hook_outputs(tr, a)
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        masks = [eng.buffer.sample_mask() for eng in tr.engines]
        assert all(m is not None for m in masks)
        _check_engine(tr, layouts, a, caps, masks, state, losses, dtype)


@pytest.mark.parametrize("mode", [dict(enable_pipeline=True), dict(enable_pipeline=True, feat_corr=True, grad_corr=True),
                                  dict(feat_corr=True, grad_corr=True), dict(halo_bits=8)])
def test_exchange_modes_layer_parity(mode):
    """P = 3: every layer's output and input gradient equal the restated layer applied to the [num_all] input the
    layer read (with --halo-bits 8 it holds the decoded halo rows) and the upstream gradient it received."""
    g, layouts = _layouts("tiny", 3)
    a = _tc_args(g, static_layer0=False, **mode)
    tr = _trainer(layouts, a)
    recs = [dict() for _ in tr.engines]

    def hook(mod, inp, out, r, i):
        rec = recs[r].setdefault(i, {})
        rec["x"], rec["out"] = inp[1].detach().clone(), out.detach().clone()
        rec.pop("gx", None)
        out.register_hook(lambda gr: rec.__setitem__("gout", gr.detach().clone()))
        if inp[1].requires_grad:
            inp[1].register_hook(lambda gr: rec.__setitem__("gx", gr.detach().clone()))

    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:a.n_layers]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: hook(mod, inp, out, r, i))
    n_checked = 0
    for _ in range(4):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        tr.run_epoch()
        torch.cuda.synchronize()
        for r, (eng, lay) in enumerate(zip(tr.engines, layouts)):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            for i, layer in enumerate(eng.model.layers[:a.n_layers]):
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                p = [state[f"layers.{i}.{k}"] for k in KEYS]
                out = ref_layer(x, *p, rows, cols, lay.num_in, layer.num_heads)
                torch.testing.assert_close(rec["out"].double(), out.detach(), rtol=2e-4, atol=2e-4)
                out.backward(rec["gout"].double())
                if "gx" in rec:
                    torch.testing.assert_close(rec["gx"].double(), x.grad, rtol=2e-4, atol=2e-5)
                    n_checked += 1
    assert n_checked > 0


# ------------------------------------------------------------------------------------------------ evaluation
def test_single_partition_logits_equal_full_graph_eval():
    from pipegcn_b200.train import create_model
    g, layouts = _layouts("tiny", 1)
    a = _tc_args(g)
    tr = _trainer(layouts, a)
    tr.run_epoch()
    eng = tr.engines[0]
    weights = create_model(eng.layer_size, a).to(DEV)       # the weights the next epoch's forward uses
    weights.load_state_dict(eng.model.state_dict())
    tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    got = _scatter(layouts, [eng.last_logits], g.n_nodes)
    ref = _full_logits(g, weights, eng.dtype)
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("P", [2, 4])
def test_partitioned_eval_equals_rank0(P):
    g, layouts = _layouts("small", P)
    a = _tc_args(g, 16, n_hidden=32, dropout=0.3, enable_pipeline=True)
    tr = _trainer(layouts, a)
    for _ in range(3):
        tr.run_epoch()
    torch.cuda.synchronize()
    got = _scatter(layouts, tr.predict(), g.n_nodes)
    ref = _full_logits(g, tr.engines[0].model, tr.engines[0].dtype)
    assert not torch.isnan(got).any()
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
    tr.release_eval()


def test_checkpoint_round_trip(tmp_path):
    from pipegcn_b200.module.model import GraphTransformer
    from pipegcn_b200.train import create_model
    g, layouts = _layouts("tiny", 2)
    a = _tc_args(g, n_linear=1)
    tr = _trainer(layouts, a)
    for _ in range(2):
        tr.run_epoch()
    torch.cuda.synchronize()
    model = tr.engines[0].model
    path = tmp_path / "transformer.pth.tar"
    saved = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    assert {k.split(".", 2)[2].split(".")[0] for k in saved if k.startswith("layers.0.")} == {
        "lin_query", "lin_key", "lin_value", "lin_skip"}
    torch.save(saved, path)
    fresh = create_model(tr.engines[0].layer_size, a).to(DEV)
    assert isinstance(fresh, GraphTransformer)
    fresh.load_state_dict(torch.load(path), strict=True)
    assert torch.equal(_full_logits(g, fresh, torch.float32), _full_logits(g, model, torch.float32))


# ------------------------------------------------------------------------------------------------ graphs, training
def test_cuda_graph_replay_equals_eager_bit_for_bit():
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit."""
    from pipegcn_b200 import ops
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    g, layouts = _layouts("tiny", 1)
    a = _tc_args(g, enable_pipeline=True)
    a.cuda_graph = True
    runs = []
    for captured in (False, True):
        ops.STEP_DEV = None
        torch.manual_seed(0)
        eng = RankEngine(layouts[0], a, LocalWorld(1, DEV).view(0), seg_len=32)
        eng.keep_logits = True
        rec = []
        for e in range(6):
            if captured and e == 3:
                eng.capture()
            loss = eng.run_epoch()
            if e >= 3:
                rec.append((loss.clone(), eng.last_logits.clone(), [p.detach().clone() for p in eng.model.parameters()]))
        torch.cuda.synchronize()
        runs.append(rec)
        ops.STEP_DEV = None
    for (l0, z0, p0), (l1, z1, p1) in zip(*runs):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def test_free_running_training_learns_planted_labels():
    """60 pipelined epochs at P = 2 on planted labels (16 classes, chance 1/16): the training accuracy must clear
    3/16, as for GAT and GATv2."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("small", planted_labels=True)
    layouts = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    a = _tc_args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True)
    a.lr = 1e-2
    tr = _trainer(layouts, a)
    for _ in range(60):
        tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    hit = tot = 0
    for eng in tr.engines:
        z = eng.last_logits[:eng.part_train].float()
        hit += int((z.argmax(1) == eng.labels).sum())
        tot += eng.part_train
    print(f"transformer planted-label training accuracy: {hit / tot:.4f}")
    assert hit / tot > 3.0 / 16, hit / tot
