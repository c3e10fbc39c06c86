"""Graph attention (`--model gat`) on the GPU: the attention kernels against an fp64 torch restatement (scatter
softmax over the CSR), the engine against a restatement of partitioned GAT training (all partitions, exchange modes,
boundary-node sampling), evaluation, checkpoints, CUDA-graph replay and free-running training."""

import pytest
import torch
import torch.nn.functional as F

from tests.test_boundary_sampling_gpu import _layouts, _trainer

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------ restatement
def ref_gat(x, w, al, ar, b, rows, cols, num_in, heads, keep=None):
    """fp64 GATConv over the edges cols -> rows: x [num_all, d_in] -> [num_in, H*D]; also (m, s) [num_in, H].  Edges
    whose source is not kept are absent."""
    if keep is not None:
        ek = keep[cols]
        rows, cols = rows[ek], cols[ek]
    z = (x @ w.T).view(x.shape[0], heads, -1)
    return ref_attend(z, al, ar, b, rows, cols, num_in)


def ref_attend(z, al, ar, b, rows, cols, num_in):
    heads = z.shape[1]
    el = (z * al.view(1, heads, -1)).sum(-1)
    er = (z[:num_in] * ar.view(1, heads, -1)).sum(-1)
    e = F.leaky_relu(el[cols] + er[rows], 0.2)
    m = torch.full((num_in, heads), float("-inf"), dtype=z.dtype, device=z.device)
    m = m.scatter_reduce(0, rows[:, None].expand(-1, heads), e, "amax")
    p = torch.exp(e - m[rows])
    s = torch.zeros(num_in, heads, dtype=z.dtype, device=z.device).index_add(0, rows, p)
    a = p / s[rows]
    out = torch.zeros(num_in, heads, z.shape[2], dtype=z.dtype, device=z.device)
    out = out.index_add(0, rows, a[..., None] * z[cols])
    return out.reshape(num_in, -1) + b, m.detach(), s.detach()


def _edges(lay_or_graph):
    indptr, indices = lay_or_graph
    rows = torch.repeat_interleave(torch.arange(indptr.numel() - 1, device=DEV), (indptr[1:] - indptr[:-1]).long())
    return rows, indices.long()


def _test_graph(num_in=300, num_halo=120, seed=0):
    """Bipartite `_U` -> `_V` graph with self loops, hub rows longer than seg_len = 32 (the fix-up path), rows whose
    only edge is the self loop, and halo rows referenced by many destinations (long CSC rows)."""
    from pipegcn_b200.graph import PartGraph
    from pipegcn_b200.partition import _csr_from_pairs
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    deg = torch.randint(1, 12, (num_in,), generator=gen)
    deg[:5] = torch.tensor([200, 90, 65, 40, 33])          # hubs
    deg[5:25] = 0                                           # self loop only
    dst = torch.repeat_interleave(torch.arange(num_in), deg)
    src = torch.randint(0, num_all, (int(deg.sum()),), generator=gen)
    src[torch.randperm(src.numel(), generator=gen)[:80]] = num_in + 3     # a halo row with a long CSC row
    pairs = torch.unique(torch.stack([dst, src], 1), dim=0)
    pairs = pairs[pairs[:, 0] != pairs[:, 1]]
    loops = torch.arange(num_in)
    dst, src = torch.cat([pairs[:, 0], loops]), torch.cat([pairs[:, 1], loops])
    indptr, indices = _csr_from_pairs(dst, src, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(src, dst, num_all, num_in)
    in_deg = torch.bincount(dst, minlength=num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, in_deg, device=DEV, seg_len=32)
    assert g.fwd.n_long > 0 and g.bwd.n_long > 0
    return g


def _tensors(g, d_in, heads, d, dtype, seed=1):
    from pipegcn_b200.graph import alloc_rows
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = alloc_rows(g.num_all, d_in, dtype, DEV)
    x.copy_(torch.randn(g.num_all, d_in, generator=gen, device=DEV))
    w = torch.randn(heads * d, d_in, generator=gen, device=DEV) / d_in ** 0.5
    al = torch.randn(1, heads, d, generator=gen, device=DEV) / d ** 0.5
    ar = torch.randn(1, heads, d, generator=gen, device=DEV) / d ** 0.5
    b = torch.randn(heads * d, generator=gen, device=DEV) * 0.1
    up = torch.randn(g.num_in, heads * d, generator=gen, device=DEV)
    return x, w, al, ar, b, up


def _keep(g, on, seed=5):
    if not on:
        return None, torch.ones(g.num_all, dtype=torch.bool, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    halo = torch.rand(g.num_all - g.num_in, generator=gen, device=DEV) < 0.5
    halo[3] = True
    return halo.to(torch.uint8).contiguous(), torch.cat([torch.ones(g.num_in, dtype=torch.bool, device=DEV), halo])


def _close(got, ref, dtype, what, rel=None):
    got, ref = got.double(), ref.double()
    if dtype == torch.float32:
        torch.testing.assert_close(got, ref, rtol=rel or 1e-4, atol=(rel or 1e-4) * max(ref.abs().max().item(), 1e-3),
                                   msg=what)
    else:
        err, scale = (got - ref).norm().item(), ref.norm().item()
        assert err <= (rel or 2e-2) * scale + 1e-6, (what, err, scale)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64])
@pytest.mark.parametrize("heads", [1, 2, 4, 8])
def test_kernels_match_fp64_restatement(heads, d, dtype, masked):
    from pipegcn_b200 import ops
    g = _test_graph()
    x, w, al, ar, b, up = _tensors(g, 24, heads, d, dtype)
    keep, keep_u = _keep(g, masked)
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    # the exchange leaves unkept halo rows zero (the layer input); their z is poisoned with NaN below, so that a leak
    # into any sum of the kernels would show
    x[~keep_u] = 0

    # ---- kernel level, on the engine's own z
    z = ops.gemm_nt(ops.presplit(x), ops.padded_weight(w, dtype))
    z[~keep_u] = float("nan")
    al32, ar32, b32 = ops._f32(al), ops._f32(ar), ops._f32(b)
    el, er = ops.gat_scores(z, al32, ar32, heads, g.num_in)
    out, m, s = ops.gat_aggregate(g, z, el, er, b32, heads, keep)
    zk = z.double().view(g.num_all, heads, d)
    kept = keep_u.nonzero().squeeze(1)
    el_ref = (zk * al.double().view(1, heads, d)).sum(-1)
    torch.testing.assert_close(el[kept].double(), el_ref[kept], rtol=1e-5, atol=1e-5)
    ek = keep_u[cols]
    zl = zk.clone().requires_grad_(True)
    zz = torch.where(keep_u[:, None, None], zl, torch.zeros_like(zl))
    o_ref, m_ref, s_ref = ref_attend(zz, al.double(), ar.double(), b.double(), rows[ek], cols[ek], g.num_in)
    torch.testing.assert_close(m.double(), m_ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(s.double(), s_ref, rtol=1e-5, atol=1e-5)
    _close(out, o_ref, dtype, "out", rel=1e-5 if dtype == torch.float32 else 1e-2)
    gu = up.to(dtype)
    der, dv = ops.gat_bwd_dst(g, z, gu, el, er, m, s, heads, keep)
    dz, dl = ops.gat_bwd_src(g, z, gu, el, er, m, s, dv, der, al32, ar32, heads, keep)
    o_ref.backward(gu.double())
    dz_ref = zl.grad.reshape(g.num_all, -1)
    _close(dz[:g.num_in], dz_ref[:g.num_in], dtype, "dz inner", rel=1e-4 if dtype == torch.float32 else 2e-2)
    _close(dz[g.num_in:], dz_ref[g.num_in:], dtype, "dz halo", rel=1e-4 if dtype == torch.float32 else 2e-2)
    if masked:
        assert torch.count_nonzero(dz[g.num_in:][~keep_u[g.num_in:]].float()) == 0

    # ---- the layer with autograd against torch.autograd in fp64
    def layer_run():
        xs = x.detach().clone().requires_grad_(True)
        ps = [t.detach().clone().requires_grad_(True) for t in (w, al, ar, b)]
        o = ops.gat_layer(xs, g, keep, heads, *ps)
        o.backward(up.to(dtype))
        return o.detach(), xs.grad, [p.grad for p in ps]

    o1, gx1, gp1 = layer_run()
    o2, gx2, gp2 = layer_run()
    assert torch.equal(o1, o2) and torch.equal(gx1, gx2) and all(torch.equal(a, b_) for a, b_ in zip(gp1, gp2))

    xr = torch.where(keep_u[:, None], x.double(), torch.zeros((), dtype=torch.float64, device=DEV))
    xr = xr.requires_grad_(True)
    wr = (w.to(dtype) if dtype == torch.bfloat16 else w).double().requires_grad_(True)
    pr = [t.double().requires_grad_(True) for t in (al, ar, b)]
    o_r, _, _ = ref_gat(xr, wr, *pr, rows, cols, g.num_in, heads, keep_u)
    o_r.backward(up.double())
    _close(o1, o_r, dtype, "layer out", rel=2e-4 if dtype == torch.float32 else 3e-2)
    kx = keep_u
    _close(gx1[kx], xr.grad[kx], dtype, "dh_all", rel=2e-4 if dtype == torch.float32 else 5e-2)
    if masked:
        assert torch.count_nonzero(gx1[~kx].float()) == 0
    for name, got, ref in zip(("dW", "d attn_l", "d attn_r", "dbias"), gp1, [wr.grad] + [p.grad for p in pr]):
        _close(got, ref, dtype, name, rel=2e-4 if dtype == torch.float32 else 5e-2)


# ------------------------------------------------------------------------------------------------ engine
def _gat_args(g, n_class=5, **kw):
    from tests.test_boundary_sampling_gpu import _args
    heads = kw.pop("n_heads", 4)
    a = _args(g, n_class, **kw)
    a.model, a.n_heads = "gat", heads
    return a


def _stored(t, dtype):
    """t rounded as the engine stores it (bf16 weights, z and activations), with the gradient passed straight
    through."""
    return t if dtype == torch.float32 else t + (t.to(dtype).double() - t).detach()


def restate_training(layouts, masks, state, a, dtype):
    """Partitioned GAT training in fp64: per rank the forward over its partition (unkept halo sources absent), loss
    and reduced gradients.  Returns per-rank per-graph-layer outputs, logits, losses and the gradients.  With bf16
    storage the weights, z and the layer inputs are rounded to bf16 where the engine stores them."""
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
                heads = params[f"layers.{i}.attn_l"].shape[1]
                xu = _stored(H[q["gid"]], dtype) * q["keep"][:, None]
                w = _stored(params[f"layers.{i}.fc.weight"], dtype)
                ek = q["keep"][q["cols"]]
                z = _stored(xu @ w.T, dtype).view(xu.shape[0], heads, -1)
                out, _, _ = ref_attend(z, params[f"layers.{i}.attn_l"], params[f"layers.{i}.attn_r"],
                                       params[f"layers.{i}.bias"], q["rows"][ek], q["cols"][ek], q["num_in"])
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


def _poison(tr):
    """NaN into every halo row the coming epoch receives (the static layer-0 store is written once, not per epoch)."""
    for eng in tr.engines:
        buf = eng.buffer
        for (layer, v), rows in buf._f_buf.items():
            if layer > 0 or not buf.static0_ready or buf.sampling:
                rows[buf._num_in:, :buf._layer_size[layer]] = float("nan")
    torch.cuda.synchronize()


def _check_engine(tr, layouts, a, caps, masks, state, losses, dtype):
    """The tolerances of test_engine_matches_sampled_graph_restatement."""
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    outs, logits, ref_losses, grads = restate_training(layouts, masks, state, a, tdt)
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
                gr = grads[name]
                assert (prm.grad.double() - gr).norm() <= 0.25 * gr.norm() + 1e-6, name


def _hook_outputs(tr, a):
    caps = [dict() for _ in tr.engines]
    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:a.n_layers - a.n_linear]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: caps[r].__setitem__(i, out.detach()))
    return caps


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
    """Synchronous training, dropout 0, 3 epochs with the engine's weights; every halo row poisoned with NaN before
    each epoch.  Layer widths 20 -> 16 (4 heads of 4) -> 16 -> 5 (one head) or a trailing linear."""
    g, layouts = _layouts("tiny", P, method)
    a = _gat_args(g, static_layer0=static0, n_linear=n_linear)
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
    """Boundary-node sampling: unkept halo sources are absent from every softmax (the keep mask reaches the
    kernels), unkept rows are poisoned with NaN."""
    g, layouts = _layouts("tiny", P, method)
    a = _gat_args(g, static_layer0=static0, sampling_rate=p)
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
        assert all(torch.equal(eng.buffer.keep_mask[:len(m)].bool(), m) for eng, m in zip(tr.engines, masks))
        _check_engine(tr, layouts, a, caps, masks, state, losses, dtype)


@pytest.mark.parametrize("mode", [dict(enable_pipeline=True), dict(enable_pipeline=True, feat_corr=True, grad_corr=True),
                                  dict(feat_corr=True, grad_corr=True)])
def test_exchange_modes_layer_parity(mode):
    """P = 3: every GAT layer's output and input gradient equal the restated layer applied to the [num_all] input and
    the upstream gradient the engine captured."""
    g, layouts = _layouts("tiny", 3)
    a = _gat_args(g, static_layer0=False, **mode)
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
                out, _, _ = ref_gat(x, state[f"layers.{i}.fc.weight"], state[f"layers.{i}.attn_l"],
                                    state[f"layers.{i}.attn_r"], state[f"layers.{i}.bias"], rows, cols, lay.num_in,
                                    layer.num_heads)
                torch.testing.assert_close(rec["out"].double(), out.detach(), rtol=2e-4, atol=2e-4)
                out.backward(rec["gout"].double())
                if "gx" in rec:
                    torch.testing.assert_close(rec["gx"].double(), x.grad, rtol=2e-4, atol=2e-5)
                    n_checked += 1
    assert n_checked > 0


# ------------------------------------------------------------------------------------------------ evaluation
def _full_logits(g, model, dtype):
    from pipegcn_b200.evaluate import EvalSet, _logits
    es = EvalSet(g, DEV, inductive=False, dtype=dtype)
    return _logits(model, es.val)


def _scatter(layouts, logits, n):
    out = torch.full((n, logits[0].shape[1]), float("nan"), device=DEV)
    for lay, z in zip(layouts, logits):
        out[lay.inner_gid.to(DEV)] = z.float()
    return out


def test_single_partition_logits_equal_full_graph_eval():
    from pipegcn_b200.train import create_model
    g, layouts = _layouts("tiny", 1)
    a = _gat_args(g)
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
    a = _gat_args(g, 16, n_hidden=32, dropout=0.3, enable_pipeline=True)
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
    from pipegcn_b200.module.model import GAT
    from pipegcn_b200.train import create_model
    g, layouts = _layouts("tiny", 2)
    a = _gat_args(g, n_linear=1)
    tr = _trainer(layouts, a)
    for _ in range(2):
        tr.run_epoch()
    torch.cuda.synchronize()
    model = tr.engines[0].model
    path = tmp_path / "gat.pth.tar"
    torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, path)
    fresh = create_model(tr.engines[0].layer_size, a).to(DEV)
    assert isinstance(fresh, GAT)
    fresh.load_state_dict(torch.load(path), strict=True)
    assert torch.equal(_full_logits(g, fresh, torch.float32), _full_logits(g, model, torch.float32))


# ------------------------------------------------------------------------------------------------ graphs, training
def test_cuda_graph_replay_equals_eager_bit_for_bit():
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit."""
    from pipegcn_b200 import ops
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    g, layouts = _layouts("tiny", 1)
    a = _gat_args(g, enable_pipeline=True)
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
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("small", planted_labels=True)
    layouts = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    a = _gat_args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True)
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
    assert hit / tot > 3.0 / 16, hit / tot
