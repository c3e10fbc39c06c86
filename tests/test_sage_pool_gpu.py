"""Max-pool GraphSAGE (`--aggregator pool`) on the GPU: the neighbour-max kernels against an fp64 torch restatement
(first-in-CSR argmax), the layer's autograd, the engine against a restatement of partitioned training (partitions,
exchange modes, boundary-node sampling), evaluation, checkpoints, CUDA-graph replay and free-running training."""

import pytest
import torch
import torch.nn.functional as F

from tests.test_boundary_sampling_gpu import _args, _layouts, _trainer
from tests.test_gat_gpu import _edges, _full_logits, _hook_outputs, _poison, _scatter, _stored

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------ restatement
def ref_argmax(q, rows, cols, num_in):
    """(M, A) [num_in, d]: the maximum of q[cols] over the edges of every destination row and the source that gives
    it, the first in edge order on a tie; the first NaN source wins; a row without edges gets M = 0, A = -1."""
    d = q.shape[1]
    qd = q.detach().double()
    vals = qd[cols]
    isnan = torch.isnan(vals)
    has_nan = torch.zeros(num_in, d, dtype=torch.float64, device=q.device).index_reduce(
        0, rows, isnan.double(), "amax", include_self=True).bool()
    clean = torch.where(isnan, torch.tensor(float("-inf"), dtype=torch.float64, device=q.device), vals)
    m = torch.full((num_in, d), float("-inf"), dtype=torch.float64, device=q.device)
    m = m.index_reduce(0, rows, clean, "amax", include_self=True)
    cand = torch.where(has_nan[rows], isnan, clean == m[rows])
    e = torch.arange(rows.numel(), device=q.device)[:, None].expand(-1, d)
    big = rows.numel()
    pos = torch.where(cand, e, torch.full_like(e, big))
    first = torch.full((num_in, d), big, dtype=torch.int64, device=q.device).index_reduce(0, rows, pos, "amin")
    has_edge = first < big
    a = torch.where(has_edge, cols[first.clamp(max=big - 1)], torch.full_like(first, -1))
    mv = torch.where(has_nan, torch.tensor(float("nan"), dtype=torch.float64, device=q.device), m)
    return torch.where(has_edge, mv, torch.zeros_like(mv)), a


def ref_hn(q, a):
    """ReLU(q[A[v, c], c]) with the gradient flowing to that one source (0 where A = -1)."""
    g = q.gather(0, a.clamp(min=0))
    return torch.where(a >= 0, F.relu(g), torch.zeros_like(g))


def ref_pool_layer(x, w1, b1, w2, b2, wp, bp, rows, cols, num_in, keep=None, dtype=torch.float32, q_stored=None):
    """fp64 SAGEConv(aggregator_type='pool') over the edges cols -> rows: x [num_all, d_in] -> [num_in, d_out].  An
    unkept source's pooled transform is 0.  `q_stored`: the engine's stored Q (its values, with the gradient of the
    restated Q)."""
    q = _stored(x @ wp.T + bp, dtype)
    if q_stored is not None:
        q = q + (q_stored.double() - q).detach()
    if keep is not None:
        q = torch.where(keep[:, None], q, torch.zeros_like(q))
    _, a = ref_argmax(q, rows, cols, num_in)
    hn = ref_hn(q, a)
    return x[:num_in] @ w1.T + b1 + _stored(hn, dtype) @ w2.T + b2


def _graph(num_in=300, num_halo=120, seed=0, hubs=(200, 90, 65, 40, 33), seg_len=32, max_deg=12):
    """Bipartite `_U` -> `_V` graph with hub rows longer than seg_len (segments and fix-up), rows without in-edges,
    and a halo row referenced by many destinations (a long CSC row)."""
    from pipegcn_b200.graph import PartGraph
    from pipegcn_b200.partition import _csr_from_pairs
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    deg = torch.randint(1, max_deg, (num_in,), generator=gen)
    deg[:len(hubs)] = torch.tensor(hubs)
    deg[len(hubs):len(hubs) + 20] = 0                       # no in-edge
    dst = torch.repeat_interleave(torch.arange(num_in), deg)
    src = torch.randint(0, num_all, (int(deg.sum()),), generator=gen)
    src[torch.randperm(src.numel(), generator=gen)[:min(80, src.numel())]] = num_in + 3
    pairs = torch.unique(torch.stack([dst, src], 1), dim=0)
    pairs = pairs[torch.randperm(pairs.shape[0], generator=gen)]       # CSR order is not source order
    dst, src = pairs[:, 0], pairs[:, 1]
    order = torch.argsort(dst, stable=True)
    dst, src = dst[order], src[order]
    indptr, indices = _csr_from_pairs(dst, src, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(src, dst, num_all, num_in)
    in_deg = torch.bincount(dst, minlength=num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, in_deg, device=DEV, seg_len=seg_len)
    assert g.fwd.n_long > 0 and g.bwd.n_long > 0
    return g


def _rows_of(n, d, dtype, values):
    from pipegcn_b200.graph import alloc_rows
    t = alloc_rows(n, d, dtype, DEV)
    t.copy_(values)
    ld = t.stride(0)
    if ld > d:                                 # NaN in the pad columns: a leak into a stored column would show
        t.as_strided((n, ld - d), (ld, 1), d).fill_(float("nan"))
    return t


# ------------------------------------------------------------------------------------------------ kernels
GRAPHS = {"small": dict(), "wide": dict(num_in=40000, num_halo=9000, seed=1, max_deg=8)}


@pytest.mark.parametrize("graph", list(GRAPHS))
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 256, 602])
def test_max_aggregate_matches_restatement(d, dtype, ties, graph):
    """hn = ReLU(M) bit for bit and A exactly; integer-valued Q forces ties, one source row holds a NaN."""
    from pipegcn_b200 import ops
    g = _graph(**GRAPHS[graph])
    gen = torch.Generator(device=DEV).manual_seed(d)
    vals = torch.randn(g.num_all, d, generator=gen, device=DEV)
    if ties:
        vals = torch.randint(-3, 4, (g.num_all, d), generator=gen, device=DEV).float()
    vals[g.num_in + 3, d // 2] = float("nan")                 # the long-CSC-row source, referenced by a hub
    q = _rows_of(g.num_all, d, dtype, vals)
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    hn, a = ops.max_aggregate(g.fwd, q)
    m_ref, a_ref = ref_argmax(q.float(), rows, cols, g.num_in)
    assert torch.equal(a, a_ref.to(torch.int32))
    hn_ref = torch.where(torch.isnan(m_ref), m_ref, F.relu(m_ref))
    torch.testing.assert_close(hn.double(), hn_ref, rtol=0, atol=0, equal_nan=True)
    assert torch.isnan(hn.float()).any()
    hn2, a2 = ops.max_aggregate(g.fwd, q)
    assert torch.equal(a, a2) and torch.equal(hn.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                                              hn2.view(torch.int16 if dtype == torch.bfloat16 else torch.int32))


@pytest.mark.parametrize("graph", list(GRAPHS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 256, 602])
def test_max_aggregate_bwd_matches_restatement(d, dtype, graph):
    """gQ against the fp64 scatter of g_neigh through the argmax, with Q == 0 exactly at some maxima (no gradient
    there) and ties; two launches are bit-identical."""
    from pipegcn_b200 import ops
    g = _graph(**GRAPHS[graph])
    gen = torch.Generator(device=DEV).manual_seed(d + 1)
    vals = torch.randint(-2, 3, (g.num_all, d), generator=gen, device=DEV).float()
    vals += torch.where(torch.rand(g.num_all, d, generator=gen, device=DEV) < 0.5, 0.0, 0.25)
    q = _rows_of(g.num_all, d, dtype, vals)
    gn = _rows_of(g.num_in, d, dtype, torch.randn(g.num_in, d, generator=gen, device=DEV))
    hn, a = ops.max_aggregate(g.fwd, q)
    assert (hn.float() == 0).logical_and(a >= 0).any()                 # Q == 0 (or < 0) at an argmax
    gq = ops.max_aggregate_bwd(g.bwd, q, a, gn)
    gq2 = ops.max_aggregate_bwd(g.bwd, q, a, gn)
    iv = torch.int16 if dtype == torch.bfloat16 else torch.int32
    assert torch.equal(gq.view(iv), gq2.view(iv))
    qd = q.double().requires_grad_(True)
    ref_hn(qd, a.long()).backward(gn.double())
    ref = qd.grad
    if dtype == torch.float32:
        bound = 4e-5 * torch.zeros_like(ref).scatter_add_(0, a.long().clamp(min=0), gn.double().abs() * (a >= 0))
        assert ((gq.double() - ref).abs() <= bound + 1e-30).all()
    else:
        torch.testing.assert_close(gq.double(), ref.to(torch.bfloat16).double(), rtol=1e-2, atol=1e-2)
    no_out = (g.bwd.indptr[1:] == g.bwd.indptr[:-1])
    assert torch.count_nonzero(gq[no_out].float()) == 0


# ------------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("drop", [0.0, 0.3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d_in,d_out", [(24, 16), (64, 64), (300, 40)])
def test_layer_autograd_matches_restatement(d_in, d_out, dtype, drop, masked):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    g = _graph()
    gen = torch.Generator(device=DEV).manual_seed(7)
    x = alloc_rows(g.num_all, d_in, dtype, DEV)
    x.copy_(torch.randn(g.num_all, d_in, generator=gen, device=DEV))
    keep, keep_u = None, torch.ones(g.num_all, dtype=torch.bool, device=DEV)
    if masked:
        halo = torch.rand(g.num_all - g.num_in, generator=gen, device=DEV) < 0.5
        keep = halo.to(torch.uint8).contiguous()
        keep_u = torch.cat([torch.ones(g.num_in, dtype=torch.bool, device=DEV), halo])
        x[~keep_u] = 0                         # the exchange leaves unkept halo rows zero
    s = d_in ** -0.5
    params = [torch.randn(d_out, d_in, generator=gen, device=DEV) * s, torch.randn(d_out, generator=gen, device=DEV) * s,
              torch.randn(d_out, d_in, generator=gen, device=DEV) * s, torch.randn(d_out, generator=gen, device=DEV) * s,
              torch.randn(d_in, d_in, generator=gen, device=DEV) * s, torch.randn(d_in, generator=gen, device=DEV) * s]
    up = torch.randn(g.num_in, d_out, generator=gen, device=DEV)
    spec = ops.DropSpec(drop, 1234) if drop > 0 else None

    def run():
        xs = x.detach().clone().requires_grad_(True)
        ps = [p.detach().clone().requires_grad_(True) for p in params]
        o = ops.sage_pool_layer(xs, g, keep, *ps, drop_bwd=spec)
        o.backward(up.to(dtype))
        return o.detach(), xs.grad, [p.grad for p in ps]

    o1, gx1, gp1 = run()
    o2, gx2, gp2 = run()
    assert torch.equal(o1, o2) and torch.equal(gx1, gx2) and all(torch.equal(a, b) for a, b in zip(gp1, gp2))
    # the Q the layer stores: the same product, launched the same way
    q_eng = ops.gemm_nt(ops.presplit(x), ops.padded_weight(params[4], dtype), bias=params[5])
    xr = x.double().requires_grad_(True)
    pr = [(p.to(dtype).double() if p.dim() == 2 else p.double()).requires_grad_(True) for p in params]
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    o_r = ref_pool_layer(xr, *pr, rows, cols, g.num_in, keep_u if masked else None, dtype, q_stored=q_eng)
    o_r.backward(up.double())
    gx_ref = xr.grad
    if spec is not None:
        gx_ref = gx_ref * torch.from_numpy(ops.dropout_keep_host(spec, None, 0, g.num_all, d_in, x.element_size())
                                           ).to(DEV) / (1 - drop)
    tol = 1e-4 if dtype == torch.float32 else 3e-2

    def close(got, ref, what):
        err, scale = (got.double() - ref).abs().max().item(), ref.abs().max().item()
        assert err <= tol * scale + 1e-6, (what, err, scale)

    close(o1, o_r.detach(), "out")
    close(gx1, gx_ref, "g_feat")
    for name, got, ref in zip(("dW1", "db1", "dW2", "db2", "dWp", "dbp"), gp1, [p.grad for p in pr]):
        close(got, ref, name)
    if masked:
        assert torch.count_nonzero(gx1[~keep_u].float()) == 0


# ------------------------------------------------------------------------------------------------ engine
def _pool_args(g, n_class=5, **kw):
    a = _args(g, n_class, **kw)
    a.aggregator = "pool"
    return a


def restate_training(layouts, masks, state, a, dtype):
    """Partitioned max-pool GraphSAGE training in fp64: per rank the forward over its partition (unkept halo rows
    pool to 0), loss and reduced gradients.  With bf16 storage the weights, Q and the activations are rounded where
    the engine stores them."""
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
                xu = _stored(H[q["gid"]], dtype) * q["keep"][:, None]
                w = [_stored(params[f"layers.{i}.{k}.weight"], dtype) for k in ("linear1", "linear2", "pool")]
                b = [params[f"layers.{i}.{k}.bias"] for k in ("linear1", "linear2", "pool")]
                out = ref_pool_layer(xu, w[0], b[0], w[1], b[1], w[2], b[2], q["rows"], q["cols"], q["num_in"],
                                     q["keep"] if masks is not None else None, dtype)
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
                gref = grads[name]
                assert (prm.grad.double() - gref).norm() <= 0.25 * gref.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype)
    (1, "random", True, 0, "fp32"),
    (1, "random", False, 1, "bf16"),
    (2, "random", True, 0, "fp32"),
    (2, "metis", False, 1, "bf16"),
    (3, "metis", False, 0, "fp32"),
    (3, "random", True, 1, "fp32"),
    (4, "metis", False, 1, "fp32"),
    (4, "random", True, 0, "bf16"),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype):
    """Synchronous training, dropout 0, 3 epochs with the engine's weights; every halo row poisoned with NaN before
    each epoch."""
    g, layouts = _layouts("tiny", P, method)
    a = _pool_args(g, static_layer0=static0, n_linear=n_linear)
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
    """Boundary-node sampling: an unkept halo row pools to 0 (the restatement of the sampled graph), every halo row
    poisoned with NaN before each epoch."""
    g, layouts = _layouts("tiny", P, method)
    a = _pool_args(g, static_layer0=static0, sampling_rate=p)
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


@pytest.mark.parametrize("mode", [dict(feat_corr=True, grad_corr=True), dict(enable_pipeline=True),
                                  dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8)])
def test_exchange_modes_layer_parity(mode):
    """P = 3: every pool layer's output and input gradient equal the restated layer applied to the rows the layer
    read (the engine's own f_buf rows) and the upstream gradient it received."""
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _pool_args(g, static_layer0=False, **mode)
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
    n_checked = 0
    for _ in range(4):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        tr.run_epoch()
        torch.cuda.synchronize()
        for r, (eng, lay) in enumerate(zip(tr.engines, layouts)):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            for i in range(n_graph):
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                p = [state[f"layers.{i}.{k}.{t}"] for k in ("linear1", "linear2", "pool") for t in ("weight", "bias")]
                out = ref_pool_layer(x, *p, rows, cols, lay.num_in)
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
    a = _pool_args(g)
    tr = _trainer(layouts, a)
    tr.run_epoch()
    eng = tr.engines[0]
    weights = create_model(eng.layer_size, a).to(DEV)
    weights.load_state_dict(eng.model.state_dict())
    tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    got = _scatter(layouts, [eng.last_logits], g.n_nodes)
    ref = _full_logits(g, weights, eng.dtype)
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("P", [2, 4])
def test_partitioned_eval_equals_rank0(P):
    g, layouts = _layouts("small", P)
    a = _pool_args(g, 16, n_hidden=32, dropout=0.3, enable_pipeline=True)
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
    from pipegcn_b200.module.model import GraphSAGE
    g, layouts = _layouts("tiny", 2)
    a = _pool_args(g, n_linear=1)
    tr = _trainer(layouts, a)
    for _ in range(2):
        tr.run_epoch()
    torch.cuda.synchronize()
    model = tr.engines[0].model
    path = tmp_path / "pool.pth.tar"
    torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, path)
    fresh = GraphSAGE(tr.engines[0].layer_size, F.relu, False, dropout=0.0, n_linear=1, aggregator="pool").to(DEV)
    fresh.load_state_dict(torch.load(path), strict=True)
    assert torch.equal(_full_logits(g, fresh, torch.float32), _full_logits(g, model, torch.float32))


# ------------------------------------------------------------------------------------------------ graphs, training
def _replay_runs(a, layouts, capture_at=3, epochs=6):
    from pipegcn_b200 import ops
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    ops.STEP_DEV = None
    torch.manual_seed(0)
    eng = RankEngine(layouts[0], a, LocalWorld(1, DEV).view(0), seg_len=32)
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


def _same(r0, r1):
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_cuda_graph_replay_equals_eager_bit_for_bit(dtype):
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit."""
    g, layouts = _layouts("tiny", 1)
    a = _pool_args(g, enable_pipeline=True)
    a.dtype = dtype
    a.cuda_graph = True
    _same(_replay_runs(a, layouts, None), _replay_runs(a, layouts, 3))


def test_explicit_mean_equals_flag_absent():
    g, layouts = _layouts("tiny", 1)
    a = _args(g, enable_pipeline=True)
    a.cuda_graph = True
    runs = [_replay_runs(a, layouts, 3)]
    a.aggregator = "mean"
    runs.append(_replay_runs(a, layouts, 3))
    _same(*runs)


def test_free_running_training_learns_planted_labels():
    """16 planted classes (chance 1/16): validation accuracy after 60 pipelined epochs on 2 partitions."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    g = make_graph("small", planted_labels=True)
    layouts = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    a = _pool_args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True)
    a.lr = 1e-2
    tr = _trainer(layouts, a)
    for _ in range(60):
        tr.run_epoch()
    torch.cuda.synchronize()
    got = _scatter(layouts, tr.predict(), g.n_nodes)
    tr.release_eval()
    val = g.val_mask.to(DEV)
    acc = (got[val].argmax(1).cpu() == g.label[val.cpu()]).float().mean().item()
    print(f"pool validation accuracy {acc:.4f}")
    assert acc > 0.3, acc
