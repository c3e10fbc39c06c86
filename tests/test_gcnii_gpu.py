"""GCNII (`--model gcnii`) on the GPU: `pg_aggregate_scaled_res` against fp64 on every dispatch path and bit for bit
against `pg_aggregate_scaled` without a residual, the row kernels, the layer autograd (teleport sum, dropout keys),
the engine against an fp64 restatement of partitioned training, full-graph equivalence, every exchange mode,
evaluation, checkpoints, CUDA-graph replay and learning at depth."""
import argparse
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_graphconv_gpu import U24, _guarded_out, _scales, _small, _widths, scaled_ref
from tests.test_kernel_conformance_gpu import AGG_IMPLS, DEV, _graph, _normal, knobs, padded, x_with_nans

pytestmark = pytest.mark.gpu

_W = {torch.float32: torch.int32, torch.bfloat16: torch.int16}


# ------------------------------------------------------------------------------------------------ residual aggregate
@pytest.mark.parametrize("impl,narrow", AGG_IMPLS)
@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("dtype,d", _widths())
@pytest.mark.parametrize("seg_len", [32, 512])
def test_aggregate_scaled_res_vs_fp64(impl, narrow, overlap, dtype, d, seg_len):
    """Empty rows, full chunks, rows around seg_len and hubs (segmented: the residual comes once, in the fix-up); NaN in
    row 0, the unreferenced rows and every pad column of x and of the residual; a guard around the output.  Without a
    residual the bits of pg_aggregate_scaled; the same bits from run to run."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(seg_len)
    gen = torch.Generator().manual_seed(d + seg_len + 3)
    n_ref = 6000
    x = x_with_nans(n_ref + 50, n_ref, d, dtype, gen)
    src, dst = _scales(n_ref + 50, gen), _scales(plan.n_rows, gen)
    res = padded(plan.n_rows, d, dtype, data=_normal((plan.n_rows, d), gen).to(dtype))     # pads: NaN
    alpha = 0.3
    bias = _normal((d,), gen).to(DEV)
    with knobs(agg_impl=impl, agg_narrow=narrow, agg_overlap=overlap):
        for b in (None, bias):
            out, check_guard = _guarded_out(plan.n_rows, d, dtype)
            ops.aggregate_scaled_res(plan, x, src, dst, res=res, alpha=alpha, bias=b, out=out)
            check_guard()
            ref, mag, lens = scaled_ref(indptr, indices, x, src, dst)
            ref = ref + alpha * res.double()
            mag = mag + alpha * res.double().abs()
            if b is not None:
                ref, mag = ref + b.double(), mag + b.double().abs()
            err = (out.double() - ref).abs()
            bound = ((lens.double() + 15) * U24)[:, None] * mag + (ref.abs() * 2.0 ** -8 if dtype == torch.bfloat16 else 0)
            assert torch.all(err <= bound), f"max excess {float((err - bound).max())}"
            again = ops.aggregate_scaled_res(plan, x, src, dst, res=res, alpha=alpha, bias=b)
            assert torch.equal(out.view(_W[dtype]), again.view(_W[dtype]))
        a = ops.aggregate_scaled(plan, x, src, dst, bias=bias)
        r = ops.aggregate_scaled_res(plan, x, src, dst, res=None, alpha=alpha, bias=bias)
        assert torch.equal(a.view(_W[dtype]), r.view(_W[dtype]))


@pytest.mark.parametrize("opts", [dict(agg_impl=2, agg_l2_hint=1), dict(agg_impl=3, agg_l2_hint=1),
                                  dict(agg_impl=1, agg_unroll=4)])
@pytest.mark.parametrize("dtype,d", [(torch.float32, 64), (torch.bfloat16, 256), (torch.bfloat16, 602)])
def test_aggregate_scaled_res_other_knobs_and_dropout(opts, dtype, d):
    """The L2-hint walkers and four rows in flight against fp64; with a dropout key the result is dropout of the
    residual sum, mask of that key (ops.dropout_keep_host)."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(32)
    gen = torch.Generator().manual_seed(d + 11)
    x = x_with_nans(6050, 6000, d, dtype, gen)
    src, dst = _scales(6050, gen), _scales(plan.n_rows, gen)
    res = padded(plan.n_rows, d, dtype, data=_normal((plan.n_rows, d), gen).to(dtype))
    spec = ops.DropSpec(0.4, 99)
    with knobs(**opts):
        out = ops.aggregate_scaled_res(plan, x, src, dst, res=res, alpha=0.1)
        outd = ops.aggregate_scaled_res(plan, x, src, dst, res=res, alpha=0.1, drop=spec)
    ref, mag, lens = scaled_ref(indptr, indices, x, src, dst)
    ref, mag = ref + 0.1 * res.double(), mag + 0.1 * res.double().abs()
    err = (out.double() - ref).abs()
    bound = ((lens.double() + 15) * U24)[:, None] * mag + (ref.abs() * 2.0 ** -8 if dtype == torch.bfloat16 else 0)
    assert torch.all(err <= bound), f"max excess {float((err - bound).max())}"
    keep = torch.from_numpy(ops.dropout_keep_host(spec, None, 0, plan.n_rows, d, x.element_size())).to(DEV)
    assert torch.all(outd[~keep] == 0)
    kept = (outd.double() - out.double() / (1 - 0.4))[keep].abs()
    assert torch.all(kept <= (out.double() / (1 - 0.4))[keep].abs() * (2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -22))


# ------------------------------------------------------------------------------------------------ row kernels
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 300])
def test_row_kernels_vs_fp64(dtype, d):
    from pipegcn_b200 import ops
    gen = torch.Generator().manual_seed(d)
    n, n_in = 70_000, 50_000
    z = padded(n, d, dtype, data=_normal((n, d), gen).to(dtype))
    spec = ops.DropSpec(0.3, 4321)
    h0, hd = ops.gcnii_relu_drop(z, spec)
    assert torch.equal(h0.view(_W[dtype]), torch.relu(z).view(_W[dtype]))
    keep = torch.from_numpy(ops.dropout_keep_host(spec, None, 0, n, d, z.element_size())).to(DEV)
    scale = 1.0 / (1.0 - torch.tensor(0.3, dtype=torch.float32))          # make_drop: fp32 arithmetic
    expect = torch.where(keep, (h0.float() * scale.to(DEV)).to(dtype), torch.zeros((), dtype=dtype, device=DEV))
    assert torch.equal(hd.view(_W[dtype]), expect.view(_W[dtype]))
    dv = -(-d // (16 // z.element_size())) * (16 // z.element_size())
    assert torch.all(h0.as_strided((n, dv), h0.stride())[:, d:].float() == 0)      # pad columns of the last vector: 0
    h0b, hdb = ops.gcnii_relu_drop(z, None)
    assert hdb is h0b and torch.equal(h0b.view(_W[dtype]), h0.view(_W[dtype]))

    ds = [padded(n_in, d, dtype, data=_normal((n_in, d), gen).to(dtype)) for _ in range(3)]
    acc = torch.empty(n_in, (d + 7) // 8 * 8, device=DEV)[:, :d]
    ref = None
    for k, t in enumerate(ds):
        ops.gcnii_teleport(t, acc, 0.15, accumulate=k > 0)
        term = 0.15 * t.double()
        ref = term if ref is None else ref + term
    assert torch.all((acc.double() - ref).abs() <= 4 * U24 * (0.15 * sum(t.double().abs() for t in ds)))

    g = padded(n, d, dtype, data=_normal((n, d), gen).to(dtype))
    dz = ops.gcnii_relu_bwd(g, h0, acc)
    full = g.double().clone()
    full[:n_in] += acc.double()
    ref = torch.where(h0.double() > 0, full, torch.zeros((), dtype=torch.float64, device=DEV))
    tol = (ref.abs() * (2.0 ** -8 if dtype == torch.bfloat16 else U24 * 2)).max()
    assert (dz.double() - ref).abs().max() <= tol


# ------------------------------------------------------------------------------------------------ layer autograd
class _Dropped(torch.autograd.Function):
    """dropout(x) under `spec` whose backward passes the gradient through: the layer's drop_bwd applies the mask."""

    @staticmethod
    def forward(ctx, x, spec):
        from pipegcn_b200 import ops
        from pipegcn_b200.graph import alloc_rows
        xp = alloc_rows(x.shape[0], x.shape[1], x.dtype, x.device)
        xp.copy_(x)
        return ops.dropout_rows(xp, spec) if spec is not None else xp

    @staticmethod
    def backward(ctx, g):
        return g, None


@pytest.mark.parametrize("drop", [0.0, 0.3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_layer_autograd_matches_restatement(dtype, drop):
    """Graph layer 0 (fc_in, ReLU, keyed dropout of h0, convolution 1) and convolution 2 on its ReLU'd output (keyed
    dropout with the mask applied by the CSC store): outputs and every gradient, the teleport sum of both
    convolutions included, against fp64 autograd; the same bits from run to run."""
    from pipegcn_b200 import ops
    from tests.test_gat_gpu import _edges, _stored
    from tests.test_sage_pool_gpu import _graph as _pool_graph
    g = _pool_graph()
    deg = torch.bincount(g.bwd.indices.long(), minlength=g.num_in)
    c = ops.sym_norm(torch.cat([deg + 1, (g.bwd.indptr[1:] - g.bwd.indptr[:-1])[g.num_in:] + 3]))
    g.set_sym_norm(c)
    alpha, lam, Fd, d = 0.2, 0.5, 40, 64
    cs = g.gcnii_norm(alpha)
    b1, b2 = ops.gcnii_beta(lam, 1), ops.gcnii_beta(lam, 2)
    gen = torch.Generator(device=DEV).manual_seed(3)
    x = padded(g.num_all, Fd, dtype, data=torch.randn(g.num_all, Fd, generator=gen, device=DEV).to(dtype))
    w_in = torch.randn(d, Fd, generator=gen, device=DEV) * Fd ** -0.5
    bi = torch.randn(d, generator=gen, device=DEV) * 0.1
    w1 = [torch.randn(d, d, generator=gen, device=DEV) * d ** -0.5 for _ in range(2)]
    bs = [torch.randn(d, generator=gen, device=DEV) for _ in range(2)]
    halo = torch.randn(g.num_all - g.num_in, d, generator=gen, device=DEV).to(dtype)
    up = torch.randn(g.num_in, d, generator=gen, device=DEV)
    s_h0 = ops.DropSpec(drop, 77) if drop else None
    s_1 = ops.DropSpec(drop, 78) if drop else None

    def run():
        ps = [t.detach().clone().requires_grad_(True) for t in [w_in, bi] + w1 + bs]
        st = ops.GCNIIState(s_h0)
        o0 = ops.gcnii_first(x, g, c, cs, ps[0], ps[1], ps[2], ps[4], alpha, b1, st)
        x1 = _Dropped.apply(torch.cat([torch.relu(o0), halo]), s_1)
        o1 = ops.gcnii_conv(x1, g, c, cs, ps[3], ps[5], alpha, b2, st, drop_bwd=s_1)
        o1.backward(up.to(dtype))
        return [o0.detach(), o1.detach()] + [p.grad for p in ps]

    r1, r2 = run(), run()
    assert all(torch.equal(p, q) for p, q in zip(r1, r2))
    rows, cols = _edges((g.fwd.indptr, g.fwd.indices))
    cd = c.double()
    ref_p = [t.double().requires_grad_(True) for t in [w_in, bi] + w1 + bs]
    m_h0 = (torch.from_numpy(ops.dropout_keep_host(s_h0, None, 0, g.num_all, d, x.element_size())).to(DEV).double()
            / (1 - drop)) if drop else 1.0
    m_1 = (torch.from_numpy(ops.dropout_keep_host(s_1, None, 0, g.num_all, d, x.element_size())).to(DEV).double()
           / (1 - drop)) if drop else 1.0
    eye = torch.eye(d, dtype=torch.float64, device=DEV)

    def conv(h, h0, w, b, beta):
        agg = torch.zeros(g.num_in, d, dtype=torch.float64, device=DEV).index_add(0, rows, cd[cols, None] * h[cols])
        s = _stored((1 - alpha) * cd[:g.num_in, None] * agg + alpha * h0[:g.num_in], dtype)
        return s @ _stored((1 - beta) * eye + beta * w, dtype) + b

    h0 = torch.relu(_stored(x.double() @ _stored(ref_p[0], dtype).t() + ref_p[1], dtype))   # rounded where stored
    o0 = conv(m_h0 * h0, h0, ref_p[2], ref_p[4], b1)
    o1 = conv(m_1 * _stored(torch.cat([torch.relu(o0), halo.double()]), dtype), h0, ref_p[3], ref_p[5], b2)
    o1.backward(up.to(dtype).double())
    tol = 1e-4 if dtype == torch.float32 else 5e-2
    for got, ref, what in zip(r1, [o0, o1] + [p.grad for p in ref_p], ["o0", "o1", "w_in", "b_in", "w1", "w2", "b1", "b2"]):
        err, scale = (got.double() - ref.detach()).abs().max().item(), ref.detach().abs().max().item()
        assert err <= tol * scale + 1e-6, (what, err, scale)


# ------------------------------------------------------------------------------------------------ engine
def _args(g, n_class, **kw):
    base = dict(model="gcnii", backend="nccl", dtype="fp32", n_layers=3, n_hidden=16, n_linear=1,
                n_feat=g.n_feat, n_class=n_class, n_train=int(g.train_mask.sum()), dropout=0.0, norm="layer",
                lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=False, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=4, log_every=10, gcnii_alpha=0.2, gcnii_lambda=0.6)
    base.update(kw)
    return argparse.Namespace(**base)


def restate_training(g, layouts, state, a, dtype):
    """Partitioned GCNII training in fp64: per rank fc_in over its [inner | halo] rows of x, the convolutions with the
    global graph's c, LayerNorm + ReLU between the layers, the trailing linears, loss and reduced gradients.  With bf16
    storage the weights (W_eff included), z, h0, S and the layer inputs are rounded where the engine stores them."""
    from tests.test_gat_gpu import _edges, _stored
    n = g.n_nodes
    c_glob = 1.0 / torch.clamp(g.in_degrees().to(DEV).double(), min=1).sqrt()
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    alpha, lam = a.gcnii_alpha, a.gcnii_lambda
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
    h0s = [None] * len(layouts)
    eye = torch.eye(a.n_hidden, dtype=torch.float64, device=DEV)
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                xu = _stored(H[q["gid"]], dtype)
                if i == 0:
                    z = _stored(xu @ _stored(params["layers.0.fc_in.weight"], dtype).T + params["layers.0.fc_in.bias"], dtype)
                    h0s[r] = xu = torch.relu(z)
                beta = math.log(lam / (i + 1) + 1)
                agg = torch.zeros(q["num_in"], a.n_hidden, dtype=torch.float64, device=DEV).index_add(
                    0, q["rows"], q["c"][q["cols"], None] * xu[q["cols"]])
                s = _stored((1 - alpha) * q["c"][:q["num_in"], None] * agg + alpha * h0s[r][:q["num_in"]], dtype)
                w_eff = _stored((1 - beta) * eye + beta * params[f"layers.{i}.weight1"], dtype)
                out = s @ w_eff + params[f"layers.{i}.bias"]
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
    # bf16: every layer's stored rows carry 2^-9 relative rounding; through 8 convolutions' backward the gradients of
    # the first layers' parameters collect more of it than through 2
    g_tol = 0.25 if a.n_layers - a.n_linear <= 4 else 0.4
    outs, logits, ref_losses, grads = restate_training(g, layouts, state, a, tdt)
    for r, eng in enumerate(tr.engines):
        got_logits = eng.last_logits.double()
        assert torch.isfinite(got_logits).all()
        if dtype == "fp32":
            for i, ref in outs[r].items():
                torch.testing.assert_close(caps[r][i].double(), ref.detach(), rtol=5e-4, atol=5e-4)
            torch.testing.assert_close(got_logits, logits[r].detach(), rtol=5e-4, atol=5e-4)
            ref_l = float(ref_losses[r].detach())
            assert abs(float(losses[r]) - ref_l) <= 2e-4 * abs(ref_l) + 1e-4
            for name, prm in eng.model.named_parameters():
                torch.testing.assert_close(prm.grad.double(), grads[name], rtol=5e-3, atol=5e-5)
        else:
            for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
                got = got_logits if i == "logits" else caps[r][i].double()
                diff, scale = (got - ref.detach()).abs(), ref.detach().abs().max().item()
                assert diff.max().item() <= 0.25 * scale and diff.mean().item() <= 2e-2 * scale, (i, diff.max())
            ref_l = float(ref_losses[r].detach())
            assert abs(float(losses[r]) - ref_l) <= 2e-2 * abs(ref_l)
            for name, prm in eng.model.named_parameters():
                gref = grads[name]
                assert (prm.grad.double() - gref).norm() <= g_tol * gref.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype, n_layers)
    (1, "random", True, 1, "fp32", 3),
    (1, "random", False, 2, "bf16", 10),
    (2, "random", True, 1, "fp32", 9),
    (2, "metis", False, 2, "bf16", 4),
    (3, "metis", False, 1, "fp32", 3),
    (3, "random", True, 2, "fp32", 10),
    (4, "metis", False, 1, "fp32", 9),
    (4, "random", True, 1, "bf16", 3),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype,n_layers", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype, n_layers):
    """Synchronous training, dropout 0, 3 epochs with the engine's weights, every halo row poisoned with NaN before
    each epoch; depth 2 and 8 convolutions.  Per-layer outputs, logits, losses and reduced gradients (fc_in's included)
    against the fp64 restatement."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, 5, static_layer0=static0, n_linear=n_linear, dtype=dtype, n_layers=n_layers)
    tr = _trainer(layouts, a)
    caps = _hook_outputs(tr, a)
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        _check_engine(g, tr, layouts, a, caps, state, losses, dtype)


@pytest.mark.parametrize("metis", [False, True])
@pytest.mark.parametrize("n_parts", [1, 2, 3, 4])
def test_full_graph_equivalence(n_parts, metis):
    """Synchronous training: every rank's logits equal whole-graph GCNII in fp64 (P = 1 is the whole graph)."""
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(n_parts, metis)
    g1, lays1 = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, n_layers=5)
    tr = LocalTrainer(lays, a, LocalWorld(n_parts, DEV))
    state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
    _, ref_logits, _, ref_grads = restate_training(g1, lays1, state, a, torch.float32)
    tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    ref = torch.zeros(g.n_nodes, n_class, dtype=torch.float64, device=DEV)
    ref[lays1[0].inner_gid.long().to(DEV)] = ref_logits[0].detach()
    for e, lay in zip(tr.engines, lays):
        torch.testing.assert_close(e.last_logits.double(), ref[lay.inner_gid.long().to(DEV)], rtol=5e-4, atol=5e-4)
    for name, p in tr.engines[0].model.named_parameters():
        torch.testing.assert_close(p.grad.double(), ref_grads[name], rtol=5e-3, atol=5e-5)


@pytest.mark.parametrize("mode", [dict(), dict(feat_corr=True, grad_corr=True), dict(enable_pipeline=True),
                                  dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8)])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_exchange_modes_layer_parity(mode, dtype):
    """P = 3, synchronous and every exchange mode (--halo-bits 8 included): every convolution >= 2's output and input
    gradient equal the fp64 convolution applied to the rows it read and the h0 of its forward, with the upstream
    gradient it received.  Losses stay finite and fall."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _edges
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _args(g, 5, static_layer0=False, dtype=dtype, n_layers=5, **mode)
    if bits is not None:
        a.halo_bits = bits
    tr = _trainer(layouts, a)
    recs = [dict() for _ in tr.engines]

    def hook(mod, inp, out, r, i):
        rec = recs[r].setdefault(i, {})
        rec["x"], rec["out"], rec["h0"] = inp[1].detach().clone(), out.detach().clone(), inp[2].h0.detach().clone()
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
    tol = 5e-4 if dtype == "fp32" else 3e-2
    eye = torch.eye(a.n_hidden, dtype=torch.float64, device=DEV)
    n_checked, losses = 0, []
    for _ in range(6):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        losses.append(sum(float(l.item()) for l in tr.run_epoch()))
        torch.cuda.synchronize()
        for r, (eng, lay) in enumerate(zip(tr.engines, layouts)):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            c = c_glob[torch.cat([lay.inner_gid, lay.halo_gid]).long().to(DEV)]
            for i in range(1, n_graph):
                rec = recs[r][i]
                beta = math.log(a.gcnii_lambda / (i + 1) + 1)
                x = rec["x"].double().requires_grad_(True)
                agg = torch.zeros(lay.num_in, a.n_hidden, dtype=torch.float64, device=DEV).index_add(
                    0, rows, c[cols, None] * x[cols])
                s = (1 - a.gcnii_alpha) * c[:lay.num_in, None] * agg + a.gcnii_alpha * rec["h0"][:lay.num_in].double()
                w_eff = ((1 - beta) * eye + beta * state[f"layers.{i}.weight1"]).to(tdt).double()
                out = s @ w_eff + state[f"layers.{i}.bias"]
                scale = out.abs().max().item()
                assert (rec["out"].double() - out.detach()).abs().max().item() <= tol * scale + 1e-6, (r, i)
                out.backward(rec["gout"].double())
                if "gx" in rec:
                    gx = x.grad
                    gs = gx.abs().max().item()
                    assert (rec["gx"].double() - gx).abs().max().item() <= tol * gs + 1e-6, (r, i)
                    n_checked += 1
    assert n_checked > 0
    assert all(l == l for l in losses) and losses[-1] < losses[0]


# ------------------------------------------------------------------------------------------------ evaluation etc.
def test_eval_paths_and_checkpoint(tmp_path):
    """Whole-graph and partitioned evaluation agree; a checkpoint loads strictly into a fresh GCNII."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.train import LocalTrainer, create_model
    from pipegcn_b200.world import LocalWorld
    g, lays = _small(3)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dropout=0.5, n_layers=6)
    tr = LocalTrainer(lays, a, LocalWorld(3, DEV))
    for _ in range(3):
        tr.run_epoch()
    torch.cuda.synchronize()
    whole = _logits(tr.engines[0].model, EvalSet(g, DEV).val)
    parts = tr.predict()
    for z, lay in zip(parts, lays):
        torch.testing.assert_close(z.float(), whole[lay.inner_gid.long().to(DEV)], rtol=5e-4, atol=5e-4)
    tr.release_eval()
    path = tmp_path / "gcnii.pt"
    torch.save(tr.engines[0].model.state_dict(), path)
    fresh = create_model(tr.engines[0].layer_size, a)
    fresh.load_state_dict(torch.load(path), strict=True)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v.to(DEV), tr.engines[0].model.state_dict()[k])


def test_inductive_matches_rank0():
    """--inductive evaluation layouts: partitioned evaluation of the validation and test graphs equals whole-graph
    evaluation."""
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
    trainer = LocalTrainer(layouts, _args(gt, 16, n_hidden=32, n_layers=5, enable_pipeline=True), LocalWorld(P, DEV))
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
        torch.testing.assert_close(got, ref, rtol=5e-4, atol=5e-4)
        trainer.release_eval(lays)


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_cuda_graph_replay_equals_eager_bit_for_bit(dtype):
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit (no dropout: the
    trailing linear's eager dropout keys its masks with a host call counter)."""
    from tests.test_graphconv_gpu import _replay_runs
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True, n_layers=5)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def test_learns_planted_labels_at_depth():
    """16 planted classes (chance 1/16), fc_in + 8 convolutions + a linear: validation accuracy after 60 pipelined
    epochs on 2 partitions."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g = make_graph("small", planted_labels=True)
    lays = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    tr = LocalTrainer(lays, _args(g, 16, n_hidden=32, n_layers=9, dropout=0.2, enable_pipeline=True),
                      LocalWorld(2, DEV))
    for _ in range(60):
        tr.run_epoch()
    val, _ = tr.evaluate()
    tr.release_eval()
    print(f"gcnii (8 convolutions) planted-label validation accuracy {val:.4f}")
    assert val > 0.3, val
