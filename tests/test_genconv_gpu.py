"""Softmax-aggregation graph convolution (`--model genconv`) on the GPU: the GENConv kernels against fp64 (every
dispatch path, past the first wave, temperatures up to a saturated softmax, NaN sources, the keep mask, empty and
self-loop-only rows, guarded outputs, two launches giving the same bits), the layer's autograd against PyG's definition
in fp64, the engine against a restatement of partitioned training (sampled too), every exchange mode layer by layer,
evaluation, checkpoints, CUDA-graph replay with a learnt temperature, and free-running training."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from pipegcn_b200 import _C
from tests.test_genconv_cpu import TEMPS, pyg_forward
from tests.test_pna_gpu import _plan_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
E32 = 2.0 ** -24
EPS = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8}


# ------------------------------------------------------------------------------------------------ kernels
def _guarded(n, d, dtype, extra_rows=3, extra_cols=8):
    """[n, d] view of a NaN-filled buffer with extra rows and a row stride of round_up(d, 8) + extra_cols."""
    ld = (d + 7) // 8 * 8 + extra_cols
    buf = torch.full((n + extra_rows, ld), float("nan"), dtype=dtype, device=DEV)
    return buf[:n, :d], buf


def _xs(num_all, d, dtype, gen, scale=6.0, nan_row=None):
    from pipegcn_b200.graph import alloc_rows
    x = scale * torch.randn(num_all, d, generator=gen)
    x[1::7] = 0.5                                 # equal sources: all-equal rows
    z = alloc_rows(num_all, d, dtype, DEV)
    z.copy_(x)
    if nan_row is not None:
        z[nan_row, ::3] = float("nan")
    return z


def _keep(g, on, seed=5):
    if not on:
        return None
    gen = torch.Generator().manual_seed(seed)
    return (torch.rand(g.num_all - g.num_in, generator=gen) < 0.6).to(torch.uint8).to(DEV)


def _aggregate(g, xs, xd, t, keep, learn):
    """pg_genconv_aggregate into guarded buffers: (s, agg, lse, var) views and their full buffers."""
    from pipegcn_b200.ops import _ptr, _scratch_ld
    n, d = g.num_in, xs.shape[1]
    s, sb = _guarded(n, d, xs.dtype)
    (agg, ab), (lse, lb) = _guarded(n, d, torch.float32), _guarded(n, d, torch.float32)
    var, vb = _guarded(n, d, torch.float32) if learn else (None, None)
    parts = 4 if learn else 3
    scratch = g.fwd.scratch(parts * d)
    _C.check(_C.lib.pg_genconv_aggregate(C.byref(g.fwd.c), xs.data_ptr(), xs.stride(0), xd.data_ptr(), xd.stride(0),
                                         d, _C.dtype_code(xs.dtype), t.data_ptr(), _ptr(keep), g.num_in, s.data_ptr(),
                                         s.stride(0), agg.data_ptr(), agg.stride(0), lse.data_ptr(), lse.stride(0),
                                         _ptr(var), var.stride(0) if learn else 0, _ptr(scratch),
                                         _scratch_ld(parts * d), _C.stream_ptr()), "genconv")
    return (s, agg, lse, var), (sb, ab, lb, vb)


def _kept(rows, cols, num_in, keep):
    if keep is None:
        return rows, cols
    ok = (cols < num_in) | keep[(cols - num_in).clamp(min=0)].bool()
    return rows[ok], cols[ok]


def _softmax_ref(xs, rows, cols, n, t):
    """fp64 (agg, L, var, row max of m, kept degree) of the messages of the stored x_src."""
    x = xs.double()
    m = torch.where(x < 0, torch.zeros_like(x), x) + 1e-7
    d = x.shape[1]
    tm = t * m[cols]
    idx = rows[:, None].expand(-1, d)
    mx = torch.full((n, d), float("-inf"), dtype=torch.float64, device=DEV).scatter_reduce(0, idx, tm, "amax")
    deg = torch.bincount(rows, minlength=n)[:, None]
    has = deg > 0
    ms = torch.where(has & torch.isfinite(mx), mx, torch.zeros_like(mx))
    w = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, torch.exp(tm - ms[rows]))
    lse = ms + torch.log(w)
    a = torch.exp(tm - lse[rows])
    agg = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, a * m[cols])
    sq = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, a * m[cols] ** 2)
    mmax = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_reduce(0, rows, m[cols], "amax")
    nan = torch.zeros(n, d, dtype=torch.int64, device=DEV).index_add(0, rows, torch.isnan(m[cols]).long()) > 0
    return agg, lse, (sq - agg ** 2).clamp(min=0), mmax, deg, has, nan


def _check(got, ref, bound, nan, what):
    ok = ~nan
    err = (got.double() - ref).abs()
    assert torch.all((err <= bound)[ok]), (what, (err - bound)[ok].max().item())
    assert torch.all(torch.isnan(got[nan].float())), what


CASES = [(dt, d, seg) for dt in (torch.float32, torch.bfloat16) for d in (5, 64, 256, 602) for seg in (64, 512)]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dtype,d,seg_len", CASES)
def test_aggregate_vs_fp64(dtype, d, seg_len, masked):
    """Every temperature of TEMPS (|t m| past 100 at t = 20), with and without the var output."""
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(300, 120, seed=d, seg_len=seg_len)
    n = g.num_in
    gen = torch.Generator().manual_seed(d + 1)
    xs = _xs(g.num_all, d, dtype, gen, nan_row=int(cols[50]))
    xd = alloc_rows(n, d, dtype, DEV)
    xd.copy_(torch.randn(n, d, generator=gen))
    keep = _keep(g, masked)
    kr, kc = _kept(rows, cols, n, keep)
    for k, t in enumerate(TEMPS):
        learn = k % 2 == 0
        tt = torch.tensor([t], dtype=torch.float32, device=DEV)
        (s, agg, lse, var), bufs = _aggregate(g, xs, xd, tt, keep, learn)
        ragg, rl, rvar, mmax, deg, has, nan = _softmax_ref(xs, kr, kc, n, t)
        # per edge: t m and t m - L each rounded once (relative 2^-24 of |t| mmax and |L|), expf within 2 ulp, W and
        # A summed in fp32 (one rounding per edge), the rescales exact up to one rounding each
        big = abs(t) * mmax + rl.abs().nan_to_num(0, 0, 0) + 1
        tol_a = (8 * big + 6 * deg) * E32 * mmax + 1e-30
        z = torch.zeros_like(ragg)
        _check(torch.where(has, agg.double(), z), torch.where(has, ragg, z), tol_a, nan & has, (t, "agg"))
        _check(torch.where(has, lse.double(), z), torch.where(has, rl, z), (8 * big + 6 * deg) * E32, nan & has,
               (t, "lse"))
        if learn:
            _check(var, torch.where(has, rvar, z), (16 * big + 8 * deg) * E32 * mmax ** 2 + 1e-30, nan & has,
                   (t, "var"))
        ref_s = torch.where(has, ragg, z) + xd.double()
        _check(s, ref_s, tol_a + EPS[dtype] * ref_s.abs() + 1e-30, nan & has, (t, "S"))
        # no (kept) in-edge: agg = 0, L = -inf, var = 0, S = x_dst exactly
        e = ~has[:, 0]
        assert torch.all(agg[e] == 0) and torch.all(lse[e] == float("-inf")) and torch.equal(s[e], xd[e])
        if learn:
            assert torch.all(var[e] == 0)
        for full in bufs:                     # only columns [0, d) of rows [0, N_in) are written
            if full is not None:
                assert torch.all(torch.isnan(full[n:].float())) and torch.all(torch.isnan(full[:, d:].float()))
        if k == 0:                            # two launches: the same bits
            (s2, agg2, lse2, var2), _ = _aggregate(g, xs, xd, tt, keep, learn)
            for a1, a2 in ((s, s2), (agg, agg2), (lse, lse2), (var, var2)):
                assert torch.equal(a1.float().nan_to_num(7.0), a2.float().nan_to_num(7.0))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_aggregate_past_the_first_wave(dtype):
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(40_000, 5_000, seed=3, hubs=(3000, 1500, 700, 200, 90, 65, 40, 33))
    gen = torch.Generator().manual_seed(7)
    d, t = 64, 1.0
    xs = _xs(g.num_all, d, dtype, gen, scale=1.0)
    xd = alloc_rows(g.num_in, d, dtype, DEV)
    xd.zero_()
    (s, agg, lse, var), _ = _aggregate(g, xs, xd, torch.tensor([t], device=DEV), None, True)
    ragg, rl, rvar, mmax, deg, has, nan = _softmax_ref(xs, rows, cols, g.num_in, t)
    big = mmax + rl.abs().nan_to_num(0, 0, 0) + 1          # rows without in-edges: L = -inf, agg = 0
    assert torch.all((agg.double() - ragg).abs() <= (8 * big + 6 * deg) * E32 * mmax + 1e-30)
    assert torch.all((lse.double() - rl).abs()[has[:, 0]] <= ((8 * big + 6 * deg) * E32)[has[:, 0]])
    assert torch.all((var.double() - rvar).abs() <= (16 * big + 8 * deg) * E32 * mmax ** 2 + 1e-30)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 256, 602])
def test_backward_passes_vs_fp64(d, dtype, masked):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(300, 120, seed=d + 5, seg_len=64)
    n, n_all = g.num_in, g.num_all
    gen = torch.Generator().manual_seed(d)
    t = 1.7 if d != 64 else 20.0
    tt = torch.tensor([t], dtype=torch.float32, device=DEV)
    xs = _xs(n_all, d, dtype, gen, scale=2.0)
    xd = alloc_rows(n, d, dtype, DEV)
    xd.copy_(torch.randn(n, d, generator=gen))
    keep = _keep(g, masked)
    s, agg, lse, var = ops.genconv_aggregate(g.fwd, xs, xd, tt, keep, n, stats=True, learn_t=True)
    gs = alloc_rows(n, d, torch.float32, DEV)
    gs.copy_(torch.randn(n, d, generator=gen))
    q, gst, dt = ops.genconv_bwd_dst(gs, agg, tt, var, dtype=dtype)
    # destination pass: Q bit for bit, g_S rounded once, dt against fp64
    assert torch.equal(q, tt * (gs * agg)) and torch.equal(gst.float(), gs.to(dtype).float())
    ref_dt = (gs.double() * var.double()).sum()
    assert abs(float(dt) - float(ref_dt)) <= 2 * E32 * abs(float(ref_dt)) + 1e-12 * float((gs.double() * var.double()).abs().sum())
    q2, _, dt2 = ops.genconv_bwd_dst(gs, agg, tt, var, dtype=dtype)
    assert torch.equal(q, q2) and torch.equal(dt, dt2)
    # source pass against fp64 sums of the kernel's own L, G, Q
    kr, kc = _kept(rows, cols, n, keep)
    m32 = torch.where(xs.float() < 0, torch.zeros_like(xs.float()), xs.float()) + 1e-7
    tm = (tt * m32).double()
    arg = tm[kc] - lse.double()[kr]
    e = torch.exp(arg)
    G, Q = gs.double()[kr], q.double()[kr]
    term = e * (G * (1 + tm[kc]) - Q)
    ref = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, kc, term)
    mag = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(
        0, kc, e * ((G * (1 + tm[kc])).abs() + Q.abs()) * (arg.abs() + tm[kc].abs() + 8))
    odeg = torch.bincount(kc, minlength=n_all)[:, None].double()
    pos = xs.double() > 0
    ref = torch.where(pos, ref, torch.zeros_like(ref))
    bound = (4 * odeg + 4) * E32 * mag + EPS[dtype] * ref.abs() + 1e-30
    dx = ops.genconv_bwd_src(g.bwd, xs, tt, lse, gs, q, keep, n)
    assert torch.all((dx.double() - ref).abs() <= bound), (dx.double() - ref).abs().max()
    assert torch.all(dx[~pos] == 0) and torch.all(dx[n_all - 5:] == 0)   # x <= 0, never-referenced sources
    if keep is not None:
        assert torch.all(dx[n + torch.nonzero(keep == 0)[:, 0]] == 0)     # unkept sources: exact zeros
    assert torch.equal(dx, ops.genconv_bwd_src(g.bwd, xs, tt, lse, gs, q, keep, n))
    # the identity form: + g_S on the inner rows, then the dropout backward, in the same store
    spec = ops.DropSpec(0.3, 77, None, 0)
    dxa = ops.genconv_bwd_src(g.bwd, xs, tt, lse, gs, q, keep, n, add=gs, drop=spec)
    plain = ops.genconv_bwd_src(g.bwd, xs, tt, lse, gs, q, keep, n, add=gs)
    ones = alloc_rows(n_all, d, dtype, DEV)
    ones.fill_(1)
    kept = ops.dropout_rows(ones, spec).float() > 0
    assert torch.all(dxa.float()[~kept] == 0)
    summed = ref + torch.cat([gs.double(), torch.zeros(n_all - n, d, dtype=torch.float64, device=DEV)])
    assert torch.all((plain.double() - summed).abs() <= bound + 2 * EPS[dtype] * summed.abs())
    if dtype == torch.float32:
        assert torch.equal(dxa, ops.dropout_rows(plain, spec))


# ------------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("learn_t", [False, True])
@pytest.mark.parametrize("d_in,d", [(24, 16), (64, 64), (300, 40)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("drop", [0.0, 0.3])
def test_layer_autograd_matches_pyg(d_in, d, dtype, drop, learn_t):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph, alloc_rows
    from pipegcn_b200.partition import _csr_from_pairs
    from tests.test_gat_gpu import _stored
    from tests.test_genconv_cpu import weights
    from tests.test_pna_cpu import graph_case
    h64, rows, cols, num_in = graph_case(seed=d_in, d=d_in)
    num_all = h64.shape[0]
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=4)
    ws, wd, w1, w2 = [w.float().to(DEV).requires_grad_(True) if w is not None else None
                      for w in weights(d_in, d, seed=d)]
    t = torch.tensor([0.9 if learn_t else -0.5], device=DEV).requires_grad_(learn_t)
    feat = alloc_rows(num_all, d_in, dtype, DEV)
    feat.copy_(h64)
    feat.requires_grad_(True)
    spec = ops.DropSpec(drop, 1234, None, 0) if drop > 0 else None
    out = ops.genconv_layer(feat, g, None, t, ws, wd, w1, w2, drop_bwd=spec)
    gout = torch.randn(num_in, d, generator=torch.Generator().manual_seed(3)).to(DEV).to(dtype)
    out.backward(gout)
    st = lambda x: _stored(x, dtype)
    leaves = [w.detach().double().requires_grad_(True) if w is not None else None for w in (ws, wd, w1, w2)]
    x64 = feat.detach().double().requires_grad_(True)
    t64 = t.detach().double()[0].requires_grad_(True)
    ref = pyg_forward(x64, rows.to(DEV), cols.to(DEV), num_in, t64,
                      *[st(w) if w is not None else None for w in leaves], store=st)
    ref.backward(gout.double())
    gh = x64.grad
    if spec is not None:
        ones = alloc_rows(num_all, d_in, dtype, DEV)
        ones.fill_(1)
        gh = gh * ops.dropout_rows(ones, spec).double()

    def close(got, want, name):
        got = got.detach().double()
        if dtype == torch.float32:
            assert (got - want).abs().max().item() <= 2e-3 * (want.abs().max().item() + 1e-12), name
        else:
            assert (got - want).norm() <= 3e-2 * want.norm() + 1e-9, (name, (got - want).norm(), want.norm())

    close(out, ref.detach(), "out")
    close(feat.grad, gh, "h")
    for name, w, leaf in zip(("w_src", "w_dst", "w1", "w2"), (ws, wd, w1, w2), leaves):
        if w is not None:
            close(w.grad, leaf.grad, name)
    if learn_t:
        close(t.grad[0], t64.grad, "t")
    else:
        assert t.grad is None


# ------------------------------------------------------------------------------------------------ engine
def _args(g, n_class=5, learn_t=True, t=0.7, **kw):
    from tests.test_boundary_sampling_gpu import _args as base
    extra = {k: kw.pop(k) for k in ("dtype", "cuda_graph") if k in kw}
    a = base(g, n_class, **kw)
    a.model, a.genconv_t = "genconv", t
    for k, v in extra.items():
        setattr(a, k, v)
    if learn_t:
        a.genconv_learn_t = True
    return a


def restate_training(layouts, masks, state, a, dtype):
    """Partitioned GENConv training in fp64 (PyG's definition): per rank the forward over its partition with the
    unkept halo sources absent, the loss and the reduced gradients, rounding to bf16 where the engine stores values."""
    from tests.test_gat_gpu import _edges, _stored
    n = sum(l.num_in for l in layouts)
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    st = lambda x: _stored(x, dtype)
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=DEV)
    for lay in layouts:
        H[lay.inner_gid.to(DEV)] = lay.feat.to(DEV).to(dtype).double()
    gr = []
    for r, lay in enumerate(layouts):
        keep = torch.ones(lay.num_all, dtype=torch.bool, device=DEV)
        if masks is not None:
            keep[lay.num_in:] = masks[r].to(DEV)
        rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
        ek = keep[cols]
        gr.append(dict(gid=torch.cat([lay.inner_gid, lay.halo_gid]).to(DEV), rows=rows[ek], cols=cols[ek],
                       inner=lay.inner_gid.to(DEV), num_in=lay.num_in))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                p = f"layers.{i}."
                w = [st(params[p + k]) if p + k in params else None
                     for k in ("lin_src.weight", "lin_dst.weight", "mlp.lins.0.weight", "mlp.lins.1.weight")]
                t = params.get(p + "aggr_module.t", torch.tensor([a.genconv_t], dtype=torch.float64, device=DEV))
                out = pyg_forward(st(H[q["gid"]]), q["rows"], q["cols"], q["num_in"], t.float().double()[0] if
                                  p + "aggr_module.t" not in params else t[0], *w, store=st)
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
    tol, gtol = (2e-3, 1e-2) if dtype == "fp32" else (6e-2, 0.25)
    for r, eng in enumerate(tr.engines):
        got_logits = eng.last_logits.double()
        assert torch.isfinite(got_logits).all()
        for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
            got = got_logits if i == "logits" else caps[r][i].double()
            assert (got - ref.detach()).abs().max().item() <= tol * ref.detach().abs().max().item() + 1e-6, (r, i)
        ref_l = float(ref_losses[r].detach())
        assert abs(float(losses[r]) - ref_l) <= tol * abs(ref_l) + 1e-4
        for name, prm in eng.model.named_parameters():
            if dtype == "bf16" and name.endswith("aggr_module.t"):
                # dt = sum g_S var cancels: its bf16 error scales with sum |g_S| var, not with |dt|
                # (test_layer_autograd_matches_pyg checks it in bf16 at the layer)
                continue
            gref = grads[name]
            assert (prm.grad.double() - gref).norm() <= gtol * gref.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype, learnt t)
    (1, "random", True, 0, "fp32", True),
    (1, "random", False, 1, "bf16", True),
    (2, "random", True, 1, "fp32", True),
    (2, "metis", False, 0, "bf16", True),
    (3, "metis", False, 0, "fp32", True),
    (3, "random", True, 1, "bf16", True),
    (4, "metis", True, 1, "fp32", True),
    (4, "random", False, 0, "fp32", True),
    (2, "metis", True, 0, "fp32", False),
    (3, "random", False, 1, "bf16", False),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype,learn_t", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype, learn_t):
    """Synchronous training with a learnt or constant t, dropout 0, 3 epochs, every halo row poisoned with NaN before
    each epoch.  Widths 20 -> 16 -> 16 -> 5: layer 0 and a last graph layer have lin_src / lin_dst, layer 1 has none."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, static_layer0=static0, n_linear=n_linear, learn_t=learn_t)
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
    """Boundary-node sampling: unkept halo sources are absent from every softmax, unkept rows are poisoned with NaN."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, static_layer0=static0, sampling_rate=p)
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


_MODES = [dict(enable_pipeline=True), dict(feat_corr=True, grad_corr=True),
          dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8),
          dict(enable_pipeline=True, halo_bits=8)]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", _MODES)
def test_exchange_modes_layer_parity(mode, dtype):
    """P = 3, dropout 0, learnt t: every graph layer >= 1's output and input gradient equal PyG's layer in fp64 applied
    to the [inner | halo] rows it read (the stale, corrected or quantised halo rows the exchange delivered) with the
    upstream gradient it received."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _edges, _stored
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _args(g, static_layer0=False, **mode)
    a.dtype = dtype
    if bits is not None:
        a.halo_bits = bits
    tr = _trainer(layouts, a)
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    recs = [dict() for _ in tr.engines]

    def keep(rec, key, t):
        # after the first epoch into the same buffers: no allocation inside a synchronous LocalWorld epoch
        if key in rec and rec[key].shape == t.shape:
            rec[key].copy_(t)
        else:
            rec[key] = t.detach().clone()

    def hook(mod, inp, out, r, i):
        rec = recs[r].setdefault(i, {})
        keep(rec, "x", inp[1].detach())
        keep(rec, "out", out.detach())
        rec["has_gx"] = False
        out.register_hook(lambda gr: keep(rec, "gout", gr))
        if inp[1].requires_grad:
            def on_gx(gr, rec=rec):
                keep(rec, "gx", gr)
                rec["has_gx"] = True
            inp[1].register_hook(on_gx)

    n_graph = a.n_layers - a.n_linear
    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:n_graph]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: hook(mod, inp, out, r, i))

    def close(got, ref):
        if dtype == "fp32":
            return (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-6
        return (got - ref).norm().item() <= 5e-2 * ref.norm().item() + 1e-6

    st = lambda x: _stored(x, tdt)
    n_checked, losses = 0, []
    for _ in range(5):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        torch.cuda.synchronize()
        losses.append(sum(float(l.item()) for l in tr.run_epoch()))
        torch.cuda.synchronize()
        for r, lay in enumerate(layouts):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            for i in range(1, n_graph):
                rec, p = recs[r][i], f"layers.{i}."
                x = rec["x"].double().requires_grad_(True)
                w = [st(state[p + k]) if p + k in state else None
                     for k in ("lin_src.weight", "lin_dst.weight", "mlp.lins.0.weight", "mlp.lins.1.weight")]
                out = pyg_forward(x, rows, cols, lay.num_in, state[p + "aggr_module.t"][0], *w, store=st)
                assert close(rec["out"].double(), out.detach()), (r, i)
                out.backward(rec["gout"].double())
                if rec["has_gx"]:
                    assert close(rec["gx"].double(), x.grad), (r, i)
                    n_checked += 1
    assert n_checked > 0
    assert all(l == l for l in losses) and losses[-1] < losses[0]


# ------------------------------------------------------------------------------------------------ evaluation etc.
@pytest.mark.parametrize("n_hidden,dtype,learn_t", [(16, "fp32", True), (10, "fp32", False), (12, "bf16", True)])
def test_single_partition_logits_equal_full_graph_eval(n_hidden, dtype, learn_t):
    """Whole-graph evaluation hands the square middle layer the contiguous [N, d] rows of F.layer_norm when the fused
    LayerNorm epilogue does not take the width (d = 10 in fp32, 12 in bf16): unaligned rows the layer must pad."""
    from pipegcn_b200.train import create_model
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _full_logits, _scatter
    g, layouts = _layouts("tiny", 1)
    a = _args(g, n_hidden=n_hidden, dtype=dtype, learn_t=learn_t)
    tr = _trainer(layouts, a)
    tr.run_epoch()
    eng = tr.engines[0]
    # the weights the next epoch's forward uses, in the engine's activation dtype
    weights = create_model(eng.layer_size, a, dtype=eng.dtype).to(DEV)
    weights.load_state_dict(eng.model.state_dict())
    tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    got = _scatter(layouts, [eng.last_logits], g.n_nodes)
    ref = _full_logits(g, weights, eng.dtype)
    if dtype == "fp32":
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
    else:       # the same bf16 roundings, sums in a relabelled order
        assert torch.isfinite(ref).all() and (got - ref).norm() <= 2e-2 * ref.norm()


@pytest.mark.parametrize("learn_t", [False, True])
@pytest.mark.parametrize("d,dtype", [(10, torch.float32), (12, torch.bfloat16), (20, torch.float32)])
def test_layer_takes_contiguous_unaligned_rows(d, dtype, learn_t):
    """The identity form (d_in == d) on a contiguous [num_all, d] input whose rows are not 16-byte vectors: output and
    gradients equal those of the same values in padded rows."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph, alloc_rows
    from pipegcn_b200.partition import _csr_from_pairs
    from tests.test_genconv_cpu import weights
    from tests.test_pna_cpu import graph_case
    h64, rows, cols, num_in = graph_case(seed=d, d=d)
    num_all = h64.shape[0]
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=4)
    _, _, w1, w2 = [w.float().to(DEV) if w is not None else None for w in weights(d, d, seed=d)]
    gout = torch.randn(num_in, d, generator=torch.Generator().manual_seed(3)).to(DEV).to(dtype)
    runs = []
    for padded in (True, False):
        feat = alloc_rows(num_all, d, dtype, DEV) if padded else torch.empty(num_all, d, dtype=dtype, device=DEV)
        feat.copy_(h64)
        assert padded or feat.stride(0) == d
        feat.requires_grad_(True)
        t = torch.tensor([0.9], device=DEV).requires_grad_(learn_t)
        ws = [w.clone().requires_grad_(True) for w in (w1, w2)]
        out = ops.genconv_layer(feat, g, None, t, None, None, *ws)
        out.backward(gout)
        runs.append([out.detach(), feat.grad, ws[0].grad, ws[1].grad] + ([t.grad] if learn_t else []))
        with torch.no_grad():
            runs[-1].append(ops.genconv_layer(feat.detach(), g, None, t, None, None, *ws))
    for x, y in zip(*runs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("P,learn_t", [(2, True), (4, True), (2, False)])
def test_eval_paths_and_checkpoint(P, learn_t, tmp_path):
    """Partitioned evaluation equals whole-graph evaluation on rank 0; a checkpoint carries every layer's learnt t (a
    constant t is not in it) and loads strictly into a fresh model that evaluates the same."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.train import LocalTrainer, create_model
    from pipegcn_b200.world import LocalWorld
    from tests.test_graphconv_gpu import _small
    g, lays = _small(P)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dropout=0.5, enable_pipeline=True, learn_t=learn_t)
    tr = LocalTrainer(lays, a, LocalWorld(P, DEV))
    for _ in range(3):
        tr.run_epoch()
    torch.cuda.synchronize()
    model = tr.engines[0].model
    if learn_t:
        assert model.layers[0].aggr_module.t.item() != a.genconv_t      # t is learnt
    else:
        t32 = torch.tensor(a.genconv_t, dtype=torch.float32).item()
        assert all(layer.t_const.item() == t32 for layer in model.layers[:model.n_graph_layers])
    whole = _logits(model, EvalSet(g, DEV).val)
    parts = tr.predict()
    for z, lay in zip(parts, lays):
        torch.testing.assert_close(z.float(), whole[lay.inner_gid.long().to(DEV)], rtol=5e-4, atol=5e-4)
    tr.release_eval()
    path = tmp_path / "genconv.pt"
    torch.save(model.state_dict(), path)
    sd = torch.load(path)
    assert all((f"layers.{i}.aggr_module.t" in sd) == learn_t for i in range(model.n_graph_layers))
    assert not any("t_const" in k for k in sd)
    fresh = create_model(tr.engines[0].layer_size, a).to(DEV)
    fresh.load_state_dict(sd, strict=True)
    assert torch.equal(fresh.layers[1].temperature(), model.layers[1].temperature())
    assert torch.equal(_logits(fresh, EvalSet(g, DEV).val), whole)


def test_inductive_matches_rank0():
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
    trainer = LocalTrainer(layouts, _args(gt, 16, n_hidden=32, enable_pipeline=True), LocalWorld(P, DEV))
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
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit, with a learnt t
    that changes every epoch: the kernels read t from the device."""
    from tests.test_graphconv_gpu import _replay_runs, _small
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    assert len(r1) >= 3
    names = [n for n, _ in _named(a, lays[0])]
    ti = [k for k, n in enumerate(names) if n.endswith("aggr_module.t")]
    assert ti
    ts = [tuple(float(p[k]) for k in ti) for _, _, p in r1]
    assert len(set(ts)) == len(ts)                                   # t changes between the replays
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def _named(a, lay):
    from pipegcn_b200.partition import get_layer_size
    from pipegcn_b200.train import create_model
    return list(create_model(get_layer_size(a.n_feat, a.n_hidden, a.n_class, a.n_layers), a).named_parameters())


def test_learns_planted_labels():
    """16 planted classes (chance 1/16): validation accuracy after 40 pipelined epochs on 2 partitions."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g = make_graph("small", planted_labels=True)
    lays = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    tr = LocalTrainer(lays, _args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True), LocalWorld(2, DEV))
    for _ in range(40):
        tr.run_epoch()
    val, _ = tr.evaluate()
    tr.release_eval()
    print(f"genconv planted-label validation accuracy {val:.4f}")
    assert val > 0.3
