"""Gaussian mixture model convolution (`--model monet`) on the GPU: the four gathers of csrc/monet.cu and their mixture
gradients against fp64, their determinism and argument checks, the layer autograd of both orders against DGL's
definition, and the engine (partitioned training, exchange modes, evaluation, checkpoints, `--inductive`, CUDA-graph
replay, learning)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from pipegcn_b200 import _C
from tests.test_monet_cpu import dgl_forward, mixture_weights, pseudo_coords
from tests.test_pna_gpu import _plan_graph
from tests.test_resgated_gpu import _hub_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
PARAMS = ("fc.weight", "mu", "inv_sigma", "bias")


def _mix(k, seed, isg=2.0):
    gen = torch.Generator().manual_seed(seed)
    mu = (0.5 + 0.3 * torch.randn(k, 2, generator=gen)).to(DEV)
    inv_sigma = (isg * (0.5 + torch.rand(k, 2, generator=gen))).to(DEV)
    return mu.contiguous(), inv_sigma.contiguous()


def _setup(g, seed):
    """Random c in (0.2, 1] for every row (set as the owners' values) and the fp64 edge data of the plan."""
    gen = torch.Generator().manual_seed(seed)
    c = (0.2 + 0.8 * torch.rand(g.num_all, generator=gen)).to(DEV)
    g.set_sym_norm(c.contiguous())
    return c.double()


def _rows(n, d, dtype, seed, scale=1.0):
    from pipegcn_b200.graph import alloc_rows
    gen = torch.Generator().manual_seed(seed)
    x = alloc_rows(n, d, dtype, DEV)
    torch.as_strided(x, (n, x.stride(0)), (x.stride(0), 1)).fill_(float("nan"))   # the row pads: never read as data
    x.copy_((scale * torch.randn(n, d, generator=gen)).to(DEV))
    return x


def _mask(like, spec):
    """The dropout key's mask over rows shaped like `like`, as fp64 0 or 1 / (1 - p) with the fp32 scale the kernels
    multiply by (a bf16 mask would round it)."""
    from pipegcn_b200 import ops
    ones = _rows(like.shape[0], like.shape[1], like.dtype, 0)
    ones.fill_(1)
    scale = float(1.0 / (1.0 - torch.tensor(spec.p, dtype=torch.float32)))
    return (ops.dropout_rows(ones, spec) != 0).double() * scale


def _within(got, ref, bound, tol, what):
    err = (got.double() - ref).abs()
    assert torch.isfinite(got).all(), what
    assert (err <= tol * bound + 1e-30).all(), (what, (err - tol * bound).max().item())


def _slices(t, k, sl, d):
    return t.reshape(t.shape[0], -1)[:, :k * sl].reshape(t.shape[0], k, sl)[:, :, :d]


def _check_kernels(g, rows, cols, d, dtype, k, seed):
    from pipegcn_b200 import ops
    c = _setup(g, seed)
    mu, isg = _mix(k, seed)
    n_in, n_all = g.num_in, g.num_all
    w = mixture_weights(pseudo_coords(c, rows, cols), mu.double(), isg.double())        # [E, K]
    rd = 1.0 / torch.bincount(rows, minlength=n_in).clamp(min=1).double()
    eps = 2.0 ** -24 if dtype == torch.float32 else 2.0 ** -8
    acc_tol = 2e-5                                     # fp32 sums of at most 700 terms
    sl = ops.monet_slice(d, dtype)
    bias = torch.randn(d, device=DEV)

    def out_tol(ref, bound):
        return eps * ref.abs() + acc_tol * bound

    # aggregate first, forward: A[v][k] = rd_v sum_u w_k x_u
    x = _rows(n_all, d, dtype, seed + 1)
    xd = x.double()
    A = ops.monet_agg_k(g, x, mu, isg)
    ref = torch.zeros(n_in, k, d, dtype=torch.float64, device=DEV).index_add(0, rows, w[:, :, None] * xd[cols][:, None])
    bnd = torch.zeros_like(ref).index_add(0, rows, w[:, :, None] * xd[cols][:, None].abs())
    ref, bnd = ref * rd[:, None, None], bnd * rd[:, None, None]
    got = A.reshape(n_in, k, sl)
    assert torch.all(got[:, :, d:] == 0)
    _within(got[:, :, :d], ref, (eps * ref.abs() + acc_tol * bnd) / 1.0, 1.0, "agg_k")

    # transform first, forward: out[v] = rd_v sum_u sum_k w_k z_u[k] + bias
    z = _rows(n_all, k * sl, dtype, seed + 2)
    zd = _slices(z, k, sl, d).double()
    out = ops.monet_agg_sum(g, z, d, mu, isg, bias)
    term = (w[:, :, None] * zd[cols]).sum(1)
    ref = torch.zeros(n_in, d, dtype=torch.float64, device=DEV).index_add(0, rows, term) * rd[:, None] + bias.double()
    bnd = torch.zeros(n_in, d, dtype=torch.float64, device=DEV).index_add(
        0, rows, (w[:, :, None] * zd[cols].abs()).sum(1)) * rd[:, None] + bias.double().abs()
    _within(out, ref, out_tol(ref, bnd), 1.0, "agg_sum")

    # mixture gradient of s_k(e) from per-edge dot products dots [E, K]
    def mix_ref(dots):
        e = pseudo_coords(c, rows, cols)
        diff = e[:, None, :] - mu.double()[None]
        a = dots * w * rd[rows][:, None]
        dmu = (a[:, :, None] * diff).sum(0) * isg.double() ** 2
        dinv = -(a[:, :, None] * diff ** 2).sum(0) * isg.double()
        bmu = (a.abs()[:, :, None] * diff.abs()).sum(0) * isg.double() ** 2
        binv = (a.abs()[:, :, None] * diff ** 2).sum(0) * isg.double()
        return dmu, dinv, bmu, binv

    # transform first, backward over the CSC: dz[u][k] = sum_v w_k rd_v G_v
    G = _rows(n_in, d, dtype, seed + 3)
    Gd = G.double()
    zb = _rows(n_all, k * sl, dtype, seed + 4)
    zbd = _slices(zb, k, sl, d).double()
    dz, dmu, dinv = ops.monet_bwd_k(g, G, zb, mu, isg)
    coef = (w * rd[rows][:, None])[:, :, None]
    ref = torch.zeros(n_all, k, d, dtype=torch.float64, device=DEV).index_add(0, cols, coef * Gd[rows][:, None])
    bnd = torch.zeros_like(ref).index_add(0, cols, coef * Gd[rows][:, None].abs())
    got = dz.reshape(n_all, k, sl)
    assert torch.all(got[:, :, d:] == 0)
    _within(got[:, :, :d], ref, eps * ref.abs() + acc_tol * bnd, 1.0, "bwd_k")
    dots = (Gd[rows][:, None, :] * zbd[cols]).sum(-1)
    rmu, rinv, bmu, binv = mix_ref(dots)
    _within(dmu, rmu, 1e-4 * bmu + 1e-6 * bmu.max(), 1.0, "bwd_k dmu")
    _within(dinv, rinv, 1e-4 * binv + 1e-6 * binv.max(), 1.0, "bwd_k dinv")
    dz2, dmu2, dinv2 = ops.monet_bwd_k(g, G, zb, mu, isg)
    assert torch.equal(dz2, dz) and torch.equal(dmu2, dmu) and torch.equal(dinv2, dinv)

    # aggregate first, backward over the CSC: dh[u] = sum_v rd_v sum_k w_k dA_v[k], with and without dropout
    dA = _rows(n_in, k * sl, dtype, seed + 5)
    dAd = _slices(dA, k, sl, d).double()
    h = _rows(n_all, d, dtype, seed + 6)
    hd = h.double()
    term = (coef * dAd[rows]).sum(1)
    ref = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, cols, term)
    bnd = torch.zeros_like(ref).index_add(0, cols, (coef * dAd[rows].abs()).sum(1))
    dh, dmu, dinv = ops.monet_bwd_sum(g, dA, h, mu, isg)
    _within(dh, ref, eps * ref.abs() + acc_tol * bnd, 1.0, "bwd_sum")
    dots = (dAd[rows] * hd[cols][:, None, :]).sum(-1)
    rmu, rinv, bmu, binv = mix_ref(dots)
    _within(dmu, rmu, 1e-4 * bmu + 1e-6 * bmu.max(), 1.0, "bwd_sum dmu")
    _within(dinv, rinv, 1e-4 * binv + 1e-6 * binv.max(), 1.0, "bwd_sum dinv")
    spec = ops.DropSpec(0.3, 1234)
    dhd, dmu_d, dinv_d = ops.monet_bwd_sum(g, dA, h, mu, isg, spec)
    mask = _mask(dh, spec)
    assert torch.equal(dmu_d, dmu) and torch.equal(dinv_d, dinv)
    assert torch.equal(dhd, (dh.float() * mask.float()).to(dtype)) or dtype == torch.bfloat16
    _within(dhd, ref * mask, (eps * ref.abs() + acc_tol * bnd) * mask, 1.0, "bwd_sum drop")
    dh2, dmu2, dinv2 = ops.monet_bwd_sum(g, dA, h, mu, isg)
    assert torch.equal(dh2, dh) and torch.equal(dmu2, dmu) and torch.equal(dinv2, dinv)


@pytest.mark.parametrize("d", [3, 64, 300])
@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernels_vs_fp64(dtype, k, d):
    """Every 16-byte vector width (4 fp32 or 8 bf16 elements, partial last vectors at d = 3 and 300), on a graph
    whose CSR and CSC both have long rows split into segments and single long rows, rows without in-edges and
    self-loop-only rows."""
    g, rows, cols = _hub_graph(400, 160, seed=k + d, seg_len=64)
    assert g.fwd.n_seg > 0 and g.bwd.n_seg > 0 and g.bwd.n_long > 0
    _check_kernels(g, rows, cols, d, dtype, k, seed=7 * k + d)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernels_past_the_first_wave(dtype):
    g, rows, cols = _plan_graph(60000, 9000, seed=3, seg_len=64)
    assert g.fwd.n_chunks > 8 * 132 * 4 and g.bwd.n_chunks > 8 * 132 * 4
    _check_kernels(g, rows, cols, 40, dtype, 3, seed=11)


def test_underflowing_weights_and_a_row_with_no_weight():
    """inv_sigma = 2000: almost every weight is exactly 0 in fp32, so is every weight of most rows; the outputs are then
    exact zeros (or the bias) and the mixture gradients stay finite."""
    from pipegcn_b200 import ops
    g, rows, cols = _hub_graph(400, 160, seed=1, seg_len=64)
    c = _setup(g, 2)
    mu = torch.stack([c[cols[:3]], c[rows[:3]]], 1).float().contiguous()
    isg = torch.full((3, 2), 2000.0, device=DEV)
    w = mixture_weights(pseudo_coords(c, rows, cols), mu.double(), isg.double())
    assert (w.float() == 0).any() and (w.float() > 0).any()
    x = _rows(g.num_all, 16, torch.float32, 3)
    A = ops.monet_agg_k(g, x, mu, isg)
    row_w = torch.zeros(g.num_in, dtype=torch.float64, device=DEV).index_add(0, rows, w.sum(1))
    assert (row_w == 0).any()
    assert torch.all(A[row_w == 0] == 0)
    G = _rows(g.num_in, 16, torch.float32, 4)
    dA = _rows(g.num_in, 3 * 16, torch.float32, 5)
    for got in (ops.monet_bwd_k(g, G, _rows(g.num_all, 48, torch.float32, 6), mu, isg),
                ops.monet_bwd_sum(g, dA, x, mu, isg)):
        assert all(torch.isfinite(t).all() for t in got)


def test_entry_points_refuse_bad_arguments():
    from pipegcn_b200 import ops
    g, _, _ = _plan_graph(300, 100, seed=0)
    _setup(g, 0)
    x = _rows(g.num_all, 8, torch.float32, 0)
    out = _rows(g.num_in, 9 * 8, torch.float32, 1)
    c, rd = g.sym_norm(), g.inv_row_degrees()
    mu9, isg9 = _mix(9, 0)
    sc = g.fwd.scratch(9 * 8)

    def agg_k(k, slice_=8, ldo=None, cptr=c.data_ptr(), xptr=x.data_ptr()):
        return _C.lib.pg_monet_agg_k(C.byref(g.fwd.c), xptr, x.stride(0), 8, _C.PG_F32, k, cptr, rd.data_ptr(),
                                     mu9.data_ptr(), isg9.data_ptr(), out.data_ptr(),
                                     out.stride(0) if ldo is None else ldo, slice_, ops._ptr(sc), 9 * 8,
                                     _C.stream_ptr())
    assert agg_k(8) == _C.PG_OK
    assert agg_k(9) != _C.PG_OK and "mixture kernels" in _C.lib.pg_last_error().decode()
    assert agg_k(0) != _C.PG_OK
    assert agg_k(3, slice_=4) != _C.PG_OK                       # slices shorter than the rows
    assert agg_k(8, ldo=7 * 8) != _C.PG_OK                      # output rows shorter than 8 slices
    assert agg_k(3, cptr=None) != _C.PG_OK and "null" in _C.lib.pg_last_error().decode()
    assert agg_k(3, xptr=None) != _C.PG_OK
    G = _rows(g.num_in, 8, torch.float32, 2)
    z, dz = _rows(g.num_all, 24, torch.float32, 3), _rows(g.num_all, 24, torch.float32, 4)
    dmu = torch.empty(3, 2, device=DEV)
    rc = _C.lib.pg_monet_bwd_k(C.byref(g.bwd.c), G.data_ptr(), G.stride(0), z.data_ptr(), z.stride(0), 8, 8,
                               _C.PG_F32, 3, c.data_ptr(), rd.data_ptr(), mu9.data_ptr(), isg9.data_ptr(),
                               dz.data_ptr(), dz.stride(0), ops._ptr(g.bwd.scratch(24)), 24, None, 0,
                               dmu.data_ptr(), dmu.data_ptr(), _C.stream_ptr())
    assert rc != _C.PG_OK and "workspace" in _C.lib.pg_last_error().decode()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ layer autograd
@pytest.mark.parametrize("d_in,d_out,k", [(24, 16, 3), (64, 8, 3), (300, 40, 1), (20, 5, 8), (16, 16, 1)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("drop", [0.0, 0.3])
def test_layer_autograd_matches_dgl(d_in, d_out, k, dtype, drop):
    """Both orders (d_in <= K d_out aggregates first) against autograd through DGL's definition in fp64, with the
    dropout backward of the layer input fused (`drop_bwd`)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.module.layer import MoNetLayer
    g, rows, cols = _plan_graph(700, 200, seed=d_in + k)
    c = _setup(g, k)
    torch.manual_seed(d_in)
    layer = MoNetLayer(d_in, d_out, k).to(DEV)
    with torch.no_grad():
        layer.mu.copy_(0.5 + 0.3 * torch.randn(k, 2))
        layer.inv_sigma.uniform_(0.5, 3.0)
        layer.bias.normal_()
    feat = _rows(g.num_all, d_in, dtype, 1).requires_grad_(True)
    spec = ops.DropSpec(drop, 77) if drop > 0 else None
    out = layer(g, feat, drop_bwd=spec)
    Gr = torch.randn(g.num_in, d_out, device=DEV)
    out.backward(Gr.to(out.dtype))
    st = (lambda t: t) if dtype == torch.float32 else (lambda t: t + (t.to(dtype).double() - t).detach())
    leaves = [p.detach().double().clone().requires_grad_(True) for p in (layer.fc.weight, layer.mu, layer.inv_sigma,
                                                                         layer.bias)]
    x = feat.detach().double().clone().requires_grad_(True)
    ref = dgl_forward(x, rows, cols, g.num_in, c, st(leaves[0]), leaves[1], leaves[2], leaves[3])
    ref.backward(Gr.to(dtype).double())
    gx = x.grad
    if spec is not None:
        gx = gx * _mask(feat, spec)

    def close(got, want, name):
        got = got.detach().double()
        if dtype == torch.float32:
            assert (got - want).abs().max().item() <= 2e-3 * (want.abs().max().item() + 1e-12), name
        else:
            assert (got - want).norm() <= 3e-2 * want.norm() + 1e-9, (name, (got - want).norm(), want.norm())

    close(out, ref.detach(), "out")
    close(feat.grad, gx, "h")
    for name, p, leaf in zip(PARAMS, (layer.fc.weight, layer.mu, layer.inv_sigma, layer.bias), leaves):
        close(p.grad, leaf.grad, name)


# ------------------------------------------------------------------------------------------------ engine
def _args(g, n_class=5, **kw):
    from tests.test_boundary_sampling_gpu import _args as base
    extra = {k: kw.pop(k) for k in ("dtype", "cuda_graph") if k in kw}
    a = base(g, n_class, **kw)
    a.model = "monet"
    for k, v in extra.items():
        setattr(a, k, v)
    return a


def _global_c(layouts, n):
    rows = []
    for lay in layouts:
        r = torch.repeat_interleave(torch.arange(lay.num_in), (lay.indptr[1:] - lay.indptr[:-1]).long())
        rows.append(lay.inner_gid.long()[r])
    return (torch.bincount(torch.cat(rows), minlength=n).clamp(min=1).double() ** -0.5).to(DEV)


def _layer_ref(params, p, x, rows, cols, num_in, c, st):
    return dgl_forward(x, rows, cols, num_in, c, st(params[p + "fc.weight"]), params[p + "mu"],
                       params[p + "inv_sigma"], params[p + "bias"])


def restate_training(layouts, state, a, dtype):
    """Partitioned MoNet training in fp64 (DGL's definition): per rank the forward over its partition with the global
    pseudo-coordinates, the loss and the reduced gradients, rounding to bf16 where the engine stores values."""
    from tests.test_gat_gpu import _edges, _stored
    n = sum(l.num_in for l in layouts)
    cg = _global_c(layouts, n)
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point()}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    st = lambda x: _stored(x, dtype)
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=DEV)
    for lay in layouts:
        H[lay.inner_gid.to(DEV)] = lay.feat.to(DEV).to(dtype).double()
    gr = []
    for lay in layouts:
        rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).to(DEV).long()
        gr.append(dict(gid=gid, rows=rows, cols=cols, inner=lay.inner_gid.to(DEV), num_in=lay.num_in, c=cg[gid]))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, a.n_hidden if i < n_layers - 1 else a.n_class, dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                out = _layer_ref(params, f"layers.{i}.", st(H[q["gid"]]), q["rows"], q["cols"], q["num_in"], q["c"],
                                 st)
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


def _check_engine(tr, layouts, a, caps, state, losses, dtype):
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    outs, logits, ref_losses, grads = restate_training(layouts, state, a, tdt)
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
            gref = grads[name]
            assert (prm.grad.double() - gref).norm() <= gtol * gref.norm() + 1e-6, name


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype)
    (1, "random", True, 0, "fp32"),
    (1, "random", False, 1, "bf16"),
    (2, "random", True, 1, "fp32"),
    (2, "metis", False, 0, "bf16"),
    (3, "metis", False, 0, "fp32"),
    (3, "random", True, 1, "bf16"),
    (4, "metis", True, 1, "fp32"),
    (4, "random", False, 0, "bf16"),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype):
    """Synchronous training, dropout 0, 3 epochs, every halo row poisoned with NaN before each epoch.  The hidden
    layers aggregate first (16 <= 3 * 16) and the logit layer transforms first (16 > 3 * 5)."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, static_layer0=static0, n_linear=n_linear)
    a.dtype = dtype
    tr = _trainer(layouts, a)
    caps = _hook_outputs(tr, a)
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        _check_engine(tr, layouts, a, caps, state, losses, dtype)


_MODES = [dict(enable_pipeline=True), dict(feat_corr=True, grad_corr=True),
          dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8),
          dict(enable_pipeline=True, halo_bits=8)]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", _MODES)
def test_exchange_modes_layer_parity(mode, dtype):
    """P = 3, dropout 0: every graph layer >= 1's output and input gradient equal DGL's layer in fp64 applied to the
    [inner | halo] rows it read (the stale, corrected or quantised halo rows the exchange delivered) with the upstream
    gradient it received."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _edges, _stored
    g, layouts = _layouts("tiny", 3)
    cg = _global_c(layouts, g.n_nodes)
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
            c = cg[torch.cat([lay.inner_gid, lay.halo_gid]).to(DEV).long()]
            for i in range(1, n_graph):
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                out = _layer_ref(state, f"layers.{i}.", x, rows, cols, lay.num_in, c, st)
                assert close(rec["out"].double(), out.detach()), (r, i)
                out.backward(rec["gout"].double())
                if rec["has_gx"]:
                    assert close(rec["gx"].double(), x.grad), (r, i)
                    n_checked += 1
    assert n_checked > 0
    assert all(l == l for l in losses)


# ------------------------------------------------------------------------------------------------ evaluation etc.
@pytest.mark.parametrize("n_hidden,dtype", [(16, "fp32"), (10, "fp32"), (12, "bf16")])
def test_single_partition_logits_equal_full_graph_eval(n_hidden, dtype):
    from pipegcn_b200.train import create_model
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _full_logits, _scatter
    g, layouts = _layouts("tiny", 1)
    a = _args(g, n_hidden=n_hidden, dtype=dtype)
    tr = _trainer(layouts, a)
    tr.run_epoch()
    eng = tr.engines[0]
    weights = create_model(eng.layer_size, a, dtype=eng.dtype).to(DEV)
    weights.load_state_dict(eng.model.state_dict())
    tr.run_epoch(keep_logits=True)
    torch.cuda.synchronize()
    got = _scatter(layouts, [eng.last_logits], g.n_nodes)
    ref = _full_logits(g, weights, eng.dtype)
    if dtype == "fp32":
        torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)
    else:
        assert torch.isfinite(ref).all() and (got - ref).norm() <= 2e-2 * ref.norm()


@pytest.mark.parametrize("P", [2, 4])
def test_eval_paths_and_checkpoint(P, tmp_path):
    """Partitioned evaluation equals whole-graph evaluation on rank 0; a checkpoint loads strictly into a fresh model
    that evaluates the same."""
    from pipegcn_b200.evaluate import EvalSet, _logits
    from pipegcn_b200.train import LocalTrainer, create_model
    from pipegcn_b200.world import LocalWorld
    from tests.test_graphconv_gpu import _small
    g, lays = _small(P)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dropout=0.5, enable_pipeline=True)
    tr = LocalTrainer(lays, a, LocalWorld(P, DEV))
    for _ in range(3):
        tr.run_epoch()
    torch.cuda.synchronize()
    model = tr.engines[0].model
    whole = _logits(model, EvalSet(g, DEV).val)
    parts = tr.predict()
    for z, lay in zip(parts, lays):
        torch.testing.assert_close(z.float(), whole[lay.inner_gid.long().to(DEV)], rtol=5e-4, atol=5e-4)
    tr.release_eval()
    path = tmp_path / "monet.pt"
    torch.save(model.state_dict(), path)
    sd = torch.load(path)
    assert all(f"layers.{i}.{k}" in sd for i in range(model.n_graph_layers) for k in PARAMS)
    fresh = create_model(tr.engines[0].layer_size, a).to(DEV)
    fresh.load_state_dict(sd, strict=True)
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
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit, while Adam
    changes mu and inv_sigma every step (the kernels read them from device memory)."""
    from tests.test_graphconv_gpu import _replay_runs, _small
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    assert len(r1) >= 3
    from pipegcn_b200.train import create_model
    names = [n for n, _ in create_model([a.n_feat, a.n_hidden, a.n_hidden, n_class], a).named_parameters()]
    mixture = [j for j, n in enumerate(names) if n.endswith(("mu", "inv_sigma"))]
    assert mixture and not torch.equal(r1[0][2][mixture[0]], r1[-1][2][mixture[0]])
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def test_learns_planted_labels():
    """16 planted classes (chance 1/16): validation accuracy after 120 pipelined epochs on 2 partitions.  The labels
    are a linear map of the own and the neighbour-mean features; MoNet has no separate self weight and learns them more
    slowly than GraphSAGE-mean (0.298 on an H100 at this seed)."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g = make_graph("small", planted_labels=True)
    lays = build_layouts(g, random_partition(g.n_nodes, 2), 2)
    torch.manual_seed(0)
    tr = LocalTrainer(lays, _args(g, 16, n_hidden=32, dropout=0.2, enable_pipeline=True), LocalWorld(2, DEV))
    for _ in range(120):
        tr.run_epoch()
    val, _ = tr.evaluate()
    tr.release_eval()
    print(f"monet planted-label validation accuracy {val:.4f}")
    assert val > 0.2
