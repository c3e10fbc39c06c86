"""Principal neighbourhood aggregation (`--model pna`) on the GPU: the PNA kernels against fp64 (every dispatch path,
past the first wave, ties, NaN, all-equal, self-loop-only and empty rows, guarded outputs), the layer's autograd
against the fp64 restatement of tests/test_pna_cpu.py, the engine against a restatement of partitioned training,
evaluation, checkpoints, CUDA-graph replay and free-running training."""
import argparse

import pytest
import torch
import torch.nn.functional as F

from pipegcn_b200 import _C
from tests.test_pna_cpu import factorised_backward, factorised_forward, graph_case, scalers64

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8}


# ------------------------------------------------------------------------------------------------ kernels
def _plan_graph(num_in, num_halo, seed, hubs=(700, 200, 90, 65, 40, 33), seg_len=64):
    """(PartGraph, rows, cols in CSR order) with hub rows split into segments (seg_len), single rows of 33..seg_len
    entries, short multi-row chunks, rows without in-edges (10..13), self-loop-only rows (14..17) and never-referenced
    halo rows (the last 5)."""
    from pipegcn_b200.graph import PartGraph
    from pipegcn_b200.partition import _csr_from_pairs
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    deg = torch.randint(1, 12, (num_in,), generator=gen)
    deg[:len(hubs)] = torch.tensor(hubs)
    deg[10:14] = 0
    rows, cols = [], []
    for v in range(num_in):
        k = int(deg[v])
        if k == 0:
            continue
        src = [v] if 14 <= v < 18 else torch.randperm(num_all - 5, generator=gen)[:k].tolist()
        rows += [v] * len(src)
        cols += src
    rows, cols = torch.tensor(rows), torch.tensor(cols)
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=seg_len)
    r = torch.repeat_interleave(torch.arange(num_in), (indptr[1:] - indptr[:-1]).long())
    return g, r.to(DEV), indices.long().to(DEV)


def _zs(num_all, d, dtype, gen, ties=True, nan_row=None):
    from pipegcn_b200.graph import alloc_rows
    x = torch.randn(num_all, d, generator=gen).to(DEV)
    if ties:                                  # many equal values: exact ties of the extremes, all-equal rows
        x[::3] = x[::3].round()
        x[1::7] = 0.5
    z = alloc_rows(num_all, d, dtype, DEV)
    z.copy_(x)
    if nan_row is not None:
        z[nan_row, ::3] = float("nan")
    return z


def _extremes_ref(zs64, rows, cols, n, sign):
    """(value, source) of the per-column max (sign 1) or min (sign -1): the first source in CSR order on a tie, the
    first NaN source when there is one."""
    d = zs64.shape[1]
    x = sign * zs64[cols]
    isn = torch.isnan(x)
    fill = torch.full((n, d), float("-inf"), dtype=x.dtype, device=DEV)
    best = fill.scatter_reduce(0, rows[:, None].expand(-1, d), torch.where(isn, fill[:1].expand_as(x), x), "amax")
    has_nan = torch.zeros(n, d, dtype=torch.int64, device=DEV).index_add(0, rows, isn.long()) > 0
    hit = torch.where(has_nan[rows], isn, (x == best[rows]) & ~isn)
    e = torch.arange(cols.numel(), device=DEV)[:, None].expand(-1, d)
    big = torch.full((n, d), cols.numel(), dtype=torch.int64, device=DEV)
    first = big.scatter_reduce(0, rows[:, None].expand(-1, d), torch.where(hit, e, big[:1].expand_as(e)), "amin")
    deg = torch.bincount(rows, minlength=n)
    src = torch.where(deg[:, None] > 0, cols[first.clamp(max=cols.numel() - 1)], torch.full_like(first, -1))
    val = torch.where(has_nan, float("nan"), sign * best)
    return torch.where(deg[:, None] > 0, val, torch.zeros_like(val)), src


def _moments_ref(zs64, rows, cols, n):
    d = zs64.shape[1]
    deg = torch.bincount(rows, minlength=n).double()[:, None]
    s = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, zs64[cols])
    mu = s / deg.clamp(min=1)
    var = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, (zs64[cols] - mu[rows]) ** 2)
    amax = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_reduce(0, rows, zs64[cols].abs(), "amax")
    return mu, var / deg.clamp(min=1), amax, deg


def _aggregate_guarded(g, zs, zd, seg_pad=0, extra_rows=3):
    """pg_pna_aggregate into NaN-filled buffers with extra rows and (seg_pad) extra columns per part: returns the
    views and the full buffers."""
    from pipegcn_b200.ops import _ptr, _scratch_ld, pna_width
    n, d = g.num_in, zs.shape[1]
    w = pna_width(d) + seg_pad
    agg = torch.full((n + extra_rows, 4 * w + 8), float("nan"), dtype=zs.dtype, device=DEV)
    mv = torch.full((n + extra_rows, 2 * w), float("nan"), dtype=torch.float32, device=DEV)
    ar = torch.full((n + extra_rows, 2 * w), -7, dtype=torch.int32, device=DEV)
    scratch = g.fwd.scratch(6 * d)
    import ctypes as C
    _C.check(_C.lib.pg_pna_aggregate(C.byref(g.fwd.c), zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), d,
                                     _C.dtype_code(zs.dtype), agg.data_ptr(), agg.stride(0), w, mv.data_ptr(),
                                     mv[:, w:].data_ptr(), mv.stride(0), ar.data_ptr(), ar[:, w:].data_ptr(),
                                     ar.stride(0), _ptr(scratch), _scratch_ld(6 * d), _C.stream_ptr()), "pna")
    return agg, mv, ar, w


CASES = [(dt, d, seg) for dt in (torch.float32, torch.bfloat16) for d in (5, 64, 256, 602) for seg in (64, 512)]


@pytest.mark.parametrize("dtype,d,seg_len", CASES)
def test_aggregate_vs_fp64(dtype, d, seg_len):
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(300, 120, seed=d, seg_len=seg_len)
    gen = torch.Generator().manual_seed(d + 1)
    zs = _zs(g.num_all, d, dtype, gen, nan_row=int(cols[50]))
    zd = alloc_rows(g.num_in, d, torch.float32, DEV)
    zd.copy_(torch.randn(g.num_in, d, generator=gen).to(DEV))
    agg, mv, ar, w = _aggregate_guarded(g, zs, zd, seg_pad=8)
    n = g.num_in
    zs64 = zs.double()
    mx, ax = _extremes_ref(zs64, rows, cols, n, 1)
    mn, an = _extremes_ref(zs64, rows, cols, n, -1)
    assert torch.equal(ar[:n, :d], ax.int()) and torch.equal(ar[:n, w:w + d], an.int())
    mu, var, amax, deg = _moments_ref(zs64, rows, cols, n)
    kmu, kvar = mv[:n, :d].double(), mv[:n, w:w + d].double()
    nanrow = torch.isnan(mu)
    ok = ~nanrow
    e32 = 2.0 ** -24
    tol_mu = 4 * deg * e32 * amax + 1e-30
    tol_var = 16 * deg * e32 * amax ** 2 + 1e-30
    assert torch.all(((kmu - mu).abs() <= tol_mu)[ok]) and torch.all(torch.isnan(kmu[nanrow]))
    assert torch.all(((kvar - var).abs() <= tol_var)[ok]) and torch.all(torch.isnan(kvar[nanrow]))
    zd64 = zd.double()
    eps = EPS[dtype]
    parts = [agg[:n, k * w:k * w + d].double() for k in range(4)]
    empty = deg == 0                                            # no in-edges: agg = 0, zd not added
    refs = [torch.where(empty, 0.0, r + zd64) for r in (mu, mx, mn)]
    tols = [tol_mu, 0 * tol_mu, 0 * tol_mu]
    for got, ref, tol in zip(parts[:3], refs, tols):
        bound = tol + 1.01 * eps * ref.abs() + 1e-30        # bf16: fp32 sum, then one rounding to bf16
        assert torch.all(((got - ref).abs() <= bound) | (torch.isnan(got) & torch.isnan(ref))), (got - ref).abs().max()
    sig = torch.sqrt(var.clamp(min=0) + 1e-30)
    bound = torch.sqrt(tol_var) + 2 * eps * sig + 1e-14
    assert torch.all(((parts[3] - sig).abs() <= bound)[ok]) and torch.all(torch.isnan(parts[3][nanrow]))
    # rows without in-edges, self-loop-only rows, guards
    assert all(torch.all(p[10:14] == 0) for p in parts)
    assert torch.all(ar[10:14, :d] == -1) and torch.all(ar[10:14, w:w + d] == -1)
    assert torch.all(mv[14:18, w:w + d] == 0)                    # one source: var exactly 0
    for k in range(4):
        assert torch.all(torch.isnan(agg[:n, k * w + d:(k + 1) * w].float())), k
    assert torch.all(torch.isnan(agg[n:].float())) and torch.all(torch.isnan(agg[:, 4 * w:].float()))
    assert torch.all(torch.isnan(mv[n:])) and torch.all(ar[n:] == -7)
    assert torch.all(torch.isnan(mv[:n, d:w])) and torch.all(ar[:n, d:w] == -7)
    # two launches: the same bits
    agg2, mv2, ar2, _ = _aggregate_guarded(g, zs, zd, seg_pad=8)
    assert torch.equal(agg.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       agg2.view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
    assert torch.equal(mv.view(torch.int32), mv2.view(torch.int32)) and torch.equal(ar, ar2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_aggregate_past_the_first_wave(dtype):
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(40_000, 5_000, seed=3, hubs=(3000, 1500, 700, 200, 90, 65, 40, 33))
    gen = torch.Generator().manual_seed(7)
    d = 64
    zs = _zs(g.num_all, d, dtype, gen)
    zd = alloc_rows(g.num_in, d, torch.float32, DEV)
    zd.zero_()
    agg, mv, ar, w = _aggregate_guarded(g, zs, zd)
    n = g.num_in
    mx, ax = _extremes_ref(zs.double(), rows, cols, n, 1)
    mn, an = _extremes_ref(zs.double(), rows, cols, n, -1)
    assert torch.equal(ar[:n, :d], ax.int()) and torch.equal(ar[:n, w:w + d], an.int())
    mu, var, amax, deg = _moments_ref(zs.double(), rows, cols, n)
    assert torch.all((mv[:n, :d].double() - mu).abs() <= 4 * deg * 2.0 ** -24 * amax + 1e-30)
    assert torch.all((mv[:n, w:w + d].double() - var).abs() <= 16 * deg * 2.0 ** -24 * amax ** 2 + 1e-30)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [5, 64, 256, 602])
def test_backward_and_row_kernels_vs_fp64(dtype, d):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    g, rows, cols = _plan_graph(300, 120, seed=d + 5, seg_len=64)
    gen = torch.Generator().manual_seed(d)
    n, n_all = g.num_in, g.num_all
    zs = _zs(n_all, d, dtype, gen)
    zd = alloc_rows(n, d, torch.float32, DEV)
    zd.copy_(torch.randn(n, d, generator=gen).to(DEV))
    agg, mu, var, amax, amin = ops.pna_aggregate(g.fwd, zs, zd)
    w = ops.pna_width(d)
    gagg = alloc_rows(n, 4 * w, torch.float32, DEV)
    gagg.copy_(torch.randn(n, 4 * w, generator=gen).to(DEV))
    pz = alloc_rows(n_all, 2 * w, dtype, DEV, zero=True)
    alpha, beta, gmx, gmn = ops.pna_bwd_dst(g.fwd.indptr, gagg, mu, var, pz[:n, w:w + d])
    ops.pna_bwd_src(g.bwd, zs, alpha, beta, amax, amin, gmx, gmn, pz[:, :d])
    # destination pass: fp32 formulas, each operation rounded once
    deg = torch.bincount(rows, minlength=n)[:, None].float()
    has = deg > 0
    gm, gx, gn, gsg = [gagg[:, k * w:k * w + d] for k in range(4)]
    sig = torch.sqrt(var.clamp(min=0) + 1e-30)
    be = torch.where(has & (var > 0), gsg / (deg * sig), torch.zeros_like(gsg))
    al = torch.where(has, gm / deg - be * mu, torch.zeros_like(gm))
    zdr = torch.where(has, (gm + gx) + gn, torch.zeros_like(gm)).to(dtype)
    assert torch.equal(alpha, al) and torch.equal(beta, be) and torch.equal(pz[:n, w:w + d], zdr)
    assert torch.equal(gmx, torch.where(has, gx, 0 * gx).to(dtype)) and torch.equal(gmn, torch.where(has, gn, 0 * gn).to(dtype))
    assert torch.all(beta[14:18] == 0)                            # var = 0: no std gradient
    # source pass against fp64 sums of the kernel's own alpha, beta, g_mx, g_mn
    a64, b64 = alpha.double(), beta.double()
    rx = torch.where(amax[rows] == cols[:, None], gmx[rows].double(), 0.0)
    rn = torch.where(amin[rows] == cols[:, None], gmn[rows].double(), 0.0)
    s1 = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, cols, a64[rows] + rx + rn)
    s1a = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, cols, a64[rows].abs() + rx.abs() + rn.abs())
    s2 = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, cols, b64[rows])
    s2a = torch.zeros(n_all, d, dtype=torch.float64, device=DEV).index_add(0, cols, b64[rows].abs())
    odeg = torch.bincount(cols, minlength=n_all)[:, None].double()
    z64 = zs.double()
    ref = s1 + z64 * s2
    bound = 3 * (odeg + 2) * 2.0 ** -24 * (s1a + z64.abs() * s2a) + EPS[dtype] * ref.abs() + 1e-30
    got = pz[:, :d].double()
    assert torch.all((got - ref).abs() <= bound), (got - ref).abs().max()
    assert torch.all(pz[n_all - 5:, :d] == 0)                    # never-referenced sources: exact zeros
    pz2 = alloc_rows(n_all, 2 * w, dtype, DEV, zero=True)
    ops.pna_bwd_dst(g.fwd.indptr, gagg, mu, var, pz2[:n, w:w + d])
    ops.pna_bwd_src(g.bwd, zs, alpha, beta, amax, amin, gmx, gmn, pz2[:, :d])
    assert torch.equal(pz.float(), pz2.float())
    # combine and grad_scale: bit for bit
    d_out = d
    sa, st = g.pna_scalers(1.7)
    y = torch.randn(n, d_out, generator=gen).to(DEV)
    z = torch.randn(n, 2 * d_out, generator=gen).to(DEV)
    out = ops.pna_combine(y, z, sa, st, dtype)
    ref = ((y + sa[:, None] * z[:, :d_out]) + st[:, None] * z[:, d_out:]).to(dtype)
    assert torch.equal(out.float(), ref.float())
    gg = alloc_rows(n, d_out, dtype, DEV)
    gg.copy_(torch.randn(n, d_out, generator=gen))
    g3 = ops.pna_grad_scale(gg, sa, st)
    wo = ops.pna_width(d_out)
    gf = gg.float()
    for k, s in enumerate((None, sa, st)):
        ref = gf if s is None else (s[:, None] * gf)
        assert torch.equal(g3[:, k * wo:k * wo + d_out].float(), ref.to(dtype).float())


# ------------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("d_in,d_out", [(24, 16), (64, 64), (300, 40)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("drop", [0.0, 0.3])
def test_layer_autograd_matches_restatement(d_in, d_out, dtype, drop):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph, alloc_rows
    from pipegcn_b200.partition import _csr_from_pairs
    h64, rows, cols, num_in = graph_case(seed=d_in, d=d_in)
    num_all = h64.shape[0]
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=4)
    gen = torch.Generator().manual_seed(d_out)
    wm = (torch.randn(d_in, 2 * d_in, generator=gen) / (2 * d_in) ** 0.5).to(DEV).requires_grad_(True)
    bm = (0.1 * torch.randn(d_in, generator=gen)).to(DEV).requires_grad_(True)
    wu = (torch.randn(d_out, 13 * d_in, generator=gen) / (13 * d_in) ** 0.5).to(DEV).requires_grad_(True)
    bu = (0.1 * torch.randn(d_out, generator=gen)).to(DEV).requires_grad_(True)
    feat = alloc_rows(num_all, d_in, dtype, DEV)
    feat.copy_(h64)
    feat.requires_grad_(True)
    delta = 1.31
    spec = ops.DropSpec(drop, 1234, None, 0) if drop > 0 else None
    out = ops.pna_layer(feat, g, delta, wm, bm, wu, bu, drop_bwd=spec)
    gout = torch.randn(num_in, d_out, generator=gen).to(DEV).to(dtype)
    out.backward(gout)
    q = (lambda t: t.detach().to(dtype).double().cpu())
    ref, st = factorised_forward(feat.detach().double().cpu(), indptr.long(), indices.long(), num_in, delta,
                                 q(wm), bm.detach().double().cpu(), q(wu), bu.detach().double().cpu(),
                                 store=lambda t: t.to(dtype).double())
    grads = factorised_backward(gout.double().cpu(), feat.detach().double().cpu(), indptr.long(), indices.long(),
                                num_in, q(wm), q(wu), st)
    gh = grads["h"]
    if spec is not None:
        ones = alloc_rows(num_all, d_in, dtype, DEV)
        ones.fill_(1)
        keep = ops.dropout_rows(ones, spec)
        gh = gh * keep.double().cpu()
    def close(got, want, name):
        got = got.detach().double().cpu()
        if dtype == torch.float32:
            scale = want.abs().max().item() + 1e-12
            assert (got - want).abs().max().item() <= 2e-3 * scale, (name, (got - want).abs().max().item(), scale)
        else:       # bf16 storage of zs, agg, G3 and [g_zs | g_zd]: 2^-9 per stored value, compared in norm
            assert (got - want).norm() <= 3e-2 * want.norm() + 1e-9, (name, (got - want).norm(), want.norm())

    close(out, ref, "out")
    close(feat.grad, gh, "h")
    close(wm.grad, grads["wm"], "wm")
    close(bm.grad, grads["bm"], "bm")
    close(wu.grad, grads["wu"], "wu")
    close(bu.grad, grads["bu"], "bu")


# ------------------------------------------------------------------------------------------------ engine
def _args(g, n_class, **kw):
    base = dict(model="pna", backend="nccl", dtype="fp32", n_layers=3, n_hidden=16, n_linear=0,
                n_feat=g.n_feat, n_class=n_class, n_train=int(g.train_mask.sum()), dropout=0.0, norm="layer",
                lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=False, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=4, log_every=10)
    base.update(kw)
    return argparse.Namespace(**base)


def _pna_ref(x, q, p, i, delta, dtype):
    """fp64 PNA layer i over one rank's [inner | halo] rows x (rounded where the engine stores values)."""
    from tests.test_gat_gpu import _stored
    d = x.shape[1]
    rows, cols, n = q["rows"], q["cols"], q["num_in"]
    wm, wu = _stored(p[f"layers.{i}.M.weight"], dtype), _stored(p[f"layers.{i}.U.weight"], dtype)
    zs = _stored(x @ wm[:, :d].T, dtype)
    zd = x[:n] @ wm[:, d:].T + p[f"layers.{i}.M.bias"]
    deg = torch.bincount(rows, minlength=n).double()[:, None]
    e = zs[cols]
    mu = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, e) / deg
    var = torch.zeros(n, d, dtype=torch.float64, device=DEV).index_add(0, rows, (e - mu[rows]) ** 2) / deg
    # the extremes as gathers of the source the kernels pick (the first in CSR order on a tie): zero halo rows, as a
    # pipelined exchange delivers before its first epoch, tie exactly
    _, ax = _extremes_ref(zs.detach(), rows, cols, n, 1)
    _, an = _extremes_ref(zs.detach(), rows, cols, n, -1)
    mx, mn = zs.gather(0, ax.clamp(min=0)), zs.gather(0, an.clamp(min=0))
    agg = _stored(torch.cat([mu + zd, mx + zd, mn + zd, torch.sqrt(var.clamp(min=0) + 1e-30)], 1), dtype)
    a, t = scalers64(deg[:, 0].long(), delta)
    a, t = a.float().double()[:, None], t.float().double()[:, None]
    return torch.cat([x[:n], agg, a * agg, t * agg], 1) @ wu.T + p[f"layers.{i}.U.bias"]


def restate_training(g, layouts, state, a, dtype, delta):
    from tests.test_gat_gpu import _edges, _stored
    n = g.n_nodes
    params = {k: v.detach().to(DEV, torch.float64).clone().requires_grad_(True) for k, v in state.items()
              if v.is_floating_point() and k != "pna_delta"}
    n_layers, n_graph = a.n_layers, a.n_layers - a.n_linear
    sizes = [a.n_feat] + [a.n_hidden] * (n_layers - 1) + [a.n_class]
    H = torch.zeros(n, a.n_feat, dtype=torch.float64, device=DEV)
    for lay in layouts:
        H[lay.inner_gid.to(DEV)] = lay.feat.to(DEV).to(dtype).double()
    gr = []
    for lay in layouts:
        rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
        gid = torch.cat([lay.inner_gid, lay.halo_gid]).long().to(DEV)
        gr.append(dict(gid=gid, rows=rows, cols=cols, inner=lay.inner_gid.long().to(DEV), num_in=lay.num_in))
    outs = [dict() for _ in layouts]
    for i in range(n_layers):
        Hn = torch.zeros(n, sizes[i + 1], dtype=torch.float64, device=DEV)
        for r, q in enumerate(gr):
            if i < n_graph:
                out = _pna_ref(_stored(H[q["gid"]], dtype), q, params, i, delta, dtype)
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


ENGINE_CASES = [  # (P, partition, static layer 0, n_linear, dtype)
    (1, "random", True, 0, "fp32"),
    (1, "random", False, 1, "bf16"),
    (2, "random", True, 1, "fp32"),
    (2, "metis", False, 0, "bf16"),
    (3, "metis", False, 0, "fp32"),
    (3, "random", True, 1, "bf16"),
    (4, "metis", True, 1, "fp32"),
    (4, "random", False, 0, "fp32"),
]


@pytest.mark.parametrize("P,method,static0,n_linear,dtype", ENGINE_CASES)
def test_engine_matches_partitioned_restatement(P, method, static0, n_linear, dtype):
    """Synchronous training, dropout 0, 3 epochs, every halo row poisoned with NaN before each epoch.  Per-layer
    outputs, logits, losses and reduced gradients against the fp64 restatement with the whole graph's delta."""
    from pipegcn_b200.ops import pna_delta
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, 5, static_layer0=static0, n_linear=n_linear, dtype=dtype)
    tr = _trainer(layouts, a)
    delta = pna_delta([torch.bincount(g.in_degrees().long()).tolist()])
    assert all(e.model.delta == delta for e in tr.engines)
    caps = _hook_outputs(tr, a)
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    for _ in range(3):
        state = {k: v.detach().clone() for k, v in tr.engines[0].model.state_dict().items()}
        _poison(tr)
        losses = tr.run_epoch(keep_logits=True)
        torch.cuda.synchronize()
        outs, logits, ref_losses, grads = restate_training(g, layouts, state, a, tdt, delta)
        for r, eng in enumerate(tr.engines):
            got_logits = eng.last_logits.double()
            assert torch.isfinite(got_logits).all()
            tol, gtol = (2e-3, 1e-2) if dtype == "fp32" else (6e-2, 0.25)
            for i, ref in list(outs[r].items()) + [("logits", logits[r])]:
                got = got_logits if i == "logits" else caps[r][i].double()
                scale = ref.detach().abs().max().item()
                assert (got - ref.detach()).abs().max().item() <= tol * scale + 1e-6, (r, i)
            ref_l = float(ref_losses[r].detach())
            assert abs(float(losses[r]) - ref_l) <= tol * abs(ref_l) + 1e-4
            for name, prm in eng.model.named_parameters():
                gref = grads[name]
                assert (prm.grad.double() - gref).norm() <= gtol * gref.norm() + 1e-6, name


@pytest.mark.parametrize("mode", [dict(), dict(feat_corr=True, grad_corr=True), dict(enable_pipeline=True),
                                  dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8),
                                  dict(enable_pipeline=True, halo_bits=8)])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_exchange_modes_train(mode, dtype):
    """P = 3 in every exchange mode (--halo-bits 8 included), dropout 0.5: losses stay finite and fall."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _args(g, 5, static_layer0=False, dtype=dtype, dropout=0.5, **mode)
    if bits is not None:
        a.halo_bits = bits
    tr = _trainer(layouts, a)
    losses = [sum(float(l.item()) for l in tr.run_epoch()) for _ in range(12)]
    assert all(l == l for l in losses) and sum(losses[-3:]) < sum(losses[:3])


_MODES = [dict(), dict(feat_corr=True, grad_corr=True), dict(enable_pipeline=True),
          dict(enable_pipeline=True, feat_corr=True, grad_corr=True), dict(halo_bits=8),
          dict(enable_pipeline=True, halo_bits=8)]
_STALL = pytest.mark.skip(reason="stalls: rank 0's layer-0 flag wait times out in epoch 1 with these gradient hooks; "
                                 "bf16 synchronous training is compared in test_engine_matches_partitioned_restatement")


@pytest.mark.parametrize("dtype,mode", [pytest.param(dt, m, marks=_STALL if (dt == "bf16" and not m) else ())
                                        for dt in ("fp32", "bf16") for m in _MODES])
def test_exchange_modes_layer_parity(mode, dtype):
    """P = 3, dropout 0, every exchange mode (--halo-bits 8 included): every graph layer >= 1's output and input
    gradient equal the fp64 PNA layer applied to the [inner | halo] rows it read -- the stale, corrected or quantised
    halo rows the exchange delivered -- with the upstream gradient it received and the whole graph's delta."""
    from pipegcn_b200.ops import pna_delta
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _edges
    g, layouts = _layouts("tiny", 3)
    mode = dict(mode)
    bits = mode.pop("halo_bits", None)
    a = _args(g, 5, static_layer0=False, dtype=dtype, **mode)
    if bits is not None:
        a.halo_bits = bits
    tr = _trainer(layouts, a)
    delta = pna_delta([torch.bincount(g.in_degrees().long()).tolist()])
    recs = [dict() for _ in tr.engines]

    def keep(rec, key, t):
        # after the first epoch into the same buffers: no allocation inside a synchronous LocalWorld epoch, where a
        # host synchronisation of the allocator would stall the ranks whose flag waits are already queued
        if key in rec and rec[key].shape == t.shape:
            rec[key].copy_(t)
        else:
            rec[key] = t.detach().clone()
        rec["has_" + key] = True

    def hook(mod, inp, out, r, i):
        rec = recs[r].setdefault(i, {})
        keep(rec, "x", inp[1].detach())
        keep(rec, "out", out.detach())
        rec["has_gx"] = False
        out.register_hook(lambda gr: keep(rec, "gout", gr))
        if inp[1].requires_grad:
            inp[1].register_hook(lambda gr: keep(rec, "gx", gr))

    n_graph = a.n_layers - a.n_linear
    for r, eng in enumerate(tr.engines):
        for i, layer in enumerate(eng.model.layers[:n_graph]):
            layer.register_forward_hook(lambda mod, inp, out, r=r, i=i: hook(mod, inp, out, r, i))
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    def close(got, ref):
        if dtype == "fp32":
            return (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-6
        # bf16: a source stored one bf16 ulp away from the fp64 restatement's may win an extreme, so the routed
        # gradients of a few elements differ; compared in norm
        return (got - ref).norm().item() <= 5e-2 * ref.norm().item() + 1e-6

    n_checked, losses = 0, []
    for _ in range(5):
        state = {k: v.detach().double() for k, v in tr.engines[0].model.state_dict().items()}
        torch.cuda.synchronize()
        losses.append(sum(float(l.item()) for l in tr.run_epoch()))
        torch.cuda.synchronize()
        for r, lay in enumerate(layouts):
            rows, cols = _edges((lay.indptr.to(DEV), lay.indices.to(DEV)))
            q = dict(rows=rows, cols=cols, num_in=lay.num_in)
            for i in range(1, n_graph):
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                out = _pna_ref(x, q, state, i, delta, tdt)
                assert close(rec["out"].double(), out.detach()), (r, i)
                out.backward(rec["gout"].double())
                if rec["has_gx"]:
                    assert close(rec["gx"].double(), x.grad), (r, i)
                    n_checked += 1
    assert n_checked > 0
    assert all(l == l for l in losses) and losses[-1] < losses[0]


# ------------------------------------------------------------------------------------------------ evaluation etc.
@pytest.mark.parametrize("P", [2, 4])
def test_eval_paths_and_checkpoint(P, tmp_path):
    """Partitioned evaluation equals whole-graph evaluation on rank 0; a checkpoint carries delta and loads strictly
    into a fresh model that evaluates the same."""
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
    path = tmp_path / "pna.pt"
    torch.save(model.state_dict(), path)
    fresh = create_model(tr.engines[0].layer_size, a).to(DEV)
    assert fresh.delta is None
    fresh.load_state_dict(torch.load(path), strict=True)
    assert fresh.delta == model.delta and float(torch.load(path)["pna_delta"]) == model.delta
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
    from tests.test_graphconv_gpu import _replay_runs, _small
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


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
    print(f"pna planted-label validation accuracy {val:.4f}")
    assert val > 0.3
