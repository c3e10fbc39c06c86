"""Residual gated graph convolution (`--model resgatedgcn`) on the GPU: the three ResGatedGCN kernels against fp64 on
every dispatch path (long rows in segments, single long rows, short rows), on every vector width, past the first wave,
with gates far into saturation, with and without a keep mask, with guarded outputs and two launches giving the same
bits; the layer's autograd against PyG's definition in fp64; the engine against a restatement of partitioned training
(sampled too); every exchange mode layer by layer; evaluation, checkpoints, `--inductive`, CUDA-graph replay and
free-running training.

The aggregate is an unnormalised sum that can cancel, so the kernels' bounds are relative to sum_u |sigmoid val| per
element (and the like for the backward passes), not to the result."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from pipegcn_b200 import _C
from tests.test_pna_gpu import _plan_graph
from tests.test_resgated_cpu import pyg_forward

pytestmark = pytest.mark.gpu
DEV = "cuda"
E32 = 2.0 ** -24
EPS = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8}
PARAMS = ("lin_key.weight", "lin_key.bias", "lin_query.weight", "lin_query.bias", "lin_value.weight",
          "lin_value.bias", "lin_skip.weight", "bias")


# ------------------------------------------------------------------------------------------------ kernels
def _layout(d, dtype, vb):
    """(half, row stride) of paired rows whose widest legal vector is vb bytes: half a multiple of the vector, the
    stride an odd multiple of it (16-byte vectors: a multiple of 8 elements)."""
    es = torch.empty((), dtype=dtype).element_size()
    v = vb // es
    half = (d + v - 1) // v * v
    ld = 2 * half + 3 * v
    if vb == 16:
        ld = (ld + 7) // 8 * 8
    elif (ld // v) % 2 == 0:
        ld += v
    return half, ld


def _guarded(n, ld, dtype, extra_rows=3):
    buf = torch.full((n + extra_rows, ld), float("nan"), dtype=dtype, device=DEV)
    return buf[:n], buf


def _operands(g, d, dtype, vb, gen, scale):
    """Paired qv [num_all] = [q | val] and ks [N_in] = [k | skip], G [N_in, d], in NaN-guarded buffers (pad columns
    NaN); |k + q| reaches past 100 at scale 30."""
    half, ld = _layout(d, dtype, vb)
    qv, _ = _guarded(g.num_all, ld, dtype)
    ks, _ = _guarded(g.num_in, ld, dtype)
    qv[:, :d] = scale * torch.randn(g.num_all, d, generator=gen).to(DEV)
    qv[:, half:half + d] = torch.randn(g.num_all, d, generator=gen).to(DEV)
    ks[:, :d] = scale * torch.randn(g.num_in, d, generator=gen).to(DEV)
    ks[:, half:half + d] = torch.randn(g.num_in, d, generator=gen).to(DEV)
    es = torch.empty((), dtype=dtype).element_size()
    gld = ld if vb == 16 else (d + vb // es - 1) // (vb // es) * (vb // es) + vb // es
    if vb < 16 and (gld // (vb // es)) % 2 == 0:
        gld += vb // es
    G, _ = _guarded(g.num_in, gld, dtype)
    G[:, :d] = torch.randn(g.num_in, d, generator=gen).to(DEV)
    return qv, ks, G[:, :d], half, ld


def _hub_graph(num_in, num_halo, seed, seg_len, hubs=(700, 200, 90, 65, 40, 33)):
    """(PartGraph, rows, cols in CSR order) of tests.test_pna_gpu._plan_graph's graph (in-hubs, rows without in-edges
    (10..13), self-loop-only rows (14..17), never-referenced halo rows (the last 5)) plus out-hubs, so that the source
    pass's CSC has long rows of its own: halo rows num_in and num_in + 1 and inner row 20 with more than seg_len
    destinations (segments), halo rows num_in + 2 and num_in + 3 with 33..seg_len (single long rows).  seg_len must
    leave room: 2 seg_len + 5 <= num_in - 8."""
    from pipegcn_b200.graph import PartGraph
    from pipegcn_b200.partition import _csr_from_pairs
    gen = torch.Generator().manual_seed(seed)
    num_all = num_in + num_halo
    deg = torch.randint(1, 12, (num_in,), generator=gen)
    deg[:len(hubs)] = torch.tensor(hubs)
    deg[10:14] = 0
    srcs = [[v] if 14 <= v < 18 else torch.randperm(num_all - 5, generator=gen)[:int(deg[v])].tolist()
            for v in range(num_in)]
    single = seg_len // 2 + 8            # with the random in-edges that reference it, still at most seg_len
    out_hubs = {num_in: 2 * seg_len + 5, num_in + 1: seg_len + seg_len // 2 + 3, 20: seg_len + 9,
                num_in + 2: single, num_in + 3: single - 1}
    eligible = torch.tensor([v for v in range(num_in) if not 10 <= v < 18])
    for u, k in out_hubs.items():
        assert k <= len(eligible)
        chosen = 0
        for v in eligible[torch.randperm(len(eligible), generator=gen)].tolist():
            if chosen == k:
                break
            if u not in srcs[v]:
                srcs[v].append(u)
                chosen += 1
        assert chosen == k
    rows = torch.tensor([v for v in range(num_in) for _ in srcs[v]])
    cols = torch.tensor([u for v in range(num_in) for u in srcs[v]])
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=seg_len)
    r = torch.repeat_interleave(torch.arange(num_in), (indptr[1:] - indptr[:-1]).long())
    return g, r.to(DEV), indices.long().to(DEV)


def _keep(g, on, seed=5):
    """The keep mask of the halo rows (60 % kept), with the out-hubs of _hub_graph split: halo rows num_in (segments)
    and num_in + 2 (a single long row) unkept, num_in + 1 and num_in + 3 kept."""
    if not on:
        return None
    gen = torch.Generator().manual_seed(seed)
    keep = (torch.rand(g.num_all - g.num_in, generator=gen) < 0.6).to(torch.uint8)
    keep[:4] = torch.tensor([0, 1, 0, 1], dtype=torch.uint8)
    return keep.to(DEV)


def _kept(rows, cols, num_in, keep):
    if keep is None:
        return rows, cols
    ok = (cols < num_in) | keep[(cols - num_in).clamp(min=0)].bool()
    return rows[ok], cols[ok]


def _run(which, g, qv, ks, G, d, half, keep, out):
    from pipegcn_b200.ops import _ptr, _scratch_ld
    plan = g.bwd if which == "src" else g.fwd
    parts = 2 if which == "src" else 1
    scratch = plan.scratch(parts * d)
    fn = {"fwd": _C.lib.pg_resgated_aggregate, "dst": _C.lib.pg_resgated_bwd_dst, "src": _C.lib.pg_resgated_bwd_src}
    head = (C.byref(plan.c), qv.data_ptr(), qv.stride(0), ks.data_ptr(), ks.stride(0), half)
    mid = (d,) if which == "fwd" else (G.data_ptr(), G.stride(0), d)
    _C.check(fn[which](*head, *mid, _C.dtype_code(qv.dtype), _ptr(keep), g.num_in, out.data_ptr(), out.stride(0),
                       _ptr(scratch), _scratch_ld(parts * d), _C.stream_ptr()), which)


def _gates(x32):
    """fp64 sigmoid and sigmoid' of the fp32 gate arguments the kernels form (k + q rounded once)."""
    x = x32.double()
    s = torch.sigmoid(x)
    return s, s * torch.sigmoid(-x)


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    assert torch.all(err <= bound), (what, (err - bound).max().item())


def _check_guards(buf, n, cols, what):
    """Only rows [0, n) and columns [0, cols) of the guarded buffer are written."""
    assert torch.all(torch.isnan(buf[n:].float())) and torch.all(torch.isnan(buf[:, cols:].float())), what


def _check_kernels(g, rows, cols, d, dtype, vb, keep, scale, seed):
    n, n_all = g.num_in, g.num_all
    gen = torch.Generator().manual_seed(seed)
    qv, ks, G, half, ld = _operands(g, d, dtype, vb, gen, scale)
    es = torch.empty((), dtype=dtype).element_size()
    full = (d + vb // es - 1) // (vb // es) * (vb // es)        # the last vector's end
    kr, kc = _kept(rows, cols, n, keep)
    kept_row = torch.ones(n_all, dtype=torch.bool, device=DEV)
    if keep is not None:                                        # an unkept halo row holds NaN: no kernel may read it
        kept_row[n:] = keep.bool()
        qv[~kept_row] = float("nan")
    q, val = qv[:, :d].float(), qv[:, half:half + d].float()
    k, skip = ks[:, :d].float(), ks[:, half:half + d].float()
    x32 = k[kr] + q[kc]
    s, ds = _gates(x32)
    if scale > 10:
        assert float(x32.abs().max()) > 100
    deg = torch.bincount(kr, minlength=n)[:, None].double()
    odeg = torch.bincount(kc, minlength=n_all)[:, None].double()
    Gd, vd = G.double(), torch.where(kept_row[:, None], val.double(), 0.0)
    z = lambda m: torch.zeros(m, d, dtype=torch.float64, device=DEV)
    tiny = 2.0 ** -140                                          # sigmoid' past its normal range, per term
    # aggregate: out = skip + sum s val
    out, ob = _guarded(n, ld, dtype)
    _run("fwd", g, qv, ks, G, d, half, keep, out)
    acc, mag = z(n).index_add(0, kr, s * vd[kc]), z(n).index_add(0, kr, (s * vd[kc]).abs())
    ref = skip.double() + acc
    _within(out[:, :d], ref, (deg + 8) * E32 * mag + EPS[dtype] * (ref.abs() + skip.double().abs()) + 1e-30, "out")
    assert torch.equal(out[:, :d][deg[:, 0] == 0], ks[:, half:half + d][deg[:, 0] == 0])   # no kept in-edge: skip
    assert torch.all(out[:, d:full] == 0)
    _check_guards(ob, n, full, "out")
    # destination pass: [dk | G]
    dkg, db = _guarded(n, ld, dtype)
    _run("dst", g, qv, ks, G, d, half, keep, dkg)
    s1, m1 = z(n).index_add(0, kr, ds * vd[kc]), z(n).index_add(0, kr, (ds * vd[kc]).abs())
    ref = Gd * s1
    _within(dkg[:, :d], ref, Gd.abs() * ((deg + 8) * E32 * m1 + deg * tiny) + EPS[dtype] * ref.abs() + 1e-30, "dk")
    assert torch.equal(dkg[:, half:half + d], G)
    assert torch.all(dkg[:, d:full] == 0) and torch.all(dkg[:, half + d:half + full] == 0)
    _check_guards(db, n, half + full, "dkg")
    # source pass: [dq | dval]
    dqv, sb = _guarded(n_all, ld, dtype)
    _run("src", g, qv, ks, G, d, half, keep, dqv)
    A, mA = z(n_all).index_add(0, kc, Gd[kr] * s), z(n_all).index_add(0, kc, (Gd[kr] * s).abs())
    B, mB = z(n_all).index_add(0, kc, Gd[kr] * ds), z(n_all).index_add(0, kc, (Gd[kr] * ds).abs())
    _within(dqv[:, half:half + d], A, (odeg + 8) * E32 * mA + EPS[dtype] * A.abs() + 1e-30, "dval")
    ref = vd * B
    _within(dqv[:, :d], ref, vd.abs() * ((odeg + 8) * E32 * mB + odeg * tiny) + EPS[dtype] * ref.abs() + 1e-30, "dq")
    assert torch.all(dqv[n_all - 5:, :d] == 0) and torch.all(dqv[n_all - 5:, half:half + d] == 0)   # no out-edges
    if keep is not None:
        unkept = n + torch.nonzero(keep == 0)[:, 0]
        assert torch.all(dqv[unkept][:, :d] == 0) and torch.all(dqv[unkept][:, half:half + d] == 0)
    assert torch.all(dqv[:, d:full] == 0) and torch.all(dqv[:, half + d:half + full] == 0)
    _check_guards(sb, n_all, half + full, "dqv")
    # two launches: the same bits
    for which, first in (("fwd", out), ("dst", dkg), ("src", dqv)):
        again, _ = _guarded(first.shape[0], ld, dtype)
        _run(which, g, qv, ks, G, d, half, keep, again)
        assert torch.equal(again.float().nan_to_num(7.0), first.float().nan_to_num(7.0)), which
    return qv, ks


VBS = [(torch.float32, vb) for vb in (16, 8, 4)] + [(torch.bfloat16, vb) for vb in (16, 8, 4, 2)]


def _check_plans(g, rows, cols, keep, seg_len):
    """Both plans have long rows in segments and single long rows (33..seg_len entries), and with a keep mask an
    unkept halo row is among the CSC's long rows of each kind."""
    for plan in (g.fwd, g.bwd):
        assert plan.n_long > 0 and plan.n_chunks_long > plan.n_seg
    if keep is not None:
        n = g.num_in
        odeg = torch.bincount(cols, minlength=g.num_all)
        unkept = n + torch.nonzero(keep == 0)[:, 0]
        assert bool((odeg[unkept] > seg_len).any()) and bool(((odeg[unkept] > 32) & (odeg[unkept] <= seg_len)).any())


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("d,seg_len,scale", [(5, 64, 30.0), (64, 128, 1.0), (602, 64, 3.0)])
@pytest.mark.parametrize("dtype,vb", VBS)
def test_kernels_vs_fp64(dtype, vb, d, seg_len, scale, masked):
    """In-hubs of 700 and 200 in-edges and out-hubs of more than seg_len destinations (in segments), rows of
    33..seg_len entries on both sides (single long rows), short rows, rows without in-edges or with a self loop only,
    never-referenced halo rows; with the mask, unkept out-hubs of both kinds whose rows hold NaN; poisoned pad
    columns; gates saturated at scale 30."""
    g, rows, cols = _hub_graph(300, 120, seed=d + vb, seg_len=seg_len)
    keep = _keep(g, masked)
    _check_plans(g, rows, cols, keep, seg_len)
    _check_kernels(g, rows, cols, d, dtype, vb, keep, scale, seed=d)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernels_past_the_first_wave(dtype):
    g, rows, cols = _hub_graph(40_000, 5_000, seed=3, seg_len=64, hubs=(3000, 1500, 700, 200, 90, 65, 40, 33))
    keep = _keep(g, True)
    _check_plans(g, rows, cols, keep, 64)
    _check_kernels(g, rows, cols, 64, dtype, 16, keep, 2.0, seed=7)


def test_entry_points_refuse_short_rows():
    from pipegcn_b200.graph import alloc_rows
    g, _, _ = _plan_graph(300, 120, seed=1)
    qv = alloc_rows(g.num_all, 16, torch.float32, DEV)
    ks = alloc_rows(g.num_in, 16, torch.float32, DEV)
    out = alloc_rows(g.num_in, 8, torch.float32, DEV)
    with pytest.raises(_C.PgError, match="shorter than its last"):
        _run("fwd", g, qv, ks, None, 6, 12, None, out)             # 16 columns < half 12 + the last vector's 8
    with pytest.raises(_C.PgError, match="bad sizes"):
        _run("fwd", g, qv, ks, None, 9, 8, None, out)              # half < d


# ------------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("d_in,d", [(24, 16), (64, 64), (300, 40), (20, 5)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("drop", [0.0, 0.3])
def test_layer_autograd_matches_pyg(d_in, d, dtype, drop):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph, alloc_rows
    from pipegcn_b200.partition import _csr_from_pairs
    from tests.test_gat_gpu import _stored
    from tests.test_pna_cpu import graph_case
    from tests.test_resgated_cpu import weights
    h64, rows, cols, num_in = graph_case(seed=d_in, d=d_in)
    num_all = h64.shape[0]
    indptr, indices = _csr_from_pairs(rows, cols, num_in, num_all)
    t_indptr, t_indices = _csr_from_pairs(cols, rows, num_all, num_in)
    g = PartGraph(num_in, num_all, indptr, indices, t_indptr, t_indices, torch.bincount(rows, minlength=num_in),
                  device=DEV, seg_len=4)
    params = [w.float().to(DEV).requires_grad_(True) for w in weights(d_in, d, seed=d, scale=2.0)]
    feat = alloc_rows(num_all, d_in, dtype, DEV)
    feat.copy_(h64)
    feat.requires_grad_(True)
    spec = ops.DropSpec(drop, 1234, None, 0) if drop > 0 else None
    out = ops.resgated_layer(feat, g, None, *params, drop_bwd=spec)
    gout = torch.randn(num_in, d, generator=torch.Generator().manual_seed(3)).to(DEV).to(dtype)
    out.backward(gout)
    st = lambda x: _stored(x, dtype)
    leaves = [p.detach().double().requires_grad_(True) for p in params]
    x64 = feat.detach().double().requires_grad_(True)
    wk, bk, wq, bq, wv, bv, ws, b = leaves
    ref = pyg_forward(x64, rows.to(DEV), cols.to(DEV), num_in, st(wk), bk, st(wq), bq, st(wv), bv, st(ws), b, store=st)
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
    for name, p, leaf in zip(("wk", "bk", "wq", "bq", "wv", "bv", "ws", "b"), params, leaves):
        close(p.grad, leaf.grad, name)


# ------------------------------------------------------------------------------------------------ engine
def _args(g, n_class=5, **kw):
    from tests.test_boundary_sampling_gpu import _args as base
    extra = {k: kw.pop(k) for k in ("dtype", "cuda_graph") if k in kw}
    a = base(g, n_class, **kw)
    a.model = "resgatedgcn"
    for k, v in extra.items():
        setattr(a, k, v)
    return a


def _layer_ref(params, p, x, rows, cols, num_in, st):
    wk, bk, wq, bq, wv, bv, ws, b = [params[p + k] for k in PARAMS]
    return pyg_forward(x, rows, cols, num_in, st(wk), bk, st(wq), bq, st(wv), bv, st(ws), b, store=st)


def restate_training(layouts, masks, state, a, dtype):
    """Partitioned ResGatedGCN training in fp64 (PyG's definition): per rank the forward over its partition with the
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
                out = _layer_ref(params, f"layers.{i}.", st(H[q["gid"]]), q["rows"], q["cols"], q["num_in"], st)
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
    """Synchronous training, dropout 0, 3 epochs, every halo row poisoned with NaN before each epoch."""
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
        _check_engine(tr, layouts, a, caps, None, state, losses, dtype)


@pytest.mark.parametrize("P,method,static0,dtype", [(3, "random", True, "fp32"), (4, "metis", False, "fp32"),
                                                    (2, "random", True, "bf16")])
def test_sampled_engine_matches_restatement(P, method, static0, dtype):
    """Boundary-node sampling at p = 0.5: unkept halo sources are absent from every sum, unkept rows are poisoned."""
    from tests.test_boundary_sampling_gpu import _layouts, _trainer
    from tests.test_gat_gpu import _hook_outputs, _poison
    g, layouts = _layouts("tiny", P, method)
    a = _args(g, static_layer0=static0, sampling_rate=0.5)
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
    """P = 3, dropout 0: every graph layer >= 1's output and input gradient equal PyG's layer in fp64 applied to the
    [inner | halo] rows it read (the stale, corrected or quantised halo rows the exchange delivered) with the upstream
    gradient it received."""
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
                rec = recs[r][i]
                x = rec["x"].double().requires_grad_(True)
                out = _layer_ref(state, f"layers.{i}.", x, rows, cols, lay.num_in, st)
                assert close(rec["out"].double(), out.detach()), (r, i)
                out.backward(rec["gout"].double())
                if rec["has_gx"]:
                    assert close(rec["gx"].double(), x.grad), (r, i)
                    n_checked += 1
    assert n_checked > 0
    assert all(l == l for l in losses) and losses[-1] < losses[0]


# ------------------------------------------------------------------------------------------------ evaluation etc.
@pytest.mark.parametrize("n_hidden,dtype", [(16, "fp32"), (10, "fp32"), (12, "bf16")])
def test_single_partition_logits_equal_full_graph_eval(n_hidden, dtype):
    """Whole-graph evaluation hands the middle layer contiguous [N, d] rows when the fused LayerNorm epilogue does not
    take the width (d = 10 in fp32, 12 in bf16)."""
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
    else:       # the same bf16 roundings, sums in a relabelled order
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
    path = tmp_path / "resgated.pt"
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
    """Three pipelined epochs replayed from captured CUDA graphs equal three eager epochs bit for bit."""
    from tests.test_graphconv_gpu import _replay_runs, _small
    g, lays = _small(1)
    n_class = int(g.label.max()) + 1
    a = _args(g, n_class, dtype=dtype, dropout=0.0, enable_pipeline=True, cuda_graph=True)
    r0, r1 = _replay_runs(a, lays[0], None), _replay_runs(a, lays[0], 3)
    assert len(r1) >= 3
    for (l0, z0, p0), (l1, z1, p1) in zip(r0, r1):
        assert torch.equal(l0, l1) and torch.equal(z0, z1)
        assert all(torch.equal(x, y) for x, y in zip(p0, p1))


def test_learns_planted_labels():
    """16 planted classes (chance 1/16): validation accuracy after 120 pipelined epochs on 2 partitions.  The labels are
    a linear map of the own and the neighbour-mean features, which GraphSAGE-mean fits directly; the gated sums learn
    it more slowly (on an H100: 0.15, 0.29 and 0.42 after 40, 80 and 120 epochs, against 0.69 for mean after 40)."""
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
    print(f"resgatedgcn planted-label validation accuracy {val:.4f}")
    assert val > 0.3
