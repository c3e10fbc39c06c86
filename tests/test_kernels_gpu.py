"""GPU parity of the individual kernels (through the C ABI) against plain fp32 torch on the host."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _random_csr(n_rows, n_cols, avg_deg, seed, hubs=0, hub_deg=0):
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 2 * avg_deg + 1, (n_rows,), generator=g)
    for h in range(hubs):
        deg[(h * 7919) % n_rows] = hub_deg
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(deg, 0)
    indices = torch.randint(0, n_cols, (int(indptr[-1]),), generator=g)
    return indptr.to(torch.int32), indices.to(torch.int32)


def _ref_agg(indptr, indices, x, div=None):
    n_rows = indptr.numel() - 1
    rows = torch.repeat_interleave(torch.arange(n_rows), (indptr[1:] - indptr[:-1]).long())
    out = torch.zeros(n_rows, x.shape[1], dtype=torch.float64)
    out.index_add_(0, rows, x.double()[indices.long()])
    if div is not None:
        out = out / div.double()[:, None]
    return out


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.bfloat16, 1.6e-2)])
@pytest.mark.parametrize("d", [1, 7, 16, 41, 64, 100, 128, 256, 602])
def test_aggregate_matches_reference(dtype, tol, d):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import CsrPlan, alloc_rows
    n_rows, n_cols = 3000, 5000
    indptr, indices = _random_csr(n_rows, n_cols, 12, seed=d, hubs=3, hub_deg=2500)
    plan = CsrPlan(indptr.to(DEV), indices.to(DEV), seg_len=512)
    assert plan.n_long == 3 and plan.n_seg == 15
    g = torch.Generator().manual_seed(d + 1)
    x = torch.randn(n_cols, d, generator=g)
    div = torch.randint(1, 50, (n_rows,), generator=g).float()
    xd = alloc_rows(n_cols, d, dtype, DEV, zero=True)
    xd.copy_(x.to(dtype))
    out = ops.aggregate(plan, xd, row_div=div.to(DEV))
    ref = _ref_agg(indptr, indices, xd.float().cpu(), div)
    scale = ref.abs().max().item()
    err = (out.float().cpu().double() - ref).abs().max().item()
    assert err <= tol * scale + 1e-6, f"max err {err} scale {scale}"
    # empty rows produce exact zeros
    empty = (indptr[1:] == indptr[:-1]).nonzero().flatten()
    assert empty.numel() > 0 and torch.count_nonzero(out[empty.to(DEV)]) == 0


def test_aggregate_unpadded_and_accumulate():
    """Contiguous (unpadded) fp32 input of odd width, plus the accumulate-into-rows mode of the backward."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import CsrPlan
    n_rows, n_cols, d = 500, 700, 37
    indptr, indices = _random_csr(n_rows, n_cols, 9, seed=5)
    plan = CsrPlan(indptr.to(DEV), indices.to(DEV), seg_len=256)
    x = torch.randn(n_cols, d)
    base = torch.randn(n_rows, d)
    out = base.clone().to(DEV)
    ops.aggregate(plan, x.to(DEV), out=out, acc_rows=300)
    ref = _ref_agg(indptr, indices, x)
    ref[:300] += base[:300].double()
    torch.testing.assert_close(out.cpu().double(), ref, rtol=1e-5, atol=1e-5)


def test_aggregate_deterministic_with_long_rows():
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import CsrPlan
    indptr, indices = _random_csr(2000, 2000, 20, seed=9, hubs=5, hub_deg=1900)
    plan = CsrPlan(indptr.to(DEV), indices.to(DEV), seg_len=256)
    x = torch.randn(2000, 256, device=DEV)
    a = ops.aggregate(plan, x).clone()
    b = ops.aggregate(plan, x).clone()
    assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_sage_aggregate_autograd_matches_oracle(dtype):
    """Forward mean and backward A^T(g/deg) against the oracle's CPU autograd (oracle/model.py)."""
    from oracle.model import OracleGraph, _CopySrcSum
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph
    from tests.helpers import small_world
    _, _, layouts, setups = small_world("tiny", 2)
    L, S = layouts[1], setups[1]
    graph = PartGraph.from_layout(L, device=DEV, seg_len=64)
    d = 24
    x = torch.randn(L.num_all, d)
    go = torch.randn(L.num_in, d)
    if dtype == torch.bfloat16:
        x, go = x.bfloat16().float(), go.bfloat16().float()
    xo = x.clone().requires_grad_(True)
    og = OracleGraph(S.u, S.v, S.num_in, S.num_all)
    ah_o = _CopySrcSum.apply(og, xo) / S.in_deg.unsqueeze(1)
    ah_o.backward(go)
    xg = x.to(DEV).to(dtype).requires_grad_(True)
    ah = ops.sage_aggregate(xg, graph)
    ah.backward(go.to(DEV).to(dtype))
    tol = dict(rtol=1e-5, atol=1e-5) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(ah.float().cpu(), ah_o.detach(), **tol)
    torch.testing.assert_close(xg.grad.float().cpu(), xo.grad, **tol)


def test_row_div():
    from pipegcn_b200 import ops
    x = torch.randn(1000, 100, device=DEV)
    div = torch.randint(1, 9, (1000,), device=DEV).float()
    out = ops.row_div(x, div)
    torch.testing.assert_close(out, x / div[:, None], rtol=3e-7, atol=0)      # reciprocal-multiply: <= 1 ulp


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 1e-2), (torch.float32, 2e-5)])
@pytest.mark.parametrize("m,n,k0,k1", [(1000, 256, 256, 256), (4097, 256, 602, 0), (300, 41, 256, 256),
                                       (128, 16, 20, 20), (77, 128, 100, 100), (5000, 64, 64, 0)])
def test_linear_tcgen05(dtype, tol, m, n, k0, k1):
    """pg_linear (wgmma/TMA) vs fp64 matmul of the same (rounded) inputs; bf16: rel 1e-2 (bf16 output
    rounding), fp32 through the 3xTF32 product: rel 2e-5."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    g = torch.Generator().manual_seed(m + n)
    def mk(r, c):
        t = alloc_rows(r, c, dtype, DEV, zero=True)
        t.copy_(torch.randn(r, c, generator=g).to(dtype))
        return t
    a0, b0 = mk(m, k0), mk(n, k0)
    a1, b1 = (mk(m, k1), mk(n, k1)) if k1 else (None, None)
    bias = torch.randn(n, generator=g).to(DEV)
    div = torch.randint(1, 9, (m,), generator=g).float().to(DEV)
    out = ops.gemm_nt(a0, b0, a1, b1, bias=bias, row_div=div, out_dtype=torch.float32)
    ref = a0.double() @ b0.double().t()
    if k1:
        ref = ref + a1.double() @ b1.double().t()
    ref = (ref + bias.double()) / div.double()[:, None]
    scale = ref.abs().max().item()
    err = (out.double() - ref).abs().max().item()
    assert err <= tol * scale, f"max err {err} vs scale {scale}"
    out2 = ops.gemm_nt(a0, b0, a1, b1, out_dtype=dtype)                 # output in the activation dtype, no epilogue
    ref2 = a0.double() @ b0.double().t() + (a1.double() @ b1.double().t() if k1 else 0)
    assert (out2.double() - ref2).abs().max().item() <= 2 * tol * ref2.abs().max().item()


def test_sage_layer_fn_matches_torch():
    """Fused layer Function (aggregate + dual GEMM, and their gradients) vs torch autograd on the same inputs."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import PartGraph
    from tests.helpers import small_world
    _, _, layouts, _ = small_world("tiny", 2)
    L = layouts[0]
    graph = PartGraph.from_layout(L, device=DEV, seg_len=64)
    d_in, d_out = 24, 16
    torch.manual_seed(0)
    feat = torch.randn(L.num_all, d_in, device=DEV, requires_grad=True)
    w1 = torch.randn(d_out, d_in, device=DEV, requires_grad=True)
    w2 = torch.randn(d_out, d_in, device=DEV, requires_grad=True)
    b1 = torch.randn(d_out, device=DEV, requires_grad=True)
    b2 = torch.randn(d_out, device=DEV, requires_grad=True)
    go = torch.randn(L.num_in, d_out, device=DEV)
    out = ops.sage_layer(feat, graph, graph.in_deg_f, w1, b1, w2, b2)
    out.backward(go)
    got = [out.detach().clone()] + [t.grad.clone() for t in (feat, w1, b1, w2, b2)]
    for t in (feat, w1, b1, w2, b2):
        t.grad = None
    rows = torch.repeat_interleave(torch.arange(L.num_in, device=DEV), (L.indptr[1:] - L.indptr[:-1]).long().to(DEV))
    A = torch.zeros(L.num_in, L.num_all, device=DEV)
    A.index_put_((rows, L.indices.long().to(DEV)), torch.ones(rows.numel(), device=DEV), accumulate=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    ah = (A @ feat) / graph.in_deg_f[:, None]
    ref = feat[: L.num_in] @ w1.t() + b1 + ah @ w2.t() + b2
    ref.backward(go)
    want = [ref.detach()] + [t.grad for t in (feat, w1, b1, w2, b2)]
    for a, b in zip(got, want):
        assert (a - b).abs().max().item() <= 1e-4 * b.abs().max().item() + 1e-5     # 3xTF32 tensor-core product


@pytest.mark.parametrize("stage", [2, 0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,d,relu", [(3000, 16, True), (3001, 256, True), (3000, 512, True), (1237, 104, True),
                                      (1001, 264, False), (513, 1024, True), (7, 256, True), (70001, 256, True)])
def test_layer_norm_relu_matches_torch(dtype, n, d, relu, stage):
    """Full / partial last vector, 1 / 2 / 4 vectors per lane, row counts that leave a ragged last group, with the
    cp.async staging ring wherever it exists (ln_stage 2; the default 1 uses it for rows of one vector per lane) and
    with plain loads (0)."""
    from pipegcn_b200 import ops, _C
    from pipegcn_b200.graph import alloc_rows
    if d * (4 if dtype == torch.float32 else 2) > 2048:
        pytest.skip("row wider than 128 vectors")
    torch.manual_seed(d)
    y = alloc_rows(n, d, dtype, DEV)
    y.copy_(torch.randn(n, d, device=DEV) * 2 + 0.5)
    gamma = (torch.rand(d, device=DEV) + 0.5).requires_grad_(True)
    beta = torch.randn(d, device=DEV).requires_grad_(True)
    go = torch.randn(n, d, device=DEV).to(dtype)
    if relu:
        # a pre-activation within rounding of zero has no defined ReLU mask (two correct implementations may disagree on
        # its sign, and the whole row's gradient with it): such rows get the data of a row without one.  Seen on an H100
        # with (n, d, dtype) = (70001, 256, fp32), torch.manual_seed(256): row 34146 held a pre-activation of 1.03e-8 in
        # torch's fp32 LayerNorm and -8.3e-9 in fp64; the kernel masked it, torch did not, and all 256 gradients of
        # that row differed (the device generator's output depends on the GPU, so other GPUs draw other rows)
        pre = torch.nn.functional.layer_norm(y.detach().float(), (d,), gamma.detach(), beta.detach(), 1e-5)
        tie = (pre.abs() < 1e-6).any(1)
        assert int(tie.sum()) <= 1 + n // 1000
        y[tie] = y[(~tie).nonzero()[0, 0]].clone()
    yq = y.detach().clone().requires_grad_(True)
    assert ops.ln_relu_supported(yq)
    _C.check(_C.lib.pg_set_option(b"ln_stage", stage))
    try:
        out = ops.layer_norm_relu(yq, gamma, beta, 1e-5, relu=relu)
        out.backward(go)
        torch.cuda.synchronize()
    finally:
        _C.lib.pg_set_option(b"ln_stage", 1)
    got = [out.detach().float(), yq.grad.float(), gamma.grad.clone(), beta.grad.clone()]
    colsum = ops._take_colsum(yq.grad)
    gamma.grad = beta.grad = None
    yr = y.detach().float().clone().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(yr, (d,), gamma, beta, 1e-5)
    if relu:
        ref = torch.relu(ref)
    ref.backward(go.float())
    want = [ref.detach(), yr.grad, gamma.grad, beta.grad]
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    for a, b in zip(got, want):
        assert (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1.0)
    assert colsum is not None
    assert (colsum - got[1].sum(0)).abs().max().item() <= 1e-3 * max(got[1].sum(0).abs().max().item(), 1.0)


@pytest.mark.parametrize("p", [0.5, 0.3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n,d", [(2049, 256), (515, 104)])
def test_layer_norm_fused_dropout_is_dropout_of_the_clean_result(dtype, n, d, p):
    """pg_ln_relu_drop_fwd writes the clean result and dropout(clean result) in one pass: both must be BIT-identical to
    the two separate kernels (p = 0.5 takes the shortcut that scales before rounding, p = 0.3 the general path)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    torch.manual_seed(n)
    y = alloc_rows(n, d, dtype, DEV)
    y.copy_(torch.randn(n, d, device=DEV) * 3 - 0.2)
    gamma, beta = torch.rand(d, device=DEV) + 0.5, torch.randn(d, device=DEV)
    step = torch.full((1,), 4, dtype=torch.int32, device=DEV)
    spec = ops.DropSpec(p, 98765, step, 1)
    out, clean = alloc_rows(n, d, dtype, DEV), alloc_rows(n, d, dtype, DEV)
    ops.layer_norm_relu(y, gamma, beta, 1e-5, True, out, clean, spec)
    plain = ops.layer_norm_relu(y, gamma, beta, 1e-5, True)
    assert torch.equal(clean, plain)
    assert torch.equal(out, ops.dropout_rows(plain, spec))
    kept = (out != 0).float().sum().item() / max((plain != 0).float().sum().item(), 1.0)
    assert abs(kept - (1 - p)) < 0.01


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_layer_norm_backward_mask_from_output_equals_recomputed_mask(dtype):
    """pg_ln_relu_bwd (ReLU mask read from the forward output) and pg_ln_relu_bwd2 (mask recomputed from y with the
    forward's own expression) give the same gradient."""
    import ctypes as C
    from pipegcn_b200 import ops, _C
    from pipegcn_b200.graph import alloc_rows
    n, d = 1501, 256
    torch.manual_seed(5)
    y = alloc_rows(n, d, dtype, DEV)
    y.copy_(torch.randn(n, d, device=DEV))
    gamma, beta = torch.rand(d, device=DEV) + 0.5, torch.randn(d, device=DEV)
    out, mean, rstd = alloc_rows(n, d, dtype, DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    code, st = _C.dtype_code(dtype), _C.stream_ptr()
    _C.check(_C.lib.pg_ln_relu_fwd(y.data_ptr(), y.stride(0), gamma.data_ptr(), beta.data_ptr(), 1e-5, 1, out.data_ptr(),
                                   out.stride(0), mean.data_ptr(), rstd.data_ptr(), n, d, code, st))
    g = alloc_rows(n, d, dtype, DEV)
    g.copy_(torch.randn(n, d, device=DEV))
    res = []
    for with_beta in (False, True):
        g_y = alloc_rows(n, d, dtype, DEV)
        red = torch.empty(3, d, device=DEV)
        partial = torch.empty(_C.lib.pg_row_grid(n) * 3 * d, device=DEV)
        if with_beta:
            _C.check(_C.lib.pg_ln_relu_bwd2(g.data_ptr(), g.stride(0), None, 0, y.data_ptr(), y.stride(0), mean.data_ptr(),
                                            rstd.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1, g_y.data_ptr(),
                                            g_y.stride(0), red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(),
                                            partial.data_ptr(), n, d, code, st))
        else:
            _C.check(_C.lib.pg_ln_relu_bwd(g.data_ptr(), g.stride(0), out.data_ptr(), out.stride(0), y.data_ptr(),
                                           y.stride(0), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), 1,
                                           g_y.data_ptr(), g_y.stride(0), red[0].data_ptr(), red[1].data_ptr(),
                                           red[2].data_ptr(), partial.data_ptr(), n, d, code, st))
        res.append((g_y.clone(), red.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("c,padded", [(41, False), (41, True), (64, True), (7, True), (172, True), (300, True), (1, True)])
def test_cross_entropy_sum_matches_torch(dtype, c, padded):
    """padded: rows from alloc_rows (16-byte aligned stride: the sub-warp kernels, 1 .. 32 lanes per row, 1 .. 2 vectors
    per lane); not padded: a contiguous [n, c] tensor whose rows are not 16-byte aligned (one warp per row)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    n, n_train = 5003, 3211
    torch.manual_seed(1)
    src = (torch.randn(n, c, device=DEV) * 3).to(dtype)
    if padded:
        z = alloc_rows(n, c, dtype, DEV)
        z.copy_(src)
        z.requires_grad_(True)
    else:
        z = src.clone().requires_grad_(True)
    labels = torch.randint(0, c, (n_train,), device=DEV)
    loss = ops.cross_entropy_sum(z, labels, n_train)
    g = torch.autograd.grad(loss * 0.5, z)[0]               # the tensor the backward produced (padded rows included)
    zr = src.float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(zr[:n_train], labels, reduction="sum")
    (ref * 0.5).backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert (g.float() - zr.grad).abs().max().item() <= tol
    assert torch.count_nonzero(g[n_train:]) == 0
    colsum = ops._take_colsum(g)
    assert colsum is not None
    want = g.float().sum(0)
    assert (colsum - want).abs().max().item() <= 1e-4 * max(want.abs().max().item(), 1.0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dropout_kernel(dtype):
    """Keep rate, scaling, and the backward regenerating the forward's mask."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    x = alloc_rows(4000, 100, dtype, DEV)
    x.fill_(1.0)
    xr = x.detach().clone().requires_grad_(True)
    assert xr.stride(0) == 100 or True
    xin = alloc_rows(4000, 100, dtype, DEV)
    xin.copy_(x)
    xin.requires_grad_(True)
    out = ops.dropout(xin, 0.3, True)
    keep = (out != 0)
    rate = keep.float().mean().item()
    assert abs(rate - 0.7) < 0.01
    assert torch.allclose(out[keep].float(), torch.full_like(out[keep], 1 / 0.7).float(), rtol=1e-2)
    out.backward(torch.ones_like(out))
    assert torch.equal(xin.grad != 0, keep)
    out2 = ops.dropout(xin, 0.3, True)
    assert not torch.equal(out2 != 0, keep)          # a new mask every call
    assert ops.dropout(xin, 0.0, True) is xin and ops.dropout(xin, 0.5, False) is xin


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [100, 256, 602])
def test_chunked_kernel_equals_row_kernel(dtype, d):
    """agg_impl 2 (chunks of whole short rows / one row / one segment per warp, indices loaded coalesced and
    broadcast by shuffles) and agg_impl 3 (long rows staged through shared memory with cp.async) sum every row in
    the same order as agg_impl 1: bit-identical results, including rows
    without entries, rows longer than the segment length, the division and the accumulate mode."""
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.graph import CsrPlan, alloc_rows
    n_rows, n_cols = 5000, 4000
    indptr, indices = _random_csr(n_rows, n_cols, 6, seed=d, hubs=4, hub_deg=1500)
    plan = CsrPlan(indptr.to(DEV), indices.to(DEV), seg_len=256)
    assert plan.n_chunks > 0 and plan.n_long == 4
    g = torch.Generator().manual_seed(3)
    x = alloc_rows(n_cols, d, dtype, DEV, zero=True)
    x.copy_(torch.randn(n_cols, d, generator=g).to(dtype))
    div = torch.randint(1, 9, (n_rows,), generator=g).float().to(DEV)
    base = alloc_rows(n_rows, d, dtype, DEV, zero=True)
    base.copy_(torch.randn(n_rows, d, generator=g).to(dtype))
    outs = []
    try:
        for impl in (1, 2, 3):
            _C.check(_C.lib.pg_set_option(b"agg_impl", impl))
            o = base.clone()
            o2 = alloc_rows(n_rows, d, dtype, DEV)
            o2.copy_(base)
            ops.aggregate(plan, x, out=o2, row_div=div, acc_rows=1234)
            outs.append((ops.aggregate(plan, x, row_div=div).clone(), o2.clone()))
    finally:
        _C.lib.pg_set_option(b"agg_impl", 2)
    for o in outs[1:]:
        assert torch.equal(outs[0][0], o[0]) and torch.equal(outs[0][1], o[1])
    ref = _ref_agg(indptr, indices, x.float().cpu(), div.cpu())
    tol = 2e-5 if dtype == torch.float32 else 1.6e-2
    assert (outs[1][0].float().cpu().double() - ref).abs().max().item() <= tol * ref.abs().max().item() + 1e-6


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("m,n,k", [(5000, 256, 256), (70000, 256, 256), (3000, 64, 256), (2500, 41, 602), (1, 16, 8),
                                   (63, 128, 100), (12345, 200, 1204)])
def test_wgrad_matches_torch(dtype, m, n, k):
    """pg_wgrad (MN-major wgmma, split-K over the rows) == g^T @ x in fp64: bf16 exact products with fp32
    accumulation (rel. 1e-5 of the output scale), fp32 through six products of bf16 terms (rel. 3e-5)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    gen = torch.Generator().manual_seed(m + n + k)
    g = alloc_rows(m, n, dtype, DEV, zero=True)
    x = alloc_rows(m, k, dtype, DEV, zero=True)
    g.copy_(torch.randn(m, n, generator=gen).to(dtype))
    x.copy_(torch.randn(m, k, generator=gen).to(dtype))
    out = ops.wgrad(g, x)
    assert out.shape == (n, k) and out.dtype == torch.float32
    ref = g.double().cpu().t() @ x.double().cpu()
    err = (out.double().cpu() - ref).abs().max().item()
    assert err <= 3e-5 * max(ref.abs().max().item(), 1.0) + 1e-6, (err, ref.abs().max().item())
    # deterministic: same partials, same order
    assert torch.equal(out, ops.wgrad(g, x))
