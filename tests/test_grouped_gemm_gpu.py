"""The grouped GEMM launches (pg_linear_group, pg_wgrad_group) give every product the bits of its own launch.

A grouped launch only reorders which CTA computes which tile, so each output must equal, bit for bit, the same product
run alone (pg_linear_drop / ops.wgrad).  Sizes run past the first wave (a few hundred thousand rows, not a multiple of
the 128-row tile) on every output width the kernels instantiate.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
M = 300_007                  # > 16 M tiles per SM on an H100, and 128 does not divide it
SHAPES = [(64, 192), (192, 256), (256, 64)]     # (n, k): every N tile of the kernels, every K width in use


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


def _rand(rows, cols, dtype, gen):
    from pipegcn_b200.graph import alloc_rows
    out = alloc_rows(rows, cols, dtype, DEV)
    out.copy_(torch.randn(rows, cols, device=DEV, generator=gen))
    return out


def _srcs(a_list, b_list):
    from pipegcn_b200 import _C
    return [_C.pg_gemm_src(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), a.shape[1])
            for a, b in zip(a_list, b_list)]


def _problem_opts(q, mixed, n, gen):
    """bias / row scale / dropout / output alignment of problem q ("mixed": a different set for every problem)."""
    if not mixed:
        return dict(bias=None, row_div=None, drop=None, aligned=True)
    from pipegcn_b200 import ops
    step = torch.tensor([4], dtype=torch.int32, device=DEV)
    return dict(bias=torch.randn(n, device=DEV, generator=gen) if q % 2 == 0 else None,
                row_div=torch.randint(1, 9, (M,), device=DEV, generator=gen).float() if q >= 1 else None,
                drop=ops.DropSpec(0.3, 0x5EED0000 + q, step, q) if q in (1, 3) else None,
                # problem 2 stores through the plain (unaligned-row) epilogue, between problems that store with TMA
                aligned=q != 2)


@pytest.mark.parametrize("mixed", [False, True], ids=["plain", "bias-rowdiv-dropout"])
@pytest.mark.parametrize("n,k", SHAPES, ids=[f"n{n}-k{k}" for n, k in SHAPES])
@pytest.mark.parametrize("n_prob", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32-3xtf32"])
def test_linear_group_bitwise(dtype, n_prob, n, k, mixed):
    from pipegcn_b200 import _C, ops
    gen = torch.Generator(device=DEV).manual_seed(1000 * n_prob + n + k + mixed)
    a = _rand(M, k, dtype, gen)
    bs = [_rand(n, k, dtype, gen) for _ in range(n_prob)]
    if dtype == torch.float32:           # the 3xTF32 product: hi*hi + hi*lo + lo*hi
        ah, al = ops.split_tf32(a)
        a_list = [ah, ah, al]
        b_lists = []
        for b in bs:
            bh, bl = ops.split_tf32(b)
            b_lists.append([bh, bl, bh])
    else:
        a_list, b_lists = [a], [[b] for b in bs]
    n_src = len(a_list)
    opts = [_problem_opts(q, mixed, n, gen) for q in range(n_prob)]
    code = _C.dtype_code(dtype)

    def output(aligned):
        ld = n + 8 if aligned else n + 1       # fp32 and bf16: n + 1 elements is not a multiple of 16 bytes
        return torch.full((M, ld), float("nan"), dtype=dtype, device=DEV)[:, :n]

    keep, outs, grouped = [], [], []
    for o in opts:
        c = output(o["aligned"])
        dc = o["drop"].c() if o["drop"] is not None else None
        keep.append(dc)
        grouped.append(c)
        outs.append(_C.pg_gemm_out(o["bias"].data_ptr() if o["bias"] is not None else None,
                                   o["row_div"].data_ptr() if o["row_div"] is not None else None,
                                   c.data_ptr(), c.stride(0), C.addressof(dc) if dc is not None else None, 7 * M))
    srcs = [s for bl in b_lists for s in _srcs(a_list, bl)]
    _C.check(_C.lib.pg_linear_group(code, code, (_C.pg_gemm_src * len(srcs))(*srcs), n_src, n_prob,
                                    (_C.pg_gemm_out * n_prob)(*outs), M, n, _C.stream_ptr()), "pg_linear_group")
    for o, bl, got in zip(opts, b_lists, grouped):
        want = output(o["aligned"])
        srcs = _srcs(a_list, bl)
        dc = o["drop"].c() if o["drop"] is not None else None
        _C.check(_C.lib.pg_linear_drop(code, code, (_C.pg_gemm_src * n_src)(*srcs), n_src,
                                       o["bias"].data_ptr() if o["bias"] is not None else None,
                                       o["row_div"].data_ptr() if o["row_div"] is not None else None,
                                       want.data_ptr(), want.stride(0), M, n, C.byref(dc) if dc is not None else None,
                                       7 * M, _C.stream_ptr()), "pg_linear_drop")
        assert not got.isnan().any()
        assert torch.equal(_bits(got), _bits(want))


def test_gemm_nt_group_matches_gemm_nt():
    """ops.gemm_nt_group (the dX products of a layer backward) == one ops.gemm_nt per product."""
    from pipegcn_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(5)
    g = _rand(M, 256, torch.bfloat16, gen)
    w1, w2 = _rand(256, 256, torch.bfloat16, gen), _rand(256, 256, torch.bfloat16, gen)
    div = torch.randint(1, 50, (M,), device=DEV, generator=gen).float()
    got = ops.gemm_nt_group(g, [w1, w2], row_divs=[None, div])
    want = [ops.gemm_nt(g, w1), ops.gemm_nt(g, w2, row_div=div)]
    for x, y in zip(got, want):
        assert torch.equal(_bits(x), _bits(y))


WGRAD_CASES = {
    "shared-g": lambda g, x, ah, dz: [(g, x), (g, ah)],                 # aggregate-first layer: g^T x, g^T ah
    "shared-x-ragged": lambda g, x, ah, dz: [(g[:251_001], x[:251_001]), (dz, x)],   # narrow layer: inner rows, all rows
}


@pytest.mark.parametrize("case", list(WGRAD_CASES))
@pytest.mark.parametrize("n,k", SHAPES, ids=[f"n{n}-k{k}" for n, k in SHAPES])
@pytest.mark.parametrize("n_prob", [1, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32-bf16x3"])
def test_wgrad_group_bitwise(dtype, n_prob, n, k, case):
    from pipegcn_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(10 * n_prob + n + k)
    g, dz = _rand(M, n, dtype, gen), _rand(M, n, dtype, gen)
    x, ah = _rand(M, k, dtype, gen), _rand(M, k, dtype, gen)
    pairs = WGRAD_CASES[case](g, x, ah, dz)[:n_prob]
    with_split = dtype == torch.float32
    if with_split:
        pairs = [(ops.Split(a), ops.Split(b)) for a, b in pairs]     # as the layers pass them in 3xTF32 mode
    got = ops.wgrad_group(pairs)
    for (a, b), out in zip(pairs, got):
        want = ops.wgrad(a, b)
        assert torch.equal(_bits(out), _bits(want))
