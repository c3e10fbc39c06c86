"""Conformance of the hot-path kernels (GEMM, weight gradient, neighbour aggregate, row kernels) with plain fp64
restatements of the same operations, past the first wave of CTAs and on every dispatch path.

Conventions:
- Inputs live in `padded` storage (the alloc_rows layout) whose pad columns hold NaN; outputs go to `Guarded` views
  whose surroundings hold a sentinel bit pattern that must survive every call bit for bit.
- Bounds are elementwise, |got - ref| <= c * mag with mag the same sum over absolute values, so that one wrong tile,
  row or column fails.  Each c is derived next to its use from the product scheme; a bf16 output adds one rounding.
- Sizes come from the device's SM count: the persistent GEMM runs min(tiles, SMs) CTAs, so "3w" = 3 * SMs * 128 rows
  gives every CTA three tiles and "2w+77" gives every CTA two tiles and some a third, ragged one.
- Where a sum over many terms would make the worst-case bound meaningless (2^17 rows, tensors past 2 GiB), the data
  are small integers: every partial sum is an integer below 2^24, exact in fp32 in any order, so the result must
  equal the fp64 one exactly.
- Options set through pg_set_option are process-wide: `knobs` restores the documented defaults afterwards.
"""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
U24 = 2.0 ** -24        # unit roundoff of an fp32 operation rounded to nearest
U23 = 2.0 ** -23        # per add of an fp32 accumulator that may truncate (tensor-core accumulation)
BF16_U = 2.0 ** -8      # one bf16 rounding to nearest (8 significant bits)

# documented defaults of pg_set_option (include/pipegcn_b200.h)
DEFAULTS = dict(agg_impl=2, agg_unroll=8, agg_pack_short=0, agg_occ=4, agg_overlap=1, agg_narrow=1, agg_l2_hint=0,
                ln_stage=1, ce_subwarp=1, gemm_epi_slabs=2)


@functools.lru_cache(None)
def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def rows_of(case: str) -> int:
    """GEMM row counts named by what they make the persistent kernel do."""
    w = sm_count() * 128
    return {"1": 1, "127": 127, "129": 129, "3w": 3 * w, "2w+77": 2 * w + 77}[case]


@contextlib.contextmanager
def knobs(fp32_gemm=None, **opts):
    """Set kernel options (and ops.FP32_GEMM) for the body; restore the defaults whatever happens."""
    from pipegcn_b200 import _C, ops
    saved = ops.FP32_GEMM
    try:
        for k, v in opts.items():
            _C.check(_C.lib.pg_set_option(k.encode(), int(v)), "pg_set_option")
        if fp32_gemm is not None:
            ops.FP32_GEMM = fp32_gemm
        yield
    finally:
        for k, v in DEFAULTS.items():
            _C.lib.pg_set_option(k.encode(), v)
        ops.FP32_GEMM = saved


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


SENTINEL = {torch.float32: 0x7FA5A5A5, torch.bfloat16: 0x7FA5}     # NaN payloads no kernel produces


def padded(n, d, dtype, fill=float("nan"), data=None):
    """An alloc_rows-shaped [n, d] view whose pad columns hold `fill`."""
    ld = (d + 7) // 8 * 8
    base = torch.full((max(n, 1), ld), fill, dtype=dtype, device=DEV)
    t = base[:n, :d]
    if data is not None:
        t.copy_(data)
    return t


class Guarded:
    """Output view [n, d] inside a larger allocation: G guard rows above and below, `col0` guard columns on the left
    and everything right of the allowed region, all holding SENTINEL.  The allowed region of a row is the header's:
    columns up to the end of the 16-byte vector holding column d-1 (`exact`: up to column d-1)."""
    G = 3

    def __init__(self, n, d, dtype, col0=0, ld=None):
        self.n, self.d, self.col0, self.dtype = n, d, col0, dtype
        self.ld = ld if ld is not None else (col0 + d + 7) // 8 * 8 + 8
        self.base = torch.empty(n + 2 * self.G, self.ld, dtype=dtype, device=DEV)
        _bits(self.base).fill_(SENTINEL[dtype])
        self.t = self.base[self.G:self.G + n, col0:col0 + d]

    def check(self, exact=False):
        v = 16 // self.base.element_size()
        end = self.col0 + (self.d if exact else (self.d + v - 1) // v * v)
        b, s, G, n = _bits(self.base), SENTINEL[self.dtype], self.G, self.n
        assert bool((b[:G] == s).all()) and bool((b[G + n:] == s).all()), "write into the guard rows"
        assert bool((b[G:G + n, :self.col0] == s).all()), "write left of the output"
        assert bool((b[G:G + n, end:] == s).all()), "write right of the allowed columns"


def assert_within(got, ref, mag, c, bf16_out, what):
    """|got - ref| <= c * mag elementwise (+ one bf16 rounding of the result for bf16 outputs)."""
    bound = c * mag
    if bf16_out:
        bound = bound + BF16_U * (ref.abs() + bound)
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound, first {idx}: got "
                             f"{got[tuple(idx)].item()} ref {ref[tuple(idx)].item()} bound {bound[tuple(idx)].item()}")


def _normal(shape, gen, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV)


def _ints(shape, lo, hi, gen):
    return torch.randint(lo, hi + 1, shape, generator=gen).to(DEV)


# ================================================ GEMM ==============================================================
def linear_c(pairs, out, bias=None, div=None, drop=None, drop_row0=0):
    """pg_linear / pg_linear_drop through the C ABI: out[m, n] = sum a_s b_s^T; pairs of [m, k_s] x [n, k_s]."""
    from pipegcn_b200 import _C
    m, n = out.shape
    srcs = (_C.pg_gemm_src * len(pairs))(*[_C.pg_gemm_src(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                                                           a.shape[1]) for a, b in pairs])
    din, dout = _C.dtype_code(pairs[0][0].dtype), _C.dtype_code(out.dtype)
    bp = bias.data_ptr() if bias is not None else None
    dp = div.data_ptr() if div is not None else None
    if drop is not None:
        rc = _C.lib.pg_linear_drop(din, dout, srcs, len(pairs), bp, dp, out.data_ptr(), out.stride(0), m, n,
                                   C.byref(drop.c()), int(drop_row0), _C.stream_ptr())
    else:
        rc = _C.lib.pg_linear(din, dout, srcs, len(pairs), bp, dp, out.data_ptr(), out.stride(0), m, n, _C.stream_ptr())
    _C.check(rc, "pg_linear")
    return out


def gemm_ref(pairs, bias=None, div=None):
    ref = sum(a.double() @ b.double().t() for a, b in pairs)
    mag = sum(a.double().abs() @ b.double().abs().t() for a, b in pairs)
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    if div is not None:
        ref, mag = ref / div.double()[:, None], mag / div.double()[:, None]
    return ref, mag


# Bounds of the product schemes, relative to mag = |A| |B|^T (+ |bias|) (/ div), K = products summed per output:
# - bf16 operands: every product is exact in fp32 (8 x 8 significant bits); the tensor core adds K of them into an
#   fp32 accumulator (each add within one ulp: U23, also if the adder truncates), then bias add, reciprocal and
#   multiply round once each: c = (K + 3) * U23.
# - 3xTF32 (hi*hi + hi*lo + lo*hi, hi = x truncated to 11 significant bits, |lo| < 2^-10 |x|): the tensor core
#   truncates lo to tf32 (relative error < 2^-10, so < 2^-20 of |x| in each of the two cross products) and drops
#   lo*lo (< 2^-20): 3 * 2^-20 per product, plus 3K accumulated products: c = 3 * 2^-20 + (3K + 3) * U23.
# - one-pass tf32: both operands truncated to 11 significant bits (< 2^-10 each): c = 2^-9 + (K + 3) * U23.
def c_bf16(K):
    return (K + 3) * U23


def c_3xtf32(K):
    return 3 * 2.0 ** -20 + (3 * K + 3) * U23


def c_tf32(K):
    return 2.0 ** -9 + (K + 3) * U23


GEMM_N = [1, 8, 41, 64, 65, 128, 129, 172, 192, 193, 256]


def _nt(n):
    return 64 if n <= 64 else 128 if n <= 128 else 192 if n <= 192 else 256


@pytest.mark.parametrize("n", GEMM_N, ids=[f"n{n}-NT{_nt(n)}" for n in GEMM_N])
@pytest.mark.parametrize("mcase", ["1", "127", "129", "3w", "2w+77"],
                         ids=["m1", "m127-one-ragged-tile", "m129-two-tiles", "m3w-three-tiles-per-CTA",
                              "m2w+77-second-and-ragged-third-tile"])
def test_gemm_tiles(mcase, n):
    """pg_linear at the edges of every N tile (NT = 64/128/192/256 for n rounded up) and with every CTA running
    several tiles (the mbarrier phases, the slab parity and the producer's next-tile prefetch carry over): bf16 with
    two pairs of different k (602 + 100) and bias + row_div into fp32, the same into bf16 without the epilogue
    operands, and fp32 through 3xTF32 (256 + 8: six sources).  Operand pad columns hold NaN; two launches agree.

    Contract note: with n % (16 / elem) != 0 the TMA store also writes (zeros into) the rest of the 16-byte vector
    holding column n-1 -- seen on an H100 for every such n here.  The header did not say so; it now does, and the
    guard check allows exactly that region (the direct epilogue writes columns [0, n) only)."""
    from pipegcn_b200 import ops
    m = rows_of(mcase)
    gen = torch.Generator().manual_seed(m * 1000 + n)
    bias = _normal((n,), gen)
    div = _ints((m,), 1, 9, gen).float()
    # bf16, two pairs of different k
    pairs = [(padded(m, k, torch.bfloat16, data=_normal((m, k), gen)), padded(n, k, torch.bfloat16, data=_normal((n, k), gen)))
             for k in (602, 100)]
    ref, mag = gemm_ref(pairs, bias, div)
    out = Guarded(m, n, torch.float32)
    ops.gemm_nt(pairs[0][0], pairs[0][1], pairs[1][0], pairs[1][1], bias=bias, row_div=div, out=out.t)
    out.check()
    assert_within(out.t, ref, mag, c_bf16(702), False, "bf16 -> fp32, bias, row_div")
    again = ops.gemm_nt(pairs[0][0], pairs[0][1], pairs[1][0], pairs[1][1], bias=bias, row_div=div,
                        out_dtype=torch.float32)
    assert torch.equal(_bits(again), _bits(out.t)), "two launches differ"
    ref2, mag2 = gemm_ref(pairs)
    out2 = Guarded(m, n, torch.bfloat16)
    ops.gemm_nt(pairs[0][0], pairs[0][1], pairs[1][0], pairs[1][1], out=out2.t)
    out2.check()
    assert_within(out2.t, ref2, mag2, c_bf16(702), True, "bf16 -> bf16")
    # fp32 operands through 3xTF32
    fp = [(padded(m, k, torch.float32, data=_normal((m, k), gen)), padded(n, k, torch.float32, data=_normal((n, k), gen)))
          for k in (256, 8)]
    ref3, mag3 = gemm_ref(fp, bias, div)
    with knobs(fp32_gemm="3xtf32"):
        out3 = ops.gemm_nt(fp[0][0], fp[0][1], fp[1][0], fp[1][1], bias=bias, row_div=div)
    assert_within(out3, ref3, mag3, c_3xtf32(264), False, "3xTF32 fp32")


@pytest.mark.parametrize("ks", [(602,), (602, 100), (8, 256), (602, 100, 8), (602, 100, 8, 256),
                                (602, 100, 8, 256, 64), (602, 100, 8, 256, 64, 72)],
                         ids=lambda ks: f"nsrc{len(ks)}-k" + "+".join(map(str, ks)))
def test_gemm_sources(ks):
    """1 to 6 independent bf16 operand pairs with different k (kb_end is built per source), NT=192, second tile."""
    m, n = rows_of("2w+77"), 172
    gen = torch.Generator().manual_seed(len(ks) + sum(ks))
    pairs = [(padded(m, k, torch.bfloat16, data=_normal((m, k), gen)), padded(n, k, torch.bfloat16, data=_normal((n, k), gen)))
             for k in ks]
    bias = _normal((n,), gen)
    div = _ints((m,), 1, 9, gen).float()
    out = Guarded(m, n, torch.float32)
    linear_c(pairs, out.t, bias, div)
    out.check()
    ref, mag = gemm_ref(pairs, bias, div)
    assert_within(out.t, ref, mag, c_bf16(sum(ks)), False, f"{len(ks)} sources")


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["out-f32", "out-bf16"])
@pytest.mark.parametrize("n", [64, 192, 256], ids=lambda n: f"NT{n}")
def test_gemm_epilogue_slabs(n, out_dtype):
    """gemm_epi_slabs = 1 (every chunk waits for the previous TMA store) and 2 (double-buffered) write the same bits,
    over three tiles per CTA."""
    m = rows_of("3w")
    gen = torch.Generator().manual_seed(n)
    pairs = [(padded(m, 256, torch.bfloat16, data=_normal((m, 256), gen)),
              padded(n, 256, torch.bfloat16, data=_normal((n, 256), gen)))]
    bias, div = _normal((n,), gen), _ints((m,), 1, 9, gen).float()
    outs = []
    for slabs in (1, 2):
        with knobs(gemm_epi_slabs=slabs):
            o = Guarded(m, n, out_dtype)
            linear_c(pairs, o.t, bias, div)
            o.check()
            outs.append(o.t)
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
    ref, mag = gemm_ref(pairs, bias, div)
    assert_within(outs[0], ref, mag, c_bf16(256), out_dtype == torch.bfloat16, "slabs = 1")


@pytest.mark.parametrize("how", ["base+1", "ldc-odd"], ids=["direct-epilogue-base-plus-one", "direct-epilogue-odd-ldc"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["out-f32", "out-bf16"])
def test_gemm_direct_epilogue(out_dtype, how):
    """Outputs whose rows are not 16-byte aligned take epilogue_direct (plain stores from the registers); it computes
    (acc + bias) * (1 / div) like the TMA epilogue, so the bits equal those of an aligned output, and it writes
    nothing outside [0, m) x [0, n)."""
    m, n = rows_of("2w+77"), 172
    gen = torch.Generator().manual_seed(7)
    pairs = [(padded(m, k, torch.bfloat16, data=_normal((m, k), gen)), padded(n, k, torch.bfloat16, data=_normal((n, k), gen)))
             for k in (256, 72)]
    bias, div = _normal((n,), gen), _ints((m,), 1, 9, gen).float()
    aligned = Guarded(m, n, out_dtype)
    linear_c(pairs, aligned.t, bias, div)
    out = Guarded(m, n, out_dtype, col0=1) if how == "base+1" else Guarded(m, n, out_dtype, ld=n + 3)
    es = out.base.element_size()
    assert out.t.data_ptr() % 16 != 0 or (out.t.stride(0) * es) % 16 != 0      # not TMA-storable: direct epilogue
    linear_c(pairs, out.t, bias, div)
    out.check(exact=True)
    assert torch.equal(_bits(out.t), _bits(aligned.t))


@pytest.mark.parametrize("n", [65, 192], ids=["NT128-edge", "NT192-full"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32-3xtf32"])
def test_gemm_nan_confined(dtype, n):
    """A NaN in one row of A (in a second-wave tile) and one row of B (the last output column) makes exactly that
    output row and column NaN; the NaN pad columns of both operands are never read."""
    from pipegcn_b200 import ops
    m = rows_of("2w+77")
    gen = torch.Generator().manual_seed(n)
    a = padded(m, 300, dtype, data=_normal((m, 300), gen))
    b = padded(n, 300, dtype, data=_normal((n, 300), gen))
    r = (sm_count() + 3) * 128 + 5                         # tile sm_count + 3: a CTA's second tile
    a[r, 77] = float("nan")
    b[n - 1, 3] = float("nan")
    with knobs(fp32_gemm="3xtf32"):
        out = ops.gemm_nt(a, b, bias=_normal((n,), gen), out_dtype=torch.float32)
    want = torch.zeros(m, n, dtype=torch.bool, device=DEV)
    want[r, :] = True
    want[:, n - 1] = True
    assert torch.equal(out.isnan(), want)


@pytest.mark.parametrize("row0", [0, 12345], ids=lambda r: f"drop_row0-{r}")
@pytest.mark.parametrize("p", [0.5, 0.3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32-3xtf32", "bf16"])
def test_gemm_fused_dropout(dtype, p, row0):
    """pg_linear_drop is bit-identical to pg_linear followed by pg_dropout_rows(row0 = drop_row0) (the kernel
    rounds a bf16 output before masking), on NT=192 with several tiles per CTA; its mask equals the host port."""
    from pipegcn_b200 import ops
    m, n = rows_of("2w+77"), 172
    gen = torch.Generator().manual_seed(row0 + int(p * 10))
    a = padded(m, 256, dtype, data=_normal((m, 256), gen))
    b = padded(n, 256, dtype, data=_normal((n, 256), gen))
    bias, div = _normal((n,), gen), _ints((m,), 1, 9, gen).float()
    step = torch.tensor([9], dtype=torch.int32, device=DEV)
    spec = ops.DropSpec(p, 0x5EED5EED12345678, step, 2)
    with knobs(fp32_gemm="3xtf32"):
        fused = ops.gemm_nt(a, b, bias=bias, row_div=div, drop=spec, drop_row0=row0)
        clean = ops.gemm_nt(a, b, bias=bias, row_div=div)
    sep = ops.dropout_rows(clean, spec, row0=row0)
    assert torch.equal(_bits(fused), _bits(sep))
    keep = torch.from_numpy(ops.dropout_keep_host(spec, 9, row0, m, n, fused.element_size())).to(DEV)
    nz = clean != 0
    assert torch.equal((fused != 0) & nz, keep & nz)


@pytest.mark.parametrize("kind", ["normal", "subnormal", "strided"])
def test_split_tf32(kind):
    """hi has its 13 low mantissa bits clear and hi + lo == x exactly."""
    from pipegcn_b200 import ops
    gen = torch.Generator().manual_seed(3)
    n, d = 3001, 77
    if kind == "normal":
        x = _normal((n, d), gen) * torch.exp2(_ints((n, d), -60, 60, gen).float())
    elif kind == "subnormal":
        x = _normal((n, d), gen) * 1e-40
        assert bool((x.abs() < 1.1754944e-38).all())
    else:
        wide = _normal((n, d + 9), gen)
        x = wide[:, 3:3 + d]                               # row stride d + 9, base not 16-byte aligned
    hi, lo = ops.split_tf32(x)
    assert bool(((_bits(hi) & 0x1FFF) == 0).all())
    assert torch.equal(hi + lo, x) and torch.equal(hi.double() + lo.double(), x.double())
    assert torch.equal(_bits(hi), _bits(x) & ~0x1FFF)


@pytest.mark.parametrize("n", [300, 602], ids=["n300-two-slices", "n602-three-slices"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gemm_nt_wider_than_one_tile(dtype, n):
    """gemm_nt splits n > 256 into 256-column products.  The result matches fp64 and keeps the layout contract of
    every other output (16-byte aligned, padded rows), so it can feed the TMA loads of the next GEMM directly.

    Regression: the slices used to be joined with torch.cat, whose rows have stride n; for bf16 with n % 8 != 0
    (n = 300) they were not 16-byte aligned, and the next pg_linear refused them."""
    from pipegcn_b200 import ops
    m = 3000
    gen = torch.Generator().manual_seed(n)
    a = padded(m, 128, dtype, data=_normal((m, 128), gen))
    b = padded(n, 128, dtype, data=_normal((n, 128), gen))
    bias, div = _normal((n,), gen), _ints((m,), 1, 9, gen).float()
    with knobs(fp32_gemm="3xtf32"):
        out = ops.gemm_nt(a, b, bias=bias, row_div=div)
    es = out.element_size()
    assert out.data_ptr() % 16 == 0 and (out.stride(0) * es) % 16 == 0 and out.stride(0) >= (n + 7) // 8 * 8
    ref, mag = gemm_ref([(a, b)], bias, div)
    c = c_3xtf32(128) if dtype == torch.float32 else c_bf16(128)
    assert_within(out, ref, mag, c, dtype == torch.bfloat16, f"n={n}")
    w = padded(16, n, dtype, data=_normal((16, n), gen))
    nxt = linear_c([(out, w)], torch.empty(m, 16, device=DEV))        # out is a TMA operand as it stands
    ref2, mag2 = gemm_ref([(out, w)])
    assert_within(nxt, ref2, mag2, c_tf32(n) if dtype == torch.float32 else c_bf16(n), False, "next GEMM")


def test_gemm_one_pass_tf32():
    """ops.FP32_GEMM = "tf32": one tf32 product per pair, with its own (coarser) bound."""
    from pipegcn_b200 import ops
    m, n = rows_of("2w+77"), 193
    gen = torch.Generator().manual_seed(11)
    pairs = [(padded(m, k, torch.float32, data=_normal((m, k), gen)), padded(n, k, torch.float32, data=_normal((n, k), gen)))
             for k in (256, 40)]
    bias, div = _normal((n,), gen), _ints((m,), 1, 9, gen).float()
    with knobs(fp32_gemm="tf32"):
        out = ops.gemm_nt(pairs[0][0], pairs[0][1], pairs[1][0], pairs[1][1], bias=bias, row_div=div)
    ref, mag = gemm_ref(pairs, bias, div)
    assert_within(out, ref, mag, c_tf32(296), False, "one-pass tf32")


# ============================================= weight gradient =====================================================
# Bounds relative to mag = |g|^T |x|, m rows summed (split-K partials, then a fixed-order reduction: every add is one
# fp32 rounding, at most m + 1 of them on any path):
# - bf16: exact products: c = (m + 1) * U23
# - fp32, six bf16 products: three bf16 terms carry every bit of an fp32 value; the omitted cross products are below
#   2^-24 of |g x|: c = 2^-22 + (6m + 1) * U23
# - fp32 one-pass, three products of two bf16 terms: each value is carried to 2^-16, the product to 3 * 2^-16:
#   c = 2^-14 + (3m + 1) * U23
WG_MODES = {"bf16": (torch.bfloat16, "3xtf32", lambda m: (m + 1) * U23),
            "f32-six-products": (torch.float32, "3xtf32", lambda m: 2.0 ** -22 + (6 * m + 1) * U23),
            "f32-one-pass-three-products": (torch.float32, "tf32", lambda m: 2.0 ** -14 + (3 * m + 1) * U23)}


@pytest.mark.parametrize("mode", list(WG_MODES))
@pytest.mark.parametrize("n,k", [(8, 41), (41, 602), (172, 256), (256, 300), (300, 172), (602, 8)],
                         ids=lambda v: str(v))
@pytest.mark.parametrize("m", [1, 63, 64, 65, 2 ** 17 + 3])
def test_wgrad(m, n, k, mode):
    """ops.wgrad (pg_wgrad, tiled in Python over 256-wide n / k blocks) against fp64 g^T x.  NaN in the pad columns
    of g and x must not reach the output; two calls give the same bits.  At m = 2^17 + 3 the data are integers in
    [-2, 2] and the result must be exact."""
    from pipegcn_b200 import ops
    dtype, fp32_gemm, cfun = WG_MODES[mode]
    gen = torch.Generator().manual_seed(m + n * 7 + k)
    exact = m > 4096
    mk = (lambda r, c: _ints((r, c), -2, 2, gen).float()) if exact else (lambda r, c: _normal((r, c), gen))
    g = padded(m, n, dtype, data=mk(m, n))
    x = padded(m, k, dtype, data=mk(m, k))
    with knobs(fp32_gemm=fp32_gemm):
        out = ops.wgrad(g, x)
        again = ops.wgrad(g, x)
    assert out.shape == (n, k)
    assert torch.equal(_bits(out), _bits(again))
    ref = g.double().t() @ x.double()
    if exact:
        assert torch.equal(out.double(), ref)
    else:
        assert_within(out, ref, g.double().abs().t() @ x.double().abs(), cfun(m), False, mode)


# =============================================== aggregate =========================================================
def structured_csr(seg_len, n_ref, seed, n_small=3000):
    """A CSR with every row structure the kernels special-case, column ids in [1, n_ref):
    empty rows; rows of exactly 32 entries; rows of 1, 2, 4, 8 and 16 entries (their chunks fill to exactly 32);
    ragged short rows; rows of 33..200 (one row per chunk, or long when seg_len = 32); rows of seg_len (not long),
    seg_len + 1 (two segments), 3 seg_len, 4 seg_len + 17 and 5 seg_len (hubs of at least 4 segments), spread over
    the row range; repeated column ids inside rows."""
    rng = np.random.default_rng(seed)
    lens = [0] * 300 + [32] * 64
    for length in (1, 2, 4, 8, 16):
        lens += [length] * (32 // length * 40)
    lens += list(rng.integers(1, 13, n_small))
    lens += list(rng.integers(33, 201, 100))
    lens = list(rng.permutation(np.array(lens)))
    longs = [seg_len, seg_len + 1, 3 * seg_len, 4 * seg_len + 17, 5 * seg_len]
    for i, length in enumerate(longs):                       # spread: some below, some above any acc_rows cut
        lens.insert((2 * i + 1) * len(lens) // (2 * len(longs)), length)
    lens = np.array(lens, dtype=np.int64)
    indptr = np.zeros(len(lens) + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(lens)
    indices = rng.integers(1, n_ref, int(indptr[-1]))
    rows32 = np.nonzero(lens == 32)[0]
    indices[indptr[rows32[0]]:indptr[rows32[0] + 1]] = 5                  # one row: 32 times the same id
    r10 = np.nonzero(lens >= 10)[0][0]
    indices[indptr[r10]:indptr[r10] + 5] = 7                              # a repeated id among others
    h = np.nonzero(lens == 4 * seg_len + 17)[0][0]
    indices[indptr[h]:indptr[h] + 3 * seg_len:3] = 9                      # repeats across a hub's segments
    return (torch.from_numpy(indptr).to(torch.int32).to(DEV), torch.from_numpy(indices).to(torch.int32).to(DEV))


@functools.lru_cache(None)
def _graph(seg_len, n_ref=6000):
    from pipegcn_b200.graph import CsrPlan
    indptr, indices = structured_csr(seg_len, n_ref, seed=seg_len)
    plan = CsrPlan(indptr, indices, seg_len=seg_len)
    assert plan.n_long >= 4 and plan.n_chunks_long > 0 and plan.n_chunks > plan.n_chunks_long
    return indptr, indices, plan


def agg_ref(indptr, indices, x, div=None):
    """fp64 (sum, sum of |.|, row lengths) of the CSR rows over the real columns of x."""
    n_rows = indptr.numel() - 1
    lens = (indptr[1:] - indptr[:-1]).long()
    rows = torch.repeat_interleave(torch.arange(n_rows, device=DEV), lens)
    xs = x.double()[indices.long()]
    ref = torch.zeros(n_rows, x.shape[1], dtype=torch.float64, device=DEV).index_add_(0, rows, xs)
    mag = torch.zeros_like(ref).index_add_(0, rows, xs.abs())
    if div is not None:
        ref, mag = ref / div.double()[:, None], mag / div.double()[:, None]
    return ref, mag, lens


def agg_bound_c(lens):
    """Per row: every kernel sums a row's entries one fp32 add each (segments, lane-group partials and the fix-up
    regroup them but add no more than len + 10 roundings along any path), then a reciprocal, a multiply and the
    accumulate add: c = (len + 13) * U24 of mag (+ |out|)."""
    return ((lens.double() + 13) * U24)[:, None]


def x_with_nans(n_cols, n_ref, d, dtype, gen, ints=False):
    """Source rows [1, n_ref) hold data; row 0, rows >= n_ref (never referenced) and every pad column hold NaN."""
    x = padded(n_cols, d, dtype)
    data = _ints((n_ref - 1, d), -3, 3, gen).float() if ints else _normal((n_ref - 1, d), gen)
    x[1:n_ref] = data.to(dtype)
    return x


def run_agg(plan, x, out, div=None, acc_rows=0, drop=None):
    from pipegcn_b200 import ops
    return ops.aggregate(plan, x, out=out, row_div=div, acc_rows=acc_rows, drop=drop)


def _vecs(d, dtype):
    return (d + 16 // (4 if dtype == torch.float32 else 2) - 1) // (16 // (4 if dtype == torch.float32 else 2))


def agg_branch(impl, narrow, dtype, d, pack_short=False, nnz_short=True):
    """The kernel dispatch_agg (csrc/aggregate.cu) picks for 16-byte vectors and a plan with a chunk table."""
    nvec = _vecs(d, dtype)
    if impl >= 2 and nvec > 16:
        vpl = 1 if nvec <= 32 else 2 if nvec <= 64 else 4
        passes = -(-nvec // (32 * vpl))
        long_k = "agg3_long (cp.async ring)" if impl == 3 else "agg2_long"
        return f"agg2_small + {long_k} VPL={vpl}, {passes} column pass(es) + fix-up"
    if impl >= 2 and narrow:
        return f"aggn_small + aggn_long G={4 if nvec <= 4 else 8 if nvec <= 8 else 16} + fix-up"
    if nvec <= 16:
        return f"agg_kernel G={4 if nvec <= 4 else 8 if nvec <= 8 else 16} VPL=1 + fix-up"
    if nvec <= 32 and pack_short and nnz_short:
        return "agg_kernel G=16 VPL=2 (packed short rows) + fix-up"
    return f"agg_kernel G=32 VPL={1 if nvec <= 32 else 2 if nvec <= 64 else 4} + fix-up"


# widths reaching every nvec branch: <= 4, <= 8, <= 16, <= 32, <= 64 vectors, one pass of 4 vectors per lane, two passes
AGG_WIDTHS = [(torch.float32, d) for d in (13, 16, 29, 41, 64, 100, 256, 500, 602, 1024)] + \
             [(torch.bfloat16, d) for d in (32, 41, 100, 256, 500, 1024, 1032)]
AGG_IMPLS = [(1, 0), (2, 0), (2, 1), (3, 0), (3, 1)]


def _agg_cases():
    out = []
    for impl, narrow in AGG_IMPLS:
        for dtype, d in AGG_WIDTHS:
            br = agg_branch(impl, narrow, dtype, d)
            if impl >= 2 and _vecs(d, dtype) > 16 and narrow:
                continue                                     # agg_narrow only matters for rows of <= 16 vectors
            out.append(pytest.param(impl, narrow, dtype, d,
                                    id=f"impl{impl}-narrow{narrow}-{str(dtype)[6:]}-d{d}: {br}"))
    return out


def _drop_check(plan, x, div, acc_rows, init, dtype, spec, step, what):
    """Fused dropout == pg_dropout_rows(pg_aggregate(...)): fp32 bit for bit; bf16 within one bf16 ulp (bit for bit
    at p = 0.5, where scaling by 2 is exact); the mask equals the host port."""
    from pipegcn_b200 import ops
    n_rows, d = init.shape
    fused = Guarded(n_rows, d, dtype)
    fused.t.copy_(init)
    run_agg(plan, x, fused.t, div, acc_rows, drop=spec)
    fused.check()
    clean = Guarded(n_rows, d, dtype)
    clean.t.copy_(init)
    run_agg(plan, x, clean.t, div, acc_rows)
    sep = ops.dropout_rows(clean.t, spec)
    if dtype == torch.float32 or spec.p == 0.5:
        assert torch.equal(_bits(fused.t), _bits(sep)), what
    else:
        # both are a bf16 rounding of v * scale: the fused one of the fp32 value, the separate one of its bf16
        # rounding; they are equal or adjacent bf16 values (one ulp <= 2^-7 of the magnitude)
        err = (fused.t.double() - sep.double()).abs()
        assert bool((err <= 2.0 ** -7 * sep.double().abs()).all()), what
    keep = torch.from_numpy(ops.dropout_keep_host(spec, step, 0, n_rows, d, x.element_size())).to(DEV)
    nz = clean.t != 0
    assert torch.equal((fused.t != 0) & nz, keep & nz), what


@pytest.mark.parametrize("impl,narrow,dtype,d", _agg_cases())
def test_aggregate_dispatch(impl, narrow, dtype, d):
    """Every dispatch branch of pg_aggregate (the case id names it) on a graph with every row structure
    (structured_csr, seg_len 256: short-row chunks, single-row chunks, long rows through the fix-up), with:
    acc_rows in {0, part, all} x row_div {absent, present} (out rows >= acc_rows start as NaN and must be overwritten),
    no write outside the allowed region, NaN in pad columns and unreferenced rows changing nothing, a NaN source row
    reaching exactly the rows that reference it, the fused dropout, two launches and agg_overlap 0 / 1 giving the
    same bits.  With agg_impl >= 2 the plan has a chunk table and both long chunks and short chunks, so the short-row
    kernel runs on the side stream under agg_overlap = 1 (n_chunks_long > 0) and on the caller's stream under 0."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(256)
    assert plan.chunks is not None and plan.n_long > 0
    n_rows, n_ref = plan.n_rows, 6000
    gen = torch.Generator().manual_seed(d * 10 + impl)
    x = x_with_nans(n_ref + 300, n_ref, d, dtype, gen)
    div = _ints((n_rows,), 1, 9, gen).float()
    base = _normal((n_rows, d), gen).to(dtype)
    sums, mag0, lens = agg_ref(indptr, indices, x)
    bf16 = dtype == torch.bfloat16
    results = {}
    for overlap in (1, 0):
        with knobs(agg_impl=impl, agg_narrow=narrow, agg_overlap=overlap):
            for acc_rows in (0, n_rows // 3, n_rows):
                for with_div in (False, True):
                    dv = div if with_div else None
                    out = Guarded(n_rows, d, dtype)
                    out.t[:acc_rows] = base[:acc_rows]
                    run_agg(plan, x, out.t, dv, acc_rows)
                    out.check()
                    ref, mag = sums.clone(), mag0.clone()
                    if with_div:
                        ref, mag = ref / div.double()[:, None], mag / div.double()[:, None]
                    ref[:acc_rows] += base[:acc_rows].double()
                    mag[:acc_rows] += base[:acc_rows].double().abs()
                    assert_within(out.t, ref, mag, agg_bound_c(lens), bf16,
                                  f"acc_rows={acc_rows} div={with_div} overlap={overlap}")
                    results[(overlap, acc_rows, with_div)] = out.t.clone()
            again = Guarded(n_rows, d, dtype)
            run_agg(plan, x, again.t, div)
            assert torch.equal(_bits(again.t), _bits(results[(overlap, 0, True)])), "two launches differ"
            if overlap == 1:
                step = torch.tensor([3], dtype=torch.int32, device=DEV)
                for p in ((0.3, 0.5) if bf16 else (0.3,)):
                    spec = ops.DropSpec(p, 0xABCDEF0123, step, 1)
                    init = Guarded(n_rows, d, dtype).t
                    init[:n_rows // 3] = base[:n_rows // 3]
                    _drop_check(plan, x, div, n_rows // 3, init, dtype, spec, 3, f"dropout p={p}")
                # one NaN source row reaches exactly the rows that reference it
                hot = int(torch.bincount(indices.long()).argmax())
                xn = padded(x.shape[0], d, dtype, data=x)     # same layout (a clone would be contiguous)
                xn[hot, :] = float("nan")
                o = run_agg(plan, xn, Guarded(n_rows, d, dtype).t)
                rows = torch.repeat_interleave(torch.arange(n_rows, device=DEV), lens)
                hit = torch.zeros(n_rows, dtype=torch.bool, device=DEV)
                hit[rows[indices.long() == hot]] = True
                assert torch.equal(o.isnan().all(1), hit) and torch.equal(o.isnan().any(1), hit)
    for key, val in results.items():
        if key[0] == 0:
            assert torch.equal(_bits(val), _bits(results[(1,) + key[1:]])), f"agg_overlap changes the bits at {key}"


@pytest.mark.parametrize("d", [41, 256], ids=["narrow", "wide"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("seg_len", [32, 256, 512])
def test_aggregate_long_rows(seg_len, impl, dtype, d):
    """Rows of seg_len, seg_len + 1 and k * seg_len entries and hubs of >= 4 segments go through the segment kernels
    and the fix-up (agg_fixup_kernel), with the accumulate mode and the fused dropout (the fix-up's store applies the
    mask).  seg_len 32 makes the 33..200-entry rows long as well."""
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(seg_len)
    lens = (indptr[1:] - indptr[:-1]).long()
    assert int((lens > seg_len).sum()) == plan.n_long and plan.n_seg >= plan.n_long + 4 * 2
    n_rows = plan.n_rows
    gen = torch.Generator().manual_seed(seg_len + impl)
    x = x_with_nans(6300, 6000, d, dtype, gen)
    div = _ints((n_rows,), 1, 9, gen).float()
    base = _normal((n_rows, d), gen).to(dtype)
    acc = n_rows // 2
    with knobs(agg_impl=impl):
        out = Guarded(n_rows, d, dtype)
        out.t[:acc] = base[:acc]
        run_agg(plan, x, out.t, div, acc)
        out.check()
        ref, mag, lens = agg_ref(indptr, indices, x, div)
        ref[:acc] += base[:acc].double()
        mag[:acc] += base[:acc].double().abs()
        assert_within(out.t, ref, mag, agg_bound_c(lens), dtype == torch.bfloat16, f"seg_len={seg_len}")
        step = torch.tensor([1], dtype=torch.int32, device=DEV)
        init = Guarded(n_rows, d, dtype).t
        init[:acc] = base[:acc]
        _drop_check(plan, x, div, acc, init, dtype, ops.DropSpec(0.5, 77, step, 0), 1, "fix-up dropout p=0.5")
        _drop_check(plan, x, None, 0, Guarded(n_rows, d, dtype).t, dtype, ops.DropSpec(0.3, 78, step, 0), 1,
                    "fix-up dropout p=0.3")


# (name, options, widths) -- every case is compared bit for bit with the same impl under the default knobs (the knobs
# change cache policies, unrolling, occupancy or lane packing, never the order of the adds) and against fp64
AGG_KNOBS = [
    # bit 31 of a pidx entry marks a hot row: the chunked kernels load it with evict_last (HINT = true instantiations)
    ("l2_hint impl2: agg2_small/agg2_long HINT", dict(agg_impl=2, agg_l2_hint=1), [(torch.float32, 100), (torch.bfloat16, 500)]),
    ("l2_hint impl3: agg3_long HINT", dict(agg_impl=3, agg_l2_hint=1), [(torch.float32, 256), (torch.bfloat16, 1032)]),
    # launch_agg: VPL == 1 (rows of <= 32 vectors) and agg_unroll 4 -> agg_kernel U = 4
    ("unroll4 impl1: agg_kernel U=4", dict(agg_impl=1, agg_unroll=4), [(torch.float32, 16), (torch.float32, 100), (torch.bfloat16, 256)]),
    # launch_agg2h: VPL == 1 (17..32 vectors) and agg_occ 5 -> agg2_long_kernel OCC = 5
    ("occ5 impl2: agg2_long OCC=5", dict(agg_impl=2, agg_occ=5), [(torch.float32, 100), (torch.bfloat16, 256)]),
    # dispatch_agg under impl 1: 17..32 vectors, nnz < 12 n_rows -> agg_kernel G=16 VPL=2
    ("pack_short impl1: agg_kernel G=16 VPL=2", dict(agg_impl=1, agg_pack_short=1), [(torch.float32, 100), (torch.bfloat16, 256)]),
]


@pytest.mark.parametrize("name,opts,dtype,d", [pytest.param(nm, o, dt, d, id=f"{nm}-{str(dt)[6:]}-d{d}")
                                                for nm, o, ws in AGG_KNOBS for dt, d in ws])
def test_aggregate_knobs(name, opts, dtype, d):
    from pipegcn_b200 import ops
    indptr, indices, plan = _graph(256)
    nvec = _vecs(d, dtype)
    if "l2_hint" in name:
        assert plan.n_hot > 0 and bool((plan.pidx < 0).any()) and nvec > 16
    if "unroll4" in name or "occ5" in name:
        assert nvec <= 32
    if "occ5" in name:
        assert 16 < nvec and plan.n_chunks_long > 0
    if "pack_short" in name:
        assert 16 < nvec <= 32 and plan.nnz < 12 * plan.n_rows
    n_rows = plan.n_rows
    gen = torch.Generator().manual_seed(d)
    x = x_with_nans(6300, 6000, d, dtype, gen)
    div = _ints((n_rows,), 1, 9, gen).float()
    base = _normal((n_rows, d), gen).to(dtype)
    acc = n_rows // 3
    outs = []
    for o in ({"agg_impl": opts["agg_impl"]}, opts):
        with knobs(**o):
            out = Guarded(n_rows, d, dtype)
            out.t[:acc] = base[:acc]
            run_agg(plan, x, out.t, div, acc)
            out.check()
            outs.append(out.t)
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), name
    ref, mag, lens = agg_ref(indptr, indices, x, div)
    ref[:acc] += base[:acc].double()
    mag[:acc] += base[:acc].double().abs()
    assert_within(outs[1], ref, mag, agg_bound_c(lens), dtype == torch.bfloat16, name)
    with knobs(**opts):
        step = torch.tensor([2], dtype=torch.int32, device=DEV)
        init = Guarded(n_rows, d, dtype).t
        init[:acc] = base[:acc]
        _drop_check(plan, x, div, acc, init, dtype, ops.DropSpec(0.3, 99, step, 0), 2, name)


@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("dtype,d,vb", [(torch.float32, 38, 8), (torch.float32, 37, 4), (torch.bfloat16, 36, 8),
                                        (torch.bfloat16, 34, 4)], ids=lambda v: str(v))
def test_aggregate_small_vectors(dtype, d, vb, impl):
    """Contiguous, unpadded rows whose byte stride is not a multiple of 16 run the 8- and 4-byte vector
    instantiations (vec_bytes); the output rows have no padding, so the allowed region is exactly [0, d)."""
    indptr, indices, plan = _graph(256)
    es = 4 if dtype == torch.float32 else 2
    assert (d * es) % 16 != 0 and (d * es) % vb == 0 and (d * es) % (2 * vb) != 0
    n_rows = plan.n_rows
    gen = torch.Generator().manual_seed(d + impl)
    xbase = torch.full((6301, d), float("nan"), dtype=dtype, device=DEV)    # contiguous: stride d
    x = xbase[1:]
    x[1:6000] = _normal((5999, d), gen).to(dtype)
    div = _ints((n_rows,), 1, 9, gen).float()
    base = _normal((n_rows, d), gen).to(dtype)
    acc = n_rows // 3
    with knobs(agg_impl=impl):
        out = Guarded(n_rows, d, dtype, ld=d)
        out.t[:acc] = base[:acc]
        run_agg(plan, x, out.t, div, acc)
        out.check(exact=True)
    ref, mag, lens = agg_ref(indptr, indices, x, div)
    ref[:acc] += base[:acc].double()
    mag[:acc] += base[:acc].double().abs()
    assert_within(out.t, ref, mag, agg_bound_c(lens), dtype == torch.bfloat16, f"{vb}-byte vectors")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_row_div(dtype):
    """pg_row_div: one reciprocal and one multiply per element (<= 2 roundings), NaN pads not spreading."""
    from pipegcn_b200 import ops
    gen = torch.Generator().manual_seed(1)
    n, d = 100003, 41
    x = padded(n, d, dtype, data=_normal((n, d), gen))
    div = _ints((n,), 1, 9, gen).float()
    out = Guarded(n, d, dtype)
    ops.row_div(x, div, out=out.t)
    out.check()
    ref = x.double() / div.double()[:, None]
    assert_within(out.t, ref, ref.abs(), 2 * U24, dtype == torch.bfloat16, "row_div")


# ============================================== row kernels ========================================================
@pytest.mark.parametrize("subwarp", [1, 0], ids=["ce_subwarp1", "ce_subwarp0-one-warp-per-row"])
@pytest.mark.parametrize("c", [41, 47, 172, 1000])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cross_entropy_at_scale(dtype, c, subwarp):
    """pg_ce_fwd / pg_ce_bwd on 300k rows (the grid-stride loops and per-CTA column partials iterate many times: the
    grid is capped at 8 CTAs per SM), pad columns holding +inf and then NaN (same bits), against fp64: lse, loss,
    gradient, column sums.  c = 1000 in fp32 has 250 vectors per row: one warp per row even with ce_subwarp."""
    from pipegcn_b200 import _C
    n_total, n_train = 300_000, 300_000 - 12_345
    gen = torch.Generator().manual_seed(c)
    zsrc = (_normal((n_total, c), gen) * 3).to(dtype)
    labels = _ints((n_train,), 0, c - 1, gen).long()
    up = torch.tensor([0.5], device=DEV)
    code, st = _C.dtype_code(dtype), _C.stream_ptr()
    grid = int(_C.lib.pg_row_grid(n_total))
    assert grid == min(-(-n_total // 8), 8 * sm_count()) and n_total > 8 * grid     # more than one resident wave
    res = []
    with knobs(ce_subwarp=subwarp):
        for fill in (float("inf"), float("nan")):
            z = padded(n_total, c, dtype, fill=fill, data=zsrc)
            lse = torch.empty(n_train, device=DEV)
            partial = torch.empty(grid * c, device=DEV)
            loss = torch.zeros(1, device=DEV)
            _C.check(_C.lib.pg_ce_fwd(z.data_ptr(), z.stride(0), labels.data_ptr(), n_train, c, code, lse.data_ptr(),
                                      partial.data_ptr(), loss.data_ptr(), st), "pg_ce_fwd")
            g = Guarded(n_total, c, dtype)
            colsum = torch.empty(c, device=DEV)
            _C.check(_C.lib.pg_ce_bwd(z.data_ptr(), z.stride(0), labels.data_ptr(), lse.data_ptr(), up.data_ptr(),
                                      n_train, n_total, c, code, g.t.data_ptr(), g.t.stride(0), colsum.data_ptr(),
                                      partial.data_ptr(), st), "pg_ce_bwd")
            g.check()
            res.append((lse, loss, g.t, colsum))
    for a, b in zip(res[0][:3], res[1][:3]):
        assert torch.equal(_bits(a), _bits(b)), "the pad fill changes the result"
    # the one-warp-per-row kernel (ce_subwarp 0, or rows of more than 128 vectors) sums the columns with
    # shared-memory atomics, whose order is not fixed; the sub-warp kernel's column sums are
    if subwarp and -(-c // (16 // zsrc.element_size())) <= 128:
        assert torch.equal(res[0][3], res[1][3])
    del res[0]
    lse, loss, g, colsum = res[0]
    zd = zsrc.double()
    lse_ref = torch.logsumexp(zd[:n_train], 1)
    zl = zd[torch.arange(n_train, device=DEV), labels]
    # per row: the max is exact, the sum of c exponentials (expf within 2 ulp) carries (c + 4) roundings, logf 2 ulp,
    # the add one: |lse - ref| <= (c + 8) * 2^-24 + 2^-23 |lse|
    e_row = (c + 8) * U24 + 2.0 ** -23 * lse_ref.abs()
    assert bool(((lse.double() - lse_ref).abs() <= e_row).all())
    # the loss: per-row errors plus the fixed-order reduction (rows of a warp, 8 warps, then the CTA partials)
    t = lse_ref - zl
    chain = -(-n_total // (8 * grid)) + 8 + grid + 8
    assert abs(loss.item() - t.sum().item()) <= float((e_row + 2.0 ** -23 * zl.abs()).sum()) + chain * U24 * float(t.abs().sum())
    # gradient: an lse error e moves p by the factor exp(e); the exp (2 ulp), the subtraction and the scale round
    p = torch.softmax(zd[:n_train], 1)
    g_ref = p.clone()
    g_ref[torch.arange(n_train, device=DEV), labels] -= 1
    g_ref *= 0.5
    bound = 0.5 * (p * (e_row[:, None] + 4 * U24) + 2 * U24)
    if dtype == torch.bfloat16:
        bound = bound + BF16_U * (g_ref.abs() + bound)
    assert bool(((g[:n_train].double() - g_ref).abs() <= bound).all())
    assert torch.count_nonzero(g[n_train:]) == 0
    # column sums of the stored gradient: rows of a lane / warp / CTA, then the CTA partials in a fixed order
    gs = g.double()
    chain = -(-n_total // grid) + grid + 16
    assert bool(((colsum.double() - gs.sum(0)).abs() <= chain * U24 * gs.abs().sum(0)).all())


@pytest.mark.parametrize("stage", [0, 2])
@pytest.mark.parametrize("d", [100, 36])
def test_layer_norm_nan_pads(d, stage):
    """pg_ln_relu_fwd / _bwd2 in fp32 with d % 8 != 0 (4 pad columns): NaN in the pad columns of y and of the
    incoming gradient changes no bit of any result."""
    from pipegcn_b200 import _C
    n = 3001
    gen = torch.Generator().manual_seed(d)
    ydata, gdata = _normal((n, d), gen) * 2 + 0.3, _normal((n, d), gen)
    gamma, beta = _normal((d,), gen).abs() + 0.5, _normal((d,), gen)
    code, st = _C.dtype_code(torch.float32), _C.stream_ptr()
    res = []
    with knobs(ln_stage=stage):
        for fill in (0.0, float("nan")):
            y, gout = padded(n, d, torch.float32, fill, ydata), padded(n, d, torch.float32, fill, gdata)
            out = Guarded(n, d, torch.float32)
            mean, rstd = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
            _C.check(_C.lib.pg_ln_relu_fwd(y.data_ptr(), y.stride(0), gamma.data_ptr(), beta.data_ptr(), 1e-5, 1,
                                           out.t.data_ptr(), out.t.stride(0), mean.data_ptr(), rstd.data_ptr(), n, d,
                                           code, st), "pg_ln_relu_fwd")
            out.check()
            g_y = Guarded(n, d, torch.float32)
            red = torch.empty(3, d, device=DEV)
            partial = torch.empty(_C.lib.pg_row_grid(n) * 3 * d, device=DEV)
            _C.check(_C.lib.pg_ln_relu_bwd2(gout.data_ptr(), gout.stride(0), None, 0, y.data_ptr(), y.stride(0),
                                            mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1,
                                            g_y.t.data_ptr(), g_y.t.stride(0), red[0].data_ptr(), red[1].data_ptr(),
                                            red[2].data_ptr(), partial.data_ptr(), n, d, code, st), "pg_ln_relu_bwd2")
            g_y.check()
            res.append([out.t, mean, rstd, g_y.t, red])
    for a, b in zip(*res):
        assert torch.equal(_bits(a), _bits(b))
    assert bool(torch.isfinite(res[1][3]).all() and torch.isfinite(res[1][4]).all())


@pytest.mark.parametrize("row0", [2 ** 31 - 3, 2 ** 32 - 5, 3 * 2 ** 32 + 7], ids=["2^31-3", "2^32-5", "3*2^32+7"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dropout_rows_far_rows(dtype, row0):
    """pg_dropout_rows with row0 past 2^31 and 2^32: the element index (row0 + r) * nvec + vector is 64-bit;
    the kernel's mask equals the host port, kept values are x * (1 / (1 - p)) rounded once."""
    from pipegcn_b200 import ops
    n, d, p = 64, 100, 0.3
    gen = torch.Generator().manual_seed(5)
    x = padded(n, d, dtype, data=torch.rand(n, d, generator=gen).to(DEV) + 0.5)
    step = torch.tensor([6], dtype=torch.int32, device=DEV)
    spec = ops.DropSpec(p, 0xFEEDFACECAFEBEEF, step, 3)
    out = Guarded(n, d, dtype)
    ops.dropout_rows(x, spec, out=out.t, row0=row0)
    out.check()
    keep = torch.from_numpy(ops.dropout_keep_host(spec, 6, row0, n, d, x.element_size())).to(DEV)
    scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    want = torch.where(keep, (x.float() * scale).to(dtype), torch.zeros((), dtype=dtype, device=DEV))
    assert torch.equal(_bits(out.t), _bits(want))


# ========================================== addresses past 2 GiB ===================================================
def _need(gib):
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")


@pytest.mark.parametrize("dtype,n_src", [(torch.float32, 2_300_000), (torch.bfloat16, 4_500_000)])
def test_aggregate_past_2gib(dtype, n_src):
    """A source tensor larger than 2^31 bytes, most referenced rows and all hub sources in its top rows (byte offsets
    past 2^31): default knobs, agg_impl 1 and agg_impl 3.  Integer data: exact sums, so every row must equal fp64."""
    d = 256
    _need(n_src * d * (4 if dtype == torch.float32 else 2) / 2 ** 30 + 2)
    rng = np.random.default_rng(1)
    n_rows = 30000
    lens = rng.integers(1, 17, n_rows)
    lens[[10, 9000, 20000, 29990]] = 3000                      # hubs: several segments each
    indptr = np.zeros(n_rows + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(lens)
    nnz = int(indptr[-1])
    top = n_src - 200_000
    idx = np.where(rng.random(nnz) < 0.8, rng.integers(top, n_src, nnz), rng.integers(0, n_src, nnz))
    for h in (10, 9000, 20000, 29990):
        idx[indptr[h]:indptr[h + 1]] = rng.integers(n_src - 50_000, n_src, 3000)
    x = None
    try:
        from pipegcn_b200.graph import CsrPlan
        ip, ix = torch.from_numpy(indptr).to(torch.int32).to(DEV), torch.from_numpy(idx).to(torch.int32).to(DEV)
        plan = CsrPlan(ip, ix, seg_len=512)
        assert plan.n_long == 4
        x = torch.empty(n_src, d, dtype=dtype, device=DEV)
        assert x.numel() * x.element_size() > 2 ** 31
        gen = torch.Generator(device=DEV).manual_seed(2)
        for i in range(0, n_src, 1 << 19):
            blk = x[i:i + (1 << 19)]
            blk.copy_(torch.randint(-2, 3, blk.shape, generator=gen, device=DEV, dtype=torch.int8))
        rows = torch.repeat_interleave(torch.arange(n_rows, device=DEV), (ip[1:] - ip[:-1]).long())
        ref = torch.zeros(n_rows, d, dtype=torch.float64, device=DEV)
        for e in range(0, nnz, 1 << 17):
            ref.index_add_(0, rows[e:e + (1 << 17)], x[ix[e:e + (1 << 17)].long()].double())
        for opts in ({}, {"agg_impl": 1}, {"agg_impl": 3}):
            with knobs(**opts):
                out = Guarded(n_rows, d, dtype)
                run_agg(plan, x, out.t)
                out.check()
            sample = torch.tensor([10, 9000, 20000, 29990, 0, n_rows - 1], device=DEV)
            # the fp32 sums are exact integers: the output is their one rounding to the dtype
            want = ref.to(dtype)
            assert torch.equal(out.t[sample], want[sample]), f"hub rows, {opts}"
            assert torch.equal(out.t, want), f"all rows, {opts}"
    finally:
        del x
        torch.cuda.empty_cache()


def test_gemm_and_wgrad_past_2gib():
    """gemm_nt and wgrad whose big operand A [4.5M, 256] bf16 spans more than 2^31 bytes (4.5M rows: about 266 tiles
    per CTA of the persistent GEMM).  Integer data: A, B in [-2, 2], g in [-1, 1]; every partial sum is an integer
    below 2^24, so both results must equal fp64 exactly (checked in row blocks)."""
    from pipegcn_b200 import ops
    _need(10)
    m, k, n = 4_500_000, 256, 64
    a = g = out = None
    try:
        gen = torch.Generator(device=DEV).manual_seed(3)
        a = torch.empty(m, k, dtype=torch.bfloat16, device=DEV)
        g = torch.empty(m, n, dtype=torch.bfloat16, device=DEV)
        assert a.numel() * 2 > 2 ** 31
        for i in range(0, m, 1 << 19):
            a[i:i + (1 << 19)].copy_(torch.randint(-2, 3, a[i:i + (1 << 19)].shape, generator=gen, device=DEV,
                                                   dtype=torch.int8))
            g[i:i + (1 << 19)].copy_(torch.randint(-1, 2, g[i:i + (1 << 19)].shape, generator=gen, device=DEV,
                                                   dtype=torch.int8))
        b = torch.randint(-2, 3, (n, k), generator=gen, device=DEV, dtype=torch.int8).to(torch.bfloat16)
        out = ops.gemm_nt(a, b, out_dtype=torch.float32)
        bd = b.double()
        for i in range(0, m, 1 << 19):
            assert torch.equal(out[i:i + (1 << 19)].double(), a[i:i + (1 << 19)].double() @ bd.t()), f"rows {i}.."
        del out
        out = None
        w = ops.wgrad(g, a)
        ref = torch.zeros(n, k, dtype=torch.float64, device=DEV)
        for i in range(0, m, 1 << 19):
            ref += g[i:i + (1 << 19)].double().t() @ a[i:i + (1 << 19)].double()
        assert torch.equal(w.double(), ref)
    finally:
        del a, g, out
        torch.cuda.empty_cache()
