"""Conformance of the halo exchange kernels (csrc/exchange.cu) with exact host restatements, through the C ABI:
pg_halo_push / pg_halo_push_drop, pg_halo_wait, pg_boundary_add, pg_scale_rows and pg_bns_mask_rows, at eight
partitions (seven peers per launch), past the first wave of CTAs and on every vector width the entry points pick.

Conventions:
- These kernels copy values or apply fp32 operations in a fixed order, so every check is bit for bit.  fp32 arithmetic
  is restated in CPU float32 tensors (one rounding per operation, no contraction); bf16 rounding is
  `tensor.to(torch.bfloat16)` (round to nearest even).  The one exception: fp32 arithmetic on a NaN gives the device's
  canonical NaN, not the host's, so an element whose reference is computed from a NaN must merely be a NaN.
- Source pad columns and unreferenced source rows hold NaN.  Every destination (message rows, EMA mirror, gradient,
  output) is a `Guarded` view whose guard rows and columns hold SENTINEL; the whole allocation is compared with its
  expected image, so the guards must survive bit for bit.
- VB (bytes) is the vector width an entry point picks: the widest that the base address and the row stride of every
  operand allow (vec_bytes / common_vec).  An operand is built for a given VB through its stride (`ld_for`) or its
  base.  The kernels write columns [0, round_up(d, VB / elem)) of a row (include/pipegcn_b200.h), so the tail of the
  last vector is written too and the case ids name VB.
- No test waits on a flag that is behind the awaited value, and none takes the timeout path.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_kernel_conformance_gpu import DEV, Guarded, _bits, padded, sm_count

pytestmark = pytest.mark.gpu

NAN = float("nan")
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
WIDTHS = [1, 3, 4, 5, 8, 9, 63, 64, 65, 100, 256, 257, 602]
VBS = {"fp32": (16, 8, 4), "bf16": (16, 8, 4, 2)}
WIDTH_CASES = [(dt, d, vb) for dt in DTYPES for d in WIDTHS for vb in VBS[dt]]
WIDTH_IDS = [f"{dt}-d{d}-VB{vb}" for dt, d, vb in WIDTH_CASES]
U32 = 0xFFFFFFFF


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def _rup(x, m):
    return (x + m - 1) // m * m


def ld_for(cols, vb, es):
    """The smallest row stride (elements) >= cols whose byte size allows vb-byte vectors and, below 16, no wider ones."""
    v = vb // es
    ld = _rup(cols, v)
    if vb < 16 and (ld * es) % (2 * vb) == 0:
        ld += v
    return ld


def picked_vb(d, es, operands):
    """vec_bytes + common_vec of the entry points for operands [(data_ptr, ld)]: the VB a case must run at."""
    vb = 16
    for p, ld in operands:
        while vb > es and (p % vb or (ld * es) % vb):
            vb //= 2
    while vb > es:
        v = vb // es
        if d % v == 0 or all(_rup(d, v) <= ld for _, ld in operands):
            break
        vb //= 2
    return vb


def source(n, d, dtype, vb, gen, scale=4.0):
    """[n, d] normal rows in storage whose stride allows exactly vb-byte vectors; pad columns hold NaN."""
    base = torch.full((max(n, 1), ld_for(d, vb, _es(dtype))), NAN, dtype=dtype, device=DEV)
    base[:n, :d] = (torch.randn(n, d, generator=gen) * scale).to(dtype).to(DEV)
    return base[:n, :d]


def guarded(n, d, dtype, vb):
    """A Guarded output [n, d] whose base and stride allow exactly vb-byte vectors, with one vector of guard columns
    on the left and at least one on the right of columns [0, round_up(d, V))."""
    v = vb // _es(dtype)
    return Guarded(n, d, dtype, col0=v, ld=ld_for(v + _rup(d, v) + v, vb, _es(dtype)))


def _nan_bits(b, dtype):
    if dtype == torch.float32:
        return (b & 0x7FFFFFFF) > 0x7F800000
    return (b.to(torch.int32) & 0x7FFF) > 0x7F80


def check_image(base, want, nan_at=None, what=""):
    """The whole allocation `base` (device) against its expected bits `want` (CPU); `nan_at`: elements that must hold
    some NaN instead (computed on the device from a NaN)."""
    got = _bits(base).cpu()
    bad = got != want
    if nan_at is not None:
        bad = torch.where(nan_at, ~_nan_bits(got, base.dtype), bad)
    if bool(bad.any()):
        r, c = bad.nonzero()[0].tolist()
        mask = 0xFFFFFFFF if base.dtype == torch.float32 else 0xFFFF
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at allocation [{r}, {c}]: got "
                             f"{int(got[r, c]) & mask:#x}, want {int(want[r, c]) & mask:#x}"
                             f"{' (any NaN)' if nan_at is not None and bool(nan_at[r, c]) else ''}")


def image(g):
    """The bits of a Guarded allocation as it stands now (CPU): the expected image before a kernel writes into it."""
    return _bits(g.base).cpu().clone()


def _fresh(img):
    """A copy of an image to fill in, and an all-False nan_at mask."""
    return img.clone(), torch.zeros(img.shape, dtype=torch.bool)


def _u32(t):
    return [int(x) & U32 for x in t.cpu().tolist()]


def _stored(x, cols):
    """The first `cols` stored columns of every row of the strided view x (its pad columns past d included)."""
    return x.as_strided((x.shape[0], cols), (x.stride(0), 1))


def _i32(values):
    """uint32 values as the int32 tensor holding their bits."""
    return torch.tensor([(int(v) & U32) - (1 << 32) if int(v) & U32 >= 1 << 31 else int(v) & U32 for v in values],
                        dtype=torch.int32, device=DEV)


def _ptr(t, row=0):
    return t.data_ptr() + row * t.stride(0) * t.element_size()


# ============================================ pg_halo_push ============================================================
class Push:
    """One launch's worth of messages (built with _MsgSet, which fills cta_begin as Buffer does) reading `src`.

    spec: [(kind, n_rows)], kind "idx" (gathered through idx: repeated ids, a descending run, the last source row)
    or "row0" (contiguous from src_row0).  Message m writes into rows [off[m], off[m] + n_rows) of one Guarded
    destination, two untouched rows apart; with `ema` its fp32 mirror rows sit in a Guarded mirror the same way."""
    GAP = 2

    def __init__(self, spec, d, dtype, vb, gen, ema=False, n_src=None, row0s=None):
        from pipegcn_b200 import _C
        from pipegcn_b200.helper.feature_buffer import _MsgSet
        self.d, self.dtype, self.es = d, dtype, _es(dtype)
        n_max = max([n for _, n in spec] + [1])
        n_src = n_src or max(2 * n_max, 600)
        self.src = source(n_src, d, dtype, vb, gen)
        assert picked_vb(d, self.es, [(self.src.data_ptr(), self.src.stride(0))]) == vb
        self.vb, self.v = vb, vb // self.es
        self.end = _rup(d, self.v)                     # columns [0, end) of a row are written
        self.rows, self.off = [], []
        o = 0
        for m, (kind, n) in enumerate(spec):
            if kind == "idx":
                ids = torch.randint(0, n_src, (n,), generator=gen)
                if n > 0:
                    ids[0] = n_src - 1                                  # the last source row
                if n > 2:
                    ids[2] = ids[1]                                     # a repeated id
                if n >= 20:
                    ids[n // 2:n // 2 + 9] = torch.arange(n_src - 20, n_src - 29, -1)    # descending
                self.rows.append(ids)
            else:
                r0 = int(torch.randint(0, n_src - n + 1, (1,), generator=gen))
                self.rows.append(torch.arange(r0, r0 + n))
            self.off.append(o)
            o += n + self.GAP
        used = torch.zeros(n_src, dtype=torch.bool)
        for r in self.rows:
            used[r] = True
        self.src[(~used).nonzero().flatten().to(DEV)] = NAN          # unreferenced rows
        self.n_dst = max(o, 1)
        self.dst = Guarded(self.n_dst, d, dtype, col0=16 // self.es)
        self.mir = None
        if ema:
            self.mir = Guarded(self.n_dst, d, torch.float32, col0=4)
            G = self.mir.G
            self.mir.base[G:G + self.n_dst, 4:4 + self.end] = torch.randn(self.n_dst, self.end, generator=gen).to(DEV)
        self.dst0, self.mir0 = image(self.dst), image(self.mir) if ema else None     # before any launch
        n_msgs = len(spec)
        self.flags = torch.zeros(n_msgs, dtype=torch.int32, device=DEV)
        self.counters = torch.zeros(n_msgs, dtype=torch.int32, device=DEV)
        self.dst_row0 = [row0s[m] if row0s else 1000 * m + 17 for m in range(n_msgs)]
        self.idx = []                                   # kept alive: the descriptors point at them
        msgs = []
        for m, (kind, n) in enumerate(spec):
            idx = self.rows[m].to(torch.int32).to(DEV) if kind == "idx" else None
            self.idx.append(idx)
            msgs.append(_C.pg_msg(idx.data_ptr() if idx is not None and n > 0 else None,
                                  int(self.rows[m][0]) if kind == "row0" and n > 0 else 0, n, 0,
                                  _ptr(self.dst.t, self.off[m]), self.dst.ld,
                                  _ptr(self.mir.t, self.off[m]) if ema else None, self.mir.ld if ema else 0,
                                  self.flags.data_ptr() + 4 * m, self.counters.data_ptr() + 4 * m, self.dst_row0[m]))
        self.ms = _MsgSet(msgs, DEV)
        self.spec = spec

    def launch(self, momentum=0.0, value=1, value_dev=None, drop=None, src=None, ld=None, d=None, n_msgs=None):
        from pipegcn_b200 import _C
        src = self.src if src is None else src
        args = (self.ms.ptr, self.ms.n_msgs if n_msgs is None else n_msgs, self.ms.n_ctas, src.data_ptr(),
                src.stride(0) if ld is None else ld, self.d if d is None else d, _C.dtype_code(self.dtype),
                momentum, float(1.0 - momentum), value, value_dev)
        if drop is not None:
            rc = _C.lib.pg_halo_push_drop(*args, C.byref(drop.c()), _C.stream_ptr())
        else:
            rc = _C.lib.pg_halo_push(*args, _C.stream_ptr())
        _C.check(rc, "pg_halo_push")
        torch.cuda.synchronize()

    def src_rows(self, m):
        """Source rows of message m as stored, columns [0, end) (pad columns included): CPU."""
        return _stored(self.src, self.end)[self.rows[m].to(DEV)].cpu()

    def check_flags(self, value):
        assert _u32(self.flags) == [value & U32] * len(self.spec), "flags"
        assert _u32(self.counters) == [0] * len(self.spec), "counters not reset"


def _dst_block(p, m):
    G, c0, n = p.dst.G, p.dst.col0, p.spec[m][1]
    return slice(G + p.off[m], G + p.off[m] + n), slice(c0, c0 + p.end)


def _mir_block(p, m):
    G, c0, n = p.mir.G, p.mir.col0, p.spec[m][1]
    return slice(G + p.off[m], G + p.off[m] + n), slice(c0, c0 + p.end)


def copy_image(p):
    want, _ = _fresh(p.dst0)
    for m in range(len(p.spec)):
        if p.spec[m][1]:
            want[_dst_block(p, m)] = _bits(p.src_rows(m))
    return want


P8 = [("idx", 33), ("row0", 0), ("idx", 257), ("row0", 1), ("idx", 31), ("row0", 255), ("idx", 32)]


@pytest.mark.parametrize("dt,d,vb", WIDTH_CASES, ids=WIDTH_IDS)
def test_push_copy(dt, d, vb):
    """Seven messages (P = 8, an empty one in the middle) of every row count class: row r of message m is its source
    row bit for bit over columns [0, round_up(d, V)) -- the last vector's tail carries the source's pad columns --, the
    rows past n_rows and the guards are untouched, every flag holds the value and every counter is back to 0."""
    gen = torch.Generator().manual_seed(d * 10 + vb)
    p = Push(P8, d, DTYPES[dt], vb, gen)
    p.launch(value=5)
    check_image(p.dst.base, copy_image(p), what="message rows")
    p.check_flags(5)


def ema_step(e, x, m):
    """The mirror update e <- fl(fl(e * m) + fl(one_minus * x)) in fp32, one_minus = (float)(1 - m) in double."""
    m32 = torch.tensor(np.float32(m))
    om = torch.tensor(np.float32(1.0 - m))
    return e * m32 + om * x


@pytest.mark.parametrize("dt,d,vb", WIDTH_CASES, ids=WIDTH_IDS)
def test_push_ema(dt, d, vb):
    """Three launches with m = 0.5, 0.9, 0.95: the mirror follows e <- fl(fl(e m) + fl((1-m) x)) (no FMA) and the
    message is e rounded to the activation dtype, bit for bit; the tails of the last vector become NaN (pad columns)."""
    dtype = DTYPES[dt]
    gen = torch.Generator().manual_seed(d * 10 + vb + 1)
    p = Push(P8, d, dtype, vb, gen, ema=True)
    e = [p.mir.base[_mir_block(p, m)].cpu().clone() for m in range(len(P8))]
    tail = torch.zeros(p.end, dtype=torch.bool)
    tail[d:] = True
    for step, mom in enumerate((0.5, 0.9, 0.95)):
        p.launch(momentum=mom, value=step + 1)
        want, nan_at = _fresh(p.dst0)
        wmir, mir_nan = _fresh(p.mir0)
        for m, (_, n) in enumerate(P8):
            if n == 0:
                continue
            e[m] = ema_step(e[m], p.src_rows(m).float(), mom)
            wmir[_mir_block(p, m)] = _bits(e[m])
            mir_nan[_mir_block(p, m)] = tail.expand(n, -1)
            want[_dst_block(p, m)] = _bits(e[m].to(dtype))
            nan_at[_dst_block(p, m)] = tail.expand(n, -1)
        check_image(p.mir.base, wmir, mir_nan, f"mirror after launch {step}")
        check_image(p.dst.base, want, nan_at, f"message after launch {step}")
        p.check_flags(step + 1)


def _drop_ref(p, m, v, spec, step):
    """keep ? T(fl(v * scale)) : +0 over columns [0, end) of message m's rows, keep from the host port of the
    receiver's mask at rows dst_row0 + r; v float32 [n, end] (CPU).  Returns the bits and where a NaN is due."""
    from pipegcn_b200 import ops
    keep = torch.from_numpy(ops.dropout_keep_host(spec, step, p.dst_row0[m], v.shape[0], p.end, p.es))
    scale = torch.tensor(np.float32(1.0) / (np.float32(1.0) - np.float32(spec.p)))
    out = torch.where(keep, v * scale, torch.zeros(())).to(p.dtype)
    return _bits(out), keep & v.isnan()


DROP_ROW0 = [3, 0, 3_000_000_017, 40, 1 << 20, 7, 123_456]     # (3e9 + r) * nvec passes 2^32: the key's high word


@pytest.mark.parametrize("ema", [False, True], ids=["copy", "ema"])
@pytest.mark.parametrize("dt,d", [(dt, d) for dt in DTYPES for d in WIDTHS], ids=[f"{dt}-d{d}-VB16" for dt in DTYPES
                                                                               for d in WIDTHS])
def test_push_drop(dt, d, ema):
    """The receiver's dropout fused into the push: message = keep ? T(fl(v * scale)) : 0 with keep the host port of
    the mask at row dst_row0 + r and v the clean row (or T(e) with EMA); without EMA also bit-identical to
    pg_dropout_rows(row0 = dst_row0) of the same rows; the mirror is bit-identical to the same launch without dropout."""
    from pipegcn_b200 import ops
    dtype = DTYPES[dt]
    step = torch.tensor([4], dtype=torch.int32, device=DEV)
    spec = ops.DropSpec(0.3, 0x1234_5678_9ABC_DEF1 + d, step, 1)
    pushes, e0 = [], None
    for drop in (spec, None):
        gen = torch.Generator().manual_seed(d * 7 + ema)
        p = Push(P8, d, dtype, 16, gen, ema=ema, row0s=DROP_ROW0)
        if ema and e0 is None:
            e0 = [p.mir.base[_mir_block(p, m)].cpu().clone() for m in range(len(P8))]
        p.launch(momentum=0.9 if ema else 0.0, value=9, drop=drop)
        p.check_flags(9)
        pushes.append(p)
    p, plain = pushes
    want, nan_at = _fresh(p.dst0)
    for m, (_, n) in enumerate(P8):
        if n == 0:
            continue
        v = p.src_rows(m).float()
        if ema:
            v = ema_step(e0[m], v, 0.9).to(dtype).float()                            # T(e)
        want[_dst_block(p, m)], nan_at[_dst_block(p, m)] = _drop_ref(p, m, v, spec, 4)
        if not ema:
            rows = padded(n, d, dtype, data=p.src[p.rows[m].to(DEV)])
            ref = ops.dropout_rows(rows, spec, row0=p.dst_row0[m])
            got = p.dst.base[_dst_block(p, m)][:, :d]
            assert torch.equal(_bits(got), _bits(ref)), f"message {m} != pg_dropout_rows"
    check_image(p.dst.base, want, nan_at, "dropped message rows")
    if ema:
        assert torch.equal(_bits(p.mir.base), _bits(plain.mir.base)), "the mirror depends on the dropout"


@pytest.mark.parametrize("dt,vb", [("fp32", 8), ("fp32", 4), ("bf16", 8), ("bf16", 4), ("bf16", 2)],
                         ids=lambda v: str(v))
def test_push_drop_refuses_narrow_vectors(dt, vb):
    """The dropout mask is defined on 16-byte vectors: a source that allows fewer bytes per vector is refused, and
    nothing is written or published."""
    from pipegcn_b200 import _C, ops
    p = Push(P8, 65, DTYPES[dt], vb, torch.Generator().manual_seed(vb))
    before = _bits(p.dst.base).clone()
    with pytest.raises(_C.PgError, match="the dropout mask is defined on 16-byte vectors"):
        p.launch(value=3, drop=ops.DropSpec(0.5, 1))
    assert torch.equal(_bits(p.dst.base), before) and _u32(p.flags) == [0] * len(P8)


def _sets():
    w = sm_count() * 8 * 32          # a wave of push CTAs: SMs x 8 resident CTAs (assumed, not measured) x 32 rows
    return {
        "one": [("idx", 257)],
        "empty-first": [("row0", 0), ("idx", 33), ("row0", 32)],
        "empty-middle": [("idx", 31), ("row0", 0), ("row0", 0), ("idx", 255)],
        "empty-last": [("idx", 1), ("row0", 257), ("idx", 0)],
        "all-empty": [("idx", 0), ("row0", 0), ("idx", 0), ("row0", 0), ("idx", 0), ("row0", 0), ("idx", 0)],
        "256-msgs": [("idx" if m % 2 else "row0", (0, 1, 31, 32, 33, 2, 0, 9)[m % 8] + m // 64) for m in range(256)],
        "4-waves": [("row0", 33), ("idx", 4 * w + 5), ("idx", 0)],
    }


SET_NAMES = ["one", "empty-first", "empty-middle", "empty-last", "all-empty", "256-msgs", "4-waves"]


@pytest.mark.parametrize("name", SET_NAMES)
@pytest.mark.parametrize("dt,vb", [("fp32", 16), ("bf16", 2)], ids=["fp32-d65-VB16", "bf16-d65-VB2"])
def test_push_message_sets(dt, vb, name):
    """Message sets from one message to the documented 256, empty messages first, in the middle and last, all
    empty (the flag-only kernel), and one message of four waves of CTAs: rows, guards, flags and counters."""
    gen = torch.Generator().manual_seed(len(name) + vb)
    spec = _sets()[name]
    p = Push(spec, 65, DTYPES[dt], vb, gen)
    assert p.ms.n_ctas == sum((n + 31) // 32 for _, n in spec)
    p.launch(value=77)
    check_image(p.dst.base, copy_image(p), what=f"message rows of {name}")
    p.check_flags(77)


def test_push_misaligned_base():
    """A 16-byte stride whose base allows only 4-byte (fp32) or 2-byte (bf16) vectors: the entry point picks them from
    the base address, and the copy is exact over [0, d)."""
    for dtype, col in ((torch.float32, 1), (torch.bfloat16, 1), (torch.bfloat16, 2), (torch.float32, 2)):
        gen = torch.Generator().manual_seed(col)
        p = Push(P8, 37, dtype, 16, gen)
        shifted = p.src.as_strided((p.src.shape[0], 37), (p.src.stride(0), 1), p.src.storage_offset() + col)
        es = _es(dtype)
        vb = picked_vb(37, es, [(shifted.data_ptr(), shifted.stride(0))])
        assert vb == col * es
        p.src, p.end = shifted, _rup(37, vb // es)
        p.launch(src=shifted, value=2)
        check_image(p.dst.base, copy_image(p), what=f"{dtype} base + {col}: VB{vb}")
        p.check_flags(2)


def test_push_flags_and_counters():
    """Flags, including those of empty messages, hold value + *value_dev after a launch; counters reset, so the same
    message set launched again publishes the new value; 0xFFFFFFFE + 3 publishes 1 (wrap-around)."""
    gen = torch.Generator().manual_seed(3)
    p = Push(P8, 64, torch.float32, 16, gen)
    dev = torch.tensor([3], dtype=torch.int32, device=DEV)
    p.launch(value=10, value_dev=dev.data_ptr())
    p.check_flags(13)
    p.launch(value=20)
    p.check_flags(20)
    p.launch(value=0xFFFFFFFE, value_dev=dev.data_ptr())
    p.check_flags(1)
    check_image(p.dst.base, copy_image(p), what="rows after three launches")
    empty = Push([("idx", 0), ("row0", 0)], 64, torch.float32, 16, gen)
    for value in (6, 0xFFFFFFFE):
        empty.launch(value=value, value_dev=dev.data_ptr())
        empty.check_flags((value + 3) & U32)


def test_push_refusals():
    """n_msgs 0 and 257, d <= 0 and ld_src < d are refused before anything is launched."""
    from pipegcn_b200 import _C
    p = Push(P8, 64, torch.float32, 16, torch.Generator().manual_seed(4))
    before = _bits(p.dst.base).clone()
    for kw, msg in ((dict(n_msgs=0), "messages per launch"), (dict(n_msgs=257), "messages per launch"),
                    (dict(d=0), "bad sizes"), (dict(d=-1), "bad sizes"), (dict(ld=63), "bad sizes")):
        with pytest.raises(_C.PgError, match=msg):
            p.launch(value=1, **kw)
    assert torch.equal(_bits(p.dst.base), before) and _u32(p.flags) == [0] * len(P8)


def test_buffer_update_bf16_odd_width():
    """Buffer.update(0, x) with x a contiguous bf16 [N_in, d] tensor of odd d (static layer-0 store off) at P = 2: the
    push reads x with 2-byte vectors, and every rank's result is cat(x_r, the peers' boundary rows) bit for bit."""
    from pipegcn_b200.helper.feature_buffer import Buffer
    from pipegcn_b200.helper.timer.comm_timer import CommTimer
    from pipegcn_b200.world import LocalWorld
    from tests.helpers import small_world
    _, _, layouts, _ = small_world("tiny", 2)
    d = 21
    world = LocalWorld(2, "cuda")
    gen = torch.Generator().manual_seed(21)
    feats = [(torch.randn(lay.num_in, d, generator=gen) * 3).to(torch.bfloat16).to(DEV) for lay in layouts]
    assert all(f.is_contiguous() and f.stride(0) == d for f in feats)
    bufs = []
    for r, lay in enumerate(layouts):
        b = Buffer(world.view(r))
        b.timer = CommTimer()
        b.timeout_ms = 5000
        b.init_buffer(lay.num_in, lay.num_all, lay.boundary, lay.recv_shape, [d, 16], dtype=torch.bfloat16)
        bufs.append(b)
    for b in bufs:           # map the peers before any flag wait is launched: nothing may synchronise while one spins
        b._connect()
    streams = [torch.cuda.Stream() for _ in layouts]
    torch.cuda.synchronize()
    outs = []
    for r, b in enumerate(bufs):
        with torch.cuda.stream(streams[r]):
            outs.append(b.update(0, feats[r]))
    torch.cuda.synchronize()
    for r, b in enumerate(bufs):
        b.check_status()
        want = torch.cat([feats[r]] + [feats[j][layouts[j].boundary[r].to(DEV)] for j in range(2) if j != r])
        assert torch.equal(_bits(outs[r]), _bits(want)), r


# ============================================ pg_halo_wait ============================================================
def _wait(ptrs, n, value, value_dev=None, status=None, wait_ns=None):
    from pipegcn_b200 import _C
    rc = _C.lib.pg_halo_wait(ptrs.data_ptr() if ptrs is not None else None, n, value, value_dev, 5000,
                             status.data_ptr() if status is not None else None,
                             wait_ns.data_ptr() if wait_ns is not None else None, _C.stream_ptr())
    _C.check(rc, "pg_halo_wait")
    torch.cuda.synchronize()


def _flag_ptrs(flags, gen):
    perm = torch.randperm(flags.numel(), generator=gen)
    return (flags.data_ptr() + 4 * perm).to(torch.int64).to(DEV)


PRESET_NS = 1 << 40


@pytest.mark.parametrize("n_flags", [1, 7, 31, 32, 33, 1024])
def test_wait_published_flags(n_flags):
    """Flags equal to or ahead of the value (by up to 2^31 - 1) return at once: status stays 0, and the blocked time
    is added to a preset wait_ns, never stored over it."""
    gen = torch.Generator().manual_seed(n_flags)
    value = 0x7000_0000
    ahead = torch.randint(0, 3, (n_flags,), generator=gen)
    ahead[-1] = 0x7FFF_FFFF
    flags = _i32((value + ahead).tolist())
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    wait_ns = torch.tensor([PRESET_NS], dtype=torch.int64, device=DEV)
    _wait(_flag_ptrs(flags, gen), n_flags, value, status=status, wait_ns=wait_ns)
    assert int(status.item()) == 0
    ns = int(wait_ns.item())
    assert PRESET_NS <= ns < PRESET_NS + 5 * 10 ** 9, ns


def test_wait_wraparound_and_device_value():
    """Flag 2 passes value 0xFFFFFFFF (signed distance); with value_dev the sum value + *value_dev is awaited, also
    across the wrap; status and wait_ns may be NULL."""
    gen = torch.Generator().manual_seed(0)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    flags = torch.tensor([2], dtype=torch.int32, device=DEV)
    _wait(_flag_ptrs(flags, gen), 1, 0xFFFFFFFF, status=status)
    dev = torch.tensor([0x20], dtype=torch.int32, device=DEV)
    flags = torch.tensor([0x10, 0x10, 0x11], dtype=torch.int32, device=DEV)
    _wait(_flag_ptrs(flags, gen), 3, 0xFFFFFFF0, dev.data_ptr(), status=status)
    _wait(_flag_ptrs(flags, gen), 3, 0xFFFFFFF0, dev.data_ptr())
    assert int(status.item()) == 0


def test_wait_counts():
    """n_flags = 0 launches nothing (wait_ns keeps its exact value); 1025 flags are refused."""
    from pipegcn_b200 import _C
    wait_ns = torch.tensor([PRESET_NS], dtype=torch.int64, device=DEV)
    _wait(None, 0, 1, wait_ns=wait_ns)
    assert int(wait_ns.item()) == PRESET_NS
    flags = torch.zeros(1025, dtype=torch.int32, device=DEV)
    with pytest.raises(_C.PgError, match="bad flag count 1025"):
        _wait(_flag_ptrs(flags, torch.Generator().manual_seed(1)), 1025, 0)


# ============================================ pg_boundary_add =========================================================
def boundary_case(dtype, d, vb, n_urow, gen):
    """grad rows urow (a scrambled subset) += the recv slots usrc[uptr[i]:uptr[i+1]] (1..7 slots, scrambled), with a
    NaN and an Inf in two slots.  Returns (grad Guarded, want bits, nan_at)."""
    from pipegcn_b200 import _C
    es = _es(dtype)
    n_grad = 2 * n_urow + 5
    counts = torch.randint(1, 8, (n_urow,), generator=gen)
    counts[0] = 1
    counts[-1] = 7
    n_slots = int(counts.sum())
    urow = torch.randperm(n_grad, generator=gen)[:n_urow]
    usrc = torch.randperm(n_slots, generator=gen)
    uptr = torch.zeros(n_urow + 1, dtype=torch.int64)
    uptr[1:] = torch.cumsum(counts, 0)
    recv = source(n_slots, d, dtype, vb, gen)
    recv[int(usrc[0]), d // 2] = NAN
    recv[int(usrc[-1]), d - 1] = float("inf")
    grad = guarded(n_grad, d, dtype, vb)
    grad.t.copy_((torch.randn(n_grad, d, generator=gen) * 4).to(dtype))
    assert picked_vb(d, es, [(grad.t.data_ptr(), grad.ld), (recv.data_ptr(), recv.stride(0))]) == vb
    want, nan_at = _fresh(image(grad))
    v = vb // es
    end = _rup(d, v)
    g = grad.t.cpu()[urow].float()
    rc = recv.cpu().float()
    for j in range(7):                        # slot order, rounding like the reference's per-peer loop
        sel = counts > j
        g[sel] = g[sel] + rc[usrc[uptr[:-1][sel] + j]]
        if dtype == torch.bfloat16:
            g[sel] = g[sel].to(dtype).float()
    rows = urow + grad.G
    c0 = grad.col0
    want[rows, c0:c0 + d] = _bits(g.to(dtype))
    nan_at[rows, c0:c0 + d] = g.isnan()
    nan_at[rows, c0 + d:c0 + end] = True                          # + the recv pad columns (NaN)
    dev = [t.to(torch.int32).to(DEV) for t in (urow, uptr, usrc)]
    rc_ = _C.lib.pg_boundary_add(grad.t.data_ptr(), grad.ld, recv.data_ptr(), recv.stride(0), d, _C.dtype_code(dtype),
                                 dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), n_urow, _C.stream_ptr())
    _C.check(rc_, "pg_boundary_add")
    torch.cuda.synchronize()
    return grad, want, nan_at


BADD_CASES = [c for c in WIDTH_CASES if c[2] != 2]


@pytest.mark.parametrize("dt,d,vb", BADD_CASES, ids=[f"{dt}-d{d}-VB{vb}" for dt, d, vb in BADD_CASES])
def test_boundary_add(dt, d, vb):
    """Ordered scatter-add of the gradient slots: fp32 sums in slot order, bf16 rounded after every add; rows outside
    urow, the columns >= round_up(d, V) and the guards untouched; a NaN and an Inf stay in their row and column."""
    for n_urow in (1, 300):
        gen = torch.Generator().manual_seed(d * 100 + vb + n_urow)
        grad, want, nan_at = boundary_case(DTYPES[dt], d, vb, n_urow, gen)
        check_image(grad.base, want, nan_at, f"n_urow {n_urow}")


@pytest.mark.parametrize("dt,vb", [("fp32", 16), ("bf16", 4)], ids=["fp32-d65-VB16", "bf16-d65-VB4"])
def test_boundary_add_waves(dt, vb):
    """Four waves of rows (8 warps per 256-thread block at 8 blocks per SM, assumed: 64 rows per SM)."""
    n_urow = 4 * 64 * sm_count()
    grad, want, nan_at = boundary_case(DTYPES[dt], 65, vb, n_urow, torch.Generator().manual_seed(5))
    check_image(grad.base, want, nan_at, "four waves")


def test_boundary_add_refuses_2byte_bf16():
    from pipegcn_b200 import _C
    gen = torch.Generator().manual_seed(2)
    recv = source(4, 9, torch.bfloat16, 2, gen)
    grad = guarded(4, 9, torch.bfloat16, 2)
    idx = torch.zeros(2, dtype=torch.int32, device=DEV)
    idx[1] = 1
    rc = _C.lib.pg_boundary_add(grad.t.data_ptr(), grad.ld, recv.data_ptr(), recv.stride(0), 9, _C.PG_BF16,
                                idx.data_ptr(), idx.data_ptr(), idx.data_ptr(), 1, _C.stream_ptr())
    assert rc == _C.PG_ERR_INVALID
    assert "bf16 rows must be 4-byte aligned" in _C.lib.pg_last_error().decode()


# ============================================ pg_scale_rows ===========================================================
def scale_c(m, k, corr):
    """c = 0 for k <= 0, 1 without corr, else float32(1 - float64(float32(m))^k).  The device evaluates the power in
    double too: exact equality is sound when no double within 2^-48 of 1 - m^k rounds to another float32."""
    if k <= 0:
        return np.float32(0.0)
    if not corr:
        return np.float32(1.0)
    y = 1.0 - float(np.float64(np.float32(m)) ** k)
    c = np.float32(y)
    assert np.float32(y - 2.0 ** -48) == c == np.float32(y + 2.0 ** -48), (m, k, "near a float32 rounding boundary")
    return c


def special_source(n, d, dtype, vb, gen):
    """source() rows with -0.0, +-Inf and NaNs with payloads (what the raw copy must keep)."""
    x = source(n, d, dtype, vb, gen)
    b = _bits(x)
    if dtype == torch.float32:
        specials = [0x80000000, 0x7FC12345, 0xFFC00001, 0x7F800000, 0xFF800000]
    else:
        specials = [0x8000, 0x7FC3, 0xFFC1, 0x7F80, 0xFF80]
    for i, s in enumerate(specials):
        if s >= (1 << (8 * _es(dtype) - 1)):
            s -= 1 << (8 * _es(dtype))
        b[(7 * i + 3) % n, (5 * i) % d] = s
    return x


def run_scale(src, d, dtype, vb, m, corr, k_host, k_dev=None):
    from pipegcn_b200 import _C
    n = src.shape[0]
    out = guarded(n, d, dtype, vb)
    assert picked_vb(d, _es(dtype), [(src.data_ptr(), src.stride(0)), (out.t.data_ptr(), out.ld)]) == vb
    out.before = image(out)
    rc = _C.lib.pg_scale_rows(src.data_ptr(), src.stride(0), out.t.data_ptr(), out.ld, n, d, _C.dtype_code(dtype), m,
                              corr, k_host, k_dev.data_ptr() if k_dev is not None else None, _C.stream_ptr())
    _C.check(rc, "pg_scale_rows")
    torch.cuda.synchronize()
    return out


def scale_image(out, src, c, vb):
    """dst = T(fl(float(src) * c)) over [0, round_up(d, V)); c == 1 is a raw copy (NaN payloads, -0.0 kept)."""
    want, nan_at = _fresh(out.before)
    n, d = src.shape
    end = _rup(d, vb // _es(src.dtype))
    full = _stored(src, end).cpu()
    blk = (slice(out.G, out.G + n), slice(out.col0, out.col0 + end))
    if c == 1:
        want[blk] = _bits(full)
    else:
        y = full.float() * torch.tensor(c)
        want[blk] = _bits(y.to(src.dtype))
        nan_at[blk] = y.isnan()
    return want, nan_at


@pytest.mark.parametrize("dt,d,vb", WIDTH_CASES, ids=WIDTH_IDS)
def test_scale_rows_widths(dt, d, vb):
    """Every VB: c = 1 - 0.95^7 scales, c = 1 (corr 0) copies raw bits."""
    dtype = DTYPES[dt]
    src = special_source(70, d, dtype, vb, torch.Generator().manual_seed(d + vb))
    for corr, k in ((1, 7), (0, 3)):
        c = scale_c(0.95, k, corr)
        out = run_scale(src, d, dtype, vb, 0.95, corr, k)
        check_image(out.base, *scale_image(out, src, c, vb), f"corr {corr} k {k}")


@pytest.mark.parametrize("k_dev", [False, True], ids=["host-k", "device-k"])
@pytest.mark.parametrize("m", [0.9, 0.95])
@pytest.mark.parametrize("corr", [0, 1])
@pytest.mark.parametrize("k", [-1, 0, 1, 2, 7, 200])
def test_scale_rows_closed_form(k, corr, m, k_dev):
    """c over k, corr and m (k split between k_host and *k_dev): c = 0 for k <= 0, and 0.9^200 rounds c to 1 (the raw
    copy)."""
    for dtype, d, vb in ((torch.float32, 65, 16), (torch.bfloat16, 9, 2)):
        src = special_source(50, d, dtype, vb, torch.Generator().manual_seed(k + 300))
        c = scale_c(m, k, corr)
        if k_dev:
            dev = torch.tensor([5], dtype=torch.int32, device=DEV)
            out = run_scale(src, d, dtype, vb, m, corr, k - 5, dev)
        else:
            out = run_scale(src, d, dtype, vb, m, corr, k)
        check_image(out.base, *scale_image(out, src, c, vb), f"{dtype} c {c}")
    if (m, k, corr) == (0.9, 200, 1):
        assert c == 1


def test_scale_rows_grid_stride():
    """n_rows * nvec past the grid (16 x SMs x 256 threads) about 2.5 times: the grid-stride loop wraps."""
    n = int(2.5 * 16 * sm_count() * 256 / 16) + 3          # d = 64 fp32 at VB16: 16 vectors per row
    src = special_source(n, 64, torch.float32, 16, torch.Generator().manual_seed(9))
    c = scale_c(0.9, 3, 1)
    out = run_scale(src, 64, torch.float32, 16, 0.9, 1, 3)
    check_image(out.base, *scale_image(out, src, c, 16), "grid-stride")


# ============================================ pg_bns_mask_rows ========================================================
def run_mask(dst, src, mask, d, dtype):
    from pipegcn_b200 import _C
    rc = _C.lib.pg_bns_mask_rows(src.data_ptr() if src is not None else None, src.stride(0) if src is not None else 0,
                                 dst.t.data_ptr(), dst.ld, dst.n, d, _C.dtype_code(dtype), mask.data_ptr(),
                                 _C.stream_ptr())
    _C.check(rc, "pg_bns_mask_rows")
    torch.cuda.synchronize()


def mask_cases(n, d, dtype, vb, gen, masks):
    """For every mask, both modes: dst = mask ? src : 0, and (src NULL) the unkept rows zeroed, the kept ones left."""
    v = vb // _es(dtype)
    end = _rup(d, v)
    src = source(n, d, dtype, vb, gen)
    full = _stored(src, end).cpu()
    for mname, mask in masks.items():
        for with_src in (True, False):
            dst = guarded(n, d, dtype, vb)
            dst.base[dst.G:dst.G + n, dst.col0:dst.col0 + end] = (torch.randn(n, end, generator=gen)).to(dtype).to(DEV)
            ops = [(src.data_ptr(), src.stride(0))] if with_src else []
            assert picked_vb(d, _es(dtype), ops + [(dst.t.data_ptr(), dst.ld)]) == vb
            want = image(dst)
            blk = want[dst.G:dst.G + n, dst.col0:dst.col0 + end]
            keep = mask.bool().cpu()
            if with_src:
                blk[keep] = _bits(full)[keep]
            blk[~keep] = 0
            run_mask(dst, src if with_src else None, mask, d, dtype)
            check_image(dst.base, want, what=f"mask {mname}, {'src' if with_src else 'src NULL'}")


def _masks(n, gen):
    return {"zeros": torch.zeros(n, dtype=torch.uint8, device=DEV), "ones": torch.ones(n, dtype=torch.uint8, device=DEV),
            "random": torch.randint(0, 2, (n,), generator=gen, dtype=torch.uint8).to(DEV)}


@pytest.mark.parametrize("dt,d,vb", WIDTH_CASES, ids=WIDTH_IDS)
def test_bns_mask_rows(dt, d, vb):
    gen = torch.Generator().manual_seed(d * 3 + vb)
    mask_cases(90, d, DTYPES[dt], vb, gen, _masks(90, gen))


def test_bns_mask_rows_grid_stride():
    """bf16 at VB2, n_rows * nvec about 2.5 grids: the grid-stride loop wraps."""
    d = 9
    n = int(2.5 * 16 * sm_count() * 256 / d) + 3
    gen = torch.Generator().manual_seed(11)
    mask_cases(n, d, torch.bfloat16, 2, gen, {"random": _masks(n, gen)["random"]})
