"""Conformance of the attention kernels (csrc/attention.cu: GAT, GATv2, the graph transformer and their shared column
sums) with plain fp64 restatements of the same operations, on every head-width instantiation, past the first wave of
CTAs and at the edges of the online softmax.

Conventions (those of tests/test_kernel_conformance_gpu.py, whose helpers are imported):
- Every pass is driven through the C ABI, so that it writes into `Guarded` views (allowed region exactly [0, H*D) of
  a row, [0, H) for the per-head statistics) that hold NaN before the call: an unwritten row shows.
- Inputs live in `padded` storage whose pad columns hold NaN; unkept halo rows and the source rows nobody references
  hold NaN as well.  No NaN may reach any output.
- Teacher forcing: every pass gets the kernel's own outputs of the pass before (m, s, dv / der, delta), and its fp64
  reference is computed from exactly those, so that an error is attributed to the pass that made it.
- Bounds are elementwise, |got - ref| <= c * mag, with mag the same sum over absolute values and c derived from the
  kernel's arithmetic (see `fwd_c` and `bwd_c`); a bf16 output adds one bf16 rounding.
- Two launches give the same bits for every output, the fp32 side outputs included.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

from tests.test_kernel_conformance_gpu import U24, Guarded, _bits, assert_within, padded, sm_count

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")
SLOPE = float(np.float32(0.2))          # kNegSlope, as the kernels hold it (0.2f)


def nj_of(d):
    return 1 if d <= 32 else 2 if d <= 64 else 4 if d <= 128 else 8 if d <= 256 else 16


def edges_per_step(fam, nj):
    """Edges a warp takes per step: GAT 32 (one per lane), GATv2 v2_edges<NJ>(), the transformer tc_edges<NJ>()."""
    if fam == "gat":
        return 32
    if fam == "gatv2":
        return 2 if nj <= 2 else 4 if nj <= 4 else 2 if nj <= 8 else 1
    return 4 if nj <= 4 else 2


# ============================================== the graph ==========================================================
NUM_IN, NUM_HALO = 3000, 1200
NUM_ALL = NUM_IN + NUM_HALO
NOSRC = 7                                           # an inner row that is nobody's source (empty CSC row)
PEAKS = np.arange(NUM_IN - 200, NUM_IN)             # inner rows referenced once: the last entry of a row of > 32
UNKEPT = np.arange(NUM_IN, NUM_IN + 100)            # halo rows always out of the sample
HUB = NUM_IN + 100                                  # a kept halo row with a long CSC row
UNREF = np.arange(NUM_ALL - 100, NUM_ALL)           # halo rows nobody references


class Graph:
    """A PartGraph with the host-side facts the references need: the forward edges (CSR order), the keep mask, the
    poisoned rows, and per plan the entries and segments of every row."""

    def __init__(self, num_in, num_all, lens, indices, keep_halo, seg_len, peak_of=None):
        from pipegcn_b200.graph import PartGraph
        self.num_in, self.num_all = num_in, num_all
        indptr = np.zeros(num_in + 1, dtype=np.int64)
        indptr[1:] = np.cumsum(lens)
        dst = np.repeat(np.arange(num_in), lens)
        order = np.argsort(indices, kind="stable")
        t_indptr = np.zeros(num_all + 1, dtype=np.int64)
        t_indptr[1:] = np.cumsum(np.bincount(indices, minlength=num_all))
        i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(torch.int32)
        self.g = PartGraph(num_in, num_all, i32(indptr), i32(indices), i32(t_indptr), i32(dst[order]),
                           torch.from_numpy(np.asarray(lens)), device=DEV, seg_len=seg_len)
        self.indptr = torch.from_numpy(indptr).to(DEV)
        self.rows = torch.from_numpy(dst).to(DEV)
        self.cols = torch.from_numpy(indices.astype(np.int64)).to(DEV)
        self.keep = torch.from_numpy(keep_halo.astype(np.uint8)).to(DEV).contiguous()
        self.keep_u = torch.cat([torch.ones(num_in, dtype=torch.bool, device=DEV), self.keep.bool()])
        refs = torch.bincount(self.cols, minlength=num_all)
        self.bad = ~self.keep_u | (refs == 0)                 # rows that hold NaN in every source tensor
        self.bad[:num_in] = False                             # inner rows are destinations too: always finite
        kept = self.keep_u[self.cols]
        self.kv, self.ku = self.rows[kept], self.cols[kept]   # the kept edges, CSR order
        self.edge_kept = kept
        self.peak_of = peak_of                                # {peak source row: its destination}
        self.n_dst, self.seg_dst = self._row_stats(self.g.fwd)
        self.n_src, self.seg_src = self._row_stats(self.g.bwd)

    @staticmethod
    def _row_stats(plan):
        n = (plan.indptr[1:] - plan.indptr[:-1]).double()
        seg = torch.zeros(plan.n_rows, dtype=torch.float64, device=DEV)
        if plan.n_long:
            seg[plan.long_row.long()] = (plan.long_seg_ptr[1:] - plan.long_seg_ptr[:-1]).double()
        return n[:, None], seg[:, None]


@functools.lru_cache(None)
def structured_graph(seg_len):
    """Every chunk kind CsrPlan._build_chunks makes: kind 0 (32 empty rows per chunk; rows of exactly 1, 2, 4, 8, 16
    and 32 entries; ragged short rows), kind 1 (33..200 entries and seg_len, one row per chunk; long at seg_len 32),
    kind 2 (seg_len + 1, 2 and 3 seg_len, hubs of 4 seg_len + 17 and 5 seg_len).  Plus: a halo row with a long CSC
    row, an inner row that is nobody's source, a repeated source inside a row, source rows referenced many times (the
    pidx hot bit), a row whose every source is unkept, a 32-edge batch and a whole hub segment of unkept sources, and
    a once-referenced "peak" source as the last entry of every row of more than 32 entries."""
    rng = np.random.default_rng(seg_len)
    tagged = [(0, "")] * 70 + [(n, "") for n in (1, 2, 4, 8, 16, 32) for _ in range(32 // n * 4)]
    tagged += [(int(n), "") for n in rng.integers(33, 201, 40)] + [(seg_len, ""), (100, "batch-unkept")]
    tagged += [(n, "") for n in (seg_len + 1, 2 * seg_len, 3 * seg_len, 4 * seg_len + 17)]
    tagged += [(5 * seg_len, "segment-unkept"), (10, "all-unkept"), (12, "repeat")]
    tagged += [(int(n), "") for n in rng.integers(1, 13, NUM_IN - len(tagged))]
    tagged = [tagged[i] for i in rng.permutation(len(tagged))]
    lens = np.array([n for n, _ in tagged], dtype=np.int64)
    tag = {t: i for i, (_, t) in enumerate(tagged) if t}
    indptr = np.zeros(NUM_IN + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(lens)
    pool = np.concatenate([np.setdiff1d(np.arange(NUM_IN - 200), [NOSRC]), np.arange(HUB + 1, UNREF[0])])
    idx = rng.choice(pool, int(indptr[-1]))
    idx[rng.choice(idx.size, 600, replace=False)] = HUB
    b = indptr[tag["repeat"]]
    idx[b:b + 5] = pool[3]
    b = indptr[tag["all-unkept"]]
    idx[b:b + 10] = rng.choice(UNKEPT, 10)
    b = indptr[tag["batch-unkept"]]
    idx[b + 32:b + 64] = rng.choice(UNKEPT, 32)
    b = indptr[tag["segment-unkept"]]
    idx[b + seg_len:b + 2 * seg_len] = rng.choice(UNKEPT, seg_len)
    peak_of = {}
    for v in np.nonzero(lens > 32)[0]:
        u = int(PEAKS[len(peak_of)])
        idx[indptr[v + 1] - 1] = u
        peak_of[u] = int(v)
    keep = rng.random(NUM_HALO) < 0.5
    keep[UNKEPT - NUM_IN] = False
    keep[HUB - NUM_IN] = True
    G = Graph(NUM_IN, NUM_ALL, lens, idx, keep, seg_len, peak_of)
    fwd, bwd = G.g.fwd, G.g.bwd
    kinds = set((fwd.chunks[:, 3] & 3).tolist())
    assert kinds == ({0, 2} if seg_len == 32 else {0, 1, 2})
    assert fwd.n_long == int((lens > seg_len).sum()) >= 5 and bwd.n_long >= 1
    hubs = fwd.long_seg_ptr[1:] - fwd.long_seg_ptr[:-1]
    assert int((hubs >= 4).sum()) >= 2 and fwd.n_seg >= fwd.n_long + 8
    empty32 = (fwd.chunks[:, 3] & 3 == 0) & (fwd.chunks[:, 1] == 0) & (fwd.chunks[:, 3] >> 2 == 32)
    assert bool(empty32.any())
    assert bool((fwd.pidx < 0).any()) and bool((bwd.pidx < 0).any())
    assert int(bwd.indptr[NOSRC + 1] - bwd.indptr[NOSRC]) == 0
    assert int(bwd.indptr[HUB + 1] - bwd.indptr[HUB]) > 2 * seg_len
    return G


@functools.lru_cache(None)
def wide_graph():
    """Short rows only, sized so that both plans have more than 16 * SMs CTAs of 4 warps (16 resident per SM at the
    most): every CTA index past the first wave runs."""
    rng = np.random.default_rng(11)
    num_in, num_halo = 120_000, 20_000
    lens = rng.integers(0, 9, num_in)
    idx = rng.integers(0, num_in + num_halo, int(lens.sum()))
    G = Graph(num_in, num_in + num_halo, lens, idx, rng.random(num_halo) < 0.5, 32)
    waves = 16 * sm_count()
    assert G.g.fwd.n_chunks // 4 > waves and G.g.bwd.n_chunks // 4 > waves
    return G


# ============================================== C ABI ==============================================================
def _call(name, *args):
    from pipegcn_b200 import _C
    _C.check(getattr(_C.lib, name)(*args, _C.stream_ptr()), name)


def _stats(n, H):
    return Guarded(n, H, torch.float32, ld=H)


def _scratch(plan, H, D):
    return torch.full((max(1, plan.n_seg * H * (4 * D + 2)),), NAN, device=DEV)


def _code(dtype):
    from pipegcn_b200 import _C
    return _C.dtype_code(dtype)


def run_gat(G, t, H, D, dtype):
    """pg_gat_aggregate, pg_gat_bwd_dst, pg_gat_bwd_src, each fed the outputs of the one before."""
    g, n_in, n_all, hd = G.g, G.num_in, G.num_all, H * D
    fwd, bwd = C.byref(g.fwd.c), C.byref(g.bwd.c)
    z, gr, code = t["z"], t["g"], _code(dtype)
    out, m, s = Guarded(n_in, hd, dtype), _stats(n_in, H), _stats(n_in, H)
    _call("pg_gat_aggregate", fwd, z.data_ptr(), z.stride(0), H, D, code, t["el"].data_ptr(), t["er"].data_ptr(),
          t["bias"].data_ptr(), G.keep.data_ptr(), n_in, out.t.data_ptr(), out.t.stride(0), m.t.data_ptr(),
          s.t.data_ptr(), _scratch(g.fwd, H, D).data_ptr())
    der, dv = _stats(n_in, H), _stats(n_in, H)
    _call("pg_gat_bwd_dst", fwd, z.data_ptr(), z.stride(0), gr.data_ptr(), gr.stride(0), H, D, code,
          t["el"].data_ptr(), t["er"].data_ptr(), m.t.data_ptr(), s.t.data_ptr(), G.keep.data_ptr(), n_in,
          der.t.data_ptr(), dv.t.data_ptr(), _scratch(g.fwd, H, D).data_ptr())
    dz, dl = Guarded(n_all, hd, dtype), _stats(n_all, H)
    _call("pg_gat_bwd_src", bwd, z.data_ptr(), z.stride(0), gr.data_ptr(), gr.stride(0), H, D, code,
          t["el"].data_ptr(), t["er"].data_ptr(), m.t.data_ptr(), s.t.data_ptr(), dv.t.data_ptr(), der.t.data_ptr(),
          t["al"].data_ptr(), t["ar"].data_ptr(), G.keep.data_ptr(), n_in, dz.t.data_ptr(), dz.t.stride(0),
          dl.t.data_ptr(), _scratch(g.bwd, H, D).data_ptr())
    return dict(out=out, m=m, s=s, der=der, dv=dv, dz=dz, del_=dl)


def run_gatv2(G, t, H, D, dtype):
    """pg_gatv2_aggregate, pg_gatv2_bwd_dst, pg_gatv2_bwd_src."""
    g, n_in, n_all, hd = G.g, G.num_in, G.num_all, H * D
    fwd, bwd = C.byref(g.fwd.c), C.byref(g.bwd.c)
    zs, zd, gr, at, code = t["zs"], t["zd"], t["g"], t["attn"], _code(dtype)
    out, m, s = Guarded(n_in, hd, dtype), _stats(n_in, H), _stats(n_in, H)
    _call("pg_gatv2_aggregate", fwd, zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), H, D, code,
          at.data_ptr(), G.keep.data_ptr(), n_in, out.t.data_ptr(), out.t.stride(0), m.t.data_ptr(), s.t.data_ptr(),
          _scratch(g.fwd, H, D).data_ptr())
    dzd, dv, pattn = Guarded(n_in, hd, dtype), _stats(n_in, H), Guarded(n_in, hd, torch.float32)
    _call("pg_gatv2_bwd_dst", fwd, zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), gr.data_ptr(),
          gr.stride(0), H, D, code, at.data_ptr(), m.t.data_ptr(), s.t.data_ptr(), G.keep.data_ptr(), n_in,
          dzd.t.data_ptr(), dzd.t.stride(0), dv.t.data_ptr(), pattn.t.data_ptr(), pattn.t.stride(0),
          _scratch(g.fwd, H, D).data_ptr())
    dzs = Guarded(n_all, hd, dtype)
    _call("pg_gatv2_bwd_src", bwd, zs.data_ptr(), zs.stride(0), zd.data_ptr(), zd.stride(0), gr.data_ptr(),
          gr.stride(0), H, D, code, at.data_ptr(), m.t.data_ptr(), s.t.data_ptr(), dv.t.data_ptr(), G.keep.data_ptr(),
          n_in, dzs.t.data_ptr(), dzs.t.stride(0), _scratch(g.bwd, H, D).data_ptr())
    return dict(out=out, m=m, s=s, dzd=dzd, dv=dv, pattn=pattn, dzs=dzs)


def run_tconv(G, t, H, D, dtype):
    """pg_tconv_aggregate, pg_tconv_bwd_dst, pg_tconv_bwd_src."""
    g, n_in, n_all, hd = G.g, G.num_in, G.num_all, H * D
    fwd, bwd = C.byref(g.fwd.c), C.byref(g.bwd.c)
    q, k, v, sk, gr, code, sc = t["q"], t["k"], t["v"], t["skip"], t["g"], _code(dtype), t["scale"]
    out, m, s = Guarded(n_in, hd, dtype), _stats(n_in, H), _stats(n_in, H)
    _call("pg_tconv_aggregate", fwd, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
          sk.data_ptr(), sk.stride(0), H, D, code, sc, G.keep.data_ptr(), n_in, out.t.data_ptr(), out.t.stride(0),
          m.t.data_ptr(), s.t.data_ptr(), _scratch(g.fwd, H, D).data_ptr())
    dq, gc, delta = Guarded(n_in, hd, dtype), Guarded(n_in, hd, dtype), _stats(n_in, H)
    _call("pg_tconv_bwd_dst", fwd, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
          gr.data_ptr(), gr.stride(0), H, D, code, sc, m.t.data_ptr(), s.t.data_ptr(), G.keep.data_ptr(), n_in,
          dq.t.data_ptr(), dq.t.stride(0), gc.t.data_ptr(), gc.t.stride(0), delta.t.data_ptr(),
          _scratch(g.fwd, H, D).data_ptr())
    dk, dv = Guarded(n_all, hd, dtype), Guarded(n_all, hd, dtype)
    _call("pg_tconv_bwd_src", bwd, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
          gr.data_ptr(), gr.stride(0), H, D, code, sc, m.t.data_ptr(), s.t.data_ptr(), delta.t.data_ptr(),
          G.keep.data_ptr(), n_in, dk.t.data_ptr(), dk.t.stride(0), dv.t.data_ptr(), dv.t.stride(0),
          _scratch(g.bwd, H, D).data_ptr())
    return dict(out=out, m=m, s=s, dq=dq, gc=gc, delta=delta, dk=dk, dv=dv)


RUN = {"gat": run_gat, "gatv2": run_gatv2, "transformer": run_tconv}


# ============================================== inputs =============================================================
REGIMES = ["normal", "large", "spread", "last", "ties"]


def make_inputs(fam, G, H, D, dtype, regime, seed):
    """The regime is planted through el / er (GAT), the magnitudes of zs (GATv2, with a positive attn of unit sum
    per head outside "normal") and of q / k (transformer):
      normal  N(0, 1) scores;
      large   scores around 100 (exp without the max subtraction overflows fp32);
      spread  scores spread over about 200 within rows (most weights underflow to 0);
      last    N(0, 1) scores and a score of about 30 for each row's last entry (its peak source): the row maximum
              arrives in the last batch of the last segment;
      ties    every source either "hi" or "lo", all hi sources the same score bits for a destination and the lo ones
              more than 104 lower (weights exactly 1 and exactly 0)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    n_in, n_all, hd = G.num_in, G.num_all, H * D
    N = lambda *shape: torch.randn(*shape, generator=gen, device=DEV)
    U = lambda lo, hi, *shape: lo + (hi - lo) * torch.rand(*shape, generator=gen, device=DEV)
    hi = torch.rand(n_all, generator=gen, device=DEV) < 0.5
    peaks = torch.tensor(sorted(G.peak_of or {}), dtype=torch.long, device=DEV)
    peak_dst = torch.tensor([G.peak_of[int(p)] for p in peaks.tolist()], dtype=torch.long, device=DEV)

    def rows(n, data, poison=True):
        t = padded(n, hd, dtype, data=data.reshape(n, hd).to(dtype))
        if poison:
            t[G.bad] = NAN
        return t

    t = {"g": rows(n_in, N(n_in, hd), False), "hi": hi}
    if fam == "gat":
        el, er = N(n_all, H), N(n_in, H)
        if regime == "large":
            el = 100 + 3 * el
        elif regime == "spread":
            el = U(-60, 200, n_all, H)
        elif regime == "last":
            el[peaks] = 30 + N(peaks.numel(), H)
        elif regime == "ties":
            el = torch.where(hi[:, None], 100.0, -100.0).expand(n_all, H).contiguous()
        el[G.bad] = NAN
        t.update(z=rows(n_all, N(n_all, hd)), el=el.contiguous(), er=er.contiguous(), bias=0.1 * N(hd),
                 al=N(hd) / math.sqrt(D), ar=N(hd) / math.sqrt(D))
    elif fam == "gatv2":
        if regime == "normal":
            attn = N(H, D) / math.sqrt(D)
        else:
            attn = U(0.5, 1.5, H, D)
            attn = attn / attn.sum(1, keepdim=True)
        zs = N(n_all, H, D)
        if regime == "large":
            zs = 100 + 3 * N(n_all, H, 1) + 0.1 * zs
        elif regime == "spread":
            zs = U(-60, 200, n_all, H, 1) + zs
        elif regime == "last":
            zs[peaks] = 30 + 0.1 * N(peaks.numel(), H, D)
        elif regime == "ties":
            eta = N(2, H, D)
            zs = torch.where(hi[:, None, None], 100 + eta[0], -100 + eta[1])
        t.update(zs=rows(n_all, zs), zd=rows(n_in, N(n_in, hd), False), attn=attn.reshape(-1).contiguous())
    else:
        scale = float(np.float32(1 / math.sqrt(D)))
        q, k = N(n_in, H, D), N(n_all, H, D)
        if regime in ("large", "spread"):
            q = 1 + 0.1 * q
            base = 100 + 3 * N(n_all, H, 1) if regime == "large" else U(-60, 200, n_all, H, 1)
            k = base / math.sqrt(D) * (1 + 0.01 * k)
        elif regime == "last":
            qv = q[peak_dst]
            k[peaks] = qv * (30 * math.sqrt(D) / (qv * qv).sum(-1, keepdim=True))
        elif regime == "ties":
            q = 0.5 + 0.5 * q.abs()
            c = 120 / math.sqrt(D)
            k = torch.where(hi[:, None, None], c, -c).expand(n_all, H, D)
        t.update(q=rows(n_in, q, False), k=rows(n_all, k), v=rows(n_all, N(n_all, hd)), skip=rows(n_in, N(n_in, hd), False),
                 scale=scale)
    return t


# ============================================== references =========================================================
def _blocks(n, width):
    step = max(1, (1 << 23) // max(width, 1))
    for i in range(0, n, step):
        yield slice(i, min(n, i + step))


def _heads(x, idx, H, D):
    return x[idx].double().view(-1, H, D)


def _amax(n, idx, val, init=0.0):
    out = torch.full((n, val.shape[1]), init, dtype=torch.float64, device=DEV)
    return out.scatter_reduce_(0, idx[:, None].expand_as(val), val, "amax")


def scores(fam, G, t, H, D):
    """fp64 score of every kept edge [Ek, H] and a bound on the kernel's error in it:
      GAT          fp32 add el + er and LeakyReLU multiply: 2 roundings of |e|
      GATv2        t = zs + zd, LeakyReLU, NJ fmaf per lane, 5 tree adds: (NJ + 7) U24 sum |attn| |LeakyReLU(t)|
      transformer  NJ fmaf per lane, 5 tree adds, the multiply by scale: (NJ + 5) U24 scale sum |q| |k| + U24 |e|"""
    v, u, nj = G.kv, G.ku, nj_of(D)
    if fam == "gat":
        x = t["el"].double()[u] + t["er"].double()[v]
        e = torch.where(x > 0, x, SLOPE * x)
        return e, 2 * U24 * e.abs()
    e = torch.empty(v.numel(), H, dtype=torch.float64, device=DEV)
    dl = torch.empty_like(e)
    for sl in _blocks(v.numel(), H * D):
        if fam == "gatv2":
            tt = _heads(t["zs"], u[sl], H, D) + _heads(t["zd"], v[sl], H, D)
            lr = torch.where(tt > 0, tt, SLOPE * tt)
            at = t["attn"].double().view(1, H, D)
            e[sl] = (at * lr).sum(-1)
            dl[sl] = (nj + 7) * U24 * (at.abs() * lr.abs()).sum(-1)
        else:
            qk = _heads(t["q"], v[sl], H, D) * _heads(t["k"], u[sl], H, D)
            e[sl] = t["scale"] * qk.sum(-1)
            dl[sl] = (nj + 5) * U24 * t["scale"] * qk.abs().sum(-1) + U24 * e[sl].abs()
    return e, dl


def fwd_c(G, e, dl, M, fam, D):
    """c of the forward per (row, head), relative to mag = sum_u a_uv |z_u| + |bias or skip|.
    The weight of an edge carries a relative error eps_v: its score's error (dl), the rounding of e - mn (U24 |e - mn|
    <= U24 W, W the row's score range) and of every later rescale argument m - mn (these telescope to at most U24 W),
    the merge arguments of fwd_merge (U24 W more), and per batch or merged segment an expf (2 ulp = 4 U24), its
    multiplies and adds (2 U24):  eps_v = max dl + 3 U24 W + 6 U24 (batches + segments + 1), batches = ceil(n / E).
    Normalising by s doubles it; s and acc add n roundings each, the fix-up 2 per segment, then the division and the
    bias add:  c = 2 eps_v + (2 n + 2 segments + 10) U24."""
    n, seg = G.n_dst, G.seg_dst
    W = _amax(G.num_in, G.kv, M[G.kv] - e)
    eps = _amax(G.num_in, G.kv, dl) + 3 * U24 * W + 6 * U24 * (torch.ceil(n / edges_per_step(fam, nj_of(D))) + seg + 1)
    return 2 * eps + (2 * n + 2 * seg + 10) * U24, eps


def fwd_ref(G, e, vals, H, D):
    """softmax-aggregate of vals over the kept edges: (out, mag, M, S), fp64 [N_in, H, D] / [N_in, H]."""
    v, u, n_in = G.kv, G.ku, G.num_in
    M = _amax(n_in, v, e, -math.inf)
    p = torch.exp(e - M[v])
    S = torch.zeros(n_in, H, dtype=torch.float64, device=DEV).index_add_(0, v, p)
    a = p / S[v]
    out = torch.zeros(n_in, H, D, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(out)
    for sl in _blocks(v.numel(), H * D):
        z = _heads(vals, u[sl], H, D)
        out.index_add_(0, v[sl], a[sl, :, None] * z)
        mag.index_add_(0, v[sl], a[sl, :, None] * z.abs())
    return out, mag, M, S


def weights(G, e, dl, m, s):
    """Backward weights w = exp(e - m) / s from the kernel's statistics, and their relative error per edge: the
    score's, the rounding of e - m, expf (4 U24) and the division."""
    v = G.kv
    mv, sv = m.double()[v], s.double()[v]
    w = torch.where(sv > 0, torch.exp(e - mv) / sv, torch.zeros((), dtype=torch.float64, device=DEV))
    return w, dl + U24 * (e - mv).abs() + 5 * U24


def bwd_c(eps_row, n, seg, D, per_edge=1):
    """c of a backward sum over a row's edges, relative to its mag (the same sum over the absolute value of every
    factor): the weight's relative error eps, a D-wide dot of NJ fmaf and 5 tree adds, one rounding per edge and
    accumulator (`per_edge` accumulations of the same output), the segments' fix-up adds, and at most 6 roundings in
    the final combination (der = A - D B, the attn / scale multiplies, the subtraction of D_v):
    c = eps + (NJ + per_edge (n + segments) + 12) U24."""
    return eps_row + (nj_of(D) + per_edge * (n + seg) + 12) * U24


UNDER = 2.0 ** -146     # a few roundings in fp32's subnormal range (its smallest subnormal is 2^-149)


def within(got, ref, mag, c, bf16_out, what, floor):
    """assert_within plus an absolute floor per row: a weight that underflows (expf of a score more than about 104
    below the maximum) is off by up to UNDER in absolute terms, not relatively -- fp64 keeps 1e-52 where fp32 has 0 --
    and so is every product it enters.  floor = UNDER * (terms + 4) * (the largest term a weight multiplies)."""
    assert_within(got, ref, mag + floor / c, c, bf16_out, what)


def _hd(x, H, D):
    """[n, H] -> [n, H * D] (per head, repeated over its columns)."""
    return x[:, :, None].expand(-1, H, D).reshape(x.shape[0], H * D)


def _flat(x):
    return x.reshape(x.shape[0], -1)


# ============================================== the checks =========================================================
def check_family(fam, G, H, D, dtype, regime, seed=1):
    t = make_inputs(fam, G, H, D, dtype, regime, seed)
    res = RUN[fam](G, t, H, D, dtype)
    again = RUN[fam](G, t, H, D, dtype)
    for name, o in res.items():
        o.check(exact=True)
        assert torch.equal(_bits(o.t), _bits(again[name].t)), f"{name}: two launches differ"
        x = o.t.float()
        ok = torch.isfinite(x) | (x == -math.inf) if name == "m" else torch.isfinite(x)     # m = -inf: empty softmax
        assert bool(ok.all()), f"{name}: NaN or an unwritten element at {(~ok).nonzero()[0].tolist()}"
    bf16 = dtype == torch.bfloat16
    n_in, n_all, hd = G.num_in, G.num_all, H * D
    e, dl = scores(fam, G, t, H, D)
    vals = t["z"] if fam == "gat" else t["zs"] if fam == "gatv2" else t["v"]
    out_r, mag, M, S = fwd_ref(G, e, vals, H, D)
    if fam == "gat":
        add = t["bias"].double().view(1, H, D).expand(n_in, H, D)
    elif fam == "gatv2":
        add = torch.zeros(n_in, H, D, dtype=torch.float64, device=DEV)
    else:
        add = t["skip"].double().view(n_in, H, D)
    out_r, mag = _flat(out_r + add), _flat(mag + add.abs())
    c_out, eps = fwd_c(G, e, dl, M, fam, D)
    # the largest term a weight multiplies: a D-wide dot of two inputs or passed-on results times a third, plus one more
    big = max([1.0] + [float(x[torch.isfinite(x)].abs().max()) for x in t.values()
                       if torch.is_tensor(x) and x.is_floating_point()]
              + [float(res[k].t.abs().max()) for k in ("dv", "der", "delta") if k in res])
    T = (D + 2) * big ** 3
    fd = UNDER * (G.n_dst + G.seg_dst + 4) * T
    fs = UNDER * (G.n_src + G.seg_src + 4) * T
    m, s, out = res["m"].t, res["s"].t, res["out"].t
    none = S == 0                                                   # rows (heads) without a kept source
    assert bool(none.any()) and bool((~none).any())
    # exact cases: no kept source -> m = -inf, s = 0, out = bias / 0 / skip rounded once
    assert bool((m[none] == -math.inf).all()) and bool((s[none] == 0).all()), "statistics of an empty softmax"
    want = (add.float().reshape(n_in, hd)).to(dtype)
    rows0 = none.all(1)
    assert torch.equal(_bits(out[rows0]), _bits(want[rows0])), "output of a row without a kept source"
    # m: GAT's is the fp32 maximum of the fp32 scores bit for bit (one IEEE add, one multiply)
    if fam == "gat":
        x32 = t["el"][G.ku] + t["er"][G.kv]
        e32 = torch.where(x32 > 0, x32, x32 * torch.tensor(SLOPE, dtype=torch.float32, device=DEV))
        m32 = torch.full((n_in, H), -math.inf, device=DEV).scatter_reduce_(0, G.kv[:, None].expand_as(e32), e32, "amax")
        assert torch.equal(m, m32), "GAT m is not the fp32 maximum of the fp32 scores"
    else:
        mx = _amax(n_in, G.kv, dl)
        bad = ~none & ~((m.double() - M).abs() <= mx)
        assert not bool(bad.any()), f"m outside its bound at {bad.nonzero()[0].tolist()}"
    S_k = torch.zeros_like(S).index_add_(0, G.kv, torch.exp(e - m.double()[G.kv]))
    nb = torch.ceil(G.n_dst / edges_per_step(fam, nj_of(D)))
    c_s = eps + (G.n_dst + nb + 6) * U24
    assert_within(torch.where(none, 0.0, s), torch.where(none, 0.0, S_k), S_k, c_s, False, f"{fam} s")
    within(out, out_r, mag, _hd(c_out, H, D), bf16, f"{fam} out", fd)
    if regime == "ties":
        check_ties(fam, G, t, H, D, dtype, res, add)
    # ---- backward, teacher-forced with the kernel's m, s (and dv / der / delta below)
    w, ew = weights(G, e, dl, m, s)
    eps_d, eps_s = _amax(n_in, G.kv, ew), _amax(n_all, G.ku, ew)
    cd = lambda k=1: bwd_c(eps_d, G.n_dst, G.seg_dst, D, k)
    cs = lambda k=1: bwd_c(eps_s, G.n_src, G.seg_src, D, k)
    BWD[fam](G, t, H, D, dtype, res, w, cd, cs, none, fd, fs)


def _zero_rows(x, rows, what):
    assert bool((x[rows] == 0).all()), f"{what}: not exactly 0"


def bwd_gat(G, t, H, D, dtype, res, w, cd, cs, none, fd, fs):
    bf16, n_in, n_all = dtype == torch.bfloat16, G.num_in, G.num_all
    v, u = G.kv, G.ku
    x = t["el"].double()[u] + t["er"].double()[v]
    sl = torch.where(x > 0, 1.0, SLOPE)
    dv_k, der_k = res["dv"].t.double(), res["der"].t.double()
    z = lambda A, n: torch.zeros(n, *A, dtype=torch.float64, device=DEV)
    Dv, magD, A, magA, B = z((H,), n_in), z((H,), n_in), z((H,), n_in), z((H,), n_in), z((H,), n_in)
    dl_r, magdl = z((H,), n_all), z((H,), n_all)
    acc, macc = z((H, D), n_all), z((H, D), n_all)
    for b in _blocks(v.numel(), H * D):
        gv, zu = _heads(t["g"], v[b], H, D), _heads(t["z"], u[b], H, D)
        dot, dab = (gv * zu).sum(-1), (gv * zu).abs().sum(-1)
        wb, sb = w[b], sl[b]
        Dv.index_add_(0, v[b], wb * dot)
        magD.index_add_(0, v[b], wb * dab)
        A.index_add_(0, v[b], wb * dot * sb)
        magA.index_add_(0, v[b], wb * dab * sb)
        B.index_add_(0, v[b], wb * sb)
        dl_r.index_add_(0, u[b], wb * (dot - dv_k[v[b]]) * sb)
        magdl.index_add_(0, u[b], wb * (dab + dv_k[v[b]].abs()) * sb)
        acc.index_add_(0, u[b], wb[:, :, None] * gv)
        macc.index_add_(0, u[b], wb[:, :, None] * gv.abs())
    within(res["dv"].t, Dv, magD, cd(), False, "gat bwd_dst dv", fd)
    within(res["der"].t, A - Dv * B, magA + magD * B, cd(), False, "gat bwd_dst der", fd)
    _zero_rows(res["dv"].t, none, "gat dv of an empty softmax")
    _zero_rows(res["der"].t, none, "gat der of an empty softmax")
    within(res["del_"].t, dl_r, magdl, cs(), False, "gat bwd_src del", fs)
    al, ar = t["al"].double().view(1, H, D), t["ar"].double().view(1, H, D)
    derp = torch.zeros(n_all, H, dtype=torch.float64, device=DEV)
    derp[:n_in] = der_k
    ref = acc + dl_r[:, :, None] * al + derp[:, :, None] * ar
    mag = macc + magdl[:, :, None] * al.abs() + (derp[:, :, None] * ar).abs()
    within(res["dz"].t, _flat(ref), _flat(mag), _hd(cs() + 3 * U24, H, D), bf16, "gat bwd_src dz", fs)
    halo0 = G.bad.clone()
    _zero_rows(res["dz"].t, halo0, "gat dz of an unkept or unreferenced halo row")
    _zero_rows(res["del_"].t, halo0, "gat del of an unkept or unreferenced halo row")
    # nobody's source: dz = fmaf(der, attn_r, +0) (one rounding; a -0 product becomes +0), rounded to the dtype
    want = (res["der"].t[NOSRC][:, None] * t["ar"].view(H, D) + 0.0).reshape(1, -1).to(dtype) \
        if G.num_in > NOSRC and int(G.g.bwd.indptr[NOSRC + 1] - G.g.bwd.indptr[NOSRC]) == 0 else None
    if want is not None:
        assert torch.equal(_bits(res["dz"].t[NOSRC:NOSRC + 1]), _bits(want)), "gat dz of a row nobody reads"


def bwd_gatv2(G, t, H, D, dtype, res, w, cd, cs, none, fd, fs):
    bf16, n_in, n_all = dtype == torch.bfloat16, G.num_in, G.num_all
    v, u = G.kv, G.ku
    dv_k = res["dv"].t.double()
    at = t["attn"].double().view(1, H, D)
    zH = lambda n: torch.zeros(n, H, dtype=torch.float64, device=DEV)
    zHD = lambda n: torch.zeros(n, H, D, dtype=torch.float64, device=DEV)
    Dv, magD = zH(n_in), zH(n_in)
    A, magA, B, Cc, magC, Q, Qa = (zHD(n_in) for _ in range(7))
    dzs, mdzs = zHD(n_all), zHD(n_all)
    for b in _blocks(v.numel(), H * D):
        gv, zsu, zdv = _heads(t["g"], v[b], H, D), _heads(t["zs"], u[b], H, D), _heads(t["zd"], v[b], H, D)
        tt = zsu + zdv
        sl = torch.where(tt > 0, 1.0, SLOPE)
        lr = tt * sl
        dot, dab = (gv * zsu).sum(-1), (gv * zsu).abs().sum(-1)
        wb = w[b]
        wd, wa = (wb * dot)[:, :, None], (wb * dab)[:, :, None]
        Dv.index_add_(0, v[b], wb * dot)
        magD.index_add_(0, v[b], wb * dab)
        A.index_add_(0, v[b], wd * sl)
        magA.index_add_(0, v[b], wa * sl)
        B.index_add_(0, v[b], wb[:, :, None] * sl)
        Cc.index_add_(0, v[b], wd * lr)
        magC.index_add_(0, v[b], wa * lr.abs())
        Q.index_add_(0, v[b], wb[:, :, None] * lr)
        Qa.index_add_(0, v[b], wb[:, :, None] * lr.abs())
        de = (wb * (dot - dv_k[v[b]]))[:, :, None]
        dem = (wb * (dab + dv_k[v[b]].abs()))[:, :, None]
        dzs.index_add_(0, u[b], wb[:, :, None] * gv + de * sl * at)
        mdzs.index_add_(0, u[b], wb[:, :, None] * gv.abs() + dem * sl * at.abs())
    within(res["dv"].t, Dv, magD, cd(), False, "gatv2 bwd_dst D_v", fd)
    c = _hd(cd(), H, D)
    Dh = Dv[:, :, None]
    within(res["dzd"].t, _flat(at * (A - Dh * B)), _flat(at.abs() * (magA + magD[:, :, None] * B)), c, bf16,
           "gatv2 bwd_dst dzd", fd)
    within(res["pattn"].t, _flat(Cc - Dh * Q), _flat(magC + magD[:, :, None] * Qa), c, False,
           "gatv2 bwd_dst pattn", fd)
    rows0 = none.all(1)
    for name in ("dv", "dzd", "pattn"):
        _zero_rows(res[name].t, rows0, f"gatv2 {name} of an empty softmax")
    within(res["dzs"].t, _flat(dzs), _flat(mdzs), _hd(cs(2), H, D), bf16, "gatv2 bwd_src dzs", fs)
    nosrc = (G.n_src[:, 0] == 0) | G.bad
    _zero_rows(res["dzs"].t, nosrc, "gatv2 dzs of an unkept, unreferenced or source-less row")


def bwd_tconv(G, t, H, D, dtype, res, w, cd, cs, none, fd, fs):
    bf16, n_in, n_all, sc = dtype == torch.bfloat16, G.num_in, G.num_all, t["scale"]
    v, u = G.kv, G.ku
    dl_k = res["delta"].t.double()
    zH = lambda n: torch.zeros(n, H, dtype=torch.float64, device=DEV)
    zHD = lambda n: torch.zeros(n, H, D, dtype=torch.float64, device=DEV)
    de, mde = zH(n_in), zH(n_in)
    A, magA, B, Ba = (zHD(n_in) for _ in range(4))
    dk, mdk, dvv, mdv = (zHD(n_all) for _ in range(4))
    for b in _blocks(v.numel(), H * D):
        gv, qv = _heads(t["g"], v[b], H, D), _heads(t["q"], v[b], H, D)
        ku, vu = _heads(t["k"], u[b], H, D), _heads(t["v"], u[b], H, D)
        gd, ga = (gv * vu).sum(-1), (gv * vu).abs().sum(-1)
        wb = w[b]
        de.index_add_(0, v[b], wb * gd)
        mde.index_add_(0, v[b], wb * ga)
        A.index_add_(0, v[b], (wb * gd)[:, :, None] * ku)
        magA.index_add_(0, v[b], (wb * ga)[:, :, None] * ku.abs())
        B.index_add_(0, v[b], wb[:, :, None] * ku)
        Ba.index_add_(0, v[b], wb[:, :, None] * ku.abs())
        cuv = (wb * (gd - dl_k[v[b]]))[:, :, None]
        cma = (wb * (ga + dl_k[v[b]].abs()))[:, :, None]
        dvv.index_add_(0, u[b], wb[:, :, None] * gv)
        mdv.index_add_(0, u[b], wb[:, :, None] * gv.abs())
        dk.index_add_(0, u[b], sc * cuv * qv)
        mdk.index_add_(0, u[b], sc * cma * qv.abs())
    within(res["delta"].t, de, mde, cd(), False, "transformer bwd_dst delta", fd)
    within(res["dq"].t, _flat(sc * (A - de[:, :, None] * B)), _flat(sc * (magA + mde[:, :, None] * Ba)),
           _hd(cd(), H, D), bf16, "transformer bwd_dst dq", fd)
    assert torch.equal(_bits(res["gc"].t), _bits(t["g"])), "transformer: the copy of g differs from g"
    rows0 = none.all(1)
    for name in ("delta", "dq"):
        _zero_rows(res[name].t, rows0, f"transformer {name} of an empty softmax")
    c = _hd(cs(), H, D)
    within(res["dv"].t, _flat(dvv), _flat(mdv), c, bf16, "transformer bwd_src dv", fs)
    within(res["dk"].t, _flat(dk), _flat(mdk), c, bf16, "transformer bwd_src dk", fs)
    nosrc = (G.n_src[:, 0] == 0) | G.bad
    for name in ("dk", "dv"):
        _zero_rows(res[name].t, nosrc, f"transformer {name} of an unkept, unreferenced or source-less row")


BWD = {"gat": bwd_gat, "gatv2": bwd_gatv2, "transformer": bwd_tconv}


def check_ties(fam, G, t, H, D, dtype, res, add):
    """Regime "ties": every weight is exactly 1 (a source of the row's maximum class) or exactly 0, so on a row that
    is not split into segments s is the count of the tied sources and acc their fp32 sum in CSR order, one rounding
    per add: out = fl(fl(acc / s) + bias or skip) bit for bit.  A reciprocal multiply in place of the division, a
    dropped rescale or a reordered sum changes bits here that no bound can see."""
    n_in, hd = G.num_in, H * D
    hi_e = t["hi"][G.cols] & G.edge_kept
    any_hi = torch.zeros(n_in, dtype=torch.bool, device=DEV).index_put_((G.rows[hi_e],), torch.ones((), dtype=torch.bool, device=DEV))
    tied = G.edge_kept & (t["hi"][G.cols] == any_hi[G.rows])
    lens = (G.indptr[1:] - G.indptr[:-1])
    short = lens <= G.g.fwd.seg_len
    vals = t["z"] if fam == "gat" else t["zs"] if fam == "gatv2" else t["v"]
    acc = torch.zeros(n_in, hd, device=DEV)
    cnt = torch.zeros(n_in, device=DEV)
    for j in range(int(lens[short].max())):
        r = torch.nonzero(short & (lens > j))[:, 0]
        e = G.indptr[r] + j
        on = tied[e]
        r, e = r[on], e[on]
        acc[r] = acc[r] + vals[G.cols[e]].float()
        cnt[r] += 1
    rows = short & (cnt > 0)
    s = res["s"].t
    assert torch.equal(s[rows], cnt[rows, None].expand(-1, H)), "ties: s is not the count of tied sources"
    want = (acc / cnt[:, None] + add.float().reshape(n_in, hd)).to(dtype)
    got = res["out"].t
    bad = rows[:, None] & (_bits(got) != _bits(want))
    assert not bool(bad.any()), (f"ties: {int(bad.sum())} outputs differ from fl(fl(acc / s) + add), first "
                                 f"{bad.nonzero()[0].tolist()}")


# ============================================== the cases ==========================================================
WIDTHS = [(1, 8), (32, 1), (33, 3), (64, 8), (65, 3), (100, 1), (128, 8), (129, 3), (172, 1), (256, 8), (257, 3),
          (400, 3), (512, 1)]
FAMILIES = ["gat", "gatv2", "transformer"]
DTYPES = [torch.float32, torch.bfloat16]


def _dname(dtype):
    return "f32" if dtype == torch.float32 else "bf16"


def _inst(fam, d):
    """What a width reaches: NJ, the edges per step and the warp_sum_n instantiations of the passes."""
    nj = nj_of(d)
    if fam == "gat":
        return f"NJ={nj}"
    e = edges_per_step(fam, nj)
    return f"NJ={nj} E={e} (fwd warp_sum_n<{e}>, bwd warp_sum_n<{2 * e}>)"


def _cases():
    out = []
    for fam in FAMILIES:
        for dtype in DTYPES:
            for d, h in WIDTHS:
                out.append(pytest.param(fam, dtype, d, h, id=f"{fam}-{_dname(dtype)}-D{d}-H{h}: {_inst(fam, d)}"))
    return out


@pytest.mark.parametrize("seg_len", [32, 256], ids=lambda s: f"seg{s}")
@pytest.mark.parametrize("fam,dtype,d,heads", _cases())
def test_attention_widths(fam, dtype, d, heads, seg_len):
    """Every pass of every family at both edges of every NJ, N(0, 1) scores, on the structured graph."""
    check_family(fam, structured_graph(seg_len), heads, d, dtype, "normal", seed=d * 7 + heads)


@pytest.mark.parametrize("seg_len", [32, 256], ids=lambda s: f"seg{s}")
@pytest.mark.parametrize("regime", REGIMES[1:])
@pytest.mark.parametrize("fam,dtype,d,heads", [pytest.param(f, dt, d, h, id=f"{f}-{_dname(dt)}-D{d}-H{h}: {_inst(f, d)}")
                                               for f in FAMILIES for dt in DTYPES for d, h in ((100, 3), (257, 3))])
def test_attention_score_regimes(fam, dtype, d, heads, regime, seg_len):
    """The softmax's edge paths: scores of about 100 (max subtraction), a spread of 200 (weights that underflow to 0:
    the pt == 0 / at == 0 skips), the maximum in the last batch of the last segment (every rescale and merge factor
    below 1), and exact ties (weights exactly 0 and 1, checked bit for bit)."""
    check_family(fam, structured_graph(seg_len), heads, d, dtype, regime, seed=d + REGIMES.index(regime))


@pytest.mark.parametrize("dtype", DTYPES, ids=_dname)
@pytest.mark.parametrize("fam", FAMILIES)
def test_attention_past_the_first_wave(fam, dtype):
    """More CTAs than one wave holds at any occupancy, for both plans, at a narrow width."""
    check_family(fam, wide_graph(), 2, 33, dtype, "normal", seed=5)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dname)
@pytest.mark.parametrize("d,heads", [(1, 8), (33, 3), (129, 3), (257, 3), (512, 1)])
def test_gat_scores(d, heads, dtype):
    """pg_gat_scores: el over every row, er over the first n_er, against fp64: NJ fmaf per lane and 5 tree adds,
    c = (NJ + 6) U24 of sum |z| |attn|; NaN rows stay in their own row; two launches agree."""
    from pipegcn_b200 import _C
    G = structured_graph(256)
    t = make_inputs("gat", G, heads, d, dtype, "normal", seed=d)
    z, n_all, n_in = t["z"], G.num_all, G.num_in
    outs = []
    for _ in range(2):
        el, er = _stats(n_all, heads), _stats(n_in, heads)
        _call("pg_gat_scores", z.data_ptr(), z.stride(0), n_all, n_in, heads, d, _C.dtype_code(dtype),
              t["al"].data_ptr(), t["ar"].data_ptr(), el.t.data_ptr(), er.t.data_ptr())
        el.check(exact=True)
        er.check(exact=True)
        outs.append((el.t, er.t))
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(*outs))
    el, er = outs[0]
    zz = z.double().view(n_all, heads, d)
    good = ~G.bad
    for got, att, rows in ((el, t["al"], slice(None)), (er, t["ar"], slice(0, n_in))):
        a = att.double().view(1, heads, d)
        ref, mag = (zz[rows] * a).sum(-1), (zz[rows] * a).abs().sum(-1)
        g = good[rows]
        assert_within(got[g], ref[g], mag[g], (nj_of(d) + 6) * U24, False, "pg_gat_scores")
        assert bool(got[~g].isnan().all())


@pytest.mark.parametrize("hd,heads", [(1, 1), (31, 1), (33, 3), (99, 3), (4096, 8)], ids=lambda v: str(v))
@pytest.mark.parametrize("n_rows", ["1", "255", "256", "257", "2w+1", "300000"])
def test_gat_colsum(n_rows, hd, heads):
    """pg_gat_colsum with and without coef, fp32 and bf16, past the block cap (2 * SMs blocks, so that rows_per grows
    past 256).  Chain of one column: a row lane adds ceil(rows_per / 8) rows (one fmaf or add each), 8 row lanes are
    added in order, then n_blocks partials: c = (ceil(rows_per / 8) + 8 + n_blocks) U24 of sum |coef x|."""
    from pipegcn_b200 import _C
    n = {"2w+1": 2 * sm_count() * 256 + 1}.get(n_rows) or int(n_rows)
    nb = int(_C.lib.pg_gat_colsum_blocks(n))
    assert nb == max(1, min(-(-n // 256), 2 * sm_count()))
    rows_per = -(-n // nb)
    c = (-(-rows_per // 8) + 8 + nb) * U24
    gen = torch.Generator(device=DEV).manual_seed(n + hd)
    for dtype in DTYPES:
        x = padded(n, hd, dtype)
        x.copy_(torch.randn(n, hd, generator=gen, device=DEV).to(dtype))
        coef = torch.randn(n, heads, generator=gen, device=DEV)
        for cf in (None, coef):
            res = []
            for _ in range(2):
                out = Guarded(1, hd, torch.float32)
                partial = torch.full((nb * hd,), NAN, device=DEV)
                _call("pg_gat_colsum", x.data_ptr(), x.stride(0), n, heads, hd // heads, _C.dtype_code(dtype),
                      cf.data_ptr() if cf is not None else None, out.t.data_ptr(), partial.data_ptr())
                out.check(exact=True)
                res.append(out.t[0])
            assert torch.equal(_bits(res[0]), _bits(res[1])), "two launches differ"
            ref = torch.zeros(hd, dtype=torch.float64, device=DEV)
            mag = torch.zeros_like(ref)
            for b in _blocks(n, hd):
                xb = x[b].double()
                if cf is not None:
                    xb = xb * _hd(cf[b].double(), heads, hd // heads)
                ref += xb.sum(0)
                mag += xb.abs().sum(0)
            assert_within(res[0], ref, mag, c, False, f"colsum {_dname(dtype)} coef={cf is not None}")


def test_head_width_past_512_is_refused():
    """D = 513 is refused before launch by every GAT and GATv2 pass (the transformer's: test_transformer_gpu)."""
    from pipegcn_b200 import _C, ops
    G = structured_graph(256)
    g = G.g
    hd = 513
    zs = torch.zeros(g.num_all, hd, device=DEV)
    zd = torch.zeros(g.num_in, hd, device=DEV)
    st = torch.zeros(g.num_all, 1, device=DEV)
    a = torch.zeros(hd, device=DEV)
    calls = [lambda: ops.gat_scores(zs, a, a, 1, g.num_in),
             lambda: ops.gat_aggregate(g, zs, st, st, a, 1),
             lambda: ops.gat_bwd_dst(g, zs, zd, st, st, st, st, 1),
             lambda: ops.gat_bwd_src(g, zs, zd, st, st, st, st, st, st, a, a, 1),
             lambda: ops.gatv2_aggregate(g, zs, zd, a, 1),
             lambda: ops.gatv2_bwd_dst(g, zs, zd, zd, a, st, st, 1),
             lambda: ops.gatv2_bwd_src(g, zs, zd, zd, a, st, st, st, 1)]
    for f in calls:
        with pytest.raises(_C.PgError, match="513"):
            f()
