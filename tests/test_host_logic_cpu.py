"""Host-side logic that needs no GPU: the chunk plan of the aggregate kernels, the on-disk partition cache,
evaluation bookkeeping and result-file naming."""
import argparse

import pytest
import torch

from pipegcn_b200.graph import CsrPlan


def _emulate(plan: CsrPlan, x: torch.Tensor) -> torch.Tensor:
    """What the chunked kernels compute, chunk by chunk, from the plan tables alone (include/pipegcn_b200.h: pg_csr)."""
    out = torch.full((plan.n_rows, x.shape[1]), float("nan"), dtype=torch.float64)
    scratch = torch.zeros(max(plan.n_seg, 1), x.shape[1], dtype=torch.float64)
    pidx, prow = plan.pidx.long() & 0x7FFFFFFF, plan.prow.long()
    seen_kind0 = False
    for i, (e, n, item, kr) in enumerate(plan.chunks.tolist()):
        kind, nr = kr & 3, kr >> 2
        assert (i < plan.n_chunks_long) == (kind != 0)            # long rows / segments first, then the short-row chunks
        if kind == 0:
            seen_kind0 = True
            assert n * nr <= 32 and nr >= 1
            for r in range(nr):
                row = prow[item + r]
                assert torch.isnan(out[row]).all()
                out[row] = x[pidx[e + r * n: e + (r + 1) * n]].sum(0) if n else 0
        elif kind == 1:
            assert not seen_kind0 and n > 32
            row = prow[item]
            assert torch.isnan(out[row]).all()
            out[row] = x[pidx[e:e + n]].sum(0)
        else:
            assert 0 < n <= plan.seg_len
            scratch[item] = x[pidx[e:e + n]].sum(0)
    for li in range(plan.n_long):
        row = plan.long_row[li].item()
        assert torch.isnan(out[row]).all()
        out[row] = scratch[plan.long_seg_ptr[li]:plan.long_seg_ptr[li + 1]].sum(0)
    return out


@pytest.mark.parametrize("n_rows,max_deg,seg_len", [(50, 5, 512), (200, 40, 16), (1000, 70, 32), (37, 3, 512), (1, 9, 4),
                                                     (300, 200, 64)])
def test_chunk_plan_covers_every_row_once(n_rows, max_deg, seg_len):
    g = torch.Generator().manual_seed(n_rows)
    n_cols = 120
    deg = torch.randint(0, max_deg, (n_rows,), generator=g)
    if n_rows > 100:
        deg[::7] = 0
    indptr = torch.zeros(n_rows + 1, dtype=torch.int32)
    indptr[1:] = torch.cumsum(deg, 0)
    indices = torch.randint(0, n_cols, (int(indptr[-1]),), generator=g, dtype=torch.int32)
    plan = CsrPlan(indptr, indices, seg_len=seg_len)
    x = torch.randn(n_cols, 3, generator=g, dtype=torch.float64)
    ref = torch.zeros(n_rows, 3, dtype=torch.float64)
    ref.index_add_(0, torch.repeat_interleave(torch.arange(n_rows), deg), x[indices.long()])
    got = _emulate(plan, x)
    assert not torch.isnan(got).any()
    torch.testing.assert_close(got, ref)
    # hot flags (bit 31) mark sources referenced at least twice
    hot = (plan.pidx.long() >> 31) & 1
    refs = torch.bincount(indices.long(), minlength=n_cols)
    assert bool((refs[(plan.pidx.long() & 0x7FFFFFFF)[hot.bool()]] >= 2).all())


def test_partition_cache_roundtrip(tmp_path, monkeypatch):
    from pipegcn_b200.helper.utils import graph_partition, partition_dir
    from pipegcn_b200.synthetic import make_graph
    monkeypatch.setenv("PG_PARTITION_ROOT", str(tmp_path))
    g = make_graph(dict(n_nodes=400, n_edges=4000, n_feat=4, n_class=3, train_frac=0.5))
    args = argparse.Namespace(partition_method="metis", partition_obj="vol", n_partitions=3, dataset="synthetic:t",
                              graph_name="", inductive=False, partition_cache=True, skip_partition=True)
    with pytest.raises(FileNotFoundError):                       # --skip-partition without a cached partition
        graph_partition(g, args, 0)
    args.skip_partition = False
    part = graph_partition(g, args, 0)
    assert (tmp_path / partition_dir(args).split("/")[-1] / "part.pt").exists()
    assert part.unique().numel() == 3
    again = graph_partition(g, args, 1)                          # another rank / a later run reads the file
    assert torch.equal(part, again)
    args.skip_partition = True
    assert torch.equal(graph_partition(g, args, 0), part)
    g2 = make_graph(dict(n_nodes=401, n_edges=4000, n_feat=4, n_class=3, train_frac=0.5))
    with pytest.raises(ValueError):                              # the cache belongs to another graph
        graph_partition(g2, args, 0)
    args.partition_method = "random"                             # random is a seeded draw: never cached
    r1, r2 = graph_partition(g, args, 0), graph_partition(g, args, 1)
    assert torch.equal(r1, r2)


def test_evaluation_bookkeeping(tmp_path, monkeypatch):
    from pipegcn_b200.evaluate import BestModel, calc_acc, result_file
    monkeypatch.chdir(tmp_path)
    logits = torch.tensor([[2.0, 1.0], [0.0, 3.0], [1.0, 0.0], [0.0, 1.0]])
    assert calc_acc(logits, torch.tensor([0, 1, 1, 1])) == 0.75                 # train.py:11-17
    a = argparse.Namespace(dataset="reddit", n_partitions=4, enable_pipeline=True, grad_corr=True, feat_corr=True,
                           graph_name="g")
    assert result_file(a) == "results/reddit_n4_p1_grad_feat.txt"               # train.py:309-316
    a.feat_corr = False
    assert result_file(a) == "results/reddit_n4_p1_grad.txt"
    a.grad_corr, a.enable_pipeline = False, False
    assert result_file(a) == "results/reddit_n4_p0.txt"
    best = BestModel()
    m = torch.nn.Linear(3, 2)
    best.offer(0.4, m)
    w = m.weight.detach().clone()
    with torch.no_grad():
        m.weight.add_(1.0)
    best.offer(0.3, m)                                                          # worse: the earlier state stays
    assert best.acc == 0.4 and torch.equal(best.state["weight"], w)
    path = best.save(a)
    assert path == "model/g_final.pth.tar" and set(torch.load(path)) == {"weight", "bias"}


def test_dropout_mask_function_statistics():
    """tools/dropout_hash_quality.py restates drop_base / drop_bits of csrc/common.cuh in numpy: the constants must be
    the kernel's, and the masks must have the right keep rate and no in-vector / neighbour / epoch correlation."""
    import importlib.util
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("dropout_hash_quality", os.path.join(root, "tools", "dropout_hash_quality.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    src = open(os.path.join(root, "pipegcn_b200", "csrc", "common.cuh")).read()
    kmul = re.search(r"kMul\[4\] = \{([^}]*)\}", src).group(1)
    assert [int(t.strip().rstrip("U"), 16) for t in kmul.split(",")] == mod.MUL
    for const in ("0x7feb352dU", "0x846ca68bU", "0x632be5abU", "0x9e3779b9U"):
        assert const in src
    mod.main(1 << 19)


def test_multi_value_warp_reduction_network():
    """csrc/rowops.cu: warp_sum_multi<K> folds K per-lane values with a halving butterfly (a lane keeps the half of the
    values its own lane bit selects and ships the other half), then broadcasts: every lane must end up with all K
    totals.  Restated on 32 numpy "lanes" with integer values (exact)."""
    import numpy as np
    rng = np.random.default_rng(0)
    lanes = np.arange(32)

    def shfl_xor(v, o):
        return v[lanes ^ o]

    for K in (1, 2, 4):
        v = [rng.integers(-1000, 1000, size=32) for _ in range(K)]
        want = [int(x.sum()) for x in v]
        if K == 1:
            t = v[0].copy()
            for o in (16, 8, 4, 2, 1):
                t = t + shfl_xor(t, o)
            got = [t]
        elif K == 2:
            up = (lanes & 16) != 0
            keep, send = np.where(up, v[1], v[0]), np.where(up, v[0], v[1])
            t = keep + shfl_xor(send, 16)
            for o in (8, 4, 2, 1):
                t = t + shfl_xor(t, o)
            got = [np.full(32, t[0]), np.full(32, t[16])]
        else:
            up = (lanes & 16) != 0
            k0, k1 = np.where(up, v[2], v[0]), np.where(up, v[3], v[1])
            s0, s1 = np.where(up, v[0], v[2]), np.where(up, v[1], v[3])
            a0, a1 = k0 + shfl_xor(s0, 16), k1 + shfl_xor(s1, 16)
            up2 = (lanes & 8) != 0
            keep, send = np.where(up2, a1, a0), np.where(up2, a0, a1)
            t = keep + shfl_xor(send, 8)
            for o in (4, 2, 1):
                t = t + shfl_xor(t, o)
            got = [np.full(32, t[src]) for src in (0, 8, 16, 24)]
        for k in range(K):
            assert np.all(got[k] == want[k]), (K, k)
