"""Boundary-node sampling (`--sampling-rate`) without a GPU: the parser flag, the refused combinations, and the
statistics of the keep hash (a host port of csrc/common.cuh: bns_key / bns_keep, pipegcn_b200.ops.bns_keep_host)."""
import argparse

import numpy as np
import pytest


def test_flag_absent_keeps_todays_namespace():
    from pipegcn_b200.helper.parser import create_parser
    base = vars(create_parser([]))
    assert "sampling_rate" not in base
    with_flag = vars(create_parser(["--sampling-rate", "0.25"]))
    assert with_flag.pop("sampling_rate") == 0.25
    assert with_flag == base
    assert create_parser(["--sampling_rate", "1"]).sampling_rate == 1.0


@pytest.mark.parametrize("bad", ["0", "-0.5", "1.5", "nan", "inf", "half"])
def test_invalid_rates_are_refused(bad):
    from pipegcn_b200.helper.parser import create_parser
    with pytest.raises(SystemExit):
        create_parser(["--sampling-rate", bad])


@pytest.mark.parametrize("flag", ["enable_pipeline", "feat_corr", "grad_corr"])
def test_unsupported_combinations_raise_before_allocation(flag):
    """RankEngine, Buffer.init_buffer and init_processes refuse before touching the layout, the world or a device."""
    from pipegcn_b200 import train
    from pipegcn_b200.helper.feature_buffer import Buffer
    args = argparse.Namespace(enable_pipeline=False, feat_corr=False, grad_corr=False, sampling_rate=0.5)
    setattr(args, flag, True)
    name = "--" + flag.replace("_", "-")
    with pytest.raises(NotImplementedError, match=name):
        train.RankEngine(None, args, None)
    with pytest.raises(NotImplementedError, match=name):
        train.init_processes(0, 2, args)
    with pytest.raises(NotImplementedError, match=name):
        Buffer().init_buffer(4, 6, None, None, [8], pipeline=args.enable_pipeline, corr_feat=args.feat_corr,
                             corr_grad=args.grad_corr, sampling_rate=0.5)
    with pytest.raises(ValueError):
        Buffer().init_buffer(4, 6, None, None, [8], sampling_rate=0.0)
    # p = 1 is today's path: every combination stays allowed
    args.sampling_rate = 1.0
    from pipegcn_b200.helper.feature_buffer import check_sampling
    assert check_sampling(1.0, True, True, True) == 1.0


def _keep(seed, t, r, rows, p):
    from pipegcn_b200 import ops
    return ops.bns_keep_host(seed, t, r, rows, ops.bns_threshold(p))


@pytest.mark.parametrize("p", [0.5, 0.1, 0.3, 0.9])
def test_keep_hash_statistics(p):
    """Keep rate within 4 sigma of p per (epoch, rank); the samples of different epochs, of different ranks and of
    neighbouring rows are uncorrelated (|z| < 4 for the correlation of the keep indicators)."""
    from pipegcn_b200 import ops
    seed = ops.bns_seed(0)
    n = 200_000
    rows = np.arange(1000, 1000 + n, dtype=np.int64)
    sigma = np.sqrt(p * (1 - p) / n)
    keeps = {}
    for t in range(4):
        for r in range(3):
            k = _keep(seed, t, r, rows, p)
            assert abs(k.mean() - p) < 4 * sigma, (t, r, k.mean())
            keeps[(t, r)] = k.astype(np.float64)

    def z(a, b):
        c = np.corrcoef(a, b)[0, 1]
        return c * np.sqrt(len(a))

    assert abs(z(keeps[(0, 0)], keeps[(1, 0)])) < 4          # epoch t vs t + 1, same rank
    assert abs(z(keeps[(0, 0)], keeps[(3, 0)])) < 4
    assert abs(z(keeps[(2, 0)], keeps[(2, 1)])) < 4          # same epoch, different ranks
    assert abs(z(keeps[(2, 1)], keeps[(2, 2)])) < 4
    a = keeps[(1, 2)]
    assert abs(z(a[:-1], a[1:])) < 4                         # neighbouring rows


def test_keep_hash_depends_on_the_seed_and_threshold_is_monotone():
    from pipegcn_b200 import ops
    rows = np.arange(50_000)
    a = _keep(ops.bns_seed(0), 0, 0, rows, 0.5)
    b = _keep(ops.bns_seed(1), 0, 0, rows, 0.5)
    assert 0.4 < (a == b).mean() < 0.6
    small, large = _keep(ops.bns_seed(0), 5, 1, rows, 0.1), _keep(ops.bns_seed(0), 5, 1, rows, 0.5)
    assert not (small & ~large).any()                        # a row kept at 0.1 is kept at 0.5
    assert ops.bns_threshold(0.5) == 2 ** 31
    with pytest.raises(ValueError):
        ops.bns_threshold(1.0)
