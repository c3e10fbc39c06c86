"""Quantised halo messages (`--halo-bits`) without a GPU: the parser flag, the refused combination, and the host port
of the quantiser (row format, stochastic rounding, special rows, 4-bit packing, byte counts)."""
import numpy as np
import pytest

from pipegcn_b200 import ops
from pipegcn_b200.helper.parser import create_parser


# ------------------------------------------------------------------------------------------------ parser
@pytest.mark.parametrize("flag", ["--halo-bits", "--halo_bits"])
@pytest.mark.parametrize("bits", [8, 4])
def test_parser_accepts_8_and_4(flag, bits):
    assert create_parser([flag, str(bits)]).halo_bits == bits


@pytest.mark.parametrize("bad", ["3", "16", "x"])
def test_parser_refuses_other_widths(bad):
    with pytest.raises(SystemExit):
        create_parser(["--halo-bits", bad])


def test_namespace_without_flag_is_unchanged():
    assert not hasattr(create_parser([]), "halo_bits")
    a = vars(create_parser(["--halo-bits", "8"]))
    a.pop("halo_bits")
    assert a == vars(create_parser([]))


# ------------------------------------------------------------------------------------------------ refusals
def test_sampling_combination_refused_before_allocation():
    from pipegcn_b200.helper.feature_buffer import Buffer, check_halo_bits
    assert check_halo_bits(None, 0.5) is None
    assert check_halo_bits(8, 1.0) == 8
    with pytest.raises(ValueError):
        check_halo_bits(6)
    with pytest.raises(NotImplementedError):
        check_halo_bits(4, 0.5)
    # Buffer.init_buffer raises before it touches the world or the device
    with pytest.raises(NotImplementedError):
        Buffer(world=None).init_buffer(1, 1, [], [], [4, 4], sampling_rate=0.5, halo_bits=8)


def test_trainer_refuses_sampling_with_quantisation():
    import argparse
    from pipegcn_b200.train import RankEngine, init_processes
    a = argparse.Namespace(sampling_rate=0.5, halo_bits=8, enable_pipeline=False, feat_corr=False, grad_corr=False,
                           model="graphsage", use_pp=False)
    with pytest.raises(NotImplementedError):
        RankEngine(None, a, None)
    with pytest.raises(NotImplementedError):
        init_processes(0, 1, a)


# ------------------------------------------------------------------------------------------------ host port
def _rows(n, d, seed=0):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32) * 3


@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("d", [5, 64, 256])
def test_decoded_within_one_step(bits, d):
    x = _rows(50, d)
    codes, lo, scale = ops.quantise_host(x, bits, 7, 1, 0, 3, 2, 100)
    assert codes.shape == (50, ops.quant_row_bytes(d, bits)) and codes.dtype == np.uint8
    np.testing.assert_array_equal(lo, x.min(1))
    y = ops.dequantise_host(codes, lo, scale, bits, d)
    assert (np.abs(y - x) <= scale[:, None] * (1 + 1e-5)).all()
    assert (y >= lo[:, None]).all()


@pytest.mark.parametrize("bits", [8, 4])
def test_rounding_is_unbiased(bits):
    x = _rows(4, 16, seed=1)
    steps = 4000
    acc = np.zeros_like(x, dtype=np.float64)
    for t in range(steps):
        c, lo, s = ops.quantise_host(x, bits, 11, 2, 1, t, 0, 0)
        acc += ops.dequantise_host(c, lo, s, bits, 16)
    mean = acc / steps
    _, _, s = ops.quantise_host(x, bits, 11, 2, 1, 0, 0, 0)
    sigma = s[:, None] / 2 / np.sqrt(steps)          # a rounding error lies in one step: std <= scale / 2
    assert (np.abs(mean - x) <= 5 * sigma + 1e-6).all()


def test_noise_independent_across_steps_rows_ranks():
    base = ops.quant_noise_host(5, 1, 0, 10, 2, np.arange(64), 64)
    assert base.dtype == np.float32 and (base >= 0).all() and (base < 1).all()
    assert abs(base.mean() - 0.5) < 0.02
    for other in (ops.quant_noise_host(5, 1, 0, 11, 2, np.arange(64), 64),          # next step
                  ops.quant_noise_host(5, 1, 0, 10, 2, np.arange(1, 65), 64),       # next rows
                  ops.quant_noise_host(5, 1, 0, 10, 3, np.arange(64), 64),          # another receiver
                  ops.quant_noise_host(5, 2, 0, 10, 2, np.arange(64), 64),          # another layer
                  ops.quant_noise_host(5, 1, 1, 10, 2, np.arange(64), 64),          # the other direction
                  ops.quant_noise_host(6, 1, 0, 10, 2, np.arange(64), 64)):         # another seed
        r = np.corrcoef(base.ravel(), other.ravel())[0, 1]
        assert abs(r) < 0.03, r
        assert not np.array_equal(base, other)
    # neighbouring elements of one row are uncorrelated too
    assert abs(np.corrcoef(base[:, :-1].ravel(), base[:, 1:].ravel())[0, 1]) < 0.03
    # at least 16 random bits per element: all 2^16 top-16-bit values show up over enough draws
    many = ops.quant_noise_host(1, 1, 0, 0, 0, np.arange(4096), 256)
    assert len(np.unique((many * 65536).astype(np.int64))) == 65536


@pytest.mark.parametrize("bits", [8, 4])
def test_special_rows(bits):
    x = _rows(5, 9)
    x[0] = 2.5                                       # constant
    x[1] = 0.0                                       # zero
    x[2, 3] = np.nan
    x[3, 0] = np.inf
    x[4, 0], x[4, 1] = -3e38, 3e38                   # finite elements, non-finite range
    codes, lo, scale = ops.quantise_host(x, bits, 0, 1, 0, 0, 0, 0)
    y = ops.dequantise_host(codes, lo, scale, bits, 9)
    assert scale[0] == 0 and (y[0] == 2.5).all()
    assert (y[1] == 0).all()
    assert np.isnan(y[2:]).all()
    # a never-written (zeroed) region decodes to exact zeros
    z = ops.dequantise_host(np.zeros((3, 16), np.uint8), np.zeros(3, np.float32), np.zeros(3, np.float32), bits, 9)
    assert (z == 0).all() and not np.signbit(z).any()


def test_four_bit_packing_round_trips():
    rng = np.random.default_rng(3)
    for d in (1, 5, 8, 33):
        x = rng.integers(0, 16, (7, d)).astype(np.float32)
        x[:, 0], x[:, -1] = 0, 15                    # range 15: scale 1, lo 0, codes = x exactly
        if d == 1:
            x[:, 0] = 3
        codes, lo, scale = ops.quantise_host(x, 4, 0, 1, 0, 0, 0, 0)
        if d > 1:
            assert (scale == 1).all() and (lo == 0).all()
            np.testing.assert_array_equal(codes[:, 0] & 15, x[:, 0].astype(np.uint8))
            np.testing.assert_array_equal(ops.dequantise_host(codes, lo, scale, 4, d), x)
        assert (codes[:, (d + 1) // 2:] == 0).all()


@pytest.mark.parametrize("d,bits,row", [(5, 8, 16), (5, 4, 16), (64, 8, 64), (64, 4, 32), (256, 8, 256), (256, 4, 128),
                                         (100, 4, 64), (17, 8, 32)])
def test_code_row_sizes(d, bits, row):
    assert ops.quant_row_bytes(d, bits) == row
    assert ops.quant_link_bytes(10, d, bits) == 10 * (row + 8)


@pytest.mark.parametrize("es", [4, 2])
def test_link_bytes_against_exact(es):
    exact = ops.quant_link_bytes(1000, 256, None, es)
    assert exact == 1000 * 256 * es
    r8, r4 = exact / ops.quant_link_bytes(1000, 256, 8), exact / ops.quant_link_bytes(1000, 256, 4)
    if es == 4:                                      # the ratios the design quotes for d = 256, fp32
        assert 3.8 < r8 < 4.0 and 7.4 < r4 < 7.6
    else:
        assert 1.9 < r8 < 2.0 and 3.7 < r4 < 3.8
