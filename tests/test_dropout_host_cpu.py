"""The host port of the counter-based dropout mask (ops.dropout_keep_host) against a scalar restatement of
csrc/common.cuh (drop_seed_hi / drop_base / drop_bits), pinned values, and its keep rate."""
import numpy as np
import pytest

from pipegcn_b200.ops import DropSpec, dropout_keep_host

M = 0xFFFFFFFF


def _mix32(x):
    x &= M
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M
    x ^= x >> 15
    x = (x * 0x846CA68B) & M
    x ^= x >> 16
    return x


def _keep_scalar(p, seed, step, step_off, row, col, elem_size, d):
    """One element, written line for line from the device code with Python integers."""
    thresh16 = int(np.float32(np.float32(p) * np.float32(65536.0) + np.float32(0.5)))
    seed_lo, seed_hi = seed & M, seed >> 32
    key = _mix32(seed_hi if step is None else (seed_hi + 0x632BE5AB * ((step + step_off + 1) & M)) & M)
    v = 16 // elem_size
    i = row * ((d + v - 1) // v) + col // v
    base = _mix32(((i & M) ^ seed_lo) + ((key + (i >> 32) * 0x9E3779B9) & M))
    h = (base * (0x9E3779B1, 0x85EBCA6B, 0xC2B2AE35, 0x27D4EB2F)[((col % v) // 2) & 3]) & M
    h ^= h >> 16
    bits = (h & 0xFFFF) if col % 2 == 0 else (h >> 16)
    return bits >= thresh16


@pytest.mark.parametrize("p,seed,step,step_off,row0,d,es", [
    (0.3, 0x0123456789ABCDEF, 5, 2, (1 << 32) - 3, 12, 4),     # row index past 2^32: the 64-bit element index
    (0.5, 42, None, 0, 0, 8, 2),                                # no step counter
    (0.1, 0xFFFFFFFFFFFFFFFF, 0xFFFFFFFF, 7, 12345, 41, 2),    # counter + offset wrap around 2^32
    (0.9, 7, 3, 0, 2 ** 40 // 11, 5, 4),                        # ragged last vector
])
def test_dropout_keep_host_matches_scalar_restatement(p, seed, step, step_off, row0, d, es):
    spec = DropSpec(p, seed, step_off=step_off)
    got = dropout_keep_host(spec, step, row0, 6, d, es)
    want = np.array([[_keep_scalar(p, seed, step, step_off, row0 + r, c, es, d) for c in range(d)] for r in range(6)])
    assert got.shape == (6, d) and np.array_equal(got, want)


def test_dropout_keep_host_pinned_values():
    """Fixed outputs of the port: a change of the mask function (which every fused kernel evaluates) shows here."""
    m = dropout_keep_host(DropSpec(0.3, 0x0123456789ABCDEF, step_off=2), 5, (1 << 32) - 3, 4, 12, 4)
    assert np.packbits(m, axis=1).tolist() == [[217, 32], [235, 0], [239, 112], [111, 112]]
    m = dropout_keep_host(DropSpec(0.5, 42), None, 0, 3, 8, 2)
    assert np.packbits(m, axis=1).tolist() == [[25], [91], [23]]


@pytest.mark.parametrize("p", [0.1, 0.3, 0.5, 0.9])
def test_dropout_keep_host_rate(p):
    n, d = 20000, 50
    keep = dropout_keep_host(DropSpec(p, 0xC0FFEE, step_off=1), 3, 777, n, d, 4)
    z = abs(keep.mean() - (1 - p)) / np.sqrt(p * (1 - p) / keep.size)
    assert z < 5, z
