"""CPU check (numpy) of the counter-based dropout mask of csrc/common.cuh (drop_base / drop_bits, ported to
the host as pipegcn_b200.ops.dropout_keep_host): keep rate per
element position, correlation between the 8 elements of a 16-byte vector, between neighbouring vectors / rows,
between epochs (the device-side step counter enters the key), and the variance of the kept count per vector.

    python tools/dropout_hash_quality.py            # prints one line per p; every z should be a few units at most
"""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from pipegcn_b200.ops import DROP_MUL, DropSpec, dropout_keep_host  # noqa: E402

MUL = list(DROP_MUL)          # drop_bits' per-pair multipliers (tests/test_host_logic_cpu.py checks them against the kernel)


def masks(n, seed, step, p):
    """Keep mask [n, 8] of the first n 16-byte bf16 vectors (one vector per row) under the key (seed, step)."""
    return dropout_keep_host(DropSpec(p, seed), step, 0, n, 8, 2).astype(np.float64)


def main(n=1 << 21):
    for p in (0.5, 0.1, 0.3, 0.9):
        ms = [masks(n, (777 << 32) | 0xdeadbeef, e, p) for e in range(5)]
        m = ms[0]
        z_mean = np.abs(m.mean(0) - (1 - p)).max() / np.sqrt(p * (1 - p) / n)
        c = np.corrcoef(m.T)
        np.fill_diagonal(c, 0)
        z_in = np.abs(c).max() * np.sqrt(n)
        z_nb = max(np.abs(np.corrcoef(m[:-s].T, m[s:].T)[:8, 8:]).max() for s in (1, 2, 32, 64)) * np.sqrt(n)
        z_ep = max(np.abs(np.corrcoef(ms[a].T, ms[b].T)[:8, 8:]).max() for a in range(5) for b in range(a + 1, 5)) * np.sqrt(n)
        var = m.sum(1).var() / (8 * p * (1 - p))
        print(f"p={p}: z_keep_rate={z_mean:.2f} z_in_vector={z_in:.2f} z_neighbours={z_nb:.2f} "
              f"z_epochs={z_ep:.2f} var_ratio={var:.4f}")
        assert z_mean < 5 and z_in < 5 and z_nb < 5 and z_ep < 5 and abs(var - 1) < 0.01


if __name__ == "__main__":
    main()
