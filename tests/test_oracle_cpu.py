"""CPU tests: the oracle's own known-answer properties (SURVEY.md §4) and host logic."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

from oracle.train import run_world
from tests.helpers import make_args, small_world

ROOT = Path(__file__).resolve().parent.parent


def _total_loss(traces, e):
    return sum(t.losses[e] for t in traces)


@pytest.mark.parametrize("n_parts", [2, 3])
def test_partition_equivalence(n_parts):
    """Non-pipelined exchange makes P-partition training exact: same loss and weights as 1 partition."""
    g, _, _, s1 = small_world("tiny", 1)
    _, _, _, sp = small_world("tiny", n_parts)
    oargs, _ = make_args(g, 5, n_epochs=3)
    t1 = run_world(s1, oargs)
    tp = run_world(sp, oargs)
    for e in range(3):
        assert abs(_total_loss(t1, e) - _total_loss(tp, e)) < 2e-4 * abs(_total_loss(t1, e))
    for k, v in t1[0].state_dict.items():
        torch.testing.assert_close(tp[0].state_dict[k], v, rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(tp[-1].state_dict[k], tp[0].state_dict[k], rtol=0, atol=0)


def test_layouts_match_oracle_setup():
    """The vectorised layout builder equals the reference's per-process procedure, bit for bit."""
    for n_parts in (1, 2, 4):
        _, _, layouts, setups = small_world("tiny", n_parts, seed_graph=n_parts)
        for L, S in zip(layouts, setups):
            assert (L.num_in, L.num_all) == (S.num_in, S.num_all)
            rows = torch.repeat_interleave(torch.arange(L.num_in), (L.indptr[1:] - L.indptr[:-1]).long())
            k1 = torch.sort(rows * L.num_all + L.indices.long()).values
            k2 = torch.sort(S.v * S.num_all + S.u).values
            assert torch.equal(k1, k2)
            trows = torch.repeat_interleave(torch.arange(L.num_all), (L.t_indptr[1:] - L.t_indptr[:-1]).long())
            k3 = torch.sort(L.t_indices.long() * L.num_all + trows).values
            assert torch.equal(k1, k3)
            assert torch.equal(L.in_deg, S.in_deg)
            assert L.recv_shape == S.recv_shape
            for a, b in zip(L.boundary, S.boundary):
                assert (a is None and b is None) or torch.equal(a, b)
            assert torch.equal(L.feat, S.node_dict["feat"])
            assert torch.equal(L.label, S.node_dict["label"])
            assert torch.equal(L.train_mask, S.node_dict["train_mask"])
            n_train = int(L.train_mask.sum())
            assert bool(L.train_mask[:n_train].all())      # move_train_first


def test_staleness_epoch0_sees_zero_halo():
    """Pipelined epoch 0 consumes zero halo rows; epoch 1 consumes epoch 0's boundary rows."""
    g, _, _, sp = small_world("tiny", 2)
    oargs, _ = make_args(g, 5, n_epochs=2, enable_pipeline=True)
    tr = run_world(sp, oargs)
    for r, s in enumerate(sp):
        f0 = tr[r].layers[0][0]["f_buf"]
        assert torch.count_nonzero(f0[s.num_in:]) == 0
        other = 1 - r
        sent = tr[other].layers[0][0]["f_buf"][: sp[other].num_in][sp[other].boundary[r]]
        got = tr[r].layers[1][0]["f_buf"][s.num_in:]
        torch.testing.assert_close(got, sent, rtol=0, atol=0)


def test_ema_closed_form():
    """feat-corr: halo rows at epoch t equal (1-m) * sum_k m^(t-1-k) x_k (no bias correction)."""
    g, _, _, sp = small_world("tiny", 2)
    m = 0.9
    oargs, _ = make_args(g, 5, n_epochs=4, enable_pipeline=True, feat_corr=True, corr_momentum=m)
    tr = run_world(sp, oargs)
    r, other = 0, 1
    xs = [tr[other].layers[e][0]["f_buf"][: sp[other].num_in][sp[other].boundary[r]] for e in range(4)]
    for t in range(1, 4):
        want = sum((1 - m) * (m ** (t - 1 - k)) * xs[k] for k in range(t))
        got = tr[r].layers[t][0]["f_buf"][sp[r].num_in:]
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)


def test_c_abi_exports_every_declared_symbol():
    """The shared library loads on a CPU-only host and exports every function of include/pipegcn_b200.h."""
    from pipegcn_b200.build import build
    lib_path = build(verbose=False)
    lib = ctypes.CDLL(str(lib_path))
    header = (ROOT / "include" / "pipegcn_b200.h").read_text()
    names = re.findall(r"^\s*(?:int|int64_t|const char\*)\s+(pg_[a-z0-9_]+)\s*\(", header, flags=re.M)
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    lib.pg_abi_version.restype = ctypes.c_int
    assert lib.pg_abi_version() == 2
    from pipegcn_b200 import _C
    assert set(_C.EXPORTS) == set(names)


def test_ops_refuse_cpu_tensors():
    """No CPU fall-back: the product ops fail loudly without a CUDA tensor."""
    from pipegcn_b200 import _C, ops
    with pytest.raises(_C.PgError):
        ops._rows(torch.zeros(4, 4))


def test_command_line_matches_reference_flags():
    """Same flags, aliases and defaults as PipeGCN/helper/parser.py (fixture tests/golden/ref_parser.json),
    except `--backend` (nccl instead of gloo: the only implemented transport) and the added `--dtype` and `--no-partition-cache`."""
    import json
    from pipegcn_b200.helper.parser import create_parser
    ref = json.loads((ROOT / "tests" / "golden" / "ref_parser.json").read_text())
    ours = vars(create_parser([]))
    for k, v in ref["defaults"].items():
        assert k in ours, f"flag {k} missing"
        if k != "backend":
            assert ours[k] == v, (k, ours[k], v)
    assert ours["backend"] == "nccl" and ours["dtype"] == "fp32"
    assert set(ours) - set(ref["defaults"]) == {"dtype", "partition_cache"}
    got = vars(create_parser(["--n_layers", "4", "--enable_pipeline", "--feat-corr", "--no-eval", "--norm", "batch"]))
    for k, v in ref["parsed_example"].items():
        if k != "backend":
            assert got[k] == v, (k, got[k], v)
