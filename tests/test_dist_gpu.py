"""Real multi-GPU parity: one process per GPU under torchrun -- CUDA IPC heaps, in-kernel
NVLink stores, NCCL all-reduce, eager and CUDA-graph replay -- against the CPU oracle (tools/dist_parity.py).
Skipped when fewer than two GPUs are visible; `bench.py --gpus N` runs the same check before timing."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def _torchrun(n, env_extra, *argv):
    env = dict(os.environ, **env_extra)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29533", str(ROOT / "tools" / "dist_parity.py"), *argv]
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("graph", ["0", "1"])
def test_two_ranks_match_oracle(graph):
    p = _torchrun(2, {"PG_PARITY_GRAPH": graph}, "tiny")
    assert p.returncode == 0 and "ALL OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
