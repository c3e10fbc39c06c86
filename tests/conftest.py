import os
import sys
from pathlib import Path

# several simulated ranks share one GPU in the LocalWorld tests, each with its own streams:
# keep them on distinct hardware queues so that a flag-wait kernel cannot block its producer
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import pytest
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
