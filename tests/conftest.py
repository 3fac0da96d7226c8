import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pytorch-segmentation_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


try:  # the oracle's ATen-CPU ops crawl with 128 oversubscribed threads on the GPU hosts (measured 10x slower than 16)
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))
except Exception:
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on the GPU box")


@pytest.fixture(scope="session")
def gpu_out_dir():
    d = os.path.join(ROOT, "gpurun_out")
    os.makedirs(d, exist_ok=True)
    return d
