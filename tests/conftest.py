import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on the GPU box")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    class G:
        bitpack = np.load(os.path.join(GOLDEN, "bitpack.npz"))
        quant = np.load(os.path.join(GOLDEN, "quantize_small.npz"))
        config1 = np.load(os.path.join(GOLDEN, "config1.npz"))
        state_dict = np.load(os.path.join(GOLDEN, "state_dict.npz"))
        degenerate = np.load(os.path.join(GOLDEN, "quantize_degenerate.npz"))  # groups on the guards of the init (quantize.py:126-131)
        heavy = np.load(os.path.join(GOLDEN, "quantize_heavy.npz"))  # heavy-tailed weights: the shrinkage's |x|^(p-1) branch is active
    return G


@pytest.fixture(scope="session")
def oracle():
    from oracle import hqq_oracle
    return hqq_oracle
