import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


os.environ.setdefault("DDN_TEST_FP32_SIMT", "1")      # the fp32 CUDA-core kernels are a test-only parity instrument


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")
    # the GPU boxes advertise 128 logical CPUs to a throttled container: 128 torch threads make the CPU oracle ~50x slower
    import torch
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
