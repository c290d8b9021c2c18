import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "slow_cpu: CPU test that takes tens of seconds")
    config.addinivalue_line("markers", "pending_gpu: GPU test of code that has not run on hardware yet; skipped unless "
                                       "SLLM_RUN_PENDING=1 (no test carries it at the moment)")


def pytest_collection_modifyitems(config, items):
    """Tests of kernels that have never run on a GPU must not be able to turn the validated suite red (the driver runs
    `-m gpu -x`).  They are opted into with SLLM_RUN_PENDING=1 and lose the marker once
    they have passed on an H100."""
    import torch
    lib_built = os.path.exists(os.path.join(ROOT, "swiftllm_b200", "libswiftllm_b200.so"))
    if not torch.cuda.is_available():
        # a plain `pytest` on a CPU box: GPU tests are skipped, not failed.  On a GPU box a missing library is NOT skipped -
        # the tests must fail loudly there (no silent fallback).
        no_gpu = pytest.mark.skip(reason="needs a CUDA device" + ("" if lib_built else " and libswiftllm_b200.so"))
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(no_gpu)
    if os.environ.get("SLLM_RUN_PENDING", "") == "1":
        return
    skip = pytest.mark.skip(reason="pending first GPU validation: set SLLM_RUN_PENDING=1 to run")
    for item in items:
        if "pending_gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        return np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    return load
