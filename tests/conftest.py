import os
import sys

import pytest

# The in-process multi-rank GPU tests launch several kernels that wait for EACH OTHER on different streams; streams that
# share a hardware work queue would order them falsely (a kernel queued behind one that waits for it). More queues
# (must be set before CUDA initialises) make that impossible for the handful of streams the tests use.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# With lazy module loading the FIRST launch of a kernel may have to wait for the context to go idle; a kernel of another
# emulated rank that is already spinning for it would then never see it start. Real ranks are separate processes with their
# own contexts; the single-process harness loads everything up front instead.
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
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
