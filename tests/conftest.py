import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


_SCRATCH = []


def scratch_dir(prefix: str) -> str:
    """Temp directory for model files written by a test; everything is removed when the session ends
    (`tempfile.mkdtemp` alone leaks one directory per test run)."""
    import tempfile
    if not _SCRATCH:
        _SCRATCH.append(tempfile.mkdtemp(prefix="gllm_b200_pytest_"))
    return tempfile.mkdtemp(prefix=prefix, dir=_SCRATCH[0])


def pytest_sessionfinish(session, exitstatus):
    import shutil
    while _SCRATCH:
        shutil.rmtree(_SCRATCH.pop(), ignore_errors=True)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
