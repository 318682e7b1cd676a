"""pytest configuration: registers the `gpu` marker and puts the oracle and the
package directory on sys.path.  GPU tests are skipped (not failed) when no CUDA device
is visible, so `-m "not gpu"` and a plain run both work on a machine without a GPU."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "chainer-faster-rcnn_b200")
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
