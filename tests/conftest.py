import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a)")


def _has_gpu() -> bool:
    try:
        from kafka_topic_analyzer_b200 import lib
        return lib().kta_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # On a machine without a GPU, gpu-marked tests are skipped.
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
