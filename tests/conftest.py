import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def _cuda_device_present() -> bool:
    """cheap probe (no torch import): the driver's control node, or an explicit override for unusual setups"""
    if os.environ.get("CERBOS_B200_TEST_GPU") in ("0", "1"):
        return os.environ["CERBOS_B200_TEST_GPU"] == "1"
    return os.path.exists("/dev/nvidiactl") or os.path.exists("/dev/nvidia0")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a device: on a host without one they are skipped, not failed (cgpu_init has no CPU fallback)."""
    if _cuda_device_present():
        return
    skip = pytest.mark.skip(reason="no CUDA device on this host (cerbos_b200 has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
