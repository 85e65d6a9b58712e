import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def load_golden(name):
    import torch

    return torch.load(os.path.join(GOLDEN, name), map_location="cpu", weights_only=False)


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_makereport(item, call):
    """When a GPU test dies, print the kernels' watchdog record (a bounded in-kernel barrier wait that timed out leaves
    {1, site, blockIdx, threadIdx, parity, spins, source tag}): the difference between "numerics" and "pipeline hang"."""
    outcome = yield
    rep = outcome.get_result()
    if rep.when == "call" and rep.failed and item.get_closest_marker("gpu") is not None:
        try:
            from perceiver_io_b200 import _lib

            rec = _lib.debug_read()
            rep.sections.append(("pcv watchdog record", f"{rec} (word 0 != 0: a barrier wait timed out; word 1 = site, "
                                                         "word 2 = block, word 3 = thread, word 6 = 0xB3D: backward kernels)"))
        except Exception as e:  # noqa: BLE001
            rep.sections.append(("pcv watchdog record", f"unavailable: {e}"))
