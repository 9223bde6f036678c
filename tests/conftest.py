import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True, scope="session")
def _program_watchdog_for_sanitizer_runs():
    """B200AWQ_WATCHDOG_S=<seconds> (runs under compute-sanitizer): lengthen the decode-program kernels' spin watchdog
    (knob 16) - under compute-sanitizer a healthy wait takes longer than the default 0.5 s."""
    secs = os.environ.get("B200AWQ_WATCHDOG_S")
    if secs:
        try:
            import torch

            if torch.cuda.is_available():
                from autoawq_b200 import ext

                ext.set_knob(16, int(secs))
        except Exception:  # noqa: BLE001
            pass
    yield
