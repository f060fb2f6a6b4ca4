import os
import sys
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parents[1]
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))


def pytest_configure(config):
    try:  # the CPU oracle is small-op bound: 128 threads on a big host only add overhead
        import torch
        torch.set_num_threads(min(16, os.cpu_count() or 1))
    except Exception:
        pass
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def hifigan_params():
    from viettts_b200 import synthetic
    return synthetic.hifigan_params(1234)


@pytest.fixture(scope="session")
def acoustic_ckpt():
    from viettts_b200 import synthetic
    return synthetic.acoustic_ckpt(1234)


@pytest.fixture(scope="session")
def golden_dir():
    return REPO / "tests" / "golden"
