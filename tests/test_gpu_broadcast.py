"""vtts_broadcast_weights (SURVEY.md 8b/8e): the start-up weight broadcast through the C ABI on two GPUs.
Skipped on single-GPU machines (run on two GPUs with `python -m pytest tests/test_gpu_broadcast.py -m gpu`)."""
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]


def test_broadcast_weights_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", str(REPO / "tests" / "helpers" / "bcast_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "BCAST_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_broadcast_weights_rejects_null_comm():
    from viettts_b200.engine import Engine
    from viettts_b200 import _lib
    e = Engine(0)
    with pytest.raises(_lib.VttsError):
        e.broadcast_weights(None, 0, True)
    e.close()
