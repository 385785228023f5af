"""Multi-GPU parity (one process per GPU, NCCL): needs >= 2 GPUs, skipped otherwise.
Run on a machine with 2+ GPUs: `python -m pytest tests -m gpu`."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.normpath(os.path.join(os.path.dirname(__file__), ".."))


def _ngpu():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("world", [2])
def test_multi_gpu_spmv_cg_spgemm(world):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "dist_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert out.stdout.count(" OK") == world
