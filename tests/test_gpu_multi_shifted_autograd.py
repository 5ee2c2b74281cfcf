"""GPU, N > 1 (skipped on boxes with fewer GPUs): the differentiable shifted solve on several ranks -- every rank's b.grad and
value gradients agree with the dense computation of the whole matrix, sigma.grad is bit-identical on every rank (one cross-GPU
sum in rank order) and agrees with it too, and dots_async is bit-identical on every rank (tests/_mgpu_shifted_autograd_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_shifted_autograd(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29930 + world
    cmd = ["timeout", "600", sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "_mgpu_shifted_autograd_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=700)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert f"MGPU_SHIFTED_AUTOGRAD_OK {world}" in p.stdout
