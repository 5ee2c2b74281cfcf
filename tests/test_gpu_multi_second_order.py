"""GPU, N > 1 (skipped on boxes with fewer GPUs): the pieces of a second backward across ranks -- the entry permutation between
a handle and its transpose is exact both ways, the weighted multiply with the handle's own values equals multiply bit for bit,
and the Hessian-vector product of a solve agrees with the dense one (tests/_mgpu_second_order_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_second_order(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29930 + world
    cmd = ["timeout", "600", sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "_mgpu_second_order_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=700)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert f"MGPU_SECOND_ORDER_OK {world}" in p.stdout
