"""GPU, N > 1 (skipped on boxes with fewer GPUs): 16-bit column codes with ghost windows -- coded solves against solves forced to
32-bit columns, bit for bit on every rank (tests/_mgpu_stream_codes_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_gpu_stream_codes(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29780 + world
    cmd = ["timeout", "600", sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "_mgpu_stream_codes_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=700)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert f"MGPU_STREAM_CODES_OK {world}" in p.stdout
