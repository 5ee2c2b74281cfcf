"""GPU, N > 1 (skipped on boxes with fewer GPUs): the transpose of a resident matrix on every rank -- its product and solve equal
those of a handle created from the blocks of the stably transposed global CSR, and the asynchronous refresh behind a value
update on the source is stream-ordered across the ranks (tests/_mgpu_transpose_worker.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_transpose(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29890 + world
    cmd = ["timeout", "600", sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "_mgpu_transpose_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=700)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert f"MGPU_TRANSPOSE_OK {world}" in p.stdout
