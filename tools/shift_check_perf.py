"""Time of bicg_shift_residuals (csrc/shift_check.cu) on the T' matrix (1 GPU), device vectors, against
    the floor 12 nnz + 8 n (L + 1) bytes (matrix once, every x_j once, b once) and
    L x bicg_spmv_time, the cost of one SpMV per shift as the reference's check does it.
CUDA events on the library's stream around each call, after warm-up; a call includes its host synchronisation and the host side
of the final sum.  The card's name and power limit are read in the same run.
usage: shift_check_perf.py [L ...]   env: SP_G (grid size, default 117), SP_REPS (timed calls per L, default 10)"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

Ls = [int(a) for a in sys.argv[1:]] or [16, 64, 512]
g = int(os.environ.get("SP_G", "117"))
reps = int(os.environ.get("SP_REPS", "10"))
if not torch.cuda.is_available():
    sys.exit("shift_check_perf: no CUDA device")
card = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
except (OSError, subprocess.TimeoutExpired):
    power = "unknown"
print(f"[shift check] card: {card}, power limit: {power}", flush=True)

B.set_options(quiet=1)
blk = B.gen_block("stencil15", g, 14.0)
n, nnz = blk.n, blk.nnz_loc
dm = B.DeviceMatrix(blk)
spmv_ms, _ = dm.spmv_time(50)
stream = torch.cuda.ExternalStream(B.lib.bicg_stream())
for L in Ls:
    sigma = (np.arange(L) + 1) * (0.01 / L)
    gen = torch.Generator(device="cuda").manual_seed(L)
    x = torch.rand((L, n), dtype=torch.float64, device="cuda", generator=gen)
    b = torch.rand(n, dtype=torch.float64, device="cuda", generator=gen)
    for _ in range(2):
        dm.shift_residuals(x, b, sigma)
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        dm.shift_residuals(x, b, sigma)
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    floor = 12.0 * nnz + 8.0 * n * (L + 1)
    print(f"[shift check] T' g={g} n={n} nnz={nnz} L={L}: {ms:.3f} ms per call (median of {reps}, min {min(times):.3f}), "
          f"floor {floor / 1e9:.3f} GB -> {floor / ms / 1e6:.0f} GB/s; {L} x SpMV = {L * spmv_ms:.3f} ms "
          f"({L * spmv_ms / ms:.1f}x)", flush=True)
    del x, b
dm.destroy()
