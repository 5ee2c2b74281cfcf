"""Call time of the shifted solvers with x_set / r in host pinned buffers, host pageable buffers and device memory (1 GPU, T' matrix).

The host paths copy x_set (L n_loc doubles) and r to the device and back on every call (bicg_shifted_solve_ex); the device path
(bicg_shifted_solve_dev) updates the caller's CUDA tensors in place.  CUDA events on the library's stream around each whole call,
after one warm-up call per mode; the three modes alternate within every repetition, and the median over the repetitions is
printed.  The card's name and power limit are read in the same run.
usage: shifted_device_perf.py [--method switching|lop ...] [L ...]   env: SP_G (grid size, default 117), SP_REPS (default 5)"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

METHODS = {"switching": "shifted_lopbicg_switching", "fixed": "shifted_lopbicg", "lop": "shifted_lopbicgstab",
           "pipe_lop": "shifted_pipe_lopbicgstab"}
ap = argparse.ArgumentParser()
ap.add_argument("--method", choices=sorted(METHODS), action="append")
ap.add_argument("L", nargs="*", type=int, default=[64, 512])
args = ap.parse_args()
methods = args.method or ["lop", "switching"]
g = int(os.environ.get("SP_G", "117"))
reps = int(os.environ.get("SP_REPS", "5"))
if not torch.cuda.is_available():
    sys.exit("shifted_device_perf: no CUDA device")
card = torch.cuda.get_device_name(0)
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
except (OSError, subprocess.TimeoutExpired):
    power = "unknown"
print(f"[shifted device] card: {card}, power limit: {power}", flush=True)

B.set_options(quiet=1, shift_tol=1e-8, shift_max_iter=300)
blk = B.gen_block("stencil15", g, 14.0)
n = blk.n
dm = B.DeviceMatrix(blk)
b = dm.spmv(np.ones(n))
stream = torch.cuda.ExternalStream(B.lib.bicg_stream())


def pinned(shape):
    return torch.empty(shape, dtype=torch.float64).pin_memory().numpy()


for L in args.L:
    sigma = (np.arange(L) + 1) * (0.01 / L)                 # main_shifted.c:95-99
    bs = b + sigma[0]
    bufs = {"pinned": (pinned((L, n)), pinned(n)), "pageable": (np.empty((L, n)), np.empty(n)),
            "device": (torch.empty((L, n), dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda"))}
    for name in methods:
        method = METHODS[name]
        times = {mode: [] for mode in bufs}
        iters = {}
        for rep in range(reps + 1):                         # rep 0 warms every mode up
            for mode, (x, r) in bufs.items():
                if mode == "device":
                    x.zero_(); r.copy_(torch.from_numpy(bs))
                    torch.cuda.synchronize()
                else:
                    x[:] = 0.0; r[:] = bs
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                k, st = dm.shifted_solve(method, x, r, sigma, 0)
                e1.record(stream)
                e1.synchronize()
                if rep:
                    times[mode].append(e0.elapsed_time(e1))
                iters[mode] = (k, st["iters"], st["loop_ms"], st["h2d_bytes"] + st["d2h_bytes"])
        assert len({v[0] for v in iters.values()}) == 1, iters
        line = ", ".join(f"{mode} {np.median(t):.1f} ms (min {min(t):.1f})" for mode, t in times.items())
        loops = ", ".join(f"{mode} {v[2]:.1f} ms" for mode, v in iters.items())
        it = iters["device"][1]
        saved = np.median(times["pageable"]) - np.median(times["device"]), np.median(times["pinned"]) - np.median(times["device"])
        print(f"[shifted device] T' g={g} n={n} {name} L={L}: {it} iterations; call time (median of {reps}): {line}; timed loop "
              f"(last call): {loops}; device saves {saved[0]:.1f} ms vs pageable, {saved[1]:.1f} ms vs pinned; host paths move "
              f"{iters['pinned'][3] / 1e9:.2f} GB, device path {iters['device'][3]} B", flush=True)
    del bufs
dm.destroy()
