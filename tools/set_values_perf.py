"""Cost of new values on a resident matrix at the benchmark's T' size (stencil15 g = 117: n = 1 601 613, nnz = 23 616 325), as
medians of alternated rounds:
  async     device time of DeviceMatrix.set_values_async from a CUDA tensor, CUDA events around `--calls` back-to-back calls
  pinned    DeviceMatrix.set_values from pinned host arrays (returns once the values are in place), host clock
  pageable  the same from ordinary (pageable) numpy arrays
  create    bicg_matrix_destroy + bicg_matrix_create of the same blocks, host clock up to a device synchronise
  solve     one T' solve (bicgstab, tol 1e-10), device loop time, for scale
and the bytes one update moves against its traffic model (one rank): 16 B per entry for the copy of the values, plus 16 B read
and 7 B written per entry by the value-table pass on packing CTAs.  The card's name and power limit are read in the same run.
usage: set_values_perf.py [--g 117] [--rounds 5] [--calls 20] [--json FILE]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def pinned_copy(a):
    p = B.lib.bicg_host_alloc(a.nbytes)
    out = np.ctypeslib.as_array((C.c_double * a.size).from_address(p))
    out[:] = a
    return p, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=117)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json")
    a = ap.parse_args()
    B.set_options(quiet=1, tol=1e-10, max_iter=1000)
    blk = B.gen_block("stencil15", a.g, 14.0)
    n, nnz = blk.n_loc, int(blk.diag.nz)
    v1 = blk.diag_arrays()[0].copy()
    v2 = v1 * 1.0009765625                                   # 1 + 2^-10: new values, the same fields as the original
    dm = B.DeviceMatrix(blk)
    t1, t2 = torch.from_numpy(v1).cuda(), torch.from_numpy(v2).cuda()
    p1, h1 = pinned_copy(v1)
    p2, h2 = pinned_copy(v2)
    b = dm.spmv(np.ones(n))
    x = np.zeros(n)
    dm.solve("bicgstab", x, b.copy())                          # warm-up: plans, first launches
    packed = dm.packed_ctas()
    dm.set_values_async(t2)                                   # warm-up of every update path
    dm.set_values(h2)
    dm.set_values(v2)
    torch.cuda.synchronize()
    samples = {k: [] for k in ("async", "pinned", "pageable", "create", "solve")}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(a.rounds):
        e0.record()
        for i in range(a.calls):
            dm.set_values_async(t2 if i % 2 else t1)
        e1.record()
        torch.cuda.synchronize()
        samples["async"].append(e0.elapsed_time(e1) / a.calls)
        for key, src in (("pinned", h1 if rnd % 2 else h2), ("pageable", v1 if rnd % 2 else v2)):
            t = time.perf_counter()
            dm.set_values(src)
            samples[key].append(1e3 * (time.perf_counter() - t))
        dm.set_values(v1)
        t = time.perf_counter()
        dm.destroy()
        dm = B.DeviceMatrix(blk)
        B.lib.bicg_synchronize()
        samples["create"].append(1e3 * (time.perf_counter() - t))
        x = np.zeros(n)
        it, st = dm.solve("bicgstab", x, b.copy())
        samples["solve"].append(st["loop_ms"])
    dm.destroy()
    B.lib.bicg_host_free(p1)
    B.lib.bicg_host_free(p2)
    name, power = card()
    med = {k: statistics.median(v) for k, v in samples.items()}
    model = 16 * nnz + 23 * nnz                              # every CTA packs on T' (checked: packed_ctas below)
    out = {"card": name, "power_limit": power, "n": n, "nnz": nnz, "rounds": a.rounds, "calls": a.calls, "packed_ctas": packed,
           "median_ms": med, "samples_ms": samples, "solve_iters": it, "model_bytes": model,
           "async_GBps": model / (med["async"] * 1e-3) / 1e9}
    print(f"{name}, power limit {power}; T' n={n} nnz={nnz}, {packed} packing CTAs")
    for k in ("async", "pinned", "pageable", "create"):
        print(f"  {k:9s} {med[k]:9.3f} ms" + (f"   {model / (med[k] * 1e-3) / 1e9:7.1f} GB/s of the {model / 1e9:.2f} GB model"
                                               if k == "async" else ""))
    print(f"  solve     {med['solve']:9.3f} ms ({it} iterations)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
