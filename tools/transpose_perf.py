"""Cost of the transpose of a resident matrix at the benchmark's T' size (stencil15 g = 117: n = 1 601 613, nnz = 23 616 325), as
medians of alternated rounds on one rank:
  create_t     bicg_matrix_create_transpose of the handle, host clock up to a device synchronise
  create       bicg_matrix_destroy + bicg_matrix_create of the same blocks, the same way
  refresh_async  device time of DeviceMatrix.transpose_values_async, CUDA events around `--calls` back-to-back calls
  refresh_sync   DeviceMatrix.transpose_values, host clock (returns once done)
  set_async    device time of DeviceMatrix.set_values_async of the same nnz from a CUDA tensor, for comparison
  set_sync     DeviceMatrix.set_values from the same CUDA tensor, host clock
and the bytes one refresh moves against its traffic model (one rank): per entry 4 B of permutation, 8 B gathered from the source
and 8 B written, plus 16 B read and 7 B written by the value-table pass on packing CTAs.  The card's name and power limit are
read in the same run.
usage: transpose_perf.py [--g 117] [--rounds 5] [--calls 20] [--json FILE]"""
import argparse
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
    t1 = torch.from_numpy(v1).cuda()
    t2 = t1 * 1.0009765625
    dm = B.DeviceMatrix(blk)
    mt = dm.transpose()                                       # warm-up: plans of the transposed shape
    mt.transpose_values_async(dm)
    mt.transpose_values(dm)
    dm.set_values_async(t2)
    dm.set_values(t1)
    x = np.zeros(n)
    mt.solve("bicgstab", x, mt.spmv(np.ones(n)))
    packed = mt.packed_ctas()
    torch.cuda.synchronize()
    samples = {k: [] for k in ("create_t", "create", "refresh_async", "refresh_sync", "set_async", "set_sync")}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(a.rounds):
        e0.record()
        for _ in range(a.calls):
            mt.transpose_values_async(dm)
        e1.record()
        torch.cuda.synchronize()
        samples["refresh_async"].append(e0.elapsed_time(e1) / a.calls)
        e0.record()
        for i in range(a.calls):
            dm.set_values_async(t2 if i % 2 else t1)
        e1.record()
        torch.cuda.synchronize()
        samples["set_async"].append(e0.elapsed_time(e1) / a.calls)
        t = time.perf_counter()
        mt.transpose_values(dm)
        samples["refresh_sync"].append(1e3 * (time.perf_counter() - t))
        t = time.perf_counter()
        dm.set_values(t2 if rnd % 2 else t1)
        samples["set_sync"].append(1e3 * (time.perf_counter() - t))
        mt.destroy()
        B.lib.bicg_synchronize()
        t = time.perf_counter()
        mt = dm.transpose()
        B.lib.bicg_synchronize()
        samples["create_t"].append(1e3 * (time.perf_counter() - t))
        dm.set_values(v1)
        t = time.perf_counter()
        dm.destroy()
        dm = B.DeviceMatrix(blk)
        B.lib.bicg_synchronize()
        samples["create"].append(1e3 * (time.perf_counter() - t))
        mt.destroy()
        mt = dm.transpose()
    mt.destroy()
    dm.destroy()
    name, power = card()
    med = {k: statistics.median(v) for k, v in samples.items()}
    model = 20 * nnz + 23 * nnz
    out = {"card": name, "power_limit": power, "n": n, "nnz": nnz, "rounds": a.rounds, "calls": a.calls, "packed_ctas": packed,
           "median_ms": med, "samples_ms": samples, "model_bytes": model,
           "refresh_async_GBps": model / (med["refresh_async"] * 1e-3) / 1e9}
    print(f"{name}, power limit {power}; T' n={n} nnz={nnz}, {packed} packing CTAs on the transpose")
    for k in ("create_t", "create", "refresh_async", "refresh_sync", "set_async", "set_sync"):
        print(f"  {k:14s} {med[k]:9.3f} ms" + (f"   {model / (med[k] * 1e-3) / 1e9:7.1f} GB/s of the {model / 1e9:.2f} GB model"
                                                if k == "refresh_async" else ""))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
