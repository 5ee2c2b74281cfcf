"""Cost of the batched multiply y_j = alpha (A + sigma_j I) x_j + beta y_j on a resident matrix at the benchmark's T' size
(stencil15 g = 117: n = 1 601 613, nnz = 23 616 325), as medians of alternated rounds, CUDA events around `--calls`
back-to-back calls on torch's current stream:
  spmv       bicg_spmv_time of the same handle (the solver's SpMV with its fused dot), per launch
  batched    DeviceMatrix.multiply_async of nvec vectors at once, per vector, for nvec in 1 2 4 8 16
  single     nvec multiply_async calls of one vector each, per vector
and the bytes each moves against the traffic model: 12 nnz + 4 n per pass over the matrix (one pass per 8 vectors), 8 n per x_j
gathered, 8 n per y_j written (beta = 0 here, so y is not read), as GB/s and as a share of the H100 SXM's 3.35 TB/s.  The card's
name and power limit are read in the same run.
usage: multiply_perf.py [--g 117] [--rounds 5] [--calls 20] [--json FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

NV_MAX = 8            # vectors per launch (MUL_NV_MAX of csrc/spmv.cuh)
PEAK = 3.35e12        # HBM3 bandwidth of the H100 SXM data sheet, B/s


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def model_bytes(nvec, n, nnz):
    passes = -(-nvec // NV_MAX)
    return passes * (12 * nnz + 4 * n) + nvec * (8 * n + 8 * n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=117)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json")
    a = ap.parse_args()
    B.set_options(quiet=1)
    blk = B.gen_block("stencil15", a.g, 14.0)
    n, nnz = blk.n_loc, int(blk.diag.nz)
    dm = B.DeviceMatrix(blk)
    nvecs = [1, 2, 4, 8, 16]
    x = torch.from_numpy(np.random.default_rng(1).standard_normal((max(nvecs), n))).cuda()
    y = torch.empty_like(x)
    for nv in nvecs:                                          # warm-up of every instantiation the timed window uses
        dm.multiply_async(x[:nv], y[:nv])
    dm.multiply_async(x[0], y[0])
    dm.spmv_time(5)
    torch.cuda.synchronize()
    samples = {"spmv": [], **{f"batched{nv}": [] for nv in nvecs}, **{f"single{nv}": [] for nv in nvecs}}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, per):
        e0.record()
        for _ in range(a.calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.calls / per

    for rnd in range(a.rounds):
        order = nvecs if rnd % 2 == 0 else nvecs[::-1]
        samples["spmv"].append(dm.spmv_time(a.calls)[0])
        for nv in order:
            xs, ys = x[:nv], y[:nv]
            singles = lambda: [dm.multiply_async(xs[j], ys[j]) for j in range(nv)]
            batched = lambda: dm.multiply_async(xs, ys)
            for key, fn in ((("single", singles), ("batched", batched)) if rnd % 2 else (("batched", batched), ("single", singles))):
                samples[f"{key}{nv}"].append(timed(fn, nv))
    dm.destroy()
    name, power = card()
    med = {k: statistics.median(v) for k, v in samples.items()}
    rows = []
    for nv in nvecs:
        for key in ("batched", "single"):
            ms = med[f"{key}{nv}"]
            by = (model_bytes(nv, n, nnz) if key == "batched" else nv * model_bytes(1, n, nnz)) / nv
            rows.append({"nvec": nv, "path": key, "ms_per_vector": ms, "model_bytes_per_vector": by,
                         "GBps": by / (ms * 1e-3) / 1e9, "share_of_3.35TBps": by / (ms * 1e-3) / PEAK})
    out = {"card": name, "power_limit": power, "n": n, "nnz": nnz, "rounds": a.rounds, "calls": a.calls,
           "spmv_time_ms": med["spmv"], "multiply_nvec1_ms": med["batched1"], "median": rows, "samples_ms": samples}
    print(f"{name}, power limit {power}; T' n={n} nnz={nnz}, medians of {a.rounds} rounds of {a.calls} calls")
    print(f"  spmv_time {med['spmv']:.4f} ms   multiply_async nvec=1 {med['batched1']:.4f} ms")
    print("  nvec  path     ms/vector   GB/s  share of 3.35 TB/s")
    for r in rows:
        print(f"  {r['nvec']:4d}  {r['path']:8s} {r['ms_per_vector']:9.4f} {r['GBps']:7.1f}  {100 * r['share_of_3.35TBps']:5.1f} %")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
