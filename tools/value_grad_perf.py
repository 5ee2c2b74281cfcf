"""Cost of the value gradient and of a differentiable solve at the benchmark's T' size (stencil15 g = 117), on one rank:
  value_grad_async against multiply_async of the same nvec (1, 2, 4, 8, 16 vectors), device time from CUDA events around
      `--calls` back-to-back calls, each against its bytes model;
  one solve_autograd forward alone against forward + loss.backward() at tol 1e-8, with the backward's three parts -- the
      transpose refresh, the adjoint solve and the value gradient -- timed on their own the same way.
Medians of `--rounds` rounds in which the order of every compared pair alternates.  The card's name and power limit are read
in the same run.

Bytes models (per call, one rank):
  value gradient, per batch of nb <= 8 vectors: 4 B of column and 8 B written per entry (+ 8 B read when beta != 0), the
      row pointers (4 (n + 1)), and 8 n per u_j read and per v_j gathered;
  multiply, per batch: 12 B per entry (value and column), the row pointers, and 8 n per x_j gathered and per y_j written.
usage: value_grad_perf.py [--g 117] [--rounds 5] [--calls 20] [--json FILE]"""
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

NV_MAX = 8


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def grad_bytes(nvec, n, nnz, beta=0.0):
    batches = (nvec + NV_MAX - 1) // NV_MAX
    per_entry = 4 + 8 + (8 if beta != 0.0 else 0)
    return batches * (per_entry * nnz + 4 * (n + 1)) + 16 * nvec * n + (batches - 1) * 8 * nnz   # later batches read out


def multiply_bytes(nvec, n, nnz):
    batches = (nvec + NV_MAX - 1) // NV_MAX
    return batches * (12 * nnz + 4 * (n + 1)) + 16 * nvec * n


def device_ms(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=117)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json")
    a = ap.parse_args()
    B.set_options(quiet=1, tol=1e-8, max_iter=1000)
    blk = B.gen_block("stencil15", a.g, 14.0)
    n, nnz = blk.n_loc, int(blk.diag.nz)
    vals = torch.from_numpy(blk.diag_arrays()[0].copy()).cuda()
    dm = B.DeviceMatrix(blk)
    dm.prepare_autograd("bicgstab")
    mt = dm._adjoint()
    rng = np.random.default_rng(0)
    xs = torch.from_numpy(rng.standard_normal((16, n))).cuda()
    us = torch.from_numpy(rng.standard_normal((16, n))).cuda()
    ys = torch.empty_like(xs)
    gd = torch.empty(nnz, dtype=torch.float64, device="cuda")
    b = torch.from_numpy(dm.spmv(np.ones(n))).cuda()
    w = torch.from_numpy(rng.standard_normal(n)).cuda()
    nvecs = (1, 2, 4, 8, 16)

    def forward():
        return B.solve_autograd(dm, b, diag_val=vals)

    def forward_backward():
        tb, tv = b.clone().requires_grad_(), vals.clone().requires_grad_()
        (B.solve_autograd(dm, tb, diag_val=tv) * w).sum().backward()

    lam, x, r = torch.zeros(n, dtype=torch.float64, device="cuda"), forward(), torch.empty(n, dtype=torch.float64, device="cuda")

    def adjoint_solve():
        lam.zero_()
        r.copy_(w)
        mt.solve_async("bicgstab", lam, r)

    parts = {"refresh": lambda: mt.transpose_values_async(dm), "adjoint_solve": adjoint_solve,
             "value_grad": lambda: dm.value_grad_async(lam, x, alpha=-1.0, diag_out=gd)}
    for nv in nvecs:                                                  # warm-up of every shape
        dm.value_grad_async(us[:nv], xs[:nv], diag_out=gd)
        dm.multiply_async(xs[:nv], ys[:nv])
    forward_backward()
    for f in parts.values():
        f()
    torch.cuda.synchronize()
    samples = {f"{k}_{nv}": [] for nv in nvecs for k in ("value_grad", "multiply")}
    samples.update({k: [] for k in ("forward", "forward_backward", *parts)})
    solve_calls = max(1, a.calls // 10)
    for rnd in range(a.rounds):
        order = nvecs if rnd % 2 == 0 else nvecs[::-1]
        for nv in order:
            pair = {"value_grad": lambda: dm.value_grad_async(us[:nv], xs[:nv], diag_out=gd),
                    "multiply": lambda: dm.multiply_async(xs[:nv], ys[:nv])}
            for k in (("value_grad", "multiply") if rnd % 2 == 0 else ("multiply", "value_grad")):
                samples[f"{k}_{nv}"].append(device_ms(pair[k], a.calls))
        for k in (("forward", "forward_backward") if rnd % 2 == 0 else ("forward_backward", "forward")):
            samples[k].append(device_ms(forward if k == "forward" else forward_backward, solve_calls))
        for k, f in parts.items():
            samples[k].append(device_ms(f, solve_calls if k == "adjoint_solve" else a.calls))
    name, power = card()
    med = {k: statistics.median(v) for k, v in samples.items()}
    print(f"{name}, power limit {power}; T' n={n} nnz={nnz}, medians of {a.rounds} alternated rounds")
    out = {"card": name, "power_limit": power, "n": n, "nnz": nnz, "rounds": a.rounds, "median_ms": med, "samples_ms": samples,
           "GBps": {}}
    for nv in nvecs:
        gb, mb = grad_bytes(nv, n, nnz), multiply_bytes(nv, n, nnz)
        g_ms, m_ms = med[f"value_grad_{nv}"], med[f"multiply_{nv}"]
        out["GBps"][nv] = {"value_grad": gb / (g_ms * 1e-3) / 1e9, "multiply": mb / (m_ms * 1e-3) / 1e9}
        print(f"  nvec {nv:2d}: value_grad {g_ms:7.3f} ms ({gb / (g_ms * 1e-3) / 1e9:6.0f} GB/s of {gb / 1e9:.3f} GB)   "
              f"multiply {m_ms:7.3f} ms ({mb / (m_ms * 1e-3) / 1e9:6.0f} GB/s of {mb / 1e9:.3f} GB)")
    print(f"  solve forward {med['forward']:.2f} ms, forward + backward {med['forward_backward']:.2f} ms; backward parts: "
          f"refresh {med['refresh']:.3f} ms, adjoint solve {med['adjoint_solve']:.2f} ms, value gradient {med['value_grad']:.3f} ms")
    dm.destroy()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
