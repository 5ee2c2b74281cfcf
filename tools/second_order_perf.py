"""Cost of the pieces a second backward adds, at the benchmark's T' size (stencil15 g = 117), on one rank:
  multiply_values_async with the handle's own values against multiply_async, at nvec 1 and 8;
  transpose_entries_async forward and reverse against transpose_values_async;
  one Hessian-vector product of a solve (forward, grad with create_graph, second grad) against one forward + first-order
      backward, at tol 1e-8.
Device time from CUDA events around `--calls` back-to-back calls (one call per HVP or backward); medians of `--rounds` rounds
in which the order of every compared pair alternates.  The card's name, power limit and max SM clock are read in the same run.
usage: second_order_perf.py [--g 117] [--rounds 5] [--calls 20] [--json FILE]"""
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return name, q


def device_ms(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def pairs(rounds, cases):
    """cases: {name: (fn, calls)}, compared in pairs (a, b) whose order alternates by round; returns medians in ms"""
    out = {k: [] for k in cases}
    names = list(cases)
    for r in range(rounds):
        for i in range(0, len(names), 2):
            pair = names[i:i + 2] if r % 2 == 0 else names[i:i + 2][::-1]
            for k in pair:
                fn, calls = cases[k]
                out[k].append(device_ms(fn, calls))
    return {k: statistics.median(v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=117)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json")
    a = ap.parse_args()
    B.set_options(quiet=1, tol=1e-8, max_iter=5000)
    blk = B.gen_block("stencil15", a.g, 14.0)
    n = blk.n_loc
    dm = B.DeviceMatrix(blk)
    dm.prepare_autograd("bicgstab")
    mt = dm._adjoint()
    vals = torch.from_numpy(blk.diag_arrays()[0].copy()).cuda()
    dm.set_values_async(vals)
    rng = np.random.default_rng(0)
    res = {}
    for nvec in (1, 8):
        x = torch.from_numpy(rng.standard_normal((nvec, n))).cuda()
        y = torch.empty_like(x)
        for fn in (lambda: dm.multiply_async(x, y), lambda: dm.multiply_values_async(vals, None, x, y)):
            fn()
        res.update({f"{k}_nvec{nvec}": v for k, v in pairs(a.rounds, {
            "multiply": (lambda: dm.multiply_async(x, y), a.calls),
            "multiply_values": (lambda: dm.multiply_values_async(vals, None, x, y), a.calls)}).items()})
    pd = torch.empty(int(mt.blk.diag.nz), dtype=torch.float64, device="cuda")
    back = torch.empty_like(vals)
    res.update(pairs(a.rounds, {
        "transpose_values": (lambda: mt.transpose_values_async(dm), a.calls),
        "entries_forward": (lambda: mt.transpose_entries_async(dm, vals, out=(pd, None)), a.calls)}))
    res.update(pairs(a.rounds, {
        "entries_forward_again": (lambda: mt.transpose_entries_async(dm, vals, out=(pd, None)), a.calls),
        "entries_reverse": (lambda: mt.transpose_entries_async(dm, pd, reverse=True, out=(back, None)), a.calls)}))
    b = torch.from_numpy(rng.standard_normal(n)).cuda()
    w, vb, vv = (torch.from_numpy(rng.standard_normal(k)).cuda() for k in (n, n, vals.numel()))

    def first():
        tb, tv = b.clone().requires_grad_(True), vals.clone().requires_grad_(True)
        x = B.solve_autograd(dm, tb, diag_val=tv)
        ((w * x).sum() + 0.5 * (x * x).sum()).backward()

    def hvp():
        tb, tv = b.clone().requires_grad_(True), vals.clone().requires_grad_(True)
        x = B.solve_autograd(dm, tb, diag_val=tv)
        g = torch.autograd.grad((w * x).sum() + 0.5 * (x * x).sum(), (tb, tv), create_graph=True)
        torch.autograd.grad((g[0] * vb).sum() + (g[1] * vv).sum(), (tb, tv))
    first(), hvp()
    torch.cuda.synchronize()
    res.update(pairs(a.rounds, {"forward_backward": (first, 1), "hvp": (hvp, 1)}))
    name, q = card()
    out = dict(card=name, power_limit_and_max_sm_clock=q, g=a.g, n=n, nnz=int(blk.diag.nz), ms=res)
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    dm.destroy()


if __name__ == "__main__":
    main()
