"""Back-to-back shifted solves of a fixed iteration count (shift_tol = 0, shift_max_iter = ITERS) in three modes, alternated in
one run, for each shifted method: `sync` (DeviceMatrix.shifted_solve on CUDA tensors: bicg_shifted_solve_dev, which returns after
a host synchronise), `async` (DeviceMatrix.shifted_solve_async on torch's current stream) and `replay` (a torch CUDA graph holding
{r <- b; x_set <- 0; shifted_solve_async}).  Wall time per solve, from N solves ending in a device synchronise, as the median of
alternated rounds.  The small Laplacian measures the per-call overhead, which is what the asynchronous path changes; the T' rows
show what staging x_set through the handle's workspace (two extra device-to-device passes over it per asynchronous solve) costs
against real work.  The card's name and power limit are read in the same run.
usage: shifted_async_perf.py [--rounds 3] [--budget-s 6] [--only NAME ...] [--methods M ...] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi_bicgstab_b200 as B

# name -> (generator kind, g, p0, number of shifts, iterations per solve)
WORKLOADS = {
    "laplace5_g64_L16": ("laplace5", 64, 0.0, 16, 20),
    "stencil15_g40_L64": ("stencil15", 40, 14.0, 64, 50),
    "Tprime_g117_L64": ("stencil15", 117, 14.0, 64, 30),
    "Tprime_g117_L512": ("stencil15", 117, 14.0, 512, 30),
}
METHODS = ("shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab")
MODES = ("sync", "async", "replay")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def run_workload(dm, n, name, method, rounds, budget_ms):
    kind, g, p0, L, iters = WORKLOADS[name]
    B.set_options(quiet=1, shift_tol=0.0, shift_max_iter=iters, shift_error=0)
    b = torch.from_numpy(dm.spmv(np.ones(n))).cuda()
    sigma_h = (np.arange(L) + 1) * (0.5 / L)
    sigma = torch.from_numpy(sigma_h).cuda()
    x, r = torch.zeros(L, n, dtype=torch.float64, device="cuda"), b.clone()
    res = torch.zeros(32, dtype=torch.uint8, device="cuda")
    dm.prepare_shifted_async(method, L)
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        r.copy_(b)
        x.zero_()
        dm.shifted_solve_async(method, x, r, sigma, 0, result=res)

    def sync_one():
        r.copy_(b); x.zero_()
        return dm.shifted_solve(method, x, r, sigma_h, 0)

    def async_one():
        r.copy_(b); x.zero_()
        dm.shifted_solve_async(method, x, r, sigma, 0, result=res)

    one = {"sync": sync_one, "async": async_one, "replay": graph.replay}
    for m in MODES:                                              # warm-up of every mode
        one[m]()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ret, st = sync_one()
    torch.cuda.synchronize()
    one_ms = (time.perf_counter() - t0) * 1e3
    graph.replay()
    torch.cuda.synchronize()
    rec = B.decode_shift_result(res)
    assert rec["ret"] == ret and rec["iters"] == st["iters"], (rec, ret, st["iters"])
    per_round = max(1, min(50, int(budget_ms / rounds / max(one_ms, 1e-3))))
    wall = {m: [] for m in MODES}
    for _ in range(rounds):
        for m in MODES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(per_round):
                one[m]()
            torch.cuda.synchronize()
            wall[m].append((time.perf_counter() - t0) * 1e3 / per_round)
    del graph
    return {"workload": name, "method": method, "n": n, "L": L, "iters_run": st["iters"], "solves_per_round": per_round,
            "rounds": rounds, "wall_ms_per_solve": {m: float(np.median(v)) for m, v in wall.items()}, "wall_ms_rounds": wall}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--budget-s", type=float, default=6.0, help="about this much solving per mode, method and workload")
    ap.add_argument("--only", nargs="+", choices=sorted(WORKLOADS))
    ap.add_argument("--methods", nargs="+", choices=METHODS, default=list(METHODS))
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("shifted_async_perf: no CUDA device")
    name, power = card()
    print(f"[shifted async perf] card: {name}, power limit: {power}", flush=True)
    out = {"card": name, "power_limit": power, "results": []}
    for w in args.only or list(WORKLOADS):
        kind, g, p0, _, _ = WORKLOADS[w]
        blk = B.gen_block(kind, g, p0)
        dm = B.DeviceMatrix(blk)
        for method in args.methods:
            rec = run_workload(dm, blk.n_loc, w, method, args.rounds, args.budget_s * 1e3)
            out["results"].append(rec)
            wm = rec["wall_ms_per_solve"]
            print(f"[shifted async perf] {w:18s} {method:26s} n={rec['n']:8d} L={rec['L']:4d} iters={rec['iters_run']:3d}  "
                  f"wall ms/solve: sync {wm['sync']:9.3f}  async {wm['async']:9.3f}  replay {wm['replay']:9.3f}", flush=True)
        dm.destroy()
    B.set_options(shift_tol=1e-12, shift_max_iter=1000)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
