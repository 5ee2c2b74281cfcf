"""Back-to-back solves of a fixed iteration count (tol = 0) in three modes, alternated in one run: DeviceMatrix.solve (returns after a
host synchronise), DeviceMatrix.solve_async on torch's current stream, and the replay of a torch CUDA graph holding one captured
solve_async.  Wall time of N solves ending in a device synchronise, per solve; also the device time of one solve from CUDA events
(synchronous: the loop_ms + h2d_ms + d2h_ms of its stats; asynchronous: events around the call on its stream).  The small
workloads measure the per-solve overhead, which is what the asynchronous path changes; the larger ones show it against real work.
The card's name and power limit are read in the same run.
usage: async_perf.py [--iters 20 300] [--solves 200] [--budget-s 20] [--only NAME ...] [--json FILE]"""
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

# name -> (generator kind, g, p0, options)
WORKLOADS = {
    "laplace5_g128": ("laplace5", 128, 0.0, {}),
    "laplace5_g512": ("laplace5", 512, 0.0, {}),
    "stencil15_g40": ("stencil15", 40, 14.0, {}),
    "Tprime_g117": ("stencil15", 117, 14.0, {}),
    "random_1M_k32": ("random", 1 << 20, 32, {}),          # long rows: the kernel-per-phase path (WHILE node when asynchronous)
}
MODES = ("sync", "async", "replay")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    return name, power


def run_workload(name, iters, solves, budget_ms, rounds=2):
    kind, g, p0, opts = WORKLOADS[name]
    B.set_options(quiet=1, tol=0.0, max_iter=iters, **opts)
    blk = B.gen_block(kind, g, p0)
    n = blk.n_loc
    dm = B.DeviceMatrix(blk)
    b = torch.from_numpy(dm.spmv(np.ones(n))).cuda()
    x, r = torch.zeros_like(b), b.clone()
    res = torch.zeros(24, dtype=torch.uint8, device="cuda")
    dm.prepare_async("bicgstab")
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        r.copy_(b)
        x.zero_()
        dm.solve_async("bicgstab", x, r, result=res)

    def sync_one():
        r.copy_(b); x.zero_()
        return dm.solve("bicgstab", x, r)[1]

    def async_one():
        r.copy_(b); x.zero_()
        dm.solve_async("bicgstab", x, r, result=res)

    one = {"sync": sync_one, "async": async_one, "replay": graph.replay}
    for m in MODES:                                              # warm-up of every mode
        one[m]()
    torch.cuda.synchronize()
    st = sync_one()
    dev = {"sync": st["loop_ms"] + st["h2d_ms"] + st["d2h_ms"]}
    for m in ("async", "replay"):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        (async_one if m == "async" else graph.replay)()
        e1.record()
        torch.cuda.synchronize()
        dev[m] = e0.elapsed_time(e1)
    ran = B.decode_result(res)["iters"]                        # < iters where the residual reaches exactly 0 (random)
    assert ran == st["iters"], (B.decode_result(res), st["iters"])
    # at most about budget_ms of solving per mode: the long solves of the large workloads are measured with fewer repetitions
    solves = max(2 * rounds, min(solves, int(budget_ms / max(dev["sync"], 1e-3))))
    wall = {m: [] for m in MODES}
    per_round = max(1, solves // rounds)
    for _ in range(rounds):
        for m in MODES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(per_round):
                one[m]()
            torch.cuda.synchronize()
            wall[m].append((time.perf_counter() - t0) * 1e3 / per_round)
    del graph
    dm.destroy()
    return {"workload": name, "n": n, "iters": iters, "iters_run": ran, "solves": per_round * rounds,
            "wall_ms_per_solve": {m: float(np.median(v)) for m, v in wall.items()},
            "wall_ms_per_solve_rounds": wall, "device_ms_one_solve": dev}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, nargs="+", default=[20, 300])
    ap.add_argument("--solves", type=int, default=200)
    ap.add_argument("--budget-s", type=float, default=20.0, help="fewer solves where one mode would take longer than this")
    ap.add_argument("--only", nargs="+", choices=sorted(WORKLOADS))
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("async_perf: no CUDA device")
    name, power = card()
    print(f"[async perf] card: {name}, power limit: {power}", flush=True)
    out = {"card": name, "power_limit": power, "results": []}
    for w in args.only or list(WORKLOADS):
        for it in args.iters:
            rec = run_workload(w, it, args.solves, args.budget_s * 1e3)
            out["results"].append(rec)
            wm, dv = rec["wall_ms_per_solve"], rec["device_ms_one_solve"]
            print(f"[async perf] {w:15s} n={rec['n']:8d} iters={rec['iters_run']:4d} solves={rec['solves']:3d}  wall ms/solve: sync {wm['sync']:.3f}  async {wm['async']:.3f}  "
                  f"replay {wm['replay']:.3f}  | device ms, one solve: sync {dv['sync']:.3f}  async {dv['async']:.3f}  "
                  f"replay {dv['replay']:.3f}", flush=True)
    B.set_options(tol=1e-15, max_iter=1000)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
