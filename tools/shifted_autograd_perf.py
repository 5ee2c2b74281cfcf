"""Cost of a differentiable shifted solve at the benchmark's T' size (stencil15 g = 117), on one rank:
  one shifted_solve_autograd forward alone against forward + loss.backward() at L = 1, 4 and 8 shifts (shifted_lopbicgstab,
      BICG_SHIFT_TOL = BICG_TOL = 1e-8; the backward runs L adjoint BiCGStab solves on A^T + sigma_j I);
  the two device operations the backward adds, each alone: shift_diagonal_async on the transpose, and dots_async over L
      vectors (L = 1, 4, 8), with the bytes dots_async reads (16 n per vector) over its time;
  one transpose refresh and one adjoint solve on A^T + sigma I, the parts the backward repeats L times.
Device time from CUDA events; medians of `--rounds` rounds in which the order of every compared pair alternates.  The card's
name and power limit are read in the same run.
usage: shifted_autograd_perf.py [--g 117] [--rounds 3] [--calls 20] [--json FILE]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mpi_bicgstab_b200 as B
from value_grad_perf import card, device_ms

METHOD = "shifted_lopbicgstab"
LS = (1, 4, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=117)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json")
    a = ap.parse_args()
    B.set_options(quiet=1, tol=1e-8, max_iter=1000, shift_tol=1e-8, shift_max_iter=1000)
    blk = B.gen_block("stencil15", a.g, 14.0)
    n, nnz = blk.n_loc, int(blk.diag.nz)
    vals = torch.from_numpy(blk.diag_arrays()[0].copy()).cuda()
    dm = B.DeviceMatrix(blk)
    rng = np.random.default_rng(0)
    b = torch.from_numpy(dm.spmv(np.ones(n))).cuda()
    sigmas = {L: torch.linspace(0.0, 2.0, L, dtype=torch.float64, device="cuda") for L in LS}
    ws = {L: torch.from_numpy(rng.standard_normal((L, n))).cuda() for L in LS}
    for L in LS:
        dm.prepare_shifted_autograd(METHOD, L)
    mt = dm._t

    def forward(L):
        return lambda: B.shifted_solve_autograd(dm, b, sigmas[L], METHOD, diag_val=vals)

    def forward_backward(L):
        def run():
            tb, ts, tv = b.clone().requires_grad_(), sigmas[L].clone().requires_grad_(), vals.clone().requires_grad_()
            (B.shifted_solve_autograd(dm, tb, ts, METHOD, diag_val=tv) * ws[L]).sum().backward()
        return run

    lam, r = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda")
    xs = {L: forward(L)().detach() for L in LS}
    outs = {L: torch.empty(L, dtype=torch.float64, device="cuda") for L in LS}

    def adjoint_solve():
        lam.zero_()
        r.copy_(ws[1][0])
        mt.solve_async("bicgstab", lam, r)

    # a zero shift, so that repeated calls leave the transpose as it is
    zero = torch.zeros(1, dtype=torch.float64, device="cuda")
    parts = {"shift_diagonal": lambda: mt.shift_diagonal_async(zero), "refresh": lambda: mt.transpose_values_async(dm),
             "adjoint_solve": adjoint_solve}
    parts.update({f"dots_{L}": (lambda L=L: dm.dots_async(ws[L], xs[L], out=outs[L])) for L in LS})
    for L in LS:                                                          # warm-up of every shape
        forward_backward(L)()
    for f in parts.values():
        f()
    torch.cuda.synchronize()
    samples = {f"{k}_{L}": [] for L in LS for k in ("forward", "forward_backward")}
    samples.update({k: [] for k in parts})
    solve_calls = max(1, a.calls // 10)
    for rnd in range(a.rounds):
        for L in (LS if rnd % 2 == 0 else LS[::-1]):
            for k in (("forward", "forward_backward") if rnd % 2 == 0 else ("forward_backward", "forward")):
                fn = forward(L) if k == "forward" else forward_backward(L)
                samples[f"{k}_{L}"].append(device_ms(fn, 1))
        for k, f in (parts.items() if rnd % 2 == 0 else list(parts.items())[::-1]):
            samples[k].append(device_ms(f, solve_calls if k == "adjoint_solve" else a.calls))
    name, power = card()
    med = {k: statistics.median(v) for k, v in samples.items()}
    print(f"{name}, power limit {power}; T' n={n} nnz={nnz}, {METHOD}, tol 1e-8, medians of {a.rounds} alternated rounds")
    out = {"card": name, "power_limit": power, "n": n, "nnz": nnz, "rounds": a.rounds, "median_ms": med, "samples_ms": samples,
           "dots_GBps": {}}
    for L in LS:
        fw, fb = med[f"forward_{L}"], med[f"forward_backward_{L}"]
        print(f"  L = {L}: forward {fw:8.2f} ms, forward + backward {fb:8.2f} ms, backward {fb - fw:8.2f} ms "
              f"({(fb - fw) / L:.2f} ms per shift)")
    for L in LS:
        byt = 16 * n * L
        out["dots_GBps"][L] = byt / (med[f"dots_{L}"] * 1e-3) / 1e9
        print(f"  dots_async over {L} vectors: {med[f'dots_{L}']:.3f} ms ({out['dots_GBps'][L]:.0f} GB/s of {byt / 1e9:.3f} GB)")
    print(f"  shift_diagonal_async {med['shift_diagonal']:.3f} ms, transpose refresh {med['refresh']:.3f} ms, adjoint solve "
          f"{med['adjoint_solve']:.2f} ms")
    dm.destroy()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
