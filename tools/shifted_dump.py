"""Digests of every shifted solver's results, for byte comparison between two builds (1 GPU).

Runs the four shifted methods on the SHIFTED_CASES of tests/helpers.py and on stencil15 g = 12 with L = 1, 513, 946, 971 and
8192 shifts (sigma_j = (j + 1) 0.01 / L, seed 0), each with shift_max_iter = 3, 9 and 1000, on host vectors, on a CUDA tensor
and on a view of one at a one-element offset (every other x_j block misaligned).  b = (A + sigma_seed I) 1 is formed on the
host.  For every solve it records the SHA-256 of x_set, r and the history, the stop iterations, the final seed, the return value
and the iteration count, and writes them as JSON.  Two builds that compute the same bits write the same file.
usage: shifted_dump.py OUT.json"""
import hashlib
import json
import os
import sys

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from helpers import SHIFTED_CASES

METHODS = ("shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab")
CASES = ([(c[0], c[1], c[2], c[3], c[4], c[5], c[6]) for c in SHIFTED_CASES] +
         [(f"stencil15_g12_L{L}", "stencil15", 12, 14.0, L, 0.01 / L, 0) for L in (1, 513, 946, 971, 8192)])
MAX_ITERS = (3, 9, 1000)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main(out):
    if not torch.cuda.is_available():
        sys.exit("shifted_dump: no CUDA device")
    B.set_options(quiet=1, autotune=0, shift_error=0, shift_tol=1e-12)
    res = {}
    for name, kind, g, p0, L, scale, seed in CASES:
        blk = B.gen_block(kind, g, p0)
        n = blk.n
        ptr, col, val = B.block_to_global_csr(blk)
        sigma = (np.arange(L) + 1) * scale
        b = sp.csr_matrix((val, col, ptr), shape=(n, n)) @ np.ones(n) + sigma[seed] * np.ones(n)
        dm = B.DeviceMatrix(blk)
        try:
            for method in METHODS:
                for mi in MAX_ITERS:
                    B.set_options(shift_max_iter=mi)
                    for path in ("host", "device", "device+1"):
                        if path == "host":
                            x, r = np.zeros((L, n)), b.copy()
                            ret, st = dm.shifted_solve(method, x, r, sigma, seed)
                        else:
                            off = 1 if path == "device+1" else 0
                            buf = torch.zeros(L * n + off, dtype=torch.float64, device="cuda")
                            xt, rt = buf[off:].view(L, n), torch.from_numpy(b.copy()).cuda()
                            torch.cuda.synchronize()
                            ret, st = dm.shifted_solve(method, xt, rt, sigma, seed)
                            x, r = xt.cpu().numpy(), rt.cpu().numpy()
                            del buf, xt, rt
                        fseed, stop = B.last_shift_info(L)
                        res[f"{name}|{method}|{mi}|{path}"] = dict(
                            ret=int(ret), iters=int(st["iters"]), seed=int(fseed), stop=digest(stop.astype(np.int32)),
                            x=digest(x), r=digest(r), hist=digest(B.last_history()))
                    print(f"[shifted-dump] {name} {method} max_iter={mi}: "
                          f"{res[f'{name}|{method}|{mi}|host']['iters']} iterations", flush=True)
        finally:
            dm.destroy()
    with open(out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"[shifted-dump] {len(res)} solves -> {out}", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
