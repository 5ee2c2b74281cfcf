"""Digests of every solver loop's results, for byte comparison between two builds (1 GPU).

Runs the four methods on the plan shapes of tests/test_gpu_loop_state.py: the persistent kernel streaming 16-bit codes and
forced to 32-bit columns, resident, with 256 threads, with 4, 8 and 32 lanes on the stencil and on the random matrix, and on
chunk tiles for 1, 4 and 32 lanes (codes and 32-bit columns); then the kernel-per-phase path on every forced stand-alone
SpMV of tests/state_check.py's STANDALONE table.  b = A 1 is formed on the host, x0 = 0.  Every case is solved with
max_iter = 3 (tol = 0) and to tol = 1e-10 (max_iter = 1000); each solve records the SHA-256 of x, r and the history and the
iteration count.  For each stand-alone variant it also records the SHA-256 of y = A 1.  Writes them as JSON: two builds
that compute the same bits write the same file.
usage: loop_dump.py OUT.json"""
import hashlib
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpi_bicgstab_b200 as B
from helpers import METHODS
from state_check import STANDALONE, cap_limit, matrix

DEFAULTS = dict(quiet=1, tol=1e-15, max_iter=1000, mega=1, resident=1, mega_threads=0, mega_lanes=0, spmv="auto",
                spmv_lanes=0, spmv_threads=0, spmv_stages=0, autotune=0)
RR = dict(krr=2, nrr=2)
SOLVES = (("k3", dict(tol=0.0, max_iter=3)), ("tol", dict(tol=1e-10, max_iter=1000)))

# (id, matrix, options at plan time, stream codes: None = as planned, False = forced 32-bit columns)
PERSISTENT = [
    ("streaming", "stencil15_g60", dict(resident=0), None),
    ("streaming-32bit", "stencil15_g60", dict(resident=0), False),
    ("resident", "stencil15_g58", dict(resident=1), None),
    ("threads256", "stencil15_g60", dict(resident=0, mega_threads=256), None),
    *[(f"lanes{l}-stencil", "stencil15_g40", dict(mega_lanes=l), None) for l in (4, 8, 32)],
    *[(f"lanes{l}-random", "random_n20011_k32", dict(mega=2, mega_lanes=l), None) for l in (4, 8, 32)],
    *[(f"chunk-l{l}{tag}", f"chunk_cap{cap_limit(512, l)}", dict(mega_lanes=l), codes)
      for l in (1, 4, 32) for tag, codes in (("", None), ("-32bit", False))],
]
CASES = ([(f"mega|{i}", name, opts, codes) for i, name, opts, codes in PERSISTENT] +
         [(f"phase|{i}", name, dict(opts, mega=0), None) for i, name, opts, _, _ in STANDALONE])


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main(out):
    res = {}
    for cid, name, opts, codes in CASES:
        B.set_options(**(DEFAULTS | opts))
        n, ptr, col, val = matrix(B, name)
        b = sp.csr_matrix((val, col, ptr), shape=(n, n)) @ np.ones(n)
        dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
        try:
            if codes is not None:
                dm.stream_codes(codes)
            if cid.startswith("phase|"):
                res[f"{cid}|A1"] = digest(dm.spmv(np.ones(n)))
            for method in METHODS:
                kw = RR if method.endswith("rr") else {}
                for tag, stop in SOLVES:
                    B.set_options(**stop)
                    x, r = np.zeros(n), b.copy()
                    it, st = dm.solve(method, x, r, **kw)
                    res[f"{cid}|{method}|{tag}"] = dict(iters=int(it), launches=int(st["kernel_launches"]), x=digest(x), r=digest(r), hist=digest(B.last_history()))
            if cid.startswith("mega|"):
                res[f"{cid}|plan"] = dict(coded_ctas=dm.coded_ctas(), resident_ctas=dm.resident_ctas())
            print(f"[loop-dump] {cid} ({name}): " +
                  ", ".join(f"{m} {res[f'{cid}|{m}|tol']['iters']}" for m in METHODS), flush=True)
        finally:
            dm.destroy()
    B.set_options(**DEFAULTS)
    with open(out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"[loop-dump] {len(res)} entries -> {out}", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
