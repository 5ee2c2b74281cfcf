"""Shared test inputs: small members of the BASELINE.json matrix families (csrc/gen.cpp)."""
import os

import numpy as np

# (name, kind, g, p0): sizes the oracle finishes in well under a second
SMALL_CASES = [
    ("stencil15_g12", "stencil15", 12, 14.0),      # Transport-like T', not diagonally dominant
    ("convdiff_g40", "convdiff", 40, 1.5),         # nonsymmetric convection-diffusion
    ("laplace5_g37", "laplace5", 37, 0.0),         # cfg 3 family, odd n
    ("random_n3001_k8", "random", 3001, 8),        # cfg 5 family, odd n
]
METHODS = ["bicgstab", "ca_bicgstab", "pipe_bicgstab", "pipe_bicgstab_rr"]
RR = dict(krr=10, nrr=3)


# shifted family (SURVEY.md 8(f) N4): (name, kind, g, p0, number of shifts, shift scale, seed index); sigma_j = (j + 1) * scale.
# The reference drivers use scale = 0.01 / L and seed 0 (main_shifted.c:95-99); the large-scale cases make the seed (the most
# diagonally dominant system) converge first, which exercises seed switching (shifted_switching_solver.c:490-527).
SHIFTED_CASES = [
    ("sh_stencil15_g12_L5", "stencil15", 12, 14.0, 5, 0.01 / 5, 0),
    ("sh_convdiff_g40_L6_switch", "convdiff", 40, 1.5, 6, 0.8, 5),
    ("sh_stencil15_g12_L4_switch", "stencil15", 12, 14.0, 4, 2.0, 3),
    ("sh_laplace5_g37_L16", "laplace5", 37, 0.0, 16, 0.01 / 16, 0),
]


def shifted_problem(O, n, ptr, col, val, L, scale, seed):
    """sigma and b = (A + sigma[seed] I) 1 as main_shifted.c:95-114 builds them."""
    sigma = (np.arange(L) + 1) * scale
    b = O.spmv(n, ptr, col, val, np.ones(n))
    O.daxpy(sigma[seed], np.ones(n), b)
    return sigma, b


# nonzero initial guesses: standard normal, or a warm start 1 + 1e-3 noise near the solution x* = 1 of b = A 1.  Either way
# r0 = b - A x0 differs from b, so the init SpMV, r# = r0, dot_zero = (r0, r0) and the b of the replacements all show.
X0_KINDS = ("normal", "warm")


def initial_guess(kind, n, seed=0):
    noise = np.random.default_rng(seed + 7919 * n).standard_normal(n)
    return noise if kind == "normal" else 1.0 + 1e-3 * noise


def initial_x_set(L, n, seed=0):
    """A nonzero initial x_set of the shifted solvers, 0.1 standard normal: no larger than the corrections they add to it."""
    return 0.1 * np.random.default_rng(seed + 7919 * n + L).standard_normal((L, n))


# the problems of tests/golden/ref_x0.npz (generator tests/golden/make_golden_x0.py): the compiled reference from nonzero
# initial guesses.  Plain solvers: (kind, g, p0, generator seed), tol, max_iter, krr / nrr of pipe_bicgstab_rr.  Shifted
# solvers: (kind, g, p0, number of shifts, shift scale, seed index), tol, max_iter; the seed switches.
X0_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_x0.npz")
X0_PLAIN, X0_PLAIN_TOL, X0_PLAIN_MAX_ITER, X0_RR = ("convdiff", 25, 2.0, 99), 1e-11, 400, dict(krr=7, nrr=2)
X0_SHIFTED, X0_SHIFTED_TOL, X0_SHIFTED_MAX_ITER = ("stencil15", 9, 14.0, 4, 2.0, 3), 1e-12, 1000


def global_csr(B, kind, g, p0, seed=12345):
    blk = B.gen_block(kind, g, p0, seed)
    ptr, col, val = B.block_to_global_csr(blk)
    return blk, blk.n, ptr, col, val


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


_BIG = {}


def big_csr(kind, g, p0, tmpdir="/dev/shm"):
    """Full-size synthetic matrix as (file, n, ptr, col, val): written once per session by the stand-alone generator
    oracle/gen_csr (binary layout of oracle.py: write_csr_bin), so neither numpy index gymnastics nor a second copy of the
    1.6 M-row matrix is needed.  The file is what oracle/_ref/ref_driver_* reads."""
    import os, subprocess, tempfile
    key = (kind, g, p0)
    if key not in _BIG:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        gen = os.path.join(root, "oracle", "gen_csr")
        if not os.path.exists(gen):
            subprocess.run(["make", "-C", os.path.join(root, "oracle"), "oracle"], check=True)
        d = tempfile.mkdtemp(dir=tmpdir if os.path.isdir(tmpdir) else None)
        f = os.path.join(d, f"{kind}_{g}.bin")
        kinds = {"stencil15": 0, "laplace5": 1, "random": 2, "convdiff": 3}
        subprocess.run([gen, str(kinds[kind]), str(int(g)), repr(float(p0)), f], check=True, capture_output=True)
        with open(f, "rb") as fh:
            n, nnz = (int(v) for v in np.fromfile(fh, dtype=np.int64, count=2))
            ptr = np.fromfile(fh, dtype=np.uint32, count=n + 1)
            col = np.fromfile(fh, dtype=np.uint32, count=nnz)
            if (n + 1 + nnz) % 2:
                np.fromfile(fh, dtype=np.uint32, count=1)
            val = np.fromfile(fh, dtype=np.float64, count=nnz)
        _BIG[key] = (f, n, ptr, col, val)
    return _BIG[key]


def x0_shifted_problem(B, O, gold_x0):
    """The shifted problem of tests/golden/ref_x0.npz: (n, ptr, col, val, b, sigma, seed, x0), x0 as stored."""
    kind, g, p0, L, scale, seed = X0_SHIFTED
    _, n, ptr, col, val = global_csr(B, kind, g, p0)
    sigma, b = shifted_problem(O, n, ptr, col, val, L, scale, seed)
    x0 = gold_x0["shifted|x0"]
    assert np.array_equal(x0, initial_x_set(L, n))
    return n, ptr, col, val, b, sigma, seed, x0
