"""What the per-iteration GPU tests share (tests/test_gpu_loop_state.py, tests/test_gpu_shifted_state.py): the test matrices,
the forced stand-alone SpMV variants, and the rule that holds a GPU result to the reference.

Tolerance: max-norm relative error for a vector, relative error for a scalar or a history entry, at most
max(FLOOR, FACTOR * spread), where spread is the same quantity between the reference and its exact evaluation (long-double
SpMV, fsum dots): the rounding the case itself amplifies.  A case whose spread exceeds MAX_SPREAD says nothing about the
kernel; _hold refuses it rather than loosening the bound.  Every assertion message carries the error, the spread and their
ratio (FACTOR * err / bound: below FACTOR passes)."""
import numpy as np
import scipy.sparse as sp

from helpers import global_csr

FACTOR, FLOOR, MAX_SPREAD = 32.0, 1e-13, 1e-9


# ---- matrices -------------------------------------------------------------------------------------------------------
def _csr(A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A.shape[0], A.indptr, A.indices, A.data


def _ragged(n, seed, max_len):
    """Diagonally dominant, 0 .. max_len off-diagonal entries per row (rows with none are common).  The diagonal's margin is
    random: with a constant one every row would sum to the same value, b = A 1 would be an eigenvector and BiCGStab would
    solve the system exactly in one step."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, max_len + 1, n)
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, n, rows.size)
    keep = cols != rows
    A = sp.csr_matrix((-rng.random(int(keep.sum())), (rows[keep], cols[keep])), shape=(n, n))
    A.sum_duplicates()
    return A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 0.5 + rng.random(n))


def cap_limit(threads, lanes):
    """Largest tile (entries) of the persistent kernel's plan: matrix.cu build_mega_plan, cap_limit."""
    smem_max, rpt = 222 * 1024, threads // lanes
    return (smem_max // 2 - (rpt + 8) * 4) // 12 // 32 * 32 - 64


CHUNK_N = 30000


def _chunk_rows(cap):
    """row -> length of the long rows around a stage's capacity `cap`; row 1 is empty (no entry at all)."""
    return {0: 3 * cap + 7, 1: 0, 2: cap + 1, 10000: cap - 1, 10001: cap, 20000: 2 * cap, CHUNK_N - 1: 2 * cap}


def _chunk_matrix(cap):
    """Ragged matrix with rows of cap - 1, cap, cap + 1, 2 cap and 3 cap + 7 entries: the first row of the matrix (first row
    of CTA 0) and its last row are long, and a long row follows an empty one.  A long row's entries weigh -2 / length next
    to a diagonal of 4, as in test_gpu_edge.py::test_rows_longer_than_a_stage, so the system stays well conditioned."""
    n = CHUNK_N
    A = sp.lil_matrix(_ragged(n, 5, 6))
    for r, length in _chunk_rows(cap).items():
        if length == 0:
            A.rows[r], A.data[r] = [], []
            continue
        c = np.round(np.linspace(0, n - 2, length - 1)).astype(np.int64)
        c = np.sort(np.append(c + (c >= r), r))
        A.rows[r] = c.tolist()
        A.data[r] = np.where(c == r, 4.0, -2.0 / length).tolist()
    return _csr(A)


def _window_matrix(far_col):
    """Band matrix (bandwidth 300) whose row 0 also holds column far_col: CTA 0's column window spans far_col + 1 columns."""
    n = 150000
    rng = np.random.default_rng(11)
    off = [-300, -1, 1, 300]
    A = sp.diags([-(0.2 + 0.6 * rng.random(n - abs(o))) for o in off], off, shape=(n, n), format="lil")
    A[0, far_col] = -0.5
    A = sp.csr_matrix(A)
    return _csr(A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 0.5 + rng.random(n)))


def _gen(kind, g, p0):
    def make(B):
        _, n, ptr, col, val = global_csr(B, kind, g, p0)
        return n, ptr, col, val
    return make


MATRICES = {
    "stencil15_g60": _gen("stencil15", 60, 14.0),          # T', 216 k rows: ~4 tiles per CTA against 2 stages
    "stencil15_g58": _gen("stencil15", 58, 14.0),          # every CTA's slice fits its shared memory
    "stencil15_g40": _gen("stencil15", 40, 14.0),
    "stencil15_g20": _gen("stencil15", 20, 14.0),
    "random_n20011_k32": _gen("random", 20011, 32),
    "stencil15_g117": _gen("stencil15", 117, 14.0),        # the benchmark matrix
    "ragged_4001": lambda B: _csr(_ragged(4001, 3, 30)),
    "window_65535": lambda B: _window_matrix(65535),
    "window_65536": lambda B: _window_matrix(65536),
    **{f"chunk_cap{cap_limit(512, l)}": (lambda B, c=cap_limit(512, l): _chunk_matrix(c)) for l in (1, 4, 32)},
    **{f"small_n{n}": (lambda B, n=n: _csr(_ragged(n, n, 8))) for n in (17, 2111, 2112, 2113)},
}
_MAT = {}
BIG = 1 << 20                                              # rows: matrices this large and their states are not kept


def matrix(B, name):
    if name in _MAT:
        return _MAT[name]
    m = MATRICES[name](B)
    if m[0] < BIG:
        _MAT[name] = m
    return m


# ---- comparison -----------------------------------------------------------------------------------------------------
def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(float(np.abs(b).max()), 1e-300))


def _hold(what, got, want, exact, at_least=0.0):
    """err <= max(FLOOR, FACTOR * spread); returns (FACTOR * err / bound, what): the ratio err / spread where the spread
    sets the bound."""
    err, spread = _rel(got, want), max(_rel(exact, want), at_least)
    assert spread <= MAX_SPREAD, f"{what}: the case's own rounding spread {spread:.3g} exceeds {MAX_SPREAD:g}: fix the case"
    bound = max(FLOOR, FACTOR * spread)
    ratio = FACTOR * err / bound
    assert err <= bound, f"{what}: err {err:.3g} > bound {bound:.3g} (spread {spread:.3g}, ratio {ratio:.3g})"
    return ratio, what


# ---- kernel-per-phase path: every stand-alone SpMV variant ------------------------------------------------------------
TMA = [(l, t, 3) for l in (1, 2, 4, 8, 16, 32) for t in (128, 256, 512)] + [(1, 256, 2), (1, 256, 4), (16, 512, 2), (32, 128, 4)]
STANDALONE = ([(f"tma-l{l}-t{t}-s{s}", "stencil15_g20", dict(spmv="tma", spmv_lanes=l, spmv_threads=t, spmv_stages=s), 0, l)
               for l, t, s in TMA] +
              [(f"rowsplit-l{l}", "stencil15_g20", dict(spmv="rowsplit", spmv_lanes=l), 1, l) for l in (1, 4, 32)] +
              [(f"rowsplit-l{l}-chunk", f"chunk_cap{cap_limit(512, 1)}", dict(spmv="rowsplit", spmv_lanes=l), 1, l) for l in (1, 4, 32)] +
              [("tma-l1-ragged", "ragged_4001", dict(spmv="tma", spmv_lanes=1), 0, 1)])
