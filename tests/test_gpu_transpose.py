"""GPU: A^T of a resident matrix as a handle of its own (bicg_matrix_create_transpose) and the refresh of its values from the
source (bicg_matrix_transpose_values, _async).  The contract: every result on the transpose is bit for bit that of a handle
created from the blocks of the global CSR of A^T built by a stable sort of A's triplets by (column, row) -- spmv, multiply,
every solve and shifted solve, their histories and which CTAs ran resident, coded and packed -- on every loop path, after
value updates on the source, synchronous, stream-ordered and captured into a CUDA graph."""
import os

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp

from helpers import METHODS, RR, initial_guess, initial_x_set

pytestmark = pytest.mark.gpu

SHIFTED = ["shifted_lopbicg_switching", "shifted_lopbicg", "shifted_lopbicgstab", "shifted_pipe_lopbicgstab"]
CASES = ["convdiff", "random", "tprime", "golden", "handmade"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "test_shifted_convdiff16.mtx")


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, tol=1e-10, max_iter=300, mega=1, resident=1, mega_lanes=0, shift_tol=1e-12,
                  shift_max_iter=300, shift_error=0)
    yield
    B.set_options(tol=1e-15, max_iter=1000, mega=1, resident=1, mega_lanes=0, shift_max_iter=1000)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def transposed_csr(n, ptr, col, val):
    """The global CSR of A^T: A's triplets stably sorted by (column, row), so equal (i, j) keep their order in row i."""
    ptr, col = np.asarray(ptr, dtype=np.int64), np.asarray(col, dtype=np.int64)
    rows = np.repeat(np.arange(n), np.diff(ptr))
    order = np.lexsort((rows, col))                     # stable: the last key is the primary one
    tptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(tptr, col + 1, 1)
    return np.cumsum(tptr), rows[order], np.asarray(val, dtype=np.float64)[order]


def _handmade():
    """7 x 7, unsorted rows, a duplicate (2, 4) twice, an explicit zero at (5, 1), and column 6 empty."""
    rows = [[(0, 4.0), (3, -1.0)], [(1, 5.0), (0, -0.5)], [(4, 1.25), (2, 6.0), (4, -0.75), (1, 0.5)], [(3, 7.0), (5, 2.0)],
            [(4, 3.0), (0, 1.0), (2, -2.0)], [(1, 0.0), (5, 8.0)], [(5, -1.5), (3, 0.25)]]
    ptr = np.cumsum([0] + [len(r) for r in rows])
    col = np.array([c for r in rows for c, _ in r], dtype=np.int64)
    val = np.array([v for r in rows for _, v in r])
    return 7, ptr, col, val


def _case_csr(B, case):
    """(n, ptr, col, val) of the global CSR of A; every case but the hand-made one is nonsymmetric in values or pattern."""
    if case == "handmade":
        return _handmade()
    if case == "golden":
        A = sp.csr_matrix(scipy.io.mmread(GOLDEN))
        A.sort_indices()
        return A.shape[0], A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64)
    kind, g, p0 = {"convdiff": ("convdiff", 24, 2.0), "random": ("random", 2500, 12), "tprime": ("stencil15", 18, 14.0)}[case]
    blk = B.gen_block(kind, g, p0)
    ptr, col, val = B.block_to_global_csr(blk)
    if case == "tprime":                              # the stencil is symmetric: scale the values by row so A^T != A
        val = val * (1.0 + (np.repeat(np.arange(blk.n), np.diff(ptr)) % 5) / 16.0)
    return blk.n, np.asarray(ptr, dtype=np.int64), np.asarray(col, dtype=np.int64), np.asarray(val, dtype=np.float64)


def _fresh_t(B, n, ptr, col, val):
    tp, tc, tv = transposed_csr(n, ptr, col, val)
    return B.DeviceMatrix(B.blocks_from_csr(n, tp, tc, tv))


def _run(B, dm, method, b, x0):
    x, r = x0.copy(), b.copy()
    it, _ = dm.solve(method, x, r, **(RR if method.endswith("rr") else {}))
    return dict(it=it, x=_bits(x), r=_bits(r), hist=_bits(B.last_history()),
                ctas=(dm.resident_ctas(), dm.coded_ctas(), dm.packed_ctas()))


def _shifted(B, dm, method, x0s, b, sigma, seed):
    x, r = x0s.copy(), b.copy()
    k, st = dm.shifted_solve(method, x, r, sigma, seed)
    seed_end, stop = B.last_shift_info(sigma.size)
    return dict(k=k, iters=st["iters"], seed=seed_end, stop=list(stop), x=_bits(x), r=_bits(r), hist=_bits(B.last_history()))


def _same_everywhere(B, mt, fresh, n, what, solves=True):
    """spmv, a batched shifted multiply, every method and every shifted method: bit-identical on mt and fresh."""
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n)
    assert _bits(mt.spmv(x)) == _bits(fresh.spmv(x)), what
    xs, ys = rng.standard_normal((3, n)), rng.standard_normal((3, n))
    sig = np.array([0.0, 0.5, -1.25])
    assert _bits(mt.multiply(xs, ys.copy(), 0.75, -0.5, sig)) == _bits(fresh.multiply(xs, ys.copy(), 0.75, -0.5, sig)), what
    if not solves:
        return
    b = fresh.spmv(np.ones(n))
    x0 = initial_guess("warm", n)
    for method in METHODS:
        got, want = _run(B, mt, method, b, x0), _run(B, fresh, method, b, x0)
        assert got == want, (what, method)
    sigma, seed = np.array([0.0, 0.3, 1.1]), 1
    x0s = initial_x_set(sigma.size, n)
    for method in SHIFTED:
        assert _shifted(B, mt, method, x0s, b, sigma, seed) == _shifted(B, fresh, method, x0s, b, sigma, seed), (what, method)


@pytest.mark.parametrize("resident", [0, 1])
@pytest.mark.parametrize("mega", [0, 1, 2])
@pytest.mark.parametrize("case", CASES)
def test_transpose_equals_fresh_handle(B, case, mega, resident):
    B.set_options(mega=mega, resident=resident)
    n, ptr, col, val = _case_csr(B, case)
    m = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt = m.transpose()
    fresh = _fresh_t(B, n, ptr, col, val)
    try:
        assert (mt.blk.n_loc, mt.blk.diag.nz, mt.blk.offd.nz) == (n, int(ptr[-1]), 0)
        _same_everywhere(B, mt, fresh, n, (case, mega, resident))
        # against scipy, and the adjoint identity (y, A x) = (A^T y, x)
        A = sp.csr_matrix((val, col, ptr), shape=(n, n))
        rng = np.random.default_rng(3)
        x, y = rng.standard_normal(n), rng.standard_normal(n)
        aty, ax = mt.spmv(y), m.spmv(x)
        scale = abs(A).T @ abs(y)
        assert np.all(np.abs(aty - A.T @ y) <= 1e-14 * scale + 1e-300), case
        bound = 1e-13 * float(abs(y) @ (abs(A) @ abs(x)))
        assert abs(float(y @ ax) - float(aty @ x)) <= bound, case
    finally:
        for d in (m, mt, fresh):
            d.destroy()


def _shift_host(n, ptr, col, val, sigma):
    """csr_shift_diagonal on a global CSR: sigma added to the first entry of every row whose column is that row."""
    val = val.copy()
    for i in range(n):
        hits = np.nonzero(col[ptr[i]:ptr[i + 1]] == i)[0]
        val[ptr[i] + hits[0]] += sigma
    return val


@pytest.mark.parametrize("refresh", ["sync", "async"])
@pytest.mark.parametrize("case", CASES)
def test_refresh_after_updates(B, case, refresh):
    """set_values and shift_diagonal on m, then the refresh: mt equals a fresh transpose of m's new values."""
    torch = _torch()
    B.set_options(mega=1, resident=1)
    n, ptr, col, val = _case_csr(B, case)
    m = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt = m.transpose()
    try:
        val2 = val * (1.0 + ((np.arange(val.size) * 5 + 1) % 7) / 64.0)
        steps = [("set", val2)]
        if case != "handmade":                      # column 6 is empty: row 6 has no diagonal entry
            steps.append(("shift", _shift_host(n, ptr, col, val2, 0.625)))
        for kind, want_val in steps:
            if kind == "set":
                if refresh == "sync":
                    m.set_values(val2)
                else:
                    m.set_values_async(torch.from_numpy(val2).cuda())
            else:
                m.shift_diagonal(0.625)
            if refresh == "sync":
                mt.transpose_values(m)
            else:
                mt.transpose_values_async(m)
                torch.cuda.current_stream().synchronize()
            fresh = _fresh_t(B, n, ptr, col, want_val)
            try:
                _same_everywhere(B, mt, fresh, n, (case, refresh, kind), solves=kind == "shift" or case == "handmade")
            finally:
                fresh.destroy()
    finally:
        m.destroy()
        mt.destroy()


def test_captured_update_refresh_and_solve_replay(B):
    """One graph of {reset x, r; m.set_values_async(buf); mt.transpose_values_async(m); mt.solve_async}, replayed with three
    value sets: every replay equals the synchronous sequence on a second pair of handles."""
    torch = _torch()
    n, ptr, col, val = _case_csr(B, "convdiff")
    sets = [val * (1.0 + ((np.arange(val.size) * (2 * k + 1) + k) % 7) / 64.0) for k in (2, 3, 4)]
    method = "bicgstab"
    m = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt = m.transpose()
    m2 = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt2 = m2.transpose()
    try:
        mt.prepare_async(method)
        x0 = torch.from_numpy(initial_guess("warm", n)).cuda()
        b = torch.ones(n, dtype=torch.float64, device="cuda")
        buf = torch.from_numpy(val.copy()).cuda()
        x, r, res = x0.clone(), b.clone(), torch.zeros(24, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            x.copy_(x0)
            r.copy_(b)
            m.set_values_async(buf)
            mt.transpose_values_async(m)
            mt.solve_async(method, x, r, result=res)
        for vals in sets:
            buf.copy_(torch.from_numpy(vals))
            g.replay()
            torch.cuda.synchronize()
            got = dict(x=_bits(x), r=_bits(r), rec=B.decode_result(res), hist=_bits(mt.history()))
            m2.set_values(vals)
            mt2.transpose_values(m2)
            fx, fr = x0.clone(), b.clone()
            fres = mt2.solve_async(method, fx, fr)
            torch.cuda.synchronize()
            want = dict(x=_bits(fx), r=_bits(fr), rec=B.decode_result(fres), hist=_bits(mt2.history()))
            assert got == want
            fresh = _fresh_t(B, n, ptr, col, vals)
            try:
                assert _bits(mt.spmv(np.ones(n))) == _bits(fresh.spmv(np.ones(n)))
            finally:
                fresh.destroy()
        del g
    finally:
        for d in (m, mt, m2, mt2):
            d.destroy()


def test_wrong_source_is_refused_and_changes_nothing(B):
    n, ptr, col, val = _case_csr(B, "random")
    m = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    other = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val * 2.0))
    mt = m.transpose()
    try:
        x = np.random.default_rng(1).standard_normal(n)
        before = _bits(mt.spmv(x))
        for src in (other, mt):
            with pytest.raises(ValueError, match="failed with -1"):
                mt.transpose_values(src)
            with pytest.raises(ValueError, match="failed with -1"):
                mt.transpose_values_async(src)
        _torch().cuda.synchronize()
        assert _bits(mt.spmv(x)) == before
    finally:
        for d in (m, other, mt):
            d.destroy()


def test_transpose_outlives_its_source(B):
    n, ptr, col, val = _case_csr(B, "golden")
    m = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt = m.transpose()
    fresh = _fresh_t(B, n, ptr, col, val)
    try:
        m.destroy()
        with pytest.raises(ValueError):
            mt.transpose_values(m)                   # a destroyed source is not a source any more
        _same_everywhere(B, mt, fresh, n, "after destroy")
        mtt = mt.transpose()                         # (A^T)^T is A again, with A's order of duplicates
        a = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
        try:
            assert _bits(mtt.spmv(np.ones(n))) == _bits(a.spmv(np.ones(n)))
        finally:
            mtt.destroy()
            a.destroy()
    finally:
        mt.destroy()
        fresh.destroy()
