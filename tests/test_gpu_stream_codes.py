"""16-bit column codes in the matrix stream of the persistent kernel (-m gpu; csrc/mega.cu).  A streaming CTA whose columns
fit a 16-bit window streams 10 bytes per entry (8-byte value + 2-byte code) instead of 12.  The arithmetic does not change, so
a coded run and a run forced to 32-bit columns (DeviceMatrix.stream_codes(False)) must agree bit for bit: x, r, the residual
history and the iteration count.  `coded_ctas` says how many CTAs really streamed codes."""
import numpy as np
import pytest
import scipy.sparse as sp

from helpers import METHODS, RR, SMALL_CASES, global_csr

pytestmark = pytest.mark.gpu

TOL = 1e-10


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count       # one persistent CTA per SM


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, tol=TOL, max_iter=1000, cache=1, mega=1, resident=0, mega_lanes=0)
    yield
    B.set_options(resident=1, tol=1e-15, max_iter=1000, mega=1, mega_lanes=0)


def _run(B, dm, method, n, codes):
    """One solve of A x = A 1 from x0 = 0: (iterations, x, r, history, coded CTAs)."""
    dm.stream_codes(codes)
    r = dm.spmv(np.ones(n))
    x = np.zeros(n)
    kw = RR if method.endswith("rr") else {}
    it, st = dm.solve(method, x, r, **kw)
    assert st["kernel_launches"] <= 8                         # the loop ran as the persistent kernel
    return it, x, r, B.last_history(), dm.coded_ctas()


def _identical(coded, plain):
    it1, x1, r1, h1, n1 = coded
    it0, x0, r0, h0, n0 = plain
    assert n0 == 0 and n1 > 0
    assert it1 == it0
    assert np.array_equal(h1, h0)
    assert np.array_equal(x1, x0)
    assert np.array_equal(r1, r0)


def _owning_ctas(B, dm, n):
    """CTAs that own rows: on these small matrices every such CTA keeps its slice resident when allowed to."""
    B.set_options(resident=1)
    try:
        _run(B, dm, "bicgstab", n, True)
        return dm.resident_ctas()
    finally:
        B.set_options(resident=0)


def _cases():
    return SMALL_CASES + [("laplace5_g300", "laplace5", 300, 0.0)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name,kind,g,p0", _cases())
def test_codes_bit_identical_to_32bit_columns(B, name, kind, g, p0, method):
    blk, n, *_ = global_csr(B, kind, g, p0)
    dm = B.DeviceMatrix(blk)
    try:
        coded = _run(B, dm, method, n, True)
        plain = _run(B, dm, method, n, False)
        owning = _owning_ctas(B, dm, n)
    finally:
        dm.destroy()
    _identical(coded, plain)
    assert coded[4] == owning, (coded[4], owning)              # every CTA that owns rows streamed codes
    assert np.abs(coded[1] - 1).max() < 1e-6


def test_transport_at_bench_size_every_cta_coded(B):
    """T' at the size of the benchmark (117^3 = 1.6 M rows, 23.6 M entries), 50 iterations: every CTA's window (~12 k own
    rows + 2 x 13 807 columns of stencil reach) fits 16 bits."""
    blk = B.gen_block("stencil15", 117, 14.0)
    n = blk.n
    B.set_options(tol=0.0, max_iter=50)
    dm = B.DeviceMatrix(blk)
    try:
        coded = _run(B, dm, "bicgstab", n, True)
        plain = _run(B, dm, "bicgstab", n, False)
    finally:
        dm.destroy()
    assert coded[4] == _sm_count()
    _identical(coded, plain)


def test_wide_windows_mix_coded_and_32bit_ctas(B, O):
    """Band matrix whose first rows also reference a column 100 000 places away (the pattern of
    test_gpu_resident.py::test_ctas_with_wide_column_windows_keep_streaming), everything streamed: the CTAs owning those rows
    cannot code their columns in 16 bits and stream 32-bit columns, the others stream codes -- in the same launch."""
    n = 150000
    rng = np.random.default_rng(11)
    off = [-300, -1, 1, 300]
    diags = [-(0.2 + 0.6 * rng.random(n - abs(o))) for o in off]
    A = sp.diags(diags, off, shape=(n, n), format="lil")
    for i in range(3000):
        A[i, i + 100000] = -0.5
    A = sp.csr_matrix(A)
    A = sp.csr_matrix(A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 0.5 + rng.random(n)))
    A.sort_indices()
    blk = B.blocks_from_csr(n, A.indptr, A.indices, A.data)
    ptr, col, val = A.indptr, A.indices, A.data
    ref = O.solve("bicgstab", n, ptr, col, val, O.spmv(n, ptr, col, val, np.ones(n)), tol=TOL, max_iter=1000)
    dm = B.DeviceMatrix(blk)
    try:
        coded = _run(B, dm, "bicgstab", n, True)
        plain = _run(B, dm, "bicgstab", n, False)
    finally:
        dm.destroy()
    _identical(coded, plain)
    assert 0 < coded[4] < _sm_count()                         # mixed: some CTAs coded, some 32-bit
    it, x, _, h, _ = coded
    m = min(10, it, ref["iters"])
    got, want = np.sqrt(h[1:m + 1]), np.sqrt(ref["hist"][1:m + 1])
    assert np.all(np.abs(got - want) <= 1e-10 * want + 1e-15), (got, want)
    assert abs(it - ref["iters"]) <= max(2, int(0.02 * ref["iters"]))
    assert np.abs(x - 1).max() < 1e-6


def _ragged(n, seed, max_len):
    rng = np.random.default_rng(seed)
    rows, cols, vals = [], [], []
    for i in range(n):
        k = int(rng.integers(0, max_len + 1))
        if k:
            c = rng.choice(n, size=min(k, n), replace=False)
            c = c[c != i]
            rows += [i] * c.size; cols += list(c); vals += list(-rng.random(c.size))
    A = sp.csr_matrix((vals, (rows, cols)), shape=(n, n))
    return A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0)


@pytest.mark.parametrize("n,long_rows", [(12000, [7]), (40000, [0, 20011, 39999])])
def test_chunked_long_rows_bit_identical(B, n, long_rows):
    """Rows longer than a stage (the shapes of test_gpu_edge.py::test_rows_longer_than_a_stage) are multiplied chunk by chunk by
    the whole CTA; the chunk path decodes the codes too."""
    A = sp.lil_matrix(_ragged(n, 5, 6))
    for r in long_rows:
        A[r, :] = -2.0 / n
        A[r, r] = 4.0
    A = sp.csr_matrix(A)
    A.sort_indices()
    blk = B.blocks_from_csr(n, A.indptr, A.indices, A.data)
    dm = B.DeviceMatrix(blk)
    try:
        coded = _run(B, dm, "bicgstab", n, True)
        plain = _run(B, dm, "bicgstab", n, False)
    finally:
        dm.destroy()
    _identical(coded, plain)
    assert np.abs(coded[1] - 1).max() < 1e-7


@pytest.mark.parametrize("lanes", [4, 8, 32])
@pytest.mark.parametrize("method", ["bicgstab", "pipe_bicgstab"])
def test_forced_lanes_bit_identical(B, lanes, method):
    """The multi-lane SpMV variants of the persistent kernel (BICG_MEGA_LANES) decode the codes in the same way."""
    blk, n, *_ = global_csr(B, "stencil15", 40, 14.0)
    B.set_options(mega_lanes=lanes)
    dm = B.DeviceMatrix(blk)                                   # the plan (and its lanes) is made with the handle
    try:
        coded = _run(B, dm, method, n, True)
        plain = _run(B, dm, method, n, False)
    finally:
        dm.destroy()
        B.set_options(mega_lanes=0)
    _identical(coded, plain)
    assert np.abs(coded[1] - 1).max() < 1e-6
