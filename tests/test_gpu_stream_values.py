"""Packed values in the matrix stream of the persistent kernel (-m gpu; csrc/mega.cu).  A streaming CTA that streams 16-bit
column codes and whose entries take at most 16 sign / exponent fields streams every value as a 4-bit index into its CTA's table
of fields plus the 52 mantissa bits: 7 bytes instead of 8, 9 per entry with the code.  The split is done on the bit pattern and
the arithmetic does not change, so a packed run and a run forced to 8-byte values (DeviceMatrix.stream_values(False), the codes
kept) must agree bit for bit: x, r, the residual history and the iteration count.  `packed_ctas` says how many CTAs really
streamed packed values."""
import numpy as np
import pytest
import scipy.sparse as sp

from helpers import METHODS, RR, SMALL_CASES, global_csr

pytestmark = pytest.mark.gpu

TOL = 1e-10
PACK_MIN_MEAN_ROW = 8.0          # csrc/matrix.cu: plans of matrices with shorter rows on average stream 8-byte values


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count       # one persistent CTA per SM


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, tol=TOL, max_iter=1000, cache=1, mega=1, resident=0, mega_lanes=0)
    yield
    B.set_options(resident=1, tol=1e-15, max_iter=1000, mega=1, mega_lanes=0)


def _run(B, dm, method, n, packed, b=None):
    """One solve of A x = b (default A 1) from x0 = 0: (iterations, x, r, history, coded CTAs, packed CTAs)."""
    dm.stream_values(packed)
    r = dm.spmv(np.ones(n)) if b is None else b.copy()
    x = np.zeros(n)
    kw = RR if method.endswith("rr") else {}
    it, st = dm.solve(method, x, r, **kw)
    assert st["kernel_launches"] <= 8                         # the loop ran as the persistent kernel
    return it, x, r, B.last_history(), dm.coded_ctas(), dm.packed_ctas()


def _identical(packed, plain, packs=True):
    it1, x1, r1, h1, c1, n1 = packed
    it0, x0, r0, h0, c0, n0 = plain
    assert n0 == 0 and (n1 > 0) == packs
    assert c1 == c0 and n1 <= c1                              # only CTAs that stream codes pack their values
    assert it1 == it0
    assert np.array_equal(h1, h0)
    assert np.array_equal(x1, x0)
    assert np.array_equal(r1, r0)


def _both(B, blk, n, method="bicgstab", b=None, packs=True):
    dm = B.DeviceMatrix(blk)
    try:
        packed = _run(B, dm, method, n, True, b)
        plain = _run(B, dm, method, n, False, b)
    finally:
        dm.destroy()
    _identical(packed, plain, packs)
    return packed


def _blk(B, A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return B.blocks_from_csr(A.shape[0], A.indptr, A.indices, A.data)


def _cases():
    return SMALL_CASES + [("laplace5_g300", "laplace5", 300, 0.0)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name,kind,g,p0", _cases())
def test_packed_values_bit_identical_to_8byte_values(B, name, kind, g, p0, method):
    blk, n, ptr, *_ = global_csr(B, kind, g, p0)
    packs = ptr[-1] / n >= PACK_MIN_MEAN_ROW
    packed = _both(B, blk, n, method, packs=packs)
    assert packed[5] == (packed[4] if packs else 0), packed[4:]   # every CTA that streams codes packs its values
    assert np.abs(packed[1] - 1).max() < 1e-6


def test_transport_at_bench_size_every_cta_packed(B):
    """T' at the size of the benchmark (117^3 = 1.6 M rows, 23.6 M entries), 50 iterations: every CTA's entries take three
    sign / exponent fields (the diagonal 14 and off-diagonals -(0.5 + u) in two binades)."""
    blk = B.gen_block("stencil15", 117, 14.0)
    B.set_options(tol=0.0, max_iter=50)
    packed = _both(B, blk, blk.n)
    assert packed[5] == packed[4] == _sm_count()


def _band(n, seed):
    """Band matrix, 9 entries per row: off-diagonals -(0.5 + 0.5 u) (one field) and a diagonal in [8.5, 15.5) (one field)."""
    rng = np.random.default_rng(seed)
    off = [-600, -300, -2, -1, 1, 2, 300, 600]
    A = sp.diags([-(0.5 + 0.5 * rng.random(n - abs(o))) for o in off], off, shape=(n, n), format="lil")
    A.setdiag(8.5 + 7.0 * rng.random(n))
    return A


@pytest.mark.parametrize("fields", [16, 17])
def test_sixteen_fields_pack_seventeen_fall_back(B, O, fields):
    """The first rows (owned by CTA 0) also hold off-diagonals in fields - 2 further binades, so CTA 0's entries take exactly
    `fields` sign / exponent fields.  With 16 it packs like every other CTA; with 17 it streams 8-byte values in the same
    launch as the packed CTAs.  Also checked against the oracle."""
    n = 150000
    A = _band(n, 21)
    rng = np.random.default_rng(22)
    for k in range(fields - 2):                               # magnitudes 2^-2 .. 2^-16: still diagonally dominant
        A[k, k + 1] = -(2.0 ** -(k + 2)) * (1.0 + 0.5 * rng.random())
    A = sp.csr_matrix(A)
    A.sort_indices()
    blk = _blk(B, A)
    packed = _both(B, blk, n)
    assert packed[4] == _sm_count()
    assert packed[5] == (packed[4] if fields <= 16 else packed[4] - 1)
    ptr, col, val = A.indptr, A.indices, A.data
    ref = O.solve("bicgstab", n, ptr, col, val, O.spmv(n, ptr, col, val, np.ones(n)), tol=TOL, max_iter=1000)
    it, x, _, h, _, _ = packed
    m = min(10, it, ref["iters"])
    got, want = np.sqrt(h[1:m + 1]), np.sqrt(ref["hist"][1:m + 1])
    assert np.all(np.abs(got - want) <= 1e-10 * want + 1e-15), (got, want)
    assert abs(it - ref["iters"]) <= max(2, int(0.02 * ref["iters"]))
    assert np.abs(x - 1).max() < 1e-6


def test_zeros_subnormals_and_largest_values_round_trip(B):
    """Stored +0.0 and -0.0, subnormals (exponent field 0, like the zeros) and the largest finite values of both signs.  The
    largest values sit in a column whose row is decoupled and has b = 0, so x, r, p, q stay exactly 0 there and the values
    multiply zeros: the solve stays finite, and a value decoded as inf or nan would turn the rows into nan."""
    n = 150000
    z = 1000                                                  # the decoupled row / column, in CTA 0's window
    A = sp.coo_matrix(_band(n, 31))
    keep = (A.row != z) & (A.col != z)
    big = np.finfo(np.float64).max
    extra_r = np.concatenate([[z], np.arange(40)])
    extra_c = np.concatenate([[z], np.full(40, z)])
    extra_v = np.concatenate([[1.0], np.where(np.arange(40) % 2 == 0, big, -big)])
    A = sp.csr_matrix((np.concatenate([A.data[keep], extra_v]),
                       (np.concatenate([A.row[keep], extra_r]), np.concatenate([A.col[keep], extra_c]))), shape=(n, n))
    A.sort_indices()
    specials = [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, -1e-310]
    for k, v in enumerate(specials):                          # over band entries (k, k + 1) of the first rows
        j = A.indptr[k] + np.searchsorted(A.indices[A.indptr[k]:A.indptr[k + 1]], k + 1)
        assert A.indices[j] == k + 1
        A.data[j] = v
    assert np.signbit(A.data).sum() > 0 and (A.data == 0).sum() == 2
    blk = B.blocks_from_csr(n, A.indptr, A.indices, A.data)
    ones = np.ones(n)
    ones[z] = 0.0
    b = A @ ones                                              # the largest values multiply the zero of column z
    packed = _both(B, blk, n, b=b)
    assert packed[5] == packed[4] == _sm_count()
    it, x, r, h, _, _ = packed
    assert np.all(np.isfinite(x)) and np.all(np.isfinite(r)) and np.all(np.isfinite(h))
    assert x[z] == 0.0 and np.abs(np.delete(x, z) - 1).max() < 1e-6


def test_shifted_diagonal_is_re_encoded(B):
    """csr_shift_diagonal changes the values in place and drops the cached upload: the next solve through the
    reference-facing call builds a new plan, whose table and packed values hold the shifted diagonal (14 -> 17, another
    binade).  Its results equal those of a fresh handle forced to 8-byte values."""
    import ctypes as C
    blk, n, *_ = global_csr(B, "stencil15", 40, 14.0)
    b = B.spmv_ovlap(blk, np.ones(n))
    x = np.zeros(n)
    r = b.copy()
    B.bicgstab(blk, x, r)                                     # caches the upload, packed
    B.lib.csr_shift_diagonal(C.byref(blk.diag), 3.0)
    x = np.zeros(n)
    r = b.copy()
    B.bicgstab(blk, x, r)
    h = B.last_history()
    dm = B.DeviceMatrix(blk)
    try:
        plain = _run(B, dm, "bicgstab", n, False, b)
        packed = _run(B, dm, "bicgstab", n, True, b)
    finally:
        dm.destroy()
    _identical(packed, plain)
    assert np.array_equal(h, plain[3]) and np.array_equal(x, plain[1])


def test_chunked_long_rows_bit_identical(B):
    """Rows longer than a stage are multiplied chunk by chunk by the whole CTA; the chunk path decodes packed values too."""
    n = 40000
    rng = np.random.default_rng(5)
    rows, cols = [], []
    for i in range(n):
        c = rng.choice(n, size=int(rng.integers(6, 15)), replace=False)
        c = c[c != i]
        rows += [i] * c.size
        cols += list(c)
    A = sp.csr_matrix((-(0.5 + 0.5 * rng.random(len(rows))), (rows, cols)), shape=(n, n))
    A = sp.lil_matrix(A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0))
    for r in (0, 20011, n - 1):
        A[r, :] = -2.0 / n
        A[r, r] = 4.0
    blk = _blk(B, A)
    packed = _both(B, blk, n)
    assert packed[5] == packed[4]
    assert np.abs(packed[1] - 1).max() < 1e-7


@pytest.mark.parametrize("lanes", [4, 8, 32])
@pytest.mark.parametrize("method", ["bicgstab", "pipe_bicgstab"])
def test_forced_lanes_random_block_bit_identical(B, lanes, method):
    """The multi-lane SpMV variants of the persistent kernel (BICG_MEGA_LANES) decode packed values in the same way: a random
    block of 32 entries per row whose values take few binades (off-diagonals -(0.5 + 0.5 u), diagonal in [17, 34))."""
    n = 20000
    rng = np.random.default_rng(7)
    rows = np.repeat(np.arange(n), 32)
    cols = rng.integers(0, n, size=rows.size)
    A = sp.csr_matrix((-(0.5 + 0.5 * rng.random(rows.size)), (rows, cols)), shape=(n, n))
    A.sum_duplicates()
    A.data = -(0.5 + 0.5 * rng.random(A.data.size))          # duplicates summed: back into one binade
    A = A + sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0 + rng.random(n))
    blk = _blk(B, A)
    B.set_options(mega_lanes=lanes)
    try:
        packed = _both(B, blk, n, method)                     # the plan (and its lanes) is made with the handle
    finally:
        B.set_options(mega_lanes=0)
    assert packed[5] == packed[4]
    assert np.abs(packed[1] - 1).max() < 1e-6
