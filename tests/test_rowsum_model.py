"""The bitwise row-sum model (tests/rowsum_model.py) held on the CPU: its fma against Fraction on adversarial triples, its row
sums at every group width against a plain per-row loop built on the Fraction fma, its exact row sums against Fraction sums.
The GPU tests of tests/test_gpu_rowsum_bits.py trust the model only as far as these tests hold it."""
import math
from fractions import Fraction

import numpy as np
import pytest

import rowsum_model as M

LANES = [1, 2, 4, 8, 16, 32]
MAX = np.finfo(np.float64).max
TINY = np.finfo(np.float64).tiny                 # 2^-1022, the smallest normal


def _ref(a, b, c):
    return np.array([M._fma_exact(x, y, z) for x, y, z in zip(a, b, c)])


def _same_bits(got, want):
    return np.ascontiguousarray(got).view(np.uint64) == np.ascontiguousarray(want).view(np.uint64)


def _short(rng, n, bits=20):
    """doubles with at most `bits` significant bits: products of two of them are exact"""
    return rng.integers(1, 2 ** bits, n) * 2.0 ** rng.integers(-60, 40, n) * rng.choice([-1.0, 1.0], n)


def _triples(seed=1):
    rng = np.random.default_rng(seed)
    out = []
    n = 30000
    # heavy cancellation: c within a few ulps of -a b
    a = rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n)
    b = rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n)
    c = -(a * b) * (1 + rng.integers(-4, 5, n) * 2.0 ** -52)
    c[::3] = rng.standard_normal(n)[::3] * 2.0 ** rng.integers(-100, 100, n)[::3]
    out.append((a, b, c))
    # cancellation to an exact zero, every sign combination, and signed-zero operands
    m = 8000
    a, b = _short(rng, m), _short(rng, m)
    out.append((a, b, -(a * b)))
    z = np.array([0.0, -0.0])
    g = np.array(np.meshgrid(np.concatenate([z, [1.5, -1.5]]), np.concatenate([z, [2.0, -2.0]]),
                             np.concatenate([z, [3.0, -3.0, -3.0 * 1.5, 3.0 * 1.5]]))).reshape(3, -1)
    out.append((np.tile(g[0], 40), np.tile(g[1], 40), np.tile(g[2], 40)))
    # results at the boundaries between binades: c = +-2^k, a b within a few ulps of 2^k's half ulp (ties included)
    m = 20000
    k = rng.integers(-200, 200, m)
    c = rng.choice([-1.0, 1.0], m) * 2.0 ** k
    a = rng.integers(1, 9, m) * rng.choice([-1.0, 1.0], m) * 2.0 ** (k - 54 - rng.integers(0, 3, m))
    b = 1.0 + rng.integers(-3, 4, m) * 2.0 ** -52
    out.append((a, b, c))
    # subnormal results and operands: products around 2^-1022 .. 2^-1080, c subnormal or cancelling into the subnormal range
    m = 20000
    a = rng.standard_normal(m) * 2.0 ** rng.integers(-560, -480, m)
    b = rng.standard_normal(m) * 2.0 ** rng.integers(-560, -480, m)
    c = np.where(rng.random(m) < 0.5, -(a * b) * (1 + rng.integers(-8, 9, m) * 2.0 ** -52),
                 rng.standard_normal(m) * 2.0 ** -1060)
    out.append((a, b, c))
    sub = rng.integers(1, 2 ** 40, m) * 2.0 ** -1074 * rng.choice([-1.0, 1.0], m)      # subnormal operand
    out.append((sub, rng.standard_normal(m) * 2.0 ** rng.integers(0, 200, m), rng.standard_normal(m) * 2.0 ** -900))
    # products just above the fast path's lower threshold (2^-960), cancelling into tiny normals and subnormals
    a = rng.standard_normal(m) * 2.0 ** -480
    b = rng.standard_normal(m) * 2.0 ** -478
    out.append((a, b, -(a * b) * (1 + rng.integers(-8, 9, m) * 2.0 ** -52)))
    # near the overflow threshold: products and c around 2^1000 .. DBL_MAX, of both signs, some overflowing
    m = 8000
    a = rng.standard_normal(m) * 2.0 ** rng.integers(490, 515, m)
    b = rng.standard_normal(m) * 2.0 ** rng.integers(490, 512, m)
    c = rng.choice([-1.0, 1.0], m) * MAX * rng.random(m)
    out.append((a, b, c))
    out.append((np.full(50, MAX), np.full(50, 1.0 + 2.0 ** -52), -MAX * (1 + np.arange(50) * 0.0)))
    # non-finite operands
    spec = np.array([np.inf, -np.inf, np.nan, 0.0, 1.0, -2.0])
    g = np.array(np.meshgrid(spec, spec, spec)).reshape(3, -1)
    out.append(tuple(g))
    return [np.concatenate(p) for p in zip(*out)]


def test_fma_against_fraction():
    a, b, c = _triples()
    assert a.size >= 100000
    got = M.fma(a, b, c)
    want = _ref(a, b, c)
    same = _same_bits(got, want) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, [(a[i].hex(), b[i].hex(), c[i].hex(), M.hexbits(got[i]), M.hexbits(want[i])) for i in bad[:5]]
    # both paths ran: most elements on the emulation, some through Fraction
    assert np.signbit(got[(got == 0)]).any() and (~np.signbit(got[(got == 0)])).any()
    assert np.isinf(got).any() and (np.abs(got[np.isfinite(got)]) < TINY).any()


def test_fma_zero_signs():
    """IEEE's sign of an exact zero: -0 only for (-0) + (-0); a nonzero exact cancellation is +0 in round to nearest"""
    assert np.signbit(M.fma(-0.0, 1.0, -0.0)) and np.signbit(M.fma(0.0, -1.0, -0.0))
    assert not np.signbit(M.fma(-0.0, 1.0, 0.0)) and not np.signbit(M.fma(0.0, 1.0, -0.0))
    assert not np.signbit(M.fma(1.5, 2.0, -3.0)) and not np.signbit(M.fma(-1.5, 2.0, 3.0))
    assert M.fma(0.0, 5.0, -7.25) == -7.25


def _loop_row_sums(ptr, col, val, x, lanes):
    """the plain per-row model: lane l from +0.0 over entries l, l + lanes, ... with the Fraction fma, then the butterfly"""
    out = np.empty(len(ptr) - 1)
    for i in range(len(ptr) - 1):
        acc = [0.0] * lanes
        for l in range(lanes):
            for j in range(int(ptr[i]) + l, int(ptr[i + 1]), lanes):
                acc[l] = M._fma_exact(val[j], x[col[j]], acc[l])
        o = lanes // 2
        while o > 0:
            acc = [acc[l] + acc[l ^ o] for l in range(lanes)]
            o //= 2
        out[i] = acc[0]
    return out


def _lengths_csr(lanes, seed):
    """rows of length 0, 1, u lanes - 1 .. u lanes + 1 for u = 1 .. 16 (the UNR of every kernel and vector count), rowsplit's
    4 lanes +- 1, and random ones; values and x over many binades, so that the order of the sums shows in the bits"""
    rng = np.random.default_rng(seed)
    lens = [0, 1, 2, 3]
    for u in (1, 2, 4, 8, 16):
        lens += [u * lanes - 1, u * lanes, u * lanes + 1]
    lens += [4 * lanes - 1, 4 * lanes + 1] + list(rng.integers(0, 3 * lanes + 5, 20))
    lens = np.maximum(np.array(lens), 0)
    n = 600
    ptr = np.concatenate([[0], np.cumsum(lens)])
    col = rng.integers(0, n, int(ptr[-1]))
    val = rng.standard_normal(col.size) * 2.0 ** rng.integers(-30, 30, col.size)
    x = rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)
    x[::17] = 0.0
    x[5::17] = -0.0
    return ptr, col, val, x


@pytest.mark.parametrize("lanes", LANES)
def test_row_sums_against_loop(lanes):
    ptr, col, val, x = _lengths_csr(lanes, lanes)
    got = M.row_sums(ptr, col, val, x, lanes)
    want = _loop_row_sums(ptr, col, val, x, lanes)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), np.flatnonzero(got.view(np.uint64) != want.view(np.uint64))
    # a subset of rows, and the shift epilogue
    rows = np.arange(1, len(ptr) - 1, 3)
    assert np.array_equal(M.row_sums(ptr, col, val, x, lanes, rows=rows).view(np.uint64), want[rows].view(np.uint64))
    sig = M.row_sums(ptr, col, val, x, lanes, sigma=-0.375)
    assert np.array_equal(sig.view(np.uint64), _ref(np.full(want.size, -0.375), x[:want.size], want).view(np.uint64))


def test_row_sums_see_the_order():
    """the lanes' order and the butterfly's order change the bits on these rows: the model would not pass a wrong order"""
    ptr, col, val, x = _lengths_csr(8, 3)
    one, eight = M.row_sums(ptr, col, val, x, 1), M.row_sums(ptr, col, val, x, 8)
    assert (one != eight).sum() > 5
    acc = M._lane_sums(np.asarray(ptr), col, val, x, 8, np.arange(len(ptr) - 1))
    v = acc.copy()
    for o in (1, 2, 4):                                      # the butterfly in the other order
        v = v + v[np.arange(8) ^ o]
    assert (v[0] != M.lanes_sum(acc)).sum() > 5


def test_signed_zero_rows():
    """rows whose products are all zeros of one sign, or cancel exactly: the sign of each zero sum"""
    ptr = np.array([0, 0, 1, 2, 4, 6, 8])
    col = np.array([0, 1, 0, 1, 2, 3, 2, 2])
    val = np.array([-0.0, 1.0, 2.0, -2.0, 1.5, -1.5, -0.0, 0.0])
    x = np.array([1.0, -0.0, 1.0, 1.0])
    want = _loop_row_sums(ptr, col, val, x, 1)
    got = M.row_sums(ptr, col, val, x, 1)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert list(np.signbit(got)) == [False, False, False, False, False, False]     # every sum starts from +0.0


def test_exact_rows_against_fraction():
    rng = np.random.default_rng(9)
    ptr, col, val, x = _lengths_csr(4, 9)
    val[:40] = 2.0 ** 600 * rng.standard_normal(40)           # products past the split's range, through Fraction
    got = M.exact_rows(ptr, col, val, x)
    for i in range(len(ptr) - 1):
        s = sum((Fraction(float(val[j])) * Fraction(float(x[col[j]])) for j in range(ptr[i], ptr[i + 1])), Fraction(0))
        assert got[i] == float(s), i


def test_componentwise_bound():
    """every group width's sums lie within gamma_k |A||x| of the exact ones; a sum off by that much more does not"""
    ptr, col, val, x = _lengths_csr(32, 4)
    rows = np.arange(len(ptr) - 1)
    for lanes in LANES:
        ok, exact, bound = M.componentwise_ok(M.row_sums(ptr, col, val, x, lanes), ptr, col, val, x, rows)
        assert ok.all(), lanes
    long = np.flatnonzero(np.diff(ptr) > 4)
    bad = exact[long] + 2 * bound[long] + np.spacing(np.abs(exact[long]))
    assert not M.componentwise_ok(bad, ptr, col, val, x, long)[0].any()
    assert math.isclose(float(M.gamma(10)), 10 * M.U / (1 - 10 * M.U))


def test_value_grad_and_multiply_epilogues():
    """the batched epilogues against the element-by-element Fraction replica they replace"""
    rng = np.random.default_rng(2)
    n, nvec = 50, 11
    rows, cols = rng.integers(0, n, 300), rng.integers(0, n, 300)
    u, v = rng.standard_normal((nvec, n)), rng.standard_normal((nvec, n))
    out0 = rng.standard_normal(300)
    got = M.value_grad(rows, cols, u, v, -0.75, 0.5, out0)
    want = None
    for j0 in (0, 8):
        t = u[j0, rows] * v[j0, cols]
        for k in range(j0 + 1, min(j0 + 8, nvec)):
            t = _ref(u[k, rows], v[k, cols], t)
        prev = (0.5 * out0) if j0 == 0 else want
        want = _ref(np.full(300, -0.75), t, prev)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    ptr, col, val, x = _lengths_csr(2, 5)
    xs = np.stack([x, -x, 2 * x])
    y0 = rng.standard_normal((3, x.size))
    sig = np.array([0.0, 0.5, -1.25])
    got = M.multiply(ptr, col, val, xs, 2, alpha=-1.5, beta=0.25, sigma=sig, y0=y0)
    for j in range(3):
        t = _ref(np.full(len(ptr) - 1, sig[j]), xs[j, :len(ptr) - 1], _loop_row_sums(ptr, col, val, xs[j], 2))
        w = _ref(np.full(t.size, -1.5), t, 0.25 * y0[j, :t.size])
        assert np.array_equal(got[j, :t.size].view(np.uint64), w.view(np.uint64)), j
