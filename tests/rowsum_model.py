"""A bitwise CPU model of the SpMV row sums (csrc/dev.cuh: row_product, lanes_sum) and of the epilogues the
header pins (include/bicgstab_b200.h: the batched multiply and the value gradient), in numpy with a correctly rounded fma.

fma(a, b, c) is Boldo and Melquiond's emulation: the exact product as two_prod (Veltkamp split) and two_sum with c, the two
low parts added in round-to-odd (np.nextafter toward the error), then one rounded add.  Elements outside its preconditions --
non-finite operands, a product or c near the overflow threshold, a product small enough for the split's error term to
underflow -- go through Fraction one by one.  An exact zero takes IEEE's sign: -0 only when a b and c are both -0.

row_sums(ptr, col, val, x, lanes) is row_product<lanes> followed by lanes_sum<lanes>: lane l of a row's group sums entries
l, l + lanes, ... in storage order, from +0.0, one fma per entry; then the butterfly v = v + v[l ^ o] for o = lanes / 2 .. 1.
UNR does not appear: it only decides how many entries one pass loads.  Rows whose order the model does not reproduce (the
persistent kernel's chunk tiles, summed by the whole CTA) are held by componentwise_ok to the exact row sum of exact_rows
instead.  The module imports nothing from the library and runs without a GPU."""
import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -53                                   # unit roundoff of round to nearest
NV_MAX = 8                                       # vectors per launch of the multiply and the value gradient (csrc/spmv.cuh)

_SPLIT = 134217729.0                             # 2^27 + 1
_BIG = 2.0 ** 995                                # beyond this the split's 2^27 a or the sums may overflow
_TINY_PROD = 2.0 ** -960                         # below this the low part of a b may not be representable


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = _SPLIT * a
    h = c - (c - a)
    return h, a - h


def two_prod(a, b):
    """(p, e) with p = fl(a b) and p + e = a b exactly, where the preconditions of fma() hold"""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _round_odd_sum(a, b):
    s, e = _two_sum(a, b)
    odd = (s.view(np.int64) & 1) == 1
    return np.where((e != 0) & ~odd, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def _fma_exact(a, b, c):
    """one element through Fraction: correctly rounded, IEEE's sign of an exact zero, IEEE's inf / nan"""
    a, b, c = float(a), float(b), float(c)
    if math.isfinite(a) and math.isfinite(b) and not math.isfinite(c):
        return c                             # the exact a b is finite, even where fl(a b) would overflow
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        with np.errstate(all="ignore"):      # an infinite or nan factor: a * b is inf or nan exactly as in the fma
            return float(np.float64(a) * np.float64(b) + np.float64(c))
    s = Fraction(a) * Fraction(b) + Fraction(c)
    if s == 0:
        prod_neg = (math.copysign(1.0, a) * math.copysign(1.0, b)) < 0
        return -0.0 if (prod_neg and (a == 0 or b == 0) and c == 0 and math.copysign(1.0, c) < 0) else 0.0
    try:
        return float(s)                          # Fraction -> float rounds to nearest, ties to even
    except OverflowError:
        return math.inf if s > 0 else -math.inf


def fma(a, b, c):
    """Correctly rounded a * b + c of doubles, elementwise (broadcasting), with IEEE's sign of an exact zero."""
    a, b, c = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64),
                                  np.asarray(c, dtype=np.float64))
    shape = a.shape
    a, b, c = a.ravel(), b.ravel(), c.ravel()
    with np.errstate(all="ignore"):
        aa, ab, ac = np.abs(a), np.abs(b), np.abs(c)
        zero_prod = (a == 0) | (b == 0)
        prod = aa * ab
        ok = np.isfinite(a) & np.isfinite(b) & np.isfinite(c) & (ac < _BIG)
        fast = ok & ~zero_prod & (aa < _BIG) & (ab < _BIG) & (prod < _BIG) & (prod >= _TINY_PROD)
        uh, ul = two_prod(a, b)
        th, tl = _two_sum(c, uh)
        out = th + _round_odd_sum(tl, ul)
        # a b is an exact zero: the result is c, or a zero whose sign IEEE fixes
        neg0 = np.signbit(a) ^ np.signbit(b)
        zres = np.where(c != 0, c, np.where(neg0 & np.signbit(c), -0.0, 0.0))
        out = np.where(ok & zero_prod, zres, out)
        # an exact zero sum of nonzero parts is +0 in round to nearest
        out = np.where(fast & (out == 0), 0.0, out)
    slow = np.flatnonzero(~fast & ~(ok & zero_prod))
    for i in slow:
        out[i] = _fma_exact(a[i], b[i], c[i])
    return out.reshape(shape)


# ---- row sums -------------------------------------------------------------------------------------------------------
def _lane_sums(ptr, col, val, x, lanes, rows):
    """(lanes, rows.size): the accumulator of every lane of every row in `rows` after row_product's loop"""
    ptr = np.asarray(ptr, dtype=np.int64)
    lens = ptr[rows + 1] - ptr[rows]
    acc = np.zeros((lanes, rows.size))
    order = np.argsort(-lens, kind="stable")     # longest first: the rows still active at step t are a prefix
    slen, sbeg = lens[order], ptr[rows][order]
    for lane in range(lanes):
        steps = np.maximum(slen - lane + lanes - 1, 0) // lanes      # entries lane, lane + lanes, ... below the length
        nsteps = int(steps.max()) if steps.size else 0
        a = np.zeros(rows.size)
        # count[t] = rows with more than t entries in this lane (steps is non-increasing)
        count = steps.size - np.searchsorted(steps[::-1], np.arange(nsteps), side="right")
        for t in range(nsteps):
            m = int(count[t])
            e = sbeg[:m] + lane + t * lanes
            a[:m] = fma(val[e], x[col[e]], a[:m])
        acc[lane, order] = a
    return acc


def lanes_sum(acc):
    """lanes_sum<L> over the lanes axis (axis 0) of acc: the butterfly v = v + v[l ^ o], o = L / 2 .. 1; lane 0's result"""
    lanes = acc.shape[0]
    v = acc.copy()
    o = lanes // 2
    idx = np.arange(lanes)
    while o > 0:
        v = v + v[idx ^ o]
        o //= 2
    return v[0]


def row_sums(ptr, col, val, x, lanes, sigma=None, rows=None):
    """row_product<lanes> + lanes_sum<lanes> of every row (or of the rows in `rows`), then fma(sigma, x[i], sum) when a
    sigma is given (the solvers' shift and the shifted seed's SpMV)"""
    assert lanes in (1, 2, 4, 8, 16, 32), lanes
    ptr = np.asarray(ptr, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    val = np.asarray(val, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    rows = np.arange(ptr.size - 1) if rows is None else np.asarray(rows, dtype=np.int64)
    y = lanes_sum(_lane_sums(ptr, col, val, x, lanes, rows))
    if sigma is not None:
        y = fma(sigma, x[rows], y)
    return y


def multiply(ptr, col, val, x, lanes, alpha=1.0, beta=0.0, sigma=None, y0=None):
    """The batched multiply's epilogue on the row sums (header: bicg_matrix_multiply): t = rowsum_j, t = fma(sigma_j, x_j, t)
    when sigma is given, y_j = alpha t when beta == 0 (y0 never read), else fma(alpha, t, beta y0_j)."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    n = len(ptr) - 1
    out = np.empty((x.shape[0], n))
    for j in range(x.shape[0]):
        t = row_sums(ptr, col, val, x[j], lanes, None if sigma is None else float(sigma[j]))
        out[j] = alpha * t if beta == 0.0 else fma(alpha, t, beta * np.asarray(y0[j][:n], dtype=np.float64))
    return out


def value_grad(rows, cols, u, v, alpha=1.0, beta=0.0, out0=None):
    """The value gradient's arithmetic (header: bicg_matrix_value_grad) for entries at (rows, cols): batches of NV_MAX vectors,
    t = u_0 v_0, then fma(u_k, v_k, t) in order; out = alpha t, or fma(alpha, t, beta out) (beta = 1 after the first batch)."""
    u = np.atleast_2d(u)
    v = np.atleast_2d(v)
    out = None
    for j0 in range(0, u.shape[0], NV_MAX):
        t = u[j0, rows] * v[j0, cols]
        for k in range(j0 + 1, min(j0 + NV_MAX, u.shape[0])):
            t = fma(u[k, rows], v[k, cols], t)
        b = beta if j0 == 0 else 1.0
        prev = out0 if j0 == 0 else out
        out = alpha * t if b == 0.0 else fma(alpha, t, b * prev)
    return out


# ---- rows held to a bound instead ------------------------------------------------------------------------------------
def _two_prod_any(a, b):
    """two_prod where it is exact, Fraction pairs elsewhere: (p, e) with p + e = a b exactly"""
    with np.errstate(all="ignore"):
        p, e = two_prod(a, b)
        pa = np.abs(p)
        bad = ~((pa < _BIG) & (pa >= _TINY_PROD) & (np.abs(a) < _BIG) & (np.abs(b) < _BIG)) & (a != 0) & (b != 0)
    e = np.where((a == 0) | (b == 0), 0.0, e)
    for i in np.flatnonzero(bad):
        exact = Fraction(float(a[i])) * Fraction(float(b[i]))
        p[i] = float(exact)
        e[i] = float(exact - Fraction(p[i]))
    return p, e


def exact_rows(ptr, col, val, x, rows=None):
    """The exact row sums, correctly rounded: math.fsum over the exact two_prod pairs of each row."""
    ptr = np.asarray(ptr, dtype=np.int64)
    rows = np.arange(ptr.size - 1) if rows is None else np.asarray(rows, dtype=np.int64)
    out = np.empty(rows.size)
    for k, i in enumerate(rows):
        s = slice(ptr[i], ptr[i + 1])
        p, e = _two_prod_any(np.asarray(val[s], dtype=np.float64), np.asarray(x, dtype=np.float64)[col[s]])
        out[k] = math.fsum(np.concatenate([p, e]).tolist())
    return out


def abs_rows(ptr, col, val, x, rows=None):
    """(|A| |x|)_i, rounded upward so that it bounds the exact value"""
    ptr = np.asarray(ptr, dtype=np.int64)
    rows = np.arange(ptr.size - 1) if rows is None else np.asarray(rows, dtype=np.int64)
    out = np.empty(rows.size)
    for k, i in enumerate(rows):
        s = slice(ptr[i], ptr[i + 1])
        t = np.abs(np.asarray(val[s], dtype=np.float64) * np.asarray(x, dtype=np.float64)[col[s]])
        out[k] = math.fsum(t.tolist()) * (1.0 + 4 * U * max(1, t.size))
    return out


def gamma(k):
    """gamma_k = k u / (1 - k u): the componentwise bound of any order of k fma's and adds"""
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def componentwise_ok(got, ptr, col, val, x, rows):
    """|got_i - y_i| <= gamma_{k_i} (|A| |x|)_i for each row i in `rows` (k_i its length, y_i the exact sum).  Returns
    (ok mask, exact sums, bounds)."""
    ptr = np.asarray(ptr, dtype=np.int64)
    rows = np.asarray(rows, dtype=np.int64)
    exact = exact_rows(ptr, col, val, x, rows)
    k = ptr[rows + 1] - ptr[rows]
    bound = gamma(np.maximum(k, 1)) * abs_rows(ptr, col, val, x, rows)
    ok = np.abs(np.asarray(got, dtype=np.float64) - exact) <= bound
    return ok, exact, bound


def hexbits(v):
    return f"{float(v).hex()} (0x{np.float64(v).view(np.uint64):016x})"
