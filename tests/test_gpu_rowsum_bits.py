"""Every SpMV kernel held bit for bit, on every row, to the CPU model of tests/rowsum_model.py (-m gpu).

Every kernel that multiplies by the matrix sums a row as csrc/dev.cuh's row_product and lanes_sum do: lane l of a group of
LANES threads sums entries l, l + LANES, ... in storage order from +0.0, one fma each, then the butterfly.  The model
reproduces that order exactly, so a row that comes out different in one bit is a kernel finding -- whatever its magnitude next
to the other rows, which a norm-wise check against the long-double oracle cannot see.  Rows of the persistent kernel's chunk
tiles are summed by the whole CTA in an order set by the plan's chunk boundaries; they are held to the componentwise bound
gamma_k (|A||x|)_i around the exact sum instead.

The matrices target where kernels go wrong: per-CTA binades (D_r A D_c with power-of-two scales stepping in blocks that are
not aligned to the CTAs, so that every persistent CTA has its own sign / exponent table and some have more than 16 fields and
fall back to 8-byte values in the same launch), row lengths around every kernel's unroll (UNR LANES - 1 .. + 1), rowsplit's
4 LANES +- 1 and the chunk-tile lengths, and rows whose products cancel to exact zeros with signed zeros, subnormal and huge
entries in x.  Every assertion message names the kernel, its configuration, the row and both bit patterns."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import rowsum_model as M
from loop_reference import ARENA
from state_check import STANDALONE, cap_limit, matrix
from test_gpu_transpose import transposed_csr

pytestmark = pytest.mark.gpu

LANES = [1, 2, 4, 8, 16, 32]
NVECS = [1, 3, M.NV_MAX, M.NV_MAX + 1, 17]
DEFAULTS = dict(quiet=1, tol=1e-15, max_iter=1000, mega=1, resident=1, mega_threads=0, mega_lanes=0, spmv="auto",
                spmv_lanes=0, spmv_threads=0, spmv_stages=0, autotune=1, cache=1)


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(**(DEFAULTS | dict(autotune=0)))
    yield
    B.set_options(**DEFAULTS)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- matrices -------------------------------------------------------------------------------------------------------
def _csr(A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A.shape[0], A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64)


def _binades():
    """D_r A D_c on a 9-point band of 150 000 rows.  A: off-diagonals -(0.5 + 0.5 u), diagonal in [8.5, 15.5): one binade
    each.  Row exponents step in blocks of 997 rows, column exponents in blocks of 4001 columns, both within +-40, so that no
    two neighbouring CTAs (about 1 140 rows each) see the same table; every fifth row block also varies its exponent over 7
    values row by row, which takes its CTAs past 16 sign / exponent fields.  Every product, dot and square of a k <= 3 solve
    stays normal and finite."""
    n = 150000
    rng = np.random.default_rng(41)
    off = [-600, -300, -2, -1, 1, 2, 300, 600]
    A = sp.diags([-(0.5 + 0.5 * rng.random(n - abs(o))) for o in off] + [8.5 + 7.0 * rng.random(n)], off + [0],
                 shape=(n, n), format="csr")
    rb = np.arange(n) // 997
    rexp = rng.integers(-40, 41, rb.max() + 1)[rb]
    busy = rb % 5 == 2
    rexp[busy] += np.arange(n)[busy] % 7
    cexp = rng.integers(-40, 41, n // 4001 + 1)[np.arange(n) // 4001]
    A = sp.diags(2.0 ** rexp) @ A @ sp.diags(2.0 ** cexp)
    return _csr(A)


def _length_list():
    """row lengths around every kernel's unroll: UNR LANES - 1 .. + 1 for UNR in 1 .. 16 (16 or 8 gathers in flight in the
    one-vector kernels, 16 / NV or 8 / NV in the batched multiply, 16 in the resident slice), rowsplit's 4 LANES +- 1, 0, 1"""
    lens = {0, 1, 2}
    for lanes in LANES:
        for u in (1, 2, 4, 8, 16):
            lens |= {u * lanes - 1, u * lanes, u * lanes + 1}
        lens |= {4 * lanes - 1, 4 * lanes + 1}
    return sorted(lens)


def _lengths():
    """20 011 rows; every 23rd row has one of _length_list()'s lengths (each one many times, at every offset in a tile), the
    others 3 .. 12 entries.  Off-diagonals over 12 binades, a diagonal that dominates them (a row of length 0 has none)."""
    n = 20011
    rng = np.random.default_rng(43)
    lens = rng.integers(3, 13, n)
    special = _length_list()
    lens[::23] = np.array(special)[np.arange(lens[::23].size) % len(special)]
    rows, cols, vals = [], [], []
    for i in range(n):
        k = int(lens[i])
        if k == 0:
            continue
        c = rng.choice(np.unique(rng.integers(0, n - 1, 2 * k + 8)), size=k - 1, replace=False)
        c = np.sort(np.append(c + (c >= i), i))
        v = -(0.5 + 0.5 * rng.random(k)) * 2.0 ** -rng.integers(0, 12, k)
        v[c == i] = np.abs(v[c != i]).sum() + 1.0 + rng.random()
        rows.append(np.full(k, i))
        cols.append(c)
        vals.append(v)
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    return _csr(A)


HOT = 31                                                        # columns 2m, 2m + 1 with m % HOT == 0 hold x = +-2^1000


def _cancel():
    """4 099 rows: rows whose products cancel to exact zero (v, -v on columns 2m and 2m + 1, which share their x), rows of
    signed zeros, and ordinary rows.  The values of the columns where x is huge (2^1000) are scaled by 2^-80, so that every
    row stays finite; x also carries signed zeros and subnormals (_cancel_x)."""
    n = 4099
    rng = np.random.default_rng(47)
    rows, cols, vals = [], [], []
    for i in range(n):
        kind = i % 5
        k = int(rng.integers(2, 40))
        c = np.sort(rng.choice(n, size=k, replace=False))
        if kind == 0:
            m = rng.choice(n // 2, size=k // 2, replace=False)
            c = np.sort(np.concatenate([2 * m, 2 * m + 1]))
            v = np.repeat(rng.standard_normal(k // 2), 2) * np.tile([1.0, -1.0], k // 2)
        elif kind == 1:
            v = rng.choice([0.0, -0.0], k)
        else:
            v = rng.standard_normal(k) * 2.0 ** rng.integers(-20, 20, k)
        rows.append(np.full(c.size, i))
        cols.append(c)
        vals.append(v)
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    A.sort_indices()                                            # explicit zeros stay
    ptr, col, val = A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64)
    val = np.where((col // 2) % HOT == 0, val * 2.0 ** -80, val)
    assert (val == 0).sum() > 1000 and np.signbit(val[val == 0]).any()
    return n, ptr, col, val


def _cancel_x(n, seed):
    """x with equal entries in columns 2m and 2m + 1: signed zeros, subnormals, +-2^1000 in the scaled columns"""
    rng = np.random.default_rng(seed)
    h = (n + 1) // 2
    half = rng.standard_normal(h) * 2.0 ** rng.integers(-10, 10, h)
    sel = rng.random(h)
    z, s = sel < 0.08, (sel >= 0.08) & (sel < 0.16)
    half[z] = rng.choice([0.0, -0.0], int(z.sum()))
    half[s] = rng.integers(1, 2 ** 30, int(s.sum())) * 2.0 ** -1074 * rng.choice([-1.0, 1.0], int(s.sum()))
    hot = np.arange(h) % HOT == 0
    half[hot] = 2.0 ** 1000 * rng.choice([-1.0, 1.0], int(hot.sum()))
    return np.repeat(half, 2)[:n]


_CACHE = {}


def csr(name):
    if name not in _CACHE:
        _CACHE[name] = {"binades": _binades, "lengths": _lengths, "cancel": _cancel}[name]()
    return _CACHE[name]


def xvec(name, n, seed=0):
    if name == "cancel":
        return _cancel_x(n, seed)
    rng = np.random.default_rng(seed + 101)
    x = rng.standard_normal(n) * 2.0 ** rng.integers(-8, 9, n)
    x[::97] = -0.0
    return x


_MODEL = {}


def model(name, x, lanes, ptr, col, val, key=None):
    k = (name, lanes, key)
    if key is None or k not in _MODEL:
        y = M.row_sums(ptr, col, val, x, lanes)
        if key is None:
            return y
        _MODEL[k] = y
    return _MODEL[k]


def assert_bits(got, want, what, rows=None):
    """bitwise equality of every row; the message names the first mismatching rows with both bit patterns"""
    got, want = np.ascontiguousarray(got, dtype=np.float64), np.ascontiguousarray(want, dtype=np.float64)
    bad = np.flatnonzero(got.view(np.uint64) != want.view(np.uint64))
    if bad.size:
        rows = np.arange(got.size) if rows is None else np.asarray(rows)
        lines = []
        for i in bad[:6]:
            lines.append(f"row {int(rows[i])}: model {M.hexbits(want[i])} kernel {M.hexbits(got[i])}")
        pytest.fail(f"{what}: {bad.size} of {got.size} rows differ from the model\n  " + "\n  ".join(lines))


# ---- stand-alone SpMV: every forced configuration -------------------------------------------------------------------
def _plan_lanes(B, dm, n):
    """the stand-alone plan's lanes and kind, from the stats of a one-iteration kernel-per-phase solve on the handle"""
    B.set_options(mega=0, tol=0.0, max_iter=1)
    x, r = np.zeros(n), np.ones(n)
    dm.solve("bicgstab", x, r)
    st = B.last_stats()
    B.set_options(mega=1, tol=1e-15, max_iter=1000)
    return st["spmv_lanes"], st["spmv_kind"]


@pytest.mark.parametrize("name", ["lengths", "cancel", "binades"])
@pytest.mark.parametrize("case", STANDALONE, ids=[c[0] for c in STANDALONE])
def test_standalone_spmv(B, case, name):
    """bicg_spmv, and bicg_debug_spmv_epi's s = A p (w for epilogue 3) under every forced stand-alone configuration"""
    cfg, _, opts, kind, lanes = case
    B.set_options(**opts)
    n, ptr, col, val = csr(name)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        got_lanes, got_kind = _plan_lanes(B, dm, n)
        assert (got_lanes, got_kind) == (lanes, kind), (cfg, got_lanes, got_kind)
        for seed in (0, 1):
            x = xvec(name, n, seed)
            assert_bits(dm.spmv(x), model(name, x, lanes, ptr, col, val, key=("x", seed)), f"spmv {cfg} on {name} x{seed}")
        if name != "cancel":
            rng = np.random.default_rng(5)
            for epi in range(4):
                buf = np.ascontiguousarray(rng.standard_normal((11, n)))
                buf[ARENA["p"]] = xvec(name, n, 2 + epi)
                p = buf[ARENA["p"]].copy()
                dots = (C.c_double * 8)()
                B.lib.bicg_debug_spmv_epi(dm.h, epi, buf.ctypes.data_as(C.c_void_p), dots)
                out = buf[ARENA["w"]] if epi == 3 else buf[ARENA["s"]]
                assert_bits(out, model(name, p, lanes, ptr, col, val, key=("epi", epi)), f"spmv_epi {epi} {cfg} on {name}")
    finally:
        dm.destroy()


@pytest.mark.parametrize("name", ["lengths", "cancel"])
def test_reference_facing_spmv_ovlap(B, name):
    """MPI_csr_spmv_ovlap on the library's own plan choice: the lanes of the plan it cached"""
    n, ptr, col, val = csr(name)
    blk = B.blocks_from_csr(n, ptr, col, val)
    x = xvec(name, n, 3)
    y = B.spmv_ovlap(blk, x)
    B.set_options(mega=0, tol=0.0, max_iter=1)
    B.bicgstab(blk, np.zeros(n), np.ones(n))                     # same cached upload: its stats name the plan
    lanes = B.last_stats()["spmv_lanes"]
    assert_bits(y, model(name, x, lanes, ptr, col, val), f"spmv_ovlap auto (lanes {lanes}) on {name}")


# ---- persistent kernel ----------------------------------------------------------------------------------------------
# (mega_lanes, resident, stream_codes, stream_values): resident slices exist only at one lane per row
COMBOS = [(1, res, codes, vals) for res in (0, 1) for codes in (True, False) for vals in (True, False)] + \
         [(l, 0, codes, vals) for l in (4, 8, 32) for codes in (True, False) for vals in (True, False)]
# arena pairs (input, output = A input) each loop leaves intact when it stops (tests/loop_reference.py)
PAIRS = {"bicgstab": [("p", "s")], "ca_bicgstab": [("s", "z"), ("r", "w")], "pipe_bicgstab": [("z", "v"), ("w", "t")]}


def _arena(B, dm, n, name):
    out = np.empty(n)
    assert B.lib.bicg_debug_get_vec(dm.h, ARENA[name], out.ctypes.data_as(C.c_void_p)) == 0
    return out


def _persistent(B, name, n, ptr, col, val, lanes, resident, codes, values, methods, chunk_rows=()):
    B.set_options(mega=2, mega_lanes=lanes, resident=resident)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    cfg = f"mega_lanes={lanes} resident={resident} codes={int(codes)} values={int(values)}"
    whole = np.setdiff1d(np.arange(n), np.asarray(chunk_rows, dtype=np.int64))
    seen = []
    try:
        dm.stream_codes(codes)
        dm.stream_values(values)
        b = np.asarray(sp.csr_matrix((val, col, ptr), shape=(n, n)) @ np.ones(n))
        for method in methods:
            for k in (1, 2, 3):
                B.set_options(tol=0.0, max_iter=k)
                x, r = np.zeros(n), b.copy()
                it, st = dm.solve(method, x, r)
                assert it == k and st["kernel_launches"] <= 8, (cfg, method, it, st["kernel_launches"])
                seen.append((dm.coded_ctas(), dm.packed_ctas(), dm.resident_ctas()))
                for src, dst in PAIRS[method]:
                    xin, y = _arena(B, dm, n, src), _arena(B, dm, n, dst)
                    assert np.all(np.isfinite(xin)), (cfg, method, k, src)
                    what = f"persistent kernel {method} k={k} {dst} = A {src}, {cfg}, {name}"
                    assert_bits(y[whole], M.row_sums(ptr, col, val, xin, lanes, rows=whole), what, rows=whole)
                    if len(chunk_rows):
                        ok, exact, bound = M.componentwise_ok(y[chunk_rows], ptr, col, val, xin, chunk_rows)
                        assert ok.all(), (f"{what}: chunk-tile rows {np.asarray(chunk_rows)[~ok]} off the exact sum by more "
                                          f"than gamma_k |A||x|: {y[chunk_rows][~ok]} vs {exact[~ok]} (bound {bound[~ok]})")
    finally:
        dm.destroy()
    return seen


@pytest.mark.parametrize("combo", COMBOS, ids=[f"l{c[0]}-res{c[1]}-codes{int(c[2])}-vals{int(c[3])}" for c in COMBOS])
def test_persistent_binades(B, combo):
    """s = A p of bicgstab, and the pairs the CA and pipelined loops leave, on the per-CTA binade matrix"""
    lanes, resident, codes, values = combo
    n, ptr, col, val = csr("binades")
    methods = list(PAIRS) if (codes and values) or resident else ["bicgstab"]
    seen = _persistent(B, "binades", n, ptr, col, val, lanes, resident, codes, values, methods)
    coded, packed, res = seen[0]
    G = _sm_count()
    if resident and res:
        assert res == G, seen[0]
    elif codes and values:
        assert 0 < packed < coded == G, f"every CTA streams codes, some but not all pack their values: {seen[0]}"
    else:
        assert packed == 0 and coded == (G if codes else 0), seen[0]


@pytest.mark.parametrize("combo", [c for c in COMBOS if c[1] == 0 and c[3]],
                         ids=[f"l{c[0]}-codes{int(c[2])}" for c in COMBOS if c[1] == 0 and c[3]])
def test_persistent_lengths(B, combo):
    lanes, resident, codes, values = combo
    n, ptr, col, val = csr("lengths")
    _persistent(B, "lengths", n, ptr, col, val, lanes, resident, codes, values, ["bicgstab"])


@pytest.mark.parametrize("lanes", [1, 4, 32])
def test_persistent_chunk_tiles(B, lanes):
    """state_check's chunk matrix for this lanes' stage capacity: whole rows bit for bit, chunk-tile rows within the bound"""
    cap = cap_limit(512, lanes)
    n, ptr, col, val = matrix(B, f"chunk_cap{cap}")
    ptr, col = np.asarray(ptr, dtype=np.int64), np.asarray(col, dtype=np.int64)
    chunk = np.flatnonzero(np.diff(ptr) > cap)
    assert chunk.size == 4
    for codes in (True, False):
        _persistent(B, f"chunk_cap{cap}", n, ptr, col, val, lanes, 1, codes, True, ["bicgstab"], chunk_rows=chunk)


# ---- batched multiply ------------------------------------------------------------------------------------------------
MUL_PLANS = [("auto", {}), ("rowsplit-l1", dict(spmv="rowsplit", spmv_lanes=1)),
             ("rowsplit-l4", dict(spmv="rowsplit", spmv_lanes=4)), ("rowsplit-l32", dict(spmv="rowsplit", spmv_lanes=32)),
             ("tma-l1", dict(spmv="tma", spmv_lanes=1)), ("tma-l2-t128", dict(spmv="tma", spmv_lanes=2, spmv_threads=128)),
             ("tma-l8", dict(spmv="tma", spmv_lanes=8)), ("tma-l16-s2", dict(spmv="tma", spmv_lanes=16, spmv_stages=2)),
             ("tma-l32", dict(spmv="tma", spmv_lanes=32))]
MUL_COMBOS = [(1.0, 0.0, False), (-0.75, 0.0, True), (-1.0, 1.0, True), (0.625, -2.5, True), (-3.0, 0.5, False)]


@pytest.mark.parametrize("name", ["lengths", "cancel"])
@pytest.mark.parametrize("plan", MUL_PLANS, ids=[p[0] for p in MUL_PLANS])
def test_multiply_every_row(B, plan, name):
    """y_j = alpha (A + sigma_j I) x_j + beta y_j for every vector count 1, 3, 8, 9, 17, on every row: sigma with zeros in it,
    negative alpha, beta != 0, and y full of NaN at beta = 0 (never read)"""
    label, opts = plan
    B.set_options(**opts)
    n, ptr, col, val = csr(name)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        lanes, _ = _plan_lanes(B, dm, n)
        rng = np.random.default_rng(7)
        for i, nvec in enumerate(NVECS):
            alpha, beta, shifted = MUL_COMBOS[i % len(MUL_COMBOS)]
            x = np.stack([xvec(name, n, 10 + j) for j in range(nvec)])
            sigma = None
            if shifted:
                sigma = rng.standard_normal(nvec)
                sigma[::3] = 0.0
            y0 = np.full((nvec, n), np.nan) if beta == 0.0 else rng.standard_normal((nvec, n))
            if beta != 0.0:
                y0[:, ::5] = -0.0
            got = dm.multiply(x, y0.copy(), alpha=alpha, beta=beta, sigma=sigma)
            want = M.multiply(ptr, col, val, x, lanes, alpha, beta, sigma, y0)
            for j in range(nvec):
                assert_bits(got[j], want[j], f"multiply {label} (lanes {lanes}) on {name}: nvec {nvec} vector {j} "
                                             f"alpha {alpha} beta {beta} sigma {None if sigma is None else sigma[j]}")
    finally:
        dm.destroy()


def test_multiply_binades(B):
    n, ptr, col, val = csr("binades")
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        lanes, _ = _plan_lanes(B, dm, n)
        x = np.stack([xvec("binades", n, 20 + j) for j in range(3)])
        sigma = np.array([0.5, 0.0, -2.0])
        y0 = np.random.default_rng(3).standard_normal((3, n))
        got = dm.multiply(x, y0.copy(), alpha=-1.5, beta=0.75, sigma=sigma)
        want = M.multiply(ptr, col, val, x, lanes, -1.5, 0.75, sigma, y0)
        for j in range(3):
            assert_bits(got[j], want[j], f"multiply auto (lanes {lanes}) on binades vector {j}")
    finally:
        dm.destroy()


# ---- transpose --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lengths", "binades"])
@pytest.mark.parametrize("plan", [("rowsplit-l4", dict(spmv="rowsplit", spmv_lanes=4)), ("tma-l1", dict(spmv="tma", spmv_lanes=1)),
                                  ("tma-l8", dict(spmv="tma", spmv_lanes=8))], ids=lambda p: p[0])
def test_transpose_spmv(B, plan, name):
    """spmv of a transpose handle against the model on the transposed CSR (A's triplets stably sorted by column, row)"""
    label, opts = plan
    B.set_options(**opts)
    n, ptr, col, val = csr(name)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    mt = dm.transpose()
    try:
        lanes, _ = _plan_lanes(B, mt, n)
        tp, tc, tv = transposed_csr(n, ptr, col, val)
        x = xvec(name, n, 30)
        assert_bits(mt.spmv(x), M.row_sums(tp, tc, tv, x, lanes), f"transpose spmv {label} (lanes {lanes}) on {name}")
    finally:
        mt.destroy()
        dm.destroy()
