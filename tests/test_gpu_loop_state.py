"""Every solver loop held to the reference iteration by iteration (-m gpu), on every plan shape of the persistent kernel
(mega.cu) and of the kernel-per-phase path (solve.cu).

A solve with tol = 0 and max_iter = k stops after exactly k iterations; then every arena vector (bicg_debug_get_vec), the
solver scalars (bicg_debug_get_scalars) and the residual history (last_history) are compared with tests/loop_reference.py
stopped at the same k.  A kernel can be wrong and still converge; it cannot be wrong and still match every vector after
every one of the first iterations.

Tolerance: max-norm relative error for a vector, relative error for a scalar or a history entry, at most
max(FLOOR, FACTOR * spread), where spread is the same quantity between the reference and its exact evaluation (long-double
SpMV, fsum dots): the rounding the case itself amplifies.  A case whose spread exceeds MAX_SPREAD says nothing about the
kernel; the test refuses it rather than loosening the bound.  Every assertion message carries the error, the spread and
their ratio (FACTOR * err / bound: below FACTOR passes).

A vector is held to its own spread.  A scalar or history entry is held to the largest spread among the scalars and history
entries of its state: they are computed from one another (beta from alpha, omega and two dots; the next alpha from beta,
omega and three dots), and one scalar's own spread can be small by chance.  Summing the reference's dots in numpy's order
instead, a correct implementation by construction, lands 175 times beta's own spread away on the 17-row case with
replacements at k = 5, and 19 times (w,w)'s on stencil15_g20; against the state's scalar spread every ratio of that
reordering stays below 2.5."""
import ctypes as C
import math

import numpy as np
import pytest

from helpers import METHODS, X0_KINDS, initial_guess
from loop_reference import ARENA, SCALARS, reference_states
from state_check import BIG, FACTOR, STANDALONE, _hold, _rel, cap_limit, matrix

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 5)
RR_KW = dict(krr=2, nrr=2)                  # replacements at k = 2 and 4, inside KS
# launches of a solve whose loop is ONE persistent kernel: the init kernels of solve.cu (Seq::bicgstab_init / capipe_init) + 1
MEGA_LAUNCHES = {"bicgstab": 3, "ca_bicgstab": 4, "pipe_bicgstab": 5, "pipe_bicgstab_rr": 5}
KERNELS_PER_ITER = {"bicgstab": 5, "ca_bicgstab": 5, "pipe_bicgstab": 4, "pipe_bicgstab_rr": 4}
DEFAULTS = dict(quiet=1, tol=1e-15, max_iter=1000, mega=1, resident=1, mega_threads=0, mega_lanes=0, spmv="auto",
                spmv_lanes=0, spmv_threads=0, spmv_stages=0, autotune=1)


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(**(DEFAULTS | dict(autotune=0)))
    yield
    B.set_options(**DEFAULTS)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count       # one persistent CTA per SM


_REF = {}


def reference(B, O, name, method, ks, krr=0, nrr=0, x0_kind=None):
    """(reference states, exact-evaluation states) for ks, computed once per matrix, method, replacement schedule and initial
    guess (x0_kind: a helpers.X0_KINDS entry, None for x0 = 0)."""
    key = (name, method, tuple(ks), krr, nrr, x0_kind)
    if key in _REF:
        return _REF[key]
    n, ptr, col, val = matrix(B, name)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    x0 = None if x0_kind is None else initial_guess(x0_kind, n)
    ref = tuple(reference_states(O, method, ptr, col, val, b, ks, krr=krr, nrr=nrr, exact=e, x0=x0) for e in (False, True))
    if n < BIG:
        _REF[key] = ref
    return ref


def check_state(B, dm, n, k, want, exact, x, r, label):
    """Every vector, scalar and history entry the solve left against the reference state after iteration k.  b (the caller's
    b, which pipe_bicgstab_rr keeps for its replacements) must be bit for bit what was passed in; every other vector, r# = r0
    and ax = A x (A x0 until the first replacement) among them, is a computed one and held to its spread."""
    what = f"{label} k={k}"
    ratio = (0.0, "")
    got = np.empty(n)
    for name, ref in want.items():
        if not isinstance(ref, np.ndarray) or name == "hist":
            continue
        assert B.lib.bicg_debug_get_vec(dm.h, ARENA[name], got.ctypes.data_as(C.c_void_p)) == 0
        if name == "b":
            assert np.array_equal(got, ref), f"{what}: b must be the caller's b bit for bit"
            continue
        ratio = max(ratio, _hold(f"{what} {name}", got, ref, exact[name]))
        if name in ("x", "r"):
            assert np.array_equal(got, x if name == "x" else r), f"{what}: returned {name} differs from the arena's"
    s13 = (C.c_double * 13)()
    B.lib.bicg_debug_get_scalars(dm.h, s13)
    gs = dict(zip(SCALARS, s13))
    names = [q for q in SCALARS if q in want]
    sspread = max([_rel(exact[q], want[q]) for q in names] + [_rel(exact["hist"][i], want["hist"][i]) for i in range(1, k + 1)])
    for name in names:
        ratio = max(ratio, _hold(f"{what} {name}", gs[name], want[name], exact[name], sspread))
    hist = B.last_history()
    assert hist.size == k + 1 and hist[0] == 1.0
    for i in range(1, k + 1):
        ratio = max(ratio, _hold(f"{what} hist[{i}]", hist[i], want["hist"][i], exact["hist"][i], sspread))
    return ratio


def solve_k(B, dm, n, method, k, b, krr=0, nrr=0, x0=None):
    B.set_options(tol=0.0, max_iter=k)
    x, r = np.zeros(n) if x0 is None else x0.copy(), b.copy()
    it, st = dm.solve(method, x, r, krr, nrr)
    assert it == st["iters"] == k, (it, k)
    return st, x, r


def assert_path(st, method, k, mega):
    if mega:
        assert st["kernel_launches"] == MEGA_LAUNCHES[method], st["kernel_launches"]     # the loop ran as ONE kernel
    else:
        assert st["kernel_launches"] >= MEGA_LAUNCHES[method] - 1 + k * KERNELS_PER_ITER[method], st["kernel_launches"]


def run_states(B, O, name, method, ks=KS, mega=1, krr=0, nrr=0, codes=None, expect=None, x0_kind=None):
    """Solve for every k in ks on a fresh handle of matrix `name`, hold each state to the reference; expect(dm, st) checks
    the plan shape.  codes=False forces 32-bit columns; x0_kind (helpers.X0_KINDS) starts from a nonzero initial guess.
    Returns ((largest ratio, where), [(x, r, history) per k])."""
    n, ptr, col, val = matrix(B, name)
    if method == "pipe_bicgstab_rr" and not krr:
        krr, nrr = RR_KW["krr"], RR_KW["nrr"]
    ref, ex = reference(B, O, name, method, ks, krr, nrr, x0_kind)
    x0 = None if x0_kind is None else initial_guess(x0_kind, n)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    B.set_options(mega=int(mega))
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    worst, outs = (0.0, ""), []
    try:
        if codes is not None:
            dm.stream_codes(codes)
        for k in ks:
            st, x, r = solve_k(B, dm, n, method, k, b, krr, nrr, x0)
            assert_path(st, method, k, bool(mega))
            if expect:
                expect(dm, st)
            worst = max(worst, check_state(B, dm, n, k, ref[k], ex[k], x, r, f"{name} {method}"))
            outs.append((x, r, B.last_history()))
    finally:
        dm.destroy()
    print(f"[loop-state] {name} {method} mega={mega} codes={codes} krr={krr} nrr={nrr} x0={x0_kind}: "
          f"largest err/spread ratio {worst[0]:.3g} ({worst[1]})")
    return worst, outs


# ---- persistent kernel ----------------------------------------------------------------------------------------------
def _all_coded(dm, st):
    assert dm.coded_ctas() == _sm_count() and dm.resident_ctas() == 0, (dm.coded_ctas(), dm.resident_ctas())


def _all_resident(dm, st):
    assert dm.resident_ctas() == _sm_count() and dm.coded_ctas() == 0, (dm.resident_ctas(), dm.coded_ctas())


PERSISTENT = [
    # (id, matrix, options at plan time, plan-shape check, iteration counts)
    ("streaming", "stencil15_g60", dict(resident=0), _all_coded, KS),
    ("resident", "stencil15_g58", dict(resident=1), _all_resident, KS),
    ("threads256", "stencil15_g60", dict(resident=0, mega_threads=256), _all_coded, KS),
    *[(f"lanes{l}-stencil", "stencil15_g40", dict(mega_lanes=l), _all_coded, KS) for l in (4, 8, 32)],
    # the pipelined loops converge by 1e-4 per iteration here: by k = 5 the case's own spread reaches 1e-6
    *[(f"lanes{l}-random", "random_n20011_k32", dict(mega=2, mega_lanes=l), _all_coded, (1, 2, 3)) for l in (4, 8, 32)],
]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_persistent_kernel_state(B, O, case, method):
    _, name, opts, expect, ks = case
    B.set_options(**opts)
    run_states(B, O, name, method, ks=ks, mega=opts.get("mega", 1), expect=expect)


def test_bench_matrix_coded_and_32bit(B, O):
    """The benchmark matrix (T' g117, 1.6 M rows), every CTA streaming codes, and forced to 32-bit columns: both match the
    reference, and each other bit for bit."""
    ks = (1, 2, 3)
    _, coded = run_states(B, O, "stencil15_g117", "bicgstab", ks=ks, codes=True, expect=_all_coded)
    _, plain = run_states(B, O, "stencil15_g117", "bicgstab", ks=ks, codes=False,
                          expect=lambda dm, st: dm.coded_ctas() == 0 or pytest.fail("forced 32-bit run streamed codes"))
    for a, b in zip(coded, plain):
        assert all(np.array_equal(u, v) for u, v in zip(a, b))


def _chunked_rows(B, n, ptr, threads, lanes):
    """{row: chunk tiles} of the CPU planner at the persistent kernel's cap_limit for (threads, lanes)."""
    ptr = np.ascontiguousarray(ptr, dtype=np.uint32)
    cap, G, rpt = cap_limit(threads, lanes), _sm_count(), threads // lanes
    tc = n + 4 * G + 64
    tr, nz, fl, ct = (C.c_int * tc)(), (C.c_uint * tc)(), (C.c_int * tc)(), (C.c_int * (G + 1))()
    mx = C.c_uint()
    nt = B.lib.bicg_plan_cta_tiles_capped(ptr.ctypes.data_as(C.POINTER(C.c_uint)), n, G, rpt, cap, tr, nz, fl, tc, ct, C.byref(mx))
    assert nt > 0 and mx.value <= cap
    out = {}
    for t in range(nt):
        if fl[t]:
            out[tr[t]] = out.get(tr[t], 0) + 1
    return out


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("lanes", [1, 4, 32])
def test_chunk_tiles_state(B, O, lanes, method):
    """Rows longer than a stage become chunk tiles that the whole CTA multiplies; every epilogue (EPI_NONE, EPI_RH_Y,
    EPI_QY_YY, EPI_CA4) runs on them under the four loops.  Coded and 32-bit columns both match the reference and each
    other."""
    cap = cap_limit(512, lanes)
    name = f"chunk_cap{cap}"
    n, ptr, *_ = matrix(B, name)
    lens = np.diff(ptr)
    want = {r: -(-int(lens[r]) // cap) for r in range(n) if lens[r] > cap}
    assert sorted(lens[r] for r in want) == [cap + 1, 2 * cap, 2 * cap, 3 * cap + 7]
    assert _chunked_rows(B, n, ptr, 512, lanes) == want          # cap - 1 and cap stay whole rows

    def expect(dm, st):
        assert dm.resident_ctas() == 0 and 0 < dm.coded_ctas() <= _sm_count()

    B.set_options(mega_lanes=lanes, resident=1)                  # a chunked plan never keeps a slice resident
    _, coded = run_states(B, O, name, method, codes=True, expect=expect)
    _, plain = run_states(B, O, name, method, codes=False, expect=lambda dm, st: dm.coded_ctas() == 0 or pytest.fail("coded"))
    for a, b in zip(coded, plain):
        assert all(np.array_equal(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("method", METHODS)
def test_code_window_boundary(B, O, method):
    """CTA 0's own-column window is exactly 65 536 columns (16-bit codes) or 65 537 (32-bit columns): one CTA less codes
    its columns.  Both match the reference and their forced-32-bit runs bit for bit."""
    coded_ctas = {}
    for name in ("window_65535", "window_65536"):
        counts = []
        B.set_options(resident=0)
        _, coded = run_states(B, O, name, method, ks=(1, 3), codes=True, expect=lambda dm, st: counts.append(dm.coded_ctas()))
        _, plain = run_states(B, O, name, method, ks=(1, 3), codes=False,
                              expect=lambda dm, st: dm.coded_ctas() == 0 or pytest.fail("coded"))
        for a, b in zip(coded, plain):
            assert all(np.array_equal(u, v) for u, v in zip(a, b))
        assert len(set(counts)) == 1
        coded_ctas[name] = counts[0]
    assert coded_ctas["window_65535"] == _sm_count()
    assert coded_ctas["window_65535"] - coded_ctas["window_65536"] == 1, coded_ctas


# ---- both loop paths --------------------------------------------------------------------------------------------------
SMALL = ["small_n17", "small_n2111", "small_n2112", "small_n2113", "ragged_4001"]


@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", SMALL)
def test_small_and_ragged_state(B, O, name, method, mega):
    """n = 17 (most CTAs own no rows), 16 x 132 - 1, 16 x 132, 16 x 132 + 1 (odd row counts take the one-row tail of the
    vector phases) and a ragged matrix with rows that hold nothing but their diagonal."""
    run_states(B, O, name, method, mega=mega)


@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("nrr", [1, 2])
@pytest.mark.parametrize("krr", [1, 2, 3])
def test_residual_replacement_every_iteration(B, O, krr, nrr, mega):
    """pipe_bicgstab_rr stopped after every iteration up to two past the last replacement (k <= krr * nrr + 2): the
    replacement branch (solver.c:494-547) runs exactly at k % krr == 0, 0 < k <= krr * nrr."""
    B.set_options(resident=0)
    run_states(B, O, "stencil15_g20", "pipe_bicgstab_rr", ks=range(1, krr * nrr + 3), mega=mega, krr=krr, nrr=nrr)


@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("method", METHODS)
def test_max_iter_stops_exactly_every_method(B, O, method, mega):
    n, ptr, col, val = matrix(B, "stencil15_g20")
    b = O.spmv(n, ptr, col, val, np.ones(n))
    B.set_options(mega=mega)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    kw = RR_KW if method.endswith("rr") else {}
    try:
        for k in (1, 4, 7, 12):
            st, *_ = solve_k(B, dm, n, method, k, b, **kw)
            assert_path(st, method, k, mega)
            assert B.last_history().size == k + 1
    finally:
        dm.destroy()


# ---- kernel-per-phase path: every stand-alone SpMV variant ------------------------------------------------------------
def _plan(kind, lanes):
    def expect(dm, st):
        assert (st["spmv_kind"], st["spmv_lanes"]) == (kind, lanes), (st["spmv_kind"], st["spmv_lanes"])
    return expect


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", STANDALONE, ids=[c[0] for c in STANDALONE])
def test_kernel_per_phase_state(B, O, case, method):
    _, name, opts, kind, lanes = case
    B.set_options(**opts)
    run_states(B, O, name, method, mega=0, expect=_plan(kind, lanes))


def _arena(rng, n):
    return np.ascontiguousarray(rng.standard_normal((11, n)))


@pytest.mark.parametrize("case", STANDALONE, ids=[c[0] for c in STANDALONE])
def test_spmv_epilogue_dots_every_variant(B, O, case):
    """y = A p with the fused epilogue dots of every loop (bicg_debug_spmv_epi, epilogues 0 to 3) on each forced stand-alone
    SpMV: y against the long-double SpMV, each dot against a sequential sum within 1e-13 of sum |x_i y_i|."""
    _, name, opts, kind, lanes = case
    B.set_options(**opts)
    n, ptr, col, val = matrix(B, name)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        for epi in range(4):
            buf = _arena(np.random.default_rng(epi + 31 * n), n)
            a = {k: buf[i].copy() for k, i in ARENA.items()}
            dots = (C.c_double * 8)()
            nd = B.lib.bicg_debug_spmv_epi(dm.h, epi, buf.ctypes.data_as(C.c_void_p), dots)
            y = O.spmv(n, ptr, col, val, a["p"], long_double=True)
            out = buf[ARENA["w"]] if epi == 3 else buf[ARENA["s"]]
            assert _rel(out, y) <= 1e-13, (epi, _rel(out, y))
            a["Y"] = O.spmv(n, ptr, col, val, a["p"])
            pairs = {0: [], 1: [("rh", "Y")], 2: [("r", "Y"), ("Y", "Y")],
                     3: [("rh", "r"), ("rh", "Y"), ("rh", "ax"), ("rh", "z")]}[epi]
            assert nd == len(pairs)
            for i, (u, v) in enumerate(pairs):
                want = math.fsum(a[u] * a[v])
                scale = float(np.abs(a[u] * a[v]).sum()) + 1e-300
                assert abs(dots[i] - want) <= 1e-13 * scale, (epi, i, u, v, dots[i], want)
    finally:
        dm.destroy()


# ---- nonzero initial guesses ------------------------------------------------------------------------------------------
# From x0 != 0 the init SpMV computes a real A x0, r0 = b - A x0 differs from b, r# = r0 and dot_zero = (r0, r0) are computed
# vectors and scalars, and the replacements of pipe_bicgstab_rr (k = 2 and 4) read the caller's b, which is no longer r0.
# (matrix, options at plan time, plan-shape check of the persistent kernel)
X0_MATRICES = [("small_n17", {}, None), ("small_n2113", {}, None), ("ragged_4001", {}, None), ("stencil15_g20", {}, None),
               ("stencil15_g58", dict(resident=1), _all_resident), ("stencil15_g60", dict(resident=0), _all_coded),
               (f"chunk_cap{cap_limit(512, 1)}", dict(mega_lanes=1), None)]


# the warm start on n = 17 under pipe_bicgstab_rr: after the replacement at k = 4 the case's own spread is 9e-10 (t), at k = 5
# 1.3e-8, so the states kept are k = 1, 2, 3 (the replacement at k = 2 among them)
X0_KS = {("small_n17", "pipe_bicgstab_rr", "warm"): (1, 2, 3)}


@pytest.mark.parametrize("x0_kind", X0_KINDS)
@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", X0_MATRICES, ids=[c[0] for c in X0_MATRICES])
def test_nonzero_x0_state(B, O, case, method, mega, x0_kind):
    name, opts, expect = case
    B.set_options(**opts)
    ks = X0_KS.get((name, method, x0_kind), KS)
    run_states(B, O, name, method, ks=ks, mega=mega, expect=expect if mega else None, x0_kind=x0_kind)


@pytest.mark.parametrize("case", STANDALONE, ids=[c[0] for c in STANDALONE])
def test_nonzero_x0_kernel_per_phase_state(B, O, case):
    """Every forced stand-alone SpMV variant computes the init's A x0; one method per variant, in turn."""
    _, name, opts, kind, lanes = case
    B.set_options(**opts)
    method = METHODS[STANDALONE.index(case) % len(METHODS)]
    run_states(B, O, name, method, ks=(1, 2), mega=0, expect=_plan(kind, lanes), x0_kind="normal")


@pytest.mark.parametrize("mega", [1, 0], ids=["mega", "multikernel"])
@pytest.mark.parametrize("method", METHODS)
def test_exact_initial_guess_does_no_iterations(B, O, method, mega):
    """x0 = x* with b = A x* from the library's own SpMV (dm.spmv: the plan and kernel of the init SpMV), so r0 = b - A x0 is
    exactly zero: 0 iterations, x returned bit for bit as given, r all zero, and a history of one entry, dot_r / dot_zero = 0 / 0,
    NaN as in the reference.  The nonzero-x0 counterpart of test_gpu_parity.py::test_zero_rhs_does_no_iterations."""
    n, ptr, col, val = matrix(B, "stencil15_g20")
    B.set_options(mega=mega, tol=1e-10, max_iter=100)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        xs = initial_guess("normal", n)
        b = dm.spmv(xs)
        x, r = xs.copy(), b.copy()
        it, st = dm.solve(method, x, r, **(RR_KW if method.endswith("rr") else {}))
        hist = B.last_history()
    finally:
        dm.destroy()
    assert it == st["iters"] == 0, it
    assert x.tobytes() == xs.tobytes()
    assert not np.any(r), np.abs(r).max()
    assert hist.size == 1 and np.isnan(hist[0]), hist
