"""The evict-first accesses of the persistent BiCGStab loop leave s = A p bit for bit at every stop (-m gpu).

mega.cu's run_bicgstab marks the r# load of s = A p, the x, y and r# accesses of the x / r update and the s load of the
p update evict-first in L2 (its policy table).  The policy changes where a line lives, never a value: a hinted access that
read or wrote the wrong address, or a stale line, shows up as rows of s that are not A p.  A solve stopped by max_iter after
iteration k ends after the beta reduction and skips that iteration's p update, so the arena's p is still the vector that
s = A p was computed from: s must equal the row sums of tests/rowsum_model.py on p bit for bit, on every row.  The
loop-state tolerances would not see a few wrong rows; this does.

The cases: a small stencil (every CTA a few 16-row groups, slices resident in shared memory), a T'-shaped stencil whose CTAs
stream their tiles like the benchmark's, and 16 x 132 + 1 rows, whose last CTA ends in a one-row tail of the vector phases."""
import ctypes as C

import numpy as np
import pytest

import rowsum_model as M
from loop_reference import ARENA
from state_check import matrix

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 5)
CASES = [("stencil15_g20", dict(resident=1)), ("stencil15_g60", dict(resident=0)), ("small_n2113", dict(resident=1))]
DEFAULTS = dict(quiet=1, tol=1e-15, max_iter=1000, mega=1, resident=1, mega_threads=0, mega_lanes=0, spmv="auto",
                spmv_lanes=0, spmv_threads=0, spmv_stages=0, autotune=1)


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(**(DEFAULTS | dict(autotune=0)))
    yield
    B.set_options(**DEFAULTS)


def _arena(B, dm, n, name):
    out = np.empty(n)
    assert B.lib.bicg_debug_get_vec(dm.h, ARENA[name], out.ctypes.data_as(C.c_void_p)) == 0
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_s_is_a_p_after_every_stop(B, O, case):
    name, opts = case
    B.set_options(mega=1, mega_lanes=1, **opts)
    n, ptr, col, val = matrix(B, name)
    b = O.spmv(n, ptr, col, val, np.ones(n))
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    try:
        for k in KS:
            B.set_options(tol=0.0, max_iter=k)
            x, r = np.zeros(n), b.copy()
            it, st = dm.solve("bicgstab", x, r)
            assert it == k and st["kernel_launches"] == 3, (k, it, st["kernel_launches"])    # the loop ran as ONE kernel
            p, s = _arena(B, dm, n, "p"), _arena(B, dm, n, "s")
            want = M.row_sums(ptr, col, val, p, 1)
            bad = np.flatnonzero(s.view(np.uint64) != want.view(np.uint64))
            assert bad.size == 0, (f"{name} k={k}: {bad.size} of {n} rows of s differ from A p, first rows "
                                   f"{bad[:8].tolist()}: {s[bad[:4]].tolist()} vs {want[bad[:4]].tolist()}")
    finally:
        dm.destroy()
