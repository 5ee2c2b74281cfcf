"""GPU: the value gradient out_e = alpha sum_j u_j[i] v_j[c] (+ beta out_e) over the stored entries of a resident matrix
(bicg_matrix_value_grad, _async).  Its arithmetic is pinned down in include/bicgstab_b200.h, so every result is checked bit for
bit against a correctly rounded replica, across vector counts that fill, split and cross batches, for host, device and
stream-ordered calls, under forced SpMV kinds and lanes and every group width of the kernel (the result must not depend on
them), with rows split into diag and offd parts as on a handle with offd entries, and on a transpose handle in its own block
order.  The cases cover banded rows, long random rows (k = 32), T' with row-scaled values, the shifted golden matrix,
three dense rows far longer than the rest, and a hand-made matrix with a duplicate entry, an explicit zero and an empty column."""
import ctypes as C

import numpy as np
import pytest

from rowsum_model import value_grad as replica      # the header's arithmetic, correctly rounded, entry by entry
from test_gpu_set_values import _chunked_matrix
from test_gpu_transpose import _case_csr, transposed_csr

pytestmark = pytest.mark.gpu

CASES = ["convdiff", "random_k32", "tprime", "golden", "chunked", "handmade"]
NV_MAX = 8                                        # vectors per launch (MUL_NV_MAX of csrc/spmv.cuh)
NVECS = [1, 3, NV_MAX, NV_MAX + 1, 17]
LANES = [1, 2, 4, 8, 16, 32]                     # the group widths value_grad_kernel is instantiated for
COMBOS = [(1.0, 0.0), (-1.0, 0.0), (-0.75, 0.5), (2.5, -1.25), (-1.0, 1.0)]


@pytest.fixture(autouse=True)
def _opts(B):
    B.set_options(quiet=1, cache=1, spmv="auto", spmv_lanes=0)
    yield
    B.set_options(spmv="auto", spmv_lanes=0)


def _torch():
    import torch
    return torch


def _bits(a):
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


def csr_of(B, case):
    """(n, ptr, col, val) of the global CSR of A"""
    if case == "chunked":
        A = _chunked_matrix()
        return A.shape[0], A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.astype(np.float64)
    if case == "random_k32":
        blk = B.gen_block("random", 3001, 32)
        ptr, col, val = B.block_to_global_csr(blk)
        return blk.n, np.asarray(ptr, dtype=np.int64), np.asarray(col, dtype=np.int64), np.asarray(val, dtype=np.float64)
    return _case_csr(B, case)


def _uv(nvec, n, seed):
    rng = np.random.default_rng(seed + 97 * nvec)
    return rng.standard_normal((nvec, n)), rng.standard_normal((nvec, n))


@pytest.fixture(scope="module", params=CASES)
def case(request, B):
    B.set_options(quiet=1, cache=1, spmv="auto", spmv_lanes=0)
    n, ptr, col, val = csr_of(B, request.param)
    dm = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
    yield request.param, n, ptr, col, val, dm
    dm.destroy()


def test_matches_replica(B, case):
    """host, device and stream-ordered calls agree bit for bit with each other and with the replica on every entry, for
    vector counts 1, 3, 8, 9, 17, negative alpha, beta != 0 and a NaN-filled output at beta = 0"""
    torch = _torch()
    name, n, ptr, col, val, dm = case
    nnz = int(ptr[-1])
    rows = np.repeat(np.arange(n), np.diff(ptr))
    idx = np.arange(nnz)                             # every entry
    for i, nvec in enumerate(NVECS):
        alpha, beta = COMBOS[i % len(COMBOS)]
        u, v = _uv(nvec, n, 1)
        out0 = np.full(nnz, np.nan) if beta == 0.0 else np.random.default_rng(nvec).standard_normal(nnz)
        got_host, off = dm.value_grad(u, v, alpha, beta, diag_out=out0.copy())
        assert off is None
        td = torch.from_numpy(out0).cuda()
        got_dev, _ = dm.value_grad(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda(), alpha, beta, diag_out=td)
        ta = torch.from_numpy(out0).cuda()
        dm.value_grad_async(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda(), alpha, beta, diag_out=ta)
        torch.cuda.synchronize()
        assert not np.isnan(got_host).any(), (name, nvec)
        assert _bits(got_dev) == _bits(got_host) and _bits(ta) == _bits(got_host), (name, nvec, alpha, beta)
        want = replica(rows[idx], col[idx], u, v, alpha, beta, out0[idx])
        assert _bits(got_host[idx]) == _bits(want), (name, nvec, alpha, beta)
    # one vector of shape (n_loc,), outputs allocated
    u, v = _uv(1, n, 2)
    g1, _ = dm.value_grad(u[0], v[0])
    assert _bits(g1[idx]) == _bits(replica(rows[idx], col[idx], u, v, 1.0, 0.0, None))


def test_independent_of_plan_and_lanes(B, case):
    """The same bits from handles created under forced SpMV kinds and lanes per row, and from the kernel forced to every
    group width it is instantiated for (1 .. 32 threads per row)."""
    torch = _torch()
    name, n, ptr, col, val, dm = case
    u, v = (torch.from_numpy(a).cuda() for a in _uv(NV_MAX + 1, n, 3))
    want, _ = dm.value_grad_async(u, v, alpha=-1.0)
    torch.cuda.synchronize()
    forced = [("rowsplit", 1), ("rowsplit", 4), ("rowsplit", 32)] + ([("tma", 1), ("tma", 8)] if name != "chunked" else [])
    for kind, lanes in forced:
        B.set_options(spmv=kind, spmv_lanes=lanes)
        other = B.DeviceMatrix(B.blocks_from_csr(n, ptr, col, val))
        try:
            got, _ = other.value_grad_async(u, v, alpha=-1.0)
            torch.cuda.synchronize()
            assert _bits(got) == _bits(want), (name, kind, lanes)
        finally:
            other.destroy()
    try:
        for lanes in LANES:
            assert B.lib.bicg_debug_value_grad_layout(dm.h, lanes, None) == 0
            got, _ = dm.value_grad_async(u, v, alpha=-1.0)
            torch.cuda.synchronize()
            assert _bits(got) == _bits(want), (name, lanes)
    finally:
        B.lib.bicg_debug_value_grad_layout(dm.h, 0, None)


def test_split_rows_through_merge_row(B, case):
    """The path of a handle with offd entries at one rank: every merged row taken as a diag part (its first half) and an offd
    part (the rest) through bicg_debug_value_grad_layout, so the kernel places each entry through merge_row, split over every
    group width.  diag_out and offd_out are the halves of the unsplit output, bit for bit."""
    torch = _torch()
    name, n, ptr, col, val, dm = case
    rl = np.diff(ptr)
    dl = rl // 2
    dptr = np.concatenate([[0], np.cumsum(dl)])
    optr = np.concatenate([[0], np.cumsum(rl - dl)])
    blk = torch.from_numpy(np.concatenate([dptr, optr]).astype(np.uint32).view(np.int32)).cuda()
    in_diag = np.arange(int(ptr[-1])) - np.repeat(ptr[:-1], rl) < np.repeat(dl, rl)
    u, v = (torch.from_numpy(a).cuda() for a in _uv(NV_MAX + 1, n, 5))
    whole, _ = dm.value_grad_async(u, v, alpha=0.5)
    torch.cuda.synchronize()
    whole = whole.cpu().numpy()
    try:
        for lanes in LANES:
            assert B.lib.bicg_debug_value_grad_layout(dm.h, lanes, C.c_void_p(blk.data_ptr())) == 0
            d = torch.full((int(dptr[-1]),), np.nan, dtype=torch.float64, device="cuda")
            o = torch.full((max(int(optr[-1]), 1),), np.nan, dtype=torch.float64, device="cuda")
            rc = B.lib.bicg_matrix_value_grad_async(dm.h, NV_MAX + 1, C.c_void_p(u.data_ptr()), C.c_void_p(v.data_ptr()),
                                                    0.5, 0.0, C.c_void_p(d.data_ptr()), C.c_void_p(o.data_ptr()),
                                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))
            assert rc == 0
            torch.cuda.synchronize()
            assert _bits(d) == _bits(whole[in_diag]), (name, lanes)
            assert _bits(o[:int(optr[-1])]) == _bits(whole[~in_diag]), (name, lanes)
    finally:
        B.lib.bicg_debug_value_grad_layout(dm.h, 0, None)
        torch.cuda.synchronize()


def test_transpose_handle_in_its_own_order(B, case):
    """A transpose's gradient is in its own block order: bit for bit that of a handle created from the transposed blocks, and
    the replica on the transposed CSR."""
    name, n, ptr, col, val, dm = case
    mt = dm.transpose()
    tp, tc, tv = transposed_csr(n, ptr, col, val)
    fresh = B.DeviceMatrix(B.blocks_from_csr(n, tp, tc, tv))
    try:
        u, v = _uv(3, n, 4)
        got, _ = mt.value_grad(u, v, alpha=-1.0)
        assert _bits(got) == _bits(fresh.value_grad(u, v, alpha=-1.0)[0]), name
        idx = np.arange(int(tp[-1]))
        trows = np.repeat(np.arange(n), np.diff(tp))
        assert _bits(got[idx]) == _bits(replica(trows[idx], tc[idx], u, v, -1.0, 0.0, None)), name
    finally:
        mt.destroy()
        fresh.destroy()
