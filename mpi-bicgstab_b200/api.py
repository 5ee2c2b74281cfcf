"""Python mirror of the reference's operator interface for the BiCGStab hot path.

Same names, argument meaning and error behaviour as solver.h:10-13 / matrix.h:44-51 of the reference, on
numpy arrays instead of raw pointers; every call goes straight through the C ABI of libbicgstab_b200.so
(include/bicgstab_b200.h) -- nothing is computed in Python.

    blk = gen_block("stencil15", 24, diag=16.0)            # or load_matrix_block("A.mtx"), or blocks_from_csr(...)
    b = spmv_ovlap(blk, np.ones(blk.n_loc))                  # main.c:109-113
    x = np.zeros(blk.n_loc)
    iters = bicgstab(blk, x, b)                              # x: solution, b: final recursive residual
"""
import ctypes as C

import numpy as np

from ._lib import ALLGATHER_FN, CSR_Matrix, INFO_Matrix, bicg_result, bicg_shift_result, bicg_stats, lib

METHODS = {"bicgstab": 0, "ca_bicgstab": 1, "pipe_bicgstab": 2, "pipe_bicgstab_rr": 3}
SHIFTED_METHODS = {"shifted_lopbicg_switching": 0, "shifted_lopbicgstab": 1, "shifted_pipe_lopbicgstab": 2}
# every method bicg_shifted_solve_ex accepts: SHIFTED_METHODS plus the fixed-seed shifted_lopbicg
SHIFTED_SOLVE_EX = dict(SHIFTED_METHODS, shifted_lopbicg=3)
GEN_KINDS = {"stencil15": 0, "laplace5": 1, "random": 2, "convdiff": 3}


def _dptr(a):
    return a.ctypes.data_as(C.c_void_p)


class MatrixBlock:
    """One rank's (A_loc_diag, A_loc_offd, A_info) triple -- what the reference's entry points take."""

    def __init__(self, world):
        self.diag = CSR_Matrix()
        self.offd = CSR_Matrix()
        self.info = INFO_Matrix()
        self._recvcounts = (C.c_int * world)()
        self._displs = (C.c_int * world)()
        self.info.recvcounts = C.cast(self._recvcounts, C.POINTER(C.c_int))
        self.info.displs = C.cast(self._displs, C.POINTER(C.c_int))
        self.world = world
        self._keep = []            # numpy arrays backing the CSR pointers (when Python owns them)
        self._lib_owned = False    # True: arrays were malloc'ed by the library -> csr_free_matrix

    # -- views ---------------------------------------------------------------------------------------
    @property
    def n_loc(self):
        return int(self.diag.rows)

    @property
    def n(self):
        return int(self.info.rows)

    @property
    def nnz_loc(self):
        return int(self.diag.nz) + int(self.offd.nz)

    @property
    def recvcounts(self):
        return np.array(self._recvcounts[:], dtype=np.int32)

    @property
    def displs(self):
        return np.array(self._displs[:], dtype=np.int32)

    @staticmethod
    def _view(m):
        nz, rows = int(m.nz), int(m.rows)
        val = np.ctypeslib.as_array(m.val, shape=(nz,)) if nz else np.zeros(0)
        col = np.ctypeslib.as_array(m.col, shape=(nz,)) if nz else np.zeros(0, dtype=np.uint32)
        ptr = np.ctypeslib.as_array(m.ptr, shape=(rows + 1,))
        return val, col, ptr

    def diag_arrays(self):
        return self._view(self.diag)

    def offd_arrays(self):
        return self._view(self.offd)

    def free(self):
        if self._lib_owned:
            lib.csr_free_matrix(C.byref(self.diag))
            lib.csr_free_matrix(C.byref(self.offd))
            self._lib_owned = False
        else:
            lib.bicg_matrix_invalidate(C.byref(self.diag))
        self._keep = []

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def plan_partition(n, world):
    """matrix.c:295-308."""
    cnt = (C.c_int * world)()
    dsp = (C.c_int * world)()
    lib.bicg_plan_partition(n, world, cnt, dsp)
    return np.array(cnt[:], dtype=np.int64), np.array(dsp[:], dtype=np.int64)


def _fill_csr(m, val, col, ptr, rows, cols, keep):
    val = np.ascontiguousarray(val, dtype=np.float64)
    col = np.ascontiguousarray(col, dtype=np.uint32)
    ptr = np.ascontiguousarray(ptr, dtype=np.uint32)
    if val.size == 0:               # keep non-null pointers like malloc(0) would
        val = np.zeros(1, dtype=np.float64)
        col = np.zeros(1, dtype=np.uint32)
    keep += [val, col, ptr]
    m.val = val.ctypes.data_as(C.POINTER(C.c_double))
    m.col = col.ctypes.data_as(C.POINTER(C.c_uint))
    m.ptr = ptr.ctypes.data_as(C.POINTER(C.c_uint))
    m.nz = int(ptr[-1])
    m.rows = rows
    m.cols = cols


def blocks_from_csr(n, ptr, col, val, rank=0, world=1):
    """Split a global CSR into rank's diag / offd blocks exactly as the reference's block loader does
    (partition matrix.c:295-308; diag: local columns, offd: global columns, in-row order kept,
    matrix.c:380-392)."""
    ptr = np.asarray(ptr, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    val = np.asarray(val, dtype=np.float64)
    cnt, dsp = plan_partition(n, world)
    lo, nloc = int(dsp[rank]), int(cnt[rank])
    hi = lo + nloc
    a, b = int(ptr[lo]), int(ptr[hi])
    c, v = col[a:b], val[a:b]
    rows = np.repeat(np.arange(nloc), np.diff(ptr[lo:hi + 1]))
    own = (c >= lo) & (c < hi)
    blk = MatrixBlock(world)
    for mask, m, shift, ncols in ((own, blk.diag, lo, nloc), (~own, blk.offd, 0, n)):
        r = rows[mask]
        p = np.zeros(nloc + 1, dtype=np.int64)
        np.add.at(p, r + 1, 1)
        p = np.cumsum(p)
        _fill_csr(m, v[mask], c[mask] - shift, p, nloc, ncols, blk._keep)
    blk.info.nz = int(ptr[-1]) & 0xFFFFFFFF
    blk.info.rows = n
    blk.info.cols = n
    blk.info.code = b"MCRG"
    for p_ in range(world):
        blk._recvcounts[p_] = int(cnt[p_])
        blk._displs[p_] = int(dsp[p_])
    return blk


def gen_block(kind, g, p0=0.0, seed=12345, rank=0, world=1):
    """Synthetic inputs of SURVEY.md 8(d) (csrc/gen.cpp), generated directly as one rank's blocks."""
    blk = MatrixBlock(world)
    rc = lib.bicg_gen_block(GEN_KINDS[kind], int(g), float(p0), int(seed), rank, world,
                            C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info))
    if rc != 0:
        raise ValueError(f"bicg_gen_block({kind}, g={g}) failed with {rc}")
    blk._lib_owned = True
    return blk


def load_matrix_block(filename, world=None):
    """MPI_csr_load_matrix_block (matrix.h:50): Matrix-Market file -> this rank's blocks."""
    world = world or lib.bicg_comm_world()
    blk = MatrixBlock(world)
    lib.MPI_csr_load_matrix_block(str(filename).encode(), C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info))
    blk._lib_owned = True
    return blk


def block_to_global_csr(blk, rank=0):
    """(ptr, col, val) of the block's rows with GLOBAL column indices, diag entries first then offd
    (the order the reference accumulates them in, matrix.c:437-440)."""
    dv, dc, dp = blk.diag_arrays()
    ov, oc, op_ = blk.offd_arrays()
    lo = int(blk.displs[rank])
    nloc = blk.n_loc
    ptr = dp.astype(np.int64) + op_.astype(np.int64)
    col = np.empty(int(ptr[-1]), dtype=np.int64)
    val = np.empty(int(ptr[-1]), dtype=np.float64)
    dlen, olen = np.diff(dp.astype(np.int64)), np.diff(op_.astype(np.int64))
    row_d = np.repeat(np.arange(nloc), dlen)
    row_o = np.repeat(np.arange(nloc), olen)
    pos_d = ptr[row_d] + (np.arange(dlen.sum()) - dp.astype(np.int64)[row_d])
    pos_o = ptr[row_o] + dlen[row_o] + (np.arange(olen.sum()) - op_.astype(np.int64)[row_o])
    col[pos_d] = dc.astype(np.int64)[:dlen.sum()] + lo
    val[pos_d] = dv[:dlen.sum()]
    col[pos_o] = oc.astype(np.int64)[:olen.sum()]
    val[pos_o] = ov[:olen.sum()]
    return ptr, col, val


# ---- the reference's entry points ------------------------------------------------------------------------
def _vec(a, n):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"] and a.size >= n, "need a contiguous float64 vector"
    return _dptr(a)


def spmv_ovlap(blk, x_loc, x_scratch=None, y_loc=None):
    """MPI_csr_spmv_ovlap (matrix.h:51): y_loc = A x.  Returns y_loc."""
    if y_loc is None:
        y_loc = np.empty(blk.n_loc)
    if x_scratch is None:
        x_scratch = np.zeros(blk.n)
    lib.MPI_csr_spmv_ovlap(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _vec(x_loc, blk.n_loc),
                           _vec(x_scratch, blk.n), _vec(y_loc, blk.n_loc))
    return y_loc


def bicgstab(blk, x_loc, r_loc):
    return lib.bicgstab(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _vec(x_loc, blk.n_loc), _vec(r_loc, blk.n_loc))


def ca_bicgstab(blk, x_loc, r_loc):
    return lib.ca_bicgstab(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _vec(x_loc, blk.n_loc), _vec(r_loc, blk.n_loc))


def pipe_bicgstab(blk, x_loc, r_loc):
    return lib.pipe_bicgstab(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _vec(x_loc, blk.n_loc), _vec(r_loc, blk.n_loc))


def pipe_bicgstab_rr(blk, x_loc, r_loc, krr, nrr):
    return lib.pipe_bicgstab_rr(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _vec(x_loc, blk.n_loc),
                                _vec(r_loc, blk.n_loc), int(krr), int(nrr))


def solve(method, blk, x_loc, r_loc, krr=0, nrr=0):
    if method == "pipe_bicgstab_rr":
        return pipe_bicgstab_rr(blk, x_loc, r_loc, krr, nrr)
    return {"bicgstab": bicgstab, "ca_bicgstab": ca_bicgstab, "pipe_bicgstab": pipe_bicgstab}[method](blk, x_loc, r_loc)


def shifted_lopbicg_switching(blk, x_set, r_loc, sigma, seed):
    """shifted_switching_solver.h:12.  x_set: (sigma_len, n_loc) C-contiguous; returns the reference's k (iterations + 1)."""
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    assert x_set.dtype == np.float64 and x_set.flags["C_CONTIGUOUS"] and x_set.shape == (sigma.size, blk.n_loc)
    return lib.shifted_lopbicg_switching(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), _dptr(x_set), _vec(r_loc, blk.n_loc),
                                         _dptr(sigma), int(sigma.size), int(seed))


def _shifted_args(blk, x_set, r_loc, sigma):
    sigma = np.ascontiguousarray(sigma, dtype=np.float64)
    assert x_set.dtype == np.float64 and x_set.flags["C_CONTIGUOUS"] and x_set.shape == (sigma.size, blk.n_loc)
    return _dptr(x_set), _vec(r_loc, blk.n_loc), sigma


def shifted_lopbicg(blk, x_set, r_loc, sigma, seed):
    """shifted_switching_solver.h:11, the fixed-seed variant of shifted_lopbicg_switching (same arguments).  Returns the
    iterations performed (not + 1)."""
    xp, rp, sigma = _shifted_args(blk, x_set, r_loc, sigma)
    return lib.shifted_lopbicg(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), xp, rp, _dptr(sigma), int(sigma.size), int(seed))


def shifted_lopbicgstab(blk, x_set, r_loc, sigma, seed):
    """shifted_solver.h:17 (LOP; its _v2 / _nooverlap twins are the same solve).  x_set: (sigma_len, n_loc) C-contiguous;
    returns the iterations performed."""
    xp, rp, sigma = _shifted_args(blk, x_set, r_loc, sigma)
    return lib.shifted_lopbicgstab(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), xp, rp, _dptr(sigma), int(sigma.size), int(seed))


def shifted_pipe_lopbicgstab(blk, x_set, r_loc, sigma, seed):
    """shifted_solver.h:20 (PIPE-LOP; its _nooverlap twin is the same solve).  Same arguments and return value as
    shifted_lopbicgstab."""
    xp, rp, sigma = _shifted_args(blk, x_set, r_loc, sigma)
    return lib.shifted_pipe_lopbicgstab(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info), xp, rp, _dptr(sigma), int(sigma.size),
                                        int(seed))


def _cuda_vectors(*args):
    """Device pointers of CUDA float64 torch tensors, given as (name, tensor, expected shape) triples, checked by
    _checked_cuda_vectors.  Then torch's current stream is synchronised, because the library works on its own stream."""
    import torch
    ptrs = _checked_cuda_vectors(*args)
    torch.cuda.current_stream(args[0][1].device).synchronize()
    return ptrs


def _checked_cuda_vectors(*args):
    """Device pointers of CUDA float64 torch tensors, given as (name, tensor, expected shape) triples.  Everything the library
    cannot check itself is checked here, before it is called: all are torch tensors, float64, contiguous, of the expected shape,
    on the library's GPU."""
    import torch
    checks = [(lambda t, s: isinstance(t, torch.Tensor), TypeError,
               lambda t, s: f"numpy arrays and torch tensors cannot be mixed in one call (got {type(t).__name__})"),
              (lambda t, s: t.dtype == torch.float64, TypeError, lambda t, s: f"need a float64 tensor, got {t.dtype}"),
              (lambda t, s: t.is_contiguous(), ValueError, lambda t, s: "need a contiguous tensor"),
              (lambda t, s: tuple(t.shape) == tuple(s), ValueError, lambda t, s: f"shape {tuple(t.shape)}, expected {tuple(s)}"),
              (lambda t, s: t.is_cuda, TypeError, lambda t, s: f"need a CUDA tensor, got one on {t.device}")]
    for ok, exc, msg in checks:              # each check over every argument before the next one
        for name, t, shape in args:
            if not ok(t, shape):
                raise exc(f"{name}: {msg(t, shape)}")
    dev = lib.bicg_device()
    for name, t, _ in args:
        if t.device.index != dev:
            raise ValueError(f"{name}: tensor on {t.device}, the library runs on cuda:{dev}")
    return [C.c_void_p(t.data_ptr()) for _, t, _ in args]


def _value_args(blk, diag_val, offd_val):
    """(name, array, expected shape) of new values for blk's blocks; offd_val may be None only where the handle has no offd
    entries (one rank, or an empty offd block)."""
    args = [("diag_val", diag_val, (int(blk.diag.nz),))]
    if offd_val is not None:
        args.append(("offd_val", offd_val, (int(blk.offd.nz),)))
    elif int(blk.offd.nz) and lib.bicg_comm_world() > 1:
        raise ValueError(f"offd_val: the offd block has {int(blk.offd.nz)} entries, got None")
    return args


def _checked_host_vectors(*args):
    """Pointers of numpy float64 arrays, given as (name, array, expected shape) triples: contiguous, of the expected shape."""
    for name, a, shape in args:
        if a.dtype != np.float64:
            raise TypeError(f"{name}: need a float64 array, got {a.dtype}")
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError(f"{name}: need a contiguous array")
        if a.shape != tuple(shape):
            raise ValueError(f"{name}: shape {a.shape}, expected {tuple(shape)}")
    return [_dptr(a) for _, a, _ in args]


def _host_sigma(sigma):
    """sigma as a contiguous float64 numpy array; a torch tensor (on any device) is copied to the host."""
    if not isinstance(sigma, np.ndarray) and hasattr(sigma, "detach"):
        sigma = sigma.detach().cpu().numpy()
    return np.ascontiguousarray(sigma, dtype=np.float64)


def last_shift_info(sigma_len):
    seed = C.c_int()
    stop = (C.c_int * sigma_len)()
    lib.bicg_last_shift_info(C.byref(seed), stop, sigma_len)
    return seed.value, np.array(stop[:])


def last_shift_error(sigma_len):
    """||(A + sigma_j I) x_j - b|| / ||b|| of every shift of the last shifted solve run with the option shift_error=1
    (BICG_SHIFT_ERROR); an empty array if it ran without it."""
    out = np.zeros(max(int(sigma_len), 1))
    n = lib.bicg_last_shift_error(out.ctypes.data_as(C.POINTER(C.c_double)), int(sigma_len))
    return out[:min(n, int(sigma_len))]


# ---- extensions ------------------------------------------------------------------------------------------
def set_option(key, value):
    if lib.bicg_set_option(str(key).encode(), str(value).encode()) != 0:
        raise KeyError(key)


def set_options(**kw):
    for k, v in kw.items():
        set_option(k.upper(), v)


def last_history():
    """dot_r/dot_zero after every iteration of the last solve on this rank (entry 0 = 1)."""
    n = lib.bicg_last_history(None, 0)
    out = np.empty(max(n, 1))
    lib.bicg_last_history(out.ctypes.data_as(C.POINTER(C.c_double)), n)
    return out[:n]


def _decode_record(t, stream, rec):
    if stream is not None:
        stream.synchronize()
    raw = bytes(t.detach().cpu().numpy().tobytes()) if hasattr(t, "detach") else bytes(np.asarray(t, dtype=np.uint8))
    if len(raw) != C.sizeof(rec):
        raise ValueError(f"a {rec.__name__} has {C.sizeof(rec)} bytes, got {len(raw)}")
    r = rec.from_buffer_copy(raw)
    return {f: getattr(r, f) for f, _ in rec._fields_ if f != "reserved"}


def decode_result(t, stream=None):
    """The bicg_result an asynchronous solve wrote into the 24-byte tensor `t`, as a dict with iters, converged, error and
    final_res.  The copy to the host is ordered after torch's current stream only: pass the stream the solve was enqueued on
    when it was another one, and it is synchronised first (or synchronise it yourself)."""
    return _decode_record(t, stream, bicg_result)


def decode_shift_result(t, stream=None):
    """The bicg_shift_result an asynchronous shifted solve wrote into the 32-byte tensor `t`, as a dict with ret, iters,
    converged, seed, error and final_res; `stream` as in decode_result."""
    return _decode_record(t, stream, bicg_shift_result)


def _result_tensor(result, nbytes, device, stream):
    """`result` checked, or a new one of nbytes that is written on `stream`"""
    import torch
    if result is None:
        result = torch.empty(nbytes, dtype=torch.uint8, device=device)
        result.record_stream(stream)          # written on `stream`, which need not be the one it was allocated on
    elif not (isinstance(result, torch.Tensor) and result.is_cuda and result.dtype == torch.uint8 and result.is_contiguous()
              and result.numel() == nbytes and result.device == device and result.data_ptr() % 8 == 0):
        raise ValueError(f"result: need a contiguous, 8-byte aligned uint8 CUDA tensor of {nbytes} elements on {device}")
    return result


def _stats_dict(s):
    return {f: getattr(s, f) for f, _ in bicg_stats._fields_}


def last_stats():
    return _stats_dict(lib.bicg_last_stats().contents)


class _CountBlock:
    def __init__(self, nz):
        self.nz = nz


class _HandleShape:
    """What a DeviceMatrix needs of its MatrixBlock, for a handle the library built (a transpose): no host arrays."""

    def __init__(self, n_loc, n, diag_nz, offd_nz):
        self.n_loc, self.n = n_loc, n
        self.diag, self.offd = _CountBlock(diag_nz), _CountBlock(offd_nz)


class DeviceMatrix:
    """A device-resident matrix handle (bicg_matrix): upload once, solve / multiply many times."""

    _t = None                  # the transpose prepare_autograd made (or the first backward that needed one)
    _src = None                # on that transpose: the handle it was made from (not owned; destroy() leaves it alone)

    def __init__(self, blk, handle=None):
        """blk: the MatrixBlock to upload; or, with `handle`, an existing bicg_matrix that this object takes over (then blk only
        describes its shape: n_loc, n and the diag.nz / offd.nz that set_values takes)."""
        self.blk = blk
        self.h = handle if handle is not None else lib.bicg_matrix_create(C.byref(blk.diag), C.byref(blk.offd), C.byref(blk.info))
        if not self.h:
            raise RuntimeError("bicg_matrix_create failed")

    def transpose(self):
        """bicg_matrix_create_transpose: a new DeviceMatrix holding A^T with this handle's row partition, its own plans and
        arena, independent of this one once created.  Row j holds the entries (i, j) of A by ascending i (equal (i, j) in
        their order in row i of A), diag columns first: results are bit-identical to a DeviceMatrix on
        blocks_from_csr of that global CSR.  Collective over the ranks."""
        h = lib.bicg_matrix_create_transpose(self.h)
        if not h:
            raise RuntimeError("bicg_matrix_create_transpose failed")
        dnz, onz = C.c_uint(), C.c_uint()
        lib.bicg_matrix_block_nz(h, C.byref(dnz), C.byref(onz))
        return DeviceMatrix(_HandleShape(self.blk.n_loc, self.blk.n, dnz.value, onz.value), handle=h)

    def transpose_values(self, src):
        """bicg_matrix_transpose_values: this transpose's values become src^T for src's current values, where src is the
        DeviceMatrix it was made from.  Returns once done.  Collective over the ranks."""
        if not isinstance(src, DeviceMatrix):
            raise TypeError(f"src: need a DeviceMatrix, got {type(src).__name__}")
        rc = lib.bicg_matrix_transpose_values(self.h, src.h)
        if rc != 0:
            raise ValueError(f"bicg_matrix_transpose_values failed with {rc} (src is not the matrix this one was transposed from)")

    def transpose_values_async(self, src, stream=None):
        """bicg_matrix_transpose_values_async: transpose_values enqueued on `stream` (default: torch's current stream) behind both
        handles' earlier work, and both handles' next work waits for it; no host synchronisation.  src's values are read in
        stream order, so a replay of a captured refresh reads them as they are then; works inside torch.cuda.graph with no
        prepare step.  Collective over the ranks."""
        import torch
        if not isinstance(src, DeviceMatrix):
            raise TypeError(f"src: need a DeviceMatrix, got {type(src).__name__}")
        if stream is None:
            stream = torch.cuda.current_stream(torch.device("cuda", lib.bicg_device()))
        rc = lib.bicg_matrix_transpose_values_async(self.h, src.h, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_transpose_values_async failed with {rc} (src is not the matrix this one was transposed "
                             f"from)")

    def set_values(self, diag_val, offd_val=None):
        """bicg_matrix_set_values: new values for the pattern the handle was created with, in the order of blk's diag and offd
        blocks (blk.diag.nz and blk.offd.nz of them; offd_val may be None where the handle has no offd entries).  Both numpy
        float64 arrays, or both contiguous CUDA float64 tensors (read after torch's current stream has been synchronised).
        Returns once the values are in place; every later result equals that of a handle freshly created from the new values.
        Rank-local: each rank sets its own rows.  blk's host arrays keep the old values: they no longer describe the device
        matrix."""
        args = _value_args(self.blk, diag_val, offd_val)
        if all(isinstance(a, np.ndarray) for _, a, _ in args):
            ptrs, dev = _checked_host_vectors(*args), 0
        else:
            ptrs, dev = _cuda_vectors(*args), 1
        rc = lib.bicg_matrix_set_values(self.h, ptrs[0], ptrs[1] if len(ptrs) > 1 else None, dev)
        if rc != 0:
            raise ValueError(f"bicg_matrix_set_values failed with {rc}")

    def set_values_async(self, diag_val, offd_val=None, stream=None):
        """bicg_matrix_set_values_async: set_values on contiguous CUDA float64 tensors only, enqueued on `stream` (default: torch's
        current stream) behind the handle's earlier work, with no host synchronisation.  The tensors are read in stream order,
        so a replay of a captured update reads them as they are then; works inside torch.cuda.graph with no prepare step.  blk's
        host arrays no longer describe the device matrix afterwards."""
        import torch
        args = _value_args(self.blk, diag_val, offd_val)
        for name, a, _ in args:
            if not isinstance(a, torch.Tensor):
                raise TypeError(f"{name}: set_values_async takes CUDA tensors only, got {type(a).__name__}")
        ptrs = _checked_cuda_vectors(*args)
        if stream is None:
            stream = torch.cuda.current_stream(diag_val.device)
        rc = lib.bicg_matrix_set_values_async(self.h, ptrs[0], ptrs[1] if len(ptrs) > 1 else None, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_set_values_async failed with {rc}")

    def shift_diagonal(self, sigma):
        """bicg_matrix_shift_diagonal: A_diag += sigma I on the device, like csr_shift_diagonal on the host blocks (the first
        entry of every own row whose column is that row; calls accumulate).  Raises ValueError, with no value changed, when a
        row of this rank has no diagonal entry.  blk's host arrays no longer describe the device matrix afterwards."""
        if lib.bicg_matrix_shift_diagonal(self.h, float(sigma)) != 0:
            raise ValueError("bicg_matrix_shift_diagonal failed: a row of this rank has no diagonal entry (no value was changed)")

    def shift_diagonal_async(self, sigma, stream=None):
        """bicg_matrix_shift_diagonal_async: shift_diagonal by the value a CUDA float64 tensor of one element holds (a view
        sigma[j:j+1] works), enqueued on `stream` (default: torch's current stream) behind the handle's earlier work, with no host
        synchronisation; the value is read in stream order, so a replay of a captured shift adds what the tensor holds then.
        Bit-identical to shift_diagonal by that value.  Inside torch.cuda.graph, call prepare_shift_diagonal_async first; an
        uncaptured call runs it itself the first time, which makes that call collective.  Raises ValueError, with no value
        changed, when a row has no diagonal entry."""
        import torch
        if not isinstance(sigma, torch.Tensor):
            raise TypeError(f"sigma: shift_diagonal_async takes a CUDA tensor, got {type(sigma).__name__}")
        (sp_,) = _checked_cuda_vectors(("sigma", sigma, (1,)))
        if stream is None:
            stream = torch.cuda.current_stream(sigma.device)
        rc = lib.bicg_matrix_shift_diagonal_async(self.h, sp_, C.c_void_p(stream.cuda_stream))
        if rc == -2:
            raise RuntimeError("shift_diagonal_async inside a stream capture needs prepare_shift_diagonal_async() first")
        if rc != 0:
            raise ValueError("bicg_matrix_shift_diagonal_async failed: a row has no diagonal entry (no value was changed)")

    def prepare_shift_diagonal_async(self):
        """bicg_matrix_shift_diagonal_async_prepare: find the diagonal positions shift_diagonal_async needs, outside any capture.
        Collective over the ranks; raises ValueError on every rank when a row of any rank has no diagonal entry."""
        if lib.bicg_matrix_shift_diagonal_async_prepare(self.h) != 0:
            raise ValueError("bicg_matrix_shift_diagonal_async_prepare failed: a row has no diagonal entry (on this or another rank)")

    def dots_async(self, u, v, out=None, stream=None):
        """bicg_matrix_dots_async: out[j] = <u_j, v_j> summed over every rank's rows, for u and v contiguous CUDA float64 tensors
        of shape (n_loc,) or (nvec, n_loc) (the rows of the x_set layout), in the fixed order the header gives; every rank gets
        the same bits.  out: a contiguous CUDA float64 tensor of shape (nvec,), allocated when None.  Enqueued on `stream`
        (default: torch's current stream) behind the handle's earlier work with no host synchronisation; works inside
        torch.cuda.graph with no prepare step.  Collective over the ranks.  Returns out."""
        import torch
        for name, t in (("u", u), ("v", v), ("out", out)):
            if t is not None and not isinstance(t, torch.Tensor):
                raise TypeError(f"{name}: dots_async takes CUDA tensors only, got {type(t).__name__}")
        shape = self._multiply_shape(u)
        nvec = shape[0] if len(shape) == 2 else 1
        given = out is not None
        if not given:
            out = u.new_empty((nvec,), dtype=u.dtype)
        up, vp, op_ = _checked_cuda_vectors(("u", u, shape), ("v", v, shape), ("out", out, (nvec,)))
        if stream is None:
            stream = torch.cuda.current_stream(u.device)
        if not given and stream != torch.cuda.current_stream(u.device):
            out.record_stream(stream)             # written on `stream`, not on the one it was allocated on
        rc = lib.bicg_matrix_dots_async(self.h, nvec, up, vp, op_, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_dots_async failed with {rc}")
        return out

    def solve(self, method, x, r, krr=0, nrr=0):
        """bicg_solve: x (initial guess in, solution out) and r (b in, final residual out) are both numpy float64 arrays, or both
        contiguous CUDA float64 torch tensors of shape (n_loc,), which are updated in place.  Returns (iterations, stats)."""
        n = self.blk.n_loc
        if isinstance(x, np.ndarray) and isinstance(r, np.ndarray):
            xp, rp, dev = _vec(x, n), _vec(r, n), 0
        else:
            (xp, rp), dev = _cuda_vectors(("x", x, (n,)), ("r", r, (n,))), 1
        st = bicg_stats()
        it = lib.bicg_solve(self.h, METHODS[method], xp, rp, krr, nrr, dev, C.byref(st))
        return it, _stats_dict(st)

    def solve_async(self, method, x, r, krr=0, nrr=0, result=None, stream=None):
        """bicg_solve_async: the solve of solve() on CUDA tensors, enqueued on `stream` (default: torch's current stream) without
        waiting for it or for anything before it.  x (initial guess in, solution out) and r (b in, final residual out) are
        contiguous CUDA float64 tensors of shape (n_loc,), updated in place in stream order.  `result`: a 24-byte uint8 CUDA
        tensor that receives the bicg_result (decode_result reads it); allocated when not given.  Works inside
        torch.cuda.graph once prepare_async(method) has been called.  Returns the result tensor."""
        import torch
        n = self.blk.n_loc
        xp, rp = _checked_cuda_vectors(("x", x, (n,)), ("r", r, (n,)))
        if stream is None:
            stream = torch.cuda.current_stream(x.device)
        result = _result_tensor(result, C.sizeof(bicg_result), x.device, stream)
        rc = lib.bicg_solve_async(self.h, METHODS[method], xp, rp, int(krr), int(nrr), C.c_void_p(stream.cuda_stream),
                                  C.c_void_p(result.data_ptr()))
        if rc == -2:
            raise RuntimeError(f"solve_async inside a stream capture needs prepare_async({method!r}) first")
        if rc != 0:
            raise ValueError(f"bicg_solve_async failed with {rc}")
        return result

    def prepare_async(self, method):
        """bicg_solve_async_prepare: build what solve_async needs for `method` under the current options, outside any capture."""
        if lib.bicg_solve_async_prepare(self.h, METHODS[method]) != 0:
            raise ValueError(f"bicg_solve_async_prepare({method}) failed")

    def history(self):
        """bicg_matrix_history: dot_r/dot_zero after every iteration of the last solve enqueued on this handle, synchronous or
        asynchronous (waits for it; entry 0 = 1)."""
        n = lib.bicg_matrix_history(self.h, None, 0)
        out = np.empty(max(n, 1))
        n = lib.bicg_matrix_history(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), n)
        return out[:n]

    def shifted_solve(self, method, x_set, r, sigma, seed):
        """bicg_shifted_solve_ex: method is a key of SHIFTED_SOLVE_EX; returns (that solver's return value, stats).  x_set
        (sigma_len, n_loc) and r (n_loc) are both numpy float64 arrays, or both contiguous CUDA float64 torch tensors, which go
        through bicg_shifted_solve_dev and are updated in place (a view at any element offset works).  sigma: numpy array or
        tensor (copied to the host)."""
        st = bicg_stats()
        if isinstance(x_set, np.ndarray) and isinstance(r, np.ndarray):
            xp, rp, sigma = _shifted_args(self.blk, x_set, r, _host_sigma(sigma))
            fn = lib.bicg_shifted_solve_ex
        else:
            sigma = _host_sigma(sigma)
            n = self.blk.n_loc
            xp, rp = _cuda_vectors(("x_set", x_set, (sigma.size, n)), ("r", r, (n,)))
            fn = lib.bicg_shifted_solve_dev
        k = fn(self.h, SHIFTED_SOLVE_EX[method], xp, rp, _dptr(sigma), int(sigma.size), int(seed), C.byref(st))
        return k, _stats_dict(st)

    def shifted_solve_async(self, method, x_set, r, sigma, seed, result=None, stop_iter=None, stream=None):
        """bicg_shifted_solve_async: the solve of shifted_solve on CUDA tensors, enqueued on `stream` (default: torch's current
        stream) without waiting for it.  x_set (sigma_len, n_loc; a view at any element offset works), r (n_loc,) and sigma
        (sigma_len,) are contiguous CUDA float64 tensors, read and written in stream order.  `result`: a 32-byte uint8 CUDA tensor
        that receives the bicg_shift_result (decode_shift_result reads it), allocated when not given; `stop_iter`: an optional
        int32 CUDA tensor of sigma_len that receives what last_shift_info reports for the same solve.  Works inside
        torch.cuda.graph once prepare_shifted_async(method, sigma_len) has been called.  Returns the result tensor."""
        import torch
        n = self.blk.n_loc
        if not isinstance(sigma, torch.Tensor):
            raise TypeError(f"sigma: need a CUDA float64 tensor, got {type(sigma).__name__}")
        if sigma.dim() != 1:
            raise ValueError(f"sigma: need a 1-d tensor, got shape {tuple(sigma.shape)}")
        L = int(sigma.numel())
        if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < L:
            raise ValueError(f"seed: need an integer in [0, {L}), got {seed!r}")
        xp, rp, sp_ = _checked_cuda_vectors(("x_set", x_set, (L, n)), ("r", r, (n,)), ("sigma", sigma, (L,)))
        if stop_iter is not None and not (isinstance(stop_iter, torch.Tensor) and stop_iter.is_cuda and stop_iter.dtype == torch.int32
                                          and stop_iter.is_contiguous() and tuple(stop_iter.shape) == (L,)
                                          and stop_iter.device == x_set.device):
            raise ValueError(f"stop_iter: need a contiguous int32 CUDA tensor of shape ({L},) on {x_set.device}")
        if stream is None:
            stream = torch.cuda.current_stream(x_set.device)
        result = _result_tensor(result, C.sizeof(bicg_shift_result), x_set.device, stream)
        if stop_iter is not None:
            stop_iter.record_stream(stream)
        rc = lib.bicg_shifted_solve_async(self.h, SHIFTED_SOLVE_EX[method], xp, rp, sp_, L, int(seed), C.c_void_p(stream.cuda_stream),
                                          C.c_void_p(result.data_ptr()),
                                          C.c_void_p(stop_iter.data_ptr()) if stop_iter is not None else None)
        if rc == -2:
            raise RuntimeError(f"shifted_solve_async inside a stream capture needs prepare_shifted_async({method!r}, {L}) first")
        if rc != 0:
            raise ValueError(f"bicg_shifted_solve_async failed with {rc}")
        return result

    def prepare_shifted_async(self, method, sigma_len):
        """bicg_shifted_solve_async_prepare: build what shifted_solve_async needs for `method` and sigma_len under the current
        options, outside any capture.  Collective over the ranks."""
        if lib.bicg_shifted_solve_async_prepare(self.h, SHIFTED_SOLVE_EX[method], int(sigma_len)) != 0:
            raise ValueError(f"bicg_shifted_solve_async_prepare({method}, {sigma_len}) failed")

    def shift_history(self):
        """bicg_matrix_shift_history: the seed history of the last asynchronous shifted solve on this handle (waits for it), the
        entries last_history returns after the synchronous solve; empty if there was none."""
        n = lib.bicg_matrix_shift_history(self.h, None, 0)
        out = np.empty(max(n, 1))
        n = lib.bicg_matrix_shift_history(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), n)
        return out[:n]

    def shift_residuals(self, x_set, b, sigma):
        """bicg_shift_residuals: ||(A + sigma_j I) x_j - b|| / ||b|| for every row x_j of x_set (sigma_len, n_loc), computed on
        the GPU in one fused pass.  x_set and b are both numpy float64 arrays or both CUDA float64 torch tensors (read in
        place).  Collective over the ranks."""
        sigma = np.ascontiguousarray(sigma, dtype=np.float64)
        n, L = self.blk.n_loc, int(sigma.size)
        out = np.empty(max(L, 1))
        if isinstance(x_set, np.ndarray):
            assert isinstance(b, np.ndarray)
            xp, bp, dev = _vec(x_set, L * n), _vec(b, n), 0
            assert x_set.size == L * n
        else:
            import torch
            for t in (x_set, b):
                assert t.is_cuda and t.dtype == torch.float64 and t.is_contiguous(), "need contiguous CUDA float64 tensors"
            assert x_set.numel() == L * n and b.numel() >= n
            xp, bp, dev = C.c_void_p(x_set.data_ptr()), C.c_void_p(b.data_ptr()), 1
            torch.cuda.current_stream().synchronize()       # the library reads them on its own stream
        rc = lib.bicg_shift_residuals(self.h, xp, bp, _dptr(sigma), L, dev, out.ctypes.data_as(C.POINTER(C.c_double)))
        if rc != 0:
            raise ValueError(f"bicg_shift_residuals failed with {rc}")
        return out[:L]

    def _multiply_shape(self, x):
        """(n_loc,) or (nvec, n_loc) as x has it; a shape that is neither is then rejected by the vector checks"""
        n = self.blk.n_loc
        shape = tuple(getattr(x, "shape", ()))
        return shape if len(shape) in (1, 2) and shape[-1] == n else (n,)

    def multiply(self, x, y=None, alpha=1.0, beta=0.0, sigma=None):
        """bicg_matrix_multiply: y_j = alpha (A + sigma_j I) x_j + beta y_j for every row x_j of x, on the GPU.  x is a numpy float64
        array or a contiguous CUDA float64 tensor of shape (n_loc,) or (nvec, n_loc); y has the same kind and shape and is
        allocated when None (then beta must be 0).  sigma: None (no shift term) or nvec values (numpy or tensor, copied to the
        host).  With sigma None, alpha = 1 and beta = 0 every y_j is bit-identical to spmv(x_j).  Tensors are read after torch's
        current stream has been synchronised.  Collective over the ranks.  Returns y."""
        shape = self._multiply_shape(x)
        nvec = shape[0] if len(shape) == 2 else 1
        if y is None:
            if beta != 0.0:
                raise ValueError("y: needed when beta != 0")
            if isinstance(x, np.ndarray):
                y = np.empty(shape)
            elif hasattr(x, "new_empty"):
                y = x.new_empty(shape, dtype=x.dtype)
        args = [("x", x, shape), ("y", y, shape)]
        if isinstance(x, np.ndarray) and isinstance(y, np.ndarray):
            (xp, yp), dev = _checked_host_vectors(*args), 0
        else:
            (xp, yp), dev = _cuda_vectors(*args), 1
        sp_ = None
        if sigma is not None:
            sigma = _host_sigma(sigma)
            if sigma.shape != (nvec,):
                raise ValueError(f"sigma: shape {sigma.shape}, expected ({nvec},)")
            sp_ = _dptr(sigma)
        rc = lib.bicg_matrix_multiply(self.h, nvec, xp, yp, float(alpha), float(beta), sp_, dev)
        if rc != 0:
            raise ValueError(f"bicg_matrix_multiply failed with {rc}")
        return y

    def multiply_async(self, x, y, alpha=1.0, beta=0.0, sigma=None, stream=None):
        """bicg_matrix_multiply_async: multiply on contiguous CUDA float64 tensors only, enqueued on `stream` (default: torch's
        current stream) behind the handle's earlier work, with no host synchronisation.  x and y as in multiply (y is required);
        sigma: None or a CUDA float64 tensor of shape (nvec,).  All are read and written in stream order, so a replay of a
        captured multiply reads them as they are then; works inside torch.cuda.graph with no prepare step.  Returns y."""
        import torch
        for name, t in (("x", x), ("y", y)) + ((("sigma", sigma),) if sigma is not None else ()):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{name}: multiply_async takes CUDA tensors only, got {type(t).__name__}")
        shape = self._multiply_shape(x)
        nvec = shape[0] if len(shape) == 2 else 1
        args = [("x", x, shape), ("y", y, shape)] + ([("sigma", sigma, (nvec,))] if sigma is not None else [])
        ptrs = _checked_cuda_vectors(*args)
        if stream is None:
            stream = torch.cuda.current_stream(x.device)
        rc = lib.bicg_matrix_multiply_async(self.h, nvec, ptrs[0], ptrs[1], float(alpha), float(beta),
                                            ptrs[2] if sigma is not None else None, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_multiply_async failed with {rc}")
        return y

    def _entry_args(self, name, diag, offd):
        """(name, tensor, expected shape) of an entry vector of this handle in its block order: diag.nz entries, then offd.nz
        entries where the handle has offd entries (offd may be None where it has none)"""
        import torch
        for n_, t in ((name + "_diag", diag), (name + "_offd", offd)):
            if t is not None and not isinstance(t, torch.Tensor):
                raise TypeError(f"{n_}: need a CUDA float64 tensor, got {type(t).__name__}")
        args = [(name + "_diag", diag, (int(self.blk.diag.nz),))]
        if offd is not None:
            args.append((name + "_offd", offd, (int(self.blk.offd.nz),)))
        elif self._has_offd():
            raise ValueError(f"{name}_offd: the offd block has {int(self.blk.offd.nz)} entries, got None")
        return args

    def multiply_values_async(self, w_diag, w_offd, x, y=None, alpha=1.0, beta=0.0, stream=None):
        """bicg_matrix_multiply_values_async: y_j = alpha A_W x_j + beta y_j for every row x_j of x, where A_W is this handle's
        pattern holding the weights W = (w_diag, w_offd) in set_values' block order instead of its values; bit-identical to
        multiply_async on a handle whose values were set to W.  Contiguous CUDA float64 tensors only: x of shape (n_loc,) or
        (nvec, n_loc), y the same (allocated when None; then beta must be 0).  Enqueued on `stream` (default: torch's current
        stream) behind the handle's earlier work with no host synchronisation.  Inside torch.cuda.graph, call
        prepare_multiply_values_async first.  Collective over the ranks.  Returns y."""
        import torch
        for name, t in (("x", x), ("y", y)):
            if t is not None and not isinstance(t, torch.Tensor):
                raise TypeError(f"{name}: multiply_values_async takes CUDA tensors only, got {type(t).__name__}")
        shape = self._multiply_shape(x)
        nvec = shape[0] if len(shape) == 2 else 1
        allocated = y is None
        if allocated:
            if beta != 0.0:
                raise ValueError("y: needed when beta != 0")
            y = x.new_empty(shape, dtype=torch.float64)
        wargs = self._entry_args("w", w_diag, w_offd)
        ptrs = _checked_cuda_vectors(("x", x, shape), ("y", y, shape), *wargs)
        if stream is None:
            stream = torch.cuda.current_stream(x.device)
        if allocated and stream != torch.cuda.current_stream(x.device):
            y.record_stream(stream)               # written on `stream`, not on the one it was allocated on
        rc = lib.bicg_matrix_multiply_values_async(self.h, nvec, ptrs[2], ptrs[3] if len(ptrs) > 3 else None, ptrs[0], ptrs[1],
                                                   float(alpha), float(beta), C.c_void_p(stream.cuda_stream))
        if rc == -2:
            raise RuntimeError("multiply_values_async inside a stream capture needs prepare_multiply_values_async() first")
        if rc != 0:
            raise ValueError(f"bicg_matrix_multiply_values_async failed with {rc}")
        return y

    def prepare_multiply_values_async(self):
        """bicg_matrix_multiply_values_async_prepare: allocate the buffer multiply_values_async stages weights into where it
        cannot read them in place (a handle with offd entries, or on the TMA tile plan), outside any capture; afterwards
        multiply_values_async works inside torch.cuda.graph with any weights."""
        if lib.bicg_matrix_multiply_values_async_prepare(self.h) != 0:
            raise ValueError("bicg_matrix_multiply_values_async_prepare failed")

    def transpose_entries_async(self, src, in_diag, in_offd=None, reverse=False, out=None, stream=None):
        """bicg_matrix_transpose_entries_async, with this handle the transpose of the DeviceMatrix src: reverse=False maps an
        entry vector (in_diag, in_offd) in src's block order to this handle's, exactly as transpose_values maps src's values;
        reverse=True maps one in this handle's order back to src's.  Pure copies: reverse after forward gives back every bit.
        out: (out_diag, out_offd) to write, allocated when None (out_offd None where the output side has no offd entries).
        Contiguous CUDA float64 tensors only, enqueued on `stream` (default: torch's current stream) behind both handles'
        earlier work with no host synchronisation; works inside torch.cuda.graph with no prepare step.  Collective over the
        ranks.  Returns (out_diag, out_offd)."""
        import torch
        if not isinstance(src, DeviceMatrix):
            raise TypeError(f"src: need a DeviceMatrix, got {type(src).__name__}")
        a, b = (self, src) if reverse else (src, self)
        iargs = a._entry_args("in", in_diag, in_offd)
        allocated = out is None
        if allocated:
            if not isinstance(in_diag, torch.Tensor):
                raise TypeError(f"in_diag: need a CUDA float64 tensor, got {type(in_diag).__name__}")
            out = (in_diag.new_empty((int(b.blk.diag.nz),)),
                   in_diag.new_empty((int(b.blk.offd.nz),)) if b._has_offd() else None)
        if not (isinstance(out, (tuple, list)) and len(out) == 2):
            raise TypeError("out: need a pair (out_diag, out_offd)")
        oargs = b._entry_args("out", out[0], out[1])
        ptrs = _checked_cuda_vectors(*iargs, *oargs)
        ip, op_ = ptrs[:len(iargs)], ptrs[len(iargs):]
        if stream is None:
            stream = torch.cuda.current_stream(in_diag.device)
        if allocated and stream != torch.cuda.current_stream(in_diag.device):
            for t in out:
                if t is not None:
                    t.record_stream(stream)       # written on `stream`, not on the one it was allocated on
        rc = lib.bicg_matrix_transpose_entries_async(self.h, src.h, 1 if reverse else 0, ip[0], ip[1] if len(ip) > 1 else None,
                                                     op_[0], op_[1] if len(op_) > 1 else None, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_transpose_entries_async failed with {rc} (src is not the matrix this one was "
                             f"transposed from, or out overlaps the input)")
        return out[0], (out[1] if len(op_) > 1 else None)

    def _has_offd(self):
        """whether the handle holds offd entries (with one rank the offd block is ignored)"""
        return int(self.blk.offd.nz) > 0 and lib.bicg_comm_world() > 1

    def _grad_outputs(self, u, beta, diag_out, offd_out):
        """(name, array, expected shape) of value_grad's outputs: diag_out, and offd_out where the handle has offd entries or
        one is given; allocated like u when None (then beta must be 0)"""
        outs = [("diag_out", diag_out, (int(self.blk.diag.nz),))]
        if offd_out is not None or self._has_offd():
            outs.append(("offd_out", offd_out, (int(self.blk.offd.nz),)))
        for k, (name, a, shape) in enumerate(outs):
            if a is None:
                if beta != 0.0:
                    raise ValueError(f"{name}: needed when beta != 0")
                if isinstance(u, np.ndarray):
                    a = np.empty(shape)
                elif hasattr(u, "new_empty"):
                    a = u.new_empty(shape, dtype=u.dtype)
                outs[k] = (name, a, shape)
        return outs

    def value_grad(self, u, v, alpha=1.0, beta=0.0, diag_out=None, offd_out=None):
        """bicg_matrix_value_grad: for every stored entry e = (i, c) of this rank's rows, out_e = alpha sum_j u_j[i] v_j[c]
        (+ beta out_e), in the block order set_values takes, so set_values(diag - eta g_diag, offd - eta g_offd) is a gradient
        step (a transpose's own order for a transpose).  u and v are numpy float64 arrays or contiguous CUDA float64 tensors of
        shape (n_loc,) or (nvec, n_loc); the outputs have the same kind, diag.nz and offd.nz elements, and are allocated when None
        (then beta must be 0).  With u = lambda = A^-T dL/dx, v = x and alpha = -1 this is dL/dA of a solve; with u = dL/dy,
        v = x and alpha = 1 the one of y = A x.  Tensors are read after torch's current stream has been synchronised.
        Collective over the ranks.  Returns (diag_out, offd_out); offd_out is None where the handle has no offd entries."""
        shape = self._multiply_shape(u)
        nvec = shape[0] if len(shape) == 2 else 1
        outs = self._grad_outputs(u, beta, diag_out, offd_out)
        args = [("u", u, shape), ("v", v, shape)] + outs
        if all(isinstance(a, np.ndarray) for _, a, _ in args):
            ptrs, dev = _checked_host_vectors(*args), 0
        else:
            ptrs, dev = _cuda_vectors(*args), 1
        rc = lib.bicg_matrix_value_grad(self.h, nvec, ptrs[0], ptrs[1], float(alpha), float(beta), ptrs[2],
                                        ptrs[3] if len(ptrs) > 3 else None, dev)
        if rc != 0:
            raise ValueError(f"bicg_matrix_value_grad failed with {rc}")
        return outs[0][1], (outs[1][1] if len(outs) > 1 else None)

    def value_grad_async(self, u, v, alpha=1.0, beta=0.0, diag_out=None, offd_out=None, stream=None):
        """bicg_matrix_value_grad_async: value_grad on contiguous CUDA float64 tensors only, enqueued on `stream` (default:
        torch's current stream) behind the handle's earlier work, with no host synchronisation.  All are read and written in
        stream order, so a replay of a captured call reads them as they are then; works inside torch.cuda.graph with no prepare
        step.  Returns (diag_out, offd_out) as value_grad does."""
        import torch
        for name, t in (("u", u), ("v", v), ("diag_out", diag_out), ("offd_out", offd_out)):
            if t is not None and not isinstance(t, torch.Tensor):
                raise TypeError(f"{name}: value_grad_async takes CUDA tensors only, got {type(t).__name__}")
        shape = self._multiply_shape(u)
        nvec = shape[0] if len(shape) == 2 else 1
        outs = self._grad_outputs(u, beta, diag_out, offd_out)
        ptrs = _checked_cuda_vectors(("u", u, shape), ("v", v, shape), *outs)
        if stream is None:
            stream = torch.cuda.current_stream(u.device)
        if stream != torch.cuda.current_stream(u.device):
            for (name, t, _), given in zip(outs, (diag_out, offd_out)):
                if given is None:
                    t.record_stream(stream)       # written on `stream`, not on the one it was allocated on
        rc = lib.bicg_matrix_value_grad_async(self.h, nvec, ptrs[0], ptrs[1], float(alpha), float(beta), ptrs[2],
                                              ptrs[3] if len(ptrs) > 3 else None, C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise ValueError(f"bicg_matrix_value_grad_async failed with {rc}")
        return outs[0][1], (outs[1][1] if len(outs) > 1 else None)

    def prepare_autograd(self, method):
        """What solve_autograd and multiply_autograd on this handle need inside torch.cuda.graph: creates and keeps this
        handle's transpose (transpose(): host work, collective over the ranks) and runs prepare_async(method) on both handles.
        Call it outside any capture.  destroy() destroys the transpose too."""
        t = self._adjoint()
        self.prepare_async(method)
        t.prepare_async(method)
        self.prepare_multiply_values_async()
        t.prepare_multiply_values_async()

    def prepare_shifted_autograd(self, method, sigma_len, adjoint_method="bicgstab"):
        """What shifted_solve_autograd on this handle needs inside torch.cuda.graph: creates and keeps the transpose as
        prepare_autograd does, runs prepare_shifted_async(method, sigma_len) here and prepare_async(adjoint_method) on the
        transpose, and finds the transpose's diagonal positions for shift_diagonal_async.  Call it outside any capture.
        Collective over the ranks; raises ValueError on every rank when a row of A^T on any rank has no diagonal entry."""
        t = self._adjoint()
        self.prepare_shifted_async(method, sigma_len)
        t.prepare_async(adjoint_method)
        if lib.bicg_matrix_shift_diagonal_async_prepare(t.h) != 0:
            raise ValueError("prepare_shifted_autograd: a row of A^T has no diagonal entry (a column of A without one, on this or "
                             "another rank), so A^T + sigma I cannot be formed by shifting stored entries")
        # a second backward solves with A + sigma_j I here; a matrix without a stored diagonal entry in every row is refused
        # then, when that shift is asked for, so first-order use of such a matrix still works
        self.prepare_async(adjoint_method)
        lib.bicg_matrix_shift_diagonal_async_prepare(self.h)
        self.prepare_multiply_values_async()
        t.prepare_multiply_values_async()

    def _adjoint(self):
        """The transpose the backward of a differentiable solve or multiply runs on: the one prepare_autograd made, else created
        here, which a stream capture cannot hold.  For a transpose made here, its source: (A^T)^T is never created."""
        if self._src is not None:
            return self._src
        if self._t is None:
            import torch
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("a backward through this DeviceMatrix inside a CUDA graph capture needs "
                                   "dm.prepare_autograd(method) before the capture: creating the transpose is host work")
            self._t = self.transpose()
            self._t._src = self
        return self._t

    def spmv(self, x_loc):
        y = np.empty(self.blk.n_loc)
        lib.bicg_spmv(self.h, _vec(x_loc, self.blk.n_loc), _dptr(y))
        return y

    def resident_ctas(self):
        """CTAs of the last persistent-kernel launch that kept their matrix slice in shared memory (BICG_RESIDENT)."""
        return int(lib.bicg_debug_resident_ctas(self.h))

    def coded_ctas(self):
        """CTAs of the last persistent-kernel launch that streamed 16-bit column codes instead of 32-bit columns."""
        return int(lib.bicg_debug_coded_ctas(self.h))

    def stream_codes(self, on):
        """Test hook: on=False makes later persistent-kernel launches on this handle stream 32-bit columns everywhere
        (the results are bit-identical); returns the previous setting."""
        return bool(lib.bicg_debug_stream_codes(self.h, 1 if on else 0))

    def packed_ctas(self):
        """CTAs of the last persistent-kernel launch that streamed 7-byte packed values instead of 8-byte values."""
        return int(lib.bicg_debug_packed_ctas(self.h))

    def stream_values(self, on):
        """Test hook: on=False makes later persistent-kernel launches on this handle stream 8-byte values everywhere while
        keeping the column codes (the results are bit-identical); returns the previous setting."""
        return bool(lib.bicg_debug_stream_values(self.h, 1 if on else 0))

    def spmv_time(self, reps=20):
        ms, by = C.c_double(), C.c_double()
        lib.bicg_spmv_time(self.h, reps, C.byref(ms), C.byref(by))
        return ms.value, by.value

    def profile(self, method, iters, krr=0, nrr=0):
        ms = (C.c_double * 3)()
        cnt = (C.c_int * 3)()
        rc = lib.bicg_profile_solve(self.h, METHODS[method], iters, int(krr), int(nrr), ms, cnt)
        if rc != 0:
            raise RuntimeError("bicg_profile_solve failed")
        return list(ms), list(cnt)

    def destroy(self):
        if self._t is not None:
            self._t.destroy()
            self._t = None
        self._src = None
        if self.h:
            lib.bicg_matrix_destroy(self.h)
            self.h = None


_CALLBACK_KEEPALIVE = []


def comm_init(rank, world, allgather_bytes):
    """Register this process as `rank` of `world`.  allgather_bytes(b: bytes) -> list[bytes] (one per rank)."""

    def _cb(_ctx, send, recv, nbytes):
        try:
            mine = C.string_at(send, nbytes)
            parts = allgather_bytes(mine)
            C.memmove(recv, b"".join(parts), nbytes * world)
            return 0
        except Exception as exc:                      # never let an exception unwind through C
            print(f"bicg allgather callback failed: {exc!r}", flush=True)
            return 1

    cb = ALLGATHER_FN(_cb)
    _CALLBACK_KEEPALIVE.append(cb)
    rc = lib.bicg_comm_init(rank, world, cb, None)
    if rc != 0:
        raise ValueError(f"bicg_comm_init({rank}, {world}) failed")


def comm_init_torch(group=None):
    """Bootstrap from an initialised torch.distributed job (one process per GPU, as torchrun starts them).
    Only the bootstrap bytes (IPC handles, halo plans) travel through torch; solver traffic is peer memory."""
    import torch
    import torch.distributed as dist

    rank, world = dist.get_rank(group), dist.get_world_size(group)
    backend = dist.get_backend(group)
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")

    def allgather_bytes(b):
        t = torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        outs = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(outs, t, group=group)
        return [o.cpu().numpy().tobytes() for o in outs]

    comm_init(rank, world, allgather_bytes)
    return rank, world


def comm_finalize():
    lib.bicg_comm_finalize()
