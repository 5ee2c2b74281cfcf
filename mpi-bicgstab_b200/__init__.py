"""mpi-bicgstab_b200 -- H100-native (sm_90a) drop-in for the BiCGStab hot path of RtrMmmt/MPI-BiCGStab.

The product is `libbicgstab_b200.so` (csrc/, C ABI in include/bicgstab_b200.h).  This package is the thin
host-side mirror of the reference's interface used by the tests and bench.py.  The directory name carries a
hyphen, so import it as `import mpi_bicgstab_b200` (alias module at the repo root) or
`importlib.import_module("mpi-bicgstab_b200")`.
"""
from . import _lib                                   # noqa: F401  (fails loudly if the .so is missing)
from .api import *                                   # noqa: F401,F403
from .api import (METHODS, GEN_KINDS, MatrixBlock, DeviceMatrix, blocks_from_csr, block_to_global_csr, gen_block,
                  load_matrix_block, plan_partition, spmv_ovlap, bicgstab, ca_bicgstab, pipe_bicgstab,
                  pipe_bicgstab_rr, solve, SHIFTED_METHODS, SHIFTED_SOLVE_EX, shifted_lopbicg_switching, shifted_lopbicg,
                  shifted_lopbicgstab, shifted_pipe_lopbicgstab, last_shift_info, last_shift_error, set_option, set_options, last_history, last_stats, comm_init,
                  comm_init_torch, comm_finalize)
from ._lib import lib, CSR_Matrix, INFO_Matrix, bicg_stats, SYMBOLS, LIB_PATH

# the differentiable entry points need torch, which importing the package does not: autograd.py is loaded on first use
_AUTOGRAD = ("solve_autograd", "multiply_autograd", "shifted_solve_autograd", "SolveFunction", "MultiplyFunction",
             "ShiftedSolveFunction")


def __getattr__(name):
    if name in _AUTOGRAD:
        from . import autograd
        return getattr(autograd, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
