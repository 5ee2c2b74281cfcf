// spmv.cuh -- argument block + launch interface of the CSR SpMV kernels (spmv.cu)
#pragma once
#include "dev.cuh"

namespace bicg {

// dots fused into the SpMV epilogue: dot[k] += U[row] * V[row] where U, V are either one of up to four
// epilogue vectors (index into vec[]) or the y just computed (index -1)
struct EpiArgs {
    int nvec;
    const double *vec[4];
    int ndot;
    int ia[4], ib[4];
};

// One argument block for both epilogues of the SpMV kernels (spmv.cu).  The solver's SpMV: y[0] = A x[0] (+ sigma[0] x[0]),
// with the dots of `epi` fused and reduced in the tail.  The batched multiply of bicg_matrix_multiply (multiply.cu):
// y_v = alpha (A + sigma_v I) x_v + beta y_v, v < nv, one pass over the matrix for nv vectors.  Both run the same plan,
// tiles and row loop, so every row sum is bit-identical between them.
constexpr int MUL_NV_MAX = 8;        // vectors one launch can take (the largest instantiated NV)
struct SpmvArgs {
    KernelCommon kc;
    // device CSR of this rank's rows over the extended local column space [own columns | ghost columns]
    // (diag block entries first, then offd entries, matrix.c:437-440 order).  val/col are padded by >= 8
    // entries so 16-byte aligned over-reads of a tile stay in bounds.
    const double   *val;
    const unsigned *col;
    const unsigned *ptr;
    int rows;
    // tile plan of the TMA kernel
    const int      *tile_row;   // ntiles + 1
    const unsigned *tile_nz;    // ntiles + 1 : ptr[tile_row[t]]
    int ntiles;
    int cap;                    // stage capacity in entries (multiple of 32)
    int stages;                 // 2..4
    int nv;                          // vectors of this launch, 1 .. MUL_NV_MAX (the solver's SpMV: 1)
    const double *x[MUL_NV_MAX];     // x_v over the extended column space; slots v >= nv repeat x[nv - 1] and are not written
    double       *y[MUL_NV_MAX];     // y_v, own rows
    const double *sigma;             // nv device values, or null: no shift term (shifted systems, shifted_switching_solver.c:386, 404)
    double alpha, beta;              // multiply epilogue; beta == 0: y is not read
    EpiArgs epi;                     // solver epilogue
    int wait_halo;                   // 1: x's ghost part is filled by peers; wait for their halo flags first
};

// epilogue slices of the solver's stages (dev.cuh: StageLayout); the multiply's stages have none
constexpr int SPMV_EPI_SLICES = 4;

// kind 0: warp-specialised TMA tile kernel, kind 1: row-split kernel.  threads (consumer threads) only matters for kind 0.
// solver: the solver's epilogue (a.nv == 1), else the multiply's for a.nv vectors.  Returns cudaError_t as int.
int launch_spmv(int kind, int lanes, int threads, int grid, size_t smem_bytes, bool solver, const SpmvArgs &a, cudaStream_t st);
// one-time opt-in to > 48 KB dynamic shared memory for every instantiation
int spmv_setup_attributes();
// add a dot term (a . b) to an epilogue; null pointer = the y just computed
void epi_add_dot(EpiArgs &e, const double *a, const double *b);

} // namespace bicg
