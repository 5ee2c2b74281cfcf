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
    const double *x;            // input vector, extended layout
    double       *y;            // output, own rows
    EpiArgs epi;
    int wait_halo;              // 1: x's ghost part is filled by peers; wait for their halo flags first
    const double *shift_sigma;  // not null: y = A x + (*shift_sigma) x  (shifted systems, shifted_switching_solver.c:386, 404)
};

// The batched multiply y_v = alpha (A + sigma_v I) x_v + beta y_v, v < nv, of bicg_matrix_multiply (multiply.cu): one pass
// over the matrix serves nv vectors.  Same plan, tiles and lanes as the SpMV above, so every row sum is bit-identical to it.
constexpr int MUL_NV_MAX = 8;        // vectors one launch can take (the largest instantiated NV)
struct MultiplyArgs {
    KernelCommon kc;                 // tail: the closing barrier with peers, none at one rank
    const double   *val;
    const unsigned *col;
    const unsigned *ptr;
    int rows;
    const int      *tile_row;
    const unsigned *tile_nz;
    int ntiles, cap, stages;
    int nv;                          // vectors of this launch, 1 .. MUL_NV_MAX
    const double *x[MUL_NV_MAX];     // x_v over the extended column space; slots v >= nv repeat x[nv - 1] and are not written
    double       *y[MUL_NV_MAX];     // y_v, own rows
    const double *sigma;             // nv device values, or null: no shift term
    double alpha, beta;              // beta == 0: y is not read
    int wait_halo;                   // 1: the ghost part of every x_v is filled by peers; wait for their halo flags first
};
// the smallest instantiated NV that holds nv vectors (nv <= MUL_NV_MAX)
int multiply_nv(int nv);
int launch_multiply(int kind, int lanes, int threads, int grid, size_t smem_bytes, int NV, const MultiplyArgs &a, cudaStream_t st);
size_t multiply_tma_smem_bytes(int cap, int stages, int threads, int lanes);

// kind 0: warp-specialised TMA tile kernel, kind 1: row-split kernel.  threads (consumer threads) only matters for kind 0.
// Returns cudaError_t as int.
int launch_spmv(int kind, int lanes, int threads, int grid, size_t smem_bytes, const SpmvArgs &a, cudaStream_t st);
// one-time opt-in to > 48 KB dynamic shared memory for every instantiation
int spmv_setup_attributes();
size_t spmv_tma_smem_bytes(int cap, int stages, int threads, int lanes);
// add a dot term (a . b) to an epilogue; null pointer = the y just computed
void epi_add_dot(EpiArgs &e, const double *a, const double *b);

} // namespace bicg
