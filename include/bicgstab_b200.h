/*
 * bicgstab_b200.h -- C ABI of libbicgstab_b200.so, the H100-native drop-in for the BiCGStab hot
 * path of RtrMmmt/MPI-BiCGStab (SpMV + BLAS-1 + iteration loops + their collectives).
 *
 * Part 1 re-declares, with identical signatures and struct layouts, the eight non-libc, non-MPI
 * symbols the reference's main.c needs (reference file:line beside each one), so that main.c
 * compiles UNCHANGED against include/compat/mpi.h + the reference's own solver.h and links against
 * this library instead of solver.c / matrix.c / vector.c.
 * Part 2 is the small extension surface (prefix bicg_) that tests, bench.py and multi-process
 * launchers use: rank/communicator bootstrap, device-resident matrices (whose values can be
 * replaced in place, pattern kept), solve statistics, synthetic-matrix generators.  No torch / CUDA types appear anywhere in this header.
 *
 * Every entry point drives hand-written sm_90a CUDA kernels; there is no CPU fallback -- if no
 * CUDA device is usable the compute entry points print an error and exit(1) (the reference's own
 * error convention, solver.c:43-46).
 */
#ifndef BICGSTAB_B200_H
#define BICGSTAB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Part 1 -- the reference's own interface
 * ---------------------------------------------------------------------------------------------- */
#ifndef MATRIX_H /* the reference's matrix.h (include guard MATRIX_H) already defines these types */

typedef char MM_typecode[4];                 /* mmio.h:16 */

/* matrix.h:19-26 -- sizeof 40; val@0 col@8 ptr@16 nz@24 rows@28 cols@32 */
typedef struct {
    double       *val;   /* nz values                                   */
    unsigned int *col;   /* nz column indices (diag: local, offd: global) */
    unsigned int *ptr;   /* rows+1 row starts, ptr[0] == 0              */
    unsigned int  nz, rows, cols;
} CSR_Matrix;

/* matrix.h:28-33 -- sizeof 32; nz@0 rows@4 cols@8 code@12 recvcounts@16 displs@24 */
typedef struct {
    unsigned int nz, rows, cols;  /* global sizes */
    MM_typecode  code;
    int         *recvcounts;      /* rows of rank p            (matrix.c:306) */
    int         *displs;          /* first global row of rank p (matrix.c:307) */
} INFO_Matrix;

/* matrix.h:44-45 (matrix.c:188-204) */
void csr_init_matrix(CSR_Matrix *m);
void csr_free_matrix(CSR_Matrix *m);
/* matrix.h:57 (matrix.c:536-551): A_diag += sigma I in place on the caller's host arrays; drops the cached device copy */
void csr_shift_diagonal(CSR_Matrix *A_diag, double sigma);

/* matrix.h:50 (matrix.c:402-419): Matrix-Market file -> this rank's diag / offd CSR blocks + partition */
void MPI_csr_load_matrix_block(char *filename, CSR_Matrix *matrix_loc_diag, CSR_Matrix *matrix_loc_offd,
                               INFO_Matrix *matrix_info);

/* matrix.h:51 (matrix.c:428-441): y_loc = A_diag x_loc + A_offd x, host pointers; x (length cols) is
 * caller-owned scratch that receives the gathered vector like the reference's allgather does. */
void MPI_csr_spmv_ovlap(CSR_Matrix *matrix_loc_diag, CSR_Matrix *matrix_loc_offd, INFO_Matrix *matrix_info,
                        double *x_loc, double *x, double *y_loc);

/* solver.h:10-13 (solver.c:35-146, 160-278, 292-417, 433-576).  Host pointers.  x_loc: initial guess in,
 * solution out.  r_loc: right-hand side in, final recursive residual out (b is destroyed, as in the
 * reference).  Return value: iterations performed.  Collective over all ranks of the job. */
int bicgstab(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc, double *r_loc);
int ca_bicgstab(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc, double *r_loc);
int pipe_bicgstab(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc, double *r_loc);
int pipe_bicgstab_rr(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc,
                     double *r_loc, int krr, int nrr);

#endif /* MATRIX_H */

/* shifted_switching_solver.h:12 (shifted_switching_solver.c:260-602): seed-switching shifted BiCGStab for (A + sigma_j I) x_j = b.
 * x_loc_set: sigma_len blocks of n_loc doubles (initial guesses in, solutions out); r_loc: b in, seed residual out; returns the
 * reference's k (iterations performed + 1).  EPS / MAX_ITER of the reference (1e-12 / 1000, :5-6) = BICG_SHIFT_TOL /
 * BICG_SHIFT_MAX_ITER.  Not needed by main.c; it is what main_shifted.c / main_repeat.c call (SURVEY.md 8(f) N4). */
int shifted_lopbicg_switching(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set,
                              double *r_loc, double *sigma, int sigma_len, int seed);
/* shifted_switching_solver.h:13 (shifted_switching_solver.c:611): the same solve without communication overlap in the reference --
 * identical arithmetic, so the same function here. */
int shifted_lopbicg_switching_noovlp(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set,
                                     double *r_loc, double *sigma, int sigma_len, int seed);
/* shifted_switching_solver.h:11 (shifted_switching_solver.c:20-257): the fixed-seed variant the shifted drivers name as the
 * alternative to the switching call (main_shifted.c:125, main_repeat.c:129, main_seed_diff.c:133).  Same arguments; until the seed
 * converges it is the switching solve line for line.  The seed never switches: when it converges first it is counted as stopped
 * but keeps iterating, since the other shifts still advance from its Krylov data, until every shift has stopped or MAX_ITER.
 * Returns k, the iterations performed (not k + 1), and prints only the `Total time` / `Avg time/iter` lines (:241-242). */
int shifted_lopbicg(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc,
                    double *sigma, int sigma_len, int seed);

/* shifted_solver.h:17-21 (shifted_solver.c:182-1085): the LOP shifted BiCGStab family for (A + sigma_j I) x_j = b.  Same arguments as
 * shifted_lopbicg_switching, but the seed never changes and every shift is advanced until max_j |1/(zeta_j pi_j)|^2 (r,r) <=
 * EPS^2 (b,b) or MAX_ITER; returns k, the iterations performed (not k + 1).  EPS / MAX_ITER: BICG_SHIFT_TOL / BICG_SHIFT_MAX_ITER.
 * shifted_lopbicgstab_v2 and _nooverlap only move the reference's per-shift updates and MPI waits; their arithmetic is that of
 * shifted_lopbicgstab, so all three are the same solve here (LOP).  shifted_pipe_lopbicgstab_nooverlap is likewise the same solve as
 * shifted_pipe_lopbicgstab (PIPE-LOP: the pipelined seed recurrences of pipe_bicgstab).  The reference's test_shifted.c calls
 * shifted_pipe_lopbicgstab_nooverlap.  shifted_bicgstab (:16) is not provided. */
int shifted_lopbicgstab(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc,
                        double *sigma, int sigma_len, int seed);
int shifted_lopbicgstab_v2(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc,
                           double *sigma, int sigma_len, int seed);
int shifted_lopbicgstab_nooverlap(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set,
                                  double *r_loc, double *sigma, int sigma_len, int seed);
int shifted_pipe_lopbicgstab(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set, double *r_loc,
                             double *sigma, int sigma_len, int seed);
int shifted_pipe_lopbicgstab_nooverlap(CSR_Matrix *A_loc_diag, CSR_Matrix *A_loc_offd, INFO_Matrix *A_info, double *x_loc_set,
                                       double *r_loc, double *sigma, int sigma_len, int seed);

/* vector.h:4-7 (vector.c:3-27) on HOST arrays: the shifted drivers build and copy their right-hand sides with these
 * (main_shifted.c:114-135, main_repeat.c:121, main_seed_diff.c:118-121), so they are exported for those programs to link
 * unchanged (csrc/hostvec.cpp).  The solvers do not use them: their vector work is fused into the device kernels. */
void    my_daxpy(int n, double alpha, const double *x, double *y);
double  my_ddot(int n, const double *x, const double *y);
void    my_dscal(int n, double alpha, double *x);
void    my_dcopy(int n, const double *x, double *y);

/* ------------------------------------------------------------------------------------------------
 * Part 2 -- extensions
 * ---------------------------------------------------------------------------------------------- */

#define BICG_ABI_VERSION 1
int bicg_abi_version(void);

/* Runtime options.  The reference fixes these with #defines (solver.c:3-9) and its signatures carry no
 * options, so they come from the environment (read once, on first use) or from bicg_set_option():
 *   BICG_TOL       (1e-15, solver.c:3)   BICG_MAX_ITER (1000, solver.c:4)   BICG_OUT_ITER (100, solver.c:9)
 *   BICG_QUIET=1   suppress the solver.c:124,135-139 stdout lines
 *   BICG_SPMV      auto | tma | rowsplit        BICG_SPMV_LANES  lanes per row (1,2,4,...,32; 0 = choose)
 *   BICG_UNROLL    iterations per body of the kernel-per-phase loop's CUDA-graph WHILE node (default 10)
 *   BICG_CACHE     1 keep uploaded matrices keyed by host pointer (default) | 0 re-upload on every call
 *   BICG_DEVICE    CUDA device ordinal (default: LOCAL_RANK if set, else 0)
 *   BICG_MEGA      1 persistent solver kernel where it wins (thread-per-row plans; default) | 2 always | 0 kernel-per-phase graph
 *   BICG_RESIDENT  1 persistent kernel keeps a CTA's matrix slice in shared memory for the whole solve when it fits (default) | 0
 *   BICG_PARTITION rows (matrix.c:295-308, default) | nnz (archive/matrix.c:407-420) in the loader and the generators
 *   BICG_PEER_TIMEOUT_S  bound of every device-side wait for another CTA / GPU (default 20)
 *   BICG_SHIFT_TOL (1e-12) / BICG_SHIFT_MAX_ITER (1000) / BICG_SHIFT_ERROR (0): the shifted solvers, see below
 *   tuning / experiments: BICG_MEGA_THREADS, BICG_MEGA_LANES, BICG_ROW_WEIGHT, BICG_BOUNDARY_WEIGHT, BICG_AUTOTUNE,
 *   BICG_SPMV_THREADS / _STAGES / _CTAS, BICG_HALO_GAP, BICG_VERBOSE,
 *   BICG_MEGA_TRACE (per-phase device timestamps of the persistent kernel on stderr)
 * Returns 0 on success, -1 for an unknown key. */
int bicg_set_option(const char *key, const char *value);

/* Multi-process bootstrap (one process = one rank = one GPU, like one MPI rank in the reference).
 * `allgather` must copy `bytes` bytes from every rank's `send` into `recv` (rank-major) and return 0;
 * the launcher supplies it (bench.py: torch.distributed; include/compat/mpi.h shim: POSIX shm).
 * Without this call the process is a single rank (world = 1). */
typedef int (*bicg_allgather_fn)(void *ctx, const void *send, void *recv, size_t bytes);
int  bicg_comm_init(int rank, int world, bicg_allgather_fn allgather, void *ctx);
void bicg_comm_finalize(void);
int  bicg_comm_rank(void);
int  bicg_comm_world(void);

/* Device-resident matrix (upload + SpMV tiling plan + halo plan); the host-pointer entry points of
 * Part 1 create and cache one of these internally. */
typedef struct bicg_matrix bicg_matrix;
bicg_matrix *bicg_matrix_create(const CSR_Matrix *diag, const CSR_Matrix *offd, const INFO_Matrix *info);
void         bicg_matrix_destroy(bicg_matrix *m);
/* drop the cached upload of a host matrix whose values were changed in place (csr_shift_diagonal,
 * matrix.c:536-551, does that) */
void         bicg_matrix_invalidate(const CSR_Matrix *diag);

/* New values on a resident matrix, same pattern: for a sequence of systems that share one sparsity pattern (implicit time
 * steps, Newton-Krylov, continuation, a diagonal shift).  The halo plan, the merged layout, the arena, the SpMV and
 * persistent-kernel plans and the column codes are kept; the merged values are rewritten and the persistent kernel's per-CTA
 * value tables and packed values rebuilt by the pass bicg_matrix_create runs, so every result on the handle afterwards is
 * bit-identical to that of a handle freshly created from blocks holding the same values.  Pointers on the handle do not
 * change: a captured solve keeps working and reads the new values when it is replayed.
 *
 * Values: diag_val holds diag.nz doubles and offd_val offd.nz doubles, in the order of the CSR_Matrix blocks the handle was
 * created from (their ptr and col are the creation's by contract and are not passed again).  diag_val must not be null;
 * offd_val may be null only when the handle has no offd entries (always with one rank, where the offd block is ignored).
 * Returns 0, or -1 for a null handle or diag_val (checked before the device is touched) or a null offd_val on a handle with
 * offd entries.
 *
 * Rank-local: neither call communicates, so neither is collective.  Each rank sets the values of its own rows; the next solve
 * is collective as before and multiplies with whatever values every rank has set.  No bootstrap exchange runs again, which is
 * what makes an update cheap on several GPUs.
 *
 * bicg_matrix_set_values: host pointers, or device pointers when device_vectors != 0.  Waits for the handle's earlier
 * asynchronous work and returns once the new values are in place.
 * bicg_matrix_set_values_async: device pointers only, enqueued on the caller's CUDA stream `stream` behind the handle's
 * previous work, with the ordering of bicg_solve_async: no host synchronisation, allocation or pageable copy, and the values
 * are read in stream order, so a replay of a captured update reads the buffers as they are at that point.  It needs no prepare
 * step and works inside a stream capture as it is (there is no -2).
 *
 * bicg_matrix_shift_diagonal: A_diag += sigma I on the handle, like csr_shift_diagonal (matrix.c:536-551) on the host arrays:
 * sigma is added to the first entry of every own row whose column is that row; repeated calls accumulate.  Synchronous and
 * rank-local.  Returns 0, or -1 for a null handle or when a row of this rank has no diagonal entry (the reference exits
 * there), and then no value has changed.
 *
 * bicg_matrix_shift_diagonal_async: the same shift by *sigma, one double in DEVICE memory read in stream order, enqueued on the
 * caller's CUDA stream `stream` with the ordering of bicg_matrix_set_values_async (no host synchronisation, allocation or
 * pageable copy), so a replay of a captured shift adds the value the buffer holds then; the persistent kernel's value tables
 * are rebuilt as by every value update, and the result is bit-identical to bicg_matrix_shift_diagonal by that value.
 * Rank-local.  Returns 0; -1 for a null m or sigma (checked before the device is touched), or when a row of this rank, or of
 * any rank at the last prepare, has no diagonal entry (then no value has changed); -2 inside a stream capture when
 * bicg_matrix_shift_diagonal_async_prepare has not run on the handle (the capture stays valid).
 * bicg_matrix_shift_diagonal_async_prepare finds the diagonal positions (once per handle; it may synchronise) outside any
 * capture; an uncaptured shift calls it itself at the handle's first asynchronous shift.  Collective: every rank returns -1
 * if any rank passed a null handle or has a row without a diagonal entry, so a refusal leaves no rank waiting in collective
 * work that would follow the shift (a transpose refresh, a solve); else 0. */
int bicg_matrix_set_values(bicg_matrix *m, const double *diag_val, const double *offd_val, int device_vectors);
int bicg_matrix_set_values_async(bicg_matrix *m, const double *diag_val, const double *offd_val, void *stream);
int bicg_matrix_shift_diagonal(bicg_matrix *m, double sigma);
int bicg_matrix_shift_diagonal_async(bicg_matrix *m, const double *sigma, void *stream);
int bicg_matrix_shift_diagonal_async_prepare(bicg_matrix *m);

/* A^T of a resident matrix as a handle of its own: for adjoint systems A^T lambda = g (the gradient of an objective of the
 * solution of A x = b, the backward of a differentiable solve), two-sided Krylov methods and the normal equations.
 *
 * bicg_matrix_create_transpose: same global size and row partition as m (its recvcounts / displs, under BICG_PARTITION=nnz
 * too), with its own plans, arena and halo.  Pattern: row j of A^T holds the entries (i, j) of A by ascending i; entries with
 * equal (i, j) keep their order in row i of A; duplicates and explicit zeros are kept; within a row, as for any handle, diag
 * columns come first, then offd columns.  So every result on it (spmv, multiply, every solve and shifted solve, histories and
 * stats apart from timings) is bit-identical to that of bicg_matrix_create on the blocks of the global CSR of A^T built by a
 * stable sort of A's global triplets by (column, row).  Once created it is independent of m: destroying m leaves it working,
 * and bicg_matrix_set_values on it takes its own block order.  Setup work, collective over the ranks like bicg_matrix_create
 * (the entries whose column another rank owns travel through the host allgather once).  Returns null for a null m, on every
 * rank if any rank passed one.
 *
 * bicg_matrix_transpose_values: mt's values become those of bicg_matrix_create_transpose(src) for src as it is at that point,
 * where src must be the handle mt was created from; the pattern is not rebuilt, only the values are copied on the device and
 * the persistent kernel's value tables rebuilt, as bicg_matrix_set_values does.  Returns 0, or -1 for a null mt or src or an
 * src that is not mt's source (then nothing is touched).  The synchronous call waits for both handles' earlier asynchronous
 * work, checks its arguments on every rank (every rank returns -1 if any rank's are bad) and returns once done; a peer timeout
 * is fatal.  bicg_matrix_transpose_values_async runs on the caller's CUDA stream behind both handles' earlier work, and both
 * handles' next work waits for it: no host synchronisation, allocation, pageable copy or output, no prepare step (there is no
 * -2), and it works inside a stream capture, where a replay reads src's values as they are then.  It checks its arguments
 * locally; a peer timeout is reported by the next synchronous call on mt.  Both are collective: with peers, each rank first
 * stores the values other ranks' rows of A^T need into their receive regions, between two empty cross-GPU reductions.
 *
 * bicg_matrix_block_nz: the entries of the diag and offd blocks of this rank's rows of a handle (offd is 0 with one rank),
 * which bicg_matrix_set_values takes; for a transpose these are not otherwise known to the caller.  -1 for a null argument. */
bicg_matrix *bicg_matrix_create_transpose(bicg_matrix *m);
int bicg_matrix_transpose_values(bicg_matrix *mt, bicg_matrix *src);
int bicg_matrix_transpose_values_async(bicg_matrix *mt, bicg_matrix *src, void *stream);
int bicg_matrix_block_nz(const bicg_matrix *m, unsigned *diag_nz, unsigned *offd_nz);

/* Entry vectors between a handle and its transpose: the permutation bicg_matrix_transpose_values applies to the values, on any
 * vector of one double per stored entry, in both directions (what differentiating through that refresh needs).
 *
 * bicg_matrix_transpose_entries_async, reverse = 0: in (in_diag, in_offd) is in src's block order (the order
 * bicg_matrix_set_values takes on src); out (out_diag, out_offd) receives, in mt's block order, exactly the values
 * bicg_matrix_transpose_values would give mt if src held `in`, so bicg_matrix_set_values(mt, out) then leaves mt with the bits
 * of that refresh.  reverse = 1: the inverse permutation, from mt's block order back to src's.  Both directions are pure
 * copies, so reverse after forward gives back every bit of `in`, duplicates and explicit zeros included.  in_offd / out_offd
 * may be null where their handle has no offd entries (always with one rank).
 *
 * Device pointers, read and written in stream order on the caller's CUDA stream `stream` behind both handles' earlier work, and
 * both handles' next work waits for it: no host synchronisation, allocation, pageable copy or output, no prepare step (there
 * is no -2), and it works inside a stream capture.  Neither handle's values change.  Returns 0, or -1 for a null mt, src,
 * in_diag or out_diag, reverse not 0 or 1, an mt that is not a transpose of src, a null in_offd or out_offd where its handle
 * has offd entries, or an output range overlapping an input range; these are checked before the device is touched.
 * Collective like bicg_matrix_transpose_values_async: with peers, the entries whose row of the other matrix another rank owns
 * are stored into that rank's receive region (forward: mt's; reverse: a second region of the transpose's arena on the source
 * entry's rank, sized at bicg_matrix_create_transpose), between two empty cross-GPU reductions.  A peer timeout is reported
 * by the next synchronous call on mt. */
int bicg_matrix_transpose_entries_async(bicg_matrix *mt, bicg_matrix *src, int reverse, const double *in_diag,
                                        const double *in_offd, double *out_diag, double *out_offd, void *stream);

enum { BICG_METHOD_BICGSTAB = 0, BICG_METHOD_CA = 1, BICG_METHOD_PIPE = 2, BICG_METHOD_PIPE_RR = 3 };

typedef struct {
    int    iters;          /* iterations performed (the reference's return value)        */
    int    converged;      /* 1 if dot_r <= tol^2 dot_zero stopped the loop               */
    double final_res;      /* sqrt(dot_r / dot_zero)  (solver.c:136)                      */
    double loop_ms;        /* CUDA-event time of the reference's timed region a14 (solver.c:69-71,129-132):
                              initial A x0 ... end of loop, device resident                */
    double h2d_ms, d2h_ms; /* host<->device copies of x, b / x, r done by this call        */
    double upload_ms;      /* matrix upload + planning done by this call (0 when cached)   */
    uint64_t h2d_bytes, d2h_bytes;
    int    kernel_launches;/* kernels launched inside the timed region.  Kernel-per-phase loop: the init kernels plus
                              every kernel of every WHILE body that ran, including those of the last body that
                              returned at once after the loop test; far above the <= 8 of a persistent-kernel
                              solve (its init kernels and the one loop kernel)                */
    int    spmv_lanes;     /* lanes per row the SpMV plan chose                             */
    int    spmv_kind;      /* 0 = tma tile kernel, 1 = rowsplit kernel                      */
} bicg_stats;

/* Solve on a device-resident matrix.  x and r are HOST pointers unless `device_vectors` != 0, in which
 * case they are device pointers (same in/out meaning as Part 1).  krr/nrr only for BICG_METHOD_PIPE_RR. */
int bicg_solve(bicg_matrix *m, int method, double *x, double *r, int krr, int nrr, int device_vectors,
               bicg_stats *stats);

/* Written by the device at the end of an asynchronous solve, in stream order (24 bytes): the iters, converged and
 * final_res that bicg_solve reports in bicg_stats for the same solve, and error = 1 if a bounded wait for a peer GPU or
 * another CTA timed out (BICG_PEER_TIMEOUT_S). */
typedef struct {
    int    iters;
    int    converged;
    int    error;
    int    reserved;
    double final_res;
} bicg_result;

/* bicg_solve with device vectors, enqueued on the caller's CUDA stream `stream` (a cudaStream_t; 0 is CUDA's default
 * stream, not the library's).  x and r are device pointers to n_loc doubles, updated in place, with the meaning of
 * bicg_solve.  `result`, if not null, is device memory that receives the solve's bicg_result.  Returns 0 once the work is
 * enqueued, with no host synchronisation, allocation, pageable copy or output; -1 for a null x / r or an unknown method
 * (PIPE_RR with krr <= 0 runs PIPE, as in bicg_solve); -2 inside a stream capture when bicg_solve_async_prepare has not
 * been called for this handle and method under the current options (the capture stays valid).  Options (TOL, MAX_ITER,
 * MEGA, RESIDENT, UNROLL, ...) are read at enqueue time; a captured solve keeps the values it was captured with.
 * The x, r and history it computes are bit-identical to bicg_solve's.
 *
 * Ordering: every call on a handle shares its device state, so each asynchronous call waits for the handle's previous
 * asynchronous work and every synchronous entry point waits for it too.  A captured solve orders its replays the same
 * way, but a replay must not run concurrently with other work on the same handle that was not enqueued after it.
 * Not updated by asynchronous solves: bicg_last_stats, bicg_last_history and the stdout lines (BICG_MEGA_TRACE and
 * bicg_profile_solve stay synchronous).  With several ranks the call is collective like bicg_solve: every rank enqueues,
 * or replays, the same sequence on the handle.
 *
 * bicg_solve_async_prepare builds, outside any capture, what the asynchronous path needs on this handle and method: the
 * graphs of the device-side loop and a history for the current MAX_ITER.  It may synchronise and allocate; an uncaptured
 * bicg_solve_async calls it itself.  The handle's first prepare also orders every later asynchronous call on it behind the
 * work already enqueued on the library's stream (the upload of bicg_matrix_create).  Raising MAX_ITER past the handle's
 * history capacity moves its history: a solve captured before that keeps writing the old one, so prepare and capture again.
 * Returns 0, or -1 for an unknown method.
 *
 * bicg_matrix_history waits for the last work enqueued on m and copies that solve's history (dot_r/dot_zero after every
 * iteration, out[0] = 1) like bicg_last_history; returns the number of entries.  A peer timeout of that solve is fatal
 * here, as it is in bicg_solve. */
int bicg_solve_async(bicg_matrix *m, int method, double *x, double *r, int krr, int nrr, void *stream, bicg_result *result);
int bicg_solve_async_prepare(bicg_matrix *m, int method);
int bicg_matrix_history(bicg_matrix *m, double *out, int cap);

/* shifted_lopbicg_switching on a resident matrix; bicg_last_shift_info: the seed the last shifted solve ended with and the
 * iteration at which every shift stopped (returns sigma_len).  The stop iteration is 1-based (the iteration after whose
 * convergence test the shift stopped), 0 for a shift that never stopped; for shifted_lopbicg the seed is the one passed in.
 * After a solve of the LOP family it is the seed passed in and 0 for every shift: there no shift stops on its own. */
int bicg_shifted_solve(bicg_matrix *m, double *x_set, double *r, const double *sigma, int sigma_len, int seed, bicg_stats *stats);
int bicg_last_shift_info(int *seed, int *stop_iter, int cap);
/* Any shifted solver on a resident matrix: BICG_SHIFTED_SWITCHING = shifted_lopbicg_switching (returns iterations + 1, like
 * bicg_shifted_solve), BICG_SHIFTED_LOP = shifted_lopbicgstab, BICG_SHIFTED_PIPE_LOP = shifted_pipe_lopbicgstab,
 * BICG_SHIFTED_LOPBICG = shifted_lopbicg (these three return the iterations performed).  -1 for an unknown method,
 * sigma_len <= 0 or seed outside [0, sigma_len).  Any sigma_len > 0 works, in every shifted entry point of this header, as
 * far as device memory holds x_set, p_j of every shift and, for the switching and fixed-seed solvers, their
 * sigma_len x (BICG_SHIFT_MAX_ITER + 1) history of pi. */
enum { BICG_SHIFTED_SWITCHING = 0, BICG_SHIFTED_LOP = 1, BICG_SHIFTED_PIPE_LOP = 2, BICG_SHIFTED_LOPBICG = 3 };
int bicg_shifted_solve_ex(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                          bicg_stats *stats);
/* bicg_shifted_solve_ex on DEVICE memory: x_set is sigma_len contiguous blocks of n_loc doubles (initial guesses in, solutions
 * out, updated in place; no padding or alignment required), r is n_loc doubles (b in, seed residual out). sigma stays a host
 * array. Same methods, return values, stdout, statistics, bicg_last_* results and BICG_SHIFT_ERROR report as
 * bicg_shifted_solve_ex, except that h2d_bytes and d2h_bytes are 0: x_set never crosses PCIe (it is staged device to device
 * through the handle's workspace, as in bicg_shifted_solve_async). Returns once the library's stream has synchronised, with the results in the caller's buffers. Collective:
 * every rank returns -1 if any rank passed a null pointer, an unknown method, sigma_len <= 0 or a seed outside
 * [0, sigma_len), or if the ranks disagree on method, sigma_len or seed. */
int bicg_shifted_solve_dev(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                           bicg_stats *stats);

/* Written by the device at the end of an asynchronous shifted solve, in stream order (32 bytes): ret is what
 * bicg_shifted_solve_dev returns for the same solve (switching: iterations + 1), iters / converged / final_res are its
 * bicg_stats fields, seed the seed the solve ended with (bicg_last_shift_info's seed), and error = 1 if a bounded wait for a
 * peer GPU or another CTA timed out (BICG_PEER_TIMEOUT_S). */
typedef struct {
    int    ret;
    int    iters;
    int    converged;
    int    seed;
    int    error;
    int    reserved;
    double final_res;
} bicg_shift_result;

/* bicg_shifted_solve_dev enqueued on the caller's CUDA stream `stream` (a cudaStream_t; 0 is CUDA's default stream).  x_set
 * (sigma_len blocks of n_loc doubles, any 8-byte alignment), r (b in, seed residual out) and sigma (sigma_len doubles) are all
 * DEVICE pointers, read and written in stream order: a replay of a captured solve picks up new values in the same buffers.
 * `result` (a bicg_shift_result) and `stop_iter` (sigma_len ints: what bicg_last_shift_info reports for the same solve) are
 * optional device memory.  x_set, r, stop_iter and the result are bit-identical to bicg_shifted_solve_dev's.  Returns 0 once the
 * work is enqueued, with no host synchronisation, allocation, pageable copy or output; -1 for a null pointer, an unknown
 * method, sigma_len <= 0 or a seed outside [0, sigma_len); -2 inside a stream capture when the handle has not been prepared
 * for this method and sigma_len under the current BICG_SHIFT_MAX_ITER (the capture stays valid).  BICG_SHIFT_TOL and
 * BICG_SHIFT_MAX_ITER are read at enqueue time; a captured solve keeps the values it was captured with.
 *
 * x_set, r and sigma are staged through buffers on the handle: copied in at the start and x_set, r copied back at the end
 * (device to device), so the call holds no pointer of the caller beyond its own enqueue.  Ordering is that of
 * bicg_solve_async: calls on one handle, synchronous or asynchronous, plain or shifted, run in the order they were made.
 * Not updated by asynchronous shifted solves: bicg_last_stats, bicg_last_history, bicg_last_shift_info and
 * bicg_last_shift_error; nothing is printed (not the seed-switch report either), and the BICG_SHIFT_ERROR check does not run
 * (call bicg_shift_residuals after synchronising).  With several ranks the call is collective like bicg_shifted_solve_dev.
 *
 * bicg_shifted_solve_async_prepare builds, outside any capture, the handle's workspace of the method's family (switching and
 * fixed seed; LOP and PIPE-LOP) for sigma_len and the current BICG_SHIFT_MAX_ITER, and the graphs of its device-side loop.  It
 * may synchronise and allocate; an uncaptured bicg_shifted_solve_async calls it itself.  Collective: every rank returns -1 if
 * any rank passed a null handle, an unknown method or sigma_len <= 0, or the ranks disagree on method or sigma_len; else 0.
 * A workspace outgrown by a new sigma_len or a larger BICG_SHIFT_MAX_ITER is replaced; after a capture on the handle the old
 * one stays allocated until the handle is destroyed, because the captured graph still uses it.
 *
 * bicg_matrix_shift_history waits for the handle's last work and copies the seed history of the last asynchronous shifted
 * solve on m, the entries bicg_last_history returns after the synchronous solve; returns their number (0 if there was none). */
int bicg_shifted_solve_async(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                             void *stream, bicg_shift_result *result, int *stop_iter);
int bicg_shifted_solve_async_prepare(bicg_matrix *m, int method, int sigma_len);
int bicg_matrix_shift_history(bicg_matrix *m, double *out, int cap);

/* out[j] = ||(A + sigma_j I) x_j - b|| / ||b||, j < sigma_len; x_set: sigma_len blocks of n_loc doubles, b: n_loc doubles, both
 * host pointers, or device pointers when device_vectors != 0.  Collective over the ranks, which pass the same sigma_len: every rank
 * returns -1 when any rank passed sigma_len <= 0 or a null pointer, or the ranks' sigma_len differ.  Any sigma_len > 0 works.
 * One fused pass over the matrix serves a batch of shifts (csrc/shift_check.cu). */
int bicg_shift_residuals(bicg_matrix *m, const double *x_set, const double *b, const double *sigma, int sigma_len,
                         int device_vectors, double *out);
/* With the option SHIFT_ERROR = 1 (BICG_SHIFT_ERROR; the reference's DISPLAY_ERROR) every shifted solver computes, after its timed
 * region, the relative error above for each of its solutions, against the b it was given, and rank 0 prints it in the reference's
 * format.  This returns those errors of the last shifted solve: sigma_len, or 0 if the option was off. */
int bicg_last_shift_error(double *out, int cap);

/* y_loc = A x_loc on a resident matrix (host pointers) -- the kernel behind MPI_csr_spmv_ovlap. */
int bicg_spmv(bicg_matrix *m, const double *x_loc, double *y_loc);

/* y_j = alpha (A + sigma_j I) x_j + beta y_j on this rank's rows, j < nvec: forming a right-hand side from the current matrix,
 * a true residual b - A x (alpha = -1, beta = 1, y = b), (A + sigma_j I) x_j for the x_set of a shifted solve.  x and y are
 * nvec contiguous blocks of n_loc doubles (the x_set layout: any 8-byte alignment, no padding).  sigma is null (no shift term)
 * or nvec doubles.  One pass over the matrix serves up to 8 vectors (csrc/multiply.cu).
 *
 * Arithmetic, per component i of vector j:
 *   t = the row sum exactly as bicg_spmv computes it on this handle (same plan, lanes and order over the merged layout), so
 *       with sigma null and alpha = 1, beta = 0, y_j is bit-identical to bicg_spmv(x_j), whatever nvec is;
 *   sigma given: t = fma(sigma_j, x_j[i], t), for every j including sigma_j = 0 (so a null sigma and a zero sigma can differ
 *       in the sign of a zero);
 *   beta == 0: y = alpha * t, and y is not read (a NaN in y does not propagate); else y = fma(alpha, t, beta * y_in).
 * Returns 0, or -1 for a null handle, x or y, nvec <= 0, or x's range overlapping y's (a gather SpMV cannot run in place);
 * these are checked before the device is touched.  bicg_last_stats, bicg_last_history and bicg_last_shift_* are not updated.
 *
 * bicg_matrix_multiply: x and y are host pointers, or device pointers when device_vectors != 0; sigma is a host array.
 * Waits for the handle's earlier asynchronous work and returns once y is in the caller's buffer.
 * bicg_matrix_multiply_async: x, y and sigma are device pointers, read and written in stream order on the caller's CUDA stream
 * `stream` behind the handle's previous work, with the ordering of bicg_solve_async: no host synchronisation, allocation,
 * pageable copy or output.  It needs no prepare step and works inside a stream capture as it is (there is no -2); a replay
 * reads x, y and sigma as they are at that point.
 *
 * Collective, like bicg_spmv: the ghost columns of every x_j come from the neighbours, and the call ends in an empty
 * cross-GPU reduction.  The synchronous call checks its arguments on every rank first: every rank returns -1 if any rank's
 * arguments are bad or the ranks disagree on nvec or on whether sigma is null; a peer timeout is fatal, as in bicg_spmv.  The
 * asynchronous call checks its arguments locally, so the ranks must agree on nvec and on whether sigma is null; a peer timeout
 * there is reported by the next synchronous call on the handle. */
int bicg_matrix_multiply(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta,
                         const double *sigma, int device_vectors);
int bicg_matrix_multiply_async(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta,
                               const double *sigma, void *stream);

/* The multiply with caller weights on the handle's pattern: y_j = alpha A_W x_j + beta y_j for j < nvec on this rank's rows,
 * where A_W is the handle's pattern holding W instead of its values.  W comes in bicg_matrix_set_values' block order: w_diag
 * has diag nz entries and w_offd offd nz entries (bicg_matrix_block_nz); w_offd may be null only where the handle has no offd
 * entries.  This is the product the derivative of bicg_matrix_value_grad needs, without a second resident copy of the matrix.
 *
 * Arithmetic: bit-identical to bicg_matrix_multiply_async with sigma null on a handle whose values were set to W (same plan,
 * lanes, order, beta and NaN rules); so with W equal to the handle's values, it is bit-identical to that multiply.  The
 * handle's values, value tables and persistent-kernel plan are not touched.
 *
 * Device pointers, with the ordering and collectivity of bicg_matrix_multiply_async (ghost columns of x_j from the neighbours,
 * an empty cross-GPU reduction per batch).  W is read in place where the merged order is the block order and the SpMV's tile
 * copies stay inside w_diag (the row-split plan, or w_diag 16-byte aligned with nnz a multiple of 4); otherwise it is first
 * staged into merged order in a buffer on the handle.  bicg_matrix_multiply_values_async_prepare allocates that buffer on
 * every handle where some W may need it (offd entries, or the tile plan), outside any capture; an uncaptured call allocates it
 * itself.  Returns 0; -1 for a null handle, w_diag, x or y, nvec <= 0, a null w_offd on a handle with offd entries, x
 * overlapping y, or W overlapping y, checked before the device is touched; -2 inside a stream capture when the prepare has
 * not run and W needs the staging buffer (the capture stays valid).  The prepare returns 0, or -1 for a null handle; it may
 * synchronise. */
int bicg_matrix_multiply_values_async(bicg_matrix *m, int nvec, const double *w_diag, const double *w_offd,
                                      const double *x, double *y, double alpha, double beta, void *stream);
int bicg_matrix_multiply_values_async_prepare(bicg_matrix *m);

/* The gradient with respect to the stored values of a resident matrix: for x_j = A^-1 b_j and a loss L, with
 * lambda_j = A^-T dL/dx_j (a solve on the handle of bicg_matrix_create_transpose), dL/da_e = -sum_j lambda_j[i] x_j[c] for every
 * stored entry e = (i, c); for y_j = A x_j, dL/da_e = sum_j (dL/dy_j)[i] x_j[c].  Both are this sampled outer product over the
 * pattern.  u (row factors) and v (column factors) are nvec contiguous blocks of n_loc doubles each (the x_set layout of
 * bicg_matrix_multiply); one pass over the pattern serves up to 8 vectors (csrc/value_grad.cu).
 *
 * Arithmetic, per stored entry e of this rank's rows at local row i and column c (own or ghost), for one batch of vectors
 * j0 .. j0 + nb - 1 (batches of up to 8, in order):
 *   t = u_j0[i] * v_j0[c];  t = fma(u_j[i], v_j[c], t) for j = j0 + 1 .. j0 + nb - 1, in that order;
 *   beta == 0: out_e = alpha * t, and out_e is not read (a NaN in it does not propagate); else out_e = fma(alpha, t, beta * out_e).
 * Every batch after the first applies with beta = 1 onto the previous batch's output.  Each output element depends only on its
 * own inputs, so the result does not depend on the launch shape, the SpMV plan or its lanes per row.
 *
 * Order: diag_out[j] belongs to diag entry j of the blocks the handle was created from, and offd_out[j] to offd entry j: the
 * order bicg_matrix_set_values takes, so set_values(diag - eta g_diag, offd - eta g_offd) is a gradient step.  A transpose's
 * order is its own (bicg_matrix_block_nz gives its counts).  offd_out may be null when the handle has no offd entries (always
 * with one rank).  Returns 0, or -1 for a null handle, u, v or diag_out, nvec <= 0, a null offd_out on a handle with offd
 * entries, or an output range overlapping u's or v's; these are checked before the device is touched.
 *
 * bicg_matrix_value_grad: u, v, diag_out and offd_out are host pointers, or device pointers when device_vectors != 0.  Waits
 * for the handle's earlier asynchronous work and returns once the outputs are in the caller's buffers.
 * bicg_matrix_value_grad_async: device pointers, read and written in stream order on the caller's CUDA stream `stream` behind
 * the handle's previous work, with the ordering of bicg_solve_async: no host synchronisation, allocation, pageable copy or
 * output.  It needs no prepare step and works inside a stream capture as it is (there is no -2).
 *
 * Collective when there are peers: the ghost columns of every v_j come from the neighbours, and every batch ends in an empty
 * cross-GPU reduction.  The synchronous call checks its arguments on every rank first: every rank returns -1 if any rank's
 * arguments are bad or the ranks disagree on nvec; a peer timeout is fatal.  The asynchronous call checks its arguments
 * locally, so the ranks must agree on nvec; a peer timeout there is reported by the next synchronous call on the handle. */
int bicg_matrix_value_grad(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta,
                           double *diag_out, double *offd_out, int device_vectors);
int bicg_matrix_value_grad_async(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta,
                                 double *diag_out, double *offd_out, void *stream);

/* Global dot products of vectors in the x_set layout: out[j] = sum over ranks of sum_i u_j[i] v_j[i] for j < nvec, where u and v
 * are nvec contiguous blocks of n_loc doubles each and out is nvec doubles, all DEVICE memory, read and written in stream order
 * on the caller's CUDA stream `stream` behind the handle's previous work, with the ordering of bicg_matrix_multiply_async: no
 * host synchronisation, allocation, pageable copy or output, no prepare step (there is no -2), and it works inside a stream
 * capture.  The handle lends its ranks and scratch: u and v need not have anything to do with its matrix.  Every rank gets the
 * same bits of every out[j].
 *
 * Arithmetic, for one vector j (csrc/dots.cu), fixed by the element index, n_loc and the rank count alone, not by the grid, the
 * SM count or the SpMV plan:
 *   chunks of 4096 elements: chunk c, thread t (t < 256) runs p_t = fma(u[e], v[e], p_t) from p_t = +0.0 over the elements
 *       e = 4096 c + t + 256 s, s = 0 .. 15, those < n_loc, in s order;
 *   the chunk's sum is the tree p_t = p_t + p_(t + h) for h = 128, 64, .., 1, t < h: p_0;
 *   the rank's sum adds the chunk sums in chunk order onto +0.0 (n_loc = 0: +0.0);
 *   out[j] adds the ranks' sums in rank order: S_0 + S_1 + ... + S_(P-1).
 * No result is -0.  Vectors go in batches of up to 8, one cross-GPU reduction each (the shifted solvers' reduction).
 *
 * Returns 0, or -1 for a null handle, u, v or out, or nvec <= 0; these are checked before the device is touched.  Collective
 * when there are peers: the ranks must agree on nvec; a peer timeout is reported by the next synchronous call on the handle. */
int bicg_matrix_dots_async(bicg_matrix *m, int nvec, const double *u, const double *v, double *out, void *stream);

/* Time `reps` launches of the fused SpMV + (r_hat, s) dot kernel (the dominant kernel of every
 * variant) with CUDA events on the library's stream; returns average ms per launch in *ms and the
 * algorithmic bytes of one launch (12 nnz + 28 n_loc, SURVEY.md 8(d) phase P1) in *bytes. */
int bicg_spmv_time(bicg_matrix *m, int reps, double *ms, double *bytes);

/* per-kernel-class device time of one kernel-per-phase solve of exactly `iters` iterations (tol = 0) from x = 0, b = 1,
 * every kernel launched from the host and bracketed by events (krr/nrr as in bicg_solve).
 * classes: 0 = SpMV(+dots), 1 = fused vector updates, 2 = other.  ms are totals over the solve. */
int bicg_profile_solve(bicg_matrix *m, int method, int iters, int krr, int nrr, double class_ms[3], int class_launches[3]);

/* Test hooks for kernel-level parity (tests/test_gpu_kernels.py); single rank.  `vecs` holds the 11 arena vectors
 * x r r# p s y|z w v t b ax (n_loc doubles each), in and out.
 *   bicg_debug_vec_phase: ONE fused vector phase (enum Phase of csrc/vec.cuh) with coef = {alpha, beta, omega}; returns the
 *                         number of dot products the phase reduces, their values in dots[].
 *   bicg_debug_spmv_epi : s = A p with the solver's epilogue dots (1: (r#,s); 2: (r,s),(s,s); 3: w = A p with
 *                         (r#,r),(r#,w),(r#,ax),(r#,z)).
 *   bicg_debug_get_vec / _get_scalars: arena vector `id` / {rTr rTr_old rTs rTy yTy rTw wTw rTz dot_r dot_zero alpha
 *                         beta omega} as the last solve on this handle left them.
 *   bicg_debug_resident_ctas: how many CTAs of the last persistent-kernel launch on this handle kept their matrix slice in
 *                         shared memory for the whole solve (BICG_RESIDENT, csrc/mega.cu).
 *   bicg_debug_coded_ctas: how many CTAs of the last persistent-kernel launch on this handle streamed 16-bit column codes
 *                         instead of 32-bit columns (csrc/mega.cu).
 *   bicg_debug_stream_codes: on = 0 makes every streaming CTA of later launches on this handle stream 32-bit columns,
 *                         on = 1 restores the default; returns the previous setting.  Both formats give bit-identical results.
 *   bicg_debug_packed_ctas: how many CTAs of the last persistent-kernel launch on this handle streamed 7-byte packed values
 *                         (a per-CTA sign / exponent table index + the 52 mantissa bits) instead of 8-byte values (csrc/mega.cu).
 *   bicg_debug_stream_values: on = 0 makes every streaming CTA of later launches on this handle stream 8-byte values (the
 *                         column codes stay), on = 1 restores the default; returns the previous setting.  Both formats give
 *                         bit-identical results.
 *   bicg_debug_value_grad_layout: later value gradients on this handle use `lanes` threads per row (1, 2, 4, ..., 32; 0: the
 *                         library's choice), and, when blk_ptr is not null, take the merged rows as split into diag and offd
 *                         parts by the device array blk_ptr = [diag row pointers | offd row pointers] (2 (n_loc + 1)
 *                         unsigned, diag_ptr[i] + offd_ptr[i] = the merged row start), writing diag_out and offd_out in
 *                         that order, as a handle with offd entries does (null: the handle's own order; device-pointer calls
 *                         only).  blk_ptr must stay
 *                         valid while it is set, and is refused (-1) on a handle with offd entries; -1 also for a null handle
 *                         or a bad lanes. */
int bicg_debug_vec_phase(bicg_matrix *m, int phase, const double coef[3], double *vecs, double dots[8]);
int bicg_debug_spmv_epi(bicg_matrix *m, int epi, double *vecs, double dots[8]);
int bicg_debug_get_vec(bicg_matrix *m, int id, double *out);
int bicg_debug_get_scalars(bicg_matrix *m, double out[13]);
int bicg_debug_resident_ctas(bicg_matrix *m);
int bicg_debug_coded_ctas(bicg_matrix *m);
int bicg_debug_stream_codes(bicg_matrix *m, int on);
int bicg_debug_packed_ctas(bicg_matrix *m);
int bicg_debug_stream_values(bicg_matrix *m, int on);
int bicg_debug_value_grad_layout(bicg_matrix *m, int lanes, const unsigned *blk_ptr);

/* full-precision history of the last solve on this rank: out[k] = dot_r/dot_zero after iteration k
 * (out[0] = 1).  Returns the number of entries available (iters + 1). */
int bicg_last_history(double *out, int cap);
const bicg_stats *bicg_last_stats(void);

/* the library's compute stream (a cudaStream_t) so callers can record their own events on it */
void *bicg_stream(void);
int   bicg_device(void);
void  bicg_synchronize(void);
/* pinned host allocations for callers that want full-rate host<->device copies */
void *bicg_host_alloc(size_t bytes);
void  bicg_host_free(void *p);

/* Host-side planning, exposed for CPU-only tests (no CUDA call inside). */
void bicg_plan_partition(int n, int world, int *counts, int *displs);          /* matrix.c:295-308 */
/* nnz-balanced contiguous partition (archive/matrix.c:407-420, DYNAMIC_ROWS): used by the loader and the generators when
 * BICG_PARTITION=nnz; row_nnz[i] = entries of global row i. */
void bicg_plan_partition_nnz(const unsigned int *row_nnz, int n, int world, int *counts, int *displs);
/* SpMV tile plan for a CSR block: tiles of <= rows_per_tile rows and <= cap_nnz entries.
 * Writes tile_row[0..ntiles] (first row of each tile); returns ntiles, or -1 if tile_row_cap is too small,
 * or -2 if a single row exceeds cap_nnz. */
int  bicg_plan_tiles(const unsigned int *ptr, int rows, int rows_per_tile, int cap_nnz, int *tile_row,
                     int tile_row_cap);
/* Tile plan of the persistent solver kernel: CTA g of `ctas` owns a contiguous row range starting at a multiple of 16
 * rows; ranges are balanced by per-row work 24*nnz(row) + 216 + extra_weight*row_extra[row] (row_extra may be NULL) and
 * cut into tiles of <= rows_per_tile rows of equal height.  tile_row[0..ntiles] (first row of each tile, then `rows`),
 * cta_tile[0..ctas] (first tile of each CTA).  Returns ntiles (or -needed ints), *max_tile_nnz = entries of the fullest tile. */
int  bicg_plan_cta_tiles(const unsigned int *ptr, int rows, int ctas, int rows_per_tile, const unsigned char *row_extra,
                         int extra_weight, int *tile_row, int tile_row_cap, int *cta_tile, unsigned int *max_tile_nnz);
/* The same with a stage capacity: tiles hold <= cap_limit entries; a row longer than cap_limit becomes a run of chunk tiles
 * (tile_flag 1 = more chunks of the row follow, 2 = last chunk, 0 = ordinary tile of whole rows); tile_nz[t] = first entry of
 * tile t.  The three tile arrays need tile_cap ints each. */
int  bicg_plan_cta_tiles_capped(const unsigned int *ptr, int rows, int ctas, int rows_per_tile, int cap_limit, int *tile_row,
                                unsigned int *tile_nz, int *tile_flag, int tile_cap, int *cta_tile, unsigned int *max_tile_nnz);
/* Halo plan of rank `self`: which global columns of the offd block it must receive, as merged runs.
 * runs_out holds triples (first_col, length, owner); returns the number of runs (or -needed if cap is small).
 * gap: runs of one owner separated by <= gap unreferenced columns are merged. */
int  bicg_plan_halo_runs(const CSR_Matrix *offd, const INFO_Matrix *info, int self, int world, int gap,
                         int *runs_out, int runs_cap);

/* The device layout of rank `self`: its diag / offd blocks merged into one CSR over [own columns | ghost slots]
 * (ghost slot g = column ghost_off + g; per row diag entries first, then offd, matrix.c:437-440).  Outputs are
 * caller-allocated: ptr_out[rows+1], col_out/val_out[diag.nz + offd.nz], recv_out quadruples (first_col, len,
 * owner, ghost_idx).  Returns the number of quadruples (or -needed ints if recv_cap is too small). */
long long bicg_plan_merge(const CSR_Matrix *diag, const CSR_Matrix *offd, const INFO_Matrix *info, int self, int world,
                          int gap, int ghost_off, unsigned int *ptr_out, unsigned int *col_out, double *val_out,
                          int *recv_out, int recv_cap, int *n_ghost_out);
/* round trip of a few bytes through the registered allgather callback; 0 = every rank's contribution arrived */
int  bicg_comm_selftest(void);

/* What rank `self` pushes to rank `dest`, derived from every rank's receive list (quadruples first_col, len,
 * owner, ghost_idx; `stride` ints reserved per rank, cnts[p] quadruples valid).  Writes triples
 * (local_src_row, len, ghost_offset_on_dest); returns their number (or -needed). */
int  bicg_plan_push_runs(const int *all_recv, const int *cnts, int stride, int self, int dest, int my_first,
                         int *out, int out_cap);

/* Synthetic inputs of SURVEY.md 8(d) / BASELINE.json configs, generated directly as one rank's blocks
 * (malloc'ed like the reference loader's, so csr_free_matrix() releases them).  info->recvcounts/displs
 * must be caller-allocated with `world` entries (main.c:82-83).
 *   kind 0: 15-point 3-D stencil on a g^3 grid ("Transport-like" T'); p0 = diagonal value
 *   kind 1: 5-point 2-D Laplacian on a g x g grid (diag 4, off -1)
 *   kind 2: random, n = g rows, k = (int)p0 entries per row incl. the diagonal (diag = k+1, off in -(0,1])
 *   kind 3: 2-D convection-diffusion g x g, upwind, p0 = Peclet-like convection strength (nonsymmetric)
 */
int bicg_gen_block(int kind, long long g, double p0, uint64_t seed, int rank, int world,
                   CSR_Matrix *diag, CSR_Matrix *offd, INFO_Matrix *info);

#ifdef __cplusplus
}
#endif
#endif /* BICGSTAB_B200_H */
