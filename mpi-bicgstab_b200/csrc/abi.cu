// abi.cu -- the extern "C" surface of libbicgstab_b200.so (include/bicgstab_b200.h).
// Part 1: the reference's own entry points (solver.h:10-13, matrix.h:51) on host pointers.
// Part 2: bicg_* extensions: communication, options, the handle's lifetime, results of the last call, the library's stream
// and host memory, and the calls around internal functions that other code calls too.  Every other bicg_* entry point on a
// handle is defined in the file that does its work.
#include "engine.hpp"

#include <cmath>
#include <cstring>
#include <ctime>

using namespace bicg;

static_assert(sizeof(CSR_Matrix) == 40, "CSR_Matrix layout must match matrix.h:19-26");
static_assert(offsetof(CSR_Matrix, col) == 8 && offsetof(CSR_Matrix, ptr) == 16 && offsetof(CSR_Matrix, nz) == 24 &&
              offsetof(CSR_Matrix, rows) == 28 && offsetof(CSR_Matrix, cols) == 32, "CSR_Matrix layout");
static_assert(sizeof(INFO_Matrix) == 32, "INFO_Matrix layout must match matrix.h:28-33");
static_assert(offsetof(INFO_Matrix, code) == 12 && offsetof(INFO_Matrix, recvcounts) == 16 &&
              offsetof(INFO_Matrix, displs) == 24, "INFO_Matrix layout");
static_assert(sizeof(bicg_result) == 24 && offsetof(bicg_result, iters) == 0 && offsetof(bicg_result, converged) == 4 &&
              offsetof(bicg_result, error) == 8 && offsetof(bicg_result, reserved) == 12 &&
              offsetof(bicg_result, final_res) == 16, "bicg_result layout of include/bicgstab_b200.h");
static_assert(sizeof(bicg_shift_result) == 32 && offsetof(bicg_shift_result, ret) == 0 && offsetof(bicg_shift_result, iters) == 4 &&
              offsetof(bicg_shift_result, converged) == 8 && offsetof(bicg_shift_result, seed) == 12 &&
              offsetof(bicg_shift_result, error) == 16 && offsetof(bicg_shift_result, reserved) == 20 &&
              offsetof(bicg_shift_result, final_res) == 24, "bicg_shift_result layout of include/bicgstab_b200.h");

namespace {

// the shifted entry points of shifted_switching_solver.h and shifted_solver.h (method = BICG_SHIFTED_*)
int run_shifted(int method, CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                int sigma_len, int seed)
{
    if (info->cols != info->rows) {   // shifted_switching_solver.c:28-31, 268-271; shifted_solver.c:190-193, 711-714
        printf("Error: matrix is not square.\n");
        exit(1);
    }
    Context &c = ctx();
    c.ensure();
    bicg_matrix *m = matrix_get_cached(D, O, info, nullptr);
    const int k = shifted_solve(m, method, x_loc_set, r_loc, sigma, sigma_len, seed, false);
    if (!c.cfg.cache) matrix_destroy(m);
    return k;
}

int run_reference_entry(int method, CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x, double *r, int krr, int nrr)
{
    if (info->cols != info->rows) {                      // solver.c:43-46
        printf("Error: matrix is not square.\n");
        exit(1);
    }
    Context &c = ctx();
    c.ensure();
    bool fresh = false;
    auto wall = [] { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec; };
    const double t0 = wall();
    bicg_matrix *m = matrix_get_cached(D, O, info, &fresh);
    const double t1 = wall();
    bicg_stats st{};
    solve(m, method, x, r, krr, nrr, 0, &st);
    const double t2 = wall();
    st.upload_ms = fresh ? matrix_upload_ms(m) : 0.0;
    st.h2d_bytes += fresh ? m->upload_bytes : 0;
    c.last_stats = st;
    print_reference_lines(st, c.last_hist);
    if (!c.cfg.cache) matrix_destroy(m);
    if (c.cfg.verbose >= 2)
        fprintf(stderr, "[bicg entry r%d] matrix %.3f ms (fresh %d), solve call %.3f ms (loop %.3f ms), destroy %.3f ms\n", c.rank,
                t1 - t0, (int)fresh, t2 - t1, st.loop_ms, wall() - t2);
    return st.iters;
}

} // namespace

extern "C" {

int bicgstab(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc, double *r_loc)
{
    return run_reference_entry(BICG_METHOD_BICGSTAB, D, O, info, x_loc, r_loc, 0, 0);
}
int ca_bicgstab(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc, double *r_loc)
{
    return run_reference_entry(BICG_METHOD_CA, D, O, info, x_loc, r_loc, 0, 0);
}
int pipe_bicgstab(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc, double *r_loc)
{
    return run_reference_entry(BICG_METHOD_PIPE, D, O, info, x_loc, r_loc, 0, 0);
}
int pipe_bicgstab_rr(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc, double *r_loc, int krr, int nrr)
{
    return run_reference_entry(BICG_METHOD_PIPE_RR, D, O, info, x_loc, r_loc, krr, nrr);
}

// shifted_switching_solver.h:12 -- same prototype, host pointers: x_loc_set holds sigma_len blocks of n_loc (initial guesses in,
// solutions out), r_loc b in / seed residual out.  Returns the reference's k (iterations + 1).
int shifted_lopbicg_switching(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                              int sigma_len, int seed)
{
    return run_shifted(BICG_SHIFTED_SWITCHING, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}

// shifted_switching_solver.h:11 -- the fixed-seed variant: same prototype and meaning, but the seed never switches (when it
// converges first it keeps iterating until every shift has stopped) and the return value is k, the iterations performed.
int shifted_lopbicg(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma, int sigma_len,
                    int seed)
{
    return run_shifted(BICG_SHIFTED_LOPBICG, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}

// shifted_switching_solver.c:611 -- the reference's twin of the function above with the halo exchange NOT overlapped with the
// diagonal block's SpMV and per-section timers; the arithmetic is the same (x, r, residual history and return value of the two
// compiled reference functions are bit-identical on the golden cases: tests/test_oracle_golden.py), and "overlapped or not" has
// no counterpart here, so it is the same solve.
int shifted_lopbicg_switching_noovlp(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                                     int sigma_len, int seed)
{
    return shifted_lopbicg_switching(D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}

// shifted_solver.h: the LOP family.  Same prototype and meaning as shifted_lopbicg_switching, but every shift is advanced until all
// have converged (no seed switch) and the return value is k, the iterations performed.  The reference's _v2 and _nooverlap twins
// differ from their first function only in where the per-shift updates and the MPI waits sit; the arithmetic is the same (x, r,
// history and return value of the compiled reference functions are bit-identical on the golden cases:
// tests/test_oracle_golden_shifted_lop.py), so each twin is the same solve here.
int shifted_lopbicgstab(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma, int sigma_len,
                        int seed)                                                         // shifted_solver.h:17
{
    return run_shifted(BICG_SHIFTED_LOP, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}
int shifted_lopbicgstab_v2(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                           int sigma_len, int seed)                                       // shifted_solver.h:18
{
    return run_shifted(BICG_SHIFTED_LOP, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}
int shifted_lopbicgstab_nooverlap(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                                  int sigma_len, int seed)                                // shifted_solver.h:19
{
    return run_shifted(BICG_SHIFTED_LOP, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}
int shifted_pipe_lopbicgstab(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc, double *sigma,
                             int sigma_len, int seed)                                     // shifted_solver.h:20
{
    return run_shifted(BICG_SHIFTED_PIPE_LOP, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}
int shifted_pipe_lopbicgstab_nooverlap(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc_set, double *r_loc,
                                       double *sigma, int sigma_len, int seed)            // shifted_solver.h:21
{
    return run_shifted(BICG_SHIFTED_PIPE_LOP, D, O, info, x_loc_set, r_loc, sigma, sigma_len, seed);
}

void MPI_csr_spmv_ovlap(CSR_Matrix *D, CSR_Matrix *O, INFO_Matrix *info, double *x_loc, double *x, double *y_loc)
{
    Context &c = ctx();
    c.ensure();
    bicg_matrix *m = matrix_get_cached(D, O, info, nullptr);
    if (x && m->world > 1) memcpy(x + info->displs[m->rank], x_loc, (size_t)m->n_loc * sizeof(double));
    spmv_host(m, x_loc, y_loc, x);
    if (!c.cfg.cache) matrix_destroy(m);
}

// ---- Part 2 ------------------------------------------------------------------------------------------

int bicg_abi_version(void) { return BICG_ABI_VERSION; }

int bicg_set_option(const char *key, const char *value) { return set_option(ctx().cfg, key, value); }

int bicg_comm_init(int rank, int world, bicg_allgather_fn allgather, void *user)
{
    if (world < 1 || world > MAX_RANKS || rank < 0 || rank >= world) return -1;
    Context &c = ctx();
    c.rank = rank; c.world = world; c.allgather = allgather; c.allgather_ctx = user;
    return 0;
}
void bicg_comm_finalize(void)
{
    Context &c = ctx();
    std::vector<bicg_matrix *> ms;
    for (auto &kv : c.cache) ms.push_back(kv.second);
    for (bicg_matrix *m : ms) matrix_destroy(m);
    c.cache.clear();
    c.release_arenas();
    c.rank = 0; c.world = 1; c.allgather = nullptr; c.allgather_ctx = nullptr;
}
int bicg_comm_selftest(void)
{
    Context &c = ctx();
    struct Probe { int rank, world; unsigned magic; } mine{c.rank, c.world, 0xB1C65AB0u + (unsigned)c.rank};
    std::vector<Probe> all((size_t)c.world);
    c.host_allgather(&mine, all.data(), sizeof(Probe));
    for (int p = 0; p < c.world; ++p)
        if (all[(size_t)p].rank != p || all[(size_t)p].world != c.world || all[(size_t)p].magic != 0xB1C65AB0u + (unsigned)p) return 1;
    return 0;
}
int bicg_comm_rank(void) { return ctx().rank; }
int bicg_comm_world(void) { return ctx().world; }

bicg_matrix *bicg_matrix_create(const CSR_Matrix *diag, const CSR_Matrix *offd, const INFO_Matrix *info)
{
    return matrix_create(diag, offd, info);
}
void bicg_matrix_destroy(bicg_matrix *m) { matrix_destroy(m); }
void bicg_matrix_invalidate(const CSR_Matrix *diag)
{
    Context &c = ctx();
    if (!diag) return;
    const void *key = diag->val ? (const void *)diag->val : (const void *)diag;
    auto it = c.cache.find(key);
    if (it == c.cache.end()) return;
    bicg_matrix *m = it->second;
    c.cache.erase(it);
    if (m->world == 1) matrix_destroy(m);       // with peers, destruction is collective: leave it to bicg_comm_finalize
    else c.cache[(const void *)m] = m;
}

int bicg_matrix_block_nz(const bicg_matrix *m, unsigned *diag_nz, unsigned *offd_nz)
{
    if (!m || !diag_nz || !offd_nz) return -1;
    *diag_nz = (unsigned)(m->nnz - m->nnz_offd);
    *offd_nz = (unsigned)m->nnz_offd;
    return 0;
}

int bicg_solve(bicg_matrix *m, int method, double *x, double *r, int krr, int nrr, int device_vectors, bicg_stats *stats)
{
    return solve(m, method, x, r, krr, nrr, device_vectors, stats);
}
int bicg_spmv(bicg_matrix *m, const double *x_loc, double *y_loc) { return spmv_host(m, x_loc, y_loc, nullptr); }
int bicg_shifted_solve(bicg_matrix *m, double *x_set, double *r, const double *sigma, int sigma_len, int seed, bicg_stats *stats)
{
    Context &c = ctx();
    const int k = shifted_solve(m, BICG_SHIFTED_SWITCHING, x_set, r, sigma, sigma_len, seed, false);
    if (stats) *stats = c.last_stats;
    return k;
}
int bicg_shifted_solve_ex(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                          bicg_stats *stats)
{
    Context &c = ctx();
    const int k = shifted_solve(m, method, x_set, r, sigma, sigma_len, seed, false);
    if (stats) *stats = c.last_stats;
    return k;
}
int bicg_shifted_solve_dev(bicg_matrix *m, int method, double *x_set, double *r, const double *sigma, int sigma_len, int seed,
                           bicg_stats *stats)
{
    Context &c = ctx();
    // collective (the solve's halo exchanges and reductions): every rank's verdict, method, sigma_len and seed
    const bool known = method == BICG_SHIFTED_SWITCHING || method == BICG_SHIFTED_LOP || method == BICG_SHIFTED_PIPE_LOP ||
                       method == BICG_SHIFTED_LOPBICG;
    if (!ranks_agree(!m || !x_set || !r || !sigma || !known || sigma_len <= 0 || seed < 0 || seed >= sigma_len,
                     {method, sigma_len, seed}))
        return -1;
    c.ensure();
    const int k = shifted_solve(m, method, x_set, r, sigma, sigma_len, seed, true);
    if (stats) *stats = c.last_stats;
    return k;
}
int bicg_last_shift_info(int *seed, int *stop_iter, int cap)
{
    Context &c = ctx();
    if (seed) *seed = c.last_shift_seed;
    const int n = (int)c.last_shift_stop.size();
    for (int i = 0; i < n && i < cap; ++i) stop_iter[i] = c.last_shift_stop[(size_t)i];
    return n;
}
int bicg_last_shift_error(double *out, int cap)
{
    Context &c = ctx();
    const int n = (int)c.last_shift_err.size();
    for (int i = 0; i < n && i < cap; ++i) out[i] = c.last_shift_err[(size_t)i];
    return n;
}
int bicg_shift_residuals(bicg_matrix *m, const double *x_set, const double *b, const double *sigma, int sigma_len, int device_vectors,
                         double *out)
{
    Context &c = ctx();
    // collective (the residual pass): every rank's verdict and sigma_len
    if (!ranks_agree(sigma_len <= 0 || !m || !x_set || !b || !sigma || !out, {sigma_len})) return -1;
    c.ensure();
    const size_t n = (size_t)m->n_loc;
    const double *dx = x_set, *db = b;
    double *tmp = nullptr;
    if (!device_vectors) {
        tmp = (double *)c.dev_alloc(((size_t)sigma_len + 1) * n * sizeof(double));
        BICG_CUDA(cudaMemcpyAsync(tmp, x_set, (size_t)sigma_len * n * sizeof(double), cudaMemcpyHostToDevice, c.stream));
        BICG_CUDA(cudaMemcpyAsync(tmp + (size_t)sigma_len * n, b, n * sizeof(double), cudaMemcpyHostToDevice, c.stream));
        dx = tmp; db = tmp + (size_t)sigma_len * n;
    }
    const std::vector<double> err = shift_relative_errors(m, dx, (long long)n, db, sigma, sigma_len);
    if (tmp) c.dev_free(tmp);
    for (int j = 0; j < sigma_len; ++j) out[j] = err[(size_t)j];
    return 0;
}

int bicg_last_history(double *out, int cap)
{
    Context &c = ctx();
    const int n = (int)c.last_hist.size();
    for (int i = 0; i < n && i < cap; ++i) out[i] = c.last_hist[(size_t)i];
    return n;
}
const bicg_stats *bicg_last_stats(void) { return &ctx().last_stats; }

void *bicg_stream(void) { Context &c = ctx(); c.ensure(); return (void *)c.stream; }
int bicg_device(void) { Context &c = ctx(); c.ensure(); return c.device; }
void bicg_synchronize(void) { Context &c = ctx(); c.ensure(); BICG_CUDA(cudaStreamSynchronize(c.stream)); }
void *bicg_host_alloc(size_t bytes)
{
    Context &c = ctx(); c.ensure();
    void *p = nullptr;
    BICG_CUDA(cudaHostAlloc(&p, bytes, cudaHostAllocDefault));
    return p;
}
void bicg_host_free(void *p) { if (p) cudaFreeHost(p); }

} // extern "C"
