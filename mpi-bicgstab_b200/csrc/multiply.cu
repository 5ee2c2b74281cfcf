// multiply.cu -- y_j = alpha (A + sigma_j I) x_j + beta y_j, j < nvec, on a resident matrix: bicg_matrix_multiply (synchronous,
// host or device vectors) and bicg_matrix_multiply_async (device vectors, on the caller's stream, capturable).
//
// The work is the SpMV kernels of spmv.cu with the multiply's epilogue, on the handle's SpMV plan: a launch takes up to
// MUL_NV_MAX vectors and streams the matrix once for all of them, so every row sum is the one bicg_spmv computes for that
// vector alone.  At one rank the
// kernels gather straight from the caller's x_j and write straight into y_j.  With peers the ghost columns of x_j come from
// the ghost tail of an arena vector (MUL_SLOT[k], the slots of shift_check.cu): the owner copies x_j's own rows into that
// vector, so the kernel reads one extended vector, and pushes the boundary runs into the same slot on its neighbours.  Each
// launch then ends in an empty cross-GPU reduction, so no rank pushes the next batch into a slot a peer is still reading.
// HaloBatches does this staging for the value gradient (value_grad.cu) too.
//
// bicg_matrix_multiply_values_async runs the same launches with caller weights W in place of the handle's values: the kernels
// read their values through SpmvArgs::val, which points at W itself where W's block order is the merged order and the tile
// kernel's bulk copies stay inside it, and otherwise at m->d_wval, into which W is first staged (merge_values).
#include "engine.hpp"

#include <algorithm>
#include <cstdint>

namespace bicg {

namespace {

// arena vectors whose ghost tails carry a batch's halo with peers (never V_R: a shifted solve returns its seed residual there)
constexpr int MUL_SLOT[MUL_NV_MAX] = {V_X, V_RH, V_P, V_S, V_Y, V_W, V_V, V_T};

// the checks both calls make before the device is touched: -1 cases of include/bicgstab_b200.h
bool bad_args(const bicg_matrix *m, int nvec, const double *x, const double *y)
{
    if (!m || !x || !y || nvec <= 0) return true;
    // a gather SpMV cannot run in place; x == y counts as overlapping even without rows
    const uintptr_t bytes = std::max<uintptr_t>((uintptr_t)nvec * (uintptr_t)m->n_loc * sizeof(double), sizeof(double));
    const uintptr_t x0 = (uintptr_t)x, y0 = (uintptr_t)y;
    return x0 < y0 + bytes && y0 < x0 + bytes;
}

// W is staged into merged order where it has offd entries, and on the tile plan unless the tile kernel's bulk copies, which
// read whole 16-byte units from 16-byte aligned addresses, stay inside w_diag: W 16-byte aligned, nnz a multiple of 4.  Only
// the row-split plan without offd entries never needs the staging buffer.
bool weights_may_stage(const bicg_matrix *m) { return m->nnz_offd || m->plan.kind == 0; }
bool weights_in_place(const bicg_matrix *m, const double *w_diag)
{
    if (m->nnz_offd) return false;
    return m->plan.kind != 0 || ((uintptr_t)w_diag % 16 == 0 && m->nnz % 4 == 0);
}

} // namespace

HaloBatches::HaloBatches(bicg_matrix *mm, cudaStream_t st) : m(mm), pl(mm, st), peers(mm->world > 1)
{
    kc = pl.common(peers ? tail_allreduce(FIN_NONE, 0) : tail_none());
    wait_halo = (peers && m->comm.recv_mask != 0) ? 1 : 0;
    if (peers) {
        // the halo push returns at once while `done` is set (as a finished solve leaves it); then wait until the peers are
        // done with the slots' ghost tails
        BICG_CUDA(cudaMemsetAsync(&m->d_sc->done, 0, sizeof(int), st));
        peer_barrier(m, st);
    }
}

void HaloBatches::stage(const double *x, int j0, int nv, const double *(&xs)[MUL_NV_MAX])
{
    const long long n = m->n_loc;
    for (int v = 0; v < MUL_NV_MAX; ++v) {
        const int k = std::min(v, nv - 1);
        xs[v] = peers ? m->vec(MUL_SLOT[k]) : x + (j0 + k) * n;
    }
    if (!peers) return;
    for (int k = 0; k < nv; ++k) {
        const double *xk = x + (j0 + k) * n;
        BICG_CUDA(cudaMemcpyAsync(m->vec(MUL_SLOT[k]), xk, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, pl.stream));
        pl.vec(PH_PUSH, tail_none(), MUL_SLOT[k], xk);
    }
}

namespace {

// every batch of one multiply on st with the values val (merged order): x, y device pointers, sigma nvec device values or null
void enqueue_multiply(bicg_matrix *m, const double *val, int nvec, const double *x, double *y, double alpha, double beta,
                      const double *sigma, cudaStream_t st)
{
    const SpmvPlan &p = m->plan;
    const long long n = m->n_loc;
    HaloBatches hb(m, st);
    SpmvArgs a{};
    a.kc = hb.kc;
    a.val = val; a.col = m->d_col; a.ptr = m->d_ptr; a.rows = m->n_loc;
    a.tile_row = p.d_tile_row; a.tile_nz = p.d_tile_nz; a.ntiles = p.ntiles; a.cap = p.cap; a.stages = p.stages;
    a.alpha = alpha; a.beta = beta;
    a.wait_halo = hb.wait_halo;
    const size_t smem = p.kind == 0 ? (size_t)p.stages * spmv_stage_bytes(p.cap, p.threads / p.lanes, 0) : 0;
    for (int j0 = 0; j0 < nvec; j0 += MUL_NV_MAX) {
        const int nv = std::min(MUL_NV_MAX, nvec - j0);
        a.nv = nv;
        a.sigma = sigma ? sigma + j0 : nullptr;
        for (int v = 0; v < MUL_NV_MAX; ++v) a.y[v] = y + (j0 + std::min(v, nv - 1)) * n;
        hb.stage(x, j0, nv, a.x);
        const int rc = launch_spmv(p.kind, p.lanes, p.threads, p.grid, smem, false, a, st);
        if (rc) fatal("bicgstab_b200: multiply launch failed (kind %d lanes %d threads %d grid %d vectors %d): %s", p.kind, p.lanes,
                      p.threads, p.grid, nv, cudaGetErrorString((cudaError_t)rc));
        ++ctx().launches;
    }
}

// m->d_wval, outside any capture
void alloc_weights(bicg_matrix *m)
{
    if (m->d_wval) return;
    Context &c = ctx();
    wait_handle(m);
    m->d_wval = (double *)c.dev_alloc((m->nnz + 16) * sizeof(double));
    BICG_CUDA(cudaMemsetAsync(m->d_wval, 0, (m->nnz + 16) * sizeof(double), c.stream));
    BICG_CUDA(cudaStreamSynchronize(c.stream));
}

} // namespace

} // namespace bicg

extern "C" int bicg_matrix_multiply(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta,
                                    const double *sigma, int device_vectors)
{
    using namespace bicg;
    Context &c = ctx();
    // collective (the halo exchange and the barrier): every rank's verdict, nvec and whether it passed sigma
    if (!ranks_agree(bad_args(m, nvec, x, y), {nvec, sigma ? 1 : 0})) return -1;
    c.ensure();
    wait_handle(m);
    const size_t bytes = (size_t)nvec * (size_t)m->n_loc * sizeof(double);
    const double *dx = x;
    double *dy = y, *tmp = nullptr, *d_sigma = nullptr;
    if (!device_vectors) {
        tmp = (double *)c.dev_alloc(2 * bytes);
        dx = tmp; dy = tmp + bytes / sizeof(double);
        c.h2d(tmp, x, bytes);
        if (beta != 0.0) c.h2d(dy, y, bytes);
    }
    if (sigma) {
        d_sigma = (double *)c.dev_alloc((size_t)nvec * sizeof(double));
        BICG_CUDA(cudaMemcpyAsync(d_sigma, sigma, (size_t)nvec * sizeof(double), cudaMemcpyHostToDevice, c.stream));
    }
    enqueue_multiply(m, m->d_val, nvec, dx, dy, alpha, beta, d_sigma, c.stream);
    if (!device_vectors) BICG_CUDA(cudaMemcpyAsync(y, dy, bytes, cudaMemcpyDeviceToHost, c.stream));
    sync_checked(m, "a multiply");
    c.dev_free(tmp); c.dev_free(d_sigma);
    return 0;
}

extern "C" int bicg_matrix_multiply_async(bicg_matrix *m, int nvec, const double *x, double *y, double alpha, double beta,
                                          const double *sigma, void *stream)
{
    using namespace bicg;
    if (bad_args(m, nvec, x, y)) return -1;
    ctx().ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    stream_ordered({m}, st, capturing(st), [&] { enqueue_multiply(m, m->d_val, nvec, x, y, alpha, beta, sigma, st); });
    return 0;
}

extern "C" int bicg_matrix_multiply_values_async_prepare(bicg_matrix *m)
{
    using namespace bicg;
    if (!m) return -1;
    ctx().ensure();
    if (weights_may_stage(m)) alloc_weights(m);
    return 0;
}

extern "C" int bicg_matrix_multiply_values_async(bicg_matrix *m, int nvec, const double *w_diag, const double *w_offd,
                                                 const double *x, double *y, double alpha, double beta, void *stream)
{
    using namespace bicg;
    if (bad_args(m, nvec, x, y) || !w_diag || (m->nnz_offd && !w_offd)) return -1;
    const size_t no = m->nnz_offd, nd = m->nnz - no;
    const size_t ybytes = (size_t)nvec * (size_t)m->n_loc * sizeof(double);
    if (overlaps(w_diag, nd * sizeof(double), y, ybytes) || (no && overlaps(w_offd, no * sizeof(double), y, ybytes))) return -1;
    ctx().ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    const bool captured = capturing(st);
    const bool in_place = weights_in_place(m, w_diag);
    if (!in_place && !m->d_wval) {
        if (captured) return -2;
        alloc_weights(m);
    }
    stream_ordered({m}, st, captured, [&] {
        if (!in_place) merge_values(m, w_diag, w_offd, m->d_wval, st);
        enqueue_multiply(m, in_place ? w_diag : m->d_wval, nvec, x, y, alpha, beta, nullptr, st);
    });
    return 0;
}
