// value_grad.cu -- the gradient with respect to a resident matrix's stored values: for every entry e = (i, c) of this rank's
// rows, out_e = alpha sum_j u_j[i] v_j[c] (+ beta out_e), j < nvec, in the caller's block order (bicg_matrix_value_grad,
// synchronous, host or device vectors; bicg_matrix_value_grad_async, device vectors, on the caller's stream, capturable).
// With u_j = lambda_j = A^-T dL/dx_j and v_j = x_j, alpha = -1, that is dL/da_e of a loss of the solutions of A x_j = b_j; with
// u_j = dL/dy_j and v_j = x_j, alpha = 1, the one of y_j = A x_j.
//
// One kernel, row-split like spmv_rowsplit_kernel: a group of LANES threads (the plan's lanes, widened to the mean row) shares
// a row, and each thread forms whole output entries, so a long row is spread over the group and no entry is summed by two
// threads.
// Each output element depends only on its own inputs: the bits do not depend on the grid, the plan or the lanes.  Vectors
// come in batches of up to MUL_NV_MAX, staged as the multiply stages them (HaloBatches: at one rank straight from the caller's
// v_j; with peers through the arena slots whose ghost tails the neighbours fill); every batch after the first adds onto the
// previous one's output with beta = 1.
#include "engine.hpp"

#include <algorithm>
#include <cstdint>

namespace bicg {

namespace {

struct ValueGradArgs {
    KernelCommon kc;                 // tail: the closing barrier with peers, none at one rank
    const unsigned *col;             // merged columns over the extended column space
    const unsigned *ptr;             // merged row pointers
    const unsigned *dptr, *optr;     // the creation's diag / offd row pointers (d_blk_ptr), or null: merged order = diag order
    int rows, nv;                    // nv: vectors of this launch, 1 .. MUL_NV_MAX
    const double *u[MUL_NV_MAX];     // u_j, own rows
    const double *v[MUL_NV_MAX];     // v_j over the extended column space (slots >= nv repeat the last; not read)
    double alpha, beta;              // beta == 0: out is not read
    double *diag_out, *offd_out;
    int wait_halo;                   // 1: the ghost part of every v_j is filled by peers; wait for their halo flags first
};

template <int LANES>
__global__ void __launch_bounds__(256) value_grad_kernel(const __grid_constant__ ValueGradArgs a)
{
    __shared__ double scratch[32];
    const int tid = threadIdx.x;
    if (a.wait_halo) {
        if (tid < 32) {
            const bool ok = halo_wait_epoch(a.kc.comm, a.kc.sc->halo_epoch);
            if (!ok && tid == 0) a.kc.sc->error = 1;
        }
        __syncthreads();
    }
    constexpr int RPB = 256 / LANES;
    const unsigned lane = (unsigned)(tid % LANES);
    const int nv = a.nv;
    for (long long base = (long long)blockIdx.x * RPB; base < a.rows; base += (long long)gridDim.x * RPB) {
        const int row = (int)base + tid / LANES;
        if (row >= a.rows) continue;
        double ui[MUL_NV_MAX];
#pragma unroll
        for (int k = 0; k < MUL_NV_MAX; ++k) ui[k] = k < nv ? a.u[k][row] : 0.0;
        // t = u_0 v_0[c], then fma(u_k, v_k[c], t) in k order; out = alpha t or fma(alpha, t, beta out)
        auto entry = [&](unsigned e, double *out) {
            const unsigned c = a.col[e];
            double t = ui[0] * ld_coherent(a.v[0] + c);
#pragma unroll
            for (int k = 1; k < MUL_NV_MAX; ++k)
                if (k < nv) t = fma(ui[k], ld_coherent(a.v[k] + c), t);
            *out = a.beta == 0.0 ? a.alpha * t : fma(a.alpha, t, a.beta * *out);
        };
        if (a.dptr)
            merge_row(row, a.dptr, a.optr, [&](unsigned k, unsigned j) { entry(k, a.diag_out + j); },
                      [&](unsigned k, unsigned j) { entry(k, a.offd_out + j); }, lane, (unsigned)LANES);
        else
            for (unsigned e = a.ptr[row] + lane; e < a.ptr[row + 1]; e += LANES) entry(e, a.diag_out + e);
    }
    if (a.kc.tail.op == TAIL_NONE) return;
    double none[1] = {0.0};
    kernel_tail<0>(a.kc, none, scratch);
}

int launch_value_grad(int lanes, int grid, const ValueGradArgs &a, cudaStream_t st)
{
    switch (lanes) {
    case 1:  value_grad_kernel<1><<<grid, 256, 0, st>>>(a); break;
    case 2:  value_grad_kernel<2><<<grid, 256, 0, st>>>(a); break;
    case 4:  value_grad_kernel<4><<<grid, 256, 0, st>>>(a); break;
    case 8:  value_grad_kernel<8><<<grid, 256, 0, st>>>(a); break;
    case 16: value_grad_kernel<16><<<grid, 256, 0, st>>>(a); break;
    case 32: value_grad_kernel<32><<<grid, 256, 0, st>>>(a); break;
    default: return (int)cudaErrorInvalidValue;
    }
    return (int)cudaGetLastError();
}

// the checks both calls make before the device is touched: -1 cases of include/bicgstab_b200.h
bool bad_args(const bicg_matrix *m, int nvec, const double *u, const double *v, const double *diag_out, const double *offd_out)
{
    if (!m || !u || !v || !diag_out || nvec <= 0) return true;
    const size_t no = m->nnz_offd, nd = m->nnz - no;
    if ((no || m->vg_blk_ptr) && !offd_out) return true;
    const size_t vec_bytes = (size_t)nvec * (size_t)m->n_loc * sizeof(double);
    for (const double *in : {u, v}) {
        if (overlaps(diag_out, nd * sizeof(double), in, vec_bytes)) return true;
        if (no && overlaps(offd_out, no * sizeof(double), in, vec_bytes)) return true;
    }
    return false;
}

// every batch of one value gradient on st: device pointers
void enqueue_value_grad(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta, double *diag_out,
                        double *offd_out, cudaStream_t st)
{
    const long long n = m->n_loc;
    HaloBatches hb(m, st);
    ValueGradArgs a{};
    a.kc = hb.kc;
    a.col = m->d_col; a.ptr = m->d_ptr; a.rows = m->n_loc;
    const unsigned *blk = m->vg_blk_ptr ? m->vg_blk_ptr : m->nnz_offd ? m->d_blk_ptr : nullptr;
    if (blk) { a.dptr = blk; a.optr = blk + (size_t)m->n_loc + 1; }
    a.alpha = alpha;
    a.diag_out = diag_out; a.offd_out = offd_out;
    a.wait_halo = hb.wait_halo;
    // the plan's lanes, or more: a group as wide as the mean row keeps a warp's column loads and output stores contiguous
    // (the SpMV streams its entries through shared memory and can take one lane per row; this kernel reads them directly)
    int lanes = m->plan.lanes;
    while (lanes < 32 && lanes < m->mean_row) lanes *= 2;
    if (m->vg_lanes) lanes = m->vg_lanes;
    const int rpb = 256 / lanes;
    const int grid = (int)std::max<long long>(1, std::min<long long>((n + rpb - 1) / rpb, (long long)ctx().sm_count * 8));
    for (int j0 = 0; j0 < nvec; j0 += MUL_NV_MAX) {
        const int nv = std::min(MUL_NV_MAX, nvec - j0);
        a.nv = nv;
        a.beta = j0 == 0 ? beta : 1.0;
        for (int k = 0; k < MUL_NV_MAX; ++k) a.u[k] = u + (j0 + std::min(k, nv - 1)) * n;
        hb.stage(v, j0, nv, a.v);
        const int rc = launch_value_grad(lanes, grid, a, st);
        if (rc) fatal("bicgstab_b200: value gradient launch failed (lanes %d grid %d vectors %d): %s", lanes, grid, nv,
                      cudaGetErrorString((cudaError_t)rc));
        ++ctx().launches;
    }
}

} // namespace

} // namespace bicg

extern "C" int bicg_matrix_value_grad(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta,
                                      double *diag_out, double *offd_out, int device_vectors)
{
    using namespace bicg;
    Context &c = ctx();
    // collective (the halo exchange and the barrier): every rank's verdict and nvec
    if (!ranks_agree(bad_args(m, nvec, u, v, diag_out, offd_out), {nvec})) return -1;
    c.ensure();
    wait_handle(m);
    const size_t vbytes = (size_t)nvec * (size_t)m->n_loc * sizeof(double);
    const size_t no = m->nnz_offd, nd = m->nnz - no;
    const double *du = u, *dv = v;
    double *dd = diag_out, *dof = offd_out, *tmp = nullptr;
    if (!device_vectors) {
        tmp = (double *)c.dev_alloc(std::max<size_t>(2 * vbytes + (nd + no) * sizeof(double), sizeof(double)));
        double *t_u = tmp, *t_v = tmp + vbytes / sizeof(double);
        dd = t_v + vbytes / sizeof(double);
        dof = dd + nd;
        c.h2d(t_u, u, vbytes);
        c.h2d(t_v, v, vbytes);
        if (beta != 0.0) {
            if (nd) c.h2d(dd, diag_out, nd * sizeof(double));
            if (no) c.h2d(dof, offd_out, no * sizeof(double));
        }
        du = t_u; dv = t_v;
    }
    enqueue_value_grad(m, nvec, du, dv, alpha, beta, dd, dof, c.stream);
    if (!device_vectors) {
        if (nd) BICG_CUDA(cudaMemcpyAsync(diag_out, dd, nd * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
        if (no) BICG_CUDA(cudaMemcpyAsync(offd_out, dof, no * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
    }
    sync_checked(m, "a value gradient");
    c.dev_free(tmp);
    return 0;
}

extern "C" int bicg_matrix_value_grad_async(bicg_matrix *m, int nvec, const double *u, const double *v, double alpha, double beta,
                                            double *diag_out, double *offd_out, void *stream)
{
    using namespace bicg;
    if (bad_args(m, nvec, u, v, diag_out, offd_out)) return -1;
    ctx().ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    stream_ordered({m}, st, capturing(st), [&] { enqueue_value_grad(m, nvec, u, v, alpha, beta, diag_out, offd_out, st); });
    return 0;
}

extern "C" int bicg_debug_value_grad_layout(bicg_matrix *m, int lanes, const unsigned *blk_ptr)
{
    if (!m || lanes < 0 || lanes > 32 || (lanes & (lanes - 1)) || (blk_ptr && m->nnz_offd)) return -1;
    m->vg_lanes = lanes;
    m->vg_blk_ptr = blk_ptr;
    return 0;
}
