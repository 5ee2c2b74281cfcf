// shift_check.cu -- the true residual of every shifted system in one pass over the matrix:
//   res2[j] = sum_i ((A x_j)_i + sigma_j x_j[i] - b[i])^2,  j < L,   and   res2[L] = sum_i b[i]^2,
// the check of shifted_switching_solver.c:570-598 (DISPLAY_ERROR) and test_shifted.c:129-154, which run one
// MPI_csr_spmv_ovlap + my_daxpy + norm loop per shift.
//
// One thread per row.  A CTA takes a block of SC_THREADS rows and walks it once per batch of SC_B shifts with the batch's
// accumulators in registers, so a row block's val / col stay in L1 / L2 between batches and the matrix streams from HBM
// about once per launch instead of once per shift.  A launch takes up to SC_LAUNCH shifts (at P = 1), which bounds its shared
// memory; more shifts take more launches.  x_j is read in place (the shifted solve's strided buffer or the caller's).
// Per component the arithmetic is that of the LANES = 1 SpMV followed by the host daxpy: the row is summed left to right
// over the merged layout (diag entries first, then offd) with fma, then fma(sigma_j, x_j[i], sum), then (... - b[i])^2.
// Only the order of the final sums differs: warp shuffles, per-warp partials in shared memory, per-CTA partials
// [grid][L + 1] added in CTA order by shift_res_sum, the ranks' L + 1 sums added in rank order on the host.
//
// With peers, the ghost columns of x_j come from the ghost tail of an arena vector (SC_SLOT): before each batch the owner
// pushes only the boundary runs of its push plan (d_push_runs) from x_j straight into that slot on its neighbours, the
// residual kernel waits for their halo flags, and ends in an empty cross-GPU reduction so that nobody pushes the next batch
// into a slot a peer is still reading.  So with peers a launch holds one batch and the matrix streams once per SC_B shifts.
// At P = 1 there is no push and no barrier.
#include "engine.hpp"

#include <algorithm>
#include <cmath>

namespace bicg {

namespace {

constexpr int SC_B = 8;              // shifts per pass over a row block (their accumulators live in registers)
constexpr int SC_THREADS = 256;      // one row per thread
constexpr int SC_WARPS = SC_THREADS / 32;
constexpr int SC_LAUNCH = 512;       // shifts per launch at P = 1: per-warp partials of SC_LAUNCH + 1 columns in shared memory
static_assert(SC_WARPS * (SC_LAUNCH + 1) * sizeof(double) <= 48 * 1024, "the partials must fit the default shared memory");
// arena vectors whose ghost tails carry the batch's halo (never V_R: a shifted solve returns its seed residual from there)
constexpr int SC_SLOT[SC_B] = {V_X, V_RH, V_P, V_S, V_Y, V_W, V_V, V_T};

struct ShiftCheckArgs {
    KernelCommon kc;                 // world > 1: halo flags + the closing barrier
    const double *val;
    const unsigned *col, *ptr;
    int n;
    const double *x;                 // x_j = x + j * ldx (own rows)
    long long ldx;
    const double *ghost[SC_B];       // world > 1: ghost column c of x_(j0 + k) is ghost[k][c]
    const double *b;
    const double *sigma;             // [L]
    int L, j0, nj;                   // this launch: shifts j0 .. j0 + nj - 1
    int with_b;                      // this launch also sums b^2 (column L)
    int wait_halo, barrier;
    double *part;                    // [gridDim.x][L + 1]
};

__global__ void __launch_bounds__(SC_THREADS) shift_res_kernel(const __grid_constant__ ShiftCheckArgs a)
{
    extern __shared__ double s_part[];                    // [SC_WARPS][nj + 1]: column nj is b^2
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int W = a.nj + 1;
    for (int t = tid; t < SC_WARPS * W; t += SC_THREADS) s_part[t] = 0.0;
    if (a.wait_halo && tid < 32) {
        const bool ok = halo_wait_epoch(a.kc.comm, a.kc.sc->halo_epoch);
        if (!ok && tid == 0) a.kc.sc->error = 1;
    }
    __syncthreads();
    double *wp = s_part + warp * W;
    for (long long r0 = (long long)blockIdx.x * SC_THREADS; r0 < a.n; r0 += (long long)gridDim.x * SC_THREADS) {
        const int row = (int)r0 + tid;
        const bool valid = row < a.n;
        unsigned pb = 0, pe = 0;
        double bi = 0.0;
        if (valid) { pb = a.ptr[row]; pe = a.ptr[row + 1]; bi = a.b[row]; }
        if (a.with_b) {
            const double s = warp_sum(bi * bi);
            if (lane == 0) wp[a.nj] += s;
        }
        for (int k0 = 0; k0 < a.nj; k0 += SC_B) {
            // shifts past the launch's last one re-read that one's vector and are dropped below
            const double *xs[SC_B], *gs[SC_B];
#pragma unroll
            for (int k = 0; k < SC_B; ++k) {
                const int kk = min(k0 + k, a.nj - 1);
                xs[k] = a.x + (long long)(a.j0 + kk) * a.ldx;
                gs[k] = a.ghost[min(kk, SC_B - 1)];              // world > 1 launches hold <= SC_B shifts
            }
            double acc[SC_B];
#pragma unroll
            for (int k = 0; k < SC_B; ++k) acc[k] = 0.0;
            for (unsigned e = pb; e < pe; ++e) {
                const unsigned c = __ldg(a.col + e);
                const double v = __ldg(a.val + e);
                const bool own = c < (unsigned)a.n;
                double xv[SC_B];
#pragma unroll
                for (int k = 0; k < SC_B; ++k) xv[k] = ld_coherent((own ? xs[k] : gs[k]) + c);
#pragma unroll
                for (int k = 0; k < SC_B; ++k) acc[k] = fma(v, xv[k], acc[k]);
            }
#pragma unroll
            for (int k = 0; k < SC_B; ++k) {
                if (k0 + k >= a.nj) break;
                double sq = 0.0;
                if (valid) {
                    const double t = fma(a.sigma[a.j0 + k0 + k], xs[k][row], acc[k]);     // my_daxpy(sigma_j, x_j, y)
                    const double d = t - bi;
                    sq = d * d;
                }
                sq = warp_sum(sq);
                if (lane == 0) wp[k0 + k] += sq;
            }
        }
    }
    __syncthreads();
    for (int j = tid; j < W; j += SC_THREADS) {
        if (j == a.nj && !a.with_b) continue;
        double s = 0.0;
        for (int w = 0; w < SC_WARPS; ++w) s += s_part[w * W + j];
        a.part[(size_t)blockIdx.x * (a.L + 1) + (j == a.nj ? a.L : a.j0 + j)] = s;
    }
    if (a.barrier) {
        double none[1] = {0.0};
        kernel_tail<0>(a.kc, none, s_part);
    }
}

// out[j] = sum of part[g][j] over g = 0 .. grid - 1 in that order
__global__ void shift_res_sum(const double *part, int grid, int W, double *out)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= W) return;
    double s = 0.0;
    for (int g = 0; g < grid; ++g) s += part[(size_t)g * W + j];
    out[j] = s;
}

// an empty cross-GPU reduction: every rank has finished what it enqueued before
__global__ void shift_barrier_kernel(const __grid_constant__ KernelCommon kc)
{
    __shared__ double scratch[1];
    double none[1] = {0.0};
    kernel_tail<0>(kc, none, scratch);
}

} // namespace

void peer_barrier(bicg_matrix *m, cudaStream_t st)
{
    PhaseLauncher pl(m, st);
    shift_barrier_kernel<<<1, 32, 0, st>>>(pl.common(tail_allreduce(FIN_NONE, 0)));
    BICG_CUDA(cudaGetLastError());
}

std::vector<double> shift_residual_sums(bicg_matrix *m, const double *d_x, long long ldx, const double *d_b, const double *sigma, int L)
{
    Context &c = ctx();
    c.ensure();
    wait_handle(m);
    const int n = m->n_loc, W = L + 1;
    const bool peers = m->world > 1;
    const int nj_max = std::min(L, peers ? SC_B : SC_LAUNCH);  // shifts per launch
    const size_t smem = (size_t)SC_WARPS * (nj_max + 1) * sizeof(double);
    int per_sm = 1;
    BICG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, shift_res_kernel, SC_THREADS, smem));
    const int grid = (int)std::max<long long>(1, std::min<long long>(((long long)n + SC_THREADS - 1) / SC_THREADS,
                                                                       (long long)c.sm_count * std::max(1, per_sm)));
    double *d_sigma = (double *)c.dev_alloc((size_t)L * sizeof(double));
    double *d_part = (double *)c.dev_alloc((size_t)grid * W * sizeof(double));
    double *d_sum = (double *)c.dev_alloc((size_t)W * sizeof(double));
    BICG_CUDA(cudaMemcpyAsync(d_sigma, sigma, (size_t)L * sizeof(double), cudaMemcpyHostToDevice, c.stream));

    PhaseLauncher pl(m);
    ShiftCheckArgs a{};
    a.kc = pl.common(peers ? tail_allreduce(FIN_NONE, 0) : tail_none());
    a.val = m->d_val; a.col = m->d_col; a.ptr = m->d_ptr; a.n = n;
    a.x = d_x; a.ldx = ldx; a.b = d_b; a.sigma = d_sigma; a.L = L; a.part = d_part;
    a.wait_halo = (peers && m->comm.recv_mask != 0) ? 1 : 0;
    a.barrier = peers ? 1 : 0;
    for (int k = 0; k < SC_B; ++k) a.ghost[k] = m->vec(SC_SLOT[k]);
    if (peers) {
        reset_scalars(m, c.cfg.tol, c.cfg.max_iter);          // clears `done`, which every launcher kernel tests first
        peer_barrier(m, c.stream);                            // the peers are done with the slots' ghost tails
    }
    for (int j0 = 0; j0 < L; j0 += nj_max) {
        a.j0 = j0; a.nj = std::min(nj_max, L - j0); a.with_b = j0 == 0;
        if (peers)
            for (int k = 0; k < a.nj; ++k) pl.vec(PH_PUSH, tail_none(), SC_SLOT[k], d_x + (long long)(j0 + k) * ldx);
        shift_res_kernel<<<grid, SC_THREADS, (size_t)SC_WARPS * (a.nj + 1) * sizeof(double), c.stream>>>(a);
        BICG_CUDA(cudaGetLastError());
    }
    shift_res_sum<<<(W + 255) / 256, 256, 0, c.stream>>>(d_part, grid, W, d_sum);
    BICG_CUDA(cudaGetLastError());
    std::vector<double> mine((size_t)W), all((size_t)W * m->world);
    BICG_CUDA(cudaMemcpyAsync(mine.data(), d_sum, (size_t)W * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
    Scalars hs{};
    if (peers) BICG_CUDA(cudaMemcpyAsync(&hs, m->d_sc, sizeof(Scalars), cudaMemcpyDeviceToHost, c.stream));
    BICG_CUDA(cudaStreamSynchronize(c.stream));
    if (hs.error) timeout_fatal(m, "the shifted residual check");
    c.dev_free(d_sigma); c.dev_free(d_part); c.dev_free(d_sum);
    c.host_allgather(mine.data(), all.data(), (size_t)W * sizeof(double));
    std::vector<double> tot(all.begin(), all.begin() + W);
    for (int p = 1; p < m->world; ++p)
        for (int j = 0; j < W; ++j) tot[(size_t)j] += all[(size_t)p * W + j];
    return tot;
}

std::vector<double> shift_relative_errors(bicg_matrix *m, const double *d_x, long long ldx, const double *d_b, const double *sigma, int L)
{
    const std::vector<double> s = shift_residual_sums(m, d_x, ldx, d_b, sigma, L);
    std::vector<double> err((size_t)L);
    for (int j = 0; j < L; ++j) err[(size_t)j] = sqrt(s[(size_t)j]) / sqrt(s[(size_t)L]);   // shifted_switching_solver.c:591
    return err;
}

} // namespace bicg
