// dots.cu -- out[j] = sum over ranks sum_i u_j[i] v_j[i], j < nvec, on the caller's stream (bicg_matrix_dots_async): the
// global dot products a caller needs next to the handle's other stream-ordered work, e.g. dL/dsigma_j = -<lambda_j, x_j> in
// the backward of a shifted solve, which with several ranks is a cross-GPU sum that no rank-local library can form.
//
// The order of every sum is fixed by the element index, n_loc and the rank count alone (include/bicgstab_b200.h):
//   chunk c holds elements c DOT_CHUNK .. (c + 1) DOT_CHUNK - 1; its thread t runs an fma chain from +0.0 over the elements
//       c DOT_CHUNK + t + DOT_THREADS s, s = 0 .. DOT_SPAN - 1 (those < n_loc), in s order;
//   the DOT_THREADS thread sums are combined by the tree p[t] = p[t] + p[t + h] for h = DOT_THREADS / 2 .. 1;
//   the chunk sums are added in chunk order onto +0.0 (dot_sum_kernel, one CTA);
//   the ranks' sums are added in rank order by the cross-GPU reduction of the shifted solvers (kernel_tail with tail_store:
//       Scalars::pend), which takes one CTA's values as they are.
// No sum can be -0 (every chain starts at +0.0), so the zeros the grid combination of kernel_tail adds change no bit.
// Vectors come in batches of up to MAX_DOTS, one reduction each.  The chunk sums go to the own part of an arena vector
// (V_T: scratch between calls, which the peers never write), so the call allocates nothing.
#include "engine.hpp"

#include <algorithm>
#include <cstdint>

namespace bicg {

namespace {

constexpr int DOT_THREADS = 256;
constexpr int DOT_SPAN = 16;                              // elements per thread and chunk
constexpr int DOT_CHUNK = DOT_THREADS * DOT_SPAN;
constexpr int DOT_TILE = 512;                             // chunk sums dot_sum_kernel stages through shared memory at a time

struct DotArgs {
    KernelCommon kc;
    const double *u[MAX_DOTS], *v[MAX_DOTS];              // this batch's vectors (slots >= nv repeat the last; not read)
    int n, nv, nchunks;
    double *part;                                          // [nv][nchunks] chunk sums
    double *out;                                           // this batch's nv results
};

__global__ void __launch_bounds__(DOT_THREADS) dot_chunk_kernel(const __grid_constant__ DotArgs a)
{
    __shared__ double s_p[MAX_DOTS][DOT_THREADS];
    const int t = threadIdx.x;
    for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
        const long long e0 = (long long)c * DOT_CHUNK + t;
        double acc[MAX_DOTS];
#pragma unroll
        for (int k = 0; k < MAX_DOTS; ++k) acc[k] = 0.0;
#pragma unroll 4
        for (int s = 0; s < DOT_SPAN; ++s) {
            const long long e = e0 + (long long)s * DOT_THREADS;
            if (e >= a.n) break;
#pragma unroll
            for (int k = 0; k < MAX_DOTS; ++k)
                if (k < a.nv) acc[k] = fma(a.u[k][e], a.v[k][e], acc[k]);
        }
#pragma unroll
        for (int k = 0; k < MAX_DOTS; ++k) s_p[k][t] = acc[k];
        __syncthreads();
        for (int h = DOT_THREADS / 2; h > 0; h >>= 1) {
            if (t < h)
                for (int k = 0; k < a.nv; ++k) s_p[k][t] = s_p[k][t] + s_p[k][t + h];
            __syncthreads();
        }
        if (t < a.nv) a.part[(size_t)t * a.nchunks + c] = s_p[t][0];
        __syncthreads();
    }
}

// one CTA: the chunk sums in chunk order, then the cross-GPU reduction in rank order into Scalars::pend, then out
__global__ void __launch_bounds__(DOT_THREADS) dot_sum_kernel(const __grid_constant__ DotArgs a)
{
    __shared__ double s_tile[MAX_DOTS][DOT_TILE + 1];
    __shared__ double scratch[32 * MAX_DOTS];
    const int t = threadIdx.x;
    double sum = 0.0;                                       // thread k < nv: vector k
    for (int c0 = 0; c0 < a.nchunks; c0 += DOT_TILE) {
        const int nc = min(DOT_TILE, a.nchunks - c0);
        for (int i = t; i < a.nv * nc; i += DOT_THREADS) s_tile[i / nc][i % nc] = a.part[(size_t)(i / nc) * a.nchunks + c0 + i % nc];
        __syncthreads();
        if (t < a.nv)
            for (int c = 0; c < nc; ++c) sum = sum + s_tile[t][c];
        __syncthreads();
    }
    if (t < MAX_DOTS) s_tile[t][0] = t < a.nv ? sum : 0.0;
    __syncthreads();
    double local[MAX_DOTS];
#pragma unroll
    for (int k = 0; k < MAX_DOTS; ++k) local[k] = s_tile[k][0];
    kernel_tail<MAX_DOTS>(a.kc, local, scratch);
    // the thread that ran the tail's finalize reads what it stored (a peer timeout leaves Scalars::error set instead)
    if (t == 0)
        for (int k = 0; k < a.nv; ++k) a.out[k] = a.kc.sc->pend[k];
}

} // namespace

} // namespace bicg

extern "C" int bicg_matrix_dots_async(bicg_matrix *m, int nvec, const double *u, const double *v, double *out, void *stream)
{
    using namespace bicg;
    if (!m || !u || !v || !out || nvec <= 0) return -1;
    Context &c = ctx();
    c.ensure();
    const cudaStream_t st = (cudaStream_t)stream;
    PhaseLauncher pl(m, st);
    const long long n = m->n_loc;
    DotArgs a{};
    a.n = m->n_loc;
    a.nchunks = (int)((n + DOT_CHUNK - 1) / DOT_CHUNK);
    a.part = m->vec(V_T);              // MAX_DOTS * nchunks <= ghost_off doubles: 8 <= 16 for n <= DOT_CHUNK, else <= n / 512 + 8 < n
    const int grid = std::max(1, std::min(a.nchunks, c.sm_count * 8));
    stream_ordered({m}, st, capturing(st), [&] {
        for (int j0 = 0; j0 < nvec; j0 += MAX_DOTS) {
            const int nv = std::min(MAX_DOTS, nvec - j0);
            a.nv = nv;
            for (int k = 0; k < MAX_DOTS; ++k) {
                a.u[k] = u + (j0 + std::min(k, nv - 1)) * n;
                a.v[k] = v + (j0 + std::min(k, nv - 1)) * n;
            }
            a.out = out + j0;
            a.kc = pl.common(tail_store(nv));
            if (a.nchunks) dot_chunk_kernel<<<grid, DOT_THREADS, 0, st>>>(a);
            BICG_CUDA(cudaGetLastError());
            dot_sum_kernel<<<1, DOT_THREADS, 0, st>>>(a);
            BICG_CUDA(cudaGetLastError());
            c.launches += 2;
        }
    });
    return 0;
}
