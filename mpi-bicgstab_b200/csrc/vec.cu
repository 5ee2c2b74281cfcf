// vec.cu -- the BLAS-1 chains of solver.c as fused single-pass kernels (sm_90a).
//
// The reference walks each length-n vector once per my_daxpy / my_dscal / my_ddot call (vector.c:3-27):
// 7 / 11 / 16 separate passes per iteration for bicgstab / ca_bicgstab / pipe_bicgstab.  Here each group of
// calls between two synchronisation points is ONE kernel: every vector is read once (double2 loads) and
// written once, the dot products that follow are accumulated in the same pass, the grid's partial sums are
// combined in a fixed order by the last CTA, which then also performs the cross-GPU reduction over peer
// memory, evaluates the scalar recurrence on the device (dev.cuh: kernel_tail) and, when the updated vector
// is the next SpMV's input, pushes the boundary runs the neighbours need straight into their ghost regions
// over NVLink (the reference: MPI_Iallgatherv of the whole vector, matrix.c:432).
//
// Per element the operation order and the FMA contraction match what gcc emits for the reference
// (y += a*x -> fma(a, x, y); x *= a -> a*x), so elementwise results are bitwise those of the CPU code.
//
//   phase          reference lines replaced
//   PH_BICG_INIT   solver.c:75-78          PH_BICG_Q    :94              PH_BICG_XR  :105-111
//   PH_BICG_P      :117-119                PH_INIT_R    :201-203         PH_CA_PS    :217-222
//   PH_QY          :225-228 / 361-364      PH_CA_XR     :233-236         PH_PIPE_1   :352-364
//   PH_PIPE_3      :370-380                PH_RR_P      :494-496         PH_RR_X     :518-519
//   PH_RR_R        :524-525                PH_RR_DOTS   :533-539
#include "vec_body.cuh"

namespace bicg {

namespace {

template <int PH>
__global__ void __launch_bounds__(256) vec_kernel(const __grid_constant__ VecArgs a)
{
    const Scalars *sc = a.kc.sc;
    if (sc->done) return;
    __shared__ double scratch[32 * MAX_DOTS];
    constexpr int ND = phase_ndot(PH);
    constexpr int NDA = ND > 0 ? ND : 1;

    Coef c;
    c.al = sc->alpha; c.be = sc->beta; c.om = sc->omega; c.nbo = -c.be * c.om;   // solver.c:119  -beta*omega

    const int lo = (int)blockIdx.x * a.chunk;
    const int hi = min(a.n, lo + a.chunk);
    double dot[NDA];
#pragma unroll
    for (int k = 0; k < NDA; ++k) dot[k] = 0.0;

    if constexpr (PH != PH_PUSH) {
        // 4 doubles (two 16-byte loads per vector) per thread and step: twice the bytes in flight of a
        // double2 loop; lo is a multiple of 4 and every vector is 128-byte aligned
        int i = lo + 4 * (int)threadIdx.x;
        for (; i + 3 < hi; i += 4 * (int)blockDim.x) body<PH, Contig<4>>(a.v, i, c, dot);
        for (; i < hi; ++i) body<PH, Contig<1>>(a.v, i, c, dot);  // < 4 trailing elements of the last chunk (one thread)
    }

    const bool pushing = a.push.npeers > 0;
    if (pushing) {
        __syncthreads();                 // this CTA's elements are final
        push_chunk(a.push, lo, hi, (int)threadIdx.x, (int)blockDim.x);
        // the peer stores are ordered before the halo flag by ONE system-scope fence per CTA: kernel_tail's
        // thread 0 fences after the __syncthreads that follows (cumulativity covers the whole CTA's stores);
        // a fence.sys in every thread costs microseconds per kernel
    }
    if (ND == 0 && a.kc.tail.op == TAIL_NONE && !a.kc.tail.signal_halo) return;
    if (ND > 0) block_sum<NDA>(dot, scratch);
    kernel_tail<ND>(a.kc, dot, scratch);
}

template <int PH>
cudaError_t launch(int grid, const VecArgs &a, cudaStream_t st)
{
    vec_kernel<PH><<<grid, 256, 0, st>>>(a);
    return cudaGetLastError();
}

} // namespace

int launch_vec(int phase, int grid, const VecArgs &a, cudaStream_t st)
{
    switch (phase) {
    case PH_BICG_INIT: return (int)launch<PH_BICG_INIT>(grid, a, st);
    case PH_BICG_Q:    return (int)launch<PH_BICG_Q>(grid, a, st);
    case PH_BICG_XR:   return (int)launch<PH_BICG_XR>(grid, a, st);
    case PH_BICG_P:    return (int)launch<PH_BICG_P>(grid, a, st);
    case PH_INIT_R:    return (int)launch<PH_INIT_R>(grid, a, st);
    case PH_CA_PS:     return (int)launch<PH_CA_PS>(grid, a, st);
    case PH_QY:        return (int)launch<PH_QY>(grid, a, st);
    case PH_CA_XR:     return (int)launch<PH_CA_XR>(grid, a, st);
    case PH_PIPE_1:    return (int)launch<PH_PIPE_1>(grid, a, st);
    case PH_PIPE_3:    return (int)launch<PH_PIPE_3>(grid, a, st);
    case PH_RR_P:      return (int)launch<PH_RR_P>(grid, a, st);
    case PH_RR_X:      return (int)launch<PH_RR_X>(grid, a, st);
    case PH_RR_R:      return (int)launch<PH_RR_R>(grid, a, st);
    case PH_RR_DOTS:   return (int)launch<PH_RR_DOTS>(grid, a, st);
    case PH_PUSH:      return (int)launch<PH_PUSH>(grid, a, st);
    default:           return (int)cudaErrorInvalidValue;
    }
}

} // namespace bicg
