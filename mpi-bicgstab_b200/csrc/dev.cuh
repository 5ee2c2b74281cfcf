// dev.cuh -- device-side building blocks shared by the SpMV and the fused-vector kernels (sm_90a).
//
//   * PTX wrappers: mbarrier + 1-D TMA bulk copies (cp.async.bulk -> SASS UBLKCP), system-scope
//     release/acquire accesses for the NVLink peer mailboxes;
//   * deterministic block / grid reductions (fixed order -> bitwise reproducible dot products);
//   * the kernel "tail": what the last CTA of a kernel does once the grid's partial dots are combined --
//     the cross-GPU all-reduce over peer memory (post / wait split-phase, summed in rank order so every
//     rank gets bitwise identical scalars), the scalar recurrences of solver.c (alpha, beta, omega, the
//     loop test), and the halo-ready signal to the peers.  This is the device-side replacement of the
//     reference's MPI_Iallreduce / MPI_Wait pairs and host-side scalar code (solver.c:89-126, 227-258,
//     363-397).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bicg {

constexpr int MAX_RANKS  = 8;     // one NVSwitch box
constexpr int MAX_DOTS   = 8;     // dot products one kernel can reduce
constexpr int MAIL_VALS  = 8;

// ------------------------------------------------------------------------------------------------
// device-resident solver state (one per matrix arena)
// ------------------------------------------------------------------------------------------------
struct Scalars {
    // reference scalars, same names as solver.c:55-56, 182-183
    double rTr, rTr_old, rTs, rTy, yTy, rTw, wTw, rTz, dot_r, dot_zero, alpha, beta, omega;
    double tol2;                 // tol * tol                                (solver.c:86)
    double pend[MAX_DOTS];       // locally reduced values waiting for a later cross-GPU reduction
    int    k, max_iter;          // iteration counter / MAX_ITER             (solver.c:4, 120)
    int    done;                 // loop test failed -> every later kernel of the batch returns at once
    int    converged;
    int    error;                // 1: peer wait timed out
    unsigned int ticket;         // last-CTA election
    unsigned int red_epoch;      // sequence number of cross-GPU reductions posted by this rank
    unsigned int red_done;       // ... completed by this rank
    unsigned int halo_epoch;     // sequence number of halo pushes issued by this rank
    unsigned int pad_;
};

// one mailbox = what rank `src` contributes to one reduction: MAIL_VALS doubles, each as TWO self-validating 8-byte
// words {flag32 | data32} (NCCL's LL protocol): an aligned 8-byte store is single-copy atomic, so a word whose flag
// equals the expected epoch carries valid data -- no fence between "flag" and data, and nothing depends on a 16-byte
// vector store arriving un-torn over NVLink.  128 B so that no two mailboxes share a line.
struct alignas(128) Mailbox { unsigned long long w[2 * MAIL_VALS]; };
struct alignas(128) HaloFlag { unsigned long long epoch; unsigned long long pad_[15]; };

// peer-memory view of the job, passed by value to every kernel
struct CommDev {
    int rank, world;
    Mailbox  *mail[MAX_RANKS];   // mail[p] = base of rank p's mailbox array [2 parities][MAX_RANKS sources]
    HaloFlag *hflag[MAX_RANKS];  // hflag[p] = base of rank p's halo flags [MAX_RANKS sources]
    unsigned send_mask;          // peers this rank pushes halo data to
    unsigned recv_mask;          // peers this rank receives halo data from
    unsigned long long timeout_ns;   // bound of every device-side wait for a peer / another CTA (BICG_PEER_TIMEOUT_S)
};

// finalize ids: which scalar recurrence the tail evaluates once the reduced values are known
enum Fin : int {
    FIN_NONE = 0,
    FIN_BICG_INIT,     // tot0=(r,r)                                   solver.c:78-83
    FIN_BICG_ALPHA,    // tot0=(r#,s)            -> alpha              solver.c:89-93
    FIN_BICG_OMEGA,    // tot0=(q,y) tot1=(y,y)  -> omega              solver.c:97-104
    FIN_BICG_BETA,     // tot0=(r,r) tot1=(r#,r) -> beta, k++, test    solver.c:108-120
    FIN_STORE_RTR,     // tot0=(r,r) -> rTr                            solver.c:203
    FIN_CAPIPE_INIT,   // tot0=(r,w) -> alpha, beta=0, omega=0, test   solver.c:206-213
    FIN_OMEGA2,        // tot0=(q,y) tot1=(y,y) -> omega               solver.c:227-232 / 363-369
    FIN_CAPIPE_END,    // tot0..3=(r#,r),(r#,w),(r#,s),(r#,z) tot4=(r,r) -> beta, alpha, k++, test   solver.c:240-253
    FIN_STORE_PEND,    // reduced values -> Scalars::pend[] (the shifted solver's own scalar kernels take it from there)
};

// what the tail does with the locally reduced dots
enum TailOp : int {
    TAIL_NONE = 0,
    TAIL_PEND,         // keep them in Scalars::pend[pend_off ...] for a later kernel (no communication)
    TAIL_ALLREDUCE,    // [pend values +] local dots -> post + wait -> finalize          (blocking sync point)
    TAIL_POST,         // [pend values +] local dots -> post only                        (MPI_Iallreduce)
    TAIL_COMPLETE,     // wait for the reduction posted earlier -> finalize              (MPI_Wait)
};

struct TailDesc {
    int op;            // TailOp
    int fin;           // Fin
    int ndot;          // local dots produced by this kernel
    int npend;         // values taken from Scalars::pend and appended after the local dots (ALLREDUCE/POST)
    int pend_off;      // TAIL_PEND: where to store
    int nred;          // TAIL_COMPLETE: number of values of the pending reduction
    int signal_halo;   // 1: this kernel pushed halo data; tell the receivers
};

struct KernelCommon {
    Scalars *sc;
    double  *partials;     // [gridDim.x][MAX_DOTS]
    double  *hist;         // hist[k] = dot_r / dot_zero
    CommDev  comm;
    TailDesc tail;
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity)
{
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    while (!mbar_try_wait(bar, parity)) { }
}
// L2 policy of one access: Plain = no hint; Hint = the access carries a createpolicy value (l2_evict_first_policy), e.g.
// evict-first for the matrix stream or for a vector whose next use is too far away for L2 to keep it (mega.cu: run_bicgstab)
struct Plain {};
struct Hint { unsigned long long pol; };

// 1-D TMA bulk copy global -> shared, completion counted in bytes on an mbarrier, optionally with an L2 policy.
// 16-byte aligned addresses and a multiple-of-16 size are required.
__device__ __forceinline__ void tma_load_1d(unsigned dst_smem, const void *src, unsigned bytes, unsigned bar, Plain = {})
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_1d(unsigned dst_smem, const void *src, unsigned bytes, unsigned bar, Hint h)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(h.pol) : "memory");
}

__device__ __forceinline__ void mbar_arrive(unsigned bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// named CTA barrier over the first `nthreads` threads: the producer warp of a warp-specialised kernel free-runs
__device__ __forceinline__ void nbar(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// ---- LL words: {flag32 | data32}; a double travels as two of them ------------------------------------------
__device__ __forceinline__ unsigned long long ll_pack(unsigned data, unsigned flag)
{
    return ((unsigned long long)flag << 32) | (unsigned long long)data;
}
__device__ __forceinline__ void ll_encode(double v, unsigned flag, unsigned long long &w0, unsigned long long &w1)
{
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    w0 = ll_pack((unsigned)b, flag);
    w1 = ll_pack((unsigned)(b >> 32), flag);
}
__device__ __forceinline__ bool ll_valid(unsigned long long w0, unsigned long long w1, unsigned flag)
{
    return (unsigned)(w0 >> 32) == flag && (unsigned)(w1 >> 32) == flag;
}
__device__ __forceinline__ double ll_decode(unsigned long long w0, unsigned long long w1)
{
    return __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
}
// both words of one value with one 16-byte access; each word validates itself, so tearing is harmless
__device__ __forceinline__ void st_ll_sys(unsigned long long *p, unsigned long long w0, unsigned long long w1)
{
    asm volatile("st.relaxed.sys.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"(w0), "l"(w1) : "memory");
}
__device__ __forceinline__ void ld_ll_sys(const unsigned long long *p, unsigned long long &w0, unsigned long long &w1)
{
    asm volatile("ld.relaxed.sys.global.v2.b64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_ll_gpu(unsigned long long *p, unsigned long long w)
{
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_ll_gpu(const unsigned long long *p)
{
    unsigned long long w;
    asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    return w;
}
__device__ __forceinline__ void ld_ll_gpu2(const unsigned long long *p, unsigned long long &w0, unsigned long long &w1)
{
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
}
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
// plain ld.global: L1-cached but never the non-coherent (.nc) path -- for vectors that other SMs / peer GPUs rewrite
// while the kernel is running (visibility comes from the acquire fence that follows the flag wait)
__device__ __forceinline__ double ld_coherent(const double *p)
{
    double v;
    asm volatile("ld.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}
// ---- L2 eviction priority of one access: ld / st .L2::cache_hint carrying a createpolicy value ------------------------
// L1 behaves as for a plain ld.global / st.global; like ld_coherent, the loads never take the non-coherent path.
__device__ __forceinline__ unsigned long long l2_evict_first_policy()
{
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ double ld_hint(const double *p, unsigned long long pol)
{
    double v;
    asm volatile("ld.global.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ double2 ld_hint2(const double *p, unsigned long long pol)
{
    double2 v;
    asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_hint(double *p, double v, unsigned long long pol)
{
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol));
}
__device__ __forceinline__ void st_hint2(double *p, double2 v, unsigned long long pol)
{
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(pol));
}
__device__ __forceinline__ unsigned long long globaltimer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ------------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// sum over the LANES consecutive threads that share one row (butterfly: every one of them gets the sum)
template <int LANES>
__device__ __forceinline__ double lanes_sum(double v)
{
#pragma unroll
    for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------
// the merged layout of a handle's rows (matrix.cu) against the diag / offd blocks it was created from
// ------------------------------------------------------------------------------------------------
// Where row i's entries land in the merged CSR: its diag entries first, then its offd entries (the reference's accumulation
// order, matrix.c:437-440), so diag entry j is merged entry optr[i] + j and offd entry j is merged entry dptr[i + 1] + j.
// diag(k, j): diag entry j is merged entry k; offd(k, j) likewise.  The merge of matrix_create, every value update and the
// value gradient (value_grad.cu) place entries through this one function.  first / step: visit only the entries first,
// first + step, ... of each block of the row (a group of step lanes sharing the row).
template <class Diag, class Offd>
__device__ __forceinline__ void merge_row(int i, const unsigned *__restrict__ dptr, const unsigned *__restrict__ optr, Diag diag,
                                          Offd offd, unsigned first = 0, unsigned step = 1)
{
    const unsigned d0 = dptr[i], d1 = dptr[i + 1], o0 = optr[i], o1 = optr[i + 1];
    for (unsigned j = d0 + first; j < d1; j += step) diag(o0 + j, j);
    for (unsigned j = o0 + first; j < o1; j += step) offd(d1 + j, j);
}

// ------------------------------------------------------------------------------------------------
// TMA-fed CSR SpMV: what the stand-alone spmv_ws_kernel (spmv.cu) and the persistent kernel (mega.cu) share
// ------------------------------------------------------------------------------------------------
constexpr int PROW_PAD = 8;       // extra ptr / epilogue slots per stage for the 16-byte alignment window

// Shared memory one CTA may opt into on sm_90, static and dynamic together (227 KB of the SM's 228 KB).
constexpr int SMEM_OPTIN_BYTES = 227 * 1024;
// What the TMA tile planner (matrix.cu: build_tma_plan) shares out among the CTAs it places on one SM, 4 KB under the SM's
// 228 KB; the planner takes a further 1536 B off each CTA's share before it sizes the CTA's stages.
constexpr long long TMA_PLAN_SMEM_BYTES = 224 * 1024;
// What the persistent kernel's planner (matrix.cu: build_mega_plan) gives its one CTA per SM, stages or resident slice:
// beside the 3.4 KB of the kernel's static shared memory it stays under SMEM_OPTIN_BYTES.
constexpr long long MEGA_PLAN_SMEM_BYTES = 222 * 1024;
// opt a kernel into the most dynamic shared memory its static shared memory leaves
template <class Kernel>
cudaError_t smem_optin(Kernel k)
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, k);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN_BYTES - (int)fa.sharedSizeBytes);
}

// One stage of a tile of rpt rows and up to cap entries, in byte offsets from the stage's start:
//   [values: cap x 8 B][nepi epilogue slices: prow x 8 B each][columns: cap x 4 B][row pointers: prow x 4 B],  prow = rpt + PROW_PAD.
// Packed values fill the value area as three planes (4-, 2- and 1-byte) at 0, vmid() and vhi(); 16-bit column codes fill
// the first half of the column area.  A stage keeps this size whatever format it holds.
constexpr int SPMV_ENTRY_BYTES = 12;   // value + column of one staged entry
__host__ __device__ constexpr size_t spmv_stage_bytes(int cap, int rpt, int nepi)
{
    return (size_t)cap * SPMV_ENTRY_BYTES + (size_t)(rpt + PROW_PAD) * (size_t)(4 + 8 * nepi);
}
struct StageLayout {
    int cap, prow, nepi;
    __host__ __device__ constexpr StageLayout(int cap_, int rpt, int nepi_) : cap(cap_), prow(rpt + PROW_PAD), nepi(nepi_) {}
    __host__ __device__ constexpr size_t bytes() const { return spmv_stage_bytes(cap, prow - PROW_PAD, nepi); }
    // the areas of the stage that starts at st
    __device__ __forceinline__ const double *vals(const unsigned char *st) const { return reinterpret_cast<const double *>(st); }
    __host__ __device__ constexpr size_t vmid_off() const { return (size_t)cap * 4u; }
    __host__ __device__ constexpr size_t vhi_off() const { return (size_t)cap * 6u; }
    __device__ __forceinline__ const unsigned char *vmid(const unsigned char *st) const { return st + vmid_off(); }
    __device__ __forceinline__ const unsigned char *vhi(const unsigned char *st) const { return st + vhi_off(); }
    __device__ __forceinline__ const double *epi(const unsigned char *st, int v = 0) const { return vals(st) + cap + v * prow; }
    __device__ __forceinline__ const unsigned *cols(const unsigned char *st) const { return reinterpret_cast<const unsigned *>(epi(st, nepi)); }
    __device__ __forceinline__ const unsigned short *codes(const unsigned char *st) const { return reinterpret_cast<const unsigned short *>(cols(st)); }
    __device__ __forceinline__ const unsigned *ptrs(const unsigned char *st) const { return cols(st) + cap; }
};

// The part of the arrays that one tile of rows [row0, row1) with entries [p0, p1) puts into a stage: entries
// [a0, a0 + cnt) and row pointers [rowa, rowa + cntp), widened to whole 16-byte units for the bulk copies.  `al` is the
// alignment mask of the entry window (TileFormat::align).
struct TileWindow { unsigned a0, cnt; int rowa, cntp; };
__device__ __forceinline__ TileWindow tile_window(int row0, int row1, unsigned p0, unsigned p1, unsigned al)
{
    TileWindow w;
    w.a0 = p0 & ~al;
    w.cnt = ((p1 + al) & ~al) - w.a0;
    w.rowa = row0 & ~3;
    w.cntp = ((row1 + 1 + 3) & ~3) - w.rowa;
    return w;
}

// What the producer put into a stage: rows [row0, row1), entries from a0 and row pointers from rowa (the TileWindow).  The
// persistent kernel's stages also carry the tile's entries [lo, hi) relative to a0 and its chunk flag (MegaArgs::tile_flag);
// the tile kernel's stages, which never hold chunk tiles, keep the 16-byte header.
struct StageHdr { int row0, row1; unsigned a0; int rowa; };
struct ChunkStageHdr : StageHdr { unsigned lo, hi; int flag; int pad_; };

// The ring of up to 4 stages, in shared memory: a "full" mbarrier per stage that the producer's bulk copies complete, an
// "empty" one on which every consumer warp arrives once it is done with the stage, and the stage headers (Hdr: StageHdr
// or ChunkStageHdr).  Visit v of the
// ring uses stage v % stages; its parity is that of v / stages.  Visits are counted in int or unsigned (I), as the caller
// counts them.
template <class Hdr>
struct StageRing {
    unsigned long long full[4], empty[4];
    Hdr hdr[4];

    // thread 0, before a CTA barrier
    __device__ __forceinline__ void init(int stages, unsigned consumer_warps)
    {
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&full[s]), 1u);
            mbar_init(smem_u32(&empty[s]), consumer_warps);
        }
        mbar_fence_init();
    }
    __device__ __forceinline__ unsigned full_bar(int s) { return smem_u32(&full[s]); }
    // producer: the stage of visit v, once the consumers have released it (from the second lap on); -1 as soon as stop()
    // is true, while waiting or after
    template <class I, class Stop>
    __device__ __forceinline__ int acquire(I v, I stages, Stop stop)
    {
        const int s = (int)(v % stages);
        if (v >= stages) {
            const unsigned par = (unsigned)(v / stages - 1) & 1u;
            while (!mbar_try_wait(smem_u32(&empty[s]), par))
                if (stop()) return -1;
        }
        return stop() ? -1 : s;
    }
    template <class I>
    __device__ __forceinline__ int acquire(I v, I stages) { return acquire(v, stages, [] { return false; }); }
    // consumer: the stage of visit v, once its bulk copies have landed
    template <class I>
    __device__ __forceinline__ int wait(I v, I stages)
    {
        const int s = (int)(v % stages);
        mbar_wait(smem_u32(&full[s]), (unsigned)(v / stages) & 1u);
        return s;
    }
    // consumer: every thread of the warp is done with stage s
    __device__ __forceinline__ void release(int s)
    {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(smem_u32(&empty[s]));
    }
};

// How a tile is streamed into its stage: 8-byte values or the three planes of packed values, 32-bit columns or 16-bit
// codes, nepi epilogue slices, and the L2 policy of the value and column copies (Plain or Hint).
template <class H = Plain>
struct TileFormat {
    bool packed, coded;
    int nepi;
    H pol;
    // a bulk copy moves whole 16-byte units: the entry window is aligned to 4 entries for 4-byte columns, 8 for 2-byte
    // codes and 16 for the 1-byte plane of packed values
    __device__ __forceinline__ unsigned align() const { return packed ? 15u : (coded ? 7u : 3u); }
    __device__ __forceinline__ unsigned col_bytes() const { return coded ? 2u : 4u; }
    __device__ __forceinline__ unsigned val_bytes() const { return packed ? 7u : 8u; }
};
// The arrays a tile is copied from: val is the 8-byte values or the low plane of packed values, col the 32-bit columns
// or the 16-bit codes.
struct TileSrc {
    const void *val;
    const unsigned short *vmid;
    const unsigned char *vhi;
    const void *col;
    const unsigned *ptr;
};
struct NoEpi { __device__ const double *operator()(int) const { return nullptr; } };
// Producer: the bulk copies of window w into stage st (layout L) and the byte count they complete on its full barrier.
// epi(v): epilogue vector v, v < f.nepi, whose rows [w.rowa, w.rowa + w.cntp) go to slice v.
template <class H, class Epi = NoEpi>
__device__ __forceinline__ void tile_issue(const unsigned char *st, const StageLayout &L, unsigned bar, const TileFormat<H> &f,
                                           const TileWindow &w, const TileSrc &src, Epi epi = {})
{
    mbar_arrive_expect_tx(bar, w.cnt * (f.val_bytes() + f.col_bytes()) + (unsigned)w.cntp * 4u + (unsigned)(f.nepi * w.cntp) * 8u);
    if (w.cnt) {
        if (f.packed) {
            tma_load_1d(smem_u32(st), (const unsigned *)src.val + w.a0, w.cnt * 4u, bar, f.pol);
            tma_load_1d(smem_u32(L.vmid(st)), src.vmid + w.a0, w.cnt * 2u, bar, f.pol);
            tma_load_1d(smem_u32(L.vhi(st)), src.vhi + w.a0, w.cnt, bar, f.pol);
        } else {
            tma_load_1d(smem_u32(L.vals(st)), (const double *)src.val + w.a0, w.cnt * 8u, bar, f.pol);
        }
        tma_load_1d(smem_u32(L.cols(st)), (const char *)src.col + (size_t)w.a0 * f.col_bytes(), w.cnt * f.col_bytes(), bar, f.pol);
    }
    tma_load_1d(smem_u32(L.ptrs(st)), src.ptr + w.rowa, (unsigned)w.cntp * 4u, bar);
    for (int v = 0; v < f.nepi; ++v)
        tma_load_1d(smem_u32(L.epi(st, v)), epi(v) + w.rowa, (unsigned)w.cntp * 8u, bar);
}

// One row's product with NV vectors x[v] over the staged entries [j, e) (j already includes the thread's offset in its
// group of LANES), summed over the group into acc[v].  This loop decides the bits of y: per vector, entries in storage
// order, one fma each, then lanes_sum.  Entry idx is read once for all NV gathers x[v][col], so UNR * NV gathers are in
// flight per thread; UNR only decides how many entries one pass loads, so acc[v] does not depend on UNR or NV.
// `column(idx)` and `value(idx)` return the column and the value of staged entry idx (a value may come as an object that
// converts to double: it is converted where it is multiplied).
template <int LANES, int UNR, int NV, class Value, class Column>
__device__ __forceinline__ void row_product(Value value, Column column, const double *const (&x)[NV], int j, int e,
                                            double (&acc)[NV])
{
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = 0.0;
    while (j < e) {
        unsigned c[UNR];
        decltype(value(0)) a[UNR];
        double xv[NV][UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            // clamp instead of predicating: unconditional loads batch freely (a predicated load per slot runs out
            // of predicate registers after 7); the FMA below is what is predicated
            const int idx = min(j + u * LANES, e - 1);
            c[u] = column(idx);
            a[u] = value(idx);
        }
#pragma unroll
        for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int u = 0; u < UNR; ++u) xv[v][u] = ld_coherent(x[v] + c[u]);
#pragma unroll
        for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (j + u * LANES < e) acc[v] = fma((double)a[u], xv[v][u], acc[v]);
        j += UNR * LANES;
    }
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = lanes_sum<LANES>(acc[v]);
}

// Sum N per-thread values over the CTA.  Result is valid in every lane of warp 0.  `scratch` holds
// 32 * N doubles.  Fixed combination order -> deterministic.
template <int N>
__device__ __forceinline__ void block_sum(double (&v)[N], double *scratch)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = warp_sum(v[k]);
    __syncthreads();                     // scratch may still be in use by a previous call
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) scratch[warp * N + k] = v[k];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            double t = (lane < nwarps) ? scratch[lane * N + k] : 0.0;
            v[k] = warp_sum(t);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// cross-GPU reduction over peer mailboxes (called by warp 0 of the last CTA, all 32 lanes)
// ------------------------------------------------------------------------------------------------
// post: lane p stores this rank's `nv` values (at least one, so a pure barrier works too) into rank p's
// mailbox[parity][me] as LL words carrying the epoch.
__device__ __forceinline__ void xg_post(const CommDev &c, unsigned epoch, const double *vals, int nv)
{
    const int lane = threadIdx.x & 31;
    if (lane < c.world) {
        Mailbox *mb = c.mail[lane] + (epoch & 1u) * MAX_RANKS + c.rank;
        const int n = nv > 0 ? nv : 1;
        for (int k = 0; k < n; ++k) {
            unsigned long long w0, w1;
            ll_encode(nv > 0 ? vals[k] : 0.0, epoch, w0, w1);
            st_ll_sys(&mb->w[2 * k], w0, w1);
        }
    }
    __syncwarp();
}
// wait: lane p polls the words rank p sent to this rank until they carry `epoch`, keeps rank p's values; lane k
// then adds value k over ranks 0..world-1 in rank order (the same order on every rank -> bitwise identical
// results everywhere).  Returns false on timeout.
__device__ __forceinline__ bool xg_wait_sum(const CommDev &c, unsigned epoch, double *vals, int nv)
{
    __shared__ double s_contrib[MAX_RANKS][MAIL_VALS];
    const int lane = threadIdx.x & 31;
    const Mailbox *mine = c.mail[c.rank] + (epoch & 1u) * MAX_RANKS;
    bool ok = true;
    if (lane < c.world) {
        const unsigned long long t0 = globaltimer_ns();
        const int n = nv > 0 ? nv : 1;
        for (int k = 0; k < n && ok; ++k) {
            unsigned long long w0, w1;
            for (;;) {
                ld_ll_sys(&mine[lane].w[2 * k], w0, w1);
                if (ll_valid(w0, w1, epoch)) break;
                if (globaltimer_ns() - t0 > c.timeout_ns) { ok = false; break; }
            }
            s_contrib[lane][k] = ll_decode(w0, w1);
        }
    }
    ok = __all_sync(0xffffffffu, ok);
    __syncwarp();
    if (ok && lane < nv) {
        double acc = s_contrib[0][lane];
        for (int p = 1; p < c.world; ++p) acc += s_contrib[p][lane];
        vals[lane] = acc;
    }
    __syncwarp();
    return ok;
}

// ------------------------------------------------------------------------------------------------
// scalar recurrences -- one thread, same operation order as the reference
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void loop_test(Scalars *s)
{
    // solver.c:86  while (dot_r > tol * tol * dot_zero && k < max_iter)
    const bool go = (s->dot_r > s->tol2 * s->dot_zero) && (s->k < s->max_iter);
    if (!go) {
        s->done = 1;
        s->converged = !(s->dot_r > s->tol2 * s->dot_zero);
    }
}

// hist == nullptr: the caller keeps a private copy of the scalars and somebody else records the history
__device__ __forceinline__ void finalize(int fin, Scalars *s, double *hist, const double *t)
{
    double hdummy;
#define BICG_HIST(i) (*(hist ? &hist[i] : &hdummy))
    switch (fin) {
    case FIN_BICG_INIT:
        s->rTr = t[0]; s->dot_r = t[0]; s->dot_zero = t[0]; s->k = 0;         // solver.c:78-83
        BICG_HIST(0) = s->dot_r / s->dot_zero;
        loop_test(s);
        break;
    case FIN_BICG_ALPHA:
        s->rTs = t[0];
        s->alpha = s->rTr / s->rTs;                                           // solver.c:93
        break;
    case FIN_BICG_OMEGA:
        s->rTy = t[0]; s->yTy = t[1];
        s->omega = s->rTy / s->yTy;                                           // solver.c:104
        break;
    case FIN_BICG_BETA:
        s->dot_r = t[0];
        s->rTr_old = s->rTr;                                                  // solver.c:110
        s->rTr = t[1];
        s->beta = (s->alpha / s->omega) * (s->rTr / s->rTr_old);              // solver.c:116
        s->k += 1;
        BICG_HIST(s->k) = s->dot_r / s->dot_zero;
        loop_test(s);
        break;
    case FIN_STORE_RTR:
        s->rTr = t[0];
        break;
    case FIN_CAPIPE_INIT:
        s->rTw = t[0];
        s->alpha = s->rTr / s->rTw;                                           // solver.c:210
        s->beta = 0.0; s->omega = 0.0;                                        // :211 (omega pinned, SURVEY 5)
        s->dot_r = s->rTr; s->dot_zero = s->rTr; s->k = 0;                    // :212-213
        BICG_HIST(0) = s->dot_r / s->dot_zero;
        loop_test(s);
        break;
    case FIN_OMEGA2:
        s->rTw = t[0]; s->wTw = t[1];
        s->omega = s->rTw / s->wTw;                                           // solver.c:232 / 369
        break;
    case FIN_CAPIPE_END:
        s->rTr_old = s->rTr;                                                  // solver.c:239
        s->rTr = t[0]; s->rTw = t[1]; s->rTs = t[2]; s->rTz = t[3];
        s->dot_r = t[4];
        s->beta = (s->alpha / s->omega) * (s->rTr / s->rTr_old);              // :248
        s->alpha = s->rTr / (s->rTw + s->beta * (s->rTs - s->omega * s->rTz)); // :249
        s->k += 1;
        BICG_HIST(s->k) = s->dot_r / s->dot_zero;
        loop_test(s);
        break;
    case FIN_STORE_PEND:
        for (int k = 0; k < MAX_DOTS; ++k) s->pend[k] = t[k];
        break;
    default: break;
    }
#undef BICG_HIST
}

// Wait until every peer in recv_mask has published halo epoch >= `expect` (called by warp 0 of a CTA).
__device__ __forceinline__ bool halo_wait_epoch(const CommDev &c, unsigned expect)
{
    const int lane = threadIdx.x & 31;
    bool ok = true;
    if (lane < c.world && ((c.recv_mask >> lane) & 1u)) {
        const unsigned long long *f = &c.hflag[c.rank][lane].epoch;
        const unsigned long long t0 = globaltimer_ns();
        while (ld_acquire_sys(f) < (unsigned long long)expect) {
            if (globaltimer_ns() - t0 > c.timeout_ns) { ok = false; break; }
        }
    }
    return __all_sync(0xffffffffu, ok);
}

// What the elected warp does once the grid's dots are combined: `tot` holds the totals in every lane.
// Runs the TailDesc: cross-GPU reduction over the peer mailboxes, scalar recurrence, halo-ready signal to the peers.
template <int NDOT>
__device__ __forceinline__ void tail_warp(const KernelCommon &kc, double (&tot)[NDOT > 0 ? NDOT : 1])
{
    Scalars *sc = kc.sc;
    const int tid = threadIdx.x & 31;
    __shared__ double s_vals[MAIL_VALS];
    const TailDesc &td = kc.tail;
    const int lane = tid;
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < NDOT; ++k) s_vals[k] = tot[k];
        if (td.op == TAIL_ALLREDUCE || td.op == TAIL_POST)
            for (int k = 0; k < td.npend; ++k) s_vals[td.ndot + k] = sc->pend[k];
    }
    __syncwarp();

    bool ok = true;
    switch (td.op) {
    case TAIL_PEND:
        if (lane == 0) for (int k = 0; k < td.ndot; ++k) sc->pend[td.pend_off + k] = s_vals[k];
        break;
    case TAIL_ALLREDUCE: {
        const int nv = td.ndot + td.npend;
        unsigned ep = sc->red_epoch + 1u;
        xg_post(kc.comm, ep, s_vals, nv);
        ok = xg_wait_sum(kc.comm, ep, s_vals, nv);
        __syncwarp();
        if (lane == 0) { sc->red_epoch = ep; sc->red_done = ep; }
        break;
    }
    case TAIL_POST: {
        const int nv = td.ndot + td.npend;
        unsigned ep = sc->red_epoch + 1u;
        xg_post(kc.comm, ep, s_vals, nv);
        if (lane == 0) sc->red_epoch = ep;
        break;
    }
    case TAIL_COMPLETE: {
        unsigned ep = sc->red_done + 1u;
        ok = xg_wait_sum(kc.comm, ep, s_vals, td.nred);
        __syncwarp();
        if (lane == 0) sc->red_done = ep;
        break;
    }
    default: break;
    }

    if (lane == 0) {
        if (!ok) { sc->error = 1; sc->done = 1; }
        else if (td.fin != FIN_NONE) finalize(td.fin, sc, kc.hist, s_vals);
    }
    if (td.signal_halo) {
        // all CTAs fenced their peer stores before taking a ticket; publish the new epoch to receivers
        const unsigned he = sc->halo_epoch + 1u;
        // every CTA that pushed fenced at system scope BEFORE its ticket, and this warp observed all tickets; the
        // flag itself is a system-scope RELEASE store so the pattern is a proper release chain at system scope
        // (one warp per kernel pays for it)
        if (lane < kc.comm.world && ((kc.comm.send_mask >> lane) & 1u))
            st_release_sys(&kc.comm.hflag[lane][kc.comm.rank].epoch, (unsigned long long)he);
        __syncwarp();
        if (lane == 0) sc->halo_epoch = he;
    }
}


// ------------------------------------------------------------------------------------------------
// kernel tail: elect the last CTA, combine the grid's partial dots in a fixed order, run the TailDesc
// ------------------------------------------------------------------------------------------------
// `local` holds this CTA's dots (valid in warp 0 after block_sum).  `scratch`: >= 32*MAX_DOTS doubles.
// Every thread of the CTA must call this.  All global writes of the CTA that the tail's signals cover
// (halo pushes) are ordered by the CTA barrier + thread 0's system-scope fence at the top of this function.
template <int NDOT>
__device__ __forceinline__ void kernel_tail(const KernelCommon &kc, double (&local)[NDOT > 0 ? NDOT : 1],
                                            double *scratch)
{
    __shared__ int s_last;
    Scalars *sc = kc.sc;
    const int tid = threadIdx.x;
    __syncthreads();                     // every thread's global / peer stores of this CTA happen-before the fence
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < NDOT; ++k) __stcg(&kc.partials[(size_t)blockIdx.x * MAX_DOTS + k], local[k]);
        if (kc.tail.signal_halo) __threadfence_system();   // peer (NVLink) stores of the halo push
        else __threadfence();
        const unsigned t = atomicAdd(&sc->ticket, 1u);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();

    // grid-level combination: thread t sums CTAs t, t+T, ... ascending, then a fixed CTA tree
    double tot[NDOT > 0 ? NDOT : 1];
#pragma unroll
    for (int k = 0; k < (NDOT > 0 ? NDOT : 1); ++k) tot[k] = 0.0;
    if (NDOT > 0) {
        for (unsigned b = tid; b < gridDim.x; b += blockDim.x) {
#pragma unroll
            for (int k = 0; k < NDOT; ++k) tot[k] += __ldcg(&kc.partials[(size_t)b * MAX_DOTS + k]);
        }
        block_sum<(NDOT > 0 ? NDOT : 1)>(tot, scratch);
    }
    if (tid >= 32) return;                       // warp 0 finishes the job
    tail_warp<NDOT>(kc, tot);
    if (tid == 0) { __threadfence(); sc->ticket = 0u; }
}

} // namespace bicg
