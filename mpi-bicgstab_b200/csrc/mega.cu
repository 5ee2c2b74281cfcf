// mega.cu -- one persistent, cooperative kernel per solve: the whole iteration loop of solver.c on the device.
//
// Why: with the matrix split over 8 GPUs an iteration is ~13 us of memory traffic; kernel boundaries, atomics and
// master/worker barriers cost several times that.  Here one CTA per SM stays resident for the entire solve and
//   * owns a fixed, contiguous, work-balanced range of rows (plan.cpp: plan_cta_tiles);
//   * runs the SpMV phases as the warp-specialised TMA pipeline of spmv.cu over its own tiles -- the producer warp
//     never stops: while the consumers are in a vector phase or wait at a synchronisation point it is already
//     streaming the first stages of the NEXT SpMV (the matrix never changes), with an L2 evict-first policy so that
//     the once-per-SpMV matrix stream does not push the (re-used) vectors out of the 50 MB L2;
//   * runs the vector phases (vec_body.cuh) on its own rows only, so nothing but the gathered x crosses SMs;
//   * keeps ITS OWN copy of the solver scalars (alpha, beta, omega, the dots, k, the loop test) in shared memory:
//     every CTA evaluates the recurrences of solver.c:93-120 itself from the same reduced values, in the same
//     order, so all CTAs (and all ranks) take bitwise identical decisions and nobody waits for a "master".
//
// Synchronisation (the replacement of MPI_Iallreduce/MPI_Wait and of the grid barriers of round 1):
//   arrive   : a CTA publishes its partial dots as self-validating LL words {generation | 32 data bits} in its own
//              128-byte slot of the generation's ring entry -- plain stores, no atomics (a release fence only where the
//              arrival also publishes rows that other CTAs gather next);
//   reduce   : (1 GPU) every CTA polls all slots of the generation (160 threads, one slot each) and adds them in a
//              fixed order; (N GPUs) only the middle CTA (the reducer) does that, posts the rank's sums into every rank's mailbox over
//              NVLink (LL words again), and every CTA of every rank polls its own GPU's 8 mailboxes and adds them in
//              rank order.  Critical path: one L2 round trip (+ one NVLink hop + one L2 round trip);
//   post / complete : the same, split (MPI_Iallreduce ... SpMV ... MPI_Wait of the pipelined variants);
//   neighbour wait  : where solver.c has no reduction but the next SpMV gathers what other CTAs just wrote (q, p,
//              s, ...), a CTA waits only for the CTAs that own the columns its rows reference (a handful for banded
//              matrices);
//   halo (N GPUs)   : boundary rows travel to the peers as LL words too (16 bytes per value, push_ll): no system-scope
//              fence, no flag -- the consumer polls exactly the ghost slots it needs.  In the BiCGStab loop the pushes
//              ride on the alpha / beta reductions and the ghost copies of q and p are advanced redundantly
//              (run_bicgstab_multi); the CA / pipelined loops unpack the LL words into the ghost tails (halo_ll, post).
// Coherence: gathered vectors are read with plain (L1-cached) loads; every neighbour wait ends in an acquire fence at gpu
// scope (SASS: MEMBAR + CCTL.IVALL), so rows rewritten by other SMs are re-fetched from L2; values from peers are taken
// from the LL words with system-scope loads and re-stored locally by the consuming CTA.
// Every wait is bounded (BICG_PEER_TIMEOUT_S, Mega::timed_out): a lost CTA or rank raises Scalars::error instead of hanging the GPU.
#include "mega.cuh"
#include "vec_body.cuh"

namespace bicg {

namespace {

constexpr int RED_THREADS = MEGA_MAX_CTAS;          // one polled slot per thread
constexpr int RED_WARPS = RED_THREADS / 32;

// Polling etiquette: the first probes go out back to back (the last arriver normally finds everything in place), after
// that the thread sleeps 64 .. 256 ns between probes -- 132 CTAs spinning flat out on the same 132 cache lines delay the
// very stores they are waiting for.
__device__ __forceinline__ void poll_pause(unsigned spins)
{
    if (spins > 2u) __nanosleep(spins > 16u ? 256u : (spins > 6u ? 128u : 64u));
}

// CTA-wide sum over the consumer threads only; result valid in every lane of warp 0
template <int N, int CT>
__device__ __forceinline__ void cblock_sum(double (&v)[N], double *scratch)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = CT / 32;
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = warp_sum(v[k]);
    nbar(1, CT);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) scratch[warp * N + k] = v[k];
    }
    nbar(1, CT);
    if (warp == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            double t = (lane < NW) ? scratch[lane * N + k] : 0.0;
            v[k] = warp_sum(t);
        }
    }
}

enum Epi : int { EPI_NONE = 0, EPI_RH_Y, EPI_QY_YY, EPI_CA4 };

struct MegaShared {
    Scalars sc;                               // this CTA's copy of the solver scalars
    double tot[MAIL_VALS];                    // reduced values of the current synchronisation point
    double red[RED_WARPS][MAIL_VALS];
    double contrib[MAX_RANKS][MAIL_VALS];
    double scratch[32 * MAX_DOTS];
    StageRing<ChunkStageHdr> ring;
    unsigned vadj[VAL_TABLE_MAX];            // the CTA's value table as PackedVal adds it (packed CTAs only)
    volatile int flags[4];                    // [1] producer stop, [2] consumed visits, [3] a wait timed out
};

// Column window of a CTA (mega_dep_kernel: the own columns [dep.x, dep.y] and the ghost slots [dep.z, dep.w] its rows
// reference).  When both spans together fit 16 bits, every column of the CTA has a 16-bit code: own column c -> c - obase
// (codes < ospan), ghost column c -> c - gbase (codes >= ospan).  The one place that decides this: the code kernel, the
// resident loader, the producer thread and the consumer threads all call it with the same dep, so a CTA's choice is the
// same everywhere.
struct ColWindow { bool ok; unsigned ospan; int obase, gbase; };
__device__ __forceinline__ ColWindow col_window(int4 dep, int ghost_off)
{
    ColWindow w;
    const bool own = dep.x <= dep.y, gh = dep.z <= dep.w;
    w.ospan = own ? (unsigned)(dep.y - dep.x + 1) : 0u;
    const unsigned gspan = gh ? (unsigned)(dep.w - dep.z + 1) : 0u;
    w.ok = w.ospan + gspan <= 65536u;
    w.obase = own ? dep.x : 0;
    w.gbase = ghost_off + (gh ? dep.z : 0) - (int)w.ospan;
    return w;
}
__device__ __forceinline__ unsigned short col_encode(const ColWindow &w, int ghost_off, unsigned c)
{
    return (unsigned short)((int)c < ghost_off ? (int)c - w.obase : (int)c - w.gbase);
}
__device__ __forceinline__ unsigned col_decode(const ColWindow &w, unsigned code)
{
    return code + (unsigned)(code < w.ospan ? w.obase : w.gbase);
}

// Resident mode (MegaArgs::resident; strong scaling, e.g. T' over 8 GPUs x 132 CTAs = 21 k entries per CTA): a CTA whose whole
// slice fits into its shared memory -- 8-byte values, the 16-bit column codes, row pointers -- loads it ONCE per solve; its
// SpMV phases then touch neither L2 nor the TMA ring for the matrix.  Decided per CTA, identically by the producer thread
// and by every consumer thread.
struct ResidentPlan { bool on; int row_lo, rows; unsigned nz_lo, nnz; ColWindow w; };
__device__ __forceinline__ ResidentPlan resident_plan(const MegaArgs &a, int t0, int t1, int lanes)
{
    ResidentPlan p;
    p.on = false; p.row_lo = 0; p.rows = 0; p.nz_lo = 0u; p.nnz = 0u;
    p.w = col_window(a.cta_dep[blockIdx.x], a.ghost_off);
    if (!a.resident || lanes != 1 || t1 <= t0 || a.tile_flag != nullptr) return p;
    p.row_lo = a.tile_row[t0];
    p.rows = a.tile_row[t1] - p.row_lo;
    if (p.rows <= 0) return p;
    p.nz_lo = a.ptr[p.row_lo];
    p.nnz = a.ptr[p.row_lo + p.rows] - p.nz_lo;
    if (mega_resident_bytes(p.nnz, p.rows) > (size_t)a.smem_bytes) return p;
    p.on = p.w.ok;                                      // columns that do not fit 16-bit codes: the CTA streams
    return p;
}
// a streaming CTA (not resident, owns tiles) streams the 16-bit codes instead of the 32-bit columns when its window fits
__device__ __forceinline__ bool streams_codes(const MegaArgs &a, const ResidentPlan &rp, int my_tiles)
{
    return a.stream_codes && a.col16 != nullptr && my_tiles > 0 && !rp.on && rp.w.ok;
}
// a CTA that streams codes and has a value table (mega_value_kernel) streams its values packed: 7 bytes instead of 8.
// Decided like streams_codes, by the producer thread and by every consumer thread from the same inputs.
__device__ __forceinline__ bool streams_values(const MegaArgs &a, bool coded)
{
    return coded && a.stream_values && a.vtab != nullptr && a.vtab[blockIdx.x].n > 0;
}
// A packed value is hi = table index << 4 | mantissa bits 51..48, mid = mantissa bits 47..32, lo = bits 31..0.
// adj[i] = (field i << 20) - (i << 20) (mod 2^32), so hi << 16 = i << 20 | (bits 51..48) << 16 plus adj[i] is the high word
// without bits 47..32, and mid fills those: the 64-bit pattern comes back exactly, with no floating-point operation.
__device__ __forceinline__ unsigned val_adj(const ValTable &t, int i)
{
    return i < t.n ? ((unsigned)t.field[i] << 20) - ((unsigned)i << 20) : 0u;
}
// As loaded from a stage, a packed value is hm = hi << 16 | mid and lo; it is put together where it is multiplied, after
// the gathers, so that it holds two registers while they are in flight, like an 8-byte value.  The planes and the table
// are read through 32-bit shared-memory addresses: one register per base instead of a 64-bit generic pointer, which is
// what keeps the 512-thread kernels within their register budget.
__device__ __forceinline__ unsigned lds_u32(unsigned p) { unsigned v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(p)); return v; }
__device__ __forceinline__ unsigned lds_u16(unsigned p) { unsigned v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(p)); return v; }
__device__ __forceinline__ unsigned lds_u8(unsigned p) { unsigned v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(p)); return v; }
struct PackedVal {
    unsigned hm, lo, adj;                         // adj: shared address of the table (MegaShared::vadj)
    __device__ __forceinline__ operator double() const
    {
        return __hiloint2double((int)(hm + lds_u32(adj + (hm >> 20) * 4u)), (int)lo);
    }
};
// entry idx of the planes of a stage that starts at shared address st (layout L)
__device__ __forceinline__ PackedVal val_load(unsigned adj, unsigned st, const StageLayout &L, unsigned idx)
{
    const unsigned lo = lds_u32(st + idx * 4u), mid = lds_u16(st + (unsigned)L.vmid_off() + idx * 2u), hi = lds_u8(st + (unsigned)L.vhi_off() + idx);
    return PackedVal{(hi << 16) | mid, lo, adj};
}

template <int CT, int LANES>
struct Mega {
    static constexpr int RPT = CT / LANES, NCW = CT / 32, UNR = (LANES == 1) ? 16 : 8;
    static_assert(CT >= RED_THREADS, "the slot reduction uses one thread per CTA slot");

    const MegaArgs &a;
    MegaShared &sh;
    unsigned char *dyn;
    int tid, lane, my_tiles, row_lo, row_hi;
    unsigned vis;                 // SpMV tile visits consumed so far (mirrors the producer's counter)
    unsigned gen;                 // arrival generation (same value in every CTA)
    unsigned red_epoch;           // cross-GPU reductions posted (same value on every rank)
    unsigned posted_gen;          // generation of the reduction posted and not yet completed
    unsigned long long halo_epoch;
    int dep_lo, dep_hi;           // CTAs owning the own columns this CTA's rows reference
    unsigned push_slots;          // push slots (peers) that need rows of this CTA
    int ghost_lo, ghost_hi;       // ghost slots this CTA's rows gather [lo, hi)
    int gs_lo, gs_hi;             // ghost slots this CTA keeps up to date itself (multi-GPU bicgstab: redundant recurrences)
    bool reads_ghost;             // this CTA's rows gather ghost columns
    bool is_reducer;              // N > 1: the CTA that adds up this GPU's slots and posts them to the peers' mailboxes
    size_t stage_bytes;
    int trace_it, trace_who;
    bool resident;                // this CTA keeps its matrix slice in shared memory (ResidentPlan)
    bool coded;                   // this CTA streams 16-bit column codes (streams_codes)
    bool packed;                  // this CTA streams 7-byte packed values (streams_values)
    ResidentPlan rp;
    const double *rs_val; const unsigned short *rs_col; const unsigned *rs_ptr;

    __device__ Mega(const MegaArgs &args, MegaShared &s) : a(args), sh(s) {}

    // the policy of run_bicgstab's evict-first accesses: made where a phase begins, not held in a register across the loop
    static __device__ __forceinline__ Hint evict_first() { return Hint{l2_evict_first_policy()}; }

    __device__ bool stop_now() const { return sh.sc.done != 0 || sh.sc.error != 0; }
    __device__ void fail() { sh.flags[3] = 1; }
    // the bound of every wait of this kernel: t0 = globaltimer_ns() when the wait began; the clock is read on every 256th
    // probe only, and a wait that sees true calls fail() and stops polling
    __device__ __forceinline__ bool timed_out(unsigned long long t0, unsigned spins) const
    {
        return (spins & 255u) == 0u && globaltimer_ns() - t0 > a.comm.timeout_ns;
    }
    // one iteration's alpha sync seen by EVERY CTA: [G][2] = arrival, release (globaltimer, per GPU)
    __device__ void snap(int which)
    {
        if (a.snap && tid == 0 && sh.sc.k == a.snap_iter) a.snap[2 * blockIdx.x + which] = globaltimer_ns();
    }
    __device__ void mark(int slot)
    {
        if (a.trace && trace_who >= 0 && tid == 0 && trace_it < MEGA_TRACE_ITERS)
            a.trace[((size_t)trace_who * MEGA_TRACE_ITERS + trace_it) * MEGA_TRACE_SLOTS + slot] = globaltimer_ns();
    }

    // ---------------------------------------------------------------- arrive ------------------------------
    // Publish NV partial sums (NV = 0: presence only) for generation ++gen.
    // release: the arrival also PUBLISHES this CTA's stores of the phase (rows that other CTAs gather after waiting for
    // it): CTA barrier + release fence before the words go out.  A pure reduction arrival does not need it: the reduced
    // values travel inside the words, nobody gathers this CTA's rows before its next releasing arrival (a neighbour wait
    // always precedes a gather), and its own earlier gathers completed before the dots that depend on them.
    template <int NV>
    __device__ void arrive(double (&dot)[NV > 0 ? NV : 1], bool release)
    {
        // a CTA barrier (inside cblock_sum, or the explicit one) puts every consumer's stores of the phase before the fence
        if (NV > 0) cblock_sum<(NV > 0 ? NV : 1), CT>(dot, sh.scratch);
        else nbar(1, CT);
        ++gen;
        if (tid < 32) {
            if (release) fence_gpu();
            MegaSlot *s = &a.sync->slot[gen & (MEGA_RING - 1)][blockIdx.x];
            constexpr int NW = NV > 0 ? 2 * NV : 1;
            if (lane < NW) {
                unsigned data = 0u;
                if (NV > 0) {
                    double v = dot[0];
#pragma unroll
                    for (int k = 1; k < NV; ++k) v = ((lane >> 1) == k) ? dot[k] : v;
                    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
                    data = (lane & 1) ? (unsigned)(b >> 32) : (unsigned)b;
                }
                st_ll_gpu(&s->w[lane], ll_pack(data, gen));
            }
        }
    }

    // ---------------------------------------------------------------- neighbour wait ----------------------
    // wait for the CTAs (of this GPU) that own the columns this CTA's rows gather
    __device__ void wait_nbr()
    {
        if (tid < 32) {
            bool ok = true;
            const unsigned long long t0 = globaltimer_ns();
            const MegaSlot *ring = a.sync->slot[gen & (MEGA_RING - 1)];
            for (int c = dep_lo + lane; c <= dep_hi; c += 32) {
                if (c == (int)blockIdx.x) continue;
                unsigned spins = 0;
                while ((unsigned)(ld_ll_gpu(&ring[c].w[0]) >> 32) != gen) {
                    poll_pause(++spins);
                    if (timed_out(t0, spins)) { ok = false; break; }
                }
            }
            fence_gpu();                                     // acquire (+ L1 invalidate): the gathers that follow see the data
            if (!__all_sync(0xffffffffu, ok) && lane == 0) fail();
        }
        nbar(1, CT);
        if (sh.flags[3]) { if (tid == 0) { sh.sc.error = 1; sh.sc.done = 1; } nbar(1, CT); }
    }
    __device__ void sync_nbr()
    {
        double d0[1] = {0.0};
        arrive<0>(d0, true);
        wait_nbr();
    }

    // ---------------------------------------------------------------- reductions --------------------------
    // All slots of generation g -> sh.tot (fixed order: thread c takes CTA c, butterfly inside each of the five
    // warps, then warp 0..4 left to right).  Called by every consumer thread; sh.tot is valid for tid 0 on return.
    template <int NV>
    __device__ void local_reduce(unsigned g)
    {
        if (tid < RED_THREADS) {
            double v[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) v[k] = 0.0;
            if (tid < (int)gridDim.x) {
                const unsigned long long *w = a.sync->slot[g & (MEGA_RING - 1)][tid].w;
                const unsigned long long t0 = globaltimer_ns();
                unsigned long long w0[NV], w1[NV];
                unsigned spins = 0;
                for (;;) {
                    bool all = true;
#pragma unroll
                    for (int k = 0; k < NV; ++k) { ld_ll_gpu2(w + 2 * k, w0[k], w1[k]); all = all && ll_valid(w0[k], w1[k], g); }
                    if (all) break;
                    ++spins;
                    if (a.comm.world == 1) poll_pause(spins);        // N > 1: only the reducer CTA polls the slots -- no crowd, no pause
                    if (timed_out(t0, spins)) { fail(); break; }
                }
#pragma unroll
                for (int k = 0; k < NV; ++k) v[k] = ll_decode(w0[k], w1[k]);
            }
#pragma unroll
            for (int k = 0; k < NV; ++k) v[k] = warp_sum(v[k]);
            if (lane == 0) {
#pragma unroll
                for (int k = 0; k < NV; ++k) sh.red[tid >> 5][k] = v[k];
            }
            nbar(2, RED_THREADS);
            if (tid == 0) {
#pragma unroll
                for (int k = 0; k < NV; ++k) {
                    double t = sh.red[0][k];
#pragma unroll
                    for (int wq = 1; wq < RED_WARPS; ++wq) t += sh.red[wq][k];
                    sh.tot[k] = t;
                }
            }
        }
    }
    // warp 0 of the reducer CTA: this rank's sums -> every rank's mailbox[parity][me]
    template <int NV>
    __device__ void post_mail()
    {
        __syncwarp();
        if (lane < a.comm.world) {
            MegaSlot *mb = a.peer_mail[0];
#pragma unroll
            for (int p = 1; p < MAX_RANKS; ++p) mb = (lane == p) ? a.peer_mail[p] : mb;
            mb += (size_t)(red_epoch & 1u) * MAX_RANKS + a.comm.rank;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                unsigned long long w0, w1;
                ll_encode(sh.tot[k], red_epoch, w0, w1);
                st_ll_sys(&mb->w[2 * k], w0, w1);
            }
        }
        __syncwarp();
    }
    // warp 0 of every CTA: the ranks' sums from this GPU's own mailboxes, added in rank order -> sh.tot
    template <int NV>
    __device__ void mail_reduce()
    {
        if (lane < a.comm.world) {
            const unsigned long long *w = a.sync->mail[red_epoch & 1u][lane].w;
            const unsigned long long t0 = globaltimer_ns();
            unsigned long long w0[NV], w1[NV];
            unsigned spins = 0;
            for (;;) {
                bool all = true;
#pragma unroll
                for (int k = 0; k < NV; ++k) { ld_ll_sys(w + 2 * k, w0[k], w1[k]); all = all && ll_valid(w0[k], w1[k], red_epoch); }
                if (all) break;
                if (++spins > 4u) __nanosleep(48);                   // 8 lines polled by 132 x 8 threads: a short pause is enough
                if (timed_out(t0, spins)) { fail(); break; }
            }
#pragma unroll
            for (int k = 0; k < NV; ++k) sh.contrib[lane][k] = ll_decode(w0[k], w1[k]);
        }
        __syncwarp();
        if (lane < NV) {
            double acc = sh.contrib[0][lane];
            for (int p = 1; p < a.comm.world; ++p) acc += sh.contrib[p][lane];
            sh.tot[lane] = acc;
        }
        __syncwarp();
    }
    // complete the reduction published at generation g and evaluate the scalar recurrence `fin` in this CTA's copy
    template <int NV>
    __device__ void finish(unsigned g, int fin, bool posted, bool tr = false)
    {
        if (a.comm.world == 1) { local_reduce<NV>(g); if (tr) mark(12); }
        else {
            if (is_reducer && !posted) { local_reduce<NV>(g); if (tr) mark(12); if (tid < 32) post_mail<NV>(); if (tr) mark(13); }
            if (tid < 32) mail_reduce<NV>();
            if (tr) mark(14);
        }
        if (tid == 0) {
            // no acquire fence here: a reduction is never directly followed by a gather of other CTAs' rows (a neighbour
            // wait with its own fence always sits in between), and the writes that follow are control-dependent on the
            // polls above
            if (sh.flags[3]) { sh.sc.error = 1; sh.sc.done = 1; }
            else finalize(fin, &sh.sc, blockIdx.x == 0 ? a.hist : nullptr, sh.tot);
        }
        nbar(1, CT);
    }
    // push_id >= 0: the boundary rows of that vector leave as LL words (push_ll) right AFTER this CTA's reduction words --
    // the consumers poll the LL words themselves, so the push need not delay the arrival; it overlaps with the reduction's
    // NVLink latency instead of preceding it
    template <int NV>
    __device__ void reduce(double (&dot)[NV], int fin, bool tr = false, int push_id = -1, int region = 0, unsigned epoch = 0u)
    {
        arrive<NV>(dot, false);
        if (tr) { mark(11); snap(0); }
        if (push_id >= 0) push_ll(push_id, region, epoch);
        if (a.comm.world > 1) ++red_epoch;
        finish<NV>(gen, fin, false, tr);
        if (tr) snap(1);
    }
    // MPI_Iallreduce + the halo of vector `id` that the SpMV hiding the reduction gathers (LL region `region`)
    template <int NV>
    __device__ void post(double (&dot)[NV], int id, int region)
    {
        const bool multi = a.comm.world > 1;
        const unsigned ep = multi ? (unsigned)(++halo_epoch) : 0u;
        arrive<NV>(dot, true);
        posted_gen = gen;
        if (multi) {
            ++red_epoch;
            if (is_reducer) { local_reduce<NV>(gen); if (tid < 32) post_mail<NV>(); }
            push_ll(id, region, ep);
        }
        wait_nbr();
        if (multi) unpack_ll(id, region, ep);
    }
    // MPI_Wait.  after_spmv: the SpMV that hid the reduction gathered a vector that the NEXT phase overwrites in place
    // (pipelined loops: y = w - alpha z is stored over w right after t = A w): the reduction was published BEFORE that
    // SpMV, so its completion says nothing about the other CTAs having finished their gathers.  A second, data-free
    // arrival after the SpMV, awaited from every CTA of this GPU (peers never gather own rows), closes the window.
    template <int NV>
    __device__ void complete(int fin, bool after_spmv)
    {
        if (after_spmv) {
            double d0[1] = {0.0};
            arrive<0>(d0, false);
            wait_all();
        }
        finish<NV>(posted_gen, fin, true);
    }
    // wait for every other CTA of this GPU to arrive at generation gen: thread c polls CTA c's slot
    __device__ __forceinline__ void wait_all()
    {
        if (tid < RED_THREADS && tid < (int)gridDim.x && tid != (int)blockIdx.x) {
            const unsigned long long *w = a.sync->slot[gen & (MEGA_RING - 1)][tid].w;
            const unsigned long long t0 = globaltimer_ns();
            unsigned spins = 0;
            while ((unsigned)(ld_ll_gpu(w) >> 32) != gen) {
                poll_pause(++spins);
                if (timed_out(t0, spins)) { fail(); break; }
            }
        }
    }

    // ---------------------------------------------------------------- SpMV over this CTA's tiles ----------
    // far: the L2 policy of the r# loads of EPI_RH_Y (run_bicgstab's table); every other access of the SpMV is plain
    template <int EPI, class F = Plain>
    __device__ void spmv(const double *x, double *y, double (&dot)[4], F far = {})
    {
        if constexpr (LANES == 1) {
            if (resident) { spmv_res<EPI>(x, y, dot, far); return; }
        }
        if (packed) spmv_impl<EPI, true, true>(x, y, dot, far);
        else if (coded) spmv_impl<EPI, true, false>(x, y, dot, far);
        else spmv_impl<EPI, false, false>(x, y, dot, far);
    }
    // one row's epilogue operands (EPI_RH_Y: r#; EPI_QY_YY: q, kept in v.r; EPI_CA4: r#, r, s, z), loaded before its gathers
    template <int EPI, class F>
    __device__ __forceinline__ void epi_load(int row, double &e0, double &e1, double &e2, double &e3, F far) const
    {
        if (EPI == EPI_RH_Y) e0 = ld1(a.v.rh + row, far);
        if (EPI == EPI_QY_YY) e0 = a.v.r[row];
        if (EPI == EPI_CA4) { e0 = a.v.rh[row]; e1 = a.v.r[row]; e2 = a.v.s[row]; e3 = a.v.z[row]; }
    }
    // one row's epilogue: y and the dots fused into the SpMV; every SpMV path of this kernel ends its rows here
    template <int EPI>
    __device__ __forceinline__ void row_done(int row, double acc, double e0, double e1, double e2, double e3, double *y, double (&dot)[4])
    {
        y[row] = acc;
        if (EPI == EPI_RH_Y) dot[0] = fma(e0, acc, dot[0]);
        if (EPI == EPI_QY_YY) { dot[0] = fma(e0, acc, dot[0]); dot[1] = fma(acc, acc, dot[1]); }
        if (EPI == EPI_CA4) {
            dot[0] = fma(e0, e1, dot[0]); dot[1] = fma(e0, acc, dot[1]);
            dot[2] = fma(e0, e2, dot[2]); dot[3] = fma(e0, e3, dot[3]);
        }
    }
    // SpMV over a shared-memory-resident slice: thread-per-row (rows tid + k CT, so neighbouring threads gather neighbouring
    // columns); a row's entries are accumulated in storage order, like spmv_impl.  Loads are unconditional on clamped indices
    // (always a valid entry of this slice; no predicate per load, so the U gathers of a pass are in flight together), only the
    // multiply-adds are guarded.
    template <int EPI, class F>
    __device__ void spmv_res(const double *x, double *y, double (&dot)[4], F far)
    {
        constexpr int U = 16;
        const double *xo = x + rp.w.obase, *xg = x + rp.w.gbase;
        const unsigned ospan = rp.w.ospan;
        const int rows = rp.rows;
        const bool empty = rp.nnz == 0u;                      // a slice of empty rows: y = 0, the dots see acc = 0
        const unsigned last = empty ? 0u : rp.nnz - 1u;
        for (int r = tid; r < rows; r += CT) {
            const int row = rp.row_lo + r;
            unsigned j = rs_ptr[r];
            const unsigned e = rs_ptr[r + 1];
            double e0 = 0.0, e1 = 0.0, e2 = 0.0, e3 = 0.0;     // epilogue operands: in flight during the gathers
            epi_load<EPI>(row, e0, e1, e2, e3, far);
            double acc = 0.0;
            while (j < e) {                                    // never entered when the slice is empty
                double xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const unsigned c = rs_col[min(min(j + (unsigned)u, e - 1u), last)];
                    xv[u] = ld_coherent((c < ospan ? xo : xg) + c);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {                  // the values come from shared memory when they are needed
                    const double v = rs_val[min(min(j + (unsigned)u, e - 1u), last)];
                    if (j + (unsigned)u < e) acc = fma(v, xv[u], acc);
                }
                j += (unsigned)U;
            }
            row_done<EPI>(row, acc, e0, e1, e2, e3, y, dot);
        }
    }

    // CODED: the stage holds the CTA's 16-bit column codes, each turned back into the column with one select and one add
    // before its gather.  PACKED (CODED CTAs only): the stage holds the three planes of the packed values, each value put
    // back together by PackedVal.
    template <int EPI, bool CODED, bool PACKED, class F>
    __device__ void spmv_impl(const double *x, double *y, double (&dot)[4], F far)
    {
        const int stages = a.stages;
        const StageLayout L(a.cap, RPT, 0);
        const int sub = tid % LANES, row_in_tile = tid / LANES;
        const ColWindow w = rp.w;
        double carry = 0.0;
        for (int lt = 0; lt < my_tiles; ++lt, ++vis) {
            const int s = sh.ring.wait(vis, (unsigned)stages);
            const unsigned char *st = dyn + (size_t)s * stage_bytes;
            const double   *sval = L.vals(st);
            const unsigned *scol = L.cols(st);
            const unsigned short *scode = L.codes(st);
            const unsigned *sptr = L.ptrs(st);
            const unsigned sts = PACKED ? smem_u32(st) : 0u, adj = PACKED ? smem_u32(sh.vadj) : 0u;
            auto column = [&](unsigned idx) { return CODED ? col_decode(w, scode[idx]) : scol[idx]; };
            auto value = [&](unsigned idx) {
                if constexpr (PACKED) return val_load(adj, sts, L, idx);
                else return sval[idx];
            };
            const ChunkStageHdr h = sh.ring.hdr[s];
            if (h.flag != 0) {
                // one chunk of a row longer than a stage: the whole CTA multiplies it, the row's partial sum is carried
                // from chunk to chunk in `carry` (same value in every thread) and the row is finished by its last chunk
                double part[1] = {0.0};
                for (unsigned jj = h.lo + (unsigned)tid; jj < h.hi; jj += 4u * CT) {
                    double pv[4], px[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const unsigned idx = min(jj + (unsigned)(u * CT), h.hi - 1u);
                        pv[u] = (double)value(idx); px[u] = ld_coherent(x + column(idx));
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        if (jj + (unsigned)(u * CT) < h.hi) part[0] = fma(pv[u], px[u], part[0]);
                }
                cblock_sum<1, CT>(part, sh.scratch);                   // fixed order; result in every lane of warp 0
                if (tid == 0) sh.red[0][0] = part[0];
                nbar(1, CT);
                carry += sh.red[0][0];
                if (h.flag == 2) {
                    if (tid == 0) {
                        double e0 = 0.0, e1 = 0.0, e2 = 0.0, e3 = 0.0;
                        epi_load<EPI>(h.row0, e0, e1, e2, e3, far);
                        row_done<EPI>(h.row0, carry, e0, e1, e2, e3, y, dot);
                    }
                    carry = 0.0;
                }
                sh.ring.release(s);
                continue;
            }
            const int row = h.row0 + row_in_tile;
            const bool valid = row < h.row1;
            int j = 0, e = 0;
            double e0 = 0.0, e1 = 0.0, e2 = 0.0, e3 = 0.0;     // epilogue operands: in flight during the gathers
            if (valid) {
                j = (int)(sptr[row - h.rowa] - h.a0) + sub;
                e = (int)(sptr[row - h.rowa + 1] - h.a0);
                if (sub == 0) epi_load<EPI>(row, e0, e1, e2, e3, far);
            }
            double acc[1];
            row_product<LANES, UNR, 1>(value, column, {x}, j, e, acc);
            if (valid && sub == 0) row_done<EPI>(row, acc[0], e0, e1, e2, e3, y, dot);
            sh.ring.release(s);
        }
    }

    // ---------------------------------------------------------------- vector phase over the CTA's own rows --
    // row_lo is a multiple of 16 and every arena vector is 128-byte aligned: 16-byte accesses, two in flight per
    // vector and thread; far: the L2 policy of the phase's far accesses (body)
    template <int PH, class F = Plain>
    __device__ void vec(double *dot, F far = {})
    {
        Coef c;
        c.al = sh.sc.alpha; c.be = sh.sc.beta; c.om = sh.sc.omega;
        c.nbo = -c.be * c.om;
        const int hi2 = row_lo + ((row_hi - row_lo) & ~1);
        int i = row_lo + 2 * tid;
        for (; i + 2 * CT < hi2; i += 4 * CT) body<PH, Pairs<2, 2 * CT>>(a.v, i, c, dot, far);
        for (; i < hi2; i += 2 * CT) body<PH, Pairs<1, 2 * CT>>(a.v, i, c, dot, far);
        if (tid == 0 && hi2 < row_hi) body<PH, Contig<1>>(a.v, hi2, c, dot, far);
    }
    // ---------------------------------------------------------------- multi-GPU helpers ---------------------
    // releasing arrival + wait for EVERY CTA of this GPU (all == true) or for the CTAs owning the gathered columns
    __device__ void sync_local(bool all)
    {
        double d0[1] = {0.0};
        arrive<0>(d0, true);
        if (!all) { wait_nbr(); return; }
        wait_all();
        if (tid < RED_THREADS) {
            nbar(2, RED_THREADS);
            if (tid < 32) fence_gpu();                 // acquire (+ L1 invalidate) after ALL pollers are through
        }
        nbar(1, CT);
        if (sh.flags[3]) { if (tid == 0) { sh.sc.error = 1; sh.sc.done = 1; } nbar(1, CT); }
    }
    // Boundary rows of vector `id` -> LL region `region` of the peers that gather them: every element travels as one
    // 16-byte pair of self-validating words {lo | epoch, hi | epoch} (dev.cuh), so the receiver needs neither a flag nor
    // a system-scope fence on the sender's side -- it polls the words of the elements it consumes.
    __device__ void push_ll(int id, int region, unsigned epoch)
    {
        if (push_slots == 0u) return;
        nbar(1, CT);                                  // the rows being pushed are final
        const double *src = a.vec_base + (long long)id * a.vstride;
#pragma unroll
        for (int s = 0; s < MAX_RANKS - 1; ++s) {
            if (!((push_slots >> s) & 1u)) continue;
            unsigned long long *dst = a.push.ll_dst[s] + 2ll * (long long)region * a.push.ll_stride[s];
            const PushRun *runs = a.push.runs[s];
            const int nr = a.push.nruns[s];
            int lo = 0, hi = nr;                      // first run that ends after row_lo
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (runs[mid].src + runs[mid].len <= row_lo) lo = mid + 1; else hi = mid; }
            for (int ri = lo; ri < nr; ++ri) {
                const PushRun r = runs[ri];
                if (r.src >= row_hi) break;
                const int b = max(r.src, row_lo), e = min(r.src + r.len, row_hi);
                for (int i = b + tid; i < e; i += CT) {
                    unsigned long long w0, w1;
                    ll_encode(src[i], epoch, w0, w1);
                    st_ll_sys(dst + 2ll * (long long)(r.dst_off + (i - r.src)), w0, w1);
                }
            }
        }
    }
    __device__ double ll_take(const unsigned long long *w, unsigned epoch, unsigned long long t0)
    {
        unsigned long long w0, w1;
        unsigned spins = 0;
        for (;;) {
            ld_ll_sys(w, w0, w1);
            if (ll_valid(w0, w1, epoch)) break;
            poll_pause(++spins);
            if (timed_out(t0, spins)) { fail(); break; }
        }
        return ll_decode(w0, w1);
    }
    // LL region -> plain ghost tail of vector `id`, for exactly the ghost slots this CTA's rows gather (several CTAs may
    // unpack the same slot: the copy is out of place and writes the same bits).  Ends with a CTA barrier.
    __device__ void unpack_ll(int id, int region, unsigned epoch)
    {
        if (ghost_hi > ghost_lo) {
            double *g = a.vec_base + (long long)id * a.vstride + a.ghost_off;
            const unsigned long long *ll = a.ll + 2ll * region * a.ll_stride;
            const unsigned long long t0 = globaltimer_ns();
            for (int i = ghost_lo + tid; i < ghost_hi; i += CT) g[i] = ll_take(ll + 2ll * i, epoch, t0);
        }
        nbar(1, CT);
    }
    // halo exchange of the CA / pipelined loops where solver.c has no reduction: boundary rows leave as LL words, the CTA waits
    // for the CTAs owning the gathered columns, then unpacks the ghost slots it gathers
    __device__ void halo_ll(int id, int region)
    {
        if (a.comm.world == 1) { sync_nbr(); return; }
        const unsigned ep = (unsigned)(++halo_epoch);
        double d0[1] = {0.0};
        arrive<0>(d0, true);
        push_ll(id, region, ep);
        wait_nbr();
        unpack_ll(id, region, ep);
    }
    // this CTA's share of the ghost slots, element-wise exactly like the owner's rows (same operands, same operation
    // order -> bitwise the values the owner computes)
    __device__ void ghost_q(int sregion, unsigned s_epoch)                 // q = r - alpha s            solver.c:94
    {
        const double al = sh.sc.alpha;
        double *r = a.v.r + a.ghost_off;
        const unsigned long long *sll = a.ll + 2ll * sregion * a.ll_stride;
        const unsigned long long t0 = globaltimer_ns();
        for (int i = gs_lo + tid; i < gs_hi; i += CT) r[i] = fma(-al, ll_take(sll + 2ll * i, s_epoch, t0), r[i]);
    }
    __device__ void ghost_p(int sregion, unsigned s_epoch, unsigned r_epoch)   // p = r + beta (p - omega s)  solver.c:117-119
    {
        const double be = sh.sc.beta, nbo = -sh.sc.beta * sh.sc.omega;
        double *p = a.v.p + a.ghost_off, *r = a.v.r + a.ghost_off;
        const unsigned long long *sll = a.ll + 2ll * sregion * a.ll_stride, *rll = a.ll + 2ll * LL_R * a.ll_stride;
        const unsigned long long t0 = globaltimer_ns();
        for (int i = gs_lo + tid; i < gs_hi; i += CT) {
            const double rn = ll_take(rll + 2ll * i, r_epoch, t0);      // the owner's new r (pushed with the beta reduction)
            const double sg = ll_take(sll + 2ll * i, s_epoch, t0);      // the same s the ghost q used (already validated)
            double t = be * p[i];
            t = fma(1.0, rn, t);
            p[i] = fma(nbo, sg, t);
            r[i] = rn;                                                   // ghost r for the next q and for nothing else
        }
    }
    // ---------------------------------------------------------------- solver.c:86-127, several GPUs ---------
    // Two halo exchanges per iteration instead of the reference's two allgathers -- and neither is waited for on its own:
    // the boundary rows of s leave with the alpha reduction, those of the new r with the beta reduction (both are known
    // before the reduction they ride on), and every rank advances its ghost copies of q and p itself with the
    // recurrences q = r - alpha s, p = r + beta (p - omega s) applied to the ghost slots (bitwise what the owner
    // computes).  So an iteration costs three NVLink-latency sync points, not five.  The boundary values travel as LL
    // words (push_ll): no system-scope fence and no flag on the sender's side (a fence.sys after NVLink stores was
    // measured at ~4.5 us), the consumer polls exactly the elements it needs.  The LL copy of s alternates between
    // two regions: a peer may already push s of iteration k + 1 while this rank still applies s of iteration k to its
    // ghost p; r needs one region (its next push follows a reduction that this rank enters after consuming it).
    // __noinline__: inlined next to run_ca, it makes bicg_mega_kernel<512, 1> spill the CTA's column window
    __device__ __noinline__ void run_bicgstab_multi()
    {
        double d4[4], d2[2], d1[1], d0[1];
        d0[0] = 0.0;
        unsigned par = 0u;
        while (true) {
            mark(0);
            d4[0] = d4[1] = d4[2] = d4[3] = 0.0;
            spmv<EPI_RH_Y>(a.v.p, a.v.s, d4);                               // s = A p, (r#,s)           :88-91
            const unsigned s_epoch = (unsigned)(++halo_epoch);
            mark(1);
            d1[0] = d4[0];
            reduce<1>(d1, FIN_BICG_ALPHA, true, V_S, LL_S0 + (int)par, s_epoch);    // alpha (+ boundary rows of s) :93
            mark(2);
            if (stop_now()) break;
            vec<PH_BICG_Q>(d0);                                             // q = r - alpha s            :94
            ghost_q(LL_S0 + (int)par, s_epoch);
            mark(3);
            sync_local(reads_ghost);
            mark(4);
            d4[0] = d4[1] = 0.0;
            spmv<EPI_QY_YY>(a.v.r, a.v.y, d4);                              // y = A q, (q,y), (y,y)      :96-102
            mark(5);
            d2[0] = d4[0]; d2[1] = d4[1];
            reduce<2>(d2, FIN_BICG_OMEGA);                                  // omega                      :104
            mark(6);
            d2[0] = d2[1] = 0.0;
            vec<PH_BICG_XR>(d2);                                            // x, r, (r,r), (r#,r)        :105-114
            const unsigned r_epoch = (unsigned)(++halo_epoch);
            mark(7);
            reduce<2>(d2, FIN_BICG_BETA, false, V_R, LL_R, r_epoch);          // beta, k++, loop test (+ boundary rows of r) :116-120
            mark(8);
            if (stop_now()) break;
            vec<PH_BICG_P>(d0);                                             // p                          :117-119
            ghost_p(LL_S0 + (int)par, s_epoch, r_epoch);
            mark(9);
            sync_local(reads_ghost);
            mark(10);
            par ^= 1u;
            ++trace_it;
        }
    }
    // ---------------------------------------------------------------- solver.c:86-127 -----------------------
    // __noinline__: inlined into the kernel body, it makes the four 512-thread kernels spill under their 96-register cap
    //
    // L2 policy of every vector access of an iteration.  Six vectors of n doubles cycle through it (p, s, r# = rh,
    // r = q, y, x: 77 MB at T', against the H100's 50 MB of L2, beside the evict-first matrix stream).  An access whose
    // next use lies behind most of the other vectors is marked evict-first, so that the four that are re-used soon
    // (p, s, r, y) keep L2 to themselves; all others are plain.
    //   phase                  access                         policy       next use of the vector
    //   SpMV s = A p           gather p, store s              plain        XR / Q
    //                          load rh (EPI_RH_Y)             evict-first  XR, behind q, y
    //   PH_BICG_Q              load r, s; store r (= q)       plain        SpMV y = A q / P
    //   SpMV y = A q           gather q, load q; store y      plain        XR
    //   PH_BICG_XR             load x; store x                evict-first  XR of the next iteration
    //                          load y                         evict-first  none: the next SpMV 2 overwrites y
    //                          load rh                        evict-first  SpMV 1 of the next iteration, behind p, s
    //                          load p, r; store r             plain        P
    //   PH_BICG_P              load s                         evict-first  none: the next SpMV 1 overwrites s
    //                          load p, r; store p             plain        SpMV s = A p
    // Each of the five demotions was measured on its own (T', H100 80GB HBM3, 700 W: 272.5 us per iteration without
    // any, 260.9 with all five, 263.5 to 265.3 with any one left plain).  The policy value is made where a phase
    // begins (evict_first()).  run_bicgstab_multi keeps plain accesses: a rank's share of the vectors is 1 / N of them.
    __device__ __noinline__ void run_bicgstab()
    {
        double d4[4], d2[2], d1[1], d0[1];
        d0[0] = 0.0;
        while (true) {
            mark(0);
            d4[0] = d4[1] = d4[2] = d4[3] = 0.0;
            spmv<EPI_RH_Y>(a.v.p, a.v.s, d4, evict_first());                // s = A p, (r#,s)           :88-91
            mark(1);
            d1[0] = d4[0];
            reduce<1>(d1, FIN_BICG_ALPHA, true);                            // alpha                      :93
            mark(2);
            if (stop_now()) break;
            vec<PH_BICG_Q>(d0);                                             // q = r - alpha s            :94
            mark(3);
            sync_nbr();
            mark(4);
            d4[0] = d4[1] = 0.0;
            spmv<EPI_QY_YY>(a.v.r, a.v.y, d4);                              // y = A q, (q,y), (y,y)      :96-102
            mark(5);
            d2[0] = d4[0]; d2[1] = d4[1];
            reduce<2>(d2, FIN_BICG_OMEGA);                                  // omega                      :104
            mark(6);
            d2[0] = d2[1] = 0.0;
            vec<PH_BICG_XR>(d2, evict_first());                             // x, r, (r,r), (r#,r)        :105-114
            mark(7);
            reduce<2>(d2, FIN_BICG_BETA);                                   // beta, k++, loop test       :116-120
            mark(8);
            if (stop_now()) break;
            vec<PH_BICG_P>(d0, evict_first());                              // p                          :117-119
            mark(9);
            sync_nbr();
            mark(10);
            ++trace_it;
        }
    }
    // ---------------------------------------------------------------- solver.c:216-259 ----------------------
    // __noinline__: inlined into the kernel body next to the packed-value SpMV, it makes the 512-thread kernels with
    // LANES > 1 spill
    __device__ __noinline__ void run_ca()
    {
        double d5[5], d4[4], d2[2], d1[1], d0[1];
        d0[0] = 0.0;
        while (true) {
            vec<PH_CA_PS>(d0);                                              // p, s                       :217-222
            halo_ll(V_S, LL_S0);
            d4[0] = 0.0;
            spmv<EPI_NONE>(a.v.s, a.v.z, d4);                               // z = A s                    :224
            nbar(1, CT);                                                    // own rows of z written by other warps
            d2[0] = d2[1] = 0.0;
            vec<PH_QY>(d2);                                                 // q, y, (q,y), (y,y)         :225-230
            reduce<2>(d2, FIN_OMEGA2);                                      // omega                      :232
            if (stop_now()) break;
            d1[0] = 0.0;
            vec<PH_CA_XR>(d1);                                              // x, r, local (r,r)          :233-236
            halo_ll(V_R, LL_R);
            d4[0] = d4[1] = d4[2] = d4[3] = 0.0;
            spmv<EPI_CA4>(a.v.r, a.v.w, d4);                                // w = A r, 4 dots            :238-247
            d5[0] = d4[0]; d5[1] = d4[1]; d5[2] = d4[2]; d5[3] = d4[3]; d5[4] = d1[0];
            reduce<5>(d5, FIN_CAPIPE_END);                                  // beta, alpha, k++, test     :248-253
            if (stop_now()) break;
        }
    }
    // ---------------------------------------------------------------- solver.c:351-398 / 494-547 ------------
    // __noinline__ for the same reason as run_bicgstab
    __device__ __noinline__ void run_pipe(bool rr)
    {
        double d5[5], d4[4], d2[2], d0[1];
        d0[0] = 0.0; d4[0] = d4[1] = d4[2] = d4[3] = 0.0;
        while (true) {
            const int k = sh.sc.k;
            const bool replace = rr && (k % a.krr == 0) && k > 0 && k <= a.krr * a.nrr;   // solver.c:498, 522
            d2[0] = d2[1] = 0.0;
            if (!replace) {
                vec<PH_PIPE_1>(d2);                                         // p,s,z,q,y + (q,y),(y,y)    :352-364
            } else {
                vec<PH_RR_P>(d0);                                           // p                          :494-496
                halo_ll(V_P, LL_P);
                spmv<EPI_NONE>(a.v.p, a.v.s, d4);                           // s = A p                    :499
                halo_ll(V_S, LL_S0);
                spmv<EPI_NONE>(a.v.s, a.v.z, d4);                           // z = A s                    :500
                nbar(1, CT);
                vec<PH_QY>(d2);                                             // q, y, (q,y), (y,y)         :509-512
            }
            post<2>(d2, V_Z, LL_Z);                                         // MPI_Iallreduce x2 (+ halo of z)
            spmv<EPI_NONE>(a.v.z, a.v.v, d4);                               // v = A z hides it           :365 / 513
            complete<2>(FIN_OMEGA2, false);                                 // MPI_Wait x2 -> omega       :366-369
            if (stop_now()) break;
            d5[0] = d5[1] = d5[2] = d5[3] = d5[4] = 0.0;
            if (!replace) {
                vec<PH_PIPE_3>(d5);                                         // x, r, w + 5 dots           :370-380
            } else {
                vec<PH_RR_X>(d0);                                           // x                          :518-519
                halo_ll(V_X, LL_X);
                spmv<EPI_NONE>(a.v.x, a.v.ax, d4);                          // Ax = A x                   :523
                nbar(1, CT);
                vec<PH_RR_R>(d0);                                           // r = b - Ax                 :524-525
                halo_ll(V_R, LL_R);
                spmv<EPI_NONE>(a.v.r, a.v.w, d4);                           // w = A r                    :526
                nbar(1, CT);
                vec<PH_RR_DOTS>(d5);                                        // 5 dots                     :533-539
            }
            post<5>(d5, V_W, LL_W);                                         // MPI_Iallreduce x5 (+ halo of w)
            spmv<EPI_NONE>(a.v.w, a.v.t, d4);                               // t = A w hides it           :381 / 540
            complete<5>(FIN_CAPIPE_END, true);                              // MPI_Wait x5 -> beta, alpha :382-388
            if (stop_now()) break;
        }
    }
};

template <int CT, int LANES>
__global__ void __launch_bounds__(CT + 32, 1) bicg_mega_kernel(const __grid_constant__ MegaArgs a)
{
    using M = Mega<CT, LANES>;
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ __align__(16) MegaShared sh;

    const int tid = threadIdx.x;
    const int stages = a.stages;
    if (tid == 0) {
        sh.flags[0] = sh.flags[1] = sh.flags[2] = sh.flags[3] = 0;
        sh.ring.init(stages, (unsigned)M::NCW);
    }
    __syncthreads();

    const int t0 = a.cta_tile[blockIdx.x], t1 = a.cta_tile[blockIdx.x + 1];
    const int my_tiles = t1 - t0;
    const StageLayout L(a.cap, M::RPT, 0);

    if (tid >= CT) {
        // ============================ producer warp: streams this CTA's tiles round and round ==============
        const ResidentPlan rp = tid == CT ? resident_plan(a, t0, t1, LANES) : ResidentPlan{};
        if (tid == CT && my_tiles > 0 && !rp.on) {
            volatile int *flags = sh.flags;
            const bool coded = streams_codes(a, rp, my_tiles);
            const bool packed = streams_values(a, coded);
            const TileFormat<Hint> f{packed, coded, 0, Hint{l2_evict_first_policy()}};
            const TileSrc src{packed ? (const void *)a.vlo : (const void *)a.val, a.vmid, a.vhi,
                              coded ? (const void *)a.col16 : (const void *)a.col, a.ptr};
            unsigned v = 0;
            for (;; ++v) {
                const int s = sh.ring.acquire(v, (unsigned)stages, [&] { return flags[1] != 0; });
                if (s < 0) break;
                const int t = t0 + (int)(v % (unsigned)my_tiles);
                const int row0 = a.tile_row[t], row1 = a.tile_row[t + 1];
                const unsigned p0 = a.tile_nz[t], p1 = a.tile_nz[t + 1];
                const TileWindow w = tile_window(row0, row1, p0, p1, f.align());
                sh.ring.hdr[s] = ChunkStageHdr{{row0, row1, w.a0, w.rowa}, p0 - w.a0, p1 - w.a0, a.tile_flag ? a.tile_flag[t] : 0, 0};
                tile_issue(dyn_smem + (size_t)s * L.bytes(), L, sh.ring.full_bar(s), f, w, src);
            }
            // drain: bulk copies already issued must land before the CTA may retire its shared memory
            for (unsigned w = (unsigned)flags[2]; w < v; ++w) sh.ring.wait(w, (unsigned)stages);
        }
    } else {
        // ============================ consumer warps: the solver ============================================
        M m(a, sh);
        m.dyn = dyn_smem; m.tid = tid; m.lane = tid & 31; m.my_tiles = my_tiles; m.vis = 0u; m.stage_bytes = L.bytes();
        m.row_lo = a.tile_row[t0]; m.row_hi = a.tile_row[t1];
        m.trace_it = 0;
        m.trace_who = blockIdx.x == 0 ? 0 : (blockIdx.x == gridDim.x / 2 ? 1 : -1);
        // counters left by the previous solve; nobody advances them before every CTA has passed its first arrive
        m.gen = a.sync->st.gen; m.red_epoch = a.sync->st.red_epoch; m.halo_epoch = a.sync->st.halo_epoch;
        m.posted_gen = m.gen;
        if (tid == 0) sh.sc = *a.sc;                  // the scalars the init kernels left (solver.c:74-83, 200-213)

        // which CTAs own the columns my rows gather, which ranks fill the ghost slots they gather
        const int4 dep = a.cta_dep[blockIdx.x];
        const int G = (int)gridDim.x;
        auto cta_of_row = [&](int r) {              // last CTA whose first row is <= r
            int lo = 0, hi = G;                     // first rows are non-decreasing; a.tile_row[a.cta_tile[G]] = rows
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (a.tile_row[a.cta_tile[mid]] <= r) lo = mid + 1; else hi = mid; }
            return lo - 1;
        };
        m.dep_lo = 1; m.dep_hi = 0;
        if (dep.x <= dep.y) { m.dep_lo = max(0, cta_of_row(dep.x)); m.dep_hi = min(G - 1, cta_of_row(dep.y)); }
        m.reads_ghost = a.comm.world > 1 && dep.z <= dep.w;
        m.ghost_lo = m.reads_ghost ? dep.z : 0; m.ghost_hi = m.reads_ghost ? dep.w + 1 : 0;
        // the reducer sits in the middle of the row range: on banded matrices the CTAs at the ends are busy pushing boundary
        // rows over NVLink (slow per SM) right before the reductions, and everybody would wait for them twice
        m.is_reducer = (int)blockIdx.x == G / 2;
        m.gs_lo = m.gs_hi = 0;
        if (a.comm.world > 1) {
            // ghost slots are shared out evenly (16-slot granules) over the CTAs
            const int ng = a.n_ghost;
            const int chunk = ((ng + G - 1) / G + 15) & ~15;
            m.gs_lo = min(ng, (int)blockIdx.x * chunk);
            m.gs_hi = min(ng, m.gs_lo + chunk);
        }
        m.push_slots = 0u;
        if (a.comm.world > 1) {
            PushDesc pd;
            pd.npeers = 1;
            for (int s = 0; s < a.push.npeers; ++s) {
                pd.runs[0] = a.push.runs[s]; pd.nruns[0] = a.push.nruns[s];
                if (m.row_hi > m.row_lo && push_touches(pd, m.row_lo, m.row_hi)) m.push_slots |= 1u << s;
            }
        }
        // resident mode: the slice goes into shared memory once (plain coalesced loads; the ring is not used by this CTA)
        m.rp = resident_plan(a, t0, t1, LANES);
        m.resident = m.rp.on;
        m.coded = streams_codes(a, m.rp, my_tiles);
        m.packed = streams_values(a, m.coded);
        if (m.packed && tid < VAL_TABLE_MAX) sh.vadj[tid] = val_adj(a.vtab[blockIdx.x], tid);
        if (m.resident) {
            const size_t nnzp = ((size_t)m.rp.nnz + 7u) & ~(size_t)7u;
            double *sv = reinterpret_cast<double *>(dyn_smem);
            unsigned short *sc16 = reinterpret_cast<unsigned short *>(sv + nnzp);
            unsigned *sp = reinterpret_cast<unsigned *>(sc16 + nnzp);
            for (unsigned i = (unsigned)tid; i < m.rp.nnz; i += (unsigned)CT) {
                sv[i] = a.val[m.rp.nz_lo + i];
                sc16[i] = a.col16[m.rp.nz_lo + i];
            }
            for (int r = tid; r <= m.rp.rows; r += CT) sp[r] = a.ptr[m.rp.row_lo + r] - m.rp.nz_lo;
            m.rs_val = sv; m.rs_col = sc16; m.rs_ptr = sp;
            if (tid == 0) atomicAdd(&a.sync->st.resident_ctas, 1);
        }
        if (m.coded && tid == 0) atomicAdd(&a.sync->st.coded_ctas, 1);
        if (m.packed && tid == 0) atomicAdd(&a.sync->st.packed_ctas, 1);
        nbar(1, CT);
        if (a.comm.world > 1 && (m.reads_ghost || m.gs_hi > m.gs_lo)) {
            // the vectors the first phases read were pushed by the init kernels (kernel-per-phase protocol)
            if (tid < 32 && !halo_wait_epoch(a.comm, sh.sc.halo_epoch) && tid == 0) { sh.sc.error = 1; sh.sc.done = 1; }
            if (tid < 32) fence_sys();
            nbar(1, CT);
        }
        if (!m.stop_now()) {                                             // solver.c:86 before the first pass
            if (a.method == 0) { if (a.comm.world > 1) m.run_bicgstab_multi(); else m.run_bicgstab(); }
            else if (a.method == 1) m.run_ca();
            else m.run_pipe(a.method == 3);
        }
        nbar(1, CT);
        if (tid == 0) {
            sh.flags[2] = (int)m.vis; __threadfence_block(); sh.flags[1] = 1;
            if (blockIdx.x == 0) {
                *a.sc = sh.sc;
                a.sync->st.gen = m.gen; a.sync->st.red_epoch = m.red_epoch; a.sync->st.halo_epoch = m.halo_epoch;
            } else if (sh.sc.error) a.sc->error = 1;
        }
    }
}

// per-CTA column ranges: min / max own column and min / max ghost slot over the CTA's entries
__global__ void __launch_bounds__(256) mega_dep_kernel(const unsigned *__restrict__ col, const unsigned *__restrict__ ptr,
                                                       const int *__restrict__ tile_row, const int *__restrict__ cta_tile,
                                                       int ghost_off, int4 *dep)
{
    __shared__ int s[4];
    if (threadIdx.x == 0) { s[0] = 0x7fffffff; s[1] = -1; s[2] = 0x7fffffff; s[3] = -1; }
    __syncthreads();
    const int r0 = tile_row[cta_tile[blockIdx.x]], r1 = tile_row[cta_tile[blockIdx.x + 1]];
    int omin = 0x7fffffff, omax = -1, gmin = 0x7fffffff, gmax = -1;
    if (r1 > r0) {
        const unsigned e0 = ptr[r0], e1 = ptr[r1];
        for (unsigned j = e0 + threadIdx.x; j < e1; j += blockDim.x) {
            const int c = (int)col[j];
            if (c < ghost_off) { omin = min(omin, c); omax = max(omax, c); }
            else { gmin = min(gmin, c - ghost_off); gmax = max(gmax, c - ghost_off); }
        }
    }
    atomicMin(&s[0], omin); atomicMax(&s[1], omax); atomicMin(&s[2], gmin); atomicMax(&s[3], gmax);
    __syncthreads();
    if (threadIdx.x == 0) dep[blockIdx.x] = make_int4(s[0], s[1], s[2], s[3]);
}

// the 16-bit column codes (col_encode) of every CTA whose column window fits them; the entries of the other CTAs are not
// written (they stream, or keep resident, nothing but their 32-bit columns)
__global__ void __launch_bounds__(256) mega_code_kernel(const unsigned *__restrict__ col, const unsigned *__restrict__ ptr,
                                                        const int *__restrict__ tile_row, const int *__restrict__ cta_tile,
                                                        int ghost_off, const int4 *__restrict__ dep, unsigned short *__restrict__ col16)
{
    const ColWindow w = col_window(dep[blockIdx.x], ghost_off);
    if (!w.ok) return;
    const int r0 = tile_row[cta_tile[blockIdx.x]], r1 = tile_row[cta_tile[blockIdx.x + 1]];
    if (r1 <= r0) return;
    const unsigned e0 = ptr[r0], e1 = ptr[r1];
    for (unsigned j = e0 + threadIdx.x; j < e1; j += blockDim.x) col16[j] = col_encode(w, ghost_off, col[j]);
}

// The value table of every CTA: the distinct sign / exponent fields (bits 63..52) of its entries, ascending -- a set, so
// it does not depend on the order in which threads find them -- or n = 0 beyond VAL_TABLE_MAX fields.  A CTA that has a
// table and column codes (col_window) also gets its entries packed; the entries of the other CTAs are not written.  The
// split works on the bit pattern, so +-0.0, subnormals and every other value round-trip exactly.
__global__ void __launch_bounds__(256) mega_value_kernel(const double *__restrict__ val, const unsigned *__restrict__ ptr,
                                                         const int *__restrict__ tile_row, const int *__restrict__ cta_tile,
                                                         int ghost_off, const int4 *__restrict__ dep, ValTable *__restrict__ vtab,
                                                         unsigned char *__restrict__ vhi, unsigned short *__restrict__ vmid,
                                                         unsigned *__restrict__ vlo)
{
    constexpr int W = 4096 / 32;
    __shared__ unsigned seen[W];                  // bit f: some entry of the CTA has field f
    __shared__ int below[W];                      // fields in the words before: the table index of field f is
    __shared__ int total;                         // below[f / 32] + the bits of seen[f / 32] under f
    for (int i = threadIdx.x; i < W; i += blockDim.x) seen[i] = 0u;
    __syncthreads();
    const int r0 = tile_row[cta_tile[blockIdx.x]], r1 = tile_row[cta_tile[blockIdx.x + 1]];
    const unsigned e0 = r1 > r0 ? ptr[r0] : 0u, e1 = r1 > r0 ? ptr[r1] : 0u;
    for (unsigned j = e0 + threadIdx.x; j < e1; j += blockDim.x) {
        const unsigned f = (unsigned)((unsigned long long)__double_as_longlong(val[j]) >> 52), b = 1u << (f & 31u);
        if (!(seen[f >> 5] & b)) atomicOr(&seen[f >> 5], b);       // a plain read first: the set is small and soon complete
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        for (int i = 0; i < W; ++i) { below[i] = n; n += __popc(seen[i]); }
        total = n;
        ValTable t;
        t.n = n <= VAL_TABLE_MAX ? n : 0;
        for (int k = 0; k < VAL_TABLE_MAX; ++k) t.field[k] = 0;
        int k = 0;
        for (int i = 0; i < W && t.n > 0; ++i)
            for (unsigned b = seen[i]; b; b &= b - 1u) t.field[k++] = (unsigned short)(i * 32 + __ffs((int)b) - 1);
        vtab[blockIdx.x] = t;
    }
    __syncthreads();
    if (total == 0 || total > VAL_TABLE_MAX || !col_window(dep[blockIdx.x], ghost_off).ok) return;
    for (unsigned j = e0 + threadIdx.x; j < e1; j += blockDim.x) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(val[j]);
        const unsigned f = (unsigned)(bits >> 52);
        const unsigned idx = (unsigned)below[f >> 5] + __popc(seen[f >> 5] & ((1u << (f & 31u)) - 1u));
        vhi[j] = (unsigned char)((idx << 4) | ((unsigned)(bits >> 48) & 15u));
        vmid[j] = (unsigned short)(bits >> 32);
        vlo[j] = (unsigned)bits;
    }
}

template <int CT, int LANES>
cudaError_t launch(const MegaArgs &a, int grid, size_t smem, cudaStream_t st)
{
    void *params[1] = {(void *)&a};
    return cudaLaunchCooperativeKernel((const void *)bicg_mega_kernel<CT, LANES>, dim3(grid), dim3(CT + 32), params, smem, st);
}
} // namespace

size_t mega_smem_bytes(int cap, int stages, int threads, int lanes)
{
    return (size_t)stages * spmv_stage_bytes(cap, threads / lanes, 0);
}

bool mega_has_variant(int threads, int lanes)
{
    if (threads == 256) return lanes == 1;
    return threads == 512 && (lanes == 1 || lanes == 4 || lanes == 8 || lanes == 32);
}

int mega_setup_attributes()
{
    cudaError_t e;
    if ((e = smem_optin(bicg_mega_kernel<256, 1>)) != cudaSuccess) return (int)e;
    if ((e = smem_optin(bicg_mega_kernel<512, 1>)) != cudaSuccess) return (int)e;
    if ((e = smem_optin(bicg_mega_kernel<512, 4>)) != cudaSuccess) return (int)e;
    if ((e = smem_optin(bicg_mega_kernel<512, 8>)) != cudaSuccess) return (int)e;
    if ((e = smem_optin(bicg_mega_kernel<512, 32>)) != cudaSuccess) return (int)e;
    return 0;
}

int launch_mega(int threads, int lanes, int grid, size_t smem, const MegaArgs &a, cudaStream_t st)
{
    if (threads == 256 && lanes == 1) return (int)launch<256, 1>(a, grid, smem, st);
    if (threads != 512) return (int)cudaErrorInvalidValue;
    switch (lanes) {
    case 1:  return (int)launch<512, 1>(a, grid, smem, st);
    case 4:  return (int)launch<512, 4>(a, grid, smem, st);
    case 8:  return (int)launch<512, 8>(a, grid, smem, st);
    case 32: return (int)launch<512, 32>(a, grid, smem, st);
    default: return (int)cudaErrorInvalidValue;
    }
}

void launch_mega_dep(const unsigned *col, const unsigned *ptr, const int *tile_row, const int *cta_tile, int grid,
                     int ghost_off, int4 *dep, cudaStream_t st)
{
    mega_dep_kernel<<<grid, 256, 0, st>>>(col, ptr, tile_row, cta_tile, ghost_off, dep);
}

void launch_mega_code(const unsigned *col, const unsigned *ptr, const int *tile_row, const int *cta_tile, int grid,
                      int ghost_off, const int4 *dep, unsigned short *col16, cudaStream_t st)
{
    mega_code_kernel<<<grid, 256, 0, st>>>(col, ptr, tile_row, cta_tile, ghost_off, dep, col16);
}

void launch_mega_values(const double *val, const unsigned *ptr, const int *tile_row, const int *cta_tile, int grid,
                        int ghost_off, const int4 *dep, ValTable *vtab, unsigned char *vhi, unsigned short *vmid,
                        unsigned *vlo, cudaStream_t st)
{
    mega_value_kernel<<<grid, 256, 0, st>>>(val, ptr, tile_row, cta_tile, ghost_off, dep, vtab, vhi, vmid, vlo);
}

} // namespace bicg
