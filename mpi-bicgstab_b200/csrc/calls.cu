// calls.cu -- what every entry point on a resident handle does around its work: the stream order of an asynchronous call, the
// agreement of the ranks on a collective call's arguments, and the timeout check at the end of a synchronous call.
#include "engine.hpp"

namespace bicg {

void wait_handle(bicg_matrix *m)
{
    if (m && m->ev_last) BICG_CUDA(cudaStreamWaitEvent(ctx().stream, m->ev_last, 0));
}

void async_handle_init(bicg_matrix *m)
{
    Context &c = ctx();
    if (!m->ev_last) {
        // the handle's first asynchronous use: matrix_create returns with the upload and the plan's encoding kernels still in
        // flight on the library's stream, and a synchronous call may have left work there too, so the handle's last work
        // starts out as everything enqueued on that stream so far
        BICG_CUDA(cudaEventCreateWithFlags(&m->ev_last, cudaEventDisableTiming));
        BICG_CUDA(cudaEventRecord(m->ev_last, c.stream));
    }
}

bool capturing(cudaStream_t st)
{
    cudaStreamCaptureStatus cs;
    BICG_CUDA(cudaStreamIsCapturing(st, &cs));
    return cs != cudaStreamCaptureStatusNone;
}

void stream_ordered(std::initializer_list<bicg_matrix *> handles, cudaStream_t st, bool captured,
                    const std::function<void()> &enqueue)
{
    for (bicg_matrix *m : handles) async_handle_init(m);
    for (bicg_matrix *m : handles) BICG_CUDA(cudaStreamWaitEvent(st, m->ev_last, captured ? cudaEventWaitExternal : 0));
    enqueue();
    for (bicg_matrix *m : handles)
        BICG_CUDA(cudaEventRecordWithFlags(m->ev_last, st, captured ? cudaEventRecordExternal : cudaEventRecordDefault));
}

bool ranks_agree(bool bad, std::initializer_list<long long> same)
{
    Context &c = ctx();
    std::vector<long long> mine(1, bad ? 1 : 0);
    mine.insert(mine.end(), same.begin(), same.end());
    const size_t k = mine.size();
    std::vector<long long> all(k * (size_t)c.world);
    c.host_allgather(mine.data(), all.data(), k * sizeof(long long));
    for (int p = 0; p < c.world; ++p) {
        const long long *o = all.data() + (size_t)p * k;
        if (o[0]) return false;
        for (size_t i = 1; i < k; ++i)
            if (o[i] != mine[i]) return false;
    }
    return true;
}

[[noreturn]] void timeout_fatal(const bicg_matrix *m, const char *during)
{
    fatal("bicgstab_b200: rank %d timed out during %s after %d s waiting for a peer GPU / another CTA (halo flag or reduction "
          "mailbox; BICG_PEER_TIMEOUT_S raises the bound)", m->rank, during, ctx().cfg.peer_timeout_s);
}

void sync_checked(bicg_matrix *m, const char *during)
{
    Context &c = ctx();
    int error = 0;
    BICG_CUDA(cudaMemcpyAsync(&error, &m->d_sc->error, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    BICG_CUDA(cudaStreamSynchronize(c.stream));
    if (error) timeout_fatal(m, during);
}

} // namespace bicg
