// shm_boot.cpp -- host-side rendezvous for multi-process jobs started without MPI or torch: a POSIX
// shared-memory segment with a sense-reversing barrier and an allgather, used (a) as the bicg_allgather_fn of
// bicg_comm_init and (b) to implement the handful of MPI calls main.c makes (include/compat/mpi.h).
// It only carries bootstrap data (IPC handles, halo plans, processor names); solver traffic never touches it.
#include "bicgstab_b200.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cerrno>
#include <csignal>
#include <cstring>
#include <fcntl.h>
#include <sched.h>
#include <string>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

namespace {

struct ShmHead {
    std::atomic<int> magic;        // SHM_READY once rank 0 has initialised THIS segment
    std::atomic<int> arrived;
    std::atomic<int> sense;
    std::atomic<int> joined;       // join tickets handed out: a fresh segment has exactly world - 1 to give
    std::atomic<int> abort;        // some rank is exiting abnormally: everybody leaves the barrier and exits
    int creator_pid;
    unsigned long long nonce;      // per-job value written by rank 0, echoed by every rank when the job starts
    char pad[32];
};
constexpr int SHM_READY = 0x42494347;     // "BICG"

struct Boot {
    int rank = 0, world = 1;
    ShmHead *head = nullptr;
    char *data = nullptr;
    size_t data_bytes = 0, total = 0;
    int local_sense = 0;
    int timeout_s = 1800;
    bool owner = false;
    std::string name;
} g;

int env_int(const char *a, const char *b, int dflt)
{
    const char *v = getenv(a);
    if (!v && b) v = getenv(b);
    return v ? atoi(v) : dflt;
}

double now_s()
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

[[noreturn]] void boot_fatal(const char *what)
{
    fprintf(stderr, "bicgstab_b200: rank %d: %s\n", g.rank, what);
    if (g.head) g.head->abort.store(1);          // the other ranks leave their barriers and exit too
    exit(1);                                     // atexit: rank 0 unlinks the segment
}

// exit path of every process that joined a job: a dying rank must not leave the others spinning, and rank 0 must not
// leave the segment behind for the next job to trip over
void at_exit_cleanup()
{
    if (!g.head) return;
    if (g.owner) shm_unlink(g.name.c_str());
}

void barrier()
{
    if (g.world == 1) return;
    g.local_sense = !g.local_sense;
    if (g.head->arrived.fetch_add(1) == g.world - 1) {
        g.head->arrived.store(0);
        g.head->sense.store(g.local_sense);
    } else {
        unsigned spins = 0;
        const double t0 = now_s();
        while (g.head->sense.load() != g.local_sense) {
            if ((++spins & 0xff) == 0) {
                sched_yield();
                if (g.head->abort.load()) { fprintf(stderr, "bicgstab_b200: rank %d: another rank aborted the job\n", g.rank); exit(1); }
                if ((spins & 0xffff) == 0 && now_s() - t0 > (double)g.timeout_s)
                    boot_fatal("host barrier timed out (a rank died or never arrived; BICG_BOOT_TIMEOUT_S raises the bound)");
            }
        }
    }
}

int shm_allgather(void *, const void *send, void *recv, size_t bytes)
{
    if (g.world == 1) { memcpy(recv, send, bytes); return 0; }
    if (bytes * (size_t)g.world > g.data_bytes) {
        fprintf(stderr, "bicgstab_b200: bootstrap allgather of %zu bytes/rank exceeds the shm segment (%zu); "
                        "raise BICG_SHM_MB\n", bytes, g.data_bytes);
        return -1;
    }
    memcpy(g.data + bytes * (size_t)g.rank, send, bytes);
    barrier();
    memcpy(recv, g.data, bytes * (size_t)g.world);
    barrier();
    return 0;
}

} // namespace

extern "C" {

// Join the job described by the environment.  Exposed so non-MPI C programs can bootstrap too.  Any failure is fatal
// (exit(1)): the reference's main.c ignores MPI_Init's return value, and a rank that silently became "rank 0 of 1"
// would solve the wrong problem.
int bicg_shm_bootstrap(void)
{
    g.rank = env_int("BICG_RANK", "RANK", 0);
    g.world = env_int("BICG_WORLD", "WORLD_SIZE", 1);
    g.timeout_s = std::max(1, env_int("BICG_BOOT_TIMEOUT_S", nullptr, 1800));
    if (g.world <= 1) { g.world = 1; g.rank = 0; return bicg_comm_init(0, 1, nullptr, nullptr); }
    if (g.world > 8) boot_fatal("more than 8 ranks: this library drives the GPUs of ONE NVSwitch box (one rank per GPU)");
    if (g.rank < 0 || g.rank >= g.world) boot_fatal("RANK outside [0, WORLD_SIZE)");
    // segment name: job id of the launcher (tools/bicgrun sets a unique one), else torchrun's port; never shared between users
    const char *job = getenv("BICG_JOB_ID");
    const char *port = getenv("MASTER_PORT");
    g.name = std::string("/bicg_b200_") + std::to_string((unsigned)getuid()) + "_" + (job ? job : (port ? port : "default"));
    const size_t mb = (size_t)env_int("BICG_SHM_MB", nullptr, 256);
    g.data_bytes = mb << 20;
    g.total = sizeof(ShmHead) + g.data_bytes;
    atexit(at_exit_cleanup);
    const double t_start = now_s();
    if (g.rank == 0) {
        shm_unlink(g.name.c_str());                       // leftovers of a crashed job (its late joiners detect the swap below)
        int fd = shm_open(g.name.c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
        if (fd < 0 || ftruncate(fd, (off_t)g.total) != 0) { perror("bicgstab_b200: shm_open"); boot_fatal("cannot create the bootstrap segment"); }
        void *map = mmap(nullptr, g.total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        close(fd);
        if (map == MAP_FAILED) { perror("bicgstab_b200: mmap"); boot_fatal("cannot map the bootstrap segment"); }
        g.owner = true;
        g.head = (ShmHead *)map;
        g.data = (char *)map + sizeof(ShmHead);
        g.head->creator_pid = (int)getpid();
        g.head->nonce = ((unsigned long long)getpid() << 32) ^ (unsigned long long)(now_s() * 1e6);
        g.head->magic.store(SHM_READY);
    } else {
        // A segment of this name may be the corpse of a crashed job (magic READY, all tickets gone) that rank 0 is about
        // to unlink and recreate.  Joining = taking one of the world - 1 tickets of a READY segment; a stale segment has
        // none left, so the joiner drops it and re-opens the name until it gets a ticket of the live one.
        for (;;) {
            if (now_s() - t_start > (double)g.timeout_s) boot_fatal("could not join the job's bootstrap segment (is rank 0 running?)");
            int fd = shm_open(g.name.c_str(), O_RDWR, 0600);
            struct stat sb;
            if (fd < 0 || fstat(fd, &sb) != 0 || (size_t)sb.st_size < g.total) { if (fd >= 0) close(fd); usleep(1000); continue; }
            void *map = mmap(nullptr, g.total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
            close(fd);
            if (map == MAP_FAILED) { usleep(1000); continue; }
            ShmHead *h = (ShmHead *)map;
            bool live = false;
            for (int spin = 0; spin < 2000 && !live; ++spin) { live = h->magic.load() == SHM_READY; if (!live) usleep(100); }
            // ... and its creator must still be alive (a job that crashed before everybody joined leaves tickets behind)
            if (live && kill((pid_t)h->creator_pid, 0) != 0 && errno == ESRCH) live = false;
            if (live && h->abort.load() == 0 && h->joined.fetch_add(1) < g.world - 1) {
                g.head = h; g.data = (char *)map + sizeof(ShmHead);
                break;
            }
            munmap(map, g.total);                         // stale or full: wait for rank 0 to replace it
            usleep(5000);
        }
    }
    barrier();
    int rc = bicg_comm_init(g.rank, g.world, shm_allgather, nullptr);
    if (rc != 0) boot_fatal("bicg_comm_init rejected the job geometry");
    // every rank echoes rank 0's nonce: proves that all of them sit in the same (fresh) segment
    unsigned long long mine = g.head->nonce;
    std::string all((size_t)g.world * sizeof(mine), '\0');
    if (shm_allgather(nullptr, &mine, &all[0], sizeof(mine)) != 0) boot_fatal("bootstrap self-test failed");
    for (int p = 0; p < g.world; ++p)
        if (memcmp(&all[(size_t)p * sizeof(mine)], &mine, sizeof(mine)) != 0) boot_fatal("ranks joined different bootstrap segments");
    return 0;
}

void bicg_shm_shutdown(void)
{
    bicg_comm_finalize();
    if (g.world > 1 && g.head) {
        barrier();
        if (g.rank == 0) { g.head->magic.store(0); shm_unlink(g.name.c_str()); g.owner = false; }
    }
}

// ---- include/compat/mpi.h -------------------------------------------------------------------------------
int bicg_shim_MPI_Init(int *, char ***) { return bicg_shm_bootstrap(); }      // failures exit(1) inside
int bicg_shim_MPI_Finalize(void) { fflush(nullptr); bicg_shm_shutdown(); return 0; }
int bicg_shim_MPI_Comm_size(int, int *size) { *size = bicg_comm_world(); return 0; }
int bicg_shim_MPI_Comm_rank(int, int *rank) { *rank = bicg_comm_rank(); return 0; }
int bicg_shim_MPI_Get_processor_name(char *name, int *len)
{
    if (gethostname(name, 127) != 0) strcpy(name, "localhost");
    name[127] = '\0';
    *len = (int)strlen(name);
    return 0;
}
double bicg_shim_MPI_Wtime(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}
int bicg_shim_MPI_Barrier(int) { barrier(); return 0; }
int bicg_shim_MPI_Gather(const void *sbuf, int scount, int st, void *rbuf, int, int, int root, int)
{
    const size_t es = (st == 1) ? 8 : (st == 3) ? 4 : 1;      // MPI_DOUBLE / MPI_INT / MPI_CHAR of compat/mpi.h
    const size_t bytes = es * (size_t)scount;
    const int world = bicg_comm_world();
    if (world == 1) { memcpy(rbuf, sbuf, bytes); return 0; }
    char *tmp = (char *)malloc(bytes * (size_t)world);
    int rc = shm_allgather(nullptr, sbuf, tmp, bytes);
    if (rc == 0 && bicg_comm_rank() == root) memcpy(rbuf, tmp, bytes * (size_t)world);
    free(tmp);
    return rc;
}
int bicg_shim_MPI_Allreduce(const void *sbuf, void *rbuf, int count, int type, int op, int)
{
    if (type != 1 || op != 1) {                                 // MPI_DOUBLE / MPI_SUM of compat/mpi.h
        fprintf(stderr, "bicgstab_b200: MPI_Allreduce supports MPI_DOUBLE with MPI_SUM only (got type %d, op %d)\n", type, op);
        exit(1);
    }
    if (count <= 0) return 0;
    const size_t bytes = (size_t)count * sizeof(double);
    const void *src = (sbuf == (const void *)-1) ? rbuf : sbuf;    // MPI_IN_PLACE
    const int world = bicg_comm_world();
    if (world == 1) { if (src != rbuf) memcpy(rbuf, src, bytes); return 0; }
    double *all = (double *)malloc(bytes * (size_t)world);
    const int rc = shm_allgather(nullptr, src, all, bytes);
    if (rc == 0) {
        double *out = (double *)rbuf;
        for (int i = 0; i < count; ++i) {
            double s = all[i];
            for (int p = 1; p < world; ++p) s += all[(size_t)p * count + i];
            out[i] = s;
        }
    }
    free(all);
    return rc;
}

} // extern "C"
