/*
 * compat/mpi.h -- the seven MPI calls the reference's main.c makes (main.c:14-28, 90-92, 150), plus the MPI_Allreduce of
 * test_shifted.c's DISPLAY_ERROR check, mapped onto libbicgstab_b200.so so that main.c compiles and links UNCHANGED on a box
 * without MPI:
 *
 *     gcc -O2 -Iinclude/compat -I<reference>/src <reference>/src/main.c -Lmpi-bicgstab_b200 -lbicgstab_b200 -o solver
 *
 * One process = one rank = one GPU.  Launch P processes with RANK / WORLD_SIZE / LOCAL_RANK in the
 * environment (tools/bicgrun does it; torchrun's variables are understood as well); with none of them set
 * the program is a single rank.  MPI_Init() bootstraps the library's communicator through a POSIX
 * shared-memory segment (csrc/shm_boot.cpp) -- the GPUs themselves then talk over NVLink peer memory.
 *
 * Everything else in <mpi.h> that the reference uses lives in solver.c / matrix.c, which this library
 * replaces, so nothing else is needed here.  The names are macro-mapped to a private prefix so a real MPI
 * in the same process cannot collide.
 */
#ifndef BICG_COMPAT_MPI_H
#define BICG_COMPAT_MPI_H
#ifdef __cplusplus
extern "C" {
#endif

typedef int MPI_Comm;
typedef int MPI_Datatype;
typedef int MPI_Op;
typedef int MPI_Request;
typedef struct { int MPI_SOURCE, MPI_TAG, MPI_ERROR; } MPI_Status;

#define MPI_COMM_WORLD 0
#define MPI_DOUBLE 1
#define MPI_CHAR 2
#define MPI_INT 3
#define MPI_SUM 1
#define MPI_SUCCESS 0
#define MPI_MAX_PROCESSOR_NAME 128
#define MPI_IN_PLACE ((void *)-1)
#define MPI_STATUS_IGNORE ((MPI_Status *)0)

#define MPI_Init               bicg_shim_MPI_Init
#define MPI_Finalize           bicg_shim_MPI_Finalize
#define MPI_Comm_size          bicg_shim_MPI_Comm_size
#define MPI_Comm_rank          bicg_shim_MPI_Comm_rank
#define MPI_Get_processor_name bicg_shim_MPI_Get_processor_name
#define MPI_Wtime              bicg_shim_MPI_Wtime
#define MPI_Gather             bicg_shim_MPI_Gather
#define MPI_Barrier            bicg_shim_MPI_Barrier
#define MPI_Allreduce          bicg_shim_MPI_Allreduce

int    MPI_Init(int *argc, char ***argv);
int    MPI_Finalize(void);
int    MPI_Comm_size(MPI_Comm comm, int *size);
int    MPI_Comm_rank(MPI_Comm comm, int *rank);
int    MPI_Get_processor_name(char *name, int *len);
double MPI_Wtime(void);
int    MPI_Gather(const void *sbuf, int scount, MPI_Datatype st, void *rbuf, int rcount, MPI_Datatype rt,
                  int root, MPI_Comm comm);
int    MPI_Barrier(MPI_Comm comm);
/* MPI_DOUBLE + MPI_SUM only (sendbuf may be MPI_IN_PLACE): the sums are added in rank order, so every rank gets the same
 * bits.  The DISPLAY_ERROR block of test_shifted.c uses it.  Any other type or op: message + exit(1). */
int    MPI_Allreduce(const void *sendbuf, void *recvbuf, int count, MPI_Datatype type, MPI_Op op, MPI_Comm comm);

#ifdef __cplusplus
}
#endif
#endif
