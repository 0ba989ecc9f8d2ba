// Collectives of the cluster-sharded solve, called from C on the library's stream.
//
// NCCL is bound at run time (dlopen/dlsym), not at link time: a host that never shards never needs
// it, and inside a PyTorch process the library must use the NCCL that process already carries
// (torch bundles its own libnccl.so.2) instead of pulling a second copy in.  Resolution order:
// an already loaded libnccl.so.2, $DIRAC_B200_NCCL_LIB, libnccl.so.2, libnccl.so.
//
// The reference merges its two GPUs' results on the host under a pthread barrier
// (lmfit_cuda.c:1544-1580,1801-1950); here every exchange is one ncclAllReduce(sum, fp64, in place)
// over NVLink / NVSwitch, enqueued behind the kernels that produced the buffer.
#include <dlfcn.h>
#include <string.h>
#include <time.h>

#include "../../include/dirac_b200.h"
#include "problem.h"

typedef struct { char internal[128]; } db_ncclUniqueId;  // ncclUniqueId, nccl.h
typedef void *db_ncclComm_t;
enum { DB_NCCL_DOUBLE = 8, DB_NCCL_SUM = 0 };            // ncclFloat64, ncclSum

static struct {
  void *lib;
  int (*GetUniqueId)(db_ncclUniqueId *);
  int (*CommInitRank)(db_ncclComm_t *, int, db_ncclUniqueId, int);
  int (*CommDestroy)(db_ncclComm_t);
  int (*AllReduce)(const void *, void *, size_t, int, int, db_ncclComm_t, cudaStream_t);
  const char *(*GetErrorString)(int);
  db_ncclComm_t comm;
  int rank, world;
} g_nccl;

static double g_comm_seconds = 0.0;   // host time spent enqueueing collectives
static unsigned long long g_comm_calls = 0, g_comm_bytes = 0;

static int nccl_bind() {
  if (g_nccl.lib) return 0;
  void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
  const char *env = getenv("DIRAC_B200_NCCL_LIB");
  if (!h && env) h = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    fprintf(stderr, "dirac_b200: cannot load NCCL (%s); set DIRAC_B200_NCCL_LIB\n", dlerror());
    return -1;
  }
  *(void **)&g_nccl.GetUniqueId = dlsym(h, "ncclGetUniqueId");
  *(void **)&g_nccl.CommInitRank = dlsym(h, "ncclCommInitRank");
  *(void **)&g_nccl.CommDestroy = dlsym(h, "ncclCommDestroy");
  *(void **)&g_nccl.AllReduce = dlsym(h, "ncclAllReduce");
  *(void **)&g_nccl.GetErrorString = dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllReduce) {
    fprintf(stderr, "dirac_b200: the NCCL library lacks a required symbol\n");
    return -1;
  }
  g_nccl.lib = h;
  return 0;
}

#define NCCL_CHECK(call)                                                                     \
  do {                                                                                       \
    int r__ = (call);                                                                        \
    if (r__ != 0) {                                                                          \
      fprintf(stderr, "dirac_b200: NCCL error %d (%s) at %s:%d\n", r__,                      \
              g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "?", __FILE__, __LINE__); \
      exit(1);                                                                               \
    }                                                                                        \
  } while (0)

// rank 0 draws the 128-byte id; the host hands it to every rank (MPI_Bcast, a file, a TCP store)
extern "C" int dirac_b200_nccl_unique_id(char *id128) {
  if (nccl_bind()) return -1;
  db_ncclUniqueId id;
  NCCL_CHECK(g_nccl.GetUniqueId(&id));
  memcpy(id128, id.internal, 128);
  return 0;
}

// collective over all ranks: binds the current CUDA device of the calling process to `rank`
extern "C" int dirac_b200_nccl_init(int rank, int world, const char *id128) {
  if (nccl_bind()) return -1;
  if (g_nccl.comm) {
    g_nccl.CommDestroy(g_nccl.comm);
    g_nccl.comm = nullptr;
  }
  db_ncclUniqueId id;
  memcpy(id.internal, id128, 128);
  NCCL_CHECK(g_nccl.CommInitRank(&g_nccl.comm, world, id, rank));
  g_nccl.rank = rank;
  g_nccl.world = world;
  return 0;
}

extern "C" void dirac_b200_nccl_finalize(void) {
  if (g_nccl.comm) {
    cudaDeviceSynchronize();
    g_nccl.CommDestroy(g_nccl.comm);
    g_nccl.comm = nullptr;
  }
}

extern "C" int dirac_b200_nccl_ready(void) { return g_nccl.comm != nullptr; }

// sum a device buffer of doubles over the ranks (no-op for a single rank); enqueued on the stream
void db_allreduce(dirac_b200_problem *pr, void *dev, long long count) {
  if (pr->world <= 1 || count <= 0) return;
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  if (pr->allreduce) {
    pr->allreduce(dev, count, (void *)pr->d.stream, pr->comm_user);
  } else {
    if (!g_nccl.comm || g_nccl.world != pr->world) {
      fprintf(stderr, "dirac_b200: sharded problem (world %d) without a communicator: call "
                      "dirac_b200_nccl_init or supply a callback to dirac_b200_set_comm\n", pr->world);
      exit(1);
    }
    NCCL_CHECK(g_nccl.AllReduce(dev, dev, (size_t)count, DB_NCCL_DOUBLE, DB_NCCL_SUM, g_nccl.comm,
                                pr->d.stream));
  }
  clock_gettime(CLOCK_MONOTONIC, &t1);
  g_comm_seconds += (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  g_comm_calls++;
  g_comm_bytes += (unsigned long long)count * 8ull;
}

void db_allreduce_world(dirac_b200_problem *pr, void *dev, long long count) {
  if (count <= 0) return;
  if (pr->allreduce) {
    pr->allreduce(dev, count, (void *)pr->d.stream, pr->comm_user);
    g_comm_calls++;
    g_comm_bytes += (unsigned long long)count * 8ull;
  } else if (g_nccl.comm && g_nccl.world > 1) {
    NCCL_CHECK(g_nccl.AllReduce(dev, dev, (size_t)count, DB_NCCL_DOUBLE, DB_NCCL_SUM, g_nccl.comm,
                                pr->d.stream));
    g_comm_calls++;
    g_comm_bytes += (unsigned long long)count * 8ull;
  }
}

// the size of the communicator of dirac_b200_nccl_init (0: none)
int db_nccl_world() { return g_nccl.comm ? g_nccl.world : 0; }

// sum a device buffer of doubles over the ranks through the host's callback, or the communicator of
// dirac_b200_nccl_init when there is none; enqueued on st
void db_allreduce_stream(dirac_b200_allreduce_fn fn, void *user, void *dev, long long count,
                         cudaStream_t st) {
  if (count <= 0) return;
  if (fn) {
    fn(dev, count, (void *)st, user);
  } else {
    if (!g_nccl.comm) {
      fprintf(stderr, "dirac_b200: an exchange without a callback or a communicator\n");
      exit(1);
    }
    NCCL_CHECK(g_nccl.AllReduce(dev, dev, (size_t)count, DB_NCCL_DOUBLE, DB_NCCL_SUM, g_nccl.comm, st));
  }
  g_comm_calls++;
  g_comm_bytes += (unsigned long long)count * 8ull;
}

// ---- overlapped exchange: all-reduces on a communication stream of the library, grouped ----------
// Used where a streaming kernel is followed by a large all-reduce of what it wrote (the LBFGS line
// model: three visibility-sized vectors per iteration): the kernel is launched in time chunks and
// every chunk's slices are summed over the ranks on a second stream while the next chunk is computed,
// so the NVLink transfer runs behind the math instead of after it.
static cudaStream_t g_comm_stream = nullptr;
int db_overlap_available(const dirac_b200_problem *pr) {
  return pr->world > 1 && !pr->allreduce && g_nccl.comm && g_nccl.world == pr->world &&
         !getenv("DIRAC_B200_NO_OVERLAP");
}
cudaStream_t db_comm_stream() {
  if (!g_comm_stream) DB_CHECK(cudaStreamCreateWithFlags(&g_comm_stream, cudaStreamNonBlocking));
  return g_comm_stream;
}
static int (*p_GroupStart)() = nullptr;
static int (*p_GroupEnd)() = nullptr;
// sums `nseg` device segments (ptr[i], count[i] doubles) over the ranks as ONE grouped NCCL operation
void db_allreduce_segments(dirac_b200_problem *pr, double **ptr, const long long *count, int nseg,
                           cudaStream_t st) {
  if (!p_GroupStart) {
    *(void **)&p_GroupStart = dlsym(g_nccl.lib, "ncclGroupStart");
    *(void **)&p_GroupEnd = dlsym(g_nccl.lib, "ncclGroupEnd");
  }
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  if (p_GroupStart && p_GroupEnd) NCCL_CHECK(p_GroupStart());
  for (int i = 0; i < nseg; i++) {
    NCCL_CHECK(g_nccl.AllReduce(ptr[i], ptr[i], (size_t)count[i], DB_NCCL_DOUBLE, DB_NCCL_SUM,
                                g_nccl.comm, st));
    g_comm_bytes += (unsigned long long)count[i] * 8ull;
  }
  if (p_GroupStart && p_GroupEnd) NCCL_CHECK(p_GroupEnd());
  clock_gettime(CLOCK_MONOTONIC, &t1);
  g_comm_seconds += (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  g_comm_calls++;
}

// host-side accounting of the collectives since the last reset: calls, bytes, seconds spent enqueueing
extern "C" void dirac_b200_comm_stats(unsigned long long *calls, unsigned long long *bytes,
                                      double *enqueue_seconds, int reset) {
  if (calls) *calls = g_comm_calls;
  if (bytes) *bytes = g_comm_bytes;
  if (enqueue_seconds) *enqueue_seconds = g_comm_seconds;
  if (reset) {
    g_comm_calls = g_comm_bytes = 0;
    g_comm_seconds = 0.0;
  }
}

// ---- host waits ------------------------------------------------------------------------------------
static double g_wait_seconds = 0.0;
static unsigned long long g_wait_calls = 0;
static inline double now_s() {
  struct timespec t;
  clock_gettime(CLOCK_MONOTONIC, &t);
  return (double)t.tv_sec + 1e-9 * (double)t.tv_nsec;
}
void db_stream_sync(cudaStream_t st) {
  const double t0 = now_s();
  DB_CHECK(cudaStreamSynchronize(st));
  g_wait_seconds += now_s() - t0;
  g_wait_calls++;
}
// wait until a kernel's last CTA has published `epoch` in host-mapped memory (its results, written
// to the same mapping before a system-wide fence, are then visible).  The stream is polled now and
// then so that a failed launch ends in the usual error exit instead of an endless spin.
void db_flag_wait(const volatile unsigned long long *flag, unsigned long long epoch,
                  cudaStream_t st) {
  const double t0 = now_s();
  unsigned spins = 0;
  while (*flag != epoch) {
    if ((++spins & 0x3fff) == 0) {
      cudaError_t e = cudaStreamQuery(st);
      if (e == cudaSuccess) {
        if (*flag != epoch) {  // kernel done without publishing: cannot happen, do not spin on it
          fprintf(stderr, "dirac_b200: result flag not published\n");
          exit(1);
        }
      } else if (e != cudaErrorNotReady) {
        DB_CHECK(e);
      }
    }
  }
  g_wait_seconds += now_s() - t0;
  g_wait_calls++;
}
void db_event_sync(cudaEvent_t ev) {
  const double t0 = now_s();
  DB_CHECK(cudaEventSynchronize(ev));
  g_wait_seconds += now_s() - t0;
  g_wait_calls++;
}
// host synchronisations since the last reset and the seconds the host spent blocked in them
extern "C" void dirac_b200_host_stats(unsigned long long *syncs, double *wait_seconds, int reset) {
  if (syncs) *syncs = g_wait_calls;
  if (wait_seconds) *wait_seconds = g_wait_seconds;
  if (reset) {
    g_wait_calls = 0;
    g_wait_seconds = 0.0;
  }
}
