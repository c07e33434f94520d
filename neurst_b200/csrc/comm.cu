// Data-parallel gradient aggregation inside the library: NCCL all-reduce (sum) of contiguous ranges of the flat fp32
// gradient arena on a dedicated communication stream, issued by the backward pass as soon as a range is final, so the
// transfers over NVLink / NVSwitch run under the remaining backward kernels.
//
// Replaces  HorovodDistributedLossScaleOptimizer._aggregate_gradients (hvd.allreduce, op=Average)
//              neurst/training/hvd_utils.py:48-62
//           MirroredStrategy(cross_device_ops=NcclAllReduce)   neurst/training/distribution_utils.py:73-98
// The 1/replicas of the average is folded into the optimizer's grad_scale.  NCCL is taken from the process (the copy
// PyTorch loads) or the system through dlopen — libb200st has no link-time dependency on it and never touches Horovod / BytePS.
#include "model.cuh"

#include <dlfcn.h>
#include <cstring>
#include <cstdlib>

namespace b200st {

namespace {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitRankConfig)(ncclComm_t*, int, ncclUniqueId, int, void*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  bool ok = false;
};
constexpr int kNcclFloat32 = 7, kNcclSum = 0;      // nccl.h: ncclFloat32 = 7, ncclSum = 0

NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);       // the copy already in the process (PyTorch's)
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return api;
  api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
  api.CommInitRankConfig = reinterpret_cast<decltype(api.CommInitRankConfig)>(dlsym(h, "ncclCommInitRankConfig"));
  api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
  api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(h, "ncclAllReduce"));
  api.Broadcast = reinterpret_cast<decltype(api.Broadcast)>(dlsym(h, "ncclBroadcast"));
  api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
  api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(dlsym(h, "ncclGetVersion"));
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce && api.Broadcast && api.GetErrorString;
  return api;
}
#define B200ST_NCCL(expr)                                                                         \
  do {                                                                                            \
    ncclResult_t _r = (expr);                                                                     \
    if (_r != 0) B200ST_FAIL(std::string(#expr ": ") + nccl().GetErrorString(_r));                \
  } while (0)
}  // namespace

// ncclConfig_t as of NCCL 2.27 (nccl.h: ncclConfig_v22700); newer libraries accept older sizes / versions
struct NcclConfig227 {
  size_t size; unsigned int magic; unsigned int version;
  int blocking, cgaClusterSize, minCTAs, maxCTAs;
  const char* netName;
  int splitShare, trafficClass;
  const char* commName;
  int collnetEnable, CTAPolicy, shrinkShare, nvlsCTAs;
};

// The all-reduces run UNDER the backward kernels: cap the SMs NCCL may take (its kernels hold an SM for the whole
// transfer, and the persistent GEMM grids are sized to the SMs that are left, see comm_reserved_sms)
constexpr int kNcclMaxCtas = 8;

struct GradSync {
  ncclComm_t comm = nullptr;
  int nranks = 1, rank = 0;
  int max_ctas = 0;               // CTAs (= SMs) the communicator may occupy; 0 = NCCL's default
  cudaStream_t cs = nullptr;
  cudaEvent_t ready = nullptr, done = nullptr;
  int64_t reduced_elems = 0;      // of the current backward pass (tests / bench)
  int calls = 0;
};

int comm_unique_id(char* out128) {
  B200ST_CHECK(nccl().ok, "libnccl.so.2 not found in the process or on the system");
  ncclUniqueId id;
  B200ST_NCCL(nccl().GetUniqueId(&id));
  std::memcpy(out128, id.internal, 128);
  return 0;
}

int comm_init(GradSync** out, const char* id128, int nranks, int rank) {
  B200ST_CHECK(nccl().ok, "libnccl.so.2 not found in the process or on the system");
  B200ST_CHECK(nranks >= 1 && rank >= 0 && rank < nranks, "bad rank / world size");
  GradSync* g = new GradSync();
  g->nranks = nranks; g->rank = rank;
  ncclUniqueId id;
  std::memcpy(id.internal, id128, 128);
  ncclResult_t r = 1;
  if (nccl().CommInitRankConfig) {
    NcclConfig227 cfg;
    const int undef = (int)0x80000000;
    cfg.size = sizeof(NcclConfig227); cfg.magic = 0xcafebeefu; cfg.version = 22703u;
    cfg.blocking = undef; cfg.cgaClusterSize = undef; cfg.minCTAs = undef; cfg.maxCTAs = kNcclMaxCtas;
    cfg.netName = nullptr; cfg.splitShare = undef; cfg.trafficClass = undef; cfg.commName = nullptr;
    cfg.collnetEnable = undef; cfg.CTAPolicy = undef; cfg.shrinkShare = undef; cfg.nvlsCTAs = undef;
    r = nccl().CommInitRankConfig(&g->comm, nranks, id, rank, &cfg);
    if (r == 0) g->max_ctas = kNcclMaxCtas;
  }
  if (r != 0) r = nccl().CommInitRank(&g->comm, nranks, id, rank);
  if (r != 0) { delete g; B200ST_FAIL(std::string("ncclCommInitRank: ") + nccl().GetErrorString(r)); }
  if (cudaStreamCreateWithFlags(&g->cs, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&g->ready, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&g->done, cudaEventDisableTiming) != cudaSuccess) {
    nccl().CommDestroy(g->comm);
    delete g;
    B200ST_FAIL("could not create the communication stream / events");
  }
  *out = g;
  return 0;
}

void comm_destroy(GradSync* g) {
  if (!g) return;
  if (g->comm) nccl().CommDestroy(g->comm);
  if (g->cs) cudaStreamDestroy(g->cs);
  if (g->ready) cudaEventDestroy(g->ready);
  if (g->done) cudaEventDestroy(g->done);
  delete g;
}

int comm_world(const GradSync* g) { return g ? g->nranks : 1; }
int comm_reserved_sms(const GradSync* g) { return g ? g->max_ctas : 0; }
int64_t comm_reduced_elems(const GradSync* g) { return g ? g->reduced_elems : 0; }
int comm_calls(const GradSync* g) { return g ? g->calls : 0; }
void comm_begin_step(GradSync* g) { if (g) { g->reduced_elems = 0; g->calls = 0; } }

// grads[lo, hi) is final once everything issued so far on `compute` (and on the optional extra events) has run: fork the
// communication stream from there and all-reduce the range in place.
int comm_reduce_range(GradSync* g, float* grads, int64_t lo, int64_t hi, cudaStream_t compute, cudaEvent_t extra0, cudaEvent_t extra1) {
  if (!g || hi <= lo) return 0;
  B200ST_CUDA(cudaEventRecord(g->ready, compute));
  B200ST_CUDA(cudaStreamWaitEvent(g->cs, g->ready, 0));
  if (extra0) B200ST_CUDA(cudaStreamWaitEvent(g->cs, extra0, 0));
  if (extra1) B200ST_CUDA(cudaStreamWaitEvent(g->cs, extra1, 0));
  B200ST_NCCL(nccl().AllReduce(grads + lo, grads + lo, (size_t)(hi - lo), kNcclFloat32, kNcclSum, g->comm, g->cs));
  g->reduced_elems += hi - lo;
  g->calls += 1;
  return 0;
}
// the consumer of the gradients (optimizer) runs on `compute`: join the communication stream back
int comm_join(GradSync* g, cudaStream_t compute) {
  if (!g) return 0;
  B200ST_CUDA(cudaEventRecord(g->done, g->cs));
  B200ST_CUDA(cudaStreamWaitEvent(compute, g->done, 0));
  return 0;
}
// rank `root` -> all (BroadcastGlobalVariablesCallback, neurst/exps/trainer.py:285)
int comm_broadcast(GradSync* g, float* buf, int64_t n, int root, cudaStream_t compute) {
  if (!g) return 0;
  B200ST_CUDA(cudaEventRecord(g->ready, compute));
  B200ST_CUDA(cudaStreamWaitEvent(g->cs, g->ready, 0));
  B200ST_NCCL(nccl().Broadcast(buf, buf, (size_t)n, kNcclFloat32, root, g->comm, g->cs));
  return comm_join(g, compute);
}

}  // namespace b200st
