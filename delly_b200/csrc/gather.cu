// gather.cu — the one exchange step of the multi-GPU path (SURVEY §8e, §8b `dgpu_gather_records`): an all-gatherv of each rank's
// finished call records before BCF emission, over the NCCL C API.
//
// Reference context: the reference is a single process; its SV list is assembled in discovery order, then `sort(svs)` and renumbered
// (src/delly.h:155-158, src/tegua.h:149-156) before vcfOutput. With the SV list sharded over ranks (contiguous id ranges, one process per
// GPU) every rank finishes its own records; this call concatenates the serialised records of all ranks IN RANK ORDER on every rank, which
// — because the shards are contiguous ranges of the reference's order — is the reference's order again (host/gather.hpp restores ids).
//
// Wire protocol: ncclAllGather of one uint64 byte count per rank, then a grouped ncclBroadcast per rank of exactly its payload
// (an all-gatherv; no padding travels). Payloads are a few bytes to tens of MB (≤ ~50 MB per genome, SURVEY §8e), so the exchange is
// latency-bound: one NVLink/NVSwitch round for the counts and one for the payloads.
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): single-GPU users of libdelly_b200.so do not need NCCL installed, and inside a
// torch process the already-loaded NCCL (same soname) is the one that is used.
#include "common.cuh"
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <mutex>

namespace {

// the handful of NCCL entry points used, with the signatures of nccl.h (2.x ABI)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;   // ncclSuccess = 0
enum { NCCL_UINT8 = 1, NCCL_UINT64 = 5 };   // ncclDataType_t: ncclInt8 0, ncclUint8 1, ncclInt32 2, ncclUint32 3, ncclInt64 4, ncclUint64 5

struct Nccl {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommCount)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*CommUserRank)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  bool ok = false;
};

Nccl& nccl() {
  static Nccl n;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) { n.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (n.h) break; }
    if (!n.h) return;
    auto sym = [&](const char* s) { return dlsym(n.h, s); };
    n.GetUniqueId = (decltype(n.GetUniqueId)) sym("ncclGetUniqueId");
    n.CommInitRank = (decltype(n.CommInitRank)) sym("ncclCommInitRank");
    n.CommDestroy = (decltype(n.CommDestroy)) sym("ncclCommDestroy");
    n.CommCount = (decltype(n.CommCount)) sym("ncclCommCount");
    n.CommUserRank = (decltype(n.CommUserRank)) sym("ncclCommUserRank");
    n.AllGather = (decltype(n.AllGather)) sym("ncclAllGather");
    n.Broadcast = (decltype(n.Broadcast)) sym("ncclBroadcast");
    n.GroupStart = (decltype(n.GroupStart)) sym("ncclGroupStart");
    n.GroupEnd = (decltype(n.GroupEnd)) sym("ncclGroupEnd");
    n.GetErrorString = (decltype(n.GetErrorString)) sym("ncclGetErrorString");
    n.GetVersion = (decltype(n.GetVersion)) sym("ncclGetVersion");
    n.ok = n.GetUniqueId && n.CommInitRank && n.CommDestroy && n.CommCount && n.CommUserRank && n.AllGather && n.Broadcast && n.GroupStart && n.GroupEnd &&
           n.GetErrorString;
  });
  return n;
}

int nccl_fail(dgpu_ctx* ctx, ncclResult_t r, const char* what) {
  if (ctx) ctx->last_error = std::string(what) + ": " + (nccl().GetErrorString ? nccl().GetErrorString(r) : "NCCL error");
  return DGPU_ERR_NCCL;
}
#define DGPU_NCCL(ctx, call, what) do { ncclResult_t r_ = (call); if (r_ != 0) return nccl_fail((ctx), r_, (what)); } while (0)

int need_nccl(dgpu_ctx* ctx) {
  if (nccl().ok) return DGPU_OK;
  if (ctx) ctx->last_error = "libnccl.so.2 could not be loaded (multi-GPU gather needs NCCL)";
  return DGPU_ERR_NCCL;
}

}  // namespace

extern "C" {

// ncclGetUniqueId: rank 0 calls this and distributes the 128 bytes to the other ranks out of band (MPI, torch.distributed, a file, ...)
// The exchange moves a few MB of records once or twice per run: two channels are plenty and the in-switch reduction engine (NVLS) is of no use to an
// all-gather, while setting both up is a good part of the communicator's start-up time (2-rank run of the reference's example: 3.7 s -> 2.7 s,
// tools/nccl_init_probe.py). Defaults only — a variable the user has set wins.
static void nccl_defaults() {
  setenv("NCCL_NVLS_ENABLE", "0", 0);
  setenv("NCCL_MAX_NCHANNELS", "2", 0);
  setenv("NCCL_MIN_NCHANNELS", "1", 0);
}

int dgpu_comm_unique_id(uint8_t* id128) {
  if (!id128) return DGPU_ERR_ARG;
  nccl_defaults();
  int rc = need_nccl(nullptr);
  if (rc) return rc;
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != 0) return DGPU_ERR_NCCL;
  memcpy(id128, id.internal, 128);
  return DGPU_OK;
}

// ncclCommInitRank on the context's device; collective over all ranks. The communicator is remembered in the context (rank / world).
int dgpu_comm_init(dgpu_ctx* ctx, int nranks, int rank, const uint8_t* id128, void** comm) {
  if (!ctx || !id128 || !comm || nranks < 1 || rank < 0 || rank >= nranks) return DGPU_ERR_ARG;
  nccl_defaults();
  int rc = need_nccl(ctx);
  if (rc) return rc;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  ncclUniqueId id;
  memcpy(id.internal, id128, 128);
  ncclComm_t c = nullptr;
  DGPU_NCCL(ctx, nccl().CommInitRank(&c, nranks, id, rank), "ncclCommInitRank");
  ctx->comm = c; ctx->rank = rank; ctx->world = nranks;
  *comm = c;
  return DGPU_OK;
}

int dgpu_comm_destroy(dgpu_ctx* ctx, void* comm) {
  if (!comm) return DGPU_OK;
  int rc = need_nccl(ctx);
  if (rc) return rc;
  if (ctx) { cudaSetDevice(ctx->device); cudaStreamSynchronize(ctx->stream); if (ctx->comm == comm) { ctx->comm = nullptr; ctx->rank = 0; ctx->world = 1; } }
  DGPU_NCCL(ctx, nccl().CommDestroy((ncclComm_t) comm), "ncclCommDestroy");
  return DGPU_OK;
}

int dgpu_nccl_version(void) {
  if (!nccl().ok || !nccl().GetVersion) return 0;
  int v = 0;
  return nccl().GetVersion(&v) == 0 ? v : 0;
}

void dgpu_free_host(void* p) { free(p); }

// All-gatherv of host byte payloads over `comm` (an ncclComm_t whose ranks each own one dgpu_ctx / GPU).
//   local / local_bytes : this rank's serialised records (host memory; may be empty)
//   *all                : malloc'd by the callee: the payloads of ranks 0..n-1 back to back (release with dgpu_free_host)
//   *counts             : malloc'd by the callee: n byte counts
//   *nranks             : n
// comm == NULL is the single-process case: the output is a copy of the input (n = 1), no NCCL needed.
// Timing (when profiling is on): dgpu_last_kernel_ms() = device time of the two collectives.
int dgpu_gather_records(dgpu_ctx* ctx, void* comm, const void* local, uint64_t local_bytes, void** all, uint64_t** counts, int* nranks) {
  if (!ctx || !all || !counts || !nranks || (local_bytes && !local)) return DGPU_ERR_ARG;
  *all = nullptr; *counts = nullptr; *nranks = 0;
  if (!comm) {
    uint64_t* c = (uint64_t*) malloc(sizeof(uint64_t));
    void* a = malloc(local_bytes ? local_bytes : 1);
    if (!c || !a) { free(c); free(a); return DGPU_ERR_CAPACITY; }
    c[0] = local_bytes;
    if (local_bytes) memcpy(a, local, local_bytes);
    *all = a; *counts = c; *nranks = 1;
    return DGPU_OK;
  }
  int rc = need_nccl(ctx);
  if (rc) return rc;
  DgpuStage s(ctx, "dgpu_gather_records", local_bytes);
  if ((rc = s.open())) return rc;
  cudaStream_t st = s.st;
  ncclComm_t c = (ncclComm_t) comm;
  int n = 0, me = 0;
  DGPU_NCCL(ctx, nccl().CommCount(c, &n), "ncclCommCount");
  DGPU_NCCL(ctx, nccl().CommUserRank(c, &me), "ncclCommUserRank");
  void* d_cnt;
  if ((rc = dgpu_reserve(ctx, SLOT_COUNTS, (size_t) (n + 1) * sizeof(uint64_t) + 1024, &d_cnt))) return rc;
  uint64_t* dc = (uint64_t*) d_cnt;   // [0..n-1] gathered counts, [n] this rank's count
  dgpu_prof_begin(ctx, st);
  DGPU_CUDA(ctx, cudaMemcpyAsync(dc + n, &local_bytes, sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  DGPU_NCCL(ctx, nccl().AllGather(dc + n, dc, 1, NCCL_UINT64, c, st), "ncclAllGather(counts)");
  ++ctx->launches;
  uint64_t* hc = (uint64_t*) malloc((size_t) n * sizeof(uint64_t));
  if (!hc) return DGPU_ERR_CAPACITY;
  cudaError_t e = cudaMemcpyAsync(hc, dc, (size_t) n * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { free(hc); return dgpu_set_cuda_error(ctx, e, "gather counts"); }
  uint64_t total = 0;
  for (int r = 0; r < n; ++r) total += hc[r];
  void* ha = malloc(total ? total : 1);
  if (!ha) { free(hc); return DGPU_ERR_CAPACITY; }
  if (total) {
    uint8_t *d_local = s.alloc<uint8_t>(local_bytes + 16), *d_all = s.alloc<uint8_t>(total + 16);
    if (s.rc) { free(hc); free(ha); return s.rc; }
    if (local_bytes) e = cudaMemcpyAsync(d_local, local, local_bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { free(hc); free(ha); return dgpu_set_cuda_error(ctx, e, "gather H2D"); }
    ncclResult_t r0 = nccl().GroupStart();
    uint64_t off = 0;
    for (int r = 0; r < n && r0 == 0; ++r) {
      if (hc[r]) r0 = nccl().Broadcast(d_local, d_all + off, (size_t) hc[r], NCCL_UINT8, r, c, st);
      off += hc[r];
    }
    ncclResult_t r1 = nccl().GroupEnd();
    if (r0 != 0 || r1 != 0) { free(hc); free(ha); return nccl_fail(ctx, r0 ? r0 : r1, "ncclBroadcast (all-gatherv)"); }
    ++ctx->launches;
    e = cudaMemcpyAsync(ha, d_all, total, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) { free(hc); free(ha); return dgpu_set_cuda_error(ctx, e, "gather D2H"); }
  }
  dgpu_prof_end(ctx, st);
  e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { free(hc); free(ha); return dgpu_set_cuda_error(ctx, e, "gather sync"); }
  *all = ha; *counts = hc; *nranks = n;
  return DGPU_OK;
}

}  // extern "C"
