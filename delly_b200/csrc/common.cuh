// common.cuh — shared device/host helpers for libdelly_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/dgpu.h"

#define DGPU_NUM_SMS_H100 132

struct DevBuf {  // grow-only device scratch buffer
  void* p = nullptr;
  size_t cap = 0;
};

struct dgpu_ctx {
  int device = 0;
  int num_sms = DGPU_NUM_SMS_H100;
  cudaStream_t stream = nullptr;
  // pipelined host-pointer calls: upload stream, download stream and their events (created on first use)
  cudaStream_t copy_stream = nullptr, out_stream = nullptr;
  std::vector<cudaEvent_t> pipe_events;
  // fork/join pool for independent launches of one batch call (the job classes of longNeedle and of the edit distance): [0] fork event,
  // [1..] join events
  std::vector<cudaStream_t> fork_streams;
  std::vector<cudaEvent_t> fork_events;
  std::string last_error;
  uint64_t launches = 0;
  std::vector<DevBuf> bufs;  // indexed by slot id (see SLOT_* below)
  void* comm = nullptr;      // ncclComm_t when multi-GPU gather is initialised
  int rank = 0, world = 1;
  uint32_t async_bound = 0;  // dgpu_set_async_bound: > 0 = the caller guarantees no sequence is longer; device-form calls then never synchronise
  // dgpu_set_ln_async_bound: > 0 = no longNeedle job exceeds ln_max_cons x ln_max_ref; the device forms then plan on the device inside a
  // workspace pool of ln_pool bytes reserved by the setter, and count their refusals in refused[DGPU_REFUSED_LN]
  uint32_t ln_max_cons = 0, ln_max_ref = 0;
  size_t ln_pool = 0;
  // dgpu_set_ep_async_bound: > 0 = no edit-path job exceeds ep_max_query x ep_max_target; the device forms then plan every Hirschberg level
  // on the device and count their refusals in refused[DGPU_REFUSED_EP]
  uint32_t ep_max_query = 0, ep_max_target = 0;
  // the refusals of the bounded forms per family (device, cumulative, allocated by dgpu_refusals_init); refused_folded[f] of them are
  // already in `unsupported`
  unsigned long long* refused = nullptr;
  unsigned long long refused_folded[2] = {0, 0};
  uint32_t msa_max_reads = 0;  // dgpu_set_msa_async_bound: > 0 = the MSA workspace slots are reserved for clusters of up to this many reads
  bool no_band = false;      // development switch (DGPU_ED_NO_BAND): long NW jobs straight to the full-matrix kernel
  uint64_t unsupported = 0;  // jobs refused per item because they exceed a device limit (dgpu_unsupported_count)
  std::vector<size_t> seg_room;  // seg_rooms (edit_path.cu): the shared memory each seg_kernel class may opt in to, [eq][class], asked once per context
  // optional CUDA-event timing of the dominant kernels of the last batch call
  bool profiling = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool ev_pending = false;
  float last_kernel_ms = 0.f;
};

// Bracket the dominant kernels of a batch call with events on the launching stream.
inline void dgpu_prof_begin(dgpu_ctx* ctx, cudaStream_t st) {
  if (ctx->profiling) cudaEventRecord(ctx->ev0, st);
}
inline void dgpu_prof_end(dgpu_ctx* ctx, cudaStream_t st) {
  if (ctx->profiling) { cudaEventRecord(ctx->ev1, st); ctx->ev_pending = true; }
}

// Scratch slots. No slot is both a staging slot and a workspace slot, so a device form may be called from inside a host form (or
// from another device form) without clobbering what the caller staged.
enum {
  // Staging slots: only DgpuStage (below) reserves these, for the caller's arrays of one host-pointer call.
  SLOT_STAGE_ARENA = 0,  // the sequence arena
  SLOT_STAGE_0,          // every other staged buffer, in the order the host form stages it: its large output buffer (ops / aln / cons,
                         // the cluster-edge columns) first, so that one slot holds it across all host forms
  SLOT_STAGE_END = SLOT_STAGE_0 + 11,
  // Workspace slots: device forms and the functions they call reserve these, each slot only in the files named beside it.
  // Inside one call a slot is re-reserved only after its previous contents are dead.
  SLOT_JOB_PERM = SLOT_STAGE_END,  // job permutation by class (edit_distance.cu, long_needle.cu)
  SLOT_COUNTS,       // class counts (edit_distance.cu, long_needle.cu); rank byte counts (gather.cu); the sink of int_peak.cu
  SLOT_LN_JOBCLS,    // per-job class bytes of longNeedle (long_needle.cu)
  SLOT_ED_STRIPES,   // stripe scratch of long edit-distance targets (edit_distance.cu)
  SLOT_ED_BAND,      // job lists of the banded NW passes (edit_distance.cu)
  SLOT_ED_SLOTS,     // per-job count slot bytes of the edit-distance classification (edit_distance.cu)
  SLOT_ED_PEQ,       // shared Peq tables of target-sharing HW job pairs: hash slots, then one entry per slot (edit_distance.cu)
  SLOT_WAVEFRONT,    // wavefront workspace of the longNeedle and segment engines; their planners count its capacity as free
                     // (long_needle.cu, edit_path.cu)
  SLOT_MSA_SEGJOBS,  // MSA warp workspace (msa.cu); segment job arrays (edit_path.cu)
  SLOT_MSA_LARGE,    // msa_large_kernel's per-CTA workspace, sized from max_reads (msa.cu)
  SLOT_EP_MIRROR,    // edit path: the reversed-sequence mirror of the HW start pass, then the traced leaf ops (edit_path.cu)
  SLOT_EP_TABLE,     // edit path: HW-start target offsets and mirror offsets, then the split selection, then the leaf table (edit_path.cu)
  SLOT_EP_COLS,      // edit path: HW-start target lengths, then the half columns of the split pass (edit_path.cu)
  SLOT_EP_BOUNDS,    // edit path: HW-start bounds and reverse end locations (edit_path.cu)
  SLOT_EP_EQTAB,     // edit path: generalised-equality tables (edit_path.cu)
  SLOT_EP_HROW,      // edit path: per-warp scratch rows of the half columns wider than the wavefront classes (edit_path.cu)
  SLOT_EP_PLAN,      // edit path under dgpu_set_ep_async_bound: the per-job, per-segment and per-level planning arrays (edit_path.cu)
  SLOT_COUNT
};

#define DGPU_FORK_STREAMS 4
int dgpu_fork_init(dgpu_ctx* ctx);  // creates the fork/join pool on first use
int dgpu_set_cuda_error(dgpu_ctx* ctx, cudaError_t e, const char* what);
// Returns device pointer of at least `bytes` bytes in `slot` (contents NOT preserved on growth).
int dgpu_reserve(dgpu_ctx* ctx, int slot, size_t bytes, void** out);
// The families whose bounded forms count refusals on the device: ctx->refused[f].
enum { DGPU_REFUSED_LN = 0, DGPU_REFUSED_EP = 1 };
// Allocates and zeroes ctx->refused on first use (synchronises the context stream).
int dgpu_refusals_init(dgpu_ctx* ctx);
// Adds the longNeedle and edit-path refusals that asynchronous calls counted on the device to ctx->unsupported (synchronises the context
// stream).
int dgpu_fold_refusals(dgpu_ctx* ctx);

#define DGPU_CUDA(ctx, call)                                            \
  do {                                                                  \
    cudaError_t _e = (call);                                            \
    if (_e != cudaSuccess) return dgpu_set_cuda_error((ctx), _e, #call); \
  } while (0)

#define DGPU_LAUNCH_CHECK(ctx, name)                                   \
  do {                                                                 \
    (ctx)->launches++;                                                 \
    cudaError_t _e = cudaGetLastError();                               \
    if (_e != cudaSuccess) return dgpu_set_cuda_error((ctx), _e, name); \
  } while (0)

// Bytes a planner may reserve in workspace `slot`: 60 % of the free device memory (cudaMemGetInfo) plus what the slot already holds.
inline size_t dgpu_workspace_budget(const dgpu_ctx* ctx, int slot, size_t free_bytes) { return (size_t) ((double) free_bytes * 0.6) + ctx->bufs[slot].cap; }

// Independent launches of one batch call, side by side on the context's fork/join pool inside the profiling bracket on `st`. begin() records
// the fork event on st; next() gives launch k pool stream k % DGPU_FORK_STREAMS, whose first launch waits for the fork event; end() makes st
// wait for every pool stream used. A caller that synchronises st therefore sees every result, and last_kernel_ms spans all launches. With
// one launch or none nothing forks and every launch goes on st.
struct DgpuFork {
  dgpu_ctx* ctx;
  cudaStream_t st;
  bool fork;
  int k = 0;  // launches handed out so far
  DgpuFork(dgpu_ctx* c, cudaStream_t s, size_t launches) : ctx(c), st(s), fork(launches > 1) {}
  int begin() {
    int rc;
    if (fork && (rc = dgpu_fork_init(ctx))) return rc;
    dgpu_prof_begin(ctx, st);
    if (fork) DGPU_CUDA(ctx, cudaEventRecord(ctx->fork_events[0], st));
    return DGPU_OK;
  }
  int next(cudaStream_t& cs) {
    cs = fork ? ctx->fork_streams[k % DGPU_FORK_STREAMS] : st;
    if (fork && k < DGPU_FORK_STREAMS) DGPU_CUDA(ctx, cudaStreamWaitEvent(cs, ctx->fork_events[0], 0));
    ++k;
    return DGPU_OK;
  }
  int end() {
    for (int s = 0; fork && s < k && s < DGPU_FORK_STREAMS; ++s) {
      DGPU_CUDA(ctx, cudaEventRecord(ctx->fork_events[1 + s], ctx->fork_streams[s]));
      DGPU_CUDA(ctx, cudaStreamWaitEvent(st, ctx->fork_events[1 + s], 0));
    }
    dgpu_prof_end(ctx, st);
    return DGPU_OK;
  }
};

// Lets `kernel` launch with `smem` bytes of dynamic shared memory (an opt-in above 48 KiB). The opt-in belongs to the kernel on its device,
// not to a context: every host thread with a context on that device shares it. So it is only ever raised, under a lock (ctx.cu), and a thread
// that needs less never lowers it under another thread's launch.
int dgpu_smem_optin_raise(dgpu_ctx* ctx, const void* kernel, size_t smem, const char* name);
template <typename K>
int dgpu_smem_optin(dgpu_ctx* ctx, K* kernel, size_t smem, const char* name) {
  if (smem <= 48 * 1024) return DGPU_OK;
  return dgpu_smem_optin_raise(ctx, (const void*) kernel, smem, name);
}

// The device side of one host-pointer call (a host form of the C ABI): the device and stream, the staged copies of the caller's arrays
// and, with DGPU_TRACE=1, one stderr line per call (name, items, wall ms): where a pipeline stage's time goes, call by call.
// A host form checks the caller's buffers, open()s, stages, runs its _dev form on `st` and finish()es. Buffers take the staging
// slots in the order they are staged; a null host array takes its slot and gives nullptr. A failing step leaves its code in `rc`
// and later steps then do nothing, so one check of `rc` after staging covers them all.
struct DgpuStage {
  const char* name; uint64_t items; double t0 = 0; bool traced = false;
  dgpu_ctx* ctx;
  cudaStream_t st = nullptr, up = nullptr;  // the call's stream (the context stream); the stream uploads go on (st unless changed)
  int rc = DGPU_OK, next = SLOT_STAGE_0;
  struct Back { void* host; const void* dev; size_t bytes; };
  std::vector<Back> back;  // copies for finish()

  DgpuStage(dgpu_ctx* c, const char* nm, uint64_t n);
  ~DgpuStage();
  // every sequence [off[i], off[i] + len[i]), i < n, inside the caller's arena; else DGPU_ERR_ARG, "<name>: a <what> lies outside the arena"
  int check_arena(uint64_t seqs_bytes, uint64_t n, const uint32_t* off, const uint32_t* len, const char* what = "sequence") {
    for (uint64_t i = 0; i < n; ++i)
      if ((uint64_t) off[i] + len[i] > seqs_bytes) { ctx->last_error = std::string(name) + ": a " + what + " lies outside the arena"; return DGPU_ERR_ARG; }
    return DGPU_OK;
  }
  int open() {
    DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
    st = up = ctx->stream;
    return DGPU_OK;
  }
  // the arena, reserved as seqs_bytes + 64 so that 16 bytes past every sequence are readable (include/dgpu.h); seqs == nullptr: no upload
  uint8_t* arena(const uint8_t* seqs, uint64_t seqs_bytes) {
    void* d = nullptr;
    if (!rc) rc = dgpu_reserve(ctx, SLOT_STAGE_ARENA, seqs_bytes + 64, &d);
    if (seqs) upload(d, seqs, seqs_bytes);
    return rc ? nullptr : (uint8_t*) d;
  }
  template <class T> T* alloc(size_t count) {  // the next staging slot
    void* d = nullptr;
    if (!rc && next >= SLOT_STAGE_END) { ctx->last_error = "DgpuStage: too many staged buffers"; rc = DGPU_ERR_ARG; }
    if (!rc) rc = dgpu_reserve(ctx, next++, count * sizeof(T), &d);
    return rc ? nullptr : (T*) d;
  }
  void upload(void* dev, const void* host, size_t bytes) {  // on `up`
    cudaError_t e = rc ? cudaSuccess : cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, up);
    if (e != cudaSuccess) rc = dgpu_set_cuda_error(ctx, e, "cudaMemcpyAsync(host to device)");
  }
  template <class T> T* in(const T* host, size_t count) {
    T* d = host ? alloc<T>(count) : (++next, nullptr);
    if (host) upload(d, host, count * sizeof(T));
    return d;
  }
  template <class T> T* out(T* host, size_t count, size_t pad = 0) {  // copied back into `host` by finish(); `pad` more elements reserved
    T* d = host ? alloc<T>(count + pad) : (++next, nullptr);
    if (host && !rc) back.push_back(Back{host, d, count * sizeof(T)});
    return d;
  }
  int finish() {  // the copies back, in the order they were staged, then a synchronise of `st`
    for (Back const& b : back) DGPU_CUDA(ctx, cudaMemcpyAsync(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost, st));
    DGPU_CUDA(ctx, cudaStreamSynchronize(st));
    return DGPU_OK;
  }
};

// ---- unaligned 16-byte chunk reader over a byte arena -------------------------------
// Reads sequence bytes [16*j, 16*j+16) of the sequence starting at `p` regardless of the
// alignment of p, with two aligned LDG.128 and PRMT realignment. Loads are clamped to the
// 16-byte blocks that contain at least one arena byte (arena_end = one past last byte).
struct ChunkReader {
  const uint4* base;   // aligned-down pointer
  uint32_t shift;      // misalignment in bytes (0..15)
  const uint8_t* end;  // arena end
  uint4 cur;           // aligned block j (already loaded)
  uint32_t j;

  __device__ __forceinline__ uint4 load(uint32_t idx) const {
    const uint4* a = base + idx;
    if ((const uint8_t*) a < end) return __ldg(a);
    return make_uint4(0, 0, 0, 0);
  }
  __device__ __forceinline__ void init(const uint8_t* p, const uint8_t* arena_end) {
    uintptr_t u = (uintptr_t) p;
    shift = (uint32_t) (u & 15);
    base = (const uint4*) (u - shift);
    end = arena_end;
    j = 0;
    cur = load(0);
  }
  // returns bytes [16j,16j+16) of the sequence and advances
  __device__ __forceinline__ uint4 next() {
    uint4 nxt = load(j + 1);
    uint4 r;
    if (shift == 0) {
      r = cur;
    } else {
      uint32_t w[8] = {cur.x, cur.y, cur.z, cur.w, nxt.x, nxt.y, nxt.z, nxt.w};
      uint32_t ws = shift >> 2, bs = (shift & 3) * 8;
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // dynamic word index resolved with selects (ws in 0..3)
        uint32_t lo = ws == 0 ? w[i] : ws == 1 ? w[i + 1] : ws == 2 ? w[i + 2] : w[i + 3];
        uint32_t hi = ws == 0 ? w[i + 1] : ws == 1 ? w[i + 2] : ws == 2 ? w[i + 3] : w[i + 4];
        o[i] = __funnelshift_r(lo, hi, bs);
      }
      r = make_uint4(o[0], o[1], o[2], o[3]);
    }
    cur = nxt;
    ++j;
    return r;
  }
};

// DNA byte -> code: A0 C1 G2 T3 N4, anything else 5 (exact byte equality is preserved by
// routing code 5 through an exact slow path in every kernel).
__device__ __forceinline__ uint32_t dna_code(uint32_t c) {
  uint32_t x = (c >> 1) & 3u;                           // A:0 C:1 T:2 G:3
  uint32_t expect = (0x47544341u >> (x * 8)) & 0xffu;   // 'A','C','T','G'
  uint32_t code = x ^ (x >> 1);                         // ->A0 C1 T3 G2
  return (c == expect) ? code : (c == 'N' ? 4u : 5u);
}
