// ctx.cu — context, error plumbing and scratch-buffer management for libdelly_b200.
#include "common.cuh"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

int dgpu_set_cuda_error(dgpu_ctx* ctx, cudaError_t e, const char* what) {
  if (ctx) {
    char buf[512];
    snprintf(buf, sizeof(buf), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
    ctx->last_error = buf;
  }
  cudaGetLastError();  // clear sticky-less errors
  return DGPU_ERR_CUDA;
}

int dgpu_reserve(dgpu_ctx* ctx, int slot, size_t bytes, void** out) {
  DevBuf& b = ctx->bufs[slot];
  if (bytes > b.cap) {
    // cudaFree synchronises the device. Callers rely on that: the edit distance's class kernels of an earlier call may still read a slot
    // from the fork/join streams, and a stream-ordered free would release the buffer under them.
    if (b.p) DGPU_CUDA(ctx, cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = bytes + (bytes >> 2) + 4096;  // 25 % headroom: batches arrive at similar sizes
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
      cudaGetLastError();
      want = bytes + 256;
      e = cudaMalloc(&b.p, want);
      if (e != cudaSuccess) return dgpu_set_cuda_error(ctx, e, "cudaMalloc(scratch)");
    }
    b.cap = want;
  }
  *out = b.p;
  return DGPU_OK;
}

int dgpu_smem_optin_raise(dgpu_ctx* ctx, const void* kernel, size_t smem, const char* name) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> granted;   // (kernel, device) -> the opt-in set so far
  std::lock_guard<std::mutex> g(mu);
  size_t& have = granted[std::make_pair(kernel, ctx->device)];
  if (smem <= have) return DGPU_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return dgpu_set_cuda_error(ctx, e, name);
  have = smem;
  return DGPU_OK;
}

int dgpu_refusals_init(dgpu_ctx* ctx) {
  if (ctx->refused) return DGPU_OK;
  DGPU_CUDA(ctx, cudaMalloc(&ctx->refused, 2 * sizeof(unsigned long long)));
  DGPU_CUDA(ctx, cudaMemsetAsync(ctx->refused, 0, 2 * sizeof(unsigned long long), ctx->stream));
  DGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return DGPU_OK;
}

int dgpu_fold_refusals(dgpu_ctx* ctx) {
  if (!ctx->refused) return DGPU_OK;
  unsigned long long v[2];
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  DGPU_CUDA(ctx, cudaMemcpyAsync(v, ctx->refused, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
  DGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int f = 0; f < 2; ++f) {
    if (v[f] <= ctx->refused_folded[f]) continue;
    const unsigned long long d = v[f] - ctx->refused_folded[f];
    ctx->unsupported += d;
    ctx->refused_folded[f] = v[f];
    if (f == DGPU_REFUSED_LN)
      ctx->last_error = "dgpu_long_needle[_ex]_dev: " + std::to_string(d) + " job(s) beyond the asynchronous bound (" + std::to_string(ctx->ln_max_cons) +
                        " x " + std::to_string(ctx->ln_max_ref) + ") or the device limits were not aligned (ok = 0)";
    else
      ctx->last_error = "dgpu_edit_path[_ex|_wide]_dev: " + std::to_string(d) + " job(s) beyond the asynchronous bound (" +
                        std::to_string(ctx->ep_max_query) + " x " + std::to_string(ctx->ep_max_target) + ") were not aligned (status 4)";
  }
  return DGPU_OK;
}

int dgpu_fork_init(dgpu_ctx* ctx) {
  while (ctx->fork_streams.size() < DGPU_FORK_STREAMS) {
    cudaStream_t s;
    DGPU_CUDA(ctx, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    ctx->fork_streams.push_back(s);
  }
  while (ctx->fork_events.size() < 1 + DGPU_FORK_STREAMS) {
    cudaEvent_t e;
    DGPU_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->fork_events.push_back(e);
  }
  return DGPU_OK;
}

extern "C" {

int dgpu_version(void) { return 1005; }

int dgpu_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return DGPU_ERR_NODEVICE; }
  return n;
}

const char* dgpu_strerror(int code) {
  switch (code) {
    case DGPU_OK: return "ok";
    case DGPU_ERR_CUDA: return "CUDA runtime error";
    case DGPU_ERR_ARG: return "invalid argument";
    case DGPU_ERR_NODEVICE: return "no usable CUDA device (this library has no CPU fallback)";
    case DGPU_ERR_CAPACITY: return "capacity exceeded";
    case DGPU_ERR_UNSUPPORTED: return "unsupported shape";
    case DGPU_ERR_NCCL: return "NCCL error";
    default: return "unknown error";
  }
}

int dgpu_ctx_create(int device, dgpu_ctx** out) {
  if (!out) return DGPU_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return DGPU_ERR_NODEVICE;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return DGPU_ERR_NODEVICE;
  if (prop.major != 9 || prop.minor != 0) return DGPU_ERR_NODEVICE;  // kernels are compiled for sm_90a only
  if (cudaSetDevice(device) != cudaSuccess) return DGPU_ERR_NODEVICE;
  dgpu_ctx* ctx = new dgpu_ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->bufs.resize(SLOT_COUNT);
  ctx->no_band = getenv("DGPU_ED_NO_BAND") != nullptr;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return DGPU_ERR_CUDA;
  }
  *out = ctx;
  return DGPU_OK;
}

void dgpu_ctx_destroy(dgpu_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (auto& b : ctx->bufs)
    if (b.p) cudaFree(b.p);
  if (ctx->refused) cudaFree(ctx->refused);
  if (ctx->ev0) { cudaEventDestroy(ctx->ev0); cudaEventDestroy(ctx->ev1); }
  for (auto e : ctx->pipe_events) cudaEventDestroy(e);
  for (auto e : ctx->fork_events) cudaEventDestroy(e);
  for (auto f : ctx->fork_streams) cudaStreamDestroy(f);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->out_stream) cudaStreamDestroy(ctx->out_stream);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int dgpu_ctx_sync(dgpu_ctx* ctx) {
  if (!ctx) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return dgpu_fold_refusals(ctx);
}

const char* dgpu_last_error(dgpu_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }

uint64_t dgpu_launch_count(dgpu_ctx* ctx) { return ctx ? ctx->launches : 0; }

uint64_t dgpu_unsupported_count(dgpu_ctx* ctx) {
  if (!ctx) return 0;
  dgpu_fold_refusals(ctx);   // a failed read leaves the count as it was and its text in last_error
  return ctx->unsupported;
}

int dgpu_set_async_bound(dgpu_ctx* ctx, uint32_t max_seq_len) {
  if (!ctx) return DGPU_ERR_ARG;
  ctx->async_bound = max_seq_len;
  return DGPU_OK;
}

int dgpu_set_profiling(dgpu_ctx* ctx, int on) {
  if (!ctx) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  if (on && !ctx->ev0) {
    DGPU_CUDA(ctx, cudaEventCreate(&ctx->ev0));
    DGPU_CUDA(ctx, cudaEventCreate(&ctx->ev1));
  }
  ctx->profiling = on != 0;
  return DGPU_OK;
}

float dgpu_last_kernel_ms(dgpu_ctx* ctx) {
  if (!ctx) return -1.f;
  if (ctx->ev_pending) {
    cudaEventSynchronize(ctx->ev1);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_kernel_ms = ms;
    ctx->ev_pending = false;
  }
  return ctx->last_kernel_ms;
}

}  // extern "C"

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
DgpuStage::DgpuStage(dgpu_ctx* c, const char* nm, uint64_t n) : name(nm), items(n), ctx(c) {
  static const bool enabled = getenv("DGPU_TRACE") != nullptr;
  if ((traced = enabled)) t0 = now_ms();
}
DgpuStage::~DgpuStage() { if (traced) fprintf(stderr, "[dgpu] %-22s %10llu items %9.2f ms\n", name, (unsigned long long) items, now_ms() - t0); }
