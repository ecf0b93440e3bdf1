// int_peak.cu — measured integer-ALU roofline denominator (LOP3 + IADD3, 8-way ILP per thread).
#include "common.cuh"

namespace {
constexpr int IP_ITERS = 4096;
// 8 independent dependent-chains per thread of LOP3 (majority, LUT 0xE8: not algebraically reducible) —
// the instruction class the Myers kernels are made of. asm volatile keeps ptxas from folding/hoisting.
__global__ void __launch_bounds__(256) int_peak_kernel(uint32_t* out, uint32_t seed) {
  uint32_t x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = seed + threadIdx.x * 8 + i;
  uint32_t y = seed ^ 0x9e3779b9u ^ threadIdx.x, z = blockIdx.x + 0x7f4a7c15u;
#pragma unroll 1
  for (int it = 0; it < IP_ITERS; ++it) {
#pragma unroll
    for (int rep = 0; rep < 4; ++rep) {
#pragma unroll
      for (int i = 0; i < 8; ++i) asm volatile("lop3.b32 %0, %0, %1, %2, 0xE8;" : "+r"(x[i]) : "r"(y), "r"(z));
#pragma unroll
      for (int i = 0; i < 8; ++i) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x[i]) : "r"(z), "r"(y));
    }
  }
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) r ^= x[i];
  if (r == 0x12345678u) out[0] = r;  // keep the chains alive
}
constexpr double IP_OPS_PER_THREAD = (double) IP_ITERS * 4 * 16;

// The same LOP3 chains with 8 independent IMAD chains interleaved (WIDE: IMAD.WIDE.U32 chains on 64-bit accumulators, each step
// multiplying the two halves so that both stay live; a 64-bit addend would be split off into IADD3s): whether the
// FMA pipe issues multiplies alongside the integer ALU pipe, which is what moving shifts and adds of the Myers column onto IMAD
// relies on. The multiplier and addend are kernel arguments, so ptxas cannot fold them into shifts or LEAs on the ALU pipe.
template <bool WIDE>
__global__ void __launch_bounds__(256) int_peak_mix_kernel(uint32_t* out, uint32_t seed, uint32_t mul, uint32_t add) {
  uint32_t x[8];
  uint32_t g[8];
  uint64_t f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    x[i] = seed + threadIdx.x * 8 + i;
    g[i] = seed ^ (threadIdx.x * 16 + i);
    f[i] = g[i];
  }
  uint32_t y = seed ^ 0x9e3779b9u ^ threadIdx.x, z = blockIdx.x + 0x7f4a7c15u;
#pragma unroll 1
  for (int it = 0; it < IP_ITERS; ++it) {
#pragma unroll
    for (int rep = 0; rep < 4; ++rep) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0xE8;" : "+r"(x[i]) : "r"(y), "r"(z));
        if (WIDE) asm volatile("{.reg .u32 l, h;\n\tmov.b64 {l, h}, %0;\n\tmul.wide.u32 %0, l, h;}" : "+l"(f[i]));
        else asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(g[i]) : "r"(mul), "r"(add));
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x[i]) : "r"(z), "r"(y));
        if (WIDE) asm volatile("{.reg .u32 l, h;\n\tmov.b64 {l, h}, %0;\n\tmul.wide.u32 %0, l, h;}" : "+l"(f[i]));
        else asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(g[i]) : "r"(mul), "r"(add));
      }
    }
  }
  uint64_t r = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) r ^= x[i] ^ g[i] ^ f[i];
  if (r == 0x12345678u) out[0] = (uint32_t) r;  // keep the chains alive
}

// best-of-4 (after one warm-up launch) kernel time in ms of `launch`
template <class F>
int time_best(dgpu_ctx* ctx, F launch, float* best) {
  cudaEvent_t e0, e1;
  DGPU_CUDA(ctx, cudaEventCreate(&e0));
  DGPU_CUDA(ctx, cudaEventCreate(&e1));
  *best = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    DGPU_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
    launch(rep);
    DGPU_LAUNCH_CHECK(ctx, "int_peak_mix");
    DGPU_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
    DGPU_CUDA(ctx, cudaEventSynchronize(e1));
    float ms;
    DGPU_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < *best) *best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return DGPU_OK;
}
}  // namespace
extern "C" int dgpu_int_peak(dgpu_ctx* ctx, double* tops) {
  if (!ctx || !tops) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  void* p;
  int rc = dgpu_reserve(ctx, SLOT_COUNTS, 32 * sizeof(uint32_t), &p);
  if (rc) return rc;
  cudaEvent_t e0, e1;
  DGPU_CUDA(ctx, cudaEventCreate(&e0));
  DGPU_CUDA(ctx, cudaEventCreate(&e1));
  const int grid = ctx->num_sms * 8;
  float best = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    DGPU_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
    int_peak_kernel<<<grid, 256, 0, ctx->stream>>>((uint32_t*) p, 17u + rep);
    DGPU_LAUNCH_CHECK(ctx, "int_peak");
    DGPU_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
    DGPU_CUDA(ctx, cudaEventSynchronize(e1));
    float ms;
    DGPU_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  double ops = (double) grid * 256.0 * IP_OPS_PER_THREAD;
  *tops = ops / (best * 1e-3) / 1e12;
  return DGPU_OK;
}

extern "C" int dgpu_int_peak_mix(dgpu_ctx* ctx, double* tops) {
  if (!ctx || !tops) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  void* p;
  int rc = dgpu_reserve(ctx, SLOT_COUNTS, 32 * sizeof(uint32_t), &p);
  if (rc) return rc;
  uint32_t* out = (uint32_t*) p;
  const int grid = ctx->num_sms * 8;
  cudaStream_t st = ctx->stream;
  float ms[3] = {0.f, 0.f, 0.f};
  rc = time_best(ctx, [&](int rep) { int_peak_kernel<<<grid, 256, 0, st>>>(out, 17u + rep); }, &ms[0]);
  if (!rc) rc = time_best(ctx, [&](int rep) { int_peak_mix_kernel<false><<<grid, 256, 0, st>>>(out, 17u + rep, 3u, 1u); }, &ms[1]);
  if (!rc) rc = time_best(ctx, [&](int rep) { int_peak_mix_kernel<true><<<grid, 256, 0, st>>>(out, 17u + rep, 3u, 1u); }, &ms[2]);
  if (rc) return rc;
  const double lop3 = (double) grid * 256.0 * IP_OPS_PER_THREAD;  // the mixed kernels issue as many IMADs again
  tops[0] = lop3 / (ms[0] * 1e-3) / 1e12;
  tops[1] = 2 * lop3 / (ms[1] * 1e-3) / 1e12;
  tops[2] = 2 * lop3 / (ms[2] * 1e-3) / 1e12;
  return DGPU_OK;
}
