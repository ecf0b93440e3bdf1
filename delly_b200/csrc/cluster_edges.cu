// cluster_edges.cu — candidate edges of Delly's clustering graphs, the data-parallel half of cluster().
//
// The reference builds its split-read and paired-end graphs with a windowed pair scan over the sorted records
// (src/cluster.h:371-431 for SRBamRecord, :551-623 for BamAlignRecord): for every record i it walks j = i+1.. until
// the window closes, tests a handful of integer predicates and, for a hit, connects (i, j) with an integer weight.
// What happens to a connected pair (component relabelling, the graphPruning cap, clique growth) is sequential and
// order-dependent and stays on the host (delly_b200/host/cluster.hpp); which pairs connect, and with what weight, is a
// pure function of the two records. That part runs here: one thread per record i, count -> exclusive scan -> fill,
// so the edges of record i come out in increasing j and the concatenation over i is exactly the order in which the
// reference's double loop meets them.
//
// Exactness: all predicates are int32 arithmetic. The two floating-point spots are reproduced as follows:
//   * SR window  uint32(std::abs(0.1 * span))  (src/cluster.h:366-367): one IEEE double multiply + truncation, identical on device;
//   * PE weight  uint32(std::log2(double(x) + 1))  (src/cluster.h:620): x + 1 is an integer in [1, 2^32); floor(log2) of
//     an integer is 31 - clz (log2 of 2^k - 1 is farther from k than any rounding error of a < 1 ulp log2).
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int CE_THREADS = 256;
constexpr int SVT_TRANS = 5;  // DELLY_SVT_TRANS (src/tags.h:20)

__host__ __device__ __forceinline__ bool ce_transloc(int svt) { return svt >= SVT_TRANS && svt < 9; }  // src/tags.h:25-28
__host__ __device__ __forceinline__ int ce_iabs(int x) { return x < 0 ? -x : x; }

struct SrArgs {
  const int32_t *chr, *pos, *chr2, *pos2, *inslen;
  uint32_t n;
  int svt;
  uint32_t maxReadSep;
};

struct PeArgs {
  const int32_t *pos, *mpos, *mtid, *alen, *median, *maxNormalISize;
  uint32_t n;
  int svt;
  uint32_t varisize;
};

// src/cluster.h:362-370
__device__ __forceinline__ uint32_t sr_varisize(const SrArgs& a, uint32_t i) {
  if (ce_transloc(a.svt)) return 2 * a.maxReadSep;
  uint32_t v = a.maxReadSep;
  double span = (a.svt == 4) ? (double) a.inslen[i] : (double) (a.pos2[i] - a.pos[i]);
  uint32_t svvar = __double2uint_rz(fabs(0.1 * span));
  if (v < svvar) v = svvar;
  if (v > 1000) v = 1000;
  return v;
}

// Visits the edges of record i in increasing j. F(j, weight).
template <typename F>
__device__ __forceinline__ void sr_scan(const SrArgs& a, uint32_t i, F f) {
  const uint32_t varisize = sr_varisize(a, i);
  const int32_t ci = a.chr[i], pi = a.pos[i], p2i = a.pos2[i], c2i = a.chr2[i], li = a.inslen[i];
  const bool tr = ce_transloc(a.svt);
  for (uint32_t j = i + 1; j < a.n; ++j) {
    if (a.chr[j] != ci) break;                                                   // the scan stays inside one chromosome (:339-342)
    const int32_t pj = a.pos[j];
    if ((uint32_t) (pj - pi) > varisize) break;                                  // :373
    if (a.svt == 4 && (uint32_t) ce_iabs(a.inslen[j] - li) > varisize) continue;  // :374
    if (tr && a.chr2[j] != c2i) continue;                                        // :375
    const int32_t d2 = ce_iabs(a.pos2[j] - p2i);
    if ((uint32_t) d2 < varisize) f(j, (uint32_t) (d2 + ce_iabs(pj - pi)));      // :376, weight :425
  }
}

__device__ __forceinline__ int32_t pe_min(int32_t pos, int32_t mpos, int svt) { return ce_transloc(svt) ? pos : min(pos, mpos); }   // src/tags.h:174-179
__device__ __forceinline__ int32_t pe_max(int32_t pos, int32_t mpos, int svt) { return ce_transloc(svt) ? mpos : max(pos, mpos); }  // src/tags.h:181-186

// src/tags.h:277-346. o1/o2 pick which pair's maxNormalISize bounds the start offset / the end offset.
__device__ __forceinline__ bool pe_disagree(int32_t min1, int32_t max1, int32_t len1, int32_t iso1, int32_t min2, int32_t max2, int32_t len2,
                                            int32_t iso2, int svt) {
  // limitStart bounds (min2 + len2 - min1); limitLo bounds the end offset when pair 2 ends first, limitHi when it ends last
  int32_t limitStart, limitLo, limitHi;
  if (ce_transloc(svt)) {
    const int ct = svt - SVT_TRANS;
    if (ct % 2 == 0) { limitStart = iso1; if (ct >= 2) { limitLo = iso1; limitHi = iso2; } else { limitLo = iso2; limitHi = iso1; } }
    else { limitStart = iso2; if (ct >= 2) { limitLo = iso2; limitHi = iso1; } else { limitLo = iso1; limitHi = iso2; } }
  } else if (svt == 0) { limitStart = iso1; limitLo = iso2; limitHi = iso1; }
  else if (svt == 1) { limitStart = iso2; limitLo = iso1; limitHi = iso2; }
  else if (svt == 2) { limitStart = iso1; limitLo = iso1; limitHi = iso2; }
  else if (svt == 3) { limitStart = iso2; limitLo = iso2; limitHi = iso1; }
  else return false;
  if ((min2 + len2 - min1) > limitStart) return true;
  if (max2 < max1) { if ((max1 + len1 - max2) > limitLo) return true; }
  else { if ((max2 + len2 - max1) > limitHi) return true; }
  if (svt == 2 && ((max1 < min2) || (max2 < min1))) return true;  // deletions: the spans must overlap (:335)
  return false;
}

template <typename F>
__device__ __forceinline__ void pe_scan(const PeArgs& a, uint32_t i, F f) {
  const int32_t aMin = pe_min(a.pos[i], a.mpos[i], a.svt), aMax = pe_max(a.pos[i], a.mpos[i], a.svt);
  const int32_t aLen = a.alen[i], aIso = a.maxNormalISize[i], aMed = a.median[i], aMtid = a.mtid[i];
  for (uint32_t j = i + 1; j < a.n; ++j) {
    const int32_t bMin = pe_min(a.pos[j], a.mpos[j], a.svt), bMax = pe_max(a.pos[j], a.mpos[j], a.svt);
    const int32_t bLen = a.alen[j];
    if (!((uint32_t) ce_iabs(bMin + bLen - aMin) <= a.varisize)) break;            // src/cluster.h:564
    if (aMtid != a.mtid[j]) continue;                                              // :566
    if (pe_disagree(aMin, aMax, aLen, aIso, bMin, bMax, bLen, a.maxNormalISize[j], a.svt)) continue;  // :569
    const uint32_t x = (uint32_t) ce_iabs(ce_iabs((bMin - aMin) - (bMax - aMax)) - ce_iabs(aMed - a.median[j])) + 1u;  // :620
    f(j, 31u - (uint32_t) __clz((int) x));
  }
}

template <bool SR, typename A>
__global__ void ce_count_kernel(A a, uint32_t* __restrict__ cnt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  uint32_t c = 0;
  if constexpr (SR) sr_scan(a, i, [&](uint32_t, uint32_t) { ++c; });
  else pe_scan(a, i, [&](uint32_t, uint32_t) { ++c; });
  cnt[i] = c;
}

template <bool SR, typename A>
__global__ void ce_fill_kernel(A a, const uint32_t* __restrict__ off, uint32_t* __restrict__ ej, uint32_t* __restrict__ ew, uint64_t cap) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  uint64_t o = off[i];
  auto put = [&](uint32_t j, uint32_t w) { if (o < cap) { ej[o] = j; ew[o] = w; } ++o; };
  if constexpr (SR) sr_scan(a, i, put);
  else pe_scan(a, i, put);
}

// ---- exclusive scan of n uint32 counts into n+1 offsets (2048 items per block; block sums scanned by one block) ----
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = CE_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t block_exclusive(uint32_t v, uint32_t* total) {
  __shared__ uint32_t wsum[CE_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    uint32_t s = lane < CE_THREADS / 32 ? wsum[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, s, d); if (lane >= d) s += t; }
    if (lane < CE_THREADS / 32) wsum[lane] = s;
  }
  __syncthreads();
  const uint32_t base = w ? wsum[w - 1] : 0;
  *total = wsum[CE_THREADS / 32 - 1];
  __syncthreads();
  return base + inc - v;
}

__global__ void scan_tiles_kernel(const uint32_t* __restrict__ cnt, uint32_t n, uint32_t* __restrict__ off, unsigned long long* __restrict__ tile_sum) {
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) { v[k] = (base + k < n) ? cnt[base + k] : 0; s += v[k]; }
  uint32_t total;
  uint32_t ex = block_exclusive(s, &total);
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) off[base + k] = ex; ex += v[k]; }
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void scan_sums_kernel(unsigned long long* tile_sum, uint32_t tiles, unsigned long long* total) {
  // one thread: a few thousand tiles at most (2048 records each)
  unsigned long long s = 0;
  for (uint32_t t = 0; t < tiles; ++t) { unsigned long long v = tile_sum[t]; tile_sum[t] = s; s += v; }
  *total = s;
}

__global__ void scan_add_kernel(uint32_t* __restrict__ off, uint32_t n, const unsigned long long* __restrict__ tile_sum, const unsigned long long* __restrict__ total) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) off[i] += (uint32_t) tile_sum[i / SCAN_TILE];
  if (i == 0) off[n] = (uint32_t) *total;
}

template <bool SR, typename A>
int ce_run(DgpuStage& s, A a, const void* const* host_cols, int ncols, uint64_t n, uint32_t* edge_off, uint32_t* edge_j, uint32_t* edge_w,
           uint64_t edge_cap, uint64_t* n_edges) {
  dgpu_ctx* ctx = s.ctx;
  int rc;
  if ((rc = s.open())) return rc;
  cudaStream_t st = s.st;
  // record columns: one device arena, ncols x n int32
  int32_t* d_cols = s.alloc<int32_t>((size_t) ncols * n);
  for (int k = 0; k < ncols; ++k) s.upload(d_cols + (size_t) k * n, host_cols[k], n * 4);
  const uint32_t tiles = (uint32_t) ((n + SCAN_TILE - 1) / SCAN_TILE);
  uint32_t* d_cnt = s.alloc<uint32_t>(n + 1);
  uint32_t* d_off = s.out(edge_off, n + 1);
  unsigned long long* d_tiles = s.alloc<unsigned long long>((size_t) tiles + 1);
  if (s.rc) return s.rc;
  const int32_t* col[8];
  for (int k = 0; k < ncols; ++k) col[k] = d_cols + (size_t) k * n;
  if constexpr (SR) { a.chr = col[0]; a.pos = col[1]; a.chr2 = col[2]; a.pos2 = col[3]; a.inslen = col[4]; }
  else { a.pos = col[0]; a.mpos = col[1]; a.mtid = col[2]; a.alen = col[3]; a.median = col[4]; a.maxNormalISize = col[5]; }
  unsigned long long* d_total = d_tiles + tiles;
  const unsigned blocks = (unsigned) ((n + CE_THREADS - 1) / CE_THREADS);
  dgpu_prof_begin(ctx, st);
  ce_count_kernel<SR, A><<<blocks, CE_THREADS, 0, st>>>(a, d_cnt);
  DGPU_LAUNCH_CHECK(ctx, "ce_count");
  scan_tiles_kernel<<<tiles, CE_THREADS, 0, st>>>(d_cnt, (uint32_t) n, d_off, d_tiles);
  DGPU_LAUNCH_CHECK(ctx, "scan_tiles");
  scan_sums_kernel<<<1, 1, 0, st>>>(d_tiles, tiles, d_total);
  DGPU_LAUNCH_CHECK(ctx, "scan_sums");
  scan_add_kernel<<<(unsigned) ((n + 1 + CE_THREADS - 1) / CE_THREADS), CE_THREADS, 0, st>>>(d_off, (uint32_t) n, d_tiles, d_total);
  DGPU_LAUNCH_CHECK(ctx, "scan_add");
  unsigned long long total = 0;
  DGPU_CUDA(ctx, cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  *n_edges = total;
  if (total >= (1ull << 32)) { ctx->last_error = "dgpu_cluster_edges: more than 2^32-1 edges"; return DGPU_ERR_CAPACITY; }
  const uint64_t fillcap = std::min<uint64_t>(total, edge_cap);
  if (fillcap) {   // the edge columns are sized by the count pass: staged (and copied back) only now
    uint32_t *d_ej = s.out(edge_j, fillcap), *d_ew = s.out(edge_w, fillcap);
    if (s.rc) return s.rc;
    ce_fill_kernel<SR, A><<<blocks, CE_THREADS, 0, st>>>(a, d_off, d_ej, d_ew, fillcap);
    DGPU_LAUNCH_CHECK(ctx, "ce_fill");
  }
  dgpu_prof_end(ctx, st);
  if ((rc = s.finish())) return rc;
  return total > edge_cap ? DGPU_ERR_CAPACITY : DGPU_OK;
}

}  // namespace

extern "C" {

int dgpu_cluster_edges_sr(dgpu_ctx* ctx, const int32_t* chr, const int32_t* pos, const int32_t* chr2, const int32_t* pos2, const int32_t* inslen,
                          uint64_t n, int svt, uint32_t max_read_sep, uint32_t* edge_off, uint32_t* edge_j, uint32_t* edge_w, uint64_t edge_cap,
                          uint64_t* n_edges) {
  DgpuStage s(ctx, "dgpu_cluster_edges_sr", n);
  if (!ctx || !edge_off || !n_edges) return DGPU_ERR_ARG;
  *n_edges = 0;
  if (n == 0) { edge_off[0] = 0; return DGPU_OK; }
  if (!chr || !pos || !chr2 || !pos2 || !inslen || n >= (1ull << 31) || svt < 0 || svt > 8 || (edge_cap && (!edge_j || !edge_w))) return DGPU_ERR_ARG;
  SrArgs a;
  a.n = (uint32_t) n; a.svt = svt; a.maxReadSep = max_read_sep;
  const void* cols[5] = {chr, pos, chr2, pos2, inslen};
  return ce_run<true>(s, a, cols, 5, n, edge_off, edge_j, edge_w, edge_cap, n_edges);
}

int dgpu_cluster_edges_pe(dgpu_ctx* ctx, const int32_t* pos, const int32_t* mpos, const int32_t* mtid, const int32_t* alen, const int32_t* median,
                          const int32_t* max_normal_isize, uint64_t n, int svt, uint32_t varisize, uint32_t* edge_off, uint32_t* edge_j,
                          uint32_t* edge_w, uint64_t edge_cap, uint64_t* n_edges) {
  DgpuStage s(ctx, "dgpu_cluster_edges_pe", n);
  if (!ctx || !edge_off || !n_edges) return DGPU_ERR_ARG;
  *n_edges = 0;
  if (n == 0) { edge_off[0] = 0; return DGPU_OK; }
  if (!pos || !mpos || !mtid || !alen || !median || !max_normal_isize || n >= (1ull << 31) || svt < 0 || svt > 8 || svt == 4 ||
      (edge_cap && (!edge_j || !edge_w)))
    return DGPU_ERR_ARG;
  PeArgs a;
  a.n = (uint32_t) n; a.svt = svt; a.varisize = varisize;
  const void* cols[6] = {pos, mpos, mtid, alen, median, max_normal_isize};
  return ce_run<false>(s, a, cols, 6, n, edge_off, edge_j, edge_w, edge_cap, n_edges);
}

}  // extern "C"
