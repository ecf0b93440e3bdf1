// edit_distance.cu — batched Myers bit-vector edit distance (NW / SHW / HW, distance + first end
// location), the device replacement for edlibAlign(..., EDLIB_TASK_DISTANCE).
//
// Reference semantics reproduced (results only; the Ukkonen band schedule of the CPU code is an
// optimisation that does not change results):
//   src/edlib.cpp:139-294  edlibAlign driver: empty-sequence rules, k auto-doubling, NW end location
//   src/edlib.cpp:407-442  calculateBlock (Myers/Hyyro advance-block)
//   src/edlib.cpp:545-702  HW/SHW: min over target columns of D[m][c], k=min(k,|q|) for HW, -1 if > k,
//                          positions in increasing order (we return the first)
//   src/edlib.cpp:728-929  NW: -1 if k < |n-m|, k=min(k,max(m,n)), D[m][n] if <= k
//
// Device design (H100, integer-ALU bound; HBM traffic is ~(|q|+|t|)/2..1 byte per 30+ int ops):
//   * jobs are binned on the device by ceil(|q|/32) (counting sort: ed_count_kernel classifies each job once, keeps its slot byte and, in its
//     last block, turns the counts into class starts; ed_scatter_kernel places the jobs from the slot bytes). The class kernels then run
//     side by side on the context's fork/join streams, costliest class first (launch_mode),
//   * |q| <= 128: ONE THREAD PER JOB. The whole DP column is one multi-word bit-vector held in
//     registers (NW = 1..4 x 32 bit, add-with-carry chain, funnel shifts), the score is read at bit
//     |q|-1 so no padding/wildcard columns are needed. The per-job match masks Peq[5][NW] live in a
//     per-thread-private, bank-conflict-free slice of shared memory; the target is streamed with
//     aligned LDG.128 + PRMT realignment (ChunkReader).
//   * HW jobs 2i and 2i+1 on the same target (a read's ALT and REF probes) with queries of one class
//     run as a pair in one thread (ed_pair_kernel): one target stream and decode, two Myers columns. Pairs whose two queries fit one
//     column of 3 or 5 words with a separator row between them (33-47 bp or 65-79 bp probe pairs) share that column (ed_pack_kernel).
//     Every read over one breakpoint has the same two probes, so the first such pair to run publishes its Peq table in a per-call hash
//     table keyed by the probes' offsets, and later pairs of that key copy it instead of building it (peq_find / peq_publish).
//   * |q| > 128: ONE WARP PER JOB, anti-diagonal wavefront: lane l owns a 64-row block and processes
//     column t-l at step t; the horizontal delta (hout) crosses lanes by shuffle. Queries longer
//     than 2048 rows are processed in 2048-row stripes, the stripe's bottom hout per column being
//     parked in a per-warp L2-resident scratch row.
//   * bytes other than ACGTN take an exact slow path (byte equality against the query), so the
//     reference's "equality is byte equality" contract holds for IUPAC / lower case too.
#include "common.cuh"
#include "myers.cuh"
#include <algorithm>
#include <array>
#include <cstdio>
#include <utility>

namespace {

constexpr int ED_THREADS = 128;
// grid cap of the one-thread-per-job kernels, in CTAs per SM. At 56-72 registers an SM holds 7-9 of these 128-thread CTAs, so the cap
// launches several waves of CTAs that each take a slice of the grid-stride loop; later waves fill the SMs whose CTAs finished early. On an
// H100 at 400 W (tools/bench_k1.py, the 10 M configs[1] jobs by class) 32 ran 8 % faster than 7 (one wave) and 3.5 % faster than 14;
// 64 was 0.8 % faster than 32, too little to tell from run-to-run noise. Results identical in every variant. ED_CTAS_PER_SM_V lets
// tools/build_variant.sh build such variants.
#ifndef ED_CTAS_PER_SM_V
#define ED_CTAS_PER_SM_V 32
#endif
constexpr int ED_CTAS_PER_SM = ED_CTAS_PER_SM_V;
// job classes: 0 trivial, 1..4 = words per thread-job, 5 = warp-per-job, ED_PAIR + 1..4 = target-sharing pairs of class 1..4 (ed_pair_kernel),
// ED_PACK + 0 / + 1 = target-sharing pairs packed into one column of 3 / 5 words (ed_pack_kernel<3, 1> / <5, 2>)
constexpr int ED_PAIR = 5;
constexpr int ED_PACK = ED_PAIR + 5;
constexpr int ED_NCLS = ED_PACK + 2;
// counts layout (SLOT_COUNTS): [0, 16) jobs per class, [ED_START, +16) class starts in perm, [ED_CUR, +16) scatter cursors, [ED_TMAX] max t_len
// of multi-stripe jobs, [ED_TICKET] blocks of ed_count_kernel done, [ED_BANDQ, +EDB_CLASSES + 1) band pass queues
constexpr int ED_START = 16, ED_CUR = 32, ED_TMAX = 48, ED_TICKET = 49, ED_BANDQ = 64, ED_COUNTS_WORDS = 128;
constexpr uint8_t ED_NO_SLOT = 0xff;  // slot byte of the odd member of a pair (ed_slot's -1)

struct EdArgs {
  const uint8_t* seqs;
  const uint8_t* seqs_end;
  const uint32_t* q_off;
  const uint32_t* q_len;
  const uint32_t* t_off;
  const uint32_t* t_len;
  const int32_t* k;
  uint32_t n;
  int32_t* dist;
  int32_t* end_loc;
  uint32_t* perm;
  uint32_t* counts;  // ED_START / ED_CUR / ED_TMAX / ED_TICKET / ED_BANDQ layout above
  uint8_t* slots;    // per job: its count slot (ed_slot) or ED_NO_SLOT, written by ed_count_kernel, read by ed_scatter_kernel
  int pair;          // HW distances without end locations or equality tables: target-sharing job pairs take ed_pair_kernel (ed_slot)
  int last_pos;     // HW/SHW: report the LAST optimal end position instead of the first (edlib's positionsSHW.back(), src/edlib.cpp:250)
  uint8_t* hbuf;     // per-warp scratch rows for multi-stripe jobs
  uint32_t hbuf_stride;
  // generalised equality (edlib's additionalEqualities, src/edlib.cpp:58-79); all jobs then take the warp-per-job kernel
  const uint32_t* eq_f;  // [256] bitmask of the pairs in which the byte is the first member (null: plain byte equality)
  const uint32_t* eq_s;  // [256] ... the second member
  const uint8_t* eq_cls; // [256] bitmask over {A,C,G,T,N} of the class symbols the byte is equal to
  int force_long;
  uint4* peq_slots;      // shared Peq tables of pairs (ED_PEQ_SLOTS_V below): hash slots, null unless pair
  uint4* peq_pool;       // one entry of ED_PEQ_WORDS words per slot
  uint32_t peq_mask;     // hash slots - 1
};

// Shared Peq tables (SLOT_ED_PEQ, calls with a.pair only). Every read over one SV breakpoint is realigned against the same ALT and REF
// probes, and the Peq table of a pair or pack slot depends only on the two probes' offsets and lengths. So the first thread of a pair that
// finds no table for it builds the table in its shared slice as before and publishes it: it claims an empty hash slot for the key
// (q_off[2i], q_off[2i + 1]) with a CAS, writes the entry of that slot, fences, and then stores the slot's tag. A later pair of the same
// key and lengths copies the entry instead of building it. Until the tag is stored, pairs of that key build their own table. Hash slots
// are uint4 {q_off[2i], q_off[2i + 1], tag, unused}, all ones when empty (no q_off is 0xffffffff: the arena is shorter than 4 GiB and a
// probe in a pair is not empty). The tag is 0x80000000 | q_len[2i] | q_len[2i + 1] << 16, so one word carries readiness and lengths. The
// call sizes the table as the power of two >= n jobs, capped at ED_PEQ_SLOTS_V, and clears it on its stream, so no entry outlives it.
#ifndef ED_PEQ_SLOTS_V
#define ED_PEQ_SLOTS_V (1u << 18)
#endif
constexpr uint32_t ED_PEQ_SLOTS_MAX = ED_PEQ_SLOTS_V, ED_PEQ_SLOTS_MIN = 256;
constexpr int ED_PEQ_PROBE = 4;                  // slots a lookup probes
constexpr int ED_PEQ_WORDS = 40;                 // words per entry: 5 symbol slots x 8 words (ed_pair_kernel<4>)
constexpr uint32_t ED_PEQ_NONE = 0xffffffffu;

__device__ __forceinline__ uint32_t peq_hash(uint32_t o0, uint32_t o1, uint32_t mask) {
  const uint32_t h = ((o0 * 0x9e3779b1u) ^ o1) * 0x85ebca6bu;
  return (h ^ (h >> 16)) & mask;
}

// The published entry of the key (o0, o1) with tag `tag`, or null. On a miss, `claim` is the first empty slot met (the one the caller
// may publish into), else ED_PEQ_NONE. Slots are read with plain loads, cached in L1: a stale slot is only an older state of it (empty, or
// claimed and not tagged yet), which sends the pair to the in-thread build. On an H100 at 700 W, reading every slot from L2 instead (ld.cg)
// made the class kernels 2.6x slower. Entries are read from L2 (copy_peq), where peq_publish's fence puts an entry before its tag, and an
// entry is read only after its tag has been seen; entries share cache lines, so an L1 copy of one could be older than the entry.
__device__ __forceinline__ const uint4* peq_find(const EdArgs& a, uint32_t o0, uint32_t o1, uint32_t tag, uint32_t& claim) {
  claim = ED_PEQ_NONE;
  uint32_t h = peq_hash(o0, o1, a.peq_mask);
#pragma unroll 1
  for (int k = 0; k < ED_PEQ_PROBE; ++k, h = (h + 1u) & a.peq_mask) {
    const uint4 s = a.peq_slots[h];
    if (s.x == o0 && s.y == o1) {
      if (s.z != tag) return nullptr;   // not published yet, or other lengths
      return a.peq_pool + (size_t) h * (ED_PEQ_WORDS / 4);
    }
    if ((s.x & s.y) == 0xffffffffu) { claim = h; return nullptr; }
  }
  return nullptr;
}

// Publishes the N words of the thread's slice pq (word e at pq[e * ED_THREADS]) as the entry of slot h for the key (o0, o1), unless
// another thread claims the slot first.
template <int N>
__device__ __forceinline__ void peq_publish(const EdArgs& a, uint32_t h, uint32_t o0, uint32_t o1, uint32_t tag, const uint32_t* pq) {
  const unsigned long long key = (unsigned long long) o0 | (unsigned long long) o1 << 32;
  if (atomicCAS((unsigned long long*) (a.peq_slots + h), ~0ull, key) != ~0ull) return;
  uint4* e = a.peq_pool + (size_t) h * (ED_PEQ_WORDS / 4);
  // rolled: once per distinct pair, and it keeps the column loop the block of the kernel with the most shared loads
#pragma unroll 1
  for (int i = 0; i < (N + 3) / 4; ++i) {
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = 4 * i + k < N ? pq[(4 * i + k) * ED_THREADS] : 0u;
    __stcg(e + i, make_uint4(w[0], w[1], w[2], w[3]));
  }
  __threadfence();
  atomicExch(&a.peq_slots[h].z, tag);
}

// An entry's first N words into the thread's slice (word e to pq[e * ED_THREADS]), 16 bytes per load.
template <int N>
__device__ __forceinline__ void copy_peq(uint32_t* pq, const uint4* e) {
#pragma unroll
  for (int i = 0; i < (N + 3) / 4; ++i) {
    const uint4 v = __ldcg(e + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (4 * i + k < N) pq[(4 * i + k) * ED_THREADS] = w[k];
  }
}

__device__ __forceinline__ int ed_class(uint32_t ql, uint32_t tl, int force_long) {
  if (ql == 0 || tl == 0) return 0;
  if (force_long) return 5;
  if (ql <= 128) return (int) ((ql + 31) >> 5);
  return 5;
}

// Apply edlib's k rules to the exact distance. mode: DGPU_MODE_*.
__device__ __forceinline__ int apply_k(int d, int k, int mode, int m, int n) {
  if (k < 0) return d;  // auto-doubling k always finds the exact distance (src/edlib.cpp:192-210)
  if (mode == DGPU_MODE_HW) {
    int kk = min(k, m);  // src/edlib.cpp:563-565
    return d <= kk ? d : -1;
  } else if (mode == DGPU_MODE_SHW) {
    return d <= k ? d : -1;
  } else {
    int diff = n > m ? n - m : m - n;
    if (k < diff) return -1;           // src/edlib.cpp:740-743
    int kk = min(k, max(m, n));        // src/edlib.cpp:745
    return d <= kk ? d : -1;
  }
}

// Whether two HW queries of a target fit one column of W words (ed_pack_kernel<W, WA>) in the order A = ma at the bottom, B = mb at the
// top: A's last row lies in word WA (32 WA < ma <= 32 WA + 31, so that the row above it, the first separator row, is in the same word),
// and at least one separator row is left between A and B (ma + mb + 1 <= 32 W).
__device__ __forceinline__ bool pack_fits(uint32_t ma, uint32_t mb, int W, int WA) {
  return ma > 32u * WA && ma <= 32u * WA + 31u && mb >= 1u && ma + mb < 32u * W;
}

// Pack class of the pair of query lengths (m0, m1) of jobs 2i and 2i + 1, in the order (m0, m1) or else (m1, m0); -1 if neither fits.
__device__ __forceinline__ int pack_class(uint32_t m0, uint32_t m1) {
  if (pack_fits(m0, m1, 3, 1) || pack_fits(m1, m0, 3, 1)) return ED_PACK;
  if (pack_fits(m0, m1, 5, 2) || pack_fits(m1, m0, 5, 2)) return ED_PACK + 1;
  return -1;
}

// Count slot of job i: its class, or, for the even member i of a pair (i, i + 1) of one-thread jobs on the same target (equal t_off and
// t_len: the ALT and REF probes of one genotyping read), the pack class if the two queries fit one (pack_class), else the pair class
// ED_PAIR + class if both are of the same class; -1 for the odd member of a pair. Indices are relative to the call.
// The words of job i and its partner o = i ^ 1 (in the same cache lines) are loaded by slot_words, separately from ed_slot, so that a
// thread can have the loads of several jobs in flight before it branches on any of them.
struct SlotWords {
  uint32_t mi, tl, to, mo, tlo, too;  // q_len, t_len, t_off of job i, then of its partner (0 if there is none)
};

__device__ __forceinline__ SlotWords slot_words(const EdArgs& a, uint32_t i) {
  const uint32_t o = i ^ 1u;
  const bool has_o = o < a.n;
  return SlotWords{a.q_len[i], a.t_len[i], a.t_off[i], has_o ? a.q_len[o] : 0u, has_o ? a.t_len[o] : 0u, has_o ? a.t_off[o] : 0u};
}

__device__ __forceinline__ int ed_slot(const EdArgs& a, uint32_t i, const SlotWords& v) {
  const uint32_t mi = v.mi, tl = v.tl, mo = v.mo;
  const int c = ed_class(mi, tl, a.force_long);
  if (!a.pair || c < 1 || c > 4) return c;
  if ((i ^ 1u) >= a.n || v.too != v.to || v.tlo != tl) return c;
  const int pk = (i & 1u) ? pack_class(mo, mi) : pack_class(mi, mo);
  if (pk >= 0) return (i & 1u) ? -1 : pk;
  if (ed_class(mo, tl, 0) != c) return c;
  return (i & 1u) ? -1 : ED_PAIR + c;
}

// Both binning kernels run ED_BIN_CTAS_PER_SM blocks of ED_BIN_THREADS per SM (one wave) and loop over their jobs, so that each block's
// global atomics on the counts line (per class, plus the ticket) are paid once per block rather than once per 256 jobs. Each thread keeps
// several jobs' loads in flight at once (ED_COUNT_UNROLL jobs in ed_count_kernel, one 4-byte word of slots in ed_scatter_kernel): with one
// job per thread the loads of a wave were too few to keep HBM busy.
constexpr int ED_BIN_THREADS = 256, ED_BIN_CTAS_PER_SM = 8, ED_COUNT_UNROLL = 2;

// The one classification of a call: each job's count slot (ed_slot) goes to a.slots, so that ed_scatter_kernel reads one byte per job instead
// of the lengths and target offsets of the job and its partner. Trivial jobs get their result here. Counts are summed per warp (one shared
// atomic per distinct slot, from the lowest lane holding it), then per block; the last block to finish (a ticket taken after a fence) turns
// the class counts into the class starts and scatter cursors.
__global__ void __launch_bounds__(ED_BIN_THREADS) ed_count_kernel(EdArgs a, int mode) {
  __shared__ uint32_t h[ED_NCLS];
  __shared__ uint32_t hmax;
  if (threadIdx.x < ED_NCLS) h[threadIdx.x] = 0;
  if (threadIdx.x == 0) hmax = 0;
  __syncthreads();
  // the loop bound is the block's first job, so every lane of a warp runs every iteration (__match_any_sync over the full warp)
  constexpr uint32_t STEP = ED_COUNT_UNROLL * ED_BIN_THREADS;
  for (uint32_t i0 = blockIdx.x * STEP; i0 < a.n; i0 += gridDim.x * STEP) {
    SlotWords v[ED_COUNT_UNROLL];
#pragma unroll
    for (int u = 0; u < ED_COUNT_UNROLL; ++u) {  // every job's loads before any branch or store
      const uint32_t i = i0 + u * ED_BIN_THREADS + threadIdx.x;
      if (i < a.n) v[u] = slot_words(a, i);
    }
#pragma unroll
    for (int u = 0; u < ED_COUNT_UNROLL; ++u) {
      const uint32_t i = i0 + u * ED_BIN_THREADS + threadIdx.x;
      const int c = i < a.n ? ed_slot(a, i, v[u]) : -1;
      if (i < a.n) {
        a.slots[i] = c >= 0 ? (uint8_t) c : ED_NO_SLOT;
        if (c == 5 && a.q_len[i] > 2048) atomicMax(&hmax, a.t_len[i]);
        if (c == 0) {
          // src/edlib.cpp:158-177: NW -> max(len), endLocations[0] = n-1; HW/SHW -> |q|, endLocations[0] = -1.
          // (this special case is taken before k is looked at)
          const uint32_t ql = a.q_len[i], tl = a.t_len[i];
          int d = (mode == DGPU_MODE_NW) ? (int) max(ql, tl) : (int) ql;
          a.dist[i] = d;
          if (a.end_loc) a.end_loc[i] = (mode == DGPU_MODE_NW) ? (int) tl - 1 : -1;
        }
      }
      const uint32_t peers = __match_any_sync(0xffffffffu, c);
      if (c >= 0 && (threadIdx.x & 31u) == (uint32_t) (__ffs(peers) - 1)) atomicAdd(&h[c], (uint32_t) __popc(peers));
    }
  }
  __syncthreads();
  if (threadIdx.x < 32) {  // warp 0 makes every global update of the block
    if (threadIdx.x < ED_NCLS && h[threadIdx.x]) atomicAdd(&a.counts[threadIdx.x], h[threadIdx.x]);
    if (threadIdx.x == 0 && hmax) atomicMax(&a.counts[ED_TMAX], hmax);
    __threadfence();
    __syncwarp();
    if (threadIdx.x == 0 && atomicAdd(&a.counts[ED_TICKET], 1u) == gridDim.x - 1) {
      // every other block's counts are in: class starts in perm, and the scatter cursors at the same place
      __threadfence();
      const volatile uint32_t* cnt = a.counts;
      uint32_t s = 0;
      for (int k = 0; k < ED_NCLS; ++k) {
        a.counts[ED_START + k] = s;
        a.counts[ED_CUR + k] = s;
        s += cnt[k];
      }
    }
  }
}

// perm entries from the slot bytes. Each block takes one contiguous range of jobs and passes over its slot bytes twice: the first pass counts
// the range's jobs per class, one global atomic per class on its scatter cursor reserves their places, and the second pass hands the places
// out. A thread reads the slots of four consecutive jobs as one word (a.slots has 16 bytes of slack past n) and takes them one at a time;
// per warp and job, one shared atomic per distinct slot (the lowest lane holding it takes room for all its peers). Any order of the jobs
// within a class segment gives the same results.
__global__ void __launch_bounds__(ED_BIN_THREADS) ed_scatter_kernel(EdArgs a) {
  constexpr uint32_t STEP = 4 * ED_BIN_THREADS;
  __shared__ uint32_t h[ED_NCLS];
  if (threadIdx.x < ED_NCLS) h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t per = ((a.n + gridDim.x - 1) / gridDim.x + STEP - 1) / STEP * STEP;
  const uint32_t lo = blockIdx.x * per, hi = min(a.n, lo + per);
  const uint32_t lane = threadIdx.x & 31u;
  // the slots of jobs i0 + 4 threadIdx.x + 0..3, byte b = job b; past the range ED_NO_SLOT
  auto word = [&](uint32_t i0) {
    const uint32_t i = i0 + 4u * threadIdx.x;
    if (i >= hi) return 0xffffffffu;
    const uint32_t w = *(const uint32_t*) (a.slots + i);
    return hi - i >= 4u ? w : w | (0xffffffffu << (8u * (hi - i)));
  };
  for (uint32_t i0 = lo; i0 < hi; i0 += STEP) {
    const uint32_t w = word(i0);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const uint32_t s = (w >> (8 * b)) & 0xffu;
      const int c = s == ED_NO_SLOT ? -1 : (int) s;
      const uint32_t peers = __match_any_sync(0xffffffffu, c);
      if (c >= 0 && (int) lane == __ffs(peers) - 1) atomicAdd(&h[c], (uint32_t) __popc(peers));
    }
  }
  __syncthreads();
  if (threadIdx.x < ED_NCLS && h[threadIdx.x]) h[threadIdx.x] = atomicAdd(&a.counts[ED_CUR + threadIdx.x], h[threadIdx.x]);
  __syncthreads();
  for (uint32_t i0 = lo; i0 < hi; i0 += STEP) {
    const uint32_t w = word(i0);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const uint32_t s = (w >> (8 * b)) & 0xffu;
      const int c = s == ED_NO_SLOT ? -1 : (int) s;
      const uint32_t peers = __match_any_sync(0xffffffffu, c);
      const int lead = __ffs(peers) - 1;
      uint32_t r = 0;
      if (c >= 0 && (int) lane == lead) r = atomicAdd(&h[c], (uint32_t) __popc(peers));
      r = __shfl_sync(0xffffffffu, r, lead) + (uint32_t) __popc(peers & ((1u << lane) - 1u));
      if (c >= 0) a.perm[r] = i0 + 4u * threadIdx.x + (uint32_t) b;
    }
  }
}

// ---- multi-word add with carry ---------------------------------------------------------
template <int NW> struct AddChain;
template <> struct AddChain<1> {
  static __device__ __forceinline__ void run(uint32_t* s, const uint32_t* x, const uint32_t* y) { s[0] = x[0] + y[0]; }
};
template <> struct AddChain<2> {
  static __device__ __forceinline__ void run(uint32_t* s, const uint32_t* x, const uint32_t* y) {
    asm("add.cc.u32 %0, %2, %4;\n\taddc.u32 %1, %3, %5;"
        : "=r"(s[0]), "=r"(s[1]) : "r"(x[0]), "r"(x[1]), "r"(y[0]), "r"(y[1]));
  }
};
template <> struct AddChain<3> {
  static __device__ __forceinline__ void run(uint32_t* s, const uint32_t* x, const uint32_t* y) {
    asm("add.cc.u32 %0, %3, %6;\n\taddc.cc.u32 %1, %4, %7;\n\taddc.u32 %2, %5, %8;"
        : "=r"(s[0]), "=r"(s[1]), "=r"(s[2])
        : "r"(x[0]), "r"(x[1]), "r"(x[2]), "r"(y[0]), "r"(y[1]), "r"(y[2]));
  }
};
template <> struct AddChain<4> {
  static __device__ __forceinline__ void run(uint32_t* s, const uint32_t* x, const uint32_t* y) {
    asm("add.cc.u32 %0, %4, %8;\n\taddc.cc.u32 %1, %5, %9;\n\taddc.cc.u32 %2, %6, %10;\n\taddc.u32 %3, %7, %11;"
        : "=r"(s[0]), "=r"(s[1]), "=r"(s[2]), "=r"(s[3])
        : "r"(x[0]), "r"(x[1]), "r"(x[2]), "r"(x[3]), "r"(y[0]), "r"(y[1]), "r"(y[2]), "r"(y[3]));
  }
};
template <> struct AddChain<5> {
  static __device__ __forceinline__ void run(uint32_t* s, const uint32_t* x, const uint32_t* y) {
    asm("add.cc.u32 %0, %5, %10;\n\taddc.cc.u32 %1, %6, %11;\n\taddc.cc.u32 %2, %7, %12;\n\taddc.cc.u32 %3, %8, %13;\n\taddc.u32 %4, %9, %14;"
        : "=r"(s[0]), "=r"(s[1]), "=r"(s[2]), "=r"(s[3]), "=r"(s[4])
        : "r"(x[0]), "r"(x[1]), "r"(x[2]), "r"(x[3]), "r"(x[4]), "r"(y[0]), "r"(y[1]), "r"(y[2]), "r"(y[3]), "r"(y[4]));
  }
};

// One DP column of the single-block Myers recurrence over NW 32-bit words, adding the column's delta of D at the query's last row to
// `score`. HIN = horizontal delta entering the top row: 0 for HW (free start), +1 for NW/SHW.
// TOP: the query's last row is bit 31 of the last word (ed_small_kernel's HW layout); otherwise it is bit `topbit` of the last word.
// The row shift across words is x * 2 + carry-in (an IMAD on the FMA pipe) with carry-out = hi(x * 2), and the bit-31 score update
// is two mad.hi by 2, which ptxas turns into two LEA.HI instead of the 5 ALU instructions of a read at a variable bit. On an H100
// (400 W) a multiplier ptxas cannot see, which keeps the mad.hi and the carries on the FMA pipe as IMAD.HI, made the K1 kernels
// 3-8 % slower than this form: dgpu_int_peak_mix shows IMADs issuing alongside LOP3s at full rate, but IMAD.WIDE.U32 not.
// SEPW >= 0: the packed layout of ed_pack_kernel, a second query A in the rows below the first separator row, bit `sep` of word SEPW.
// The shift carries A's last-row Ph / Mh into that row; clearing the bit in the new Pv and Mv keeps it at Pv = Mv = 0, so the separator
// stays inert (ed_pack_kernel). A's delta is added to score_a: A's last row, bit s of word SEPW, moves to bit 31 with a plain IMAD by
// mula = 2^(31 - s) on the FMA pipe, then read as above.
template <int NW, int HIN, bool TOP, int SEPW = -1>
__device__ __forceinline__ void myers_column(uint32_t (&Pv)[NW], uint32_t (&Mv)[NW], const uint32_t (&Eq)[NW], uint32_t topbit,
                                             int& score, uint32_t sep = 0, uint32_t mula = 0, int* score_a = nullptr) {
  uint32_t Xv[NW], t[NW], sum[NW], Ph[NW], Mh[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    Xv[w] = Eq[w] | Mv[w];
    t[w] = Eq[w] & Pv[w];
  }
  AddChain<NW>::run(sum, t, Pv);
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    uint32_t Xh = (sum[w] ^ Pv[w]) | Eq[w];
    Ph[w] = Mv[w] | ~(Xh | Pv[w]);
    Mh[w] = Pv[w] & Xh;
  }
  if (TOP) {
    // score += Ph >> 31 (unsigned high word of Ph * 2) - Mh >> 31 (signed high word of Mh * 2: -1 iff bit 31 is set)
    asm("mad.hi.u32 %0, %1, 2, %0;" : "+r"(score) : "r"(Ph[NW - 1]));
    asm("mad.hi.s32 %0, %1, 2, %0;" : "+r"(score) : "r"(Mh[NW - 1]));
  } else {
    score += (int) ((Ph[NW - 1] >> topbit) & 1u) - (int) ((Mh[NW - 1] >> topbit) & 1u);
  }
  if constexpr (SEPW >= 0) {
    const uint32_t pa = Ph[SEPW] * mula, ma = Mh[SEPW] * mula;
    asm("mad.hi.u32 %0, %1, 2, %0;" : "+r"(*score_a) : "r"(pa));
    asm("mad.hi.s32 %0, %1, 2, %0;" : "+r"(*score_a) : "r"(ma));
  }
  // shift Ph / Mh up by one row across the words. Every index is a constant after unrolling, so the column stays in registers
  // (a backward loop with a w == 0 case was left rolled by ptxas and put the arrays on the stack).
  uint32_t ph[NW], mh[NW], cp = HIN, cm = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    ph[w] = Ph[w] * 2u + cp;
    mh[w] = Mh[w] * 2u + cm;
    cp = __umulhi(Ph[w], 2u);
    cm = __umulhi(Mh[w], 2u);
  }
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    Pv[w] = mh[w] | ~(Xv[w] | ph[w]);
    Mv[w] = ph[w] & Xv[w];
    if (w == SEPW) {
      Pv[w] &= ~sep;
      Mv[w] &= ~sep;
    }
  }
}

// symbol slot in the shared Peq table: A0 C1 T2 G3 N4 — the order ((c >> 1) & 3) yields for ACGT, so the fast path
// can turn four target bytes into four table offsets with packed arithmetic
__device__ __forceinline__ uint32_t peq_slot(uint32_t code) { return code < 4 ? (code ^ (code >> 1)) : code; }

// match bits of the four bytes of x that equal the byte s (s < 0x80), byte b -> bit b. Exact: a byte of v = x ^ s*0x01010101 is zero iff
// its low seven bits carry nothing into bit 7 when 0x7f is added and its own bit 7 (that of x) is clear. The multiply moves bits 7, 15, 23,
// 31 to 28..31 without overlapping any other product term.
__device__ __forceinline__ uint32_t match4(uint32_t x, uint32_t s) {
  const uint32_t t = ((x & 0x7f7f7f7fu) ^ (s * 0x01010101u)) + 0x7f7f7f7fu;
  const uint32_t z = ~(t | x) & 0x80808080u;
  return (z * 0x00204081u) >> 28;
}

// x = the slots ((c >> 1) & 3) of four bytes; returns the four bytes ACGT would have at those slots. The byte of slot x is
// 0x41 + 2 x + 15 [x == 2] ('A' 'C' 'T' 'G'), two multiply-adds, so a word is all ACGT iff it equals acgt_bytes((w >> 1) & 0x03030303).
__device__ __forceinline__ uint32_t acgt_bytes(uint32_t x) {
  const uint32_t is_t = (x >> 1) & ~x & 0x01010101u;
  return x * 2u + 0x41414141u + is_t * 15u;
}

// match bits of 32 bytes against the byte s, byte b -> bit b: the exact Peq word of a query word holding a byte outside ACGT. Out of line,
// since such words are rare and the Peq build stays one straight block without them.
__device__ __noinline__ uint32_t match32(uint4 lo, uint4 hi, uint32_t s) {
  const uint32_t wv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  uint32_t e = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) e |= match4(wv[k], s) << (k * 4);
  return e;
}

// exact slow path for a target byte outside ACGTN: byte equality against the query rows q[0..len), len <= 32, bit i = row i. Kept out of
// line so the column loop holds calls instead of one copy of the loop per column slot; one word per call, so the result comes back in a
// register rather than through a stack frame.
__device__ __noinline__ uint32_t eq_word_by_bytes(const uint8_t* q, uint32_t len, uint32_t c) {
  uint32_t e = 0;
  for (uint32_t i = 0; i < len; ++i)
    if (__ldg(q + i) == (uint8_t) c) e |= 1u << i;
  return e;
}

// ed_small_kernel's HW layout: the m query rows move up by p = 32 NW - m (0..31) rows, so that the last one is bit 31 of the last word,
// and the p rows below them become virtual rows that match every target byte (vmask). With HIN = 0 such rows keep Pv = Mv = 0 in every
// column, compute Ph = Mh = 0 and carry nothing into the add chain, so they shift a 0 into the first query row, as the free top row of
// HW does: bit 31 reads D[m][c] in every column. Rows past |q| drop out of the top. With HIN = 1 the rows would not be inert.
template <int NW>
__device__ __forceinline__ void rows_to_top(uint32_t (&e)[NW], uint32_t p, uint32_t vmask) {
#pragma unroll
  for (int w = NW - 1; w > 0; --w) e[w] = __funnelshift_l(e[w - 1], e[w], p);
  e[0] = (e[0] << p) | vmask;
}

// Match masks of one query for the Peq table, in slot order A0 C1 T2 G3 N4; word w of slot s goes to pq[(s * SW + w) * ED_THREADS].
// Per query word: bits 1 and 2 of the 32 bytes are gathered into two 32-row planes (one multiply per plane and 4-byte group moves bit
// 8i + k of the group to bit 28 + i, as match4 does; a funnel shift appends the group below the later ones), and each of A C T G is one
// LOP3 of the planes, with no N row. A word with any byte outside ACGT is built exactly by match32 instead (N rows get the N mask, other
// bytes no bit). Rows past |q| read whatever follows the query in the arena (the reader stays inside it); the last word is masked to |q|, or
// in the HW layout those rows are shifted out.
template <int NW>
__device__ __forceinline__ void peq_words(uint32_t (&pm)[5][NW], const uint8_t* q, const uint8_t* seqs_end) {
  ChunkReader qr;
  qr.init(q, seqs_end);
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    const uint4 lo = qr.next(), hi = qr.next();
    const uint32_t wv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    uint32_t p1 = 0, p2 = 0, bad = 0;
#pragma unroll
    for (int g = 7; g >= 0; --g) {
      const uint32_t x = (wv[g] >> 1) & 0x03030303u;
      bad |= wv[g] ^ acgt_bytes(x);
      p1 = __funnelshift_l((x & 0x01010101u) * 0x10204080u, p1, 4);
      p2 = __funnelshift_l((x & 0x02020202u) * 0x08102040u, p2, 4);
    }
    if (bad == 0) {
      pm[0][w] = ~(p1 | p2);
      pm[1][w] = p1 & ~p2;
      pm[2][w] = p2 & ~p1;
      pm[3][w] = p1 & p2;
      pm[4][w] = 0;
    } else {
      pm[0][w] = match32(lo, hi, 'A');
      pm[1][w] = match32(lo, hi, 'C');
      pm[2][w] = match32(lo, hi, 'T');
      pm[3][w] = match32(lo, hi, 'G');
      pm[4][w] = match32(lo, hi, 'N');
    }
  }
}

template <int NW, bool TOP>
__device__ __forceinline__ void build_peq(uint32_t* pq, int SW, const uint8_t* q, const uint8_t* seqs_end, uint32_t topbit, uint32_t p,
                                          uint32_t vmask) {
  uint32_t pm[5][NW];
  peq_words<NW>(pm, q, seqs_end);
#pragma unroll
  for (int s = 0; s < 5; ++s) {
    if (TOP) rows_to_top<NW>(pm[s], p, vmask);
    else pm[s][NW - 1] &= (2u << topbit) - 1u;
#pragma unroll
    for (int w = 0; w < NW; ++w) pq[(s * SW + w) * ED_THREADS] = pm[s][w];
  }
}

// ---- ed_pack_kernel's layout: two HW queries of one target in one column of R = 32 W rows ----------------------------------------------
// A in rows 0 .. mA-1 (its last row in word WA), B in rows R-mB .. R-1 (its last row bit 31 of word W-1, as in ed_small_kernel's HW
// layout), and between them at least one separator row. Separator rows are virtual rows like those below a query in the HW layout: Eq = 1
// for every byte, Pv = Mv = 0 at the start. The first one (bit mA & 31 of word WA) would take A's last-row Ph / Mh through the shift, so
// myers_column clears it in Pv and Mv (SEPW); every other separator row computes Ph = Mh = 0, carries nothing, and shifts a 0 into the
// row above it, so B's first row sees HW's free top row just as A's row 0 does at the bottom of the column.

// bits of word w that are rows in [lo, hi)
__device__ __forceinline__ uint32_t rows_in(uint32_t w, uint32_t lo, uint32_t hi) {
  auto below = [](int x) { return x <= 0 ? 0u : x >= 32 ? 0xffffffffu : (1u << x) - 1u; };
  return below((int) hi - (int) (32u * w)) & ~below((int) lo - (int) (32u * w));
}

// B's Peq words in the HW layout of its own class, NB = ceil(mB / 32) words, stored as the top NB words of the W-word column (NBMAX >= NB)
template <int W, int NBMAX>
__device__ __forceinline__ void build_peq_top(uint32_t* pq, const uint8_t* q, uint32_t m, const uint8_t* seqs_end) {
  if constexpr (NBMAX > 1) {
    if (m <= 32u * (NBMAX - 1)) {
      build_peq_top<W, NBMAX - 1>(pq, q, m, seqs_end);
      return;
    }
  }
  const uint32_t p = 32u * NBMAX - m;
  build_peq<NBMAX, true>(pq + (W - NBMAX) * ED_THREADS, W, q, seqs_end, 0, p, (1u << p) - 1u);
}

// The packed Peq table of one thread (pq = peq + tid, W words per symbol slot): B's words at the top, words of separator rows only all
// ones, then A's words from the bottom, A's last word WA taking the separator and B rows above mA from what is stored there.
template <int W, int WA>
__device__ __forceinline__ void build_pack_peq(uint32_t* pq, const uint8_t* qa, uint32_t ma, const uint8_t* qb, uint32_t mb,
                                               const uint8_t* seqs_end) {
  build_peq_top<W, W - WA>(pq, qb, mb, seqs_end);
  const uint32_t nb = (mb + 31u) >> 5;
#pragma unroll 1
  for (uint32_t w = WA; w < W - nb; ++w)
#pragma unroll
    for (int s = 0; s < 5; ++s) pq[(s * W + w) * ED_THREADS] = 0xffffffffu;
  uint32_t pm[5][WA + 1];
  peq_words<WA + 1>(pm, qa, seqs_end);
  const uint32_t low = (2u << ((ma - 1u) & 31u)) - 1u;
#pragma unroll
  for (int s = 0; s < 5; ++s) {
#pragma unroll
    for (int w = 0; w < WA; ++w) pq[(s * W + w) * ED_THREADS] = pm[s][w];
    uint32_t& top = pq[(s * W + WA) * ED_THREADS];
    top = (pm[s][WA] & low) | (top & ~low);
  }
}

// word w of the packed column's match mask for a target byte c outside ACGTN (the exact slow path): byte equality in A's and B's rows,
// 1 in the separator rows. Out of line, like eq_word_by_bytes.
__device__ __noinline__ uint32_t pack_eq_word(const uint8_t* qa, uint32_t ma, const uint8_t* qb, uint32_t b0, uint32_t w, uint32_t c) {
  uint32_t e = 0;
  for (uint32_t i = 0; i < 32; ++i) {
    const uint32_t r = 32u * w + i;
    const bool eq = r < ma ? __ldg(qa + r) == (uint8_t) c : r < b0 ? true : __ldg(qb + (r - b0)) == (uint8_t) c;
    e |= (uint32_t) eq << i;
  }
  return e;
}

// NJ (1 or 2) jobs of one thread that share a target: jobs perm[i], ..., perm[i] + NJ - 1 of the class `cls` segment of perm. One target stream,
// one byte decode and one Peq address per column feed NJ independent Myers columns. The Peq table of the thread holds, per symbol slot,
// the NW words of each job's query: peq[(slot * NJ NW + j NW + w) * ED_THREADS + tid].
// WA >= 0 (ed_pack_kernel, NJ = 2, HW): the two queries share ONE column of NW words (the packed layout above build_pack_peq), A = job 0 in
// the bottom rows with its last row in word WA, B = job 1 at the top; job 0 is the call's job perm[i] if the pair fits in that order
// (pack_fits), else perm[i] + 1. The Peq table then holds NW words per slot.
template <int NW, int MODE, bool WANT_END, int NJ, int WA = -1>
__device__ __forceinline__ void ed_small_jobs(const EdArgs& a, uint32_t* peq, int cls) {
  constexpr int HIN = (MODE == DGPU_MODE_HW) ? 0 : 1;
  constexpr bool TOP = (MODE == DGPU_MODE_HW);  // query rows at the top of the bit-vector (rows_to_top)
  constexpr bool PACK = WA >= 0;
  constexpr int NC = PACK ? 1 : NJ;              // Myers columns per thread
  constexpr int SW = NC * NW;                    // Peq words per symbol slot
  static_assert(!PACK || (NJ == 2 && MODE == DGPU_MODE_HW && !WANT_END), "a packed column holds two HW distances");
  static_assert(NJ == 1 || (MODE == DGPU_MODE_HW && !WANT_END), "target-sharing pairs are HW distances");
  const uint32_t cnt = a.counts[cls];
  const uint32_t start = a.counts[ED_START + cls];
  const uint32_t tid = threadIdx.x;
  for (uint32_t idx = blockIdx.x * ED_THREADS + tid; idx < cnt; idx += gridDim.x * ED_THREADS) {
    const uint32_t job0 = a.perm[start + idx];
    const uint32_t n = a.t_len[job0];
    const uint8_t* t = a.seqs + a.t_off[job0];
    uint32_t m[NJ], jid[NJ], topbit[NC], p[NC], vmask[NC];
    const uint8_t* q[NJ];
    uint32_t Pv[NC][NW], Mv[NC][NW];
    uint32_t sep = 0, mula = 0;
    int score[NJ], best[NJ], bpos[NJ], prev[NJ];
    if constexpr (NJ == 2) {
      // a pair or pack slot (HW): the shared Peq table of its two probes if one is published (peq_find), else built here and published
      const uint32_t m0 = a.q_len[job0], m1 = a.q_len[job0 + 1];
      const uint32_t o0 = a.q_off[job0], o1 = a.q_off[job0 + 1];
      const uint32_t sw = PACK && !pack_fits(m0, m1, NW, WA) ? 1u : 0u;
      jid[0] = job0 + sw;
      jid[1] = job0 + (sw ^ 1u);
      m[0] = sw ? m1 : m0;
      m[1] = sw ? m0 : m1;
      q[0] = a.seqs + (sw ? o1 : o0);
      q[1] = a.seqs + (sw ? o0 : o1);
      const uint32_t tag = 0x80000000u | m0 | m1 << 16;
      uint32_t claim;
      const uint4* ent = peq_find(a, o0, o1, tag, claim);
      if (ent) {
        copy_peq<5 * SW>(peq + tid, ent);
      } else {
        if constexpr (PACK) {
          build_pack_peq<NW, WA>(peq + tid, q[0], m[0], q[1], m[1], a.seqs_end);
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint32_t pj = 32u * NW - m[j];
            build_peq<NW, true>(peq + j * NW * ED_THREADS + tid, SW, q[j], a.seqs_end, 0, pj, (1u << pj) - 1u);
          }
        }
        if (claim != ED_PEQ_NONE) peq_publish<5 * SW>(a, claim, o0, o1, tag, peq + tid);
      }
    }
    if constexpr (PACK) {
      p[0] = 32u * NW - m[1];  // first row of B; the separator is rows m[0] .. p[0] - 1
#pragma unroll
      for (int w = 0; w < NW; ++w) { Pv[0][w] = ~rows_in(w, m[0], p[0]); Mv[0][w] = 0; }
      // both through a mov that ptxas cannot see into: a multiplier it knows to be 1 << x becomes a variable SHF.L on the ALU pipe again,
      // and a mask it can rebuild from m[0] is recomputed in the column loop (two ALU instructions per four columns)
      asm("mov.b32 %0, %1;" : "=r"(sep) : "r"(1u << (m[0] & 31u)));
      asm("mov.b32 %0, %1;" : "=r"(mula) : "r"(1u << (31u - ((m[0] - 1u) & 31u))));
      topbit[0] = 0;
      vmask[0] = 0;
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if constexpr (!PACK) {
        if constexpr (NJ == 1) {
          jid[j] = job0 + j;
          m[j] = a.q_len[job0 + j];
          q[j] = a.seqs + a.q_off[job0 + j];
        }
        topbit[j] = (m[j] - 1) & 31u;
        p[j] = 32u * NW - m[j];  // jobs of this class have 32 (NW - 1) < |q| <= 32 NW
        vmask[j] = TOP ? (1u << p[j]) - 1u : 0u;
        if constexpr (NJ == 1) build_peq<NW, TOP>(peq + j * NW * ED_THREADS + tid, SW, q[j], a.seqs_end, topbit[j], p[j], vmask[j]);
#pragma unroll
        for (int w = 0; w < NW; ++w) { Pv[j][w] = 0xffffffffu; Mv[j][w] = 0; }
        Pv[j][0] = ~vmask[j];  // virtual rows start at Pv = Mv = 0
      }
      score[j] = (int) m[j];
      // candidate end position -1 (score m) exists iff |q| % 64 != 0 (edlib's padding columns)
      best[j] = (m[j] & 63u) ? (int) m[j] : 0x7fffffff;
      bpos[j] = -1;
      prev[j] = 0;
    }

    auto track = [&](int j, uint32_t col) {
      if (MODE != DGPU_MODE_NW) {
        if (WANT_END) { if (score[j] < best[j] || (a.last_pos && score[j] == best[j])) { best[j] = score[j]; bpos[j] = (int) col; } }
        else best[j] = min(best[j], score[j]);
      }
    };
    // one column through the table (ACGTN) or the exact slow path (any other byte)
    // column j's Myers step; it updates the score of job j, or in the packed layout those of both jobs (B through the top row, A through
    // word WA)
    auto column = [&](int j, const uint32_t (&Eq)[NW]) {
      myers_column<NW, HIN, TOP, WA>(Pv[j], Mv[j], Eq, topbit[j], score[PACK ? 1 : j], sep, mula, &score[0]);
    };
    auto step = [&](uint32_t c, uint32_t col) {
      const uint32_t code = dna_code(c);
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        uint32_t Eq[NW];
        if (code < 5) {
#pragma unroll
          for (int w = 0; w < NW; ++w) Eq[w] = peq[(peq_slot(code) * SW + j * NW + w) * ED_THREADS + tid];
        } else if (PACK) {
#pragma unroll
          for (int w = 0; w < NW; ++w) Eq[w] = pack_eq_word(q[0], m[0], q[1], p[0], w, c);
        } else {
#pragma unroll
          for (int w = 0; w < NW; ++w) Eq[w] = eq_word_by_bytes(q[j] + w * 32, min(32u, m[j] - w * 32), c);
          if (TOP) rows_to_top<NW>(Eq, p[j], vmask[j]);
        }
        column(j, Eq);
#pragma unroll
        for (int s = PACK ? 0 : j; s < (PACK ? NJ : j + 1); ++s) track(s, col);
      }
    };
    const uint32_t base2 = (tid * 4u) * 0x00010001u;  // this thread's slot offset in both 16-bit halves
    // the four columns of target bytes wd, the first being column col
    auto group4 = [&](uint32_t wd, uint32_t col) {
      // four bytes at once: x = slot of each byte if it is one of ACGT
      const uint32_t x = (wd >> 1) & 0x03030303u;
      if (wd == acgt_bytes(x)) {
        // byte offsets of the four Peq rows, two per register: slot * (SW*512) + tid*4
        const uint32_t offA = (x & 0x00ff00ffu) * (uint32_t) (SW * 4 * ED_THREADS) + base2;          // columns 0 and 2
        const uint32_t offB = ((x >> 8) & 0x00ff00ffu) * (uint32_t) (SW * 4 * ED_THREADS) + base2;   // columns 1 and 3
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const uint32_t pk = (b & 1) ? offB : offA;
          const uint32_t off = (b & 2) ? (pk >> 16) : (pk & 0xffffu);
#pragma unroll
          for (int j = 0; j < NC; ++j) {
            uint32_t Eq[NW];
#pragma unroll
            for (int w = 0; w < NW; ++w) Eq[w] = *(const uint32_t*) ((const char*) peq + off + (j * NW + w) * 4 * ED_THREADS);
            column(j, Eq);
#pragma unroll
            for (int s = PACK ? 0 : j; s < (PACK ? NJ : j + 1); ++s) {
              if (MODE != DGPU_MODE_NW) {
                if (WANT_END) track(s, col + b);
                else if (b & 1) best[s] = min(best[s], min(prev[s], score[s]));  // two columns per three-input min
                else prev[s] = score[s];
              }
            }
          }
        }
      } else {
        // a byte outside ACGT among the four: one rolled copy of the general step per word
#pragma unroll 1
        for (uint32_t b = 0; b < 4; ++b) step((wd >> (b * 8)) & 0xffu, col + b);
      }
    };

    ChunkReader tr;
    tr.init(t, a.seqs_end);
    uint32_t c0 = 0;
    for (; c0 + 16 <= n; c0 += 16) {
      const uint4 v = tr.next();
      const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q4 = 0; q4 < 4; ++q4) group4(wv[q4], c0 + q4 * 4);
    }
    if (c0 < n) {
      // the last 1..15 columns: whole words of four through the same fast block, then 0..3 single columns. No column past |t| is run.
      const uint4 v = tr.next();
      uint32_t w0 = v.x, w1 = v.y, w2 = v.z;
#pragma unroll 1
      for (; c0 + 4 <= n; c0 += 4) {
        group4(w0, c0);
        w0 = w1; w1 = w2; w2 = v.w;
      }
#pragma unroll 1
      for (; c0 < n; ++c0, w0 >>= 8) step(w0 & 0xffu, c0);
    }

#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      int d, e;
      if (MODE == DGPU_MODE_NW) { d = score[j]; e = (int) n - 1; }
      else { d = best[j]; e = bpos[j]; }
      const int kk = a.k ? a.k[jid[j]] : -1;
      d = apply_k(d, kk, MODE, (int) m[j], (int) n);
      a.dist[jid[j]] = d;
      if (a.end_loc) a.end_loc[jid[j]] = (d < 0) ? -1 : e;
    }
  }
}

// Register budget: no occupancy floor (min 1 CTA), so ptxas keeps the column and the job state of every class in registers (56 / 64 / 72
// registers for NW = 1 / 2 / 3, 0 spills). On an H100 (400 W) floors of 8 and 9 CTAs per SM (64 and 56 registers, still no spills) ran
// NW = 1 and 2 at the same speed and NW = 3 1 % slower; floors of 10 and more spill. Without any bound ptxas aims at a higher occupancy
// and spills in some instantiations.
template <int NW, int MODE, bool WANT_END>
__global__ void __launch_bounds__(ED_THREADS, 1) ed_small_kernel(EdArgs a) {
  __shared__ uint32_t peq[5 * NW * ED_THREADS];
  ed_small_jobs<NW, MODE, WANT_END, 1>(a, peq, NW);
}

// One thread per pair of HW jobs on one target (ed_slot): the ALT and REF probes of a genotyping read are realigned in one pass over the
// read, so the target load, its decode, the Peq addresses, the job setup and the tail are paid once for two jobs.
template <int NW>
__global__ void __launch_bounds__(ED_THREADS, 1) ed_pair_kernel(EdArgs a) {
  __shared__ uint32_t peq[5 * 2 * NW * ED_THREADS];
  ed_small_jobs<NW, DGPU_MODE_HW, false, 2>(a, peq, ED_PAIR + NW);
}

// One thread per pair of HW jobs on one target whose two queries fit one column of W words (pack_fits): W = 3 for a 33-63 bp query with a
// partner of up to 95 - |q| bp, W = 5 for 65-95 bp with up to 159 - |q|. Two 33-47 bp probes then take 3 words instead of 2 x 2, two
// 65-79 bp probes 5 instead of 2 x 3, and every word of the column needs one Peq load per target column for both jobs.
template <int W, int WA>
__global__ void __launch_bounds__(ED_THREADS, 1) ed_pack_kernel(EdArgs a) {
  __shared__ uint32_t peq[5 * W * ED_THREADS];
  ed_small_jobs<W, DGPU_MODE_HW, false, 2, WA>(a, peq, W == 3 ? ED_PACK : ED_PACK + 1);
}

// ---- warp-per-job wavefront for |q| > 128 -------------------------------------------
constexpr int EDL_WARPS = 4;  // warps per CTA in the long kernel

template <int MODE, bool EQ>
__global__ void __launch_bounds__(EDL_WARPS * 32) ed_long_kernel(EdArgs a, const uint32_t* list, const uint32_t* list_cnt) {
  __shared__ uint64_t peq_s[EDL_WARPS][5][32];
  // job list: the class-5 segment of perm, or (NW with band passes in front) what the band passes left over
  const uint32_t cnt = list ? *list_cnt : a.counts[5];
  if (!list) list = a.perm + a.counts[ED_START + 5];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const uint32_t gwarp = blockIdx.x * EDL_WARPS + wib;
  const uint32_t nwarps = gridDim.x * EDL_WARPS;
  volatile int8_t* hrow = a.hbuf ? (volatile int8_t*) a.hbuf + (size_t) gwarp * a.hbuf_stride : nullptr;
  const EqTabs tabs = {a.eq_f, a.eq_s, a.eq_cls};

  for (uint32_t idx = gwarp; idx < cnt; idx += nwarps) {
    const uint32_t job = list[idx];
    const uint32_t m = a.q_len[job], n = a.t_len[job];
    const int topbit = (int) ((m - 1) & 63u);
    int score = (int) m;  // D[m][0]; only meaningful on the lane that owns row m-1
    int best = (m & 63u) ? (int) m : 0x7fffffff, bpos = -1;  // end position -1 exists iff |q| % 64 != 0
    stripes<EQ>(peq_s[wib], hrow, a.seqs + a.q_off[job], a.seqs + a.t_off[job], m, n, false, MODE == DGPU_MODE_HW ? 0 : 1, tabs,
                [&](int col, uint64_t Ph, uint64_t Mh) {
                  score += (int) ((Ph >> topbit) & 1ull) - (int) ((Mh >> topbit) & 1ull);   // delta of row m-1
                  if (MODE != DGPU_MODE_NW && (score < best || (a.last_pos && score == best))) { best = score; bpos = col; }
                },
                [](uint32_t, int, uint64_t, uint64_t) {});
    // broadcast the result from the lane that owns row m-1
    const int owner = (int) (((m - 1) & 2047u) >> 6);
    int d = (MODE == DGPU_MODE_NW) ? score : best;
    int e = (MODE == DGPU_MODE_NW) ? (int) n - 1 : bpos;
    d = __shfl_sync(0xffffffffu, d, owner);
    e = __shfl_sync(0xffffffffu, e, owner);
    if (lane == 0) {
      const int kk = a.k ? a.k[job] : -1;
      d = apply_k(d, kk, MODE, (int) m, (int) n);
      a.dist[job] = d;
      if (a.end_loc) a.end_loc[job] = (d < 0) ? -1 : e;
    }
  }
}

// ---- banded passes for long NW jobs (Ukkonen band, src/edlib.cpp:728-929 computes the same cells block-wise) ------------------------
// The reference computes, for a threshold k, only the blocks that intersect the diagonals a path of cost <= k can touch, and doubles
// k (from 64) until the result is <= k (src/edlib.cpp:192-210). The device form of the same idea:
//   * a band pass of class G gives a job to G lanes (32/G jobs per warp). The band is a STAIRCASE of G 64-row blocks: during the 64
//     target columns of chunk J lane p holds block J - A + p (A = blocks above the diagonal, chosen per job from |t| - |q|); lanes
//     are skewed by one step so that a block's horizontal delta reaches the block below by shuffle; after the chunk every lane takes
//     over the block of the lane below (Pv, Mv and the absolute score of the block's last row travel through shared memory), the
//     last lane opens a new block with Pv = 1..1 (the cells left of it are outside the band: +1 per row is an upper bound).
//   * the pass covers every diagonal in [-64(G-1-A), 64A] at every column, so its result s is the exact distance whenever
//     s <= kvalid = 2 * min(64A - max(0,d), 64(G-1-A) - max(0,-d)) + |d|, d = |t| - |q| (Ukkonen's argument), or when the
//     staircase covers the whole matrix. Otherwise the job goes to the next class (band twice as wide), finally to ed_long_kernel.
//   * the first class of a job comes from a cheap upper bound (mismatches on the main diagonal + |d|, ed_band_plan_kernel): when it
//     fits a class that class is certain to succeed; otherwise classes are tried from kvalid >= 64 upwards like the reference does.
// counts[ED_BANDQ + c] = jobs queued for band class c (c < EDB_CLASSES), counts[ED_BANDQ + EDB_CLASSES] = jobs left to ed_long_kernel
__device__ __forceinline__ void band_queue(const EdArgs& a, uint32_t* lists, uint32_t cap, int c, uint32_t job) {
  lists[(size_t) c * cap + atomicAdd(&a.counts[ED_BANDQ + c], 1u)] = job;
}

// first class, from c0 on, that can hold the job and (need >= 0) certifies distances up to `need`, or covers the whole matrix
__device__ __forceinline__ int band_first_class(int c0, int m, int n, int need) {
  const int nblk = (m + 63) >> 6;
  for (int c = c0; c < EDB_CLASSES; ++c) {
    if (nblk > edb_block_cap(c)) continue;
    const BandPlan b = band_plan(edb_lanes(c), m, n);
    if (b.whole || b.kvalid >= need) return c;
  }
  return EDB_CLASSES;
}

__global__ void __launch_bounds__(256) ed_band_plan_kernel(EdArgs a, uint32_t* lists, uint32_t cap) {
  const uint32_t cnt = a.counts[5], start = a.counts[ED_START + 5];
  const int lane = threadIdx.x & 31;
  const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t idx = gwarp; idx < cnt; idx += nwarps) {
    const uint32_t job = a.perm[start + idx];
    const int m = (int) a.q_len[job], n = (int) a.t_len[job];
    const uint8_t* q = a.seqs + a.q_off[job];
    const uint8_t* t = a.seqs + a.t_off[job];
    const int d = n > m ? n - m : m - n;
    int kk = a.k ? a.k[job] : -1;
    if (kk >= 0 && kk < d) {                      // src/edlib.cpp:740-743
      if (lane == 0) { a.dist[job] = -1; if (a.end_loc) a.end_loc[job] = -1; }
      continue;
    }
    const int len = min(m, n);
    int mis = 0;
    for (int i = lane; i < len; i += 32) mis += __ldg(q + i) != __ldg(t + i);
    for (int o = 16; o; o >>= 1) mis += __shfl_xor_sync(0xffffffffu, mis, o);
    int need = mis + d;                           // cost of the gap-free alignment + end gap: an upper bound of the distance
    if (kk >= 0) need = min(need, min(kk, max(m, n)));   // beyond the caller's k the answer is -1 whatever the distance is
    if (lane == 0) {
      int c = band_first_class(0, m, n, need);
      if (c == EDB_CLASSES) c = band_first_class(0, m, n, 64);   // no class certifies the bound: widen step by step like the reference
      band_queue(a, lists, cap, c, job);
    }
  }
}

template <int G, bool EQ>
__global__ void __launch_bounds__(EDB_WARPS * 32) ed_band_kernel(EdArgs a, uint32_t* lists, uint32_t cap) {
  constexpr int CLS = (G == 2) ? 0 : (G == 4) ? 1 : (G == 8) ? 2 : (G == 16) ? 3 : 4;
  constexpr int JPW = 32 / G;                      // jobs per warp
  constexpr int PEQ_JOB = EDB_PEQ_WORDS / JPW;     // Peq words per job
  __shared__ uint64_t peq_s[EDB_WARPS][EDB_PEQ_WORDS];
  __shared__ uint64_t hoP[EDB_WARPS][32], hoM[EDB_WARPS][32];
  __shared__ int hoS[EDB_WARPS][32];
  const uint32_t cnt = a.counts[ED_BANDQ + CLS];
  const uint32_t* list = lists + (size_t) CLS * cap;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int p = lane & (G - 1), grp = lane / G;
  const uint32_t gwarp = blockIdx.x * EDB_WARPS + wib, nwarps = gridDim.x * EDB_WARPS;
  uint64_t* peq = &peq_s[wib][grp * PEQ_JOB];
  const EqTabs tabs = {a.eq_f, a.eq_s, a.eq_cls};

  for (uint32_t base = gwarp * JPW; base < cnt; base += nwarps * JPW) {
    const bool have = base + grp < cnt;
    const uint32_t job = have ? list[base + grp] : 0;
    const int m = have ? (int) a.q_len[job] : 0, n = have ? (int) a.t_len[job] : 0;
    const uint8_t* q = a.seqs + (have ? a.q_off[job] : 0);
    const uint8_t* t = a.seqs + (have ? a.t_off[job] : 0);
    const BandPlan bp = band_plan(G, max(m, 1), max(n, 1));

    __syncwarp();
    band_build_peq<G>(peq, q, m, false, p);
    __syncwarp();

    uint64_t Pv, Mv;
    int sc, blk, plast;
    band_pass<G, EQ>(peq, q, t, m, n, false, bp, hoP[wib], hoM[wib], hoS[wib], tabs, Pv, Mv, sc, blk, [](int, uint64_t, uint64_t) {});
    const int s = band_corner<G>(Pv, Mv, sc, m, n, bp, plast);
    if (have && p == 0) {
      const int kk = a.k ? a.k[job] : -1;
      if (plast >= 0 && plast < G && (bp.whole || s <= bp.kvalid)) {
        const int dd = apply_k(s, kk, DGPU_MODE_NW, m, n);
        a.dist[job] = dd;
        if (a.end_loc) a.end_loc[job] = dd < 0 ? -1 : n - 1;
      } else if (kk >= 0 && min(kk, max(m, n)) <= bp.kvalid) {
        a.dist[job] = -1;                          // every path of cost <= k lies inside the band, and the band found none
        if (a.end_loc) a.end_loc[job] = -1;
      } else {
        band_queue(a, lists, cap, band_first_class(CLS + 1, m, n, bp.kvalid + 1), job);
      }
    }
  }
}

// ---- pipelined host-pointer call: arena prefix needed by each job index range ----------------------------------
constexpr int ED_PIPE_MAX_CHUNKS = 16;          // job index ranges per call
constexpr uint64_t ED_PIPE_MIN_JOBS = 1u << 18; // smallest range worth a separate launch
constexpr int ED_PIPE_PIECES = 32;              // arena upload pieces

__global__ void ed_extent_kernel(const uint32_t* __restrict__ q_off, const uint32_t* __restrict__ q_len,
                                 const uint32_t* __restrict__ t_off, const uint32_t* __restrict__ t_len,
                                 uint32_t n, uint32_t jobs_per, uint32_t arena_bytes, uint32_t* __restrict__ ext) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t e = 0, c = 0;
  if (i < n) {
    const uint64_t a = (uint64_t) q_off[i] + q_len[i], b = (uint64_t) t_off[i] + t_len[i];
    const uint64_t m = a > b ? a : b;
    if (m > arena_bytes) ext[ED_PIPE_MAX_CHUNKS] = 1;   // a sequence outside the caller's arena: the call is refused before any kernel reads it
    e = (uint32_t) (m < arena_bytes ? m : arena_bytes);
    c = i / jobs_per;
  }
  // a block of 256 consecutive jobs spans at most two ranges: reduce per warp when the warp is uniform
  const uint32_t c0 = __shfl_sync(0xffffffffu, c, 0);
  if (__all_sync(0xffffffffu, c == c0 || i >= n)) {
    for (int o = 16; o; o >>= 1) e = max(e, __shfl_xor_sync(0xffffffffu, e, o));
    if ((threadIdx.x & 31) == 0 && e) atomicMax(&ext[c0], e);
  } else if (i < n && e) atomicMax(&ext[c], e);
}

int dgpu_pipe_init(dgpu_ctx* ctx) {
  if (!ctx->copy_stream) DGPU_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  if (!ctx->out_stream) DGPU_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->out_stream, cudaStreamNonBlocking));
  const size_t want = 1 + ED_PIPE_PIECES + ED_PIPE_MAX_CHUNKS;
  while (ctx->pipe_events.size() < want) {
    cudaEvent_t e;
    DGPU_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->pipe_events.push_back(e);
  }
  return DGPU_OK;
}

// The class kernels that take EdArgs alone, [class][want_end]: ed_small for classes 1..4, ed_pair and ed_pack for the target-sharing
// pairs. Pairs return no end locations (EdArgs::pair needs end_loc == nullptr), so their kernel fills both columns. Class 5 is a chain of
// its own (launch_mode).
using EdKernel = void (*)(EdArgs);
template <int MODE>
constexpr EdKernel ED_KERNELS[ED_NCLS][2] = {
    {nullptr, nullptr},
    {ed_small_kernel<1, MODE, false>, ed_small_kernel<1, MODE, true>}, {ed_small_kernel<2, MODE, false>, ed_small_kernel<2, MODE, true>},
    {ed_small_kernel<3, MODE, false>, ed_small_kernel<3, MODE, true>}, {ed_small_kernel<4, MODE, false>, ed_small_kernel<4, MODE, true>},
    {nullptr, nullptr},
    {ed_pair_kernel<1>, ed_pair_kernel<1>}, {ed_pair_kernel<2>, ed_pair_kernel<2>}, {ed_pair_kernel<3>, ed_pair_kernel<3>},
    {ed_pair_kernel<4>, ed_pair_kernel<4>}, {ed_pack_kernel<3, 1>, ed_pack_kernel<3, 1>}, {ed_pack_kernel<5, 2>, ed_pack_kernel<5, 2>}};

// Class 5's kernels: the band pass of each band class and the full matrix, [0] without and [1] with equality tables
using EdBandKernel = void (*)(EdArgs, uint32_t*, uint32_t);
template <bool EQ, size_t... C>
constexpr std::array<EdBandKernel, EDB_CLASSES> ed_band_kernels(std::index_sequence<C...>) {
  return {{ed_band_kernel<edb_lanes(C), EQ>...}};
}
constexpr std::array<EdBandKernel, EDB_CLASSES> ED_BAND_KERNELS[2] = {ed_band_kernels<false>(std::make_index_sequence<EDB_CLASSES>()),
                                                                      ed_band_kernels<true>(std::make_index_sequence<EDB_CLASSES>())};
using EdLongKernel = void (*)(EdArgs, const uint32_t*, const uint32_t*);
template <int MODE>
constexpr EdLongKernel ED_LONG_KERNELS[2] = {ed_long_kernel<MODE, false>, ed_long_kernel<MODE, true>};

template <int MODE>
int launch_mode(dgpu_ctx* ctx, EdArgs& a, const uint32_t* hc, cudaStream_t st) {
  const int sms = ctx->num_sms;
  auto grid_for = [&](uint32_t cnt, int per_block, int max_per_sm) {
    uint32_t need = (cnt + per_block - 1) / per_block;
    uint32_t cap = (uint32_t) (sms * max_per_sm);
    return need < cap ? need : cap;
  };
  const bool want_end = (a.end_loc != nullptr);
  const bool eq = (a.eq_cls != nullptr);
  // Scratch of class 5, reserved before any class kernel of this call is launched (see the note on dgpu_reserve where perm is reserved).
  const bool band = MODE == DGPU_MODE_NW && !ctx->no_band;
  const uint32_t g5 = grid_for(hc[5], EDL_WARPS, 8);
  uint32_t* lists = nullptr;
  a.hbuf = nullptr;
  a.hbuf_stride = 0;
  if (hc[5] && hc[ED_TMAX]) {
    a.hbuf_stride = (hc[ED_TMAX] + 255u) & ~255u;
    void* hb;
    int rc = dgpu_reserve(ctx, SLOT_ED_STRIPES, (size_t) g5 * EDL_WARPS * a.hbuf_stride, &hb);
    if (rc) return rc;
    a.hbuf = (uint8_t*) hb;
  }
  if (hc[5] && band) {
    void* lp;
    int rc = dgpu_reserve(ctx, SLOT_ED_BAND, (size_t) (EDB_CLASSES + 1) * hc[5] * sizeof(uint32_t), &lp);
    if (rc) return rc;
    lists = (uint32_t*) lp;
  }

  // one class on stream cs: ed_small / ed_pair / ed_pack, or class 5's chain in order on one stream (band passes narrowest first, as a
  // pass queues what it could not certify for the next one, then the full matrix; without band passes the full matrix alone)
  auto launch = [&](int c, cudaStream_t cs) -> int {
    if (c != 5) {
      const EdKernel k = ED_KERNELS<MODE>[c][want_end];
      k<<<grid_for(hc[c], ED_THREADS, ED_CTAS_PER_SM), ED_THREADS, 0, cs>>>(a);
      DGPU_LAUNCH_CHECK(ctx, c <= 4 ? "ed_small" : c < ED_PACK ? "ed_pair" : "ed_pack");
      return DGPU_OK;
    }
    const uint32_t *list = nullptr, *list_cnt = nullptr;   // ed_long_kernel's jobs: class 5 of perm, or what the band passes left
    if (band) {
      const uint32_t cap = hc[5];
      ed_band_plan_kernel<<<grid_for(hc[5], 8, 8), 256, 0, cs>>>(a, lists, cap);
      DGPU_LAUNCH_CHECK(ctx, "ed_band_plan");
      for (int bc = 0; bc < EDB_CLASSES; ++bc) {
        const EdBandKernel k = ED_BAND_KERNELS[eq][bc];
        k<<<grid_for(hc[5], EDB_WARPS * (32 / edb_lanes(bc)), 5), EDB_WARPS * 32, 0, cs>>>(a, lists, cap);
        DGPU_LAUNCH_CHECK(ctx, "ed_band");
      }
      list = lists + (size_t) EDB_CLASSES * cap;
      list_cnt = a.counts + ED_BANDQ + EDB_CLASSES;
    }
    const EdLongKernel k = ED_LONG_KERNELS<MODE>[eq];
    k<<<g5, EDL_WARPS * 32, 0, cs>>>(a, list, list_cnt);
    DGPU_LAUNCH_CHECK(ctx, "ed_long");
    return DGPU_OK;
  };

  // The classes are independent once perm is scattered, so they run side by side on the fork/join pool (DgpuFork).
  // Costliest class per job first: the block scheduler starts the CTAs of earlier launches first, so the classes launched last fill the
  // SMs while the long ones drain, where one stream let every class drain the GPU alone.
  static constexpr int order[] = {ED_PACK + 1, ED_PAIR + 2, ED_PAIR + 3, ED_PAIR + 4, ED_PACK, ED_PAIR + 1, 4, 3, 2, 1, 5};
  int nl = 0;
  for (int c : order) nl += hc[c] != 0;
  DgpuFork fork(ctx, st, nl);
  int rc;
  if ((rc = fork.begin())) return rc;
  for (int c : order) {
    if (!hc[c]) continue;
    cudaStream_t cs;
    if ((rc = fork.next(cs)) || (rc = launch(c, cs))) return rc;
  }
  return fork.end();
}

}  // namespace

// Internal entry shared with edit_path.cu: last_pos selects the last optimal end position; async_bound > 0 launches without reading the class
// counts back, with the stripe scratch sized for sequences of up to that length (dgpu_set_async_bound).
int dgpu_edit_distance_impl(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* q_off, const uint32_t* q_len,
                            const uint32_t* t_off, const uint32_t* t_len,
                            const int32_t* k, int mode, uint64_t n,
                            int32_t* dist, int32_t* end_loc, void* stream, int last_pos, const uint32_t* eq_tabs, uint32_t async_bound);

extern "C" {

int dgpu_edit_distance_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                           const uint32_t* q_off, const uint32_t* q_len,
                           const uint32_t* t_off, const uint32_t* t_len,
                           const int32_t* k, int mode, uint64_t n,
                           int32_t* dist, int32_t* end_loc, void* stream) {
  return dgpu_edit_distance_impl(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, k, mode, n, dist, end_loc, stream, 0, nullptr, ctx ? ctx->async_bound : 0);
}

}  // extern "C"

int dgpu_edit_distance_impl(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* q_off, const uint32_t* q_len,
                            const uint32_t* t_off, const uint32_t* t_len,
                            const int32_t* k, int mode, uint64_t n,
                            int32_t* dist, int32_t* end_loc, void* stream, int last_pos, const uint32_t* eq_tabs, uint32_t async_bound) {
  if (!ctx) return DGPU_ERR_ARG;
  if (mode != DGPU_MODE_NW && mode != DGPU_MODE_SHW && mode != DGPU_MODE_HW) return DGPU_ERR_ARG;
  if (n == 0) return DGPU_OK;
  if (n >= (1ull << 31) || seqs_bytes >= (1ull << 32)) return DGPU_ERR_ARG;
  if (!seqs || !q_off || !q_len || !t_off || !t_len || !dist) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t) stream : ctx->stream;

  EdArgs a;
  a.seqs = seqs; a.seqs_end = seqs + seqs_bytes;
  a.q_off = q_off; a.q_len = q_len; a.t_off = t_off; a.t_len = t_len; a.k = k;
  a.n = (uint32_t) n; a.dist = dist; a.end_loc = end_loc;
  a.hbuf = nullptr; a.hbuf_stride = 0;
  a.last_pos = last_pos;
  a.pair = (mode == DGPU_MODE_HW && !end_loc && !eq_tabs) ? 1 : 0;
  // eq_tabs (device): uint32 f[256], uint32 s[256], then uint8 cls[256]
  a.eq_f = eq_tabs; a.eq_s = eq_tabs ? eq_tabs + 256 : nullptr; a.eq_cls = eq_tabs ? (const uint8_t*) (eq_tabs + 512) : nullptr;
  a.force_long = eq_tabs ? 1 : 0;
  // The class kernels of an earlier call may still run on the pool streams (launch_mode) and read this scratch. A call on the same stream
  // is ordered after them by the join. A slot that has to grow is freed with cudaFree, which synchronises the whole device, so the old
  // buffer is idle whichever stream the earlier call used. dgpu_reserve must keep freeing that way.
  void* p;
  int rc = dgpu_reserve(ctx, SLOT_JOB_PERM, n * sizeof(uint32_t), &p);
  if (rc) return rc;
  a.perm = (uint32_t*) p;
  rc = dgpu_reserve(ctx, SLOT_COUNTS, ED_COUNTS_WORDS * sizeof(uint32_t), &p);
  if (rc) return rc;
  a.counts = (uint32_t*) p;
  rc = dgpu_reserve(ctx, SLOT_ED_SLOTS, n + 16, &p);   // ed_scatter_kernel reads whole words
  if (rc) return rc;
  a.slots = (uint8_t*) p;

  DGPU_CUDA(ctx, cudaMemsetAsync(a.counts, 0, ED_COUNTS_WORDS * sizeof(uint32_t), st));
  a.peq_slots = a.peq_pool = nullptr;
  a.peq_mask = 0;
  if (a.pair) {   // the shared Peq tables of pairs (ED_PEQ_SLOTS_V), cleared on st: no entry outlives the call
    uint32_t hs = ED_PEQ_SLOTS_MIN;
    while (hs < n && hs < ED_PEQ_SLOTS_MAX) hs <<= 1;
    rc = dgpu_reserve(ctx, SLOT_ED_PEQ, (size_t) hs * (sizeof(uint4) + ED_PEQ_WORDS * sizeof(uint32_t)), &p);
    if (rc) return rc;
    a.peq_slots = (uint4*) p;
    a.peq_pool = a.peq_slots + hs;
    a.peq_mask = hs - 1;
    DGPU_CUDA(ctx, cudaMemsetAsync(a.peq_slots, 0xff, (size_t) hs * sizeof(uint4), st));
  }
  const uint32_t cb = (uint32_t) std::min<uint64_t>((n + ED_BIN_THREADS - 1) / ED_BIN_THREADS, (uint64_t) ctx->num_sms * ED_BIN_CTAS_PER_SM);
  ed_count_kernel<<<cb, ED_BIN_THREADS, 0, st>>>(a, mode);
  DGPU_LAUNCH_CHECK(ctx, "ed_count");
  ed_scatter_kernel<<<cb, ED_BIN_THREADS, 0, st>>>(a);
  DGPU_LAUNCH_CHECK(ctx, "ed_scatter");
  uint32_t hc[ED_TMAX + 1];
  if (async_bound) {
    // Asynchronous form (dgpu_set_async_bound, or the edit path's bound): no host round trip. Every class is launched with a grid sized from the job count (the kernels
    // read their own class counts on the device and an empty class returns at once), the stripe scratch of long targets from the caller's bound.
    for (uint32_t& c : hc) c = 0;
    const uint32_t bound = async_bound;
    hc[1] = hc[2] = (uint32_t) n;
    if (bound > 64) hc[3] = (uint32_t) n;
    if (bound > 96) hc[4] = (uint32_t) n;
    if (bound > 128 || a.force_long) { hc[5] = (uint32_t) n; if (bound > 2048) hc[ED_TMAX] = bound; }
    if (a.pair) {   // a pair takes two jobs
      hc[ED_PAIR + 1] = hc[ED_PAIR + 2] = (uint32_t) (n / 2);
      if (bound > 64) hc[ED_PAIR + 3] = (uint32_t) (n / 2);
      if (bound > 96) hc[ED_PAIR + 4] = (uint32_t) (n / 2);
      hc[ED_PACK] = (uint32_t) (n / 2);
      if (bound > 64) hc[ED_PACK + 1] = (uint32_t) (n / 2);
    }
  } else {
    // One small D2H so that launches are sized exactly and empty classes cost nothing.
    DGPU_CUDA(ctx, cudaMemcpyAsync(hc, a.counts, sizeof(hc), cudaMemcpyDeviceToHost, st));
    DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  }

  if (mode == DGPU_MODE_HW) return launch_mode<DGPU_MODE_HW>(ctx, a, hc, st);
  if (mode == DGPU_MODE_SHW) return launch_mode<DGPU_MODE_SHW>(ctx, a, hc, st);
  return launch_mode<DGPU_MODE_NW>(ctx, a, hc, st);
}

extern "C" {

int dgpu_edit_distance(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                       const uint32_t* q_off, const uint32_t* q_len,
                       const uint32_t* t_off, const uint32_t* t_len,
                       const int32_t* k, int mode, uint64_t n,
                       int32_t* dist, int32_t* end_loc) {
  DgpuStage s(ctx, "dgpu_edit_distance", n);
  if (!ctx) return DGPU_ERR_ARG;
  if (n == 0) return DGPU_OK;
  if (!seqs || !q_off || !q_len || !t_off || !t_len || !dist) return DGPU_ERR_ARG;
  if (n >= (1ull << 31) || seqs_bytes >= (1ull << 32)) return DGPU_ERR_ARG;
  const uint64_t njc = std::min<uint64_t>(ED_PIPE_MAX_CHUNKS, n / ED_PIPE_MIN_JOBS);
  const bool pipelined = njc >= 2 && seqs_bytes >= (32u << 20);
  int rc;
  // caller buffers: every sequence inside the arena. Small batches are checked here; the pipelined path below checks on the device while it
  // reduces the arena extents (a host loop over 10 M jobs would read 160 MB before the first upload)
  if (!pipelined && ((rc = s.check_arena(seqs_bytes, n, q_off, q_len)) || (rc = s.check_arena(seqs_bytes, n, t_off, t_len)))) return rc;
  if ((rc = s.open())) return rc;
  cudaStream_t st = s.st;
  if (pipelined) {   // the job metadata goes up on the copy stream, the arena piece by piece below
    if ((rc = dgpu_pipe_init(ctx))) return rc;
    s.up = ctx->copy_stream;
  }
  uint8_t* d_seqs = s.arena(pipelined ? nullptr : seqs, seqs_bytes);
  uint32_t *d_qoff = s.in(q_off, n), *d_qlen = s.in(q_len, n), *d_toff = s.in(t_off, n), *d_tlen = s.in(t_len, n);
  int32_t* d_k = s.in(k, n);
  int32_t *d_dist = s.out(dist, n), *d_end = s.out(end_loc, n);
  uint32_t* d_ext = pipelined ? s.alloc<uint32_t>(ED_PIPE_MAX_CHUNKS + 1) : nullptr;
  if (s.rc) { cudaStreamSynchronize(s.up); return s.rc; }   // uploads already queued read the caller's arrays

  // Small batches: one copy-in, one pass, one copy-out on the context stream.
  if (!pipelined) {
    if ((rc = dgpu_edit_distance_dev(ctx, d_seqs, seqs_bytes, d_qoff, d_qlen, d_toff, d_tlen, d_k, mode, n, d_dist, d_end, st))) return rc;
    return s.finish();
  }

  // Large batches (the genotyping batch of src/coverage.h:412-454 is 131072 x threads jobs): the call is PCIe-bound
  // (about 100 input bytes per job against 0.5 ns of kernel time), so the arena upload is pipelined against the
  // kernels. The job metadata goes first; the arena follows in ED_PIPE_PIECES pieces on a copy stream; the jobs
  // are cut into njc index ranges, and range c is launched as soon as the arena prefix it reads (its largest
  // q_off+q_len / t_off+t_len, reduced on the device from the uploaded metadata) has arrived. Results of a
  // finished range go back on a third stream, not through s.finish(). Any job order is correct; arena-ordered
  // jobs (the way batches are built: reads appended as they are scanned) overlap fully.
  cudaStream_t cs = ctx->copy_stream, os = ctx->out_stream;
  cudaEvent_t* ev = ctx->pipe_events.data();  // [0] metadata, [1..PIECES] arena pieces, [1+PIECES..] range done
  DGPU_CUDA(ctx, cudaEventRecord(ev[0], cs));
  const uint64_t piece = (((seqs_bytes + ED_PIPE_PIECES - 1) / ED_PIPE_PIECES) + 0xfffffull) & ~0xfffffull;  // 1 MiB multiple
  int npieces = 0;
  for (uint64_t o = 0; o < seqs_bytes; o += piece, ++npieces) {
    const uint64_t len = std::min<uint64_t>(piece, seqs_bytes - o);
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_seqs + o, seqs + o, len, cudaMemcpyHostToDevice, cs));
    DGPU_CUDA(ctx, cudaEventRecord(ev[1 + npieces], cs));
  }
  // an even range size, so that no range starts on the odd member of a target-sharing pair (ed_slot pairs jobs 2i and 2i + 1 of a call)
  const uint64_t jobs_per = (((n + njc - 1) / njc) + 1) & ~1ull;
  DGPU_CUDA(ctx, cudaStreamWaitEvent(st, ev[0], 0));
  DGPU_CUDA(ctx, cudaMemsetAsync(d_ext, 0, (ED_PIPE_MAX_CHUNKS + 1) * sizeof(uint32_t), st));
  ed_extent_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(d_qoff, d_qlen, d_toff, d_tlen, (uint32_t) n, (uint32_t) jobs_per, (uint32_t) seqs_bytes, d_ext);
  DGPU_LAUNCH_CHECK(ctx, "ed_extent");
  uint32_t h_ext[ED_PIPE_MAX_CHUNKS + 1];
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_ext, d_ext, sizeof(h_ext), cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  if (h_ext[ED_PIPE_MAX_CHUNKS]) {
    cudaStreamSynchronize(cs);   // the arena upload reads the caller's buffer only inside seqs_bytes; let it drain
    ctx->last_error = "dgpu_edit_distance: a sequence lies outside the arena";
    return DGPU_ERR_ARG;
  }
  for (uint64_t c = 0; c < njc; ++c) {
    const uint64_t j0 = c * jobs_per;
    if (j0 >= n) break;
    const uint64_t cnt = std::min<uint64_t>(jobs_per, n - j0);
    const int need = h_ext[c] ? (int) ((h_ext[c] - 1) / piece) : 0;   // last arena piece this range reads
    DGPU_CUDA(ctx, cudaStreamWaitEvent(st, ev[1 + std::min(need, npieces - 1)], 0));
    rc = dgpu_edit_distance_dev(ctx, d_seqs, seqs_bytes, d_qoff + j0, d_qlen + j0, d_toff + j0, d_tlen + j0, d_k ? d_k + j0 : nullptr, mode, cnt,
                                d_dist + j0, d_end ? d_end + j0 : nullptr, st);
    if (rc) { cudaStreamSynchronize(cs); return rc; }
    cudaEvent_t done = ev[1 + ED_PIPE_PIECES + c];
    DGPU_CUDA(ctx, cudaEventRecord(done, st));
    DGPU_CUDA(ctx, cudaStreamWaitEvent(os, done, 0));
    DGPU_CUDA(ctx, cudaMemcpyAsync(dist + j0, d_dist + j0, cnt * 4, cudaMemcpyDeviceToHost, os));
    if (end_loc) DGPU_CUDA(ctx, cudaMemcpyAsync(end_loc + j0, d_end + j0, cnt * 4, cudaMemcpyDeviceToHost, os));
  }
  DGPU_CUDA(ctx, cudaStreamSynchronize(cs));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(os));
  return DGPU_OK;
}

}  // extern "C"
