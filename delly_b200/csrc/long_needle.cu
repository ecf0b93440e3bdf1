// long_needle.cu — batched consensus-vs-SV-reference split alignment, the device replacement for
// longNeedle() (src/needle.h:45-222) as instantiated by _consRefAlignment (src/split.h:540-558):
// AlignConfig<true,false>, DnaScore(1,-1,-1,-1) => linear gaps, row 0 free, last row moves right free.
//
// Reference semantics reproduced bit-for-bit:
//   * forward DP on (s1,s2) and a second DP on (revcomp s1, revcomp s2) (needle.h:59-81, revcomp per
//     src/util.h:549-563 incl. its handling of non-ACGTN bytes);
//   * false if mat[m][n] != rev[m][n] (:83-86);
//   * best join: first strict maximum in row-major order of prefmax(mat[row])[col] +
//     prefmax(rev[m-row])[n-col] (:88-115); refRight = LAST right in [0,n-refLeft] with
//     mat[consLeft][refLeft] + rev[consRight][right] == bestScore (:116-123); false if no gain (:152);
//   * tracebacks with priority vertical > horizontal > diagonal (:155-192) and the stitched
//     2 x alilen alignment (:196-219), bytes other than ACGTN- in the reverse part left as '\0'.
//
// Device design (see wavefront.cuh): ONE WARP (short-read shapes) or one CTA (long-read shapes) PER
// ALIGNMENT, anti-diagonal wavefront with C columns per thread held in registers. The reverse pass stores,
// per cell, the running prefix maximum of its row (int16, column-mirrored) plus a 4-bit nibble (traceback
// direction + "cell equals the row maximum so far"); the forward pass never materialises mat: it carries the
// running maximum of its own row across threads and evaluates the join of needle.h:104-115 on the fly
// against the stored reverse maxima, keeping a per-thread arg-max in row-major first-max order that is
// reduced once at the end. refRight (needle.h:116-123) is recovered from the stored maxima and the
// "equals maximum" bits. Workspace ~3 B per DP cell (0.8 MB for 300x1100; a batch in flight exceeds L2 and streams
// through HBM at about 1 TB/s, far below the roof).
// Job geometry (ln_geom): up to 1273 reference columns one warp with C = 8..40 columns per lane;
// up to 2041 two warps x C=32; up to 4089 four warps x C=32; up to 16377 eight warps x C = 24..64 (ln_ups: C >= 48 keeps the
// scalar engine's previous-row state in shared memory), chosen so that at least 3/4 of the lanes own columns. Warps of one CTA hand the
// boundary column over through a shared-memory ring (wavefront.cuh), not a block barrier. The two tracebacks are
// warp-cooperative (a diagonal window of direction words per round of loads). Job classes of one call run concurrently on
// forked streams.
#include "common.cuh"
#include "wavefront.cuh"
#include "wavefront2.cuh"
#include <algorithm>
#include <array>
#include <string>
#include <utility>
#include <vector>

namespace {

constexpr int LN_NCLS = 16;  // 0 trivial; 1..15 the rows of ln_geom
constexpr int LN_GEN = 16;   // class + LN_GEN: the same geometry for jobs with a byte outside ACGTN (scalar engine, byte compares)

// Workspace plan of one class (ln_fit): the class's slabs start at `base` inside the workspace, and only the first `grid` CTAs of its launch
// take jobs.
struct LnPlan {
  unsigned long long base, work_stride, off_dirsR, off_dirsF, off_trace;
  uint32_t grid;
};

struct LnArgs {
  const uint8_t* seqs;
  const uint32_t* c_off;
  const uint32_t* c_len;
  const uint32_t* r_off;
  const uint32_t* r_len;
  uint32_t n;
  uint8_t* aln;             // output arena
  const uint64_t* aln_off;  // per job: offset of row 0; row 1 at +(m+n)
  uint32_t* aln_len;
  uint8_t* ok;
  int32_t* info;            // optional per job [consLeft, refLeft, refRight, bestScore] (may be NULL)
  uint32_t* perm;
  uint32_t* counts;              // [0..31] class counts (16.. = generic), [32..63] starts, [64..95] cursors
  unsigned long long* maxcells;  // per class max: [0..31] prefix-maxima bytes (wide class: slab bytes), [32..63] direction bytes of one pass,
                                 // [64..95] m+n, [96..127] m
  uint8_t* jobcls;               // per job: its class (0..31), written by the count kernel
  uint8_t* work;                 // per-CTA workspace slabs
  size_t work_stride;
  size_t off_dirsR, off_dirsF, off_trace;  // offsets inside a slab (reverse prefix maxima at 0)
  uint32_t max_ref;              // widest window the wide engine takes (0: none, the dgpu_long_needle forms)
  unsigned long long wide_budget;  // workspace bytes one wide job may take
  uint32_t bound_cons, bound_ref;  // dgpu_set_ln_async_bound (0: none): jobs beyond it are refused
  const LnPlan* plan;            // per class, under the bound (the PLAN kernels); else work / work_stride / off_* and the launch grid hold
};

// The workspace slab of this CTA and the CTAs that take jobs, from the plan (PLAN) or from the arguments and the launch. The class kernels
// are compiled both ways, so that reading the plan costs the kernels of the synchronous forms no registers.
struct LnCta { uint8_t* slab; size_t off_dirsR, off_dirsF, off_trace; uint32_t grid; };
template <bool PLAN>
__device__ __forceinline__ LnCta ln_cta(const LnArgs& a, int cls) {
  if (!PLAN) return {a.work + (size_t) blockIdx.x * a.work_stride, a.off_dirsR, a.off_dirsF, a.off_trace, gridDim.x};
  const LnPlan& p = a.plan[cls];
  return {a.work + p.base + (size_t) blockIdx.x * p.work_stride, (size_t) p.off_dirsR, (size_t) p.off_dirsF, (size_t) p.off_trace, p.grid};
}

// Geometry of the wavefront job classes: a job whose n reference columns satisfy n + 7 <= cap (7 columns of slack for the aligned
// forward blocks) and not the previous row's cap takes the row's class, C columns per lane and T threads per CTA (MULTI: T > 32).
// Classes 1..5 one warp; 6..8 two warps x C=32 (one warp with C = 48..64 would spill); 9 four warps; 10..15 eight warps. Multi-warp
// CTAs are sized so that at least 3/4 of their lanes own columns (idle lanes are idle issue slots).
struct LnGeom { uint32_t cap; int C, T; };
__host__ __device__ constexpr LnGeom ln_geom(int cls) {
  constexpr LnGeom rows[LN_NCLS] = {{0, 0, 0},
                                    {256, 8, 32}, {512, 16, 32}, {768, 24, 32}, {1024, 32, 32}, {1280, 40, 32},
                                    {1536, 32, 64}, {1792, 32, 64}, {2048, 32, 64},
                                    {4096, 32, 128},
                                    {6144, 24, 256}, {8192, 32, 256}, {10240, 40, 256}, {12288, 48, 256}, {14336, 56, 256}, {16384, 64, 256}};
  return rows[cls];
}
// Packed engine: CTAs per SM its register allocation is sized for (12 warps per SM; one 8-warp CTA), and the depth of its partner ring
// (wavefront2.cuh).
__host__ __device__ constexpr int ln2_occ(int T) { return 12 * 32 / T; }
constexpr int LN_PART_D = 2;
// Scalar engine: CTAs per SM of the grid cap (8 warps per SM at up to 255 registers per thread), and whether the C columns of row state do
// not fit the register file and live in shared memory (wavefront.cuh).
__host__ __device__ constexpr int ln_per_sm(int T) { return T == 32 ? 16 : 256 / T; }
__host__ __device__ constexpr bool ln_ups(int C, int T) { return T > 32 && C >= 48; }
// row geometry for n reference columns with C columns per thread (see wavefront.cuh)
__host__ __device__ inline uint32_t ln_nact(uint32_t n, uint32_t C) { return (n + C - 1) / C; }
__host__ __device__ inline uint32_t ln_P(uint32_t n, uint32_t C) { return 1 + ln_nact(n, C) * C; }
__host__ __device__ inline uint32_t ln_bstride(uint32_t n, uint32_t C) { return ln_nact(n, C) * C + C + 16; }  // P-1 .. + pad for overhanging forward blocks
__host__ __device__ inline uint32_t ln_dstride(uint32_t n, uint32_t C) { return (ln_nact(n, C) + 1) * (C / 8); }

// class by number of reference columns n: -1 unsupported
__host__ __device__ inline int ln_class(uint32_t m, uint32_t n) {
  if (m == 0 || n == 0) return 0;
  if ((uint64_t) m + n > 32000u) return -1;  // int16 score storage
  for (int c = 1; c < LN_NCLS; ++c)
    if (n + 7 <= ln_geom(c).cap) return c;
  return -1;
}

// Dynamic shared memory of ln_kernel2, carved in this order: the partner ring of the forward pass (bytes), the row scratch of the join's
// arg-max search (words), the row string of the current pass (m bytes).
struct Ln2Smem {
  size_t ring, scr;
  size_t bytes(size_t mmax) const { return ring + scr * sizeof(uint32_t) + ((mmax + 15) & ~(size_t) 15); }
};
__host__ __device__ inline Ln2Smem ln2_smem(int C, int T) { return {(size_t) wf2::part_slots(C, LN_PART_D, T) * sizeof(uint4), (size_t) (C + 1) * T}; }
// Dynamic shared memory of ln_kernel: the previous-row state (ln_ups classes), then the row string of the current pass (m bytes).
__host__ __device__ constexpr size_t ln_smem_ups(int C, int T) { return ln_ups(C, T) ? (size_t) C * T * sizeof(int) : 0; }
// Workspace of one job: the reverse pass's prefix maxima and the direction nibbles of one pass. The packed engine's workspace is step-major
// (wavefront2.cuh), the scalar engine's row-major.
struct LnParts { unsigned long long rev, dirs; };
__host__ __device__ inline LnParts ln2_parts(int C, int T, uint32_t m) { return {wf2::ws_brev_bytes(C, (int) m, T), wf2::ws_dirs_bytes(C, (int) m, T)}; }
__host__ __device__ inline LnParts ln_parts(int C, uint32_t m, uint32_t n) {
  return {(m + 1ull) * ln_bstride(n, C) * sizeof(int16_t), (m + 1ull) * ln_dstride(n, C) * sizeof(uint32_t)};
}
// Slab layout of a class from the maxima over its jobs: prefix maxima, reverse direction nibbles, forward direction nibbles, then the four
// trace strings of m + n bytes.
__host__ __device__ inline void ln_slab(LnPlan& a, unsigned long long rev, unsigned long long dirs, unsigned long long mn) {
  auto al = [](unsigned long long x) { return (x + 255) & ~255ull; };
  a.off_dirsR = al(rev + 1024);
  a.off_dirsF = a.off_dirsR + al(dirs + 1024);
  a.off_trace = a.off_dirsF + al(dirs + 1024);
  a.work_stride = a.off_trace + al(4 * mn + 64);
}

// ---- wide-window engine geometry (lnw_kernel below) --------------------------------------------------------------------------------
// Jobs beyond ln_class's shapes. One 512-thread CTA per job computes the DP one whole ROW at a time: thread t owns J consecutive chunks
// of 8 columns, the row's horizontal dependency is resolved by a block-wide max-scan, and the previous row lives in shared memory as int16
// row-shifted scores U = H + r in [0, 2m]. So |cons| <= 16383 (LNW_MAX_CONS) is what int16 allows, and the window is bounded only by
// shared memory (DGPU_LN_MAX_REF). Reverse prefix maxima are stored column-mirrored (element x at index n + 7 - x) and the reverse pass's
// chunks start at column o <= 1 (o = n mod 8), so that both the reverse pass's stores and the forward pass's partner loads are aligned
// 16-byte vectors. Workspace per job: 2 B (prefix maxima) + 2 x 0.5 B (direction nibbles) per cell.
constexpr int LN_WIDE = LN_GEN;           // job class of the wide engine (class 0 + LN_GEN is never a class of the wavefront kernels)
constexpr int LNW_THREADS = 512;
constexpr int LNW_JMAX = 17;              // chunks per thread at DGPU_LN_MAX_REF: ceil(8193 / 512), odd
constexpr uint32_t LNW_MAX_CONS = 16383;  // int16 row-shifted scores: U <= 2m <= 32766
static_assert(((DGPU_LN_MAX_REF + 6) / 8 + 1 + LNW_THREADS - 1) / LNW_THREADS <= LNW_JMAX, "LNW_JMAX below the chunks of the widest window");

struct LnwGeom {
  int o;                     // first column of the reverse pass's chunk grid (o <= 1, o = n mod 8); the forward grid starts at 1
  uint32_t nqR, nqF;         // chunks of 8 columns of the reverse / forward pass
  uint32_t bstride;          // int16 per row of reverse prefix maxima
  uint32_t dstride;          // nibble words per row of directions
  unsigned long long off_dirsR, off_dirsF, off_trace, bytes;   // slab layout
};
__host__ __device__ inline unsigned long long lnw_al(unsigned long long x) { return (x + 255) & ~255ull; }
__host__ __device__ inline LnwGeom lnw_geom(uint32_t m, uint32_t n) {
  LnwGeom g;
  g.o = 1 - (int) ((1u - n) & 7u);
  g.nqR = (uint32_t) ((int) n - g.o) / 8 + 1;
  g.nqF = (n + 7) / 8;
  g.bstride = (n + 15 + 7) & ~7u;     // mirrored indices reach n + 13 (the grid's columns <= 0)
  g.dstride = g.nqR;
  const unsigned long long rows = (unsigned long long) m + 1;
  g.off_dirsR = lnw_al(rows * g.bstride * 2);
  g.off_dirsF = g.off_dirsR + lnw_al(rows * g.dstride * 4);
  g.off_trace = g.off_dirsF + lnw_al(rows * g.dstride * 4);
  g.bytes = g.off_trace + lnw_al(4ull * (m + n) + 64);
  return g;
}
// dynamic shared memory of lnw_kernel for windows up to max_ref and consensus up to mmax
inline size_t lnw_smem(uint32_t max_ref, size_t mmax) {
  const size_t nq = (max_ref + 6) / 8 + 1;
  return ((2 * (8 * nq + 8) + 15) & ~(size_t) 15) + 8 * nq + ((mmax + 15) & ~(size_t) 15);
}

// one WARP per job: class by shape, and whether every byte of both sequences is one of ACGTN (then the packed engine applies)
__global__ void ln_count_kernel(LnArgs a, unsigned long long* unsupported) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= a.n) return;
  const uint32_t m = a.c_len[i], n = a.r_len[i];
  int c = ln_class(m, n);
  if (c < 0 && n <= a.max_ref && m <= LNW_MAX_CONS && lnw_geom(m, n).bytes <= a.wide_budget) c = LN_WIDE;
  if (a.bound_cons && (m > a.bound_cons || n > a.bound_ref)) c = -1;
  if (c < 0) {   // beyond the kernel's shapes: this ONE job is reported as not aligned (ok = 0, info[2] = -1) and counted; the batch goes on
    if (lane == 0) {
      atomicAdd(unsupported, 1ull);
      a.jobcls[i] = 0; atomicAdd(&a.counts[0], 1u);
      a.ok[i] = 0; a.aln_len[i] = 0;
      if (a.info) { a.info[4 * i] = 0; a.info[4 * i + 1] = 0; a.info[4 * i + 2] = -1; a.info[4 * i + 3] = 0; }
    }
    return;
  }
  if (c > 0 && c != LN_WIDE) {   // (the wide engine compares bytes)
    bool bad = false;
    const uint8_t* s1 = a.seqs + a.c_off[i];
    const uint8_t* s2 = a.seqs + a.r_off[i];
    for (uint32_t k = lane; k < m; k += 32) bad |= !wf2::hot_ok(__ldg(s1 + k));
    for (uint32_t k = lane; k < n; k += 32) bad |= !wf2::hot_ok(__ldg(s2 + k));
    if (__any_sync(0xffffffffu, bad)) c += LN_GEN;
  }
  if (lane != 0) return;
  a.jobcls[i] = (uint8_t) c;
  atomicAdd(&a.counts[c], 1u);
  if (c == 0) { a.ok[i] = 0; a.aln_len[i] = 0; return; }
  atomicMax(&a.maxcells[96 + c], (unsigned long long) m);
  if (c == LN_WIDE) {   // slab bytes: the wide kernel lays its slab out per job (lnw_geom)
    atomicMax(&a.maxcells[c], lnw_geom(m, n).bytes);
    return;
  }
  const LnGeom g = ln_geom(c & (LN_GEN - 1));
  const LnParts p = c < LN_GEN ? ln2_parts(g.C, g.T, m) : ln_parts(g.C, m, n);
  atomicMax(&a.maxcells[c], p.rev);
  atomicMax(&a.maxcells[32 + c], p.dirs);
  atomicMax(&a.maxcells[64 + c], (unsigned long long) (m + n));
}

__global__ void ln_offsets_kernel(uint32_t* counts) {
  uint32_t s = 0;
  for (int c = 0; c < 32; ++c) { counts[32 + c] = s; counts[64 + c] = s; s += counts[c]; }
}

__global__ void ln_scatter_kernel(LnArgs a) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int c = a.jobcls[i];
  uint32_t p = atomicAdd(&a.counts[64 + c], 1u);
  a.perm[p] = i;
}

// The workspace plan pl[2 * LN_NCLS] of both forms from the class counts and the maxima over each class's jobs (ln_count_kernel's layout),
// within `limit` bytes; cap[c] = the most CTAs class c may take (0: not launched). Returns the bytes the plan takes. Every launched non-empty
// class gets the slab of its largest job and min(count, cap) CTAs. The wide class's slabs are hundreds of MB, so it takes what the ordinary
// classes leave, keeping them up to half of the limit and never less than one CTA each; if the ordinary classes still ask for more than the
// rest, each keeps one CTA and the CTAs above that are cut by one factor, so that the plan fits. A limit that cannot hold one CTA of every
// class leaves each class one CTA, and the plan takes more than the limit.
__host__ __device__ inline unsigned long long ln_fit(const uint32_t* counts, const unsigned long long* maxc, const uint32_t* cap, unsigned long long limit,
                                                     LnPlan* pl) {
  typedef unsigned long long u64;
  auto sub = [](u64 a, u64 b) { return a > b ? a - b : 0ull; };   // saturating
  auto lo = [](u64 a, u64 b) { return a < b ? a : b; };
  u64 ord = 0, base = 0;   // ordinary classes: bytes asked for, bytes of one CTA each
  for (int c = 0; c < 2 * LN_NCLS; ++c) {
    LnPlan& p = pl[c];
    p.base = p.work_stride = p.off_dirsR = p.off_dirsF = p.off_trace = 0;
    p.grid = 0;
    if (c == 0 || !cap[c] || !counts[c]) continue;
    if (c == LN_WIDE) p.work_stride = maxc[c];   // the slab is the largest job's (lnw_geom), laid out per job by the kernel
    else ln_slab(p, maxc[c], maxc[32 + c], maxc[64 + c]);
    p.grid = (uint32_t) lo(counts[c], cap[c]);
    if (c != LN_WIDE) { ord += p.grid * p.work_stride; base += p.work_stride; }
  }
  u64 wide_total = 0;
  LnPlan& w = pl[LN_WIDE];
  if (w.grid) {
    const u64 keep = lo(ord, limit / 2);
    w.grid = (uint32_t) lo(w.grid, sub(limit, keep > base ? keep : base) / w.work_stride);
    if (!w.grid) w.grid = 1;
    wide_total = w.grid * w.work_stride;
  }
  const u64 rest = sub(limit, wide_total);
  if (ord > rest)
    for (int c = 1; c < 2 * LN_NCLS; ++c)
      if (c != LN_WIDE && pl[c].grid) pl[c].grid = 1 + (uint32_t) (rest > base ? (pl[c].grid - 1ull) * (rest - base) / (ord - base) : 0);
  u64 off = 0;
  for (int c = 0; c < 2 * LN_NCLS; ++c) { pl[c].base = off; off += pl[c].grid * pl[c].work_stride; }
  return off;
}

// Device-side planning under dgpu_set_ln_async_bound: ln_fit by one thread, from the counts and maxima the synchronous form reads back.
// gmax[c] = the CTAs class c is launched with (0: not launched); pool = the workspace the setter reserved, sized for one bound-shaped CTA of
// every class the bound admits, so the plan fits it.
struct LnPlanIn { uint32_t gmax[2 * LN_NCLS]; unsigned long long pool; };
__global__ void ln_plan_kernel(const uint32_t* __restrict__ counts, const unsigned long long* __restrict__ maxc, LnPlanIn in, LnPlan* plan) {
  if (threadIdx.x == 0) ln_fit(counts, maxc, in.gmax, in.pool, plan);
}

// src/util.h:549-563 applied to position i of the output
__device__ __forceinline__ uint8_t revcomp_at(const uint8_t* s, uint32_t L, uint32_t i) {
  uint8_t c = s[L - 1 - i];
  if (c >= 'a' && c <= 'z') c -= 32;  // boost::to_upper_copy, "C" locale
  switch (c) {
    case 'A': return 'T';
    case 'C': return 'G';
    case 'G': return 'C';
    case 'T': return 'A';
    case 'N': return 'N';
    default: return s[i];  // the reference leaves the original (un-reversed) byte in place
  }
}

// needle.h:207-216: complement of an alignment character of the reverse part; other bytes stay unwritten (0)
__device__ __forceinline__ uint8_t comp_aln(uint8_t c) {
  switch (c) {
    case 'A': return 'T';
    case 'C': return 'G';
    case 'G': return 'C';
    case 'T': return 'A';
    case 'N': return 'N';
    case '-': return '-';
    default: return 0;
  }
}

// Warp-cooperative traceback over the direction nibbles from (rr,cc) to (0,0); emits alignment characters in
// traceback order and returns the number of columns (same value in every lane). Executed by one full warp.
//   * the warp stages a window of direction words that follows the diagonal (lane i: row rr-i, the two words around
//     column cc-i) with ONE round of loads, so the walk pays one memory latency per <= 32 steps instead of one per step;
//   * lane 0 walks the window (shared memory) and records which steps consumed a row / a column as two bit masks;
//   * all lanes then expand the masks in parallel: lane t derives the coordinates of step t by popcount, fetches the two
//     sequence bytes and stores the alignment characters (coalesced), so no load sits on the walk's dependency chain;
//   * once row 0 or column 0 is reached the rest is a pure gap run, filled in by all lanes.
// REVSTR: sequences are the reverse complements (the reverse matrix of src/needle.h:74-82).
template <bool REVSTR>
__device__ __forceinline__ uint32_t ln_traceback_warp(const uint32_t* __restrict__ dirs, uint32_t dstride, int cstart, const uint8_t* s1, uint32_t m,
                                                      const uint8_t* s2, uint32_t n, uint32_t rr0, uint32_t cc0, uint8_t* tA, uint8_t* tB,
                                                      uint32_t* win /* 64 words of shared memory owned by this warp */, int lane) {
  int rr = (int) rr0, cc = (int) cc0;
  uint32_t k = 0;
  auto chA = [&](int r) -> uint8_t { uint8_t a = REVSTR ? revcomp_at(s1, m, (uint32_t) r) : s1[r]; return REVSTR ? comp_aln(a) : a; };
  auto chB = [&](int c) -> uint8_t { uint8_t b = REVSTR ? revcomp_at(s2, n, (uint32_t) c) : s2[c]; return REVSTR ? comp_aln(b) : b; };
  const uint8_t gap = '-';
  while (rr > 0 && cc > 0) {
    {
      const int ri = rr - lane;
      const int wi = (max(cc - lane, 1) - cstart) >> 3;
      uint32_t w1 = 0, w0 = 0;
      if (ri >= 1) {
        const uint32_t* drow = dirs + (size_t) ri * dstride;
        w1 = __ldcg(drow + wi);
        if (wi > 0) w0 = __ldcg(drow + wi - 1);
      }
      win[2 * lane] = w0; win[2 * lane + 1] = w1;
    }
    __syncwarp();
    uint32_t maskR = 0, maskC = 0;
    int steps = 0;
    const int row0 = rr, col0 = cc;
    if (lane == 0) {
      int r = rr, c = cc;
      while (r > 0 && c > 0 && steps < 32) {
        const int i = row0 - r;
        if (i >= 32) break;
        const int k2 = c - cstart;
        const int wsel = (k2 >> 3) - ((max(col0 - i, 1) - cstart) >> 3) + 1;
        if (wsel < 0 || wsel > 1) break;
        const uint32_t code = (win[2 * i + wsel] >> ((k2 & 7) * 4)) & 3u;
        const uint32_t dr = (code != 2u), dc = (code != 1u);
        maskR |= dr << steps; maskC |= dc << steps;
        r -= (int) dr; c -= (int) dc;
        ++steps;
      }
    }
    maskR = __shfl_sync(0xffffffffu, maskR, 0);
    maskC = __shfl_sync(0xffffffffu, maskC, 0);
    steps = __shfl_sync(0xffffffffu, steps, 0);
    if (lane < steps) {
      const uint32_t below = (1u << lane) - 1u;
      const int r = row0 - __popc(maskR & below), c = col0 - __popc(maskC & below);   // coordinates before step `lane`
      tA[k + lane] = ((maskR >> lane) & 1u) ? chA(r - 1) : gap;
      tB[k + lane] = ((maskC >> lane) & 1u) ? chB(c - 1) : gap;
    }
    rr = row0 - __popc(maskR); cc = col0 - __popc(maskC);
    k += (uint32_t) steps;
    __syncwarp();
  }
  // row 0: horizontal run; column 0: vertical run (needle.h:159-171 with one index exhausted)
  for (int t = lane; t < cc; t += 32) { tA[k + t] = gap; tB[k + t] = chB(cc - 1 - t); }
  for (int t = lane; t < rr; t += 32) { tA[k + t] = chA(rr - 1 - t); tB[k + t] = gap; }
  return k + (uint32_t) cc + (uint32_t) rr;
}

// (a register cap tight enough for more single-warp CTAs per SM would spill the DP state that lives in registers)
// MAXT = threads per CTA the register allocation is sized for: a multi-warp CTA of 8 warps may use 255 registers per
// thread (the DP state of C columns lives in registers), 16 warps would be capped at 128 and spill.
template <int C, bool MULTI, int MAXT, bool PLAN>
__global__ void __launch_bounds__(MAXT, 1) ln_kernel(LnArgs a, int cls) {
  extern __shared__ uint8_t sm_dyn[];
  constexpr int UPS = ln_ups(C, MAXT) ? MAXT : 0;   // wide column blocks: previous-row state in shared memory (wavefront.cuh)
  int* sm_up = (int*) sm_dyn;                         // [C][UPS]
  uint8_t* sm_rows = sm_dyn + ln_smem_ups(C, MAXT);  // row string of the current pass (m bytes)
  __shared__ int sm_x[wf::WF_SMX];
  __shared__ int sm_pub[8];
  __shared__ uint32_t sm_win[128];  // traceback windows (one per tracing warp)
  __shared__ wf::Best sm_best[16];
  const int tid = threadIdx.x;
  const int T = blockDim.x;
  const int lane = tid & 31;
  const uint32_t cnt = a.counts[cls], start = a.counts[32 + cls];
  const LnCta cta = ln_cta<PLAN>(a, cls);
  if (PLAN && blockIdx.x >= cta.grid) return;
  int16_t* brev = (int16_t*) cta.slab;
  uint32_t* dirsR = (uint32_t*) (cta.slab + cta.off_dirsR);
  uint32_t* dirsF = (uint32_t*) (cta.slab + cta.off_dirsF);
  uint8_t* trace = cta.slab + cta.off_trace;
  const wf::Scoring sc = {1, -1, true, true};  // DnaScore(1,-1,-1,-1), AlignConfig<true,false> (src/split.h:541-542)

  for (uint32_t idx = blockIdx.x; idx < cnt; idx += cta.grid) {
    const uint32_t job = a.perm[start + idx];
    const uint32_t m = a.c_len[job], n = a.r_len[job];
    const uint8_t* s1 = a.seqs + a.c_off[job];
    const uint8_t* s2 = a.seqs + a.r_off[job];
    const uint32_t bstride = ln_bstride(n, C), dstride = ln_dstride(n, C);
    const int P = (int) ln_P(n, C);
    const int delta = P - 1 - (int) n;
    const int cstartF = ((delta + 1) & ~7) - delta;  // forward blocks are aligned to the mirrored storage
    __syncthreads();
    // ---- reverse pass on (revcomp s1, revcomp s2) ----
    for (uint32_t i = tid; i < m; i += T) sm_rows[i] = revcomp_at(s1, m, i);
    __syncthreads();
    wf::Best dummy;
    int revCorner, matCorner;
    wf::pass<C, MULTI, wf::REV, false, UPS>([&](int i) { return sm_rows[i]; }, [&](int i) { return revcomp_at(s2, n, (uint32_t) i); }, (int) m, (int) n, sc,
                                            1, dirsR, dstride, brev, bstride, P, sm_x, dummy, revCorner, nullptr, nullptr, sm_up);
    __syncthreads();
    // ---- forward pass with the fused join ----
    for (uint32_t i = tid; i < m; i += T) sm_rows[i] = s1[i];
    __syncthreads();
    wf::Best best;
    wf::pass<C, MULTI, wf::FWD, false, UPS>([&](int i) { return sm_rows[i]; }, [&](int i) { return s2[i]; }, (int) m, (int) n, sc, cstartF, dirsF, dstride,
                                            brev, bstride, P, sm_x, best, matCorner, nullptr, nullptr, sm_up);
    // reduce the per-thread arg-max (row-major first max)
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      wf::Best o;
      o.val = __shfl_xor_sync(0xffffffffu, best.val, d);
      o.row = __shfl_xor_sync(0xffffffffu, best.row, d);
      o.col = __shfl_xor_sync(0xffffffffu, best.col, d);
      o.bm = __shfl_xor_sync(0xffffffffu, best.bm, d);
      if (wf::best_before(o, best)) best = o;
    }
    if (MULTI) {
      if (lane == 0) sm_best[tid >> 5] = best;
      __syncthreads();
      best = sm_best[0];
      for (int w = 1; w < (T >> 5); ++w)
        if (wf::best_before(sm_best[w], best)) best = sm_best[w];
      __syncthreads();
    }
    const int gbest = best.val, consLeft = best.row, refLeft = best.col, matv = best.bm;
    const bool ok = (matCorner == revCorner) && (gbest != matCorner);  // needle.h:83-86, :152
    if (!ok) {
      if (tid == 0) {
        a.ok[job] = 0; a.aln_len[job] = 0;
        if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = 0; a.info[4 * job + 3] = gbest; }
      }
      continue;
    }
    // refRight: last right in [0, n-refLeft] with matv + rev[consRight][right] == gbest (needle.h:116-123);
    // rev[cR][x] == target  <=>  prefixmax[cR][x] == target and the cell carries the "equals maximum" bit
    const uint32_t consRight = m - (uint32_t) consLeft;
    {
      const int16_t* brow = brev + (size_t) consRight * bstride;
      const uint32_t* drow = dirsR + (size_t) consRight * dstride;
      const int target = gbest - matv + (int) consRight;   // stored prefix maxima carry their row index as a shift (wavefront.cuh)
      int bestRight = 0;
      for (uint32_t x = tid; x <= n - (uint32_t) refLeft; x += T) {
        if ((int) __ldcg(brow + (P - 1 - (int) x)) != target) continue;
        bool eq = true;
        if (x > 0) { uint32_t w = __ldcg(drow + ((x - 1) >> 3)); eq = ((w >> (((x - 1) & 7) * 4)) & 4u) != 0; }
        if (eq) bestRight = max(bestRight, (int) x);
      }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) bestRight = max(bestRight, __shfl_xor_sync(0xffffffffu, bestRight, d));
      if (MULTI) {
        if (lane == 0) sm_x[tid >> 5] = bestRight;
        __syncthreads();
        for (int w = 0; w < (T >> 5); ++w) bestRight = max(bestRight, sm_x[w]);
        __syncthreads();
      }
      if (tid == 0) sm_pub[2] = bestRight;
      __syncthreads();
    }
    const uint32_t refRight = (uint32_t) sm_pub[2];
    uint8_t* tFA = trace;
    uint8_t* tFB = trace + (m + n);
    uint8_t* tRA = trace + 2 * (size_t) (m + n);
    uint8_t* tRB = trace + 3 * (size_t) (m + n);
    // two warp-cooperative tracebacks: warps 0 and 1 of a CTA side by side, or one after the other in the single warp
    if (!MULTI || tid < 32) {
      const uint32_t v = ln_traceback_warp<false>(dirsF, dstride, cstartF, s1, m, s2, n, (uint32_t) consLeft, (uint32_t) refLeft, tFA, tFB, sm_win, lane);
      if (lane == 0) sm_pub[3] = (int) v;
    }
    if (!MULTI || (tid >= 32 && tid < 64)) {
      const uint32_t v = ln_traceback_warp<true>(dirsR, dstride, 1, s1, m, s2, n, consRight, refRight, tRA, tRB, sm_win + (MULTI ? 64 : 0), lane);
      if (lane == 0) sm_pub[4] = (int) v;
    }
    __syncthreads();
    const uint32_t Lf = (uint32_t) sm_pub[3], Lr = (uint32_t) sm_pub[4];
    const uint32_t gapref = (n - refRight) - (uint32_t) refLeft;
    const uint32_t L = Lf + gapref + Lr;
    uint8_t* o0 = a.aln + a.aln_off[job];
    uint8_t* o1 = o0 + (m + n);
    for (uint32_t i = tid; i < L; i += T) {
      uint8_t x, y;
      if (i < Lf) { x = tFA[Lf - 1 - i]; y = tFB[Lf - 1 - i]; }
      else if (i < Lf + gapref) { x = '-'; y = s2[refLeft + (i - Lf)]; }
      else { x = tRA[i - Lf - gapref]; y = tRB[i - Lf - gapref]; }
      o0[i] = x; o1[i] = y;
    }
    if (tid == 0) {
      a.ok[job] = 1; a.aln_len[job] = L;
      if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = (int) refRight; a.info[4 * job + 3] = gbest; }
    }
  }
}


// ---- second-generation kernel on the packed two-row engine (wavefront2.cuh) ------------------------------------------------------
// Same job anatomy as ln_kernel (reverse pass storing mirrored prefix maxima + nibbles, forward pass with the fused join, refRight,
// two warp-cooperative tracebacks, stitched output); what differs: nibbles hold the differences (X - up, X - left) and even rows are
// rotated by one column inside a thread's group (wf2::nib_index), there is no "equals the row maximum" bit — refRight (needle.h:116-123)
// rebuilds the one row it needs from the horizontal differences with a block-wide scan — and the partner rows of the forward pass are staged
// through shared memory with cp.async.
template <int C, bool REVSTR>
__device__ __forceinline__ uint32_t ln_traceback_warp2(const uint32_t* __restrict__ dirs, int T, int cstart, const uint8_t* s1, uint32_t m,
                                                       const uint8_t* s2, uint32_t n, uint32_t rr0, uint32_t cc0, uint8_t* tA, uint8_t* tB,
                                                       uint32_t* win /* 64 words of shared memory owned by this warp */, int lane) {
  int rr = (int) rr0, cc = (int) cc0;
  uint32_t k = 0;
  auto chA = [&](int r) -> uint8_t { uint8_t a = REVSTR ? revcomp_at(s1, m, (uint32_t) r) : s1[r]; return REVSTR ? comp_aln(a) : a; };
  auto chB = [&](int c) -> uint8_t { uint8_t b = REVSTR ? revcomp_at(s2, n, (uint32_t) c) : s2[c]; return REVSTR ? comp_aln(b) : b; };
  const uint8_t gap = '-';
  while (rr > 0 && cc > 0) {
    {
      const int ri = rr - lane;
      uint32_t w1 = 0, w0 = 0;
      if (ri >= 1) {
        const int wi = wf2::nib_index<C>(ri, max(cc - lane, 1), cstart) >> 3;
        w1 = wf2::nib_word<C>(dirs, ri, wi, T);
        if (wi > 0) w0 = wf2::nib_word<C>(dirs, ri, wi - 1, T);
      }
      win[2 * lane] = w0; win[2 * lane + 1] = w1;
    }
    __syncwarp();
    uint32_t maskR = 0, maskC = 0;
    int steps = 0;
    const int row0 = rr, col0 = cc;
    if (lane == 0) {
      int r = rr, c = cc;
      while (r > 0 && c > 0 && steps < 32) {
        const int i = row0 - r;
        if (i >= 32) break;
        const int idx = wf2::nib_index<C>(r, c, cstart);
        const int wsel = (idx >> 3) - (wf2::nib_index<C>(r, max(col0 - i, 1), cstart) >> 3) + 1;
        if (wsel < 0 || wsel > 1) break;
        const uint32_t code = wf2::nib_dir((win[2 * i + wsel] >> ((idx & 7) * 4)) & 15u);
        const uint32_t dr = (code != 2u), dc = (code != 1u);
        maskR |= dr << steps; maskC |= dc << steps;
        r -= (int) dr; c -= (int) dc;
        ++steps;
      }
    }
    maskR = __shfl_sync(0xffffffffu, maskR, 0);
    maskC = __shfl_sync(0xffffffffu, maskC, 0);
    steps = __shfl_sync(0xffffffffu, steps, 0);
    if (steps == 0) {   // the staged window missed the very first cell (block wrap of an even row): take one step straight from memory
      uint32_t code = 0;
      if (lane == 0) {
        const int idx = wf2::nib_index<C>(rr, cc, cstart);
        code = wf2::nib_dir((wf2::nib_word<C>(dirs, rr, idx >> 3, T) >> ((idx & 7) * 4)) & 15u);
      }
      code = __shfl_sync(0xffffffffu, code, 0);
      maskR = (code != 2u); maskC = (code != 1u); steps = 1;
    }
    if (lane < steps) {
      const uint32_t below = (1u << lane) - 1u;
      const int r = row0 - __popc(maskR & below), c = col0 - __popc(maskC & below);
      tA[k + lane] = ((maskR >> lane) & 1u) ? chA(r - 1) : gap;
      tB[k + lane] = ((maskC >> lane) & 1u) ? chB(c - 1) : gap;
    }
    rr = row0 - __popc(maskR); cc = col0 - __popc(maskC);
    k += (uint32_t) steps;
    __syncwarp();
  }
  for (int t = lane; t < cc; t += 32) { tA[k + t] = gap; tB[k + t] = chB(cc - 1 - t); }
  for (int t = lane; t < rr; t += 32) { tA[k + t] = chA(rr - 1 - t); tB[k + t] = gap; }
  return k + (uint32_t) cc + (uint32_t) rr;
}

template <int C, bool MULTI, int MAXT, bool PLAN>
__global__ void __launch_bounds__(MAXT, ln2_occ(MAXT)) ln_kernel2(LnArgs a, int cls) {
  extern __shared__ uint8_t sm_dyn[];
  const int tid = threadIdx.x;
  const int T = blockDim.x;
  const int lane = tid & 31;
  const Ln2Smem L = ln2_smem(C, T);
  uint4* sm_part = (uint4*) sm_dyn;                  // partner ring of the forward pass
  uint32_t* sm_scr = (uint32_t*) (sm_dyn + L.ring);  // row scratch of the join's arg-max search
  uint8_t* sm_rows = (uint8_t*) (sm_scr + L.scr);    // one-hot codes of the row string of the current pass
  __shared__ int sm_x[wf::WF_SMX];
  __shared__ int sm_pub[8];
  __shared__ uint32_t sm_win[128];
  __shared__ wf::Best sm_best[16];
  __shared__ int sm_scan[16];
  const uint32_t cnt = a.counts[cls], start = a.counts[32 + cls];
  const LnCta cta = ln_cta<PLAN>(a, cls);
  if (PLAN && blockIdx.x >= cta.grid) return;
  uint4* brev4 = (uint4*) cta.slab;                     // step-major workspace (wavefront2.cuh)
  uint32_t* dirsR = (uint32_t*) (cta.slab + cta.off_dirsR);
  uint32_t* dirsF = (uint32_t*) (cta.slab + cta.off_dirsF);
  uint8_t* trace = cta.slab + cta.off_trace;

  for (uint32_t idx = blockIdx.x; idx < cnt; idx += cta.grid) {
    const uint32_t job = a.perm[start + idx];
    const uint32_t m = a.c_len[job], n = a.r_len[job];
    const uint8_t* s1 = a.seqs + a.c_off[job];
    const uint8_t* s2 = a.seqs + a.r_off[job];
    const int P = (int) ln_P(n, C);
    const int delta = P - 1 - (int) n;
    const int cstartF = ((delta + 1) & ~7) - delta;
    __syncthreads();
    // ---- reverse pass on (revcomp s1, revcomp s2) ----
    for (uint32_t i = tid; i < m; i += T) sm_rows[i] = (uint8_t) wf2::hot(revcomp_at(s1, m, i));
    __syncthreads();
    wf::Best dummy;
    int revCorner, matCorner;
    wf2::pass<C, MULTI, wf2::REV, LN_PART_D>(sm_rows, [&](int i) { return revcomp_at(s2, n, (uint32_t) i); }, (int) m, (int) n, 1, dirsR, brev4, P, sm_x, sm_part, sm_scr, dummy, revCorner);
    __syncthreads();
    // ---- forward pass with the fused join ----
    for (uint32_t i = tid; i < m; i += T) sm_rows[i] = (uint8_t) wf2::hot(s1[i]);
    wf2::synth_groups<C>(brev4, (int) m);
    if (cstartF < 0) {
      // The forward blocks start at column cstartF <= 1 (aligned to the mirrored groups); its dummy columns c < 0 would pair with the elements
      // x = n - c > n of the reverse rows — prefix maxima of columns that do not exist. They are no join candidates: mark them once per job.
      const int nd = -cstartF, nactR = (P - 1) / C;
      for (int i = tid; i < (int) (m + 1) * nd; i += T) {
        const int r = i / nd, idxm = P - 1 - ((int) n + 1 + i % nd), g = idxm >> 3;
        ((int16_t*) (brev4 + wf2::grp_index<C>(r, nactR - 1 - g / (C / 8), g % (C / 8), T)))[idxm & 7] = (int16_t) -32768;
      }
    }
    __syncthreads();
    wf::Best best;
    wf2::pass<C, MULTI, wf2::FWD, LN_PART_D>(sm_rows, [&](int i) { return s2[i]; }, (int) m, (int) n, cstartF, dirsF, brev4, P, sm_x, sm_part, sm_scr, best, matCorner);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      wf::Best o;
      o.val = __shfl_xor_sync(0xffffffffu, best.val, d);
      o.row = __shfl_xor_sync(0xffffffffu, best.row, d);
      o.col = __shfl_xor_sync(0xffffffffu, best.col, d);
      o.bm = __shfl_xor_sync(0xffffffffu, best.bm, d);
      if (wf::best_before(o, best)) best = o;
    }
    if (MULTI) {
      if (lane == 0) sm_best[tid >> 5] = best;
      __syncthreads();
      best = sm_best[0];
      for (int w = 1; w < (T >> 5); ++w)
        if (wf::best_before(sm_best[w], best)) best = sm_best[w];
      __syncthreads();
    }
    const int gbest = best.val, consLeft = best.row, refLeft = best.col, matv = best.bm;
    const bool ok = (matCorner == revCorner) && (gbest != matCorner);  // needle.h:83-86, :152
    if (!ok) {
      if (tid == 0) {
        a.ok[job] = 0; a.aln_len[job] = 0;
        if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = 0; a.info[4 * job + 3] = gbest; }
      }
      continue;
    }
    // refRight: last right in [0, n-refLeft] with matv + rev[consRight][right] == gbest (needle.h:116-123). Row consRight of the reverse matrix
    // is rebuilt from its horizontal differences: H(cR, x) = H(cR, x-1) + (nibble >> 2) - g, H(cR, 0) = -cR (block-wide prefix scan).
    const uint32_t consRight = m - (uint32_t) consLeft;
    {
      const int target = gbest - matv;
      const int xmax = (int) n - refLeft;
      int bestRight = 0;
      if (consRight == 0) { if (target == 0) bestRight = xmax; }
      else {
        const int g = (consRight == m) ? 0 : 1;
        const int per = (xmax + T) / T;                       // columns per thread (x = 1 .. xmax)
        const int xa = 1 + tid * per, xb = min(xmax, xa + per - 1);
        int sum = 0;
        for (int x = xa; x <= xb; ++x) {
          const int ni = wf2::nib_index<C>((int) consRight, x, 1);
          sum += (int) ((wf2::nib_word<C>(dirsR, (int) consRight, ni >> 3, T) >> ((ni & 7) * 4 + 2)) & 3u) - g;
        }
        int incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
        int base = incl - sum;
        if (MULTI) {
          if (lane == 31) sm_scan[tid >> 5] = incl;
          __syncthreads();
          for (int w = 0; w < (tid >> 5); ++w) base += sm_scan[w];
          __syncthreads();
        }
        int h = -(int) consRight + base;                       // H(cR, xa - 1)
        if (tid == 0 && h == target) bestRight = 0;            // x = 0 (always within range)
        for (int x = xa; x <= xb; ++x) {
          const int ni = wf2::nib_index<C>((int) consRight, x, 1);
          h += (int) ((wf2::nib_word<C>(dirsR, (int) consRight, ni >> 3, T) >> ((ni & 7) * 4 + 2)) & 3u) - g;
          if (h == target) bestRight = x;
        }
      }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) bestRight = max(bestRight, __shfl_xor_sync(0xffffffffu, bestRight, d));
      if (MULTI) {
        if (lane == 0) sm_x[tid >> 5] = bestRight;
        __syncthreads();
        for (int w = 0; w < (T >> 5); ++w) bestRight = max(bestRight, sm_x[w]);
        __syncthreads();
      }
      if (tid == 0) sm_pub[2] = bestRight;
      __syncthreads();
    }
    const uint32_t refRight = (uint32_t) sm_pub[2];
    uint8_t* tFA = trace;
    uint8_t* tFB = trace + (m + n);
    uint8_t* tRA = trace + 2 * (size_t) (m + n);
    uint8_t* tRB = trace + 3 * (size_t) (m + n);
    if (!MULTI || tid < 32) {
      const uint32_t v = ln_traceback_warp2<C, false>(dirsF, T, cstartF, s1, m, s2, n, (uint32_t) consLeft, (uint32_t) refLeft, tFA, tFB, sm_win, lane);
      if (lane == 0) sm_pub[3] = (int) v;
    }
    if (!MULTI || (tid >= 32 && tid < 64)) {
      const uint32_t v = ln_traceback_warp2<C, true>(dirsR, T, 1, s1, m, s2, n, consRight, refRight, tRA, tRB, sm_win + (MULTI ? 64 : 0), lane);
      if (lane == 0) sm_pub[4] = (int) v;
    }
    __syncthreads();
    const uint32_t Lf = (uint32_t) sm_pub[3], Lr = (uint32_t) sm_pub[4];
    const uint32_t gapref = (n - refRight) - (uint32_t) refLeft;
    const uint32_t L = Lf + gapref + Lr;
    uint8_t* o0 = a.aln + a.aln_off[job];
    uint8_t* o1 = o0 + (m + n);
    for (uint32_t i = tid; i < L; i += T) {
      uint8_t x, y;
      if (i < Lf) { x = tFA[Lf - 1 - i]; y = tFB[Lf - 1 - i]; }
      else if (i < Lf + gapref) { x = '-'; y = s2[refLeft + (i - Lf)]; }
      else { x = tRA[i - Lf - gapref]; y = tRB[i - Lf - gapref]; }
      o0[i] = x; o1[i] = y;
    }
    if (tid == 0) {
      a.ok[job] = 1; a.aln_len[job] = L;
      if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = (int) refRight; a.info[4 * job + 3] = gbest; }
    }
  }
}

// ---- wide-window kernel (geometry and layout: lnw_geom) -------------------------------------------------------------------------------
// Block-wide exclusive max-scan over the (at most 32) warps of the CTA: max(init, v of every lower thread). One block barrier; sm_w = 32 ints.
__device__ __forceinline__ int lnw_excl_max(int v, int init, int* sm_w) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl = max(incl, o); }
  int excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = init;
  if (lane == 31) sm_w[w] = incl;
  __syncthreads();
  int pw = (lane < w) ? sm_w[lane] : init;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) pw = max(pw, __shfl_xor_sync(0xffffffffu, pw, d));
  return max(max(excl, pw), init);
}

// One DP pass of the wide engine over rows 1..m. Shared rows prepared by the caller: sm_rows[r-1] = row byte, sm_col[k] = byte of column
// o + k (0 outside 1..n), sm_u[8 + k] = U of column o + k in the previous row (row 0: all 0), sm_u[7] = column o - 1.
// Thread t owns chunks q = t*J .. t*J+J-1 (columns o + 8q .. o + 8q + 7); J is odd, so the 16-byte shared accesses of a warp are free of
// bank conflicts. Per row, three sweeps over the thread's chunks:
//   1. D = max(U_diag + (match ? 2 : 0), U_up), X = D + g*c; block max-scan of X: U[c] = max_{k<=c} X[k] - g*c (column 0: X = U = 0);
//   2. U and its direction (vertical > horizontal > diagonal, as wavefront.cuh), U written over the previous row in place; block max-scan of U;
//   3. the row's prefix maxima: REV stores them mirrored with the "equals the row maximum" bit, FWD evaluates the join of needle.h:104-115
//      against the stored reverse row m - r, keeping the first maximum in row-major order.
// Grid columns <= 0 (only the reverse grid has them) are pinned to the column-0 value U = 0. *corner receives H[m][n].
template <bool REVP>
__device__ __forceinline__ void lnw_pass(const uint8_t* sm_rows, const uint8_t* sm_col, int16_t* sm_u, int* sm_w, const int m, const int n, const int o,
                                         const int nq, const int J, int16_t* __restrict__ brev, const uint32_t bstride, uint32_t* __restrict__ dirs,
                                         const uint32_t dstride, wf::Best& best, int* corner) {
  const int tid = threadIdx.x;
  const int qa = tid * J;
  for (int r = 1; r <= m; ++r) {
    const int g = (r == m) ? 0 : 1;   // AlignConfig<true,false>: horizontal moves in the last row are free
    const uint32_t a = sm_rows[r - 1];
    const int u0 = (qa < nq) ? (int) sm_u[8 * qa + 7] : 0;   // previous row, column left of the first chunk (read before anyone overwrites it)
    // ---- sweep 1: the row maximum of X per thread
    int xmax = wf::NEG;
    {
      int pd = u0;
#pragma unroll
      for (int j = 0; j < LNW_JMAX; ++j) {
        const int q = qa + j;
        if (j < J && q < nq) {
          const int cb = o + 8 * q;
          const uint4 pv = *(const uint4*) (sm_u + 8 * q + 8);
          const uint2 cv = *(const uint2*) (sm_col + 8 * q);
          const uint32_t pw[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int up = (int) ((pw[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            const uint32_t b = (((i < 4) ? cv.x : cv.y) >> ((i & 3) * 8)) & 0xffu;
            const int c = cb + i;
            const int x = max(pd + (a == b ? 2 : 0), up) + g * c;
            pd = up;
            if (c >= 1) xmax = max(xmax, x);
          }
        }
      }
    }
    const int carry = lnw_excl_max(xmax, 0, sm_w);
    // ---- sweep 2: scores, directions, the row maximum of U per thread
    int rmax = wf::NEG;
    uint32_t dc[(LNW_JMAX + 1) / 2];   // 2-bit directions, two chunks per word (expanded to nibbles in sweep 3)
#pragma unroll
    for (int j = 0; j < (LNW_JMAX + 1) / 2; ++j) dc[j] = 0;
    {
      int pd = u0, pm = carry;
      int ul = carry - g * (o + 8 * qa - 1);   // U of the column left of the first chunk, this row
#pragma unroll
      for (int j = 0; j < LNW_JMAX; ++j) {
        const int q = qa + j;
        if (j < J && q < nq) {
          const int cb = o + 8 * q;
          const uint4 pv = *(const uint4*) (sm_u + 8 * q + 8);
          const uint2 cv = *(const uint2*) (sm_col + 8 * q);
          const uint32_t pw[4] = {pv.x, pv.y, pv.z, pv.w};
          uint32_t uw[4] = {0, 0, 0, 0};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int up = (int) ((pw[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            const uint32_t b = (((i < 4) ? cv.x : cv.y) >> ((i & 3) * 8)) & 0xffu;
            const int c = cb + i;
            const int x = max(pd + (a == b ? 2 : 0), up) + g * c;
            pd = up;
            int U = 0;
            if (c >= 1) { pm = max(pm, x); U = pm - g * c; }
            const uint32_t code = (U == up) ? 1u : ((U == ul - g) ? 2u : 0u);
            ul = U;
            rmax = max(rmax, U);
            dc[j >> 1] |= code << ((j & 1) * 16 + i * 2);
            uw[i >> 1] |= (uint32_t) U << ((i & 1) * 16);
            if (r == m && c == n) *corner = U - m;
          }
          *(uint4*) (sm_u + 8 * q + 8) = make_uint4(uw[0], uw[1], uw[2], uw[3]);
        }
      }
    }
    const int carry2 = lnw_excl_max(rmax, 0, sm_w + 32);
    // ---- sweep 3: prefix maxima
    int rm = carry2;
    if (!REVP && tid == 0) {   // column 0 (H = -r, shifted 0) against reverse row m - r at x = n (index 7)
      const int v = (int) __ldcg(brev + (size_t) (m - r) * bstride + 7) - m;
      if (v > best.val) { best.val = v; best.row = r; best.col = 0; best.bm = -r; }
    }
#pragma unroll
    for (int j = 0; j < LNW_JMAX; ++j) {
      const int q = qa + j;
      if (j < J && q < nq) {
        const int cb = o + 8 * q;
        const uint4 uv = *(const uint4*) (sm_u + 8 * q + 8);
        const uint32_t uw[4] = {uv.x, uv.y, uv.z, uv.w};
        uint32_t dw = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) dw |= ((dc[j >> 1] >> ((j & 1) * 16 + i * 2)) & 3u) << (i * 4);
        if (REVP) {
          uint32_t sw[4] = {0, 0, 0, 0};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int U = (int) ((uw[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            rm = max(rm, U);
            if (U == rm) dw |= 4u << (i * 4);
            const int h = 7 - i;   // column cb + i is element x = cb + i at index n + 7 - x = (n - cb) + h
            sw[h >> 1] |= (uint32_t) rm << ((h & 1) * 16);
          }
          *(uint4*) (brev + (size_t) r * bstride + (n - cb)) = make_uint4(sw[0], sw[1], sw[2], sw[3]);
        } else {
          const uint4 pv = __ldcg((const uint4*) (brev + (size_t) (m - r) * bstride + cb + 7));   // partners x = n - c of columns cb ..
          const uint32_t pw[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int U = (int) ((uw[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            rm = max(rm, U);
            const int c = cb + i;
            const int v = rm + (int) (int16_t) ((pw[i >> 1] >> ((i & 1) * 16)) & 0xffffu) - m;
            if (c <= n && v > best.val) { best.val = v; best.row = r; best.col = c; best.bm = rm - r; }
          }
        }
        dirs[(size_t) r * dstride + q] = dw;
      }
    }
    if (REVP && tid == 0) brev[(size_t) r * bstride + n + 7] = 0;   // x = 0: H = -r, shifted 0
  }
}

// One CTA per wide job: reverse pass, forward pass with the join, refRight, the two warp tracebacks and the stitched output, with the
// semantics of ln_kernel (see the head of this file).
template <bool PLAN>
__global__ void __launch_bounds__(LNW_THREADS, 1) lnw_kernel(LnArgs a) {
  extern __shared__ uint8_t sm_dyn[];
  const uint32_t nqmax = (a.max_ref + 6) / 8 + 1;
  int16_t* sm_u = (int16_t*) sm_dyn;                                        // [8 * nqmax + 8]
  uint8_t* sm_col = sm_dyn + ((2 * (8 * (size_t) nqmax + 8) + 15) & ~(size_t) 15);   // [8 * nqmax]
  uint8_t* sm_rows = sm_col + 8 * (size_t) nqmax;                            // [m]
  __shared__ int sm_w[64];
  __shared__ int sm_pub[8];
  __shared__ uint32_t sm_win[128];
  __shared__ wf::Best sm_best[LNW_THREADS / 32];
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const uint32_t cnt = a.counts[LN_WIDE], start = a.counts[32 + LN_WIDE];
  const LnCta cta = ln_cta<PLAN>(a, LN_WIDE);   // (the slab's layout is per job: lnw_geom)
  if (PLAN && blockIdx.x >= cta.grid) return;
  uint8_t* slab = cta.slab;

  for (uint32_t idx = blockIdx.x; idx < cnt; idx += cta.grid) {
    const uint32_t job = a.perm[start + idx];
    const uint32_t m = a.c_len[job], n = a.r_len[job];
    const uint8_t* s1 = a.seqs + a.c_off[job];
    const uint8_t* s2 = a.seqs + a.r_off[job];
    const LnwGeom G = lnw_geom(m, n);
    int16_t* brev = (int16_t*) slab;
    uint32_t* dirsR = (uint32_t*) (slab + G.off_dirsR);
    uint32_t* dirsF = (uint32_t*) (slab + G.off_dirsF);
    uint8_t* trace = slab + G.off_trace;
    const int J = (int) (((G.nqR + LNW_THREADS - 1) / LNW_THREADS) | 1u);
    __syncthreads();
    // ---- reverse pass on (revcomp s1, revcomp s2) ----
    for (uint32_t i = tid; i < m; i += LNW_THREADS) sm_rows[i] = revcomp_at(s1, m, i);
    for (uint32_t k = tid; k < 8 * G.nqR; k += LNW_THREADS) {
      const int c = G.o + (int) k;
      sm_col[k] = (c >= 1 && c <= (int) n) ? revcomp_at(s2, n, (uint32_t) (c - 1)) : 0;
    }
    for (uint32_t k = tid; k < 8 * G.nqR + 8; k += LNW_THREADS) sm_u[k] = 0;
    for (uint32_t k = tid; k < G.bstride; k += LNW_THREADS) brev[k] = 0;              // row 0: prefix maxima 0
    for (uint32_t k = tid; k < G.dstride; k += LNW_THREADS) dirsR[k] = 0x44444444u;   // row 0: every cell equals its row maximum
    __syncthreads();
    wf::Best dummy;
    lnw_pass<true>(sm_rows, sm_col, sm_u, sm_w, (int) m, (int) n, G.o, (int) G.nqR, J, brev, G.bstride, dirsR, G.dstride, dummy, &sm_pub[0]);
    __syncthreads();
    // ---- forward pass with the fused join ----
    for (uint32_t i = tid; i < m; i += LNW_THREADS) sm_rows[i] = s1[i];
    for (uint32_t k = tid; k < 8 * G.nqF; k += LNW_THREADS) sm_col[k] = (k < n) ? s2[k] : 0;   // grid origin 1: column k + 1
    for (uint32_t k = tid; k < 8 * G.nqF + 8; k += LNW_THREADS) sm_u[k] = 0;
    wf::Best best;
    best.val = wf::NEG; best.row = 0; best.col = 0; best.bm = 0;
    {  // join candidates of row 0: bestMat[0][c] = 0 against reverse row m at x = n - c (index c + 7)
      const int16_t* prow = brev + (size_t) m * G.bstride;
      for (uint32_t c = tid; c <= n; c += LNW_THREADS) {
        const int v = (int) __ldcg(prow + c + 7) - (int) m;
        if (v > best.val) { best.val = v; best.row = 0; best.col = (int) c; best.bm = 0; }
      }
    }
    __syncthreads();
    lnw_pass<false>(sm_rows, sm_col, sm_u, sm_w, (int) m, (int) n, 1, (int) G.nqF, J, brev, G.bstride, dirsF, G.dstride, best, &sm_pub[1]);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      wf::Best o;
      o.val = __shfl_xor_sync(0xffffffffu, best.val, d);
      o.row = __shfl_xor_sync(0xffffffffu, best.row, d);
      o.col = __shfl_xor_sync(0xffffffffu, best.col, d);
      o.bm = __shfl_xor_sync(0xffffffffu, best.bm, d);
      if (wf::best_before(o, best)) best = o;
    }
    if (lane == 0) sm_best[tid >> 5] = best;
    __syncthreads();
    best = sm_best[0];
    for (int w = 1; w < LNW_THREADS / 32; ++w)
      if (wf::best_before(sm_best[w], best)) best = sm_best[w];
    const int revCorner = sm_pub[0], matCorner = sm_pub[1];
    __syncthreads();
    const int gbest = best.val, consLeft = best.row, refLeft = best.col, matv = best.bm;
    const bool ok = (matCorner == revCorner) && (gbest != matCorner);  // needle.h:83-86, :152
    if (!ok) {
      if (tid == 0) {
        a.ok[job] = 0; a.aln_len[job] = 0;
        if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = 0; a.info[4 * job + 3] = gbest; }
      }
      continue;
    }
    // refRight (needle.h:116-123) from the stored prefix maxima and "equals maximum" bits, as in ln_kernel
    const uint32_t consRight = m - (uint32_t) consLeft;
    {
      const int16_t* brow = brev + (size_t) consRight * G.bstride;
      const uint32_t* drow = dirsR + (size_t) consRight * G.dstride;
      const int target = gbest - matv + (int) consRight;
      int bestRight = 0;
      for (uint32_t x = tid; x <= n - (uint32_t) refLeft; x += LNW_THREADS) {
        if ((int) __ldcg(brow + (n + 7 - x)) != target) continue;
        bool eq = true;
        if (x > 0) { const uint32_t k = (uint32_t) ((int) x - G.o); eq = ((__ldcg(drow + (k >> 3)) >> ((k & 7) * 4)) & 4u) != 0; }
        if (eq) bestRight = max(bestRight, (int) x);
      }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) bestRight = max(bestRight, __shfl_xor_sync(0xffffffffu, bestRight, d));
      if (lane == 0) sm_w[tid >> 5] = bestRight;
      __syncthreads();
      for (int w = 0; w < LNW_THREADS / 32; ++w) bestRight = max(bestRight, sm_w[w]);
      if (tid == 0) sm_pub[2] = bestRight;
      __syncthreads();
    }
    const uint32_t refRight = (uint32_t) sm_pub[2];
    uint8_t* tFA = trace;
    uint8_t* tFB = trace + (m + n);
    uint8_t* tRA = trace + 2 * (size_t) (m + n);
    uint8_t* tRB = trace + 3 * (size_t) (m + n);
    if (tid < 32) {
      const uint32_t v = ln_traceback_warp<false>(dirsF, G.dstride, 1, s1, m, s2, n, (uint32_t) consLeft, (uint32_t) refLeft, tFA, tFB, sm_win, lane);
      if (lane == 0) sm_pub[3] = (int) v;
    } else if (tid < 64) {
      const uint32_t v = ln_traceback_warp<true>(dirsR, G.dstride, G.o, s1, m, s2, n, consRight, refRight, tRA, tRB, sm_win + 64, lane);
      if (lane == 0) sm_pub[4] = (int) v;
    }
    __syncthreads();
    const uint32_t Lf = (uint32_t) sm_pub[3], Lr = (uint32_t) sm_pub[4];
    const uint32_t gapref = (n - refRight) - (uint32_t) refLeft;
    const uint32_t L = Lf + gapref + Lr;
    uint8_t* o0 = a.aln + a.aln_off[job];
    uint8_t* o1 = o0 + (m + n);
    for (uint32_t i = tid; i < L; i += LNW_THREADS) {
      uint8_t x, y;
      if (i < Lf) { x = tFA[Lf - 1 - i]; y = tFB[Lf - 1 - i]; }
      else if (i < Lf + gapref) { x = '-'; y = s2[refLeft + (i - Lf)]; }
      else { x = tRA[i - Lf - gapref]; y = tRB[i - Lf - gapref]; }
      o0[i] = x; o1[i] = y;
    }
    if (tid == 0) {
      a.ok[job] = 1; a.aln_len[job] = L;
      if (a.info) { a.info[4 * job] = consLeft; a.info[4 * job + 1] = refLeft; a.info[4 * job + 2] = (int) refRight; a.info[4 * job + 3] = gbest; }
    }
  }
}

// The wavefront kernel of each job class, its template arguments read from ln_geom: classes 1..15 on the packed engine, 17..31 the same
// geometries on the scalar engine; the PLAN kernels for calls under dgpu_set_ln_async_bound.
using LnKernel = void (*)(LnArgs, int);
template <bool PLAN, size_t... G>
constexpr std::array<LnKernel, 2 * LN_NCLS> ln_kernels(std::index_sequence<G...>) {
  return {{nullptr, ln_kernel2<ln_geom(G + 1).C, (ln_geom(G + 1).T > 32), ln_geom(G + 1).T, PLAN>..., nullptr,
           ln_kernel<ln_geom(G + 1).C, (ln_geom(G + 1).T > 32), ln_geom(G + 1).T, PLAN>...}};
}
constexpr std::array<LnKernel, 2 * LN_NCLS> LN_KERNELS[2] = {ln_kernels<false>(std::make_index_sequence<LN_NCLS - 1>()),
                                                             ln_kernels<true>(std::make_index_sequence<LN_NCLS - 1>())};

int check_max_ref(dgpu_ctx* ctx, uint32_t max_ref) {
  if (max_ref >= 1 && max_ref <= DGPU_LN_MAX_REF) return DGPU_OK;
  ctx->last_error = "dgpu_long_needle_ex: max_ref must be 1 .. " + std::to_string(DGPU_LN_MAX_REF);
  return DGPU_ERR_ARG;
}

// Launch shape of class c for consensus strings up to mmax bytes (wide class: windows up to max_ref): threads, dynamic shared memory and
// the CTAs per SM its grid is capped at.
struct LnShape { unsigned threads; size_t smem; int per_sm; };
LnShape ln_shape(int c, size_t mmax, uint32_t max_ref) {
  if (c == LN_WIDE) return {(unsigned) LNW_THREADS, lnw_smem(max_ref, mmax), 1};   // one 512-thread CTA per SM
  const LnGeom g = ln_geom(c & (LN_GEN - 1));
  if (c < LN_GEN) {
    const size_t smem = ln2_smem(g.C, g.T).bytes(mmax);
    return {(unsigned) g.T, smem, std::max(1, std::min<int>(ln2_occ(g.T), (int) ((200 * 1024) / (smem + 2048))))};
  }
  return {(unsigned) g.T, ln_smem_ups(g.C, g.T) + ((mmax + 15) & ~(size_t) 15), ln_per_sm(g.T)};
}

int ln_optin(dgpu_ctx* ctx, int c, bool plan, size_t smem) {
  if (c == LN_WIDE) return dgpu_smem_optin(ctx, plan ? lnw_kernel<true> : lnw_kernel<false>, smem, "cudaFuncSetAttribute(lnw_kernel)");
  return dgpu_smem_optin(ctx, LN_KERNELS[plan][c], smem, c < LN_GEN ? "cudaFuncSetAttribute(ln_kernel2)" : "cudaFuncSetAttribute(ln_kernel)");
}

int ln_launch(dgpu_ctx* ctx, int c, const LnArgs& a, unsigned grid, const LnShape& s, cudaStream_t cs) {
  const bool plan = a.plan != nullptr;
  int rc;
  if ((rc = ln_optin(ctx, c, plan, s.smem))) return rc;
  if (c == LN_WIDE) {
    (plan ? lnw_kernel<true> : lnw_kernel<false>)<<<grid, s.threads, s.smem, cs>>>(a);
    DGPU_LAUNCH_CHECK(ctx, "lnw_kernel");
  } else {
    LN_KERNELS[plan][c]<<<grid, s.threads, s.smem, cs>>>(a, c);
    DGPU_LAUNCH_CHECK(ctx, c < LN_GEN ? "ln_kernel2" : "ln_kernel");
  }
  return DGPU_OK;
}

// The classes a bound of max_cons x max_ref admits, each with its launch shape at the bound and the slab bytes of a bound-shaped job of
// the class: the wavefront classes whose narrowest window fits max_ref (both engines), and the wide class when the bound exceeds the
// wavefront shapes. The shapes are the same for both forms; dgpu_long_needle_dev takes only bounds without the wide class.
struct LnBoundClass { int c; LnShape s; unsigned long long slab; };
std::vector<LnBoundClass> ln_bound_classes(uint32_t max_cons, uint32_t max_ref) {
  std::vector<LnBoundClass> v;
  for (int c = 1; c < LN_NCLS; ++c) {
    const uint32_t nlo = c == 1 ? 1 : ln_geom(c - 1).cap - 6;   // the narrowest window of the class: n + 7 > the previous row's cap
    if (nlo > max_ref || nlo >= 32000) continue;
    const LnGeom g = ln_geom(c);
    const uint32_t n = std::min(max_ref, g.cap - 7), m = std::min(max_cons, 32000 - nlo);
    for (int e : {c, c + LN_GEN}) {
      const LnParts p = e < LN_GEN ? ln2_parts(g.C, g.T, m) : ln_parts(g.C, m, n);
      LnPlan pl;
      ln_slab(pl, p.rev, p.dirs, (unsigned long long) m + n);
      v.push_back({e, ln_shape(e, max_cons, max_ref), pl.work_stride});
    }
  }
  if (ln_class(max_cons, max_ref) < 0) v.push_back({LN_WIDE, ln_shape(LN_WIDE, max_cons, max_ref), lnw_geom(max_cons, max_ref).bytes});
  return v;
}

// the device form of both entry points; max_ref = 0: no wide engine (dgpu_long_needle_dev)
int ln_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off,
           const uint32_t* r_len, uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_len, uint8_t* ok, int32_t* info,
           uint32_t max_ref, void* stream) {
  if (n == 0) return DGPU_OK;
  if (n >= (1ull << 31) || seqs_bytes >= (1ull << 32)) return DGPU_ERR_ARG;
  if (!seqs || !c_off || !c_len || !r_off || !r_len || !aln || !aln_off || !aln_len || !ok) return DGPU_ERR_ARG;
  const bool bound = ctx->ln_max_cons != 0;   // dgpu_set_ln_async_bound: plan on the device, no readback
  if (bound && !max_ref && ln_class(ctx->ln_max_cons, ctx->ln_max_ref) < 0) {
    ctx->last_error = "dgpu_long_needle_dev: the asynchronous bound exceeds the wavefront shapes (|ref| <= 16377, |cons| + |ref| <= 32000); "
                      "use dgpu_long_needle_ex_dev";
    return DGPU_ERR_ARG;
  }
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t) stream : ctx->stream;
  LnArgs a{};
  a.seqs = seqs;
  a.c_off = c_off; a.c_len = c_len; a.r_off = r_off; a.r_len = r_len; a.n = (uint32_t) n;
  a.aln = aln; a.aln_off = aln_off; a.aln_len = aln_len; a.ok = ok; a.info = info;
  a.max_ref = max_ref; a.wide_budget = 0;
  a.bound_cons = ctx->ln_max_cons; a.bound_ref = ctx->ln_max_ref;
  a.plan = nullptr;
  void* p;
  int rc;
  if (bound) {   // every wide job inside the bound fits the pool (the setter sized it so)
    a.max_ref = std::min(max_ref, ctx->ln_max_ref);
    if (max_ref) a.wide_budget = lnw_geom(ctx->ln_max_cons, ctx->ln_max_ref).bytes;
  } else if (max_ref) {   // a wide job may take half of the workspace budget below; one that needs more is refused alone
    size_t free0 = 0, total0 = 0;
    cudaMemGetInfo(&free0, &total0);
    a.wide_budget = dgpu_workspace_budget(ctx, SLOT_WAVEFRONT, free0) / 2;
  }
  if ((rc = dgpu_reserve(ctx, SLOT_JOB_PERM, n * sizeof(uint32_t), &p))) return rc;
  a.perm = (uint32_t*) p;
  if ((rc = dgpu_reserve(ctx, SLOT_COUNTS, 2048 + 2 * LN_NCLS * sizeof(LnPlan), &p))) return rc;
  a.counts = (uint32_t*) p;                                   // 96 uint32 = 384 B
  a.maxcells = (unsigned long long*) ((uint8_t*) p + 512);     // 128 uint64 = 1024 B
  unsigned long long* d_unsupported = bound ? ctx->refused + DGPU_REFUSED_LN : (unsigned long long*) ((uint8_t*) p + 1536);
  LnPlan* d_plan = (LnPlan*) ((uint8_t*) p + 2048);
  DGPU_CUDA(ctx, cudaMemsetAsync(p, 0, 2048, st));
  void* pc;
  if ((rc = dgpu_reserve(ctx, SLOT_LN_JOBCLS, n + 64, &pc))) return rc;
  a.jobcls = (uint8_t*) pc;
  const uint32_t cb = (uint32_t) ((n + 255) / 256);
  ln_count_kernel<<<(uint32_t) ((n * 32 + 255) / 256), 256, 0, st>>>(a, d_unsupported);
  DGPU_LAUNCH_CHECK(ctx, "ln_count");
  ln_offsets_kernel<<<1, 1, 0, st>>>(a.counts);
  DGPU_LAUNCH_CHECK(ctx, "ln_offsets");
  ln_scatter_kernel<<<cb, 256, 0, st>>>(a);
  DGPU_LAUNCH_CHECK(ctx, "ln_scatter");
  if (bound) {
    // Launch every class the bound admits with its grid cap and the shared memory of the bound; ln_plan_kernel gives each its slabs and
    // its active CTAs in the pool, and the CTAs above them (all of an empty class's) return at once.
    std::vector<LnBoundClass> cls = ln_bound_classes(ctx->ln_max_cons, ctx->ln_max_ref);
    if (!max_ref && !cls.empty() && cls.back().c == LN_WIDE) cls.pop_back();
    LnPlanIn in{};
    for (const LnBoundClass& k : cls) in.gmax[k.c] = (uint32_t) ctx->num_sms * k.s.per_sm;
    in.pool = ctx->ln_pool;
    if ((rc = dgpu_reserve(ctx, SLOT_WAVEFRONT, ctx->ln_pool, &p))) return rc;
    a.work = (uint8_t*) p;
    ln_plan_kernel<<<1, 32, 0, st>>>(a.counts, a.maxcells, in, d_plan);
    DGPU_LAUNCH_CHECK(ctx, "ln_plan");
    a.plan = d_plan;
    DgpuFork fork(ctx, st, cls.size());
    if ((rc = fork.begin())) return rc;
    for (const LnBoundClass& k : cls) {
      cudaStream_t cs;
      if ((rc = fork.next(cs)) || (rc = ln_launch(ctx, k.c, a, in.gmax[k.c], k.s, cs))) return rc;
    }
    return fork.end();
  }
  struct { uint32_t counts[128]; unsigned long long maxc[128]; unsigned long long unsupported; } h;
  DGPU_CUDA(ctx, cudaMemcpyAsync(&h, p, sizeof(h), cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  if (h.unsupported) {   // per-item refusal: those jobs come back with ok = 0 (and info[2] = -1); never a silent approximation, never a failed batch
    ctx->unsupported += h.unsupported;
    ctx->last_error = max_ref
        ? "dgpu_long_needle_ex: " + std::to_string(h.unsupported) + " job(s) with |ref| > max_ref (" + std::to_string(max_ref) + "), |cons| > " +
              std::to_string(LNW_MAX_CONS) + " or a workspace beyond the device budget were not aligned (ok = 0)"
        : "dgpu_long_needle: " + std::to_string(h.unsupported) + " job(s) with |cons|+|ref| > 32000 or |ref| > 16377 were not aligned (ok = 0)";
  }
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  // Plan every non-empty class first (ln_fit within the workspace budget). The classes then run CONCURRENTLY on a small pool of
  // streams forked from `st` (each class has its own region of the workspace): a batch of a few hundred SVs spread over
  // several classes would otherwise run as a sequence of under-filled launches.
  // Classes 1..15: jobs over ACGTN only -> packed two-row engine (ln_kernel2); 17..31: the same geometries for jobs with other bytes -> scalar engine.
  LnShape shape[2 * LN_NCLS];
  uint32_t cap[2 * LN_NCLS] = {};
  size_t nplans = 0;
  for (int c = 1; c < 2 * LN_NCLS; ++c)
    if (h.counts[c]) {
      shape[c] = ln_shape(c, (size_t) h.maxc[96 + c], max_ref);
      cap[c] = (uint32_t) ctx->num_sms * shape[c].per_sm;
      ++nplans;
    }
  LnPlan pl[2 * LN_NCLS];
  const size_t total = ln_fit(h.counts, h.maxc, cap, dgpu_workspace_budget(ctx, SLOT_WAVEFRONT, free_b), pl);
  if ((rc = dgpu_reserve(ctx, SLOT_WAVEFRONT, total, &p))) return rc;
  DgpuFork fork(ctx, st, nplans);
  if ((rc = fork.begin())) return rc;
  for (int c = 1; c < 2 * LN_NCLS; ++c) {
    if (!pl[c].grid) continue;
    LnArgs ac = a;
    ac.work = (uint8_t*) p + pl[c].base;
    ac.work_stride = pl[c].work_stride; ac.off_dirsR = pl[c].off_dirsR; ac.off_dirsF = pl[c].off_dirsF; ac.off_trace = pl[c].off_trace;
    cudaStream_t cs;
    if ((rc = fork.next(cs)) || (rc = ln_launch(ctx, c, ac, pl[c].grid, shape[c], cs))) return rc;
  }
  return fork.end();
}

// the host form of both entry points (max_ref = 0: dgpu_long_needle)
int ln_host(dgpu_ctx* ctx, const char* name, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* c_off, const uint32_t* c_len,
            const uint32_t* r_off, const uint32_t* r_len, uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_len,
            uint8_t* ok, int32_t* info, uint32_t max_ref) {
  DgpuStage s(ctx, name, n);
  if (!ctx) return DGPU_ERR_ARG;
  if (n == 0) return DGPU_OK;
  if (!seqs || !c_off || !c_len || !r_off || !r_len || !aln || !aln_off || !aln_len || !ok) return DGPU_ERR_ARG;
  int rc;
  if ((rc = s.check_arena(seqs_bytes, n, c_off, c_len)) || (rc = s.check_arena(seqs_bytes, n, r_off, r_len))) return rc;
  for (uint64_t i = 0; i < n; ++i)   // alignment slots (2 rows of |cons| + |ref|) inside aln_bytes
    if (aln_off[i] + 2ull * ((uint64_t) c_len[i] + r_len[i]) > aln_bytes) { ctx->last_error = std::string(name) + ": alignment slot beyond aln_bytes"; return DGPU_ERR_CAPACITY; }
  if ((rc = s.open())) return rc;
  const uint8_t* d_seqs = s.arena(seqs, seqs_bytes);
  uint8_t* d_aln = s.out(aln, aln_bytes, 64);
  const uint32_t *d_coff = s.in(c_off, n), *d_clen = s.in(c_len, n), *d_roff = s.in(r_off, n), *d_rlen = s.in(r_len, n);
  const uint64_t* d_aoff = s.in(aln_off, n);
  uint32_t* d_alen = s.out(aln_len, n);
  uint8_t* d_ok = s.out(ok, n);
  int32_t* d_info = s.out(info, n * 4);   // null when the caller wants no info rows
  if (s.rc) return s.rc;
  if ((rc = ln_dev(ctx, d_seqs, seqs_bytes, d_coff, d_clen, d_roff, d_rlen, n, d_aln, d_aoff, d_alen, d_ok, d_info, max_ref, s.st))) return rc;
  return s.finish();
}

}  // namespace

extern "C" {

int dgpu_set_ln_async_bound(dgpu_ctx* ctx, uint32_t max_cons, uint32_t max_ref) {
  if (!ctx) return DGPU_ERR_ARG;
  if (!max_cons && !max_ref) { ctx->ln_max_cons = ctx->ln_max_ref = 0; ctx->ln_pool = 0; return DGPU_OK; }
  if (!max_cons || !max_ref || max_cons > LNW_MAX_CONS || max_ref > DGPU_LN_MAX_REF) {
    ctx->last_error = "dgpu_set_ln_async_bound: max_cons must be 1 .. " + std::to_string(LNW_MAX_CONS) + " and max_ref 1 .. " +
                      std::to_string(DGPU_LN_MAX_REF) + " (or both 0)";
    return DGPU_ERR_ARG;
  }
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  // The pool: every admitted class at its grid cap with bound-shaped slabs, within the workspace budget, but never less than one
  // bound-shaped slab per class (ln_plan_kernel relies on that).
  unsigned long long one = 0, all = 0;
  int rc;
  for (const LnBoundClass& k : ln_bound_classes(max_cons, max_ref)) {
    if ((rc = ln_optin(ctx, k.c, true, k.s.smem))) return rc;
    one += k.slab;
    all += (unsigned long long) ctx->num_sms * k.s.per_sm * k.slab;
  }
  size_t free_b = 0, total_b = 0;
  DGPU_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  const size_t pool = std::max<size_t>(one, std::min<size_t>(all, dgpu_workspace_budget(ctx, SLOT_WAVEFRONT, free_b)));
  void* p;
  if ((rc = dgpu_reserve(ctx, SLOT_WAVEFRONT, pool, &p)) || (rc = dgpu_reserve(ctx, SLOT_COUNTS, 2048 + 2 * LN_NCLS * sizeof(LnPlan), &p)) ||
      (rc = dgpu_fork_init(ctx)) || (rc = dgpu_refusals_init(ctx)))
    return rc;
  ctx->ln_max_cons = max_cons; ctx->ln_max_ref = max_ref; ctx->ln_pool = pool;
  return DGPU_OK;
}

int dgpu_long_needle_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                         const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off, const uint32_t* r_len,
                         uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_len, uint8_t* ok,
                         int32_t* info, void* stream) {
  if (!ctx) return DGPU_ERR_ARG;
  return ln_dev(ctx, seqs, seqs_bytes, c_off, c_len, r_off, r_len, n, aln, aln_off, aln_len, ok, info, 0, stream);
}

int dgpu_long_needle_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off, const uint32_t* r_len,
                            uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_len, uint8_t* ok,
                            int32_t* info, uint32_t max_ref, void* stream) {
  if (!ctx) return DGPU_ERR_ARG;
  int rc;
  if ((rc = check_max_ref(ctx, max_ref))) return rc;
  return ln_dev(ctx, seqs, seqs_bytes, c_off, c_len, r_off, r_len, n, aln, aln_off, aln_len, ok, info, max_ref, stream);
}

int dgpu_long_needle(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                     const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off, const uint32_t* r_len,
                     uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_len, uint8_t* ok,
                     int32_t* info) {
  return ln_host(ctx, "dgpu_long_needle", seqs, seqs_bytes, c_off, c_len, r_off, r_len, n, aln, aln_off, aln_bytes, aln_len, ok, info, 0);
}

int dgpu_long_needle_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                        const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off, const uint32_t* r_len,
                        uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_len, uint8_t* ok,
                        int32_t* info, uint32_t max_ref) {
  if (!ctx) return DGPU_ERR_ARG;
  int rc;
  if ((rc = check_max_ref(ctx, max_ref))) return rc;
  return ln_host(ctx, "dgpu_long_needle_ex", seqs, seqs_bytes, c_off, c_len, r_off, r_len, n, aln, aln_off, aln_bytes, aln_len, ok, info, max_ref);
}

}  // extern "C"
