// edit_path.cu — batched edlibAlign(..., EDLIB_TASK_PATH): edit distance, start/end location and the
// edit-operation path (0 match, 1 insert, 2 delete, 3 mismatch). Problems whose estimated alignment data is below
// 1 MiB are traced back directly, larger ones are split with Hirschberg's recursion exactly where the reference
// splits them (src/edlib.cpp:1189-1212, :1232-1397): target halved, FIRST query row (interior rows ascending, then the
// -1 boundary, then the last row) whose left and right half-column distances add up to the optimum, recursion on the
// upper-left and lower-right sub-problems with those two distances as their optima.
//
// Reference semantics reproduced:
//   * distance and first end location as dgpu_edit_distance (src/edlib.cpp:545-702, :728-929);
//   * HW start location: end - (LAST optimal end of the reversed query in the reversed target prefix, SHW,
//     k = distance) (src/edlib.cpp:226-254); end location -1 -> start 0 and an all-insert path (:241);
//     SHW and NW start at 0;
//   * the path is the global alignment of the query against target[start..end] traced back from the bottom
//     right cell with priority up (insert) > left (delete) > diagonal (src/edlib.cpp:1021-1131); the band the
//     reference restricts itself to never changes that choice because every cell that can be chosen has a
//     value <= the optimum and is therefore exact.
// The traceback matrix is produced by the same anti-diagonal wavefront engine as longNeedle (wavefront.cuh)
// with scoring (match 0, mismatch -1, gap -1), i.e. score = -distance.
#include "common.cuh"
#include "myers.cuh"
#include "wavefront.cuh"
#include <algorithm>
#include <array>
#include <utility>

int dgpu_edit_distance_impl(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* q_off, const uint32_t* q_len,
                            const uint32_t* t_off, const uint32_t* t_len, const int32_t* k, int mode, uint64_t n, int32_t* dist,
                            int32_t* end_loc, void* stream, int last_pos, const uint32_t* eq_tabs, uint32_t async_bound);

#include <vector>

namespace {

// ------------------------------------------------------------------------------------------------------------
// Device side of stages 1-2 (distance, end, HW start) — unchanged semantics, see header comment.
// Job w's sequence seqs[off[w] .. +len[w]) reversed into mirror[dst[w] ..]. Every job has its own mirror bytes: sequences may share arena
// bytes (a query inside its target, overlapping windows of one contig), and a reversal written back at the arena address would overwrite them.
__global__ void ep_mirror_kernel(const uint8_t* seqs, uint8_t* mirror, const uint32_t* off, const uint32_t* len, const uint32_t* dst, uint32_t n) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n) return;
  const uint32_t o = off[w], L = len[w], d = dst[w];
  for (uint32_t i = lane; i < L; i += 32) mirror[d + i] = seqs[o + L - 1 - i];
}

// mt_off: where the reversed target starts in the mirror
__global__ void ep_hwstart_jobs_kernel(const uint32_t* mt_off, const uint32_t* t_len, const int32_t* dist, const int32_t* end_loc, uint32_t n,
                                       uint32_t* t2_off, uint32_t* t2_len, int32_t* k2) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int e = end_loc[i], d = dist[i];
  if (d < 0 || e < 0) { t2_off[i] = mt_off[i]; t2_len[i] = 0; k2[i] = 0; return; }
  t2_off[i] = mt_off[i] + (t_len[i] - (uint32_t) e - 1);
  t2_len[i] = (uint32_t) e + 1;
  k2[i] = d;
}

__global__ void ep_start_kernel(int mode, const uint32_t* q_len, const uint32_t* t_len, const int32_t* dist, const int32_t* end_loc, const int32_t* rev_pos,
                                uint32_t n, int32_t* start_loc) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = dist[i], e = end_loc[i];
  if (q_len[i] == 0 || t_len[i] == 0 || d < 0) { start_loc[i] = -1; return; }  // edlibAlign returns before locations exist (src/edlib.cpp:158-177)
  start_loc[i] = (mode == DGPU_MODE_HW && e >= 0) ? e - rev_pos[i] : 0;
}

// NW distance through the wavefront engine when generalised equalities are in play (score-only pass)
// and the segment work below share one job description.
struct SegJobs {
  const uint8_t* seqs;
  const uint32_t* q_off;   // query slice
  const uint32_t* q_len;
  const uint32_t* t_off;   // target slice
  const uint32_t* t_len;
  const uint8_t* rev;      // 1: run on the reversed slices (Hirschberg's right half)
  const uint8_t* kind;     // 0: traceback -> ops ; 1: last column -> colbuf
  const uint64_t* out_off; // kind 0: byte offset in tmp ops ; kind 1: int offset in colbuf
  uint32_t* out_len;       // kind 0: number of ops written
  int32_t* corner;         // -distance of the slice (both kinds)
  uint8_t* tmp_ops;
  int* colbuf;
  const uint32_t* list;    // job indices of this class
  uint32_t count;
  uint8_t* work;
  size_t work_stride, off_trace;
  wf::EqTables eq;
  // banded bit-parallel segments (seg_band_kernel)
  const uint32_t* plan_m;  // rows / columns of the problem whose band the segment lives in: its own for a leaf, the parent's for a half column
  const uint32_t* plan_n;
  const uint8_t* eq_cls;   // class table of the generalised equality (null: byte equality)
  const uint32_t* plan_count;  // PLAN kernels (asynchronous form): the number of jobs in `list`, on the device; `count` is not read
};

// the job count of a class kernel: a.count, or the count the device planned (PLAN)
template <bool PLAN>
__device__ __forceinline__ uint32_t seg_count(const SegJobs& a) { return PLAN ? *a.plan_count : a.count; }

// Geometry of the seg_kernel classes: a segment of n target columns takes the first row with n <= cap (class 0: n = 0), with C columns
// per lane, T threads per CTA (MULTI: T > 32) and a grid of at most per_sm CTAs per SM.
struct SegGeom { uint32_t cap; int C, T, per_sm; };
constexpr int SEG_NCLS = 12;
constexpr SegGeom SEG_GEOM[SEG_NCLS] = {{0, 0, 0, 0},
                                        {256, 8, 32, 16}, {512, 16, 32, 16}, {768, 24, 32, 16}, {1024, 32, 32, 16},
                                        {1280, 40, 32, 16}, {1536, 48, 32, 16}, {1792, 56, 32, 16}, {2048, 64, 32, 16},
                                        {4096, 32, 128, 4}, {8192, 32, 256, 2}, {16384, 32, 512, 1}};
__host__ __device__ inline uint32_t seg_dstride(uint32_t n, uint32_t C) { return ((n + C - 1) / C + 1) * (C / 8); }
// the first row of SEG_GEOM whose cap holds n; -1: none (written out for device code, checked against the table below)
__host__ __device__ constexpr int seg_class(uint32_t n) {
  return n <= 2048 ? (int) ((n + 255) / 256) : n <= 4096 ? 9 : n <= 8192 ? 10 : n <= 16384 ? 11 : -1;
}
constexpr bool seg_class_matches_geom() {
  for (int c = 1; c < SEG_NCLS; ++c)
    if (seg_class(SEG_GEOM[c].cap) != c || seg_class(SEG_GEOM[c - 1].cap + 1) != c) return false;
  return seg_class(0) == 0 && seg_class(SEG_GEOM[SEG_NCLS - 1].cap + 1) == -1;
}
static_assert(seg_class_matches_geom(), "seg_class and SEG_GEOM disagree");

template <int C, bool MULTI, bool EQ, bool PLAN = false>
__global__ void __launch_bounds__(MULTI ? 512 : 32) seg_kernel(SegJobs a) {
  extern __shared__ uint8_t sm_rows[];
  __shared__ int sm_x[wf::WF_SMX];
  __shared__ int sm_pub[4];
  const int tid = threadIdx.x, T = blockDim.x;
  uint8_t* slab = a.work + (size_t) blockIdx.x * a.work_stride;
  uint32_t* dirs = (uint32_t*) slab;
  uint8_t* trace = slab + a.off_trace;
  const wf::Scoring sc = {0, -1, false, false};
  const uint32_t count = seg_count<PLAN>(a);
  for (uint32_t idx = blockIdx.x; idx < count; idx += gridDim.x) {
    const uint32_t job = a.list[idx];
    const uint32_t m = a.q_len[job], n = a.t_len[job];
    const uint8_t* q = a.seqs + a.q_off[job];
    const uint8_t* t = a.seqs + a.t_off[job];
    const bool rev = a.rev[job] != 0;
    const int kind = a.kind[job];
    const uint32_t dstride = seg_dstride(n, C);
    __syncthreads();
    for (uint32_t i = tid; i < m; i += T) sm_rows[i] = rev ? q[m - 1 - i] : q[i];
    __syncthreads();
    wf::Best dummy;
    int corner;
    auto rowc = [&](int i) { return sm_rows[i]; };
    if (rev) {
      wf::pass<C, MULTI, wf::PLAIN, EQ>(rowc, [&](int j) { return t[n - 1 - j]; }, (int) m, (int) n, sc, 1, kind == 0 ? dirs : nullptr, dstride, nullptr, 0, 0,
                                        sm_x, dummy, corner, &a.eq, kind == 1 ? a.colbuf + a.out_off[job] : nullptr);
    } else {
      wf::pass<C, MULTI, wf::PLAIN, EQ>(rowc, [&](int j) { return t[j]; }, (int) m, (int) n, sc, 1, kind == 0 ? dirs : nullptr, dstride, nullptr, 0, 0, sm_x,
                                        dummy, corner, &a.eq, kind == 1 ? a.colbuf + a.out_off[job] : nullptr);
    }
    __syncthreads();
    if (kind == 0) {
      if (tid == 0) {
        // traceback: up (insert, 1) > left (delete, 2) > diagonal (match 0 / mismatch 3), src/edlib.cpp:1021-1131
        uint32_t rr = m, cc = n, k = 0;
        while (rr > 0 || cc > 0) {
          uint32_t code;
          if (rr == 0) code = 2;
          else if (cc == 0) code = 1;
          else {
            uint32_t w = __ldcg(dirs + (size_t) rr * dstride + ((cc - 1) >> 3));
            code = (w >> (((cc - 1) & 7) * 4)) & 3u;
          }
          uint8_t op;
          if (code == 1) { --rr; op = 1; }
          else if (code == 2) { --cc; op = 2; }
          else {
            --rr; --cc;
            const uint32_t x = sm_rows[rr], y = t[cc];
            op = (EQ ? a.eq.equal(x, y) : (x == y)) ? 0 : 3;
          }
          trace[k++] = op;
        }
        sm_pub[0] = (int) k;
      }
      __syncthreads();
      const uint32_t L = (uint32_t) sm_pub[0];
      uint8_t* o = a.tmp_ops + a.out_off[job];
      for (uint32_t i = tid; i < L; i += T) o[i] = trace[L - 1 - i];
      if (tid == 0) a.out_len[job] = L;
    }
    if (tid == 0) a.corner[job] = corner;
  }
}

// ---- banded bit-parallel segments -------------------------------------------------------------------------------------------------------
// The same staircase band as ed_band_kernel (edit_distance.cu), on Hirschberg's segments. A segment's optimum is known before it is run
// (a leaf's from the split that produced it, a half column's parent from the distance pass), so the host picks the narrowest class whose
// certified range contains it and ONE pass is exact for every cell an optimal path can touch:
//   kind 1 (half column): the last DP column, exact on the rows optimal paths of the parent cross, over-estimated (or "infinite")
//     elsewhere — hb_select_kernel only ever tests l + r == optimum, which over-estimates cannot satisfy. Both halves of a parent use the
//     parent's band (the reversed problem maps it onto itself).
//   kind 0 (leaf): every lane stores, per column, its block's vertical deltas after the column (Pv) and the horizontal deltas into the
//     column (Ph): 2 bits per cell, all leaf_trace needs. Ops are written from the END of the job's slot backwards (out_len says how
//     many); the host shifts the leaf offset.
constexpr int SEGB_WARPS = 2;

template <int G, bool EQ, bool PLAN = false>
__global__ void __launch_bounds__(SEGB_WARPS * 32) seg_band_kernel(SegJobs a) {
  constexpr int JPW = 32 / G;
  constexpr int PEQ_JOB = EDB_PEQ_WORDS / JPW;
  constexpr int WCOLS = (4 * G < 32) ? 4 * G : 32;
  __shared__ uint64_t peq_s[SEGB_WARPS][EDB_PEQ_WORDS];
  __shared__ uint64_t hoP[SEGB_WARPS][32], hoM[SEGB_WARPS][32];
  __shared__ int hoS[SEGB_WARPS][32];
  __shared__ uint4 win_s[SEGB_WARPS][JPW * WCOLS];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int p = lane & (G - 1), grp = lane / G;
  const uint32_t gwarp = blockIdx.x * SEGB_WARPS + wib, nwarps = gridDim.x * SEGB_WARPS;
  uint64_t* peq = &peq_s[wib][grp * PEQ_JOB];
  uint4* win = &win_s[wib][grp * WCOLS];
  uint4* store = (uint4*) (a.work + ((size_t) gwarp * JPW + grp) * a.work_stride);
  const EqTabs tabs = {a.eq.f, a.eq.s, a.eq_cls};

  for (uint32_t base = gwarp * JPW; base < seg_count<PLAN>(a); base += nwarps * JPW) {   // the count is read where it is used, as a.count was
    const bool have = base + grp < seg_count<PLAN>(a);
    const uint32_t job = have ? a.list[base + grp] : 0;
    const int m = have ? (int) a.q_len[job] : 0, n = have ? (int) a.t_len[job] : 0;
    const uint8_t* q = a.seqs + (have ? a.q_off[job] : 0);
    const uint8_t* t = a.seqs + (have ? a.t_off[job] : 0);
    const bool rev = have && a.rev[job] != 0;
    const int kind = have ? (int) a.kind[job] : 1;
    const int nblk = (m + 63) >> 6;
    const BandPlan bp = band_plan(G, have ? (int) a.plan_m[job] : 1, have ? (int) a.plan_n[job] : 1);

    __syncwarp();
    band_build_peq<G>(peq, q, m, rev, p);
    __syncwarp();

    uint64_t Pv, Mv;
    int sc, blk, plast;
    band_pass<G, EQ>(peq, q, t, m, n, rev, bp, hoP[wib], hoM[wib], hoS[wib], tabs, Pv, Mv, sc, blk, [&](int st, uint64_t pv, uint64_t ph) {
      if (kind == 0) store[(size_t) st * G + p] = make_uint4((uint32_t) pv, (uint32_t) (pv >> 32), (uint32_t) ph, (uint32_t) (ph >> 32));
    });
    __threadfence_block();
    __syncwarp();

    // corner: D[m][n] when the band holds it (a leaf's always does), reported as a score like the wavefront kernels do
    const int s = band_corner<G>(Pv, Mv, sc, m, n, bp, plast);
    if (have && p == 0) a.corner[job] = (plast >= 0 && plast < G) ? -s : 1;

    if (kind == 1 && have) {
      int* colv = a.colbuf + a.out_off[job];
      for (int i = p; i <= m; i += G) colv[i] = -(1 << 28);
    }
    __syncwarp();
    if (kind == 1 && have) {
      int* colv = a.colbuf + a.out_off[job];
      if (p == 0) colv[0] = -n;
      if (blk >= 0 && blk < nblk) {
        int v = sc;
        for (int j = 63; j >= 0; --j) {
          const int i = 64 * blk + j + 1;
          if (i <= m) colv[i] = -v;
          v -= (int) ((Pv >> j) & 1ull) - (int) ((Mv >> j) & 1ull);
        }
      }
    }

    const bool act = have && kind == 0;
    const uint32_t k = leaf_trace<G, WCOLS, EQ>(act, q, t, m, n, rev, a.eq, win, a.tmp_ops + (have ? a.out_off[job] : 0), [&](int col, int b) {
      const int Jc = col >> 6, pp = b - (Jc - bp.A);
      return pp >= 0 && pp < G ? __ldcg(store + ((size_t) (65 * Jc + (col & 63) + pp) * G + pp)) : make_uint4(0, 0, 0, 0);
    });
    if (act && p == 0) a.out_len[job] = k;
    __syncwarp();
  }
}

// ---- segments wider than the wavefront classes (n > 16384 columns) that no band class certifies ---------------------------------------
// Hirschberg only produces these from slices wider than 16384 columns: half columns of any height and width, and leaves of at most two
// 64-row blocks (20 ceil(m/64) n + 8 n < 2^20 with n > 16384 forces m <= 128).
constexpr int EPW_WARPS = 4;     // warps per CTA of seg_half_wide_kernel
constexpr int EPL_WARPS = 2;     // warps per CTA of seg_leaf_wide_kernel
constexpr int EPL_G = 2;         // lanes per leaf: one per 64-row block
constexpr int EPL_WCOLS = 32;    // traceback window, columns

// Half column (kind 1) of an unbanded segment: one warp per segment on ed_long_kernel's striped wavefront (stripes), its bottom deltas
// parked in the warp's scratch row (n bytes). NW top boundary (D[0][j] = j), rows / columns read back to front when rev. After each
// stripe the lanes' final Pv / Mv are the vertical deltas of column n, which give colbuf[out_off + i] = -D[i][n] for every row of the
// stripe, run on from the stripe above; the column is exact on every row.
template <bool EQ, bool PLAN = false>
__global__ void __launch_bounds__(EPW_WARPS * 32) seg_half_wide_kernel(SegJobs a, size_t hrow_stride) {
  __shared__ uint64_t peq_s[EPW_WARPS][5][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t gwarp = blockIdx.x * EPW_WARPS + wib, nwarps = gridDim.x * EPW_WARPS;
  volatile int8_t* hrow = (volatile int8_t*) (a.work + (size_t) gwarp * hrow_stride);
  const EqTabs tabs = {a.eq.f, a.eq.s, a.eq_cls};
  const uint32_t count = seg_count<PLAN>(a);
  for (uint32_t idx = gwarp; idx < count; idx += nwarps) {
    const uint32_t job = a.list[idx];
    const uint32_t m = a.q_len[job], n = a.t_len[job];
    const uint8_t* q = a.seqs + a.q_off[job];
    const uint8_t* t = a.seqs + a.t_off[job];
    const bool rev = a.rev[job] != 0;
    int* colv = a.colbuf + a.out_off[job];
    if (lane == 0) colv[0] = -(int) n;
    int top = (int) n;   // D[s * 2048][n]: the column value above the current stripe
    stripes<EQ>(peq_s[wib], hrow, q, t, m, n, rev, 1, tabs, [](int, uint64_t, uint64_t) {},
                [&](uint32_t row0, int rows, uint64_t Pv, uint64_t Mv) {
                  // this stripe's rows of column n: exclusive prefix of the lanes' delta sums, then each lane writes its own rows
                  const uint64_t valid = rows == 64 ? ~0ull : ((1ull << rows) - 1);
                  const int sum = __popcll(Pv & valid) - __popcll(Mv & valid);
                  int incl = sum;
                  for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                  }
                  int v = top + incl - sum;
                  for (int j = 0; j < rows; ++j) {
                    v += (int) ((Pv >> j) & 1ull) - (int) ((Mv >> j) & 1ull);
                    colv[row0 + j + 1] = -v;
                  }
                  top += __shfl_sync(0xffffffffu, incl, 31);
                });
    if (lane == 0) a.corner[job] = -top;
  }
}

// Leaf (kind 0) of at most two 64-row blocks and any width: EPL_G = 2 lanes per leaf, 16 leaves per warp. Lane p holds block p over the
// whole column (lane 1 one step behind lane 0, its horizontal delta arriving by shuffle) and stores (Pv after the column, Ph into the
// column) for every column, 16 B per lane-column. The traceback is seg_band_kernel's (leaf_trace, a window of EPL_WCOLS columns).
template <bool EQ, bool PLAN = false>
__global__ void __launch_bounds__(EPL_WARPS * 32) seg_leaf_wide_kernel(SegJobs a) {
  constexpr int G = EPL_G, JPW = 32 / G;
  __shared__ uint64_t peq_s[EPL_WARPS][JPW * G * EDB_BLOCK_WORDS];
  __shared__ uint4 win_s[EPL_WARPS][JPW * EPL_WCOLS];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int p = lane & (G - 1), grp = lane / G;
  const uint32_t gwarp = blockIdx.x * EPL_WARPS + wib, nwarps = gridDim.x * EPL_WARPS;
  uint64_t* peq = &peq_s[wib][grp * G * EDB_BLOCK_WORDS];
  uint4* win = &win_s[wib][grp * EPL_WCOLS];
  uint4* store = (uint4*) (a.work + ((size_t) gwarp * JPW + grp) * a.work_stride);
  const EqTabs tabs = {a.eq.f, a.eq.s, a.eq_cls};

  const uint32_t count = seg_count<PLAN>(a);
  for (uint32_t base = gwarp * JPW; base < count; base += nwarps * JPW) {
    const bool have = base + grp < count;
    const uint32_t job = have ? a.list[base + grp] : 0;
    const int m = have ? (int) a.q_len[job] : 0, n = have ? (int) a.t_len[job] : 0;
    const uint8_t* q = a.seqs + (have ? a.q_off[job] : 0);
    const uint8_t* t = a.seqs + (have ? a.t_off[job] : 0);
    const bool rev = have && a.rev[job] != 0;
    const int nblk = (m + 63) >> 6;
    const bool mine = p < nblk;   // this lane holds a block of the leaf

    __syncwarp();
    band_build_peq<G>(peq, q, m, rev, p);
    __syncwarp();

    int steps = have ? n + G - 1 : 0;
    for (int o = 16; o; o >>= 1) steps = max(steps, __shfl_xor_sync(0xffffffffu, steps, o));
    uint64_t Pv = ~0ull, Mv = 0;
    int hout = 1, sc = m;   // sc: D[m][col + 1] on the lane of the last block
    const int tb = (m - 1) & 63;
    uint32_t chn = (have && n > 0) ? __ldg(rev ? t + (n - 1) : t) : 0u;
    for (int st = 0; st < steps; ++st) {
      const int hin_sh = __shfl_up_sync(0xffffffffu, hout, 1, G);
      const int col = st - p;
      if (mine && col >= 0 && col < n) {
        const uint32_t ch = chn;
        if (col + 1 < n) chn = __ldg(rev ? t + (n - 2 - col) : t + col + 1);
        const uint64_t Eq = band_eq<EQ>(peq, p, ch, q, m, rev, tabs);
        uint64_t Ph, Mh;
        hout = block64(Pv, Mv, Eq, p == 0 ? 1 : hin_sh, Ph, Mh);
        if (p == nblk - 1) sc += (int) ((Ph >> tb) & 1ull) - (int) ((Mh >> tb) & 1ull);
        store[(size_t) col * nblk + p] = make_uint4((uint32_t) Pv, (uint32_t) (Pv >> 32), (uint32_t) Ph, (uint32_t) (Ph >> 32));
      }
    }
    __threadfence_block();
    __syncwarp();
    {
      const int s = __shfl_sync(0xffffffffu, sc, grp * G + ((nblk - 1) & (G - 1)));
      if (have && p == 0) a.corner[job] = -s;
    }

    const uint32_t k = leaf_trace<G, EPL_WCOLS, EQ>(have, q, t, m, n, rev, a.eq, win, a.tmp_ops + (have ? a.out_off[job] : 0),
                                                    [&](int col, int b) { return __ldcg(store + (size_t) col * nblk + b); });
    if (have && p == 0) a.out_len[job] = k;
    __syncwarp();
  }
}

// Hirschberg split row (src/edlib.cpp:1303-1338): F = forward half column (F[i] = -fcol[i]), B = reverse half column
// (B[i] = -bcol[m-i]); interior rows i = 1..m-1 ascending, then i = 0, then i = m. One warp per segment. PLAN: the segment count is
// *plan_nseg, on the device.
template <bool PLAN = false>
__global__ void hb_select_kernel(const int* colbuf, const uint64_t* f_off, const uint64_t* b_off, const uint32_t* m_arr, const uint32_t* h_arr,
                                 const uint32_t* n_arr, const int32_t* best_arr, uint32_t nseg, const uint32_t* plan_nseg, int32_t* out3) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= (PLAN ? *plan_nseg : nseg)) return;
  const int* F = colbuf + f_off[w];
  const int* B = colbuf + b_off[w];
  const int m = (int) m_arr[w], h = (int) h_arr[w], n = (int) n_arr[w], best = best_arr[w];
  int found = -2, ls = 0, rs = 0;
  for (int i0 = 1; i0 < m && found == -2; i0 += 32) {
    const int i = i0 + lane;
    bool ok = false;
    int l = 0, r = 0;
    if (i < m) { l = -F[i]; r = -B[m - i]; ok = (l + r == best); }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (bal) {
      const int src = __ffs(bal) - 1;
      found = i0 + src;
      ls = __shfl_sync(0xffffffffu, l, src);
      rs = __shfl_sync(0xffffffffu, r, src);
    }
  }
  if (found == -2) {
    const int r0 = -B[m];  // i = 0: whole query against the right half
    if (h + r0 == best) { found = 0; ls = h; rs = r0; }
    else {
      const int lm = -F[m];  // i = m: whole query against the left half
      if (lm + (n - h) == best) { found = m; ls = lm; rs = n - h; }
    }
  }
  if (lane == 0) { out3[3 * w] = found; out3[3 * w + 1] = ls; out3[3 * w + 2] = rs; }
}

// Concatenate the leaves of every job into its final ops array. One warp per job.
__global__ void hb_concat_kernel(const uint8_t* tmp_ops, const uint32_t* job_leaf_lo, const uint32_t* leaf_kind /*0 traced,1 all insert,2 all delete*/,
                                 const uint64_t* leaf_off, const uint32_t* leaf_len, uint32_t njobs, uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= njobs) return;
  uint8_t* o = ops + ops_off[w];
  uint32_t pos = 0;
  for (uint32_t l = job_leaf_lo[w]; l < job_leaf_lo[w + 1]; ++l) {
    const uint32_t L = leaf_len[l], kd = leaf_kind[l];
    if (kd == 0) { const uint8_t* src = tmp_ops + leaf_off[l]; for (uint32_t i = lane; i < L; i += 32) o[pos + i] = src[i]; }
    else { const uint8_t v = (kd == 1) ? 1 : 2; for (uint32_t i = lane; i < L; i += 32) o[pos + i] = v; }
    pos += L;
  }
  if (lane == 0) ops_len[w] = pos;
}

struct Seg { uint32_t job, qoff, qlen, toff, tlen; int32_t score; };

// Runs a set of SegJobs (already on the host) class by class.
struct SegRunner {
  dgpu_ctx* ctx;
  cudaStream_t st;
  const uint8_t* seqs;
  wf::EqTables eq;
  bool use_eq;
  std::vector<uint32_t> qoff, qlen, toff, tlen;
  std::vector<uint8_t> rev, kind;
  std::vector<uint64_t> out_off;
  std::vector<uint32_t> plan_m, plan_n;  // problem whose band the segment lives in (seg_band_kernel)
  std::vector<int32_t> bound;            // optimum of that problem
  std::vector<uint8_t> tail_ops;         // set by run(): the segment went through seg_band_kernel or seg_leaf_wide_kernel (a leaf's ops then end at
                                         // the end of its slot)
  const uint8_t* eq_cls = nullptr;
  void clear() { qoff.clear(); qlen.clear(); toff.clear(); tlen.clear(); rev.clear(); kind.clear(); out_off.clear(); plan_m.clear(); plan_n.clear(); bound.clear(); tail_ops.clear(); }
  size_t add(uint32_t qo, uint32_t ql, uint32_t to, uint32_t tl, bool r, int kd, uint64_t oo, uint32_t pm, uint32_t pn, int32_t k) {
    qoff.push_back(qo); qlen.push_back(ql); toff.push_back(to); tlen.push_back(tl); rev.push_back(r); kind.push_back((uint8_t) kd); out_off.push_back(oo);
    plan_m.push_back(pm); plan_n.push_back(pn); bound.push_back(k);
    return qoff.size() - 1;
  }
  // device outputs
  uint32_t* d_out_len = nullptr;
  int32_t* d_corner = nullptr;
  int run(uint8_t* tmp_ops, int* colbuf);
};

// seg_kernel of each class, [0] without and [1] with equality tables, its template arguments read from SEG_GEOM
using SegKernel = void (*)(SegJobs);
template <bool EQ, bool PLAN, size_t... G>
constexpr std::array<SegKernel, SEG_NCLS> seg_kernels(std::index_sequence<G...>) {
  return {{nullptr, seg_kernel<SEG_GEOM[G + 1].C, (SEG_GEOM[G + 1].T > 32), EQ, PLAN>...}};
}
// [PLAN][eq]: the PLAN copies serve the asynchronous form
constexpr std::array<SegKernel, SEG_NCLS> SEG_KERNELS_P[2][2] = {
    {seg_kernels<false, false>(std::make_index_sequence<SEG_NCLS - 1>()), seg_kernels<true, false>(std::make_index_sequence<SEG_NCLS - 1>())},
    {seg_kernels<false, true>(std::make_index_sequence<SEG_NCLS - 1>()), seg_kernels<true, true>(std::make_index_sequence<SEG_NCLS - 1>())}};

// seg_band_kernel of each band class (G = edb_lanes), [0] without and [1] with equality tables
template <bool EQ, bool PLAN, size_t... C>
constexpr std::array<SegKernel, EDB_CLASSES> segb_kernels(std::index_sequence<C...>) {
  return {{seg_band_kernel<edb_lanes(C), EQ, PLAN>...}};
}
constexpr std::array<SegKernel, EDB_CLASSES> SEGB_KERNELS_P[2][2] = {
    {segb_kernels<false, false>(std::make_index_sequence<EDB_CLASSES>()), segb_kernels<true, false>(std::make_index_sequence<EDB_CLASSES>())},
    {segb_kernels<false, true>(std::make_index_sequence<EDB_CLASSES>()), segb_kernels<true, true>(std::make_index_sequence<EDB_CLASSES>())}};
// the segments wider than the wavefront classes, [PLAN][eq]
using SegHalfKernel = void (*)(SegJobs, size_t);
constexpr SegHalfKernel SEG_HALF_WIDE_KERNELS_P[2][2] = {{seg_half_wide_kernel<false>, seg_half_wide_kernel<true>},
                                                         {seg_half_wide_kernel<false, true>, seg_half_wide_kernel<true, true>}};
constexpr SegKernel SEG_LEAF_WIDE_KERNELS_P[2][2] = {{seg_leaf_wide_kernel<false>, seg_leaf_wide_kernel<true>},
                                                     {seg_leaf_wide_kernel<false, true>, seg_leaf_wide_kernel<true, true>}};

// narrowest band class that holds the segment's rows and certifies the optimum `k` of the problem (pm x pn) it belongs to; -1: none
__host__ __device__ inline int seg_band_class(uint32_t m, uint32_t pm, uint32_t pn, int32_t k) {
  if (k < 0) return -1;
  const int nblk = (int) ((m + 63) >> 6);
  for (int c = 0; c < EDB_CLASSES; ++c) {
    if (nblk > edb_block_cap(c)) continue;
    if (band_plan(edb_lanes(c), (int) pm, (int) pn).kvalid >= k) return c;
  }
  return -1;
}

// The dynamic shared memory each seg_kernel class may opt in to ([class], class 0 unused): the device's per-block maximum less the kernel's
// static shared memory, asked once per context.
const size_t* seg_rooms(dgpu_ctx* ctx, bool eq) {
  if (ctx->seg_room.empty()) {
    ctx->seg_room.assign(2 * SEG_NCLS, 0);
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device);
    for (int e = 0; e < 2; ++e)
      for (int c = 1; c < SEG_NCLS; ++c) {
        cudaFuncAttributes fa{};
        cudaFuncGetAttributes(&fa, (const void*) SEG_KERNELS_P[0][e][c]);
        ctx->seg_room[e * SEG_NCLS + c] = (size_t) optin - fa.sharedSizeBytes;
      }
  }
  return ctx->seg_room.data() + (eq ? SEG_NCLS : 0);
}

// Whether seg_kernel cannot stage m query rows in shared memory: the launch's opt-in of (m + 15) & ~15 dynamic bytes would exceed the
// device's per-block maximum less the kernel's static shared memory (`room`), and the whole call would fail. Such half columns (Hirschberg
// over a query of more than ~230 kb) run on seg_half_wide_kernel instead; every segment seg_kernel can launch still runs there.
__host__ __device__ inline bool seg_rows_exceed(uint32_t m, size_t room) {
  const size_t smem = ((size_t) m + 15) & ~(size_t) 15;
  return smem > 48 * 1024 && smem > room;
}

// The kernel a segment runs on: a band class that certifies its optimum (0 .. EDB_CLASSES - 1), else the wavefront class c of its width
// (EPK_SEG + c) unless a half column's rows do not fit its shared memory, else seg_half_wide_kernel (EPK_HALF) or seg_leaf_wide_kernel
// (EPK_LEAF); -1: a leaf of more than two row blocks and more than 16384 columns, which Hirschberg's split rule never leaves.
constexpr int EPK_HALF = EDB_CLASSES, EPK_LEAF = EDB_CLASSES + 1, EPK_SEG = EDB_CLASSES + 1, EPK_N = EPK_SEG + SEG_NCLS;
__host__ __device__ inline int seg_kind(uint32_t qlen, uint32_t tlen, int kind, uint32_t pm, uint32_t pn, int32_t bound, bool no_band,
                                        const size_t* room) {
  const int bc = no_band ? -1 : seg_band_class(qlen, pm, pn, bound);
  if (bc >= 0) return bc;
  const int c = seg_class(tlen);
  if (c > 0 && !(kind == 1 && seg_rows_exceed(qlen, room[c]))) return EPK_SEG + c;
  if (kind == 1) return EPK_HALF;
  return qlen > 64 * EPL_G ? -1 : EPK_LEAF;
}
// whether kind k writes a traced leaf's ops from the end of its slot (seg_band_kernel, seg_leaf_wide_kernel)
__host__ __device__ inline bool seg_kind_tail(int k) { return k < EDB_CLASSES || k == EPK_LEAF; }

// The largest extents the jobs of one kind can have (0 where its jobs need none: half columns store no trace and no directions): a traced
// leaf's columns (band classes), a leaf's trace cells of one uint4 per row block and column (seg_leaf_wide_kernel), a half column's width
// (seg_half_wide_kernel), a leaf's direction words, the rows staged in shared memory and m + n (seg_kernel).
struct SegExtent { size_t cols, cells, half, words, rows, mn; };

// Launch geometry of kind `id`: a CTA takes `per_cta` jobs, each with `stride` bytes of workspace in `slot` (a wide half column's scratch
// row, a leaf's trace storage, a seg_kernel job's directions and, from off_trace on, its trace); the grid is at most per_sm CTAs per SM.
struct SegKindGeom {
  size_t per_cta; int per_sm, slot; size_t stride, off_trace; unsigned threads; size_t smem;
  SegKernel k; SegHalfKernel half;   // seg_half_wide_kernel (half) takes the stride as its row stride
  const char* name;
};
SegKindGeom seg_kind_geom(int id, bool eq, bool plan, SegExtent const& x) {
  auto al = [](size_t v) { return (v + 255) & ~(size_t) 255; };
  if (id < EDB_CLASSES) {   // a leaf's trace storage: one uint4 per lane and step
    const int G = edb_lanes(id);
    const size_t steps = x.cols ? 65 * ((x.cols - 1) >> 6) + ((x.cols - 1) & 63) + G : 0;
    return {(size_t) (32 / G) * SEGB_WARPS, 8, SLOT_WAVEFRONT, steps * G * sizeof(uint4), 0, SEGB_WARPS * 32, 0, SEGB_KERNELS_P[plan][eq][id], nullptr,
            "seg_band_kernel"};
  }
  if (id == EPK_HALF)   // one warp per half column, a scratch row of n bytes per warp
    return {EPW_WARPS, 4, SLOT_EP_HROW, al(x.half), 0, EPW_WARPS * 32, 0, nullptr, SEG_HALF_WIDE_KERNELS_P[plan][eq], "seg_half_wide_kernel"};
  if (id == EPK_LEAF)
    return {(size_t) (32 / EPL_G) * EPL_WARPS, 8, SLOT_WAVEFRONT, x.cells * sizeof(uint4), 0, EPL_WARPS * 32, 0, SEG_LEAF_WIDE_KERNELS_P[plan][eq], nullptr,
            "seg_leaf_wide_kernel"};
  const SegGeom& g = SEG_GEOM[id - EPK_SEG];
  const size_t off_trace = al(x.words * 4 + 1024);
  return {1, g.per_sm, SLOT_WAVEFRONT, off_trace + al(x.mn + 64), off_trace, (unsigned) g.T, (x.rows + 15) & ~(size_t) 15,
          SEG_KERNELS_P[plan][eq][id - EPK_SEG], nullptr, "seg_kernel"};
}

// The grid of kind k: at most `ctas` CTAs and per_sm per SM, cut to the CTAs whose workspace `avail` bytes of its slot hold (at least one).
size_t seg_grid(const dgpu_ctx* ctx, SegKindGeom const& k, size_t ctas, size_t avail) {
  size_t grid = std::min(ctas, (size_t) ctx->num_sms * k.per_sm);
  const size_t per_block = k.per_cta * k.stride;
  if (per_block) grid = std::max<size_t>(1, std::min(grid, avail / per_block));
  return grid;
}

// Kind k on st over `list`, with seg_grid's grid and its workspace reserved: `count` jobs, or the PLAN copies the count the plan wrote at
// plan_count.
int seg_launch(dgpu_ctx* ctx, cudaStream_t st, SegJobs a, SegKindGeom const& k, size_t ctas, size_t avail, const uint32_t* list, uint32_t count,
               const uint32_t* plan_count) {
  int rc;
  const size_t grid = seg_grid(ctx, k, ctas, avail);
  void* w;   // at least 256 bytes: a band class of half columns alone stores no trace (the other kinds always take more)
  if ((rc = dgpu_reserve(ctx, k.slot, std::max<size_t>(grid * k.per_cta * k.stride, 256), &w))) return rc;
  a.work = (uint8_t*) w;
  a.list = list;
  a.count = count;
  a.plan_count = plan_count;
  a.work_stride = k.stride;
  a.off_trace = k.off_trace;
  if (!k.half && (rc = dgpu_smem_optin(ctx, k.k, k.smem, "cudaFuncSetAttribute(seg_kernel)"))) return rc;
  if (k.half) k.half<<<(unsigned) grid, k.threads, 0, st>>>(a, k.stride);
  else k.k<<<(unsigned) grid, k.threads, k.smem, st>>>(a);
  DGPU_LAUNCH_CHECK(ctx, k.name);
  return DGPU_OK;
}

// development switch: no band classes (wavefront and wide kernels only)
inline bool ep_no_band() {
  static const bool no_band = getenv("DGPU_EP_NO_BAND") != nullptr;
  return no_band;
}

int SegRunner::run(uint8_t* tmp_ops, int* colbuf) {
  const size_t N = qoff.size();
  if (!N) return DGPU_OK;
  int rc;
  // upload job arrays (one packed scratch buffer)
  const size_t bytes = N * (6 * 4 + 2 + 8 + 4 + 4) + 64 * 16;
  void* p;
  if ((rc = dgpu_reserve(ctx, SLOT_MSA_SEGJOBS, bytes + N * 4, &p))) return rc;
  uint8_t* base = (uint8_t*) p;
  auto carve = [&](size_t nbytes) { uint8_t* r = base; base += (nbytes + 15) & ~(size_t) 15; return r; };
  uint32_t* d_qoff = (uint32_t*) carve(N * 4); uint32_t* d_qlen = (uint32_t*) carve(N * 4);
  uint32_t* d_toff = (uint32_t*) carve(N * 4); uint32_t* d_tlen = (uint32_t*) carve(N * 4);
  uint64_t* d_oo = (uint64_t*) carve(N * 8);
  uint8_t* d_rev = carve(N); uint8_t* d_kind = carve(N);
  d_out_len = (uint32_t*) carve(N * 4); d_corner = (int32_t*) carve(N * 4);
  uint32_t* d_list = (uint32_t*) carve(N * 4);
  uint32_t* d_pm = (uint32_t*) carve(N * 4); uint32_t* d_pn = (uint32_t*) carve(N * 4);
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_pm, plan_m.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_pn, plan_n.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_qoff, qoff.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_qlen, qlen.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_toff, toff.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_tlen, tlen.data(), N * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_oo, out_off.data(), N * 8, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_rev, rev.data(), N, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_kind, kind.data(), N, cudaMemcpyHostToDevice, st));
  // the jobs of each kind (seg_kind), listed back to back in d_list in kind order
  std::vector<std::vector<uint32_t> > lists(EPK_N);
  tail_ops.assign(N, 0);
  const bool no_band = ep_no_band();
  const size_t* room = seg_rooms(ctx, use_eq);
  for (size_t i = 0; i < N; ++i) {
    const int kd = seg_kind(qlen[i], tlen[i], kind[i], plan_m[i], plan_n[i], bound[i], no_band, room);
    if (kd < 0) return DGPU_ERR_UNSUPPORTED;
    lists[kd].push_back((uint32_t) i);
    tail_ops[i] = seg_kind_tail(kd);
  }
  std::vector<uint32_t> flat;
  for (std::vector<uint32_t> const& L : lists) flat.insert(flat.end(), L.begin(), L.end());
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_list, flat.data(), flat.size() * 4, cudaMemcpyHostToDevice, st));
  SegJobs a;
  a.seqs = seqs; a.q_off = d_qoff; a.q_len = d_qlen; a.t_off = d_toff; a.t_len = d_tlen; a.rev = d_rev; a.kind = d_kind; a.out_off = d_oo;
  a.out_len = d_out_len; a.corner = d_corner; a.tmp_ops = tmp_ops; a.colbuf = colbuf; a.eq = eq;
  a.plan_m = d_pm; a.plan_n = d_pn; a.eq_cls = eq_cls;
  // One launch per non-empty kind, in turn on st: band classes G = 2 .. 32, wide half columns, wide leaves, seg_kernel classes; the geometry
  // of the largest extents its jobs have, the grid shrunk to the workspace budget.
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  size_t lo = 0;
  for (int id = 0; id < EPK_N; lo += lists[id].size(), ++id) {
    std::vector<uint32_t> const& L = lists[id];
    if (L.empty()) continue;
    SegExtent x{};
    for (uint32_t i : L) {
      if (kind[i] == 0) {   // leaves
        x.cols = std::max<size_t>(x.cols, tlen[i]);
        x.cells = std::max<size_t>(x.cells, (size_t) tlen[i] * ((qlen[i] + 63) >> 6));
        if (id > EPK_SEG) x.words = std::max(x.words, (size_t) (qlen[i] + 1) * seg_dstride(tlen[i], SEG_GEOM[id - EPK_SEG].C));
      }
      x.half = std::max<size_t>(x.half, tlen[i]);
      x.rows = std::max<size_t>(x.rows, qlen[i]);
      x.mn = std::max<size_t>(x.mn, (size_t) qlen[i] + tlen[i]);
    }
    const SegKindGeom k = seg_kind_geom(id, use_eq, false, x);
    if ((rc = seg_launch(ctx, st, a, k, (L.size() + k.per_cta - 1) / k.per_cta, dgpu_workspace_budget(ctx, k.slot, free_b), d_list + lo,
                         (uint32_t) L.size(), nullptr)))
      return rc;
  }
  return DGPU_OK;
}

__host__ __device__ inline bool seg_needs_split(uint32_t m, uint32_t n) {  // src/edlib.cpp:1189-1191
  const long long est = 20ll * ((m + 63) / 64) * n + 8ll * n;
  return est >= 1024 * 1024;
}

// Bytes of one run of the HW start-pass mirror. The mirror holds a private copy of every job's query and target, so jobs that share a
// sequence (many reads against one window) need more than the arena; runs bound that and keep offsets 32-bit.
constexpr uint64_t EP_MIRROR_RUN = 1ull << 30;

int check_max_slice(dgpu_ctx* ctx, uint32_t max_slice) {
  if (max_slice >= 1 && max_slice <= DGPU_EP_MAX_SLICE) return DGPU_OK;
  if (ctx) ctx->last_error = "dgpu_edit_path_wide: max_slice must be 1 .. " + std::to_string(DGPU_EP_MAX_SLICE);
  return DGPU_ERR_ARG;
}

// Distance and first end location of every job, then its start location (HW: a reversed SHW pass per mirror run); host copies of all three.
int ep_locate(dgpu_ctx* ctx, cudaStream_t st, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* q_off, const uint32_t* q_len,
              const uint32_t* t_off, const uint32_t* t_len, int mode, const uint32_t* d_eqtabs, uint64_t n, std::vector<uint32_t> const& h_qlen,
              std::vector<uint32_t> const& h_tlen, int32_t* dist, int32_t* start_loc, int32_t* end_loc, std::vector<int32_t>& h_dist,
              std::vector<int32_t>& h_start, std::vector<int32_t>& h_end) {
  int rc;
  const uint32_t nb = (uint32_t) ((n + 255) / 256);
  // 1. distance + first end location (k = -1 at every PATH call site of the reference); generalised equalities ride along as tables
  if ((rc = dgpu_edit_distance_impl(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, nullptr, mode, n, dist, end_loc, st, 0, d_eqtabs,
                                    ctx->async_bound))) return rc;
  void* d_rev = nullptr;
  // mirror layout of the HW start pass: job i's reversed query at mq[i], its reversed target right after it, jobs back to back in runs
  // of at most EP_MIRROR_RUN bytes; each run is mirrored and searched in one SHW pass (offsets relative to the run)
  std::vector<uint32_t> h_moff;
  std::vector<uint64_t> run_lo, run_bytes;
  if (mode == DGPU_MODE_HW) {
    h_moff.resize(2 * n);
    uint64_t pos = 0;
    for (uint64_t i = 0; i < n; ++i) {
      const uint64_t need = (uint64_t) h_qlen[i] + h_tlen[i];
      if (need > EP_MIRROR_RUN) { ctx->last_error = "dgpu_edit_path: a HW job's query and target exceed the start-pass mirror"; return DGPU_ERR_CAPACITY; }
      if (i == 0 || pos + need > EP_MIRROR_RUN) {
        if (i) run_bytes.push_back(pos);
        run_lo.push_back(i);
        pos = 0;
      }
      h_moff[i] = (uint32_t) pos; h_moff[n + i] = (uint32_t) (pos + h_qlen[i]);
      pos += need;
    }
    run_bytes.push_back(pos);
    run_lo.push_back(n);
    const uint64_t run_max = *std::max_element(run_bytes.begin(), run_bytes.end());
    // 2. start location: reversed query vs reversed target prefix, SHW, k = distance, LAST optimal end
    void *d_mirror, *d_t2off, *d_t2len, *d_k2;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_MIRROR, run_max + 64, &d_mirror))) return rc;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_TABLE, n * 12, &d_t2off))) return rc;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_COLS, n * 4, &d_t2len))) return rc;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_BOUNDS, n * 8, &d_k2))) return rc;
    d_rev = (uint8_t*) d_k2 + n * 4;
    uint32_t* d_mq = (uint32_t*) d_t2off + n;
    uint32_t* d_mt = d_mq + n;
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_mq, h_moff.data(), 2 * n * 4, cudaMemcpyHostToDevice, st));
    ep_hwstart_jobs_kernel<<<nb, 256, 0, st>>>(d_mt, t_len, dist, end_loc, (uint32_t) n, (uint32_t*) d_t2off, (uint32_t*) d_t2len, (int32_t*) d_k2);
    DGPU_LAUNCH_CHECK(ctx, "ep_hwstart_jobs");
    for (size_t r = 0; r + 1 < run_lo.size(); ++r) {   // a run reuses the mirror after the previous run's pass on the same stream
      const uint64_t j0 = run_lo[r], cnt = run_lo[r + 1] - j0;
      const uint32_t wb = (uint32_t) ((cnt * 32 + 255) / 256);
      ep_mirror_kernel<<<wb, 256, 0, st>>>(seqs, (uint8_t*) d_mirror, q_off + j0, q_len + j0, d_mq + j0, (uint32_t) cnt);
      DGPU_LAUNCH_CHECK(ctx, "ep_mirror(q)");
      ep_mirror_kernel<<<wb, 256, 0, st>>>(seqs, (uint8_t*) d_mirror, t_off + j0, t_len + j0, d_mt + j0, (uint32_t) cnt);
      DGPU_LAUNCH_CHECK(ctx, "ep_mirror(t)");
      if ((rc = dgpu_edit_distance_impl(ctx, (const uint8_t*) d_mirror, run_bytes[r], d_mq + j0, q_len + j0, (const uint32_t*) d_t2off + j0,
                                        (const uint32_t*) d_t2len + j0, (const int32_t*) d_k2 + j0, DGPU_MODE_SHW, cnt, start_loc + j0,
                                        (int32_t*) d_rev + j0, st, 1, d_eqtabs, ctx->async_bound))) return rc;
    }
  }
  ep_start_kernel<<<nb, 256, 0, st>>>(mode, q_len, t_len, dist, end_loc, (const int32_t*) d_rev, (uint32_t) n, start_loc);
  DGPU_LAUNCH_CHECK(ctx, "ep_start");
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_dist.data(), dist, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_start.data(), start_loc, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_end.data(), end_loc, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  return DGPU_OK;
}

// Hirschberg splitting of every job's aligned slice, level by level, until each segment is a leaf (status 2: slice wider than max_slice).
int ep_split(dgpu_ctx* ctx, cudaStream_t st, SegRunner& R, uint64_t n, std::vector<uint32_t> const& h_qoff, std::vector<uint32_t> const& h_qlen,
             std::vector<uint32_t> const& h_toff, std::vector<uint32_t> const& h_tlen, std::vector<int32_t> const& h_dist, std::vector<int32_t> const& h_start,
             std::vector<int32_t> const& h_end, uint32_t max_slice, std::vector<std::vector<Seg> >& perjob, std::vector<uint32_t>& h_status) {
  int rc;
  bool any_split = false;
  for (uint64_t i = 0; i < n; ++i) {
    if (h_qlen[i] == 0 || h_tlen[i] == 0 || h_dist[i] < 0) continue;  // no path at all (edlib returns early)
    const int s = h_start[i], e = h_end[i];
    Seg sg; sg.job = (uint32_t) i; sg.qoff = h_qoff[i]; sg.qlen = h_qlen[i]; sg.toff = h_toff[i] + (uint32_t) s; sg.tlen = (uint32_t) (e - s + 1); sg.score = h_dist[i];
    if (sg.tlen > max_slice) { h_status[i] = 2; continue; }
    perjob[i].push_back(sg);
    if (sg.qlen && sg.tlen && seg_needs_split(sg.qlen, sg.tlen)) any_split = true;
  }
  while (any_split) {
    any_split = false;
    // collect the segments to split
    struct Ref { uint32_t job, idx; };
    std::vector<Ref> todo;
    R.clear();
    std::vector<uint64_t> f_off, b_off;
    std::vector<uint32_t> sm_, sh_, sn_;
    std::vector<int32_t> sbest;
    uint64_t colpos = 0;
    for (uint64_t i = 0; i < n; ++i)
      for (uint32_t k = 0; k < perjob[i].size(); ++k) {
        Seg const& g = perjob[i][k];
        if (!(g.qlen && g.tlen && seg_needs_split(g.qlen, g.tlen))) continue;
        const uint32_t h = g.tlen / 2;
        todo.push_back(Ref{(uint32_t) i, k});
        f_off.push_back(colpos); R.add(g.qoff, g.qlen, g.toff, h, false, 1, colpos, g.qlen, g.tlen, g.score); colpos += g.qlen + 1;
        b_off.push_back(colpos); R.add(g.qoff, g.qlen, g.toff + h, g.tlen - h, true, 1, colpos, g.qlen, g.tlen, g.score); colpos += g.qlen + 1;
        sm_.push_back(g.qlen); sh_.push_back(h); sn_.push_back(g.tlen); sbest.push_back(g.score);
      }
    if (todo.empty()) break;
    void* d_col;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_COLS, (colpos + 16) * sizeof(int), &d_col))) return rc;
    if ((rc = R.run(nullptr, (int*) d_col))) return rc;
    const size_t S = todo.size();
    void* d_sel;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_TABLE, S * (8 + 8 + 4 + 4 + 4 + 4 + 12) + 256, &d_sel))) return rc;
    uint8_t* bp = (uint8_t*) d_sel;
    uint64_t* d_foff = (uint64_t*) bp; bp += S * 8;
    uint64_t* d_boff = (uint64_t*) bp; bp += S * 8;
    uint32_t* d_m = (uint32_t*) bp; bp += S * 4;
    uint32_t* d_h = (uint32_t*) bp; bp += S * 4;
    uint32_t* d_n = (uint32_t*) bp; bp += S * 4;
    int32_t* d_best = (int32_t*) bp; bp += S * 4;
    int32_t* d_out3 = (int32_t*) bp;
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_foff, f_off.data(), S * 8, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_boff, b_off.data(), S * 8, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_m, sm_.data(), S * 4, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_h, sh_.data(), S * 4, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_n, sn_.data(), S * 4, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_best, sbest.data(), S * 4, cudaMemcpyHostToDevice, st));
    hb_select_kernel<<<(unsigned) ((S * 32 + 255) / 256), 256, 0, st>>>((const int*) d_col, d_foff, d_boff, d_m, d_h, d_n, d_best, (uint32_t) S, nullptr,
                                                                        d_out3);
    DGPU_LAUNCH_CHECK(ctx, "hb_select");
    std::vector<int32_t> out3(3 * S);
    DGPU_CUDA(ctx, cudaMemcpyAsync(out3.data(), d_out3, S * 12, cudaMemcpyDeviceToHost, st));
    DGPU_CUDA(ctx, cudaStreamSynchronize(st));
    // replace every split segment by its two children (processed back to front so indices stay valid)
    for (size_t t = S; t-- > 0;) {
      std::vector<Seg>& v = perjob[todo[t].job];
      const Seg g = v[todo[t].idx];
      const int i = out3[3 * t];
      if (i < 0) { h_status[g.job] = 3; v.clear(); continue; }  // no split row reproduces the optimum: internal error
      const uint32_t h = g.tlen / 2;
      Seg ul = g, lr = g;
      ul.qlen = (uint32_t) i; ul.tlen = h; ul.score = out3[3 * t + 1];
      lr.qoff = g.qoff + (uint32_t) i; lr.qlen = g.qlen - (uint32_t) i; lr.toff = g.toff + h; lr.tlen = g.tlen - h; lr.score = out3[3 * t + 2];
      v[todo[t].idx] = ul;
      v.insert(v.begin() + todo[t].idx + 1, lr);
    }
    for (uint64_t i = 0; i < n && !any_split; ++i)
      for (Seg const& g : perjob[i])
        if (g.qlen && g.tlen && seg_needs_split(g.qlen, g.tlen)) { any_split = true; break; }
  }
  return DGPU_OK;
}

// Traceback (or trivial run) of every leaf, the check that it reproduces its distance, the concatenation per job into ops, then status.
int ep_leaves(dgpu_ctx* ctx, cudaStream_t st, SegRunner& R, uint64_t n, std::vector<std::vector<Seg> > const& perjob, std::vector<uint32_t>& h_status,
              uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status) {
  int rc;
  R.clear();
  std::vector<uint32_t> job_lo(n + 1, 0), leaf_kind, leaf_len_h;
  std::vector<uint64_t> leaf_off;
  std::vector<size_t> leaf_slot;
  uint64_t tmp_bytes = 0;
  for (uint64_t i = 0; i < n; ++i) {
    job_lo[i] = (uint32_t) leaf_kind.size();
    if (h_status[i]) continue;
    for (Seg const& g : perjob[i]) {
      if (g.qlen == 0 || g.tlen == 0) {  // src/edlib.cpp:1169-1176
        leaf_kind.push_back(g.qlen == 0 ? 2u : 1u); leaf_len_h.push_back(g.qlen + g.tlen); leaf_off.push_back(0); leaf_slot.push_back((size_t) -1);
      } else {
        leaf_kind.push_back(0u); leaf_len_h.push_back(0); leaf_off.push_back(tmp_bytes);
        leaf_slot.push_back(R.add(g.qoff, g.qlen, g.toff, g.tlen, false, 0, tmp_bytes, g.qlen, g.tlen, g.score));
        tmp_bytes += g.qlen + g.tlen;
      }
    }
  }
  job_lo[n] = (uint32_t) leaf_kind.size();
  void* d_tmp;
  if ((rc = dgpu_reserve(ctx, SLOT_EP_MIRROR, tmp_bytes + 64, &d_tmp))) return rc;
  dgpu_prof_begin(ctx, st);
  if ((rc = R.run((uint8_t*) d_tmp, nullptr))) return rc;
  dgpu_prof_end(ctx, st);
  const size_t NL = leaf_kind.size();
  std::vector<uint32_t> traced_len(R.qoff.size());
  std::vector<int32_t> traced_corner(R.qoff.size());
  if (!traced_len.empty()) {
    DGPU_CUDA(ctx, cudaMemcpyAsync(traced_len.data(), R.d_out_len, traced_len.size() * 4, cudaMemcpyDeviceToHost, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(traced_corner.data(), R.d_corner, traced_len.size() * 4, cudaMemcpyDeviceToHost, st));
    DGPU_CUDA(ctx, cudaStreamSynchronize(st));
  }
  {
    // consistency: every traced leaf must reproduce the distance Hirschberg assigned to it
    size_t li = 0;
    for (uint64_t i = 0; i < n; ++i) {
      if (h_status[i]) continue;
      for (Seg const& g : perjob[i]) {
        if (leaf_slot[li] != (size_t) -1) {
          leaf_len_h[li] = traced_len[leaf_slot[li]];
          if (-traced_corner[leaf_slot[li]] != g.score) h_status[i] = 3;
          else if (R.tail_ops[leaf_slot[li]]) leaf_off[li] += (uint64_t) g.qlen + g.tlen - traced_len[leaf_slot[li]];   // seg_band_kernel / seg_leaf_wide_kernel write from the end of the slot
        }
        ++li;
      }
    }
  }
  void* d_leaf;
  if ((rc = dgpu_reserve(ctx, SLOT_EP_TABLE, (n + 1) * 4 + NL * 16 + 256, &d_leaf))) return rc;
  uint8_t* lp = (uint8_t*) d_leaf;
  uint64_t* d_loff = (uint64_t*) lp; lp += NL * 8;
  uint32_t* d_lo = (uint32_t*) lp; lp += (n + 1) * 4;
  uint32_t* d_lkind = (uint32_t*) lp; lp += NL * 4;
  uint32_t* d_llen = (uint32_t*) lp;
  if (NL) {
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_loff, leaf_off.data(), NL * 8, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_lkind, leaf_kind.data(), NL * 4, cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_llen, leaf_len_h.data(), NL * 4, cudaMemcpyHostToDevice, st));
  }
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_lo, job_lo.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st));
  hb_concat_kernel<<<(unsigned) ((n * 32 + 255) / 256), 256, 0, st>>>((const uint8_t*) d_tmp, d_lo, d_lkind, d_loff, d_llen, (uint32_t) n, ops, ops_off, ops_len);
  DGPU_LAUNCH_CHECK(ctx, "hb_concat");
  DGPU_CUDA(ctx, cudaMemcpyAsync(status, h_status.data(), n * 4, cudaMemcpyHostToDevice, st));
  DGPU_CUDA(ctx, cudaStreamSynchronize(st));  // host vectors above are copy sources
  return DGPU_OK;
}

// ---- asynchronous form (dgpu_set_ep_async_bound) --------------------------------------------------------------------------------------
// Under a bound (max_query x max_target) the device form reads nothing back. Everything ep_locate / ep_split / ep_leaves decide on the host
// from copied-back values is decided here by kernels, in arrays whose sizes follow from n and the bound alone:
//   * a job's segments live in slots j << l .. (j << l) + cnt[j] - 1 at level l (a level at most doubles them), so no segment list is
//     compacted across jobs; the number of levels is the largest any admitted slice can need (ep_bound_levels);
//   * ep_plan_kernel (one CTA) compacts the segments that still need a split, in job order, into hb_select_kernel's inputs and two half
//     columns each, and appends every half column to the list of the kernel that runs it (seg_kind), in that order;
//   * the half columns of a job's segment k start at 2 ((qoff_k - q_off[j]) + k) in the job's colbuf region, a traced leaf's ops at
//     (qoff_k - q_off[j]) + (toff_k - t_off[j]) in its tmp-ops region: the segments of a job partition its query and its slice in order;
//   * every kind the bound can reach at a level is launched with the grid of the bound (the PLAN copies read their job count from the plan,
//     and CTAs beyond it find no work).
// job status while planning: 0, 2 (slice wider than max_slice), 3 (no split row / leaf distance reproduces the optimum), 4 (refused)
struct EpBound {
  uint32_t mq, mt;   // the bound
  uint32_t w;        // widest slice a call traces: min(max_target, max_slice)
  int levels;        // Hirschberg levels any admitted slice can need
};

// the number of Hirschberg levels after which no segment of at most mq rows and w columns needs a split
inline int ep_bound_levels(uint32_t mq, uint32_t w) {
  int l = 0;
  while (seg_needs_split(mq, (uint32_t) ((w + (1ull << l) - 1) >> l))) ++l;
  return l;
}
// the widest segment of nblk row blocks that needs no split
inline uint32_t leaf_nmax(uint32_t nblk) { return (uint32_t) ((1024u * 1024u - 1) / (20u * nblk + 8)); }

// Launch geometry (PLAN copies) of kind `id` under a bound: the largest extents any segment of that kind can have, for half columns or for
// leaves.
SegKindGeom bound_kind(int id, bool leaves, bool eq, uint32_t mq, uint32_t w, const size_t* room) {
  SegExtent x{};
  if (id < EDB_CLASSES) x.cols = leaves ? std::min(w, leaf_nmax(1)) : 0;
  else if (id == EPK_HALF) x.half = (w + 1) / 2;
  else if (id == EPK_LEAF) x.cells = std::max<size_t>(std::min(w, leaf_nmax(1)), 2 * (size_t) std::min(w, leaf_nmax(2)));
  else {
    const int c = id - EPK_SEG;
    const SegGeom& g = SEG_GEOM[c];
    const uint32_t N = std::min(g.cap, w);
    for (uint32_t nb = 1; leaves && nb <= (mq + 63) / 64; ++nb)   // a leaf's rows and columns are bounded by mq, N and the split rule
      x.words = std::max(x.words, (size_t) (std::min(mq, 64 * nb) + 1) * seg_dstride(std::min(N, leaf_nmax(nb)), g.C));
    x.rows = seg_rows_exceed(mq, room[c]) ? room[c] & ~(size_t) 15 : mq;   // the most rows a segment of this class stages
    x.mn = (size_t) mq + N;
  }
  return seg_kind_geom(id, eq, true, x);
}

// The kinds the segments of a level (leaves: the leaves) can reach under the bound.
std::vector<int> bound_kinds(EpBound const& b, int level, bool leaves, const size_t* room) {
  std::vector<int> ids;
  if (!ep_no_band())
    for (int bc = 0; bc < EDB_CLASSES; ++bc) ids.push_back(bc);
  uint32_t lo = 0, hi;   // widths of the segments
  if (leaves) hi = std::min(b.w, leaf_nmax(1));
  else {
    uint32_t nmin = 1;   // narrowest segment of at most mq rows that needs a split; its half columns are at least half as wide
    while (!seg_needs_split(b.mq, nmin)) ++nmin;
    lo = nmin / 2;
    hi = (uint32_t) ((b.w + (2ull << level) - 1) >> (level + 1));
  }
  bool wide = hi > SEG_GEOM[SEG_NCLS - 1].cap;
  for (int c = 1; c < SEG_NCLS; ++c)
    if (SEG_GEOM[c].cap >= lo && SEG_GEOM[c - 1].cap < hi) {
      ids.push_back(EPK_SEG + c);
      if (!leaves && seg_rows_exceed(b.mq, room[c])) wide = true;
    }
  if (wide) ids.push_back(leaves ? EPK_LEAF : EPK_HALF);
  return ids;
}

struct EpPlan {
  uint64_t n;
  const uint32_t *q_off, *q_len, *t_off, *t_len;   // q_len / t_len: 0 for a refused job
  uint32_t* jst;                                    // job status
  // segments of the level (in) and of the next one (out), slot (j << shift) + k
  uint32_t shift;
  const uint32_t* cnt; const uint32_t *sq, *sql, *st, *stl; const int32_t* ssc;
  uint32_t* cnt2; uint32_t *oq, *oql, *ot, *otl; int32_t* osc;
  uint32_t* pre;                                    // splits before each slot, in job order (n << shift) + 1
  // the jobs of the class kernels (half columns or leaves) and their per-kind lists
  uint32_t *jq, *jql, *jt, *jtl, *jpm, *jpn; int32_t* jbound; uint8_t *jrev, *jkind, *jtail; uint64_t* joff;
  uint32_t* out_len; int32_t* corner;
  uint32_t* lists; uint64_t list_cap; uint32_t* counts;   // counts[EPK_N]: the splits of the level
  // hb_select_kernel's inputs and outputs
  uint64_t *f_off, *b_off; uint32_t *sm, *sh, *sn; int32_t *sbest, *out3;
  uint64_t col_stride, tmp_stride;   // ints of colbuf, bytes of tmp ops per job
  // leaves
  uint32_t* leaf_lo; uint32_t* leaf_kind; uint64_t* leaf_off; uint32_t* leaf_len;
  size_t room[SEG_NCLS]; bool no_band;
};

constexpr int EPP_THREADS = 1024;
struct EpPlanShared { uint32_t scan[32], wc[32][EPK_N], run[EPK_N]; };

// exclusive prefix of v over the CTA (EPP_THREADS threads); total: the sum
__device__ uint32_t cta_exscan(uint32_t v, EpPlanShared& sh, uint32_t& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) sh.scan[w] = x;
  __syncthreads();
  if (w == 0) {
    uint32_t s = sh.scan[lane];
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    sh.scan[lane] = s;
  }
  __syncthreads();
  const uint32_t ex = x - v + (w ? sh.scan[w - 1] : 0);
  total = sh.scan[31];
  __syncthreads();
  return ex;
}

// appends item `it` to the list of kind k (-1: none), in thread order; every thread of the CTA calls it
__device__ void plan_append(EpPlan const& p, EpPlanShared& sh, int k, uint32_t it) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned peers = __match_any_sync(0xffffffffu, k);
  const uint32_t rank = __popc(peers & ((1u << lane) - 1));
  if (k >= 0 && rank == 0) sh.wc[w][k] = __popc(peers);
  __syncthreads();
  if (threadIdx.x < EPK_N) {
    uint32_t s = sh.run[threadIdx.x];
    for (int x = 0; x < 32; ++x) { const uint32_t c = sh.wc[x][threadIdx.x]; sh.wc[x][threadIdx.x] = s; s += c; }
    sh.run[threadIdx.x] = s;
  }
  __syncthreads();
  if (k >= 0) p.lists[k * p.list_cap + sh.wc[w][k] + rank] = it;
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * EPK_N; i += EPP_THREADS) (&sh.wc[0][0])[i] = 0;
  __syncthreads();
}

// One level of Hirschberg's recursion planned (leaves = false) or the leaves planned (leaves = true). One CTA.
template <bool LEAVES>
__global__ void __launch_bounds__(EPP_THREADS) ep_plan_kernel(EpPlan p) {
  __shared__ EpPlanShared sh;
  for (int i = threadIdx.x; i < 32 * EPK_N; i += EPP_THREADS) (&sh.wc[0][0])[i] = 0;
  if (threadIdx.x < EPK_N) sh.run[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t nslots = p.n << p.shift;
  const uint32_t kmask = (1u << p.shift) - 1;
  if (LEAVES) {
    // every slot gets a leaf entry (an unused one an empty run), so that hb_concat_kernel finds a job's leaves at j << shift
    for (uint64_t j = threadIdx.x; j <= p.n; j += EPP_THREADS) p.leaf_lo[j] = (uint32_t) (j << p.shift);
    for (uint64_t b = 0; b < nslots; b += EPP_THREADS) {
      const uint64_t i = b + threadIdx.x;
      int kd = -1;
      if (i < nslots) {
        const uint32_t j = (uint32_t) (i >> p.shift), k = (uint32_t) i & kmask;
        uint32_t lk = 1, len = 0;
        if (k < p.cnt[j] && !p.jst[j]) {
          const uint32_t m = p.sql[i], n = p.stl[i];
          if (m == 0 || n == 0) { lk = m == 0 ? 2 : 1; len = m + n; }   // src/edlib.cpp:1169-1176
          else {
            const int32_t sc = p.ssc[i];
            kd = seg_kind(m, n, 0, m, n, sc, p.no_band, p.room);
            if (kd > EPK_SEG && seg_rows_exceed(m, p.room[kd - EPK_SEG])) kd = -1;   // the synchronous form fails such a launch
            if (kd < 0) p.jst[j] = 3;   // Hirschberg's split rule leaves no such leaf
            else {
              lk = 0;
              const uint64_t off = j * p.tmp_stride + (p.sq[i] - p.q_off[j]) + (p.st[i] - p.t_off[j]);
              p.leaf_off[i] = off;
              p.jq[i] = p.sq[i]; p.jql[i] = m; p.jt[i] = p.st[i]; p.jtl[i] = n; p.jrev[i] = 0; p.jkind[i] = 0; p.joff[i] = off;
              p.jpm[i] = m; p.jpn[i] = n; p.jbound[i] = sc; p.jtail[i] = seg_kind_tail(kd);
            }
          }
        }
        p.leaf_kind[i] = lk;
        if (lk) { p.leaf_len[i] = len; p.leaf_off[i] = 0; }
      }
      plan_append(p, sh, kd, (uint32_t) i);
    }
  } else {
    // the segments that need a split, in job order: hb_select_kernel's inputs and the two half columns of each
    uint32_t nsplit = 0;
    for (uint64_t b = 0; b < nslots; b += EPP_THREADS) {
      const uint64_t i = b + threadIdx.x;
      uint32_t need = 0, j = 0, k = 0;
      if (i < nslots) {
        j = (uint32_t) (i >> p.shift); k = (uint32_t) i & kmask;
        if (k < p.cnt[j] && !p.jst[j]) { const uint32_t m = p.sql[i], n = p.stl[i]; need = m && n && seg_needs_split(m, n); }
      }
      uint32_t total;
      const uint32_t s = nsplit + cta_exscan(need, sh, total);
      if (i < nslots) p.pre[i] = s;
      if (need) {
        const uint32_t qo = p.sq[i], m = p.sql[i], to = p.st[i], n = p.stl[i], h = n / 2;
        const int32_t sc = p.ssc[i];
        const uint64_t f = j * p.col_stride + 2 * ((uint64_t) (qo - p.q_off[j]) + k), bo = f + m + 1;
        p.f_off[s] = f; p.b_off[s] = bo; p.sm[s] = m; p.sh[s] = h; p.sn[s] = n; p.sbest[s] = sc;
        for (int r = 0; r < 2; ++r) {
          const uint32_t x = 2 * s + r;
          p.jq[x] = qo; p.jql[x] = m; p.jt[x] = r ? to + h : to; p.jtl[x] = r ? n - h : h; p.jrev[x] = (uint8_t) r; p.jkind[x] = 1;
          p.joff[x] = r ? bo : f; p.jpm[x] = m; p.jpn[x] = n; p.jbound[x] = sc;
        }
      }
      nsplit += total;
    }
    if (threadIdx.x == 0) { p.pre[nslots] = nsplit; p.counts[EPK_N] = nsplit; }
    __syncthreads();
    for (uint32_t b = 0; b < 2 * nsplit; b += EPP_THREADS) {
      const uint32_t x = b + threadIdx.x;
      const int kd = x < 2 * nsplit ? seg_kind(p.jql[x], p.jtl[x], 1, p.jpm[x], p.jpn[x], p.jbound[x], p.no_band, p.room) : -1;
      plan_append(p, sh, kd, x);
    }
  }
  if (threadIdx.x < EPK_N) p.counts[threadIdx.x] = sh.run[threadIdx.x];
}

// every split segment replaced by its two children (hb_select_kernel's row and distances), the others copied: the next level's slots
__global__ void ep_split_kernel(EpPlan p) {
  const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (p.n << p.shift)) return;
  const uint32_t j = (uint32_t) (i >> p.shift), k = (uint32_t) i & ((1u << p.shift) - 1), cnt = p.cnt[j];
  if (k == 0 && cnt == 0) p.cnt2[j] = 0;
  if (k >= cnt) return;
  const uint32_t pre0 = p.pre[(uint64_t) j << p.shift], s = p.pre[i], split = p.pre[i + 1] - s;
  const uint64_t o = ((uint64_t) j << (p.shift + 1)) + k + (s - pre0);
  const uint32_t qo = p.sq[i], m = p.sql[i], to = p.st[i], n = p.stl[i];
  if (!split) { p.oq[o] = qo; p.oql[o] = m; p.ot[o] = to; p.otl[o] = n; p.osc[o] = p.ssc[i]; }
  else {
    const int32_t row = p.out3[3 * s];
    if (row < 0) p.jst[j] = 3;   // no split row reproduces the optimum: internal error
    else {
      const uint32_t h = n / 2, r = (uint32_t) row;
      p.oq[o] = qo; p.oql[o] = r; p.ot[o] = to; p.otl[o] = h; p.osc[o] = p.out3[3 * s + 1];
      p.oq[o + 1] = qo + r; p.oql[o + 1] = m - r; p.ot[o + 1] = to + h; p.otl[o + 1] = n - h; p.osc[o + 1] = p.out3[3 * s + 2];
    }
  }
  if (k == cnt - 1) p.cnt2[j] = cnt + (s + split - pre0);
}

// a traced leaf's length, the check that it reproduces the distance Hirschberg assigned to it, and the offset of ops written from the end
// of the slot (seg_band_kernel, seg_leaf_wide_kernel)
__global__ void ep_leaf_done_kernel(EpPlan p) {
  const uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (p.n << p.shift) || p.leaf_kind[i] != 0) return;
  const uint32_t L = p.out_len[i];
  if (-p.corner[i] != p.jbound[i]) p.jst[i >> p.shift] = 3;
  else if (p.jtail[i]) p.leaf_off[i] += (uint64_t) p.jql[i] + p.jtl[i] - L;
  p.leaf_len[i] = L;
}

// refusals, the lengths every later pass reads (0 for a refused job) and the HW start-pass mirror offsets: job j at (j % run_jobs) x
// (max_query + max_target) of its run
__global__ void ep_async_jobs_kernel(const uint32_t* q_len, const uint32_t* t_len, uint64_t n, uint32_t mq, uint32_t mt, uint32_t run_jobs,
                                     uint32_t* ql2, uint32_t* tl2, uint32_t* mq_off, uint32_t* mt_off, uint32_t* jst, unsigned long long* refused) {
  const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const bool out = q_len[j] > mq || t_len[j] > mt;
  if (out) atomicAdd(refused, 1ull);
  ql2[j] = out ? 0 : q_len[j];
  tl2[j] = out ? 0 : t_len[j];
  jst[j] = out ? 4 : 0;
  mq_off[j] = (uint32_t) (j % run_jobs) * (mq + mt);
  mt_off[j] = mq_off[j] + mq;
}

// level 0: each job's aligned slice as its one segment (ep_split's first loop)
__global__ void ep_seg_init_kernel(EpPlan p, const int32_t* dist, const int32_t* start_loc, const int32_t* end_loc, uint32_t max_slice) {
  const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= p.n) return;
  uint32_t c = 0;
  if (!p.jst[j] && p.q_len[j] && p.t_len[j] && dist[j] >= 0) {
    const int s = start_loc[j], e = end_loc[j];
    const uint32_t w = (uint32_t) (e - s + 1);
    if (w > max_slice) p.jst[j] = 2;
    else { p.oq[j] = p.q_off[j]; p.oql[j] = p.q_len[j]; p.ot[j] = p.t_off[j] + (uint32_t) s; p.otl[j] = w; p.osc[j] = dist[j]; c = 1; }
  }
  p.cnt2[j] = c;
}

__global__ void ep_status_kernel(const uint32_t* jst, uint64_t n, uint32_t* status, int32_t* dist, int32_t* start_loc, int32_t* end_loc, uint32_t* ops_len) {
  const uint64_t j = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  status[j] = jst[j];
  if (jst[j] == 4) { dist[j] = start_loc[j] = end_loc[j] = -1; ops_len[j] = 0; }
}

// the generalised-equality tables of ep_dev (f[256], s[256], cls[256 bytes]) from pairs passed by value. 256 threads.
struct EqPairs { uint8_t p[64]; uint32_t n; };
__global__ void ep_eqtab_kernel(EqPairs e, uint32_t* tab) {
  const uint32_t b = threadIdx.x;
  auto fs = [&](uint32_t x, int side) { uint32_t v = 0; for (uint32_t i = 0; i < e.n; ++i) v |= (uint32_t) (e.p[2 * i + side] == x) << i; return v; };
  const uint32_t f = fs(b, 0), s = fs(b, 1);
  tab[b] = f; tab[256 + b] = s;
  const uint8_t sym[5] = {'A', 'C', 'G', 'T', 'N'};
  uint8_t cls = 0;
  for (int sy = 0; sy < 5; ++sy)
    if (b == sym[sy] || (f & fs(sym[sy], 1)) || (s & fs(sym[sy], 0))) cls |= (uint8_t) (1u << sy);
  ((uint8_t*) (tab + 512))[b] = cls;
}
constexpr size_t EP_EQTAB_BYTES = (512 + 64) * 4;

// The equality tables of n_eq > 0 pairs, built on st into SLOT_EP_EQTAB; *tab: f[256], s[256], cls[256 bytes].
int ep_eqtabs(dgpu_ctx* ctx, cudaStream_t st, const uint8_t* eq_pairs, uint32_t n_eq, const uint32_t** tab) {
  EqPairs e;
  for (uint32_t i = 0; i < 2 * n_eq; ++i) e.p[i] = eq_pairs[i];
  e.n = n_eq;
  void* d_tab;
  int rc;
  if ((rc = dgpu_reserve(ctx, SLOT_EP_EQTAB, EP_EQTAB_BYTES, &d_tab))) return rc;
  ep_eqtab_kernel<<<1, 256, 0, st>>>(e, (uint32_t*) d_tab);
  DGPU_LAUNCH_CHECK(ctx, "ep_eqtab");
  *tab = (const uint32_t*) d_tab;
  return DGPU_OK;
}

// The kinds in `ids` on st, with the lists and counts the plan wrote. Each grid is the largest the workspace the setter reserved holds.
int run_bound(dgpu_ctx* ctx, cudaStream_t st, SegJobs a, std::vector<int> const& ids, bool leaves, bool eq, EpBound const& b, const size_t* room,
              const uint32_t* lists, uint64_t list_cap, const uint32_t* counts) {
  int rc;
  for (int id : ids) {
    const SegKindGeom k = bound_kind(id, leaves, eq, b.mq, b.w, room);
    if ((rc = seg_launch(ctx, st, a, k, SIZE_MAX, ctx->bufs[k.slot].cap, lists + id * list_cap, 0, counts + id))) return rc;
  }
  return DGPU_OK;
}

int ep_dev_async(dgpu_ctx* ctx, cudaStream_t st, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* q_off, const uint32_t* q_len,
                 const uint32_t* t_off, const uint32_t* t_len, int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist,
                 int32_t* start_loc, int32_t* end_loc, uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status, uint32_t max_slice) {
  int rc;
  EpBound b;
  b.mq = ctx->ep_max_query; b.mt = ctx->ep_max_target; b.w = std::min(b.mt, max_slice);
  b.levels = ep_bound_levels(b.mq, b.w);
  const bool eq = n_eq > 0;
  const size_t* room = seg_rooms(ctx, eq);
  const uint64_t S = 1ull << b.levels, NS = n * S;   // segment slots per job and in all
  const uint64_t qt = (uint64_t) b.mq + b.mt;
  const uint32_t run_jobs = (uint32_t) std::min<uint64_t>(EP_MIRROR_RUN / qt, n);
  const unsigned nb = (unsigned) ((n + 255) / 256), sb = (unsigned) ((NS + 255) / 256);

  // the per-call arrays, all sized from n and the bound
  void* base;
  const size_t plan_bytes = n * 4 * 12 + NS * (4 * 10 + 4 * 19 + 8 * 3 + 3 + 4 * EPK_N) + 4 * (EPK_N + 1) + 64 * 32;
  if ((rc = dgpu_reserve(ctx, SLOT_EP_PLAN, plan_bytes, &base))) return rc;
  uint8_t* cur = (uint8_t*) base;
  auto carve = [&](size_t nbytes) { uint8_t* r = cur; cur += (nbytes + 15) & ~(size_t) 15; return (void*) r; };
  uint32_t *ql2 = (uint32_t*) carve(n * 4), *tl2 = (uint32_t*) carve(n * 4), *mq_off = (uint32_t*) carve(n * 4), *mt_off = (uint32_t*) carve(n * 4);
  uint32_t *t2off = (uint32_t*) carve(n * 4), *t2len = (uint32_t*) carve(n * 4);
  int32_t *k2 = (int32_t*) carve(n * 4), *rev_pos = (int32_t*) carve(n * 4);
  uint32_t* cnt[2] = {(uint32_t*) carve(n * 4), (uint32_t*) carve(n * 4)};
  EpPlan p;
  p.n = n; p.q_off = q_off; p.q_len = ql2; p.t_off = t_off; p.t_len = tl2;
  p.jst = (uint32_t*) carve(n * 4);
  p.leaf_lo = (uint32_t*) carve((n + 1) * 4);
  uint32_t* sq[2]; uint32_t* sql[2]; uint32_t* sto[2]; uint32_t* stl[2]; int32_t* ssc[2];
  for (int x = 0; x < 2; ++x) {
    sq[x] = (uint32_t*) carve(NS * 4); sql[x] = (uint32_t*) carve(NS * 4); sto[x] = (uint32_t*) carve(NS * 4); stl[x] = (uint32_t*) carve(NS * 4);
    ssc[x] = (int32_t*) carve(NS * 4);
  }
  p.pre = (uint32_t*) carve((NS + 1) * 4);
  p.jq = (uint32_t*) carve(NS * 4); p.jql = (uint32_t*) carve(NS * 4); p.jt = (uint32_t*) carve(NS * 4); p.jtl = (uint32_t*) carve(NS * 4);
  p.jpm = (uint32_t*) carve(NS * 4); p.jpn = (uint32_t*) carve(NS * 4); p.jbound = (int32_t*) carve(NS * 4);
  p.out_len = (uint32_t*) carve(NS * 4); p.corner = (int32_t*) carve(NS * 4);
  p.sm = (uint32_t*) carve(NS * 4); p.sh = (uint32_t*) carve(NS * 4); p.sn = (uint32_t*) carve(NS * 4); p.sbest = (int32_t*) carve(NS * 4);
  p.leaf_kind = (uint32_t*) carve(NS * 4); p.leaf_len = (uint32_t*) carve(NS * 4);
  p.out3 = (int32_t*) carve(NS * 12);
  p.joff = (uint64_t*) carve(NS * 8); p.f_off = (uint64_t*) carve(NS * 8); p.b_off = (uint64_t*) carve(NS * 8);
  p.leaf_off = p.f_off;   // the leaves come after the last split
  p.jrev = (uint8_t*) carve(NS); p.jkind = (uint8_t*) carve(NS); p.jtail = (uint8_t*) carve(NS);
  p.list_cap = NS;
  p.lists = (uint32_t*) carve(NS * 4 * EPK_N);
  p.counts = (uint32_t*) carve(4 * (EPK_N + 1));
  p.col_stride = 2 * ((uint64_t) b.mq + S / 2);
  p.tmp_stride = qt;
  for (int c = 0; c < SEG_NCLS; ++c) p.room[c] = room[c];
  p.no_band = ep_no_band();
  void *d_col = nullptr, *d_mirror;
  if (b.levels && (rc = dgpu_reserve(ctx, SLOT_EP_COLS, (n * p.col_stride + 16) * sizeof(int), &d_col))) return rc;
  if ((rc = dgpu_reserve(ctx, SLOT_EP_MIRROR, n * qt + 64, &d_mirror))) return rc;   // the HW mirror, then the traced leaves' ops

  SegJobs a;
  a.seqs = seqs; a.q_off = p.jq; a.q_len = p.jql; a.t_off = p.jt; a.t_len = p.jtl; a.rev = p.jrev; a.kind = p.jkind; a.out_off = p.joff;
  a.out_len = p.out_len; a.corner = p.corner; a.tmp_ops = nullptr; a.colbuf = (int*) d_col; a.plan_m = p.jpm; a.plan_n = p.jpn;
  a.eq.f = nullptr; a.eq.s = nullptr; a.eq_cls = nullptr;
  const uint32_t* d_eqtabs = nullptr;
  if (eq) {
    if ((rc = ep_eqtabs(ctx, st, eq_pairs, n_eq, &d_eqtabs))) return rc;
    a.eq.f = d_eqtabs; a.eq.s = d_eqtabs + 256; a.eq_cls = (const uint8_t*) (d_eqtabs + 512);
  }

  // distance, end and start locations (ep_locate), on the lengths with refused jobs emptied
  ep_async_jobs_kernel<<<nb, 256, 0, st>>>(q_len, t_len, n, b.mq, b.mt, run_jobs, ql2, tl2, mq_off, mt_off, p.jst, ctx->refused + DGPU_REFUSED_EP);
  DGPU_LAUNCH_CHECK(ctx, "ep_async_jobs");
  const uint32_t ed_bound = std::max(b.mq, b.mt);
  if ((rc = dgpu_edit_distance_impl(ctx, seqs, seqs_bytes, q_off, ql2, t_off, tl2, nullptr, mode, n, dist, end_loc, st, 0, d_eqtabs, ed_bound))) return rc;
  if (mode == DGPU_MODE_HW) {
    ep_hwstart_jobs_kernel<<<nb, 256, 0, st>>>(mt_off, tl2, dist, end_loc, (uint32_t) n, t2off, t2len, k2);
    DGPU_LAUNCH_CHECK(ctx, "ep_hwstart_jobs");
    for (uint64_t j0 = 0; j0 < n; j0 += run_jobs) {   // a run reuses the mirror after the previous run's pass on the same stream
      const uint64_t c = std::min<uint64_t>(run_jobs, n - j0);
      const uint32_t wb = (uint32_t) ((c * 32 + 255) / 256);
      ep_mirror_kernel<<<wb, 256, 0, st>>>(seqs, (uint8_t*) d_mirror, q_off + j0, ql2 + j0, mq_off + j0, (uint32_t) c);
      DGPU_LAUNCH_CHECK(ctx, "ep_mirror(q)");
      ep_mirror_kernel<<<wb, 256, 0, st>>>(seqs, (uint8_t*) d_mirror, t_off + j0, tl2 + j0, mt_off + j0, (uint32_t) c);
      DGPU_LAUNCH_CHECK(ctx, "ep_mirror(t)");
      if ((rc = dgpu_edit_distance_impl(ctx, (const uint8_t*) d_mirror, c * qt, mq_off + j0, ql2 + j0, t2off + j0, t2len + j0, k2 + j0, DGPU_MODE_SHW, c,
                                        start_loc + j0, rev_pos + j0, st, 1, d_eqtabs, ed_bound))) return rc;
    }
  }
  ep_start_kernel<<<nb, 256, 0, st>>>(mode, ql2, tl2, dist, end_loc, rev_pos, (uint32_t) n, start_loc);
  DGPU_LAUNCH_CHECK(ctx, "ep_start");

  // Hirschberg's levels (ep_split)
  p.shift = 0; p.cnt2 = cnt[0]; p.oq = sq[0]; p.oql = sql[0]; p.ot = sto[0]; p.otl = stl[0]; p.osc = ssc[0];
  ep_seg_init_kernel<<<nb, 256, 0, st>>>(p, dist, start_loc, end_loc, max_slice);
  DGPU_LAUNCH_CHECK(ctx, "ep_seg_init");
  int in = 0;
  for (int l = 0; l < b.levels; ++l, in ^= 1) {
    p.shift = (uint32_t) l;
    p.cnt = cnt[in]; p.sq = sq[in]; p.sql = sql[in]; p.st = sto[in]; p.stl = stl[in]; p.ssc = ssc[in];
    p.cnt2 = cnt[in ^ 1]; p.oq = sq[in ^ 1]; p.oql = sql[in ^ 1]; p.ot = sto[in ^ 1]; p.otl = stl[in ^ 1]; p.osc = ssc[in ^ 1];
    const uint64_t slots = n << l;
    ep_plan_kernel<false><<<1, EPP_THREADS, 0, st>>>(p);
    DGPU_LAUNCH_CHECK(ctx, "ep_plan");
    const std::vector<int> ids = bound_kinds(b, l, false, room);
    if ((rc = run_bound(ctx, st, a, ids, false, eq, b, room, p.lists, p.list_cap, p.counts))) return rc;
    hb_select_kernel<true><<<(unsigned) ((slots * 32 + 255) / 256), 256, 0, st>>>((const int*) d_col, p.f_off, p.b_off, p.sm, p.sh, p.sn, p.sbest, 0,
                                                                               p.counts + EPK_N, p.out3);
    DGPU_LAUNCH_CHECK(ctx, "hb_select");
    ep_split_kernel<<<(unsigned) ((slots + 255) / 256), 256, 0, st>>>(p);
    DGPU_LAUNCH_CHECK(ctx, "ep_split");
  }

  // the leaves (ep_leaves)
  p.shift = (uint32_t) b.levels;
  p.cnt = cnt[in]; p.sq = sq[in]; p.sql = sql[in]; p.st = sto[in]; p.stl = stl[in]; p.ssc = ssc[in];
  ep_plan_kernel<true><<<1, EPP_THREADS, 0, st>>>(p);
  DGPU_LAUNCH_CHECK(ctx, "ep_plan");
  a.tmp_ops = (uint8_t*) d_mirror;
  a.colbuf = nullptr;
  dgpu_prof_begin(ctx, st);
  const std::vector<int> leaf_ids = bound_kinds(b, 0, true, room);
  if ((rc = run_bound(ctx, st, a, leaf_ids, true, eq, b, room, p.lists, p.list_cap, p.counts))) return rc;
  dgpu_prof_end(ctx, st);
  ep_leaf_done_kernel<<<sb, 256, 0, st>>>(p);
  DGPU_LAUNCH_CHECK(ctx, "ep_leaf_done");
  hb_concat_kernel<<<(unsigned) ((n * 32 + 255) / 256), 256, 0, st>>>((const uint8_t*) d_mirror, p.leaf_lo, p.leaf_kind, p.leaf_off, p.leaf_len,
                                                                      (uint32_t) n, ops, ops_off, ops_len);
  DGPU_LAUNCH_CHECK(ctx, "hb_concat");
  ep_status_kernel<<<nb, 256, 0, st>>>(p.jst, n, status, dist, start_loc, end_loc, ops_len);
  DGPU_LAUNCH_CHECK(ctx, "ep_status");
  return DGPU_OK;
}

// The device form of every entry point: a job whose aligned target slice is wider than max_slice gets status 2 alone.
int ep_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
           const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
           int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
           uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status, uint32_t max_slice, void* stream) {
  if (!ctx) return DGPU_ERR_ARG;
  if (n == 0) return DGPU_OK;
  if (n >= (1ull << 31) || seqs_bytes >= (1ull << 32)) return DGPU_ERR_ARG;
  if (mode != DGPU_MODE_NW && mode != DGPU_MODE_SHW && mode != DGPU_MODE_HW) return DGPU_ERR_ARG;
  if (!seqs || !q_off || !q_len || !t_off || !t_len || !dist || !start_loc || !end_loc || !ops || !ops_off || !ops_len || !status) return DGPU_ERR_ARG;
  if (n_eq > 32 || (n_eq && !eq_pairs)) return DGPU_ERR_ARG;
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t) stream : ctx->stream;
  if (ctx->ep_max_query)
    return ep_dev_async(ctx, st, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off, ops_len,
                        status, max_slice);
  int rc;
  // host copies of the job geometry
  std::vector<uint32_t> h_qoff(n), h_qlen(n), h_toff(n), h_tlen(n);
  std::vector<uint64_t> h_opsoff(n);
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_qoff.data(), q_off, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_qlen.data(), q_len, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_toff.data(), t_off, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_tlen.data(), t_len, n * 4, cudaMemcpyDeviceToHost, st));
  DGPU_CUDA(ctx, cudaMemcpyAsync(h_opsoff.data(), ops_off, n * 8, cudaMemcpyDeviceToHost, st));
  SegRunner R;
  R.ctx = ctx; R.st = st; R.seqs = seqs; R.use_eq = n_eq > 0; R.eq.f = nullptr; R.eq.s = nullptr;
  const uint32_t* d_eqtabs = nullptr;
  if (n_eq) {
    if ((rc = ep_eqtabs(ctx, st, eq_pairs, n_eq, &d_eqtabs))) return rc;
    R.eq.f = d_eqtabs; R.eq.s = d_eqtabs + 256; R.eq_cls = (const uint8_t*) (d_eqtabs + 512);
  }
  std::vector<int32_t> h_dist(n), h_start(n), h_end(n);
  if ((rc = ep_locate(ctx, st, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, d_eqtabs, n, h_qlen, h_tlen, dist, start_loc, end_loc, h_dist,
                      h_start, h_end))) return rc;
  std::vector<std::vector<Seg> > perjob(n);
  std::vector<uint32_t> h_status(n, 0);
  if ((rc = ep_split(ctx, st, R, n, h_qoff, h_qlen, h_toff, h_tlen, h_dist, h_start, h_end, max_slice, perjob, h_status))) return rc;
  return ep_leaves(ctx, st, R, n, perjob, h_status, ops, ops_off, ops_len, status);
}

// The host form of every entry point.
int ep_host(dgpu_ctx* ctx, const char* name, const uint8_t* seqs, uint64_t seqs_bytes,
            const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
            int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
            uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes, uint32_t* ops_len, uint32_t* status, uint32_t max_slice) {
  DgpuStage s(ctx, name, n);
  if (!ctx) return DGPU_ERR_ARG;
  if (n == 0) return DGPU_OK;
  if (!seqs || !q_off || !q_len || !t_off || !t_len || !dist || !start_loc || !end_loc || !ops || !ops_off || !ops_len || !status) return DGPU_ERR_ARG;
  int rc;
  if ((rc = s.check_arena(seqs_bytes, n, q_off, q_len)) || (rc = s.check_arena(seqs_bytes, n, t_off, t_len))) return rc;
  for (uint64_t i = 0; i < n; ++i)   // op slots (capacity |q| + |t|) inside ops_bytes
    if (ops_off[i] + q_len[i] + t_len[i] > ops_bytes) { ctx->last_error = std::string(name) + ": op slot beyond ops_bytes"; return DGPU_ERR_CAPACITY; }
  if ((rc = s.open())) return rc;
  const uint8_t* d_seqs = s.arena(seqs, seqs_bytes);
  uint8_t* d_ops = s.out(ops, ops_bytes, 64);
  const uint32_t *d_qoff = s.in(q_off, n), *d_qlen = s.in(q_len, n), *d_toff = s.in(t_off, n), *d_tlen = s.in(t_len, n);
  const uint64_t* d_opsoff = s.in(ops_off, n);
  int32_t *d_dist = s.out(dist, n), *d_start = s.out(start_loc, n), *d_end = s.out(end_loc, n);
  uint32_t *d_opslen = s.out(ops_len, n), *d_status = s.out(status, n);
  if (s.rc) return s.rc;
  if ((rc = ep_dev(ctx, d_seqs, seqs_bytes, d_qoff, d_qlen, d_toff, d_tlen, mode, eq_pairs, n_eq, n, d_dist, d_start, d_end, d_ops, d_opsoff, d_opslen,
                   d_status, max_slice, s.st)))
    return rc;
  return s.finish();
}

}  // namespace

extern "C" {

int dgpu_set_ep_async_bound(dgpu_ctx* ctx, uint32_t max_query, uint32_t max_target) {
  if (!ctx) return DGPU_ERR_ARG;
  if (!max_query && !max_target) { ctx->ep_max_query = ctx->ep_max_target = 0; return DGPU_OK; }
  if (max_query < 1 || max_target < 1 || max_query > DGPU_EP_MAX_SLICE || max_target > DGPU_EP_MAX_SLICE) {
    ctx->last_error = "dgpu_set_ep_async_bound: max_query and max_target must be 1 .. " + std::to_string(DGPU_EP_MAX_SLICE) + ", or both 0";
    return DGPU_ERR_ARG;
  }
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  int rc;
  if ((rc = dgpu_refusals_init(ctx))) return rc;
  // every kind any level or the leaves can reach, with or without equalities: its shared-memory opt-in and its workspace at the full grid
  // within the budget, at least one bound-shaped slab
  EpBound b;
  b.mq = max_query; b.mt = b.w = max_target; b.levels = ep_bound_levels(b.mq, b.w);
  size_t free_b = 0, total_b = 0;
  DGPU_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  std::vector<size_t> need(SLOT_COUNT, 0);
  for (int eq = 0; eq < 2; ++eq) {
    const size_t* room = seg_rooms(ctx, eq);
    for (int l = 0; l <= b.levels; ++l) {
      const bool leaves = l == b.levels;
      for (int id : bound_kinds(b, leaves ? 0 : l, leaves, room)) {
        const SegKindGeom k = bound_kind(id, leaves, eq, b.mq, b.w, room);
        const size_t grid = seg_grid(ctx, k, SIZE_MAX, dgpu_workspace_budget(ctx, k.slot, free_b));
        need[k.slot] = std::max(need[k.slot], std::max<size_t>(grid * k.per_cta * k.stride, 256));
        if (!k.half && (rc = dgpu_smem_optin(ctx, k.k, k.smem, "cudaFuncSetAttribute(seg_kernel)"))) return rc;
      }
    }
  }
  need[SLOT_EP_EQTAB] = EP_EQTAB_BYTES;
  for (int slot = 0; slot < SLOT_COUNT; ++slot) {
    void* w;
    if (need[slot] && (rc = dgpu_reserve(ctx, slot, need[slot], &w))) return rc;
  }
  ctx->ep_max_query = max_query;
  ctx->ep_max_target = max_target;
  return DGPU_OK;
}

int dgpu_edit_path_wide_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                            int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                            uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status, uint32_t max_slice, void* stream) {
  int rc;
  if ((rc = check_max_slice(ctx, max_slice))) return rc;
  return ep_dev(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off, ops_len, status,
                max_slice, stream);
}

int dgpu_edit_path_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                          const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                          int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                          uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status, void* stream) {
  return ep_dev(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off, ops_len, status,
                DGPU_EP_CLASSIC_SLICE, stream);
}

int dgpu_edit_path_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                       const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                       int mode, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                       uint8_t* ops, const uint64_t* ops_off, uint32_t* ops_len, uint32_t* status, void* stream) {
  return ep_dev(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, nullptr, 0, n, dist, start_loc, end_loc, ops, ops_off, ops_len, status,
                DGPU_EP_CLASSIC_SLICE, stream);
}

int dgpu_edit_path_wide(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                        const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                        int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                        uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes, uint32_t* ops_len, uint32_t* status, uint32_t max_slice) {
  int rc;
  if ((rc = check_max_slice(ctx, max_slice))) return rc;
  return ep_host(ctx, "dgpu_edit_path_wide", seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off,
                 ops_bytes, ops_len, status, max_slice);
}

int dgpu_edit_path_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                      const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                      int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                      uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes, uint32_t* ops_len, uint32_t* status) {
  return ep_host(ctx, "dgpu_edit_path", seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off,
                 ops_bytes, ops_len, status, DGPU_EP_CLASSIC_SLICE);
}

int dgpu_edit_path(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                   const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off, const uint32_t* t_len,
                   int mode, uint64_t n, int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                   uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes, uint32_t* ops_len, uint32_t* status) {
  return ep_host(ctx, "dgpu_edit_path", seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, nullptr, 0, n, dist, start_loc, end_loc, ops, ops_off,
                 ops_bytes, ops_len, status, DGPU_EP_CLASSIC_SLICE);
}

}  // extern "C"
