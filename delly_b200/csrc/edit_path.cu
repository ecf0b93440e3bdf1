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
                            int32_t* end_loc, void* stream, int last_pos, const uint32_t* eq_tabs);

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
};

// Geometry of the seg_kernel classes: a segment of n target columns takes the first row with n <= cap (class 0: n = 0), with C columns
// per lane, T threads per CTA (MULTI: T > 32) and a grid of at most per_sm CTAs per SM.
struct SegGeom { uint32_t cap; int C, T, per_sm; };
constexpr int SEG_NCLS = 12;
constexpr SegGeom SEG_GEOM[SEG_NCLS] = {{0, 0, 0, 0},
                                        {256, 8, 32, 16}, {512, 16, 32, 16}, {768, 24, 32, 16}, {1024, 32, 32, 16},
                                        {1280, 40, 32, 16}, {1536, 48, 32, 16}, {1792, 56, 32, 16}, {2048, 64, 32, 16},
                                        {4096, 32, 128, 4}, {8192, 32, 256, 2}, {16384, 32, 512, 1}};
__host__ __device__ inline uint32_t seg_dstride(uint32_t n, uint32_t C) { return ((n + C - 1) / C + 1) * (C / 8); }
inline int seg_class(uint32_t n) {
  for (int c = 0; c < SEG_NCLS; ++c)
    if (n <= SEG_GEOM[c].cap) return c;
  return -1;
}

template <int C, bool MULTI, bool EQ>
__global__ void __launch_bounds__(MULTI ? 512 : 32) seg_kernel(SegJobs a) {
  extern __shared__ uint8_t sm_rows[];
  __shared__ int sm_x[wf::WF_SMX];
  __shared__ int sm_pub[4];
  const int tid = threadIdx.x, T = blockDim.x;
  uint8_t* slab = a.work + (size_t) blockIdx.x * a.work_stride;
  uint32_t* dirs = (uint32_t*) slab;
  uint8_t* trace = slab + a.off_trace;
  const wf::Scoring sc = {0, -1, false, false};
  for (uint32_t idx = blockIdx.x; idx < a.count; idx += gridDim.x) {
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

template <int G, bool EQ>
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

  for (uint32_t base = gwarp * JPW; base < a.count; base += nwarps * JPW) {
    const bool have = base + grp < a.count;
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
template <bool EQ>
__global__ void __launch_bounds__(EPW_WARPS * 32) seg_half_wide_kernel(SegJobs a, size_t hrow_stride) {
  __shared__ uint64_t peq_s[EPW_WARPS][5][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t gwarp = blockIdx.x * EPW_WARPS + wib, nwarps = gridDim.x * EPW_WARPS;
  volatile int8_t* hrow = (volatile int8_t*) (a.work + (size_t) gwarp * hrow_stride);
  const EqTabs tabs = {a.eq.f, a.eq.s, a.eq_cls};
  for (uint32_t idx = gwarp; idx < a.count; idx += nwarps) {
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
template <bool EQ>
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

  for (uint32_t base = gwarp * JPW; base < a.count; base += nwarps * JPW) {
    const bool have = base + grp < a.count;
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
// (B[i] = -bcol[m-i]); interior rows i = 1..m-1 ascending, then i = 0, then i = m. One warp per segment.
__global__ void hb_select_kernel(const int* colbuf, const uint64_t* f_off, const uint64_t* b_off, const uint32_t* m_arr, const uint32_t* h_arr,
                                 const uint32_t* n_arr, const int32_t* best_arr, uint32_t nseg, int32_t* out3) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= nseg) return;
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
template <bool EQ, size_t... G>
constexpr std::array<SegKernel, SEG_NCLS> seg_kernels(std::index_sequence<G...>) {
  return {{nullptr, seg_kernel<SEG_GEOM[G + 1].C, (SEG_GEOM[G + 1].T > 32), EQ>...}};
}
constexpr std::array<SegKernel, SEG_NCLS> SEG_KERNELS[2] = {seg_kernels<false>(std::make_index_sequence<SEG_NCLS - 1>()),
                                                            seg_kernels<true>(std::make_index_sequence<SEG_NCLS - 1>())};

// seg_band_kernel of each band class (G = edb_lanes), [0] without and [1] with equality tables
template <bool EQ, size_t... C>
constexpr std::array<SegKernel, EDB_CLASSES> segb_kernels(std::index_sequence<C...>) {
  return {{seg_band_kernel<edb_lanes(C), EQ>...}};
}
constexpr std::array<SegKernel, EDB_CLASSES> SEGB_KERNELS[2] = {segb_kernels<false>(std::make_index_sequence<EDB_CLASSES>()),
                                                                segb_kernels<true>(std::make_index_sequence<EDB_CLASSES>())};
// the segments wider than the wavefront classes, [eq]
using SegHalfKernel = void (*)(SegJobs, size_t);
constexpr SegHalfKernel SEG_HALF_WIDE_KERNELS[2] = {seg_half_wide_kernel<false>, seg_half_wide_kernel<true>};
constexpr SegKernel SEG_LEAF_WIDE_KERNELS[2] = {seg_leaf_wide_kernel<false>, seg_leaf_wide_kernel<true>};

// narrowest band class that holds the segment's rows and certifies the optimum `k` of the problem (pm x pn) it belongs to; -1: none
inline int seg_band_class(uint32_t m, uint32_t pm, uint32_t pn, int32_t k) {
  if (k < 0) return -1;
  const int nblk = (int) ((m + 63) >> 6);
  for (int c = 0; c < EDB_CLASSES; ++c) {
    if (nblk > edb_block_cap(c)) continue;
    if (band_plan(edb_lanes(c), (int) pm, (int) pn).kvalid >= k) return c;
  }
  return -1;
}

// Whether seg_kernel cannot stage m query rows in shared memory: the launch's opt-in of (m + 15) & ~15 dynamic bytes would exceed the
// device's per-block maximum less the kernel's static shared memory, and the whole call would fail. Such half columns (Hirschberg over a
// query of more than ~230 kb) run on seg_half_wide_kernel instead; every segment seg_kernel can launch still runs there.
bool seg_rows_exceed(dgpu_ctx* ctx, uint32_t m, int cls, bool eq) {
  if (ctx->seg_room.empty()) ctx->seg_room.assign(SEG_NCLS * 2, 0);
  size_t& r = ctx->seg_room[cls * 2 + eq];   // [class][eq]: dynamic shared memory the class's seg_kernel may opt in to
  if (!r) {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device);
    cudaFuncAttributes fa{};
    cudaFuncGetAttributes(&fa, (const void*) SEG_KERNELS[eq][cls]);
    r = (size_t) optin - fa.sharedSizeBytes;
  }
  const size_t smem = ((size_t) m + 15) & ~(size_t) 15;
  return smem > 48 * 1024 && smem > r;
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
  // class lists
  // lists[1..11]: wavefront classes by target length (SEG_GEOM); lists[12..16]: band classes G = 2, 4, 8, 16, 32
  // wide_half / wide_leaf: unbanded segments wider than the wavefront classes (seg_half_wide_kernel, seg_leaf_wide_kernel)
  std::vector<std::vector<uint32_t> > lists(SEG_NCLS + EDB_CLASSES);
  std::vector<uint32_t> wide_half, wide_leaf;
  tail_ops.assign(N, 0);
  static const bool no_band = getenv("DGPU_EP_NO_BAND") != nullptr;   // development switch: no band classes (wavefront and wide kernels only)
  for (size_t i = 0; i < N; ++i) {
    const int bc = no_band ? -1 : seg_band_class(qlen[i], plan_m[i], plan_n[i], bound[i]);
    if (bc >= 0) { lists[SEG_NCLS + bc].push_back((uint32_t) i); tail_ops[i] = 1; continue; }
    const int c = seg_class(tlen[i]);
    if (c > 0 && !(kind[i] == 1 && seg_rows_exceed(ctx, qlen[i], c, use_eq))) { lists[c].push_back((uint32_t) i); continue; }
    if (kind[i] == 1) { wide_half.push_back((uint32_t) i); continue; }
    if (qlen[i] > 64 * EPL_G) return DGPU_ERR_UNSUPPORTED;   // Hirschberg's split rule leaves no such leaf
    wide_leaf.push_back((uint32_t) i);
    tail_ops[i] = 1;
  }
  std::vector<uint32_t> flat;
  std::vector<size_t> lo(SEG_NCLS + 1 + EDB_CLASSES, 0);
  for (int c = 1; c < SEG_NCLS + EDB_CLASSES; ++c) { lo[c] = flat.size(); flat.insert(flat.end(), lists[c].begin(), lists[c].end()); }
  lo[SEG_NCLS + EDB_CLASSES] = flat.size();
  const size_t lo_half = flat.size();
  flat.insert(flat.end(), wide_half.begin(), wide_half.end());
  const size_t lo_leaf = flat.size();
  flat.insert(flat.end(), wide_leaf.begin(), wide_leaf.end());
  DGPU_CUDA(ctx, cudaMemcpyAsync(d_list, flat.data(), flat.size() * 4, cudaMemcpyHostToDevice, st));
  SegJobs a;
  a.seqs = seqs; a.q_off = d_qoff; a.q_len = d_qlen; a.t_off = d_toff; a.t_len = d_tlen; a.rev = d_rev; a.kind = d_kind; a.out_off = d_oo;
  a.out_len = d_out_len; a.corner = d_corner; a.tmp_ops = tmp_ops; a.colbuf = colbuf; a.eq = eq;
  a.plan_m = d_pm; a.plan_n = d_pn; a.eq_cls = eq_cls;
  // One launch per kind of segment, in turn on st: band classes G = 2 .. 32, wide half columns, wide leaves, seg_kernel classes. A kind's CTA
  // takes `per_cta` jobs, each with `stride` bytes of workspace in `slot` (a wide half column's scratch row, a leaf's trace storage, a
  // seg_kernel job's directions and, from off_trace on, its trace); the grid is at most per_sm CTAs per SM, shrunk to the workspace budget.
  struct Kind {
    const std::vector<uint32_t>* jobs; size_t lo;   // the jobs and their offset in d_list
    size_t per_cta; int per_sm, slot; size_t stride, off_trace; unsigned threads; size_t smem;
    SegKernel k; SegHalfKernel half;                 // seg_half_wide_kernel (half) takes the stride as its row stride
    const char* name;
  };
  std::vector<Kind> kinds;
  for (int bc = 0; bc < EDB_CLASSES; ++bc) {
    std::vector<uint32_t> const& L = lists[SEG_NCLS + bc];
    if (L.empty()) continue;
    const int G = edb_lanes(bc), jpw = 32 / G;
    size_t maxsteps = 0;   // trace storage of a leaf: one uint4 per lane and step
    for (uint32_t i : L)
      if (kind[i] == 0) maxsteps = std::max<size_t>(maxsteps, 65 * (size_t) ((tlen[i] - 1) >> 6) + ((tlen[i] - 1) & 63) + G);
    kinds.push_back({&L, lo[SEG_NCLS + bc], (size_t) jpw * SEGB_WARPS, 8, SLOT_WAVEFRONT, maxsteps * G * sizeof(uint4), 0, SEGB_WARPS * 32, 0,
                     SEGB_KERNELS[use_eq][bc], nullptr, "seg_band_kernel"});
  }
  if (!wide_half.empty()) {   // one warp per half column, a scratch row of n bytes per warp
    size_t nmax = 0;
    for (uint32_t i : wide_half) nmax = std::max<size_t>(nmax, tlen[i]);
    kinds.push_back({&wide_half, lo_half, EPW_WARPS, 4, SLOT_EP_HROW, (nmax + 255) & ~(size_t) 255, 0, EPW_WARPS * 32, 0, nullptr,
                     SEG_HALF_WIDE_KERNELS[use_eq], "seg_half_wide_kernel"});
  }
  if (!wide_leaf.empty()) {   // trace storage of a leaf: one uint4 per block and column
    size_t maxcells = 0;
    for (uint32_t i : wide_leaf) maxcells = std::max<size_t>(maxcells, (size_t) tlen[i] * ((qlen[i] + 63) >> 6));
    kinds.push_back({&wide_leaf, lo_leaf, (size_t) (32 / EPL_G) * EPL_WARPS, 8, SLOT_WAVEFRONT, maxcells * sizeof(uint4), 0, EPL_WARPS * 32, 0,
                     SEG_LEAF_WIDE_KERNELS[use_eq], nullptr, "seg_leaf_wide_kernel"});
  }
  for (int c = 1; c < SEG_NCLS; ++c) {
    if (lists[c].empty()) continue;
    const SegGeom& g = SEG_GEOM[c];
    size_t maxwords = 0, mmax = 0, mnmax = 0;
    for (uint32_t i : lists[c]) {
      if (kind[i] == 0) maxwords = std::max(maxwords, (size_t) (qlen[i] + 1) * seg_dstride(tlen[i], g.C));   // half columns store no directions
      mmax = std::max<size_t>(mmax, qlen[i]);
      mnmax = std::max<size_t>(mnmax, (size_t) qlen[i] + tlen[i]);
    }
    auto al = [](size_t x) { return (x + 255) & ~(size_t) 255; };
    const size_t off_trace = al(maxwords * 4 + 1024);
    kinds.push_back({&lists[c], lo[c], 1, g.per_sm, SLOT_WAVEFRONT, off_trace + al(mnmax + 64), off_trace, (unsigned) g.T, (mmax + 15) & ~(size_t) 15,
                     SEG_KERNELS[use_eq][c], nullptr, "seg_kernel"});
  }
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  for (Kind const& k : kinds) {
    size_t grid = std::min<size_t>((k.jobs->size() + k.per_cta - 1) / k.per_cta, (size_t) ctx->num_sms * k.per_sm);
    const size_t per_block = k.per_cta * k.stride;
    const size_t budget = dgpu_workspace_budget(ctx, k.slot, free_b);
    if (per_block && grid * per_block > budget) grid = std::max<size_t>(1, budget / per_block);
    void* w;   // at least 256 bytes: a band class of half columns alone stores no trace (the other kinds always take more)
    if ((rc = dgpu_reserve(ctx, k.slot, std::max<size_t>(grid * per_block, 256), &w))) return rc;
    a.work = (uint8_t*) w;
    a.list = d_list + k.lo;
    a.count = (uint32_t) k.jobs->size();
    a.work_stride = k.stride;
    a.off_trace = k.off_trace;
    if (!k.half && (rc = dgpu_smem_optin(ctx, k.k, k.smem, "cudaFuncSetAttribute(seg_kernel)"))) return rc;
    if (k.half) k.half<<<(unsigned) grid, k.threads, 0, st>>>(a, k.stride);
    else k.k<<<(unsigned) grid, k.threads, k.smem, st>>>(a);
    DGPU_LAUNCH_CHECK(ctx, k.name);
  }
  return DGPU_OK;
}

inline bool seg_needs_split(uint32_t m, uint32_t n) {  // src/edlib.cpp:1189-1191
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
  if ((rc = dgpu_edit_distance_impl(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, nullptr, mode, n, dist, end_loc, st, 0, d_eqtabs))) return rc;
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
                                        (int32_t*) d_rev + j0, st, 1, d_eqtabs))) return rc;
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
    hb_select_kernel<<<(unsigned) ((S * 32 + 255) / 256), 256, 0, st>>>((const int*) d_col, d_foff, d_boff, d_m, d_h, d_n, d_best, (uint32_t) S, d_out3);
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
  const uint32_t* d_eqtabs = nullptr;  // f[256], s[256], cls[256 bytes]
  if (n_eq) {
    uint32_t tab[512 + 64] = {0};
    for (uint32_t p = 0; p < n_eq; ++p) { tab[eq_pairs[2 * p]] |= 1u << p; tab[256 + eq_pairs[2 * p + 1]] |= 1u << p; }
    uint8_t* cls = (uint8_t*) (tab + 512);
    static const uint8_t sym[5] = {'A', 'C', 'G', 'T', 'N'};
    for (uint32_t b = 0; b < 256; ++b)
      for (int sy = 0; sy < 5; ++sy)
        if (b == sym[sy] || (tab[b] & tab[256 + sym[sy]]) || (tab[256 + b] & tab[sym[sy]])) cls[b] |= (uint8_t) (1u << sy);
    void* d_tab;
    if ((rc = dgpu_reserve(ctx, SLOT_EP_EQTAB, sizeof(tab), &d_tab))) return rc;
    DGPU_CUDA(ctx, cudaMemcpyAsync(d_tab, tab, sizeof(tab), cudaMemcpyHostToDevice, st));
    DGPU_CUDA(ctx, cudaStreamSynchronize(st));  // tab is a stack array
    R.eq.f = (const uint32_t*) d_tab; R.eq.s = (const uint32_t*) d_tab + 256; R.eq_cls = (const uint8_t*) ((const uint32_t*) d_tab + 512);
    d_eqtabs = (const uint32_t*) d_tab;
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
