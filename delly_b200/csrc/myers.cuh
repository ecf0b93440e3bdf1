// myers.cuh — pieces shared by the bit-parallel kernels (edit_distance.cu, edit_path.cu): Myers' 64-row block update, the geometry and the
// pass of the banded staircase (G 64-row blocks per job on a sub-warp lane group; see the comment above ed_band_kernel), the striped warp
// wavefront and the leaf traceback.
#pragma once
#include "common.cuh"

// 64-row block update with signed hin/hout (src/edlib.cpp:407-442, Myers' Advance_Block).
__device__ __forceinline__ int block64(uint64_t& Pv, uint64_t& Mv, uint64_t Eq, int hin, uint64_t& PhOut, uint64_t& MhOut) {
  uint64_t hinNeg = (uint64_t) ((uint32_t) hin >> 31);
  uint64_t Xv = Eq | Mv;
  Eq |= hinNeg;
  uint64_t Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
  uint64_t Ph = Mv | ~(Xh | Pv);
  uint64_t Mh = Pv & Xh;
  PhOut = Ph;  // pre-shift horizontal deltas: bit r = delta of row r of this block
  MhOut = Mh;
  int hout = (int) (Ph >> 63) - (int) (Mh >> 63);
  Ph <<= 1;
  Mh <<= 1;
  Mh |= hinNeg;
  Ph |= (uint64_t) ((uint32_t) (hin + 1) >> 1);
  Pv = Mh | ~(Xv | Ph);
  Mv = Ph & Xv;
  return hout;
}


constexpr int EDB_WARPS = 4;
constexpr int EDB_CLASSES = 5;          // G = 2, 4, 8, 16, 32
#ifndef EDB_PEQ_WORDS_V
#define EDB_PEQ_WORDS_V 1280
#endif
constexpr int EDB_PEQ_WORDS = EDB_PEQ_WORDS_V;   // 64-bit Peq words per warp, split over the warp's 32/G jobs
constexpr int EDB_BLOCK_WORDS = 6;      // per 64-row block: match masks of A, C, G, T, N + the rows holding any other byte
__host__ __device__ constexpr int edb_lanes(int c) { return 2 << c; }
__host__ __device__ constexpr int edb_block_cap(int c) { return EDB_PEQ_WORDS / EDB_BLOCK_WORDS / (32 / edb_lanes(c)); }  // 13, 26, 53, 106, 213 blocks

struct BandPlan { int A; int kvalid; bool whole; };

__host__ __device__ inline BandPlan band_plan(int G, int m, int n) {
  const int d = n - m, up = d > 0 ? d : 0, lo = d < 0 ? -d : 0;
  BandPlan b; b.A = 0; int best = -0x7fffffff;
  for (int A = 0; A < G; ++A) {
    const int h1 = 64 * A - up, h2 = 64 * (G - 1 - A) - lo;
    const int h = h1 < h2 ? h1 : h2;
    if (h > best) { best = h; b.A = A; }
  }
  b.kvalid = best >= 0 ? 2 * best + up + lo : -1;
  b.whole = ((n - 1) >> 6) <= b.A && 64 * (G - b.A) >= m;
  return b;
}


// generalised equality (edlib's additionalEqualities, src/edlib.cpp:58-79) as three 256-entry tables; cls == nullptr: plain byte equality
struct EqTabs {
  const uint32_t* f;   // bitmask of the pairs in which the byte is the first member
  const uint32_t* s;   // ... the second member
  const uint8_t* cls;  // bitmask over {A,C,G,T,N} of the class symbols the byte is equal to
};

// Rows of a 64-row block equal to the target byte ch. word(sy): the block's rows holding symbol sy of {A,C,G,T,N}; other: the rows holding
// any other byte (IUPAC, lower case, gaps), compared byte by byte through row(i), under EQ with the pair tables too. An ACGTN byte equals
// no row outside ACGTN, so without EQ only a column byte outside ACGTN compares them.
template <bool EQ, typename Word, typename Row>
__device__ __forceinline__ uint64_t match_mask(uint32_t ch, uint64_t other, const EqTabs& tabs, Word word, Row row) {
  uint64_t Eq = 0;
  if (EQ) {
    const uint32_t cm = tabs.cls[ch & 0xffu];
#pragma unroll
    for (int sy = 0; sy < 5; ++sy)
      if ((cm >> sy) & 1u) Eq |= word(sy);
  } else {
    const uint32_t code = dna_code(ch);
    if (code < 5) return word(code);
  }
  if (other) {
    const uint32_t cf = EQ ? tabs.f[ch & 0xffu] : 0u, cs = EQ ? tabs.s[ch & 0xffu] : 0u;
    while (other) {
      const int i = __ffsll((long long) other) - 1;
      other &= other - 1;
      const uint32_t qb = row(i);
      if (qb == (ch & 0xffu) || (EQ && ((tabs.f[qb] & cs) || (tabs.s[qb] & cf)))) Eq |= 1ull << i;
    }
  }
  return Eq;
}

// Match masks of the job's 64-row blocks: lane p of the G-lane group builds blocks p, p+G, ... (rows read back to front when rev).
template <int G>
__device__ __forceinline__ void band_build_peq(uint64_t* peq, const uint8_t* q, int m, bool rev, int p) {
  const int nblk = (m + 63) >> 6;
  for (int bb = p; bb < nblk; bb += G) {
    uint32_t pl[EDB_BLOCK_WORDS] = {0, 0, 0, 0, 0, 0}, ph[EDB_BLOCK_WORDS] = {0, 0, 0, 0, 0, 0};
    const int r0 = bb * 64, rows = min(64, m - r0);
    for (int i = 0; i < rows; ++i) {
      const uint32_t code = dna_code(__ldg(rev ? q + (m - 1 - r0 - i) : q + r0 + i));
      const uint32_t bit = 1u << (i & 31);
#pragma unroll
      for (int sy = 0; sy < EDB_BLOCK_WORDS; ++sy) {
        const uint32_t v = (code == (uint32_t) sy) ? bit : 0u;
        if (i < 32) pl[sy] |= v; else ph[sy] |= v;
      }
    }
#pragma unroll
    for (int sy = 0; sy < EDB_BLOCK_WORDS; ++sy) peq[bb * EDB_BLOCK_WORDS + sy] = ((uint64_t) ph[sy] << 32) | pl[sy];
  }
}

// Rows of block blk equal to the target byte ch.
template <bool EQ>
__device__ __forceinline__ uint64_t band_eq(const uint64_t* peq, int blk, uint32_t ch, const uint8_t* q, int m, bool rev, const EqTabs& tabs) {
  const uint64_t* w = peq + blk * EDB_BLOCK_WORDS;
  return match_mask<EQ>(ch, w[5], tabs, [&](int sy) { return w[sy]; }, [&](int i) {
    const int row = blk * 64 + i;
    return (uint32_t) __ldg(rev ? q + (m - 1 - row) : q + row);
  });
}

// Staircase band pass of one job (q rows x t columns, both read back to front when rev) on its G-lane group, see the comment above
// ed_band_kernel. peq: the group's match masks (band_build_peq); hoP / hoM / hoS: the warp's hand-over rows, which take a block's Pv, Mv and
// last-row score to the lane above at the end of every 64-column chunk. step(st, Pv, Ph) runs after every block update (Ph: the pre-shift
// horizontal deltas into the column). On return the lane's last block is blk, its vertical deltas after column n-1 are Pv / Mv and sc is
// D[last row of the block][n].
template <int G, bool EQ, typename Step>
__device__ __forceinline__ void band_pass(const uint64_t* peq, const uint8_t* q, const uint8_t* t, int m, int n, bool rev, const BandPlan& bp,
                                          uint64_t* hoP, uint64_t* hoM, int* hoS, const EqTabs& tabs, uint64_t& Pv, uint64_t& Mv, int& sc,
                                          int& blk, Step step) {
  const int lane = threadIdx.x & 31, p = lane & (G - 1);
  const int nblk = (m + 63) >> 6;
  int steps = n > 0 ? 65 * ((n - 1) >> 6) + ((n - 1) & 63) + G : 0;
  for (int o = 16; o; o >>= 1) steps = max(steps, __shfl_xor_sync(0xffffffffu, steps, o));

  Pv = ~0ull; Mv = 0;
  blk = p - bp.A;
  int J = 0, c = -p;                              // c < 0: waiting for the skew; 0..63: column 64J + c; 64: hand-over slot
  sc = 64 * (blk + 1);                            // D[last row of the block][column before the current one]
  int hout = 1;
  uint32_t chn = n > 0 ? __ldg(rev ? t + (n - 1) : t) : 0u;
  for (int st = 0; st < steps; ++st) {
    const int hin_sh = __shfl_up_sync(0xffffffffu, hout, 1, G);
    if (c >= 0 && c < 64) {
      const int col = (J << 6) + c;
      if (col < n) {
        const uint32_t ch = chn;
        if (col + 1 < n) chn = __ldg(rev ? t + (n - 2 - col) : t + col + 1);
        if (blk >= 0 && blk < nblk) {
          const uint64_t Eq = band_eq<EQ>(peq, blk, ch, q, m, rev, tabs);
          const int hin = (p == 0 || blk == 0) ? 1 : hin_sh;   // above: the matrix border or a cell outside the band
          uint64_t Ph, Mh;
          hout = block64(Pv, Mv, Eq, hin, Ph, Mh);
          sc += hout;
          step(st, Pv, Ph);
        }
      }
    }
    const bool give = (c == 63), take = (c == 64) && (((J + 1) << 6) < n);
    if (__any_sync(0xffffffffu, give || take)) {
      if (give) { hoP[lane] = Pv; hoM[lane] = Mv; hoS[lane] = sc; }
      __syncwarp();
      if (take) {
        if (p < G - 1) { Pv = hoP[lane + 1]; Mv = hoM[lane + 1]; sc = hoS[lane + 1]; }
        else { Pv = ~0ull; Mv = 0; sc += 64; }
        ++blk; ++J; c = -1;
      }
      __syncwarp();
    }
    ++c;
  }
}

// D[m][n] after band_pass: the block holding row m-1, corrected by the vertical deltas of the rows below it inside the block, broadcast over
// the group from lane plast of the group, which holds that block. plast outside [0, G): the band does not reach the corner.
template <int G>
__device__ __forceinline__ int band_corner(uint64_t Pv, uint64_t Mv, int sc, int m, int n, const BandPlan& bp, int& plast) {
  const int tb = (m - 1) & 63;
  const uint64_t below = tb == 63 ? 0ull : (~0ull << (tb + 1));
  const int s = sc - __popcll(Pv & below) + __popcll(Mv & below);
  plast = (((m + 63) >> 6) - 1) - (((n - 1) >> 6) - bp.A);
  return __shfl_sync(0xffffffffu, s, ((threadIdx.x & 31) & ~(G - 1)) + (plast & (G - 1)));
}

// Striped warp wavefront of one job (q rows x t columns, both read back to front when rev): one warp, lane = 64-row block, 2048-row
// stripes, each lane one step behind the lane above (hout by shuffle), the column bytes loaded 32 at a time and passed down the lanes by
// shuffle. peq: the warp's symbol-major [5][32] match masks (no bank conflicts in the inner loop). hin0: the top row's horizontal delta (0
// for HW, 1 otherwise); each stripe's bottom deltas are parked in hrow (n bytes) for the stripe below. cell(col, Ph, Mh) runs on the lane
// owning row m-1 after each of its block updates (pre-shift horizontal deltas); stripe_end(row0, rows, Pv, Mv) runs on every lane after
// each stripe with its block's first row, its row count (0 on idle lanes) and its vertical deltas after column n-1.
template <bool EQ, typename Cell, typename StripeEnd>
__device__ __forceinline__ void stripes(uint64_t (*peq)[32], volatile int8_t* hrow, const uint8_t* q, const uint8_t* t, uint32_t m, uint32_t n,
                                        bool rev, int hin0, const EqTabs& tabs, Cell cell, StripeEnd stripe_end) {
  const int lane = threadIdx.x & 31;
  const uint32_t nstripes = (m + 2047) / 2048;
  for (uint32_t s = 0; s < nstripes; ++s) {
    const uint32_t row0 = s * 2048 + (uint32_t) lane * 64;
    const int nb = (int) min(32u, (m - s * 2048 + 63) / 64);   // active lanes in this stripe
    const bool active = lane < nb, last = lane == nb - 1 && s + 1 == nstripes, park = lane == nb - 1 && s + 1 < nstripes;
    const int rows = active ? (int) min(64u, m - row0) : 0;
    auto qrow = [&](int i) { return (uint32_t) __ldg(rev ? q + (m - 1 - row0 - i) : q + row0 + i); };
    uint64_t other = 0;   // rows holding a byte outside ACGTN
    {
      uint64_t pm[5] = {0, 0, 0, 0, 0};
      for (int i = 0; i < rows; ++i) {
        const uint32_t code = dna_code(qrow(i));
#pragma unroll
        for (int sy = 0; sy < 5; ++sy) pm[sy] |= (code == (uint32_t) sy) ? (1ull << i) : 0ull;
        if (code == 5u) other |= 1ull << i;
      }
      __syncwarp();
#pragma unroll
      for (int sy = 0; sy < 5; ++sy) peq[sy][lane] = pm[sy];
      __syncwarp();
    }
    uint64_t Pv = ~0ull, Mv = 0;
    int hout = 0;
    uint32_t cbuf = 0;   // 32 target bytes, one per lane, refreshed every 32 steps
    uint32_t cchar = 0;  // this lane's current column byte
    const uint32_t nsteps = n + (uint32_t) nb - 1;
    for (uint32_t st = 0; st < nsteps; ++st) {
      if ((st & 31u) == 0) {
        const uint32_t p = st + (uint32_t) lane;
        cbuf = (p < n) ? (uint32_t) __ldg(rev ? t + (n - 1 - p) : t + p) : 0u;
      }
      const uint32_t newc = __shfl_sync(0xffffffffu, cbuf, (int) (st & 31u));
      const uint32_t upc = __shfl_up_sync(0xffffffffu, cchar, 1);
      cchar = (lane == 0) ? newc : upc;
      const int hin_sh = __shfl_up_sync(0xffffffffu, hout, 1);
      const int col = (int) st - lane;
      if (active && col >= 0 && col < (int) n) {
        const int hin = lane ? hin_sh : (s == 0 ? hin0 : (int) hrow[col]);
        const uint64_t Eq = match_mask<EQ>(cchar, other, tabs, [&](int sy) { return peq[sy][lane]; }, qrow);
        uint64_t Ph, Mh;
        hout = block64(Pv, Mv, Eq, hin, Ph, Mh);
        if (last) cell(col, Ph, Mh);
        if (park) hrow[col] = (int8_t) hout;
      }
    }
    __syncwarp();
    __threadfence_block();
    stripe_end(row0, rows, Pv, Mv);
  }
}

// Traceback of a leaf (src/edlib.cpp:1021-1131: up = insert 1, left = delete 2, diagonal = match 0 / mismatch 3) over the stored (Pv after
// the column, Ph into the column) words of its 64-row blocks: up iff the Pv bit, else left iff the Ph bit, else diagonal. The G lanes of a
// group walk the path together through a window of WCOLS columns of the current block staged in win (fetch(col, block): the stored word).
// act: the group traces a leaf; under EQ a diagonal step matches by eq.equal. Ops are written from the END of the slot out[0 .. m + n)
// backwards; returns how many.
template <int G, int WCOLS, bool EQ, typename Tabs, typename Fetch>
__device__ __forceinline__ uint32_t leaf_trace(bool act, const uint8_t* q, const uint8_t* t, int m, int n, bool rev, const Tabs& eq, uint4* win,
                                               uint8_t* out, Fetch fetch) {
  const int p = threadIdx.x & (G - 1);
  int r = m - 1, cc = n - 1;
  uint32_t k = 0;
  const uint32_t cap = (uint32_t) (m + n);
  int wb = -1, wc0 = -1;
  while (__any_sync(0xffffffffu, act && r >= 0 && cc >= 0)) {
    const bool go = act && r >= 0 && cc >= 0;
    const int b = r >> 6;
    const bool need = go && (b != wb || cc > wc0 || cc <= wc0 - WCOLS);
    if (__any_sync(0xffffffffu, need)) {
      if (need) {
        for (int x = p; x < WCOLS; x += G) {
          const int col = cc - x;
          win[x] = col >= 0 ? fetch(col, b) : make_uint4(0, 0, 0, 0);
        }
        wb = b; wc0 = cc;
      }
      __syncwarp();
    }
    if (go) {
      const uint4 w = win[wc0 - cc];
      const int bit = r & 63;
      const uint32_t pv = ((bit < 32 ? w.x : w.y) >> (bit & 31)) & 1u;
      const uint32_t ph = ((bit < 32 ? w.z : w.w) >> (bit & 31)) & 1u;
      uint8_t op;
      if (pv) { op = 1; --r; }
      else if (ph) { op = 2; --cc; }
      else {
        const uint32_t x = __ldg(rev ? q + (m - 1 - r) : q + r), y = __ldg(rev ? t + (n - 1 - cc) : t + cc);
        op = (EQ ? eq.equal(x, y) : (x == y)) ? 0 : 3;
        --r; --cc;
      }
      if (p == 0) out[cap - 1 - k] = op;
      ++k;
    }
    __syncwarp();
  }
  if (act) {
    for (int i = p; i <= r; i += G) out[cap - 1 - (k + (uint32_t) i)] = 1;    // column 0 reached: the remaining rows are inserts
    if (r >= 0) k += (uint32_t) (r + 1);
    for (int i = p; i <= cc; i += G) out[cap - 1 - (k + (uint32_t) i)] = 2;   // row 0 reached: the remaining columns are deletes
    if (cc >= 0) k += (uint32_t) (cc + 1);
  }
  return k;
}
