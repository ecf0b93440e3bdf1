// wavefront2.cuh — the longNeedle DP engine, second generation: TWO DP ROWS PER INSTRUCTION.
//
// Same decomposition as wavefront.cuh (thread t owns C consecutive DP columns, anti-diagonal wavefront across the threads, one shuffle
// hand-off per step), but a thread now advances a PAIR of rows (rA = 2k-1, rB = 2k) in one sweep over its columns, with the two cells of an
// iteration packed as int16x2 in one register: lane A (low half) computes cell (rA, c0+j), lane B (high half) cell (rB, c0+j-1) — the two
// cells of one anti-diagonal, which are independent. Every arithmetic instruction of the recurrence is a 16x2 SIMD-in-register DPX op
// (VIMNMX3.S16x2, VIMNMX.S16x2, VIADDMNMX.S16x2) or a plain 32-bit op that acts on both halves without cross-talk:
//
//     mm   = min.u16x2(colpair[j] & rowpair, 1)            match flags of both cells (one-hot base codes)
//     T    = diag + 2*mm                                    diagonal + (match ? 2 : 0)        [scores are row-shifted: U = H + r + 8]
//     X    = max3.s16x2(T, up, left)                        both cells
//     acc += (5X - up - 4left) << 4(j&3)                    both direction nibbles: (X-up) | (X-left) << 2, three IMADs on the FMA pipe
//     run  = max.s16x2(run, X)                              running row maxima (bestMat / bestRev of src/needle.h:88-103)
//     REV: every second iteration one PRMT packs two prefix maxima of a row for the mirrored int16 store
//     FWD: vmax = max(vmax, run + partner)                  one PRMT + one VIADDMNMX.S16x2: the fused join of src/needle.h:104-115
//     up'  = prmt(S[j+1], X) ; diag' = up ; left' = X - g   operands of the next iteration (lane B's `up` is lane A's result)
//
// i.e. ~10 instructions per TWO cells where the scalar engine spends ~12 per cell, and the per-thread state is C packed registers (previous
// row) + C+1 column-pair registers, so twice as many warps fit on an SM.
//
// Exactness notes:
//  * U = H + r + 8 >= 8 for every cell of a semiglobal matrix with a free first row (H >= -r), and <= 2m + 8: all packed values are positive
//    15-bit numbers; plain 32-bit add / subtract / multiply-add never carries between the halves, and the linear form 5X - up - 4left
//    yields both nibbles exactly (the differences X - up and X - left are in 0..3 by the DP's Lipschitz bounds: match +1, gaps -1).
//  * The direction nibble stores the DIFFERENCES, not a decoded direction: vertical iff (X - up) == 0, else horizontal iff (X - left) == 0,
//    else diagonal — longNeedle's priority (src/needle.h:159-171). Decoding happens in the traceback (O(m + n) cells).
//  * Lane B lags one column: its nibble for column c0+j-1 is produced in iteration j. Within a thread's C-nibble group the nibbles of an
//    EVEN row are therefore rotated by one (slot k holds column c0 + k - 1, slot 0 holds column c0 + C - 1); nib_index() maps (row, column).
//  * Lane B of iteration 0 and lane A of iteration C are not cells of this thread; their operands are arranged so that they reproduce the
//    neighbour's boundary value (B) / contribute a zero nibble (A) — see the operand set-up below.
//  * Bases are one-hot coded (A C G T N); a job with any other byte goes through the scalar engine (wavefront.cuh), which compares bytes.
#pragma once
#include "common.cuh"
#include "wavefront.cuh"

namespace wf2 {

using wf::Best;
using wf::best_before;

// partner-row ring depth in steps (FWD): rows are fetched PART_D - 1 steps ahead with cp.async (template parameter of pass())
constexpr int BIAS = 8;          // U = H + row + BIAS
constexpr uint32_t NEG16x2 = 0x80008000u;

enum Mode { REV = 1, FWD = 2 };

__device__ __forceinline__ uint32_t hot(uint32_t ch) {
  return ch == 'A' ? 1u : ch == 'C' ? 2u : ch == 'G' ? 4u : ch == 'T' ? 8u : ch == 'N' ? 16u : 0u;
}
__host__ __device__ __forceinline__ bool hot_ok(uint8_t ch) { return ch == 'A' || ch == 'C' || ch == 'G' || ch == 'T' || ch == 'N'; }

// position of cell (r, c) inside the nibble row of r (cstart = first column of thread 0); see the header for the rotation of even rows
template <int C>
__device__ __forceinline__ int nib_index(int r, int c, int cstart) {
  const int k = c - cstart;
  const int t = k / C;
  int o = k - t * C;
  if (!(r & 1)) o = (o + 1 == C) ? 0 : o + 1;
  return t * C + o;
}
// decoded direction of a nibble: 1 vertical, 2 horizontal, 0 diagonal
__device__ __forceinline__ uint32_t nib_dir(uint32_t nib) { return ((nib & 3u) == 0u) ? 1u : (((nib >> 2) & 3u) == 0u ? 2u : 0u); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const uint32_t s = (uint32_t) __cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async16s(uint32_t smem32, const void* gmem) {   // destination given as a shared-window address
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem32), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// shared memory a pass needs for the partner ring (FWD), in uint4
__host__ __device__ constexpr int part_slots(int C, int part_d, int T) { return part_d * 2 * (C / 8) * T; }

// ---- workspace layout: STEP-MAJOR ("diagonal") ---------------------------------------------------------------------------
// At one step of the wavefront the threads of a warp work on DIFFERENT rows (thread t on row pair s - t), so a row-major workspace makes
// every warp-wide store touch 32 cache lines (one 16-byte piece per line): the reverse pass was bound by the load/store unit, not by the
// arithmetic. The workspace is therefore indexed by STEP first: the 16-byte group (row r, thread t, group w)
// — eight mirrored prefix maxima, or eight direction nibbles x 4 bits = one word — lives at
//     prefix maxima (uint4 units):  ((step * 2 + ab) * WPT + w) * T + t        step = pair(r) + t, pair(r) = (r + 1) >> 1, ab = 0 for odd r (lane A), 1 for even r
//     nibble words  (uint32 units): ((step * 2 + ab) * T + t) * WPT + w
// so that what the 32 lanes of a warp store in one instruction is contiguous. The forward pass reads the partner row m - r of its own row r;
// under the mirroring all lanes of a warp then read groups of the SAME reverse step, again contiguous. Row 0 is "pair 0, lane B".
// Sizes: (K + T + 1) * 2 * WPT * T groups resp. * T * WPT words with K = (m + 1) / 2 row pairs, and behind the groups the
// (WPT + 1) * T constant groups of synth_groups().
__host__ __device__ __forceinline__ size_t ws_steps(int m, int T) { return (size_t) ((m + 1) / 2 + T + 1); }
__host__ __device__ __forceinline__ int ws_synth_groups(int C, int T) { return (C / 8 + 1) * T; }
__host__ __device__ __forceinline__ size_t ws_brev_bytes(int C, int m, int T) { return (ws_steps(m, T) * 2 * (C / 8) * T + ws_synth_groups(C, T)) * 16; }
__host__ __device__ __forceinline__ size_t ws_dirs_bytes(int C, int m, int T) { return ws_steps(m, T) * 2 * (C / 8) * T * 4; }
template <int C> __device__ __forceinline__ size_t grp_index(int r, int t, int w, int T) {
  return ((size_t) ((((r + 1) >> 1) + t) * 2 + ((r & 1) ^ 1)) * (C / 8) + w) * T + t;
}
template <int C> __device__ __forceinline__ size_t nibw_index(int r, int t, int w, int T) {
  return ((size_t) ((((r + 1) >> 1) + t) * 2 + ((r & 1) ^ 1)) * T + t) * (C / 8) + w;
}
// nibble word gw (= thread * WPT + w) of row r
template <int C> __device__ __forceinline__ uint32_t nib_word(const uint32_t* __restrict__ dirs, int r, int gw, int T) {
  return __ldcg(dirs + nibw_index<C>(r, gw / (C / 8), gw % (C / 8), T));
}
// one stored prefix maximum of the reverse pass: row r, mirrored index idx (element x = nactR * C - idx); idx == nactR * C is column 0 (U = BIAS)
template <int C> __device__ __forceinline__ int brev_at(const uint4* __restrict__ brev4, int r, int idx, int nactR, int T) {
  if (idx >= nactR * C) return idx == nactR * C ? BIAS : -32768;
  const int g = idx >> 3;
  const int16_t* p = (const int16_t*) (brev4 + grp_index<C>(r, nactR - 1 - g / (C / 8), g % (C / 8), T));
  return (int) __ldcg(p + (idx & 7));
}

// The constant groups the forward pass reads where no reverse thread stored one (see pass(): synth0). Called by every thread of the CTA after the
// reverse pass of the job, before the forward pass; the caller synchronises.
template <int C> __device__ __forceinline__ void synth_groups(uint4* __restrict__ brev4, int m) {
  constexpr int WPT = C / 8;
  constexpr uint32_t NEG2 = 0x80008000u;
  const int T = blockDim.x, tid = threadIdx.x;
  uint4* g = brev4 + ws_steps(m, T) * 2 * WPT * T;
  for (int i = tid; i < ws_synth_groups(C, T); i += T) g[i] = make_uint4(i == 0 ? ((NEG2 & 0xffff0000u) | (uint32_t) BIAS) : NEG2, NEG2, NEG2, NEG2);
}

// rowHot: one-hot codes of the row string (shared memory, m bytes); colChar(c-1) = column byte.
// Scoring is longNeedle's: match 1, mismatch -1, gap 1, first row free, last row horizontally free (src/needle.h:59-66).
// REV (cstart = 1): stores per row the running prefix maxima (int16, mirrored: element x at index P-1-x, value U-shifted) and the nibbles.
// FWD (cstart = idx0 - delta, see wavefront.cuh): nibbles + fused join against the stored maxima of REV; best = per-thread arg-max.
template <int C, bool MULTI, int MODE, int PART_D, typename TB>
__device__ __forceinline__ void pass(const uint8_t* rowHot, TB colChar, const int m, const int n, const int cstart, uint32_t* __restrict__ dirs,
                                     uint4* __restrict__ brev4, const int P, int* sm_x /* MULTI: WF_SMX ints */,
                                     uint4* sm_part /* FWD: part_slots(C, PART_D, T) uint4 */, uint32_t* sm_scr /* FWD: (C + 1) * T words */, Best& best, int& corner) {
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int T = blockDim.x;
  const int c0 = cstart + tid * C;
  constexpr int WPT = C / 8;
  const int delta = P - 1 - n;
  const bool first = (tid == 0);
  const bool owns = (c0 <= n) && (c0 + C - 1 >= 1);
  const int K = (m + 1) >> 1;                       // row pairs
  const int nactR = (P - 1) / C;                    // threads of the reverse pass that own columns (P - 1 = nactR * C)
  const int nact = (n - cstart + C) / C;
  const int nsteps = K + min(T, nact) - 1;
  constexpr uint32_t B2 = (uint32_t) BIAS | ((uint32_t) BIAS << 16);

  // column pairs: low half = one-hot of column c0+j (lane A), high half = one-hot of column c0+j-1 (lane B); 0 = matches nothing
  uint32_t colp[C + 1];
#pragma unroll
  for (int j = 0; j <= C; ++j) {
    const int ca = c0 + j, cb = c0 + j - 1;
    const uint32_t a = (j < C && ca >= 1 && ca <= n) ? hot((uint32_t) colChar(ca - 1)) : 0u;
    const uint32_t b = (j > 0 && cb >= 1 && cb <= n) ? hot((uint32_t) colChar(cb - 1)) : 0u;
    colp[j] = a | (b << 16);
  }
  uint32_t S[C];   // S[j]: high half = U(row above the current pair, column c0+j); low half = U(rA of the last pair, column c0+j+1)
#pragma unroll
  for (int j = 0; j < C; ++j) S[j] = B2;
  uint32_t X0 = B2;            // iteration-0 result of the last pair (lane A: column c0)
  uint32_t handH = B2, handX = B2, prevRecvHi = BIAS;
  best.val = wf::NEG; best.row = 0; best.col = 0; best.bm = 0;

  // ---- row 0 ------------------------------------------------------------------------------------------------------------
  if (MODE == REV) {
    if (owns) {   // prefix maxima of row 0: U = 0 + 0 + BIAS ("pair 0, lane B")
#pragma unroll
      for (int w = 0; w < WPT; ++w) brev4[grp_index<C>(0, tid, w, T)] = make_uint4(B2, B2, B2, B2);
    }
  }
  if (MODE == FWD) {
    // join candidates of row 0: bestMat[0][c] = 0, partner = element (m, n-c) at index c + delta of row m (stored with shift m + BIAS)
    if (first && c0 == 1) { const int v = brev_at<C>(brev4, m, delta, nactR, T) - m - BIAS; if (v > best.val) { best.val = v; best.row = 0; best.col = 0; best.bm = 0; } }
    if (owns) {
      for (int j = 0; j < C; ++j) {
        const int c = c0 + j;
        if (c >= 0 && c <= n) {
          const int v = brev_at<C>(brev4, m, c + delta, nactR, T) - m - BIAS;
          if (v > best.val) { best.val = v; best.row = 0; best.col = c; best.bm = 0; }
        }
      }
    }
  }

  // ---- FWD: partner rows through a shared-memory ring, PART_D - 1 steps ahead ------------------------------------------
  // Source of the partner groups: this thread's groups g0 .. g0+WPT-1 of a reverse row were written by at most two reverse threads
  // (tqa for the first `split` groups, tqa - 1 for the rest); inside a row the uint4 index of group w is rowbase(r') + w*T + (w < split ? offA : offB)
  // (see grp_index: rowbase = (pair(r')*2 + ab) * WPT * T). Threads with tq < 0 have no stored group there: column 0 (U = BIAS) or beyond the row.
  const int g0 = (c0 + delta) >> 3;               // first mirrored group of this thread's columns (c0 + delta is a multiple of 8)
  const int tqa = nactR - 1 - g0 / WPT, wa0 = g0 % WPT;
  const int split = WPT - wa0;
  // As uint4 indices relative to brev4 a group's source is base + w*T (+ the row's base when a reverse thread stored it). Groups nobody stored
  // (column 0: U = BIAS as first element; beyond the row: no partner) are read from a small constant region behind the job's rows
  // (synth_groups below: entry 0 = the column-0 group, every other entry = "no partner"), so that the prefetch is branch-free.
  const int synth0 = (int) (ws_steps(m, T) * 2 * WPT * T);
  const bool dynA = tqa >= 0, dynB = tqa >= 1;
  const int baseA = dynA ? (2 * tqa * WPT + wa0) * T + tqa : ((tqa == -1 && wa0 == 0) ? synth0 : synth0 + 1);
  const int baseB = dynB ? (2 * (tqa - 1) * WPT - split) * T + (tqa - 1) : ((tqa == 0) ? synth0 - split * T : synth0 + 1);
  const uint32_t part32 = (uint32_t) __cvta_generic_to_shared(sm_part + tid);   // this thread's column of the ring, as a shared-window address
  auto fetch_row = [&](uint32_t dst32, int rp) {   // partner row rp -> ring slot (dst32 = this thread's first group of the row)
    const int rowbase = ((((rp + 1) >> 1) * 2 + ((rp & 1) ^ 1)) * WPT) * T;
    const int bA = baseA + (dynA ? rowbase : 0), bB = baseB + (dynB ? rowbase : 0);
#pragma unroll
    for (int w = 0; w < WPT; ++w) cp_async16s(dst32 + (uint32_t) (w * T) * 16u, brev4 + ((w < split ? bA : bB) + w * T));
  };
  int pslot = 1;   // ring slot of the next prefetch (= step % PART_D, kept as a counter)
  auto prefetch = [&](int sp) {   // partner rows of step sp (pair kp = sp - tid): rows m - rA, m - rB, this thread's columns
    if (MODE == FWD) {
      const int kp = sp - tid;
      if (owns && kp >= 1 && kp <= K) {
        const uint32_t dst32 = part32 + (uint32_t) (pslot * 2 * WPT * T) * 16u;
        fetch_row(dst32, m - (2 * kp - 1));
        if (2 * kp <= m) fetch_row(dst32 + (uint32_t) (WPT * T) * 16u, m - 2 * kp);
      }
      cp_async_commit();
      pslot = (pslot + 1 == PART_D) ? 0 : pslot + 1;
    }
  };
  int cslot = 0;   // ring slot of the current step (advanced at the top of every step)
  int gk = wf::NEG; // FWD: best join value any lane of this warp has seen so far
  if (MODE == FWD) {
#pragma unroll
    for (int sp = 1; sp < PART_D; ++sp) prefetch(sp);
  }
#if WF_RING
  if (MULTI) {
    __syncthreads();
    if (tid < 2 * wf::WF_MAXW) sm_x[wf::WF_MAXW * wf::RING_D * 2 + tid] = 0;
    __syncthreads();
  }
#endif

  for (int s = 1; s <= nsteps; ++s) {
    // ---- hand-off from the left neighbour (what it produced in the previous step, for the same row pair) -------------------
    uint32_t recvH = __shfl_up_sync(0xffffffffu, handH, 1);
    uint32_t recvX = __shfl_up_sync(0xffffffffu, handX, 1);
    if (MULTI) {
      const int w = tid >> 5;
      volatile int* ring = sm_x;
      volatile int* prod = sm_x + wf::WF_MAXW * wf::RING_D * 2;
      volatile int* cons = prod + wf::WF_MAXW;
      const int nw = T >> 5;
      if (lane == 31 && w + 1 < nw) {
        while (cons[w + 1] < s - wf::RING_D) { }
        ring[(w * wf::RING_D + (s % wf::RING_D)) * 2] = (int) handH;
        ring[(w * wf::RING_D + (s % wf::RING_D)) * 2 + 1] = (int) handX;
        __threadfence_block();
        prod[w] = s;
      }
      if (lane == 0 && w > 0) {
        while (prod[w - 1] < s) { }
        recvH = (uint32_t) ring[((w - 1) * wf::RING_D + (s % wf::RING_D)) * 2];
        recvX = (uint32_t) ring[((w - 1) * wf::RING_D + (s % wf::RING_D)) * 2 + 1];
        __threadfence_block();
        cons[w] = s;
      }
      __syncwarp();
    }
    if (MODE == FWD) { prefetch(s + PART_D - 1); cp_async_wait<PART_D - 1>(); cslot = (cslot + 1 == PART_D) ? 0 : cslot + 1; }
    const int k = s - tid;
    int candA = wf::NEG, candB = wf::NEG, candRow = 0;   // FWD: join maxima of the two rows of this step (idle lanes: none)
    uint32_t candRX = 0;
    if (k >= 1 && k <= K && owns) {
      const int rA = 2 * k - 1, rB = 2 * k;
      const bool hasB = (rB <= m);
      const uint32_t gvec = ((rA == m) ? 0u : 1u) | (((rB == m) ? 0u : 1u) << 16);        // horizontal gap: free in the last row
      const uint32_t rowpair = (uint32_t) rowHot[rA - 1] | (hasB ? ((uint32_t) rowHot[rB - 1] << 16) : 0u);
      const uint32_t rH = first ? B2 : recvH;       // (U(rA, c0-1), U(rB, c0-1)); column 0 / the dummy columns of thread 0 are U = BIAS
      const uint32_t rX = first ? B2 : recvX;
      // iteration 0 operands. Lane B has no cell here: up.hi = U(rA,c0-1), left.hi = U(rB,c0-1) (no gap), T.hi = 0 < both, so X.hi = U(rB,c0-1),
      // which is exactly lane B's `left` source for iteration 1, and up.hi its diagonal.
      uint32_t diag = (first ? (uint32_t) BIAS : prevRecvHi);                                // lo = U(rA-1, c0-1); hi = 0
      uint32_t up = __byte_perm(S[0], rH, 0x5432);                                           // lo = S[0].hi = U(rA-1, c0); hi = rH.lo
      uint32_t left = rH - (gvec & 0xffffu);
      uint32_t run = rX;
      uint32_t acc[C / 4];
#pragma unroll
      for (int q = 0; q < C / 4; ++q) acc[q] = 0;
      acc[0] = 0u - (((rH >> 16) - (rH & 0xffffu)) << 16);   // cancels lane B's iteration-0 term (X - up).hi = U(rB,c0-1) - U(rA,c0-1)
      uint32_t runPrev = 0, keepA = 0, vmax = NEG16x2;
      uint32_t wA[4], wB[4];                         // REV: packed prefix maxima of the two rows, one 16-byte group at a time (mirrored word order)
      uint32_t pav[4], pbv[4], pbLast = NEG16x2;     // FWD: partner words of the current 8-column block
      uint4* const stA = brev4 + (size_t) (s * 2 * WPT) * T + tid;   // REV: this step's groups (lane A rows first, then lane B)
      const uint4* const pbase = sm_part + (size_t) (cslot * 2 * WPT) * T + tid;   // FWD: this step's partner groups in the ring
      if (MODE == FWD && first && c0 == 1) {
        // column 0 is not inside thread 0's block: candidates (r, 0) = H[r][0] + element (m-r, n)
        const int vA = brev_at<C>(brev4, m - rA, delta, nactR, T) - m - BIAS;
        if (vA > best.val) { best.val = vA; best.row = rA; best.col = 0; best.bm = -rA; }
        if (hasB) {
          const int vB = brev_at<C>(brev4, m - rB, delta, nactR, T) - m - BIAS;
          if (vB > best.val) { best.val = vB; best.row = rB; best.col = 0; best.bm = -rB; }
        }
      }
#pragma unroll
      for (int j = 0; j <= C; ++j) {
        const uint32_t mm = __vminu2(colp[j] & rowpair, 0x00010001u);
        const uint32_t Tv = mm * 2u + diag;
        const uint32_t X = __vimax3_s16x2(Tv, up, left);
        {
          constexpr int unused = 0; (void) unused;
          const int q = (j == C) ? 0 : (j >> 2);
          const int sh = (j == C) ? 0 : 4 * (j & 3);
          acc[q] += X * (5u << sh);
          acc[q] -= up * (1u << sh);
          acc[q] -= left * (4u << sh);
        }
        run = __vmaxs2(run, X);
        if (MODE == REV) {
          // a row's prefix maxima leave in 16-byte groups as soon as the four words of a group exist (word index descends with j)
          if (j < C && (j & 1)) {
            const int q = (C - 1 - j) >> 1;
            wA[q & 3] = __byte_perm(run, runPrev, 0x5410);           // columns (j, j-1) of row rA
            if ((q & 3) == 0) stA[(q >> 2) * T] = make_uint4(wA[0], wA[1], wA[2], wA[3]);
          }
          if (j >= 2 && !(j & 1)) {
            const int q = (C - j) >> 1;
            wB[q & 3] = __byte_perm(run, runPrev, 0x7632);            // columns (j-1, j-2) of row rB
            if ((q & 3) == 0 && hasB) stA[(WPT + (q >> 2)) * T] = make_uint4(wB[0], wB[1], wB[2], wB[3]);
          }
          runPrev = run;
        }
        if (MODE == FWD) {
          if (j < C && (j & 7) == 0) {
            pbLast = (j == 0) ? NEG16x2 : pbv[3];
            const uint4 a4 = pbase[(j >> 3) * T];
            pav[0] = a4.x; pav[1] = a4.y; pav[2] = a4.z; pav[3] = a4.w;
            const uint4 b4 = pbase[(WPT + (j >> 3)) * T];
            pbv[0] = b4.x; pbv[1] = b4.y; pbv[2] = b4.z; pbv[3] = b4.w;
          }
          uint32_t pv;
          if (j == C) pv = __byte_perm(NEG16x2, pbv[3], 0x7610);                                          // A: none; B: column C-1
          else if ((j & 1) == 0) pv = __byte_perm(pav[(j & 7) >> 1], ((j & 7) == 0) ? pbLast : pbv[((j & 7) >> 1) - 1], 0x7610);   // A: lo of word e; B: hi of the word before
          else pv = __byte_perm(pav[(j & 7) >> 1], pbv[(j & 7) >> 1], 0x5432);                          // A: hi of word e; B: lo of word e
          vmax = __viaddmax_s16x2(run, pv, vmax);
        }
        if (j == 0) X0 = X;
        if (j > 0) S[j - 1] = X;
        if (j == C - 1) keepA = X;
        if (j < C) {
          const uint32_t nl = X - gvec;
          diag = up;
          if (j + 1 == C) { diag = up & 0xffff0000u; up = __byte_perm(nl, X, 0x5410); }      // lane A idles: up.lo = left.lo, T.lo = 0 -> zero nibble
          else up = __byte_perm(S[j + 1], X, 0x5432);
          left = nl;
        } else {
          handH = __byte_perm(keepA, X, 0x7610);       // (U(rA, c0+C-1), U(rB, c0+C-1))
          handX = run;
        }
      }
      prevRecvHi = rH >> 16;
      // ---- nibble rows --------------------------------------------------------------------------------------------------
      {
        uint32_t* dA = dirs + ((size_t) (s * 2 + 0) * T + tid) * WPT;
#pragma unroll
        for (int w = 0; w < WPT; ++w) dA[w] = __byte_perm(acc[2 * w], acc[2 * w + 1], 0x5410);
        if (hasB) {
          uint32_t* dB = dirs + ((size_t) (s * 2 + 1) * T + tid) * WPT;
#pragma unroll
          for (int w = 0; w < WPT; ++w) dB[w] = __byte_perm(acc[2 * w], acc[2 * w + 1], 0x7632);
        }
      }
      if (MODE == FWD) {
        const int off = m + 2 * BIAS;
        candA = (int) (int16_t) (vmax & 0xffffu) - off;
        candB = hasB ? (int) (int16_t) (vmax >> 16) - off : wf::NEG;
        candRX = rX; candRow = rA;
      }
    }
    if (MODE == FWD) {
      // A row of this pair improves the thread's best -> find the first column that attains the row's maximum (row rA before rB). Only
      // candidates that reach the best value any lane of the warp has seen so far can be the global arg-max (ties are decided later, in
      // row-major order, between the per-thread bests), which filters the many gradual improvements of threads far from the optimum.
      // The row values go through a small shared scratch so that the search is a short rolled loop.
      const int cm = max(candA, candB);
      gk = max(gk, __reduce_max_sync(0xffffffffu, cm));
      if ((candA > best.val || candB > best.val) && cm >= gk) {
        const int off = m + 2 * BIAS;
        const int rA = candRow, rB = candRow + 1;
        const uint4* const pbase = sm_part + (size_t) (cslot * 2 * WPT) * T + tid;
        uint32_t* sc = sm_scr + tid;
        sc[0] = X0;
#pragma unroll
        for (int j = 0; j < C; ++j) sc[(j + 1) * T] = S[j];
        if (candA > best.val && candA >= gk) {
          int rn = (int) (candRX & 0xffffu);
#pragma unroll 1
          for (int j = 0; j < C; ++j) {
            rn = max(rn, (int) (sc[j * T] & 0xffffu));
            const int pvv = (int) ((const int16_t*) (pbase + (j >> 3) * T))[j & 7];
            if (rn + pvv - off == candA) { best.val = candA; best.row = rA; best.col = c0 + j; best.bm = rn - rA - BIAS; break; }
          }
        }
        if (candB > best.val && candB >= gk) {
          int rn = (int) (candRX >> 16);
#pragma unroll 1
          for (int j = 0; j < C; ++j) {
            rn = max(rn, (int) (sc[(j + 1) * T] >> 16));
            const int pvv = (int) ((const int16_t*) (pbase + (WPT + (j >> 3)) * T))[j & 7];
            if (rn + pvv - off == candB) { best.val = candB; best.row = rB; best.col = c0 + j; best.bm = rn - rB - BIAS; break; }
          }
        }
      }
    }
  }
  if (MODE == FWD) cp_async_wait<0>();
  // corner H[m][n]: lane A of the last pair if m is odd, lane B if even
  {
    const int owner = (n - cstart) / C;
    __shared__ int sm_corner2;
    if (tid == owner) {
      const int jn = (n - cstart) % C;
      uint32_t v = (m & 1) ? (X0 & 0xffffu) : (S[0] >> 16);
#pragma unroll
      for (int j = 1; j < C; ++j)
        if (j == jn) v = (m & 1) ? (S[j - 1] & 0xffffu) : (S[j] >> 16);
      sm_corner2 = (int) v - m - BIAS;
    }
    __syncthreads();
    corner = sm_corner2;
    __syncthreads();
  }
}

}  // namespace wf2
