// msa.cu — batched per-cluster multiple sequence alignment + consensus, the device replacement for
// msa() (src/msa.h:185-239) as called per SV by assembleSplitReads (src/shortpe.h:185,252).
//
// Reference semantics reproduced bit-for-bit, ONE WARP PER CLUSTER (4 independent clusters per CTA):
//   * distanceMatrix: d[i][j] = lcs(si,sj)*100 / min(|si|,|sj|) (src/msa.h:10-44). LCS length is
//     computed bit-parallel (Allison-Dix/Hyyro: V' = (V + (V & M)) | (V & ~M), LCS = #zeros),
//     one lane per read pair; the value is the same LCS length the reference's DP returns.
//   * upgma: first strict maximum in row-major order, integer-average update, -1 masking (:46-89).
//   * palign: progressive gotoh(left,right) over the guide tree (:91-109). Nodes are evaluated in
//     creation order (children always precede parents), which yields the same alignments as the
//     reference's post-order recursion because each node is a pure function of its children.
//   * gotoh with AlignConfig<true,true> (free end gaps both ways), DnaScore(match,mismatch,go,ge)
//     (src/gotoh.h:71-174): exact s/v/h values, the 4 trace bitsets with the reference's tie rules
//     (bit3 before bit4; bit1/bit2 = "gap was opened here"), the h/v/s traceback state machine, and
//     _createAlignment's row order (src/align.h:202-229).
//   * _score: char compare when both sides have one row, else the float profile product summed
//     k1-outer/k2-inner in IEEE single without contraction and truncated (src/align.h:96-111);
//     _createProfile incl. the first..last aligned span rule (src/align.h:128-171).
//   * consensus: coverage threshold max(2,min(minCliqueSize,rows)), first-max vote over A,C,G,T,other,
//     gaps dropped (src/msa.h:111-173).
//
// DP parallelisation: anti-diagonal wavefront inside the warp — lane l owns C consecutive DP columns in
// registers and computes row (step - l) for them; the affine state (s, h) of its last column reaches lane l+1
// by shuffle, the vertical state v stays in registers. No block barriers anywhere; a CTA is just four
// independent warps sharing an SM slot. The 25-term float _score is evaluated once per pair of DISTINCT column
// profiles (columns whose integer counts agree have bit-identical float profiles) into an int8 table in shared
// memory and looked up per cell. Trace nibbles go to an L2-resident per-warp slab.
//
// Clusters of 33 .. max_reads (<= MSA_LARGE_MAXR) reads go to msa_large_kernel instead, ONE CTA PER CLUSTER: the LCS pairs are
// spread over all warps, UPGMA takes a CTA-wide arg-max per merge over the still-active nodes, and the guide tree is aligned level
// by level (a node's level = 1 + its deeper child's), each warp running the same DP, traceback and profile code as msa_kernel on one
// node of the level. Node alignments are not kept per node: every read owns two row buffers and a bank bit, a new node writes its
// rows into the other bank of each of its reads, and a node's row order ("rows of a1, then rows of a2") is a linked list over read
// ids, so the workspace grows as reads x columns.
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int MSA_WARPS = 4;        // independent clusters per CTA
#ifndef MSA_PER_SM
#define MSA_PER_SM 5
#endif
constexpr int MSA_T = 32 * MSA_WARPS;
constexpr int MSA_MAXR = 32;        // reads per cluster (reference default maxReadPerSV = 20)
constexpr int MSA_LCAP = 1023;      // max alignment columns (DP has LCAP+1 columns)
constexpr int MSA_N = 2 * MSA_MAXR + 1;
constexpr int MSA_NEGINF = 1000000; // DnaScore::inf (src/align.h:21)
constexpr int LCS_W = 8;            // 32-bit words per read in the bit-parallel LCS (<= 256 bp)
constexpr int MSA_UMAX = 64;        // distinct column profiles per side the de-duplication tracks (more: every column is its own profile)
constexpr int MSA_SSMEM = MSA_UMAX * MSA_UMAX;  // score-table entries that fit shared memory; larger tables live in the warp's slab
constexpr int MSA_HASH = 128;       // open-addressing slots for the profile de-duplication
constexpr int MSA_LARGE_MAXR = DGPU_MSA_LARGE_MAXR;  // reads per cluster of msa_large_kernel: 10-bit profile-key fields, int16 node ids
constexpr int MSA_LN = 2 * MSA_LARGE_MAXR + 1;
constexpr int MSA_LWARPS = 8;       // warps of one msa_large_kernel CTA (one cluster)
constexpr int MSA_LT = 32 * MSA_LWARPS;

constexpr int ST_OK = 0, ST_TOO_MANY = 1, ST_TOO_LONG = 2, ST_BAD_CHAR = 3;

struct MsaArgs {
  const uint8_t* seqs;
  const uint32_t* read_off;
  const uint32_t* read_len;
  const uint32_t* cluster_off;  // nclusters+1 indices into the read arrays
  uint32_t nclusters;
  int match, mismatch, go, ge, min_clique;
  int max_reads;            // clusters above it: status 1; 33 .. max_reads: msa_large_kernel's
  uint8_t* cons;
  const uint64_t* cons_off;
  uint32_t* cons_len;
  uint32_t* n_rows;
  uint32_t* status;
  uint8_t* aln;             // optional root alignment dump
  const uint64_t* aln_off;
  uint32_t* aln_cols;
  uint8_t* work;            // one slab per warp
  size_t work_stride;
  size_t off_prof, off_trace, off_lcs, off_keys, off_src, off_bnd, off_tab, off_spans;
  size_t aln_cap;           // bytes of node alignment storage per warp (at slab offset 0)
};

struct NodeAln {
  const uint8_t* p;  // rows x L, row stride L
  int R, L;
  __device__ __forceinline__ const uint8_t* row(int r) const { return p + (size_t) r * L; }
};

// The rows of a msa_large_kernel node: row r is read rid[r]'s buffer in its current bank.
struct NodeRows {
  const uint8_t* buf;    // per read: two row buffers of MSA_LCAP + 1 bytes
  const int16_t* rid;    // read id of every row, in row order
  const uint8_t* bank;   // per read: which of its two buffers holds its current row
  int R, L;
  __device__ __forceinline__ const uint8_t* row(int r) const { const int k = rid[r]; return buf + ((size_t) k * 2 + bank[k]) * (MSA_LCAP + 1); }
};

// Per-warp state of the profile scoring, in shared memory
struct ProfSm {
  union {
    int8_t S[MSA_UMAX * MSA_UMAX];         // exact _score per pair of distinct column profiles
    struct {                               // profile de-duplication (finished before S is built)
      unsigned long long hkey[MSA_HASH];
      int hval[MSA_HASH];
      int hcount;
    } h;
  } t;
  unsigned long long uniq1[MSA_UMAX], uniq2[MSA_UMAX];
};

// Per-warp shared state (about 10 KB, so that five 4-warp CTAs fit one SM)
constexpr int MSA_TRI = MSA_N * (MSA_N - 1) / 2;
struct WarpSm {
  int8_t d[MSA_TRI];                       // guide-tree similarity matrix, upper triangle (values -2..100)
  int8_t par[MSA_N], lc[MSA_N], rc[MSA_N];
  uint8_t nodeR[MSA_N];
  uint16_t nodeL[MSA_N];
  uint32_t nodeP[MSA_N];                   // leaf: offset into the read arena; inner node: offset into the warp's slab
  int16_t first1[MSA_MAXR], last1[MSA_MAXR], first2[MSA_MAXR], last2[MSA_MAXR];
  uint32_t win[64];                        // traceback window: 32 rows x 2 trace words
  union {
    uint32_t peq[MSA_MAXR * 5 * LCS_W];    // LCS phase
    ProfSm g;
  } u;
};

// Shared state of one msa_large_kernel CTA (one cluster of up to MSA_LARGE_MAXR reads, MSA_LN nodes)
struct LargeSm {
  int16_t lc[MSA_LN], rc[MSA_LN];
  uint16_t nodeR[MSA_LN], nodeL[MSA_LN];
  int16_t head[MSA_LN], tail[MSA_LN];      // a node's rows: the linked list head .. tail over next[]
  int16_t lev[MSA_LN], order[MSA_LN];      // tree level of every node; inner nodes sorted by level
  int16_t act[2][MSA_LN];                  // UPGMA: the active nodes in increasing id order (double-buffered)
  int16_t levoff[MSA_LARGE_MAXR + 2];
  int16_t next[MSA_LARGE_MAXR], first[MSA_LARGE_MAXR], last[MSA_LARGE_MAXR];  // per read: next row, first/last aligned column
  uint8_t bank[MSA_LARGE_MAXR + 1];
  unsigned long long red[MSA_LWARPS];
  int status;
  uint32_t win[MSA_LWARPS][64];
  ProfSm g[MSA_LWARPS];
};

__device__ __forceinline__ int tri(int i, int j, int n) {  // i < j < n
  return i * (2 * n - i - 1) / 2 + (j - i - 1);
}
__device__ __forceinline__ int tri(int i, int j) { return tri(i, j, MSA_N); }

// _createProfile (src/align.h:128-171) in integer form: key[j] = the six integers column j's profile is made of (counts of
// A,C,G,T,N and the covering-row count over the first..last aligned span of each row, KB bits each: 6 while a node has at most
// 63 rows, 10 up to 1023). The float profile p[k][j] = count_k / rows is a pure function of the key, so two columns with equal
// keys have bit-identical profiles — which is what the score table exploits. The '-' row of the reference's profile is never read
// by _score. Rows: NodeAln or NodeRows.
template <int KB, class Rows>
__device__ void make_profile_keys(const Rows& a, const int16_t* first, const int16_t* last, unsigned long long* key, int lane) {
  for (int j = lane; j < a.L; j += 32) {
    int cnt[5] = {0, 0, 0, 0, 0};
    int sum = 0;
    for (int r = 0; r < a.R; ++r) {
      int f = first[r], l = last[r];
      if (f < 0) { f = -1; l = a.L; }  // all-gap row: the reference's initial values cover everything
      if (f <= j && j <= l) {
        ++sum;
        uint8_t c = a.row(r)[j];
        if (c == 'A' || c == 'a') ++cnt[0];
        else if (c == 'C' || c == 'c') ++cnt[1];
        else if (c == 'G' || c == 'g') ++cnt[2];
        else if (c == 'T' || c == 't') ++cnt[3];
        else if (c == 'N' || c == 'n') ++cnt[4];
        else if (c == '-') {}
        else --sum;
      }
    }
    unsigned long long kk = (unsigned long long) (uint32_t) sum;
#pragma unroll
    for (int k = 0; k < 5; ++k) kk = (kk << KB) | (unsigned long long) (uint32_t) cnt[k];
    key[j] = kk + 1ull;  // never 0: 0 marks an empty hash slot
  }
  __syncwarp();
}

// Map every column to the index of its distinct profile through a small open-addressing table.
// Returns the number of distinct profiles, or -1 if there are more than MSA_UMAX (the caller then treats every column as its own profile).
__device__ int dedup_profiles(ProfSm& g, const unsigned long long* key, int L, uint16_t* ids, unsigned long long* uniq, int lane) {
  for (int i = lane; i < MSA_HASH; i += 32) { g.t.h.hkey[i] = 0ull; g.t.h.hval[i] = -1; }
  if (lane == 0) g.t.h.hcount = 0;
  __syncwarp();
  bool overflow = false;
  for (int j0 = 0; j0 < L; j0 += 32) {
    const int j = j0 + lane;
    if (j < L) {
      const unsigned long long k = key[j];
      uint32_t h = (uint32_t) ((k * 0x9E3779B97F4A7C15ull) >> 57);  // 7 bits
      int id = -1;
      for (int probe = 0; probe < MSA_HASH; ++probe) {
        const unsigned long long prev = atomicCAS(&g.t.h.hkey[h], 0ull, k);
        if (prev == 0ull) {  // this lane created the slot
          const int nid = atomicAdd(&g.t.h.hcount, 1);
          if (nid < MSA_UMAX) uniq[nid] = k;
          __threadfence_block();
          atomicExch(&g.t.h.hval[h], nid);
          id = nid;
          break;
        }
        if (prev == k) {  // somebody (maybe in this very instruction) owns the slot: wait for its id
          int v;
          do { v = atomicAdd(&g.t.h.hval[h], 0); } while (v < 0);
          id = v;
          break;
        }
        h = (h + 1) & (MSA_HASH - 1);
      }
      if (id < 0 || id >= MSA_UMAX) overflow = true; else ids[j] = (uint16_t) id;
    }
    __syncwarp();
  }
  overflow = __any_sync(0xffffffffu, overflow);
  const int U = g.t.h.hcount;
  __syncwarp();
  return (overflow || U > MSA_UMAX) ? -1 : U;
}

// Exact _score (src/align.h:104-109) for every pair of distinct profiles: S[u1 * U2 + u2] (fits int8: |score| <= max(|match|,|mismatch|)).
// The 25 products are summed k1-outer / k2-inner in IEEE single without contraction, then truncated, as the reference does per cell.
// KB: the key field width of make_profile_keys.
template <int KB>
__device__ void build_score_table(const unsigned long long* uniq1, int U1, const unsigned long long* uniq2, int U2, int match, int mismatch, int8_t* S, int lane) {
  const float fm = (float) match, fx = (float) mismatch;
  constexpr unsigned long long mask = (1ull << KB) - 1ull;
  for (int x = lane; x < U1 * U2; x += 32) {
    const int u1 = x / U2, u2 = x % U2;
    float p1[5], p2[5];
    unsigned long long k1 = uniq1[u1] - 1ull, k2 = uniq2[u2] - 1ull;
    const float s1 = (float) (uint32_t) (k1 >> (5 * KB)), s2 = (float) (uint32_t) (k2 >> (5 * KB));
#pragma unroll
    for (int k = 4; k >= 0; --k) {
      p1[k] = __fdiv_rn((float) (uint32_t) (k1 & mask), s1); k1 >>= KB;
      p2[k] = __fdiv_rn((float) (uint32_t) (k2 & mask), s2); k2 >>= KB;
    }
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 5; ++a)
#pragma unroll
      for (int b = 0; b < 5; ++b) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(p1[a], p2[b]), (a == b) ? fm : fx));
    S[x] = (int8_t) (int) acc;
  }
  __syncwarp();
}

// The DP of gotoh() as a warp wavefront over one strip of 32*C columns starting at cbase: lane l owns columns
// cbase + l*C .. cbase + l*C + C-1 (column 0 of the matrix is the fixed boundary s = v = 0, h = -inf). Strips after the
// first take the (s, h) of the column left of them from bnd_in[row] and every strip that has a successor leaves its last
// column in bnd_out[row]. Writes one trace nibble per cell: bit0 = bit1, bit1 = bit2, bit2 = bit3, bit3 = bit4 of
// src/gotoh.h:135-138. tr: row-major, rowwords words per row, cell (r,c) at word c/8, nibble c%8.
// The substitution score of cell (r,c) is S[id1[r-1] * sstride + id2[c-1]].
#define MSA_SETBIT_GT(dw, a, b, imm) asm("{.reg .pred p; setp.gt.s32 p, %1, %2; @p or.b32 %0, %0, %3;}" : "+r"(dw) : "r"(a), "r"(b), "r"(imm))
#define MSA_SETBIT_EQ(dw, a, b, imm) asm("{.reg .pred p; setp.eq.s32 p, %1, %2; @p or.b32 %0, %0, %3;}" : "+r"(dw) : "r"(a), "r"(b), "r"(imm))

// BIG = false: the score table is in shared memory (32-bit addressing, one add + one load per cell);
// BIG = true: it is in the warp's global slab (more than MSA_SSMEM distinct profile pairs; rare).
// Trace bit 3 is stored as plain (s == v); the traceback tests bit 2 (s == h) first, as the reference's else-if does.
template <int C, bool BIG>
__device__ __noinline__ void gotoh_wave(const int m, const int n, const int o, const int e, uint32_t* __restrict__ tr, const int rowwords,
                                        const uint16_t* __restrict__ id1, const uint16_t* __restrict__ id2, const int8_t* S, const int sstride,
                                        const int cbase, const int2* __restrict__ bnd_in, int2* __restrict__ bnd_out, const int lane) {
  const int c0 = cbase + lane * C;
  constexpr int WPT = (C + 7) / 8;
  const bool owns = c0 <= n;
  const bool has_next = cbase + 32 * C <= n;
  const int nact = min(32, (n - cbase) / C + 1);  // lanes that own a column <= n
  const uint32_t sbase = BIG ? 0u : (uint32_t) __cvta_generic_to_shared(S);

  uint32_t cx[C];   // the column's distinct-profile index (plus the table's shared-memory address when !BIG)
  int vgo[C], vge[C];  // vertical gap costs: zero in the last column (free end gaps, AlignConfig<true,true>)
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int c = c0 + j;
    cx[j] = sbase + ((c >= 1 && c <= n) ? (uint32_t) id2[c - 1] : 0u);
    vgo[j] = (c == n) ? 0 : o;
    vge[j] = (c == n) ? 0 : e;
  }
  int sprev[C], vprev[C];
#pragma unroll
  for (int j = 0; j < C; ++j) { sprev[j] = 0; vprev[j] = -MSA_NEGINF; }
  // row 0: bit3 for every column >= 1 (src/gotoh.h:113-117)
  if (owns) {
    if (C >= 8) {
#pragma unroll
      for (int w = 0; w < WPT; ++w) {
        uint32_t bits = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) { const int c = c0 + 8 * w + q; if (c >= 1 && c <= n) bits |= 4u << (4 * q); }
        if (c0 + 8 * w <= n) tr[(c0 >> 3) + w] = bits;
      }
    } else {  // C == 4: half a trace word per lane
      uint32_t bits = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) { const int c = c0 + q; if (c >= 1 && c <= n) bits |= 4u << (4 * q); }
      ((uint16_t*) tr)[c0 >> 2] = (uint16_t) bits;
    }
  }
  int lastS = 0, lastH = 0, prevRecvS = 0;
  const int nsteps = m + nact - 1;
  int2 nextb = make_int2(0, 0);
  if (cbase > 0 && lane == 0) nextb = bnd_in[1];
  // the row profile index is fetched one step ahead of its use
  int nextid = 0;
  if (owns && lane == 0) nextid = id1[0];
  for (int st = 1; st <= nsteps; ++st) {
    int recvS = __shfl_up_sync(0xffffffffu, lastS, 1);
    int recvH = __shfl_up_sync(0xffffffffu, lastH, 1);
    if (cbase > 0 && lane == 0) {
      recvS = nextb.x; recvH = nextb.y;
      if (st < m) nextb = bnd_in[st + 1];
    }
    const int r = st - lane;
    const int roff = nextid * sstride;
    if (owns && r >= 0 && r < m) nextid = id1[r];  // for row r + 1
    if (r >= 1 && r <= m && owns) {
      const int er = (r == m) ? 0 : e;
      const int orr = (r == m) ? 0 : o;
      int sc[C];
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (BIG) sc[j] = (int) S[roff + (int) cx[j]];
        else asm("ld.shared.s8 %0, [%1];" : "=r"(sc[j]) : "r"(cx[j] + (uint32_t) roff));
      }
      int sleft = recvS, hleft = recvH, diag = prevRecvS;
      uint32_t dw[WPT];
#pragma unroll
      for (int w = 0; w < WPT; ++w) dw[w] = 0;
#pragma unroll
      for (int j = 0; j < C; ++j) {
        const int vext = vprev[j] + vge[j];
        const int vopen = sprev[j] + vgo[j];
        int v = max(vopen, vext);
        const int hext = hleft + er;
        const int hopen = sleft + orr;
        int h = max(hopen, hext);
        int s = max(max(diag + sc[j], h), v);
        if (j == 0) {  // column 0 of the matrix (src/gotoh.h:118-123) sits in lane 0 of the first strip
          uint32_t b0 = 0;
          MSA_SETBIT_GT(b0, hopen, hext, 1);
          MSA_SETBIT_GT(b0, vopen, vext, 2);
          MSA_SETBIT_EQ(b0, s, h, 4);
          MSA_SETBIT_EQ(b0, s, v, 8);
          const bool z = (c0 == 0);
          s = z ? 0 : s; v = z ? 0 : v; h = z ? -MSA_NEGINF : h;
          dw[0] = z ? 8u : b0;
        } else {
          MSA_SETBIT_GT(dw[j >> 3], hopen, hext, 1 << ((j & 7) * 4));
          MSA_SETBIT_GT(dw[j >> 3], vopen, vext, 2 << ((j & 7) * 4));
          MSA_SETBIT_EQ(dw[j >> 3], s, h, 4 << ((j & 7) * 4));
          MSA_SETBIT_EQ(dw[j >> 3], s, v, 8 << ((j & 7) * 4));
        }
        diag = sprev[j];
        sprev[j] = s; vprev[j] = v;
        sleft = s; hleft = h;
      }
      lastS = sleft; lastH = hleft;
      if (C >= 8) {
        uint32_t* drow = tr + (size_t) r * rowwords + (c0 >> 3);
#pragma unroll
        for (int w = 0; w < WPT; ++w)
          if (c0 + 8 * w <= n) drow[w] = dw[w];
      } else {
        ((uint16_t*) (tr + (size_t) r * rowwords))[c0 >> 2] = (uint16_t) dw[0];
      }
      if (has_next && lane == 31) bnd_out[r] = make_int2(lastS, lastH);
    }
    prevRecvS = recvS;
  }
  __syncwarp();
}

// Substitution scores: _score (src/align.h:96-111) compares raw characters when both sides hold one row and otherwise
// multiplies the float column profiles. Either way the score depends only on (kind of row column, kind of column column):
// number the kinds (ids1, ids2) and tabulate. Returns the table (g.t.S, or bigtab when it does not fit there) and its row stride.
// first/last: the aligned span of every row (read only when a side has more than one row); KB: see make_profile_keys.
template <int KB, class Rows>
__device__ __forceinline__ const int8_t* score_table(const Rows& a1, const int16_t* first1, const int16_t* last1,
                                                     const Rows& a2, const int16_t* first2, const int16_t* last2, const MsaArgs& A, ProfSm& g,
                                                     unsigned long long* keys1, unsigned long long* keys2, uint16_t* ids1, uint16_t* ids2,
                                                     int8_t* bigtab, int& sstride, const int lane) {
  const int m = a1.L, n = a2.L;
  if (a1.R == 1 && a2.R == 1) {
    const uint8_t *p1 = a1.row(0), *p2 = a2.row(0);
    for (int j = lane; j < m; j += 32) { const uint8_t ch = p1[j]; ids1[j] = (uint16_t) (dna_code(ch) + ((ch & 0x20) ? 5u : 0u)); }
    for (int j = lane; j < n; j += 32) { const uint8_t ch = p2[j]; ids2[j] = (uint16_t) (dna_code(ch) + ((ch & 0x20) ? 5u : 0u)); }
    for (int x = lane; x < 100; x += 32) g.t.S[x] = (int8_t) ((x / 10 == x % 10) ? A.match : A.mismatch);
    sstride = 10;
    __syncwarp();
    return g.t.S;
  }
  make_profile_keys<KB>(a1, first1, last1, keys1, lane);
  make_profile_keys<KB>(a2, first2, last2, keys2, lane);
  const unsigned long long* u1 = g.uniq1;
  const unsigned long long* u2 = g.uniq2;
  int U1 = dedup_profiles(g, keys1, m, ids1, g.uniq1, lane);
  if (U1 < 0) { for (int j = lane; j < m; j += 32) ids1[j] = (uint16_t) j; U1 = m; u1 = keys1; }
  int U2 = dedup_profiles(g, keys2, n, ids2, g.uniq2, lane);
  if (U2 < 0) { for (int j = lane; j < n; j += 32) ids2[j] = (uint16_t) j; U2 = n; u2 = keys2; }
  __syncwarp();
  int8_t* Sw = (U1 * U2 <= MSA_SSMEM) ? g.t.S : bigtab;
  build_score_table<KB>(u1, U1, u2, U2, A.match, A.mismatch, Sw, lane);
  sstride = U2;
  return Sw;
}

__device__ __forceinline__ void gotoh_dp(const int m, const int n, const MsaArgs& A, uint32_t* tr, const int rowwords,
                                         const uint16_t* id1, const uint16_t* id2, const int8_t* S, const int sstride, const bool big, int2* bnd, const int lane) {
  const int o = A.go + A.ge, e = A.ge;
  if (n + 1 <= 32 * 4) {
    if (!big) gotoh_wave<4, false>(m, n, o, e, tr, rowwords, id1, id2, S, sstride, 0, nullptr, nullptr, lane);
    else gotoh_wave<4, true>(m, n, o, e, tr, rowwords, id1, id2, S, sstride, 0, nullptr, nullptr, lane);
  } else {
    int2* bin = bnd;
    int2* bout = bnd + (MSA_LCAP + 1);
    for (int cbase = 0; cbase <= n; cbase += 32 * 8) {
      if (!big) gotoh_wave<8, false>(m, n, o, e, tr, rowwords, id1, id2, S, sstride, cbase, bin, bout, lane);
      else gotoh_wave<8, true>(m, n, o, e, tr, rowwords, id1, id2, S, sstride, cbase, bin, bout, lane);
      int2* t = bin; bin = bout; bout = t;
    }
  }
}

// bit-parallel LCS length of reads a (Peq masks in pa[5][LCS_W]) and b (codes 0..4)
__device__ int lcs_bitpar(const uint32_t* pa, int la, const uint8_t* b, int lb) {
  const int nw = (la + 31) >> 5;
  uint32_t V[LCS_W];
#pragma unroll
  for (int w = 0; w < LCS_W; ++w) V[w] = 0xffffffffu;
  for (int j = 0; j < lb; ++j) {
    const uint32_t code = dna_code(b[j]);
    uint32_t carry = 0;
#pragma unroll
    for (int w = 0; w < LCS_W; ++w) {
      if (w < nw) {
        const uint32_t M = (code < 5) ? pa[code * LCS_W + w] : 0u;
        const uint32_t u = V[w] & M;
        const uint32_t s1 = V[w] + u;
        const uint32_t c1 = s1 < u;
        const uint32_t s2 = s1 + carry;
        const uint32_t c2 = s2 < carry;
        V[w] = s2 | (V[w] & ~M);
        carry = c1 | c2;
      }
    }
  }
  int zeros = 0;
#pragma unroll
  for (int w = 0; w < LCS_W; ++w) {
    if (w < nw) {
      uint32_t x = ~V[w];
      if (w == nw - 1 && (la & 31)) x &= (1u << (la & 31)) - 1u;
      zeros += __popc(x);
    }
  }
  return zeros;
}

// plain LCS DP for a pair of two reads longer than the bit vectors (e.g. 2 x 300 bp libraries); row: lb + 1 ints of scratch
__device__ __forceinline__ int lcs_dp(const uint8_t* a, int la, const uint8_t* b, int lb, int* row) {
  for (int c = 0; c <= lb; ++c) row[c] = 0;
  for (int i = 1; i <= la; ++i) {
    int diag = 0;
    const uint8_t ca = a[i - 1];
    for (int c = 1; c <= lb; ++c) {
      const int up = row[c];
      row[c] = (ca == b[c - 1]) ? diag + 1 : max(up, row[c - 1]);
      diag = up;
    }
  }
  return row[lb];
}

// read r's status bits, this lane's share: 2 = empty or longer than MSA_LCAP, 1 = a byte outside ACGTN (the reference's float
// profile is NaN there)
__device__ __forceinline__ int read_flags(const MsaArgs& A, const uint32_t r, const int lane) {
  const uint32_t L = A.read_len[r];
  int bad = (L > MSA_LCAP || L == 0) ? 2 : 0;
  const uint8_t* s = A.seqs + A.read_off[r];
  for (uint32_t j = lane; j < L; j += 32)
    if (dna_code(s[j]) > 4) bad |= 1;
  return bad;
}

// Peq masks of one read for lcs_bitpar (one warp; reads longer than the bit vectors get none)
__device__ __forceinline__ void build_peq(const uint8_t* s, const uint32_t L, uint32_t* peq, const int lane) {
  if (L > 32 * LCS_W) return;
  for (uint32_t j0 = 0; j0 < L; j0 += 32) {
    uint32_t j = j0 + lane;
    uint32_t code = (j < L) ? dna_code(s[j]) : 7u;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      unsigned b = __ballot_sync(0xffffffffu, code == (uint32_t) k);
      if (lane == 0) peq[k * LCS_W + (j0 >> 5)] = b;
    }
  }
}

// traceback (src/gotoh.h:141-167) of the m x n trace the warp's gotoh_dp left in tr: lane 0 runs the state machine over a window of
// trace words the warp stages in win (shared memory, 32 rows x 2 words following the diagonal); once the path reaches row 0 or
// column 0 the rest is a pure gap run (row 0 holds only bit3, column 0 only bit4) and is filled in by all lanes.
// src1/src2[k]: the row / column of alignment column L-1-k (-1: gap). Returns L.
__device__ __forceinline__ int msa_traceback(const uint32_t* tr, const int rowwords, const int m, const int n, uint32_t* win,
                                             int16_t* src1, int16_t* src2, const int lane) {
  int row = m, col = n, k = 0, tst = 0;  // tst: 0 = 's', 1 = 'h', 2 = 'v'
  while (row > 0 && col > 0) {
    {
      const int ri = row - lane;
      const int wi = max(col - lane, 0) >> 3;
      uint32_t w1 = 0, w0 = 0;
      if (ri >= 0) {
        const uint32_t* trow = tr + (size_t) ri * rowwords;
        w1 = __ldcg(trow + wi);
        if (wi > 0) w0 = __ldcg(trow + wi - 1);
      }
      win[2 * lane] = w0; win[2 * lane + 1] = w1;
    }
    __syncwarp();
    if (lane == 0) {
      const int row0 = row, col0 = col;
      while (row > 0 && col > 0) {
        const int i = row0 - row;
        if (i >= 32) break;
        const int wsel = (col >> 3) - (max(col0 - i, 0) >> 3) + 1;
        if (wsel < 0 || wsel > 1) break;
        const uint32_t nb = (win[2 * i + wsel] >> ((col & 7) * 4)) & 0xfu;
        // branch-free form of the reference's loop: an 's' state that sees bit3/bit4 switches to 'h'/'v' and that
        // state consumes the same cell, so every iteration emits exactly one alignment column
        const int mode = (tst != 0) ? tst : ((nb & 4u) ? 1 : ((nb & 8u) ? 2 : 0));
        const int drow = (mode != 1), dcol = (mode != 2);
        row -= drow; col -= dcol;
        src1[k] = (int16_t) (drow ? row : -1);
        src2[k] = (int16_t) (dcol ? col : -1);
        ++k;
        tst = (mode == 0 || ((nb >> (mode - 1)) & 1u)) ? 0 : mode;
      }
    }
    __syncwarp();   // lane 0's reads of the staged window are done before the next refill (racecheck: write-after-read on win)
    row = __shfl_sync(0xffffffffu, row, 0);
    col = __shfl_sync(0xffffffffu, col, 0);
    k = __shfl_sync(0xffffffffu, k, 0);
  }
  for (int t = lane; t < col; t += 32) { src1[k + t] = -1; src2[k + t] = (int16_t) (col - 1 - t); }
  for (int t = lane; t < row; t += 32) { src1[k + t] = (int16_t) (row - 1 - t); src2[k + t] = -1; }
  __syncwarp();
  return k + row + col;
}

// gapped consensus, columns j0, j0 + stride, ... (src/msa.h:111-173): rows covering j (first..last aligned span) vote, first
// maximum over A,C,G,T,other; '-' below the coverage threshold or when "other" wins
template <class Rows>
__device__ __forceinline__ void consensus_columns(const Rows& ra, const int16_t* first, const int16_t* last, const int thr, uint8_t* gapped,
                                                  const int j0, const int stride) {
  for (int j = j0; j < ra.L; j += stride) {
    int cov = 0;
    int cnt[5] = {0, 0, 0, 0, 0};
    for (int r = 0; r < ra.R; ++r) {
      if (first[r] >= 0 && first[r] <= j && j <= last[r]) {
        ++cov;
        const uint8_t c = ra.row(r)[j];
        if (c == 'A' || c == 'a') ++cnt[0];
        else if (c == 'C' || c == 'c') ++cnt[1];
        else if (c == 'G' || c == 'g') ++cnt[2];
        else if (c == 'T' || c == 't') ++cnt[3];
        else ++cnt[4];
      }
    }
    uint8_t g = '-';
    if (cov >= thr) {
      int mi = 0;
#pragma unroll
      for (int x = 1; x < 5; ++x) if (cnt[x] > cnt[mi]) mi = x;
      if (mi == 0) g = 'A'; else if (mi == 1) g = 'C'; else if (mi == 2) g = 'G'; else if (mi == 3) g = 'T';
    }
    gapped[j] = g;
  }
}

// ordered compaction of the non-gap consensus letters gapped[0..L) into o (ballot prefix, one warp); returns their number
__device__ __forceinline__ uint32_t compact_consensus(const uint8_t* gapped, const int L, uint8_t* o, const int lane) {
  uint32_t k = 0;
  for (int j0 = 0; j0 < L; j0 += 32) {
    const int j = j0 + lane;
    const uint8_t g = (j < L) ? gapped[j] : (uint8_t) '-';
    const unsigned b = __ballot_sync(0xffffffffu, g != '-');
    if (g != '-') o[k + __popc(b & ((1u << lane) - 1u))] = g;
    k += __popc(b);
  }
  return k;
}

__global__ void __launch_bounds__(MSA_T, MSA_PER_SM) msa_kernel(MsaArgs A) {
  extern __shared__ __align__(16) uint8_t msa_smem[];
  WarpSm* wsm = reinterpret_cast<WarpSm*>(msa_smem);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  WarpSm& w = wsm[wib];
  const uint32_t gwarp = blockIdx.x * MSA_WARPS + wib, nwarps = gridDim.x * MSA_WARPS;
  uint8_t* slab = A.work + (size_t) gwarp * A.work_stride;
  uint8_t* alnbuf = slab;
  uint8_t* gapped = slab + A.off_prof;
  uint16_t* ids1 = (uint16_t*) (slab + A.off_prof + (MSA_LCAP + 1));
  uint16_t* ids2 = ids1 + (MSA_LCAP + 1);
  int8_t* bigtab = (int8_t*) (slab + A.off_tab);
  uint32_t* tr = (uint32_t*) (slab + A.off_trace);
  int* lcsrow = (int*) (slab + A.off_lcs);                          // 32 DP rows (one per lane) for the long-pair LCS
  int8_t* lcstmp = (int8_t*) (lcsrow + 32 * (MSA_LCAP + 2));      // its results, before they enter the similarity matrix
  unsigned long long* keys1 = (unsigned long long*) (slab + A.off_keys);
  unsigned long long* keys2 = keys1 + (MSA_LCAP + 1);
  int16_t* src1 = (int16_t*) (slab + A.off_src);
  int16_t* src2 = src1 + (2 * MSA_LCAP + 4);
  int2* bnd = (int2*) (slab + A.off_bnd);
  int16_t* spans = (int16_t*) (slab + A.off_spans);  // per node: first[MSA_MAXR], last[MSA_MAXR]

  for (uint32_t cl = gwarp; cl < A.nclusters; cl += nwarps) {
    __syncwarp();
    const uint32_t rbeg = A.cluster_off[cl], rend = A.cluster_off[cl + 1];
    const int num = (int) (rend - rbeg);
    int status = ST_OK;
    if (num > A.max_reads) status = ST_TOO_MANY;
    else if (num > MSA_MAXR) continue;  // msa_large_kernel's
    if (status == ST_OK) {
      int bad = 0;
      for (int i = 0; i < num; ++i) bad |= read_flags(A, rbeg + i, lane);
      bad = __reduce_or_sync(0xffffffffu, (unsigned) bad);
      if (bad & 2) status = ST_TOO_LONG; else if (bad & 1) status = ST_BAD_CHAR;
    }
    if (status != ST_OK || num == 0) {
      if (lane == 0) { A.status[cl] = status; A.cons_len[cl] = 0; A.n_rows[cl] = 0; if (A.aln_cols) A.aln_cols[cl] = 0; }
      continue;
    }
    const int N = 2 * num + 1;

    // ---- distance matrix (src/msa.h:32-44, :190-195) ---------------------------------
    for (int x = lane; x < MSA_TRI; x += 32) w.d[x] = -1;
    for (int x = lane; x < N; x += 32) { w.par[x] = -1; w.lc[x] = -1; w.rc[x] = -1; }
    for (int x = lane; x < num * 5 * LCS_W; x += 32) w.u.peq[x] = 0;
    __syncwarp();
    for (int i = 0; i < num; ++i) build_peq(A.seqs + A.read_off[rbeg + i], A.read_len[rbeg + i], &w.u.peq[i * 5 * LCS_W], lane);
    __syncwarp();
    {
      const int npairs = num * (num - 1) / 2;
      for (int pidx = lane; pidx < npairs; pidx += 32) {
        int i = 0, rem = pidx;  // unrank (i<j) in row-major order
        while (rem >= num - 1 - i) { rem -= num - 1 - i; ++i; }
        const int j = i + 1 + rem;
        const int li = (int) A.read_len[rbeg + i], lj = (int) A.read_len[rbeg + j];
        int l;
        if (li <= 32 * LCS_W) l = lcs_bitpar(&w.u.peq[i * 5 * LCS_W], li, A.seqs + A.read_off[rbeg + j], lj);
        else if (lj <= 32 * LCS_W) l = lcs_bitpar(&w.u.peq[j * 5 * LCS_W], lj, A.seqs + A.read_off[rbeg + i], li);
        else l = -2;  // long pair: plain DP below
        w.d[tri(i, j)] = (l >= 0) ? (int8_t) ((l * 100) / min(li, lj)) : (int8_t) -2;
      }
      __syncwarp();
      {  // plain LCS DP for pairs of two long reads (reads beyond the 256-column bit vectors, e.g. 2 x 300 bp libraries): one pair per lane,
         // each lane with its own DP row in the warp's slab
        int* myrow = lcsrow + (size_t) lane * (MSA_LCAP + 2);
        int seen = 0;
        for (int i = 0; i < num; ++i)
          for (int j = i + 1; j < num; ++j)
            if (w.d[tri(i, j)] == -2) {
              if ((seen++ & 31) != lane) continue;
              const int li = (int) A.read_len[rbeg + i], lj = (int) A.read_len[rbeg + j];
              const int l = lcs_dp(A.seqs + A.read_off[rbeg + i], li, A.seqs + A.read_off[rbeg + j], lj, myrow);
              lcstmp[tri(i, j)] = (int8_t) ((l * 100) / min(li, lj));   // into the matrix after the scan: the other lanes still count the -2 marks
            }
        __syncwarp();
        for (int x = lane; x < MSA_TRI; x += 32)
          if (w.d[x] == -2) w.d[x] = lcstmp[x];
      }
      __syncwarp();
    }

    // ---- UPGMA (src/msa.h:46-89) ---------------------------------------------------------
    int nn = num;
    for (; nn < N; ++nn) {
      unsigned long long key = 0;
      for (int x = lane; x < nn * nn; x += 32) {
        int i = x / nn, j = x % nn;
        if (j > i) {
          int v = w.d[tri(i, j)];
          unsigned long long k2 = ((unsigned long long) (uint32_t) (v + 2) << 32) | (uint32_t) (0x7fffffff - (i * MSA_N + j));
          key = k2 > key ? k2 : key;
        }
      }
#pragma unroll
      for (int dd = 16; dd >= 1; dd >>= 1) {
        unsigned long long y = __shfl_xor_sync(0xffffffffu, key, dd);
        key = y > key ? y : key;
      }
      const int dMax = (int) (uint32_t) (key >> 32) - 2;
      if (key == 0 || dMax == -1) break;
      const int code = 0x7fffffff - (int) (uint32_t) (key & 0xffffffffu);
      const int dI = code / MSA_N, dJ = code % MSA_N;
      if (lane == 0) { w.par[dI] = (int8_t) nn; w.par[dJ] = (int8_t) nn; w.lc[nn] = (int8_t) dI; w.rc[nn] = (int8_t) dJ; }
      __syncwarp();
      for (int i = lane; i < nn; i += 32)
        if (w.par[i] == -1)
          w.d[tri(i, nn)] = (int8_t) ((((dI < i) ? w.d[tri(dI, i)] : w.d[tri(i, dI)]) + ((dJ < i) ? w.d[tri(dJ, i)] : w.d[tri(i, dJ)])) / 2);
      __syncwarp();
      for (int i = lane; i < nn + 1; i += 32) {
        if (i < dI) w.d[tri(i, dI)] = -1;
        if (i > dI) w.d[tri(dI, i)] = -1;
        if (i < dJ) w.d[tri(i, dJ)] = -1;
        if (i > dJ) w.d[tri(dJ, i)] = -1;
      }
      __syncwarp();
    }
    const int root = (nn > 0) ? nn - 1 : 0;

    // ---- progressive alignment in node-creation order ---------------------------------------
    if (lane < num) {
      w.nodeR[lane] = 1;
      w.nodeL[lane] = (uint16_t) A.read_len[rbeg + lane];
      w.nodeP[lane] = A.read_off[rbeg + lane];
      spans[2 * MSA_MAXR * lane] = 0;  // a read has no gaps: aligned span = the whole read
      spans[2 * MSA_MAXR * lane + MSA_MAXR] = (int16_t) (A.read_len[rbeg + lane] - 1);
    }
    __syncwarp();
    size_t bump = 0;
    for (int node = num; node <= root && status == ST_OK; ++node) {
      NodeAln a1, a2;
      const int c1 = w.lc[node], c2 = w.rc[node];
      {
        a1.p = (c1 < num ? A.seqs : alnbuf) + w.nodeP[c1]; a1.R = w.nodeR[c1]; a1.L = w.nodeL[c1];
        a2.p = (c2 < num ? A.seqs : alnbuf) + w.nodeP[c2]; a2.R = w.nodeR[c2]; a2.L = w.nodeL[c2];
      }
      const int m = a1.L, n = a2.L;
      if (a1.R > 1 || a2.R > 1) {
        if (lane < a1.R) { w.first1[lane] = spans[2 * MSA_MAXR * c1 + lane]; w.last1[lane] = spans[2 * MSA_MAXR * c1 + MSA_MAXR + lane]; }
        if (lane < a2.R) { w.first2[lane] = spans[2 * MSA_MAXR * c2 + lane]; w.last2[lane] = spans[2 * MSA_MAXR * c2 + MSA_MAXR + lane]; }
        __syncwarp();
      }
      int sstride;
      const int8_t* Sptr = score_table<6>(a1, w.first1, w.last1, a2, w.first2, w.last2, A, w.u.g, keys1, keys2, ids1, ids2, bigtab, sstride, lane);
      const int rowwords = (n + 1 + 7) >> 3;
      gotoh_dp(m, n, A, tr, rowwords, ids1, ids2, Sptr, sstride, Sptr != w.u.g.t.S, bnd, lane);
      const int L = msa_traceback(tr, rowwords, m, n, w.win, src1, src2, lane);
      const int R = a1.R + a2.R;
      if (L > MSA_LCAP) { status = ST_TOO_LONG; break; }   // every node of at most MSA_LCAP columns fits A.aln_cap
      uint8_t* out = alnbuf + bump;
      bump += ((size_t) R * L + 15) & ~(size_t) 15;
      // _createAlignment (src/align.h:202-229): rows of a1, then rows of a2
      int16_t* inv1 = (int16_t*) keys1;  // child column -> column of the new alignment (the keys are dead after the DP)
      int16_t* inv2 = (int16_t*) keys2;
      for (int ai = lane; ai < L; ai += 32) {
        const int kk = L - 1 - ai;
        const int s1 = src1[kk], s2 = src2[kk];
        for (int i = 0; i < a1.R; ++i) out[(size_t) i * L + ai] = (s1 >= 0) ? a1.p[(size_t) i * a1.L + s1] : (uint8_t) '-';
        for (int i = 0; i < a2.R; ++i) out[(size_t) (a1.R + i) * L + ai] = (s2 >= 0) ? a2.p[(size_t) i * a2.L + s2] : (uint8_t) '-';
        if (s1 >= 0) inv1[s1] = (int16_t) ai;
        if (s2 >= 0) inv2[s2] = (int16_t) ai;
      }
      __syncwarp();
      // first/last aligned column of every row (src/align.h:137-150), carried over from the children
      if (lane < R) {
        const bool left = lane < a1.R;
        const int16_t* cs = spans + 2 * MSA_MAXR * (left ? c1 : c2);
        const int rr = left ? lane : lane - a1.R;
        const int16_t* inv = left ? inv1 : inv2;
        spans[2 * MSA_MAXR * node + lane] = inv[cs[rr]];
        spans[2 * MSA_MAXR * node + MSA_MAXR + lane] = inv[cs[MSA_MAXR + rr]];
      }
      if (lane == 0) { w.nodeR[node] = (uint8_t) R; w.nodeL[node] = (uint16_t) L; w.nodeP[node] = (uint32_t) (out - alnbuf); }
      __syncwarp();
    }
    if (status != ST_OK) {
      if (lane == 0) { A.status[cl] = status; A.cons_len[cl] = 0; A.n_rows[cl] = 0; if (A.aln_cols) A.aln_cols[cl] = 0; }
      continue;
    }

    // ---- consensus (src/msa.h:111-173) -------------------------------------------------------
    NodeAln ra;
    ra.p = (root < num ? A.seqs : alnbuf) + w.nodeP[root]; ra.R = w.nodeR[root]; ra.L = w.nodeL[root];
    if (lane < ra.R) { w.first1[lane] = spans[2 * MSA_MAXR * root + lane]; w.last1[lane] = spans[2 * MSA_MAXR * root + MSA_MAXR + lane]; }
    __syncwarp();
    const int thr = max(2, min(A.min_clique, ra.R));
    // consensus_columns' vote, written out: calling it here adds spills to msa_kernel and cost 0.8 % of K2 throughput on an H100
    for (int j = lane; j < ra.L; j += 32) {
      int cov = 0;
      int cnt[5] = {0, 0, 0, 0, 0};
      for (int r = 0; r < ra.R; ++r) {
        if (w.first1[r] >= 0 && w.first1[r] <= j && j <= w.last1[r]) {
          ++cov;
          const uint8_t c = ra.p[(size_t) r * ra.L + j];
          if (c == 'A' || c == 'a') ++cnt[0];
          else if (c == 'C' || c == 'c') ++cnt[1];
          else if (c == 'G' || c == 'g') ++cnt[2];
          else if (c == 'T' || c == 't') ++cnt[3];
          else ++cnt[4];
        }
      }
      uint8_t g = '-';
      if (cov >= thr) {
        int mi = 0;
#pragma unroll
        for (int x = 1; x < 5; ++x) if (cnt[x] > cnt[mi]) mi = x;
        if (mi == 0) g = 'A'; else if (mi == 1) g = 'C'; else if (mi == 2) g = 'G'; else if (mi == 3) g = 'T';
      }
      gapped[j] = g;
    }
    __syncwarp();
    {
      const uint32_t k = compact_consensus(gapped, ra.L, A.cons + A.cons_off[cl], lane);
      if (lane == 0) {
        A.cons_len[cl] = k;
        A.n_rows[cl] = (uint32_t) ra.R;
        A.status[cl] = ST_OK;
        if (A.aln_cols) A.aln_cols[cl] = (uint32_t) ra.L;
      }
    }
    if (A.aln) {
      uint8_t* o = A.aln + A.aln_off[cl];
      for (int x = lane; x < ra.R * ra.L; x += 32) o[x] = ra.p[x];
    }
  }
}

// Global workspace of msa_large_kernel: one slab per CTA (sized for max_reads), holding the similarity triangle at offset 0, then
// the Peq masks, the two row buffers of every read, the gapped consensus and one slab per warp. A warp's slab holds the trace at
// offset 0 (in the LCS phase: the 32 DP rows of its lanes) and the same per-node arrays as a msa_kernel warp's.
struct MsaLargeWork {
  uint8_t* work;
  size_t cta_stride, off_peq, off_rows, off_gapped, off_warps;
  size_t warp_stride, w_tab, w_keys, w_ids, w_src, w_bnd, w_rows;
};

__global__ void __launch_bounds__(MSA_LT, 1) msa_large_kernel(MsaArgs A, MsaLargeWork W) {
  extern __shared__ __align__(16) uint8_t msa_smem[];
  LargeSm& S = *reinterpret_cast<LargeSm*>(msa_smem);
  const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
  constexpr int RS = MSA_LCAP + 1;  // row buffer bytes
  uint8_t* cta = W.work + (size_t) blockIdx.x * W.cta_stride;
  int8_t* d = (int8_t*) cta;
  uint32_t* peq = (uint32_t*) (cta + W.off_peq);
  uint8_t* rowbuf = cta + W.off_rows;
  uint8_t* gapped = cta + W.off_gapped;
  uint8_t* slab = cta + W.off_warps + (size_t) wib * W.warp_stride;
  uint32_t* tr = (uint32_t*) slab;
  int* lcsrow = (int*) slab + (size_t) lane * (MSA_LCAP + 2);
  int8_t* bigtab = (int8_t*) (slab + W.w_tab);
  unsigned long long* keys1 = (unsigned long long*) (slab + W.w_keys);
  unsigned long long* keys2 = keys1 + RS;
  uint16_t* ids1 = (uint16_t*) (slab + W.w_ids);
  uint16_t* ids2 = ids1 + RS;
  int16_t* src1 = (int16_t*) (slab + W.w_src);
  int16_t* src2 = src1 + (2 * MSA_LCAP + 4);
  int2* bnd = (int2*) (slab + W.w_bnd);
  int16_t* rid1 = (int16_t*) (slab + W.w_rows);  // per node: read id, first and last aligned column of every row of each child
  int16_t *rid2 = rid1 + RS, *f1 = rid2 + RS, *l1 = f1 + RS, *f2 = l1 + RS, *l2 = f2 + RS;
  int16_t* root_rid = (int16_t*) (cta + W.off_warps + W.w_rows);  // the root's rows, in warp 0's arrays
  int16_t *root_f = root_rid + 2 * RS, *root_l = root_f + RS;

  for (uint32_t cl = blockIdx.x; cl < A.nclusters; cl += gridDim.x) {
    const uint32_t rbeg = A.cluster_off[cl];
    const int num = (int) (A.cluster_off[cl + 1] - rbeg);
    if (num <= MSA_MAXR || num > A.max_reads) continue;  // msa_kernel's
    __syncthreads();  // the previous cluster is finished with the shared state
    int bad = 0;
    for (int i = wib; i < num; i += MSA_LWARPS) bad |= read_flags(A, rbeg + i, lane);
    const int too_long = __syncthreads_or(bad & 2), bad_char = __syncthreads_or(bad & 1);
    int status = too_long ? ST_TOO_LONG : (bad_char ? ST_BAD_CHAR : ST_OK);
    if (status != ST_OK) {
      if (tid == 0) { A.status[cl] = status; A.cons_len[cl] = 0; A.n_rows[cl] = 0; if (A.aln_cols) A.aln_cols[cl] = 0; }
      continue;
    }
    const int NN = 2 * num + 1;

    // ---- distance matrix (src/msa.h:32-44, :190-195); leaves: one row each, copied into bank 0 of its read ----------
    for (int x = tid; x < num * 5 * LCS_W; x += MSA_LT) peq[x] = 0;
    for (int i = tid; i < num; i += MSA_LT) {
      const int len = (int) A.read_len[rbeg + i];
      S.nodeR[i] = 1; S.nodeL[i] = (uint16_t) len; S.head[i] = S.tail[i] = (int16_t) i; S.lev[i] = 0;
      S.next[i] = -1; S.first[i] = 0; S.last[i] = (int16_t) (len - 1); S.bank[i] = 0;
      S.act[0][i] = (int16_t) i;
    }
    __syncthreads();
    for (int i = wib; i < num; i += MSA_LWARPS) {
      const uint32_t len = A.read_len[rbeg + i];
      const uint8_t* s = A.seqs + A.read_off[rbeg + i];
      build_peq(s, len, peq + i * 5 * LCS_W, lane);
      for (uint32_t x = lane; x < len; x += 32) rowbuf[(size_t) i * 2 * RS + x] = s[x];
    }
    __syncthreads();
    for (int i = wib; i < num; i += MSA_LWARPS) {
      const int li = (int) A.read_len[rbeg + i];
      const uint8_t* si = A.seqs + A.read_off[rbeg + i];
      for (int j = i + 1 + lane; j < num; j += 32) {
        const int lj = (int) A.read_len[rbeg + j];
        const uint8_t* sj = A.seqs + A.read_off[rbeg + j];
        int l;
        if (li <= 32 * LCS_W) l = lcs_bitpar(peq + i * 5 * LCS_W, li, sj, lj);
        else if (lj <= 32 * LCS_W) l = lcs_bitpar(peq + j * 5 * LCS_W, lj, si, li);
        else l = lcs_dp(si, li, sj, lj, lcsrow);
        d[tri(i, j, NN)] = (int8_t) ((l * 100) / min(li, lj));
      }
    }
    __syncthreads();

    // ---- UPGMA (src/msa.h:46-89) over the active nodes ----------------------------------------------------------------
    // Only entries between two active nodes are ever read, so merged nodes are dropped from the list instead of masked with -1.
    // The list is in increasing id order, so row-major order over list positions (a, b) is row-major order over node ids: the
    // first strict maximum is the reference's.
    int nact = num, cur = 0, nn = num;
    for (; nn < NN; ++nn) {
      const int16_t* act = S.act[cur];
      unsigned long long key = 0;
      for (int a = wib; a < nact; a += MSA_LWARPS) {
        const int i = act[a];
        for (int b = a + 1 + lane; b < nact; b += 32) {
          const int v = d[tri(i, act[b], NN)];
          const unsigned long long k2 = ((unsigned long long) (uint32_t) (v + 2) << 32) | (uint32_t) (0x7fffffff - (a * MSA_LN + b));
          key = k2 > key ? k2 : key;
        }
      }
#pragma unroll
      for (int dd = 16; dd >= 1; dd >>= 1) {
        unsigned long long y = __shfl_xor_sync(0xffffffffu, key, dd);
        key = y > key ? y : key;
      }
      if (lane == 0) S.red[wib] = key;
      __syncthreads();
      for (int x = 0; x < MSA_LWARPS; ++x) key = S.red[x] > key ? S.red[x] : key;
      const int dMax = (int) (uint32_t) (key >> 32) - 2;
      if (key == 0 || dMax == -1) break;
      const int code = 0x7fffffff - (int) (uint32_t) (key & 0xffffffffu);
      const int pa = code / MSA_LN, pb = code % MSA_LN;
      const int dI = act[pa], dJ = act[pb];
      int16_t* nxt = S.act[cur ^ 1];
      for (int t = tid; t < nact; t += MSA_LT) {
        if (t == pa || t == pb) continue;
        const int i = act[t];
        d[tri(i, nn, NN)] = (int8_t) ((d[(dI < i) ? tri(dI, i, NN) : tri(i, dI, NN)] + d[(dJ < i) ? tri(dJ, i, NN) : tri(i, dJ, NN)]) / 2);
        nxt[t - (t > pa) - (t > pb)] = (int16_t) i;
      }
      if (tid == 0) { S.lc[nn] = (int16_t) dI; S.rc[nn] = (int16_t) dJ; S.lev[nn] = (int16_t) (1 + max(S.lev[dI], S.lev[dJ])); nxt[nact - 2] = (int16_t) nn; }
      __syncthreads();
      cur ^= 1;
      --nact;
    }
    const int root = nn - 1;

    // ---- progressive alignment, level by level: the nodes of one level are independent --------------------------------
    const int maxlev = S.lev[root];
    if (tid == 0) {  // inner nodes sorted by level (counting sort; levels 1 .. maxlev start at levoff[level])
      for (int l = 0; l <= maxlev + 1; ++l) S.levoff[l] = 0;
      for (int node = num; node <= root; ++node) ++S.levoff[S.lev[node] + 1];
      for (int l = 0; l <= maxlev; ++l) { S.levoff[l + 1] += S.levoff[l]; S.act[0][l] = S.levoff[l]; }
      for (int node = num; node <= root; ++node) S.order[S.act[0][S.lev[node]]++] = (int16_t) node;
    }
    __syncthreads();
    for (int lv = 1; lv <= maxlev; ++lv) {
      int err = 0;
      for (int q = S.levoff[lv] + wib; q < S.levoff[lv + 1]; q += MSA_LWARPS) {
        const int node = S.order[q], c1 = S.lc[node], c2 = S.rc[node];
        const int R1 = S.nodeR[c1], R2 = S.nodeR[c2], m = S.nodeL[c1], n = S.nodeL[c2];
        if (lane == 0) {
          for (int i = 0, r = S.head[c1]; i < R1; ++i, r = S.next[r]) rid1[i] = (int16_t) r;
          for (int i = 0, r = S.head[c2]; i < R2; ++i, r = S.next[r]) rid2[i] = (int16_t) r;
        }
        __syncwarp();
        for (int i = lane; i < R1; i += 32) { f1[i] = S.first[rid1[i]]; l1[i] = S.last[rid1[i]]; }
        for (int i = lane; i < R2; i += 32) { f2[i] = S.first[rid2[i]]; l2[i] = S.last[rid2[i]]; }
        __syncwarp();
        const NodeRows a1{rowbuf, rid1, S.bank, R1, m}, a2{rowbuf, rid2, S.bank, R2, n};
        int sstride;
        const int8_t* Sptr = score_table<10>(a1, f1, l1, a2, f2, l2, A, S.g[wib], keys1, keys2, ids1, ids2, bigtab, sstride, lane);
        const int rowwords = (n + 1 + 7) >> 3;
        gotoh_dp(m, n, A, tr, rowwords, ids1, ids2, Sptr, sstride, Sptr != S.g[wib].t.S, bnd, lane);
        const int L = msa_traceback(tr, rowwords, m, n, S.win[wib], src1, src2, lane);
        if (L > MSA_LCAP) { err = 1; break; }
        // _createAlignment (src/align.h:202-229): rows of a1, then rows of a2, each written into the other bank of its read
        int16_t* inv1 = (int16_t*) keys1;  // child column -> column of the new alignment (the keys are dead after the DP)
        int16_t* inv2 = (int16_t*) keys2;
        for (int ai = lane; ai < L; ai += 32) {
          const int kk = L - 1 - ai;
          const int s1 = src1[kk], s2 = src2[kk];
          if (s1 >= 0) inv1[s1] = (int16_t) ai;
          if (s2 >= 0) inv2[s2] = (int16_t) ai;
        }
        for (int i = 0; i < R1 + R2; ++i) {
          const bool left = i < R1;
          const int r = left ? rid1[i] : rid2[i - R1];
          const int16_t* sv = left ? src1 : src2;
          const uint8_t* from = rowbuf + ((size_t) r * 2 + S.bank[r]) * RS;
          uint8_t* to = rowbuf + ((size_t) r * 2 + (S.bank[r] ^ 1)) * RS;
          for (int ai = lane; ai < L; ai += 32) { const int s = sv[L - 1 - ai]; to[ai] = (s >= 0) ? from[s] : (uint8_t) '-'; }
        }
        __syncwarp();
        // first/last aligned column of every row (src/align.h:137-150), carried over from the children
        for (int i = lane; i < R1 + R2; i += 32) {
          const bool left = i < R1;
          const int r = left ? rid1[i] : rid2[i - R1];
          const int16_t* inv = left ? inv1 : inv2;
          S.first[r] = inv[S.first[r]]; S.last[r] = inv[S.last[r]]; S.bank[r] ^= 1;
        }
        if (lane == 0) {
          S.next[S.tail[c1]] = S.head[c2]; S.head[node] = S.head[c1]; S.tail[node] = S.tail[c2];
          S.nodeR[node] = (uint16_t) (R1 + R2); S.nodeL[node] = (uint16_t) L;
        }
        __syncwarp();
      }
      if (__syncthreads_or(err)) { status = ST_TOO_LONG; break; }
    }
    if (status != ST_OK) {
      if (tid == 0) { A.status[cl] = status; A.cons_len[cl] = 0; A.n_rows[cl] = 0; if (A.aln_cols) A.aln_cols[cl] = 0; }
      continue;
    }

    // ---- consensus (src/msa.h:111-173) -------------------------------------------------------------------------------
    const int R = S.nodeR[root], L = S.nodeL[root];
    if (tid == 0)
      for (int i = 0, r = S.head[root]; i < R; ++i, r = S.next[r]) root_rid[i] = (int16_t) r;
    __syncthreads();
    for (int i = tid; i < R; i += MSA_LT) { root_f[i] = S.first[root_rid[i]]; root_l[i] = S.last[root_rid[i]]; }
    __syncthreads();
    const NodeRows ra{rowbuf, root_rid, S.bank, R, L};
    const int thr = max(2, min(A.min_clique, R));
    consensus_columns(ra, root_f, root_l, thr, gapped, tid, MSA_LT);
    if (A.aln) {
      uint8_t* o = A.aln + A.aln_off[cl];
      for (int r = wib; r < R; r += MSA_LWARPS) {
        const uint8_t* p = ra.row(r);
        for (int x = lane; x < L; x += 32) o[(size_t) r * L + x] = p[x];
      }
    }
    __syncthreads();
    if (wib == 0) {
      const uint32_t k = compact_consensus(gapped, L, A.cons + A.cons_off[cl], lane);
      if (lane == 0) {
        A.cons_len[cl] = k;
        A.n_rows[cl] = (uint32_t) R;
        A.status[cl] = ST_OK;
        if (A.aln_cols) A.aln_cols[cl] = (uint32_t) L;
      }
    }
  }
}

int check_max_reads(dgpu_ctx* ctx, uint32_t max_reads) {
  if (max_reads >= 1 && max_reads <= (uint32_t) MSA_LARGE_MAXR) return DGPU_OK;
  ctx->last_error = "dgpu_msa_ex: max_reads must be 1 .. " + std::to_string(MSA_LARGE_MAXR);
  return DGPU_ERR_ARG;
}

constexpr size_t MSA_B_TRACE = ((size_t) (MSA_LCAP + 1) * ((MSA_LCAP + 8) / 8) * 4 + 255) & ~(size_t) 255;   // traceback bits of one alignment

// Slab layout of msa_kernel's warps (fixed: sized for MSA_MAXR reads and MSA_LCAP columns).
void msa_warp_layout(MsaArgs& A) {
  auto al = [](size_t x) { return (x + 255) & ~(size_t) 255; };
  // node alignments of one cluster, never freed: a node takes R x L bytes rounded up to 16, at most R x (MSA_LCAP + 1). The R of all
  // nodes sum to the leaves' depths, at most 2 + 3 + .. + MSA_MAXR for a chain-shaped guide tree.
  A.aln_cap = al((size_t) (MSA_MAXR * (MSA_MAXR + 1) / 2 - 1) * (MSA_LCAP + 1));
  A.off_prof = A.aln_cap;
  const size_t b_prof = al((size_t) (MSA_LCAP + 1) * 5);  // gapped consensus + the two column-kind arrays
  A.off_trace = A.off_prof + b_prof;
  A.off_lcs = A.off_trace + MSA_B_TRACE;
  A.off_keys = A.off_lcs + al((size_t) 32 * (MSA_LCAP + 2) * sizeof(int) + MSA_TRI);
  A.off_src = A.off_keys + al((size_t) (MSA_LCAP + 1) * 16);
  A.off_bnd = A.off_src + al((size_t) (2 * MSA_LCAP + 4) * 4);
  A.off_tab = A.off_bnd + al((size_t) 2 * (MSA_LCAP + 1) * 8);
  A.off_spans = A.off_tab + al((size_t) MSA_LCAP * MSA_LCAP);
  A.work_stride = A.off_spans + al((size_t) MSA_N * 2 * MSA_MAXR * 2);
}

// Slab layout of one msa_large_kernel CTA for clusters of up to max_reads reads.
MsaLargeWork msa_large_layout(size_t max_reads) {
  auto al = [](size_t x) { return (x + 255) & ~(size_t) 255; };
  MsaLargeWork W{};
  const size_t nmax = max_reads, nn = 2 * nmax + 1;
  W.off_peq = al(nn * (nn - 1) / 2);
  W.off_rows = W.off_peq + al(nmax * 5 * LCS_W * 4);
  W.off_gapped = W.off_rows + al(nmax * 2 * (MSA_LCAP + 1));
  W.off_warps = W.off_gapped + al(MSA_LCAP + 1);
  W.w_tab = std::max(MSA_B_TRACE, al((size_t) 32 * (MSA_LCAP + 2) * sizeof(int)));  // the trace, or the LCS phase's DP rows
  W.w_keys = W.w_tab + al((size_t) MSA_LCAP * MSA_LCAP);
  W.w_ids = W.w_keys + al((size_t) (MSA_LCAP + 1) * 16);
  W.w_src = W.w_ids + al((size_t) (MSA_LCAP + 1) * 4);
  W.w_bnd = W.w_src + al((size_t) (2 * MSA_LCAP + 4) * 4);
  W.w_rows = W.w_bnd + al((size_t) 2 * (MSA_LCAP + 1) * 8);
  W.warp_stride = W.w_rows + al((size_t) 6 * (MSA_LCAP + 1) * 2);
  W.cta_stride = W.off_warps + MSA_LWARPS * W.warp_stride;
  return W;
}

}  // namespace

extern "C" {

int dgpu_set_msa_async_bound(dgpu_ctx* ctx, uint32_t max_reads, uint32_t max_read_len) {
  if (!ctx) return DGPU_ERR_ARG;
  if (!max_reads && !max_read_len) { ctx->msa_max_reads = 0; return DGPU_OK; }
  if (!max_reads || !max_read_len || max_reads > (uint32_t) MSA_LARGE_MAXR || max_read_len > (uint32_t) MSA_LCAP) {
    ctx->last_error = "dgpu_set_msa_async_bound: max_reads must be 1 .. " + std::to_string(MSA_LARGE_MAXR) + " and max_read_len 1 .. " +
                      std::to_string(MSA_LCAP) + " (or both 0)";
    return DGPU_ERR_ARG;
  }
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  // the slots of the largest grids dgpu_msa_ex_dev launches (their slabs are sized for MSA_LCAP columns whatever the read length)
  MsaArgs A;
  msa_warp_layout(A);
  void* p;
  int rc;
  if ((rc = dgpu_smem_optin(ctx, msa_kernel, sizeof(WarpSm) * MSA_WARPS, "cudaFuncSetAttribute(msa_kernel)")) ||
      (rc = dgpu_reserve(ctx, SLOT_MSA_SEGJOBS, (size_t) ctx->num_sms * MSA_PER_SM * MSA_WARPS * A.work_stride, &p)))
    return rc;
  if (max_reads > (uint32_t) MSA_MAXR &&
      ((rc = dgpu_smem_optin(ctx, msa_large_kernel, sizeof(LargeSm), "cudaFuncSetAttribute(msa_large_kernel)")) ||
       (rc = dgpu_reserve(ctx, SLOT_MSA_LARGE, (size_t) ctx->num_sms * msa_large_layout(max_reads).cta_stride, &p))))
    return rc;
  ctx->msa_max_reads = max_reads;
  return DGPU_OK;
}

int dgpu_msa_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                    const uint32_t* read_off, const uint32_t* read_len, const uint32_t* cluster_off, uint32_t nclusters,
                    int match, int mismatch, int go, int ge, int min_clique,
                    uint8_t* cons, const uint64_t* cons_off, uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
                    uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_cols, uint32_t max_reads, void* stream) {
  if (!ctx) return DGPU_ERR_ARG;
  int rc;
  if ((rc = check_max_reads(ctx, max_reads))) return rc;
  if (nclusters == 0) return DGPU_OK;
  if (!seqs || !read_off || !read_len || !cluster_off || !cons || !cons_off || !cons_len || !n_rows || !status) return DGPU_ERR_ARG;
  if (seqs_bytes >= (1ull << 32)) return DGPU_ERR_ARG;
  if (match > 127 || match < -127 || mismatch > 127 || mismatch < -127) return DGPU_ERR_UNSUPPORTED;  // the score table is int8
  DGPU_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t) stream : ctx->stream;
  if (ctx->msa_max_reads) max_reads = std::min(max_reads, ctx->msa_max_reads);   // inside the slots dgpu_set_msa_async_bound reserved
  MsaArgs A;
  A.seqs = seqs; A.read_off = read_off; A.read_len = read_len; A.cluster_off = cluster_off; A.nclusters = nclusters;
  A.match = match; A.mismatch = mismatch; A.go = go; A.ge = ge; A.min_clique = min_clique; A.max_reads = (int) max_reads;
  A.cons = cons; A.cons_off = cons_off; A.cons_len = cons_len; A.n_rows = n_rows; A.status = status;
  A.aln = aln; A.aln_off = aln_off; A.aln_cols = aln_cols;
  msa_warp_layout(A);
  const int per_sm = MSA_PER_SM;  // CTAs of four independent warps
  const size_t smem = sizeof(WarpSm) * MSA_WARPS;
  if ((rc = dgpu_smem_optin(ctx, msa_kernel, smem, "cudaFuncSetAttribute(msa_kernel)"))) return rc;   // per device: set on the first call
  size_t grid = std::min<size_t>((nclusters + MSA_WARPS - 1) / MSA_WARPS, (size_t) ctx->num_sms * per_sm);
  void* p;
  if ((rc = dgpu_reserve(ctx, SLOT_MSA_SEGJOBS, grid * MSA_WARPS * A.work_stride, &p))) return rc;
  A.work = (uint8_t*) p;
  // clusters of 33 .. max_reads reads: one CTA each, workspace sized for max_reads (nothing when max_reads <= 32)
  MsaLargeWork W{};
  size_t lgrid = 0, lsmem = sizeof(LargeSm);
  if (max_reads > (uint32_t) MSA_MAXR) {
    W = msa_large_layout(max_reads);
    lgrid = std::min<size_t>(nclusters, (size_t) ctx->num_sms);
    if ((rc = dgpu_smem_optin(ctx, msa_large_kernel, lsmem, "cudaFuncSetAttribute(msa_large_kernel)"))) return rc;
    if ((rc = dgpu_reserve(ctx, SLOT_MSA_LARGE, lgrid * W.cta_stride, &p))) return rc;
    W.work = (uint8_t*) p;
  }
  dgpu_prof_begin(ctx, st);
  msa_kernel<<<(unsigned) grid, MSA_T, smem, st>>>(A);
  DGPU_LAUNCH_CHECK(ctx, "msa_kernel");
  if (lgrid) {
    msa_large_kernel<<<(unsigned) lgrid, MSA_LT, lsmem, st>>>(A, W);
    DGPU_LAUNCH_CHECK(ctx, "msa_large_kernel");
  }
  dgpu_prof_end(ctx, st);
  return DGPU_OK;
}

int dgpu_msa_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                 const uint32_t* read_off, const uint32_t* read_len, const uint32_t* cluster_off, uint32_t nclusters,
                 int match, int mismatch, int go, int ge, int min_clique,
                 uint8_t* cons, const uint64_t* cons_off, uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
                 uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_cols, void* stream) {
  return dgpu_msa_ex_dev(ctx, seqs, seqs_bytes, read_off, read_len, cluster_off, nclusters, match, mismatch, go, ge, min_clique, cons, cons_off,
                         cons_len, n_rows, status, aln, aln_off, aln_cols, MSA_MAXR, stream);
}

int dgpu_msa_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                const uint32_t* read_off, const uint32_t* read_len, uint32_t nreads,
                const uint32_t* cluster_off, uint32_t nclusters,
                int match, int mismatch, int go, int ge, int min_clique,
                uint8_t* cons, const uint64_t* cons_off, uint64_t cons_bytes, uint32_t* cons_len, uint32_t* n_rows,
                uint32_t* status, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_cols, uint32_t max_reads) {
  DgpuStage s(ctx, "dgpu_msa", nclusters);
  if (!ctx) return DGPU_ERR_ARG;
  int rc;
  if ((rc = check_max_reads(ctx, max_reads))) return rc;
  if (nclusters == 0) return DGPU_OK;
  if (!seqs || !read_off || !read_len || !cluster_off || !cons || !cons_off || !cons_len || !n_rows || !status) return DGPU_ERR_ARG;
  if ((rc = s.check_arena(seqs_bytes, nreads, read_off, read_len, "read"))) return rc;
  for (uint32_t i = 0; i < nclusters; ++i) {   // consensus slots (capacity = the cluster's total read length) inside cons_bytes
    if (cluster_off[i] > cluster_off[i + 1] || cluster_off[i + 1] > nreads) { ctx->last_error = "dgpu_msa: cluster_off is not a partition of the reads"; return DGPU_ERR_ARG; }
    uint64_t cap = 0;
    for (uint32_t r = cluster_off[i]; r < cluster_off[i + 1]; ++r) cap += read_len[r];
    if (cons_off[i] + cap > cons_bytes) { ctx->last_error = "dgpu_msa: consensus slot beyond cons_bytes"; return DGPU_ERR_CAPACITY; }
  }
  if (aln && (!aln_off || !aln_cols)) return DGPU_ERR_ARG;
  if ((rc = s.open())) return rc;
  const uint8_t* d_seqs = s.arena(seqs, seqs_bytes);
  uint8_t* d_cons = s.out(cons, cons_bytes, 64);
  const uint32_t *d_roff = s.in(read_off, nreads), *d_rlen = s.in(read_len, nreads), *d_coff = s.in(cluster_off, (size_t) nclusters + 1);
  const uint64_t* d_consoff = s.in(cons_off, nclusters);
  uint32_t *d_conslen = s.out(cons_len, nclusters), *d_nrows = s.out(n_rows, nclusters), *d_status = s.out(status, nclusters);
  uint8_t* d_aln = s.out(aln, aln_bytes, 64);
  const uint64_t* d_alnoff = s.in(aln ? aln_off : nullptr, nclusters);
  uint32_t* d_alncols = s.out(aln ? aln_cols : nullptr, nclusters);
  if (s.rc) return s.rc;
  if ((rc = dgpu_msa_ex_dev(ctx, d_seqs, seqs_bytes, d_roff, d_rlen, d_coff, nclusters, match, mismatch, go, ge, min_clique, d_cons, d_consoff,
                            d_conslen, d_nrows, d_status, d_aln, d_alnoff, d_alncols, max_reads, s.st)))
    return rc;
  return s.finish();
}

int dgpu_msa(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
             const uint32_t* read_off, const uint32_t* read_len, uint32_t nreads,
             const uint32_t* cluster_off, uint32_t nclusters,
             int match, int mismatch, int go, int ge, int min_clique,
             uint8_t* cons, const uint64_t* cons_off, uint64_t cons_bytes, uint32_t* cons_len, uint32_t* n_rows,
             uint32_t* status, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_cols) {
  return dgpu_msa_ex(ctx, seqs, seqs_bytes, read_off, read_len, nreads, cluster_off, nclusters, match, mismatch, go, ge, min_clique, cons, cons_off,
                     cons_bytes, cons_len, n_rows, status, aln, aln_off, aln_bytes, aln_cols, MSA_MAXR);
}

}  // extern "C"
