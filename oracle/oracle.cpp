// oracle.cpp — CPU restatement of the reference algorithms on the hot path.
//
// *** TEST INFRASTRUCTURE ONLY ***  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library. The product (libdelly_b200.so and
// delly_b200/host) never links or calls it.
//
// Parity pin: every function here is checked against oracle/_ref/libdelly_ref.so — the reference's
// own sources (dellytools/delly @ 3a22fe2) compiled verbatim — on seeded inputs in
// tests/test_oracle_vs_ref.py, and against the committed vectors in tests/golden/ that were
// generated from that build (tests/golden/make_golden.py). The reference ships no tests or golden
// vectors of its own (SURVEY.md §4), so these are the only pins that exist.
//
// Each function is written from the algorithm's definition (plain full-matrix DP, no banding, no
// bit-vectors) and cites the reference lines whose observable behaviour it restates.
#include <algorithm>
#include <array>
#include <atomic>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

namespace {

typedef std::vector<std::string> Rows;  // an alignment: equal-length rows over ACGTN-

// ---------------------------------------------------------------------------------------
// Edit distance, edlib semantics (src/edlib.cpp:139-294, :545-702, :728-929).
// mode 0 NW (global), 1 SHW (prefix: free gap after query), 2 HW (infix: free gaps around query).
// Returns distance or -1 if it exceeds k (k < 0: unbounded); *end0 = first optimal end position.
int edit_distance(const uint8_t* q, int m, const uint8_t* t, int n, int k, int mode, int* end0) {
  *end0 = -1;
  if (m == 0 || n == 0) {  // src/edlib.cpp:158-177 (decided before k is applied)
    if (mode == 0) { *end0 = n - 1; return std::max(m, n); }
    return m;
  }
  std::vector<int> prev(m + 1), cur(m + 1);
  for (int i = 0; i <= m; ++i) prev[i] = i;  // column 0
  // HW/SHW candidates are the end positions -1..n-1 with score D[m][pos+1]; the first minimum wins.
  // Position -1 (empty target prefix, score m) exists only when |q| is not a multiple of 64: edlib
  // sees column -1 through its W = 64*ceil(m/64)-m wildcard padding columns (src/edlib.cpp:656-671).
  int best = INT_MAX, bpos = -1;
  if (m % 64 != 0) best = m;
  for (int c = 1; c <= n; ++c) {
    cur[0] = (mode == 2) ? 0 : c;
    for (int i = 1; i <= m; ++i) {
      int sub = prev[i - 1] + (q[i - 1] == t[c - 1] ? 0 : 1);
      cur[i] = std::min(sub, std::min(prev[i] + 1, cur[i - 1] + 1));
    }
    if (cur[m] < best) { best = cur[m]; bpos = c - 1; }
    prev.swap(cur);
  }
  int d, e;
  if (mode == 0) { d = prev[m]; e = n - 1; } else { d = best; e = bpos; }
  if (k >= 0) {
    if (mode == 2) { if (d > std::min(k, m)) d = -1; }              // src/edlib.cpp:563-565
    else if (mode == 1) { if (d > k) d = -1; }
    else {
      if (k < std::abs(n - m)) d = -1;                               // src/edlib.cpp:740-743
      else if (d > std::min(k, std::max(m, n))) d = -1;              // src/edlib.cpp:745
    }
  }
  if (d >= 0) *end0 = e;
  return d;
}

// ---------------------------------------------------------------------------------------
inline char comp(char c) {
  switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; default: return c; }
}
// src/util.h:549-563 — upper-cases, complements ACGT, keeps N; any other byte keeps the
// ORIGINAL (un-reversed) character at that index (the reference's `default: break` quirk).
std::string revcomp(std::string const& s) {
  std::string out = s;
  size_t L = s.size();
  for (size_t i = 0; i < L; ++i) {
    char c = (char) std::toupper((unsigned char) s[L - 1 - i]);
    switch (c) {
      case 'A': out[i] = 'T'; break;
      case 'C': out[i] = 'G'; break;
      case 'G': out[i] = 'C'; break;
      case 'T': out[i] = 'A'; break;
      case 'N': out[i] = 'N'; break;
      default: break;
    }
  }
  return out;
}

// Linear-gap semiglobal DP of longNeedle (src/needle.h:59-66, :74-81) with AlignConfig<true,false>,
// score (1,-1,-1): row 0 free, last row moves right for free, vertical gaps always -1.
void ln_matrix(std::string const& a, std::string const& b, std::vector<int32_t>& M) {
  size_t m = a.size(), n = b.size(), W = n + 1;
  M.assign((m + 1) * W, 0);
  for (size_t r = 1; r <= m; ++r) M[r * W] = M[(r - 1) * W] - 1;
  for (size_t r = 1; r <= m; ++r) {
    int hg = (r == m) ? 0 : -1;
    for (size_t c = 1; c <= n; ++c) {
      int d = M[(r - 1) * W + c - 1] + (a[r - 1] == b[c - 1] ? 1 : -1);
      int u = M[(r - 1) * W + c] - 1;
      int l = M[r * W + c - 1] + hg;
      M[r * W + c] = std::max(std::max(d, u), l);
    }
  }
}

// Traceback with priority vertical > horizontal > diagonal (src/needle.h:155-171, :178-192).
// Emits alignment rows for a[0..rr) vs b[0..cc).
void ln_trace(std::vector<int32_t> const& M, std::string const& a, std::string const& b, size_t m, size_t n,
              size_t rr, size_t cc, std::string& ra, std::string& rb) {
  size_t W = n + 1;
  std::string ta, tb;
  while (rr > 0 || cc > 0) {
    int hg = (rr == 0 || rr == m) ? 0 : -1;
    if (rr > 0 && M[rr * W + cc] == M[(rr - 1) * W + cc] - 1) { --rr; ta.push_back(a[rr]); tb.push_back('-'); }
    else if (cc > 0 && M[rr * W + cc] == M[rr * W + cc - 1] + hg) { --cc; ta.push_back('-'); tb.push_back(b[cc]); }
    else { --rr; --cc; ta.push_back(a[rr]); tb.push_back(b[cc]); }
  }
  ra.assign(ta.rbegin(), ta.rend());
  rb.assign(tb.rbegin(), tb.rend());
}

// longNeedle (src/needle.h:45-222). Returns false when fwd/rev scores disagree or no split improves.
bool long_needle(std::string const& s1, std::string const& s2, std::string& row0, std::string& row1) {
  size_t m = s1.size(), n = s2.size(), W = n + 1;
  std::vector<int32_t> mat, rev;
  ln_matrix(s1, s2, mat);
  std::string r1 = revcomp(s1), r2 = revcomp(s2);
  ln_matrix(r1, r2, rev);
  if (mat[m * W + n] != rev[m * W + n]) return false;            // :83-86
  // prefix maxima (:88-103)
  std::vector<int32_t> bm(mat), br(rev);
  for (size_t r = 0; r <= m; ++r)
    for (size_t c = 1; c <= n; ++c) {
      if (bm[r * W + c] <= bm[r * W + c - 1]) bm[r * W + c] = bm[r * W + c - 1];
      if (br[r * W + c] <= br[r * W + c - 1]) br[r * W + c] = br[r * W + c - 1];
    }
  int32_t bestScore = mat[m * W + n];
  size_t consLeft = 0, refLeft = 0;
  for (size_t r = 0; r <= m; ++r)                                 // :104-115 first strict max, row-major
    for (size_t c = 0; c <= n; ++c) {
      int32_t v = bm[r * W + c] + br[(m - r) * W + (n - c)];
      if (v > bestScore) { bestScore = v; consLeft = r; refLeft = c; }
    }
  size_t consRight = m - consLeft, refRight = 0;
  for (size_t right = 0; right <= n - refLeft; ++right)           // :116-123 last matching right
    if (mat[consLeft * W + refLeft] + rev[consRight * W + right] == bestScore) refRight = right;
  if (bestScore == mat[m * W + n]) return false;                  // :152
  std::string fa, fb, va, vb;
  ln_trace(mat, s1, s2, m, n, consLeft, refLeft, fa, fb);
  ln_trace(rev, r1, r2, m, n, consRight, refRight, va, vb);
  row0 = fa; row1 = fb;
  for (size_t j = refLeft; j < n - refRight; ++j) { row0.push_back('-'); row1.push_back(s2[j]); }   // :203-206
  // reverse-complemented, reversed rev alignment (:207-217). Characters outside ACGTN- are left
  // unwritten by the reference (boost::multi_array zero-initialises char -> '\0').
  for (size_t j = 0; j < va.size(); ++j) {
    char x = va[va.size() - 1 - j], y = vb[vb.size() - 1 - j];
    auto cv = [](char ch) -> char {
      switch (ch) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A';
                    case 'N': return 'N'; case '-': return '-'; default: return '\0'; }
    };
    row0.push_back(cv(x)); row1.push_back(cv(y));
  }
  return true;
}

// longestHomology (src/needle.h:13-42): banded (|i-j| <= k) unit-cost DP, returns row-1 at the first
// row whose best banded score drops below the threshold, 0 if that never happens.
int longest_homology(std::string const& s1, std::string const& s2, int thr) {
  int m = (int) s1.size(), n = (int) s2.size(), k = std::abs(thr);
  const int NEG = -1000000;
  std::vector<int> prev(n + 2, NEG), cur(n + 2, NEG);
  for (int c = 0; c <= std::min(k, n); ++c) prev[c] = -c;
  for (int r = 1; r <= m; ++r) {
    std::fill(cur.begin(), cur.end(), NEG);
    if (r <= k) cur[0] = -r;
    int bestCol = thr - 1;
    for (int c = std::max(1, r - k); c <= std::min(n, r + k); ++c) {
      int v = prev[c - 1] + (s1[r - 1] == s2[c - 1] ? 0 : -1);
      if (std::abs(r - 1 - c) <= k) v = std::max(v, prev[c] - 1);
      if (std::abs(r - c + 1) <= k) v = std::max(v, cur[c - 1] - 1);
      cur[c] = v;
      if (v > bestCol) bestCol = v;
    }
    if (bestCol < thr) return r - 1;
    prev.swap(cur);
  }
  return 0;
}

// ---------------------------------------------------------------------------------------
// LCS length (src/msa.h:10-30).
int lcs(std::string const& a, std::string const& b) {
  size_t m = a.size(), n = b.size();
  std::vector<int> prev(n + 1, 0), cur(n + 1, 0);
  for (size_t i = 1; i <= m; ++i) {
    for (size_t j = 1; j <= n; ++j)
      cur[j] = (a[i - 1] == b[j - 1]) ? prev[j - 1] + 1 : std::max(prev[j], cur[j - 1]);
    prev.swap(cur);
  }
  return prev[n];
}

// Column profile of an alignment (src/align.h:128-171): per column the fraction of A,C,G,T,N,'-'
// among rows whose first..last non-gap span covers the column; other characters are not counted.
void profile(Rows const& a, std::vector<float>& p /* 6 x L */) {
  size_t R = a.size(), L = a[0].size();
  p.assign(6 * L, 0.0f);
  std::vector<long> first(R, -1), last(R, (long) L);
  for (size_t i = 0; i < R; ++i)
    for (size_t j = 0; j < L; ++j)
      if (a[i][j] != '-') { if (first[i] == -1) first[i] = (long) j; last[i] = (long) j; }
  for (size_t j = 0; j < L; ++j) {
    int sum = 0;
    for (size_t i = 0; i < R; ++i) {
      if (first[i] <= (long) j && (long) j <= last[i]) {
        ++sum;
        char c = a[i][j];
        if (c == 'A' || c == 'a') p[0 * L + j] += 1;
        else if (c == 'C' || c == 'c') p[1 * L + j] += 1;
        else if (c == 'G' || c == 'g') p[2 * L + j] += 1;
        else if (c == 'T' || c == 't') p[3 * L + j] += 1;
        else if (c == 'N' || c == 'n') p[4 * L + j] += 1;
        else if (c == '-') p[5 * L + j] += 1;
        else --sum;
      }
    }
    for (int k = 0; k < 6; ++k) p[k * L + j] /= sum;
  }
}

// Gotoh affine DP with free end gaps on both sequences and the reference's trace-bit semantics
// (src/gotoh.h:71-174, instantiated as AlignConfig<true,true>, src/msa.h:106-107).
// Substitution score: char compare if both inputs have one row, else the float profile product
// summed k1-outer/k2-inner and truncated to int (src/align.h:96-111).
int gotoh(Rows const& a1, Rows const& a2, int match, int mismatch, int go, int ge, Rows& out) {
  const int INF = 1000000;
  size_t m = a1[0].size(), n = a2[0].size(), W = n + 1;
  bool prof = !(a1.size() == 1 && a2.size() == 1);
  std::vector<float> p1, p2;
  if (prof) { profile(a1, p1); profile(a2, p2); }
  auto score = [&](size_t r, size_t c) -> int {
    if (!prof) return a1[0][r] == a2[0][c] ? match : mismatch;
    volatile float s = 0;  // volatile: forbid contraction/reassociation, keep IEEE single steps
    for (int k1 = 0; k1 < 5; ++k1)
      for (int k2 = 0; k2 < 5; ++k2) {
        volatile float t = p1[k1 * m + r] * p2[k2 * n + c];
        t = t * (float) (k1 == k2 ? match : mismatch);
        s = s + t;
      }
    return (int) s;
  };
  auto hgap = [&](size_t row, int cost) { return (row == 0 || row == m) ? 0 : cost; };
  auto vgap = [&](size_t col, int cost) { return (col == 0 || col == n) ? 0 : cost; };
  std::vector<int> s(W, 0), v(W, 0);
  std::vector<uint8_t> b1((m + 1) * W, 0), b2((m + 1) * W, 0), b3((m + 1) * W, 0), b4((m + 1) * W, 0);
  int newhoz = 0, prevsub = 0;
  for (size_t row = 0; row <= m; ++row) {
    for (size_t col = 0; col <= n; ++col) {
      if (row == 0 && col == 0) { s[0] = 0; v[0] = -INF; newhoz = -INF; b1[0] = 1; b2[0] = 1; }
      else if (row == 0) { v[col] = -INF; s[col] = hgap(0, go + (int) col * ge); newhoz = s[col]; b3[col] = 1; }
      else if (col == 0) {
        newhoz = -INF; s[0] = vgap(0, go + (int) row * ge); prevsub = (row == 1) ? 0 : vgap(0, go + (int) (row - 1) * ge);
        v[0] = s[0]; b4[row * W] = 1;
      } else {
        int prevhoz = newhoz, prevver = v[col], diag = prevsub;
        prevsub = s[col];
        newhoz = std::max(s[col - 1] + hgap(row, go + ge), prevhoz + hgap(row, ge));
        v[col] = std::max(prevsub + vgap(col, go + ge), prevver + vgap(col, ge));
        s[col] = std::max(std::max(diag + score(row - 1, col - 1), newhoz), v[col]);
        size_t x = row * W + col;
        if (s[col] == newhoz) b3[x] = 1; else if (s[col] == v[col]) b4[x] = 1;
        if (newhoz != prevhoz + hgap(row, ge)) b1[x] = 1;
        if (v[col] != prevver + vgap(col, ge)) b2[x] = 1;
      }
    }
  }
  // traceback state machine (src/gotoh.h:141-167)
  std::string tr;
  size_t row = m, col = n;
  char st = 's';
  while (row > 0 || col > 0) {
    size_t x = row * W + col;
    if (st == 's') {
      if (b3[x]) st = 'h'; else if (b4[x]) st = 'v';
      else { --row; --col; tr.push_back('s'); }
    } else if (st == 'h') { if (b1[x]) st = 's'; --col; tr.push_back('h'); }
    else { if (b2[x]) st = 's'; --row; tr.push_back('v'); }
  }
  // merged alignment: rows of a1 then rows of a2 (src/align.h:202-229)
  size_t R1 = a1.size(), R2 = a2.size(), L = tr.size();
  out.assign(R1 + R2, std::string(L, '-'));
  size_t r = 0, c = 0;
  for (size_t ai = 0; ai < L; ++ai) {
    char op = tr[L - 1 - ai];
    if (op == 's' || op == 'v') { for (size_t i = 0; i < R1; ++i) out[i][ai] = a1[i][r]; }
    if (op == 's' || op == 'h') { for (size_t i = 0; i < R2; ++i) out[R1 + i][ai] = a2[i][c]; }
    if (op != 'h') ++r;
    if (op != 'v') ++c;
  }
  return s[n];
}

// Consensus of an alignment (src/msa.h:111-173).
void consensus(Rows const& a, int minClique, std::string& gapped, std::string& cs) {
  size_t R = a.size(), L = a[0].size();
  std::vector<int> cov(L, 0);
  std::vector<long> st(R), en(R);
  for (size_t i = 0; i < R; ++i) {
    long s = 0, e = -1;
    for (size_t j = 0; j < L; ++j) { if (a[i][j] != '-') e = (long) j; else if (e == -1) s = (long) j + 1; }
    st[i] = s; en[i] = e;
    for (long j = s; j <= e; ++j) ++cov[j];
  }
  int thr = std::max(2, std::min(minClique, (int) R));
  gapped.assign(L, '-');
  for (size_t j = 0; j < L; ++j) {
    if (cov[j] < thr) continue;
    int cnt[5] = {0, 0, 0, 0, 0};
    for (size_t i = 0; i < R; ++i) {
      if (st[i] <= (long) j && (long) j <= en[i]) {
        char c = a[i][j];
        if (c == 'A' || c == 'a') ++cnt[0]; else if (c == 'C' || c == 'c') ++cnt[1];
        else if (c == 'G' || c == 'g') ++cnt[2]; else if (c == 'T' || c == 't') ++cnt[3]; else ++cnt[4];
      }
    }
    int mi = 0;
    for (int x = 1; x < 5; ++x) if (cnt[x] > cnt[mi]) mi = x;
    if (mi < 4) gapped[j] = "ACGT"[mi];
  }
  cs.clear();
  for (char c : gapped) if (c != '-') cs.push_back(c);
}

// Number of distinct column profiles of an alignment, counted on the integers profile() divides (the A,C,G,T,N counts and the number
// of covering rows): columns with equal integers have bit-identical float profiles.
int distinct_profiles(Rows const& a) {
  size_t R = a.size(), L = a[0].size();
  std::vector<long> first(R, -1), last(R, (long) L);
  for (size_t i = 0; i < R; ++i)
    for (size_t j = 0; j < L; ++j)
      if (a[i][j] != '-') { if (first[i] == -1) first[i] = (long) j; last[i] = (long) j; }
  std::vector<std::array<int, 6>> keys(L);
  for (size_t j = 0; j < L; ++j) {
    std::array<int, 6> k{};
    for (size_t i = 0; i < R; ++i) {
      if (first[i] <= (long) j && (long) j <= last[i]) {
        ++k[5];
        char c = a[i][j];
        if (c == 'A' || c == 'a') ++k[0];
        else if (c == 'C' || c == 'c') ++k[1];
        else if (c == 'G' || c == 'g') ++k[2];
        else if (c == 'T' || c == 't') ++k[3];
        else if (c == 'N' || c == 'n') ++k[4];
        else if (c != '-') --k[5];
      }
    }
    keys[j] = k;
  }
  std::sort(keys.begin(), keys.end());
  return (int) (std::unique(keys.begin(), keys.end()) - keys.begin());
}

// One inner node of the guide tree: its rows and columns, the columns of its two children (the DP's rows and columns) and their
// distinct column profiles (0 when both children are single reads, which gotoh compares character by character).
struct NodeInfo { int R, L, L1, L2, U1, U2; };

// msa (src/msa.h:185-239): LCS similarity matrix, UPGMA guide tree, progressive gotoh, consensus.
// nodes (optional): every inner node in creation order.
int msa(std::vector<std::string> const& reads, int minClique, int match, int mismatch, int go, int ge,
        std::string& cs, Rows* alnOut, std::vector<NodeInfo>* nodes = nullptr) {
  int num = (int) reads.size(), N = 2 * num + 1;
  std::vector<int> d((size_t) N * N, -1);
  for (int i = 0; i < num; ++i)
    for (int j = i + 1; j < num; ++j)
      d[i * N + j] = (lcs(reads[i], reads[j]) * 100) / (int) std::min(reads[i].size(), reads[j].size());   // msa.h:41
  std::vector<int> par(N, -1), lc(N, -1), rc(N, -1);
  int nn = num;
  for (; nn < N; ++nn) {                                       // upgma, msa.h:74-89
    int dMax = -1, dI = 0, dJ = 0;
    for (int i = 0; i < nn; ++i)
      for (int j = i + 1; j < nn; ++j)
        if (d[i * N + j] > dMax) { dMax = d[i * N + j]; dI = i; dJ = j; }
    if (dMax == -1) break;
    par[dI] = nn; par[dJ] = nn; lc[nn] = dI; rc[nn] = dJ;
    for (int i = 0; i < nn; ++i)                               // msa.h:61-72
      if (par[i] == -1)
        d[i * N + nn] = (((dI < i) ? d[dI * N + i] : d[i * N + dI]) + ((dJ < i) ? d[dJ * N + i] : d[i * N + dJ])) / 2;
    for (int i = 0; i < dI; ++i) d[i * N + dI] = -1;
    for (int i = dI + 1; i < nn + 1; ++i) d[dI * N + i] = -1;
    for (int i = 0; i < dJ; ++i) d[i * N + dJ] = -1;
    for (int i = dJ + 1; i < nn + 1; ++i) d[dJ * N + i] = -1;
  }
  int root = (nn > 0) ? nn - 1 : 0;
  // post-order progressive alignment (msa.h:91-109)
  struct Rec {
    static void run(int node, std::vector<int> const& lc, std::vector<int> const& rc, std::vector<std::string> const& reads,
                    int match, int mismatch, int go, int ge, Rows& out, std::vector<NodeInfo>* info) {
      if (lc[node] == -1 && rc[node] == -1) { out.assign(1, reads[node]); return; }
      Rows a, b;
      run(lc[node], lc, rc, reads, match, mismatch, go, ge, a, info);
      run(rc[node], lc, rc, reads, match, mismatch, go, ge, b, info);
      gotoh(a, b, match, mismatch, go, ge, out);
      if (info) {
        const bool prof = a.size() > 1 || b.size() > 1;
        (*info)[node] = NodeInfo{(int) out.size(), (int) out[0].size(), (int) a[0].size(), (int) b[0].size(),
                                 prof ? distinct_profiles(a) : 0, prof ? distinct_profiles(b) : 0};
      }
    }
  };
  Rows aln;
  std::vector<NodeInfo> info(nodes ? N : 0);
  Rec::run(root, lc, rc, reads, match, mismatch, go, ge, aln, nodes ? &info : nullptr);
  if (nodes) nodes->assign(info.begin() + num, info.begin() + std::max(num, root + 1));
  std::string gapped;
  consensus(aln, minClique, gapped, cs);
  if (alnOut) *alnOut = aln;
  return (int) aln.size();
}

template <typename F>
void parallel_for(uint64_t n, int threads, F f) {
  std::atomic<uint64_t> next(0);
  auto work = [&]() { for (;;) { uint64_t i = next.fetch_add(1, std::memory_order_relaxed); if (i >= n) break; f(i); } };
  if (threads <= 1) { work(); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < threads; ++t) th.emplace_back(work);
  for (auto& x : th) x.join();
}

Rows to_rows(const char* rows, int r, int L) {
  Rows a(r);
  for (int i = 0; i < r; ++i) a[i].assign(rows + (size_t) i * L, L);
  return a;
}

}  // namespace

extern "C" {

int ora_edit_distance(const uint8_t* q, int m, const uint8_t* t, int n, int k, int mode, int* end0) {
  return edit_distance(q, m, t, n, k, mode, end0);
}

void ora_edit_distance_batch(const uint8_t* arena, const uint32_t* q_off, const uint32_t* q_len,
                             const uint32_t* t_off, const uint32_t* t_len, const int32_t* k, int mode,
                             uint64_t n, int32_t* dist, int32_t* end_loc, int threads) {
  parallel_for(n, threads, [&](uint64_t i) {
    int e;
    dist[i] = edit_distance(arena + q_off[i], (int) q_len[i], arena + t_off[i], (int) t_len[i], k ? k[i] : -1, mode, &e);
    if (end_loc) end_loc[i] = e;
  });
}

int ora_long_needle(const char* s1, int m, const char* s2, int n, char* rows, long cap, int* alilen) {
  std::string r0, r1;
  *alilen = 0;
  if (!long_needle(std::string(s1, m), std::string(s2, n), r0, r1)) return 0;
  *alilen = (int) r0.size();
  if ((long) (2 * r0.size()) > cap) return -1;
  memcpy(rows, r0.data(), r0.size());
  memcpy(rows + r0.size(), r1.data(), r1.size());
  return 1;
}

int ora_longest_homology(const char* s1, int m, const char* s2, int n, int thr) {
  return longest_homology(std::string(s1, m), std::string(s2, n), thr);
}

int ora_lcs(const char* a, int m, const char* b, int n) { return lcs(std::string(a, m), std::string(b, n)); }

int ora_gotoh(const char* rows1, int r1, int L1, const char* rows2, int r2, int L2,
              int match, int mismatch, int go, int ge, char* out, long cap, int* outL, int* score) {
  Rows o;
  *score = gotoh(to_rows(rows1, r1, L1), to_rows(rows2, r2, L2), match, mismatch, go, ge, o);
  *outL = (int) o[0].size();
  if ((long) (o.size() * o[0].size()) > cap) return -1;
  for (size_t i = 0; i < o.size(); ++i) memcpy(out + i * o[0].size(), o[i].data(), o[0].size());
  return 0;
}

int ora_consensus(const char* rows, int r, int L, int minClique, char* gapped, char* cs, int* cs_len) {
  std::string g, s;
  consensus(to_rows(rows, r, L), minClique, g, s);
  memcpy(gapped, g.data(), g.size());
  memcpy(cs, s.data(), s.size());
  *cs_len = (int) s.size();
  return 0;
}

int ora_msa(const char* arena, const uint32_t* off, const uint32_t* len, int nreads, int minClique,
            int match, int mismatch, int go, int ge, char* cons, int cons_cap, int* cons_len,
            char* aln_out, long aln_cap, int* alnL) {
  std::vector<std::string> reads;
  for (int i = 0; i < nreads; ++i) reads.push_back(std::string(arena + off[i], len[i]));
  std::string cs;
  Rows aln;
  int rows = msa(reads, minClique, match, mismatch, go, ge, cs, &aln);
  *cons_len = (int) cs.size();
  if ((int) cs.size() > cons_cap) return -1;
  memcpy(cons, cs.data(), cs.size());
  if (aln_out) {
    *alnL = (int) aln[0].size();
    if ((long) (aln.size() * aln[0].size()) > aln_cap) return -1;
    for (size_t i = 0; i < aln.size(); ++i) memcpy(aln_out + i * aln[0].size(), aln[i].data(), aln[0].size());
  }
  return rows;
}

// The guide tree's inner nodes of ora_msa's cluster in creation order: (R, L, L1, L2, U1, U2) per node at nodes[6 * k], see NodeInfo.
// Returns the number of nodes, or -1 if there are more than cap.
int ora_msa_nodes(const char* arena, const uint32_t* off, const uint32_t* len, int nreads, int match, int mismatch, int go, int ge,
                  int* nodes, int cap) {
  std::vector<std::string> reads;
  for (int i = 0; i < nreads; ++i) reads.push_back(std::string(arena + off[i], len[i]));
  std::string cs;
  std::vector<NodeInfo> info;
  msa(reads, 2, match, mismatch, go, ge, cs, nullptr, &info);
  if ((int) info.size() > cap) return -1;
  for (size_t k = 0; k < info.size(); ++k) {
    const NodeInfo& x = info[k];
    int* o = nodes + 6 * k;
    o[0] = x.R; o[1] = x.L; o[2] = x.L1; o[3] = x.L2; o[4] = x.U1; o[5] = x.U2;
  }
  return (int) info.size();
}

int ora_hardware_threads() { return (int) std::thread::hardware_concurrency(); }

}  // extern "C"
