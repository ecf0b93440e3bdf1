// msaedlib.hpp — long-read per-SV consensus (SURVEY.md §8 a11): msaEdlib (src/assemble.h:385-473) with
// consensusEdlib (:202-268) and convertAlignment (:24-88), batched over all SV clusters of a chromosome:
//   1 dgpu_edit_distance call  : all-pairs global edit distances of every cluster (src/assemble.h:388-395)
//   host                        : median-distance centroid, order by distance to it, drop the poorest 20 % (:397-422)
//   <= maxReads-1 rounds        : round i aligns the i-th selected read of every cluster against the IUPAC consensus of
//                                 its growing alignment with ONE dgpu_edit_path_ex call (NW, 20 extra equality pairs, :425-447)
//   host                        : coverage-thresholded consensus (src/msa.h:111-173) and the 5 % end trim (:463-467)
// msaWfa (insertions, :549-725) is not mirrored yet.
#pragma once
#include <algorithm>
#include <array>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/dgpu.h"
#include "split.hpp"
#include "splitalign.hpp"

namespace dellyb200 {

// src/assemble.h:202-268 — per column majority over A,C,G,T,other; ambiguous columns become the extended IUPAC letter
inline void consensusEdlib(TAlign const& align, std::string& cons) {
  static const char amb[5][5] = {{0, 'M', 'R', 'W', 'B'}, {0, 0, 'S', 'Y', 'D'}, {0, 0, 0, 'K', 'E'}, {0, 0, 0, 0, 'F'}, {0, 0, 0, 0, 0}};
  const std::size_t L = align.empty() ? 0 : align[0].size();
  cons.assign(L, '-');
  for (std::size_t j = 0; j < L; ++j) {
    int32_t count[5] = {0, 0, 0, 0, 0};
    for (std::string const& row : align) {
      switch (row[j]) {
        case 'A': case 'a': ++count[0]; break;
        case 'C': case 'c': ++count[1]; break;
        case 'G': case 'g': ++count[2]; break;
        case 'T': case 't': ++count[3]; break;
        default: ++count[4]; break;
      }
    }
    uint32_t maxIdx = 0, sndIdx = 1;
    if (count[0] < count[1]) { maxIdx = 1; sndIdx = 0; }
    for (uint32_t i = 2; i < 5; ++i) {
      if (count[i] > count[maxIdx]) { sndIdx = maxIdx; maxIdx = i; }
      else if (count[i] > count[sndIdx]) sndIdx = i;
    }
    if (2 * count[sndIdx] < count[maxIdx]) cons[j] = (maxIdx < 4) ? "ACGT"[maxIdx] : '-';
    else {
      const uint32_t k1 = std::min(maxIdx, sndIdx), k2 = std::max(maxIdx, sndIdx);
      cons[j] = amb[k1][k2] ? amb[k1][k2] : '-';
    }
  }
}

// The same vote from per-column letter counts (A, C, G, T, other) — what consensusEdlib computes from the rows. msaEdlibBatch keeps the counts of a
// growing alignment up to date (one pass over the edit path per added row) instead of re-reading every row in every round.
typedef std::array<int32_t, 5> TColCount;
inline int edlibBucket(char ch) {
  switch (ch) {
    case 'A': case 'a': return 0;
    case 'C': case 'c': return 1;
    case 'G': case 'g': return 2;
    case 'T': case 't': return 3;
    default: return 4;
  }
}
inline void consensusFromCounts(std::vector<TColCount> const& counts, std::string& cons) {
  static const char amb[5][5] = {{0, 'M', 'R', 'W', 'B'}, {0, 0, 'S', 'Y', 'D'}, {0, 0, 0, 'K', 'E'}, {0, 0, 0, 0, 'F'}, {0, 0, 0, 0, 0}};
  const std::size_t L = counts.size();
  cons.assign(L, '-');
  for (std::size_t j = 0; j < L; ++j) {
    TColCount const& count = counts[j];
    uint32_t maxIdx = 0, sndIdx = 1;
    if (count[0] < count[1]) { maxIdx = 1; sndIdx = 0; }
    for (uint32_t i = 2; i < 5; ++i) {
      if (count[i] > count[maxIdx]) { sndIdx = maxIdx; maxIdx = i; }
      else if (count[i] > count[sndIdx]) sndIdx = i;
    }
    if (2 * count[sndIdx] < count[maxIdx]) cons[j] = (maxIdx < 4) ? "ACGT"[maxIdx] : '-';
    else {
      const uint32_t k1 = std::min(maxIdx, sndIdx), k2 = std::max(maxIdx, sndIdx);
      cons[j] = amb[k1][k2] ? amb[k1][k2] : '-';
    }
  }
}
// the counts after convertAlignmentNW(query, align, ops): an inserted column holds a gap in every earlier row
inline void countsAfterRow(std::string const& query, std::size_t rowsBefore, std::string const& ops, std::vector<TColCount>& counts) {
  std::vector<TColCount> out(ops.size());
  int32_t tIdx = -1, qIdx = -1;
  for (std::size_t j = 0; j < ops.size(); ++j) {
    if (ops[j] != 1) out[j] = counts[(std::size_t) ++tIdx];
    else { out[j] = TColCount{{0, 0, 0, 0, (int32_t) rowsBefore}}; }
    ++out[j][(ops[j] != 2) ? edlibBucket(query[(std::size_t) ++qIdx]) : 4];
  }
  counts.swap(out);
}

// src/assemble.h:24-88 for EDLIB_MODE_NW: add `query` as a new last row along the path (ops against the consensus string)
inline void convertAlignmentNW(std::string const& query, TAlign& align, std::string const& ops) {
  const std::size_t R = align.size(), L = ops.size();
  TAlign out(R + 1, std::string(L, '-'));
  int32_t tIdx = -1, qIdx = -1;
  for (std::size_t j = 0; j < L; ++j) {
    if (ops[j] != 1) { ++tIdx; for (std::size_t r = 0; r < R; ++r) out[r][j] = align[r][tIdx]; }
    if (ops[j] != 2) out[R][j] = query[++qIdx];
  }
  align.swap(out);
}

// src/msa.h:111-173 (host flavour; the short-read path runs the same vote inside dgpu_msa)
inline void consensusRows(Config const& c, TAlign const& align, std::string& gapped, std::string& cs) {
  const std::size_t R = align.size(), L = R ? align[0].size() : 0;
  std::vector<int> cov(L, 0);
  std::vector<long> st(R), en(R);
  for (std::size_t i = 0; i < R; ++i) {
    long s = 0, e = -1;
    for (std::size_t j = 0; j < L; ++j) { if (align[i][j] != '-') e = (long) j; else if (e == -1) s = (long) j + 1; }
    st[i] = s; en[i] = e;
    for (long j = s; j <= e; ++j) ++cov[j];
  }
  const int thr = std::max(2, std::min((int) c.minCliqueSize, (int) R));
  gapped.assign(L, '-');
  for (std::size_t j = 0; j < L; ++j) {
    if (cov[j] < thr) continue;
    int cnt[5] = {0, 0, 0, 0, 0};
    for (std::size_t i = 0; i < R; ++i) {
      if (st[i] > (long) j || (long) j > en[i]) continue;
      switch (align[i][j]) {
        case 'A': case 'a': ++cnt[0]; break;
        case 'C': case 'c': ++cnt[1]; break;
        case 'G': case 'g': ++cnt[2]; break;
        case 'T': case 't': ++cnt[3]; break;
        default: ++cnt[4]; break;
      }
    }
    int mi = 0;
    for (int x = 1; x < 5; ++x) if (cnt[x] > cnt[mi]) mi = x;
    if (mi < 4) gapped[j] = "ACGT"[mi];
  }
  cs.clear();
  for (char ch : gapped) if (ch != '-') cs.push_back(ch);
}

// Batched msaEdlib: clusters[i] = reads of SV i (caller's order). consensus[i], rows[i] = msaEdlib's cs and return value.
inline int msaEdlibBatch(dgpu_ctx* ctx, Config const& c, std::vector<std::vector<std::string> > const& clusters, std::vector<std::string>& consensus,
                         std::vector<int>& rows) {
  static const uint8_t iupac[40] = {'M', 'A', 'M', 'C', 'R', 'A', 'R', 'G', 'W', 'A', 'W', 'T', 'B', 'A', 'B', '-', 'S', 'C', 'S', 'G',
                                    'Y', 'C', 'Y', 'T', 'D', 'C', 'D', '-', 'K', 'G', 'K', 'T', 'E', 'G', 'E', '-', 'F', 'T', 'F', '-'};
  const std::size_t N = clusters.size();
  consensus.assign(N, std::string());
  rows.assign(N, 0);
  if (!N) return DGPU_OK;
  int rc;
  // stage clock (DGPU_TIMING=1: one line on stderr)
  const bool timing = getenv("DGPU_TIMING") != nullptr;
  double tDist = 0, tSelect = 0, tFold = 0, tPath = 0, tConvert = 0, tFinal = 0;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  double t0 = now();
  auto lap = [&](double& acc) { const double t = now(); acc += t - t0; t0 = t; };
  // ---- all-pairs global edit distances ----------------------------------------------------------------------------
  std::vector<std::vector<int32_t> > edit(N);
  {
    std::string arena;
    std::vector<std::vector<uint32_t> > off(N);
    for (std::size_t i = 0; i < N; ++i)
      for (std::string const& r : clusters[i]) { off[i].push_back((uint32_t) arena.size()); arena += r; }
    std::vector<uint32_t> qo, ql, to, tl;
    for (std::size_t i = 0; i < N; ++i) {
      const std::size_t S = clusters[i].size();
      for (std::size_t a = 0; a < S; ++a)
        for (std::size_t b = a + 1; b < S; ++b) {
          qo.push_back(off[i][a]); ql.push_back((uint32_t) clusters[i][a].size());
          to.push_back(off[i][b]); tl.push_back((uint32_t) clusters[i][b].size());
        }
    }
    std::vector<int32_t> dist(qo.size());
    if (!qo.empty()) {
      rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), nullptr, DGPU_MODE_NW, qo.size(),
                              dist.data(), nullptr);
      if (rc) return rc;
    }
    std::size_t k = 0;
    for (std::size_t i = 0; i < N; ++i) {
      const std::size_t S = clusters[i].size();
      edit[i].assign(S * S, 0);
      for (std::size_t a = 0; a < S; ++a)
        for (std::size_t b = a + 1; b < S; ++b) { edit[i][a * S + b] = edit[i][b * S + a] = dist[k++]; }
    }
  }
  lap(tDist);
  // ---- centroid, ordering, selection (src/assemble.h:397-422) --------------------------------------------------------------
  std::vector<std::vector<uint32_t> > sel(N);
  std::vector<TAlign> aligns(N);
  std::vector<std::vector<TColCount> > colCounts(N);   // letter counts per column of aligns[i], kept in step with it
  std::vector<uint8_t> broken(N, 0);   // a progressive round of this cluster exceeded a device limit: no consensus (counted in deviceLimitLog)
  std::size_t maxSel = 0;
  for (std::size_t i = 0; i < N; ++i) {
    std::vector<std::string> const& sps = clusters[i];
    const std::size_t S = sps.size();
    if (!S) continue;
    uint32_t bestIdx = 0;
    int32_t bestVal = (int32_t) sps[0].size();
    for (uint32_t a = 0; a < S; ++a) {
      std::vector<int32_t> d(edit[i].begin() + a * S, edit[i].begin() + (a + 1) * S);
      std::sort(d.begin(), d.end());
      if (d[S / 2] < bestVal) { bestVal = d[S / 2]; bestIdx = a; }
    }
    std::vector<std::pair<int32_t, int32_t> > qs;
    qs.push_back(std::make_pair(0, (int32_t) bestIdx));
    for (uint32_t j = 0; j < S; ++j) if (j != bestIdx) qs.push_back(std::make_pair(edit[i][bestIdx * S + j], (int32_t) j));
    std::sort(qs.begin(), qs.end());
    uint32_t lastIdx = (uint32_t) (0.8 * qs.size());
    if (lastIdx < 3) lastIdx = 3;
    for (uint32_t k = 0; k < qs.size() && k < lastIdx; ++k) sel[i].push_back((uint32_t) qs[k].second);
    aligns[i].assign(1, sps[sel[i][0]]);
    colCounts[i].assign(aligns[i][0].size(), TColCount{{0, 0, 0, 0, 0}});
    for (std::size_t j = 0; j < aligns[i][0].size(); ++j) ++colCounts[i][j][edlibBucket(aligns[i][0][j])];
    maxSel = std::max(maxSel, sel[i].size());
  }
  lap(tSelect);
  // ---- progressive rounds -----------------------------------------------------------------------------------------------
  for (std::size_t round = 1; round < maxSel; ++round) {
    std::vector<uint32_t> who;
    std::string arena;
    std::vector<uint32_t> qo, ql, to, tl;
    std::vector<uint64_t> oo;
    uint64_t obytes = 0;
    std::vector<std::string> alignStrs(N);
    parallelFor(N, [&](std::size_t i) { if (!((sel[i].size() <= round) || broken[i])) consensusFromCounts(colCounts[i], alignStrs[i]); });
    for (std::size_t i = 0; i < N; ++i) {
      if ((sel[i].size() <= round) || broken[i]) continue;
      std::string const& alignStr = alignStrs[i];
      std::string const& q = clusters[i][sel[i][round]];
      who.push_back((uint32_t) i);
      qo.push_back((uint32_t) arena.size()); ql.push_back((uint32_t) q.size()); arena += q;
      to.push_back((uint32_t) arena.size()); tl.push_back((uint32_t) alignStr.size()); arena += alignStr;
      oo.push_back(obytes); obytes += q.size() + alignStr.size();
    }
    lap(tFold);
    const std::size_t J = who.size();
    std::vector<int32_t> dist(J), st(J), en(J);
    std::vector<uint32_t> olen(J), status(J);
    std::vector<uint8_t> ops(obytes + 1);
    rc = editPathCall(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), DGPU_MODE_NW, iupac, 20, J, dist.data(),
                      st.data(), en.data(), ops.data(), oo.data(), obytes, olen.data(), status.data());
    if (rc) return rc;
    lap(tPath);
    for (std::size_t k = 0; k < J; ++k)
      if (status[k]) { ++deviceLimitLog().pathJobs; aligns[who[k]].clear(); broken[who[k]] = 1; }   // this cluster yields no consensus
    parallelFor(J, [&](std::size_t k) {   // a cluster appears once per round
      if (broken[who[k]]) return;
      const std::string path((const char*) ops.data() + oo[k], olen[k]);
      countsAfterRow(clusters[who[k]][sel[who[k]][round]], aligns[who[k]].size(), path, colCounts[who[k]]);
      convertAlignmentNW(clusters[who[k]][sel[who[k]][round]], aligns[who[k]], path);
    });
    lap(tConvert);
  }
  // ---- consensus + trim (src/assemble.h:458-467) ---------------------------------------------------------------------------
  parallelFor(N, [&](std::size_t i) {
    if (aligns[i].empty()) return;
    std::string gapped, cs;
    consensusRows(c, aligns[i], gapped, cs);
    int32_t trim = (int32_t) (0.05 * cs.size());
    if (trim > 50) trim = 50;
    const int32_t len = (int32_t) cs.size() - 2 * trim;
    if (len > 100) cs = cs.substr(trim, len);
    consensus[i] = cs;
    rows[i] = (int) aligns[i].size();
  });
  lap(tFinal);
  if (timing) fprintf(stderr, "[msaEdlibBatch] clusters %zu: all-pairs distance %.1f ms, selection %.1f, consensus of the growing alignments %.1f, path rounds %.1f, convert %.1f, final %.1f\n",
                      N, tDist, tSelect, tFold, tPath, tConvert, tFinal);
  return DGPU_OK;
}

}  // namespace dellyb200
