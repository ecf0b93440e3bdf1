// splitalign.hpp — consensus-vs-reference alignment for insertions (SURVEY.md §8 a10): splitAlign,
// editDistanceVec, glueAlignment, infixStart/infixEnd with the six per-SV edlib PATH calls of the reference
// (src/split.h:378-537, src/util.h:86-99) replaced by THREE batched dgpu_edit_path rounds over all SVs:
//   round 1  prefix third / suffix third of the SV reference inside the consensus (HW)   -> consensus core [csStart, csEnd)
//   round 2  SV reference vs core, forward and reverse-complemented (SHW)                 -> per-position edit counts, best join
//   round 3  left / right part of the SV reference inside the consensus (HW)              -> glued 2-row alignment
#pragma once
#include <string>
#include <vector>

#include "../../include/dgpu.h"
#include "split.hpp"

namespace dellyb200 {

struct EdPath {  // what the reference reads from an EdlibAlignResult of a PATH call
  int32_t editDistance = -1, start = -1, end = -1;
  std::string ops;  // 0 match, 1 insert, 2 delete, 3 mismatch
  bool failed = false;  // the job exceeded a device limit (counted in deviceLimitLog): the caller treats the alignment as failed
};

// One batched edlibAlign(query, target, k=-1, mode, EDLIB_TASK_PATH[, additionalEqualities]) round.
inline int editPathBatch(dgpu_ctx* ctx, std::vector<std::pair<std::string, std::string> > const& qt, int mode, std::vector<EdPath>& out,
                         const uint8_t* eq_pairs = nullptr, uint32_t n_eq = 0) {
  const std::size_t N = qt.size();
  out.assign(N, EdPath());
  if (!N) return DGPU_OK;
  std::string arena;
  std::vector<uint32_t> qo(N), ql(N), to(N), tl(N);
  std::vector<uint64_t> oo(N);
  uint64_t obytes = 0;
  for (std::size_t i = 0; i < N; ++i) {
    qo[i] = (uint32_t) arena.size(); ql[i] = (uint32_t) qt[i].first.size(); arena += qt[i].first;
    to[i] = (uint32_t) arena.size(); tl[i] = (uint32_t) qt[i].second.size(); arena += qt[i].second;
    oo[i] = obytes; obytes += qt[i].first.size() + qt[i].second.size();
  }
  std::vector<int32_t> dist(N), st(N), en(N);
  std::vector<uint32_t> olen(N), status(N);
  std::vector<uint8_t> ops(obytes + 1);
  int rc = editPathCall(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), mode, eq_pairs, n_eq, N, dist.data(),
                        st.data(), en.data(), ops.data(), oo.data(), obytes, olen.data(), status.data());
  if (rc) return rc;
  for (std::size_t i = 0; i < N; ++i) {
    if (status[i]) { ++deviceLimitLog().pathJobs; out[i].failed = true; out[i].end = 0; out[i].start = 0; continue; }   // never approximated: failed, counted
    out[i].editDistance = dist[i]; out[i].start = st[i]; out[i].end = en[i];
    out[i].ops.assign((const char*) ops.data() + oo[i], olen[i]);
  }
  return DGPU_OK;
}

// src/util.h:86-99
inline uint32_t infixStart(EdPath const& c) {
  int32_t tIdx = c.end;
  for (char op : c.ops) if (op != 1) --tIdx;
  return (tIdx >= 0) ? (uint32_t) (tIdx + 1) : 0u;
}
inline uint32_t infixEnd(EdPath const& c) { return (uint32_t) c.end; }

// src/split.h:378-406 — running edit count at every query position along the path
inline void editDistanceVec(std::string const& seqI, std::string const& seqJ, EdPath const& c, std::vector<uint32_t>& dist) {
  dist.assign(seqI.size(), 0);
  int32_t t = -1, q = -1;
  uint32_t edits = 0;
  for (char op : c.ops) {
    if (op == 2) { ++t; ++edits; }
    else if (op == 1) { ++q; ++edits; dist[q] = edits; }
    else { ++t; ++q; if (seqI[q] != seqJ[t]) ++edits; dist[q] = edits; }
  }
}

// src/split.h:408-477 — stitch the left and right infix alignments of the query parts around `gaplen` unaligned target bases
inline void glueAlignment(std::string const& query, std::string const& target, uint32_t gaplen, EdPath const& left, EdPath const& right, TAlign& align) {
  int32_t tIdx = left.end;
  for (char op : left.ops) if (op != 1) --tIdx;
  const uint32_t missingStart = (tIdx >= 0) ? (uint32_t) (tIdx + 1) : 0u;
  uint32_t missingEnd = (uint32_t) right.end;
  if (missingEnd < target.size()) missingEnd = (uint32_t) (target.size() - missingEnd - 1);
  std::string rowQ, rowT;
  int32_t qIdx = -1;
  rowT.assign(target, 0, missingStart); rowQ.assign(missingStart, '-');
  auto emit = [&](EdPath const& c) {
    for (char op : c.ops) {
      rowT.push_back(op == 1 ? '-' : target[++tIdx]);
      rowQ.push_back(op == 2 ? '-' : query[++qIdx]);
    }
  };
  emit(left);
  for (uint32_t j = 0; j < gaplen; ++j) { rowQ.push_back('-'); rowT.push_back(target[++tIdx]); }
  emit(right);
  for (uint32_t j = 0; j < missingEnd; ++j) { rowT.push_back(target[++tIdx]); rowQ.push_back('-'); }
  align.assign(2, std::string());
  align[0] = rowQ; align[1] = rowT;
}

// Batched splitAlign (src/split.h:480-537): ok[i] and aligns[i] (row 0 = SV reference, row 1 = consensus, as the reference
// leaves them before _consRefAlignment swaps the rows, src/split.h:546-553).
inline int splitAlignBatch(dgpu_ctx* ctx, std::vector<std::string> const& cons, std::vector<std::string> const& refs, std::vector<uint8_t>& ok,
                           std::vector<TAlign>& aligns) {
  const std::size_t N = cons.size();
  ok.assign(N, 0);
  aligns.assign(N, TAlign());
  if (!N) return DGPU_OK;
  int rc;
  // ---- round 1 -------------------------------------------------------------------------------------------
  std::vector<std::pair<std::string, std::string> > qt;
  for (std::size_t i = 0; i < N; ++i) {
    qt.push_back(std::make_pair(refs[i].substr(0, refs[i].size() / 3), cons[i]));
    qt.push_back(std::make_pair(refs[i].substr(2 * refs[i].size() / 3), cons[i]));
  }
  std::vector<EdPath> r1;
  if ((rc = editPathBatch(ctx, qt, DGPU_MODE_HW, r1))) return rc;
  std::vector<uint32_t> live;
  std::vector<std::string> cs;
  for (std::size_t i = 0; i < N; ++i) {
    if (r1[2 * i].failed || r1[2 * i + 1].failed) continue;
    const uint32_t csStart = infixStart(r1[2 * i]), csEnd = infixEnd(r1[2 * i + 1]);
    if (csStart >= csEnd) continue;
    live.push_back((uint32_t) i);
    cs.push_back(csStart <= cons[i].size() ? cons[i].substr(csStart, csEnd - csStart) : std::string());
  }
  // ---- round 2 -------------------------------------------------------------------------------------------
  qt.clear();
  for (std::size_t k = 0; k < live.size(); ++k) {
    std::string rr = refs[live[k]], cr = cs[k];
    reverseComplement(rr); reverseComplement(cr);
    qt.push_back(std::make_pair(refs[live[k]], cs[k]));
    qt.push_back(std::make_pair(rr, cr));
  }
  std::vector<EdPath> r2;
  if ((rc = editPathBatch(ctx, qt, DGPU_MODE_SHW, r2))) return rc;
  std::vector<uint32_t> bestJoin(live.size(), 0);
  std::vector<uint8_t> dead(live.size(), 0);
  for (std::size_t k = 0; k < live.size(); ++k) {
    if (r2[2 * k].failed || r2[2 * k + 1].failed) { dead[k] = 1; continue; }
    std::vector<uint32_t> fwd, rev;
    editDistanceVec(qt[2 * k].first, qt[2 * k].second, r2[2 * k], fwd);
    editDistanceVec(qt[2 * k + 1].first, qt[2 * k + 1].second, r2[2 * k + 1], rev);
    uint32_t bj = 0;
    const std::size_t S = fwd.size();
    for (uint32_t i = 1; i + 1 < S; ++i)
      if (fwd[i] + rev[S - i - 2] < fwd[bj] + rev[S - bj - 2]) bj = i;
    bestJoin[k] = bj;
  }
  // ---- round 3 -------------------------------------------------------------------------------------------
  qt.clear();
  for (std::size_t k = 0; k < live.size(); ++k) {
    const std::string& r = refs[live[k]];
    qt.push_back(std::make_pair(r.substr(0, bestJoin[k] + 1), cons[live[k]]));
    qt.push_back(std::make_pair(r.substr(bestJoin[k] + 1), cons[live[k]]));
  }
  std::vector<EdPath> r3;
  if ((rc = editPathBatch(ctx, qt, DGPU_MODE_HW, r3))) return rc;
  for (std::size_t k = 0; k < live.size(); ++k) {
    if (dead[k] || r3[2 * k].failed || r3[2 * k + 1].failed) continue;
    const uint32_t leftEnd = infixEnd(r3[2 * k]), rightStart = infixStart(r3[2 * k + 1]);
    if (leftEnd + 15 >= rightStart) continue;
    glueAlignment(refs[live[k]], cons[live[k]], rightStart - leftEnd - 1, r3[2 * k], r3[2 * k + 1], aligns[live[k]]);
    ok[live[k]] = 1;
  }
  return DGPU_OK;
}

}  // namespace dellyb200
