// split.hpp — consensus-to-reference breakpoint refinement around the batched device alignment
// (SURVEY.md §8 a9 + the alignConsensus driver). Same names and argument meaning as the reference:
//   src/util.h:549-563   reverseComplement
//   src/split.h:70-163   _getSVRef            (SV-type specific reference window)
//   src/split.h:166-244  _coordTransform
//   src/split.h:247-260  _validSRAlignment, _checkSVGap
//   src/split.h:262-280  _findHomology  -> src/needle.h:13-42 longestHomology
//   src/split.h:282-316  _percentIdentity
//   src/split.h:319-375  _findSplit
//   src/split.h:560-672  _alignConsensus / alignConsensus   (here: alignConsensusBatch, one device call per batch)
// The per-SV longNeedle call (src/split.h:555) is replaced by ONE dgpu_long_needle call for the whole
// batch; everything after it is O(alignment length) host work done exactly as the reference does it
// (including the single float division of _percentIdentity).
#pragma once
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/dgpu.h"
#include "editpath.hpp"
#include "types.hpp"

namespace dellyb200 {

typedef std::vector<std::string> TAlign;  // TAlign[0] = consensus row, TAlign[1] = reference row

inline void reverseComplement(std::string& sequence) {
  const std::string orig = sequence;
  const std::size_t L = orig.size();
  for (std::size_t i = 0; i < L; ++i) {
    switch (std::toupper((unsigned char) orig[L - 1 - i])) {
      case 'A': sequence[i] = 'T'; break;
      case 'C': sequence[i] = 'G'; break;
      case 'G': sequence[i] = 'C'; break;
      case 'T': sequence[i] = 'A'; break;
      case 'N': sequence[i] = 'N'; break;
      default: break;  // the reference keeps the original byte at this index
    }
  }
}

namespace detail {
inline std::string upperSlice(const char* ref, int32_t b, int32_t e) {
  std::string s(ref + b, ref + e);
  for (char& c : s) c = (char) std::toupper((unsigned char) c);
  return s;
}
// Upper-cased slice, reversed and complemented the way _getSVRef does it (src/split.h:78-90): bytes other
// than ACGTN keep the forward-slice byte at that index.
inline std::string rcSlice(const char* ref, int32_t b, int32_t e) {
  const std::string fwd = upperSlice(ref, b, e);
  std::string out = fwd;
  const std::size_t L = fwd.size();
  for (std::size_t i = 0; i < L; ++i) {
    switch (fwd[L - 1 - i]) {
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
}  // namespace detail

// src/split.h:70-163. `ref` is the sequence of contig `refIndex`.
inline std::string _getSVRef(Config const& c, const char* ref, Breakpoint const& bp, int32_t refIndex, int32_t svt) {
  using detail::rcSlice;
  using detail::upperSlice;
  if (_translocation(svt)) {
    const uint8_t ct = _getSpanOrientation(svt);
    if (bp.chr == refIndex) {
      if (ct == 0 || ct == 2) return upperSlice(ref, bp.svStartBeg, bp.svStartEnd) + bp.part1;
      if (ct == 1) return rcSlice(ref, bp.svStartBeg, bp.svStartEnd) + bp.part1;
      return bp.part1 + upperSlice(ref, bp.svStartBeg, bp.svStartEnd);
    }
    if (ct == 0) return rcSlice(ref, bp.svEndBeg, bp.svEndEnd);
    return upperSlice(ref, bp.svEndBeg, bp.svEndEnd);
  }
  const bool large = (bp.svEnd - bp.svStart) > c.minConsWindow;
  switch (svt) {
    case 2:
      if (bp.svEnd - bp.svStart <= c.indelsize) return upperSlice(ref, bp.svStartBeg, bp.svEndEnd);
      return upperSlice(ref, bp.svStartBeg, bp.svStartEnd) + upperSlice(ref, bp.svEndBeg, bp.svEndEnd);
    case 4: return upperSlice(ref, bp.svStartBeg, bp.svEndEnd);
    case 3: return upperSlice(ref, bp.svEndBeg, bp.svEndEnd) + upperSlice(ref, bp.svStartBeg, bp.svStartEnd);
    case 0:
      if (large) return upperSlice(ref, bp.svStartBeg, bp.svStartEnd) + rcSlice(ref, bp.svEndBeg, bp.svEndEnd);
      return upperSlice(ref, bp.svStartBeg, bp.svStartEnd) + rcSlice(ref, bp.svStart, bp.svEndEnd) + upperSlice(ref, bp.svEnd, bp.svEndEnd);
    case 1:
      if (large) return rcSlice(ref, bp.svStartBeg, bp.svStartEnd) + upperSlice(ref, bp.svEndBeg, bp.svEndEnd);
      return upperSlice(ref, bp.svStartBeg, bp.svStart) + rcSlice(ref, bp.svStartBeg, bp.svEnd) + upperSlice(ref, bp.svEndBeg, bp.svEndEnd);
    default: return "";
  }
}

// src/split.h:166-244
inline bool _coordTransform(Config const& c, std::string const& ref, Breakpoint const& sv, AlignDescriptor const& ad, uint32_t& finalGapStart,
                            uint32_t& finalGapEnd, int32_t svt) {
  const int32_t annStart = sv.svStartEnd - sv.svStartBeg;
  const int32_t annEnd = sv.svEndEnd - sv.svEndBeg;
  auto straddles = [&](int32_t annealed) { return !((ad.rStart >= annealed) || (ad.rEnd < annealed)); };
  // the four junction geometries, named by the translocation connection type they correspond to
  auto geo0 = [&]() { if (!straddles(annStart)) return false; finalGapStart = sv.svStartBeg + ad.rStart; finalGapEnd = sv.svEndBeg + (ref.size() - ad.rEnd) + 1; return true; };
  auto geo1 = [&](int32_t annealed) { if (!straddles(annealed)) return false; finalGapStart = sv.svStartBeg + (annealed - ad.rStart) + 1; finalGapEnd = sv.svEndBeg + (ad.rEnd - annealed); return true; };
  auto geo2 = [&]() { if (!straddles(annStart)) return false; finalGapStart = sv.svStartBeg + ad.rStart; finalGapEnd = sv.svEndBeg + (ad.rEnd - annStart); return true; };
  auto geo3 = [&]() { if (!straddles(annEnd)) return false; finalGapStart = sv.svStartBeg + (ad.rEnd - annEnd); finalGapEnd = sv.svEndBeg + ad.rStart; return true; };
  if (_translocation(svt)) {
    switch (_getSpanOrientation(svt)) {
      case 0: return geo0();
      case 1: return geo1(annStart);
      case 2: return geo2();
      case 3: return geo3();
      default: return false;
    }
  }
  switch (svt) {
    case 2:
      if (sv.svEnd - sv.svStart > c.indelsize) return geo2();
      finalGapStart = sv.svStartBeg + ad.rStart; finalGapEnd = sv.svStartBeg + ad.rEnd; return true;
    case 3: return geo3();
    case 0:
      if ((sv.svEnd - sv.svStart) > c.minConsWindow) return geo0();
      if (!straddles(annStart)) return false;
      finalGapStart = sv.svStartBeg + ad.rStart; finalGapEnd = sv.svEndEnd - (ad.rEnd - annStart); return true;
    case 1:
      if ((sv.svEnd - sv.svStart) > c.minConsWindow) return geo1(annStart);
      return geo1((sv.svStart - sv.svStartBeg) + (sv.svEnd - sv.svStartBeg));
    case 4: finalGapStart = sv.svStartBeg + ad.rStart; finalGapEnd = sv.svStartBeg + ad.rEnd; return true;
    default: return true;
  }
}

inline bool _validSRAlignment(int32_t cStart, int32_t cEnd, int32_t rStart, int32_t rEnd, int32_t svt) {
  if (svt == 4) return ((rEnd - rStart) < 5) && ((cEnd - cStart) > 15);
  return ((cEnd - cStart) < 5) && ((rEnd - rStart) > 15);
}

// src/needle.h:13-42 — banded (|row-col| <= k) unit-cost DP; number of leading rows whose best banded
// score stays >= scoreThreshold (row-1 at the first failure, 0 if it never fails). Rolling rows; cells
// outside the band are never read, like in the reference's full matrix.
inline int32_t longestHomology(std::string const& s1, std::string const& s2, int32_t scoreThreshold) {
  const int32_t m = (int32_t) s1.size(), n = (int32_t) s2.size(), k = std::abs(scoreThreshold);
  std::vector<int32_t> prev(n + 2, 0), cur(n + 2, 0);
  for (int32_t col = 1; col <= std::min(k, n); ++col) prev[col] = prev[col - 1] - 1;
  for (int32_t row = 1; row <= m; ++row) {
    if (row <= k) cur[0] = -row;
    int32_t bestCol = scoreThreshold - 1;
    for (int32_t col = std::max(1, row - k); col <= std::min(n, row + k); ++col) {
      int32_t v = prev[col - 1] + (s1[row - 1] == s2[col - 1] ? 0 : -1);
      if (std::abs(row - 1 - col) <= k) v = std::max(v, prev[col] - 1);
      if (std::abs(row - col + 1) <= k) v = std::max(v, cur[col - 1] - 1);
      cur[col] = v;
      bestCol = std::max(bestCol, v);
    }
    if (bestCol < scoreThreshold) return row - 1;
    prev.swap(cur);
  }
  return 0;
}

// src/split.h:262-280
inline void _findHomology(std::string const& consensus, std::string const& svRefStr, AlignDescriptor& ad, int32_t svt) {
  std::string sufC, sufR, preC, preR;
  if (svt == 4) {
    sufC = consensus.substr(ad.cStart); sufR = svRefStr.substr(ad.rEnd - 1);
    preC = consensus.substr(0, ad.cEnd - 1); preR = svRefStr.substr(0, ad.rStart);
  } else {
    sufC = consensus.substr(ad.cEnd - 1); sufR = svRefStr.substr(ad.rStart);
    preC = consensus.substr(0, ad.cStart); preR = svRefStr.substr(0, ad.rEnd - 1);
  }
  ad.homRight = longestHomology(sufC, sufR, -1);
  std::reverse(preC.begin(), preC.end());
  std::reverse(preR.begin(), preR.end());
  ad.homLeft = longestHomology(preC, preR, -1);
}

// src/split.h:282-316 — identity of the flanks outside alignment columns [gS, gE]; every other internal gap
// counts its length as mismatches once the gap closes.
inline void _percentIdentity(TAlign const& align, int32_t gS, int32_t gE, float& percId) {
  bool varSeen = false, refSeen = false, inGap = false;
  uint32_t gapMM = 0, mm = 0, ma = 0;
  const int32_t L = (int32_t) align[0].size();
  for (int32_t j = 0; j < L; ++j) {
    if (j >= gS && j <= gE) continue;
    const char a = align[0][j], b = align[1][j];
    if (a != '-') varSeen = true;
    if (b != '-') refSeen = true;
    if (a == '-' || b == '-') {
      if (refSeen && varSeen) {
        if (!inGap) { inGap = true; gapMM = 0; }
        gapMM += 1;
      }
    } else {
      if (inGap) { mm += gapMM; inGap = false; }
      if (a == b) ma += 1; else mm += 1;
    }
  }
  percId = (float) ma / (float) (ma + mm);
}

// src/split.h:319-375
inline bool _findSplit(Config const& c, std::string const& consensus, std::string const& svRefStr, TAlign const& align, AlignDescriptor& ad,
                       int32_t svt) {
  int32_t gS = 0, gE = 0, refIndex = 0, varIndex = 0, gapStartRef = 0, gapStartVar = 0, a1 = 0;
  bool inGap = false;
  const int32_t L = (int32_t) align[0].size();
  for (int32_t j = 0; j < L; ++j) {
    const bool v = align[0][j] != '-', r = align[1][j] != '-';
    if (v) ++varIndex;
    if (r) ++refIndex;
    if ((!v || !r) && refIndex > 0 && varIndex > 0) {
      if (!inGap) {
        gapStartVar = v ? varIndex - 1 : varIndex;
        gapStartRef = r ? refIndex - 1 : refIndex;
        a1 = j;
        inGap = true;
      }
    } else {
      if (inGap) {
        const bool better = (svt == 4) ? ((varIndex - gapStartVar) > (ad.cEnd - ad.cStart)) : ((refIndex - gapStartRef) > (ad.rEnd - ad.rStart));
        if (better) {
          ad.rStart = gapStartRef; ad.rEnd = refIndex; ad.cStart = gapStartVar; ad.cEnd = varIndex;
          gS = a1; gE = j - 1;
        }
      }
      inGap = false;
    }
  }
  if (ad.rEnd <= ad.rStart) return false;
  if (!_validSRAlignment(ad.cStart, ad.cEnd, ad.rStart, ad.rEnd, svt)) return false;
  _percentIdentity(align, gS, gE, ad.percId);
  if (ad.percId < c.flankQuality) return false;
  _findHomology(consensus, svRefStr, ad, svt);
  if ((ad.homLeft + c.minimumFlankSize > ad.cStart) || (varIndex < ad.cEnd + ad.homRight + c.minimumFlankSize)) return false;
  if ((ad.homLeft + c.minimumFlankSize > ad.rStart) || (refIndex < ad.rEnd + ad.homRight + c.minimumFlankSize)) return false;
  return true;
}

// Everything of _alignConsensus after the alignment exists (src/split.h:583-644).
inline bool _finishAlignConsensus(Config const& c, std::string const& consensus, std::string const& svRefStr, TAlign const& align,
                                  StructuralVariantRecord& sv, Breakpoint const& bp) {
  AlignDescriptor ad;
  if (!_findSplit(c, consensus, svRefStr, align, ad, sv.svt)) return false;
  uint32_t finalGapStart = 0, finalGapEnd = 0;
  if (!_coordTransform(c, svRefStr, bp, ad, finalGapStart, finalGapEnd, sv.svt)) return false;
  if (!(_translocation(sv.svt) || (finalGapStart < finalGapEnd))) return false;
  if ((sv.svEnd - sv.svStart <= c.indelsize) && (sv.svt == 2 || sv.svt == 4)) {
    std::string refVCF, altVCF;
    int32_t cpos = 0;
    bool inSV = false;
    for (std::size_t j = 0; j < align[0].size(); ++j) {
      if (align[0][j] != '-') {
        ++cpos;
        if (cpos == ad.cStart) inSV = true;
        else if (cpos == ad.cEnd) inSV = false;
      }
      if (inSV) {
        if (align[0][j] != '-') altVCF += align[0][j];
        if (align[1][j] != '-') refVCF += align[1][j];
      }
    }
    sv.alleles = refVCF + "," + altVCF;  // _addAlleles(ref, alt), src/util.h:250-253
  }
  sv.precise = true;
  sv.svStart = (int32_t) finalGapStart;
  sv.svEnd = (int32_t) finalGapEnd;
  sv.srAlignQuality = ad.percId;
  sv.insLen = ad.cEnd - ad.cStart - 1;
  sv.consBp = ad.cStart;
  sv.homLen = std::max(0, ad.homLeft + ad.homRight - 2);
  const int32_t ci = std::max(ad.homLeft, ad.homRight);
  sv.ciposlow = -ci; sv.ciposhigh = ci; sv.ciendlow = -ci; sv.ciendhigh = ci;
  return true;
}

inline int splitAlignBatch(dgpu_ctx* ctx, std::vector<std::string> const& cons, std::vector<std::string> const& refs, std::vector<uint8_t>& ok,
                           std::vector<TAlign>& aligns);  // defined in splitalign.hpp (include it with this header)

// Batched _consRefAlignment (src/split.h:540-558): align[0] = consensus row, align[1] = reference row.
// Insertions (svt 4) go through splitAlignBatch (three dgpu_edit_path rounds; rows swapped afterwards, :548-552),
// everything else through ONE dgpu_long_needle (or, with windows beyond its shapes, dgpu_long_needle_ex) call. ok[k] = the reference
// function's return value.
inline int consRefAlignmentBatch(dgpu_ctx* ctx, std::vector<int32_t> const& svt, std::vector<const std::string*> const& cons,
                                 std::vector<const std::string*> const& refs, std::vector<uint8_t>& ok, std::vector<TAlign>& aligns) {
  const std::size_t N = svt.size();
  ok.assign(N, 0);
  aligns.assign(N, TAlign());
  int rc;
  {
    std::vector<uint32_t> ins;
    std::vector<std::string> ic, ir;
    for (std::size_t i = 0; i < N; ++i) if (svt[i] == 4) { ins.push_back((uint32_t) i); ic.push_back(*cons[i]); ir.push_back(*refs[i]); }
    if (!ins.empty()) {
      std::vector<uint8_t> iok;
      std::vector<TAlign> ial;
      rc = splitAlignBatch(ctx, ic, ir, iok, ial);
      if (rc) return rc;
      for (std::size_t k = 0; k < ins.size(); ++k) {
        if (!iok[k]) continue;
        TAlign align(2);
        align[0] = ial[k][1]; align[1] = ial[k][0];
        aligns[ins[k]].swap(align);
        ok[ins[k]] = 1;
      }
    }
  }
  std::vector<uint32_t> idx;
  for (std::size_t i = 0; i < N; ++i) if (svt[i] != 4) idx.push_back((uint32_t) i);
  if (idx.empty()) return DGPU_OK;
  std::string arena;
  std::vector<uint32_t> co, cl, ro, rl;
  std::vector<uint64_t> ao;
  uint64_t abytes = 0;
  for (uint32_t i : idx) {
    co.push_back((uint32_t) arena.size()); cl.push_back((uint32_t) cons[i]->size()); arena += *cons[i];
    ro.push_back((uint32_t) arena.size()); rl.push_back((uint32_t) refs[i]->size()); arena += *refs[i];
    ao.push_back(abytes);
    abytes += 2 * (uint64_t) (cons[i]->size() + refs[i]->size());
  }
  std::vector<uint8_t> aln(abytes + 1), okk(idx.size());
  std::vector<uint32_t> alen(idx.size());
  // Windows beyond the wavefront kernels' shapes (|ref| > 16377 or |cons| + |ref| > 32000) need dgpu_long_needle_ex, with max_ref = the
  // batch's widest window. Every other batch goes through dgpu_long_needle, the entry point every binding of the ABI provides, including
  // the CPU suite's stand-in of it (tests/standin/host_standin.cpp forwards dgpu_long_needle to the reference's longNeedle).
  bool wide = false;
  uint32_t widest = 0;
  for (std::size_t k = 0; k < idx.size(); ++k) {
    widest = std::max(widest, rl[k]);
    wide |= rl[k] > 16377 || (uint64_t) cl[k] + rl[k] > 32000;
  }
  const uint64_t refusedBefore = dgpu_unsupported_count(ctx);
  rc = wide ? dgpu_long_needle_ex(ctx, (const uint8_t*) arena.data(), arena.size(), co.data(), cl.data(), ro.data(), rl.data(), idx.size(), aln.data(),
                                  ao.data(), abytes, alen.data(), okk.data(), nullptr, std::max<uint32_t>(1, std::min<uint32_t>(widest, DGPU_LN_MAX_REF)))
            : dgpu_long_needle(ctx, (const uint8_t*) arena.data(), arena.size(), co.data(), cl.data(), ro.data(), rl.data(), idx.size(), aln.data(),
                               ao.data(), abytes, alen.data(), okk.data(), nullptr);
  if (rc) return rc;
  deviceLimitLog().needleJobs += dgpu_unsupported_count(ctx) - refusedBefore;   // jobs beyond the kernel's shapes come back as failed alignments (ok = 0)
  for (std::size_t k = 0; k < idx.size(); ++k) {
    if (!okk[k]) continue;
    const uint64_t half = (uint64_t) cl[k] + rl[k];
    TAlign align(2);
    align[0].assign((const char*) aln.data() + ao[k], alen[k]);
    align[1].assign((const char*) aln.data() + ao[k] + half, alen[k]);
    aligns[idx[k]].swap(align);
    ok[idx[k]] = 1;
  }
  return DGPU_OK;
}

// Batched alignConsensus (src/split.h:646-672 + :560-644). chrseq[tid] = contig sequence (may be NULL for
// contigs no SV of this batch touches), exactly what the reference passes as seq / sndSeq.
// ok[i] = alignConsensus' return value for svs[i]. Insertions (svt 4) go through splitAlignBatch (three
// dgpu_edit_path rounds), everything else through one dgpu_long_needle call.
inline int alignConsensusBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<const char*> const& chrseq,
                               std::vector<StructuralVariantRecord>& svs, bool realign, std::vector<uint8_t>& ok) {
  const std::size_t N = svs.size();
  ok.assign(N, 0);
  std::vector<Breakpoint> bps(N);
  std::vector<std::string> refs(N);
  std::vector<uint32_t> idx;  // SVs that reach the alignment
  for (std::size_t i = 0; i < N; ++i) {
    StructuralVariantRecord& sv = svs[i];
    if ((int32_t) sv.consensus.size() < (2 * c.minimumFlankSize + sv.insLen)) continue;  // src/split.h:648
    Breakpoint bp(sv);
    if (sv.svt == 4) _initBreakpoint(target_len, bp, std::max((int32_t) ((sv.consensus.size() - sv.insLen) / 3), c.minimumFlankSize), sv.svt);
    else _initBreakpoint(target_len, bp, (int32_t) sv.consensus.size(), sv.svt);
    if (bp.chr != bp.chr2) bp.part1 = _getSVRef(c, chrseq[bp.chr2], bp, bp.chr2, sv.svt);
    refs[i] = _getSVRef(c, chrseq[bp.chr], bp, bp.chr, sv.svt);
    bps[i] = bp;
    idx.push_back((uint32_t) i);
  }
  if (idx.empty()) return DGPU_OK;
  int rc;
  if (realign) {
    // orientation check (src/split.h:563-571): two global edit distances, reference window as the query
    std::string arena;
    std::vector<uint32_t> qo, ql, to, tl;
    std::vector<std::string> rcs(idx.size());
    for (std::size_t k = 0; k < idx.size(); ++k) {
      const std::string& cons = svs[idx[k]].consensus;
      rcs[k] = cons;
      reverseComplement(rcs[k]);
      const uint32_t ro = (uint32_t) arena.size(); arena += refs[idx[k]];
      const uint32_t fo = (uint32_t) arena.size(); arena += cons;
      const uint32_t vo = (uint32_t) arena.size(); arena += rcs[k];
      for (int rep = 0; rep < 2; ++rep) {
        qo.push_back(ro); ql.push_back((uint32_t) refs[idx[k]].size());
        to.push_back(rep ? vo : fo); tl.push_back((uint32_t) cons.size());
      }
    }
    std::vector<int32_t> dist(qo.size());
    rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), nullptr,
                            DGPU_MODE_NW, qo.size(), dist.data(), nullptr);
    if (rc) return rc;
    for (std::size_t k = 0; k < idx.size(); ++k)
      if (dist[2 * k + 1] < dist[2 * k]) svs[idx[k]].consensus = rcs[k];
  }
  // _consRefAlignment for every SV that got this far, then the host logic per SV
  std::vector<int32_t> svts;
  std::vector<const std::string*> cp, rp;
  for (uint32_t i : idx) { svts.push_back(svs[i].svt); cp.push_back(&svs[i].consensus); rp.push_back(&refs[i]); }
  std::vector<uint8_t> aok;
  std::vector<TAlign> aligns;
  rc = consRefAlignmentBatch(ctx, svts, cp, rp, aok, aligns);
  if (rc) return rc;
  for (std::size_t k = 0; k < idx.size(); ++k) {
    if (!aok[k]) continue;
    const uint32_t i = idx[k];
    ok[i] = _finishAlignConsensus(c, svs[i].consensus, refs[i], aligns[k], svs[i], bps[i]) ? 1 : 0;
  }
  return DGPU_OK;
}

}  // namespace dellyb200
