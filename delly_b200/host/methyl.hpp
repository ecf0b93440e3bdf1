// methyl.hpp — CpG methylation around SV breakpoints from the MM / ML tags of long reads (SURVEY §8f row 4), the host
// mirror of
//   src/methyl.h:35-81    MethylInfo, MethylAccum
//   src/methyl.h:118-216  buildMethylCalls        (MM / ML tags -> one call per read base: 1 = 5mC, 0 = C, -1 = no call)
//   src/methyl.h:219-259  collectMethylFromWindows (calls of the aligned bases inside reference windows)
//   src/methyl.h:262-414  collectMethylFromInsertionEdlib (calls of the inserted bases, placed on the consensus through an
//                         edlibAlign HW + PATH of the read's inserted segment against the consensus insertion)
//   src/methyl.h:417-440  clusterAndFilterCpG, :443-470 finalizeMethylInfo, :473-568 accumulateMethyl
// as genotypeLR uses them (src/genotype.h:306-324, :383-388): every read that supports REF or ALT of an SV adds its calls
// to that SV's windows.
//
// The reference aligns one insertion-carrying read at a time inside the genotyping loop. Here accumulateMethyl does the
// window part at once (byte loops over the CIGAR: host) and QUEUES the insertion part as an InsertionJob; after the read
// scan all queued jobs go to the device in ONE dgpu_edit_path call (HW), and their CpG calls are added afterwards. All
// accumulators are sums and per-position counters, so the order of the additions is immaterial.
#pragma once
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/dgpu.h"
#include "split.hpp"
#include "types.hpp"

namespace dellyb200 {

struct MethylConfig {  // src/tegua.h:44,60,248-249 (+ minCpgDepth of the genotyping options)
  uint16_t methylProb = 128;
  int32_t methylWindow = 1000;
  uint32_t minCpgDepth = 1;
};

struct MethylInfo {  // src/methyl.h:35-55; -1 = no call. Index 0..3 = SV start left / right, SV end left / right
  int32_t alt[4] = {-1, -1, -1, -1};   // ALT methylation percent
  int32_t ref[4] = {-1, -1, -1, -1};   // REF methylation percent
  int32_t mnc[4] = {-1, -1, -1, -1};   // CpG sites seen (REF and ALT reads together)
  int32_t mdp[4] = {-1, -1, -1, -1};   // mean read depth per CpG site
};

struct MethylAccum {  // src/methyl.h:58-81
  uint32_t altM[4] = {0, 0, 0, 0}, altT[4] = {0, 0, 0, 0}, refM[4] = {0, 0, 0, 0}, refT[4] = {0, 0, 0, 0};
  std::unordered_map<int32_t, uint32_t> cpg[4];
};

// The part of one alignment record the methylation code reads (the genotyping record plus its two tags).
struct MethylRead {
  int32_t pos = 0;
  bool reverse = false;
  std::vector<std::pair<uint8_t, uint32_t> > const* cigar = nullptr;
  std::string const* seq = nullptr;   // read bases as stored in the record
  bool hasMM = false, hasML = false;  // MM present with type Z; ML present as a B:C array
  std::string const* mm = nullptr;
  std::vector<uint8_t> const* ml = nullptr;
};

namespace detail {
inline char complementBase(char b) {  // src/methyl.h:94-103
  switch (std::toupper((unsigned char) b)) {
    case 'A': return 'T';
    case 'C': return 'G';
    case 'G': return 'C';
    case 'T': return 'A';
    default: return b;
  }
}
// boost::split(out, s, is_any_of(sep)) without token compression: n separators give n + 1 tokens
inline std::vector<std::string> splitAny(std::string const& s, char sep) {
  std::vector<std::string> out(1);
  for (char ch : s) {
    if (ch == sep) out.emplace_back();
    else out.back().push_back(ch);
  }
  return out;
}
}  // namespace detail

// src/methyl.h:118-216. methCall is indexed in the ORIGINAL read orientation (fwdseq).
inline bool buildMethylCalls(MethylRead const& r, uint8_t probModTh, std::vector<int8_t>& methCall) {
  const int32_t l = (int32_t) r.seq->size();
  methCall.assign((std::size_t) l, (int8_t) -1);
  if (!r.hasMM) return false;
  std::string fwdseq = *r.seq;
  if (r.reverse) reverseComplement(fwdseq);
  std::unordered_map<char, std::vector<int32_t> > basepos;
  for (int32_t i = 0; i < l; ++i) basepos[(char) std::toupper((unsigned char) fwdseq[i])].push_back(i);

  struct ModHit { int32_t pos; char code; uint8_t prob; bool rev; char base; };
  std::vector<ModHit> hits;
  bool skipStatus5mC = false;  // "C+m?" / "C+m.": unlisted cytosines carry no call
  for (std::string const& tok : detail::splitAny(*r.mm, ';')) {
    if (tok.size() < 2) continue;
    const char base = tok[0];
    const bool revMod = (tok[1] == '-');
    std::size_t idx = 2;
    std::string codes;
    bool hasSkip = false;
    while (idx < tok.size() && tok[idx] != ',') {
      const char ch = tok[idx++];
      if (ch == '?' || ch == '.') hasSkip = true;
      else if (std::isalpha((unsigned char) ch)) codes.push_back(ch);
    }
    if (hasSkip)
      for (char cd : codes)
        if (cd == 'm' || cd == 'M') skipStatus5mC = true;
    if (idx < tok.size() && tok[idx] == ',') {
      const std::string rest = tok.substr(idx + 1);
      if (!rest.empty()) {
        int32_t current = -1;
        for (std::string const& pt : detail::splitAny(rest, ',')) {
          if (pt.empty()) continue;
          current += std::stoi(pt) + 1;
          for (char cd : codes) hits.push_back(ModHit{current, cd, (uint8_t) 255, revMod, base});
        }
      }
    }
  }
  if (!skipStatus5mC)
    for (int32_t i = 0; i < l; ++i)
      if (std::toupper((unsigned char) fwdseq[i]) == 'C') methCall[i] = 0;
  if (r.hasML) {  // probabilities in hit order
    const std::size_t n = std::min(r.ml->size(), hits.size());
    for (std::size_t i = 0; i < n; ++i) hits[i].prob = (*r.ml)[i];
  }
  for (ModHit const& h : hits) {
    if (h.code != 'm' && h.code != 'M') continue;
    const char ub = (char) std::toupper((unsigned char) h.base);
    const char target = h.rev ? detail::complementBase(ub) : ub;
    auto it = basepos.find(target);
    if (it == basepos.end()) continue;
    if (h.pos < 0 || (std::size_t) h.pos >= it->second.size()) continue;
    methCall[it->second[h.pos]] = (h.prob >= probModTh) ? 1 : 0;
  }
  return true;
}

// src/methyl.h:219-259
inline void collectMethylFromWindows(MethylRead const& r, std::vector<int8_t> const& methCall, std::vector<std::pair<int32_t, int32_t> > const& wins,
                                     std::vector<uint32_t>& meth, std::vector<uint32_t>& tot, std::vector<std::unordered_map<int32_t, uint32_t> >& cpgPos) {
  meth.assign(wins.size(), 0);
  tot.assign(wins.size(), 0);
  cpgPos.assign(wins.size(), std::unordered_map<int32_t, uint32_t>());
  if (wins.empty() || methCall.empty()) return;
  const int32_t l = (int32_t) r.seq->size();
  int32_t maxEnd = 0;
  for (auto const& w : wins) maxEnd = std::max(maxEnd, w.second);
  int32_t rp = r.pos, sp = 0;
  for (auto const& cg : *r.cigar) {
    const int32_t len = (int32_t) cg.second;
    if (cg.first == 0 || cg.first == 7 || cg.first == 8) {
      for (int32_t k = 0; k < len; ++k, ++rp, ++sp) {
        if (rp >= maxEnd) return;
        const int32_t fwdPos = r.reverse ? (l - sp - 1) : sp;
        if (fwdPos < 0 || fwdPos >= l) continue;
        const int8_t call = methCall[fwdPos];
        if (call < 0) continue;
        for (std::size_t wi = 0; wi < wins.size(); ++wi) {
          if (rp >= wins[wi].first && rp < wins[wi].second) {
            ++tot[wi];
            if (call == 1) ++meth[wi];
            ++cpgPos[wi][rp];
          }
        }
      }
    } else if (cg.first == 2 || cg.first == 3) {
      rp += len;
      if (rp >= maxEnd) return;
    } else if (cg.first == 1 || cg.first == 4) {
      sp += len;
    }
  }
}

// One queued insertion alignment (src/methyl.h:262-321): the read's inserted segment against the consensus insertion.
struct InsertionJob {
  uint32_t svid = 0;
  bool reverse = false;
  int32_t insReadStart = 0, readLen = 0, insLen = 0;
  std::string readIns, consIns;
  std::vector<int8_t> methCall;  // this read's calls (original orientation)
};

// The locate-the-insertion half of collectMethylFromInsertionEdlib (:262-321): returns false when the read shows no
// insertion (or clipped segment) to place.
inline bool locateInsertion(MethylConfig const& mc, MethylRead const& r, std::vector<int8_t> const& methCall, StructuralVariantRecord const& sv,
                            InsertionJob& job) {
  const int32_t l = (int32_t) r.seq->size();
  const int32_t insLen = sv.insLen;
  if (l == 0 || insLen <= 0) return false;
  if (sv.consBp < 0 || (sv.consBp + insLen) > (int32_t) sv.consensus.size()) return false;
  int32_t insReadStart = -1, insReadLen = 0;
  int32_t minOpLen = std::min(insLen / 2, mc.methylWindow / 2);
  if (minOpLen < 1) minOpLen = 1;
  const bool mapsBeforeBp = (r.pos < sv.svStart);
  int32_t rp = r.pos, sp = 0;
  const int32_t nCigar = (int32_t) r.cigar->size();
  for (int32_t ci = 0; ci < nCigar; ++ci) {
    const uint8_t op = (*r.cigar)[ci].first;
    const int32_t len = (int32_t) (*r.cigar)[ci].second;
    if (op == 0 || op == 7 || op == 8) { rp += len; sp += len; }
    else if (op == 2 || op == 3) rp += len;
    else if (op == 1) {
      if (rp == sv.svStart && len >= minOpLen) { insReadStart = sp; insReadLen = len; break; }
      sp += len;
    } else if (op == 4) {
      if (len >= minOpLen) {
        const bool wantFirst = !mapsBeforeBp;
        if ((wantFirst && ci == 0) || (!wantFirst && ci == nCigar - 1)) {
          if (len > insReadLen) { insReadStart = sp; insReadLen = len; }
        }
      }
      sp += len;
    }
  }
  if (insReadStart < 0) return false;
  insReadLen = std::min(insReadLen, l - insReadStart);
  if (insReadLen <= 0) return false;
  job.svid = (uint32_t) sv.id;
  job.reverse = r.reverse;
  job.insReadStart = insReadStart;
  job.readLen = l;
  job.insLen = insLen;
  job.readIns = r.seq->substr((std::size_t) insReadStart, (std::size_t) insReadLen);
  job.consIns = sv.consensus.substr((std::size_t) sv.consBp, (std::size_t) insLen);
  job.methCall = methCall;
  return true;
}

// src/methyl.h:473-568: the calls of one REF- or ALT-supporting read for one SV. `candidates` are the breakpoint
// positions of the SV this read spans on chromosome refIndex.
inline void accumulateMethyl(MethylConfig const& mc, MethylRead const& r, std::vector<int8_t> const& methCall, StructuralVariantRecord const& sv, int32_t refIndex,
                             int32_t chromLen, bool isAlt, std::vector<int32_t> const& candidates, MethylAccum& acc, std::vector<InsertionJob>& queue) {
  if (methCall.empty()) return;
  const bool isTrans = _translocation(sv.svt), isIns = (sv.svt == 4), isDel = (sv.svt == 2);
  bool onStart = false, onEnd = false;
  for (int32_t cand : candidates) {
    if (cand == sv.svStart && sv.chr == refIndex) onStart = true;
    if (cand == sv.svEnd && sv.chr2 == refIndex) onEnd = true;
  }
  if (!onStart && !onEnd) return;
  const int32_t W = mc.methylWindow;
  std::vector<std::pair<int32_t, int32_t> > wins;
  std::vector<int32_t> field;
  auto add = [&](int32_t b, int32_t e, int32_t f) { if (e > b) { wins.emplace_back(b, e); field.push_back(f); } };
  const bool inner = !isIns && !(isAlt && isDel);  // the windows inside the SV exist for this allele
  if (onStart) {
    add(std::max(0, sv.svStart - W), sv.svStart, 0);
    if (inner) add(sv.svStart, !isTrans ? std::min(sv.svStart + W, sv.svEnd) : std::min(sv.svStart + W, chromLen), 1);
  }
  if (onEnd) {
    if (inner) add(!isTrans ? std::max(sv.svStart, sv.svEnd - W) : std::max(0, sv.svEnd - W), sv.svEnd, 2);
    add(sv.svEnd, std::min(sv.svEnd + W, chromLen), 3);
  }
  if (!wins.empty()) {
    std::vector<uint32_t> meth, tot;
    std::vector<std::unordered_map<int32_t, uint32_t> > cpgPos;
    collectMethylFromWindows(r, methCall, wins, meth, tot, cpgPos);
    for (std::size_t i = 0; i < field.size(); ++i) {
      const int32_t f = field[i];
      if (isAlt) { acc.altM[f] += meth[i]; acc.altT[f] += tot[i]; }
      else { acc.refM[f] += meth[i]; acc.refT[f] += tot[i]; }
      for (auto const& kv : cpgPos[i]) acc.cpg[f][kv.first] += kv.second;
    }
  }
  if (isIns && isAlt && sv.insLen > 0 && !r.seq->empty() && !sv.consensus.empty()) {
    InsertionJob job;
    if (locateInsertion(mc, r, methCall, sv, job)) queue.push_back(std::move(job));
  }
}

// The second half of collectMethylFromInsertionEdlib (:323-413) for all queued jobs: ONE dgpu_edit_path call (HW), then
// consensus -> read coordinates from the path and the tolerant CpG lookup (+-8 read bases). Adds to acc[svid].
inline int flushInsertionJobs(dgpu_ctx* ctx, MethylConfig const& mc, std::vector<InsertionJob> const& queue, std::vector<MethylAccum>& acc) {
  if (queue.empty()) return DGPU_OK;
  if (!ctx) return DGPU_ERR_NODEVICE;
  const std::size_t J = queue.size();
  std::string arena;
  std::vector<uint32_t> qo(J), ql(J), to(J), tl(J), opsLen(J), status(J);
  std::vector<uint64_t> opsOff(J);
  uint64_t opsBytes = 0;
  for (std::size_t j = 0; j < J; ++j) {
    qo[j] = (uint32_t) arena.size(); ql[j] = (uint32_t) queue[j].readIns.size(); arena += queue[j].readIns;
    to[j] = (uint32_t) arena.size(); tl[j] = (uint32_t) queue[j].consIns.size(); arena += queue[j].consIns;
    opsOff[j] = opsBytes;
    opsBytes += (uint64_t) ql[j] + tl[j];
  }
  std::vector<int32_t> dist(J), startLoc(J), endLoc(J);
  std::vector<uint8_t> ops(opsBytes + 1);
  int rc = editPathCall(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), DGPU_MODE_HW, nullptr, 0, J,
                        dist.data(), startLoc.data(), endLoc.data(), ops.data(), opsOff.data(), opsBytes, opsLen.data(), status.data());
  if (rc) return rc;
  for (std::size_t j = 0; j < J; ++j)
    if (status[j] != 0) ++deviceLimitLog().pathJobs;   // e.g. a consensus insertion above DGPU_EP_MAX_SLICE columns: no calls from this read
  static const int32_t CPGTOL = 8;
  for (std::size_t j = 0; j < J; ++j) {
    InsertionJob const& jb = queue[j];
    if ((dist[j] < 0) || (status[j] != 0)) continue;
    const int32_t insLen = jb.insLen, nRead = (int32_t) jb.readIns.size(), l = jb.readLen;
    std::vector<int32_t> consToRead((std::size_t) insLen, -1);
    {
      int32_t qi = 0, ti = startLoc[j];
      const uint8_t* a = ops.data() + opsOff[j];
      for (int32_t ai = 0; ai < (int32_t) opsLen[j] && qi < nRead && ti < insLen; ++ai) {
        if (a[ai] == 0 || a[ai] == 3) { consToRead[ti] = qi; ++qi; ++ti; }  // match / mismatch
        else if (a[ai] == 1) { consToRead[ti] = -1; ++ti; }                 // EDLIB_EDOP_INSERT: target base without a read base
        else ++qi;
      }
    }
    MethylAccum& A = acc[jb.svid];
    const int32_t wlen = std::min(mc.methylWindow, insLen);
    auto up = [](char ch) { return (char) std::toupper((unsigned char) ch); };
    for (int32_t window = 0; window < 2; ++window) {
      const int32_t winStart = window ? (insLen - wlen) : 0, winEnd = window ? insLen : wlen;
      const int32_t f = window ? 2 : 1;  // start-right / end-left
      for (int32_t k = winStart; k < winEnd - 1; ++k) {
        if (up(jb.consIns[k]) != 'C' || up(jb.consIns[k + 1]) != 'G') continue;
        int8_t call = -1;
        const int32_t centre = jb.reverse ? consToRead[k + 1] : consToRead[k];  // reverse reads carry the call on the G's partner
        if (centre < 0) continue;
        for (int32_t delta = 0; delta <= CPGTOL && call < 0; ++delta) {
          for (int32_t sign : {0, -1, 1}) {
            if ((delta == 0) != (sign == 0)) continue;
            const int32_t p = centre + delta * sign;
            int32_t idx;
            if (!jb.reverse) {
              if (p < 0 || p + 1 >= nRead) continue;
              if (up(jb.readIns[p]) != 'C' || up(jb.readIns[p + 1]) != 'G') continue;
              idx = jb.insReadStart + p;
            } else {
              if (p < 1 || p >= nRead) continue;
              if (up(jb.readIns[p - 1]) != 'C' || up(jb.readIns[p]) != 'G') continue;
              idx = l - 1 - (jb.insReadStart + p);
            }
            if (idx < 0 || idx >= l) continue;
            if (jb.methCall[idx] < 0) continue;
            call = jb.methCall[idx];
            break;
          }
        }
        if (call < 0) continue;
        ++A.cpg[f][k];
        ++A.altT[f];
        if (call == 1) ++A.altM[f];
      }
    }
  }
  return DGPU_OK;
}

// src/methyl.h:417-440: CpG sites = runs of positions (p, p + 1) — the two strands of one site — with enough depth
inline int32_t clusterAndFilterCpG(std::unordered_map<int32_t, uint32_t> const& cpgMap, uint32_t minDepth) {
  if (cpgMap.empty()) return 0;
  std::vector<std::pair<int32_t, uint32_t> > sites(cpgMap.begin(), cpgMap.end());
  std::sort(sites.begin(), sites.end());
  int32_t count = 0, clusterStart = sites[0].first;
  uint32_t depth = sites[0].second;
  for (std::size_t i = 1; i < sites.size(); ++i) {
    if (sites[i].first <= clusterStart + 1) depth += sites[i].second;
    else {
      if (depth >= minDepth) ++count;
      clusterStart = sites[i].first;
      depth = sites[i].second;
    }
  }
  if (depth >= minDepth) ++count;
  return count;
}

// src/methyl.h:443-470
inline void finalizeMethylInfo(MethylAccum const& a, MethylInfo& mi, uint32_t minCpgDepth) {
  for (int f = 0; f < 4; ++f) {
    mi.alt[f] = (a.altT[f] > 0) ? (int32_t) std::round(100.0f * (float) a.altM[f] / (float) a.altT[f]) : -1;
    mi.ref[f] = (a.refT[f] > 0) ? (int32_t) std::round(100.0f * (float) a.refM[f] / (float) a.refT[f]) : -1;
    mi.mnc[f] = clusterAndFilterCpG(a.cpg[f], minCpgDepth);
    mi.mdp[f] = (mi.mnc[f] <= 0) ? -1 : (int32_t) std::round((float) (a.altT[f] + a.refT[f]) / (float) mi.mnc[f]);
  }
}

// The MA / MR / MNC / MDV FORMAT values of one sample (src/modvcf.h:622-665); INT32_MIN = missing
inline void methylFormat(MethylInfo const& mi, int32_t svt, uint32_t minCpgDepth, int32_t* ma, int32_t* mr, int32_t* mnc, int32_t* mdv) {
  const int32_t missing = INT32_MIN;
  const bool isIns = (svt == 4), isDel = (svt == 2);
  for (int f = 0; f < 4; ++f) {
    auto gate = [&](int32_t pct) { return (pct < 0 || mi.mdp[f] < 0 || (uint32_t) mi.mdp[f] < minCpgDepth) ? missing : pct; };
    mnc[f] = (mi.mnc[f] < 0) ? missing : mi.mnc[f];
    mdv[f] = (mi.mdp[f] < 0) ? missing : mi.mdp[f];
    const bool innerField = (f == 1 || f == 2);
    ma[f] = (innerField && isDel) ? missing : gate(mi.alt[f]);
    mr[f] = (innerField && isIns) ? missing : gate(mi.ref[f]);
  }
}

}  // namespace dellyb200
