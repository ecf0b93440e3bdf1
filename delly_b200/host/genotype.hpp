// genotype.hpp — short-read genotyping realignment, the batch seam of the reference
// (AlignJob / AlignResult / process_batch, src/coverage.h:87-115, :412-454), with the two
// _editDistanceHW calls per job replaced by ONE dgpu_edit_distance call for the whole batch.
// Also _editDistanceNW for the long-read path (src/genotype.h:22-29).
#pragma once
#include <cmath>
#include <map>
#include <set>
#include <string>
#include <tuple>
#include <atomic>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/dgpu.h"
#include "methyl.hpp"
#include "shard.hpp"
#include "split.hpp"
#include "types.hpp"

namespace dellyb200 {

struct AlignJob {  // src/coverage.h:87-96
  std::string consProbe, refProbe, sequence;
  uint32_t fileIndex, svId;
  uint8_t qual;
};

struct AlignResult {  // src/coverage.h:98-105
  uint32_t fileIndex = 0, svId = 0;
  char type = 'N';  // 'R' ref, 'A' alt, 'N' none
  uint8_t qual = 0;
};

// k exactly as edlibNewAlignConfig receives it at src/coverage.h:111: int(2 * 0.95f * |q|) evaluated in float
inline int32_t _hwBound(Config const& c, std::size_t qsize) { return (int32_t) (2 * c.flankQuality * qsize); }

// score of _editDistanceHW (src/coverage.h:109-113) from the device's edit distance
inline double _hwScore(Config const& c, std::size_t qsize, int32_t editDistance) {
  if (editDistance == -1) return 0;
  return ((1.0 - c.flankQuality) * (double) qsize) / (double) (editDistance + 1);
}

// process_batch (src/coverage.h:412-441): results[i] for jobs[i]; the merge into countMap (:442-453) stays with the caller.
inline int processBatch(dgpu_ctx* ctx, Config const& c, std::vector<AlignJob> const& jobs, std::vector<AlignResult>& results) {
  const std::size_t J = jobs.size();
  results.assign(J, AlignResult());
  if (!J) return DGPU_OK;
  std::string arena;
  std::vector<uint32_t> qo(2 * J), ql(2 * J), to(2 * J), tl(2 * J);
  std::vector<int32_t> k(2 * J), dist(2 * J);
  for (std::size_t i = 0; i < J; ++i) {
    const AlignJob& j = jobs[i];
    const uint32_t so = (uint32_t) arena.size(); arena += j.sequence;
    qo[2 * i] = (uint32_t) arena.size(); ql[2 * i] = (uint32_t) j.consProbe.size(); arena += j.consProbe;
    qo[2 * i + 1] = (uint32_t) arena.size(); ql[2 * i + 1] = (uint32_t) j.refProbe.size(); arena += j.refProbe;
    to[2 * i] = to[2 * i + 1] = so; tl[2 * i] = tl[2 * i + 1] = (uint32_t) j.sequence.size();
    k[2 * i] = _hwBound(c, j.consProbe.size()); k[2 * i + 1] = _hwBound(c, j.refProbe.size());
  }
  int rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), k.data(),
                              DGPU_MODE_HW, 2 * J, dist.data(), nullptr);
  if (rc) return rc;
  for (std::size_t i = 0; i < J; ++i) {
    const double scoreAlt = _hwScore(c, jobs[i].consProbe.size(), dist[2 * i]);
    const double scoreRef = _hwScore(c, jobs[i].refProbe.size(), dist[2 * i + 1]);
    if ((scoreRef > 0.7) || (scoreAlt > 0.7)) {
      results[i].svId = jobs[i].svId;
      results[i].fileIndex = jobs[i].fileIndex;
      const bool isRef = scoreRef > scoreAlt;
      results[i].type = isRef ? 'R' : 'A';
      results[i].qual = (uint8_t) std::min(255, std::min((int) ((isRef ? scoreRef : scoreAlt) * 35), (int) jobs[i].qual));
    }
  }
  return DGPU_OK;
}

// Batched _editDistanceNW (src/genotype.h:22-29): global edit distance of (query, target) pairs.
inline int editDistanceNWBatch(dgpu_ctx* ctx, std::vector<std::pair<std::string, std::string> > const& pairs, std::vector<int32_t>& dist) {
  dist.assign(pairs.size(), 0);
  if (pairs.empty()) return DGPU_OK;
  std::string arena;
  std::vector<uint32_t> qo, ql, to, tl;
  for (auto const& p : pairs) {
    qo.push_back((uint32_t) arena.size()); ql.push_back((uint32_t) p.first.size()); arena += p.first;
    to.push_back((uint32_t) arena.size()); tl.push_back((uint32_t) p.second.size()); arena += p.second;
  }
  return dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), nullptr, DGPU_MODE_NW,
                            pairs.size(), dist.data(), nullptr);
}

// ---- REF / ALT probes of the genotyping pass (src/coverage.h:117-263) ------------------------------------------

struct BpRegion {  // src/coverage.h:49-67; sorted by bppos only (std::sort, unstable for ties like the reference)
  int32_t regionStart = 0, regionEnd = 0, bppos = 0, homLeft = 0, homRight = 0, svt = 0;
  uint32_t id = 0;
  uint8_t bpPoint = 0;
  BpRegion() {}
  BpRegion(int32_t rs, int32_t re, int32_t bpos, int32_t hl, int32_t hr, int32_t s, uint32_t identifier, uint8_t bpp)
      : regionStart(rs), regionEnd(re), bppos(bpos), homLeft(hl), homRight(hr), svt(s), id(identifier), bpPoint(bpp) {}
  bool operator<(BpRegion const& o) const { return bppos < o.bppos; }
};

// src/coverage.h:117-160: which end of the reference gap a breakpoint's REF probe is centred on
inline bool _cutAtREnd(unsigned int bpPoint, int32_t svt) {
  const bool flipped = _translocation(svt) ? (_getSpanOrientation(svt) == 3) : (svt == 3);
  return flipped ? !bpPoint : (bpPoint != 0);
}
inline int32_t _cutRefStart(int32_t rStart, int32_t rEnd, int32_t offset, unsigned int bpPoint, int32_t svt) {
  return (_cutAtREnd(bpPoint, svt) ? rEnd : rStart) - offset;
}
inline int32_t _cutRefEnd(int32_t rStart, int32_t rEnd, int32_t offset, unsigned int bpPoint, int32_t svt) {
  return (_cutAtREnd(bpPoint, svt) ? rEnd : rStart) + offset;
}

inline std::string _addID(int32_t svt) {  // src/util.h:237-246
  if (svt == 0 || svt == 1) return "INV";
  if (svt == 2) return "DEL";
  if (svt == 3) return "DUP";
  if (svt == 4) return "INS";
  if (svt == 9) return "CNV";
  return "BND";
}

// symbolic / breakend ALT allele (src/util.h:253-272)
inline std::string _addAlleles(std::string const& ref, std::string const& chr2, StructuralVariantRecord const& sv, int32_t svt) {
  if (_translocation(svt)) {
    const uint8_t ct = _getSpanOrientation(svt);
    const std::string pos = std::to_string(sv.svEnd);
    if (ct == 0) return ref + "," + ref + "]" + chr2 + ":" + pos + "]";
    if (ct == 1) return ref + "," + "[" + chr2 + ":" + pos + "[" + ref;
    if (ct == 2) return ref + "," + ref + "[" + chr2 + ":" + pos + "[";
    if (ct == 3) return ref + "," + "]" + chr2 + ":" + pos + "]" + ref;
  }
  return ref + ",<" + _addID(svt) + ">";
}

// std::string::substr with the reference's argument conversion (int32 -> size_t): pos > size throws there
// (std::out_of_range aborts delly); here it is reported so a batch never dies half-way.
inline bool _substrChecked(std::string const& s, int32_t start, int32_t len, std::string& out) {
  const std::size_t pos = (std::size_t) start;   // negative start wraps like the implicit conversion does
  if (pos > s.size()) return false;
  out = s.substr(pos, (std::size_t) len);
  return true;
}

// _generateProbes (src/coverage.h:164-263) for a whole SV list: the per-precise-SV _consRefAlignment + _findSplit is ONE
// consRefAlignmentBatch call (one dgpu_long_needle + the splitAlign rounds) instead of |svs| sequential DPs.
//   svs            in/out: alleles filled when empty (:185-187)
//   refProbeArr / consProbeArr   [2][svs.size()], indexed by sv.id like the reference
//   bpRegion       [n_targets], each sorted by bppos; svOnChr[n_targets]
//   bad            ids whose probe cut fell outside the string (the reference would have thrown)
//   want           (may be null) the SVs whose probes are needed, by index; the others get their alleles only. A rank of a contig-sharded run
//                  wants the SVs with a breakpoint on its contigs: the breakpoint regions of those contigs are then the single-process ones.
inline int generateProbesBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                               std::vector<const char*> const& chrseq, std::vector<StructuralVariantRecord>& svs,
                               std::vector<std::vector<std::string> >& refProbeArr, std::vector<std::vector<std::string> >& consProbeArr,
                               std::vector<std::vector<BpRegion> >& bpRegion, std::vector<bool>& svOnChr, std::vector<uint32_t>& bad,
                               std::vector<uint8_t> const* want = nullptr) {
  const std::size_t N = svs.size();
  refProbeArr.assign(2, std::vector<std::string>(N));
  consProbeArr.assign(2, std::vector<std::string>(N));
  bpRegion.assign(target_len.size(), std::vector<BpRegion>());
  svOnChr.assign(target_len.size(), false);
  bad.clear();
  std::vector<uint32_t> idx;
  std::vector<std::string> refs;
  for (std::size_t i = 0; i < N; ++i) {
    StructuralVariantRecord& sv = svs[i];
    svOnChr[sv.chr] = true;
    svOnChr[sv.chr2] = true;
    if (sv.alleles.empty()) sv.alleles = _addAlleles(detail::upperSlice(chrseq[sv.chr], sv.svStart - 1, sv.svStart), target_name[sv.chr2], sv, sv.svt);
    if (!sv.precise || (want && !(*want)[i])) continue;
    Breakpoint bp(sv);
    if (sv.svt == 4) _initBreakpoint(target_len, bp, std::max((int32_t) ((sv.consensus.size() - sv.insLen) / 3), c.minimumFlankSize), sv.svt);
    else _initBreakpoint(target_len, bp, (int32_t) sv.consensus.size(), sv.svt);
    // translocations: the chr2 part is cut first, with the breakpoint initialised from the full consensus length (:193-197)
    // (the reference visits contigs in index order and fills the chr2 part while on contig chr2, so it exists only if chr2 < chr)
    if (sv.chr != sv.chr2 && sv.chr2 < sv.chr) {
      Breakpoint bp2(sv);
      _initBreakpoint(target_len, bp2, (int32_t) sv.consensus.size(), sv.svt);
      bp.part1 = _getSVRef(c, chrseq[sv.chr2], bp2, sv.chr2, sv.svt);
    }
    refs.push_back(_getSVRef(c, chrseq[sv.chr], bp, sv.chr, sv.svt));
    idx.push_back((uint32_t) i);
  }
  if (!idx.empty()) {
    std::vector<int32_t> svts;
    std::vector<const std::string*> cp, rp;
    for (std::size_t k = 0; k < idx.size(); ++k) { svts.push_back(svs[idx[k]].svt); cp.push_back(&svs[idx[k]].consensus); rp.push_back(&refs[k]); }
    std::vector<uint8_t> aok;
    std::vector<TAlign> aligns;
    int rc = consRefAlignmentBatch(ctx, svts, cp, rp, aok, aligns);
    if (rc) return rc;
    // The reference walks contigs in index order and, per contig, the SVs whose chr is that contig (:176-254): breakpoint
    // regions are appended in that order before the (unstable) sort by bppos, so the same order is kept here.
    std::vector<uint32_t> order(idx.size());
    for (std::size_t k = 0; k < idx.size(); ++k) order[k] = (uint32_t) k;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return svs[idx[a]].chr < svs[idx[b]].chr; });
    for (uint32_t k : order) {
      if (!aok[k]) continue;
      StructuralVariantRecord const& sv = svs[idx[k]];
      std::string const& svRefStr = refs[k];
      AlignDescriptor ad;
      if (!_findSplit(c, sv.consensus, svRefStr, aligns[k], ad, sv.svt)) continue;
      for (unsigned int bpPoint = 0; bpPoint < 2; ++bpPoint) {
        int32_t regionChr, regionStart, regionEnd, cutConsStart, cutConsEnd, bppos;
        if (bpPoint) {
          regionChr = sv.chr2;
          regionStart = std::max(0, sv.svEnd - c.minimumFlankSize);
          regionEnd = (int32_t) std::min((uint32_t) (sv.svEnd + c.minimumFlankSize), target_len[sv.chr2]);
          cutConsStart = ad.cEnd - ad.homLeft - c.minimumFlankSize;
          cutConsEnd = ad.cEnd + ad.homRight + c.minimumFlankSize;
          bppos = sv.svEnd;
        } else {
          regionChr = sv.chr;
          regionStart = std::max(0, sv.svStart - c.minimumFlankSize);
          regionEnd = (int32_t) std::min((uint32_t) (sv.svStart + c.minimumFlankSize), target_len[sv.chr]);
          cutConsStart = ad.cStart - ad.homLeft - c.minimumFlankSize;
          cutConsEnd = ad.cStart + ad.homRight + c.minimumFlankSize;
          bppos = sv.svStart;
        }
        const int32_t cutRefStart = _cutRefStart(ad.rStart, ad.rEnd, ad.homLeft + c.minimumFlankSize, bpPoint, sv.svt);
        const int32_t cutRefEnd = _cutRefEnd(ad.rStart, ad.rEnd, ad.homRight + c.minimumFlankSize, bpPoint, sv.svt);
        if (!_substrChecked(sv.consensus, cutConsStart, cutConsEnd - cutConsStart, consProbeArr[bpPoint][sv.id]) ||
            !_substrChecked(svRefStr, cutRefStart, cutRefEnd - cutRefStart, refProbeArr[bpPoint][sv.id])) {
          bad.push_back(sv.id);
          break;
        }
        bpRegion[regionChr].push_back(BpRegion(regionStart, regionEnd, bppos, ad.homLeft, ad.homRight, sv.svt, sv.id, (uint8_t) bpPoint));
      }
    }
  }
  for (auto& r : bpRegion) std::sort(r.begin(), r.end());
  return DGPU_OK;
}


// ---- long-read genotyping pass (genotypeLR, src/genotype.h:93-397) ---------------------------------------------------

constexpr uint32_t BAMF_REVERSE = 0x10, BAMF_SECONDARY = 0x100, BAMF_QCFAIL = 0x200, BAMF_DUP = 0x400, BAMF_UNMAP = 0x4, BAMF_SUPPLEMENTARY = 0x800;

struct LrRecord {  // what genotypeLR reads from one bam1_t
  int32_t tid = 0, pos = 0;
  uint32_t flag = 0;
  uint8_t mapq = 0;
  std::vector<std::pair<uint8_t, uint32_t> > cigar;  // (BAM op code, length)
  std::string seq;                                    // read bases as decoded by bam_seqi ("=ACMGRSVTWYHKDBN")
  uint8_t hp = 0;                                     // HP tag (0 = none)
  int32_t ps = -1;                                    // PS tag (-1 = none)
  bool hasMM = false, hasML = false;                  // MM tag present with type Z; ML tag present as a B:C array
  std::string mm;                                     // MM: base-modification positions (SAM tags spec)
  std::vector<uint8_t> ml;                            // ML: modification probabilities
};

struct JunctionCount {  // src/coverage.h:74-85
  std::vector<uint8_t> ref, alt, hp1ref, hp1alt, hp2ref, hp2alt;
  int32_t ps = -1;
};

struct ReadCount {  // src/util.h:69-76
  int32_t leftRC = 0, rc = 0, rightRC = 0;
};

// One ALT-supporting read of an SV, for the SV-read dump (host/svreaddump.hpp)
struct SvReadEvent {
  uint32_t rec;    // index into the genotyped record list
  uint32_t svid;
  int32_t svt;     // the type the reference names the id after (_addID)
};

// src/genotype.h:30-41
inline int32_t _readStart(LrRecord const& r) {
  uint32_t rp = (uint32_t) r.pos;
  if (!r.cigar.empty() && (r.cigar[0].first == 4 || r.cigar[0].first == 5)) {
    if (rp > r.cigar[0].second) rp -= r.cigar[0].second;
    else rp = 0;
  }
  return (int32_t) rp;
}
// src/genotype.h:43-56
inline int32_t _readEnd(LrRecord const& r) {
  uint32_t rp = (uint32_t) r.pos;
  if (!r.cigar.empty()) {
    for (auto const& c : r.cigar)
      if (c.first == 0 || c.first == 7 || c.first == 8 || c.first == 2 || c.first == 3) rp += c.second;
    if (r.cigar.back().first == 4 || r.cigar.back().first == 5) rp += r.cigar.back().second;
  }
  return (int32_t) rp;
}
// src/genotype.h:58-90: read coordinate of reference position pos
inline int32_t _findSeqBp(LrRecord const& r, uint32_t pos) {
  uint32_t rp = (uint32_t) r.pos, sp = 0;
  if (!r.cigar.empty()) {
    for (auto const& c : r.cigar) {
      const uint8_t op = c.first;
      const uint32_t len = c.second;
      if (op == 0 || op == 7 || op == 8) {
        if (rp >= pos) return (int32_t) sp;             // first base of the block
        if (pos - rp < len) return (int32_t) (sp + (pos - rp));
        rp += len; sp += len;
      } else if (op == 2 || op == 3) {
        rp += len;
        if (rp >= pos) return (int32_t) sp;
      } else if (op == 1 || op == 4 || op == 5) sp += len;
    }
    if (r.cigar.back().first == 4 || r.cigar.back().first == 5) return (int32_t) (sp - r.cigar.back().second);
  }
  return -1;
}

// The exchange of a contig-sharded genotypeLR: every rank sends, for the SVs with a breakpoint on its contigs, its decided qualities in job
// order (REF / ALT, per haplotype, the phase set of its first phased ALT read), the read-depth (non-zero on the rank of sv.chr only) and its
// methylation sums; the lists are concatenated in rank order, the sums added (finalizeMethylInfo sorts the CpG positions, so the sum of the
// per-rank counts is exact).
inline int mergeLrGenotypes(ContigShard const& cs, int localRc, std::vector<StructuralVariantRecord> const& svs, bool wantMethyl, std::vector<JunctionCount>& jctMap,
                            std::vector<ReadCount>& covMap, std::vector<MethylAccum>& acc) {
  ByteWriter w;
  auto putQ = [&](std::vector<uint8_t> const& v) { w.bytes(v); };
  for (uint32_t i = 0; i < svs.size(); ++i) {
    if (!cs.owns(svs[i].chr) && !cs.owns(svs[i].chr2)) continue;
    JunctionCount const& j = jctMap[i];
    w.pod(i);
    putQ(j.ref); putQ(j.alt); putQ(j.hp1ref); putQ(j.hp1alt); putQ(j.hp2ref); putQ(j.hp2alt); w.pod(j.ps);
    w.pod(covMap[i].leftRC); w.pod(covMap[i].rc); w.pod(covMap[i].rightRC);
    if (wantMethyl) {
      MethylAccum const& a = acc[i];
      for (int f = 0; f < 4; ++f) {
        w.pod(a.altM[f]); w.pod(a.altT[f]); w.pod(a.refM[f]); w.pod(a.refT[f]);
        w.pod<uint32_t>((uint32_t) a.cpg[f].size());
        for (auto const& kv : a.cpg[f]) { w.pod(kv.first); w.pod(kv.second); }
      }
    }
  }
  std::vector<std::string> parts;
  int rc = cs.exchange(localRc, w.buf, parts);
  if (rc) return rc;
  jctMap.assign(svs.size(), JunctionCount());
  covMap.assign(svs.size(), ReadCount());
  if (wantMethyl) acc.assign(svs.size(), MethylAccum());
  auto add = [](std::vector<uint8_t>& to, std::vector<uint8_t> const& v) { to.insert(to.end(), v.begin(), v.end()); };
  for (int r = 0; r < cs.nranks; ++r) {
    ByteReader rd(parts[r].data(), parts[r].size());
    while (rd.ok() && !rd.done()) {
      const uint32_t i = rd.pod<uint32_t>();
      if (!rd.ok() || i >= svs.size()) return DGPU_ERR_NCCL;
      JunctionCount& j = jctMap[i];
      add(j.ref, rd.bytes()); add(j.alt, rd.bytes()); add(j.hp1ref, rd.bytes()); add(j.hp1alt, rd.bytes()); add(j.hp2ref, rd.bytes()); add(j.hp2alt, rd.bytes());
      const int32_t ps = rd.pod<int32_t>();
      if (j.ps < 0) j.ps = ps;
      covMap[i].leftRC += rd.pod<int32_t>(); covMap[i].rc += rd.pod<int32_t>(); covMap[i].rightRC += rd.pod<int32_t>();
      if (wantMethyl) {
        MethylAccum& a = acc[i];
        for (int f = 0; f < 4; ++f) {
          a.altM[f] += rd.pod<uint32_t>(); a.altT[f] += rd.pod<uint32_t>(); a.refM[f] += rd.pod<uint32_t>(); a.refT[f] += rd.pod<uint32_t>();
          const uint32_t n = rd.pod<uint32_t>();
          for (uint32_t k = 0; k < n && rd.ok(); ++k) { const int32_t pos = rd.pod<int32_t>(); a.cpg[f][pos] += rd.pod<uint32_t>(); }
        }
      }
    }
    if (!rd.ok()) return DGPU_ERR_NCCL;
  }
  return DGPU_OK;
}

// genotypeLR for ONE sample: records sorted like a coordinate-sorted BAM (by tid, then pos). The read scan, the
// coverage track and the candidate selection run on the host exactly as the reference does; every
// (read, SV, breakpoint) candidate contributes two global edit distances (REF window vs read window, ALT window vs read
// window), and all of them go to the device in ONE dgpu_edit_distance call (NW) — the reference calls edlib twice per
// candidate, serially. The scores are then folded back in read order, so jctMap receives its qualities in the
// reference's order.
// The reference's first cap test (ref.size() + alt.size() >= maxGenoReadCount, :231) is implied by its second
// (reads seen for this SV, :233) because a read adds at most one quality after it has been counted; only the second
// is evaluated here, which is what makes the candidates independent of the scores.
// dump: receives the ALT-supporting (read, SV) groups in evaluation order (src/genotype.h:325-331)
// cs != nullptr (contig sharding): recs holds this rank's contigs only. A read only ever counts toward the SVs with a breakpoint on its own
// contig, so the per-SV cap needs a count from another rank only for an SV whose two breakpoints lie on two ranks' contigs (a translocation,
// or a BND site): the rank of the lower contig first sends the number of reads it will count for it (no alignment is needed for that), the
// rank of the higher contig starts its cap there. Every rank then realigns the reads of its contigs and sends, per SV, its decided qualities
// in job order, the read-depth of the SVs whose first breakpoint is on its contigs, and its methylation sums; every rank merges them in rank
// order (= contig order).
inline int genotypeLRBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                           std::vector<const char*> const& chrseq, std::vector<StructuralVariantRecord>& svs, std::vector<LrRecord> const& recs,
                           std::vector<JunctionCount>& jctMap, std::vector<ReadCount>& covMap, MethylConfig const* methylCfg = nullptr,
                           std::vector<MethylInfo>* methylMap = nullptr, std::vector<SvReadEvent>* dump = nullptr, ContigShard const* cs = nullptr) {
  jctMap.assign(svs.size(), JunctionCount());
  covMap.assign(svs.size(), ReadCount());
  const bool wantMethyl = (methylCfg != nullptr) && (methylMap != nullptr);
  if (wantMethyl) methylMap->assign(svs.size(), MethylInfo());
  if (svs.empty()) return DGPU_OK;
  if (cs && dump) return DGPU_ERR_ARG;
  auto bpMapOf = [&](int32_t refIndex, std::multimap<int32_t, int32_t>& bpMap) {
    for (auto const& sv : svs) {
      if (sv.chr == refIndex) bpMap.insert(std::make_pair(sv.svStart, sv.id));
      if (sv.chr2 == refIndex) bpMap.insert(std::make_pair(sv.svEnd, sv.id));
    }
  };
  // the SVs whose breakpoints a genotyping read spans (:189-222); false for a read that decides nothing
  auto spanned = [&](LrRecord const& rec, std::multimap<int32_t, int32_t> const& bpMap, std::set<int32_t>& process, int32_t& rStart, int32_t& rEnd) {
    if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP | BAMF_SUPPLEMENTARY | BAMF_SECONDARY)) return false;
    if (rec.mapq < c.minMapQual) return false;
    if ((int32_t) rec.seq.size() < 2 * c.minimumFlankSize) return false;
    rStart = _readStart(rec) + c.minimumFlankSize;
    rEnd = _readEnd(rec);
    if (rEnd > c.minimumFlankSize) {
      rEnd -= c.minimumFlankSize;
      if (rStart < rEnd) {
        auto itB = bpMap.lower_bound(rStart);
        auto itE = bpMap.upper_bound(rEnd);
        for (; (itB != itE) && (itB != bpMap.end()); ++itB) process.insert(itB->second);
      }
    }
    return true;
  };
  std::vector<uint32_t> readSV(svs.size(), 0);
  int rc = DGPU_OK;
  if (cs) {   // the counts of the SVs whose lower breakpoint contig is this rank's and whose other one a higher rank's
    auto split = [&](StructuralVariantRecord const& sv) { return cs->owner(sv.chr) != cs->owner(sv.chr2); };
    std::vector<uint32_t> lowerCount(svs.size(), 0);
    std::size_t ri = 0;
    for (int32_t refIndex = 0; refIndex < (int32_t) target_len.size(); ++refIndex) {
      const std::size_t rlo = ri;
      while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;
      if (rlo == ri || !cs->owns(refIndex)) continue;
      std::multimap<int32_t, int32_t> bpMap;
      for (auto const& sv : svs)
        if (split(sv) && std::min(sv.chr, sv.chr2) == refIndex) {
          if (sv.chr == refIndex) bpMap.insert(std::make_pair(sv.svStart, sv.id));
          if (sv.chr2 == refIndex) bpMap.insert(std::make_pair(sv.svEnd, sv.id));
        }
      if (bpMap.empty()) continue;
      for (std::size_t k = rlo; k < ri; ++k) {
        std::set<int32_t> process;
        int32_t rStart, rEnd;
        if (!spanned(recs[k], bpMap, process, rStart, rEnd)) continue;
        for (int32_t svid : process) if (lowerCount[svid] < c.maxGenoReadCount) ++lowerCount[svid];
      }
    }
    ByteWriter w;
    for (uint32_t i = 0; i < svs.size(); ++i) if (lowerCount[i]) { w.pod(i); w.pod(lowerCount[i]); }
    std::vector<std::string> parts;
    if ((rc = cs->exchange(DGPU_OK, w.buf, parts))) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      ByteReader rd(parts[r].data(), parts[r].size());
      while (rd.ok() && !rd.done()) {
        const uint32_t i = rd.pod<uint32_t>(), n = rd.pod<uint32_t>();
        if (!rd.ok() || i >= svs.size()) return DGPU_ERR_NCCL;
        if (cs->owns(std::max(svs[i].chr, svs[i].chr2))) readSV[i] = n;
      }
      if (!rd.ok()) return DGPU_ERR_NCCL;
    }
  }
  std::vector<std::vector<int32_t> > groupCands;  // the breakpoints of the SV each (read, SV) group spans (methylation windows)
  struct Cand { uint32_t rec, svid; uint32_t refSize, altSize; };
  std::vector<Cand> cands;                 // in the reference's evaluation order
  std::vector<uint32_t> groupEnd;          // cands of one (read, SV) pair end here
  std::vector<std::pair<uint32_t, uint32_t> > groupKey;  // (record, svid) per group
  std::string arena;
  std::vector<uint32_t> qo, ql, to, tl;
  std::size_t ri = 0;
  for (int32_t refIndex = 0; refIndex < (int32_t) target_len.size(); ++refIndex) {
    std::size_t rlo = ri;
    while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;   // this contig's records (tid < 0 never matches)
    std::multimap<int32_t, int32_t> bpMap;
    bpMapOf(refIndex, bpMap);
    if (bpMap.empty()) continue;
    const char* seq = chrseq[refIndex];
    for (auto& sv : svs)   // the alleles only slice the reference: every rank fills them for every SV
      if ((sv.chr == refIndex) && sv.alleles.empty())
        sv.alleles = _addAlleles(detail::upperSlice(seq, sv.svStart - 1, sv.svStart), target_name[sv.chr2], sv, sv.svt);
    if (cs && !cs->owns(refIndex)) continue;
    const uint32_t tlen = target_len[refIndex];
    std::vector<uint16_t> covBases(tlen, 0);
    const uint32_t maxCoverage = 65535;
    for (std::size_t k = rlo; k < ri; ++k) {
      LrRecord const& rec = recs[k];
      if (rec.flag & (BAMF_SECONDARY | BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP)) continue;
      if (rec.mapq < c.minMapQual) continue;
      {  // coverage track (:176-188)
        uint32_t rp = (uint32_t) rec.pos;
        for (auto const& cg : rec.cigar) {
          if (cg.first == 0 || cg.first == 7 || cg.first == 8) {
            for (uint32_t q = 0; q < cg.second; ++q, ++rp)
              if ((rp < tlen) && (covBases[rp] < maxCoverage - 1)) ++covBases[rp];
          } else if (cg.first == 2 || cg.first == 3) rp += cg.second;
        }
      }
      std::set<int32_t> process;
      int32_t rStart, rEnd;
      if (!spanned(rec, bpMap, process, rStart, rEnd)) continue;
      const int32_t lq = (int32_t) rec.seq.size();
      for (int32_t svid : process) {
        if (readSV[svid] >= c.maxGenoReadCount) continue;
        ++readSV[svid];
        StructuralVariantRecord const& sv = svs[svid];
        std::vector<int32_t> candidates;
        if ((sv.chr == refIndex) && (sv.svStart >= rStart) && (sv.svStart <= rEnd)) candidates.push_back(sv.svStart);
        if ((sv.chr2 == refIndex) && (sv.svEnd >= rStart) && (sv.svEnd <= rEnd)) candidates.push_back(sv.svEnd);
        if (candidates.empty()) continue;
        const std::size_t before = cands.size();
        for (int32_t pos : candidates) {
          const int32_t spBp = _findSeqBp(rec, (uint32_t) pos);
          int32_t consBp = sv.consBp;
          if (pos == sv.svEnd) consBp += sv.insLen;
          const int32_t rStartOffset = pos - std::max(0, pos - spBp);
          const int32_t rEndOffset = std::min(pos + lq - spBp, (int32_t) tlen) - pos;
          const int32_t cStartOffset = consBp - std::max(0, consBp - spBp);
          const int32_t cEndOffset = std::min(consBp + lq - spBp, (int32_t) sv.consensus.size()) - consBp;
          const int32_t offset = std::min(std::min(rStartOffset, cStartOffset), std::min(rEndOffset, cEndOffset));
          if (offset < c.minimumFlankSize) continue;
          if (!_translocation(sv.svt) && (2 * offset < c.minConsWindow)) continue;
          const std::string ref = detail::upperSlice(seq, pos - offset, pos + offset);
          const std::string alt = sv.consensus.substr((std::size_t) (consBp - offset), (std::size_t) (2 * offset));
          std::string probe = rec.seq.substr((std::size_t) (spBp - offset), (std::size_t) (2 * offset));
          // _editDistanceNW(ref, probe): the first argument is edlib's query
          qo.push_back((uint32_t) arena.size()); ql.push_back((uint32_t) ref.size()); arena += ref;
          to.push_back((uint32_t) arena.size()); tl.push_back((uint32_t) probe.size()); arena += probe;
          if (((sv.svt == 0) && (pos == sv.svEnd)) || ((sv.svt == 1) && (pos == sv.svStart)) || ((sv.svt == 5) && (pos == sv.svEnd)) ||
              ((sv.svt == 6) && (pos == sv.svStart)))
            reverseComplement(probe);
          qo.push_back((uint32_t) arena.size()); ql.push_back((uint32_t) alt.size()); arena += alt;
          to.push_back((uint32_t) arena.size()); tl.push_back((uint32_t) probe.size()); arena += probe;
          cands.push_back(Cand{(uint32_t) k, (uint32_t) svid, (uint32_t) ref.size(), (uint32_t) alt.size()});
        }
        if (cands.size() > before) {
          groupEnd.push_back((uint32_t) cands.size()); groupKey.push_back(std::make_pair((uint32_t) k, (uint32_t) svid));
          if (wantMethyl) groupCands.push_back(candidates);
        }
      }
    }
    // read-depth of the SV body and its flanks (:347-381)
    for (auto const& sv : svs) {
      if (sv.chr != refIndex) continue;
      const bool pointLike = _translocation(sv.svt) || (sv.svt == 4);
      int32_t halfSize = (sv.svEnd - sv.svStart) / 2;
      if (pointLike) halfSize = 500;
      auto sum = [&](int32_t b, int32_t e) { int32_t s = 0; for (uint32_t q = (uint32_t) b; (q < (uint32_t) e) && (q < tlen); ++q) s += covBases[q]; return s; };
      covMap[sv.id].leftRC = sum(std::max(sv.svStart - halfSize, 0), sv.svStart);
      if (pointLike) {
        covMap[sv.id].rc = sum(std::max(sv.svStart - halfSize, 0), std::min(sv.svStart + halfSize, (int32_t) tlen));
        covMap[sv.id].rightRC = sum(sv.svStart, std::min(sv.svStart + halfSize, (int32_t) tlen));
      } else {
        covMap[sv.id].rc = sum(sv.svStart, sv.svEnd);
        covMap[sv.id].rightRC = sum(sv.svEnd, std::min(sv.svEnd + halfSize, (int32_t) tlen));
      }
    }
  }
  std::vector<int32_t> dist(qo.size());
  if (!cands.empty())   // (no device call when no read reached a decision)
    rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), nullptr, DGPU_MODE_NW,
                            qo.size(), dist.data(), nullptr);
  if (rc && !cs) return rc;
  // fold the distances back per (read, SV) in evaluation order (:283-337)
  std::size_t ci = 0;
  std::vector<MethylAccum> methylAccum(wantMethyl ? svs.size() : 0);
  std::vector<InsertionJob> insQueue;
  std::vector<int8_t> methCall;          // calls of the record methCallRec (built once per read, :309-313)
  int64_t methCallRec = -1;
  bool hasMethyl = false;
  for (std::size_t g = 0; g < groupEnd.size() && !rc; ++g) {
    int32_t refedsum = 0, altedsum = 0, nInform = 0;
    for (; ci < groupEnd[g]; ++ci) {
      const int32_t refScore = dist[2 * ci], altScore = dist[2 * ci + 1];
      double scoreA = (1.0 - c.flankQuality) * cands[ci].altSize;
      double scoreR = (1.0 - c.flankQuality) * cands[ci].refSize;
      scoreA = scoreA / (double) (altScore + 1);
      scoreR = scoreR / (double) (refScore + 1);
      if ((scoreR > 0.6) || (scoreA > 0.6)) { refedsum += refScore; altedsum += altScore; ++nInform; }
    }
    if (nInform == 0) continue;
    const int32_t delta = refedsum - altedsum;
    const int32_t adelta = (delta < 0) ? -delta : delta;
    const double w = std::log10((double) c.flankQuality / (double) (1.0 - c.flankQuality));
    double ex = (double) adelta * w;
    if (ex > 4.0) ex = 4.0;
    uint32_t mq = (uint32_t) (10.0 * std::log10(1.0 + std::pow(10.0, ex)));
    if (mq > (uint32_t) c.genoCap) mq = (uint32_t) c.genoCap;
    const uint8_t qual = (uint8_t) mq;
    LrRecord const& rec = recs[groupKey[g].first];
    JunctionCount& jc = jctMap[groupKey[g].second];
    if (wantMethyl) {  // :306-324: the calls of this read go to the SV's windows under the allele it supports
      MethylRead mr;
      mr.pos = rec.pos; mr.reverse = (rec.flag & BAMF_REVERSE) != 0; mr.cigar = &rec.cigar; mr.seq = &rec.seq;
      mr.hasMM = rec.hasMM; mr.hasML = rec.hasML; mr.mm = &rec.mm; mr.ml = &rec.ml;
      if (methCallRec != (int64_t) groupKey[g].first) {
        methCallRec = (int64_t) groupKey[g].first;
        hasMethyl = buildMethylCalls(mr, (uint8_t) methylCfg->methylProb, methCall);
      }
      if (hasMethyl)
        accumulateMethyl(*methylCfg, mr, methCall, svs[groupKey[g].second], rec.tid, (int32_t) target_len[rec.tid], delta > 0, groupCands[g],
                         methylAccum[groupKey[g].second], insQueue);
    }
    if (delta <= 0) {
      jc.ref.push_back(qual);
      if (rec.hp == 1) jc.hp1ref.push_back(qual);
      else if (rec.hp == 2) jc.hp2ref.push_back(qual);
    } else {
      if (dump) dump->push_back(SvReadEvent{groupKey[g].first, groupKey[g].second, svs[groupKey[g].second].svt});
      jc.alt.push_back(qual);
      if (rec.hp == 1) jc.hp1alt.push_back(qual);
      else if (rec.hp == 2) jc.hp2alt.push_back(qual);
      if ((rec.hp > 0) && (rec.ps >= 0) && (jc.ps < 0)) jc.ps = rec.ps;
    }
  }
  if (wantMethyl && !rc) rc = flushInsertionJobs(ctx, *methylCfg, insQueue, methylAccum);
  if (rc && !cs) return rc;
  if (cs && (rc = mergeLrGenotypes(*cs, rc, svs, wantMethyl, jctMap, covMap, methylAccum))) return rc;
  if (wantMethyl)
    for (std::size_t i = 0; i < svs.size(); ++i) finalizeMethylInfo(methylAccum[i], (*methylMap)[i], methylCfg->minCpgDepth);
  return DGPU_OK;
}


// ---- short-read genotyping pass, junction reads (annotateCoverage, src/coverage.h:265-548 + :412-454, :671-675) -------------

constexpr uint32_t BAMF_MUNMAP = 0x8;

struct SrRecord {  // what annotateCoverage reads from one bam1_t
  int32_t tid = 0, pos = 0;
  uint32_t flag = 0;
  uint8_t mapq = 0;
  std::vector<std::pair<uint8_t, uint32_t> > cigar;
  std::string seq;              // junction-read half only
  int32_t lqseq = 0;            // l_qseq (= seq.size() when the bases are present)
  int32_t mtid = 0, mpos = 0, isize = 0;
  uint64_t name = 0;            // query-name identity: mates share it (the reference hashes the name, src/tags.h:260-267)
  uint32_t nameHash32 = 0;      // hash_string(qname) (src/tags.h:260-267); only scanPEandSRBatch needs the actual value, see there
  std::size_t seed = 0;         // hash_sr(rec) (src/util.h:519-527); 0 = derive from name and the read-2 flag
};

struct LibraryInfo {  // src/util.h:29-41
  int32_t rs = 0, median = 0, mad = 0, minNormalISize = 0, minISizeCutoff = 0, maxNormalISize = 0, maxISizeCutoff = 0;
  uint32_t abnormal_pairs = 0;
};

struct SpanningCount {  // src/coverage.h:69-72
  std::vector<uint8_t> ref, alt;
};

// src/split.h:55-68
inline void _adjustOrientation(std::string& sequence, unsigned int bpPoint, int32_t svt) {
  if (_translocation(svt)) {
    const uint8_t ct = _getSpanOrientation(svt);
    if (((ct == 0) && bpPoint) || ((ct == 1) && !bpPoint)) reverseComplement(sequence);
  } else if (svt == 0) { if (bpPoint) reverseComplement(sequence); }
  else if (svt == 1) { if (!bpPoint) reverseComplement(sequence); }
}

// The junction-read half of annotateCoverage for ONE sample: probes (generateProbesBatch), the read scan that turns every
// read over a breakpoint region into an AlignJob, the batched realignment (processBatch: one dgpu_edit_distance per
// batch) and the merge into countMap with the reference's reference-bias rule (every second REF read is dropped, :448).
// Batches are flushed exactly where the reference flushes them — when 131072 x maxThreads jobs are buffered and at the end
// of every contig — because the scan consults countMap (the maxGenoReadCount cap, :501) between batches, so the batch
// boundaries are part of the result. The spanning-pair and read-depth half (:551-733) is not part of this function.
// The probes of an SV list (the reference computes them once, before the loop over the files: src/coverage.h:164-263)
struct JunctionProbes {
  std::vector<std::vector<std::string> > refProbeArr, consProbeArr;
  std::vector<std::vector<BpRegion> > bpRegion;
  std::vector<bool> svOnChr;
};
inline int prepareJunctionProbes(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                                 std::vector<const char*> const& chrseq, std::vector<StructuralVariantRecord>& svs, JunctionProbes& p,
                                 std::vector<uint8_t> const* want = nullptr) {
  std::vector<uint32_t> bad;
  int rc = generateProbesBatch(ctx, c, target_len, target_name, chrseq, svs, p.refProbeArr, p.consProbeArr, p.bpRegion, p.svOnChr, bad, want);
  if (rc) return rc;
  if (!bad.empty()) return DGPU_ERR_ARG;  // the reference would have thrown (std::out_of_range in substr)
  return DGPU_OK;
}

inline int annotateJunctionReadsWithProbes(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, JunctionProbes const& probes, std::size_t nSv,
                                           std::vector<SrRecord> const& recs, std::vector<JunctionCount>& countMap, std::vector<SvReadEvent>* dump = nullptr,
                                           ContigShard const* cs = nullptr);

inline int annotateJunctionReadsBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                                      std::vector<const char*> const& chrseq, std::vector<StructuralVariantRecord>& svs, std::vector<SrRecord> const& recs,
                                      std::vector<JunctionCount>& countMap, std::vector<SvReadEvent>* dump = nullptr) {
  JunctionProbes probes;
  int rc = prepareJunctionProbes(ctx, c, target_len, target_name, chrseq, svs, probes);
  if (rc) return rc;
  return annotateJunctionReadsWithProbes(ctx, c, target_len, probes, svs.size(), recs, countMap, dump);
}

// the per-file pass (src/coverage.h:346-548, :671-675) over probes prepared once.
// Structure (results identical to the reference's, cheaper to produce):
//  * the read scan of every contig runs on its own host thread and only records WHICH (read, breakpoint) pairs become jobs — no strings are copied;
//  * the reference flushes its job buffer every 131072 x threads jobs and at the end of a contig, and consults the per-SV cap both when it queues a
//    job and when it merges a result. Results are merged in job order and a job that is skipped at queue time because the cap was reached would
//    have been dropped at the merge anyway, so neither the flush points nor the queue-time check change the outcome: here every job is queued,
//    all jobs go to the device in as few dgpu_edit_distance calls as the 4 GiB arena allows, and the merge applies the cap in job order;
//  * the arena holds every probe once and every read once per orientation (the ALT and REF job of a read share it; BAM_FREVERSE-dependent
//    orientation per breakpoint is src/split.h:55-68), instead of three strings per job.
// dump: receives the ALT junction reads in job order (src/coverage.h:528-532). The reference aligns one job at a time when it dumps and checks
// the cap against exact counts before each alignment; the merge below applies the same check to the same jobs in the same order.
// cs != nullptr (contig sharding): recs holds this rank's contigs only; the rank aligns the jobs of its contigs, and the decided jobs of all
// ranks (SV, REF / ALT, quality) are gathered and merged in job order — contig order is rank order — on every rank.
inline int annotateJunctionReadsWithProbes(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, JunctionProbes const& probes, std::size_t nSv,
                                           std::vector<SrRecord> const& recs, std::vector<JunctionCount>& countMap, std::vector<SvReadEvent>* dump,
                                           ContigShard const* cs) {
  std::vector<std::vector<std::string> > const& refProbeArr = probes.refProbeArr;
  std::vector<std::vector<std::string> > const& consProbeArr = probes.consProbeArr;
  std::vector<std::vector<BpRegion> > const& bpRegion = probes.bpRegion;
  std::vector<bool> const& svOnChr = probes.svOnChr;
  countMap.assign(nSv, JunctionCount());
  struct LightJob { uint32_t rec, svId; int32_t svt; uint8_t bpPoint, qual; };
  const int32_t nchr = (int32_t) target_len.size();
  std::vector<std::size_t> lo((std::size_t) nchr + 1, recs.size());
  {
    std::size_t ri = 0;
    for (int32_t refIndex = 0; refIndex < nchr; ++refIndex) { lo[refIndex] = ri; while (ri < recs.size() && recs[ri].tid == refIndex) ++ri; }
    lo[nchr] = ri;
  }
  std::vector<std::vector<LightJob> > jobsOf((std::size_t) nchr);
  auto scanContig = [&](int32_t refIndex) {
    if (!svOnChr[refIndex] || (cs && !cs->owns(refIndex))) return;
    const int32_t tlen = (int32_t) target_len[refIndex];
    // the union of the breakpoint regions as sorted disjoint intervals: "does the read touch a region" is one binary search
    std::vector<std::pair<int32_t, int32_t> > iv;
    for (BpRegion const& b : bpRegion[refIndex]) if (b.regionEnd > b.regionStart) iv.push_back(std::make_pair(b.regionStart, b.regionEnd));
    std::sort(iv.begin(), iv.end());
    std::vector<int32_t> ivStart, ivEnd;
    for (auto const& x : iv) {
      if (!ivEnd.empty() && x.first <= ivEnd.back()) ivEnd.back() = std::max(ivEnd.back(), x.second);
      else { ivStart.push_back(x.first); ivEnd.push_back(x.second); }
    }
    std::vector<LightJob>& out = jobsOf[(std::size_t) refIndex];
    for (std::size_t q = lo[refIndex]; q < lo[refIndex + 1]; ++q) {
      SrRecord const& rec = recs[q];
      if (rec.flag & (BAMF_SECONDARY | BAMF_QCFAIL | BAMF_DUP | BAMF_SUPPLEMENTARY | BAMF_UNMAP | BAMF_MUNMAP)) continue;
      if (rec.mapq < c.minGenoQual) continue;
      bool hasSoftClip = false, hasClip = false;
      int32_t leadingSC = 0;
      for (std::size_t i = 0; i < rec.cigar.size(); ++i) {
        if (rec.cigar[i].first == 4) { hasClip = true; hasSoftClip = true; if (i == 0) leadingSC = (int32_t) rec.cigar[i].second; }
        else if (rec.cigar[i].first == 5) hasClip = true;
      }
      const int32_t lq = (int32_t) rec.seq.size();
      if (lq < 2 * c.minimumFlankSize) continue;
      const int32_t rbegin = std::max(0, rec.pos - leadingSC);
      const int32_t rend = std::min(rec.pos + lq, tlen);
      if (rend <= rbegin) continue;
      {
        const std::size_t u = (std::size_t) (std::upper_bound(ivEnd.begin(), ivEnd.end(), rbegin) - ivEnd.begin());   // first interval ending after rbegin
        if ((u == ivEnd.size()) || (ivStart[u] >= rend)) continue;
      }
      BpRegion probe; probe.bppos = rbegin;
      auto itBp = std::lower_bound(bpRegion[refIndex].begin(), bpRegion[refIndex].end(), probe);
      for (; (itBp != bpRegion[refIndex].end()) && (rec.pos + lq >= itBp->bppos); ++itBp) {
        if (hasSoftClip || ((!hasClip) && (rec.pos + c.minimumFlankSize + itBp->homLeft <= itBp->bppos) &&
                            (rec.pos + lq >= itBp->bppos + c.minimumFlankSize + itBp->homRight)))
          out.push_back(LightJob{(uint32_t) q, itBp->id, itBp->svt, itBp->bpPoint, rec.mapq});
      }
    }
  };
  {
    const unsigned hw = hostThreads();
    std::atomic<int32_t> next(0);
    auto worker = [&]() { for (int32_t r = next++; r < nchr; r = next++) scanContig(r); };
    std::vector<std::thread> pool;
    const unsigned nth = std::min<unsigned>(hw, (unsigned) nchr);
    for (unsigned t = 1; t < nth; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
  }
  // ---- arena: probes once, reads once per orientation; jobs in the reference's order (contig, read, breakpoint) ------------------------------
  std::vector<uint32_t> refAlignedReadCount(nSv, 0);
  // the merge of one decided job into the SV's lists (src/coverage.h:442-453); true = an ALT read was added
  auto merge = [&](uint32_t svId, bool isRef, uint8_t qual) {
    JunctionCount& jc = countMap[svId];
    if ((jc.ref.size() + jc.alt.size()) >= c.maxGenoReadCount) return false;
    if (!isRef) { jc.alt.push_back(qual); return true; }
    if (++refAlignedReadCount[svId] % 2) jc.ref.push_back(qual);
    return false;
  };
  ByteWriter votes;   // contig sharding: this rank's decided jobs, in job order
  int rc = DGPU_OK;
  std::vector<LightJob> jobs;
  for (auto& v : jobsOf) { jobs.insert(jobs.end(), v.begin(), v.end()); std::vector<LightJob>().swap(v); }
  const std::size_t J = jobs.size();
  std::size_t done = 0;
  while (done < J) {
    std::string arena;
    std::unordered_map<uint64_t, uint32_t> probeOff, readOff;   // (svId, bpPoint, which) -> offset; (rec, flipped) -> offset
    std::vector<uint32_t> qo, ql, to, tl;
    std::vector<int32_t> k;
    std::size_t end = done;
    auto placeProbe = [&](std::string const& p, uint64_t key) -> uint32_t {
      auto it = probeOff.find(key);
      if (it != probeOff.end()) return it->second;
      const uint32_t off = (uint32_t) arena.size();
      arena += p;
      probeOff.emplace(key, off);
      return off;
    };
    for (; end < J; ++end) {
      LightJob const& j = jobs[end];
      if (arena.size() > 3000000000ull) break;   // dgpu_edit_distance takes arenas below 4 GiB
      std::string const& cons = consProbeArr[j.bpPoint][j.svId];
      std::string const& ref = refProbeArr[j.bpPoint][j.svId];
      // does _adjustOrientation flip this read for this breakpoint? (src/split.h:55-68)
      bool flip = false;
      if (_translocation(j.svt)) { const uint8_t ct = _getSpanOrientation(j.svt); flip = ((ct == 0) && j.bpPoint) || ((ct == 1) && !j.bpPoint); }
      else if (j.svt == 0) flip = (j.bpPoint != 0);
      else if (j.svt == 1) flip = (j.bpPoint == 0);
      const uint64_t rkey = ((uint64_t) j.rec << 1) | (flip ? 1u : 0u);
      uint32_t so;
      auto itR = readOff.find(rkey);
      if (itR != readOff.end()) so = itR->second;
      else {
        so = (uint32_t) arena.size();
        if (flip) { std::string sq = recs[j.rec].seq; reverseComplement(sq); arena += sq; }
        else arena += recs[j.rec].seq;
        readOff.emplace(rkey, so);
      }
      const uint64_t pkey = (((uint64_t) j.svId << 1) | j.bpPoint) << 1;
      qo.push_back(placeProbe(cons, pkey)); ql.push_back((uint32_t) cons.size());
      qo.push_back(placeProbe(ref, pkey | 1u)); ql.push_back((uint32_t) ref.size());
      const uint32_t sl = (uint32_t) recs[j.rec].seq.size();
      to.push_back(so); tl.push_back(sl); to.push_back(so); tl.push_back(sl);
      k.push_back(_hwBound(c, cons.size())); k.push_back(_hwBound(c, ref.size()));
    }
    const std::size_t n = end - done;
    std::vector<int32_t> dist(2 * n);
    rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), qo.data(), ql.data(), to.data(), tl.data(), k.data(), DGPU_MODE_HW, 2 * n,
                            dist.data(), nullptr);
    if (rc && !cs) return rc;
    if (rc) break;
    for (std::size_t i = 0; i < n; ++i) {   // processBatch scoring (src/coverage.h:412-441) and the merge (:442-453), in job order
      LightJob const& j = jobs[done + i];
      const double scoreAlt = _hwScore(c, ql[2 * i], dist[2 * i]);
      const double scoreRef = _hwScore(c, ql[2 * i + 1], dist[2 * i + 1]);
      if (!((scoreRef > 0.7) || (scoreAlt > 0.7))) continue;
      const bool isRef = scoreRef > scoreAlt;
      const uint8_t qual = (uint8_t) std::min(255, std::min((int) ((isRef ? scoreRef : scoreAlt) * 35), (int) j.qual));
      if (cs) { votes.pod(j.svId); votes.pod<uint8_t>(isRef); votes.pod(qual); continue; }
      if (merge(j.svId, isRef, qual) && dump) dump->push_back(SvReadEvent{j.rec, j.svId, j.svt});
    }
    done = end;
  }
  if (cs) {
    std::vector<std::string> parts;
    if ((rc = cs->exchange(rc, votes.buf, parts))) return rc;
    for (std::string const& part : parts) {
      ByteReader rd(part.data(), part.size());
      while (rd.ok() && !rd.done()) {
        const uint32_t svId = rd.pod<uint32_t>();
        const bool isRef = rd.pod<uint8_t>() != 0;
        const uint8_t qual = rd.pod<uint8_t>();
        if (!rd.ok() || svId >= nSv) return DGPU_ERR_NCCL;
        merge(svId, isRef, qual);
      }
    }
  }
  return DGPU_OK;
}


// src/tags.h:217-226 on the record's own fields
inline uint8_t getSVType(SrRecord const& r) {
  const bool rev = (r.flag & BAMF_REVERSE) != 0, mrev = (r.flag & 0x20) != 0;  // BAM_FMREVERSE
  if (!rev) return !mrev ? 0 : ((r.pos < r.mpos) ? 2 : 3);
  return !mrev ? ((r.pos > r.mpos) ? 2 : 3) : 1;
}
// src/tags.h:228-258
inline int32_t _isizeMappingPos(SrRecord const& r, int32_t isize) {
  if (r.tid != r.mtid) {
    const uint8_t orient = getSVType(r);
    if (orient == 0) return DELLY_SVT_TRANS + 0;
    if (orient == 1) return DELLY_SVT_TRANS + 1;
    const bool fwd = !(r.flag & BAMF_REVERSE);
    if (r.tid > r.mtid) return fwd ? DELLY_SVT_TRANS + 2 : DELLY_SVT_TRANS + 3;
    return fwd ? DELLY_SVT_TRANS + 3 : DELLY_SVT_TRANS + 2;
  }
  if (r.pos == r.mpos) return -1;
  const uint8_t orient = getSVType(r);
  if (orient == 0) return 0;
  if (orient == 1) return 1;
  if (orient == 2) return (isize > std::abs(r.isize)) ? -1 : 2;
  return (std::abs(r.pos - r.mpos) < 100) ? -1 : 3;
}

// The spanning-pair and read-depth half of annotateCoverage (src/coverage.h:368-406, :456-470, :551-668, :681-733) for ONE sample —
// pure host logic (no alignment): mate bookkeeping (first/second read of a pair, clip flags, pair quality), fragment and
// base coverage tracks, REF-spanning pairs over a breakpoint (every second one kept, :616), ALT-spanning abnormal pairs of the
// SV's type whose mate lands near the other breakpoint, and the left / body / right read-depth of every SV.
// svOnChr as produced by generateProbesBatch. The reference keys its mate table by a hash of (name, tid, pos, mtid, mpos);
// here the key is the tuple itself.
// dump: receives the ALT-spanning pair events in contig order, record order within a contig (src/coverage.h:652-657)
// cs != nullptr (contig sharding): recs holds this rank's contigs only. The inter-chromosomal first observations go to the rank of the mate's
// contig, the rank walks its own contigs, and the events of every contig and the read-depth of every SV (counted on contig sv.chr) are gathered
// and replayed in contig order on every rank.
inline int annotateSpanningAndDepth(Config const& c, LibraryInfo const& lib, std::vector<uint32_t> const& target_len,
                                    std::vector<StructuralVariantRecord> const& svs, std::vector<bool> const& svOnChr, std::vector<SrRecord> const& recs,
                                    std::vector<ReadCount>& covCount, std::vector<SpanningCount>& spanMap, std::vector<SvReadEvent>* dump = nullptr,
                                    ContigShard const* cs = nullptr) {
  covCount.assign(svs.size(), ReadCount());
  spanMap.assign(svs.size(), SpanningCount());
  typedef std::map<TPairKey, std::pair<bool, uint8_t> > TClipQual;
  struct SpanPoint { int32_t bppos, svt; uint32_t id; int32_t chr2, otherBppos; bool operator<(SpanPoint const& o) const { return bppos < o.bppos; } };
  struct SpanEvent { uint32_t id; uint8_t alt, quality; };   // one push_back of the reference, replayed in contig order below
  const uint32_t maxCoverage = 65535;
  const int32_t nchr = (int32_t) target_len.size();
  // The reference walks the contigs one after the other; the contigs are independent except for (1) the mate table of inter-chromosomal pairs
  // (filled on the contig with the smaller index, read and erased on the mate's contig) and (2) the order in which qualities are appended
  // to an SV's lists when two contigs touch it. So: record ranges and the inter-chromosomal first observations first (sequential, one cheap pass;
  // the table is split by the contig that will read it), then the contigs in parallel with their appends recorded, then the appends in contig order.
  std::vector<std::size_t> lo((std::size_t) nchr + 1, recs.size());
  {
    std::size_t ri = 0;
    for (int32_t refIndex = 0; refIndex < nchr; ++refIndex) {
      lo[refIndex] = ri;
      while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;
    }
    lo[nchr] = ri;
  }
  auto softClipped = [](SrRecord const& rec) { for (auto const& cg : rec.cigar) if (cg.first == 4) return true; return false; };
  std::vector<TClipQual> cliptraOf((std::size_t) nchr);
  for (int32_t refIndex = 0; refIndex < nchr; ++refIndex) {
    if (!svOnChr[refIndex]) continue;
    for (std::size_t q = lo[refIndex]; q < lo[refIndex + 1]; ++q) {
      SrRecord const& rec = recs[q];
      if (rec.tid >= rec.mtid || rec.mtid >= nchr) continue;   // first observation of an inter-chromosomal pair: tid < mtid
      if (rec.flag & (BAMF_SECONDARY | BAMF_QCFAIL | BAMF_DUP | BAMF_SUPPLEMENTARY | BAMF_UNMAP | BAMF_MUNMAP)) continue;
      if (rec.mapq < c.minGenoQual) continue;
      if ((!(rec.flag & 0x1)) || (!svOnChr[rec.mtid])) continue;
      cliptraOf[rec.mtid][TPairKey(rec.name, rec.tid, rec.pos, rec.mtid, rec.mpos)] = std::make_pair(softClipped(rec), rec.mapq);
    }
  }
  int rc = DGPU_OK;
  if (cs && (rc = shareMateTables(*cs, DGPU_OK, cliptraOf))) return rc;
  std::vector<std::vector<SpanEvent> > events((std::size_t) nchr);
  std::vector<std::vector<SvReadEvent> > dumpOf(dump ? (std::size_t) nchr : 0);
  auto doContig = [&](std::size_t refIndexU) {
    const int32_t refIndex = (int32_t) refIndexU;
    if (!svOnChr[refIndex] || (cs && !cs->owns(refIndex))) return;
    const std::size_t rlo = lo[refIndex], ri = lo[refIndex + 1];
    TClipQual clip;
    TClipQual& cliptra = cliptraOf[refIndex];
    std::vector<SpanEvent>& ev = events[refIndex];
    std::vector<SvReadEvent>* dumpEv = dump ? &dumpOf[refIndex] : nullptr;
    const int32_t tlen = (int32_t) target_len[refIndex];
    std::vector<uint16_t> covFragment((std::size_t) tlen, 0), covBases((std::size_t) tlen, 0);
    // base coverage as a difference array (one +1 / -1 per aligned block instead of one increment per base); the reference's saturating
    // counter (++ only below maxCoverage - 1) is min(count, maxCoverage - 1), applied when the array is integrated after the scan
    std::vector<int32_t> covDiff((std::size_t) tlen + 1, 0);
    std::vector<SpanPoint> spanPoint;
    for (auto const& sv : svs) {
      if (sv.peSupport == 0) continue;
      if ((sv.chr == refIndex) && (sv.svStart < tlen)) spanPoint.push_back(SpanPoint{sv.svStart, sv.svt, (uint32_t) sv.id, sv.chr2, sv.svEnd});
      if ((sv.chr2 == refIndex) && (sv.svEnd < tlen)) spanPoint.push_back(SpanPoint{sv.svEnd, sv.svt, (uint32_t) sv.id, sv.chr, sv.svStart});
    }
    std::sort(spanPoint.begin(), spanPoint.end());
    int32_t lastAlignedPos = 0;
    std::set<uint64_t> lastAlignedPosReads;
    for (std::size_t q = rlo; q < ri; ++q) {
      SrRecord const& rec = recs[q];
      if (rec.flag & (BAMF_SECONDARY | BAMF_QCFAIL | BAMF_DUP | BAMF_SUPPLEMENTARY | BAMF_UNMAP | BAMF_MUNMAP)) continue;
      if (rec.mapq < c.minGenoQual) continue;
      {  // aligned bases (:461-475: only M counts, D and N skip)
        uint32_t rp = 0;
        for (auto const& cg : rec.cigar) {
          if (cg.first == 0) {
            const int64_t b0 = (int64_t) rec.pos + rp, b1 = std::min<int64_t>(b0 + cg.second, tlen);
            if (b0 < b1) { ++covDiff[(std::size_t) b0]; --covDiff[(std::size_t) b1]; }
            rp += cg.second;
          } else if (cg.first == 2 || cg.first == 3) rp += cg.second;
        }
      }
      const bool hasSoftClip = softClipped(rec);
      if ((!(rec.flag & 0x1)) || (rec.mtid < 0) || (!svOnChr[rec.mtid])) continue;  // BAM_FPAIRED; (a negative mtid would index out of bounds in the reference)
      if (rec.pos > lastAlignedPos) { lastAlignedPosReads.clear(); lastAlignedPos = rec.pos; }
      const bool firstObs = (rec.tid == rec.mtid) ? ((rec.pos < rec.mpos) || ((rec.pos == rec.mpos) && !lastAlignedPosReads.count(rec.name))) : (rec.tid < rec.mtid);
      if (firstObs) {
        lastAlignedPosReads.insert(rec.name);
        if (rec.tid == rec.mtid) clip[TPairKey(rec.name, rec.tid, rec.pos, rec.mtid, rec.mpos)] = std::make_pair(hasSoftClip, rec.mapq);
        continue;   // inter-chromosomal first observations are already in the mate's table
      }
      const TPairKey hv(rec.name, rec.mtid, rec.mpos, rec.tid, rec.pos);
      TClipQual& tab = (rec.tid == rec.mtid) ? clip : cliptra;
      auto itCM = tab.find(hv);
      if (itCM == tab.end()) continue;  // mate discarded
      const uint8_t pairQuality = std::min((uint8_t) itCM->second.second, rec.mapq);
      const bool pairClip = itCM->second.first || hasSoftClip;
      tab.erase(itCM);
      if (pairQuality < c.minGenoQual) continue;
      if (rec.tid == rec.mtid) {  // fragment mid point (:589-593); halfAlignmentLength = (M,=,X,D,N lengths) / 2
        uint32_t alen = 0;
        for (auto const& cg : rec.cigar) if (cg.first == 0 || cg.first == 7 || cg.first == 8 || cg.first == 2 || cg.first == 3) alen += cg.second;
        const int32_t midPoint = rec.pos + (int32_t) (alen / 2);
        if ((midPoint < tlen) && (covFragment[(std::size_t) midPoint] < maxCoverage - 1)) ++covFragment[(std::size_t) midPoint];
      }
      int32_t outerISize = (rec.pos < rec.mpos) ? rec.mpos + rec.lqseq - rec.pos : rec.pos + rec.lqseq - rec.mpos;
      if (lib.median == 0) continue;
      const uint8_t svType = getSVType(rec);
      if ((!pairClip) && (svType == 2) && (outerISize >= lib.minNormalISize) && (outerISize <= lib.maxNormalISize) && (rec.tid == rec.mtid)) {
        const int32_t spanlen = (int32_t) (0.8 * outerISize);
        const int32_t pbegin = std::min(rec.pos, rec.mpos);
        const int32_t st = pbegin + (outerISize - spanlen) / 2;
        auto itSpan = std::lower_bound(spanPoint.begin(), spanPoint.end(), SpanPoint{st, 0, 0, 0, 0});
        // a breakpoint inside [st, st + spanlen) (and on the contig): the sorted breakpoint list answers it without walking the interval
        const bool spanvalid = (itSpan != spanPoint.end()) && (itSpan->bppos < std::min(st + spanlen, tlen));
        if (spanvalid) {
          for (; (itSpan != spanPoint.end()) && (st + spanlen >= itSpan->bppos); ++itSpan) ev.push_back(SpanEvent{itSpan->id, 0, pairQuality});
        }
      }
      if ((svType != 2) || (outerISize < lib.minNormalISize) || (outerISize > lib.maxNormalISize) || (rec.tid != rec.mtid)) {
        const int32_t svt = _isizeMappingPos(rec, lib.maxISizeCutoff);
        if (svt == -1) continue;
        int32_t pbegin = rec.pos;
        int32_t pend = std::min(rec.pos + lib.maxNormalISize, tlen);
        if (rec.flag & BAMF_REVERSE) {
          pbegin = std::max(0, rec.pos + rec.lqseq - lib.maxNormalISize);
          pend = std::min(rec.pos + rec.lqseq, tlen);
        }
        auto itSpan = std::lower_bound(spanPoint.begin(), spanPoint.end(), SpanPoint{pbegin, 0, 0, 0, 0});
        const bool spanvalid = (itSpan != spanPoint.end()) && (itSpan->bppos < pend);
        if (spanvalid) {
          for (; (itSpan != spanPoint.end()) && (pend >= itSpan->bppos); ++itSpan)
            if ((svt == itSpan->svt) && (rec.mtid == itSpan->chr2) && (std::abs(rec.mpos - itSpan->otherBppos) < lib.maxNormalISize)) {
              ev.push_back(SpanEvent{itSpan->id, 1, pairQuality});
              if (dumpEv) dumpEv->push_back(SvReadEvent{(uint32_t) q, itSpan->id, itSpan->svt});
            }
        }
      }
    }
    {
      int64_t run = 0;
      for (int32_t k = 0; k < tlen; ++k) { run += covDiff[(std::size_t) k]; covBases[(std::size_t) k] = (uint16_t) std::min<int64_t>(run, maxCoverage - 1); }
    }
    // fragment / base counts left of, inside and right of every SV of this contig (:681-733)
    for (auto const& sv : svs) {
      if (sv.chr != refIndex) continue;
      bool smallSV = false;
      int32_t halfSize = (sv.svEnd - sv.svStart) / 2;
      const bool pointLike = _translocation(sv.svt) || (sv.svt == 4);
      if (pointLike) { halfSize = 500; smallSV = true; }
      else if ((sv.svEnd - sv.svStart) <= c.indelsize) smallSV = true;
      auto sum = [&](int32_t b, int32_t e) {
        int32_t s = 0;
        for (uint32_t k = (uint32_t) b; (k < (uint32_t) e) && (k < (uint32_t) tlen); ++k) s += smallSV ? covBases[k] : covFragment[k];
        return s;
      };
      covCount[sv.id].leftRC = sum(std::max(sv.svStart - halfSize, 0), sv.svStart);
      if (pointLike) {
        covCount[sv.id].rc = sum(std::max(sv.svStart - halfSize, 0), std::min(sv.svStart + halfSize, tlen));
        covCount[sv.id].rightRC = sum(sv.svStart, std::min(sv.svStart + halfSize, tlen));
      } else {
        covCount[sv.id].rc = sum(sv.svStart, sv.svEnd);
        covCount[sv.id].rightRC = sum(sv.svEnd, std::min(sv.svEnd + halfSize, tlen));
      }
    }
  };
  {
    // every worker holds the coverage arrays of one contig (8 bytes per base): at most eight at a time
    std::atomic<std::size_t> next(0);
    auto worker = [&]() { for (std::size_t r = next++; r < (std::size_t) nchr; r = next++) doContig(r); };
    const std::size_t nth = std::min<std::size_t>(std::min<std::size_t>(hostThreads(), 8), (std::size_t) std::max(1, nchr));
    std::vector<std::thread> pool;
    for (std::size_t t = 1; t < nth; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
  }
  if (cs) {   // the other ranks' contig events and read-depth
    ByteWriter w;
    for (std::size_t refIndex = cs->lo(); refIndex < cs->hi(); ++refIndex) {
      w.pod<uint64_t>((uint64_t) events[refIndex].size());
      for (SpanEvent const& e : events[refIndex]) { w.pod(e.id); w.pod(e.alt); w.pod(e.quality); }
    }
    for (auto const& sv : svs) if (cs->owns(sv.chr)) w.pod(covCount[sv.id]);
    std::vector<std::string> parts;
    if ((rc = cs->exchange(DGPU_OK, w.buf, parts))) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      if (r == cs->rank) continue;
      ByteReader rd(parts[r].data(), parts[r].size());
      for (std::size_t refIndex = cs->bounds[r]; refIndex < cs->bounds[r + 1]; ++refIndex) {
        const uint64_t n = rd.pod<uint64_t>();
        for (uint64_t k = 0; k < n && rd.ok(); ++k) {
          SpanEvent e;
          e.id = rd.pod<uint32_t>(); e.alt = rd.pod<uint8_t>(); e.quality = rd.pod<uint8_t>();
          if (e.id >= svs.size()) return DGPU_ERR_NCCL;
          events[refIndex].push_back(e);
        }
      }
      for (auto const& sv : svs)
        if (sv.chr >= (int32_t) cs->bounds[r] && sv.chr < (int32_t) cs->bounds[r + 1]) covCount[sv.id] = rd.pod<ReadCount>();
      if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
    }
  }
  std::vector<uint32_t> refAlignedSpanCount(svs.size(), 0);
  for (int32_t refIndex = 0; refIndex < nchr; ++refIndex)
    for (SpanEvent const& e : events[refIndex]) {
      if (e.alt) spanMap[e.id].alt.push_back(e.quality);
      else if (++refAlignedSpanCount[e.id] % 2) spanMap[e.id].ref.push_back(e.quality);
    }
  for (auto const& v : dumpOf) dump->insert(dump->end(), v.begin(), v.end());
  return DGPU_OK;
}

}  // namespace dellyb200
