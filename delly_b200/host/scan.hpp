// scan.hpp — the discovery front end of `delly sr` (scanPEandSR, src/shortpe.h:285-533) over an in-memory record list:
// per record the CIGAR junction scan and the abnormal-pair bookkeeping, then junction selection, split-read and paired-end
// clustering and the split-read store that assembleSplitReads consumes. Host logic throughout (the only heavy part, the
// windowed pair scans inside cluster(), can run on the device: pass a context).
#pragma once
#include <algorithm>
#include <map>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "assemble.hpp"
#include "cluster.hpp"
#include "genotype.hpp"
#include "junction.hpp"

namespace dellyb200 {

// recs sorted like a coordinate-sorted BAM (tid, pos). svs receives the paired-end SVs, srSVs the split-read SVs, srStore[tid]
// the (read start, read id) -> SV id entries of the assigned split reads. lib.abnormal_pairs counts the pairs kept (:446).
// ctx != nullptr: the pair scans of both cluster() flavours run on the device (clusterGpu); results are identical.
//
// Containers follow the reference where their iteration order reaches the output: junctions per read live in an unordered
// map keyed by the read id (the select* functions iterate it; the reference uses boost::unordered_map, the oracle build and
// this code std::unordered_map — SURVEY section 0: parity is defined against one build).
// One reference quirk is kept: the "same start position" tie-break of pairs (_firstPairObs, src/tags.h:269-274) looks up
// hash_string(qname) in a set that scanPEandSR fills with hash_sr ids (:409), so it only fires on a hash coincidence.
// The per-file half of scanPEandSR (:318-463): junction scan and abnormal-pair bookkeeping of ONE sample, junction selection; the
// sample's split-read and paired-end records are appended to srBR / bamRecord (the reference concatenates the files in order, :468-477).
// cs != nullptr (contig sharding): recs holds this rank's contigs only; the inter-chromosomal first observations go to the rank of the mate's
// contig before the contig logs are built, and the logs of all ranks are gathered and replayed in contig order on every rank.
inline int scanSamplePEandSR(Config const& c, LibraryInfo& lib, std::vector<uint32_t> const& target_len, std::vector<SrRecord> const& recs, TSvtSRBamRecord& srBRAll,
                             std::vector<std::vector<BamAlignRecord> >& bamRecord, ContigShard const* cs = nullptr) {
  typedef std::map<TPairKey, std::pair<uint8_t, int32_t> > TMateMap;
  std::unordered_map<std::size_t, TJunctionVector> readBp;
  TSvtSRBamRecord srBR(2 * DELLY_SVT_TRANS);
  auto alignmentLength = [](SrRecord const& r) {  // src/util.h:440-447
    uint32_t alen = 0;
    for (auto const& cg : r.cigar) if (cg.first == 0 || cg.first == 7 || cg.first == 8 || cg.first == 2 || cg.first == 3) alen += cg.second;
    return alen;
  };
  // The reference walks the contigs one after the other. A contig's records are independent of the other contigs' except for (1) the order in
  // which junctions enter the per-read table (its iteration order reaches the output), (2) the order of the pair records per SV type and (3) the
  // mate table of inter-chromosomal pairs (filled on the contig with the smaller index, read and erased on the mate's). So the contigs are scanned
  // in parallel into per-contig logs — junction insertions and pair records in record order — with the inter-chromosomal first observations
  // collected beforehand (one cheap sequential pass, the table split by the contig that reads it), and the logs are replayed in contig order.
  const int32_t nchr = (int32_t) target_len.size();
  std::vector<std::size_t> lo((std::size_t) nchr + 1, recs.size());
  {
    std::size_t ri = 0;
    for (int32_t refIndex = 0; refIndex < nchr; ++refIndex) {
      lo[refIndex] = ri;
      while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;
    }
    lo[nchr] = ri;
  }
  // what a record must pass before the pair bookkeeping looks at it (:392-407); returns the SV type or -1
  auto pairType = [&](SrRecord const& rec) -> int32_t {
    if (!(rec.flag & 0x1)) return -1;                                 // BAM_FPAIRED
    if (lib.median == 0) return -1;
    if (rec.flag & (BAMF_SECONDARY | BAMF_SUPPLEMENTARY)) return -1;
    if ((rec.mtid < 0) || (rec.flag & BAMF_MUNMAP)) return -1;
    if (c.mateExcluded(rec.mtid)) return -1;                          // :399
    if ((rec.tid != rec.mtid) && (rec.mapq < c.minTraQual)) return -1;
    const int32_t svt = _isizeMappingPos(rec, lib.maxISizeCutoff);
    if (svt == -1) return -1;
    if (!c.wantSvt(svt)) return -1;   // :405
    if ((svt == 2) && (lib.maxISizeCutoff > std::abs(rec.isize))) return -1;
    return svt;
  };
  std::vector<TMateMap> matetraOf((std::size_t) nchr);
  for (int32_t refIndex = 0; refIndex < nchr; ++refIndex)
    for (std::size_t q = lo[refIndex]; q < lo[refIndex + 1]; ++q) {
      SrRecord const& rec = recs[q];
      if (rec.tid >= rec.mtid || rec.mtid >= nchr) continue;          // first observation of an inter-chromosomal pair: tid < mtid
      if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP)) continue;
      if (rec.mapq < c.minMapQual) continue;
      if (pairType(rec) < 0) continue;
      matetraOf[rec.mtid][TPairKey(rec.name, rec.tid, rec.pos, rec.mtid, rec.mpos)] = std::make_pair(rec.mapq, (int32_t) alignmentLength(rec));
    }
  int rc = DGPU_OK;
  if (cs && (rc = shareMateTables(*cs, DGPU_OK, matetraOf))) return rc;
  struct ContigLog { JunctionLog junctions; std::vector<std::pair<int32_t, BamAlignRecord> > pairs; };
  std::vector<ContigLog> logs((std::size_t) nchr);
  parallelFor((std::size_t) nchr, [&](std::size_t refIndexU) {
    const int32_t refIndex = (int32_t) refIndexU;
    if (cs && !cs->owns(refIndex)) return;
    ContigLog& log = logs[refIndexU];
    TMateMap mateMap;
    TMateMap& matetra = matetraOf[refIndexU];
    int32_t lastAlignedPos = 0;
    std::unordered_set<std::size_t> lastAlignedPosReads;
    for (std::size_t q = lo[refIndex]; q < lo[refIndex + 1]; ++q) {
      SrRecord const& rec = recs[q];
      if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP)) continue;
      if (rec.mapq < c.minMapQual) continue;
      const std::size_t seed = srSeed(rec);
      cigarJunctions(log.junctions, seed, rec.flag, rec.tid, rec.pos, rec.mapq, rec.cigar, c.minClip, c.minRefSep);   // :360-389
      const int32_t svt = pairType(rec);
      if (svt < 0) continue;
      if (rec.pos > lastAlignedPos) { lastAlignedPosReads.clear(); lastAlignedPos = rec.pos; }
      const bool firstObs = (rec.tid == rec.mtid)
                                ? ((rec.pos < rec.mpos) || ((rec.pos == rec.mpos) && !lastAlignedPosReads.count((std::size_t) rec.nameHash32)))
                                : (rec.tid < rec.mtid);
      if (firstObs) {
        lastAlignedPosReads.insert(seed);
        if (!_translocation(svt)) mateMap[TPairKey(rec.name, rec.tid, rec.pos, rec.mtid, rec.mpos)] = std::make_pair(rec.mapq, (int32_t) alignmentLength(rec));
        // (inter-chromosomal first observations are already in the table of the mate's contig)
      } else {
        const TPairKey hv(rec.name, rec.mtid, rec.mpos, rec.tid, rec.pos);
        TMateMap& tab = _translocation(svt) ? matetra : mateMap;
        auto itMM = tab.find(hv);
        if ((itMM == tab.end()) || (!(itMM->second.first))) continue;  // mate discarded (or its quality was 0)
        const uint8_t pairQuality = std::min((uint8_t) itMM->second.first, rec.mapq);
        const int32_t alenmate = itMM->second.second;
        tab.erase(itMM);
        BamAlignRecord b;  // src/cluster.h:36: the two alignment lengths pass through uint16_t parameters
        b.tid = rec.tid; b.pos = rec.pos; b.mtid = rec.mtid; b.mpos = rec.mpos; b.alen = (uint16_t) alignmentLength(rec); b.malen = (uint16_t) alenmate;
        b.Median = lib.median; b.Mad = lib.mad; b.maxNormalISize = lib.maxNormalISize; b.flag = rec.flag; b.MapQuality = pairQuality;
        log.pairs.emplace_back(svt, b);
      }
    }
  });
  if (cs) {   // the logs of the other ranks' contigs
    ByteWriter w;
    for (std::size_t refIndex = cs->lo(); refIndex < cs->hi(); ++refIndex) {
      ContigLog const& log = logs[refIndex];
      putJunctionLog(w, log.junctions);
      w.pod<uint64_t>((uint64_t) log.pairs.size());
      for (auto const& pr : log.pairs) { w.pod(pr.first); w.pod(pr.second); }
    }
    std::vector<std::string> parts;
    if ((rc = cs->exchange(DGPU_OK, w.buf, parts))) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      if (r == cs->rank) continue;
      ByteReader rd(parts[r].data(), parts[r].size());
      for (std::size_t refIndex = cs->bounds[r]; refIndex < cs->bounds[r + 1]; ++refIndex) {
        ContigLog& log = logs[refIndex];
        getJunctionLog(rd, log.junctions);
        const uint64_t np = rd.pod<uint64_t>();
        for (uint64_t k = 0; k < np && rd.ok(); ++k) { const int32_t svt = rd.pod<int32_t>(); log.pairs.emplace_back(svt, rd.pod<BamAlignRecord>()); }
      }
      if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
    }
  }
  for (int32_t refIndex = 0; refIndex < nchr; ++refIndex) {
    for (auto const& e : logs[refIndex].junctions.ev) readBp[e.first].push_back(e.second);
    for (auto const& pr : logs[refIndex].pairs) { bamRecord[pr.first].push_back(pr.second); ++lib.abnormal_pairs; }
  }
  for (auto& kv : readBp) std::sort(kv.second.begin(), kv.second.end());
  if (c.wantSvt(2)) selectDeletions(c, readBp, srBR);   // :457-461 (no insertion bridging in the short-read path)
  if (c.wantSvt(3)) selectDuplications(c, readBp, srBR);
  if (c.svtset.empty() || c.svtset.count(0) || c.svtset.count(1)) selectInversions(c, readBp, srBR);
  if (c.wantSvt(4)) selectInsertions(c, readBp, srBR);
  if (c.svtset.empty() || c.svtset.count(5) || c.svtset.count(6) || c.svtset.count(7) || c.svtset.count(8)) selectTranslocations(c, readBp, srBR);
  for (std::size_t svt = 0; svt < srBR.size(); ++svt) srBRAll[svt].insert(srBRAll[svt].end(), srBR[svt].begin(), srBR[svt].end());
  return DGPU_OK;
}

// The joint half (:479-527): per SV type sort + cluster of the pooled records, and the read store assembleSplitReads consumes.
// varisize = getVariability over all libraries (src/util.h:759-768).
inline int clusterScannedPEandSR(dgpu_ctx* ctx, Config const& c, int32_t varisize, std::vector<uint32_t> const& target_len, TSvtSRBamRecord& srBR,
                                 std::vector<std::vector<BamAlignRecord> >& bamRecord, std::vector<StructuralVariantRecord>& svs,
                                 std::vector<StructuralVariantRecord>& srSVs, std::vector<TPosReadSV>& srStore) {
  int rc;
  for (uint32_t svt = 0; svt < srBR.size(); ++svt) {
    if (!c.wantSvt((int32_t) svt)) continue;   // :486
    if (srBR[svt].empty()) continue;
    std::sort(srBR[svt].begin(), srBR[svt].end());
    if (ctx) { if ((rc = clusterGpu(ctx, c, srBR[svt], srSVs, (int32_t) svt))) return rc; }
    else cluster(c, srBR[svt], srSVs, (int32_t) svt);
  }
  for (int32_t svt = 0; svt < (int32_t) bamRecord.size(); ++svt) {
    if (!c.wantSvt(svt)) continue;   // :503
    if (bamRecord[svt].empty()) continue;
    std::sort(bamRecord[svt].begin(), bamRecord[svt].end());
    if (ctx) { if ((rc = clusterGpu(ctx, c, bamRecord[svt], svs, (uint32_t) varisize, svt))) return rc; }
    else cluster(c, bamRecord[svt], svs, (uint32_t) varisize, svt);
  }
  srStore.assign(target_len.size(), TPosReadSV());
  for (auto const& v : srBR)
    for (SRBamRecord const& r : v) {
      if ((r.svid == -1) || (r.rstart == -1)) continue;
      if (r.rstart < (int32_t) target_len[r.chr]) srStore[r.chr].insert(std::make_pair(std::make_pair(r.rstart, r.id), r.svid));
      if ((r.chr != r.chr2) && (r.rstart < (int32_t) target_len[r.chr2])) srStore[r.chr2].insert(std::make_pair(std::make_pair(r.rstart, r.id), r.svid));
    }
  return DGPU_OK;
}

// scanPEandSR over the samples of a call set (libs[f] belongs to samples[f]).
// cs: contig sharding (scanSamplePEandSR); the pooled records and the clustering are then the same on every rank.
inline int scanPEandSRBatch(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo>& libs, std::vector<uint32_t> const& target_len,
                            std::vector<std::vector<SrRecord> const*> const& samples, std::vector<StructuralVariantRecord>& svs,
                            std::vector<StructuralVariantRecord>& srSVs, std::vector<TPosReadSV>& srStore, ContigShard const* cs = nullptr) {
  TSvtSRBamRecord srBR(2 * DELLY_SVT_TRANS);
  std::vector<std::vector<BamAlignRecord> > bamRecord(2 * DELLY_SVT_TRANS);
  int32_t varisize = 0;
  for (std::size_t f = 0; f < samples.size(); ++f) {
    const int rc = scanSamplePEandSR(c, libs[f], target_len, *samples[f], srBR, bamRecord, cs);
    if (rc) return rc;
    varisize = std::max(varisize, std::max(libs[f].maxNormalISize, libs[f].rs));
  }
  const int rc = clusterScannedPEandSR(ctx, c, varisize, target_len, srBR, bamRecord, svs, srSVs, srStore);
  if (rc && cs) {   // a device failure of this rank alone: the next exchange of the other ranks (the assembly's) carries it to them
    std::vector<std::string> parts;
    cs->exchange(rc, std::string(), parts);
  }
  return rc;
}

inline int scanPEandSRBatch(dgpu_ctx* ctx, Config const& c, LibraryInfo& lib, std::vector<uint32_t> const& target_len, std::vector<SrRecord> const& recs,
                            std::vector<StructuralVariantRecord>& svs, std::vector<StructuralVariantRecord>& srSVs, std::vector<TPosReadSV>& srStore) {
  std::vector<LibraryInfo> libs(1, lib);
  const int rc = scanPEandSRBatch(ctx, c, libs, target_len, std::vector<std::vector<SrRecord> const*>(1, &recs), svs, srSVs, srStore);
  lib = libs[0];
  return rc;
}


// mergeSort (src/shortpe.h:536-621): paired-end SVs are refined by a matching split-read SV (same type and contigs, both
// breakpoints inside the paired-end confidence intervals); split-read SVs without a paired-end partner are appended unless a
// better-supported precise duplicate exists within 10 bp. The repeated sort of `pe` after every append is the reference's.
inline void mergeSort(std::vector<StructuralVariantRecord>& pe, std::vector<StructuralVariantRecord>& sr) {
  std::sort(pe.begin(), pe.end());
  std::sort(sr.begin(), sr.end());
  for (int32_t svt = 0; svt < 10; ++svt) {
    for (int32_t i = 0; i < (int32_t) sr.size(); ++i) {
      if (sr[i].svt != svt) continue;
      if ((sr[i].srSupport == 0) || (sr[i].srAlignQuality == 0)) continue;
      const int32_t searchWindow = 500;
      bool svExists = false;
      StructuralVariantRecord key;   // the (chr, svStart, svEnd) look-up record (src/tags.h:122): chr2 = chr, supports 0
      key.chr = sr[i].chr; key.svStart = std::max(0, sr[i].svStart - searchWindow); key.chr2 = sr[i].chr; key.svEnd = sr[i].svEnd;
      key.peSupport = 0; key.srSupport = 0;
      auto itOther = std::lower_bound(pe.begin(), pe.end(), key);
      for (; (itOther != pe.end()) && (std::abs(itOther->svStart - sr[i].svStart) < searchWindow); ++itOther) {
        if ((itOther->svt != svt) || (itOther->precise)) continue;
        if ((sr[i].chr != itOther->chr) || (sr[i].chr2 != itOther->chr2)) continue;
        if ((itOther->svStart + itOther->ciposlow < sr[i].svStart) && (sr[i].svStart < itOther->svStart + itOther->ciposhigh) &&
            (itOther->svEnd + itOther->ciendlow < sr[i].svEnd) && (sr[i].svEnd < itOther->svEnd + itOther->ciendhigh)) {
          svExists = true;
          itOther->svStart = sr[i].svStart; itOther->svEnd = sr[i].svEnd;
          itOther->ciposlow = sr[i].ciposlow; itOther->ciposhigh = sr[i].ciposhigh; itOther->ciendlow = sr[i].ciendlow; itOther->ciendhigh = sr[i].ciendhigh;
          itOther->srMapQuality = sr[i].srMapQuality; itOther->srSupport = sr[i].srSupport; itOther->insLen = sr[i].insLen; itOther->homLen = sr[i].homLen;
          itOther->srAlignQuality = sr[i].srAlignQuality; itOther->precise = true; itOther->consensus = sr[i].consensus; itOther->consBp = sr[i].consBp;
          itOther->mapq += sr[i].mapq;
        }
      }
      if (svExists) continue;
      const int32_t precSearchWindow = 10;
      bool preciseDuplicate = false;
      auto better = [&](int32_t j) { return (sr[i].srSupport < sr[j].srSupport) || ((i < j) && (sr[i].srSupport == sr[j].srSupport)); };
      for (int32_t j = i + 1; j < (int32_t) sr.size(); ++j) {
        if (std::abs(sr[i].svStart - sr[j].svStart) > precSearchWindow) break;
        if (sr[i].svt != sr[j].svt) continue;
        if ((sr[i].chr != sr[j].chr) || (sr[i].chr2 != sr[j].chr2)) continue;
        if ((sr[j].svStart + sr[j].ciposlow <= sr[i].svStart) && (sr[i].svStart <= sr[j].svStart + sr[j].ciposhigh) &&
            (sr[j].svEnd + sr[j].ciendlow <= sr[i].svEnd) && (sr[i].svEnd <= sr[j].svEnd + sr[j].ciendhigh) && better(j))
          preciseDuplicate = true;
      }
      for (int32_t j = i - 1; j >= 0; --j) {
        if (std::abs(sr[i].svStart - sr[j].svStart) > precSearchWindow) break;
        if (sr[i].svt != sr[j].svt) continue;
        if ((sr[i].chr != sr[j].chr) || (sr[i].chr2 != sr[j].chr2)) continue;
        if ((sr[j].svStart + sr[j].ciposlow < sr[i].svStart) && (sr[i].svStart < sr[j].svStart + sr[j].ciposhigh) &&
            (sr[j].svEnd + sr[j].ciendlow < sr[i].svEnd) && (sr[i].svEnd < sr[j].svEnd + sr[j].ciendhigh) && better(j))
          preciseDuplicate = true;
      }
      if (!preciseDuplicate) {
        pe.push_back(sr[i]);
        std::sort(pe.begin(), pe.end());
      }
    }
  }
}


// getLibraryParams (src/util.h:771-891) for one sample: read length (median of l_qseq) and insert-size median / MAD of the first
// up to 10^6 read-1 alignments (primary, mapped, not duplicate / QC-fail), the normal-pair window and the deletion cut-off
// derived from them. A library whose pairs are mostly not in FR orientation keeps median = 0 (the reference warns and treats
// it as single-end). recs sorted like a coordinate-sorted BAM.
// The screen is a state (LibraryScreen) so that it can be continued: a contig-sharded run (getLibraryParamsSharded) continues it rank after
// rank, where the ranks of the lower contigs left it. The screened values are kept as histograms (value -> count): the medians are order
// statistics, which a histogram gives exactly, and a histogram of insert sizes is a few kB where the values are millions.
struct LibraryScreen {
  uint32_t alignmentCount = 0, processedNumPairs = 0, processedNumReads = 0, rplus = 0, nonrplus = 0;
  bool characterized = false;
  std::unordered_map<uint32_t, uint32_t> readSize, isize;
};
inline void continueLibraryScreen(std::vector<uint32_t> const& target_len, std::vector<SrRecord> const& recs, LibraryScreen& s) {
  const uint32_t maxAlignmentsScreened = 10000000, maxNumAlignments = 1000000;
  std::size_t ri = 0;
  for (int32_t refIndex = 0; (refIndex < (int32_t) target_len.size()) && !s.characterized; ++refIndex) {
    const std::size_t rlo = ri;
    while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;
    for (std::size_t q = rlo; q < ri; ++q) {
      SrRecord const& rec = recs[q];
      if ((rec.flag & 0x80) || !(rec.lqseq < 65000)) continue;
      if (rec.flag & (BAMF_SECONDARY | BAMF_QCFAIL | BAMF_DUP | BAMF_SUPPLEMENTARY | BAMF_UNMAP)) continue;
      if ((s.alignmentCount > maxAlignmentsScreened) || ((s.processedNumReads >= maxNumAlignments) && (s.processedNumPairs == 0)) ||
          (s.processedNumPairs >= maxNumAlignments)) {
        s.characterized = true;
        break;
      }
      ++s.alignmentCount;
      if (s.processedNumReads < maxNumAlignments) { ++s.readSize[(uint32_t) rec.lqseq]; ++s.processedNumReads; }
      if ((rec.flag & 0x1) && !(rec.flag & BAMF_MUNMAP) && (rec.tid == rec.mtid) && (s.processedNumPairs < maxNumAlignments)) {
        ++s.isize[(uint32_t) std::abs(rec.isize)];
        if (getSVType(rec) == 2) ++s.rplus; else ++s.nonrplus;
        ++s.processedNumPairs;
      }
    }
  }
}
inline void libraryFromScreen(Config const& c, LibraryScreen const& s, LibraryInfo& lib) {
  const uint32_t minNumAlignments = 1000;
  lib = LibraryInfo();
  auto kth = [](std::unordered_map<uint32_t, uint32_t> const& h, uint64_t k) {   // the element a full sort would put at index k
    std::vector<std::pair<uint32_t, uint32_t> > v(h.begin(), h.end());
    std::sort(v.begin(), v.end());
    for (auto const& kv : v) { if (k < kv.second) return kv.first; k -= kv.second; }
    return 0u;
  };
  if (s.processedNumReads >= minNumAlignments) lib.rs = (int32_t) kth(s.readSize, s.processedNumReads / 2);
  if (s.processedNumPairs >= minNumAlignments) {
    const int32_t median = (int32_t) kth(s.isize, s.processedNumPairs / 2);
    std::unordered_map<uint32_t, uint32_t> absDev;
    for (auto const& kv : s.isize) absDev[(uint32_t) std::abs((int32_t) kv.first - median)] += kv.second;
    const int32_t mad = (int32_t) kth(absDev, s.processedNumPairs / 2);
    if ((median >= 50) && (median <= 100000) && !(s.rplus < s.nonrplus)) {
      lib.median = median; lib.mad = mad;
      lib.maxNormalISize = median + (c.madNormalCutoff * mad);
      lib.minNormalISize = std::max(median - (c.madNormalCutoff * mad), 0);
      lib.maxISizeCutoff = median + (c.madCutoff * mad);
      lib.minISizeCutoff = median - (c.madCutoff * mad);
      lib.maxISizeCutoff = std::max(lib.maxISizeCutoff, 2 * lib.rs);
      lib.maxISizeCutoff = std::max(lib.maxISizeCutoff, 500);
      if (lib.minISizeCutoff < 0) lib.minISizeCutoff = 0;
    }
  }
}
inline void getLibraryParams(Config const& c, std::vector<uint32_t> const& target_len, std::vector<SrRecord> const& recs, LibraryInfo& lib) {
  LibraryScreen s;
  continueLibraryScreen(target_len, recs, s);
  libraryFromScreen(c, s, lib);
}

// the screen over a contig-sharded genome: rank r continues it (over its own contigs) from the state rank r - 1 left, until the library is
// characterized — usually inside the first rank's contigs: one exchange
inline int getLibraryParamsSharded(Config const& c, std::vector<uint32_t> const& target_len, std::vector<SrRecord> const& recs, ContigShard const& cs,
                                   LibraryInfo& lib) {
  LibraryScreen s;
  for (int r = 0; r < cs.nranks && !s.characterized; ++r) {
    ByteWriter w;
    if (r == cs.rank) {
      continueLibraryScreen(target_len, recs, s);
      const uint32_t f[5] = {s.alignmentCount, s.processedNumPairs, s.processedNumReads, s.rplus, s.nonrplus};
      for (uint32_t x : f) w.pod(x);
      w.pod<uint8_t>(s.characterized);
      for (auto const* h : {&s.readSize, &s.isize}) {
        w.pod<uint64_t>((uint64_t) h->size());
        for (auto const& kv : *h) { w.pod(kv.first); w.pod(kv.second); }
      }
    }
    std::vector<std::string> parts;
    const int rc = cs.exchange(DGPU_OK, w.buf, parts);
    if (rc) return rc;
    ByteReader rd(parts[r].data(), parts[r].size());
    s.alignmentCount = rd.pod<uint32_t>(); s.processedNumPairs = rd.pod<uint32_t>(); s.processedNumReads = rd.pod<uint32_t>(); s.rplus = rd.pod<uint32_t>();
    s.nonrplus = rd.pod<uint32_t>();
    s.characterized = rd.pod<uint8_t>() != 0;
    for (auto* h : {&s.readSize, &s.isize}) {
      h->clear();
      const uint64_t n = rd.pod<uint64_t>();
      for (uint64_t k = 0; k < n && rd.ok(); ++k) { const uint32_t v = rd.pod<uint32_t>(); (*h)[v] = rd.pod<uint32_t>(); }
    }
    if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
  }
  libraryFromScreen(c, s, lib);
  return DGPU_OK;
}

}  // namespace dellyb200
