// types.hpp — record types and small predicates of Delly's split-read path, field-for-field
// (SURVEY.md §8 a15). Host side of delly-b200; plain C++17, no Boost, no htslib.
//
// Mirrors (names, field order, sort orders, argument meaning):
//   src/tags.h:25-57   _translocation, _getSpanOrientation, Junction (+operator<)
//   src/tags.h:62-80   SRBamRecord (+operator<)
//   src/tags.h:82-130  SVAnno, StructuralVariantRecord (+operator<)
//   src/tags.h:132-172 Breakpoint, _initBreakpoint
//   src/tags.h:174-210 _minCoord/_maxCoord, _svSizeCheck (PE and SR flavours)
//   src/tags.h:277-346 _pairsDisagree
//   src/cluster.h:24-65 BamAlignRecord, EdgeRecord
//   src/split.h:15-25  AlignDescriptor
//   src/align.h:11-25  DnaScore
#pragma once
#include <atomic>
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <functional>
#include <set>
#include <string>
#include <thread>
#include <vector>

namespace dellyb200 {

// Host-side loop over independent items (per-SV folding between device rounds): up to 16 threads (DGPU_HOST_THREADS overrides), the calling
// thread included; fn(i) must only touch item i. The reference runs these loops serially per SV; the results do not depend on the order.
// The budget is the process's; a rank thread of a several-rank process (`delly_b200 --devices`) sets its share of it (rankHostThreads), so
// that the ranks together run no more host threads than one rank alone.
inline unsigned processHostThreads() {
  static const unsigned n = [] {
    const char* e = getenv("DGPU_HOST_THREADS");
    if (e && atoi(e) > 0) return (unsigned) atoi(e);
    const unsigned hw = std::thread::hardware_concurrency();
    return std::max(1u, std::min(hw ? hw : 1u, 16u));
  }();
  return n;
}
inline unsigned& rankHostThreads() { thread_local unsigned n = 0; return n; }   // 0 = the whole process budget
inline unsigned hostThreads() { return rankHostThreads() ? rankHostThreads() : processHostThreads(); }
template <typename F>
inline void parallelFor(std::size_t n, F&& fn, std::size_t minPerThread = 1) {
  const std::size_t nth = std::min<std::size_t>(hostThreads(), std::max<std::size_t>(1, n / std::max<std::size_t>(1, minPerThread)));
  if (nth <= 1) { for (std::size_t i = 0; i < n; ++i) fn(i); return; }
  std::atomic<std::size_t> next(0);
  auto worker = [&]() { for (std::size_t i = next++; i < n; i = next++) fn(i); };
  std::vector<std::thread> pool;
  for (std::size_t t = 1; t < nth; ++t) pool.emplace_back(worker);
  worker();
  for (auto& th : pool) th.join();
}


// Items that exceeded a device limit (include/dgpu.h, "Device limits"). The reference has no such limits; an item beyond one is never
// computed some other way and never aborts the run: it is treated as a FAILED alignment of that one SV / read (the reference's own
// behaviour when an alignment fails: the SV stays imprecise or is dropped), counted here, and the binding reports the counts on stderr.
// One log per process: the ranks of a several-rank process (`delly_b200 --devices`) all count into it, so it holds the sum over the ranks.
struct DeviceLimitLog {
  std::atomic<uint64_t> msaClusters{0};   // dgpu_msa_ex status != 0: > DGPU_MSA_LARGE_MAXR reads, > 1023 alignment columns, a byte outside ACGTN
  std::atomic<uint64_t> pathJobs{0};      // dgpu_edit_path[_wide] status != 0: target slice beyond DGPU_EP_MAX_SLICE columns
  std::atomic<uint64_t> needleJobs{0};    // dgpu_long_needle[_ex]: |cons| > 16383, |ref| > DGPU_LN_MAX_REF, or a workspace beyond the device budget
  uint64_t total() const { return msaClusters.load() + pathJobs.load() + needleJobs.load(); }
};
inline DeviceLimitLog& deviceLimitLog() { static DeviceLimitLog log; return log; }

constexpr int32_t DELLY_SVT_TRANS = 5;

inline bool _translocation(int32_t svt) { return (DELLY_SVT_TRANS <= svt) && (svt < 9); }
inline uint8_t _getSpanOrientation(int32_t svt) { return (uint8_t) (_translocation(svt) ? svt - DELLY_SVT_TRANS : svt); }

struct DnaScore {
  int32_t match = 5, mismatch = -4, go = -10, ge = -1, inf = 1000000;
  DnaScore() {}
  DnaScore(int32_t m, int32_t mm, int32_t o, int32_t e) : match(m), mismatch(mm), go(o), ge(e) {}
};

// The fields of the reference's Config / TeguaConfig that the hot path reads
// (src/delly.h:49-82, :393-398; src/tegua.h:39-74, :230-243).
struct Config {
  DnaScore aliscore;
  uint16_t minCliqueSize = 2;
  uint32_t minRefSep = 25;
  uint32_t maxReadSep = 40;
  uint32_t graphPruning = 1000;
  uint32_t maxGenoReadCount = 250;
  uint32_t maxReadPerSV = 20;  // src/delly.h:224 (lr: 15, src/tegua.h:237)
  uint16_t minMapQual = 1;    // src/delly.h:229 / src/tegua.h:246
  uint16_t minGenoQual = 5;   // src/delly.h:230
  uint16_t minTraQual = 20;   // src/delly.h:218
  uint16_t madCutoff = 9, madNormalCutoff = 5;   // src/delly.h:201,219
  uint32_t minClip = 25;      // src/delly.h:220
  uint32_t maxThreads = 4;    // src/delly.h:212 — only sizes the genotyping batches (131072 x threads jobs, src/coverage.h:271)
  int32_t genoCap = 25;       // long-read per-read genotype quality cap (src/tegua.h:266)
  int32_t nchr = 0;
  int32_t minimumFlankSize = 13;
  int32_t indelsize = 1000;
  int32_t minConsWindow = 100;
  float flankQuality = 0.95f;
  std::set<int32_t> svtset;   // `-t`: SV types to compute (empty = all; src/delly.h:73, src/util.h:370-395)
  bool wantSvt(int32_t svt) const { return svtset.empty() || svtset.count(svt); }
  // contigs without any valid region (exclude file, src/util.h:666-741): pairs whose mate lies on one are skipped (src/shortpe.h:399). Empty: none.
  std::vector<uint8_t> contigExcluded;
  bool mateExcluded(int32_t mtid) const { return !contigExcluded.empty() && mtid >= 0 && (std::size_t) mtid < contigExcluded.size() && contigExcluded[mtid]; }
  static Config shortRead() { return Config(); }
  static Config longRead() {  // src/tegua.h:230-243
    Config c;
    c.minimumFlankSize = 100; c.minConsWindow = 1000; c.flankQuality = 0.9f; c.indelsize = 10000; c.maxReadSep = 500;
    return c;
  }
};

struct Junction {
  bool forward, scleft;
  int32_t refidx, rstart, refpos, seqpos;
  uint16_t qual;
  Junction(bool fw, bool cl, int32_t idx, int32_t rst, int32_t r, int32_t s, uint16_t q)
      : forward(fw), scleft(cl), refidx(idx), rstart(rst), refpos(r), seqpos(s), qual(q) {}
  bool operator<(Junction const& o) const {  // (seqpos, refidx, refpos, scleft)
    if (seqpos != o.seqpos) return seqpos < o.seqpos;
    if (refidx != o.refidx) return refidx < o.refidx;
    if (refpos != o.refpos) return refpos < o.refpos;
    return scleft < o.scleft;
  }
};

struct SRBamRecord {
  int32_t chr, pos, chr2, pos2, rstart, sstart, qual, inslen, svid, primaryChr;
  std::size_t id;
  SRBamRecord(int32_t c, int32_t p, int32_t c2, int32_t p2, int32_t rst, int32_t sst, int32_t q, int32_t il, std::size_t idval)
      : chr(c), pos(p), chr2(c2), pos2(p2), rstart(rst), sstart(sst), qual(q), inslen(il), svid(-1), primaryChr(-1), id(idval) {}
  bool operator<(SRBamRecord const& o) const {  // (chr, pos, chr2, pos2)
    if (chr != o.chr) return chr < o.chr;
    if (pos != o.pos) return pos < o.pos;
    if (chr2 != o.chr2) return chr2 < o.chr2;
    return pos2 < o.pos2;
  }
};

struct SVAnno {
  bool isRC = false;
  int32_t seqType = 0, homLen = 0, trPeriod = 0;
  float trCopies = 0.0f;
};

struct StructuralVariantRecord {
  int32_t chr = 0, svStart = 0, chr2 = 0, svEnd = 0;
  int32_t ciposlow = 0, ciposhigh = 0, ciendlow = 0, ciendhigh = 0;
  int32_t srSupport = 0, srMapQuality = 0, mapq = 0, insLen = 0, svt = -1, id = 0, homLen = 0;
  int32_t peSupport = 0, peMapQuality = 0, consBp = 0, alleleid = -1, nallele = 1;
  float srAlignQuality = 0;
  bool precise = false;
  std::string alleles, consensus;
  SVAnno anno;
  StructuralVariantRecord() {}
  // the SR-cluster constructor (src/tags.h:125): precise defaults to true there
  StructuralVariantRecord(int32_t c1, int32_t s, int32_t c2, int32_t e, int32_t cipl, int32_t ciph, int32_t ciel, int32_t cieh,
                          int32_t sup, int32_t srmapq, int32_t qval, int32_t ilen, int32_t svtype, int32_t idval)
      : chr(c1), svStart(s), chr2(c2), svEnd(e), ciposlow(cipl), ciposhigh(ciph), ciendlow(ciel), ciendhigh(cieh), srSupport(sup),
        srMapQuality(srmapq), mapq(qval), insLen(ilen), svt(svtype), id(idval), precise(true) {}
  bool operator<(StructuralVariantRecord const& o) const {  // (chr, svStart, chr2, svEnd, -peSupport, -srSupport)
    if (chr != o.chr) return chr < o.chr;
    if (svStart != o.svStart) return svStart < o.svStart;
    if (chr2 != o.chr2) return chr2 < o.chr2;
    if (svEnd != o.svEnd) return svEnd < o.svEnd;
    if (peSupport != o.peSupport) return peSupport > o.peSupport;
    return srSupport > o.srSupport;
  }
};

struct Breakpoint {
  int32_t svStartBeg = 0, svStartEnd = 0, svEndBeg = 0, svEndEnd = 0, svStart = 0, svEnd = 0, peSupport = 0, svt = -1, chr = 0, chr2 = 0;
  std::string part1;
  Breakpoint() {}
  explicit Breakpoint(StructuralVariantRecord const& sv)
      : svStartBeg(sv.svStart), svStartEnd(sv.svStart), svEndBeg(sv.svEnd), svEndEnd(sv.svEnd), svStart(sv.svStart), svEnd(sv.svEnd),
        peSupport(sv.peSupport), svt(sv.svt), chr(sv.chr), chr2(sv.chr2) {}
};

// Window around both breakpoints (src/tags.h:151-172). target_len plays the role of hdr->target_len.
inline void _initBreakpoint(std::vector<uint32_t> const& target_len, Breakpoint& bp, int32_t boundary, int32_t svt) {
  bp.svStartBeg = std::max(0, bp.svStart - boundary);
  bp.svEndEnd = std::min((int32_t) target_len[bp.chr2], bp.svEnd + boundary);
  if (_translocation(svt) || svt == 4) {
    bp.svStartEnd = std::min((int32_t) target_len[bp.chr], bp.svStart + boundary);
    bp.svEndBeg = std::max(0, bp.svEnd - boundary);
  } else {
    const int32_t mid = (bp.svStart + bp.svEnd) / 2;
    bp.svStartEnd = std::min(bp.svStart + boundary, mid);
    bp.svEndBeg = std::max(mid + 1, bp.svEnd - boundary);
  }
}

template <typename T> inline T _minCoord(T position, T matePosition, int32_t svt) { return _translocation(svt) ? position : std::min(position, matePosition); }
template <typename T> inline T _maxCoord(T position, T matePosition, int32_t svt) { return _translocation(svt) ? matePosition : std::max(position, matePosition); }

// paired-end size check (src/tags.h:189-198)
inline bool _svSizeCheck(int32_t s, int32_t e, int32_t svt) {
  if (svt >= 0 && svt <= 2) return (e - s) >= 300;
  if (svt == 3) return (e - s) >= 100;
  return true;
}
// split-read size check (src/tags.h:200-210)
inline bool _svSizeCheck(int32_t s, int32_t e, int32_t svt, int32_t inslen) {
  if (svt >= 0 && svt <= 3) return (e - s) >= 15;
  if (svt == 4) return inslen >= 15;
  return true;
}

struct BamAlignRecord {
  int32_t tid, pos, mtid, mpos, alen, malen, Median, Mad, maxNormalISize;
  uint32_t flag;
  uint8_t MapQuality;
  bool operator<(BamAlignRecord const& o) const {  // src/cluster.h:39-49
    if (tid == mtid) {
      const int32_t a = std::min(pos, mpos), b = std::min(o.pos, o.mpos);
      if (a != b) return a < b;
      const int32_t c = std::max(pos, mpos), d = std::max(o.pos, o.mpos);
      if (c != d) return c < d;
      return maxNormalISize < o.maxNormalISize;
    }
    if (pos != o.pos) return pos < o.pos;
    if (mpos != o.mpos) return mpos < o.mpos;
    return maxNormalISize < o.maxNormalISize;
  }
};

struct EdgeRecord {
  uint32_t source, target, weight;
  bool operator<(EdgeRecord const& o) const {  // (weight, source, target)
    if (weight != o.weight) return weight < o.weight;
    if (source != o.source) return source < o.source;
    return target < o.target;
  }
};

struct AlignDescriptor {
  int32_t cStart = 0, cEnd = 0, rStart = 0, rEnd = 0, homLeft = 0, homRight = 0;
  float percId = 0;
};

// Can two abnormal pairs support the same SV? (src/tags.h:277-346). The per-type rules differ only in
// which pair's insert-size bound limits which offset; the table below encodes that choice.
inline bool _pairsDisagree(int32_t p1Min, int32_t p1Max, int32_t p1Len, int32_t p1ISize, int32_t p2Min, int32_t p2Max, int32_t p2Len,
                           int32_t p2ISize, int32_t svt) {
  // bound on the left offset, on the right offset when pair2 ends first, and when pair1 ends first
  int32_t bLeft, bRightP2First, bRightP1First;
  bool needOverlap = false;
  if (_translocation(svt)) {
    const uint8_t ct = _getSpanOrientation(svt);
    const bool even = (ct % 2 == 0), hi = (ct >= 2);
    bLeft = even ? p1ISize : p2ISize;
    // even&&hi: (p1,p2) ; even&&!hi: (p2,p1) ; odd&&hi: (p2,p1) ; odd&&!hi: (p1,p2)
    const bool p1first = (even == hi);
    bRightP2First = p1first ? p1ISize : p2ISize;
    bRightP1First = p1first ? p2ISize : p1ISize;
  } else if (svt == 0) { bLeft = p1ISize; bRightP2First = p2ISize; bRightP1First = p1ISize; }
  else if (svt == 1) { bLeft = p2ISize; bRightP2First = p1ISize; bRightP1First = p2ISize; }
  else if (svt == 2) { bLeft = p1ISize; bRightP2First = p1ISize; bRightP1First = p2ISize; needOverlap = true; }
  else if (svt == 3) { bLeft = p2ISize; bRightP2First = p2ISize; bRightP1First = p1ISize; }
  else return false;
  if ((p2Min + p2Len - p1Min) > bLeft) return true;
  if (p2Max < p1Max) { if ((p1Max + p1Len - p2Max) > bRightP2First) return true; }
  else { if ((p2Max + p2Len - p1Max) > bRightP1First) return true; }
  if (needOverlap && ((p1Max < p2Min) || (p2Max < p1Min))) return true;
  return false;
}

}  // namespace dellyb200
