// shard.hpp — cutting a batch of independent jobs into contiguous per-rank ranges (SURVEY §8e), shared by the sharded stage mirrors; the
// wire format and the all-gather every exchange between ranks goes through, and its in-process form (SimExchange); the contig partition of
// the contig-sharded `delly sr`.
#pragma once
#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/dgpu.h"
#include "types.hpp"

namespace dellyb200 {

// Contiguous ranges of [0, n) with (nearly) equal total cost: bounds[r] .. bounds[r+1] belongs to rank r. Prefix cut at the multiples of
// total / nranks; deterministic, identical on every rank (every rank computes it from the same list).
inline std::vector<std::size_t> partitionByCost(std::vector<uint64_t> const& cost, int nranks) {
  const std::size_t n = cost.size();
  std::vector<std::size_t> bounds((std::size_t) nranks + 1, n);
  bounds[0] = 0;
  uint64_t total = 0;
  for (uint64_t c : cost) total += std::max<uint64_t>(c, 1);
  uint64_t acc = 0;
  std::size_t i = 0;
  for (int r = 1; r < nranks; ++r) {
    const uint64_t target = (uint64_t) (((unsigned __int128) total * (unsigned) r) / (unsigned) nranks);
    while (i < n && acc + std::max<uint64_t>(cost[i], 1) / 2 < target) { acc += std::max<uint64_t>(cost[i], 1); ++i; }
    bounds[r] = i;
  }
  return bounds;
}

// The split-read assembly of one rank (assembleSplitReadsBatch / assembleLRBatch): the queued SVs are cut by cost, the rank builds the
// consensus and aligns it for its range only, `exchange` all-gathers the finished records (mine -> all, in queue order).
struct AssembleShard {
  int rank = 0, nranks = 1;
  std::function<int(std::vector<StructuralVariantRecord> const& mineWork, std::vector<uint8_t> const& mineOk, std::vector<std::size_t> const& bounds,
                    std::vector<StructuralVariantRecord>& allWork, std::vector<uint8_t>& allOk)> exchange;
};

// all-gatherv of one byte string per rank: parts[r] = rank r's payload, same on every rank. Returns DGPU_OK or an error code.
typedef std::function<int(std::string const& local, std::vector<std::string>& parts)> GatherFn;

// The all-gatherv between N ranks that are host threads of one process (`delly_b200 --devices`, the in-process test hooks): every rank
// leaves its payload in its slot, the last one to arrive publishes all slots. fail() releases every rank waiting now or later with
// DGPU_ERR_NCCL, so that one rank's error never leaves the others blocked in an exchange it will not join.
struct SimExchange {
  std::mutex mu; std::condition_variable cv;
  std::vector<std::string> slots; int arrived = 0; long generation = 0; int n;
  bool failed = false;
  explicit SimExchange(int nranks) : slots(nranks), n(nranks) {}
  int gather(int rank, std::string const& local, std::vector<std::string>& parts) {
    std::unique_lock<std::mutex> lk(mu);
    if (failed) return DGPU_ERR_NCCL;
    const long gen = generation;
    slots[rank] = local;
    if (++arrived == n) { published = slots; arrived = 0; ++generation; cv.notify_all(); }
    else cv.wait(lk, [&] { return generation != gen || failed; });
    if (failed) return DGPU_ERR_NCCL;
    parts = published;
    return DGPU_OK;
  }
  void fail() { std::lock_guard<std::mutex> lk(mu); failed = true; cv.notify_all(); }
  GatherFn of(int rank) { return [this, rank](std::string const& local, std::vector<std::string>& parts) { return gather(rank, local, parts); }; }
  std::vector<std::string> published;
};

// ---- wire format (little endian, host order; all ranks are the same binary on the same box) ----------------------------------------
class ByteWriter {
 public:
  std::string buf;
  template <typename T> void pod(T const& v) { buf.append(reinterpret_cast<const char*>(&v), sizeof(T)); }
  void str(std::string const& s) { pod<uint32_t>((uint32_t) s.size()); buf.append(s); }
  void bytes(std::vector<uint8_t> const& v) { pod<uint32_t>((uint32_t) v.size()); if (!v.empty()) buf.append(reinterpret_cast<const char*>(v.data()), v.size()); }
};
class ByteReader {
 public:
  ByteReader(const char* p, std::size_t n) : p_(p), end_(p + n) {}
  bool ok() const { return ok_; }
  bool done() const { return p_ >= end_; }
  template <typename T> T pod() { T v = T(); if (p_ + sizeof(T) > end_) { ok_ = false; return v; } std::memcpy(&v, p_, sizeof(T)); p_ += sizeof(T); return v; }
  std::string str() { const uint32_t n = pod<uint32_t>(); if (!ok_ || p_ + n > end_) { ok_ = false; return std::string(); } std::string s(p_, n); p_ += n; return s; }
  std::vector<uint8_t> bytes() { const uint32_t n = pod<uint32_t>(); if (!ok_ || p_ + n > end_) { ok_ = false; return {}; } std::vector<uint8_t> v(p_, p_ + n); p_ += n; return v; }
 private:
  const char* p_; const char* end_; bool ok_ = true;
};

inline void putSv(ByteWriter& w, StructuralVariantRecord const& v) {
  const int32_t f[20] = {v.chr, v.svStart, v.chr2, v.svEnd, v.ciposlow, v.ciposhigh, v.ciendlow, v.ciendhigh, v.srSupport, v.srMapQuality,
                         v.mapq, v.insLen, v.svt, v.id, v.homLen, v.peSupport, v.peMapQuality, v.consBp, v.alleleid, v.nallele};
  for (int32_t x : f) w.pod(x);
  w.pod(v.srAlignQuality);
  w.pod<uint8_t>(v.precise ? 1 : 0);
  w.pod<uint8_t>(v.anno.isRC ? 1 : 0); w.pod(v.anno.seqType); w.pod(v.anno.homLen); w.pod(v.anno.trPeriod); w.pod(v.anno.trCopies);   // SVAnno (src/tags.h:82-91)
  w.str(v.alleles); w.str(v.consensus);
}
inline void getSv(ByteReader& r, StructuralVariantRecord& v) {
  int32_t f[20];
  for (int32_t& x : f) x = r.pod<int32_t>();
  v.chr = f[0]; v.svStart = f[1]; v.chr2 = f[2]; v.svEnd = f[3]; v.ciposlow = f[4]; v.ciposhigh = f[5]; v.ciendlow = f[6]; v.ciendhigh = f[7]; v.srSupport = f[8];
  v.srMapQuality = f[9]; v.mapq = f[10]; v.insLen = f[11]; v.svt = f[12]; v.id = f[13]; v.homLen = f[14]; v.peSupport = f[15]; v.peMapQuality = f[16]; v.consBp = f[17];
  v.alleleid = f[18]; v.nallele = f[19];
  v.srAlignQuality = r.pod<float>();
  v.precise = r.pod<uint8_t>() != 0;
  v.anno.isRC = r.pod<uint8_t>() != 0; v.anno.seqType = r.pod<int32_t>(); v.anno.homLen = r.pod<int32_t>(); v.anno.trPeriod = r.pod<int32_t>(); v.anno.trCopies = r.pod<float>();
  v.alleles = r.str(); v.consensus = r.str();
}

// ---- contig sharding (`delly_b200 sr --shard-by contig`) --------------------------------------------------------------------------
// The reference walks the contigs one after the other in every stage that reads alignments (scanPEandSR, assembleSplitReads,
// annotateCoverage), and the stage mirrors already split that walk into per-contig logs replayed in contig order. A rank owns a contiguous
// range of contigs, holds only the alignments of those contigs, runs the per-contig part of every stage on them and exchanges the logs;
// everything that depends on the whole genome (junction selection, clustering, mergeSort, sort + renumbering) runs on every rank over the
// same gathered inputs.

// Contiguous contig ranges balanced by weight (mapped reads per contig, summed over the input files): bounds[r] .. bounds[r+1] are rank r's
// contigs. Every rank computes the same cut; with more ranks than contigs some ranges are empty.
inline std::vector<std::size_t> partitionContigs(std::vector<uint64_t> const& weight, int nranks) { return partitionByCost(weight, nranks); }

// The exclude flags of an exclude set (1 = the contig has no valid region: it is excluded as a whole). The scan consults them for the MATE's
// contig (src/shortpe.h:399), which may be any rank's, so a contig-sharded run takes them from the genome-wide lists, before keepOwnContigs.
template <typename TRegions>
std::vector<uint8_t> excludedContigs(TRegions const& valid) {
  std::vector<uint8_t> excluded(valid.size(), 0);
  for (std::size_t t = 0; t < valid.size(); ++t) excluded[t] = valid[t].empty();
  return excluded;
}
// A rank's share of the per-contig region lists (one list of intervals per contig) of a contig-sharded run: the lists of the other ranks'
// contigs are emptied, so the rank reads its own contigs only.
template <typename TRegions>
void keepOwnContigs(std::vector<std::size_t> const& bounds, int rank, TRegions& valid, TRegions& whole) {
  for (std::size_t t = 0; t < valid.size(); ++t)
    if (t < bounds[rank] || t >= bounds[rank + 1]) { valid[t].clear(); whole[t].clear(); }
}

struct ContigShard {
  int rank = 0, nranks = 1;
  std::vector<std::size_t> bounds;   // partitionContigs
  GatherFn gather;
  std::size_t lo() const { return bounds[rank]; }
  std::size_t hi() const { return bounds[rank + 1]; }
  bool owns(int32_t tid) const { return tid >= 0 && (std::size_t) tid >= lo() && (std::size_t) tid < hi(); }
  // the rank whose range holds contig tid (the last rank of an empty range at tid never does)
  int owner(int32_t tid) const {
    for (int r = 0; r < nranks; ++r) if ((std::size_t) tid >= bounds[r] && (std::size_t) tid < bounds[r + 1]) return r;
    return nranks;
  }
  // One all-gather with a status word in front of every payload, so that a rank whose local work failed still takes part in the exchange
  // and every rank leaves it with the same error. parts[r] = rank r's payload without the status word.
  int exchange(int localRc, std::string const& payload, std::vector<std::string>& parts) const {
    std::string msg(sizeof(int32_t), '\0');
    const int32_t st = localRc;
    std::memcpy(&msg[0], &st, sizeof(st));
    if (!localRc) msg += payload;
    std::vector<std::string> raw;
    int rc = gather(msg, raw);
    if (rc) return rc;
    if ((int) raw.size() != nranks) return DGPU_ERR_NCCL;
    parts.assign(raw.size(), std::string());
    for (std::size_t r = 0; r < raw.size(); ++r) {
      if (raw[r].size() < sizeof(int32_t)) return DGPU_ERR_NCCL;
      int32_t s;
      std::memcpy(&s, raw[r].data(), sizeof(s));
      if (s) return s;
      parts[r] = raw[r].substr(sizeof(int32_t));
    }
    return DGPU_OK;
  }
};

// The per-read junction table of the scans (readBp, an unordered_map whose iteration order depends on the order of its insertions) as a log:
// (read id, junction) in insertion order. A contig's log is built on its owner, and replaying the logs in contig order into one table repeats
// the insertions of the sequential walk.
struct JunctionLog {
  std::vector<std::pair<std::size_t, Junction> > ev;
  struct Slot { JunctionLog* log; std::size_t seed; void push_back(Junction const& j) { log->ev.emplace_back(seed, j); } };
  Slot operator[](std::size_t seed) { return Slot{this, seed}; }
};
inline void putJunctionLog(ByteWriter& w, JunctionLog const& log) {
  w.pod<uint64_t>((uint64_t) log.ev.size());
  for (auto const& e : log.ev) {
    Junction const& j = e.second;
    w.pod<uint64_t>((uint64_t) e.first); w.pod<uint8_t>(j.forward); w.pod<uint8_t>(j.scleft); w.pod(j.refidx); w.pod(j.rstart); w.pod(j.refpos); w.pod(j.seqpos); w.pod(j.qual);
  }
}
inline void getJunctionLog(ByteReader& rd, JunctionLog& log) {
  const uint64_t nj = rd.pod<uint64_t>();
  for (uint64_t k = 0; k < nj && rd.ok(); ++k) {
    const std::size_t seed = (std::size_t) rd.pod<uint64_t>();
    const bool fw = rd.pod<uint8_t>() != 0, cl = rd.pod<uint8_t>() != 0;
    const int32_t refidx = rd.pod<int32_t>(), rstart = rd.pod<int32_t>(), refpos = rd.pod<int32_t>(), seqpos = rd.pod<int32_t>();
    const uint16_t qual = rd.pod<uint16_t>();
    log.ev.emplace_back(seed, Junction(fw, cl, refidx, rstart, refpos, seqpos, qual));
  }
}

// The mate tables of inter-chromosomal pairs (scanPEandSR, annotateCoverage): the first observation of a pair (tid < mtid) is put, on the
// contig of the read, into the table of the mate's contig, which is read when that contig is walked. `tables[mtid]` holds this rank's first
// observations; after the exchange the tables of the rank's own contigs hold every rank's, entered in contig order of the reads (rank order),
// so a key seen twice keeps the value the sequential walk leaves.
typedef std::tuple<uint64_t, int32_t, int32_t, int32_t, int32_t> TPairKey;
template <typename A, typename B>
int shareMateTables(ContigShard const& cs, int localRc, std::vector<std::map<TPairKey, std::pair<A, B> > >& tables) {
  ByteWriter w;
  for (std::size_t m = 0; m < tables.size(); ++m) {
    if (tables[m].empty() || cs.owns((int32_t) m)) continue;
    w.pod<uint32_t>((uint32_t) m); w.pod<uint64_t>((uint64_t) tables[m].size());
    for (auto const& kv : tables[m]) {
      w.pod(std::get<0>(kv.first)); w.pod(std::get<1>(kv.first)); w.pod(std::get<2>(kv.first)); w.pod(std::get<3>(kv.first)); w.pod(std::get<4>(kv.first));
      w.pod(kv.second.first); w.pod(kv.second.second);
    }
  }
  std::vector<std::string> parts;
  int rc = cs.exchange(localRc, w.buf, parts);
  if (rc) return rc;
  // a rank's reads come before a later rank's: the entries of lower ranks first, then this rank's own, then higher ranks' (a later
  // assignment to the same key wins, as in the sequential walk)
  std::vector<std::map<TPairKey, std::pair<A, B> > > own(tables.size());
  for (std::size_t m = cs.lo(); m < cs.hi() && m < tables.size(); ++m) own[m].swap(tables[m]);
  for (int r = 0; r < cs.nranks; ++r) {
    if (r == cs.rank) {
      for (std::size_t m = cs.lo(); m < cs.hi() && m < tables.size(); ++m)
        for (auto const& kv : own[m]) tables[m][kv.first] = kv.second;
      continue;
    }
    ByteReader rd(parts[r].data(), parts[r].size());
    while (rd.ok() && !rd.done()) {
      const uint32_t m = rd.pod<uint32_t>();
      const uint64_t n = rd.pod<uint64_t>();
      for (uint64_t k = 0; k < n && rd.ok(); ++k) {
        const uint64_t a = rd.pod<uint64_t>(); const int32_t b = rd.pod<int32_t>(), c = rd.pod<int32_t>(), d = rd.pod<int32_t>(), e = rd.pod<int32_t>();
        const A x = rd.pod<A>(); const B y = rd.pod<B>();
        if (m < tables.size() && cs.owns((int32_t) m)) tables[m][TPairKey(a, b, c, d, e)] = std::make_pair(x, y);
      }
    }
    if (!rd.ok()) return DGPU_ERR_NCCL;
  }
  for (std::size_t m = 0; m < tables.size(); ++m) if (!cs.owns((int32_t) m)) tables[m].clear();
  return DGPU_OK;
}

}  // namespace dellyb200
