// assemble.hpp — the split-read assembly stage of `delly sr` (assembleSplitReads, src/shortpe.h:48-282), batched:
// the reference collects the split reads of every SV from the BAM, then runs msa() + alignConsensus() per SV on its thread pool
// (:172-201, :246-271). Here the collection is the same host code over an in-memory record list, and ALL SVs go through
// ONE msaBatch (one dgpu_msa) and ONE alignConsensusBatch (one dgpu_long_needle + the splitAlign rounds for insertions).
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <unordered_set>
#include <vector>

#include "genotype.hpp"
#include "msa.hpp"
#include "shard.hpp"
#include "split.hpp"
#include "splitalign.hpp"

namespace dellyb200 {

typedef std::map<std::pair<int32_t, std::size_t>, int32_t> TPosReadSV;  // (position, read id) -> SV id, per contig (src/shortpe.h:462-476)

// read id as the reference derives it (hash_sr, src/util.h:519-527: read 2 of a pair = read 1 + 1)
// (a caller that already has the reference's id passes it in SrRecord::seed)
inline std::size_t srSeed(SrRecord const& r) { return r.seed ? r.seed : (std::size_t) r.name * 2 + ((r.flag & 0x80) ? 1 : 0); }

// samples: the alignment lists of all input files, in file order (the reference walks contig by contig and, inside a contig, file by
// file: src/shortpe.h:81-156), each sorted like a coordinate-sorted BAM.
// cs != nullptr (contig sharding): samples hold this rank's contigs only and an SV belongs to the rank of sv.chr. The split reads a rank
// collects for a translocation on its contigs are gathered by every rank and replayed in contig order into the owner's read set, so msa sees
// the set of the single-process walk; the owner assembles its SVs and the finished records of all ranks are gathered.
inline int assembleSplitReadsBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<const char*> const& chrseq,
                                   std::vector<TPosReadSV> const& srStore, std::vector<StructuralVariantRecord>& svs,
                                   std::vector<std::vector<SrRecord> const*> const& samples, AssembleShard const* shard = nullptr,
                                   ContigShard const* cs = nullptr) {
  // The reference keeps the reads of an SV in a std::unordered_set<std::string>; its iteration order is the order msa() sees
  // (and it de-duplicates identical reads). The same container with the same insertion sequence gives the same order.
  typedef std::unordered_set<std::string> TSequences;
  const std::size_t N = svs.size();
  std::vector<TSequences> traStore(N);
  std::vector<std::vector<uint8_t> > traQualStore(N);
  std::vector<std::vector<std::string> > traOrder(cs ? N : 0);   // contig sharding: the translocation reads in insertion order
  std::vector<uint32_t> queued;                          // SV ids that reach msa + alignConsensus
  std::vector<std::vector<std::string> > clusters;       // their reads, in the set's iteration order
  std::vector<std::vector<uint8_t> > quals;
  auto reset = [&](StructuralVariantRecord& sv) { sv.consensus = ""; sv.srSupport = 0; sv.srAlignQuality = 0; };
  std::vector<std::size_t> ri(samples.size(), 0), rlo(samples.size(), 0);
  for (int32_t refIndex = 0; refIndex < (int32_t) target_len.size(); ++refIndex) {
    for (std::size_t f = 0; f < samples.size(); ++f) {
      std::vector<SrRecord> const& recs = *samples[f];
      rlo[f] = ri[f];
      while (ri[f] < recs.size() && recs[ri[f]].tid == refIndex) ++ri[f];
    }
    if (srStore[refIndex].empty() || (cs && !cs->owns(refIndex))) continue;
    std::vector<bool> hits(target_len[refIndex], false);
    for (auto const& kv : srStore[refIndex]) hits[(std::size_t) kv.first.first] = true;
    std::vector<TSequences> seqStore(N);
    std::vector<std::vector<uint8_t> > qualStore(N);
    for (std::size_t f = 0; f < samples.size(); ++f)
    for (std::size_t q = rlo[f]; q < ri[f]; ++q) {
      SrRecord const& rec = (*samples[f])[q];
      if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP | BAMF_SECONDARY | BAMF_SUPPLEMENTARY)) continue;
      if (rec.mapq < c.minMapQual) continue;
      if (!hits[(std::size_t) rec.pos]) continue;
      auto it = srStore[refIndex].find(std::make_pair(rec.pos, srSeed(rec)));
      if (it == srStore[refIndex].end()) continue;
      const int32_t svid = it->second;
      StructuralVariantRecord const& sv = svs[svid];
      if (svid != sv.id) continue;
      std::string sequence = rec.seq;
      bool bpPoint = false;   // :115-131
      if (_translocation(sv.svt)) { if (rec.tid == sv.chr2) bpPoint = true; }
      else if (sv.svt == 0) bpPoint = (rec.pos + 25 > sv.svStart);
      else if (sv.svt == 1) bpPoint = (rec.pos + 25 > sv.svEnd);
      _adjustOrientation(sequence, bpPoint ? 1u : 0u, sv.svt);
      if (seqStore[svid].size() < c.maxReadPerSV) {   // (the cap looks at seqStore for translocations too, :140)
        if (_translocation(sv.svt)) {
          if (cs) { if (traStore[svid].insert(sequence).second) { traQualStore[svid].push_back(rec.mapq); traOrder[svid].push_back(std::move(sequence)); } }
          else if (traStore[svid].insert(std::move(sequence)).second) traQualStore[svid].push_back(rec.mapq);
        }
        else { if (seqStore[svid].insert(std::move(sequence)).second) qualStore[svid].push_back(rec.mapq); }
      }
    }
    for (uint32_t svid = 0; svid < N; ++svid) {
      if (_translocation(svs[svid].svt)) continue;
      if (svs[svid].chr != refIndex) continue;
      if (seqStore[svid].size() <= 1) { reset(svs[svid]); continue; }
      queued.push_back(svid);
      clusters.push_back(std::vector<std::string>(seqStore[svid].begin(), seqStore[svid].end()));
      quals.push_back(qualStore[svid]);
    }
  }
  int rc = DGPU_OK;
  if (cs) {   // every rank's translocation reads, replayed in rank (= contig) order into the read sets of this rank's translocations
    ByteWriter w;
    for (uint32_t svid = 0; svid < N; ++svid) {
      if (traOrder[svid].empty()) continue;
      w.pod(svid); w.pod<uint32_t>((uint32_t) traOrder[svid].size());
      for (std::size_t k = 0; k < traOrder[svid].size(); ++k) { w.str(traOrder[svid][k]); w.pod(traQualStore[svid][k]); }
    }
    std::vector<std::string> parts;
    if ((rc = cs->exchange(DGPU_OK, w.buf, parts))) return rc;
    for (uint32_t svid = 0; svid < N; ++svid) { traStore[svid].clear(); traQualStore[svid].clear(); }
    for (int r = 0; r < cs->nranks; ++r) {
      ByteReader rd(parts[r].data(), parts[r].size());
      while (rd.ok() && !rd.done()) {
        const uint32_t svid = rd.pod<uint32_t>(), n = rd.pod<uint32_t>();
        if (svid >= N) return DGPU_ERR_NCCL;
        for (uint32_t k = 0; k < n && rd.ok(); ++k) {
          std::string sq = rd.str();
          const uint8_t q = rd.pod<uint8_t>();
          if (cs->owns(svs[svid].chr) && traStore[svid].insert(std::move(sq)).second) traQualStore[svid].push_back(q);
        }
      }
      if (!rd.ok()) return DGPU_ERR_NCCL;
    }
  }
  for (int32_t refIndex2 = 0; refIndex2 < (int32_t) target_len.size(); ++refIndex2)
    for (int32_t refIndex = refIndex2 + 1; refIndex < (int32_t) target_len.size(); ++refIndex)
      for (uint32_t svid = 0; svid < N; ++svid) {
        if (!_translocation(svs[svid].svt) || (cs && !cs->owns(refIndex))) continue;
        if ((svs[svid].chr != refIndex) || (svs[svid].chr2 != refIndex2)) continue;
        if (traStore[svid].size() <= 1) { reset(svs[svid]); continue; }
        queued.push_back(svid);
        clusters.push_back(std::vector<std::string>(traStore[svid].begin(), traStore[svid].end()));
        quals.push_back(traQualStore[svid]);
      }
  if (queued.empty() && !cs) return DGPU_OK;
  // The two device batches — msa() and alignConsensus() of every queued SV — are what a rank shards (SURVEY §8e): the read collection above is
  // host work every rank repeats; of the queue a rank processes one contiguous range, cut by cost (all-pairs LCS + progressive alignment grow with
  // reads^2 x length^2), and the finished records of all ranks are exchanged once.
  std::size_t lo = 0, hi = queued.size();
  std::vector<std::size_t> bounds;
  if (shard && shard->nranks > 1) {
    std::vector<uint64_t> cost(queued.size());
    for (std::size_t k = 0; k < queued.size(); ++k) {
      uint64_t L = 0;
      for (auto const& s : clusters[k]) L = std::max<uint64_t>(L, s.size());
      cost[k] = (uint64_t) clusters[k].size() * clusters[k].size() * L * L;
    }
    bounds = partitionByCost(cost, shard->nranks);
    lo = bounds[shard->rank]; hi = bounds[shard->rank + 1];
  }
  std::vector<std::string> consensus;
  std::vector<int> rows;
  std::vector<StructuralVariantRecord> work(hi - lo);
  std::vector<uint8_t> ok;
  if (hi > lo) {
    std::vector<std::vector<std::string> > mine(clusters.begin() + lo, clusters.begin() + hi);
    rc = msaBatch(ctx, c, mine, consensus, rows);
    if (!rc) {
      for (std::size_t k = lo; k < hi; ++k) { work[k - lo] = svs[queued[k]]; work[k - lo].consensus = consensus[k - lo]; }
      rc = alignConsensusBatch(ctx, c, target_len, chrseq, work, false, ok);
    }
    if (rc && !cs) return rc;   // (contig sharding: the error travels with the exchange below)
  }
  if (shard && shard->nranks > 1) {
    std::vector<StructuralVariantRecord> allWork;
    std::vector<uint8_t> allOk;
    if ((rc = shard->exchange(work, ok, bounds, allWork, allOk))) return rc;
    if (allWork.size() != queued.size()) return DGPU_ERR_NCCL;
    work.swap(allWork); ok.swap(allOk);
  }
  for (std::size_t k = 0; k < queued.size() && !rc; ++k) {
    StructuralVariantRecord& sv = svs[queued[k]];
    sv = work[k];
    if (!ok[k]) { reset(sv); continue; }
    std::vector<uint8_t>& qv = quals[k];
    sv.mapq = 0;
    for (uint8_t q : qv) sv.mapq += q;
    if (!qv.empty()) { const std::size_t n = qv.size() / 2; std::nth_element(qv.begin(), qv.begin() + n, qv.end()); sv.srMapQuality = qv[n]; }   // medianVector, src/util.h:78-84
    else sv.srMapQuality = 0;
    sv.srSupport = (int32_t) clusters[k].size();
  }
  if (cs) {   // the records of every rank's SVs
    ByteWriter w;
    for (uint32_t svid = 0; svid < N; ++svid)
      if (cs->owns(svs[svid].chr)) putSv(w, svs[svid]);
    std::vector<std::string> parts;
    if ((rc = cs->exchange(rc, w.buf, parts))) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      if (r == cs->rank) continue;
      ByteReader rd(parts[r].data(), parts[r].size());
      for (uint32_t svid = 0; svid < N; ++svid) {
        if (svs[svid].chr < (int32_t) cs->bounds[r] || svs[svid].chr >= (int32_t) cs->bounds[r + 1]) continue;
        getSv(rd, svs[svid]);
      }
      if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
    }
  }
  return DGPU_OK;
}

inline int assembleSplitReadsBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<const char*> const& chrseq,
                                   std::vector<TPosReadSV> const& srStore, std::vector<StructuralVariantRecord>& svs, std::vector<SrRecord> const& recs) {
  return assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, svs, std::vector<std::vector<SrRecord> const*>(1, &recs));
}

}  // namespace dellyb200
