// assemblelr.hpp — the long-read assembly stage of `delly lr` (assemble, src/assemble.h:736-964), batched.
// The reference computes an SV's consensus inside its BAM scan, the moment enough reads have been collected (:832-873), and
// handles left-overs and translocations after each contig (:881-946); every consensus is msaEdlib (msaWfa for insertions)
// followed by alignConsensus. The collection rules decide WHICH reads reach the MSA and are mirrored exactly; the consensus
// work of an SV depends on nothing but its own reads, so all SVs are queued during the scan and then run through ONE
// msaEdlibBatch, ONE msaWfaBatch and two alignConsensusBatch calls (realign on / off).
#pragma once
#include "shard.hpp"
#include <algorithm>
#include <map>
#include <numeric>
#include <string>
#include <vector>

#include "genotype.hpp"
#include "msaedlib.hpp"
#include "msawfa.hpp"
#include "split.hpp"
#include "splitalign.hpp"

namespace dellyb200 {

struct SeqSlice {  // src/assemble.h:14-22
  int32_t svid = -1, sstart = -1, inslen = -1, qual = -1;
  SeqSlice() {}
  SeqSlice(int32_t sv, int32_t sst, int32_t il, int32_t q) : svid(sv), sstart(sst), inslen(il), qual(q) {}
};
typedef std::map<std::pair<int32_t, std::size_t>, std::vector<SeqSlice> > TPosReadSlices;  // (read start, read id) -> slices, per contig

// src/assemble.h:369-381
inline void selectBestReads(std::vector<std::string>& seqs, std::vector<int32_t>& scores, int32_t maxReads) {
  if ((int32_t) seqs.size() <= maxReads) return;
  std::vector<uint32_t> idx(seqs.size());
  std::iota(idx.begin(), idx.end(), 0);
  std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return scores[a] > scores[b]; });
  std::vector<std::string> sel;
  sel.reserve(maxReads);
  for (int32_t k = 0; k < maxReads; ++k) sel.push_back(std::move(seqs[idx[k]]));
  seqs = std::move(sel);
  scores.clear();
}

// recs: LrRecord list sorted by (tid, pos); LrRecord::ps is unused here; the read id is LrRecord-independent: ids[i] for recs[i].
// cs != nullptr (contig sharding): recs holds this rank's contigs only, and an SV belongs to the rank that owns sv.chr — its collection ends
// during the walk of that contig (inline trigger or left-over loop), so the reads of later contigs never reach it. Collection is append-only
// under the cap maxCandidates, so what an SV holds when its own contig is walked is the first maxCandidates entries of the lower contigs'
// entries in contig order: every rank first collects, on its own contigs, at most maxCandidates entries for each SV of a higher rank and sends
// them to the owner, which puts the lower ranks' entries in rank order in front of its own walk. The owner then queues, builds and aligns the
// consensus of its SVs, and the final records of every rank's SVs are exchanged.
inline int assembleLRBatch(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<const char*> const& chrseq,
                           std::vector<StructuralVariantRecord>& svs, std::vector<TPosReadSlices> const& srStore, std::vector<LrRecord> const& recs,
                           std::vector<std::size_t> const& ids, AssembleShard const* shard = nullptr, ContigShard const* cs = nullptr) {
  const std::size_t N = svs.size();
  std::vector<std::vector<std::string> > seqStore(N);
  std::vector<std::vector<int32_t> > scoreStore(N);
  const int32_t maxCandidates = (int32_t) c.maxReadPerSV * 4;
  std::vector<bool> svcons(N, false);
  struct Job { uint32_t svid; bool inlineTrigger; std::vector<std::string> reads; };
  std::vector<Job> jobs;
  auto reset = [&](StructuralVariantRecord& sv) { sv.consensus = ""; sv.srSupport = 0; sv.srAlignQuality = 0; };
  auto finish = [&](uint32_t svid) { seqStore[svid].clear(); scoreStore[svid].clear(); svcons[svid] = true; };
  // the contigs walked here and the SVs collected for: every contig and SV in one process; with cs, first (pass 0) the SVs of higher ranks,
  // then (pass 1) this rank's own
  auto take = [&](uint32_t svid, int pass) {
    if (!cs) return true;
    const int o = cs->owner(svs[svid].chr);
    return pass == 0 ? o > cs->rank : o == cs->rank;
  };
  auto walk = [&](int pass) {
    std::size_t ri = 0;
    for (int32_t refIndex = 0; refIndex < (int32_t) target_len.size(); ++refIndex) {
      const std::size_t rlo = ri;
      while (ri < recs.size() && recs[ri].tid == refIndex) ++ri;
      if (srStore[refIndex].empty()) continue;
      if (cs && !cs->owns(refIndex)) continue;
      std::vector<bool> hits(target_len[refIndex], false);
      for (auto const& kv : srStore[refIndex]) hits[(std::size_t) kv.first.first] = true;
      for (std::size_t q = rlo; q < ri; ++q) {
        LrRecord const& rec = recs[q];
        if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP | BAMF_SECONDARY | BAMF_SUPPLEMENTARY)) continue;
        if (!hits[(std::size_t) rec.pos]) continue;
        auto it = srStore[refIndex].find(std::make_pair(rec.pos, ids[q]));
        if (it == srStore[refIndex].end()) continue;
        const int32_t readlen = (int32_t) rec.seq.size();
        for (SeqSlice const& seqsl : it->second) {
          const int32_t svid = seqsl.svid;
          StructuralVariantRecord& sv = svs[svid];
          if (!take((uint32_t) svid, pass)) continue;
          if (svcons[svid] || ((int32_t) seqStore[svid].size() >= maxCandidates)) continue;
          int32_t window = c.minConsWindow;
          window += std::max(sv.ciposhigh - sv.ciposlow, sv.ciendhigh - sv.ciendlow);
          window += seqsl.inslen;
          const int32_t origCenter = (rec.flag & BAMF_REVERSE) ? (readlen - seqsl.sstart) : seqsl.sstart;
          int32_t sPos = std::max(origCenter - window, 0);
          int32_t ePos = std::min(origCenter + window, readlen);
          if ((ePos - sPos) <= window) continue;
          const int32_t anchorLen = origCenter - sPos, svSideLen = ePos - origCenter;
          std::string subseq = rec.seq.substr((std::size_t) sPos, (std::size_t) (ePos - sPos));
          if (_translocation(sv.svt)) {
            const uint8_t ct = _getSpanOrientation(sv.svt);
            if ((ct == 0 && refIndex == sv.chr2) || (ct == 1 && refIndex == sv.chr)) reverseComplement(subseq);
          } else if (sv.svt == 0) { if (rec.pos > (sv.svStart + sv.svEnd) / 2) reverseComplement(subseq); }
          else if (sv.svt == 1) { if (rec.flag & BAMF_REVERSE) reverseComplement(subseq); }
          seqStore[svid].push_back(std::move(subseq));
          scoreStore[svid].push_back(std::min(anchorLen, svSideLen));
          if ((!_translocation(sv.svt)) && (sv.chr == refIndex) &&
              (((int32_t) seqStore[svid].size() == maxCandidates) || ((int32_t) seqStore[svid].size() == sv.srSupport))) {   // enough split reads (:832-834)
            if (seqStore[svid].size() > 1) {
              selectBestReads(seqStore[svid], scoreStore[svid], (int32_t) c.maxReadPerSV);
              jobs.push_back(Job{(uint32_t) svid, true, seqStore[svid]});
            } else reset(sv);
            finish((uint32_t) svid);
          }
        }
      }
      if (pass == 0) continue;
      // left-overs and translocations whose second contig is this one (:881-946)
      for (int32_t refIndex2 = 0; refIndex2 <= refIndex; ++refIndex2)
        for (uint32_t svid = 0; svid < N; ++svid) {
          if (svcons[svid] || seqStore[svid].size() <= 1) continue;
          StructuralVariantRecord const& sv = svs[svid];
          const bool compute = _translocation(sv.svt) ? ((refIndex2 != refIndex) && (sv.chr == refIndex) && (sv.chr2 == refIndex2))
                                                      : ((refIndex2 == refIndex) && (sv.chr == refIndex) && (sv.chr2 == refIndex2));
          if (!compute) continue;
          selectBestReads(seqStore[svid], scoreStore[svid], (int32_t) c.maxReadPerSV);
          jobs.push_back(Job{svid, false, seqStore[svid]});
          finish(svid);
        }
    }
  };
  int rc;
  if (cs) {   // the entries of this rank's contigs for the SVs of higher ranks, to their owners
    walk(0);
    ByteWriter w;
    for (uint32_t svid = 0; svid < N; ++svid) {
      if (seqStore[svid].empty() || !take(svid, 0)) continue;
      w.pod(svid); w.pod<uint32_t>((uint32_t) seqStore[svid].size());
      for (std::size_t k = 0; k < seqStore[svid].size(); ++k) { w.str(seqStore[svid][k]); w.pod(scoreStore[svid][k]); }
      seqStore[svid].clear(); scoreStore[svid].clear();
    }
    std::vector<std::string> parts;
    if ((rc = cs->exchange(DGPU_OK, w.buf, parts))) return rc;
    for (int r = 0; r < cs->rank; ++r) {   // lower ranks first, in rank order (= contig order), under the cap
      ByteReader rd(parts[r].data(), parts[r].size());
      while (rd.ok() && !rd.done()) {
        const uint32_t svid = rd.pod<uint32_t>(), n = rd.pod<uint32_t>();
        if (!rd.ok() || svid >= N) return DGPU_ERR_NCCL;
        for (uint32_t k = 0; k < n && rd.ok(); ++k) {
          std::string sq = rd.str();
          const int32_t score = rd.pod<int32_t>();
          if (!take(svid, 1) || (int32_t) seqStore[svid].size() >= maxCandidates) continue;
          seqStore[svid].push_back(std::move(sq)); scoreStore[svid].push_back(score);
        }
      }
      if (!rd.ok()) return DGPU_ERR_NCCL;
    }
  }
  walk(1);
  for (uint32_t svid = 0; svid < N; ++svid) if (!svcons[svid]) reset(svs[svid]);   // unfinished SVs (:956-963)
  if (jobs.empty() && !cs) return DGPU_OK;   // the queue is built from replicated data: empty on every rank or on none

  // ---- consensus of every queued SV: msaEdlib (msaWfa for insertions), then alignConsensus ------------------------------
  // What a rank shards (SURVEY section 8e): the read collection above is host work every rank repeats; the queue is cut into contiguous
  // ranges of (nearly) equal cost (all-pairs distances + progressive paths: reads^2 x length^2), a rank runs the device batches of its
  // range, the finished records are exchanged in queue order. (With cs every queued job is this rank's own.)
  std::size_t jlo = 0, jhi = jobs.size();
  std::vector<std::size_t> bounds;
  if (shard && shard->nranks > 1 && !cs) {
    std::vector<uint64_t> cost(jobs.size());
    for (std::size_t k = 0; k < jobs.size(); ++k) {
      uint64_t L = 0;
      for (auto const& r : jobs[k].reads) L = std::max<uint64_t>(L, r.size());
      cost[k] = (uint64_t) jobs[k].reads.size() * jobs[k].reads.size() * L * L + 1;
    }
    bounds = partitionByCost(cost, shard->nranks);
    jlo = bounds[shard->rank]; jhi = bounds[shard->rank + 1];
  }
  std::vector<uint32_t> ed, wf;   // job indices
  for (uint32_t k = (uint32_t) jlo; k < (uint32_t) jhi; ++k) (svs[jobs[k].svid].svt != 4 ? ed : wf).push_back(k);
  std::vector<uint8_t> success(jobs.size(), 0);
  auto runJobs = [&]() -> int {
    int rc;
    if (!ed.empty()) {
      std::vector<std::vector<std::string> > clusters;
      for (uint32_t k : ed) clusters.push_back(jobs[k].reads);
      std::vector<std::string> consensus; std::vector<int> rows;
      if ((rc = msaEdlibBatch(ctx, c, clusters, consensus, rows))) return rc;
      std::vector<StructuralVariantRecord> work(ed.size());
      std::vector<std::string> tmpCons(ed.size());
      std::vector<int32_t> offsetTmp(ed.size(), 0);
      for (std::size_t i = 0; i < ed.size(); ++i) {
        work[i] = svs[jobs[ed[i]].svid];
        work[i].consensus = consensus[i];
        const int32_t svSize = work[i].svEnd - work[i].svStart;
        if (((work[i].svt == 0) || (work[i].svt == 1)) && (svSize < (int32_t) work[i].consensus.size())) {   // small inversions (:841-848)
          offsetTmp[i] = ((int32_t) work[i].consensus.size() - svSize) / 2;
          tmpCons[i] = work[i].consensus;
          work[i].consensus = work[i].consensus.substr((std::size_t) offsetTmp[i], (std::size_t) svSize);
        }
      }
      std::vector<uint8_t> ok;
      if ((rc = alignConsensusBatch(ctx, c, target_len, chrseq, work, true, ok))) return rc;
      for (std::size_t i = 0; i < ed.size(); ++i) {
        if (!tmpCons[i].empty()) { work[i].consensus = tmpCons[i]; work[i].consBp += offsetTmp[i]; }
        svs[jobs[ed[i]].svid] = work[i];
        success[ed[i]] = ok[i];
      }
    }
    if (!wf.empty()) {
      std::vector<std::vector<std::string> > clusters;
      std::vector<std::string> prefix, suffix;
      for (uint32_t k : wf) {
        StructuralVariantRecord const& sv = svs[jobs[k].svid];
        const char* seq = chrseq[sv.chr];
        const int32_t seqlen = (int32_t) target_len[sv.chr];
        clusters.push_back(jobs[k].reads);
        prefix.push_back(detail::upperSlice(seq, std::max(sv.svStart - c.minConsWindow, 0), sv.svStart));
        suffix.push_back(detail::upperSlice(seq, sv.svStart, std::min(seqlen, sv.svStart + c.minConsWindow)));
      }
      std::vector<std::string> consensus; std::vector<int> rows;
      if ((rc = msaWfaBatch(ctx, c, clusters, prefix, suffix, consensus, rows))) return rc;
      std::vector<StructuralVariantRecord> work;
      std::vector<uint32_t> which;
      for (std::size_t i = 0; i < wf.size(); ++i) {
        StructuralVariantRecord& sv = svs[jobs[wf[i]].svid];
        sv.consensus = consensus[i];
        // the in-scan path aligns any non-empty consensus (:858), the left-over path only a consensus shorter than insLen + 4 windows (:927)
        const bool go = jobs[wf[i]].inlineTrigger ? !sv.consensus.empty() : ((int32_t) sv.consensus.size() < sv.insLen + 4 * c.minConsWindow);
        if (go) { work.push_back(sv); which.push_back(wf[i]); }
      }
      if (!work.empty()) {
        std::vector<uint8_t> ok;
        if ((rc = alignConsensusBatch(ctx, c, target_len, chrseq, work, false, ok))) return rc;
        for (std::size_t i = 0; i < work.size(); ++i) { svs[jobs[which[i]].svid] = work[i]; success[which[i]] = ok[i]; }
      }
    }
    return DGPU_OK;
  };
  rc = runJobs();
  if (cs) {   // the final records of every rank's SVs (consensus, breakpoints, support, or the reset of an unfinished / failed SV)
    if (!rc) for (uint32_t k = 0; k < jobs.size(); ++k) if (!success[k]) reset(svs[jobs[k].svid]);
    ByteWriter w;
    for (uint32_t svid = 0; svid < N; ++svid) if (take(svid, 1)) putSv(w, svs[svid]);
    std::vector<std::string> parts;
    if ((rc = cs->exchange(rc, w.buf, parts))) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      if (r == cs->rank) continue;
      ByteReader rd(parts[r].data(), parts[r].size());
      for (uint32_t svid = 0; svid < N; ++svid) if (cs->owner(svs[svid].chr) == r) getSv(rd, svs[svid]);
      if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
    }
    return DGPU_OK;
  }
  if (rc) return rc;
  if (shard && shard->nranks > 1) {
    std::vector<StructuralVariantRecord> mine, all;
    std::vector<uint8_t> mineOk, allOk;
    for (std::size_t k = jlo; k < jhi; ++k) { mine.push_back(svs[jobs[k].svid]); mineOk.push_back(success[k]); }
    if ((rc = shard->exchange(mine, mineOk, bounds, all, allOk))) return rc;
    if (all.size() != jobs.size() || allOk.size() != jobs.size()) return DGPU_ERR_NCCL;
    for (std::size_t k = 0; k < jobs.size(); ++k) { svs[jobs[k].svid] = all[k]; success[k] = allOk[k]; }
  }
  for (uint32_t k = 0; k < jobs.size(); ++k) if (!success[k]) reset(svs[jobs[k].svid]);
  return DGPU_OK;
}

}  // namespace dellyb200
