// gather.hpp — the sharded (one process per GPU) form of the call chains and its one exchange step (SURVEY §8e).
//
// After the SV list exists every SV is independent for consensus building, consensus alignment and genotyping, so the list is cut into
// CONTIGUOUS ranges balanced by estimated cost; each rank runs the batched stage mirrors on its range only (its own GPU) and the finished
// records — the full StructuralVariantRecord (src/tags.h:82-130 incl. SVAnno, consensus, alleles) plus the per-sample count vectors
// (JunctionCount / SpanningCount, src/coverage.h:69-85; ReadCount, src/util.h:69-76; MethylInfo, src/methyl.h:35-55) — are exchanged with ONE
// all-gatherv (dgpu_gather_records over NCCL in the product; any GatherFn in the tests). Because the ranges are contiguous ranges of the
// reference's order (the list is sorted and renumbered BEFORE it is cut, exactly where the reference sorts: src/delly.h:155-158), restoring
// the reference's order is the concatenation of the ranks' records in rank order, and the id of a record is its local index plus the
// exclusive prefix sum of the range sizes.
//
// What is replicated on every rank: reading the alignments, the junction scan and the (sequential, order-dependent) clustering — host work
// whose result every rank needs in full. What is sharded: every device batch (msa, longNeedle / splitAlign, probe generation, the junction
// read realignment, read-depth and spanning-pair bookkeeping of the rank's own SVs).
// The contig-sharded form (Shard::contigBounds, `--shard-by contig`) removes the replicated reading and scan: a rank holds the alignments of its
// own contigs only and the per-contig logs of every stage travel between the ranks (genotypeSrSitesByContig below, host/scan.hpp,
// host/assemble.hpp, host/genotype.hpp); only junction selection, clustering, mergeSort and the sort stay replicated.
//
// Exactness: the N-rank result equals the 1-rank result record for record, unconditionally. The only cross-SV coupling in the genotyping
// pass is the batching of the junction-read jobs (flushed every 131072 x threads jobs and at the end of a contig, src/coverage.h:271,446,671):
// the per-SV cap is consulted both when a job is queued and when its result is merged, results are merged in job order, and a job that is
// not queued because the cap was already reached would have been dropped at the merge anyway — so the final lists of an SV depend only on
// that SV's own jobs in order, not on where the flushes fall. Every SV's jobs stay on one rank, in the reference's order.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "pipeline.hpp"
#include "shard.hpp"

namespace dellyb200 {

struct Shard {
  int rank = 0, nranks = 1;
  GatherFn gather;   // empty = single process
  // --shard-by contig: the contig ranges of the ranks (partitionContigs); empty = the SV list is cut by cost (--shard-by svs). The contig
  // mode holds from one rank up (one rank owns every contig and exchanges with itself).
  std::vector<std::size_t> contigBounds;
  bool active() const { return nranks > 1 && (bool) gather; }
  bool byContig() const { return !contigBounds.empty() && (bool) gather; }
  ContigShard contigShard() const { ContigShard cs; cs.rank = rank; cs.nranks = nranks; cs.bounds = contigBounds; cs.gather = gather; return cs; }
};

// wall-clock of the chain's stages (for the pipeline-level benchmark): name -> milliseconds, in call order
struct StageClock {
  std::vector<std::pair<std::string, double> > ms;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  void lap(const char* name) {
    const auto t1 = std::chrono::steady_clock::now();
    ms.push_back(std::make_pair(std::string(name), std::chrono::duration<double, std::milli>(t1 - t0).count()));
    t0 = t1;
  }
};

// ---- wire format (ByteWriter / ByteReader, host/shard.hpp) --------------------------------------------------------------------------
inline void putJct(ByteWriter& w, JunctionCount const& j) { w.bytes(j.ref); w.bytes(j.alt); w.bytes(j.hp1ref); w.bytes(j.hp1alt); w.bytes(j.hp2ref); w.bytes(j.hp2alt); w.pod(j.ps); }
inline void getJct(ByteReader& r, JunctionCount& j) { j.ref = r.bytes(); j.alt = r.bytes(); j.hp1ref = r.bytes(); j.hp1alt = r.bytes(); j.hp2ref = r.bytes(); j.hp2alt = r.bytes(); j.ps = r.pod<int32_t>(); }
inline void putMethyl(ByteWriter& w, MethylInfo const& m) { for (int k = 0; k < 4; ++k) { w.pod(m.alt[k]); w.pod(m.ref[k]); w.pod(m.mnc[k]); w.pod(m.mdp[k]); } }
inline void getMethyl(ByteReader& r, MethylInfo& m) { for (int k = 0; k < 4; ++k) { m.alt[k] = r.pod<int32_t>(); m.ref[k] = r.pod<int32_t>(); m.mnc[k] = r.pod<int32_t>(); m.mdp[k] = r.pod<int32_t>(); } }

// One rank's finished records: its SVs (ids already global) and, per sample, the count vectors of those SVs.
struct ShardRecords {
  std::vector<StructuralVariantRecord> svs;
  struct Sample { std::vector<JunctionCount> jct; std::vector<SpanningCount> span; std::vector<ReadCount> rc; std::vector<MethylInfo> methyl; };
  std::vector<Sample> sample;
};

inline std::string packShardRecords(ShardRecords const& s) {
  ByteWriter w;
  w.pod<uint32_t>(0x44475055u);   // "DGPU"
  w.pod<uint32_t>((uint32_t) s.svs.size());
  w.pod<uint32_t>((uint32_t) s.sample.size());
  for (auto const& v : s.svs) putSv(w, v);
  for (auto const& sm : s.sample) {
    const uint8_t has[4] = {(uint8_t) !sm.jct.empty(), (uint8_t) !sm.span.empty(), (uint8_t) !sm.rc.empty(), (uint8_t) !sm.methyl.empty()};
    for (uint8_t h : has) w.pod(h);
    if (has[0]) for (auto const& j : sm.jct) putJct(w, j);
    if (has[1]) for (auto const& sp : sm.span) { w.bytes(sp.ref); w.bytes(sp.alt); }
    if (has[2]) for (auto const& rc : sm.rc) { w.pod(rc.leftRC); w.pod(rc.rc); w.pod(rc.rightRC); }
    if (has[3]) for (auto const& m : sm.methyl) putMethyl(w, m);
  }
  return w.buf;
}

inline bool unpackShardRecords(std::string const& buf, ShardRecords& s) {
  ByteReader r(buf.data(), buf.size());
  if (r.pod<uint32_t>() != 0x44475055u) return false;
  const uint32_t n = r.pod<uint32_t>(), F = r.pod<uint32_t>();
  if (!r.ok()) return false;
  s.svs.assign(n, StructuralVariantRecord());
  for (auto& v : s.svs) getSv(r, v);
  s.sample.assign(F, ShardRecords::Sample());
  for (auto& sm : s.sample) {
    uint8_t has[4];
    for (uint8_t& h : has) h = r.pod<uint8_t>();
    if (has[0]) { sm.jct.resize(n); for (auto& j : sm.jct) getJct(r, j); }
    if (has[1]) { sm.span.resize(n); for (auto& sp : sm.span) { sp.ref = r.bytes(); sp.alt = r.bytes(); } }
    if (has[2]) { sm.rc.resize(n); for (auto& rc : sm.rc) { rc.leftRC = r.pod<int32_t>(); rc.rc = r.pod<int32_t>(); rc.rightRC = r.pod<int32_t>(); } }
    if (has[3]) { sm.methyl.resize(n); for (auto& m : sm.methyl) getMethyl(r, m); }
  }
  return r.ok() && r.done();
}

// Genotyping cost model of one SV, in DP cell units: the probe alignment of a precise SV (longNeedle of the consensus against the SV
// window: 3 matrices of |cons| x (|cons| + 2 x window), SURVEY §8d) plus the junction-read realignments of both breakpoints
// (≈ coverage x read length cells per probe; a constant per SV at a given depth).
inline uint64_t genotypingCost(StructuralVariantRecord const& sv, Config const& c) {
  uint64_t cost = 20000;
  if (sv.precise && !sv.consensus.empty()) cost += 3ull * sv.consensus.size() * (sv.consensus.size() + 2ull * (uint64_t) std::max(c.minConsWindow, 1));
  return cost;
}

// the genotype fields of one sample from its count vectors (src/modvcf.h:667-715): precise SVs from junction reads, imprecise ones from
// spanning pairs
inline void srSampleFormat(std::vector<StructuralVariantRecord> const& svs, SrSampleCounts& sc) {
  static const BoLog bl;
  sc.format.resize(svs.size());
  for (std::size_t i = 0; i < svs.size(); ++i) {
    JunctionCount const& j = sc.jctMap[i];
    std::vector<uint8_t> const& rr = svs[i].precise ? j.ref : sc.spanMap[i].ref;
    std::vector<uint8_t> const& aa = svs[i].precise ? j.alt : sc.spanMap[i].alt;
    sc.format[i] = sampleFormat(bl, rr, aa, j.ps, (int32_t) j.hp1alt.size(), (int32_t) j.hp2alt.size(), sc.rcMap[i].leftRC, sc.rcMap[i].rc, sc.rcMap[i].rightRC);
  }
}

// ---- contig-sharded genotyping (--shard-by contig) -----------------------------------------------------------------------------------
// The complete, sorted and renumbered SV list on a rank that holds the alignments of its own contigs only: the probes of the SVs with a
// breakpoint on those contigs, then per sample the junction-read pass and the spanning-pair / read-depth pass over the rank's contigs, each
// with its exchange (host/genotype.hpp). Every rank ends with the complete count vectors and genotype fields.
inline int genotypeSrSitesByContig(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo> const& libs, std::vector<uint32_t> const& target_len,
                                   std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq,
                                   std::vector<std::vector<SrRecord> const*> const& samples, ContigShard const& cs, SrMultiCallSet& out, StageClock* clock) {
  const std::size_t F = samples.size();
  out.sample.assign(F, SrSampleCounts());
  if (out.svs.empty()) return DGPU_OK;
  std::vector<uint8_t> want(out.svs.size());
  for (std::size_t i = 0; i < out.svs.size(); ++i) want[i] = cs.owns(out.svs[i].chr) || cs.owns(out.svs[i].chr2);
  JunctionProbes probes;
  int rc = prepareJunctionProbes(ctx, c, target_len, target_name, chrseq, out.svs, probes, &want);
  if (rc) {   // this rank alone may fail (a probe cut outside its consensus): the first exchange of the other ranks carries the error to them
    std::vector<std::string> parts;
    cs.exchange(rc, std::string(), parts);
    return rc;
  }
  if (clock) clock->lap("probes");
  std::vector<bool> svOnChr(target_len.size(), false);
  for (auto const& sv : out.svs) { svOnChr[sv.chr] = true; svOnChr[sv.chr2] = true; }
  for (std::size_t f = 0; f < F; ++f) {
    SrSampleCounts& sc = out.sample[f];
    if ((rc = annotateJunctionReadsWithProbes(ctx, c, target_len, probes, out.svs.size(), *samples[f], sc.jctMap, nullptr, &cs))) return rc;
    if ((rc = annotateSpanningAndDepth(c, libs[f], target_len, out.svs, svOnChr, *samples[f], sc.rcMap, sc.spanMap, nullptr, &cs))) return rc;
    srSampleFormat(out.svs, sc);
  }
  if (clock) clock->lap("genotype");
  return DGPU_OK;
}

// ---- sharded genotyping of a sorted, renumbered SV list (one or several samples) ---------------------------------------------------
// in/out: cs.svs = the COMPLETE list, sorted and renumbered, identical on every rank. On return every rank holds the complete result.
// dump: the SV-read events of every sample (one process only: the order of tied breakpoints depends on the whole SV list, see DESIGN §8).
inline int genotypeSrSitesSharded(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo> const& libs, std::vector<uint32_t> const& target_len,
                                  std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq,
                                  std::vector<std::vector<SrRecord> const*> const& samples, Shard const& shard, SrMultiCallSet& cs, StageClock* clock = nullptr,
                                  SvReadDump* dump = nullptr) {
  const std::size_t F = samples.size();
  if (dump && (shard.active() || shard.byContig())) return DGPU_ERR_ARG;
  if (shard.byContig()) return genotypeSrSitesByContig(ctx, c, libs, target_len, target_name, chrseq, samples, shard.contigShard(), cs, clock);
  cs.sample.assign(F, SrSampleCounts());
  if (dump) dump->file.assign(F, SvReadDump::File());
  if (cs.svs.empty()) return DGPU_OK;
  if (!shard.active()) {
    JunctionProbes probes;
    int rc = prepareJunctionProbes(ctx, c, target_len, target_name, chrseq, cs.svs, probes);
    if (rc) return rc;
    if (clock) clock->lap("probes");
    for (std::size_t f = 0; f < F; ++f) {
      SrCallSet one; one.svs = cs.svs;
      if ((rc = genotypeSrSites(ctx, c, libs[f], target_len, target_name, chrseq, *samples[f], one, &probes, dump ? &dump->file[f] : nullptr))) return rc;
      cs.sample[f].jctMap.swap(one.jctMap); cs.sample[f].spanMap.swap(one.spanMap); cs.sample[f].rcMap.swap(one.rcMap); cs.sample[f].format.swap(one.format);
    }
    if (clock) clock->lap("genotype");
    return DGPU_OK;
  }
  std::vector<uint64_t> cost(cs.svs.size());
  for (std::size_t i = 0; i < cs.svs.size(); ++i) cost[i] = genotypingCost(cs.svs[i], c);
  const std::vector<std::size_t> bounds = partitionByCost(cost, shard.nranks);
  const std::size_t lo = bounds[shard.rank], hi = bounds[shard.rank + 1];
  // this rank's range with rank-local ids 0..k-1 (the count maps are indexed by id)
  ShardRecords mine;
  mine.svs.assign(cs.svs.begin() + lo, cs.svs.begin() + hi);
  for (std::size_t i = 0; i < mine.svs.size(); ++i) mine.svs[i].id = (int32_t) i;
  mine.sample.assign(F, ShardRecords::Sample());
  int rc = DGPU_OK;
  if (!mine.svs.empty()) {
    JunctionProbes probes;
    if ((rc = prepareJunctionProbes(ctx, c, target_len, target_name, chrseq, mine.svs, probes))) return rc;
    if (clock) clock->lap("probes");
    for (std::size_t f = 0; f < F; ++f) {
      SrCallSet one; one.svs = mine.svs;
      if ((rc = genotypeSrSites(ctx, c, libs[f], target_len, target_name, chrseq, *samples[f], one, &probes))) return rc;
      mine.sample[f].jct.swap(one.jctMap); mine.sample[f].span.swap(one.spanMap); mine.sample[f].rc.swap(one.rcMap);
    }
  }
  if (clock) clock->lap("genotype");
  // ids become global: local index + exclusive prefix sum of the range sizes (= lo)
  for (std::size_t i = 0; i < mine.svs.size(); ++i) mine.svs[i].id = (int32_t) (lo + i);
  std::vector<std::string> parts;
  if ((rc = shard.gather(packShardRecords(mine), parts))) return rc;
  if ((int) parts.size() != shard.nranks) return DGPU_ERR_NCCL;
  if (clock) clock->lap("gather_records");
  // restore the reference's order: concatenation in rank order (the ranges are contiguous ranges of the sorted list)
  std::vector<StructuralVariantRecord> all;
  for (std::size_t f = 0; f < F; ++f) { cs.sample[f].jctMap.clear(); cs.sample[f].spanMap.clear(); cs.sample[f].rcMap.clear(); }
  for (int r = 0; r < shard.nranks; ++r) {
    ShardRecords part;
    if (!unpackShardRecords(parts[r], part)) return DGPU_ERR_NCCL;
    if (part.svs.size() != bounds[r + 1] - bounds[r] || (part.sample.size() != F && !part.svs.empty())) return DGPU_ERR_NCCL;
    for (std::size_t i = 0; i < part.svs.size(); ++i) {
      if (part.svs[i].id != (int32_t) (bounds[r] + i)) return DGPU_ERR_NCCL;
      all.push_back(part.svs[i]);
    }
    for (std::size_t f = 0; f < F && !part.svs.empty(); ++f) {
      cs.sample[f].jctMap.insert(cs.sample[f].jctMap.end(), part.sample[f].jct.begin(), part.sample[f].jct.end());
      cs.sample[f].spanMap.insert(cs.sample[f].spanMap.end(), part.sample[f].span.begin(), part.sample[f].span.end());
      cs.sample[f].rcMap.insert(cs.sample[f].rcMap.end(), part.sample[f].rc.begin(), part.sample[f].rc.end());
    }
  }
  if (all.size() != cs.svs.size()) return DGPU_ERR_NCCL;
  cs.svs.swap(all);
  for (std::size_t f = 0; f < F; ++f) srSampleFormat(cs.svs, cs.sample[f]);
  return DGPU_OK;
}

// `delly sr -v sites.bcf` sharded over ranks (BASELINE configs[3]: genotype mode, cluster-sharded)
inline int dellySrGenotypeSharded(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo> const& libs, std::vector<uint32_t> const& target_len,
                                  std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq, std::vector<VcfSite> const& sites,
                                  bool headerHasConsBp, std::vector<std::vector<SrRecord> const*> const& samples, Shard const& shard, SrMultiCallSet& out,
                                  StageClock* clock = nullptr, SvReadDump* dump = nullptr) {
  out = SrMultiCallSet();
  if (dump && (shard.active() || shard.byContig())) return DGPU_ERR_ARG;
  const bool ok = vcfParseSites(sites, headerHasConsBp, target_name, out.svs);
  for (auto const& sv : out.svs)
    if (sv.chr < 0 || sv.chr2 < 0) return DGPU_ERR_ARG;
  std::sort(out.svs.begin(), out.svs.end());   // src/delly.h:155-158, on every rank identically, BEFORE the list is cut
  for (std::size_t i = 0; i < out.svs.size(); ++i) out.svs[i].id = (int32_t) i;
  if (clock) clock->lap("parse_sort_sites");
  const int rc = genotypeSrSitesSharded(ctx, c, libs, target_len, target_name, chrseq, samples, shard, out, clock, dump);
  if (rc) return rc;
  return ok ? DGPU_OK : DGPU_ERR_ARG;
}

inline AssembleShard makeAssembleShard(Shard const& shard);

// `delly sr` discovery + genotyping sharded over ranks. --shard-by svs: scan + clustering replicated (host), split-read assembly and genotyping
// cut by cost. --shard-by contig: every rank holds, scans, assembles and genotypes the alignments of its own contigs, the per-contig logs are
// exchanged (host/scan.hpp, host/assemble.hpp, host/genotype.hpp), junction selection, clustering, mergeSort and the sort run on every rank.
inline int dellySrCallSharded(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo>& libs, std::vector<uint32_t> const& target_len,
                              std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq,
                              std::vector<std::vector<SrRecord> const*> const& samples, Shard const& shard, SrMultiCallSet& out, StageClock* clock = nullptr,
                              std::vector<std::vector<SrRecord> const*> const* genoSamples = nullptr, SvReadDump* dump = nullptr) {
  // samples: the records of the valid regions (scan, clustering, assembly); genoSamples: the records of the whole contigs for the genotyping pass
  // (src/coverage.h reads every contig end to end) — the same lists unless an exclude file is in play. dump: indexes into genoSamples.
  std::vector<StructuralVariantRecord> srSVs;
  std::vector<TPosReadSV> srStore;
  out = SrMultiCallSet();
  if (dump && (shard.active() || shard.byContig())) return DGPU_ERR_ARG;
  const ContigShard cs = shard.contigShard();
  int rc = scanPEandSRBatch(ctx, c, libs, target_len, samples, out.svs, srSVs, srStore, shard.byContig() ? &cs : nullptr);
  if (rc) return rc;
  if (clock) clock->lap("scan_cluster");
  if (shard.byContig()) {
    if ((rc = assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, srSVs, samples, nullptr, &cs))) return rc;
  } else if (shard.active()) {
    AssembleShard as = makeAssembleShard(shard);
    if ((rc = assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, srSVs, samples, &as))) return rc;
  } else if ((rc = assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, srSVs, samples))) return rc;
  if (clock) clock->lap("assemble");
  mergeSort(out.svs, srSVs);
  std::sort(out.svs.begin(), out.svs.end());
  for (std::size_t i = 0; i < out.svs.size(); ++i) out.svs[i].id = (int32_t) i;
  if (clock) clock->lap("merge_sort");
  return genotypeSrSitesSharded(ctx, c, libs, target_len, target_name, chrseq, genoSamples ? *genoSamples : samples, shard, out, clock, dump);
}

// The exchange of an assembly queue cut by cost (AssembleShard): every rank sends the finished records of its range and receives all of them in
// queue order.
inline AssembleShard makeAssembleShard(Shard const& shard) {
  AssembleShard as;
  as.rank = shard.rank; as.nranks = shard.nranks;
  as.exchange = [shard](std::vector<StructuralVariantRecord> const& mineWork, std::vector<uint8_t> const& mineOk, std::vector<std::size_t> const& bounds,
                        std::vector<StructuralVariantRecord>& allWork, std::vector<uint8_t>& allOk) -> int {
    ByteWriter w;
    w.pod<uint32_t>((uint32_t) mineWork.size());
    for (std::size_t k = 0; k < mineWork.size(); ++k) { putSv(w, mineWork[k]); w.pod<uint8_t>(mineOk[k]); }
    std::vector<std::string> parts;
    int r2 = shard.gather(w.buf, parts);
    if (r2) return r2;
    if ((int) parts.size() != shard.nranks) return DGPU_ERR_NCCL;
    allWork.clear(); allOk.clear();
    for (int r = 0; r < shard.nranks; ++r) {
      ByteReader rd(parts[r].data(), parts[r].size());
      const uint32_t n = rd.pod<uint32_t>();
      if (!rd.ok() || n != bounds[r + 1] - bounds[r]) return DGPU_ERR_NCCL;
      for (uint32_t k = 0; k < n; ++k) { StructuralVariantRecord v; getSv(rd, v); allWork.push_back(v); allOk.push_back(rd.pod<uint8_t>()); }
      if (!rd.ok()) return DGPU_ERR_NCCL;
    }
    return DGPU_OK;
  };
  return as;
}

// ---- long reads (`delly lr`) ------------------------------------------------------------------------------------------------------------
// Sharded genotyping + annotation of an SV list whose ids are its indices (discovery: sorted and renumbered, src/tegua.h:150-156; -v: file order).
// A rank takes a contiguous range by cost, genotypes it in every sample with rank-local ids (genotypeLR fills the alleles, annotateSV reads them),
// ids become local index + range start, one all-gatherv of the complete records and count vectors, concatenation in rank order.
inline int genotypeLrSitesSharded(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                                  std::vector<const char*> const& chrseq, std::vector<LrSample> const& samples, Shard const& shard, LrMultiCallSet& cs,
                                  MeiTemplates const* mei, AnnoConfig const& annoCfg, MethylConfig const* methylCfg, bool annotateBeforeFormat,
                                  SvReadDump* dump = nullptr) {
  const std::size_t F = samples.size();
  if (dump && shard.active()) return DGPU_ERR_ARG;
  cs.sample.assign(F, LrSampleCounts());
  if (dump) dump->file.assign(F, SvReadDump::File());
  int rc;
  auto runRange = [&](std::vector<StructuralVariantRecord>& svs, std::vector<LrSampleCounts>& out) -> int {
    out.assign(F, LrSampleCounts());
    for (std::size_t f = 0; f < F; ++f) {
      LrSampleCounts& sc = out[f];
      int r = genotypeLRBatch(ctx, c, target_len, target_name, chrseq, svs, *samples[f].recs, sc.jctMap, sc.rcMap, methylCfg, methylCfg ? &sc.methyl : nullptr,
                              dump ? &dump->file[f].sr : nullptr);
      if (r) return r;
    }
    if (mei) { int r = annotateSVs(ctx, annoCfg, *mei, chrseq, target_len, svs); if (r) return r; }
    return DGPU_OK;
  };
  (void) annotateBeforeFormat;
  if (!shard.active()) {
    if ((rc = runRange(cs.svs, cs.sample))) return rc;
  } else {
    std::vector<uint64_t> cost(cs.svs.size());
    for (std::size_t i = 0; i < cs.svs.size(); ++i) cost[i] = genotypingCost(cs.svs[i], c);
    const std::vector<std::size_t> bounds = partitionByCost(cost, shard.nranks);
    const std::size_t lo = bounds[shard.rank], hi = bounds[shard.rank + 1];
    ShardRecords mine;
    mine.svs.assign(cs.svs.begin() + lo, cs.svs.begin() + hi);
    for (std::size_t i = 0; i < mine.svs.size(); ++i) mine.svs[i].id = (int32_t) i;
    std::vector<LrSampleCounts> local;
    if ((rc = runRange(mine.svs, local))) return rc;
    mine.sample.assign(F, ShardRecords::Sample());
    for (std::size_t f = 0; f < F; ++f) { mine.sample[f].jct.swap(local[f].jctMap); mine.sample[f].rc.swap(local[f].rcMap); mine.sample[f].methyl.swap(local[f].methyl); }
    for (std::size_t i = 0; i < mine.svs.size(); ++i) mine.svs[i].id = (int32_t) (lo + i);
    std::vector<std::string> parts;
    if ((rc = shard.gather(packShardRecords(mine), parts))) return rc;
    if ((int) parts.size() != shard.nranks) return DGPU_ERR_NCCL;
    std::vector<StructuralVariantRecord> all;
    for (int r = 0; r < shard.nranks; ++r) {
      ShardRecords part;
      if (!unpackShardRecords(parts[r], part)) return DGPU_ERR_NCCL;
      if (part.svs.size() != bounds[r + 1] - bounds[r] || (part.sample.size() != F && !part.svs.empty())) return DGPU_ERR_NCCL;
      for (std::size_t i = 0; i < part.svs.size(); ++i) {
        if (part.svs[i].id != (int32_t) (bounds[r] + i)) return DGPU_ERR_NCCL;
        all.push_back(part.svs[i]);
      }
      for (std::size_t f = 0; f < F && !part.svs.empty(); ++f) {
        LrSampleCounts& sc = cs.sample[f];
        sc.jctMap.insert(sc.jctMap.end(), part.sample[f].jct.begin(), part.sample[f].jct.end());
        sc.rcMap.insert(sc.rcMap.end(), part.sample[f].rc.begin(), part.sample[f].rc.end());
        sc.methyl.insert(sc.methyl.end(), part.sample[f].methyl.begin(), part.sample[f].methyl.end());
      }
    }
    if (all.size() != cs.svs.size()) return DGPU_ERR_NCCL;
    cs.svs.swap(all);
  }
  for (std::size_t f = 0; f < F; ++f) lrSampleFormat(cs.svs, cs.sample[f].jctMap, cs.sample[f].rcMap, cs.sample[f].format);
  return DGPU_OK;
}

// ---- contig-sharded long reads (`delly_b200 lr --shard-by contig`) ---------------------------------------------------------------------
// A rank holds the long reads of its own contigs only. Discovery: the junction logs are gathered and replayed in contig order
// (clusterSRReadsLR), the read collection of an SV ends on the rank of sv.chr, which receives the lower ranks' candidates and builds the
// consensus (assembleLRBatch). Genotyping per file: the cap counts of SVs split over two ranks, then the decided qualities, read-depth and
// methylation sums (genotypeLRBatch). Annotation below. Junction selection, clustering, the sort, the near-duplicate filter and the
// renumbering run on every rank over the same inputs.

// annotateSVs over the SVs whose first breakpoint is on this rank's contigs; the annotations of every rank's SVs are exchanged
inline int annotateSVsByContig(dgpu_ctx* ctx, AnnoConfig const& annoCfg, MeiTemplates const& mei, std::vector<const char*> const& chrseq,
                               std::vector<uint32_t> const& target_len, std::vector<StructuralVariantRecord>& svs, ContigShard const& cs) {
  std::vector<int32_t> which;
  for (std::size_t i = 0; i < svs.size(); ++i)
    if (!_translocation(svs[i].svt) && cs.owns(svs[i].chr)) which.push_back((int32_t) i);
  int rc = which.empty() ? DGPU_OK : annotateSVBatch(ctx, annoCfg, mei, chrseq, target_len, svs, which);
  ByteWriter w;
  for (int32_t i : which) { SVAnno const& a = svs[i].anno; w.pod<uint8_t>(a.isRC ? 1 : 0); w.pod(a.seqType); w.pod(a.homLen); w.pod(a.trPeriod); w.pod(a.trCopies); }
  std::vector<std::string> parts;
  if ((rc = cs.exchange(rc, w.buf, parts))) return rc;
  for (int r = 0; r < cs.nranks; ++r) {
    if (r == cs.rank) continue;
    ByteReader rd(parts[r].data(), parts[r].size());
    for (StructuralVariantRecord& sv : svs) {
      if (_translocation(sv.svt) || cs.owner(sv.chr) != r) continue;
      sv.anno.isRC = rd.pod<uint8_t>() != 0; sv.anno.seqType = rd.pod<int32_t>(); sv.anno.homLen = rd.pod<int32_t>(); sv.anno.trPeriod = rd.pod<int32_t>();
      sv.anno.trCopies = rd.pod<float>();
    }
    if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
  }
  return DGPU_OK;
}

// genotyping (every file) + annotation of a complete SV list whose ids are its indices, on a rank that holds its own contigs' reads
inline int genotypeLrSitesByContig(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                                   std::vector<const char*> const& chrseq, std::vector<LrSample> const& samples, ContigShard const& cs, LrMultiCallSet& out,
                                   MeiTemplates const* mei, AnnoConfig const& annoCfg, MethylConfig const* methylCfg, StageClock* clock) {
  out.sample.assign(samples.size(), LrSampleCounts());
  int rc;
  for (std::size_t f = 0; f < samples.size(); ++f) {
    LrSampleCounts& sc = out.sample[f];
    if ((rc = genotypeLRBatch(ctx, c, target_len, target_name, chrseq, out.svs, *samples[f].recs, sc.jctMap, sc.rcMap, methylCfg, methylCfg ? &sc.methyl : nullptr,
                              nullptr, &cs)))
      return rc;
    lrSampleFormat(out.svs, sc.jctMap, sc.rcMap, sc.format);
  }
  if (mei && (rc = annotateSVsByContig(ctx, annoCfg, *mei, chrseq, target_len, out.svs, cs))) return rc;
  if (clock) clock->lap("genotype");
  return DGPU_OK;
}

// `delly lr` discovery + genotyping, contig-sharded: the result equals dellyLrCallMulti's on every rank
inline int dellyLrCallByContig(dgpu_ctx* ctx, Config const& c, float indelExtension, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                               std::vector<const char*> const& chrseq, std::vector<LrSample> const& samples, ContigShard const& cs, LrMultiCallSet& out,
                               MeiTemplates const* mei, AnnoConfig const& annoCfg, MethylConfig const* methylCfg, std::vector<LrSample> const* genoSamples,
                               StageClock* clock) {
  out = LrMultiCallSet();
  std::vector<LrRecord> stream;
  std::vector<std::size_t> streamIds;
  buildLrStream(target_len, samples, stream, streamIds);
  int rc = discoverLrSVs(ctx, c, indelExtension, target_len, chrseq, stream, streamIds, out.svs, nullptr, &cs);
  if (rc) return rc;
  if (clock) clock->lap("discover");
  return genotypeLrSitesByContig(ctx, c, target_len, target_name, chrseq, genoSamples ? *genoSamples : samples, cs, out, mei, annoCfg, methylCfg, clock);
}

// `delly lr` over ranks. --shard-by svs: the record stream, the junction clustering and the read collection replicated (host), the per-SV
// consensus + consensus alignment and the genotyping / annotation sharded by cost. --shard-by contig: dellyLrCallByContig.
inline int dellyLrCallSharded(dgpu_ctx* ctx, Config const& c, float indelExtension, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                              std::vector<const char*> const& chrseq, std::vector<LrSample> const& samples, Shard const& shard, LrMultiCallSet& out,
                              MeiTemplates const* mei = nullptr, AnnoConfig const& annoCfg = AnnoConfig(), MethylConfig const* methylCfg = nullptr,
                              std::vector<LrSample> const* genoSamples = nullptr, SvReadDump* dump = nullptr, StageClock* clock = nullptr) {
  out = LrMultiCallSet();
  if (dump && (shard.active() || shard.byContig())) return DGPU_ERR_ARG;
  if (shard.byContig())
    return dellyLrCallByContig(ctx, c, indelExtension, target_len, target_name, chrseq, samples, shard.contigShard(), out, mei, annoCfg, methylCfg, genoSamples, clock);
  std::vector<LrRecord> stream;
  std::vector<std::size_t> streamIds;
  buildLrStream(target_len, samples, stream, streamIds);
  AssembleShard as;
  if (shard.active()) as = makeAssembleShard(shard);
  int rc = discoverLrSVs(ctx, c, indelExtension, target_len, chrseq, stream, streamIds, out.svs, shard.active() ? &as : nullptr);
  if (rc) return rc;
  if (clock) clock->lap("discover");
  rc = genotypeLrSitesSharded(ctx, c, target_len, target_name, chrseq, genoSamples ? *genoSamples : samples, shard, out, mei, annoCfg, methylCfg, true, dump);
  if (!rc && clock) clock->lap("genotype");
  return rc;
}

// `delly lr -v sites.bcf` over ranks (ids = file order, src/tegua.h:157)
inline int dellyLrGenotypeSharded(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                                  std::vector<const char*> const& chrseq, std::vector<VcfSite> const& sites, bool headerHasConsBp, std::vector<LrSample> const& samples,
                                  Shard const& shard, LrMultiCallSet& out, MeiTemplates const* mei = nullptr, AnnoConfig const& annoCfg = AnnoConfig(),
                                  MethylConfig const* methylCfg = nullptr, SvReadDump* dump = nullptr, StageClock* clock = nullptr) {
  out = LrMultiCallSet();
  if (dump && (shard.active() || shard.byContig())) return DGPU_ERR_ARG;
  const bool ok = vcfParseSites(sites, headerHasConsBp, target_name, out.svs);
  for (auto const& sv : out.svs)
    if (sv.chr < 0 || sv.chr2 < 0) return DGPU_ERR_ARG;
  for (std::size_t i = 0; i < out.svs.size(); ++i)
    if (out.svs[i].id != (int32_t) i) return DGPU_ERR_ARG;   // the count vectors are indexed by id
  if (clock) clock->lap("parse_sites");
  const int rc = shard.byContig()
                     ? genotypeLrSitesByContig(ctx, c, target_len, target_name, chrseq, samples, shard.contigShard(), out, mei, annoCfg, methylCfg, clock)
                     : genotypeLrSitesSharded(ctx, c, target_len, target_name, chrseq, samples, shard, out, mei, annoCfg, methylCfg, false, dump);
  if (rc) return rc;
  if (clock && !shard.byContig()) clock->lap("genotype");
  return ok ? DGPU_OK : DGPU_ERR_ARG;
}

}  // namespace dellyb200
