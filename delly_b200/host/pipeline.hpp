// pipeline.hpp — the stage sequence of `delly sr` discovery + genotyping (dellyRun, src/delly.h:86-196) over in-memory
// alignments of one sample: scanPEandSR -> assembleSplitReads -> mergeSort -> sort + renumber -> annotateCoverage ->
// per-sample genotype fields (what vcfOutput derives, src/modvcf.h:667-715). File handling, exclude intervals, library
// estimation (getLibraryParams) and the BCF writer stay with the caller; every stage is the batched mirror of this repository.
#pragma once
#include "assemble.hpp"
#include "assemblelr.hpp"
#include "genotype.hpp"
#include "gl.hpp"
#include "scan.hpp"
#include "svanno.hpp"
#include "svreaddump.hpp"
#include "vcfparse.hpp"

namespace dellyb200 {

struct SrCallSet {
  std::vector<StructuralVariantRecord> svs;   // sorted, ids renumbered (src/delly.h:155-158)
  std::vector<JunctionCount> jctMap;          // junction-read support per SV
  std::vector<SpanningCount> spanMap;         // spanning-pair support per SV
  std::vector<ReadCount> rcMap;               // read-depth left / inside / right of the SV
  std::vector<SampleFormat> format;           // GT / GL / GQ / PL / FT / RCN of the sample
};

// The part of dellyRun after the SV list exists (src/delly.h:155-178): sort + renumber, annotateCoverage, per-sample genotype fields.
// out.svs holds the SVs on entry (from discovery or from a site list).
// `probes`: the junction probes of the (already sorted and renumbered) SV list when the caller prepared them once for several samples.
// `dump`: receives this sample's SV-read events.
inline int genotypeSrSites(dgpu_ctx* ctx, Config const& c, LibraryInfo const& lib, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                           std::vector<const char*> const& chrseq, std::vector<SrRecord> const& recs, SrCallSet& out, JunctionProbes const* probes = nullptr,
                           SvReadDump::File* dump = nullptr) {
  int rc = DGPU_OK;
  if (!probes) {
    std::sort(out.svs.begin(), out.svs.end());
    for (std::size_t i = 0; i < out.svs.size(); ++i) out.svs[i].id = (int32_t) i;
  }
  if (out.svs.empty()) return DGPU_OK;
  // annotateCoverage = junction-read half + spanning / read-depth half (independent of each other)
  if (probes) rc = annotateJunctionReadsWithProbes(ctx, c, target_len, *probes, out.svs.size(), recs, out.jctMap, dump ? &dump->sr : nullptr);
  else rc = annotateJunctionReadsBatch(ctx, c, target_len, target_name, chrseq, out.svs, recs, out.jctMap, dump ? &dump->sr : nullptr);
  if (rc) return rc;
  std::vector<bool> svOnChr(target_len.size(), false);
  for (auto const& sv : out.svs) { svOnChr[sv.chr] = true; svOnChr[sv.chr2] = true; }
  annotateSpanningAndDepth(c, lib, target_len, out.svs, svOnChr, recs, out.rcMap, out.spanMap, dump ? &dump->pe : nullptr);
  static const BoLog bl;
  out.format.resize(out.svs.size());
  for (std::size_t i = 0; i < out.svs.size(); ++i) {
    JunctionCount const& j = out.jctMap[i];
    // precise SVs are genotyped from junction reads, imprecise ones from spanning pairs (src/modvcf.h:668-669)
    std::vector<uint8_t> const& r = out.svs[i].precise ? j.ref : out.spanMap[i].ref;
    std::vector<uint8_t> const& a = out.svs[i].precise ? j.alt : out.spanMap[i].alt;
    out.format[i] = sampleFormat(bl, r, a, j.ps, (int32_t) j.hp1alt.size(), (int32_t) j.hp2alt.size(), out.rcMap[i].leftRC, out.rcMap[i].rc, out.rcMap[i].rightRC);
  }
  return DGPU_OK;
}

// `delly sr` discovery + genotyping of one sample (src/delly.h:130-178 without a site list)
inline int dellySrCall(dgpu_ctx* ctx, Config const& c, LibraryInfo& lib, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                       std::vector<const char*> const& chrseq, std::vector<SrRecord> const& recs, SrCallSet& out) {
  std::vector<StructuralVariantRecord> srSVs;
  std::vector<TPosReadSV> srStore;
  out = SrCallSet();
  int rc = scanPEandSRBatch(ctx, c, lib, target_len, recs, out.svs, srSVs, srStore);
  if (rc) return rc;
  if ((rc = assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, srSVs, recs))) return rc;
  mergeSort(out.svs, srSVs);
  return genotypeSrSites(ctx, c, lib, target_len, target_name, chrseq, recs, out);
}

// ---- several samples in one call set (tumour / normal, trios, cohorts: `delly call a.bam b.bam ...`) -----------------------------
// Discovery pools the samples (per-file scans concatenated in file order before sorting and clustering, src/shortpe.h:318-477; the
// split-read collection walks contig by contig and file by file, :81-156); genotyping is independent per file (annotateCoverage's outer
// loop is the file, src/coverage.h:346-352), so every sample gets its own count maps and genotype fields over the SAME SV list.
struct SrSampleCounts {
  std::vector<JunctionCount> jctMap;
  std::vector<SpanningCount> spanMap;
  std::vector<ReadCount> rcMap;
  std::vector<SampleFormat> format;
};
struct SrMultiCallSet {
  std::vector<StructuralVariantRecord> svs;
  std::vector<SrSampleCounts> sample;   // one per input file
};

inline int genotypeSrSitesMulti(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo> const& libs, std::vector<uint32_t> const& target_len,
                                std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq,
                                std::vector<std::vector<SrRecord> const*> const& samples, SrMultiCallSet& out) {
  std::sort(out.svs.begin(), out.svs.end());
  for (std::size_t i = 0; i < out.svs.size(); ++i) out.svs[i].id = (int32_t) i;
  out.sample.assign(samples.size(), SrSampleCounts());
  if (out.svs.empty()) return DGPU_OK;
  JunctionProbes probes;   // once for all samples, like the reference (src/coverage.h:164-263 precedes the loop over the files)
  int rc = prepareJunctionProbes(ctx, c, target_len, target_name, chrseq, out.svs, probes);
  if (rc) return rc;
  for (std::size_t f = 0; f < samples.size(); ++f) {
    SrCallSet one;
    one.svs = out.svs;
    if ((rc = genotypeSrSites(ctx, c, libs[f], target_len, target_name, chrseq, *samples[f], one, &probes))) return rc;
    out.sample[f].jctMap.swap(one.jctMap); out.sample[f].spanMap.swap(one.spanMap); out.sample[f].rcMap.swap(one.rcMap); out.sample[f].format.swap(one.format);
  }
  return DGPU_OK;
}

inline int dellySrCallMulti(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo>& libs, std::vector<uint32_t> const& target_len,
                            std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq,
                            std::vector<std::vector<SrRecord> const*> const& samples, SrMultiCallSet& out) {
  std::vector<StructuralVariantRecord> srSVs;
  std::vector<TPosReadSV> srStore;
  out = SrMultiCallSet();
  int rc = scanPEandSRBatch(ctx, c, libs, target_len, samples, out.svs, srSVs, srStore);
  if (rc) return rc;
  if ((rc = assembleSplitReadsBatch(ctx, c, target_len, chrseq, srStore, srSVs, samples))) return rc;
  mergeSort(out.svs, srSVs);
  return genotypeSrSitesMulti(ctx, c, libs, target_len, target_name, chrseq, samples, out);
}

// `delly sr -v sites.bcf` (genotyping mode, src/delly.h:151 -> vcfParse): the site list of a Delly BCF genotyped in one sample.
// Returns DGPU_ERR_ARG when the sites are not from a Delly (>= v1.1.7) file (the reference prints an error and genotypes what it parsed so far;
// that list is in out.svs).
inline int dellySrGenotype(dgpu_ctx* ctx, Config const& c, LibraryInfo const& lib, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                           std::vector<const char*> const& chrseq, std::vector<VcfSite> const& sites, bool headerHasConsBp, std::vector<SrRecord> const& recs,
                           SrCallSet& out) {
  out = SrCallSet();
  const bool ok = vcfParseSites(sites, headerHasConsBp, target_name, out.svs);
  for (auto const& sv : out.svs)
    if (sv.chr < 0 || sv.chr2 < 0) return DGPU_ERR_ARG;  // a site on a contig the alignments do not have
  int rc = genotypeSrSites(ctx, c, lib, target_len, target_name, chrseq, recs, out);
  if (rc) return rc;
  return ok ? DGPU_OK : DGPU_ERR_ARG;
}


// genotyping mode over several samples (`delly call -v sites.bcf a.bam b.bam ...`)
inline int dellySrGenotypeMulti(dgpu_ctx* ctx, Config const& c, std::vector<LibraryInfo> const& libs, std::vector<uint32_t> const& target_len,
                                std::vector<std::string> const& target_name, std::vector<const char*> const& chrseq, std::vector<VcfSite> const& sites,
                                bool headerHasConsBp, std::vector<std::vector<SrRecord> const*> const& samples, SrMultiCallSet& out) {
  out = SrMultiCallSet();
  const bool ok = vcfParseSites(sites, headerHasConsBp, target_name, out.svs);
  for (auto const& sv : out.svs)
    if (sv.chr < 0 || sv.chr2 < 0) return DGPU_ERR_ARG;
  const int rc = genotypeSrSitesMulti(ctx, c, libs, target_len, target_name, chrseq, samples, out);
  if (rc) return rc;
  return ok ? DGPU_OK : DGPU_ERR_ARG;
}

// ---- `delly lr` ---------------------------------------------------------------------------------------------------------

// _clusterSRReads without alternate alignments (src/junction.h:495-623 -> :476-492, :593-621): the CIGAR junction scan of every
// record (findJunctions), junction selection (fetchSVs), per SV type sort + cluster, and the read store that assemble() consumes.
// ids[i] = read id of recs[i] (hash_lr in the reference). ctx != nullptr: pair scans on the device.
inline int clusterSRReadsLR(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<LrRecord> const& recs,
                            std::vector<std::size_t> const& ids, float indelExtension, std::vector<StructuralVariantRecord>& svc,
                            std::vector<TPosReadSlices>& srStore, ContigShard const* cs = nullptr) {
  std::unordered_map<std::size_t, TJunctionVector> readBp;
  if (!cs) {
    for (std::size_t i = 0; i < recs.size(); ++i) {
      LrRecord const& rec = recs[i];
      if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP)) continue;
      if ((rec.mapq < c.minMapQual) || (rec.tid < 0)) continue;
      cigarJunctionsLR(readBp, ids[i], rec.flag, rec.tid, rec.pos, rec.mapq, rec.cigar, c.minClip, c.minRefSep, indelExtension);
    }
  } else {
    // contig sharding: the records (this rank's contigs, in stream order) fill one insertion log per contig; the logs of every rank are
    // gathered and replayed in contig order, which is the sequence of insertions of the walk over the whole stream. A read's supplementary
    // alignments on other ranks' contigs join its junctions there.
    std::vector<JunctionLog> logs(target_len.size());
    for (std::size_t i = 0; i < recs.size(); ++i) {
      LrRecord const& rec = recs[i];
      if (rec.flag & (BAMF_QCFAIL | BAMF_DUP | BAMF_UNMAP)) continue;
      if ((rec.mapq < c.minMapQual) || !cs->owns(rec.tid)) continue;
      cigarJunctionsLR(logs[rec.tid], ids[i], rec.flag, rec.tid, rec.pos, rec.mapq, rec.cigar, c.minClip, c.minRefSep, indelExtension);
    }
    ByteWriter w;
    for (std::size_t t = cs->lo(); t < cs->hi(); ++t) putJunctionLog(w, logs[t]);
    std::vector<std::string> parts;
    int rc = cs->exchange(DGPU_OK, w.buf, parts);
    if (rc) return rc;
    for (int r = 0; r < cs->nranks; ++r) {
      if (r == cs->rank) continue;
      ByteReader rd(parts[r].data(), parts[r].size());
      for (std::size_t t = cs->bounds[r]; t < cs->bounds[r + 1]; ++t) getJunctionLog(rd, logs[t]);
      if (!rd.ok() || !rd.done()) return DGPU_ERR_NCCL;
    }
    for (auto const& log : logs)
      for (auto const& e : log.ev) readBp[e.first].push_back(e.second);
  }
  for (auto& kv : readBp) std::sort(kv.second.begin(), kv.second.end());
  TSvtSRBamRecord srBR(2 * DELLY_SVT_TRANS);
  fetchSVs(c, readBp, srBR);
  srStore.assign(target_len.size(), TPosReadSlices());
  for (uint32_t svt = 0; svt < srBR.size(); ++svt) {
    if (srBR[svt].empty()) continue;
    std::sort(srBR[svt].begin(), srBR[svt].end());
    if (ctx) {
      const int rc = clusterGpu(ctx, c, srBR[svt], svc, (int32_t) svt);
      if (rc && cs) {   // a device failure of this rank alone: the next exchange of the other ranks (the assembly's) carries it to them
        std::vector<std::string> parts;
        cs->exchange(rc, std::string(), parts);
      }
      if (rc) return rc;
    }
    else cluster(c, srBR[svt], svc, (int32_t) svt);
    for (SRBamRecord const& r : srBR[svt]) {
      if ((r.svid == -1) || (r.rstart == -1)) continue;
      const int32_t insertChr = (r.primaryChr != -1) ? r.primaryChr : r.chr;
      if (r.rstart < (int32_t) target_len[insertChr]) srStore[insertChr][std::make_pair(r.rstart, r.id)].push_back(SeqSlice(r.svid, r.sstart, r.inslen, r.qual));
    }
  }
  return DGPU_OK;
}

struct LrCallSet {
  std::vector<StructuralVariantRecord> svs;
  std::vector<JunctionCount> jctMap;
  std::vector<ReadCount> rcMap;
  std::vector<SampleFormat> format;
  std::vector<MethylInfo> methyl;   // per SV, when the records carry MM / ML tags and a MethylConfig is given
};

// runTegua's stage sequence for one sample (src/tegua.h:104-193): _clusterSRReads -> assemble -> sort -> drop near-identical
// neighbours of the same type (:121-141) -> sort + renumber -> genotypeLR -> genotype fields.
// discovery half: the SV list, sorted and renumbered
inline int discoverLrSVs(dgpu_ctx* ctx, Config const& c, float indelExtension, std::vector<uint32_t> const& target_len, std::vector<const char*> const& chrseq,
                         std::vector<LrRecord> const& recs, std::vector<std::size_t> const& ids, std::vector<StructuralVariantRecord>& svsOut,
                         AssembleShard const* shard = nullptr, ContigShard const* cs = nullptr) {
  struct { std::vector<StructuralVariantRecord> svs; } out;
  std::vector<StructuralVariantRecord> svc;
  std::vector<TPosReadSlices> srStore;
  int rc = clusterSRReadsLR(ctx, c, target_len, recs, ids, indelExtension, svc, srStore, cs);
  if (rc) return rc;
  if ((rc = assembleLRBatch(ctx, c, target_len, chrseq, svc, srStore, recs, ids, shard, cs))) return rc;
  std::sort(svc.begin(), svc.end());
  std::map<int32_t, StructuralVariantRecord> lastSVperType;
  for (auto const& sv : svc) {
    if ((sv.srSupport == 0) && (sv.peSupport == 0)) continue;
    if (!out.svs.empty()) {
      auto lt = lastSVperType.find(sv.svt);
      if (lt != lastSVperType.end()) {
        StructuralVariantRecord const& last = lt->second;
        if ((last.chr == sv.chr) && (last.chr2 == sv.chr2) && (std::abs(sv.svStart - last.svStart) < (int32_t) c.minRefSep) &&
            (std::abs(sv.svEnd - last.svEnd) < (int32_t) c.minRefSep)) {
          const int32_t len1 = (sv.svt == 4) ? sv.insLen : (sv.svEnd - sv.svStart);
          const int32_t len2 = (last.svt == 4) ? last.insLen : (last.svEnd - last.svStart);
          int32_t lengthvar = (int32_t) std::min(0.1 * len1, 0.1 * len2);
          const int32_t lengthdiff = std::abs(len1 - len2);
          if (lengthvar < 15) lengthvar = 15;
          if (lengthdiff < lengthvar) continue;
        }
      }
    }
    lastSVperType[sv.svt] = sv;
    out.svs.push_back(sv);
  }
  std::sort(out.svs.begin(), out.svs.end());
  for (std::size_t i = 0; i < out.svs.size(); ++i) out.svs[i].id = (int32_t) i;
  svsOut.swap(out.svs);
  return DGPU_OK;
}

// the genotype fields of one sample from its junction counts and read-depth (src/modvcf.h:667-715; long reads have no spanning pairs)
inline void lrSampleFormat(std::vector<StructuralVariantRecord> const& svs, std::vector<JunctionCount> const& jctMap, std::vector<ReadCount> const& rcMap,
                           std::vector<SampleFormat>& format) {
  static const BoLog bl;
  static const std::vector<uint8_t> none;
  format.resize(svs.size());
  for (std::size_t i = 0; i < svs.size(); ++i) {
    JunctionCount const& j = jctMap[i];
    format[i] = sampleFormat(bl, svs[i].precise ? j.ref : none, svs[i].precise ? j.alt : none, j.ps, (int32_t) j.hp1alt.size(), (int32_t) j.hp2alt.size(), rcMap[i].leftRC,
                             rcMap[i].rc, rcMap[i].rightRC);
  }
}

inline int dellyLrCall(dgpu_ctx* ctx, Config const& c, float indelExtension, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                       std::vector<const char*> const& chrseq, std::vector<LrRecord> const& recs, std::vector<std::size_t> const& ids, LrCallSet& out,
                       MeiTemplates const* mei = nullptr, AnnoConfig const& annoCfg = AnnoConfig(), MethylConfig const* methylCfg = nullptr) {
  out = LrCallSet();
  int rc = discoverLrSVs(ctx, c, indelExtension, target_len, chrseq, recs, ids, out.svs);
  if (rc) return rc;
  if ((rc = genotypeLRBatch(ctx, c, target_len, target_name, chrseq, out.svs, recs, out.jctMap, out.rcMap, methylCfg, methylCfg ? &out.methyl : nullptr))) return rc;
  // annotateSV (src/genotype.h:159-163) reads the alleles genotypeLR has just filled and nothing the genotyping writes, so it
  // runs here for all chromosomes at once; the templates are the caller's (class MEI of the reference), none = no annotation
  if (mei && (rc = annotateSVs(ctx, annoCfg, *mei, chrseq, target_len, out.svs))) return rc;
  lrSampleFormat(out.svs, out.jctMap, out.rcMap, out.format);
  return DGPU_OK;
}

// Several long-read samples in one call set. Every discovery stage of the reference walks contig by contig and, inside a contig, file by
// file into shared containers (src/junction.h:345-350, :646-649, :702-705; src/assemble.h:783-787), which is the single-sample code over the
// record stream ordered by (contig, file, position): that stream is built here. Genotyping (and methylation) is per file (src/genotype.h:164).
struct LrSampleCounts {
  std::vector<JunctionCount> jctMap;
  std::vector<ReadCount> rcMap;
  std::vector<SampleFormat> format;
  std::vector<MethylInfo> methyl;
};
struct LrMultiCallSet {
  std::vector<StructuralVariantRecord> svs;
  std::vector<LrSampleCounts> sample;
};
struct LrSample {
  std::vector<LrRecord> const* recs;
  std::vector<std::size_t> const* ids;
};

// the record stream ordered by (contig, file, position) that the reference's discovery loops see over several files
inline void buildLrStream(std::vector<uint32_t> const& target_len, std::vector<LrSample> const& samples, std::vector<LrRecord>& stream, std::vector<std::size_t>& streamIds) {
  std::vector<std::size_t> ri(samples.size(), 0);
  for (int32_t refIndex = 0; refIndex < (int32_t) target_len.size(); ++refIndex)
    for (std::size_t f = 0; f < samples.size(); ++f) {
      std::vector<LrRecord> const& r = *samples[f].recs;
      for (; ri[f] < r.size() && r[ri[f]].tid == refIndex; ++ri[f]) { stream.push_back(r[ri[f]]); streamIds.push_back((*samples[f].ids)[ri[f]]); }
    }
}

inline int dellyLrCallMulti(dgpu_ctx* ctx, Config const& c, float indelExtension, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                            std::vector<const char*> const& chrseq, std::vector<LrSample> const& samples, LrMultiCallSet& out, MeiTemplates const* mei = nullptr,
                            AnnoConfig const& annoCfg = AnnoConfig(), MethylConfig const* methylCfg = nullptr, std::vector<LrSample> const* genoSamples = nullptr) {
  // samples: the records of the valid regions (discovery, src/tegua.h:119-122); genoSamples: the whole contigs for the genotyping pass when an
  // exclude file makes the two differ
  out = LrMultiCallSet();
  std::vector<LrRecord> stream;
  std::vector<std::size_t> streamIds;
  buildLrStream(target_len, samples, stream, streamIds);
  int rc = discoverLrSVs(ctx, c, indelExtension, target_len, chrseq, stream, streamIds, out.svs);
  if (rc) return rc;
  out.sample.assign(samples.size(), LrSampleCounts());
  std::vector<LrSample> const& geno = genoSamples ? *genoSamples : samples;
  for (std::size_t f = 0; f < samples.size(); ++f) {
    LrSampleCounts& sc = out.sample[f];
    if ((rc = genotypeLRBatch(ctx, c, target_len, target_name, chrseq, out.svs, *geno[f].recs, sc.jctMap, sc.rcMap, methylCfg, methylCfg ? &sc.methyl : nullptr))) return rc;
    lrSampleFormat(out.svs, sc.jctMap, sc.rcMap, sc.format);
  }
  if (mei && (rc = annotateSVs(ctx, annoCfg, *mei, chrseq, target_len, out.svs))) return rc;
  return DGPU_OK;
}

// `delly lr -v sites.bcf`: the site list genotyped in every sample (src/tegua.h:159-193; unlike the short-read mode the list is NOT sorted or
// renumbered: the ids are the file order, as vcfParse assigns them). Returns DGPU_ERR_ARG for a site list that is not from a Delly file or
// names a contig the alignments do not have.
inline int dellyLrGenotype(dgpu_ctx* ctx, Config const& c, std::vector<uint32_t> const& target_len, std::vector<std::string> const& target_name,
                           std::vector<const char*> const& chrseq, std::vector<VcfSite> const& sites, bool headerHasConsBp, std::vector<LrSample> const& samples,
                           LrMultiCallSet& out, MeiTemplates const* mei = nullptr, AnnoConfig const& annoCfg = AnnoConfig(), MethylConfig const* methylCfg = nullptr) {
  out = LrMultiCallSet();
  const bool ok = vcfParseSites(sites, headerHasConsBp, target_name, out.svs);
  for (auto const& sv : out.svs)
    if (sv.chr < 0 || sv.chr2 < 0) return DGPU_ERR_ARG;
  out.sample.assign(samples.size(), LrSampleCounts());
  int rc;
  for (std::size_t f = 0; f < samples.size(); ++f) {
    LrSampleCounts& sc = out.sample[f];
    if ((rc = genotypeLRBatch(ctx, c, target_len, target_name, chrseq, out.svs, *samples[f].recs, sc.jctMap, sc.rcMap, methylCfg, methylCfg ? &sc.methyl : nullptr))) return rc;
    lrSampleFormat(out.svs, sc.jctMap, sc.rcMap, sc.format);
  }
  if (mei && (rc = annotateSVs(ctx, annoCfg, *mei, chrseq, target_len, out.svs))) return rc;
  return ok ? DGPU_OK : DGPU_ERR_ARG;
}

}  // namespace dellyb200
