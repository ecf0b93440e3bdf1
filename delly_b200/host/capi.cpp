// capi.cpp — flat C hooks over the C++ host mirror (delly_b200/host/*.hpp) so the parity tests can drive it
// through ctypes next to the compiled reference. Built into libdelly_b200_host.so, which links
// libdelly_b200.so (the CUDA library); nothing here touches oracle/.
#include <cmath>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <map>
#include <mutex>
#include <thread>

#include "cluster.hpp"
#include "genotype.hpp"
#include "assemble.hpp"
#include "assemblelr.hpp"
#include "scan.hpp"
#include "pipeline.hpp"
#include "vcf.hpp"
#include "gl.hpp"
#include "junction.hpp"
#include "msa.hpp"
#include "split.hpp"
#include "splitalign.hpp"
#include "msaedlib.hpp"
#include "msawfa.hpp"
#include "svanno.hpp"
#include "seqidentity.hpp"
#include "edlib_compat.hpp"
#include "gather.hpp"

using namespace dellyb200;

extern "C" {

// cluster(c, br, sv, svt) — layout as oracle/ref_wrap2.cpp::ref_cluster_sr
int dh_cluster_sr(const int32_t* br8, const uint64_t* ids, int n, int svt, int minClique, int maxReadSep, int graphPruning, int nchr,
                  int32_t* svid_out, int32_t* sv_out, int cap) {
  Config c; c.minCliqueSize = (uint16_t) minClique; c.maxReadSep = maxReadSep; c.graphPruning = graphPruning; c.nchr = nchr;
  std::vector<SRBamRecord> br;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = br8 + 8 * i;
    br.push_back(SRBamRecord(r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], (std::size_t) ids[i]));
  }
  std::vector<StructuralVariantRecord> sv;
  cluster(c, br, sv, svt);
  for (int i = 0; i < n; ++i) svid_out[i] = br[i].svid;
  if ((int) sv.size() > cap) return -1;
  for (std::size_t i = 0; i < sv.size(); ++i) {
    int32_t* o = sv_out + 14 * i;
    o[0] = sv[i].chr; o[1] = sv[i].svStart; o[2] = sv[i].chr2; o[3] = sv[i].svEnd; o[4] = sv[i].ciposlow; o[5] = sv[i].ciposhigh;
    o[6] = sv[i].ciendlow; o[7] = sv[i].ciendhigh; o[8] = sv[i].srSupport; o[9] = sv[i].srMapQuality; o[10] = sv[i].mapq; o[11] = sv[i].insLen;
    o[12] = sv[i].svt; o[13] = sv[i].id;
  }
  return (int) sv.size();
}

int dh_cluster_pe(const int32_t* rec11, int n, int svt, int minClique, int graphPruning, uint32_t varisize, int32_t* sv_out, int cap) {
  Config c; c.minCliqueSize = (uint16_t) minClique; c.graphPruning = graphPruning;
  std::vector<BamAlignRecord> v(n);
  for (int i = 0; i < n; ++i) {
    const int32_t* r = rec11 + 11 * i;
    v[i].tid = r[0]; v[i].pos = r[1]; v[i].mtid = r[2]; v[i].mpos = r[3]; v[i].alen = (uint16_t) r[4]; v[i].malen = (uint16_t) r[5];
    v[i].Median = r[6]; v[i].Mad = r[7]; v[i].maxNormalISize = r[8]; v[i].flag = (uint32_t) r[9]; v[i].MapQuality = (uint8_t) r[10];
  }
  std::vector<StructuralVariantRecord> sv;
  cluster(c, v, sv, varisize, svt);
  if ((int) sv.size() > cap) return -1;
  for (std::size_t i = 0; i < sv.size(); ++i) {
    int32_t* o = sv_out + 12 * i;
    o[0] = sv[i].chr; o[1] = sv[i].svStart; o[2] = sv[i].chr2; o[3] = sv[i].svEnd; o[4] = sv[i].ciposlow; o[5] = sv[i].ciposhigh;
    o[6] = sv[i].ciendlow; o[7] = sv[i].ciendhigh; o[8] = sv[i].peSupport; o[9] = sv[i].peMapQuality; o[10] = sv[i].mapq; o[11] = sv[i].svt;
  }
  return (int) sv.size();
}

// clusterGpu — same layouts as dh_cluster_sr / dh_cluster_pe, pair scan on the device
int dh_cluster_sr_gpu(dgpu_ctx* ctx, const int32_t* br8, const uint64_t* ids, int n, int svt, int minClique, int maxReadSep, int graphPruning, int nchr,
                      int32_t* svid_out, int32_t* sv_out, int cap) {
  Config c; c.minCliqueSize = (uint16_t) minClique; c.maxReadSep = maxReadSep; c.graphPruning = graphPruning; c.nchr = nchr;
  std::vector<SRBamRecord> br;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = br8 + 8 * i;
    br.push_back(SRBamRecord(r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], (std::size_t) ids[i]));
  }
  std::vector<StructuralVariantRecord> sv;
  int rc = clusterGpu(ctx, c, br, sv, svt);
  if (rc) return rc - 1;
  for (int i = 0; i < n; ++i) svid_out[i] = br[i].svid;
  if ((int) sv.size() > cap) return -1;
  for (std::size_t i = 0; i < sv.size(); ++i) {
    int32_t* o = sv_out + 14 * i;
    o[0] = sv[i].chr; o[1] = sv[i].svStart; o[2] = sv[i].chr2; o[3] = sv[i].svEnd; o[4] = sv[i].ciposlow; o[5] = sv[i].ciposhigh;
    o[6] = sv[i].ciendlow; o[7] = sv[i].ciendhigh; o[8] = sv[i].srSupport; o[9] = sv[i].srMapQuality; o[10] = sv[i].mapq; o[11] = sv[i].insLen;
    o[12] = sv[i].svt; o[13] = sv[i].id;
  }
  return (int) sv.size();
}

int dh_cluster_pe_gpu(dgpu_ctx* ctx, const int32_t* rec11, int n, int svt, int minClique, int graphPruning, uint32_t varisize, int32_t* sv_out, int cap) {
  Config c; c.minCliqueSize = (uint16_t) minClique; c.graphPruning = graphPruning;
  std::vector<BamAlignRecord> v(n);
  for (int i = 0; i < n; ++i) {
    const int32_t* r = rec11 + 11 * i;
    v[i].tid = r[0]; v[i].pos = r[1]; v[i].mtid = r[2]; v[i].mpos = r[3]; v[i].alen = (uint16_t) r[4]; v[i].malen = (uint16_t) r[5];
    v[i].Median = r[6]; v[i].Mad = r[7]; v[i].maxNormalISize = r[8]; v[i].flag = (uint32_t) r[9]; v[i].MapQuality = (uint8_t) r[10];
  }
  std::vector<StructuralVariantRecord> sv;
  int rc = clusterGpu(ctx, c, v, sv, varisize, svt);
  if (rc) return rc - 1;
  if ((int) sv.size() > cap) return -1;
  for (std::size_t i = 0; i < sv.size(); ++i) {
    int32_t* o = sv_out + 12 * i;
    o[0] = sv[i].chr; o[1] = sv[i].svStart; o[2] = sv[i].chr2; o[3] = sv[i].svEnd; o[4] = sv[i].ciposlow; o[5] = sv[i].ciposhigh;
    o[6] = sv[i].ciendlow; o[7] = sv[i].ciendhigh; o[8] = sv[i].peSupport; o[9] = sv[i].peMapQuality; o[10] = sv[i].mapq; o[11] = sv[i].svt;
  }
  return (int) sv.size();
}

// The per-record part of findJunctions (lr, src/junction.h:352-437) / of scanPEandSR's CIGAR scan (sr, src/shortpe.h:355-389)
// over a record list — layout as oracle/ref_wrap2.cpp::ref_find_junctions; seeds = the caller's read ids.
int dh_find_junctions(const int32_t* rec7, const uint64_t* seeds, int n, const uint32_t* cigar, int minMapQual, int minClip, int minRefSep,
                      float indelExtension, int lr, uint64_t* read_seed, uint32_t* read_off, int read_cap, int32_t* junc7, int junc_cap, int* n_reads) {
  std::map<std::size_t, TJunctionVector> readBp;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = rec7 + 7 * i;
    const uint32_t flag = (uint32_t) r[2];
    if (flag & (0x200 | 0x400 | 0x4)) continue;                 // BAM_FQCFAIL | BAM_FDUP | BAM_FUNMAP
    if ((r[3] < minMapQual) || (r[0] < 0)) continue;
    std::vector<std::pair<uint8_t, uint32_t> > cg;
    for (int k = 0; k < r[6]; ++k) cg.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    if (lr) cigarJunctionsLR(readBp, (std::size_t) seeds[i], flag, r[0], r[1], (uint8_t) r[3], cg, (uint32_t) minClip, (uint32_t) minRefSep, indelExtension);
    else cigarJunctions(readBp, (std::size_t) seeds[i], flag, r[0], r[1], (uint8_t) r[3], cg, (uint32_t) minClip, (uint32_t) minRefSep);
  }
  for (auto& kv : readBp) std::sort(kv.second.begin(), kv.second.end());   // src/junction.h:449
  int k = 0, pos = 0;
  read_off[0] = 0;
  for (auto const& kv : readBp) {
    if (k >= read_cap) return -1;
    read_seed[k] = kv.first;
    for (auto const& j : kv.second) {
      if (pos >= junc_cap) return -1;
      int32_t* o = junc7 + 7 * pos++;
      o[0] = j.forward; o[1] = j.scleft; o[2] = j.refidx; o[3] = j.rstart; o[4] = j.refpos; o[5] = j.seqpos; o[6] = j.qual;
    }
    read_off[++k] = (uint32_t) pos;
  }
  *n_reads = k;
  return pos;
}

int dh_select_junctions(const int32_t* junc7, const uint32_t* read_off, const uint64_t* read_id, int nreads, int maxReadSep, int minRefSep,
                        int32_t* out9, uint64_t* out_id, int cap, int32_t* out_cnt) {
  Config c; c.maxReadSep = maxReadSep; c.minRefSep = minRefSep;
  std::map<std::size_t, TJunctionVector> readBp;  // ascending read id, like the oracle wrapper
  for (int r = 0; r < nreads; ++r) {
    TJunctionVector v;
    for (uint32_t k = read_off[r]; k < read_off[r + 1]; ++k) {
      const int32_t* j = junc7 + 7 * k;
      v.push_back(Junction(j[0] != 0, j[1] != 0, j[2], j[3], j[4], j[5], (uint16_t) j[6]));
    }
    readBp.insert(std::make_pair((std::size_t) read_id[r], v));
  }
  TSvtSRBamRecord br(2 * DELLY_SVT_TRANS);
  fetchSVs(c, readBp, br);
  int pos = 0;
  for (int svt = 0; svt < 9; ++svt) {
    out_cnt[svt] = (int32_t) br[svt].size();
    for (auto const& x : br[svt]) {
      if (pos >= cap) return -1;
      int32_t* o = out9 + 9 * pos;
      o[0] = x.chr; o[1] = x.pos; o[2] = x.chr2; o[3] = x.pos2; o[4] = x.rstart; o[5] = x.sstart; o[6] = x.qual; o[7] = x.inslen; o[8] = x.primaryChr;
      out_id[pos] = x.id;
      ++pos;
    }
  }
  return pos;
}

// _getSVRef on a two-contig toy genome (layout as ref_get_sv_ref)
int dh_get_sv_ref(const char* seq, int seqlen, const char* sndSeq, int sndlen, const int32_t* sv_in, int conslen, int minimumFlankSize, int indelsize,
                  int minConsWindow, char* out, int cap, int* outlen) {
  Config c; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  std::vector<uint32_t> tl = {(uint32_t) seqlen, (uint32_t) sndlen};
  StructuralVariantRecord sv;
  sv.chr = sv_in[0]; sv.svStart = sv_in[1]; sv.chr2 = sv_in[2]; sv.svEnd = sv_in[3]; sv.svt = sv_in[4]; sv.insLen = sv_in[5];
  Breakpoint bp(sv);
  if (sv.svt == 4) _initBreakpoint(tl, bp, std::max((int32_t) ((conslen - sv.insLen) / 3), c.minimumFlankSize), sv.svt);
  else _initBreakpoint(tl, bp, conslen, sv.svt);
  if (bp.chr != bp.chr2) bp.part1 = _getSVRef(c, sndSeq, bp, bp.chr2, sv.svt);
  std::string s = _getSVRef(c, seq, bp, bp.chr, sv.svt);
  *outlen = (int) s.size();
  if ((int) s.size() > cap) return -1;
  memcpy(out, s.data(), s.size());
  return 0;
}

// _findSplit on a given 2-row alignment (layout as ref_find_split)
int dh_find_split(const char* cons, int m, const char* ref, int n, const char* rows, int L, int svt, float flankQuality, int minimumFlankSize,
                  int32_t* ad6, float* percId) {
  Config c; c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize;
  TAlign a(2);
  a[0].assign(rows, L); a[1].assign(rows + L, L);
  AlignDescriptor ad;
  bool ok = _findSplit(c, std::string(cons, m), std::string(ref, n), a, ad, svt);
  ad6[0] = ad.cStart; ad6[1] = ad.cEnd; ad6[2] = ad.rStart; ad6[3] = ad.rEnd; ad6[4] = ad.homLeft; ad6[5] = ad.homRight;
  *percId = ad.percId;
  return ok ? 1 : 0;
}

// _consRefAlignment for one (consensus, SV reference) pair: svt 4 -> splitAlign, else longNeedle; rows as the reference returns them
int dh_cons_ref_alignment(dgpu_ctx* ctx, const char* cons, int m, const char* ref, int n, int svt, char* rows, long cap, int* alilen) {
  *alilen = 0;
  if (svt == 4) {
    std::vector<uint8_t> ok; std::vector<TAlign> al;
    int rc = splitAlignBatch(ctx, std::vector<std::string>(1, std::string(cons, m)), std::vector<std::string>(1, std::string(ref, n)), ok, al);
    if (rc) return rc;
    if (al[0].size() == 2) {
      *alilen = (int) al[0][0].size();
      if (2l * *alilen > cap) return -100;
      memcpy(rows, al[0][1].data(), *alilen);            // swapped: row 0 = consensus (target of the glue), row 1 = reference
      memcpy(rows + *alilen, al[0][0].data(), *alilen);
    }
    return ok[0] ? 1 : 0;
  }
  return -101;
}

// splitAlign (src/split.h:480-537) over n insertion consensus / reference-window pairs of one arena; ok_out[i] = 1 if aligned, alilen_out[i] = columns
int dh_split_align_batch(dgpu_ctx* ctx, const char* arena, const uint32_t* cons_off, const uint32_t* cons_len, const uint32_t* ref_off, const uint32_t* ref_len, int n,
                         uint8_t* ok_out, int32_t* alilen_out) {
  std::vector<std::string> cons((size_t) n), refs((size_t) n);
  for (int i = 0; i < n; ++i) { cons[i].assign(arena + cons_off[i], cons_len[i]); refs[i].assign(arena + ref_off[i], ref_len[i]); }
  std::vector<uint8_t> ok; std::vector<TAlign> al;
  int rc = splitAlignBatch(ctx, cons, refs, ok, al);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) { ok_out[i] = ok[i]; alilen_out[i] = (al[i].size() == 2) ? (int32_t) al[i][0].size() : 0; }
  return 0;
}

int dh_longest_homology(const char* s1, int m, const char* s2, int n, int thr) { return longestHomology(std::string(s1, m), std::string(s2, n), thr); }

// alignConsensusBatch on the toy two-contig genome (seq = contig 0, sndSeq = contig 1): n SVs, sv_in n x 6, consensus arena;
// outputs as ref_align_consensus per SV.
int dh_align_consensus_batch(dgpu_ctx* ctx, const char* seq, int seqlen, const char* sndSeq, int sndlen, int n, const int32_t* sv_in,
                             const char* cons_arena, const uint32_t* cons_off, const uint32_t* cons_len, int realign, float flankQuality,
                             int minimumFlankSize, int indelsize, int minConsWindow, int32_t* sv_out, float* srq, char* alleles, int alleles_stride,
                             int32_t* alleles_len, char* cons_out, int cons_stride, int32_t* cons_out_len, uint8_t* ok_out) {
  Config c; c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  std::vector<uint32_t> tl = {(uint32_t) seqlen, (uint32_t) sndlen};
  std::vector<const char*> chr = {seq, sndSeq};
  std::vector<StructuralVariantRecord> svs(n);
  for (int i = 0; i < n; ++i) {
    const int32_t* s = sv_in + 6 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5];
    svs[i].consensus.assign(cons_arena + cons_off[i], cons_len[i]);
  }
  std::vector<uint8_t> ok;
  int rc = alignConsensusBatch(ctx, c, tl, chr, svs, realign != 0, ok);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    int32_t* o = sv_out + 10 * i;
    StructuralVariantRecord const& sv = svs[i];
    o[0] = sv.svStart; o[1] = sv.svEnd; o[2] = sv.insLen; o[3] = sv.consBp; o[4] = sv.homLen; o[5] = sv.ciposlow; o[6] = sv.ciposhigh;
    o[7] = sv.ciendlow; o[8] = sv.ciendhigh; o[9] = sv.precise ? 1 : 0;
    srq[i] = sv.srAlignQuality;
    alleles_len[i] = (int32_t) sv.alleles.size();
    memcpy(alleles + (size_t) i * alleles_stride, sv.alleles.data(), std::min<size_t>(sv.alleles.size(), alleles_stride));
    cons_out_len[i] = (int32_t) sv.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, sv.consensus.data(), std::min<size_t>(sv.consensus.size(), cons_stride));
    ok_out[i] = ok[i];
  }
  return 0;
}

// generateProbesBatch — layout as oracle/ref_wrap3.cpp::ref_generate_probes (contig 0 "chrA", contig 1 "chrB").
// Returns the number of regions, -1 on capacity, -2 if some probe cut fell outside its string, < -2 device error.
int dh_generate_probes(dgpu_ctx* ctx, const char* seq0, int len0, const char* seq1, int len1, int n, const int32_t* sv_in, const uint8_t* cons_arena,
                       const uint32_t* cons_off, const uint32_t* cons_len, float flankQuality, int minimumFlankSize, int indelsize,
                       int minConsWindow, uint8_t* arena, uint64_t arena_cap, uint64_t* p_off, uint32_t* p_len, int32_t* regions, int cap,
                       uint8_t* alleles, int32_t* alleles_len, uint8_t* svOnChrOut) {
  Config c; c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  std::vector<uint32_t> tl = {(uint32_t) len0, (uint32_t) len1};
  std::vector<std::string> names = {"chrA", "chrB"};
  std::vector<const char*> chr = {seq0, seq1};
  std::vector<StructuralVariantRecord> svs(n);
  for (int i = 0; i < n; ++i) {
    const int32_t* s = sv_in + 8 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5];
    svs[i].precise = s[6] != 0; svs[i].id = s[7];
    svs[i].consensus.assign((const char*) cons_arena + cons_off[i], cons_len[i]);
  }
  std::vector<std::vector<std::string> > refProbeArr, consProbeArr;
  std::vector<std::vector<BpRegion> > bpRegion;
  std::vector<bool> svOnChr;
  std::vector<uint32_t> bad;
  int rc = generateProbesBatch(ctx, c, tl, names, chr, svs, refProbeArr, consProbeArr, bpRegion, svOnChr, bad);
  if (rc) return rc - 2;
  if (!bad.empty()) return -2;
  uint64_t pos = 0;
  for (int i = 0; i < n; ++i) {
    const std::string* p[4] = {&consProbeArr[0][i], &refProbeArr[0][i], &consProbeArr[1][i], &refProbeArr[1][i]};
    for (int k = 0; k < 4; ++k) {
      if (pos + p[k]->size() > arena_cap) return -1;
      p_off[4 * i + k] = pos; p_len[4 * i + k] = (uint32_t) p[k]->size();
      memcpy(arena + pos, p[k]->data(), p[k]->size());
      pos += p[k]->size();
    }
    alleles_len[i] = (int32_t) svs[i].alleles.size();
    memcpy(alleles + 256 * (size_t) i, svs[i].alleles.data(), std::min<std::size_t>(256, svs[i].alleles.size()));
  }
  int r = 0;
  for (int k = 0; k < 2; ++k) {
    svOnChrOut[k] = svOnChr[k] ? 1 : 0;
    for (auto const& b : bpRegion[k]) {
      if (r >= cap) return -1;
      int32_t* o = regions + 9 * r++;
      o[0] = k; o[1] = b.regionStart; o[2] = b.regionEnd; o[3] = b.bppos; o[4] = b.homLeft; o[5] = b.homRight; o[6] = b.svt; o[7] = (int32_t) b.id; o[8] = b.bpPoint;
    }
  }
  return r;
}

// annotateJunctionReadsBatch — layout as oracle/ref_wrap3.cpp::ref_annotate_junction_reads
int dh_annotate_junction_reads(dgpu_ctx* ctx, const char* seq0, int len0, const char* seq1, int len1, const int32_t* rec10, int nrec, const uint32_t* cigar,
                               const char* reads, const int32_t* sv9, int nsv, const uint8_t* cons_arena, const uint32_t* cons_off, const uint32_t* cons_len,
                               float flankQuality, int minimumFlankSize, int indelsize, int minConsWindow, int minGenoQual, int maxGenoReadCount, int maxThreads,
                               uint8_t* qual_out, int qual_cap, uint32_t* ref_off, uint32_t* alt_off) {
  Config c; c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  c.minGenoQual = (uint16_t) minGenoQual; c.maxGenoReadCount = (uint32_t) maxGenoReadCount; c.maxThreads = (uint32_t) maxThreads;
  std::vector<uint32_t> tl = {(uint32_t) len0, (uint32_t) len1};
  std::vector<std::string> names = {"chrA", "chrB"};
  std::vector<const char*> chr = {seq0, seq1};
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec10 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
  }
  std::vector<StructuralVariantRecord> svs(nsv);
  for (int i = 0; i < nsv; ++i) {
    const int32_t* s = sv9 + 9 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5];
    svs[i].precise = s[6] != 0; svs[i].id = s[7]; svs[i].peSupport = s[8];
    svs[i].consensus.assign((const char*) cons_arena + cons_off[i], cons_len[i]);
  }
  std::vector<JunctionCount> countMap;
  int rc = annotateJunctionReadsBatch(ctx, c, tl, names, chr, svs, recs, countMap);
  if (rc) return rc - 2;
  int pos = 0;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t* off = pass ? alt_off : ref_off;
    for (int i = 0; i < nsv; ++i) {
      off[i] = (uint32_t) pos;
      std::vector<uint8_t> const& v = pass ? countMap[i].alt : countMap[i].ref;
      if (pos + (int) v.size() > qual_cap) return -1;
      for (uint8_t q : v) qual_out[pos++] = q;
    }
    off[nsv] = (uint32_t) pos;
  }
  return pos;
}

// annotateSpanningAndDepth — the spanning-pair / read-depth outputs of oracle/ref_wrap3.cpp::ref_annotate_junction_reads (pure host).
// svOnChr is derived like _generateProbes does (src/coverage.h:179): a contig carries an SV end.
int dh_annotate_spanning(int len0, int len1, const int32_t* rec12, int nrec, const uint32_t* cigar, const int32_t* sv9, int nsv, int indelsize, int minGenoQual,
                         const int32_t* lib4, uint8_t* span_out, int span_cap, uint32_t* sref_off, uint32_t* salt_off, int32_t* rc_out) {
  Config c; c.indelsize = indelsize; c.minGenoQual = (uint16_t) minGenoQual;
  LibraryInfo lib; lib.median = lib4[0]; lib.minNormalISize = lib4[1]; lib.maxNormalISize = lib4[2]; lib.maxISizeCutoff = lib4[3];
  std::vector<uint32_t> tl = {(uint32_t) len0, (uint32_t) len1};
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
  }
  std::vector<StructuralVariantRecord> svs(nsv);
  std::vector<bool> svOnChr(2, false);
  for (int i = 0; i < nsv; ++i) {
    const int32_t* s = sv9 + 9 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5];
    svs[i].precise = s[6] != 0; svs[i].id = s[7]; svs[i].peSupport = s[8];
    svOnChr[s[0]] = true; svOnChr[s[2]] = true;
  }
  std::vector<ReadCount> cov; std::vector<SpanningCount> span;
  annotateSpanningAndDepth(c, lib, tl, svs, svOnChr, recs, cov, span);
  int sp = 0;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t* off = pass ? salt_off : sref_off;
    for (int i = 0; i < nsv; ++i) {
      off[i] = (uint32_t) sp;
      std::vector<uint8_t> const& v = pass ? span[i].alt : span[i].ref;
      if (sp + (int) v.size() > span_cap) return -1;
      for (uint8_t q : v) span_out[sp++] = q;
    }
    off[nsv] = (uint32_t) sp;
  }
  for (int i = 0; i < nsv; ++i) { rc_out[3 * i] = cov[i].leftRC; rc_out[3 * i + 1] = cov[i].rc; rc_out[3 * i + 2] = cov[i].rightRC; }
  return sp;
}

// assembleSplitReadsBatch — layout as oracle/ref_wrap5.cpp::ref_assemble_split_reads
int dh_assemble_split_reads(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                            int nrec, const uint32_t* cigar, const char* reads, const int32_t* store5, int nstore, const int32_t* sv7, int nsv, int maxReadPerSV,
                            int minMapQual, int minCliqueSize, float flankQuality, int minimumFlankSize, int indelsize, int minConsWindow, int32_t* sv_out,
                            float* srq, char* cons_out, int cons_stride, int32_t* cons_len, char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  Config c; c.maxReadPerSV = (uint32_t) maxReadPerSV; c.minMapQual = (uint16_t) minMapQual; c.minCliqueSize = (uint16_t) minCliqueSize;
  c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  std::vector<uint32_t> tl; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
  }
  std::vector<StructuralVariantRecord> svs(nsv);
  for (int i = 0; i < nsv; ++i) {
    const int32_t* s = sv7 + 7 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5]; svs[i].id = s[6];
    svs[i].precise = false;
  }
  std::vector<TPosReadSV> srStore(ncontig);
  for (int i = 0; i < nstore; ++i) {
    const int32_t* e = store5 + 5 * i;
    srStore[e[0]].insert(std::make_pair(std::make_pair(e[1], (std::size_t) e[2] * 2 + (e[3] ? 1 : 0)), e[4]));
  }
  int rc = assembleSplitReadsBatch(ctx, c, tl, chr, srStore, svs, recs);
  if (rc) return rc;
  for (int i = 0; i < nsv; ++i) {
    StructuralVariantRecord const& sv = svs[i];
    int32_t* o = sv_out + 13 * i;
    o[0] = sv.svStart; o[1] = sv.svEnd; o[2] = sv.srSupport; o[3] = sv.mapq; o[4] = sv.srMapQuality; o[5] = sv.insLen; o[6] = sv.homLen; o[7] = sv.consBp;
    o[8] = sv.precise ? 1 : 0; o[9] = sv.ciposlow; o[10] = sv.ciposhigh; o[11] = sv.ciendlow; o[12] = sv.ciendhigh;
    srq[i] = sv.srAlignQuality;
    cons_len[i] = (int32_t) sv.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, sv.consensus.data(), std::min<size_t>(sv.consensus.size(), cons_stride));
    alleles_len[i] = (int32_t) sv.alleles.size();
    memcpy(alleles_out + (size_t) i * alleles_stride, sv.alleles.data(), std::min<size_t>(sv.alleles.size(), alleles_stride));
  }
  return 0;
}

// scanPEandSRBatch — layout as oracle/ref_wrap5.cpp::ref_scan_pe_sr; seeds / nameHash per record from the caller
// (ctx may be NULL: host pair scans)
int dh_scan_pe_sr(dgpu_ctx* ctx, const uint32_t* contig_len, int ncontig, const int32_t* rec12, const uint64_t* seeds, const uint32_t* name_hash, int nrec,
                  const uint32_t* cigar, const int32_t* lib5, int minMapQual, int minTraQual, int minClip, int minRefSep, int maxReadSep, int minCliqueSize,
                  int graphPruning, int32_t* pe_out, int32_t* sr_out, int cap, int32_t* store_out, uint64_t* store_seed, int store_cap, int32_t* n_out,
                  uint32_t* abnormal_pairs) {
  Config c; c.minMapQual = (uint16_t) minMapQual; c.minTraQual = (uint16_t) minTraQual; c.minClip = (uint32_t) minClip; c.minRefSep = (uint32_t) minRefSep;
  c.maxReadSep = (uint32_t) maxReadSep; c.minCliqueSize = (uint16_t) minCliqueSize; c.graphPruning = (uint32_t) graphPruning; c.nchr = ncontig;
  LibraryInfo lib; lib.rs = lib5[0]; lib.median = lib5[1]; lib.mad = lib5[2]; lib.maxNormalISize = lib5[3]; lib.maxISizeCutoff = lib5[4];
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
    recs[i].seed = (std::size_t) seeds[i]; recs[i].nameHash32 = name_hash[i];
  }
  std::vector<StructuralVariantRecord> svs, srSVs;
  std::vector<TPosReadSV> srStore;
  int rc = scanPEandSRBatch(ctx, c, lib, tl, recs, svs, srSVs, srStore);
  if (rc) return rc - 1;
  if ((int) svs.size() > cap || (int) srSVs.size() > cap) return -1;
  for (std::size_t i = 0; i < svs.size(); ++i) {
    int32_t* o = pe_out + 12 * i; StructuralVariantRecord const& v = svs[i];
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.peMapQuality; o[10] = v.mapq; o[11] = v.svt;
  }
  for (std::size_t i = 0; i < srSVs.size(); ++i) {
    int32_t* o = sr_out + 14 * i; StructuralVariantRecord const& v = srSVs[i];
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.srSupport; o[9] = v.srMapQuality; o[10] = v.mapq; o[11] = v.insLen; o[12] = v.svt; o[13] = v.id;
  }
  int k = 0;
  for (int t = 0; t < ncontig; ++t)
    for (auto const& kv : srStore[t]) {
      if (k >= store_cap) return -1;
      store_out[3 * k] = t; store_out[3 * k + 1] = kv.first.first; store_out[3 * k + 2] = kv.second; store_seed[k] = (uint64_t) kv.first.second;
      ++k;
    }
  n_out[0] = (int32_t) svs.size(); n_out[1] = (int32_t) srSVs.size(); n_out[2] = k;
  *abnormal_pairs = lib.abnormal_pairs;
  return 0;
}

// mergeSort — layout as oracle/ref_wrap5.cpp::ref_merge_sort
int dh_merge_sort(const int32_t* pe20, int npe, const int32_t* sr20, int nsr, int32_t* out20, int cap) {
  auto load = [](const int32_t* r) {
    StructuralVariantRecord v;
    v.chr = r[0]; v.svStart = r[1]; v.chr2 = r[2]; v.svEnd = r[3]; v.ciposlow = r[4]; v.ciposhigh = r[5]; v.ciendlow = r[6]; v.ciendhigh = r[7];
    v.peSupport = r[8]; v.srSupport = r[9]; v.peMapQuality = r[10]; v.srMapQuality = r[11]; v.mapq = r[12]; v.insLen = r[13]; v.homLen = r[14]; v.svt = r[15];
    v.precise = r[16] != 0; v.consBp = r[17]; v.consensus = std::to_string(r[18]); v.srAlignQuality = (float) r[19] / 1000.0f;
    return v;
  };
  std::vector<StructuralVariantRecord> pe, sr;
  for (int i = 0; i < npe; ++i) pe.push_back(load(pe20 + 20 * i));
  for (int i = 0; i < nsr; ++i) sr.push_back(load(sr20 + 20 * i));
  mergeSort(pe, sr);
  if ((int) pe.size() > cap) return -1;
  for (std::size_t i = 0; i < pe.size(); ++i) {
    int32_t* o = out20 + 20 * i; StructuralVariantRecord const& v = pe[i];
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.consensus.empty() ? -1 : std::stoi(v.consensus); o[19] = (int32_t) std::lround(v.srAlignQuality * 1000.0f);
  }
  return (int) pe.size();
}

// dellySrCall — layout as oracle/ref_wrap5.cpp::ref_delly_sr_call
// `-t`: SV types of the following chain hooks (bit svt = wanted; 0 = all), as oracle/ref_wrap5.cpp::ref_set_svtset
static uint32_t g_svtmask = 0;
void dh_set_svtset(uint32_t mask) { g_svtmask = mask; }
static void apply_svtset(Config& c) { for (int b = 0; b < 10; ++b) if (g_svtmask & (1u << b)) c.svtset.insert(b); }

// flat site rows -> VcfSite (layout: oracle/ref_wrap7.cpp::ref_vcf_parse)
static std::vector<VcfSite> sites_from_rows(const int32_t* site22, int nsite, const char* strs, const uint32_t* str_off) {
  std::vector<VcfSite> sites((size_t) nsite);
  for (int i = 0; i < nsite; ++i) {
    const int32_t* r = site22 + 22 * i; VcfSite& s = sites[i];
    const uint32_t mask = (uint32_t) r[3];
    auto has = [&](int bit) { return (mask >> bit) & 1u; };
    auto str = [&](int k) { return std::string(strs + str_off[7 * i + k], strs + str_off[7 * i + k + 1]); };
    s.chrom = "chr" + std::to_string(r[0]); s.pos0 = r[1]; memcpy(&s.qual, r + 2, 4); s.precise = r[21] != 0;
    s.ref = str(0); s.alt = str(1);
    s.svMethod.present = has(0); s.svMethod.value = str(2); s.svType.present = has(1); s.svType.value = str(3); s.ct.present = has(2); s.ct.value = str(4);
    s.chr2.present = has(9); s.chr2.value = str(5); s.consensus.present = has(11); s.consensus.value = str(6);
    s.pe.present = has(3); s.pe.value = r[4]; s.insLen.present = has(4); s.insLen.value = r[5]; s.svLen.present = has(5); s.svLen.value = r[6];
    s.homLen.present = has(6); s.homLen.value = r[7]; s.sr.present = has(7); s.sr.value = r[8]; s.end.present = has(8); s.end.value = r[9];
    s.pos2.present = has(10); s.pos2.value = r[10]; s.consBp.present = has(12); s.consBp.value = r[11];
    s.hasCipos = has(13); s.cipos[0] = r[12]; s.cipos[1] = r[13]; s.hasCiend = has(14); s.ciend[0] = r[14]; s.ciend[1] = r[15];
    s.mapq.present = has(15); s.mapq.value = r[16]; s.srMapq.present = has(16); s.srMapq.value = r[17];
    s.srq.present = has(17); memcpy(&s.srq.value, r + 18, 4);
    s.alleleId.present = has(18); s.alleleId.value = r[19]; s.nAllele.present = has(19); s.nAllele.value = r[20];
  }
  return sites;
}

// vcfParseSites — layout as oracle/ref_wrap7.cpp::ref_vcf_parse
int dh_vcf_parse(int ncontig, const int32_t* site22, int nsite, const char* strs, const uint32_t* str_off, int headerHasConsBp, int32_t* sv_out, int cap,
                 char* alleles_out, int astride, int32_t* alen, char* cons_out, int cstride, int32_t* clen) {
  std::vector<std::string> names;
  for (int k = 0; k < ncontig; ++k) names.push_back("chr" + std::to_string(k));
  std::vector<StructuralVariantRecord> svs;
  vcfParseSites(sites_from_rows(site22, nsite, strs, str_off), headerHasConsBp != 0, names, svs);
  const int n = (int) svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = svs[i];
    int32_t* o = sv_out + 22 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; memcpy(o + 19, &v.srAlignQuality, 4); o[20] = v.alleleid; o[21] = v.nallele;
    alen[i] = (int32_t) v.alleles.size(); memcpy(alleles_out + (size_t) i * astride, v.alleles.data(), std::min<size_t>(v.alleles.size(), astride));
    clen[i] = (int32_t) v.consensus.size(); memcpy(cons_out + (size_t) i * cstride, v.consensus.data(), std::min<size_t>(v.consensus.size(), cstride));
  }
  return n;
}

static int delly_sr_hook(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, const uint32_t* name_hash, int nrec, const uint32_t* cigar, const char* reads, const int32_t* lib6, int32_t* sv_out,
                     int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const int32_t* site22, int nsite,
                     const char* strs, const uint32_t* str_off) {
  Config c;   // short-read defaults (src/delly.h:212-232)
  c.nchr = ncontig; c.maxThreads = 1;
  apply_svtset(c);
  LibraryInfo lib; lib.rs = lib6[0]; lib.median = lib6[1]; lib.mad = lib6[2]; lib.minNormalISize = lib6[3]; lib.maxNormalISize = lib6[4]; lib.maxISizeCutoff = lib6[5];
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
    recs[i].seed = (std::size_t) seeds[i]; recs[i].nameHash32 = name_hash[i];
  }
  SrCallSet cs;
  int rc = site22 ? dellySrGenotype(ctx, c, lib, tl, names, chr, sites_from_rows(site22, nsite, strs, str_off), true, recs, cs)
                  : dellySrCall(ctx, c, lib, tl, names, chr, recs, cs);
  if (rc) return rc - 1;
  const int n = (int) cs.svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    int32_t* o = sv_out + 20 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; o[19] = 0;
    memcpy(o + 19, &v.srAlignQuality, 4);
    SampleFormat const& f = cs.format[i];
    int32_t* q = fmt_out + 14 * i;
    q[0] = f.gt[0]; q[1] = f.gt[1]; q[2] = f.gq; q[3] = f.pl[0]; q[4] = f.pl[1]; q[5] = f.pl[2]; q[6] = f.rcn; q[7] = f.pass ? 1 : 0;
    q[8] = (int32_t) cs.spanMap[i].ref.size(); q[9] = (int32_t) cs.spanMap[i].alt.size(); q[10] = (int32_t) cs.jctMap[i].ref.size(); q[11] = (int32_t) cs.jctMap[i].alt.size();
    q[12] = cs.rcMap[i].rc; q[13] = cs.rcMap[i].leftRC + cs.rcMap[i].rightRC;
    for (int k = 0; k < 3; ++k) gl_out[3 * i + k] = f.gl[k];
    cons_len[i] = (int32_t) v.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, v.consensus.data(), std::min<size_t>(v.consensus.size(), cons_stride));
  }
  return n;
}

int dh_delly_sr_call(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, const uint32_t* name_hash, int nrec, const uint32_t* cigar, const char* reads, const int32_t* lib6, int32_t* sv_out,
                     int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return delly_sr_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, nrec, cigar, reads, lib6, sv_out, cap, fmt_out, gl_out, cons_out,
                       cons_stride, cons_len, nullptr, 0, nullptr, nullptr);
}

// several samples in one call set — layout as oracle/ref_wrap5.cpp::ref_delly_sr_call_multi (records grouped by file, fmt_out / gl_out file-major)
static int delly_sr_multi_hook(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                           const uint64_t* seeds, const uint32_t* name_hash, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads,
                           const int32_t* lib6, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len,
                           const int32_t* site22, int nsite, const char* strs, const uint32_t* str_off) {
  Config c;
  c.nchr = ncontig; c.maxThreads = 1;
  apply_svtset(c);
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<LibraryInfo> libs((size_t) nfile);
  std::vector<std::vector<SrRecord> > recs((size_t) nfile);
  std::vector<std::vector<SrRecord> const*> samples;
  for (int f = 0; f < nfile; ++f) {
    const int32_t* l = lib6 + 6 * f;
    libs[f].rs = l[0]; libs[f].median = l[1]; libs[f].mad = l[2]; libs[f].minNormalISize = l[3]; libs[f].maxNormalISize = l[4]; libs[f].maxISizeCutoff = l[5];
    for (uint32_t i = file_off[f]; i < file_off[f + 1]; ++i) {
      const int32_t* r = rec12 + 12 * (size_t) i;
      SrRecord rec;
      rec.tid = r[0]; rec.pos = r[1]; rec.flag = (uint32_t) r[2]; rec.mapq = (uint8_t) r[3];
      for (int k = 0; k < r[6]; ++k) rec.cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
      rec.seq.assign(reads + r[7], (std::size_t) r[4]);
      rec.lqseq = r[4]; rec.mtid = r[8]; rec.mpos = r[9]; rec.isize = r[10]; rec.name = (uint64_t) r[11];
      rec.seed = (std::size_t) seeds[i]; rec.nameHash32 = name_hash[i];
      recs[f].push_back(rec);
    }
  }
  for (int f = 0; f < nfile; ++f) samples.push_back(&recs[f]);
  SrMultiCallSet cs;
  int rc = site22 ? dellySrGenotypeMulti(ctx, c, libs, tl, names, chr, sites_from_rows(site22, nsite, strs, str_off), true, samples, cs)
                  : dellySrCallMulti(ctx, c, libs, tl, names, chr, samples, cs);
  if (rc) return rc - 1;
  const int n = (int) cs.svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    int32_t* o = sv_out + 20 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; o[19] = 0;
    memcpy(o + 19, &v.srAlignQuality, 4);
    for (int f = 0; f < nfile; ++f) {
      SrSampleCounts const& sc = cs.sample[f];
      SampleFormat const& fm = sc.format[i];
      int32_t* q = fmt_out + 14 * ((size_t) f * cap + i);
      q[0] = fm.gt[0]; q[1] = fm.gt[1]; q[2] = fm.gq; q[3] = fm.pl[0]; q[4] = fm.pl[1]; q[5] = fm.pl[2]; q[6] = fm.rcn; q[7] = fm.pass ? 1 : 0;
      q[8] = (int32_t) sc.spanMap[i].ref.size(); q[9] = (int32_t) sc.spanMap[i].alt.size(); q[10] = (int32_t) sc.jctMap[i].ref.size(); q[11] = (int32_t) sc.jctMap[i].alt.size();
      q[12] = sc.rcMap[i].rc; q[13] = sc.rcMap[i].leftRC + sc.rcMap[i].rightRC;
      for (int k = 0; k < 3; ++k) gl_out[3 * ((size_t) f * cap + i) + k] = fm.gl[k];
    }
    cons_len[i] = (int32_t) v.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, v.consensus.data(), std::min<size_t>(v.consensus.size(), cons_stride));
  }
  return n;
}

int dh_delly_sr_call_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                           const uint64_t* seeds, const uint32_t* name_hash, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads,
                           const int32_t* lib6, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return delly_sr_multi_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, file_off, nfile, cigar, reads, lib6, sv_out, cap, fmt_out, gl_out,
                             cons_out, cons_stride, cons_len, nullptr, 0, nullptr, nullptr);
}
// genotyping mode over several samples (site rows as dh_vcf_parse)
int dh_delly_sr_genotype_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                               const uint64_t* seeds, const uint32_t* name_hash, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads,
                               const int32_t* lib6, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len,
                               const int32_t* site22, int nsite, const char* strs, const uint32_t* str_off) {
  return delly_sr_multi_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, file_off, nfile, cigar, reads, lib6, sv_out, cap, fmt_out, gl_out,
                             cons_out, cons_stride, cons_len, site22, nsite, strs, str_off);
}

// genotyping mode: the same outputs for a given site list (rows as dh_vcf_parse) instead of discovery
int dh_delly_sr_genotype(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                         const uint64_t* seeds, const uint32_t* name_hash, int nrec, const uint32_t* cigar, const char* reads, const int32_t* lib6, int32_t* sv_out,
                         int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const int32_t* site22, int nsite,
                         const char* strs, const uint32_t* str_off) {
  return delly_sr_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, nrec, cigar, reads, lib6, sv_out, cap, fmt_out, gl_out, cons_out,
                       cons_stride, cons_len, site22, nsite, strs, str_off);
}

// assembleLRBatch — layout as oracle/ref_wrap5.cpp::ref_assemble_lr (read id = name id here)
int dh_assemble_lr(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec,
                   const uint32_t* cigar, const char* reads, const int32_t* store6, int nstore, const int32_t* sv12, int nsv, int maxReadPerSV, int minCliqueSize,
                   float flankQuality, int minimumFlankSize, int indelsize, int minConsWindow, int32_t* sv_out, float* srq, char* cons_out, int cons_stride,
                   int32_t* cons_len, char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  Config c; c.maxReadPerSV = (uint32_t) maxReadPerSV; c.minCliqueSize = (uint16_t) minCliqueSize;
  c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  std::vector<uint32_t> tl; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<LrRecord> recs(nrec);
  std::vector<std::size_t> ids(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    ids[i] = (std::size_t) r[11];
  }
  std::vector<StructuralVariantRecord> svs(nsv);
  for (int i = 0; i < nsv; ++i) {
    const int32_t* s = sv12 + 12 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5]; svs[i].id = s[6];
    svs[i].srSupport = s[7]; svs[i].ciposlow = s[8]; svs[i].ciposhigh = s[9]; svs[i].ciendlow = s[10]; svs[i].ciendhigh = s[11];
    svs[i].precise = false;
  }
  std::vector<TPosReadSlices> srStore(ncontig);
  for (int i = 0; i < nstore; ++i) {
    const int32_t* e = store6 + 6 * i;
    srStore[e[0]][std::make_pair(e[1], (std::size_t) e[2])].push_back(SeqSlice(e[3], e[4], e[5], 60));
  }
  int rc = assembleLRBatch(ctx, c, tl, chr, svs, srStore, recs, ids);
  if (rc) return rc;
  for (int i = 0; i < nsv; ++i) {
    StructuralVariantRecord const& sv = svs[i];
    int32_t* o = sv_out + 13 * i;
    o[0] = sv.svStart; o[1] = sv.svEnd; o[2] = sv.srSupport; o[3] = sv.mapq; o[4] = sv.srMapQuality; o[5] = sv.insLen; o[6] = sv.homLen; o[7] = sv.consBp;
    o[8] = sv.precise ? 1 : 0; o[9] = sv.ciposlow; o[10] = sv.ciposhigh; o[11] = sv.ciendlow; o[12] = sv.ciendhigh;
    srq[i] = sv.srAlignQuality;
    cons_len[i] = (int32_t) sv.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, sv.consensus.data(), std::min<size_t>(sv.consensus.size(), cons_stride));
    alleles_len[i] = (int32_t) sv.alleles.size();
    memcpy(alleles_out + (size_t) i * alleles_stride, sv.alleles.data(), std::min<size_t>(sv.alleles.size(), alleles_stride));
  }
  return 0;
}

// dellyLrCall — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call; seeds = the read ids (hash_lr of the query names)
// set (per thread) by the sharded test hook: the chain then runs as one rank of a sharded run
static thread_local Shard const* g_lr_shard = nullptr;

static int delly_lr_call_hook(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, int nrec, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, float indelExtension,
                     int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const uint8_t* tagflags,
                     const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off, int methylWindow, int methylProb,
                     int minCpgDepth, const char* tpl_arena, const uint32_t* tpl_off, float meiMinFrac, float trMinFrac, int32_t* anno_out, int32_t* methyl_out,
                     char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  Config c;
  c.minMapQual = (uint16_t) cfg12[0]; c.minClip = (uint32_t) cfg12[1]; c.minRefSep = (uint32_t) cfg12[2]; c.maxReadSep = (uint32_t) cfg12[3];
  c.minCliqueSize = (uint16_t) cfg12[4]; c.graphPruning = (uint32_t) cfg12[5]; c.maxReadPerSV = (uint32_t) cfg12[6]; c.minimumFlankSize = cfg12[7];
  c.indelsize = cfg12[8]; c.minConsWindow = cfg12[9]; c.maxGenoReadCount = (uint32_t) cfg12[10]; c.genoCap = cfg12[11];
  c.flankQuality = flankQuality; c.nchr = ncontig;
  apply_svtset(c);
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<LrRecord> recs(nrec);
  std::vector<std::size_t> ids(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    ids[i] = (std::size_t) seeds[i];
    if (tagflags && (tagflags[i] & 1)) { recs[i].hasMM = true; recs[i].mm.assign(mm_arena + mm_off[i], mm_arena + mm_off[i + 1]); }
    if (tagflags && (tagflags[i] & 2)) { recs[i].hasML = true; recs[i].ml.assign(ml_arena + ml_off[i], ml_arena + ml_off[i + 1]); }
  }
  LrCallSet cs;
  MeiTemplates mei;
  AnnoConfig acfg; acfg.meiMinFrac = meiMinFrac; acfg.trMinFrac = trMinFrac;
  MethylConfig mcfg; mcfg.methylWindow = methylWindow; mcfg.methylProb = (uint16_t) methylProb; mcfg.minCpgDepth = (uint32_t) minCpgDepth;
  if (tpl_arena) {
    for (int t = 1; t <= 6; ++t) mei.seq[t].assign(tpl_arena + tpl_off[t - 1], tpl_arena + tpl_off[t]);
    mei.polyA.assign(tpl_arena + tpl_off[6], tpl_arena + tpl_off[7]);
  }
  int rc;
  if (g_lr_shard) {
    LrMultiCallSet ms;
    std::vector<LrSample> samples(1, LrSample{&recs, &ids});
    rc = dellyLrCallSharded(ctx, c, indelExtension, tl, names, chr, samples, *g_lr_shard, ms, tpl_arena ? &mei : nullptr, acfg, tagflags ? &mcfg : nullptr);
    if (!rc) { cs.svs.swap(ms.svs); cs.jctMap.swap(ms.sample[0].jctMap); cs.rcMap.swap(ms.sample[0].rcMap); cs.format.swap(ms.sample[0].format); cs.methyl.swap(ms.sample[0].methyl); }
  } else rc = dellyLrCall(ctx, c, indelExtension, tl, names, chr, recs, ids, cs, tpl_arena ? &mei : nullptr, acfg, tagflags ? &mcfg : nullptr);
  if (rc) return rc - 1;
  const int n = (int) cs.svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    int32_t* o = sv_out + 20 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; o[19] = 0;
    memcpy(o + 19, &v.srAlignQuality, 4);
    SampleFormat const& f = cs.format[i];
    int32_t* q = fmt_out + 14 * i;
    q[0] = f.gt[0]; q[1] = f.gt[1]; q[2] = f.gq; q[3] = f.pl[0]; q[4] = f.pl[1]; q[5] = f.pl[2]; q[6] = f.rcn; q[7] = f.pass ? 1 : 0;
    q[8] = 0; q[9] = 0; q[10] = (int32_t) cs.jctMap[i].ref.size(); q[11] = (int32_t) cs.jctMap[i].alt.size();
    q[12] = cs.rcMap[i].rc; q[13] = cs.rcMap[i].leftRC + cs.rcMap[i].rightRC;
    for (int k = 0; k < 3; ++k) gl_out[3 * i + k] = f.gl[k];
    cons_len[i] = (int32_t) v.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, v.consensus.data(), std::min<size_t>(v.consensus.size(), cons_stride));
    if (anno_out) {
      int32_t* a = anno_out + 5 * i;
      a[0] = v.anno.isRC ? 1 : 0; a[1] = v.anno.seqType; a[2] = v.anno.homLen; a[3] = v.anno.trPeriod; memcpy(a + 4, &v.anno.trCopies, 4);
    }
    if (methyl_out && !cs.methyl.empty()) {
      MethylInfo const& mi = cs.methyl[v.id];
      memcpy(methyl_out + 16 * i, mi.alt, 16); memcpy(methyl_out + 16 * i + 4, mi.ref, 16); memcpy(methyl_out + 16 * i + 8, mi.mnc, 16); memcpy(methyl_out + 16 * i + 12, mi.mdp, 16);
    }
    if (alleles_out) {
      alleles_len[i] = (int32_t) v.alleles.size();
      memcpy(alleles_out + (size_t) i * alleles_stride, v.alleles.data(), std::min<size_t>(v.alleles.size(), alleles_stride));
    }
  }
  return n;
}

int dh_delly_lr_call(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, int nrec, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, float indelExtension,
                     int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return delly_lr_call_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, nrec, cigar, reads, cfg12, flankQuality, indelExtension, sv_out, cap, fmt_out,
                            gl_out, cons_out, cons_stride, cons_len, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nullptr, nullptr, 0.f, 0.f, nullptr, nullptr,
                            nullptr, 0, nullptr);
}

// the complete long-read chain — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call_ex plus the template sequences
int dh_delly_lr_call_ex(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                        const uint64_t* seeds, int nrec, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, float indelExtension,
                        int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const uint8_t* tagflags,
                        const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off, int methylWindow, int methylProb,
                        int minCpgDepth, const char* tpl_arena, const uint32_t* tpl_off, float meiMinFrac, float trMinFrac, int32_t* anno_out, int32_t* methyl_out,
                        char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  return delly_lr_call_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, nrec, cigar, reads, cfg12, flankQuality, indelExtension, sv_out, cap, fmt_out,
                            gl_out, cons_out, cons_stride, cons_len, tagflags, mm_arena, mm_off, ml_arena, ml_off, methylWindow, methylProb, minCpgDepth, tpl_arena,
                            tpl_off, meiMinFrac, trMinFrac, anno_out, methyl_out, alleles_out, alleles_stride, alleles_len);
}

// several long-read samples — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call_multi
int dh_delly_lr_call_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                           const uint64_t* seeds, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality,
                           float indelExtension, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  Config c;
  c.minMapQual = (uint16_t) cfg12[0]; c.minClip = (uint32_t) cfg12[1]; c.minRefSep = (uint32_t) cfg12[2]; c.maxReadSep = (uint32_t) cfg12[3];
  c.minCliqueSize = (uint16_t) cfg12[4]; c.graphPruning = (uint32_t) cfg12[5]; c.maxReadPerSV = (uint32_t) cfg12[6]; c.minimumFlankSize = cfg12[7];
  c.indelsize = cfg12[8]; c.minConsWindow = cfg12[9]; c.maxGenoReadCount = (uint32_t) cfg12[10]; c.genoCap = cfg12[11];
  c.flankQuality = flankQuality; c.nchr = ncontig;
  apply_svtset(c);
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<std::vector<LrRecord> > recs((size_t) nfile);
  std::vector<std::vector<std::size_t> > ids((size_t) nfile);
  for (int f = 0; f < nfile; ++f)
    for (uint32_t i = file_off[f]; i < file_off[f + 1]; ++i) {
      const int32_t* r = rec12 + 12 * (size_t) i;
      LrRecord rec;
      rec.tid = r[0]; rec.pos = r[1]; rec.flag = (uint32_t) r[2]; rec.mapq = (uint8_t) r[3];
      for (int k = 0; k < r[6]; ++k) rec.cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
      rec.seq.assign(reads + r[7], (std::size_t) r[4]);
      recs[f].push_back(rec); ids[f].push_back((std::size_t) seeds[i]);
    }
  std::vector<LrSample> samples;
  for (int f = 0; f < nfile; ++f) samples.push_back(LrSample{&recs[f], &ids[f]});
  LrMultiCallSet cs;
  int rc = dellyLrCallMulti(ctx, c, indelExtension, tl, names, chr, samples, cs);
  if (rc) return rc - 1;
  const int n = (int) cs.svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    int32_t* o = sv_out + 20 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; o[19] = 0;
    memcpy(o + 19, &v.srAlignQuality, 4);
    for (int f = 0; f < nfile; ++f) {
      LrSampleCounts const& sc = cs.sample[f];
      SampleFormat const& fm = sc.format[i];
      int32_t* q = fmt_out + 14 * ((size_t) f * cap + i);
      q[0] = fm.gt[0]; q[1] = fm.gt[1]; q[2] = fm.gq; q[3] = fm.pl[0]; q[4] = fm.pl[1]; q[5] = fm.pl[2]; q[6] = fm.rcn; q[7] = fm.pass ? 1 : 0;
      q[8] = 0; q[9] = 0; q[10] = (int32_t) sc.jctMap[i].ref.size(); q[11] = (int32_t) sc.jctMap[i].alt.size();
      q[12] = sc.rcMap[i].rc; q[13] = sc.rcMap[i].leftRC + sc.rcMap[i].rightRC;
      for (int k = 0; k < 3; ++k) gl_out[3 * ((size_t) f * cap + i) + k] = fm.gl[k];
    }
    cons_len[i] = (int32_t) v.consensus.size();
    memcpy(cons_out + (size_t) i * cons_stride, v.consensus.data(), std::min<size_t>(v.consensus.size(), cons_stride));
  }
  return n;
}

// long-read genotyping mode: one sample, the outputs of dh_delly_lr_call for a given site list (rows as dh_vcf_parse)
int dh_delly_lr_genotype(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec,
                         const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, const int32_t* site22, int nsite, const char* strs,
                         const uint32_t* str_off, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out) {
  Config c;
  c.minMapQual = (uint16_t) cfg12[0]; c.minClip = (uint32_t) cfg12[1]; c.minRefSep = (uint32_t) cfg12[2]; c.maxReadSep = (uint32_t) cfg12[3];
  c.minCliqueSize = (uint16_t) cfg12[4]; c.graphPruning = (uint32_t) cfg12[5]; c.maxReadPerSV = (uint32_t) cfg12[6]; c.minimumFlankSize = cfg12[7];
  c.indelsize = cfg12[8]; c.minConsWindow = cfg12[9]; c.maxGenoReadCount = (uint32_t) cfg12[10]; c.genoCap = cfg12[11];
  c.flankQuality = flankQuality; c.nchr = ncontig;
  apply_svtset(c);
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<LrRecord> recs(nrec);
  std::vector<std::size_t> ids(nrec, 0);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
  }
  LrMultiCallSet cs;
  int rc = dellyLrGenotype(ctx, c, tl, names, chr, sites_from_rows(site22, nsite, strs, str_off), true, std::vector<LrSample>(1, LrSample{&recs, &ids}), cs);
  if (rc) return rc - 1;
  const int n = (int) cs.svs.size();
  if (n > cap) return -1;
  for (int i = 0; i < n; ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    int32_t* o = sv_out + 20 * i;
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
    o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id; o[19] = 0;
    memcpy(o + 19, &v.srAlignQuality, 4);
    LrSampleCounts const& sc = cs.sample[0];
    SampleFormat const& fm = sc.format[i];
    int32_t* q = fmt_out + 14 * i;
    q[0] = fm.gt[0]; q[1] = fm.gt[1]; q[2] = fm.gq; q[3] = fm.pl[0]; q[4] = fm.pl[1]; q[5] = fm.pl[2]; q[6] = fm.rcn; q[7] = fm.pass ? 1 : 0;
    q[8] = 0; q[9] = 0; q[10] = (int32_t) sc.jctMap[i].ref.size(); q[11] = (int32_t) sc.jctMap[i].alt.size();
    q[12] = sc.rcMap[i].rc; q[13] = sc.rcMap[i].leftRC + sc.rcMap[i].rightRC;
    for (int k = 0; k < 3; ++k) gl_out[3 * i + k] = fm.gl[k];
  }
  return n;
}

// clusterSRReadsLR — layout as oracle/ref_wrap5.cpp::ref_cluster_sr_reads (ctx may be NULL: host pair scans)
int dh_cluster_sr_reads(dgpu_ctx* ctx, const uint32_t* contig_len, int ncontig, const int32_t* rec12, const uint64_t* seeds, int nrec, const uint32_t* cigar,
                        const int32_t* cfg12, float indelExtension, int32_t* sv_out, int cap, int32_t* store_out, uint64_t* store_seed, int store_cap, int32_t* n_out) {
  Config c;
  c.minMapQual = (uint16_t) cfg12[0]; c.minClip = (uint32_t) cfg12[1]; c.minRefSep = (uint32_t) cfg12[2]; c.maxReadSep = (uint32_t) cfg12[3];
  c.minCliqueSize = (uint16_t) cfg12[4]; c.graphPruning = (uint32_t) cfg12[5]; c.nchr = ncontig;
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<LrRecord> recs(nrec);
  std::vector<std::size_t> ids(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    ids[i] = (std::size_t) seeds[i];
  }
  std::vector<StructuralVariantRecord> svc;
  std::vector<TPosReadSlices> srStore;
  int rc = clusterSRReadsLR(ctx, c, tl, recs, ids, indelExtension, svc, srStore);
  if (rc) return rc - 1;
  if ((int) svc.size() > cap) return -1;
  for (std::size_t i = 0; i < svc.size(); ++i) {
    int32_t* o = sv_out + 14 * i; StructuralVariantRecord const& v = svc[i];
    o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
    o[8] = v.srSupport; o[9] = v.srMapQuality; o[10] = v.mapq; o[11] = v.insLen; o[12] = v.svt; o[13] = v.id;
  }
  int k = 0;
  for (int t = 0; t < ncontig; ++t)
    for (auto const& kv : srStore[t])
      for (auto const& sl : kv.second) {
        if (k >= store_cap) return -1;
        int32_t* o = store_out + 6 * k;
        o[0] = t; o[1] = kv.first.first; o[2] = sl.svid; o[3] = sl.sstart; o[4] = sl.inslen; o[5] = sl.qual;
        store_seed[k++] = (uint64_t) kv.first.second;
      }
  n_out[0] = (int32_t) svc.size(); n_out[1] = k;
  return 0;
}

// getLibraryParams — layout as oracle/ref_wrap6.cpp::ref_get_library_params
int dh_get_library_params(const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec, const uint32_t* cigar, int madCutoff, int madNormalCutoff,
                          int32_t* out7) {
  Config c; c.madCutoff = (uint16_t) madCutoff; c.madNormalCutoff = (uint16_t) madNormalCutoff;
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<SrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec12 + 12 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    recs[i].lqseq = r[4]; recs[i].mtid = r[8]; recs[i].mpos = r[9]; recs[i].isize = r[10]; recs[i].name = (uint64_t) r[11];
  }
  LibraryInfo l;
  getLibraryParams(c, tl, recs, l);
  out7[0] = l.rs; out7[1] = l.median; out7[2] = l.mad; out7[3] = l.minNormalISize; out7[4] = l.minISizeCutoff; out7[5] = l.maxNormalISize; out7[6] = l.maxISizeCutoff;
  return 0;
}

// vcfRecords — layout as oracle/ref_wrap7.cpp::ref_vcf_output
static int vcf_output_hook(const uint32_t* contig_len, int ncontig, const int32_t* sv25, int n, const char* alleles, int astride, const int32_t* alen, const char* cons,
                  int cstride, const int32_t* clen, const uint8_t* quals, const uint32_t* jr_off, const uint32_t* ja_off, const uint32_t* sr_off,
                  const uint32_t* sa_off, const int32_t* hp5, const int32_t* rc3, int hasVcfFile, char* out, int cap, const int32_t* anno_tr,
                  const int32_t* methyl16, int minCpgDepth, int nfile) {
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<std::string> names;
  for (int k = 0; k < ncontig; ++k) names.push_back("chr" + std::to_string(k));
  std::vector<StructuralVariantRecord> svs(n);
  std::vector<std::vector<JunctionCount> > jctF((size_t) nfile, std::vector<JunctionCount>(n));
  std::vector<std::vector<SpanningCount> > spanF((size_t) nfile, std::vector<SpanningCount>(n));
  std::vector<std::vector<ReadCount> > rcmF((size_t) nfile, std::vector<ReadCount>(n));
  for (int i = 0; i < n; ++i) {
    const int32_t* r = sv25 + 25 * i; StructuralVariantRecord& v = svs[i];
    v.chr = r[0]; v.svStart = r[1]; v.chr2 = r[2]; v.svEnd = r[3]; v.ciposlow = r[4]; v.ciposhigh = r[5]; v.ciendlow = r[6]; v.ciendhigh = r[7];
    v.peSupport = r[8]; v.srSupport = r[9]; v.peMapQuality = r[10]; v.srMapQuality = r[11]; v.mapq = r[12]; v.insLen = r[13]; v.homLen = r[14]; v.svt = r[15];
    v.precise = r[16] != 0; v.consBp = r[17]; v.id = r[18]; memcpy(&v.srAlignQuality, r + 19, 4); v.alleleid = r[20]; v.nallele = r[21];
    v.anno.homLen = r[22]; v.anno.seqType = r[23]; v.anno.isRC = r[24] != 0;
    if (anno_tr) { v.anno.trPeriod = anno_tr[2 * i]; memcpy(&v.anno.trCopies, anno_tr + 2 * i + 1, 4); }
    v.alleles.assign(alleles + (size_t) i * astride, (size_t) alen[i]); v.consensus.assign(cons + (size_t) i * cstride, (size_t) clen[i]);
    const int id = v.id;
    for (int f = 0; f < nfile; ++f) {   // per-sample arrays file-major, as in oracle/ref_wrap7.cpp
      const uint32_t* jr = jr_off + (size_t) f * (n + 1); const uint32_t* ja = ja_off + (size_t) f * (n + 1);
      const uint32_t* sr = sr_off + (size_t) f * (n + 1); const uint32_t* sa = sa_off + (size_t) f * (n + 1);
      const int32_t* hp = hp5 + (size_t) f * 5 * n; const int32_t* rc = rc3 + (size_t) f * 3 * n;
      JunctionCount& jc = jctF[f][id];
      jc.ref.assign(quals + jr[i], quals + jr[i + 1]); jc.alt.assign(quals + ja[i], quals + ja[i + 1]);
      spanF[f][id].ref.assign(quals + sr[i], quals + sr[i + 1]); spanF[f][id].alt.assign(quals + sa[i], quals + sa[i + 1]);
      jc.hp1ref.assign(hp[5 * i], 30); jc.hp1alt.assign(hp[5 * i + 1], 30); jc.hp2ref.assign(hp[5 * i + 2], 30); jc.hp2alt.assign(hp[5 * i + 3], 30);
      jc.ps = hp[5 * i + 4];
      rcmF[f][id].leftRC = rc[3 * i]; rcmF[f][id].rc = rc[3 * i + 1]; rcmF[f][id].rightRC = rc[3 * i + 2];
    }
  }
  std::vector<std::vector<MethylInfo> > methylF((size_t) nfile);
  if (methyl16)
    for (int f = 0; f < nfile; ++f) {
      methylF[f].resize(n);
      for (int i = 0; i < n; ++i) {
        MethylInfo& mi = methylF[f][svs[i].id];
        const int32_t* m = methyl16 + 16 * ((size_t) f * n + i);
        memcpy(mi.alt, m, 16); memcpy(mi.ref, m + 4, 16); memcpy(mi.mnc, m + 8, 16); memcpy(mi.mdp, m + 12, 16);
      }
    }
  std::vector<VcfSample> samples((size_t) nfile);
  for (int f = 0; f < nfile; ++f) {
    samples[f].name = "sample" + std::to_string(f + 1); samples[f].jctMap = &jctF[f]; samples[f].rcMap = &rcmF[f]; samples[f].spanMap = &spanF[f];
    samples[f].methylMap = methyl16 ? &methylF[f] : nullptr;
  }
  const std::string text = vcfRecords(svs, samples, names, tl, "in-memory.fa", "00000000", hasVcfFile != 0, (uint32_t) minCpgDepth);
  memcpy(out, text.data(), std::min<size_t>(text.size(), (size_t) cap));
  return (int) text.size();
}

int dh_vcf_output(const uint32_t* contig_len, int ncontig, const int32_t* sv25, int n, const char* alleles, int astride, const int32_t* alen, const char* cons,
                  int cstride, const int32_t* clen, const uint8_t* quals, const uint32_t* jr_off, const uint32_t* ja_off, const uint32_t* sr_off,
                  const uint32_t* sa_off, const int32_t* hp5, const int32_t* rc3, int hasVcfFile, char* out, int cap) {
  return vcf_output_hook(contig_len, ncontig, sv25, n, alleles, astride, alen, cons, cstride, clen, quals, jr_off, ja_off, sr_off, sa_off, hp5, rc3, hasVcfFile, out,
                         cap, nullptr, nullptr, 0, 1);
}

// as oracle/ref_wrap7.cpp::ref_vcf_output_ex: plus the tandem-repeat annotation and the sample's MethylInfo
int dh_vcf_output_ex(const uint32_t* contig_len, int ncontig, const int32_t* sv25, int n, const char* alleles, int astride, const int32_t* alen, const char* cons,
                     int cstride, const int32_t* clen, const uint8_t* quals, const uint32_t* jr_off, const uint32_t* ja_off, const uint32_t* sr_off,
                     const uint32_t* sa_off, const int32_t* hp5, const int32_t* rc3, int hasVcfFile, char* out, int cap, const int32_t* anno_tr,
                     const int32_t* methyl16, int minCpgDepth) {
  return vcf_output_hook(contig_len, ncontig, sv25, n, alleles, astride, alen, cons, cstride, clen, quals, jr_off, ja_off, sr_off, sa_off, hp5, rc3, hasVcfFile, out,
                         cap, anno_tr, methyl16, minCpgDepth, 1);
}

// several samples — layout as oracle/ref_wrap7.cpp::ref_vcf_output_multi
int dh_vcf_output_multi(const uint32_t* contig_len, int ncontig, const int32_t* sv25, int n, const char* alleles, int astride, const int32_t* alen, const char* cons,
                        int cstride, const int32_t* clen, const uint8_t* quals, const uint32_t* jr_off, const uint32_t* ja_off, const uint32_t* sr_off,
                        const uint32_t* sa_off, const int32_t* hp5, const int32_t* rc3, int hasVcfFile, char* out, int cap, const int32_t* anno_tr,
                        const int32_t* methyl16, int minCpgDepth, int nfile) {
  return vcf_output_hook(contig_len, ncontig, sv25, n, alleles, astride, alen, cons, cstride, clen, quals, jr_off, ja_off, sr_off, sa_off, hp5, rc3, hasVcfFile, out,
                         cap, anno_tr, methyl16, minCpgDepth, nfile);
}

// genotypeLRBatch — layout as oracle/ref_wrap4.cpp::ref_genotype_lr (contigs named "chr0", "chr1", ...)
static int genotype_lr_hook(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec10, int nrec,
                   const uint32_t* cigar, const char* reads, const int32_t* sv8, int nsv, const char* cons_arena, const uint32_t* cons_off,
                   const uint32_t* cons_len, int minMapQual, int minimumFlankSize, int minConsWindow, int maxGenoReadCount, float flankQuality, int genoCap,
                   uint8_t* qual_out, int qual_cap, uint32_t* ref_off, uint32_t* alt_off, int32_t* hp_out, int32_t* rc_out, const uint8_t* tagflags,
                   const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off, int methylWindow, int methylProb,
                   int minCpgDepth, int32_t* methyl_out) {
  Config c; c.minMapQual = (uint16_t) minMapQual; c.minimumFlankSize = minimumFlankSize; c.minConsWindow = minConsWindow;
  c.maxGenoReadCount = (uint32_t) maxGenoReadCount; c.flankQuality = flankQuality; c.genoCap = genoCap;
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  for (int k = 0; k < ncontig; ++k) { tl.push_back(contig_len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(contig_arena + contig_off[k]); }
  std::vector<LrRecord> recs(nrec);
  for (int i = 0; i < nrec; ++i) {
    const int32_t* r = rec10 + 10 * i;
    recs[i].tid = r[0]; recs[i].pos = r[1]; recs[i].flag = (uint32_t) r[2]; recs[i].mapq = (uint8_t) r[3];
    for (int k = 0; k < r[6]; ++k) recs[i].cigar.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
    recs[i].seq.assign(reads + r[7], (std::size_t) r[4]);
    recs[i].hp = (uint8_t) (r[8] > 0 ? r[8] : 0); recs[i].ps = r[9];
    if (tagflags && (tagflags[i] & 1)) { recs[i].hasMM = true; recs[i].mm.assign(mm_arena + mm_off[i], mm_arena + mm_off[i + 1]); }
    if (tagflags && (tagflags[i] & 2)) { recs[i].hasML = true; recs[i].ml.assign(ml_arena + ml_off[i], ml_arena + ml_off[i + 1]); }
  }
  std::vector<StructuralVariantRecord> svs(nsv);
  for (int i = 0; i < nsv; ++i) {
    const int32_t* s = sv8 + 8 * i;
    svs[i].chr = s[0]; svs[i].svStart = s[1]; svs[i].chr2 = s[2]; svs[i].svEnd = s[3]; svs[i].svt = s[4]; svs[i].insLen = s[5]; svs[i].consBp = s[6]; svs[i].id = s[7];
    svs[i].consensus.assign(cons_arena + cons_off[i], cons_len[i]);
    svs[i].precise = true;
  }
  std::vector<JunctionCount> jct; std::vector<ReadCount> cov;
  MethylConfig mcfg; mcfg.methylWindow = methylWindow; mcfg.methylProb = (uint16_t) methylProb; mcfg.minCpgDepth = (uint32_t) minCpgDepth;
  std::vector<MethylInfo> methyl;
  int rc = genotypeLRBatch(ctx, c, tl, names, chr, svs, recs, jct, cov, tagflags ? &mcfg : nullptr, tagflags ? &methyl : nullptr);
  if (rc) return rc - 1;
  if (tagflags && methyl_out)
    for (int i = 0; i < nsv; ++i) {
      memcpy(methyl_out + 16 * i, methyl[i].alt, 16); memcpy(methyl_out + 16 * i + 4, methyl[i].ref, 16);
      memcpy(methyl_out + 16 * i + 8, methyl[i].mnc, 16); memcpy(methyl_out + 16 * i + 12, methyl[i].mdp, 16);
    }
  int pos = 0;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t* off = pass ? alt_off : ref_off;
    for (int i = 0; i < nsv; ++i) {
      off[i] = (uint32_t) pos;
      std::vector<uint8_t> const& v = pass ? jct[i].alt : jct[i].ref;
      if (pos + (int) v.size() > qual_cap) return -1;
      for (uint8_t q : v) qual_out[pos++] = q;
    }
    off[nsv] = (uint32_t) pos;
  }
  for (int i = 0; i < nsv; ++i) {
    hp_out[5 * i] = (int32_t) jct[i].hp1ref.size(); hp_out[5 * i + 1] = (int32_t) jct[i].hp1alt.size(); hp_out[5 * i + 2] = (int32_t) jct[i].hp2ref.size();
    hp_out[5 * i + 3] = (int32_t) jct[i].hp2alt.size(); hp_out[5 * i + 4] = jct[i].ps;
    rc_out[3 * i] = cov[i].leftRC; rc_out[3 * i + 1] = cov[i].rc; rc_out[3 * i + 2] = cov[i].rightRC;
  }
  return pos;
}

int dh_genotype_lr(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec10, int nrec,
                   const uint32_t* cigar, const char* reads, const int32_t* sv8, int nsv, const char* cons_arena, const uint32_t* cons_off,
                   const uint32_t* cons_len, int minMapQual, int minimumFlankSize, int minConsWindow, int maxGenoReadCount, float flankQuality, int genoCap,
                   uint8_t* qual_out, int qual_cap, uint32_t* ref_off, uint32_t* alt_off, int32_t* hp_out, int32_t* rc_out) {
  return genotype_lr_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec10, nrec, cigar, reads, sv8, nsv, cons_arena, cons_off, cons_len, minMapQual,
                          minimumFlankSize, minConsWindow, maxGenoReadCount, flankQuality, genoCap, qual_out, qual_cap, ref_off, alt_off, hp_out, rc_out, nullptr,
                          nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nullptr);
}

// genotypeLRBatch with MM / ML tags — layout as oracle/ref_wrap4.cpp::ref_genotype_lr_methyl
int dh_genotype_lr_methyl(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec10,
                          int nrec, const uint32_t* cigar, const char* reads, const int32_t* sv8, int nsv, const char* cons_arena, const uint32_t* cons_off,
                          const uint32_t* cons_len, int minMapQual, int minimumFlankSize, int minConsWindow, int maxGenoReadCount, float flankQuality,
                          int genoCap, uint8_t* qual_out, int qual_cap, uint32_t* ref_off, uint32_t* alt_off, int32_t* hp_out, int32_t* rc_out,
                          const uint8_t* tagflags, const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off,
                          int methylWindow, int methylProb, int minCpgDepth, int32_t* methyl_out) {
  return genotype_lr_hook(ctx, contig_arena, contig_off, contig_len, ncontig, rec10, nrec, cigar, reads, sv8, nsv, cons_arena, cons_off, cons_len, minMapQual,
                          minimumFlankSize, minConsWindow, maxGenoReadCount, flankQuality, genoCap, qual_out, qual_cap, ref_off, alt_off, hp_out, rc_out, tagflags,
                          mm_arena, mm_off, ml_arena, ml_off, methylWindow, methylProb, minCpgDepth, methyl_out);
}

// _seqIdentity / _bestSeqIdentity / _minRotation (src/merge.h:187-243) for n pairs: sequences in one arena, (offset, length) per side
int dh_seq_identity_batch(dgpu_ctx* ctx, const char* arena, const uint32_t* a_off, const uint32_t* a_len, const uint32_t* b_off, const uint32_t* b_len,
                          const int32_t* pos_off, int n, double minId, int seqCutoff, int best, double* out) {
  std::vector<IdentityPair> pairs((size_t) n);
  for (int i = 0; i < n; ++i) { pairs[i].a.assign(arena + a_off[i], a_len[i]); pairs[i].b.assign(arena + b_off[i], b_len[i]); pairs[i].posOff = pos_off ? pos_off[i] : 0; }
  std::vector<double> id;
  const int rc = best ? bestSeqIdentityBatch(ctx, pairs, minId, seqCutoff, id) : seqIdentityBatch(ctx, pairs, minId, id);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) out[i] = id[i];
  return 0;
}
int dh_min_rotation(const char* s, int n, char* out) {
  const std::string r = _minRotation(std::string(s, s + n));
  memcpy(out, r.data(), r.size());
  return (int) r.size();
}

// MA / MR / MNC / MDV FORMAT values from one MethylInfo (16 ints, field order alt, ref, mnc, mdp)
void dh_methyl_format(const int32_t* mi16, int svt, int minCpgDepth, int32_t* out16) {
  MethylInfo mi;
  memcpy(mi.alt, mi16, 16); memcpy(mi.ref, mi16 + 4, 16); memcpy(mi.mnc, mi16 + 8, 16); memcpy(mi.mdp, mi16 + 12, 16);
  methylFormat(mi, svt, (uint32_t) minCpgDepth, out16, out16 + 4, out16 + 8, out16 + 12);
}

// _computeGLs for one sample — layout as oracle/ref_wrap3.cpp::ref_compute_gls
void dh_compute_gls(const uint8_t* refq, int nref, const uint8_t* altq, int nalt, float* gls3, int32_t* gq, int32_t* gts2) {
  static BoLog bl;
  std::vector<uint8_t> r(refq, refq + nref), a(altq, altq + nalt);
  _computeGLs(bl, r, a, gls3, gq, gts2);
}

// sampleFormat for n samples: qualities as arenas with n+1 offsets; extra = n x [ps, hp1alt, hp2alt, rcl, rc, rcr];
// out = n x [gt0, gt1, gq, pl0, pl1, pl2, rcn, pass, glMissing], gls = n x 3
void dh_sample_format(int n, const uint8_t* refq, const uint32_t* ref_off, const uint8_t* altq, const uint32_t* alt_off, const int32_t* extra,
                      int32_t* out, float* gls) {
  static BoLog bl;
  for (int i = 0; i < n; ++i) {
    std::vector<uint8_t> r(refq + ref_off[i], refq + ref_off[i + 1]), a(altq + alt_off[i], altq + alt_off[i + 1]);
    const int32_t* e = extra + 6 * i;
    SampleFormat f = sampleFormat(bl, r, a, e[0], e[1], e[2], e[3], e[4], e[5]);
    int32_t* o = out + 9 * i;
    o[0] = f.gt[0]; o[1] = f.gt[1]; o[2] = f.gq; o[3] = f.pl[0]; o[4] = f.pl[1]; o[5] = f.pl[2]; o[6] = f.rcn; o[7] = f.pass ? 1 : 0; o[8] = f.glMissing ? 1 : 0;
    for (int k = 0; k < 3; ++k) gls[3 * i + k] = f.gl[k];
  }
}

// processBatch: jobs as three arenas; results type/qual per job
int dh_process_batch(dgpu_ctx* ctx, int n, const char* arena, const uint32_t* cons_off, const uint32_t* cons_len, const uint32_t* ref_off,
                     const uint32_t* ref_len, const uint32_t* seq_off, const uint32_t* seq_len, const uint8_t* qual, float flankQuality,
                     char* type_out, uint8_t* qual_out) {
  Config c; c.flankQuality = flankQuality;
  std::vector<AlignJob> jobs(n);
  for (int i = 0; i < n; ++i) {
    jobs[i].consProbe.assign(arena + cons_off[i], cons_len[i]);
    jobs[i].refProbe.assign(arena + ref_off[i], ref_len[i]);
    jobs[i].sequence.assign(arena + seq_off[i], seq_len[i]);
    jobs[i].fileIndex = 0; jobs[i].svId = (uint32_t) i; jobs[i].qual = qual[i];
  }
  std::vector<AlignResult> res;
  int rc = processBatch(ctx, c, jobs, res);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) { type_out[i] = res[i].type; qual_out[i] = res[i].qual; }
  return 0;
}

// msaBatch: clusters as (arena, read_off, read_len, cluster_off)
int dh_msa_batch(dgpu_ctx* ctx, const char* arena, const uint32_t* read_off, const uint32_t* read_len, const uint32_t* cluster_off, int ncl,
                 int minClique, char* cons, int cons_stride, int32_t* cons_len, int32_t* rows) {
  Config c; c.minCliqueSize = (uint16_t) minClique;
  std::vector<std::vector<std::string> > cl(ncl);
  for (int i = 0; i < ncl; ++i)
    for (uint32_t r = cluster_off[i]; r < cluster_off[i + 1]; ++r) cl[i].push_back(std::string(arena + read_off[r], read_len[r]));
  std::vector<std::string> cs;
  std::vector<int> rw;
  int rc = msaBatch(ctx, c, cl, cs, rw);
  if (rc) return rc;
  for (int i = 0; i < ncl; ++i) {
    cons_len[i] = (int32_t) cs[i].size(); rows[i] = rw[i];
    memcpy(cons + (size_t) i * cons_stride, cs[i].data(), std::min<size_t>(cs[i].size(), cons_stride));
  }
  return 0;
}

// msaEdlibBatch: clusters as (arena, read_off, read_len, cluster_off)
int dh_msa_edlib_batch(dgpu_ctx* ctx, const char* arena, const uint32_t* read_off, const uint32_t* read_len, const uint32_t* cluster_off, int ncl,
                       int minClique, char* cons, int cons_stride, int32_t* cons_len, int32_t* rows) {
  Config c = Config::longRead(); c.minCliqueSize = (uint16_t) minClique;
  std::vector<std::vector<std::string> > cl(ncl);
  for (int i = 0; i < ncl; ++i)
    for (uint32_t r = cluster_off[i]; r < cluster_off[i + 1]; ++r) cl[i].push_back(std::string(arena + read_off[r], read_len[r]));
  std::vector<std::string> cs;
  std::vector<int> rw;
  int rc = msaEdlibBatch(ctx, c, cl, cs, rw);
  if (rc) return rc;
  for (int i = 0; i < ncl; ++i) {
    cons_len[i] = (int32_t) cs[i].size(); rows[i] = rw[i];
    memcpy(cons + (size_t) i * cons_stride, cs[i].data(), std::min<size_t>(cs[i].size(), cons_stride));
  }
  return 0;
}

// msaWfaBatch: clusters as (arena, read_off, read_len, cluster_off); flanks as fixed-stride arrays (flank_len 0: 5 % trim)
int dh_msa_wfa_batch(dgpu_ctx* ctx, const char* arena, const uint32_t* read_off, const uint32_t* read_len, const uint32_t* cluster_off, int ncl,
                     int minClique, const char* prefix, const char* suffix, int flank_stride, const int32_t* prefix_len, const int32_t* suffix_len,
                     char* cons, int cons_stride, int32_t* cons_len, int32_t* rows) {
  Config c = Config::longRead(); c.minCliqueSize = (uint16_t) minClique;
  std::vector<std::vector<std::string> > cl(ncl);
  std::vector<std::string> pre(ncl), suf(ncl);
  for (int i = 0; i < ncl; ++i) {
    for (uint32_t r = cluster_off[i]; r < cluster_off[i + 1]; ++r) cl[i].push_back(std::string(arena + read_off[r], read_len[r]));
    pre[i].assign(prefix + (size_t) i * flank_stride, prefix_len[i]);
    suf[i].assign(suffix + (size_t) i * flank_stride, suffix_len[i]);
  }
  std::vector<std::string> cs;
  std::vector<int> rw;
  int rc = msaWfaBatch(ctx, c, cl, pre, suf, cs, rw);
  if (rc) return rc;
  for (int i = 0; i < ncl; ++i) {
    cons_len[i] = (int32_t) cs[i].size(); rows[i] = rw[i];
    memcpy(cons + (size_t) i * cons_stride, cs[i].data(), std::min<size_t>(cs[i].size(), cons_stride));
  }
  return 0;
}

// annotateSVBatch for the SVs of one chromosome — layout as oracle/ref_wrap8.cpp::ref_annotate_sv, plus the mobile-element
// templates the reference holds (class MEI): tpl_arena / tpl_off[8] = sequences 1..6 and the polyA tail (slot 7).
// ctx may be NULL when no inserted sequence needs a device distance (deletions, symbolic or short insertions).
int dh_annotate_sv(dgpu_ctx* ctx, const char* tpl_arena, const uint32_t* tpl_off, const char* seq, int chrLen, const int32_t* sv3, int nsv,
                   const char* alleles, const uint32_t* al_off, float meiMinFrac, float trMinFrac, int32_t* out5) {
  MeiTemplates mei;
  if (tpl_arena && tpl_off) {
    for (int t = 1; t <= 6; ++t) mei.seq[t].assign(tpl_arena + tpl_off[t - 1], tpl_arena + tpl_off[t]);
    mei.polyA.assign(tpl_arena + tpl_off[6], tpl_arena + tpl_off[7]);
  }
  AnnoConfig c; c.meiMinFrac = meiMinFrac; c.trMinFrac = trMinFrac;
  std::vector<StructuralVariantRecord> svs(nsv);
  std::vector<int32_t> which(nsv);
  for (int i = 0; i < nsv; ++i) {
    svs[i].svt = sv3[3 * i]; svs[i].svStart = sv3[3 * i + 1]; svs[i].svEnd = sv3[3 * i + 2];
    svs[i].alleles.assign(alleles + al_off[i], alleles + al_off[i + 1]);
    which[i] = i;
  }
  std::vector<const char*> chrseq(1, seq);
  std::vector<uint32_t> tlen(1, (uint32_t) chrLen);
  int rc = annotateSVBatch(ctx, c, mei, chrseq, tlen, svs, which);
  if (rc) return rc;
  for (int i = 0; i < nsv; ++i) {
    int32_t* o = out5 + 5 * i;
    o[0] = svs[i].anno.isRC ? 1 : 0; o[1] = svs[i].anno.seqType; o[2] = svs[i].anno.homLen; o[3] = svs[i].anno.trPeriod;
    memcpy(&o[4], &svs[i].anno.trCopies, 4);
  }
  return 0;
}

int dh_detect_tandem_repeat(const char* s, int n, int maxPeriod, float minFraction, float* copies) {
  std::pair<int32_t, float> r = detectTandemRepeat(std::string(s, s + n), maxPeriod, minFraction);
  *copies = r.second;
  return r.first;
}

#include "capi_sharded.inc"

// edit-path jobs refused so far by a device limit (DeviceLimitLog::pathJobs; the binding reports it on stderr)
uint64_t dh_path_jobs_refused(void) { return deviceLimitLog().pathJobs.load(); }

}  // extern "C"
