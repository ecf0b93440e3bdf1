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

// ---- the flat rows of the hooks below --------------------------------------------------------------------------------------------------

// CIGAR of a record row: r[5] = first op in the packed array (BAM encoding: length << 4 | op), r[6] = number of ops
static std::vector<std::pair<uint8_t, uint32_t> > row_cigar(const int32_t* r, const uint32_t* cigar) {
  std::vector<std::pair<uint8_t, uint32_t> > cg;
  for (int k = 0; k < r[6]; ++k) cg.push_back(std::make_pair((uint8_t) (cigar[r[5] + k] & 0xf), cigar[r[5] + k] >> 4));
  return cg;
}

// Short-read row i (tid, pos, flag, mapq, length, cigar first, cigar count, read offset, mtid, mpos, isize, name id). cigar, reads, seeds and
// name_hash may be NULL: the fields they fill keep their defaults.
static SrRecord sr_record(const int32_t* r, const uint32_t* cigar, const char* reads, const uint64_t* seeds, const uint32_t* name_hash, std::size_t i) {
  SrRecord rec;
  rec.tid = r[0]; rec.pos = r[1]; rec.flag = (uint32_t) r[2]; rec.mapq = (uint8_t) r[3];
  if (cigar) rec.cigar = row_cigar(r, cigar);
  if (reads) rec.seq.assign(reads + r[7], (std::size_t) r[4]);
  rec.lqseq = r[4]; rec.mtid = r[8]; rec.mpos = r[9]; rec.isize = r[10]; rec.name = (uint64_t) r[11];
  if (seeds) rec.seed = (std::size_t) seeds[i];
  if (name_hash) rec.nameHash32 = name_hash[i];
  return rec;
}

// MM / ML tags of long-read rows (flags NULL = none): flags[i] bit 0 = MM, bit 1 = ML, each the arena slice [off[i], off[i + 1])
struct LrTags { const uint8_t* flags; const char* mm; const uint32_t* mm_off; const uint8_t* ml; const uint32_t* ml_off; };

// Long-read row i: [0..7] as sr_record; with hpps, [8] = HP tag (0 = none) and [9] = PS tag (-1 = none). reads may be NULL.
static LrRecord lr_record(const int32_t* r, const uint32_t* cigar, const char* reads, bool hpps, LrTags const& tags, std::size_t i) {
  LrRecord rec;
  rec.tid = r[0]; rec.pos = r[1]; rec.flag = (uint32_t) r[2]; rec.mapq = (uint8_t) r[3];
  rec.cigar = row_cigar(r, cigar);
  if (reads) rec.seq.assign(reads + r[7], (std::size_t) r[4]);
  if (hpps) { rec.hp = (uint8_t) (r[8] > 0 ? r[8] : 0); rec.ps = r[9]; }
  if (tags.flags && (tags.flags[i] & 1)) { rec.hasMM = true; rec.mm.assign(tags.mm + tags.mm_off[i], tags.mm + tags.mm_off[i + 1]); }
  if (tags.flags && (tags.flags[i] & 2)) { rec.hasML = true; rec.ml.assign(tags.ml + tags.ml_off[i], tags.ml + tags.ml_off[i + 1]); }
  return rec;
}

// contigs "chr0", "chr1", ... as arena + offsets + lengths
struct Genome {
  std::vector<uint32_t> tl; std::vector<std::string> names; std::vector<const char*> chr;
  Genome(const char* arena, const uint32_t* off, const uint32_t* len, int n) {
    for (int k = 0; k < n; ++k) { tl.push_back(len[k]); names.push_back("chr" + std::to_string(k)); chr.push_back(arena + off[k]); }
  }
};

// mobile-element templates: arena slices off[t - 1] .. off[t] are sequences 1..6, off[6] .. off[7] the polyA tail
static void load_mei(MeiTemplates& mei, const char* arena, const uint32_t* off) {
  for (int t = 1; t <= 6; ++t) mei.seq[t].assign(arena + off[t - 1], arena + off[t]);
  mei.polyA.assign(arena + off[6], arena + off[7]);
}

// the 20-int SV row: chr, start, chr2, end, ciposlow/high, ciendlow/high, PE, SR, PE mapq, SR mapq, mapq, insLen, homLen, svt, precise,
// consBp, id, srAlignQuality (float bits)
static void put_sv(int32_t* o, StructuralVariantRecord const& v) {
  o[0] = v.chr; o[1] = v.svStart; o[2] = v.chr2; o[3] = v.svEnd; o[4] = v.ciposlow; o[5] = v.ciposhigh; o[6] = v.ciendlow; o[7] = v.ciendhigh;
  o[8] = v.peSupport; o[9] = v.srSupport; o[10] = v.peMapQuality; o[11] = v.srMapQuality; o[12] = v.mapq; o[13] = v.insLen; o[14] = v.homLen; o[15] = v.svt;
  o[16] = v.precise ? 1 : 0; o[17] = v.consBp; o[18] = v.id;
  memcpy(o + 19, &v.srAlignQuality, 4);
}

// the 14-int FORMAT row: gt0, gt1, gq, pl0..2, rcn, pass, [8] and [9] as the chain defines them (c89), junction REF / ALT reads, rc,
// left + right rc; and the GL triple
static void put_format(int32_t* q, float* gl, SampleFormat const& f, std::pair<int32_t, int32_t> c89, JunctionCount const& j, ReadCount const& rc) {
  q[0] = f.gt[0]; q[1] = f.gt[1]; q[2] = f.gq; q[3] = f.pl[0]; q[4] = f.pl[1]; q[5] = f.pl[2]; q[6] = f.rcn; q[7] = f.pass ? 1 : 0;
  q[8] = c89.first; q[9] = c89.second; q[10] = (int32_t) j.ref.size(); q[11] = (int32_t) j.alt.size(); q[12] = rc.rc; q[13] = rc.leftRC + rc.rightRC;
  for (int k = 0; k < 3; ++k) gl[k] = f.gl[k];
}

// FORMAT [8], [9]: spanning REF / ALT pairs (sr); zeros (lr); ALT reads of haplotype 1 + 100 x those of haplotype 2 and the phase set (the
// lr contig hooks)
static std::pair<int32_t, int32_t> cols_spanning(SrSampleCounts const& s, int i) { return {(int32_t) s.spanMap[i].ref.size(), (int32_t) s.spanMap[i].alt.size()}; }
static std::pair<int32_t, int32_t> cols_zero(LrSampleCounts const&, int) { return {0, 0}; }
static std::pair<int32_t, int32_t> cols_haplotype(LrSampleCounts const& s, int i) {
  JunctionCount const& j = s.jctMap[i];
  return {(int32_t) j.hp1alt.size() + 100 * (int32_t) j.hp2alt.size(), j.ps};
}

// fixed-stride string slot i, cut at the stride; len[i] = the full length
static void put_bytes(char* out, int stride, int32_t* len, std::size_t i, std::string const& s) {
  len[i] = (int32_t) s.size();
  memcpy(out + i * stride, s.data(), std::min<size_t>(s.size(), stride));
}

// the assembled SVs of dh_assemble_split_reads / dh_assemble_lr: 13-int rows (start, end, SR, mapq, SR mapq, insLen, homLen, consBp, precise,
// ciposlow/high, ciendlow/high), srAlignQuality, consensus and alleles
static void put_assembled(std::vector<StructuralVariantRecord> const& svs, int32_t* sv_out, float* srq, char* cons_out, int cons_stride, int32_t* cons_len,
                          char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  for (std::size_t i = 0; i < svs.size(); ++i) {
    StructuralVariantRecord const& sv = svs[i];
    int32_t* o = sv_out + 13 * i;
    o[0] = sv.svStart; o[1] = sv.svEnd; o[2] = sv.srSupport; o[3] = sv.mapq; o[4] = sv.srMapQuality; o[5] = sv.insLen; o[6] = sv.homLen; o[7] = sv.consBp;
    o[8] = sv.precise ? 1 : 0; o[9] = sv.ciposlow; o[10] = sv.ciposhigh; o[11] = sv.ciendlow; o[12] = sv.ciendhigh;
    srq[i] = sv.srAlignQuality;
    put_bytes(cons_out, cons_stride, cons_len, i, sv.consensus);
    put_bytes(alleles_out, alleles_stride, alleles_len, i, sv.alleles);
  }
}

// one MethylInfo as 16 ints: alt, ref, mnc, mdp
static void put_methyl(int32_t* m, MethylInfo const& mi) { memcpy(m, mi.alt, 16); memcpy(m + 4, mi.ref, 16); memcpy(m + 8, mi.mnc, 16); memcpy(m + 12, mi.mdp, 16); }

// per-SV quality lists (T: JunctionCount / SpanningCount) as one arena: the REF lists of all SVs, then the ALT lists; ref_off / alt_off[nsv + 1].
// Returns the arena size, or -1 when it exceeds cap.
template <typename T>
static int put_qual_lists(std::vector<T> const& v, int nsv, uint8_t* out, int cap, uint32_t* ref_off, uint32_t* alt_off) {
  int pos = 0;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t* off = pass ? alt_off : ref_off;
    for (int i = 0; i < nsv; ++i) {
      off[i] = (uint32_t) pos;
      std::vector<uint8_t> const& q = pass ? v[i].alt : v[i].ref;
      if (pos + (int) q.size() > cap) return -1;
      for (uint8_t x : q) out[pos++] = x;
    }
    off[nsv] = (uint32_t) pos;
  }
  return pos;
}

// Where a chain hook writes its n SVs: sv[cap][20]; per file, file-major with stride cap, fmt[nfile][cap][14] and gl[nfile][cap][3]; the
// consensus cons[cap][cons_stride] + cons_len[cap] (cons may be NULL). The lr extras, each may be NULL: anno[cap][5], methyl[nfile][cap][16],
// alleles[cap][alleles_stride] + alleles_len[cap]. A single-sample hook is nfile = 1.
struct ChainOut {
  int32_t* sv; int cap; int32_t* fmt; float* gl; char* cons; int cons_stride; int32_t* cons_len;
  int nfile = 1;
  int32_t* anno = nullptr; int32_t* methyl = nullptr; char* alleles = nullptr; int alleles_stride = 0; int32_t* alleles_len = nullptr;
};

// The SV rows, FORMAT rows + GLs of every file and consensus of a multi-sample call set; cols89(sample, i) gives FORMAT [8], [9].
// Returns the number of SVs, or -1 (nothing written) when they exceed cap.
template <typename TCallSet, typename TCols89>
static int write_calls(TCallSet const& cs, ChainOut const& o, TCols89 cols89) {
  const int n = (int) cs.svs.size();
  if (n > o.cap) return -1;
  for (int i = 0; i < n; ++i) {
    put_sv(o.sv + 20 * i, cs.svs[i]);
    for (std::size_t f = 0; f < cs.sample.size(); ++f) {
      const std::size_t row = f * o.cap + i;
      put_format(o.fmt + 14 * row, o.gl + 3 * row, cs.sample[f].format[i], cols89(cs.sample[f], i), cs.sample[f].jctMap[i], cs.sample[f].rcMap[i]);
    }
    if (o.cons) put_bytes(o.cons, o.cons_stride, o.cons_len, i, cs.svs[i].consensus);
  }
  return n;
}

// the lr extras the hook has: annotation (isRC, seqType, homLen, trPeriod, trCopies as float bits), the methylation of every file that has
// one, the alleles
static void write_lr_extras(LrMultiCallSet const& cs, ChainOut const& o) {
  for (std::size_t i = 0; i < cs.svs.size(); ++i) {
    StructuralVariantRecord const& v = cs.svs[i];
    if (o.anno) {
      int32_t* a = o.anno + 5 * i;
      a[0] = v.anno.isRC ? 1 : 0; a[1] = v.anno.seqType; a[2] = v.anno.homLen; a[3] = v.anno.trPeriod; memcpy(a + 4, &v.anno.trCopies, 4);
    }
    if (o.methyl)
      for (std::size_t f = 0; f < cs.sample.size(); ++f)
        if (!cs.sample[f].methyl.empty()) put_methyl(o.methyl + 16 * (f * o.cap + i), cs.sample[f].methyl[v.id]);
    if (o.alleles) put_bytes(o.alleles, o.alleles_stride, o.alleles_len, i, v.alleles);
  }
}

// a single-sample call set as the one-file multi-sample set
static SrMultiCallSet one_sample(SrCallSet& cs) {
  SrMultiCallSet m; m.svs.swap(cs.svs); m.sample.resize(1);
  m.sample[0].jctMap.swap(cs.jctMap); m.sample[0].spanMap.swap(cs.spanMap); m.sample[0].rcMap.swap(cs.rcMap); m.sample[0].format.swap(cs.format);
  return m;
}
static LrMultiCallSet one_sample(LrCallSet& cs) {
  LrMultiCallSet m; m.svs.swap(cs.svs); m.sample.resize(1);
  m.sample[0].jctMap.swap(cs.jctMap); m.sample[0].rcMap.swap(cs.rcMap); m.sample[0].format.swap(cs.format); m.sample[0].methyl.swap(cs.methyl);
  return m;
}

// ---- in-process ranks ------------------------------------------------------------------------------------------------------------------

// N ranks as N host threads of one process, exchanging through a SimExchange: rank r runs run(r, gather, outs[r]) -> rc. The first rank to
// fail releases the others. Returns the first negative rank code; -100 when a rank's code or output differs from rank 0's (same(a, b) =
// equal); else rank 0's code, with its output moved to out0.
template <typename TOut, typename TRun, typename TSame>
static int run_ranks(int nranks, TRun run, TSame same, TOut& out0) {
  SimExchange ex(nranks);
  std::vector<TOut> outs((size_t) nranks);
  std::vector<int> rcs((size_t) nranks, 0);
  std::vector<std::thread> th;
  for (int r = 0; r < nranks; ++r) th.emplace_back([&, r] { rcs[r] = run(r, ex.of(r), outs[r]); if (rcs[r] < 0) ex.fail(); });
  for (auto& t : th) t.join();
  for (int r = 0; r < nranks; ++r) if (rcs[r] < 0) return rcs[r];
  for (int r = 1; r < nranks; ++r) if (rcs[r] != rcs[0] || !same(outs[r], outs[0])) return -100;
  out0 = std::move(outs[0]);
  return rcs[0];
}

// A rank's own zeroed copy of a chain hook's outputs, shaped by the hook's ChainOut (with every lr extra; copy_to copies those the hook
// has); compared with GL bits
struct ChainCopy {
  std::vector<int32_t> sv, fmt, cl, anno, methyl, al; std::vector<float> gl; std::vector<char> cons, alleles;
  ChainOut view(ChainOut const& like) {
    const std::size_t C = (std::size_t) like.cap, F = (std::size_t) like.nfile;
    sv.assign(C * 20, 0); fmt.assign(F * C * 14, 0); gl.assign(F * C * 3, 0.f); cons.assign(C * like.cons_stride, 0); cl.assign(C, 0);
    anno.assign(C * 5, 0); methyl.assign(F * C * 16, 0); alleles.assign(C * std::max(like.alleles_stride, 1), 0); al.assign(C, 0);
    return ChainOut{sv.data(), like.cap, fmt.data(), gl.data(), cons.data(), like.cons_stride, cl.data(), like.nfile, anno.data(), methyl.data(), alleles.data(),
                    like.alleles_stride, al.data()};
  }
  bool operator==(ChainCopy const& o) const {
    return sv == o.sv && fmt == o.fmt && cl == o.cl && cons == o.cons && anno == o.anno && methyl == o.methyl && alleles == o.alleles && al == o.al &&
           gl.size() == o.gl.size() && !memcmp(gl.data(), o.gl.data(), gl.size() * 4);
  }
  void copy_to(ChainOut const& d) const {
    memcpy(d.sv, sv.data(), sv.size() * 4); memcpy(d.fmt, fmt.data(), fmt.size() * 4); memcpy(d.gl, gl.data(), gl.size() * 4);
    memcpy(d.cons, cons.data(), cons.size()); memcpy(d.cons_len, cl.data(), cl.size() * 4);
    if (d.anno) memcpy(d.anno, anno.data(), anno.size() * 4);
    if (d.methyl) memcpy(d.methyl, methyl.data(), methyl.size() * 4);
    if (d.alleles) { memcpy(d.alleles, alleles.data(), (size_t) d.cap * d.alleles_stride); memcpy(d.alleles_len, al.data(), al.size() * 4); }
  }
};

// run_ranks over a chain hook: run(r, gather, out) writes rank r's outputs to out; rank 0's reach dst
template <typename TRun>
static int run_chain_ranks(int nranks, ChainOut const& dst, TRun run) {
  ChainCopy out;
  const int n = run_ranks(nranks, [&](int r, GatherFn gather, ChainCopy& o) { return run(r, gather, o.view(dst)); }, std::equal_to<ChainCopy>(), out);
  if (n >= 0) out.copy_to(dst);
  return n;
}

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
    const std::vector<std::pair<uint8_t, uint32_t> > cg = row_cigar(r, cigar);
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
  std::vector<SrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(sr_record(rec10 + 12 * i, cigar, reads, nullptr, nullptr, i));
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
  return put_qual_lists(countMap, nsv, qual_out, qual_cap, ref_off, alt_off);
}

// annotateSpanningAndDepth — the spanning-pair / read-depth outputs of oracle/ref_wrap3.cpp::ref_annotate_junction_reads (pure host).
// svOnChr is derived like _generateProbes does (src/coverage.h:179): a contig carries an SV end.
int dh_annotate_spanning(int len0, int len1, const int32_t* rec12, int nrec, const uint32_t* cigar, const int32_t* sv9, int nsv, int indelsize, int minGenoQual,
                         const int32_t* lib4, uint8_t* span_out, int span_cap, uint32_t* sref_off, uint32_t* salt_off, int32_t* rc_out) {
  Config c; c.indelsize = indelsize; c.minGenoQual = (uint16_t) minGenoQual;
  LibraryInfo lib; lib.median = lib4[0]; lib.minNormalISize = lib4[1]; lib.maxNormalISize = lib4[2]; lib.maxISizeCutoff = lib4[3];
  std::vector<uint32_t> tl = {(uint32_t) len0, (uint32_t) len1};
  std::vector<SrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(sr_record(rec12 + 12 * i, cigar, nullptr, nullptr, nullptr, i));
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
  const int sp = put_qual_lists(span, nsv, span_out, span_cap, sref_off, salt_off);
  if (sp < 0) return sp;
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
  const Genome g(contig_arena, contig_off, contig_len, ncontig);
  std::vector<SrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(sr_record(rec12 + 12 * i, cigar, reads, nullptr, nullptr, i));
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
  int rc = assembleSplitReadsBatch(ctx, c, g.tl, g.chr, srStore, svs, recs);
  if (rc) return rc;
  put_assembled(svs, sv_out, srq, cons_out, cons_stride, cons_len, alleles_out, alleles_stride, alleles_len);
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
  std::vector<SrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(sr_record(rec12 + 12 * i, cigar, nullptr, seeds, name_hash, i));
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
    put_sv(o, v); o[20] = v.alleleid; o[21] = v.nallele;
    put_bytes(alleles_out, astride, alen, i, v.alleles);
    put_bytes(cons_out, cstride, clen, i, v.consensus);
  }
  return n;
}

// The inputs of an sr chain hook. Records grouped by file: file_off[nfile + 1] (a single-sample hook is nfile = 1, file_off = {0, nrec});
// site22 (NULL = discovery): the sites of genotyping mode, rows as dh_vcf_parse. geno_* (may be NULL): a second record set, the whole
// contigs, for the genotyping pass when an exclude set restricts the first to the valid regions; valid_intervals (may be NULL = no exclude
// set): per contig, the number of valid regions the exclude set leaves.
struct SrInput {
  const char* contig_arena; const uint32_t* contig_off; const uint32_t* contig_len; int ncontig;
  const int32_t* rec12; const uint64_t* seeds; const uint32_t* name_hash; const uint32_t* file_off; int nfile;
  const uint32_t* cigar; const char* reads; const int32_t* lib6;
  const int32_t* site22; int nsite; const char* strs; const uint32_t* str_off;
  const int32_t* geno_rec12 = nullptr; const uint64_t* geno_seeds = nullptr; const uint32_t* geno_name_hash = nullptr; const uint32_t* geno_file_off = nullptr;
  const int32_t* valid_intervals = nullptr;
};

// What the sr entry points take, built from an SrInput. own (NULL = every row): keep only the rows of contigs [own[0], own[1]);
// held[ncontig] (may be NULL) counts the records kept, both sets.
struct SrRun {
  Config c; Genome g; std::vector<LibraryInfo> libs; std::vector<VcfSite> sites;
  std::vector<std::vector<SrRecord> > recs, geno; std::vector<std::vector<SrRecord> const*> samples, genoSamples;
  SrRun(SrRun const&) = delete;
  SrRun(SrInput const& in, const std::size_t* own, int64_t* held) : g(in.contig_arena, in.contig_off, in.contig_len, in.ncontig) {
    c.nchr = in.ncontig; c.maxThreads = 1;   // short-read defaults (src/delly.h:212-232)
    apply_svtset(c);
    if (in.valid_intervals) {   // the genome-wide region lists of the binding (dummy intervals: what matters is which lists are empty)
      std::vector<std::vector<int> > valid((size_t) in.ncontig);
      for (int t = 0; t < in.ncontig; ++t) valid[t].assign((size_t) in.valid_intervals[t], 0);
      c.contigExcluded = excludedContigs(valid);
    }
    if (in.site22) sites = sites_from_rows(in.site22, in.nsite, in.strs, in.str_off);
    auto read = [&](const int32_t* rec12, const uint64_t* seeds, const uint32_t* nh, uint32_t b, uint32_t e, std::vector<SrRecord>& out) {
      for (uint32_t i = b; i < e; ++i) {
        const int32_t* r = rec12 + 12 * (size_t) i;
        if (own && (r[0] < 0 || (std::size_t) r[0] < own[0] || (std::size_t) r[0] >= own[1])) continue;
        out.push_back(sr_record(r, in.cigar, in.reads, seeds, nh, i));
        if (held) ++held[r[0]];
      }
    };
    const std::size_t F = (std::size_t) in.nfile;
    libs.resize(F); recs.resize(F); geno.resize(in.geno_rec12 ? F : 0);
    for (std::size_t f = 0; f < F; ++f) {
      const int32_t* l = in.lib6 + 6 * f;
      libs[f].rs = l[0]; libs[f].median = l[1]; libs[f].mad = l[2]; libs[f].minNormalISize = l[3]; libs[f].maxNormalISize = l[4]; libs[f].maxISizeCutoff = l[5];
      read(in.rec12, in.seeds, in.name_hash, in.file_off[f], in.file_off[f + 1], recs[f]);
      samples.push_back(&recs[f]);
      if (in.geno_rec12) {
        read(in.geno_rec12, in.geno_seeds, in.geno_name_hash, in.geno_file_off[f], in.geno_file_off[f + 1], geno[f]);
        genoSamples.push_back(&geno[f]);
      }
    }
  }
};

// dellySrCall / dellySrGenotype (site22 != NULL) — layout as oracle/ref_wrap5.cpp::ref_delly_sr_call; genotyping sites as dh_vcf_parse
int dh_delly_sr_genotype(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                         const uint64_t* seeds, const uint32_t* name_hash, int nrec, const uint32_t* cigar, const char* reads, const int32_t* lib6, int32_t* sv_out,
                         int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const int32_t* site22, int nsite,
                         const char* strs, const uint32_t* str_off) {
  const uint32_t file_off[2] = {0, (uint32_t) nrec};
  const SrInput in{contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, file_off, 1, cigar, reads, lib6, site22, nsite, strs, str_off};
  SrRun s(in, nullptr, nullptr);
  SrCallSet cs;
  int rc = site22 ? dellySrGenotype(ctx, s.c, s.libs[0], s.g.tl, s.g.names, s.g.chr, s.sites, true, s.recs[0], cs)
                  : dellySrCall(ctx, s.c, s.libs[0], s.g.tl, s.g.names, s.g.chr, s.recs[0], cs);
  if (rc) return rc - 1;
  return write_calls(one_sample(cs), ChainOut{sv_out, cap, fmt_out, gl_out, cons_out, cons_stride, cons_len}, cols_spanning);
}

int dh_delly_sr_call(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, const uint32_t* name_hash, int nrec, const uint32_t* cigar, const char* reads, const int32_t* lib6, int32_t* sv_out,
                     int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return dh_delly_sr_genotype(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, nrec, cigar, reads, lib6, sv_out, cap, fmt_out, gl_out,
                              cons_out, cons_stride, cons_len, nullptr, 0, nullptr, nullptr);
}

// several samples in one call set — layout as oracle/ref_wrap5.cpp::ref_delly_sr_call_multi (records grouped by file, fmt_out / gl_out
// file-major); site22 != NULL = genotyping mode
int dh_delly_sr_genotype_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                               const uint64_t* seeds, const uint32_t* name_hash, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads,
                               const int32_t* lib6, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len,
                               const int32_t* site22, int nsite, const char* strs, const uint32_t* str_off) {
  const SrInput in{contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, file_off, nfile, cigar, reads, lib6, site22, nsite, strs, str_off};
  SrRun s(in, nullptr, nullptr);
  SrMultiCallSet cs;
  int rc = site22 ? dellySrGenotypeMulti(ctx, s.c, s.libs, s.g.tl, s.g.names, s.g.chr, s.sites, true, s.samples, cs)
                  : dellySrCallMulti(ctx, s.c, s.libs, s.g.tl, s.g.names, s.g.chr, s.samples, cs);
  if (rc) return rc - 1;
  return write_calls(cs, ChainOut{sv_out, cap, fmt_out, gl_out, cons_out, cons_stride, cons_len, nfile}, cols_spanning);
}

int dh_delly_sr_call_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                           const uint64_t* seeds, const uint32_t* name_hash, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads,
                           const int32_t* lib6, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return dh_delly_sr_genotype_multi(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, name_hash, file_off, nfile, cigar, reads, lib6, sv_out, cap,
                                    fmt_out, gl_out, cons_out, cons_stride, cons_len, nullptr, 0, nullptr, nullptr);
}

// assembleLRBatch — layout as oracle/ref_wrap5.cpp::ref_assemble_lr (read id = name id here)
int dh_assemble_lr(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec,
                   const uint32_t* cigar, const char* reads, const int32_t* store6, int nstore, const int32_t* sv12, int nsv, int maxReadPerSV, int minCliqueSize,
                   float flankQuality, int minimumFlankSize, int indelsize, int minConsWindow, int32_t* sv_out, float* srq, char* cons_out, int cons_stride,
                   int32_t* cons_len, char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  Config c; c.maxReadPerSV = (uint32_t) maxReadPerSV; c.minCliqueSize = (uint16_t) minCliqueSize;
  c.flankQuality = flankQuality; c.minimumFlankSize = minimumFlankSize; c.indelsize = indelsize; c.minConsWindow = minConsWindow;
  const Genome g(contig_arena, contig_off, contig_len, ncontig);
  std::vector<LrRecord> recs;
  std::vector<std::size_t> ids;
  for (int i = 0; i < nrec; ++i) {
    recs.push_back(lr_record(rec12 + 12 * i, cigar, reads, false, LrTags(), i));
    ids.push_back((std::size_t) rec12[12 * i + 11]);
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
  int rc = assembleLRBatch(ctx, c, g.tl, g.chr, svs, srStore, recs, ids);
  if (rc) return rc;
  put_assembled(svs, sv_out, srq, cons_out, cons_stride, cons_len, alleles_out, alleles_stride, alleles_len);
  return 0;
}

// The inputs of an lr chain hook: contigs, records, file_off and sites as SrInput (seeds NULL = read ids 0); cfg12 = minMapQual, minClip,
// minRefSep, maxReadSep, minCliqueSize, graphPruning, maxReadPerSV, minimumFlankSize, indelsize, minConsWindow, maxGenoReadCount, genoCap.
// tags.flags NULL = no MM / ML tags (and no methylation); tpl_arena NULL = no MEI templates (tpl_off[8] as load_mei); hpps: rows [8] / [9]
// are the HP / PS tags; valid (may be NULL = no exclude set): 1 for the records inside the valid regions of an exclude set (discovery
// sees those, genotyping all).
struct LrInput {
  const char* contig_arena; const uint32_t* contig_off; const uint32_t* contig_len; int ncontig;
  const int32_t* rec12; const uint64_t* seeds; const uint32_t* file_off; int nfile;
  const uint32_t* cigar; const char* reads; const int32_t* cfg12; float flankQuality, indelExtension;
  const int32_t* site22; int nsite; const char* strs; const uint32_t* str_off;
  LrTags tags = LrTags(); int methylWindow = 0, methylProb = 0, minCpgDepth = 0;
  const char* tpl_arena = nullptr; const uint32_t* tpl_off = nullptr; float meiMinFrac = 0.f, trMinFrac = 0.f;
  bool hpps = false; const uint8_t* valid = nullptr;
};

// What the lr entry points take, built from an LrInput; own and held as for SrRun (held counts a record of both lists twice)
struct LrRun {
  Config c; Genome g; std::vector<VcfSite> sites;
  MeiTemplates mei; AnnoConfig acfg; MethylConfig mcfg;
  MeiTemplates const* meiP; MethylConfig const* mcfgP;   // NULL without templates / tags
  std::vector<std::vector<LrRecord> > recs, whole; std::vector<std::vector<std::size_t> > ids, wholeIds; std::vector<LrSample> samples, genoSamples;
  LrRun(LrRun const&) = delete;
  LrRun(LrInput const& in, const std::size_t* own, int64_t* held) : g(in.contig_arena, in.contig_off, in.contig_len, in.ncontig) {
    const int32_t* k = in.cfg12;
    c.minMapQual = (uint16_t) k[0]; c.minClip = (uint32_t) k[1]; c.minRefSep = (uint32_t) k[2]; c.maxReadSep = (uint32_t) k[3];
    c.minCliqueSize = (uint16_t) k[4]; c.graphPruning = (uint32_t) k[5]; c.maxReadPerSV = (uint32_t) k[6]; c.minimumFlankSize = k[7];
    c.indelsize = k[8]; c.minConsWindow = k[9]; c.maxGenoReadCount = (uint32_t) k[10]; c.genoCap = k[11];
    c.flankQuality = in.flankQuality; c.nchr = in.ncontig;
    apply_svtset(c);
    if (in.site22) sites = sites_from_rows(in.site22, in.nsite, in.strs, in.str_off);
    if (in.tpl_arena) load_mei(mei, in.tpl_arena, in.tpl_off);
    acfg.meiMinFrac = in.meiMinFrac; acfg.trMinFrac = in.trMinFrac;
    mcfg.methylWindow = in.methylWindow; mcfg.methylProb = (uint16_t) in.methylProb; mcfg.minCpgDepth = (uint32_t) in.minCpgDepth;
    meiP = in.tpl_arena ? &mei : nullptr;
    mcfgP = in.tags.flags ? &mcfg : nullptr;
    const std::size_t F = (std::size_t) in.nfile;
    recs.resize(F); ids.resize(F); whole.resize(in.valid ? F : 0); wholeIds.resize(in.valid ? F : 0);
    for (std::size_t f = 0; f < F; ++f) {
      for (uint32_t i = in.file_off[f]; i < in.file_off[f + 1]; ++i) {
        const int32_t* r = in.rec12 + 12 * (size_t) i;
        if (own && (r[0] < 0 || (std::size_t) r[0] < own[0] || (std::size_t) r[0] >= own[1])) continue;
        const LrRecord rec = lr_record(r, in.cigar, in.reads, in.hpps, in.tags, i);
        const std::size_t id = in.seeds ? (std::size_t) in.seeds[i] : 0;
        if (!in.valid || in.valid[i]) { recs[f].push_back(rec); ids[f].push_back(id); if (held) ++held[r[0]]; }
        if (in.valid) { whole[f].push_back(rec); wholeIds[f].push_back(id); if (held) ++held[r[0]]; }
      }
      samples.push_back(LrSample{&recs[f], &ids[f]});
      if (in.valid) genoSamples.push_back(LrSample{&whole[f], &wholeIds[f]});
    }
  }
};

// dellyLrCall over one file, or dellyLrCallSharded as one rank of a sharded run (shard != NULL)
static int delly_lr_call(dgpu_ctx* ctx, LrInput const& in, Shard const* shard, ChainOut const& o) {
  LrRun s(in, nullptr, nullptr);
  LrMultiCallSet cs;
  int rc;
  if (shard) rc = dellyLrCallSharded(ctx, s.c, in.indelExtension, s.g.tl, s.g.names, s.g.chr, s.samples, *shard, cs, s.meiP, s.acfg, s.mcfgP);
  else {
    LrCallSet one;
    rc = dellyLrCall(ctx, s.c, in.indelExtension, s.g.tl, s.g.names, s.g.chr, s.recs[0], s.ids[0], one, s.meiP, s.acfg, s.mcfgP);
    cs = one_sample(one);
  }
  if (rc) return rc - 1;
  const int n = write_calls(cs, o, cols_zero);
  if (n >= 0) write_lr_extras(cs, o);
  return n;
}

// the complete long-read chain — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call_ex plus the template sequences; seeds = the read ids
// (hash_lr of the query names)
int dh_delly_lr_call_ex(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                        const uint64_t* seeds, int nrec, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, float indelExtension,
                        int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len, const uint8_t* tagflags,
                        const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off, int methylWindow, int methylProb,
                        int minCpgDepth, const char* tpl_arena, const uint32_t* tpl_off, float meiMinFrac, float trMinFrac, int32_t* anno_out, int32_t* methyl_out,
                        char* alleles_out, int alleles_stride, int32_t* alleles_len) {
  const uint32_t file_off[2] = {0, (uint32_t) nrec};
  const LrInput in{contig_arena, contig_off, contig_len, ncontig, rec12, seeds, file_off, 1, cigar, reads, cfg12, flankQuality, indelExtension, nullptr, 0, nullptr,
                   nullptr, LrTags{tagflags, mm_arena, mm_off, ml_arena, ml_off}, methylWindow, methylProb, minCpgDepth, tpl_arena, tpl_off, meiMinFrac, trMinFrac};
  return delly_lr_call(ctx, in, nullptr, ChainOut{sv_out, cap, fmt_out, gl_out, cons_out, cons_stride, cons_len, 1, anno_out, methyl_out, alleles_out, alleles_stride,
                                                  alleles_len});
}

// dellyLrCall — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call
int dh_delly_lr_call(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                     const uint64_t* seeds, int nrec, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, float indelExtension,
                     int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  return dh_delly_lr_call_ex(ctx, contig_arena, contig_off, contig_len, ncontig, rec12, seeds, nrec, cigar, reads, cfg12, flankQuality, indelExtension, sv_out, cap,
                             fmt_out, gl_out, cons_out, cons_stride, cons_len, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nullptr, nullptr, 0.f, 0.f,
                             nullptr, nullptr, nullptr, 0, nullptr);
}

// several long-read samples — layout as oracle/ref_wrap5.cpp::ref_delly_lr_call_multi
int dh_delly_lr_call_multi(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12,
                           const uint64_t* seeds, const uint32_t* file_off, int nfile, const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality,
                           float indelExtension, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out, char* cons_out, int cons_stride, int32_t* cons_len) {
  const LrInput in{contig_arena, contig_off, contig_len, ncontig, rec12, seeds, file_off, nfile, cigar, reads, cfg12, flankQuality, indelExtension, nullptr, 0,
                   nullptr, nullptr};
  LrRun s(in, nullptr, nullptr);
  LrMultiCallSet cs;
  int rc = dellyLrCallMulti(ctx, s.c, indelExtension, s.g.tl, s.g.names, s.g.chr, s.samples, cs);
  if (rc) return rc - 1;
  return write_calls(cs, ChainOut{sv_out, cap, fmt_out, gl_out, cons_out, cons_stride, cons_len, nfile}, cols_zero);
}

// long-read genotyping mode: one sample, the outputs of dh_delly_lr_call for a given site list (rows as dh_vcf_parse) except the consensus
int dh_delly_lr_genotype(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec,
                         const uint32_t* cigar, const char* reads, const int32_t* cfg12, float flankQuality, const int32_t* site22, int nsite, const char* strs,
                         const uint32_t* str_off, int32_t* sv_out, int cap, int32_t* fmt_out, float* gl_out) {
  const uint32_t file_off[2] = {0, (uint32_t) nrec};
  const LrInput in{contig_arena, contig_off, contig_len, ncontig, rec12, nullptr, file_off, 1, cigar, reads, cfg12, flankQuality, 0.f, site22, nsite, strs, str_off};
  LrRun s(in, nullptr, nullptr);
  LrMultiCallSet cs;
  int rc = dellyLrGenotype(ctx, s.c, s.g.tl, s.g.names, s.g.chr, s.sites, true, s.samples, cs);
  if (rc) return rc - 1;
  return write_calls(cs, ChainOut{sv_out, cap, fmt_out, gl_out, nullptr, 0, nullptr}, cols_zero);
}

// clusterSRReadsLR — layout as oracle/ref_wrap5.cpp::ref_cluster_sr_reads (ctx may be NULL: host pair scans)
int dh_cluster_sr_reads(dgpu_ctx* ctx, const uint32_t* contig_len, int ncontig, const int32_t* rec12, const uint64_t* seeds, int nrec, const uint32_t* cigar,
                        const int32_t* cfg12, float indelExtension, int32_t* sv_out, int cap, int32_t* store_out, uint64_t* store_seed, int store_cap, int32_t* n_out) {
  Config c;
  c.minMapQual = (uint16_t) cfg12[0]; c.minClip = (uint32_t) cfg12[1]; c.minRefSep = (uint32_t) cfg12[2]; c.maxReadSep = (uint32_t) cfg12[3];
  c.minCliqueSize = (uint16_t) cfg12[4]; c.graphPruning = (uint32_t) cfg12[5]; c.nchr = ncontig;
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<LrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(lr_record(rec12 + 12 * i, cigar, nullptr, false, LrTags(), i));
  std::vector<std::size_t> ids(seeds, seeds + nrec);
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

// LibraryInfo as 7 ints: rs, median, mad, minNormalISize, minISizeCutoff, maxNormalISize, maxISizeCutoff
static void put_lib7(LibraryInfo const& l, int32_t* o) {
  o[0] = l.rs; o[1] = l.median; o[2] = l.mad; o[3] = l.minNormalISize; o[4] = l.minISizeCutoff; o[5] = l.maxNormalISize; o[6] = l.maxISizeCutoff;
}

// getLibraryParams — layout as oracle/ref_wrap6.cpp::ref_get_library_params (the screen reads no CIGAR)
int dh_get_library_params(const uint32_t* contig_len, int ncontig, const int32_t* rec12, int nrec, const uint32_t* cigar, int madCutoff, int madNormalCutoff,
                          int32_t* out7) {
  Config c; c.madCutoff = (uint16_t) madCutoff; c.madNormalCutoff = (uint16_t) madNormalCutoff;
  std::vector<uint32_t> tl(contig_len, contig_len + ncontig);
  std::vector<SrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(sr_record(rec12 + 12 * i, nullptr, nullptr, nullptr, nullptr, i));
  LibraryInfo l;
  getLibraryParams(c, tl, recs, l);
  put_lib7(l, out7);
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

// genotypeLRBatch with MM / ML tags (tagflags may be NULL) — layout as oracle/ref_wrap4.cpp::ref_genotype_lr_methyl (contigs named "chr0",
// "chr1", ...; record rows of 10: [8] = HP, [9] = PS)
int dh_genotype_lr_methyl(dgpu_ctx* ctx, const char* contig_arena, const uint32_t* contig_off, const uint32_t* contig_len, int ncontig, const int32_t* rec10,
                          int nrec, const uint32_t* cigar, const char* reads, const int32_t* sv8, int nsv, const char* cons_arena, const uint32_t* cons_off,
                          const uint32_t* cons_len, int minMapQual, int minimumFlankSize, int minConsWindow, int maxGenoReadCount, float flankQuality,
                          int genoCap, uint8_t* qual_out, int qual_cap, uint32_t* ref_off, uint32_t* alt_off, int32_t* hp_out, int32_t* rc_out,
                          const uint8_t* tagflags, const char* mm_arena, const uint32_t* mm_off, const uint8_t* ml_arena, const uint32_t* ml_off,
                          int methylWindow, int methylProb, int minCpgDepth, int32_t* methyl_out) {
  Config c; c.minMapQual = (uint16_t) minMapQual; c.minimumFlankSize = minimumFlankSize; c.minConsWindow = minConsWindow;
  c.maxGenoReadCount = (uint32_t) maxGenoReadCount; c.flankQuality = flankQuality; c.genoCap = genoCap;
  const Genome g(contig_arena, contig_off, contig_len, ncontig);
  const LrTags tags{tagflags, mm_arena, mm_off, ml_arena, ml_off};
  std::vector<LrRecord> recs;
  for (int i = 0; i < nrec; ++i) recs.push_back(lr_record(rec10 + 10 * i, cigar, reads, true, tags, i));
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
  int rc = genotypeLRBatch(ctx, c, g.tl, g.names, g.chr, svs, recs, jct, cov, tagflags ? &mcfg : nullptr, tagflags ? &methyl : nullptr);
  if (rc) return rc - 1;
  if (tagflags && methyl_out) for (int i = 0; i < nsv; ++i) put_methyl(methyl_out + 16 * i, methyl[i]);
  const int pos = put_qual_lists(jct, nsv, qual_out, qual_cap, ref_off, alt_off);
  if (pos < 0) return pos;
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
  return dh_genotype_lr_methyl(ctx, contig_arena, contig_off, contig_len, ncontig, rec10, nrec, cigar, reads, sv8, nsv, cons_arena, cons_off, cons_len, minMapQual,
                               minimumFlankSize, minConsWindow, maxGenoReadCount, flankQuality, genoCap, qual_out, qual_cap, ref_off, alt_off, hp_out, rc_out,
                               nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nullptr);
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
  if (tpl_arena && tpl_off) load_mei(mei, tpl_arena, tpl_off);
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
