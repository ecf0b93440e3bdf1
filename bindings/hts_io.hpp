// hts_io.hpp — the htslib side of the binding (BAM / FASTA / BCF in, BCF / VCF out). Everything here is IO glue around the batched
// host mirrors of delly_b200/host: it turns what the reference's drivers read per bam1_t into the record lists the mirrors take, and the
// field-by-field record description of host/vcf.hpp into the htslib calls vcfOutput makes. References:
//   src/shortpe.h:349-352, src/junction.h:347-350  record iteration (sam_itr_queryi per contig over the valid regions)
//   src/util.h:519-542                              read ids (hash_sr, hash_lr)
//   src/tags.h:260-267                              hash_string
//   src/util.h:626-664, :194-205                    getSMTag, checkSampleNames
//   src/util.h:666-741                              _parseExcludeIntervals
//   src/modvcf.h:156-339                            vcfParse (the bcf_get_info_* calls; the per-record rules are host/vcfparse.hpp)
//   src/modvcf.h:344-791                            vcfOutput (the bcf_hdr_append / bcf_update_* / bcf_write1 calls)
// htslib is the reference's own IO dependency and stays what it is (tools/build_htslib.sh builds the vendored 1.21).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <fstream>
#include <functional>
#include <iostream>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include <htslib/faidx.h>
#include <htslib/sam.h>
#include <htslib/vcf.h>

#include "../delly_b200/host/pipeline.hpp"
#include "../delly_b200/host/vcf.hpp"

namespace dellyb200 {
namespace io {

// ---- read ids --------------------------------------------------------------------------------------------------------------
// boost::hash_combine / hash_range as the oracle build defines them (oracle/shim11/boost/filesystem.hpp): the classic formula over
// std::hash. The ids are opaque; what matters is that containers keyed by them iterate in the same order on both sides.
template <typename T> inline void hashCombine(std::size_t& seed, T const& v) { seed ^= std::hash<T>()(v) + 0x9e3779b9 + (seed << 6) + (seed >> 2); }

inline unsigned hashString(const char* s) {  // src/tags.h:260-267
  unsigned h = 37;
  while (*s) { h = (h * 54059) ^ (s[0] * 76963); s++; }
  return h;
}

inline std::size_t hashSr(bam1_t const* rec) {  // src/util.h:519-527
  const char* q = bam_get_qname(rec);
  std::size_t seed = hashString(q);
  std::size_t prehash = 0;
  for (const char* p = q; *p; ++p) hashCombine(prehash, *p);
  hashCombine(seed, prehash);
  if ((rec->core.flag & BAM_FREAD1) && (seed > 0)) --seed;
  return seed;
}

inline std::size_t hashLr(bam1_t const* rec) {  // src/util.h:529-535
  const std::string qname = bam_get_qname(rec);
  std::size_t seed = hashString(qname.c_str());
  hashCombine(seed, std::hash<std::string>()(qname));
  return seed;
}

inline void decodeSeq(bam1_t const* rec, std::string& out) {  // "=ACMGRSVTWYHKDBN"[bam_seqi(seq, i)], as every stage of the reference decodes it
  const int32_t l = rec->core.l_qseq;
  out.resize((std::size_t) l);
  const uint8_t* seq = bam_get_seq(rec);
  for (int32_t i = 0; i < l; ++i) out[i] = "=ACMGRSVTWYHKDBN"[bam_seqi(seq, i)];
}

template <typename TRec> inline void fillCore(bam1_t const* rec, TRec& r) {
  r.tid = rec->core.tid; r.pos = (int32_t) rec->core.pos; r.flag = rec->core.flag; r.mapq = rec->core.qual;
  const uint32_t* cigar = bam_get_cigar(rec);
  r.cigar.resize(rec->core.n_cigar);
  for (uint32_t i = 0; i < rec->core.n_cigar; ++i) r.cigar[i] = std::make_pair((uint8_t) bam_cigar_op(cigar[i]), (uint32_t) bam_cigar_oplen(cigar[i]));
  decodeSeq(rec, r.seq);
}

inline void toSrRecord(bam1_t const* rec, SrRecord& r) {
  fillCore(rec, r);
  r.lqseq = rec->core.l_qseq; r.mtid = rec->core.mtid; r.mpos = (int32_t) rec->core.mpos; r.isize = (int32_t) rec->core.isize;
  r.name = (uint64_t) std::hash<std::string>()(bam_get_qname(rec));
  r.nameHash32 = hashString(bam_get_qname(rec));
  r.seed = hashSr(rec);
}

inline void toLrRecord(bam1_t const* rec, LrRecord& r) {
  fillCore(rec, r);
  // src/genotype.h:219-222
  uint8_t* hpTag = bam_aux_get(rec, "HP");
  if (hpTag) r.hp = (uint8_t) bam_aux2i(hpTag);
  uint8_t* psTag = bam_aux_get(rec, "PS");
  if (psTag) r.ps = (int32_t) bam_aux2i(psTag);
  // src/methyl.h:126-127, :189-199
  uint8_t* mm = bam_aux_get(rec, "MM");
  if (mm && (*mm == 'Z')) { r.hasMM = true; r.mm = reinterpret_cast<const char*>(mm + 1); }
  uint8_t* ml = bam_aux_get(rec, "ML");
  if (ml && (*ml == 'B') && (*reinterpret_cast<char*>(ml + 1) == 'C')) {
    const uint8_t* p = ml + 2;
    const int32_t n = (int32_t) (p[0] | ((uint32_t) p[1] << 8) | ((uint32_t) p[2] << 16) | ((uint32_t) p[3] << 24));
    r.hasML = true;
    r.ml.assign(p + 4, p + 4 + (n > 0 ? n : 0));
  }
}

// ---- alignment file -------------------------------------------------------------------------------------------------------
struct Interval { uint32_t lo, hi; };
typedef std::vector<std::vector<Interval> > TRegionsGenome;

struct AlignmentFile {
  samFile* fp = nullptr;
  hts_idx_t* idx = nullptr;
  bam_hdr_t* hdr = nullptr;
  std::string path;
  ~AlignmentFile() { if (hdr) bam_hdr_destroy(hdr); if (idx) hts_idx_destroy(idx); if (fp) sam_close(fp); }
  bool open(std::string const& p, std::string const& genome, int ioThreads) {
    path = p;
    fp = sam_open(p.c_str(), "r");
    if (!fp) { std::cerr << "Fail to open file " << p << std::endl; return false; }
    hts_set_fai_filename(fp, genome.c_str());
    if (ioThreads > 1) hts_set_threads(fp, ioThreads);   // bgzf decompression off the scan thread (SURVEY §8f row 1)
    idx = sam_index_load(fp, p.c_str());
    if (!idx) { std::cerr << "Fail to open index for " << p << std::endl; return false; }
    hdr = sam_hdr_read(fp);
    if (!hdr) { std::cerr << "Fail to open header for " << p << std::endl; return false; }
    return true;
  }
  // The same record stream read by several threads (SURVEY section 8f row 1: BAM ingestion is the end-to-end wall of the reference): every valid
  // region is cut into chunks of `chunk` bp, each chunk is read through its own file handle and iterator, and a record belongs to the chunk that
  // contains its start position (an iterator also returns the reads that merely overlap its interval; of those a later chunk keeps only what
  // starts inside it, the first chunk of a region keeps everything — exactly what the single iterator over the region returns, in its order).
  // names: the query name of every record, kept only for the SV-read dump (a sample has millions of records).
  template <typename TRec, typename TFill>
  bool readRegionsParallel(std::string const& genome, TRegionsGenome const& regions, std::vector<TRec>& out, TFill fill, int threads, std::vector<std::size_t>* ids = nullptr,
                           std::size_t (*idfn)(bam1_t const*) = nullptr, uint32_t chunk = 0, std::vector<std::string>* names = nullptr) {
    if (!chunk) {   // about four chunks per thread, between 256 kbp and 4 Mbp
      uint64_t total = 0;
      for (auto const& v : regions) for (Interval const& iv : v) total += iv.hi - iv.lo;
      chunk = (uint32_t) std::min<uint64_t>(4000000, std::max<uint64_t>(262144, total / (4 * (uint64_t) std::max(1, threads))));
    }
    struct Task { int32_t tid; uint32_t lo, hi; bool firstOfRegion; std::vector<TRec> recs; std::vector<std::size_t> ids; std::vector<std::string> names; };
    std::vector<Task> tasks;
    for (int32_t refIndex = 0; refIndex < hdr->n_targets; ++refIndex)
      for (Interval const& iv : regions[refIndex])
        for (uint32_t b = iv.lo; b < iv.hi; b += chunk) { Task t; t.tid = refIndex; t.lo = b; t.hi = std::min<uint64_t>((uint64_t) b + chunk, iv.hi); t.firstOfRegion = (b == iv.lo); tasks.push_back(std::move(t)); }
    if (threads < 2 || tasks.size() < 2) { readRegions(regions, out, fill, ids, idfn, names); return true; }
    std::atomic<std::size_t> next(0);
    std::atomic<bool> failed(false);
    auto worker = [&]() {
      samFile* f = sam_open(path.c_str(), "r");
      if (!f) { failed = true; return; }
      hts_set_fai_filename(f, genome.c_str());
      hts_idx_t* ix = sam_index_load(f, path.c_str());
      bam_hdr_t* h = sam_hdr_read(f);
      if (!ix || !h) { failed = true; if (h) bam_hdr_destroy(h); if (ix) hts_idx_destroy(ix); sam_close(f); return; }
      bam1_t* rec = bam_init1();
      for (std::size_t k = next++; k < tasks.size(); k = next++) {
        Task& t = tasks[k];
        hts_itr_t* iter = sam_itr_queryi(ix, t.tid, t.lo, t.hi);
        while (sam_itr_next(f, iter, rec) >= 0) {
          if (!t.firstOfRegion && (rec->core.pos < (hts_pos_t) t.lo)) continue;   // belongs to an earlier chunk
          t.recs.emplace_back();
          fill(rec, t.recs.back());
          if (ids) t.ids.push_back(idfn(rec));
          if (names) t.names.emplace_back(bam_get_qname(rec));
        }
        hts_itr_destroy(iter);
      }
      bam_destroy1(rec); bam_hdr_destroy(h); hts_idx_destroy(ix); sam_close(f);
    };
    std::vector<std::thread> pool;
    for (int i = 0; i < threads; ++i) pool.emplace_back(worker);
    for (auto& th : pool) th.join();
    if (failed) return false;
    // the tasks' records into one list in task order: slices moved in parallel
    std::vector<std::size_t> off(tasks.size() + 1, out.size());
    for (std::size_t k = 0; k < tasks.size(); ++k) off[k + 1] = off[k] + tasks[k].recs.size();
    out.resize(off[tasks.size()]);
    if (ids) ids->resize(off[tasks.size()]);
    if (names) names->resize(off[tasks.size()]);
    std::atomic<std::size_t> nextMove(0);
    auto mover = [&]() {
      for (std::size_t k = nextMove++; k < tasks.size(); k = nextMove++) {
        std::move(tasks[k].recs.begin(), tasks[k].recs.end(), out.begin() + (std::ptrdiff_t) off[k]);
        if (ids) std::copy(tasks[k].ids.begin(), tasks[k].ids.end(), ids->begin() + (std::ptrdiff_t) off[k]);
        if (names) std::move(tasks[k].names.begin(), tasks[k].names.end(), names->begin() + (std::ptrdiff_t) off[k]);
        std::vector<TRec>().swap(tasks[k].recs);
      }
    };
    std::vector<std::thread> movers;
    for (int i = 1; i < threads; ++i) movers.emplace_back(mover);
    mover();
    for (auto& th : movers) th.join();
    return true;
  }
  // every record the reference's iterators return: contig by contig, region by region (a read over two regions comes twice, as there)
  template <typename TRec, typename TFill>
  void readRegions(TRegionsGenome const& regions, std::vector<TRec>& out, TFill fill, std::vector<std::size_t>* ids = nullptr, std::size_t (*idfn)(bam1_t const*) = nullptr,
                   std::vector<std::string>* names = nullptr) {
    bam1_t* rec = bam_init1();
    for (int32_t refIndex = 0; refIndex < hdr->n_targets; ++refIndex) {
      for (Interval const& iv : regions[refIndex]) {
        hts_itr_t* iter = sam_itr_queryi(idx, refIndex, iv.lo, iv.hi);
        while (sam_itr_next(fp, iter, rec) >= 0) {
          out.emplace_back();
          fill(rec, out.back());
          if (ids) ids->push_back(idfn(rec));
          if (names) names->emplace_back(bam_get_qname(rec));
        }
        hts_itr_destroy(iter);
      }
    }
    bam_destroy1(rec);
  }
};

inline void getSMTag(std::string const& header, std::string const& fileName, std::string& sampleName) {  // src/util.h:626-664
  std::set<std::string> smIdentifiers;
  bool rgPresent = false;
  std::size_t b = 0;
  while (b <= header.size()) {
    std::size_t e = header.find('\n', b);
    if (e == std::string::npos) e = header.size();
    const std::string line = header.substr(b, e - b);
    if (line.find("@RG") == 0) {
      std::size_t kb = 0;
      while (kb <= line.size()) {
        std::size_t ke = line.find('\t', kb);
        if (ke == std::string::npos) ke = line.size();
        const std::string kv = line.substr(kb, ke - kb);
        const std::size_t sp = kv.find(':');
        if ((sp != std::string::npos) && (kv.substr(0, sp) == "SM")) { rgPresent = true; smIdentifiers.insert(kv.substr(sp + 1)); }
        kb = ke + 1;
      }
    }
    b = e + 1;
  }
  if (!rgPresent) sampleName = fileName;
  else if (smIdentifiers.size() == 1) sampleName = *smIdentifiers.begin();
  else if (smIdentifiers.size() > 1) { sampleName = *smIdentifiers.begin(); std::cerr << "Warning: Multiple sample names (@RG:SM) present in the BAM file!" << std::endl; }
}

inline std::string fileStem(std::string const& p) {  // boost::filesystem::path::stem
  const std::size_t k = p.rfind('/');
  std::string f = (k == std::string::npos) ? p : p.substr(k + 1);
  const std::size_t d = f.rfind('.');
  return (d == std::string::npos || d == 0) ? f : f.substr(0, d);
}

inline void checkSampleNames(std::vector<std::string>& sampleName) {  // src/util.h:194-205
  uint32_t ucount = 0;
  std::set<std::string> snames;
  for (std::string& nm : sampleName) {
    while (snames.count(nm)) {
      std::cerr << "Warning: Duplicate sample names: " << nm << std::endl;
      nm += "_" + std::to_string(ucount++);
      std::cerr << "Warning: Changing sample name to " << nm << std::endl;
    }
    snames.insert(nm);
  }
}

// src/util.h:666-741. Exclude lines: "chr" (whole contig) or "chr start end", separated by blank / tab / ',' / ';'.
inline bool parseExcludeIntervals(bool hasExcludeFile, std::string const& exclude, bam_hdr_t* hdr, TRegionsGenome& validRegions) {
  const int32_t n = hdr->n_targets;
  validRegions.assign(n, std::vector<Interval>());
  std::vector<std::vector<Interval> > exclg(n);
  std::vector<bool> validChr(n, true);
  auto insertJoined = [](std::vector<Interval>& v, Interval iv) {   // boost::icl::interval_set::insert: joins overlapping and touching intervals
    std::vector<Interval> out;
    bool placed = false;
    for (Interval const& x : v) {
      if (x.hi < iv.lo) out.push_back(x);
      else if (iv.hi < x.lo) { if (!placed) { out.push_back(iv); placed = true; } out.push_back(x); }
      else { if (x.lo < iv.lo) iv.lo = x.lo; if (iv.hi < x.hi) iv.hi = x.hi; }
    }
    if (!placed) out.push_back(iv);
    v.swap(out);
  };
  if (hasExcludeFile) {
    std::ifstream chrFile(exclude.c_str());
    std::string line;
    while (chrFile.good()) {
      std::getline(chrFile, line);
      std::vector<std::string> tok;
      std::string cur;
      for (char ch : line) {
        if (std::strchr(" \t,;", ch)) { if (!cur.empty()) tok.push_back(cur); cur.clear(); }
        else cur.push_back(ch);
      }
      if (!cur.empty()) tok.push_back(cur);
      if (tok.empty()) continue;
      const int32_t tid = bam_name2id(hdr, tok[0].c_str());
      if (tid < 0) continue;
      if (tok.size() == 1) { validChr[tid] = false; continue; }
      auto bad = [&]() { std::cerr << "Exclude file needs to be in tab-delimited format: chr, start, end" << std::endl << "Offending line: " << line << std::endl; return false; };
      auto toInt = [](std::string const& s, int32_t& v) { std::istringstream is(s); is >> v; return !is.fail() && is.eof(); };
      int32_t start = 0, end = 0;
      if (!toInt(tok[1], start)) return bad();
      if (tok.size() < 3) return bad();
      if (!toInt(tok[2], end)) return bad();
      if (start < end) insertJoined(exclg[tid], Interval{(uint32_t) start, (uint32_t) end});
      else { std::cerr << "Exclude file needs to be in tab-delimited format (chr, start, end) and start < end." << std::endl << "Offending line: " << line << std::endl; return false; }
    }
  }
  for (int32_t i = 0; i < n; ++i) {
    if (!validChr[i]) continue;
    uint32_t istart = 0;
    for (Interval const& it : exclg[i]) {
      if (istart + 1 < it.lo) insertJoined(validRegions[i], Interval{istart, it.lo - 1});
      istart = it.hi;
    }
    if (istart + 1 < hdr->target_len[i]) insertJoined(validRegions[i], Interval{istart, hdr->target_len[i]});
  }
  return true;
}

// ---- reference genome ------------------------------------------------------------------------------------------------------
struct Genome {
  std::vector<char*> seq;          // faidx_fetch_seq buffers, one per BAM contig (nullptr when the FASTA lacks it)
  std::vector<const char*> cseq;
  ~Genome() { for (char* s : seq) if (s) free(s); }
  // Loads the contigs named by the BAM header whole (the reference loads them one at a time per stage; every stage reads the same bytes).
  bool load(std::string const& fasta, bam_hdr_t* hdr, bool requireAll) {
    faidx_t* fai = fai_load(fasta.c_str());
    if (!fai) { std::cerr << "Fail to open genome fai index for " << fasta << std::endl; return false; }
    static const char empty[1] = {0};
    for (int32_t i = 0; i < hdr->n_targets; ++i) {
      char* s = nullptr;
      if (faidx_has_seq(fai, hdr->target_name[i])) {
        int32_t seqlen = -1;
        s = faidx_fetch_seq(fai, hdr->target_name[i], 0, hdr->target_len[i], &seqlen);
      } else if (requireAll) {
        std::cerr << "BAM file chromosome " << hdr->target_name[i] << " is NOT present in your reference file " << fasta << std::endl;
        fai_destroy(fai);
        return false;
      } else std::cerr << "Warning: BAM file chromosome " << hdr->target_name[i] << " is NOT present in your reference file " << fasta << " and will be skipped." << std::endl;
      seq.push_back(s);
      cseq.push_back(s ? s : empty);
    }
    fai_destroy(fai);
    return true;
  }
};

// ---- site list (`-v`) ------------------------------------------------------------------------------------------------------
inline bool isKeyPresent(bcf_hdr_t const* hdr, std::string const& key) {  // src/modvcf.h:139-150 (_isKeyPresent)
  for (int i = 0; i < hdr->n[BCF_DT_ID]; ++i) {
    const std::string k(hdr->id[BCF_DT_ID][i].key);
    if (k == key) return true;
  }
  return false;
}

inline bool readSites(std::string const& vcffile, std::vector<VcfSite>& sites, bool& headerHasConsBp) {
  htsFile* ifile = bcf_open(vcffile.c_str(), "r");
  if (!ifile) { std::cerr << "Fail to open file " << vcffile << std::endl; return false; }
  bcf_hdr_t* hdr = bcf_hdr_read(ifile);
  if (!hdr) { std::cerr << "Fail to open index file " << vcffile << std::endl; bcf_close(ifile); return false; }
  headerHasConsBp = isKeyPresent(hdr, "CONSBP");
  bcf1_t* rec = bcf_init();
  int32_t ni = 0; int32_t* vi = nullptr;
  int32_t nf = 0; float* vf = nullptr;
  int32_t ns = 0; char* vs = nullptr;
  auto getInt = [&](const char* key, VcfOpt<int32_t>& o) { if (bcf_get_info_int32(hdr, rec, key, &vi, &ni) > 0) { o.present = true; o.value = *vi; } };
  auto getStr = [&](const char* key, VcfOpt<std::string>& o) { if (bcf_get_info_string(hdr, rec, key, &vs, &ns) > 0) { o.present = true; o.value = std::string(vs); } };
  while (bcf_read(ifile, hdr, rec) == 0) {
    bcf_unpack(rec, BCF_UN_INFO);
    VcfSite s;
    s.chrom = bcf_hdr_id2name(hdr, rec->rid);
    s.pos0 = (int32_t) rec->pos;
    s.qual = rec->qual;
    s.ref = rec->d.allele[0];
    if (rec->n_allele > 1) s.alt = rec->d.allele[1];
    s.precise = bcf_get_info_flag(hdr, rec, "PRECISE", 0, 0) > 0;
    getStr("SVMETHOD", s.svMethod); getStr("SVTYPE", s.svType); getStr("CT", s.ct); getStr("CHR2", s.chr2); getStr("CONSENSUS", s.consensus);
    getInt("PE", s.pe); getInt("INSLEN", s.insLen); getInt("SVLEN", s.svLen); getInt("HOMLEN", s.homLen); getInt("SR", s.sr); getInt("END", s.end);
    getInt("POS2", s.pos2); getInt("CONSBP", s.consBp); getInt("MAPQ", s.mapq); getInt("SRMAPQ", s.srMapq); getInt("ALLELEID", s.alleleId); getInt("NALLELE", s.nAllele);
    if (bcf_get_info_float(hdr, rec, "SRQ", &vf, &nf) > 0) { s.srq.present = true; s.srq.value = *vf; }
    if (bcf_get_info_int32(hdr, rec, "CIPOS", &vi, &ni) > 0) { s.hasCipos = true; s.cipos[0] = vi[0]; s.cipos[1] = vi[1]; }
    if (bcf_get_info_int32(hdr, rec, "CIEND", &vi, &ni) > 0) { s.hasCiend = true; s.ciend[0] = vi[0]; s.ciend[1] = vi[1]; }
    sites.push_back(s);
  }
  free(vi); free(vf); free(vs);
  bcf_destroy(rec);
  bcf_hdr_destroy(hdr);
  bcf_close(ifile);
  return true;
}

// ---- BCF / VCF output ------------------------------------------------------------------------------------------------------
// The Sink of host/vcf.hpp::vcfRecordsTo: each described field becomes the htslib call vcfOutput makes, in the same order.
class HtsVcfWriter {
 public:
  HtsVcfWriter(std::string const& outfile, std::vector<std::string> const& target_name) : outfile_(outfile), target_name_(target_name) {
    fp_ = hts_open(outfile.c_str(), (outfile == "-") ? "w" : "wb");   // src/modvcf.h:355-357
    hdr_ = bcf_hdr_init("w");
    rec_ = bcf_init();
  }
  ~HtsVcfWriter() { close(); }
  bool ok() const { return fp_ != nullptr && !failed_; }
  void header(std::string const& line) { bcf_hdr_append(hdr_, line.c_str()); }
  void sample(std::string const& s) { bcf_hdr_add_sample(hdr_, s.c_str()); ++nsamples_; }
  void headerWritten() {
    bcf_hdr_add_sample(hdr_, NULL);
    if (bcf_hdr_write(fp_, hdr_) != 0) std::cerr << "Error: Failed to write BCF header!" << std::endl;
  }
  void begin(int32_t rid, int64_t pos) { rec_->rid = bcf_hdr_name2id(hdr_, target_name_[rid].c_str()); rec_->pos = pos; }
  void str(const char* kind, const char* key, std::string const& v) {
    if (!kind[0]) {
      if (!std::strcmp(key, "ID")) bcf_update_id(hdr_, rec_, v.c_str());
      else if (!std::strcmp(key, "ALLELES")) bcf_update_alleles_str(hdr_, rec_, v.c_str());
    } else if (kind[0] == 'I') {
      if (!std::strcmp(key, "PRECISE") || !std::strcmp(key, "IMPRECISE")) bcf_update_info_flag(hdr_, rec_, key, NULL, 1);
      else bcf_update_info_string(hdr_, rec_, key, v.c_str());
    } else {   // FORMAT string (FT): one value per sample, comma-separated in the description
      std::vector<std::string> parts;
      std::string cur;
      for (char ch : v) { if (ch == ',') { parts.push_back(cur); cur.clear(); } else cur.push_back(ch); }
      parts.push_back(cur);
      std::vector<const char*> p;
      for (auto const& s : parts) p.push_back(s.c_str());
      bcf_update_format_string(hdr_, rec_, key, p.data(), (int) p.size());
    }
  }
  void ints(const char* kind, const char* key, const int32_t* v, int n) {
    if (!kind[0]) {   // FILTER: 0 = PASS, 1 = LowQual
      int32_t tmpi = bcf_hdr_id2int(hdr_, BCF_DT_ID, v[0] ? "LowQual" : "PASS");
      bcf_update_filter(hdr_, rec_, &tmpi, 1);
    } else if (kind[0] == 'I') bcf_update_info_int32(hdr_, rec_, key, v, n);
    else if (!std::strcmp(key, "GT")) bcf_update_genotypes(hdr_, rec_, v, n);
    else bcf_update_format_int32(hdr_, rec_, key, v, n);
  }
  void flt(const char*, const char* key, float v) { bcf_update_info_float(hdr_, rec_, key, &v, 1); }
  void write(int32_t, int64_t, float qual) {
    rec_->qual = qual;
    if (bcf_write1(fp_, hdr_, rec_) != 0) { std::cerr << "Error: Failed to write BCF record!" << std::endl; failed_ = true; }
    bcf_clear1(rec_);
  }
  void close() {
    if (!fp_) return;
    bcf_destroy1(rec_);
    bcf_hdr_destroy(hdr_);
    hts_close(fp_);
    fp_ = nullptr;
    if (outfile_ != "-") bcf_index_build(outfile_.c_str(), 14);   // src/modvcf.h:778
  }
 private:
  std::string outfile_;
  std::vector<std::string> target_name_;
  htsFile* fp_ = nullptr;
  bcf_hdr_t* hdr_ = nullptr;
  bcf1_t* rec_ = nullptr;
  int nsamples_ = 0;
  bool failed_ = false;
};

inline std::string todayIso() {   // boost::gregorian::to_iso_string(today) (src/modvcf.h:360-364)
  std::time_t t = std::time(nullptr);
  std::tm tmv;
  localtime_r(&t, &tmv);
  char b[32];
  std::snprintf(b, sizeof(b), "%04d%02d%02d", tmv.tm_year + 1900, tmv.tm_mon + 1, tmv.tm_mday);
  return b;
}

}  // namespace io
}  // namespace dellyb200
