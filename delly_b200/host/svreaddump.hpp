// svreaddump.hpp — the SV-read dump of `delly sr|lr -d`: the reads that support each called SV, as the genotyping passes classify them.
// The stage mirrors record one SvReadEvent (host/genotype.hpp) per ALT-supporting read where they append its quality to the SV's list; the
// lines are rendered here in the reference's order.
//   src/coverage.h:336-341, :517-537, :652-662   short reads: SR lines (junction reads), PE lines (ALT-spanning pairs)
//   src/genotype.h:127-133, :325-331             long reads: SR lines
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "genotype.hpp"

namespace dellyb200 {

struct SvReadDump {
  struct File { std::vector<SvReadEvent> sr, pe; };   // each in record order; long reads have SR events only
  std::vector<File> file;                             // one per input file, in command-line order
};

// _addID(svt) followed by the id zero-padded to 8 digits
inline std::string svReadId(int32_t svt, uint32_t id) {
  std::string n = std::to_string(id);
  if (n.size() < 8) n.insert(n.begin(), 8 - n.size(), '0');
  return _addID(svt) + n;
}

// Hands the rendered text to put(const char*, std::size_t) in blocks of about 1 MiB.
template <typename Put> class DumpText {
 public:
  explicit DumpText(Put& put) : put_(put) {}
  ~DumpText() { flush(); }
  DumpText& operator<<(std::string const& s) { buf_ += s; if (buf_.size() >= (1u << 20)) flush(); return *this; }
  DumpText& operator<<(const char* s) { return *this << std::string(s); }
  template <typename T> DumpText& operator<<(T v) { return *this << std::to_string(v); }
  void flush() { if (!buf_.empty()) put_(buf_.data(), buf_.size()); buf_.clear(); }
 private:
  Put& put_;
  std::string buf_;
};

// Short reads: file by file; within a file, record by record (the lists are in contig, then BAM order); within a record its SR lines, then
// its PE lines. The reference reads target_name[mtid] for an unpaired read (mtid = -1) as well; that is undefined, "*" is written here.
template <typename Put>
void writeSrReadDump(Put put, SvReadDump const& d, std::vector<std::string> const& paths, std::vector<std::vector<SrRecord> const*> const& recs,
                     std::vector<std::vector<std::string> > const& names, std::vector<std::string> const& target_name) {
  DumpText<Put> out(put);
  out << "#svid\tbam\tqname\tchr\tpos\tmatechr\tmatepos\tmapq\ttype\n";
  for (std::size_t f = 0; f < d.file.size(); ++f) {
    std::vector<SvReadEvent> const& sr = d.file[f].sr;
    std::vector<SvReadEvent> const& pe = d.file[f].pe;
    std::size_t i = 0, j = 0;
    while (i < sr.size() || j < pe.size()) {
      const bool isSr = (j == pe.size()) || (i < sr.size() && sr[i].rec <= pe[j].rec);
      SvReadEvent const& e = isSr ? sr[i++] : pe[j++];
      SrRecord const& r = (*recs[f])[e.rec];
      out << svReadId(e.svt, e.svid) << "\t" << paths[f] << "\t" << names[f][e.rec] << "\t" << target_name[r.tid] << "\t" << r.pos << "\t"
          << (r.mtid >= 0 ? target_name[r.mtid] : std::string("*")) << "\t" << r.mpos << "\t" << (int32_t) r.mapq << (isSr ? "\tSR\n" : "\tPE\n");
    }
  }
}

// Long reads: contig by contig; within a contig, file by file; within a file, record by record, and SV id ascending within a record.
template <typename Put>
void writeLrReadDump(Put put, SvReadDump const& d, std::vector<std::string> const& paths, std::vector<std::vector<LrRecord> const*> const& recs,
                     std::vector<std::vector<std::string> > const& names, std::vector<std::string> const& target_name) {
  DumpText<Put> out(put);
  out << "#svid\tbam\tqname\tchr\tpos\tmapq\ttype\n";
  std::vector<std::size_t> next(d.file.size(), 0);
  for (int32_t refIndex = 0; refIndex < (int32_t) target_name.size(); ++refIndex)
    for (std::size_t f = 0; f < d.file.size(); ++f) {
      std::vector<SvReadEvent> const& sr = d.file[f].sr;
      for (std::size_t& i = next[f]; i < sr.size() && (*recs[f])[sr[i].rec].tid == refIndex; ++i) {
        LrRecord const& r = (*recs[f])[sr[i].rec];
        out << svReadId(sr[i].svt, sr[i].svid) << "\t" << paths[f] << "\t" << names[f][sr[i].rec] << "\t" << target_name[r.tid] << "\t" << r.pos << "\t"
            << (int32_t) r.mapq << "\tSR\n";
      }
    }
}

}  // namespace dellyb200
