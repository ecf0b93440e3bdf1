// delly_b200 — the drop-in binding: the `delly sr` / `delly lr` command-line surface (BAM + FASTA in, BCF out) over the batched
// H100 path. It is what a maintainer gets by replacing the per-item alignment calls of the reference's drivers with the batched
// C ABI (include/dgpu.h): htslib reads the alignments into record lists (bindings/hts_io.hpp), the stage mirrors of delly_b200/host
// run the reference's stage sequence with every alignment batch on the device, htslib writes the BCF.
//   src/delly.h:199-400  `delly sr` options and checks -> dellyRun (:86-196)
//   src/tegua.h:209-440  `delly lr` options and checks -> runTegua (:78-207)
// Parity: tests/test_bcf_parity.py compares the BCF written here byte for byte (uncompressed stream, ##fileDate aside) with the BCF the
// reference's own drivers write (oracle/_ref/delly_ref = src/delly.h + src/tegua.h compiled verbatim against the same htslib).
// No CPU fallback: without an sm_90 device dgpu_ctx_create fails and so does this program.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <cstring>
#include <iostream>
#include <string>
#include <sys/resource.h>
#include <sys/stat.h>
#include <unistd.h>
#include <thread>
#include <vector>
#include <zlib.h>

#include "hts_io.hpp"
#include "../delly_b200/host/gather.hpp"
#include "../include/dgpu.h"

using namespace dellyb200;

namespace {

struct Options {
  bool lr = false;
  std::string svtype = "ALL", mode = "ont";
  std::string genome, exclude, outfile = "-", vcffile, dumpfile, meifile;
  std::vector<std::string> files;
  bool hasExclude = false, hasVcf = false, hasOutfile = false, help = false;
  int device = 0, ioThreads = 16;
  int rank = 0, nranks = 1;          // one process per GPU: --rank r --nranks N --comm-file path (rank 0 publishes the NCCL id there)
  std::string commFile, timingFile;  // --timing file: stage wall-clock times as one JSON object
  std::string shardBy = "svs";       // --shard-by svs|contig: what the ranks divide
  bool readShareOnly = false;        // --read-share-only: read this rank's share of the alignments, write --timing, stop (measuring a share alone)
  std::vector<int> devices;          // --devices LIST: rank r runs on devices[r]; every rank is a thread of this process (no NCCL, no comm file)
  float indelExtension = 0.5f;
  MethylConfig methyl;
  AnnoConfig anno;
  Config c;
};

bool fileOk(std::string const& p) { struct stat st; return ::stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode) && st.st_size > 0; }

// src/util.h:370-395 (_svTypesToCompute): DEL -> 2, INS -> 4, DUP -> 3, INV -> 0,1, BND -> 5..8, ALL -> no restriction
bool svTypesToCompute(Config& c, std::string const& svtype) {
  c.svtset.clear();
  std::size_t b = 0;
  bool all = false;
  while (b <= svtype.size()) {
    std::size_t e = svtype.find(',', b);
    if (e == std::string::npos) e = svtype.size();
    const std::string t = svtype.substr(b, e - b);
    if (t == "ALL") all = true;
    else if (t == "DEL") c.svtset.insert(2);
    else if (t == "INS") c.svtset.insert(4);
    else if (t == "DUP") c.svtset.insert(3);
    else if (t == "INV") { c.svtset.insert(0); c.svtset.insert(1); }
    else if (t == "BND") { c.svtset.insert(5); c.svtset.insert(6); c.svtset.insert(7); c.svtset.insert(8); }
    else return false;
    b = e + 1;
  }
  if (all) c.svtset.clear();
  return true;
}

void usage(Options const& o) {
  std::cerr << "\nUsage: delly_b200 " << (o.lr ? "lr" : "sr") << " [OPTIONS] -g <ref.fa> <sample1.sort.bam> <sample2.sort.bam> ...\n"
            << "  options follow `delly " << (o.lr ? "lr" : "sr") << "` (same letters and defaults), including -d <reads.gz> (gzipped list of the reads"
            << " that support each SV); extra: --device N, --io-threads N" << (o.lr ? ", --mei <templates.fa>" : "") << "\n"
            << "  several GPUs, one process each: --rank r --nranks N --comm-file <path> [--shard-by svs|contig] [--timing <file>]\n"
            << "  several GPUs, one process: --devices LIST (e.g. 0-7 or 0,1,2,3; rank r runs on entry r, an index may repeat) [--shard-by svs|contig]\n"
            << "    [--timing <file>]; not with --device, --rank, --nranks or --comm-file. The ranks split --io-threads and the host-stage threads"
               " (DGPU_HOST_THREADS, default min(cores, 16)) evenly, at least one each; --shard-by svs reads the BAM once, with all --io-threads\n"
            << "  --read-share-only: read this rank's share (--shard-by contig), write --timing and stop: no device, no exchange\n";
}

// --devices LIST: comma-separated device indices and ranges a-b (a <= b); entry r is the device of rank r. At most 1024 ranks.
bool parseDeviceList(std::string const& s, std::vector<int>& out) {
  out.clear();
  std::size_t b = 0;
  auto number = [](std::string const& t, int& v) {
    if (t.empty() || t.size() > 4 || t.find_first_not_of("0123456789") != std::string::npos) return false;
    v = std::stoi(t);
    return true;
  };
  while (b <= s.size()) {
    std::size_t e = s.find(',', b);
    if (e == std::string::npos) e = s.size();
    const std::string t = s.substr(b, e - b);
    const std::size_t dash = t.find('-');
    int lo = 0, hi = 0;
    if (dash == std::string::npos) { if (!number(t, lo)) return false; hi = lo; }
    else if (!number(t.substr(0, dash), lo) || !number(t.substr(dash + 1), hi) || hi < lo) return false;
    for (int d = lo; d <= hi; ++d) { if (out.size() >= 1024) return false; out.push_back(d); }
    b = e + 1;
  }
  return !out.empty();
}

// `delly sr` (src/delly.h:207-246) and `delly lr` (src/tegua.h:215-275) share most letters; the long names are the reference's.
bool parse(int argc, char** argv, Options& o) {
  Config& c = o.c;
  if (o.lr) { c = Config::longRead(); c.minCliqueSize = 3; c.minRefSep = 30; c.maxReadPerSV = 15; }
  else c = Config::shortRead();
  c.maxThreads = 4;
  o.methyl.methylProb = 128; o.methyl.methylWindow = 1000; o.methyl.minCpgDepth = 5;
  auto need = [&](int& i) -> const char* { if (i + 1 >= argc) { std::cerr << "missing value for " << argv[i] << std::endl; std::exit(2); } return argv[++i]; };
  std::vector<std::string> processRank;   // the options of the one-process-per-GPU mode that were given (--devices excludes them)
  bool hasDevices = false;
  std::string deviceList;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    std::string v;
    bool inl = false;
    if (a.size() > 2 && a[0] == '-' && a[1] == '-') { const std::size_t e = a.find('='); if (e != std::string::npos) { v = a.substr(e + 1); a = a.substr(0, e); inl = true; } }
    else if (a.size() > 2 && a[0] == '-' && a[1] != '-') { v = a.substr(2); a = a.substr(0, 2); inl = true; }
    auto val = [&]() -> std::string { return inl ? v : std::string(need(i)); };
    auto is = [&](const char* s, const char* l) { return a == s || a == l; };
    if (a.empty() || a[0] != '-' || a == "-") { o.files.push_back(a); continue; }
    if (is("-?", "--help")) o.help = true;
    else if (is("-t", "--svtype")) o.svtype = val();
    else if (is("-g", "--genome")) o.genome = val();
    else if (is("-x", "--exclude")) { o.exclude = val(); o.hasExclude = true; }
    else if (is("-o", "--outfile")) { o.outfile = val(); o.hasOutfile = true; }
    else if (is("-q", "--map-qual")) c.minMapQual = (uint16_t) std::stoi(val());
    else if (is("-c", "--minclip")) c.minClip = (uint32_t) std::stoul(val());
    else if (is("-z", "--min-clique-size")) c.minCliqueSize = (uint16_t) std::stoi(val());
    else if (is("-m", "--minrefsep")) c.minRefSep = (uint32_t) std::stoul(val());
    else if (is("-n", "--maxreadsep")) c.maxReadSep = (uint32_t) std::stoul(val());
    else if (is("-p", "--max-reads")) c.maxReadPerSV = (uint32_t) std::stoul(val());
    else if (is("-v", "--vcffile")) { o.vcffile = val(); o.hasVcf = true; }
    else if (is("-u", "--geno-qual")) c.minGenoQual = (uint16_t) std::stoi(val());
    else if (is("-d", "--dump")) o.dumpfile = val();
    else if (is("-w", "--cons-window")) c.minConsWindow = std::stoi(val());
    else if (a == "--device") { o.device = std::stoi(val()); processRank.push_back(a); }
    else if (a == "--devices") { deviceList = val(); hasDevices = true; }
    else if (a == "--io-threads") o.ioThreads = std::stoi(val());
    else if (a == "--rank") { o.rank = std::stoi(val()); processRank.push_back(a); }
    else if (a == "--nranks") { o.nranks = std::stoi(val()); processRank.push_back(a); }
    else if (a == "--comm-file") { o.commFile = val(); processRank.push_back(a); }
    else if (a == "--timing") o.timingFile = val();
    else if (a == "--shard-by") o.shardBy = val();
    else if (a == "--read-share-only") o.readShareOnly = true;
    else if (!o.lr && is("-h", "--threads")) c.maxThreads = (uint32_t) std::stoul(val());
    else if (!o.lr && is("-r", "--qual-tra")) c.minTraQual = (uint16_t) std::stoi(val());
    else if (!o.lr && is("-s", "--mad-cutoff")) c.madCutoff = (uint16_t) std::stoi(val());
    else if (!o.lr && is("-a", "--max-geno-count")) c.maxGenoReadCount = (uint32_t) std::stoul(val());
    else if (!o.lr && is("-j", "--pruning")) c.graphPruning = (uint32_t) std::stoul(val());
    else if (o.lr && is("-y", "--technology")) o.mode = val();
    else if (o.lr && is("-f", "--flank-size")) c.minimumFlankSize = std::stoi(val());
    else if (o.lr && is("-a", "--flank-quality")) c.flankQuality = std::stof(val());
    else if (o.lr && is("-i", "--indel-size")) c.indelsize = std::stoi(val());
    else if (o.lr && is("-k", "--mei-minfrac")) o.anno.meiMinFrac = std::stof(val());
    else if (o.lr && is("-r", "--tr-minfrac")) o.anno.trMinFrac = std::stof(val());
    else if (o.lr && is("-j", "--methyl-window")) o.methyl.methylWindow = std::stoi(val());
    else if (o.lr && is("-e", "--methyl-prob")) o.methyl.methylProb = (uint16_t) std::stoi(val());
    else if (o.lr && a == "--min-cpg-depth") o.methyl.minCpgDepth = (uint32_t) std::stoul(val());
    else if (o.lr && is("-b", "--max-geno-count")) c.maxGenoReadCount = (uint32_t) std::stoul(val());
    else if (o.lr && a == "--pruning") c.graphPruning = (uint32_t) std::stoul(val());
    else if (o.lr && a == "--extension") o.indelExtension = std::stof(val());
    else if (o.lr && a == "--read-cap") c.genoCap = std::stoi(val());
    else if (o.lr && a == "--mei") o.meifile = val();
    else if (o.lr && is("-l", "--alt-align")) { std::cerr << "alternate alignments (-l) are outside the accelerated path (SURVEY section 2)" << std::endl; return false; }
    else { std::cerr << "unrecognised option '" << argv[i] << "'" << std::endl; return false; }
  }
  if (hasDevices) {
    if (!processRank.empty()) {
      std::cerr << "--devices cannot be combined with " << processRank[0] << ": --devices runs every rank in this process, --device / --rank / --nranks /"
                   " --comm-file run one rank per process" << std::endl;
      return false;
    }
    if (!parseDeviceList(deviceList, o.devices)) {
      std::cerr << "--devices takes a comma-separated list of device indices and ranges a-b with a <= b (e.g. 0,1,2,3 or 0-7), not '" << deviceList << "'" << std::endl;
      return false;
    }
    if (!o.dumpfile.empty() && o.devices.size() > 1) {
      std::cerr << "the SV-read dump (-d) needs a single rank: over --devices with several entries every rank genotypes a part of the SV list, and the"
                   " order of the dump lines depends on the whole list" << std::endl;
      return false;
    }
    if (o.devices.size() == 1) { o.device = o.devices[0]; o.devices.clear(); }   // one rank: the single-process run on that device
    else o.nranks = (int) o.devices.size();
  }
  if (o.shardBy != "svs" && o.shardBy != "contig") { std::cerr << "--shard-by takes svs or contig" << std::endl; return false; }
  if (o.readShareOnly && o.shardBy != "contig") { std::cerr << "--read-share-only measures a share of --shard-by contig" << std::endl; return false; }
  if (!o.dumpfile.empty() && o.shardBy == "contig") {
    std::cerr << "the SV-read dump (-d) needs --shard-by svs: the order of the dump lines depends on the whole SV list and the whole record list" << std::endl;
    return false;
  }
  if (!o.dumpfile.empty() && o.nranks > 1) {
    std::cerr << "the SV-read dump (-d) needs a single process: over --nranks > 1 every rank genotypes a part of the SV list, and the order of"
                 " the dump lines depends on the whole list" << std::endl;
    return false;
  }
  return true;
}

// the template sequences of the reference's annotation step (class MEI, src/svanno.h:30-39) are data of the reference; the build
// extracts them into a FASTA next to the binary (tools/extract_mei.py), `--mei` names another file. Records: >alu >line1 >sva >numt >soloLTR >hervk >polyA
bool loadMei(std::string const& path, MeiTemplates& mei) {
  std::ifstream f(path.c_str());
  if (!f.is_open()) return false;
  std::string line, name;
  int found = 0;
  while (std::getline(f, line)) {
    if (line.empty()) continue;
    if (line[0] == '>') { name = line.substr(1); continue; }
    int k = (name == "alu") ? 1 : (name == "line1") ? 2 : (name == "sva") ? 3 : (name == "numt") ? 4 : (name == "soloLTR") ? 5 : (name == "hervk") ? 6 : (name == "polyA") ? 0 : -1;
    if (k < 0) continue;
    if (k == 0) mei.polyA += line; else mei.seq[k] += line;
    ++found;
  }
  return found >= 7;
}

std::string exeDir(const char* argv0) {
  char buf[4096];
  const ssize_t n = ::readlink("/proc/self/exe", buf, sizeof(buf) - 1);
  std::string p = (n > 0) ? std::string(buf, (std::size_t) n) : std::string(argv0);
  const std::size_t k = p.rfind('/');
  return (k == std::string::npos) ? "." : p.substr(0, k);
}

// The device side of a rank starts while the host reads its inputs: creating the CUDA context (and, with one process per rank, the NCCL
// communicator plus one tiny warm-up exchange that sets up the NVLink connections) costs 0.5 - 2 s; a background thread pays it during the BAM scan.
// With `ex` (--devices) the rank is a thread of a several-rank process and exchanges through it: no communicator.
class DeviceSession {
 public:
  DeviceSession(Options const& o, SimExchange* ex = nullptr) : o_(o), ex_(ex) { th_ = std::thread([this] { start(); }); }
  ~DeviceSession() {
    if (th_.joinable()) th_.join();
    if (comm_) dgpu_comm_destroy(commCtx_, comm_);
    if (commCtx_) dgpu_ctx_destroy(commCtx_);
    if (ctx_) dgpu_ctx_destroy(ctx_);
  }
  // the compute context (needed by the first device stage); the communicator keeps starting in the background until the first exchange needs it
  bool wait() { waitFor(1); return ctx_ != nullptr; }
  bool waitComm() { waitFor(2); return commOk_; }
  dgpu_ctx* ctx() { return ctx_; }
  Shard shard() {
    Shard sh;
    if (o_.nranks > 1 && ex_) {
      sh.rank = o_.rank; sh.nranks = o_.nranks;
      sh.gather = ex_->of(o_.rank);
#ifdef DELLY_B200_FAIL_HOOK
      // test builds only (tests/test_devices.py): DELLY_B200_FAIL_RANK=r makes rank r's first exchange fail on the host, so that the release
      // of the other ranks can be checked without a device error
      const char* failRank = getenv("DELLY_B200_FAIL_RANK");
      if (failRank && std::atoi(failRank) == o_.rank)
        sh.gather = [](std::string const&, std::vector<std::string>&) { std::cerr << "delly_b200: exchange failed (DELLY_B200_FAIL_RANK)" << std::endl; return (int) DGPU_ERR_NCCL; };
#endif
    } else if (o_.nranks > 1) {
      sh.rank = o_.rank; sh.nranks = o_.nranks;
      sh.gather = [this](std::string const& local, std::vector<std::string>& parts) -> int {
        if (!waitComm()) return DGPU_ERR_NCCL;
        return gatherStrings(commCtx_, comm_, local, parts);
      };
    }
    return sh;
  }
  static int gatherStrings(dgpu_ctx* ctx, void* comm, std::string const& local, std::vector<std::string>& parts) {
    void* all = nullptr; uint64_t* counts = nullptr; int n = 0;
    const int grc = dgpu_gather_records(ctx, comm, local.data(), (uint64_t) local.size(), &all, &counts, &n);
    if (grc) return grc;
    parts.clear();
    const char* p = (const char*) all;
    for (int r = 0; r < n; ++r) { parts.emplace_back(p, (std::size_t) counts[r]); p += counts[r]; }
    dgpu_free_host(all); dgpu_free_host(counts);
    return DGPU_OK;
  }
 private:
  void start();
  void reach(int stage) { { std::lock_guard<std::mutex> g(m_); stage_ = stage; } cv_.notify_all(); }
  void waitFor(int stage) { std::unique_lock<std::mutex> g(m_); cv_.wait(g, [&] { return stage_ >= stage; }); }
  const Options o_;   // a copy: the rank's options, whatever the caller does with its own afterwards
  SimExchange* ex_;
  std::thread th_;
  std::mutex m_;
  std::condition_variable cv_;
  int stage_ = 0;              // 1: compute context ready (or failed), 2: communicator ready (or failed / not needed)
  dgpu_ctx* ctx_ = nullptr;
  dgpu_ctx* commCtx_ = nullptr;   // the exchange has its own context (stream, staging buffers): it starts while the compute context already works
  void* comm_ = nullptr;
  bool commOk_ = false;
};

struct Inputs {
  std::vector<io::AlignmentFile> files;
  std::vector<std::string> sampleName;
  std::vector<uint32_t> target_len;
  std::vector<std::string> target_name;
  io::TRegionsGenome validRegions, wholeContigs;
  io::Genome genome;
};

bool openInputs(Options& o, Inputs& in) {
  if (!fileOk(o.genome)) { std::cerr << "Reference file is missing: " << o.genome << std::endl; return false; }
  {
    faidx_t* fai = fai_load(o.genome.c_str());
    if (!fai) { if (fai_build(o.genome.c_str()) == -1) { std::cerr << "Fail to open genome fai index for " << o.genome << std::endl; return false; } }
    else fai_destroy(fai);
  }
  in.files.resize(o.files.size());
  in.sampleName.resize(o.files.size());
  o.c.nchr = 0;
  for (std::size_t f = 0; f < o.files.size(); ++f) {
    if (!fileOk(o.files[f])) { std::cerr << "Alignment file is missing: " << o.files[f] << std::endl; return false; }
    if (!in.files[f].open(o.files[f], o.genome, o.ioThreads)) return false;
    if (!o.c.nchr) o.c.nchr = in.files[f].hdr->n_targets;
    else if (o.c.nchr != in.files[f].hdr->n_targets) { std::cerr << "BAM files have different number of chromosomes!" << std::endl; return false; }
    std::string sampleName = "unknown";
    io::getSMTag(std::string(in.files[f].hdr->text ? in.files[f].hdr->text : sam_hdr_str(in.files[f].hdr)), io::fileStem(o.files[f]), sampleName);
    in.sampleName[f] = sampleName;
  }
  io::checkSampleNames(in.sampleName);
  if (o.hasExclude && !fileOk(o.exclude)) { std::cerr << "Exclude file is missing: " << o.exclude << std::endl; return false; }
  if (o.hasVcf && !fileOk(o.vcffile)) { std::cerr << "Input VCF/BCF file is missing: " << o.vcffile << std::endl; return false; }
  bam_hdr_t* hdr = in.files[0].hdr;
  for (int32_t i = 0; i < hdr->n_targets; ++i) { in.target_len.push_back(hdr->target_len[i]); in.target_name.push_back(hdr->target_name[i]); }
  if (!io::parseExcludeIntervals(o.hasExclude, o.exclude, hdr, in.validRegions)) { std::cerr << "Delly couldn't parse exclude intervals!" << std::endl; return false; }
  in.wholeContigs.assign(hdr->n_targets, std::vector<io::Interval>());
  for (int32_t i = 0; i < hdr->n_targets; ++i) in.wholeContigs[i].push_back(io::Interval{0u, hdr->target_len[i]});
  return in.genome.load(o.genome, hdr, o.lr);
}


// The SV-read dump (-d) as one gzip stream; render(put) hands it the text.
template <typename TRender> bool writeDump(std::string const& path, TRender render) {
  gzFile gz = gzopen(path.c_str(), "wb");
  if (!gz) { std::cerr << "cannot open the SV-read dump file " << path << std::endl; return false; }
  bool ok = true;
  render([&](const char* p, std::size_t n) { if (ok && gzwrite(gz, p, (unsigned) n) != (int) n) ok = false; });
  if (gzclose(gz) != Z_OK) ok = false;
  if (!ok) std::cerr << "cannot write the SV-read dump file " << path << std::endl;
  return ok;
}

// what this rank holds and sends (--timing): its records (both lists with -x), its peak resident memory, and the bytes it contributed to the
// exchanges of each stage (the stage clock's lap names)
struct ShareStats {
  std::size_t records = 0;
  std::map<std::size_t, uint64_t> sentAtLap;   // bytes handed to the gather while the stage clock had k laps: the stage of lap k sent them
};

void writeTiming(Options const& o, StageClock const& clock, std::size_t nsv, ShareStats const* share = nullptr) {
  if (o.timingFile.empty()) return;
  std::ofstream f((o.timingFile + (o.nranks > 1 ? "." + std::to_string(o.rank) : std::string())).c_str());
  double total = 0;
  f << "{\"rank\": " << o.rank << ", \"nranks\": " << o.nranks << ", \"svs\": " << nsv << ", \"stages_ms\": {";
  for (std::size_t i = 0; i < clock.ms.size(); ++i) { f << (i ? ", " : "") << "\"" << clock.ms[i].first << "\": " << clock.ms[i].second; total += clock.ms[i].second; }
  f << "}, \"total_ms\": " << total;
  if (share) {
    struct rusage ru;
    getrusage(RUSAGE_SELF, &ru);
    f << ", \"records\": " << share->records << ", \"peak_rss_kb\": " << ru.ru_maxrss << ", \"sent_bytes\": {";
    bool first = true;
    for (auto const& kv : share->sentAtLap) {
      f << (first ? "" : ", ") << "\"" << (kv.first < clock.ms.size() ? clock.ms[kv.first].first : std::string("end")) << "\": " << kv.second;
      first = false;
    }
    f << "}";
  }
  f << "}" << std::endl;
}

// One process per GPU: rank 0 creates the NCCL id and publishes it in --comm-file (written under a temporary name, then renamed); the other
// ranks wait for the file. The communicator lives as long as the process.
bool initComm(Options const& o, dgpu_ctx* ctx, void** comm) {
  uint8_t id[128];
  if (o.commFile.empty()) { std::cerr << "--nranks > 1 needs --comm-file" << std::endl; return false; }
  if (o.rank == 0) {
    if (dgpu_comm_unique_id(id) != DGPU_OK) { std::cerr << "NCCL is not available (libnccl.so.2)" << std::endl; return false; }
    const std::string tmp = o.commFile + ".tmp";
    { std::ofstream f(tmp.c_str(), std::ios::binary); f.write((const char*) id, 128); }
    if (std::rename(tmp.c_str(), o.commFile.c_str()) != 0) { std::cerr << "cannot publish " << o.commFile << std::endl; return false; }
  } else {
    for (int tries = 0; tries < 6000; ++tries) {
      std::ifstream f(o.commFile.c_str(), std::ios::binary);
      if (f.good()) { f.read((char*) id, 128); if (f.gcount() == 128) break; }
      if (tries == 5999) { std::cerr << "timed out waiting for " << o.commFile << std::endl; return false; }
      usleep(10000);
    }
  }
  const int rc = dgpu_comm_init(ctx, o.nranks, o.rank, id, comm);
  if (rc != DGPU_OK) { std::cerr << "dgpu_comm_init failed (" << rc << "): " << dgpu_last_error(ctx) << std::endl; return false; }
  return true;
}

void DeviceSession::start() {
  if (o_.readShareOnly) { reach(2); return; }   // nothing on the device
  const int rc = dgpu_ctx_create(o_.device, &ctx_);
  if (rc != DGPU_OK) { std::cerr << "delly_b200: no usable sm_90 device (dgpu_ctx_create = " << rc << "); there is no CPU fallback on this path" << std::endl; ctx_ = nullptr; reach(2); return; }
  reach(1);
  if (o_.nranks > 1 && !ex_) {
    std::vector<std::string> parts;
    if (dgpu_ctx_create(o_.device, &commCtx_) != DGPU_OK) { commCtx_ = nullptr; std::cerr << "delly_b200: cannot create the exchange context" << std::endl; }
    else if (!initComm(o_, commCtx_, &comm_)) { }
    else if (gatherStrings(commCtx_, comm_, std::string("warm-up"), parts) != DGPU_OK || (int) parts.size() != o_.nranks) std::cerr << "NCCL warm-up exchange failed: " << dgpu_last_error(commCtx_) << std::endl;
    else commOk_ = true;
  } else commOk_ = true;
  reach(2);
}

// --shard-by contig: the contig ranges of the ranks, balanced by the mapped reads of the BAM indexes summed over the files; by the contig
// lengths when an index has no read counts (one unit for every contig). Every rank computes the same cut from the same files.
std::vector<std::size_t> contigCut(Options const& o, Inputs const& in) {
  std::vector<uint64_t> w(in.target_len.size(), 0);
  bool counted = true;
  for (auto const& f : in.files)
    for (int32_t t = 0; t < (int32_t) w.size() && counted; ++t) {
      uint64_t mapped = 0, unmapped = 0;
      if (hts_idx_get_stat(f.idx, t, &mapped, &unmapped) != 0) counted = false;
      else w[t] += mapped;
    }
  if (!counted) w.assign(in.target_len.begin(), in.target_len.end());
  return partitionContigs(w, o.nranks);
}

// The record lists of an sr run, as the reference's iterators return them: the valid regions' (scan, clustering, assembly, library estimate,
// src/shortpe.h:349, src/util.h:810) and, with an exclude file, the whole contigs' for the genotyping pass (src/coverage.h) — a second list.
// names: the query names of the genotyped records (-d).
struct SrReads {
  std::vector<std::vector<SrRecord> > recs, recsWhole;
  std::vector<std::vector<std::string> > names;
};

bool readSr(Options const& o, std::vector<io::AlignmentFile>& files, io::TRegionsGenome const& valid, io::TRegionsGenome const& whole, SrReads& r) {
  const std::size_t F = files.size();
  const bool dump = !o.dumpfile.empty();
  r.recs.assign(F, std::vector<SrRecord>());
  r.recsWhole.assign(o.hasExclude ? F : 0, std::vector<SrRecord>());
  r.names.assign(dump ? F : 0, std::vector<std::string>());
  for (std::size_t f = 0; f < F; ++f)
    if (!files[f].readRegionsParallel(o.genome, valid, r.recs[f], io::toSrRecord, o.ioThreads, nullptr, nullptr, 0, (dump && !o.hasExclude) ? &r.names[f] : nullptr)) {
      std::cerr << "cannot read " << o.files[f] << std::endl;
      return false;
    }
  for (std::size_t f = 0; f < F && o.hasExclude; ++f)
    if (!files[f].readRegionsParallel(o.genome, whole, r.recsWhole[f], io::toSrRecord, o.ioThreads, nullptr, nullptr, 0, dump ? &r.names[f] : nullptr)) {
      std::cerr << "cannot read " << o.files[f] << std::endl;
      return false;
    }
  return true;
}

// The long reads of an lr run with their read ids: the valid regions' and, with an exclude file, the whole contigs' (the genotyping pass).
struct LrReads {
  std::vector<std::vector<LrRecord> > recs, recsWhole;
  std::vector<std::vector<std::size_t> > ids, idsWhole;
  std::vector<std::vector<std::string> > names;
};

bool readLr(Options const& o, std::vector<io::AlignmentFile>& files, io::TRegionsGenome const& valid, io::TRegionsGenome const& whole, LrReads& r) {
  const std::size_t F = files.size();
  const bool dump = !o.dumpfile.empty();
  r.recs.assign(F, std::vector<LrRecord>()); r.ids.assign(F, std::vector<std::size_t>());
  r.recsWhole.assign(o.hasExclude ? F : 0, std::vector<LrRecord>()); r.idsWhole.assign(o.hasExclude ? F : 0, std::vector<std::size_t>());
  r.names.assign(dump ? F : 0, std::vector<std::string>());
  for (std::size_t f = 0; f < F; ++f)
    if (!files[f].readRegionsParallel(o.genome, valid, r.recs[f], io::toLrRecord, o.ioThreads, &r.ids[f], io::hashLr, 0, (dump && !o.hasExclude) ? &r.names[f] : nullptr)) {
      std::cerr << "cannot read " << o.files[f] << std::endl;
      return false;
    }
  for (std::size_t f = 0; f < F && o.hasExclude; ++f)
    if (!files[f].readRegionsParallel(o.genome, whole, r.recsWhole[f], io::toLrRecord, o.ioThreads, &r.idsWhole[f], io::hashLr, 0, dump ? &r.names[f] : nullptr)) {
      std::cerr << "cannot read " << o.files[f] << std::endl;
      return false;
    }
  return true;
}

// What the ranks of a --devices process share, read-only once they start: the inputs opened once (headers, region lists, the genome loaded
// once) and, with --shard-by svs, where every rank needs every record, the record lists read once. clock: the stages the process ran for
// all ranks before they started (every rank's --timing begins with them).
struct SharedInputs {
  Inputs in;
  bool haveReads = false;
  SrReads sr;
  LrReads lr;
  StageClock clock;
  std::atomic<bool> outputOpened{false};   // rank 0 has created the BCF (removed again when another rank fails)
};

// The inputs of one rank: opened by the rank itself (one process per rank) or shared (--devices). A rank of a --devices process that reads
// its own share (--shard-by contig) does so through its own file handles, beside the other ranks' reads.
struct RankInputs {
  Inputs own;
  Inputs& in;
  std::vector<io::AlignmentFile> ownFiles;
  io::TRegionsGenome valid, whole;   // this rank's region lists (cut to its contigs by keepOwnContigs)
  explicit RankInputs(SharedInputs* shared) : in(shared ? shared->in : own) {}
  bool open(Options& o, SharedInputs* shared) {
    if (!shared && !openInputs(o, own)) return false;
    valid = in.validRegions; whole = in.wholeContigs;
    return true;
  }
  std::vector<io::AlignmentFile>& files(Options const& o, SharedInputs* shared) {
    if (!shared) return in.files;
    if (ownFiles.empty()) {
      ownFiles.resize(o.files.size());
      for (std::size_t f = 0; f < o.files.size(); ++f) if (!ownFiles[f].open(o.files[f], o.genome, o.ioThreads)) { ownFiles.clear(); break; }
    }
    return ownFiles;
  }
};

// this rank's contigs and records (--shard-by contig), one line on stderr
void reportShare(Options const& o, Inputs const& in, std::vector<std::size_t> const& bounds, std::size_t n) {
  const std::size_t lo = bounds[o.rank], hi = bounds[o.rank + 1];
  std::ostringstream s;   // one write: the ranks of a --devices process report side by side
  s << "rank " << o.rank << "/" << o.nranks << ": contigs ";
  if (lo < hi) s << lo << "-" << hi - 1 << " (" << in.target_name[lo] << ".." << in.target_name[hi - 1] << ")";
  else s << "none";
  s << ", " << n << " records\n";
  std::cerr << s.str() << std::flush;
}

int runSr(Options& o, DeviceSession& dev, SharedInputs* shared = nullptr) {
  StageClock clock = shared ? shared->clock : StageClock();
  clock.t0 = std::chrono::steady_clock::now();
  RankInputs ri(shared);
  if (!ri.open(o, shared)) return 1;
  Inputs& in = ri.in;
  if (!shared) clock.lap("open_inputs");
  Config& c = o.c;
  const std::size_t F = in.files.size();
  const bool byContig = o.shardBy == "contig";
  Shard shard = dev.shard();
  ShareStats share;
  // exclude file: contigs without a valid region are excluded as a whole; the scan skips pairs whose mate is there (src/shortpe.h:399)
  if (o.hasExclude) c.contigExcluded = excludedContigs(in.validRegions);
  if (byContig) {   // this rank reads its own contigs only (the exclude flags above are the whole genome's)
    shard.contigBounds = contigCut(o, in);
    if (o.nranks == 1) shard.gather = [](std::string const& local, std::vector<std::string>& parts) { parts.assign(1, local); return (int) DGPU_OK; };
    keepOwnContigs(shard.contigBounds, o.rank, ri.valid, ri.whole);
    GatherFn g = shard.gather;
    shard.gather = [g, &share, &clock](std::string const& local, std::vector<std::string>& parts) {
      share.sentAtLap[clock.ms.size()] += local.size();
      return g(local, parts);
    };
  }
  const bool dump = !o.dumpfile.empty();
  SrReads ownReads;
  const bool readHere = !(shared && shared->haveReads);
  if (readHere) {
    std::vector<io::AlignmentFile>& files = ri.files(o, shared);
    if (files.size() != F || !readSr(o, files, ri.valid, ri.whole, ownReads)) return 1;
    clock.lap("read_bam");
  }
  SrReads const& rd = readHere ? ownReads : shared->sr;
  std::vector<std::vector<SrRecord> const*> samples, genoSamples;
  for (std::size_t f = 0; f < F; ++f) {
    samples.push_back(&rd.recs[f]);
    if (o.hasExclude) genoSamples.push_back(&rd.recsWhole[f]);
  }
  if (byContig) {
    std::size_t n = 0;
    for (std::size_t f = 0; f < F; ++f) n += rd.recs[f].size() + (o.hasExclude ? rd.recsWhole[f].size() : 0);
    reportShare(o, in, shard.contigBounds, n);
    share.records = n;
    if (o.readShareOnly) { writeTiming(o, clock, 0, &share); return 0; }
  }
  std::vector<LibraryInfo> libs(F);
  for (std::size_t f = 0; f < F; ++f) {
    if (byContig) {   // the first alignments in contig order may lie on other ranks' contigs: the screen continues rank after rank
      const int lrc = getLibraryParamsSharded(c, in.target_len, rd.recs[f], shard.contigShard(), libs[f]);
      if (lrc) { std::cerr << "delly_b200: the library exchange failed (" << lrc << ")" << std::endl; return 1; }
    } else getLibraryParams(c, in.target_len, rd.recs[f], libs[f]);
    if (libs[f].rs == 0) { std::cerr << "Sample has not enough data to estimate library parameters! File: " << o.files[f] << std::endl; return 1; }
  }
  clock.lap("library");
  if (!dev.wait()) return 3;
  clock.lap("wait_device");
  dgpu_ctx* ctx = dev.ctx();
  SrMultiCallSet cs;
  SvReadDump reads;
  int rc;
  if (!o.hasVcf)
    rc = dellySrCallSharded(ctx, c, libs, in.target_len, in.target_name, in.genome.cseq, samples, shard, cs, &clock, o.hasExclude ? &genoSamples : nullptr, dump ? &reads : nullptr);
  else {
    std::vector<VcfSite> sites;
    bool hasConsBp = false;
    if (!io::readSites(o.vcffile, sites, hasConsBp)) return 1;
    rc = dellySrGenotypeSharded(ctx, c, libs, in.target_len, in.target_name, in.genome.cseq, sites, hasConsBp, o.hasExclude ? genoSamples : samples, shard, cs, &clock,
                                dump ? &reads : nullptr);
    if (rc == DGPU_ERR_ARG && !cs.sample.empty()) { std::cerr << "Error: Delly genotyping requires a Delly BCF file from v1.1.7 or later!" << std::endl; rc = DGPU_OK; }
  }
  if (rc) { std::cerr << "delly_b200: device path failed (" << rc << "): " << dgpu_last_error(ctx) << std::endl; return 1; }
  if (o.rank != 0) { writeTiming(o, clock, cs.svs.size(), byContig ? &share : nullptr); return 0; }   // every rank holds the complete call set; rank 0 writes it
  if (dump && !cs.svs.empty()) {   // the reference opens the dump in annotateCoverage, which an empty SV list skips (src/delly.h:176)
    std::vector<std::vector<SrRecord> const*> const& geno = o.hasExclude ? genoSamples : samples;
    if (!writeDump(o.dumpfile, [&](auto put) { writeSrReadDump(put, reads, o.files, geno, rd.names, in.target_name); })) return 1;
    clock.lap("write_dump");
  }
  // src/delly.h:161-178: the count maps stay empty (and the header gets no sample column) when there is nothing to genotype
  std::vector<VcfSample> vs;
  if (!cs.svs.empty())
    for (std::size_t f = 0; f < F; ++f) {
      VcfSample s; s.name = in.sampleName[f]; s.jctMap = &cs.sample[f].jctMap; s.rcMap = &cs.sample[f].rcMap; s.spanMap = &cs.sample[f].spanMap;
      vs.push_back(s);
    }
  if (shared) shared->outputOpened = true;
  io::HtsVcfWriter w(o.outfile, in.target_name);
  if (!w.ok()) { std::cerr << "cannot open " << o.outfile << std::endl; return 1; }
  vcfRecordsTo(w, cs.svs, vs, in.target_name, in.target_len, o.genome, io::todayIso(), o.hasVcf, 0);
  w.close();
  clock.lap("write_bcf");
  writeTiming(o, clock, cs.svs.size(), byContig ? &share : nullptr);
  for (std::size_t f = 0; f < F; ++f)
    std::cerr << "Sample:" << in.sampleName[f] << ",ReadSize=" << libs[f].rs << ",Median=" << libs[f].median << ",MAD=" << libs[f].mad << ",UniqueDiscordantPairs=" << libs[f].abnormal_pairs << std::endl;
  return 0;
}

int runLr(Options& o, DeviceSession& dev, const char* argv0, SharedInputs* shared = nullptr) {
  StageClock clock = shared ? shared->clock : StageClock();
  clock.t0 = std::chrono::steady_clock::now();
  RankInputs ri(shared);
  if (!ri.open(o, shared)) return 1;
  Inputs& in = ri.in;
  if (!shared) clock.lap("open_inputs");
  Config& c = o.c;
  const std::size_t F = in.files.size();
  if (o.mode == "pb") o.indelExtension = 0.7f;
  else if (o.mode == "ont") o.indelExtension = 0.5f;
  MeiTemplates mei;
  const std::string meiPath = o.meifile.empty() ? exeDir(argv0) + "/../data/_mei_templates.fa" : o.meifile;
  if (!loadMei(meiPath, mei)) { std::cerr << "cannot read the annotation templates " << meiPath << " (see --mei)" << std::endl; return 1; }
  const bool byContig = o.shardBy == "contig";
  Shard shard = dev.shard();
  ShareStats share;
  if (byContig) {   // this rank reads its own contigs only: its valid regions, and its whole contigs with -x
    shard.contigBounds = contigCut(o, in);
    if (o.nranks == 1) shard.gather = [](std::string const& local, std::vector<std::string>& parts) { parts.assign(1, local); return (int) DGPU_OK; };
    keepOwnContigs(shard.contigBounds, o.rank, ri.valid, ri.whole);
    GatherFn g = shard.gather;
    shard.gather = [g, &share, &clock](std::string const& local, std::vector<std::string>& parts) {
      share.sentAtLap[clock.ms.size()] += local.size();
      return g(local, parts);
    };
  }
  const bool dump = !o.dumpfile.empty();
  LrReads ownReads;
  const bool readHere = !(shared && shared->haveReads);
  if (readHere) {
    std::vector<io::AlignmentFile>& files = ri.files(o, shared);
    if (files.size() != F || !readLr(o, files, ri.valid, ri.whole, ownReads)) return 1;
    clock.lap("read_bam");
  }
  LrReads const& rd = readHere ? ownReads : shared->lr;
  std::vector<LrSample> samples, genoSamples;
  for (std::size_t f = 0; f < F; ++f) {
    samples.push_back(LrSample{&rd.recs[f], &rd.ids[f]});
    if (o.hasExclude) genoSamples.push_back(LrSample{&rd.recsWhole[f], &rd.idsWhole[f]});
  }
  if (byContig) {
    std::size_t n = 0;
    for (std::size_t f = 0; f < F; ++f) n += rd.recs[f].size() + (o.hasExclude ? rd.recsWhole[f].size() : 0);
    reportShare(o, in, shard.contigBounds, n);
    share.records = n;
    if (o.readShareOnly) { writeTiming(o, clock, 0, &share); return 0; }
  }
  if (!dev.wait()) return 3;
  clock.lap("wait_device");
  dgpu_ctx* ctx = dev.ctx();
  LrMultiCallSet cs;
  SvReadDump reads;
  int rc;
  if (!o.hasVcf)
    rc = dellyLrCallSharded(ctx, c, o.indelExtension, in.target_len, in.target_name, in.genome.cseq, samples, shard, cs, &mei, o.anno, &o.methyl,
                            o.hasExclude ? &genoSamples : nullptr, dump ? &reads : nullptr, &clock);
  else {
    std::vector<VcfSite> sites;
    bool hasConsBp = false;
    if (!io::readSites(o.vcffile, sites, hasConsBp)) return 1;
    rc = dellyLrGenotypeSharded(ctx, c, in.target_len, in.target_name, in.genome.cseq, sites, hasConsBp, o.hasExclude ? genoSamples : samples, shard, cs, &mei, o.anno,
                                &o.methyl, dump ? &reads : nullptr, &clock);
    if (rc == DGPU_ERR_ARG && !cs.sample.empty()) { std::cerr << "Error: Delly genotyping requires a Delly BCF file from v1.1.7 or later!" << std::endl; rc = DGPU_OK; }
  }
  if (rc) { std::cerr << "delly_b200: device path failed (" << rc << "): " << dgpu_last_error(ctx) << std::endl; return 1; }
  if (o.rank != 0) { writeTiming(o, clock, cs.svs.size(), byContig ? &share : nullptr); return 0; }   // every rank holds the complete call set; rank 0 writes it
  if (dump && !cs.svs.empty()) {   // genotypeLR returns before it opens the dump when the SV list is empty (src/genotype.h:97, :127-133)
    std::vector<std::vector<LrRecord> const*> geno;
    for (LrSample const& s : (o.hasExclude ? genoSamples : samples)) geno.push_back(s.recs);
    if (!writeDump(o.dumpfile, [&](auto put) { writeLrReadDump(put, reads, o.files, geno, rd.names, in.target_name); })) return 1;
    clock.lap("write_dump");
  }
  // long reads have no spanning pairs: empty lists per SV (src/tegua.h:173-190)
  std::vector<SpanningCount> noSpan(cs.svs.size());
  std::vector<VcfSample> vs;
  for (std::size_t f = 0; f < F; ++f) {
    VcfSample s; s.name = in.sampleName[f]; s.jctMap = &cs.sample[f].jctMap; s.rcMap = &cs.sample[f].rcMap; s.spanMap = &noSpan; s.methylMap = &cs.sample[f].methyl;
    vs.push_back(s);
  }
  if (shared) shared->outputOpened = true;
  io::HtsVcfWriter w(o.outfile, in.target_name);
  if (!w.ok()) { std::cerr << "cannot open " << o.outfile << std::endl; return 1; }
  vcfRecordsTo(w, cs.svs, vs, in.target_name, in.target_len, o.genome, io::todayIso(), o.hasVcf, o.methyl.minCpgDepth);
  w.close();
  clock.lap("write_bcf");
  writeTiming(o, clock, cs.svs.size(), byContig ? &share : nullptr);
  return 0;
}

// --devices: every rank a host thread of this process, on its own device and context (sessions[r], started by main so that the contexts are
// created while the inputs are read), exchanging through `ex`. The process opens the inputs once and, with --shard-by svs, reads the record
// lists once; with --shard-by contig every rank reads its own contigs, all at the same time. The ranks split the IO and host-stage thread
// budgets. The first rank to fail releases the others (ex.fail()); the process then reports that rank and leaves no BCF behind.
int runDevices(Options& o, std::vector<std::unique_ptr<DeviceSession> >& sessions, SimExchange& ex, const char* argv0) {
  const int N = (int) o.devices.size();
  SharedInputs shared;
  if (!openInputs(o, shared.in)) { ex.fail(); return 1; }
  shared.clock.lap("open_inputs");
  if (o.shardBy == "svs") {   // every rank needs every record: one read, with the whole IO budget
    const bool ok = o.lr ? readLr(o, shared.in.files, shared.in.validRegions, shared.in.wholeContigs, shared.lr)
                         : readSr(o, shared.in.files, shared.in.validRegions, shared.in.wholeContigs, shared.sr);
    if (!ok) { ex.fail(); return 1; }
    shared.haveReads = true;
    shared.clock.lap("read_bam");
  }
  const unsigned hostShare = std::max(1u, processHostThreads() / (unsigned) N);
  std::vector<int> rcs((std::size_t) N, 0);
  std::atomic<int> firstFailed(-1);
  std::vector<std::thread> th;
  for (int r = 0; r < N; ++r)
    th.emplace_back([&, r] {
      rankHostThreads() = hostShare;
      Options ro = o;
      ro.rank = r; ro.device = o.devices[r]; ro.ioThreads = std::max(1, o.ioThreads / N);
      rcs[r] = o.lr ? runLr(ro, *sessions[r], argv0, &shared) : runSr(ro, *sessions[r], &shared);
      if (rcs[r]) {
        int none = -1;
        firstFailed.compare_exchange_strong(none, r);
        ex.fail();
      }
    });
  for (auto& t : th) t.join();
  const int bad = firstFailed.load();
  if (bad < 0) return 0;
  std::cerr << "delly_b200: rank " << bad << " of " << N << " (device " << o.devices[bad] << ") failed; the other ranks were stopped" << std::endl;
  if (shared.outputOpened && o.outfile != "-") { std::remove(o.outfile.c_str()); std::remove((o.outfile + ".csi").c_str()); }
  return rcs[bad];
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2 || (std::strcmp(argv[1], "sr") && std::strcmp(argv[1], "lr"))) { std::cerr << "usage: delly_b200 sr|lr [OPTIONS] -g <ref.fa> <in.bam> ..." << std::endl; return 1; }
  Options o;
  o.lr = !std::strcmp(argv[1], "lr");
  if (!parse(argc - 1, argv + 1, o)) return 1;
  if (o.help || o.files.empty() || o.genome.empty()) { usage(o); return 0; }
  if (!svTypesToCompute(o.c, o.svtype)) { std::cerr << "Please specify a valid SV type, i.e., -t INV or -t DEL,INV without spaces." << std::endl; return 1; }
  const uint32_t hw = std::thread::hardware_concurrency() ? std::thread::hardware_concurrency() : 1;
  o.c.maxThreads = std::min<uint32_t>(std::max<uint32_t>(1, o.c.maxThreads), hw);   // src/delly.h:268
  if (o.c.minCliqueSize < 2) o.c.minCliqueSize = 2;
  if (o.c.minMapQual > o.c.minTraQual) o.c.minTraQual = o.c.minMapQual;
  if (o.c.minGenoQual < 5 && !o.lr) o.c.minGenoQual = 5;   // src/delly.h:386
  if (!o.devices.empty()) {   // before any input is read
    const int ndev = dgpu_device_count();   // < 0: no CUDA driver here; creating the contexts reports that
    for (int d : o.devices)
      if (ndev >= 0 && d >= ndev) { std::cerr << "--devices: there is no device " << d << " (this process sees " << ndev << ")" << std::endl; return 1; }
  }
  std::unique_ptr<SimExchange> ex;
  std::vector<std::unique_ptr<DeviceSession> > sessions;   // one per rank, creating its context from here on
  if (o.devices.empty()) sessions.emplace_back(new DeviceSession(o));
  else {
    ex.reset(new SimExchange((int) o.devices.size()));
    for (std::size_t k = 0; k < o.devices.size(); ++k) {
      Options ro = o;
      ro.rank = (int) k; ro.device = o.devices[k];
      sessions.emplace_back(new DeviceSession(ro, ex.get()));
    }
  }
  const int r = !o.devices.empty() ? runDevices(o, sessions, *ex, argv[0]) : o.lr ? runLr(o, *sessions[0], argv[0]) : runSr(o, *sessions[0]);
  DeviceLimitLog const& lim = deviceLimitLog();   // the sum over the ranks of a --devices run
  if (lim.total())
    std::cerr << "Warning: " << lim.msaClusters.load() << " read cluster(s) (over " << DGPU_MSA_LARGE_MAXR << " reads, over 1023 alignment columns or a byte"
              << " outside ACGTN), " << lim.pathJobs.load() << " edit-path job(s) (an aligned target slice over " << DGPU_EP_MAX_SLICE
              << " bases) and " << lim.needleJobs.load()
              << " consensus alignment(s) (a consensus over 16383 bases or a reference window over " << DGPU_LN_MAX_REF << " bases) exceeded a device limit (include/dgpu.h) and were treated as failed alignments of their SV / read; the reference"
                 " has no such limits, so these records may differ from its output." << std::endl;
  // Every output is written and closed at this point. Tearing the CUDA context, the NCCL communicator and a few GB of device scratch down
  // costs a few hundred ms and produces nothing: leave that to the operating system (DGPU_CLEAN_EXIT=1 keeps the orderly teardown, e.g. under
  // compute-sanitizer).
  if (!getenv("DGPU_CLEAN_EXIT")) { std::cout.flush(); std::cerr.flush(); fflush(nullptr); _exit(r); }
  return r;
}
