// msa.hpp — per-SV split-read consensus (src/msa.h:185-239 as called from src/shortpe.h:185,252), batched:
// msaBatch(ctx, c, clusters, consensus, rows) runs every cluster of a chromosome in one dgpu_msa_ex call.
// The caller passes each cluster's reads in the iteration order of the reference's
// std::unordered_set<std::string> (src/shortpe.h:68-70) — order matters for the guide tree ties.
#pragma once
#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/dgpu.h"
#include "types.hpp"

namespace dellyb200 {

inline int msaBatch(dgpu_ctx* ctx, Config const& c, std::vector<std::vector<std::string> > const& clusters, std::vector<std::string>& consensus,
                    std::vector<int>& rows) {
  const std::size_t N = clusters.size();
  consensus.assign(N, std::string());
  rows.assign(N, 0);
  if (!N) return DGPU_OK;
  std::string arena;
  std::vector<uint32_t> roff, rlen, coff(1, 0);
  std::vector<uint64_t> cons_off(N);
  uint64_t cbytes = 0;
  std::size_t largest = 0;
  for (std::size_t i = 0; i < N; ++i) {
    cons_off[i] = cbytes;
    largest = std::max(largest, clusters[i].size());
    for (std::string const& r : clusters[i]) {
      roff.push_back((uint32_t) arena.size()); rlen.push_back((uint32_t) r.size()); arena += r;
      cbytes += r.size();
    }
    coff.push_back((uint32_t) roff.size());
  }
  std::vector<uint8_t> cons(cbytes + 1);
  std::vector<uint32_t> clen(N), nrows(N), status(N);
  // every cluster the device can take: the large-cluster workspace is sized for the largest one. A batch without clusters of more
  // than 32 reads goes through dgpu_msa (= dgpu_msa_ex with max_reads 32), the entry point every binding of the ABI provides,
  // including the CPU suite's stand-in of it (tests/standin/host_standin.cpp forwards dgpu_msa to the reference's msa).
  const uint32_t max_reads = (uint32_t) std::min<std::size_t>(largest, DGPU_MSA_LARGE_MAXR);
  const int rc = max_reads > 32
      ? dgpu_msa_ex(ctx, (const uint8_t*) arena.data(), arena.size(), roff.data(), rlen.data(), (uint32_t) roff.size(), coff.data(), (uint32_t) N,
                    c.aliscore.match, c.aliscore.mismatch, c.aliscore.go, c.aliscore.ge, c.minCliqueSize, cons.data(), cons_off.data(), cbytes,
                    clen.data(), nrows.data(), status.data(), nullptr, nullptr, 0, nullptr, max_reads)
      : dgpu_msa(ctx, (const uint8_t*) arena.data(), arena.size(), roff.data(), rlen.data(), (uint32_t) roff.size(), coff.data(), (uint32_t) N,
                 c.aliscore.match, c.aliscore.mismatch, c.aliscore.go, c.aliscore.ge, c.minCliqueSize, cons.data(), cons_off.data(), cbytes,
                 clen.data(), nrows.data(), status.data(), nullptr, nullptr, 0, nullptr);
  if (rc) return rc;
  for (std::size_t i = 0; i < N; ++i) {
    if (status[i]) { ++deviceLimitLog().msaClusters; consensus[i].clear(); rows[i] = 0; continue; }   // this SV gets no consensus (counted, reported)
    consensus[i].assign((const char*) cons.data() + cons_off[i], clen[i]);
    rows[i] = (int) nrows[i];
  }
  return DGPU_OK;
}

}  // namespace dellyb200
