// edlib_compat.hpp — implementation of include/dgpu_edlib.h: the edlib C API (src/edlib.h) as single-job calls into the
// batched C ABI. See the header for the contract (per-thread context, no CPU fallback, first location only).
#pragma once
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dgpu.h"
#include "editpath.hpp"
#define DGPU_EDLIB_NO_ALIASES
#include "../../include/dgpu_edlib.h"

namespace dellyb200 {
namespace detail {
// Test seam: the context the compat layer uses instead of creating its own (set by the CPU stand-in build, whose device entry points
// ignore it). Null = create one on first use. One per process, read by every thread that aligns through the compat layer: atomic.
inline std::atomic<dgpu_ctx*>& edlibCompatCtxOverride() { static std::atomic<dgpu_ctx*> p{nullptr}; return p; }
inline dgpu_ctx* edlibCompatCtx() {
  if (edlibCompatCtxOverride()) return edlibCompatCtxOverride();
  thread_local dgpu_ctx* ctx = nullptr;
  thread_local bool tried = false;
  if (!ctx && !tried) {
    tried = true;
    const char* dev = std::getenv("DGPU_DEVICE");
    if (dgpu_ctx_create(dev ? std::atoi(dev) : 0, &ctx) != DGPU_OK) ctx = nullptr;
  }
  return ctx;
}
}  // namespace detail
}  // namespace dellyb200

extern "C" {

EdlibAlignConfig dgpu_edlibNewAlignConfig(int k, EdlibAlignMode mode, EdlibAlignTask task, const EdlibEqualityPair* additionalEqualities,
                                          int additionalEqualitiesLength) {
  EdlibAlignConfig c;
  c.k = k; c.mode = mode; c.task = task;
  c.additionalEqualities = additionalEqualities; c.additionalEqualitiesLength = additionalEqualitiesLength;
  return c;
}

EdlibAlignConfig dgpu_edlibDefaultAlignConfig(void) { return dgpu_edlibNewAlignConfig(-1, EDLIB_MODE_NW, EDLIB_TASK_DISTANCE, nullptr, 0); }

EdlibAlignResult dgpu_edlibAlign(const char* query, int queryLength, const char* target, int targetLength, const EdlibAlignConfig config) {
  EdlibAlignResult r;
  r.status = EDLIB_STATUS_OK; r.editDistance = -1; r.endLocations = nullptr; r.startLocations = nullptr; r.numLocations = 0;
  r.alignment = nullptr; r.alignmentLength = 0; r.alphabetLength = 0;
  if (queryLength < 0 || targetLength < 0 || (config.mode != EDLIB_MODE_NW && config.mode != EDLIB_MODE_SHW && config.mode != EDLIB_MODE_HW)) {
    r.status = EDLIB_STATUS_ERROR;
    return r;
  }
  bool seen[256] = {false};
  for (int i = 0; i < queryLength; ++i) seen[(unsigned char) query[i]] = true;
  for (int i = 0; i < targetLength; ++i) seen[(unsigned char) target[i]] = true;
  for (int b = 0; b < 256; ++b) r.alphabetLength += seen[b];
  dgpu_ctx* ctx = dellyb200::detail::edlibCompatCtx();
  if (!ctx) { r.status = EDLIB_STATUS_ERROR; return r; }
  std::string arena(query, query + queryLength);
  arena.append(target, target + targetLength);
  arena.push_back('\0');
  const uint32_t qo = 0, ql = (uint32_t) queryLength, to = (uint32_t) queryLength, tl = (uint32_t) targetLength;
  const int32_t k = config.k;
  int32_t dist = -1, start = -1, end = -1;
  const bool wantPath = (config.task == EDLIB_TASK_PATH), wantStart = wantPath || (config.task == EDLIB_TASK_LOC);
  const bool hasEq = config.additionalEqualitiesLength > 0;
  const bool emptySide = (queryLength == 0 || targetLength == 0);   // edlib returns before start locations / a path exist (src/edlib.cpp:158-177)
  int rc;
  if (emptySide || (!wantStart && !hasEq)) {
    // the distance entry point: DISTANCE without additional equalities, and every empty-sequence case
    rc = dgpu_edit_distance(ctx, (const uint8_t*) arena.data(), arena.size(), &qo, &ql, &to, &tl, &k, (int) config.mode, 1, &dist, &end);
    if (rc) { r.status = EDLIB_STATUS_ERROR; return r; }
    r.editDistance = dist;
    if (dist >= 0) { r.endLocations = (int*) std::malloc(sizeof(int)); r.endLocations[0] = end; r.numLocations = 1; }
    return r;
  }
  // the path entry point (it also carries the additional equalities, which the distance entry point does not take)
  std::vector<uint8_t> ops((size_t) queryLength + (size_t) targetLength + 1);
  const uint64_t opsOff = 0;
  uint32_t opsLen = 0, status = 0;
  std::vector<uint8_t> eq;
  for (int i = 0; i < config.additionalEqualitiesLength; ++i) { eq.push_back((uint8_t) config.additionalEqualities[i].first); eq.push_back((uint8_t) config.additionalEqualities[i].second); }
  rc = dellyb200::editPathCall(ctx, (const uint8_t*) arena.data(), arena.size(), &qo, &ql, &to, &tl, (int) config.mode, eq.empty() ? nullptr : eq.data(),
                               (uint32_t) (eq.size() / 2), 1, &dist, &start, &end, ops.data(), &opsOff, ops.size(), &opsLen, &status);
  if (rc || status) { r.status = EDLIB_STATUS_ERROR; return r; }
  if (k >= 0 && dist > k) dist = -1;   // the path entry points are unbounded; edlib reports -1 (and no locations) beyond k
  r.editDistance = dist;
  if (dist < 0) return r;
  r.endLocations = (int*) std::malloc(sizeof(int)); r.endLocations[0] = end; r.numLocations = 1;
  if (wantStart) { r.startLocations = (int*) std::malloc(sizeof(int)); r.startLocations[0] = start; }
  if (wantPath) {
    r.alignment = (unsigned char*) std::malloc(opsLen ? opsLen : 1);
    std::memcpy(r.alignment, ops.data(), opsLen);
    r.alignmentLength = (int) opsLen;
  }
  return r;
}

void dgpu_edlibFreeAlignResult(EdlibAlignResult result) {
  std::free(result.endLocations);
  std::free(result.startLocations);
  std::free(result.alignment);
}

char* dgpu_edlibAlignmentToCigar(const unsigned char* alignment, int alignmentLength, EdlibCigarFormat cigarFormat) {
  if (cigarFormat != EDLIB_CIGAR_EXTENDED && cigarFormat != EDLIB_CIGAR_STANDARD) return nullptr;
  const char* sym = (cigarFormat == EDLIB_CIGAR_STANDARD) ? "MIDM" : "=IDX";
  std::string out;
  int i = 0;
  while (i < alignmentLength) {
    if (alignment[i] > 3) return nullptr;
    const char ch = sym[alignment[i]];
    int run = 0;
    // a run ends where the SYMBOL changes (match and mismatch share 'M' in the standard format)
    while (i < alignmentLength && alignment[i] <= 3 && sym[alignment[i]] == ch) { ++run; ++i; }
    out += std::to_string(run);
    out.push_back(ch);
  }
  char* c = (char*) std::malloc(out.size() + 1);
  std::memcpy(c, out.c_str(), out.size() + 1);
  return c;
}

}  // extern "C"
