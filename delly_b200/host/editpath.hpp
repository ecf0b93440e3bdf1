// editpath.hpp — the one rule by which the host mirrors pick the edit-path entry point for a batch of edlibAlign(..., EDLIB_TASK_PATH) calls.
#pragma once
#include <cstdint>

#include "../../include/dgpu.h"

namespace dellyb200 {

// dgpu_edit_path_wide with the widest slice the device traces when a target is wider than DGPU_EP_CLASSIC_SLICE (an aligned slice is never
// wider than its target), otherwise dgpu_edit_path_ex, which computes those batches the same way. A job still beyond the cap comes back
// with status 2.
inline int editPathCall(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* qo, const uint32_t* ql, const uint32_t* to,
                        const uint32_t* tl, int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* st, int32_t* en,
                        uint8_t* ops, const uint64_t* oo, uint64_t obytes, uint32_t* olen, uint32_t* status) {
  bool wide = false;
  for (uint64_t i = 0; i < n && !wide; ++i) wide = tl[i] > DGPU_EP_CLASSIC_SLICE;
  if (wide)
    return dgpu_edit_path_wide(ctx, seqs, seqs_bytes, qo, ql, to, tl, mode, eq_pairs, n_eq, n, dist, st, en, ops, oo, obytes, olen, status, DGPU_EP_MAX_SLICE);
  return dgpu_edit_path_ex(ctx, seqs, seqs_bytes, qo, ql, to, tl, mode, eq_pairs, n_eq, n, dist, st, en, ops, oo, obytes, olen, status);
}

}  // namespace dellyb200
