// tests/standin/edit_path_wide_standin.cpp — TEST INFRASTRUCTURE ONLY (CPU suite). Linked next to host_standin.cpp by
// tests/test_edit_path_wide.py: dgpu_edit_path_wide forwarded to the stand-in's dgpu_edit_path_ex (the reference's own edlib, which has no
// slice limit), so that the host mirrors' path calls with targets wider than 16384 columns are served on a machine without a GPU. A job whose
// aligned slice is wider than max_slice gets status 2 and no ops, as from the device.
#include <cstdint>
#include "../../include/dgpu.h"

extern "C" int dgpu_edit_path_wide(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* q_off, const uint32_t* q_len, const uint32_t* t_off,
                                   const uint32_t* t_len, int mode, const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n, int32_t* dist, int32_t* start_loc,
                                   int32_t* end_loc, uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes, uint32_t* ops_len, uint32_t* status,
                                   uint32_t max_slice) {
  if (max_slice < 1 || max_slice > DGPU_EP_MAX_SLICE) return DGPU_ERR_ARG;
  const int rc = dgpu_edit_path_ex(ctx, seqs, seqs_bytes, q_off, q_len, t_off, t_len, mode, eq_pairs, n_eq, n, dist, start_loc, end_loc, ops, ops_off, ops_bytes,
                                   ops_len, status);
  for (uint64_t i = 0; i < n && rc == DGPU_OK; ++i)
    if (status[i] == 0 && dist[i] >= 0 && end_loc[i] >= 0 && (int64_t) end_loc[i] - start_loc[i] + 1 > (int64_t) max_slice) { status[i] = 2; ops_len[i] = 0; }
  return rc;
}
