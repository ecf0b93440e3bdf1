// tests/standin/long_needle_ex_standin.cpp — TEST INFRASTRUCTURE ONLY (CPU suite). Linked next to host_standin.cpp by
// tests/test_long_needle_wide.py: dgpu_long_needle_ex forwarded to the stand-in's dgpu_long_needle (the reference's own longNeedle, which has
// no window limit), so that the host mirrors' calls for windows beyond the wavefront kernels' shapes are served on a machine without a GPU.
#include <cstdint>
#include "../../include/dgpu.h"

extern "C" int dgpu_long_needle_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* c_off, const uint32_t* c_len, const uint32_t* r_off,
                                   const uint32_t* r_len, uint64_t n, uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_len, uint8_t* ok,
                                   int32_t* info, uint32_t) {
  return dgpu_long_needle(ctx, seqs, seqs_bytes, c_off, c_len, r_off, r_len, n, aln, aln_off, aln_bytes, aln_len, ok, info);
}
