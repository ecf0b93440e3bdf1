// tests/standin/msa_ex_standin.cpp — TEST INFRASTRUCTURE ONLY (CPU suite). Linked next to host_standin.cpp or binding_standin.cpp by
// tests/test_msa_large.py: dgpu_msa_ex forwarded to the stand-in's dgpu_msa (the reference's own msa, which has no read-count limit),
// so that the host mirrors' calls for clusters of more than 32 reads are served on a machine without a GPU.
#include <cstdint>
#include "../../include/dgpu.h"

extern "C" int dgpu_msa_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes, const uint32_t* read_off, const uint32_t* read_len, uint32_t nreads,
                           const uint32_t* cluster_off, uint32_t nclusters, int match, int mismatch, int go, int ge, int min_clique, uint8_t* cons,
                           const uint64_t* cons_off, uint64_t cons_bytes, uint32_t* cons_len, uint32_t* n_rows, uint32_t* status, uint8_t* aln,
                           const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_cols, uint32_t) {
  return dgpu_msa(ctx, seqs, seqs_bytes, read_off, read_len, nreads, cluster_off, nclusters, match, mismatch, go, ge, min_clique, cons, cons_off, cons_bytes,
                  cons_len, n_rows, status, aln, aln_off, aln_bytes, aln_cols);
}
