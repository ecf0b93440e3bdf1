/*
 * dgpu.h — C ABI of libdelly_b200: batched, H100-native (sm_90a) replacements for the
 * per-item alignment calls on Delly's split-read / consensus realignment path.
 *
 * The reference (dellytools/delly @ 3a22fe2) has no FFI; it is one translation unit of
 * inline templates. Each entry point below names the reference call site(s) it replaces
 * (paths relative to the reference root). A maintainer binds them by replacing the
 * per-item loop at that call site with one batched call (see INTEGRATION.md).
 *
 * Conventions
 *  - extern "C", plain pointers and sizes only. Return 0 (DGPU_OK) or a negative
 *    DGPU_ERR_* code; no exceptions cross the boundary.
 *  - Sequences are 1 byte per base in one packed arena (`seqs`); equality is byte
 *    equality exactly like edlib / the reference's char compares (so IUPAC codes,
 *    'N' and lower case keep the reference's semantics). Sequences may share or overlap
 *    bytes anywhere in the arena (a query inside its target, windows of one contig).
 *  - Every batch call exists in two forms:
 *      dgpu_<op>        host pointers in/out; the call stages H2D, launches, copies the
 *                       results D2H and returns when they are in the caller's buffers.
 *                       Pinned caller buffers are DMA'd directly.
 *      dgpu_<op>_dev    device pointers in/out, enqueued on `stream`
 *                       (a cudaStream_t passed as void*; NULL = the context's stream).
 *  - Caller buffers. Host forms check every job against the sizes given (sequences inside `seqs_bytes`, output slots inside `ops_bytes` /
 *    `aln_bytes` / `cons_bytes`) and return DGPU_ERR_ARG / DGPU_ERR_CAPACITY before anything is launched. Device forms trust their arguments
 *    (checking would need a device round trip); their arena must be readable in whole 16-byte words: 16-byte aligned, with >= 16 readable bytes
 *    after `seqs_bytes` (the kernels fetch the arena with aligned 128-bit loads).
 *  - A context is bound to one CUDA device and must not be shared between host threads
 *    (same contract as one edlib call per pool worker, src/coverage.h:420-426).
 *  - There is NO CPU fallback: if no CUDA device is usable, dgpu_ctx_create fails.
 */
#ifndef DGPU_H
#define DGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGPU_OK 0
#define DGPU_ERR_CUDA (-1)        /* a CUDA runtime call failed; see dgpu_last_error() */
#define DGPU_ERR_ARG (-2)         /* invalid argument */
#define DGPU_ERR_NODEVICE (-3)    /* no usable sm_90 device */
#define DGPU_ERR_CAPACITY (-4)    /* an output/workspace capacity was exceeded */
#define DGPU_ERR_UNSUPPORTED (-5) /* shape outside what the device path supports */
#define DGPU_ERR_NCCL (-6)

/* Alignment modes and tasks: numerically identical to EdlibAlignMode / EdlibAlignTask
 * (src/edlib.h:36-71) so call sites can pass their existing enum values. */
#define DGPU_MODE_NW 0
#define DGPU_MODE_SHW 1
#define DGPU_MODE_HW 2

typedef struct dgpu_ctx dgpu_ctx;

/* ---- context ------------------------------------------------------------------ */
int dgpu_ctx_create(int device, dgpu_ctx** out);
void dgpu_ctx_destroy(dgpu_ctx* ctx);
/* Block until everything queued on the context's stream has finished. */
int dgpu_ctx_sync(dgpu_ctx* ctx);
/* Text of the last CUDA/NCCL error seen by this context (never NULL). */
const char* dgpu_last_error(dgpu_ctx* ctx);
const char* dgpu_strerror(int code);
/* ABI version (major*1000+minor). */
int dgpu_version(void);
/* Number of CUDA devices this process can see (any architecture), or DGPU_ERR_NODEVICE when the runtime cannot count them (no driver). */
int dgpu_device_count(void);
/* Number of kernel launches issued through this context so far (bench accounting). */
uint64_t dgpu_launch_count(dgpu_ctx* ctx);
/* jobs refused PER ITEM so far because they exceed a device limit (the call still succeeds; the item comes back flagged: ok = 0 / status != 0).
 * Refusals of longNeedle and edit-path calls under dgpu_set_ln_async_bound / dgpu_set_ep_async_bound are read from the device here (a synchronisation of the context stream):
 * synchronise the stream such a call was enqueued on first. */
uint64_t dgpu_unsupported_count(dgpu_ctx* ctx);
/* Stream-asynchronous device forms. By default dgpu_edit_distance_dev reads its job-class counts back once per call (one small D2H + stream
 * synchronisation) so that it launches exactly the kernels the batch needs. With max_seq_len > 0 the caller guarantees that no query or target of
 * later calls is longer; the call then enqueues everything on `stream` and returns without any host synchronisation (scratch buffers are sized from
 * the bound and grown only between calls; it can be followed by further work on the stream, overlapped with copies on other streams, or captured
 * into a CUDA graph once the scratch exists). 0 switches back. dgpu_long_needle[_ex]_dev and dgpu_msa[_ex]_dev have bounds of their own,
 * below, and so has dgpu_edit_path[_ex|_wide]_dev (dgpu_set_ep_async_bound). */
int dgpu_set_async_bound(dgpu_ctx* ctx, uint32_t max_seq_len);
/* The same for the edit paths. With (max_query, max_target) set, the caller guarantees that no job of a later dgpu_edit_path[_ex|_wide][_dev]
 * call has q_len > max_query or t_len > max_target. The device forms then enqueue everything on `stream` and return without any host
 * synchronisation, read-back or copy from host memory: the distance passes run their asynchronous branch sized from max(max_query,
 * max_target), and every Hirschberg level is planned on the device, as many levels as the bound can need, each launching the half-column
 * kernels the bound can reach at that level with the grid and shared memory of the bound. The setter opts those kernels in to their shared
 * memory and reserves their workspace (within the workspace budget, at least one bound-shaped slab per kernel). The per-job scratch grows with
 * the number of jobs, so a call may be captured into a CUDA graph after one call with at least as many jobs. A job beyond the bound is refused
 * alone: status 4, dist = start = end = -1, ops_len = 0; the device forms count such refusals on the device, and dgpu_unsupported_count and
 * dgpu_ctx_sync add them once the work that made them has finished. The host forms take the same path and return the same bytes. Rules:
 * 1 <= max_query, max_target <= DGPU_EP_MAX_SLICE, else DGPU_ERR_ARG; (0, 0) switches back to the synchronous forms. The bound applies to
 * every edit-path call of the context and leaves dgpu_set_async_bound's meaning for dgpu_edit_distance* unchanged. */
int dgpu_set_ep_async_bound(dgpu_ctx* ctx, uint32_t max_query, uint32_t max_target);
/* The same for longNeedle. With (max_cons, max_ref) set, the caller guarantees that no job of a later dgpu_long_needle[_ex][_dev] call has
 * c_len > max_cons or r_len > max_ref. The device forms then read nothing back: one small kernel plans the workspace on the device from the
 * batch's per-class counts and largest shapes, and every job class the bound admits is launched with the grid and shared memory of the
 * bound (CTAs a class does not need return at once). The setter opts every such kernel in to its shared memory and reserves the workspace
 * pool: each admitted class at its full grid with bound-shaped slabs, within the workspace budget (0.6 x free memory), but at least one
 * bound-shaped slab per class. The per-job scratch grows with the number of jobs, so a call may be captured into a CUDA graph after one call
 * with at least as many jobs. Rules: max_cons <= 16383, max_ref <= DGPU_LN_MAX_REF, both > 0, else DGPU_ERR_ARG; (0, 0) switches back.
 * The bound applies to every longNeedle call of the context. dgpu_long_needle[_dev] (no wide engine) returns DGPU_ERR_ARG under a bound
 * its wavefront kernels cannot take, max_ref > 16377 or max_cons + max_ref > 32000; the _ex forms take any bound, and their max_ref
 * argument still limits the wide engine. A job beyond the bound or the limits below is refused alone (ok = 0, aln_len = 0, info[2] = -1).
 * The device forms count such refusals on the device: dgpu_unsupported_count and dgpu_ctx_sync add them to the count (and set
 * dgpu_last_error) once the work that made them has finished, not when the call returns. */
int dgpu_set_ln_async_bound(dgpu_ctx* ctx, uint32_t max_cons, uint32_t max_ref);
/* The same for the MSA. dgpu_msa[_ex]_dev read nothing back, but grow their workspace slots (which synchronises the device) the first time
 * a call needs more. With (max_reads, max_read_len) set, the setter reserves the slots of the largest grids for clusters of up to
 * max_reads reads, and later calls never grow them; a call's max_reads above the bound is lowered to it, so a larger cluster gets status 1.
 * Reads longer than 1023 bases get status 2 as always; the slots are sized for 1023-column alignments whatever max_read_len is.
 * Rules: max_reads <= DGPU_MSA_LARGE_MAXR, max_read_len <= 1023, both > 0, else DGPU_ERR_ARG; (0, 0) switches back. */
int dgpu_set_msa_async_bound(dgpu_ctx* ctx, uint32_t max_reads, uint32_t max_read_len);
/* Measurement hooks (bench.py): when profiling is on, every batch call brackets its dominant
 * kernels (not the staging copies or the binning pre-pass) with CUDA events on the launching
 * stream; dgpu_last_kernel_ms waits for and returns that span for the most recent call. */
int dgpu_set_profiling(dgpu_ctx* ctx, int on);
float dgpu_last_kernel_ms(dgpu_ctx* ctx);
/* Measured integer-ALU peak of this device: a LOP3/IADD3 micro-kernel, result in 1e12 int32 op/s.
 * MEASURED_PEAKS.json carries no integer peak, and this path is integer-pipe bound. */
int dgpu_int_peak(dgpu_ctx* ctx, double* tera_ops_per_s);
/* Whether IMADs issue to the FMA pipe alongside the integer ALU pipe: 1e12 instructions/s of [0] the LOP3 chains of dgpu_int_peak,
 * [1] the same LOP3 chains with as many IMAD chains interleaved, [2] the same with IMAD.WIDE.U32 in place of the IMADs. */
int dgpu_int_peak_mix(dgpu_ctx* ctx, double tera_instr_per_s[3]);

/* ---- Myers bit-vector edit distance (replaces edlibAlign with EDLIB_TASK_DISTANCE) --
 * Call sites: _editDistanceHW, src/coverage.h:107-115 (two per AlignJob in process_batch,
 * :412-441, and the dump path :520-521); _editDistanceNW, src/genotype.h:22-29
 * (:276,:284); orientation check src/split.h:567-568; msaEdlib pairs src/assemble.h:390.
 *
 * Job i aligns query seqs[q_off[i] .. +q_len[i]) against target seqs[t_off[i] .. +t_len[i])
 * in `mode` with bound k[i] (k < 0: unbounded, like edlib's auto-doubling k,
 * src/edlib.cpp:192-210). dist[i] = edit distance, or -1 if it exceeds k — bit-identical to
 * EdlibAlignResult.editDistance, including the HW clamp k=min(k,|q|) (src/edlib.cpp:563-565),
 * the NW rules (src/edlib.cpp:740-746) and the empty-sequence rules (src/edlib.cpp:158-177).
 * end_loc (may be NULL): endLocations[0] (leftmost optimal end, src/edlib.cpp:656-691), -1 if none.
 * `k` may be NULL (all unbounded). Offsets are 32-bit: one arena is at most 4 GiB.
 */
int dgpu_edit_distance(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                       const uint32_t* q_off, const uint32_t* q_len,
                       const uint32_t* t_off, const uint32_t* t_len,
                       const int32_t* k, int mode, uint64_t n,
                       int32_t* dist, int32_t* end_loc);
int dgpu_edit_distance_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                           const uint32_t* q_off, const uint32_t* q_len,
                           const uint32_t* t_off, const uint32_t* t_len,
                           const int32_t* k, int mode, uint64_t n,
                           int32_t* dist, int32_t* end_loc, void* stream);

/* ---- edit distance + locations + alignment path (replaces edlibAlign with EDLIB_TASK_PATH) --
 * Call sites (all with k = -1): splitAlign, src/split.h:485,489,497,507,524,527 (HW and SHW);
 * _trimConsensus src/assemble.h:351,356; msaEdlib/msaWfa src/assemble.h:447,656,693 (NW/HW).
 * Per job: dist (editDistance), start_loc / end_loc (startLocations[0] / endLocations[0], src/edlib.cpp:213-258),
 * ops = the alignment array (0 match, 1 insert, 2 delete, 3 mismatch; src/edlib.h:84-87) at ops + ops_off[i]
 * (reserve q_len + t_len bytes), ops_len (alignmentLength). Problems above edlib's 1 MiB switch are split with
 * Hirschberg's recursion exactly like the reference (src/edlib.cpp:1189-1212, :1232-1397), so paths are identical
 * at every size. status: 0 ok; 2 = aligned target slice t[start..end] wider than DGPU_EP_CLASSIC_SLICE = 16384 columns (_wide forms: wider than
 * max_slice); the job keeps the reference's distance and locations, its path is NOT produced; 3 = internal consistency failure;
 * 4 = refused under dgpu_set_ep_async_bound (q_len or t_len beyond the bound): dist = start = end = -1, ops_len = 0.
 * The _ex forms take edlib's additionalEqualities (src/edlib.h:100-106) as 2*n_eq bytes (first,second pairs,
 * n_eq <= 32) in every mode — the reference's call sites are src/assemble.h:425-447 (NW, msaEdlib) and
 * src/assemble.h:663-693 (HW, msaWfa).
 * The *_dev forms stage job geometry through the host between device rounds (they synchronise the stream).
 */
int dgpu_edit_path(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                   const uint32_t* q_off, const uint32_t* q_len,
                   const uint32_t* t_off, const uint32_t* t_len, int mode, uint64_t n,
                   int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                   uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes,
                   uint32_t* ops_len, uint32_t* status);
int dgpu_edit_path_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                       const uint32_t* q_off, const uint32_t* q_len,
                       const uint32_t* t_off, const uint32_t* t_len, int mode, uint64_t n,
                       int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                       uint8_t* ops, const uint64_t* ops_off,
                       uint32_t* ops_len, uint32_t* status, void* stream);

int dgpu_edit_path_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                      const uint32_t* q_off, const uint32_t* q_len,
                      const uint32_t* t_off, const uint32_t* t_len, int mode,
                      const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n,
                      int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                      uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes,
                      uint32_t* ops_len, uint32_t* status);
int dgpu_edit_path_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                          const uint32_t* q_off, const uint32_t* q_len,
                          const uint32_t* t_off, const uint32_t* t_len, int mode,
                          const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n,
                          int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                          uint8_t* ops, const uint64_t* ops_off,
                          uint32_t* ops_len, uint32_t* status, void* stream);
/* The _wide forms take the _ex arguments plus max_slice, the widest aligned target slice the caller wants traced (1 .. DGPU_EP_MAX_SLICE,
 * else DGPU_ERR_ARG); a job with a wider slice gets status 2 alone. The other forms are the _wide forms with max_slice =
 * DGPU_EP_CLASSIC_SLICE. Hirschberg segments of up to 16384 columns run on the band and wavefront engines as they always did; unbanded
 * segments wider than that run on a warp-per-segment half-column engine (a scratch row of one byte per column) and a two-lanes-per-leaf
 * traceback engine (leaves of at most 128 rows, 16 B per block and column). In every form, a half column with more query rows than the
 * wavefront engine can stage in shared memory (about 230 k; such a call used to fail with DGPU_ERR_CUDA) also runs on the half-column engine.
 * Cap: no buffer of these engines is sized by the slice width beyond O(m + n) scratch per segment, and their 32-bit arithmetic (int32 end
 * locations and step counts, the -(1<<28) over-estimate of banded half columns) would hold up to 2^27 columns. What bounds the cap is time:
 * an unbanded half column takes one warp for (m / 2048) x n steps, so a path's time grows with the square of the width. One 8 %-divergent NW
 * pair at 2^18 columns takes 15.7 s on an H100 80GB HBM3 at 700 W (profiles/h100_bench_epw.json); 2^19 would take about four times that
 * per path. DGPU_EP_MAX_SLICE is the widest slice the test suite checks against the reference. */
#define DGPU_EP_CLASSIC_SLICE 16384   /* the slice limit of dgpu_edit_path[_ex][_dev] */
#define DGPU_EP_MAX_SLICE 262144
int dgpu_edit_path_wide(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                        const uint32_t* q_off, const uint32_t* q_len,
                        const uint32_t* t_off, const uint32_t* t_len, int mode,
                        const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n,
                        int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                        uint8_t* ops, const uint64_t* ops_off, uint64_t ops_bytes,
                        uint32_t* ops_len, uint32_t* status, uint32_t max_slice);
int dgpu_edit_path_wide_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* q_off, const uint32_t* q_len,
                            const uint32_t* t_off, const uint32_t* t_len, int mode,
                            const uint8_t* eq_pairs, uint32_t n_eq, uint64_t n,
                            int32_t* dist, int32_t* start_loc, int32_t* end_loc,
                            uint8_t* ops, const uint64_t* ops_off,
                            uint32_t* ops_len, uint32_t* status, uint32_t max_slice, void* stream);

/* ---- consensus vs SV-reference split alignment (replaces longNeedle) --------------------
 * Call sites: _consRefAlignment for svt != 4, src/split.h:555 (reached from alignConsensus,
 * src/shortpe.h:186,253, src/assemble.h:849,859,916,926) and _generateProbes, src/coverage.h:214.
 * Implements longNeedle(cons, svRef, align, AlignConfig<true,false>, DnaScore(1,-1,-1,-1)),
 * src/needle.h:45-222, bit-for-bit (DP, forward/reverse score check, best-join tie rules,
 * traceback priority, stitched alignment).
 *
 * Job i aligns consensus seqs[c_off[i]..+c_len[i]) (rows) against the SV reference window
 * seqs[r_off[i]..+r_len[i]) (columns). Outputs per job:
 *   ok[i]       1 = longNeedle returned true; 0 = false (scores disagree / no split found)
 *   aln_len[i]  alignment columns L (0 when ok == 0)
 *   aln         row 0 (consensus) at aln + aln_off[i], row 1 (reference) at aln + aln_off[i] +
 *               (c_len[i] + r_len[i]); the caller reserves 2*(c_len+r_len) bytes per job.
 *   info        optional [consLeft, refLeft, refRight, bestScore] per job (white-box tests)
 * Limits of dgpu_long_needle / dgpu_long_needle_dev: r_len <= 16377 and c_len + r_len <= 32000 (the wavefront kernels' shapes). A job
 * beyond them is refused alone: ok = 0, aln_len = 0, info[2] = -1, dgpu_unsupported_count + 1; the call succeeds.
 */
int dgpu_long_needle(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                     const uint32_t* c_off, const uint32_t* c_len,
                     const uint32_t* r_off, const uint32_t* r_len, uint64_t n,
                     uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes,
                     uint32_t* aln_len, uint8_t* ok, int32_t* info);
int dgpu_long_needle_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                         const uint32_t* c_off, const uint32_t* c_len,
                         const uint32_t* r_off, const uint32_t* r_len, uint64_t n,
                         uint8_t* aln, const uint64_t* aln_off,
                         uint32_t* aln_len, uint8_t* ok, int32_t* info, void* stream);
/* The _ex forms take max_ref, the widest reference window the caller wants computed (1 .. DGPU_LN_MAX_REF, else DGPU_ERR_ARG).
 * Jobs inside the wavefront kernels' shapes run exactly as in dgpu_long_needle; jobs beyond them with r_len <= max_ref and
 * c_len <= 16383 run on the wide-window engine (one CTA per job computing whole DP rows, ~3 B of workspace per cell). Any other job,
 * and a job whose workspace alone exceeds half of the device budget (0.6 x free memory), is refused alone as above.
 * Caps: c_len <= 16383 because the wide engine keeps row-shifted scores U = H + r in [0, 2 c_len] as int16; DGPU_LN_MAX_REF because it
 * keeps the previous DP row (int16) and both sequences of a job in shared memory, about 213 KB at 65535 columns (227 KB per CTA on sm_90). */
#define DGPU_LN_MAX_REF 65535
int dgpu_long_needle_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                        const uint32_t* c_off, const uint32_t* c_len,
                        const uint32_t* r_off, const uint32_t* r_len, uint64_t n,
                        uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes,
                        uint32_t* aln_len, uint8_t* ok, int32_t* info, uint32_t max_ref);
int dgpu_long_needle_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                            const uint32_t* c_off, const uint32_t* c_len,
                            const uint32_t* r_off, const uint32_t* r_len, uint64_t n,
                            uint8_t* aln, const uint64_t* aln_off,
                            uint32_t* aln_len, uint8_t* ok, int32_t* info, uint32_t max_ref, void* stream);

/* ---- per-cluster MSA + consensus (replaces msa) -----------------------------------------
 * Call sites: msa(c, seqStore[svid], consensus), src/shortpe.h:185 and :252 (one call per SV
 * inside the thread-pool workers of assembleSplitReads). Implements src/msa.h:185-239 bit-for-bit:
 * LCS similarity matrix, UPGMA guide tree, progressive end-gap-free affine gotoh() on column
 * profiles (src/gotoh.h:71-174, src/align.h:96-171) and the coverage-thresholded consensus vote.
 *
 * Cluster i consists of reads cluster_off[i] .. cluster_off[i+1]-1 (indices into read_off/read_len),
 * IN THE ORDER THE REFERENCE ITERATES ITS std::unordered_set (the caller preserves that order).
 * Outputs per cluster: consensus bytes at cons + cons_off[i] (reserve sum of the cluster's read
 * lengths), cons_len[i], n_rows[i] (= msa()'s return value), status[i]:
 *   0 ok; 1 more than max_reads reads (32 for dgpu_msa / dgpu_msa_dev); 2 a read is empty or a read or an intermediate alignment
 *   exceeds 1023 columns; 3 a read contains a byte outside ACGTN (the reference's float profile is
 *   NaN there) — such clusters are NOT computed and the caller must treat them as errors.
 * Optional white-box output: the root alignment (n_rows x aln_cols, row-major) at aln + aln_off[i].
 * Scoring: (match, mismatch, go, ge) = DnaScore, e.g. (5,-4,-10,-1); requires go <= 0 and ge <= 0.
 */
int dgpu_msa(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
             const uint32_t* read_off, const uint32_t* read_len, uint32_t nreads,
             const uint32_t* cluster_off, uint32_t nclusters,
             int match, int mismatch, int go, int ge, int min_clique,
             uint8_t* cons, const uint64_t* cons_off, uint64_t cons_bytes,
             uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
             uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_cols);
int dgpu_msa_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                 const uint32_t* read_off, const uint32_t* read_len,
                 const uint32_t* cluster_off, uint32_t nclusters,
                 int match, int mismatch, int go, int ge, int min_clique,
                 uint8_t* cons, const uint64_t* cons_off,
                 uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
                 uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_cols, void* stream);
/* The _ex forms take max_reads, the largest cluster the caller wants computed (1 .. DGPU_MSA_LARGE_MAXR, else DGPU_ERR_ARG):
 * clusters of up to 32 reads run one warp each, clusters of 33 .. max_reads one CTA each, larger ones get status 1. max_reads
 * also sizes the large-cluster workspace (none when it is <= 32; about 17 MB per SM at 1023), so the device form needs no
 * readback. dgpu_msa / dgpu_msa_dev are the _ex forms with max_reads = 32. */
#define DGPU_MSA_LARGE_MAXR 1023
int dgpu_msa_ex(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                const uint32_t* read_off, const uint32_t* read_len, uint32_t nreads,
                const uint32_t* cluster_off, uint32_t nclusters,
                int match, int mismatch, int go, int ge, int min_clique,
                uint8_t* cons, const uint64_t* cons_off, uint64_t cons_bytes,
                uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
                uint8_t* aln, const uint64_t* aln_off, uint64_t aln_bytes, uint32_t* aln_cols, uint32_t max_reads);
int dgpu_msa_ex_dev(dgpu_ctx* ctx, const uint8_t* seqs, uint64_t seqs_bytes,
                    const uint32_t* read_off, const uint32_t* read_len,
                    const uint32_t* cluster_off, uint32_t nclusters,
                    int match, int mismatch, int go, int ge, int min_clique,
                    uint8_t* cons, const uint64_t* cons_off,
                    uint32_t* cons_len, uint32_t* n_rows, uint32_t* status,
                    uint8_t* aln, const uint64_t* aln_off, uint32_t* aln_cols, uint32_t max_reads, void* stream);

/* ---- clustering graphs: candidate edges ------------------------------------------
 * Replaces the windowed pair scans inside cluster() — src/cluster.h:371-431 (SRBamRecord) and :551-623
 * (BamAlignRecord): which pairs (i, j > i) of the SORTED records connect, and the edge weight. Records are passed
 * column-wise (int32). edge_off[n+1] receives the CSR offsets (edges of record i at edge_off[i] .. edge_off[i+1],
 * in increasing j — the order the reference's double loop meets them), edge_j / edge_w the targets and weights.
 * *n_edges = total number of edges; if it exceeds edge_cap the call fills nothing beyond edge_cap and returns
 * DGPU_ERR_CAPACITY (call again with larger arrays; edge_cap = 0 just counts). The component bookkeeping,
 * graphPruning and clique growth that consume the edges are sequential and stay with the caller
 * (delly_b200/host/cluster.hpp: clusterGpu).
 *   SR: chr, pos, chr2, pos2, inslen of SRBamRecord (src/tags.h:62-80), svt 0..8, max_read_sep = c.maxReadSep.
 *   PE: pos, mpos, mtid, alen, Median, maxNormalISize of BamAlignRecord (src/cluster.h:24-50), svt 0..3 / 5..8,
 *       varisize as passed to cluster() (src/shortpe.h:512-515). */
int dgpu_cluster_edges_sr(dgpu_ctx* ctx, const int32_t* chr, const int32_t* pos, const int32_t* chr2, const int32_t* pos2,
                          const int32_t* inslen, uint64_t n, int svt, uint32_t max_read_sep,
                          uint32_t* edge_off, uint32_t* edge_j, uint32_t* edge_w, uint64_t edge_cap, uint64_t* n_edges);
int dgpu_cluster_edges_pe(dgpu_ctx* ctx, const int32_t* pos, const int32_t* mpos, const int32_t* mtid, const int32_t* alen,
                          const int32_t* median, const int32_t* max_normal_isize, uint64_t n, int svt, uint32_t varisize,
                          uint32_t* edge_off, uint32_t* edge_j, uint32_t* edge_w, uint64_t edge_cap, uint64_t* n_edges);

/* ---- multi-GPU: the one exchange step ----------------------------------------------
 * The reference is one process: it builds the SV list, sorts and renumbers it (src/delly.h:155-158, src/tegua.h:149-156) and writes
 * the BCF. Sharded over GPUs (one process per GPU; contiguous ranges of the sorted SV list per rank, delly_b200/host/gather.hpp) every
 * rank finishes the records of its own range; this is the exchange that brings them together before emission: an all-gatherv of one
 * serialised byte string per rank over NCCL (ncclAllGather of the byte counts, then a grouped ncclBroadcast of exactly each payload).
 *   dgpu_comm_unique_id / dgpu_comm_init / dgpu_comm_destroy  thin wrappers of ncclGetUniqueId / ncclCommInitRank / ncclCommDestroy
 *       for callers that have no communicator yet (rank 0 creates the 128-byte id and hands it to the other ranks out of band). NCCL is
 *       bound at run time (dlopen libnccl.so.2): without it these calls return DGPU_ERR_NCCL and the rest of the library is unaffected.
 *   dgpu_gather_records  local / local_bytes = this rank's payload (host memory); *all = the payloads of ranks 0..n-1 back to back and
 *       *counts = their n sizes, both malloc'd by the callee (release with dgpu_free_host); *nranks = n. comm == NULL: single process
 *       (the output is a copy of the input). Collective: every rank of `comm` must call it, with its own context. */
int dgpu_comm_unique_id(uint8_t* id128);
int dgpu_comm_init(dgpu_ctx* ctx, int nranks, int rank, const uint8_t* id128, void** comm);
int dgpu_comm_destroy(dgpu_ctx* ctx, void* comm);
int dgpu_nccl_version(void);   /* ncclGetVersion of the bound library, 0 if NCCL is not available */
int dgpu_gather_records(dgpu_ctx* ctx, void* comm /* ncclComm_t */, const void* local, uint64_t local_bytes, void** all, uint64_t** counts, int* nranks);
void dgpu_free_host(void* p);

#ifdef __cplusplus
}
#endif
#endif /* DGPU_H */
