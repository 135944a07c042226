/*
 * daachorse_b200.h -- C ABI of libdaachorse_b200.so
 *
 * An H100-native (sm_90a) double-array Aho-Corasick matcher that is a drop-in for the
 * scan path of the Rust crate daac-tools/daachorse 4.0.0.  The reference has no FFI of
 * its own: its boundary is the crate's public Rust API.  Each entry point below names the
 * reference item it replaces (file:line relative to the crate root) -- INTEGRATION.md
 * shows the `extern "C"` block and the thin Rust wrappers a crate maintainer would add.
 *
 * Conventions
 *   - every function returns a dach_status (0 = OK) unless documented otherwise;
 *   - handles are opaque, created/destroyed by the library; all data buffers are
 *     caller-owned; no torch / C++ types cross the boundary;
 *   - V (the pattern value type of the crate) is fixed to u32;
 *   - match positions are u32 byte offsets inside one haystack (haystacks <= 4 GiB - 1);
 *     per-haystack result ranges are u64 offsets into the match array;
 *   - there is NO CPU scan path in this library: scanning requires a CUDA device and
 *     fails with DACH_CUDA_ERROR otherwise.
 */
#ifndef DAACHORSE_B200_H
#define DAACHORSE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DACH_ABI_VERSION 2

/* Status codes.  1-4 mirror DaachorseError (src/errors.rs:10-22); 5 stands for the
 * `assert!(self.match_kind.is_standard())` / `is_leftmost()` panics of
 * src/bytewise.rs:194-197,299-302,551-554 and src/charwise.rs:188-191,297-300,557-560
 * (a Rust shim turns it back into a panic). */
typedef enum {
    DACH_OK = 0,
    DACH_INVALID_ARGUMENT = 1,
    DACH_AUTOMATON_SCALE = 2,
    DACH_INVALID_CONVERSION = 3,
    DACH_INVALID_AUTOMATON = 4,
    DACH_MATCH_KIND_MISMATCH = 5,
    DACH_OUTPUT_OVERFLOW = 6, /* out_cap too small; *needed holds the required capacity */
    DACH_CUDA_ERROR = 7
} dach_status;

/* MatchKind, #[repr(u8)] (src/lib.rs:324-346) */
typedef enum {
    DACH_STANDARD = 0,
    DACH_LEFTMOST_LONGEST = 1,
    DACH_LEFTMOST_FIRST = 2
} dach_match_kind;

/* Which iterator of the crate a batch scan reproduces. */
typedef enum {
    DACH_FIND = 0,                       /* find_iter                        src/bytewise.rs:190, src/charwise.rs:184 */
    DACH_FIND_OVERLAPPING = 1,           /* find_overlapping_iter            src/bytewise.rs:292, src/charwise.rs:290 */
    DACH_FIND_OVERLAPPING_NO_SUFFIX = 2, /* find_overlapping_no_suffix_iter  src/bytewise.rs:410, src/charwise.rs:412 */
    DACH_LEFTMOST_FIND = 3               /* leftmost_find_iter               src/bytewise.rs:547, src/charwise.rs:553 */
} dach_scan_mode;

/* One reported match: Match<u32>{length,end,value} seen through start()/end()/value()
 * (src/lib.rs:287-320); start = end - length. */
typedef struct {
    uint32_t start;
    uint32_t end;
    uint32_t value;
} dach_match;

typedef struct dach_pma dach_pma; /* host-side automaton  (DoubleArrayAhoCorasick / Charwise...) */
typedef struct dach_dev dach_dev; /* device-resident scan image of one automaton            */

/* ---- construction (host) --------------------------------------------------------- */

/* DoubleArrayAhoCorasickBuilder::new().match_kind(k).num_free_blocks(n).build_with_values()
 * (src/bytewise/builder.rs:57,90,112,152,204); DoubleArrayAhoCorasick::new / with_values
 * (src/bytewise.rs:103,145) are the match_kind = Standard, num_free_blocks = 16 case.
 * Patterns: one byte blob + n+1 offsets.  values == NULL associates value i with pattern i.
 * num_free_blocks == 0 -> DACH_INVALID_ARGUMENT (the crate panics, builder.rs:113). */
int dach_bytewise_build(const uint8_t *pattern_bytes, const uint64_t *pattern_offs,
                        const uint32_t *values, uint32_t n_patterns, uint8_t match_kind,
                        uint32_t num_free_blocks, dach_pma **out);

/* CharwiseDoubleArrayAhoCorasickBuilder (src/charwise/builder.rs:55,71,89,129,178);
 * CharwiseDoubleArrayAhoCorasick::new / with_values (src/charwise.rs:100,139).
 * Patterns must be valid UTF-8 (the crate takes &str); invalid UTF-8 ->
 * DACH_INVALID_ARGUMENT. */
int dach_charwise_build(const uint8_t *pattern_bytes, const uint64_t *pattern_offs,
                        const uint32_t *values, uint32_t n_patterns, uint8_t match_kind,
                        uint32_t num_free_blocks, dach_pma **out);

/* deserialize (src/bytewise.rs:868-964, src/charwise.rs:896-952): parses the crate's own
 * wire format, runs the same validation, rebuilds root_table.  *consumed receives the
 * number of bytes read (the crate returns the remaining slice).  This is the hand-off a
 * Rust caller uses: pma.serialize() -> dach_pma_deserialize -> dach_dev_upload.
 * deserialize_unchecked (src/bytewise.rs:1009, src/charwise.rs:997) maps to this same
 * checked entry point: device loads are unchecked too, so validation is mandatory. */
int dach_pma_deserialize(const uint8_t *src, size_t len, int charwise, dach_pma **out,
                         size_t *consumed);

/* serialize (src/bytewise.rs:801-820, src/charwise.rs:831-848): byte-identical to the
 * crate's output.  dach_pma_serialized_bytes gives the exact size. */
size_t dach_pma_serialized_bytes(const dach_pma *pma);
int dach_pma_serialize(const dach_pma *pma, uint8_t *dst, size_t cap, size_t *written);

/* match_kind (src/bytewise.rs:747, src/charwise.rs:762), num_states (:785 / :779),
 * heap_bytes (:764 / :813), num_elements (src/charwise.rs:796; double-array length for
 * both variants). */
uint8_t dach_pma_match_kind(const dach_pma *pma);
uint32_t dach_pma_num_states(const dach_pma *pma);
size_t dach_pma_heap_bytes(const dach_pma *pma);
size_t dach_pma_num_elements(const dach_pma *pma);
int dach_pma_is_charwise(const dach_pma *pma);
uint32_t dach_pma_max_pattern_len(const dach_pma *pma); /* longest pattern in bytes */
/* The output records (src/nfa_builder.rs:203-222): one per pattern the builder kept -- duplicates get
 * a record each; LeftmostFirst drops patterns that extend a shorter one.  dach_pma_outputs copies
 * record i's value, length (bytes) and parent (0 = none, else the parent's 1-based index; a parent
 * comes before its child) to values[i] / lengths[i] / parents[i]; any array may be NULL.
 * n < dach_pma_num_outputs -> DACH_INVALID_ARGUMENT.  These label DACH_KEY_OUTPUT histograms. */
uint32_t dach_pma_num_outputs(const dach_pma *pma);
int dach_pma_outputs(const dach_pma *pma, uint32_t *values, uint32_t *lengths, uint32_t *parents,
                     uint32_t n);
void dach_pma_free(dach_pma *pma);

/* ---- device image ---------------------------------------------------------------- */

/* Builds the scan image of `pma` (records repacked for the kernels, root table, mapper,
 * outputs) and uploads it once to CUDA device `device`. */
int dach_dev_upload(const dach_pma *pma, int device, dach_dev **out);
void dach_dev_free(dach_dev *dev);
size_t dach_dev_image_bytes(const dach_dev *dev); /* bytes resident in HBM for the automaton */

/* ---- batch scan (the hot path) ---------------------------------------------------- */

/* Scans n haystacks that are ALREADY RESIDENT on the device and writes, for haystack i,
 * exactly the matches the crate's iterator `mode` yields on it, in the same order, to
 * d_out[d_out_offs[i] .. d_out_offs[i+1]).
 *
 *   d_text      device pointer, the haystack bytes back to back
 *   d_offs      device pointer, n+1 u64 byte offsets into d_text (ascending)
 *   text_bytes  total byte length of d_text (== offs[n]); the kernel never reads past it
 *   d_out       device pointer, capacity out_cap matches
 *   d_out_offs  device pointer, n+1 u64
 *   needed      host pointer; receives the total number of matches (exact, also past 2^32)
 *   stream      cudaStream_t (NULL = default stream); the call synchronises the stream
 *               before returning
 *
 * Returns DACH_OUTPUT_OVERFLOW (and *needed) when out_cap is too small; nothing useful is
 * in d_out then, and nothing at or past d_out + out_cap is written.  A haystack that yields
 * 2^32 or more matches cannot be placed (per-haystack match indices are u32): the call
 * returns DACH_INVALID_ARGUMENT with the exact *needed and writes no match; count such
 * batches with dach_dev_count_batch / dach_dev_hist_batch.  Stream chunks, the host form and
 * jobs behave the same.  DACH_MATCH_KIND_MISMATCH mirrors the crate's panics.  Charwise
 * haystacks must be valid UTF-8 (as &str guarantees in the crate). */
int dach_dev_scan_batch(dach_dev *dev, int mode, const uint8_t *d_text, const uint64_t *d_offs,
                        uint64_t n, uint64_t text_bytes, dach_match *d_out, uint64_t out_cap,
                        uint64_t *d_out_offs, uint64_t *needed, void *stream);

/* Same contract with HOST buffers (pageable or pinned): copies text/offsets to the
 * device in slices overlapped with scanning, copies matches and offsets back.  This is
 * the call the crate-facing wrappers use and the one bench.py times as `e2e`. */
int dach_scan_batch_host(dach_dev *dev, int mode, const uint8_t *text, const uint64_t *offs,
                         uint64_t n, dach_match *out, uint64_t out_cap, uint64_t *out_offs,
                         uint64_t *needed);

/* Chunks of streams -- the batch form of the crate's steppers (FindStepper /
 * FindOverlappingStepper, src/bytewise/iter.rs:344-475, constructors src/bytewise.rs:627-729;
 * charwise: src/charwise/iter.rs:403-534, constructors src/charwise.rs:638,734): haystack i is
 * the next chunk of stream i.  Standard automata; mode is DACH_FIND or DACH_FIND_OVERLAPPING.
 * A chunk of a charwise stream holds whole chars (the charwise steppers consume chars).
 *   d_state  device pointer, n u32, in/out: the stepper's state_id.  In: the state the
 *            previous chunk of the stream ended in (0 = ROOT for a new stream).  Out: the
 *            state after the chunk's last byte.  State ids are the crate's (the bytewise device
 *            image is renumbered hot-first; ids are translated at the boundary), so chunks may
 *            alternate between this library and the crate's own steppers.
 *   d_pos    device pointer, n u32, or NULL: the stepper's pos at the chunk's first byte;
 *            it is added to start and end of the chunk's matches (stream coordinates,
 *            modulo 2^32).  NULL = positions relative to the chunk.
 * What is reported: for every byte (char) of the chunk, consume() followed by matches() -- the
 * matches() of the incoming state belong to the previous chunk and are not repeated.  All
 * other arguments, the output layout and the return codes are those of dach_dev_scan_batch;
 * on DACH_OUTPUT_OVERFLOW d_state has been advanced already (keep a copy to retry).
 * DACH_INVALID_ARGUMENT where no Standard lane machine applies (more than 2^24 states; bytewise:
 * a ROOT without children; DACH_FIND with an empty pattern in the set). */
int dach_dev_scan_stream(dach_dev *dev, int mode, const uint8_t *d_text, const uint64_t *d_offs,
                         uint64_t n, uint64_t text_bytes, uint32_t *d_state, const uint32_t *d_pos,
                         dach_match *d_out, uint64_t out_cap, uint64_t *d_out_offs,
                         uint64_t *needed, void *stream);

/* ---- counts and first matches ----------------------------------------------------------------
 *
 * Two questions that need no match list.  Same batch layout, modes, d_offs checks and errors as
 * dach_dev_scan_batch (DACH_INVALID_ARGUMENT for bad offsets, DACH_MATCH_KIND_MISMATCH, DACH_CUDA_ERROR
 * without a device), but no capacity: there is no DACH_OUTPUT_OVERFLOW.  The calls synchronise `stream`.
 *
 *   count  d_counts[i] (u64) = the number of matches iterator `mode` yields on haystack i, i.e. exactly
 *          out_offs[i+1] - out_offs[i] of dach_dev_scan_batch; *total = their sum.  u64 because
 *          overlapping lists make more than 2^32 matches on one haystack reachable.
 *   first  d_first[i] = the first match iterator `mode` yields on haystack i (`iter.next()`), d_found[i] = 1
 *          if there is one; otherwise d_found[i] = 0 and d_first[i] = {0xffffffff x 3}.  *n_found = the
 *          haystacks with a match.  The scan of a haystack stops at its first match.  For Standard automata
 *          the three Standard modes have the same first match (the head of the first output list reached,
 *          ROOT's empty pattern at position 0 included).
 *
 * The host forms copy text and offsets to the device in the slices of dach_scan_batch_host; only the
 * per-haystack results come back (8 B, or 13 B, per haystack; dach_dev_last_h2d_bytes / _d2h_bytes).
 * Option kernel = 1, 2 or 4 runs the default lane machines here (kernel = 3); kernel = 0 the lane-per-haystack
 * kernels.  Stream chunks, jobs and shard groups have no count / first form. */
int dach_dev_count_batch(dach_dev *dev, int mode, const uint8_t *d_text, const uint64_t *d_offs, uint64_t n,
                         uint64_t text_bytes, uint64_t *d_counts, uint64_t *total, void *stream);
int dach_count_batch_host(dach_dev *dev, int mode, const uint8_t *text, const uint64_t *offs, uint64_t n,
                          uint64_t *counts, uint64_t *total);
int dach_dev_first_batch(dach_dev *dev, int mode, const uint8_t *d_text, const uint64_t *d_offs, uint64_t n,
                         uint64_t text_bytes, dach_match *d_first, uint8_t *d_found, uint64_t *n_found, void *stream);
int dach_first_batch_host(dach_dev *dev, int mode, const uint8_t *text, const uint64_t *offs, uint64_t n,
                          dach_match *first, uint8_t *found, uint64_t *n_found);

/* ---- per-pattern occurrence counts ------------------------------------------------------------
 *
 * How often each pattern occurs in a batch, with no match list: hist[k] += the number of matches
 * iterator `mode` yields over all n haystacks whose key is k.
 *   DACH_KEY_OUTPUT  k = the index of the match's output record (dach_pma_outputs); n_hist must be at
 *                    least dach_pma_num_outputs.
 *   DACH_KEY_VALUE   k = the match's value: exactly a bincount of the values of dach_dev_scan_batch.
 *                    n_hist must exceed the largest value.  For automata made by `new` the value is the
 *                    pattern index.
 * The counts are ADDED into the caller's zeroed (or earlier) histogram, so calls on batches A and B
 * leave what one call on A ++ B would: a corpus accumulates on the device across batches (and across
 * GPUs with an ordinary all-reduce).  *total = the matches added (== the dach_dev_count_batch total).
 * A too-small n_hist or an unknown key is DACH_INVALID_ARGUMENT before anything runs; offsets, modes
 * and the missing device as dach_dev_count_batch.  The calls synchronise `stream`.
 * The host form uses the slices of dach_scan_batch_host, adds them up on the device and copies
 * n_hist x 8 bytes back once (dach_dev_last_d2h_bytes).  Option hist_smem (default 1024; 0 = off):
 * events of the leading compact states are counted in shared memory per CTA first.  Options kernel and
 * the fallbacks as dach_dev_count_batch.  Stream chunks, jobs and shard groups have no histogram form. */
typedef enum {
    DACH_KEY_OUTPUT = 0,
    DACH_KEY_VALUE = 1
} dach_hist_key;
int dach_dev_hist_batch(dach_dev *dev, int mode, int key, const uint8_t *d_text, const uint64_t *d_offs,
                        uint64_t n, uint64_t text_bytes, uint64_t *d_hist, uint64_t n_hist, uint64_t *total,
                        void *stream);
int dach_hist_batch_host(dach_dev *dev, int mode, int key, const uint8_t *text, const uint64_t *offs,
                         uint64_t n, uint64_t *hist, uint64_t n_hist, uint64_t *total);

/* ---- asynchronous scans (jobs) ----------------------------------------------------------
 *
 * dach_dev_scan_batch is one call that synchronises its stream and serialises per handle.  A job is
 * the same pipeline cut in two phases that only ENQUEUE work, with a workspace of its own, so that
 * host threads, streams and GPUs overlap (the crate's iterators are `&self`: any number of scans run
 * concurrently on one automaton -- src/bytewise.rs:190-197 takes `&self`).
 *   dach_job_scan   enqueues items + scan kernel + offsets on `stream`; returns at once.
 *                   cap_matches sizes the staging pool (as out_cap does in dach_dev_scan_batch).
 *   dach_job_place  enqueues the gather on `stream` (may differ from the scan's stream; ordered by an
 *                   event): matches -> d_out + *d_base, offsets (+ *d_base) -> d_out_offs[0..n].
 *                   d_base is a DEVICE pointer to the index of this batch's first match in d_out, or
 *                   NULL for 0; d_out / d_out_offs may be peer-mapped memory of another GPU.
 *   dach_job_wait   blocks until the placement is done; status and *needed as dach_dev_scan_batch.
 * A job holds one scan at a time: scan -> place -> (wait) -> scan ...; the next dach_job_scan is
 * ordered after the previous placement by the library.  Options are read from the dach_dev.
 * A job keeps its dach_dev alive: dach_dev_free may come first (as a garbage collector may order
 * it); the device image is then released by the last dach_job_free of that device. */
typedef struct dach_job dach_job;
int dach_job_create(dach_dev *dev, dach_job **out);
void dach_job_free(dach_job *job);
int dach_job_scan(dach_job *job, int mode, const uint8_t *d_text, const uint64_t *d_offs, uint64_t n,
                  uint64_t text_bytes, uint64_t cap_matches, void *stream);
int dach_job_place(dach_job *job, dach_match *d_out, uint64_t out_cap, uint64_t *d_out_offs,
                   const uint64_t *d_base, void *stream);
int dach_job_wait(dach_job *job, uint64_t *needed);
double dach_job_scan_kernel_ms(const dach_job *job); /* CUDA-event time of the job's last scan kernel */
double dach_job_push_ms(const dach_job *job);        /* ... of its last peer push (dach_group_place), 0 if none */
/* ms since the handle's first dach_job_scan of {scan kernel start, scan kernel end, peer push start, peer push end}
 * of the job's last step: the timeline of a pipelined run (bench.py config.timeline) */
int dach_job_times(const dach_job *job, double out[4]);

/* ---- shard groups: the exchange step of a batch sharded over the GPUs of one node ---------
 *
 * Haystacks are independent, so a batch shards with no data-path collective; the one exchange is
 * the gather of the per-shard match buffers to rank 0 (north_star).  Here that gather is not a
 * separate collective: every rank's placement kernel stores its matches straight into rank 0's
 * dense result buffer over NVLink peer memory, at the base it learns from the lower ranks' counts
 * (published into every rank's control block with system-scope releases, polled locally).  Rank 0
 * ends a step holding exactly what one GPU would have produced for the concatenated batch:
 * matches dense and in shard order, n_total + 1 rebased offsets.
 *
 *   create   every rank: control block; rank 0 also the result buffers (match_cap matches,
 *            n_haystacks_total + 1 offsets).
 *   export / connect   DACH_GROUP_HANDLE_BYTES per rank, exchanged by the caller (any transport:
 *            torch.distributed, MPI, a pipe), passed in rank order.  Ranks may be processes (CUDA IPC)
 *            or handles inside one process (peer access).
 *   place    the exchange step of one job: hay_base = index of the shard's first haystack in the
 *            whole batch, last = this shard ends the batch (it also writes offsets[n_total]).
 *            Calling place for step s releases the result of step s-1 (rank 0).  On ranks other
 *            than 0 the call BLOCKS until the rank's host knows where its matches go -- its own scan
 *            is done, the lower ranks have published their counts, rank 0 has released the previous
 *            result -- because the packed tuples then leave through a copy engine (no SM, LSU slot or
 *            L1 line is taken from the scan running beside the exchange).  Pipelining callers enqueue
 *            the next dach_job_scan before they call place; one thread driving several ranks places
 *            them in rank order.  (Environment DACH_GROUP_PUSH=sm keeps everything on the device:
 *            k_push, destination-aligned 16-byte peer stores, no host round trip.)
 *   finish   rank 0: enqueues the wait for all ranks on `stream`, synchronises it, reports the total
 *            (DACH_OUTPUT_OVERFLOW if it exceeds match_cap); other ranks: synchronise `stream`.
 *   result   rank 0's device pointers. */
#define DACH_GROUP_HANDLE_BYTES 256
typedef struct dach_group dach_group;
int dach_group_create(int rank, int world, int device, uint64_t match_cap, uint64_t n_haystacks_total,
                      dach_group **out);
int dach_group_export(const dach_group *group, void *handle);
int dach_group_connect(dach_group *group, const void *handles);
int dach_group_place(dach_group *group, dach_job *job, uint64_t hay_base, int last, void *stream);
int dach_group_finish(dach_group *group, uint64_t *total, void *stream);
int dach_group_result(const dach_group *group, dach_match **d_out, uint64_t **d_offs);
void dach_group_free(dach_group *group);

/* ---- introspection for the bench / tests ------------------------------------------ */

/* Number of kernels this handle has launched so far (bench.py's gpu_launches). */
uint64_t dach_dev_kernel_launches(const dach_dev *dev);
/* Device time (ms, CUDA events on the launch stream) of the scan kernel alone and of the
 * whole device-side pipeline in the most recent dach_dev_scan_batch call. */
double dach_dev_last_scan_kernel_ms(const dach_dev *dev);
double dach_dev_last_total_ms(const dach_dev *dev);
/* Bytes moved host<->device by the most recent dach_scan_batch_host call. */
uint64_t dach_dev_last_h2d_bytes(const dach_dev *dev);
uint64_t dach_dev_last_d2h_bytes(const dach_dev *dev);
/* Tuning knobs: kernel (3 = StdMachine3, the default; 2, 1 = its predecessors; 0 = lane per haystack),
 * hot_entries (records of the hot region staged in shared memory, default 6144), threads, ctas_per_sm, seg_len
 * (segment length for intra-haystack chunking of find_overlapping), l2_hints, slice_mib, ... */
int dach_dev_set_option(dach_dev *dev, const char *name, int64_t value);

/* Human-readable text of the last error on this thread ("" if none). */
const char *dach_last_error(void);
int dach_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DAACHORSE_B200_H */
