/*
 * acb200.h -- C ABI of the H100-native multi-pattern matcher (libacb200.so).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference
 * (G-Research/ahocorasick_rs) has no C ABI of its own: its PyO3 shim
 * (src/lib.rs) calls straight into the Rust crate `aho-corasick` 1.1.4.  Each
 * entry point below names the reference call site it stands in for; a
 * maintainer of the reference would bind these from src/lib.rs through
 * `extern "C"` (see INTEGRATION.md) or, as this repo does, from Python with
 * ctypes (ahocorasick_rs_b200/_capi.py).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *   - every function returns ACB_OK (0) or a negative ACB_E* code; text for the
 *     last error on the calling thread comes from acb_last_error();
 *   - "dev_" pointers are CUDA device pointers on the current device; the
 *     library never allocates device memory: the caller (PyTorch's caching
 *     allocator in this repo) owns every buffer and says how big it is;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it
 *     and nothing synchronises unless stated;
 *   - there is no CPU fallback: scan entry points fail with ACB_ECUDA when no
 *     device is usable.
 */
#ifndef ACB200_H
#define ACB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACB_OK 0
#define ACB_EINVAL (-1)      /* bad argument */
#define ACB_EBUILD (-2)      /* automaton construction failed (reference: BuildError -> ValueError, src/lib.rs:215,406) */
#define ACB_EUNSUPPORTED (-3) /* overlapping search on a non-Standard automaton (reference: MatchError -> ValueError, src/lib.rs:36-39,52-54) */
#define ACB_ECUDA (-4)       /* CUDA runtime error / no device */
#define ACB_ECAPACITY (-5)   /* a caller-provided buffer is too small */

/* MatchKind (reference: src/lib.rs:92-98) */
#define ACB_STANDARD 0
#define ACB_LEFTMOST_FIRST 1
#define ACB_LEFTMOST_LONGEST 2

/* Implementation (reference: src/lib.rs:111-118). -1 = None (heuristic).
 * Here it selects the device table layout only; results never depend on it. */
#define ACB_IMPL_AUTO (-1)
#define ACB_IMPL_NONCONTIGUOUS_NFA 0
#define ACB_IMPL_CONTIGUOUS_NFA 1
#define ACB_IMPL_DFA 2

typedef struct acb_automaton acb_automaton;

/* One match, as the reference's (pattern, start, end) tuple (src/lib.rs:240-246,
 * 431) plus the haystack it belongs to.  16 bytes, written with one store. */
typedef struct acb_match {
    uint32_t haystack; /* index into the batch (0 for single-haystack calls) */
    uint32_t pattern;  /* index into the pattern list given to acb_build */
    uint32_t start;    /* byte offset, or code point index when codepoints != 0 */
    uint32_t end;      /* exclusive */
} acb_match;

const char *acb_last_error(void);
const char *acb_version(void);

/*
 * Build an automaton on the host.
 * Stands in for AhoCorasickBuilder::new().kind(..).match_kind(..).build(..)
 * at src/lib.rs:186-215 (str) and 401-406 (bytes).
 * Pattern i is blob[offsets[i] .. offsets[i+1]); ids are input order.  Empty
 * patterns are an error here too (the reference rejects them before the crate
 * sees them, src/lib.rs:204-207,386-389).
 */
int acb_build(const uint8_t *blob, const uint64_t *offsets, uint64_t n_patterns, int match_kind,
              int implementation, acb_automaton **out);
void acb_free(acb_automaton *a);

/* Facts about a built automaton. */
uint64_t acb_num_patterns(const acb_automaton *a);
uint64_t acb_num_states(const acb_automaton *a);
uint32_t acb_num_columns(const acb_automaton *a);
uint32_t acb_max_pattern_len(const acb_automaton *a);
uint32_t acb_min_pattern_len(const acb_automaton *a);
int acb_match_kind(const acb_automaton *a);

/*
 * The device image: the flat tables the kernels read (column map, dense
 * transition rows, per-state match lists, pattern lengths), serialised into
 * one buffer.  The caller allocates acb_image_bytes() on the device, fills it
 * from acb_image_write()'s host copy ("table uploaded once to HBM"), and
 * passes it to every scan.
 */
uint64_t acb_image_bytes(const acb_automaton *a);
int acb_image_write(const acb_automaton *a, void *host_dst, uint64_t dst_bytes);

/*
 * The hot image: the rows of the table the staged kernel keeps in shared memory,
 * hottest first.  "Hot" is decided from data: acb_profile() walks a sample of a
 * device-resident input through the automaton and counts state visits into
 * dev_visits (u32[acb_num_states], zeroed by the call); the caller copies the
 * counts to the host and hands them to acb_hot_build() (host_visits == NULL:
 * no profile, shallowest states first), then uploads the result and passes it,
 * with its row count, to the scans.  Which rows are hot changes speed only --
 * everything the fast path cannot prove uneventful is redone by the exact
 * scanner -- never results.  dev_hot == NULL selects the plain kernel.
 */
int acb_profile(const acb_automaton *a, const void *dev_image, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                int64_t n_haystacks, uint64_t total_bytes, int overlapping, uint32_t *dev_visits, void *stream);
uint64_t acb_hot_bytes(const acb_automaton *a, uint32_t max_rows);
int acb_hot_build(const acb_automaton *a, const uint32_t *host_visits, uint32_t max_rows, void *host_dst,
                  uint64_t dst_bytes);
uint32_t acb_hot_rows(const void *host_hot);

/* What a hot image holds (read from its host copy; passed along with the device copy). */
typedef struct acb_hot_desc {
    uint32_t rows;     /* rows of the compact table (column-indexed) */
    uint32_t rows128;  /* rows of the byte-indexed 128-wide table (0: patterns use bytes >= 0x7f) */
    uint32_t visited;  /* rows the profile actually saw; the rest is filler */
    uint32_t reserved; /* flags set by the caller: bit 0 = the hot rows do not cover this data (dense automaton on
                          adversarial input): with tuning.kernel = 0 the scan then runs from the image in global
                          memory / L2 (kernel 4) instead of the shared-memory table */
} acb_hot_desc;
int acb_hot_describe(const void *host_hot, acb_hot_desc *desc);

/*
 * The sieve image: the position-parallel form of the matcher (csrc/sieve.h).  Instead of walking an automaton -- one
 * DEPENDENT table load per haystack byte -- every byte position is tested independently: the W bytes ending there are
 * hashed into a Bloom filter of the patterns' suffixes held in shared memory; survivors walk on through the filter's
 * deeper levels and are finally verified, exactly, against a reverse trie in global memory / L2, which names every
 * pattern ending at that position in the reference's order.  That is the overlapping match list
 * (try_find_overlapping_iter, src/lib.rs:52-54); the non-overlapping lists (try_find_iter, src/lib.rs:58-60) are
 * selected from it per haystack for all three match kinds.  This is the compact (non-DFA) table format: a few tens of
 * bytes per trie node instead of a dense row per state.
 * acb_sieve_build builds (or rebuilds, when the arguments change) the image on the host and returns its size (0 on
 * error): bloom_bytes_max = shared memory the filters may take when the scan keeps one 512-byte window of text per warp
 * on chip (the caller knows the device: shared memory per block minus 46 KB; the builder uses less for sparse pattern sets,
 * which leaves the scan a deeper ring of text), w_max = cap on the primary window in bytes (0 = automatic).  The caller uploads acb_sieve_write()'s copy and passes the device pointer to the
 * scans as dev_sieve (NULL = use the table kernels).
 */
uint64_t acb_sieve_build(acb_automaton *a, uint32_t bloom_bytes_max, uint32_t w_max);
int acb_sieve_write(acb_automaton *a, void *host_dst, uint64_t dst_bytes);
typedef struct acb_sieve_desc {
    uint32_t window;         /* W: bytes hashed per position by the fast path */
    uint32_t last_level;     /* longest suffix length held by the on-chip filter */
    uint32_t probes;         /* Bloom probes per key */
    uint32_t bloom_bytes;
    uint32_t nodes;          /* reverse-trie nodes (depth >= W) */
    uint32_t keys;           /* distinct W-byte suffixes = hash table entries */
    uint32_t filter_entries;
    uint32_t table_slots;
} acb_sieve_desc;
int acb_sieve_describe(const void *host_sieve, acb_sieve_desc *desc);

/*
 * How a scan is cut up.  The byte stream [offsets[0], offsets[n]) is divided into
 * fixed-size SEGMENTS on a grid anchored at the 64-byte aligned address at or
 * before dev_bytes; one GPU lane scans one segment, so the work per lane is the
 * same whatever the haystack lengths are (one huge haystack, a ragged batch, a
 * million short lines).  A segment that begins inside a haystack starts from a
 * speculated automaton state that is verified -- and, when wrong, repaired --
 * before results are delivered; see DESIGN.md.  The plan depends only on
 * host-known quantities: the automaton, the address of the byte buffer, its
 * length and the number of haystacks.
 */
typedef struct acb_plan {
    uint64_t n_segments;
    uint64_t n_units;       /* entries the unit arrays of the workspace need */
    uint64_t scratch_words; /* u64 words dev_scratch needs */
    uint32_t segment_bytes;
    uint32_t warm_bytes;    /* bytes scanned before a segment to guess its start state (>= longest pattern) */
    uint32_t lane_stride;   /* segments between neighbouring lanes of a warp */
    uint32_t task_bytes;    /* the sieve kernel's unit of work: bytes of the stream one warp walks (a multiple of 512) */
} acb_plan;

int acb_plan_scan(const acb_automaton *a, const void *dev_bytes, uint64_t total_bytes, uint64_t n_haystacks,
                  acb_plan *plan);

/* Caller-provided device workspace for one scan, sized from the plan. */
typedef struct acb_workspace {
    acb_match *dev_raw;      /* [raw_capacity] unordered matches as kernels emit them */
    uint32_t *dev_raw_seq;   /* [raw_capacity] rank of each raw match inside its unit */
    uint32_t *dev_raw_unit;  /* [raw_capacity] unit (segment slot / haystack) each raw match belongs to */
    uint32_t *dev_raw_aux;   /* [raw_capacity] code point bookkeeping per raw match */
    uint64_t raw_capacity;
    uint32_t *dev_unit_counts;   /* [plan.n_units] */
    uint64_t *dev_unit_offsets;  /* [plan.n_units + 1] */
    void *dev_seg_info;          /* [plan.n_segments * 32 bytes] per-segment summaries */
    uint64_t *dev_scratch;       /* [plan.scratch_words]; its first 8 words must be ZERO the first time a workspace is
                                    used: they hold the kernels' counters, and every completed scan leaves them zeroed
                                    again (so a scan needs no clearing launch in front of it) */
    uint64_t *dev_total;         /* [8]: [0] = matches found, [1] = 1 when dev_out holds all of them (0: buffers too
                                    small, retry), [2] = 16-byte groups in the stream, [3] = times a lane left the hot table
                                    for the exact scanner, [4] = raw matches emitted, [5] = segment boundaries repaired */
    acb_match *dev_out;          /* [out_capacity] final matches in the reference's order */
    uint64_t out_capacity;
    uint64_t *dev_match_offsets; /* [n_haystacks + 1] haystack h's matches are dev_out[off[h] .. off[h+1]) */
} acb_workspace;

/*
 * Scan a batch of haystacks resident in device memory:
 * haystack h = dev_bytes[dev_offsets[h] .. dev_offsets[h+1]); total_bytes =
 * length of the dev_bytes buffer (>= dev_offsets[n]).  One haystack of many
 * gigabytes is just n_haystacks = 1.
 *
 * Per haystack this is the drain of the reference's iterator: get_matches
 * (src/lib.rs:42-68) choosing try_find_iter (58-60) or
 * try_find_overlapping_iter (52-54), collected at 238-248 (str) / 433 (bytes).
 * codepoints != 0 reports start/end as code point indexes, i.e. it also does
 * the work of get_byte_to_code_point (src/lib.rs:73-88) for valid UTF-8.
 *
 * On return (after the stream has run): ws->dev_out holds
 * min(total, out_capacity) matches ordered by haystack and then in the
 * reference's iteration order; ws->dev_match_offsets brackets each haystack's
 * matches; ws->dev_total[0] is the true total.  If the matches did not fit
 * raw_capacity / out_capacity nothing is lost silently: dev_total[1] is 0 and
 * dev_total[0] / [4] say how much room a second call needs.
 * overlapping on a non-Standard automaton returns ACB_EUNSUPPORTED before any
 * byte is read, like the reference.  (overlapping = 2 asks for the overlapping LIST of any automaton -- the input of
 * acb_select_non_overlapping; it needs dev_sieve.)
 */
int acb_scan_batch(const acb_automaton *a, const void *dev_image, const void *dev_hot, const acb_hot_desc *hot_desc,
                   const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes,
                   int overlapping, int codepoints, const acb_plan *plan, const acb_workspace *ws, void *stream);

/*
 * One haystack too large for one call (more than 2^31 bytes), non-overlapping search: the caller scans it as an
 * OVERLAPPING search in windows (exact: the matches ending at a position depend on max_pattern_len - 1 bytes before it),
 * concatenates the lists -- rows of four int64 (haystack, pattern, start, end), in the reference's order -- and this call
 * selects from them what the reference's non-overlapping iterator (try_find_iter, src/lib.rs:58-60) reports for the
 * automaton's match kind: dev_out gets the selected rows, *dev_count their number.  dev_out needs room for n_rows rows.
 */
int acb_select_non_overlapping(const acb_automaton *a, const int64_t *dev_rows, uint64_t n_rows, int64_t *dev_out, uint64_t *dev_count,
                                void *stream);

/*
 * Which haystacks contain an occurrence of any pattern.  Stands in for the crate's AhoCorasick::is_match, once per
 * haystack of a device-resident batch (haystack h = dev_bytes[dev_offsets[h] .. dev_offsets[h+1]); total_bytes =
 * length of the dev_bytes buffer, below 2^31).  The answer does not depend on the match kind (a haystack has a
 * non-overlapping match of any kind iff some pattern occurs in it), so every automaton is accepted.  It needs the sieve
 * image (acb_sieve_build / acb_sieve_write) and runs the sieve kernel in its any-match mode: one launch, no match list,
 * no epilogue; the task size comes from acb_plan_scan (acb_tuning.segment_bytes applies when tuning.kernel = 5).
 *
 * dev_flags = u8[n_haystacks], read and written: a haystack whose flag is nonzero on entry is not scanned and keeps its
 * flag; the call sets flag h to 1 when haystack h contains a pattern, and never clears one (zero the array for a fresh
 * answer; OR-accumulating lets several calls -- windows of one haystack, several automata -- share one array).
 * dev_scratch = u64[3], any contents: the call clears it (cudaMemsetAsync) and leaves
 *   [0] its task counter (low 32 bits: tasks claimed, one more per warp than there are tasks);
 *   [1] tasks skipped whole: tasks of task_bytes (a grid anchored at the 512-byte aligned address at or before dev_bytes)
 *       whose part of the stream [dev_offsets[0], dev_offsets[n]) lies inside one haystack whose flag was set when a
 *       warp claimed the task;
 *   [2] windows not scanned: in the other tasks, the 512-byte windows of the grid from the first one, past the task's
 *       first, that lies inside the haystack holding the rest of the task, if that haystack's flag was set when the
 *       previous window was loaded, through the task's last window.
 * Skipping changes speed only, never the flags.  Returns ACB_EINVAL, before any CUDA call, for a null pointer (a null
 * dev_bytes is accepted when total_bytes == 0: an empty buffer), n_haystacks outside [0, 2^32 - 2],
 * total_bytes >= 2^31 or an automaton without a sieve image.  n_haystacks == 0 or total_bytes == 0 launches nothing.
 */
int acb_any_match(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                  int64_t n_haystacks, uint64_t total_bytes, uint8_t *dev_flags, uint64_t *dev_scratch, void *stream);

/*
 * Each haystack's first match for the automaton's match kind: the first record the reference's non-overlapping
 * iterator (try_find_iter, src/lib.rs:58-60) yields, i.e. the crate's AhoCorasick::find, once per haystack of a
 * device-resident batch (haystack h = dev_bytes[dev_offsets[h] .. dev_offsets[h+1]); total_bytes = length of the
 * dev_bytes buffer, below 2^31).  Three calls:
 *
 * acb_find_first runs the sieve kernel in its first-match mode: one launch, no match list, no epilogue, no
 * synchronisation, every match kind.  dev_keys = u64[n_haystacks], read and written: key h is lowered (atomic minimum)
 * to the best match found in haystack h and never raised; ~0 (UINT64_MAX) = no match.  Positions in a key are byte
 * offsets relative to the haystack's start, and a smaller key is a better match:
 *   ACB_STANDARD           end << 32 | (0xffffffff - (end - start))   earliest end, then the longest pattern
 *   ACB_LEFTMOST_FIRST     start << 32 | pattern                       leftmost start, then the lowest pattern index
 *   ACB_LEFTMOST_LONGEST   start << 32 | (0xffffffff - end)            leftmost start, then the longest pattern
 * (patterns with the same bytes are ranked by index).  A key given on entry is a bound: positions that cannot beat it
 * are not scanned -- a position whose haystack-relative end is e gives a key whose high word is at least e (Standard)
 * or e - max_pattern_len (the leftmost kinds), and it cannot beat a key whose high word is strictly below that.  Fill
 * the array with ~0 for a fresh answer; min-accumulating lets the windows of one haystack share a key.
 * dev_scratch = u64[3], any contents: as acb_any_match's, with "flag set" read as "no position from the task's first
 * byte (the window's first byte) on can beat the key":
 *   [0] its task counter; [1] tasks skipped whole: tasks whose part of the stream lies inside one haystack, and whose
 *   first byte's position could not beat that haystack's key when a warp claimed the task; [2] windows not scanned: in
 *   the other tasks, the 512-byte windows of the grid from the first one, past the task's first, that lies inside the
 *   haystack holding the rest of the task, if its first byte's position could not beat that haystack's key when the
 *   previous window was loaded, through the task's last window.
 * Skipping changes speed only, never the keys.  Argument checks, the 2^31 limit and the empty cases are acb_any_match's.
 *
 * acb_first_rows decodes the keys into dev_rows = int64[n_haystacks][3] = (pattern, start, end), byte offsets relative
 * to the haystack, and (-1, -1, -1) where the key is ~0.  It reads the sieve image (pattern lengths, and the reverse
 * trie that names the pattern of a Standard or LeftmostLongest key) and, for those two kinds, the bytes of the
 * haystacks with a match; dev_bytes and dev_offsets must be the buffers the keys were found in.  One launch.
 *
 * acb_rows_to_codepoints converts such rows, of a UTF-8 batch, to code point indexes (what codepoints != 0 gives
 * acb_scan_batch): dev_cp_rows (same shape, not dev_rows) gets dev_rows with start and end lowered by the continuation
 * bytes of the haystack before them.  Positions are 64-bit: total_bytes may exceed 2^31.  Work is the bytes before each
 * row's end, spread over the whole grid.  One device-to-device copy and one launch, no synchronisation.
 *
 * All three return ACB_EINVAL, before any CUDA call, for a null pointer or n_haystacks outside [0, 2^32 - 2].
 */
int acb_find_first(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_keys, uint64_t *dev_scratch, void *stream);
int acb_first_rows(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                   int64_t n_haystacks, const uint64_t *dev_keys, int64_t *dev_rows, void *stream);
int acb_rows_to_codepoints(const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes,
                           const int64_t *dev_rows, int64_t *dev_cp_rows, void *stream);

/*
 * How many matches each haystack has: len(find_matches_as_indexes(haystack, overlapping)) of the reference
 * (get_matches, src/lib.rs:42-68), once per haystack of a device-resident batch, without the match list.  Counts are
 * the same in bytes and in code points.  Three calls:
 *
 * acb_count_overlapping counts the overlapping matches (try_find_overlapping_iter, src/lib.rs:52-54): one launch of the
 * sieve kernel in its count mode -- no records, no epilogue, no synchronisation, nothing skipped.  Standard automata
 * only: any other kind returns ACB_EUNSUPPORTED before any byte is read, like the reference.  dev_counts =
 * u64[n_haystacks], read and written: haystack h's count is ADDED to dev_counts[h] (zero the array for a fresh answer;
 * accumulating lets the windows of one haystack share a counter).  dev_scratch = u64[3], any contents: the call clears
 * it and leaves its task counter in [0].  Argument checks, the 2^31 limit and the empty cases are acb_any_match's.
 *
 * acb_count_non_overlapping counts the non-overlapping matches (try_find_iter, src/lib.rs:58-60) for every match kind:
 * the sieve's list scan, as acb_scan_batch runs it (same plan, same workspace, kernel 5 whatever the tuning), then a
 * count epilogue that places the overlapping list and counts each haystack's selection without packing it.  A haystack
 * whose overlapping list has more than ACB_LONG_STRETCH records is counted by the whole grid (successor of every
 * record, then pointer jumping), the others by one thread each.  dev_counts = u64[n_haystacks] is WRITTEN.  ws->dev_total:
 * [0] = the sum of the counts, [1] = 1 when the counts are complete (0: the workspace was too small, every count is
 * zero and [0] / [4] say how much room a second call needs, as for acb_scan_batch), [2] = haystacks counted by the
 * whole grid, [3] = [5] = 0, [4] = records of the overlapping list.  Two launches, no synchronisation.  ws->dev_out and
 * ws->dev_raw are overwritten; ws->dev_match_offsets is not used.
 *
 * acb_count_rows counts what acb_select_non_overlapping would select from the rows of ONE haystack (same shape and
 * order): *dev_count = the count.  dev_scratch = 16 * n_rows bytes.  The work is spread over the grid (pointer jumping,
 * as above) in one cooperative launch.
 *
 * All three return ACB_EINVAL, before any CUDA call, for a null pointer (a null dev_bytes is accepted when total_bytes
 * == 0; dev_rows and dev_scratch may be null when n_rows == 0), n_haystacks outside [0, 2^32 - 2], total_bytes >= 2^31,
 * n_rows >= 2^32 - 1, a workspace with a null buffer or a plan that acb_plan_scan does not give for these arguments.
 */
#define ACB_LONG_STRETCH 4096
int acb_count_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                          int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_counts, uint64_t *dev_scratch, void *stream);
int acb_count_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                              int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                              uint64_t *dev_counts, void *stream);
int acb_count_rows(const acb_automaton *a, const int64_t *dev_rows, uint64_t n_rows, uint64_t *dev_scratch, uint64_t *dev_count,
                   void *stream);

/*
 * How often each pattern matches in a device-resident batch, without the match list: dev_pattern_counts =
 * u64[acb_num_patterns(a)], read and written, and entry p is ADDED the number of records with pattern p in the
 * reference's result (get_matches, src/lib.rs:42-68), summed over the batch's haystacks.  Patterns with the same bytes
 * keep their own ids and are each counted as the reference reports them.  Accumulating lets runs of haystacks, windows
 * of one haystack and several devices total one corpus.  Two calls:
 *
 * acb_pattern_counts_overlapping counts the overlapping matches: one launch of the sieve kernel in its pattern mode, no
 * records, no epilogue, no synchronisation, nothing skipped.  Standard automata only: any other kind returns
 * ACB_EUNSUPPORTED before any byte is read.  dev_scratch = u64[3], as for acb_count_overlapping.
 *
 * acb_pattern_counts_non_overlapping counts the non-overlapping matches for every match kind: the sieve's list scan
 * (plan and workspace as for acb_count_non_overlapping), then an epilogue that places the overlapping list, selects each
 * haystack's matches without packing a result, and adds the selected records' patterns.  A haystack whose overlapping
 * list has more than ACB_LONG_STRETCH records is selected by the whole grid (successors, pointer jumping, and marks
 * that follow the chain of selected records), the others by one thread each.  ws->dev_total: [0] = records added (the
 * total of the selection), [1] = 1 when the counts were added (0: the workspace was too small, NOTHING was added, and
 * [0] / [4] say how much room a second call needs), [2] = haystacks selected by the whole grid, [3] = [5] = 0, [4] =
 * records of the overlapping list.  Two launches, no synchronisation.  ws->dev_out, ws->dev_raw, ws->dev_raw_seq and
 * ws->dev_match_offsets are overwritten.
 *
 * Argument checks, the 2^31 limit and the empty cases are those of acb_count_overlapping and acb_count_non_overlapping
 * (ACB_EINVAL before any CUDA call); an empty batch adds nothing.
 */
int acb_pattern_counts_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_pattern_counts, uint64_t *dev_scratch,
                                   void *stream);
int acb_pattern_counts_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                       int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                       uint64_t *dev_pattern_counts, void *stream);

/*
 * Which patterns each haystack contains, and how often: for haystack h, with R_h the reference's result
 * find_matches_as_indexes(h, overlapping) (get_matches, src/lib.rs:42-68), the HITS of h are the pairs (p, c) where p
 * is a pattern id occurring in R_h and c the number of records of R_h with pattern p, p ascending.  Patterns with the
 * same bytes keep their own ids (non-overlapping: the lower id takes the match).  The row sums are the per-haystack
 * counts of acb_count_*; the column sums are acb_pattern_counts_*.  The list is never handed back.
 *
 * The sieve's list scan (plan and workspace as for acb_count_non_overlapping, kernel 5 whatever the tuning), then one
 * epilogue that places the overlapping list, selects each haystack's matches (overlapping: all of them) and aggregates
 * their patterns.  A haystack whose overlapping list has at most ACB_LONG_STRETCH records is aggregated by one warp
 * (a sort of its pids); a longer one gets a counter row in dev_rows.  A row is acb_pattern_hit_row_words(n_patterns)
 * u32 words: n_patterns counters, padded to an even count, then 8-byte bookkeeping (the haystack, then one word per
 * 2048 counters).  dev_rows must be 8-byte aligned and hold row_words words; it may be null when row_words == 0.
 *
 * Outputs: ws->dev_out = the hits as acb_pattern_hit records, grouped by haystack, patterns ascending within each;
 * ws->dev_match_offsets = u64[n_haystacks + 1] bracketing each haystack's hits.  ws->dev_total: [0] = hits, [1] = 1
 * when the result is complete (0: the list did not fit the workspace or row_words was too small; NOTHING valid was
 * written, and [4] / [5] say how much room a second call needs), [2] = haystacks selected on the grid (lists of more than
 * ACB_LONG_STRETCH records), [3] = haystacks aggregated in a counter row, [4] = records of the overlapping list, [5] =
 * counter-row words needed (known once the list fits; at most [4] / (ACB_LONG_STRETCH + 1) rows).  ws->dev_raw,
 * ws->dev_raw_seq and dev_rows are overwritten.  Two launches, no synchronisation.  A u32 count suffices: one call
 * addresses fewer than 2^31 bytes, and a pattern matches at most once per end position.
 *
 * overlapping = 1 on a leftmost automaton returns ACB_EUNSUPPORTED before any byte is read, like the reference.
 * Argument checks, the 2^31 limit and the empty cases are those of acb_count_non_overlapping (ACB_EINVAL before any
 * CUDA call), plus overlapping outside {0, 1} and a misaligned dev_rows.
 */
typedef struct acb_pattern_hit {
    uint32_t haystack; /* index into the batch */
    uint32_t pattern;  /* pattern id */
    uint32_t count;    /* records of the haystack's result with this pattern */
    uint32_t reserved; /* 0 */
} acb_pattern_hit;     /* 16 bytes, like acb_match */
uint64_t acb_pattern_hit_row_words(uint64_t n_patterns);
int acb_pattern_hits(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                     int64_t n_haystacks, uint64_t total_bytes, int overlapping, const acb_plan *plan, const acb_workspace *ws,
                     uint32_t *dev_rows, uint64_t row_words, void *stream);

/*
 * Stream search: matches in data that arrives in chunks, for many streams at once.  A stream is the concatenation of
 * the chunks fed to it; positions are absolute within it and 64-bit.  The crate the reference wraps has the single-stream,
 * Standard, non-overlapping form (AhoCorasick::stream_find_iter); here every match kind and overlapping Standard are
 * served, and the rows a stream releases over all its feeds are exactly the one-shot result on the concatenation
 * (get_matches, src/lib.rs:42-68), in the reference's order.  A feed gives each stream one chunk (maybe empty) of a
 * device-resident batch: chunk i = dev_bytes[dev_offsets[i] .. dev_offsets[i + 1]); total_bytes = length of the dev_bytes
 * buffer, below 2^31.
 *
 * Release rule, in bytes whatever the positions are reported in: after a feed that brings a stream to F bytes, the rows
 * it has released are the rows of the one-shot result with end <= F (Standard, overlapping or not), or with
 * start + max_pattern_len <= F (LeftmostFirst, LeftmostLongest: no later match can start before such a row).  A feed
 * that ends a stream (dev_last[i] != 0) releases the rest and leaves its carry zero: the slot starts a new stream.
 *
 * The caller owns the state of each stream, zero-filled before its first feed (halo = acb_max_pattern_len - 1):
 *   dev_carry = int64[n_streams][4]: [0] bytes fed so far F, [1] the restart point of the non-overlapping selection
 *     (absolute byte offset), [2] tail length T = min(F, halo), [3] UTF-8 continuation bytes before the tail's start
 *     (kept when codepoints != 0, else 0);
 *   dev_tail = uint8[n_streams][halo]: stream i's last T bytes at dev_tail + i * halo (may be null when halo == 0).
 *
 * A feed is four calls on one CUDA stream:
 *   1. acb_stream_seams writes each stream's seam -- its tail, then the chunk's first min(chunk length, halo) bytes --
 *      packed into dev_seam_bytes (room for n_streams * 2 * halo bytes; may be null when halo == 0), and
 *      dev_seam_offsets = int64[n_streams + 1] brackets them: a batch of n_streams haystacks.  Three launches.
 *   2. acb_scan_batch with overlapping = 2, codepoints = 0 (the overlapping list of any automaton, in bytes) on the
 *      chunks (dev_bytes, dev_offsets) as they are, and
 *   3. the same on the seams (dev_seam_bytes, dev_seam_offsets), each with its own workspace: both lists are read in 4.
 *   4. acb_stream_resolve merges, per stream, its seam's records with its chunk's records that end past the seam (every
 *      match ending in the chunk starts at most halo bytes before it, so it lies in tail || chunk), continues the
 *      selection from the carried restart point (one thread per stream: the selection is a chain), and writes
 *      dev_rows = int64[k][4] = (stream, pattern, start, end), grouped by stream in the reference's order, and
 *      dev_row_offsets = int64[n_streams + 1] bracketing each stream's rows (k = dev_row_offsets[n_streams]).  With
 *      codepoints != 0 (UTF-8 data, chunks may be cut inside a character) start and end are code point indexes: the
 *      byte offset minus the continuation bytes before it in the stream; it needs dev_image (pattern lengths in code
 *      points).  Then it updates the carry and the tail.  dev_seam_list / dev_chunk_list and their match offsets are
 *      ws->dev_out / ws->dev_match_offsets of the scans in 2 and 3.  With R = the two lists' lengths added
 *      (dev_seam_match_offsets[n] + dev_chunk_match_offsets[n]), dev_rows needs room for R rows and dev_scratch =
 *      int64[2 + 6 * n_streams + 4 * R] (int64[2 + 6 * n_streams] for overlapping = 1, whose rows are read from the
 *      lists directly): it leaves [0] = list records the selection considered, [1] = streams holding something back
 *      (a leftmost pick not yet released, or a restart point past the new tail's start).  dev_last = uint8[n_streams]
 *      or null (no stream ends).  A memset and four kernel launches (select, prefix, rows, carry); with code points
 *      the rows are written by the carry kernel and acb_rows_to_codepoints' copy and launch replace the rows kernel.
 *      No synchronisation.
 *
 * Both return ACB_EINVAL, before any CUDA call, for a null pointer (dev_bytes may be null when total_bytes == 0),
 * n_streams outside [0, 2^32 - 2], total_bytes >= 2^31, overlapping other than 0 / 1 or codepoints without dev_image;
 * acb_stream_resolve returns ACB_EUNSUPPORTED for overlapping = 1 on a leftmost automaton, like the reference.
 */
int acb_stream_seams(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                     const int64_t *dev_carry, const uint8_t *dev_tail, uint8_t *dev_seam_bytes, int64_t *dev_seam_offsets, void *stream);
int acb_stream_resolve(const acb_automaton *a, const void *dev_image, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams,
                       uint64_t total_bytes, const uint8_t *dev_last, int overlapping, int codepoints, int64_t *dev_carry, uint8_t *dev_tail,
                       const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, const acb_match *dev_seam_list,
                       const uint64_t *dev_seam_match_offsets, const acb_match *dev_chunk_list, const uint64_t *dev_chunk_match_offsets,
                       int64_t *dev_scratch, int64_t *dev_rows, int64_t *dev_row_offsets, void *stream);

/*
 * Stream queries: is_match, find_first and count_matches per stream, without the rows.  They keep the stream search's
 * carry and tail (dev_carry, dev_tail above; word [1] is used by the non-overlapping count only) and its seams: a feed
 * starts with acb_stream_seams and ends with acb_stream_advance.  Let C be a stream's concatenation so far, F = len(C).
 *
 * acb_stream_advance updates the carry without a selection: the new tail, F and T, and with codepoints != 0 the
 * continuation bytes before the tail (dev_scratch = int64[6 * n_streams], else it may be null).  A stream with
 * dev_last[i] != 0 gets a zero carry.  It reads the seams, so it runs after the feed's scans.  With code points a
 * launch, acb_rows_to_codepoints' copy and launch, then one launch; without, one launch.
 *
 * is_match: acb_any_match on the seams and on the chunks, with the same persistent dev_flags (u8[n_streams], zero for
 * a new stream): flag i is then is_match(C), and a stream already flagged has its chunk tasks skipped whole.  The
 * caller reads the flags, and zeroes those of the streams that end.
 *
 * find_first: per stream, dev_best = int64[n_streams][6], zero for a new stream: [0] state (0 no candidate, 1 a pending
 * one, 2 the final answer), [1] pattern, [2] start, [3] end (absolute byte offsets), [4] start, [5] end in code points
 * (the byte offsets without codepoints).  dev_seam_keys and dev_chunk_keys = u64[n_streams], ~0 for a new stream, are
 * the keys of acb_find_first on the seams and on the chunks; acb_stream_first_resolve leaves them ready for the next
 * feed: 0 where that scan can be skipped (a final answer: both; a pending leftmost candidate: the chunk's, whose
 * records all start after it), ~0 elsewhere.  A feed: acb_stream_seams, acb_find_first on the seams and on the
 * chunks, acb_stream_first_resolve, acb_stream_advance.  The resolve decodes both keys (acb_first_rows; keys that
 * were pre-set to 0 are ignored), converts them to code points (acb_rows_to_codepoints; the carried continuation
 * count gives the part before the seam), takes the best of the carried candidate and the two under the kind's key
 * order above, and applies the release rule: Standard is final at once (end <= F), the leftmost kinds once start +
 * max_pattern_len <= F, every candidate on dev_last.  dev_rows = int64[n_streams][3] gets each final answer
 * (pattern, start, end) -- code point indexes with codepoints != 0 -- and (-1, -1, -1) elsewhere; a stream that ends
 * gets its final answer and a zero dev_best.  dev_seam_bytes, dev_seam_offsets are the seams' buffers,
 * seam_buffer_bytes the length of dev_seam_bytes (below 2^31).  dev_scratch = int64[2 + 12 * n_streams]: it leaves
 * [1] = streams with a pending candidate.  A memset and seven launches (eleven with code points: two copies and two
 * launches of acb_rows_to_codepoints), no synchronisation.
 *
 * count_matches: dev_running = int64[n_streams], zero for a new stream.  acb_stream_count adds this feed's count and
 * writes dev_counts = int64[n_streams]: the number of rows the stream search would have released so far (after a
 * feed with dev_last[i], len(find_matches_as_indexes(C, overlapping))); it zeroes dev_running[i] of a stream that
 * ends, and acb_stream_advance follows it.
 *   overlapping = 1 (Standard only; a leftmost automaton returns ACB_EUNSUPPORTED): a feed is acb_stream_seams,
 *     acb_scan_batch (overlapping = 2) on the seams, acb_count_overlapping on the chunks into zeroed dev_chunk_counts
 *     = u64[n_streams], acb_stream_count, acb_stream_advance.  The count adds the chunk's and the seam records that
 *     cross the tail / head join (start < T < end).  dev_chunk_list and its offsets may be null.  dev_scratch =
 *     int64[4].  A memset and one launch.
 *   overlapping = 0, every kind: the two scans of the stream search (acb_scan_batch, overlapping = 2, on the chunks
 *     and on the seams), then acb_stream_count, which continues the selection from the carried restart point (word
 *     [1]) and counts the picks the release rule allows.  A stream whose sequence has at most ACB_LONG_STRETCH
 *     records is counted by one thread; a longer one by the whole grid (successors, pointer jumping, marks on the
 *     selected chain, as acb_pattern_counts_non_overlapping).  dev_chunk_counts may be null.  dev_scratch =
 *     int64[scratch_words], scratch_words >= 4 + 6 * n_streams + 4 * R, R = the two lists' lengths added.  A memset
 *     and one cooperative launch.
 *   dev_scratch leaves [0] = list records considered, [1] = streams holding a pick the release rule does not allow
 *   yet, [2] = streams counted on the whole grid.
 *
 * All three return ACB_EINVAL, before any CUDA call, for a null pointer (dev_bytes may be null when total_bytes == 0,
 * dev_tail and dev_seam_bytes when max_pattern_len == 1), n_streams outside [0, 2^32 - 2], total_bytes >= 2^31,
 * overlapping other than 0 / 1 or a dev_scratch too small; acb_stream_first_resolve also for an automaton without a
 * sieve image.  n_streams == 0 launches nothing.
 */
int acb_stream_advance(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                       const uint8_t *dev_last, int codepoints, int64_t *dev_carry, uint8_t *dev_tail, const uint8_t *dev_seam_bytes,
                       const int64_t *dev_seam_offsets, int64_t *dev_scratch, void *stream);
int acb_stream_first_resolve(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                             int64_t n_streams, uint64_t total_bytes, const uint8_t *dev_last, int codepoints, const int64_t *dev_carry,
                             const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, uint64_t seam_buffer_bytes,
                             uint64_t *dev_seam_keys, uint64_t *dev_chunk_keys, int64_t *dev_best, int64_t *dev_scratch, int64_t *dev_rows,
                             void *stream);
int acb_stream_count(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                     const uint8_t *dev_last, int overlapping, int64_t *dev_carry, const int64_t *dev_seam_offsets,
                     const acb_match *dev_seam_list, const uint64_t *dev_seam_match_offsets, const acb_match *dev_chunk_list,
                     const uint64_t *dev_chunk_match_offsets, const uint64_t *dev_chunk_counts, int64_t *dev_running, int64_t *dev_counts,
                     int64_t *dev_scratch, uint64_t scratch_words, void *stream);

/*
 * Token ids: a byte format that makes a search over token-id sequences an exact byte search (csrc/tokens.cuh).  Id t,
 * 0 <= t < ACB_TOKEN_ID_LIMIT, becomes ACB_TOKEN_BYTES bytes: 0x80 | (t >> 14), (t >> 7) & 0x7f, t & 0x7f.  Only a
 * token's first byte has its high bit set, so every occurrence of an encoded pattern in an encoded haystack starts and
 * ends on a token boundary: the byte search's rows, divided by ACB_TOKEN_BYTES, are the token search's, for every
 * match kind, overlapping or not, and for every query and stream form.
 *
 * acb_tokens_encode writes ACB_TOKEN_BYTES * n_tokens bytes to dev_out from the ids at dev_tokens: token_bytes = 2
 * (uint16), 4 (int32) or 8 (int64).  dev_bad = u64, which the caller presets to ~0: an id outside [0, 2^21) lowers
 * it, with atomicMin, to that id's index, so after the call it holds the smallest bad index (or still ~0); the bytes of
 * a bad id are undefined.  One launch (none for n_tokens == 0); 16-byte loads and 32-bit stores when dev_tokens is
 * 16-byte aligned and dev_out 4-byte aligned, one id at a time otherwise.  No synchronisation.
 * acb_tokens_encode_host is the same on host memory (host_bad preset by the caller too), on the calling thread.
 * Both return ACB_EINVAL, before any CUDA call, for a token_bytes other than 2, 4 or 8, n_tokens >= 2^60 or a null
 * pointer (the ids and the output may be null when n_tokens == 0).
 */
/*
 * Pattern sets: each haystack (or stream) searches for its own subset of the automaton's patterns.  For haystack h with
 * set S, every covered query returns exactly what it would return from an automaton built from only the patterns in S,
 * with the same match kind and in the same relative order (LeftmostFirst priority is kept), reporting ids of the FULL
 * automaton.  The descriptor:
 *   dev_set_bits   u32[n_sets][words_per_set], words_per_set = ceil(n_patterns / 32): bit p % 32 of word p / 32 of
 *                  row s = pattern p is in set s
 *   dev_set_index  int32 (index_bytes 4) or int64 (8) [n_haystacks]: haystack h uses row dev_set_index[h]; an index
 *                  outside [0, n_sets) admits no pattern (the kernels never read outside the bitset)
 * The *_filtered entry points take it as their last argument before `stream` and are otherwise the calls they are
 * named after; a NULL filter is exactly that call.  A filtered call always runs the sieve (the table images hold every
 * pattern): acb_scan_batch_filtered takes kernel 5 whatever the tuning and needs dev_sieve.  acb_first_rows_filtered
 * must get the filter its keys were found with (the node's lowest ADMITTED pid is reported), and
 * acb_stream_first_resolve_filtered passes it on to the two acb_first_rows calls it makes.  ACB_EINVAL, before any
 * device work: n_sets == 0, a null dev_set_bits, a null dev_set_index with n_haystacks > 0, index_bytes not 4 or 8.
 * (The is_match stream needs no filtered resolve: it is acb_any_match_filtered on the seams and the chunks.)
 */
typedef struct acb_pattern_filter {
    const uint32_t *dev_set_bits;
    uint64_t n_sets;
    const void *dev_set_index;
    int index_bytes;
} acb_pattern_filter;
int acb_scan_batch_filtered(const acb_automaton *a, const void *dev_image, const void *dev_hot, const acb_hot_desc *hot_desc,
                            const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks,
                            uint64_t total_bytes, int overlapping, int codepoints, const acb_plan *plan, const acb_workspace *ws,
                            const acb_pattern_filter *filter, void *stream);
int acb_any_match_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                           int64_t n_haystacks, uint64_t total_bytes, uint8_t *dev_flags, uint64_t *dev_scratch,
                           const acb_pattern_filter *filter, void *stream);
int acb_find_first_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                            int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_keys, uint64_t *dev_scratch,
                            const acb_pattern_filter *filter, void *stream);
int acb_first_rows_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                            int64_t n_haystacks, const uint64_t *dev_keys, int64_t *dev_rows, const acb_pattern_filter *filter, void *stream);
int acb_count_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_counts, uint64_t *dev_scratch,
                                   const acb_pattern_filter *filter, void *stream);
int acb_count_non_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                       int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                       uint64_t *dev_counts, const acb_pattern_filter *filter, void *stream);
int acb_stream_first_resolve_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                      int64_t n_streams, uint64_t total_bytes, const uint8_t *dev_last, int codepoints, const int64_t *dev_carry,
                                      const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, uint64_t seam_buffer_bytes,
                                      uint64_t *dev_seam_keys, uint64_t *dev_chunk_keys, int64_t *dev_best, int64_t *dev_scratch,
                                      int64_t *dev_rows, const acb_pattern_filter *filter, void *stream);

/*
 * Match masks: which bytes of a device-resident batch lie inside a match.  For haystack h, with R_h the reference's
 * result find_matches_as_indexes(h, overlapping) (with a filter: R_h for h's set), byte offsets[h] + p is COVERED when
 * start <= p < end for some record of R_h.  Bytes outside every haystack are not covered.  The mask is a u32 bitmask
 * that every call OR-accumulates into: bit bit_base + q (bit q % 32 of word q / 32) stands for byte q of dev_bytes,
 * and the caller zeroes the mask once.  So runs of haystacks, windows of one haystack and several code paths can fill
 * one mask.  The list is never handed back.
 *
 * acb_match_mask_overlapping covers the overlapping matches: one launch of the sieve kernel in its cover mode -- at
 * each end position the longest match ending there covers every shorter one, so its bytes are OR-ed in and no chain
 * is walked.  No records, no epilogue, no synchronisation, nothing skipped.  Standard automata only: any other kind
 * returns ACB_EUNSUPPORTED before any byte is read.  dev_scratch = u64[3], as for acb_count_overlapping.
 *
 * acb_match_mask_non_overlapping covers the non-overlapping matches for every match kind: the sieve's list scan (plan
 * and workspace as for acb_count_non_overlapping), then an epilogue that places the overlapping list, selects each
 * haystack's matches as acb_pattern_counts_non_overlapping does (stretches of more than ACB_LONG_STRETCH records on the
 * whole grid) and ORs the selected records' bytes.  ws->dev_total is that call's: [0] = records selected, [1] = 1 when
 * the mask was written (0: the workspace was too small, NOTHING was OR-ed, and [0] / [4] say how much room a second
 * call needs), [2] = haystacks selected by the whole grid, [4] = records of the overlapping list.  Two launches, no
 * synchronisation.
 *
 * acb_mask_rows ORs the bytes of rows that are already selected: row_bytes 4 = acb_match records, 8 = int64 rows
 * (haystack, pattern, start, end), positions haystack-relative bytes; row r covers bits bit_base + dev_offsets[h] +
 * [start, end).  Rows naming a haystack outside [0, n_haystacks) or an empty span are skipped.  One launch.
 *
 * acb_mask_unpack turns bits into bytes: dev_out[i] = bit bit_base + stride * i of dev_mask (0 or 1), i < n.  stride 1
 * for bytes, ACB_TOKEN_BYTES for token ids (an occurrence starts and ends on a token boundary).  One launch.
 *
 * ACB_EINVAL, before any CUDA call: a null pointer (dev_bytes may be null when total_bytes == 0, dev_rows when n_rows
 * == 0, dev_mask and dev_out when n == 0), n_haystacks outside [0, 2^32 - 2], total_bytes >= 2^31, a malformed filter,
 * a workspace with a null buffer or a plan acb_plan_scan does not give for these arguments, row_bytes not 4 or 8,
 * stride 0.
 */
int acb_match_mask_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                               int64_t n_haystacks, uint64_t total_bytes, uint32_t *dev_mask, uint64_t bit_base, uint64_t *dev_scratch,
                               void *stream);
int acb_match_mask_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                        int64_t n_haystacks, uint64_t total_bytes, uint32_t *dev_mask, uint64_t bit_base,
                                        uint64_t *dev_scratch, const acb_pattern_filter *filter, void *stream);
int acb_match_mask_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                   uint32_t *dev_mask, uint64_t bit_base, void *stream);
int acb_match_mask_non_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes,
                                            const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan,
                                            const acb_workspace *ws, uint32_t *dev_mask, uint64_t bit_base,
                                            const acb_pattern_filter *filter, void *stream);
int acb_mask_rows(const void *dev_rows, int row_bytes, uint64_t n_rows, const int64_t *dev_offsets, int64_t n_haystacks, uint32_t *dev_mask,
                  uint64_t bit_base, void *stream);
int acb_mask_unpack(const uint32_t *dev_mask, uint64_t bit_base, uint64_t stride, uint64_t n, uint8_t *dev_out, void *stream);

/*
 * Match-mask streams: the match mask of each stream's concatenation, flag by flag, released once no later data can
 * change it.  Let halo = acb_max_pattern_len - 1 and F the bytes a stream has been fed.  After a feed the stream has
 * released the positions [0, R), R = F - T = max(0, F - halo) (T = dev_carry[2]); a feed with dev_last[i] != 0 sets
 * R = F, releases everything still held and starts the slot again at position 0.  A released flag is final: it equals
 * the mask of the whole concatenation (acb_match_mask_*, overlapping or not, with a filter the stream's set).  A match
 * covering p < R starts at most p, so start + max_pattern_len <= F and end <= F: the stream search has released it.
 *
 * State: the stream search's dev_carry, dev_tail and seams (above), and the HELD flags, uint8[n_streams][halo] twice:
 * byte k of stream i's row in the read buffer is the flag of position R + k, k < T.  Each feed reads one buffer and
 * writes the other (a chunk shorter than the tail shifts it); the caller swaps them.  Both zero-filled at first (may
 * be null when halo == 0).  A feed, on one CUDA stream, with dev_chunk_mask = u32[ceil(total_bytes / 32)] and
 * dev_seam_mask = u32[ceil(seam buffer bytes / 32)] zero-filled for it (bit q: byte q of that buffer):
 *   1. acb_stream_seams.
 *   2. overlapping = 1 (Standard): acb_match_mask_overlapping(_filtered) on the chunks into dev_chunk_mask and on the
 *      seams into dev_seam_mask, bit_base 0.  Every match that ends past the old F lies wholly in one of them; matches
 *      that end before were OR-ed by earlier feeds, and their bits past the old R are in the held flags.
 *      overlapping = 0 (every kind): the stream search's two list scans and acb_stream_resolve with codepoints = 0,
 *      after copying dev_carry (int64[n_streams][4]) to dev_carry_before; then acb_stream_mask_rows ORs each released
 *      row into the bit spaces: the part in the old tail into dev_seam_mask, the rest into dev_chunk_mask.  A row this
 *      feed releases starts at or after the old R, so it lies in old tail || chunk.  One launch, grid-stride over the
 *      rows (their count is read on the device).
 *   3. acb_stream_mask_emit writes the flags of the positions in [R_old, R_new) that are multiples of stride (1: a flag
 *      per byte; ACB_TOKEN_BYTES: a flag per token id, read at its first byte), packed by stream into dev_flags (room
 *      for total_bytes + n_streams * halo flags), dev_flag_offsets = int64[n_streams + 1] bracketing each stream's and
 *      dev_flag_starts = int64[n_streams] = the index of each stream's first one (ceil(R_old / stride)).  The flag of
 *      byte p is, in the old tail, its held flag OR its seam bit; in the chunk, its chunk bit OR (overlapping = 1) the
 *      seam bit of the head byte it is.  It writes the held flags of [R_new, F_new) to dev_held_out.  It reads F and T
 *      from dev_carry_before, the carry as it was before this feed: dev_carry itself on the overlapping path, where it
 *      runs before step 4; the copy on the other, whose resolve has already moved the carry (and zeroed it on
 *      dev_last).  Three launches (count, prefix, the flags and held flags on the whole grid), no synchronisation.
 *   4. overlapping = 1: acb_stream_advance (codepoints = 0).  overlapping = 0: nothing, the resolve advanced the carry.
 *
 * ACB_EINVAL, before any CUDA call: a null pointer (dev_last may be null: no stream ends; the held buffers when halo
 * == 0), the same buffer for dev_held_in and dev_held_out, overlapping other than 0 / 1, stride outside [1, 2^32 - 1],
 * n_streams outside [0, 2^32 - 2].  acb_stream_mask_emit returns ACB_EUNSUPPORTED for overlapping = 1 on a leftmost
 * automaton.  n_streams == 0 launches nothing (the emit zeroes dev_flag_offsets[0]).
 */
int acb_stream_mask_rows(const int64_t *dev_offsets, int64_t n_streams, const int64_t *dev_carry_before, const int64_t *dev_seam_offsets,
                         const int64_t *dev_rows, const int64_t *dev_row_offsets, uint32_t *dev_chunk_mask, uint32_t *dev_seam_mask,
                         void *stream);
int acb_stream_mask_emit(const acb_automaton *a, const int64_t *dev_offsets, int64_t n_streams, const uint8_t *dev_last, int overlapping,
                         uint64_t stride, const int64_t *dev_carry_before, const int64_t *dev_seam_offsets, const uint32_t *dev_chunk_mask,
                         const uint32_t *dev_seam_mask, const uint8_t *dev_held_in, uint8_t *dev_held_out, uint8_t *dev_flags,
                         int64_t *dev_flag_offsets, int64_t *dev_flag_starts, void *stream);

#define ACB_TOKEN_ID_LIMIT (1u << 21)
#define ACB_TOKEN_BYTES 3
int acb_tokens_encode(const void *dev_tokens, int token_bytes, uint64_t n_tokens, uint8_t *dev_out, uint64_t *dev_bad, void *stream);
int acb_tokens_encode_host(const void *host_tokens, int token_bytes, uint64_t n_tokens, uint8_t *host_out, uint64_t *host_bad);

/*
 * Completing tokens: for each row of token-id histories, the next ids that would complete a pattern.  With C a row's
 * history and S its admitted patterns (all, or with a filter the row's set), id t COMPLETES a pattern when some p in S
 * is a suffix of C || [t]: p[:-1] is a suffix of C and p[-1] == t.  That is a new match ending right after C, for any
 * match kind -- it does not depend on the automaton's.  Only the last K - 1 ids of C matter (K = the longest pattern
 * in tokens); an id outside [0, ACB_TOKEN_ID_LIMIT) equals no pattern token.  The automaton's patterns must be in the
 * token format (acb_tokens_encode_host of each pattern).
 *
 * The completions image (csrc/completions.h) is a reverse trie over every pattern's p[:-1] at token granularity.
 * acb_completions_build builds it once on the host and writes its size to *image_bytes (ACB_EINVAL when a pattern is
 * not in the token format); the caller uploads acb_completions_write()'s copy and passes the device pointer as
 * dev_image.  acb_completions_describe reads a host copy's node and entry counts, depth = K - 1 and max_last = the
 * largest id that ends a pattern (0 without patterns).
 *
 * The three calls walk the image for every row, one warp per row: row i is dev_tokens[a, b) with a, b =
 * dev_offsets[i], dev_offsets[i + 1] clamped to [0, n_tokens] (b < a: an empty history), token_bytes 2 (uint16), 4
 * (int32) or 8 (int64).  Offsets are never checked on the device and nothing outside the ids is read.  Filter: as
 * acb_pattern_filter, one set per row (an index outside [0, n_sets) admits nothing).  One launch each, nothing
 * synchronises, nothing is allocated.
 *   acb_completions_count   dev_counts[i] = the number of distinct completing ids of row i (int64[n_rows])
 *   acb_completions_emit    those ids, written to dev_ids from dev_row_offsets[i] (int64[n_rows]: the exclusive prefix
 *                           sum of the counts), each once, ascending within a trie node (not overall)
 *   acb_completions_mask    logits[i * row_stride + t] = value for every completing id t of row i; every other element
 *                           untouched.  dev_logits: logits_dtype ACB_LOGITS_F32 / _F16 / _BF16, rows of `vocab`
 *                           elements row_stride elements apart.
 *   acb_completions_bias    a signed bias per pattern (a sequence-bias logits processor): with P_t the admitted pids
 *                           that t completes, ordered longest pattern first, ties by ascending pid (p1 .. pk),
 *                           s = dev_bias[p1], then s = fl32(s + dev_bias[pj]) for j = 2 .. k (the sum starts from its
 *                           first term, not from 0), and logits[i * row_stride + t] = round(fl32(logits[..] + s)) to
 *                           the logits dtype, nearest-even, once; every other element untouched.  dev_bias:
 *                           float32[n_patterns].  Each element is written by one thread: no atomics, the result is
 *                           the same bit for bit on every run.  All -inf biases give the mask's -inf.
 * ACB_EINVAL, before any CUDA call: a null pointer (dev_tokens may be null when n_tokens == 0, the per-row pointers
 * when n_rows == 0), acb_completions_build not called, token_bytes not 2, 4 or 8, n_tokens >= 2^60, n_rows outside
 * [0, 2^32 - 2], a malformed filter, and for the mask and the bias a logits_dtype not listed, vocab outside [1, 2^62),
 * row_stride outside [0, 2^62) or vocab <= max_last (the image has an id the rows cannot hold).  n_rows == 0 launches
 * nothing.
 */
#define ACB_LOGITS_F32 0
#define ACB_LOGITS_F16 1
#define ACB_LOGITS_BF16 2
typedef struct acb_completions_desc {
    uint32_t nodes;      /* reverse-trie nodes, the root included */
    uint32_t entries;    /* (last token, pattern) entries: the number of patterns */
    uint32_t depth;      /* K - 1: the history ids a walk may read */
    uint32_t max_last;   /* the largest id that ends a pattern */
} acb_completions_desc;
int acb_completions_build(acb_automaton *a, uint64_t *image_bytes);
int acb_completions_write(acb_automaton *a, void *host_dst, uint64_t dst_bytes);
int acb_completions_describe(const void *host_image, acb_completions_desc *desc);
int acb_completions_count(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                          const int64_t *dev_offsets, int64_t n_rows, int64_t *dev_counts, const acb_pattern_filter *filter, void *stream);
int acb_completions_emit(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, const int64_t *dev_row_offsets, int64_t *dev_ids,
                         const acb_pattern_filter *filter, void *stream);
int acb_completions_mask(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, void *dev_logits, int logits_dtype, int64_t row_stride, int64_t vocab,
                         float value, const acb_pattern_filter *filter, void *stream);
int acb_completions_bias(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, const float *dev_bias, void *dev_logits, int logits_dtype,
                         int64_t row_stride, int64_t vocab, const acb_pattern_filter *filter, void *stream);

/*
 * Vocabulary masks: for each row of token-id histories, the next ids whose BYTES would complete a pattern of a byte
 * (or UTF-8 string) automaton.  A vocabulary is n_vocab byte strings: vocab[t] holds the bytes of id t (an entry may
 * be empty).  Row i's history C is dev_tokens[a, b), clamped exactly as for acb_completions_mask.  An id outside
 * [0, n_vocab) (a negative pad, say) is a BREAK: it decodes to nothing and no occurrence may span it.  An empty entry
 * neither breaks nor adds bytes.  T = the bytes of C after its last break (only its last max_pattern_len - 1 bytes can
 * matter).  Id t COMPLETES a pattern for the row when some admitted pattern (all, or with a filter the row's set)
 * occurs in T || vocab[t] with its end inside vocab[t]: a Standard overlapping search of T || vocab[t] by an automaton
 * of the admitted patterns has a match ending past len(T).  So a token that holds a pattern is banned after every
 * history, an empty entry never is, and the answer does not depend on the automaton's match kind.  The candidates are
 * t < min(vocab, n_vocab): columns at or above n_vocab are never written; ids at or above vocab still decode in
 * histories.  Masking before every sampling step keeps every sampled token from ending a pattern in the decoded text.
 *
 * The vocabulary image (csrc/vocab.h) holds a Standard dense DFA (a copy of the automaton's own when its kind is
 * Standard; otherwise one built once from its patterns and kept with the automaton), the depth of every state, each
 * id's offset and length, each id's tail_hit (the last byte at which the walk from the root over vocab[t] enters a
 * match state, -1 for none) and the entry bytes.  blob holds the entries back to back, entry t at
 * blob[offsets[t], offsets[t + 1]); offsets = u64[n_vocab + 1] with offsets[0] = 0, non-decreasing.  The format's 32-bit
 * index widths hold at most ACB_VOCAB_MAX_IDS ids and ACB_VOCAB_MAX_BYTES entry bytes.  acb_vocab_build checks the
 * vocabulary and writes the image's size to *image_bytes (it reads the offsets, not the bytes); acb_vocab_write writes
 * the image (ACB_ECAPACITY when dst_bytes is short); the caller uploads it and passes the device pointer as dev_image.
 * acb_vocab_describe reads a host copy: n_vocab, the DFA's states and columns, max_pattern_len, the bytes of a DFA
 * built for the vocabulary (0 when it copies the automaton's own) and the ids with tail_hit >= 0.  ACB_EINVAL for a
 * null pointer (blob may be null when the entries hold no bytes), n_vocab above ACB_VOCAB_MAX_IDS, offsets[0] != 0,
 * decreasing offsets or more than ACB_VOCAB_MAX_BYTES bytes; ACB_EBUILD when the Standard DFA cannot be built.
 *
 * acb_vocab_mask writes logits[i * row_stride + t] = value (rounded to the logits dtype) for every completing id t of
 * row i; every other element is untouched.  dev_image must be the upload of acb_vocab_write(a, ...) for this `a`.
 * dev_state = u32[n_rows], the caller's scratch (the rows' DFA states between the two launches).  Logits as for
 * acb_completions_mask; any vocab >= 1 is valid.  Two launches (the rows' states, then the mask), no synchronisation,
 * no allocation.  ACB_EINVAL, before any CUDA call: a null pointer (dev_tokens may be null when n_tokens == 0, the
 * per-row pointers when n_rows == 0), token_bytes not 2, 4 or 8, n_tokens >= 2^60, n_rows outside [0, 2^32 - 2], a
 * malformed filter or one of 2^32 - 1 sets or more, a logits_dtype not listed, vocab outside [1, 2^62) or row_stride
 * outside [0, 2^62).  n_rows == 0 launches nothing.
 *
 * acb_vocab_stop finds each row's stop string: the first of its new ids whose bytes end an admitted pattern.  Row i is
 * clamped as for acb_vocab_mask; its last n = min(max(new_i, 0), b - a) ids are new, new_i = dev_new[i] (int64[n_rows])
 * or n_new when dev_new is null, the first at f = (b - a) - n.  Decoding the row (each break starts a fresh text), an
 * occurrence of an admitted pattern counts when a Standard overlapping search of its break-free text finds it and its
 * last byte lies in a new id's bytes; it may start in older ids.  The stop is the counted occurrence with the earliest
 * last byte, then the longest, then the lowest pid.  dev_out = int64[n_rows * 4]: row i gets (pattern, token, end,
 * length): `token` the index from a of the id holding the match's last byte (>= f), `end` that id's bytes up to and
 * including it (1 .. its length), `length` the pattern's bytes; -1 four times for none.  The answer does not depend on
 * the automaton's match kind.  For n = 1, row h || [t] has a stop exactly when acb_vocab_mask bans t after h under the
 * same filter.  One launch, no synchronisation, no allocation.  ACB_EINVAL, before any CUDA call: a null pointer (as
 * for acb_vocab_mask; dev_new may be null), token_bytes not 2, 4 or 8, n_tokens >= 2^60, n_rows outside
 * [0, 2^32 - 2], a malformed filter, or n_new < 0 when dev_new is null.  n_rows == 0 launches nothing.
 */
#define ACB_VOCAB_MAX_IDS 0x7fffffffull
#define ACB_VOCAB_MAX_BYTES 0x7fffffffull
typedef struct acb_vocab_desc {
    uint32_t n_vocab;
    uint32_t states;            /* of the Standard DFA */
    uint32_t columns;
    uint32_t max_pattern_len;   /* bytes; 0 without patterns */
    uint64_t extra_dfa_bytes;   /* a DFA built for the vocabulary (the automaton's kind is not Standard); 0 otherwise */
    uint32_t tail_hit_ids;      /* ids whose own bytes enter a match state from the root */
    uint32_t reserved;
} acb_vocab_desc;
int acb_vocab_build(acb_automaton *a, const uint8_t *blob, const uint64_t *offsets, uint64_t n_vocab, uint64_t *image_bytes);
int acb_vocab_write(acb_automaton *a, const uint8_t *blob, const uint64_t *offsets, uint64_t n_vocab, void *host_dst, uint64_t dst_bytes);
int acb_vocab_describe(const void *host_image, acb_vocab_desc *desc);
int acb_vocab_mask(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                   const int64_t *dev_offsets, int64_t n_rows, uint32_t *dev_state, void *dev_logits, int logits_dtype, int64_t row_stride,
                   int64_t vocab, float value, const acb_pattern_filter *filter, void *stream);
int acb_vocab_stop(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                   const int64_t *dev_offsets, int64_t n_rows, int64_t n_new, const int64_t *dev_new, int64_t *dev_out,
                   const acb_pattern_filter *filter, void *stream);

/*
 * Multi-GPU: the fixed-size block a rank contributes to the gather of the per-shard match lists (the only exchange
 * of the sharded path; NCCL all-gather over NVLink).  dev_block holds (cap + 1) records of 16 bytes: record 0 =
 * (match count, hay_base, complete flag, 0), then the first `cap` matches of a finished scan (dev_total / dev_out of
 * its workspace).  One launch on `stream`, no host round trip.
 */
int acb_pack_gather_block(const uint64_t *dev_total, const acb_match *dev_out, uint32_t hay_base, uint64_t cap, void *dev_block,
                          void *stream);

/* Kernel launch bookkeeping for bench.py's "gpu_launches". */
uint64_t acb_launch_count(void);

/*
 * Device-side timing of the scan kernel alone (CUDA events recorded on the
 * caller's stream around the scan kernel of every subsequent scan call), for
 * the roofline figure.  acb_timing_read synchronises on the recorded events,
 * returns their summed duration and count, and clears them.
 */
int acb_timing_enable(int on);
int acb_timing_read(double *total_ms, uint64_t *n_scans);

/* Tuning knobs (0 = library default), per calling thread. Affects speed only, never results. */
typedef struct acb_tuning {
    int kernel;        /* 0 auto (the sieve when dev_sieve is given), 1 = plain (one thread per haystack, table in global/L2),
                          2 = staged segments (hot rows in shared memory), 3 = staged, two segments per lane, 4 = segments
                          straight from global/L2, 5 = sieve (position-parallel filter + exact verification) */
    int hot_rows;      /* cap on rows kept in shared memory */
    int segment_bytes; /* segment size (rounded up to a multiple of 64 and to 8 x the warm-up); kernel 5: task size (multiple of 512) */
    int table;         /* 0 auto, 1 = column-indexed compact table only, 2 = byte-indexed 128-wide table when available */
    int sieve_ring;    /* cap on the sieve's ring depth (512-byte windows of text each warp keeps in shared memory), rounded
                          down to a power of two in [1, 8] (0 or less: as many as fit); it never raises the ring above what
                          fits next to the filters (see acb_sieve_ring) */
} acb_tuning;
int acb_set_tuning(const acb_tuning *t);

/*
 * The ring depth every sieve scan on this thread runs with for filters of bloom_bytes (acb_sieve_desc.bloom_bytes) on
 * a device with smem_optin bytes of opt-in shared memory per block: the largest power of two up to 8 whose ring fits
 * next to the filters, capped by the calling thread's acb_tuning.sieve_ring.  0 = the filters do not fit at all.
 */
uint32_t acb_sieve_ring(uint32_t bloom_bytes, uint32_t smem_optin);

#ifdef __cplusplus
}
#endif
#endif /* ACB200_H */
