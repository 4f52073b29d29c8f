/*
 * acb200.h -- C ABI of the GPU-native Aho-Corasick search path (libacb200.so).
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference has no
 * FFI in-tree; the seam its hot path sits behind is the sealed trait
 * `unsafe trait Automaton` (src/automaton.rs:198) reached from `AhoCorasick`
 * through `Arc<dyn AcAutomaton>` (src/ahocorasick.rs:177-180) with exactly two
 * virtual entry points on the search path -- `try_find` and
 * `try_find_overlapping` (src/ahocorasick.rs:2757-2772).  Every export below
 * cites the reference interface it replaces.  Plain pointers and sizes only,
 * no exceptions/panics cross the boundary, handles are immutable after
 * creation and safe for concurrent searches (the reference's automata are
 * Send + Sync, src/lib.rs:274-326).
 *
 * There is no CPU fallback: every search entry point returns ACG_E_CUDA /
 * ACG_E_NO_DEVICE if no CUDA device is usable.
 */
#ifndef ACB200_H
#define ACB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* src/util/search.rs:1052 MatchKind */
enum { ACG_STANDARD = 0, ACG_LEFTMOST_FIRST = 1, ACG_LEFTMOST_LONGEST = 2 };
/* src/util/search.rs:1133 StartKind */
enum { ACG_START_UNANCHORED = 0, ACG_START_ANCHORED = 1, ACG_START_BOTH = 2 };
/* src/ahocorasick.rs:2624 AhoCorasickKind (0 = None / auto, :2213-2261) */
enum { ACG_KIND_AUTO = 0, ACG_KIND_NONCONTIGUOUS_NFA = 1, ACG_KIND_CONTIGUOUS_NFA = 2, ACG_KIND_DFA = 3 };
/* which prefilter the reference would have built, src/util/prefilter.rs:163-305 */
enum { ACG_PRE_NONE = 0, ACG_PRE_MEMMEM = 1, ACG_PRE_START_BYTES = 2, ACG_PRE_RARE_BYTES = 3, ACG_PRE_PACKED = 4 };
/* device engines (acg_set_engine / acg_last_engine) */
enum {
  ACG_ENGINE_AUTO = 0,
  ACG_ENGINE_WALK = 1,      /* sharded DFA state-transition scan (K1) */
  ACG_ENGINE_PREFILTER = 2, /* k-gram prefilter + anchored DFA verify (K3/K3b), the packed/Teddy role */
  ACG_ENGINE_SEQUENTIAL = 3 /* single-lane restatement of the reference loop (anchored inputs, empty patterns) */
};

/* Error convention: 0 = OK; negative codes map 1:1 to BuildError
 * (src/util/error.rs:23-49) and MatchErrorKind (:200-223), plus boundary codes. */
enum {
  ACG_OK = 0,
  ACG_E_STATE_ID_OVERFLOW = -1,
  ACG_E_PATTERN_ID_OVERFLOW = -2,
  ACG_E_PATTERN_TOO_LONG = -3,
  ACG_E_INVALID_INPUT_ANCHORED = -10,
  ACG_E_INVALID_INPUT_UNANCHORED = -11,
  ACG_E_UNSUPPORTED_STREAM = -12,
  ACG_E_UNSUPPORTED_OVERLAPPING = -13,
  ACG_E_UNSUPPORTED_EMPTY = -14,
  ACG_E_INVALID_SPAN = -20, /* the reference panics, src/util/search.rs:332-343 */
  ACG_E_OVERFLOW = -21,     /* out buffer too small; *n_out holds the required count */
  ACG_E_INVALID_ARG = -22,
  ACG_E_CUDA = -30,
  ACG_E_NO_DEVICE = -31,
  ACG_E_NOMEM = -32
};

/* `Match { pattern: PatternID, span: Span }`, src/util/search.rs:825-830 */
typedef struct {
  uint32_t pid;
  uint32_t _pad;
  uint64_t start;
  uint64_t end;
} acg_match;

/* AhoCorasickBuilder knobs, src/ahocorasick.rs:2135-2617 */
typedef struct {
  int32_t match_kind;             /* default ACG_STANDARD */
  int32_t start_kind;             /* default ACG_START_UNANCHORED */
  int32_t ascii_case_insensitive; /* default 0 */
  int32_t byte_classes;           /* default 1 */
  int32_t prefilter;              /* default 1 */
  int32_t kind;                   /* default ACG_KIND_AUTO; the device always executes a DFA */
  int64_t dense_depth;            /* accepted for API parity; has no effect on a DFA */
} acg_build_opts;

/* The data `DFA` exposes through the Automaton trait (src/dfa.rs:91-132,
 * 192-302).  This is what a Rust `-sys` shim passes after building the
 * automaton with the reference's own builder. */
typedef struct {
  const uint32_t* trans;        /* premultiplied next-state ids, row-major [state_len][1<<stride2] */
  uint64_t trans_len;
  uint32_t stride2;
  uint32_t alphabet_len;
  uint8_t byte_classes[256];
  uint32_t max_special_id, max_match_id, start_unanchored_id, start_anchored_id;
  const uint32_t* match_offsets; /* CSR over match states 2..=max_match_id>>stride2: [n+1] */
  const uint32_t* match_pids;
  const uint32_t* pattern_lens;
  uint32_t n_patterns;
  uint32_t match_kind;
  uint32_t start_kind;
  uint32_t prefilter_kind;       /* informative (ACG_PRE_*) */
  uint64_t min_pattern_len, max_pattern_len;
} acg_dfa_desc;

typedef struct acg_dfa acg_dfa;

void acg_build_opts_default(acg_build_opts* o);

/* AhoCorasickBuilder::build (src/ahocorasick.rs:2171-2207) with kind=DFA:
 * noncontiguous construction (src/nfa/noncontiguous.rs:963-1051) followed by
 * dfa::Builder::build_from_noncontiguous (src/dfa.rs:431-540), then upload.
 * The host tables are bit-identical to the reference's. */
int acg_build(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
              const acg_build_opts* opts, acg_dfa** out);
/* Same, host tables only (no CUDA needed): for table-parity checks. Searches
 * on such a handle return ACG_E_NO_DEVICE. */
int acg_build_host(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                   const acg_build_opts* opts, acg_dfa** out);
/* acg_build with the dense transition table produced on the GPU (SURVEY section 8f.2): the host
 * runs the noncontiguous construction (trie, failure links, match lists, state permutation:
 * src/nfa/noncontiguous.rs:963-1481) and ships that compact form; the cells of
 * dfa::Builder::finish_build_one_start (src/dfa.rs:544-593) -- next_state for every (state, class)
 * -- are filled by a kernel, one launch per trie level, each row inheriting the finished row of
 * its failure state.  Same table bit for bit (acg_dfa_table fetches it back on demand); nothing of
 * size state_len x stride is built on or copied from the host.  Applies to StartKind::Unanchored
 * (the other start kinds take the acg_build path). */
int acg_build_on_device(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                        const acg_build_opts* opts, acg_dfa** out);
/* Adopt a DFA built by the reference itself (pointers borrowed for the call). */
int acg_dfa_create(const acg_dfa_desc* desc, acg_dfa** out);
void acg_dfa_free(acg_dfa* dfa);

/* Host view of the tables held by the handle (borrowed until acg_dfa_free). */
int acg_dfa_table(const acg_dfa* dfa, acg_dfa_desc* out);
uint64_t acg_dfa_state_len(const acg_dfa* dfa);
/* getters, src/ahocorasick.rs:1867-2021 */
int acg_kind(const acg_dfa* dfa); /* what AhoCorasick::kind() would report for these options */
int acg_match_kind(const acg_dfa* dfa);
int acg_start_kind(const acg_dfa* dfa);
uint64_t acg_patterns_len(const acg_dfa* dfa);
uint64_t acg_min_pattern_len(const acg_dfa* dfa);
uint64_t acg_max_pattern_len(const acg_dfa* dfa);
uint64_t acg_memory_usage(const acg_dfa* dfa);
int acg_prefilter_kind(const acg_dfa* dfa);
/* Teddy variant the reference would pick (src/packed/teddy/builder.rs:98-231); 0 if not packed */
int acg_packed_variant(const acg_dfa* dfa, int* fat, int* mask_len);

/* Engine override (default AUTO) and introspection for tests/bench. */
int acg_set_engine(acg_dfa* dfa, int engine);
int acg_last_engine(const acg_dfa* dfa);

/* ---- searches over HOST buffers (copies are part of the call) ------------- */

/* AhoCorasick::try_find_overlapping_iter(...).collect()
 * (src/ahocorasick.rs:1350 -> src/automaton.rs:397-423, 954-970, 1423-1537):
 * all matches in the reference's iteration order. Two-call protocol on
 * ACG_E_OVERFLOW. */
int acg_find_overlapping(const acg_dfa* dfa, const uint8_t* hay, uint64_t hay_len,
                         uint64_t span_start, uint64_t span_end, int anchored,
                         acg_match* out, uint64_t cap, uint64_t* n_out);
/* AhoCorasick::try_find_iter(...).collect()
 * (src/ahocorasick.rs:1275 -> src/automaton.rs:844-936, 1259-1420). */
int acg_find_iter(const acg_dfa* dfa, const uint8_t* hay, uint64_t hay_len,
                  uint64_t span_start, uint64_t span_end, int anchored,
                  acg_match* out, uint64_t cap, uint64_t* n_out);
/* AhoCorasick::try_find (src/ahocorasick.rs:1021) / is_match (:311, earliest=1). */
int acg_find(const acg_dfa* dfa, const uint8_t* hay, uint64_t hay_len,
             uint64_t span_start, uint64_t span_end, int anchored, int earliest,
             acg_match* out, int* found);

/* ---- searches over DEVICE-resident haystacks (roofline measurement; no H2D) -
 * d_hay points at haystack byte 0 in device memory.  Results are written to the
 * host array `out` (matches are sparse); *kernel_ms, if non-NULL, receives the
 * CUDA-event time of the scan kernels on the library's stream. */
int acg_find_overlapping_dev(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                             uint64_t span_start, uint64_t span_end,
                             acg_match* out, uint64_t cap, uint64_t* n_out, float* kernel_ms);
int acg_find_iter_dev(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                      uint64_t span_start, uint64_t span_end,
                      acg_match* out, uint64_t cap, uint64_t* n_out, float* kernel_ms);
/* Same as acg_find_overlapping_dev but the ordered matches stay on the device: d_out is a device
 * array of acg_match (cap entries); only matches with end > min_end are kept (shard ownership
 * by end offset, SURVEY.md section 8e) and `offset_add` is added to start/end (global offsets of
 * a sliced haystack).  *n_out receives the number written.  Feeds the NCCL gather directly. */
int acg_find_overlapping_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                                uint64_t span_start, uint64_t span_end, uint64_t min_end,
                                uint64_t offset_add, void* d_out, uint64_t cap, uint64_t* n_out,
                                float* kernel_ms);
/* Count-only variants: scan + order on the device, return the number of matches
 * and an FNV-1a checksum of the ordered (pid,start,end) stream computed on the
 * device-ordered tuples (host side folds it).  `d_out`/cap may be 0/NULL. */
int acg_count_overlapping_dev(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                              uint64_t span_start, uint64_t span_end,
                              uint64_t* n_out, uint64_t* fnv, float* kernel_ms);

/* ---- batched search: many independent documents in one call -----------------
 * A batch is one byte buffer plus CSR offsets doc_offsets[n_docs + 1] (host memory, non-decreasing,
 * doc_offsets[n_docs] <= hay_len); document d is hay[doc_offsets[d] .. doc_offsets[d + 1]), empty
 * documents allowed.  For every d, the records tagged doc == d are exactly what the single-haystack
 * call returns on that document alone -- same (pid, start, end), offsets relative to the document's
 * first byte, same order -- and the records appear in ascending d.  Error codes are those of the
 * single calls; decreasing offsets or offsets past hay_len give ACG_E_INVALID_SPAN, n_docs >= 2^32
 * ACG_E_INVALID_ARG.  hay_on_device != 0: `hay` is a device pointer to byte 0.  Results go to host
 * memory; two-call protocol on ACG_E_OVERFLOW (*n_out holds the required count).
 * Engine: the prefilter engine when the automaton has a prefilter plan and the input is unanchored,
 * else (and with ACG_ENGINE_SEQUENTIAL) one thread per document running the reference's loop --
 * a single very long document is then one thread's sequential walk. */
typedef struct {
  uint32_t pid;
  uint32_t doc; /* acg_match layout, the document index in the pad */
  uint64_t start;
  uint64_t end;
} acg_doc_match;
/* AhoCorasick::try_find_iter(doc) for every document */
int acg_find_iter_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                        const uint64_t* doc_offsets, uint64_t n_docs, int anchored,
                        acg_doc_match* out, uint64_t cap, uint64_t* n_out);
/* AhoCorasick::try_find_overlapping_iter(doc) for every document */
int acg_find_overlapping_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                               const uint64_t* doc_offsets, uint64_t n_docs, int anchored,
                               acg_doc_match* out, uint64_t cap, uint64_t* n_out);
/* AhoCorasick::is_match(doc) for every document: flags[d] = 0 / 1 */
int acg_is_match_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                       const uint64_t* doc_offsets, uint64_t n_docs, int anchored, uint8_t* flags);
/* AhoCorasick::try_find(Input::new(doc).anchored(a).earliest(e)) for every document.
 * found[d] = 1 and out[d] = {pid, d, start, end} (offsets relative to the document) when the
 * single-haystack acg_find on document d alone, span (0, len), reports a match; otherwise
 * found[d] = 0 and out[d] = {0, d, 0, 0}.  Both arrays have n_docs entries in host memory.
 * One output slot per document: no overflow protocol.  `earliest` follows acg_find, including its
 * packed-prefilter rule; an ACG_ENGINE_PREFILTER override the input cannot use (anchored, no
 * prefilter plan, `earliest` on a leftmost automaton) gives ACG_E_INVALID_ARG. */
int acg_find_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                   const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int earliest,
                   acg_doc_match* out, uint8_t* found);

/* Batched search with device-resident inputs and results.  d_hay: device pointer to byte 0.
 * doc_offsets: [n_docs + 1] CSR bounds, in host memory (offsets_on_device == 0) or device memory
 * (!= 0, 8-byte aligned); device offsets are used by the kernels where they are, without a copy.
 * Same contract and error codes as the acg_*_batch calls above:
 * - per document, the same records in the same order;
 * - decreasing offsets or offsets past hay_len give ACG_E_INVALID_SPAN, detected on the device
 *   when the offsets are there;
 * - n_docs >= 2^32 gives ACG_E_INVALID_ARG.
 * All outputs are device pointers.  The call returns once they are written.
 * find_iter / overlapping: d_out[0 .. *n_out) holds the acg_doc_match records, in the order and
 * layout acg_*_batch writes to host memory, and d_match_offsets[n_docs + 1] their CSR index by
 * document: the records of document d are d_out[d_match_offsets[d] .. d_match_offsets[d + 1]).
 * If *n_out > cap the call returns ACG_E_OVERFLOW with the required count in *n_out and writes
 * neither array (two-call protocol).  n_out is a host pointer: the only result that crosses to the
 * host.  is_match / find: d_flags / d_found and d_out have n_docs entries, as in acg_is_match_batch /
 * acg_find_batch. */
int acg_find_iter_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                               const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                               int anchored, acg_doc_match* d_out, uint64_t cap,
                               uint64_t* d_match_offsets, uint64_t* n_out);
int acg_find_overlapping_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                                      const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                                      int anchored, acg_doc_match* d_out, uint64_t cap,
                                      uint64_t* d_match_offsets, uint64_t* n_out);
int acg_is_match_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                              const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                              int anchored, uint8_t* d_flags);
int acg_find_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                          const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                          int anchored, int earliest, acg_doc_match* d_out, uint8_t* d_found);

/* How often each pattern occurs in each document of a batch, as a sparse CSR matrix
 * [n_docs x patterns_len].  Let R be the records acg_find_overlapping_batch (overlapping != 0) or
 * acg_find_iter_batch (overlapping == 0) returns for the same dfa, haystack, offsets and anchored.
 * Document d's entries are pids[row_offsets[d] .. row_offsets[d + 1]), strictly ascending;
 * counts[i] (>= 1) is the number of records of R with doc == d and pid == pids[i].
 * *nnz = row_offsets[n_docs] = number of distinct (doc, pid) pairs in R.
 * row_offsets has n_docs + 1 entries, pids and counts cap entries each.  If *nnz > cap the call
 * returns ACG_E_OVERFLOW with the required count in *nnz and writes none of the three arrays;
 * cap == 0 with NULL pids / counts is a size query.  Error codes, their order and the engine are
 * those of the batch call `overlapping` selects.  The counts are computed on the device without
 * materialising the records: the result's size depends on the number of distinct pairs only.
 * _devout: the three arrays are device pointers, doc_offsets as in the other _devout calls; nnz is
 * a host pointer. */
int acg_pattern_counts_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int overlapping,
                             uint64_t* row_offsets, uint32_t* pids, uint64_t* counts, uint64_t cap,
                             uint64_t* nnz);
int acg_pattern_counts_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                                    const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                                    int anchored, int overlapping, uint64_t* d_row_offsets,
                                    uint32_t* d_pids, uint64_t* d_counts, uint64_t cap, uint64_t* nnz);

/* How much of each document of a batch its matches cover.  Let R be the records
 * acg_find_overlapping_batch (overlapping != 0) or acg_find_iter_batch (overlapping == 0) returns
 * for the same dfa, haystack, offsets and anchored.  covered[d] (n_docs entries) is the number of
 * bytes of document d that lie in [start, end) of at least one record of R with doc == d: the
 * size of the union of the matches, not the sum of their lengths; empty matches cover nothing.
 * mask (optional, NULL for none) is indexed like hay: for every i in
 * [doc_offsets[0], doc_offsets[n_docs]) mask[i] = 1 if byte i lies in a match of its document
 * and 0 otherwise; entries outside that range are left untouched.  The output has a fixed size,
 * so there is no overflow protocol.  Error codes, their order and the engine are those of the
 * batch call `overlapping` selects; a NULL covered with n_docs > 0 is ACG_E_INVALID_ARG, and
 * n_docs == 0 writes nothing.  The union is computed on the device from the matches, without
 * materialising the records.
 * _devout: covered and mask are device pointers, doc_offsets as in the other _devout calls. */
int acg_match_coverage_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int overlapping,
                             uint64_t* covered, uint8_t* mask);
int acg_match_coverage_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                                    const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                                    int anchored, int overlapping, uint64_t* d_covered, uint8_t* d_mask);

/* replace_all_bytes of every document of a batch.  Let R be the records acg_find_iter_batch
 * returns for the same dfa, haystack and offsets with anchored = 0.  Document d's result is
 * document d with every record of R of that document replaced by its pattern's replacement, in
 * order, as the reference's try_replace_all_bytes builds it: the bytes before the first match,
 * the replacement, the bytes between the first and the second match, ..., the bytes after the
 * last one.  Empty matches insert their replacement; replacements are not searched again.
 * Replacement i (n_reps == patterns_len entries) is rep_bytes[rep_offsets[i] .. rep_offsets[i + 1]);
 * the table is in host memory for both calls.  n_reps != patterns_len, decreasing rep_offsets, a
 * NULL rep_offsets or a NULL rep_bytes with replacement bytes give ACG_E_INVALID_ARG.
 * The results are in the CSR form every batch call takes: document d's bytes are
 * out[out_offsets[d] .. out_offsets[d + 1]), out_offsets has n_docs + 1 entries, out_offsets[0] = 0
 * and *out_len = out_offsets[n_docs].  If *out_len > cap the call returns ACG_E_OVERFLOW with the
 * required size in *out_len and writes neither out nor out_offsets; cap == 0 with a NULL out is a
 * size query.  A NULL out with cap > 0, a NULL out_offsets or a NULL out_len is ACG_E_INVALID_ARG.
 * Otherwise the error codes, their order and the engine are those of acg_find_iter_batch with
 * anchored = 0 (an automaton built with ACG_START_ANCHORED gives ACG_E_INVALID_INPUT_UNANCHORED).
 * n_docs == 0 writes out_offsets[0] = 0 and *out_len = 0.  The output is spliced on the device
 * from the matches, without materialising the records.
 * out must not overlap the haystack: the input is still read while the output is written.
 * _devout: out and out_offsets are device pointers, doc_offsets as in the other _devout calls;
 * out_len is a host pointer. */
int acg_replace_all_batch(const acg_dfa* dfa, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                          const uint64_t* doc_offsets, uint64_t n_docs,
                          const uint8_t* rep_bytes, const uint64_t* rep_offsets, uint64_t n_reps,
                          uint8_t* out, uint64_t cap, uint64_t* out_offsets, uint64_t* out_len);
int acg_replace_all_batch_devout(const acg_dfa* dfa, const void* d_hay, uint64_t hay_len,
                                 const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                                 const uint8_t* rep_bytes, const uint64_t* rep_offsets, uint64_t n_reps,
                                 uint8_t* d_out, uint64_t cap, uint64_t* d_out_offsets, uint64_t* out_len);

/* ---- stream sets: many byte streams, each searched as its bytes arrive ----------------------
 * A stream set holds n_streams streams over one automaton, in find_iter mode (overlapping == 0:
 * the matches of try_find_iter, Standard semantics) or overlapping mode (the matches of
 * try_find_overlapping_iter).  Let X_s be the bytes stream s has received since the set was
 * created or the stream was last reset.  A feed takes one chunk per stream, in the batch form:
 * chunk s is hay[chunk_offsets[s] .. chunk_offsets[s + 1]), empty chunks allowed.  A successful
 * feed that takes X_s from n0 to n1 bytes returns, for every s, exactly the matches of the mode's
 * iterator over all of X_s whose end lies in (n0, n1], as acg_doc_match records with doc = s and
 * start / end absolute offsets into X_s, in ascending s and, within a stream, in the iterator's
 * order.  So a stream's records over all its feeds, concatenated, are the iterator over X_s, and
 * in find_iter mode also what try_stream_find_iter yields over X_s: a match that starts in one
 * feed's bytes and ends in a later one's is returned once, by the later feed.
 * Creation (the restrictions of StreamChunkIter::new and try_find_overlapping_iter):
 * - a leftmost automaton gives ACG_E_UNSUPPORTED_STREAM (find_iter) or
 *   ACG_E_UNSUPPORTED_OVERLAPPING (overlapping);
 * - an automaton with the empty pattern gives ACG_E_UNSUPPORTED_EMPTY;
 * - an automaton built with ACG_START_ANCHORED gives ACG_E_INVALID_INPUT_UNANCHORED;
 * - n_streams == 0 or n_streams >= 2^32 gives ACG_E_INVALID_ARG;
 * - ACG_E_NOMEM when the state does not fit: 16 bytes and max_pattern_len - 1 tail bytes per
 *   stream, on the automaton's device.  The automaton must outlive the set.
 * Feeds: hay_on_device != 0 (always for _devout): hay is a device pointer to byte 0.  Decreasing
 * chunk offsets or offsets past hay_len give ACG_E_INVALID_SPAN (detected on the device when the
 * offsets are there); n_streams other than the set's, a NULL n_out, a NULL out with cap > 0 or a
 * NULL d_match_offsets give ACG_E_INVALID_ARG.  If *n_out > cap the call returns ACG_E_OVERFLOW
 * with the required count in *n_out and writes nothing (two-call protocol): a retry with room
 * returns what the first call would have.  Every error leaves every stream as it was, except
 * ACG_E_CUDA, after which the set's state is undefined until acg_streams_reset(set, NULL, 0).
 * _devout: d_out and d_match_offsets[n_streams + 1] (the CSR index of the records by stream, as in
 * the batch _devout calls) are device pointers, chunk_offsets as doc_offsets there; n_out is a
 * host pointer.  The engine is that of the batch calls, chosen per feed.
 * One call at a time per set (feed, reset, positions): the caller serialises them.  Different sets,
 * also on one automaton, may be fed from different threads at once.
 * acg_streams_reset: ids (host memory, n_ids entries) restart from zero bytes; ids == NULL resets
 * every stream.  An id >= n_streams gives ACG_E_INVALID_ARG and resets none.
 * acg_streams_positions: pos[s] = the length of X_s, pos in host memory with n_streams entries. */
typedef struct acg_streams acg_streams;
int acg_streams_create(const acg_dfa* dfa, uint64_t n_streams, int overlapping, acg_streams** out);
void acg_streams_free(acg_streams* set);
int acg_streams_reset(acg_streams* set, const uint64_t* ids, uint64_t n_ids);
int acg_streams_positions(const acg_streams* set, uint64_t* pos);
int acg_streams_feed(acg_streams* set, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                     const uint64_t* chunk_offsets, uint64_t n_streams, acg_doc_match* out, uint64_t cap,
                     uint64_t* n_out);
int acg_streams_feed_devout(acg_streams* set, const void* d_hay, uint64_t hay_len, const uint64_t* chunk_offsets,
                            int offsets_on_device, uint64_t n_streams, acg_doc_match* d_out, uint64_t cap,
                            uint64_t* d_match_offsets, uint64_t* n_out);

/* ---- replace sets: try_stream_replace_all over many streams, spliced on the device ----------
 * A replace set is a find_iter stream set that writes text instead of records.  For stream s let
 * X_s be the bytes it has received since creation, its last reset or its last flush, pos_s = |X_s|,
 * c_s the end of the last find_iter match of X_s (0 if none), and h_s = max(c_s, pos_s -
 * (max_pattern_len - 1)), floored at 0: the emit boundary.  Everything before h_s is settled; the
 * held bytes X_s[h_s, pos_s), at most max_pattern_len - 1 of them, hold no match yet.
 * acg_streams_create_replace: the checks of acg_streams_create in find_iter mode, in its order, then
 * the replacement table as acg_replace_all_batch checks it (one per pattern, offsets that do not
 * decrease, rep_bytes non-NULL when there are bytes; else ACG_E_INVALID_ARG), then ACG_E_NOMEM.  The
 * table is copied to the device; the caller's arrays are not kept.
 * acg_streams_replace_feed(_devout): a feed in the form of acg_streams_feed(_devout) that takes stream
 * s from (pos, h) to (pos', h') writes X_s[h, h') with every find_iter match of X_s in that range
 * replaced by its pattern's replacement (empty ones delete; replacements are not searched again):
 * stream s's bytes are out[out_offsets[s] .. out_offsets[s + 1]), out_offsets[n_streams + 1],
 * out_offsets[0] = 0, *out_len = out_offsets[n_streams].  Every match lies wholly inside or outside
 * that range.  So a stream's outputs over all its feeds, followed by its flush, are
 * replace_all_bytes(X_s), what try_stream_replace_all writes for X_s.  The output is bytes: h may
 * split a multi-byte UTF-8 character between one feed's output and the next.  *out_len > cap
 * returns ACG_E_OVERFLOW with the required size, writes nothing and changes no stream.  The other
 * errors, their order and the offset rules are those of acg_streams_feed(_devout); a NULL
 * out_offsets is ACG_E_INVALID_ARG.  _devout: out and out_offsets are device pointers.  out must not
 * overlap the chunks.
 * acg_streams_flush: for each id in ids (ids == NULL: every stream, in order) the stream's held
 * bytes X_s[h, pos), raw, in the same CSR form into host memory (n_ids + 1 or n_streams + 1
 * offsets); those streams then restart from zero bytes.  An id >= n_streams, a duplicate id, a NULL
 * out_offsets or out_len, or a NULL out with cap > 0 gives ACG_E_INVALID_ARG and touches no stream;
 * *out_len > cap gives ACG_E_OVERFLOW with the required size and resets no stream.
 * acg_streams_held: held[s] = pos_s - h_s, held in host memory with n_streams entries.
 * acg_streams_positions, acg_streams_reset (which discards the held bytes unemitted) and
 * acg_streams_free take replace sets.  acg_streams_feed(_devout) on a replace set, and the calls
 * above on another set, give ACG_E_INVALID_ARG. */
int acg_streams_create_replace(const acg_dfa* dfa, uint64_t n_streams, const uint8_t* rep_bytes,
                               const uint64_t* rep_offsets, uint64_t n_reps, acg_streams** out);
int acg_streams_replace_feed(acg_streams* set, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* chunk_offsets, uint64_t n_streams, uint8_t* out, uint64_t cap,
                             uint64_t* out_offsets, uint64_t* out_len);
int acg_streams_replace_feed_devout(acg_streams* set, const void* d_hay, uint64_t hay_len,
                                    const uint64_t* chunk_offsets, int offsets_on_device, uint64_t n_streams,
                                    uint8_t* d_out, uint64_t cap, uint64_t* d_out_offsets, uint64_t* out_len);
int acg_streams_flush(acg_streams* set, const uint64_t* ids, uint64_t n_ids, uint8_t* out, uint64_t cap,
                      uint64_t* out_offsets, uint64_t* out_len);
int acg_streams_held(const acg_streams* set, uint64_t* held);

/* ---- lookahead: which of a fixed set of candidate chunks would complete a match ------------
 * A candidate set is a fixed list of byte strings (a tokenizer's vocabulary, say), uploaded once
 * and reused by every call: candidate i is bytes[offsets[i] .. offsets[i + 1]).
 * acg_candidates_create: n_cands >= 2^32, decreasing offsets, a NULL offsets or out, or a NULL
 * bytes with bytes to copy give ACG_E_INVALID_ARG; ACG_E_NOMEM when they do not fit.  The
 * candidates are copied to the automaton's device, mapped through its byte classes, so the set is
 * bound to that automaton, which must outlive it; the caller's arrays are not kept.
 * acg_streams_lookahead(_devout): for a stream or replace set whose stream s has received X_s
 * (pos_s = |X_s|), row k of the output is stream ids[k] (ids == NULL: n_streams rows, row k is
 * stream k; ids in host memory, duplicates and any order allowed), and
 *   out[k * n_cands + c] = 1 iff a feed that gave that stream candidate c as its chunk would
 *   return at least one match for it: the set's iterator (find_iter with its restart point, or
 *   overlapping; find_iter for a replace set) over X_s | c has a match whose end lies in
 *   (pos_s, pos_s + |c|]; else 0.
 * Empty candidates never match, so a caller whose logits are wider than its vocabulary pads the
 * list with empty candidates.  out holds n_rows * n_cands bytes, row-major, 0 or 1 each: host memory
 * for acg_streams_lookahead, device memory for _devout.  The call reads the streams and changes
 * none of them.  A candidate set from another automaton, a NULL set or candidate set, an id
 * >= n_streams, n_ids >= 2^32 or a NULL out with n_rows * n_cands > 0 give ACG_E_INVALID_ARG and
 * write nothing; a workspace that cannot grow gives ACG_E_NOMEM.  One call at a time per stream
 * set, as for feeds; a candidate set may be shared by concurrent calls on different sets.
 * acg_last_stats: the mask kernel in scan_ms, the rest of the device work (the rows' states, their
 * dedupe and the copy of shared rows) in order_ms. */
typedef struct acg_candidates acg_candidates;
int acg_candidates_create(const acg_dfa* dfa, const uint8_t* bytes, const uint64_t* offsets, uint64_t n_cands,
                          acg_candidates** out);
void acg_candidates_free(acg_candidates* cands);
int acg_streams_lookahead(const acg_streams* set, const acg_candidates* cands, const uint64_t* ids, uint64_t n_ids,
                          uint8_t* out);
int acg_streams_lookahead_devout(const acg_streams* set, const acg_candidates* cands, const uint64_t* ids,
                                 uint64_t n_ids, uint8_t* d_out);

/* ---- multi-GPU: haystack slices + gather of match buffers to rank 0 (SURVEY.md section 8e) ----
 * One process (or thread) per GPU.  The path shards naturally: rank g owns the matches whose END
 * lies in (own_lo, own_hi] (rank 0 also owns end == span_start: empty-pattern matches of the start
 * state, src/automaton.rs:1456-1464), scans [read_lo, own_hi) from a cold start with
 * read_lo = own_lo - (max_pattern_len - 1), and never exchanges haystack bytes.  The only
 * exchange is the gather of the per-rank match buffers to rank 0; concatenated in rank order they
 * are the list AhoCorasick::find_overlapping_iter yields on the whole haystack
 * (src/automaton.rs:954-970, 1423-1537).
 * Transport: the records are stored by each rank's expand kernel directly into rank 0's receive
 * buffer through a cudaIpc peer mapping (NVLink / NVSwitch); NCCL carries the 8-byte counts and the
 * closing barrier, and the payload too (ncclSend / ncclRecv) if the peer mapping is unavailable. */
enum { ACG_TRANSPORT_NONE = 0, ACG_TRANSPORT_PEER = 1, ACG_TRANSPORT_NCCL = 2 };
#define ACG_COMM_ID_BYTES 128
typedef struct acg_comm acg_comm;
/* Rank 0 creates the rendezvous token (an ncclUniqueId) and hands it to the other ranks by whatever
 * channel launched them (MPI, torch.distributed, a file). */
int acg_comm_unique_id(uint8_t id[ACG_COMM_ID_BYTES]);
/* Collective over all ranks; binds to the calling thread's current CUDA device. */
int acg_comm_init(const uint8_t id[ACG_COMM_ID_BYTES], int rank, int nranks, acg_comm** out);
void acg_comm_free(acg_comm* comm);
int acg_comm_rank(const acg_comm* comm);
int acg_comm_size(const acg_comm* comm);
int acg_comm_transport(const acg_comm* comm); /* ACG_TRANSPORT_* */
/* Slice of rank `rank` out of `nranks` for the span [span_start, span_end): the rank owns ends in
 * (own_lo, own_hi] and must hold the haystack bytes [read_lo, own_hi).  Pure arithmetic. */
int acg_shard_plan(uint64_t span_start, uint64_t span_end, int nranks, int rank, uint64_t max_pattern_len,
                   uint64_t* own_lo, uint64_t* own_hi, uint64_t* read_lo);
typedef struct {
  uint64_t local_matches;  /* records this rank contributed */
  uint64_t total_matches;  /* records in rank 0's buffer (known to every rank) */
  uint64_t candidates;
  float scan_ms, order_ms; /* this rank's scan kernel(s) / ordering */
  float gather_ms;         /* count exchange + expand into rank 0's buffer + closing barrier */
  int32_t transport;
  int32_t launches;
} acg_shard_stats;
/* Collective.  `hay` holds this rank's slice of the global haystack: its byte 0 is global offset
 * `hay_global_offset`, `hay_len` bytes are readable, and it must cover the rank's
 * [read_lo, own_hi) of acg_shard_plan for the span (ACG_E_INVALID_SPAN otherwise).  hay_on_device
 * != 0: `hay` is a device pointer on the communicator's device; 0: a host pointer (the copy is
 * pipelined with the scan, as in acg_find_overlapping).  On rank 0, *d_matches receives a device
 * pointer to *n_total acg_match records in GLOBAL offsets, in the reference's iteration order,
 * valid until the next call on this communicator; if h_out != NULL they are also copied to the host
 * (ACG_E_OVERFLOW with *n_total set if h_cap is too small; acg_comm_fetch then gets them without
 * another scan).  Other ranks receive NULL / the total. */
int acg_find_overlapping_sharded(const acg_dfa* dfa, acg_comm* comm, const void* hay, int hay_on_device,
                                 uint64_t hay_len, uint64_t hay_global_offset, uint64_t span_start,
                                 uint64_t span_end, const acg_match** d_matches, uint64_t* n_total,
                                 acg_match* h_out, uint64_t h_cap, acg_shard_stats* stats);
/* The same search in two halves, for callers that run one sharded search after another (a stream of
 * haystack batches): _begin returns once this rank's records are on their way into rank 0's buffer,
 * _wait completes the step.  Up to two steps may be in flight, so the scan of batch k + 1 overlaps
 * the NVLink transfer of batch k's records (rank 0's buffer has two halves; the records of a step
 * stay valid until the step after the next begins).  Both are collective; every rank must issue
 * begin / wait in the same order.  *ticket identifies the step for _wait. */
int acg_find_overlapping_sharded_begin(const acg_dfa* dfa, acg_comm* comm, const void* hay, int hay_on_device,
                                       uint64_t hay_len, uint64_t hay_global_offset, uint64_t span_start,
                                       uint64_t span_end, int* ticket);
int acg_find_overlapping_sharded_wait(acg_comm* comm, int ticket, const acg_match** d_matches, uint64_t* n_total,
                                      acg_match* h_out, uint64_t h_cap, acg_shard_stats* stats);
/* In the begin / wait form the records travel by copy engine: the expand kernel writes them into this
 * rank's own HBM and one device-to-device copy over NVLink puts them at their place in rank 0's
 * buffer, so the next step's scan has every SM while they are under way (the blocking call stores them
 * from the kernel itself, which is the shorter path for a single step).
 *
 * Device timestamps around a stream of steps: acg_comm_mark(comm, 0) before the first _begin and
 * acg_comm_mark(comm, 1) after the last _wait each wait for the device to drain and record a CUDA
 * event; acg_comm_mark_elapsed_ms gives the time between them on the device's clock. */
int acg_comm_mark(acg_comm* comm, int which);
int acg_comm_mark_elapsed_ms(const acg_comm* comm, float* ms);
/* Rank 0: copy the records of the most recent sharded search to the host; *n_out = their number. */
int acg_comm_fetch(const acg_comm* comm, acg_match* out, uint64_t cap, uint64_t* n_out);
/* Rank 0: the same records in page-locked host memory owned by the communicator (one full-speed
 * device-to-host copy, no staging through pageable memory); *view stays valid until the next
 * acg_comm_fetch_view or sharded search on this communicator. */
int acg_comm_fetch_view(acg_comm* comm, const acg_match** view, uint64_t* n_out);
/* Count + FNV-1a of the ordered (pid, start, end) stream of the most recent sharded search
 * (rank 0), comparable with acg_count_overlapping_dev on one GPU over the same haystack. */
int acg_comm_checksum(const acg_comm* comm, uint64_t* n_out, uint64_t* fnv);

/* ---- packed searcher: packed::Config / Builder / Searcher, src/packed/api.rs ----------------
 * The reference's standalone "packed" API is Teddy (or Rabin-Karp) over a small pattern set with
 * leftmost semantics.  On the device its role is played by the same K3/K3b kernel pair that serves
 * AhoCorasick (a fingerprint prefilter feeding the DFA verifier); what this API keeps from the
 * reference is the construction contract -- when Builder::build returns None -- and the search
 * results, which are the leftmost-first / leftmost-longest non-overlapping matches. */
enum { ACG_PACKED_FORCE_NONE = 0, ACG_PACKED_FORCE_TEDDY = 1, ACG_PACKED_FORCE_RABINKARP = 2 };
typedef struct {
  int32_t match_kind;               /* ACG_LEFTMOST_FIRST (default) | ACG_LEFTMOST_LONGEST, api.rs:28-46 */
  int32_t force;                    /* Config::only_teddy / only_rabin_karp, api.rs:143-190 */
  int32_t only_teddy_fat;           /* -1 = None, 0 / 1 = Some(false / true), api.rs:158 */
  int32_t only_teddy_256bit;        /* -1 = None, 0 / 1 = Some(false / true), api.rs:170 */
  int32_t heuristic_pattern_limits; /* default 1, api.rs:196 */
} acg_packed_config;
typedef struct acg_packed acg_packed;
void acg_packed_config_default(acg_packed_config* c);
/* Builder::extend + Builder::build (api.rs:253-345).  Returns ACG_OK with *out == NULL where the
 * reference returns None: no patterns, an empty pattern, more than 128 patterns, or a pattern set
 * Teddy declines (teddy/builder.rs:98-231, decided as on x86-64 with AVX2). */
int acg_packed_build(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                     const acg_packed_config* cfg, acg_packed** out);
/* Same decision and tables without CUDA; searches return ACG_E_NO_DEVICE. */
int acg_packed_build_host(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                          const acg_packed_config* cfg, acg_packed** out);
void acg_packed_free(acg_packed* s);
/* Searcher::find_iter (api.rs:580) -- and find_in (:529) applied repeatedly for a sub-span:
 * non-overlapping leftmost matches inside [span_start, span_end).  Two-call protocol on
 * ACG_E_OVERFLOW; ACG_E_INVALID_SPAN where the reference's slice indexing panics. */
int acg_packed_find_iter(const acg_packed* s, const uint8_t* hay, uint64_t hay_len,
                         uint64_t span_start, uint64_t span_end, acg_match* out, uint64_t cap,
                         uint64_t* n_out);
/* Searcher::find (api.rs:491) / find_in (:529). */
int acg_packed_find(const acg_packed* s, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
                    uint64_t span_end, acg_match* out, int* found);
int acg_packed_match_kind(const acg_packed* s);        /* api.rs:612 */
uint64_t acg_packed_minimum_len(const acg_packed* s);  /* api.rs:627: 0 for Rabin-Karp, else Teddy's */
uint64_t acg_packed_memory_usage(const acg_packed* s); /* api.rs:634 (heap of the device engine's tables) */
uint64_t acg_packed_patterns_len(const acg_packed* s);
/* Which searcher the reference would run: returns 1 for Teddy (and fills fat / mask_len /
 * vector_bytes), 0 for Rabin-Karp. */
int acg_packed_searcher_variant(const acg_packed* s, int* fat, int* mask_len, int* vector_bytes);

/* per-call statistics of the most recent search on this handle (bench glue) */
typedef struct {
  int32_t engine;
  int32_t launches;          /* kernels launched by the library in the call */
  uint64_t candidates;       /* prefilter survivors (ACG_ENGINE_PREFILTER) */
  uint64_t raw_matches;      /* tuples appended before ordering/stitching */
  float scan_ms;             /* dominant scan kernel(s) */
  float order_ms;            /* ordering / compaction */
  float h2d_ms;
  float d2h_ms;              /* expansion of the records and their copy to the host */
} acg_stats;
int acg_last_stats(const acg_dfa* dfa, acg_stats* out);

const char* acg_strerror(int code);
/* number of CUDA devices visible (0 if none / driver missing) */
int acg_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
