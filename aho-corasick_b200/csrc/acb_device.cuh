// acb_device.cuh -- device-side views shared by the kernels and the C-ABI layer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace acb {

// Packed 64-bit ordering key of one emitted match: (end - span_start) in the
// high 40 bits, a 24-bit tie-break in the low bits.  Sorting the keys ascending
// reproduces the reference's emission order:
//   * walk engine:      tie-break = index into the match state's pattern list
//                        (src/automaton.rs:1475-1481 reports list entries in order)
//   * prefilter engine: tie-break = (max_len - len) * dup_cap + index among the
//                        node's own (equal-length) patterns, which orders equal
//                        ends by (length desc, list order) -- the order in which
//                        src/nfa/noncontiguous.rs:490-523 concatenates lists.
constexpr int kTieBits = 24;
constexpr uint64_t kTieMask = (1ull << kTieBits) - 1;
constexpr uint64_t kInvalidKey = ~0ull;

// (start, end) in haystack offsets of tuple (key, pid) of a search of the span from span_start.  Key
// layouts (ChainLaunch::mode): 1 = start_rel << 24 | len, otherwise end_rel << 24 | tie.
struct MatchSpan {
  uint64_t start, end;
};
__host__ __device__ __forceinline__ MatchSpan decode_key(uint64_t key, uint32_t pid, int key_mode, uint64_t span_start,
                                                         const uint32_t* pattern_lens) {
  const uint64_t at = span_start + (key >> kTieBits);
  if (key_mode == 1) return MatchSpan{at, at + (key & kTieMask)};
  return MatchSpan{at - pattern_lens[pid], at};
}

// The ordered tuples a search left in the workspace: first member of every launch struct that reads them.
struct TupleList {
  const uint64_t* keys;
  const uint32_t* pids;
  const uint32_t* pattern_lens;
  uint64_t n;
};

struct DfaDev {
  const uint32_t* trans;          // premultiplied ids, as shipped (src/dfa.rs:92-95)
  const uint8_t* classes;         // [256] byte -> class (src/util/alphabet.rs)
  const uint32_t* match_offsets;  // CSR over match-state rows 2..
  const uint32_t* match_pids;
  const uint32_t* pattern_lens;
  const uint16_t* depth16;        // trie depth per row (prefilter engine's anchored walk)
  uint32_t stride2;
  uint32_t max_match_id;
  uint32_t start_unanchored_id;
  uint32_t start_anchored_id;
  uint32_t max_pattern_len;
  uint32_t min_pattern_len;
  // Anchor map (prefilter engine): open-addressing hash table from the first k haystack bytes at a
  // candidate offset to the trie state those bytes lead to, so that the verifier starts at depth
  // k with one lookup instead of k dependent table reads.  Entry = (key, premultiplied state id),
  // empty slots hold id 0 (DEAD is never a target).  nullptr: walk from the start state.
  const uint2* amap;
  uint32_t amap_shift;            // slot = hash3(key) >> amap_shift
  uint32_t amap_mask;             // capacity - 1
  uint32_t amap_k;                // key length in bytes (1..4)
  uint32_t amap_kmask;            // mask of the low amap_k bytes
};

// ---- launch wrappers (acb_kernels.cu) --------------------------------------

struct WalkLaunch {
  const uint8_t* hay;   // device pointer to haystack byte 0
  uint64_t hay_len;     // bytes readable behind `hay`
  uint64_t span_start, span_end;
  uint64_t seg_len;     // bytes owned per lane
  uint64_t n_segs;
  uint64_t* keys;       // [cap]
  uint32_t* pids;       // [cap]
  unsigned long long* counter;  // total tuples wanted (may exceed cap => overflow)
  uint64_t cap;
};
cudaError_t launch_walk_overlapping(const DfaDev& dfa, const WalkLaunch& p, cudaStream_t s);

// Dense-table construction on the device (SURVEY section 8f.2; the cells of src/dfa.rs:544-593):
// one launch per BFS level of the trie, one warp per table row: copy the row of the failure state
// (complete since an earlier level) or fill with a constant, then overlay the row's own edges.
struct FillLaunch {
  uint32_t* trans;              // [state_len << stride2], zero-initialised
  uint32_t stride2, alphabet_len;
  const uint32_t* row;          // per entry of this level: row to produce
  const uint32_t* inherit_row;  // UINT32_MAX: fill with fill_id
  const uint32_t* fill_id;
  const uint32_t* edge_off;     // [n + 1], indexes edge_class / edge_to (absolute offsets)
  const uint8_t* edge_class;
  const uint32_t* edge_to;
  uint32_t n;                   // rows in this level
};
cudaError_t launch_dfa_fill_level(const FillLaunch& f, cudaStream_t s);

// Sequential engine: single-lane restatement of FindIter (src/automaton.rs:857-936) over try_find_fwd
// (:1259-1420) -- anchored inputs, automata containing the empty pattern -- one thread per document.
// A batch (acg_*_batch when the prefilter engine does not apply) takes two launches: the count pass
// (incl == nullptr) fills counts[n_docs] -- or flags[n_docs] for is_match -- and after an inclusive scan
// of the counts the fill pass writes each document's records at out[incl[doc - 1] * 3] as
// (pid | doc << 32, start, end) with offsets relative to the document, the acg_doc_match layout.
// find: one launch (`find`).  A single document (a single-haystack search) takes one launch: the count
// pass given `out` also writes the records, from index 0.  A long document is one thread's walk.
struct SeqDocsLaunch {
  const uint8_t* hay;
  const uint64_t* doc_offsets;  // [n_docs + 1], haystack offsets
  uint64_t n_docs;
  int anchored;
  int match_kind;
  int overlapping;              // 1: find_overlapping_iter, 0: find_iter
  int single;                   // 1: stop at the first match (is_match, find)
  int earliest;                 // find_iter, find: as acg_find's `earliest` (forced on for Standard)
  int find;                     // find (with single): one pass, the first match or (0 | doc << 32, 0, 0) at
                                // out[doc * 3] and flags[doc] = found
  unsigned long long* counts;   // count pass: [n_docs]
  uint8_t* flags;               // count pass, is_match / find: [n_docs] instead of counts
  const unsigned long long* incl;   // fill pass: [n_docs] inclusive scan of counts
  uint64_t* out;                // [cap * 3]; nullptr in the count pass of a batch
  uint64_t cap;                 // records
};
cudaError_t launch_seq_docs(const DfaDev& dfa, const SeqDocsLaunch& p, cudaStream_t s);
cudaError_t inclusive_sum_u64(void* d_temp, size_t& temp_bytes, const unsigned long long* in, unsigned long long* out,
                              uint64_t n, cudaStream_t s);

// is_match over a batch on the prefilter engine: flags[doc] = 1 for the document of each of n tuples.
// find over a batch (best != nullptr): the tuple with the smallest key of each document -- its first match,
// since the keys of one document order its candidates as try_find prefers them -- written at out[doc * 3] in
// the acg_doc_match layout, flags[doc] = found; (0 | doc << 32, 0, 0) and 0 for a document without one.
struct DocFlagsLaunch {
  TupleList t;
  int mode;                     // key layout as ChainLaunch::mode
  uint64_t span_start;
  const uint64_t* doc_offsets;  // [n_docs + 1]
  uint64_t n_docs;
  uint8_t* flags;
  unsigned long long* best = nullptr;  // find: [n_docs] scratch, the smallest key per document
  uint64_t* out = nullptr;             // find: [n_docs * 3]
};
cudaError_t launch_doc_flags(const DocFlagsLaunch& f, cudaStream_t s);
// find: three launches (clear, per-document minimum key, write the minimum's record)
cudaError_t launch_doc_first(const DocFlagsLaunch& f, cudaStream_t s);

// Device-resident batch results (acg_find_iter_batch_devout / acg_find_overlapping_batch_devout, prefilter
// engine): the n ordered tuples, document-major, become acg_doc_match records out[i * 3] = (pid | doc << 32,
// start, end), offsets relative to the document, and match_offsets[d] = the index of document d's first record
// (match_offsets[n_docs] = n).  Record i writes match_offsets[d] = i for every d in (doc of i - 1, doc of i], the
// last one also (doc of n - 1, n_docs]: every entry is written once, with no atomics.  n > 0.
struct DocRecordsLaunch {
  TupleList t;
  int mode;                     // key layout as ChainLaunch::mode
  uint64_t span_start;
  const uint64_t* doc_offsets;  // [n_docs + 1]
  uint64_t n_docs;
  uint64_t* out;                // [n * 3]
  uint64_t* match_offsets;      // [n_docs + 1]
};
cudaError_t launch_doc_records(const DocRecordsLaunch& e, cudaStream_t s);

// Offsets in device memory: result[0] = 1 if some offs[i] > offs[i + 1] or offs[n_docs] > hay_len (left as it
// was otherwise: the caller clears it), result[1] = offs[0], result[2] = offs[n_docs].
cudaError_t launch_check_offsets(const uint64_t* offs, uint64_t n_docs, uint64_t hay_len,
                                 unsigned long long* result, cudaStream_t s);

// K3/K3b: position-parallel k-gram prefilter fused with the anchored DFA verify.
// Plays the role of the reference's packed/Teddy prefilter (src/packed/teddy/
// generic.rs:114-713 candidate + :820-870 verify): a cheap per-position
// fingerprint test with no false negatives, then exact verification -- except
// that the fingerprint is a hashed k-gram bitmap in shared memory (one LDS per
// position) instead of PSHUFB nybble masks, and the verifier is the shipped DFA
// walked from the candidate position while it stays on the trie path.
struct PrefilterLaunch {
  const uint8_t* hay;
  uint64_t hay_len;             // bytes readable behind `hay`
  uint64_t span_start, span_end;
  const uint32_t* bitmap;       // global copy, staged into shared memory per CTA
  uint32_t log_bits;            // bitmap size = 1 << log_bits bits
  uint32_t k;                   // fingerprint length in bytes (1..4), <= min_pattern_len
  uint32_t stride;              // 1: probe every offset with the k-gram; 2: probe even offsets with
                                // 3-byte fingerprints of pattern bytes [0,3) and [1,4) (k == 4 only)
  uint16_t geom;                // stride 2 only: 0 narrow, 1 wide (2 KiB tiles / 512 threads / 16 KiB bitmap: rare
                                // first-stage hits)
  uint16_t pair;                // (unused)
  uint32_t kmask;               // mask of the low k bytes
  uint32_t fold;                // 0 or 0x20202020 (ASCII case folding of the fingerprint)
  uint32_t mult;                // first Bloom hash: gram * mult
  uint32_t mult3;               // stride 2: multiplier of the 3-byte first-stage fingerprint
  uint32_t shift;               // hash >> shift = byte offset into the bitmap (= 35 - log_bits)
  int dense;                    // many fingerprints: survivors of both probes are filtered once more
                                // (anchor-map lookup) before the warp-wide verification
  int brute;                    // 1: skip the bitmap, every position is a candidate
  int mode;                     // 0: all occurrences (overlapping); 1: best match per start (leftmost)
  int first_only;               // mode 0 for a non-overlapping consumer (find_iter / find): of several equal
                                // patterns ending at a node only the first can ever be yielded -- skip the rest
  uint32_t dup_shift;           // log2 of the per-node duplicate capacity in the tie-break
  uint64_t scan_lo, scan_hi;      // start offsets this launch is responsible for (within the span)
  uint64_t region_lo, region_hi;  // 16-byte aligned filter region inside [scan_lo, scan_hi)
  uint64_t* keys;
  uint32_t* pids;
  unsigned long long* counter;  // [0] tuples, [1] candidates, [2] super-tiles handed out (dynamic tile distribution)
  uint64_t cap;
  uint32_t dyn;                 // tile distribution: 0 static, 1 per-CTA counter, 2 global super-tiles from counter[2] (see prefilter_kernel)
  // byte-set scan (bytescan_kernel, the memchr-class start-bytes / rare-bytes prefilter): bs_n needles,
  // each replicated into the four bytes of a word; a pattern that shows needle i at offset q starts in
  // [q - bs_back[i], q] (0 for start bytes, <= 15)
  uint32_t bs_n;
  uint32_t bs_needle[3];
  uint32_t bs_back[3];
  uint32_t key_shift;           // stride 2: first-stage hash = window * (mult3 << key_shift).  8: the fourth window
                                // byte drops out (3-byte keys); 5: its low 3 bits stay in the key (experiment).
  // Bucketed emission (bucket_shift != 0, see Emitter in acb_prefilter.cu): a tuple whose key offset is o goes to
  // bucket o >> bucket_shift, slots [b << bucket_log, (b + 1) << bucket_log) of keys / pids, counted in
  // counter[kBucketCountersAt + b]; a tuple whose bucket is full is appended to the overflow list behind the
  // buckets (keys[bucket_slots + i], i counted in counter[0]).  0: one list counted in counter[0].
  uint32_t bucket_shift;
  uint32_t bucket_log;
  uint64_t bucket_slots;        // n_buckets << bucket_log
  // Batched search (acg_*_batch): CSR document bounds in haystack offsets, [n_docs + 1] on the device; a match is
  // reported only if it ends inside the document its start lies in.  nullptr / 0: one haystack.
  const uint64_t* doc_offsets;
  uint64_t n_docs;
};
cudaError_t launch_prefilter(const DfaDev& dfa, const PrefilterLaunch& p, int sm_count, cudaStream_t s);
cudaError_t launch_bytescan(const DfaDev& dfa, const PrefilterLaunch& p, int sm_count, cudaStream_t s);

// Non-overlapping iteration (FindIter, src/automaton.rs:857-936) over ordered candidate tuples.
// mode 1 (leftmost): keys = (start_rel << 24 | len), sorted by start;
// mode 0 (standard): keys = (end_rel << 24 | tie), sorted by (end, len desc, list order).
// Writes flags[i] = 1 for the tuples the reference's iterator would yield.
struct ChainLaunch {
  TupleList t;
  int mode;
  uint64_t* scratch_end;   // [n] end offsets (leftmost) -> inclusive prefix max
  uint8_t* flags;          // [n]
};
cudaError_t launch_chain_ends(const ChainLaunch& c, cudaStream_t s);
cudaError_t launch_chain_select(const ChainLaunch& c, cudaStream_t s);
cudaError_t scan_max_u64(void* d_temp, size_t& temp_bytes, uint64_t* data, uint64_t n, cudaStream_t s);
cudaError_t select_flagged(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, const uint32_t* pids_in,
                           const uint8_t* flags, uint64_t* keys_out, uint32_t* pids_out,
                           unsigned long long* d_num_out, uint64_t n, cudaStream_t s);

// Expand ordered (end_rel << 24 | tie, pid) tuples into 24-byte match records on the device,
// keeping only ends > min_end (writes compacted output; order preserved because kept tuples are a
// suffix of the end-sorted list).
struct ExpandLaunch {
  TupleList t;
  uint64_t first;        // index of the first kept tuple (host-side binary search result)
  uint64_t span_start;
  uint64_t offset_add;
  uint64_t* out;         // [ (n-first) * 3 ] as (pid, start, end) u64 triples == acg_match layout
  int small = 0;         // > 0: that many 128-thread CTAs at most (one per SM: each fits beside a persistent scan
                         // CTA, pipelined sharded steps); 0: one 256-thread CTA per 256 records
};
cudaError_t launch_expand(const ExpandLaunch& e, cudaStream_t s);
// number of leading tuples whose end_rel <= bound (keys sorted ascending)
cudaError_t launch_lower_bound(const uint64_t* keys, uint64_t n, uint64_t bound_key,
                               unsigned long long* d_result, cudaStream_t s);

// K4 on bucketed tuples (PrefilterLaunch::bucket_shift).  Bucket b holds the keys with offsets in
// [b << bucket_shift, (b + 1) << bucket_shift); its count is bucket_count[b] (may exceed bucket_cap: the rest
// went to the overflow list).
constexpr int kBucketCountersAt = 8;   // index of bucket 0's counter in the workspace's counter array
constexpr uint32_t kMaxBuckets = 1024;
constexpr uint32_t kOrderLog = 14;
constexpr uint32_t kOrderCap = 1u << kOrderLog;  // tuples one CTA of order_buckets_kernel sorts in shared memory
struct OrderLaunch {
  const uint64_t* keys_in;             // buffer 0: bucket b at [b * bucket_cap, ...), then the overflow list
  const uint32_t* pids_in;
  uint64_t* keys_out;                  // [sum of the counts], (offset << 24 | tie, pid) ascending
  uint32_t* pids_out;
  const unsigned long long* bucket_count;  // [n_buckets]
  const unsigned long long* overflow_count;
  uint32_t n_buckets, bucket_shift, bucket_cap;
  uint32_t tie_bits;                   // the tie-break occupies the low tie_bits bits of the key
  uint64_t bucket_slots;               // n_buckets * bucket_cap: start of the overflow list
};
// One CTA per bucket sorts it in shared memory and stores it at the bucket's prefix offset.  Needs every
// count <= bucket_cap <= kOrderCap (an empty overflow list).
cudaError_t launch_order_buckets(const OrderLaunch& o, cudaStream_t s);
// Fallback: the buckets and the overflow list, concatenated into keys_out / pids_out (unordered).
cudaError_t launch_compact_buckets(const OrderLaunch& o, cudaStream_t s);

// key/pid pair sort (K4). temp storage is queried with d_temp == nullptr.
cudaError_t sort_pairs(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, uint64_t* keys_out,
                       const uint32_t* vals_in, uint32_t* vals_out, uint64_t n, int end_bit,
                       cudaStream_t s);

}  // namespace acb
