// acb_kernels.cu -- sm_90a kernels of the Aho-Corasick search path.
//
//   K1  walk_overlapping_kernel   sharded DFA state-transition scan; replaces the
//                                 loop of try_find_overlapping_fwd_imp
//                                 (src/automaton.rs:1491-1534) + DFA::next_state
//                                 (src/dfa.rs:218-226) + match expansion (:275-286)
//   Kseq seq_docs_kernel          single-lane FindIter/try_find (anchored inputs,
//                                 empty-pattern automata), one thread per document
//        doc_flags_kernel         per-document is_match / first match of a batch's
//        doc_first_kernel         prefilter tuples
//        doc_records_kernel       device-resident batch records + their CSR index by document
//        count_keys_kernel        pattern counts of a batch: (document, pattern) keys, runs of
//        run_heads_kernel         equal sorted keys, the CSR row index by document
//        count_runs_kernel
//        count_rows_kernel
//        cover_keys_kernel        match coverage of a batch: (start, length) per match, ends,
//        cover_ends_kernel        each match's uncovered part counted per document and written
//        cover_runs_kernel        to the byte mask
//        cover_mask_kernel
//        replace_keys_kernel      replace of a batch: per match its document, pid, end and length change,
//        replace_rows_kernel      the output offsets by document, the first match of every output tile,
//        replace_tiles_kernel     and the output spliced tile by tile
//        replace_splice_kernel
//        stream_docs_kernel       a stream set's feed: the combined documents tail | chunk, gathered, the
//        stream_gather_kernel     records that a previous feed has not returned, rebased to stream offsets,
//        stream_keep_kernel       and every stream's new position, cursor and tail
//        stream_records_kernel
//        stream_state_kernel
//        stream_hold_kernel       a replace set's feed: the records of D with each stream's held bytes as a
//                                 deletion after them, for the replace kernels to splice
//        stream_flush_kernel      a replace set's flush: the listed streams' tails out, their state zeroed
//        look_state_kernel        a stream set's lookahead: every row's state from its stream's tail, the
//        look_heads_kernel        distinct states (after a sort) with one row each, the candidates walked
//        look_compact_kernel      from every distinct state into that row, and the row copied to the rows
//        look_mask_kernel         that share its state
//        look_copy_kernel
//        check_offsets_kernel     validation of document offsets in device memory
//   K4  sort_pairs                ordering of the appended tuples (CUB radix sort)
#include "acb_device.cuh"
#ifndef ACB_PTX_HEADER
#define ACB_PTX_HEADER "acb_ptx.cuh"
#endif
#include ACB_PTX_HEADER

#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace acb {

namespace {

// Append the whole pattern list of match state `sid` (entered after consuming the byte at
// absolute offset end-1) to the tuple buffer.  Lanes of a warp that report in the same step share
// one atomic (warp-ballot + warp-aggregated append), list entry by list entry.  Out of line: matches
// are rare (one per 4 KiB in the BASELINE workloads) and the walk loop must stay small.
__device__ __noinline__ void emit_state_matches(const uint32_t* match_offsets, const uint32_t* match_pids,
                                                uint32_t row, uint64_t end_rel, uint64_t* keys, uint32_t* pids,
                                                unsigned long long* counter, uint64_t cap) {
  const uint32_t lo = match_offsets[row], hi = match_offsets[row + 1];
  const int lane = threadIdx.x & 31;
  for (uint32_t i = lo; i < hi; ++i) {
    const unsigned m = __activemask();
    const int leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(m));
    base = __shfl_sync(m, base, leader);
    const unsigned long long g = base + __popc(m & ((1u << lane) - 1));
    if (g < cap) {  // overflow: the host sees counter > cap and retries
      keys[g] = (end_rel << kTieBits) | (uint64_t)(i - lo);
      pids[g] = match_pids[i];
    }
  }
}

constexpr int kWalkThreads = 256;

// One lane per haystack shard.  A lane starts cold (start state) at most
// max_pattern_len-1 bytes before its shard -- the Aho-Corasick state depends on
// at most that many trailing bytes -- and only reports matches whose end lies
// inside its shard, so every end offset is owned by exactly one lane.
// The loop is one dependent table load per byte.  Everything below the first two trie levels is an
// L2 hit, one 32-byte sector per byte, so the kernel is bound by random-sector traffic out of L2 and
// more loads in flight do not help.  Tried and dropped as slower: the start / depth-1 rows staged in
// shared memory behind a flagged table copy, and four independent shards per lane with speculative
// 16-byte blocks.
__global__ void __launch_bounds__(kWalkThreads, 5)
walk_overlapping_kernel(DfaDev d, WalkLaunch p) {
  __shared__ uint8_t s_cls[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cls[i] = d.classes[i];
  __syncthreads();

  const uint64_t seg = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (seg >= p.n_segs) return;
  const uint64_t g0 = p.span_start + seg * p.seg_len;
  uint64_t g1 = g0 + p.seg_len;
  if (g1 > p.span_end) g1 = p.span_end;
  const uint64_t back = d.max_pattern_len > 0 ? (uint64_t)d.max_pattern_len - 1 : 0;
  uint64_t pos = (g0 - p.span_start > back) ? g0 - back : p.span_start;

  const uint32_t* __restrict__ trans = d.trans;
  const uint32_t max_match = d.max_match_id;
  uint32_t sid = d.start_unanchored_id;

  // matches of the start state itself (empty patterns) at the very beginning of
  // the span are reported before the first byte (src/automaton.rs:1456-1464)
  if (seg == 0 && sid != 0 && sid <= max_match)
    emit_state_matches(d.match_offsets, d.match_pids, (sid >> d.stride2) - 2, 0, p.keys, p.pids, p.counter, p.cap);

  auto next = [&](uint32_t from, uint32_t byte) -> uint32_t { return __ldg(trans + from + s_cls[byte]); };

#define ACB_STEP(byte_expr)                                                          \
  do {                                                                               \
    sid = next(sid, (byte_expr));                                                    \
    if (sid <= max_match) {                                                          \
      if (sid == 0) { pos = g1; break; }                                             \
      if (pos >= g0)                                                                 \
        emit_state_matches(d.match_offsets, d.match_pids, (sid >> d.stride2) - 2, pos + 1 - p.span_start, p.keys, p.pids, p.counter, p.cap); \
    }                                                                                \
    ++pos;                                                                           \
  } while (0)

  const uint8_t* __restrict__ hay = p.hay;
  while (pos < g1 && ((reinterpret_cast<uintptr_t>(hay + pos)) & 15)) ACB_STEP(hay[pos]);
  while (pos + 16 <= g1) {
    const uint4 v = ptx::ld_nc_u4(hay + pos);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    bool dead = false;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const uint32_t b = (w[k >> 2] >> ((k & 3) * 8)) & 0xFF;
      sid = next(sid, b);
      if (sid <= max_match) {
        if (sid == 0) { dead = true; break; }
        if (pos >= g0)
          emit_state_matches(d.match_offsets, d.match_pids, (sid >> d.stride2) - 2, pos + 1 - p.span_start, p.keys, p.pids, p.counter, p.cap);
      }
      ++pos;
    }
    if (dead) { pos = g1; break; }
  }
  while (pos < g1) ACB_STEP(hay[pos]);
#undef ACB_STEP
}

// ---- dense-table construction (one BFS level per launch) -------------------------
constexpr int kFillThreads = 256;

__global__ void __launch_bounds__(kFillThreads) dfa_fill_level_kernel(FillLaunch f) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t w = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= f.n) return;
  uint32_t* dst = f.trans + ((size_t)f.row[w] << f.stride2);
  const uint32_t inherit = f.inherit_row[w];
  if (inherit != UINT32_MAX) {
    const uint32_t* src = f.trans + ((size_t)inherit << f.stride2);  // written by an earlier launch
    for (uint32_t c = lane; c < f.alphabet_len; c += 32) dst[c] = src[c];
  } else {
    const uint32_t v = f.fill_id[w];
    for (uint32_t c = lane; c < f.alphabet_len; c += 32) dst[c] = v;
  }
  __syncwarp();
  for (uint32_t e = f.edge_off[w] + lane; e < f.edge_off[w + 1]; e += 32) dst[f.edge_class[e]] = f.edge_to[e];
}

// ---- sequential engine -------------------------------------------------------

struct SeqMatch {
  uint32_t pid;
  uint64_t start, end;
};

__device__ __forceinline__ bool seq_is_match(const DfaDev& d, uint32_t sid) {
  return sid != 0 && sid <= d.max_match_id;
}
__device__ __forceinline__ SeqMatch seq_get_match(const DfaDev& d, uint32_t sid, uint32_t idx, uint64_t at) {
  const uint32_t row = (sid >> d.stride2) - 2;
  const uint32_t pid = d.match_pids[d.match_offsets[row] + idx];
  SeqMatch m;
  m.pid = pid;
  m.start = at - d.pattern_lens[pid];
  m.end = at;
  return m;
}

// try_find_fwd_imp, src/automaton.rs:1285-1420 (prefilter-free instance)
__device__ __forceinline__ bool seq_try_find(const DfaDev& d, const uint8_t* hay, uint64_t start, uint64_t end,
                             bool anchored, bool earliest, SeqMatch* out) {
  if (start > end) return false;
  uint32_t sid = anchored ? d.start_anchored_id : d.start_unanchored_id;
  uint64_t at = start;
  bool have = false;
  SeqMatch mat;
  if (seq_is_match(d, sid)) {
    mat = seq_get_match(d, sid, 0, at);
    have = true;
    if (earliest) { *out = mat; return true; }
  }
  while (at < end) {
    sid = d.trans[sid + d.classes[hay[at]]];
    if (sid <= d.max_match_id) {
      if (sid == 0) break;
      SeqMatch m = seq_get_match(d, sid, 0, at + 1);
      if (!(anchored && m.start > start)) {
        mat = m;
        have = true;
        if (earliest) break;
      }
    }
    ++at;
  }
  if (have) *out = mat;
  return have;
}

// FindIter (src/automaton.rs:857-936) over [span_start, span_end): writes the i-th match as
// (pid | tag, start - base, end - base) at out[(first + i) * 3] while first + i < cap (out may be
// null: count only) and returns the number of matches.
__device__ __forceinline__ unsigned long long seq_find_iter(const DfaDev& d, const uint8_t* hay, uint64_t span_start, uint64_t span_end,
                                            bool anchored, bool earliest, bool single, uint64_t* out,
                                            unsigned long long first, uint64_t cap, uint64_t tag, uint64_t base) {
  uint64_t start = span_start;
  unsigned long long n = 0;
  bool have_last = false;
  uint64_t last_end = 0;
  for (;;) {
    SeqMatch m;
    if (!seq_try_find(d, hay, start, span_end, anchored, earliest, &m)) break;
    if (!single && m.start == m.end && have_last && m.end == last_end) {
      // FindIter::handle_overlapping_empty_match, src/automaton.rs:910-920
      start += 1;
      if (!seq_try_find(d, hay, start, span_end, anchored, earliest, &m)) break;
    }
    if (out && first + n < cap) {
      out[(first + n) * 3 + 0] = m.pid | tag;
      out[(first + n) * 3 + 1] = m.start - base;
      out[(first + n) * 3 + 2] = m.end - base;
    }
    ++n;
    if (single) break;
    start = m.end;
    last_end = m.end;
    have_last = true;
  }
  return n;
}

// try_find_overlapping_fwd_imp (src/automaton.rs:1443-1537) run to the end of [lo, hi), unanchored:
// the start state's matches at lo, then every list entry of each match state entered, in list order.
// Same output convention as seq_find_iter.
__device__ __forceinline__ unsigned long long seq_overlapping(const DfaDev& d, const uint8_t* hay, uint64_t lo, uint64_t hi,
                                              uint64_t* out, unsigned long long first, uint64_t cap, uint64_t tag) {
  unsigned long long n = 0;
  uint32_t sid = d.start_unanchored_id;
  bool report = seq_is_match(d, sid);  // the start state's matches end at lo
  for (uint64_t at = lo;;) {           // `at`: end offset of the matches of sid
    if (report) {
      const uint32_t row = (sid >> d.stride2) - 2;
      for (uint32_t i = d.match_offsets[row]; i < d.match_offsets[row + 1]; ++i, ++n) {
        if (!out || first + n >= cap) continue;
        const uint32_t pid = d.match_pids[i];
        out[(first + n) * 3 + 0] = pid | tag;
        out[(first + n) * 3 + 1] = at - d.pattern_lens[pid] - lo;
        out[(first + n) * 3 + 2] = at - lo;
      }
    }
    if (at >= hi) break;
    sid = d.trans[sid + d.classes[hay[at]]];
    ++at;
    if (sid == 0) break;  // DEAD
    report = sid <= d.max_match_id;
  }
  return n;
}

struct SumOp {
  __device__ __forceinline__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; }
};

// One thread per document of a batch.  Count pass (incl == nullptr): counts[doc] = its number of
// matches, or flags[doc] = (a match exists) when flags is given.  Fill pass: the document's records from
// index incl[doc - 1] (the matches of the documents before it) on, tagged with the document
// (doc << 32 in the pid word, offsets relative to the document's first byte).  find: the count pass with
// flags, the document's one record written at index doc.  A count pass given `out` writes from index 0 (one
// document).
constexpr int kSeqDocThreads = 128;
template <bool OVERLAPPING>
__global__ void __launch_bounds__(kSeqDocThreads) seq_docs_kernel(DfaDev d, SeqDocsLaunch p) {
  const uint64_t doc = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (doc >= p.n_docs) return;
  const uint64_t lo = p.doc_offsets[doc], hi = p.doc_offsets[doc + 1];
  const bool fill = p.incl != nullptr;
  uint64_t* out = p.out;
  const unsigned long long first = p.find ? doc : (fill && doc ? p.incl[doc - 1] : 0);
  const uint64_t tag = doc << 32;
  if (p.find) {  // the record of "no match", overwritten by the match if there is one
    out[doc * 3 + 0] = tag;
    out[doc * 3 + 1] = 0;
    out[doc * 3 + 2] = 0;
  }
  unsigned long long n;
  if constexpr (OVERLAPPING) {
    n = seq_overlapping(d, p.hay, lo, hi, out, first, p.cap, tag);
  } else {
    const bool earliest = p.match_kind == 0 || p.earliest != 0;
    n = seq_find_iter(d, p.hay, lo, hi, p.anchored != 0, earliest, p.single != 0, out, first, p.cap, tag, lo);
  }
  if (fill) return;
  if (p.flags) p.flags[doc] = n != 0;
  else p.counts[doc] = n;
}

#ifdef ACB_EMULATE
// The dry-run runtime (tests/emu) has no atomicMin; it runs one thread at a time between synchronisation
// points, so a plain read-modify-write is atomic there.
inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  const unsigned long long o = *p;
  if (v < o) *p = v;
  return o;
}
#endif

// The document that holds haystack offset s, which lies in [doc_offsets[0], doc_offsets[n_docs]): the
// last one that starts at or before s, found by an upper-bound search for the first document end past s.
// (An empty document's end is its start, so the search never stops at one.)
__device__ __forceinline__ uint64_t doc_of(const uint64_t* offs, uint64_t n_docs, uint64_t s) {
  uint64_t lo = 1, hi = n_docs;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (offs[mid] > s) hi = mid; else lo = mid + 1;
  }
  return lo - 1;
}

// The haystack offsets of tuple i.
__device__ __forceinline__ MatchSpan tuple_span(const DocFlagsLaunch& f, uint64_t i) {
  return decode_key(f.t.keys[i], f.t.pids[i], f.mode, f.span_start, f.t.pattern_lens);
}

// Over the n tuples of a prefilter scan.  is_match: flags[doc] = 1 for the document of every tuple.
// find (best != nullptr): best[doc] = the smallest key of the document's tuples.
__global__ void doc_flags_kernel(DocFlagsLaunch f) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.t.n) return;
  const uint64_t doc = doc_of(f.doc_offsets, f.n_docs, tuple_span(f, i).start);
  if (f.best) atomicMin(f.best + doc, (unsigned long long)f.t.keys[i]);
  else f.flags[doc] = 1;
}

// find: clear best[] and flags[], and give every document the record of "no match".
__global__ void doc_first_clear_kernel(DocFlagsLaunch f) {
  const uint64_t doc = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (doc >= f.n_docs) return;
  f.best[doc] = ~0ull;
  f.flags[doc] = 0;
  f.out[doc * 3 + 0] = doc << 32;
  f.out[doc * 3 + 1] = 0;
  f.out[doc * 3 + 2] = 0;
}

// find, after doc_flags_kernel: the tuple holding its document's smallest key writes the document's record
// (decoded as acg_find decodes its first tuple, offsets relative to the document).  Keys are unique within
// a document, so one tuple per document writes.
__global__ void doc_first_kernel(DocFlagsLaunch f) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.t.n) return;
  const MatchSpan m = tuple_span(f, i);
  const uint64_t doc = doc_of(f.doc_offsets, f.n_docs, m.start);
  if (f.t.keys[i] != f.best[doc]) return;
  const uint64_t base = f.doc_offsets[doc];
  f.out[doc * 3 + 0] = (uint64_t)f.t.pids[i] | doc << 32;
  f.out[doc * 3 + 1] = m.start - base;
  f.out[doc * 3 + 2] = m.end - base;
  f.flags[doc] = 1;
}

// Ordered tuples of a batch -> acg_doc_match records and their CSR index by document, in one pass (see
// DocRecordsLaunch).  No match crosses a document end, so the documents of the records do not decrease.
__global__ void doc_records_kernel(DocRecordsLaunch e) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= e.t.n) return;
  const uint32_t pid = e.t.pids[i];
  const MatchSpan m = decode_key(e.t.keys[i], pid, e.mode, e.span_start, e.t.pattern_lens);
  const uint64_t doc = doc_of(e.doc_offsets, e.n_docs, m.start);
  const uint64_t base = e.doc_offsets[doc];
  e.out[i * 3 + 0] = (uint64_t)pid | doc << 32;
  e.out[i * 3 + 1] = m.start - base;
  e.out[i * 3 + 2] = m.end - base;
  uint64_t d = 0;
  if (i) d = doc_of(e.doc_offsets, e.n_docs, decode_key(e.t.keys[i - 1], e.t.pids[i - 1], e.mode, e.span_start, e.t.pattern_lens).start) + 1;
  for (; d <= doc; ++d) e.match_offsets[d] = i;
  if (i + 1 == e.t.n)
    for (d = doc + 1; d <= e.n_docs; ++d) e.match_offsets[d] = e.t.n;
}

// Pattern counts, step 1 (CountKeysLaunch): the (document, pattern) key of match i and its pid.
__global__ void count_keys_kernel(CountKeysLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.t.n) return;
  uint64_t doc;
  uint32_t pid;
  if (c.rec) {
    const uint64_t w0 = c.rec[i * 3];
    pid = (uint32_t)w0;
    doc = w0 >> 32;
  } else {
    pid = c.t.pids[i];
    doc = doc_of(c.doc_offsets, c.n_docs, decode_key(c.t.keys[i], pid, c.mode, c.span_start, c.t.pattern_lens).start);
  }
  c.keys_out[i] = doc << c.pid_bits | pid;
  c.pids_out[i] = pid;
}

// The first index in [lo, hi) whose key is >= v (hi if none); keys ascending.
__device__ __forceinline__ uint64_t lower_bound_key(const uint64_t* keys, uint64_t lo, uint64_t hi, uint64_t v) {
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (keys[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void run_heads_kernel(CountRunsLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  c.heads[i] = i == 0 || c.keys[i] != c.keys[i - 1];
}

// The head of each run writes its entry: the pid, and the run's length -- the next head's start (the first
// greater key, or n after the last run) minus its own.
__global__ void count_runs_kernel(CountRunsLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.n) return;
  const uint64_t key = c.keys[i];
  if (i && c.keys[i - 1] == key) return;
  const uint64_t r = c.run_index[i] - 1;
  c.pids[r] = c.key_pids[i];
  c.counts[r] = lower_bound_key(c.keys, i + 1, c.n, key + 1) - i;
}

// One thread per document d <= n_docs: the first key of a document >= d heads a run, whose index is the number
// of runs before it (nnz when there is none).
__global__ void count_rows_kernel(CountRunsLaunch c) {
  const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d > c.n_docs) return;
  const uint64_t i = lower_bound_key(c.keys, 0, c.n, d << c.pid_bits);
  c.row_offsets[d] = i < c.n ? c.run_index[i] - 1 : c.nnz;
}

// Match coverage, step 1 (CoverLaunch): the start of match i relative to the span, and its length.
__global__ void cover_keys_kernel(CoverLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.t.n) return;
  uint64_t start, len;
  if (c.rec) {
    const uint64_t* r = c.rec + i * 3;
    start = c.doc_offsets[r[0] >> 32] - c.span_start + r[1];
    len = r[2] - r[1];
  } else {
    const MatchSpan m = decode_key(c.t.keys[i], c.t.pids[i], c.mode, c.span_start, c.t.pattern_lens);
    start = m.start - c.span_start;
    len = m.end - m.start;
  }
  c.starts[i] = start;
  c.lens[i] = (uint32_t)len;
}

__global__ void cover_ends_kernel(CoverLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.t.n) return;
  c.max_end[i] = c.starts[i] + c.lens[i];
}

// The part of match i that no earlier match covers: [max(s_i, M_{i-1}), e_i), empty when M_{i-1} >= e_i.
__device__ __forceinline__ uint64_t cover_part_lo(const CoverLaunch& c, uint64_t i, uint64_t s) {
  if (i == 0) return s;
  const uint64_t m = c.max_end[i - 1];
  return m > s ? m : s;
}

// Each match adds the length of its uncovered part to its document's count.  The matches are in start order,
// so the documents of a warp's lanes do not decrease: a segmented inclusive scan over equal documents leaves
// each run's sum in its last lane, which alone adds it (one atomic per document per warp).  Every lane takes
// part in the shuffles, so none returns early.
__global__ void cover_runs_kernel(CoverLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint64_t doc = ~0ull, part = 0;
  if (i < c.t.n) {
    const uint64_t s = c.starts[i], e = s + c.lens[i], lo = cover_part_lo(c, i, s);
    part = e > lo ? e - lo : 0;
    doc = doc_of(c.doc_offsets, c.n_docs, c.span_start + s);
  }
  for (int o = 1; o < 32; o <<= 1) {
    const int src = lane >= o ? lane - o : lane;
    const uint64_t d2 = __shfl_sync(0xffffffffu, doc, src), p2 = __shfl_sync(0xffffffffu, part, src);
    if (lane >= o && d2 == doc) part += p2;
  }
  const uint64_t next = __shfl_sync(0xffffffffu, doc, lane < 31 ? lane + 1 : lane);
  if (i < c.t.n && part && (lane == 31 || next != doc)) atomicAdd(c.covered + doc, (unsigned long long)part);
}

// One warp per match writes its uncovered part of the mask: the parts are disjoint, so every covered byte is
// written once, and a 64 KiB match is 2 K coalesced stores per lane rather than one thread's 64 K.
__global__ void cover_mask_kernel(CoverLaunch c) {
  const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t lane = threadIdx.x & 31;
  if (i >= c.t.n) return;
  const uint64_t s = c.starts[i], e = s + c.lens[i];
  uint8_t* m = c.mask + c.span_start;
  for (uint64_t j = cover_part_lo(c, i, s) + lane; j < e; j += 32) m[j] = 1;
}

// Replace, step 1 (ReplaceLaunch): match i's document, pid, end, a_i = end - rep_len and delta_i.  On the prefilter
// engine `e` and `docs` are the tuple buffers being read: each thread reads its own tuple before it writes there.
__global__ void replace_keys_kernel(ReplaceLaunch r) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.t.n) return;
  uint64_t start, end, doc;
  uint32_t pid;
  if (r.rec) {
    const uint64_t* q = r.rec + i * 3;
    pid = (uint32_t)q[0];
    doc = q[0] >> 32;
    const uint64_t base = r.doc_offsets[doc] - r.span_start;
    start = base + q[1];
    end = base + q[2];
  } else {
    pid = r.t.pids[i];
    const MatchSpan m = decode_key(r.t.keys[i], pid, r.mode, r.span_start, r.t.pattern_lens);
    doc = doc_of(r.doc_offsets, r.n_docs, m.start);  // tuples are never empty: the start is inside the document
    start = m.start - r.span_start;
    end = m.end - r.span_start;
  }
  const uint64_t rep_len = r.rep_offsets[pid + 1] - r.rep_offsets[pid];
  r.a[i] = end - rep_len;
  r.e[i] = end;
  r.pids[i] = pid;
  r.docs[i] = (uint32_t)doc;
  r.incl[i] = rep_len - (end - start);
}

// One thread per document d <= n_docs: its output starts where its first byte lands, behind the length changes of
// the matches of the documents before it (those below the first match whose document is >= d).
__global__ void replace_rows_kernel(ReplaceLaunch r) {
  const uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d > r.n_docs) return;
  uint64_t lo = 0, hi = r.t.n;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (r.docs[mid] < d) lo = mid + 1; else hi = mid;
  }
  r.out_offsets[d] = r.doc_offsets[d] - r.span_start + (lo ? r.incl[lo - 1] : 0);
}

// The splice writes the output in tiles of kSpliceTile bytes of the output's 16-byte aligned address space: CTA b
// owns the bytes o with o + mis in [b * kSpliceTile, (b + 1) * kSpliceTile), mis = the output's address mod 16, and
// each thread one aligned 16-byte chunk of it.
constexpr int kSpliceThreads = 256;
constexpr uint64_t kSpliceTile = kSpliceThreads * 16;

__device__ __forceinline__ uint64_t replace_q(const ReplaceLaunch& r, uint64_t i) { return r.a[i] + r.incl[i]; }

// The last match i in [lo, hi) with q_i <= o, or lo - 1 if there is none (q is non-decreasing).
__device__ __forceinline__ int64_t replace_last_at(const ReplaceLaunch& r, int64_t lo, int64_t hi, uint64_t o) {
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (replace_q(r, mid) <= o) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

__device__ __forceinline__ uint64_t splice_tile_start(uint64_t tile, uint64_t mis) {
  const uint64_t v = tile * kSpliceTile;
  return v > mis ? v - mis : 0;
}

// One thread per tile t <= n_tiles: first[t] = the last match whose q is at or before the tile's first byte (-1:
// none).  The tile's bytes lie in the segments of matches first[t] .. first[t + 1].
__global__ void replace_tiles_kernel(ReplaceLaunch r, uint64_t n_tiles, uint64_t mis) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_tiles) return;
  r.tile_first[t] = replace_last_at(r, 0, (int64_t)r.t.n, splice_tile_start(t, mis));
}

// 16 input bytes from any address: the two aligned words that hold them, shifted together.
__device__ __forceinline__ uint4 load16(const uint8_t* p) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
  const uint4* w = reinterpret_cast<const uint4*>(addr & ~uintptr_t(15));
  const uint32_t sh = (uint32_t)(addr & 15);
  const uint4 x = __ldg(w);
  if (sh == 0) return x;
  const uint4 y = __ldg(w + 1);  // holds byte p[15]: inside the input
  const uint32_t v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
  const uint32_t k = sh >> 2, bits = (sh & 3) * 8;
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t lo = k == 0 ? v[j] : k == 1 ? v[j + 1] : k == 2 ? v[j + 2] : v[j + 3];
    const uint32_t hi = k == 0 ? v[j + 1] : k == 1 ? v[j + 2] : k == 2 ? v[j + 3] : v[j + 4];
    o[j] = __funnelshift_r(lo, hi, bits);
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// Replace, last step: every output byte written once.  A thread finds the segment of its chunk's first byte with
// one search among the tile's matches, and moves to the next segment with another only where one starts inside
// its chunk, so the work per tile is bounded by its 4 KiB of output and the logarithm of its number of matches,
// whatever the lengths of the documents, gaps and replacements.  A chunk inside one gap is one 16-byte copy.
__global__ void __launch_bounds__(kSpliceThreads) replace_splice_kernel(ReplaceLaunch r, uint64_t mis) {
  const uint64_t v = (uint64_t)blockIdx.x * kSpliceTile + threadIdx.x * 16;
  const uint64_t o = v > mis ? v - mis : 0;
  const uint64_t o_end = v + 16 - mis < r.out_len ? v + 16 - mis : r.out_len;
  if (o >= o_end) return;
  const int64_t f = r.tile_first[blockIdx.x];
  const int64_t lo = f > 0 ? f : 0, hi = r.tile_first[blockIdx.x + 1] + 1;
  int64_t i = replace_last_at(r, lo, hi, o);
  // the segment of match i: its replacement [rep_lo, rep_hi), then the gap up to next_q, input byte o - inc
  uint64_t inc = 0, rep_lo = 0, rep_hi = 0, rep_at = 0, next_q = ~0ull;
  auto enter = [&]() {
    if (i >= 0) {
      inc = r.incl[i];
      rep_lo = r.a[i] + inc;
      rep_hi = r.e[i] + inc;
      if (rep_hi > rep_lo) rep_at = r.rep_offsets[r.pids[i]] - r.rep_offsets[0];
    }
    next_q = i + 1 < hi ? replace_q(r, i + 1) : ~0ull;
  };
  enter();
  uint8_t* dst = r.out + o;
  const uint64_t n = o_end - o;
  if (n == 16 && o >= rep_hi && o + 16 <= next_q) {
    *reinterpret_cast<uint4*>(dst) = load16(r.in + (o - inc));
    return;
  }
  uint64_t w0 = 0, w1 = 0;
  for (uint64_t j = 0; j < n; ++j) {
    const uint64_t p = o + j;
    if (p >= next_q) {
      i = replace_last_at(r, i + 1, hi, p);
      enter();
    }
    const uint64_t b = p < rep_hi ? r.rep_bytes[rep_at + (p - rep_lo)] : r.in[p - inc];
    if (j < 8) w0 |= b << (8 * j); else w1 |= b << (8 * (j - 8));
  }
  if (n == 16) {
    *reinterpret_cast<uint4*>(dst) = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
  } else {
    for (uint64_t j = 0; j < n; ++j) dst[j] = (uint8_t)((j < 8 ? w0 >> (8 * j) : w1 >> (8 * (j - 8))) & 0xFF);
  }
}

// ---- stream sets (StreamLaunch) ----
__device__ __forceinline__ uint64_t stream_tail_len(const StreamLaunch& p, uint64_t s) {
  const uint64_t k = p.pos[s] - p.cursor[s];
  return k < p.back ? k : p.back;
}

__global__ void stream_docs_kernel(StreamLaunch p) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0) p.doc_offsets[0] = 0;
  if (s >= p.n) return;
  p.doc_offsets[s + 1] = stream_tail_len(p, s) + (p.chunk_offsets[s + 1] - p.chunk_offsets[s]);
}

// The last stream s in [lo, hi) with doc_offsets[s] <= o (lo - 1 if none): for o < docs_len the one whose D holds o.
__device__ __forceinline__ int64_t stream_at(const StreamLaunch& p, int64_t lo, int64_t hi, uint64_t o) {
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (p.doc_offsets[mid] <= o) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

// D in tiles of kSpliceTile bytes, one aligned 16-byte chunk per thread.  Two threads find the streams of the tile's
// first and last byte, so each thread searches only among the tile's streams.  A chunk inside one stream's chunk or
// tail bytes is one 16-byte copy; one that crosses a boundary is gathered byte by byte.
__global__ void __launch_bounds__(kSpliceThreads) stream_gather_kernel(StreamLaunch p) {
  __shared__ int64_t s_range[2];
  const uint64_t tile0 = (uint64_t)blockIdx.x * kSpliceTile;
  if (threadIdx.x < 2) {
    const uint64_t last = (tile0 + kSpliceTile < p.docs_len ? tile0 + kSpliceTile : p.docs_len) - 1;
    s_range[threadIdx.x] = stream_at(p, 0, (int64_t)p.n, threadIdx.x ? last : tile0);
  }
  __syncthreads();
  const uint64_t o = tile0 + threadIdx.x * 16;
  if (o >= p.docs_len) return;
  const uint64_t n = p.docs_len - o < 16 ? p.docs_len - o : 16;
  int64_t s = stream_at(p, s_range[0], s_range[1] + 1, o);
  // the bytes of stream s: tail [d0, c0), chunk [c0, d1)
  uint64_t d0, c0, d1;
  const uint8_t *tail, *chunk;
  auto enter = [&]() {
    d0 = p.doc_offsets[s];
    d1 = p.doc_offsets[s + 1];
    c0 = d0 + stream_tail_len(p, (uint64_t)s);
    tail = p.tail + (uint64_t)s * p.back;
    chunk = p.chunks + p.chunk_offsets[s];
  };
  enter();
  uint8_t* dst = p.docs + o;
  if (n == 16 && o >= c0 && o + 16 <= d1) {
    *reinterpret_cast<uint4*>(dst) = load16(chunk + (o - c0));
    return;
  }
  if (n == 16 && o + 16 <= c0) {
    *reinterpret_cast<uint4*>(dst) = load16(tail + (o - d0));
    return;
  }
  uint64_t w0 = 0, w1 = 0;
  for (uint64_t j = 0; j < n; ++j) {
    const uint64_t q = o + j;
    while (q >= d1) {
      ++s;
      enter();
    }
    const uint64_t b = q < c0 ? tail[q - d0] : chunk[q - c0];
    if (j < 8) w0 |= b << (8 * j); else w1 |= b << (8 * (j - 8));
  }
  if (n == 16) {
    *reinterpret_cast<uint4*>(dst) = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
  } else {
    for (uint64_t j = 0; j < n; ++j) dst[j] = (uint8_t)((j < 8 ? w0 >> (8 * j) : w1 >> (8 * (j - 8))) & 0xFF);
  }
}

__global__ void stream_keep_kernel(StreamLaunch p) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.m) return;
  const uint64_t* r = p.rec + i * 3;
  p.keep[i] = r[2] > stream_tail_len(p, r[0] >> 32);
}

// Thread i < m: record i, if kept, at its place among the kept ones; thread i <= n: out_index[i], the kept records
// before stream i's first one.
__global__ void stream_records_kernel(StreamLaunch p) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.m) {
    const uint64_t* r = p.rec + i * 3;
    const bool kept = !p.keep || p.keep[i] != (i ? p.keep[i - 1] : 0ull);
    if (kept) {
      const uint64_t j = p.keep ? p.keep[i] - 1 : i, s = r[0] >> 32;
      const uint64_t base = p.pos[s] - stream_tail_len(p, s);
      p.out[j * 3 + 0] = r[0];
      p.out[j * 3 + 1] = base + r[1];
      p.out[j * 3 + 2] = base + r[2];
    }
  }
  if (p.out_index && i <= p.n) {
    const uint64_t first = p.rec_index[i];
    p.out_index[i] = p.keep ? (first ? p.keep[first - 1] : 0) : first;
  }
}

// Stream s after the feed, from the records of D: its position pos' = base + |D_s| (base = pos - L_s, where D_s
// starts), its cursor' and the start of its new tail t = max(pos' - back, cursor'), which is also a replace set's
// emit boundary.  The state kernel and the hold kernel both take t from here, so the tail a replace feed holds back
// is the one the state keeps.
struct StreamNext {
  uint64_t base, pos, cursor, t;
};
__device__ __forceinline__ StreamNext stream_next(const StreamLaunch& p, uint64_t s) {
  StreamNext x;
  x.base = p.pos[s] - stream_tail_len(p, s);
  x.pos = x.base + (p.doc_offsets[s + 1] - p.doc_offsets[s]);
  x.cursor = p.cursor[s];
  if (!p.overlapping) {
    const uint64_t lo = p.rec_index[s], hi = p.rec_index[s + 1];
    if (hi > lo) x.cursor = x.base + p.rec[(hi - 1) * 3 + 2];
  }
  x.t = x.pos > p.back ? x.pos - p.back : 0;
  if (x.cursor > x.t) x.t = x.cursor;
  return x;
}

// One warp per stream: every lane reads the old state, then the new tail is copied and lane 0 stores pos and cursor.
__global__ void stream_state_kernel(StreamLaunch p) {
  const uint64_t s = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (s >= p.n) return;
  const uint64_t d0 = p.doc_offsets[s];
  const StreamNext x = stream_next(p, s);
  const uint64_t base = x.base, pos = x.pos, cursor = x.cursor, t = x.t;
  const uint8_t* src = p.docs + d0 + (t - base);
  uint8_t* dst = p.tail + s * p.back;
  for (uint64_t k = lane; k < pos - t; k += 32) dst[k] = src[k];
  __syncwarp();
  if (lane == 0) {
    p.pos[s] = pos;
    p.cursor[s] = cursor;
  }
}

// Thread i < m: record i of D, moved past the hold records of the streams before its own; thread s < n: stream s's
// hold record [t - base, |D_s|) after its last record.  D's find_iter records all end at or before cursor' <= t, so
// the list stays in start order within every stream.
__global__ void stream_hold_kernel(StreamLaunch p) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.m) {
    const uint64_t* r = p.rec + i * 3;
    uint64_t* q = p.held + (i + (r[0] >> 32)) * 3;
    q[0] = r[0];
    q[1] = r[1];
    q[2] = r[2];
  }
  if (i < p.n) {
    const StreamNext x = stream_next(p, i);
    uint64_t* q = p.held + (p.rec_index[i + 1] + i) * 3;
    q[0] = (i << 32) | p.hold_pid;
    q[1] = x.t - x.base;
    q[2] = x.pos - x.base;
  }
}

// One warp per listed stream: its tail to the output, then lane 0 zeroes its state.
__global__ void stream_flush_kernel(StreamLaunch p, const uint64_t* ids, uint64_t n_ids, const uint64_t* out_offsets,
                                    uint8_t* out) {
  const uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if (k >= n_ids) return;
  const uint64_t s = ids ? ids[k] : k, o = out_offsets[k], len = out_offsets[k + 1] - o;
  const uint8_t* src = p.tail + s * p.back;
  for (uint64_t j = lane; j < len; j += 32) out[o + j] = src[j];
  if (lane == 0) {
    p.pos[s] = 0;
    p.cursor[s] = 0;
  }
}

// ---- lookahead of a stream set (LookLaunch) ----
// Thread k: the state row k's stream is in, walked from the unanchored start over its tail.
constexpr int kLookThreads = 256;
__global__ void __launch_bounds__(kLookThreads) look_state_kernel(DfaDev d, LookLaunch p) {
  __shared__ uint8_t s_cls[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cls[i] = d.classes[i];
  __syncthreads();
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p.n_rows) return;
  const uint64_t s = p.ids ? p.ids[k] : k, len = stream_tail_len(p.st, s);
  const uint8_t* tail = p.st.tail + s * p.st.back;
  uint32_t sid = d.start_unanchored_id;
  for (uint64_t j = 0; j < len; ++j) sid = __ldg(d.trans + sid + s_cls[tail[j]]);
  p.keys[k] = sid;
  p.rows[k] = (uint32_t)k;
}

__global__ void look_heads_kernel(LookLaunch p) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.n_rows) p.heads[i] = i == 0 || p.skeys[i] != p.skeys[i - 1];
}

// After the scan heads[i] is 1 + the run of entry i: the head of run u stores its state and row, every entry its run.
__global__ void look_compact_kernel(LookLaunch p) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_rows) return;
  const uint64_t u = p.heads[i] - 1;
  const uint32_t row = p.srows[i];
  p.row_u[row] = u;
  if (i == 0 || p.heads[i - 1] != p.heads[i]) {
    p.keys[u] = p.skeys[i];
    p.rows[u] = row;
  }
}

// Warp item (u, g), items in that order so that neighbouring warps share a state: lane c walks candidate 32 g + c
// from state keys[u] and stops at the first match state (DEAD ends the walk without one).  The candidates' bytes are
// class ids already.  U is read here, so the grid does not depend on it.
__global__ void __launch_bounds__(kLookThreads) look_mask_kernel(DfaDev d, LookLaunch p) {
  const uint64_t n_u = p.heads[p.n_rows - 1], groups = (p.n_cands + 31) >> 5, items = n_u * groups;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t* __restrict__ trans = d.trans;
  const uint32_t max_match = d.max_match_id;
  for (uint64_t it = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; it < items; it += warps) {
    const uint64_t u = it / groups, c = (it - u * groups) * 32 + lane;
    if (c >= p.n_cands) continue;
    uint32_t sid = (uint32_t)p.keys[u];
    uint8_t hit = 0;
    const uint64_t hi = __ldg(p.cand_offsets + c + 1);
    for (uint64_t q = __ldg(p.cand_offsets + c); q < hi; ++q) {
      sid = __ldg(trans + sid + __ldg(p.cand_classes + q));
      if (sid <= max_match) {
        hit = sid != 0;
        break;
      }
    }
    p.out[(uint64_t)p.rows[u] * p.n_cands + c] = hit;
  }
}

// Item (row, tile): a row whose run is written by another row copies that row's tile of kSpliceTile bytes, one
// 16-byte piece per thread.
__global__ void __launch_bounds__(kSpliceThreads) look_copy_kernel(LookLaunch p) {
  const uint64_t tiles = (p.n_cands + kSpliceTile - 1) / kSpliceTile;
  for (uint64_t it = blockIdx.x; it < p.n_rows * tiles; it += gridDim.x) {
    const uint64_t k = it / tiles, o = (it - k * tiles) * kSpliceTile + threadIdx.x * 16;
    const uint64_t r = p.rows[p.row_u[k]];
    if (r == k || o >= p.n_cands) continue;
    const uint8_t* src = p.out + r * p.n_cands + o;
    uint8_t* dst = p.out + k * p.n_cands + o;
    const uint64_t n = p.n_cands - o < 16 ? p.n_cands - o : 16;
    if (n == 16 && !((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15)) {
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    } else {
      for (uint64_t j = 0; j < n; ++j) dst[j] = src[j];
    }
  }
}

__global__ void check_offsets_kernel(const uint64_t* offs, uint64_t n_docs, uint64_t hay_len,
                                     unsigned long long* result) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    result[1] = offs[0];
    result[2] = offs[n_docs];
    if (offs[n_docs] > hay_len) result[0] = 1;
  }
  if (i < n_docs && offs[i] > offs[i + 1]) result[0] = 1;  // every writer stores the same word
}

// Records built in shared memory and stored as 16-byte vectors: the target may be another GPU's HBM
// (peer mapping of rank 0's receive buffer, acb_comm.hpp), where full lines per warp store matter
// more than at home.  256 records per CTA.  Record = acg_match { u32 pid; u32 pad; u64 start; u64 end }.
constexpr int kExpandThreads = 256;
__global__ void __launch_bounds__(kExpandThreads) expand_kernel(ExpandLaunch e) {
  __shared__ uint64_t s_rec[kExpandThreads * 3];
  const uint64_t m = e.t.n - e.first;
  // grid-stride over blocks of kExpandThreads records
  for (uint64_t base = (uint64_t)blockIdx.x * kExpandThreads; base < m; base += (uint64_t)gridDim.x * kExpandThreads) {
    const uint64_t i = base + threadIdx.x;
    if (i < m) {
      const uint32_t pid = e.t.pids[e.first + i];
      const MatchSpan span = decode_key(e.t.keys[e.first + i], pid, e.mode, e.span_start + e.offset_add, e.t.pattern_lens);
      s_rec[threadIdx.x * 3 + 0] = (uint64_t)pid;
      s_rec[threadIdx.x * 3 + 1] = span.start;
      s_rec[threadIdx.x * 3 + 2] = span.end;
    }
    __syncthreads();
    const uint64_t cnt = m - base < kExpandThreads ? m - base : kExpandThreads;  // records of this block
    uint64_t* dst = e.out + base * 3;
    const uint32_t words = (uint32_t)cnt * 3;  // 8-byte words
    // 16-byte vector stores from the first 16-byte boundary of the destination on (a rank's offset
    // in the global list can be odd, and a record is 24 bytes)
    const uint32_t head = (uint32_t)((reinterpret_cast<uintptr_t>(dst) >> 3) & 1);  // 8-byte words before the boundary
    if (head && threadIdx.x == 0 && words) dst[0] = s_rec[0];
    for (uint32_t w = head + threadIdx.x * 2; w + 1 < words; w += 2 * kExpandThreads)
      *reinterpret_cast<ulonglong2*>(dst + w) = make_ulonglong2(s_rec[w], s_rec[w + 1]);
    if (words > head && ((words - head) & 1) && threadIdx.x == 0) dst[words - 1] = s_rec[words - 1];
    __syncthreads();
  }
}

// keys are sorted: count the tuples with key < bound_key (single block, strided binary chunks)
__global__ void lower_bound_kernel(const uint64_t* keys, uint64_t n, uint64_t bound_key,
                                   unsigned long long* result) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (keys[mid] < bound_key) lo = mid + 1; else hi = mid;
  }
  *result = lo;
}

}  // namespace

cudaError_t launch_expand(const ExpandLaunch& e, cudaStream_t s) {
  const uint64_t m = e.t.n - e.first;
  if (m == 0) return cudaSuccess;
  ACB_LAUNCH(expand_kernel, (unsigned)((m + kExpandThreads - 1) / kExpandThreads), kExpandThreads, 0, s, e);
  return cudaGetLastError();
}
cudaError_t launch_lower_bound(const uint64_t* keys, uint64_t n, uint64_t bound_key,
                               unsigned long long* d_result, cudaStream_t s) {
  ACB_LAUNCH(lower_bound_kernel, 1, 32, 0, s, keys, n, bound_key, d_result);
  return cudaGetLastError();
}

cudaError_t launch_walk_overlapping(const DfaDev& dfa, const WalkLaunch& p, cudaStream_t s) {
  const uint64_t blocks = (p.n_segs + kWalkThreads - 1) / kWalkThreads;
  ACB_LAUNCH(walk_overlapping_kernel, (unsigned)blocks, kWalkThreads, 0, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_dfa_fill_level(const FillLaunch& f, cudaStream_t s) {
  if (f.n == 0) return cudaSuccess;
#ifdef ACB_EMULATE
  if (getenv("ACB_EMU_TRACE")) fprintf(stderr, "launch_dfa_fill_level rows %u\n", f.n);
#endif
  const uint64_t blocks = ((uint64_t)f.n * 32 + kFillThreads - 1) / kFillThreads;
  ACB_LAUNCH(dfa_fill_level_kernel, (unsigned)blocks, kFillThreads, 0, s, f);
  return cudaGetLastError();
}

cudaError_t launch_seq_docs(const DfaDev& dfa, const SeqDocsLaunch& p, cudaStream_t s) {
  if (p.n_docs == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((p.n_docs + kSeqDocThreads - 1) / kSeqDocThreads);
  if (p.overlapping) ACB_LAUNCH(seq_docs_kernel<true>, blocks, kSeqDocThreads, 0, s, dfa, p);
  else ACB_LAUNCH(seq_docs_kernel<false>, blocks, kSeqDocThreads, 0, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_doc_flags(const DocFlagsLaunch& f, cudaStream_t s) {
  if (f.t.n == 0) return cudaSuccess;
  ACB_LAUNCH(doc_flags_kernel, (unsigned)((f.t.n + 255) / 256), 256, 0, s, f);
  return cudaGetLastError();
}

cudaError_t launch_doc_first(const DocFlagsLaunch& f, cudaStream_t s) {
  if (f.n_docs == 0) return cudaSuccess;
  ACB_LAUNCH(doc_first_clear_kernel, (unsigned)((f.n_docs + 255) / 256), 256, 0, s, f);
  if (f.t.n == 0) return cudaGetLastError();
  ACB_LAUNCH(doc_flags_kernel, (unsigned)((f.t.n + 255) / 256), 256, 0, s, f);
  ACB_LAUNCH(doc_first_kernel, (unsigned)((f.t.n + 255) / 256), 256, 0, s, f);
  return cudaGetLastError();
}

cudaError_t launch_doc_records(const DocRecordsLaunch& e, cudaStream_t s) {
  if (e.t.n == 0) return cudaSuccess;
  ACB_LAUNCH(doc_records_kernel, (unsigned)((e.t.n + 255) / 256), 256, 0, s, e);
  return cudaGetLastError();
}

cudaError_t launch_count_keys(const CountKeysLaunch& c, cudaStream_t s) {
  if (c.t.n == 0) return cudaSuccess;
  ACB_LAUNCH(count_keys_kernel, (unsigned)((c.t.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_run_heads(const CountRunsLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(run_heads_kernel, (unsigned)((c.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_count_runs(const CountRunsLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(count_runs_kernel, (unsigned)((c.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_count_rows(const CountRunsLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(count_rows_kernel, (unsigned)((c.n_docs + 1 + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_cover_keys(const CoverLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(cover_keys_kernel, (unsigned)((c.t.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_cover_ends(const CoverLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(cover_ends_kernel, (unsigned)((c.t.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_cover_runs(const CoverLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(cover_runs_kernel, (unsigned)((c.t.n + 255) / 256), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_cover_mask(const CoverLaunch& c, cudaStream_t s) {
  ACB_LAUNCH(cover_mask_kernel, (unsigned)((c.t.n + 7) / 8), 256, 0, s, c);
  return cudaGetLastError();
}

cudaError_t launch_replace_keys(const ReplaceLaunch& r, cudaStream_t s) {
  ACB_LAUNCH(replace_keys_kernel, (unsigned)((r.t.n + 255) / 256), 256, 0, s, r);
  return cudaGetLastError();
}

cudaError_t launch_replace_rows(const ReplaceLaunch& r, cudaStream_t s) {
  ACB_LAUNCH(replace_rows_kernel, (unsigned)((r.n_docs + 1 + 255) / 256), 256, 0, s, r);
  return cudaGetLastError();
}

uint64_t replace_splice_tiles(const uint8_t* out, uint64_t out_len) {
  return ((reinterpret_cast<uintptr_t>(out) & 15) + out_len + kSpliceTile - 1) / kSpliceTile;
}

cudaError_t launch_replace_splice(const ReplaceLaunch& r, cudaStream_t s) {
  const uint64_t mis = reinterpret_cast<uintptr_t>(r.out) & 15, n_tiles = replace_splice_tiles(r.out, r.out_len);
  ACB_LAUNCH(replace_tiles_kernel, (unsigned)((n_tiles + 1 + 255) / 256), 256, 0, s, r, n_tiles, mis);
  ACB_LAUNCH(replace_splice_kernel, (unsigned)n_tiles, kSpliceThreads, 0, s, r, mis);
  return cudaGetLastError();
}

cudaError_t launch_stream_docs(const StreamLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(stream_docs_kernel, (unsigned)((p.n + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_gather(const StreamLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(stream_gather_kernel, (unsigned)((p.docs_len + kSpliceTile - 1) / kSpliceTile), kSpliceThreads, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_keep(const StreamLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(stream_keep_kernel, (unsigned)((p.m + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_records(const StreamLaunch& p, cudaStream_t s) {
  const uint64_t n = p.m > p.n + 1 ? p.m : p.n + 1;
  ACB_LAUNCH(stream_records_kernel, (unsigned)((n + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_state(const StreamLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(stream_state_kernel, (unsigned)((p.n * 32 + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_hold(const StreamLaunch& p, cudaStream_t s) {
  const uint64_t n = p.m > p.n ? p.m : p.n;
  ACB_LAUNCH(stream_hold_kernel, (unsigned)((n + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_stream_flush(const StreamLaunch& p, const uint64_t* ids, uint64_t n_ids,
                                const uint64_t* out_offsets, uint8_t* out, cudaStream_t s) {
  ACB_LAUNCH(stream_flush_kernel, (unsigned)((n_ids * 32 + 255) / 256), 256, 0, s, p, ids, n_ids, out_offsets, out);
  return cudaGetLastError();
}

cudaError_t launch_look_state(const DfaDev& dfa, const LookLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(look_state_kernel, (unsigned)((p.n_rows + kLookThreads - 1) / kLookThreads), kLookThreads, 0, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_look_heads(const LookLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(look_heads_kernel, (unsigned)((p.n_rows + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_look_compact(const LookLaunch& p, cudaStream_t s) {
  ACB_LAUNCH(look_compact_kernel, (unsigned)((p.n_rows + 255) / 256), 256, 0, s, p);
  return cudaGetLastError();
}

// Eight CTAs of 256 threads fill an SM; no more warps than the largest U (n_rows) could use.
cudaError_t launch_look_mask(const DfaDev& dfa, const LookLaunch& p, cudaStream_t s) {
  const uint64_t warps = p.n_rows * ((p.n_cands + 31) >> 5), per_cta = kLookThreads / 32;
  const uint64_t grid = std::min<uint64_t>((uint64_t)p.sm_count * 8, (warps + per_cta - 1) / per_cta);
  ACB_LAUNCH(look_mask_kernel, (unsigned)grid, kLookThreads, 0, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_look_copy(const LookLaunch& p, cudaStream_t s) {
  const uint64_t items = p.n_rows * ((p.n_cands + kSpliceTile - 1) / kSpliceTile);
  const uint64_t grid = std::min<uint64_t>((uint64_t)p.sm_count * 8, items);
  ACB_LAUNCH(look_copy_kernel, (unsigned)grid, kSpliceThreads, 0, s, p);
  return cudaGetLastError();
}

cudaError_t launch_check_offsets(const uint64_t* offs, uint64_t n_docs, uint64_t hay_len,
                                 unsigned long long* result, cudaStream_t s) {
  ACB_LAUNCH(check_offsets_kernel, (unsigned)(n_docs / 256 + 1), 256, 0, s, offs, n_docs, hay_len, result);
  return cudaGetLastError();
}

cudaError_t inclusive_sum_u64(void* d_temp, size_t& temp_bytes, const unsigned long long* in, unsigned long long* out,
                              uint64_t n, cudaStream_t s) {
  return cub::DeviceScan::InclusiveScan(d_temp, temp_bytes, in, out, SumOp(), (int64_t)n, s);
}

cudaError_t sort_pairs(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, uint64_t* keys_out,
                       const uint32_t* vals_in, uint32_t* vals_out, uint64_t n, int end_bit,
                       cudaStream_t s) {
  return cub::DeviceRadixSort::SortPairs(d_temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, n,
                                         0, end_bit, s);
}

}  // namespace acb
