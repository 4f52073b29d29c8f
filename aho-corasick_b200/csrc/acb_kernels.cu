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
// more than at home.  Two sizes: 256 records per CTA, and a small one -- 128 threads, 3 KB of shared
// memory -- that fits beside the persistent scan CTA of the next sharded step on the same SM, so that
// the transfer overlaps that scan.  Record = acg_match { u32 pid; u32 pad; u64 start; u64 end }.
template <int kExpandThreads>
__global__ void __launch_bounds__(kExpandThreads) expand_kernel(ExpandLaunch e) {
  __shared__ uint64_t s_rec[kExpandThreads * 3];
  const uint64_t m = e.t.n - e.first;
  // grid-stride over blocks of kExpandThreads records (the small form runs one CTA per SM)
  for (uint64_t base = (uint64_t)blockIdx.x * kExpandThreads; base < m; base += (uint64_t)gridDim.x * kExpandThreads) {
    const uint64_t i = base + threadIdx.x;
    if (i < m) {
      const uint32_t pid = e.t.pids[e.first + i];
      const MatchSpan span = decode_key(e.t.keys[e.first + i], pid, 0, e.span_start + e.offset_add, e.t.pattern_lens);
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
  if (e.small) {
    // one small CTA per SM at most: the persistent scan CTA of the next step must still fit beside it
    const uint64_t blocks = (m + 127) / 128;
    ACB_LAUNCH(expand_kernel<128>, (unsigned)(blocks < (uint64_t)e.small ? blocks : (uint64_t)e.small), 128, 0, s, e);
  } else {
    ACB_LAUNCH(expand_kernel<256>, (unsigned)((m + 255) / 256), 256, 0, s, e);
  }
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
