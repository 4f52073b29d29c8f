// acb_api.cu -- the extern "C" boundary (include/acb200.h): handle management,
// input validation with the reference's error behaviour, device orchestration.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <pthread.h>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <new>
#include <optional>
#include <vector>

#include "../../include/acb200.h"
#include "../../include/acb200_debug.h"
#include "acb_build.hpp"
#include "acb_comm.hpp"
#include "acb_device.cuh"
#include "acb_plan.hpp"

using acb::DfaDev;
using acb::HostDfa;

namespace {

#define CK(expr)                                                                       \
  do {                                                                                 \
    cudaError_t e_ = (expr);                                                           \
    if (e_ != cudaSuccess) {                                                           \
      std::fprintf(stderr, "acb200: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e_), \
                   __FILE__, __LINE__, cudaGetErrorString(e_));                        \
      return ACG_E_CUDA;                                                               \
    }                                                                                  \
  } while (0)

// counters of a search: [0] tuples (bucketed emission: the overflow list), [1] candidates, [2] super-tiles,
// [kBucketCountersAt + b] the tuples of bucket b
constexpr size_t kCounterBytes = 8 * (acb::kBucketCountersAt + acb::kMaxBuckets);

// A buffer that owns its memory -- device, or page-locked host -- and only grows.  A grow discards the
// contents; after a failed allocation the buffer is empty, so a capacity never outlives its memory.
template <class T, bool kPinned>
struct Buf {
  T* p = nullptr;
  uint64_t cap = 0;  // elements
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  ~Buf() { release(); }
  operator T*() const { return p; }
  void release() {
    if (p) kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  int reserve(uint64_t n) {
    if (n <= cap) return ACG_OK;
    release();
    const cudaError_t e = kPinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e != cudaSuccess) p = nullptr;
    CK(e);
    cap = n;
    return ACG_OK;
  }
};
template <class T> using DevBuf = Buf<T, false>;
template <class T> using PinnedBuf = Buf<T, true>;

// Room for n elements in each of several buffers that share a sizing policy, or none of them: the ones that
// are too small are all released before the first is allocated (a grow never holds the old and the new memory
// together), and when an allocation fails the whole group is released, so that the next search starts from
// nothing instead of from a capacity that only some of the group have.
template <class... B>
int reserve_all(uint64_t n, B&... b) {
  ((b.cap < n ? b.release() : void()), ...);
  int rc = ACG_OK;
  ((rc = rc ? rc : b.reserve(n)), ...);
  if (rc) (b.release(), ...);
  return rc;
}

struct Workspace {
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
  DevBuf<uint64_t> d_keys[2];  // the tuple lists: all four of one capacity, or all empty (reserve_tuples)
  DevBuf<uint32_t> d_pids[2];
  uint64_t tuple_cap() const { return d_keys[0].cap; }
  DevBuf<unsigned long long> d_counter;
  PinnedBuf<unsigned long long> h_counter;
  DevBuf<uint8_t> d_temp;  // CUB temporary storage (cub_call): a search's CUB calls run in order on `stream`;
                           // after the last of them, the replace splice's tile index
  DevBuf<uint8_t> d_hay;  // staging of host haystacks
  DevBuf<uint64_t> d_scratch;  // chain resolution: end offsets / prefix max
  DevBuf<uint8_t> d_flags;
  DevBuf<uint64_t> d_rec;  // records of a host-output search, three words each, and their staging on the host
  PinnedBuf<uint64_t> h_rec;
  acg_stats stats{};  // of the search that holds (or last held) this workspace
  // pageable host haystacks: page-locked staging ring filled by host threads (run_prefilter)
  PinnedBuf<uint8_t> h_stage[2];
  cudaEvent_t stage_ev[2] = {nullptr, nullptr};
  // batched search, per document: offsets, counts, their inclusive scan, flags
  DevBuf<uint64_t> d_doc_offs;
  DevBuf<unsigned long long> d_doc_counts, d_doc_incl;
  DevBuf<uint8_t> d_doc_flags;
  // replace of a batch: the replacement table (offsets, then the bytes) and a host-output call's output
  DevBuf<uint64_t> d_rep;
  DevBuf<uint8_t> d_out;  // also a host-output stream feed's records
  // a stream feed: the combined documents tail | chunk, their offsets and the chunk offsets given on the host
  DevBuf<uint8_t> d_sdocs;
  DevBuf<uint64_t> d_soffs;
  DevBuf<uint64_t> d_held;  // a replace set's feed: the records of D with every stream's hold record
};

}  // namespace

struct acg_dfa {
  HostDfa h;
  std::vector<uint16_t> depth16;
  acb::PrefilterPlan pf;
  uint32_t* d_bitmap = nullptr;
  uint2* d_amap = nullptr;
  bool has_empty = false;
  uint32_t max_list_len = 0;
  bool on_device = false;
  bool dev_touched = false;  // upload() started: device resources may exist even if it failed
  int device = -1;
  uint32_t* d_trans = nullptr;
  uint8_t* d_classes = nullptr;
  uint32_t* d_moff = nullptr;
  uint32_t* d_mpids = nullptr;
  uint32_t* d_plens = nullptr;
  uint16_t* d_depth16 = nullptr;
  DfaDev dev{};
  int engine_override = ACG_ENGINE_AUTO;
  uint64_t pipeline_chunk = 64ull << 20;  // H2D chunk of the pipelined host path (acg_debug_set_pipeline_chunk)
  mutable bool bytescan_inert = false;    // the needles turned out to be frequent in a haystack: fingerprint filter from then on
  uint32_t experiment = 0;                // ACG_EXP_* kernel variants awaiting measurement (acg_debug_set_experiment)
  mutable std::mutex mu;  // configuration (engine / experiment knobs, lazy table fetch) and the workspace pool
  // Searches run through `&self` from many threads (the reference's automata are Send + Sync,
  // src/lib.rs:274-326): every search leases a workspace -- its own stream pair, events, tuple
  // buffers and haystack staging -- from this pool, so concurrent callers overlap on the device
  // instead of queueing behind one mutex.  Workspaces are created on demand, at most kMaxWorkspaces.
  static constexpr size_t kMaxWorkspaces = 4;
  mutable std::vector<Workspace*> ws_all, ws_free;
  mutable std::condition_variable ws_cv;
  mutable acg_stats last_stats{};  // of the search that finished last (acg_last_stats from another thread)
};

// A stream set (acg_streams_create): the state of StreamLaunch (acb_device.cuh) on the automaton's device.
// A replace set (acg_streams_create_replace) is a find_iter set that also holds its replacement table.
struct acg_streams {
  const acg_dfa* a = nullptr;
  uint64_t n = 0, back = 0;
  bool overlapping = false;
  bool replace = false;
  uint64_t* d_state = nullptr;  // [2 * n]: pos, then cursor
  uint8_t* d_tail = nullptr;    // [n * back]
  // replace sets: the caller's rep_offsets [patterns_len + 1], the last one again (the empty replacement of the
  // hold records, pid patterns_len), then the replacement bytes
  uint64_t* d_rep = nullptr;
};

// A candidate set (acg_candidates_create) on the automaton's device: the offsets, from 0, and the bytes already mapped
// through the automaton's byte classes, which is why it is bound to that automaton.
struct acg_candidates {
  const acg_dfa* a = nullptr;
  uint64_t n = 0;
  uint64_t* d_offs = nullptr;   // [n + 1]
  uint8_t* d_classes = nullptr;  // [d_offs[n]]
};

namespace {

// The workspace leased by the search running on this thread (WsLease below).
thread_local Workspace* tls_ws = nullptr;
thread_local const acg_dfa* tls_stats_owner = nullptr;
thread_local acg_stats tls_stats{};
Workspace& cur_ws() { return *tls_ws; }

int init_workspace(Workspace& w) {
  CK(cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&w.copy_stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&w.ev0));
  CK(cudaEventCreate(&w.ev1));
  CK(cudaEventCreate(&w.ev2));
  CK(cudaEventCreate(&w.ev3));
  int rc = w.d_counter.reserve(kCounterBytes / 8);
  return rc ? rc : w.h_counter.reserve(kCounterBytes / 8);
}

// The buffers free themselves when the workspace is deleted: right after this, on the handle's device.
void destroy_workspace(Workspace& w) {
  if (w.stream) cudaStreamSynchronize(w.stream);
  for (int i = 0; i < 2; ++i)
    if (w.stage_ev[i]) cudaEventDestroy(w.stage_ev[i]);
  if (w.ev0) cudaEventDestroy(w.ev0);
  if (w.ev1) cudaEventDestroy(w.ev1);
  if (w.ev2) cudaEventDestroy(w.ev2);
  if (w.ev3) cudaEventDestroy(w.ev3);
  if (w.stream) cudaStreamDestroy(w.stream);
  if (w.copy_stream) cudaStreamDestroy(w.copy_stream);
}

// RAII lease of one workspace of the handle for the duration of a search.
struct WsLease {
  const acg_dfa* a;
  Workspace* w = nullptr;
  Workspace* prev;
  int rc = ACG_OK;
  explicit WsLease(const acg_dfa* a_) : a(a_), prev(tls_ws) {
    std::unique_lock<std::mutex> lk(a->mu);
    for (;;) {
      if (!a->ws_free.empty()) { w = a->ws_free.back(); a->ws_free.pop_back(); break; }
      if (a->ws_all.size() < acg_dfa::kMaxWorkspaces) {
        w = new (std::nothrow) Workspace();
        if (!w) { rc = ACG_E_NOMEM; return; }
        a->ws_all.push_back(w);
        lk.unlock();
        int prev_dev = -1;
        cudaGetDevice(&prev_dev);
        if (prev_dev != a->device) cudaSetDevice(a->device);
        rc = init_workspace(*w);
        if (prev_dev != a->device && prev_dev >= 0) cudaSetDevice(prev_dev);
        break;  // a half-initialised workspace stays in ws_all and is destroyed with the handle
      }
      a->ws_cv.wait(lk);
    }
    if (rc == ACG_OK) { w->stats = acg_stats{}; tls_ws = w; }
  }
  // Keep the workspace beyond this scope (a sharded step whose expand kernel is still reading its
  // tuples); release_workspace() hands it back.
  Workspace* detach() {
    Workspace* out = w;
    if (w) { tls_stats = w->stats; tls_stats_owner = a; tls_ws = prev; }
    w = nullptr;
    return out;
  }
  ~WsLease() {
    if (!w) return;
    tls_stats = w->stats;
    tls_stats_owner = a;
    tls_ws = prev;
    std::lock_guard<std::mutex> lk(a->mu);
    a->last_stats = w->stats;
    if (rc == ACG_OK) a->ws_free.push_back(w);
    a->ws_cv.notify_one();
  }
};

void release_workspace(const acg_dfa* a, Workspace* w) {
  if (!w) return;
  std::lock_guard<std::mutex> lk(a->mu);
  a->last_stats = w->stats;
  a->ws_free.push_back(w);
  a->ws_cv.notify_one();
}

void derive_metadata(acg_dfa* a) {
  HostDfa& h = a->h;
  a->has_empty = h.min_pattern_len == 0 && !h.pattern_lens.empty();
  a->max_list_len = 0;
  for (size_t i = 0; i + 1 < h.match_offsets.size(); ++i)
    a->max_list_len = std::max(a->max_list_len, h.match_offsets[i + 1] - h.match_offsets[i]);
  // Trie depth of every row = BFS distance from the unanchored start row: one transition
  // deepens the longest-suffix state by at most one byte, and a state of depth d is reached by
  // its own d bytes.  The builder hands it over for tables it built; adopted tables are walked.
  const uint32_t s2 = h.stride2;
  const size_t rows = size_t(h.state_len);
  auto bfs_depth = [&]() {
    std::vector<uint32_t> dist(rows, UINT32_MAX);
    std::vector<uint32_t> q;
    if (h.start_unanchored_id) {
      dist[h.start_unanchored_id >> s2] = 0;
      q.push_back(h.start_unanchored_id >> s2);
    }
    for (size_t qi = 0; qi < q.size(); ++qi) {
      const uint32_t r = q[qi];
      const uint32_t* row = h.trans.data() + (size_t(r) << s2);
      for (uint32_t c = 0; c < h.alphabet_len; ++c) {
        const uint32_t nr = row[c] >> s2;
        if (nr == 0 || dist[nr] != UINT32_MAX) continue;
        dist[nr] = dist[r] + 1;
        q.push_back(nr);
      }
    }
    std::vector<uint16_t> out(rows, 0xFFFF);
    for (size_t r = 0; r < rows; ++r)
      if (dist[r] != UINT32_MAX) out[r] = uint16_t(std::min<uint32_t>(dist[r], 0xFFFE));
    return out;
  };
  if (h.row_depth.size() == rows) {
    a->depth16 = h.row_depth;  // tests/test_adopt_tables_host.py: equals bfs_depth() of the same table
  } else {
    a->depth16 = bfs_depth();
  }
  a->pf = acb::plan_prefilter(h, a->depth16, (a->experiment & ACG_EXP_KEY24) != 0);
}

// Dense table produced on the device from the builder's DenseFillPlan (acb_build.hpp): one
// launch per BFS level.  The plan's arrays are freed afterwards; the host never holds the table
// unless acg_dfa_table asks for it (fetch_table).
int fill_table_on_device(acg_dfa* a) {
  HostDfa& h = a->h;
  const acb::DenseFillPlan& f = h.fill;
  const size_t n = f.row.size();
  uint32_t *d_row = nullptr, *d_inh = nullptr, *d_fill = nullptr, *d_eoff = nullptr, *d_eto = nullptr;
  uint8_t* d_ecls = nullptr;
  auto release = [&]() {
    cudaFree(d_row); cudaFree(d_inh); cudaFree(d_fill); cudaFree(d_eoff); cudaFree(d_eto); cudaFree(d_ecls);
  };
  auto up = [&](auto** dptr, const void* src, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(dptr), std::max<size_t>(bytes, 16));
    if (e != cudaSuccess) return e;
    if (bytes) e = cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice);
    return e;
  };
  cudaError_t e = cudaMalloc(&a->d_trans, std::max<size_t>(size_t(h.trans_len) * 4, 16));
  if (e == cudaSuccess) e = cudaMemset(a->d_trans, 0, size_t(h.trans_len) * 4);
  if (e == cudaSuccess) e = up(&d_row, f.row.data(), n * 4);
  if (e == cudaSuccess) e = up(&d_inh, f.inherit_row.data(), n * 4);
  if (e == cudaSuccess) e = up(&d_fill, f.fill_id.data(), n * 4);
  if (e == cudaSuccess) e = up(&d_eoff, f.edge_off.data(), f.edge_off.size() * 4);
  if (e == cudaSuccess) e = up(&d_eto, f.edge_to.data(), f.edge_to.size() * 4);
  if (e == cudaSuccess) e = up(&d_ecls, f.edge_class.data(), f.edge_class.size());
  for (size_t l = 0; e == cudaSuccess && l + 1 < f.level_off.size(); ++l) {
    const uint32_t lo = f.level_off[l], hi = f.level_off[l + 1];
    acb::FillLaunch p;
    p.trans = a->d_trans;
    p.stride2 = h.stride2;
    p.alphabet_len = h.alphabet_len;
    p.row = d_row + lo;
    p.inherit_row = d_inh + lo;
    p.fill_id = d_fill + lo;
    p.edge_off = d_eoff + lo;
    p.edge_class = d_ecls;
    p.edge_to = d_eto;
    p.n = hi - lo;
    e = acb::launch_dfa_fill_level(p, nullptr);  // default stream: levels run in order
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  release();
  if (e != cudaSuccess) { cudaGetLastError(); return ACG_E_CUDA; }
  // the per-row arrays have served their purpose; `shallow` stays (the plan can be re-derived)
  acb::DenseFillPlan& fp = h.fill;
  std::vector<uint32_t>().swap(fp.level_off);
  std::vector<uint32_t>().swap(fp.row);
  std::vector<uint32_t>().swap(fp.inherit_row);
  std::vector<uint32_t>().swap(fp.fill_id);
  std::vector<uint32_t>().swap(fp.edge_off);
  std::vector<uint8_t>().swap(fp.edge_class);
  std::vector<uint32_t>().swap(fp.edge_to);
  return ACG_OK;
}

int upload(acg_dfa* a) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return ACG_E_NO_DEVICE;
  }
  CK(cudaGetDevice(&a->device));
  a->dev_touched = true;
  HostDfa& h = a->h;
  auto up = [&](auto** dptr, const void* src, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(dptr), std::max<size_t>(bytes, 16));
    if (e != cudaSuccess) return e;
    if (bytes) e = cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice);
    return e;
  };
  if (h.fill.valid) {
    int rc = fill_table_on_device(a);
    if (rc) return rc;
  } else {
    CK(up(&a->d_trans, h.trans.data(), h.trans.size() * 4));
  }
  CK(up(&a->d_classes, h.classes, 256));
  CK(up(&a->d_moff, h.match_offsets.data(), h.match_offsets.size() * 4));
  CK(up(&a->d_mpids, h.match_pids.data(), h.match_pids.size() * 4));
  CK(up(&a->d_plens, h.pattern_lens.data(), h.pattern_lens.size() * 4));
  CK(up(&a->d_depth16, a->depth16.data(), a->depth16.size() * 2));
  if (a->pf.supported && !a->pf.bitmap.empty()) CK(up(&a->d_bitmap, a->pf.bitmap.data(), a->pf.bitmap.size() * 4));
  if (a->pf.supported && !a->pf.amap.empty()) CK(up(&a->d_amap, a->pf.amap.data(), a->pf.amap.size() * 8));
  DfaDev& d = a->dev;
  d.trans = a->d_trans;
  d.classes = a->d_classes;
  d.match_offsets = a->d_moff;
  d.match_pids = a->d_mpids;
  d.pattern_lens = a->d_plens;
  d.depth16 = a->d_depth16;
  d.stride2 = h.stride2;
  d.max_match_id = h.max_match_id;
  d.start_unanchored_id = h.start_unanchored_id;
  d.start_anchored_id = h.start_anchored_id;
  d.max_pattern_len = uint32_t(std::min<uint64_t>(h.max_pattern_len, UINT32_MAX));
  d.min_pattern_len = uint32_t(std::min<uint64_t>(h.min_pattern_len, UINT32_MAX));
  d.amap = a->d_amap;
  acb::plan_device_fields(a->pf, d);
  a->on_device = true;
  return ACG_OK;
}

int reserve_tuples(Workspace& w, uint64_t cap) {
  return reserve_all(cap, w.d_keys[0], w.d_pids[0], w.d_keys[1], w.d_pids[1]);
}

// One CUB call `f(d_temp, temp_bytes)` on the workspace's temporary storage: sized by a query
// (d_temp == nullptr, which CUB answers without doing the work) and grown if the call needs more.
template <class F>
int cub_call(Workspace& w, F f) {
  size_t tb = 0;
  CK(f(nullptr, tb));
  int rc = w.d_temp.reserve(std::max<size_t>(tb, 16));
  if (rc) return rc;
  tb = w.d_temp.cap;
  CK(f(w.d_temp, tb));
  return ACG_OK;
}

// host output: room for n records on the device and on their way to the caller
int reserve_rec(Workspace& w, uint64_t n) {
  n = std::max<uint64_t>(n, 1 << 16) * 3;
  int rc = w.d_rec.reserve(n);
  return rc ? rc : w.h_rec.reserve(n);
}

// batched search: room for n entries in each per-document array
int reserve_docs(Workspace& w, uint64_t n) {
  return reserve_all(std::max<uint64_t>(n, 1 << 12), w.d_doc_offs, w.d_doc_counts, w.d_doc_incl, w.d_doc_flags);
}

// enforce_anchored_consistency, src/ahocorasick.rs:2778-2789
int check_anchored(int have, int want_anchored) {
  if (have == ACG_START_BOTH) return ACG_OK;
  if (have == ACG_START_UNANCHORED) return want_anchored ? ACG_E_INVALID_INPUT_ANCHORED : ACG_OK;
  return want_anchored ? ACG_OK : ACG_E_INVALID_INPUT_UNANCHORED;
}
// Input::set_span, src/util/search.rs:332-343 (the reference panics; we return a code)
bool span_ok(uint64_t hay_len, uint64_t s, uint64_t e) { return e <= hay_len && s <= e + 1; }
// DFA::start_state, src/dfa.rs:192-215
int check_start(const HostDfa& h, int anchored) {
  if (anchored) return h.start_anchored_id == 0 ? ACG_E_INVALID_INPUT_ANCHORED : ACG_OK;
  return h.start_unanchored_id == 0 ? ACG_E_INVALID_INPUT_UNANCHORED : ACG_OK;
}

struct TupleResult {
  uint64_t n = 0;
  int sorted_buf = 0;
};

// A batched search's documents (device copy of the CSR offsets) as seen by the prefilter engine.
struct DocBatch {
  const uint64_t* d_offsets = nullptr;
  uint64_t n = 0;
  bool unordered = false;  // is_match: one list, no order step (only the documents of the tuples matter)
};

// Bucketed emission of the prefilter engine (PrefilterLaunch::bucket_shift): the span's key offsets
// [0, n_bytes] are cut into `n` ranges of 2^shift bytes, fixed before the first launch, and each
// bucket is given 2^log slots of tuple buffer 0, so that K4 is one shared-memory sort per bucket
// (order_buckets_kernel) instead of a radix sort of the whole list.
// The shift: 2^25 bytes (32 MiB) -- about 8 K tuples at the BASELINE density of one match per 4 KiB,
// half of what one CTA sorts (kOrderCap = 16 K) -- unless the 32-bit sort key needs smaller buckets
// (2^shift << tie_bits <= 2^32) or more than kMaxBuckets of them would be needed (then larger ones).
// When the tie-break needs more than 10 bits (patterns of 1 KiB and more, or many duplicates) the
// buckets would be under 4 MiB and their slots would outnumber the list's default capacity (one
// tuple per 256 bytes): the single list and the radix sort then stay.  So do the walk engine and
// the global super-tile distribution.  A bucket that fills up sends its further tuples to an
// overflow list behind the buckets, and K4 falls back to the radix sort.
struct BucketPlan {
  uint32_t shift = 0;  // 0: a single list
  uint32_t n = 0, log = 0, tie_bits = 0;  // buckets, log2 of the slots per bucket, bits of the tie-break
  uint64_t slots() const { return uint64_t(n) << log; }
};

BucketPlan plan_buckets(const acg_dfa* a, uint64_t n_bytes) {
  BucketPlan b;
  if (a->experiment & ACG_EXP_GLOBAL_TILES) return b;
  const uint32_t tie_bits = uint32_t(acb::bit_width(a->h.max_pattern_len)) + a->pf.dup_shift;
  if (tie_bits >= 32) return b;
  const uint32_t max_shift = 32 - tie_bits;
  uint32_t shift = std::min<uint32_t>(25, max_shift);
  uint32_t min_shift = 22;
  uint32_t log = acb::kOrderLog;
#ifdef ACB_EMULATE
  // dry run: smaller buckets / capacities, so that kilobyte inputs cross many buckets and overflow them
  if (const char* e = getenv("ACB_EMU_BUCKETSHIFT")) { shift = std::min<uint32_t>(uint32_t(atoi(e)), max_shift); min_shift = 1; }
  if (const char* e = getenv("ACB_EMU_BUCKETLOG")) log = std::min<uint32_t>(uint32_t(std::max(atoi(e), 0)), acb::kOrderLog);
#endif
  if (shift < min_shift) return b;
  while ((n_bytes >> shift) + 1 > acb::kMaxBuckets) {
    if (shift >= max_shift) return b;
    ++shift;
  }
  b.shift = shift;
  b.n = uint32_t((n_bytes >> shift) + 1);
  b.log = log;
  b.tie_bits = tie_bits;
  return b;
}

// Enqueue one K3/K3b launch covering the start offsets [scan_lo, scan_hi) of the span.
int enqueue_prefilter_range(const acg_dfa* a, const uint8_t* d_hay, uint64_t readable,
                            uint64_t span_start, uint64_t span_end, uint64_t scan_lo,
                            uint64_t scan_hi, int mode, int dev_sms, const BucketPlan& bp,
                            const DocBatch* docs) {
  Workspace& w = cur_ws();
  const acb::PrefilterPlan& pf = a->pf;
  // 16-byte aligned filter region whose 4-byte look-ahead stays inside the readable bytes
  const uintptr_t base = reinterpret_cast<uintptr_t>(d_hay);
  uint64_t lo = scan_lo + ((16 - ((base + scan_lo) & 15)) & 15);
  const uint64_t limit = std::min<uint64_t>(scan_hi, readable >= 20 ? readable - 20 : 0);
  uint64_t hi = lo;
  if (limit > lo) hi = lo + ((limit - lo) & ~15ull);
  if (lo > scan_hi) { lo = scan_hi; hi = scan_hi; }
  acb::PrefilterLaunch p;
  p.hay = d_hay;
  p.hay_len = readable;
  p.span_start = span_start;
  p.span_end = span_end;
  p.bitmap = a->d_bitmap;
  p.log_bits = pf.log_bits;
  p.k = pf.k;
  p.stride = pf.stride;
  // kernel geometry as planned; second-stage organisation and tile distribution: see prefilter_kernel
  p.geom = pf.wide ? 1 : 0;
  p.dyn = (a->experiment & ACG_EXP_STATIC_TILES) ? 0 : ((a->experiment & ACG_EXP_GLOBAL_TILES) ? 2 : 1);
  p.kmask = pf.kmask;
  p.fold = pf.fold;
  p.mult = pf.mult;
  p.mult3 = pf.mult3;
  p.key_shift = pf.key_shift;
  p.shift = pf.shift;
  p.dense = pf.dense ? 1 : 0;
  p.brute = pf.brute ? 1 : 0;
  p.mode = mode == 1 ? 1 : 0;
  p.first_only = mode == 2 ? 1 : 0;  // mode 2: all occurrences for a non-overlapping consumer
  p.dup_shift = pf.dup_shift;
  p.scan_lo = scan_lo;
  p.scan_hi = scan_hi;
  p.region_lo = lo;
  p.region_hi = hi;
  p.keys = w.d_keys[0];
  p.pids = w.d_pids[0];
  p.counter = w.d_counter;
  p.cap = w.tuple_cap();
  p.bucket_shift = bp.shift;
  p.bucket_log = bp.log;
  p.bucket_slots = bp.slots();
  p.doc_offsets = docs ? docs->d_offsets : nullptr;
  p.n_docs = docs ? docs->n : 0;
  p.bs_n = 0;
  for (int i = 0; i < 3; ++i) { p.bs_needle[i] = 0; p.bs_back[i] = 0; }
  if (pf.bs_n && !a->bytescan_inert && !(a->experiment & ACG_EXP_NO_BYTESCAN)) {
    p.bs_n = pf.bs_n;
    for (uint32_t i = 0; i < pf.bs_n; ++i) { p.bs_needle[i] = uint32_t(pf.bs_byte[i]) * 0x01010101u; p.bs_back[i] = pf.bs_back[i]; }
    CK(acb::launch_bytescan(a->dev, p, dev_sms, w.stream));
  } else {
    // counter[2]: the launch's global super-tile counter (dynamic tile distribution), zero at launch
    if (p.dyn == 2) CK(cudaMemsetAsync(w.d_counter + 2, 0, 8, w.stream));
    CK(acb::launch_prefilter(a->dev, p, dev_sms, w.stream));
  }
  cur_ws().stats.launches += 1;
  return ACG_OK;
}

// K4: order the appended tuples; `want` tuples sit in buffer 0 -- as one list, or (bucketed) in the
// buckets of `bp` and, `overflow` of them, in the overflow list behind the buckets.  Leaves them ordered
// in buffer res->sorted_buf.  Everything between ev2 and ev3 is the order time.
int order_tuples(const acg_dfa* a, uint64_t want, uint64_t n_bytes, TupleResult* res, const BucketPlan& bp,
                 uint64_t overflow) {
  Workspace& w = cur_ws();
  res->n = want;
  cur_ws().stats.raw_matches = want;
  res->sorted_buf = 0;
  if (want <= 1 && (bp.shift == 0 || want == 0)) return ACG_OK;  // (one bucketed tuple still has to move to slot 0)
  const int end_bit = std::min(64, acb::kTieBits + acb::bit_width(n_bytes + 1));
  float ms = 0;
  CK(cudaEventRecord(w.ev2, w.stream));
  // the list in buffer `from`, ordered into the other one
  auto sort_list = [&](int from) {
    return cub_call(w, [&](void* t, size_t& tb) {
      return acb::sort_pairs(t, tb, w.d_keys[from], w.d_keys[1 - from], w.d_pids[from], w.d_pids[1 - from], want,
                             end_bit, w.stream);
    });
  };
  int rc;
  if (bp.shift == 0) {
    if ((rc = sort_list(0))) return rc;
    cur_ws().stats.launches += 8;  // radix passes (library code, upper bound)
    res->sorted_buf = 1;
  } else {
    acb::OrderLaunch o;
    o.keys_in = w.d_keys[0];
    o.pids_in = w.d_pids[0];
    o.keys_out = w.d_keys[1];
    o.pids_out = w.d_pids[1];
    o.bucket_count = w.d_counter + acb::kBucketCountersAt;
    o.overflow_count = w.d_counter;
    o.n_buckets = bp.n;
    o.bucket_shift = bp.shift;
    o.bucket_cap = 1u << bp.log;
    o.tie_bits = bp.tie_bits;
    o.bucket_slots = bp.slots();
    if (overflow == 0) {
      // every bucket within what one CTA sorts: the buckets' order is the keys' order already
      CK(acb::launch_order_buckets(o, w.stream));
      cur_ws().stats.launches += 1;
      res->sorted_buf = 1;
    } else {
      // a bucket overflowed: concatenate buckets and overflow list, radix sort of the whole list
      CK(acb::launch_compact_buckets(o, w.stream));
      if ((rc = sort_list(1))) return rc;
      cur_ws().stats.launches += 9;
      res->sorted_buf = 0;
    }
  }
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  cur_ws().stats.order_ms = ms;
  return ACG_OK;
}

// K1 + K4 on a device-resident haystack; leaves `n` ordered tuples in
// ws.d_keys[sorted_buf] / ws.d_pids[sorted_buf].
int run_walk_overlapping(const acg_dfa* a, const uint8_t* d_hay, uint64_t readable, uint64_t span_start,
                         uint64_t span_end, TupleResult* res) {
  Workspace& w = cur_ws();
  const uint64_t n_bytes = span_end - span_start;
  if (a->max_list_len >= (1u << acb::kTieBits)) return ACG_E_INVALID_ARG;
  if (n_bytes >= (1ull << (64 - acb::kTieBits))) return ACG_E_INVALID_ARG;
  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, a->device);
  const uint64_t target_lanes = uint64_t(dev_sms) * 2048;
  uint64_t seg_len = (n_bytes + target_lanes - 1) / std::max<uint64_t>(target_lanes, 1);
  seg_len = std::max<uint64_t>(seg_len, 256);
  seg_len = (seg_len + 15) & ~15ull;
  // shard starts are placed so that (d_hay + span_start + k*seg_len) keeps the 16-byte
  // phase of the first shard; the kernel handles the unaligned head per lane.
  const uint64_t n_segs = std::max<uint64_t>((n_bytes + seg_len - 1) / seg_len, 1);
  uint64_t cap = std::max<uint64_t>(w.tuple_cap(), std::max<uint64_t>(1 << 20, n_bytes / 256));
  for (int attempt = 0; attempt < 8; ++attempt) {
    int rc = reserve_tuples(w, cap);
    if (rc) return rc;
    CK(cudaMemsetAsync(w.d_counter, 0, 8, w.stream));
    acb::WalkLaunch p;
    p.hay = d_hay;
    p.hay_len = readable;
    p.span_start = span_start;
    p.span_end = span_end;
    p.seg_len = seg_len;
    p.n_segs = n_segs;
    p.keys = w.d_keys[0];
    p.pids = w.d_pids[0];
    p.counter = w.d_counter;
    p.cap = w.tuple_cap();
    CK(cudaEventRecord(w.ev0, w.stream));
    CK(acb::launch_walk_overlapping(a->dev, p, w.stream));
    CK(cudaEventRecord(w.ev1, w.stream));
    CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 8, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    cur_ws().stats.launches += 1;
    const uint64_t want = *w.h_counter;
    if (want > w.tuple_cap()) { cap = want + want / 8 + 1024; continue; }  // overflow: grow and rescan
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev0, w.ev1);
    cur_ws().stats.scan_ms = ms;
    return order_tuples(a, want, n_bytes, res, BucketPlan{}, 0);
  }
  return ACG_E_NOMEM;
}

// ---- pageable host haystacks ---------------------------------------------------------------------
// cudaMemcpyAsync from pageable memory is staged by the driver through its own page-locked buffers by
// a single thread, several times slower than a copy from pinned memory.  A caller that
// hands over an ordinary allocation (a Rust Vec<u8>, a numpy array) gets the same pipeline with the
// staging done here: host threads copy each chunk into a page-locked ring buffer while the previous
// chunk is on its way over PCIe.
class CopyPool {
 public:
  static CopyPool& get() {
    // never destroyed: the workers wait on its condition variable for the life of the process, and
    // destroying a condition variable that has waiters blocks (exit would hang).  A forked child has
    // none of the parent's threads: it drops the inherited object and starts its own pool on demand.
    static std::once_flag once;
    std::call_once(once, [] { pthread_atfork(nullptr, nullptr, [] { instance().store(nullptr); }); });
    CopyPool* p = instance().load(std::memory_order_acquire);
    if (!p) {
      CopyPool* fresh = new CopyPool;
      if (instance().compare_exchange_strong(p, fresh)) p = fresh;
      // (lost the race: `fresh` stays allocated -- its workers are parked for good, a few KB once)
    }
    return *p;
  }
  // dst[0, n) = src[0, n), split over the pool's threads; returns when done
  void copy(uint8_t* dst, const uint8_t* src, size_t n) {
    if (n < (4u << 20) || workers_.empty()) { std::memcpy(dst, src, n); return; }
    std::unique_lock<std::mutex> lk(mu_);
    busy_cv_.wait(lk, [&] { return !active_; });  // one copy at a time: the pool is shared by all handles
    active_ = true;
    dst_ = dst; src_ = src; n_ = n;
    next_.store(0);
    pending_ = int(workers_.size());
    ++epoch_;
    cv_.notify_all();
    done_cv_.wait(lk, [&] { return pending_ == 0; });
    active_ = false;
    busy_cv_.notify_one();
  }

 private:
  static std::atomic<CopyPool*>& instance() {
    static std::atomic<CopyPool*> p{nullptr};
    return p;
  }
  CopyPool() {
    unsigned n = std::thread::hardware_concurrency();
    n = n >= 16 ? 8 : (n >= 4 ? n / 2 : 0);
    for (unsigned i = 0; i < n; ++i) workers_.emplace_back([this] { run(); });
    for (auto& t : workers_) t.detach();  // process-lifetime pool
  }
  void run() {
    uint64_t seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> lk(mu_);
      cv_.wait(lk, [&] { return epoch_ != seen; });
      seen = epoch_;
      uint8_t* dst = dst_;
      const uint8_t* src = src_;
      const size_t n = n_;
      lk.unlock();
      constexpr size_t kSlice = 1u << 20;
      for (;;) {
        const size_t off = next_.fetch_add(kSlice);
        if (off >= n) break;
        std::memcpy(dst + off, src + off, std::min(kSlice, n - off));
      }
      lk.lock();
      if (--pending_ == 0) done_cv_.notify_one();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_, done_cv_, busy_cv_;
  std::vector<std::thread> workers_;
  uint8_t* dst_ = nullptr;
  const uint8_t* src_ = nullptr;
  size_t n_ = 0;
  std::atomic<size_t> next_{0};
  int pending_ = 0;
  uint64_t epoch_ = 0;
  bool active_ = false;
};

bool is_pageable_host(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return attr.type == cudaMemoryTypeUnregistered;
}

// The staging ring of a pageable host haystack: two buffers of `bytes`, and the event that guards each.
int reserve_stage(Workspace& w, uint64_t bytes) {
  for (int i = 0; i < 2; ++i) {
    int rc = w.h_stage[i].reserve(bytes);
    if (rc) return rc;
    if (!w.stage_ev[i]) CK(cudaEventCreateWithFlags(&w.stage_ev[i], cudaEventDisableTiming));
  }
  return ACG_OK;
}

// K3/K3b (+ K4): prefilter engine.  mode 0 leaves all occurrences ordered like
// find_overlapping_iter; mode 1 leaves the best match per start offset ordered by start (input of
// the chain resolution).  When `h_hay` is given the span is first copied from (pinned) host
// memory in chunks on the copy stream, and each chunk is scanned as soon as it has landed, so the
// H2D copy and the scan overlap.
int run_prefilter(const acg_dfa* a, const uint8_t* d_hay, uint64_t readable, uint64_t span_start,
                  uint64_t span_end, int mode, TupleResult* res, const uint8_t* h_hay = nullptr,
                  uint64_t scan_lo = UINT64_MAX, uint64_t scan_hi = UINT64_MAX, const DocBatch* docs = nullptr) {
  if (scan_lo == UINT64_MAX) { scan_lo = span_start; scan_hi = span_end; }
  const bool unordered = docs && docs->unordered;
  Workspace& w = cur_ws();
  const uint64_t n_bytes = span_end - span_start;
  if (n_bytes >= (1ull << (64 - acb::kTieBits))) return ACG_E_INVALID_ARG;
  int dev_sms = 132;
  cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, a->device);
  // one tuple per 256 haystack bytes to start with (the BASELINE workloads have one per 4 KiB);
  // denser outputs are detected through the counter and the scan is repeated with room
  uint64_t cap = std::max<uint64_t>(w.tuple_cap(), std::max<uint64_t>(1 << 20, (scan_hi - scan_lo) / 256));
  // bucketed emission: the buckets' slots, then at least 64 K slots of overflow list
  const BucketPlan bp = unordered ? BucketPlan{} : plan_buckets(a, n_bytes);
  cap = std::max<uint64_t>(cap, bp.slots() + (bp.shift ? (1u << 16) : 0));
  const size_t counter_bytes = bp.shift ? 8 * (acb::kBucketCountersAt + size_t(bp.n)) : 16;
  bool copied = h_hay == nullptr;
  for (int attempt = 0; attempt < 8; ++attempt) {
    int rc = reserve_tuples(w, cap);
    if (rc) return rc;
    CK(cudaMemsetAsync(w.d_counter, 0, counter_bytes, w.stream));
    CK(cudaEventRecord(w.ev0, w.stream));
    if (copied) {
      if ((rc = enqueue_prefilter_range(a, d_hay, readable, span_start, span_end, scan_lo, scan_hi, mode,
                                        dev_sms, bp, docs)))
        return rc;
    } else {
      // chunked H2D on the copy stream; a chunk's start offsets are scanned once the bytes a
      // verification can touch (max_pattern_len + fingerprint look-ahead) have landed
      const uint64_t chunk = a->pipeline_chunk;
      const uint64_t tail = std::min<uint64_t>(a->h.max_pattern_len, 1u << 30) + 64;
      uint64_t scanned = span_start;
      // pageable source: the chunk goes through a page-locked ring buffer filled by host threads
      const bool staged = span_end - span_start >= std::min<uint64_t>(8u << 20, chunk) && is_pageable_host(h_hay + span_start);
      if (staged && (rc = reserve_stage(w, std::min<uint64_t>(chunk, span_end - span_start)))) return rc;
      bool stage_used[2] = {false, false};
      int stage_i = 0;
      CK(cudaEventRecord(w.ev2, w.copy_stream));
      for (uint64_t c0 = span_start; c0 < span_end; c0 += chunk) {
        const uint64_t c1 = std::min(span_end, c0 + chunk);
        const uint8_t* src = h_hay + c0;
        if (staged) {
          if (stage_used[stage_i]) CK(cudaEventSynchronize(w.stage_ev[stage_i]));  // its previous H2D copy has left the buffer
          CopyPool::get().copy(w.h_stage[stage_i], h_hay + c0, size_t(c1 - c0));
          src = w.h_stage[stage_i];
        }
        CK(cudaMemcpyAsync(const_cast<uint8_t*>(d_hay) + c0, src, c1 - c0, cudaMemcpyHostToDevice,
                           w.copy_stream));
        if (staged) {
          CK(cudaEventRecord(w.stage_ev[stage_i], w.copy_stream));
          stage_used[stage_i] = true;
          stage_i ^= 1;
        }
        CK(cudaEventRecord(w.ev3, w.copy_stream));
        CK(cudaStreamWaitEvent(w.stream, w.ev3, 0));
        const uint64_t upto = c1 == span_end ? span_end : (c1 > scanned + tail ? c1 - tail : scanned);
        if (upto > scanned || c1 == span_end) {
          if ((rc = enqueue_prefilter_range(a, d_hay, c1 == span_end ? readable : c1, span_start, span_end,
                                            scanned, upto, mode, dev_sms, bp, docs)))
            return rc;
          scanned = upto;
        }
      }
      copied = true;
    }
    CK(cudaEventRecord(w.ev1, w.stream));
    CK(cudaMemcpyAsync(w.h_counter, w.d_counter, counter_bytes, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    // bucketed: counter[0] is the length of the overflow list, the buckets' counters include the tuples
    // that went there
    uint64_t want = w.h_counter[0], overflow = 0, room = w.tuple_cap();
    if (bp.shift) {
      overflow = want;
      want = 0;
      for (uint32_t i = 0; i < bp.n; ++i) want += w.h_counter[acb::kBucketCountersAt + i];
      room = w.tuple_cap() - bp.slots();
    }
    cur_ws().stats.candidates = w.h_counter[1];
    // the reference retires a prefilter that keeps reporting candidates (PrefilterState,
    // src/util/prefilter.rs): needles in more than one offset out of 64 => fingerprint filter next time
    // (beyond that the verifications cost more than the fingerprint probes they replace)
    if (a->pf.bs_n && !a->bytescan_inert && scan_hi - scan_lo >= (1u << 16) && w.h_counter[1] > (scan_hi - scan_lo) / 64)
      a->bytescan_inert = true;
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev0, w.ev1);
    cur_ws().stats.scan_ms = ms;  // with a host haystack this is the overlapped copy+scan time
    if (bp.shift ? overflow > room : want > w.tuple_cap()) {
      const uint64_t need = bp.shift ? overflow : want;
      cap = (w.tuple_cap() - room) + need + need / 8 + 1024;
      continue;
    }
    if (unordered) {  // one list in buffer 0, in emission order
      res->n = want;
      res->sorted_buf = 0;
      cur_ws().stats.raw_matches = want;
      return ACG_OK;
    }
    return order_tuples(a, want, n_bytes, res, bp, overflow);
  }
  return ACG_E_NOMEM;
}

// The ordered tuples of `r` as the kernels that read them take them.
acb::TupleList tuple_list(const acg_dfa* a, const Workspace& w, const TupleResult& r) {
  return acb::TupleList{w.d_keys[r.sorted_buf], w.d_pids[r.sorted_buf], a->d_plens, r.n};
}

// FindIter over ordered candidate tuples, on the device: marks the tuples the reference's
// iterator yields and compacts them into the other tuple buffer.
int run_chain(const acg_dfa* a, int mode, TupleResult* r) {
  Workspace& w = cur_ws();
  if (r->n == 0) return ACG_OK;
  int rc = reserve_all(std::max<uint64_t>(r->n, 1 << 16), w.d_scratch, w.d_flags);
  if (rc) return rc;
  const int dst = 1 - r->sorted_buf;
  acb::ChainLaunch c;
  c.t = tuple_list(a, w, *r);
  c.mode = mode;
  c.scratch_end = w.d_scratch;
  c.flags = w.d_flags;
  CK(cudaEventRecord(w.ev2, w.stream));
  CK(cudaMemsetAsync(w.d_flags, 0, r->n, w.stream));
  CK(acb::launch_chain_ends(c, w.stream));
  if ((rc = cub_call(w, [&](void* t, size_t& tb) { return acb::scan_max_u64(t, tb, w.d_scratch, r->n, w.stream); })))
    return rc;
  CK(acb::launch_chain_select(c, w.stream));
  if ((rc = cub_call(w, [&](void* t, size_t& tb) {
         return acb::select_flagged(t, tb, c.t.keys, c.t.pids, w.d_flags, w.d_keys[dst], w.d_pids[dst], w.d_counter,
                                    r->n, w.stream);
       })))
    return rc;
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 8, cudaMemcpyDeviceToHost, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  cur_ws().stats.order_ms += ms;
  cur_ws().stats.launches += 8;
  r->n = *w.h_counter;
  r->sorted_buf = dst;
  return ACG_OK;
}

// Host output: the n records the device wrote to w.d_rec, copied to the caller's `out` through their page-locked
// staging -- or, for count_overlapping (`fnv`), only the FNV-1a of their words.  The time from ev0, which the
// caller records before the records are written, to the end of the copy goes to d2h_ms.
int copy_out(uint64_t n, acg_match* out, uint64_t* fnv) {
  Workspace& w = cur_ws();
  if (n) CK(cudaMemcpyAsync(w.h_rec, w.d_rec, n * 24, cudaMemcpyDeviceToHost, w.stream));
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms += ms;
  if (fnv) {
    uint64_t hsh = 0xcbf29ce484222325ull;
    for (uint64_t i = 0; i < n * 3; ++i)
      for (int k = 0; k < 8; ++k) { hsh ^= (w.h_rec[i] >> (8 * k)) & 0xFF; hsh *= 0x100000001b3ull; }
    *fnv = hsh;
  } else if (n) {
    CopyPool::get().copy(reinterpret_cast<uint8_t*>(out), reinterpret_cast<const uint8_t*>(w.h_rec.p), n * 24);
  }
  return ACG_OK;
}

// The sequential engine over [span_start, span_end): the one-document form of seq_docs_kernel, which counts
// and writes the records in the same walk.
int run_seq(const acg_dfa* a, const uint8_t* d_hay, uint64_t span_start, uint64_t span_end,
            int anchored, int earliest, int single, acg_match* out, uint64_t cap, uint64_t* n_out) {
  Workspace& w = cur_ws();
  uint64_t scap = cap;
  int rc = reserve_docs(w, 2);
  if (rc) return rc;
  const uint64_t bounds[2] = {span_start, span_end};
  CK(cudaMemcpyAsync(w.d_doc_offs, bounds, sizeof(bounds), cudaMemcpyHostToDevice, w.stream));
  for (int attempt = 0; attempt < 4; ++attempt) {
    if ((rc = reserve_rec(w, scap))) return rc;
    acb::SeqDocsLaunch p{};
    p.hay = d_hay;
    p.doc_offsets = w.d_doc_offs;
    p.n_docs = 1;
    p.anchored = anchored;
    p.match_kind = a->h.match_kind;
    p.earliest = earliest;
    p.single = single;
    p.counts = w.d_counter;
    p.out = w.d_rec;
    p.cap = w.d_rec.cap / 3;
    CK(cudaEventRecord(w.ev0, w.stream));
    CK(acb::launch_seq_docs(a->dev, p, w.stream));
    CK(cudaEventRecord(w.ev1, w.stream));
    CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 8, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    cur_ws().stats.launches += 1;
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev0, w.ev1);
    cur_ws().stats.scan_ms = ms;
    const uint64_t n = *w.h_counter;
    *n_out = n;
    cur_ws().stats.raw_matches = n;
    if (n > cap) return ACG_E_OVERFLOW;  // caller retries with a bigger buffer (two-call protocol)
    if (n > w.d_rec.cap / 3) { scap = n; continue; }
    if (n) {
      CK(cudaMemcpyAsync(w.h_rec, w.d_rec, n * 24, cudaMemcpyDeviceToHost, w.stream));
      CK(cudaStreamSynchronize(w.stream));
      for (uint64_t i = 0; i < n; ++i) {
        out[i].pid = uint32_t(w.h_rec[i * 3]);
        out[i]._pad = 0;
        out[i].start = span_start + w.h_rec[i * 3 + 1];
        out[i].end = span_start + w.h_rec[i * 3 + 2];
      }
    }
    return ACG_OK;
  }
  return ACG_E_NOMEM;
}

// Stage [span_start, span_end) of a host haystack on the device; returns a
// pointer that can be indexed with ABSOLUTE haystack offsets in that range.
int stage_host_span(const acg_dfa* a, const uint8_t* hay, uint64_t span_start, uint64_t span_end,
                    const uint8_t** d_base, bool alloc_only = false) {
  Workspace& w = cur_ws();
  // keep the 16-byte phase of the host offsets so vector loads stay aligned
  const uint64_t lead = span_start & 15;
  const uint64_t bytes = span_end - span_start;
  const uint64_t need = bytes + lead + 64;
  if (need > w.d_hay.cap) {  // whole MiB, one past what is needed
    int rc = w.d_hay.reserve(((need + (1ull << 20)) >> 20) << 20);
    if (rc) return rc;
  }
  *d_base = w.d_hay + lead - span_start;  // never dereferenced outside [span_start, span_end + slack)
  if (alloc_only) return ACG_OK;
  CK(cudaEventRecord(w.ev0, w.stream));
  if (bytes)
    CK(cudaMemcpyAsync(w.d_hay + lead, hay + span_start, bytes, cudaMemcpyHostToDevice, w.stream));
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  cur_ws().stats.h2d_ms = ms;
  return ACG_OK;
}

// Where the kernels read the haystack: `base`, indexed with absolute offsets, and `readable` bytes behind it.
// A host haystack is staged in the workspace; `pipelined` only allocates the room and leaves the copy from
// `h_src` to run_prefilter, which overlaps it with the scan.
struct Placement {
  const uint8_t* base = nullptr;
  uint64_t readable = 0;
  const uint8_t* h_src = nullptr;
};

int place_input(const acg_dfa* a, const uint8_t* hay, bool on_device, uint64_t hay_len, uint64_t span_start,
                uint64_t span_end, bool pipelined, Placement* p) {
  if (on_device) {
    p->base = hay;
    p->readable = hay_len;
    return ACG_OK;
  }
  p->readable = span_end + 32;  // the staging buffer has slack behind the span
  if (pipelined) p->h_src = hay;
  return stage_host_span(a, hay, span_start, span_end, &p->base, pipelined);
}

// acg_find / acg_find_batch: where the reference attaches its packed (Teddy) prefilter -- leftmost kinds
// only -- an unanchored try_find returns what the prefilter reports, a confirmed leftmost match
// (Candidate::Match, src/automaton.rs:1304-1309), whether or not `earliest` was asked for.
int find_earliest(const acg_dfa* a, int anchored, int earliest) {
  const bool packed = !anchored && a->h.match_kind != ACG_STANDARD && a->h.prefilter_kind == ACG_PRE_PACKED;
  return earliest && !packed;
}

// The engine of a search, or ACG_E_INVALID_ARG.  The prefilter engine serves unanchored input of an
// automaton with a plan, but not `earliest` on a leftmost automaton: that reports the first match STATE
// entered (src/automaton.rs:1381-1383), which the per-start formulation does not model.  Otherwise the
// call's `other` engine runs (the walk or the sequential engine), as does an override of it.  An
// ACG_ENGINE_PREFILTER override the input cannot use is an error when `strict`, else `other` runs.
int choose_engine(const acg_dfa* a, int anchored, int earliest, int other, bool strict) {
  const bool pf_ok = a->pf.supported && !anchored && !(earliest && a->h.match_kind != ACG_STANDARD);
  const int forced = a->engine_override;
  if (forced == other) return other;
  if (forced == ACG_ENGINE_PREFILTER && !pf_ok && strict) return ACG_E_INVALID_ARG;
  return pf_ok ? ACG_ENGINE_PREFILTER : other;
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int validate_common(const acg_dfa* a, uint64_t hay_len, uint64_t s, uint64_t e, int anchored) {
  if (!a) return ACG_E_INVALID_ARG;
  if (!span_ok(hay_len, s, e)) return ACG_E_INVALID_SPAN;
  int rc = check_anchored(a->h.start_kind, anchored);
  if (rc) return rc;
  return ACG_OK;
}

struct DevOut {
  void* d_out = nullptr;
  uint64_t min_end = 0;
  uint64_t offset_add = 0;
};

// The overlapping search of [span_start, span_end): engine, placement, the walk or prefilter scan, leaving
// r->n ordered tuples; *first = the number of them that end at or before `min_end`.
int scan_overlapping(const acg_dfa* a, const uint8_t* hay, bool on_device, uint64_t hay_len, uint64_t span_start,
                     uint64_t span_end, bool strict, uint64_t min_end, TupleResult* r, uint64_t* first) {
  Workspace& w = cur_ws();
  *first = 0;
  const int engine = choose_engine(a, 0, 0, ACG_ENGINE_WALK, strict);
  if (engine < 0) return engine;
  w.stats.engine = engine;
  Placement pl;
  int rc = place_input(a, hay, on_device, hay_len, span_start, span_end, engine == ACG_ENGINE_PREFILTER, &pl);
  if (rc) return rc;
  if (engine == ACG_ENGINE_PREFILTER) rc = run_prefilter(a, pl.base, pl.readable, span_start, span_end, 0, r, pl.h_src);
  else rc = run_walk_overlapping(a, pl.base, pl.readable, span_start, span_end, r);
  if (rc || r->n == 0 || min_end <= span_start) return rc;
  const uint64_t bound_key = (min_end - span_start + 1) << acb::kTieBits;  // first key with end > min_end
  CK(acb::launch_lower_bound(tuple_list(a, w, *r).keys, r->n, bound_key, w.d_counter, w.stream));
  CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 8, cudaMemcpyDeviceToHost, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  *first = *w.h_counter;
  return ACG_OK;
}

// The records of the ordered tuples of r from index `first` on (key layout `mode`), expanded into the caller's
// device buffer (`devout`), or into the workspace and copied to the host `out` -- count_overlapping (`fnv`) only
// hashes them.  On overflow nothing is written: the caller retries with room for *n_out.
int expand_out(const acg_dfa* a, const TupleResult& r, uint64_t first, int mode, uint64_t span_start,
               const DevOut* devout, acg_match* out, uint64_t cap, uint64_t* n_out, uint64_t* fnv) {
  Workspace& w = cur_ws();
  const uint64_t n = r.n - first;
  *n_out = n;
  if (!fnv && n > cap) return ACG_E_OVERFLOW;
  if (!devout && !fnv && n && !out) return ACG_E_INVALID_ARG;
  int rc = devout ? ACG_OK : reserve_rec(w, n);
  if (rc) return rc;
  acb::ExpandLaunch e;
  e.t = tuple_list(a, w, r);
  e.first = first;
  e.mode = mode;
  e.span_start = span_start;
  e.offset_add = devout ? devout->offset_add : 0;
  e.out = devout ? static_cast<uint64_t*>(devout->d_out) : w.d_rec.p;
  CK(cudaEventRecord(w.ev0, w.stream));
  CK(acb::launch_expand(e, w.stream));
  if (!devout) {
    w.stats.launches += 1;
    return copy_out(n, out, fnv);
  }
  CK(cudaStreamSynchronize(w.stream));
  w.stats.launches += 2;
  return ACG_OK;
}

int overlapping_impl(const acg_dfa* a, const uint8_t* hay, bool hay_on_device, uint64_t hay_len,
                     uint64_t span_start, uint64_t span_end, int anchored, acg_match* out,
                     uint64_t cap, uint64_t* n_out, uint64_t* fnv, float* kernel_ms,
                     const DevOut* devout = nullptr) {
  if (!n_out) return ACG_E_INVALID_ARG;
  *n_out = 0;
  int rc = validate_common(a, hay_len, span_start, span_end, anchored);
  if (rc) return rc;
  // Automaton::try_find_overlapping_iter, src/automaton.rs:397-423
  if (a->h.match_kind != ACG_STANDARD) return ACG_E_UNSUPPORTED_OVERLAPPING;
  if (anchored) return ACG_E_INVALID_INPUT_ANCHORED;
  if ((rc = check_start(a->h, 0))) return rc;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  if (fnv) *fnv = 0xcbf29ce484222325ull;
  if (span_start > span_end) return ACG_OK;  // Input::is_done
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;
  // devout: keep the matches on the device, drop ends <= min_end (owned by the previous shard), expand
  TupleResult r;
  uint64_t first = 0;
  if ((rc = scan_overlapping(a, hay, hay_on_device, hay_len, span_start, span_end, true, devout ? devout->min_end : 0,
                             &r, &first)))
    return rc;
  if (kernel_ms) *kernel_ms = cur_ws().stats.scan_ms + cur_ws().stats.order_ms;
  return expand_out(a, r, first, 0, span_start, devout, out, cap, n_out, fnv);
}

// acg_shard_plan: the slice arithmetic shared by every rank (SURVEY.md section 8e).  Interior
// boundaries are rounded down to 64 bytes relative to the span start so device loads stay vectorisable.
void shard_plan(uint64_t span_start, uint64_t span_end, int nranks, int rank, uint64_t max_pattern_len,
                uint64_t* own_lo, uint64_t* own_hi, uint64_t* read_lo) {
  const uint64_t n = span_end - span_start;
  const uint64_t back = max_pattern_len ? max_pattern_len - 1 : 0;
  auto cut = [&](int g) -> uint64_t {
    if (g <= 0) return span_start;
    if (g >= nranks) return span_end;
    const unsigned __int128 q = (unsigned __int128)n * (unsigned)g / (unsigned)nranks;
    return span_start + (uint64_t(q) & ~63ull);
  };
  *own_lo = cut(rank);
  *own_hi = cut(rank + 1);
  *read_lo = (*own_lo - span_start > back) ? *own_lo - back : span_start;
}

// The sharded overlapping search of one rank, first half: scan the slice, keep the matches this
// rank owns, learn the global offsets, and enqueue the expand kernel that stores the records into
// rank 0's buffer (half `slot`) plus the closing barrier.  Returns without waiting for the transfer:
// the step's workspace stays leased (the expand kernel reads its tuples) until sharded_wait.
int sharded_begin(const acg_dfa* a, acg_comm* c, const uint8_t* hay, bool hay_on_device, uint64_t hay_len,
                  uint64_t hay_off, uint64_t span_start, uint64_t span_end, bool streaming, int* slot_out) {
  if (!a || !c || !slot_out) return ACG_E_INVALID_ARG;
  // checks that do not depend on the rank come first, so that all ranks fail together
  if (span_start > span_end) return ACG_E_INVALID_SPAN;
  if (a->h.match_kind != ACG_STANDARD) return ACG_E_UNSUPPORTED_OVERLAPPING;
  int rc = check_anchored(a->h.start_kind, 0);
  if (rc) return rc;
  if ((rc = check_start(a->h, 0))) return rc;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  if (a->device != c->device) return ACG_E_INVALID_ARG;
  const int slot = int(c->step_seq & 1);
  acg_comm::Step& step = c->steps[slot];
  if (step.active) return ACG_E_INVALID_ARG;  // two steps in flight at most: wait for the older one first
  uint64_t own_lo, own_hi, read_lo;
  shard_plan(span_start, span_end, c->nranks, c->rank, a->h.max_pattern_len, &own_lo, &own_hi, &read_lo);
  // an empty slice (more ranks than 64-byte blocks) still takes part in the collectives
  const bool covered = own_hi == own_lo || (read_lo >= hay_off && own_hi <= hay_off + hay_len);
  TupleResult r;
  uint64_t first = 0;
  uint64_t lspan_s = 0;
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;  // (a rank that cannot even get a stream cannot join the exchange either)
  if (covered && own_hi > own_lo) {
    // the local scan, in local offsets: span [read_lo, own_hi) - hay_off
    // an unusable prefilter override falls back to the walk; ends <= own_lo belong to the previous rank
    lspan_s = read_lo - hay_off;
    rc = scan_overlapping(a, hay, hay_on_device, hay_len, lspan_s, own_hi - hay_off, false, own_lo - hay_off, &r,
                          &first);
  }
  if (!covered) rc = ACG_E_INVALID_SPAN;
  // a failed rank still joins the exchange (with the error flag in the top bit) so that nobody hangs
  const uint64_t mine = rc ? 0 : r.n - first;
  cudaEventRecord(step.begun, c->stream);
  uint64_t total = 0, my_off = 0;
  int rc2 = acb::comm_exchange_counts(c, mine | (rc ? (1ull << 63) : 0), &total, &my_off);
  if (rc2) return rc ? rc : rc2;
  bool any_failed = false;
  total = 0; my_off = 0;
  for (int g = 0; g < c->nranks; ++g) {
    if (c->counts[size_t(g)] >> 63) any_failed = true;
    c->counts[size_t(g)] &= ~(1ull << 63);
    if (g < c->rank) my_off += c->counts[size_t(g)];
    total += c->counts[size_t(g)];
  }
  if (any_failed) return rc ? rc : ACG_E_CUDA;  // some other rank failed: nothing was gathered
  if ((rc = acb::comm_ensure_recv(c, total))) return rc;  // every rank takes the same branch (same totals)
  uint8_t* target = nullptr;
  if ((rc = acb::comm_record_target(c, slot, my_off, mine, streaming, &target))) return rc;
  if (mine) {
    Workspace& w = cur_ws();
    acb::ExpandLaunch e;
    e.t = tuple_list(a, w, r);
    e.first = first;
    e.mode = 0;
    e.span_start = lspan_s;
    e.offset_add = hay_off;
    e.out = reinterpret_cast<uint64_t*>(target);
    // blocking step: the kernel stores the records straight into rank 0's buffer.  Stream of steps
    // (begin / wait): it expands into local memory -- short, HBM-bound -- and a copy engine ships the
    // records, so that the next step's scan, which starts right behind, finds every SM free.
    CK(acb::launch_expand(e, c->stream));
  }
  bool flagged = false;
  if ((rc = acb::comm_enqueue_close(c, slot, my_off, mine, streaming, c->step_seq + 1, &flagged))) return rc;
  cudaEventRecord(step.done, c->stream);
  step.seq = c->step_seq + 1;
  step.flagged = flagged;
  cur_ws().stats.launches += 3;
  step.mine = mine;
  step.total = total;
  step.scan_ms = cur_ws().stats.scan_ms;
  step.order_ms = cur_ws().stats.order_ms;
  step.candidates = cur_ws().stats.candidates;
  step.launches = cur_ws().stats.launches;
  step.dfa = a;
  step.lease = lease.detach();
  step.active = true;
  ++c->step_seq;
  *slot_out = slot;
  return ACG_OK;
}

// Second half: wait until every rank's records of step `slot` are in rank 0's buffer.
int sharded_wait(acg_comm* c, int slot, const acg_match** d_matches, uint64_t* n_total, acg_match* h_out,
                 uint64_t h_cap, acg_shard_stats* st) {
  if (!c || slot < 0 || slot > 1 || !n_total) return ACG_E_INVALID_ARG;
  acg_comm::Step& step = c->steps[slot];
  if (!step.active) return ACG_E_INVALID_ARG;
  DeviceGuard guard(c->device);
  const cudaError_t e = cudaEventSynchronize(step.done);
  release_workspace(static_cast<const acg_dfa*>(step.dfa), static_cast<Workspace*>(step.lease));
  step.lease = nullptr;
  step.active = false;
  if (e != cudaSuccess) { cudaGetLastError(); return ACG_E_CUDA; }
  // begin / wait form: the other ranks' records are in once their flag words say so
  if (step.flagged) {
    const int frc = acb::comm_wait_flags(c, step.seq);
    if (frc) return frc;
  }
  float gms = 0;
  cudaEventElapsedTime(&gms, step.begun, step.done);
  c->last_gather_ms = gms;
  *n_total = step.total;
  if (d_matches) *d_matches = nullptr;
  if (st) {
    st->local_matches = step.mine;
    st->total_matches = step.total;
    st->candidates = step.candidates;
    st->scan_ms = step.scan_ms;
    st->order_ms = step.order_ms;
    st->gather_ms = gms;
    st->transport = c->transport;
    st->launches = step.launches;
  }
  if (c->rank == 0) {
    c->last_result = acb::comm_half(c, slot);
    c->last_total = step.total;
    if (d_matches) *d_matches = reinterpret_cast<const acg_match*>(c->last_result);
    if (h_out) {
      if (step.total > h_cap) return ACG_E_OVERFLOW;
      if (step.total) CK(cudaMemcpy(h_out, c->last_result, size_t(step.total) * sizeof(acg_match), cudaMemcpyDeviceToHost));
    }
  }
  return ACG_OK;
}

int find_iter_impl(const acg_dfa* a, const uint8_t* hay, bool hay_on_device, uint64_t hay_len,
                   uint64_t span_start, uint64_t span_end, int anchored, acg_match* out,
                   uint64_t cap, uint64_t* n_out, float* kernel_ms) {
  if (!n_out) return ACG_E_INVALID_ARG;
  *n_out = 0;
  int rc = validate_common(a, hay_len, span_start, span_end, anchored);
  if (rc) return rc;
  if ((rc = check_start(a->h, anchored))) return rc;  // FindIter::new, src/automaton.rs:861-870
  if (!a->on_device) return ACG_E_NO_DEVICE;
  if (span_start > span_end) return ACG_OK;
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;
  const int engine = choose_engine(a, anchored, 0, ACG_ENGINE_SEQUENTIAL, true);
  if (engine < 0) return engine;
  cur_ws().stats.engine = engine;
  Placement pl;
  if ((rc = place_input(a, hay, hay_on_device, hay_len, span_start, span_end, engine == ACG_ENGINE_PREFILTER, &pl)))
    return rc;
  if (engine == ACG_ENGINE_SEQUENTIAL) {
    rc = run_seq(a, pl.base, span_start, span_end, anchored, 0, 0, out, cap, n_out);
    if (kernel_ms) *kernel_ms = cur_ws().stats.scan_ms;
    return rc;
  }
  // Standard: all occurrences in (end, len desc, list) order, then the iterator's greedy choice;
  // leftmost kinds: best match per start offset ordered by start, then the same greedy choice.
  const int mode = a->h.match_kind == ACG_STANDARD ? 0 : 1;
  TupleResult r;
  if ((rc = run_prefilter(a, pl.base, pl.readable, span_start, span_end, mode == 0 ? 2 : 1, &r, pl.h_src))) return rc;
  if ((rc = run_chain(a, mode, &r))) return rc;
  if (kernel_ms) *kernel_ms = cur_ws().stats.scan_ms + cur_ws().stats.order_ms;
  return expand_out(a, r, 0, mode, span_start, nullptr, out, cap, n_out, nullptr);
}

// acg_find (include/acb200.h)
int find_impl(const acg_dfa* a, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
              uint64_t span_end, int anchored, int earliest, acg_match* out, int* found) {
  if (!out || !found) return ACG_E_INVALID_ARG;
  *found = 0;
  int rc = validate_common(a, hay_len, span_start, span_end, anchored);
  if (rc) return rc;
  if ((rc = check_start(a->h, anchored))) return rc;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  if (span_start > span_end) return ACG_OK;
  earliest = find_earliest(a, anchored, earliest);
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;
  Workspace& w = cur_ws();
  const int engine = choose_engine(a, anchored, earliest, ACG_ENGINE_SEQUENTIAL, false);
  w.stats.engine = engine;
  // the prefilter engine's window-by-window copy below only takes the room
  Placement pl;
  if ((rc = place_input(a, hay, false, hay_len, span_start, span_end, engine == ACG_ENGINE_PREFILTER, &pl))) return rc;
  if (engine == ACG_ENGINE_SEQUENTIAL) {
    uint64_t n = 0;
    rc = run_seq(a, pl.base, span_start, span_end, anchored, earliest, 1, out, 1, &n);
    if (rc == ACG_OK && n) *found = 1;
    return rc;
  }
  // The reference's try_find is lazy (it stops reading at the first match, SURVEY.md section
  // 7h); the eager device scan therefore works through geometrically growing windows of start
  // offsets (1 MiB, 16 MiB, 256 MiB, ...), copying only what a window needs.
  const int mode = a->h.match_kind == ACG_STANDARD ? 0 : 1;
  const uint64_t look = a->h.max_pattern_len + 64;
  uint64_t copied_hi = span_start;
  // Scan the start offsets [lo, hi) and fetch the first tuple (*n: the number of tuples).
  auto first_in = [&](uint64_t lo, uint64_t hi, uint64_t* key, uint32_t* pid, uint64_t* n) -> int {
    const uint64_t upto = std::min(hi + look, span_end);
    if (upto > copied_hi) {
      CK(cudaMemcpyAsync(const_cast<uint8_t*>(pl.base) + copied_hi, hay + copied_hi, upto - copied_hi,
                         cudaMemcpyHostToDevice, w.stream));
      copied_hi = upto;
    }
    TupleResult r;
    int rc = run_prefilter(a, pl.base, copied_hi == span_end ? span_end + 32 : copied_hi, span_start, span_end,
                           mode == 0 ? 2 : 1, &r, nullptr, lo, hi);
    *n = r.n;
    if (rc || r.n == 0) return rc;
    const acb::TupleList t = tuple_list(a, w, r);
    CK(cudaMemcpyAsync(w.h_counter, t.keys, 8, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaMemcpyAsync(w.h_counter + 1, t.pids, 4, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    *key = w.h_counter[0];
    *pid = uint32_t(w.h_counter[1]);
    return ACG_OK;
  };
  const uint32_t* plens = a->h.pattern_lens.data();
  uint64_t lo = span_start, win = 1ull << 20;
  while (lo < span_end) {
    const uint64_t hi = std::min(span_end, lo + win);
    uint64_t key = 0, n = 0;
    uint32_t pid = 0;
    if ((rc = first_in(lo, hi, &key, &pid, &n))) return rc;
    if (n) {
      const uint64_t end = acb::decode_key(key, pid, mode, span_start, plens).end;
      if (mode == 0 && end > hi && hi < span_end) {
        // Standard: a match that starts in [hi, end) could still end earlier -- scan those starts
        uint64_t key2 = 0, n2 = 0;
        uint32_t pid2 = 0;
        if ((rc = first_in(hi, std::min(span_end, end), &key2, &pid2, &n2))) return rc;
        if (n2 && key2 < key) { key = key2; pid = pid2; }
      }
      const acb::MatchSpan m = acb::decode_key(key, pid, mode, span_start, plens);
      out->pid = pid;
      out->_pad = 0;
      out->start = m.start;
      out->end = m.end;
      *found = 1;
      return ACG_OK;
    }
    lo = hi;
    win = std::min<uint64_t>(win * 16, 1ull << 30);
  }
  return ACG_OK;
}

enum BatchKind { kBatchFindIter = 0, kBatchOverlapping = 1, kBatchIsMatch = 2, kBatchFind = 3 };

// acg_*_batch_devout: the results stay in device memory -- `out` / `flags` are device pointers, and find_iter /
// overlapping also fill the records' CSR index by document -- and the offsets may be there too.
struct BatchDevOut {
  bool offsets_on_device = false;
  uint64_t* match_offsets = nullptr;  // find_iter / overlapping: [n_docs + 1]
};

// acg_pattern_counts_batch(_devout): instead of the records of a find_iter / overlapping batch, how often each
// pattern occurs in each document, as a CSR matrix (host or device arrays, as the call's other outputs).
struct BatchCounts {
  uint64_t* row_offsets;  // [n_docs + 1]
  uint32_t* pids;         // [cap]
  uint64_t* counts;       // [cap]
};

// The n matches of a batch -- the tuples `t` of the prefilter engine, or (t.keys == nullptr) the records the
// sequential engine left at w.d_rec -- counted by (document, pattern) into `co` (CountKeysLaunch and
// CountRunsLaunch, acb_device.cuh).  Host output goes through w.d_rec: [row_offsets | counts | pids] there, one
// copy to page-locked staging, then to the caller's arrays.  *nnz > cap: ACG_E_OVERFLOW, nothing written.
int count_matches(const acg_dfa* a, const acb::TupleList& t, int sorted_buf, int mode, uint64_t span_start,
                  const uint64_t* d_offs, uint64_t n_docs, const BatchCounts& co, bool dev_out, uint64_t cap,
                  uint64_t* nnz) {
  Workspace& w = cur_ws();
  const uint64_t n = t.n, nd1 = n_docs + 1;
  const uint32_t pid_bits = uint32_t(acb::bit_width(std::max<uint64_t>(a->h.pattern_lens.size(), 1) - 1));
  int rc;
  float ms = 0;
  // the time between ev2 and ev3, to order_ms
  auto lap = [&]() -> int {
    CK(cudaEventRecord(w.ev3, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    cudaEventElapsedTime(&ms, w.ev2, w.ev3);
    w.stats.order_ms += ms;
    return ACG_OK;
  };
  acb::CountRunsLaunch c{};
  if (n) {
    // tuples in buffer b: keys into the other one, sorted back into b; records: keys into 0, sorted into 1
    const int b = t.keys ? sorted_buf : 1;
    if (!t.keys && (rc = reserve_tuples(w, std::max<uint64_t>(n, w.tuple_cap())))) return rc;
    if ((rc = reserve_all(std::max<uint64_t>(n, 1 << 16), w.d_scratch, w.d_flags))) return rc;
    CK(cudaEventRecord(w.ev2, w.stream));
    acb::CountKeysLaunch k;
    k.t = t;
    k.rec = t.keys ? nullptr : w.d_rec.p;
    k.mode = mode;
    k.span_start = span_start;
    k.doc_offsets = d_offs;
    k.n_docs = n_docs;
    k.pid_bits = pid_bits;
    k.keys_out = w.d_keys[1 - b];
    k.pids_out = w.d_pids[1 - b];
    CK(acb::launch_count_keys(k, w.stream));
    const int end_bit = std::max(1, int(pid_bits) + acb::bit_width(n_docs - 1));
    if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
           return acb::sort_pairs(tmp, tb, w.d_keys[1 - b], w.d_keys[b], w.d_pids[1 - b], w.d_pids[b], n, end_bit,
                                  w.stream);
         })))
      return rc;
    c.keys = w.d_keys[b];
    c.key_pids = w.d_pids[b];
    c.n = n;
    c.heads = reinterpret_cast<unsigned long long*>(w.d_keys[1 - b].p);  // the unsorted keys are spent
    c.run_index = reinterpret_cast<unsigned long long*>(w.d_scratch.p);
    c.pid_bits = pid_bits;
    c.n_docs = n_docs;
    CK(acb::launch_run_heads(c, w.stream));
    if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
           return acb::inclusive_sum_u64(tmp, tb, c.heads, c.run_index, n, w.stream);
         })))
      return rc;
    CK(cudaMemcpyAsync(w.h_counter, c.run_index + n - 1, 8, cudaMemcpyDeviceToHost, w.stream));
    if ((rc = lap())) return rc;
    w.stats.launches += 11;  // keys, radix passes (upper bound), heads, scan
    c.nnz = *w.h_counter;
  }
  *nnz = c.nnz;
  if (c.nnz > cap) return ACG_E_OVERFLOW;
  if (dev_out) {
    c.row_offsets = co.row_offsets;
    c.counts = co.counts;
    c.pids = co.pids;
  } else {
    if ((rc = reserve_rec(w, std::max(nd1, c.nnz)))) return rc;  // 3 words each: room for 1 + 1 + 1/2 of them
    c.row_offsets = w.d_rec;
    c.counts = w.d_rec + nd1;
    c.pids = reinterpret_cast<uint32_t*>(w.d_rec + nd1 + c.nnz);
  }
  CK(cudaEventRecord(w.ev2, w.stream));
  if (n) {
    CK(acb::launch_count_runs(c, w.stream));
    CK(acb::launch_count_rows(c, w.stream));
    w.stats.launches += 2;
  } else {
    CK(cudaMemsetAsync(c.row_offsets, 0, nd1 * 8, w.stream));
  }
  if ((rc = lap())) return rc;
  if (dev_out) return ACG_OK;
  const uint64_t bytes = nd1 * 8 + c.nnz * 12;
  CK(cudaEventRecord(w.ev0, w.stream));
  CK(cudaMemcpyAsync(w.h_rec, w.d_rec, bytes, cudaMemcpyDeviceToHost, w.stream));
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms += ms;
  const uint8_t* h = reinterpret_cast<const uint8_t*>(w.h_rec.p);
  CopyPool::get().copy(reinterpret_cast<uint8_t*>(co.row_offsets), h, nd1 * 8);
  if (c.nnz) {
    CopyPool::get().copy(reinterpret_cast<uint8_t*>(co.counts), h + nd1 * 8, c.nnz * 8);
    CopyPool::get().copy(reinterpret_cast<uint8_t*>(co.pids), h + (nd1 + c.nnz) * 8, c.nnz * 4);
  }
  return ACG_OK;
}

// acg_match_coverage_batch(_devout): instead of the records of a find_iter / overlapping batch, the bytes of each
// document they cover (host or device arrays, as the call's other outputs).
struct BatchCoverage {
  uint64_t* covered;  // [n_docs]
  uint8_t* mask;      // indexed like the haystack, or nullptr
};

// n bytes from the device at `src` to the host at `dst`: in one copy when `dst` is page-locked, else chunk by chunk
// through the workspace's staging ring (two page-locked buffers of one pipeline chunk), each chunk's copy to the
// caller overlapping the next one's transfer.
int copy_to_host(const acg_dfa* a, uint8_t* dst, const uint8_t* src, uint64_t n) {
  Workspace& w = cur_ws();
  if (!is_pageable_host(dst)) {
    CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    return ACG_OK;
  }
  const uint64_t chunk = std::min<uint64_t>(a->pipeline_chunk, n);
  int rc = reserve_stage(w, chunk);
  if (rc) return rc;
  uint64_t at[2] = {0, 0}, len[2] = {0, 0};
  auto drain = [&](int i) -> int {
    if (!len[i]) return ACG_OK;
    CK(cudaEventSynchronize(w.stage_ev[i]));
    CopyPool::get().copy(dst + at[i], w.h_stage[i], size_t(len[i]));
    len[i] = 0;
    return ACG_OK;
  };
  int i = 0;
  for (uint64_t c0 = 0; c0 < n; c0 += chunk, i ^= 1) {
    if ((rc = drain(i))) return rc;
    at[i] = c0;
    len[i] = std::min(chunk, n - c0);
    CK(cudaMemcpyAsync(w.h_stage[i], src + c0, len[i], cudaMemcpyDeviceToHost, w.stream));
    CK(cudaEventRecord(w.stage_ev[i], w.stream));
  }
  if ((rc = drain(i))) return rc;  // the older chunk first
  return drain(i ^ 1);
}

// The n matches of a batch -- the tuples `t` of the prefilter engine, or (t.keys == nullptr) the records the
// sequential engine left at w.d_rec -- turned into the bytes of each document they cover, and the mask (CoverLaunch,
// acb_device.cuh).  `ordered`: the matches are in start order already (find_iter), so there is no sort.  Scratch:
// (start, length) pairs in the tuple buffers, ends in w.d_scratch.  Host output: the counts in w.d_doc_counts and
// the mask in the haystack staging buffer (the haystack is spent by now), copied to the caller from there.
int cover_matches(const acg_dfa* a, const acb::TupleList& t, int sorted_buf, int mode, bool ordered,
                  uint64_t span_start, uint64_t span_end, const uint64_t* d_offs, uint64_t n_docs,
                  const BatchCoverage& cv, bool dev_out) {
  Workspace& w = cur_ws();
  const uint64_t n = t.n;
  int rc;
  acb::CoverLaunch c{};
  c.t = t;
  c.rec = t.keys ? nullptr : w.d_rec.p;
  c.mode = mode;
  c.span_start = span_start;
  c.doc_offsets = d_offs;
  c.n_docs = n_docs;
  c.covered = dev_out ? reinterpret_cast<unsigned long long*>(cv.covered) : w.d_doc_counts.p;
  c.mask = cv.mask;
  if (cv.mask && !dev_out) {
    const uint8_t* base = nullptr;
    if ((rc = stage_host_span(a, nullptr, span_start, span_end, &base, true))) return rc;
    c.mask = const_cast<uint8_t*>(base);
  }
  // tuples in buffer b: (start, length) into the other one, sorted back into b; records: into 0, sorted into 1
  const int b = t.keys ? sorted_buf : 1;
  if (n) {
    if (!t.keys && (rc = reserve_tuples(w, std::max<uint64_t>(n, w.tuple_cap())))) return rc;
    if ((rc = reserve_all(std::max<uint64_t>(n, 1 << 16), w.d_scratch, w.d_flags))) return rc;
  }
  CK(cudaEventRecord(w.ev2, w.stream));
  CK(cudaMemsetAsync(c.covered, 0, n_docs * 8, w.stream));
  if (c.mask) CK(cudaMemsetAsync(c.mask + span_start, 0, span_end - span_start, w.stream));
  if (n) {
    c.starts = w.d_keys[1 - b];
    c.lens = w.d_pids[1 - b];
    c.max_end = w.d_scratch;
    CK(acb::launch_cover_keys(c, w.stream));
    w.stats.launches += 1;
    if (!ordered) {
      const int end_bit = std::max(1, acb::bit_width(span_end - span_start));
      if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
             return acb::sort_pairs(tmp, tb, w.d_keys[1 - b], w.d_keys[b], w.d_pids[1 - b], w.d_pids[b], n, end_bit,
                                    w.stream);
           })))
        return rc;
      c.starts = w.d_keys[b];
      c.lens = w.d_pids[b];
      w.stats.launches += 8;  // radix passes (upper bound)
    }
    CK(acb::launch_cover_ends(c, w.stream));
    if ((rc = cub_call(w, [&](void* tmp, size_t& tb) { return acb::scan_max_u64(tmp, tb, c.max_end, n, w.stream); })))
      return rc;
    CK(acb::launch_cover_runs(c, w.stream));
    w.stats.launches += 3;  // ends, scan, runs
    if (c.mask) {
      CK(acb::launch_cover_mask(c, w.stream));
      w.stats.launches += 1;
    }
  }
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  w.stats.order_ms += ms;
  if (dev_out) return ACG_OK;
  if ((rc = reserve_rec(w, (n_docs + 2) / 3))) return rc;  // 3 words per record: room for n_docs words
  CK(cudaEventRecord(w.ev0, w.stream));
  CK(cudaMemcpyAsync(w.h_rec, c.covered, n_docs * 8, cudaMemcpyDeviceToHost, w.stream));
  if (cv.mask && (rc = copy_to_host(a, cv.mask + span_start, c.mask + span_start, span_end - span_start))) return rc;
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms += ms;
  CopyPool::get().copy(reinterpret_cast<uint8_t*>(cv.covered), reinterpret_cast<const uint8_t*>(w.h_rec.p),
                       n_docs * 8);
  return ACG_OK;
}

// acg_replace_all_batch(_devout): instead of the records of a find_iter batch, the documents with every match
// replaced (the output arrays in host or device memory, as the call's other outputs; the table in host memory).
struct BatchReplace {
  const uint8_t* rep_bytes;
  const uint64_t* rep_offsets;  // [n_reps + 1]
  uint64_t n_reps;
  uint8_t* out;                 // [cap]
  uint64_t* out_offsets;        // [n_docs + 1]
};

// One replacement per pattern, with offsets that do not decrease and bytes behind them (the reference asserts the
// count, src/automaton.rs:443-448).
bool replacements_ok(const acg_dfa* a, const BatchReplace& rp) {
  if (!rp.rep_offsets || rp.n_reps != a->h.pattern_lens.size()) return false;
  for (uint64_t i = 0; i < rp.n_reps; ++i)
    if (rp.rep_offsets[i + 1] < rp.rep_offsets[i]) return false;
  return rp.rep_bytes || rp.rep_offsets[rp.n_reps] == rp.rep_offsets[0];
}

// A batch's replacement table into w.d_rep: the offsets, then the bytes (replace_matches takes them from there).
int upload_replacements(Workspace& w, const BatchReplace& rp) {
  const uint64_t n_reps = rp.n_reps, rep_total = rp.rep_offsets[n_reps] - rp.rep_offsets[0];
  int rc = w.d_rep.reserve(n_reps + 1 + (rep_total + 7) / 8);
  if (rc) return rc;
  CK(cudaMemcpyAsync(w.d_rep, rp.rep_offsets, (n_reps + 1) * 8, cudaMemcpyHostToDevice, w.stream));
  if (rep_total)
    CK(cudaMemcpyAsync(w.d_rep + n_reps + 1, rp.rep_bytes + rp.rep_offsets[0], rep_total, cudaMemcpyHostToDevice,
                       w.stream));
  return ACG_OK;
}

// The n find_iter matches of a batch -- the tuples `t` of the prefilter engine, in start order after the chain, or
// (t.keys == nullptr) the acg_doc_match records at `rec` -- spliced with their replacements into the output
// (ReplaceLaunch, acb_device.cuh).  `d_in`: the input at span_start, still being read.  The table is on the device:
// `rep_offsets` as the caller gave them, `rep_bytes` the bytes behind them.  Scratch: a_i and e_i in the tuple
// buffers' keys, pids and documents in their pids, the deltas and their sum in w.d_scratch, the tile index in
// w.d_temp.  Host output: the bytes in w.d_out and out_offsets in w.d_doc_incl (free once the search has run, and
// not w.d_rec, which still holds a stream feed's records for its state step), copied to the caller from there.
// *out_len > cap: ACG_E_OVERFLOW, nothing written.
int replace_matches(const acg_dfa* a, const acb::TupleList& t, const uint64_t* rec, int sorted_buf, int mode,
                    uint64_t span_start, uint64_t span_end, const uint8_t* d_in, const uint64_t* d_offs,
                    uint64_t n_docs, const uint64_t* rep_offsets, const uint8_t* rep_bytes, const BatchReplace& rp,
                    bool dev_out, uint64_t cap, uint64_t* out_len) {
  Workspace& w = cur_ws();
  const uint64_t n = t.n, nd1 = n_docs + 1;
  int rc;
  float ms = 0;
  // the time between ev2 and ev3, to order_ms
  auto lap = [&]() -> int {
    CK(cudaEventRecord(w.ev3, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    cudaEventElapsedTime(&ms, w.ev2, w.ev3);
    w.stats.order_ms += ms;
    return ACG_OK;
  };
  acb::ReplaceLaunch r{};
  r.t = t;
  r.rec = t.keys ? nullptr : rec;
  r.mode = mode;
  r.span_start = span_start;
  r.doc_offsets = d_offs;
  r.n_docs = n_docs;
  r.rep_offsets = rep_offsets;
  r.rep_bytes = rep_bytes;
  r.in = d_in;
  uint64_t total = span_end - span_start;
  CK(cudaEventRecord(w.ev2, w.stream));
  if (n) {
    // tuples in buffer b: a_i and pids into the other one, e_i and documents over the tuples; records: 0 and 1
    const int b = t.keys ? sorted_buf : 1;
    if (!t.keys && (rc = reserve_tuples(w, std::max<uint64_t>(n, w.tuple_cap())))) return rc;
    if ((rc = reserve_all(std::max<uint64_t>(n, 1 << 16), w.d_scratch, w.d_flags))) return rc;
    r.a = w.d_keys[1 - b];
    r.pids = w.d_pids[1 - b];
    r.e = w.d_keys[b];
    r.docs = w.d_pids[b];
    r.incl = reinterpret_cast<unsigned long long*>(w.d_scratch.p);
    CK(acb::launch_replace_keys(r, w.stream));
    if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
           return acb::inclusive_sum_u64(tmp, tb, r.incl, r.incl, n, w.stream);
         })))
      return rc;
    CK(cudaMemcpyAsync(w.h_counter, r.incl + n - 1, 8, cudaMemcpyDeviceToHost, w.stream));
    if ((rc = lap())) return rc;
    w.stats.launches += 2;
    total += w.h_counter[0];  // the sum of the length changes, mod 2^64: the output is never shorter than 0
  }
  *out_len = total;
  if (total > cap) return ACG_E_OVERFLOW;
  r.out_len = total;
  if (dev_out) {
    r.out = rp.out;
    r.out_offsets = rp.out_offsets;
  } else {
    if ((rc = w.d_out.reserve(std::max<uint64_t>(total, 1 << 20)))) return rc;
    if ((rc = w.h_rec.reserve(nd1))) return rc;
    r.out = w.d_out;
    r.out_offsets = reinterpret_cast<uint64_t*>(w.d_doc_incl.p);  // nd1 entries (reserve_docs)
  }
  const uint64_t n_tiles = total ? acb::replace_splice_tiles(r.out, total) : 0;
  if ((rc = w.d_temp.reserve(std::max<uint64_t>((n_tiles + 1) * 8, 16)))) return rc;
  r.tile_first = reinterpret_cast<int64_t*>(w.d_temp.p);
  CK(cudaEventRecord(w.ev2, w.stream));
  CK(acb::launch_replace_rows(r, w.stream));
  w.stats.launches += 1;
  if (total) {
    CK(acb::launch_replace_splice(r, w.stream));
    w.stats.launches += 2;
  }
  if ((rc = lap())) return rc;
  if (dev_out) return ACG_OK;
  CK(cudaEventRecord(w.ev0, w.stream));
  CK(cudaMemcpyAsync(w.h_rec, r.out_offsets, nd1 * 8, cudaMemcpyDeviceToHost, w.stream));
  if (total && (rc = copy_to_host(a, rp.out, r.out, total))) return rc;
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms += ms;
  CopyPool::get().copy(reinterpret_cast<uint8_t*>(rp.out_offsets), reinterpret_cast<const uint8_t*>(w.h_rec.p),
                       nd1 * 8);
  return ACG_OK;
}

// acg_streams_feed(_devout): the batch is the feed's combined documents D in the workspace (offsets on the device,
// `docs_len` bytes), and its records become the feed's (StreamLaunch, acb_device.cuh).  `out` and `out_index` are
// the caller's device arrays, or (!dev_out) `out` is the caller's host array.  acg_streams_replace_feed(_devout)
// (`replace`, the set): `out` is the output bytes and `out_index` their offsets, both host arrays unless dev_out.
struct BatchStreams {
  acb::StreamLaunch launch;  // the set, the chunks and D; the records and outputs are filled in by stream_records
  uint64_t docs_len;
  void* out;
  uint64_t* out_index;
  bool dev_out;
  const acg_streams* replace;
};

// A replace set's feed, once D is searched: the records of D and the hold records (launch_stream_hold), spliced
// with the set's table into the feed's output, then the state of every stream.  *out_len > cap: ACG_E_OVERFLOW,
// and nothing -- state included -- is written.
int stream_replace(const acg_dfa* a, const BatchStreams& st, acb::StreamLaunch& p, uint64_t cap, uint64_t* out_len) {
  Workspace& w = cur_ws();
  const uint64_t n_rec = p.m + p.n;
  int rc = w.d_held.reserve(std::max<uint64_t>(n_rec, 1 << 16) * 3);
  if (rc) return rc;
  p.held = w.d_held;
  p.hold_pid = static_cast<uint32_t>(a->h.pattern_lens.size());
  CK(acb::launch_stream_hold(p, w.stream));
  w.stats.launches += 1;
  const uint64_t* rep_offsets = st.replace->d_rep;
  const uint8_t* rep_bytes = reinterpret_cast<const uint8_t*>(rep_offsets + p.hold_pid + 2);
  const BatchReplace rp{nullptr, nullptr, p.hold_pid, static_cast<uint8_t*>(st.out), st.out_index};
  if ((rc = replace_matches(a, acb::TupleList{nullptr, nullptr, nullptr, n_rec}, p.held, 0, 0, 0, p.docs_len, p.docs,
                            reinterpret_cast<const uint64_t*>(p.doc_offsets), p.n, rep_offsets, rep_bytes, rp,
                            st.dev_out, cap, out_len)))
    return rc;
  float ms = 0;
  CK(cudaEventRecord(w.ev2, w.stream));
  CK(acb::launch_stream_state(p, w.stream));
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  w.stats.order_ms += ms;
  w.stats.launches += 1;
  return ACG_OK;
}

// The m records of D at `rec` with their index: the ones a previous feed has not returned (overlapping: those that
// end after their tail), rebased and tagged, then the state of every stream.  ms_to gets the batch's time from ev2
// to ev3.  *n_out > cap: ACG_E_OVERFLOW, and nothing -- state included -- is written.
int stream_records(const acg_dfa* a, const BatchStreams& st, const uint64_t* rec, const uint64_t* rec_index,
                   uint64_t m, uint64_t cap, uint64_t* n_out, float& ms_to) {
  Workspace& w = cur_ws();
  float ms = 0;
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  ms_to += ms;
  acb::StreamLaunch p = st.launch;
  p.rec = rec;
  p.rec_index = rec_index;
  p.m = m;
  p.keep = nullptr;
  if (st.replace) return stream_replace(a, st, p, cap, n_out);
  uint64_t kept = m;
  int rc;
  CK(cudaEventRecord(w.ev2, w.stream));
  if (p.overlapping && m) {
    if ((rc = reserve_all(std::max<uint64_t>(m, 1 << 16), w.d_scratch, w.d_flags))) return rc;
    p.keep = reinterpret_cast<unsigned long long*>(w.d_scratch.p);
    CK(acb::launch_stream_keep(p, w.stream));
    if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
           return acb::inclusive_sum_u64(tmp, tb, p.keep, p.keep, m, w.stream);
         })))
      return rc;
    CK(cudaMemcpyAsync(w.h_counter, p.keep + m - 1, 8, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    w.stats.launches += 2;
    kept = w.h_counter[0];
  }
  *n_out = kept;
  if (kept > cap) return ACG_E_OVERFLOW;
  if (kept && !st.out) return ACG_E_INVALID_ARG;
  const bool dev_out = st.dev_out;
  if (!dev_out && (rc = w.d_out.reserve(std::max<uint64_t>(kept * 24, 1 << 20)))) return rc;
  p.out = dev_out ? static_cast<uint64_t*>(st.out) : reinterpret_cast<uint64_t*>(w.d_out.p);
  p.out_index = st.out_index;
  CK(acb::launch_stream_records(p, w.stream));
  CK(acb::launch_stream_state(p, w.stream));
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  w.stats.order_ms += ms;
  w.stats.launches += 2;
  if (dev_out || !kept) return ACG_OK;
  CK(cudaEventRecord(w.ev0, w.stream));
  if ((rc = copy_to_host(a, reinterpret_cast<uint8_t*>(st.out), w.d_out, kept * 24))) return rc;
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms += ms;
  return ACG_OK;
}

// acg_find_iter_batch / acg_find_overlapping_batch / acg_is_match_batch / acg_find_batch (include/acb200.h), and
// with `co` acg_pattern_counts_batch, with `cv` acg_match_coverage_batch (what: kBatchFindIter or
// kBatchOverlapping, the records they aggregate; `cap` and `n_out` are those of the counts) or with `rp`
// acg_replace_all_batch (kBatchFindIter; `cap` and `n_out` in output bytes).  is_match and find give one result
// per document: flags[n_docs] (find: found) and, for find, out[n_docs].  With `st` a stream feed, which holds the
// workspace already, searches its combined documents (`hay`, `offs` on the device; `cap` and `n_out` those of the
// feed's records).
int batch_impl(const acg_dfa* a, int what, const uint8_t* hay, bool hay_on_device, uint64_t hay_len,
               const uint64_t* offs, uint64_t n_docs, int anchored, acg_match* out, uint64_t cap, uint64_t* n_out,
               uint8_t* flags, int earliest = 0, const BatchDevOut* dv = nullptr, const BatchCounts* co = nullptr,
               const BatchCoverage* cv = nullptr, const BatchReplace* rp = nullptr, const BatchStreams* st = nullptr) {
  const bool per_doc = what == kBatchIsMatch || what == kBatchFind;
  if (!a || !offs || (per_doc ? n_docs && (!flags || (what == kBatchFind && !out)) : !n_out))
    return ACG_E_INVALID_ARG;
  if (rp ? !rp->out_offsets || (!rp->out && cap) || !replacements_ok(a, *rp)
         : cv ? n_docs && !cv->covered
              : co ? !co->row_offsets || ((!co->pids || !co->counts) && cap)
                   : dv && !per_doc && (!dv->match_offsets || (!out && cap)))
    return ACG_E_INVALID_ARG;
  if (n_out) *n_out = 0;
  if (n_docs >= (1ull << 32)) return ACG_E_INVALID_ARG;
  const bool offs_on_device = (dv && dv->offsets_on_device) || st;
  if (offs_on_device) {
    if (reinterpret_cast<uintptr_t>(offs) & 7) return ACG_E_INVALID_ARG;
  } else {
    for (uint64_t i = 0; i < n_docs; ++i)
      if (offs[i + 1] < offs[i]) return ACG_E_INVALID_SPAN;
    if (offs[n_docs] > hay_len) return ACG_E_INVALID_SPAN;
  }
  int rc = check_anchored(a->h.start_kind, anchored);
  if (rc) return rc;
  if (what == kBatchOverlapping) {  // Automaton::try_find_overlapping_iter, src/automaton.rs:397-423
    if (a->h.match_kind != ACG_STANDARD) return ACG_E_UNSUPPORTED_OVERLAPPING;
    if (anchored) return ACG_E_INVALID_INPUT_ANCHORED;
  }
  if ((rc = check_start(a->h, anchored))) return rc;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  if (n_docs == 0 && !dv) {
    if (co) co->row_offsets[0] = 0;
    if (rp) rp->out_offsets[0] = 0;
    return ACG_OK;
  }
  earliest = find_earliest(a, anchored, earliest);
  const int engine = n_docs ? choose_engine(a, anchored, earliest, ACG_ENGINE_SEQUENTIAL, true) : ACG_ENGINE_SEQUENTIAL;
  if (engine < 0) return engine;
  const bool use_pf = engine == ACG_ENGINE_PREFILTER;
  DeviceGuard guard(a->device);
  std::optional<WsLease> lease;
  if (!st) {
    lease.emplace(a);
    if (lease->rc) return lease->rc;
  }
  Workspace& w = cur_ws();
  w.stats.engine = engine;
  const uint64_t nd1 = n_docs + 1;
  if ((rc = reserve_docs(w, nd1))) return rc;
  uint64_t span_start, span_end;
  const uint64_t* d_offs = w.d_doc_offs;
  unsigned long long* const d_counts = w.d_doc_counts;
  unsigned long long* const d_incl = w.d_doc_incl;
  // The results go to the caller's device arrays, or to the workspace's and from there to the host at the end.
  // The records (find: one per document, at index doc) get their place once their number is known; on overflow
  // nothing is written, and the caller retries with room for *n_out.  Records that are counted or covered stay
  // in the workspace.
  uint8_t* const d_flags = dv ? flags : w.d_doc_flags.p;
  uint64_t* const d_index = dv ? dv->match_offsets : reinterpret_cast<uint64_t*>(d_counts);
  uint64_t* d_rec = nullptr;
  uint64_t n_rec = 0;
  const bool aggregated = co || cv || rp;
  auto records = [&](uint64_t n) -> int {
    const bool to_caller = dv && !aggregated;
    if (!aggregated && !st && n > cap) return ACG_E_OVERFLOW;
    if (!aggregated && !st && n && !out) return ACG_E_INVALID_ARG;
    n_rec = n;
    const int e = to_caller ? ACG_OK : reserve_rec(w, n);
    d_rec = to_caller ? reinterpret_cast<uint64_t*>(out) : w.d_rec.p;
    return e;
  };
  if (what == kBatchFind && (rc = records(n_docs))) return rc;
  if (st) {  // built by the feed: bounds known to hold
    span_start = 0;
    span_end = st->docs_len;
    d_offs = offs;
  } else if (offs_on_device) {
    // checked where they are; the span bounds come back with the verdict (placement and the scan plan need them)
    CK(cudaMemsetAsync(w.d_counter, 0, 8, w.stream));
    CK(acb::launch_check_offsets(offs, n_docs, hay_len, w.d_counter, w.stream));
    CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 24, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    w.stats.launches += 1;
    if (w.h_counter[0]) return ACG_E_INVALID_SPAN;
    span_start = w.h_counter[1];
    span_end = w.h_counter[2];
    d_offs = offs;
  } else {
    span_start = offs[0];
    span_end = offs[n_docs];
    CK(cudaMemcpyAsync(w.d_doc_offs, offs, nd1 * 8, cudaMemcpyHostToDevice, w.stream));
  }
  if (n_docs == 0) {  // device output: the index of no records
    if (!per_doc && !cv)
      CK(cudaMemsetAsync(co ? co->row_offsets : rp ? rp->out_offsets : dv->match_offsets, 0, 8, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    return ACG_OK;
  }
  Placement pl;
  if ((rc = place_input(a, hay, hay_on_device, hay_len, span_start, span_end, use_pf, &pl))) return rc;
  if (rp && (rc = upload_replacements(w, *rp))) return rc;
  const uint64_t* rep_offsets = w.d_rep;
  const uint8_t* rep_bytes = rp ? reinterpret_cast<const uint8_t*>(w.d_rep + rp->n_reps + 1) : nullptr;
  // The end of a batch: the time between ev2 and ev3 to `ms_to` -- the sequential engine's scan, the order time
  // of the prefilter engine's per-document step -- and for host output the copy of the flags and the records.
  auto finish = [&](float& ms_to) -> int {
    if (dv) {
      CK(cudaStreamSynchronize(w.stream));
    } else {
      CK(cudaEventRecord(w.ev0, w.stream));
      if (per_doc) CK(cudaMemcpyAsync(flags, d_flags, n_docs, cudaMemcpyDeviceToHost, w.stream));
      if (int e = copy_out(n_rec, out, nullptr)) return e;
    }
    float ms = 0;
    cudaEventElapsedTime(&ms, w.ev2, w.ev3);
    ms_to += ms;
    return ACG_OK;
  };
  if (!use_pf) {
    // one thread per document: count, inclusive scan, fill at each document's offset
    acb::SeqDocsLaunch p{};
    p.hay = pl.base;
    p.doc_offsets = d_offs;
    p.n_docs = n_docs;
    p.anchored = anchored;
    p.match_kind = a->h.match_kind;
    p.overlapping = what == kBatchOverlapping;
    p.single = per_doc;
    p.earliest = what == kBatchIsMatch || earliest;
    CK(cudaEventRecord(w.ev2, w.stream));
    if (per_doc) {
      p.flags = d_flags;
      if (what == kBatchFind) {
        p.find = 1;
        p.out = d_rec;
        p.cap = n_docs;
      }
      CK(acb::launch_seq_docs(a->dev, p, w.stream));
      CK(cudaEventRecord(w.ev3, w.stream));
      w.stats.launches += 1;
      return finish(w.stats.scan_ms);
    }
    p.counts = d_counts;
    CK(acb::launch_seq_docs(a->dev, p, w.stream));
    if ((rc = cub_call(w, [&](void* t, size_t& tb) {
           return acb::inclusive_sum_u64(t, tb, d_counts, d_incl, n_docs, w.stream);
         })))
      return rc;
    CK(cudaMemcpyAsync(w.h_counter, d_incl + n_docs - 1, 8, cudaMemcpyDeviceToHost, w.stream));
    CK(cudaStreamSynchronize(w.stream));
    const uint64_t total = w.h_counter[0];
    if (!co) *n_out = total;
    w.stats.raw_matches = total;
    w.stats.launches += 2;
    if ((rc = records(total))) return rc;
    if (total) {
      p.incl = d_incl;
      p.out = d_rec;
      p.cap = total;
      CK(acb::launch_seq_docs(a->dev, p, w.stream));
      w.stats.launches += 1;
    }
    CK(cudaEventRecord(w.ev3, w.stream));
    if (aggregated) {
      CK(cudaStreamSynchronize(w.stream));
      cudaEventElapsedTime(&w.stats.scan_ms, w.ev2, w.ev3);
      const acb::TupleList recs{nullptr, nullptr, nullptr, total};
      if (cv)  // find_iter records are in start order; overlapping ones in end order
        return cover_matches(a, recs, 0, 0, what == kBatchFindIter, span_start, span_end, d_offs, n_docs, *cv,
                             dv != nullptr);
      if (rp)
        return replace_matches(a, recs, d_rec, 0, 0, span_start, span_end, pl.base + span_start, d_offs, n_docs,
                               rep_offsets, rep_bytes, *rp, dv != nullptr, cap, n_out);
      return count_matches(a, recs, 0, 0, span_start, d_offs, n_docs, *co, dv != nullptr, cap, n_out);
    }
    // the CSR index is the inclusive scan behind a zero
    CK(cudaMemsetAsync(d_index, 0, 8, w.stream));
    CK(cudaMemcpyAsync(d_index + 1, d_incl, n_docs * 8, cudaMemcpyDeviceToDevice, w.stream));
    if (st) return stream_records(a, *st, d_rec, d_index, n_rec, cap, n_out, w.stats.scan_ms);
    return finish(w.stats.scan_ms);
  }
  // prefilter engine over the whole span, each match bounded by its document (PrefilterLaunch::doc_offsets)
  const int chain_mode = what == kBatchOverlapping || a->h.match_kind == ACG_STANDARD ? 0 : 1;
  const int pf_mode = what == kBatchOverlapping ? 0 : (chain_mode == 0 ? 2 : 1);
  DocBatch docs;
  docs.d_offsets = d_offs;
  docs.n = n_docs;
  docs.unordered = per_doc || (aggregated && what == kBatchOverlapping);  // counts and coverage do not depend on it
  TupleResult r;
  if ((rc = run_prefilter(a, pl.base, pl.readable, span_start, span_end, pf_mode, &r, pl.h_src, UINT64_MAX,
                          UINT64_MAX, &docs)))
    return rc;
  if (per_doc) {
    // is_match: the documents of the tuples.  find: per document, the tuple with the smallest key (mode 1: the
    // best match at the smallest start; mode 2: the smallest end, longest first, then list order -- entry 0 of
    // the first match state entered), the first tuple acg_find takes from the same keys in sorted order.
    acb::DocFlagsLaunch f;
    f.t = tuple_list(a, w, r);
    f.mode = chain_mode;
    f.span_start = span_start;
    f.doc_offsets = d_offs;
    f.n_docs = n_docs;
    f.flags = d_flags;
    CK(cudaEventRecord(w.ev2, w.stream));
    if (what == kBatchFind) {
      f.best = d_counts;
      f.out = d_rec;
      CK(acb::launch_doc_first(f, w.stream));
      w.stats.launches += 3;
    } else {
      CK(cudaMemsetAsync(d_flags, 0, n_docs, w.stream));
      CK(acb::launch_doc_flags(f, w.stream));
      w.stats.launches += 1;
    }
    CK(cudaEventRecord(w.ev3, w.stream));
    return finish(w.stats.order_ms);
  }
  if (what == kBatchFindIter && (rc = run_chain(a, chain_mode, &r))) return rc;
  if (cv)  // the tuples of find_iter are in start order: the chain's matches neither overlap nor go backwards
    return cover_matches(a, tuple_list(a, w, r), r.sorted_buf, chain_mode, what == kBatchFindIter, span_start,
                         span_end, d_offs, n_docs, *cv, dv != nullptr);
  if (co)
    return count_matches(a, tuple_list(a, w, r), r.sorted_buf, chain_mode, span_start, d_offs, n_docs, *co,
                         dv != nullptr, cap, n_out);
  if (rp)  // the chain's matches in start order: the splice's segments follow each other
    return replace_matches(a, tuple_list(a, w, r), nullptr, r.sorted_buf, chain_mode, span_start, span_end,
                           pl.base + span_start, d_offs, n_docs, rep_offsets, rep_bytes, *rp, dv != nullptr, cap,
                           n_out);
  *n_out = r.n;
  if ((rc = records(r.n))) return rc;
  CK(cudaEventRecord(w.ev2, w.stream));
  if (r.n == 0) {
    CK(cudaMemsetAsync(d_index, 0, nd1 * 8, w.stream));
  } else {
    acb::DocRecordsLaunch e;
    e.t = tuple_list(a, w, r);
    e.mode = chain_mode;
    e.span_start = span_start;
    e.doc_offsets = d_offs;
    e.n_docs = n_docs;
    e.out = d_rec;
    e.match_offsets = d_index;
    CK(acb::launch_doc_records(e, w.stream));
    w.stats.launches += 1;
  }
  CK(cudaEventRecord(w.ev3, w.stream));
  if (st) return stream_records(a, *st, d_rec, d_index, r.n, cap, n_out, w.stats.order_ms);
  return finish(w.stats.order_ms);
}

// acg_streams_feed / acg_streams_feed_devout (include/acb200.h).  dev_out: `out` and `match_offsets` are device
// arrays, else `out` is a host array.  With `replace`, acg_streams_replace_feed(_devout): `out` is the output bytes
// and `match_offsets` their offsets, both host arrays unless dev_out.  The chunk offsets are checked (on the device when they are there) and D's
// length fetched in one round trip; D is gathered, searched by batch_impl and its records finished by
// stream_records.  Staging and gather time go to h2d_ms.
int streams_feed_impl(acg_streams* set, const uint8_t* hay, bool hay_on_device, uint64_t hay_len,
                      const uint64_t* chunk_offsets, bool offsets_on_device, uint64_t n_streams, void* out,
                      uint64_t cap, uint64_t* match_offsets, bool dev_out, bool replace, uint64_t* n_out) {
  if (!set || set->replace != replace || !chunk_offsets || !n_out || n_streams != set->n ||
      ((dev_out || replace) && !match_offsets) || (!out && cap))
    return ACG_E_INVALID_ARG;
  *n_out = 0;
  const uint64_t n = set->n, n1 = n + 1;
  if (offsets_on_device) {
    if (reinterpret_cast<uintptr_t>(chunk_offsets) & 7) return ACG_E_INVALID_ARG;
  } else {
    for (uint64_t i = 0; i < n; ++i)
      if (chunk_offsets[i + 1] < chunk_offsets[i]) return ACG_E_INVALID_SPAN;
    if (chunk_offsets[n] > hay_len) return ACG_E_INVALID_SPAN;
  }
  const acg_dfa* a = set->a;
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;
  Workspace& w = cur_ws();
  int rc = w.d_soffs.reserve(2 * n1);
  if (rc) return rc;
  acb::StreamLaunch p{};
  p.n = n;
  p.back = set->back;
  p.overlapping = set->overlapping;
  p.pos = set->d_state;
  p.cursor = set->d_state + n;
  p.tail = set->d_tail;
  p.doc_offsets = reinterpret_cast<unsigned long long*>(w.d_soffs.p);
  CK(cudaEventRecord(w.ev0, w.stream));
  if (offsets_on_device) {
    p.chunk_offsets = chunk_offsets;
    CK(cudaMemsetAsync(w.d_counter, 0, 8, w.stream));
    CK(acb::launch_check_offsets(chunk_offsets, n, hay_len, w.d_counter, w.stream));
    CK(cudaMemcpyAsync(w.h_counter, w.d_counter, 24, cudaMemcpyDeviceToHost, w.stream));
    w.stats.launches += 1;
  } else {
    p.chunk_offsets = w.d_soffs + n1;
    CK(cudaMemcpyAsync(w.d_soffs + n1, chunk_offsets, n1 * 8, cudaMemcpyHostToDevice, w.stream));
  }
  CK(acb::launch_stream_docs(p, w.stream));
  if ((rc = cub_call(w, [&](void* tmp, size_t& tb) {
         return acb::inclusive_sum_u64(tmp, tb, p.doc_offsets + 1, p.doc_offsets + 1, n, w.stream);
       })))
    return rc;
  CK(cudaMemcpyAsync(w.h_counter + 3, p.doc_offsets + n, 8, cudaMemcpyDeviceToHost, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  w.stats.launches += 2;
  uint64_t chunks_lo = offsets_on_device ? w.h_counter[1] : chunk_offsets[0];
  uint64_t chunks_hi = offsets_on_device ? w.h_counter[2] : chunk_offsets[n];
  if (offsets_on_device && w.h_counter[0]) return ACG_E_INVALID_SPAN;
  p.docs_len = w.h_counter[3];
  // host chunks: staged in the workspace, read from there with their absolute offsets
  Placement pl;
  if ((rc = place_input(a, hay, hay_on_device, hay_len, chunks_lo, chunks_hi, false, &pl))) return rc;
  p.chunks = pl.base;
  if ((rc = w.d_sdocs.reserve(((p.docs_len + 64 + (1ull << 20)) >> 20) << 20))) return rc;
  p.docs = w.d_sdocs;
  if (p.docs_len) {
    CK(acb::launch_stream_gather(p, w.stream));
    w.stats.launches += 1;
  }
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.h2d_ms = ms;
  BatchStreams st{p, p.docs_len, out, dev_out || replace ? match_offsets : nullptr, dev_out, replace ? set : nullptr};
  return batch_impl(a, set->overlapping ? kBatchOverlapping : kBatchFindIter, p.docs, true, p.docs_len,
                    w.d_soffs, n, 0, reinterpret_cast<acg_match*>(out), cap, n_out, nullptr, 0, nullptr, nullptr,
                    nullptr, nullptr, &st);
}

// acg_streams_create, and with `rp` (its table only) acg_streams_create_replace.
int streams_create(const acg_dfa* a, uint64_t n_streams, int overlapping, const BatchReplace* rp, acg_streams** out) {
  if (!a || !out || n_streams == 0 || n_streams >= (1ull << 32)) return ACG_E_INVALID_ARG;
  *out = nullptr;
  // StreamChunkIter::new, src/automaton.rs:1087-1103, and try_find_overlapping_iter, :397-423
  if (a->h.match_kind != ACG_STANDARD) return overlapping ? ACG_E_UNSUPPORTED_OVERLAPPING : ACG_E_UNSUPPORTED_STREAM;
  if (a->has_empty) return ACG_E_UNSUPPORTED_EMPTY;
  int rc = check_anchored(a->h.start_kind, 0);
  if (rc || (rc = check_start(a->h, 0))) return rc;
  if (rp && !replacements_ok(a, *rp)) return ACG_E_INVALID_ARG;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  acg_streams* s = new (std::nothrow) acg_streams();
  if (!s) return ACG_E_NOMEM;
  s->a = a;
  s->n = n_streams;
  s->back = a->h.max_pattern_len ? a->h.max_pattern_len - 1 : 0;
  s->overlapping = overlapping != 0;
  s->replace = rp != nullptr;
  DeviceGuard guard(a->device);
  cudaError_t e = cudaMalloc(&s->d_state, n_streams * 16);
  if (e != cudaSuccess) s->d_state = nullptr;
  if (e == cudaSuccess && (e = cudaMalloc(&s->d_tail, std::max<uint64_t>(n_streams * s->back, 16))) != cudaSuccess)
    s->d_tail = nullptr;
  if (e == cudaSuccess) e = cudaMemset(s->d_state, 0, n_streams * 16);
  if (e == cudaSuccess && rp) {
    const uint64_t n_reps = rp->n_reps, rep_total = rp->rep_offsets[n_reps] - rp->rep_offsets[0];
    std::vector<uint64_t> offs(rp->rep_offsets, rp->rep_offsets + n_reps + 1);
    offs.push_back(offs.back());
    if ((e = cudaMalloc(&s->d_rep, (n_reps + 2) * 8 + rep_total)) != cudaSuccess) s->d_rep = nullptr;
    if (e == cudaSuccess) e = cudaMemcpy(s->d_rep, offs.data(), (n_reps + 2) * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && rep_total)
      e = cudaMemcpy(s->d_rep + n_reps + 2, rp->rep_bytes + rp->rep_offsets[0], rep_total, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    acg_streams_free(s);
    return e == cudaErrorMemoryAllocation ? ACG_E_NOMEM : ACG_E_CUDA;
  }
  *out = s;
  return ACG_OK;
}

// acg_streams_lookahead(_devout): the LookLaunch steps (acb_device.cuh) into `out` (dev_out) or into the workspace's
// output buffer, copied to the host `out` from there.  Scratch: the tuple buffers (states and rows, sorted and not),
// the per-document counts (run starts, then the run index), d_scratch (the run of every row) and d_soffs (the ids).
// Nothing of the set is written.
int streams_lookahead_impl(const acg_streams* set, const acg_candidates* c, const uint64_t* ids, uint64_t n_ids,
                           uint8_t* out, bool dev_out) {
  if (!set || !c || c->a != set->a) return ACG_E_INVALID_ARG;
  const uint64_t n_rows = ids ? n_ids : set->n;
  if (n_rows >= (1ull << 32)) return ACG_E_INVALID_ARG;
  for (uint64_t i = 0; ids && i < n_ids; ++i)
    if (ids[i] >= set->n) return ACG_E_INVALID_ARG;
  const uint64_t total = n_rows * c->n;
  if (total && !out) return ACG_E_INVALID_ARG;
  if (!total) return ACG_OK;
  const acg_dfa* a = set->a;
  DeviceGuard guard(a->device);
  WsLease lease(a);
  if (lease.rc) return lease.rc;
  Workspace& w = cur_ws();
  int rc = reserve_tuples(w, std::max<uint64_t>(n_rows, 1 << 12));
  if (rc || (rc = reserve_docs(w, n_rows)) || (rc = w.d_scratch.reserve(std::max<uint64_t>(n_rows, 1 << 12))) ||
      (ids && (rc = w.d_soffs.reserve(n_rows))) || (!dev_out && (rc = w.d_out.reserve(total)))) {
    cudaGetLastError();  // a failed allocation: the buffers are empty again, the error is not sticky
    return ACG_E_NOMEM;
  }
  acb::LookLaunch p{};
  p.st.n = set->n;
  p.st.back = set->back;
  p.st.overlapping = set->overlapping;
  p.st.pos = set->d_state;
  p.st.cursor = set->d_state + set->n;
  p.st.tail = set->d_tail;
  p.ids = ids ? w.d_soffs.p : nullptr;
  p.n_rows = n_rows;
  p.cand_offsets = c->d_offs;
  p.cand_classes = c->d_classes;
  p.n_cands = c->n;
  p.keys = w.d_keys[0];
  p.rows = w.d_pids[0];
  p.skeys = w.d_keys[1];
  p.srows = w.d_pids[1];
  p.heads = w.d_doc_counts;
  p.row_u = w.d_scratch;
  p.out = dev_out ? out : w.d_out.p;
  p.sm_count = 132;
  cudaDeviceGetAttribute(&p.sm_count, cudaDevAttrMultiProcessorCount, a->device);
  const uint64_t max_id = (a->h.state_len - 1) << a->h.stride2;
  int end_bit = 1;
  while (end_bit < 64 && (max_id >> end_bit)) ++end_bit;
  if (ids) CK(cudaMemcpyAsync(w.d_soffs, ids, n_rows * 8, cudaMemcpyHostToDevice, w.stream));
  CK(cudaEventRecord(w.ev0, w.stream));
  CK(acb::launch_look_state(a->dev, p, w.stream));
  if ((rc = cub_call(w, [&](void* t, size_t& tb) {
         return acb::sort_pairs(t, tb, p.keys, p.skeys, p.rows, p.srows, n_rows, end_bit, w.stream);
       })))
    return rc;
  CK(acb::launch_look_heads(p, w.stream));
  if ((rc = cub_call(w, [&](void* t, size_t& tb) {
         return acb::inclusive_sum_u64(t, tb, p.heads, p.heads, n_rows, w.stream);
       })))
    return rc;
  CK(acb::launch_look_compact(p, w.stream));
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(acb::launch_look_mask(a->dev, p, w.stream));
  CK(cudaEventRecord(w.ev2, w.stream));
  CK(acb::launch_look_copy(p, w.stream));
  CK(cudaEventRecord(w.ev3, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, w.ev1, w.ev2);
  w.stats.scan_ms = ms;
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.order_ms = ms;
  cudaEventElapsedTime(&ms, w.ev2, w.ev3);
  w.stats.order_ms += ms;
  w.stats.launches = 7;
  if (dev_out) return ACG_OK;
  CK(cudaEventRecord(w.ev0, w.stream));
  if ((rc = copy_to_host(a, out, w.d_out, total))) return rc;
  CK(cudaEventRecord(w.ev1, w.stream));
  CK(cudaStreamSynchronize(w.stream));
  cudaEventElapsedTime(&ms, w.ev0, w.ev1);
  w.stats.d2h_ms = ms;
  return ACG_OK;
}

}  // namespace

extern "C" {

void acg_build_opts_default(acg_build_opts* o) {
  o->match_kind = ACG_STANDARD;
  o->start_kind = ACG_START_UNANCHORED;
  o->ascii_case_insensitive = 0;
  o->byte_classes = 1;
  o->prefilter = 1;
  o->kind = ACG_KIND_AUTO;
  o->dense_depth = 3;
}

static int build_common(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                        const acg_build_opts* opts, bool to_device, acg_dfa** out, bool device_fill = false) {
  if (!out) return ACG_E_INVALID_ARG;
  *out = nullptr;
  acg_build_opts def;
  acg_build_opts_default(&def);
  if (!opts) opts = &def;
  if (n && (!patterns || !lens)) return ACG_E_INVALID_ARG;
  acb::BuildOptions bo;
  bo.match_kind = opts->match_kind;
  bo.start_kind = opts->start_kind;
  bo.ascii_case_insensitive = opts->ascii_case_insensitive != 0;
  bo.byte_classes = opts->byte_classes != 0;
  bo.prefilter = opts->prefilter != 0;
  bo.kind = opts->kind;
  bo.defer_dense = device_fill && to_device;
  std::vector<acb::PatternRef> pats(n);
  for (uint64_t i = 0; i < n; ++i) pats[i] = acb::PatternRef{patterns[i], lens[i]};
  acg_dfa* a = new (std::nothrow) acg_dfa();
  if (!a) return ACG_E_NOMEM;
  int rc = ACG_OK;
  static const bool trace = std::getenv("ACB_BUILD_TRACE") != nullptr;
  auto t0 = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!trace) return;
    const auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "acb200 build: %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t0).count());
    t0 = now;
  };
  try {
    rc = acb::build_dfa(pats, bo, &a->h);
    lap("build_dfa total");
    if (rc == ACG_OK) derive_metadata(a);
    lap("derive_metadata (device plan)");
  } catch (const std::bad_alloc&) {
    rc = ACG_E_NOMEM;
  }
  if (rc == ACG_OK && to_device) rc = upload(a);
  lap("upload / device fill");
  if (rc != ACG_OK) { acg_dfa_free(a); return rc; }
  *out = a;
  return ACG_OK;
}

int acg_build(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
              const acg_build_opts* opts, acg_dfa** out) {
  return build_common(patterns, lens, n, opts, true, out);
}
int acg_build_host(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                   const acg_build_opts* opts, acg_dfa** out) {
  return build_common(patterns, lens, n, opts, false, out);
}
int acg_build_on_device(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                        const acg_build_opts* opts, acg_dfa** out) {
  return build_common(patterns, lens, n, opts, true, out, true);
}

// Structural checks of an adopted table (the layout facts of src/dfa.rs:91-132 the kernels rely
// on): a malformed descriptor is rejected instead of being indexed out of bounds on the device.
static bool desc_is_consistent(const acg_dfa_desc* d) {
  if (!d->trans || !d->match_offsets || (!d->pattern_lens && d->n_patterns)) return false;
  if (d->stride2 > 8 || d->alphabet_len == 0 || d->alphabet_len > (1u << d->stride2)) return false;
  const uint64_t stride = 1ull << d->stride2;
  if (d->trans_len == 0 || (d->trans_len & (stride - 1)) || d->trans_len > (1ull << 32)) return false;
  const uint64_t rows = d->trans_len >> d->stride2;
  if (rows < 4) return false;  // DEAD, FAIL and the two start rows always exist
  if (d->match_kind > ACG_LEFTMOST_LONGEST || d->start_kind > ACG_START_BOTH) return false;
  for (int b = 0; b < 256; ++b)
    if (d->byte_classes[b] >= d->alphabet_len) return false;
  // Row 1 is the FAIL sentinel of the noncontiguous NFA (src/dfa.rs:101-108): it is never the target
  // of a DFA transition nor a start state.  Its id is non-zero and <= max_match_id, so a kernel
  // would take it for a match state and index match_offsets[row - 2] out of bounds.
  auto id_ok = [&](uint32_t id) { return (id & (stride - 1)) == 0 && id < d->trans_len; };
  auto target_ok = [&](uint32_t id) { return id_ok(id) && id != stride; };
  if (!id_ok(d->max_match_id) || !target_ok(d->start_unanchored_id) || !target_ok(d->start_anchored_id) ||
      !id_ok(d->max_special_id))
    return false;
  const uint64_t max_match_row = d->max_match_id >> d->stride2;
  if (max_match_row < 1 || max_match_row >= rows) return false;
  for (uint64_t i = 0; i < d->trans_len; ++i)
    if (!target_ok(d->trans[i])) return false;
  const uint64_t nms = max_match_row - 1;  // match rows are 2 ..= max_match_row
  if (d->match_offsets[0] != 0) return false;
  for (uint64_t m = 0; m < nms; ++m)
    if (d->match_offsets[m + 1] < d->match_offsets[m]) return false;
  const uint64_t n_pids = d->match_offsets[nms];
  if (n_pids && !d->match_pids) return false;
  for (uint64_t i = 0; i < n_pids; ++i)
    if (d->match_pids[i] >= d->n_patterns) return false;
  for (uint32_t i = 0; i < d->n_patterns; ++i)
    if (d->pattern_lens[i] < d->min_pattern_len || d->pattern_lens[i] > d->max_pattern_len) return false;
  return true;
}

int acg_dfa_create(const acg_dfa_desc* d, acg_dfa** out) {
  if (!d || !out) return ACG_E_INVALID_ARG;
  *out = nullptr;
  if (!desc_is_consistent(d)) return ACG_E_INVALID_ARG;
  acg_dfa* a = new (std::nothrow) acg_dfa();
  if (!a) return ACG_E_NOMEM;
  HostDfa& h = a->h;
  try {
    h.trans.assign(d->trans, d->trans + d->trans_len);
    h.trans_len = d->trans_len;
    h.stride2 = d->stride2;
    h.alphabet_len = d->alphabet_len;
    std::memcpy(h.classes, d->byte_classes, 256);
    h.max_special_id = d->max_special_id;
    h.max_match_id = d->max_match_id;
    h.start_unanchored_id = d->start_unanchored_id;
    h.start_anchored_id = d->start_anchored_id;
    const size_t nms = size_t(d->max_match_id >> d->stride2) - 1;
    h.match_offsets.assign(d->match_offsets, d->match_offsets + nms + 1);
    h.match_pids.assign(d->match_pids, d->match_pids + h.match_offsets[nms]);
    h.pattern_lens.assign(d->pattern_lens, d->pattern_lens + d->n_patterns);
    h.match_kind = int(d->match_kind);
    h.start_kind = int(d->start_kind);
    h.prefilter_kind = int(d->prefilter_kind);
    h.reported_kind = ACG_KIND_DFA;
    h.min_pattern_len = d->min_pattern_len;
    h.max_pattern_len = d->max_pattern_len;
    h.state_len = d->trans_len >> d->stride2;
    derive_metadata(a);
  } catch (const std::bad_alloc&) {
    delete a;
    return ACG_E_NOMEM;
  }
  int rc = upload(a);
  if (rc != ACG_OK && rc != ACG_E_NO_DEVICE) { acg_dfa_free(a); return rc; }
  *out = a;  // without a device the handle is host-only (searches report ACG_E_NO_DEVICE)
  return ACG_OK;
}

void acg_dfa_free(acg_dfa* a) {
  if (!a) return;
  if (a->on_device || a->dev_touched) {
    DeviceGuard guard(a->device);
    for (Workspace* w : a->ws_all) { destroy_workspace(*w); delete w; }
    cudaFree(a->d_trans); cudaFree(a->d_classes); cudaFree(a->d_moff); cudaFree(a->d_mpids);
    cudaFree(a->d_plens); cudaFree(a->d_depth16); cudaFree(a->d_bitmap); cudaFree(a->d_amap);
  }
  delete a;
}

namespace {
// The table of a handle whose dense fill ran on the device, fetched on demand.
int fetch_table(const acg_dfa* a) {
  HostDfa& h = const_cast<acg_dfa*>(a)->h;
  if (!h.fill.valid || !h.trans.empty()) return ACG_OK;
  if (!a->d_trans) return ACG_E_NO_DEVICE;
  std::lock_guard<std::mutex> lock(a->mu);
  if (!h.trans.empty()) return ACG_OK;
  DeviceGuard guard(a->device);
  std::vector<uint32_t> t(size_t(h.trans_len));
  if (cudaMemcpy(t.data(), a->d_trans, t.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
    cudaGetLastError();
    return ACG_E_CUDA;
  }
  h.trans.swap(t);
  return ACG_OK;
}

}  // namespace

int acg_dfa_table(const acg_dfa* a, acg_dfa_desc* o) {
  if (!a || !o) return ACG_E_INVALID_ARG;
  if (int rc = fetch_table(a)) return rc;
  const HostDfa& h = a->h;
  o->trans = h.trans.data();
  o->trans_len = h.trans.size();
  o->stride2 = h.stride2;
  o->alphabet_len = h.alphabet_len;
  std::memcpy(o->byte_classes, h.classes, 256);
  o->max_special_id = h.max_special_id;
  o->max_match_id = h.max_match_id;
  o->start_unanchored_id = h.start_unanchored_id;
  o->start_anchored_id = h.start_anchored_id;
  o->match_offsets = h.match_offsets.data();
  o->match_pids = h.match_pids.data();
  o->pattern_lens = h.pattern_lens.data();
  o->n_patterns = uint32_t(h.pattern_lens.size());
  o->match_kind = uint32_t(h.match_kind);
  o->start_kind = uint32_t(h.start_kind);
  o->prefilter_kind = uint32_t(h.prefilter_kind);
  o->min_pattern_len = h.min_pattern_len;
  o->max_pattern_len = h.max_pattern_len;
  return ACG_OK;
}

uint64_t acg_dfa_state_len(const acg_dfa* a) { return a ? a->h.state_len : 0; }
int acg_kind(const acg_dfa* a) { return a ? a->h.reported_kind : 0; }
int acg_match_kind(const acg_dfa* a) { return a ? a->h.match_kind : 0; }
int acg_start_kind(const acg_dfa* a) { return a ? a->h.start_kind : 0; }
uint64_t acg_patterns_len(const acg_dfa* a) { return a ? a->h.pattern_lens.size() : 0; }
uint64_t acg_min_pattern_len(const acg_dfa* a) { return a ? a->h.min_pattern_len : 0; }
uint64_t acg_max_pattern_len(const acg_dfa* a) { return a ? a->h.max_pattern_len : 0; }
uint64_t acg_memory_usage(const acg_dfa* a) {
  if (!a) return 0;  // DFA::memory_usage, src/dfa.rs:289-297 (heap of the tables)
  const HostDfa& h = a->h;
  return h.trans_len * 4 + (h.match_offsets.size() - 1) * 24 + h.match_pids.size() * 4 +
         h.pattern_lens.size() * 4;
}
int acg_prefilter_kind(const acg_dfa* a) { return a ? a->h.prefilter_kind : 0; }
int acg_packed_variant(const acg_dfa* a, int* fat, int* mask_len) {
  if (!a || !a->h.packed.active) return 0;
  if (fat) *fat = a->h.packed.fat;
  if (mask_len) *mask_len = a->h.packed.mask_len;
  return 1;
}

int acg_debug_prefilter_plan(const acg_dfa* a, acg_prefilter_plan* out) {
  if (!a || !out) return ACG_E_INVALID_ARG;
  const acb::PrefilterPlan& pf = a->pf;
  *out = acg_prefilter_plan{};
  out->supported = pf.supported ? 1 : 0;
  out->brute = pf.brute ? 1 : 0;
  out->dense = pf.dense ? 1 : 0;
  out->stride = int32_t(pf.stride);
  out->wide = pf.wide ? 1 : 0;
  out->k = pf.k; out->kmask = pf.kmask; out->fold = pf.fold;
  out->mult = pf.mult; out->mult3 = pf.mult3; out->key_shift = pf.key_shift; out->shift = pf.shift; out->log_bits = pf.log_bits;
  out->bitmap = pf.bitmap.data(); out->bitmap_words = pf.bitmap.size();
  out->amap = pf.amap.data(); out->amap_log = pf.amap_log;
  out->depth16 = a->depth16.data(); out->n_rows = a->depth16.size();
  out->dup_shift = pf.dup_shift;
  out->bs_n = (pf.bs_n && !a->bytescan_inert) ? pf.bs_n : 0;
  for (int i = 0; i < 3; ++i) { out->bs_byte[i] = pf.bs_byte[i]; out->bs_back[i] = pf.bs_back[i]; }
  return ACG_OK;
}

int acg_debug_set_pipeline_chunk(acg_dfa* a, uint64_t bytes) {
  if (!a || bytes < 4096 || (bytes & 4095)) return ACG_E_INVALID_ARG;
  a->pipeline_chunk = bytes;
  return ACG_OK;
}

int acg_debug_set_experiment(acg_dfa* a, uint32_t flags) {
  if (!a || (flags & ~uint32_t(ACG_EXP_KEY24 | ACG_EXP_STATIC_TILES | ACG_EXP_NO_BYTESCAN | ACG_EXP_GLOBAL_TILES))) return ACG_E_INVALID_ARG;
  std::lock_guard<std::mutex> lock(a->mu);
  const uint32_t changed = a->experiment ^ flags;
  a->experiment = flags;
  if (changed & ACG_EXP_KEY24) {
    // the first-stage keys are part of the plan: rebuild it and refresh the device copy of the bitmap
    const size_t old_words = a->pf.bitmap.size();
    a->pf = acb::plan_prefilter(a->h, a->depth16, (flags & ACG_EXP_KEY24) != 0);
    if (a->on_device && a->d_bitmap && a->pf.supported) {
      if (a->pf.bitmap.size() != old_words) return ACG_E_INVALID_ARG;  // the geometry does not depend on the keys
      DeviceGuard guard(a->device);
      if (cudaMemcpy(a->d_bitmap, a->pf.bitmap.data(), old_words * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaGetLastError();
        return ACG_E_CUDA;
      }
    }
  }
  return ACG_OK;
}

int acg_set_engine(acg_dfa* a, int engine) {
  if (!a || engine < ACG_ENGINE_AUTO || engine > ACG_ENGINE_SEQUENTIAL) return ACG_E_INVALID_ARG;
  a->engine_override = engine;
  return ACG_OK;
}
// Statistics of the most recent search on this handle: the calling thread's own last search if it
// made one (concurrent callers do not see each other's numbers), else the search that finished last.
static acg_stats stats_for(const acg_dfa* a) {
  if (tls_stats_owner == a) return tls_stats;
  std::lock_guard<std::mutex> lk(a->mu);
  return a->last_stats;
}
int acg_last_engine(const acg_dfa* a) { return a ? stats_for(a).engine : 0; }
int acg_last_stats(const acg_dfa* a, acg_stats* out) {
  if (!a || !out) return ACG_E_INVALID_ARG;
  *out = stats_for(a);
  return ACG_OK;
}

int acg_find_overlapping(const acg_dfa* a, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
                         uint64_t span_end, int anchored, acg_match* out, uint64_t cap,
                         uint64_t* n_out) {
  return overlapping_impl(a, hay, false, hay_len, span_start, span_end, anchored, out, cap, n_out,
                          nullptr, nullptr);
}
int acg_find_overlapping_dev(const acg_dfa* a, const void* d_hay, uint64_t hay_len,
                             uint64_t span_start, uint64_t span_end, acg_match* out, uint64_t cap,
                             uint64_t* n_out, float* kernel_ms) {
  return overlapping_impl(a, static_cast<const uint8_t*>(d_hay), true, hay_len, span_start, span_end,
                          0, out, cap, n_out, nullptr, kernel_ms);
}
int acg_find_overlapping_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len,
                                uint64_t span_start, uint64_t span_end, uint64_t min_end,
                                uint64_t offset_add, void* d_out, uint64_t cap, uint64_t* n_out,
                                float* kernel_ms) {
  if (!d_out && cap) return ACG_E_INVALID_ARG;
  DevOut dv;
  dv.d_out = d_out;
  dv.min_end = min_end;
  dv.offset_add = offset_add;
  return overlapping_impl(a, static_cast<const uint8_t*>(d_hay), true, hay_len, span_start, span_end, 0,
                          nullptr, cap, n_out, nullptr, kernel_ms, &dv);
}
int acg_count_overlapping_dev(const acg_dfa* a, const void* d_hay, uint64_t hay_len,
                              uint64_t span_start, uint64_t span_end, uint64_t* n_out, uint64_t* fnv,
                              float* kernel_ms) {
  uint64_t dummy_fnv = 0;
  return overlapping_impl(a, static_cast<const uint8_t*>(d_hay), true, hay_len, span_start, span_end,
                          0, nullptr, 0, n_out, fnv ? fnv : &dummy_fnv, kernel_ms);
}

int acg_find_iter(const acg_dfa* a, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
                  uint64_t span_end, int anchored, acg_match* out, uint64_t cap, uint64_t* n_out) {
  return find_iter_impl(a, hay, false, hay_len, span_start, span_end, anchored, out, cap, n_out,
                        nullptr);
}
int acg_find_iter_dev(const acg_dfa* a, const void* d_hay, uint64_t hay_len, uint64_t span_start,
                      uint64_t span_end, acg_match* out, uint64_t cap, uint64_t* n_out,
                      float* kernel_ms) {
  return find_iter_impl(a, static_cast<const uint8_t*>(d_hay), true, hay_len, span_start, span_end, 0,
                        out, cap, n_out, kernel_ms);
}

int acg_find_iter_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                        const uint64_t* doc_offsets, uint64_t n_docs, int anchored, acg_doc_match* out, uint64_t cap,
                        uint64_t* n_out) {
  return batch_impl(a, kBatchFindIter, hay, hay_on_device != 0, hay_len, doc_offsets, n_docs, anchored,
                    reinterpret_cast<acg_match*>(out), cap, n_out, nullptr);
}
int acg_find_overlapping_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                               const uint64_t* doc_offsets, uint64_t n_docs, int anchored, acg_doc_match* out,
                               uint64_t cap, uint64_t* n_out) {
  return batch_impl(a, kBatchOverlapping, hay, hay_on_device != 0, hay_len, doc_offsets, n_docs, anchored,
                    reinterpret_cast<acg_match*>(out), cap, n_out, nullptr);
}
int acg_is_match_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                       const uint64_t* doc_offsets, uint64_t n_docs, int anchored, uint8_t* flags) {
  return batch_impl(a, kBatchIsMatch, hay, hay_on_device != 0, hay_len, doc_offsets, n_docs, anchored, nullptr, 0,
                    nullptr, flags);
}
int acg_find_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                   const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int earliest, acg_doc_match* out,
                   uint8_t* found) {
  return batch_impl(a, kBatchFind, hay, hay_on_device != 0, hay_len, doc_offsets, n_docs, anchored,
                    reinterpret_cast<acg_match*>(out), n_docs, nullptr, found, earliest != 0);
}

int acg_find_iter_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                               int offsets_on_device, uint64_t n_docs, int anchored, acg_doc_match* d_out,
                               uint64_t cap, uint64_t* d_match_offsets, uint64_t* n_out) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  dv.match_offsets = d_match_offsets;
  return batch_impl(a, kBatchFindIter, static_cast<const uint8_t*>(d_hay), true, hay_len, doc_offsets, n_docs,
                    anchored, reinterpret_cast<acg_match*>(d_out), cap, n_out, nullptr, 0, &dv);
}
int acg_find_overlapping_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len,
                                      const uint64_t* doc_offsets, int offsets_on_device, uint64_t n_docs,
                                      int anchored, acg_doc_match* d_out, uint64_t cap, uint64_t* d_match_offsets,
                                      uint64_t* n_out) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  dv.match_offsets = d_match_offsets;
  return batch_impl(a, kBatchOverlapping, static_cast<const uint8_t*>(d_hay), true, hay_len, doc_offsets, n_docs,
                    anchored, reinterpret_cast<acg_match*>(d_out), cap, n_out, nullptr, 0, &dv);
}
int acg_is_match_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                              int offsets_on_device, uint64_t n_docs, int anchored, uint8_t* d_flags) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  return batch_impl(a, kBatchIsMatch, static_cast<const uint8_t*>(d_hay), true, hay_len, doc_offsets, n_docs,
                    anchored, nullptr, 0, nullptr, d_flags, 0, &dv);
}
int acg_find_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                          int offsets_on_device, uint64_t n_docs, int anchored, int earliest, acg_doc_match* d_out,
                          uint8_t* d_found) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  return batch_impl(a, kBatchFind, static_cast<const uint8_t*>(d_hay), true, hay_len, doc_offsets, n_docs,
                    anchored, reinterpret_cast<acg_match*>(d_out), n_docs, nullptr, d_found, earliest != 0, &dv);
}

int acg_pattern_counts_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int overlapping,
                             uint64_t* row_offsets, uint32_t* pids, uint64_t* counts, uint64_t cap, uint64_t* nnz) {
  const BatchCounts co{row_offsets, pids, counts};
  return batch_impl(a, overlapping ? kBatchOverlapping : kBatchFindIter, hay, hay_on_device != 0, hay_len, doc_offsets,
                    n_docs, anchored, nullptr, cap, nnz, nullptr, 0, nullptr, &co);
}
int acg_pattern_counts_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                                    int offsets_on_device, uint64_t n_docs, int anchored, int overlapping,
                                    uint64_t* d_row_offsets, uint32_t* d_pids, uint64_t* d_counts, uint64_t cap,
                                    uint64_t* nnz) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  const BatchCounts co{d_row_offsets, d_pids, d_counts};
  return batch_impl(a, overlapping ? kBatchOverlapping : kBatchFindIter, static_cast<const uint8_t*>(d_hay), true,
                    hay_len, doc_offsets, n_docs, anchored, nullptr, cap, nnz, nullptr, 0, &dv, &co);
}

int acg_match_coverage_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* doc_offsets, uint64_t n_docs, int anchored, int overlapping,
                             uint64_t* covered, uint8_t* mask) {
  const BatchCoverage cv{covered, mask};
  uint64_t unused = 0;
  return batch_impl(a, overlapping ? kBatchOverlapping : kBatchFindIter, hay, hay_on_device != 0, hay_len, doc_offsets,
                    n_docs, anchored, nullptr, 0, &unused, nullptr, 0, nullptr, nullptr, &cv);
}
int acg_match_coverage_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                                    int offsets_on_device, uint64_t n_docs, int anchored, int overlapping,
                                    uint64_t* d_covered, uint8_t* d_mask) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  const BatchCoverage cv{d_covered, d_mask};
  uint64_t unused = 0;
  return batch_impl(a, overlapping ? kBatchOverlapping : kBatchFindIter, static_cast<const uint8_t*>(d_hay), true,
                    hay_len, doc_offsets, n_docs, anchored, nullptr, 0, &unused, nullptr, 0, &dv, nullptr, &cv);
}

int acg_replace_all_batch(const acg_dfa* a, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                          const uint64_t* doc_offsets, uint64_t n_docs, const uint8_t* rep_bytes,
                          const uint64_t* rep_offsets, uint64_t n_reps, uint8_t* out, uint64_t cap,
                          uint64_t* out_offsets, uint64_t* out_len) {
  const BatchReplace rp{rep_bytes, rep_offsets, n_reps, out, out_offsets};
  return batch_impl(a, kBatchFindIter, hay, hay_on_device != 0, hay_len, doc_offsets, n_docs, 0, nullptr, cap,
                    out_len, nullptr, 0, nullptr, nullptr, nullptr, &rp);
}
int acg_replace_all_batch_devout(const acg_dfa* a, const void* d_hay, uint64_t hay_len, const uint64_t* doc_offsets,
                                 int offsets_on_device, uint64_t n_docs, const uint8_t* rep_bytes,
                                 const uint64_t* rep_offsets, uint64_t n_reps, uint8_t* d_out, uint64_t cap,
                                 uint64_t* d_out_offsets, uint64_t* out_len) {
  BatchDevOut dv;
  dv.offsets_on_device = offsets_on_device != 0;
  const BatchReplace rp{rep_bytes, rep_offsets, n_reps, d_out, d_out_offsets};
  return batch_impl(a, kBatchFindIter, static_cast<const uint8_t*>(d_hay), true, hay_len, doc_offsets, n_docs, 0,
                    nullptr, cap, out_len, nullptr, 0, &dv, nullptr, nullptr, &rp);
}

int acg_streams_create(const acg_dfa* a, uint64_t n_streams, int overlapping, acg_streams** out) {
  return streams_create(a, n_streams, overlapping, nullptr, out);
}

int acg_streams_create_replace(const acg_dfa* a, uint64_t n_streams, const uint8_t* rep_bytes,
                               const uint64_t* rep_offsets, uint64_t n_reps, acg_streams** out) {
  const BatchReplace rp{rep_bytes, rep_offsets, n_reps, nullptr, nullptr};
  return streams_create(a, n_streams, 0, &rp, out);
}

void acg_streams_free(acg_streams* s) {
  if (!s) return;
  {
    DeviceGuard guard(s->a->device);
    cudaFree(s->d_state);
    cudaFree(s->d_tail);
    cudaFree(s->d_rep);
  }
  delete s;
}

int acg_streams_reset(acg_streams* s, const uint64_t* ids, uint64_t n_ids) {
  if (!s) return ACG_E_INVALID_ARG;
  if (ids)
    for (uint64_t i = 0; i < n_ids; ++i)
      if (ids[i] >= s->n) return ACG_E_INVALID_ARG;
  DeviceGuard guard(s->a->device);
  if (!ids) {
    CK(cudaMemset(s->d_state, 0, s->n * 16));
    return ACG_OK;
  }
  std::vector<uint64_t> st(2 * s->n);
  CK(cudaMemcpy(st.data(), s->d_state, s->n * 16, cudaMemcpyDeviceToHost));
  for (uint64_t i = 0; i < n_ids; ++i) st[ids[i]] = st[s->n + ids[i]] = 0;
  CK(cudaMemcpy(s->d_state, st.data(), s->n * 16, cudaMemcpyHostToDevice));
  return ACG_OK;
}

int acg_streams_positions(const acg_streams* s, uint64_t* pos) {
  if (!s || !pos) return ACG_E_INVALID_ARG;
  DeviceGuard guard(s->a->device);
  CK(cudaMemcpy(pos, s->d_state, s->n * 8, cudaMemcpyDeviceToHost));
  return ACG_OK;
}

int acg_streams_feed(acg_streams* s, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                     const uint64_t* chunk_offsets, uint64_t n_streams, acg_doc_match* out, uint64_t cap,
                     uint64_t* n_out) {
  return streams_feed_impl(s, hay, hay_on_device != 0, hay_len, chunk_offsets, false, n_streams, out, cap, nullptr,
                           false, false, n_out);
}

int acg_streams_feed_devout(acg_streams* s, const void* d_hay, uint64_t hay_len, const uint64_t* chunk_offsets,
                            int offsets_on_device, uint64_t n_streams, acg_doc_match* d_out, uint64_t cap,
                            uint64_t* d_match_offsets, uint64_t* n_out) {
  return streams_feed_impl(s, static_cast<const uint8_t*>(d_hay), true, hay_len, chunk_offsets,
                           offsets_on_device != 0, n_streams, d_out, cap, d_match_offsets, true, false, n_out);
}

int acg_streams_replace_feed(acg_streams* s, const uint8_t* hay, int hay_on_device, uint64_t hay_len,
                             const uint64_t* chunk_offsets, uint64_t n_streams, uint8_t* out, uint64_t cap,
                             uint64_t* out_offsets, uint64_t* out_len) {
  return streams_feed_impl(s, hay, hay_on_device != 0, hay_len, chunk_offsets, false, n_streams, out, cap,
                           out_offsets, false, true, out_len);
}

int acg_streams_replace_feed_devout(acg_streams* s, const void* d_hay, uint64_t hay_len,
                                    const uint64_t* chunk_offsets, int offsets_on_device, uint64_t n_streams,
                                    uint8_t* d_out, uint64_t cap, uint64_t* d_out_offsets, uint64_t* out_len) {
  return streams_feed_impl(s, static_cast<const uint8_t*>(d_hay), true, hay_len, chunk_offsets,
                           offsets_on_device != 0, n_streams, d_out, cap, d_out_offsets, true, true, out_len);
}

int acg_streams_held(const acg_streams* s, uint64_t* held) {
  if (!s || !s->replace || !held) return ACG_E_INVALID_ARG;
  std::vector<uint64_t> st(2 * s->n);
  DeviceGuard guard(s->a->device);
  CK(cudaMemcpy(st.data(), s->d_state, s->n * 16, cudaMemcpyDeviceToHost));
  for (uint64_t i = 0; i < s->n; ++i) held[i] = std::min(s->back, st[i] - st[s->n + i]);
  return ACG_OK;
}

// The held bytes of the listed streams are their tails (L_s = held_s): their lengths and offsets are worked out on
// the host from the state, and one kernel gathers the tails and zeroes the state.
int acg_streams_flush(acg_streams* s, const uint64_t* ids, uint64_t n_ids, uint8_t* out, uint64_t cap,
                      uint64_t* out_offsets, uint64_t* out_len) {
  if (!s || !s->replace || !out_offsets || !out_len || (!out && cap)) return ACG_E_INVALID_ARG;
  const uint64_t n = s->n, k = ids ? n_ids : n;
  if (ids) {
    std::vector<uint8_t> seen(n, 0);
    for (uint64_t i = 0; i < n_ids; ++i)
      if (ids[i] >= n || seen[ids[i]]++) return ACG_E_INVALID_ARG;
  }
  *out_len = 0;
  const acg_dfa* a = s->a;
  DeviceGuard guard(a->device);
  std::vector<uint64_t> st(2 * n), offs(k + 1, 0);
  CK(cudaMemcpy(st.data(), s->d_state, n * 16, cudaMemcpyDeviceToHost));
  for (uint64_t j = 0; j < k; ++j) {
    const uint64_t i = ids ? ids[j] : j;
    offs[j + 1] = offs[j] + std::min(s->back, st[i] - st[n + i]);
  }
  const uint64_t total = offs[k];
  *out_len = total;
  if (total > cap) return ACG_E_OVERFLOW;
  if (k) {
    WsLease lease(a);
    if (lease.rc) return lease.rc;
    Workspace& w = cur_ws();
    int rc = w.d_soffs.reserve(2 * k + 1);
    if (rc || (rc = w.d_out.reserve(std::max<uint64_t>(total, 1 << 20)))) return rc;
    acb::StreamLaunch p{};
    p.n = n;
    p.back = s->back;
    p.pos = s->d_state;
    p.cursor = s->d_state + n;
    p.tail = s->d_tail;
    uint64_t* d_ids = w.d_soffs + (k + 1);
    CK(cudaMemcpyAsync(w.d_soffs, offs.data(), (k + 1) * 8, cudaMemcpyHostToDevice, w.stream));
    if (ids) CK(cudaMemcpyAsync(d_ids, ids, k * 8, cudaMemcpyHostToDevice, w.stream));
    CK(acb::launch_stream_flush(p, ids ? d_ids : nullptr, k, w.d_soffs, w.d_out, w.stream));
    if (total && (rc = copy_to_host(a, out, w.d_out, total))) return rc;
    CK(cudaStreamSynchronize(w.stream));
  }
  std::copy(offs.begin(), offs.end(), out_offsets);
  return ACG_OK;
}

int acg_candidates_create(const acg_dfa* a, const uint8_t* bytes, const uint64_t* offsets, uint64_t n_cands,
                          acg_candidates** out) {
  if (!a || !out || !offsets || n_cands >= (1ull << 32)) return ACG_E_INVALID_ARG;
  *out = nullptr;
  for (uint64_t i = 0; i < n_cands; ++i)
    if (offsets[i + 1] < offsets[i]) return ACG_E_INVALID_ARG;
  const uint64_t total = offsets[n_cands] - offsets[0];
  if (total && !bytes) return ACG_E_INVALID_ARG;
  if (!a->on_device) return ACG_E_NO_DEVICE;
  std::vector<uint64_t> offs;
  std::vector<uint8_t> cls;
  try {
    offs.resize(n_cands + 1);
    cls.resize(total);
  } catch (const std::bad_alloc&) {
    return ACG_E_NOMEM;
  }
  for (uint64_t i = 0; i <= n_cands; ++i) offs[i] = offsets[i] - offsets[0];
  for (uint64_t i = 0; i < total; ++i) cls[i] = a->h.classes[bytes[offsets[0] + i]];
  acg_candidates* c = new (std::nothrow) acg_candidates();
  if (!c) return ACG_E_NOMEM;
  c->a = a;
  c->n = n_cands;
  DeviceGuard guard(a->device);
  cudaError_t e = cudaMalloc(&c->d_offs, (n_cands + 1) * 8);
  if (e != cudaSuccess) c->d_offs = nullptr;
  if (e == cudaSuccess && (e = cudaMalloc(&c->d_classes, std::max<uint64_t>(total, 16))) != cudaSuccess)
    c->d_classes = nullptr;
  if (e == cudaSuccess) e = cudaMemcpy(c->d_offs, offs.data(), (n_cands + 1) * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && total) e = cudaMemcpy(c->d_classes, cls.data(), total, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaGetLastError();
    acg_candidates_free(c);
    return e == cudaErrorMemoryAllocation ? ACG_E_NOMEM : ACG_E_CUDA;
  }
  *out = c;
  return ACG_OK;
}

void acg_candidates_free(acg_candidates* c) {
  if (!c) return;
  {
    DeviceGuard guard(c->a->device);
    cudaFree(c->d_offs);
    cudaFree(c->d_classes);
  }
  delete c;
}

int acg_streams_lookahead(const acg_streams* s, const acg_candidates* c, const uint64_t* ids, uint64_t n_ids,
                          uint8_t* out) {
  return streams_lookahead_impl(s, c, ids, n_ids, out, false);
}

int acg_streams_lookahead_devout(const acg_streams* s, const acg_candidates* c, const uint64_t* ids, uint64_t n_ids,
                                 uint8_t* d_out) {
  return streams_lookahead_impl(s, c, ids, n_ids, d_out, true);
}

int acg_find(const acg_dfa* a, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
             uint64_t span_end, int anchored, int earliest, acg_match* out, int* found) {
  return find_impl(a, hay, hay_len, span_start, span_end, anchored, earliest, out, found);
}

// ---- packed searcher (src/packed/api.rs) ----------------------------------------------------

struct acg_packed {
  acg_dfa* inner = nullptr;  // leftmost DFA over the same patterns: the device engine
  int match_kind = ACG_LEFTMOST_FIRST;
  bool teddy = false;
  bool fat = false;
  int mask_len = 0;
  int vector_bytes = 0;
  uint64_t minimum_len = 0;
};

void acg_packed_config_default(acg_packed_config* c) {
  c->match_kind = ACG_LEFTMOST_FIRST;
  c->force = ACG_PACKED_FORCE_NONE;
  c->only_teddy_fat = -1;
  c->only_teddy_256bit = -1;
  c->heuristic_pattern_limits = 1;
}

static int packed_build_common(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                               const acg_packed_config* cfg, bool to_device, acg_packed** out) {
  if (!out) return ACG_E_INVALID_ARG;
  *out = nullptr;
  acg_packed_config def;
  acg_packed_config_default(&def);
  if (!cfg) cfg = &def;
  if (n && (!patterns || !lens)) return ACG_E_INVALID_ARG;
  if (cfg->match_kind != ACG_LEFTMOST_FIRST && cfg->match_kind != ACG_LEFTMOST_LONGEST) return ACG_E_INVALID_ARG;
  // Builder::add (api.rs:303-322): the builder turns inert -- and build() returns None -- once a
  // 129th pattern or an empty pattern is offered; build() also returns None without patterns.
  constexpr uint64_t kPatternLimit = 128;  // PATTERN_LIMIT, api.rs:15
  if (n == 0 || n > kPatternLimit) return ACG_OK;
  uint64_t min_len = UINT64_MAX;
  for (uint64_t i = 0; i < n; ++i) {
    if (lens[i] == 0) return ACG_OK;
    min_len = std::min(min_len, lens[i]);
  }
  acg_packed plan;
  plan.match_kind = cfg->match_kind;
  if (cfg->force != ACG_PACKED_FORCE_RABINKARP) {
    // teddy::Builder::build_imp (teddy/builder.rs:98-231) as it decides on x86-64 with AVX2
    const bool limits = cfg->heuristic_pattern_limits != 0;
    if (limits && n > 64) return ACG_OK;
    const int mask_len = int(std::min<uint64_t>(4, min_len));
    const bool use_256 = cfg->only_teddy_256bit != 0;  // None -> AVX2 is available
    bool fat;
    if (cfg->only_teddy_fat < 0) fat = use_256 && n > 32;
    else if (cfg->only_teddy_fat == 0) fat = false;
    else { if (!use_256) return ACG_OK; fat = true; }
    if (limits && mask_len == 1 && n > 16) return ACG_OK;
    plan.teddy = true;
    plan.fat = fat;
    plan.mask_len = mask_len;
    // Slim SSSE3: 16 lanes; Slim AVX2: 32; Fat AVX2: 16 (two 128-bit halves), teddy/generic.rs:94-96, 427-429
    plan.vector_bytes = use_256 ? 32 : 16;
    const int width = (use_256 && !fat) ? 32 : 16;
    plan.minimum_len = uint64_t(width + mask_len - 1);
  }
  acg_build_opts o;
  acg_build_opts_default(&o);
  o.match_kind = cfg->match_kind;
  o.kind = ACG_KIND_DFA;
  acg_dfa* inner = nullptr;
  const int rc = to_device ? acg_build(patterns, lens, n, &o, &inner) : acg_build_host(patterns, lens, n, &o, &inner);
  if (rc != ACG_OK) return rc;
  acg_packed* s = new (std::nothrow) acg_packed(plan);
  if (!s) { acg_dfa_free(inner); return ACG_E_NOMEM; }
  s->inner = inner;
  *out = s;
  return ACG_OK;
}

int acg_packed_build(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                     const acg_packed_config* cfg, acg_packed** out) {
  return packed_build_common(patterns, lens, n, cfg, true, out);
}
int acg_packed_build_host(const uint8_t* const* patterns, const uint64_t* lens, uint64_t n,
                          const acg_packed_config* cfg, acg_packed** out) {
  return packed_build_common(patterns, lens, n, cfg, false, out);
}
void acg_packed_free(acg_packed* s) {
  if (!s) return;
  acg_dfa_free(s->inner);
  delete s;
}
int acg_packed_find_iter(const acg_packed* s, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
                         uint64_t span_end, acg_match* out, uint64_t cap, uint64_t* n_out) {
  if (!s) return ACG_E_INVALID_ARG;
  return acg_find_iter(s->inner, hay, hay_len, span_start, span_end, 0, out, cap, n_out);
}
int acg_packed_find(const acg_packed* s, const uint8_t* hay, uint64_t hay_len, uint64_t span_start,
                    uint64_t span_end, acg_match* out, int* found) {
  if (!s) return ACG_E_INVALID_ARG;
  return acg_find(s->inner, hay, hay_len, span_start, span_end, 0, 0, out, found);
}
int acg_packed_match_kind(const acg_packed* s) { return s ? s->match_kind : 0; }
uint64_t acg_packed_minimum_len(const acg_packed* s) { return s ? s->minimum_len : 0; }
uint64_t acg_packed_memory_usage(const acg_packed* s) { return s ? acg_memory_usage(s->inner) : 0; }
uint64_t acg_packed_patterns_len(const acg_packed* s) { return s ? acg_patterns_len(s->inner) : 0; }
int acg_packed_searcher_variant(const acg_packed* s, int* fat, int* mask_len, int* vector_bytes) {
  if (!s || !s->teddy) return 0;
  if (fat) *fat = s->fat ? 1 : 0;
  if (mask_len) *mask_len = s->mask_len;
  if (vector_bytes) *vector_bytes = s->vector_bytes;
  return 1;
}

// ---- multi-GPU (SURVEY.md section 8e) ---------------------------------------------------------

int acg_comm_unique_id(uint8_t id[ACG_COMM_ID_BYTES]) { return acb::comm_unique_id(id); }
int acg_comm_init(const uint8_t id[ACG_COMM_ID_BYTES], int rank, int nranks, acg_comm** out) {
  return acb::comm_create(id, rank, nranks, out);
}
void acg_comm_free(acg_comm* c) {
  if (!c) return;
  for (auto& step : c->steps) {  // steps nobody waited for: let their kernels finish, hand the workspaces back
    if (!step.active) continue;
    DeviceGuard guard(c->device);
    cudaEventSynchronize(step.done);
    release_workspace(static_cast<const acg_dfa*>(step.dfa), static_cast<Workspace*>(step.lease));
    step.active = false;
  }
  acb::comm_destroy(c);
}
int acg_comm_rank(const acg_comm* c) { return c ? c->rank : -1; }
int acg_comm_size(const acg_comm* c) { return c ? c->nranks : 0; }
int acg_comm_transport(const acg_comm* c) { return c ? c->transport : ACG_TRANSPORT_NONE; }

int acg_shard_plan(uint64_t span_start, uint64_t span_end, int nranks, int rank, uint64_t max_pattern_len,
                   uint64_t* own_lo, uint64_t* own_hi, uint64_t* read_lo) {
  if (!own_lo || !own_hi || !read_lo || nranks < 1 || rank < 0 || rank >= nranks || span_start > span_end)
    return ACG_E_INVALID_ARG;
  shard_plan(span_start, span_end, nranks, rank, max_pattern_len, own_lo, own_hi, read_lo);
  return ACG_OK;
}

int acg_find_overlapping_sharded(const acg_dfa* a, acg_comm* c, const void* hay, int hay_on_device,
                                 uint64_t hay_len, uint64_t hay_global_offset, uint64_t span_start,
                                 uint64_t span_end, const acg_match** d_matches, uint64_t* n_total,
                                 acg_match* h_out, uint64_t h_cap, acg_shard_stats* stats) {
  if (!n_total) return ACG_E_INVALID_ARG;
  *n_total = 0;
  if (d_matches) *d_matches = nullptr;
  if (stats) *stats = acg_shard_stats{};
  int slot = 0;
  int rc = sharded_begin(a, c, static_cast<const uint8_t*>(hay), hay_on_device != 0, hay_len, hay_global_offset,
                         span_start, span_end, /*streaming=*/false, &slot);
  if (rc == ACG_E_OVERFLOW && c && (c->steps[0].active || c->steps[1].active)) rc = ACG_E_INVALID_ARG;
  if (rc) return rc;
  return sharded_wait(c, slot, d_matches, n_total, h_out, h_cap, stats);
}

int acg_find_overlapping_sharded_begin(const acg_dfa* a, acg_comm* c, const void* hay, int hay_on_device,
                                       uint64_t hay_len, uint64_t hay_global_offset, uint64_t span_start,
                                       uint64_t span_end, int* ticket) {
  // ACB_GATHER_STORE=1: ship the records with the expand kernel's own peer stores, as the blocking
  // call does (kept for measurements; the copy-engine payload is what lets the next scan run undisturbed)
  static const bool store = getenv("ACB_GATHER_STORE") != nullptr;
  return sharded_begin(a, c, static_cast<const uint8_t*>(hay), hay_on_device != 0, hay_len, hay_global_offset,
                       span_start, span_end, /*streaming=*/!store, ticket);
}

int acg_comm_mark(acg_comm* c, int which) {
  if (!c || which < 0 || which > 1) return ACG_E_INVALID_ARG;
  DeviceGuard guard(c->device);
  if (!c->mark[which]) CK(cudaEventCreate(&c->mark[which]));
  // behind everything the device has been given so far (searches run on their handles' own streams)
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(c->mark[which], c->stream));
  CK(cudaEventSynchronize(c->mark[which]));
  return ACG_OK;
}

int acg_comm_mark_elapsed_ms(const acg_comm* c, float* ms) {
  if (!c || !ms || !c->mark[0] || !c->mark[1]) return ACG_E_INVALID_ARG;
  DeviceGuard guard(c->device);
  CK(cudaEventElapsedTime(ms, c->mark[0], c->mark[1]));
  return ACG_OK;
}
int acg_find_overlapping_sharded_wait(acg_comm* c, int ticket, const acg_match** d_matches, uint64_t* n_total,
                                      acg_match* h_out, uint64_t h_cap, acg_shard_stats* stats) {
  if (n_total) *n_total = 0;
  if (stats) *stats = acg_shard_stats{};
  return sharded_wait(c, ticket, d_matches, n_total, h_out, h_cap, stats);
}

int acg_comm_fetch(const acg_comm* c, acg_match* out, uint64_t cap, uint64_t* n_out) {
  if (!c || !n_out) return ACG_E_INVALID_ARG;
  const uint64_t total = c->last_total;
  *n_out = total;
  if (c->rank != 0) return ACG_E_INVALID_ARG;
  if (total > cap || (total && !out)) return ACG_E_OVERFLOW;
  DeviceGuard guard(c->device);
  if (total) CK(cudaMemcpy(out, c->last_result, size_t(total) * sizeof(acg_match), cudaMemcpyDeviceToHost));
  return ACG_OK;
}

int acg_comm_fetch_view(acg_comm* c, const acg_match** view, uint64_t* n_out) {
  if (!c || !view || !n_out || c->rank != 0) return ACG_E_INVALID_ARG;
  const uint64_t total = c->last_total;
  *n_out = total;
  *view = nullptr;
  DeviceGuard guard(c->device);
  if (total > c->h_view_cap) {
    if (c->h_view) { cudaFreeHost(c->h_view); c->h_view = nullptr; c->h_view_cap = 0; }
    const uint64_t cap = total + total / 8 + 1024;
    CK(cudaMallocHost(&c->h_view, size_t(cap) * sizeof(acg_match)));
    c->h_view_cap = cap;
  }
  if (total) {
    CK(cudaMemcpyAsync(c->h_view, c->last_result, size_t(total) * sizeof(acg_match), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  *view = reinterpret_cast<const acg_match*>(c->h_view);
  return ACG_OK;
}

int acg_comm_checksum(const acg_comm* c, uint64_t* n_out, uint64_t* fnv) {
  if (!c || !n_out || !fnv || c->rank != 0) return ACG_E_INVALID_ARG;
  const uint64_t total = c->last_total;
  *n_out = total;
  uint64_t hsh = 0xcbf29ce484222325ull;
  auto mix = [&](uint64_t v) {
    for (int k = 0; k < 8; ++k) { hsh ^= (v >> (8 * k)) & 0xFF; hsh *= 0x100000001b3ull; }
  };
  DeviceGuard guard(c->device);
  std::vector<acg_match> buf;
  const uint64_t chunk = 1 << 20;
  try { buf.resize(size_t(std::min<uint64_t>(chunk, std::max<uint64_t>(total, 1)))); } catch (const std::bad_alloc&) { return ACG_E_NOMEM; }
  for (uint64_t i = 0; i < total; i += chunk) {
    const uint64_t m = std::min(chunk, total - i);
    CK(cudaMemcpy(buf.data(), c->last_result + i * sizeof(acg_match), size_t(m) * sizeof(acg_match), cudaMemcpyDeviceToHost));
    for (uint64_t j = 0; j < m; ++j) { mix(buf[j].pid); mix(buf[j].start); mix(buf[j].end); }
  }
  *fnv = hsh;
  return ACG_OK;
}

const char* acg_strerror(int code) {
  switch (code) {
    case ACG_OK: return "ok";
    case ACG_E_STATE_ID_OVERFLOW: return "state identifier overflow";
    case ACG_E_PATTERN_ID_OVERFLOW: return "pattern identifier overflow";
    case ACG_E_PATTERN_TOO_LONG: return "pattern exceeds the maximum pattern length";
    case ACG_E_INVALID_INPUT_ANCHORED: return "anchored searches are not supported or enabled";
    case ACG_E_INVALID_INPUT_UNANCHORED: return "unanchored searches are not supported or enabled";
    case ACG_E_UNSUPPORTED_STREAM: return "match kind does not support stream searching";
    case ACG_E_UNSUPPORTED_OVERLAPPING: return "match kind does not support overlapping searches";
    case ACG_E_UNSUPPORTED_EMPTY: return "matching with an empty pattern string is not supported here";
    case ACG_E_INVALID_SPAN: return "invalid span for haystack";
    case ACG_E_OVERFLOW: return "output buffer too small";
    case ACG_E_INVALID_ARG: return "invalid argument";
    case ACG_E_CUDA: return "CUDA error";
    case ACG_E_NO_DEVICE: return "no usable CUDA device (there is no CPU fallback)";
    case ACG_E_NOMEM: return "out of memory";
    default: return "unknown error";
  }
}

int acg_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // extern "C"
