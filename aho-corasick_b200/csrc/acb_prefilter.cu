// acb_prefilter.cu -- K3/K3b: position-parallel k-gram prefilter fused with the
// anchored DFA verify, and the non-overlapping chain resolution.
//
// Why this shape on a GPU: the reference's per-byte loop (src/automaton.rs:1310-1418,
// 1491-1534) is one dependent table load per haystack byte -- latency bound, and
// on a GPU it forces one lane per shard with strided haystack reads.  Testing
// every *start position* independently instead reads the haystack exactly once,
// fully coalesced (16 B per lane), costs one shared-memory probe per position and
// leaves the dependent DFA walk to the few positions that survive (the role the
// packed/Teddy prefilter plays in the reference, src/packed/teddy/README.md).
// Exactness comes from the verifier, which walks the shipped DFA from the
// candidate offset while the state stays on the trie path that starts there
// (depth(state) == bytes consumed) and reports the node's own patterns -- the set
// of patterns that are a prefix of the haystack at that offset.
#include "acb_device.cuh"
#include "acb_fingerprint.cuh"
#ifndef ACB_PTX_HEADER
#define ACB_PTX_HEADER "acb_ptx.cuh"
#endif
#include ACB_PTX_HEADER

#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

namespace acb {
namespace {

// Kernel geometry.  NARROW (0): 1 024 threads, 1 KiB tile per warp step (2 x 16 positions per lane;
// stride 2 takes two such tiles per step, see PfPass);
// WIDE (1, stride 2 only): 512 threads, 2 KiB tile per warp step (4 x 16 positions per lane, 32
// probes), 16 KiB bitmap, two CTAs per SM -- the per-step bookkeeping is spread over twice as many
// positions, which pays when first-stage hits are rare (few patterns); with frequent hits the 32
// resident warps of the narrow geometry hide the latency of the second stage and the verifier
// better.  (A third geometry -- the 2 KiB tile with the 128 KiB bitmap, 20 warps -- lost to the
// narrow one on cfg 2 and cfg 3 and was dropped.)
enum : int { kGeomNarrow = 0, kGeomWide = 1 };
template <int GEOM> struct PfGeom {
  static constexpr int kThreads = GEOM == kGeomNarrow ? 1024 : 512;
  static constexpr int kWarps = kThreads / 32;
  static constexpr int kGroups = GEOM == kGeomNarrow ? 2 : 4;  // 16-byte groups per lane and step
  static constexpr int kTile = kGroups * 512;           // haystack bytes per warp step
  static constexpr int kStageBytes = kTile + 16;        // + fingerprint look-ahead
  static constexpr int kMinCtas = GEOM == kGeomWide ? 2 : 1;
  // Bloom bitmap size: a compile-time constant, so that the byte index (hash >> shift) and the
  // shared-memory base fold into one address instruction
  static constexpr uint32_t kLogBits = GEOM == kGeomWide ? kWideLogBits : kNarrowLogBits;
};
// per-warp queue sizes: first-probe hits of one step handled by the compacted second probe, and
// verified-candidate entries (the dense variant stores 8-byte entries, so fewer of them fit
// beside the 128 KiB bitmap)
template <bool DENSE> struct PfCfg {
  static constexpr int kSlots = 256;
  static constexpr int kQ2 = DENSE ? 64 : 96;
};

// Queued offsets are 32-bit, inside a window of 2^kWinShift bytes of the chunk (prefilter_kernel).
// The dry run can shrink the window (ACB_EMU_WINSHIFT) so that small inputs cross many of them.
#ifdef ACB_EMULATE
static const uint32_t kWinShift = getenv("ACB_EMU_WINSHIFT") ? (uint32_t)atoi(getenv("ACB_EMU_WINSHIFT")) : 31u;
#else
constexpr uint32_t kWinShift = 31;
#endif

constexpr int kPfStages = 2;            // ring depth per warp (TMA bulk copies + mbarriers, acb_ptx.cuh)

// The haystack bytes one warp step probes before it compacts their hits.  Stride 2 on the narrow
// geometry takes 2 KiB per step -- both 1 KiB halves of the warp's ring, filled by one bulk copy --
// so that each lane collects 32 hit bits, as the wide geometry does: the ballots, syncs and loop
// set-up of the hit path, the tile draw and the copy issue are paid once per 2 KiB instead of once
// per KiB.  The ring is then a single stage (the warp waits for its next 2 KiB, the other 31 warps
// of the SM issue meanwhile).  Stride 1 has 32 hit bits per lane with 1 KiB already.
template <int GEOM, int STRIDE> struct PfPass {
  static constexpr bool kPair = STRIDE == 2 && GEOM == kGeomNarrow;
  static constexpr int kStages = kPair ? 1 : kPfStages;               // ring stages in use
  static constexpr int kGroups = PfGeom<GEOM>::kGroups * (kPair ? 2 : 1);  // 16-byte groups per lane and step
  static constexpr int kTile = kGroups * 512;                           // haystack bytes per warp step
  static_assert(kStages * (kTile + 16) <= kPfStages * PfGeom<GEOM>::kStageBytes, "a step's tiles fit the warp's ring");
};

template <bool BUCKETED = true>  // false: the single list only (kernels that never bucket)
struct Emitter {
  uint64_t* g_keys;
  uint32_t* g_pids;
  unsigned long long* g_counter;
  uint64_t cap;
  uint32_t bucket_shift, bucket_log;  // see PrefilterLaunch
  uint64_t bucket_slots;
  // Matches are sparse (about one per 4 KiB in the BASELINE workloads) while candidates are
  // verified by whole warps, so lanes that found something aggregate their append into one
  // atomic per warp step (warp-ballot + warp-aggregated atomic).
  // Bucketed: the append goes to the bucket of the key's offset, so that the order step only sorts
  // inside buckets (order_buckets_kernel).  A warp verifies offsets that lie close together, so its
  // lanes nearly always share the bucket and keep the single atomic; lanes of different buckets
  // append one by one.  A full bucket sends the tuple to the overflow list (never dropped; the order
  // step then falls back to the radix sort of everything).
  __device__ __forceinline__ void emit(uint64_t key, uint32_t pid) {
    const unsigned m = __activemask();
    const int leader = __ffs(m) - 1;
    const int lane = threadIdx.x & 31;
    const bool bucketed = BUCKETED && bucket_shift != 0;
    unsigned long long* cnt = g_counter;
    uint64_t first = 0;  // the bucket's first slot
    bool together = true;
    if (bucketed) {
      const uint32_t b = (uint32_t)(key >> (kTieBits + bucket_shift));
      cnt += kBucketCountersAt + b;
      first = (uint64_t)b << bucket_log;
      together = __ballot_sync(m, b == (uint32_t)__shfl_sync(m, b, leader)) == m;
    }
    unsigned long long g;
    if (together) {
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(cnt, (unsigned long long)__popc(m));
      base = __shfl_sync(m, base, leader);
      g = base + __popc(m & ((1u << lane) - 1));
    } else {
      g = atomicAdd(cnt, 1ull);
    }
    uint64_t slot = first + g;
    if (bucketed && g >> bucket_log) slot = bucket_slots + atomicAdd(g_counter, 1ull);
    if (slot < cap) { g_keys[slot] = key; g_pids[slot] = pid; }
  }
};

// Anchor-map lookup (acb_fingerprint.cuh): the state reached from the start state by `key`, the raw
// first k bytes at an offset; 0 if those bytes are not the beginning of any pattern.
__device__ __forceinline__ uint32_t anchor_lookup_key(const DfaDev& d, uint32_t key) {
  uint32_t slot = amap_slot(key, d.amap_shift);
  for (;;) {
    const uint2 e = __ldg(d.amap + slot);
    if (e.y == 0 || e.x == key) return e.y;
    slot = amap_next(slot, d.amap_mask);
  }
}

// The same lookup for the k bytes at haystack offset `s`.
__device__ __forceinline__ uint32_t anchor_lookup(const DfaDev& d, const PrefilterLaunch& p, uint64_t s) {
  if (s + d.amap_k > p.span_end) return 0;  // no pattern fits any more
  // the k bytes at s: two aligned word loads when both words lie inside the haystack buffer,
  // byte loads within a word of its edges (nothing outside [hay, hay + hay_len) is ever read)
  const uintptr_t a = reinterpret_cast<uintptr_t>(p.hay + s);
  const uintptr_t lo_edge = reinterpret_cast<uintptr_t>(p.hay), hi_edge = lo_edge + p.hay_len;
  const uintptr_t wa = a & ~uintptr_t(3);
  uint32_t key;
  if (wa >= lo_edge && wa + ((a & 3) ? 8 : 4) <= hi_edge) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(wa);
    const uint32_t lo = __ldg(w);
    const uint32_t hi = (a & 3) ? __ldg(w + 1) : 0u;
    key = __funnelshift_r(lo, hi, (uint32_t)(a & 3) * 8) & d.amap_kmask;
  } else {
    key = 0;
    for (uint32_t i = 0; i < d.amap_k; ++i) key |= (uint32_t)__ldg(p.hay + s + i) << (8 * i);
  }
  return anchor_lookup_key(d, key);
}

// Batched search: the end of the document that contains start offset s, i.e. doc_offsets[i] for the
// first i with doc_offsets[i] > s (the span is [doc_offsets[0], doc_offsets[n_docs]), so i exists).
// Only candidates that reach a match state pay for it.  (Out of line, the call makes ptxas spill
// around it in every prefilter_kernel instantiation.)
__device__ __forceinline__ uint64_t doc_end_of(const uint64_t* __restrict__ offs, uint64_t n_docs, uint64_t s) {
  uint64_t lo = 1, hi = n_docs;  // answer in [1, n_docs]
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(offs + mid) > s) hi = mid; else lo = mid + 1;
  }
  return __ldg(offs + lo);
}

// Verify one candidate start offset `s` (K3b): walk the shipped DFA while the state stays on the
// trie path anchored at s (depth == bytes consumed), starting from state `sid` at depth `j`
// (the start state, or the state the anchor map gave for the first j bytes).
// Batched search (p.doc_offsets): a match must end inside the document s lies in; the walk stops at
// the first match state past that end (any longer match ends later still).  The end is looked up at
// each match state the walk reaches (most candidates that match reach one).
template <int MODE, class EM>
__device__ __forceinline__ void verify_from(const DfaDev& d, const PrefilterLaunch& p, const uint8_t* s_cls,
                                            uint64_t s, uint32_t sid, uint32_t j, EM& em) {
  const uint8_t* __restrict__ hay = p.hay;
  const uint32_t* __restrict__ trans = d.trans;
  uint64_t pos = s + j;
  uint32_t best_pid = 0, best_len = 0;
  bool entered = j != 0;  // the anchor state may itself hold patterns of length j
  for (;;) {
    if (!entered) {
      if (pos >= p.span_end) break;
      const uint32_t b = __ldg(hay + pos);
      sid = __ldg(trans + sid + s_cls[b]);
      ++j;
      ++pos;
      if (sid == 0) break;  // DEAD (leftmost automata): nothing longer can start at s
      if (__ldg(d.depth16 + (sid >> d.stride2)) != j) break;  // left the trie path anchored at s
    }
    entered = false;
    if (sid <= d.max_match_id) {
      // (no end cached across the loop: a live 64-bit value there costs the single-haystack scans)
      if (p.doc_offsets != nullptr && pos > doc_end_of(p.doc_offsets, p.n_docs, s)) break;
      const uint32_t row = sid >> d.stride2;
      const uint32_t lo = __ldg(d.match_offsets + row - 2), hi = __ldg(d.match_offsets + row - 1);
      if (MODE == 0) {
        // the node's own patterns come first in its list and all have length j
        for (uint32_t i = lo; i < hi; ++i) {
          const uint32_t pid = __ldg(d.match_pids + i);
          if (__ldg(d.pattern_lens + pid) != j) break;
          if (p.first_only && i > lo) break;  // duplicates of one pattern: the iterator can only yield the first
          const uint64_t tie = ((uint64_t)(d.max_pattern_len - j) << p.dup_shift) | (uint64_t)(i - lo);
          em.emit(((pos - p.span_start) << kTieBits) | tie, pid);
        }
      } else {
        const uint32_t pid = __ldg(d.match_pids + lo);
        if (__ldg(d.pattern_lens + pid) == j) { best_pid = pid; best_len = j; }
      }
    }
  }
  if (MODE == 1 && best_len) em.emit(((s - p.span_start) << kTieBits) | best_len, best_pid);
}

template <int MODE, class EM>
__device__ __forceinline__ void verify_at(const DfaDev& d, const PrefilterLaunch& p, const uint8_t* s_cls,
                                          uint64_t s, EM& em) {
  if (d.amap != nullptr) {
    const uint32_t sid = anchor_lookup(d, p, s);
    if (sid != 0) verify_from<MODE>(d, p, s_cls, s, sid, d.amap_k, em);
  } else {
    verify_from<MODE>(d, p, s_cls, s, d.start_unanchored_id, 0, em);
  }
}

// Bloom probe of a 32-bit hash, bloom_bit(h, h, SHIFT): the byte comes from the top (log_bits-3)
// bits, the bit inside the byte from the low 3 bits.  The probe loads that byte, replicates it
// into all four byte lanes with a multiply (FMA pipe) and rotates by the raw hash (the hardware
// uses the shift amount mod 32), which puts bit (h & 7) of the byte at bit 0 -- one shift, one
// byte load, one multiply and one rotate per position, no masking.
template <uint32_t SHIFT>
__device__ __forceinline__ bool bloom_test(const uint32_t* s_bitmap, uint32_t h) {
  const uint32_t byte = reinterpret_cast<const uint8_t*>(s_bitmap)[h >> SHIFT];
  const uint32_t rep = byte * 0x01010101u;  // the rotate below then finds bit (h & 7) at bit 0
  return (__funnelshift_r(rep, rep, h) & 1u) != 0;
}

// One CTA owns a contiguous chunk of the filter region; each warp streams 512 B of it per step
// (a 1 KiB tile staged in shared memory by a TMA bulk copy, double buffered per warp) and probes
// the k-gram Bloom bitmap once per position.  The hits of a step are compacted (lane t takes hit
// t), re-probed with the second Bloom hash out of the staged tile, and the survivors go to a
// per-warp queue that
// is verified 32 at a time, so the dependent DFA walks always run with full warps.  There is no
// block-wide barrier in the steady state: a warp waiting on a verification overlaps with the
// other warps' fingerprint work.
// Second stage: compacted (hit, start offset) items, one per lane.  Stride 1 / stride 2: tested with
// one / two more Bloom hashes of the 4-byte fingerprint in the shared-memory bitmap.  DENSE: looked up
// in the anchor map (exact: one L2 access tells whether the k bytes begin a pattern and at which
// trie state), two items per lane in flight.
// (Tried and dropped: a lane-local second stage without compaction, a paired one, and the
// anchor-map second stage for the stride-2 kernel -- slower on cfg 2, the L2 latency outweighs the
// sparser bitmap.)
// Tile distribution DYN:
//   0  static: warp w of a CTA takes the tiles w, w + W, w + 2W, ... of the CTA's chunk.  The
//      scheduler favours some warps, nothing hands their neighbours' work over, and the kernel ends
//      with its slowest warp.
//   1  (default) the warps of a CTA draw tiles of the CTA's chunk from a shared-memory counter, four
//      per atomic: faster than the static split on cfg 2, cfg 3 and cfg 5.
//   2  tiles numbered over the whole region, super-tiles of 256 per CTA from a global counter
//      (prefetched half-way through the current one), batches of four per warp from a 64-bit
//      shared-memory word.  A CTA that starts late or shares its SM with another kernel simply ends
//      up with fewer super-tiles -- meant for the pipelined multi-GPU steps -- but the heavier draw
//      costs what the better balance wins: on cfg 2 it is slower than (1) and no faster than (0).
//      Kept selectable (ACG_EXP_GLOBAL_TILES).
template <int MODE, bool MASKED, bool DENSE, int STRIDE, int GEOM, int DYN = 0>
__global__ void __launch_bounds__(PfGeom<GEOM>::kThreads, PfGeom<GEOM>::kMinCtas)  // wide: two CTAs per SM (64 registers)
prefilter_kernel(DfaDev d, PrefilterLaunch p) {
  static_assert(STRIDE == 1 || STRIDE == 2, "fingerprint stride");
  static_assert(GEOM == kGeomNarrow || STRIDE == 2, "the 2 KiB tile needs the stride-2 first stage (32 hit bits per lane)");
  constexpr bool ANCH = DENSE;  // second stage = anchor-map lookup, queue entries carry the trie state
  constexpr int kPfThreads = PfGeom<GEOM>::kThreads;
  constexpr int kPfWarps = PfGeom<GEOM>::kWarps;
  constexpr int kRingBytes = kPfStages * PfGeom<GEOM>::kStageBytes;  // per warp
  constexpr int kStages = PfPass<GEOM, STRIDE>::kStages;
  constexpr int kPfTile = PfPass<GEOM, STRIDE>::kTile;
  constexpr int kPfStageBytes = kPfTile + 16;  // + fingerprint look-ahead
  constexpr int kGroups = PfPass<GEOM, STRIDE>::kGroups;
  constexpr int kPfSlots = PfCfg<DENSE>::kSlots;
  constexpr int kPfQ2 = PfCfg<ANCH>::kQ2;
  constexpr uint32_t kBloomShift = bloom_shift(PfGeom<GEOM>::kLogBits);
  using Q2Entry = typename std::conditional<ANCH, uint2, uint32_t>::type;  // (offset[, trie state of its first k bytes])
  ACB_DYNAMIC_SMEM(smem_raw);
  unsigned char* s_ring = smem_raw;                                    // [kPfWarps][kRingBytes]
  uint64_t* s_bars = reinterpret_cast<uint64_t*>(s_ring + kPfWarps * kRingBytes);  // [kPfWarps][kPfStages]
  uint32_t* s_tile_of = reinterpret_cast<uint32_t*>(s_bars + kPfWarps * kPfStages);  // DYN: tile number staged in [warp][stage]
  uint32_t* s_next_tile = s_tile_of + kPfWarps * kPfStages;                        // DYN: draw state (u64), prefetched super-tile (u32), pad
  Q2Entry* s_queue2 = reinterpret_cast<Q2Entry*>(s_next_tile + 4);  // [kPfWarps][kPfQ2]
  uint16_t* s_slots = reinterpret_cast<uint16_t*>(s_queue2 + kPfWarps * kPfQ2);  // [kPfWarps][kPfSlots]
  uint32_t* s_bitmap = reinterpret_cast<uint32_t*>(s_slots + kPfWarps * kPfSlots);
  __shared__ uint8_t s_cls[256];

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const uint32_t bitmap_words = p.brute ? 0u : (1u << (p.log_bits - 5));
  for (uint32_t i = tid; i < bitmap_words; i += kPfThreads) s_bitmap[i] = p.bitmap[i];
  if (tid < 256) s_cls[tid] = d.classes[tid];
  if (tid < kPfWarps * kPfStages) ptx::mbar_init(ptx::smem_addr(&s_bars[tid]), 1);
  // DYN draw state (64 bits at s_next_tile): this CTA starts with super-tile blockIdx.x; whether that
  // one exists is checked when the first batch is drawn (tiles >= n_tiles are skipped)
  if (tid == 0) {
    *reinterpret_cast<uint64_t*>(s_next_tile) = DYN == 2 ? (uint64_t)blockIdx.x << 32 : 0ull;  // (DYN 1: a 32-bit tile counter)
    s_next_tile[2] = 0xFFFFFFFEu;  // no super-tile prefetched yet
  }
  ptx::mbar_init_fence();
  ptx::fence_proxy_async();
  __syncthreads();

  // (the global super-tile distribution keeps the single list, see plan_buckets in acb_api.cu)
  Emitter<DYN != 2> em{p.keys, p.pids, p.counter, p.cap, p.bucket_shift, p.bucket_log, p.bucket_slots};
  unsigned long long cand_total = 0;

  // head / tail positions outside the aligned filter region are unconditional candidates
  // (with stride 2 the last probe of the region is at region_hi-2 and covers the starts
  // region_hi-3 and region_hi-2, so region_hi-1 joins the tail)
  if (blockIdx.x == 0) {
    const uint64_t tail_lo = (p.region_hi > p.region_lo && !p.brute) ? p.region_hi - (STRIDE - 1) : p.region_hi;
    const uint64_t head_n = p.region_lo - p.scan_lo;
    const uint64_t tail_n = p.scan_hi > tail_lo ? p.scan_hi - tail_lo : 0;
    for (uint64_t i = tid; i < head_n + tail_n; i += kPfThreads) {
      const uint64_t s = i < head_n ? p.scan_lo + i : tail_lo + (i - head_n);
      verify_at<MODE>(d, p, s_cls, s, em);
    }
  }

  // The chunk of the span this CTA's tile numbers refer to.  Static split: a contiguous 1/gridDim of
  // the region, in units of 16-byte blocks (the brute-force path always takes it).  DYN 2: the whole
  // region -- tiles are handed out globally -- known at compile time, so that its bounds stay launch
  // parameters instead of registers.
  const uint64_t n_blocks16 = (p.region_hi - p.region_lo) >> 4;
  const uint64_t per_cta = (n_blocks16 + gridDim.x - 1) / gridDim.x;
  const uint64_t b0 = (uint64_t)blockIdx.x * per_cta;
  const uint64_t b1 = min(b0 + per_cta, n_blocks16);
  const uint64_t split_lo = p.region_lo + (b0 << 4);
  const uint64_t split_hi = b0 < b1 ? p.region_lo + (b1 << 4) : split_lo;

  if (p.brute) {
    for (uint64_t s = split_lo + tid; s < split_hi; s += kPfThreads) verify_at<MODE>(d, p, s_cls, s, em);
    if (tid == 0 && split_hi > split_lo) atomicAdd(p.counter + 1, (unsigned long long)(split_hi - split_lo));
    return;
  }
  constexpr bool whole = DYN == 2;
  const uint64_t chunk_lo = whole ? p.region_lo : split_lo;
  const uint64_t chunk_hi = whole ? p.region_hi : split_hi;

  const uint32_t kmask = p.kmask, fold = p.fold, mult = p.mult;
  const uint32_t fold1 = p.fold & 0x00FFFFFFu;  // stride 2: the first stage fingerprints 3 bytes
  // stride 2: multiplying by (mult3 << 8) drops the window's fourth byte for free; the bit inside
  // the bitmap byte then comes from the fingerprint's own low bits (the product's are zero)
  const uint32_t mult8 = key_mult(p.mult3, p.key_shift);  // 8: 24-bit keys; 5: 27-bit keys (default)
  // queue offsets are relative to chunk_base: a stride-2 probe at the first byte of the chunk
  // also owns the start one byte before it
  // (unsigned arithmetic: for chunk_lo == 0 the base wraps to 2^64 - 1 and base + rel, rel >= 1, is the
  // offset again; rel == 0 -- the byte before the region -- is never queued, the head owns it)
  const uint64_t chunk_base = chunk_lo - (uint64_t)(STRIDE - 1);
  const uint32_t rel_bias = (uint32_t)(STRIDE - 1);
  const uint8_t* s_bytes = reinterpret_cast<const uint8_t*>(s_bitmap);
  unsigned char* ring = s_ring + warp * kRingBytes;
  uint64_t* bars = s_bars + warp * kPfStages;
  uint16_t* slots = s_slots + warp * kPfSlots;
  Q2Entry* q2 = s_queue2 + warp * kPfQ2;
  uint32_t q2len = 0;  // warp-uniform
  // queued offsets are 32-bit, relative to chunk_base + (q2win << kWinShift): a warp's tiles only
  // move forward, so the queue is drained when a tile lies in the next 2 GiB window of the chunk
  uint32_t q2win = 0;  // warp-uniform

  auto drain2 = [&]() {  // verify the queued survivors (K3b), one per lane
    __syncwarp();
    const uint64_t win_base = chunk_base + ((uint64_t)q2win << kWinShift);
    for (uint32_t i = lane; i < q2len; i += 32) {
      if constexpr (ANCH) {
        // (offset, trie state of its first k bytes): the anchor map was consulted when the entry was queued
        const uint2 e = q2[i];
        if (e.y != 0) verify_from<MODE>(d, p, s_cls, win_base + e.x, e.y, d.amap_k, em);
        else verify_at<MODE>(d, p, s_cls, win_base + e.x, em);
      } else {
        verify_at<MODE>(d, p, s_cls, win_base + q2[i], em);
      }
    }
    cand_total += q2len;
    q2len = 0;
    __syncwarp();
  };

  // ---- K3 main loop.  Each warp streams its share of the chunk through a two-stage ring of
  // tiles (+16 B look-ahead) filled by TMA bulk copies (cp.async.bulk, completion on an
  // mbarrier): no load instructions or address arithmetic per lane, and the next tile is in
  // flight while the current one is probed.  Lane L owns the 16-byte groups at tile offsets
  // g*512 + 16L, so its 16-byte shared-memory reads are conflict free.
  // Tile t of the chunk covers [chunk_lo + t * kPfTile, + kPfTile) cut at chunk_hi; only the last
  // tile can be short.  Static split: step i of warp w handles tile w + i * kPfWarps.
  const uint64_t chunk_bytes = chunk_hi - chunk_lo;
  const uint32_t n_tiles = (uint32_t)((chunk_bytes + kPfTile - 1) / kPfTile);
  const uint32_t last_valid = n_tiles ? (uint32_t)(chunk_bytes - (uint64_t)(n_tiles - 1) * kPfTile) : 0;
  const bool use_windows = (chunk_bytes >> kWinShift) != 0;  // queued 32-bit offsets need more than one window
  // shared addresses of this warp's barriers and ring, and of the lane's first 16-byte group;
  // opaque to the compiler so that they stay in registers instead of being re-derived from the
  // thread index at every use
  uint32_t bar0 = ptx::smem_addr(bars), ring0 = ptx::smem_addr(ring), lane0 = ring0 + (uint32_t)lane * 16u;
  ptx::keep_in_registers(bar0, ring0, lane0);
  // Refilling a stage needs no proxy fence: every lane has consumed its shared-memory reads of the
  // tile (their values fed the probes) before the __syncwarp that precedes the copy.
  const uint8_t* chunk_src = p.hay + chunk_lo;
  // Lane 0 copies tile t into `stage` and asks L2 for t_next, the tile of the warp's next copy (if
  // known and inside the chunk; no shared memory, only bytes the kernel reads anyway): the copy of t_next
  // then reads L2 instead of waiting a DRAM round trip.  In flight at any time: one tile per warp,
  // 132 x 32 x 2 KiB = 8.6 MB of L2 on an H100 for the stride-2 kernel.  Not in the dense variant:
  // its second stage and verifier live on the anchor map and table in L2, and the prefetch cost it
  // 1.4 % on cfg 5.  (The dry run has no L2.)
  constexpr bool kPrefetch = !DENSE;
  auto issue = [&](uint32_t t, uint32_t stage, uint32_t t_next) {  // lane 0 only; t < n_tiles
    const uint32_t bytes = (t + 1 < n_tiles ? (uint32_t)kPfTile : last_valid) + 16;
    const uint32_t bar = bar0 + stage * 8, dst = ring0 + stage * kPfStageBytes;
    ptx::mbar_arrive_expect_tx(bar, bytes);
    ptx::tma_load_1d(dst, chunk_src + (uint64_t)t * kPfTile, bytes, bar);
#ifndef ACB_EMULATE
    if (kPrefetch && t_next < n_tiles)
      ptx::bulk_prefetch_l2(chunk_src + (uint64_t)t_next * kPfTile, (t_next + 1 < n_tiles ? (uint32_t)kPfTile : last_valid) + 16);
#else
    (void)t_next;
#endif
  };
  // DYN: tiles are numbered over the whole region and handed out on two levels.  A CTA holds one
  // super-tile of kSuper consecutive tiles at a time (shared 64-bit state: super-tile index | next
  // offset inside it) and takes the next one from a global counter when it runs out; lane 0 of a warp
  // draws kDrawBatch consecutive tiles per shared-memory atomic.  A CTA that starts late, or shares
  // its SM with another kernel, simply ends up with fewer super-tiles: no second wave, no straggler.
  // The tile number for a stage is left in s_tile_of[warp][stage] for the warp to read when it gets
  // to that stage.
  constexpr uint32_t kDrawBatch = 4, kSuper = 256;
  static_assert(kSuper % (2 * kDrawBatch) == 0, "batches never straddle a super-tile or its half-way mark");
  uint32_t* tile_of = s_tile_of + warp * kPfStages;
  const uint32_t draw_a = ptx::smem_addr(s_next_tile), next_a = draw_a + 8;
  const uint32_t n_super = (n_tiles + kSuper - 1) / kSuper;
  constexpr uint64_t kNoMore = 0xFFFFFFFFull << 32;
  constexpr uint32_t kUnpublished = 0xFFFFFFFEu, kNone = 0xFFFFFFFFu;
  uint32_t batch_next = 0, batch_left = 0;  // lane 0's current batch
  bool exhausted = false;
  // The global fetch-and-add for the CTA's next super-tile is issued half-way through the current
  // one by whichever warp draws that batch, and its result is only looked at one step later, when
  // that warp publishes it in shared memory: the ~1 us round trip to L2 never stalls anybody.
  unsigned long long pend_g = 0;
  bool have_pend = false;
  auto publish = [&]() {  // lane 0 only
    if (have_pend) {
      ptx::sts32_volatile(next_a, pend_g < n_super ? (uint32_t)pend_g : kNone);
      have_pend = false;
    }
  };
  auto draw = [&](uint32_t stage) {  // lane 0 only
    if constexpr (DYN == 1) {
      // tiles of this CTA's chunk from the CTA's counter, kDrawBatch per atomic
      // (with the L2 prefetch the next batch is drawn with the last tile of the current one, so that
      // the tile after t is always known)
      if (batch_left == 0) {
        batch_next = ptx::atoms_add(draw_a, kDrawBatch);
        batch_left = kDrawBatch;
      }
      const uint32_t t = batch_next++;
      if (--batch_left == 0 && kPrefetch) {
        batch_next = ptx::atoms_add(draw_a, kDrawBatch);
        batch_left = kDrawBatch;
      }
      tile_of[stage] = t;
      if (t < n_tiles) issue(t, stage, batch_next);
      return;
    }
    publish();
    while (batch_left == 0 && !exhausted) {
      const uint64_t v = ptx::atoms_add64(draw_a, kDrawBatch);
      const uint32_t sup = (uint32_t)(v >> 32), off = (uint32_t)v;
      if (sup == kNone) { exhausted = true; break; }
      if (off == kSuper / 2) { pend_g = atomicAdd(p.counter + 2, 1ull) + gridDim.x; have_pend = true; }
      if (off < kSuper) { batch_next = sup * kSuper + off; batch_left = kDrawBatch; break; }
      if (off == kSuper) {
        // the first draw past the end installs the prefetched super-tile (published long ago, normally)
        uint32_t g;
        while ((g = ptx::lds32_volatile(next_a)) == kUnpublished) {}
        ptx::sts32_volatile(next_a, kUnpublished);
        if (g != kNone) {
          ptx::atoms_exch64(draw_a, ((uint64_t)g << 32) | kDrawBatch);  // (this warp keeps the first batch)
          batch_next = g * kSuper;
          batch_left = kDrawBatch;
        } else {
          ptx::atoms_exch64(draw_a, kNoMore);
          exhausted = true;
        }
        break;
      }
      while ((uint32_t)(ptx::lds64_volatile(draw_a) >> 32) == sup) {}  // the install is under way
    }
    uint32_t t = n_tiles;
    if (!exhausted) { t = batch_next++; --batch_left; }
    tile_of[stage] = t;
    // prefetched only inside the current batch: the next one may need a super-tile install
    if (t < n_tiles) issue(t, stage, batch_left ? batch_next : n_tiles);
  };
  if (lane == 0) {
    if constexpr (DYN) {
      draw(0);
      if (kStages > 1) draw(1);
    } else {
      const uint32_t w = (uint32_t)warp, step = (uint32_t)kPfWarps;
      if (w < n_tiles) issue(w, 0, w + step);
      if (kStages > 1 && w + step < n_tiles) issue(w + step, 1, w + 2 * step);
    }
  }
  __syncwarp();
  constexpr int kBitsPerGroup = 16 / STRIDE;
  constexpr int kHitBits = kGroups * kBitsPerGroup;
  for (uint32_t it = 0;; ++it) {
    const uint32_t stage = kStages == 1 ? 0u : it & 1;
    const uint32_t parity = (kStages == 1 ? it : it >> 1) & 1;
    uint32_t t;
    if constexpr (DYN) t = *reinterpret_cast<volatile uint32_t*>(tile_of + stage);
    else t = (uint32_t)warp + it * (uint32_t)kPfWarps;
    if (t >= n_tiles) break;  // tile numbers only grow: nothing is in flight for this warp any more
    const uint64_t wbase = chunk_lo + (uint64_t)t * kPfTile;
    uint32_t win = 0;
    if (use_windows) {  // (a chunk below 2 GiB -- every CTA chunk of a span under 264 GiB on 132 SMs -- has one window)
      win = (uint32_t)(((uint64_t)t * kPfTile) >> kWinShift);
      if (win != q2win) {  // warp-uniform
        if (q2len) drain2();
        q2win = win;
      }
    }
    while (!ptx::mbar_try_wait(bar0 + stage * 8, parity)) {}
    const uint32_t stage_off = stage * (uint32_t)kPfStageBytes;
    const uint32_t tile_a = ring0 + stage_off;
    uint32_t wv[kGroups][5];
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
      const uint32_t ga = lane0 + stage_off + g * 512;
      const uint4 v = ptx::lds128(ga);
      wv[g][0] = v.x; wv[g][1] = v.y; wv[g][2] = v.z; wv[g][3] = v.w;
      wv[g][4] = ptx::lds32(ga + 16);  // look-ahead word behind the group
    }
    // hit mask of this lane, kBitsPerGroup bits per group.  Stride 1: bit 16g+o = offset o of
    // group g.  Stride 2: only even offsets are probed (3-byte fingerprints of the pattern bytes
    // [0,3) and [1,4): a pattern starting at an odd offset is caught by its second fingerprint at
    // the next even offset); bit 8g+i = offset 2i of group g.
    uint32_t mask = 0;
#define ACB_WIN(o, lo, hi) (((o) & 3) ? __funnelshift_r(lo, hi, ((o) & 3) * 8) : (lo))
#define ACB_PROBE(o, lo, hi)                                                                  \
  do {                                                                                        \
    uint32_t gm, h, sel;                                                                      \
    if constexpr (STRIDE == 2) {                                                              \
      gm = MASKED ? (ACB_WIN(o, lo, hi) | fold1) : ACB_WIN(o, lo, hi);                        \
      h = gm * mult8;                                                                         \
      sel = gm;                                                                               \
    } else {                                                                                  \
      gm = MASKED ? ((ACB_WIN(o, lo, hi) | fold) & kmask) : ACB_WIN(o, lo, hi);               \
      h = gm * mult;                                                                          \
      sel = h;                                                                                \
    }                                                                                         \
    if constexpr (DENSE) {                                                                    \
      /* blocked filter: one word per key (top bits of the product), two bits inside it (low    \
         bits of the product's high half) -- both tested with this one load; the rotates take    \
         their amounts mod 32, which are the bits dense_bit_a(ph) and dense_bit_b(ph) */         \
      const uint32_t ph = __umulhi(gm, mult);                                                  \
      const uint32_t bw = s_bitmap[dense_word(h, kBloomShift)];                                \
      mask = __funnelshift_r(mask, __funnelshift_r(bw, bw, ph) & __funnelshift_r(bw, bw, ph >> 5), 1); \
    } else {                                                                                  \
      const uint32_t rep = (uint32_t)s_bytes[h >> kBloomShift] * 0x01010101u;                 \
      mask = __funnelshift_r(mask, __funnelshift_r(rep, rep, sel), 1);                        \
    }                                                                                         \
  } while (0)
#pragma unroll
    for (int g = 0; g < kGroups; ++g) {
#pragma unroll
      for (int wi = 0; wi < 4; ++wi) {
        if constexpr (STRIDE == 1) {
          ACB_PROBE(0, wv[g][wi], wv[g][wi + 1]); ACB_PROBE(1, wv[g][wi], wv[g][wi + 1]);
          ACB_PROBE(2, wv[g][wi], wv[g][wi + 1]); ACB_PROBE(3, wv[g][wi], wv[g][wi + 1]);
        } else {
          ACB_PROBE(0, wv[g][wi], wv[g][wi + 1]); ACB_PROBE(2, wv[g][wi], wv[g][wi + 1]);
        }
      }
    }
#undef ACB_PROBE
#undef ACB_WIN
    // the probes were funnelled in from the top: move the first one down to bit 0
    if constexpr (kHitBits < 32) mask >>= (32 - kHitBits);
    if (t + 1 == n_tiles) {
      // the last tile may be short: drop the hit bits of groups behind its end
      uint32_t ok_bits = 0;
#pragma unroll
      for (int g = 0; g < kGroups; ++g)
        if ((uint32_t)(g * 512 + lane * 16) < last_valid) ok_bits |= (uint32_t)((1ull << kBitsPerGroup) - 1) << (g * kBitsPerGroup);
      mask &= ok_bits;
    }
    // tile offset of hit bit `b` of lane `ln`
    auto hit_offset = [&](uint32_t b, uint32_t ln) -> uint32_t {
      return (b / kBitsPerGroup) * 512 + ln * 16 + (b % kBitsPerGroup) * STRIDE;
    };
    // slot allocation for this step's first-probe hits without touching shared memory: the
    // per-lane counts (almost always < 8) are summed across the warp bit plane by bit plane with
    // ballots; a lane with more hits than the planes cover sends the step down the unselective path
    const uint32_t cnt = __popc(mask);
    const uint32_t lt = (1u << lane) - 1;
    constexpr int kPlanes = DENSE ? 4 : 3;  // per-lane hit counts the ballot prefix sum covers (dense: 32 probes per lane)
    uint32_t slot = 0, total = 0;
#pragma unroll
    for (int b = 0; b < kPlanes; ++b) {
      const uint32_t bl = __ballot_sync(0xffffffffu, (cnt >> b) & 1u);
      slot += __popc(bl & lt) << b;
      total += __popc(bl) << b;
    }
    if (__any_sync(0xffffffffu, (cnt >> kPlanes) != 0)) total = (uint32_t)kPfSlots + 1;
    if (total) {
      // the very first probe of the region has no start before it
      const bool region_first = (whole || blockIdx.x == 0) && t == 0;
      if (total > (uint32_t)kPfSlots) {
        // fingerprints not selective here: verify this step's hits in place
        uint32_t nver = 0;
        while (mask) {
          const int b = __ffs(mask) - 1;
          mask &= mask - 1;
          const uint64_t e = wbase + hit_offset((uint32_t)b, (uint32_t)lane);
#pragma unroll
          for (int j = 0; j < STRIDE; ++j)
            if (e >= p.region_lo + j) { verify_at<MODE>(d, p, s_cls, e - j, em); ++nver; }
        }
        cand_total += __reduce_add_sync(0xffffffffu, nver);
      } else {
        // hit t of the step is recorded as (lane << 5 | bit); the consumer decodes the offset
        {
          uint16_t* sp = slots + slot;
          const uint32_t tag = (uint32_t)lane << 5;
          while (mask) {
            const uint32_t b = (uint32_t)__ffs(mask) - 1;
            mask &= mask - 1;
            *sp++ = (uint16_t)(tag | b);
          }
        }
        __syncwarp();
        // second stage, compacted: the work items are (hit, start offset the hit owns) -- the
        // probed offset and, with stride 2, the one before it -- one per lane.  Each is tested
        // with two Bloom hashes of its 4-byte fingerprint, re-read from the staged tile.
        const uint32_t wrel = (use_windows ? (uint32_t)((wbase - chunk_lo) - ((uint64_t)win << kWinShift)) : (uint32_t)(wbase - chunk_lo)) + rel_bias;
        const uint32_t n_items = total * STRIDE;
        if constexpr (ANCH) {
          // Anchor-map second stage: the answer is an L2 access away, so every lane takes two items
          // per round and has both first probes of the table in flight before it looks at either.
          for (uint32_t base = 0; base < n_items; base += 64) {
            uint32_t rel2[2], key2[2], slot2[2], sid2[2];
            bool look[2], pass2[2];
            uint2 ent[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const uint32_t w = base + 32u * u + lane;
              const uint32_t j = STRIDE == 2 ? (w & 1u) : 0u;
              look[u] = false; pass2[u] = false; rel2[u] = 0; key2[u] = 0; slot2[u] = 0; sid2[u] = 0;
              ent[u] = make_uint2(0, 0);
              if (w < n_items) {
                const uint32_t raw = slots[STRIDE == 2 ? (w >> 1) : w];
                const uint32_t e = hit_offset(raw & 31u, raw >> 5);
                rel2[u] = wrel + e - j;
                if (STRIDE == 2 && e < j) {
                  // the start lies one byte before the tile (at most one item per step): the
                  // verifier decides -- unless it would fall before the filter region
                  pass2[u] = !region_first;
                } else if (d.amap == nullptr) {
                  pass2[u] = true;
                } else if (chunk_base + ((uint64_t)win << kWinShift) + rel2[u] + d.amap_k <= p.span_end) {
                  const uint32_t off = e - j;
                  const uint32_t sa = tile_a + (off & ~3u);
                  key2[u] = __funnelshift_r(ptx::lds32(sa), ptx::lds32(sa + 4), (off & 3) * 8) & d.amap_kmask;
                  slot2[u] = amap_slot(key2[u], d.amap_shift);
                  look[u] = true;
                }
              }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u)
              if (look[u]) ent[u] = __ldg(d.amap + slot2[u]);
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              if (look[u]) {
                while (ent[u].y != 0 && ent[u].x != key2[u]) {  // open addressing, empty slot = miss
                  slot2[u] = amap_next(slot2[u], d.amap_mask);
                  ent[u] = __ldg(d.amap + slot2[u]);
                }
                sid2[u] = ent[u].y;
                pass2[u] = sid2[u] != 0;
              }
              const uint32_t bal = __ballot_sync(0xffffffffu, pass2[u]);
              if (bal) {
                if (pass2[u]) q2[q2len + __popc(bal & lt)] = make_uint2(rel2[u], sid2[u]);
                q2len += __popc(bal);
                if (q2len > (uint32_t)(kPfQ2 - 32)) drain2();
              }
            }
          }
        } else
        for (uint32_t base = 0; base < n_items; base += 32) {
          const uint32_t w = base + lane;
          const uint32_t j = STRIDE == 2 ? (w & 1u) : 0u;
          bool pass = false;
          uint32_t e = 0;
          if (w < n_items) {
            const uint32_t raw = slots[STRIDE == 2 ? (w >> 1) : w];
            e = hit_offset(raw & 31u, raw >> 5);
            if (STRIDE == 2 && e < j) {
              // the start lies one byte before the tile (at most one item per step): no second
              // probe, the verifier decides -- unless it would fall before the filter region
              pass = !region_first;
            } else {
              const uint32_t off = e - j;
              const uint32_t sa = tile_a + (off & ~3u);
              uint32_t gram = __funnelshift_r(ptx::lds32(sa), ptx::lds32(sa + 4), (off & 3) * 8);
              if (MASKED) gram = (gram | fold) & kmask;
              // stride 2: the first stage saw only three of the four bytes, so the cheap
              // multiplicative hash of the whole fingerprint rejects most items before the mix
              if (STRIDE == 2) pass = bloom_test<kBloomShift>(s_bitmap, gram * mult) && bloom_test<kBloomShift>(s_bitmap, bloom_hash2(gram));
              else pass = bloom_test<kBloomShift>(s_bitmap, bloom_hash2(gram));
            }
          }
          const uint32_t bal = __ballot_sync(0xffffffffu, pass);
          if (bal) {
            if (pass) {
              const uint32_t rel = wrel + e - j;
              if constexpr (!ANCH) q2[q2len + __popc(bal & lt)] = rel;
            }
            q2len += __popc(bal);
            if (q2len > (uint32_t)(kPfQ2 - 32)) drain2();
          }
        }
      }
    }
    __syncwarp();  // every lane is done with this stage: refill it with the tile kStages steps ahead
    if (lane == 0) {
      if constexpr (DYN) draw(stage);
      else if (t + kStages * kPfWarps < n_tiles) issue(t + kStages * kPfWarps, stage, t + (kStages + 1) * kPfWarps);
    }
    if constexpr (DYN && kStages == 1) __syncwarp();  // the tile number just drawn is the next step's
  }
  if constexpr (DYN == 2) { if (lane == 0) publish(); }  // a prefetched super-tile index somebody may be waiting for
  if (q2len) drain2();
  if (lane == 0 && cand_total) atomicAdd(p.counter + 1, cand_total);  // cand_total is warp-uniform
}

// ---- byte-set scan: the memchr-class prefilters ------------------------------------------------
// The reference skips ahead with memchr / memchr2 / memchr3 over the patterns' start bytes or over
// up to three "rare" bytes with their largest offsets (src/util/prefilter.rs:665-731, 855-904, chosen
// by :163-305 for automata with at most three such bytes), and runs the automaton from each
// candidate.  The same first stage here is a streaming compare: every lane takes 16 bytes per step
// (one coalesced 512-byte load per warp), flags the bytes that equal a needle with three integer
// instructions per word and needle, and the flagged offsets -- widened to the start offsets
// [q - back, q] they can belong to -- go through the same per-warp queue and anchored DFA verifier
// (K3b) as the fingerprint prefilter's survivors.  No shared-memory table, no staging: the kernel is
// bound by the haystack read as long as the needles are as rare as the reference's heuristics assume.
constexpr int kBsThreads = 512;
constexpr int kBsWarps = kBsThreads / 32;
constexpr int kBsQueue = 128;  // queued start offsets per warp (8 bytes each)

template <int MODE>
__global__ void __launch_bounds__(kBsThreads, 2) bytescan_kernel(DfaDev d, PrefilterLaunch p) {
  __shared__ uint8_t s_cls[256];
  __shared__ uint64_t s_q[kBsWarps * kBsQueue];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 256) s_cls[tid] = d.classes[tid];
  __syncthreads();
  Emitter<> em{p.keys, p.pids, p.counter, p.cap, p.bucket_shift, p.bucket_log, p.bucket_slots};
  unsigned long long cand_total = 0;
  // head / tail positions outside the aligned region are unconditional candidates
  if (blockIdx.x == 0) {
    const uint64_t head_n = p.region_lo - p.scan_lo;
    const uint64_t tail_n = p.scan_hi > p.region_hi ? p.scan_hi - p.region_hi : 0;
    for (uint64_t i = tid; i < head_n + tail_n; i += kBsThreads)
      verify_at<MODE>(d, p, s_cls, i < head_n ? p.scan_lo + i : p.region_hi + (i - head_n), em);
  }
  uint64_t* q = s_q + warp * kBsQueue;
  uint32_t qlen = 0;  // warp-uniform
  auto drain = [&]() {
    __syncwarp();
    for (uint32_t i = lane; i < qlen; i += 32) verify_at<MODE>(d, p, s_cls, q[i], em);
    cand_total += qlen;
    qlen = 0;
    __syncwarp();
  };
  const uint32_t n_needles = p.bs_n;
  const uint32_t max_back = max(p.bs_back[0], max(p.bs_back[1], p.bs_back[2]));
  // A warp step covers `owned` lanes x 16 bytes of start offsets.  With offsets (rare bytes) the last
  // lane only supplies the look-ahead of lane 30, and the next step begins at its 16 bytes.
  const uint32_t owned_lanes = max_back ? 31u : 32u;
  const uint64_t step_bytes = (uint64_t)owned_lanes * 16;
  const uint64_t region_bytes = p.region_hi - p.region_lo;
  const uint64_t n_steps = (region_bytes + step_bytes - 1) / step_bytes;
  const uint32_t lt = (1u << lane) - 1;
  // bytes past the region's end belong to the tail (verified above); a look-ahead lane may read up
  // to 16 bytes behind region_hi, which enqueue_prefilter_range keeps readable
  const uint64_t load_end = p.region_hi + (max_back ? 16 : 0);
  auto load = [&](uint64_t base) -> uint4 {
    return base < load_end ? ptx::ld_nc_u4(p.hay + base) : make_uint4(0, 0, 0, 0);
  };
  auto process = [&](uint64_t base, const uint4& v) {
    const bool in_range = base < load_end;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    // Zero-byte test per word and needle: (x - 0x01..) & ~x & 0x80.. has bit 7 set in every byte of
    // x = word ^ needle that is zero (and possibly in the byte above a true hit: a spurious
    // candidate the verifier rejects, never a missed one).  Most steps have no needle in the warp's
    // 512 bytes at all: one vote and on to the next load.
    uint32_t zany = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (j >= (int)n_needles) break;
      const uint32_t needle = p.bs_needle[j];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t x = w[k] ^ needle;
        zany |= (x - 0x01010101u) & ~x & 0x80808080u;
      }
    }
    if (!__any_sync(0xffffffffu, zany != 0 && in_range)) return;
    // flagged bytes, one 16-bit mask per needle (bit i = byte i of the lane's 16)
    uint32_t cand = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (j >= (int)n_needles) break;
      const uint32_t needle = p.bs_needle[j];
      uint32_t m = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t x = w[k] ^ needle;
        const uint32_t z = (x - 0x01010101u) & ~x & 0x80808080u;
        m |= ((((z >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * k);  // gather the four flags
      }
      if (!in_range) m = 0;
      const uint32_t back = p.bs_back[j];
      if (back == 0) {
        cand |= m;
      } else {
        // start offsets [q - back, q] of a flag at q: the flags of the next 16 bytes count for the
        // last `back` offsets of this lane
        const uint32_t both = m | (__shfl_down_sync(0xffffffffu, m, 1) << 16);
        uint32_t smear = both;
        for (uint32_t sft = 1; sft <= back; ++sft) smear |= both >> sft;
        cand |= smear & 0xFFFFu;
      }
    }
    if (lane >= (int)owned_lanes || base >= p.region_hi) cand = 0;  // look-ahead only / the tail's offsets
    const uint32_t cnt = __popc(cand);
    if (__any_sync(0xffffffffu, cnt != 0)) {
      // warp-wide slot allocation by ballot bit planes (counts <= 16)
      uint32_t slot = 0, total = 0;
#pragma unroll
      for (int b = 0; b < 5; ++b) {
        const uint32_t bl = __ballot_sync(0xffffffffu, (cnt >> b) & 1u);
        slot += __popc(bl & lt) << b;
        total += __popc(bl) << b;
      }
      if (qlen + total > (uint32_t)kBsQueue) drain();
      if (total > (uint32_t)kBsQueue) {
        // needles everywhere (the reference would have retired such a prefilter): verify in place
        uint32_t c = cand, nver = 0;
        while (c) {
          const int bit = __ffs(c) - 1;
          c &= c - 1;
          verify_at<MODE>(d, p, s_cls, base + bit, em);
          ++nver;
        }
        cand_total += __reduce_add_sync(0xffffffffu, nver);
      } else {
        uint64_t* dst = q + qlen + slot;
        uint32_t c = cand;
        while (c) {
          const int bit = __ffs(c) - 1;
          c &= c - 1;
          *dst++ = base + bit;
        }
        qlen += total;
        if (qlen >= 64) drain();
      }
    }
  };
  // Software pipeline: the loads of the next two steps are issued before the current two are
  // examined, so every warp keeps 1-2 KiB in flight while it computes (the compare phase of a warp is
  // about as long as a DRAM round trip; without the prefetch half of the latency is exposed).
  const uint64_t stride = (uint64_t)gridDim.x * kBsWarps;
  auto base_of = [&](uint64_t st) { return p.region_lo + st * step_bytes + (uint64_t)lane * 16; };  // this lane's 16 bytes
  uint64_t st = (uint64_t)blockIdx.x * kBsWarps + warp;
  uint4 cur[2], nxt[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) cur[u] = st + u * stride < n_steps ? load(base_of(st + u * stride)) : make_uint4(0, 0, 0, 0);
  for (; st < n_steps; st += 2 * stride) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint64_t sn = st + (2 + u) * stride;
      nxt[u] = sn < n_steps ? load(base_of(sn)) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u)
      if (st + u * stride < n_steps) process(base_of(st + u * stride), cur[u]);
    cur[0] = nxt[0];
    cur[1] = nxt[1];
  }
  if (qlen) drain();
  if (lane == 0 && cand_total) atomicAdd(p.counter + 1, cand_total);
}

// ---- chain resolution ---------------------------------------------------------

__device__ __forceinline__ void tuple_span(const ChainLaunch& c, uint64_t i, uint64_t* s, uint64_t* e) {
  const uint64_t key = c.t.keys[i];
  if (c.mode == 1) {
    *s = key >> kTieBits;
    *e = *s + (key & kTieMask);
  } else {
    *e = key >> kTieBits;
    *s = *e - c.t.pattern_lens[c.t.pids[i]];
  }
}

__global__ void chain_ends_kernel(ChainLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.t.n) return;
  uint64_t s, e;
  tuple_span(c, i, &s, &e);
  c.scratch_end[i] = e;
}

// Entry j is an "anchor" when every earlier tuple ends at or before its start:
// the iterator's cursor is then <= start(j) whatever it did before, so j is
// yielded and the search restarts at end(j) (src/automaton.rs:927-935).  Each
// anchor's thread resolves the short run of mutually overlapping tuples after it.
__global__ void chain_select_kernel(ChainLaunch c) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.t.n) return;
  uint64_t s, e;
  tuple_span(c, i, &s, &e);
  if (i > 0 && c.scratch_end[i - 1] > s) return;  // not an anchor: an earlier anchor's thread decides
  c.flags[i] = 1;
  uint64_t cur_end = e;
  for (uint64_t j = i + 1; j < c.t.n; ++j) {
    uint64_t sj, ej;
    tuple_span(c, j, &sj, &ej);
    if (c.scratch_end[j - 1] <= sj) break;  // next anchor
    if (sj >= cur_end) { c.flags[j] = 1; cur_end = ej; } else c.flags[j] = 0;
  }
}

struct MaxOp {
  __device__ __forceinline__ uint64_t operator()(uint64_t a, uint64_t b) const { return a > b ? a : b; }
};

// ---- K4 on bucketed tuples ------------------------------------------------------------------------
// The prefilter kernels append every tuple to the bucket of its key's offset (Emitter), so the buckets
// are already in key order among themselves and only their insides need sorting: one CTA per bucket
// loads it into shared memory as 32-bit keys ((offset - bucket base) << tie_bits | tie: the bucket's
// range is planned to fit), sorts (key, 16-bit index) pairs by LSD radix with 8-bit digits, and stores
// the tuples in their unchanged 64-bit form at the bucket's prefix offset.  One pass: every warp ranks
// its own consecutive items (the lanes with the same digit found with eight ballots, a per-warp count
// per digit in shared memory), the (digit, warp) counts are scanned in that order, and every item is
// scattered to its digit's offset for its warp plus its rank -- stable, so the passes compose.
constexpr int kOrdThreads = 1024;
constexpr int kOrdWarps = kOrdThreads / 32;
constexpr int kOrdRounds = (int)kOrderCap / kOrdThreads;  // items per lane and pass at most
constexpr int kOrdBatch = 8;                               // global loads in flight per thread

__global__ void __launch_bounds__(kOrdThreads, 1) order_buckets_kernel(OrderLaunch o) {
  ACB_DYNAMIC_SMEM(smem_raw);
  const uint32_t cap = o.bucket_cap;
  uint32_t* ka = reinterpret_cast<uint32_t*>(smem_raw);  // [cap] x 2: keys, ping-pong
  uint32_t* kb = ka + cap;
  uint16_t* ia = reinterpret_cast<uint16_t*>(kb + cap);  // [cap] x 2: index of the tuple in the bucket
  uint16_t* ib = ia + cap;
  uint16_t* s_cnt = ib + cap;                            // [256 digits][kOrdWarps], then their exclusive scan
  uint32_t* s_sum = reinterpret_cast<uint32_t*>(s_cnt + 256 * kOrdWarps);  // [kOrdWarps]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t lt = (1u << lane) - 1;
  const uint32_t b = blockIdx.x;
  const uint32_t n = (uint32_t)o.bucket_count[b];
  if (n == 0) return;

  // output offset: the tuples of the buckets before this one
  uint32_t part = 0;
  for (uint32_t i = tid; i < b; i += kOrdThreads) part += (uint32_t)o.bucket_count[i];
  part = __reduce_add_sync(0xffffffffu, part);
  if (lane == 0) s_sum[warp] = part;
  __syncthreads();
  uint64_t out0 = 0;
  for (int w = 0; w < kOrdWarps; ++w) out0 += s_sum[w];

  const uint64_t in0 = (uint64_t)b * cap;
  const uint64_t off0 = (uint64_t)b << o.bucket_shift;
  const uint32_t tie_bits = o.tie_bits;
  const uint64_t tie_mask = (1ull << tie_bits) - 1;
  for (uint32_t j0 = 0; j0 < n; j0 += kOrdBatch * kOrdThreads) {
    uint64_t k[kOrdBatch];
#pragma unroll
    for (int u = 0; u < kOrdBatch; ++u) {
      const uint32_t j = j0 + u * kOrdThreads + tid;
      k[u] = j < n ? o.keys_in[in0 + j] : 0;
    }
#pragma unroll
    for (int u = 0; u < kOrdBatch; ++u) {
      const uint32_t j = j0 + u * kOrdThreads + tid;
      if (j < n) {
        ka[j] = (uint32_t)((((k[u] >> kTieBits) - off0) << tie_bits) | (k[u] & tie_mask));
        ia[j] = (uint16_t)j;
      }
    }
  }

  // warp w ranks the items [w_lo, w_hi), 32 per round
  const uint32_t per_warp = (n + kOrdWarps - 1) / kOrdWarps;
  const uint32_t w_lo = min(warp * per_warp, n), w_hi = min(w_lo + per_warp, n);
  const uint32_t rounds = (per_warp + 31) / 32;
  const uint32_t key_bits = o.bucket_shift + tie_bits;
  for (uint32_t sh = 0; sh < key_bits; sh += 8) {
    for (int i = tid; i < 256 * kOrdWarps / 2; i += kOrdThreads) reinterpret_cast<uint32_t*>(s_cnt)[i] = 0;
    __syncthreads();  // counts cleared, keys in place
    uint32_t rd[kOrdRounds];  // digit << 16 | rank among the warp's items of that digit
#pragma unroll
    for (int r = 0; r < kOrdRounds; ++r) {
      rd[r] = 0;
      if ((uint32_t)r < rounds) {  // warp-uniform
        const uint32_t i = w_lo + r * 32 + lane;
        const bool valid = i < w_hi;
        const uint32_t digit = valid ? (ka[i] >> sh) & 0xFFu : 0u;
        uint32_t peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
        for (int bit = 0; bit < 8; ++bit) {
          const uint32_t bb = __ballot_sync(0xffffffffu, (digit >> bit) & 1u);
          peers &= ((digit >> bit) & 1u) ? bb : ~bb;
        }
        uint16_t* c = s_cnt + digit * kOrdWarps + warp;
        const uint32_t base = valid ? *c : 0u;
        __syncwarp();
        if (valid && (peers & lt) == 0) *c = (uint16_t)(base + __popc(peers));
        __syncwarp();
        rd[r] = (digit << 16) | (base + __popc(peers & lt));
      }
    }
    __syncthreads();
    {  // exclusive scan of the counts in (digit, warp) order, 8 per thread
      constexpr int kPer = 256 * kOrdWarps / kOrdThreads;
      uint16_t* c = s_cnt + tid * kPer;
      uint32_t v[kPer], sum = 0;
#pragma unroll
      for (int u = 0; u < kPer; ++u) { v[u] = c[u]; sum += v[u]; }
      uint32_t incl = sum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t x = (uint32_t)__shfl_sync(0xffffffffu, incl, lane >= d ? lane - d : lane);
        if (lane >= d) incl += x;
      }
      if (lane == 31) s_sum[warp] = incl;
      __syncthreads();
      uint32_t run = incl - sum;
      for (int w = 0; w < warp; ++w) run += s_sum[w];
#pragma unroll
      for (int u = 0; u < kPer; ++u) { c[u] = (uint16_t)run; run += v[u]; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kOrdRounds; ++r) {
      const uint32_t i = w_lo + r * 32 + lane;
      if ((uint32_t)r < rounds && i < w_hi) {
        const uint32_t dst = s_cnt[(rd[r] >> 16) * kOrdWarps + warp] + (rd[r] & 0xFFFFu);
        kb[dst] = ka[i];
        ib[dst] = ia[i];
      }
    }
    __syncthreads();  // scattered; the counts may be cleared
    uint32_t* tk = ka; ka = kb; kb = tk;
    uint16_t* ti = ia; ia = ib; ib = ti;
  }

  for (uint32_t j0 = 0; j0 < n; j0 += kOrdBatch * kOrdThreads) {
    uint32_t pid[kOrdBatch];
#pragma unroll
    for (int u = 0; u < kOrdBatch; ++u) {
      const uint32_t j = j0 + u * kOrdThreads + tid;
      pid[u] = j < n ? o.pids_in[in0 + ia[j]] : 0u;
    }
#pragma unroll
    for (int u = 0; u < kOrdBatch; ++u) {
      const uint32_t j = j0 + u * kOrdThreads + tid;
      if (j < n) {
        const uint32_t sk = ka[j];
        o.keys_out[out0 + j] = ((off0 + (sk >> tie_bits)) << kTieBits) | (sk & tie_mask);
        o.pids_out[out0 + j] = pid[u];
      }
    }
  }
}

// Fallback of the order step (a bucket overflowed): CTA b < n_buckets copies bucket b, CTA n_buckets
// the overflow list, each to its prefix offset; the radix sort of the whole list follows.
constexpr int kCompactThreads = 256;
__global__ void __launch_bounds__(kCompactThreads) compact_buckets_kernel(OrderLaunch o) {
  __shared__ unsigned long long s_part[kCompactThreads];
  const uint32_t b = blockIdx.x;
  const int tid = threadIdx.x;
  unsigned long long part = 0;
  for (uint32_t i = tid; i < b && i < o.n_buckets; i += kCompactThreads) part += min(o.bucket_count[i], (unsigned long long)o.bucket_cap);
  s_part[tid] = part;
  __syncthreads();
  uint64_t dst = 0;
  for (int i = 0; i < kCompactThreads; ++i) dst += s_part[i];
  const uint64_t n = b < o.n_buckets ? min(o.bucket_count[b], (unsigned long long)o.bucket_cap) : *o.overflow_count;
  const uint64_t src = b < o.n_buckets ? (uint64_t)b * o.bucket_cap : o.bucket_slots;
  for (uint64_t j = tid; j < n; j += kCompactThreads) {
    o.keys_out[dst + j] = o.keys_in[src + j];
    o.pids_out[dst + j] = o.pids_in[src + j];
  }
}

}  // namespace

cudaError_t launch_prefilter(const DfaDev& dfa, const PrefilterLaunch& p, int sm_count, cudaStream_t s) {
  const bool dense = p.dense != 0;
  const int geom = p.stride == 2 ? p.geom : kGeomNarrow;
  if (geom < kGeomNarrow || geom > kGeomWide) return cudaErrorInvalidValue;
  const uint32_t want_log = geom == kGeomWide ? PfGeom<kGeomWide>::kLogBits : PfGeom<kGeomNarrow>::kLogBits;
  if (!p.brute && (p.log_bits != want_log || p.shift != bloom_shift(want_log))) return cudaErrorInvalidValue;
  const size_t bitmap_bytes = p.brute ? 0 : (size_t(1) << (p.log_bits - 3));
  static const int kThreadsOf[2] = {PfGeom<0>::kThreads, PfGeom<1>::kThreads};
  static const int kStageOf[2] = {PfGeom<0>::kStageBytes, PfGeom<1>::kStageBytes};
  const int threads = kThreadsOf[geom];
  const int warps = threads / 32;
  const int stage_bytes = kStageOf[geom];
  const int tile = geom == kGeomWide ? PfPass<kGeomWide, 2>::kTile
                   : p.stride == 2 ? PfPass<kGeomNarrow, 2>::kTile : PfPass<kGeomNarrow, 1>::kTile;  // bytes per warp step
  const int q2_bytes = dense ? PfCfg<true>::kQ2 * 8 : PfCfg<false>::kQ2 * 4;
  const int slot_bytes = PfCfg<false>::kSlots * 2;
  const size_t smem = size_t(warps) * (kPfStages * stage_bytes + kPfStages * 12 + q2_bytes + slot_bytes) + 16 + bitmap_bytes;
  if (smem > 227 * 1024 - 1024) return cudaErrorInvalidValue;  // static shared memory: byte classes, tile numbers
  const bool masked = p.fold != 0 || p.kmask != 0xFFFFFFFFu;
  using KernT = void (*)(DfaDev, PrefilterLaunch);
  // [mode][masked][dyn][variant]: 0 stride 1, 1 stride 1 + dense, 2 stride 2 narrow, 3 stride 2 wide
  // (stride 2 is never combined with the dense variant)
#define ACB_PF_ROW(M, K, D)                                                                                 \
  {prefilter_kernel<M, K, false, 1, kGeomNarrow, D>, prefilter_kernel<M, K, true, 1, kGeomNarrow, D>, \
   prefilter_kernel<M, K, false, 2, kGeomNarrow, D>, prefilter_kernel<M, K, false, 2, kGeomWide, D>}
  static const KernT table[2][2][3][4] = {
      {{ACB_PF_ROW(0, false, 0), ACB_PF_ROW(0, false, 1), ACB_PF_ROW(0, false, 2)},
       {ACB_PF_ROW(0, true, 0), ACB_PF_ROW(0, true, 1), ACB_PF_ROW(0, true, 2)}},
      {{ACB_PF_ROW(1, false, 0), ACB_PF_ROW(1, false, 1), ACB_PF_ROW(1, false, 2)},
       {ACB_PF_ROW(1, true, 0), ACB_PF_ROW(1, true, 1), ACB_PF_ROW(1, true, 2)}}};
#undef ACB_PF_ROW
  if (p.dyn > 2) return cudaErrorInvalidValue;
  if (p.stride == 2 && dense) return cudaErrorInvalidValue;
  int variant = dense ? 1 : 0;
  if (p.stride == 2) variant = geom == kGeomWide ? 3 : 2;
  KernT kern = table[p.mode ? 1 : 0][masked ? 1 : 0][p.dyn][variant];
#ifdef ACB_EMULATE
  if (getenv("ACB_EMU_TRACE")) fprintf(stderr, "launch_prefilter variant %d dyn %d threads %d smem %zu\n", variant, (int)p.dyn, threads, smem);
#endif
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int per_sm = 1;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) per_sm = 1;
  uint64_t grid = (uint64_t)sm_count * per_sm;
  const uint64_t cta_step = uint64_t(warps) * tile;
  const uint64_t warp_steps = ((p.region_hi - p.region_lo) + cta_step - 1) / cta_step;
  if (grid > warp_steps) grid = warp_steps ? warp_steps : 1;
  ACB_LAUNCH(kern, (unsigned)grid, threads, smem, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_bytescan(const DfaDev& dfa, const PrefilterLaunch& p, int sm_count, cudaStream_t s) {
  if (p.bs_n < 1 || p.bs_n > 3) return cudaErrorInvalidValue;
  for (uint32_t j = 0; j < 3; ++j)
    if (p.bs_back[j] > 15) return cudaErrorInvalidValue;
  uint64_t grid = (uint64_t)sm_count * 2;
  const uint64_t steps = ((p.region_hi - p.region_lo) + 16 * 31 - 1) / (16 * 31);
  const uint64_t ctas = (steps + kBsWarps - 1) / kBsWarps;
  if (grid > ctas) grid = ctas ? ctas : 1;
  if (p.mode) ACB_LAUNCH(bytescan_kernel<1>, (unsigned)grid, kBsThreads, 0, s, dfa, p);
  else ACB_LAUNCH(bytescan_kernel<0>, (unsigned)grid, kBsThreads, 0, s, dfa, p);
  return cudaGetLastError();
}

cudaError_t launch_chain_ends(const ChainLaunch& c, cudaStream_t s) {
  const unsigned blocks = (unsigned)((c.t.n + 255) / 256);
  ACB_LAUNCH(chain_ends_kernel, blocks, 256, 0, s, c);
  return cudaGetLastError();
}
cudaError_t launch_chain_select(const ChainLaunch& c, cudaStream_t s) {
  const unsigned blocks = (unsigned)((c.t.n + 255) / 256);
  ACB_LAUNCH(chain_select_kernel, blocks, 256, 0, s, c);
  return cudaGetLastError();
}
cudaError_t launch_order_buckets(const OrderLaunch& o, cudaStream_t s) {
  if (o.n_buckets == 0 || o.n_buckets > kMaxBuckets || o.bucket_cap == 0 || o.bucket_cap > kOrderCap ||
      o.bucket_shift + o.tie_bits > 32)
    return cudaErrorInvalidValue;
  const size_t smem = size_t(o.bucket_cap) * 12 + 256 * kOrdWarps * 2 + kOrdWarps * 4;
  cudaError_t e = cudaFuncSetAttribute(order_buckets_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  ACB_LAUNCH(order_buckets_kernel, o.n_buckets, kOrdThreads, smem, s, o);
  return cudaGetLastError();
}
cudaError_t launch_compact_buckets(const OrderLaunch& o, cudaStream_t s) {
  ACB_LAUNCH(compact_buckets_kernel, o.n_buckets + 1, kCompactThreads, 0, s, o);
  return cudaGetLastError();
}
cudaError_t scan_max_u64(void* d_temp,size_t& temp_bytes, uint64_t* data, uint64_t n, cudaStream_t s) {
  return cub::DeviceScan::InclusiveScan(d_temp, temp_bytes, data, data, MaxOp(), (int64_t)n, s);
}
cudaError_t select_flagged(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, const uint32_t* pids_in,
                           const uint8_t* flags, uint64_t* keys_out, uint32_t* pids_out,
                           unsigned long long* d_num_out, uint64_t n, cudaStream_t s) {
  size_t a = 0, b = 0;
  if (d_temp == nullptr) {
    cudaError_t e = cub::DeviceSelect::Flagged(nullptr, a, keys_in, flags, keys_out, d_num_out, (int64_t)n, s);
    if (e != cudaSuccess) return e;
    e = cub::DeviceSelect::Flagged(nullptr, b, pids_in, flags, pids_out, d_num_out, (int64_t)n, s);
    temp_bytes = a > b ? a : b;
    return e;
  }
  cudaError_t e = cub::DeviceSelect::Flagged(d_temp, temp_bytes, keys_in, flags, keys_out, d_num_out, (int64_t)n, s);
  if (e != cudaSuccess) return e;
  return cub::DeviceSelect::Flagged(d_temp, temp_bytes, pids_in, flags, pids_out, d_num_out, (int64_t)n, s);
}

}  // namespace acb
