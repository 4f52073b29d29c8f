// acb_fingerprint.cuh -- the prefilter's fingerprint format, one definition for the plan that lays the
// tables out on the host (acb_plan.hpp) and the kernels that probe them (acb_prefilter.cu).  nvcc compiles
// it for host and device; a plain C++ compiler (the dry run in tests/emu) as host code.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define ACB_FP_FN __host__ __device__ __forceinline__
#else
#define ACB_FP_FN inline
#endif

namespace acb {

// Bloom bitmap sizes: 2^20 bits (128 KiB) for the narrow kernel geometry, 2^17 bits (16 KiB) for the wide
// one, which is only chosen for small pattern sets and then leaves room for two CTAs per SM.
constexpr uint32_t kNarrowLogBits = 20, kWideLogBits = 17;
// A hash's byte in the bitmap is its top (log_bits - 3) bits: hash >> bloom_shift(log_bits).
ACB_FP_FN constexpr uint32_t bloom_shift(uint32_t log_bits) { return 35 - log_bits; }
// More fingerprints than this: the dense blocked filter instead of the two-probe Bloom filter.
constexpr uint64_t kDenseGrams = 8192;
// First Bloom hash of a fingerprint: gram * kMult, a single multiply for the per-position probe.
constexpr uint32_t kMult = 0x9E3779B1u;

// Second Bloom hash: a full avalanche mix (evaluated only for first-probe hits, so its cost is irrelevant).
ACB_FP_FN uint32_t bloom_hash2(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// The anchor map's hash.
ACB_FP_FN uint32_t bloom_hash3(uint32_t x) {
  x ^= x >> 15;
  x *= 0x2c1b3c6du;
  x ^= x >> 12;
  x *= 0x297a2d39u;
  x ^= x >> 15;
  return x;
}

// Bit index of hash `h` in the byte-addressed bitmap (little-endian words): the byte from the top bits of
// `h`, the bit inside it from the low 3 bits of `sel` -- `h` itself for a Bloom probe, the key for a
// stride-2 first-stage probe, whose hash window * key_mult(mult3, key_shift) has zero low bits.  The
// shifted multiplier drops the window's fourth byte (key_shift 8) or all of it but its low 3 bits (5).
ACB_FP_FN uint32_t bloom_bit(uint32_t h, uint32_t sel, uint32_t shift) { return (h >> shift) * 8 + (sel & 7); }
ACB_FP_FN uint32_t key_mult(uint32_t mult3, uint32_t key_shift) { return mult3 << key_shift; }

// Dense blocked filter: a fingerprint owns one 32-bit word, picked by the top bits of the low half `lo` of
// gram * kMult, and two bits inside it, picked by the high half `hi`.
ACB_FP_FN uint32_t dense_word(uint32_t lo, uint32_t shift) { return lo >> (shift + 2); }
ACB_FP_FN uint32_t dense_bit_a(uint32_t hi) { return hi & 31; }
ACB_FP_FN uint32_t dense_bit_b(uint32_t hi) { return (hi >> 5) & 31; }

ACB_FP_FN int bit_width(uint64_t v) { int b = 0; for (; v; v >>= 1) ++b; return b; }

// Anchor map: 2^amap_log slots (at least 16) of (key, premultiplied state id), a 64-bit word with the key in its low
// half (a uint2 on the device); id 0 marks an empty slot.  A key's home slot is the top amap_log bits of
// its hash (amap_shift = 32 - amap_log), a lookup walks on slot by slot to the key or an empty slot.  The
// load factor stays at or below 1/4: a lookup of a key that is not there (the common case) ends at the
// first slot three times out of four, and every further slot is another dependent L2 access.
ACB_FP_FN uint32_t amap_log_for(uint64_t n_keys) { return uint32_t(bit_width((n_keys * 4 - 1) | 15)); }
ACB_FP_FN uint32_t amap_slot(uint32_t key, uint32_t amap_shift) { return bloom_hash3(key) >> amap_shift; }
ACB_FP_FN uint32_t amap_next(uint32_t slot, uint32_t amap_mask) { return (slot + 1) & amap_mask; }
ACB_FP_FN uint64_t amap_entry(uint32_t key, uint32_t id) { return uint64_t(key) | (uint64_t(id) << 32); }

}  // namespace acb
