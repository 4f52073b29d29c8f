// acb_plan.hpp -- the prefilter engine's plan for one automaton, derived from the host tables alone (so it
// also works for DFAs adopted through acg_dfa_create): which fingerprints the kernels probe, in which
// bitmap, and the anchor map their verifier starts from.  Its tables have the format of
// acb_fingerprint.cuh.  Host code, defined here and compiled with its one user, acb_api.cu.
#pragma once
#include <algorithm>

#include "acb_build.hpp"
#include "acb_device.cuh"
#include "acb_fingerprint.cuh"

namespace acb {

struct PrefilterPlan {
  bool supported = false;
  uint32_t k = 0, kmask = 0, fold = 0, mult = 1, mult3 = 1, shift = 0, log_bits = 0;
  uint32_t stride = 1;
  uint32_t key_shift = 8;  // stride 2: first-stage hash = window * (mult3 << key_shift); 5: the key also
                           // holds the low 3 bits of the window's fourth byte (default; 8 with ACG_EXP_KEY24)
  bool wide = false;
  bool brute = false;
  uint32_t dup_shift = 0;
  std::vector<uint32_t> bitmap;
  bool dense = false;  // many fingerprints: the kernel filters survivors through the anchor map
  // anchor map: (k-byte haystack prefix -> trie state at depth k), open addressing, see DfaDev::amap
  std::vector<uint64_t> amap;  // low word = key, high word = premultiplied state id (0 = empty)
  uint32_t amap_log = 0;
  // byte-set scan (bytescan_kernel): the needles of the reference's start-bytes / rare-bytes prefilter
  // when it would have picked one (bs_n == 0: fingerprint filter)
  uint32_t bs_n = 0;
  uint8_t bs_byte[3] = {0, 0, 0};
  uint8_t bs_back[3] = {0, 0, 0};
};

namespace plan_detail {

// bit `bit` of a bitmap of 32-bit words
inline void set_bit(std::vector<uint32_t>& bm, uint32_t bit) { bm[bit >> 5] |= 1u << (bit & 31); }
inline uint32_t test_bit(const std::vector<uint32_t>& bm, uint32_t bit) { return (bm[bit >> 5] >> (bit & 31)) & 1u; }

// The two-probe Bloom bitmap of 2^log_bits bits over the fingerprints `grams`: gram * kMult (a single
// multiply for the per-position probe) and the full mix bloom_hash2 (which only first-probe hits pay for).
inline std::vector<uint32_t> bloom_bitmap(const std::vector<uint32_t>& grams, uint32_t log_bits) {
  const uint32_t shift = bloom_shift(log_bits);
  std::vector<uint32_t> bm(size_t(1) << (log_bits - 5), 0u);
  for (uint32_t g : grams) {
    const uint32_t h1 = g * kMult, h2 = bloom_hash2(g);
    set_bit(bm, bloom_bit(h1, h1, shift));
    set_bit(bm, bloom_bit(h2, h2, shift));
  }
  return bm;
}

// Dense blocked filter: the word of fingerprint g and the mask of its two bits in that word.
struct DenseBits { uint32_t word, mask; };
inline DenseBits dense_bits(uint32_t g, uint32_t shift) {
  const uint64_t prod = uint64_t(g) * kMult;
  const uint32_t hi = uint32_t(prod >> 32);
  return {dense_word(uint32_t(prod), shift), (1u << dense_bit_a(hi)) | (1u << dense_bit_b(hi))};
}

// The distinct byte values, ascending, at each of the first n positions of the grams, and the number of
// strings they spell.
struct Alphabets {
  std::vector<uint8_t> at[4];
  double space = 1.0;
};
inline Alphabets alphabets(const std::vector<uint32_t>& grams, uint32_t n) {
  Alphabets out;
  for (uint32_t j = 0; j < n; ++j) {
    bool seen[256] = {false};
    for (uint32_t g : grams) seen[(g >> (8 * j)) & 0xFF] = true;
    for (uint32_t b = 0; b < 256; ++b)
      if (seen[b]) out.at[j].push_back(uint8_t(b));
    out.space *= double(std::max<size_t>(out.at[j].size(), 1));
  }
  return out;
}

// Pass-rate estimates: kTrials fingerprints drawn with a fixed-seed LCG; trial(next) draws one through
// next() -- as many steps as it likes -- and returns 1 if it passes the filter.
constexpr int kTrials = 65536;
template <class Trial>
uint64_t count_passes(Trial trial) {
  uint64_t x = 0x9E3779B97F4A7C15ull, pass = 0;
  auto next = [&x]() { return x = x * 6364136223846793005ull + 1442695040888963407ull; };
  for (int i = 0; i < kTrials; ++i) pass += trial(next);
  return pass;
}

}  // namespace plan_detail

// The plan of automaton `h`, whose rows have the trie depths `depth16`.  key24: 24-bit stride-2
// first-stage keys (ACG_EXP_KEY24) instead of 27-bit ones.
inline PrefilterPlan plan_prefilter(const HostDfa& h, const std::vector<uint16_t>& depth16, bool key24) {
  using namespace plan_detail;
  PrefilterPlan pf;
  if (h.pattern_lens.empty() || h.start_unanchored_id == 0) return pf;
  if (h.max_pattern_len >= 0xFFFE || h.min_pattern_len == 0) return pf;
  const uint32_t s2 = h.stride2;
  const size_t rows = size_t(h.state_len);
  // tie-break layout: (max_len - len) << dup_shift | index among the node's own patterns
  uint32_t max_dups = 1;
  for (size_t m = 0; m + 1 < h.match_offsets.size(); ++m) {
    const uint32_t lo = h.match_offsets[m], hi = h.match_offsets[m + 1];
    const uint32_t dep = (m + 2 < rows) ? depth16[m + 2] : 0xFFFF;
    uint32_t own = 0;
    for (uint32_t i = lo; i < hi && h.pattern_lens[h.match_pids[i]] == dep; ++i) ++own;
    max_dups = std::max(max_dups, own);
  }
  pf.dup_shift = uint32_t(bit_width(max_dups - 1));
  if (bit_width(h.max_pattern_len) + int(pf.dup_shift) > kTieBits) return pf;

  // Trie edges out of a row, bytes ascending: f(byte, child row) for every child that is not DEAD.  From
  // the table, or -- deferred dense fill, the table does not exist on the host -- from the builder's
  // shallow trie edges (grouped by source row, bytes ascending), the same transitions "one byte deeper".
  std::vector<uint32_t> sh_first;  // first shallow edge of a row, +1 (0: none)
  if (h.fill.valid) {
    sh_first.assign(rows, 0);
    for (size_t i = h.fill.shallow.size(); i-- > 0;) sh_first[h.fill.shallow[i].from_row] = uint32_t(i + 1);
  }
  auto for_each_edge = [&](uint32_t row, auto&& f) {
    if (h.fill.valid) {
      for (size_t i = sh_first[row]; i != 0 && i <= h.fill.shallow.size() && h.fill.shallow[i - 1].from_row == row; ++i)
        if (h.fill.shallow[i - 1].to_row != 0) f(h.fill.shallow[i - 1].byte, h.fill.shallow[i - 1].to_row);
      return;
    }
    const uint32_t* tr = h.trans.data() + (size_t(row) << s2);
    for (uint32_t b = 0; b < 256; ++b) {
      const uint32_t nr = tr[h.classes[b]] >> s2;
      if (nr != 0) f(b, nr);
    }
  };

  // k-gram fingerprints: every trie path of length k from the start row, over raw bytes
  const uint32_t kmax = uint32_t(std::min<uint64_t>(4, h.min_pattern_len));
  struct Item { uint32_t row; uint32_t gram; };
  std::vector<std::vector<uint32_t>> grams(kmax + 1);
  std::vector<std::vector<Item>> level(kmax + 1);  // (row, raw bytes) of every trie path of that length
  std::vector<Item> cur{{h.start_unanchored_id >> s2, 0u}}, nxt;
  for (uint32_t j = 0; j < kmax; ++j) {
    nxt.clear();
    for (const Item& it : cur)
      for_each_edge(it.row, [&](uint32_t b, uint32_t nr) {
        if (depth16[nr] == j + 1) nxt.push_back(Item{nr, it.gram | (b << (8 * j))});
      });
    cur.swap(nxt);
    level[j + 1] = cur;
    auto& g = grams[j + 1];
    g.reserve(cur.size());
    for (const Item& it : cur) g.push_back(it.gram);
    std::sort(g.begin(), g.end());
    g.erase(std::unique(g.begin(), g.end()), g.end());
    if (cur.size() > (64u << 20)) break;  // pathological fan-out: give up on longer fingerprints
  }
  // pick the fingerprint length with the sparsest bitmap (ties -> longer)
  double fill = 2.0;  // fraction of the probes that pass (~ candidate rate on random input)
  std::vector<uint32_t> best_set;
  for (uint32_t k = 1; k <= kmax; ++k) {
    if (grams[k].empty()) continue;
    const uint32_t kmask = k == 4 ? 0xFFFFFFFFu : ((1u << (8 * k)) - 1);
    std::vector<uint32_t> folded = grams[k];
    for (uint32_t& g : folded) g |= 0x20202020u & kmask;
    std::sort(folded.begin(), folded.end());
    folded.erase(std::unique(folded.begin(), folded.end()), folded.end());
    const bool use_fold = folded.size() * 3 < grams[k].size() * 2;
    const std::vector<uint32_t>& set = use_fold ? folded : grams[k];  // (k bytes each)
    std::vector<uint32_t> bm = bloom_bitmap(set, kNarrowLogBits);
    uint64_t set_bits = 0;
    for (uint32_t w : bm) set_bits += uint64_t(__builtin_popcount(w));
    double f = double(set_bits) / double(uint64_t(1) << kNarrowLogBits);
    f = f * f;  // both probes must hit
    // expected candidate rate on text drawn from the patterns' own alphabet: Bloom false positives
    // plus genuine k-gram prefix hits (fingerprints / prod_j |bytes seen at position j|)
    f += std::min(1.0, double(set.size()) / alphabets(set, k).space);
    if (f <= fill) {
      fill = f;
      pf.k = k; pf.kmask = kmask; pf.fold = use_fold ? (0x20202020u & kmask) : 0u;
      pf.mult = kMult; pf.shift = bloom_shift(kNarrowLogBits); pf.log_bits = kNarrowLogBits;
      pf.bitmap.swap(bm);
      best_set = set;
      for (uint32_t& g : best_set) g &= kmask;
    }
  }
  if (pf.k == 0) return pf;
  // Dense sets (more fingerprints than a two-probe Bloom filter of 2^20 bits can keep apart; cfg 5:
  // 10^5): the blocked filter instead, so that the per-position probe settles both bits with a single
  // shared-memory load; the second stage is then the exact anchor-map lookup.
  const bool dense = best_set.size() > kDenseGrams;
  if (dense) {
    std::fill(pf.bitmap.begin(), pf.bitmap.end(), 0u);
    for (uint32_t g : best_set) { const DenseBits d = dense_bits(g, pf.shift); pf.bitmap[d.word] |= d.mask; }
    // pass rate on text drawn from the bytes the patterns use at each fingerprint position
    const Alphabets alpha = alphabets(best_set, pf.k);
    fill = double(count_passes([&](auto& next) {
             uint32_t g = 0;
             for (uint32_t j = 0; j < pf.k; ++j) g |= uint32_t(alpha.at[j][(next() >> 33) % alpha.at[j].size()]) << (8 * j);
             const DenseBits d = dense_bits(g, pf.shift);
             return uint32_t((pf.bitmap[d.word] & d.mask) == d.mask);
           })) / kTrials;
  }
  pf.brute = fill > 0.25;
  pf.supported = true;
  // Stride-2 first stage: with 4-byte fingerprints and patterns of at least 4 bytes, probing only
  // every other offset with the 3-byte fingerprints of pattern bytes [0,3) and [1,4) still sees
  // every occurrence (a pattern that starts at an odd offset shows its second fingerprint at the
  // next even one) and halves the per-position probe work.  Worth it while those 3-grams stay rare.
  if (!pf.brute && pf.k == 4 && !dense) {
    std::vector<uint32_t> g3;
    g3.reserve(best_set.size() * 2);
    const uint32_t f3 = pf.fold & 0x00FFFFFFu;
    for (uint32_t g : best_set) {
      g3.push_back((g & 0x00FFFFFFu) | f3);
      g3.push_back((g >> 8) | f3);
    }
    std::sort(g3.begin(), g3.end());
    g3.erase(std::unique(g3.begin(), g3.end()), g3.end());
    const Alphabets alpha = alphabets(g3, 3);
    const double n_bits_set = double(g3.size()) + 2.0 * double(best_set.size());
    const double true3 = double(g3.size()) / alpha.space;
    const double pass1 = n_bits_set / double(uint64_t(1) << pf.log_bits) + true3;  // per probed offset
    if (pass1 < 0.07) {  // beyond that the second stage costs more than the halved probe count saves
      pf.stride = 2;
      // rare hits even with a 16 KiB bitmap: the wide geometry (2 KiB tiles, two CTAs per SM)
      // amortises the per-step bookkeeping better
      pf.wide = n_bits_set / double(uint64_t(1) << kWideLogBits) + true3 < 0.01;
      if (pf.wide) {
        pf.log_bits = kWideLogBits;
        pf.shift = bloom_shift(kWideLogBits);
        pf.bitmap = bloom_bitmap(best_set, kWideLogBits);
      }
      // First-stage keys.  24-bit keys (ACG_EXP_KEY24): the 3-byte fingerprints.  Default (faster on
      // cfg 2 and cfg 3): 27-bit keys -- the 3 bytes plus the low 3 bits of the window's fourth byte,
      // which a shift of 5 instead of 8 in the multiplier keeps at no cost in the kernel.  For a pattern
      // that starts at the probed (even) offset the fourth byte is its own fourth byte; for one that
      // starts one byte earlier it is the pattern's fifth byte -- any of the 8 values if the pattern
      // ends after four bytes.  Genuine 3-byte prefix hits (the bulk of the first-stage hits of cfg 2)
      // drop 8-fold.
      pf.key_shift = key24 ? 8 : 5;
      std::vector<uint32_t> keys1;
      if (key24) {
        keys1 = g3;
      } else {
        for (const Item& it : level[4]) {
          const uint32_t g = it.gram;
          keys1.push_back(((g & 0x00FFFFFFu) | f3) | (((g >> 24) & 7u) << 24));
          uint32_t xs = 0;  // bit x: some pattern through this 4-gram continues with a byte whose low bits are x
          if (it.row >= 2 && (it.row << s2) <= h.max_match_id) {
            const uint32_t lo = h.match_offsets[it.row - 2], hi = h.match_offsets[it.row - 1];
            if (lo < hi && h.pattern_lens[h.match_pids[lo]] == 4) xs = 0xFF;  // a 4-byte pattern ends here
          }
          if (xs != 0xFF)
            for_each_edge(it.row, [&](uint32_t b, uint32_t nr) {
              if (depth16[nr] == 5) xs |= 1u << (b & 7);
            });
          for (uint32_t x = 0; x < 8; ++x)
            if (xs >> x & 1) keys1.push_back(((g >> 8) | f3) | (x << 24));
        }
        std::sort(keys1.begin(), keys1.end());
        keys1.erase(std::unique(keys1.begin(), keys1.end()), keys1.end());
      }
      // The bit of a first-stage key: byte index from the key times (mult3 << key_shift), bit inside the
      // byte from the key's own low bits.  A multiplicative hash of such short keys is sensitive to the
      // constant, so pick the candidate that lets through the fewest keys drawn from the bytes the
      // patterns use at each position.
      static const uint32_t kCand[] = {0x1B873593u, 0x27D4EB2Fu, 0x165667B1u, 0x9E3779B1u, 0x2C1B3C6Du,
                                       0xB5297A4Du, 0x85EBCA6Bu, 0x5BD1E995u, 0x7FEB352Du, 0xCC9E2D51u,
                                       0x1B56C4E9u, 0xC2B2AE35u};
      auto key_bit = [&](uint32_t g, uint32_t m) { return bloom_bit(g * key_mult(m, pf.key_shift), g, pf.shift); };
      uint32_t best_m = kCand[0];
      uint64_t best_pass = UINT64_MAX;
      std::vector<uint32_t> trial;
      for (uint32_t m : kCand) {
        trial = pf.bitmap;
        for (uint32_t g : keys1) set_bit(trial, key_bit(g, m));
        const uint64_t pass = count_passes([&](auto& next) {
          const uint64_t x = next();
          const uint32_t r = uint32_t(x >> 33);
          uint32_t g = uint32_t(alpha.at[0][r % alpha.at[0].size()]) |
                       uint32_t(alpha.at[1][(r >> 10) % alpha.at[1].size()]) << 8 |
                       uint32_t(alpha.at[2][(r >> 20) % alpha.at[2].size()]) << 16;
          if (!key24) g |= uint32_t((x >> 20) & 7) << 24;
          return test_bit(trial, key_bit(g, m));
        });
        if (pass < best_pass) { best_pass = pass; best_m = m; }
      }
      pf.mult3 = best_m;
      for (uint32_t g : keys1) set_bit(pf.bitmap, key_bit(g, best_m));
    }
  }
  pf.dense = !pf.brute && dense;
  // Anchor map: the verifier looks the first k bytes at a candidate offset up here and starts at
  // depth k.  Keys are raw (unfolded) byte strings: one entry per trie path of length k.
  const std::vector<Item>& paths = level[pf.k];
  if (!paths.empty() && paths.size() <= (4u << 20)) {
    pf.amap_log = amap_log_for(paths.size());
    pf.amap.assign(size_t(1) << pf.amap_log, 0ull);
    const uint32_t shift = 32 - pf.amap_log, mask = (1u << pf.amap_log) - 1;
    for (const Item& it : paths) {
      const uint32_t key = it.gram & pf.kmask;
      uint32_t slot = amap_slot(key, shift);
      while (pf.amap[slot] != 0 && uint32_t(pf.amap[slot]) != key) slot = amap_next(slot, mask);
      pf.amap[slot] = amap_entry(key, it.row << s2);
    }
  }
  // Byte-set scan for the automata the reference gives a start-bytes / rare-bytes prefilter
  // (src/util/prefilter.rs:163-305).  Tables built here carry the set; for an adopted table that
  // reports start bytes the set is read off the start row (the first bytes of all patterns).
  if (h.prefilter_kind == kPreStartBytes || h.prefilter_kind == kPreRareBytes) {
    if (h.pre_n) {
      // Needles with offsets (rare bytes in the middle of patterns) turn every occurrence into
      // back + 1 start offsets to verify; on BASELINE config 1's automaton over uniform printable text
      // that is slower than the fingerprint filter, so the scan is reserved for needles that mark a
      // pattern's first byte (bs_back stays 0).
      if (std::all_of(h.pre_back, h.pre_back + h.pre_n, [](uint8_t back) { return back == 0; })) {
        pf.bs_n = h.pre_n;
        std::copy(h.pre_byte, h.pre_byte + h.pre_n, pf.bs_byte);
      }
    } else if (h.prefilter_kind == kPreStartBytes && !level[1].empty() && grams[1].size() <= 3) {
      pf.bs_n = uint32_t(grams[1].size());
      std::copy(grams[1].begin(), grams[1].end(), pf.bs_byte);
    }
  }
  return pf;
}

// The anchor-map fields of the kernels' view of the automaton (d.amap is the device copy of pf.amap).
inline void plan_device_fields(const PrefilterPlan& pf, DfaDev& d) {
  d.amap_shift = pf.amap_log ? 32 - pf.amap_log : 0;
  d.amap_mask = pf.amap_log ? (1u << pf.amap_log) - 1 : 0;
  d.amap_k = pf.k;
  d.amap_kmask = pf.kmask;
}

}  // namespace acb
