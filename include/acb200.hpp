// acb200.hpp -- header-only C++ facade over the C ABI (acb200.h).
//
// Mirrors the search surface of BurntSushi/aho-corasick 1.1.3 (the reference is Rust; there is no
// Rust toolchain in the build image, so the host side above the C ABI is C++):
//
//   reference (src/ahocorasick.rs)                        here
//   ---------------------------------------------------  -----------------------------------------
//   AhoCorasick::new(patterns)                    :243   acb200::AhoCorasick::create(patterns)
//   AhoCorasick::builder()                        :268   acb200::AhoCorasick::builder()
//   AhoCorasickBuilder::{match_kind, start_kind,          acb200::AhoCorasickBuilder (same knobs,
//     ascii_case_insensitive, kind, prefilter,              same defaults)
//     dense_depth, byte_classes, build}      :2171-2616
//   find / try_find / is_match           :311, 404, 1021   find / try_find / is_match
//   find_iter / try_find_iter                 :562, 1275   find_iter / try_find_iter
//   find_overlapping_iter / try_...           :609, 1350   find_overlapping_iter / try_...
//   kind, start_kind, match_kind, min/max_pattern_len,     same names
//     patterns_len, memory_usage              :1867-2021
//   Match { pattern(), start(), end(), span(), ... }       acb200::Match (src/util/search.rs:825-1000)
//   Input { span, anchored, earliest }   search.rs:83-88   acb200::Input
//   MatchError / BuildError          src/util/error.rs     acb200::MatchError / acb200::BuildError
//
// The `find_*` methods panic in the reference where the `try_*` methods return Err; here `find_*`
// throw the same exception the `try_*` variants report through acb200::Result.  Iterators are
// cursors over the materialised, already ordered match list (the device scan is eager; results are
// identical to the reference's lazy iteration).
#pragma once
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <algorithm>
#include <string_view>
#include <utility>
#include <vector>

#include "acb200.h"

namespace acb200 {

enum class MatchKind : int { Standard = ACG_STANDARD, LeftmostFirst = ACG_LEFTMOST_FIRST, LeftmostLongest = ACG_LEFTMOST_LONGEST };
enum class StartKind : int { Unanchored = ACG_START_UNANCHORED, Anchored = ACG_START_ANCHORED, Both = ACG_START_BOTH };
enum class AhoCorasickKind : int { NoncontiguousNFA = ACG_KIND_NONCONTIGUOUS_NFA, ContiguousNFA = ACG_KIND_CONTIGUOUS_NFA, DFA = ACG_KIND_DFA };
enum class Anchored : int { No = 0, Yes = 1 };

// src/util/error.rs:23-49
class BuildError : public std::runtime_error {
 public:
  explicit BuildError(int code) : std::runtime_error(acg_strerror(code)), code_(code) {}
  int code() const { return code_; }
 private:
  int code_;
};

// src/util/error.rs:140-223
enum class MatchErrorKind { InvalidInputAnchored, InvalidInputUnanchored, UnsupportedStream, UnsupportedOverlapping, UnsupportedEmpty, Boundary };
class MatchError : public std::runtime_error {
 public:
  explicit MatchError(int code) : std::runtime_error(acg_strerror(code)), code_(code) {}
  int code() const { return code_; }
  MatchErrorKind kind() const {
    switch (code_) {
      case ACG_E_INVALID_INPUT_ANCHORED: return MatchErrorKind::InvalidInputAnchored;
      case ACG_E_INVALID_INPUT_UNANCHORED: return MatchErrorKind::InvalidInputUnanchored;
      case ACG_E_UNSUPPORTED_STREAM: return MatchErrorKind::UnsupportedStream;
      case ACG_E_UNSUPPORTED_OVERLAPPING: return MatchErrorKind::UnsupportedOverlapping;
      case ACG_E_UNSUPPORTED_EMPTY: return MatchErrorKind::UnsupportedEmpty;
      default: return MatchErrorKind::Boundary;
    }
  }
 private:
  int code_;
};
// device / boundary failures (no CPU fallback exists)
class DeviceError : public std::runtime_error {
 public:
  explicit DeviceError(int code) : std::runtime_error(acg_strerror(code)), code_(code) {}
  int code() const { return code_; }
 private:
  int code_;
};

// `Match`, src/util/search.rs:825-1000
class Match {
 public:
  Match() = default;
  Match(uint32_t pid, uint64_t start, uint64_t end) : pid_(pid), start_(start), end_(end) {}
  uint32_t pattern() const { return pid_; }
  uint64_t start() const { return start_; }
  uint64_t end() const { return end_; }
  std::pair<uint64_t, uint64_t> span() const { return {start_, end_}; }
  uint64_t len() const { return end_ - start_; }
  bool is_empty() const { return start_ == end_; }
  bool operator==(const Match& o) const { return pid_ == o.pid_ && start_ == o.start_ && end_ == o.end_; }
 private:
  uint32_t pid_ = 0;
  uint64_t start_ = 0, end_ = 0;
};

// `Input`, src/util/search.rs:83-88, builder-style setters :148-330
class Input {
 public:
  // implicit on purpose, like `impl<'h, H: AsRef<[u8]>> From<&'h H> for Input<'h>` (search.rs:656)
  Input(std::string_view haystack) : hay_(haystack), start_(0), end_(haystack.size()) {}  // NOLINT
  Input(const std::string& haystack) : Input(std::string_view(haystack)) {}                // NOLINT
  Input(const char* haystack) : Input(std::string_view(haystack)) {}                       // NOLINT
  Input(const uint8_t* p, size_t n) : hay_(reinterpret_cast<const char*>(p), n), start_(0), end_(n) {}
  Input& span(uint64_t start, uint64_t end) { start_ = start; end_ = end; return *this; }
  Input& range(uint64_t start, uint64_t end) { return span(start, end); }
  Input& anchored(Anchored a) { anchored_ = a; return *this; }
  Input& earliest(bool yes) { earliest_ = yes; return *this; }
  std::string_view haystack() const { return hay_; }
  uint64_t start() const { return start_; }
  uint64_t end() const { return end_; }
  Anchored get_anchored() const { return anchored_; }
  bool get_earliest() const { return earliest_; }
 private:
  std::string_view hay_;
  uint64_t start_, end_;
  Anchored anchored_ = Anchored::No;
  bool earliest_ = false;
};

template <class T>
struct Result {  // Result<T, MatchError>
  T value{};
  int error = 0;
  bool is_ok() const { return error == 0; }
  bool is_err() const { return error != 0; }
  T& unwrap() {
    if (error) throw_error(error);
    return value;
  }
  static void throw_error(int e) {
    if (e <= ACG_E_INVALID_INPUT_ANCHORED && e >= ACG_E_UNSUPPORTED_EMPTY) throw MatchError(e);
    if (e == ACG_E_INVALID_SPAN) throw std::out_of_range(acg_strerror(e));  // the reference panics
    throw DeviceError(e);
  }
};

// FindIter / FindOverlappingIter (src/automaton.rs:844-970): cursor over the ordered matches.
class MatchIter {
 public:
  MatchIter() = default;
  explicit MatchIter(std::vector<Match> m) : m_(std::move(m)) {}
  // Iterator::next -> Option<Match>
  bool next(Match* out) {
    if (i_ >= m_.size()) return false;
    *out = m_[i_++];
    return true;
  }
  std::vector<Match>::const_iterator begin() const { return m_.begin(); }
  std::vector<Match>::const_iterator end() const { return m_.end(); }
  size_t count() const { return m_.size(); }
  const std::vector<Match>& collect() const { return m_; }
 private:
  std::vector<Match> m_;
  size_t i_ = 0;
};
using FindIter = MatchIter;
using FindOverlappingIter = MatchIter;

// `OverlappingState`, src/automaton.rs:782-840: the cursor of a resumable overlapping search.  The
// device scan is eager, so the state holds the ordered match list of the search it was first used
// with and hands out one match per try_find_overlapping call -- the sequence the reference's state
// machine produces.  As in the reference, reuse a state only with the same automaton and input.
class OverlappingState {
 public:
  static OverlappingState start() { return OverlappingState(); }  // :817
  std::optional<Match> get_match() const { return mat_; }         // :829
 private:
  friend class AhoCorasick;
  bool started_ = false;
  std::vector<Match> matches_;
  size_t next_ = 0;
  std::optional<Match> mat_;
};

namespace detail {
// `str::is_char_boundary` on UTF-8 bytes
inline bool is_char_boundary(std::string_view s, uint64_t i) {
  if (i == 0 || i == s.size()) return true;
  return i < s.size() && (static_cast<unsigned char>(s[i]) & 0xC0) != 0x80;
}
// The loop of try_replace_all_with{,_bytes} (src/automaton.rs:498-550) over a materialised match
// list: `f(match, matched text, dst) -> bool`, false stops after that match.  With
// `char_boundaries` (the &str flavour) matches that split a UTF-8 code point are skipped (:514-518).
template <class F>
void splice(std::string_view hay, const std::vector<Match>& matches, std::string& dst, F&& f, bool char_boundaries) {
  uint64_t last = 0;
  for (const Match& m : matches) {
    if (char_boundaries && !(is_char_boundary(hay, m.start()) && is_char_boundary(hay, m.end()))) continue;
    dst.append(hay.substr(last, m.start() - last));
    last = m.end();
    if (!f(m, hay.substr(m.start(), m.end() - m.start()), dst)) break;
  }
  dst.append(hay.substr(last));
}
}  // namespace detail

class AhoCorasick;

// `AhoCorasickBuilder`, src/ahocorasick.rs:2135-2617
class AhoCorasickBuilder {
 public:
  AhoCorasickBuilder() { acg_build_opts_default(&o_); }
  AhoCorasickBuilder& match_kind(MatchKind k) { o_.match_kind = int(k); return *this; }
  AhoCorasickBuilder& start_kind(StartKind k) { o_.start_kind = int(k); return *this; }
  AhoCorasickBuilder& ascii_case_insensitive(bool yes) { o_.ascii_case_insensitive = yes; return *this; }
  AhoCorasickBuilder& kind(AhoCorasickKind k) { o_.kind = int(k); return *this; }
  AhoCorasickBuilder& kind_auto() { o_.kind = ACG_KIND_AUTO; return *this; }  // kind(None)
  AhoCorasickBuilder& prefilter(bool yes) { o_.prefilter = yes; return *this; }
  AhoCorasickBuilder& dense_depth(uint64_t d) { o_.dense_depth = int64_t(d); return *this; }
  AhoCorasickBuilder& byte_classes(bool yes) { o_.byte_classes = yes; return *this; }
  // device-side knob with no counterpart in the reference: fill the dense table on the GPU
  // (acg_build_on_device) instead of on the host; same table, same results
  AhoCorasickBuilder& device_fill(bool yes) { device_fill_ = yes; return *this; }
  template <class Patterns>
  AhoCorasick build(const Patterns& patterns) const;
 private:
  acg_build_opts o_;
  bool device_fill_ = false;
};

// `AhoCorasick`, src/ahocorasick.rs:177-2082 (search surface)
class AhoCorasick {
 public:
  AhoCorasick() = default;
  AhoCorasick(AhoCorasick&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  AhoCorasick& operator=(AhoCorasick&& o) noexcept {
    if (this != &o) { reset(); h_ = o.h_; o.h_ = nullptr; }
    return *this;
  }
  AhoCorasick(const AhoCorasick&) = delete;
  AhoCorasick& operator=(const AhoCorasick&) = delete;
  ~AhoCorasick() { reset(); }

  template <class Patterns>
  static AhoCorasick create(const Patterns& patterns) { return AhoCorasickBuilder().build(patterns); }  // ::new
  static AhoCorasickBuilder builder() { return AhoCorasickBuilder(); }

  AhoCorasickKind kind() const { return AhoCorasickKind(acg_kind(h_)); }
  StartKind start_kind() const { return StartKind(acg_start_kind(h_)); }
  MatchKind match_kind() const { return MatchKind(acg_match_kind(h_)); }
  uint64_t min_pattern_len() const { return acg_min_pattern_len(h_); }
  uint64_t max_pattern_len() const { return acg_max_pattern_len(h_); }
  uint64_t patterns_len() const { return acg_patterns_len(h_); }
  uint64_t memory_usage() const { return acg_memory_usage(h_); }

  // try_find, src/ahocorasick.rs:1021
  Result<std::pair<bool, Match>> try_find(const Input& in) const {
    Result<std::pair<bool, Match>> r;
    acg_match m{};
    int found = 0;
    r.error = acg_find(h_, hay(in), in.haystack().size(), in.start(), in.end(), int(in.get_anchored()),
                       in.get_earliest(), &m, &found);
    r.value = {found != 0, Match(m.pid, m.start, m.end)};
    return r;
  }
  // find, :404 (panics in the reference where this throws)
  bool find(const Input& in, Match* out) const {
    auto r = try_find(in).unwrap();
    if (r.first && out) *out = r.second;
    return r.first;
  }
  // is_match, :311
  bool is_match(const Input& in) const {
    Input e = in;
    e.earliest(match_kind() == MatchKind::Standard);  // existence is all that is reported
    return try_find(e).unwrap().first;
  }
  // try_find_iter, :1275
  Result<FindIter> try_find_iter(const Input& in) const { return collect(acg_find_iter, in); }
  FindIter find_iter(const Input& in) const { return std::move(try_find_iter(in).unwrap()); }  // :562
  // try_find_overlapping_iter, :1350
  Result<FindOverlappingIter> try_find_overlapping_iter(const Input& in) const {
    return collect(acg_find_overlapping, in);
  }
  FindOverlappingIter find_overlapping_iter(const Input& in) const {  // :609
    return std::move(try_find_overlapping_iter(in).unwrap());
  }

  // try_find_overlapping, :1184: advance `state` to the next overlapping match (or to none)
  Result<bool> try_find_overlapping(const Input& in, OverlappingState& state) const {
    Result<bool> r;
    if (!state.started_) {
      auto it = try_find_overlapping_iter(in);
      if (it.is_err()) { r.error = it.error; return r; }
      state.matches_ = it.value.collect();
      state.next_ = 0;
      state.started_ = true;
    }
    if (state.next_ < state.matches_.size()) state.mat_ = state.matches_[state.next_++];
    else state.mat_.reset();
    r.value = state.mat_.has_value();
    return r;
  }
  void find_overlapping(const Input& in, OverlappingState& state) const { try_find_overlapping(in, state).unwrap(); }  // :470

  // Batched search (acg_*_batch, include/acb200.h): many documents in one device call.  `offsets` are the
  // CSR bounds [n_docs + 1] into `haystack`; per document the result is the single-haystack call's on that
  // document alone, offsets relative to it.
  using PerDoc = std::vector<std::vector<Match>>;
  Result<PerDoc> try_find_iter_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                     Anchored a = Anchored::No) const {
    return collect_batch(acg_find_iter_batch, haystack, offsets, a);
  }
  Result<PerDoc> try_find_overlapping_iter_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                                 Anchored a = Anchored::No) const {
    return collect_batch(acg_find_overlapping_batch, haystack, offsets, a);
  }
  Result<std::vector<bool>> try_is_match_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                               Anchored a = Anchored::No) const {
    Result<std::vector<bool>> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    std::vector<uint8_t> flags(offsets.size());
    r.error = acg_is_match_batch(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(),
                                 offsets.data(), offsets.size() - 1, int(a), flags.data());
    if (r.error == 0) r.value.assign(flags.begin(), flags.end() - 1);
    return r;
  }
  PerDoc find_iter_batch(std::string_view haystack, const std::vector<uint64_t>& offsets, Anchored a = Anchored::No) const {
    return std::move(try_find_iter_batch(haystack, offsets, a).unwrap());
  }
  PerDoc find_overlapping_iter_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                     Anchored a = Anchored::No) const {
    return std::move(try_find_overlapping_iter_batch(haystack, offsets, a).unwrap());
  }
  std::vector<bool> is_match_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                   Anchored a = Anchored::No) const {
    return std::move(try_is_match_batch(haystack, offsets, a).unwrap());
  }
  // try_find of every document (acg_find_batch): its first match, or nullopt
  using FirstPerDoc = std::vector<std::optional<Match>>;
  Result<FirstPerDoc> try_find_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                     Anchored a = Anchored::No, bool earliest = false) const {
    Result<FirstPerDoc> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    const uint64_t n_docs = offsets.size() - 1;
    std::vector<acg_doc_match> out(n_docs);
    std::vector<uint8_t> found(n_docs);
    r.error = acg_find_batch(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(), offsets.data(),
                             n_docs, int(a), int(earliest), out.data(), found.data());
    if (r.error == 0) {
      r.value.resize(n_docs);
      for (uint64_t d = 0; d < n_docs; ++d)
        if (found[d]) r.value[d] = Match(out[d].pid, out[d].start, out[d].end);
    }
    return r;
  }
  FirstPerDoc find_batch(std::string_view haystack, const std::vector<uint64_t>& offsets, Anchored a = Anchored::No,
                         bool earliest = false) const {
    return std::move(try_find_batch(haystack, offsets, a, earliest).unwrap());
  }
  // How often each pattern occurs in each document (acg_pattern_counts_batch): the records of
  // find_overlapping_iter_batch (`overlapping`) or find_iter_batch counted by (document, pattern), as a CSR
  // matrix -- document d's patterns are pids[row_offsets[d] .. row_offsets[d + 1]), ascending, each counts[i] times.
  struct PatternCounts {
    std::vector<uint64_t> row_offsets;  // [n_docs + 1]
    std::vector<uint32_t> pids;
    std::vector<uint64_t> counts;
  };
  Result<PatternCounts> try_pattern_counts_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                                 bool overlapping = false, Anchored a = Anchored::No) const {
    Result<PatternCounts> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    PatternCounts& c = r.value;
    c.row_offsets.resize(offsets.size());
    uint64_t nnz = 0;
    for (uint64_t cap = cap_hint_;; cap = nnz) {
      c.pids.resize(cap);
      c.counts.resize(cap);
      r.error = acg_pattern_counts_batch(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(),
                                         offsets.data(), offsets.size() - 1, int(a), int(overlapping),
                                         c.row_offsets.data(), c.pids.data(), c.counts.data(), cap, &nnz);
      if (r.error != ACG_E_OVERFLOW) break;  // two-call protocol: nnz is the required count
    }
    c.pids.resize(r.error ? 0 : nnz);
    c.counts.resize(r.error ? 0 : nnz);
    return r;
  }
  PatternCounts pattern_counts_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                     bool overlapping = false, Anchored a = Anchored::No) const {
    return std::move(try_pattern_counts_batch(haystack, offsets, overlapping, a).unwrap());
  }
  // How much of each document its matches cover (acg_match_coverage_batch): covered[d] is the number of bytes of
  // document d inside at least one record of find_overlapping_iter_batch (`overlapping`) or find_iter_batch; with
  // `with_mask`, mask[i] (one entry per haystack byte) is 1 where byte i lies in a match of its document.
  struct MatchCoverage {
    std::vector<uint64_t> covered;  // [n_docs]
    std::vector<uint8_t> mask;      // [haystack.size()], or empty
  };
  Result<MatchCoverage> try_match_coverage_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                                 bool overlapping = false, Anchored a = Anchored::No,
                                                 bool with_mask = false) const {
    Result<MatchCoverage> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    MatchCoverage& c = r.value;
    c.covered.resize(offsets.size() - 1);
    if (with_mask) c.mask.assign(haystack.size(), 0);
    r.error = acg_match_coverage_batch(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(),
                                       offsets.data(), offsets.size() - 1, int(a), int(overlapping), c.covered.data(),
                                       with_mask ? c.mask.data() : nullptr);
    if (r.error) c = MatchCoverage{};
    return r;
  }
  MatchCoverage match_coverage_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                     bool overlapping = false, Anchored a = Anchored::No, bool with_mask = false) const {
    return std::move(try_match_coverage_batch(haystack, offsets, overlapping, a, with_mask).unwrap());
  }
  // replace_all_bytes of every document (acg_replace_all_batch): the documents with their find_iter matches
  // replaced by replacements[pattern], spliced on the device, as a batch: document d's result is
  // bytes[offsets[d] .. offsets[d + 1]).  One replacement per pattern, or ACG_E_INVALID_ARG.
  struct ReplacedBatch {
    std::string bytes;
    std::vector<uint64_t> offsets;  // [n_docs + 1]
  };
  template <class Replacements>
  Result<ReplacedBatch> try_replace_all_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                              const Replacements& replacements) const {
    Result<ReplacedBatch> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    std::string table;
    std::vector<uint64_t> at{0};
    for (const auto& x : replacements) {
      table.append(std::string_view(x));
      at.push_back(table.size());
    }
    ReplacedBatch& b = r.value;
    b.offsets.resize(offsets.size());
    const uint64_t span = offsets.back() >= offsets.front() ? offsets.back() - offsets.front() : 0;
    uint64_t need = 0;
    for (uint64_t cap = span + span / 8 + 4096;; cap = need) {
      b.bytes.resize(cap);
      r.error = acg_replace_all_batch(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(),
                                      offsets.data(), offsets.size() - 1,
                                      reinterpret_cast<const uint8_t*>(table.data()), at.data(), at.size() - 1,
                                      reinterpret_cast<uint8_t*>(b.bytes.data()), cap, b.offsets.data(), &need);
      if (r.error != ACG_E_OVERFLOW) break;  // two-call protocol: need is the required size
    }
    if (r.error) b = ReplacedBatch{};
    else b.bytes.resize(need);
    return r;
  }
  template <class Replacements>
  ReplacedBatch replace_all_batch(std::string_view haystack, const std::vector<uint64_t>& offsets,
                                  const Replacements& replacements) const {
    return std::move(try_replace_all_batch(haystack, offsets, replacements).unwrap());
  }

  // replace_all_with / replace_all_with_bytes, :834 / :887 (src/automaton.rs:498-550)
  template <class F>
  void replace_all_with(std::string_view haystack, std::string& dst, F&& replace_with) const {
    detail::splice(haystack, find_iter(Input(haystack)).collect(), dst, replace_with, true);
  }
  template <class F>
  void replace_all_with_bytes(std::string_view haystack, std::string& dst, F&& replace_with) const {
    detail::splice(haystack, find_iter(Input(haystack)).collect(), dst, replace_with, false);
  }
  // replace_all / replace_all_bytes, :651 / :693: one replacement per pattern (the reference panics
  // otherwise, src/automaton.rs:443-448)
  template <class Replacements>
  std::string replace_all(std::string_view haystack, const Replacements& replace_with) const {
    return replace_impl(haystack, replace_with, true);
  }
  template <class Replacements>
  std::string replace_all_bytes(std::string_view haystack, const Replacements& replace_with) const {
    return replace_impl(haystack, replace_with, false);
  }

  acg_dfa* raw() const { return h_; }

 private:
  friend class AhoCorasickBuilder;
  template <class Replacements>
  std::string replace_impl(std::string_view haystack, const Replacements& replace_with, bool char_boundaries) const {
    std::vector<std::string_view> reps;
    for (const auto& r : replace_with) reps.emplace_back(r);
    if (reps.size() != patterns_len())
      throw std::invalid_argument("replace_all requires a replacement for every pattern in the automaton");
    std::string dst;
    dst.reserve(haystack.size());
    detail::splice(haystack, find_iter(Input(haystack)).collect(), dst,
                   [&](const Match& m, std::string_view, std::string& out) { out.append(reps[m.pattern()]); return true; },
                   char_boundaries);
    return dst;
  }
  explicit AhoCorasick(acg_dfa* h) : h_(h) {}
  void reset() {
    if (h_) acg_dfa_free(h_);
    h_ = nullptr;
  }
  static const uint8_t* hay(const Input& in) { return reinterpret_cast<const uint8_t*>(in.haystack().data()); }
  using SearchFn = int (*)(const acg_dfa*, const uint8_t*, uint64_t, uint64_t, uint64_t, int, acg_match*, uint64_t, uint64_t*);
  Result<MatchIter> collect(SearchFn fn, const Input& in) const {
    Result<MatchIter> r;
    // room for one match per 256 haystack bytes from the start (the device sizes its own tuple buffer
    // the same way): an ACG_E_OVERFLOW retry repeats the whole copy + scan, so it should be the exception
    const uint64_t span_len = in.end() > in.start() ? in.end() - in.start() : 0;
    std::vector<acg_match> buf(std::max<uint64_t>(cap_hint_, span_len / 256 + 64));
    uint64_t n = 0;
    for (;;) {
      int rc = fn(h_, hay(in), in.haystack().size(), in.start(), in.end(), int(in.get_anchored()), buf.data(),
                  buf.size(), &n);
      if (rc == ACG_E_OVERFLOW) {  // two-call protocol: n is the required count
        cap_hint_ = n + n / 8 + 64;
        buf.resize(cap_hint_);
        continue;
      }
      r.error = rc;
      break;
    }
    if (r.error == 0) {
      std::vector<Match> out;
      out.reserve(n);
      for (uint64_t i = 0; i < n; ++i) out.emplace_back(buf[i].pid, buf[i].start, buf[i].end);
      r.value = MatchIter(std::move(out));
    }
    return r;
  }
  using BatchFn = int (*)(const acg_dfa*, const uint8_t*, int, uint64_t, const uint64_t*, uint64_t, int, acg_doc_match*,
                          uint64_t, uint64_t*);
  Result<PerDoc> collect_batch(BatchFn fn, std::string_view haystack, const std::vector<uint64_t>& offsets, Anchored a) const {
    Result<PerDoc> r;
    if (offsets.empty()) { r.error = ACG_E_INVALID_ARG; return r; }
    const uint64_t n_docs = offsets.size() - 1;
    std::vector<acg_doc_match> buf(std::max<uint64_t>(cap_hint_, haystack.size() / 256 + 64));
    uint64_t n = 0;
    for (;;) {
      const int rc = fn(h_, reinterpret_cast<const uint8_t*>(haystack.data()), 0, haystack.size(), offsets.data(), n_docs,
                        int(a), buf.data(), buf.size(), &n);
      if (rc == ACG_E_OVERFLOW) {
        cap_hint_ = n + n / 8 + 64;
        buf.resize(cap_hint_);
        continue;
      }
      r.error = rc;
      break;
    }
    if (r.error == 0) {
      r.value.resize(n_docs);
      for (uint64_t i = 0; i < n; ++i) r.value[buf[i].doc].emplace_back(buf[i].pid, buf[i].start, buf[i].end);
    }
    return r;
  }
  acg_dfa* h_ = nullptr;
  mutable uint64_t cap_hint_ = 4096;
};

// A candidate set (acg_candidates_create, include/acb200.h): a fixed list of byte strings -- a tokenizer's vocabulary,
// say -- on the automaton's device, for the lookahead of that automaton's stream sets.  The automaton must outlive it.
class Candidates {
 public:
  template <class Strings>
  Candidates(const AhoCorasick& ac, const Strings& cands) {
    std::string bytes;
    std::vector<uint64_t> at{0};
    for (const auto& x : cands) {
      bytes.append(std::string_view(x));
      at.push_back(bytes.size());
    }
    Result<int> r;
    r.error = acg_candidates_create(ac.raw(), reinterpret_cast<const uint8_t*>(bytes.data()), at.data(),
                                    at.size() - 1, &h_);
    r.unwrap();
    n_ = at.size() - 1;
  }
  Candidates(Candidates&& o) noexcept : h_(o.h_), n_(o.n_) { o.h_ = nullptr; }
  Candidates& operator=(Candidates&& o) noexcept {
    if (this != &o) { close(); h_ = o.h_; n_ = o.n_; o.h_ = nullptr; }
    return *this;
  }
  Candidates(const Candidates&) = delete;
  Candidates& operator=(const Candidates&) = delete;
  ~Candidates() { close(); }

  uint64_t size() const { return n_; }
  acg_candidates* raw() const { return h_; }

 private:
  void close() {
    if (h_) acg_candidates_free(h_);
    h_ = nullptr;
  }
  acg_candidates* h_ = nullptr;
  uint64_t n_ = 0;
};

namespace detail {
// acg_streams_lookahead: rows(ids) x cands.size() bytes, row-major, 1 where feeding that row's stream that candidate
// would return a match.  An empty `ids` takes every one of the set's n streams.
inline Result<std::vector<uint8_t>> lookahead(const acg_streams* set, uint64_t n, const Candidates& cands,
                                              const std::vector<uint64_t>& ids) {
  Result<std::vector<uint8_t>> r;
  r.value.resize((ids.empty() ? n : ids.size()) * cands.size());
  r.error = acg_streams_lookahead(set, cands.raw(), ids.empty() ? nullptr : ids.data(), ids.size(), r.value.data());
  return r;
}
}  // namespace detail

// A stream set (acg_streams_*, include/acb200.h): n streams searched on the device as their bytes arrive.  feed()
// takes one chunk per stream -- CSR `offsets` [n + 1] into `chunks` -- and returns, per stream, the matches of the
// mode's iterator (find_iter, or find_overlapping_iter when `overlapping`) over all the stream's bytes that end in
// this chunk, with offsets into the whole stream.  The automaton must outlive the set; one call at a time per set.
class Streams {
 public:
  Streams(const AhoCorasick& ac, uint64_t n_streams, bool overlapping = false) {
    Result<int> r;
    r.error = acg_streams_create(ac.raw(), n_streams, overlapping, &h_);
    r.unwrap();
    n_ = n_streams;
  }
  Streams(Streams&& o) noexcept : h_(o.h_), n_(o.n_), cap_hint_(o.cap_hint_) { o.h_ = nullptr; }
  Streams& operator=(Streams&& o) noexcept {
    if (this != &o) { close(); h_ = o.h_; n_ = o.n_; cap_hint_ = o.cap_hint_; o.h_ = nullptr; }
    return *this;
  }
  Streams(const Streams&) = delete;
  Streams& operator=(const Streams&) = delete;
  ~Streams() { close(); }

  uint64_t n_streams() const { return n_; }

  using PerStream = std::vector<std::vector<Match>>;
  Result<PerStream> try_feed(std::string_view chunks, const std::vector<uint64_t>& offsets) {
    Result<PerStream> r;
    std::vector<acg_doc_match> buf(std::max<uint64_t>(cap_hint_, 64));
    uint64_t n = 0;
    for (;;) {
      const uint64_t n_chunks = offsets.empty() ? 0 : offsets.size() - 1;
      const int rc = acg_streams_feed(h_, reinterpret_cast<const uint8_t*>(chunks.data()), 0, chunks.size(),
                                      offsets.empty() ? nullptr : offsets.data(), n_chunks, buf.data(), buf.size(), &n);
      if (rc == ACG_E_OVERFLOW) {  // nothing was fed: retry with room for n
        cap_hint_ = n + n / 8 + 64;
        buf.resize(cap_hint_);
        continue;
      }
      r.error = rc;
      break;
    }
    if (r.error == 0) {
      r.value.resize(n_);
      for (uint64_t i = 0; i < n; ++i) r.value[buf[i].doc].emplace_back(buf[i].pid, buf[i].start, buf[i].end);
    }
    return r;
  }
  PerStream feed(std::string_view chunks, const std::vector<uint64_t>& offsets) {
    return std::move(try_feed(chunks, offsets).unwrap());
  }
  // Restart the given streams from zero bytes; reset() restarts every stream.
  void reset(const std::vector<uint64_t>& ids) {
    if (ids.empty()) return;
    Result<int> r;
    r.error = acg_streams_reset(h_, ids.data(), ids.size());
    r.unwrap();
  }
  void reset() {
    Result<int> r;
    r.error = acg_streams_reset(h_, nullptr, 0);
    r.unwrap();
  }
  // The bytes every stream has received.
  std::vector<uint64_t> positions() const {
    std::vector<uint64_t> pos(n_);
    Result<int> r;
    r.error = acg_streams_positions(h_, pos.data());
    r.unwrap();
    return pos;
  }
  // For every row -- stream ids[k], or every stream when ids is empty -- and every candidate c: 1 if feeding that
  // stream c would return a match, row-major.  No stream changes.
  Result<std::vector<uint8_t>> try_lookahead(const Candidates& cands, const std::vector<uint64_t>& ids = {}) const {
    return detail::lookahead(h_, n_, cands, ids);
  }
  std::vector<uint8_t> lookahead(const Candidates& cands, const std::vector<uint64_t>& ids = {}) const {
    return std::move(try_lookahead(cands, ids).unwrap());
  }
  acg_streams* raw() const { return h_; }

 private:
  void close() {
    if (h_) acg_streams_free(h_);
    h_ = nullptr;
  }
  acg_streams* h_ = nullptr;
  uint64_t n_ = 0;
  uint64_t cap_hint_ = 4096;
};

// A replace set (acg_streams_create_replace, include/acb200.h): n streams whose text is replaced on the device as
// their bytes arrive.  feed() takes one chunk per stream -- CSR `offsets` [n + 1] into `chunks` -- and returns per
// stream the text this feed settled, with every find_iter match replaced by replacements[pattern]; flush() returns
// the bytes the streams still hold back and restarts them.  A stream's feeds followed by its flush give
// replace_all_bytes of everything it received.  The automaton must outlive the set; one call at a time per set.
class ReplaceStreams {
 public:
  template <class Replacements>
  ReplaceStreams(const AhoCorasick& ac, uint64_t n_streams, const Replacements& replacements) {
    std::string table;
    std::vector<uint64_t> at{0};
    for (const auto& x : replacements) {
      table.append(std::string_view(x));
      at.push_back(table.size());
    }
    Result<int> r;
    r.error = acg_streams_create_replace(ac.raw(), n_streams, reinterpret_cast<const uint8_t*>(table.data()),
                                         at.data(), at.size() - 1, &h_);
    r.unwrap();
    n_ = n_streams;
  }
  ReplaceStreams(ReplaceStreams&& o) noexcept : h_(o.h_), n_(o.n_) { o.h_ = nullptr; }
  ReplaceStreams& operator=(ReplaceStreams&& o) noexcept {
    if (this != &o) { close(); h_ = o.h_; n_ = o.n_; o.h_ = nullptr; }
    return *this;
  }
  ReplaceStreams(const ReplaceStreams&) = delete;
  ReplaceStreams& operator=(const ReplaceStreams&) = delete;
  ~ReplaceStreams() { close(); }

  uint64_t n_streams() const { return n_; }

  Result<std::vector<std::string>> try_feed(std::string_view chunks, const std::vector<uint64_t>& offsets) {
    const uint64_t n_chunks = offsets.empty() ? 0 : offsets.size() - 1;
    const uint64_t span = offsets.empty() ? 0 : offsets.back() - offsets.front();
    return collect(span + span / 8 + 4096, [&](uint8_t* out, uint64_t cap, uint64_t* out_offs, uint64_t* need) {
      return acg_streams_replace_feed(h_, reinterpret_cast<const uint8_t*>(chunks.data()), 0, chunks.size(),
                                      offsets.empty() ? nullptr : offsets.data(), n_chunks, out, cap, out_offs, need);
    }, n_);
  }
  std::vector<std::string> feed(std::string_view chunks, const std::vector<uint64_t>& offsets) {
    return std::move(try_feed(chunks, offsets).unwrap());
  }
  // The held bytes of the given streams, raw, and those streams restarted from zero bytes; flush() takes every
  // stream.
  std::vector<std::string> flush(const std::vector<uint64_t>& ids) {
    if (ids.empty()) return {};
    return std::move(collect(0, [&](uint8_t* out, uint64_t cap, uint64_t* out_offs, uint64_t* need) {
      return acg_streams_flush(h_, ids.data(), ids.size(), out, cap, out_offs, need);
    }, ids.size()).unwrap());
  }
  std::vector<std::string> flush() {
    return std::move(collect(0, [&](uint8_t* out, uint64_t cap, uint64_t* out_offs, uint64_t* need) {
      return acg_streams_flush(h_, nullptr, 0, out, cap, out_offs, need);
    }, n_).unwrap());
  }
  // Restart the given streams from zero bytes, discarding what they hold back; reset() restarts every stream.
  void reset(const std::vector<uint64_t>& ids) {
    if (ids.empty()) return;
    Result<int> r;
    r.error = acg_streams_reset(h_, ids.data(), ids.size());
    r.unwrap();
  }
  void reset() {
    Result<int> r;
    r.error = acg_streams_reset(h_, nullptr, 0);
    r.unwrap();
  }
  // The bytes every stream has received.
  std::vector<uint64_t> positions() const {
    std::vector<uint64_t> pos(n_);
    Result<int> r;
    r.error = acg_streams_positions(h_, pos.data());
    r.unwrap();
    return pos;
  }
  // The bytes every stream holds back: positions() - held() is where its output has reached.
  std::vector<uint64_t> held() const {
    std::vector<uint64_t> h(n_);
    Result<int> r;
    r.error = acg_streams_held(h_, h.data());
    r.unwrap();
    return h;
  }
  // As Streams::lookahead: 1 where feeding the row's stream the candidate would replace a match.
  Result<std::vector<uint8_t>> try_lookahead(const Candidates& cands, const std::vector<uint64_t>& ids = {}) const {
    return detail::lookahead(h_, n_, cands, ids);
  }
  std::vector<uint8_t> lookahead(const Candidates& cands, const std::vector<uint64_t>& ids = {}) const {
    return std::move(try_lookahead(cands, ids).unwrap());
  }
  acg_streams* raw() const { return h_; }

 private:
  // The two-call protocol in output bytes: `call(out, cap, out_offsets, &need)` until it fits, split per entry.
  template <class Call>
  static Result<std::vector<std::string>> collect(uint64_t cap, Call call, uint64_t n_out) {
    Result<std::vector<std::string>> r;
    std::string bytes;
    std::vector<uint64_t> offs(n_out + 1);
    uint64_t need = 0;
    for (;; cap = need) {
      bytes.resize(cap);
      r.error = call(reinterpret_cast<uint8_t*>(bytes.data()), cap, offs.data(), &need);
      if (r.error != ACG_E_OVERFLOW) break;
    }
    if (r.error == 0) {
      r.value.reserve(n_out);
      for (uint64_t i = 0; i < n_out; ++i) r.value.emplace_back(bytes.substr(offs[i], offs[i + 1] - offs[i]));
    }
    return r;
  }
  void close() {
    if (h_) acg_streams_free(h_);
    h_ = nullptr;
  }
  acg_streams* h_ = nullptr;
  uint64_t n_ = 0;
};

template <class Patterns>
AhoCorasick AhoCorasickBuilder::build(const Patterns& patterns) const {
  std::vector<const uint8_t*> ptrs;
  std::vector<uint64_t> lens;
  for (const auto& p : patterns) {
    std::string_view v(p);
    ptrs.push_back(reinterpret_cast<const uint8_t*>(v.data()));
    lens.push_back(v.size());
  }
  acg_dfa* h = nullptr;
  int rc = (device_fill_ ? acg_build_on_device : acg_build)(ptrs.data(), lens.data(), ptrs.size(), &o_, &h);
  if (rc == ACG_E_STATE_ID_OVERFLOW || rc == ACG_E_PATTERN_ID_OVERFLOW || rc == ACG_E_PATTERN_TOO_LONG)
    throw BuildError(rc);
  if (rc) throw DeviceError(rc);
  return AhoCorasick(h);
}

// ---- `aho_corasick::packed`, src/packed/api.rs --------------------------------------------------
namespace packed {

enum class MatchKind : int { LeftmostFirst = ACG_LEFTMOST_FIRST, LeftmostLongest = ACG_LEFTMOST_LONGEST };  // :28-46

class Builder;
class Searcher;

// `packed::Config`, :87-230
class Config {
 public:
  Config() { acg_packed_config_default(&c_); }
  Builder builder() const;                                                                       // :127
  Config& match_kind(MatchKind k) { c_.match_kind = int(k); return *this; }                       // :132
  Config& only_teddy(bool yes) { c_.force = yes ? ACG_PACKED_FORCE_TEDDY : ACG_PACKED_FORCE_NONE; return *this; }  // :143
  Config& only_teddy_fat(std::optional<bool> yes) { c_.only_teddy_fat = yes ? int(*yes) : -1; return *this; }      // :158
  Config& only_teddy_256bit(std::optional<bool> yes) { c_.only_teddy_256bit = yes ? int(*yes) : -1; return *this; }  // :170
  Config& only_rabin_karp(bool yes) { c_.force = yes ? ACG_PACKED_FORCE_RABINKARP : ACG_PACKED_FORCE_NONE; return *this; }  // :181
  Config& heuristic_pattern_limits(bool yes) { c_.heuristic_pattern_limits = yes; return *this; }  // :196
  // not in the reference: decide and build the tables without touching CUDA
  Config& host_only(bool yes) { host_only_ = yes; return *this; }
 private:
  friend class Builder;
  acg_packed_config c_;
  bool host_only_ = false;
};

// `packed::Searcher`, :396-660
class Searcher {
 public:
  Searcher(Searcher&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  Searcher& operator=(Searcher&& o) noexcept {
    if (this != &o) { if (h_) acg_packed_free(h_); h_ = o.h_; o.h_ = nullptr; }
    return *this;
  }
  Searcher(const Searcher&) = delete;
  Searcher& operator=(const Searcher&) = delete;
  ~Searcher() { if (h_) acg_packed_free(h_); }

  template <class Patterns>
  static std::optional<Searcher> create(const Patterns& patterns);  // Searcher::new, :440
  static Config config() { return Config(); }                       // :451
  static Builder builder();                                         // :458

  // find_in, :529 (the span of `in`; anchored / earliest do not exist for packed searchers)
  bool find_in(const Input& in, Match* out) const {
    acg_match m{};
    int found = 0;
    const int rc = acg_packed_find(h_, hay(in), in.haystack().size(), in.start(), in.end(), &m, &found);
    if (rc) Result<int>::throw_error(rc);
    if (found && out) *out = Match(m.pid, m.start, m.end);
    return found != 0;
  }
  bool find(std::string_view haystack, Match* out) const { return find_in(Input(haystack), out); }  // :491
  // find_iter, :580
  MatchIter find_iter(const Input& in) const {
    const uint64_t span_len = in.end() > in.start() ? in.end() - in.start() : 0;
    std::vector<acg_match> buf(std::max<uint64_t>(cap_hint_, span_len / 256 + 64));
    uint64_t n = 0;
    for (;;) {
      const int rc = acg_packed_find_iter(h_, hay(in), in.haystack().size(), in.start(), in.end(), buf.data(),
                                          buf.size(), &n);
      if (rc == ACG_E_OVERFLOW) { cap_hint_ = n + n / 8 + 64; buf.resize(cap_hint_); continue; }
      if (rc) Result<int>::throw_error(rc);
      break;
    }
    std::vector<Match> out;
    out.reserve(n);
    for (uint64_t i = 0; i < n; ++i) out.emplace_back(buf[i].pid, buf[i].start, buf[i].end);
    return MatchIter(std::move(out));
  }
  MatchKind match_kind() const { return MatchKind(acg_packed_match_kind(h_)); }  // :612
  uint64_t minimum_len() const { return acg_packed_minimum_len(h_); }            // :627
  uint64_t memory_usage() const { return acg_packed_memory_usage(h_); }          // :634
  uint64_t patterns_len() const { return acg_packed_patterns_len(h_); }

 private:
  friend class Builder;
  explicit Searcher(acg_packed* h) : h_(h) {}
  static const uint8_t* hay(const Input& in) { return reinterpret_cast<const uint8_t*>(in.haystack().data()); }
  acg_packed* h_ = nullptr;
  mutable uint64_t cap_hint_ = 4096;
};

// `packed::Builder`, :232-357
class Builder {
 public:
  Builder() = default;
  explicit Builder(const Config& c) : cfg_(c) {}
  Builder& add(std::string_view pattern) { pats_.emplace_back(pattern); return *this; }  // :303
  template <class Patterns>
  Builder& extend(const Patterns& patterns) {                                            // :337
    for (const auto& p : patterns) add(std::string_view(p));
    return *this;
  }
  size_t len() const { return pats_.size(); }                                            // :349
  size_t minimum_len() const {                                                           // :354
    size_t m = 0;
    for (size_t i = 0; i < pats_.size(); ++i) m = (i == 0 || pats_[i].size() < m) ? pats_[i].size() : m;
    return m;
  }
  // build, :253: nullopt where the reference returns None
  std::optional<Searcher> build() const {
    std::vector<const uint8_t*> ptrs;
    std::vector<uint64_t> lens;
    for (const auto& p : pats_) {
      ptrs.push_back(reinterpret_cast<const uint8_t*>(p.data()));
      lens.push_back(p.size());
    }
    acg_packed* h = nullptr;
    const int rc = (cfg_.host_only_ ? acg_packed_build_host : acg_packed_build)(ptrs.data(), lens.data(), ptrs.size(),
                                                                                &cfg_.c_, &h);
    if (rc == ACG_E_STATE_ID_OVERFLOW || rc == ACG_E_PATTERN_ID_OVERFLOW || rc == ACG_E_PATTERN_TOO_LONG)
      throw BuildError(rc);
    if (rc) throw DeviceError(rc);
    if (!h) return std::nullopt;
    return Searcher(h);
  }
 private:
  Config cfg_;
  std::vector<std::string> pats_;
};

inline Builder Config::builder() const { return Builder(*this); }
inline Builder Searcher::builder() { return Builder(); }
template <class Patterns>
std::optional<Searcher> Searcher::create(const Patterns& patterns) { return Builder().extend(patterns).build(); }

}  // namespace packed

}  // namespace acb200
