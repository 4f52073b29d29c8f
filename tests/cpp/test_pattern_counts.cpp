// Pattern counts through the C++ facade (include/acb200.hpp): pattern_counts_batch / try_pattern_counts_batch
// on a few documents, each row checked against the facade's own per-document records.  Built with g++ against
// libacb200.so (or the dry-run library) by tests/test_gpu_cpp_pattern_counts.py.
#include <cstdio>
#include <map>
#include <string>
#include <vector>

#include "acb200.hpp"

using namespace acb200;

static int failures = 0;
#define CHECK(cond)                                                        \
  do {                                                                     \
    if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
  } while (0)

// The counts against the batch records of the same call, grouped here
static void check_against_records(const AhoCorasick& ac, const std::string& hay, const std::vector<uint64_t>& offs,
                                  bool overlapping, Anchored a) {
  auto got = ac.try_pattern_counts_batch(hay, offs, overlapping, a);
  auto rec = overlapping ? ac.try_find_overlapping_iter_batch(hay, offs, a) : ac.try_find_iter_batch(hay, offs, a);
  CHECK(got.is_ok() && rec.is_ok());
  if (!got.is_ok() || !rec.is_ok()) return;
  const auto& c = got.value;
  CHECK(c.row_offsets.size() == offs.size());
  CHECK(c.row_offsets.front() == 0 && c.row_offsets.back() == c.pids.size() && c.pids.size() == c.counts.size());
  for (size_t d = 0; d + 1 < offs.size(); ++d) {
    std::map<uint32_t, uint64_t> want;
    for (const Match& m : rec.value[d]) ++want[m.pattern()];
    std::map<uint32_t, uint64_t> row;
    for (uint64_t i = c.row_offsets[d]; i < c.row_offsets[d + 1]; ++i) {
      if (i > c.row_offsets[d]) CHECK(c.pids[i] > c.pids[i - 1]);
      row[c.pids[i]] = c.counts[i];
    }
    CHECK(row == want);
  }
}

int main() {
  const std::vector<std::string> patterns = {"abcd", "bc", "ab", "b"};
  const std::string hay = std::string("abcdab") + "" + "xxbcxbc" + "zzz" + "abcabb" + "a";
  const std::vector<uint64_t> offs = {0, 6, 6, 13, 16, 22, 23};
  {
    AhoCorasick ac = AhoCorasick::create(patterns);
    // overlapping: abcdab = abcd, bc, ab x2, b x2
    auto c = ac.pattern_counts_batch(hay, offs, true);
    CHECK((c.row_offsets == std::vector<uint64_t>{0, 4, 4, 6, 6, 9, 9}));
    CHECK((std::vector<uint32_t>(c.pids.begin(), c.pids.begin() + 4) == std::vector<uint32_t>{0, 1, 2, 3}));
    CHECK((std::vector<uint64_t>(c.counts.begin(), c.counts.begin() + 4) == std::vector<uint64_t>{1, 1, 2, 2}));
    for (bool ov : {false, true}) check_against_records(ac, hay, offs, ov, Anchored::No);
    // unanchored-only automaton, anchored input: the error of the batch call
    auto r = ac.try_pattern_counts_batch(hay, offs, false, Anchored::Yes);
    CHECK(r.is_err() && r.error == ACG_E_INVALID_INPUT_ANCHORED);
    CHECK(ac.try_pattern_counts_batch(hay, {}).is_err());
    auto none = ac.pattern_counts_batch(hay, {0});
    CHECK(none.row_offsets == std::vector<uint64_t>{0} && none.pids.empty() && none.counts.empty());
  }
  for (MatchKind k : {MatchKind::LeftmostFirst, MatchKind::LeftmostLongest}) {
    AhoCorasick ac = AhoCorasick::builder().match_kind(k).start_kind(StartKind::Both).build(patterns);
    auto r = ac.try_pattern_counts_batch(hay, offs, true);
    CHECK(r.is_err() && r.error == ACG_E_UNSUPPORTED_OVERLAPPING);
    for (Anchored a : {Anchored::No, Anchored::Yes}) check_against_records(ac, hay, offs, false, a);
  }
  if (failures) {
    std::printf("%d checks failed\n", failures);
    return 1;
  }
  std::printf("all checks passed\n");
  return 0;
}
