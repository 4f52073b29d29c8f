// Match coverage through the C++ facade (include/acb200.hpp): match_coverage_batch / try_match_coverage_batch on
// a few documents, each document checked against the facade's own per-document records.  Built with g++ against
// libacb200.so (or the dry-run library) by tests/test_gpu_cpp_match_coverage.py.
#include <cstdio>
#include <string>
#include <vector>

#include "acb200.hpp"

using namespace acb200;

static int failures = 0;
#define CHECK(cond)                                                        \
  do {                                                                     \
    if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
  } while (0)

// The coverage and the mask against the union of the batch records of the same call, taken here
static void check_against_records(const AhoCorasick& ac, const std::string& hay, const std::vector<uint64_t>& offs,
                                  bool overlapping, Anchored a) {
  auto got = ac.try_match_coverage_batch(hay, offs, overlapping, a, true);
  auto rec = overlapping ? ac.try_find_overlapping_iter_batch(hay, offs, a) : ac.try_find_iter_batch(hay, offs, a);
  CHECK(got.is_ok() && rec.is_ok());
  if (!got.is_ok() || !rec.is_ok()) return;
  const auto& c = got.value;
  CHECK(c.covered.size() + 1 == offs.size() && c.mask.size() == hay.size());
  std::vector<uint8_t> want(hay.size(), 0);
  for (size_t d = 0; d + 1 < offs.size(); ++d)
    for (const Match& m : rec.value[d])
      for (uint64_t i = offs[d] + m.start(); i < offs[d] + m.end(); ++i) want[i] = 1;
  CHECK(c.mask == want);
  for (size_t d = 0; d + 1 < offs.size(); ++d) {
    uint64_t n = 0;
    for (uint64_t i = offs[d]; i < offs[d + 1]; ++i) n += want[i];
    CHECK(c.covered[d] == n);
  }
  auto no_mask = ac.match_coverage_batch(hay, offs, overlapping, a);
  CHECK(no_mask.covered == c.covered && no_mask.mask.empty());
}

int main() {
  const std::vector<std::string> patterns = {"abcd", "bc", "ab", "b"};
  const std::string hay = std::string("abcdab") + "" + "xxbcxbc" + "zzz" + "abcabb" + "a";
  const std::vector<uint64_t> offs = {0, 6, 6, 13, 16, 22, 23};
  {
    AhoCorasick ac = AhoCorasick::create(patterns);
    // overlapping: abcdab is covered entirely; xxbcxbc in bc twice; abcabb in ab, bc, ab, b
    auto c = ac.match_coverage_batch(hay, offs, true, Anchored::No, true);
    CHECK((c.covered == std::vector<uint64_t>{6, 0, 4, 0, 6, 0}));
    for (bool ov : {false, true}) check_against_records(ac, hay, offs, ov, Anchored::No);
    // unanchored-only automaton, anchored input: the error of the batch call
    auto r = ac.try_match_coverage_batch(hay, offs, false, Anchored::Yes);
    CHECK(r.is_err() && r.error == ACG_E_INVALID_INPUT_ANCHORED);
    CHECK(ac.try_match_coverage_batch(hay, {}).is_err());
    auto none = ac.match_coverage_batch(hay, {0}, false, Anchored::No, true);
    CHECK(none.covered.empty() && none.mask == std::vector<uint8_t>(hay.size(), 0));
  }
  for (MatchKind k : {MatchKind::LeftmostFirst, MatchKind::LeftmostLongest}) {
    AhoCorasick ac = AhoCorasick::builder().match_kind(k).start_kind(StartKind::Both).build(patterns);
    auto r = ac.try_match_coverage_batch(hay, offs, true);
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
