// Batched find through the C++ facade (include/acb200.hpp): find_batch / try_find_batch on a few documents,
// each checked against try_find on that document alone.  Built with g++ against libacb200.so (or the
// dry-run library) by tests/test_gpu_cpp_find_batch.py.
#include <cstdio>
#include <optional>
#include <string>
#include <tuple>
#include <vector>

#include "acb200.hpp"

using namespace acb200;
using T3 = std::tuple<unsigned, unsigned long, unsigned long>;

static int failures = 0;
#define CHECK(cond)                                                        \
  do {                                                                     \
    if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
  } while (0)

static std::vector<std::optional<T3>> tuples(const std::vector<std::optional<Match>>& v) {
  std::vector<std::optional<T3>> out;
  for (const auto& m : v) {
    if (m) out.emplace_back(T3{m->pattern(), m->start(), m->end()});
    else out.emplace_back(std::nullopt);
  }
  return out;
}

// find_batch against try_find on every document alone
static void check_against_single(const AhoCorasick& ac, const std::string& hay, const std::vector<uint64_t>& offs,
                                 Anchored a, bool earliest) {
  auto got = ac.try_find_batch(hay, offs, a, earliest);
  CHECK(got.is_ok());
  if (!got.is_ok()) return;
  CHECK(got.value.size() == offs.size() - 1);
  for (size_t d = 0; d + 1 < offs.size() && d < got.value.size(); ++d) {
    const std::string doc = hay.substr(offs[d], offs[d + 1] - offs[d]);
    auto one = ac.try_find(Input(doc).anchored(a).earliest(earliest));
    CHECK(one.is_ok());
    CHECK(bool(got.value[d]) == one.value.first);
    if (got.value[d] && one.value.first) {
      CHECK(got.value[d]->pattern() == one.value.second.pattern());
      CHECK(got.value[d]->start() == one.value.second.start());
      CHECK(got.value[d]->end() == one.value.second.end());
    }
  }
}

int main() {
  const std::vector<std::string> patterns = {"abcd", "bc", "ab"};
  const std::string hay = std::string("abcd") + "" + "xxbcx" + "zzz" + "abcab" + "a";
  const std::vector<uint64_t> offs = {0, 4, 4, 9, 12, 17, 18};
  using O = std::optional<T3>;
  {
    AhoCorasick ac = AhoCorasick::create(patterns);  // Standard: the first match state entered
    CHECK(tuples(ac.find_batch(hay, offs)) ==
          (std::vector<O>{T3{2, 0, 2}, std::nullopt, T3{1, 2, 4}, std::nullopt, T3{2, 0, 2}, std::nullopt}));
    check_against_single(ac, hay, offs, Anchored::No, false);
    check_against_single(ac, hay, offs, Anchored::No, true);
    // unanchored-only automaton, anchored input: the error acg_find gives
    auto r = ac.try_find_batch(hay, offs, Anchored::Yes);
    CHECK(r.is_err() && r.error == ACG_E_INVALID_INPUT_ANCHORED);
    CHECK(ac.try_find_batch(hay, {}).is_err());
    CHECK(ac.find_batch(hay, {0}).empty());
  }
  for (MatchKind k : {MatchKind::LeftmostFirst, MatchKind::LeftmostLongest}) {
    AhoCorasick ac = AhoCorasick::builder().match_kind(k).start_kind(StartKind::Both).build(patterns);
    CHECK(tuples(ac.find_batch(hay, offs))[0] == O(T3{0, 0, 4}));  // abcd: listed before ab, and longer
    for (Anchored a : {Anchored::No, Anchored::Yes})
      for (bool earliest : {false, true}) check_against_single(ac, hay, offs, a, earliest);
  }
  if (failures) {
    std::printf("%d checks failed\n", failures);
    return 1;
  }
  std::printf("all checks passed\n");
  return 0;
}
