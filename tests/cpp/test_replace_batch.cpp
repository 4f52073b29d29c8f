// Replace per document through the C++ facade (include/acb200.hpp): replace_all_batch / try_replace_all_batch on a
// few documents, each document checked against the facade's own replace_all_bytes of that document alone.  Built
// with g++ against libacb200.so (or the dry-run library) by tests/test_gpu_cpp_replace.py.
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

// The batch against replace_all_bytes of every document alone
static void check_against_glue(const AhoCorasick& ac, const std::string& hay, const std::vector<uint64_t>& offs,
                               const std::vector<std::string>& reps) {
  auto got = ac.try_replace_all_batch(hay, offs, reps);
  CHECK(got.is_ok());
  if (!got.is_ok()) return;
  const auto& b = got.value;
  CHECK(b.offsets.size() == offs.size() && b.offsets.front() == 0 && b.offsets.back() == b.bytes.size());
  if (b.offsets.size() != offs.size()) return;
  for (size_t d = 0; d + 1 < offs.size(); ++d) {
    const std::string want = ac.replace_all_bytes(std::string_view(hay).substr(offs[d], offs[d + 1] - offs[d]), reps);
    CHECK(b.bytes.substr(b.offsets[d], b.offsets[d + 1] - b.offsets[d]) == want);
  }
}

int main() {
  const std::vector<std::string> app = {"append", "appendage", "app"};
  {
    // src/ahocorasick.rs:651-760 as one-document batches
    AhoCorasick lf = AhoCorasick::builder().match_kind(MatchKind::LeftmostFirst).build(app);
    auto b = lf.replace_all_batch("append the app to the appendage", {0, 31}, std::vector<std::string>{"x", "y", "z"});
    CHECK(b.bytes == "x the z to the xage" && (b.offsets == std::vector<uint64_t>{0, 19}));
    AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{"fox", "brown", "quick"});
    b = ac.replace_all_batch("The quick brown fox.", {0, 20}, std::vector<std::string>{"sloth", "grey", "slow"});
    CHECK(b.bytes == "The slow grey sloth.");
  }
  const std::vector<std::string> patterns = {"abcd", "bc", "ab", "b"};
  const std::string hay = std::string("abcdab") + "" + "xxbcxbc" + "zzz" + "abcabb" + "a";
  const std::vector<uint64_t> offs = {0, 6, 6, 13, 16, 22, 23};
  const std::vector<std::string> reps = {"", "BCBC", "a", "[b]"};
  for (MatchKind k : {MatchKind::Standard, MatchKind::LeftmostFirst, MatchKind::LeftmostLongest}) {
    AhoCorasick ac = AhoCorasick::builder().match_kind(k).build(patterns);
    check_against_glue(ac, hay, offs, reps);
    check_against_glue(ac, hay, offs, std::vector<std::string>{"", "", "", ""});
    check_against_glue(ac, hay, {0}, reps);
    auto r = ac.try_replace_all_batch(hay, offs, std::vector<std::string>{"x"});  // one per pattern
    CHECK(r.is_err() && r.error == ACG_E_INVALID_ARG);
    CHECK(ac.try_replace_all_batch(hay, {}, reps).is_err());
  }
  {
    // the empty pattern: its replacement at every position, into the empty document too
    AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{""});
    auto b = ac.replace_all_batch("abc", {0, 2, 2, 3}, std::vector<std::string>{"-"});
    CHECK(b.bytes == "-a-b---c-" && (b.offsets == std::vector<uint64_t>{0, 5, 6, 9}));
    // an anchored-only automaton: the error of find_iter_batch with unanchored input
    AhoCorasick an = AhoCorasick::builder().start_kind(StartKind::Anchored).build(patterns);
    auto r = an.try_replace_all_batch(hay, offs, reps);
    CHECK(r.is_err() && r.error == ACG_E_INVALID_INPUT_UNANCHORED);
  }
  {
    // an output much longer than the input: the overflow retry of the facade
    AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{"a"});
    const std::string big(10000, 'R');
    auto b = ac.replace_all_batch("aaaa", {0, 1, 4}, std::vector<std::string>{big});
    CHECK(b.bytes == big + big + big + big && (b.offsets == std::vector<uint64_t>{0, 10000, 40000}));
  }
  if (failures) {
    std::printf("%d checks failed\n", failures);
    return 1;
  }
  std::printf("all checks passed\n");
  return 0;
}
