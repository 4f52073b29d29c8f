// Lookahead through the C++ facade (include/acb200.hpp): acb200::Candidates and lookahead() on Streams and
// ReplaceStreams, every bit checked against a twin set with the same history that is fed the candidate.  Built with
// g++ against libacb200.so (or the dry-run library) by tests/test_gpu_cpp_lookahead.py.
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

static std::string join(const std::vector<std::string>& v, std::vector<uint64_t>& offs) {
  std::string s;
  offs.assign(1, 0);
  for (const std::string& x : v) {
    s += x;
    offs.push_back(s.size());
  }
  return s;
}

// For every candidate, a twin find_iter / overlapping set fed `history` and then the candidate on every stream:
// the streams it returns matches for are that candidate's column.
static void check_against_twins(const AhoCorasick& ac, const std::vector<std::string>& history, bool overlapping,
                                const std::vector<std::string>& cands, const std::vector<uint8_t>& mask) {
  const size_t n = history.size();
  for (size_t c = 0; c < cands.size(); ++c) {
    Streams twin(ac, n, overlapping);
    std::vector<uint64_t> offs;
    const std::string h = join(history, offs);
    twin.feed(h, offs);
    const std::string again = join(std::vector<std::string>(n, cands[c]), offs);
    const auto got = twin.feed(again, offs);
    for (size_t s = 0; s < n; ++s) CHECK((mask[s * cands.size() + c] != 0) == !got[s].empty());
  }
}

int main() {
  AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{"abc", "bcd", "zz", "hello world"});
  const std::vector<std::string> history = {"abc", "xbc", "", "hello wor", "z", "abcab"};
  const std::vector<std::string> cands = {"d", "", "bcd", "ld", "z", "c", "q", "hello world", "zzz"};
  Candidates cs(ac, cands);
  CHECK(cs.size() == cands.size());
  std::vector<uint64_t> offs;
  const std::string h = join(history, offs);
  for (bool overlapping : {false, true}) {
    Streams set(ac, history.size(), overlapping);
    set.feed(h, offs);
    const std::vector<uint64_t> pos = set.positions();
    const std::vector<uint8_t> mask = set.lookahead(cs);
    CHECK(mask.size() == history.size() * cands.size());
    check_against_twins(ac, history, overlapping, cands, mask);
    // {"abc", "bcd"}, stream fed "abc", candidate "d": only overlapping mode sees bcd
    CHECK(mask[0 * cands.size() + 0] == (overlapping ? 1 : 0));
    // rows by id: duplicates and any order
    const std::vector<uint8_t> some = set.lookahead(cs, {5, 0, 5});
    for (size_t c = 0; c < cands.size(); ++c) {
      CHECK(some[c] == mask[5 * cands.size() + c]);
      CHECK(some[cands.size() + c] == mask[c]);
      CHECK(some[2 * cands.size() + c] == mask[5 * cands.size() + c]);
    }
    CHECK(set.try_lookahead(cs, {6}).error == ACG_E_INVALID_ARG);
    CHECK(set.positions() == pos);
  }
  {
    // a replace set's bits are its find_iter matches
    ReplaceStreams rs(ac, history.size(), std::vector<std::string>{"1", "2", "3", "4"});
    Streams fi(ac, history.size());
    rs.feed(h, offs);
    fi.feed(h, offs);
    CHECK(rs.lookahead(cs) == fi.lookahead(cs));
    const std::vector<uint64_t> held = rs.held();
    rs.lookahead(cs);
    CHECK(rs.held() == held);
  }
  {
    // a candidate set of another automaton
    AhoCorasick other = AhoCorasick::create(std::vector<std::string>{"abc"});
    Candidates foreign(other, cands);
    Streams set(ac, 2);
    CHECK(set.try_lookahead(foreign).error == ACG_E_INVALID_ARG);
  }
  if (failures) return 1;
  std::printf("all checks passed\n");
  return 0;
}
