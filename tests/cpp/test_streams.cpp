// Stream sets through the C++ facade (include/acb200.hpp): acb200::Streams fed a few streams chunk by chunk, each
// stream's matches over all its feeds checked against the facade's find_iter / find_overlapping_iter over the
// concatenated stream.  Built with g++ against libacb200.so (or the dry-run library) by
// tests/test_gpu_cpp_streams.py.
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

static bool same(const std::vector<Match>& a, const std::vector<Match>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); ++i)
    if (a[i].pattern() != b[i].pattern() || a[i].start() != b[i].start() || a[i].end() != b[i].end()) return false;
  return true;
}

// Deal every stream into chunks of 0 to 6 bytes, feed them, and compare with the whole-stream iterator.
static void check_streams(const AhoCorasick& ac, const std::vector<std::string>& streams, bool overlapping) {
  Streams set(ac, streams.size(), overlapping);
  std::vector<std::vector<Match>> got(streams.size());
  std::vector<size_t> at(streams.size(), 0);
  unsigned seed = 7;
  for (bool more = true; more;) {
    more = false;
    std::string chunks;
    std::vector<uint64_t> offs{0};
    for (size_t s = 0; s < streams.size(); ++s) {
      seed = seed * 1103515245u + 12345u;
      const size_t k = std::min<size_t>((seed >> 16) % 7, streams[s].size() - at[s]);
      chunks += streams[s].substr(at[s], k);
      at[s] += k;
      offs.push_back(chunks.size());
      more |= at[s] < streams[s].size();
    }
    auto r = set.try_feed(chunks, offs);
    CHECK(r.is_ok());
    if (!r.is_ok()) return;
    for (size_t s = 0; s < streams.size(); ++s)
      for (const Match& m : r.value[s]) got[s].push_back(m);
  }
  const std::vector<uint64_t> pos = set.positions();
  for (size_t s = 0; s < streams.size(); ++s) {
    CHECK(pos[s] == streams[s].size());
    const std::vector<Match> want =
        overlapping ? ac.find_overlapping_iter(Input(streams[s])).collect() : ac.find_iter(Input(streams[s])).collect();
    CHECK(same(got[s], want));
  }
}

int main() {
  AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{"abcab", "bca", "ab", "zzzz", "the lazy dog"});
  const std::vector<std::string> streams = {"xxabcabcabzzzzzz", "", "the lazy dog and the lazy dog", "zzabcabzz" "zz"};
  check_streams(ac, streams, false);
  check_streams(ac, streams, true);
  {
    // reset: a stream starts again from zero bytes; the others go on
    Streams set(ac, 2);
    set.feed("abcthe la", {0, 3, 9});
    set.reset(std::vector<uint64_t>{0});
    auto r = set.feed("bcazy dog", {0, 3, 9});
    CHECK(r[0].size() == 1 && r[0][0].start() == 0 && r[0][0].end() == 3);
    CHECK(r[1].size() == 1 && r[1][0].start() == 0 && r[1][0].end() == 12);
    CHECK((set.positions() == std::vector<uint64_t>{3, 12}));
    set.reset();
    CHECK((set.positions() == std::vector<uint64_t>{0, 0}));
    // one chunk per stream
    auto bad = set.try_feed("abc", {0, 3});
    CHECK(bad.error == ACG_E_INVALID_ARG);
  }
  {
    bool threw = false;
    AhoCorasick lf = AhoCorasick::builder().match_kind(MatchKind::LeftmostFirst).build(std::vector<std::string>{"a"});
    try {
      Streams set(lf, 1);
    } catch (const MatchError&) {
      threw = true;
    }
    CHECK(threw);
  }
  if (failures) return 1;
  std::printf("all checks passed\n");
  return 0;
}
