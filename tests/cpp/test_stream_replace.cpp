// Replace sets through the C++ facade (include/acb200.hpp): acb200::ReplaceStreams fed a few streams chunk by
// chunk, each stream's outputs over all its feeds and its flush checked against the facade's replace_all_bytes of
// the concatenated stream, and every output checked to end at the stream's emit boundary (positions - held).
// Built with g++ against libacb200.so (or the dry-run library) by tests/test_gpu_cpp_stream_replace.py.
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

// Deal every stream into chunks of 0 to 6 bytes, feed them, flush, and compare with replace_all_bytes.
static void check_streams(const AhoCorasick& ac, const std::vector<std::string>& streams,
                          const std::vector<std::string>& reps) {
  ReplaceStreams set(ac, streams.size(), reps);
  std::vector<std::string> got(streams.size());
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
    const std::vector<uint64_t> pos = set.positions(), held = set.held();
    for (size_t s = 0; s < streams.size(); ++s) {
      got[s] += r.value[s];
      CHECK(pos[s] == at[s]);
      CHECK(held[s] <= ac.max_pattern_len() - 1);
      // everything before the emit boundary is settled: what is out is the replacement of exactly that prefix
      CHECK(got[s] == ac.replace_all_bytes(streams[s].substr(0, pos[s] - held[s]), reps));
    }
  }
  const std::vector<std::string> tails = set.flush();
  CHECK(tails.size() == streams.size());
  for (size_t s = 0; s < streams.size() && s < tails.size(); ++s)
    CHECK(got[s] + tails[s] == ac.replace_all_bytes(streams[s], reps));
  CHECK((set.positions() == std::vector<uint64_t>(streams.size(), 0)));
}

int main() {
  AhoCorasick ac = AhoCorasick::create(std::vector<std::string>{"abcab", "bca", "ab", "zzzz", "the lazy dog"});
  const std::vector<std::string> reps = {"<1>", "", "AB", "zz", "[the sleepy cat]"};
  const std::vector<std::string> streams = {"xxabcabcabzzzzzz", "", "the lazy dog and the lazy dog", "zzabcabzz" "zz"};
  check_streams(ac, streams, reps);
  {
    ReplaceStreams set(ac, 2, reps);
    // "the lazy d" is held back whole; "abc" is out but "ab" could still become "abcab"
    auto r = set.feed("xabcthe lazy d", {0, 4, 14});
    CHECK(r[0] == "xAB" && r[1] == "");
    CHECK((set.held() == std::vector<uint64_t>{1, 10}));
    // "bca" would start before the restart point of find_iter: no match, and "ca" is held
    auto r2 = set.feed("aog", {0, 1, 3});
    CHECK(r2[0] == "" && r2[1] == "[the sleepy cat]");
    CHECK((set.held() == std::vector<uint64_t>{2, 0}));
    // flush of one stream: its held bytes raw, then it starts again
    auto f = set.flush(std::vector<uint64_t>{0});
    CHECK(f.size() == 1 && f[0] == "ca");
    CHECK((set.positions() == std::vector<uint64_t>{0, 12}));
    set.reset();
    CHECK((set.positions() == std::vector<uint64_t>{0, 0}));
    // one chunk per stream; a duplicate flush id
    CHECK(set.try_feed("abc", {0, 3}).error == ACG_E_INVALID_ARG);
    bool threw = false;
    try {
      set.flush(std::vector<uint64_t>{1, 1});
    } catch (const DeviceError&) {
      threw = true;
    }
    CHECK(threw);
  }
  {
    bool threw = false;
    try {
      ReplaceStreams set(ac, 1, std::vector<std::string>{"x"});  // one replacement for five patterns
    } catch (const DeviceError&) {
      threw = true;
    }
    CHECK(threw);
  }
  if (failures) return 1;
  std::printf("all checks passed\n");
  return 0;
}
