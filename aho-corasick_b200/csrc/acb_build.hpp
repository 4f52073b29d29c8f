// acb_build.hpp -- host-side automaton construction for the GPU search path.
//
// Produces the dense DFA the device kernels consume, with tables that are
// bit-identical to what the reference's own builder produces for the same
// patterns and options (AhoCorasickBuilder::build with kind = DFA:
// src/ahocorasick.rs:2171-2207 -> src/nfa/noncontiguous.rs:963-1051 ->
// src/dfa.rs:431-540).  The implementation is an independent design (explicit
// trie with per-node sorted edge lists, failure links by BFS, DFA rows filled
// by row inheritance from the failure state) -- it shares no code with the
// test oracle under oracle/, which restates the reference's data structures.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace acb {

enum : int { kStandard = 0, kLeftmostFirst = 1, kLeftmostLongest = 2 };
enum : int { kStartUnanchored = 0, kStartAnchored = 1, kStartBoth = 2 };
enum : int { kPreNone = 0, kPreMemmem = 1, kPreStartBytes = 2, kPreRareBytes = 3, kPrePacked = 4 };

struct BuildOptions {
  int match_kind = kStandard;
  int start_kind = kStartUnanchored;
  bool ascii_case_insensitive = false;
  bool byte_classes = true;
  bool prefilter = true;
  int kind = 0;  // AhoCorasickKind requested (0 auto); only reported back
  // Leave the dense table unfilled and describe it by a DenseFillPlan instead (unanchored start
  // kind only; ignored otherwise): the rows are then produced on the device (acb_kernels.cu:
  // dfa_fill_level_kernel), level by level.
  bool defer_dense = false;
};

// Compact description of the dense transition table of src/dfa.rs:544-593 (finish_build_one_start:
// every cell is delta(state, class)), in the row-inheritance form of this builder: row(v) is
// row(fail(v)) -- complete one BFS level earlier -- overlaid with v's own trie edges.
struct DenseFillPlan {
  bool valid = false;
  std::vector<uint32_t> level_off;    // [levels + 1] offsets into the per-row arrays (level 0: the two start rows)
  std::vector<uint32_t> row;          // table row to produce
  std::vector<uint32_t> inherit_row;  // row to copy first, UINT32_MAX: fill with fill_id instead
  std::vector<uint32_t> fill_id;      // premultiplied id for every class when nothing is inherited
  std::vector<uint32_t> edge_off;     // [rows + 1] CSR over the row's own edges
  std::vector<uint8_t> edge_class;
  std::vector<uint32_t> edge_to;      // premultiplied id
  // trie edges that leave nodes of depth < 5, by raw byte (ascending per source row): what the
  // device engine needs to enumerate pattern beginnings without the dense table
  struct ShallowEdge { uint32_t from_row; uint32_t byte; uint32_t to_row; };
  std::vector<ShallowEdge> shallow;
};

// Which packed (Teddy) searcher the reference would construct as a prefilter
// (src/packed/api.rs:253-322, src/packed/teddy/builder.rs:98-231).
struct PackedPlan {
  bool active = false;
  bool fat = false;
  int mask_len = 0;
};

struct HostDfa {
  std::vector<uint32_t> trans;  // premultiplied ids, [state_len << stride2]
  uint32_t stride2 = 0;
  uint32_t alphabet_len = 0;
  uint8_t classes[256] = {0};
  uint32_t max_special_id = 0, max_match_id = 0, start_unanchored_id = 0, start_anchored_id = 0;
  std::vector<uint32_t> match_offsets;  // [num_match_states + 1]
  std::vector<uint32_t> match_pids;
  std::vector<uint32_t> pattern_lens;
  int match_kind = kStandard;
  int start_kind = kStartUnanchored;
  int reported_kind = 3;
  uint64_t min_pattern_len = UINT64_MAX, max_pattern_len = 0;
  uint64_t state_len = 0;
  int prefilter_kind = kPreNone;
  PackedPlan packed;
  // The byte set of the reference's start-bytes / rare-bytes prefilter when it picks one of them
  // (src/util/prefilter.rs:535-575, 784-824): up to three bytes; pre_back[i] = the largest offset at
  // which pre_byte[i] occurs in any pattern (RareByteOffsets, :460-520; 0 for start bytes), i.e. a
  // pattern that shows the byte at haystack offset q starts in [q - pre_back[i], q].
  uint32_t pre_n = 0;
  uint8_t pre_byte[3] = {0, 0, 0};
  uint8_t pre_back[3] = {0, 0, 0};
  // Trie depth of every table row that is reachable from the unanchored start state (0xFFFF for
  // the others), when the builder knows it (unanchored start kind); empty otherwise.  Equals the
  // BFS distance from the start row that acb_api.cu derives for adopted tables.
  std::vector<uint16_t> row_depth;
  uint64_t trans_len = 0;  // state_len << stride2 (== trans.size() unless the fill was deferred)
  DenseFillPlan fill;      // valid => `trans` is empty
};

struct PatternRef {
  const uint8_t* p;
  uint64_t n;
};

// Returns 0 or a negative ACG_E_* build error code.
int build_dfa(const std::vector<PatternRef>& patterns, const BuildOptions& opts, HostDfa* out);

}  // namespace acb
