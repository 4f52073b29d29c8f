/*
 * ac_oracle.h -- CPU oracle for the GPU Aho-Corasick hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a plain-C restatement of the reference
 * algorithm (BurntSushi/aho-corasick 1.1.3) for the DFA-scan / packed hot path.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference leg may load it -- and there only as the checker / CPU comparator,
 * never as the thing shipped.  The product (aho-corasick_b200/) has its own,
 * independent builder and never links or calls anything in this directory.
 *
 * Parity status: PINNED against the reference's own golden vectors
 * (src/tests.rs:96-642, src/packed/tests.rs:129-368 incl. the 3x261 "Z"
 * padding variations, README/doc examples) via tests/test_oracle_golden.py.
 * The reference itself (Rust) is not built, so there is no oracle/_ref.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * the root of the reference crate).
 */
#ifndef AC_ORACLE_H
#define AC_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* src/util/search.rs:1052 (MatchKind), :1133 (StartKind) */
enum { ORC_STANDARD = 0, ORC_LEFTMOST_FIRST = 1, ORC_LEFTMOST_LONGEST = 2 };
enum { ORC_START_UNANCHORED = 0, ORC_START_ANCHORED = 1, ORC_START_BOTH = 2 };
/* src/ahocorasick.rs:2624 (AhoCorasickKind); 0 = auto (build_auto :2213) */
enum { ORC_KIND_AUTO = 0, ORC_KIND_NFA = 1, ORC_KIND_CONTIGUOUS = 2, ORC_KIND_DFA = 3 };
/* which prefilter the reference would construct, src/util/prefilter.rs:163-305 */
enum { ORC_PRE_NONE = 0, ORC_PRE_MEMMEM = 1, ORC_PRE_START_BYTES = 2,
       ORC_PRE_RARE_BYTES = 3, ORC_PRE_PACKED = 4 };

/* error codes: src/util/error.rs:23-49 (build), :200-223 (match) */
enum {
  ORC_OK = 0,
  ORC_E_STATE_ID_OVERFLOW = -1,
  ORC_E_PATTERN_ID_OVERFLOW = -2,
  ORC_E_PATTERN_TOO_LONG = -3,
  ORC_E_INVALID_INPUT_ANCHORED = -10,
  ORC_E_INVALID_INPUT_UNANCHORED = -11,
  ORC_E_UNSUPPORTED_STREAM = -12,
  ORC_E_UNSUPPORTED_OVERLAPPING = -13,
  ORC_E_UNSUPPORTED_EMPTY = -14,
  ORC_E_INVALID_SPAN = -20,
  ORC_E_OVERFLOW = -21,
  ORC_E_UNSUPPORTED_KIND = -22
};

typedef struct {
  int match_kind;             /* default Standard */
  int start_kind;             /* default Unanchored */
  int ascii_case_insensitive; /* default 0 */
  int byte_classes;           /* default 1 */
  int prefilter;              /* default 1 */
  int kind;                   /* default ORC_KIND_AUTO */
  int64_t dense_depth;        /* default 3; <0 means usize::MAX */
} orc_opts;

typedef struct {
  uint32_t pid;
  uint32_t _pad;
  uint64_t start;
  uint64_t end;
} orc_match;

typedef struct orc_ac orc_ac;

void orc_opts_default(orc_opts* o);

/* AhoCorasickBuilder::build, src/ahocorasick.rs:2171-2207 */
int orc_build(const uint8_t* const* pats, const size_t* lens, size_t n,
              const orc_opts* opts, orc_ac** out);
void orc_free(orc_ac* ac);

/* getters, src/ahocorasick.rs:1867-2021 */
int orc_kind(const orc_ac* ac);        /* ORC_KIND_NFA or ORC_KIND_DFA (contiguous is not restated; auto falls to NFA search semantics) */
int orc_match_kind(const orc_ac* ac);
int orc_start_kind(const orc_ac* ac);
size_t orc_patterns_len(const orc_ac* ac);
size_t orc_min_pattern_len(const orc_ac* ac);
size_t orc_max_pattern_len(const orc_ac* ac);
int orc_prefilter_kind(const orc_ac* ac);
/* 1 if the packed prefilter would be Teddy; *fat, *mask_len filled (src/packed/teddy/builder.rs:98-231) */
int orc_packed_variant(const orc_ac* ac, int* fat, int* mask_len, int* vbytes);

/* DFA table view (valid only when orc_kind()==ORC_KIND_DFA), src/dfa.rs:91-132 */
typedef struct {
  const uint32_t* trans;
  uint64_t trans_len;
  uint32_t stride2;
  uint32_t alphabet_len;
  const uint8_t* byte_classes;   /* [256] */
  uint32_t max_special_id, max_match_id, start_unanchored_id, start_anchored_id;
  const uint32_t* match_offsets; /* [num_match_states + 1] */
  const uint32_t* match_pids;
  uint32_t num_match_states;
  const uint32_t* pattern_lens;
  uint32_t n_patterns;
  uint32_t match_kind;
  uint64_t min_pattern_len, max_pattern_len;
  uint64_t state_len;
} orc_dfa_view;
int orc_dfa_get(const orc_ac* ac, orc_dfa_view* v);

/* AhoCorasick::try_find, src/ahocorasick.rs:1021 -> src/automaton.rs:1259-1420 */
int orc_try_find(const orc_ac* ac, const uint8_t* hay, size_t hay_len,
                 size_t span_start, size_t span_end, int anchored, int earliest,
                 orc_match* out, int* found);
/* AhoCorasick::try_find_iter, src/ahocorasick.rs:1275 -> src/automaton.rs:844-936.
 * Returns ORC_E_OVERFLOW (with *n_out = required count) if cap is too small. */
int orc_find_iter(const orc_ac* ac, const uint8_t* hay, size_t hay_len,
                  size_t span_start, size_t span_end, int anchored,
                  orc_match* out, size_t cap, size_t* n_out);
/* AhoCorasick::try_find_overlapping_iter, src/ahocorasick.rs:1350 ->
 * src/automaton.rs:397-423, 954-970, 1423-1537 */
int orc_find_overlapping_iter(const orc_ac* ac, const uint8_t* hay, size_t hay_len,
                              size_t span_start, size_t span_end, int anchored,
                              orc_match* out, size_t cap, size_t* n_out);

/* Raw DFA scan loops used as the CPU baseline (count-only; no iterator
 * overhead): one pass of src/automaton.rs:1491-1534 over [start,end) reporting
 * the number of matches and an FNV-1a checksum of the (pid,start,end) stream. */
int orc_scan_overlapping_count(const orc_ac* ac, const uint8_t* hay, size_t hay_len,
                               size_t span_start, size_t span_end,
                               uint64_t* n_matches, uint64_t* fnv);

/* ---- packed (src/packed/api.rs) ------------------------------------- */
enum { ORC_PACKED_LEFTMOST_FIRST = 0, ORC_PACKED_LEFTMOST_LONGEST = 1 };
enum { ORC_FORCE_NONE = 0, ORC_FORCE_TEDDY = 1, ORC_FORCE_RABINKARP = 2 };
typedef struct {
  int kind;
  int force;                    /* ForceAlgorithm, api.rs:143-199 */
  int only_teddy_fat;           /* -1 None, 0 Some(false), 1 Some(true) */
  int only_teddy_256bit;        /* -1 None, 0 Some(false), 1 Some(true) */
  int heuristic_pattern_limits; /* default 1 */
} orc_packed_config;
typedef struct orc_packed orc_packed;
void orc_packed_config_default(orc_packed_config* c);
/* packed::Builder::build, api.rs:253-282. Returns NULL in *out when the reference returns None. */
int orc_packed_build(const uint8_t* const* pats, const size_t* lens, size_t n,
                     const orc_packed_config* cfg, orc_packed** out);
void orc_packed_free(orc_packed* p);
size_t orc_packed_minimum_len(const orc_packed* p);
/* Searcher::find_in, api.rs:529-546 */
int orc_packed_find_in(const orc_packed* p, const uint8_t* hay, size_t hay_len,
                       size_t span_start, size_t span_end, orc_match* out, int* found);
/* Searcher::find_iter, api.rs:548-556 + FindIter :661-687 */
int orc_packed_find_iter(const orc_packed* p, const uint8_t* hay, size_t hay_len,
                         orc_match* out, size_t cap, size_t* n_out);

#ifdef __cplusplus
}
#endif
#endif
