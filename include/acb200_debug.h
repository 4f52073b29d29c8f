/*
 * acb200_debug.h -- introspection of the device engine's derived tables (libacb200.so).
 *
 * Test infrastructure, not part of the drop-in boundary (include/acb200.h): it lets the CPU test
 * suite check the contract between the host-side table construction and the kernels' probe
 * functions (no false negatives in the fingerprint bitmap, anchor map == DFA walk) on handles
 * built without a GPU (acg_build_host).
 */
#ifndef ACB200_DEBUG_H
#define ACB200_DEBUG_H

#include "acb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int32_t supported; /* 0: the automaton runs on the walk / sequential engines only */
  int32_t brute;     /* fingerprints not selective: every offset is verified */
  int32_t dense;     /* > 8192 fingerprints: survivors are compacted through the anchor map */
  int32_t stride;    /* 1 or 2 (first-stage probe stride) */
  int32_t wide;      /* stride 2 only: 2 KiB tiles, 16 KiB bitmap */
  uint32_t k;        /* fingerprint length in bytes, 1..4 */
  uint32_t kmask, fold, mult, mult3, shift, log_bits;
  const uint32_t* bitmap; /* 1 << (log_bits - 5) words, borrowed until acg_dfa_free */
  uint64_t bitmap_words;
  const uint64_t* amap;   /* 1 << amap_log entries: low word key, high word premultiplied state id */
  uint32_t amap_log;
  const uint16_t* depth16; /* trie depth per table row */
  uint64_t n_rows;
  uint32_t dup_shift;      /* tie-break layout: (max_len - len) << dup_shift | index among equal patterns */
  uint32_t key_shift;      /* stride 2: first-stage hash = window * (mult3 << key_shift); 5, or 8 with ACG_EXP_KEY24 */
  uint32_t bs_n;           /* byte-set scan (start-bytes / rare-bytes role): number of needles, 0 = fingerprint filter */
  uint8_t bs_byte[3];
  uint8_t bs_back[3];      /* largest offset of the needle in any pattern (0 for start bytes) */
} acg_prefilter_plan;

/* Fills *out with views of the handle's derived tables.  Works on host-only handles. */
int acg_debug_prefilter_plan(const acg_dfa* dfa, acg_prefilter_plan* out);

/* Size of the H2D chunks of the pipelined host path (default 64 MiB; a multiple of 4096).  Lets
 * tests exercise the multi-chunk logic on small inputs. */
int acg_debug_set_pipeline_chunk(acg_dfa* dfa, uint64_t bytes);

/* Kernel / plan variants that never change results, only which instantiation of the prefilter kernel
 * runs or how its first-stage keys are formed; kept switchable so that tools/ab_inproc.py can time
 * them against each other in one process.  (Earlier variants TALL = 1, PAIR = 2, WALK_HOT = 4 and
 * LOCAL2 = 16, and an anchor-map second stage for the stride-2 kernel, lost such comparisons and
 * are gone.) */
#define ACG_EXP_KEY24 8u         /* stride-2 first stage keyed by the 3 fingerprint bytes only; default: 27 bits (3 bytes +
                                  * low 3 bits of the fourth).  Rebuilds the bitmap. */
#define ACG_EXP_STATIC_TILES 32u /* warp w of a CTA takes tiles w, w + W, ...; default: the warps of a CTA draw their tiles
                                  * from a shared-memory counter. */
#define ACG_EXP_GLOBAL_TILES 16u  /* tiles numbered over the whole region, super-tiles per CTA from a global counter */
#define ACG_EXP_NO_BYTESCAN 64u  /* automata with a start-bytes / rare-bytes set: use the fingerprint filter anyway */
int acg_debug_set_experiment(acg_dfa* dfa, uint32_t flags);

#ifdef __cplusplus
}
#endif
#endif
