"""The prefilter kernels against the oracle on bytes outside printable ASCII.

Every other kernel-level suite draws its patterns and haystacks from printable ASCII (0x20 .. 0x7E), yet
several steps of the plan and the kernels depend on byte content: the case fold x | 0x20 (which also
merges @ / `, [ / {, \\ / |, ] / }, ^ / ~, _ / DEL and every high byte with its partner 0x20 away, while
the verifier's case insensitivity covers letters only), the fold the plan applies to a case-sensitive
automaton whose spellings collapse, the low 3 bits of the fourth window byte in the 27-bit stride-2 keys,
the start-state walk the verifier takes when a plan ships no anchor map, and the SWAR compare of the
byte-set scan, which flags a byte equal to needle ^ 0x01 just above a needle as well (the exact verifier
drops it).  The families of tests/byte_families.py put those bytes in front of every variant:

  high bytes     0x80 .. 0xFF     stride-2 narrow, stride-2 wide, dense, stride 1 with k = 3 and k = 2
                                  (masked), and k = 1, which is always brute mode: the plan's estimate
                                  of the 1-gram pass rate is the set size over the bytes seen, i.e. 1
  full range     0x00 .. 0xFF     stride-2 narrow, stride-2 wide, dense, stride 1 with k = 3
  fold mix       CI, letters + fold-pair non-letters + high bytes: stride-2 narrow and dense, fold != 0
  spellings      case-sensitive, three spellings a word: stride 1, k = 4, fold != 0
  4-byte keys    4-byte patterns and their 5-byte continuations: stride 2, 27-bit and 24-bit keys
  no anchor map  270 000 CI patterns with distinct first four letters (16 trie paths each, over the
                 4 Mi an anchor map holds): brute mode with no map.  The dense variant without a map
                 cannot be reached: more than 4 Mi fingerprints (or 262 144 folded 4-grams of letters,
                 whose own pass rate is over a half) saturate the blocked filter, and the plan goes brute
  needles        rare-bytes prefilter with first-byte needles 0xFF, 0x00, 0x7F: the byte-set scan, then
                 retired; four needles as the control (bs_n == 0).  A 0xFF needle needs the pattern
                 b"\\xff" (0xFF is the most common byte by the reference's ranks), so k = 1 and the kernel
                 behind the scan is brute mode
  256 columns    byte_classes(false) on the high-byte sets: narrow, wide, dense
  StartKind::Both, searched unanchored, on the high-byte narrow set.

Each row asserts the plan it gets (so its id names the kernel that ran) and compares, tuple for tuple and
in order, with the oracle built with the same knobs: find_overlapping_iter (Standard) and find_iter of its
match kinds at pointer phases 0, 1 and 13 into one device buffer and on an odd sub-span whose ends lie
inside planted patterns; try_find and is_match on both spans; one batched call over documents whose
bounds fall inside planted patterns.  The haystack is drawn from the family's own byte distribution;
planted into it are every pattern (where there is room) at starts that cover every residue mod 32 and
every 16-byte group of a 2 KiB tile, decoys the verifier must reject (a byte swapped for its fold partner
or for another case spelling, the last byte changed, bits 3 .. 7 of the fourth or fifth byte changed, runs
of needle, needle ^ 0x01) and a pattern cut off by the end of the buffer.

Under the dry run (ACB_EMULATE=1, tests/emu/) the same tests run on the CPU build at reduced sizes."""
import functools
import time
from types import SimpleNamespace

import numpy as np
import pytest

import aho_corasick_b200 as ab
import byte_families as F
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import sampled_docs_match_the_oracle
from test_gpu_kernel_matrix import KEY24, ON_GPU
from test_gpu_parity import assert_np_equal, to_device
from test_prefilter_plan import plan_of, set_experiment

# one haystack per row: 64 MiB + an odd remainder on the device, 512 KiB + the same on the dry run
N = ((64 << 20) if ON_GPU else (512 << 10)) + 4093
NO_AMAP_N = ((4 << 20) if ON_GPU else (64 << 10)) + 4093
NO_AMAP_PATTERNS = 270000
PHASES = (0, 1, 13)
PREFILTER = int(ab.Engine.Prefilter)


def _pats(name):
    return {
        "high-narrow": lambda: F.high(5000, 0xB1), "high-wide": lambda: F.high(50, 0xB2),
        "high-dense": lambda: F.high(20000, 0xB3), "high-k3": lambda: F.high(300, 0xB4, 3, 12),
        "high-k2": lambda: F.high(300, 0xB5, 2, 12), "high-k1": lambda: F.high(300, 0xB6, 1, 12),
        "full-narrow": lambda: F.full(5000, 0xF1), "full-wide": lambda: F.full(50, 0xF2),
        "full-dense": lambda: F.full(20000, 0xF3), "full-k3": lambda: F.full(300, 0xF4, 3, 12),
        "fold-narrow": lambda: F.fold_mix(5000, 0xC1), "fold-dense": lambda: F.fold_mix(20000, 0xC2),
        "spellings": lambda: F.spellings(1700, 0x5E),
        "keys4": lambda: F.keys4(2000, 0x4B),
        "needles3": lambda: F.needles(F.NEEDLES3, 300, 0x3D), "needles4": lambda: F.needles(F.NEEDLES4, 300, 0x4D),
    }[name]()


M32, M24, M16 = 0xFFFFFFFF, 0xFFFFFF, 0xFFFF
NARROW = dict(stride=2, wide=0, dense=0, brute=0, k=4, kmask=M32, amap=True)
WIDE = dict(stride=2, wide=1, dense=0, brute=0, k=4, kmask=M32, amap=True)
DENSE = dict(stride=1, wide=0, dense=1, brute=0, k=4, kmask=M32, amap=True)
STRIDE1 = dict(stride=1, wide=0, dense=0, brute=0, amap=True)
BRUTE = dict(stride=1, wide=0, dense=0, brute=1)

# (id, pattern set, CI, byte classes, start kind, match kinds, experiment flags, expected plan)
ROWS = [
    ("high-narrow", "high-narrow", False, True, O.START_UNANCHORED, (0, 1), 0, dict(NARROW, fold=0, bs_n=0)),
    ("high-wide", "high-wide", False, True, O.START_UNANCHORED, (0,), 0, dict(WIDE, fold=0, bs_n=0)),
    ("high-dense", "high-dense", False, True, O.START_UNANCHORED, (0, 2), 0, dict(DENSE, fold=0, bs_n=0)),
    ("high-stride1-k3", "high-k3", False, True, O.START_UNANCHORED, (0,), 0, dict(STRIDE1, k=3, kmask=M24, fold=0, bs_n=0)),
    ("high-stride1-k2", "high-k2", False, True, O.START_UNANCHORED, (1,), 0, dict(STRIDE1, k=2, kmask=M16, fold=0, bs_n=0)),
    ("high-brute-k1", "high-k1", False, True, O.START_UNANCHORED, (0,), 0, dict(BRUTE, k=1, kmask=0xFF, fold=0x20, amap=True, bs_n=0)),
    ("full-narrow", "full-narrow", False, True, O.START_UNANCHORED, (0, 1), 0, dict(NARROW, fold=0, bs_n=0)),
    ("full-wide", "full-wide", False, True, O.START_UNANCHORED, (1,), 0, dict(WIDE, fold=0, bs_n=0)),
    ("full-dense", "full-dense", False, True, O.START_UNANCHORED, (0, 1), 0, dict(DENSE, fold=0, bs_n=0)),
    ("full-stride1-k3", "full-k3", False, True, O.START_UNANCHORED, (0,), 0, dict(STRIDE1, k=3, kmask=M24, fold=0, bs_n=0)),
    ("fold-ci-narrow", "fold-narrow", True, True, O.START_UNANCHORED, (0, 1, 2), 0, dict(NARROW, fold=0x20202020, bs_n=0)),
    ("fold-ci-dense", "fold-dense", True, True, O.START_UNANCHORED, (0, 1, 2), 0, dict(DENSE, fold=0x20202020, bs_n=0)),
    ("fold-no-ci-stride1", "spellings", False, True, O.START_UNANCHORED, (0, 1), 0, dict(STRIDE1, k=4, kmask=M32, fold=0x20202020, bs_n=0)),
    ("keys4-key27", "keys4", False, True, O.START_UNANCHORED, (0, 1), 0, dict(NARROW, fold=0, bs_n=0, key_shift=5)),
    ("keys4-key24", "keys4", False, True, O.START_UNANCHORED, (0,), KEY24, dict(NARROW, fold=0, bs_n=0, key_shift=8)),
    ("needles3-bytescan", "needles3", False, True, O.START_UNANCHORED, (0,), 0, dict(BRUTE, k=1, bs_n=3)),
    ("needles4-control", "needles4", False, True, O.START_UNANCHORED, (0,), 0, dict(BRUTE, k=1, bs_n=0)),
    ("nobc-narrow", "high-narrow", False, False, O.START_UNANCHORED, (0,), 0, dict(NARROW, fold=0, bs_n=0)),
    ("nobc-wide", "high-wide", False, False, O.START_UNANCHORED, (1,), 0, dict(WIDE, fold=0, bs_n=0)),
    ("nobc-dense", "high-dense", False, False, O.START_UNANCHORED, (2,), 0, dict(DENSE, fold=0, bs_n=0)),
    ("both-high-narrow", "high-narrow", False, True, O.START_BOTH, (0,), 0, dict(NARROW, fold=0, bs_n=0)),
]
ROWS = [SimpleNamespace(id=r[0], set=r[1], ci=r[2], bc=r[3], sk=r[4], kinds=r[5], flags=r[6], plan=r[7]) for r in ROWS]


def builder(kind, ci, bc=True, sk=O.START_UNANCHORED):
    return (ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).byte_classes(bc)
            .start_kind(ab.StartKind(sk)).kind(ab.AhoCorasickKind.DFA))


def oracle(pats, kind, ci, bc=True, sk=O.START_UNANCHORED):
    return O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, byte_classes=bc, start_kind=sk, kind=O.KIND_DFA)


def plan_fields(p):
    return dict(stride=p.stride, wide=p.wide, dense=p.dense, brute=p.brute, k=p.k, kmask=p.kmask, fold=p.fold,
                amap=p.amap_log != 0, bs_n=p.bs_n, key_shift=p.key_shift, supported=p.supported)


def assert_plan(ac, want, ctx):
    got = plan_fields(plan_of(ac))
    assert got["supported"] == 1, (ctx, got)
    assert {k: got[k] for k in want} == want, (ctx, got)


# ---- haystacks -------------------------------------------------------------------------------------------
def decoys(p, j, ci, spelled, needle_set):
    """Near misses of planted pattern p (the j-th plant)."""
    out = []
    if spelled:   # another case spelling of a word: flip one letter's case
        i = j % len(p)
        out.append(p[:i] + bytes([p[i] ^ 0x20 if F.is_letter(p[i]) else p[i]]) + p[i + 1:])
    else:         # one byte for its fold partner, where the verifier tells them apart
        cand = [i for i, c in enumerate(p) if F.has_partner(c, ci)]
        if cand:
            i = cand[j % len(cand)]
            out.append(p[:i] + bytes([p[i] ^ 0x20]) + p[i + 1:])
    out.append(p[:-1] + bytes([p[-1] ^ (1 << (j % 8))]))                    # last byte changed
    i = 3 + (j & 1)
    if i < len(p):                                                        # bits 3 .. 7 of byte 4 or 5
        out.append(p[:i] + bytes([p[i] ^ (0x08 << (j % 5))]) + p[i + 1:])
    if needle_set:
        nd = needle_set[j % len(needle_set)]
        out.append(bytes([nd, nd ^ 1]) * (1 + j % 3))                      # the SWAR compare over-flags nd ^ 1
    return out


def make_haystack(row, pats, n, seed):
    """Filler from the family's byte distribution (for the needle rows: its bytes but the needles), plants
    and decoys every ~gap bytes, a pattern cut off by the buffer's end.  Returns (hay, plant starts, plant
    lengths) -- plants are the patterns, not the decoys."""
    rng = np.random.default_rng(seed)
    w = F.byte_weights(pats)
    needle_set = F.NEEDLES3 if row.set.startswith("needles") else b""
    if needle_set:
        w[list(F.NEEDLES4)] = 0
        w /= w.sum()
    hay = rng.choice(256, size=n, p=w).astype(np.uint8)
    spelled = row.set == "spellings"
    gap = 1024 if needle_set else 96   # needle rows: keep the candidates under the scan's retirement rate
    order = rng.permutation(len(pats))
    starts, lens = [], []
    pos, j = int(rng.integers(0, 32)), 0
    end = n - 64
    while pos < end:
        p = pats[order[j % len(pats)]]
        pos += (len(starts) - pos) % 32   # the j-th plant starts at j mod 32
        if pos + len(p) > end:
            break
        for i, x in enumerate([p] + decoys(p, j, row.ci, spelled, needle_set)):
            if pos + len(x) > end:
                break
            hay[pos: pos + len(x)] = np.frombuffer(x, dtype=np.uint8)
            if i == 0:
                starts.append(pos)
                lens.append(len(x))
            pos += len(x) + int(rng.integers(0, 2 * gap))
        j += 1
    # a match at the first byte of pointer phases 1 and 13 (the verifier reads the bytes within a word of
    # the buffer's edges one at a time), a pattern cut off by the buffer's end
    short = [p for p in pats if len(p) <= 12]
    for ph, p in zip(PHASES[1:], short[:2]):
        hay[ph: ph + len(p)] = np.frombuffer(p, dtype=np.uint8)
    longest = max(pats, key=len)
    hay[n - (len(longest) - 1):] = np.frombuffer(longest[:-1], dtype=np.uint8)
    if row.ci:
        W.flip_case(hay, seed + 1)   # letters in either case: still matches under CI
    starts, lens = np.array(starts, dtype=np.int64), np.array(lens, dtype=np.int64)
    assert set(np.unique(starts % 32)) == set(range(32)), row.id
    if starts.size >= 2048:   # where there is room: every 16-byte group of a 1 KiB and a 2 KiB tile
        assert set(np.unique((starts % 2048) // 16)) == set(range(128)), row.id
    if ON_GPU and len(pats) <= 20000:
        assert j >= len(pats), (row.id, j)   # every pattern planted
    return hay, starts, lens


def inside(starts, lens, at, odd=True):
    """An offset inside the first planted pattern of 3+ bytes at or after `at` (odd if asked)."""
    i = int(np.searchsorted(starts, at))
    while lens[i] < 3:
        i += 1
    s = int(starts[i]) + 1
    return s + 1 if odd and s % 2 == 0 else s


def doc_bounds(starts, lens, n, every):
    """Document bounds inside every `every`-th planted pattern."""
    sel = np.arange(0, starts.size, every)
    sel = sel[lens[sel] >= 2]
    cut = starts[sel] + 1 + (sel % (lens[sel] - 1))
    return np.unique(np.concatenate([[0], cut, [n]])).astype(np.int64)


_CACHE = {}


def haystack(row, pats, n=N):
    """One haystack at a time (keyed by pattern set, case knob and size), with its device copy."""
    import torch
    key = (row.set, row.ci, n)
    if _CACHE.get("key") != key:
        _CACHE.clear()
        if ON_GPU:
            torch.cuda.empty_cache()
        hay, starts, lens = make_haystack(row, pats, n, sum(row.set.encode()) * 131 + int(row.ci))
        d = to_device(torch.from_numpy(hay))
        assert d.data_ptr() % 16 == 0
        sub = (inside(starts, lens, n // 8), inside(starts, lens, n // 4 + 999))
        offs = doc_bounds(starts, lens, n, 16 if n == N else 4)
        _CACHE.update(key=key, hay=hay, d=d, sub=sub, offs=offs)
    return SimpleNamespace(**_CACHE)


# ---- the checks ------------------------------------------------------------------------------------------
def apis(kind):
    return ("overlapping", "iter") if kind == 0 else ("iter",)


def check_row(ac, o, h, kind, ctx, engines):
    """Every search of one handle: phases 0, 1, 13 and the odd sub-span, try_find / is_match on both spans,
    one batched call."""
    n = h.hay.size
    for api in apis(kind):
        fn = ac.find_overlapping_iter_dev_np if api == "overlapping" else ac.find_iter_dev_np
        ofn = o.find_overlapping_iter_np if api == "overlapping" else o.find_iter_np
        for off, span in [(ph, None) for ph in PHASES] + [(0, h.sub)]:
            want = ofn(h.hay[off:], span)
            got = fn(h.d.data_ptr() + off, n - off, span)[0]
            engines.append(ac.last_stats()["engine"])
            assert_np_equal(got, want, (ctx, api, off, span))
            if span is None:
                assert len(want) > n // 4096, (ctx, api, off, len(want))
    for span in (None, h.sub):
        m = ac.try_find(h.hay, span=span)
        engines.append(ac.last_stats()["engine"])
        assert (m.as_tuple() if m else None) == o.try_find(h.hay, span), (ctx, "try_find", span)
        assert ac.is_match(h.hay, span) == (m is not None), (ctx, "is_match", span)
        engines.append(ac.last_stats()["engine"])
    what = "overlapping" if kind == 0 else "iter"
    batch = (h.d if ON_GPU else h.hay, h.offs)
    got = (ac.find_overlapping_iter_batch_np if kind == 0 else ac.find_iter_batch_np)(batch)
    engines.append(ac.last_stats()["engine"])
    assert len(got) > 0, ctx
    sampled_docs_match_the_oracle(got, o, h.hay, h.offs, what, n=200)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("row", ROWS, ids=[r.id for r in ROWS])
def test_byte_content_row(row):
    pats = _pats(row.set)
    h = haystack(row, pats)
    for kind in row.kinds:
        ac = set_experiment(builder(kind, row.ci, row.bc, row.sk).build(pats), row.flags)
        assert_plan(ac, row.plan, (row.id, kind))
        o = oracle(pats, kind, row.ci, row.bc, row.sk)
        engines = []
        check_row(ac, o, h, kind, (row.id, kind), engines)
        assert set(engines) == {PREFILTER}, (row.id, kind, engines)
        if row.plan["bs_n"]:
            assert_plan(ac, row.plan, (row.id, kind, "not retired"))
            retire_and_check(ac, o, h, kind, row)


def retire_and_check(ac, o, h, kind, row):
    """A needle-dense search of 256 KiB (runs of needle, needle ^ 0x01) retires the byte-set scan; the
    kernel behind it then gives the same results on the same handle."""
    import torch
    rng = np.random.default_rng(kind)
    nd = np.frombuffer(F.NEEDLES3, dtype=np.uint8)
    pairs = np.stack([nd, nd ^ 1], 1)[rng.integers(0, nd.size, size=128 << 10)]
    dense = np.ascontiguousarray(pairs.reshape(-1))
    dd = to_device(torch.from_numpy(dense))
    assert_np_equal(ac.find_iter_dev_np(dd.data_ptr(), dense.size)[0], o.find_iter_np(dense), (row.id, "needle-dense"))
    assert ac.last_stats()["engine"] == PREFILTER
    assert plan_of(ac).bs_n == 0, (row.id, "retired")
    engines = []
    check_row(ac, o, h, kind, (row.id, kind, "retired"), engines)
    assert set(engines) == {PREFILTER}, (row.id, engines)


@functools.lru_cache(maxsize=1)
def no_amap_set():
    """The 270 000-pattern set, its handle and its oracle, built once per module."""
    pats = F.no_amap(NO_AMAP_PATTERNS, 0xA0)
    t0 = time.perf_counter()
    ac = builder(0, True).build(pats)
    t1 = time.perf_counter()
    o = oracle(pats, 0, True)
    t2 = time.perf_counter()
    print("no-anchor-map set: %d patterns, %.1f MiB of tables, library build %.2f s, oracle build %.2f s" % (
        len(pats), ac.memory_usage() / 2 ** 20, t1 - t0, t2 - t1))
    return pats, ac, o


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_no_anchor_map():
    """More than 4 Mi trie paths of length k: the plan ships no anchor map and the kernel verifies from
    the start state (brute mode: the dense variant cannot be reached, see the module docstring)."""
    pats, ac, o = no_amap_set()
    assert_plan(ac, dict(BRUTE, k=4, fold=0x20202020, amap=False, bs_n=0), "no-amap")
    row = SimpleNamespace(id="no-amap", set="no-amap", ci=True)
    h = haystack(row, pats, NO_AMAP_N)
    engines = []
    check_row(ac, o, h, 0, "no-amap", engines)
    assert set(engines) == {PREFILTER}, engines
