"""CPU checks of the device engine's derived tables (include/acb200_debug.h).

The kernels in csrc/acb_prefilter.cu and the plan built by csrc/acb_plan.hpp share a contract, written
down once in csrc/acb_fingerprint.cuh: how a fingerprint is hashed into the shared-memory Bloom bitmap
and how the anchor map is probed.  The probe functions are restated here independently (they are a
handful of integer operations) and checked against the tables the library builds -- no false
negatives for any pattern beginning, and the anchor map must agree with a walk of the DFA table
(which itself is bit-identical to the oracle's, tests/test_product_host.py).  Runs without a GPU on
host-only handles.
"""
import ctypes as C
import random
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import aho_corasick_b200 as ab  # noqa: E402
from aho_corasick_b200 import workload as W  # noqa: E402

sys.path.insert(0, str(ROOT / "tests"))
import byte_families as F  # noqa: E402

M32 = 0xFFFFFFFF


class Plan(C.Structure):
    _fields_ = [("supported", C.c_int32), ("brute", C.c_int32), ("dense", C.c_int32), ("stride", C.c_int32),
                ("wide", C.c_int32), ("k", C.c_uint32), ("kmask", C.c_uint32), ("fold", C.c_uint32),
                ("mult", C.c_uint32), ("mult3", C.c_uint32), ("shift", C.c_uint32), ("log_bits", C.c_uint32),
                ("bitmap", C.POINTER(C.c_uint32)), ("bitmap_words", C.c_uint64),
                ("amap", C.POINTER(C.c_uint64)), ("amap_log", C.c_uint32),
                ("depth16", C.POINTER(C.c_uint16)), ("n_rows", C.c_uint64), ("dup_shift", C.c_uint32),
                ("key_shift", C.c_uint32), ("bs_n", C.c_uint32), ("bs_byte", C.c_uint8 * 3), ("bs_back", C.c_uint8 * 3)]


def plan_of(ac):
    lib = ab._lib
    lib.acg_debug_prefilter_plan.argtypes = [C.c_void_p, C.POINTER(Plan)]
    p = Plan()
    assert lib.acg_debug_prefilter_plan(ac._h, C.byref(p)) == 0
    return p


def hash2(x):  # bloom_hash2 in acb_fingerprint.cuh
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def hash3(x):  # bloom_hash3
    x ^= x >> 15
    x = (x * 0x2C1B3C6D) & M32
    x ^= x >> 12
    x = (x * 0x297A2D39) & M32
    x ^= x >> 15
    return x


def bit_set(p, byte_index, bit):
    i = byte_index * 8 + bit
    assert i < (1 << p.log_bits)
    return (p.bitmap[i >> 5] >> (i & 31)) & 1


def probe_full(p, gram):
    """bloom_test(): byte from the hash's top bits, bit from its low 3 bits."""
    return bit_set(p, gram >> p.shift, gram & 7)


def first_stage_hit(p, window):
    """The per-position probe of prefilter_kernel for a 4-byte little-endian window."""
    if p.stride == 2:
        gm = (window | (p.fold & 0x00FFFFFF)) & M32
        h = (gm * ((p.mult3 << p.key_shift) & M32)) & M32   # key_shift 8: 3-byte key; 5: + 3 bits of the 4th byte
        return bit_set(p, h >> p.shift, gm & 7)
    gm = (window | p.fold) & p.kmask
    if p.dense:
        # blocked filter: the word from the top bits of the product, two bits from its high half
        prod = gm * p.mult
        lo, hi = prod & M32, (prod >> 32) & M32
        w = p.bitmap[lo >> (32 - (p.log_bits - 5))]
        return (w >> (hi & 31)) & (w >> ((hi >> 5) & 31)) & 1
    h = (gm * p.mult) & M32
    return bit_set(p, h >> p.shift, h & 7)


def second_stage_hit(p, window):
    if p.dense:
        return True   # the dense variant's second stage is the (exact) anchor-map lookup
    gram = (window | p.fold) & p.kmask
    ok = probe_full(p, hash2(gram))
    if p.stride == 2:
        ok = ok and probe_full(p, (gram * p.mult) & M32)
    return ok


def anchor_lookup(p, key):
    if not p.amap_log:
        return None
    mask = (1 << p.amap_log) - 1
    slot = hash3(key) >> (32 - p.amap_log)
    for _ in range(mask + 1):
        e = p.amap[slot]
        if (e >> 32) == 0:
            return 0
        if (e & M32) == key:
            return e >> 32
        slot = (slot + 1) & mask
    raise AssertionError("anchor map has no empty slot")


def walk(t, data):
    """DFA walk from the unanchored start over `data`; returns the premultiplied state id."""
    sid = int(t["start_unanchored_id"])
    for b in data:
        sid = int(t["trans"][sid + int(t["byte_classes"][b])])
    return sid


def le32(b4):
    return int.from_bytes(bytes(b4) + b"\0" * (4 - len(b4)), "little")


def case_variants(rng, b, n, partners=False):
    """Spellings of b that match it under ascii_case_insensitive (letters flipped at random); with
    `partners`, (spelling, is_match) pairs that add b with one non-letter swapped for its fold partner
    (x ^ 0x20: the twelve punctuation / DEL bytes and every high byte), which must not match."""
    out = {bytes(b)}
    for _ in range(n):
        out.add(bytes((c ^ 0x20) if (chr(c).isalpha() and c < 128 and rng.random() < 0.5) else c for c in b))
    if not partners:
        return out
    pairs = {(v, True) for v in out}
    for i, c in enumerate(b):
        if not (chr(c).isalpha() and c < 128):
            pairs.add((bytes(b[:i]) + bytes([c ^ 0x20]) + bytes(b[i + 1:]), False))
    return pairs


def set_experiment(ac, flags):
    ab._lib.acg_debug_set_experiment.argtypes = [C.c_void_p, C.c_uint32]
    assert ab._lib.acg_debug_set_experiment(ac._h, flags) == 0
    return ac


def check(pats, experiment=0, **knobs):
    b = ab.AhoCorasick.builder().host_only().kind(ab.AhoCorasickKind.DFA)
    for k, v in knobs.items():
        getattr(b, k)(v)
    ac = set_experiment(b.build(pats), experiment)
    p = plan_of(ac)
    assert p.key_shift == (5 if (not experiment & 8 and p.stride == 2) else 8)
    t = ac.tables()
    ci = bool(knobs.get("ascii_case_insensitive"))
    if not p.supported:
        return p
    assert 1 <= p.k <= 4 and p.k <= min(len(x) for x in pats)
    assert p.bitmap_words == 1 << (p.log_bits - 5) and p.shift == 35 - p.log_bits
    assert p.log_bits == (17 if (p.stride == 2 and p.wide) else 20)
    rng = random.Random(len(pats))
    stride2 = int(t["stride2"])
    for pat in pats:
        for v, spelling in (case_variants(rng, pat, 3, partners=True) if ci else {(bytes(pat), True)}):
            # the text "v + tail" at an even and at an odd offset: the probes that must fire.  A fold
            # partner spelling is merged with the pattern by the fold; without one it may miss.
            w0 = le32(v[:4])
            if not spelling:
                if p.fold == (0x20202020 & p.kmask) and not p.brute:
                    if p.stride == 2:
                        assert first_stage_hit(p, w0)
                        if len(v) > 4:
                            assert first_stage_hit(p, le32(v[1:5]))
                    else:
                        assert first_stage_hit(p, w0)
                    assert second_stage_hit(p, w0)
                # the anchor map is keyed by raw bytes: a state only if the spelling is itself a pattern start
                sid = anchor_lookup(p, w0 & p.kmask)
                if sid is not None:
                    key = v[:p.k]
                    on_path = walk(t, key) != 0 and p.depth16[walk(t, key) >> stride2] == p.k
                    assert sid == (walk(t, key) if on_path else 0), (pat, v)
                continue
            if not p.brute:
                if p.stride == 2:
                    assert p.k == 4
                    assert first_stage_hit(p, w0)        # start at an even offset: bytes [0,3) (+ the pattern's 4th)
                    # start at an odd offset: bytes [1,4) at the next even one, followed by the pattern's
                    # fifth byte -- or by any text if the pattern ends there
                    tails = [v[4:5]] if len(v) > 4 else [bytes([x]) for x in (0, 0x41, 0x7A, 0x20, 0xFF, 3, 0x35, 0x66)]
                    for tail in tails:
                        assert first_stage_hit(p, le32(v[1:4] + tail))
                else:
                    assert first_stage_hit(p, w0)
                assert second_stage_hit(p, w0)
            sid = anchor_lookup(p, w0 & p.kmask)
            if sid is not None:
                assert sid == walk(t, v[:p.k]) and sid != 0
                assert p.depth16[sid >> stride2] == p.k
    # keys that are not pattern beginnings must miss
    if p.amap_log:
        starts = {bytes(x[:p.k]) for x in pats}
        alphabet = sorted({c for x in pats for c in x}) or [0]
        miss = 0
        for _ in range(300):
            key = bytes(rng.choice(alphabet) for _ in range(p.k))
            sid = anchor_lookup(p, le32(key) & p.kmask)
            on_path = p.depth16[walk(t, key) >> stride2] == p.k and walk(t, key) != 0
            assert (sid != 0) == on_path
            if ci:
                continue
            assert (sid != 0) == (key in starts)
            miss += sid == 0
    return p


GOLDEN_SETS = [
    [b"apple", b"maple", b"Snapple"],
    [b"append", b"appendage", b"app"],
    [b"abcd", b"bcde", b"cdef", b"abcdefgh", b"xyzw"],
    [b"ab", b"abc", b"b"],
    [b"a"],
    [b"Sam", b"Samwise", b"sam"],
]


@pytest.mark.parametrize("kind", [ab.MatchKind.Standard, ab.MatchKind.LeftmostFirst, ab.MatchKind.LeftmostLongest])
@pytest.mark.parametrize("ci", [False, True])
def test_plan_on_small_sets(kind, ci):
    for pats in GOLDEN_SETS:
        check(pats, match_kind=kind, ascii_case_insensitive=ci)


def test_plan_cfg2_like():
    pats = W.make_patterns(5000, 0xAC5000)
    p = check(pats)
    assert p.stride == 2 and not p.wide and not p.dense and not p.brute and p.k == 4


def test_plan_cfg3_like():
    pats = W.make_patterns(5000, 0xAC5000)
    p = check(pats, match_kind=ab.MatchKind.LeftmostFirst, ascii_case_insensitive=True)
    assert p.k == 4 and p.fold == 0x20202020 and not p.dense


def test_plan_cfg4_like():
    pats = W.make_patterns(50, 0xAC0050)
    p = check(pats, match_kind=ab.MatchKind.LeftmostFirst)
    assert p.stride == 2 and p.wide and p.log_bits == 17


def test_plan_dense():
    pats = W.make_patterns(20000, 0xAC1000)
    p = check(pats)
    assert p.dense and p.stride == 1 and p.amap_log >= 15


def test_plan_short_patterns_and_unsupported():
    p = check([b"ab", b"cd", b"efg"])
    assert p.k == 2
    p = check([b"", b"ab"])
    assert not p.supported  # the empty pattern: every offset matches, walk / sequential engines only


def test_first_stage_pass_rate_is_low_on_random_text():
    """Selectivity sanity check for the cfg2-like set: the restated probe on random printable text."""
    pats = W.make_patterns(5000, 0xAC5000)
    ac = ab.AhoCorasick.builder().host_only().kind(ab.AhoCorasickKind.DFA).build(pats)
    p = plan_of(ac)
    rng = np.random.default_rng(3)
    txt = rng.integers(0x20, 0x7F, size=(20000, 4), dtype=np.uint32)
    wins = txt[:, 0] | (txt[:, 1] << 8) | (txt[:, 2] << 16) | (txt[:, 3] << 24)
    hits = sum(first_stage_hit(p, int(w)) for w in wins)
    assert hits / len(wins) < 0.05


@pytest.mark.parametrize("knobs", [dict(), dict(match_kind=ab.MatchKind.LeftmostFirst, ascii_case_insensitive=True),
                                   dict(match_kind=ab.MatchKind.LeftmostLongest)])
def test_plan_with_27_bit_first_stage_keys(knobs):
    """Default plan: the first-stage key also holds the low 3 bits of the window's fourth byte.
    No false negatives at either alignment, whatever follows a 4-byte pattern; fewer random hits.
    ACG_EXP_KEY24 = 8 goes back to 3-byte keys."""
    for pats in (W.make_patterns(5000, 0xAC5000), W.make_patterns(50, 0xAC0050),
                 [b"abcd", b"bcde", b"cdef", b"abcdefgh", b"xyzw", b"abcdX", b"abcdY"],
                 W.make_patterns(700, 11, lo=4, hi=5)):
        p = check(pats, experiment=0, **knobs)
        assert p.stride == 2 and p.key_shift == 5
        p = check(pats, experiment=8, **knobs)
        assert p.stride == 2 and p.key_shift == 8


def test_27_bit_keys_cut_the_first_stage_pass_rate():
    pats = W.make_patterns(5000, 0xAC5000)
    ac = ab.AhoCorasick.builder().host_only().kind(ab.AhoCorasickKind.DFA).build(pats)
    rng = np.random.default_rng(3)
    txt = rng.integers(0x20, 0x7F, size=(40000, 4), dtype=np.uint32)
    wins = txt[:, 0] | (txt[:, 1] << 8) | (txt[:, 2] << 16) | (txt[:, 3] << 24)
    k27 = sum(first_stage_hit(plan_of(ac), int(w)) for w in wins)
    set_experiment(ac, 8)
    base = sum(first_stage_hit(plan_of(ac), int(w)) for w in wins)
    set_experiment(ac, 0)
    again = sum(first_stage_hit(plan_of(ac), int(w)) for w in wins)
    print("first-stage pass rate on random printable text: 24-bit keys %.4f, 27-bit keys %.4f" % (base / len(wins), k27 / len(wins)))
    # the genuine 3-byte prefix hits (10 000 fingerprints in 95^3) all but disappear; what remains are the
    # Bloom false positives of a bitmap that also carries the second stage's two bits per 4-gram
    assert again == k27 and k27 < base * 0.97


# the families of the device rows in test_gpu_byte_content.py (all but the 270 000-pattern set, whose
# per-pattern restated probes take minutes in Python): (patterns, knobs, experiment flags, expected plan)
BYTE_FAMILIES = {
    "high-narrow": (lambda: F.high(5000, 0xB1), {}, 0, dict(stride=2, wide=0, dense=0, fold=0)),
    "high-wide": (lambda: F.high(50, 0xB2), {}, 0, dict(stride=2, wide=1, fold=0)),
    "high-dense": (lambda: F.high(20000, 0xB3), {}, 0, dict(stride=1, dense=1, fold=0)),
    "high-k3": (lambda: F.high(300, 0xB4, 3, 12), {}, 0, dict(stride=1, dense=0, k=3)),
    "high-k2": (lambda: F.high(300, 0xB5, 2, 12), {}, 0, dict(stride=1, dense=0, k=2)),
    "high-k1": (lambda: F.high(300, 0xB6, 1, 12), {}, 0, dict(brute=1, k=1, fold=0x20)),
    "full-narrow": (lambda: F.full(5000, 0xF1), {}, 0, dict(stride=2, wide=0, dense=0)),
    "full-wide": (lambda: F.full(50, 0xF2), {}, 0, dict(stride=2, wide=1)),
    "full-dense": (lambda: F.full(20000, 0xF3), {}, 0, dict(stride=1, dense=1)),
    "full-k3": (lambda: F.full(300, 0xF4, 3, 12), {}, 0, dict(stride=1, dense=0, k=3)),
    "fold-ci-narrow": (lambda: F.fold_mix(5000, 0xC1), dict(ascii_case_insensitive=True), 0,
                       dict(stride=2, wide=0, dense=0, fold=0x20202020)),
    "fold-ci-dense": (lambda: F.fold_mix(20000, 0xC2), dict(ascii_case_insensitive=True), 0,
                      dict(stride=1, dense=1, fold=0x20202020)),
    "fold-ci-leftmost": (lambda: F.fold_mix(5000, 0xC1),
                         dict(ascii_case_insensitive=True, match_kind=ab.MatchKind.LeftmostLongest), 0,
                         dict(stride=2, wide=0, fold=0x20202020)),
    "spellings": (lambda: F.spellings(1700, 0x5E), {}, 0, dict(stride=1, dense=0, k=4, fold=0x20202020)),
    "keys4-key27": (lambda: F.keys4(2000, 0x4B), {}, 0, dict(stride=2, key_shift=5)),
    "keys4-key24": (lambda: F.keys4(2000, 0x4B), {}, 8, dict(stride=2, key_shift=8)),
    "needles3": (lambda: F.needles(F.NEEDLES3, 300, 0x3D), {}, 0, dict(brute=1, bs_n=3)),
    "needles4": (lambda: F.needles(F.NEEDLES4, 300, 0x4D), {}, 0, dict(brute=1, bs_n=0)),
    "nobc-narrow": (lambda: F.high(5000, 0xB1), dict(byte_classes=False), 0, dict(stride=2, wide=0, dense=0)),
    "nobc-dense": (lambda: F.high(20000, 0xB3), dict(byte_classes=False), 0, dict(stride=1, dense=1)),
}


@pytest.mark.parametrize("family", list(BYTE_FAMILIES))
def test_plan_on_byte_content_families(family):
    """High bytes, NUL / DEL, fold-pair non-letters, case spellings, 4-byte keys and needle sets: no false
    negatives at either stride-2 alignment; under case insensitivity the fold-partner spellings of
    non-letters and high bytes reach the first stage and get no anchor-map state."""
    make, knobs, experiment, want = BYTE_FAMILIES[family]
    p = check(make(), experiment=experiment, **knobs)
    assert p.supported
    got = {k: getattr(p, k) for k in want}
    assert got == want, (family, got)
