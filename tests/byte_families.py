"""Pattern families over the whole byte range, shared by the device rows (test_gpu_byte_content.py) and the
CPU plan check (test_prefilter_plan.py).

workload.make_patterns and fill_haystack draw printable ASCII only.  These families put the bytes that
printable text never shows in front of the fingerprint probes: high bytes, NUL and DEL, the non-letters
that case folding (x | 0x20) merges with a partner, case spellings of one word, 4-byte patterns that are
prefixes of longer ones, and first bytes for the byte-set scan.  Every generator is deterministic."""
import numpy as np

from aho_corasick_b200 import workload as W

# the non-letter bytes whose partner 0x20 away is also a non-letter: x | 0x20 merges each pair, the
# verifier (ascii_case_insensitive covers letters only) must not
FOLD12 = b"@`[{\\|]}^~_\x7f"
LETTERS = bytes(range(0x41, 0x5B)) + bytes(range(0x61, 0x7B))


def is_letter(c):
    return 0x61 <= (c | 0x20) <= 0x7A


def has_partner(c, ci):
    """c ^ 0x20 is a different byte to the verifier: under case insensitivity every byte but a letter."""
    return not (ci and is_letter(c))


def _marked(pats, marks):
    """Every other pattern gets one of `marks` at position 0 .. 4 (where it is long enough)."""
    out = []
    for i, p in enumerate(pats):
        if i % 2 == 0:
            pos = (i // 2) % 5
            if pos < len(p):
                p = p[:pos] + bytes([marks[(i // 10) % len(marks)]]) + p[pos + 1:]
        out.append(p)
    return out


def high(n, seed, lo=4, hi=16):
    """Bytes 0x80 .. 0xFF, with 0x80, 0xFF and the fold pair 0xC1 / 0xE1 at positions 0 .. 4."""
    return _marked(W.make_patterns(n, seed, lo, hi, alphabet=(0x80, 0xFF)), b"\x80\xff\xc1\xe1")


def full(n, seed, lo=4, hi=16):
    """Bytes uniform over 0x00 .. 0xFF, with NUL, DEL, 0xFF and 0x80 at positions 0 .. 4."""
    return _marked(W.make_patterns(n, seed, lo, hi, alphabet=(0x00, 0xFF)), b"\x00\x7f\xff\x80")


def fold_mix(n, seed, lo=4, hi=16):
    """For ascii_case_insensitive(true): letters mixed with the twelve fold-pair non-letters (twice as
    likely each) and with high bytes."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(LETTERS + FOLD12 * 2 + bytes(range(0x80, 0x100)), dtype=np.uint8)
    return [bytes(rng.choice(pool, size=int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def spellings(n, seed):
    """For ascii_case_insensitive(false): n lower-case words, each also in upper case and capitalised, so
    that folding shrinks the fingerprint set by two thirds and the plan folds a case-sensitive automaton."""
    out = []
    for w in W.make_patterns(n, seed, 4, 12, alphabet=(0x61, 0x7A)):
        out += [w, w.upper(), w[:1].upper() + w[1:]]
    return out


def keys4(n, seed):
    """4-byte patterns (two of every three 4-grams) and, behind every 4-gram, two longer patterns whose
    fifth bytes differ only in one of bits 3 .. 7: the 27-bit stride-2 keys carry the low 3 bits of that
    byte, the second probe and the verifier tell them apart."""
    rng = np.random.default_rng(seed)
    out = []
    for i, b in enumerate(W.make_patterns(n, seed, 4, 4, alphabet=(0x00, 0xFF))):
        if i % 3 != 2:
            out.append(b)
        f = int(rng.integers(256))
        tail = bytes(rng.integers(0, 256, size=int(rng.integers(0, 6)), dtype=np.uint8))
        out += [b + bytes([f]) + tail, b + bytes([f ^ (0x08 << (i % 5))]) + tail]
    return out


def no_amap(n, seed):
    """For ascii_case_insensitive(true): n patterns of 5 .. 6 letters with distinct (case-folded) first
    four letters.  Each such 4-gram is 16 trie paths, so 270 000 of them exceed the 4 Mi paths an anchor
    map may hold."""
    rng = np.random.default_rng(seed)
    low = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    idx = rng.choice(26 ** 4, size=n, replace=False)
    body = np.stack([low[(idx // 26 ** j) % 26] for j in range(4)] +
                    [low[rng.integers(0, 26, size=n)], low[rng.integers(0, 26, size=n)]], 1)
    lens = 5 + (rng.integers(0, 2, size=n))
    up = rng.integers(0, 2, size=body.shape).astype(bool)   # spelled in mixed case; the automaton folds
    body = np.where(up, body ^ 0x20, body)
    return [bytes(body[i, :lens[i]]) for i in range(n)]


# The byte-set scan takes the reference's rare-bytes prefilter when every needle is a first byte only.  A
# pattern's rare byte is its rarest by the reference's frequency ranks (0x7F, then 0x00, are among the
# rarest; 0xFF is the most common byte of all) unless it already holds a needle.  So the single-byte
# pattern 0xFF comes first: it makes 0xFF a needle, and every later pattern that begins with 0xFF reuses it.
# The tails are lower-case letters, ranked far above the needles.
NEEDLES3 = b"\xff\x00\x7f"
NEEDLES4 = b"\xff\x00\x7f\x1b"


def needles(first, n, seed):
    rng = np.random.default_rng(seed)
    tails = W.make_patterns(n, seed, 3, 11, alphabet=(0x61, 0x7A))
    return [b"\xff"] + [bytes([first[i % len(first)]]) + t for i, t in enumerate(tails)]


def byte_weights(pats):
    """The bytes of the patterns, counted: the haystack filler's distribution."""
    h = np.bincount(np.frombuffer(b"".join(pats), dtype=np.uint8), minlength=256).astype(np.float64)
    return h / h.sum()
