"""Lookahead of stream sets (acg_candidates_*, acg_streams_lookahead(_devout)) on the dry-run build of the kernels
(tests/emu/).

The reference for every bit is its definition, computed with the oracle: with X the bytes the row's stream has
received since it was created, reset or (replace sets) flushed, the bit of candidate c is 1 iff the set's iterator
(find_iter, overlapping for an overlapping set) over X | c has a match that ends after |X|.  On small cases every
column is also checked against a twin set with the same history that is actually fed c.  Calls alternate between
host and "device" output (the dry run's device memory is host memory), with sentinels on both sides of every
output, and every call must leave the set as it found it."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import byte_families as BF  # noqa: E402
import oracle_py as O  # noqa: E402
from test_emulated_batch import emulated_library  # noqa: E402,F401
from test_emulated_kernels import VARIANTS, workload  # noqa: E402
from test_emulated_streams import NESTED, STANDARD_BYTESCAN, STANDARD_VARIANTS, split_hay  # noqa: E402
from test_kernel_resources import ptxas_info  # noqa: E402

SENTINEL = 0xA5
PAD = 48  # output bytes on either side that no call may touch
E_INVALID_ARG = -22
MODES = ("find_iter", "overlapping", "replace")


class History:
    """A set of `mode` over `ac` and what each of its streams has received since it last started from zero bytes."""

    def __init__(self, ac, n, mode):
        self.ac, self.mode, self.n = ac, mode, n
        self.st = self.make()
        self.data = [b""] * n
        self.log = []  # ("feed", chunks) / ("restart", ids) to replay on a twin

    def make(self):
        if self.mode == "replace":
            return self.ac.replace_streams(self.n, [b"<>"] * self.ac.patterns_len())
        return self.ac.streams(self.n, self.mode == "overlapping")

    def feed(self, chunks):
        chunks = [bytes(c) for c in chunks]
        self.st.feed(chunks)
        self.data = [d + c for d, c in zip(self.data, chunks)]
        self.log.append(("feed", chunks))

    def restart(self, ids):
        """reset, or for a replace set flush: the streams start again from zero bytes."""
        if self.mode == "replace":
            self.st.flush(ids)
        else:
            self.st.reset(ids)
        for i in ids:
            self.data[i] = b""
        self.log.append(("restart", list(ids)))

    def twin(self):
        """A find_iter or overlapping set with the same history: a replace set's matches are its find_iter matches,
        and its flush restarts a stream as a reset does."""
        t = self.ac.streams(self.n, self.mode == "overlapping")
        for what, x in self.log:
            if what == "feed":
                t.feed(x)
            else:
                t.reset(x)
        return t


def oracle_bit(o, x, c, overlapping):
    if not c:
        return False
    h = np.frombuffer(x + c, np.uint8).copy()
    r = o.find_overlapping_iter_np(h) if overlapping else o.find_iter_np(h)
    return bool(len(r)) and int(r["end"].max()) > len(x)


def oracle_mask(o, hist, cands, ids=None):
    rows = range(hist.n) if ids is None else ids
    ov = hist.mode == "overlapping"
    return np.array([[oracle_bit(o, hist.data[s], c, ov) for c in cands] for s in rows], dtype=bool).reshape(
        len(rows), len(cands))


def raw_look(st, cs, ids, form):
    """One raw call into a sentinel-framed buffer: (rc, the mask as bool [rows, n_cands], the whole buffer)."""
    a = None if ids is None else np.asarray(ids, np.uint64)
    rows = st.n_streams if a is None else a.size
    buf = np.full(rows * cs.n + 2 * PAD, SENTINEL, np.uint8)
    fn = ab._lib.acg_streams_lookahead if form == "host" else ab._lib.acg_streams_lookahead_devout
    rc = fn(st._h, cs._h, None if a is None else a.ctypes.data, 0 if a is None else a.size, buf[PAD:].ctypes.data)
    assert (buf[:PAD] == SENTINEL).all() and (buf[PAD + rows * cs.n:] == SENTINEL).all(), (form, "sentinels")
    body = buf[PAD:PAD + rows * cs.n]
    if rc == 0:
        assert np.isin(body, (0, 1)).all(), "bytes other than 0 and 1"
    return rc, body.astype(bool).reshape(rows, cs.n), buf


def state_of(hist):
    st = hist.st
    return st.positions().tolist(), (st.held().tolist() if hist.mode == "replace" else None)


def check(o, hist, cands, cs=None, ids=None, twin=False):
    """The mask of `cands` in both output forms against the oracle (and, with `twin`, every column against a twin set
    fed that candidate); the set is unchanged by the calls."""
    own = cs is None
    cs = cs or hist.ac.candidates(cands)
    before = state_of(hist)
    want = oracle_mask(o, hist, cands, ids)
    for form in ("host", "devout"):
        rc, got, _ = raw_look(hist.st, cs, ids, form)
        assert rc == 0, (form, rc)
        if not np.array_equal(got, want):
            k, c = np.argwhere(got != want)[0]
            s = k if ids is None else ids[k]
            raise AssertionError((form, hist.mode, "row", int(k), "stream", int(s), hist.data[s][-40:],
                                  "candidate", cands[c], "got", bool(got[k, c])))
    assert np.array_equal(hist.st.lookahead_np(cs, ids), want)
    assert state_of(hist) == before, "a lookahead changed the set"
    if twin:
        rows = list(range(hist.n)) if ids is None else list(ids)
        for j, c in enumerate(cands):
            t = hist.twin()
            got = t.feed([c] * hist.n)
            assert [bool(got[s]) for s in rows] == want[:, j].tolist(), ("twin", c)
            t.close()
    if own:
        cs.close()
    return want


def candidate_list(pats, rng, max_len, singles=True):
    """Empty; every single byte; prefixes, suffixes and infixes of patterns; whole patterns inside longer strings;
    strings longer than max_pattern_len."""
    out = [b""]
    if singles:
        out += [bytes([b]) for b in range(256)]
    for p in pats[:: max(1, len(pats) // 24)][:24]:
        k = int(rng.integers(1, len(p) + 1))
        i = int(rng.integers(0, len(p)))
        out += [p[:k], p[-k:], p[i:i + k], b"qq" + p + b"q", p]
    filler = bytes(rng.integers(97, 123, size=max_len + 5, dtype=np.uint8))
    out += [filler, filler[:max_len // 2] + pats[0] + filler[:max_len], b""]
    return out


def seeded(hist, hay, rng, n_feeds=3, restart=True):
    """Streams filled from `hay` over a few feeds: stream 0 never fed, stream 1 restarted at the end."""
    parts = split_hay(hay, hist.n, rng)
    parts[0] = b""
    for i in range(n_feeds):
        chunks = []
        for p in parts:
            a, b = len(p) * i // n_feeds, len(p) * (i + 1) // n_feeds
            chunks.append(p[a:b])
        hist.feed(chunks)
    if restart:
        hist.restart([1])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", STANDARD_VARIANTS)
def test_prefilter_variants(name, mode):
    n, seed, _, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, 12 << 10, ci)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    rng = np.random.default_rng(seed)
    hist = History(ac, 6, mode)
    seeded(hist, hay, rng)
    want = check(o, hist, candidate_list(pats, rng, ac.max_pattern_len()))
    assert want.any() and not want.all()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,pats,kw", STANDARD_BYTESCAN)
def test_bytescan_sets(name, pats, kw, mode):
    ci = kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=6 << 10)].copy()
    for i in range(0, hay.size - 64, 331):
        p = pats[(i // 331) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).build(pats)
    o = O.Oracle(pats, ascii_case_insensitive=ci)
    hist = History(ac, 5, mode)
    seeded(hist, hay, rng)
    check(o, hist, candidate_list(pats, rng, ac.max_pattern_len()))


def test_modes_differ_where_the_cursor_has_moved():
    """{"abc", "bcd"}, stream fed "abc", candidate "d": bcd ends in the d, but find_iter restarts at 3."""
    pats = [b"abc", b"bcd"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    bits = {}
    for mode in MODES:
        hist = History(ac, 2, mode)
        hist.feed([b"abc", b"xbc"])
        bits[mode] = check(o, hist, [b"d", b"", b"bcd", b"ab"], twin=True)
    assert bits["overlapping"].tolist() == [[True, False, True, False], [True, False, True, False]]
    assert bits["find_iter"].tolist() == [[False, False, True, False], [True, False, True, False]]
    assert np.array_equal(bits["replace"], bits["find_iter"])


@pytest.mark.parametrize("mode", MODES)
def test_split_inside_pattern_at_every_point(mode):
    """Stream k holds the text up to k bytes into a planted long pattern, built over a few feeds; the candidates
    finish it at every point, and cut it short by one byte."""
    long = b"the quick brown fox jumps over the lazy dog"
    pats = NESTED + [long]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    body = b"xx" + b"abcabcabcabzzzzz" + long + b"abcabz"
    at = body.index(long)
    n = len(long) + 1
    hist = History(ac, n, mode)
    hist.feed([body[:at // 2]] * n)
    hist.feed([body[at // 2:at + k] for k in range(n)])
    cands = sorted({long[k:] for k in range(n)} | {long[k:-1] for k in range(n)} | {b"z", b"zz", b"bca", b"q"})
    check(o, hist, cands)
    small = History(ac, 8, mode)
    small.feed([body[:at + k] for k in range(0, 40, 5)])
    check(o, small, [long[k:] for k in range(0, 40, 5)] + [b"z", b"ab"], twin=True)


@pytest.mark.parametrize("mode", MODES)
def test_patterns_at_the_tail_limit(mode):
    """A 65 533-byte pattern: streams hold back exactly max_pattern_len - 1 bytes of it, and the candidates are its
    last byte, its last two bytes, and a byte that does not finish it."""
    plen = 65533
    rng = np.random.default_rng(plen)
    p = rng.integers(97, 101, size=plen, dtype=np.uint8).tobytes()
    pats = [p, b"wxyz"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    hist = History(ac, 4, mode)
    filler = rng.integers(101, 110, size=plen, dtype=np.uint8).tobytes()
    hist.feed([filler[:100] + p[:plen // 2], filler[:7] + p[:plen - 2], b"wx", b""])
    hist.feed([p[plen // 2:-1], p[plen - 2:plen - 1], b"y", b"x" + p[:-1]])
    want = check(o, hist, [p[-1:], p[-2:], b"z", b"e", b"wxyz", p], twin=True)
    assert want[0, 0] and want[1, 0] and want[2, 2] and want[3, 0]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("family", ["high", "full", "fold_mix"])
def test_byte_families(family, mode):
    """High and control bytes, and case-insensitive sets that mix letters with the fold-pair non-letters."""
    ci = family == "fold_mix"
    pats = getattr(BF, family)(40, 11)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    rng = np.random.default_rng(3)
    pieces = []
    for i in range(60):
        q = pats[int(rng.integers(0, len(pats)))]
        if ci:
            q = bytes(b ^ 0x20 if BF.is_letter(b) and rng.random() < 0.5 else b for b in q)
        pieces += [bytes(rng.integers(0, 256, size=int(rng.integers(0, 9)), dtype=np.uint8)), q]
    hay = np.frombuffer(b"".join(pieces), np.uint8)
    hist = History(ac, 5, mode)
    seeded(hist, hay, rng)
    cands = candidate_list(pats, rng, ac.max_pattern_len())
    if ci:
        cands += [c.swapcase() for c in cands[257:]]
    check(o, hist, cands)


def test_ids_subsets_duplicates_and_order():
    pats = [b"abc", b"bcd", b"zz", b"hello world"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    hist = History(ac, 5, "overlapping")
    hist.feed([b"xab", b"hello wor", b"z", b"", b"abcab"])
    cands = [b"c", b"ld", b"z", b"cd", b""] + [b"q"] * 30  # 35: not a multiple of 32
    with ac.candidates(cands) as cs:
        full = check(o, hist, cands, cs)
        for ids in ([3], [4, 0], [2, 2, 2, 0, 2], list(range(5))[::-1], []):
            assert np.array_equal(check(o, hist, cands, cs, ids=ids), full[ids].reshape(len(ids), len(cands)))
        for form in ("host", "devout"):
            rc, _, buf = raw_look(hist.st, cs, [0, 5, 1], form)
            assert rc == E_INVALID_ARG and (buf == SENTINEL).all(), form
        with pytest.raises(Exception):
            hist.st.lookahead_np(cs, [1, 7])


@pytest.mark.parametrize("n_cands", [0, 1, 31, 32, 33, 100])
def test_candidate_counts(n_cands):
    pats = [b"ab", b"bc", b"cab"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(n_cands)
    cands = [bytes(rng.choice(list(b"abcx"), size=int(rng.integers(0, 5)))) for _ in range(n_cands)]
    for mode in MODES:
        hist = History(ac, 3, mode)
        hist.feed([b"ca", b"", b"xxa"])
        got = check(o, hist, cands, twin=n_cands <= 33)
        assert got.shape == (3, n_cands)


@pytest.mark.parametrize("mode", MODES)
def test_the_set_is_unchanged_by_lookahead(mode):
    """A set that looks ahead between its feeds gives the same feeds, positions and held bytes as a twin that never
    does."""
    pats, hay = workload(300, 17, 8 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    rng = np.random.default_rng(17)
    parts = split_hay(hay, 4, rng)
    a, b = History(ac, 4, mode), History(ac, 4, mode)
    with ac.candidates(candidate_list(pats, rng, ac.max_pattern_len(), singles=False)) as cs:
        for i in range(4):
            chunks = [p[len(p) * i // 4:len(p) * (i + 1) // 4] for p in parts]
            a.st.lookahead_np(cs)
            a.st.lookahead_np(cs, [3, 0, 0])
            assert a.st.feed(chunks) == b.st.feed(chunks)
            assert state_of(a) == state_of(b)
            if i == 2:
                a.restart([2])
                b.restart([2])
        if mode == "replace":
            assert a.st.flush() == b.st.flush()


def test_errors():
    pats = [b"abc", b"bcd"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    other = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    st = ac.streams(2)
    out = np.zeros(16, np.uint8)
    with other.candidates([b"a", b"b"]) as foreign, ac.candidates([b"a", b"b"]) as cs:
        for fn in (ab._lib.acg_streams_lookahead, ab._lib.acg_streams_lookahead_devout):
            assert fn(st._h, foreign._h, None, 0, out.ctypes.data) == E_INVALID_ARG
            assert fn(None, cs._h, None, 0, out.ctypes.data) == E_INVALID_ARG
            assert fn(st._h, None, None, 0, out.ctypes.data) == E_INVALID_ARG
            assert fn(st._h, cs._h, None, 0, None) == E_INVALID_ARG
            ids = np.array([0], np.uint64)
            assert fn(st._h, cs._h, ids.ctypes.data, 0, None) == 0  # no rows: nothing to write
        assert (out == 0).all()
        with pytest.raises(ValueError):
            st.lookahead_np(foreign)
        st.close()
        with pytest.raises(ValueError):
            st.lookahead_np(cs)
    h = ctypes.c_void_p()
    b = np.frombuffer(b"abcd", np.uint8)
    offs = np.array([0, 2, 4], np.uint64)
    create = ab._lib.acg_candidates_create
    assert create(ac._h, b.ctypes.data, offs.ctypes.data, 1 << 32, ctypes.byref(h)) == E_INVALID_ARG
    assert create(ac._h, b.ctypes.data, np.array([0, 3, 2], np.uint64).ctypes.data, 2,
                  ctypes.byref(h)) == E_INVALID_ARG
    assert create(ac._h, None, offs.ctypes.data, 2, ctypes.byref(h)) == E_INVALID_ARG
    assert create(ac._h, b.ctypes.data, offs.ctypes.data, 2, None) == E_INVALID_ARG
    assert create(ac._h, None, np.zeros(3, np.uint64).ctypes.data, 2, ctypes.byref(h)) == 0  # two empty candidates
    ab._lib.acg_candidates_free(h)
    # offsets need not start at 0
    with ac.candidates((b, np.array([1, 3, 4], np.uint64))) as cs, ac.streams(1, True) as s1:
        s1.feed([b"a"])
        assert s1.lookahead_np(cs).tolist() == [[True, False]]  # "bc" finishes abc, "d" nothing


def test_stats():
    pats = [b"abc", b"bcd"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    with ac.streams(3) as st, ac.candidates([b"c", b"d"]) as cs:
        st.feed([b"ab", b"", b"b"])
        assert st.lookahead_np(cs).tolist() == [[True, False], [False, False], [False, False]]
        s = ac.last_stats()
        assert s["launches"] == 7 and s["scan_ms"] >= 0 and s["order_ms"] >= 0


def test_new_kernels_do_not_spill():
    info = {k: v for k, v in ptxas_info("acb_kernels.cu").items() if "look_" in k}
    assert len(info) == 5, sorted(info)
    for name, v in info.items():
        assert v["spill"] == 0, name
