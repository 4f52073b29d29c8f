"""Replace sets (acg_streams_create_replace, acg_streams_replace_feed(_devout), acg_streams_flush, acg_streams_held)
on the dry-run build of the kernels (tests/emu/).

Two references, computed from the oracle:
- per feed, the exact bytes the feed must release.  With X the stream's bytes so far, c the end of the last
  find_iter match of X (0 if none) and h = max(c, |X| - (max_pattern_len - 1)), the stream's output up to now is X[:h]
  with the oracle's find_iter matches of X spliced in (they all end at or before h).  This checks when bytes are
  released, not only what they add up to; held() must be |X| - h;
- per stream, its outputs followed by its flush: the splice over the oracle's find_iter matches of all its bytes,
  and for short streams also the host glue stream_replace_all over an io.BytesIO of them.
Feeds cycle through host output, device output with host offsets, device output with "device" offsets (the dry
run's device memory is host memory) and the Python list form, with sentinels around every output array and exactly
the room the feed needs."""
import ctypes
import io
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from test_emulated_batch import emulated_library  # noqa: E402,F401
from test_emulated_kernels import VARIANTS, workload  # noqa: E402
from test_emulated_replace import splice  # noqa: E402
from test_emulated_streams import (NESTED, STANDARD_BYTESCAN, STANDARD_VARIANTS, dealt,  # noqa: E402
                                   split_hay)
from test_prefilter_plan import plan_of  # noqa: E402

SENTINEL = 0xA5A5A5A5A5A5A5A5
BYTE_SENTINEL = 0xA5
PAD = 40  # output bytes on either side that no call may touch
FORMS = ("host", "devout", "devout_dev_offsets", None)  # None: ReplaceStreams.feed
E_INVALID_ARG, E_INVALID_SPAN = -22, -20


def raw_feed(st, chunks, form, cap):
    """One raw replace feed of the given form into sentinel-filled arrays: (rc, out_len, output buffer with PAD bytes
    on either side, out_offsets with one entry on either side)."""
    pieces = [bytes(c) for c in chunks]
    offs = np.r_[0, np.cumsum([len(c) for c in pieces])].astype(np.uint64)
    hay = np.frombuffer(b"".join(pieces) + b"\0", np.uint8)[:-1].copy()
    buf = np.full(cap + 2 * PAD, BYTE_SENTINEL, np.uint8)
    oo = np.full(len(pieces) + 3, SENTINEL, np.uint64)
    n = ctypes.c_uint64(12345)
    hp = hay.ctypes.data if hay.size else None
    if form == "host":
        rc = ab._lib.acg_streams_replace_feed(st._h, hp, 0, hay.size, offs.ctypes.data, len(pieces),
                                              buf[PAD:].ctypes.data, cap, oo[1:].ctypes.data, ctypes.byref(n))
    else:
        rc = ab._lib.acg_streams_replace_feed_devout(st._h, hp, hay.size, offs.ctypes.data,
                                                     int(form == "devout_dev_offsets"), len(pieces),
                                                     buf[PAD:].ctypes.data, cap, oo[1:].ctypes.data, ctypes.byref(n))
    return rc, int(n.value), buf, oo


def raw_flush(st, ids, cap):
    """One raw flush into sentinel-filled arrays, as raw_feed."""
    k = st.n_streams if ids is None else len(ids)
    u = None if ids is None else np.array(ids, np.uint64)
    buf = np.full(cap + 2 * PAD, BYTE_SENTINEL, np.uint8)
    oo = np.full(k + 3, SENTINEL, np.uint64)
    n = ctypes.c_uint64(12345)
    rc = ab._lib.acg_streams_flush(st._h, None if u is None else u.ctypes.data, k if u is not None else 0,
                                   buf[PAD:].ctypes.data, cap, oo[1:].ctypes.data, ctypes.byref(n))
    return rc, int(n.value), buf, oo


def check_sentinels(buf, oo, got, rc):
    assert (buf[:PAD] == BYTE_SENTINEL).all(), "sentinel before the output"
    assert oo[0] == SENTINEL and oo[-1] == SENTINEL, "sentinels around out_offsets"
    if rc == 0:
        assert (buf[PAD + got:] == BYTE_SENTINEL).all(), "sentinel after the output"
    else:
        assert (buf == BYTE_SENTINEL).all() and (oo == SENTINEL).all(), "a failed call wrote"


class Run:
    """A replace set and, per stream, its bytes and its output so far; every feed and flush checked on its own."""

    def __init__(self, ac, o, reps, n):
        self.ac, self.o, self.n = ac, o, n
        self.reps = [r.encode() if isinstance(r, str) else bytes(r) for r in reps]
        self.back = ac.max_pattern_len() - 1
        self.st = ac.replace_streams(n, reps)
        self.data = [b""] * n
        self.out = [b""] * n
        self.i = 0

    def settled(self, x):
        """(h, X[:h] with X's find_iter matches spliced in) for a stream's bytes x."""
        r = self.o.find_iter_np(np.frombuffer(x + b"\0", np.uint8)[:-1].copy())
        c = int(r["end"][-1]) if r.size else 0
        h = max(c, len(x) - self.back, 0)
        assert r.size == 0 or int(r["end"].max()) <= h
        return h, splice(x[:h], r["start"].tolist(), r["end"].tolist(), r["pid"].tolist(), self.reps)

    def feed(self, chunks, form="cycle"):
        if form == "cycle":
            form = FORMS[self.i % len(FORMS)]
        self.i += 1
        data = [d + bytes(c) for d, c in zip(self.data, chunks)]
        want, hs = [], []
        for s in range(self.n):
            h, so_far = self.settled(data[s])
            assert so_far.startswith(self.out[s]), ("an earlier feed released bytes that changed", s)
            want.append(so_far[len(self.out[s]):])
            hs.append(h)
        if form is None:
            got = self.st.feed(chunks)
        else:
            need = sum(map(len, want))
            rc, n, buf, oo = raw_feed(self.st, chunks, form, need)
            check_sentinels(buf, oo, n, rc)
            assert rc == 0 and n == need, (form, rc, n, need)
            o = oo[1:-1].astype(np.int64)
            assert o[0] == 0 and o[-1] == n and (np.diff(o) >= 0).all(), (form, "out_offsets")
            b = buf[PAD:PAD + n].tobytes()
            got = [b[o[s]:o[s + 1]] for s in range(self.n)]
        for s in range(self.n):
            assert got[s] == want[s], ("feed", self.i, form, s, got[s][:80], want[s][:80])
        self.data = data
        self.out = [a + g for a, g in zip(self.out, got)]
        pos, held = self.st.positions(), self.st.held()
        assert pos.tolist() == [len(d) for d in data]
        assert (held <= self.back).all()
        assert (pos - held).tolist() == hs, "positions() - held() is the emit boundary"
        return got

    def flush(self, ids=None, raw=False):
        """Flush `ids` (all: None); every flushed stream must come out whole and restart from zero bytes."""
        held = self.st.held()
        sel = list(range(self.n)) if ids is None else list(ids)
        if raw:
            need = int(sum(held[s] for s in sel))
            rc, n, buf, oo = raw_flush(self.st, ids, need)
            check_sentinels(buf, oo, n, rc)
            assert rc == 0 and n == need
            o = oo[1:-1].astype(np.int64)
            b = buf[PAD:PAD + n].tobytes()
            got = [b[o[k]:o[k + 1]] for k in range(len(sel))]
        else:
            got = self.st.flush(ids)
        assert len(got) == len(sel)
        for k, s in enumerate(sel):
            x = self.data[s]
            assert got[k] == x[len(x) - int(held[s]):], ("flush returns the held bytes raw", s)
            self.check_whole(s, self.out[s] + got[k])
            self.data[s], self.out[s] = b"", b""
        pos = self.st.positions()
        assert all(pos[s] == 0 for s in sel) and all(self.st.held()[s] == 0 for s in sel)
        return got

    def check_whole(self, s, text, glue=None):
        x = self.data[s]
        r = self.o.find_iter_np(np.frombuffer(x + b"\0", np.uint8)[:-1].copy())
        want = splice(x, r["start"].tolist(), r["end"].tolist(), r["pid"].tolist(), self.reps)
        assert text == want, ("whole stream", s, len(text), len(want))
        if glue if glue is not None else len(x) < (16 << 10):
            w = io.BytesIO()
            self.ac.stream_replace_all(io.BytesIO(x), w, self.reps, chunk_bytes=997)
            assert text == w.getvalue(), ("host glue", s)

    def close(self):
        self.flush()
        self.st.close()


def run_feeds(ac, o, reps, feeds, between=None):
    """Feed `feeds` to a new replace set, cycling through the forms, then flush every stream; returns each stream's
    whole output."""
    run = Run(ac, o, reps, len(feeds[0]))
    for i, f in enumerate(feeds):
        if between:
            between(i, run)
        run.feed(f)
    whole = list(run.out)
    tails = run.flush()
    run.st.close()
    return [w + t for w, t in zip(whole, tails)]


def mixed_reps(n, rng, longest=40):
    """Deletions, same-length-ish and longer tags, by pattern."""
    reps = []
    for p in range(n):
        k = p % 4
        reps.append(b"" if k == 0 else b"<%d>" % p if k == 1 else bytes(rng.integers(33, 127, size=int(
            rng.integers(0, longest))).astype(np.uint8)) if k == 2 else b"#")
    return reps


@pytest.mark.parametrize("name", STANDARD_VARIANTS)
def test_prefilter_variants(name):
    """Every Standard prefilter variant, streams cut at random points, on the prefilter and sequential engines."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, 32 << 10, ci)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    assert plan_of(ac).supported
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    rng = np.random.default_rng(seed)
    reps = mixed_reps(len(pats), rng)
    feeds = dealt(split_hay(hay, 7, rng), rng, 6)
    got = run_feeds(ac, o, reps, feeds)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    ac.set_engine(ab.Engine.Sequential)
    assert run_feeds(ac, o, reps, feeds) == got
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


@pytest.mark.parametrize("name,pats,kw", STANDARD_BYTESCAN)
def test_bytescan_sets(name, pats, kw):
    ci = kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=16 << 10)].copy()
    for i in range(0, hay.size - 64, 331):
        p = pats[(i // 331) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).build(pats)
    assert plan_of(ac).bs_n >= 1
    o = O.Oracle(pats, ascii_case_insensitive=ci)
    run_feeds(ac, o, mixed_reps(len(pats), rng), dealt(split_hay(hay, 5, rng), rng, 8))
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_split_inside_pattern_at_every_point(engine):
    """Stream k holds the same bytes and is cut at k bytes into a planted long pattern: every split point of it at
    once, then chunks of 0 to 3 bytes, shorter than the held bytes, so that matches spread over many feeds."""
    pats = NESTED + [b"the quick brown fox jumps over the lazy dog"]
    reps = [b"", b"BCA", b"[cabcabc]", b"", b"<11>", b"", b"ZZ", b"5", b"the slow red fox"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats).set_engine(engine)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    body = b"xx" + b"abcabcabcabzzzzz" + b"the quick brown fox jumps over the lazy dog" + b"abcabz" * 3 + b"q"
    at = body.index(b"the quick")
    streams = 44
    feeds = [[body[:at + k] for k in range(streams)]]
    rest = [body[at + k:] for k in range(streams)]
    rng = np.random.default_rng(5)
    while any(rest):
        nxt = []
        for s in range(streams):
            k = int(rng.integers(0, 4))
            nxt.append(rest[s][:k])
            rest[s] = rest[s][k:]
        feeds.append(nxt)
    got = run_feeds(ac, o, reps, feeds)
    assert all(g == got[0] for g in got) and b"the slow red fox" in got[0]


@pytest.mark.parametrize("pats", [[b"abcd", b"bc"], [b"ab", b"abcdef"], [b"abcdef", b"def", b"cdefg"]],
                         ids=["suffix-inside", "prefix", "chain"])
def test_prefix_and_suffix_patterns_across_a_boundary(pats):
    """One pattern inside, a prefix or a suffix of another: Standard reports the earliest end, so a shorter match
    that ends first wins over a longer one, wherever the chunk boundary falls -- including a match that ends exactly
    at the end of a feed."""
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    reps = [b"<%d>" % i for i in range(len(pats))]
    body = b"xabcdefgabcdabcdefy" * 2
    n = len(body) + 1
    feeds = [[body[:k] for k in range(n)], [body[k:k + 2] for k in range(n)], [body[k + 2:] for k in range(n)]]
    got = run_feeds(ac, o, reps, feeds)
    assert all(g == got[0] for g in got)


def test_decode_steps_and_empty_feeds():
    """1-byte decode steps, empty chunks and feeds where every chunk is empty, on periodic text where find_iter's
    restart point matters."""
    pats = [b"aa", b"aaa", b"aba", b"abab", b"baba", b"b"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(11)
    streams = [bytes(rng.choice(np.frombuffer(b"ab", np.uint8), size=int(rng.integers(0, 120)))) for _ in range(6)]
    feeds = []
    at = [0] * 6
    while any(at[s] < len(streams[s]) for s in range(6)):
        if len(feeds) % 7 == 3:
            feeds.append([b""] * 6)
            continue
        f = []
        for s in range(6):
            k = int(rng.integers(0, 2)) if s % 2 else 1
            f.append(streams[s][at[s]:at[s] + k])
            at[s] += k
        feeds.append(f)
    run_feeds(ac, o, [b"", b"A", b"xyz", b"", b"BABA!", b"c"], feeds)


@pytest.mark.parametrize("plen", [1024, 4096, 65533])
def test_long_patterns_held_at_back(plen):
    """1 KiB to 64 KiB patterns with replacements up to several KiB: a feed ends one byte before the end of a
    pattern, so the set holds exactly back = max_pattern_len - 1 bytes, and the match comes out with the next
    feed's first byte."""
    rng = np.random.default_rng(plen)
    p = rng.integers(97, 101, size=plen, dtype=np.uint8).tobytes()
    pats = [p, b"wxyz"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    back = plen - 1
    filler = rng.integers(101, 110, size=3 * plen, dtype=np.uint8).tobytes()
    stream0 = filler[:plen] + p + b"wxyz" + filler[plen:2 * plen] + p + p[: plen // 2]
    first = plen + back
    stream1 = b"x" + p + filler[:100]
    reps = [bytes(rng.integers(33, 127, size=6000, dtype=np.uint8)), b""]
    run = Run(ac, o, reps, 2)
    run.feed([stream0[:first], stream1[:1]])
    assert run.st.held()[0] == back
    run.feed([stream0[first:first + 1], stream1[1:2]])
    assert run.out[0].endswith(reps[0])
    run.feed([stream0[first + 1:first + 1 + plen // 3], stream1[2:]])
    run.feed([stream0[first + 1 + plen // 3:], b""])
    assert run.st.held()[0] == plen // 2  # the half pattern after the last match
    run.close()


@pytest.mark.parametrize("table", ["deletions", "same-length", "longer", "all-empty"])
def test_replacement_tables(table):
    pats, hay = workload(5000, 0xAC5000, 24 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(7)
    if table == "deletions":
        reps = [b"" if i % 2 else b"-" for i in range(len(pats))]
    elif table == "same-length":
        reps = [b"*" * len(p) for p in pats]
    elif table == "longer":
        reps = [bytes(rng.integers(33, 127, size=len(p) + int(rng.integers(1, 3000)), dtype=np.uint8))
                for p in pats]
    else:
        reps = [b""] * len(pats)
    got = run_feeds(ac, o, reps, dealt(split_hay(hay, 4, rng), rng, 5))
    total = sum(map(len, got))
    assert total < hay.size if table in ("deletions", "all-empty") else total >= hay.size


@pytest.mark.parametrize("ci", [False, True])
def test_high_and_control_bytes(ci):
    """Patterns and text over the whole byte range, case-insensitive automata included."""
    rng = np.random.default_rng(31 + ci)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(40)]
    pats += [b"\x00\x00", b"\xff\xfe\xff", b"Ab\xc3\xa9", b"\r\n\r\n"]
    pats = list(dict.fromkeys(pats))
    hay = rng.integers(0, 256, size=12 << 10, dtype=np.uint8)
    for i in range(0, hay.size - 16, 97):
        q = pats[(i // 97) % len(pats)]
        hay[i:i + len(q)] = np.frombuffer(q, np.uint8)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    run_feeds(ac, o, mixed_reps(len(pats), rng), dealt(split_hay(hay, 4, rng), rng, 6))


def test_reset_and_flush_between_feeds():
    """Flushes and resets of some streams and of all, between feeds: a flushed stream comes out whole, restarts at
    offset 0, and its later outputs are those of a fresh stream given the same bytes."""
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(NESTED)
    o = O.Oracle(NESTED, kind=O.KIND_DFA)
    reps = [b"<%d>" % i if i % 3 else b"" for i in range(len(NESTED))]
    rng = np.random.default_rng(8)
    alpha = np.frombuffer(b"abcz", np.uint8)
    feeds = dealt([bytes(rng.choice(alpha, size=150)) for _ in range(5)], rng, 12)
    run = Run(ac, o, reps, 5)
    fresh = Run(ac, o, reps, 5)
    for i, f in enumerate(feeds):
        if i == 3:
            run.flush([1, 3])
        if i == 5:
            run.flush([4, 0], raw=True)
        if i == 7:
            run.st.reset([2])  # the held bytes are discarded unemitted
            run.data[2], run.out[2] = b"", b""
            assert run.st.positions()[2] == 0
        if i == 9:
            run.flush()
            fresh.flush()
        got = run.feed(f)
        if i >= 9:
            assert got == fresh.feed(f), "a flushed stream goes on as a fresh one"
    run.close()
    fresh.close()


@pytest.mark.parametrize("form", FORMS[:3])
def test_overflow_writes_nothing_and_changes_nothing(form):
    """cap = needed - 1: ACG_E_OVERFLOW with the exact size, nothing written, positions and held unchanged; the
    retry gives what a run without the overflow gives.  The same for flush."""
    pats, hay = workload(5000, 0xAC5000, 24 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(4)
    reps = mixed_reps(len(pats), rng, 400)
    feeds = dealt(split_hay(hay, 5, rng), rng, 4)
    clean = Run(ac, o, reps, 5)
    want = [clean.feed(f, form) for f in feeds]
    st = ac.replace_streams(5, reps)
    for i, f in enumerate(feeds):
        need = sum(map(len, want[i]))
        pos, held = st.positions(), st.held()
        if need:
            rc, n, buf, oo = raw_feed(st, f, form, need - 1)
            check_sentinels(buf, oo, n, rc)
            assert rc == ab.E_OVERFLOW and n == need, (rc, n, need)
            assert np.array_equal(st.positions(), pos) and np.array_equal(st.held(), held)
        # the size query: no output at all
        rc, n, _, _ = raw_feed(st, f, form, 0)
        assert (rc, n) == ((ab.E_OVERFLOW, need) if need else (0, 0))
        if not need:
            continue
        rc, n, buf, oo = raw_feed(st, f, form, need)
        o_ = oo[1:-1].astype(np.int64)
        b = buf[PAD:PAD + n].tobytes()
        assert rc == 0 and [b[o_[s]:o_[s + 1]] for s in range(5)] == want[i], i
    held = st.held()
    need = int(held.sum())
    assert need
    rc, n, buf, oo = raw_flush(st, None, need - 1)
    check_sentinels(buf, oo, n, rc)
    assert rc == ab.E_OVERFLOW and n == need and np.array_equal(st.held(), held)
    assert st.flush() == clean.flush()
    st.close()
    clean.st.close()


def test_error_codes_change_nothing():
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(NESTED)
    reps = [b"x"] * len(NESTED)
    st = ac.replace_streams(3, reps)
    st.feed([b"xxabcab", b"zzz", b"abca"])
    pos, held = st.positions(), st.held()
    hay = np.frombuffer(b"abcabcabzzzz" * 4, np.uint8).copy()
    out = np.zeros(256, np.uint8)
    oo = np.zeros(4, np.uint64)
    n = ctypes.c_uint64()
    f, g = ab._lib.acg_streams_replace_feed, ab._lib.acg_streams_replace_feed_devout
    u = np.array([0, 3, 6, 9], np.uint64)
    hp, up, op, oop, np_ = hay.ctypes.data, u.ctypes.data, out.ctypes.data, oo.ctypes.data, ctypes.byref(n)
    # decreasing offsets and offsets past the haystack, with the offsets on the host and "on the device"
    for offs in ([0, 9, 4, 20], [0, 5, 9, 49], [3, 2, 2, 2]):
        b = np.array(offs, np.uint64)
        assert f(st._h, hp, 0, hay.size, b.ctypes.data, 3, op, 256, oop, np_) == E_INVALID_SPAN
        for on_dev in (0, 1):
            assert g(st._h, hp, hay.size, b.ctypes.data, on_dev, 3, op, 256, oop, np_) == E_INVALID_SPAN
    assert f(st._h, hp, 0, hay.size, up, 2, op, 256, oop, np_) == E_INVALID_ARG       # n_streams
    assert f(st._h, hp, 0, hay.size, up, 3, None, 256, oop, np_) == E_INVALID_ARG     # NULL out with cap
    assert f(st._h, hp, 0, hay.size, up, 3, op, 256, None, np_) == E_INVALID_ARG      # NULL out_offsets
    assert f(st._h, hp, 0, hay.size, up, 3, op, 256, oop, None) == E_INVALID_ARG      # NULL out_len
    assert f(st._h, hp, 0, hay.size, None, 3, op, 256, oop, np_) == E_INVALID_ARG     # NULL chunk offsets
    assert g(st._h, hp, hay.size, up, 0, 3, op, 256, None, np_) == E_INVALID_ARG
    # the find_iter feed on a replace set, and the replace calls on find_iter and overlapping sets
    rec = np.zeros(64, ab.DOC_MATCH_DTYPE)
    assert ab._lib.acg_streams_feed(st._h, hp, 0, hay.size, up, 3, rec.ctypes.data, 64, np_) == E_INVALID_ARG
    assert ab._lib.acg_streams_feed_devout(st._h, hp, hay.size, up, 0, 3, rec.ctypes.data, 64, oop,
                                           np_) == E_INVALID_ARG
    for overlapping in (False, True):
        with ac.streams(3, overlapping) as other:
            assert f(other._h, hp, 0, hay.size, up, 3, op, 256, oop, np_) == E_INVALID_ARG
            assert g(other._h, hp, hay.size, up, 0, 3, op, 256, oop, np_) == E_INVALID_ARG
            assert ab._lib.acg_streams_flush(other._h, None, 0, op, 256, oop, np_) == E_INVALID_ARG
            assert ab._lib.acg_streams_held(other._h, oop) == E_INVALID_ARG
            assert not other.positions().any()
    # flush: an id out of range, a duplicate, NULL out_offsets / out_len, NULL out with cap
    fl = ab._lib.acg_streams_flush
    for ids in ([3], [0, 2, 0], [1, 1]):
        a = np.array(ids, np.uint64)
        assert fl(st._h, a.ctypes.data, a.size, op, 256, oop, np_) == E_INVALID_ARG, ids
    assert fl(st._h, None, 0, op, 256, None, np_) == E_INVALID_ARG
    assert fl(st._h, None, 0, op, 256, oop, None) == E_INVALID_ARG
    assert fl(st._h, None, 0, None, 256, oop, np_) == E_INVALID_ARG
    assert ab._lib.acg_streams_held(st._h, None) == E_INVALID_ARG
    assert np.array_equal(st.positions(), pos) and np.array_equal(st.held(), held)
    assert st.flush() == [b"xxabcab"[-int(held[0]):] if held[0] else b"", b"zzz"[3 - int(held[1]):],
                          b"abca"[4 - int(held[2]):]]
    st.close()


def test_creation_errors():
    def code(ac, n=4, reps=None, table=None):
        h = ctypes.c_void_p()
        _, rptr, roffs = ac._replacement_table(reps if reps is not None else [b"x"] * ac.patterns_len())
        if table is not None:
            rptr, roffs = table
        rc = ab._lib.acg_streams_create_replace(ac._h, n, rptr, None if roffs is None else roffs.ctypes.data,
                                                0 if roffs is None else roffs.size - 1, ctypes.byref(h))
        if rc == 0:
            ab._lib.acg_streams_free(h)
        return rc

    for kind in (ab.MatchKind.LeftmostFirst, ab.MatchKind.LeftmostLongest):
        ac = ab.AhoCorasick.builder().match_kind(kind).build([b"abc"])
        assert code(ac) == -12 and code(ac, table=(None, None)) == -12
        with pytest.raises(ab.MatchError):
            ac.replace_streams(2, [b"x"])
    ac = ab.AhoCorasick.builder().build([b"abc", b""])
    assert code(ac) == -14
    ac = ab.AhoCorasick.builder().start_kind(ab.StartKind.Anchored).build([b"abc"])
    assert code(ac) == -11
    ac = ab.AhoCorasick.builder().build([b"abc", b"de"])
    assert code(ac, 0) == E_INVALID_ARG and code(ac, 1 << 32) == E_INVALID_ARG
    # the table: a wrong count, decreasing offsets, NULL offsets, NULL bytes behind non-empty offsets
    data = np.frombuffer(b"xyz", np.uint8).copy()
    assert code(ac, table=(data.ctypes.data, np.array([0, 1], np.uint64))) == E_INVALID_ARG
    assert code(ac, table=(data.ctypes.data, np.array([0, 2, 1], np.uint64))) == E_INVALID_ARG
    assert code(ac, table=(data.ctypes.data, None)) == E_INVALID_ARG
    assert code(ac, table=(None, np.array([0, 1, 3], np.uint64))) == E_INVALID_ARG
    assert code(ac, table=(None, np.array([5, 5, 5], np.uint64))) == 0          # all empty: no bytes needed
    assert code(ac, table=(data.ctypes.data - 1, np.array([1, 2, 4], np.uint64))) == 0  # offsets need not start at 0
    assert code(ac, 1) == 0
    ac2 = ab.AhoCorasick.builder().start_kind(ab.StartKind.Both).build([b"abc"])
    assert code(ac2) == 0


def test_table_is_copied_and_offsets_need_not_start_at_zero():
    """The set keeps its own copy of the table: the caller's arrays can change after creation."""
    ac = ab.AhoCorasick.builder().build([b"abc", b"de"])
    data = np.frombuffer(b"__XY-", np.uint8).copy()
    offs = np.array([2, 4, 5], np.uint64)
    h = ctypes.c_void_p()
    assert ab._lib.acg_streams_create_replace(ac._h, 1, data.ctypes.data, offs.ctypes.data, 2, ctypes.byref(h)) == 0
    data[:] = ord("!")
    offs[:] = 0
    out = np.zeros(64, np.uint8)
    oo = np.zeros(2, np.uint64)
    n = ctypes.c_uint64()
    hay = np.frombuffer(b"abcde", np.uint8).copy()
    u = np.array([0, 5], np.uint64)
    assert ab._lib.acg_streams_replace_feed(h, hay.ctypes.data, 0, 5, u.ctypes.data, 1, out.ctypes.data, 64,
                                            oo.ctypes.data, ctypes.byref(n)) == 0
    assert out[:n.value].tobytes() == b"XY-"
    ab._lib.acg_streams_free(h)


def test_python_surface():
    """ReplaceStreams: ValueError for a wrong table; feed, feed_np, flush and flush_np agree with each other and
    with the list and (values, offsets) input forms; str replacements; closed sets refuse calls."""
    ac = ab.AhoCorasick.builder().build(NESTED)
    with pytest.raises(ValueError):
        ac.replace_streams(2, ["x"])
    reps = ["<%d>" % i for i in range(len(NESTED))]
    with ac.replace_streams(3, reps) as a, ac.replace_streams(3, reps) as b:
        for chunk in ([b"abca", b"", b"zz"], [b"b", b"cabc", b"zz"], [b"abcabz", b"a", b""]):
            lists = a.feed(chunk)
            vals = np.frombuffer(b"".join(chunk), np.uint8).copy()
            offs = np.r_[0, np.cumsum([len(c) for c in chunk])]
            v, o = b.feed_np((vals, offs))
            assert o.dtype == np.uint64 and o.size == 4 and o[-1] == v.size
            assert lists == [v.tobytes()[o[i]:o[i + 1]] for i in range(3)]
        assert np.array_equal(a.positions(), b.positions()) and np.array_equal(a.held(), b.held())
        v, o = b.flush_np([2, 0])
        assert a.flush([2, 0]) == [v.tobytes()[o[i]:o[i + 1]] for i in range(2)]
        assert a.flush([]) == [] and a.positions()[1] == b.positions()[1] != 0
        with pytest.raises(ValueError):
            a.feed([b"abc"])
        with pytest.raises(ValueError):
            a.flush([-1])
        with pytest.raises(ab.DeviceError):
            a.flush([1, 1])
    with pytest.raises(ValueError):
        a.feed([b"a", b"b", b"c"])
    with pytest.raises(ValueError):
        a.held()
