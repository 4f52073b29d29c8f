"""Stream sets (acg_streams_*) on the dry-run build of the kernels (tests/emu/).

The reference result for every stream is the oracle's find_iter / find_overlapping_iter over the concatenation of
the chunks the stream received since it was created or reset, and in find_iter mode also the host glue
stream_find_iter over an io.BytesIO of it.  Every feed is checked on its own as well: its records come in ascending
stream order, and each ends in the bytes the feed brought -- in find_iter mode that is the claim that no record of
a combined document ends inside its tail, which the device path relies on instead of filtering.  Feeds alternate
between host output, device output with host offsets and device output with "device" offsets (the dry run's device
memory is host memory), with sentinels around every output array."""
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
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402
from test_prefilter_plan import plan_of  # noqa: E402

SENTINEL = 0xA5A5A5A5A5A5A5A5
PAD = 3  # sentinel records / index entries on either side of every output
FORMS = ("host", "devout", "devout_dev_offsets")
E_INVALID_ARG, E_INVALID_SPAN = -22, -20


def raw_feed(st, chunks, form, cap=None):
    """One raw feed call of the given form into sentinel-filled arrays: (rc, n_out, records, index or None).  The
    records are a DOC_MATCH_DTYPE array of `cap` entries (default: enough), the index has n_streams + 1 entries."""
    pieces = [bytes(c) for c in chunks]
    offs = np.r_[0, np.cumsum([len(c) for c in pieces])].astype(np.uint64)
    hay = np.frombuffer(b"".join(pieces) + b"\0", np.uint8)[:-1].copy()
    if cap is None:
        cap = 4 * int(offs[-1]) + 64
    buf = np.full((cap + 2 * PAD) * 3, SENTINEL, np.uint64)
    idx = np.full(st.n_streams + 1 + 2 * PAD, SENTINEL, np.uint64)
    n = ctypes.c_uint64(12345)
    hp = hay.ctypes.data if hay.size else None
    optr = buf[PAD * 3:].ctypes.data
    if form == "host":
        rc = ab._lib.acg_streams_feed(st._h, hp, 0, hay.size, offs.ctypes.data, st.n_streams, optr, cap,
                                      ctypes.byref(n))
    else:
        rc = ab._lib.acg_streams_feed_devout(st._h, hp, hay.size, offs.ctypes.data, int(form == "devout_dev_offsets"),
                                             st.n_streams, optr, cap, idx[PAD:].ctypes.data, ctypes.byref(n))
    got = int(n.value)
    assert (buf[:PAD * 3] == SENTINEL).all(), (form, "sentinel before the records")
    if rc == 0:
        assert (buf[(PAD + got) * 3:] == SENTINEL).all(), (form, "sentinel after the records")
    assert (idx[:PAD] == SENTINEL).all() and (idx[PAD + st.n_streams + 1:] == SENTINEL).all(), (form, "index sentinels")
    rec = buf[PAD * 3:(PAD + min(got, cap)) * 3].view(ab.DOC_MATCH_DTYPE)
    return rc, got, buf, (idx[PAD:PAD + st.n_streams + 1] if form != "host" else None), rec


def feed_checked(st, chunks, form, before):
    """One feed of `form` (or the Python list form when form is None): its records, checked against the feed
    contract given the positions `before`; returns (records per stream, positions after)."""
    n = st.n_streams
    if form is None:
        rec = st.feed_np(chunks)
    else:
        rc, got, _, idx, rec = raw_feed(st, chunks, form)
        assert rc == 0, (form, rc)
        if idx is not None:
            assert np.array_equal(idx, np.searchsorted(rec["doc"], np.arange(n + 1))), (form, "index")
    after = st.positions()
    assert np.array_equal(after, before + np.array([len(c) for c in chunks], np.uint64)), "positions"
    doc = rec["doc"].astype(np.int64)
    assert (np.diff(doc) >= 0).all(), "records in ascending stream order"
    assert (rec["end"] > before[doc]).all(), "a record ends in bytes an earlier feed brought"
    assert (rec["end"] <= after[doc]).all() and (rec["start"] <= rec["end"]).all(), "a record ends past the stream"
    per = [rec[doc == s] for s in range(n)]
    return per, after


def oracle_stream(o, data, overlapping):
    h = np.frombuffer(bytes(data) + b"\0", np.uint8)[:-1].copy()
    r = o.find_overlapping_iter_np(h) if overlapping else o.find_iter_np(h)
    return [(int(p), int(s), int(e)) for p, s, e in zip(r["pid"], r["start"], r["end"])]


def tuples(recs):
    return [(int(p), int(s), int(e)) for p, s, e in zip(recs["pid"], recs["start"], recs["end"])]


def run_feeds(ac, o, feeds, overlapping, forms=FORMS, between=None, glue=None):
    """Feed `feeds` (a list of feeds, each one chunk per stream) to a new set, cycling through `forms`; checks
    every feed, then every stream against the oracle over its bytes (and the host glue in find_iter mode).
    `between(i, st)` runs before feed i.  Returns the records per stream."""
    n = len(feeds[0])
    with ac.streams(n, overlapping) as st:
        pos = np.zeros(n, np.uint64)
        got = [[] for _ in range(n)]
        data = [b"" for _ in range(n)]
        for i, chunks in enumerate(feeds):
            if between:
                between(i, st)
            per, pos = feed_checked(st, chunks, forms[i % len(forms)], pos)
            for s in range(n):
                got[s] += tuples(per[s])
                data[s] += bytes(chunks[s])
    for s in range(n):
        want = oracle_stream(o, data[s], overlapping)
        assert got[s] == want, ("stream", s, len(got[s]), len(want))
        if not overlapping and (glue if glue is not None else len(data[s]) < (16 << 10)):
            g = [m.as_tuple() for m in ac.stream_find_iter(io.BytesIO(data[s]), chunk_bytes=997)]
            assert got[s] == g, ("host glue", s)
    return got


def cut(data, rng, n_feeds):
    """`data` cut into n_feeds chunks at random points: empty and 1-byte chunks included."""
    pts = sorted(int(x) for x in rng.integers(0, len(data) + 1, size=n_feeds - 1))
    for i in range(0, len(pts), 5):  # some 1-byte chunks
        if pts[i] + 1 <= len(data):
            pts.insert(i + 1, pts[i] + 1)
    pts = sorted(pts)[:n_feeds - 1]
    b = [0] + pts + [len(data)]
    return [data[b[i]:b[i + 1]] for i in range(n_feeds)]


def dealt(streams, rng, n_feeds):
    """Each stream's bytes cut into n_feeds chunks, transposed into feeds."""
    cuts = [cut(s, rng, n_feeds) for s in streams]
    return [[c[i] for c in cuts] for i in range(n_feeds)]


def split_hay(hay, n_streams, rng):
    b = np.sort(rng.integers(0, hay.size + 1, size=n_streams - 1))
    b = np.r_[0, b, hay.size]
    return [hay[b[i]:b[i + 1]].tobytes() for i in range(n_streams)]


STANDARD_VARIANTS = [k for k, v in VARIANTS.items() if v[3] == 0]
STANDARD_BYTESCAN = [(name, pats, kw) for name, pats, kw in BYTESCAN_SETS if kw.get("kind", 0) == 0]


@pytest.mark.parametrize("overlapping", [False, True])
@pytest.mark.parametrize("name", STANDARD_VARIANTS)
def test_prefilter_variants(name, overlapping):
    """Every Standard prefilter variant, streams cut at random points, on the prefilter and sequential engines."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, 48 << 10, ci)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    assert plan_of(ac).supported
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    rng = np.random.default_rng(seed)
    feeds = dealt(split_hay(hay, 9, rng), rng, 7)
    got = run_feeds(ac, o, feeds, overlapping)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert sum(map(len, got)) > 20
    ac.set_engine(ab.Engine.Sequential)
    assert run_feeds(ac, o, feeds, overlapping) == got
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


@pytest.mark.parametrize("overlapping", [False, True])
@pytest.mark.parametrize("name,pats,kw", STANDARD_BYTESCAN)
def test_bytescan_sets(name, pats, kw, overlapping):
    ci = kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=24 << 10)].copy()
    for i in range(0, hay.size - 64, 331):
        p = pats[(i // 331) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    ac = ab.AhoCorasick.builder().ascii_case_insensitive(ci).build(pats)
    assert plan_of(ac).bs_n >= 1
    o = O.Oracle(pats, ascii_case_insensitive=ci)
    feeds = dealt(split_hay(hay, 5, rng), rng, 9)
    run_feeds(ac, o, feeds, overlapping)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


# a set where matches overlap, nest and chain: prefixes, suffixes and a periodic pattern
NESTED = [b"abcab", b"bca", b"cabcabc", b"ab", b"abcabcabcab", b"zzzz", b"zz", b"bcabz"]


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
@pytest.mark.parametrize("overlapping", [False, True])
def test_split_inside_pattern_at_every_point(overlapping, engine):
    """Stream k holds the same bytes and is cut at k bytes into a planted long pattern: every split point of it at
    once, plus tiny chunks afterwards so that the tail is built over several feeds."""
    pats = NESTED + [b"the quick brown fox jumps over the lazy dog"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats).set_engine(engine)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    body = b"xx" + b"abcabcabcabzzzzz" + b"the quick brown fox jumps over the lazy dog" + b"abcabz" * 3 + b"q"
    at = body.index(b"the quick")
    L = 43
    streams = L + 1
    feeds = [[body[:at + k] for k in range(streams)]]
    rest = [body[at + k:] for k in range(streams)]
    rng = np.random.default_rng(5)
    while any(rest):  # 0 to 3 bytes per stream and feed: shorter than back
        nxt = []
        for s in range(streams):
            k = int(rng.integers(0, 4))
            nxt.append(rest[s][:k])
            rest[s] = rest[s][k:]
        feeds.append(nxt)
    got = run_feeds(ac, o, feeds, overlapping)
    assert all(g == got[0] for g in got)
    assert (pats.index(pats[-1]), at, at + L) in got[0]


@pytest.mark.parametrize("overlapping", [False, True])
def test_repetitive_text_tiny_chunks(overlapping):
    """Periodic text, where find_iter's restart point matters: chunks of 0 to 2 bytes across many feeds."""
    pats = [b"aa", b"aaa", b"aba", b"abab", b"baba", b"b"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(11)
    streams = [bytes(rng.choice(np.frombuffer(b"ab", np.uint8), size=int(rng.integers(0, 300)))) for _ in range(6)]
    run_feeds(ac, o, dealt(streams, rng, 40), overlapping)


@pytest.mark.parametrize("plen", [1024, 4096, 65533])
@pytest.mark.parametrize("overlapping", [False, True])
def test_long_patterns_at_the_tail_limit(plen, overlapping):
    """1 KiB to 64 KiB patterns: chunks end exactly where the tail holds back = max_pattern_len - 1 bytes of a
    pattern, so the match ends with the first byte of the next feed; and matches cut at both ends of the tail."""
    rng = np.random.default_rng(plen)
    p = rng.integers(97, 101, size=plen, dtype=np.uint8).tobytes()
    # overlapping mode also reports a prefix of the pattern; in find_iter mode that prefix would end the match early
    pats = [p, b"wxyz", p[: plen // 2]] if overlapping else [p, b"wxyz"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    back = plen - 1
    filler = rng.integers(101, 110, size=3 * plen, dtype=np.uint8).tobytes()
    stream0 = filler[:plen] + p + b"wxyz" + filler[plen:2 * plen] + p + p[: plen // 2]
    # stream 0: the first feed ends one byte before the end of the pattern -- the tail is exactly `back` bytes
    first = plen + back
    # stream 1: a 1-byte chunk, then the pattern's first byte only, then the rest
    stream1 = b"x" + p + filler[:100]
    feeds = [[stream0[:first], stream1[:1]], [stream0[first:first + 1], stream1[1:2]],
             [stream0[first + 1:first + 1 + plen // 3], stream1[2:]], [stream0[first + 1 + plen // 3:], b""]]
    got = run_feeds(ac, o, feeds, overlapping, glue=False)
    assert (0, plen, 2 * plen) in got[0] and (0, 1, 1 + plen) in got[1]


@pytest.mark.parametrize("overlapping", [False, True])
def test_chunks_across_tiles_and_windows(overlapping):
    """Chunks of hundreds of KiB: combined documents over many gather tiles and prefilter tiles, with the
    pipeline chunk of host staging below the chunk size."""
    pats, hay = workload(5000, 0xAC5000, 640 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    ab._lib.acg_debug_set_pipeline_chunk(ac._h, 64 << 10)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(3)
    feeds = dealt(split_hay(hay, 3, rng), rng, 3)
    got = run_feeds(ac, o, feeds, overlapping)
    assert sum(map(len, got)) > 100


def test_engine_switch_between_feeds():
    pats, hay = workload(5000, 0xAC5000, 32 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(9)
    feeds = dealt(split_hay(hay, 4, rng), rng, 8)
    engines = [ab.Engine.Auto, ab.Engine.Sequential, ab.Engine.Prefilter]
    for overlapping in (False, True):
        run_feeds(ac, o, feeds, overlapping, between=lambda i, st: ac.set_engine(engines[i % 3]))
    ac.set_engine(ab.Engine.Auto)


@pytest.mark.parametrize("form", FORMS)
def test_overflow_writes_nothing_and_changes_nothing(form):
    """cap = needed - 1: ACG_E_OVERFLOW with the count, nothing written, positions unchanged, and the retry and the
    feeds after it give what a run without the overflow gives."""
    pats, hay = workload(5000, 0xAC5000, 32 << 10)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    rng = np.random.default_rng(4)
    feeds = dealt(split_hay(hay, 5, rng), rng, 4)
    for overlapping in (False, True):
        clean = []
        with ac.streams(5, overlapping) as st:
            for f in feeds:
                clean.append(raw_feed(st, f, form)[4].copy())
        with ac.streams(5, overlapping) as st:
            for i, f in enumerate(feeds):
                need = len(clean[i])
                if need:
                    pos = st.positions()
                    rc, n, buf, idx, _ = raw_feed(st, f, form, cap=need - 1)
                    assert rc == ab.E_OVERFLOW and n == need, (rc, n, need)
                    assert (buf == SENTINEL).all(), "overflow wrote records"
                    assert idx is None or (idx == SENTINEL).all(), "overflow wrote the index"
                    assert np.array_equal(st.positions(), pos)
                rc, n, _, _, rec = raw_feed(st, f, form, cap=need)
                assert rc == 0 and n == need and np.array_equal(rec, clean[i]), (overlapping, i)


@pytest.mark.parametrize("form", FORMS)
def test_bad_chunk_offsets_change_nothing(form):
    pats = NESTED
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    streams = [b"xxabcabcabcabzz" * 3, b"zzzzabcab" * 4, b""]
    rng = np.random.default_rng(2)
    feeds = dealt(streams, rng, 5)

    def bad(i, st):
        pos = st.positions()
        hay = np.frombuffer(b"abcabcabzzzz" * 4, np.uint8).copy()
        out = np.zeros(64, ab.DOC_MATCH_DTYPE)
        idx = np.zeros(4, np.uint64)
        n = ctypes.c_uint64()
        for offs in ([0, 9, 4, 20], [0, 5, 9, 49], [3, 2, 2, 2]):
            u = np.array(offs, np.uint64)
            if form == "host":
                rc = ab._lib.acg_streams_feed(st._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 3,
                                              out.ctypes.data, 64, ctypes.byref(n))
            else:
                rc = ab._lib.acg_streams_feed_devout(st._h, hay.ctypes.data, hay.size, u.ctypes.data,
                                                     int(form == "devout_dev_offsets"), 3, out.ctypes.data, 64,
                                                     idx.ctypes.data, ctypes.byref(n))
            assert rc == E_INVALID_SPAN, (offs, rc)
        assert np.array_equal(st.positions(), pos)

    for overlapping in (False, True):
        run_feeds(ac, o, feeds, overlapping, between=bad)


def test_argument_errors():
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(NESTED)
    hay = np.frombuffer(b"abcabc", np.uint8).copy()
    u = np.array([0, 3, 6], np.uint64)
    out = np.zeros(16, ab.DOC_MATCH_DTYPE)
    idx = np.zeros(4, np.uint64)
    n = ctypes.c_uint64()
    with ac.streams(2) as st:
        f = ab._lib.acg_streams_feed
        assert f(st._h, hay.ctypes.data, 0, 6, u.ctypes.data, 3, out.ctypes.data, 16, ctypes.byref(n)) == E_INVALID_ARG
        assert f(st._h, hay.ctypes.data, 0, 6, u.ctypes.data, 2, None, 16, ctypes.byref(n)) == E_INVALID_ARG
        assert f(st._h, hay.ctypes.data, 0, 6, u.ctypes.data, 2, out.ctypes.data, 16, None) == E_INVALID_ARG
        assert f(st._h, hay.ctypes.data, 0, 6, None, 2, out.ctypes.data, 16, ctypes.byref(n)) == E_INVALID_ARG
        g = ab._lib.acg_streams_feed_devout
        assert g(st._h, hay.ctypes.data, 6, u.ctypes.data, 0, 2, out.ctypes.data, 16, None,
                 ctypes.byref(n)) == E_INVALID_ARG
        assert g(st._h, hay.ctypes.data, 6, u.ctypes.data, 0, 1, out.ctypes.data, 16, idx.ctypes.data,
                 ctypes.byref(n)) == E_INVALID_ARG
        assert np.array_equal(st.positions(), [0, 0])
        # the size query: cap 0 and no output
        assert f(st._h, hay.ctypes.data, 0, 6, u.ctypes.data, 2, None, 0, ctypes.byref(n)) == ab.E_OVERFLOW
        assert n.value == 2 and np.array_equal(st.positions(), [0, 0])
        bad = np.array([0, 2], np.uint64)
        assert ab._lib.acg_streams_reset(st._h, bad.ctypes.data, 2) == E_INVALID_ARG
        assert ab._lib.acg_streams_positions(st._h, None) == E_INVALID_ARG
        with pytest.raises(ValueError):
            st.feed([b"abc"])
    with pytest.raises(ValueError):
        st.feed([b"a", b"b"])


def test_reset_of_some_streams():
    """Streams 1 and 3 are reset in the middle of a run: from then on they are new streams, the others go on."""
    pats = NESTED
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(8)
    alpha = np.frombuffer(b"abcz", np.uint8)
    streams = [bytes(rng.choice(alpha, size=200)) for _ in range(5)]
    feeds = dealt(streams, rng, 10)
    for overlapping in (False, True):
        with ac.streams(5, overlapping) as st:
            got = [[] for _ in range(5)]
            data = [b""] * 5
            pos = np.zeros(5, np.uint64)
            for i, f in enumerate(feeds):
                if i == 5:
                    st.reset([1, 3])
                    pos = st.positions()
                    assert pos[1] == 0 and pos[3] == 0
                    for s in (1, 3):
                        got[s], data[s] = [], b""
                per, pos = feed_checked(st, f, FORMS[i % 3], pos)
                for s in range(5):
                    got[s] += tuples(per[s])
                    data[s] += f[s]
            for s in range(5):
                assert got[s] == oracle_stream(o, data[s], overlapping), (overlapping, s)
            st.reset()
            assert not st.positions().any()
            want = list(ac.find_overlapping_iter(b"abcab") if overlapping else ac.find_iter(b"abcab"))
            assert st.feed([b"abcab"] * 5) == [want] * 5


def test_creation_errors():
    def code(ac, n=4, overlapping=0):
        h = ctypes.c_void_p()
        rc = ab._lib.acg_streams_create(ac._h, n, overlapping, ctypes.byref(h))
        if rc == 0:
            ab._lib.acg_streams_free(h)
        return rc

    for kind in (ab.MatchKind.LeftmostFirst, ab.MatchKind.LeftmostLongest):
        ac = ab.AhoCorasick.builder().match_kind(kind).build([b"abc"])
        assert code(ac) == -12 and code(ac, overlapping=1) == -13
        with pytest.raises(ab.MatchError):
            ac.streams(2)
    ac = ab.AhoCorasick.builder().build([b"abc", b""])
    assert code(ac) == -14 and code(ac, overlapping=1) == -14
    ac = ab.AhoCorasick.builder().start_kind(ab.StartKind.Anchored).build([b"abc"])
    assert code(ac) == -11 and code(ac, overlapping=1) == -11
    ac = ab.AhoCorasick.builder().build([b"abc"])
    assert code(ac, 0) == E_INVALID_ARG and code(ac, 1 << 32) == E_INVALID_ARG
    assert code(ac, 1) == 0
    ac2 = ab.AhoCorasick.builder().start_kind(ab.StartKind.Both).build([b"abc"])
    assert code(ac2) == 0


def test_list_and_torch_free_forms_agree():
    """feed() and feed_np() give the raw calls' records; (values, offsets) chunks as the batch calls take them."""
    ac = ab.AhoCorasick.builder().build(NESTED)
    with ac.streams(3) as a, ac.streams(3) as b:
        for chunk in ([b"abca", b"", b"zz"], [b"b", b"cabc", b"zz"], [b"abcabz", b"a", b""]):
            lists = a.feed(chunk)
            vals = np.frombuffer(b"".join(chunk), np.uint8).copy()
            offs = np.r_[0, np.cumsum([len(c) for c in chunk])]
            rec = b.feed_np((vals, offs))
            assert lists == ab.AhoCorasick._per_doc(rec, 3)
        assert np.array_equal(a.positions(), b.positions())
