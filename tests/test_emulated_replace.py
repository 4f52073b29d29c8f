"""Replace per document (acg_replace_all_batch / _devout) on the dry-run build of the kernels (tests/emu/).

Every result is compared with three independent computations: the splice of src/automaton.rs:525-550 run in
numpy over the same handle's find_iter_batch_np records, the same splice over the oracle's find_iter on sampled
documents alone, and the host glue replace_all_bytes(document) on sampled documents.  Host output, device output
with host offsets and device output with "device" offsets (the dry run's device memory is host memory) must give
the same bytes, and no call may write outside its output: the output and out_offsets carry sentinels on both
sides."""
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
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import workload as W  # noqa: E402
from test_emulated_batch import build, doc_offsets, emulated_library, plant_at_boundaries  # noqa: E402,F401
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402

SENTINEL = 0xA5A5A5A5A5A5A5A5
BYTE_SENTINEL = 0xA5
PAD = 40  # output bytes on either side that no call may touch


def splice(doc, starts, ends, pids, reps):
    """The loop of try_replace_all_bytes over one document's matches."""
    out, last = [], 0
    for s, e, p in zip(starts, ends, pids):
        out += [doc[last:s], reps[p]]
        last = e
    out.append(doc[last:])
    return b"".join(out)


def from_records(rec, hay, offs, reps):
    """(values, offsets) of the splice over batch records, document by document."""
    hb = hay.tobytes()
    n_docs = offs.size - 1
    at = np.searchsorted(rec["doc"], np.arange(n_docs + 1))
    parts = []
    for d in range(n_docs):
        r = rec[at[d]:at[d + 1]]
        parts.append(splice(hb[offs[d]:offs[d + 1]], r["start"].tolist(), r["end"].tolist(), r["pid"].tolist(), reps))
    return b"".join(parts), np.r_[0, np.cumsum([len(p) for p in parts], dtype=np.uint64)].astype(np.uint64)


def raw(ac, hay, offs, reps, cap, dev=False, on_dev=False, at=PAD, out=True):
    """One raw call into sentinel-filled arrays: (rc, out_len, out buffer with `at` bytes before, out_offsets with
    one entry before and after)."""
    _, rptr, roffs = ac._replacement_table(reps)
    u = np.ascontiguousarray(offs, dtype=np.int64).astype(np.uint64)
    n_docs = u.size - 1
    buf = np.full(cap + at + PAD, BYTE_SENTINEL, np.uint8)
    oo = np.full(n_docs + 3, SENTINEL, np.uint64)
    n = ctypes.c_uint64(12345)
    hp = hay.ctypes.data if hay.size else None
    optr = buf[at:].ctypes.data if out else None
    if dev:
        rc = ab._lib.acg_replace_all_batch_devout(ac._h, hp, hay.size, u.ctypes.data, int(on_dev), n_docs, rptr,
                                                  roffs.ctypes.data, roffs.size - 1, optr, cap, oo[1:].ctypes.data,
                                                  ctypes.byref(n))
    else:
        rc = ab._lib.acg_replace_all_batch(ac._h, hp, 0, hay.size, u.ctypes.data, n_docs, rptr, roffs.ctypes.data,
                                           roffs.size - 1, optr, cap, oo[1:].ctypes.data, ctypes.byref(n))
    return rc, int(n.value), buf, oo


def check_raw(ac, hay, offs, reps, values, out_offsets, ctx):
    """The raw calls, host and device output, with exactly the room needed (at two alignments), one byte less,
    and none (the size query)."""
    need = values.size
    want_oo = np.r_[SENTINEL, out_offsets, SENTINEL].astype(np.uint64)
    for dev, on_dev, at in ((False, False, PAD), (True, False, PAD + 3), (True, True, PAD + 9), (False, False, 7)):
        rc, n, buf, oo = raw(ac, hay, offs, reps, need, dev, on_dev, at)
        assert rc == 0 and n == need, (ctx, dev, on_dev, rc, n, need)
        assert buf[at:at + need].tobytes() == values.tobytes(), (ctx, dev, on_dev, "bytes")
        assert (buf[:at] == BYTE_SENTINEL).all() and (buf[at + need:] == BYTE_SENTINEL).all(), (ctx, "sentinels")
        assert np.array_equal(oo, want_oo), (ctx, dev, on_dev, "out_offsets")
        if need:  # one byte short: the required size, nothing written
            rc, n, buf, oo = raw(ac, hay, offs, reps, need - 1, dev, on_dev, at)
            assert rc == ab.E_OVERFLOW and n == need, (ctx, dev, "overflow", rc, n)
            assert (buf == BYTE_SENTINEL).all() and (oo == SENTINEL).all(), (ctx, dev, "overflow wrote")
        rc, n, buf, oo = raw(ac, hay, offs, reps, 0, dev, on_dev, at, out=False)  # size query
        assert n == need and rc == (ab.E_OVERFLOW if need else 0), (ctx, dev, "size query", rc, n)
        assert (buf == BYTE_SENTINEL).all(), (ctx, dev, "size query wrote")
        assert np.array_equal(oo, want_oo) if not need else (oo == SENTINEL).all(), (ctx, dev, "size query offsets")


def check(ac, o, hay, offs, reps, ctx, sample=12, glue=True):
    """replace_all_batch_np against the records' splice, the oracle and the host glue on sampled documents; the
    list form and the raw calls against it.  Returns (values, offsets)."""
    offs = np.asarray(offs, dtype=np.int64)
    n_docs = offs.size - 1
    reps = [r.encode() if isinstance(r, str) else bytes(r) for r in reps]
    values, out_offsets = ac.replace_all_batch_np((hay, offs), reps)
    assert values.dtype == np.uint8 and out_offsets.dtype == np.uint64 and out_offsets.shape == (n_docs + 1,), ctx
    want, want_offs = from_records(ac.find_iter_batch_np((hay, offs)), hay, offs, reps)
    assert np.array_equal(out_offsets, want_offs), (ctx, "offsets", np.flatnonzero(out_offsets != want_offs)[:10])
    assert values.tobytes() == want, (ctx, "bytes")
    rng = np.random.default_rng(n_docs)
    docs = set(rng.integers(0, n_docs, size=min(sample, n_docs)).tolist()) if n_docs else set()
    docs |= {0, n_docs - 1} if n_docs else set()
    vb = values.tobytes()
    for d in sorted(docs):
        lo, hi = int(offs[d]), int(offs[d + 1])
        doc = hay[lo:hi].tobytes()
        got = vb[out_offsets[d]:out_offsets[d + 1]]
        r = o.find_iter_np(np.frombuffer(doc, np.uint8).copy())
        assert got == splice(doc, r["start"].tolist(), r["end"].tolist(), r["pid"].tolist(), reps), (ctx, "oracle", d)
        if glue:
            assert got == ac.replace_all_bytes(doc, reps), (ctx, "replace_all_bytes", d)
    if n_docs:
        assert ac.replace_all_batch((hay, offs), reps) == [vb[out_offsets[d]:out_offsets[d + 1]]
                                                           for d in range(n_docs)], ctx
    check_raw(ac, hay, offs, reps, values, out_offsets, ctx)
    return values, out_offsets


def mixed_reps(pats, seed):
    """One replacement per pattern: deletions, shorter, same-length and longer ones, some holding the pattern."""
    rng = np.random.default_rng(seed)
    out = []
    for i, p in enumerate(pats):
        k = int(rng.integers(0, 5))
        out.append((b"", p[: len(p) // 2], b"#" * len(p), b"[%d]" % i + p + p, p[::-1])[k])
    return out


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants(name):
    """Every prefilter kernel variant, matches across, at and next to document boundaries; then the sequential
    engine forced on the same batch."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, min(nbytes, 64 << 10), ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    offs = doc_offsets(hay.size, seed)
    plant_at_boundaries(hay, offs, pats, seed)
    if ci:
        W.flip_case(hay, 7)
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    reps = mixed_reps(pats, seed)
    want = check(ac, o, hay, offs, reps, name, glue=False)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert len(ac.find_iter_batch_np((hay, offs))) > 20, name
    ac.set_engine(ab.Engine.Sequential)
    got = check(ac, o, hay, offs, reps, (name, "sequential"), glue=False)
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
    assert all(np.array_equal(g, w) for g, w in zip(got, want)), (name, "engines")


@pytest.mark.parametrize("name,pats,kw", BYTESCAN_SETS[:3] + BYTESCAN_SETS[4:5])
def test_bytescan_automata(name, pats, kw):
    kind, ci = kw.get("kind", 0), kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=24 << 10)].copy()
    for i in range(0, hay.size - 64, 577):
        p = pats[(i // 577) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    offs = doc_offsets(hay.size, 3, max_len=1024)
    plant_at_boundaries(hay, offs, pats, 4)
    ac = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).build(pats)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci)
    check(ac, o, hay, offs, mixed_reps(pats, 9), name)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


def test_match_kinds_case_insensitive_and_duplicates():
    rng = np.random.default_rng(11)
    hay = np.frombuffer(b"abcABC", np.uint8)[rng.integers(0, len(b"abcABC"), size=5000)]
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab", b"ab"]
    reps = [b"", b"XYZW", b"b", b"..", b"abcab", b"Q"]
    for kind in (0, 1, 2):
        for ci in (False, True):
            for engine in (ab.Engine.Auto, ab.Engine.Sequential):
                ac = build(pats, kind, ci, engine=engine)
                o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
                check(ac, o, hay, offs, reps, (kind, ci, engine))


def test_empty_pattern_inserts_everywhere():
    """The empty pattern: its replacement goes in at every position, into empty documents too, on the
    sequential engine the automaton leaves no plan for."""
    ac = build([b""])
    assert ac.replace_all_batch([b"ab", b"", b"c", b""], [b"-"]) == [b"-a-b-", b"-", b"-c-", b"-"]
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
    assert ac.replace_all_batch([b"ab", b""], [b""]) == [b"ab", b""]
    rng = np.random.default_rng(21)
    hay = np.frombuffer(b"abc", np.uint8)[rng.integers(0, len(b"abc"), size=3000)]
    offs = doc_offsets(hay.size, 22, max_len=48)
    pats = [b"ab", b"", b"ca", b"abc"]
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        values, _ = check(ac, o, hay, offs, [b"<>", b"_", b"", b"ABCD"], (kind, "empty pattern"))
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        check(ac, o, hay, offs, [b"", b"", b"", b""], (kind, "deleting"))
    ac = build([b""])
    values, out_offsets = check(ac, O.Oracle([b""], kind=O.KIND_DFA), hay, offs, [b"|"], "only the empty pattern")
    assert values.size == hay.size + hay.size + offs.size - 1


def test_replacement_lengths_and_no_rescan():
    """Deletions, shorter, equal and longer replacements, a 64 KiB one, replacements made of pattern bytes (the
    output is not searched again), and an output shorter than the input."""
    rng = np.random.default_rng(64)
    hay = np.frombuffer(b"abcd xyz", np.uint8)[rng.integers(0, len(b"abcd xyz"), size=12 << 10)]
    offs = doc_offsets(hay.size, 65, max_len=900)
    pats = [b"ab", b"xyz", b"d d", b"ca"]
    big = bytes(rng.integers(0, 256, size=64 << 10, dtype=np.uint8))
    for kind in (0, 1):
        for engine in (ab.Engine.Auto, ab.Engine.Sequential):
            ac = build(pats, kind, engine=engine)
            o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
            shorter, _ = check(ac, o, hay, offs, [b"", b"X", b"", b"c"], (kind, engine, "shorter"))
            assert shorter.size < hay.size
            same, _ = check(ac, o, hay, offs, [b"AB", b"XYZ", b"D-D", b"CA"], (kind, engine, "same"))
            assert same.size == hay.size
            check(ac, o, hay, offs, [b"abab", b"xyzxyz", b"d dd d", b"abcab"], (kind, engine, "pattern bytes"))
            check(ac, o, hay, offs, [big, b"", b"12345678901234567", big[:1000]], (kind, engine, "64 KiB"),
                  sample=4)
    ac = build([b"ab"])
    assert ac.replace_all_batch([b"aabb", b"abab", b"xab"], [b"ab"]) == [b"aabb", b"abab", b"xab"]
    assert ac.replace_all_batch([b"aabb"], [b"a"]) == [b"aab"]  # not searched again


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_batch_shapes(engine):
    """No document, one, all empty, documents without a match (a shifted copy), one document holding every
    match; the host output through a staging ring of 4 KiB chunks."""
    pats, hay = workload(5000, 0xAC5000, 24 << 10)
    W.plant(hay, pats, 3, period=97, window=40)
    ac = build(pats, 0, engine=engine)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    reps = mixed_reps(pats, 5)
    for offs in ([0], [17], [hay.size]):
        values, out_offsets = check(ac, o, hay, np.array(offs), reps, (engine, offs))
        assert values.size == 0 and out_offsets.tolist() == [0]
    check(ac, o, np.zeros(0, np.uint8), np.array([0]), reps, (engine, "empty buffer"))
    check(ac, o, np.zeros(0, np.uint8), np.array([0, 0, 0]), reps, (engine, "empty documents of an empty buffer"))
    check(ac, o, hay, np.array([300, hay.size - 333]), reps, (engine, "one document"))
    values, out_offsets = check(ac, o, hay, np.array([5, 5, 5, 5]), reps, (engine, "all empty"))
    assert values.size == 0 and out_offsets.tolist() == [0, 0, 0, 0]
    # without a match in the batch: a copy of the span
    clean = np.full(9000, ord("."), np.uint8)
    values, out_offsets = check(ac, o, clean, np.array([3, 100, 100, 4000, 8999]), reps, (engine, "no match"))
    assert values.tobytes() == clean[3:8999].tobytes() and out_offsets.tolist() == [0, 97, 97, 3997, 8996]
    # documents without a match between others, and one document holding every match
    offs = np.r_[np.zeros(40, np.int64), np.arange(0, 64, 2), hay.size, [hay.size] * 7]
    check(ac, o, hay, offs, reps, (engine, "every match in one document"))
    ab._lib.acg_debug_set_pipeline_chunk.argtypes = [ctypes.c_void_p, ctypes.c_uint64]
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 4096) == 0
    check(ac, o, hay, doc_offsets(hay.size, 31), [r + r for r in reps], (engine, "staging ring"), sample=4)


def test_doc_examples_as_one_document_batches():
    # src/ahocorasick.rs:651-760, replace_all / replace_all_bytes
    app, app_hay = ["append", "appendage", "app"], b"append the app to the appendage"
    lf = ab.AhoCorasick.builder().match_kind(ab.MatchKind.LeftmostFirst).build(app)
    assert lf.replace_all_batch([app_hay], [b"x", b"y", b"z"]) == [b"x the z to the xage"]
    assert lf.replace_all_batch([app_hay], ["x", "y", "z"]) == [lf.replace_all_bytes(app_hay, ["x", "y", "z"])]
    ac = ab.AhoCorasick.new(["fox", "brown", "quick"])
    assert ac.replace_all_batch([b"The quick brown fox."], ["sloth", "grey", "slow"]) == [b"The slow grey sloth."]
    values, offs = ac.replace_all_batch_np([b"The quick brown fox.", b"", b"a fox"], ["sloth", "grey", "slow"])
    assert values.tobytes() == b"The slow grey sloth.a sloth" and offs.tolist() == [0, 20, 20, 27]


def test_error_codes():
    pats = [b"abcd", b"bcd"]
    docs = [b"xabcdx", b"", b"bcd"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    reps = [b"1", b"22"]
    # the errors of acg_find_iter_batch with anchored = 0
    cases = [build(pats, start_kind=ab.StartKind.Anchored),  # InvalidInputUnanchored
             build(pats + [b""], engine=ab.Engine.Prefilter)]  # an override the automaton cannot use
    for ac in cases:
        r = reps + [b""] * (ac.patterns_len() - len(reps))
        with pytest.raises((ab.MatchError, ab.DeviceError)) as want:
            ac.find_iter_batch_np((hay, offs))
        with pytest.raises(type(want.value)) as got:
            ac.replace_all_batch_np((hay, offs), r)
        assert got.value.code == want.value.code
        for dev, on_dev in ((False, False), (True, False), (True, True)):
            rc, n, buf, oo = raw(ac, hay, offs, r, 64, dev, on_dev)
            assert rc == want.value.code and (buf == BYTE_SENTINEL).all() and (oo == SENTINEL).all(), (dev, on_dev)
    ac = build(pats)
    with pytest.raises(ValueError):  # one replacement per pattern, as the host glue
        ac.replace_all_batch_np((hay, offs), [b"1"])
    for bad in ([0, 5, 3, 9], [0, 4, 10], [2, 1], [10]):
        with pytest.raises(ValueError):
            ac.replace_all_batch_np((hay, np.array(bad)), reps)
        for dev, on_dev in ((True, False), (True, True)):
            rc, n, buf, oo = raw(ac, hay, np.array(bad), reps, 64, dev, on_dev)
            assert rc == -20 and (buf == BYTE_SENTINEL).all() and (oo == SENTINEL).all(), (bad, on_dev)
    lib = ab._lib
    u = np.array([0, 6, 6, hay.size], np.uint64)
    out = np.zeros(64, np.uint8)
    oo = np.zeros(8, np.uint64)
    n = ctypes.c_uint64()
    good = np.array([0, 1, 3], np.uint64)
    data = np.frombuffer(b"122", np.uint8)

    def host(h=ac._h, offsets=u.ctypes.data, n_docs=3, rb=data.ctypes.data, ro=good.ctypes.data, nr=2,
             o=out.ctypes.data, cap=64, oop=oo.ctypes.data, nl=ctypes.byref(n)):
        return lib.acg_replace_all_batch(h, hay.ctypes.data, 0, hay.size, offsets, n_docs, rb, ro, nr, o, cap, oop, nl)

    def devout(h=ac._h, offsets=u.ctypes.data, n_docs=3, rb=data.ctypes.data, ro=good.ctypes.data, nr=2,
               o=out.ctypes.data, cap=64, oop=oo.ctypes.data, nl=ctypes.byref(n), on_dev=0):
        return lib.acg_replace_all_batch_devout(h, hay.ctypes.data, hay.size, offsets, on_dev, n_docs, rb, ro, nr, o,
                                                cap, oop, nl)

    want = [ac.replace_all_bytes(d, reps) for d in docs]
    assert want == [b"x1x", b"", b"22"]
    assert host() == 0 and n.value == 5 and out[:5].tobytes() == b"x1x22" and oo[:4].tolist() == [0, 3, 3, 5]
    for call in (host, devout):
        assert call(nr=1) == -22 and call(nr=3) == -22  # n_reps != patterns_len
        dec = np.array([0, 2, 1], np.uint64)
        assert call(ro=dec.ctypes.data) == -22  # decreasing rep_offsets
        assert call(ro=None) == -22 and call(rb=None) == -22  # no table, no bytes behind it
        assert call(rb=None, ro=np.array([5, 5, 5], np.uint64).ctypes.data) == 0  # empty replacements need none
        assert call(o=None) == -22  # no output with room
        assert call(oop=None) == -22 and call(nl=None) == -22 and call(h=None) == -22 and call(offsets=None) == -22
        assert call(n_docs=1 << 32) == -22  # before the offsets are read, as the batch calls
        oo[:] = 7
        assert call(n_docs=0, o=None, cap=0) == 0 and oo[0] == 0 and n.value == 0
    assert devout(n_docs=1 << 32, on_dev=1) == -22
    # the table's first offset need not be 0
    shifted = np.frombuffer(b"....122", np.uint8)
    assert host(rb=shifted.ctypes.data, ro=np.array([4, 5, 7], np.uint64).ctypes.data) == 0
    assert out[:5].tobytes() == b"x1x22"
