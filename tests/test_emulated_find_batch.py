"""Batched find (acg_find_batch) on the dry-run build of the kernels (tests/emu/), document by document
against the oracle's try_find on each document alone.

The contract: found[d] and out[d] are what try_find returns on document d alone (offsets relative to it),
with (0, d, 0, 0) for a document without a match.  Both engines are covered: the prefilter engine's
unordered scan reduced to the smallest key per document, and the per-document sequential kernel (anchored
inputs, the empty pattern, `earliest` on leftmost automata, Engine.Sequential)."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import workload as W  # noqa: E402
from test_emulated_batch import _DevView, build, doc_offsets, emulated_library, plant_at_boundaries  # noqa: E402,F401
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402
from test_prefilter_plan import plan_of  # noqa: E402


def expected_first(o, hay, offs, anchored=False, earliest=False):
    """The oracle's try_find on every document alone: (found [n_docs], records [n_docs, 4] as doc, pid,
    start, end)."""
    n = offs.size - 1
    found = np.zeros(n, bool)
    rec = np.zeros((n, 4), np.uint64)
    rec[:, 0] = np.arange(n)
    for d in range(n):
        m = o.try_find(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]), anchored=anchored, earliest=earliest)
        if m is not None:
            found[d] = True
            rec[d, 1:] = m
    return found, rec


def records(r):
    return np.stack([r["doc"].astype(np.uint64), r["pid"].astype(np.uint64), r["start"].astype(np.uint64),
                     r["end"].astype(np.uint64)], axis=1) if len(r) else np.zeros((0, 4), np.uint64)


def check_first(ac, o, hay, offs, ctx, anchored=False, earliest=False, device=True):
    """find_batch_np on a host haystack (and a device-resident one) against the oracle; returns the
    engine the call took."""
    want_found, want = expected_first(o, hay, offs, anchored, earliest)
    views = [hay, _DevView(hay)] if device else [hay]
    engine = None
    for v in views:
        found, r = ac.find_batch_np((v, offs), anchored=anchored, earliest=earliest)
        assert found.dtype == bool and found.shape == (offs.size - 1,), ctx
        assert np.array_equal(found, want_found), (ctx, type(v).__name__, np.flatnonzero(found != want_found)[:5])
        bad = np.flatnonzero((records(r) != want).any(axis=1))
        assert bad.size == 0, (ctx, type(v).__name__, bad[:5], records(r)[bad[:3]], want[bad[:3]])
        engine = ac.last_stats()["engine"]
    return want_found, engine


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants(name):
    """Every prefilter kernel variant, planted matches across, at and next to document boundaries, with and
    without `earliest`; the per-document sequential kernel gives the same answer."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, min(nbytes, 256 << 10), ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    offs = doc_offsets(hay.size, seed)
    plant_at_boundaries(hay, offs, pats, seed)
    if ci:
        W.flip_case(hay, 7)
    ac = build(pats, kind, ci)
    plan = plan_of(ac)
    assert plan.supported and not plan.brute
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    found, engine = check_first(ac, o, hay, offs, name)
    assert engine == int(ab.Engine.Prefilter)
    assert found.sum() > 50 and (~found).sum() > 50
    # `earliest`: Standard stays on the prefilter engine; a leftmost automaton takes the sequential one unless
    # the reference gives it the packed prefilter (then `earliest` is ignored)
    packed = kind != 0 and ac.prefilter_kind() == 4
    _, engine = check_first(ac, o, hay, offs, (name, "earliest"), earliest=True)
    assert engine == int(ab.Engine.Prefilter if kind == 0 or packed else ab.Engine.Sequential), (name, engine)
    if packed:
        assert ac.find_batch_np((hay, offs), earliest=True)[1].tobytes() == \
            ac.find_batch_np((hay, offs))[1].tobytes()
    ac.set_engine(ab.Engine.Sequential)
    check_first(ac, o, hay, offs, (name, "sequential"), device=False)
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


@pytest.mark.parametrize("name,pats,kw", BYTESCAN_SETS[:3] + BYTESCAN_SETS[4:5])
def test_bytescan_automata(name, pats, kw):
    kind, ci = kw.get("kind", 0), kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=64 << 10)].copy()
    for i in range(0, hay.size - 64, 577):
        p = pats[(i // 577) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    offs = doc_offsets(hay.size, 3, max_len=1024)
    plant_at_boundaries(hay, offs, pats, 4)
    ac = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).build(pats)
    assert plan_of(ac).bs_n >= 1
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci)
    found, engine = check_first(ac, o, hay, offs, name)
    assert engine == int(ab.Engine.Prefilter) and found.any()


def test_match_kinds_differ():
    """`abcd` and `bc` on `abcd`: Standard reports the first match state entered (bc), the leftmost kinds the
    match at the smallest start; `ab` / `abcd` separate leftmost-first from leftmost-longest."""
    cases = {
        (b"abcd", b"bc"): {0: (1, 1, 3), 1: (0, 0, 4), 2: (0, 0, 4)},
        (b"ab", b"abcd"): {0: (0, 0, 2), 1: (0, 0, 2), 2: (1, 0, 4)},
    }
    docs = [b"abcd", b"", b"xxabcdxx", b"abc", b"a", b"zzzzabcd"]
    for pats, want in cases.items():
        for kind, first in want.items():
            for engine in (ab.Engine.Auto, ab.Engine.Sequential):
                ac = build(list(pats), kind, engine=engine)
                got = [m.as_tuple() if m else None for m in ac.find_batch(docs)]
                o = O.Oracle(list(pats), match_kind=kind, kind=O.KIND_DFA)
                assert got == [o.try_find(d) for d in docs], (pats, kind, engine)
                assert got[0] == first, (pats, kind, engine, got)


def test_short_documents_and_earliest():
    """Thousands of documents shorter than 16 bytes (empty and 1-byte ones among them), every match kind,
    with and without `earliest`."""
    pats = [b"abcd", b"bcde", b"cdab", b"dd", b"abcdabcd", b"bc"] + W.make_patterns(300, 5)
    rng = np.random.default_rng(9)
    hay = rng.choice(np.frombuffer(b"abcde", dtype=np.uint8), size=40000)
    offs = np.concatenate([[0], np.cumsum(rng.integers(0, 16, size=6000))]).astype(np.int64)
    offs = offs[offs <= hay.size]
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        for earliest in (False, True):
            found, engine = check_first(ac, o, hay, offs, (kind, earliest), earliest=earliest)
            assert found.any() and not found.all()
            assert engine == int(ab.Engine.Sequential if earliest and kind else ab.Engine.Prefilter)


def test_packed_prefilter_ignores_earliest():
    """A leftmost automaton the reference gives its packed (Teddy) prefilter: an unanchored try_find returns
    the confirmed leftmost match whether or not `earliest` is asked for, so the prefilter engine serves it."""
    pats = [b"sam", b"frodo", b"pippin", b"merry", b"gandalf", b"sauron", b"samwise"]
    docs = [b"samwise and frodo", b"", b"foo gandalf", b"sa", b"mer", b"merry pippin", b"ssamwise"]
    ac = build(pats, 1)
    o = O.Oracle(pats, match_kind=1, kind=O.KIND_DFA)
    assert ac.prefilter_kind() == 4 and o.prefilter_kind == O.PRE_PACKED
    got = [m.as_tuple() if m else None for m in ac.find_batch(docs, earliest=True)]
    assert got == [o.try_find(d, earliest=True) for d in docs]
    assert got == [m.as_tuple() if m else None for m in ac.find_batch(docs)]
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    # the same automaton without the packed prefilter: `earliest` reports the first match state entered
    o2 = O.Oracle(pats, match_kind=1, kind=O.KIND_DFA, prefilter=False)
    ac2 = ab.AhoCorasick.builder().match_kind(1).kind(ab.AhoCorasickKind.DFA).prefilter(False).build(pats)
    got2 = [m.as_tuple() if m else None for m in ac2.find_batch(docs, earliest=True)]
    assert got2 == [o2.try_find(d, earliest=True) for d in docs]
    assert got2[0] == (0, 0, 3)


def test_anchored_and_empty_pattern_automata():
    """The per-document sequential kernel: anchored input (StartKind Anchored / Both), the empty pattern (a
    single try_find has no empty-match rule: (pid, 0, 0) where the oracle reports it), Engine.Sequential."""
    rng = np.random.default_rng(11)
    hay = rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=6000)
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab"]
    for kind in (0, 1, 2):
        for sk in (ab.StartKind.Anchored, ab.StartKind.Both):
            ac = build(pats, kind, start_kind=sk)
            o = O.Oracle(pats, match_kind=kind, start_kind=int(sk), kind=O.KIND_DFA)
            for earliest in (False, True):
                found, engine = check_first(ac, o, hay, offs, (kind, sk, earliest), anchored=True, earliest=earliest)
                assert engine == int(ab.Engine.Sequential) and found.any() and not found.all()
            if sk == ab.StartKind.Both:
                check_first(ac, o, hay, offs, (kind, sk, "unanchored"))
        ac = build(pats + [b""], kind)
        o = O.Oracle(pats + [b""], match_kind=kind, kind=O.KIND_DFA)
        assert not plan_of(ac).supported
        for earliest in (False, True):
            found, engine = check_first(ac, o, hay, offs, (kind, "empty pattern", earliest), earliest=earliest)
            assert engine == int(ab.Engine.Sequential) and found.all()
        empty = ab.AhoCorasick.builder().match_kind(kind).build([b""])
        assert [m.as_tuple() for m in empty.find_batch([b"", b"abc"])] == [(0, 0, 0), (0, 0, 0)]


def test_prefilter_override_and_error_codes():
    pats = [b"abcd", b"bcd"]
    docs = [b"xabcdx", b"", b"bcd"]
    # Walk means Auto here
    assert [m and m.as_tuple() for m in build(pats, engine=ab.Engine.Walk).find_batch(docs)] == \
        [(0, 1, 5), None, (1, 0, 3)]
    # a prefilter override the input cannot use: anchored, no plan, `earliest` on a leftmost automaton
    with pytest.raises(ab.DeviceError) as e:
        build(pats, start_kind=ab.StartKind.Both, engine=ab.Engine.Prefilter).find_batch(docs, anchored=ab.Anchored.Yes)
    assert e.value.code == -22
    with pytest.raises(ab.DeviceError):
        build(pats + [b""], engine=ab.Engine.Prefilter).find_batch(docs)
    with pytest.raises(ab.DeviceError):   # (no packed prefilter, so `earliest` is not ignored)
        build(pats, 1, engine=ab.Engine.Prefilter, prefilter=False).find_batch(docs, earliest=True)
    assert [m.as_tuple() for m in build(pats, 1, engine=ab.Engine.Prefilter).find_batch(docs)[::2]] == \
        [(0, 1, 5), (1, 0, 3)]
    assert build(pats, 0, engine=ab.Engine.Prefilter).find_batch(docs, earliest=True)[0].as_tuple() == (0, 1, 5)
    # StartKind errors, as acg_find gives them
    with pytest.raises(ab.MatchError) as e:
        build(pats).find_batch(docs, anchored=ab.Anchored.Yes)
    assert e.value.kind == "InvalidInputAnchored"
    with pytest.raises(ab.MatchError) as e:
        build(pats, start_kind=ab.StartKind.Anchored).find_batch(docs)
    assert e.value.kind == "InvalidInputUnanchored"


def test_offsets_and_document_counts():
    ac = build([b"abcd"])
    hay = np.frombuffer(b"abcdabcd", dtype=np.uint8).copy()
    for offs in ([0, 5, 3, 8], [0, 4, 9], [2, 1], [0, 8, 8, 9]):
        with pytest.raises(ValueError):
            ac.find_batch_np((hay, np.array(offs)))
    # n_docs >= 2^32 is refused before the offsets are read
    offs = np.zeros(2, np.uint64)
    out = np.zeros(1, ab.DOC_MATCH_DTYPE)
    found = np.zeros(1, np.uint8)
    assert ab._lib.acg_find_batch(ac._h, hay.ctypes.data, 0, hay.size, offs.ctypes.data, 1 << 32, 0, 0,
                                  out.ctypes.data, found.ctypes.data) == -22
    # no documents: nothing written
    out[:] = 7
    found[:] = 7
    for o in ([0], [5]):
        offs = np.array(o, np.uint64)
        assert ab._lib.acg_find_batch(ac._h, hay.ctypes.data, 0, hay.size, offs.ctypes.data, 0, 0, 0,
                                      out.ctypes.data, found.ctypes.data) == 0
    assert found[0] == 7 and out["pid"][0] == 7
    assert ac.find_batch([]) == [] and ac.find_batch_np((hay, np.array([3])))[0].shape == (0,)
    # one document: the single-haystack try_find, offsets relative to the document
    pats, big = workload(5000, 0xAC5000, 96 << 10)
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        for s, e in ((1000, big.size - 333), (5, 9), (77, 77)):
            found, r = ac.find_batch_np((big, np.array([s, e])))
            m = ac.try_find(np.ascontiguousarray(big[s:e]))
            assert bool(found[0]) == (m is not None), (kind, s, e)
            assert (r["doc"][0], r["pid"][0], r["start"][0], r["end"][0]) == \
                ((0,) + m.as_tuple() if m else (0, 0, 0, 0)), (kind, s, e)


def test_documents_across_buckets_and_list_input(monkeypatch):
    """256-byte order buckets (the find scan is unordered, so they must not matter) and str / bytes lists."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    n, seed, nbytes, kind, ci = VARIANTS["stride2_narrow"]
    pats, hay = workload(n, seed, 96 << 10)
    W.plant(hay, pats, 8, period=61, window=40)
    offs = doc_offsets(hay.size, 21, max_len=700)
    plant_at_boundaries(hay, offs, pats, 22)
    for kind in (0, 1):
        check_first(build(pats, kind), O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, ("buckets", kind))
    ac = build([b"ab", b"b"])
    assert [m and m.as_tuple() for m in ac.find_batch(["xab", b"b", "", "q"])] == [(0, 1, 3), (1, 0, 1), None, None]


@pytest.mark.skipif(os.environ.get("ACB_EMU_WINSHIFT") is not None, reason="runs inside the subprocess below")
def test_documents_across_queue_windows():
    """4 KiB queue windows (2 GiB on the device; the window size is fixed when the library loads, hence
    a fresh process) with 2 KiB buckets."""
    env = dict(os.environ, ACB_EMU_WINSHIFT="12", ACB_EMU_BUCKETSHIFT="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", str(Path(__file__)), "-k",
                        "prefilter_variants or short_documents"], capture_output=True, text=True, env=env,
                       timeout=1800, cwd=str(ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
