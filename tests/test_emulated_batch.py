"""Batched search (acg_find_iter_batch / acg_find_overlapping_batch / acg_is_match_batch) on the dry-run
build of the kernels (tests/emu/), document by document against the oracle run on each document alone.

The batch contract: the records tagged doc == d are exactly the single-haystack call's list on document d
(offsets relative to it, same order), documents ascending.  Both engines are covered: the prefilter
engine over the whole buffer with every match bounded by its document, and the per-document sequential
kernel (anchored inputs, the empty pattern, Engine.Sequential)."""
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
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import packed, workload as W  # noqa: E402
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402
from test_prefilter_plan import plan_of  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    import build_emu
    lib = ctypes.CDLL(str(build_emu.build(asan=os.environ.get("ACB_EMU_ASAN") == "1")))
    ab._declare(lib)
    packed._declare(lib)
    saved = ab._lib, packed._lib
    ab._lib = packed._lib = lib
    try:
        yield lib
    finally:
        ab._lib, packed._lib = saved


def doc_offsets(n_bytes, seed, max_len=4096):
    """CSR bounds over [0, n_bytes): log-uniform lengths in [1, max_len], with empty, 1-byte and runs of
    short (< 16 B) documents mixed in."""
    rng = np.random.default_rng(seed)
    lens = []
    total = 0
    while total < n_bytes:
        r = rng.random()
        if r < 0.05:
            run = [0] * int(rng.integers(1, 3))
        elif r < 0.10:
            run = [1]
        elif r < 0.15:
            run = list(rng.integers(0, 16, size=int(rng.integers(4, 40))))
        else:
            run = [int(np.exp(rng.uniform(0, np.log(max_len))))]
        for x in run:
            lens.append(int(min(x, n_bytes - total)))
            total += lens[-1]
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def plant_at_boundaries(hay, offs, pats, seed):
    """Patterns that straddle a document boundary, end exactly at a document's end, or start exactly at
    a document's start."""
    rng = np.random.default_rng(seed)
    for i, b in enumerate(offs[1:-1]):
        p = np.frombuffer(pats[int(rng.integers(len(pats)))], dtype=np.uint8)
        at = (b - len(p) // 2, b - len(p), b)[i % 3]
        if 0 <= at and at + len(p) <= hay.size:
            hay[at:at + len(p)] = p


def expected(o, hay, offs, what, anchored=False):
    """The oracle on every document alone, as (doc, pid, start, end) records."""
    fn = o.find_overlapping_iter_np if what == "overlapping" else o.find_iter_np
    parts = []
    for d in range(offs.size - 1):
        doc = np.ascontiguousarray(hay[offs[d]:offs[d + 1]])
        r = fn(doc, anchored=anchored)
        if len(r):
            parts.append(np.stack([np.full(len(r), d, np.uint64), r["pid"].astype(np.uint64),
                                   r["start"].astype(np.uint64), r["end"].astype(np.uint64)], axis=1))
    return np.concatenate(parts) if parts else np.zeros((0, 4), np.uint64)


def records(got):
    return np.stack([got["doc"].astype(np.uint64), got["pid"].astype(np.uint64), got["start"].astype(np.uint64),
                     got["end"].astype(np.uint64)], axis=1) if len(got) else np.zeros((0, 4), np.uint64)


def expected_flags(o, hay, offs, anchored=False):
    return np.array([len(o.find_iter_np(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]), anchored=anchored)) > 0
                     for d in range(offs.size - 1)], dtype=bool)


def eq(got, want, ctx=None):
    g = records(got)
    assert g.shape == want.shape, (g.shape, want.shape, ctx)
    assert np.array_equal(g, want), ctx


def check_all(ac, o, hay, offs, kind, ctx, anchored=False, device=True):
    """find_iter (host and device-resident haystack), overlapping (Standard), is_match."""
    batch = (hay, offs)
    want = expected(o, hay, offs, "iter", anchored)
    eq(ac.find_iter_batch_np(batch, anchored=anchored), want, (ctx, "find_iter"))
    if device:
        eq(ac.find_iter_batch_np((_DevView(hay), offs), anchored=anchored), want, (ctx, "find_iter, device"))
    if kind == 0 and not anchored:
        eq(ac.find_overlapping_iter_batch_np(batch), expected(o, hay, offs, "overlapping"), (ctx, "overlapping"))
    flags = ac.is_match_batch(batch, anchored=anchored)
    assert np.array_equal(flags, expected_flags(o, hay, offs, anchored)), (ctx, "is_match")
    return want


class _DevView:
    """A host array presented as a CUDA tensor (hay_on_device = 1): the dry run's device memory is host
    memory, so this takes the device-resident path of the library."""
    is_cuda = True
    dtype = "torch.uint8"

    def __init__(self, a):
        self.a = a

    def is_contiguous(self):
        return True

    def data_ptr(self):
        return self.a.ctypes.data

    def numel(self):
        return self.a.size


def build(pats, kind=0, ci=False, engine=ab.Engine.Auto, **kw):
    b = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA)
    for k, v in kw.items():
        getattr(b, k)(v)
    return b.build(pats).set_engine(engine)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants(name):
    """Every prefilter kernel variant, planted matches across, at and next to document boundaries; the
    per-document sequential kernel on the same batch gives the same answer."""
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
    want = check_all(ac, o, hay, offs, kind, name)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert len(want) > 100
    # matches the concatenated search would report across boundaries exist, and none is reported here
    whole = o.find_overlapping_iter_np(hay) if kind == 0 else o.find_iter_np(hay)
    doc_of = np.searchsorted(offs, whole["start"].astype(np.int64), side="right") - 1
    assert (whole["end"].astype(np.int64) > offs[doc_of + 1]).sum() > 10
    ac.set_engine(ab.Engine.Sequential)
    check_all(ac, o, hay, offs, kind, (name, "sequential"), device=False)
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
    check_all(ac, o, hay, offs, kind, name)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


def test_short_documents_inside_one_tile():
    """Thousands of documents shorter than 16 bytes: many documents per probed 16-byte group."""
    pats = [b"abcd", b"bcde", b"cdab", b"dd", b"abcdabcd"] + W.make_patterns(300, 5)
    rng = np.random.default_rng(9)
    hay = np.frombuffer(bytes(rng.choice(list(b"abcde"), size=40000)), dtype=np.uint8).copy()
    offs = np.concatenate([[0], np.cumsum(rng.integers(0, 16, size=6000))]).astype(np.int64)
    offs = offs[offs <= hay.size]
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        check_all(ac, o, hay, offs, kind, kind)


def test_anchored_and_empty_pattern_automata():
    """The automata the prefilter engine cannot serve: anchored input (StartKind Anchored / Both) and the
    empty pattern -- the per-document sequential kernel."""
    rng = np.random.default_rng(11)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=6000)), dtype=np.uint8).copy()
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab"]
    for kind in (0, 1, 2):
        for sk in (ab.StartKind.Anchored, ab.StartKind.Both):
            ac = build(pats, kind, start_kind=sk)
            o = O.Oracle(pats, match_kind=kind, start_kind=int(sk), kind=O.KIND_DFA)
            check_all(ac, o, hay, offs, kind, (kind, sk), anchored=True)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
            if sk == ab.StartKind.Both:
                check_all(ac, o, hay, offs, kind, (kind, sk, "unanchored"))
        ac = build(pats + [b""], kind)
        o = O.Oracle(pats + [b""], match_kind=kind, kind=O.KIND_DFA)
        assert not plan_of(ac).supported
        check_all(ac, o, hay, offs, kind, (kind, "empty pattern"))
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


def test_error_codes_are_those_of_the_single_calls():
    pats = [b"abcd", b"bcd"]
    docs = [b"xabcdx", b"", b"bcd"]
    lf = build(pats, 1)
    with pytest.raises(ab.MatchError) as e:
        lf.find_overlapping_iter_batch(docs)
    assert e.value.kind == "UnsupportedOverlapping"
    with pytest.raises(ab.MatchError) as e:
        build(pats).find_iter_batch(docs, anchored=ab.Anchored.Yes)
    assert e.value.kind == "InvalidInputAnchored"
    with pytest.raises(ab.MatchError) as e:
        build(pats, start_kind=ab.StartKind.Anchored).is_match_batch(docs)
    assert e.value.kind == "InvalidInputUnanchored"
    # a prefilter override the automaton cannot serve
    with pytest.raises(ab.DeviceError):
        build(pats + [b""], engine=ab.Engine.Prefilter).find_iter_batch(docs)
    # the Walk override means Auto here
    assert [[m.as_tuple() for m in d] for d in build(pats, engine=ab.Engine.Walk).find_iter_batch(docs)] == \
        [[(0, 1, 5)], [], [(1, 0, 3)]]


def test_invalid_offsets_raise_value_error():
    ac = build([b"abcd"])
    hay = np.frombuffer(b"abcdabcd", dtype=np.uint8).copy()
    for offs in ([0, 5, 3, 8], [0, 4, 9], [2, 1], [0, 8, 8, 9]):
        for fn in (ac.find_iter_batch_np, ac.find_overlapping_iter_batch_np, ac.is_match_batch):
            with pytest.raises(ValueError):
                fn((hay, np.array(offs)))
    with pytest.raises(ValueError):
        ac.find_iter_batch((hay, np.array([0, -1])))
    # n_docs >= 2^32 is refused before the offsets are read
    cnt = ctypes.c_uint64()
    offs = np.zeros(2, np.uint64)
    rc = ab._lib.acg_find_iter_batch(ac._h, hay.ctypes.data, 0, hay.size, offs.ctypes.data, 1 << 32, 0, None, 0,
                                     ctypes.byref(cnt))
    assert rc == -22


def test_no_documents_and_one_document():
    pats, hay = workload(5000, 0xAC5000, 96 << 10)
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        for offs in ([0], [17]):
            assert len(ac.find_iter_batch_np((hay, np.array(offs)))) == 0
            assert ac.find_iter_batch((hay, np.array(offs))) == []
            assert ac.is_match_batch((hay, np.array(offs))).shape == (0,)
        assert ac.find_iter_batch([]) == []
        # one document: the single-haystack call, bit for bit (offsets relative to the document)
        s, e = 1000, hay.size - 333
        got = ac.find_iter_batch_np((hay, np.array([s, e])))
        single = ac.try_find_iter_np(np.ascontiguousarray(hay[s:e]))
        assert len(got) == len(single) > 50 and (got["doc"] == 0).all()
        for k in ("pid", "start", "end"):
            assert np.array_equal(got[k], single[k]), (kind, k)
        if kind == 0:
            got = ac.find_overlapping_iter_batch_np((hay, np.array([0, hay.size])))
            single = ac.try_find_overlapping_iter_np(hay)
            assert got.tobytes() == single.tobytes()   # same layout, doc 0 in the pad


def test_overflow_retry_and_list_input():
    """More matches than the first output buffer holds: the two-call protocol on both engines."""
    docs = [b"a" * 3000, b"", "aaa", b"ba" * 1000, b"a"]
    want = [[(0, i, i + 1) for i in range(len(d))] if d != b"ba" * 1000 else [(0, 2 * i + 1, 2 * i + 2) for i in range(1000)]
            for d in docs]
    for engine in (ab.Engine.Auto, ab.Engine.Sequential):
        ac = build([b"a"], engine=engine)
        ac._cap_hint = 16
        got = ac.find_overlapping_iter_batch(docs)
        assert [[m.as_tuple() for m in d] for d in got] == want, engine
        assert [[m.as_tuple() for m in d] for d in ac.find_iter_batch(docs)] == want, engine
        assert ac.is_match_batch(docs).tolist() == [True, False, True, True, True]


def test_documents_across_buckets(monkeypatch):
    """256-byte order buckets: documents and their matches spread over many buckets."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    n, seed, nbytes, kind, ci = VARIANTS["stride2_narrow"]
    pats, hay = workload(n, seed, 96 << 10)
    W.plant(hay, pats, 8, period=61, window=40)
    offs = doc_offsets(hay.size, 21, max_len=700)
    plant_at_boundaries(hay, offs, pats, 22)
    for kind in (0, 1):
        ac = build(pats, kind)
        check_all(ac, O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, kind, ("buckets", kind))


@pytest.mark.skipif(os.environ.get("ACB_EMU_WINSHIFT") is not None, reason="runs inside the subprocess below")
def test_documents_across_queue_windows():
    """4 KiB queue windows (2 GiB on the device; the window size is fixed when the library loads, hence
    a fresh process) with 2 KiB buckets."""
    env = dict(os.environ, ACB_EMU_WINSHIFT="12", ACB_EMU_BUCKETSHIFT="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", str(Path(__file__)), "-k",
                        "prefilter_variants or short_documents"], capture_output=True, text=True, env=env,
                       timeout=1800, cwd=str(ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
