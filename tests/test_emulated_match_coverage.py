"""Match coverage per document (acg_match_coverage_batch / _devout) on the dry-run build of the kernels
(tests/emu/).

Every result is compared with two independent computations: the union of the same handle's find_iter_batch_np /
find_overlapping_iter_batch_np records, taken on the host with numpy (+1 at each start, -1 at each end, a running
sum), and the oracle run on sampled documents alone.  Host output, device output with host offsets and device
output with "device" offsets (the dry run's device memory is host memory) must give the same bytes, and no call
may write a mask entry outside [offsets[0], offsets[n_docs])."""
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
from test_emulated_batch_devout import offsets_arg  # noqa: E402
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402

SENTINEL = 0xA5A5A5A5A5A5A5A5
MASK_SENTINEL = 0xA5
PAD = 40  # mask bytes on either side of the haystack that no call may touch


def union(starts, ends, size):
    """The byte mask of the union of the half-open intervals [starts, ends) over [0, size)."""
    d = np.zeros(size + 1, np.int64)
    np.add.at(d, starts.astype(np.int64), 1)
    np.add.at(d, ends.astype(np.int64), -1)
    return np.cumsum(d[:-1]) > 0


def from_records(rec, offs, size):
    """(covered, mask) of batch records: their union, per document."""
    base = offs[rec["doc"].astype(np.int64)].astype(np.int64)
    mask = union(base + rec["start"].astype(np.int64), base + rec["end"].astype(np.int64), size)
    cs = np.r_[0, np.cumsum(mask)]
    covered = (cs[offs[1:]] - cs[offs[:-1]]).astype(np.uint64)
    inside = np.zeros(size, bool)
    if offs.size > 1:
        inside[offs[0]:offs[-1]] = True
    return covered, mask & inside


def raw_host(ac, hay, offs, ov, anchored=ab.Anchored.No, with_mask=True):
    """acg_match_coverage_batch into sentinel-filled host arrays: (rc, covered, mask with PAD bytes each side)."""
    u = np.ascontiguousarray(offs, dtype=np.int64).astype(np.uint64)
    covered = np.full(max(u.size - 1, 1), SENTINEL, np.uint64)
    mask = np.full(hay.size + 2 * PAD, MASK_SENTINEL, np.uint8)
    rc = ab._lib.acg_match_coverage_batch(ac._h, hay.ctypes.data if hay.size else None, 0, hay.size, u.ctypes.data,
                                          u.size - 1, int(anchored), int(ov), covered.ctypes.data,
                                          mask[PAD:].ctypes.data if with_mask else None)
    return rc, covered[:u.size - 1], mask


def devout(ac, hay, offs, on_dev, ov, anchored=ab.Anchored.No, with_mask=True):
    """The coverage into sentinel-filled "device" arrays: (covered, mask with PAD bytes each side)."""
    keep, arg, n_docs = offsets_arg(offs, on_dev)
    covered = np.full(max(n_docs, 1), SENTINEL, np.uint64)
    mask = np.full(hay.size + 2 * PAD, MASK_SENTINEL, np.uint8)
    ac.match_coverage_batch_devout(hay.ctypes.data if hay.size else 0, hay.size, arg, covered.ctypes.data,
                                   mask[PAD:].ctypes.data if with_mask else None, overlapping=ov, anchored=anchored,
                                   n_docs=n_docs)
    return covered[:n_docs], mask


def padded(mask, offs):
    """What a sentinel-filled padded mask must hold after a call that writes `mask` over [offs[0], offs[-1])."""
    want = np.full(mask.size + 2 * PAD, MASK_SENTINEL, np.uint8)
    if offs.size > 1:
        lo, hi = int(offs[0]), int(offs[-1])
        want[PAD + lo:PAD + hi] = mask[lo:hi]
    return want


def check(ac, o, hay, offs, overlapping, ctx, anchored=ab.Anchored.No, sample=12, min_covered=0):
    """Host output against the records' union and the oracle; the raw host call and device output (both offset
    placements, with and without a mask) byte for byte against it.  Returns (covered, mask)."""
    offs = np.asarray(offs, dtype=np.int64)
    n_docs = offs.size - 1
    records = (ac.find_overlapping_iter_batch_np if overlapping else ac.find_iter_batch_np)((hay, offs),
                                                                                           anchored=anchored)
    covered, mask = ac.match_coverage_batch_np((hay, offs), overlapping=overlapping, anchored=anchored, mask=True)
    want_cov, want_mask = from_records(records, offs, hay.size)
    assert covered.dtype == np.uint64 and covered.shape == (n_docs,), ctx
    assert mask.dtype == bool and mask.shape == (hay.size,), ctx
    assert np.array_equal(covered, want_cov), (ctx, "covered", np.flatnonzero(covered != want_cov)[:10])
    assert np.array_equal(mask, want_mask), (ctx, "mask", np.flatnonzero(mask != want_mask)[:10])
    assert int(covered.sum()) >= min_covered, (ctx, int(covered.sum()))
    assert np.array_equal(ac.match_coverage_batch_np((hay, offs), overlapping=overlapping, anchored=anchored),
                          covered), (ctx, "without mask")
    rng = np.random.default_rng(n_docs)
    docs = set(rng.integers(0, n_docs, size=min(sample, n_docs)).tolist()) if n_docs else set()
    docs |= {0, n_docs - 1} if n_docs else set()
    fn = o.find_overlapping_iter_np if overlapping else o.find_iter_np
    for d in sorted(docs):
        lo, hi = int(offs[d]), int(offs[d + 1])
        r = fn(np.ascontiguousarray(hay[lo:hi]), anchored=bool(anchored))
        m = union(r["start"], r["end"], hi - lo)
        assert covered[d] == m.sum() and np.array_equal(mask[lo:hi], m), (ctx, "oracle doc", d)
    want_padded = padded(mask.view(np.uint8), offs)
    rc, cov_raw, mask_raw = raw_host(ac, hay, offs, overlapping, anchored)
    assert rc == 0 and cov_raw.tobytes() == covered.tobytes(), (ctx, "raw host", rc)
    assert mask_raw.tobytes() == want_padded.tobytes(), (ctx, "raw host mask")
    for on_dev in (False, True):
        cov_dv, mask_dv = devout(ac, hay, offs, on_dev, overlapping, anchored)
        assert cov_dv.tobytes() == covered.tobytes(), (ctx, "devout", on_dev)
        assert mask_dv.tobytes() == want_padded.tobytes(), (ctx, "devout mask", on_dev)
        cov_dv, mask_dv = devout(ac, hay, offs, on_dev, overlapping, anchored, with_mask=False)
        assert cov_dv.tobytes() == covered.tobytes() and (mask_dv == MASK_SENTINEL).all(), (ctx, "no mask", on_dev)
    return covered, mask


def flags_of(kind):
    return (False, True) if kind == 0 else (False,)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants(name):
    """Every prefilter kernel variant, with matches across, at and next to document boundaries; then the
    sequential engine forced on the same batch."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, min(nbytes, 96 << 10), ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    offs = doc_offsets(hay.size, seed)
    plant_at_boundaries(hay, offs, pats, seed)
    if ci:
        W.flip_case(hay, 7)
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    for ov in flags_of(kind):
        want = check(ac, o, hay, offs, ov, (name, ov), min_covered=100)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        ac.set_engine(ab.Engine.Sequential)
        got = check(ac, o, hay, offs, ov, (name, ov, "sequential"))
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), (name, ov, "engines")
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac.set_engine(ab.Engine.Auto)


@pytest.mark.parametrize("name,pats,kw", BYTESCAN_SETS[:3] + BYTESCAN_SETS[4:5])
def test_bytescan_automata(name, pats, kw):
    kind, ci = kw.get("kind", 0), kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=32 << 10)].copy()
    for i in range(0, hay.size - 64, 577):
        p = pats[(i // 577) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    offs = doc_offsets(hay.size, 3, max_len=1024)
    plant_at_boundaries(hay, offs, pats, 4)
    ac = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).build(pats)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci)
    for ov in flags_of(kind):
        check(ac, o, hay, offs, ov, (name, ov), min_covered=100)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


def test_anchored_empty_and_duplicate_patterns():
    """The sequential engine chosen by anchored input and by the empty pattern (whose matches cover nothing);
    duplicate patterns; all three match kinds."""
    rng = np.random.default_rng(11)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=4000)), dtype=np.uint8).copy()
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab", b"ab"]
    for kind in (0, 1, 2):
        for sk in (ab.StartKind.Anchored, ab.StartKind.Both):
            ac = build(pats, kind, start_kind=sk)
            o = O.Oracle(pats, match_kind=kind, start_kind=int(sk), kind=O.KIND_DFA)
            check(ac, o, hay, offs, False, (kind, sk), anchored=ab.Anchored.Yes, min_covered=20)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac = build(pats + [b""], kind)
        o = O.Oracle(pats + [b""], match_kind=kind, kind=O.KIND_DFA)
        for ov in flags_of(kind):
            check(ac, o, hay, offs, ov, (kind, "empty pattern", ov), min_covered=0 if kind == 0 and not ov else 20)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac = build(pats, kind)
        for ov in flags_of(kind):
            check(ac, O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, ov, (kind, "duplicates", ov),
                  min_covered=100)
    ac = build([b""])
    for ov in (False, True):
        covered, mask = check(ac, O.Oracle([b""], kind=O.KIND_DFA), hay, offs, ov, ("only the empty pattern", ov))
        assert not covered.any() and not mask.any()


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_nested_chained_and_full_cover(engine):
    """Prefix-closed and suffix-closed sets (every match nested in a longer one), matches that end exactly where
    the next starts, matches ending at the document end, and documents covered completely."""
    docs = [b"xabcdx", b"abcdabcd", b"abab", b"ababa", b"", b"xxabcd", b"dcba", b"abcdxabc", b"a", b"bcd"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    sets = {"prefix-closed": [b"a", b"ab", b"abc", b"abcd"], "suffix-closed": [b"d", b"cd", b"bcd", b"abcd"],
            "chains": [b"ab", b"ba", b"cd", b"x", b"bc"]}
    for name, pats in sets.items():
        for kind in (0, 1, 2):
            ac = build(pats, kind, engine=engine)
            o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
            for ov in flags_of(kind):
                covered, mask = check(ac, o, hay, offs, ov, (engine, name, kind, ov))
                if name == "chains":  # ab|cd|ab|cd and ab|ab: each match ends where the next starts
                    assert covered[1] == 8 and covered[2] == 4
                if ov and name == "prefix-closed":  # every match nested in abcd, or ab
                    assert covered[1] == 8 and covered[2] == 4
                if ov and name == "suffix-closed":  # ending at the document end
                    assert covered[1] == 8 and covered[5] == 4 and covered[9] == 3
    # random dense sets over a two-letter alphabet: long runs of overlapping, nested and touching matches
    rng = np.random.default_rng(5)
    hay = np.frombuffer(bytes(rng.choice(list(b"ab"), size=6000)), dtype=np.uint8).copy()
    offs = doc_offsets(hay.size, 6, max_len=300)
    pats = sorted({bytes(rng.choice(list(b"ab"), size=int(rng.integers(2, 9)))) for _ in range(12)})
    for kind in (0, 1, 2):
        ac = build(pats, kind, engine=engine)
        for ov in flags_of(kind):
            check(ac, O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, ov, (engine, "ab", kind, ov),
                  min_covered=1000)


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_batch_shapes(engine):
    """No document, one, all empty, empty documents at the start / middle / end, one document holding every match."""
    pats, hay = workload(5000, 0xAC5000, 24 << 10)
    W.plant(hay, pats, 3, period=97, window=40)
    ac = build(pats, 0, engine=engine)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for ov in (False, True):
        for offs in ([0], [17], [hay.size]):
            covered, mask = check(ac, o, hay, np.array(offs), ov, (engine, ov, offs))
            assert covered.size == 0 and not mask.any()
        check(ac, o, np.zeros(0, np.uint8), np.array([0]), ov, (engine, ov, "empty buffer"))
        check(ac, o, hay, np.array([300, hay.size - 333]), ov, (engine, ov, "one document"), min_covered=100)
        covered, _ = check(ac, o, hay, np.array([5, 5, 5, 5]), ov, (engine, ov, "all empty"))
        assert covered.tolist() == [0, 0, 0]
        m = hay.size // 2
        offs = np.array([0, 0, 0, 100, m, m, m + 50, hay.size, hay.size, hay.size])
        covered, _ = check(ac, o, hay, offs, ov, (engine, ov, "empty documents"), min_covered=100)
        assert covered[0] == covered[1] == covered[4] == covered[7] == covered[8] == 0
        offs = np.r_[np.zeros(40, np.int64), np.arange(0, 64, 2), hay.size, [hay.size] * 7]
        covered, _ = check(ac, o, hay, offs, ov, (engine, ov, "every match in one document"), min_covered=100)
        assert covered[:71].sum() == 0 and covered[72:].sum() == 0


def test_long_patterns_and_the_staging_ring():
    """1 KiB patterns planted across and at the ends of documents, nested in each other; the host mask through
    a staging ring of several 4 KiB chunks, and through one chunk."""
    rng = np.random.default_rng(1024)
    base = bytes(rng.integers(97, 123, size=1100, dtype=np.uint8))
    pats = [base[:1024], base[50:1074], base[:1050], base[1000:1100] + b"zz"]
    hay = np.frombuffer(bytes(rng.integers(97, 123, size=24 << 10, dtype=np.uint8)), dtype=np.uint8).copy()
    for at in (0, 1500, 3000, 3040, 7000, 11000, 15000, 20000):
        hay[at:at + len(base)] = np.frombuffer(base, dtype=np.uint8)
    offs = np.array([0, 1100, 1500, 2600, 2600, 4200, 8074, 12100, 15000, 16100, 20000, 21024, hay.size])
    ab._lib.acg_debug_set_pipeline_chunk.argtypes = [ctypes.c_void_p, ctypes.c_uint64]
    for kind in (0, 1, 2):
        for engine in (ab.Engine.Auto, ab.Engine.Sequential):
            ac = build(pats, kind, engine=engine)
            o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
            for chunk in (4096, 64 << 20):
                assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, chunk) == 0
                for ov in flags_of(kind):
                    covered, _ = check(ac, o, hay, offs, ov, (kind, engine, chunk, ov), sample=20, min_covered=5000)
                    # [0, 1024), [50, 1074) and [0, 1050): their union, or the match each kind yields first
                    assert covered[0] == (1074 if ov else (1050 if kind == 2 else 1024)), (kind, ov)


def test_error_codes_are_those_of_the_batch_calls():
    pats = [b"abcd", b"bcd"]
    docs = [b"xabcdx", b"", b"bcd"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    cases = [(build(pats, 1), True, ab.Anchored.No),   # UnsupportedOverlapping
             (build(pats, start_kind=ab.StartKind.Both), True, ab.Anchored.Yes),  # InvalidInputAnchored
             (build(pats), False, ab.Anchored.Yes),
             (build(pats, start_kind=ab.StartKind.Anchored), False, ab.Anchored.No),
             (build(pats + [b""], engine=ab.Engine.Prefilter), False, ab.Anchored.No),  # an override it cannot use
             (build(pats + [b""], engine=ab.Engine.Prefilter), True, ab.Anchored.No)]
    for ac, ov, anchored in cases:
        host = ac.find_overlapping_iter_batch_np if ov else ac.find_iter_batch_np
        with pytest.raises((ab.MatchError, ab.DeviceError)) as want:
            host((hay, offs), anchored=anchored)
        for mask in (False, True):
            with pytest.raises(type(want.value)) as got:
                ac.match_coverage_batch_np((hay, offs), overlapping=ov, anchored=anchored, mask=mask)
            assert got.value.code == want.value.code, (ov, anchored)
            rc, covered, m = raw_host(ac, hay, offs, ov, anchored, with_mask=mask)
            assert rc == want.value.code and (covered == SENTINEL).all() and (m == MASK_SENTINEL).all()
        for on_dev in (False, True):
            with pytest.raises(type(want.value)) as got:
                devout(ac, hay, offs, on_dev, ov, anchored)
            assert got.value.code == want.value.code, (ov, anchored, on_dev)
    ac = build(pats)
    for bad in ([0, 5, 3, 9], [0, 4, 10], [2, 1], [10]):
        for ov in (False, True):
            with pytest.raises(ValueError):
                ac.match_coverage_batch_np((hay, np.array(bad)), overlapping=ov, mask=True)
            for on_dev in (False, True):
                with pytest.raises(ValueError):
                    devout(ac, hay, np.array(bad), on_dev, ov)
    lib = ab._lib
    buf = np.zeros(16, np.uint64)
    u = np.array([0, 3, hay.size], np.uint64)
    # n_docs >= 2^32 is refused before the offsets are read, as by the batch calls
    cnt = ctypes.c_uint64()
    assert lib.acg_find_iter_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1 << 32, 0, None, 0,
                                   ctypes.byref(cnt)) == -22
    assert lib.acg_match_coverage_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1 << 32, 0, 0,
                                        buf.ctypes.data, None) == -22
    for on_dev in (0, 1):
        assert lib.acg_match_coverage_batch_devout(ac._h, hay.ctypes.data, hay.size, u.ctypes.data, on_dev, 1 << 32,
                                                   0, 1, buf.ctypes.data, None) == -22
    # no covered array: refused with documents, nothing to write without
    for ov in (0, 1):
        assert lib.acg_match_coverage_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 2, 0, ov, None,
                                            None) == -22
        assert lib.acg_match_coverage_batch_devout(ac._h, hay.ctypes.data, hay.size, u.ctypes.data, 0, 2, 0, ov, None,
                                                   None) == -22
        assert lib.acg_match_coverage_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 0, 0, ov, None,
                                            None) == 0
        assert lib.acg_match_coverage_batch_devout(ac._h, hay.ctypes.data, hay.size, u.ctypes.data, 1, 0, 0, ov, None,
                                                   None) == 0
    assert lib.acg_match_coverage_batch(None, hay.ctypes.data, 0, hay.size, u.ctypes.data, 2, 0, 0, buf.ctypes.data,
                                        None) == -22
    assert lib.acg_match_coverage_batch(ac._h, hay.ctypes.data, 0, hay.size, None, 2, 0, 0, buf.ctypes.data,
                                        None) == -22


def test_find_iter_coverage_through_the_radix_sort_fallback(monkeypatch):
    """2-slot order buckets of 256 bytes overflow, so the order step of the scan takes the radix-sort fallback
    before the chain and the coverage."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    monkeypatch.setenv("ACB_EMU_BUCKETLOG", "1")
    n, seed, nbytes, kind, ci = VARIANTS["stride2_narrow"]
    pats, hay = workload(n, seed, 32 << 10)
    W.plant(hay, pats, 8, period=61, window=40)
    offs = doc_offsets(hay.size, 21, max_len=700)
    plant_at_boundaries(hay, offs, pats, 22)
    for kind in (0, 1):
        ac = build(pats, kind)
        check(ac, O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, False, ("fallback", kind),
              min_covered=1000)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
