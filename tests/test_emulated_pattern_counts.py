"""Pattern counts per document (acg_pattern_counts_batch / _devout) on the dry-run build of the kernels
(tests/emu/).

Every result is compared with two independent computations: the same handle's find_iter_batch_np /
find_overlapping_iter_batch_np records grouped on the host with np.unique(doc << 32 | pid), and the oracle
run on sampled documents alone.  Host output, device output with host offsets and device output with
"device" offsets (the dry run's device memory is host memory) must give the same bytes."""
import ctypes
import os
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
SENTINEL32 = 0xA5A5A5A5


def grouped(rec, n_docs):
    """(row_offsets, pids, counts) of batch records, grouped on the host."""
    key = rec["doc"].astype(np.uint64) << np.uint64(32) | rec["pid"].astype(np.uint64)
    u, c = np.unique(key, return_counts=True)
    rows = np.searchsorted(u >> np.uint64(32), np.arange(n_docs + 1, dtype=np.uint64), side="left")
    return rows.astype(np.uint64), (u & np.uint64(0xFFFFFFFF)).astype(np.uint32), c.astype(np.uint64)


def devout(ac, hay, offs, on_dev, overlapping, anchored=ab.Anchored.No, cap=None):
    """The counts into sentinel-filled "device" arrays; cap None: the size query first."""
    keep, arg, n_docs = offsets_arg(offs, on_dev)
    rows = np.full(n_docs + 1, SENTINEL, np.uint64)
    if cap is None:
        try:
            cap = ac.pattern_counts_batch_devout(hay.ctypes.data, hay.size, arg, rows.ctypes.data, None, None, 0,
                                                 overlapping=overlapping, anchored=anchored, n_docs=n_docs)
        except OverflowError as e:
            cap = e.args[0]
    pids = np.full(max(cap, 1), SENTINEL32, np.uint32)
    counts = np.full(max(cap, 1), SENTINEL, np.uint64)
    nnz = ac.pattern_counts_batch_devout(hay.ctypes.data, hay.size, arg, rows.ctypes.data, pids.ctypes.data,
                                         counts.ctypes.data, cap, overlapping=overlapping, anchored=anchored,
                                         n_docs=n_docs)
    assert nnz == cap
    return rows, pids[:nnz], counts[:nnz]


def same(got, want, ctx):
    for g, w, name in zip(got, want, ("row_offsets", "pids", "counts")):
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g, w), (ctx, name, g[:20], w[:20])


def check(ac, o, hay, offs, overlapping, ctx, anchored=ab.Anchored.No, sample=12, min_nnz=0):
    """Host output against the grouped records and the oracle; device output (both offset placements) byte for
    byte against host output.  Returns the host result."""
    n_docs = offs.size - 1
    records = (ac.find_overlapping_iter_batch_np if overlapping else ac.find_iter_batch_np)((hay, offs),
                                                                                           anchored=anchored)
    got = ac.pattern_counts_batch_np((hay, offs), overlapping=overlapping, anchored=anchored)
    same(got, grouped(records, n_docs), (ctx, "records"))
    rows, pids, counts = got
    assert rows[-1] == len(pids) >= min_nnz, ctx
    assert (counts >= 1).all(), ctx
    within_row = ~np.isin(np.arange(1, len(pids)), rows)
    assert (np.diff(pids.astype(np.int64))[within_row] > 0).all(), (ctx, "pids ascending in each row")
    rng = np.random.default_rng(n_docs)
    docs = set(rng.integers(0, n_docs, size=min(sample, n_docs)).tolist()) if n_docs else set()
    docs |= {0, n_docs - 1} if n_docs else set()
    fn = o.find_overlapping_iter_np if overlapping else o.find_iter_np
    for d in sorted(docs):
        r = fn(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]), anchored=bool(anchored))
        u, c = np.unique(r["pid"].astype(np.uint32), return_counts=True)
        lo, hi = int(rows[d]), int(rows[d + 1])
        assert np.array_equal(pids[lo:hi], u) and np.array_equal(counts[lo:hi], c.astype(np.uint64)), (ctx, "doc", d)
    for on_dev in (False, True):
        dv = devout(ac, hay, offs, on_dev, overlapping, anchored)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(dv, got)), (ctx, "devout", on_dev)
    return got


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
        want = check(ac, o, hay, offs, ov, (name, ov), min_nnz=30)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        ac.set_engine(ab.Engine.Sequential)
        same(check(ac, o, hay, offs, ov, (name, ov, "sequential")), want, (name, ov, "engines"))
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
        check(ac, o, hay, offs, ov, (name, ov), min_nnz=20)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


def test_anchored_empty_and_duplicate_patterns():
    """The sequential engine chosen by anchored input and by the empty pattern; duplicate patterns count under
    each of their ids as the records report them; all three match kinds."""
    rng = np.random.default_rng(11)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=4000)), dtype=np.uint8).copy()
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab", b"ab"]
    for kind in (0, 1, 2):
        for sk in (ab.StartKind.Anchored, ab.StartKind.Both):
            ac = build(pats, kind, start_kind=sk)
            o = O.Oracle(pats, match_kind=kind, start_kind=int(sk), kind=O.KIND_DFA)
            check(ac, o, hay, offs, False, (kind, sk), anchored=ab.Anchored.Yes, min_nnz=20)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac = build(pats + [b""], kind)
        o = O.Oracle(pats + [b""], match_kind=kind, kind=O.KIND_DFA)
        for ov in flags_of(kind):
            check(ac, o, hay, offs, ov, (kind, "empty pattern", ov), min_nnz=20)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac = build(pats, kind)
        for ov in flags_of(kind):
            check(ac, O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), hay, offs, ov, (kind, "duplicates", ov))


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_batch_shapes(engine):
    """No document, one, all empty, empty rows at the start / middle / end, one document holding every match."""
    pats, hay = workload(5000, 0xAC5000, 24 << 10)
    ac = build(pats, 0, engine=engine)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for ov in (False, True):
        for offs in ([0], [17], [hay.size]):
            rows, pids, counts = check(ac, o, hay, np.array(offs), ov, (engine, ov, offs))
            assert rows.tolist() == [0] and len(pids) == len(counts) == 0
        check(ac, o, np.zeros(0, np.uint8), np.array([0]), ov, (engine, ov, "empty buffer"))
        check(ac, o, hay, np.array([300, hay.size - 333]), ov, (engine, ov, "one document"), min_nnz=10)
        rows, _, _ = check(ac, o, hay, np.array([5, 5, 5, 5]), ov, (engine, ov, "all empty"))
        assert rows.tolist() == [0, 0, 0, 0]
        m = hay.size // 2
        offs = np.array([0, 0, 0, 100, m, m, m + 50, hay.size, hay.size, hay.size])
        rows, _, _ = check(ac, o, hay, offs, ov, (engine, ov, "empty rows"), min_nnz=10)
        assert rows[0] == rows[1] == rows[2] and rows[4] == rows[5] and rows[-1] == rows[-2] == rows[-3]
        offs = np.r_[np.zeros(40, np.int64), np.arange(0, 64, 2), hay.size, [hay.size] * 7]
        rows, _, _ = check(ac, o, hay, offs, ov, (engine, ov, "every match in one document"), min_nnz=10)
        assert rows[71] == 0 and rows[72] == rows[-1]


@pytest.mark.parametrize("n_pats", [1, 2, 4096, 4097])
def test_key_width_edges(n_pats):
    """pid_bits 0, 1, 12 and 13, and n_docs one below, at and one above a power of two (the sort's end bit)."""
    pats = [b"ab"] if n_pats == 1 else ([b"ab", b"b"] if n_pats == 2 else W.make_patterns(n_pats, n_pats))
    ac = build(pats, 0)
    pats_arr = [np.frombuffer(p, dtype=np.uint8) for p in (pats[:1] + pats[-1:])]
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for n_docs in (255, 256, 257):
        rng = np.random.default_rng(n_docs + n_pats)
        hay = np.empty(n_docs * 48, np.uint8)
        W.fill_haystack(hay, n_docs)
        for i in range(0, hay.size - 20, 37):
            p = pats_arr[(i // 37) % 2]
            hay[i:i + p.size] = p
        offs = np.r_[0, np.sort(rng.integers(0, hay.size, size=n_docs - 1)), hay.size]
        for ov in (False, True):
            rows, pids, _ = check(ac, o, hay, offs, ov, (n_pats, n_docs, ov), sample=4, min_nnz=n_docs // 4)
            assert pids.max() == n_pats - 1


def test_overflow_protocol():
    """cap = nnz - 1 returns E_OVERFLOW with nnz and writes none of the arrays; cap = nnz succeeds; cap 0 with
    no arrays is a size query.  Host and device output, both engines."""
    docs = [b"a" * 300, b"", b"ba" * 100, b"a", b"abc"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    lib, cnt = ab._lib, ctypes.c_uint64()
    for engine in (ab.Engine.Auto, ab.Engine.Sequential):
        ac = build([b"a", b"aa", b"b", b"c", b"x"], engine=engine)
        for ov in (False, True):
            want = ac.pattern_counts_batch_np((hay, offs), overlapping=ov)
            nnz = len(want[1])
            assert nnz >= 7
            for on_dev in (False, True):
                keep, arg, n_docs = offsets_arg(offs, on_dev)
                rows = np.full(n_docs + 1, SENTINEL, np.uint64)
                pids = np.full(nnz, SENTINEL32, np.uint32)
                counts = np.full(nnz, SENTINEL, np.uint64)
                with pytest.raises(OverflowError) as e:
                    ac.pattern_counts_batch_devout(hay.ctypes.data, hay.size, arg, rows.ctypes.data, pids.ctypes.data,
                                                   counts.ctypes.data, nnz - 1, overlapping=ov, n_docs=n_docs)
                assert e.value.args[0] == nnz
                assert (rows == SENTINEL).all() and (pids == SENTINEL32).all() and (counts == SENTINEL).all()
                got = devout(ac, hay, offs, on_dev, ov, cap=nnz)
                assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want)), (engine, ov, on_dev)
            # host output: the same protocol
            for cap, rc_want in ((nnz - 1, ab.E_OVERFLOW), (0, ab.E_OVERFLOW), (nnz, 0)):
                rows = np.full(offs.size, SENTINEL, np.uint64)
                pids = np.full(max(cap, 1), SENTINEL32, np.uint32)
                counts = np.full(max(cap, 1), SENTINEL, np.uint64)
                args = (pids.ctypes.data, counts.ctypes.data) if cap else (None, None)
                rc = lib.acg_pattern_counts_batch(ac._h, hay.ctypes.data, 0, hay.size, offs.astype(np.uint64).ctypes.data,
                                                  offs.size - 1, 0, int(ov), rows.ctypes.data, *args, cap,
                                                  ctypes.byref(cnt))
                assert rc == rc_want and cnt.value == nnz, (engine, ov, cap, rc)
                if rc:
                    assert (rows == SENTINEL).all() and (pids == SENTINEL32).all() and (counts == SENTINEL).all()
                else:
                    assert rows.tobytes() == want[0].tobytes() and pids.tobytes() == want[1].tobytes()
        # the Python retry loop from a one-entry first guess
        ac._cap_hint = 1
        same(ac.pattern_counts_batch_np(docs, overlapping=True),
             grouped(ac.find_overlapping_iter_batch_np(docs), len(docs)), (engine, "retry"))


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
        with pytest.raises(type(want.value)) as got:
            ac.pattern_counts_batch_np((hay, offs), overlapping=ov, anchored=anchored)
        assert got.value.code == want.value.code, (ov, anchored)
        for on_dev in (False, True):
            with pytest.raises(type(want.value)) as got:
                devout(ac, hay, offs, on_dev, ov, anchored, cap=16)
            assert got.value.code == want.value.code, (ov, anchored, on_dev)
    ac = build(pats)
    for bad in ([0, 5, 3, 9], [0, 4, 10], [2, 1], [10]):
        for ov in (False, True):
            with pytest.raises(ValueError):
                ac.pattern_counts_batch_np((hay, np.array(bad)), overlapping=ov)
            for on_dev in (False, True):
                with pytest.raises(ValueError):
                    devout(ac, hay, np.array(bad), on_dev, ov, cap=16)
    lib, cnt = ab._lib, ctypes.c_uint64()
    rows = np.zeros(8, np.uint64)
    buf = np.zeros(16, np.uint64)
    u = np.zeros(2, np.uint64)
    # n_docs >= 2^32 is refused before the offsets are read, as by the batch calls
    assert lib.acg_pattern_counts_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1 << 32, 0, 0,
                                        rows.ctypes.data, buf.ctypes.data, buf.ctypes.data, 4, ctypes.byref(cnt)) == -22
    assert lib.acg_find_iter_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1 << 32, 0, None, 0,
                                   ctypes.byref(cnt)) == -22
    for on_dev in (0, 1):
        assert lib.acg_pattern_counts_batch_devout(ac._h, hay.ctypes.data, hay.size, u.ctypes.data, on_dev, 1 << 32, 0,
                                                   1, rows.ctypes.data, buf.ctypes.data, buf.ctypes.data, 4,
                                                   ctypes.byref(cnt)) == -22
    # no row index, or entries without room
    assert lib.acg_pattern_counts_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1, 0, 0, None,
                                        buf.ctypes.data, buf.ctypes.data, 4, ctypes.byref(cnt)) == -22
    assert lib.acg_pattern_counts_batch(ac._h, hay.ctypes.data, 0, hay.size, u.ctypes.data, 1, 0, 0,
                                        rows.ctypes.data, None, buf.ctypes.data, 4, ctypes.byref(cnt)) == -22


def test_find_iter_counts_through_the_radix_sort_fallback(monkeypatch):
    """2-slot order buckets of 256 bytes overflow, so the order step of the find_iter scan takes the radix-sort
    fallback before the chain and the counts."""
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
              min_nnz=100)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
