"""Batched search with device-resident results (acg_*_batch_devout) on the dry-run build of the kernels
(tests/emu/), whose device memory is host memory: numpy buffers stand in for the device arrays.

The devout contract: the records are byte for byte what the host-output batch call returns on the same batch,
d_match_offsets is their CSR index by document, and flags / first matches equal is_match_batch / find_batch --
with the document offsets in host memory and "on the device" (used by the kernels where they are)."""
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
from aho_corasick_b200 import packed, workload as W  # noqa: E402
from test_emulated_batch import build, doc_offsets, plant_at_boundaries  # noqa: E402
from test_emulated_kernels import VARIANTS, BYTESCAN_SETS, workload  # noqa: E402

SENTINEL = np.uint64(0xDEADBEEFDEADBEEF)


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


def offsets_arg(offs, on_device):
    """(keepalive, offsets argument, n_docs): the host array, or the address of a uint64 copy ("device")."""
    u = np.ascontiguousarray(offs, dtype=np.int64).astype(np.uint64)
    return u, (u.ctypes.data if on_device else offs), u.size - 1


def devout(ac, what, hay, offs, on_device, anchored=ab.Anchored.No, cap=None):
    """(records, match_offsets) of find_iter / overlapping into sentinel-filled "device" buffers."""
    fn = ac.find_overlapping_iter_batch_devout if what == "overlapping" else ac.find_iter_batch_devout
    keep, arg, n_docs = offsets_arg(offs, on_device)
    if cap is None:  # the two-call protocol
        try:
            cap = fn(hay.ctypes.data, hay.size, arg, None, 0, np.zeros(n_docs + 1, np.uint64).ctypes.data,
                     anchored=anchored, n_docs=n_docs)
        except OverflowError as e:
            cap = e.args[0]
    out = np.full(max(cap, 1) * 3, SENTINEL, np.uint64)
    mo = np.full(n_docs + 1, SENTINEL, np.uint64)
    n = fn(hay.ctypes.data, hay.size, arg, out.ctypes.data, cap, mo.ctypes.data, anchored=anchored, n_docs=n_docs)
    assert n == cap
    return out.view(ab.DOC_MATCH_DTYPE)[:n], mo


def devout_flags(ac, hay, offs, on_device, anchored=ab.Anchored.No):
    keep, arg, n_docs = offsets_arg(offs, on_device)
    flags = np.full(max(n_docs, 1), 7, np.uint8)
    ac.is_match_batch_devout(hay.ctypes.data, hay.size, arg, flags.ctypes.data, anchored=anchored, n_docs=n_docs)
    return flags[:n_docs]


def devout_find(ac, hay, offs, on_device, anchored=ab.Anchored.No, earliest=False):
    keep, arg, n_docs = offsets_arg(offs, on_device)
    found = np.full(max(n_docs, 1), 7, np.uint8)
    out = np.full(max(n_docs, 1) * 3, SENTINEL, np.uint64)
    ac.find_batch_devout(hay.ctypes.data, hay.size, arg, out.ctypes.data, found.ctypes.data, anchored=anchored,
                         earliest=earliest, n_docs=n_docs)
    return found[:n_docs], out.view(ab.DOC_MATCH_DTYPE)[:n_docs]


def csr_of(rec, n_docs):
    return np.searchsorted(rec["doc"].astype(np.int64), np.arange(n_docs + 1), side="left").astype(np.uint64)


def check_devout(ac, hay, offs, kind, ctx, anchored=ab.Anchored.No, min_records=0):
    """Every devout call against the host-output batch call on the same batch, offsets on both sides."""
    batch = (hay, offs)
    n_docs = offs.size - 1
    whats = ["iter", "overlapping"] if kind == 0 and not anchored else ["iter"]
    want = {w: (ac.find_overlapping_iter_batch_np if w == "overlapping" else ac.find_iter_batch_np)(
        batch, anchored=anchored) for w in whats}
    assert len(want["iter"]) >= min_records, ctx
    want_flags = ac.is_match_batch(batch, anchored=anchored)
    want_find = {e: ac.find_batch_np(batch, anchored=anchored, earliest=e) for e in (False, True)}
    for on_dev in (False, True):
        c = (ctx, "offsets on the device" if on_dev else "host offsets")
        assert np.array_equal(devout_flags(ac, hay, offs, on_dev, anchored), want_flags.astype(np.uint8)), c
        for e, (wf, wr) in want_find.items():
            found, rec = devout_find(ac, hay, offs, on_dev, anchored, e)
            assert np.array_equal(found, wf.astype(np.uint8)) and rec.tobytes() == wr.tobytes(), (c, "find", e)
        for w in whats:  # last, so that last_stats() tells the engine of a records call
            got, mo = devout(ac, w, hay, offs, on_dev, anchored)
            assert got.tobytes() == want[w].tobytes(), (c, w)
            assert np.array_equal(mo, csr_of(want[w], n_docs)), (c, w)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants(name):
    """Every prefilter kernel variant (doc_records_kernel in the key layout of the call), then the per-document
    sequential kernel on the same batch."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, min(nbytes, 128 << 10), ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    offs = doc_offsets(hay.size, seed)
    plant_at_boundaries(hay, offs, pats, seed)
    if ci:
        W.flip_case(hay, 7)
    ac = build(pats, kind, ci)
    check_devout(ac, hay, offs, kind, name, min_records=50)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    ac.set_engine(ab.Engine.Sequential)
    check_devout(ac, hay, offs, kind, (name, "sequential"))
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


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
    check_devout(ac, hay, offs, kind, name, min_records=20)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)


def test_anchored_and_empty_pattern_automata():
    rng = np.random.default_rng(11)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=4000)), dtype=np.uint8).copy()
    offs = doc_offsets(hay.size, 12, max_len=64)
    pats = [b"ab", b"abc", b"b", b"ca", b"cab"]
    for kind in (0, 1, 2):
        for sk in (ab.StartKind.Anchored, ab.StartKind.Both):
            ac = build(pats, kind, start_kind=sk)
            check_devout(ac, hay, offs, kind, (kind, sk), anchored=ab.Anchored.Yes, min_records=20)
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        ac = build(pats + [b""], kind)
        check_devout(ac, hay, offs, kind, (kind, "empty pattern"), min_records=20)
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
def test_edge_batches(engine):
    """Zero documents, one document, all documents empty, no match anywhere."""
    pats, hay = workload(5000, 0xAC5000, 48 << 10)
    empty = np.zeros(0, np.uint8)
    for kind in (0, 1):
        ac = build(pats, kind, engine=engine)
        for offs in ([0], [17], [hay.size]):
            check_devout(ac, hay, np.array(offs), kind, (engine, kind, offs))
        check_devout(ac, empty, np.array([0]), kind, (engine, kind, "empty buffer"))
        check_devout(ac, hay, np.array([1000, hay.size - 333]), kind, (engine, kind, "one document"), min_records=10)
        check_devout(ac, hay, np.array([5, 5, 5, 5]), kind, (engine, kind, "all empty"))
        check_devout(ac, hay, np.array([0, 3, 3, 7, 9]), kind, (engine, kind, "no match"))
        # one match in the last of many documents: the last record's index fills the whole front of the CSR
        tail = np.frombuffer(b"x" * 3000 + pats[0], dtype=np.uint8).copy()
        offs = np.r_[np.arange(0, 3000, 3), tail.size]
        got, mo = devout(ac, "iter", tail, offs, True)
        assert len(got) >= 1 and (got["doc"] == offs.size - 2).all()
        assert (mo[:-1] == 0).all() and mo[-1] == len(got)


def test_overflow_protocol():
    """cap one short raises OverflowError(count) and writes neither array; a retry with that count succeeds."""
    docs = [b"a" * 300, b"", b"ba" * 100, b"a"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    for engine in (ab.Engine.Auto, ab.Engine.Sequential):
        ac = build([b"a", b"aa"], engine=engine)
        for what in ("iter", "overlapping"):
            for on_dev in (False, True):
                want, _ = devout(ac, what, hay, offs, on_dev)
                count = len(want)
                assert count > 300
                keep, arg, n_docs = offsets_arg(offs, on_dev)
                fn = ac.find_overlapping_iter_batch_devout if what == "overlapping" else ac.find_iter_batch_devout
                out = np.full((count - 1) * 3 + 3, SENTINEL, np.uint64)
                mo = np.full(n_docs + 1, SENTINEL, np.uint64)
                with pytest.raises(OverflowError) as e:
                    fn(hay.ctypes.data, hay.size, arg, out.ctypes.data, count - 1, mo.ctypes.data, n_docs=n_docs)
                assert e.value.args[0] == count
                assert (out == SENTINEL).all() and (mo == SENTINEL).all()
                with pytest.raises(OverflowError) as e:  # the count alone: no output buffer at all
                    fn(hay.ctypes.data, hay.size, arg, None, 0, mo.ctypes.data, n_docs=n_docs)
                assert e.value.args[0] == count and (mo == SENTINEL).all()
                got, mo = devout(ac, what, hay, offs, on_dev, cap=count)
                assert got.tobytes() == want.tobytes() and mo[-1] == count


def test_invalid_input():
    ac = build([b"abcd"])
    hay = np.frombuffer(b"abcdabcd", dtype=np.uint8).copy()
    out = np.zeros(64, np.uint64)
    mo = np.full(8, SENTINEL, np.uint64)
    flags = np.zeros(8, np.uint8)
    for offs in ([0, 5, 3, 8], [0, 4, 9], [2, 1], [0, 8, 8, 9], [9]):
        for on_dev in (False, True):
            keep, arg, n_docs = offsets_arg(offs, on_dev)
            for fn in (ac.find_iter_batch_devout, ac.find_overlapping_iter_batch_devout):
                with pytest.raises(ValueError):
                    fn(hay.ctypes.data, hay.size, arg, out.ctypes.data, 16, mo.ctypes.data, n_docs=n_docs)
            with pytest.raises(ValueError):
                ac.is_match_batch_devout(hay.ctypes.data, hay.size, arg, flags.ctypes.data, n_docs=n_docs)
            with pytest.raises(ValueError):
                ac.find_batch_devout(hay.ctypes.data, hay.size, arg, out.ctypes.data, flags.ctypes.data,
                                     n_docs=n_docs)
    assert (mo == SENTINEL).all()
    lib, cnt = ab._lib, ctypes.c_uint64()
    offs = np.zeros(2, np.uint64)
    # n_docs >= 2^32 is refused before the offsets are read; so are device offsets that are not 8-byte aligned
    for on_dev in (0, 1):
        assert lib.acg_find_iter_batch_devout(ac._h, hay.ctypes.data, hay.size, offs.ctypes.data, on_dev, 1 << 32, 0,
                                              out.ctypes.data, 16, mo.ctypes.data, ctypes.byref(cnt)) == -22
        assert lib.acg_is_match_batch_devout(ac._h, hay.ctypes.data, hay.size, offs.ctypes.data, on_dev, 1 << 32, 0,
                                             flags.ctypes.data) == -22
    assert lib.acg_find_iter_batch_devout(ac._h, hay.ctypes.data, hay.size, offs.ctypes.data + 4, 1, 1, 0,
                                          out.ctypes.data, 16, mo.ctypes.data, ctypes.byref(cnt)) == -22
    # no index array, or records without room
    assert lib.acg_find_iter_batch_devout(ac._h, hay.ctypes.data, hay.size, offs.ctypes.data, 0, 1, 0,
                                          out.ctypes.data, 16, None, ctypes.byref(cnt)) == -22
    assert lib.acg_find_iter_batch_devout(ac._h, hay.ctypes.data, hay.size, offs.ctypes.data, 0, 1, 0,
                                          None, 16, mo.ctypes.data, ctypes.byref(cnt)) == -22


def test_error_codes_are_those_of_the_host_output_calls():
    pats = [b"abcd", b"bcd"]
    docs = [b"xabcdx", b"", b"bcd"]
    hay = np.frombuffer(b"".join(docs), dtype=np.uint8).copy()
    offs = np.r_[0, np.cumsum([len(d) for d in docs])]
    out = np.zeros(64, np.uint64)
    mo = np.zeros(8, np.uint64)
    flags = np.zeros(8, np.uint8)
    cases = [(build(pats, 1), "overlapping", ab.Anchored.No),
             (build(pats), "iter", ab.Anchored.Yes),
             (build(pats, start_kind=ab.StartKind.Anchored), "is_match", ab.Anchored.No),
             (build(pats + [b""], engine=ab.Engine.Prefilter), "iter", ab.Anchored.No),
             (build(pats + [b""], engine=ab.Engine.Prefilter), "find", ab.Anchored.No)]
    for ac, what, anchored in cases:
        host = {"iter": ac.find_iter_batch_np, "overlapping": ac.find_overlapping_iter_batch_np,
                "is_match": ac.is_match_batch, "find": ac.find_batch_np}[what]
        with pytest.raises((ab.MatchError, ab.DeviceError)) as want:
            host((hay, offs), anchored=anchored)
        for on_dev in (False, True):
            keep, arg, n_docs = offsets_arg(offs, on_dev)
            with pytest.raises(type(want.value)) as got:
                if what in ("iter", "overlapping"):
                    fn = ac.find_overlapping_iter_batch_devout if what == "overlapping" else ac.find_iter_batch_devout
                    fn(hay.ctypes.data, hay.size, arg, out.ctypes.data, 16, mo.ctypes.data, anchored=anchored,
                       n_docs=n_docs)
                elif what == "is_match":
                    ac.is_match_batch_devout(hay.ctypes.data, hay.size, arg, flags.ctypes.data, anchored=anchored,
                                             n_docs=n_docs)
                else:
                    ac.find_batch_devout(hay.ctypes.data, hay.size, arg, out.ctypes.data, flags.ctypes.data,
                                         anchored=anchored, n_docs=n_docs)
            assert got.value.code == want.value.code, (what, on_dev)


def test_documents_across_buckets(monkeypatch):
    """256-byte order buckets: documents and their records spread over many buckets."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    n, seed, nbytes, kind, ci = VARIANTS["stride2_narrow"]
    pats, hay = workload(n, seed, 32 << 10)
    W.plant(hay, pats, 8, period=61, window=40)
    offs = doc_offsets(hay.size, 21, max_len=700)
    plant_at_boundaries(hay, offs, pats, 22)
    for kind in (0, 1):
        check_devout(build(pats, kind), hay, offs, kind, ("buckets", kind), min_records=100)


@pytest.mark.skipif(os.environ.get("ACB_EMU_WINSHIFT") is not None, reason="runs inside the subprocess below")
def test_documents_across_queue_windows():
    """4 KiB queue windows (fixed when the library loads, hence a fresh process) with 2 KiB buckets."""
    env = dict(os.environ, ACB_EMU_WINSHIFT="12", ACB_EMU_BUCKETSHIFT="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", str(Path(__file__)), "-k",
                        "prefilter_variants and (stride2_narrow or dense)"], capture_output=True, text=True, env=env,
                       timeout=1800, cwd=str(ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
