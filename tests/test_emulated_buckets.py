"""Bucketed emission and the shared-memory order step (order_buckets_kernel), on the dry-run build of
the kernels (tests/emu/), against the oracle.

On the device a bucket covers 32 MiB of key offsets and holds 16 K tuples; ACB_EMU_BUCKETSHIFT and
ACB_EMU_BUCKETLOG shrink both in the dry run (read at every search), so that kilobyte inputs cross
many buckets and can fill one.  Which order path ran shows in the launch count of the search: the
scan, then one order launch (buckets), or the compaction and the radix sort (overflow)."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import packed, workload as W  # noqa: E402

ORDER_BUCKETS = 2   # launches of a device-resident search: scan + order_buckets_kernel
EXPAND = 1          # + expand_kernel, which writes the records of a host-output search
ORDER_FALLBACK = 10  # scan + compaction + radix sort (counted as 8)


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    import build_emu
    lib = ctypes.CDLL(str(build_emu.build(asan=os.environ.get("ACB_EMU_ASAN") == "1")))
    ab._declare(lib)
    packed._declare(lib)
    lib.acg_debug_set_experiment.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
    saved = ab._lib, packed._lib
    ab._lib = packed._lib = lib
    try:
        yield lib
    finally:
        ab._lib, packed._lib = saved


def eq(got, want, ctx=None):
    assert len(got) == len(want), (len(got), len(want), ctx)
    for k in ("pid", "start", "end"):
        assert np.array_equal(got[k], want[k]), (k, ctx)


def launches(ac):
    return int(ac.last_stats()["launches"])


@pytest.mark.parametrize("kind,ci", [(0, False), (1, True), (2, False)])
def test_matches_across_small_buckets(monkeypatch, kind, ci):
    """256-byte buckets: planted matches every 61 bytes, many of them starting in one bucket and ending
    in the next; overlapping search and every find_iter mode, whole span and a sub-span."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    pats = W.make_patterns(5000, 0xAC5000)
    hay = np.empty(96 << 10, dtype=np.uint8)
    W.fill_haystack(hay, 5)
    W.plant(hay, pats, 8, period=61, window=40)   # (a period that does not divide the bucket)
    if ci:
        W.flip_case(hay, 7)
    ac = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    ptr = hay.ctypes.data
    if kind == 0:
        want = o.find_overlapping_iter_np(hay)
        crossing = (want["start"] >> 8) != ((want["end"] - 1) >> 8)
        assert crossing.sum() > 20
        eq(ac.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, "overlapping")
        assert launches(ac) == ORDER_BUCKETS + EXPAND
        eq(ac.try_find_overlapping_iter_np(hay), want, "overlapping, host input")
    want = o.find_iter_np(hay)
    assert len(want) > 100
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], want, "find_iter")
    assert launches(ac) == ORDER_BUCKETS + 8 + EXPAND   # + the chain resolution
    eq(ac.try_find_iter_np(hay), want, "find_iter, host input")
    s, e = 3000, hay.size - 1500
    eq(ac.find_iter_dev_np(ptr, hay.size, span=(s, e))[0], o.find_iter_np(hay, span=(s, e)), "sub-span")


def test_one_tuple_and_no_tuple(monkeypatch):
    """A single match in a late bucket still ends up at the front of the ordered list."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "8")
    hay = np.frombuffer(b"x" * 5000 + b"needle" + b"y" * 300, dtype=np.uint8).copy()
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build([b"needle", b"thread"])
    o = O.Oracle([b"needle", b"thread"], kind=O.KIND_DFA)
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "one")
    empty = np.frombuffer(b"z" * 4096, dtype=np.uint8).copy()
    assert len(ac.find_overlapping_iter_dev_np(empty.ctypes.data, empty.size)[0]) == 0


@pytest.mark.parametrize("n_a,experiment", [(3000, 0), (3000, 64), (90000, 64)])
def test_full_bucket_takes_the_fallback(monkeypatch, n_a, experiment):
    """`aa` over a run of `a`s: 64-slot buckets of 1 KiB fill up, the rest of their tuples go to the
    overflow list, and the order step compacts everything and radix-sorts it.  With 90 000 `a`s the
    overflow list outgrows its room as well, and the scan is repeated with more.  Experiment 64: the
    fingerprint filter instead of the byte-set scan."""
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", "10")
    monkeypatch.setenv("ACB_EMU_BUCKETLOG", "6")
    pats = [b"aa", b"ab", b"ba", b"aaa"]
    hay = np.frombuffer(b"b" * 700 + b"a" * n_a + b"b" * 900 + b"ab" * 200, dtype=np.uint8).copy()
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    assert ab._lib.acg_debug_set_experiment(ac._h, experiment) == 0
    o = O.Oracle(pats, kind=O.KIND_DFA)
    want = o.find_overlapping_iter_np(hay)
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], want, "overlapping")
    assert launches(ac) >= ORDER_FALLBACK
    eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), "find_iter")
    # the same search with room in every bucket takes the bucket sort again
    monkeypatch.setenv("ACB_EMU_BUCKETLOG", "14")
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], want, "roomy buckets")
    assert launches(ac) == ORDER_BUCKETS + EXPAND


def test_buckets_across_queue_windows():
    """Spans larger than one queue window (2 GiB on the device, 4 KiB here) with 2 KiB buckets: every
    prefilter kernel variant and tile distribution of tests/emu_window_check.py."""
    env = dict(os.environ, ACB_EMU_WINSHIFT="12", ACB_EMU_BUCKETSHIFT="11")
    r = subprocess.run([sys.executable, str(ROOT / "tests" / "emu_window_check.py")], capture_output=True, text=True,
                       env=env, timeout=1800)
    assert r.returncode == 0 and "WINDOWS OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
