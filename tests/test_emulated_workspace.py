"""The search workspace on the dry-run build of the library (tests/emu/): what one handle's buffers go
through in its life -- grown one after the other, and an allocation that fails half way through a grow of
several -- with every result compared with the oracle.  The dry-run runtime counts allocation calls and can
make the n-th one fail (tests/emu/README.md)."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from test_emulated_batch import expected, records  # noqa: E402
from test_emulated_kernels import build, emulated_library, eq, workload  # noqa: E402,F401

DEVICE, PINNED = 0, 1


def allocations():
    return ab._lib.acb_emu_alloc_calls(DEVICE), ab._lib.acb_emu_alloc_calls(PINNED)


def test_failed_staging_ring_allocation_leaves_a_usable_workspace():
    """A pageable host haystack goes through a ring of two page-locked buffers.  When the second of them cannot
    be allocated while the ring grows, that search fails -- and the next one that fits the old ring must find a
    ring again, not the capacity of the one that was freed."""
    pats, hay = workload(5000, 0xAC5000, 256 << 10)
    small = hay[: 24 << 10]
    o = O.Oracle(pats, kind=O.KIND_DFA)
    ac = build(pats)
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 4096) == 0
    eq(ac.try_find_overlapping_iter_np(small), o.find_overlapping_iter_np(small), "ring of 4 KiB")
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 64 << 10) == 0
    ab._lib.acb_emu_fail_alloc(PINNED, 2)  # the grow's first allocation succeeds, its second does not
    with pytest.raises(ab.DeviceError):
        ac.try_find_overlapping_iter_np(hay)
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 4096) == 0
    eq(ac.try_find_overlapping_iter_np(small), o.find_overlapping_iter_np(small), "after the failed grow")
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 64 << 10) == 0
    eq(ac.try_find_overlapping_iter_np(hay), o.find_overlapping_iter_np(hay), "ring of 64 KiB")


def test_failed_tuple_list_allocation_is_forgotten_by_the_next_search():
    """More matches than the tuple lists hold: the scan is repeated with four larger lists.  When the second of
    them cannot be allocated that search fails, and the workspace must not remember the capacity of the first:
    the next, short search starts again from four lists of the default capacity, and the long one then succeeds."""
    pats = [b"a", b"b", b"ab", b"ba", b"aba"]
    hay = np.frombuffer(b"ab" * (300 << 10), dtype=np.uint8)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    want, want_short = o.find_overlapping_iter_np(hay), o.find_overlapping_iter_np(hay[:1000])
    assert len(want) > (1 << 20)  # the tuple lists' first capacity
    ac = build(pats)
    ptr = hay.ctypes.data  # "device" memory is host memory in the dry run: no haystack staging to allocate
    eq(ac.find_overlapping_iter_dev_np(ptr, 1000)[0], want_short, "short")
    ab._lib.acb_emu_fail_alloc(DEVICE, 2)
    with pytest.raises(ab.DeviceError):
        ac.find_overlapping_iter_dev_np(ptr, hay.size)
    before = allocations()
    eq(ac.find_overlapping_iter_dev_np(ptr, 1000)[0], want_short, "short, after the failed grow")
    assert allocations() == (before[0] + 4, before[1])
    eq(ac.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, "grown after all")


def test_buffers_grow_one_after_the_other_in_one_handles_life():
    """One handle, one thread, hence one workspace: a short search, then more matches than the tuple lists
    hold (rescan; sort storage, tuple staging and haystack staging grow with it), then batches of more
    documents than the per-document arrays and the per-document records start with, then a find_iter whose
    candidates outnumber the chain scratch.  The same calls again find every buffer large enough: nothing is
    allocated."""
    pats = [b"a", b"b", b"ab", b"ba", b"aba"]
    hay = np.frombuffer(b"ab" * (300 << 10), dtype=np.uint8)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    ac = build(pats)
    want = o.find_overlapping_iter_np(hay)
    assert len(want) > (1 << 20)  # the tuple lists' first capacity
    n_docs = (1 << 12) + 904
    offs = np.arange(n_docs + 1, dtype=np.int64) * 13
    docs = np.ascontiguousarray(hay[: offs[-1]])
    want_docs = expected(o, docs, offs, "overlapping")
    part = hay[: 64 << 10]
    assert len(o.find_overlapping_iter_np(part)) > (1 << 16)  # the candidates; the chain scratch's first capacity
    for again in (False, True):
        before = allocations()
        eq(ac.try_find_overlapping_iter_np(hay[:1000]), o.find_overlapping_iter_np(hay[:1000]), "short")
        eq(ac.try_find_overlapping_iter_np(hay), want, "tuple lists regrown")
        assert np.array_equal(records(ac.find_overlapping_iter_batch_np((docs, offs))), want_docs)
        assert ac.is_match_batch((docs, offs)).all()
        found, first = ac.find_batch_np((docs, offs))
        assert found.all() and np.array_equal(first["end"], np.ones(n_docs))  # "a" or "b" at the start of every document
        eq(ac.try_find_iter_np(part), o.find_iter_np(part), "chain scratch regrown")
        assert (allocations() == before) == again
