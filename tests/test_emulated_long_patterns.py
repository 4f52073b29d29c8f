"""Long patterns on the dry-run build of the kernels (tests/emu/): the families, length and tie-break limits and
placements of tests/test_gpu_long_patterns.py at reduced sizes, and the sharded search, which needs several
devices there, with threads as ranks.

For the order-path cases buckets shrink to 4 or 32 KiB of key offsets and 256 slots (ACB_EMU_BUCKETSHIFT /
ACB_EMU_BUCKETLOG), so that kilobyte inputs reach the order step's buckets, their fallback and the single list;
the pipelined host path runs with 4 KiB and 64 KiB chunks, shorter than the longest patterns."""
import ctypes
import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import packed, sharded as S  # noqa: E402
import test_gpu_long_patterns as LP  # noqa: E402
from test_sharded_emulated import eq, run_ranks  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    import build_emu
    lib = ctypes.CDLL(str(build_emu.build(asan=os.environ.get("ACB_EMU_ASAN") == "1")))
    ab._declare(lib)
    packed._declare(lib)
    saved = ab._lib, packed._lib, LP.RUN.on_gpu
    ab._lib = packed._lib = lib
    LP.RUN.on_gpu = False   # dry-run sizes and host buffers as "device" memory, whether or not the host has a GPU
    try:
        yield lib
    finally:
        ab._lib, packed._lib, LP.RUN.on_gpu = saved


def small_buckets(monkeypatch, shift):
    monkeypatch.setenv("ACB_EMU_BUCKETSHIFT", str(shift))
    monkeypatch.setenv("ACB_EMU_BUCKETLOG", "8")


@pytest.mark.parametrize("case", LP.FAMILY_CASES, ids=[LP.family_case_id(c) for c in LP.FAMILY_CASES])
def test_long_pattern_families(case):
    LP.run_family_case(*case)


def test_long_patterns_case_insensitive():
    LP.run_family_case("mixed", 4096, LP.plan(dense=1, dup_shift=1), ci=True)


@pytest.mark.parametrize("row", LP.BOUNDARIES, ids=[r[0] for r in LP.BOUNDARIES])
def test_length_and_tie_boundaries(monkeypatch, row):
    small_buckets(monkeypatch, 15)
    LP.run_boundary(row)


@pytest.mark.parametrize("L", [1023, 65533])
def test_walk_shards_cold_start(L):
    LP.run_walk_shards(L)


@pytest.mark.parametrize("L", [4097, 65533])
def test_pipelined_chunks_shorter_than_the_tail(L):
    LP.run_pipelined(L, [4096, 65536] if L > 65536 - 64 else [4096])


@pytest.mark.parametrize("L", [4096, 65533])
def test_find_windows(L):
    LP.run_find_windows(L)


def test_order_buckets_with_long_patterns(monkeypatch):
    small_buckets(monkeypatch, 12)
    LP.run_order_buckets()


def test_sharded_read_back_across_slices():
    """Six ranks over 72 KiB: slices of 12 KiB, shorter than the longest pattern (30 000 bytes), so that a rank's
    read-back of max_len - 1 bytes crosses two or three slices.  Matches that straddle one, two and three slice
    boundaries each appear once in the gathered list, which equals the oracle's and the single search's."""
    world, L = 6, 30000
    fam = LP.FAMILIES["prefix"](L, 0x5A4D)
    hay = LP.base_haystack(fam, 72 << 10, 11)
    plan = S.slice_plan(0, hay.size, world, L)
    bounds = [lo for lo, _, _ in plan[1:]]
    assert all(hi - lo < L for lo, hi, _ in plan)
    assert all(lo - rd >= L - 1 for lo, _, rd in plan[1:] if lo >= L)   # read-back of max_len - 1 bytes
    p = np.frombuffer(fam.pats[-1], np.uint8)
    for at in (bounds[0] - 3000, hay.size - L):
        hay[at: at + L] = p
    want = O.Oracle(fam.pats, kind=O.KIND_DFA).find_overlapping_iter_np(hay)
    st, en = want["start"].astype(np.int64), want["end"].astype(np.int64)
    crossed = sum(((st < b) & (en > b)).astype(np.int64) for b in bounds)
    for k in (1, 2, 3):
        assert (crossed == k).sum() > 0, (k, np.bincount(crossed))
    single = LP.builder(0).build(fam.pats).find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0]
    LP.assert_np_equal(single, want, "single search")
    res = run_ranks(world, fam.pats, hay, (0, hay.size))
    n, out, _, _ = res[0]
    assert n == len(want)
    eq(out, want)
    assert sum(r[2]["local_matches"] for r in res) == n
