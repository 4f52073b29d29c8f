"""Dry run (tests/emu/) of the stride-2 narrow prefilter kernel's tile bookkeeping with one CTA, so
that tile t starts at region_lo + t * 2 KiB: a warp step probes one 2 KiB tile staged by one bulk copy
(plus 16 bytes of look-ahead), draws its tiles four at a time and draws the next four with the last
tile of a batch (the tile of the next copy is then known for the L2 prefetch).  Checked against the
oracle for overlapping, leftmost-first and leftmost-longest search: hits at the first and last bytes
of a tile at both parities, steps with several times the usual number of first-stage hits, and spans
whose last tile is short."""
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
from aho_corasick_b200 import packed, workload as W  # noqa: E402
from test_prefilter_plan import plan_of  # noqa: E402

TILE = 2048   # bytes per warp step of the stride-2 narrow kernel
KINDS = (0, 1, 2)  # overlapping (Standard), leftmost-first, leftmost-longest


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


@pytest.fixture
def one_cta(monkeypatch):
    """One emulated SM: one CTA whose chunk is the whole region, so tile t starts at region_lo + t * TILE."""
    monkeypatch.setenv("ACB_EMU_SMS", "1")


PATS = W.make_patterns(5000, 0xAC5000)


def searchers():
    out = []
    for kind in KINDS:
        ac = ab.AhoCorasick.builder().match_kind(kind).kind(ab.AhoCorasickKind.DFA).build(PATS)
        p = plan_of(ac)
        assert p.supported and not p.brute and (p.stride, bool(p.wide), bool(p.dense)) == (2, False, False), kind
        out.append((kind, ac, O.Oracle(PATS, match_kind=kind, kind=O.KIND_DFA)))
    return out


def eq(got, want, ctx):
    assert len(got) == len(want), (len(got), len(want), ctx)
    for k in ("pid", "start", "end"):
        assert np.array_equal(got[k], want[k]), (k, ctx)


@pytest.fixture(scope="module")
def engines(emulated_library):
    return searchers()


def check_all(engines, view, ctx, min_matches=1):
    for kind, ac, o in engines:
        ptr = view.ctypes.data
        if kind == 0:
            want = o.find_overlapping_iter_np(view)
            eq(ac.find_overlapping_iter_dev_np(ptr, view.size)[0], want, (ctx, kind))
            assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        else:
            want = o.find_iter_np(view)
            eq(ac.find_iter_dev_np(ptr, view.size)[0], want, (ctx, kind))
        assert len(want) >= min_matches, (ctx, kind)


def aligned(backing, phase, n):
    """n bytes of `backing` starting `phase` bytes past a 64-byte boundary."""
    off = (-backing.ctypes.data) % 64 + phase
    return backing[off:off + n]


def region_lo(view):
    return (16 - view.ctypes.data % 16) % 16


def put(view, at, pat):
    if 0 <= at and at + len(pat) <= view.size:
        view[at:at + len(pat)] = np.frombuffer(pat, dtype=np.uint8)


def first_stage_hits_per_tile(view, ac):
    """The stride-2 first-stage probe restated (as tests/test_prefilter_plan.py does) over the tiles of
    a one-CTA launch: hits per TILE bytes from region_lo."""
    p = plan_of(ac)
    bitmap = np.ctypeslib.as_array(ctypes.cast(p.bitmap, ctypes.POINTER(ctypes.c_uint32)), shape=(int(p.bitmap_words),))
    lo = region_lo(view)
    n_tiles = (view.size - lo - 20) // TILE
    h = view[lo: lo + n_tiles * TILE + 4].astype(np.uint32)
    pos = np.arange(0, n_tiles * TILE, 2)
    win = h[pos] | (h[pos + 1] << 8) | (h[pos + 2] << 16) | (h[pos + 3] << 24)
    gm = (win | (p.fold & 0x00FFFFFF)) & 0xFFFFFFFF
    hh = (gm.astype(np.uint64) * ((p.mult3 << p.key_shift) & 0xFFFFFFFF)) & 0xFFFFFFFF
    bit = (hh >> p.shift) * 8 + (gm & 7)
    hit = (bitmap[(bit >> 5).astype(np.int64)] >> (bit & 31).astype(np.uint32)) & 1
    return hit.reshape(n_tiles, TILE // 2).sum(axis=1)


@pytest.mark.parametrize("phase", [0, 1, 2, 3])
def test_hits_at_the_first_and_last_bytes_of_a_tile(engines, one_cta, phase):
    """Patterns that start at tile offsets -3 .. 3 (offset -1 is the start one byte before the tile,
    owned by the tile's first probe) and that end on a tile's last byte or run into its look-ahead,
    at every tile boundary of a one-CTA launch, at four pointer phases."""
    rng = np.random.default_rng(100 + phase)
    backing = np.empty((48 << 10) + 128, dtype=np.uint8)
    view = aligned(backing, phase, 48 << 10)
    W.fill_haystack(view, 11 + phase)
    W.plant(view, PATS, 12 + phase, period=512, window=256)
    lo = region_lo(view)
    # one plant per tile boundary b, cycling through the offsets d: a pattern that starts at b + d,
    # then one that ends at b + d (d < 0: on the last bytes of the tile before b)
    cases = [(d, ends) for ends in (False, True) for d in (-3, -2, -1, 0, 1, 2, 3)]
    for i, b in enumerate(range(lo + TILE, view.size - 64, TILE)):
        d, ends = cases[i % len(cases)]
        pat = PATS[int(rng.integers(len(PATS)))]
        put(view, b + d - (len(pat) if ends else 0), pat)
    assert (view.size - 64 - lo) // TILE >= len(cases)
    check_all(engines, view, ("phase", phase), min_matches=100)


def test_steps_dense_in_first_stage_hits(engines, one_cta):
    """Segments planted with a pattern every 16 .. 96 bytes: 2 KiB steps with two to ten times the
    22 first-stage hits of a cfg 2 step."""
    backing = np.empty((96 << 10) + 128, dtype=np.uint8)
    view = aligned(backing, 0, 96 << 10)
    W.fill_haystack(view, 21)
    seg = 8 << 10
    for i, period in enumerate([96, 16, 64, 32, 48, 24, 80, 40, 56, 20, 72, 28]):
        part = view[i * seg: (i + 1) * seg]
        W.plant(part, PATS, 30 + i, period=period, window=period - 16 if period > 32 else 1)
    _, ac, _ = engines[0]
    hits = first_stage_hits_per_tile(view, ac)
    assert (hits > 128).sum() >= 4 and ((hits > 44) & (hits <= 128)).sum() >= 8, hits
    check_all(engines, view, "dense", min_matches=1000)


@pytest.mark.parametrize("last", [16, 32, 528, 1040, 2032])
def test_short_last_tile(engines, one_cta, last):
    """Regions of n full tiles plus `last` bytes, with patterns at the last tile's first bytes, on
    its last bytes and across the end of the region into the tail."""
    rng = np.random.default_rng(last)

    def pick():
        return PATS[int(rng.integers(len(PATS)))]
    backing = np.empty((24 << 10) + 256, dtype=np.uint8)
    end = 10 * TILE + last      # region_lo = 0 (phase 0); region_hi = end: 20 readable bytes behind it
    view = aligned(backing, 0, end + 20)
    W.fill_haystack(view, 40 + last)
    W.plant(view, PATS, 41 + last, period=512, window=256)
    for at in (10 * TILE - 1, 10 * TILE + 1):   # around the last tile's first probe
        put(view, at, pick())
    pat = pick()
    put(view, end - 24 - len(pat), pat)         # ends shortly before the region's end
    put(view, end - 3, pick())                  # starts in the last bytes and runs into the tail
    pat = pick()
    put(view, view.size - len(pat), pat)        # ends on the last byte
    check_all(engines, view, ("last", last), min_matches=10)
    for cut in (1, 2, 3, 7, 16):   # the same bytes with the region ending earlier
        check_all(engines, view[: view.size - cut], ("last", last, "cut", cut))
