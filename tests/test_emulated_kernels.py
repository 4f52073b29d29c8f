"""The product's kernel sources executed on the CPU (tests/emu/: g++ build of csrc/*.cu against a
dry-run CUDA runtime, CUDA threads as fibers) and compared with the oracle.

This is a check of the kernels' *logic* -- chunk/tile partitioning, ownership of start offsets at
every alignment, the stride-1 / stride-2 / wide / dense variants, queues and overflow paths,
ordering keys, chain resolution, the device-resident and sharded entry points, the pipelined host
path -- on machines without a GPU.  It models neither the hardware's concurrency nor its memory
model; the `-m gpu` suite on an H100 remains the parity gate."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "emu"))
import aho_corasick_b200 as ab  # noqa: E402
import oracle_py as O  # noqa: E402
from aho_corasick_b200 import packed, sharded as S, workload as W  # noqa: E402
from test_prefilter_plan import plan_of  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def emulated_library():
    import build_emu
    import os
    lib = ctypes.CDLL(str(build_emu.build(asan=os.environ.get("ACB_EMU_ASAN") == "1")))
    ab._declare(lib)
    packed._declare(lib)
    lib.acg_debug_set_pipeline_chunk.argtypes = [ctypes.c_void_p, ctypes.c_uint64]
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


def workload(n_pat, seed, nbytes, ci=False):
    pats = W.make_patterns(n_pat, seed)
    hay = np.empty(nbytes, dtype=np.uint8)
    W.fill_haystack(hay, 5)
    W.plant(hay, pats, 6, period=1024, window=512)
    if ci:
        W.flip_case(hay, 7)
    return pats, hay


def build(pats, kind=0, ci=False, engine=ab.Engine.Auto):
    return (ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci)
            .kind(ab.AhoCorasickKind.DFA).build(pats).set_engine(engine))


# name -> (patterns, seed, bytes, match kind, case-insensitive, expected plan)
VARIANTS = {
    "stride2_narrow": (5000, 0xAC5000, 768 << 10, 0, False),
    "stride2_narrow_ci_leftmost": (5000, 0xAC5000, 512 << 10, 1, True),
    "stride2_wide": (50, 0xAC0050, 768 << 10, 1, False),
    "stride1_short_patterns": (300, 31, 256 << 10, 2, False),
    "dense": (20000, 0xAC1000, 384 << 10, 0, False),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_prefilter_variants_device_and_host_paths(name):
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, nbytes, ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    ac = build(pats, kind, ci)
    plan = plan_of(ac)   # the variant must really be the kernel instantiation its name says
    assert plan.supported and not plan.brute
    assert (plan.stride, bool(plan.wide), bool(plan.dense), plan.k) == {
        "stride2_narrow": (2, False, False, 4), "stride2_narrow_ci_leftmost": (2, False, False, 4),
        "stride2_wide": (2, True, False, 4), "stride1_short_patterns": (1, False, False, 3),
        "dense": (1, False, True, 4)}[name]
    assert bool(plan.fold) == ci
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    ptr = hay.ctypes.data  # "device" memory is host memory in the dry run
    if kind == 0:
        want = o.find_overlapping_iter_np(hay)
        got, _ = ac.find_overlapping_iter_dev_np(ptr, hay.size)
        eq(got, want, name)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        eq(ac.try_find_overlapping_iter_np(hay), want, name + " host")
        cnt, fnv, _ = ac.count_overlapping_dev(ptr, hay.size)
        ocnt, ofnv = o.scan_overlapping_count(hay)
        assert (cnt, fnv) == (ocnt, ofnv)
        ac.set_engine(ab.Engine.Walk)
        eq(ac.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, name + " walk")
        ac.set_engine(ab.Engine.Auto)
    want = o.find_iter_np(hay)
    assert len(want) > 100
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], want, name)
    eq(ac.try_find_iter_np(hay), want, name + " host")
    s, e = 4099, hay.size - 777
    eq(ac.find_iter_dev_np(ptr, hay.size, span=(s, e))[0], o.find_iter_np(hay, span=(s, e)), name + " span")


@pytest.mark.parametrize("name", ["stride2_narrow", "stride2_wide", "stride1_short_patterns"])
def test_every_alignment_of_the_device_pointer(name):
    """Head / aligned region / tail bookkeeping: the same bytes at 18 different pointer phases and
    span ends, against the oracle."""
    n, seed, _, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, 40 << 10, ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    W.plant(hay, pats, 8, period=64, window=32)   # dense matches, also across every boundary
    ac = build(pats, 0, ci)
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    backing = np.zeros(hay.size + 64, dtype=np.uint8)
    for phase in range(18):
        view = backing[phase:phase + hay.size]
        view[:] = hay
        for cut in (0, 1, 2, 3, 15, 16, 17, 33):
            sub = view[:hay.size - cut]
            eq(ac.find_overlapping_iter_dev_np(sub.ctypes.data, sub.size)[0], o.find_overlapping_iter_np(sub), (phase, cut))


def test_sharded_slices_reproduce_the_whole():
    """acg_find_overlapping_devout with ownership by end offset (SURVEY section 8e): the
    concatenation of the ranks' outputs equals the single-device stream."""
    pats, hay = workload(5000, 0xAC5000, 512 << 10)
    ac = build(pats)
    want = O.Oracle(pats, kind=O.KIND_DFA).find_overlapping_iter_np(hay)
    back = int(ac.max_pattern_len()) - 1
    for world in (2, 3, 5):
        parts = []
        for lo, hi, read_lo in S.slice_plan(0, hay.size, world, ac.max_pattern_len()):
            piece = np.ascontiguousarray(hay[read_lo:hi])
            out = np.zeros(len(want) + 16, ab.MATCH_DTYPE)
            n, _ = ac.find_overlapping_devout(piece.ctypes.data, piece.size, (0, piece.size), lo - read_lo, read_lo,
                                              out.ctypes.data, out.size)
            parts.append(out[:n])
            assert read_lo == max(0, lo - back)
        eq(np.concatenate(parts), want, world)


def test_pipelined_host_path_with_many_chunks():
    """The chunked H2D + scan overlap of the host entry points, with the chunk shrunk so that a
    1 MiB haystack takes many launches with their own scan ranges."""
    pats, hay = workload(5000, 0xAC5000, 1 << 20)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for chunk in (4096, 64 << 10, 200 << 12):
        ac = build(pats)
        assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, chunk) == 0
        eq(ac.try_find_overlapping_iter_np(hay), o.find_overlapping_iter_np(hay), chunk)
        eq(ac.try_find_iter_np(hay, span=(123, hay.size - 5)), o.find_iter_np(hay, span=(123, hay.size - 5)), chunk)
    lf = build(pats, 1)
    ab._lib.acg_debug_set_pipeline_chunk(lf._h, 8192)
    eq(lf.try_find_iter_np(hay), O.Oracle(pats, match_kind=1, kind=O.KIND_DFA).find_iter_np(hay), "leftmost-first")


def test_pageable_host_source_goes_through_the_copy_pool():
    """A host haystack in ordinary (not page-locked) memory is staged by the library's copy threads into
    a page-locked ring, chunk by chunk (run_prefilter; every pointer counts as pageable in the dry run).
    Chunks of 6 MiB are above the pool's threshold, so the worker threads really split them; the ring is
    reused from the third chunk on, and the last chunk is partial."""
    pats, hay = workload(5000, 0xAC5000, (20 << 20) + 12345)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    ac = build(pats)
    assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, 6 << 20) == 0
    eq(ac.try_find_overlapping_iter_np(hay), o.find_overlapping_iter_np(hay))
    eq(ac.try_find_overlapping_iter_np(hay, span=(5 << 20, hay.size - 7)),
       o.find_overlapping_iter_np(hay, span=(5 << 20, hay.size - 7)), "sub-span")


def test_tuple_buffer_overflow_rescan_and_brute_mode():
    """More matches than the initial tuple capacity (counter overflow -> regrow -> rescan) and a
    pattern set whose fingerprints cannot be selective (every offset is verified)."""
    hay = np.frombuffer(b"ab" * (1 << 19), dtype=np.uint8)           # 1 Mi bytes, a match at every offset
    pats = [b"a", b"b", b"ab", b"ba", b"aba"]
    ac = build(pats)
    want = O.Oracle(pats, kind=O.KIND_DFA).find_overlapping_iter_np(hay[: 600 << 10])
    assert len(want) > (1 << 20)
    eq(ac.try_find_overlapping_iter_np(hay[: 600 << 10]), want)
    eq(build(pats, 2).try_find_iter_np(hay[: 64 << 10]), O.Oracle(pats, match_kind=2, kind=O.KIND_DFA).find_iter_np(hay[: 64 << 10]))


@pytest.mark.parametrize("name", ["stride2_narrow", "stride2_wide", "stride1_short_patterns", "dense"])
def test_exact_size_device_buffers(name):
    """Haystacks that fill their allocation exactly, with a pattern ending on the last byte: every
    read the kernels make must stay inside [0, hay_len) (under ACB_EMU_ASAN=1 an over-read aborts
    the run; without the sanitizer this still checks the tiny and ragged sizes)."""
    n, seed, _, kind, ci = VARIANTS[name]
    pats = W.make_patterns(n, seed)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    ac = build(pats, 0, ci)
    o = O.Oracle(pats, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    rng = np.random.default_rng(17)
    for size in list(range(0, 70)) + [127, 128, 129, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 33000]:
        hay = np.empty(size, dtype=np.uint8)          # its own allocation of exactly `size` bytes
        hay[:] = rng.integers(0x20, 0x7F, size=size, dtype=np.uint8)
        for p in (pats[size % len(pats)], pats[(size * 7 + 1) % len(pats)]):
            if len(p) <= size:
                hay[size - len(p):] = np.frombuffer(p, dtype=np.uint8)   # ends on the last byte
                break
        want = o.find_overlapping_iter_np(hay)
        got, _ = ac.find_overlapping_iter_dev_np(hay.ctypes.data if size else 0, size)
        eq(got, want, (name, size))
        eq(ac.try_find_overlapping_iter_np(hay), want, (name, size, "host"))
        if size in (0, 1, 5, 17, 64, 129, 1025, 4097):
            ac.set_engine(ab.Engine.Walk)
            eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data if size else 0, size)[0], want, (name, size, "walk"))
            ac.set_engine(ab.Engine.Sequential)
            eq(ac.find_iter_dev_np(hay.ctypes.data if size else 0, size)[0], o.find_iter_np(hay), (name, size, "seq"))
            ac.set_engine(ab.Engine.Auto)
            eq(ac.find_iter_dev_np(hay.ctypes.data if size else 0, size)[0], o.find_iter_np(hay), (name, size, "iter"))


def test_random_sets_on_exact_size_buffers():
    """Randomized differential on haystacks that fill their allocation exactly: small alphabets,
    duplicates, 1-byte patterns, all match kinds, every entry point family."""
    import random
    rng = random.Random(4242)
    for it in range(90):
        alphabet = [b"ab", b"abcd", b"aAbBcC ", bytes(range(256)), b"abcdefghijklmnopqrstuvwxyz"][it % 5]
        npat = rng.choice([1, 2, 5, 20, 200])
        pats = [bytes(rng.choice(alphabet) for _ in range(rng.randint(1, rng.choice([3, 8, 20])))) for _ in range(npat)]
        if it % 4 == 0:
            pats += [pats[0], pats[-1][:2]]
        size = rng.choice([0, 1, 2, 3, 4, 5, 7, 15, 16, 17, 31, 33, 100, 1000, 5000, 40000])
        hay = np.empty(size, dtype=np.uint8)
        hay[:] = np.frombuffer(bytes(rng.choice(alphabet) for _ in range(size)), dtype=np.uint8)
        ptr = hay.ctypes.data if size else 0
        kind = it % 3
        ci = it % 7 == 0
        ac = build(pats, kind, ci)
        o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
        lo = rng.randrange(0, size + 1)
        hi = rng.randrange(lo, size + 1)
        for span in ((0, size), (lo, hi)):
            if kind == 0:
                eq(ac.find_overlapping_iter_dev_np(ptr, size, span=span)[0], o.find_overlapping_iter_np(hay, span=span), (it, span))
            eq(ac.find_iter_dev_np(ptr, size, span=span)[0], o.find_iter_np(hay, span=span), (it, span))
            eq(ac.try_find_iter_np(hay, span=span), o.find_iter_np(hay, span=span), (it, span, "host"))
            m = ac.try_find(hay, span=span)
            assert (m.as_tuple() if m else None) == o.try_find(hay, span=span), (it, span)


@pytest.mark.parametrize("kind", [0, 1])
def test_unselective_steps_verify_in_place(kind):
    """A selective fingerprint set (so the Bloom path is taken) on a haystack made of pattern
    beginnings: every probe hits, the per-step hit count exceeds the slot queue and the step falls
    back to verifying its hits in place (the `total > kPfSlots` path), for stride 2 and stride 1."""
    for extra, stride in ((W.make_patterns(300, 5), 2), ([p[:3] for p in W.make_patterns(150, 5)], 1)):
        pats = [b"abab", b"baba", b"ababab", b"bab"][: 3 if stride == 2 else 4] + extra
        ac = build(pats, kind)
        plan = plan_of(ac)
        assert plan.supported and not plan.brute and plan.stride == stride
        hay = np.frombuffer(b"ab" * 20000 + b"xyz" + b"ba" * 3000, dtype=np.uint8).copy()
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        if kind == 0:
            eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), stride)
            assert ac.last_stats()["candidates"] > hay.size // 2   # (nearly) every offset was verified
        eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), stride)


# ---- switchable kernel / plan variants (include/acb200_debug.h: ACG_EXP_KEY24 = 8, ACG_EXP_GLOBAL_TILES = 16, ACG_EXP_STATIC_TILES = 32,
# ACG_EXP_NO_BYTESCAN = 64)
def set_experiment(ac, flags):
    ab._lib.acg_debug_set_experiment.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
    assert ab._lib.acg_debug_set_experiment(ac._h, flags) == 0
    return ac


@pytest.mark.parametrize("flags", [8, 16, 24, 32, 40])
@pytest.mark.parametrize("name", ["stride2_narrow", "stride2_narrow_ci_leftmost"])
def test_experimental_variants_match_the_oracle(name, flags):
    """24-bit first-stage keys and the static tile split (the non-default variants) on the
    cfg 2 / cfg 3 pattern sets: overlapping, find_iter, sub-span, host path, count + FNV."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, nbytes, ci)
    W.plant(hay[: 64 << 10], pats, 9, period=96, window=40)   # a stretch with dense matches
    ac = set_experiment(build(pats, kind, ci), flags)
    assert plan_of(ac).stride == 2 and not plan_of(ac).wide
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    ptr = hay.ctypes.data
    if kind == 0:
        want = o.find_overlapping_iter_np(hay)
        eq(ac.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, (name, flags))
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        eq(ac.try_find_overlapping_iter_np(hay), want, (name, flags, "host"))
        cnt, fnv, _ = ac.count_overlapping_dev(ptr, hay.size)
        assert (cnt, fnv) == o.scan_overlapping_count(hay)
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], o.find_iter_np(hay), (name, flags))
    s, e = 4099, hay.size - 777
    eq(ac.find_iter_dev_np(ptr, hay.size, span=(s, e))[0], o.find_iter_np(hay, span=(s, e)), (name, flags, "span"))
    # the default kernel on the same handle gives the same candidates-independent answer
    set_experiment(ac, 0)
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], o.find_iter_np(hay), (name, "default"))


@pytest.mark.parametrize("flags", [0, 8, 16, 32, 40])
def test_experimental_variants_at_every_alignment(flags):
    """Ownership of the start one byte before a tile / chunk / region (the e == 0 corner of the
    lane-local second stage, tiles drawn dynamically) at 18 pointer phases x 8 span ends."""
    n, seed, _, kind, ci = VARIANTS["stride2_narrow"]
    pats, hay = workload(n, seed, 72 << 10, ci)
    W.plant(hay, pats, 8, period=64, window=32)
    ac = set_experiment(build(pats, 0, ci), flags)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    backing = np.zeros(hay.size + 64, dtype=np.uint8)
    for phase in range(18):
        view = backing[phase:phase + hay.size]
        view[:] = hay
        for cut in (0, 1, 2, 3, 15, 16, 17, 33):
            sub = view[:hay.size - cut]
            eq(ac.find_overlapping_iter_dev_np(sub.ctypes.data, sub.size)[0], o.find_overlapping_iter_np(sub), (flags, phase, cut))


def test_27_bit_keys_on_the_wide_geometry_and_short_pattern_tails():
    """27-bit first-stage keys (the default) with the 16 KiB bitmap (cfg 4's plan), and 4-byte patterns
    at odd offsets followed by every possible byte."""
    n, seed, nbytes, kind, ci = VARIANTS["stride2_wide"]
    pats, hay = workload(n, seed, 256 << 10, ci)
    ac = build(pats, kind, ci)
    assert plan_of(ac).wide and plan_of(ac).key_shift == 5
    o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
    eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), "wide key27")
    pats = [b"abcd", b"bcde", b"wxyz", b"abcdq"] + W.make_patterns(5000, 0xAC5000)
    body = b"".join(b" " * (i % 2) + p + bytes([x]) for i, p in enumerate(pats[:4] * 64) for x in (i * 37 % 256,))
    hay = np.frombuffer(body + bytes(range(256)) * 4, dtype=np.uint8).copy()
    ac = build(pats, 0)
    assert plan_of(ac).stride == 2 and plan_of(ac).key_shift == 5
    o = O.Oracle(pats, kind=O.KIND_DFA)
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "tails")


@pytest.mark.parametrize("flags", [0, 16, 32])
def test_experimental_variants_unselective_steps(flags):
    pats = [b"abab", b"baba", b"ababab"] + W.make_patterns(5000, 0xAC5000)
    ac = set_experiment(build(pats, 0), flags)
    assert plan_of(ac).stride == 2 and not plan_of(ac).wide
    hay = np.frombuffer(b"ab" * 20000 + b"xyz" + b"ba" * 3000, dtype=np.uint8).copy()
    o = O.Oracle(pats, kind=O.KIND_DFA)
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), flags)
    eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), flags)


@pytest.mark.parametrize("name", ["stride2_wide", "stride1_short_patterns", "dense"])
def test_dynamic_tiles_on_the_other_variants(name):
    """ACG_EXP_STATIC_TILES = 32 and ACG_EXP_GLOBAL_TILES = 16 with the wide, stride-1 and dense instantiations."""
    n, seed, nbytes, kind, ci = VARIANTS[name]
    pats, hay = workload(n, seed, min(nbytes, 256 << 10), ci)
    if name == "stride1_short_patterns":
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    ac = set_experiment(build(pats, kind, ci), 16)
    eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), (name, 'global tiles'))
    ac = set_experiment(build(pats, kind, ci), 32)
    eq(ac.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), name)
    if kind == 0:
        eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), name)
        s, e = 4099, hay.size - 777
        eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size, span=(s, e))[0], o.find_overlapping_iter_np(hay, span=(s, e)), name)


# ---- dense table produced on the "device" (acg_build_on_device, SURVEY section 8f.2) -------------
def _builder(kind, ci, **kw):
    b = ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA)
    for k, v in kw.items():
        getattr(b, k)(v)
    return b


def _same_tables(a, b, ctx):
    ta, tb = a.tables(), b.tables()
    assert set(ta) == set(tb)
    for k in ta:
        va, vb = ta[k], tb[k]
        if isinstance(va, np.ndarray):
            assert np.array_equal(va, vb), (k, ctx)
        else:
            assert va == vb, (k, ctx)


def _same_plan(a, b, ctx):
    pa, pb = plan_of(a), plan_of(b)
    for f in ("supported", "brute", "dense", "stride", "wide", "k", "kmask", "fold", "mult", "mult3", "shift",
              "log_bits", "bitmap_words", "amap_log", "n_rows", "dup_shift"):
        assert getattr(pa, f) == getattr(pb, f), (f, ctx)
    if pa.supported:
        n = int(pa.bitmap_words)
        assert np.array_equal(np.ctypeslib.as_array(pa.bitmap, shape=(n,)), np.ctypeslib.as_array(pb.bitmap, shape=(n,))), ctx
        if pa.amap_log:
            m = 1 << pa.amap_log
            assert np.array_equal(np.ctypeslib.as_array(pa.amap, shape=(m,)), np.ctypeslib.as_array(pb.amap, shape=(m,))), ctx
    assert np.array_equal(np.ctypeslib.as_array(pa.depth16, shape=(int(pa.n_rows),)),
                          np.ctypeslib.as_array(pb.depth16, shape=(int(pb.n_rows),))), ctx


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("ci", [False, True])
def test_device_fill_reproduces_the_host_table(kind, ci):
    """Table, derived prefilter plan and search results of acg_build_on_device == acg_build, on the
    golden-style corner sets (1-byte patterns, duplicates, prefixes, empty pattern) and random sets."""
    import random
    rng = random.Random(1000 + kind * 2 + ci)
    sets = [[b"apple", b"maple", b"Snapple"], [b"a", b"ab", b"abc", b"b", b"bca", b"a"], [b"", b"ab", b"b"], [b"x"],
            [b"append", b"appendage", b"app"], W.make_patterns(400, 3), W.make_patterns(60, 4, lo=1, hi=5)]
    for _ in range(25):
        sets.append([bytes(rng.choice(b"abAB") for _ in range(rng.randint(1, 7))) for _ in range(rng.randint(1, 40))])
    for pats in sets:
        host = _builder(kind, ci).build(pats)
        dev = _builder(kind, ci, device_fill=True).build(pats)
        ctx = (pats[:4], kind, ci)
        _same_plan(host, dev, ctx)     # before the table is fetched: derived from the trie alone
        _same_tables(host, dev, ctx)   # acg_dfa_table fetches the device-built table
        assert host.memory_usage() == dev.memory_usage()
        hay = np.frombuffer(b"xxabcaBAbab Snapple appendage maple" * 40 + bytes(rng.choice(b"abAB") for _ in range(3000)),
                            dtype=np.uint8).copy()
        o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
        eq(dev.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), ctx)
        if kind == 0:
            eq(dev.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), ctx)


def test_device_fill_on_the_baseline_pattern_sets():
    for n, seed, kind, ci in ((5000, 0xAC5000, 0, False), (5000, 0xAC5000, 1, True), (50, 0xAC0050, 1, False),
                              (20000, 0xAC1000, 0, False)):
        pats, hay = workload(n, seed, 192 << 10, ci)
        host = _builder(kind, ci).build(pats)
        dev = _builder(kind, ci, device_fill=True).build(pats)
        _same_plan(host, dev, n)
        o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
        eq(dev.find_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_iter_np(hay), n)
        if kind == 0:   # both engines read the device-built table
            eq(dev.set_engine(ab.Engine.Walk).find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0],
               o.find_overlapping_iter_np(hay), n)
        _same_tables(host, dev, n)


def test_device_fill_with_a_rebuilt_plan():
    """ACG_EXP_KEY24 re-derives the prefilter plan after the build: on a device-filled handle that runs
    off the builder's shallow trie edges (the fill plan's per-row arrays are gone by then)."""
    pats, hay = workload(5000, 0xAC5000, 192 << 10)
    host = set_experiment(_builder(0, False).build(pats), 8)
    dev = set_experiment(_builder(0, False, device_fill=True).build(pats), 8)
    assert plan_of(dev).key_shift == 8
    _same_plan(host, dev, "key24")
    o = O.Oracle(pats, kind=O.KIND_DFA)
    eq(dev.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "key24 dev fill")
    set_experiment(dev, 0)
    assert plan_of(dev).key_shift == 5
    _same_plan(set_experiment(host, 0), dev, "back to 27-bit keys")
    eq(dev.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "default dev fill")


def test_device_fill_falls_back_for_other_start_kinds():
    pats = [b"abcd", b"bcd", b"cd", b"b"]
    for sk in (ab.StartKind.Both, ab.StartKind.Anchored):
        host = _builder(1, False, start_kind=sk).build(pats)
        dev = _builder(1, False, start_kind=sk, device_fill=True).build(pats)
        _same_tables(host, dev, sk)


# ---- the reference's regression tests around its memchr-class prefilters, src/tests.rs:1537-1660:
# results only (the device engine has no such prefilters), through the product on the dry-run library
def test_reference_regressions():
    pat = "Tsubaki House-Triple Shot Vol01校花三姐妹".encode()
    assert ab.AhoCorasick.builder().ascii_case_insensitive(True).build([pat]).find(b"") is None
    assert ab.AhoCorasick.new([b"ab/j/", b"x/"]).is_match(b"ab/j/")      # issue 53
    for c in range(ord("a"), ord("z"), 3):
        for c2 in range(ord("a"), ord("z"), 2):
            needle = bytes([c, c2])
            ac = ab.AhoCorasick.builder().ascii_case_insensitive(True).prefilter(True).build([needle])
            assert len(ac.find_iter(needle.upper())) == 1, needle


def test_reference_regression_stream_across_reads():
    """src/tests.rs:1588-1660 (issue 64): a match that straddles two reads of a stream."""
    magic, begin = b"1234j", 65535

    class Reader:
        def __init__(self):
            self.pos = 0

        def read(self, n):
            if self.pos > 100000:
                return b""
            out = bytearray(n)
            lo, hi = max(begin, self.pos), min(begin + len(magic), self.pos + n)
            if lo < hi:
                out[lo - self.pos:hi - self.pos] = magic[lo - begin:hi - begin]
            self.pos += n
            return bytes(out)

    ac = ab.AhoCorasick.builder().byte_classes(False).build([magic])
    whole = bytearray()
    r = Reader()
    while True:
        b = r.read(8192)
        if not b:
            break
        whole += b
    from_whole = ac.find_iter(bytes(whole))[0].start()
    assert from_whole == begin
    for chunk in (8192, 65536, 65535 + 2, 4096 + 1):
        first = next(iter(ac.stream_find_iter(Reader(), chunk_bytes=chunk)))
        assert first.start() == from_whole, chunk


def test_verify_equality_vectors_of_packed_pattern_rs():
    """src/packed/pattern.rs:422-480 (is_equal / is_prefix, the memcmp behind Teddy's verify): the
    same vectors against the device verifier -- a candidate whose last byte differs must not match."""
    base = b"abcdefghijklmn"
    for n in range(1, len(base) + 1):
        x, y = base[:n], base[:n - 1] + b"x"
        for searcher in (ab.AhoCorasick.builder().match_kind(ab.MatchKind.LeftmostFirst).build([x]),
                         packed.Searcher.new([x])):
            assert searcher.find(y) is None and searcher.find(x).as_tuple() == (0, 0, n), n
            assert searcher.find(b"zz" + x + y).as_tuple() == (0, 2, 2 + n)
            assert [m.as_tuple() for m in searcher.find_iter(y + x + y + x)] == [(0, n, 2 * n), (0, 3 * n, 4 * n)]
    foo = packed.Searcher.new([b"foo"])
    assert foo.find(b"foobar").as_tuple() == (0, 0, 3) and foo.find(b"fobfo") is None


def test_walk_engine_at_every_alignment():
    """K1 walks four shards per lane on a 16-byte grid anchored below the span start: every pointer
    phase x span start / end inside a block, spans shorter than one shard, 1-byte and empty patterns."""
    pats = W.make_patterns(300, 21) + [b"a", b"ab", b""]
    hay = np.empty(20 << 10, dtype=np.uint8)
    W.fill_haystack(hay, 12, alphabet=(0x61, 0x66))
    W.plant(hay, pats[:300], 13, period=128, window=64)
    ac = build(pats, 0, engine=ab.Engine.Walk)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    backing = np.zeros(hay.size + 64, dtype=np.uint8)
    for phase in (0, 1, 3, 7, 8, 15, 16, 17):
        view = backing[phase:phase + hay.size]
        view[:] = hay
        for s, e in ((0, hay.size), (1, hay.size - 1), (5, 6), (17, 40), (33, 33), (4097, 9001), (hay.size - 3, hay.size)):
            got, _ = ac.find_overlapping_iter_dev_np(view.ctypes.data, view.size, span=(s, e))
            eq(got, o.find_overlapping_iter_np(view, span=(s, e)), (phase, s, e))
            assert ac.last_stats()["engine"] == int(ab.Engine.Walk)


def test_concurrent_searches_lease_separate_workspaces():
    """Searches through one handle from several threads (Send + Sync, src/lib.rs:274-326) each lease
    a workspace of the handle's pool; results are the oracle's and acg_last_stats is per caller."""
    from concurrent.futures import ThreadPoolExecutor
    import random
    rng = random.Random(5)
    pats = [bytes(rng.choice(b"abcd") for _ in range(rng.randint(2, 6))) for _ in range(40)]
    hays = [np.frombuffer(bytes(rng.choice(b"abcd") for _ in range(rng.choice([10, 500, 20000]))), dtype=np.uint8).copy()
            for _ in range(12)]
    ac = build(pats, 0)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    want = [(o.find_overlapping_iter_np(h), o.find_iter_np(h)) for h in hays]

    def work(i):
        h = hays[i % len(hays)]
        a = ac.try_find_overlapping_iter_np(h)
        raw = ac.last_stats()["raw_matches"]       # this thread's own search, whatever the others are doing
        b = ac.try_find_iter_np(h)
        return i % len(hays), a, raw, b

    with ThreadPoolExecutor(6) as ex:
        for i, a, raw, b in ex.map(work, range(72)):
            eq(a, want[i][0], i)
            eq(b, want[i][1], i)
            assert raw == len(want[i][0]), (i, raw)


# ---- byte-set scan: the start-bytes / rare-bytes prefilter role (bytescan_kernel) -----------------
BYTESCAN_SETS = [
    ("start3", [b"Quartz", b"Xenon", b"Zanzibar"], dict()),                     # start bytes Q, X, Z
    ("start1", [b"xylophone", b"xyz", b"xx"], dict()),
    ("start_ci", [b"Sam", b"samwise"], dict(ci=True)),                          # S, s
    ("start2", [b"Quartz", b"Quebec", b"Zanzibar"], dict()),
    ("leftmost", [b"apple", b"app", b"maple syrup", b"ma"], dict(kind=1)),
    ("leftmost_longest", [b"apple", b"app", b"maple syrup", b"ma"], dict(kind=2)),
]


@pytest.mark.parametrize("name,pats,kw", BYTESCAN_SETS)
def test_bytescan_engine(name, pats, kw):
    kind, ci = kw.get("kind", 0), kw.get("ci", False)
    rng = np.random.default_rng(len(name))
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz SMQ.,", dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=96 << 10)].copy()
    for i in range(0, hay.size - 64, 977):      # plant occurrences at many alignments
        p = pats[(i // 977) % len(pats)]
        hay[i:i + len(p)] = np.frombuffer(p, dtype=np.uint8)
    ac = (ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).build(pats))
    plan = plan_of(ac)
    assert plan.bs_n >= 1, (name, ac.prefilter_kind())
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci)
    ptr = hay.ctypes.data
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], o.find_iter_np(hay), name)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    cand = ac.last_stats()["candidates"]
    assert 0 < cand < hay.size // 4
    if kind == 0:
        eq(ac.find_overlapping_iter_dev_np(ptr, hay.size)[0], o.find_overlapping_iter_np(hay), name)
        eq(ac.try_find_overlapping_iter_np(hay), o.find_overlapping_iter_np(hay), (name, "host"))
    # every pointer phase x span ends inside a block
    backing = np.zeros(hay.size + 64, dtype=np.uint8)
    small = hay[: 20 << 10]
    for phase in (0, 1, 5, 15, 16, 17, 31):
        view = backing[phase:phase + small.size]
        view[:] = small
        for s, e in ((0, small.size), (3, small.size - 5), (977, 977 + 40), (4097, 9001), (small.size - 20, small.size)):
            eq(ac.find_iter_dev_np(view.ctypes.data, view.size, span=(s, e))[0], o.find_iter_np(view, span=(s, e)), (name, phase, s, e))
    # the fingerprint filter on the same handle agrees
    set_experiment(ac, 64)
    eq(ac.find_iter_dev_np(ptr, hay.size)[0], o.find_iter_np(hay), (name, "fingerprints"))
    set_experiment(ac, 0)


def test_bytescan_retires_when_needles_are_everywhere():
    """Needles in more than one offset out of eight: the scan still answers correctly and the handle
    goes back to the fingerprint filter for later searches (the reference's PrefilterState)."""
    pats = [b"aaab", b"aab"]
    ac = ab.AhoCorasick.builder().build(pats)
    assert plan_of(ac).bs_n == 1
    hay = np.frombuffer(b"aaaaab" * 30000, dtype=np.uint8).copy()
    assert ab.AhoCorasick.builder().build([b"apple", b"maple", b"Snapple"]).prefilter_kind() == 3   # rare bytes with
    assert plan_of(ab.AhoCorasick.builder().build([b"apple", b"maple", b"Snapple"])).bs_n == 0       # offsets: fingerprints
    o = O.Oracle(pats)
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "dense needles")
    assert plan_of(ac).bs_n == 0
    eq(ac.find_overlapping_iter_dev_np(hay.ctypes.data, hay.size)[0], o.find_overlapping_iter_np(hay), "after retiring")


@pytest.mark.parametrize("shift", [12, 14])
def test_queue_windows_on_small_inputs(shift):
    """The 32-bit queued offsets of the prefilter kernel live in windows of the chunk (2 GiB on the
    device); tests/emu_window_check.py runs the variants with the window shrunk to 4 / 16 KiB."""
    import os
    import subprocess
    env = dict(os.environ, ACB_EMU_WINSHIFT=str(shift))
    r = subprocess.run([sys.executable, str(ROOT / "tests" / "emu_window_check.py")], capture_output=True, text=True,
                       env=env, timeout=1200)
    assert r.returncode == 0 and "WINDOWS OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
