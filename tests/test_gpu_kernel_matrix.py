"""Every prefilter_kernel instantiation on the device against the oracle, at tile, chunk and span edges.

launch_prefilter (csrc/acb_prefilter.cu) picks one of 48 instantiations of
prefilter_kernel<MODE, MASKED, DENSE, STRIDE, GEOM, DYN> from table[mode][masked][dyn][variant]:
  mode     1 for leftmost find_iter / find, 0 otherwise (Standard find_iter is mode 0 with first_only);
  masked   fold != 0 or kmask != 0xFFFFFFFF (case-insensitive, or fingerprints shorter than 4 bytes);
  dyn      tile draw: 0 static split (ACG_EXP_STATIC_TILES), 1 per-CTA counter (default), 2 global
           super-tiles (ACG_EXP_GLOBAL_TILES);
  variant  0 stride 1, 1 dense, 2 stride-2 narrow, 3 stride-2 wide.
Brute mode is a runtime branch of the stride-1 kernel and the byte-set scan is a kernel pair of its own.

The ledger (CPU) restates that choice from the host plan and shows that the case table below reaches
all 48, brute in both modes and the byte-set scan in both modes.  The matrix (GPU) runs every
(variant, masked, mode) row under every tile draw on one device-resident haystack large enough that the
global draw installs several super-tiles per CTA, and compares tuple for tuple, order included, with the
oracle: the full span, an odd sub-span, three pointer phases, spans of a few bytes to a few CTA rounds,
and the batched entry points over the same bytes cut into documents.

Under the dry run (ACB_EMULATE=1, tests/emu/) the same tests run at reduced sizes on the CPU library."""
import itertools
import os
from types import SimpleNamespace

import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import sampled_docs_match_the_oracle
from test_gpu_find_batch import first_records, same as same_first
from test_gpu_parity import assert_np_equal, to_device
from test_prefilter_plan import plan_of, set_experiment

KEY24, GLOBAL_TILES, STATIC_TILES, NO_BYTESCAN = 8, 16, 32, 64   # include/acb200_debug.h
DYN_FLAGS = {0: STATIC_TILES, 1: 0, 2: GLOBAL_TILES}


def _on_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


ON_GPU = _on_gpu()
# the haystack of every row: 256 MiB on the device; the dry run executes kernels one CTA at a time on
# the CPU and takes 4 MiB (with its 3 emulated SMs, still more super-tiles than CTAs in every geometry)
N = (256 << 20) if ON_GPU else (4 << 20)
BRUTE_N = (4 << 20) if ON_GPU else (256 << 10)
BYTESET_N = (64 << 20) if ON_GPU else (1 << 20)
PHASE_LEN = (8 << 20) if ON_GPU else (512 << 10)
DENSE_SEG = (2 << 20) if ON_GPU else (96 << 10)


def sm_count():
    if ON_GPU:
        import torch
        return torch.cuda.get_device_properties(0).multi_processor_count
    return int(os.environ.get("ACB_EMU_SMS", "3"))   # tests/emu/cuda_runtime.h


# ---- launch geometry, restated from csrc/acb_prefilter.cu (PfGeom, PfPass, launch_prefilter) ----------
# variant -> (warps per CTA, bytes per warp step, CTAs per SM)
GEOM = {0: (32, 1024, 1), 1: (32, 1024, 1), 2: (32, 2048, 1), 3: (16, 2048, 2)}
SUPER = 256   # tiles per super-tile of the global draw (kSuper)


def region(base, readable, scan_lo, scan_hi):
    """[region_lo, region_hi) of enqueue_prefilter_range: the 16-byte aligned filter region whose 4-byte
    look-ahead stays inside the readable bytes; the rest of [scan_lo, scan_hi) is head and tail."""
    lo = scan_lo + ((16 - ((base + scan_lo) & 15)) & 15)
    limit = min(scan_hi, readable - 20 if readable >= 20 else 0)
    hi = lo + ((limit - lo) & ~15) if limit > lo else lo
    if lo > scan_hi:
        lo = hi = scan_hi
    return lo, hi


def grid(variant, region_bytes):
    warps, tile, per_sm = GEOM[variant]
    steps = -(-region_bytes // (warps * tile))
    return min(sm_count() * per_sm, steps or 1)


def tile_edges(variant, lo, hi):
    """Start offsets of every tile of a launch over [lo, hi): the global draw numbers tiles from region_lo,
    the per-CTA draws and the static split from each CTA's chunk (a 1/grid share in 16-byte blocks)."""
    _, tile, _ = GEOM[variant]
    edges = [np.arange(lo, hi, tile, dtype=np.int64)]
    g = grid(variant, hi - lo)
    per_cta = -(-((hi - lo) >> 4) // g)
    for c in range(g):
        a, b = lo + c * per_cta * 16, min(hi, lo + (c + 1) * per_cta * 16)
        edges.append(np.arange(a, b, tile, dtype=np.int64))
    return np.concatenate(edges)


# ---- the ledger: which kernel a search launches ----------------------------------------------------
def launch_of(p, flags, mode):
    """The kernel a search in `mode` launches on a handle with plan `p` and experiment flags `flags`
    (enqueue_prefilter_range + launch_prefilter): ("bytescan", mode), ("brute", mode) or
    ("prefilter", mode, masked, dyn, variant)."""
    assert p.supported
    if p.bs_n and not flags & NO_BYTESCAN:
        return ("bytescan", mode)
    if p.brute:
        return ("brute", mode)
    masked = int(p.fold != 0 or p.kmask != 0xFFFFFFFF)
    dyn = 0 if flags & STATIC_TILES else (2 if flags & GLOBAL_TILES else 1)
    variant = (3 if p.wide else 2) if p.stride == 2 else (1 if p.dense else 0)
    return ("prefilter", mode, masked, dyn, variant)


def api_mode(kind, api):
    return 0 if api == "overlapping" or kind == 0 else 1


def alpha12():
    return [bytes((97 + (i * 7 + j * 5 + (i >> j)) % 12) for j in range(4 + i % 5)) for i in range(300)]


def short300():
    pats = W.make_patterns(300, 31)
    return [p[:3] for p in pats[:150]] + pats[150:]


SETS = {
    "narrow": lambda: W.make_patterns(5000, 0xAC5000),    # stride-2 narrow, k = 4
    "wide": lambda: W.make_patterns(50, 0xAC0050),        # stride-2 wide
    "dense": lambda: W.make_patterns(20000, 0xAC1000),    # dense (blocked filter + anchor map)
    "short": short300,                                    # stride 1, k = 3 (masked)
    "alpha12": alpha12,                                   # stride 1, k = 4, unmasked
    "brute": lambda: [bytes([b]) for b in range(256)] + [b"abc", b"zz"],
    "byteset": lambda: [bytes(t) for t in itertools.product(b"ab", repeat=4)] + [b"abbaab", b"bbbbbbb"],
}

# (set, variant, masked, mode, case-insensitive, match kinds, extra flags)
ROWS = [
    ("narrow", 2, 0, 0, False, (0,), 0), ("narrow", 2, 0, 1, False, (1, 2), 0),
    ("narrow", 2, 1, 0, True, (0,), 0), ("narrow", 2, 1, 1, True, (1, 2), 0),
    ("wide", 3, 0, 0, False, (0,), 0), ("wide", 3, 0, 1, False, (1,), 0),
    ("wide", 3, 1, 0, True, (0,), 0), ("wide", 3, 1, 1, True, (1,), 0),
    ("dense", 1, 0, 0, False, (0,), 0), ("dense", 1, 0, 1, False, (1, 2), 0),
    ("dense", 1, 1, 0, True, (0,), 0), ("dense", 1, 1, 1, True, (1, 2), 0),
    ("short", 0, 1, 0, False, (0,), 0), ("short", 0, 1, 1, False, (1,), 0),
    # kind 0 over this set gets a three-needle byte-set plan: the fingerprint kernel needs NO_BYTESCAN
    ("alpha12", 0, 0, 0, False, (0,), NO_BYTESCAN), ("alpha12", 0, 0, 1, False, (1,), 0),
]
ROWS = [SimpleNamespace(set=s, variant=v, masked=m, mode=md, ci=ci, kinds=k, flags=f) for s, v, m, md, ci, k, f in ROWS]
MATRIX = [(r, d) for r in ROWS for d in (1, 0, 2)]


def row_id(rd):
    r, d = rd
    return "%s-%s-mode%d-dyn%d" % (r.set, "masked" if r.masked else "plain", r.mode, d)


def apis(kind):
    return ("overlapping", "iter") if kind == 0 else ("iter",)


def key_widths(variant):
    return (0, KEY24) if variant in (2, 3) else (0,)


def builder(kind, ci):
    return ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA)


def ledger_cases():
    """(name, set, kind, ci, flags, api, expected launch) of every search the device tests make."""
    for r, dyn in MATRIX:
        for kind in r.kinds:
            for kw in key_widths(r.variant):
                for api in apis(kind):
                    yield (row_id((r, dyn)), r.set, kind, r.ci, DYN_FLAGS[dyn] | r.flags | kw, api,
                           ("prefilter", r.mode, r.masked, dyn, r.variant))
    for kind in (0, 1):
        for dyn in (0, 1, 2):
            yield ("brute", "brute", kind, False, DYN_FLAGS[dyn], "iter", ("brute", kind))
        yield ("byteset", "byteset", kind, False, 0, "iter", ("bytescan", kind))


def test_ledger_covers_every_instantiation():
    """Host-only plans: the case table reaches all 48 instantiations, brute and the byte-set scan in both modes."""
    pats = {}
    handles = {}
    seen = {}
    for name, s, kind, ci, flags, api, want in ledger_cases():
        if s not in pats:
            pats[s] = SETS[s]()
        if (s, kind, ci) not in handles:
            handles[s, kind, ci] = builder(kind, ci).host_only().build(pats[s])
        ac = set_experiment(handles[s, kind, ci], flags)
        got = launch_of(plan_of(ac), flags, api_mode(kind, api))
        assert got == want, (name, kind, api, flags)
        seen.setdefault(got, set()).add(name)
    every = {("prefilter", m, k, d, v) for m in (0, 1) for k in (0, 1) for d in (0, 1, 2) for v in range(4)}
    assert len(every) == 48 and every <= set(seen), sorted(every - set(seen))
    for extra in (("brute", 0), ("brute", 1), ("bytescan", 0), ("bytescan", 1)):
        assert extra in seen, extra
    print("ledger: %d/48 instantiations, brute x%d, byte-set x%d" % (
        len(every & set(seen)), sum(k[0] == "brute" for k in seen), sum(k[0] == "bytescan" for k in seen)))


# ---- haystacks ---------------------------------------------------------------------------------------
def put_many(hay, pats, starts, pids):
    """Write pats[pids[i]] at starts[i] (those that fit; later writes win where they overlap)."""
    lens = np.array([len(p) for p in pats], dtype=np.int64)
    starts, pids = np.asarray(starts, dtype=np.int64), np.asarray(pids, dtype=np.int64)
    ok = (starts >= 0) & (starts + lens[pids] <= hay.size)
    starts, pids = starts[ok], pids[ok]
    table = np.zeros((len(pats), int(lens.max())), dtype=np.uint8)
    for i, p in enumerate(pats):
        table[i, :len(p)] = np.frombuffer(p, dtype=np.uint8)
    for L in np.unique(lens[pids]):
        sel = lens[pids] == L
        hay[starts[sel][:, None] + np.arange(L)[None, :]] = table[pids[sel], :L]


def plant_edges(hay, pats, edges, rng):
    """At edge b, cycling: a pattern that starts at b + d, then one that ends at b + d, d in -3 .. 3."""
    cases = [(d, ends) for ends in (False, True) for d in range(-3, 4)]
    pids = rng.integers(len(pats), size=edges.size)
    lens = np.array([len(p) for p in pats], dtype=np.int64)[pids]
    d = np.array([c[0] for c in cases])[np.arange(edges.size) % len(cases)]
    ends = np.array([c[1] for c in cases])[np.arange(edges.size) % len(cases)]
    put_many(hay, pats, edges + d - np.where(ends, lens, 0), pids)


def plant_dense_segment(hay, pats, at, nbytes, seed):
    """Patterns every 16 .. 96 bytes: first-stage hits at nearly every probe, slot overflow, several
    second-stage rounds per step and full queues."""
    seg = 8 << 10
    periods = [96, 16, 64, 32, 48, 24, 80, 40, 56, 20, 72, 28]
    for i in range(nbytes // seg):
        p = periods[i % len(periods)]
        W.plant(hay[at + i * seg: at + (i + 1) * seg], pats, seed + i, period=p, window=p - 16 if p > 32 else 1)


SUB = (N // 8 + 4099, N // 4 + 3333)                                   # odd start, odd end
PHASES = {1: (PHASE_LEN + 101, 3), 7: (PHASE_LEN + 2033, 1), 15: (PHASE_LEN + 4077, 2)}  # length, tail start
DENSE_AT = N // 2
SMALL_AT = DENSE_AT + 5


def small_spans(variant):
    warps, tile, _ = GEOM[variant]
    round_ = warps * tile   # one CTA round: every warp of one CTA takes one step
    lens = list(range(41)) + [1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097]
    lens += [round_ - 16, round_, round_ + 16, 5 * round_ + 16]
    return [(SMALL_AT, SMALL_AT + L) for L in lens]


def make_haystack(name, ci, variant, n):
    """W.fill_haystack + one planted match per 512 bytes; patterns around every tile / CTA-chunk edge of
    the full span's launch in this row's geometry; a segment of dense hits; patterns at the region ends
    of the spans the test searches (start at region_hi - 1, - 2, - 3 and region_lo - 1)."""
    pats = SETS[name]()
    seed = sum(name.encode()) * 7 + int(ci)
    rng = np.random.default_rng(seed)
    hay = np.empty(n, dtype=np.uint8)
    W.fill_haystack(hay, seed)
    W.plant(hay, pats, seed + 1, period=512, window=256)
    offs = W.doc_offsets(n, seed)
    if n != N:   # (the brute-mode haystack: planted matches only)
        return pats, hay, offs
    lo, hi = region(0, n, 0, n)
    plant_edges(hay, pats, tile_edges(variant, lo, hi), rng)
    plant_dense_segment(hay, pats, DENSE_AT, DENSE_SEG, seed + 2)
    b = offs[1:-1:7]   # across, ending at and starting at document boundaries
    pids = rng.integers(len(pats), size=b.size)
    lens = np.array([len(p) for p in pats], dtype=np.int64)[pids]
    put_many(hay, pats, np.choose(np.arange(b.size) % 3, [b - lens // 2, b - lens, b]), pids)
    ends = [hi - 1]
    s_lo, s_hi = region(0, n, *SUB)
    ends += [s_hi - 2, s_lo - 1]
    for ph, (L, k) in PHASES.items():
        p_lo, p_hi = region(ph, L, 0, L)
        ends += [ph + p_hi - k, ph + p_lo - 1]
    put_many(hay, pats, ends, rng.integers(len(pats), size=len(ends)))
    if ci:
        W.flip_case(hay, seed + 3)
    return pats, hay, offs


_CACHE = {}


def haystack(name, ci, variant, n=N):
    """One (set, case) haystack at a time, with its device copy and the oracle lists computed on it."""
    import torch
    key = (name, ci, variant, n)
    if _CACHE.get("key") != key:
        _CACHE.clear()
        if ON_GPU:
            torch.cuda.empty_cache()
        pats, hay, offs = make_haystack(name, ci, variant, n)
        d = to_device(torch.from_numpy(hay))
        assert d.data_ptr() % 16 == 0   # region(): the haystack's 16-byte phase is the offset's
        _CACHE.update(key=key, pats=pats, hay=hay, offs=offs, d=d, oracles={}, lists={})
    return SimpleNamespace(**_CACHE)


def oracle_list(h, kind, ci, api, off, length, span):
    """The oracle's list for one search, computed once per haystack and reused across tile draws and key widths."""
    key = (kind, ci, api, off, length, span)
    if key not in h.lists:
        if (kind, ci) not in h.oracles:
            h.oracles[kind, ci] = O.Oracle(h.pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
        o = h.oracles[kind, ci]
        view = h.hay[off: off + length]
        fn = o.find_overlapping_iter_np if api == "overlapping" else o.find_iter_np
        h.lists[key] = fn(view, span)
    return h.lists[key]


def search(ac, h, api, off, length, span):
    fn = ac.find_overlapping_iter_dev_np if api == "overlapping" else ac.find_iter_dev_np
    return fn(h.d.data_ptr() + off, length, span)[0]


def views(variant, n):
    """(pointer offset, readable length, span) of every search of a row."""
    out = [(0, n, None), (0, n, SUB)]
    out += [(ph, L, None) for ph, (L, _) in PHASES.items()]
    out += [(0, n, s) for s in small_spans(variant)]
    return out


def check_views(ac, h, kind, ci, api, variant, ctx, n=N):
    for off, length, span in views(variant, n):
        want = oracle_list(h, kind, ci, api, off, length, span)
        got = search(ac, h, api, off, length, span)
        assert_np_equal(got, want, (ctx, api, off, length, span))
        if span is None or span[1] > span[0]:
            assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter), (ctx, api, off, span)
        if span is None and off == 0:
            assert len(want) >= n // 512, (ctx, api, len(want))


def batch_input(h):
    return (h.d if ON_GPU else h.hay, h.offs)


def check_batches(ac, h, kind, ci, ctx):
    """The same bytes cut into documents: the document bound of the verifier, and the unbucketed emitter
    of the unordered scans (find_batch)."""
    batch = batch_input(h)
    n_docs = h.offs.size - 1
    if kind == 0:
        single = oracle_list(h, kind, ci, "overlapping", 0, h.hay.size, None)
        got = ac.find_overlapping_iter_batch_np(batch)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter), ctx
        doc = np.searchsorted(h.offs, single["start"].astype(np.int64), side="right") - 1
        keep = single["end"].astype(np.int64) <= h.offs[doc + 1]
        assert (~keep).sum() > 0, ctx
        want = single[keep]
        assert len(got) == len(want), (ctx, len(got), len(want))
        base = h.offs[got["doc"].astype(np.int64)].astype(np.uint64)
        assert np.array_equal(got["pid"], want["pid"]), ctx
        assert np.array_equal(got["start"] + base, want["start"]), ctx
        assert np.array_equal(got["end"] + base, want["end"]), ctx
    it = ac.find_iter_batch_np(batch)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter), ctx
    assert len(it) > n_docs // 2, ctx
    o = h.oracles.get((kind, ci)) or O.Oracle(h.pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    sampled_docs_match_the_oracle(it, o, h.hay, h.offs, "iter", n=200)
    first = ac.find_batch_np(batch)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter), ctx
    same_first(first, first_records(it, n_docs), ctx)


# ---- the matrix ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("rd", MATRIX, ids=[row_id(rd) for rd in MATRIX])
def test_kernel_matrix(rd):
    r, dyn = rd
    ctx = row_id(rd)
    h = haystack(r.set, r.ci, r.variant)
    lo, hi = region(h.d.data_ptr(), N, 0, N)
    _, tile, _ = GEOM[r.variant]
    n_super = -(-((hi - lo) // tile) // SUPER)
    # the global draw must install further super-tiles (the prefetch / publish / install path), and the
    # per-CTA draws must split the region over the whole grid
    assert n_super > grid(r.variant, hi - lo) == sm_count() * GEOM[r.variant][2], (n_super, grid(r.variant, hi - lo))
    for kind in r.kinds:
        ac = builder(kind, r.ci).build(h.pats)
        for kw in key_widths(r.variant):
            flags = DYN_FLAGS[dyn] | r.flags | kw
            set_experiment(ac, flags)
            for api in apis(kind):
                assert launch_of(plan_of(ac), flags, api_mode(kind, api)) == ("prefilter", r.mode, r.masked, dyn, r.variant)
                check_views(ac, h, kind, r.ci, api, r.variant, (ctx, kind, kw))
        set_experiment(ac, DYN_FLAGS[dyn] | r.flags)
        check_batches(ac, h, kind, r.ci, (ctx, kind, "batch"))
    if (r.set, r.masked, r.mode) == ("narrow", 0, 0) and dyn != 1:
        # the same filter under another tile draw verifies as many candidates, give or take the
        # unconditional ones (hits that own the start one byte before a tile depend on the tiling)
        ac = builder(0, False).build(h.pats)
        set_experiment(ac, DYN_FLAGS[dyn])
        search(ac, h, "overlapping", 0, N, None)
        cand = ac.last_stats()["candidates"]
        set_experiment(ac, 0)
        search(ac, h, "overlapping", 0, N, None)
        c1 = ac.last_stats()["candidates"]
        assert abs(cand - c1) <= c1 // 10, (cand, c1)


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind", [0, 1])
def test_brute_mode_verifies_every_offset(kind):
    """All 256 single bytes: no selective fingerprint, the stride-1 kernel verifies every offset of the
    region (one candidate each), under every tile draw."""
    h = haystack("brute", False, 0, BRUTE_N)
    ac = builder(kind, False).build(h.pats)
    for dyn in (0, 1, 2):
        set_experiment(ac, DYN_FLAGS[dyn])
        for api in apis(kind):
            assert launch_of(plan_of(ac), DYN_FLAGS[dyn], api_mode(kind, api)) == ("brute", kind)
            for off, length, span in [(0, BRUTE_N, None), (0, BRUTE_N, (4099, BRUTE_N - 777)), (7, BRUTE_N // 2 + 33, None)]:
                got = search(ac, h, api, off, length, span)
                assert_np_equal(got, oracle_list(h, kind, False, api, off, length, span), (kind, dyn, api, off, span))
                st = ac.last_stats()
                assert st["engine"] == int(ab.Engine.Prefilter)
                lo, hi = region(h.d.data_ptr() + off, length, *(span or (0, length)))
                assert st["candidates"] == hi - lo, (kind, dyn, api, off, span, st["candidates"], hi - lo)


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind", [0, 1])
def test_byteset_scan_and_its_retirement(kind):
    """Two needle bytes (a, b): bytescan_kernel in both modes against the oracle on text where the needles
    are rare; then, on one handle, a needle-dense search of 256 KiB retires the byte-set scan, and the next
    search runs the kernel behind it with the same results."""
    import torch
    pats = SETS["byteset"]()
    hay = np.empty(BYTESET_N, dtype=np.uint8)
    W.fill_haystack(hay, 77, alphabet=(0x41, 0x5A))   # upper-case text: no needle byte
    W.plant(hay, pats, 78, period=1024, window=512)
    d = to_device(torch.from_numpy(hay))
    o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
    ac = builder(kind, False).build(pats)
    for api in apis(kind):
        assert launch_of(plan_of(ac), 0, api_mode(kind, api)) == ("bytescan", kind)
        fn = ac.find_overlapping_iter_dev_np if api == "overlapping" else ac.find_iter_dev_np
        ofn = o.find_overlapping_iter_np if api == "overlapping" else o.find_iter_np
        for off, length, span in [(0, BYTESET_N, None), (0, BYTESET_N, (4099, BYTESET_N - 777)), (15, BYTESET_N // 2 + 9, None)]:
            want = ofn(hay[off: off + length], span)
            assert_np_equal(fn(d.data_ptr() + off, length, span)[0], want, (kind, api, off, span))
            assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
            assert len(want) > 0
        assert launch_of(plan_of(ac), 0, api_mode(kind, api)) == ("bytescan", kind)   # not retired
    rng = np.random.default_rng(kind)
    dense = np.frombuffer(bytes(rng.choice(list(b"ab"), size=256 << 10)), dtype=np.uint8).copy()
    dd = to_device(torch.from_numpy(dense))
    api = apis(kind)[-1]
    want = o.find_iter_np(dense)
    ac = builder(kind, False).build(pats)
    fn = ac.find_iter_dev_np
    assert launch_of(plan_of(ac), 0, api_mode(kind, api)) == ("bytescan", kind)
    first = fn(dd.data_ptr(), dense.size)[0]
    assert_np_equal(first, want, (kind, "needle-dense"))
    after = launch_of(plan_of(ac), 0, api_mode(kind, api))
    assert after[0] != "bytescan", after
    again = fn(dd.data_ptr(), dense.size)[0]
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert_np_equal(again, want, (kind, "retired"))
    assert_np_equal(fn(d.data_ptr(), BYTESET_N)[0], o.find_iter_np(hay), (kind, "retired, sparse"))
