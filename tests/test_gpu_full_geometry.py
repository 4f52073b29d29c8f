"""Device tests at production geometry: 2 GiB queue windows, offsets past 4 GiB, full order-step buckets.

Three parts of the device path change behaviour only at sizes the rest of the GPU suite never reaches:
  1. prefilter_kernel queues second-stage survivors as 32-bit offsets inside 2 GiB windows of its chunk
     (kWinShift, use_windows, q2win, drain2).  Only the global super-tile draw (ACG_EXP_GLOBAL_TILES),
     whose chunk is the whole region, has a chunk above 2 GiB;
  2. haystack, document and span offsets of 2^32 and more (40-bit key offsets, the staged host base,
     acg_find's growing windows);
  3. the order step at its real capacity: 16 384 tuples per bucket (order_buckets_kernel, 16 rounds per
     warp), one more tuple (compact_buckets_kernel + radix sort), bucket shifts 22 to 25 and the single list.
Every assertion compares with a reference: the CPU oracle on slices, an independent device path (another
tile draw, engine or span), or a result known by construction that the oracle confirms.

Under the dry run (ACB_EMULATE=1, tests/emu/) groups 1 and 3 run at the sizes ACB_EMU_WINSHIFT,
ACB_EMU_BUCKETSHIFT and ACB_EMU_BUCKETLOG give them, e.g.
  ACB_EMULATE=1 ACB_EMU_WINSHIFT=12 ACB_EMU_BUCKETSHIFT=12 ACB_EMU_BUCKETLOG=6 pytest tests/test_gpu_full_geometry.py -k "window or bucket"
With 4 KiB windows a warp's draw of four consecutive tiles crosses window edges; with 16 KiB windows and the
dry run's few tiles per warp the queue never carries entries into the next window (drain2 is not exercised).
"""
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_emulated_buckets import EXPAND, ORDER_BUCKETS, ORDER_FALLBACK
from test_gpu_find_batch import first_records, same as same_first
from test_gpu_kernel_matrix import (DYN_FLAGS, ON_GPU, ROWS, SETS, api_mode, apis, builder, key_widths,
                                    launch_of, plant_dense_segment, put_many, region)
from test_gpu_parity import assert_np_equal, to_device
from test_prefilter_plan import plan_of, set_experiment

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))

GIB = 1 << 30
T32 = 1 << 32


def _geometry(var, device_value):
    """The device constant, or under the dry run the value the emulated library reads from `var`."""
    v = None if ON_GPU else os.environ.get(var)
    return int(v) if v else device_value


# queue window (kWinShift, acb_prefilter.cu); bucket bytes and slots (plan_buckets / kOrderLog, acb_api.cu)
WIN_SHIFT = _geometry("ACB_EMU_WINSHIFT", 31)
BUCKET_SHIFT_ENV = None if ON_GPU else os.environ.get("ACB_EMU_BUCKETSHIFT")
BUCKET_LOG = min(_geometry("ACB_EMU_BUCKETLOG", 14), 14)
WIN = 1 << WIN_SHIFT
SLOTS = 1 << BUCKET_LOG
RADIX = ORDER_FALLBACK - ORDER_BUCKETS   # launches counted for the radix sort of a whole list
CHAIN = 8                                # launches counted for find_iter's chain resolution


def engine(ac):
    return ac.last_stats()["engine"]


def launches(ac):
    return int(ac.last_stats()["launches"])


def write(buf, at, arr):
    """Host bytes into the (device) haystack buffer."""
    if ON_GPU:
        import torch
        buf[at: at + arr.size].copy_(torch.from_numpy(arr))
        torch.cuda.synchronize()
    else:
        buf[at: at + arr.size] = arr


def ptr_of(buf):
    return buf.data_ptr() if ON_GPU else buf.ctypes.data


def dev_search(ac, ptr, api, length, span=None):
    fn = ac.find_overlapping_iter_dev_np if api == "overlapping" else ac.find_iter_dev_np
    return fn(ptr, length, span)[0]


def i64(a):
    return a.astype(np.int64)


def inside(lst, lo, hi):
    """The matches of `lst` that lie wholly inside [lo, hi)."""
    return lst[(i64(lst["start"]) >= lo) & (i64(lst["end"]) <= hi)]


def same_shifted(got, want, shift, ctx):
    """got (offsets in one haystack) == want (offsets in a slice that begins at `shift`), tuple for tuple."""
    assert len(got) == len(want), (len(got), len(want), ctx)
    assert np.array_equal(got["pid"], want["pid"]), ctx
    assert np.array_equal(i64(got["start"]) - shift, i64(want["start"])), ctx
    assert np.array_equal(i64(got["end"]) - shift, i64(want["end"])), ctx


def iter_window_matches(full, o, hay_slice, slice_at, maxlen, ctx, at_span_start=False):
    """find_iter: from the first reported match end in the slice (the iterator's cursor there; the slice's
    own start if it is the span's), the oracle on the rest of the slice agrees with `full` on the matches
    that start at least maxlen bytes before the slice's end.  Returns the number compared."""
    st, en = i64(full["start"]), i64(full["end"])
    hi = slice_at + hay_slice.size
    if at_span_start:
        ws = slice_at
    else:
        i0 = int(np.searchsorted(en, slice_at))
        if i0 >= len(full) or en[i0] >= hi - maxlen:
            return 0
        ws = int(en[i0])
    want = o.find_iter_np(np.ascontiguousarray(hay_slice[ws - slice_at:]))
    safe = hi - maxlen
    want = want[i64(want["start"]) + ws < safe]
    got = full[(st >= ws) & (st < safe)]
    same_shifted(got, want, ws, ctx)
    return len(want)


def straddle_free(single, offs):
    """The single-haystack overlapping list minus the matches that cross a document bound, as acg_doc_match
    records (doc, pid, start, end relative to the document)."""
    doc = np.searchsorted(offs, i64(single["start"]), side="right") - 1
    keep = i64(single["end"]) <= offs[doc + 1]
    out = np.zeros(int(keep.sum()), ab.DOC_MATCH_DTYPE)
    out["doc"], out["pid"] = doc[keep], single["pid"][keep]
    out["start"] = i64(single["start"][keep]) - offs[doc[keep]]
    out["end"] = i64(single["end"][keep]) - offs[doc[keep]]
    return out, int((~keep).sum())


def same_docs(got, want, ctx):
    assert len(got) == len(want), (len(got), len(want), ctx)
    for k in ("doc", "pid", "start", "end"):
        assert np.array_equal(i64(got[k]), i64(want[k])), (k, ctx)


# =====================================================================================================
# 1. Queue windows: the global tile draw over a region of at least three 2 GiB windows
# =====================================================================================================
N1 = 2 * WIN + WIN // 2 + 13                 # not a multiple of 16; 5 GiB + 13 on the device
NB_HALF = min(128 << 10, WIN // 8)           # half a neighbourhood: 128 KiB on the device
DSEG = (64 << 10) if ON_GPU else (8 << 10)   # dense segment across the first window edge
SUB1 = (3 * WIN // 16 + 99, N1 - 78)      # window edges not at multiples of 2^31 from the buffer start
WIN_VIEWS = {"full": (0, N1, None), "sub": (0, N1, SUB1), "phase1": (1, N1 - 1, None), "phase15": (15, N1 - 15, None)}


def window_edges(ptr, view, variant):
    """(region_lo, region_hi, first byte of every window's first tile after window 0) of a DYN 2 launch over
    `view`, offsets relative to the view's pointer.  The chunk is the whole region and window k holds the
    queued offsets chunk_base + k * 2^31 + rel, chunk_base = region_lo - (STRIDE - 1)."""
    off, length, span = view
    lo, hi = region(ptr + off, length, *(span or (0, length)))
    n_win = ((hi - 1 - lo) >> WIN_SHIFT) + 1   # window of a tile: its offset from region_lo >> kWinShift
    return lo, hi, [lo + k * WIN for k in range(1, n_win)], n_win


def neighbourhoods(points, total, dense_at):
    """Merged [a, b) intervals of NB_HALF bytes around every point and the dense segment (buffer offsets)."""
    iv = sorted([(max(0, p - NB_HALF), min(total, p + NB_HALF)) for p in points]
                + [(max(0, dense_at - NB_HALF), min(total, dense_at + DSEG + NB_HALF))])
    out = []
    for a, b in iv:
        if out and a <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], b))
        else:
            out.append((a, b))
    return out


@pytest.fixture(scope="class")
def window_haystack():
    """One buffer of N1 (+ 3) bytes with cfg 2's fill, on the device or, in the dry run, on the host."""
    n_alloc = (N1 + 7) & ~7
    pats = W.config_patterns("cfg2")
    if ON_GPU:
        import torch
        torch.cuda.empty_cache()
        try:
            buf = torch.empty(n_alloc, dtype=torch.uint8, device="cuda")
        except RuntimeError:
            pytest.skip("not enough device memory for the %d-byte haystack" % n_alloc)
        W.torch_fill_config("cfg2", buf, pats)
    else:
        buf = W.make_config("cfg2", n_alloc)[1]
    yield buf
    del buf
    if ON_GPU:
        import torch
        torch.cuda.empty_cache()


def window_row_id(r):
    return "%s-%s-mode%d" % (r.set, "masked" if r.masked else "plain", r.mode)


@pytest.mark.gpu
class TestQueueWindows:
    @pytest.mark.timeout(1200)
    @pytest.mark.parametrize("r", ROWS, ids=[window_row_id(r) for r in ROWS])
    def test_queue_windows(self, window_haystack, r):
        """Every (variant, masked, mode) row under the global tile draw, with and without 24-bit keys, over a
        region of >= 3 windows: the full span, pointer phases 1 and 15 and a sub-span.  Patterns start and end
        at edge + d (d = -3 .. 3, one d per round) of every window's first tile and of the region ends, inside
        host-built neighbourhoods; a dense segment crosses the first window edge.  Against the same handle at
        DYN 1 (one window only) tuple for tuple, the oracle on every neighbourhood, and the batched calls."""
        buf = window_haystack
        ptr = ptr_of(buf)
        pats = SETS[r.set]()
        lens = np.array([len(p) for p in pats], dtype=np.int64)
        maxlen = int(lens.max())
        seed = sum(r.set.encode()) * 11 + r.mode * 3 + int(r.ci)
        rng = np.random.default_rng(seed)
        geo = {}
        for name, view in WIN_VIEWS.items():
            lo, hi, edges, n_win = window_edges(ptr, view, r.variant)
            assert n_win >= 3 and len(edges) >= 2, (name, n_win)   # every DYN 2 launch crosses >= 2 window edges
            geo[name] = SimpleNamespace(lo=lo, hi=hi, edges=edges, n_win=n_win)
        dense_at = geo["full"].edges[0] - DSEG // 2
        points = []
        for name, (off, _, _) in WIN_VIEWS.items():
            g = geo[name]
            points += [off + e for e in g.edges] + [off + g.lo, off + g.hi]
        nbs = neighbourhoods(points, N1, dense_at)
        # base bytes of each neighbourhood: text, one planted pattern per 512 bytes, the dense segment
        base = []
        for k, (a, b) in enumerate(nbs):
            h = np.empty(b - a, dtype=np.uint8)
            W.fill_haystack(h, seed + 17 * k)
            W.plant(h, pats, seed + 100 + k, period=512, window=256)
            if a <= dense_at and dense_at + DSEG <= b:
                plant_dense_segment(h, pats, dense_at - a, DSEG, seed + 7)
            base.append(h)
        assert any(a <= dense_at and dense_at + DSEG <= b for a, b in nbs)
        oracles = {}

        def oracle(kind):
            if kind not in oracles:
                oracles[kind] = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=r.ci, kind=O.KIND_DFA)
            return oracles[kind]

        handles = {kind: builder(kind, r.ci).build(pats) for kind in r.kinds}
        compared = 0
        for name, view in WIN_VIEWS.items():
            off, length, span = view
            g = geo[name]
            s_lo, s_hi = span or (0, length)
            seen = {e: set() for e in g.edges}
            for d in range(-3, 4):
                hs = [h.copy() for h in base]
                for e in g.edges + [g.lo, g.hi]:
                    at = off + e
                    k = next(i for i, (a, b) in enumerate(nbs) if a <= at < b)
                    a = nbs[k][0]
                    pid_end, pid_start = rng.integers(len(pats), size=2)
                    # one pattern that ends at edge + d, one that starts there (for stride 2 and d = -1 at a
                    # window's first tile: the start one byte before it, queued with rel == 0)
                    put_many(hs[k], pats, [at + d - a - lens[pid_end], at + d - a], [pid_end, pid_start])
                for k, (a, b) in enumerate(nbs):
                    if r.ci:
                        W.flip_case(hs[k], seed + 31 * k)
                    write(buf, a, hs[k])
                for kind, ac in handles.items():
                    for api in apis(kind):
                        set_experiment(ac, DYN_FLAGS[1] | r.flags)
                        ref = dev_search(ac, ptr + off, api, length, span)
                        assert engine(ac) == int(ab.Engine.Prefilter)
                        for kw in key_widths(r.variant):
                            flags = DYN_FLAGS[2] | r.flags | kw
                            set_experiment(ac, flags)
                            assert launch_of(plan_of(ac), flags, api_mode(kind, api)) == \
                                ("prefilter", r.mode, r.masked, 2, r.variant)
                            got = dev_search(ac, ptr + off, api, length, span)
                            assert engine(ac) == int(ab.Engine.Prefilter)
                            assert_np_equal(got, ref, (name, d, kind, api, kw, "DYN 2 vs DYN 1"))
                        st, en = i64(got["start"]), i64(got["end"])
                        for e in g.edges:
                            for x in np.concatenate([st[(st >= e - 3) & (st <= e + 3)], en[(en >= e - 3) & (en <= e + 3)]]):
                                seen[e].add(int(x) - e)
                        # the oracle on every neighbourhood, cut to the searched span
                        for k, (a, b) in enumerate(nbs):
                            lo, hi = max(a - off, s_lo), min(b - off, s_hi)
                            if hi - lo < 4 * maxlen:
                                continue
                            hb = hs[k][lo + off - a: hi + off - a]
                            if api == "overlapping":
                                want = oracle(kind).find_overlapping_iter_np(hb)
                                same_shifted(inside(got, lo, hi), want, lo, (name, d, kind, "nb", a))
                                compared += len(want)
                            else:
                                compared += iter_window_matches(got, oracle(kind), hb, lo, maxlen,
                                                                (name, d, kind, "nb", a), at_span_start=lo == s_lo)
            # matches within 3 bytes on both sides of every window edge (all seven d for overlapping search)
            for e, ds in seen.items():
                assert any(x < 0 for x in ds) and any(x >= 0 for x in ds), (name, e, sorted(ds))
                if 0 in r.kinds:
                    assert set(range(-3, 4)) <= ds, (name, e, sorted(ds))
        assert compared > 1000, compared
        self._check_batches(buf, handles, pats, r, nbs, base, oracle)
        print("windows %s: %d windows per launch, %d neighbourhoods, %d oracle matches"
              % (window_row_id(r), geo["full"].n_win, len(nbs), compared))

    @staticmethod
    def _check_batches(buf, handles, pats, r, nbs, base, oracle):
        """The bytes of the last round cut into documents: the DYN 2 batch against the DYN 1 single list minus
        the straddlers (overlapping), against the DYN 1 batch and the oracle on documents inside the
        neighbourhoods (find_iter)."""
        offs = W.doc_offsets(N1, 0xD0C5 + r.mode, hi=min(16384, WIN >> 4))
        docs = (buf, offs)
        ptr = ptr_of(buf)
        for kind, ac in handles.items():
            if kind == 0:
                set_experiment(ac, DYN_FLAGS[1] | r.flags)
                single = dev_search(ac, ptr, "overlapping", N1)
                want, n_straddle = straddle_free(single, offs)
                assert n_straddle > 0
                set_experiment(ac, DYN_FLAGS[2] | r.flags)
                got = ac.find_overlapping_iter_batch_np(docs)
                assert engine(ac) == int(ab.Engine.Prefilter)
                same_docs(got, want, (kind, "overlapping batch"))
            set_experiment(ac, DYN_FLAGS[1] | r.flags)
            ref = ac.find_iter_batch_np(docs)
            set_experiment(ac, DYN_FLAGS[2] | r.flags)
            got = ac.find_iter_batch_np(docs)
            assert engine(ac) == int(ab.Engine.Prefilter)
            same_docs(got, ref, (kind, "find_iter batch"))
            checked = 0
            for (a, b), h in zip(nbs, base):
                d0 = int(np.searchsorted(offs, a, side="left"))
                for dd in range(d0, min(d0 + 40, offs.size - 1)):
                    if offs[dd + 1] > b:
                        break
                    # (the bytes of the last round: read back from the buffer)
                    db = buf[offs[dd]: offs[dd + 1]].cpu().numpy() if ON_GPU else buf[offs[dd]: offs[dd + 1]]
                    want = oracle(kind).find_iter_np(np.ascontiguousarray(db))
                    lo = np.searchsorted(got["doc"], dd, side="left")
                    hi = np.searchsorted(got["doc"], dd, side="right")
                    part = got[lo:hi]
                    assert len(part) == len(want), (kind, dd)
                    for k in ("pid", "start", "end"):
                        assert np.array_equal(i64(part[k]), i64(want[k])), (kind, dd, k)
                    checked += 1
            assert checked > 0, checked
            set_experiment(ac, 0)


# =====================================================================================================
# 2. Offsets past 4 GiB on one device
# =====================================================================================================
N2 = 6 * GIB + (256 << 20) + 4099           # resident haystack past 3 * 2^31, plus an odd remainder
SITES = (T32, 3 << 31)                       # planted straddlers
RELOC = (T32 - (3 << 20), T32 + (5 << 20))   # relocated range


def spans_spell(d, n, full, pats, ci=False):
    """Every reported span holds its pattern's bytes (ASCII case folded if ci), checked on the device."""
    import torch
    st, en, pid = i64(full["start"]), i64(full["end"]), i64(full["pid"])
    lens = np.array([len(p) for p in pats], dtype=np.int64)
    assert np.array_equal(en - st, lens[pid])
    maxlen = int(lens.max())
    table = np.zeros((len(pats), maxlen), dtype=np.uint8)
    for i, p in enumerate(pats):
        table[i, :len(p)] = np.frombuffer(p, dtype=np.uint8)

    def fold(x):
        return torch.where((x >= 65) & (x <= 90), x + 32, x) if ci else x
    t_table = torch.from_numpy(table).cuda()
    t_st, t_pid, t_len = torch.from_numpy(st).cuda(), torch.from_numpy(pid).cuda(), torch.from_numpy(en - st).cuda()
    ar = torch.arange(maxlen, device="cuda")
    for lo in range(0, len(full), 1 << 18):
        sl = slice(lo, lo + (1 << 18))
        mask = ar[None, :] < t_len[sl][:, None]
        idx = (t_st[sl][:, None] + ar[None, :]).clamp_(max=n - 1)
        assert bool(torch.all((fold(d[idx]) == fold(t_table[t_pid[sl]])) | ~mask))


@pytest.fixture(scope="class")
def past4g():
    """cfg 2's fill over N2 bytes on the device; at each site S a length-5 pattern from S - 3 to S + 2 and one
    more pattern at S + 16 (offset S exactly in the view that begins 16 bytes into the buffer)."""
    import torch
    torch.cuda.empty_cache()
    pats = W.config_patterns("cfg2")
    try:
        d = torch.empty((N2 + 7) & ~7, dtype=torch.uint8, device="cuda")
    except RuntimeError:
        pytest.skip("not enough device memory for the 6.25 GiB haystack")
    W.torch_fill_config("cfg2", d, pats)
    p5 = next(i for i, p in enumerate(pats) if len(p) == 5)
    at16 = 77
    for s in SITES:
        d[s - 3: s + 2] = torch.frombuffer(bytearray(pats[p5]), dtype=torch.uint8).cuda()
        d[s + 16: s + 16 + len(pats[at16])] = torch.frombuffer(bytearray(pats[at16]), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()
    ac = builder(0, False).build(pats)
    full = ac.find_overlapping_iter_dev_np(d.data_ptr(), N2)[0]
    assert engine(ac) == int(ab.Engine.Prefilter)
    yield SimpleNamespace(d=d, pats=pats, ac=ac, full=full, p5=p5, at16=at16, o=O.Oracle(pats, kind=O.KIND_DFA))
    del d
    torch.cuda.empty_cache()


@pytest.mark.gpu
class TestPast4GiB:
    @pytest.mark.timeout(900)
    def test_overlapping_past_4gib(self, past4g):
        """Whole-span overlapping search over 6.25 GiB: two engines agree on count and FNV-1a, the host list's
        count and FNV-1a are count_overlapping_dev's, whole = left + right + straddlers at cuts 2^32 - 1, 2^32,
        2^32 + 1, the oracle on 8 MiB windows, a span that starts past 2^32, the same search 16 bytes further
        into the buffer, and a relocated copy of the bytes around 2^32."""
        import torch
        from bench_docs import fnv1a
        h = past4g
        d, ac, full, ptr = h.d, h.ac, h.full, h.d.data_ptr()
        st, en = i64(full["start"]), i64(full["end"])
        assert int(en.max()) > T32 + GIB, int(en.max())
        for s in SITES:   # the planted straddler and its neighbour are reported
            assert ((st == s - 3) & (en == s + 2) & (i64(full["pid"]) == h.p5)).any(), s
            assert ((st == s + 16) & (i64(full["pid"]) == h.at16)).any(), s
        cnt_p, fnv_p, _ = ac.count_overlapping_dev(ptr, N2)
        assert engine(ac) == int(ab.Engine.Prefilter)
        ac.set_engine(ab.Engine.Walk)
        cnt_w, fnv_w, _ = ac.count_overlapping_dev(ptr, N2)
        assert engine(ac) == int(ab.Engine.Walk)
        ac.set_engine(ab.Engine.Auto)
        assert (cnt_p, fnv_p) == (cnt_w, fnv_w)
        assert cnt_p == len(full) and fnv_p == fnv1a(full)
        for cut in (T32 - 1, T32, T32 + 1):
            left = ac.find_overlapping_iter_dev_np(ptr, N2, span=(0, cut))[0]
            right = ac.find_overlapping_iter_dev_np(ptr, N2, span=(cut, N2))[0]
            straddle = (st < cut) & (en > cut)
            assert straddle.sum() > 0, cut
            assert len(left) + len(right) + int(straddle.sum()) == len(full), cut
            assert_np_equal(left, full[en <= cut], ("left", cut))
            assert_np_equal(right, full[st >= cut], ("right", cut))
        for off in (T32 - (4 << 20), (3 << 31) - (4 << 20) + 5, N2 - (8 << 20)):
            w = d[off: off + (8 << 20)].cpu().numpy()
            same_shifted(inside(full, off, off + w.size), h.o.find_overlapping_iter_np(w), off, ("oracle", off))
        late = (T32 + 12345, N2)
        assert_np_equal(ac.find_overlapping_iter_dev_np(ptr, N2, span=late)[0], full[st >= late[0]], "late span")
        # 16 bytes further into the buffer: offset 2^32 is the planted pattern's start
        v16 = ac.find_overlapping_iter_dev_np(ptr + 16, N2 - 16)[0]
        same_shifted(full[st >= 16], v16, 16, "view + 16")
        assert ((i64(v16["start"]) == T32) & (i64(v16["pid"]) == h.at16)).any()
        # relocation: the bytes of RELOC in a fresh buffer at the same 16-byte phase
        a, b = RELOC
        small = torch.empty(b - a + 64, dtype=torch.uint8, device="cuda")
        assert (small.data_ptr() - (ptr + a)) % 16 == 0
        small[: b - a].copy_(d[a:b])
        torch.cuda.synchronize()
        host = d[a:b].cpu().numpy()
        for kind in (0, 1, 2):
            o = O.Oracle(h.pats, match_kind=kind, kind=O.KIND_DFA)
            hk = ac if kind == 0 else builder(kind, False).build(h.pats)
            for api in apis(kind):
                big = dev_search(hk, ptr, api, N2, span=RELOC)
                rel = dev_search(hk, small.data_ptr(), api, b - a)
                same_shifted(big, rel, a, (kind, api, "relocated"))
                want = o.find_overlapping_iter_np(host) if api == "overlapping" else o.find_iter_np(host)
                assert_np_equal(rel, want, (kind, api, "relocated vs oracle"))
        del small
        # device output past 2^32: records with end > min_end, offsets moved by offset_add
        min_end, add = T32 - 1000, 3 << 31
        keep = full[en > min_end]
        out = torch.empty((len(keep) + 16, 3), dtype=torch.int64, device="cuda")
        n, _ = ac.find_overlapping_devout(ptr, N2, None, min_end, add, out.data_ptr(), len(keep) + 16)
        assert n == len(keep)
        rec = out[:n].cpu().numpy()
        assert np.array_equal(rec[:, 0], i64(keep["pid"]))
        assert np.array_equal(rec[:, 1], i64(keep["start"]) + add) and np.array_equal(rec[:, 2], i64(keep["end"]) + add)
        assert int(rec[:, 2].max()) > T32 + (3 << 31)
        print("past 4 GiB: %d matches, last end %d" % (len(full), int(en.max())))

    @pytest.mark.timeout(900)
    @pytest.mark.parametrize("kind", [0, 1, 2])
    def test_find_iter_past_4gib(self, past4g, kind):
        """find_iter over 6.25 GiB: ordered, non-overlapping, every span spells its pattern (on the device); on
        windows past 2^32 that begin at a reported match end, the oracle and the sequential engine agree."""
        h = past4g
        ptr = h.d.data_ptr()
        ac = builder(kind, False).build(h.pats)
        full = ac.find_iter_dev_np(ptr, N2)[0]
        assert engine(ac) == int(ab.Engine.Prefilter)
        st, en = i64(full["start"]), i64(full["end"])
        assert bool(np.all(st[1:] >= en[:-1])) and bool(np.all(en > st)) and int(en.max()) > T32 + GIB
        spans_spell(h.d, N2, full, h.pats)
        o = O.Oracle(h.pats, match_kind=kind, kind=O.KIND_DFA)
        maxlen = max(len(p) for p in h.pats)
        win = 4 << 20
        for off in (T32 - 4096, T32 + (1 << 20) + 7, (3 << 31) - 999, N2 - win - 4096):
            i0 = int(np.searchsorted(en, off))
            ws, we = int(en[i0]), min(N2, int(en[i0]) + win)
            assert iter_window_matches(full, o, h.d[ws:we].cpu().numpy(), ws, maxlen, (kind, off),
                                       at_span_start=True) > 500
            ac.set_engine(ab.Engine.Sequential)
            seq = ac.find_iter_dev_np(ptr, N2, span=(ws, we))[0]
            assert engine(ac) == int(ab.Engine.Sequential)
            ac.set_engine(ab.Engine.Auto)
            pf = ac.find_iter_dev_np(ptr, N2, span=(ws, we))[0]
            assert_np_equal(seq, pf, (kind, off, "sequential vs prefilter"))
            safe = we - maxlen
            assert_np_equal(seq[i64(seq["start"]) < safe], full[(st >= ws) & (st < safe)], (kind, off, "window vs full"))

    @pytest.mark.timeout(1200)
    def test_batches_past_4gib(self, past4g):
        """About 2.8 M documents over the 6.25 GiB buffer, one of them across 2^32; host and device offsets, host
        and device output, prefilter and sequential engines; and a batch that begins past 2^32 and ends before
        the buffer does."""
        import torch
        from test_gpu_batch_devout import host_records
        h = past4g
        d, full = h.d, h.full
        offs = W.doc_offsets(N2, 0xB16)
        near = np.abs(offs - T32) < 64
        offs = offs[~near]   # the document of the straddler at 2^32 - 3 .. 2^32 + 2 crosses 2^32
        k = int(np.searchsorted(offs, T32))
        assert offs[k - 1] < T32 - 3 and offs[k] > T32 + 2
        n_docs = offs.size - 1
        d_offs = torch.from_numpy(offs).cuda()
        want, n_straddle = straddle_free(full, offs)
        assert n_straddle > 0 and len(want) > 1_000_000
        ac0 = builder(0, False).build(h.pats)
        for eng in (ab.Engine.Auto, ab.Engine.Sequential):
            ac0.set_engine(eng)
            got = ac0.find_overlapping_iter_batch_np((d, offs))
            assert engine(ac0) == int(ab.Engine.Prefilter if eng == ab.Engine.Auto else eng)
            same_docs(got, want, ("overlapping batch", eng))
        ac0.set_engine(ab.Engine.Auto)
        bm = ac0.find_overlapping_iter_batch_torch((d, d_offs))
        assert host_records(bm.records).tobytes() == got.tobytes()
        flags = ac0.is_match_batch((d, offs))
        want_flags = np.bincount(i64(want["doc"]), minlength=n_docs) > 0
        assert np.array_equal(flags, want_flags)
        assert np.array_equal(ac0.is_match_batch_torch((d, d_offs)).cpu().numpy(), want_flags)
        # find_iter / find: prefilter, sequential and device output agree; sampled documents past 2^32 are the oracle's
        ac1 = builder(1, False).build(h.pats)
        it = ac1.find_iter_batch_np((d, offs))
        assert engine(ac1) == int(ab.Engine.Prefilter)
        ac1.set_engine(ab.Engine.Sequential)
        same_docs(ac1.find_iter_batch_np((d, offs)), it, "find_iter batch, sequential")
        assert engine(ac1) == int(ab.Engine.Sequential)
        ac1.set_engine(ab.Engine.Auto)
        assert host_records(ac1.find_iter_batch_torch((d, d_offs)).records).tobytes() == it.tobytes()
        first = first_records(it, n_docs)
        same_first(ac1.find_batch_np((d, offs)), first, "find_batch")
        found, rec = ac1.find_batch_torch((d, d_offs))
        assert np.array_equal(found.cpu().numpy(), first[0])
        assert host_records(rec).tobytes() == first[1].tobytes()
        o1 = O.Oracle(h.pats, match_kind=1, kind=O.KIND_DFA)
        late = np.flatnonzero(offs[:-1] >= T32 - (1 << 20))
        sample = np.unique(np.concatenate([[k - 1, k], np.random.default_rng(5).choice(late, 100)]))
        for dd in sample:
            w = o1.find_iter_np(d[offs[dd]: offs[dd + 1]].cpu().numpy())
            part = it[np.searchsorted(it["doc"], dd): np.searchsorted(it["doc"], dd, side="right")]
            same_docs(part, np.array([(x["pid"], dd, x["start"], x["end"]) for x in w], dtype=ab.DOC_MATCH_DTYPE),
                      ("oracle doc", int(dd)))
        # a batch from past 2^32 to before the end of the buffer
        i, j = int(np.searchsorted(offs, T32 + 12345)), int(np.searchsorted(offs, N2 - (7 << 20)))
        sub = offs[i: j + 1]
        assert sub[0] > T32 and sub[-1] < N2
        got = ac0.find_overlapping_iter_batch_np((d, sub))
        part = want[(i64(want["doc"]) >= i) & (i64(want["doc"]) < j)].copy()
        part["doc"] -= i
        same_docs(got, part, "batch past 2^32")
        bm = ac0.find_overlapping_iter_batch_torch((d, torch.from_numpy(sub).cuda()))
        assert host_records(bm.records).tobytes() == got.tobytes()

    @pytest.mark.timeout(900)
    def test_host_input_past_4gib(self):
        """A host haystack of 4 GiB + 64 MiB, zero except [2^32 - 32 MiB, 2^32 + 32 MiB):
        spans inside that range against the oracle, try_find / is_match from offset 0 across acg_find's growing
        windows to the one match past 2^32, and a host batch of documents past 2^32."""
        import torch
        torch.cuda.empty_cache()

        def rss():
            with open("/proc/self/statm") as f:
                return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")
        before = rss()
        hz = np.zeros(T32 + (64 << 20), dtype=np.uint8)
        a, b = T32 - (32 << 20), T32 + (32 << 20)
        pats = W.config_patterns("cfg2")
        W.fill_haystack(hz[a:b], 0xAC4611, a)
        W.plant(hz[a:b], pats, 0x5EED, a, period=1024, window=512)
        span = (T32 - (20 << 20) + 5, T32 + (20 << 20) + 3)
        view = hz[span[0]: span[1]]
        for kind in (0, 1):
            ac = builder(kind, False).build(pats)
            o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
            if kind == 0:
                got = ac.try_find_overlapping_iter_np(hz, span=span)
                same_shifted(got, o.find_overlapping_iter_np(view), span[0], "host overlapping")
            got = ac.try_find_iter_np(hz, span=span)
            assert len(got) > 10000
            same_shifted(got, o.find_iter_np(view), span[0], ("host find_iter", kind))
            assert engine(ac) == int(ab.Engine.Prefilter)
        # a batch of host documents past 2^32
        offs = T32 + (1 << 20) + W.doc_offsets(24 << 20, 0xF00)
        ac = builder(0, False).build(pats)
        single = ac.try_find_overlapping_iter_np(hz, span=(int(offs[0]), int(offs[-1])))
        want, _ = straddle_free(single, offs)
        same_docs(ac.find_overlapping_iter_batch_np((hz, offs)), want, "host batch past 2^32")
        # try_find / is_match from 0: near misses across acg_find's window edges, one match past 2^32.  The
        # text in [a, b) holds no byte below 0x20, so only the planted bytes can match.
        fp = [b"\x01needle\x02", b"\x01need\x03", b"\x04\x04\x04"]
        edges = [1 << 20, 17 << 20, 273 << 20] + [(273 << 20) + k * GIB for k in range(1, 4)]
        for e in edges + [T32 - 8]:
            hz[e - 3: e + 3] = np.frombuffer(b"\x01needl", dtype=np.uint8)
        at = T32 + 1003
        hz[at: at + 8] = np.frombuffer(fp[0], dtype=np.uint8)
        o = O.Oracle(fp, kind=O.KIND_DFA)
        for e in edges:
            assert o.try_find(hz[e - 4096: e + 4096]) is None
        assert o.try_find(hz[T32: T32 + (1 << 20)]) == (0, at - T32, at + 8 - T32)
        for kind in (0, 1, 2):
            ac = builder(kind, False).build(fp)
            m = ac.try_find(hz)
            assert m is not None and m.as_tuple() == (0, at, at + 8), (kind, m)
            assert ac.is_match(hz) and not ac.is_match(hz, span=(0, at + 7))
        # Reading the zero pages through the driver's pageable copies backs them (measured on the H100 host: the
        # resident set grows by about the array's size).  Nothing beyond that: no host copy of the span is kept.
        grown = rss() - before
        assert grown < hz.nbytes + (512 << 20), grown
        print("host input past 4 GiB: RSS grew by %d MiB" % (grown >> 20))
        del hz


# =====================================================================================================
# 3. The order step at its real capacity
# =====================================================================================================
TARGETS = sorted({c for c in (0, 1, 31, 32, 33, 1023, 1025, SLOTS - 1, SLOTS) if c <= SLOTS})
SPAN3_START = 4099                       # buckets are relative to the span start: not bucket-aligned
# max pattern length per set: bits_for(max_len) + dup_shift (1: one duplicated pattern) = 7 .. 11 tie bits
TIE_SETS = {7: 37, 8: 69, 9: 133, 10: 261, 11: 517}
DEVICE_SHIFT = {7: 25, 8: 24, 9: 23, 10: 22, 11: None}
GROUP = [b"qrstuv", b"rstuv", b"stuv"]   # suffixes of each other: one planting ends three patterns (four with the
                                         # duplicate of the first) at one offset, and starts three


def bits_for(v):
    return int(v).bit_length()


def bucket_plan(ac, n_bytes, flags=0):
    """plan_buckets (acb_api.cu) restated from the handle's plan: (shift, number of buckets), or None for the
    single list."""
    if flags & DYN_FLAGS[2]:
        return None
    tie = bits_for(ac.max_pattern_len()) + plan_of(ac).dup_shift
    if tie >= 32:
        return None
    max_shift = 32 - tie
    shift, min_shift = min(25, max_shift), 22
    if BUCKET_SHIFT_ENV:
        shift, min_shift = min(int(BUCKET_SHIFT_ENV), max_shift), 1
    if shift < min_shift:
        return None
    while (n_bytes >> shift) + 1 > 1024:
        if shift >= max_shift:
            return None
        shift += 1
    return shift, (n_bytes >> shift) + 1


def bucket_patterns(max_len):
    """Upper-case singles none of which contains another, the suffix group with a duplicate, and one long
    pattern of a byte that is never planted: no byte of any pattern is zero."""
    singles = []
    for p in W.make_patterns(200, 0xB0C, lo=5, hi=8, alphabet=(0x41, 0x5A)):
        if p not in singles and not any(p in q or q in p for q in singles):
            singles.append(p)
    singles = singles[:48]
    return singles + GROUP + [GROUP[0], b"~" * max_len], len(singles)


def bucket_layout(pats, shift, keyed_by, n_single, extra=0):
    """Plantings (position, pattern index) that put TARGETS[i] tuples in bucket i (the SLOTS bucket `extra`
    more), none in the next and one in the last, keyed by end (overlapping) or by start (leftmost).  Each
    bucket has a match whose key is the bucket's first offset and one that crosses into it (overlapping) or
    out of it (leftmost), in alternate buckets; suffix groups give tuples that share an end."""
    B = 1 << shift
    group_tuples = 4 if keyed_by == "end" else 3
    span_len = (len(TARGETS) + 1) * B + B // 2
    plants = []

    def put(key, pi, plen):
        start = key - plen if keyed_by == "end" else key
        plants.append((SPAN3_START + start, pi))

    single = 0
    for b, c in enumerate(TARGETS + [0, 1]):
        if b == len(TARGETS) + 1:
            b = span_len >> shift   # the last bucket
        c += extra if c == SLOTS else 0
        # (an edge match of one bucket and a crossing one of its neighbour would share bytes: they alternate)
        if keyed_by == "end":
            units = [("edge" if b % 2 == 0 else "cross", 1)][:c]
        else:
            units = [("edge", 1), ("cross", 1)][:c if b % 2 == 0 else 0]
        rest = c - len(units)
        n_groups = (rest // 2) // group_tuples
        units += [("group", group_tuples)] * n_groups + [("single", 1)] * (rest - n_groups * group_tuples)
        step = (B - 64) // (len(units) + 1)
        assert not units or step >= 16, (B, len(units))
        for i, (what, _) in enumerate(units):
            if what == "edge":
                key = b * B
            elif what == "cross":
                key = b * B + 2 if keyed_by == "end" else (b + 1) * B - 3
            else:
                key = b * B + 32 + i * step
            if what == "group":
                put(key, n_single, len(GROUP[0]))
            else:
                pi = single % n_single
                single += 1
                put(key, pi, len(pats[pi]))
        assert sum(u for _, u in units) == c
    return plants, span_len


def bucket_haystack(pats, shift, keyed_by, n_single, extra=0):
    plants, span_len = bucket_layout(pats, shift, keyed_by, n_single, extra)
    hay = np.zeros(SPAN3_START + span_len + 97, dtype=np.uint8)
    for pos, pi in plants:
        hay[pos: pos + len(pats[pi])] = np.frombuffer(pats[pi], dtype=np.uint8)
    return hay, (SPAN3_START, SPAN3_START + span_len)


def tuples_per_bucket(o_all, hay, span, shift, keyed_by):
    """Tuples the scan emits per bucket, from the oracle: every (pattern, end) of the overlapping list keyed by
    end, or every start offset at which some pattern matches keyed by start."""
    allm = o_all.find_overlapping_iter_np(hay, span)
    key = i64(allm["end"]) if keyed_by == "end" else np.unique(i64(allm["start"]))
    return np.bincount((key - span[0]) >> shift)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("tie_bits", list(TIE_SETS), ids=["tie%d" % t for t in TIE_SETS])
def test_order_buckets_at_capacity(tie_bits):
    """Buckets with 0, 1, 31, 32, 33, 1023, 1025, 16383 and 16384 tuples (SLOTS = 16 K slots on the device), an
    empty bucket and one tuple in the last: order_buckets_kernel runs and the result is the oracle's for
    overlapping search and find_iter kinds 1 and 2; one tuple more in the full bucket takes the compaction and
    radix sort with the same result; the same bytes as a batch give the same records (doc_records_kernel); a
    search without a match.  Sets of 7 .. 11 tie-break bits plan shifts 25, 24, 23, 22 and the single list."""
    import torch
    pats, n_single = bucket_patterns(TIE_SETS[tie_bits])
    o_all = O.Oracle(pats, kind=O.KIND_DFA)
    handles = {kind: builder(kind, False).build(pats) for kind in (0, 1, 2)}
    for ac in handles.values():
        assert ac.max_pattern_len() == TIE_SETS[tie_bits]
        assert bits_for(ac.max_pattern_len()) + plan_of(ac).dup_shift == tie_bits
    probe = bucket_plan(handles[0], 0)
    if ON_GPU:
        assert (probe[0] if probe else None) == DEVICE_SHIFT[tie_bits], probe
    shift = probe[0] if probe else (22 if ON_GPU else int(BUCKET_SHIFT_ENV or 22))
    for keyed_by, kinds in (("end", (0,)), ("start", (1, 2))):
        for extra in (0, 1):
            hay, span = bucket_haystack(pats, shift, keyed_by, n_single, extra)
            n_bytes = span[1] - span[0]
            plan = bucket_plan(handles[0], n_bytes)
            assert plan == (None if probe is None else (shift, (n_bytes >> shift) + 1)), (plan, probe)
            per = tuples_per_bucket(o_all, hay, span, shift, keyed_by)
            want_counts = [c + (extra if c == SLOTS else 0) for c in TARGETS] + [0]
            assert list(per[: len(want_counts)]) == want_counts, (keyed_by, extra, list(per[: len(want_counts)]))
            assert per[len(want_counts):].sum() == 1 and per[-1] == 1 and len(per) == (n_bytes >> shift) + 1
            d = to_device(torch.from_numpy(hay)) if ON_GPU else hay
            ptr = ptr_of(d)
            for kind in kinds:
                ac = handles[kind]
                o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
                api = "overlapping" if kind == 0 else "iter"
                want = o.find_overlapping_iter_np(hay, span) if api == "overlapping" else o.find_iter_np(hay, span)
                got = dev_search(ac, ptr, api, hay.size, span)
                assert engine(ac) == int(ab.Engine.Prefilter)
                assert_np_equal(got, want, (tie_bits, keyed_by, extra, kind))
                chain = CHAIN if api == "iter" else 0
                n_l = launches(ac) - chain
                if plan is None:
                    assert n_l == 1 + RADIX + EXPAND, (n_l, "single list")
                elif extra:
                    assert n_l >= ORDER_FALLBACK + EXPAND, (n_l, "fallback")
                else:
                    assert n_l == ORDER_BUCKETS + EXPAND, (n_l, "buckets")
                if kind == 0:
                    # the same bytes as documents: records from doc_records_kernel
                    offs = span[0] + W.doc_offsets(n_bytes, 0xD0C + extra, lo=64, hi=1 << max(7, shift - 6))
                    recs, n_straddle = straddle_free(got, offs)
                    same_docs(ac.find_overlapping_iter_batch_np((d, offs)), recs, (tie_bits, "batch", extra))
                    assert engine(ac) == int(ab.Engine.Prefilter)
                if extra == 0:
                    # nothing ends (overlapping) or starts (leftmost) in bucket 0: a search of its bytes finds nothing
                    empty = (span[0], span[0] + (1 << shift) - 16)
                    assert len(dev_search(ac, ptr, api, hay.size, empty)) == 0
            del d
    print("buckets tie%d: shift %s, %d tuples in the fullest bucket" % (tie_bits, probe and probe[0], SLOTS))
