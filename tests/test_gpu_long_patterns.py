"""Long patterns (1 KiB to 64 KiB) on every device path, against the oracle, at the plan and tie-break limits.

The device path changes behaviour with max_pattern_len in many places, and none of them is reached by a short
pattern:
  * plan_prefilter (acb_plan.hpp): no plan when max_len >= 0xFFFE or bit_width(max_len) + dup_shift > 24;
  * verify_from (acb_prefilter.cu): walks up to 65 533 bytes on the trie path, 16-bit depths against a 32-bit
    count, tie-breaks (max_len - len) << dup_shift | index, and the document bound of batched searches;
  * plan_buckets (acb_api.cu): 10 tie bits still give buckets (shift 22, 32-bit in-bucket keys), 11 the single
    list and the radix sort;
  * walk_overlapping_kernel: every lane reads max_len - 1 bytes back, across many 256-byte shards, clamped at
    the span start;
  * run_prefilter's pipelined host path: a tail of max_len + 64 bytes longer than the H2D chunk;
  * acg_find: look-ahead of max_len + 64 bytes past each window (1 MiB, 16 MiB, ...) and the Standard rescan of
    the starts in [hi, end) when the first match found ends past the window;
  * chain_select_kernel on periodic patterns, where every start is a candidate.
Every result is compared with the oracle (KIND_DFA) tuple for tuple, order included, and every case asserts the
engine it ran on, the prefilter plan and, where it applies, the order path (from the launch count).

Under the dry run (tests/test_emulated_long_patterns.py) the same checks run at smaller sizes on the CPU build of
the kernels."""
import os
import time
from types import SimpleNamespace

import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_emulated_buckets import EXPAND, ORDER_BUCKETS, ORDER_FALLBACK
from test_emulated_batch import _DevView
from test_gpu_kernel_matrix import ON_GPU
from test_gpu_parity import assert_np_equal
from test_prefilter_plan import plan_of

RADIX = ORDER_FALLBACK - ORDER_BUCKETS   # launches counted for the radix sort of a whole list
CHAIN = 8                                # launches counted for find_iter's chain resolution
MIB = 1 << 20
AUTO, WALK, PREFILTER, SEQUENTIAL = (int(e) for e in (ab.Engine.Auto, ab.Engine.Walk, ab.Engine.Prefilter,
                                                      ab.Engine.Sequential))

# Where the searches run: on the device, or on the dry-run library (tests/test_emulated_long_patterns.py sets
# on_gpu False whatever the host has, so that its "device" buffers are host memory).  Read at every call.
RUN = SimpleNamespace(on_gpu=ON_GPU)

# haystack sizes: the device runs the real geometry, the dry run (one CTA at a time on the CPU) a reduced one
SIZES = {"hay": (4 * MIB, 128 << 10), "walk": (MIB, 64 << 10), "pipe": (4 * MIB, 512 << 10),
         "bucket": (16 * MIB + 4096, 48 << 10)}


def size(name):
    return SIZES[name][0 if RUN.on_gpu else 1]


def sm_count():
    if RUN.on_gpu:
        import torch
        return torch.cuda.get_device_properties(0).multi_processor_count
    return int(os.environ.get("ACB_EMU_SMS", "3"))   # tests/emu/cuda_runtime.h


# ---- handles, inputs and the engine / plan / order path of a search -----------------------------------------
def builder(kind, ci=False):
    return ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA)


def oracle(pats, kind=0, ci=False, prefilter=True):
    return O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA, prefilter=prefilter)


def engine(ac):
    return int(ac.last_stats()["engine"])


def launches(ac):
    return int(ac.last_stats()["launches"])


def device_copy(hay):
    """(keepalive, address) of the haystack in device memory (host memory under the dry run)."""
    if RUN.on_gpu:
        import torch
        t = torch.from_numpy(hay).cuda()
        torch.cuda.synchronize()
        return t, t.data_ptr()
    return hay, hay.ctypes.data


def pinned_copy(hay):
    """The haystack in page-locked host memory (a plain copy under the dry run)."""
    if RUN.on_gpu:
        import torch
        t = torch.from_numpy(hay).pin_memory()
        return t.numpy()
    return hay.copy()


def env_int(name):
    v = None if RUN.on_gpu else os.environ.get(name)
    return int(v) if v else None


def bucket_plan(ac, n_bytes):
    """plan_buckets (acb_api.cu) restated: (shift, log2 of the slots per bucket), or None for the single list.
    Under the dry run ACB_EMU_BUCKETSHIFT / ACB_EMU_BUCKETLOG shrink both, as in the library."""
    tie = int(ac.max_pattern_len()).bit_length() + plan_of(ac).dup_shift
    if tie >= 32:
        return None
    max_shift = 32 - tie
    shift, min_shift, log = min(25, max_shift), 22, 14
    if env_int("ACB_EMU_BUCKETSHIFT") is not None:
        shift, min_shift = min(env_int("ACB_EMU_BUCKETSHIFT"), max_shift), 1
    if env_int("ACB_EMU_BUCKETLOG") is not None:
        log = min(env_int("ACB_EMU_BUCKETLOG"), 14)
    if shift < min_shift:
        return None
    while (n_bytes >> shift) + 1 > 1024:
        if shift >= max_shift:
            return None
        shift += 1
    return shift, log


def expected_order_launches(ac, n_bytes, keys):
    """Launches of a device-resident search whose scan emits tuples with these span-relative keys (end offsets
    for overlapping search, start offsets for leftmost find_iter), without the chain resolution: the order step
    in shared memory, its fallback when a bucket overflows, or the single list.  Returns (path, launches)."""
    bp = bucket_plan(ac, n_bytes)
    if bp is None:
        return "single", 1 + RADIX + EXPAND
    shift, log = bp
    per = np.bincount(np.asarray(keys, dtype=np.int64) >> shift) if len(keys) else np.zeros(1, np.int64)
    if int(per.max()) > (1 << log):
        return "fallback", None
    return "buckets", ORDER_BUCKETS + EXPAND


def assert_order_path(ac, n_bytes, keys, extra, ctx):
    path, want = expected_order_launches(ac, n_bytes, keys)
    got = launches(ac) - extra
    if want is None:
        assert got >= ORDER_FALLBACK + EXPAND, (got, path, ctx)
    else:
        assert got == want, (got, path, ctx)
    return path


def plan_fields(ac):
    p = plan_of(ac)
    return dict(supported=p.supported, brute=p.brute, dense=p.dense, stride=p.stride, wide=p.wide, bs_n=p.bs_n,
                dup_shift=p.dup_shift)


def assert_plan(ac, want, ctx):
    got = plan_fields(ac)
    if not want.get("supported", 1):   # no plan: only what made it so is pinned
        assert got["supported"] == 0 and got["dup_shift"] == want.get("dup_shift", got["dup_shift"]), (got, ctx)
        return got
    for k, v in want.items():
        assert got[k] == v, (k, got, want, ctx)
    return got


# ---- pattern families ---------------------------------------------------------------------------------------
def rand_bytes(rng, alphabet, n):
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def rand_hay(rng, alphabet, n):
    return np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)].copy()


def fam_random(alphabet):
    """a. One random long pattern over `alphabet`, its first half, its last third and a 12-byte piece."""
    def make(L, seed):
        rng = np.random.default_rng(seed)
        p = rand_bytes(rng, alphabet, L)
        q = L // 4
        pats = [p, p[: max(1, L // 2)], p[-max(1, L // 3):], p[q: q + 12]]
        return SimpleNamespace(pats=pats, long=[p], hay_alphabet=alphabet, near=True)
    return make


def fam_closed(which):
    """b. One long pattern and its prefixes (or suffixes) of 1, 2, 4, ..., L bytes: one end (or start) offset
    closes many patterns and leftmost-first prunes."""
    def make(L, seed):
        rng = np.random.default_rng(seed)
        p = rand_bytes(rng, b"abcdefgh", L)
        lens = sorted({1 << i for i in range(L.bit_length()) if (1 << i) < L} | {L})
        pats = [p[:n] if which == "prefix" else p[-n:] for n in lens]
        return SimpleNamespace(pats=pats, long=[p], hay_alphabet=b"abcdefgh", near=False)
    return make


def fam_periodic(L, seed):
    """c. (ab)^n, (ba)^n, a^L and a^(L/2) on a haystack of periodic runs: every start is a candidate."""
    n = L // 2
    pats = [b"ab" * n, b"ba" * n, b"a" * L, b"a" * max(1, L // 2)]
    return SimpleNamespace(pats=pats, long=pats[:3], hay_alphabet=None, near=False)


def fam_mixed(L, seed):
    """e. A keyword list (9 000 cfg-like patterns: more than 8 192 fingerprints, the dense plan) with three long
    sentences in it."""
    rng = np.random.default_rng(seed)
    words = W.make_patterns(9000, 0x1057 + seed, lo=4, hi=16)
    longs = [bytes(rng.integers(0x20, 0x7F, L, dtype=np.uint8)) for _ in range(2)] + \
        [bytes(rng.integers(0x20, 0x7F, max(4, L // 3), dtype=np.uint8))]
    return SimpleNamespace(pats=words[:4000] + longs + words[4000:], long=longs, hay_alphabet=None, near=True,
                           text=True)


FAMILIES = {
    "ab": fam_random(b"ab"),
    "acgt": fam_random(b"acgt"),
    "bytes": fam_random(bytes(range(256))),
    "prefix": fam_closed("prefix"),
    "suffix": fam_closed("suffix"),
    "periodic": fam_periodic,
    "mixed": fam_mixed,
}


def near_miss(p):
    """d. The pattern with its last byte changed: the verifier walks the whole length and fails."""
    return p[:-1] + bytes([p[-1] ^ 1 if p[-1] ^ 1 != p[-1] else 0])


def base_haystack(fam, n, seed):
    rng = np.random.default_rng(seed)
    if getattr(fam, "text", False):
        hay = np.empty(n, np.uint8)
        W.fill_haystack(hay, seed)
        W.plant(hay, fam.pats, seed + 1, period=512, window=256)
        return hay
    if fam.hay_alphabet is None:   # periodic runs of (ab)*, (ba)*, a* and a few random bytes
        parts, total = [], 0
        while total < n:
            r = int(rng.integers(1, 4 * max(len(p) for p in fam.pats)))
            unit = [b"ab", b"ba", b"a", b"ab"][int(rng.integers(0, 4))]
            parts.append((unit * (r // len(unit) + 1))[:r] + bytes([int(rng.integers(0x61, 0x64))]))
            total += r + 1
        return np.frombuffer(b"".join(parts)[:n], np.uint8).copy()
    return rand_hay(rng, fam.hay_alphabet, n)


def tile_edges(n):
    """Offsets where the prefilter cuts its region: the 1 KiB (stride 1) and 2 KiB (stride 2) tiles, and the
    CTA chunks of each variant's grid (one 16-byte-block share per CTA, acb_prefilter.cu)."""
    edges = set(range(1024, n, 1024))
    for warps, tile, per_sm in ((32, 1024, 1), (32, 2048, 1), (16, 2048, 2)):
        g = min(sm_count() * per_sm, max(1, -(-n // (warps * tile))))
        per_cta = -(-(n >> 4) // g) * 16
        edges |= {c * per_cta for c in range(1, g)}
    return sorted(e for e in edges if 0 < e < n)


def plant_at_edges(hay, fam, edges, rng):
    """Each long pattern (and, for families that have one, its near miss right after it) starting or ending at
    edge + d, d in -1, 0, +1, for as many edges as fit without overlapping.  Returns the plantings."""
    out, busy_to = [], 0
    k = 0
    for e in edges:
        p = fam.long[k % len(fam.long)]
        d = (k % 3) - 1
        at = e + d if (k // 3) % 2 == 0 else e + d - len(p)
        span = len(p) * (2 if fam.near else 1) + 1
        if at < busy_to or at < 0 or at + span > hay.size:
            continue
        hay[at: at + len(p)] = np.frombuffer(p, np.uint8)
        if fam.near:
            hay[at + len(p) + 1: at + 2 * len(p) + 1] = np.frombuffer(near_miss(p), np.uint8)
        out.append((at, len(p)))
        busy_to = at + span
        k += 1
    return out


# ---- the entry points ---------------------------------------------------------------------------------------
def check_single(pats, hay, ctx, plan_want, ci=False, span=None, host=True, kinds=(0, 1, 2), order=True):
    """Overlapping search on Auto and Walk, find_iter of `kinds` on Auto and Sequential, device, pinned and
    pageable input; try_find with and without earliest and is_match; each against the oracle, with the engine
    and plan asserted.  Returns the overlapping oracle list and the order path of the overlapping search."""
    n = hay.size
    s0 = 0 if span is None else span[0]
    keep, ptr = device_copy(hay)
    pin = pinned_copy(hay) if host else None
    ac0 = builder(0, ci).build(pats)
    got_plan = assert_plan(ac0, plan_want, ctx)
    supported = bool(got_plan["supported"])
    want = oracle(pats, 0, ci).find_overlapping_iter_np(hay, span)
    path = None
    for eng in (ab.Engine.Auto, ab.Engine.Walk):
        ac0.set_engine(eng)
        ex = PREFILTER if (supported and eng == ab.Engine.Auto) else WALK
        assert_np_equal(ac0.find_overlapping_iter_dev_np(ptr, n, span)[0], want, (ctx, "overlapping dev", int(eng)))
        assert engine(ac0) == ex, (ctx, int(eng))
        if ex == PREFILTER and order:
            path = assert_order_path(ac0, (span[1] - s0) if span else n, want["end"].astype(np.int64) - s0, 0,
                                     (ctx, "overlapping order"))
        if host:
            for name, x in (("pinned", pin), ("pageable", hay)):
                assert_np_equal(ac0.try_find_overlapping_iter_np(x, span), want, (ctx, "overlapping", name, int(eng)))
                assert engine(ac0) == ex
    ac0.set_engine(ab.Engine.Auto)
    for kind in kinds:
        ac = ac0 if kind == 0 else builder(kind, ci).build(pats)
        w_it = oracle(pats, kind, ci, prefilter=False).find_iter_np(hay, span)
        for eng in (ab.Engine.Auto, ab.Engine.Sequential):
            ac.set_engine(eng)
            ex = PREFILTER if (supported and eng == ab.Engine.Auto) else SEQUENTIAL
            assert_np_equal(ac.find_iter_dev_np(ptr, n, span)[0], w_it, (ctx, "find_iter dev", kind, int(eng)))
            assert engine(ac) == ex, (ctx, kind, int(eng))
            if host:
                for name, x in (("pinned", pin), ("pageable", hay)):
                    assert_np_equal(ac.try_find_iter_np(x, span), w_it, (ctx, "find_iter", name, kind, int(eng)))
        ac.set_engine(ab.Engine.Auto)
        of = oracle(pats, kind, ci)
        for earliest in (False, True):
            m = ac.try_find(hay, span=span, earliest=earliest)
            assert (m.as_tuple() if m else None) == of.try_find(hay, span, earliest=earliest), (ctx, kind, earliest)
            assert engine(ac) == try_find_engine(ac, supported, kind, earliest), (ctx, "try_find", kind, earliest)
        assert ac.is_match(hay, span) == (of.try_find(hay, span) is not None), (ctx, kind)
    return want, path


def try_find_engine(ac, supported, kind, earliest):
    """find_earliest + choose_engine (acb_api.cu): `earliest` on a leftmost automaton runs the sequential engine,
    unless the automaton has the packed prefilter, whose confirmed leftmost match is returned either way."""
    earliest = earliest and not (kind and ac.prefilter_kind() == 4)
    return PREFILTER if supported and not (earliest and kind) else SEQUENTIAL


def doc_records(lists):
    """Per-document oracle lists -> DOC_MATCH_DTYPE records in document order."""
    n = sum(len(x) for x in lists)
    out = np.zeros(n, ab.DOC_MATCH_DTYPE)
    i = 0
    for d, x in enumerate(lists):
        out["doc"][i: i + len(x)] = d
        for k in ("pid", "start", "end"):
            out[k][i: i + len(x)] = x[k]
        i += len(x)
    return out


def same_docs(got, want, ctx):
    assert len(got) == len(want), (len(got), len(want), ctx)
    for k in ("doc", "pid", "start", "end"):
        if not np.array_equal(got[k].astype(np.int64), want[k].astype(np.int64)):
            i = int(np.nonzero(got[k].astype(np.int64) != want[k].astype(np.int64))[0][0])
            raise AssertionError((k, i, got[max(0, i - 2): i + 3], want[max(0, i - 2): i + 3], ctx))


def counts_of(lists, n_pats):
    rows, pids, counts = [0], [], []
    for x in lists:
        c = np.bincount(x["pid"].astype(np.int64), minlength=n_pats)
        nz = np.flatnonzero(c)
        pids += nz.tolist()
        counts += c[nz].tolist()
        rows.append(len(pids))
    return np.array(rows, np.uint64), np.array(pids, np.uint32), np.array(counts, np.uint64)


def check_batches(pats, hay, offs, ctx, plan_want, ci=False, kinds=(0, 1, 2)):
    """Every batched entry point over the documents hay[offs[d]:offs[d + 1]], host and device input, prefilter
    and sequential engines, against the oracle on each document alone.  (Device input under the dry run: the host
    array presented as a device tensor, whose address the library reads as device memory.)"""
    keep, ptr = device_copy(hay)
    docs = [np.ascontiguousarray(hay[offs[d]: offs[d + 1]]) for d in range(offs.size - 1)]
    n_docs = len(docs)
    inputs = [("host", (hay, offs)), ("device", (keep if RUN.on_gpu else _DevView(hay), offs))]
    ac0 = builder(0, ci).build(pats)
    supported = bool(assert_plan(ac0, plan_want, ctx)["supported"])
    o0 = oracle(pats, 0, ci)
    ov = [o0.find_overlapping_iter_np(x) for x in docs]
    want_ov = doc_records(ov)
    for eng in (ab.Engine.Auto, ab.Engine.Sequential):
        ex = PREFILTER if (supported and eng == ab.Engine.Auto) else SEQUENTIAL
        ac0.set_engine(eng)
        for name, inp in inputs:
            same_docs(ac0.find_overlapping_iter_batch_np(inp), want_ov, (ctx, "overlapping batch", name, int(eng)))
            assert engine(ac0) == ex, (ctx, int(eng))
            rows, pids, counts = ac0.pattern_counts_batch_np(inp, overlapping=True)
            w = counts_of(ov, len(pats))
            assert all(np.array_equal(a.astype(np.int64), b.astype(np.int64)) for a, b in zip((rows, pids, counts), w)), \
                (ctx, "overlapping counts", name)
    ac0.set_engine(ab.Engine.Auto)
    if RUN.on_gpu:
        _check_batches_torch(ac0, keep, offs, want_ov, None, None, ov, len(pats), ctx, overlapping=True)
    for kind in kinds:
        ac = ac0 if kind == 0 else builder(kind, ci).build(pats)
        o_it, of = oracle(pats, kind, ci, prefilter=False), oracle(pats, kind, ci)
        it = [o_it.find_iter_np(x) for x in docs]
        want_it = doc_records(it)
        first = [of.try_find(x) for x in docs]
        for eng in (ab.Engine.Auto, ab.Engine.Sequential):
            ex = PREFILTER if (supported and eng == ab.Engine.Auto) else SEQUENTIAL
            ac.set_engine(eng)
            for name, inp in inputs:
                same_docs(ac.find_iter_batch_np(inp), want_it, (ctx, "find_iter batch", kind, name, int(eng)))
                assert engine(ac) == ex, (ctx, kind, int(eng))
                found, rec = ac.find_batch_np(inp)
                got_first = [(int(r["pid"]), int(r["start"]), int(r["end"])) if f else None for f, r in zip(found, rec)]
                assert got_first == first, (ctx, "find_batch", kind, name, int(eng))
                flags = ac.is_match_batch(inp)
                assert flags.tolist() == [f is not None for f in first], (ctx, "is_match_batch", kind, name)
                rows, pids, counts = ac.pattern_counts_batch_np(inp, overlapping=False)
                w = counts_of(it, len(pats))
                assert all(np.array_equal(a.astype(np.int64), b.astype(np.int64)) for a, b in zip((rows, pids, counts), w)), \
                    (ctx, "counts", kind, name)
        ac.set_engine(ab.Engine.Auto)
        if RUN.on_gpu:
            _check_batches_torch(ac, keep, offs, want_it, first, n_docs, it, len(pats), ctx)
    return want_ov


def _check_batches_torch(ac, d, offs, want, first, n_docs, lists, n_pats, ctx, overlapping=False):
    """The _torch device-output forms with device offsets: the same records, first matches, flags and counts."""
    import torch
    from test_gpu_batch_devout import host_records
    d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
    if overlapping:
        bm = ac.find_overlapping_iter_batch_torch((d, d_offs))
    else:
        bm = ac.find_iter_batch_torch((d, d_offs))
        found, rec = ac.find_batch_torch((d, d_offs))
        f, r = found.cpu().numpy(), rec.cpu().numpy()
        got_first = [(int(r[i, 0] & 0xFFFFFFFF), int(r[i, 1]), int(r[i, 2])) if f[i] else None for i in range(n_docs)]
        assert got_first == first, (ctx, "find_batch_torch")
        assert ac.is_match_batch_torch((d, d_offs)).cpu().numpy().tolist() == [x is not None for x in first], ctx
    assert host_records(bm.records).tobytes() == want.tobytes(), (ctx, "batch torch", overlapping)
    csr = ac.pattern_counts_batch_torch((d, d_offs), overlapping=overlapping)
    rows, pids, counts = counts_of(lists, n_pats)
    assert np.array_equal(csr.crow_indices().cpu().numpy(), rows.astype(np.int64)), (ctx, "counts torch")
    assert np.array_equal(csr.col_indices().cpu().numpy(), pids.astype(np.int64)), (ctx, "counts torch")
    assert np.array_equal(csr.values().cpu().numpy(), counts.astype(np.int64)), (ctx, "counts torch")


# ---- the cases ----------------------------------------------------------------------------------------------
# (family, max_pattern_len, expected plan fields); a plan field absent from the dict is not pinned
def plan(brute=0, dense=0, stride=1, bs_n=0, dup_shift=0):
    """The plan fields of a handle with a plan (none of these cases has stride-2 wide tiles)."""
    return dict(supported=1, brute=brute, dense=dense, stride=stride, wide=0, bs_n=bs_n, dup_shift=dup_shift)


FAMILY_CASES = [
    ("ab", 1023, plan(bs_n=2)),              # start bytes a, b: the byte-set scan, then the fingerprint filter
    ("ab", 65533, plan(bs_n=2)),
    ("acgt", 2049, plan(bs_n=3)),
    ("acgt", 65533, plan(bs_n=3)),
    ("bytes", 4096, plan(stride=2)),         # stride-2 fingerprints, 2 KiB tiles
    ("prefix", 4096, plan(brute=1, bs_n=1)),  # a 1-byte pattern: k = 1
    ("suffix", 65533, plan(brute=1)),
    ("periodic", 4096, plan(bs_n=2)),
    ("mixed", 5000, plan(dense=1)),          # more than 8 192 fingerprints: the dense plan
]


def family_case_id(c):
    return "%s-%d" % (c[0], c[1])


def run_family_case(fam_name, L, plan_want, ci=False):
    fam = FAMILIES[fam_name](L, 0xF00 + L)
    assert max(len(p) for p in fam.pats) == L
    hay = base_haystack(fam, max(size("hay"), 6 * L + 8192), L)
    plants = plant_at_edges(hay, fam, tile_edges(hay.size), np.random.default_rng(L))
    assert len(plants) >= 2, plants
    pats = fam.pats
    if ci:
        W.flip_case(hay, L)
    ctx = (fam_name, L, ci)
    want, path = check_single(pats, hay, ctx, plan_want, ci=ci)
    lens = np.array([len(p) for p in pats])
    assert (lens[want["pid"]] == L).sum() >= len(plants) // 2, ctx   # the long matches are there
    # a sub-span that begins inside a planted long match and ends inside another
    a, b = plants[0][0] + 1, plants[-1][0] + plants[-1][1] - 1
    if b > a:
        check_single(pats, hay, ctx + ("span",), plan_want, ci=ci, span=(a, b), host=False, kinds=(1,))
    # (filler for the periodic and mixed sets: bytes that cannot extend a periodic match)
    check_document_forms(pats, pats.index(fam.long[0]), fam.hay_alphabet or b"xyz", ctx, plan_want, ci=ci)
    return path


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", FAMILY_CASES, ids=[family_case_id(c) for c in FAMILY_CASES])
def test_long_pattern_families(case):
    """Families a-e with long matches and near misses planted across tile and CTA-chunk edges: every
    single-haystack entry point, both engines, device, pinned and pageable input; every batched entry point over
    documents built around the long pattern."""
    t = time.time()
    path = run_family_case(*case)
    print("family %s: order path %s, %.1f s" % (family_case_id(case), path, time.time() - t))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_long_patterns_case_insensitive():
    """The mixed family with ASCII case folded in haystack and automaton."""
    run_family_case("mixed", 4096, plan(dense=1, dup_shift=1), ci=True)   # case folding makes duplicates


# The boundary table: (id, max_pattern_len, copies of a short pattern, expected plan, expected order path of the
# overlapping search on the device).  "buckets22": buckets of 4 MiB, the in-bucket key uses all 32 bits.
def boundary_pats(L, dups):
    rng = np.random.default_rng(L + dups)
    p = rand_bytes(rng, b"acgt", L)
    return [p, p[: L // 2], p[-(L // 3):], p[L // 4: L // 4 + 16]] + [b"acgtacgtac"] * dups


BOUNDARIES = [
    ("len1023", 1023, 1, plan(bs_n=3), 10),
    ("len1024", 1024, 1, plan(), 11),
    ("len2049", 2049, 1, plan(bs_n=2), 12),
    ("len4096", 4096, 1, plan(bs_n=3), 13),
    ("len65533", 65533, 1, plan(bs_n=3), 16),
    ("len65534", 65534, 1, dict(supported=0), None),
    ("len65533-dup256", 65533, 256, plan(bs_n=3, dup_shift=8), 24),
    ("len65533-dup257", 65533, 257, dict(supported=0, dup_shift=9), None),
]


def run_boundary(row):
    name, L, dups, plan_want, tie = row
    pats = boundary_pats(L, dups)
    ac = builder(0).build(pats)
    assert ac.max_pattern_len() == L
    p = plan_of(ac)
    assert p.supported == plan_want["supported"], (name, p.supported)
    if tie is not None:
        assert L.bit_length() + p.dup_shift == tie
    hay_bytes = max(size("hay"), 6 * L + 8192)
    bp = bucket_plan(ac, hay_bytes)
    if RUN.on_gpu and tie is not None:
        # the device's plan_buckets: 10 tie bits still give buckets (shift 22), 11 and more the single list
        assert (bp[0] if bp else None) == (22 if tie == 10 else None), (name, bp)
    fam = SimpleNamespace(pats=pats, long=[pats[0]], hay_alphabet=b"acgt", near=True)
    hay = base_haystack(fam, hay_bytes, L)
    plants = plant_at_edges(hay, fam, tile_edges(hay.size), np.random.default_rng(L))
    assert plants
    want, path = check_single(pats, hay, name, plan_want)
    if tie is not None:
        assert path == ("single" if bp is None else "buckets"), (name, path, bp)
    check_document_forms(pats, 0, b"acgt", (name,), plan_want, kinds=(0, 1))
    return path


def document_batch(p, alphabet, seed, reps=2):
    """(haystack, offsets, forms): documents built around the long pattern p, each of one form:
      exact       p alone;
      at_end      filler + p: the match ends exactly at the document end;
      one_past    filler + p[:-1], and the next document (next) begins with p's last byte: the match would end
                  one byte past the document end;
      plus_before one byte + p (the pattern + 1 byte, ending at the end);
      plus_after  p + one byte;
      shorter     p[:-1] and p[1:], one byte shorter than the pattern;
      near        p with its last byte changed;
      short       a few bytes of filler."""
    rng = np.random.default_rng(seed)

    def filler(n):
        return rand_bytes(rng, alphabet, n)
    docs = []
    for r in range(reps):
        k = 1 + 29 * r
        docs += [("exact", p), ("at_end", filler(k + 36) + p), ("one_past", filler(k + 22) + p[:-1]),
                 ("next", p[-1:] + filler(k + 40)), ("plus_before", filler(1) + p), ("plus_after", p + filler(1)),
                 ("shorter", p[:-1]), ("shorter", p[1:]), ("near", near_miss(p)), ("short", filler(k + 6))]
    forms = [f for f, _ in docs]
    lens = np.array([len(x) for _, x in docs], np.int64)
    offs = np.zeros(len(docs) + 1, np.int64)
    offs[1:] = np.cumsum(lens)
    hay = np.frombuffer(b"".join(x for _, x in docs), np.uint8).copy()
    return hay, offs, forms


def assert_doc_forms(pats, hay, offs, forms, long_pid, ci=False):
    """Each form holds its long match where it should, by the oracle over the whole batch: at the document end
    (exact, at_end, plus_before), one byte before it (plus_after), one byte past it (one_past), nowhere inside
    (one_past, shorter, near)."""
    L = len(pats[long_pid])
    whole = oracle(pats, 0, ci).find_overlapping_iter_np(hay)
    longs = whole[whole["pid"] == long_pid]
    ends = set(longs["end"].astype(np.int64).tolist())
    for d, f in enumerate(forms):
        a, b = int(offs[d]), int(offs[d + 1])
        inside = any(a <= e - L and e <= b for e in ends)
        if f in ("exact", "at_end", "plus_before"):
            assert b in ends and b - L >= a, (f, d)
        elif f == "plus_after":
            assert b - 1 in ends and b - 1 - L >= a, (f, d)
        elif f == "one_past":
            assert b + 1 in ends and not inside, (f, d)
        elif f in ("shorter", "near"):
            assert not inside, (f, d)
    assert {"exact", "at_end", "one_past", "plus_before", "plus_after", "shorter", "near"} <= set(forms)


def check_document_forms(pats, long_pid, alphabet, ctx, plan_want, ci=False, kinds=(0, 1, 2)):
    hay, offs, forms = document_batch(pats[long_pid], alphabet, len(pats[long_pid]))
    if ci:
        W.flip_case(hay, 5)
    assert_doc_forms(pats, hay, offs, forms, long_pid, ci)
    check_batches(pats, hay, offs, ctx + ("documents",), plan_want, ci=ci, kinds=kinds)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("row", BOUNDARIES, ids=[r[0] for r in BOUNDARIES])
def test_length_and_tie_boundaries(row):
    """Each row of the plan and tie-break limits: the plan (or its absence), the engine and the order path,
    and every single-haystack and batched entry point against the oracle."""
    t = time.time()
    path = run_boundary(row)
    print("boundary %s: order path %s, %.1f s" % (row[0], path, time.time() - t))


# ---- placements ---------------------------------------------------------------------------------------------
def walk_seg_len(n_bytes):
    """run_walk_overlapping: max(ceil(n / (SMs * 2048)), 256) bytes per lane, rounded up to 16."""
    lanes = sm_count() * 2048
    seg = max(-(-n_bytes // lanes), 256)
    return (seg + 15) & ~15


def run_walk_shards(L):
    """Long matches around walk shard edges (a lane owns the ends in (g0, g1]): ending at g0, g0 + 1, g1 - 1 and g1
    of shards more than L bytes past the span start, and a shorter piece ending at g0 + 1 of a shard whose cold
    start is clamped at the span start; a span that is exactly one pattern long."""
    fam = FAMILIES["acgt"](L, 0x3A1 + L)
    p, piece = fam.pats[0], fam.pats[2]   # the pattern and its last third
    hay = base_haystack(fam, max(size("walk"), 6 * L), L + 5)
    ac = builder(0).build(fam.pats)
    ac.set_engine(ab.Engine.Walk)
    o = oracle(fam.pats)
    s0 = 37   # span start
    seg = walk_seg_len(hay.size - s0)
    assert seg < L
    far = L // seg + 3   # shards apart, so that one planting does not cover the next
    planted = []
    for i, d in enumerate((0, 1, -1, 0)):
        e = s0 + (i + 2) * far * seg + d
        hay[e - L: e] = np.frombuffer(p, np.uint8)
        planted.append((e, L))
    k = len(piece) // seg + 1   # clamped: g0 - s0 < L - 1
    e = s0 + k * seg + 1
    assert k * seg < L - 1 and e - len(piece) >= s0
    hay[e - len(piece): e] = np.frombuffer(piece, np.uint8)
    planted.append((e, len(piece)))
    keep, ptr = device_copy(hay)
    t_walk = []
    for span in ((s0, hay.size), (0, hay.size), (planted[1][0] - L, planted[1][0])):
        want = o.find_overlapping_iter_np(hay, span)
        t = time.time()
        got = ac.find_overlapping_iter_dev_np(ptr, hay.size, span)[0]
        t_walk.append(time.time() - t)
        assert engine(ac) == WALK
        assert_np_equal(got, want, ("walk shards", L, span))
        have = set(zip(want["end"].tolist(), (want["end"] - want["start"]).tolist()))
        assert {(e, n) for e, n in planted if e - n >= span[0] and e <= span[1]} <= have, span
    return t_walk


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("L", [1023, 65533])
def test_walk_shards_cold_start(L):
    """The walk engine with lanes whose max_len - 1 byte back-read spans hundreds of shards (timed: the cold
    start is about L dependent loads per lane)."""
    t = run_walk_shards(L)
    print("walk L=%d: %s s per search (%d-byte shards)" % (L, ["%.3f" % x for x in t], walk_seg_len(size("walk"))))


def run_pipelined(L, chunks):
    """Host haystacks copied chunk by chunk with chunks shorter than the tail a chunk's scan waits for
    (max_len + 64 bytes): whole chunks land before any of their start offsets may be scanned.  A long match
    across every chunk edge, at offsets -1, 0, +1; pinned and pageable (the staged ring) input."""
    fam = FAMILIES["ab"](L, 0x919 + L)
    p = fam.pats[0]
    hay = base_haystack(fam, size("pipe"), L + 9)
    step = L + 2
    for k, at in enumerate(range(3000, hay.size - L, step)):
        at += (k % 3) - 1
        hay[at: at + L] = np.frombuffer(p, np.uint8)
    pin = pinned_copy(hay)
    o0, o1 = oracle(fam.pats), oracle(fam.pats, 1, prefilter=False)
    w0, w1 = o0.find_overlapping_iter_np(hay), None
    ac0, ac1 = builder(0).build(fam.pats), builder(1).build(fam.pats)
    w1 = o1.find_iter_np(hay)
    span = (4095, hay.size - 4097)
    w0s = o0.find_overlapping_iter_np(hay, span)
    for chunk in chunks:
        assert chunk < L + 64   # the tail of run_prefilter's pipelined path is longer than a chunk
        for ac in (ac0, ac1):
            assert ab._lib.acg_debug_set_pipeline_chunk(ac._h, chunk) == 0
        for name, x in (("pinned", pin), ("pageable", hay)):
            assert_np_equal(ac0.try_find_overlapping_iter_np(x), w0, ("pipelined overlapping", L, chunk, name))
            assert engine(ac0) == PREFILTER
            assert_np_equal(ac0.try_find_overlapping_iter_np(x, span), w0s, ("pipelined span", L, chunk, name))
            assert_np_equal(ac1.try_find_iter_np(x), w1, ("pipelined find_iter", L, chunk, name))
            assert engine(ac1) == PREFILTER
    assert (w0["end"] - w0["start"] == L).sum() > 4


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("L", [4097, 65533])
def test_pipelined_chunks_shorter_than_the_tail(L):
    run_pipelined(L, [4096, 65536] if L > 65536 - 64 else [4096])


FIND_EDGES = (1 << 20, 17 << 20)   # acg_find's window edges: 1 MiB, then 16 MiB more


def run_find_windows(L):
    """try_find / is_match from offset 0 on a host haystack: a long match that starts at edge - 1 and one that ends
    at edge + 1, for both window edges.  A 64-byte piece of the long pattern starts 2 bytes into it: under
    Standard that short match ends first, and when the long one starts at edge - 1 the short one starts in
    [hi, end), which only the second scan of those starts finds."""
    rng = np.random.default_rng(L)
    p = rand_bytes(rng, b"acgt", L)
    pats = [p, p[2:66]]
    hay = np.zeros(FIND_EDGES[1] + 2 * L + 4096, np.uint8)
    handles = {kind: builder(kind).build(pats) for kind in (0, 1, 2)}
    oracles = {kind: oracle(pats, kind) for kind in (0, 1, 2)}
    for e in FIND_EDGES:
        for what, at in (("start", e - 1), ("end", e + 1 - L)):
            hay[at: at + L] = np.frombuffer(p, np.uint8)
            for kind, ac in handles.items():
                want = oracles[kind].try_find(hay)
                assert want == ((1, at + 2, at + 66) if kind == 0 else (0, at, at + L)), (what, e, kind, want)
                for earliest in (False, True):
                    w = oracles[kind].try_find(hay, earliest=earliest)
                    m = ac.try_find(hay, earliest=earliest)
                    assert (m.as_tuple() if m else None) == w, (what, e, kind, earliest, m, w)
                    assert engine(ac) == try_find_engine(ac, True, kind, earliest)
                assert ac.is_match(hay)
                assert not ac.is_match(hay, span=(0, at + 65))
            hay[at: at + L] = 0


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("L", [4096, 65533])
def test_find_windows(L):
    run_find_windows(L)


def run_order_buckets():
    """max_len 1 023 (10 tie bits): long matches that cross bucket edges, keyed by end (overlapping) and by start
    (leftmost find_iter): at bucket edge E, one ends at E + d and one starts at E + d (d = -1, 0, +1 from edge to
    edge).  The order step in shared memory runs, not its fallback."""
    L = 1023
    rng = np.random.default_rng(77)
    p = rand_bytes(rng, b"acgt", L)
    pats = [p, p[100:140], p[-24:]]
    fam = SimpleNamespace(pats=pats, long=[p], hay_alphabet=b"acgt", near=False)
    hay = base_haystack(fam, size("bucket"), 5)
    ac0 = builder(0).build(pats)
    bp = bucket_plan(ac0, hay.size)
    assert bp is not None
    shift = bp[0]
    if RUN.on_gpu:
        assert shift == 22
    B = 1 << shift
    n_edges = (hay.size - L) // B
    assert n_edges >= 3
    pb = np.frombuffer(p, np.uint8)
    for b in range(1, n_edges + 1):
        e = b * B + (b % 3) - 1
        hay[e - L: e] = pb   # ends at the edge + d
        hay[e: e + L] = pb   # starts there
    keep, ptr = device_copy(hay)
    want = oracle(pats).find_overlapping_iter_np(hay)
    assert_np_equal(ac0.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, "order buckets overlapping")
    assert engine(ac0) == PREFILTER
    assert assert_order_path(ac0, hay.size, want["end"].astype(np.int64), 0, "by end") == "buckets"
    st, en = want["start"].astype(np.int64), want["end"].astype(np.int64)
    # one long match across each edge with d != 0: ending at E + 1, or starting at E - 1
    assert ((st >> shift) != ((en - 1) >> shift)).sum() >= sum(b % 3 != 1 for b in range(1, n_edges + 1))
    for kind in (1, 2):
        ac = builder(kind).build(pats)
        w = oracle(pats, kind, prefilter=False).find_iter_np(hay)
        assert_np_equal(ac.find_iter_dev_np(ptr, hay.size)[0], w, ("order buckets", kind))
        assert engine(ac) == PREFILTER
        assert assert_order_path(ac, hay.size, np.unique(st), CHAIN, ("by start", kind)) == "buckets"


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_order_buckets_with_long_patterns():
    run_order_buckets()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("fam_name,L", [("ab", 4096), ("ab", 65533), ("prefix", 4096), ("suffix", 65533)])
def test_device_fill_long_patterns(fam_name, L):
    """acg_build_on_device (one dfa_fill_level_kernel launch per trie level, up to 65 533 of them): tables
    bit-identical to the host builder's, and the oracle's results from them."""
    fam = FAMILIES[fam_name](L, 0xF111 + L)
    host = builder(0).host_only(True).build(fam.pats)
    t = time.time()
    dev = builder(0).device_fill(True).build(fam.pats)
    t_fill = time.time() - t
    th, td = host.tables(), dev.tables()
    for k in th:
        if isinstance(th[k], np.ndarray):
            assert np.array_equal(th[k], td[k]), (fam_name, L, k)
        else:
            assert th[k] == td[k], (fam_name, L, k)
    hay = base_haystack(fam, size("hay") // 4, 3)
    plant_at_edges(hay, fam, tile_edges(hay.size), None)
    keep, ptr = device_copy(hay)
    want = oracle(fam.pats).find_overlapping_iter_np(hay)
    assert_np_equal(dev.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, (fam_name, L, "device fill"))
    assert engine(dev) == PREFILTER
    dev.set_engine(ab.Engine.Walk)
    assert_np_equal(dev.find_overlapping_iter_dev_np(ptr, hay.size)[0], want, (fam_name, L, "device fill, walk"))
    print("device fill %s L=%d: %.2f s" % (fam_name, L, t_fill))
