"""Batched search on the H100 (acg_find_iter_batch / acg_find_overlapping_batch / acg_is_match_batch):
device-resident batches of 64-256 MiB cut into log-uniform documents, every prefilter kernel variant and
the per-document sequential kernel, against the oracle on sampled documents and against the
single-haystack call; and the full-size docs workload of tools/bench_docs.py (cfg 2's automaton and 4 GiB haystack)."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W

pytestmark = pytest.mark.gpu

# name -> (patterns, seed, MiB, match kind, case-insensitive): the prefilter variants of
# tests/test_emulated_kernels.py (stride-2 narrow, case-insensitive leftmost, wide, stride 1, dense)
VARIANTS = {
    "stride2_narrow": (5000, 0xAC5000, 256, 0, False),
    "stride2_narrow_ci_leftmost": (5000, 0xAC5000, 128, 1, True),
    "stride2_wide": (50, 0xAC0050, 128, 1, False),
    "stride1_short_patterns": (300, 31, 64, 2, False),
    "dense": (20000, 0xAC1000, 64, 0, False),
}


def batch_workload(n, seed, mib, ci, short=False):
    import torch
    pats = W.make_patterns(n, seed)
    if short:
        pats = [p[:3] for p in pats[:150]] + pats[150:]
    hay = np.empty(mib << 20, dtype=np.uint8)
    W.fill_haystack(hay, 5)
    W.plant(hay, pats, 6, period=1024, window=512)
    offs = W.doc_offsets(hay.size, seed & 0xFFFF)
    rng = np.random.default_rng(seed)
    for i, b in enumerate(offs[1:-1:7]):   # across, ending at and starting at document boundaries
        p = np.frombuffer(pats[int(rng.integers(len(pats)))], dtype=np.uint8)
        at = (b - len(p) // 2, b - len(p), b)[i % 3]
        if at >= 0 and at + len(p) <= hay.size:
            hay[at:at + len(p)] = p
    if ci:
        W.flip_case(hay, 7)
    return pats, hay, offs, torch.from_numpy(hay).cuda()


def build(pats, kind=0, ci=False):
    return ab.AhoCorasick.builder().match_kind(kind).ascii_case_insensitive(ci).kind(ab.AhoCorasickKind.DFA).build(pats)


def same(a, b, ctx):
    assert len(a) == len(b), (len(a), len(b), ctx)
    for k in ("doc", "pid", "start", "end"):
        assert np.array_equal(a[k], b[k]), (k, ctx)


def sampled_docs_match_the_oracle(got, o, hay, offs, what, n=200, seed=0):
    rng = np.random.default_rng(seed)
    docs = np.unique(rng.integers(0, offs.size - 1, size=n))
    lo = np.searchsorted(got["doc"], docs, side="left")
    hi = np.searchsorted(got["doc"], docs, side="right")
    fn = o.find_overlapping_iter_np if what == "overlapping" else o.find_iter_np
    for d, a, b in zip(docs, lo, hi):
        want = fn(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]))
        part = got[a:b]
        assert len(part) == len(want), (what, d)
        for k in ("pid", "start", "end"):
            assert np.array_equal(part[k], want[k]), (what, d, k)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_batch_variants(name):
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    dev = (d_hay, offs)
    whats = ["iter", "overlapping"] if kind == 0 else ["iter"]
    for what in whats:
        fn = ac.find_overlapping_iter_batch_np if what == "overlapping" else ac.find_iter_batch_np
        got = fn(dev)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        assert len(got) > 1000 and np.all(np.diff(got["doc"].astype(np.int64)) >= 0)
        sampled_docs_match_the_oracle(got, o, hay, offs, what)
        same(fn((hay, offs)), got, (name, what, "host haystack"))
        ac.set_engine(ab.Engine.Sequential)
        same(fn(dev), got, (name, what, "sequential"))
        ac.set_engine(ab.Engine.Auto)
    flags = ac.is_match_batch(dev)
    want = np.zeros(offs.size - 1, bool)
    want[ac.find_iter_batch_np(dev)["doc"]] = True
    assert np.array_equal(flags, want)
    ac.set_engine(ab.Engine.Sequential)
    assert np.array_equal(ac.is_match_batch(dev), want)


def test_anchored_and_empty_pattern_batches():
    import torch
    rng = np.random.default_rng(3)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=4 << 20)), dtype=np.uint8).copy()
    offs = W.doc_offsets(hay.size, 4, lo=1, hi=256)
    d_hay = torch.from_numpy(hay).cuda()
    pats = [b"ab", b"abc", b"b", b"ca", b"cab"]
    for kind in (0, 1, 2):
        ac = ab.AhoCorasick.builder().match_kind(kind).start_kind(ab.StartKind.Both).build(pats)
        o = O.Oracle(pats, match_kind=kind, start_kind=int(ab.StartKind.Both))
        got = ac.find_iter_batch_np((d_hay, offs), anchored=ab.Anchored.Yes)
        docs = np.random.default_rng(kind).integers(0, offs.size - 1, size=300)
        for d in docs:
            part = got[got["doc"] == d]
            want = o.find_iter_np(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]), anchored=True)
            assert len(part) == len(want) and np.array_equal(part["start"], want["start"]), (kind, d)
        e = ab.AhoCorasick.builder().match_kind(kind).build(pats + [b""])
        oe = O.Oracle(pats + [b""], match_kind=kind)
        got = e.find_iter_batch_np((d_hay, offs))
        for d in docs[:100]:
            part = got[got["doc"] == d]
            want = oe.find_iter_np(np.ascontiguousarray(hay[offs[d]:offs[d + 1]]))
            assert len(part) == len(want) and np.array_equal(part["end"], want["end"]), (kind, d)


def test_full_size_docs_workload():
    """tools/bench_docs.py's workload: cfg 2's automaton and 4 GiB haystack cut into ~1.8 M documents.  The
    batch list, mapped back to global offsets, is cfg 2's single-haystack list minus the matches that
    straddle a document boundary; the prefilter and per-document sequential engines agree."""
    import torch
    n = 4 << 30
    pats = W.config_patterns("cfg2")
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg2", d_hay, pats)
    offs = W.doc_offsets(n, 0xD0C5)
    assert 1_600_000 < offs.size < 2_000_000
    ac = build(pats)
    single, _ = ac.find_overlapping_iter_dev_np(d_hay.data_ptr(), n)
    got = ac.find_overlapping_iter_batch_np((d_hay, offs))
    doc = np.searchsorted(offs, single["start"].astype(np.int64), side="right") - 1
    keep = single["end"].astype(np.int64) <= offs[doc + 1]
    assert (~keep).sum() > 100
    want = single[keep]
    assert len(got) == len(want)
    base = offs[got["doc"].astype(np.int64)].astype(np.uint64)
    assert np.array_equal(got["pid"], want["pid"])
    assert np.array_equal(got["start"] + base, want["start"])
    assert np.array_equal(got["end"] + base, want["end"])
    ac.set_engine(ab.Engine.Sequential)
    same(ac.find_overlapping_iter_batch_np((d_hay, offs)), got, "sequential engine, overlapping")
    ac.set_engine(ab.Engine.Auto)
    # sampled documents against the oracle, on their own bytes
    o = O.Oracle(pats, kind=O.KIND_DFA)
    rng = np.random.default_rng(1)
    for d in rng.integers(0, offs.size - 1, size=200):
        part = got[got["doc"] == d]
        doc_bytes = d_hay[int(offs[d]):int(offs[d + 1])].cpu().numpy()
        want_d = o.find_overlapping_iter_np(doc_bytes)
        assert len(part) == len(want_d) and np.array_equal(part["end"], want_d["end"]), d
    del d_hay
    torch.cuda.empty_cache()
