"""Match coverage per document on the H100 (acg_match_coverage_batch / _devout and the torch form).

Every result is compared with a torch computation, on the device, from the same handle's *_batch_torch records
(sorted by start, torch.cummax of the ends, scatter_add of each match's uncovered part per document; the mask
from index_add of +1 / -1 at the starts and ends, a cumsum and > 0, one window of the haystack at a time) and
with the oracle on sampled documents.  Host output, the raw device-output call and the torch form must agree.
Covered: the prefilter kernel variants of tests/test_gpu_batch.py on both engines, and the full-size shapes --
cfg 2's 1.8 M documents (overlapping) and cfg 3's (find_iter) in 4 GiB with the mask, cfg 5's 100 000 patterns
over 2 GiB, one 4 GiB document, a batch whose span and mask run past 2^32, and 4 KiB and 64 KiB patterns at
document edges."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu

WINDOW = 512 << 20  # bytes of the mask the torch reference builds at a time


def torch_coverage(ac, d_hay, offs, overlapping, anchored=ab.Anchored.No):
    """(covered int64 [n_docs], starts, ends): the union of the batch records with torch on the device."""
    import torch
    r = ac.find_overlapping_iter_batch_torch((d_hay, offs)) if overlapping else \
        ac.find_iter_batch_torch((d_hay, offs), anchored=anchored)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(d_hay.device)
    s, order = torch.sort(d_offs[r.doc] + r.start)
    e, doc = (d_offs[r.doc] + r.end)[order], r.doc[order]
    m = torch.cummax(e, 0).values
    prev = torch.cat([torch.zeros(1, dtype=m.dtype, device=m.device), m[:-1]])
    part = (e - torch.maximum(s, prev)).clamp_(min=0)
    covered = torch.zeros(offs.size - 1, dtype=torch.int64, device=d_hay.device).scatter_add_(0, doc, part)
    return covered, s, e


def mask_matches(mask, s, e, lo, hi):
    """mask (CUDA bool, indexed like the haystack) over [lo, hi) equals the union of [s, e), window by window."""
    import torch
    for w0 in range(lo, hi, WINDOW):
        w1 = min(hi, w0 + WINDOW)
        keep = (s < w1) & (e > w0) & (e > s)
        d = torch.zeros(w1 - w0 + 1, dtype=torch.int32, device=mask.device)
        one = torch.ones(int(keep.sum()), dtype=torch.int32, device=mask.device)
        d.index_add_(0, s[keep].clamp(min=w0) - w0, one)
        d.index_add_(0, e[keep].clamp(max=w1) - w0, -one)
        if not torch.equal(mask[w0:w1], torch.cumsum(d[:-1], 0, dtype=torch.int32) > 0):
            return False
    return True


def check(ac, d_hay, offs, overlapping, o, ctx, n_sample=100, anchored=ab.Anchored.No, min_covered=1, host=True):
    """The torch form (with the mask) against the records' union and the oracle; the raw device-output call and
    (host) the host-output call against the torch form.  Returns covered as a numpy array."""
    import torch
    covered, mask = ac.match_coverage_batch_torch((d_hay, offs), overlapping=overlapping, anchored=anchored)
    assert covered.dtype == torch.int64 and mask.dtype == torch.bool and mask.numel() == d_hay.numel()
    want, s, e = torch_coverage(ac, d_hay, offs, overlapping, anchored)
    assert torch.equal(covered, want), ctx
    lo, hi = int(offs[0]), int(offs[-1])
    assert mask_matches(mask, s, e, lo, hi), (ctx, "mask")
    assert not mask[:lo].any() and not mask[hi:].any(), (ctx, "mask outside the documents")
    del s, e
    got = covered.cpu().numpy()
    assert int(got.sum()) >= min_covered, (ctx, int(got.sum()))
    fn = o.find_overlapping_iter_np if overlapping else o.find_iter_np
    for d in np.random.default_rng(offs.size).integers(0, offs.size - 1, size=n_sample):
        a, b = int(offs[d]), int(offs[d + 1])
        r = fn(d_hay[a:b].cpu().numpy(), anchored=bool(anchored))
        m = np.zeros(b - a, bool)
        for x, y in zip(r["start"].tolist(), r["end"].tolist()):
            m[x:y] = True
        assert got[d] == m.sum() and np.array_equal(mask[a:b].cpu().numpy(), m), (ctx, int(d))
    # the raw device-output call with device offsets, into a mask with sentinels around [lo, hi)
    d_cov = torch.full((offs.size - 1,), -1, dtype=torch.int64, device=d_hay.device)
    d_mask = torch.full((d_hay.numel(),), 7, dtype=torch.uint8, device=d_hay.device)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(d_hay.device)
    torch.cuda.synchronize()  # the sentinels are written before the library's stream reads or writes the arrays
    ac.match_coverage_batch_devout(d_hay.data_ptr(), d_hay.numel(), d_offs.data_ptr(), d_cov.data_ptr(),
                                   d_mask.data_ptr(), overlapping=overlapping, anchored=anchored,
                                   n_docs=offs.size - 1)
    assert torch.equal(d_cov, covered) and torch.equal(d_mask[lo:hi], mask[lo:hi].to(torch.uint8)), (ctx, "devout")
    assert (d_mask[:lo] == 7).all() and (d_mask[hi:] == 7).all(), (ctx, "devout sentinels")
    del d_mask, mask
    if host:
        h_cov, h_mask = ac.match_coverage_batch_np((d_hay, offs), overlapping=overlapping, anchored=anchored,
                                                   mask=True)
        assert np.array_equal(h_cov.astype(np.int64), got), (ctx, "host")
        h = torch.from_numpy(h_mask).to(d_hay.device)
        d_mask2 = ac.match_coverage_batch_torch((d_hay, offs), overlapping=overlapping, anchored=anchored)[1]
        assert torch.equal(h, d_mask2), (ctx, "host mask")
    return got


@pytest.mark.parametrize("name", list(VARIANTS))
def test_coverage_variants(name):
    """Every prefilter variant and then the sequential engine: the union of the records, and equal engines."""
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    for ov in ((False, True) if kind == 0 else (False,)):
        want = check(ac, d_hay, offs, ov, o, (name, ov), min_covered=10_000)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        ac.set_engine(ab.Engine.Sequential)
        got = ac.match_coverage_batch_np((d_hay, offs), overlapping=ov)
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        assert np.array_equal(got.astype(np.int64), want), (name, ov, "sequential")
        ac.set_engine(ab.Engine.Auto)


def test_anchored_batches_on_the_sequential_engine():
    import torch
    rng = np.random.default_rng(3)
    hay = np.frombuffer(bytes(rng.choice(list(b"abc"), size=4 << 20)), dtype=np.uint8).copy()
    offs = W.doc_offsets(hay.size, 4, lo=1, hi=256)
    d_hay = torch.from_numpy(hay).cuda()
    pats = [b"ab", b"abc", b"b", b"ca", b"cab", b"ab"]
    for kind in (0, 1, 2):
        ac = ab.AhoCorasick.builder().match_kind(kind).start_kind(ab.StartKind.Both).build(pats)
        o = O.Oracle(pats, match_kind=kind, start_kind=int(ab.StartKind.Both))
        check(ac, d_hay, offs, False, o, kind, anchored=ab.Anchored.Yes, min_covered=10_000)
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)


def _config_batch(name, n):
    import torch
    pats = W.config_patterns(name)
    b = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA)
    if name == "cfg3":
        b.ascii_case_insensitive(True).match_kind(ab.MatchKind.LeftmostFirst)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config(name, d_hay, pats)
    return pats, b.build(pats), d_hay


@pytest.mark.parametrize("name", ["cfg2", "cfg3"])
def test_full_size_docs_workload(name):
    """tools/bench_docs.py's documents: 4 GiB cut into ~1.8 M, with the mask; cfg 2 covers with
    find_overlapping_iter, cfg 3 with find_iter (leftmost-first, case-insensitive)."""
    import torch
    n = 4 << 30
    pats, ac, d_hay = _config_batch(name, n)
    offs = W.doc_offsets(n, 0xD0C5)
    assert 1_600_000 < offs.size < 2_000_000
    o = O.Oracle(pats, match_kind=int(ac.match_kind()), ascii_case_insensitive=name == "cfg3", kind=O.KIND_DFA)
    check(ac, d_hay, offs, name == "cfg2", o, name, n_sample=60, min_covered=1_000_000)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    del d_hay
    torch.cuda.empty_cache()


def test_full_size_cfg5():
    """cfg 5's 100 000 patterns over 2 GiB cut into documents."""
    import torch
    n = 2 << 30
    pats, ac, d_hay = _config_batch("cfg5", n)
    assert ac.patterns_len() == 100_000
    offs = W.doc_offsets(n, 0xC5)
    check(ac, d_hay, offs, True, O.Oracle(pats, kind=O.KIND_DFA), "cfg5", n_sample=30, min_covered=100_000,
          host=False)
    del d_hay
    torch.cuda.empty_cache()


def test_one_4_gib_document_and_a_batch_past_4_gib():
    """One 4 GiB document: covered is the union of the single-haystack find_overlapping_iter records.  Then a
    batch of documents whose span starts before and ends past 2^32, with mask entries past 2^32."""
    import torch
    n = (4 << 30) + (192 << 20)
    pats, ac, d_hay = _config_batch("cfg2", n)
    whole = 4 << 30
    single, _ = ac.find_overlapping_iter_dev_np(d_hay.data_ptr(), whole)
    assert len(single) > 500_000
    s = single["start"].astype(np.int64)
    order = np.argsort(s, kind="stable")
    s, e = s[order], single["end"].astype(np.int64)[order]
    prev = np.r_[0, np.maximum.accumulate(e)[:-1]]
    want = int(np.clip(e - np.maximum(s, prev), 0, None).sum())
    covered, _ = ac.match_coverage_batch_torch((d_hay, np.array([0, whole])), overlapping=True, mask=False)
    assert covered.tolist() == [want]
    assert ac.match_coverage_batch_np((d_hay, np.array([0, whole])), overlapping=True).tolist() == [want]
    # documents from 2^32 - 160 MiB to the end of the buffer, past 2^32
    offs = (whole - (160 << 20)) + W.doc_offsets(n - whole + (160 << 20), 0x4AB)
    assert offs[0] < 1 << 32 < offs[-1] == n
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for ov in (True, False):
        check(ac, d_hay, offs, ov, o, ("past 4 GiB", ov), n_sample=60, min_covered=100_000)
        _, mask = ac.match_coverage_batch_torch((d_hay, offs), overlapping=ov)
        assert mask[1 << 32:].any() and mask[: 1 << 32].any()
        del mask
    del d_hay
    torch.cuda.empty_cache()


@pytest.mark.parametrize("plen", [4096, 65536])
def test_long_patterns_at_document_edges(plen):
    """A 4 KiB or 64 KiB pattern, and a copy shifted by 3 bytes, planted across, at the end of and at the start
    of documents: each document's coverage is its planted bytes, on both engines."""
    import torch
    rng = np.random.default_rng(plen)
    base = rng.integers(97, 123, size=plen + 3, dtype=np.uint8)
    pats = [base[:plen].tobytes(), base[3:plen + 3].tobytes(), b"zzzq"]
    n = 64 * (plen + 512)
    hay = np.full(n, ord("."), np.uint8)
    offs, at = [0], 0
    while at + 2 * plen + 64 < n:
        doc = int(rng.integers(plen + 8, 2 * plen))
        where = (0, doc - plen - 3, (doc - plen - 3) // 2)[len(offs) % 3]  # start, end, middle
        hay[at + where:at + where + plen + 3] = base
        offs.append(at + doc)
        at += doc
    offs.append(n)
    offs = np.array(offs, np.int64)
    d_hay = torch.from_numpy(hay).cuda()
    for kind in (0, 1):
        ac = build(pats, kind)
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        for ov in ((False, True) if kind == 0 else (False,)):
            got = check(ac, d_hay, offs, ov, o, (plen, kind, ov), n_sample=20, min_covered=10 * plen)
            assert set(got[:-1].tolist()) == {plen + 3 if ov else plen}, (plen, kind, ov)
            ac.set_engine(ab.Engine.Sequential)
            assert np.array_equal(ac.match_coverage_batch_np((d_hay, offs), overlapping=ov).astype(np.int64), got)
            ac.set_engine(ab.Engine.Auto)
