"""Pattern counts per document on the H100 (acg_pattern_counts_batch / _devout and the torch sparse CSR form).

Every result is compared with a torch grouping, computed on the device, of the same handle's *_batch_torch
records (torch.unique(doc * P + pid, return_counts=True)) and with the oracle on sampled documents.  Host
output, the raw device-output call and the sparse tensor must agree.  Covered: the prefilter kernel variants
of tests/test_gpu_batch.py on both engines, and the full-size shapes -- cfg 2's 1.8 M documents (overlapping)
and cfg 3's (find_iter) in 4 GiB, cfg 5's 100 000 patterns over 2 GiB, one 4 GiB document and a batch whose
span ends past 4 GiB."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu


def grouped_records(ac, d_hay, offs, overlapping, anchored=ab.Anchored.No):
    """(rows, pids, counts) int64 CUDA tensors: the batch records grouped with torch.unique on the device."""
    import torch
    n_docs, n_pats = offs.size - 1, ac.patterns_len()
    r = ac.find_overlapping_iter_batch_torch((d_hay, offs)) if overlapping else \
        ac.find_iter_batch_torch((d_hay, offs), anchored=anchored)
    keys, counts = torch.unique(r.doc * n_pats + r.pid, return_counts=True)
    docs = keys // n_pats
    rows = torch.searchsorted(docs, torch.arange(n_docs + 1, device=docs.device), right=False)
    return rows, keys % n_pats, counts


def counts_everywhere(ac, d_hay, offs, overlapping, anchored=ab.Anchored.No):
    """The sparse tensor's (crow, col, values); host output and the raw device-output call, checked equal to it."""
    import torch
    sp = ac.pattern_counts_batch_torch((d_hay, offs), overlapping=overlapping, anchored=anchored)
    assert sp.layout == torch.sparse_csr and sp.shape == (offs.size - 1, ac.patterns_len())
    rows, pids, counts = sp.crow_indices(), sp.col_indices(), sp.values()
    assert rows.dtype == pids.dtype == counts.dtype == torch.int64
    h_rows, h_pids, h_counts = ac.pattern_counts_batch_np((d_hay, offs), overlapping=overlapping, anchored=anchored)
    assert np.array_equal(h_rows.astype(np.int64), rows.cpu().numpy())
    assert np.array_equal(h_pids.astype(np.int64), pids.cpu().numpy())
    assert np.array_equal(h_counts.astype(np.int64), counts.cpu().numpy())
    nnz = len(h_pids)
    d_rows = torch.empty(offs.size, dtype=torch.int64, device=d_hay.device)
    d_pids = torch.empty(max(nnz, 1), dtype=torch.int32, device=d_hay.device)
    d_counts = torch.empty(max(nnz, 1), dtype=torch.int64, device=d_hay.device)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(d_hay.device)
    got = ac.pattern_counts_batch_devout(d_hay.data_ptr(), d_hay.numel(), d_offs.data_ptr(), d_rows.data_ptr(),
                                         d_pids.data_ptr(), d_counts.data_ptr(), nnz, overlapping=overlapping,
                                         anchored=anchored, n_docs=offs.size - 1)
    assert got == nnz and torch.equal(d_rows, rows) and torch.equal(d_pids[:nnz].long(), pids) \
        and torch.equal(d_counts[:nnz], counts)
    return rows, pids, counts


def check(ac, d_hay, offs, overlapping, o, ctx, n_sample=100, anchored=ab.Anchored.No, min_nnz=1):
    import torch
    rows, pids, counts = counts_everywhere(ac, d_hay, offs, overlapping, anchored)
    want = grouped_records(ac, d_hay, offs, overlapping, anchored)
    for g, w, name in zip((rows, pids, counts), want, ("rows", "pids", "counts")):
        assert torch.equal(g, w), (ctx, name)
    assert int(rows[-1]) >= min_nnz, ctx
    rows, pids, counts = rows.cpu().numpy(), pids.cpu().numpy(), counts.cpu().numpy()
    fn = o.find_overlapping_iter_np if overlapping else o.find_iter_np
    for d in np.random.default_rng(offs.size).integers(0, offs.size - 1, size=n_sample):
        doc = d_hay[int(offs[d]):int(offs[d + 1])].cpu().numpy()
        u, c = np.unique(fn(doc, anchored=bool(anchored))["pid"].astype(np.int64), return_counts=True)
        lo, hi = rows[d], rows[d + 1]
        assert np.array_equal(pids[lo:hi], u) and np.array_equal(counts[lo:hi], c), (ctx, d)
    return rows, pids, counts


@pytest.mark.parametrize("name", list(VARIANTS))
def test_counts_variants(name):
    """Every prefilter variant and then the sequential engine: the same matrix as the grouped records."""
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    for ov in ((False, True) if kind == 0 else (False,)):
        want = check(ac, d_hay, offs, ov, o, (name, ov), min_nnz=1000)
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
        ac.set_engine(ab.Engine.Sequential)
        got = counts_everywhere(ac, d_hay, offs, ov)
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        assert all(np.array_equal(g.cpu().numpy(), w) for g, w in zip(got, want)), (name, ov, "sequential")
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
        check(ac, d_hay, offs, False, o, kind, anchored=ab.Anchored.Yes, min_nnz=1000)
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
    """tools/bench_docs.py's documents: 4 GiB cut into ~1.8 M; cfg 2 counts find_overlapping_iter, cfg 3
    find_iter (leftmost-first, case-insensitive)."""
    import torch
    n = 4 << 30
    pats, ac, d_hay = _config_batch(name, n)
    offs = W.doc_offsets(n, 0xD0C5)
    assert 1_600_000 < offs.size < 2_000_000
    o = O.Oracle(pats, match_kind=int(ac.match_kind()), ascii_case_insensitive=name == "cfg3", kind=O.KIND_DFA)
    check(ac, d_hay, offs, name == "cfg2", o, name, n_sample=60, min_nnz=100_000)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    del d_hay
    torch.cuda.empty_cache()


def test_full_size_cfg5_pid_bits_17():
    """cfg 5's 100 000 patterns (17 pid bits) over 2 GiB cut into documents."""
    import torch
    n = 2 << 30
    pats, ac, d_hay = _config_batch("cfg5", n)
    assert ac.patterns_len() == 100_000
    offs = W.doc_offsets(n, 0xC5)
    _, pids, _ = check(ac, d_hay, offs, True, O.Oracle(pats, kind=O.KIND_DFA), "cfg5", n_sample=30,
                       min_nnz=10_000)
    assert pids.max() >= 1 << 16
    del d_hay
    torch.cuda.empty_cache()


def test_one_4_gib_document_and_a_batch_past_4_gib():
    """One 4 GiB document: its row is np.bincount of the single-haystack find_overlapping_iter pids.  Then a
    batch of documents whose span starts before and ends past 2^32."""
    import torch
    n = (4 << 30) + (192 << 20)
    pats, ac, d_hay = _config_batch("cfg2", n)
    whole = 4 << 30
    sp = ac.pattern_counts_batch_torch((d_hay, np.array([0, whole])), overlapping=True)
    single, _ = ac.find_overlapping_iter_dev_np(d_hay.data_ptr(), whole)
    assert len(single) > 500_000
    bc = np.bincount(single["pid"].astype(np.int64), minlength=len(pats))
    want_pids = np.flatnonzero(bc)
    assert sp.crow_indices().tolist() == [0, len(want_pids)]
    assert np.array_equal(sp.col_indices().cpu().numpy(), want_pids)
    assert np.array_equal(sp.values().cpu().numpy(), bc[want_pids])
    h_rows, h_pids, h_counts = ac.pattern_counts_batch_np((d_hay, np.array([0, whole])), overlapping=True)
    assert np.array_equal(h_pids, want_pids) and np.array_equal(h_counts, bc[want_pids])
    # documents from 2^32 - 160 MiB to the end of the buffer, past 2^32
    offs = (whole - (160 << 20)) + W.doc_offsets(n - whole + (160 << 20), 0x4AB)
    assert offs[0] < 1 << 32 < offs[-1] == n
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for ov in (True, False):
        check(ac, d_hay, offs, ov, o, ("past 4 GiB", ov), n_sample=60, min_nnz=10_000)
    del d_hay
    torch.cuda.empty_cache()
