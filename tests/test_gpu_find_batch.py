"""Batched find on the H100 (acg_find_batch): the device-resident batches of tests/test_gpu_batch.py (every
prefilter kernel variant), the per-document sequential kernel, and the full-size docs workload of
tools/bench_docs.py (cfg 2 and cfg 3 over 4 GiB).  For every document, find_batch is the first record
find_iter_batch gives it (or no match), and on sampled documents it is the oracle's try_find."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu


def first_records(rec, n_docs):
    """(found, records) of the first record of every document in a find_iter_batch list, in find_batch's form."""
    found = np.zeros(n_docs, bool)
    first = np.zeros(n_docs, ab.DOC_MATCH_DTYPE)
    first["doc"] = np.arange(n_docs)
    if len(rec):
        idx = np.flatnonzero(np.r_[True, rec["doc"][1:] != rec["doc"][:-1]])
        docs = rec["doc"][idx].astype(np.int64)
        found[docs] = True
        first[docs] = rec[idx]
    return found, first


def same(got, want, ctx):
    assert np.array_equal(got[0], want[0]), (ctx, np.flatnonzero(got[0] != want[0])[:5])
    assert got[1].tobytes() == want[1].tobytes(), (ctx, np.flatnonzero(got[1] != want[1])[:5])


def sampled_docs_match_the_oracle(got, o, doc_bytes, n_docs, ctx, anchored=False, earliest=False, n=200, seed=0):
    found, r = got
    for d in np.unique(np.random.default_rng(seed).integers(0, n_docs, size=n)):
        m = o.try_find(doc_bytes(d), anchored=anchored, earliest=earliest)
        assert bool(found[d]) == (m is not None), (ctx, d)
        assert (int(r["doc"][d]), int(r["pid"][d]), int(r["start"][d]), int(r["end"][d])) == \
            ((int(d),) + tuple(m) if m is not None else (int(d), 0, 0, 0)), (ctx, d)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_find_batch_variants(name):
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    n_docs = offs.size - 1
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    dev = (d_hay, offs)
    doc_bytes = lambda d: np.ascontiguousarray(hay[offs[d]:offs[d + 1]])  # noqa: E731
    got = ac.find_batch_np(dev)
    st = ac.last_stats()
    assert st["engine"] == int(ab.Engine.Prefilter) and st["raw_matches"] > 0
    assert got[0].sum() > 1000 and (~got[0]).sum() > 0
    same(got, first_records(ac.find_iter_batch_np(dev), n_docs), (name, "find_iter_batch"))
    sampled_docs_match_the_oracle(got, o, doc_bytes, n_docs, name)
    same(ac.find_batch_np((hay, offs)), got, (name, "host haystack"))
    # `earliest`: Standard is earliest already; a leftmost automaton takes the sequential engine unless the
    # reference gives it the packed prefilter, which ignores `earliest`
    early = ac.find_batch_np(dev, earliest=True)
    packed = ac.prefilter_kind() == 4
    if kind == 0 or packed:
        same(early, got, (name, "earliest"))
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter if kind == 0 or packed else ab.Engine.Sequential)
    sampled_docs_match_the_oracle(early, o, doc_bytes, n_docs, (name, "earliest"), earliest=True, seed=1)
    ac.set_engine(ab.Engine.Sequential)
    same(ac.find_batch_np(dev), got, (name, "sequential"))
    same(ac.find_batch_np(dev, earliest=True), early, (name, "sequential, earliest"))


def test_sequential_path_batches():
    """Anchored input, the empty pattern and `earliest` on leftmost automata: the per-document kernel."""
    import torch
    rng = np.random.default_rng(3)
    hay = rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=4 << 20)
    offs = W.doc_offsets(hay.size, 4, lo=1, hi=256)
    n_docs = offs.size - 1
    d_hay = torch.from_numpy(hay).cuda()
    dev = (d_hay, offs)
    doc_bytes = lambda d: np.ascontiguousarray(hay[offs[d]:offs[d + 1]])  # noqa: E731
    pats = [b"ab", b"abc", b"b", b"ca", b"cab"]
    for kind in (0, 1, 2):
        ac = ab.AhoCorasick.builder().match_kind(kind).start_kind(ab.StartKind.Both).build(pats)
        o = O.Oracle(pats, match_kind=kind, start_kind=int(ab.StartKind.Both))
        got = ac.find_batch_np(dev, anchored=ab.Anchored.Yes)
        assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        same(got, first_records(ac.find_iter_batch_np(dev, anchored=ab.Anchored.Yes), n_docs), (kind, "anchored"))
        sampled_docs_match_the_oracle(got, o, doc_bytes, n_docs, (kind, "anchored"), anchored=True, n=300)
        early = ac.find_batch_np(dev, earliest=True)
        if kind:
            assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
        sampled_docs_match_the_oracle(early, o, doc_bytes, n_docs, (kind, "earliest"), earliest=True, n=300)
        e = ab.AhoCorasick.builder().match_kind(kind).build(pats + [b""])
        oe = O.Oracle(pats + [b""], match_kind=kind)
        got = e.find_batch_np(dev)
        assert got[0].all() and e.last_stats()["engine"] == int(ab.Engine.Sequential)
        sampled_docs_match_the_oracle(got, oe, doc_bytes, n_docs, (kind, "empty pattern"), n=100)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_full_size_docs_workload(cfg):
    """tools/bench_docs.py's workload: the automaton and 4 GiB haystack of cfg 2 (Standard) or cfg 3
    (leftmost-first, case-insensitive) cut into ~1.8 M documents."""
    import torch
    n = 4 << 30
    pats = W.config_patterns(cfg)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config(cfg, d_hay, pats)
    offs = W.doc_offsets(n, 0xD0C5)
    n_docs = offs.size - 1
    kind, ci = (1, True) if cfg == "cfg3" else (0, False)
    ac = build(pats, kind, ci)
    got = ac.find_batch_np((d_hay, offs))
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert 100_000 < got[0].sum() < n_docs
    same(got, first_records(ac.find_iter_batch_np((d_hay, offs)), n_docs), cfg)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    doc_bytes = lambda d: d_hay[int(offs[d]):int(offs[d + 1])].cpu().numpy()  # noqa: E731
    sampled_docs_match_the_oracle(got, o, doc_bytes, n_docs, cfg, seed=1)
    del d_hay
    torch.cuda.empty_cache()
