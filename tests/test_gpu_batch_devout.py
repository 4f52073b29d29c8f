"""Batched search with device-resident results on the H100 (acg_*_batch_devout through the torch forms):
record for record what the host-output batch calls return, with the document offsets as a CUDA tensor and as a
host array, on the batches of tests/test_gpu_batch.py; and the full-size docs workload of tools/bench_docs.py."""
import sys
from pathlib import Path

import numpy as np
import pytest

import aho_corasick_b200 as ab
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))


def host_records(t):
    """int64 [n, 3] CUDA records -> DOC_MATCH_DTYPE ndarray (same bytes)."""
    return np.ascontiguousarray(t.cpu().numpy()).view(np.uint8).reshape(-1).view(ab.DOC_MATCH_DTYPE)


def check_matches(bm, want, n_docs, device, ctx):
    import torch
    for t in (bm.records, bm.offsets, bm.pid, bm.doc, bm.start, bm.end):
        assert t.device == device, ctx
    got = host_records(bm.records)
    assert len(got) == len(want) and got.tobytes() == want.tobytes(), ctx
    want_offs = np.searchsorted(want["doc"].astype(np.int64), np.arange(n_docs + 1), side="left")
    assert np.array_equal(bm.offsets.cpu().numpy(), want_offs), ctx
    assert torch.equal(bm.pid.cpu(), torch.from_numpy(want["pid"].astype(np.int64))), ctx
    assert torch.equal(bm.doc.cpu(), torch.from_numpy(want["doc"].astype(np.int64))), ctx
    assert torch.equal(bm.end.cpu() - bm.start.cpu(), torch.from_numpy((want["end"] - want["start"]).astype(np.int64)))


@pytest.mark.parametrize("name", list(VARIANTS))
def test_torch_forms_match_the_host_output_calls(name):
    import torch
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    ac = build(pats, kind, ci)
    n_docs = offs.size - 1
    d_offs = torch.from_numpy(offs).to(d_hay.device)
    host = (d_hay, offs)
    whats = ["iter", "overlapping"] if kind == 0 else ["iter"]
    for engine in (ab.Engine.Auto, ab.Engine.Sequential):
        ac.set_engine(engine)
        want = {w: (ac.find_overlapping_iter_batch_np if w == "overlapping" else ac.find_iter_batch_np)(host)
                for w in whats}
        want_flags = ac.is_match_batch(host)
        want_find = ac.find_batch_np(host)
        for offsets in (d_offs, offs):
            ctx = (name, engine, "cuda offsets" if offsets is d_offs else "host offsets")
            batch = (d_hay, offsets)
            for w in whats:
                fn = ac.find_overlapping_iter_batch_torch if w == "overlapping" else ac.find_iter_batch_torch
                bm = fn(batch)
                assert ac.last_stats()["engine"] == (int(ab.Engine.Prefilter) if engine == ab.Engine.Auto
                                                     else int(ab.Engine.Sequential)), ctx
                assert len(want[w]) > 1000
                check_matches(bm, want[w], n_docs, d_hay.device, (ctx, w))
            flags = ac.is_match_batch_torch(batch)
            assert flags.dtype == torch.bool and flags.device == d_hay.device
            assert np.array_equal(flags.cpu().numpy(), want_flags), ctx
            found, rec = ac.find_batch_torch(batch)
            assert found.device == d_hay.device and rec.device == d_hay.device
            assert np.array_equal(found.cpu().numpy(), want_find[0]), ctx
            assert host_records(rec).tobytes() == want_find[1].tobytes(), ctx
    # invalid device offsets are found on the device
    bad = d_offs.clone()
    bad[n_docs // 2] = bad[n_docs // 2 + 1] + 1
    with pytest.raises(ValueError):
        ac.find_iter_batch_torch((d_hay, bad))
    with pytest.raises(ValueError):
        ac.is_match_batch_torch((d_hay, d_offs + 1))


def test_full_size_docs_workload():
    """tools/bench_docs.py's workload: cfg 2's automaton and 4 GiB haystack cut into ~1.8 M documents, offsets
    a CUDA tensor.  The device list equals the host-output list in count and FNV-1a, and the doc column of the
    records is what the CSR index implies."""
    import torch
    from bench_docs import fnv1a
    n = 4 << 30
    pats = W.config_patterns("cfg2")
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg2", d_hay, pats)
    offs = W.doc_offsets(n, 0xD0C5)
    n_docs = offs.size - 1
    ac = build(pats)
    want = ac.find_overlapping_iter_batch_np((d_hay, offs))
    bm = ac.find_overlapping_iter_batch_torch((d_hay, torch.from_numpy(offs).cuda()))
    got = host_records(bm.records)
    assert len(got) == len(want) > 1_000_000
    assert fnv1a(got) == fnv1a(want)
    counts = bm.offsets[1:] - bm.offsets[:-1]
    implied = torch.repeat_interleave(torch.arange(n_docs, device="cuda"), counts)
    assert torch.equal(bm.doc, implied)
    assert int(bm.offsets[0]) == 0 and int(bm.offsets[-1]) == len(got)
    del d_hay, bm
    torch.cuda.empty_cache()
