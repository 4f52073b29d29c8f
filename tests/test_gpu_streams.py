"""Stream sets on the H100 (acg_streams_*, AhoCorasick.streams).

Every stream is a contiguous range of a device haystack, cut into one chunk per feed at seeded points; a feed's
chunks are gathered from the haystack in torch.  The reference for all streams at once is one batch call over the
per-stream ranges (find_iter_batch_torch / find_overlapping_iter_batch_torch, whose offsets are relative to each
range, as the streams' are), and sampled streams are compared with the oracle.  A stream's records over all feeds,
concatenated (a stable sort by stream of every feed's records), must equal the batch's records for it.  Covered:
the Standard prefilter variants of tests/test_gpu_batch.py on both engines; cfg 2's 1.8 M documents in 4 GiB dealt
to 65 536 streams in 16 rounds (overlapping); cfg 4 as a decode step (4 096 streams, 1 000 feeds of 1 to 8 bytes,
find_iter); one stream fed 9 x 512 MiB, past 2^32; and cfg 5's 100 000 patterns over 2 GiB in 8 rounds."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu


def cuts_for(bounds, n_rounds, seed):
    """[n_rounds + 1, n_streams] cut points: stream s's chunk of round r is [cuts[r, s], cuts[r + 1, s]), cut at
    random points of the stream [bounds[s], bounds[s + 1])."""
    rng = np.random.default_rng(seed)
    n = bounds.size - 1
    inner = np.sort(rng.random((n_rounds - 1, n)), axis=0)
    c = bounds[:-1] + (inner * (bounds[1:] - bounds[:-1])).astype(np.int64)
    return np.vstack([bounds[:-1], c, bounds[1:]]).astype(np.int64)


def round_chunks(d_hay, cuts, r, device_offsets=True):
    """(values, offsets) of round r: the chunks gathered into one CUDA buffer, offsets on the device or the host."""
    import torch
    lo, hi = cuts[r], cuts[r + 1]
    lens = hi - lo
    offs = np.r_[0, np.cumsum(lens)].astype(np.int64)
    total = int(offs[-1])
    dev = d_hay.device
    if total:
        shift = torch.repeat_interleave(torch.from_numpy(lo - offs[:-1]).to(dev), torch.from_numpy(lens).to(dev),
                                        output_size=total)
        values = d_hay[torch.arange(total, device=dev) + shift]
        del shift
    else:
        values = torch.empty(0, dtype=torch.uint8, device=dev)
    return values, (torch.from_numpy(offs).to(dev) if device_offsets else offs)


def stable_by_stream(parts):
    import torch
    rec = torch.cat(parts) if parts else torch.empty((0, 3), dtype=torch.int64, device="cuda")
    order = torch.sort(rec[:, 0] >> 32, stable=True).indices
    return rec[order]


def feed_all(ac, d_hay, cuts, overlapping, forms=("torch",), between=None):
    """Feed every round; returns the records of all feeds in stream order (CUDA int64 [n, 3])."""
    import torch
    n = cuts.shape[1]
    parts = []
    with ac.streams(n, overlapping) as st:
        for r in range(cuts.shape[0] - 1):
            if between:
                between(r)
            form = forms[r % len(forms)]
            values, offs = round_chunks(d_hay, cuts, r, device_offsets=form == "torch")
            if form == "torch":
                got = st.feed_torch((values, offs))
                rec = got.records
                assert torch.equal(got.offsets.cpu(), torch.searchsorted(
                    rec[:, 0] >> 32, torch.arange(n + 1, device=rec.device)).cpu())
            else:
                h = st.feed_np((values, offs))
                rec = torch.from_numpy(np.stack([h["pid"].astype(np.int64) | (h["doc"].astype(np.int64) << 32),
                                                 h["start"].astype(np.int64), h["end"].astype(np.int64)], axis=1)
                                       .reshape(-1, 3)).to(d_hay.device)
            parts.append(rec.clone())
            del values
        assert np.array_equal(st.positions().astype(np.int64), cuts[-1] - cuts[0])
    return stable_by_stream(parts)


def check(ac, d_hay, bounds, cuts, overlapping, o, n_sample=20, **kw):
    import torch
    got = feed_all(ac, d_hay, cuts, overlapping, **kw)
    fn = ac.find_overlapping_iter_batch_torch if overlapping else ac.find_iter_batch_torch
    want = fn((d_hay, torch.from_numpy(bounds).to(d_hay.device))).records
    assert got.shape == want.shape, (got.shape, want.shape)
    assert torch.equal(got, want)
    rng = np.random.default_rng(n_sample)
    doc = (got[:, 0] >> 32).cpu().numpy()
    g = got.cpu().numpy()
    for s in np.unique(rng.integers(0, bounds.size - 1, size=n_sample)):
        h = d_hay[int(bounds[s]):int(bounds[s + 1])].cpu().numpy()
        w = o.find_overlapping_iter_np(h) if overlapping else o.find_iter_np(h)
        mine = g[doc == s]
        assert len(mine) == len(w), s
        assert np.array_equal(mine[:, 0] & 0xFFFFFFFF, w["pid"]) and np.array_equal(mine[:, 1], w["start"]) \
            and np.array_equal(mine[:, 2], w["end"]), s
    return got


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
@pytest.mark.parametrize("name", [k for k, v in VARIANTS.items() if v[3] == 0])
def test_stream_variants(name, engine):
    import torch
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, min(mib, 32), ci)
    ac = build(pats, kind, ci).set_engine(engine)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    bounds = offs[::max(1, (offs.size - 1) // 512)]
    bounds = np.r_[bounds[bounds < hay.size], hay.size].astype(np.int64)
    cuts = cuts_for(bounds, 6, seed)
    for overlapping in (False, True):
        check(ac, d_hay, bounds, cuts, overlapping, o, forms=("torch", "host"))
        assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter if engine == ab.Engine.Auto
                                                else ab.Engine.Sequential)
    del d_hay
    torch.cuda.empty_cache()


def _config(name, n):
    import torch
    pats = W.config_patterns(name)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config(name, d_hay, pats)
    return pats, ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats), d_hay


def test_cfg2_4gib_in_65536_streams_16_rounds():
    """cfg 2's 1.8 M documents in 4 GiB, dealt in order to 65 536 streams (about 27 documents each), fed in 16
    rounds that cut at document boundaries, overlapping mode."""
    import torch
    n = 4 << 30
    pats, ac, d_hay = _config("cfg2", n)
    offs = W.doc_offsets(n, 0xD0C5)
    n_docs = offs.size - 1
    assert 1_600_000 < n_docs < 2_000_000
    first = (np.arange(65537) * n_docs) // 65536  # stream s: documents [first[s], first[s + 1])
    bounds = offs[first].astype(np.int64)
    rounds = 16
    cuts = np.stack([offs[first[:-1] + ((first[1:] - first[:-1]) * r) // rounds] for r in range(rounds)]
                    + [bounds[1:]]).astype(np.int64)
    got = check(ac, d_hay, bounds, cuts, True, O.Oracle(pats, kind=O.KIND_DFA), n_sample=20)
    assert got.shape[0] > 500_000
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    del d_hay
    torch.cuda.empty_cache()


def test_cfg4_decode_steps():
    """4 096 streams fed 1 000 times 1 to 8 bytes each, from CUDA tensors, find_iter mode."""
    import torch
    pats, ac, d_hay = _config("cfg4", 4096 * 8 * 1000)
    k = np.random.default_rng(4).integers(1, 9, size=(1000, 4096))
    bounds = np.r_[0, np.cumsum(k.sum(axis=0))].astype(np.int64)
    cuts = (bounds[:-1] + np.r_[np.zeros((1, 4096), np.int64), np.cumsum(k, axis=0)]).astype(np.int64)
    assert np.array_equal(cuts[-1], bounds[1:])
    check(ac, d_hay, bounds, cuts, False, O.Oracle(pats, kind=O.KIND_DFA), n_sample=40)
    del d_hay
    torch.cuda.empty_cache()


def test_one_stream_past_4_gib():
    """One stream fed 9 x 512 MiB in both modes: absolute offsets past 2^32, against the single-haystack calls."""
    import torch
    piece = 512 << 20
    n = 9 * piece
    pats, ac, d_hay = _config("cfg2", n)
    with ac.streams(1, overlapping=True) as ov, ac.streams(1) as it:
        parts_ov, parts_it = [], []
        for r in range(9):
            chunk = (d_hay[r * piece:(r + 1) * piece], np.array([0, piece]))
            parts_ov.append(ov.feed_np(chunk))
            parts_it.append(it.feed_np(chunk))
        assert ov.positions()[0] == n and it.positions()[0] == n
    for parts, fn in ((parts_ov, ac.find_overlapping_iter_dev_np), (parts_it, ac.find_iter_dev_np)):
        got = np.concatenate(parts)
        want, _ = fn(d_hay.data_ptr(), n)
        assert len(got) == len(want) and got["end"].max() > (1 << 32)
        for k in ("pid", "start", "end"):
            assert np.array_equal(got[k], want[k]), k
    del d_hay
    torch.cuda.empty_cache()


def test_cfg5_2gib_in_8_rounds():
    """cfg 5's 100 000 patterns over 2 GiB: 4 096 streams of 512 KiB, 8 rounds, both modes."""
    import torch
    n = 2 << 30
    pats, ac, d_hay = _config("cfg5", n)
    assert ac.patterns_len() == 100_000
    bounds = np.linspace(0, n, 4097).astype(np.int64)
    cuts = cuts_for(bounds, 8, 5)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    for overlapping in (False, True):
        check(ac, d_hay, bounds, cuts, overlapping, o, n_sample=6)
    del d_hay
    torch.cuda.empty_cache()
