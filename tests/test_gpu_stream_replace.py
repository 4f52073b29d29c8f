"""Replace sets on the H100 (acg_streams_create_replace, AhoCorasick.replace_streams).

Every stream is a contiguous range of a device haystack, cut into one chunk per feed at seeded points (the chunks
gathered in torch, as in tests/test_gpu_streams.py).  After the last feed every stream is flushed.  A stream's
outputs over all its feeds followed by its flush must equal replace_all_bytes of its range, and the reference for
all streams at once is one replace_all_batch_torch call over the per-stream ranges; sampled streams are also
compared with the oracle's find_iter spliced on the host.  Covered: the Standard prefilter variants on both engines;
cfg 2's 4 GiB dealt to 65 536 streams in 16 rounds; cfg 4 as a decode step (4 096 streams, 1 000 feeds of 1 to 8
bytes); cfg 5's 100 000 patterns over 1 GiB; one stream fed past 2^32 with a match across that offset; 64 KiB
patterns; and the overflow retry with device output."""
import ctypes

import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from test_gpu_batch import VARIANTS, batch_workload, build
from test_gpu_streams import _config, cuts_for, round_chunks

pytestmark = pytest.mark.gpu


def splice(doc, starts, ends, pids, reps):
    """The loop of try_replace_all_bytes over one document's matches."""
    out, last = [], 0
    for s, e, p in zip(starts, ends, pids):
        out += [doc[last:s], reps[p]]
        last = e
    out.append(doc[last:])
    return b"".join(out)


def tag_table(pats):
    """Deletions, same-length replacements and tags longer than their patterns, some by hundreds of bytes."""
    reps = []
    for i, p in enumerate(pats):
        k = i % 4
        reps.append(b"" if k == 0 else b"*" * len(p) if k == 1 else b"<PII:%d>" % i if k == 2
                    else b"[" + b"redacted " * (1 + i % 50) + b"]")
    return reps


def assemble(pieces, n):
    """Each stream's pieces -- one (values, offsets) per feed and the flush, on the device -- concatenated in order,
    as one (values, int64 offsets [n + 1]) batch in stream order."""
    import torch
    dev = pieces[0][1].device
    lens = torch.stack([o[1:] - o[:-1] for _, o in pieces])  # [feeds + 1, n]
    per = lens.sum(0)
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    offsets[1:] = torch.cumsum(per, 0)
    within = torch.cumsum(lens, 0) - lens
    out = torch.empty(int(offsets[-1]), dtype=torch.uint8, device=dev)
    for r, (v, o) in enumerate(pieces):
        if v.numel():
            base = offsets[:-1] + within[r] - o[:-1]
            out[torch.repeat_interleave(base, lens[r], output_size=v.numel())
                + torch.arange(v.numel(), device=dev)] = v
    return out, offsets


def feed_all(ac, d_hay, cuts, reps, forms=("torch",)):
    """Feed every round and flush: the stream-order (values, offsets) of all outputs."""
    import torch
    n = cuts.shape[1]
    back = ac.max_pattern_len() - 1
    dev = d_hay.device
    pieces = []
    with ac.replace_streams(n, reps) as st:
        for r in range(cuts.shape[0] - 1):
            form = forms[r % len(forms)]
            values, offs = round_chunks(d_hay, cuts, r, device_offsets=form == "torch")
            if form == "torch":
                out, oo = st.feed_torch((values, offs))
            else:
                v, o = st.feed_np((values, offs))
                out, oo = torch.from_numpy(v).to(dev), torch.from_numpy(o.astype(np.int64)).to(dev)
            pieces.append((out, oo))
            del values
        assert np.array_equal(st.positions().astype(np.int64), cuts[-1] - cuts[0])
        assert (st.held() <= back).all()
        v, o = st.flush_np()
        pieces.append((torch.from_numpy(v).to(dev), torch.from_numpy(o.astype(np.int64)).to(dev)))
        assert not st.positions().any()
    return assemble(pieces, n)


def check(ac, d_hay, bounds, cuts, reps, o, n_sample=20, **kw):
    import torch
    got_v, got_o = feed_all(ac, d_hay, cuts, reps, **kw)
    want_v, want_o = ac.replace_all_batch_torch((d_hay, torch.from_numpy(bounds).to(d_hay.device)), reps)
    assert torch.equal(got_o, want_o)
    assert torch.equal(got_v, want_v)
    rng = np.random.default_rng(n_sample)
    go = got_o.cpu().numpy()
    for s in np.unique(rng.integers(0, bounds.size - 1, size=n_sample)):
        h = d_hay[int(bounds[s]):int(bounds[s + 1])].cpu().numpy()
        w = o.find_iter_np(h)
        want = splice(h.tobytes(), w["start"].tolist(), w["end"].tolist(), w["pid"].tolist(), reps)
        assert got_v[int(go[s]):int(go[s + 1])].cpu().numpy().tobytes() == want, s
    return got_v, got_o


@pytest.mark.parametrize("engine", [ab.Engine.Auto, ab.Engine.Sequential])
@pytest.mark.parametrize("name", [k for k, v in VARIANTS.items() if v[3] == 0])
def test_replace_set_variants(name, engine):
    import torch
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, min(mib, 32), ci)
    ac = build(pats, kind, ci).set_engine(engine)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    bounds = offs[::max(1, (offs.size - 1) // 512)]
    bounds = np.r_[bounds[bounds < hay.size], hay.size].astype(np.int64)
    check(ac, d_hay, bounds, cuts_for(bounds, 6, seed), tag_table(pats), o, forms=("torch", "host"))
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter if engine == ab.Engine.Auto
                                            else ab.Engine.Sequential)
    del d_hay
    torch.cuda.empty_cache()


def test_cfg2_4gib_in_65536_streams_16_rounds():
    """cfg 2's 1.8 M documents in 4 GiB, dealt in order to 65 536 streams, fed in 16 rounds cut at random points."""
    import torch
    from aho_corasick_b200 import workload as W
    n = 4 << 30
    pats, ac, d_hay = _config("cfg2", n)
    offs = W.doc_offsets(n, 0xD0C5)
    first = (np.arange(65537) * (offs.size - 1)) // 65536
    bounds = offs[first].astype(np.int64)
    reps = tag_table(pats)
    got_v, _ = check(ac, d_hay, bounds, cuts_for(bounds, 16, 2), reps, O.Oracle(pats, kind=O.KIND_DFA))
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    del d_hay, got_v
    torch.cuda.empty_cache()


def test_cfg4_decode_steps():
    """4 096 streams fed 1 000 times 1 to 8 bytes each, from CUDA tensors."""
    import torch
    pats, ac, d_hay = _config("cfg4", 4096 * 8 * 1000)
    k = np.random.default_rng(4).integers(1, 9, size=(1000, 4096))
    bounds = np.r_[0, np.cumsum(k.sum(axis=0))].astype(np.int64)
    cuts = (bounds[:-1] + np.r_[np.zeros((1, 4096), np.int64), np.cumsum(k, axis=0)]).astype(np.int64)
    check(ac, d_hay, bounds, cuts, tag_table(pats), O.Oracle(pats, kind=O.KIND_DFA), n_sample=40)
    del d_hay
    torch.cuda.empty_cache()


def test_cfg5_1gib_in_8_rounds():
    """cfg 5's 100 000 patterns over 1 GiB: 4 096 streams of 256 KiB, 8 rounds."""
    import torch
    n = 1 << 30
    pats, ac, d_hay = _config("cfg5", n)
    assert ac.patterns_len() == 100_000
    bounds = np.linspace(0, n, 4097).astype(np.int64)
    check(ac, d_hay, bounds, cuts_for(bounds, 8, 5), tag_table(pats), O.Oracle(pats, kind=O.KIND_DFA), n_sample=6)
    del d_hay
    torch.cuda.empty_cache()


def test_one_stream_past_4_gib():
    """One stream fed 9 x 512 MiB, with a pattern planted across offset 2^32, which is also a feed boundary."""
    import torch
    piece = 512 << 20
    n = 9 * piece
    pats, ac, d_hay = _config("cfg2", n)
    p = max(pats, key=len)
    at = (1 << 32) - len(p) // 2
    d_hay[at:at + len(p)] = torch.frombuffer(bytearray(p), dtype=torch.uint8).cuda()
    reps = tag_table(pats)
    pieces = []
    with ac.replace_streams(1, reps) as st:
        for r in range(9):
            out, oo = st.feed_torch((d_hay[r * piece:(r + 1) * piece], np.array([0, piece])))
            pieces.append(out)
        assert st.positions()[0] == n
        tail = st.flush()[0]
    got = torch.cat(pieces + [torch.frombuffer(bytearray(tail), dtype=torch.uint8).cuda()] if tail else pieces)
    want, wo = ac.replace_all_batch_torch((d_hay, np.array([0, n])), reps)
    assert torch.equal(got, want)
    w0 = at - 64
    window = d_hay[w0:at + len(p) + 64].cpu().numpy().tobytes()
    assert any(w0 + m.start() < (1 << 32) < w0 + m.end() for m in ac.find_iter(window)), "no match across 2^32"
    del d_hay, got, want
    torch.cuda.empty_cache()


def test_64kib_patterns():
    """64 KiB patterns among short ones: streams held at back = 65 535 bytes, and matches across many feeds."""
    import torch
    rng = np.random.default_rng(64)
    longs = [rng.integers(97, 101, size=65536, dtype=np.uint8).tobytes() for _ in range(3)]
    pats = longs + [b"abcd", b"dcba", b"bad"]
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    n_streams, per = 64, 1 << 20
    hay = rng.integers(97, 101, size=n_streams * per, dtype=np.uint8)
    for s in range(n_streams):
        for j in range(3):
            at = s * per + 4096 + j * 300_000 + s * 17
            hay[at:at + 65536] = np.frombuffer(longs[(s + j) % 3], np.uint8)
    d_hay = torch.from_numpy(hay).cuda()
    bounds = np.arange(n_streams + 1, dtype=np.int64) * per
    reps = [b"[long %d]" % i for i in range(3)] + [b"", b"DCBA", b"<bad>"]
    check(ac, d_hay, bounds, cuts_for(bounds, 40, 64), reps, O.Oracle(pats, kind=O.KIND_DFA), n_sample=4)
    del d_hay
    torch.cuda.empty_cache()


def test_overflow_retry_on_device():
    """Device output with cap one byte short: ACG_E_OVERFLOW with the exact size, no stream changed, and the retry
    gives what a set that never overflowed gives."""
    import torch
    pats, ac, d_hay = _config("cfg2", 64 << 20)
    reps = tag_table(pats)
    bounds = np.linspace(0, d_hay.numel(), 257).astype(np.int64)
    cuts = cuts_for(bounds, 4, 9)
    with ac.replace_streams(256, reps) as clean, ac.replace_streams(256, reps) as st:
        for r in range(4):
            values, offs = round_chunks(d_hay, cuts, r)
            want_v, want_o = clean.feed_torch((values, offs))
            need = want_v.numel()
            pos, held = st.positions(), st.held()
            out = torch.full((need + 64,), 0xA5, dtype=torch.uint8, device="cuda")
            oo = torch.full((258,), -1, dtype=torch.int64, device="cuda")
            cnt = ctypes.c_uint64()
            rc = ab._lib.acg_streams_replace_feed_devout(st._h, values.data_ptr(), values.numel(), offs.data_ptr(), 1,
                                                         256, out.data_ptr(), need - 1, oo.data_ptr(),
                                                         ctypes.byref(cnt))
            assert rc == ab.E_OVERFLOW and cnt.value == need
            assert (out == 0xA5).all() and (oo == -1).all()
            assert np.array_equal(st.positions(), pos) and np.array_equal(st.held(), held)
            rc = ab._lib.acg_streams_replace_feed_devout(st._h, values.data_ptr(), values.numel(), offs.data_ptr(), 1,
                                                         256, out.data_ptr(), need, oo.data_ptr(), ctypes.byref(cnt))
            assert rc == 0 and cnt.value == need
            assert torch.equal(out[:need], want_v) and torch.equal(oo[:257], want_o) and (out[need:] == 0xA5).all()
        assert st.flush() == clean.flush()
    del d_hay
    torch.cuda.empty_cache()
