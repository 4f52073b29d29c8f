"""Replace per document on the H100 (acg_replace_all_batch / _devout and the torch form).

Every result is compared with a torch splice, on the device, of the same handle's find_iter_batch_torch records
(the length change delta of each match, its exclusive cumsum D and q = start + D; for each output byte o,
i = searchsorted(q, o, right) - 1, and the replacement's byte if o < q_i + rep_len_i, else input byte
o - (D_i + delta_i)), built one window of at most 256 MiB of output at a time, and with the oracle on sampled
documents.  Host output, the raw device-output call and the torch form must agree.  Covered: the prefilter kernel
variants of tests/test_gpu_batch.py on both engines, and the full-size shapes -- cfg 2's 1.8 M documents in
4 GiB, cfg 3's (leftmost-first, case-insensitive), cfg 5's 100 000 patterns over 2 GiB, one 4 GiB document, a
batch whose output runs past 2^32, and 4 KiB and 64 KiB patterns at document edges."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from test_gpu_batch import VARIANTS, batch_workload, build

pytestmark = pytest.mark.gpu

WINDOW = 256 << 20  # output bytes the torch reference builds at a time


def mixed_reps(pats, seed, long=0):
    """A seeded table: deletions, shorter, same-length and longer replacements (`long` extra bytes)."""
    rng = np.random.default_rng(seed)
    out = []
    for i, p in enumerate(pats):
        k = int(rng.integers(0, 4))
        out.append((b"", p[: len(p) // 2], b"#" * len(p), b"<%d>" % i + p + b"=" * long)[k])
    return out


def torch_reference(ac, d_hay, offs, reps):
    """(out_offsets int64, a function yielding (w0, expected bytes of [w0, w1)) windows, out_len)."""
    import torch
    dev = d_hay.device
    r = ac.find_iter_batch_torch((d_hay, offs))
    assert r.records.shape[0] > 0
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    rep_len = torch.tensor([len(x) for x in reps], dtype=torch.int64, device=dev)
    rep_at = torch.cumsum(rep_len, 0) - rep_len
    joined = b"".join(reps) or b"\0"
    rep_data = torch.frombuffer(bytearray(joined), dtype=torch.uint8).to(dev)
    lo = int(offs[0])
    base = d_offs[r.doc] - lo
    s, e, pid = base + r.start, base + r.end, r.pid
    delta = rep_len[pid] - (e - s)
    incl = torch.cumsum(delta, 0)
    q = s + incl - delta
    incl0 = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), incl])
    out_offsets = d_offs - lo + incl0[r.offsets]
    out_len = int(out_offsets[-1])
    span = int(offs[-1]) - lo

    def windows():
        for w0 in range(0, out_len, WINDOW):
            o = torch.arange(w0, min(out_len, w0 + WINDOW), dtype=torch.int64, device=dev)
            i = torch.searchsorted(q, o, right=True) - 1
            ok = i >= 0
            ic = i.clamp(min=0)
            qi = torch.where(ok, q[ic], 0)
            p = pid[ic]
            in_rep = ok & (o < qi + rep_len[p])
            src = o - torch.where(ok, incl[ic], 0)
            from_rep = rep_data[(rep_at[p] + o - qi).clamp(0, rep_data.numel() - 1)]
            from_hay = d_hay[lo + src.clamp(0, max(span - 1, 0))]
            yield w0, torch.where(in_rep, from_rep, from_hay)
            del o, i, ic, qi, p, in_rep, src, from_rep, from_hay
    return out_offsets, windows, out_len


def check(ac, d_hay, offs, reps, o, ctx, n_sample=100, host=True):
    """The torch form against the torch splice and the oracle; the raw device-output call with device offsets,
    into a buffer with sentinels, and (host) the host-output call against the torch form.  Returns the torch
    (values, offsets)."""
    import torch
    values, out_offsets = ac.replace_all_batch_torch((d_hay, offs), reps)
    assert values.dtype == torch.uint8 and out_offsets.dtype == torch.int64 and values.device == d_hay.device
    want_offs, windows, out_len = torch_reference(ac, d_hay, offs, reps)
    assert torch.equal(out_offsets, want_offs), ctx
    assert values.numel() == out_len, (ctx, values.numel(), out_len)
    for w0, want in windows():
        assert torch.equal(values[w0:w0 + want.numel()], want), (ctx, "window", w0)
        del want
    got_offs = out_offsets.cpu().numpy()
    for d in np.random.default_rng(offs.size).integers(0, offs.size - 1, size=n_sample):
        a, b = int(offs[d]), int(offs[d + 1])
        doc = d_hay[a:b].cpu().numpy()
        r = o.find_iter_np(doc)
        parts, last = [], 0
        for x, y, p in zip(r["start"].tolist(), r["end"].tolist(), r["pid"].tolist()):
            parts += [doc[last:x].tobytes(), reps[p]]
            last = y
        parts.append(doc[last:].tobytes())
        assert values[got_offs[d]:got_offs[d + 1]].cpu().numpy().tobytes() == b"".join(parts), (ctx, int(d))
    # the raw device-output call: device offsets, an output 3 bytes past a 16-byte boundary, sentinels around it
    n_docs = offs.size - 1
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(d_hay.device)
    buf = torch.full((out_len + 67,), 7, dtype=torch.uint8, device=d_hay.device)
    d_oo = torch.full((n_docs + 3,), -1, dtype=torch.int64, device=d_hay.device)
    torch.cuda.synchronize()  # the sentinels are written before the library's stream touches the arrays
    with pytest.raises(OverflowError) as e:
        ac.replace_all_batch_devout(d_hay.data_ptr(), d_hay.numel(), d_offs.data_ptr(), reps, buf[35:].data_ptr(),
                                    out_len - 1, d_oo[1:].data_ptr(), n_docs=n_docs)
    assert e.value.args[0] == out_len and (buf == 7).all() and (d_oo == -1).all(), (ctx, "overflow")
    n = ac.replace_all_batch_devout(d_hay.data_ptr(), d_hay.numel(), d_offs.data_ptr(), reps, buf[35:].data_ptr(),
                                    out_len, d_oo[1:].data_ptr(), n_docs=n_docs)
    assert n == out_len and torch.equal(buf[35:35 + out_len], values), (ctx, "devout")
    assert (buf[:35] == 7).all() and (buf[35 + out_len:] == 7).all(), (ctx, "devout sentinels")
    assert torch.equal(d_oo[1:-1], out_offsets) and d_oo[0] == -1 and d_oo[-1] == -1, (ctx, "devout offsets")
    del buf
    if host:
        h_values, h_offs = ac.replace_all_batch_np((d_hay, offs), reps)
        assert np.array_equal(h_offs.astype(np.int64), got_offs), (ctx, "host offsets")
        assert torch.equal(torch.from_numpy(h_values).to(d_hay.device), values), (ctx, "host")
    return values, out_offsets


@pytest.mark.parametrize("name", list(VARIANTS))
def test_replace_variants(name):
    """Every prefilter variant and then the sequential engine: the splice of the records, and equal engines."""
    import torch
    n, seed, mib, kind, ci = VARIANTS[name]
    pats, hay, offs, d_hay = batch_workload(n, seed, mib, ci, short=name == "stride1_short_patterns")
    ac = build(pats, kind, ci)
    o = O.Oracle(pats, match_kind=kind, ascii_case_insensitive=ci, kind=O.KIND_DFA)
    reps = mixed_reps(pats, seed)
    values, out_offsets = check(ac, d_hay, offs, reps, o, name)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    ac.set_engine(ab.Engine.Sequential)
    v2, o2 = ac.replace_all_batch_torch((d_hay, offs), reps)
    assert ac.last_stats()["engine"] == int(ab.Engine.Sequential)
    assert torch.equal(v2, values) and torch.equal(o2, out_offsets), (name, "sequential")


def test_empty_pattern_on_the_sequential_engine():
    import torch
    rng = np.random.default_rng(3)
    hay = np.frombuffer(b"abc", np.uint8)[rng.integers(0, len(b"abc"), size=4 << 20)]
    offs = W.doc_offsets(hay.size, 4, lo=1, hi=256)
    offs = np.sort(np.r_[offs, offs[1:200:7]])  # and empty documents
    d_hay = torch.from_numpy(hay).cuda()
    pats = [b"ab", b"", b"cab", b"ab"]
    for kind in (0, 1, 2):
        ac = build(pats, kind)
        check(ac, d_hay, offs, [b"XY", b"-", b"", b"Q"], O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA), kind)
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
    """tools/bench_docs.py's documents: 4 GiB cut into ~1.8 M, with tools/bench_docs.py's table."""
    import torch
    n = 4 << 30
    pats, ac, d_hay = _config_batch(name, n)
    offs = W.doc_offsets(n, 0xD0C5)
    assert 1_600_000 < offs.size < 2_000_000
    o = O.Oracle(pats, match_kind=int(ac.match_kind()), ascii_case_insensitive=name == "cfg3", kind=O.KIND_DFA)
    values, _ = check(ac, d_hay, offs, mixed_reps(pats, 0xBE4C), o, name, n_sample=60)
    assert ac.last_stats()["engine"] == int(ab.Engine.Prefilter)
    assert values.numel() != n
    del d_hay, values
    torch.cuda.empty_cache()


def test_full_size_cfg5():
    """cfg 5's 100 000 patterns over 2 GiB cut into documents."""
    import torch
    n = 2 << 30
    pats, ac, d_hay = _config_batch("cfg5", n)
    assert ac.patterns_len() == 100_000
    offs = W.doc_offsets(n, 0xC5)
    check(ac, d_hay, offs, mixed_reps(pats, 5), O.Oracle(pats, kind=O.KIND_DFA), "cfg5", n_sample=30, host=False)
    del d_hay
    torch.cuda.empty_cache()


def test_one_4_gib_document_and_an_output_past_4_gib():
    """One 4 GiB document against the single-haystack records spliced in torch; then documents whose
    lengthening replacements take the output past 2^32."""
    import torch
    n = 4 << 30
    pats, ac, d_hay = _config_batch("cfg2", n)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    check(ac, d_hay, np.array([0, n]), mixed_reps(pats, 1), o, "one document", n_sample=1, host=False)
    del d_hay
    torch.cuda.empty_cache()
    m = 3 << 30
    pats, ac, d_hay = _config_batch("cfg2", m)
    offs = W.doc_offsets(m, 0x4AB)
    reps = [p + b"+" * 4096 for p in pats]
    values, _ = check(ac, d_hay, offs, reps, o, "past 4 GiB", n_sample=30, host=False)
    assert values.numel() > 1 << 32
    del d_hay, values
    torch.cuda.empty_cache()


@pytest.mark.parametrize("plen", [4096, 65536])
def test_long_patterns_at_document_edges(plen):
    """A 4 KiB or 64 KiB pattern, and a copy shifted by 3 bytes, planted across, at the end of and at the start
    of documents, replaced by something short and something long, on both engines."""
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
    reps = [b"<short>", base.tobytes() * 2, b""]
    for kind in (0, 1):
        ac = build(pats, kind)
        o = O.Oracle(pats, match_kind=kind, kind=O.KIND_DFA)
        values, out_offsets = check(ac, d_hay, offs, reps, o, (plen, kind), n_sample=20)
        ac.set_engine(ab.Engine.Sequential)
        v2, o2 = ac.replace_all_batch_torch((d_hay, offs), reps)
        assert torch.equal(v2, values) and torch.equal(o2, out_offsets), (plen, kind, "sequential")
