"""Lookahead of stream sets on the H100 (acg_streams_lookahead(_devout), Streams / ReplaceStreams.lookahead_*).

The reference is an independent walk of ac.tables() in torch (tests/lookahead_ref.py): each stream's tail -- its
last max_pattern_len - 1 bytes after its find_iter restart point, tracked here from the feeds' records -- gives a
state, and every candidate is walked from it.  Sampled pairs are also checked against the oracle over the stream's
whole history.  Covered: cfg 4 as a decode loop (4 096 streams, a 128 256-candidate vocabulary, 1 000 steps in both
modes, where every step's mask must predict which streams the step's feed returns a record for); cfg 2 and cfg 5
streams filled from documents, with a replace set beside the find_iter set; and a mask of 36 000 rows, past 4 GiB."""
import numpy as np
import pytest

import aho_corasick_b200 as ab
import oracle_py as O
from aho_corasick_b200 import workload as W
from lookahead_ref import TorchWalk, vocabulary

pytestmark = pytest.mark.gpu
N_VOCAB = 128256


class Tracker:
    """Per stream: position, find_iter restart point and the last `back` bytes; full histories of a few streams."""

    def __init__(self, n, back, overlapping, keep=()):
        self.n, self.back, self.overlapping = n, back, overlapping
        self.pos = np.zeros(n, np.int64)
        self.cursor = np.zeros(n, np.int64)
        self.last = [b""] * n
        self.full = {s: b"" for s in keep}

    def fed(self, chunks, rec):
        """After a feed of `chunks` (bytes per stream) that returned records `rec` (int64 [m, 3] on the host)."""
        for s, c in enumerate(chunks):
            if c:
                self.last[s] = (self.last[s] + c)[-self.back:] if self.back else b""
                self.pos[s] += len(c)
            if s in self.full:
                self.full[s] += c
        if not self.overlapping and len(rec):
            docs = rec[:, 0] >> 32
            tail = np.r_[docs[1:] != docs[:-1], True]
            self.cursor[docs[tail]] = rec[tail, 2]

    def tails(self, rows=None):
        out = []
        for s in (range(self.n) if rows is None else rows):
            k = int(min(self.back, self.pos[s] - self.cursor[s]))
            out.append(self.last[s][len(self.last[s]) - k:] if k else b"")
        return out


def oracle_pairs(o, tr, cands, got, rows, cols, overlapping):
    for s in rows:
        x = tr.full[s]
        for c in cols:
            h = np.frombuffer(x + cands[c], np.uint8).copy()
            r = o.find_overlapping_iter_np(h) if overlapping else o.find_iter_np(h)
            want = bool(len(r)) and int(r["end"].max()) > len(x)
            assert bool(got[s][c]) == want, ("oracle", s, cands[c])


def chunk_tensors(vocab_bytes, vocab_offs, tok):
    """(values, offsets) on the device: candidate tok[s] as stream s's chunk."""
    import torch
    lo = vocab_offs[tok]
    lens = vocab_offs[tok + 1] - lo
    offs = torch.zeros(tok.numel() + 1, dtype=torch.int64, device=tok.device)
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    if not total:
        return torch.empty(0, dtype=torch.uint8, device=tok.device), offs
    shift = torch.repeat_interleave(lo - offs[:-1], lens, output_size=total)
    return vocab_bytes[torch.arange(total, device=tok.device) + shift], offs


@pytest.mark.parametrize("overlapping", [False, True])
def test_decode_steps_cfg4(overlapping):
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    pats = W.config_patterns("cfg4")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    vocab = vocabulary(pats, N_VOCAB, 41)
    walk = TorchWalk(ac, vocab, dev)
    lens = np.fromiter(map(len, vocab), np.int64, count=len(vocab))
    vocab_offs = torch.from_numpy(np.r_[0, np.cumsum(lens)]).to(dev)
    vocab_bytes = torch.from_numpy(np.frombuffer(b"".join(vocab), np.uint8).copy()).to(dev)
    n = 4096
    rng = np.random.default_rng(7 + overlapping)
    # single bytes a quarter as likely as each longer token
    weights = np.where(np.arange(N_VOCAB) < 256, 1.0, 4.0)
    weights /= weights.sum()
    sample = [0, 1, 17, 1000, 4095]
    tr = Tracker(n, walk.back, overlapping, keep=sample)
    hits = 0
    with ac.streams(n, overlapping) as st, ac.candidates(vocab) as cs:
        for step in range(1000):
            mask = st.lookahead_torch(cs)
            tok_h = rng.choice(N_VOCAB, size=n, p=weights)
            tok = torch.from_numpy(tok_h).to(dev)
            bits = mask[torch.arange(n, device=dev), tok]
            if step % 50 == 0:
                want = walk.mask(walk.states(tr.tails()))
                assert torch.equal(mask, want), ("table walk", step, int((mask != want).sum()))
                cols = rng.choice(N_VOCAB, size=48, replace=False).tolist() + list(range(250, 256))
                oracle_pairs(o, tr, vocab, {s: mask[s].cpu().numpy() for s in sample}, sample, cols, overlapping)
            values, offs = chunk_tensors(vocab_bytes, vocab_offs, tok)
            got = st.feed_torch((values, offs))
            rec = got.records
            has = torch.zeros(n, dtype=torch.bool, device=dev)
            if rec.shape[0]:
                has[rec[:, 0] >> 32] = True
            assert torch.equal(has, bits), ("step", step, int((has != bits).sum()))
            hits += int(has.sum())
            tr.fed([vocab[t] for t in tok_h.tolist()], rec.cpu().numpy())
        assert np.array_equal(st.positions().astype(np.int64), tr.pos)
    assert hits > 1000


def fill_streams(ac, pats, name, n, rounds, seed, sets):
    """Feeds `rounds` rounds of document pieces of config `name` to every set of `sets` ((set, overlapping) pairs, the
    same chunks to each); returns a tracker per stream set, None for a replace set."""
    rng = np.random.default_rng(seed)
    hay = np.empty(n * 64 * rounds, np.uint8)
    W.make_config(name, hay.size, out=hay)
    trs = [None if isinstance(st, ab.ReplaceStreams) else
           Tracker(n, max(ac.max_pattern_len() - 1, 0), ov, keep=range(0, n, n // 8)) for st, ov in sets]
    at = 0
    for r in range(rounds):
        lens = rng.integers(0, 96, size=n)
        chunks = []
        for s in range(n):
            chunks.append(hay[at:at + lens[s]].tobytes())
            at = (at + int(lens[s])) % (hay.size - 128)
        for (st, ov), tr in zip(sets, trs):
            if tr is None:
                st.feed(chunks)
            else:
                h = st.feed_np(chunks)
                rec = np.stack([h["pid"].astype(np.int64) | (h["doc"].astype(np.int64) << 32),
                                h["start"].astype(np.int64), h["end"].astype(np.int64)], axis=1).reshape(-1, 3)
                tr.fed(chunks, rec)
    return trs


@pytest.mark.parametrize("name,rows", [("cfg2", None), ("cfg5", 512)])
def test_streams_from_documents(name, rows):
    """cfg 2 (5 000 patterns) in full and cfg 5 (100 000 patterns) on sampled rows, find_iter and overlapping sets;
    a replace set fed the same chunks gives the find_iter set's mask, in both output forms."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    pats = W.config_patterns(name)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    o = O.Oracle(pats, kind=O.KIND_DFA)
    vocab = vocabulary(pats, N_VOCAB, 43)
    walk = TorchWalk(ac, vocab, dev)
    n = 4096
    fi, ov = ac.streams(n), ac.streams(n, True)
    rp = ac.replace_streams(n, [b"*"] * len(pats))
    trs = fill_streams(ac, pats, name, n, 3, 5, [(fi, False), (ov, True), (rp, False)])
    with ac.candidates(vocab) as cs:
        ids = None if rows is None else np.random.default_rng(1).choice(n, size=rows, replace=False)
        for st, tr, overlapping in ((fi, trs[0], False), (ov, trs[1], True)):
            got = st.lookahead_torch(cs, ids)
            want = walk.mask(walk.states(tr.tails(ids)))
            assert torch.equal(got, want), (name, overlapping, int((got != want).sum()))
            assert ac.last_stats()["launches"] == 7
            keep = sorted(tr.full)
            full = st.lookahead_np(cs, keep)
            oracle_pairs(o, tr, vocab, dict(zip(keep, full)), keep, list(range(0, N_VOCAB, 2500)), overlapping)
        m_fi = fi.lookahead_torch(cs)
        assert torch.equal(rp.lookahead_torch(cs), m_fi)
        assert np.array_equal(rp.lookahead_np(cs, [5, 5, 3]), m_fi[[5, 5, 3]].cpu().numpy())
        assert np.array_equal(ov.positions(), trs[1].pos.astype(np.uint64))
    for s in (fi, ov, rp):
        s.close()


def test_mask_past_4_gib():
    """36 000 rows x 128 256 candidates = 4.6 GB of mask: the last rows (byte offsets past 2^32) and the first ones
    equal the table walk."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    pats = W.config_patterns("cfg4")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    vocab = vocabulary(pats, N_VOCAB, 47)
    walk = TorchWalk(ac, vocab, dev)
    n = 36000
    assert n * N_VOCAB > (1 << 32)
    rng = np.random.default_rng(3)
    hay = np.empty(n * 24, np.uint8)
    W.make_config("cfg4", hay.size, out=hay)
    lens = rng.integers(0, 24, size=n)
    chunks = [hay[24 * s:24 * s + lens[s]].tobytes() for s in range(n)]
    with ac.streams(n, True) as st, ac.candidates(vocab) as cs:
        st.feed(chunks)
        tr = Tracker(n, walk.back, True)
        tr.fed(chunks, np.zeros((0, 3), np.int64))
        got = st.lookahead_torch(cs)
        for rows in (list(range(n - 300, n)), list(range(200))):
            want = walk.mask(walk.states(tr.tails(rows)))
            assert torch.equal(got[rows], want), (rows[0], int((got[rows] != want).sum()))
        del got
