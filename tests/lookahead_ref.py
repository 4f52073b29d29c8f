"""Helpers of the lookahead checks on the GPU (tests/test_gpu_lookahead.py, tools/bench_lookahead.py): a seeded
synthetic vocabulary, and the lookahead computed in torch by walking the tables of AhoCorasick.tables() -- what a
caller without acg_streams_lookahead would write, and an independent reference for it."""
import numpy as np

from aho_corasick_b200 import workload as W

MAX_TOKEN = 64


def vocabulary(patterns, n, seed):
    """n byte strings, 0 to MAX_TOKEN bytes: every single byte first, then pieces of the patterns (prefixes, suffixes,
    infixes, whole ones with text around them) and of workload text, with a few empty ones."""
    rng = np.random.default_rng(seed)
    text = np.empty(1 << 20, np.uint8)
    W.fill_haystack(text, seed)
    text = text.tobytes()
    out = [bytes([b]) for b in range(256)]
    while len(out) < n:
        r = rng.random()
        p = patterns[int(rng.integers(0, len(patterns)))]
        k = int(rng.integers(1, len(p) + 1))
        if r < 0.01:
            out.append(b"")
        elif r < 0.2:
            out.append(p[:k])
        elif r < 0.4:
            out.append(p[-k:])
        elif r < 0.5:
            i = int(rng.integers(0, len(p)))
            out.append(p[i:i + k])
        elif r < 0.6:
            a = int(rng.integers(0, 8))
            i = int(rng.integers(0, len(text) - 64))
            out.append((text[i:i + a] + p + text[i + a:i + 2 * a])[:MAX_TOKEN])
        else:
            i = int(rng.integers(0, len(text) - 64))
            out.append(text[i:i + int(rng.integers(1, 17 if r < 0.95 else MAX_TOKEN + 1))])
    return out[:n]


class TorchWalk:
    """The lookahead by table walk in torch on `device`: the candidates as class ids padded to the longest one."""

    def __init__(self, ac, cands, device):
        import torch
        t = ac.tables()
        self.device = device
        self.trans = torch.from_numpy(t["trans"].astype(np.int64)).to(device)
        self.classes = torch.from_numpy(t["byte_classes"].astype(np.int64)).to(device)
        self.start = int(t["start_unanchored_id"])
        self.max_match = int(t["max_match_id"])
        self.back = max(int(t["max_pattern_len"]) - 1, 0)
        width = max(1, max(map(len, cands)))
        pad = np.zeros((len(cands), width), np.uint8)
        lens = np.zeros(len(cands), np.int64)
        for i, c in enumerate(cands):
            pad[i, :len(c)] = np.frombuffer(c, np.uint8)
            lens[i] = len(c)
        self.cls = self.classes[torch.from_numpy(pad).to(device).long()]
        self.lens = torch.from_numpy(lens).to(device)
        self.width = width

    def states(self, tails):
        """The state after walking each tail (bytes) from the unanchored start state: int64 [len(tails)]."""
        import torch
        width = max([1] + [len(t) for t in tails])
        pad = np.zeros((len(tails), width), np.uint8)
        lens = np.zeros(len(tails), np.int64)
        for i, t in enumerate(tails):
            pad[i, :len(t)] = np.frombuffer(t, np.uint8)
            lens[i] = len(t)
        cls = self.classes[torch.from_numpy(pad).to(self.device).long()]
        n = torch.from_numpy(lens).to(self.device)
        s = torch.full((len(tails),), self.start, dtype=torch.int64, device=self.device)
        for j in range(width):
            s = torch.where(j < n, self.trans[s + cls[:, j]], s)
        return s

    def mask(self, states, block=256):
        """bool [len(states), n_cands]: a walk from each state over every candidate enters a match state."""
        import torch
        out = torch.empty((states.numel(), self.lens.numel()), dtype=torch.bool, device=self.device)
        for b0 in range(0, states.numel(), block):
            s = states[b0:b0 + block, None].expand(-1, self.lens.numel()).contiguous()
            hit = torch.zeros_like(s, dtype=torch.bool)
            for j in range(self.width):
                live = (j < self.lens)[None, :]
                s = torch.where(live, self.trans[s + self.cls[None, :, j]], s)
                hit |= live & (s != 0) & (s <= self.max_match)
            out[b0:b0 + block] = hit
        return out
