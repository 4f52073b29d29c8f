"""Deterministic synthetic inputs for the BASELINE configs (SURVEY.md section 8d).

Counter-based SplitMix64: every 8-byte word of the haystack is a pure function of
(seed, word index), so any rank can reproduce any slice of a 32 GiB haystack without
generating what precedes it.  Bench/test glue -- not part of the search path.
"""
from __future__ import annotations

import numpy as np

_M = np.uint64(0xFFFFFFFFFFFFFFFF)
_G = np.uint64(0x9E3779B97F4A7C15)


def _mix(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = x + _G
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _words(seed: int, first_word: int, n_words: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        idx = np.arange(first_word, first_word + n_words, dtype=np.uint64)
        return _mix(np.uint64(seed) + idx * _G)


def make_patterns(n: int, seed: int, lo: int = 4, hi: int = 16, alphabet=(0x20, 0x7E)):
    """n patterns, length uniform in [lo, hi], bytes uniform in the alphabet range; duplicates kept."""
    a0, a1 = alphabet
    span = a1 - a0 + 1
    r = _words(seed, 0, n * (hi + 1))
    pats = []
    for i in range(n):
        base = i * (hi + 1)
        ln = lo + int(r[base] % np.uint64(hi - lo + 1))
        body = (a0 + (r[base + 1: base + 1 + ln] >> np.uint64(11)) % np.uint64(span)).astype(np.uint8)
        pats.append(body.tobytes())
    return pats


def fill_haystack(out: np.ndarray, seed: int, global_offset: int = 0, alphabet=(0x20, 0x7E),
                  chunk: int = 1 << 26):
    """Fill `out` (uint8) with the bytes [global_offset, global_offset+len(out)) of the stream."""
    assert out.dtype == np.uint8 and global_offset % 8 == 0
    lut = _alphabet_lut(alphabet)
    n = out.size
    pos = 0
    while pos < n:
        m = min(chunk, n - pos)
        nw = (m + 7) // 8
        w = _words(seed, (global_offset + pos) // 8, nw)
        np.take(lut, w.view(np.uint8)[:m], out=out[pos:pos + m])
        pos += m
    return out


def _alphabet_lut(alphabet):
    """uniform byte -> alphabet byte: a0 + (b * span >> 8)."""
    a0, a1 = alphabet
    span = a1 - a0 + 1
    return (a0 + ((np.arange(256, dtype=np.uint32) * span) >> 8)).astype(np.uint8)


def plant(out: np.ndarray, patterns, seed: int, global_offset: int = 0, period: int = 4096,
          window: int = 2048):
    """Plant a pseudo-randomly chosen pattern at every offset k*period + (r % window) that falls
    entirely inside this slice (plants never overlap: max pattern length << period - window)."""
    n = out.size
    k0 = global_offset // period
    k1 = (global_offset + n + period - 1) // period
    ks = np.arange(k0, k1, dtype=np.uint64)
    r = _mix(np.uint64(seed) ^ (ks * _G))
    offs = (ks * np.uint64(period) + (r % np.uint64(window))).astype(np.int64) - global_offset
    pid = ((r >> np.uint64(32)) % np.uint64(len(patterns))).astype(np.int64)
    lens = np.array([len(p) for p in patterns], dtype=np.int64)
    maxlen = int(lens.max())
    table = np.zeros((len(patterns), maxlen), dtype=np.uint8)
    for i, p in enumerate(patterns):
        table[i, :len(p)] = np.frombuffer(p, dtype=np.uint8)
    ok = (offs >= 0) & (offs + lens[pid] <= n)
    offs, pid = offs[ok], pid[ok]
    for L in np.unique(lens[pid]):
        sel = lens[pid] == L
        o, p = offs[sel], pid[sel]
        idx = o[:, None] + np.arange(L)[None, :]
        out[idx] = table[p, :L]
    return int(ok.sum())


def flip_case(out: np.ndarray, seed: int, global_offset: int = 0, chunk: int = 1 << 26):
    """Flip the ASCII case of each letter with probability 1/2 (config 3)."""
    n = out.size
    pos = 0
    while pos < n:
        m = min(chunk, n - pos)
        nw = (m + 7) // 8
        w = _words(seed, (global_offset + pos) // 8, nw).view(np.uint8)[:m]
        v = out[pos:pos + m]
        is_alpha = ((v | 0x20) >= ord("a")) & ((v | 0x20) <= ord("z"))
        flip = is_alpha & ((w & 1) == 1)
        out[pos:pos + m] = np.where(flip, v ^ 0x20, v)
        pos += m
    return out


CONFIGS = {
    # BASELINE config 1's automaton (README example; the reference gives it a start-bytes prefilter: a, m, S)
    # over a synthetic haystack: the byte-set scan's workload
    "cfg1": dict(patterns=[b"apple", b"maple", b"Snapple"], n_patterns=3, pattern_seed=0, hay_seed=0xAC4611,
                 alphabet=(0x20, 0x7E)),
    # three capitalised words in lower-case text: the reference gives this automaton a start-bytes
    # prefilter (memchr for 'Q') and the needle is as rare as that heuristic hopes -- the byte-set scan's workload
    "cfg1s": dict(patterns=[b"Quartz", b"Quebec", b"Quixote"], n_patterns=3, pattern_seed=0, hay_seed=0xAC4611,
                  alphabet=(0x61, 0x7A)),
    # name: (n_patterns, pattern_seed, haystack_seed, alphabet)
    "cfg2": dict(n_patterns=5000, pattern_seed=0xAC5000, hay_seed=0xAC4611, alphabet=(0x20, 0x7E)),
    "cfg2b": dict(n_patterns=5000, pattern_seed=0xAC5000, hay_seed=0xAC4611, alphabet=(0x61, 0x7A)),
    "cfg3": dict(n_patterns=5000, pattern_seed=0xAC5000, hay_seed=0xAC4611, alphabet=(0x20, 0x7E),
                 case_seed=0xAC3C45),
    "cfg4": dict(n_patterns=50, pattern_seed=0xAC0050, hay_seed=0xAC4611, alphabet=(0x20, 0x7E)),
    "cfg5": dict(n_patterns=100000, pattern_seed=0xAC1000, hay_seed=0xAC4611, alphabet=(0x20, 0x7E)),
}


def doc_offsets(n_bytes: int, seed: int, lo: int = 16, hi: int = 16384) -> np.ndarray:
    """CSR bounds (int64, [n_docs + 1]) cutting [0, n_bytes) into documents whose lengths are log-uniform
    in [lo, hi] (the last one is cut short); mean (hi - lo) / ln(hi / lo), about 2.3 KiB by default."""
    rng = np.random.default_rng(seed)
    mean = (hi - lo) / np.log(hi / lo)
    lens = np.exp(rng.uniform(np.log(lo), np.log(hi + 1), size=int(n_bytes / mean * 1.1) + 16)).astype(np.int64)
    ends = np.cumsum(lens)
    while ends[-1] < n_bytes:  # (not reached for sizes above a few MiB)
        more = np.exp(rng.uniform(np.log(lo), np.log(hi + 1), size=1024)).astype(np.int64)
        ends = np.concatenate([ends, ends[-1] + np.cumsum(more)])
    k = int(np.searchsorted(ends, n_bytes))
    return np.concatenate([[0], ends[:k], [n_bytes]]).astype(np.int64)


def config_patterns(name: str):
    """The pattern set of a named configuration."""
    c = CONFIGS[name]
    if "patterns" in c:
        return list(c["patterns"])
    return make_patterns(c["n_patterns"], c["pattern_seed"], alphabet=c["alphabet"])


def make_config(name: str, hay_bytes: int, out: np.ndarray | None = None, global_offset: int = 0):
    c = CONFIGS[name]
    pats = config_patterns(name)
    if out is None:
        out = np.empty(hay_bytes, dtype=np.uint8)
    fill_haystack(out, c["hay_seed"], global_offset, alphabet=c["alphabet"])
    planted = plant(out, pats, c["hay_seed"] ^ 0x5EED, global_offset)
    if "case_seed" in c:
        flip_case(out, c["case_seed"], global_offset)
    return pats, out, planted


# ---- the same streams generated on the GPU with torch (bench: 4 GiB in well under a second) ----
def _t_mix(x):
    import torch
    def lsr(v, k):
        return (v >> k) & ((1 << (64 - k)) - 1)
    G = -7046029254386353131          # 0x9E3779B97F4A7C15 as int64
    z = x + G
    z = (z ^ lsr(z, 30)) * -4658895280553007687   # 0xBF58476D1CE4E5B9
    z = (z ^ lsr(z, 27)) * -7723592293110705685   # 0x94D049BB133111EB
    return z ^ lsr(z, 31)


def _to_i64(v: int) -> int:
    v &= 0xFFFFFFFFFFFFFFFF
    return v - (1 << 64) if v >= (1 << 63) else v


def torch_fill_config(name: str, out, patterns, global_offset: int = 0, chunk: int = 1 << 28):
    """Fill the CUDA uint8 tensor `out` with the same bytes make_config() produces on the host."""
    import torch
    c = CONFIGS[name]
    dev = out.device
    n = out.numel()
    assert global_offset % 8 == 0 and n % 8 == 0
    G = -7046029254386353131
    lut = torch.from_numpy(_alphabet_lut(c["alphabet"])).to(dev)
    pos = 0
    while pos < n:
        m = min(chunk, n - pos)
        idx = torch.arange((global_offset + pos) // 8, (global_offset + pos + m) // 8, dtype=torch.int64, device=dev)
        w = _t_mix(_to_i64(c["hay_seed"]) + idx * G)
        out[pos:pos + m] = lut[w.view(torch.uint8).long()]
        pos += m
        del idx, w
    # plants
    period, window = 4096, 2048
    k0 = global_offset // period
    k1 = (global_offset + n + period - 1) // period
    ks = torch.arange(k0, k1, dtype=torch.int64, device=dev)
    r = _t_mix(_to_i64(c["hay_seed"] ^ 0x5EED) ^ (ks * G))
    offs = ks * period + (r & (window - 1)) - global_offset
    hi32 = (r >> 32) & 0xFFFFFFFF
    pid = hi32 % len(patterns)
    lens_np = np.array([len(p) for p in patterns], dtype=np.int64)
    maxlen = int(lens_np.max())
    table_np = np.zeros((len(patterns), maxlen), dtype=np.uint8)
    for i, p in enumerate(patterns):
        table_np[i, :len(p)] = np.frombuffer(p, dtype=np.uint8)
    lens = torch.from_numpy(lens_np).to(dev)
    table = torch.from_numpy(table_np).to(dev)
    pl = lens[pid]
    ok = (offs >= 0) & (offs + pl <= n)
    offs, pid, pl = offs[ok], pid[ok], pl[ok]
    ar = torch.arange(maxlen, device=dev)
    mask = ar[None, :] < pl[:, None]
    idx = (offs[:, None] + ar[None, :])[mask]
    out[idx] = table[pid][mask]
    if "case_seed" in c:
        pos = 0
        while pos < n:
            m = min(chunk, n - pos)
            idx = torch.arange((global_offset + pos) // 8, (global_offset + pos + m) // 8, dtype=torch.int64, device=dev)
            w = _t_mix(_to_i64(c["case_seed"]) + idx * G).view(torch.uint8)
            v = out[pos:pos + m]
            low = v | 0x20
            flip = (low >= ord("a")) & (low <= ord("z")) & ((w & 1) == 1)
            out[pos:pos + m] = torch.where(flip, v ^ 0x20, v)
            pos += m
            del idx, w
    return int(ok.sum().item())
