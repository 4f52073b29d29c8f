#!/usr/bin/env python3
"""Lookahead of stream sets (acg_streams_lookahead_devout through Streams.lookahead_torch) on two workloads.

    python tools/bench_lookahead.py [--workload decode|cfg2|both] [--calls 1000] [--warmup 20]

decode: cfg 4 (50 patterns), 4 096 streams in find_iter mode, a seeded 128 256-candidate vocabulary
        (tests/lookahead_ref.py).  Every step takes the mask and then feeds each stream a token drawn from the
        vocabulary, so the streams' states move as in a decode loop; only the lookahead call is timed.
cfg2:   cfg 2 (5 000 patterns), 4 096 find_iter streams filled with three rounds of document pieces, the same
        vocabulary; the same set is asked again and again.

Reported per workload:
- the card's name, power limit and SM clock, read in the same run;
- the wall time per call, median and p90: the host clock around a call, which ends in a device synchronise;
- the device time per call from the library's CUDA events (acg_last_stats: scan_ms is the mask kernel, order_ms the
  state walk, the dedupe and the copy of shared rows);
- U, the distinct tail states per call (the rows the mask kernel walks), from the torch reference's states;
- the per-kernel split from torch.profiler over 50 calls, in a run of its own;
- the mask's write rate (its bytes over the device time) against a torch.zeros of the same size timed with CUDA
  events in the same run;
- the torch table walk (tests/lookahead_ref.py) on the same states, timed with CUDA events on 10 calls, and whether
  its masks equal the library's.
Prints one JSON line per workload."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.dont_write_bytecode = True

N_STREAMS = 4096
N_VOCAB = 128256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    f = (q[0].split(", ") + ["?"] * 4)[:4] if q else ["?"] * 4
    return {"name": f[0], "power_limit": f[1], "sm_clock": f[2], "sm_clock_max": f[3]}


def tails(st_pos, cursor, last, back):
    out = []
    for s in range(len(last)):
        k = int(min(back, st_pos[s] - cursor[s]))
        out.append(last[s][len(last[s]) - k:] if k else b"")
    return out


def events_ms(fn, reps):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def run(workload, calls, warmup):
    import torch
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W
    from lookahead_ref import TorchWalk, vocabulary
    dev = torch.device("cuda", torch.cuda.current_device())
    name = "cfg4" if workload == "decode" else "cfg2"
    pats = W.config_patterns(name)
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    vocab = vocabulary(pats, N_VOCAB, 41)
    walk = TorchWalk(ac, vocab, dev)
    back = walk.back
    st = ac.streams(N_STREAMS)
    cs = ac.candidates(vocab)
    rng = np.random.default_rng(11)
    pos = np.zeros(N_STREAMS, np.int64)
    cursor = np.zeros(N_STREAMS, np.int64)
    last = [b""] * N_STREAMS

    def feed(chunks):
        h = st.feed_np(chunks)
        for s, c in enumerate(chunks):
            if c:
                last[s] = (last[s] + c)[-back:] if back else b""
                pos[s] += len(c)
        if len(h):
            docs = h["doc"].astype(np.int64)
            end = np.r_[docs[1:] != docs[:-1], True]
            cursor[docs[end]] = h["end"][end].astype(np.int64)

    if workload == "cfg2":
        hay = np.empty(N_STREAMS * 64 * 3, np.uint8)
        W.make_config("cfg2", hay.size, out=hay)
        at = 0
        for _ in range(3):
            lens = rng.integers(0, 96, size=N_STREAMS)
            chunks = []
            for s in range(N_STREAMS):
                chunks.append(hay[at:at + lens[s]].tobytes())
                at = (at + int(lens[s])) % (hay.size - 128)
            feed(chunks)

    def step():
        if workload == "decode":
            feed([vocab[t] for t in rng.integers(0, N_VOCAB, size=N_STREAMS).tolist()])

    for _ in range(warmup):
        st.lookahead_torch(cs)
        step()
    wall, dev_ms, scan_ms, uniq = [], [], [], []
    checks = []
    for i in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = st.lookahead_torch(cs)
        wall.append((time.perf_counter() - t0) * 1e3)
        s = ac.last_stats()
        dev_ms.append(s["scan_ms"] + s["order_ms"])
        scan_ms.append(s["scan_ms"])
        states = walk.states(tails(pos, cursor, last, back))
        uniq.append(int(torch.unique(states).numel()))
        if i % max(1, calls // 10) == 0:  # the torch baseline on the same states, and the two masks compared
            ref = None

            def base():
                nonlocal ref
                ref = walk.mask(states)
            checks.append((events_ms(base, 1), bool(torch.equal(ref, m))))
            del ref
        del m
        step()
    mask_bytes = N_STREAMS * N_VOCAB
    zeros_ms = events_ms(lambda: torch.zeros(mask_bytes, dtype=torch.uint8, device=dev), 20)
    # per-kernel split, a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            st.lookahead_torch(cs)
            step()
        torch.cuda.synchronize()
    split = {}
    for e in prof.events():
        if e.device_type.name != "CUDA" or "memcpy" in e.name.lower() or "memset" in e.name.lower():
            continue
        if not any(k in e.name for k in ("look_", "Radix", "Scan", "radix", "scan")):
            continue
        key = next((k for k in ("look_state", "look_heads", "look_compact", "look_mask", "look_copy") if k in e.name),
                   "cub " + ("sort" if "adix" in e.name else "scan"))
        split[key] = split.get(key, 0.0) + e.device_time_total / 1000.0 / 50
    med = float(np.median(dev_ms))
    out = {
        "workload": workload, "card": card(), "streams": N_STREAMS, "candidates": N_VOCAB, "calls": calls,
        "wall_ms_median": float(np.median(wall)), "wall_ms_p90": float(np.percentile(wall, 90)),
        "device_ms_median": med, "device_ms_p90": float(np.percentile(dev_ms, 90)),
        "mask_kernel_ms_median": float(np.median(scan_ms)),
        "U_median": float(np.median(uniq)), "U_min": int(np.min(uniq)), "U_max": int(np.max(uniq)),
        "kernel_ms_per_call": {k: round(v, 4) for k, v in sorted(split.items())},
        "mask_GBps": mask_bytes / (med * 1e-3) / 1e9, "torch_zeros_GBps": mask_bytes / (zeros_ms * 1e-3) / 1e9,
        "torch_walk_ms_median": float(np.median([c[0] for c in checks])),
        "torch_walk_equal": all(c[1] for c in checks), "torch_walk_checks": len(checks),
    }
    st.close()
    cs.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="both", choices=["decode", "cfg2", "both"])
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_lookahead.py needs a CUDA device")
    for w in (["decode", "cfg2"] if a.workload == "both" else [a.workload]):
        print(json.dumps(run(w, a.calls, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
